"""GPU tests of the vertex normals and the hard Phong pass (csrc/shade.cu, recmv_b200.raster.vertex_normals /
shade_meshes, the HardPhongShader / SoftSilhouetteShader of compat/MaskRender.py) against the float64 oracle
(oracle/shade_oracle.py).  The oracle shades the GPU's own fragments, so the comparison does not depend on the
rasterizer's coverage decisions (tested in tests/test_gpu_raster.py).

Bounds are about 3x the maxima measured on an H100 80GB HBM3 and are printed with the measured values:
NORMAL_ANGLE (radians, vertex normals of the deformed 257^3 marching-cubes mesh against float64), RGB_TOL (absolute,
shaded colours against float64 shading of the same fragments with float64 normals; shininess 64 amplifies the fp32
error of R . V near a highlight)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import shade_oracle as so
from recmv_b200 import _lib, ops, synth
from recmv_b200.model import LBSkinner
from recmv_b200.raster import Fragments, rasterize_meshes, shade_meshes, vertex_normals

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

NORMAL_ANGLE = 6e-7      # measured 2.0e-7
FAN_ANGLE = 3.5e-6       # measured 1.2e-6 (1e5 faces summed on one vertex)
RGB_TOL = 2.5e-5         # measured 8.0e-6
SILHOUETTE_TOL = 2e-7    # measured 6.4e-8


def _skinner():
    Js, parents, init = synth.skeleton()
    ws = synth.skinning_voxel((17, 33, 21), seed=7)
    return LBSkinner(ws, [-1.1] * 3, [1.1] * 3, Js, parents, init_pose=init,
                     bbox_extend=torch.tensor(synth.BBOX_EXTEND), bbox_center=torch.tensor(synth.BBOX_CENTER)).to(DEV)


@pytest.fixture(scope="module")
def mesh():
    sdf = synth.sphere_sdf_grid(257, num=8, seed=3, device=DEV)
    h = 2.0 / 256
    verts, faces = ops.mc_gpu(sdf, h, h, h, -1.0, -1.0, -1.0, 0.0)
    return verts, faces


def deform(verts, N, seed):
    sk = _skinner()
    poses, trans = synth.poses_trans(N, seed=seed)
    V = verts.shape[0]
    with torch.no_grad():
        d = sk(verts.repeat(N, 1), [poses.to(DEV), trans.to(DEV)], torch.arange(N, device=DEV).repeat_interleave(V))
    return d.view(N, V, 3).contiguous()


class _Cams:
    """The attributes of the reference's RectifiedPerspectiveCameras the renderer reads."""

    def __init__(self, rows):
        self.focal_length, self.principal_point = rows[:, 0:2], rows[:, 2:4]
        self.R, self.T = rows[:, 4:13].reshape(-1, 3, 3), rows[:, 13:16]


def cameras(N, H, W, seed):
    """A camera per frame in the reference's convention (R close to diag(-1, -1, 1), the body ~2.6 in front)."""
    g = np.random.default_rng(seed)
    rows = []
    for n in range(N):
        a = g.normal(size=3) * 0.15
        K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        Q = np.linalg.qr(np.eye(3) + K)[0]
        Q = Q * np.sign(np.diag(Q))
        R = np.diag([-1.0, -1.0, 1.0]) @ Q
        f = 0.9 * min(H, W) * (1 + 0.1 * n)
        T = np.array([0.02 * n, -0.03, 2.6 + 0.1 * n])
        rows.append(np.concatenate([[f, f * 1.02, W / 2 - 0.5 + n, H / 2 - 0.5 - n], R.reshape(-1), T]))
    return torch.tensor(np.stack(rows), dtype=torch.float32, device=DEV)


def centre(cam):
    c = cam.double().cpu().numpy()
    return -np.einsum("nij,nj->ni", c[:, 4:13].reshape(-1, 3, 3), c[:, 13:16])


def angle(a, b):
    """Angle between the rows of a and b (0 where both are 0)."""
    a, b = a.reshape(-1, 3), b.reshape(-1, 3)
    return np.arctan2(np.linalg.norm(np.cross(a, b), axis=1), np.sum(a * b, axis=1))


class _Lights:
    def __init__(self, location, ambient=(0.5,) * 3, diffuse=(0.3,) * 3, specular=(0.2,) * 3):
        self.location = torch.as_tensor(location, dtype=torch.float32).reshape(-1, 3)
        self.ambient_color, self.diffuse_color, self.specular_color = (
            torch.as_tensor(x, dtype=torch.float32).reshape(-1, 3) for x in (ambient, diffuse, specular))


# ---- vertex normals -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("N", [1, 3])
def test_normals_against_oracle(mesh, N):
    verts, faces = mesh
    d = deform(verts, N, 20 + N)
    n = vertex_normals(d, faces)
    ref = so.vertex_normals(d.double().cpu().numpy(), faces.cpu().numpy())
    got = n.double().cpu().numpy()
    err = angle(got, ref).max()
    refn = np.linalg.norm(ref, axis=-1)
    print(f"[normals N={N}] V={d.shape[1]} F={faces.shape[0]} max angle to float64 {err:.2e} rad "
          f"(bound {NORMAL_ANGLE:.0e}); |n| - 1 max {np.abs(np.linalg.norm(got, axis=-1) - 1)[refn > 0.5].max():.2e}")
    assert err < NORMAL_ANGLE
    assert np.all(got[refn == 0] == 0)
    assert torch.equal(n, vertex_normals(d, faces))                       # bit-identical across calls
    for k in range(N):                                                    # N frames = N one-frame calls
        assert torch.equal(n[k:k + 1], vertex_normals(d[k:k + 1].contiguous(), faces))


def test_normals_unreferenced_zero_area_and_out_of_range_faces():
    g = np.random.default_rng(5)
    V = 40
    v = torch.tensor(g.normal(size=(2, V, 3)), dtype=torch.float32, device=DEV)
    v[:, 30] = v[:, 31]                                                   # coincident vertices: a zero-area face
    faces = [[0, 1, 2], [2, 1, 3], [3, 4, 5], [30, 31, 6], [7, 7, 8], [9, 10, 11], [12, 13, 14],
             [0, 1, V], [-1, 4, 5], [3, 1 << 40, 2], [15, 16, 17]]          # three faces with an index out of range
    f = torch.tensor(faces, dtype=torch.int64, device=DEV)
    n = vertex_normals(v, f).cpu().numpy()
    ref = so.vertex_normals(v.double().cpu().numpy(), faces)
    used = np.zeros(V, bool)
    used[np.array([x for x in faces if all(0 <= i < V for i in x)]).reshape(-1)] = True
    assert np.all(n[:, ~used] == 0) and np.all(ref[:, ~used] == 0)        # unreferenced (and only out-of-range) vertices
    assert np.all(n[:, 8] == 0) and np.all(n[:, 7] == 0)                  # (7, 7, 8) has zero area
    assert np.abs(n - ref).max() < 1e-5


def test_normals_fan_of_1e5_faces_around_one_vertex():
    K = 100_000
    th = np.linspace(0, 2 * np.pi, K, endpoint=False)
    ring = np.stack([np.cos(th), np.sin(th), 0.1 * np.sin(7 * th)], 1)
    v = torch.tensor(np.concatenate([[[0.0, 0.0, 0.3]], ring])[None], dtype=torch.float32, device=DEV)
    i = np.arange(K)
    f = torch.tensor(np.stack([np.zeros(K, np.int64), 1 + i, 1 + (i + 1) % K], 1), device=DEV)
    vertex_normals(v, f)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    n = vertex_normals(v, f)
    b.record()
    b.synchronize()
    ref = so.vertex_normals(v.double().cpu().numpy(), f.cpu().numpy())
    err = angle(n.double().cpu().numpy(), ref)
    print(f"[normals fan] {K} faces on one vertex: {a.elapsed_time(b):.3f} ms, centre angle {err[0]:.2e}, "
          f"max angle {err.max():.2e} rad (bound {FAN_ANGLE:.0e})")
    assert err.max() < FAN_ANGLE
    assert torch.equal(n, vertex_normals(v, f))


# ---- Phong ----------------------------------------------------------------------------------------------------------

def oracle_phong(fr, d, faces, cam, colors, lights, background=(1.0, 1.0, 1.0)):
    nrm = so.vertex_normals(d.double().cpu().numpy(), faces.cpu().numpy())
    return so.phong(fr.pix_to_face[..., 0].cpu().numpy(), fr.bary_coords[..., 0, :].double().cpu().numpy(),
                    d.double().cpu().numpy(), nrm, None if colors is None else colors.double().cpu().numpy(),
                    faces.cpu().numpy(), centre(cam), lights.location.double().numpy(),
                    lights.ambient_color.double().numpy(), lights.diffuse_color.double().numpy(),
                    lights.specular_color.double().numpy(), background=background)


def check_image(img, ref, fr, background, label):
    img = img.cpu()
    bg = fr.pix_to_face[..., 0].cpu() < 0
    err = float((img.double() - torch.from_numpy(ref)).abs().max())
    worst = np.unravel_index(int((img.double() - torch.from_numpy(ref)).abs().amax(-1).argmax()), img.shape[:3])
    print(f"[phong {label}] {tuple(img.shape)} covered={int((~bg).sum())} max |rgb - f64| {err:.2e} "
          f"(bound {RGB_TOL:.0e}) at {tuple(int(x) for x in worst)} f64 {ref[worst][:3]}; f64 rgb max {ref[..., :3].max():.3f}")
    assert err < RGB_TOL
    assert torch.equal(img[bg][:, :3], torch.tensor(background, dtype=torch.float32).expand(int(bg.sum()), 3))
    assert bool((img[..., 3] == 1).all())


@pytest.mark.parametrize("H,W", [(1080, 1080), (333, 517)])
def test_phong_against_oracle(mesh, H, W):
    verts, faces = mesh
    d = deform(verts, 1, 30)
    cam = cameras(1, H, W, 30)
    fr = rasterize_meshes(d, faces, _Cams(cam), (H, W))
    colors = torch.rand((1, d.shape[1], 3), generator=synth.generator(4)).to(DEV)
    lights = _Lights([[0.4, -0.8, -1.5]])                 # between the camera and the body: highlights in view
    bgc = (0.25, 0.5, 0.75)
    img = shade_meshes(d, faces, fr, _Cams(cam), colors=colors, lights=lights, background=bgc)
    check_image(img, oracle_phong(fr, d, faces, cam, colors, lights, bgc), fr, bgc, f"{H}x{W}")
    assert torch.equal(img, shade_meshes(d, faces, fr, _Cams(cam), colors=colors, lights=lights, background=bgc))


def test_phong_per_frame_cameras_lights_and_broadcast(mesh):
    verts, faces = mesh
    N, H, W = 3, 400, 360
    d = deform(verts, N, 31)
    cam = cameras(N, H, W, 31)
    fr = rasterize_meshes(d, faces, _Cams(cam), (H, W))
    lights = _Lights([[0.4, -0.8, -1.5], [-0.5, 0.2, -2.0], [0.0, 1.0, 0.0]], ambient=[[0.5] * 3, [0.4] * 3, [0.2] * 3],
                     diffuse=[[0.3] * 3, [0.5, 0.4, 0.3], [0.6] * 3], specular=[[0.2] * 3, [0.3] * 3, [0.1, 0.2, 0.3]])
    img = shade_meshes(d, faces, fr, _Cams(cam), lights=lights)
    check_image(img, oracle_phong(fr, d, faces, cam, None, lights), fr, (1.0, 1.0, 1.0), f"N={N} per-frame")
    # one broadcast row (camera, lights, materials, colours) = N equal rows, bit for bit
    one = _Lights([[0.4, -0.8, -1.5]])
    rep = _Lights([[0.4, -0.8, -1.5]] * N, ambient=[[0.5] * 3] * N, diffuse=[[0.3] * 3] * N, specular=[[0.2] * 3] * N)
    col = torch.rand((1, d.shape[1], 3), generator=synth.generator(6)).to(DEV)
    a = shade_meshes(d, faces, fr, _Cams(cam[:1]), colors=col, lights=one)
    b = shade_meshes(d, faces, fr, _Cams(cam[:1].expand(N, 16).contiguous()), colors=col.expand(N, -1, -1).contiguous(),
                     lights=rep)
    assert torch.equal(a, b)


class _Meshes:
    def __init__(self, verts, faces, textures=None):
        self._v, self._f, self.textures = verts, faces, textures

    def verts_padded(self):
        return self._v

    def faces_list(self):
        return [self._f] * self._v.shape[0]


def test_shader_camera_is_the_shaders_own_unless_passed(mesh):
    from recmv_b200.compat.MaskRender import HardPhongShader, mask_renderer
    verts, faces = mesh
    N, H, W = 2, 300, 400
    d = deform(verts, N, 32)
    cam_r, cam_s, cam_k = cameras(N, H, W, 32), cameras(N, H, W, 33), cameras(N, H, W, 34)
    ren = mask_renderer((H, W))
    ren.shader = HardPhongShader(DEV, _Cams(cam_s))                     # infer_fl.py:167
    ren.rasterizer.cameras = _Cams(cam_r)                               # infer_garment reassigns only this one
    imgs, fr = ren(_Meshes(d, faces))
    assert torch.equal(imgs, shade_meshes(d, faces, fr, _Cams(cam_s)))
    assert not torch.equal(imgs, shade_meshes(d, faces, fr, _Cams(cam_r)))
    imgs_k, fr_k = ren(_Meshes(d, faces), cameras=_Cams(cam_k))          # cameras= reaches both
    assert all(torch.equal(x, y) for x, y in zip(fr_k, rasterize_meshes(d, faces, _Cams(cam_k), (H, W))))
    assert torch.equal(imgs_k, shade_meshes(d, faces, fr_k, _Cams(cam_k)))


def test_outputs_stay_in_bounds_and_bad_indices_give_background(mesh):
    verts, faces = mesh
    N, H, W = 2, 70, 90
    d = deform(verts, N, 35)
    cam = cameras(N, H, W, 35)
    fr = rasterize_meshes(d, faces, _Cams(cam), (H, W))
    F, V = faces.shape[0], d.shape[1]
    bad = torch.cat([faces, torch.tensor([[0, 1, V], [-1, 1, 2]], device=DEV)]).contiguous()
    p2f = fr.pix_to_face.clone()
    p2f[p2f >= F] += 2                                                   # frame 1 in the packing of F + 2 faces
    p2f[0, 0, :5, 0] = torch.tensor([-5, F, F + 1, 2 * (F + 2), 1 << 40], device=DEV)   # bad faces / out of range
    fr2 = Fragments(p2f, fr.zbuf, fr.bary_coords, fr.dists)
    nrm = vertex_normals(d, bad)
    assert torch.equal(nrm, vertex_normals(d, faces))                    # faces with a bad index add nothing
    params = torch.tensor([[0.0] * 3 + [0.4, -0.8, -1.5] + [0.5] * 3 + [0.3] * 3 + [0.2] * 3 + [1.0] * 9 + [64.0] +
                           [0.1, 0.2, 0.3]] * N, device=DEV)
    params[:, :3] = torch.tensor(centre(cam), dtype=torch.float32, device=DEV)
    lib = _lib.load()
    G = 4096
    npix = N * H * W
    out = torch.full((4 * npix + 2 * G,), float("nan"), device=DEV)
    ptr = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off * t.element_size())   # noqa: E731
    _lib.check(lib.recmv_shade_phong(ptr(p2f), ptr(fr.bary_coords), N, H, W, ptr(d), ptr(nrm), None, V, ptr(bad),
                                     F + 2, ptr(params), ptr(out, G), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    assert bool(out[:G].isnan().all()) and bool(out[out.numel() - G:].isnan().all())
    body = out[G:G + 4 * npix].view(N, H, W, 4)
    assert not bool(body.isnan().any())
    assert torch.equal(body[0, 0, :5], torch.tensor([[0.1, 0.2, 0.3, 1.0]] * 5, device=DEV))
    assert torch.equal(body, ops.shade_phong(fr2, d, nrm, None, bad, params))
    ref = so.phong(p2f[..., 0].cpu().numpy(), fr.bary_coords[..., 0, :].double().cpu().numpy(), d.double().cpu().numpy(),
                   nrm.double().cpu().numpy(), None, bad.cpu().numpy(), centre(cam), [0.4, -0.8, -1.5],
                   background=(0.1, 0.2, 0.3))
    assert float((body.cpu().double() - torch.from_numpy(ref)).abs().max()) < RGB_TOL
    # a CPU tensor or a wrong shape is refused before any launch
    with pytest.raises(RuntimeError):
        ops.shade_phong(fr2, d.cpu(), nrm, None, bad, params)
    with pytest.raises(RuntimeError):
        ops.shade_phong(fr2, d, nrm[:, :-1].contiguous(), None, bad, params)
    with pytest.raises(RuntimeError):
        ops.vertex_normals(d, bad.int())


# ---- the drop-in, driven the way infer_garment drives it ------------------------------------------------------------

def test_drop_in_like_infer_garment(mesh):
    from recmv_b200.compat.MaskRender import (HardPhongShader, PointLights, SoftSilhouetteShader, TexturesVertex,
                                              mask_renderer)
    from recmv_b200.utils import FindSurfacePs
    verts, faces = mesh
    N, H, W = 2, 540, 720
    V, F = verts.shape[0], faces.shape[0]
    # the merged two-garment mesh: the sphere mesh and a shrunken, shifted copy, each with a constant colour
    tv = torch.cat([verts, verts * 0.5 + torch.tensor([0.3, 0.2, -0.6], device=DEV)])
    tf = torch.cat([faces, faces + V]).contiguous()
    d = deform(tv, N, 36)
    color = torch.cat([torch.tensor([0.8, 0.3, 0.3], device=DEV).expand(V, 3), torch.tensor([0.3, 0.3, 0.8],
                                                                                           device=DEV).expand(V, 3)])
    meshes = _Meshes(d, tf, TexturesVertex([color for _ in range(N)]))
    cam = cameras(N, H, W, 36)
    ren = mask_renderer((H, W))
    ren.shader = HardPhongShader(DEV, _Cams(cam))
    ren.rasterizer.cameras = _Cams(cam)
    bare = mask_renderer((H, W), _Cams(cam))
    with torch.no_grad():
        imgs, frags = ren(meshes)
        none, frags0 = bare(meshes)
    assert none is None and imgs.shape == (N, H, W, 4) and imgs[..., :3].shape == (N, H, W, 3)
    assert all(torch.equal(x, y) for x, y in zip(frags, frags0))
    assert all(torch.equal(x, y) for x, y in zip(frags, rasterize_meshes(d, tf, _Cams(cam), (H, W))))
    a, b = FindSurfacePs(tv, tf, frags), FindSurfacePs(tv, tf, frags0)
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and a[0].numel() > 1000
    lt = _Lights([[0.0, 1.0, 0.0]])
    ref = oracle_phong(frags, d, tf, cam, color.expand(N, -1, -1), lt)
    check_image(imgs, ref, frags, (1.0, 1.0, 1.0), "drop-in merged")
    # def1imgs: canonical-pose render with cameras= and lights= passed by keyword
    newT = torch.tensor([[0.0, 0.1, 2.8]], device=DEV).repeat(N, 1)
    Rn = torch.tensor([[-1.0, 0, 0], [0, 1, 0], [0, 0, -1]], device=DEV).repeat(N, 1, 1)
    newcam = torch.cat([cam[:, :4], Rn.reshape(N, 9), newT], 1).contiguous()
    white = _Meshes(d, tf, TexturesVertex([torch.ones_like(tv) for _ in range(N)]))
    with torch.no_grad():
        def1imgs, fr1 = ren(white, cameras=_Cams(newcam), lights=PointLights(device=DEV, location=((0, 1, 2.8),)))
    assert def1imgs.shape == (N, H, W, 4) and bool((fr1.pix_to_face >= 0).any())
    ref1 = so.phong(fr1.pix_to_face[..., 0].cpu().numpy(), fr1.bary_coords[..., 0, :].double().cpu().numpy(),
                    d.double().cpu().numpy(), so.vertex_normals(d.double().cpu().numpy(), tf.cpu().numpy()), None,
                    tf.cpu().numpy(), centre(newcam), [0, 1, 2.8])
    check_image(def1imgs, ref1, fr1, (1.0, 1.0, 1.0), "def1imgs")
    # the silhouette shader of model/network.py:316-322
    ren.shader = SoftSilhouetteShader()
    sil, fr2 = ren(meshes)
    assert all(torch.equal(x, y) for x, y in zip(fr2, frags0))
    ref2 = so.silhouette(fr2.pix_to_face[..., 0].cpu().numpy(), fr2.dists[..., 0].double().cpu().numpy(), 1e-4)
    es = float((sil.cpu().double() - torch.from_numpy(ref2)).abs().max())
    print(f"[silhouette] max |rgba - f64| {es:.2e} (bound {SILHOUETTE_TOL:.0e})")
    assert es < SILHOUETTE_TOL and bool((sil[..., :3] == 1).all()) and bool((sil[..., 3][fr2.pix_to_face[..., 0] < 0] == 0).all())
    # an unknown shader is refused by name
    ren.shader = object()
    with pytest.raises(NotImplementedError, match="object"):
        ren(meshes)
