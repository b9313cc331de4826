"""GPU tests of the mesh rasterizer (csrc/raster.cu, recmv_b200.raster) against the float64 oracle
(oracle/raster_oracle.py).

Pixels whose decision is ambiguous at fp32 precision -- a pixel centre within MARGIN_PX pixels of an edge of a face it
might belong to, or a runner-up zbuf within ZTOL * zbuf of the winner's -- are counted, printed and bounded; on every
other pixel pix_to_face is bit-equal to the oracle and bary / zbuf / dists are within the float64 bounds of DESIGN
section 6 (about 3x the maxima measured on an H100).

Scenes: the marching-cubes mesh of synth.sphere_sdf_grid at 257^3 (201 548 faces) deformed by LBSkinner at 1, 3 and 4
frames with their own poses and cameras; adversarial scenes (a face over the whole image, a fan of 1e5 slivers through
one pixel, sub-pixel faces, faces off-screen and behind the camera, zero-area faces, coincident copies, no faces,
ragged and 1x1 images, a pair list that has to grow); bit-exact invariances; NaN-guarded output bounds through the C ABI;
and the path to FindSurfacePs."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import raster_oracle as ro
from recmv_b200 import _lib, ops, synth
from recmv_b200.model import LBSkinner
from recmv_b200.raster import Fragments, rasterize_meshes

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

MARGIN_PX = 2e-3          # decision margin of the coverage test, in pixels
ZTOL = 1e-6               # relative decision margin of the depth test
AMBIGUOUS_SHARE = 0.12    # of the covered pixels
BARY_TOL, ZBUF_TOL, DISTS_TOL = 7e-3, 2e-5, 1.2e-3   # on unambiguous pixels: bary abs, zbuf rel, dists rel (floor 1e-6)


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


def compare(verts, faces, cam, H, W, want_dists=True, label="", z_clip=1e-6, area_eps=1e-8):
    p2f, zbuf, bary, dists, counts = ops.rasterize_meshes(verts, faces, cam, H, W, z_clip, area_eps, want_dists)
    ref = ro.rasterize(verts.double().cpu().numpy(), faces.cpu().numpy(), cam.double().cpu().numpy(), H, W,
                       z_clip=z_clip, area_eps=area_eps, margin_px=MARGIN_PX, ztol=ZTOL)
    p = p2f[..., 0].cpu().numpy()
    amb = ref["ambiguous"]
    ok = ~amb
    cov_ref = ref["pix_to_face"] >= 0
    n_cov = max(int(cov_ref.sum()), 1)
    mism = int((p[ok] != ref["pix_to_face"][ok]).sum())
    hit = ok & cov_ref
    eb = float(np.abs(bary[..., 0, :].cpu().double().numpy()[hit] - ref["bary"][hit]).max()) if hit.any() else 0.0
    ez = float((np.abs(zbuf[..., 0].cpu().double().numpy()[hit] - ref["zbuf"][hit]) / ref["zbuf"][hit]).max()) \
        if hit.any() else 0.0
    ed = float((np.abs(dists[..., 0].cpu().double().numpy()[hit] - ref["dists"][hit])
                / np.maximum(np.abs(ref["dists"][hit]), 1e-6)).max()) if (hit.any() and want_dists) else 0.0
    print(f"[raster {label}] N={p.shape[0]} {H}x{W} F={faces.shape[0]} covered={n_cov} pairs={counts['pairs']} "
          f"skipped={counts['skipped']} (f64 {ref['skipped']} +- {ref['skipped_ambiguous']}) ambiguous={int(amb.sum())} "
          f"({amb.sum() / n_cov:.2e}, depth {int(ref['ambiguous_z'].sum())}) mismatches={mism} "
          f"bary={eb:.2e} zbuf={ez:.2e} dists={ed:.2e}")
    assert mism == 0
    assert abs(counts["skipped"] - ref["skipped"]) <= ref["skipped_ambiguous"]
    bg = p < 0
    assert np.array_equal(bg[ok], ~cov_ref[ok])
    for t in (zbuf[..., 0], dists[..., 0] if want_dists else None):
        if t is not None:
            assert bool((t.cpu().numpy()[bg] == -1).all())
    assert bool((bary[..., 0, :].cpu().numpy()[bg] == -1).all())
    assert counts["covered"] == int((~bg).sum())
    assert eb < BARY_TOL and ez < ZBUF_TOL and ed < DISTS_TOL, (eb, ez, ed)
    return (p2f, zbuf, bary, dists, counts), ref


@pytest.mark.parametrize("N,H,W,seed", [(1, 512, 512, 1), (3, 1080, 1080, 2), (4, 540, 960, 3)])
def test_deformed_mc_mesh_against_oracle(mesh, N, H, W, seed):
    verts, faces = mesh
    d = deform(verts, N, seed)
    (p2f, *_), ref = compare(d, faces, cameras(N, H, W, seed), H, W, label="mc")
    cov = int((ref["pix_to_face"] >= 0).sum())
    assert cov > 0.05 * N * H * W
    assert ref["ambiguous"].sum() < AMBIGUOUS_SHARE * cov


def screen_scene(tris_screen, depths, H, W):
    """World vertices for screen-space triangles [F,3,2] at view depths [F,3] under one fixed camera."""
    cam = torch.tensor([[0.8 * W, 0.8 * W, W / 2 + 0.25, H / 2 - 0.25, -1, 0, 0, 0, -1, 0, 0, 0, 1, 0.1, -0.2, 2.0]],
                       dtype=torch.float64)
    s = torch.as_tensor(tris_screen, dtype=torch.float64).reshape(-1, 2)
    z = torch.as_tensor(depths, dtype=torch.float64).reshape(-1)
    fx, fy, px, py = cam[0, :4]
    Xv = torch.stack([(px - s[:, 0]) * z / fx, (py - s[:, 1]) * z / fy, z], 1)
    R, T = cam[0, 4:13].view(3, 3), cam[0, 13:]
    X = (Xv - T) @ R.T
    faces = torch.arange(X.shape[0]).view(-1, 3)
    return X.float()[None].to(DEV).contiguous(), faces.to(DEV), cam.float().to(DEV)


def test_one_face_over_the_whole_image():
    H, W = 300, 200
    v, f, c = screen_scene([[[-500, -400], [900, -300], [-200, 1200]]], [[2.0, 3.0, 2.5]], H, W)
    (p2f, *_rest), _ = compare(v, f, c, H, W, label="full")
    assert bool((p2f == 0).all()) and _rest[-1]["pairs"] == ((W + 31) // 32) * ((H + 7) // 8)


def test_fan_of_slivers_through_one_pixel():
    K, H, W = 100_000, 64, 96
    g = np.random.default_rng(3)
    th = g.uniform(0, 2 * np.pi, K)
    u, v = np.stack([np.cos(th), np.sin(th)], 1), np.stack([-np.sin(th), np.cos(th)], 1)
    c = np.array([40.0, 20.0])
    tris = np.stack([c - 0.5 * u, c + 3 * u + 0.2 * v, c + 3 * u - 0.2 * v], 1)
    depth = np.repeat(g.uniform(2.0, 3.0, K)[:, None], 3, 1)
    vv, f, cam = screen_scene(tris, depth, H, W)
    (p2f, zbuf, _b, _d, counts), ref = compare(vv, f, cam, H, W, label="fan")
    assert counts["pairs"] >= K
    assert int(p2f[0, 20, 40, 0]) == int(np.argmin(depth[:, 0]))


def test_subpixel_offscreen_behind_camera_and_zero_area_faces():
    H, W = 77, 101
    g = np.random.default_rng(4)
    small = g.uniform(0, [W, H], (3000, 1, 2)) + g.normal(size=(3000, 3, 2)) * 0.3        # sub-pixel faces
    large = g.uniform(-W, 2 * W, (300, 3, 2))                                             # partly / fully off-screen
    flat = np.repeat(g.uniform(0, [W, H], (200, 1, 2)), 3, 1)                              # zero area
    tris = np.concatenate([small, large, flat])
    depth = g.uniform(2.0, 4.0, (tris.shape[0], 3))
    depth[3000:3100, 1] = g.uniform(-1.0, 0.0, 100)                                       # a vertex behind the camera
    v, f, cam = screen_scene(tris, depth, H, W)
    (_p, _z, _b, _d, counts), ref = compare(v, f, cam, H, W, label="mixed")
    assert counts["skipped"] >= 300


def test_coincident_copies_pick_the_lower_copy(mesh):
    verts, faces = mesh
    d = deform(verts, 2, 5)
    F = faces.shape[0]
    (p2f, *_), _ = compare(d, torch.cat([faces, faces]).contiguous(), cameras(2, 256, 320, 5), 256, 320, label="copies")
    p = p2f[..., 0]
    hit = p >= 0
    n = torch.arange(2, device=DEV).view(2, 1, 1).expand_as(p)
    assert bool(hit.any()) and bool(((p - n * 2 * F)[hit] < F).all())


@pytest.mark.parametrize("H,W", [(1, 1), (33, 65), (7, 31), (1080, 1)])
def test_ragged_and_tiny_images(mesh, H, W):
    verts, faces = mesh
    compare(deform(verts, 2, 6), faces, cameras(2, max(H, 8), max(W, 8), 6), H, W, label=f"{H}x{W}")


def test_no_faces():
    v = torch.randn((2, 10, 3), device=DEV)
    cam = cameras(2, 16, 16, 1)
    for faces in (torch.zeros((0, 3), dtype=torch.int64, device=DEV),):
        p2f, zbuf, bary, dists, counts = ops.rasterize_meshes(v, faces, cam, 16, 24)
        assert bool((p2f == -1).all() and (zbuf == -1).all() and (bary == -1).all() and (dists == -1).all())
        assert counts == {"covered": 0, "skipped": 0, "pairs": 0}
    p2f, *_ = ops.rasterize_meshes(torch.zeros((2, 0, 3), device=DEV), faces, cam, 5, 7)
    assert p2f.shape == (2, 5, 7, 1) and bool((p2f == -1).all())


def test_pair_list_regrows_to_the_same_result(mesh):
    verts, faces = mesh
    d = deform(verts, 3, 7)
    cam = cameras(3, 400, 400, 7)
    big = ops.rasterize_meshes(d, faces, cam, 400, 400, capacity=10_000_000)
    ops._scratch_cache.clear()                         # a fresh workspace that must grow inside the call
    small = ops.rasterize_meshes(d, faces, cam, 400, 400, capacity=16)
    assert small[4] == big[4] and small[4]["pairs"] > 16
    for a, b in zip(big[:4], small[:4]):
        assert torch.equal(a, b)


def test_invariances(mesh):
    verts, faces = mesh
    N, H, W = 3, 360, 480
    d = deform(verts, N, 8)
    cam = cameras(N, H, W, 8)
    F = faces.shape[0]
    a = ops.rasterize_meshes(d, faces, cam, H, W)
    b = ops.rasterize_meshes(d, faces, cam, H, W)
    for x, y in zip(a[:4], b[:4]):
        assert torch.equal(x, y)                                          # two runs
    for n in range(N):                                                    # N frames = N one-frame launches
        s = ops.rasterize_meshes(d[n:n + 1].contiguous(), faces, cam[n:n + 1].contiguous(), H, W)
        p = s[0].clone()
        p[p >= 0] += n * F
        assert torch.equal(p, a[0][n:n + 1])
        for x, y in zip(s[1:4], a[1:4]):
            assert torch.equal(x, y[n:n + 1])
    nd = ops.rasterize_meshes(d, faces, cam, H, W, want_dists=False)     # dists off: the rest unchanged
    assert nd[3] is None and all(torch.equal(x, y) for x, y in zip(nd[:3], a[:3]))
    perm = torch.randperm(F, generator=synth.generator(9)).to(DEV)       # permuted faces
    pp = ops.rasterize_meshes(d, faces[perm].contiguous(), cam, H, W)
    q, q0 = pp[0][..., 0], a[0][..., 0]
    nF = torch.arange(N, device=DEV).view(N, 1, 1) * F
    mapped = torch.where(q >= 0, perm[(q - nF).clamp_min(0)] + nF, q)
    diff = mapped != q0
    assert bool((pp[1][..., 0][diff] == a[1][..., 0][diff]).all())      # only exact z-ties may differ
    print(f"[raster permutation] z-tie pixels that changed face: {int(diff.sum())}")
    assert int(diff.sum()) <= 1e-4 * int((q0 >= 0).sum())     # none measured
    keep = ~diff
    assert torch.equal(pp[1][keep], a[1][keep]) and torch.equal(pp[2][keep], a[2][keep])


def test_outputs_stay_in_bounds_through_the_c_abi(mesh):
    verts, faces = mesh
    N, H, W = 2, 70, 90
    d = deform(verts, N, 10)
    cam = cameras(N, H, W, 10)
    lib = _lib.load()
    G = 4096
    npix = N * H * W
    p2f = torch.full((npix + 2 * G,), -7, dtype=torch.int64, device=DEV)
    zb, di = (torch.full((npix + 2 * G,), float("nan"), device=DEV) for _ in range(2))
    ba = torch.full((3 * npix + 2 * G,), float("nan"), device=DEV)
    cap = 1 << 20
    nbytes = ctypes.c_size_t(0)
    _lib.check(lib.recmv_raster_workspace_bytes(N, faces.shape[0], H, W, cap, ctypes.byref(nbytes)))
    ws = torch.empty((nbytes.value,), dtype=torch.uint8, device=DEV)
    ctr = torch.full((4,), 99, dtype=torch.int32, device=DEV)
    ptr = lambda t, off=G: ctypes.c_void_p(t.data_ptr() + off * t.element_size())   # noqa: E731
    _lib.check(lib.recmv_rasterize_meshes(ptr(d, 0), d.shape[1], ptr(faces, 0), faces.shape[0], N, ptr(cam, 0), H, W, 1e-6,
                                          1e-8, ptr(ws, 0), cap, ptr(p2f), ptr(zb), ptr(ba), ptr(di), ptr(ctr, 0),
                                          ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    for t in (p2f, zb, di, ba):
        assert bool((t[:G] == -7).all()) if t.dtype == torch.int64 else bool(t[:G].isnan().all())
        tail = t[t.numel() - G:]
        assert bool((tail == -7).all()) if t.dtype == torch.int64 else bool(tail.isnan().all())
        body = t[G:t.numel() - G]
        assert bool((body != -7).all()) if t.dtype == torch.int64 else not bool(body.isnan().any())
    ref = ops.rasterize_meshes(d, faces, cam, H, W)
    assert torch.equal(p2f[G:G + npix], ref[0].view(-1)) and torch.equal(ba[G:G + 3 * npix], ref[2].view(-1))
    assert int(ctr[3]) == 0 and int(ctr[0]) == ref[4]["covered"]
    # argument checks before any CUDA call
    assert lib.recmv_rasterize_meshes(None, 0, None, 0, 1, None, 0, W, 0.0, 0.0, None, 0, None, None, None, None,
                                      ptr(ctr, 0), None) == -3
    assert lib.recmv_rasterize_meshes(ptr(d, 0), d.shape[1], ptr(faces, 0), faces.shape[0], N, None, H, W, 0.0, 0.0,
                                      ptr(ws, 0), cap, ptr(p2f), ptr(zb), ptr(ba), None, ptr(ctr, 0), None) == -1


def test_python_api_rejects_cpu_and_non_contiguous(mesh):
    verts, faces = mesh
    d = deform(verts, 2, 11)
    cam = (torch.tensor([[500.0, 500.0]]), torch.tensor([[200.0, 150.0]]), torch.diag(torch.tensor([-1.0, -1.0, 1.0]))[None],
           torch.tensor([[0.0, 0.0, 2.6]]))
    with pytest.raises(RuntimeError):
        rasterize_meshes(d.cpu(), faces.cpu(), cam, (300, 400))
    with pytest.raises(RuntimeError):
        rasterize_meshes(d.transpose(0, 1).contiguous().transpose(0, 1), faces, cam, (300, 400))
    with pytest.raises(RuntimeError):
        rasterize_meshes(d, faces.t().contiguous().t(), cam, (300, 400))
    fr = rasterize_meshes(d, faces, cam, (300, 400))                     # one camera shared by both frames
    assert isinstance(fr, Fragments) and fr.pix_to_face.shape == (2, 300, 400, 1) and fr.bary_coords.shape[-2:] == (1, 3)


class _Cams:
    """The attributes of the reference's RectifiedPerspectiveCameras the rasterizer reads."""

    def __init__(self, rows):
        self.focal_length, self.principal_point = rows[:, 0:2], rows[:, 2:4]
        self.R, self.T = rows[:, 4:13].reshape(-1, 3, 3), rows[:, 13:16]


class _Meshes:
    def __init__(self, verts, faces):
        self._v, self._f = verts, faces

    def verts_padded(self):
        return self._v

    def faces_list(self):
        return [self._f] * self._v.shape[0]


def test_end_to_end_fragment_decode_and_find_surface(mesh):
    from recmv_b200.compat.MaskRender import mask_renderer
    from recmv_b200.utils import FindSurfacePs, FindSurfacePsMesh, FindSurfacePsRays
    verts, faces = mesh
    N, H, W = 2, 540, 720
    d = deform(verts, N, 12)
    cam = cameras(N, H, W, 12)
    fr = rasterize_meshes(d, faces, _Cams(cam), (H, W))
    # the device decode equals the CPU path of FindSurfacePs on our fragments
    dev = FindSurfacePs(verts, faces, fr)
    cpu = FindSurfacePs(verts.cpu(), faces.cpu(), Fragments(*(t.cpu() for t in fr)))
    for x, y in zip(dev[:3] + dev[4:], cpu[:3] + cpu[4:]):
        assert torch.equal(x.cpu(), y)
    assert (dev[3].cpu() - cpu[3]).abs().max() < 1e-6 and dev[0].numel() > 10000
    # FindSurfacePsMesh = rasterize + FindSurfacePsRays, bit for bit (with and without the mask)
    mask = (torch.rand((N, H, W), generator=synth.generator(3)) > 0.2).float().to(DEV)
    c0 = cam[0].cpu()
    for m in (None, mask):
        a = FindSurfacePsMesh(verts, faces, d, _Cams(cam), H, W, m)
        b = FindSurfacePsRays(verts, faces, fr, (c0[0], c0[1], c0[2], c0[3], c0[4:13].view(3, 3)), m)
        assert len(a) == 6 and all(torch.equal(x, y) for x, y in zip(a, b))
    # each pixel's observation-space seed point (on the deformed mesh) lies on its view ray from cam_pos
    b, r, c, pts, fi, rays = FindSurfacePsRays(d[0], faces, Fragments(fr.pix_to_face[:1], fr.zbuf[:1], fr.bary_coords[:1],
                                                                         None), (c0[0], c0[1], c0[2], c0[3],
                                                                                 c0[4:13].view(3, 3)))
    R, T = c0[4:13].view(3, 3).double(), c0[13:16].double()
    cp = -(R @ T)
    v = pts.cpu().double() - cp
    off = (torch.linalg.cross(v, rays.cpu().double(), dim=1).norm(dim=1) / v.norm(dim=1)).max().item()
    print(f"[raster seed points] max angle to the view ray {off:.2e} rad over {pts.shape[0]} pixels")
    assert off < 4e-7
    # the compat renderer driven the way find_surface_ps drives it
    ren = mask_renderer((H, W))
    ren.rasterizer.cameras = _Cams(cam)
    imgs, fr2 = ren(_Meshes(d, faces))
    assert imgs is None and ren.rasterizer.raster_settings.image_size == (H, W)
    assert all(torch.equal(x, y) for x, y in zip(fr, fr2))
    assert all(torch.equal(x, y) for x, y in zip(fr, ren(_Meshes(d, faces), cameras=_Cams(cam))[1]))
