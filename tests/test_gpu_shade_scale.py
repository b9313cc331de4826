"""The shading kernels bit for bit against their float32 restatement (tests/shade_f32.py).

vertex_normals must equal the restatement on every vertex of every mesh below; shade_phong on every pixel, given the
kernel's own powf values, which a material with only a specular term reads back (each channel is then exactly
powf(sa, shininess)).  Those powf values are held to the correctly rounded power of the restated sa within POW_ULP.
Zeros compare with ==: a +0 / -0 difference is not a finding; every other value compares by its bits (NaN included).
The restatement itself is held to float64 by tests/test_shade_f32_cpu.py.

Restated on subsets where the whole would be slow: of the 64-frame mc sphere, frames 0, 1, 32 and 63.
"""
import numpy as np
import pytest
import torch

import shade_f32 as sf
import shade_scenes as ss
from oracle import shade_oracle as so
from recmv_b200 import ops, synth
from recmv_b200.model import LBSkinner
from recmv_b200.raster import Fragments, rasterize_meshes

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# largest |powf(sa, n) - pow_rn(sa, n)| in float32 ulps of the correctly rounded value, over every covered pixel of
# the tests below; measured on an H100 80GB HBM3 at 700 W: 1 ulp (0 at shininess 0 and 1).  __powf measured 10 to 181
# ulp there, and NaN for powf(0, 0).
POW_ULP = 2
_pow = {"ulp": 0}


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    eq = (a.view(np.uint32) == b.view(np.uint32)) | ((a == 0) & (b == 0)) | (np.isnan(a) & np.isnan(b))
    bad = np.argwhere(~eq)
    return (None if not len(bad) else (tuple(bad[0]), a[tuple(bad[0])], b[tuple(bad[0])], int(len(bad))))


def t(x, dt=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x)).to(DEV, dt).contiguous()


# ---- meshes ---------------------------------------------------------------------------------------------------------
def _skinner():
    Js, parents, init = synth.skeleton()
    ws = synth.skinning_voxel((17, 33, 21), seed=7)
    return LBSkinner(ws, [-1.1] * 3, [1.1] * 3, Js, parents, init_pose=init,
                     bbox_extend=torch.tensor(synth.BBOX_EXTEND), bbox_center=torch.tensor(synth.BBOX_CENTER)).to(DEV)


@pytest.fixture(scope="module")
def mc_sphere():
    sdf = synth.sphere_sdf_grid(257, num=8, seed=3, device=DEV)
    h = 2.0 / 256
    verts, faces = ops.mc_gpu(sdf, h, h, h, -1.0, -1.0, -1.0, 0.0)
    return verts.float().contiguous(), faces.contiguous()


def deform(verts, N, seed):
    poses, trans = synth.poses_trans(N, seed=seed)
    V = verts.shape[0]
    with torch.no_grad():
        d = _skinner()(verts.repeat(N, 1), [poses.to(DEV), trans.to(DEV)],
                       torch.arange(N, device=DEV).repeat_interleave(V))
    return d.view(N, V, 3).contiguous()


def check_normals(verts, faces, label, frames=None):
    """vertex_normals on the GPU against the restatement on `frames` (default all)."""
    verts = verts.cpu().numpy() if torch.is_tensor(verts) else np.asarray(verts, np.float32)
    faces = faces.cpu().numpy() if torch.is_tensor(faces) else np.asarray(faces, np.int64)
    got = ops.vertex_normals(t(verts), t(faces, torch.int64)).cpu().numpy()
    frames = range(verts.shape[0]) if frames is None else frames
    for n in frames:
        ref = sf.vertex_normals(verts[n:n + 1], faces)
        d = same_bits(got[n:n + 1], ref)
        assert d is None, (label, n, d)
    print(f"[normals {label}] N={verts.shape[0]} V={verts.shape[1]} F={faces.shape[0]}: bit-exact on frames "
          f"{list(frames) if len(frames) < 8 else 'all'}")
    return got


@pytest.mark.parametrize("N", [1, 3, 64])
def test_mc_sphere_normals_bit_exact(mc_sphere, N):
    verts, faces = mc_sphere
    d = deform(verts, N, 40 + N)
    check_normals(d, faces, f"mc sphere N={N}", frames=[0, 1, 32, 63] if N == 64 else None)


def test_fan_of_1e5_faces_bit_exact():
    v, f = ss.fan(100_000)
    check_normals(v, f, "fan 1e5")


def test_adversarial_normals_bit_exact():
    v, f = ss.adversarial_mesh()
    got = check_normals(v, f, "adversarial")
    assert np.isnan(got[0]).any() and np.isfinite(got[1]).all()


@pytest.mark.parametrize("V,F", [(1, 1), (1, 2000), (256, 1365), (257, 1366), (65536, 100_000), (65537, 30_000),
                                 ((1 << 24) + 1, 200_000)])
def test_sort_shapes_bit_exact(V, F):
    """V sets the sort's key bits (V itself is the key of an invalid face) and 3F its single-tile or onesweep path."""
    g = np.random.default_rng(V + F)
    v = g.normal(size=(1, V, 3)).astype(np.float32)
    f = g.integers(0, V, size=(F, 3))
    f[g.random(F) < 0.01, 1] = V                                                   # invalid faces
    f[0] = V - 1                                                                   # the highest valid key
    check_normals(v, f, f"V={V} F={F}")


# ---- Phong ----------------------------------------------------------------------------------------------------------
def params_rows(N, centre, light, shininess=64.0, amb=(0.5,) * 3, dif=(0.3,) * 3, spc=(0.2,) * 3,
                mat=((1.0,) * 3, (1.0,) * 3, (1.0,) * 3), bg=(0.25, 0.5, 0.75)):
    p = np.zeros((N, 28), np.float32)
    p[:, 0:3], p[:, 3:6] = centre, light
    p[:, 6:9], p[:, 9:12], p[:, 12:15] = amb, dif, spc
    p[:, 15:18], p[:, 18:21], p[:, 21:24] = mat
    p[:, 24], p[:, 25:28] = shininess, bg
    return p


def check_phong(p2f, bary, verts, normals, colors, faces, params, label):
    """Bit-exact Phong given the kernel's powf, powf within POW_ULP of the correctly rounded power, and the specular
    material 0 bit-exact with no powf at all.  Returns the restated image."""
    N, H, W = p2f.shape
    fr = Fragments(t(p2f, torch.int64)[..., None], None, t(bary)[..., None, :], None)
    args = (t(verts), t(normals), None if colors is None else t(colors), t(faces, torch.int64))
    cov = sf._fragments(p2f, faces, N, verts.shape[1], np.asarray(faces).reshape(-1, 3).shape[0])[0].reshape(N, H, W)
    spec = ops.shade_phong(fr, *args[:2], args[2], args[3], t(sf.spec_only_params(params))).cpu().numpy()
    assert same_bits(spec[cov][:, 0], spec[cov][:, 1]) is None and same_bits(spec[cov][:, 0], spec[cov][:, 2]) is None
    img = ops.shade_phong(fr, *args[:2], args[2], args[3], t(params)).cpu().numpy()
    ref, sa = sf.phong(p2f, bary, verts, normals, colors, faces, params, spec=spec[..., 0])
    d = same_bits(img, ref)
    assert d is None, (label, "rgba", d)
    # powf against the correctly rounded power of the restated sa, on covered pixels
    sh = np.broadcast_to(np.asarray(params, np.float32)[:, 24][:, None, None], (N, H, W))
    exact = sf.pow_rn(sa, sh)
    got = spec[..., 0]
    ulp = np.spacing(np.abs(exact).astype(np.float32))
    with np.errstate(invalid="ignore"):
        e = np.where(got == exact, 0.0, np.abs(got.astype(np.float64) - exact) / ulp)[cov]
    worst = float(e.max(initial=0.0))
    _pow["ulp"] = max(_pow["ulp"], worst)
    assert worst <= POW_ULP, (label, worst)
    # no specular material: powf cannot matter
    p0 = np.array(params, copy=True)
    p0[:, 21:24] = 0
    img0 = ops.shade_phong(fr, *args[:2], args[2], args[3], t(p0)).cpu().numpy()
    assert same_bits(img0, sf.phong(p2f, bary, verts, normals, colors, faces, p0)[0]) is None, label
    print(f"[phong {label}] N={N} {H}x{W} covered={int(cov.sum())}: bit-exact; powf max {worst:.0f} ulp "
          f"(bound {POW_ULP})")
    return ref


class _Cams:
    def __init__(self, rows):
        self.focal_length, self.principal_point = rows[:, 0:2], rows[:, 2:4]
        self.R, self.T = rows[:, 4:13].reshape(-1, 3, 3), rows[:, 13:16]


def camera(H, W):
    R = np.diag([-1.0, -1.0, 1.0])
    f = 0.9 * min(H, W)
    return np.concatenate([[f, f, W / 2 - 0.5, H / 2 - 0.5], R.reshape(-1), [0.02, -0.03, 2.6]])[None]


@pytest.mark.parametrize("shininess", [0.0, 1.0, 10.5, 64.0])
def test_phong_mc_sphere_1080_bit_exact(mc_sphere, shininess):
    verts, faces = mc_sphere
    H = W = 1080
    d = deform(verts, 1, 30)
    cam = camera(H, W)
    fr = rasterize_meshes(d, faces, _Cams(torch.tensor(cam, dtype=torch.float32, device=DEV)), (H, W))
    nrm = ops.vertex_normals(d, faces)
    colors = torch.rand((1, d.shape[1], 3), generator=synth.generator(4)).numpy()
    centre = -cam[0, 4:13].reshape(3, 3) @ cam[0, 13:16]
    params = params_rows(1, centre, [0.4, -0.8, -1.5], shininess)
    check_phong(fr.pix_to_face[..., 0].cpu().numpy(), fr.bary_coords[..., 0, :].cpu().numpy(), d.cpu().numpy(),
                nrm.cpu().numpy(), colors, faces.cpu().numpy(), params, f"mc sphere 1080^2 n={shininess}")


@pytest.mark.parametrize("shininess", [0.0, 1.0, 10.5, 64.0])
def test_phong_hand_built_bit_exact(shininess):
    p2f, bary, verts, normals, colors, faces, centre, light = ss.hand_fragments()
    N = p2f.shape[0]
    params = params_rows(N, centre, light, shininess, amb=np.tile([0.5, 0.4, 0.3], (N, 1)))
    ref = check_phong(p2f, bary, verts, normals, colors, faces, params, f"hand-built n={shininess}")
    check_phong(p2f, bary, verts, normals, None, faces, params, f"hand-built no colours n={shininess}")
    # cos exactly 0 (frame 3): no diffuse and, for shininess > 0, no specular; shininess 0 gives powf(0, 0) = 1
    _, sa = sf.phong(p2f, bary, verts, normals, colors, faces, params)
    assert sa[3, 0, 1] == 0
    spec = 1.0 if shininess == 0 else 0.0
    assert np.allclose(ref[3, 0, 1, :3], np.array([0.5, 0.4, 0.3]) * colors[3, 6] + 0.2 * spec, rtol=1e-6, atol=0)


def test_shininess_0_matches_pytorch3d_and_the_oracle():
    """pytorch3d's phong_shading takes torch.pow(relu(cos) * mask, shininess): 0^0 = 1 on every covered pixel, lit or
    not.  The kernel's powf(0, 0) gives the same, as does the float64 oracle."""
    p2f, bary, verts, normals, colors, faces, centre, light = ss.hand_fragments(1)
    N = p2f.shape[0]
    params = sf.spec_only_params(params_rows(N, centre, light, 0.0))
    fr = Fragments(t(p2f, torch.int64)[..., None], None, t(bary)[..., None, :], None)
    img = ops.shade_phong(fr, t(verts), t(normals), t(colors), t(faces, torch.int64), t(params)).cpu().numpy()
    cov = sf._fragments(p2f, faces, N, verts.shape[1], len(faces))[0].reshape(p2f.shape)
    assert (img[cov][:, :3] == 1).all()
    assert float(torch.pow(torch.zeros(()), torch.zeros(()))) == 1.0
    ref = so.phong(p2f, bary, verts, normals, colors, faces, params[:, 0:3], params[:, 3:6], params[:, 6:9],
                   params[:, 9:12], params[:, 12:15], params[:, 15:18], params[:, 18:21], params[:, 21:24],
                   params[:, 24:25], params[:, 25:28])
    assert (ref[cov][:, :3] == 1).all()


def test_measured_pow_ulp_printed():
    print(f"[phong powf] largest measured error over the Phong tests run: {_pow['ulp']:.0f} ulp (bound {POW_ULP})")
