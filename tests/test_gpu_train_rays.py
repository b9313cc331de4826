"""GPU tests of the training-ray sampler (csrc/train_rays.cu, DESIGN section 1j) and the `sample_train_ray` drop-in
(recmv_b200.utils.make_sample_train_ray): kept rows bit for bit against the oracle (oracle/train_rays_oracle.py), rays
bit for bit against the fragment decode's and within 1e-6 of the torch expression (the bound of
tests/test_gpu_boundary.py), the drop-in against the reference's own function (tests/golden/train_rays_ref.npz), the
learnable-camera branch, run-to-run identity, the one host read, and a binomial check of the keep rate."""
import sys
import types
import warnings

import numpy as np
import pytest
import torch
from scipy import stats

from conftest import load_golden
from oracle import train_rays_oracle as tro
from recmv_b200 import ops
from recmv_b200.utils import make_sample_train_ray

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = 0x9E3779B97F4A7C15
_q = np.array([0.9, -0.1, 0.35, 0.2]) / np.linalg.norm([0.9, -0.1, 0.35, 0.2])
_R = np.array([[1 - 2 * (_q[2] ** 2 + _q[3] ** 2), 2 * (_q[1] * _q[2] - _q[3] * _q[0]), 2 * (_q[1] * _q[3] + _q[2] * _q[0])],
               [2 * (_q[1] * _q[2] + _q[3] * _q[0]), 1 - 2 * (_q[1] ** 2 + _q[3] ** 2), 2 * (_q[2] * _q[3] - _q[1] * _q[0])],
               [2 * (_q[1] * _q[3] - _q[2] * _q[0]), 2 * (_q[2] * _q[3] + _q[1] * _q[0]), 1 - 2 * (_q[1] ** 2 + _q[2] ** 2)]])
CAM = np.concatenate([[1100.0, 1087.5, 540.25, 531.5], (_R @ np.diag([1., -1., -1.])).ravel()]).astype(np.float32)


@pytest.fixture(autouse=True)
def _no_aborted_launch():
    yield
    torch.cuda.synchronize()
    ops.check_async_errors()


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _scene(seed, G, N, H, W, cover, mask_p=(0.4, 0.5, 0.1), nan=0.0, P=None):
    """G garments: masks [N,H,W] with values (0, 1, -1) at mask_p (a share `nan` of NaN), and lists of the covered
    pixels in (n, row, col) order (or P random rows, repeats allowed, when P is given)."""
    g = np.random.default_rng(seed)
    out = []
    for _ in range(G):
        mask = g.choice(np.array([0., 1., -1.], np.float32), size=(N, H, W), p=mask_p)
        if nan:
            mask[g.uniform(size=mask.shape) < nan] = np.nan
        if P is None:
            b, r, c = np.nonzero(g.uniform(size=(N, H, W)) < cover)
        else:
            flat = np.sort(g.integers(0, N * H * W, size=P))
            b, r, c = flat // (H * W), flat // W % H, flat % W
        pts = g.standard_normal((len(b), 3)).astype(np.float32)
        out.append((mask, b.astype(np.int64), r.astype(np.int64), c.astype(np.int64), pts))
    return out


def _run(scene, target, seed=SEED, offset=0, cam=CAM):
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(DEV)  # noqa: E731
    return ops.train_rays_sample([t(s[1]) for s in scene], [t(s[2]) for s in scene], [t(s[3]) for s in scene],
                                 [t(s[4]) for s in scene], [t(s[0]) for s in scene], t(cam), target, seed, offset)


def _check(scene, target, seed=SEED, offset=0):
    got = _run(scene, target, seed, offset)
    want, _ = tro.sample([s[0] for s in scene], [s[1] for s in scene], [s[2] for s in scene], [s[3] for s in scene],
                         target, seed, offset, CAM)
    for g, ((mask, b, r, c, pts), (keep, rays), out) in enumerate(zip(scene, want, got)):
        ob, orow, ocol, opts, orays = (x.cpu().numpy() for x in out)
        for name, a, e in (("batch", ob, b[keep]), ("row", orow, r[keep]), ("col", ocol, c[keep]),
                           ("pts", opts, pts[keep]), ("rays", orays, rays.astype(np.float32))):
            assert _same(a, e), f"garment {g}: {name} differs ({len(a)} vs {len(e)} rows)"
    return got, want


def _pnum(scene, g=0):
    s = scene[g]
    return len(tro.candidates(s[0], s[1], s[2], s[3]))


CASES = {
    "G1_N1_1080": lambda: (_scene(1, 1, 1, 1080, 1080, 0.4), 2048),
    "G2_N4_1080": lambda: (_scene(2, 2, 4, 1080, 1080, 0.35), 3072 * 4),
    "G2_N4_1080_keep_all": lambda: (_scene(3, 2, 4, 1080, 1080, 0.005), 3072 * 4),
    "T0": lambda: (_scene(4, 2, 1, 64, 64, 0.5), 0),
    "empty_first_list": lambda: ([(np.ones((1, 64, 64), np.float32),) + tuple(np.zeros(0, np.int64) for _ in range(3))
                                  + (np.zeros((0, 3), np.float32),)] + _scene(5, 1, 1, 64, 64, 0.5), 100),
    "all_zero_masks": lambda: ([(np.zeros_like(s[0]),) + s[1:] for s in _scene(6, 2, 2, 64, 64, 0.5)], 10),
    "nan_masks": lambda: (_scene(7, 2, 2, 128, 128, 0.6, nan=0.5), 500),
    "ragged_blocks": lambda: ([_scene(8, 1, 1, 64, 64, 0, P=P)[0] for P in (1, 255, 256, 257, 511, 1025, 4097)], 50),
    "G9_two_groups": lambda: (_scene(9, 9, 2, 96, 96, 0.5), 800),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_bit_identical_to_the_oracle(case):
    scene, target = CASES[case]()
    got, want = _check(scene, target, SEED, (1 << 32) - 1000 if case == "G2_N4_1080" else 77)
    if case == "T0" or case == "all_zero_masks":
        assert all(len(k) == 0 for k, _ in want)
    if case == "G2_N4_1080":
        assert all(_pnum(scene, g) > target for g in range(2))
    if case == "G2_N4_1080_keep_all":
        assert all(0 < _pnum(scene, g) <= target for g in range(2))


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_pnum_just_below_at_and_just_above_target(delta):
    scene = _scene(10, 2, 1, 200, 200, 0.5)
    target = _pnum(scene, 0) - delta           # pnum = T - 1, T, T + 1 for garment 0
    got, want = _check(scene, target, SEED, 5)
    n0 = len(want[0][0])
    if delta <= 0:
        assert n0 == _pnum(scene, 0)            # no draw: every candidate
    else:
        assert n0 < _pnum(scene, 0)


def test_lists_longer_than_2_pow_24_rows():
    scene = _scene(11, 1, 16, 1080, 1080, 0, mask_p=(0.3, 0.6, 0.1), P=(1 << 24) + 4097)
    assert len(scene[0][1]) > 1 << 24
    _check(scene, 1 << 22, SEED, 3)


def test_repeat_calls_are_bit_identical():
    scene = _scene(12, 2, 4, 1080, 1080, 0.3)
    a = _run(scene, 8192, SEED, 99)
    b = _run(scene, 8192, SEED, 99)
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert torch.equal(u.view(torch.uint8) if u.dtype == torch.float32 else u,
                               v.view(torch.uint8) if v.dtype == torch.float32 else v)


def test_keep_rate_is_binomial():
    scene = _scene(13, 1, 4, 1080, 1080, 0.5)
    pnum, target = _pnum(scene), 6144 * 4
    kept = len(_run(scene, target, SEED, 0)[0][0])
    p = float(tro.threshold(target, pnum))
    assert stats.binomtest(kept, pnum, p).pvalue > 1e-4, (kept, pnum, p)


def test_rays_equal_the_fragment_decode_and_the_torch_expression():
    N, H, W = 2, 1080, 1080
    g = np.random.default_rng(14)
    covered = g.uniform(size=(N, H, W)) < 0.3
    p2f = torch.from_numpy(np.where(covered, 0, -1)).to(DEV).view(N, H, W, 1).long()
    bary = torch.full((N, H, W, 1, 3), 1.0 / 3.0, device=DEV)
    verts = torch.tensor([[0., 0., 0.], [1., 0., 0.], [0., 1., 0.]], device=DEV)
    faces = torch.tensor([[0, 1, 2]], device=DEV)
    R = CAM[4:13].reshape(3, 3)
    b, r, c, p, _, rays = ops.fragment_decode(p2f, bary, verts, faces, None, (*CAM[:4].tolist(), torch.tensor(R)))
    ones = torch.ones((N, H, W), device=DEV)
    kb, kr, kc, kp, krays = ops.train_rays_sample([b], [r], [c], [p], [ones], torch.tensor(CAM, device=DEV),
                                                  1 << 40, SEED)[0]
    assert torch.equal(kb, b) and torch.equal(kr, r) and torch.equal(kc, c)
    assert torch.equal(krays.view(torch.int32), rays.view(torch.int32))
    # CameraMine.view_rays as torch evaluates it on the GPU
    f, pp, Rt = torch.tensor(CAM[:2], device=DEV), torch.tensor(CAM[2:4], device=DEV), torch.tensor(R, device=DEV)
    ps = torch.cat([kc.view(-1, 1), kr.view(-1, 1), torch.ones_like(kc.view(-1, 1))], -1).float()
    v = torch.zeros_like(ps)
    v[:, 0] = -ps[:, 0] / f[0] + ps[:, 2] * pp[0] / f[0]
    v[:, 1] = -ps[:, 1] / f[1] + ps[:, 2] * pp[1] / f[1]
    v[:, 2] = ps[:, 2]
    v = (v / torch.norm(v, p=2, dim=1, keepdim=True)).matmul(Rt.transpose(0, 1))
    assert float((krays - v).abs().max()) <= 1e-6


def test_bad_arguments_raise():
    scene = _scene(15, 1, 1, 16, 16, 0.5)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.train_rays_sample([torch.from_numpy(scene[0][1])], [torch.from_numpy(scene[0][2])],
                              [torch.from_numpy(scene[0][3])], [torch.from_numpy(scene[0][4])],
                              [torch.from_numpy(scene[0][0])], torch.tensor(CAM, device=DEV), 10, 0)
    t = lambda x: torch.from_numpy(x).to(DEV)  # noqa: E731
    with pytest.raises(RuntimeError, match="row"):
        ops.train_rays_sample([t(scene[0][1])], [t(scene[0][2][:-1])], [t(scene[0][3])], [t(scene[0][4])],
                              [t(scene[0][0])], torch.tensor(CAM, device=DEV), 10, 0)
    assert ops.train_rays_sample([], [], [], [], [], torch.tensor(CAM, device=DEV), 10, 0) == []


# ---- the drop-in -------------------------------------------------------------------------------------------------
class RectifiedPerspectiveCameras:
    """Stands in for the reference's camera class (looked up in the bound class's module): its parameters and its
    `view_rays` formula (model/CameraMine.py:146-167)."""

    def __init__(self, focal_length, principal_point, R, T, image_size=None):
        self.focal_length, self.principal_point, self.R, self.T = focal_length, principal_point, R, T

    def to(self, device):
        return self

    def view_rays(self, ps, cam_id=0):
        rays = torch.zeros_like(ps)
        rays[:, 0] = -ps[:, 0] / self.focal_length[cam_id, 0] + ps[:, 2] * self.principal_point[cam_id, 0] / self.focal_length[cam_id, 0]
        rays[:, 1] = -ps[:, 1] / self.focal_length[cam_id, 1] + ps[:, 2] * self.principal_point[cam_id, 1] / self.focal_length[cam_id, 1]
        rays[:, 2] = ps[:, 2]
        rays = rays / torch.norm(rays, p=2, dim=1, keepdim=True)
        return rays.matmul(self.R[cam_id].transpose(0, 1))


class _Net:
    sample_train_ray = make_sample_train_ray()


assert sys.modules[_Net.__module__].RectifiedPerspectiveCameras is RectifiedPerspectiveCameras


class _Conf:
    def __init__(self, d):
        self.d = d

    def get_int(self, key):
        return int(self.d[key])

    def __contains__(self, key):
        return key in self.d


def _self(z, name, pc=True, grad=False):
    k = lambda s: z[f"{name}/{s}"]  # noqa: E731
    cam = [torch.tensor(k(s), device=DEV) for s in ("focal", "pp", "R", "T")]
    if grad:
        cam[0].requires_grad_(True)
        cam[2].requires_grad_(True)
    H, W = k("mask_0").shape[1:]

    def get_camera_parameters(n, dev):
        return (cam[0].view(1, 2).expand(n, 2), cam[1].view(1, 2).expand(n, 2), cam[2].view(1, 3, 3).expand(n, 3, 3),
                cam[3].view(1, 3).expand(n, 3), H, W)

    s = _Net()
    s.conf = _Conf({} if int(k("conf_pix")) < 0 else {"sample_pix_num": int(k("conf_pix"))})
    s.garment_size = int(k("garment_size"))
    s.dataset = types.SimpleNamespace(get_camera_parameters=get_camera_parameters)
    s.maskRender = types.SimpleNamespace(rasterizer=types.SimpleNamespace(cameras=None))
    s.pcRender = types.SimpleNamespace(rasterizer=types.SimpleNamespace(cameras=None)) if pc else None
    args = [int(k("N")), int(k("arg_pix"))] + [[torch.tensor(k(f"{x}_{g}"), device=DEV) for g in range(2)]
                                               for x in ("mask", "batch", "row", "col", "pts")]
    return s, args + [torch.arange(int(k("N")), device=DEV), DEV], cam


def _bound(z, name):
    fn = _Net.sample_train_ray
    fn.stream.update(seed=int(z[f"{name}/seed"]), offset=int(z[f"{name}/offset"]))
    return fn


@pytest.mark.parametrize("name", ["below", "above", "mixed"])
def test_drop_in_matches_the_reference(name):
    z = load_golden("train_rays_ref.npz")
    s, args, _ = _self(z, name, pc=name != "mixed")
    fn = _bound(z, name)
    out = s.sample_train_ray(*args)
    assert len(out) == 6 and all(len(x) == 2 for x in out[:5])
    cams = out[5]
    assert isinstance(cams, RectifiedPerspectiveCameras) and s.maskRender.rasterizer.cameras is cams
    if s.pcRender is not None:
        assert s.pcRender.rasterizer.cameras is cams
    assert fn.stream["offset"] == int(z[f"{name}/offset"]) + sum(len(z[f"{name}/batch_{g}"]) for g in range(2))
    for g in range(2):
        for j, key in enumerate(("batch", "row", "col", "pts")):
            assert _same(out[j][g].cpu().numpy(), z[f"{name}/ref_{key}_{g}"]), (g, key)
        assert float(np.abs(out[4][g].cpu().numpy() - z[f"{name}/ref_rays_{g}"]).max(initial=0)) <= 1e-6


def test_drop_in_learnable_camera_keeps_the_reference_graph():
    z = load_golden("train_rays_ref.npz")
    s, args, cam = _self(z, "above", grad=True)
    _bound(z, "above")
    out = s.sample_train_ray(*args)
    rays = out[4]
    assert all(r.requires_grad for r in rays)
    w = [torch.linspace(-1, 1, r.numel(), device=DEV).view_as(r) for r in rays]
    sum((r * x).sum() for r, x in zip(rays, w)).backward()
    gf, gR = cam[0].grad.clone(), cam[2].grad.clone()
    # the same expression on the reference's kept pixels
    f2, R2 = cam[0].detach().clone().requires_grad_(True), cam[2].detach().clone().requires_grad_(True)
    c2 = RectifiedPerspectiveCameras(f2.view(1, 2), cam[1].view(1, 2), R2.view(1, 3, 3), cam[3].view(1, 3))
    ref = [c2.view_rays(torch.stack([torch.tensor(z[f"above/ref_col_{g}"], device=DEV),
                                     torch.tensor(z[f"above/ref_row_{g}"], device=DEV),
                                     torch.ones(len(z[f"above/ref_col_{g}"]), dtype=torch.int64, device=DEV)],
                                    1).float()) for g in range(2)]
    sum((r * x).sum() for r, x in zip(ref, w)).backward()
    assert torch.equal(gf, f2.grad) and torch.equal(gR, R2.grad)
    assert float(gf.abs().max()) > 0 and float(gR.abs().max()) > 0
    for r, e in zip(rays, ref):
        assert torch.equal(r.detach(), e.detach())


def test_drop_in_repeats_from_the_same_stream_and_seeds_from_torch():
    z = load_golden("train_rays_ref.npz")
    runs = []
    for _ in range(2):
        torch.manual_seed(4321)
        _Net.sample_train_ray = make_sample_train_ray()
        s, args, _ = _self(z, "above")
        a = s.sample_train_ray(*args)
        b = s.sample_train_ray(*args)
        runs.append((s.sample_train_ray.stream["seed"], [x.cpu() for x in a[0] + a[3]], [x.cpu() for x in b[0] + b[3]]))
    assert runs[0][0] == runs[1][0]
    for x, y in zip(runs[0][1] + runs[0][2], runs[1][1] + runs[1][2]):
        assert torch.equal(x, y)
    assert not all(torch.equal(x, y) for x, y in zip(runs[0][1], runs[0][2]))    # the second call draws anew


def test_drop_in_reads_the_host_once():
    z = load_golden("train_rays_ref.npz")
    s, args, _ = _self(z, "above")
    _bound(z, "above")
    s.sample_train_ray(*args)                     # warm-up: workspace, pinned counters
    torch.cuda.synchronize()
    before = ops.launch_count()
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            s.sample_train_ray(*args)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [w for w in rec if str(w.message).startswith("called a synchronizing CUDA operation")]
    assert len(syncs) == 1, [str(w.message) for w in syncs]
    assert ops.launch_count() - before == 5
