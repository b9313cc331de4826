"""GPU tests of the surface sampler (csrc/surface_sample.cu, DESIGN section 1h) and the curve-aware drop-in
(recmv_b200.utils.make_curve_aware_loss): every sample bit for bit against the float64 oracle (oracle/sample_oracle.py)
rounded to float32, the stream's batching and offset rules, run-to-run identity, and the drop-in against the
reference's own `curve_aware_loss` (tests/golden/curve_aware_ref.npz, tests/golden/make_golden_curve_aware.py).

Bounds of the drop-in (max |a - b| / max |b| per tensor, as tests/test_gpu_train.py measures): the loss within
LOSS_TOL; the SDF parameters' gradients within GRAD_TOL = the training tolerance 3e-5 plus three samples whose
|sdf + r| changes sign between the tensor-core network and the reference's fp32 CPU run (each moves 2/S of the
cotangent mass, 4e-5 of the gradient at S = 50 000)."""
import types

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import sample_oracle as so
from recmv_b200 import ops, raster, testing
from recmv_b200.model import getTmpSdf
from recmv_b200.utils import make_curve_aware_loss

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CURVE_AWARE = {'female_outfit1': 'bottom_curve', 'female_outfit3': 'bottom_curve', 'anran_dance': 'bottom_curve'}
LOSS_TOL = 1e-5
GRAD_TOL = 3e-5 + 3 * 2 / 50000
SEED = 0x9E3779B97F4A7C15


@pytest.fixture(autouse=True)
def _no_aborted_launch():
    yield
    torch.cuda.synchronize()
    ops.check_async_errors()


def _same(a, b):
    """Bit equality, NaN included."""
    a, b = np.ascontiguousarray(a, dtype=np.float32), np.ascontiguousarray(b, dtype=np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _gpu(verts, faces, S, seed=SEED, offset=0):
    v = torch.tensor(np.asarray(verts, dtype=np.float32), device=DEV)
    f = torch.tensor(np.asarray(faces, dtype=np.int64), device=DEV)
    return ops.surface_sample(v.reshape(-1, v.shape[-2], 3).contiguous(), f, S, seed, offset).cpu().numpy()


def _grid_mesh(n, seed):
    """An n x n height-field sheet: 2 (n-1)^2 faces of unequal areas."""
    g = np.random.default_rng(seed)
    x, y = np.meshgrid(np.linspace(0, 1, n) ** 1.5, np.linspace(0, 2, n))
    z = 0.1 * g.standard_normal((n, n))
    v = np.stack([x, y, z], -1).reshape(-1, 3).astype(np.float32)
    i = np.arange(n * n).reshape(n, n)
    a, b, c, d = i[:-1, :-1].ravel(), i[:-1, 1:].ravel(), i[1:, :-1].ravel(), i[1:, 1:].ravel()
    return v, np.concatenate([np.stack([a, b, c], 1), np.stack([b, d, c], 1)]).astype(np.int64)


def _fan_of(seed, P=200):
    g = np.random.default_rng(seed)
    t = np.linspace(0, 2 * np.pi, P, endpoint=False)
    r = 0.5 + 0.1 * np.sin(5 * t) + 0.02 * g.standard_normal(P)
    return so.fan(np.stack([r * np.cos(t), 0.05 * g.standard_normal(P), r * np.sin(t)], 1))


def _degenerate():
    v, f = _grid_mesh(9, 3)
    f = f.copy()
    v[f[5]] = v[f[5, 0]]            # zero area
    f[9, 0] = -3                    # invalid index
    f[17, 2] = len(v)               # invalid index
    v[f[20, 1]] = np.nan            # non-finite area
    return v, f


CASES = {
    "one_triangle": lambda: (np.array([[[0, 0, 0], [1, 0, 0], [0.25, 2, 0.5]]], np.float32), np.array([[0, 1, 2]]),
                             4096, 0),
    "fan_200_S50000": lambda: (_fan_of(1)[0][None], _fan_of(1)[1], 50000, 77),
    "fan_M3_one_launch": lambda: (np.stack([_fan_of(s)[0] for s in (2, 3, 4)]), _fan_of(2)[1], 20000, (1 << 32) - 30000),
    "S1": lambda: (_fan_of(5)[0][None], _fan_of(5)[1], 1, 5),
    "S_ragged": lambda: (_fan_of(6)[0][None], _fan_of(6)[1], 777, 0),
    "degenerate_faces": lambda: (_degenerate()[0][None], _degenerate()[1], 30000, 0),
    "all_degenerate": lambda: (np.zeros((1, 4, 3), np.float32), np.array([[0, 1, 2], [1, 2, 3]]), 300, 0),
    "all_degenerate_invalid_face0": lambda: (np.zeros((1, 4, 3), np.float32), np.array([[0, 1, 4], [1, 2, 3]]), 300, 0),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_bit_identical_to_the_oracle(case):
    verts, faces, S, offset = CASES[case]()
    got = _gpu(verts, faces, S, SEED, offset)
    want = so.sample_surface(verts, faces, S, SEED, offset).astype(np.float32)
    assert _same(got, want), f"{case}: {int((got.view(np.uint32) != want.view(np.uint32)).any(-1).sum())} samples differ"
    if case == "all_degenerate_invalid_face0":
        assert np.isnan(got).all()
    if case == "degenerate_faces":
        assert np.isfinite(got).all()


def test_2e5_faces_at_1e6_samples():
    v, f = _grid_mesh(317, 8)              # 2 * 316^2 = 199 712 faces, 781 chunks
    assert len(f) > 199_000
    got = _gpu(v[None], f, 1_000_000, SEED, 123456789)
    want = so.sample_surface(v[None], f, 1_000_000, SEED, 123456789).astype(np.float32)
    assert _same(got, want)
    again = _gpu(v[None], f, 1_000_000, SEED, 123456789)
    assert _same(got, again)


def test_batched_equals_sequential_and_split_equals_whole():
    verts = np.stack([_fan_of(s)[0] for s in (7, 8, 9)])
    faces = _fan_of(7)[1]
    S, off = 5000, 31
    whole = _gpu(verts, faces, S, SEED, off)
    for m in range(3):
        assert _same(whole[m], _gpu(verts[m][None], faces, S, SEED, off + m * S)[0])
    S1 = 1234
    a = _gpu(verts[:1], faces, S1, SEED, off)
    b = _gpu(verts[:1], faces, S - S1, SEED, off + S1)
    assert _same(np.concatenate([a[0], b[0]]), whole[0])


def test_raster_sample_surface_is_the_op():
    v, f = _fan_of(10)
    vt = torch.tensor(v, device=DEV)[None]
    ft = torch.tensor(f, device=DEV)
    assert _same(raster.sample_surface(vt, ft, 999, seed=3, offset=4).cpu().numpy(),
                 ops.surface_sample(vt, ft, 999, 3, 4).cpu().numpy())


def test_cpu_tensors_and_empty_faces_raise():
    v, f = _fan_of(11)
    with pytest.raises(RuntimeError, match="CUDA"):
        raster.sample_surface(torch.tensor(v)[None], torch.tensor(f), 10)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.surface_sample(torch.tensor(v)[None], torch.tensor(f), 10, 0, 0)
    with pytest.raises(RuntimeError):
        ops.surface_sample(torch.tensor(v, device=DEV)[None], torch.tensor(f), 10, 0, 0)   # CPU faces
    with pytest.raises(RuntimeError, match="empty"):
        ops.surface_sample(torch.tensor(v, device=DEV)[None], torch.zeros((0, 3), dtype=torch.int64, device=DEV), 10,
                           0, 0)


# ---- the drop-in -------------------------------------------------------------------------------------------------
class _Conf:
    def __init__(self, d):
        self.d = d

    def get_float(self, key):
        v = self.d
        for k in key.split("."):
            v = v[k]
        return float(v)

    def __contains__(self, key):
        return key in self.d


class _Curves:
    def __init__(self, pts):
        self.pts = pts

    def forward(self):
        return self.pts


def _net():
    return testing.build_sdf(getTmpSdf, seed=0, perturb_seed=101).to(DEV)


def _make(z, name, net, isfine=None, weight=None):
    """The method's `self` for one fixture case, its curves on the GPU."""
    k = lambda s: z[f"{name}/{s}"]  # noqa: E731
    return types.SimpleNamespace(
        conf=_Conf({"pc_weight": {"curve_aware_weight": float(k("weight")) if weight is None else weight}}),
        fl_names=[str(s) for s in k("fl_names")], garment_type=str(k("garment_type")),
        isfine=bool(k("isfine")) if isfine is None else isfine,
        inter_free_curve=_Curves(torch.tensor(k("curves"), device=DEV)), garment_nets=[net],
        sdfShrinkRadius=float(k("shrink")), info={})


def _merr(a, b):
    a = torch.as_tensor(a, dtype=torch.float64).detach().cpu()
    b = torch.as_tensor(b, dtype=torch.float64).detach().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


@pytest.mark.parametrize("name", ["one", "two", "fallthrough"])
def test_drop_in_matches_the_reference(name):
    z = load_golden("curve_aware_ref.npz")
    net = _net()
    s = _make(z, name, net)
    fn = make_curve_aware_loss(CURVE_AWARE)
    fn.stream.update(seed=int(z[f"{name}/seed"]), offset=int(z[f"{name}/offset"]))
    loss = fn(s, {"sdfRatio": 0.7})
    assert net.last_path == "fused-train"
    loss.backward()
    terms = [str(t) for t in z[f"{name}/terms"]]
    assert list(s.info) == terms
    assert fn.stream["offset"] == int(z[f"{name}/offset"]) + 50000 * len(terms)
    rows = [("loss", _merr(loss, z[f"{name}/loss"]), LOSS_TOL)]
    rows += [(t, _merr(s.info[t], z[f"{name}/term_loss"][i]), LOSS_TOL) for i, t in enumerate(terms)]
    for l in range(9):
        lin = getattr(net, f"lin{l}")
        rows.append((f"lin{l}.bias", _merr(lin.bias.grad, z[f"{name}/lin{l}_bias"]), GRAD_TOL))
        rows.append((f"lin{l}.weight_g", _merr(lin.weight_g.grad, z[f"{name}/lin{l}_weight_g"]), GRAD_TOL))
        rows.append((f"lin{l}.weight_v", _merr(lin.weight_v.grad[::32, ::16], z[f"{name}/lin{l}_weight_v"]), GRAD_TOL))
    table = "\n".join(f"{name}/{n}: {e:.2e} (bound {b:.1e})" for n, e, b in rows)
    print(table)
    assert all(e <= b for _, e, b in rows), table
    # the points themselves: the reference's fans (its own centroids) through the kernel give its samples bit for bit
    fans = torch.tensor(np.stack([z[f"{name}/fan_{t}"] for t in range(len(terms))]), device=DEV)
    P = fans.shape[1] - 1
    i = torch.arange(P, device=DEV)
    faces = torch.stack([i, (i + 1) % P, torch.full_like(i, P)], 1)
    pts = ops.surface_sample(fans, faces, 50000, int(z[f"{name}/seed"]), int(z[f"{name}/offset"])).cpu().numpy()
    for t in range(len(terms)):
        assert _same(pts[t, ::50], z[f"{name}/samples_{t}"])


def test_drop_in_isfine_off_and_weight_zero():
    z = load_golden("curve_aware_ref.npz")
    net = _net()
    fn = make_curve_aware_loss(CURVE_AWARE)
    fn.stream.update(seed=int(z["two/seed"]), offset=int(z["two/offset"]))
    s = _make(z, "two", net, isfine=False)
    loss = fn(s, {"sdfRatio": 0.7})
    assert list(s.info) == ["pc_upper_bottom_circle_loss_sdf"]
    want = float(z["two/term_loss"][0]) * float(z["two/weight"])
    assert abs(loss.item() - want) <= LOSS_TOL * abs(want)
    before = ops.launch_count()
    s0 = _make(z, "two", net, weight=0.0)
    assert fn(s0, {"sdfRatio": 0.7}) == 0. and s0.info == {}
    assert ops.launch_count() == before


def test_drop_in_has_no_host_synchronisation():
    z = load_golden("curve_aware_ref.npz")
    net = _net()
    fn = make_curve_aware_loss(CURVE_AWARE)
    fn(_make(z, "two", net), {"sdfRatio": 0.7}).backward()    # warm-up: seed draw, workspace growth, weight packing
    s = _make(z, "two", net)                                  # its curves' upload synchronises, outside the window
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = fn(s, {"sdfRatio": 0.7})
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_drop_in_launch_count_does_not_depend_on_the_curves():
    z = load_golden("curve_aware_ref.npz")
    net = _net()
    fn = make_curve_aware_loss(CURVE_AWARE)
    fn(_make(z, "two", net), {"sdfRatio": 0.7}).backward()
    counts = {}
    for name in ("one", "two"):
        before = ops.launch_count()
        fn(_make(z, name, net), {"sdfRatio": 0.7}).backward()
        counts[name] = ops.launch_count() - before
    assert counts["one"] == counts["two"], counts


def test_drop_in_seed_comes_from_torch_and_the_stream_advances():
    z = load_golden("curve_aware_ref.npz")
    net = _net()
    runs = []
    for _ in range(2):
        torch.manual_seed(1234)
        fn = make_curve_aware_loss(CURVE_AWARE)
        a = fn(_make(z, "two", net), {"sdfRatio": 0.7}).detach()
        b = fn(_make(z, "two", net), {"sdfRatio": 0.7}).detach()
        runs.append((fn.stream["seed"], a.item(), b.item()))
        assert fn.stream["offset"] == 4 * 50000
    assert runs[0] == runs[1]
    assert runs[0][1] != runs[0][2]      # the second call draws new points
