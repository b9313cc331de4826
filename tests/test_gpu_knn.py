"""GPU tests of the nearest-neighbour kernel (csrc/knn.cu) and the layers over it (ops.KnnNearestFunction,
recmv_b200.knn, recmv_b200.utils.fl_proj_loss) against oracle/knn_oracle.py: the forward bit for bit against the
float32 restatement, the backward against the float64 closed form on the kernel's own idx, chamfer_distance against
the float64 formula, and fl_proj_loss against the reference's own function (tests/golden/fl_proj_ref.npz).

Bounds are about 3x the maxima measured on an H100 80GB HBM3 and are printed with the measured values:
DIST_F64 (kernel dists against the float64 minimum, relative to the largest distance of the sample), GRAD_TOL
(gradients against float64, relative to the sum of |terms| of each entry), CHAMFER_TOL / FL_TOL / FL_GRAD_TOL
(relative, chamfer values, the loss and its gradient against float64), LOOP_TOL (the same loss built per frame from
chamfer_distance calls, as the reference builds it)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import knn_oracle as ko
from recmv_b200 import _lib, ops
from recmv_b200.knn import chamfer_distance, knn_gather, knn_points
from recmv_b200.utils import fl_proj_loss

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

DIST_F64 = 5e-8       # measured 1.4e-8
GRAD_TOL = 3.5e-7     # measured 1.05e-7 (dp1 and the 1e4-query hub of dp2)
CHAMFER_TOL = 1e-6    # measured 1.2e-7 (values), 3.0e-7 (gradients)
FL_TOL = 2e-7         # measured 6.5e-8
FL_GRAD_TOL = 3e-7    # measured 1.0e-7
LOOP_TOL = 6e-7       # measured 1.8e-7 (value), 1.5e-7 (gradient): the per-frame loop sums in another order


def _cloud(g, N, P, D, scale=1.0):
    return (g.normal(size=(N, P, D)) * scale).astype(np.float32)


def _run(p1, p2, l1=None, l2=None):
    t = lambda a: torch.tensor(a, device=DEV)  # noqa: E731
    d, i = ops.knn_nearest(t(p1), t(p2), None if l1 is None else t(np.asarray(l1, dtype=np.int64)),
                           None if l2 is None else t(np.asarray(l2, dtype=np.int64)))
    torch.cuda.synchronize()
    return d.cpu().numpy(), i.cpu().numpy()


def _bit_equal(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


CASES = [   # (N, P1, P2, ragged)
    (1, 1, 1, False),
    (1, 255, 257, False),
    (3, 300, 517, True),
    (64, 37, 259, True),
    (2, 1000, 5000, True),     # splits of P2
    (1, 3000, 100000, False),  # many splits
]


@pytest.mark.parametrize("D", [2, 3])
@pytest.mark.parametrize("N,P1,P2,ragged", CASES)
def test_forward_bit_exact(D, N, P1, P2, ragged):
    g = np.random.default_rng(N * 7 + P1 + D)
    p1, p2 = _cloud(g, N, P1, D), _cloud(g, N, P2, D)
    # duplicated candidates and queries that sit exactly on a candidate: exact ties
    p2[:, P2 // 2] = p2[:, 0]
    p1[:, 0] = p2[:, P2 // 2]
    l1 = l2 = None
    if ragged:
        l1 = g.integers(0, P1 + 1, size=N)
        l2 = g.integers(0, P2 + 1, size=N)
        l1[0], l2[-1] = 0, 0
        if N > 2:
            l1[1], l2[1] = 1, 1
            l1[2], l2[2] = P1 + 5, -3   # clamped to [0, P]
    d, i = _run(p1, p2, l1, l2)
    rd, ri = ko.nearest_f32(p1, p2, l1, l2)
    assert np.array_equal(i, ri)
    assert _bit_equal(d, rd)
    if not ragged:
        assert np.all(i[:, 0] == 0)   # the query on the duplicated point takes the lower index


def test_forward_1e5_by_1e5():
    g = np.random.default_rng(11)
    P = 100000
    p1, p2 = _cloud(g, 1, P, 3), _cloud(g, 1, P, 3)
    d, i = _run(p1, p2)
    rows = np.sort(g.choice(P, 2000, replace=False))
    rd, ri = ko.nearest_f32(p1, p2, rows=rows)
    assert np.array_equal(i[0, rows], ri[0, rows])
    assert _bit_equal(d[0, rows], rd[0, rows])
    q = p1[0, rows].astype(np.float64)
    d64 = np.empty(len(rows))
    for s in range(0, len(rows), 250):
        d64[s:s + 250] = ((q[s:s + 250, None] - p2[0, None].astype(np.float64)) ** 2).sum(-1).min(1)
    err = np.abs(d[0, rows] - d64).max() / d64.max()
    print(f"1e5 x 1e5: max |d - d64| / max d64 = {err:.2e} (bound {DIST_F64:.0e})")
    assert err < DIST_F64
    assert np.all((i >= 0) & (i < P))


def test_non_finite_coordinates_keep_the_index_in_range():
    g = np.random.default_rng(2)
    p1, p2 = _cloud(g, 2, 300, 3), _cloud(g, 2, 400, 3)
    p1[0, :10] = np.nan
    p1[0, 10:20] = np.inf
    p2[1, ::3] = np.nan
    p2[1, 1::3] = -np.inf
    l2 = np.array([400, 350])
    d, i = _run(p1, p2, None, l2)
    assert np.all((i >= 0) & (i < l2[:, None]))


def test_outputs_stay_inside_guarded_buffers():
    g = np.random.default_rng(4)
    N, P1, P2, D, G = 3, 333, 129, 3, 64
    p1 = torch.tensor(_cloud(g, N, P1, D), device=DEV)
    p2 = torch.tensor(_cloud(g, N, P2, D), device=DEV)
    l1 = torch.tensor([333, 0, 100], device=DEV)
    l2 = torch.tensor([129, 5, 0], device=DEV)
    lib = _lib.load()
    nbytes = ctypes.c_size_t(0)
    assert lib.recmv_knn_workspace_bytes(N, P1, P2, ctypes.byref(nbytes)) == 0
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=DEV)
    dist = torch.full((N * P1 + 2 * G,), float("nan"), device=DEV)
    idx = torch.full((N * P1 + 2 * G,), -7, dtype=torch.int64, device=DEV)
    g1 = torch.full((N * P1 * D + 2 * G,), float("nan"), device=DEV)
    g2 = torch.full((N * P2 * D + 2 * G,), float("nan"), device=DEV)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ptr = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off * t.element_size())  # noqa: E731
    assert lib.recmv_knn_nearest(ptr(p1), ptr(p2), ptr(l1), ptr(l2), N, P1, P2, D, ptr(ws), ptr(dist, G), ptr(idx, G),
                                 st) == 0
    grad = torch.rand(N, P1, device=DEV)
    assert lib.recmv_knn_nearest_backward(ptr(p1), ptr(p2), ptr(idx, G), ptr(grad), N, P1, P2, D, ptr(ws),
                                          ptr(g1, G), ptr(g2, G), st) == 0
    torch.cuda.synchronize()
    for t, fill in ((dist, None), (g1, None), (g2, None), (idx, -7)):
        head, tail = t[:G], t[-G:]
        if fill is None:
            assert torch.isnan(head).all() and torch.isnan(tail).all()
            assert not torch.isnan(t[G:-G]).any()
        else:
            assert (head == fill).all() and (tail == fill).all() and (t[G:-G] >= -1).all()
    rd, ri = ko.nearest_f32(p1.cpu().numpy(), p2.cpu().numpy(), l1.cpu().numpy(), l2.cpu().numpy())
    assert np.array_equal(idx[G:-G].view(N, P1).cpu().numpy(), ri)


def _grad_err(got, want, scale):
    return float((np.abs(got - want) / np.maximum(scale, 1e-30)).max())


def _abs_scale(p1, p2, idx, grad):
    a1, a2 = ko.nearest_backward_f64(np.abs(p1), -np.abs(p2), idx, np.abs(grad))   # sum of |terms| per entry
    return np.abs(a1), np.abs(a2)


@pytest.mark.parametrize("D", [2, 3])
def test_backward_against_closed_form_with_a_hub(D):
    g = np.random.default_rng(20 + D)
    N, P1, P2 = 2, 12000, 3000
    p2 = _cloud(g, N, P2, D, scale=10.0)
    p2[:, 7] = 0.0                                    # the hub: 1e4 queries cluster around candidate 7
    p1 = _cloud(g, N, P1, D, scale=10.0)
    p1[:, :10000] = _cloud(g, N, 10000, D, scale=1e-3)
    l1, l2 = np.array([P1, 11000]), np.array([P2, 2500])
    t1 = torch.tensor(p1, device=DEV, requires_grad=True)
    t2 = torch.tensor(p2, device=DEV, requires_grad=True)
    gd = torch.tensor(g.normal(size=(N, P1)).astype(np.float32), device=DEV)
    L1, L2 = torch.tensor(l1, device=DEV), torch.tensor(l2, device=DEV)
    runs = []
    for _ in range(2):
        d, i = ops.KnnNearestFunction.apply(t1, t2, L1, L2)
        g1, g2 = torch.autograd.grad(d, (t1, t2), gd)
        runs.append((g1.cpu().numpy(), g2.cpu().numpy(), i.cpu().numpy()))
    assert np.array_equal(runs[0][0].view(np.uint32), runs[1][0].view(np.uint32))
    assert np.array_equal(runs[0][1].view(np.uint32), runs[1][1].view(np.uint32))
    g1, g2, idx = runs[0]
    assert (idx[:, :10000] == 7).all()
    w1, w2 = ko.nearest_backward_f64(p1, p2, idx, gd.cpu().numpy())
    s1, s2 = _abs_scale(p1.astype(np.float64), p2.astype(np.float64), idx, gd.cpu().numpy())
    e1, e2 = _grad_err(g1, w1, s1), _grad_err(g2, w2, s2)
    print(f"D={D} backward: dp1 err {e1:.2e}, dp2 err {e2:.2e} (relative to sum |terms|; bound {GRAD_TOL:.0e})")
    assert e1 < GRAD_TOL and e2 < GRAD_TOL
    assert np.all(g1[1, 11000:] == 0) and np.all(g2[1, 2500:] == 0)


@pytest.mark.parametrize("point_reduction", ["sum", "mean"])
@pytest.mark.parametrize("batch_reduction", [None, "sum", "mean"])
def test_chamfer_distance_against_float64(batch_reduction, point_reduction):
    g = np.random.default_rng(31)
    N = 4
    x, y = _cloud(g, N, 150, 2, 50.0), _cloud(g, N, 90, 2, 50.0)
    lx, ly = np.array([150, 1, 77, 150]), np.array([90, 90, 13, 1])
    tx = torch.tensor(x, device=DEV, requires_grad=True)
    ty = torch.tensor(y, device=DEV, requires_grad=True)
    got, none = chamfer_distance(tx, ty, torch.tensor(lx, device=DEV), torch.tensor(ly, device=DEV),
                                 batch_reduction=batch_reduction, point_reduction=point_reduction)
    assert none is None
    rx = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    ry = torch.tensor(y, dtype=torch.float64, requires_grad=True)
    want = ko.chamfer_f64(rx, ry, torch.tensor(lx), torch.tensor(ly), batch_reduction=batch_reduction,
                          point_reduction=point_reduction)[0]
    err = float(((got.detach().cpu().double() - want.detach()).abs() / want.detach().abs()).max())
    gw = torch.randn(want.shape, dtype=torch.float64)
    gx, gy = torch.autograd.grad(got, (tx, ty), gw.float().to(DEV))
    wx, wy = torch.autograd.grad(want, (rx, ry), gw)
    ge = max(float((a.cpu().double() - b).abs().max() / b.abs().max()) for a, b in ((gx, wx), (gy, wy)))
    print(f"chamfer {batch_reduction}/{point_reduction}: value err {err:.2e}, grad err {ge:.2e}")
    assert err < CHAMFER_TOL and ge < CHAMFER_TOL


def test_chamfer_empty_cloud_gives_nan_for_mean_and_zero_for_sum():
    x, y = torch.randn(2, 5, 2, device=DEV), torch.randn(2, 4, 2, device=DEV)
    lx = torch.tensor([5, 0], device=DEV)
    s = chamfer_distance(x, y, lx, None, batch_reduction=None, point_reduction="sum")[0]
    m = chamfer_distance(x, y, lx, None, batch_reduction=None, point_reduction="mean")[0]
    assert s[1].item() == 0 and torch.isnan(m[1]) and torch.isfinite(m[0])


def test_knn_points_and_gather_registration_shape():
    g = np.random.default_rng(8)
    src = torch.tensor(_cloud(g, 1, 40000, 3), device=DEV, requires_grad=True)
    tgt = torch.tensor(_cloud(g, 1, 30000, 3), device=DEV)
    nn = knn_points(src, tgt)
    assert nn.dists.shape == (1, 40000, 1) and nn.idx.shape == (1, 40000, 1) and nn.knn is None
    near = knn_gather(tgt, nn.idx)[:, :, 0]
    d = ((src - near) ** 2).sum(-1)
    assert torch.equal(d.detach().cpu() == 0, nn.dists[..., 0].cpu() == 0)
    nn.dists.sum().backward()
    assert torch.allclose(src.grad, 2 * (src - near).detach(), rtol=0, atol=1e-5)


def _fixture(golden, N=None, curves=None):
    z = golden("fl_proj_ref.npz")
    C = len(z["weights"])
    cs = list(range(C)) if curves is None else curves
    n = slice(None) if N is None else slice(0, N)
    pts = [torch.tensor(z[f"pts_{c}"][n], device=DEV, requires_grad=True) for c in cs]
    gts = [torch.tensor(z[f"gt_{c}"][n], device=DEV) for c in cs]
    masks = [torch.tensor(z[f"mask_{c}"][n], device=DEV)[..., None].expand(-1, -1, 3) for c in cs]
    return z, pts, gts, masks, [float(z["weights"][c]) for c in cs]


def test_fl_proj_loss_matches_the_reference(golden):
    z, pts, gts, masks, w = _fixture(golden)
    loss = fl_proj_loss(pts, gts, masks, w)
    grads = torch.autograd.grad(loss, pts)
    err = abs(loss.item() - float(z["loss"])) / abs(float(z["loss"]))
    ge = max(float(np.abs(gr.cpu().numpy() - z[f"grad_{c}"]).max() / np.abs(z[f"grad_{c}"]).max())
             for c, gr in enumerate(grads) if np.abs(z[f"grad_{c}"]).max() > 0)
    print(f"fl_proj_loss: value err {err:.2e} (bound {FL_TOL:.0e}), grad err {ge:.2e} (bound {FL_GRAD_TOL:.0e})")
    assert err < FL_TOL and ge < FL_GRAD_TOL
    assert all(float(gr[..., 2].abs().max()) == 0 for gr in grads)
    assert float(grads[3].abs().max()) == 0     # the invisible curve


def test_fl_proj_loss_has_no_host_synchronisation(golden):
    z, pts, gts, masks, w = _fixture(golden)
    fl_proj_loss(pts, gts, masks, w).backward()     # warm-up: workspace growth and lazy initialisation
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = fl_proj_loss(pts, gts, masks, w)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_fl_proj_launch_count_does_not_depend_on_frames_or_curves(golden):
    counts = {}
    for N in (1, 3):
        for curves in ([0, 4], [0, 1, 2, 3, 4, 5]):
            z, pts, gts, masks, w = _fixture(golden, N, curves)
            before = ops.launch_count()
            fl_proj_loss(pts, gts, masks, w).backward()
            counts[(N, len(curves))] = ops.launch_count() - before
    assert len(set(counts.values())) == 1, counts


def test_chamfer_with_an_empty_cloud_back_propagates():
    # the reference's per-frame call on a frame with no visible point: x = pts[mask].view(1, -1, 2) with an all-False
    # mask, an empty tensor whose data pointer may be NULL, that still requires grad
    pts = torch.randn(1, 6, 2, device=DEV, requires_grad=True)
    y = torch.randn(1, 4, 2, device=DEV, requires_grad=True)
    for x in (pts[torch.zeros(1, 6, 2, dtype=torch.bool, device=DEV)].view(1, -1, 2),
              torch.empty(1, 0, 2, device=DEV, requires_grad=True)):
        loss = chamfer_distance(x, y, point_reduction="sum")[0]
        gp, gy = torch.autograd.grad(loss, (pts, y), allow_unused=True)
        assert loss.item() == 0
        assert gy is not None and float(gy.abs().max()) == 0
        assert gp is None or float(gp.abs().max()) == 0
    # the same through the C ABI: P2 = 0 with a NULL candidate pointer is accepted by both directions
    lib = _lib.load()
    nbytes = ctypes.c_size_t(0)
    assert lib.recmv_knn_workspace_bytes(1, 4, 0, ctypes.byref(nbytes)) == 0
    ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=DEV)
    d = torch.full((1, 4), float("nan"), device=DEV)
    i = torch.full((1, 4), -7, dtype=torch.int64, device=DEV)
    g1 = torch.full((1, 4, 2), float("nan"), device=DEV)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    y2 = y.detach().contiguous()
    assert lib.recmv_knn_nearest(p(y2), None, None, None, 1, 4, 0, 2, p(ws), p(d), p(i), st) == 0
    assert lib.recmv_knn_nearest_backward(p(y2), None, p(i), p(torch.ones(1, 4, device=DEV)), 1, 4, 0, 2, p(ws), p(g1),
                                          None, st) == 0
    torch.cuda.synchronize()
    assert (i == -1).all() and (d == 0).all() and (g1 == 0).all()


def test_per_frame_chamfer_loop_matches_the_reference(golden):
    # the reference's fl_proj_loss structure, one chamfer_distance call per frame and curve on the boolean-selected
    # visible points (point_reduction="sum"), including the frame and the curve with no visible point
    z, pts, gts, masks, w = _fixture(golden)
    loss = 0.0
    for p, gt, m, wc in zip(pts, gts, masks, w):
        vis = m[..., 0]
        S = sum(chamfer_distance(p[n][vis[n]][:, :2].view(1, -1, 2), gt[n].view(1, -1, 2), point_reduction="sum")[0]
                for n in range(p.shape[0]))
        V, Q = int((vis.sum(1) > 0).sum()), int(vis.sum())
        loss = loss + wc * S / max(V, 1) / max(Q, 1)
    loss = loss / len(pts)
    grads = torch.autograd.grad(loss, pts)
    err = abs(loss.item() - float(z["loss"])) / abs(float(z["loss"]))
    ge = max(float(np.abs(gr.cpu().numpy() - z[f"grad_{c}"]).max() / np.abs(z[f"grad_{c}"]).max())
             for c, gr in enumerate(grads) if np.abs(z[f"grad_{c}"]).max() > 0)
    print(f"per-frame chamfer loop: value err {err:.2e}, grad err {ge:.2e} (bound {LOOP_TOL:.0e})")
    assert err < LOOP_TOL and ge < LOOP_TOL


@pytest.mark.parametrize("D", [2, 3])
def test_strided_inputs_are_accepted(D):
    g = np.random.default_rng(40 + D)
    a = torch.tensor(_cloud(g, 2, 300, 4), device=DEV)
    b = torch.tensor(_cloud(g, 2, 200, 4), device=DEV)
    sa, sb = a[..., :D], b[:, ::2, 1:1 + D]
    assert not sa.is_contiguous() and not sb.is_contiguous()
    got, want = knn_points(sa, sb), knn_points(sa.contiguous(), sb.contiguous())
    assert torch.equal(got.idx, want.idx) and torch.equal(got.dists, want.dists)
    assert torch.equal(chamfer_distance(sa, sb)[0], chamfer_distance(sa.contiguous(), sb.contiguous())[0])
