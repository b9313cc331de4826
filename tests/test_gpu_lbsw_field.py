"""GPU tests of the skinning-voxel construction (csrc/lbsw_field.cu): the kNN blend and the smoothing kernel against
float64, end to end against the reference's own output (tests/golden/lbsw_ref.npz), bit-exact repeatability, output
bounds, and the skinner built from a body."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(HERE, "golden"))

from make_golden_lbsw import CASES  # noqa: E402
from oracle import lbsw_torch as lt  # noqa: E402
from recmv_b200 import _lib, ops, synth, utils  # noqa: E402
from recmv_b200.model import Deformer  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
G = np.load(os.path.join(HERE, "golden", "lbsw_ref.npz"))
BMIN, BMAX = G["bmin"].tolist(), G["bmax"].tolist()
GAP = 1e-5      # float64 gap between the k-th and (k+1)-th distance above which the neighbour set is unambiguous


def body():
    v, w = synth.body_points()
    return v.to(DEV), w.to(DEV)


def f64_neighbours(res, ac, k, sel):
    """float64 distances of the voxels `sel`, sorted stably: (sorted distances [n,V], their indices [n,V])."""
    v, _ = synth.body_points()
    c = lt.voxel_centres(BMIN, BMAX, res, ac, torch.float64, DEV)[sel]
    d = (c[:, None, :] - v.double().to(DEV)[None]).norm(dim=-1)
    return torch.sort(d, dim=-1, stable=True)


KNN_SHAPES = [((13, 25, 9), False), ((13, 25, 9), True), ((13, 1, 9), False), ((1, 17, 6), False),
              ((129, 225, 65), False)]


@pytest.mark.parametrize("k", [1, 5, 30, 32])
@pytest.mark.parametrize("res,ac", KNN_SHAPES)
def test_knn_blend_vs_float64(res, ac, k):
    v, w = body()
    out, idx = ops.lbsw_knn_blend(v, w, BMIN, BMAX, res, k, ac, want_idx=True)
    N = res[0] * res[1] * res[2]
    g = torch.Generator().manual_seed(k)
    sel = torch.arange(N) if N <= 4096 else torch.randperm(N, generator=g)[:4096]
    sel = sel.to(DEV)
    ds, order = f64_neighbours(res, ac, k, sel)
    mine = idx[sel].long()
    # the chosen distances, in float64
    vd = v.double()
    c = lt.voxel_centres(BMIN, BMAX, res, ac, torch.float64, DEV)[sel]
    dmine = (c[:, None, :] - vd[mine]).norm(dim=-1)
    # nearest first, and no chosen vertex farther than an unchosen one (up to fp32 rounding of the distance)
    assert (dmine[:, 1:] >= dmine[:, :-1] - 1e-6).all()
    dk1 = ds[:, k] if k < ds.shape[1] else torch.full_like(ds[:, 0], float("inf"))
    assert (dmine.max(1).values <= dk1 + 1e-6).all()
    clear = (dk1 - ds[:, k - 1]) > GAP
    print(f"\n{res} ac={ac} k={k}: {int((~clear).sum())} of {len(sel)} voxels near a tie at the k-th distance")
    assert torch.equal(mine[clear].sort(1).values, order[clear, :k].sort(1).values)
    # blend of the kernel's own neighbour set in float64.  Measured on an H100: max |diff| 1.1e-6 (production grid,
    # k = 32), 2e-7 - 9.7e-7 elsewhere
    inv = 1.0 / dmine.clamp(1e-4, 1.0)
    wts = inv / inv.sum(1, keepdim=True)
    ref = (w.double()[mine] * wts[..., None]).sum(1)
    err = (out.view(N, 24)[sel].double() - ref).abs().max().item()
    print(f"  blend max |err| vs float64: {err:.3e}")
    assert err < 3.5e-6


def test_knn_ties_go_to_the_lower_index():
    v, w = body()
    V0 = 3000
    vv = torch.cat([v[:V0], v[:V0]]).contiguous()          # every distance twice: i and i + V0
    ww = torch.cat([w[:V0], w[:V0].flip(1)]).contiguous()
    for k in (1, 3, 8, 31):
        _, idx = ops.lbsw_knn_blend(vv, ww, BMIN, BMAX, (9, 13, 7), k, want_idx=True)
        rows = idx.tolist()
        for row in rows:
            assert row[0] < V0                               # the nearest distance: its lower copy comes first
            for p, j in enumerate(row):
                if j >= V0:                                  # an upper copy only after its lower copy
                    assert j - V0 in row[:p]


def random_field(shape, seed):
    D, H, W = shape
    g = torch.Generator().manual_seed(seed)
    x = torch.rand((1, 24, D, H, W), generator=g) ** 4
    return (x / x.sum(1, keepdim=True)).to(DEV)


@pytest.mark.parametrize("zero_below", [0.0, 5e-3])
@pytest.mark.parametrize("times", [0, 1, 2, 30])
@pytest.mark.parametrize("shape", [(9, 25, 13), (9, 2, 13), (1, 5, 6)])
def test_smooth_vs_float64(shape, times, zero_below):
    x = random_field(shape, 3 + times)
    out, out_cl = ops.lbsw_smooth(ops.voxel_to_channels_last(x), times, zero_below)
    assert torch.equal(out_cl, ops.voxel_to_channels_last(out))
    ref = lt.smooth_weights(x.double(), times, zero_below)
    f32 = lt.smooth_weights(x.cpu(), times, zero_below).to(DEV)
    err = (out.double() - ref).abs()
    near = (x.double() - zero_below).abs().amin() < 1e-6 if zero_below else False
    print(f"\n{shape} times={times} zero_below={zero_below}: max |err| vs float64 {err.max().item():.3e}; "
          f"bit-identical to the fp32 CPU restatement: {torch.equal(out, f32)}")
    # measured on an H100: max 1.8e-7 (30 passes)
    assert near or err.max().item() < 4e-7
    if min(shape) < 3:
        # no interior: every pass is a renormalisation only
        y = x.double()
        for _ in range(times):
            y = y / y.sum(1, keepdim=True)
        if zero_below:
            y[y < zero_below] = 0
        assert (out.double() - y).abs().max().item() < 4e-7
    if times == 0 and not zero_below:
        assert torch.equal(out, x)                       # the reference's loop does not run: values untouched


@pytest.mark.parametrize("name", list(CASES))
def test_end_to_end_vs_reference(name):
    variant, res, ac, k, times = CASES[name]
    v, w = torch.from_numpy(G["verts"]).to(DEV), torch.from_numpy(G["vert_ws"]).to(DEV)
    fn = Deformer.compute_lbswField if variant == "model" else utils.compute_lbswField
    out = fn(BMIN, BMAX, res, v, w, align_corners=ac, mean_neighbor=k, smooth_times=times)
    ref = torch.from_numpy(G[name]).to(DEV)
    assert out.shape == ref.shape
    err = (out - ref).abs().max().item()
    print(f"\n{name}: max |err| vs the reference's output {err:.3e}")
    # the kernel's distances and sums round differently from torch's norm / sum.  Measured on an H100: 3.6e-7
    # (times = 0), 1.8e-7 in the three smoothed cases
    assert err < 1.2e-6


def test_repeatable_streams_and_output_bounds():
    v, w = body()
    res, k, G_ = (13, 25, 9), 30, 7
    W, H, D = res
    N = W * H * D
    a = ops.lbsw_knn_blend(v, w, BMIN, BMAX, res, k, want_idx=True)
    b = ops.lbsw_knn_blend(v, w, BMIN, BMAX, res, k, want_idx=True)
    s = torch.cuda.Stream(DEV)
    with torch.cuda.stream(s):
        c = ops.lbsw_knn_blend(v, w, BMIN, BMAX, res, k, want_idx=True)
    s.synchronize()
    for x, y in ((a, b), (a, c)):
        assert torch.equal(x[0], y[0]) and torch.equal(x[1], y[1])
    sa = ops.lbsw_smooth(a[0].clone(), 30)
    with torch.cuda.stream(s):
        sc = ops.lbsw_smooth(a[0].clone(), 30)
    s.synchronize()
    assert torch.equal(sa[0], sc[0]) and torch.equal(sa[1], sc[1])

    # guard regions of NaN around every output; every element inside must be written
    lib = _lib.load()
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    st = ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    cl = torch.full((N + 2 * G_, 24), float("nan"), device=DEV)
    ix = torch.full((N + 2 * G_, k), -7, dtype=torch.int32, device=DEV)
    lo, hi = (ctypes.c_float * 3)(*BMIN), (ctypes.c_float * 3)(*BMAX)
    assert lib.recmv_lbsw_knn_blend(P(v), P(w), v.shape[0], 24, lo, hi, W, H, D, 0, k, P(cl[G_:]), P(ix[G_:]), st) == 0
    torch.cuda.synchronize()
    assert torch.isnan(cl[:G_]).all() and torch.isnan(cl[G_ + N:]).all() and not torch.isnan(cl[G_:G_ + N]).any()
    assert (ix[:G_] == -7).all() and (ix[G_ + N:] == -7).all() and (ix[G_:G_ + N] >= 0).all()
    assert torch.equal(cl[G_:G_ + N].view(D, H, W, 24), a[0]) and torch.equal(ix[G_:G_ + N], a[1])
    for times in (0, 1, 4):
        bufa = torch.full((N + 2 * G_, 24), float("nan"), device=DEV)
        bufa[G_:G_ + N] = a[0].view(N, 24)
        bufb = torch.full_like(bufa, float("nan"))
        ocl = torch.full_like(bufa, float("nan"))
        onc = torch.full((24 * N + 2 * G_,), float("nan"), device=DEV)
        assert lib.recmv_lbsw_smooth(P(bufa[G_:]), P(bufb[G_:]), D, H, W, times, 0.0, P(onc[G_:]), P(ocl[G_:]), st) == 0
        torch.cuda.synchronize()
        for t in (bufa, bufb, ocl):
            assert torch.isnan(t[:G_]).all() and torch.isnan(t[G_ + N:]).all()
        assert torch.isnan(onc[:G_]).all() and torch.isnan(onc[G_ + 24 * N:]).all()
        assert not torch.isnan(ocl[G_:G_ + N]).any() and not torch.isnan(onc[G_:G_ + 24 * N]).any()
        ref = ops.lbsw_smooth(a[0].clone(), times)
        assert torch.equal(onc[G_:G_ + 24 * N].view(1, 24, D, H, W), ref[0])
        assert torch.equal(ocl[G_:G_ + N].view(D, H, W, 24), ref[1])


def test_skinner_from_body_matches_plain_constructor():
    v, w = body()
    Js, parents, init = synth.skeleton()
    sk, verts, faces = Deformer.skinner_from_body(v, w, Js, parents, init, (33, 57, 17))
    assert faces is None and verts.shape == (6890, 3)
    assert sk.ws.shape == (1, 24, 17, 57, 33)
    assert torch.allclose(sk.bbox_extend, (v.max(0).values - v.min(0).values).max() * 1.1)
    assert torch.equal(sk.ws, Deformer.compute_lbswField(v.min(0).values.tolist(), v.max(0).values, (33, 57, 17), v, w,
                                                         mean_neighbor=30, smooth_times=30))
    sk = sk.to(DEV)
    seeded = sk._ws_cl
    assert seeded is not None and sk.ws_channels_last() is seeded      # the cache is used, not rebuilt
    assert torch.equal(seeded, ops.voxel_to_channels_last(sk.ws))
    plain = Deformer.LBSkinner(sk.ws.clone(), sk.b_min, sk.b_max, Js, parents, init_pose=init,
                               bbox_extend=sk.bbox_extend, bbox_center=sk.bbox_center).to(DEV)
    poses, trans = synth.poses_trans(2, seed=11)
    poses, trans = poses.to(DEV), trans.to(DEV)
    g = torch.Generator().manual_seed(1)
    ps = ((torch.rand((2, 500, 3), generator=g) - 0.5) * 1.6).to(DEV)
    with torch.no_grad():
        assert torch.equal(sk(ps, [poses, trans]), plain(ps, [poses, trans]))
        xa, oka = sk.inverse(ps, [poses, trans])
        xb, okb = plain.inverse(ps, [poses, trans])
    assert torch.equal(xa, xb) and torch.equal(oka, okb)
