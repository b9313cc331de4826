"""Pins the float64 skinning oracle (tests/skinning_oracle.py) on the CPU.

Its forward, inverse, backward and VJP equal ot.lbs_forward / ot.lbs_inverse and their first- and second-order float64
autograd to 1e-12.  The comparison uses a box of extend 2 centred at 0 and dyadic points, so that the fp32 voxel
coordinate the oracle evaluates at is exact and equals ot's float64 one; the points stay off lattice planes, where the
one-sided derivatives of the two could differ.  Separately, the oracle's fp32 coordinate equals ot._unnormalize_clip
computed in fp32 with the production box, and its absolute twins bound the outputs they belong to."""
import numpy as np
import pytest
import torch

import skinning_oracle as so
import skinning_scenes as sc
from oracle import oracle_torch as ot

SHAPE = (17, 33, 21)
CENTER = (0.0, 0.0, 0.0)
EXTEND = 2.0


def _scene(P=600, F=3, seed=0):
    g = torch.Generator().manual_seed(seed)
    ws = sc.voxel("toy")
    k = torch.randint(-1150, 1150, (P, 3), generator=g)
    ps = (k.double() / 1024).float()                              # dyadic: exact in every fp32 step of the coordinate
    size = torch.tensor([SHAPE[2], SHAPE[1], SHAPE[0]], dtype=torch.float64)
    uu = ((ps.double() / EXTEND * 2 + 1) * size - 1) / 2
    keep = ((uu - uu.round()).abs() > 1e-3).all(1)                # off every lattice plane
    ps = ps[keep].contiguous()
    A, trans = sc.bone_A(F)
    A = A + 0.05 * torch.randn(A.shape, generator=g) * torch.tensor([1.0, 1, 1, 0]).view(4, 1)   # not rigid
    f = torch.randint(0, F, (ps.shape[0],), generator=g)
    return ws, ps, A.contiguous(), trans, f


def _skin(ws):
    return so.Skin(sc.channels_last(ws), CENTER, EXTEND)


def test_coord32_equals_the_fp32_sampler_coordinate():
    ps = sc.random_points(20000, seed=3, spread=1.4)
    for a, size in enumerate(sc.sizes_xyz(sc.SHAPES["prod"])):
        u = so.coord32(ps[:, a], int(size), float(sc.CENTER[a]), float(sc.EXTEND))
        g = ((ps[:, a] - float(sc.CENTER[a])) / torch.full_like(ps[:, a], float(sc.EXTEND))) * 2.0
        assert torch.equal(ot._unnormalize_clip(g, int(size)), u.clamp(0, float(size) - 1))
        assert np.array_equal(u.numpy(), sc.coords32(ps.numpy(), sc.SHAPES["prod"])[:, a])


@pytest.mark.parametrize("with_tps", [False, True])
def test_forward_and_backward_equal_autograd(with_tps):
    ws, ps, A, trans, f = _scene()
    g = torch.Generator().manual_seed(1)
    tps = (ps + (torch.randint(-40, 40, ps.shape, generator=g).float() / 1024)) if with_tps else None
    if with_tps:
        size = torch.tensor([SHAPE[2], SHAPE[1], SHAPE[0]], dtype=torch.float64)
        uu = ((tps.double() / EXTEND * 2 + 1) * size - 1) / 2
        keep = ((uu - uu.round()).abs() > 1e-3).all(1)
        ps, tps, f = ps[keep].contiguous(), tps[keep].contiguous(), f[keep]
    cot = torch.randn(ps.shape, generator=g)
    sk = _skin(ws)
    out, S, w = so.forward(sk, ps, A, trans, f, tps)
    p = ps.double().requires_grad_(True)
    t = tps.double().requires_grad_(True) if with_tps else None
    a = A.double().requires_grad_(True)
    tr = trans.double().requires_grad_(True)
    ref = ot.lbs_forward(p, a, tr, ws.double(), torch.tensor(CENTER).double(), EXTEND, f, t)
    assert (out - ref.detach()).abs().max() < 1e-12
    assert ((ref.detach().abs() <= S * (1 + 1e-12))).all()
    wref = ot.skin_weights(ws.double(), (t if with_tps else p).detach(), torch.tensor(CENTER).double(), EXTEND)
    assert (w - wref).abs().max() < 1e-12
    (dps, dtps, dA, dtr), (Sp, St, SA, Str) = so.backward(sk, ps, A, cot, f, A.shape[0], tps)
    ins = [x for x in (p, t, a, tr) if x is not None]
    gr = torch.autograd.grad(ref, ins, cot.double())
    exp = [gr[0], gr[1] if with_tps else None, gr[-2], gr[-1]]
    for k, (mine, r, s) in enumerate(zip((dps, dtps, dA, dtr), exp, (Sp, St, SA, Str))):
        if r is None:
            assert mine is None
            continue
        assert (mine - r).abs().max() < 1e-12 * max(1.0, float(r.abs().max())), k
        assert (r.abs() <= s * (1 + 1e-12) + 1e-300).all(), k


@pytest.mark.parametrize("with_tps", [False, True])
def test_vjp_equals_double_autograd(with_tps):
    ws, ps, A, trans, f = _scene(P=400, seed=2)
    g = torch.Generator().manual_seed(3)
    tps = None
    if with_tps:
        tps = (ps + (torch.randint(-40, 40, ps.shape, generator=g).float() / 1024))
        size = torch.tensor([SHAPE[2], SHAPE[1], SHAPE[0]], dtype=torch.float64)
        uu = ((tps.double() / EXTEND * 2 + 1) * size - 1) / 2
        keep = ((uu - uu.round()).abs() > 1e-3).all(1)
        ps, tps, f = ps[keep].contiguous(), tps[keep].contiguous(), f[keep]
    cg, u = torch.randn(ps.shape, generator=g), torch.randn(ps.shape, generator=g)
    v = torch.randn(ps.shape, generator=g) if with_tps else None
    sk = _skin(ws)
    (dg, dps, dtps, dA), (Sg, Sp, St, SA) = so.vjp(sk, ps, A, cg, u, f, A.shape[0], tps, v)
    F_ = A.shape[0]
    p = ps.double().requires_grad_(True)
    t = tps.double().requires_grad_(True) if with_tps else None
    a = A.double().requires_grad_(True)
    gg = cg.double().requires_grad_(True)
    out = ot.lbs_forward(p, a, torch.zeros((F_, 3), dtype=torch.float64), ws.double(), torch.tensor(CENTER).double(),
                         EXTEND, f, t)
    firsts = torch.autograd.grad(out, [p] + ([t] if with_tps else []), gg, create_graph=True)
    phi = (firsts[0] * u.double()).sum() + ((firsts[1] * v.double()).sum() if with_tps else 0)
    ins = [gg, p] + ([t] if with_tps else []) + [a]
    d = torch.autograd.grad(phi, ins, allow_unused=True)
    d = [x if x is not None else torch.zeros_like(i) for x, i in zip(d, ins)]
    exp = (d[0], d[1], d[2] if with_tps else None, d[-1])
    for k, (mine, r, s) in enumerate(zip((dg, dps, dtps, dA), exp, (Sg, Sp, St, SA))):
        if r is None:
            assert mine is None
            continue
        assert (mine - r).abs().max() < 1e-12 * max(1.0, float(r.abs().max())), k
        assert (r.abs() <= s * (1 + 1e-12) + 1e-300).all(), k


def test_inverse_equals_ot():
    ws, ps, A, trans, f = _scene(seed=4)
    F = 16
    Ai, tri = sc.inverse_A(F, singular=(3,), nan=(7,))
    f = torch.arange(ps.shape[0]) % F
    sk = _skin(ws)
    xc, ok, det, detS, cond, scale = so.inverse(sk, ps, Ai, tri, f)
    rx, rok = ot.lbs_inverse(ps.double(), Ai.double(), tri.double(), ws.double(), torch.tensor(CENTER).double(), EXTEND, f)
    assert torch.equal(ok, rok)
    assert torch.equal(torch.isnan(xc), torch.isnan(rx))
    fin = torch.isfinite(rx).all(1) & ok
    # two float64 evaluations of a system of condition number cond differ by about cond * 1e-16
    assert ((xc - rx).abs().amax(1)[fin] <= 1e-13 * (cond * scale)[fin]).all()
    assert (xc[f == 3] == 0).all() and not ok[f == 3].any()            # singular: invalid, 0
    assert ok[f == 7].all() and torch.isnan(xc[f == 7]).all()          # NaN: valid, NaN (FastMinv)
    assert (det.abs() <= detS * (1 + 1e-12))[torch.isfinite(det)].all()
    good = ok & torch.isfinite(xc).all(1)
    assert (xc[good].abs().amax(1) <= scale[good] * (1 + 1e-9)).all() and (cond[good] >= 1 - 1e-12).all()
