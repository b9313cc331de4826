"""The skinning kernels (csrc/lbs.cu: recmv_lbs_fwd, recmv_lbs_inverse, recmv_lbs_backward, recmv_lbs_vjp_backward)
on the production voxel, across the voxel border, over many frames and at many-wave sizes, against the float64
oracle of tests/skinning_oracle.py on the scenes of tests/skinning_scenes.py.

Metric: every entry must satisfy |y_kernel - y_64| <= kappa 2^-24 S, with S the oracle's absolute twin of that entry
(the sum of the magnitudes of the terms it adds), and one kappa per kernel and output, about 3x the value measured on
an H100.  Each check prints the measured kappa and, beside it, the older max|a - b| / max|b|.  NaN patterns must be
equal, and so must infinities.  The bit-exact checks (multi-wave launches against one-wave slices, permutations, the
three ways of naming a frame, NULL optional outputs, two runs of a reduction) need no tolerance."""
import ctypes
import functools

import numpy as np
import pytest
import torch

import skinning_oracle as so
import skinning_scenes as sc
from oracle import oracle_torch as ot
from recmv_b200 import _lib, ops, synth
from recmv_b200.model import LBSkinner
from recmv_b200.utils import compute_Jacobian

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = 2.0 ** -24
CENTER = [float(x) for x in sc.CENTER]
EXTEND = float(sc.EXTEND)
# kappa bounds, about 3x the largest value measured on an H100 80GB HBM3 (700 W); see DESIGN section 6
KAPPA = {
    "fwd.out": 22, "fwd.w": 18,                                   # measured 7.4, 5.8
    "inv.xc": 15,                                                 # 5.0
    "bwd.dps": 23, "bwd.dtps": 9, "bwd.dA": 33, "bwd.dtrans": 8,  # 7.6, 2.8, 11.0, 2.6
    "vjp.dg": 17, "vjp.dps": 15, "vjp.dtps": 10, "vjp.dA": 19,    # 5.7, 5.1, 3.5, 6.5
}
# LBSkinner end to end, max|a - b| / max|b| against float64 (the chain kernel's fp32 bone matrices included)
# (measured 4.8e-7, 8.1e-7, 1.8e-7, 2.5e-7, 4.8e-6, 1.1e-6)
E2E = {"fwd": 1.5e-6, "dtmpl": 2.5e-6, "dposes": 6e-7, "dtrans": 8e-7, "cg.dps": 1.5e-5, "cg.dposes": 3.5e-6}
MEASURED = {}


@functools.lru_cache(maxsize=None)
def _ws(name):
    return sc.channels_last(sc.voxel(name)).to(DEV)


@functools.lru_cache(maxsize=None)
def _skin(name):
    return so.Skin(_ws(name), CENTER, EXTEND)


def _wave():
    return torch.cuda.get_device_properties(0).multi_processor_count * 8 * 128


class Checks:
    """Collects every comparison of a test, prints it, and fails at the end with all the violations."""

    def __init__(self):
        self.bad = []

    def kappa(self, key, label, k, y, S):
        k = k.detach().double().reshape(y.shape).to(y.device)
        nan_k, nan_y = torch.isnan(k), torch.isnan(y)
        if not torch.equal(nan_k, nan_y):
            self.bad.append(f"{label} {key}: NaN pattern differs at {int((nan_k != nan_y).sum())} entries")
            return
        inf_y = torch.isinf(y)
        if not torch.equal(torch.isinf(k), inf_y) or not torch.equal(k[inf_y], y[inf_y]):
            self.bad.append(f"{label} {key}: infinities differ")
            return
        fin = torch.isfinite(y) & torch.isfinite(S)
        d = (k - y).abs()[fin]
        s = S[fin]
        zero = s == 0
        if (d[zero] != 0).any():
            self.bad.append(f"{label} {key}: {int((d[zero] != 0).sum())} entries with S = 0 are not exact")
        kap = float((d[~zero] / (EPS * s[~zero])).max()) if (~zero).any() else 0.0
        old = float(d.max() / y[fin].abs().max().clamp_min(1e-30)) if d.numel() else 0.0
        MEASURED[key] = max(MEASURED.get(key, 0.0), kap)
        print(f"{label} {key}: kappa {kap:.3g} (bound {KAPPA[key]})  max|a-b|/max|b| {old:.2e}")
        if not kap <= KAPPA[key]:
            self.bad.append(f"{label} {key}: kappa {kap:.3g} > {KAPPA[key]}")
        return kap

    def true(self, cond, what):
        if not cond:
            self.bad.append(what)

    def done(self):
        assert not self.bad, "\n".join(self.bad)


def _t(x, dtype=None):
    t = torch.as_tensor(x)
    return (t if dtype is None else t.to(dtype)).to(DEV).contiguous()


def _fwd(ws, ps, A, trans, bi=None, ppf=0, tps=None, weights=True):
    return ops.lbs_forward(ps, A, trans, ws, CENTER, EXTEND, bi, ppf, tps, want_weights=weights)


# ------------------------------------------------------------------ recmv_lbs_fwd
@pytest.mark.parametrize("vox", ["prod", "sharp", "small"])
def test_forward_coordinate_classes(vox):
    """Every coordinate class, with and without tps, over 33 frames of random layout with out-of-range indices."""
    c = Checks()
    ws, sk = _ws(vox), _skin(vox)
    ps, cls, _ = sc.classed_points(sc.SHAPES[vox], per_class=128, seed=1)
    P = ps.shape[0]
    F = 33
    A, trans = sc.bone_A(F, seed=2)
    bi = sc.frames(P, F, "random", seed=3, out_of_range=True)
    f = _t(sc.clamp_frames(bi, F))
    A, trans, bi = _t(A), _t(trans), _t(bi)
    ps = _t(ps)
    for tps_form in (False, True):
        if tps_form:
            tps, p = ps, _t(sc.random_points(P, seed=4))
        else:
            tps, p = None, ps
        out, w = _fwd(ws, p, A, trans, bi, 0, tps)
        y, S, wy = so.forward(sk, p, A, trans, f, tps)
        c.kappa("fwd.out", f"{vox} tps={tps_form}", out, y, S)
        c.kappa("fwd.w", f"{vox} tps={tps_form}", w, wy, wy)
        c.true(torch.isfinite(w).all(), "weights finite at every coordinate")
    c.done()


@pytest.mark.parametrize("F", sc.FRAME_COUNTS)
def test_forward_frame_layouts(F):
    c = Checks()
    ws, sk = _ws("prod"), _skin("prod")
    P = 33 * 256 + 5
    A, trans = sc.bone_A(F, seed=F)
    A, trans = _t(A), _t(trans)
    p = _t(sc.random_points(P, seed=F))
    for layout in sc.LAYOUTS:
        for oor in (False, True):
            bi = sc.frames(P, F, layout, seed=F, out_of_range=oor)
            out, w = _fwd(ws, p, A, trans, _t(bi))
            y, S, wy = so.forward(sk, p, A, trans, _t(sc.clamp_frames(bi, F)))
            c.kappa("fwd.out", f"F={F} {layout} oor={oor}", out, y, S)
            # out-of-range indices select the clamped frames, bit for bit
            ref = _fwd(ws, p, A, trans, _t(sc.clamp_frames(bi, F)))[0]
            c.true(torch.equal(out, ref), f"F={F} {layout}: out-of-range indices do not select the clamped frames")
    c.done()


def _sizes():
    w = _wave()
    return [1, 255, 256, 257, 33 * 256, w - 1, w, w + 1, 3 * w + 77, 10 ** 6 + 77]


def test_forward_sizes_slices_and_permutations():
    c = Checks()
    ws, sk = _ws("prod"), _skin("prod")
    w = _wave()
    F = 3
    A, trans = sc.bone_A(F, seed=5)
    A, trans = _t(A), _t(trans)
    for P in _sizes():
        p = _t(sc.random_points(P, seed=P % 1000))
        tps = (p + 0.02 * torch.randn(p.shape, device=DEV, generator=torch.Generator(DEV).manual_seed(P))).contiguous()
        bi = _t(sc.frames(P, F, "random", seed=P))
        for t in (None, tps):
            out, wo = _fwd(ws, p, A, trans, bi, 0, t)
            y, S, wy = so.forward(sk, p, A, trans, bi, t)
            c.kappa("fwd.out", f"P={P} tps={t is not None}", out, y, S)
            c.kappa("fwd.w", f"P={P} tps={t is not None}", wo, wy, wy)
            if P > w:
                # a multi-wave launch equals one-wave slices, and a permutation permutes
                parts = [_fwd(ws, p[i:i + w], A, trans, bi[i:i + w], 0, None if t is None else t[i:i + w])
                         for i in range(0, P, w)]
                c.true(torch.equal(out, torch.cat([q[0] for q in parts])) and
                       torch.equal(wo, torch.cat([q[1] for q in parts])), f"P={P}: slices differ")
                perm = torch.randperm(P, device=DEV, generator=torch.Generator(DEV).manual_seed(1))
                o2, w2 = _fwd(ws, p[perm], A, trans, bi[perm], 0, None if t is None else t[perm])
                c.true(torch.equal(o2, out[perm]) and torch.equal(w2, wo[perm]), f"P={P}: permutation differs")
    c.done()


@pytest.mark.parametrize("ppf", sc.PPFS)
def test_forward_ppf_batch_inds_and_out_of_range_agree(ppf):
    c = Checks()
    ws, sk = _ws("prod"), _skin("prod")
    F = 3
    P = ppf * F + 77                                       # a tail beyond ppf * F: clamped into the last frame
    A, trans = sc.bone_A(F, seed=6)
    A, trans = _t(A), _t(trans)
    p = _t(sc.random_points(P, seed=7))
    f = sc.ppf_frames(P, ppf, F)
    a = _fwd(ws, p, A, trans, None, ppf)
    b = _fwd(ws, p, A, trans, _t(f))
    oor = f.copy()
    oor[f == F - 1] = np.where(np.arange((f == F - 1).sum()) % 2 == 0, F, 1 << 40)
    oor[f == 0] = np.where(np.arange((f == 0).sum()) % 2 == 0, -1, 0)
    d = _fwd(ws, p, A, trans, _t(oor))
    c.true(all(torch.equal(x, y) for x, y in zip(a, b)) and all(torch.equal(x, y) for x, y in zip(a, d)),
           f"ppf={ppf}: the three frame forms differ")
    y, S, _ = so.forward(sk, p, A, trans, _t(f))
    c.kappa("fwd.out", f"ppf={ppf}", a[0], y, S)
    c.done()


def _guarded(n, *shape, dtype=torch.float32, fill=float("nan")):
    return torch.full((n + 2 * 512,) + shape, fill, dtype=dtype, device=DEV)


def _vox(ws):
    return ops.make_voxel(ws, CENTER, EXTEND)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _in(t):
    return None if t is None else ctypes.c_void_p(t[512:].data_ptr())


def test_forward_and_inverse_guarded_buffers_and_null_outputs():
    c = Checks()
    ws = _ws("prod")
    P, F = 3 * _wave() + 77, 3
    A, trans = sc.bone_A(F, seed=8)
    A, trans = _t(A), _t(trans)
    p = _t(sc.random_points(P, seed=9))
    bi = _t(sc.frames(P, F, "random", seed=10))
    vox = _vox(ws)
    lib = _lib.load()
    out, wo = _guarded(P, 3), _guarded(P, 24)
    _lib.check(lib.recmv_lbs_fwd(ops._ptr(p), None, ops._ptr(A), ops._ptr(trans), ops._ptr(bi), 0, F, ctypes.byref(vox),
                                 _in(out), _in(wo), P, _stream()))
    out2 = _guarded(P, 3)
    _lib.check(lib.recmv_lbs_fwd(ops._ptr(p), None, ops._ptr(A), ops._ptr(trans), ops._ptr(bi), 0, F, ctypes.byref(vox),
                                 _in(out2), None, P, _stream()))
    xc, va = _guarded(P, 3), _guarded(P, dtype=torch.uint8, fill=0xAB)
    _lib.check(lib.recmv_lbs_inverse(ops._ptr(p), ops._ptr(A), ops._ptr(trans), ops._ptr(bi), 0, F, ctypes.byref(vox),
                                     _in(xc), _in(va), P, _stream()))
    xc2 = _guarded(P, 3)
    _lib.check(lib.recmv_lbs_inverse(ops._ptr(p), ops._ptr(A), ops._ptr(trans), ops._ptr(bi), 0, F, ctypes.byref(vox),
                                     _in(xc2), None, P, _stream()))
    torch.cuda.synchronize()
    for name, o in (("out", out), ("weights", wo), ("out (weights NULL)", out2), ("xc", xc), ("xc (valid NULL)", xc2)):
        c.true(torch.isnan(o[:512]).all() and torch.isnan(o[512 + P:]).all(), f"{name}: guard written")
        c.true(torch.isfinite(o[512:512 + P]).all(), f"{name}: row not written")
    c.true((va[:512] == 0xAB).all() and (va[512 + P:] == 0xAB).all() and (va[512:512 + P] <= 1).all(), "valid guards")
    c.true(torch.equal(out[512:512 + P], out2[512:512 + P]), "weights_out = NULL changes out")
    c.true(torch.equal(xc[512:512 + P], xc2[512:512 + P]), "valid = NULL changes xc")
    c.done()


# ------------------------------------------------------------------ recmv_lbs_inverse
def _inverse_check(c, label, xc, va, sk, x, A, trans, f, may_be_ambiguous=None):
    """xc / valid against the oracle.  Rows whose float64 |det| lies within fp32's rounding bound of det (16 eps times
    its twin) of the 1e-4 gate are ambiguous: counted, and allowed only in `may_be_ambiguous` (else at most 16)."""
    y, ok, det, detS, cond, scale = so.inverse(sk, x, A, trans, f)
    va = va.to(y.device)
    amb = ((det.abs() - 1e-4).abs() <= 16 * EPS * detS) & torch.isfinite(det)
    mism = (va != ok) & ~amb
    c.true(not mism.any(), f"{label}: valid differs on {int(mism.sum())} rows away from the gate")
    n_amb = int(amb.sum())
    print(f"{label}: {n_amb} of {len(ok)} rows within fp32 rounding of the 1e-4 gate, valid differs on "
          f"{int((amb & (va != ok)).sum())} of them")
    if may_be_ambiguous is None:
        c.true(n_amb <= 16, f"{label}: {n_amb} ambiguous rows")
    else:
        c.true(not (amb & ~may_be_ambiguous).any(), f"{label}: ambiguous rows outside the frames at the gate")
    both = va & ok & ~amb
    k = xc.double()[both]
    yy = y[both]
    c.true(torch.equal(torch.isnan(k), torch.isnan(yy)), f"{label}: NaN pattern of xc differs")
    inv_ = ~va & ~amb
    c.true((xc[inv_] == 0).all(), f"{label}: an invalid row is not 0")
    fin = torch.isfinite(yy).all(1) & torch.isfinite(scale[both]) & torch.isfinite(cond[both])
    err = (k - yy).abs().amax(1)[fin]
    bound = EPS * cond[both][fin] * scale[both][fin]
    kap = float((err / bound).max()) if fin.any() else 0.0
    MEASURED["inv.xc"] = max(MEASURED.get("inv.xc", 0.0), kap)
    old = float(err.max() / yy[fin].abs().max()) if fin.any() else 0.0
    print(f"{label} inv.xc: kappa {kap:.3g} (bound {KAPPA['inv.xc']}, per row against cond |M^-1|(|x|+|trans|+|t|))"
          f"  max|a-b|/max|b| {old:.2e}")
    c.true(kap <= KAPPA["inv.xc"], f"{label}: inverse kappa {kap:.3g}")
    return ok, amb


def test_inverse_determinant_sweep_singular_and_nan_rows():
    c = Checks()
    ws, sk = _ws("prod"), _skin("prod")
    F = 300
    sing, nanf = (7, 150), (11, 280)
    A, trans = sc.inverse_A(F, singular=sing, nan=nanf, gate=True)
    A, trans = _t(A), _t(trans)
    P = 3 * _wave() + 77
    x = _t(sc.random_points(P, seed=12, spread=1.05))
    bi = _t(sc.frames(P, F, "random", seed=13))
    xc, va = ops.lbs_inverse(x, A, trans, ws, CENTER, EXTEND, bi)
    n_gate = len(sc.GATE_OFFSETS)
    at_gate = bi >= F - n_gate
    ok, amb = _inverse_check(c, "inverse det sweep", xc, va, sk, x, A, trans, bi, may_be_ambiguous=at_gate)
    # the frames at the gate: rows on both sides of it, rows inside fp32's rounding of it, and the +-10 % frames
    # decided exactly like float64
    c.true(va[at_gate].any() and (~va[at_gate]).any() and amb[at_gate].any(), "the gate frames do not probe the gate")
    for i, off in enumerate(sc.GATE_OFFSETS):
        if abs(off) >= 0.1:
            m = bi == F - n_gate + i
            c.true(not amb[m].any() and torch.equal(va[m], ok[m]), f"gate frame {off}: undecided")
    for fs in sing:
        m = bi == fs
        c.true(m.any() and (~va[m]).all() and (xc[m] == 0).all(), f"singular frame {fs}: not 0 and invalid")
    for fs in nanf:
        m = bi == fs
        c.true(m.any() and va[m].all() and torch.isnan(xc[m]).all(), f"NaN frame {fs}: not NaN and valid")
    c.true((~va).sum() > 0.2 * P and va.sum() > 0.2 * P, "the sweep does not cross the gate")
    # multi-wave against one-wave slices, and a permutation
    w = _wave()
    parts = [ops.lbs_inverse(x[i:i + w], A, trans, ws, CENTER, EXTEND, bi[i:i + w]) for i in range(0, P, w)]
    c.true(torch.equal(xc.nan_to_num(7.0), torch.cat([q[0] for q in parts]).nan_to_num(7.0)) and
           torch.equal(va, torch.cat([q[1] for q in parts])), "inverse slices differ")
    perm = torch.randperm(P, device=DEV, generator=torch.Generator(DEV).manual_seed(2))
    x2, v2 = ops.lbs_inverse(x[perm], A, trans, ws, CENTER, EXTEND, bi[perm])
    c.true(torch.equal(x2.nan_to_num(7.0), xc[perm].nan_to_num(7.0)) and torch.equal(v2, va[perm]),
           "inverse permutation differs")
    c.done()


@pytest.mark.parametrize("vox", ["prod", "small"])
def test_inverse_coordinate_classes(vox):
    c = Checks()
    ws, sk = _ws(vox), _skin(vox)
    ps, cls, _ = sc.classed_points(sc.SHAPES[vox], per_class=128, seed=14)
    P = ps.shape[0]
    F = 3
    A, trans = sc.bone_A(F, seed=15)
    A, trans, x = _t(A), _t(trans), _t(ps)
    bi = _t(sc.frames(P, F, "interleaved"))
    xc, va = ops.lbs_inverse(x, A, trans, ws, CENTER, EXTEND, bi, 0)
    _inverse_check(c, f"inverse classes {vox}", xc, va, sk, x, A, trans, bi)
    c.done()


# ------------------------------------------------------------------ recmv_lbs_backward
def _bwd_run(c, label, ws, sk, p, A, g, bi, f, F, tps=None, ppf=0):
    k = ops.lbs_backward(p, A, g, ws, CENTER, EXTEND, bi, ppf, tps)
    (dps, dtps, dA, dtr), (Sp, St, SA, Str) = so.backward(sk, p, A, g, f, F, tps)
    c.kappa("bwd.dps", label, k[0], dps, Sp)
    if tps is not None:
        c.kappa("bwd.dtps", label, k[1], dtps, St)
    c.kappa("bwd.dA", label, k[2], dA, SA)
    c.kappa("bwd.dtrans", label, k[3], dtr, Str)
    c.true((k[2][:, :, 3] == 0).all(), f"{label}: row 3 of dA")
    empty = torch.bincount(f, minlength=F) == 0
    if empty.any():
        c.true((k[2][empty] == 0).all() and (k[3][empty] == 0).all(), f"{label}: a frame with no point is not 0")
    return k


@pytest.mark.parametrize("F", sc.FRAME_COUNTS)
def test_backward_frame_layouts(F):
    """Every layout at F frames; P = 33 chunks + 5 points (F > 256: slot numbers up to 255 per chunk)."""
    c = Checks()
    ws, sk = _ws("prod"), _skin("prod")
    P = 33 * 256 + 5
    A, trans = sc.bone_A(F, seed=F + 1)
    A = _t(A)
    p = _t(sc.random_points(P, seed=F + 2))
    gen = torch.Generator(DEV).manual_seed(F)
    g = torch.randn((P, 3), device=DEV, generator=gen)
    tps_all = (p + 0.03 * torch.randn((P, 3), device=DEV, generator=gen)).contiguous()
    for i, layout in enumerate(sc.LAYOUTS):
        for oor in (False, True):
            bi = sc.frames(P, F, layout, seed=F, out_of_range=oor)
            f = _t(sc.clamp_frames(bi, F))
            tps = tps_all if (i + oor) % 2 else None
            k = _bwd_run(c, f"F={F} {layout} oor={oor} tps={tps is not None}", ws, sk, p, A, g, _t(bi), f, F, tps)
            if oor:
                ref = ops.lbs_backward(p, A, g, ws, CENTER, EXTEND, f, 0, tps)
                c.true(all(torch.equal(a, b) for a, b in zip(k, ref) if a is not None),
                       f"F={F} {layout}: out-of-range indices differ from the clamped ones")
            d, w = sc.chunk_stats(f.cpu().numpy())
            if F >= 256 and layout == "interleaved" and not oor:
                c.true(d.max() == 256 and w.max() == 8, "interleaved layout does not fill the slots")
    c.done()


@pytest.mark.parametrize("vox", ["prod", "sharp", "small"])
def test_backward_coordinate_classes(vox):
    """Every coordinate class as the sampling point: as ps (the finite classes: lattice planes, the border, outside) and
    as tps (all of them, with +-inf, NaN and 1e30), over 33 frames of random layout with out-of-range indices."""
    c = Checks()
    ws, sk = _ws(vox), _skin(vox)
    ps, cls, _ = sc.classed_points(sc.SHAPES[vox], per_class=128, seed=30)
    fin = np.isfinite(ps).all(1)
    F = 33
    A, _ = sc.bone_A(F, seed=31)
    A = _t(A)
    gen = torch.Generator(DEV).manual_seed(32)
    for tps_form in (False, True):
        s = _t(ps if tps_form else ps[fin])
        P = s.shape[0]
        tps, p = (s, _t(sc.random_points(P, seed=33))) if tps_form else (None, s)
        g = torch.randn((P, 3), device=DEV, generator=gen)
        bi = sc.frames(P, F, "random", seed=34, out_of_range=True)
        _bwd_run(c, f"{vox} classes tps={tps_form}", ws, sk, p, A, g, _t(bi), _t(sc.clamp_frames(bi, F)), F, tps)
        if tps_form:
            # a NaN or infinite sampling coordinate has no weight derivative on its axis
            k = ops.lbs_backward(p, A, g, ws, CENTER, EXTEND, _t(bi), 0, tps)[1]
            c.true((k[~torch.isfinite(tps)] == 0).all(), f"{vox}: dtps not 0 on a non-finite axis")
    c.done()


@pytest.mark.parametrize("P", [1, 5 * 256 - 3, 32 * 256, 33 * 256, 10 ** 6 + 77])
def test_backward_sizes_invariances(P):
    """5 chunks (fewer than the reduce's 32 rows), 32, 33 and 3 907 chunks; per-point outputs slice- and
    permutation-invariant, dA / dtrans bit-identical across runs and between the ppf and batch_inds forms."""
    c = Checks()
    ws, sk = _ws("prod"), _skin("prod")
    F = 3
    ppf = max(P // F - 5, 1)
    A, _ = sc.bone_A(F, seed=16)
    A = _t(A)
    p = _t(sc.random_points(P, seed=17))
    gen = torch.Generator(DEV).manual_seed(P)
    g = torch.randn((P, 3), device=DEV, generator=gen)
    tps = (p + 0.03 * torch.randn((P, 3), device=DEV, generator=gen)).contiguous()
    f = _t(sc.ppf_frames(P, ppf, F))
    for t in (None, tps):
        k = _bwd_run(c, f"P={P} tps={t is not None}", ws, sk, p, A, g, None, f, F, t, ppf)
        k2 = ops.lbs_backward(p, A, g, ws, CENTER, EXTEND, None, ppf, t)
        k3 = ops.lbs_backward(p, A, g, ws, CENTER, EXTEND, f, 0, t)
        c.true(all(torch.equal(a, b) for a, b in zip(k, k2) if a is not None), f"P={P}: two runs differ")
        c.true(all(torch.equal(a, b) for a, b in zip(k, k3) if a is not None), f"P={P}: ppf and batch_inds differ")
        if P > 1:
            perm = torch.randperm(P, device=DEV, generator=torch.Generator(DEV).manual_seed(3))
            kp = ops.lbs_backward(p[perm], A, g[perm], ws, CENTER, EXTEND, f[perm], 0, None if t is None else t[perm])
            c.true(torch.equal(kp[0], k[0][perm]) and (t is None or torch.equal(kp[1], k[1][perm])),
                   f"P={P}: permuted per-point outputs differ")
            h = P // 2 + 1
            s1 = ops.lbs_backward(p[:h], A, g[:h], ws, CENTER, EXTEND, f[:h], 0, None if t is None else t[:h])
            s2 = ops.lbs_backward(p[h:], A, g[h:], ws, CENTER, EXTEND, f[h:], 0, None if t is None else t[h:])
            c.true(torch.equal(torch.cat([s1[0], s2[0]]), k[0]), f"P={P}: sliced dps differs")
    c.done()


# ------------------------------------------------------------------ recmv_lbs_vjp_backward
def _vjp_run(c, label, ws, sk, p, A, g, u, bi, f, F, tps=None, v=None, ppf=0):
    k = ops.lbs_vjp_backward(p, A, g, ws, CENTER, EXTEND, bi, ppf, tps, u, v)
    (dg, dps, dtps, dA), (Sg, Sp, St, SA) = so.vjp(sk, p, A, g, u, f, F, tps, v)
    c.kappa("vjp.dg", label, k[0], dg, Sg)
    c.kappa("vjp.dps", label, k[1], dps, Sp)
    if tps is not None:
        c.kappa("vjp.dtps", label, k[2], dtps, St)
    c.kappa("vjp.dA", label, k[3], dA, SA)
    c.true((k[3][:, :, 3] == 0).all(), f"{label}: row 3 of dA")
    empty = torch.bincount(f, minlength=F) == 0
    if empty.any():
        c.true((k[3][empty] == 0).all(), f"{label}: a frame with no point is not 0")
    return k


@pytest.mark.parametrize("vox", ["prod", "sharp", "toy"])
def test_vjp_voxels_and_layouts(vox):
    """The production and sharp voxels (the toy voxel's figures printed beside them), over every frame count and
    layout, with and without out-of-range indices, and every coordinate class in tps."""
    c = Checks()
    ws, sk = _ws(vox), _skin(vox)
    P = 33 * 256 + 5
    p = _t(sc.random_points(P, seed=18, spread=1.0))
    gen = torch.Generator(DEV).manual_seed(19)
    g, u, v = (torch.randn((P, 3), device=DEV, generator=gen) for _ in range(3))
    tps = (p + 0.03 * torch.randn((P, 3), device=DEV, generator=gen)).contiguous()
    for F in sc.FRAME_COUNTS:
        A, _ = sc.bone_A(F, seed=F + 3)
        A = _t(A)
        for i, layout in enumerate(sc.LAYOUTS):
            for oor in (False, True):
                bi = sc.frames(P, F, layout, seed=F, out_of_range=oor)
                f = _t(sc.clamp_frames(bi, F))
                t = tps if (i + oor) % 2 else None
                vv = v if t is not None else None
                k = _vjp_run(c, f"{vox} F={F} {layout} oor={oor} tps={t is not None}", ws, sk, p, A, g, u, _t(bi), f,
                             F, t, vv)
                if oor:
                    ref = ops.lbs_vjp_backward(p, A, g, ws, CENTER, EXTEND, f, 0, t, u, vv)
                    c.true(all(torch.equal(a, b) for a, b in zip(k, ref) if a is not None),
                           f"{vox} F={F} {layout}: out-of-range indices differ from the clamped ones")
    if vox != "toy":
        cp, _, _ = sc.classed_points(sc.SHAPES[vox], per_class=128, seed=20)
        cp = _t(cp)
        n = cp.shape[0]
        A, _ = sc.bone_A(3, seed=21)
        A = _t(A)
        f = _t(sc.frames(n, 3, "random", seed=22))
        pa = _t(sc.random_points(n, seed=23, spread=1.0))
        _vjp_run(c, f"{vox} classes in tps", ws, sk, pa, A, g[:n], u[:n], f, f, 3, cp, v[:n])
    c.done()


@pytest.mark.parametrize("vox", ["prod", "sharp"])
def test_vjp_sizes_invariances(vox):
    c = Checks()
    ws, sk = _ws(vox), _skin(vox)
    F = 3
    A, _ = sc.bone_A(F, seed=24)
    A = _t(A)
    for P in (1, 5 * 256 - 3, 32 * 256, 33 * 256, 10 ** 6 + 77):
        p = _t(sc.random_points(P, seed=25))
        gen = torch.Generator(DEV).manual_seed(P)
        g, u, v = (torch.randn((P, 3), device=DEV, generator=gen) for _ in range(3))
        tps = (p + 0.03 * torch.randn((P, 3), device=DEV, generator=gen)).contiguous()
        ppf = max(P // F - 3, 1)
        f = _t(sc.ppf_frames(P, ppf, F))
        for t in (None, tps):
            vv = v if t is not None else None
            k = _vjp_run(c, f"{vox} P={P} tps={t is not None}", ws, sk, p, A, g, u, None, f, F, t, vv, ppf)
            k2 = ops.lbs_vjp_backward(p, A, g, ws, CENTER, EXTEND, f, 0, t, u, vv)
            c.true(all(torch.equal(a, b) for a, b in zip(k, k2) if a is not None), f"P={P}: ppf and batch_inds differ")
            if P > 1:
                perm = torch.randperm(P, device=DEV, generator=torch.Generator(DEV).manual_seed(4))
                kp = ops.lbs_vjp_backward(p[perm], A, g[perm], ws, CENTER, EXTEND, f[perm], 0,
                                          None if t is None else t[perm], u[perm], None if vv is None else vv[perm])
                c.true(all(torch.equal(a, b[perm]) for a, b in zip(kp[:3], k[:3]) if a is not None),
                       f"P={P}: permuted per-point outputs differ")
                h = P // 2 + 1
                parts = [ops.lbs_vjp_backward(p[s], A, g[s], ws, CENTER, EXTEND, f[s], 0, None if t is None else t[s],
                                              u[s], None if vv is None else vv[s]) for s in (slice(0, h), slice(h, P))]
                c.true(all(torch.equal(torch.cat([parts[0][j], parts[1][j]]), k[j]) for j in range(3)
                           if k[j] is not None), f"P={P}: sliced per-point outputs differ")
    c.done()


# ------------------------------------------------------------------ LBSkinner end to end
def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def test_lbskinner_production_template():
    """A 55 233-vertex template x 3 frames on the production voxel: the fused forward, the fused-train gradients
    (template, poses, trans; the chain kernel included) and the fused create_graph input gradient, against float64."""
    c = Checks()
    Js, parents, ip = sc._skeleton()
    sk = LBSkinner(sc.voxel("prod"), [-1.1] * 3, [1.1] * 3, Js, parents, init_pose=ip,
                   bbox_extend=torch.tensor(EXTEND), bbox_center=torch.tensor(CENTER)).to(DEV)
    V, F = sc.TEMPLATE_V, 3
    gen = synth.generator(26)
    tmpl = ((torch.rand((1, V, 3), generator=gen) - 0.5) * 2.0).to(DEV)
    poses, trans = synth.poses_trans(F, seed=27)
    poses, trans = poses.to(DEV), trans.to(DEV)
    cot = torch.randn((F, V, 3), generator=gen).to(DEV)
    skin = _skin("prod")
    f = torch.arange(F, device=DEV).repeat_interleave(V)
    p64 = poses.double().cpu().requires_grad_(True)
    A64 = ot.bone_matrices(p64, Js.double(), parents, ip.double())
    Ad = A64.detach().to(DEV)
    ps = tmpl.expand(F, V, 3).reshape(-1, 3).contiguous()
    # forward
    with torch.no_grad():
        out = sk(tmpl.expand(F, V, 3), [poses, trans], None)
    c.true(sk.last_path == "fused", "forward path")
    y, S, _ = so.forward(skin, ps, Ad, trans, f)
    e = _rel(out.reshape(-1, 3), y)
    print(f"LBSkinner fused forward: max|a-b|/max|b| {e:.2e} (bound {E2E['fwd']})")
    c.true(e < E2E["fwd"], f"forward {e:.2e}")
    # fused-train gradients
    t = tmpl.clone().requires_grad_(True)
    pd, td = poses.clone().requires_grad_(True), trans.clone().requires_grad_(True)
    o = sk(t.expand(F, V, 3), [pd, td], None)
    c.true(sk.last_path == "fused-train", "train path")
    gt, gp, gtr = torch.autograd.grad(o, (t, pd, td), cot)
    (dps, _, dA, dtr), _ = so.backward(skin, ps, Ad, cot.reshape(-1, 3), f, F)
    (rp,) = torch.autograd.grad(A64, p64, dA.cpu(), retain_graph=True)
    for name, k, r in (("dtmpl", gt, dps.view(F, V, 3).sum(0, keepdim=True)), ("dposes", gp, rp), ("dtrans", gtr, dtr)):
        e = _rel(k, r)
        print(f"LBSkinner fused-train {name}: max|a-b|/max|b| {e:.2e} (bound {E2E[name]})")
        c.true(e < E2E[name], f"{name} {e:.2e}")
    # the fused create_graph input gradient (train-phase normals) against float64 and the composite
    cotJ = torch.randn((F * V, 3, 3), generator=gen).to(DEV)
    cotD = torch.randn((F * V, 3), generator=gen).to(DEV)
    res = {}
    for fused in (True, False):
        sk.second_order_fused = fused
        x = ps.clone().requires_grad_(True)
        pd = poses.clone().requires_grad_(True)
        D = sk(x.view(F, V, 3), [pd, trans], None).reshape(-1, 3)
        J = compute_Jacobian(x, D, True, True)
        if fused:
            c.true(sk.last_backward == "fused (create_graph, input gradient)", sk.last_backward)
        loss = (J * cotJ).sum() + (D * cotD).sum()
        res[fused] = torch.autograd.grad(loss, (x, pd))
    sk.second_order_fused = False
    (dps, _, dA, _), _ = so.backward(skin, ps, Ad, cotD, f, F)
    for i in range(3):
        e_i = torch.zeros((F * V, 3), dtype=torch.float32, device=DEV)
        e_i[:, i] = 1
        (_, d2, _, dA2), _ = so.vjp(skin, ps, Ad, e_i, cotJ[:, i, :].contiguous(), f, F)
        dps, dA = dps + d2, dA + dA2
    (rp,) = torch.autograd.grad(A64, p64, dA.cpu())
    for name, k, r, comp in (("cg.dps", res[True][0], dps, res[False][0]), ("cg.dposes", res[True][1], rp, res[False][1])):
        e, ec = _rel(k, r), _rel(comp, r)
        print(f"LBSkinner create_graph {name}: fused {e:.2e}  composite fp32 {ec:.2e} (bound {E2E[name]})")
        c.true(e < E2E[name], f"{name} {e:.2e}")
    c.done()


def test_zz_print_measured():
    print("measured kappa:", {k: round(v, 3) for k, v in sorted(MEASURED.items())})
