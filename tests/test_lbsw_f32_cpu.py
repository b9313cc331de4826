"""The float32 restatement of the skinning-voxel kernels (tests/lbsw_f32.py) against float64.  No GPU.

The neighbour lists equal a float64 brute force wherever the float64 gap between the k-th and (k+1)-th distance is
clear of the float32 rounding of the distance, and the NumPy and torch scans of the restatement agree everywhere.  The
blend and the smoothing are held, entry by entry, to |v32 - v64| <= kappa u S, u = 2^-24, with S the running bound of
the kernels' operation order (render_f32.Rb): the blend of the restatement's own neighbours, and the smoothing passes.
Each kappa is about 3x the largest ratio measured here (printed next to it).
"""
import numpy as np
import pytest
import torch

import lbsw_f32 as lf
import render_f32 as rf
from render_f32 import Rb
from recmv_b200 import synth

BMIN, BMAX = [-0.85, -0.9, -0.15], [0.85, 0.85, 0.2]
# measured: blend 0.22, smooth 0.34 (one pass)
KAPPA = dict(blend=0.7, smooth=1.0)


def ratio(a, b, S):
    a, b, S = (np.asarray(x, np.float64) for x in (a, b, S))
    d = np.abs(a - b)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(d == 0, 0.0, d / (rf.U * S))
    return float(r.max(initial=0.0))


@pytest.mark.parametrize("ac", [False, True])
def test_knn_restatement_against_float64(ac):
    v, w = (x.numpy() for x in synth.body_points())
    res = (13, 25, 9)
    sel = np.arange(13 * 25 * 9)
    c = lf.centres(sel, res, ac, BMIN, BMAX)
    s, ids = lf.neighbours(c, v)
    st, it = lf.neighbours(torch.as_tensor(c), torch.as_tensor(v), xp=torch)
    assert np.array_equal(s.view(np.uint32), st.view(np.uint32)) and np.array_equal(ids, it)
    d64 = np.linalg.norm(c.astype(np.float64)[:, None] - v.astype(np.float64)[None], axis=-1)
    o = np.argsort(d64, axis=1, kind="stable")
    ds = np.take_along_axis(d64, o, 1)
    worst = 0.0
    for k in (1, 5, 8, 16, 30, 32):
        clear = ds[:, k] - ds[:, k - 1] > 1e-5
        assert np.array_equal(np.sort(ids[clear, :k], 1), np.sort(o[clear, :k], 1))
        out, _ = lf.blend(s, ids, w, k)
        # float64 blend of the same neighbours, from the float64 distances, with its running bound
        dk = Rb(np.linalg.norm(c.astype(np.float64)[:, None] - v.astype(np.float64)[ids[:, :k]], axis=-1))
        dk = Rb(dk.v, dk.e + 4 * dk.v)               # the float32 distance: three roundings and a square root
        cl = Rb(np.clip(dk.v, 1e-4, 1.0), np.where((dk.v > 1e-4) & (dk.v < 1.0), dk.e, 0.0))
        r = 1.0 / cl
        tot = Rb(np.zeros(len(sel)))
        for i in range(k):
            tot = tot + r[:, i]
        acc = Rb(np.zeros((len(sel), 24)))
        for i in range(k):
            wi = r[:, i] / tot
            acc = acc + Rb(w[ids[:, i]]) * Rb(wi.v[:, None], wi.e[:, None])
        worst = max(worst, ratio(out, acc.v, acc.e))
    print(f"[f32 knn ac={ac}] kappa blend {worst:.3f} (bound {KAPPA['blend']})")
    assert worst <= KAPPA["blend"], worst


@pytest.mark.parametrize("times", [0, 1, 2, 30])
def test_smooth_restatement_against_float64(times):
    g = np.random.default_rng(times)
    x = g.random((9, 25, 13, 24), dtype=np.float32) ** 4
    x = (x / x.sum(-1, keepdims=True)).astype(np.float32)
    out = lf.smooth(x, times)
    w = Rb(x.astype(np.float64))
    for _ in range(times):
        c = w[1:-1, 1:-1, 1:-1]
        sum6 = ((((w[2:, 1:-1, 1:-1] + w[:-2, 1:-1, 1:-1]) + w[1:-1, 2:, 1:-1]) + w[1:-1, :-2, 1:-1])
                + w[1:-1, 1:-1, 2:]) + w[1:-1, 1:-1, :-2]
        mean = sum6 / 6.0
        new = ((c - mean) * Rb(float(np.float32(0.7)))) + mean
        v, e = w.v.copy(), w.e.copy()
        v[1:-1, 1:-1, 1:-1], e[1:-1, 1:-1, 1:-1] = new.v, new.e
        w = Rb(v, e)
        tot = Rb(np.zeros(w.v.shape[:3]))
        for ch in range(24):
            tot = tot + w[..., ch]
        w = w / Rb(tot.v[..., None], tot.e[..., None])
    k = ratio(out, w.v, w.e)
    print(f"[f32 smooth times={times}] kappa {k:.3f} (bound {KAPPA['smooth']})")
    assert k <= KAPPA["smooth"], k
    if times == 0:
        assert np.array_equal(out, x)
