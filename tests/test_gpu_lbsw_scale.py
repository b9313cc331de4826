"""The skinning-voxel kernels (csrc/lbsw_field.cu) bit for bit against their float32 restatement (tests/lbsw_f32.py).

kNN blend: every checked voxel's 24 weights and its out_idx list must equal the restatement, on the production voxel
at k = 1, 7, 8, 9, 15, 16, 17, 30, 31 and 32 (both sides of the TopK<8> / <16> / <32> dispatch) with both values of
align_corners, and on adversarial vertex sets.  Smoothing: every voxel of the output, on the production grid and on
small and ragged grids.  The restatement itself is held to float64 by tests/test_lbsw_f32_cpu.py.

Restated on subsets where the whole would be slow: of the production voxel's 1.9 M kNN voxels, the z = 0 and z = 32
slices, the x = 0 and x = 128 slices, the grid's 12 edges (its corners included) and 50 000 random voxels; the 30
smoothing passes on the 30^3 boxes at the low and the high corner of the grid (restated from a 60^3 crop: a voxel
30 or more voxels inside a crop face is unaffected by that face after 30 passes).
"""
import os

import numpy as np
import pytest
import torch

import lbsw_f32 as lf
from recmv_b200 import _lib, ops, synth

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, "golden", "lbsw_ref.npz"))
BMIN, BMAX = G["bmin"].astype(np.float32).tolist(), G["bmax"].astype(np.float32).tolist()
PROD = (129, 225, 65)          # (W, H, D) of the production voxel
KS = [1, 7, 8, 9, 15, 16, 17, 30, 31, 32]


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    eq = (a.view(np.uint32) == b.view(np.uint32)) | ((a == 0) & (b == 0)) | (np.isnan(a) & np.isnan(b))
    bad = np.argwhere(~eq)
    return None if not len(bad) else (tuple(bad[0]), a[tuple(bad[0])], b[tuple(bad[0])], int(len(bad)))


def body():
    v, w = synth.body_points()
    return v.numpy(), w.numpy()


def production_voxels(seed=0):
    W, H, D = PROD
    x, y, z = np.meshgrid(np.arange(W), np.arange(H), np.arange(D), indexing="ij")
    x, y, z = x.ravel(), y.ravel(), z.ravel()
    flat = (z * H + y) * W + x
    on = (z == 0) | (z == 32) | (x == 0) | (x == W - 1)
    edge = (((x == 0) | (x == W - 1)).astype(int) + ((y == 0) | (y == H - 1)) + ((z == 0) | (z == D - 1))) >= 2
    rnd = np.random.default_rng(seed).choice(W * H * D, 50_000, replace=False)
    return np.unique(np.concatenate([flat[on | edge], rnd]))


def check_knn(verts, ws, res, ks, ac, sel=None, label=""):
    """Runs the kernel at each k and compares the voxels `sel` (default all) with the restatement."""
    W, H, D = res
    sel = np.arange(W * H * D) if sel is None else sel
    c = lf.centres(sel, res, ac, BMIN, BMAX)
    s, ids = lf.neighbours(torch.as_tensor(c, device=DEV), torch.as_tensor(verts, device=DEV), xp=torch)
    vt, wt = torch.as_tensor(verts, device=DEV).contiguous(), torch.as_tensor(ws, device=DEV).contiguous()
    sel_t = torch.as_tensor(sel, device=DEV)
    for k in ks:
        out, idx = ops.lbsw_knn_blend(vt, wt, BMIN, BMAX, res, k, ac, want_idx=True)
        got = out.view(-1, 24)[sel_t].cpu().numpy()
        gi = idx[sel_t].cpu().numpy()
        ref, ri = lf.blend(s, ids, ws, k)
        bad = np.nonzero((gi != ri).any(1))[0]
        assert not len(bad), (label, k, ac, int(sel[bad[0]]), gi[bad[0]], ri[bad[0]], len(bad))
        d = same_bits(got, ref)
        assert d is None, (label, k, ac, d)
    print(f"[knn {label}] res={res} ac={ac} V={len(verts)} k={ks}: {len(sel)} voxels bit-exact (weights and indices)")


@pytest.mark.parametrize("ac", [False, True])
def test_production_voxel_knn_bit_exact(ac):
    v, w = body()
    check_knn(v, w, PROD, KS, ac, production_voxels(int(ac)), "production")


RES_SMALL = (9, 13, 7)


def _rows(g, V):
    v, w = body()
    i = g.choice(len(v), V, replace=False)
    return v[i].copy(), w[i].copy()


@pytest.mark.parametrize("V", [1, 2, 3, 4, 5])
def test_every_tail_of_the_4_wide_scan(V):
    v, w = _rows(np.random.default_rng(V), V)
    check_knn(v, w, RES_SMALL, [k for k in (1, 2, 3, 4, 5) if k <= V], False, label=f"V={V}")


@pytest.mark.parametrize("k", [7, 8, 9, 16, 17, 32])
def test_k_equals_v(k):
    v, w = _rows(np.random.default_rng(100 + k), k)
    check_knn(v, w, RES_SMALL, [k], True, label=f"V=k={k}")


def test_shared_memory_limit():
    """14 336 vertices (224 KB of float4) is the most the kernel takes; 14 337 is refused with RECMV_E_RANGE."""
    g = np.random.default_rng(7)
    v0, w0 = body()
    i = g.integers(0, len(v0), 14_337)
    v = (v0[i] + g.normal(scale=0.01, size=(len(i), 3))).astype(np.float32)
    w = w0[i]
    sel = np.random.default_rng(8).choice(33 * 57 * 17, 4000, replace=False)
    check_knn(v[:14_336], w[:14_336], (33, 57, 17), [1, 8, 16, 32], False, sel, label="V=14336")
    with pytest.raises(_lib.RecmvError):
        ops.lbsw_knn_blend(torch.as_tensor(v, device=DEV), torch.as_tensor(w, device=DEV), BMIN, BMAX, (9, 13, 7), 4)


def test_adversarial_vertices():
    """Duplicated vertices (exact ties go to the lower index), voxel centres exactly on vertices (the 1e-4 clamp), all
    distances above 1 (the clamp to 1: equal weights), and a NaN vertex (never a neighbour)."""
    g = np.random.default_rng(9)
    res = (9, 13, 7)
    v0, w0 = _rows(g, 600)
    dup = np.concatenate([v0, v0[::-1], v0[:40]])                                 # every distance 2 or 3 times
    wd = np.concatenate([w0, w0[::-1, ::-1], w0[:40]])
    check_knn(dup.copy(), wd.copy(), res, KS, False, label="duplicated")
    on = lf.centres(np.arange(0, 9 * 13 * 7, 5), res, False, BMIN, BMAX)         # vertices on voxel centres
    von = np.concatenate([on, v0[: 600 - len(on)]]).astype(np.float32)
    check_knn(von, w0.copy(), res, [1, 8, 9, 32], False, label="on centres")
    far = (v0 * 0.1 + np.float32(3.0)).astype(np.float32)                        # every distance > 1
    check_knn(far, w0.copy(), res, [1, 9, 32], True, label="far")
    vn = v0.copy()
    vn[[0, 17, 599], 1] = np.nan
    check_knn(vn, w0.copy(), res, [1, 8, 16, 32], False, label="NaN vertices")
    check_knn(vn[:8].copy(), w0[:8].copy(), res, [8], False, label="NaN vertex, k = V")


# ---- smoothing ------------------------------------------------------------------------------------------------------
def random_field(shape, seed):
    g = np.random.default_rng(seed)
    x = g.random(tuple(shape) + (24,), dtype=np.float32) ** 4
    return (x / x.sum(-1, keepdims=True)).astype(np.float32)


def smooth_gpu(x, times, zero_below):
    _, out_cl = ops.lbsw_smooth(torch.as_tensor(x, device=DEV).contiguous(), times, zero_below)
    return out_cl.cpu().numpy()


@pytest.mark.parametrize("zero_below", [0.0, 5e-3])
@pytest.mark.parametrize("times", [0, 1, 2])
def test_production_grid_smooth_bit_exact(times, zero_below):
    W, H, D = PROD
    x = random_field((D, H, W), 20 + times)
    d = same_bits(smooth_gpu(x, times, zero_below), lf.smooth(x, times, zero_below))
    assert d is None, (times, zero_below, d)


@pytest.mark.parametrize("zero_below", [0.0, 5e-3])
def test_production_grid_30_passes_bit_exact(zero_below):
    W, H, D = PROD
    x = random_field((D, H, W), 30)
    got = smooth_gpu(x, 30, zero_below)
    B, T = 30, 30
    lo = lf.smooth(x[:B + T, :B + T, :B + T], 30, zero_below)[:B, :B, :B]
    hi = lf.smooth(x[D - B - T:, H - B - T:, W - B - T:], 30, zero_below)[T:, T:, T:]
    assert same_bits(got[:B, :B, :B], lo) is None
    assert same_bits(got[D - B:, H - B:, W - B:], hi) is None


@pytest.mark.parametrize("shape", [(1, 1, 1), (2, 9, 9), (9, 2, 9), (9, 9, 2), (3, 3, 3), (5, 7, 11), (17, 3, 5)])
@pytest.mark.parametrize("times", [0, 1, 2, 30])
def test_small_and_ragged_grids_smooth_bit_exact(shape, times):
    """No interior voxel, a single interior voxel (3^3), and voxel counts that are not a multiple of 256."""
    x = random_field(shape, times)
    for zb in (0.0, 5e-3):
        d = same_bits(smooth_gpu(x, times, zb), lf.smooth(x, times, zb))
        assert d is None, (shape, times, zb, d)
