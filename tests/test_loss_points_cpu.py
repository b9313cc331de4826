"""CPU tests of the loss-point oracle (oracle/loss_points_oracle.py, DESIGN section 1k), which the GPU tests hold the
sampler to bit for bit: the float32 threshold rule torch applies, the normal sampler's distribution, the range of the
global points, the counters of lanes, garments and successive calls, the frame means' VJPs against finite
differences, and the oracle against the reference's own `surface_render_loss` (tests/golden/
surface_render_loss_ref.npz): its kept rows, torch's own threshold comparison, and the fixture's regeneration."""
import os

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import loss_points_oracle as lpo, refload

SEED = 0x0123456789ABCDEF


def test_threshold_is_the_float32_quotient():
    S, V = 2048, 80000
    thr = lpo.threshold(S, V)
    assert thr == np.float32(S / V) and float(thr) < S / V       # rounds below the double quotient
    assert not (thr < thr)                                        # a uniform equal to it is not kept
    assert lpo.threshold(2048, 2048) == 1.0 and lpo.threshold(2048, 2047) > 1.0
    with pytest.raises(ValueError):
        lpo.threshold(2048, 0)


def test_every_vertex_is_kept_at_or_below_S():
    for V in (2047, 2048):
        assert len(lpo.draw(SEED, 0, 0, lpo.E_DRAW, V + 10, V, 2048)) == V
    keep = lpo.draw(SEED, 0, 0, lpo.E_DRAW, 80010, 80000, 2048)
    assert abs(len(keep) - 2048) < 5 * np.sqrt(2048) and np.all(np.diff(keep) > 0)


def test_normals_are_standard_normal_and_rarely_flagged():
    z, flag = lpo.normals(SEED, np.arange(200000, dtype=np.uint64))
    for k in range(3):
        assert stats.kstest(z[:, k].astype(np.float64), "norm").pvalue > 1e-3
    assert abs(float(np.corrcoef(z[:, 0], z[:, 1])[0, 1])) < 0.01
    assert flag.sum() <= 3


def test_global_points_lie_in_range():
    g = lpo.global_points(SEED, np.arange(100000, dtype=np.uint64))
    assert g.dtype == np.float32 and g.min() >= -1.8 and g.max() < 1.8
    # the extremes of u: 0 -> -1.8f, 1 - 2^-24 -> 1.8f - 2^-22
    u = np.array([0, 0xFFFFFFFF], np.uint32)
    ext = lpo.unit24(u) * np.float32(3.6) - np.float32(1.8)
    assert ext[0] == np.float32(-1.8) and ext[1] == np.float32(1.8) - np.float32(2.0 ** -22)


def test_counters_are_disjoint_across_lanes_garments_and_calls():
    rng = np.random.default_rng(0)
    Ms, Vs = (37, 0, 120), (300, 10, 2500)
    used, offset = [], (1 << 32) - 900
    for call in range(2):
        base = 0
        for M, V in zip(Ms, Vs):
            C = M + V
            n = {lpo.E_DRAW: V, lpo.D_DRAW: V, lpo.E_LOCAL: C, lpo.E_GLOBAL: C // 6, lpo.D_LOCAL: C}
            for lane, k in n.items():
                used.append(lpo.counters(offset, base, lane, C, k))
            base += lpo.LANES * C
        out, nxt = lpo.sample([rng.standard_normal((M, 3)) for M in Ms], [rng.standard_normal((V, 3)) for V in Vs],
                              [rng.uniform(size=M) < 0.5 for M in Ms], SEED, offset)
        assert nxt == offset + base
        offset = nxt
    allc = np.concatenate(used)
    assert len(np.unique(allc)) == len(allc) and allc.max() > (1 << 32)


def test_sample_layout():
    rng = np.random.default_rng(1)
    P, V = rng.standard_normal((50, 3)).astype(np.float32), rng.standard_normal((9000, 3)).astype(np.float32)
    check = rng.uniform(size=50) < 0.6
    (o,), _ = lpo.sample([P], [V], [check], SEED, 11)
    nE, nD = 50 + len(o["keep_e"]), 50 + len(o["keep_d"])
    assert o["X_E"].shape == (nE + nE // 6, 3) and o["X_D"].shape == (2 * nD, 3)
    assert np.array_equal(o["X_D"][:50], P) and np.array_equal(o["X_D"][50:nD], V[o["keep_d"]])
    assert np.abs(o["X_E"][:50] - P).max() < 0.1 and np.abs(o["X_D"][nD:] - o["X_D"][:nD]).max() < 0.1
    assert not np.array_equal(o["keep_e"], o["keep_d"])
    assert np.array_equal(o["checked"], np.flatnonzero(check))


def _fd(f, x, eps=1e-6):
    g = np.zeros_like(x)
    for i in np.ndindex(x.shape):
        xp, xm = x.copy(), x.copy()
        xp[i] += eps
        xm[i] -= eps
        g[i] = (f(xp) - f(xm)) / (2 * eps)
    return g


def test_frame_mean_vjps_match_finite_differences():
    rng = np.random.default_rng(2)
    M, N = 12, 4
    b = rng.integers(0, N, M)
    b[b == 2] = 0                                                # an empty frame
    gtn = rng.standard_normal((M, 3))
    gtn[0] *= 1e-6                                               # invalid
    J = np.eye(3) + 0.3 * rng.standard_normal((M, 3, 3))
    nx = rng.standard_normal((M, 3))
    w = rng.uniform(size=M)
    L, dg, dJ, dnx = lpo.normal_mean(gtn, J, nx, w, b, N, 1.0)
    assert np.allclose(dg, _fd(lambda x: lpo._frame_mean_normal(x, J, nx, w, b, N), gtn), atol=1e-6)
    assert np.allclose(dJ, _fd(lambda x: lpo._frame_mean_normal(gtn, x, nx, w, b, N), J), atol=1e-6)
    assert np.allclose(dnx, _fd(lambda x: lpo._frame_mean_normal(gtn, J, x, w, b, N), nx), atol=1e-6)
    H, W = 3, 4
    gt = rng.uniform(size=(N, H, W, 3)).astype(np.float32)
    r, c = rng.integers(0, H, M), rng.integers(0, W, M)
    col = rng.uniform(size=(M, 3)).astype(np.float32)
    L, dcol = lpo.color_mean(gt, b, r, c, col, N)
    e = np.abs(gt[b, r, c].astype(np.float64) - col).sum(1)
    n = np.bincount(b, minlength=N)
    assert abs(L - sum(e[b == f].sum() / max(n[f], 1) for f in range(N)) / N) < 1e-6
    assert np.allclose(np.abs(dcol).sum(1), 3 / (N * n[b]))


# ---- the reference's own surface_render_loss (tests/golden/surface_render_loss_ref.npz) ----------------------------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURE = os.path.join(GOLDEN, "surface_render_loss_ref.npz")


def test_oracle_reproduces_the_fixtures_kept_rows():
    z = np.load(FIXTURE)
    seed, offset = int(z["seed"]), int(z["offset"])
    P = [z[f"in/P_{g}"] for g in range(2)]
    V = [z[f"in/V_{g}"] for g in range(2)]
    chk = [z[f"in/check_{g}"] for g in range(2)]
    out, _ = lpo.sample(P, V, chk, seed, offset)
    for tag in ("f32", "f64"):
        for g, o in enumerate(out):
            # the points the reference's own `TmpVs[torch.rand(V) < S / V]` kept, bit for bit
            for lane, keep in (("B_E", o["keep_e"]), ("B_D", o["keep_d"])):
                want = np.concatenate([P[g], V[g][keep]]).astype(z[f"{tag}/{lane}_{g}"].dtype)
                assert np.array_equal(z[f"{tag}/{lane}_{g}"], want), (tag, lane, g)
            k = o["checked"]
            assert np.array_equal(z[f"{tag}/TmpPs_{g}"], P[g][k].astype(z[f"{tag}/TmpPs_{g}"].dtype))
            assert np.array_equal(z[f"{tag}/rays_c_{g}"], z[f"in/rays_{g}"][k].astype(z[f"{tag}/rays_c_{g}"].dtype))
            for key in ("batch", "row", "col"):
                assert np.array_equal(z[f"{tag}/{key}_c_{g}"], z[f"in/{key}_{g}"][k])
            if tag == "f32":   # the reference's local samples are the oracle's rows bit for bit
                nE = len(P[g]) + len(o["keep_e"])
                z_e = np.asarray(o["X_E"][:nE])
                assert np.array_equal(z_e[~o["flag_e"][:nE]], lpo.local(z["f32/B_E_" + str(g)], lpo.normals(
                    seed, lpo.counters(offset, 5 * sum(len(P[h]) + len(V[h]) for h in range(g)), lpo.E_LOCAL,
                                       len(P[g]) + len(V[g]), nE))[0])[~o["flag_e"][:nE]])


def test_torch_keeps_what_the_threshold_rule_keeps():
    """`torch.rand(V) < float(S) / float(V)` on the CPU, evaluated by torch itself: a uniform equal to fp32(S / V) and
    its float32 neighbours are kept exactly as lpo.draw's `u < threshold(S, V)` keeps them."""
    for S, V in ((2048, 80000), (2048, 2300), (4096, 4097), (1365, 80001)):
        thr = lpo.threshold(S, V)
        u = np.concatenate([lpo.unit24(np.arange(0, 1 << 32, 4099, dtype=np.uint64).astype(np.uint32)),
                            [np.nextafter(thr, np.float32(0)), thr, np.nextafter(thr, np.float32(1))]]).astype(np.float32)
        u = u[u < 1]
        kept_torch = (torch.from_numpy(u) < float(S) / float(V)).numpy()
        assert np.array_equal(kept_torch, u < thr), (S, V)


@pytest.mark.skipif(not refload.available(), reason="needs the reference source tree")
def test_surface_render_loss_generator_reproduces_the_fixture():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_surface_render_loss",
                                                  os.path.join(GOLDEN, "make_golden_surface_render_loss.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    new = gen.generate()
    z = np.load(FIXTURE)
    assert sorted(new) == sorted(z.files)
    for key in z.files:
        a, b = new[key], z[key]
        if "/grad/" in key or "/loss" in key or "/info/" in key:
            # CPU torch may split its sums by thread count: float32 values to 1e-4 of the tensor's scale, float64 to 1e-10
            tol = (1e-4 if key.startswith("f32") else 1e-10) * max(float(np.abs(b).max(initial=0)), 1e-30)
            assert float(np.abs(a - b).max(initial=0)) <= tol, key
        else:
            assert np.array_equal(a, b), key
