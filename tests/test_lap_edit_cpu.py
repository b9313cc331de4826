"""CPU: the float64 Laplacian-editing oracle (tests/lap_edit_oracle.py, DESIGN section 1g) against the reference's dense
formula on hand-built meshes, the fitting loop against the reference's own (tests/golden/lap_edit_ref.npz), and the
NumPy restatement of the kernel's chunked PCG against the oracle."""
import numpy as np
import pytest

import lap_edit_oracle as lo

# (faces, V, cidx, targets): every component holds a constraint, so the reference's dense inverse exists
HAND = {
    "lone_triangle": ([[0, 1, 2]], 3, [0, 2], [[0.1, 0.0, 0.2], [1.0, 1.2, -0.1]]),
    "strip_with_isolated_vertex": ([[0, 1, 2], [2, 1, 3]], 5, [0, 3, 4], [[0.0, 0.1, 0.0], [1.1, 0.9, 0.3],
                                                                         [2.0, 2.0, 2.0]]),
    "repeated_index_face": ([[0, 0, 1], [0, 1, 2]], 3, [2], [[0.5, -0.5, 0.25]]),
    "duplicate_constraints": ([[0, 1, 2], [1, 3, 2]], 4, [3, 0, 3, 3], [[1.0, 1.0, 0.0], [0.0, 0.0, 0.1],
                                                                       [1.2, 0.8, 0.1], [0.9, 1.1, -0.1]]),
}


def _verts(V, seed=0):
    return np.random.default_rng(seed).uniform(-1, 1, (V, 3))


@pytest.mark.parametrize("name", sorted(HAND))
@pytest.mark.parametrize("c", [1.0, 10.0])
@pytest.mark.parametrize("smooth", [False, True])
def test_oracle_equals_dense_reference(name, c, smooth):
    faces, V, cidx, tgt = HAND[name]
    x = _verts(V)
    y = lo.solve(x, faces, cidx, tgt, c, smooth)
    ref = lo.dense_reference(x, faces, cidx, tgt, c, smooth)
    np.testing.assert_allclose(y, ref, rtol=0, atol=1e-11)


def test_isolated_vertex_and_self_edge_rules():
    # an isolated vertex: L row -e_i, so it is solved on its own ((1 + c n) y = x + c sum u) and smoothed to 0
    faces, V, cidx, tgt = HAND["strip_with_isolated_vertex"]
    x = _verts(V)
    y = lo.solve(x, faces, cidx, tgt, 2.0)
    np.testing.assert_allclose(y[4], (x[4] + 2.0 * np.asarray(tgt[2])) / 3.0, atol=1e-14)
    assert np.array_equal(lo.solve(x, faces, cidx, tgt, 2.0, True)[4], np.zeros(3))
    # the self edge (0, 0) counts twice in deg_0 = 4 but is dropped from the smoothing sum with the diagonal
    faces, V, cidx, tgt = HAND["repeated_index_face"]
    y = lo.solve(_verts(V), faces, cidx, tgt)
    L, adj = lo.laplacian(faces, V)
    assert adj["deg"][0] == 4
    np.testing.assert_allclose(lo.smooth(y, L)[0], (y[1] + y[2]) / 4.0, atol=1e-15)


def test_unconstrained_component_is_unchanged():
    # two triangles with no shared vertex; only the first is constrained
    faces = [[0, 1, 2], [3, 4, 5]]
    x = _verts(6)
    y = lo.solve(x, faces, [0, 1], [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])
    assert np.array_equal(y[3:], x[3:])
    ref = lo.dense_reference(x[:3], [[0, 1, 2]], [0, 1], [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])
    np.testing.assert_allclose(y[:3], ref, atol=1e-12)
    yp, st = lo.pcg(x, faces, [0, 1], [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])
    assert np.array_equal(yp[3:], x[3:]) and st[6] == 1.0
    np.testing.assert_allclose(yp[:3], ref, atol=1e-9)


def test_out_of_range_constraints_are_skipped():
    faces, V, cidx, tgt = HAND["lone_triangle"]
    x = _verts(V)
    y = lo.solve(x, faces, cidx + [-1, 3, 7], tgt + [[9.0, 9, 9]] * 3)
    np.testing.assert_allclose(y, lo.solve(x, faces, cidx, tgt), atol=0)
    _, st = lo.pcg(x, faces, cidx + [-1, 3, 7], tgt + [[9.0, 9, 9]] * 3)
    assert st[7] == 3


@pytest.mark.parametrize("case", [0, 1, 2, 3])
def test_fitting_loop_matches_the_reference(golden, case):
    z = golden("lap_edit_ref.npz")
    fields = dict(waist=z["waist"], hem=z["hem"])
    targets = dict(waist=z["tgt_waist"], hem=z["tgt_hem"])
    r = lo.fit(z["src_v"], z["src_f"], fields, targets, int(z["epoch"]), float(z[f"c_{case}"]),
               bool(z[f"smooth_{case}"]))
    scale = np.abs(z[f"final_v_{case}"] - z["src_v"]).max()
    assert np.array_equal(np.concatenate(r["idx"]), z[f"idx_{case}"])
    assert np.array_equal(np.concatenate(r["tgt"]), z[f"tgt_{case}"])
    assert np.abs(r["epoch_v"] - z[f"epoch_v_{case}"]).max() < 1e-11 * scale
    assert np.abs(r["final_v"] - z[f"final_v_{case}"]).max() < 1e-11 * scale
    # the reference's own fp32 run, for scale: its dense fp32 inverse is far from float64
    assert np.abs(z[f"final_v32_{case}"] - z[f"final_v_{case}"]).max() < 2e-3 * scale


@pytest.mark.parametrize("case", [0, 3])
def test_numpy_pcg_reaches_the_oracle_on_the_fixture(golden, case):
    z = golden("lap_edit_ref.npz")
    n = z[f"count_{case}"]
    c, smooth = float(z[f"c_{case}"]), bool(z[f"smooth_{case}"])
    for e in range(int(z["epoch"])):
        sl = slice(int(n[:e].sum()), int(n[:e + 1].sum()))
        x = z[f"epoch_v_{case}"][e]
        ref = lo.solve(x, z["src_f"], z[f"idx_{case}"][sl], z[f"tgt_{case}"][sl], c, smooth)
        y, st = lo.pcg(x, z["src_f"], z[f"idx_{case}"][sl], z[f"tgt_{case}"][sl], c, smooth_out=smooth)
        assert st[6] == 1.0 and (st[3:6] <= 1e-10).all() and st[7] == 0
        np.testing.assert_allclose(y, ref, rtol=0, atol=1e-8)


def test_numpy_pcg_on_a_tube():
    v, f, loops = lo.tube(60, 30)
    cidx, u = lo.loop_targets(v, loops)
    ref = lo.solve(v, f, cidx, u)
    y, st = lo.pcg(v, f, cidx, u)
    assert st[6] == 1.0 and 0 < st[:3].min() and st[:3].max() < 3000
    np.testing.assert_allclose(y, ref, rtol=0, atol=1e-8)
    # the stop rule is bounded: max_iter ends the solve with the flag at 0
    _, st = lo.pcg(v, f, cidx, u, max_iter=5)
    assert st[6] == 0.0 and st[:3].max() == 5
    # a non-finite input ends it at once with the flag at -1
    x = v.copy()
    x[7, 1] = np.nan
    y, st = lo.pcg(x, f, cidx, u)
    assert st[6] == -1.0 and st[1] == 0 and np.isnan(y[7, 1])
