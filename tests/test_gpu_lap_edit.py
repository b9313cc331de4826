"""GPU: the Laplacian-editing solve (csrc/lap_edit.cu, DESIGN section 1g) against the float64 oracle
(tests/lap_edit_oracle.py) and the reference's own fitting loop (tests/golden/lap_edit_ref.npz), on hand-built meshes
and on tubes of 5e3 and 5.5e4 vertices; the drop-in Laplacian_Optimizer; unconstrained components, skipped indices and
non-finite input; determinism across runs and grid sizes; launch count and host synchronisation; argument errors."""
import ctypes

import numpy as np
import pytest
import torch

import lap_edit_oracle as lo
from recmv_b200 import _lib, ops
from recmv_b200.registration import Laplacian_Optimizer

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _cuda(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), device=DEV).to(dtype)


def _solve(x, faces, cidx, ctgt, c=1.0, smooth=True, **kw):
    V = len(x)
    adj = ops.mesh_adjacency(_cuda(np.asarray(faces, dtype=np.int64).reshape(-1, 3), torch.int64), V)
    y, st = ops.laplacian_edit(_cuda(x), adj, _cuda(np.asarray(cidx, dtype=np.int64), torch.int64),
                               _cuda(np.asarray(ctgt).reshape(-1, 3)), c, smooth, **kw)
    return y.cpu().numpy().astype(np.float64), st.cpu().numpy()


def _f32(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


HAND = {
    "lone_triangle": ([[0, 1, 2]], 3, [0, 2], [[0.1, 0.0, 0.2], [1.0, 1.2, -0.1]]),
    "strip_with_isolated_vertex": ([[0, 1, 2], [2, 1, 3]], 5, [0, 3, 4], [[0.0, 0.1, 0.0], [1.1, 0.9, 0.3],
                                                                         [2.0, 2.0, 2.0]]),
    "repeated_index_face": ([[0, 0, 1], [0, 1, 2]], 3, [2], [[0.5, -0.5, 0.25]]),
    "duplicate_constraints": ([[0, 1, 2], [1, 3, 2]], 4, [3, 0, 3, 3], [[1.0, 1.0, 0.0], [0.0, 0.0, 0.1],
                                                                       [1.2, 0.8, 0.1], [0.9, 1.1, -0.1]]),
}


@pytest.mark.parametrize("name", sorted(HAND))
@pytest.mark.parametrize("c,smooth", [(1.0, False), (10.0, True)])
def test_hand_meshes_against_the_oracle(name, c, smooth):
    faces, V, cidx, tgt = HAND[name]
    x = _f32(np.random.default_rng(0).uniform(-1, 1, (V, 3)))
    ref = lo.dense_reference(x, faces, cidx, _f32(tgt), c, smooth)
    y, st = _solve(x, faces, cidx, tgt, c, smooth)
    assert st[6] == 1.0 and st[7] == 0, st
    np.testing.assert_allclose(y, ref, rtol=0, atol=3e-7)   # the fp32 store of values below 3


def _fixture_case(z, case):
    n = z[f"count_{case}"]
    for e in range(int(z["epoch"])):
        sl = slice(int(n[:e].sum()), int(n[:e + 1].sum()))
        yield e, z[f"idx_{case}"][sl], z[f"tgt_{case}"][sl]


@pytest.mark.parametrize("case", [0, 1, 2, 3])
def test_fixture_replayed_through_ops(golden, case):
    z = golden("lap_edit_ref.npz")
    c, smooth = float(z[f"c_{case}"]), bool(z[f"smooth_{case}"])
    scale = np.abs(z[f"final_v_{case}"] - z["src_v"]).max()
    worst = 0.0
    for e, idx, tgt in _fixture_case(z, case):
        nxt = z[f"epoch_v_{case}"][e + 1] if e + 1 < int(z["epoch"]) else z[f"final_v_{case}"]
        y, st = _solve(_f32(z[f"epoch_v_{case}"][e]), z["src_f"], idx, tgt, c, smooth)
        assert st[6] == 1.0 and st[7] == 0
        worst = max(worst, np.abs(y - nxt).max() / scale)
    ref32 = np.abs(z[f"final_v32_{case}"] - z[f"final_v_{case}"]).max() / scale
    print(f"case {case}: ours {worst:.3e} of the displacement per epoch, the reference's fp32 run {ref32:.3e}")
    assert worst < 2e-5   # the fp32 rounding of the input and the output


def test_drop_in_on_the_fixture(golden, tmp_path, monkeypatch):
    z = golden("lap_edit_ref.npz")
    monkeypatch.chdir(tmp_path)
    for case in range(4):
        tmpl = lo.Template(z["src_v"], z["src_f"], dict(waist=z["waist"], hem=z["hem"]), dtype=torch.float32,
                           device=DEV)
        curves = [lo.Curve(_cuda(z["tgt_waist"])), lo.Curve(_cuda(z["tgt_hem"]))]
        opt = Laplacian_Optimizer(epoch=int(z["epoch"]), constrain_weight=float(z[f"c_{case}"]),
                                  smooth=bool(z[f"smooth_{case}"]))
        out = opt(source_fl_meshes=[tmpl], target_meshes=curves, source_type=["skirt"],
                  target_fl_type=["waist", "hem"], outlayer=True)
        assert out["source_fl_meshes"][0] is tmpl and tmpl.updates == int(z["epoch"])
        scale = np.abs(z[f"final_v_{case}"] - z["src_v"]).max()
        assert np.array_equal(np.concatenate([m[1] for m in tmpl.matches]), z[f"idx_{case}"])
        assert np.abs(tmpl.vertices.cpu().numpy() - z[f"final_v_{case}"]).max() < 2e-5 * scale
        assert opt.stats[6].item() == 1.0
    # the debug files of the last epoch: vertex-only binary PLYs of the matched source points and the targets
    idx, tgt = tmpl.matches[-1][1], tmpl.matches[-1][2]
    for name, pts in (("source_0.ply", tmpl.matches[-1][0][idx]), ("target_0.ply", tgt)):
        raw = (tmp_path / "debug" / "register" / name).read_bytes()
        head, body = raw.split(b"end_header\n")
        assert b"element vertex %d" % len(idx) in head
        np.testing.assert_array_equal(np.frombuffer(body, dtype="<f4").reshape(-1, 3), np.float32(pts))


def _tube(nt, nz):
    v, f, loops = lo.tube(nt, nz)
    cidx, u = lo.loop_targets(v, loops)
    return _f32(v), f, cidx, _f32(u)


@pytest.mark.parametrize("nt,nz", [(100, 50), (330, 168)])
def test_tubes_against_spsolve(nt, nz):
    x, f, cidx, u = _tube(nt, nz)
    ref = lo.solve(x, f, cidx, u, 1.0)
    y, st = _solve(x, f, cidx, u, 1.0, smooth=False)
    err = np.abs(y - ref).max()
    print(f"V={len(x)}: iterations {st[:3]}, relative residuals {st[3:6]}, max error {err:.3e}, "
          f"displacement {np.abs(ref - x).max():.3f}")
    assert st[6] == 1.0 and (st[3:6] <= 1e-10).all()
    assert err < 1e-6


def test_unconstrained_component_is_bit_unchanged():
    x, f, cidx, u = _tube(40, 20)
    V = len(x)
    f2 = np.concatenate([f, f + V])
    x2 = np.concatenate([x, x + 2.0])
    y, st = _solve(x2, f2, cidx, u, 1.0, smooth=False)
    assert st[6] == 1.0
    assert np.array_equal(np.float32(y[V:]), np.float32(x2[V:]))
    np.testing.assert_allclose(y[:V], lo.solve(x, f, cidx, u), rtol=0, atol=1e-6)


def test_out_of_range_indices_are_skipped_and_counted():
    x, f, cidx, u = _tube(40, 20)
    V = len(x)
    bad = np.array([-5, V, V + 100, -1])
    y0, s0 = _solve(x, f, cidx, u, smooth=False)
    y1, s1 = _solve(x, f, np.concatenate([bad[:2], cidx, bad[2:]]), np.concatenate([np.ones((2, 3)), u,
                                                                                    np.ones((2, 3))]), smooth=False)
    assert s0[7] == 0 and s1[7] == 4
    assert np.array_equal(y0, y1)


def test_non_finite_input_ends_with_a_flag():
    x, f, cidx, u = _tube(40, 20)
    x[7, 1] = np.nan
    y, st = _solve(x, f, cidx, u, smooth=False)
    assert st[6] == -1.0 and st[1] == 0
    assert np.isnan(y[7, 1])
    u2 = u.copy()
    u2[3, 0] = np.inf
    _, st = _solve(_tube(40, 20)[0], f, cidx, u2, smooth=False)
    assert st[6] == -1.0


def test_max_iter_bounds_the_solve():
    x, f, cidx, u = _tube(100, 50)
    _, st = _solve(x, f, cidx, u, smooth=False, max_iter=7)
    assert st[6] == 0.0 and st[:3].max() == 7
    _, st_np = lo.pcg(x, f, cidx, u, max_iter=7)
    assert np.array_equal(st[:3], st_np[:3])


def test_bit_identical_across_runs_and_grid_sizes():
    x, f, cidx, u = _tube(100, 50)
    adj = ops.mesh_adjacency(_cuda(f, torch.int64), len(x))
    args = (_cuda(x), adj, _cuda(cidx, torch.int64), _cuda(u))
    runs = [ops.laplacian_edit(*args, 10.0, True, max_blocks=b) for b in (0, 0, 1, 7)]
    y0, s0 = runs[0]
    assert s0[6].item() == 1.0
    for y, s in runs[1:]:
        assert torch.equal(y, y0) and torch.equal(s, s0)
    # and the iteration counts follow the NumPy restatement of the algorithm
    _, st_np = lo.pcg(x, f, cidx, u, 10.0)
    assert np.abs(s0[:3].cpu().numpy() - st_np[:3]).max() <= 0.02 * st_np[:3].max() + 2


def test_no_host_sync_and_three_launches():
    x, f, cidx, u = _tube(100, 50)
    adj = ops.mesh_adjacency(_cuda(f, torch.int64), len(x))
    args = (_cuda(x), adj, _cuda(cidx, torch.int64), _cuda(u))
    stats = torch.zeros(ops.LAP_EDIT_STATS, device=DEV)
    ops.laplacian_edit(*args, stats=stats)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        l0 = ops.launch_count()
        y, st = ops.laplacian_edit(*args, stats=stats)
        launches = ops.launch_count() - l0
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert launches == 3 and st is stats
    assert stats[6].item() == 1.0


def test_abi_and_wrapper_argument_errors():
    lib = _lib.load()
    x, f, cidx, u = _tube(20, 10)
    V, M = len(x), len(cidx)
    xd, ci, ud = _cuda(x), _cuda(np.sort(cidx), torch.int64), _cuda(u)
    row_ptr, col, deg, _ = adj = ops.mesh_adjacency(_cuda(f, torch.int64), V)
    nb = ctypes.c_size_t(0)
    assert lib.recmv_lap_edit_workspace_bytes(V, M, ctypes.byref(nb)) == 0
    assert lib.recmv_lap_edit_workspace_bytes(-1, M, ctypes.byref(nb)) == -3
    assert lib.recmv_lap_edit_workspace_bytes(V, M, None) == -1
    assert lib.recmv_lap_edit_workspace_bytes(V, M, ctypes.byref(nb)) == 0
    ws = torch.empty(nb.value, dtype=torch.uint8, device=DEV)
    out = torch.empty((V, 3), device=DEV)
    stats = torch.empty(8, device=DEV)
    p = ops._ptr
    st = ops._stream(xd)
    good = [p(xd), V, p(row_ptr), p(col), p(deg), p(ci), p(ud), M, 1.0, 1e-10, 100, 1, 0, p(ws), p(out), p(stats), st]
    assert lib.recmv_lap_edit_solve(*good) == 0
    for k, val, code in ((0, None, -1), (2, None, -1), (5, None, -1), (13, None, -1), (15, None, -1), (1, -1, -3),
                         (7, -1, -3), (10, 0, -3), (9, 0.0, -3), (9, -1e-3, -3), (8, -1.0, -3), (12, -2, -3)):
        bad = list(good)
        bad[k] = val
        assert lib.recmv_lap_edit_solve(*bad) == code, (k, val)
    with pytest.raises(RuntimeError):
        ops.laplacian_edit(xd.cpu(), adj, ci, ud)
    with pytest.raises(RuntimeError):
        ops.laplacian_edit(xd.double(), adj, ci, ud)
    with pytest.raises(RuntimeError):
        ops.laplacian_edit(xd, adj, ci.int(), ud)
    with pytest.raises(RuntimeError):
        ops.laplacian_edit(xd, adj, ci, ud[:-1])
    with pytest.raises(RuntimeError):
        ops.laplacian_edit(xd[:-1], adj, ci, ud)
    with pytest.raises(RuntimeError):
        ops.laplacian_edit(xd, adj, ci, ud, max_iter=0)
