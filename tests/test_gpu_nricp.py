"""GPU: the NRICP kernels (csrc/nricp.cu, DESIGN section 1f) against the float64 oracle (tests/nricp_oracle.py) and
the reference's own loop (tests/golden/nricp_ref.npz), the C ABI's guards and errors, determinism, launch count and
host synchronisation, and a production-shaped fit against the reference loop restated in torch."""
import contextlib
import ctypes
import io
import os
import sys

import numpy as np
import pytest
import torch

import nricp_oracle as no
from recmv_b200 import _lib, ops
from recmv_b200.registration import NRICP_Optimizer_AdamW

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import bench_nricp  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
LR = 1e-4


def _adj(faces, V):
    f = torch.as_tensor(np.asarray(faces, dtype=np.int64).reshape(-1, 3), device=DEV)
    return ops.mesh_adjacency(f, V)


def _check_adjacency(faces, V):
    row_ptr, col, deg, boundary = (t.cpu().numpy() for t in _adj(faces, V))
    r = no.adjacency(faces, V)
    E2 = row_ptr[-1]
    assert np.array_equal(row_ptr, r["row_ptr"])
    assert np.array_equal(col[:E2], r["col"]) and (col[E2:] == -1).all()
    assert np.array_equal(deg, r["deg"])
    assert np.array_equal(boundary, r["boundary"])


@pytest.mark.parametrize("faces,V", [([[0, 1, 2]], 3), ([[0, 1, 2], [2, 1, 3]], 5), ([[0, 0, 1]], 2),
                                     ([[0, 1, 2], [1, 2, 5], [-1, 0, 1]], 4), ([[3, 3, 3]], 4),
                                     (np.zeros((0, 3), dtype=np.int64), 3)])
def test_adjacency_hand_meshes(faces, V):
    _check_adjacency(faces, V)


def test_adjacency_production_mesh_bit_equal():
    src_v, src_f, tgt_v, tgt_f = bench_nricp.sphere_scene(DEV)
    for f, V in ((src_f, src_v.shape[0]), (tgt_f, tgt_v.shape[0])):
        _check_adjacency(f.cpu().numpy(), V)
    # the open half has a boundary rim, the closed sphere none
    assert _adj(src_f.cpu().numpy(), src_v.shape[0])[3].any()
    assert not _adj(tgt_f.cpu().numpy(), tgt_v.shape[0])[3].any()


def _fixture_state(z, seed, perturb=0.02):
    g = np.random.default_rng(seed)
    x = z["src_v"]
    V = len(x)
    X = no.identity_affine(V) + perturb * g.standard_normal((V, 3, 4))
    n = no.shade_oracle.vertex_normals(x[None], z["src_f"])[0]
    tn = no.shade_oracle.vertex_normals(z["tgt_v"][None], z["tgt_f"])[0]
    keep = z["masks"] > 0
    tv, tn = z["tgt_v"][keep], tn[keep]
    j = no.nearest(no.warp(X, x), tv)
    return X, x, n, tv, tn, j


def _cuda(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), device=DEV).to(dtype)


@pytest.mark.parametrize("gamma,step", [(1.0, 1), (2.0, 1), (1.0, 5)])
def test_one_step_against_float64(golden, gamma, step):
    z = golden("nricp_ref.npz")
    X, x, n, tv, tn, j = _fixture_state(z, 7)
    # round the state to fp32 first, so both sides start from the same numbers
    X, x, n, tv, tn = (np.asarray(np.float32(a), dtype=np.float64) for a in (X, x, n, tv, tn))
    V = len(x)
    adj = no.adjacency(z["src_f"], V)
    L = no.laplacian(adj["edges"], V)
    sw, lw, thr = 5.0, 25.0, 0.3
    g, t = no.gradient(X, x, n, tv[j], tn[j], adj, L, sw, lw, gamma, thr)
    rng = np.random.default_rng(1)
    st = tuple(np.float32(a).astype(np.float64) for a in
               (1e-3 * rng.standard_normal(X.shape), 1e-4 * rng.random(X.shape), 2e-4 * rng.random(X.shape)))
    st = (st[0], st[1], np.maximum(st[1], st[2]))
    if step == 1:
        st = (np.zeros_like(X),) * 3
    X1, st1 = no.adamw_step(X, g, st, step)

    Xd = _cuda(X)
    mom = tuple(_cuda(a) for a in st)
    d_adj = _adj(z["src_f"], V)
    stats = ops.nricp_step(_cuda(x), _cuda(n), _cuda(tv), _cuda(tn), _cuda(j, torch.int64), d_adj, Xd, mom, step, sw,
                           lw, gamma=gamma, threshold=thr).cpu().numpy()
    # the gate: vertices whose cosine is within fp32 rounding of the threshold may go either way
    _, n2, ok = no.warp(X, x, n)
    cos = no.cosine(tn[j], n2)
    ambiguous = int((np.abs(cos - thr) < 1e-5).sum())
    assert abs(stats[4] - t["w"].sum()) <= ambiguous
    terms = [abs(stats[k] - ref) / abs(ref) for k, ref in
             ((0, t["data"]), (1, t["stiff"]), (2, t["lap"]), (3, t["loss"]), (5, t["S"]))]
    upd = np.abs(Xd.cpu().numpy() - X1).max() / LR
    msg = f"terms rel {max(terms):.3e} update/lr {upd:.3e} gate {stats[4]} vs {t['w'].sum()} (ambiguous {ambiguous})"
    if step == 1:   # exp_avg = (1 - beta1) g exactly: the gradient itself
        gd = mom[0].cpu().numpy().astype(np.float64) / 0.1
        gerr = np.abs(gd - g).max() / np.abs(g).max()
        msg += f" grad rel {gerr:.3e}"
        assert gerr <= 1.5e-5   # measured 4.6e-6 on an H100
    print(msg)
    assert max(terms) <= 3e-7   # measured 8.0e-8
    # the update in units of lr: Adam's normalisation turns gradient noise near eps into step-sized differences
    assert upd <= 4e-3   # measured 1.3e-3


def test_zero_S_gives_nan_like_torch():
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "nricp_ref.npz"))
    x = z["src_v"]
    V = len(x)
    X = _cuda(no.identity_affine(V))
    mom = tuple(torch.zeros_like(X) for _ in range(3))
    stats = ops.nricp_step(_cuda(x), _cuda(np.ones((V, 3))), _cuda(x), _cuda(np.ones((V, 3))),
                           torch.arange(V, device=DEV), _adj(z["src_f"], V), X, mom, 1, 5.0, 25.0, threshold=2.0)
    assert stats[5].item() == 0.0 and stats[4].item() == 0.0
    assert torch.isnan(X).all()   # s = 1 / (2 sqrt(0)) = +inf times zero residuals, as torch's sqrt backward gives


def _replay(z, case):
    """The fitting loop on ops, recording the vertices at every epoch start."""
    x = _cuda(z["src_v"])
    f = _cuda(z["src_f"], torch.int64)
    tv, tf = _cuda(z["tgt_v"]), _cuda(z["tgt_f"], torch.int64)
    n = ops.vertex_normals(x[None], f)[0]
    tn = ops.vertex_normals(tv[None], tf)[0]
    keep = _cuda(z["masks"]) > 0
    tv, tn = tv[keep].contiguous(), tn[keep].contiguous()
    V = x.shape[0]
    adj = ops.mesh_adjacency(f, V)
    X = _cuda(no.identity_affine(V))
    mom = tuple(torch.empty_like(X) for _ in range(3))
    stats = torch.zeros(ops.NRICP_STATS, device=DEV)
    sws, lws, mile = list(z["stiffness_weight"]), list(z["laplacian_weight"]), list(z["mile_stone"])
    out, mi, launches = [], 0, set()
    for e in range(int(z["epoch"])):
        v = ops.nricp_warp(X, x)
        out.append(v.cpu().numpy())
        _, idx = ops.knn_nearest(v[None], tv[None])
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for t in range(1, (100 if e == 0 else int(z["inner_iter"])) + 1):
                l0 = ops.launch_count()
                ops.nricp_step(x, n, tv, tn, idx[0], adj, X, mom, t, float(sws[mi]), float(lws[mi]),
                               gamma=float(z[f"gamma_{case}"]), threshold=float(z[f"threshold_{case}"]), stats=stats)
                launches.add(ops.launch_count() - l0)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        if e + 1 in mile:
            mi += 1
    return np.stack(out), ops.nricp_warp(X, x).cpu().numpy(), X, stats, launches


@pytest.mark.parametrize("case", [0, 1])
def test_fixture_replay_fp32(golden, case):
    z = golden("nricp_ref.npz")
    ev, fv, X, stats, launches = _replay(z, case)
    assert launches == {2}
    scale = np.abs(z[f"final_v_{case}"] - z["src_v"]).max()
    err = max(np.abs(ev - z[f"epoch_v_{case}"]).max(), np.abs(fv - z[f"final_v_{case}"]).max()) / scale
    print(f"case {case}: max vertex error / total displacement = {err:.3e}")
    assert err < 7e-4   # measured 2.1e-4 (case 0) and 1.5e-4 (case 1)
    # two runs are bit-identical
    ev2, fv2, X2, stats2, _ = _replay(z, case)
    assert np.array_equal(ev, ev2) and np.array_equal(fv, fv2)
    assert torch.equal(X, X2) and torch.equal(stats, stats2)


def test_drop_in_on_the_fixture(golden, tmp_path, capsys):
    z = golden("nricp_ref.npz")
    opt = NRICP_Optimizer_AdamW(epoch=int(z["epoch"]), dense_pcl=1, use_normal=True,
                                stiffness_weight=list(z["stiffness_weight"]), mile_stone=list(z["mile_stone"]),
                                inner_iter=int(z["inner_iter"]), laplacian_weight=list(z["laplacian_weight"]),
                                gamma=float(z["gamma_0"]), threshold=float(z["threshold_0"]))
    src = bench_nricp.Mesh(_cuda(z["src_v"]), _cuda(z["src_f"], torch.int64))
    loss, out = opt(smpl_slice=src, cano_meshes=bench_nricp.Mesh(_cuda(z["tgt_v"]), _cuda(z["tgt_f"], torch.int64)),
                    save_path=str(tmp_path), garment_name="patch", static_pts_type=[], nricp_masks=_cuda(z["masks"]))
    assert loss.dim() == 0 and loss.is_cuda
    scale = np.abs(z["final_v_0"] - z["src_v"]).max()
    assert np.abs(out.vertices.cpu().numpy() - z["final_v_0"]).max() < 7e-4 * scale
    lines = [s for s in capsys.readouterr().out.splitlines() if "NRICP avg_update" in s]
    assert len(lines) == int(z["epoch"])
    obj = tmp_path / "nricp_deform" / "patch" / f"{int(z['epoch'])}.obj"
    recs = obj.read_text().splitlines()
    assert sum(r.startswith("v ") for r in recs) == len(z["src_v"])
    assert sum(r.startswith("f ") for r in recs) == len(z["src_f"])
    # unsupported inputs
    with pytest.raises(NotImplementedError):
        NRICP_Optimizer_AdamW(epoch=1, dense_pcl=1, use_normal=False, stiffness_weight=[1.0],
                              laplacian_weight=[1.0])(smpl_slice=src, cano_meshes=src, save_path=None,
                                                      garment_name="p", static_pts_type=[], nricp_masks=None)
    with pytest.raises(ValueError):
        opt(smpl_slice=src, cano_meshes=bench_nricp.Mesh(_cuda(z["tgt_v"]), _cuda(z["tgt_f"], torch.int64)),
            save_path=None, garment_name="p", static_pts_type=[], nricp_masks=torch.zeros(len(z["tgt_v"]), device=DEV))


def test_guarded_buffers_and_argument_errors(golden):
    z = golden("nricp_ref.npz")
    lib = _lib.load()
    x = _cuda(z["src_v"])
    f = _cuda(z["src_f"], torch.int64)
    V, F = x.shape[0], f.shape[0]
    G = 64
    nan = float("nan")

    def guarded(n, dtype=torch.float32, fill=nan):
        return torch.full((n + 2 * G,), fill, dtype=dtype, device=DEV)

    row_ptr, col, deg = guarded(V + 1, torch.int32, -7), guarded(6 * F, torch.int32, -7), guarded(V, torch.int32, -7)
    bnd = guarded(V, torch.uint8, 7)
    nb = ctypes.c_size_t(0)
    assert lib.recmv_mesh_adjacency_workspace_bytes(V, F, ctypes.byref(nb)) == 0
    ws = torch.empty(nb.value, dtype=torch.uint8, device=DEV)
    p = lambda t, o=G: ctypes.c_void_p(t.data_ptr() + o * t.element_size())  # noqa: E731
    st = ops._stream(x)
    assert lib.recmv_mesh_adjacency(p(f, 0), F, V, p(ws, 0), p(row_ptr), p(col), p(deg), p(bnd), st) == 0
    X = guarded(12 * V)
    X[G:G + 12 * V] = _cuda(no.identity_affine(V)).reshape(-1)
    v_out, n_out, ok = guarded(3 * V), guarded(3 * V), guarded(V, torch.uint8, 7)
    n = ops.vertex_normals(x[None], f)[0]
    assert lib.recmv_nricp_warp(p(X), p(x, 0), p(n, 0), V, p(v_out), p(n_out), p(ok), st) == 0
    mom = [guarded(12 * V) for _ in range(3)]
    stats = guarded(8)
    assert lib.recmv_nricp_workspace_bytes(V, ctypes.byref(nb)) == 0
    ws2 = torch.empty(nb.value, dtype=torch.uint8, device=DEV)
    idx = torch.arange(V, device=DEV)
    tv = (x + 0.01).contiguous()   # a non-zero residual: S > 0
    prm = _lib.NricpParams(5.0, 25.0, 1.0, 0.3, 1e-4, 0.9, 0.999, 1e-8, 1e-2, 1)
    args = [p(x, 0), p(n, 0), p(tv, 0), p(n, 0), V, p(idx, 0), p(row_ptr), p(col), p(bnd), V, ctypes.byref(prm), p(X),
            p(mom[0]), p(mom[1]), p(mom[2]), p(ws2, 0), p(stats), st]
    assert lib.recmv_nricp_step(*args) == 0
    torch.cuda.synchronize()
    for t, n_in in ((row_ptr, V + 1), (col, 6 * F), (deg, V), (bnd, V), (X, 12 * V), (v_out, 3 * V), (n_out, 3 * V),
                    (ok, V), (mom[0], 12 * V), (mom[1], 12 * V), (mom[2], 12 * V), (stats, 8)):
        head, body, tail = t[:G], t[G:G + n_in], t[G + n_in:]
        if t.dtype == torch.float32:
            assert torch.isnan(head).all() and torch.isnan(tail).all() and torch.isfinite(body).all()
        else:
            assert (head == head[0]).all() and (tail == head[0]).all()
    assert torch.equal(v_out[G:G + 3 * V], x.reshape(-1))   # identity warp
    # argument errors
    assert lib.recmv_mesh_adjacency(p(f, 0), -1, V, p(ws, 0), p(row_ptr), p(col), p(deg), p(bnd), st) == -3
    assert lib.recmv_mesh_adjacency(None, F, V, p(ws, 0), p(row_ptr), p(col), p(deg), p(bnd), st) == -1
    assert lib.recmv_nricp_warp(None, p(x, 0), None, V, p(v_out), None, None, st) == -1
    assert lib.recmv_nricp_warp(p(X), p(x, 0), None, -1, p(v_out), None, None, st) == -3
    bad = list(args)
    bad[10] = None
    assert lib.recmv_nricp_step(*bad) == -1
    prm0 = _lib.NricpParams(5.0, 25.0, 1.0, 0.3, 1e-4, 0.9, 0.999, 1e-8, 1e-2, 0)
    bad[10] = ctypes.byref(prm0)
    assert lib.recmv_nricp_step(*bad) == -3
    adj = ops.mesh_adjacency(f, V)
    Xt = _cuda(no.identity_affine(V))
    m3 = tuple(torch.zeros_like(Xt) for _ in range(3))
    with pytest.raises(RuntimeError):
        ops.mesh_adjacency(f.int(), V)
    with pytest.raises(RuntimeError):
        ops.nricp_warp(Xt.double(), x)
    with pytest.raises(RuntimeError):
        ops.nricp_step(x, n, x, n, idx.int(), adj, Xt, m3, 1, 1.0, 1.0)
    with pytest.raises(RuntimeError):
        ops.nricp_step(x, n, x, n, idx, adj, Xt[:-1], m3, 1, 1.0, 1.0)
    with pytest.raises(RuntimeError):
        ops.nricp_step(x.cpu(), n, x, n, idx, adj, Xt, m3, 1, 1.0, 1.0)


def test_production_fit_against_torch_loop():
    src_v, src_f, tgt_v, tgt_f = bench_nricp.sphere_scene(DEV)
    V = src_v.shape[0]
    assert 4e4 <= V <= 7e4
    sched = dict(epoch=3, inner_iter=50, stiffness_weight=[50.0, 20.0], laplacian_weight=[250.0, 250.0],
                 mile_stone=[2], threshold=0.3)
    ref_v, ref_w = bench_nricp.torch_fit(src_v, src_f, tgt_v, tgt_f, **sched)
    opt = NRICP_Optimizer_AdamW(dense_pcl=4e4, use_normal=True, **sched)
    with contextlib.redirect_stdout(io.StringIO()) as buf:
        _, out = opt(smpl_slice=bench_nricp.Mesh(src_v.clone(), src_f), cano_meshes=bench_nricp.Mesh(tgt_v, tgt_f),
                     save_path=None, garment_name="sphere", static_pts_type=[],
                     nricp_masks=torch.ones(tgt_v.shape[0], device=DEV))
    ours = out.vertices

    def dist(v):   # mean distance to the nearest target point
        d, _ = ops.knn_nearest(v[None].contiguous(), tgt_v[None])
        return d.sqrt().mean().item()

    d0, d_ref, d_ours = dist(src_v), dist(ref_v), dist(ours)
    count = int(buf.getvalue().splitlines()[-1].split("valid")[1].split("/")[0])
    print(f"mean distance: start {d0:.5f} torch {d_ref:.5f} fused {d_ours:.5f}; gate torch {int(ref_w.sum())} "
          f"fused {count}; max vertex difference {(ours - ref_v).abs().max().item():.3e}")
    assert d_ours < 0.9 * d0
    assert abs(d_ours - d_ref) <= 2e-3 * d_ref   # measured 6e-4 relative (0.03178 vs 0.03180)
    assert abs(count - int(ref_w.sum())) <= 1e-3 * V   # measured equal (54 621)
