"""GPU: the callers either side of the fused kernels -- Newton-like surface solve (A10), cardinal rays and
deformed normals (A7), coarse-to-fine sweep + marching cubes (A11/A13) -- against goldens produced by the
reference's own functions on its own modules (tests/golden/make_golden.py)."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_golden, norm_err
sys.path.insert(0, GOLDEN)
import make_golden as mg  # noqa: E402  (scene builders shared with the generator)
from oracle import oracle_torch as ot  # noqa: E402
from recmv_b200 import _lib, ops, synth  # noqa: E402
from recmv_b200 import model as M  # noqa: E402
from recmv_b200 import utils as U  # noqa: E402
from recmv_b200.MCAcc import Seg3dLossless  # noqa: E402
from recmv_b200.discretize import discretize_sdf  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


class _Mods:  # the scene builder expects module namespaces
    getTmpSdf = staticmethod(M.getTmpSdf)
    MLPTranslator, LBSkinner, CompositeDeformer = M.MLPTranslator, M.LBSkinner, M.CompositeDeformer


def _scene():
    sdf, deformer = mg.surface_scene(_Mods, _Mods, device="cpu")
    return sdf.to(DEV), deformer.to(DEV)


RATIO = {"sdfRatio": 0.8, "deformerRatio": 0.6, "renderRatio": 0.9}


@pytest.mark.parametrize("mode,min_agree", [(_lib.MLP_FP32_SIMT, 0.99), (_lib.MLP_TC_F16X3, 0.97)])
def test_surface_solve_matches_reference(mode, min_agree):
    g = load_golden("surface.npz")
    t = {k: torch.from_numpy(v).to(DEV) for k, v in g.items()}
    sdf, deformer = _scene()
    sdf.mlp_mode = mode
    defconds = [t["conds"], [t["poses"], t["trans"]]]
    cam = torch.tensor(synth.CAM_POS, device=DEV)
    ps, ok = U.OptimizeGarmentSurfaceSinlge(cam, t["rays"], t["seeds"].clone(), t["batch_inds"], sdf, RATIO,
                                            deformer, defconds, dthreshold=1.e-4, athreshold=0.05, w1=3.05,
                                            w2=1., times=10, offset_type="body")
    agree = (ok == t["ok"]).float().mean().item()
    both = ok & t["ok"]
    print(f"mode {mode}: converged {int(ok.sum())} (reference {int(t['ok'].sum())}), flag agreement {agree:.4f}, "
          f"max |dp| on common {(ps - t['ps'])[both].abs().max().item():.2e}")
    assert agree >= min_agree
    # fp32 mode takes the very same iterations as the reference.  In tc3 mode a point can pass the acceptance
    # test one iteration earlier or later (|sdf| < 1e-4 with ~1e-5 arithmetic noise), so positions agree to
    # within the acceptance ball: angle < 0.05 deg at ~2.4 units from the camera = 2.1e-3.
    assert (ps - t["ps"])[both].abs().max() < (2e-6 if mode == _lib.MLP_FP32_SIMT else 2.1e-3)
    # single iteration: deterministic update formula p <- p - L g/|g|^2
    ps1, ok1 = U.OptimizeSurfacePs(cam, t["rays"], t["seeds"].clone(), t["batch_inds"], sdf, RATIO,
                                   lambda p, c, i, **kw: deformer(p, c, i, ratio=kw["ratio"], offset_type="body"),
                                   defconds, dthreshold=1.e-4, athreshold=0.05, times=1)
    assert (ok1 == t["ok_1it"]).float().mean() >= min_agree
    # tc3: |f| of a seed can be ~1e-5 = the arithmetic noise, where sign(f) (hence that one step) may flip
    assert (ps1 - t["ps_1it"]).abs().max() < (5e-5 if mode == _lib.MLP_FP32_SIMT else 1e-3)


def test_cardinal_rays_and_normals_match_reference():
    g = load_golden("surface.npz")
    t = {k: torch.from_numpy(v).to(DEV) for k, v in g.items()}
    sdf, deformer = _scene()
    defconds = [t["conds"], [t["poses"], t["trans"]]]
    pts = t["ps"].clone().requires_grad_(True)
    crays, ds = U.compute_cardinal_rays(deformer, pts, t["rays"], defconds, t["batch_inds"], RATIO, "test", "body")
    assert norm_err(ds, t["ds"]) < 1e-4 and (crays - t["crays"]).abs().max() < 2e-4
    pts2 = t["ps"].clone().requires_grad_(True)
    nrm, _ = U.compute_deformed_normals(sdf, deformer, pts2, defconds, t["batch_inds"], RATIO, "test", "body")
    assert (nrm - t["normals"]).abs().max() < 2e-4
    # train phase builds the second-order graph through the CUDA sampler's double backward
    pts3 = t["ps"][:64].clone().requires_grad_(True)
    cr, _ = U.compute_cardinal_rays(deformer, pts3, t["rays"][:64], [t["conds"], [t["poses"], t["trans"]]],
                                    t["batch_inds"][:64], RATIO, "train", "body")
    cr.pow(2).sum().backward()
    assert torch.isfinite(pts3.grad).all()


def test_c2f_sweep_and_discretize_on_gpu():
    sys.path.insert(0, os.path.dirname(__file__))
    from test_c2f_cpu import KW, sphere_query
    eng = Seg3dLossless(sphere_query, **KW).to(DEV)
    out = eng.forward()
    # the CPU sweep's grid, which tests/test_c2f_cpu.py pins bit for bit to the reference class's
    gold = Seg3dLossless(sphere_query, **KW).forward()[0, 0].to(DEV)
    assert (out[0, 0] - gold).abs().max() < 2e-6 and bool(((out[0, 0] > 0) == (gold > 0)).all())
    # network as query function: fused launches, watertight mesh close to the analytic level set
    sdf = M.getTmpSdf(DEV, 6, 0.6, 256)
    eng2 = Seg3dLossless(None, b_min=[-1, -1, -1], b_max=[1, 1, 1], resolutions=[17, 33, 65, 129],
                         align_corners=False, balance_value=0.0).to(DEV)
    v, f = discretize_sdf(sdf, eng2, None)
    assert sdf.last_path == "fused" and v.shape[0] > 1000 and f.min() >= 0
    e = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]).sort(dim=1).values
    assert bool((torch.unique(e, dim=0, return_counts=True)[1] == 2).all())
    with torch.no_grad():
        assert sdf(v, None).abs().max() < 2e-3       # vertices sit on the zero level set (cell size 0.0155)
    assert sum(s[3] for s in eng2.stats) < 0.25 * 129 ** 3


@pytest.mark.parametrize("resolutions", [[17, 33, 65, 129], [(15, 21, 9), (29, 41, 17), (57, 81, 33), (113, 161, 65)],
                                         # the full production 'coarse' pyramid of train.py:42-48
                                         [(15, 21, 9), (29, 41, 17), (57, 81, 33), (113, 161, 65), (225, 321, 129)]])
def test_c2f_device_worklist_is_bit_identical_to_the_torch_path(resolutions):
    """Seg3dLossless with the sweep as a device worklist (recmv_c2f_refine / recmv_sdf_mlp_fwd_counted /
    recmv_c2f_scatter_list / recmv_c2f_mark_conflicts): same voxels re-queried, same query-point arithmetic -> the grid equals
    the torch-op path's (itself bit-identical to the reference class, tests/test_c2f_cpu.py) bit for bit, per-level
    statistics included; isotropic pyramid and the anisotropic 'coarse' pyramid of train.py:42-48 (halved)."""
    from recmv_b200 import testing
    sdf = testing.build_sdf(M.getTmpSdf, seed=0, perturb_seed=101).to(DEV)
    aniso = not isinstance(resolutions[0], int)
    eng = Seg3dLossless(None, b_min=[-0.7, -1.0, -0.4] if aniso else [-1, -1, -1], b_max=[0.7, 1.0, 0.4] if aniso else [1, 1, 1],
                        resolutions=resolutions, align_corners=False, balance_value=0.0).to(DEV)

    def q(points):
        with torch.no_grad():
            return sdf.forward(points.reshape(-1, 3), 0.8).reshape(1, 1, -1)
    eng.query_func = q
    with torch.no_grad():
        g_torch = eng.forward().clone()
    assert eng.last_sweep_path == "fused"
    st_torch = list(eng.stats)
    q.recmv_sdf = (sdf, 0.8)
    with torch.no_grad():
        g_dev = eng.forward()
    assert eng.last_sweep_path == "device-worklist"
    assert torch.equal(g_dev, g_torch)
    assert list(eng.stats) == st_torch
    ops.check_async_errors()


def test_fused_translator_and_deformer_match_reference():
    """A4 / A5: MLPTranslator alone (golden from the reference class) and the CompositeDeformer = translator +
    LBS in one launch (golden `ds` from the reference CompositeDeformer)."""
    g = load_golden("translator.npz")
    torch.manual_seed(1)
    tr = M.MLPTranslator(128, 6)
    from recmv_b200 import testing
    testing.perturb_module(tr, 202, scale=0.5)
    tr = tr.to(DEV)
    t = {k: torch.from_numpy(v).to(DEV) for k, v in g.items() if k not in ("param_names", "param_sums")}
    with torch.no_grad():
        out = tr(t["p"], t["conds"], t["batch_inds"], ratio={"deformerRatio": 0.6}, offset_type="body")
    assert tr.last_path == "fused"
    print(f"translator: out {norm_err(out, t['out']):.2e} offset {norm_err(tr.offset['body'], t['offset']):.2e}")
    assert norm_err(out, t["out"]) < 1e-4 and norm_err(tr.offset["body"], t["offset"]) < 2e-4
    with torch.no_grad():   # [N,V,3] call form
        out2 = tr(t["p"][:1500].view(3, 500, 3), t["conds"], None, ratio={"deformerRatio": 0.6}, offset_type="b2")
    ref2 = None
    tr.mlp_mode = _lib.MLP_FP32_SIMT   # explicit composite path for comparison
    with torch.no_grad():
        ref2 = tr(t["p"][:1500].view(3, 500, 3), t["conds"], None, ratio={"deformerRatio": 0.6}, offset_type="b3")
    assert tr.last_path == "autograd-composite" and norm_err(out2, ref2) < 1e-4
    # composite deformer
    gs = load_golden("surface.npz")
    ts = {k: torch.from_numpy(v).to(DEV) for k, v in gs.items()}
    sdf, deformer = _scene()
    with torch.no_grad():
        ds = deformer(ts["ps"], [ts["conds"], [ts["poses"], ts["trans"]]], ts["batch_inds"], ratio=RATIO,
                      offset_type="body")
    assert deformer.defs[0].last_path == "fused-deformer"
    print(f"composite deformer: {norm_err(ds, ts['ds']):.2e}")
    assert norm_err(ds, ts["ds"]) < 1e-4
    ops.check_async_errors()


def test_fused_rendernet_matches_reference():
    """A8: the colour MLP in one tensor-core launch vs the golden of the reference class (same seeds => same params),
    plus a ragged size (not a multiple of the 128-row tile) against the torch composite on the same module."""
    from recmv_b200 import testing
    g = dict(load_golden("rendernet.npz"), **load_golden("rendernet_feats.npz"))
    torch.manual_seed(2)
    rn = M.RenderingNetwork_view_norm(256, d_in=9, d_out=3, dims=[512] * 4, mode="idr", weight_norm=True,
                                      multires_v=4, multires_n=0)
    testing.perturb_module(rn, 303)
    rn = rn.to(DEV)
    t = {k: torch.from_numpy(g[k]).to(DEV) for k in ("points", "normals", "view_dirs", "feats", "out")}
    with torch.no_grad():
        col = rn(t["points"], t["normals"], t["view_dirs"], t["feats"], {"renderRatio": 0.8})
    assert rn.last_path == "fused"
    err = norm_err(col, t["out"])
    print(f"rendernet fused vs reference golden: max abs err / rms {err:.2e}")
    assert err < 1e-4
    n = 777
    with torch.no_grad():
        a = rn(t["points"][:n], t["normals"][:n], t["view_dirs"][:n], t["feats"][:n], {"renderRatio": None})
        rn.mlp_mode = _lib.MLP_FP32_SIMT   # no SIMT colour kernel: selects the torch composite
        b = rn(t["points"][:n], t["normals"][:n], t["view_dirs"][:n], t["feats"][:n], {"renderRatio": None})
    assert rn.last_path == "autograd-composite" and norm_err(a, b) < 1e-4
    ops.check_async_errors()


def test_fused_deformer_jacobian_matches_autograd():
    """A7: D(p) and J = dD/dp from ONE forward-mode launch of the fused deformer vs three autograd passes through
    the torch translator + CUDA sampler (utils.compute_Jacobian, the reference's procedure); then the reference
    goldens of the quantities built from J (cardinal rays, deformed normals) through the fused path."""
    g = load_golden("surface.npz")
    t = {k: torch.from_numpy(v).to(DEV) for k, v in g.items()}
    sdf, deformer = _scene()
    defconds = [t["conds"], [t["poses"], t["trans"]]]
    with torch.no_grad():
        ds, J = deformer.value_and_jacobian(t["ps"], defconds, t["batch_inds"], ratio=RATIO, offset_type="body")
    assert deformer.defs[0].last_path == "fused-deformer-jvp"
    pts = t["ps"].clone().requires_grad_(True)
    ds_ref = deformer(pts, defconds, t["batch_inds"], ratio=RATIO, offset_type="body")
    assert deformer.defs[0].last_path == "fused-train"      # translator on the tensor-core training path, LBS on the CUDA sampler
    J_ref = U.compute_Jacobian(pts, ds_ref, False, False)
    print(f"fused deformer JVP: ds {norm_err(ds, ds_ref):.2e}  J {norm_err(J, J_ref):.2e}")
    assert norm_err(ds, t["ds"]) < 1e-4 and norm_err(J, J_ref) < 2e-4
    crays, ds2 = U.compute_cardinal_rays(deformer, t["ps"].clone().requires_grad_(True), t["rays"], defconds,
                                         t["batch_inds"], RATIO, "test", "body")
    assert deformer.defs[0].last_path == "fused-deformer-jvp"
    assert norm_err(ds2, t["ds"]) < 1e-4 and (crays - t["crays"]).abs().max() < 2e-4
    nrm, _ = U.compute_deformed_normals(sdf, deformer, t["ps"].clone().requires_grad_(True), defconds,
                                        t["batch_inds"], RATIO, "test", "body")
    assert (nrm - t["normals"]).abs().max() < 2e-4
    ops.check_async_errors()


def test_interp2x_boundary3d_and_fused_sweep_bookkeeping():
    """A11 helpers: order 0 == the restated reference kernel (bit-exact), order 1 == F.interpolate on the values and
    on the occupancy flags (bit-exact: the default sweep stays bit-identical), backward, the dilated todo mask, the
    drop-in module under its reference name, and the whole sweep with / without the fused bookkeeping."""
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(4)
    for shape in ((1, 1, 9, 10, 11), (2, 3, 5, 4, 6), (1, 1, 33, 33, 33)):
        x = torch.randn(shape, generator=g)
        o_ref, f_ref = ot.interp2x_boundary3d(x, 0.1)
        xd = x.to(DEV)
        o0, f0 = ops.interp2x_boundary3d_forward(xd, 0.1, 0)
        assert torch.equal(o0.cpu(), o_ref) and torch.equal(f0.cpu(), f_ref)
        size = tuple(2 * s - 1 for s in shape[2:])
        o1, f1 = ops.interp2x_boundary3d_forward(xd, 0.1, 1)
        t_val = F.interpolate(xd, size=size, mode="trilinear", align_corners=True)
        t_valid = F.interpolate((xd > 0.1).float(), size=size, mode="trilinear", align_corners=True)
        assert torch.equal(o1, t_val) and torch.equal(f1, (t_valid > 0) & (t_valid < 1))
        go = torch.randn(o_ref.shape, generator=g)
        gi = ops.interp2x_boundary3d_backward(go.to(DEV))
        assert (gi.cpu() - ot.interp2x_boundary3d_backward(go)).abs().max() < 1e-5
        if shape[:2] == (1, 1):
            done = (torch.rand(o_ref.shape[2:], generator=g) < 0.3).to(DEV)
            smooth = torch.ones(1, 1, 3, 3, 3, device=DEV) / 27.0
            want = (F.conv3d(f1.float(), smooth, padding=1) > 0)[0, 0] & ~done
            assert torch.equal(ops.c2f_todo_mask(f1[0, 0].contiguous(), done), want)
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(__file__)), "recmv_b200", "compat"))
    import interp2x_boundary3d as ext                      # the reference's module name
    out, fl = ext.forward(xd, 0.1)
    assert torch.equal(out, o0) and fl.dtype == torch.bool and ext.backward(go.to(DEV)).shape == xd.shape
    # the sweep: fused bookkeeping (default on CUDA) vs torch ops on the same device, same query function
    sys.path.insert(0, os.path.dirname(__file__))
    from test_c2f_cpu import KW, sphere_query
    eng = Seg3dLossless(sphere_query, **KW).to(DEV)
    a = eng.forward()
    assert eng.last_sweep_path == "fused"
    real = ops.interp2x_boundary3d_forward

    def torch_path(inp, balance, order):
        size = tuple(2 * s - 1 for s in inp.shape[2:])
        v = F.interpolate((inp > balance).float(), size=size, mode="trilinear", align_corners=True)
        return [F.interpolate(inp, size=size, mode="trilinear", align_corners=True), (v > 0) & (v < 1)]
    ops.interp2x_boundary3d_forward = torch_path
    try:
        b = eng.forward()
    finally:
        ops.interp2x_boundary3d_forward = real
    assert torch.equal(a, b)
    eng_c = Seg3dLossless(sphere_query, **{**KW, "use_cuda_impl": True}).to(DEV)   # the reference's optional path
    c = eng_c.forward()
    assert (c - a).abs().max() < 1e-5 and bool(((c > 0) == (a > 0)).all())


def test_surface_grad_coeffs_kernel_and_fused_pipeline():
    """SURVEY 8f rank 1: the per-ray algebra of propagateTmpPsGrad in one kernel vs its torch restatement (oracle,
    fp32 and fp64), incl. FastMinv's singular flag; then the whole autograd-free pipeline (two forward-mode launches +
    the kernel) vs the reference procedure (autograd gradient of f, three autograd passes for J, torch algebra)."""
    g = torch.Generator().manual_seed(9)
    n = 4099
    gl, gf, v, dc = (torch.randn((n, 3), generator=g) for _ in range(4))
    v = v / v.norm(dim=1, keepdim=True)
    J = torch.eye(3).expand(n, 3, 3) + 0.3 * torch.randn((n, 3, 3), generator=g)
    J[:7] = 0.0                                   # singular systems: b^T b has rank 1 -> flag false, zeros
    coef, vec, rg, ok = ops.surface_grad_coeffs(gl.to(DEV), gf.to(DEV), J.to(DEV), v.to(DEV), dc.to(DEV))
    c_o, v_o, r_o, ok_o = ot.surface_grad_coeffs(gl, gf, J, v, dc)
    c64, v64, r64, ok64 = ot.surface_grad_coeffs(gl.double(), gf.double(), J.double(), v.double(), dc.double())
    assert not ok[:7].any() and float(coef[:7].abs().max()) == 0.0
    agree = ok.cpu() == ok_o
    assert agree.float().mean() > 0.999           # |det| within rounding of the 1e-4 threshold may flip
    bm = torch.cat([gf.view(-1, 1, 3), ot.cross_matrix(v).matmul(J)], dim=1).double()
    det = torch.linalg.det(bm.permute(0, 2, 1).matmul(bm))
    sel = (ok.cpu() & ok_o & ok64 & (det.abs() > 5e-2))   # well-conditioned systems (fp32 loses its digits near the threshold)
    assert sel.float().mean() > 0.6
    for a, b in ((coef, c64), (vec, v64), (rg, r64)):
        err = (a.cpu().double()[sel] - b[sel]).abs().max() / b[sel].abs().max()
        assert err < 1e-3, err                     # conditioning of b^T b amplifies fp32 rounding; the fp32 oracle:
    print("kernel vs fp32 restatement:", float((coef.cpu()[sel] - c_o[sel]).abs().max() / c_o[sel].abs().max()))
    # whole pipeline on the scene of the surface goldens
    gs = load_golden("surface.npz")
    t = {k: torch.from_numpy(x).to(DEV) for k, x in gs.items()}
    sdf, deformer = _scene()
    defconds = [t["conds"], [t["poses"], t["trans"]]]
    cam = torch.tensor(synth.CAM_POS, device=DEV)
    glp = torch.randn((t["ps"].shape[0], 3), generator=g).to(DEV)
    coef, vec, rg, ok, d = U.implicit_surface_grad_coeffs(sdf, deformer, t["ps"], t["rays"], glp, defconds,
                                                          t["batch_inds"], RATIO, "body", cam)
    p = t["ps"].clone().requires_grad_(True)
    f = sdf(p, RATIO)
    gfp = torch.autograd.grad(f, p, torch.ones_like(f))[0]
    dd = deformer(p, defconds, t["batch_inds"], ratio=RATIO, offset_type="body")
    Jr = U.compute_Jacobian(p, dd, False, False)
    c_r, v_r, r_r, ok_r = ot.surface_grad_coeffs(glp.cpu(), gfp.cpu(), Jr.cpu(), t["rays"].cpu(), (dd.detach() - cam).cpu())
    bm = torch.cat([gfp.cpu().view(-1, 1, 3), ot.cross_matrix(t["rays"].cpu()).matmul(Jr.cpu())], dim=1).double()
    det = torch.linalg.det(bm.permute(0, 2, 1).matmul(bm))
    sel = ok.cpu() & ok_r & (det.abs() > 5e-2)
    print("pipeline: well-conditioned rays", float(sel.float().mean()))
    assert sel.float().mean() > 0.5
    for a, b in ((coef, c_r), (vec, v_r), (rg, r_r)):
        assert (a.cpu()[sel] - b[sel]).abs().max() / b[sel].abs().max() < 2e-3
    ops.check_async_errors()


def test_device_surface_solve_matches_reference_and_torch_loop():
    """A10 as ONE C call (recmv_surface_solve): against the reference's golden run (same bounds as the tc3 torch
    loop: a point may pass the acceptance test one step earlier or later), against the step-by-step loop on the same
    device, the single-step case, a single-frame call without batch indices, and timing of both."""
    import time
    import importlib
    FSP = importlib.import_module("recmv_b200.utils.FindSurfacePs")   # the module (utils re-exports a function of that name)
    g = load_golden("surface.npz")
    t = {k: torch.from_numpy(v).to(DEV) for k, v in g.items()}
    sdf, deformer = _scene()
    defconds = [t["conds"], [t["poses"], t["trans"]]]
    cam = torch.tensor(synth.CAM_POS, device=DEV)
    kw = dict(dthreshold=1.e-4, athreshold=0.05, w1=3.05, w2=1., times=10, offset_type="body")

    def run(device_solve):
        FSP.DEVICE_SOLVE = device_solve
        try:
            n0 = ops.launch_count()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ps, ok = U.OptimizeGarmentSurfaceSinlge(cam, t["rays"], t["seeds"].clone(), t["batch_inds"], sdf, RATIO,
                                                    deformer, defconds, **kw)
            torch.cuda.synchronize()
            return ps, ok, (time.perf_counter() - t0) * 1e3, ops.launch_count() - n0
        finally:
            FSP.DEVICE_SOLVE = True
    run(True); run(False)                                   # warm-up (weight packing, allocator)
    ps_d, ok_d, ms_d, n_d = run(True)
    ps_t, ok_t, ms_t, n_t = run(False)
    print(f"device solve: {ms_d:.2f} ms, {n_d} launches | torch loop: {ms_t:.2f} ms, {n_t} launches | "
          f"converged {int(ok_d.sum())} / {int(ok_t.sum())} / reference {int(t['ok'].sum())}")
    assert n_d == 3 * 11 + 1 and n_t != n_d                 # bone matrices + (2 forward-mode launches + update) x (times + 1) rounds
    for ps, ok in ((ps_d, ok_d),):
        agree = (ok == t["ok"]).float().mean().item()
        both = ok & t["ok"]
        assert agree >= 0.97 and (ps - t["ps"])[both].abs().max() < 2.1e-3
    both = ok_d & ok_t
    assert (ok_d == ok_t).float().mean() >= 0.97 and (ps_d - ps_t)[both].abs().max() < 2.1e-3
    # converged points satisfy the acceptance test when re-evaluated
    with torch.no_grad():
        f = sdf(ps_d[ok_d], RATIO).view(-1)
        dd = deformer(ps_d[ok_d], defconds, t["batch_inds"][ok_d], ratio=RATIO, offset_type="body") - cam
    up = torch.cross(dd, t["rays"][ok_d], dim=1)
    ang = torch.arcsin(up.norm(dim=1) / dd.norm(dim=1)) * 180. / np.pi
    assert f.abs().max() < 1.2e-4 and ang.max() < 0.051
    # one step
    sdf2, def2 = sdf, deformer
    ps1, ok1 = U.OptimizeGarmentSurfaceSinlge(cam, t["rays"], t["seeds"].clone(), t["batch_inds"], sdf2, RATIO, def2,
                                              defconds, dthreshold=1.e-4, athreshold=0.05, times=1, offset_type="body")
    assert (ok1 == t["ok_1it"]).float().mean() >= 0.97 and (ps1 - t["ps_1it"]).abs().max() < 1e-3
    # one frame, no batch indices
    m = t["batch_inds"] == 0
    ps0, ok0 = ops.surface_solve(cam, t["rays"][m], t["seeds"][m], None, sdf.packed_weights(), sdf._pe_weights(RATIO),
                                 *deformer.device_solve_args([t["conds"][:1], [t["poses"][:1], t["trans"][:1]]], RATIO)[:4],
                                 1.e-4, 0.05, 3.05, 1., 10)
    assert (ok0 == ok_d[m]).float().mean() >= 0.97
    ops.check_async_errors()
