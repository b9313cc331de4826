"""GPU tests of the feature-curve kernels (csrc/curve_fit.cu, csrc/curve_project.cu, DESIGN section 1n) and the
`project_2d_loss` drop-in (utils.make_project_2d_loss): the curves, the regulariser and their backward against the
float64 oracle (oracle/curve_oracle.py) and torch's float32 autograd at the kinks; the screen points, flags and
compacted clouds against the oracle and `fl_proj_loss`'s own compaction; the projection backward against the float64
Jacobian; run-to-run identity; the refusals; and the drop-in of both classes against the reference's method restated
in torch on the same networks (tests/project_2d_scene.py), with its host synchronisations counted."""
import os
import sys
import warnings

import numpy as np
import pytest
import torch

from oracle import curve_oracle as co
from recmv_b200 import _lib, ops, utils

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
DEV = torch.device("cuda", 0)


def _ulps(got, ref):
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    return (np.abs(got - ref) / np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)).max()


def _rel(got, ref):
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    return np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30)


# ---- the curve kernel -----------------------------------------------------------------------------------------------

def _curve_inputs(C, S, seed, case="random"):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    th = torch.linspace(0, 2 * np.pi, S + 1)[:-1]
    ring = torch.stack([th.cos(), th.sin(), 0.05 * (3 * th).sin()], -1)
    center = r(C, 1, 3) * 0.3
    verts = center + ring[None] * (0.1 + 0.2 * torch.rand(C, 1, 1, generator=g)) + r(C, S, 3) * 1e-3
    dirs = (verts - center) / ((verts - center).norm(dim=-1, keepdim=True) + 1e-6)
    init_scale = ((verts - center) * dirs).sum(-1, keepdim=True).clamp_min(0.)
    nx = torch.nn.functional.normalize(r(C, 1, 3), dim=-1)
    scale = 1.0 + 0.05 * r(C, S, 1)
    nx_scale = 0.01 * r(C, S, 1)
    if case == "kinks":
        scale[0, 3] = 0.                                             # relu(0)
        scale[1, 7:9] = 0.                                           # three equal points: two zero-length segments
        dirs[1, 7:10] = dirs[1, 9]
        init_scale[1, 7:10] = init_scale[1, 9]
        nx_scale[1, 7:10] = nx_scale[1, 9]
        scale[1, 9] = 0.
        dirs[2, 10:20] = dirs[2, 10]                                 # collinear: ten points on one ray
        nx_scale[2, 10:20] = 0.
    return [t.contiguous().to(DEV) for t in (center, dirs, init_scale, nx, scale, nx_scale)]


def _oracle_args(ins):
    center, dirs, s0, nx, scale, t = (x.double().cpu().numpy() for x in ins)
    C, S = dirs.shape[:2]
    return center.reshape(C, 3), dirs, s0.reshape(C, S), nx.reshape(C, 3), scale.reshape(C, S), t.reshape(C, S)


@pytest.mark.parametrize("C,S", [(6, 200), (1, 2), (3, 1024), (5, 37)])
def test_curve_forward_within_2_ulp_of_float64(C, S):
    ins = _curve_inputs(C, S, seed=C * 1000 + S)
    v, reg = ops.curve_fit(*ins)
    center, dirs, s0, nx, scale, t = _oracle_args(ins)
    vo = co.curve_points(center, dirs, s0, nx, scale, t)
    do, ceno = co.regularizer(vo, center)
    assert _ulps(v.cpu(), vo) <= 2
    assert _ulps(reg[:, 0].cpu(), do) <= 2
    assert _ulps(reg[:, 1].cpu(), ceno) <= 2


@pytest.mark.parametrize("C,S", [(6, 200), (1, 2), (3, 1024)])
def test_curve_backward_against_float64_vjp(C, S):
    ins = _curve_inputs(C, S, seed=7 + S)
    g = torch.Generator().manual_seed(S)
    dv = torch.randn(C, S, 3, generator=g).to(DEV)
    dreg = torch.randn(C, 2, generator=g).to(DEV)
    dscale, dnx = ops.curve_fit_backward(*ins, dv, dreg)
    center, dirs, s0, nx, scale, t = _oracle_args(ins)
    vo = co.curve_points(center, dirs, s0, nx, scale, t)
    gv = co.regularizer_vjp(vo, center, dreg[:, 0].double().cpu().numpy(), dreg[:, 1].double().cpu().numpy())
    ds, dt = co.curve_vjp(dirs, s0, nx, scale, gv + dv.double().cpu().numpy())
    assert _rel(dscale.view(C, S).cpu(), ds) <= 4e-7
    assert _rel(dnx.view(C, S).cpu(), dt) <= 4e-7


def test_curve_backward_at_the_kinks_against_float64_vjp():
    # relu(0), two zero-length segments (gradients of ~1e14) and collinear points: each curve to its own largest entry
    ins = _curve_inputs(3, 64, seed=3, case="kinks")
    g = torch.Generator().manual_seed(4)
    dv = torch.randn(3, 64, 3, generator=g).to(DEV)
    dreg = torch.randn(3, 2, generator=g).to(DEV)
    dscale, dnx = ops.curve_fit_backward(*ins, dv, dreg)
    center, dirs, s0, nx, scale, t = _oracle_args(ins)
    vo = co.curve_points(center, dirs, s0, nx, scale, t)
    gv = co.regularizer_vjp(vo, center, dreg[:, 0].double().cpu().numpy(), dreg[:, 1].double().cpu().numpy())
    ds, dt = co.curve_vjp(dirs, s0, nx, scale, gv + dv.double().cpu().numpy())
    assert dscale[0, 3, 0] == 0 and ds[0, 3] == 0
    assert np.abs(dt[1]).max() > 1e6 * np.abs(dt[0]).max()       # the zero-length segments' ~1e14 gradients
    for c in range(3):
        assert _rel(dscale[c].view(-1).cpu(), ds[c]) <= 4e-7, c
        assert _rel(dnx[c].view(-1).cpu(), dt[c]) <= 4e-7, c


def test_curve_kinks_match_torch_float32_autograd():
    import project_2d_scene as ps
    ins = _curve_inputs(3, 64, seed=3, case="kinks")
    scale = ins[4].clone().requires_grad_()
    t = ins[5].clone().requires_grad_()
    curve = ps.Curve.__new__(ps.Curve)
    torch.nn.Module.__init__(curve)
    for name, x in zip(("cano_verts_center", "cano_v_dirs", "init_scale", "cano_nx"), ins[:4]):
        curve.register_buffer(name, x)
    curve.scale, curve.nx_scale = torch.nn.Parameter(scale), torch.nn.Parameter(t)
    g = torch.Generator().manual_seed(4)
    dv = torch.randn(3, 64, 3, generator=g).to(DEV)
    ref_reg = curve.regularization(torch.ones(1, device=DEV))
    (ref_reg['diff_a_loss'] * 0.7 + (curve() * dv).sum()).backward()
    s2, t2 = ins[4].clone().requires_grad_(), ins[5].clone().requires_grad_()
    v, reg = ops.CurveFitFunction.apply(*ins[:4], s2, t2)
    (reg[:, 0].sum() * 0.7 + (v * dv).sum()).backward()
    assert s2.grad[0, 3, 0] == 0 and curve.scale.grad[0, 3, 0] == 0           # relu'(0) = 0
    assert torch.isfinite(s2.grad).all()
    # the zero-length segments put gradients of ~1e14 on curve 1; each curve is held to its own largest entry.  The
    # float32 reference rounds every difference of nearby points (1e-5 relative at these spacings), the kernel does not
    for c in range(3):
        assert _rel(s2.grad[c].cpu(), curve.scale.grad[c].cpu()) <= 1e-4, c
        assert _rel(t2.grad[c].cpu(), curve.nx_scale.grad[c].cpu()) <= 1e-4, c
    assert abs(reg[:, 0].sum().item() - ref_reg['diff_a_loss'].item()) <= 1e-5 * abs(ref_reg['diff_a_loss'].item())


def test_curve_runs_are_bit_identical():
    ins = _curve_inputs(6, 200, seed=11)
    dv = torch.randn(6, 200, 3, device=DEV)
    dreg = torch.randn(6, 2, device=DEV)
    a = ops.curve_fit(*ins) + ops.curve_fit_backward(*ins, dv, dreg)
    b = ops.curve_fit(*ins) + ops.curve_fit_backward(*ins, dv, dreg)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_curve_refusals():
    ins = _curve_inputs(2, 16, seed=1)
    with pytest.raises(RuntimeError):
        ops.curve_fit(*[x.cpu() for x in ins])
    with pytest.raises(RuntimeError):
        ops.curve_fit(ins[0], ins[1].double(), *ins[2:])
    with pytest.raises(RuntimeError):
        ops.curve_fit(ins[0], ins[1], ins[2][:, :8].contiguous(), *ins[3:])
    one = _curve_inputs(1, 2, seed=1)
    with pytest.raises(RuntimeError):                                    # S = 1
        ops.curve_fit(*[x[:, :1].contiguous() if x.shape[1] == 2 else x for x in one])


# ---- the projection kernel ------------------------------------------------------------------------------------------

def _project_case(N, S, sizes=(4, 2), W=1080, H=1080, seed=0):
    """Rows of len(sizes) garments (garment, frame, curve, point), the table, cameras, masks and body checks."""
    g = torch.Generator().manual_seed(seed)
    K = sum(sizes)
    table, base = [], 0
    col = 0
    for Cg in sizes:
        for c in range(Cg):
            table.append((base + c * S, Cg * S, col))
            col += 1
        base += N * Cg * S
    R = base
    X = torch.randn(R, 3, generator=g) * 0.3
    ang = 0.2 * torch.arange(N) - 0.1
    Rm = torch.zeros(N, 3, 3)
    Rm[:, 0, 0], Rm[:, 0, 2], Rm[:, 1, 1], Rm[:, 2, 0], Rm[:, 2, 2] = ang.cos(), -ang.sin(), 1, ang.sin(), ang.cos()
    f = 1.25 * min(H, W)
    cams = torch.cat([torch.tensor([[f, f * 1.01, W / 2 + 0.35, H / 2 - 0.4]]).expand(N, 4), Rm.reshape(N, 9),
                      torch.tensor([[0.02, 0.05, 3.0]]).expand(N, 3)], 1)
    masks = torch.ones(N, K)
    masks[:, 1] = 0.                         # curve 1 unlabelled in every frame
    body = torch.rand(R, generator=g) * 0.2 - 0.05
    thresholds = [0.1, 0.05, 0.05, 0.08, 0.05, 0.05, 0.1, 0.05][:K]
    if N > 1:
        masks[1, :] = 0.                     # frame 1 has no visible point
    body[table[2][0]:table[2][0] + S] = 1.0  # curve 2, frame 0: every point behind the body
    return [X.to(DEV), cams.to(DEV).contiguous(), W, H, table, thresholds, S, masks.to(DEV), body.to(DEV)]


def _dense_rows(table, N, S):
    """[K, N, S] row indices of the table."""
    return np.array([[[b + n * st + s for s in range(S)] for n in range(N)] for b, st, _ in table])


@pytest.mark.parametrize("N,S,W,H", [(3, 200, 1080, 1080), (1, 200, 1283, 721), (2, 5, 64, 48), (3, 1500, 1080, 1080)])
def test_projection_flags_and_clouds(N, S, W, H):
    args = _project_case(N, S, W=W, H=H, seed=N + S)
    X, cams, _, _, table, thresholds, _, masks, body = args
    args[2], args[3] = W, H
    screen, visible, slot, clouds, counts = ops.curve_project(*args)
    rows = _dense_rows(table, N, S)
    K = len(table)
    Xr = X.double().cpu().numpy()[rows]                                      # [K,N,S,3]
    camsd = cams.double().cpu().numpy()
    ref = np.stack([co.screen(Xr[k], camsd, W, H) for k in range(K)])
    got = screen.cpu().numpy()[rows]
    assert _ulps(got, ref) <= 2
    flags = np.stack([(masks[:, c].cpu().numpy()[:, None] != 0) & (body.cpu().numpy()[rows[k]] < np.float32(thr))
                      for k, ((_, _, c), thr) in enumerate(zip(table, thresholds))])
    assert np.array_equal(visible.cpu().numpy()[rows], flags)
    # fl_proj_loss's own compaction of the same screen points
    xy = screen[torch.as_tensor(rows.reshape(K * N, S), device=DEV)][..., :2]
    vis = visible[torch.as_tensor(rows.reshape(K * N, S), device=DEV)]
    order = torch.argsort((~vis).to(torch.uint8), dim=1, stable=True)
    xc = torch.gather(xy, 1, order[..., None].expand(-1, -1, 2))
    assert torch.equal(counts, vis.sum(1))
    cl, ref_cl = clouds.cpu(), xc.cpu()
    for b in range(K * N):
        n = int(counts[b])
        assert torch.equal(cl[b, :n], ref_cl[b, :n])
        assert not cl[b, n:].any()
    cnt = counts.view(K, N).cpu()
    assert (cnt[1] == 0).all()                                 # the curve unlabelled everywhere
    if N > 1:
        assert (cnt[:, 1] == 0).all()                          # the frame without a visible point
    assert cnt[2, 0] == 0
    assert (slot.cpu().numpy()[rows] >= 0).sum() == int(counts.sum())


@pytest.mark.parametrize("N,S", [(3, 200), (1, 37)])
def test_projection_backward_against_float64_jacobian(N, S):
    args = _project_case(N, S, seed=5 * N + S)
    X, cams, W, H, table, thresholds, _, masks, body = args
    Xg = X.clone().requires_grad_()
    screen, visible, counts, clouds = ops.CurveProjectFunction.apply(Xg, cams, W, H, table, thresholds, S, masks, body)
    assert not screen.requires_grad and not visible.requires_grad and not counts.requires_grad
    dcl = torch.randn(clouds.shape, device=DEV)
    (clouds * dcl).sum().backward()
    rows = _dense_rows(table, N, S)
    K = len(table)
    vis = visible.cpu().numpy()[rows]
    ref = np.zeros((X.shape[0], 3))
    dcl_np = dcl.double().cpu().numpy().reshape(K, N, S, 2)
    camsd = cams.double().cpu().numpy()
    for k in range(K):
        for n in range(N):
            idx = np.nonzero(vis[k, n])[0]
            d = np.zeros((1, S, 2))
            d[0, idx] = dcl_np[k, n, :len(idx)]
            g = co.screen_vjp(X.double().cpu().numpy()[rows[k, n]][None], camsd[n:n + 1], W, H, d)[0]
            ref[rows[k, n]] = g * vis[k, n][:, None]
    got = Xg.grad.double().cpu().numpy()
    assert _rel(got, ref) <= 4e-7
    assert not got[~visible.cpu().numpy()].any()


def test_projection_runs_are_bit_identical():
    args = _project_case(3, 200, seed=2)
    a = ops.curve_project(*args)
    b = ops.curve_project(*args)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    dcl = torch.randn(a[3].shape, device=DEV)
    assert torch.equal(ops.curve_project_backward(args[0], args[1], 6, 200, a[2], dcl),
                       ops.curve_project_backward(args[0], args[1], 6, 200, a[2], dcl))


def test_projection_refusals():
    args = _project_case(2, 16, seed=1)
    bad = list(args)
    bad[0] = args[0].cpu()
    with pytest.raises(RuntimeError):
        ops.curve_project(*bad)
    bad = list(args)
    bad[0] = args[0].double()
    with pytest.raises(RuntimeError):
        ops.curve_project(*bad)
    bad = list(args)
    bad[8] = args[8][:-1].contiguous()                                       # body of the wrong length
    with pytest.raises(RuntimeError):
        ops.curve_project(*bad)
    bad = list(args)
    bad[4] = args[4][:-1]                                                    # the table misses rows
    bad[5] = args[5][:-1]
    with pytest.raises(_lib.RecmvError):
        ops.curve_project(*bad)
    bad = list(args)
    bad[4] = [(b, s, 99) for b, s, _ in args[4]]                             # a mask column past M
    with pytest.raises(_lib.RecmvError):
        ops.curve_project(*bad)
    bad = list(args)
    bad[7] = args[7][:1].contiguous()                                        # masks for the wrong frame count
    with pytest.raises(RuntimeError):
        ops.curve_project(*bad)


# ---- the drop-in ----------------------------------------------------------------------------------------------------

def _count(fn, counted=()):
    """(result, host synchronisations of the whole call, of each wrapped (obj, attr) in `counted`)."""
    rec = []
    inner = {}
    for obj, attr in counted:
        f = getattr(obj, attr)
        inner[(id(obj), attr)] = 0

        def wrapped(*a, f=f, key=(id(obj), attr), **k):
            n0 = sum("synchroniz" in str(w.message) for w in rec)
            out = f(*a, **k)
            inner[key] += sum("synchroniz" in str(w.message) for w in rec) - n0
            return out

        setattr(obj, attr, wrapped)
    torch.cuda.synchronize()
    try:
        with warnings.catch_warnings(record=True) as caught:
            rec = caught
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                out = fn()
            finally:
                torch.cuda.set_sync_debug_mode("default")
    finally:
        for obj, attr in counted:
            delattr(obj, attr)          # back to the class's method
    rec[:] = [w for w in rec if "prototype" not in str(w.message)]     # the debug mode's own notice
    total = sum("synchroniz" in str(w.message) for w in rec)
    return out, total, list(inner.values()), [(w.filename, w.lineno) for w in rec if "synchroniz" in str(w.message)]


def _fixture(N):
    from conftest import load_golden
    z = load_golden("project_2d_ref.npz")
    p = f"n{N}/"
    return {k[len(p):]: v for k, v in z.items() if k.startswith(p)}


def _fixture_scene(d):
    """The fixture's `self` and arguments on this package's networks, renderer and z-buffer binding."""
    import project_2d_scene as ps
    import surface_render_scene as srs
    from oracle import zbuf_oracle as zo
    from recmv_b200.compat.MaskRender import mask_renderer
    sdf, deformer, _ = srs.networks(DEV)
    t = lambda k: torch.from_numpy(np.ascontiguousarray(d[k])).to(DEV)  # noqa: E731
    N = int(d["in/poses"].shape[0])
    H, W = 96, 120
    curve = ps.Curve(t("in/curve_verts"), ps.FL_NAMES)
    with torch.no_grad():
        for k in ("cano_smpl_verts", "cano_verts_center", "cano_v_dirs", "cano_nx", "init_scale"):
            getattr(curve, k).copy_(t("in/buf_" + k))
        curve.scale.copy_(t("in/scale"))
        curve.nx_scale.copy_(t("in/nx_scale"))
    poses, trans = t("in/poses").requires_grad_(True), t("in/trans").requires_grad_(True)
    conds = [t("in/conds")[k].requires_grad_(True) for k in range(3)]
    c = t("in/cam")
    cam = zo.Camera(c[:, 0:2].contiguous(), c[:, 2:4].contiguous(), c[:, 4:13].reshape(-1, 3, 3).contiguous(),
                    c[:, 13:16].contiguous(), (W, H))
    me = ps.Model(
        garment_size=2, garment_names=list(ps.GARMENTS), garment_nets=[sdf, sdf], fl_names=list(ps.FL_NAMES),
        garment_vs=[t("in/V_0"), t("in/V_1")], garment_fs=[t("in/F_0"), t("in/F_1")], tmpBodyVs=t("in/body_v"),
        tmpBodyFs=t("in/body_f"), deformer=deformer, conf=ps.Conf(ps.CONF), info={}, sdfShrinkRadius=0.01,
        inter_free_curve=curve, maskRender=mask_renderer((H, W), cameras=cam),
        fl_optimizer=torch.optim.AdamW([curve.scale, curve.nx_scale], lr=1e-4),
        dataset=__import__("types").SimpleNamespace(fl_weights=dict(ps.FL_WEIGHTS)),
        get_grad_parameters=lambda frame_ids, device: (conds, poses, trans, None))
    args = (N, H, W, torch.arange(N, device=DEV), ps.RATIO, cam, t("in/fl_masks"), t("in/gt_fl_pts"), DEV)
    return me, args, dict(poses=poses, trans=trans, conds=conds, deformer=deformer, curve=curve, sdf=sdf)


@pytest.mark.parametrize("cls,weights", [("base", (10., 1.)), ("large", (0., 0.))],
                         ids=["OptimGarmentNetwork", "LargePose"])
@pytest.mark.parametrize("N", [1, 3])
def test_drop_in_reproduces_the_reference_project_2d_loss(cls, weights, N):
    import project_2d_scene as ps
    d = _fixture(N)
    me, args, st = _fixture_scene(d)
    got = utils.make_project_2d_loss(*weights)(me, *args)
    f = f"{cls}/f64/"
    keys = sorted(k[len(f + "info/"):] for k in d if k.startswith(f + "info/"))
    assert set(me.info) == {"fl_loss"} and sorted(me.info["fl_loss"]) == keys and len(keys) == 8
    for k in keys:
        v, ref = me.info["fl_loss"][k], float(d[f + "info/" + k])
        assert isinstance(v, torch.Tensor) and v.dim() == 0 and not v.requires_grad
        # the SDF terms go through the garment SDF network on the tensor cores, whose own error (about 1e-6 of the
        # output's scale, as smoke() reports it) is 2.4e-5 of the pants' mean |f + r|: 5e-5 there, 1e-5 elsewhere
        tol = 5e-5 if k.endswith("_loss_sdf") else 1e-5
        assert abs(v.item() - ref) <= tol * abs(ref), (k, v.item(), ref)
    assert len(got) == 4
    for g, garment in enumerate(ps.GARMENTS):
        names = ps.FL_EXTRACT[garment]
        assert len(got[0][g]) == len(got[1][g]) == len(got[2][g]) == len(names)
        for c, name in enumerate(names):
            col = ps.FL_NAMES.index(name)
            scr, vis, lab = got[0][g][c], got[1][g][c], got[2][g][c]
            assert scr.shape == (N, 200, 3) and scr.dtype == torch.float32 and not scr.requires_grad
            _close = _rel(scr.cpu(), d[f"{f}screen_{g}_{c}"])
            assert _close <= 1e-5, (garment, name, _close)
            assert vis.shape == (N, 200, 3) and vis.dtype == torch.bool
            assert np.array_equal(vis.cpu().numpy(), d[f"{f}visible_{g}_{c}"]), (garment, name)
            assert lab.shape == (N, 200, 3) and lab.dtype == torch.bool
            assert torch.equal(lab, args[6][:, None, col:col + 1].expand(N, 200, 3))
        assert np.array_equal(got[3][g].cpu().numpy(), d[f"{f}gt_{g}"])
    # gradients, each to its own largest entry; an all-zero reference (the Large-Pose weights) must be matched by zeros
    pairs = [("scale", st["curve"].scale.grad), ("nx_scale", st["curve"].nx_scale.grad), ("poses", st["poses"].grad),
             ("trans", st["trans"].grad), ("cond1", st["conds"][1].grad), ("cond2", st["conds"][2].grad)]
    pairs += [(f"translator.{n}", p.grad) for n, p in st["deformer"].defs[0].named_parameters()]
    pairs += [(f"sdf.{n}", p.grad) for n, p in st["sdf"].named_parameters()]
    checked, errs = 0, {}
    for name, grad in pairs:
        key = f"{f}grad/{name}"
        if key not in d:
            assert grad is None or not grad.any(), name
            continue
        ref = d[key]
        got_g = grad.detach().reshape(-1)
        got_g = got_g if got_g.numel() == ref.size else got_g[::257]
        got_g = got_g.double().cpu().numpy().reshape(ref.shape)
        errs[name] = 0. if not ref.any() and not got_g.any() else _rel(got_g, ref)
        checked += 1
    print("gradient errors", {k: float(v) for k, v in errs.items()})
    assert checked >= 20
    # the curve parameters (this change's kernels) to 2.5e-5.  The network, pose and condition gradients sum chamfer
    # residuals 2 (x - y) of about a pixel whose float32 position error is 1e-4 px: the reference's own float32 run
    # misses float64 on them by up to 8.7e-5 (translator biases, N = 3), and this package's networks add their
    # tensor-core error, so they are held to 5e-4
    bad = {k: v for k, v in errs.items() if v > (2.5e-5 if k in ("scale", "nx_scale") else 5e-4)}
    assert not bad, bad
    for name in ("scale", "nx_scale"):
        g = np.abs(d[f"{f}grad/{name}"])
        sel = g > 1e-3 * g.max() if g.max() > 0 else np.ones_like(g, dtype=bool)
        after = getattr(st["curve"], name).detach().cpu().numpy()
        assert np.abs(after[sel] - d[f"{f}{name}_after"][sel]).max() <= 1e-6, name
    tr = me.deformer.defs[0].offset
    for n in ps.FL_NAMES:
        assert tr[n].shape == (N, 200, 3)
        assert _rel(tr[n].detach().cpu(), d[f"{f}offset/{n}"]) <= 1e-5, n


def test_drop_in_makes_no_host_synchronisation():
    import project_2d_scene as ps
    me, args, _ = ps.scene(DEV, N=3)
    fn = utils.make_project_2d_loss()
    fn(me, *args)                                # warm: library load, workspaces, the deformer's host caches
    _, total, (adamw,), where = _count(lambda: fn(me, *args), counted=[(me.fl_optimizer, "step")])
    print("host synchronisations: drop-in", total - adamw, "AdamW.step", adamw)
    assert total - adamw == 0, where
    ref_self, ref_args, _ = ps.scene(DEV, N=3)
    ps.reference_flow(ref_self, *ref_args)
    _, ref_total, _, _ = _count(lambda: ps.reference_flow(ref_self, *ref_args))
    print("host synchronisations: reference flow", ref_total)
    assert ref_total >= 12


def test_drop_in_refusals():
    import project_2d_scene as ps
    me, args, _ = ps.scene(DEV, N=1)
    fn = utils.make_project_2d_loss()
    me.conf.d["fl_visible_method"] = "surface"
    with pytest.raises(NotImplementedError):
        fn(me, *args)
    me.conf.d["fl_visible_method"] = "zbuff"
    bad = list(args)
    bad[6] = args[6].cpu()
    with pytest.raises(RuntimeError):
        fn(me, *bad)

