"""GPU tests of the skinning's training path: the kinematic-chain VJP kernel (recmv_bone_matrices_backward), the fused
skinning backward (recmv_lbs_backward) and their autograd wiring (ops.BoneMatricesFunction, ops.LbsTrainFunction,
LBSkinner / CompositeDeformer), against float64 autograd of the oracle, the reference's own gradients (lbs_grad.npz)
and the torch composite (train_fused=False).  Each bound sits above the error measured on an H100; the composite's own
fp32 distance from float64 is printed beside the kernel's."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F
from torch.utils._python_dispatch import TorchDispatchMode

from conftest import load_golden
from oracle import oracle_torch as ot
from recmv_b200 import _lib, ops, synth
from recmv_b200.model import CompositeDeformer, LBSkinner, MLPTranslator
from recmv_b200.utils import compute_cardinal_rays, compute_deformed_normals

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RATIO = {"deformerRatio": 0.6}
# skinning backward against float64, relative to the largest reference entry.  H100: at most 2.4e-6 (dps with one
# frame; the composite in fp32 7.8e-7 there, and up to 1.3e-5 on dA at V = 120 000 where the kernel measured 3.4e-7)
SKIN_BOUND = 6e-6


def _skinner(init=True):
    Js, parents, ip = synth.skeleton()
    ws = synth.skinning_voxel((17, 33, 21), seed=7)
    sk = LBSkinner(ws, [-1.1] * 3, [1.1] * 3, Js, parents, init_pose=ip,
                   bbox_extend=torch.tensor(synth.BBOX_EXTEND), bbox_center=torch.tensor(synth.BBOX_CENTER)).to(DEV)
    if not init:
        sk.init_pose = None
    return sk


def _rel(a, b):
    a = torch.as_tensor(a).detach().double().cpu()
    b = torch.as_tensor(b).detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


# ------------------------------------------------------------------ kinematic-chain VJP
def _chain_t(poses, sk):
    """(G, A) by autograd-able oracle ops in the dtype of `poses`; A follows LBSkinner (init pose or G - [0 | G J])."""
    dt = poses.dtype
    Js = sk.Js.to(dt).cpu()
    G = ot.bone_matrices(poses, Js, sk.parents, torch.eye(4, dtype=dt).expand(24, 4, 4))
    if sk.init_pose is not None:
        return G, G @ sk.init_pose.to(dt).cpu().view(1, 24, 4, 4)
    Jw0 = torch.cat([Js.view(1, 24, 3, 1).expand(G.shape[0], 24, 3, 1), torch.zeros(G.shape[0], 24, 1, 1, dtype=dt)], 2)
    return G, G - F.pad(G @ Jw0, [3, 0])


def _poses(n, seed):
    poses, _ = synth.poses_trans(n, seed=seed)
    axis = torch.tensor([0.48, -0.6, 0.64])
    poses[0, 0] = 0.0                                   # the |theta + 1e-8| branch
    poses[0, 1] = 1e-6 * axis                           # tiny angle
    poses[0, 2] = (math.pi - 1e-3) * axis               # near pi
    poses[0, 3] = math.pi * axis
    poses[0, 4] = (2 * math.pi + 0.4) * axis            # beyond 2 pi
    poses[0, 5] = -(2 * math.pi + 1.3) * axis.flip(0)
    return poses


@pytest.mark.parametrize("init", [True, False])
@pytest.mark.parametrize("which", ["dA", "dG", "both"])
@pytest.mark.parametrize("F_", [1, 5, 90, 1000])
def test_chain_vjp_matches_float64(F_, which, init):
    sk = _skinner(init)
    poses = _poses(F_, seed=F_)
    gen = synth.generator(77 + F_)
    dG = torch.randn((F_, 24, 4, 4), generator=gen) if which != "dA" else None
    dA = torch.randn((F_, 24, 4, 4), generator=gen) if which != "dG" else None
    pd = poses.to(DEV)
    G, A = ops.bone_matrices(pd, sk.Js, sk._parents_dev(pd.device), sk.init_pose)
    d = ops.bone_matrices_backward(pd, sk.Js, sk._parents_dev(pd.device), sk.init_pose, G,
                                   None if dG is None else dG.to(DEV), None if dA is None else dA.to(DEV))
    grads = []
    for dt in (torch.float64, torch.float32):      # fp32: the torch chain's own distance from float64
        p = poses.to(dt).requires_grad_(True)
        Gt, At = _chain_t(p, sk)
        outs = [t for t, c in ((Gt, dG), (At, dA)) if c is not None]
        grads.append(torch.autograd.grad(outs, p, [c.to(dt) for c in (dG, dA) if c is not None])[0])
    ref, tch = grads
    err = _rel(d, ref)
    print(f"chain VJP F={F_} {which} init={init}: kernel {err:.2e}  torch chain fp32 {_rel(tch, ref):.2e}")
    assert torch.isfinite(d).all()
    assert err < 2e-6          # H100: at most 5.2e-7 (F = 1000); the torch chain in fp32 5.4e-7


def test_chain_forward_and_vjp_match_torch_chain():
    """The kernel chain against the torch chain (train_fused=False): forward A and posedSkeleton, and the pose gradient."""
    for init in (True, False):
        sk = _skinner(init)
        poses = _poses(7, seed=3).to(DEV)
        gen = synth.generator(5)
        cA, cJ = torch.randn((7, 24, 4, 4), generator=gen).to(DEV), torch.randn((7, 24, 3), generator=gen).to(DEV)
        res = {}
        for fused in (True, False):
            sk.train_fused = fused
            p = poses.clone().requires_grad_(True)
            A = sk.bone_matrices(p)
            J = sk.posedSkeleton([p, torch.zeros((7, 3), device=DEV)])
            (gA,) = torch.autograd.grad(A, p, cA)
            (gJ,) = torch.autograd.grad(J, p, cJ)
            res[fused] = (A.detach(), J.detach(), gA, gJ)
        f, t = res[True], res[False]
        assert (f[0] - t[0]).abs().max() < 2e-6 and (f[1] - t[1]).abs().max() < 2e-6
        assert _rel(f[2], t[2]) < 4e-6 and _rel(f[3], t[3]) < 4e-6


# ------------------------------------------------------------------ skinning backward
def _scene(P_extra_faces=64, seed=9):
    """The lbs.npz scene (about 8 % of its points outside the voxel) plus points exactly on the voxel's box faces."""
    g = load_golden("lbs.npz")
    ps = torch.from_numpy(g["ps"])
    gen = synth.generator(seed)
    c, e = torch.tensor(synth.BBOX_CENTER), float(torch.tensor(synth.BBOX_EXTEND))
    face = (torch.rand((P_extra_faces, 3), generator=gen) - 0.5) * e
    ax = torch.arange(P_extra_faces) % 3
    sign = torch.where(torch.arange(P_extra_faces) % 2 == 0, 1.0, -1.0)
    face[torch.arange(P_extra_faces), ax] = c[ax] + sign * (e / 2)
    ps = torch.cat([ps, face])
    bi = torch.cat([torch.from_numpy(g["batch_inds"]), torch.randint(0, 3, (P_extra_faces,), generator=gen)])
    return ps, bi, torch.from_numpy(g["A"]), torch.from_numpy(g["trans"])


def _oracle_grads(ps, tps, A, trans, bi, cot):
    """float64 autograd of ot.lbs_forward: (dps, dtps or None, dA, dtrans); frames clamped like the kernels."""
    ws = synth.skinning_voxel((17, 33, 21), seed=7).double()
    center = torch.tensor(synth.BBOX_CENTER).double()
    extend = float(torch.tensor(synth.BBOX_EXTEND))
    p = ps.double().requires_grad_(True)
    t = tps.double().requires_grad_(True) if tps is not None else None
    a = A.double().requires_grad_(True)
    tr = trans.double().requires_grad_(True)
    out = ot.lbs_forward(p, a, tr, ws, center, extend, bi.clamp(0, A.shape[0] - 1), t)
    ins = [x for x in (p, t, a, tr) if x is not None]
    gr = list(torch.autograd.grad(out, ins, cot.double()))
    return gr[0], (gr[1] if t is not None else None), gr[-2], gr[-1]


def _composite_grads(sk, ps, tps, A, trans, bi, cot):
    """The torch composite in fp32 (FrozenVoxelSampleFunction + blend) on the device."""
    p = ps.to(DEV).requires_grad_(True)
    t = tps.to(DEV).requires_grad_(True) if tps is not None else None
    a = A.to(DEV).requires_grad_(True)
    tr = trans.to(DEV).requires_grad_(True)
    out = sk._composite(p, p if t is None else t, a, tr, bi.clamp(0, A.shape[0] - 1).to(DEV))
    ins = [x for x in (p, t, a, tr) if x is not None]
    gr = list(torch.autograd.grad(out, ins, cot.to(DEV)))
    return gr[0], (gr[1] if t is not None else None), gr[-2], gr[-1]


def _kernel_grads(sk, ps, tps, A, bi, cot, ppf=0):
    center, extend = sk.bbox_host()
    return ops.lbs_backward(ps.to(DEV), A.to(DEV), cot.to(DEV), sk.ws_channels_last(), center, extend,
                            None if bi is None else bi.to(DEV), ppf, None if tps is None else tps.to(DEV))


def _check(name, kern, ref, comp, bound):
    for k, r, c, lab in zip(kern, ref, comp, ("dps", "dtps", "dA", "dtrans")):
        if r is None:
            assert k is None
            continue
        ek, ec = _rel(k.reshape(r.shape), r), _rel(c.reshape(r.shape), r)
        print(f"{name} {lab}: kernel {ek:.2e}  composite fp32 {ec:.2e}")
        assert ek < bound, (name, lab, ek)


@pytest.mark.parametrize("case", ["sorted-list", "unsorted-list", "out-of-range", "tps-ps"])
def test_lbs_backward_matches_float64(case):
    sk = _skinner()
    ps, bi, A, trans = _scene()
    gen = synth.generator(31)
    tps = None
    if case == "sorted-list":
        bi = bi.sort().values
    elif case == "out-of-range":
        bi = bi.clone()
        bi[::7] = -2
        bi[3::11] = 5
    elif case == "tps-ps":
        tps = ps + 0.05 * torch.randn(ps.shape, generator=gen)
    cot = torch.randn(ps.shape, generator=gen)
    kern = _kernel_grads(sk, ps, tps, A, bi, cot)
    ref = _oracle_grads(ps, tps, A, trans, bi, cot)
    comp = _composite_grads(sk, ps, tps, A, trans, bi, cot)
    _check(case, kern, ref, comp, SKIN_BOUND)


def test_lbs_backward_expanded_template_multi_wave():
    """[3, V, 3] garment vertices expanded from one template (V = 120 000: 1407 chunks, more than one wave)."""
    sk = _skinner()
    V = 120000
    gen = synth.generator(12)
    tmpl = (torch.rand((1, V, 3), generator=gen) - 0.5) * 2.4
    poses, trans = synth.poses_trans(3, seed=4)
    A = ot.bone_matrices(poses, sk.Js.cpu(), sk.parents, sk.init_pose.cpu())
    cot = torch.randn((3 * V, 3), generator=gen)
    ps = tmpl.expand(3, V, 3).reshape(-1, 3)
    bi = torch.arange(3).repeat_interleave(V)
    kern = _kernel_grads(sk, ps, None, A, None, cot, ppf=V)
    ref = _oracle_grads(ps, None, A, trans, bi, cot)
    comp = _composite_grads(sk, ps, None, A, trans, bi, cot)
    _check("expanded V=120000", kern, ref, comp, SKIN_BOUND)
    # the same through LBSkinner, with the gradient reaching the unexpanded template
    t = tmpl.to(DEV).requires_grad_(True)
    pd, td = poses.to(DEV).requires_grad_(True), trans.to(DEV).requires_grad_(True)
    out = sk(t.expand(3, V, 3), [pd, td], None)
    assert sk.last_path == "fused-train"
    out.backward(cot.view(3, V, 3).to(DEV))
    assert sk.last_backward == "fused" and t.grad.shape == (1, V, 3)
    assert _rel(t.grad, ref[0].view(3, V, 3).sum(0, keepdim=True)) < SKIN_BOUND


def _guarded(n, *shape):
    return torch.full((n + 2 * 512,) + shape, float("nan"), device=DEV)


def _raw(sk, ps, tps, A, bi, g, dps, dtps, dA, dtrans, work, ppf=0):
    center, extend = sk.bbox_host()
    vox = ops.make_voxel(sk.ws_channels_last(), center, extend)
    P = ps.shape[0]

    def ptr(t, rows=512):
        return None if t is None else ctypes.c_void_p(t[rows:].data_ptr())
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(_lib.load().recmv_lbs_backward(
        ops._ptr(ps), ops._ptr(tps), ops._ptr(A), None, ops._ptr(bi), ppf, A.shape[0], ctypes.byref(vox), ops._ptr(g),
        ptr(dps), ptr(dtps), ptr(dA), ptr(dtrans), ops._ptr(work), P, st), "recmv_lbs_backward")


@pytest.mark.parametrize("tps_form", [False, True])
def test_lbs_backward_bounds_determinism_and_null_outputs(tps_form):
    sk = _skinner()
    ps, bi, A, _ = _scene()
    gen = synth.generator(41)
    P, F_ = ps.shape[0], A.shape[0]
    ps, bi, A = ps.to(DEV), bi.to(DEV), A.to(DEV)
    tps = (ps + 0.03 * torch.randn(ps.shape, generator=gen).to(DEV)).contiguous() if tps_form else None
    g = torch.randn(ps.shape, generator=gen).to(DEV)
    nbytes = ctypes.c_size_t(0)
    _lib.load().recmv_lbs_backward_workspace_bytes(P, F_, ctypes.byref(nbytes))
    work = torch.full((nbytes.value // 4 + 4,), float("nan"), device=DEV)   # stale contents must not matter

    def run(want=(True, True, True, True)):
        outs = [_guarded(P, 3), _guarded(P, 3), _guarded(F_, 24, 4, 4), _guarded(F_, 3)]
        outs = [o if w else None for o, w in zip(outs, want)]
        _raw(sk, ps, tps, A, bi, g, *outs, work)
        torch.cuda.synchronize()
        return outs
    full = run()
    for o, n, written in zip(full, (P, P, F_, F_), (True, tps_form, True, True)):
        assert torch.isnan(o[:512]).all() and torch.isnan(o[512 + n:]).all()     # guards untouched
        if written:
            assert torch.isfinite(o[512:512 + n]).all()
        else:
            assert torch.isnan(o[512:512 + n]).all()                            # dtps without tps: not written
    assert (full[2][512:512 + F_, :, 3] == 0).all()                               # row 3 of dA
    again = run()
    for a, b in zip(full, again):
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0))                  # bit-identical
    for k in range(4):                                                            # one output alone
        want = [i == k for i in range(4)]
        one = run(want)[k]
        assert torch.equal(one.nan_to_num(7.0), full[k].nan_to_num(7.0))
    ref = ops.lbs_backward(ps, A, g, sk.ws_channels_last(), *sk.bbox_host(), bi, 0, tps)
    for a, r, n in zip(full, ref, (P, P, F_, F_)):
        if r is not None:
            assert torch.equal(a[512:512 + n], r)


def test_lbs_backward_empty_and_single_frame():
    sk = _skinner()
    center, extend = sk.bbox_host()
    ws = sk.ws_channels_last()
    A = torch.randn((2, 24, 4, 4), device=DEV)
    e = torch.empty((0, 3), device=DEV)
    dps, dtps, dA, dtrans = ops.lbs_backward(e, A, e, ws, center, extend, torch.empty(0, dtype=torch.long, device=DEV))
    assert dps.shape == (0, 3) and dtps is None and (dA == 0).all() and (dtrans == 0).all()
    ps, bi, A3, trans = _scene()
    cot = torch.randn(ps.shape, generator=synth.generator(2))
    A1, tr1 = A3[1:2], trans[1:2]
    kern = _kernel_grads(sk, ps, None, A1, None, cot, ppf=0)
    ref = _oracle_grads(ps, None, A1, tr1, torch.zeros_like(bi), cot)
    comp = _composite_grads(sk, ps, None, A1, tr1, torch.zeros_like(bi), cot)
    _check("F=1", kern, ref, comp, SKIN_BOUND)


# ------------------------------------------------------------------ LBSkinner against the reference's own gradients
@pytest.mark.parametrize("form", ["list", "batch"])
def test_lbskinner_gradients_match_reference_golden(form):
    g = load_golden("lbs_grad.npz")
    s = load_golden("lbs.npz")
    sk = _skinner()
    ps = torch.from_numpy(s["ps"]).to(DEV).requires_grad_(True)
    poses = torch.from_numpy(s["poses"]).to(DEV).requires_grad_(True)
    trans = torch.from_numpy(s["trans"]).to(DEV).requires_grad_(True)
    if form == "list":
        out = sk(ps, [poses, trans], torch.from_numpy(s["batch_inds"]).to(DEV))
    else:
        out = sk(ps.view(3, 1000, 3), [poses, trans], None).reshape(-1, 3)
    assert sk.last_path == "fused-train"
    gr = torch.autograd.grad(out, (ps, poses, trans), torch.from_numpy(g["cot"]).to(DEV))
    assert sk.last_backward == "fused"
    for name, k in zip(("dps", "dposes", "dtrans"), gr):
        e64, e32 = _rel(k, g[f"{form}_f64_{name}"]), _rel(g[f"{form}_f32_{name}"], g[f"{form}_f64_{name}"])
        print(f"golden {form} {name}: kernel {e64:.2e}  reference fp32 {e32:.2e}")
        assert e64 < 4e-6      # H100: at most 1.1e-6 (dps); the reference's own fp32 run 1.1e-6
    p = torch.from_numpy(s["poses"]).to(DEV).requires_grad_(True)
    J = sk.posedSkeleton([p, trans.detach()])
    (gJ,) = torch.autograd.grad(J, p, torch.from_numpy(g["cot_J"]).to(DEV))
    assert _rel(gJ, g["skel_f64_dposes"]) < 2e-6


# ------------------------------------------------------------------ the deformer as the training step uses it
class _Count(TorchDispatchMode):
    def __init__(self):
        super().__init__()
        self.n = 0

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        self.n += 1
        return func(*args, **(kwargs or {}))


def _deformer(V=3000, seed=3):
    torch.manual_seed(seed)
    tr = MLPTranslator(128, 6)
    sk = _skinner()
    d = CompositeDeformer([tr, sk]).to(DEV)
    gen = synth.generator(seed)
    tmpl = ((torch.rand((1, V, 3), generator=gen) - 0.5) * 2.0).to(DEV)
    poses, trans = synth.poses_trans(3, seed=seed)
    conds = (torch.randn((3, 128), generator=gen) * 0.1).to(DEV)
    return d, tr, sk, tmpl, poses.to(DEV), trans.to(DEV), conds


def _step(d, tr, sk, tmpl, poses, trans, conds, fused):
    tr.train_fused = sk.train_fused = fused
    p, t, c = (x.clone().requires_grad_(True) for x in (poses, trans, conds))
    out = d(tmpl.expand(3, -1, 3), [c, [p, t]], None, ratio=RATIO, offset_type="garment")
    path = sk.last_path
    loss = (out * torch.linspace(-1, 1, out.numel(), device=DEV).view(out.shape)).sum()
    params = list(tr.parameters())
    gr = torch.autograd.grad(loss, [p, t, c] + params)
    return out.detach(), path, gr


def test_deformer_training_step_matches_composite_and_skips_torch_chain(monkeypatch):
    d, tr, sk, tmpl, poses, trans, conds = _deformer()
    o_f, path_f, g_f = _step(d, tr, sk, tmpl, poses, trans, conds, True)
    o_c, path_c, g_c = _step(d, tr, sk, tmpl, poses, trans, conds, False)
    assert path_f == "fused-train" and path_c == "autograd-composite"
    assert (o_f - o_c).abs().max() < 1e-4
    names = ["poses", "trans", "conds"] + [n for n, _ in tr.named_parameters()]
    for n, a, b in zip(names, g_f, g_c):
        e = _rel(a, b)
        print(f"deformer {n}: fused vs composite {e:.2e}")
        # poses / trans: the skinning alone (measured 8.6e-7); conds and the translator's parameters also carry the
        # translator's tensor-core GEMMs against cuBLAS (measured at most 5.5e-4)
        assert e < (5e-6 if n in ("poses", "trans") else 2e-3), (n, e)
    # float64: the skinning stage alone, fed the translated points of the fused step
    with torch.no_grad():
        x = tr(tmpl.expand(3, -1, 3), conds, None, ratio=RATIO, offset_type="x")
    V = tmpl.shape[1]
    g = torch.linspace(-1, 1, 3 * V * 3, device=DEV).view(-1, 3).cpu()
    p64 = poses.cpu().double().requires_grad_(True)
    t64 = trans.cpu().double().requires_grad_(True)
    A64 = ot.bone_matrices(p64, sk.Js.double().cpu(), sk.parents, sk.init_pose.double().cpu())
    o64 = ot.lbs_forward(x.reshape(-1, 3).cpu().double(), A64, t64, sk.ws.double().cpu(),
                         torch.tensor(synth.BBOX_CENTER).double(), float(torch.tensor(synth.BBOX_EXTEND)),
                         torch.arange(3).repeat_interleave(V))
    r_p, r_t = torch.autograd.grad(o64, (p64, t64), g.double())
    pk, tk = poses.clone().requires_grad_(True), trans.clone().requires_grad_(True)
    sk.train_fused = True
    ok = sk(x, [pk, tk], None)
    gp, gt = torch.autograd.grad(ok, (pk, tk), g.view(ok.shape).to(DEV))
    print(f"deformer skinning vs float64: poses {_rel(gp, r_p):.2e} trans {_rel(gt, r_t):.2e}")
    assert _rel(gp, r_p) < SKIN_BOUND and _rel(gt, r_t) < SKIN_BOUND
    # the fused path never builds the torch chain, and dispatches far fewer ops
    counts = {}
    for fused in (True, False):
        sk.train_fused = fused
        p = poses.clone().requires_grad_(True)
        c = _Count()
        with c:
            out = sk(x, [p, trans], None)
            out.sum().backward()
        counts[fused] = c.n
    print(f"aten ops of one LBSkinner forward + backward: fused {counts[True]}, composite {counts[False]}")
    assert counts[True] * 10 < counts[False]
    monkeypatch.setattr(sk, "_chain", lambda *a: (_ for _ in ()).throw(AssertionError("torch chain used")))
    sk.train_fused = True
    p = poses.clone().requires_grad_(True)
    sk(x, [p, trans], None).sum().backward()
    sk.posedSkeleton([p, trans]).sum().backward()


@pytest.mark.parametrize("which", ["cardinal_rays", "deformed_normals"])
def test_train_phase_jacobians_use_composite_create_graph(which):
    d, tr, sk, tmpl, poses, trans, conds = _deformer(V=500, seed=5)
    sdf = lambda x, ratio: (x * x).sum(-1, keepdim=True) - 0.3            # noqa: E731  (smooth, nonzero gradient)
    gen = synth.generator(6)
    P = 600
    ps0 = ((torch.rand((P, 3), generator=gen) - 0.5) * 1.6).to(DEV)
    bi = torch.randint(0, 3, (P,), generator=gen).to(DEV)
    rays = F.normalize(torch.randn((P, 3), generator=gen), dim=1).to(DEV)
    res = {}
    for fused in (True, False):
        tr.train_fused = sk.train_fused = fused
        ps = ps0.clone().requires_grad_(True)
        p, t, c = (x.clone().requires_grad_(True) for x in (poses, trans, conds))
        if which == "cardinal_rays":
            v, ds = compute_cardinal_rays(d, ps, rays, [c, [p, t]], bi, RATIO, "train", "x")
        else:
            v, ds = compute_deformed_normals(sdf, d, ps, [c, [p, t]], bi, RATIO, "train", "x")
        if fused:
            assert sk.last_path == "fused-train" and sk.last_backward == "autograd-composite (create_graph)"
        loss = (v * rays).sum() + (ds * rays).sum()
        gr = torch.autograd.grad(loss, [p, t, c, ps])
        if fused:
            assert sk.last_backward == "fused"
        res[fused] = (v.detach(), gr)
    assert (res[True][0] - res[False][0]).abs().max() < 1e-4
    for n, a, b in zip(("poses", "trans", "conds", "ps"), res[True][1], res[False][1]):
        e = _rel(a, b)
        print(f"{which} {n}: fused vs composite {e:.2e}")
        assert e < 5e-5, (n, e)   # H100: at most 8.3e-6 (conds)
