"""GPU tests of the skinning's second-order path: the VJP of the skinning backward's point gradients
(recmv_lbs_vjp_backward) and its autograd wiring (ops.LbsVjpFunction, LbsTrainFunction under create_graph with
LBSkinner.second_order_fused), against float64 autograd of the oracle applied twice, the reference's own second-order
gradients (lbs_grad2.npz) and the torch composite (second_order_fused=False).  Each bound sits above the error
measured on an H100; the composite's own fp32 distance from float64 is printed beside the kernel's."""
import ctypes

import pytest
import torch
import torch.nn.functional as F
from torch.utils._python_dispatch import TorchDispatchMode

from conftest import load_golden
from oracle import oracle_torch as ot
from recmv_b200 import _lib, ops, synth
from recmv_b200.model import CompositeDeformer, LBSkinner, MLPTranslator
from recmv_b200.utils import compute_cardinal_rays, compute_Jacobian, compute_deformed_normals

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RATIO = {"deformerRatio": 0.6}
LABEL = "fused (create_graph, input gradient)"
# the second-order skinning against float64, relative to the largest reference entry.  H100: at most 2.3e-5 (dtps of
# P = 255; the fp32 composite at most 4.9e-6 on these cases), d g and dA at most 2.6e-6; the reference golden 9.9e-6
# (dps; the reference's own fp32 run 7.4e-6)
VJP_BOUND = 6e-5


def _skinner():
    Js, parents, ip = synth.skeleton()
    ws = synth.skinning_voxel((17, 33, 21), seed=7)
    return LBSkinner(ws, [-1.1] * 3, [1.1] * 3, Js, parents, init_pose=ip,
                     bbox_extend=torch.tensor(synth.BBOX_EXTEND), bbox_center=torch.tensor(synth.BBOX_CENTER)).to(DEV)


def _rel(a, b):
    a = torch.as_tensor(a).detach().double().cpu()
    b = torch.as_tensor(b).detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _scene(seed=9):
    """The lbs.npz scene (about 8 % of its points outside the voxel) plus points exactly on the voxel's box faces."""
    g = load_golden("lbs.npz")
    ps = torch.from_numpy(g["ps"])
    gen = synth.generator(seed)
    c, e = torch.tensor(synth.BBOX_CENTER), float(torch.tensor(synth.BBOX_EXTEND))
    n = 64
    face = (torch.rand((n, 3), generator=gen) - 0.5) * e
    ax = torch.arange(n) % 3
    sign = torch.where(torch.arange(n) % 2 == 0, 1.0, -1.0)
    face[torch.arange(n), ax] = c[ax] + sign * (e / 2)
    ps = torch.cat([ps, face])
    bi = torch.cat([torch.from_numpy(g["batch_inds"]), torch.randint(0, 3, (n,), generator=gen)])
    return ps, bi, torch.from_numpy(g["A"])


def _beyond_faces(P, seed):
    """Points beyond every box face: each point leaves the box through one, two or three axes, on either side."""
    gen = synth.generator(seed)
    e = float(torch.tensor(synth.BBOX_EXTEND))
    ps = (torch.rand((P, 3), generator=gen) - 0.5) * 0.9 * e
    for k in range(P):
        axes = [k % 3] if k % 4 else [0, 1, 2][: 1 + (k // 4) % 3]
        for a in axes:
            side = 1.0 if (k // 3) % 2 == 0 else -1.0
            ps[k, a] = side * (e / 2 + 0.02 + 0.3 * float(torch.rand((1,), generator=gen)))
    return ps


def _oracle(ps, tps, A, bi, g, u, v):
    """float64 autograd twice of ot.lbs_forward: (d g, d ps, d tps or None, d A) of <V(ps, tps, A, g), (u, v)>."""
    ws = synth.skinning_voxel((17, 33, 21), seed=7).double()
    center = torch.tensor(synth.BBOX_CENTER).double()
    extend = float(torch.tensor(synth.BBOX_EXTEND))
    F_ = A.shape[0]
    p = ps.double().requires_grad_(True)
    t = tps.double().requires_grad_(True) if tps is not None else None
    a = A.double().requires_grad_(True)
    gg = g.double().requires_grad_(True)
    out = ot.lbs_forward(p, a, torch.zeros((F_, 3), dtype=torch.float64), ws, center, extend, bi.clamp(0, F_ - 1), t)
    firsts = torch.autograd.grad(out, [p] + ([t] if t is not None else []), gg, create_graph=True)
    phi = (firsts[0] * u.double()).sum()
    if t is not None:
        phi = phi + (firsts[1] * v.double()).sum()
    ins = [gg, p] + ([t] if t is not None else []) + [a]
    d = [x if x is not None else torch.zeros_like(i) for x, i in zip(torch.autograd.grad(phi, ins, allow_unused=True), ins)]
    return d[0], d[1], (d[2] if t is not None else None), d[-1]


def _composite(sk, ps, tps, A, bi, g, u, v):
    """The same by the fp32 torch composite (the CUDA sampler's bwd / bwd2 plus the blend) on the device."""
    F_ = A.shape[0]
    p = ps.to(DEV).requires_grad_(True)
    t = tps.to(DEV).requires_grad_(True) if tps is not None else None
    a = A.to(DEV).requires_grad_(True)
    gg = g.to(DEV).requires_grad_(True)
    out = sk._composite(p, p if t is None else t, a, torch.zeros((F_, 3), device=DEV), bi.clamp(0, F_ - 1).to(DEV))
    firsts = torch.autograd.grad(out, [p] + ([t] if t is not None else []), gg, create_graph=True)
    phi = (firsts[0] * u.to(DEV)).sum()
    if t is not None:
        phi = phi + (firsts[1] * v.to(DEV)).sum()
    ins = [gg, p] + ([t] if t is not None else []) + [a]
    d = [x if x is not None else torch.zeros_like(i) for x, i in zip(torch.autograd.grad(phi, ins, allow_unused=True), ins)]
    return d[0], d[1], (d[2] if t is not None else None), d[-1]


def _kernel(sk, ps, tps, A, bi, g, u, v, ppf=0):
    center, extend = sk.bbox_host()
    return ops.lbs_vjp_backward(ps.to(DEV), A.to(DEV), g.to(DEV), sk.ws_channels_last(), center, extend,
                                None if bi is None else bi.to(DEV), ppf, None if tps is None else tps.to(DEV),
                                u.to(DEV), None if v is None else v.to(DEV))


def _check(name, kern, ref, comp, bound=VJP_BOUND):
    for k, r, c, lab in zip(kern, ref, comp, ("d_grad_out", "dps", "dtps", "dA")):
        if r is None:
            assert k is None
            continue
        assert torch.isfinite(k).all(), (name, lab)
        ek = _rel(k.reshape(r.shape), r)
        ec = _rel(c.reshape(r.shape), r) if c is not None else float("nan")
        print(f"{name} {lab}: kernel {ek:.2e}  composite fp32 {ec:.2e}")
        assert ek < bound, (name, lab, ek)


@pytest.mark.parametrize("case", ["sorted-list", "unsorted-list", "out-of-range", "tps-ps", "batch-ppf",
                                  "beyond-faces", "beyond-faces-tps", "F1"])
def test_lbs_vjp_backward_matches_float64(case):
    sk = _skinner()
    ps, bi, A = _scene()
    gen = synth.generator(53)
    tps, ppf = None, 0
    if case == "sorted-list":
        bi = bi.sort().values
    elif case == "out-of-range":
        bi = bi.clone()
        bi[::7] = -2
        bi[3::11] = 5
    elif case == "tps-ps":
        tps = ps + 0.05 * torch.randn(ps.shape, generator=gen)
    elif case == "batch-ppf":
        ps = ps[:3 * 1000]
        bi, ppf = torch.arange(3).repeat_interleave(1000), 1000
    elif case.startswith("beyond-faces"):
        ps = _beyond_faces(900, seed=3)
        bi = torch.randint(0, 3, (900,), generator=gen)
        if case.endswith("tps"):
            tps, ps = ps, (torch.rand((900, 3), generator=gen) - 0.5) * 2.0
    elif case == "F1":
        A, bi = A[1:2], torch.zeros_like(bi)
    g = torch.randn(ps.shape, generator=gen)
    u = torch.randn(ps.shape, generator=gen)
    v = torch.randn(ps.shape, generator=gen) if tps is not None else None
    kern = _kernel(sk, ps, tps, A, None if ppf else bi, g, u, v, ppf)
    ref = _oracle(ps, tps, A, bi, g, u, v)
    comp = _composite(sk, ps, tps, A, bi, g, u, v)
    _check(case, kern, ref, comp)
    if case.startswith("beyond-faces"):
        # every sampling point is clamped on at least one axis; the all-clamped ones have no weight derivative at all
        s = ps if tps is None else tps
        out = (s.abs() > float(torch.tensor(synth.BBOX_EXTEND)) / 2).all(1)
        assert out.any()
        if tps is not None:
            assert (kern[2].cpu()[out] == 0).all()


@pytest.mark.parametrize("P", [0, 1, 255, 257, 120000])
@pytest.mark.parametrize("tps_form", [False, True])
def test_lbs_vjp_backward_sizes(P, tps_form):
    """P = 0, a single point, one partial chunk, a chunk and a point, and 3 x 40 000 (many waves)."""
    sk = _skinner()
    gen = synth.generator(100 + P)
    ps = (torch.rand((P, 3), generator=gen) - 0.5) * 2.4
    tps = (ps + 0.05 * torch.randn((P, 3), generator=gen)) if tps_form else None
    A = ot.bone_matrices(synth.poses_trans(3, seed=4)[0], sk.Js.cpu(), sk.parents, sk.init_pose.cpu())
    bi = torch.randint(0, 3, (P,), generator=gen)
    g, u = torch.randn((P, 3), generator=gen), torch.randn((P, 3), generator=gen)
    v = torch.randn((P, 3), generator=gen) if tps_form else None
    kern = _kernel(sk, ps, tps, A, bi, g, u, v)
    if P == 0:
        assert kern[0].shape == (0, 3) and (kern[3] == 0).all()
        return
    ref = _oracle(ps, tps, A, bi, g, u, v)
    _check(f"P={P} tps={tps_form}", kern, ref, [None] * 4)


# ------------------------------------------------------------------ output contract of the raw entry
def _guarded(n, *shape):
    return torch.full((n + 2 * 512,) + shape, float("nan"), device=DEV)


@pytest.mark.parametrize("tps_form", [False, True])
def test_lbs_vjp_backward_bounds_nulls_workspace_and_determinism(tps_form):
    sk = _skinner()
    ps, bi, A = _scene()
    gen = synth.generator(41)
    P, F_ = ps.shape[0], A.shape[0]
    ps, bi, A = ps.to(DEV), bi.to(DEV), A.to(DEV)
    tps = (ps + 0.03 * torch.randn(ps.shape, generator=gen).to(DEV)).contiguous() if tps_form else None
    g, u = torch.randn(ps.shape, generator=gen).to(DEV), torch.randn(ps.shape, generator=gen).to(DEV)
    v = torch.randn(ps.shape, generator=gen).to(DEV) if tps_form else None
    center, extend = sk.bbox_host()
    vox = ops.make_voxel(sk.ws_channels_last(), center, extend)
    nbytes = ctypes.c_size_t(0)
    _lib.load().recmv_lbs_backward_workspace_bytes(P, F_, ctypes.byref(nbytes))

    def run(want=(True, True, True, True), work_fill=0.0):
        work = torch.full((nbytes.value // 4 + 4,), work_fill, device=DEV)
        outs = [_guarded(P, 3), _guarded(P, 3), _guarded(P, 3) if tps_form else None, _guarded(F_, 24, 4, 4)]
        outs = [o if w else None for o, w in zip(outs, want)]

        def ptr(t):
            return None if t is None else ctypes.c_void_p(t[512:].data_ptr())
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(_lib.load().recmv_lbs_vjp_backward(
            ops._ptr(ps), ops._ptr(tps), ops._ptr(A), ops._ptr(bi), 0, F_, ctypes.byref(vox), ops._ptr(g), ops._ptr(u),
            ops._ptr(v), *[ptr(o) for o in outs], ops._ptr(work), P, st), "recmv_lbs_vjp_backward")
        torch.cuda.synchronize()
        return outs
    full = run()
    for o, n in zip(full, (P, P, P, F_)):
        if o is None:
            continue
        assert torch.isnan(o[:512]).all() and torch.isnan(o[512 + n:]).all()     # guards untouched
        assert torch.isfinite(o[512:512 + n]).all()
    assert (full[3][512:512 + F_, :, 3] == 0).all()                               # row 3 of dA
    for a, b in zip(full, run(work_fill=float("nan"))):                           # stale workspace; a second run
        if a is not None:
            assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0))
    for k in range(4):                                                            # one output alone
        if full[k] is None:
            continue
        one = run([i == k for i in range(4)])[k]
        assert torch.equal(one.nan_to_num(7.0), full[k].nan_to_num(7.0))
    for k in range(4):                                                            # one output dropped
        if full[k] is None:
            continue
        rest = run([i != k for i in range(4)])
        for i in range(4):
            if i != k and full[i] is not None:
                assert torch.equal(rest[i].nan_to_num(7.0), full[i].nan_to_num(7.0))
    ref = ops.lbs_vjp_backward(ps, A, g, sk.ws_channels_last(), center, extend, bi, 0, tps, u, v)
    for a, r, n in zip(full, ref, (P, P, P, F_)):
        if r is not None:
            assert torch.equal(a[512:512 + n], r)


# ------------------------------------------------------------------ the reference's own second-order gradients
@pytest.mark.parametrize("form", ["list", "batch"])
def test_lbskinner_second_order_matches_reference_golden(form):
    g = load_golden("lbs_grad2.npz")
    s = load_golden("lbs.npz")
    sk = _skinner()
    sk.second_order_fused = True
    ps = torch.from_numpy(s["ps"]).to(DEV).requires_grad_(True)
    poses = torch.from_numpy(s["poses"]).to(DEV).requires_grad_(True)
    trans = torch.from_numpy(s["trans"]).to(DEV).requires_grad_(True)
    if form == "list":
        D = sk(ps, [poses, trans], torch.from_numpy(s["batch_inds"]).to(DEV))
    else:
        D = sk(ps.view(3, 1000, 3), [poses, trans], None).reshape(-1, 3)
    assert sk.last_path == "fused-train"
    J = compute_Jacobian(ps, D, True, True)
    assert sk.last_backward == LABEL
    loss = (J * torch.from_numpy(g["cot_J"]).to(DEV)).sum() + (D * torch.from_numpy(g["cot_D"]).to(DEV)).sum()
    gr = torch.autograd.grad(loss, (ps, poses, trans))
    for name, k in zip(("dps", "dposes", "dtrans"), gr):
        e64, e32 = _rel(k, g[f"{form}_f64_{name}"]), _rel(g[f"{form}_f32_{name}"], g[f"{form}_f64_{name}"])
        print(f"golden2 {form} {name}: kernel {e64:.2e}  reference fp32 {e32:.2e}")
        assert e64 < VJP_BOUND


# ------------------------------------------------------------------ the deformer as the training step uses it
class _Count(TorchDispatchMode):
    def __init__(self):
        super().__init__()
        self.n = 0

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        self.n += 1
        return func(*args, **(kwargs or {}))


def _deformer(V=500, seed=5):
    torch.manual_seed(seed)
    tr = MLPTranslator(128, 6)
    sk = _skinner()
    d = CompositeDeformer([tr, sk]).to(DEV)
    gen = synth.generator(seed)
    poses, trans = synth.poses_trans(3, seed=seed)
    conds = (torch.randn((3, 128), generator=gen) * 0.1).to(DEV)
    return d, tr, sk, poses.to(DEV), trans.to(DEV), conds


def _train_phase(d, tr, sk, poses, trans, conds, which, fused, P=600):
    """One train-phase block: the Jacobian call site, then the loss's backward.  Returns (value, gradients, labels)."""
    sk.second_order_fused = fused
    sdf = lambda x, ratio: (x * x).sum(-1, keepdim=True) - 0.3            # noqa: E731  (smooth, nonzero gradient)
    gen = synth.generator(6)
    ps = ((torch.rand((P, 3), generator=gen) - 0.5) * 1.6).to(DEV).requires_grad_(True)
    bi = torch.randint(0, 3, (P,), generator=gen).to(DEV)
    rays = F.normalize(torch.randn((P, 3), generator=gen), dim=1).to(DEV)
    p, t, c = (x.clone().requires_grad_(True) for x in (poses, trans, conds))
    if which == "cardinal_rays":
        v, ds = compute_cardinal_rays(d, ps, rays, [c, [p, t]], bi, RATIO, "train", "x")
        label = sk.last_backward
        loss = (v * rays).sum() + (ds * rays).sum()
    elif which == "deformed_normals":
        v, ds = compute_deformed_normals(sdf, d, ps, [c, [p, t]], bi, RATIO, "train", "x")
        label = sk.last_backward
        loss = (v * rays).sum() + (ds * rays).sum()
    else:   # the normal loss: J = compute_Jacobian(ps, ds, True, True), then J^T n
        ds = d(ps, [c, [p, t]], bi, ratio=RATIO, offset_type="x")
        J = compute_Jacobian(ps, ds, True, True)
        label = sk.last_backward
        v = (J.transpose(1, 2) @ rays.unsqueeze(-1)).squeeze(-1)
        loss = (v * v).sum() + (ds * rays).sum()
    gr = torch.autograd.grad(loss, [p, t, c, ps] + list(tr.parameters()))
    return v.detach(), gr, label


@pytest.mark.parametrize("which", ["cardinal_rays", "deformed_normals", "normal_loss"])
def test_train_phase_jacobians_fused_match_composite(which, monkeypatch):
    d, tr, sk, poses, trans, conds = _deformer()
    v_c, g_c, lab_c = _train_phase(d, tr, sk, poses, trans, conds, which, False)
    assert lab_c == "autograd-composite (create_graph)"
    with monkeypatch.context() as m:
        m.setattr(sk, "_composite", lambda *a: (_ for _ in ()).throw(AssertionError("composite used")))
        v_f, g_f, lab_f = _train_phase(d, tr, sk, poses, trans, conds, which, True)
        _, g_f2, _ = _train_phase(d, tr, sk, poses, trans, conds, which, True)
    assert lab_f == LABEL
    assert (v_f - v_c).abs().max() < 1e-4
    names = ["poses", "trans", "conds", "ps"] + [n for n, _ in tr.named_parameters()]
    for n, a, b in zip(names, g_f, g_c):
        e = _rel(a, b)
        print(f"{which} {n}: fused vs composite {e:.2e}")
        assert e < 5e-5, (n, e)
    for k in (0, 3):                                                  # poses and ps: bit-identical across runs
        assert torch.equal(g_f[k], g_f2[k])
    counts = {}
    for fused in (True, False):
        c = _Count()
        with c:
            _train_phase(d, tr, sk, poses, trans, conds, which, fused)
        counts[fused] = c.n
    print(f"{which}: aten ops of one train-phase block: fused {counts[True]}, composite {counts[False]}")
    assert counts[True] < counts[False]


def test_composite_kept_without_input_grad_only_or_second_order(monkeypatch):
    d, tr, sk, poses, trans, conds = _deformer()
    sk.second_order_fused = True
    gen = synth.generator(7)
    P = 300
    bi = torch.randint(0, 3, (P,), generator=gen).to(DEV)
    x = ((torch.rand((P, 3), generator=gen) - 0.5) * 1.6).to(DEV)
    # a raw create_graph request outside input_grad_only(): the pose gradient may be wanted too
    ps, p = x.clone().requires_grad_(True), poses.clone().requires_grad_(True)
    out = sk(ps, [p, trans], bi)
    (gps,) = torch.autograd.grad(out, ps, torch.ones_like(out), create_graph=True)
    assert sk.last_backward == "autograd-composite (create_graph)"
    gps.sum().backward()
    assert p.grad is not None and torch.isfinite(p.grad).all()
    # RECMV_SECOND_ORDER=0 (ops.SECOND_ORDER_FUSED false) keeps the torch graph even inside input_grad_only()
    monkeypatch.setattr(ops, "SECOND_ORDER_FUSED", False)
    ps, p = x.clone().requires_grad_(True), poses.clone().requires_grad_(True)
    out = sk(ps, [p, trans], bi)
    compute_Jacobian(ps, out, True, True)
    assert sk.last_backward == "autograd-composite (create_graph)"
