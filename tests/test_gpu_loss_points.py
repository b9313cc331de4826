"""GPU tests of surface_render_loss on the device (DESIGN section 1k): the loss-point sampler and check compaction
(csrc/loss_points.cu) bit for bit against oracle/loss_points_oracle.py, the per-frame means (csrc/frame_loss.cu)
against float64 with their backward, and the drop-in utils.make_surface_render_loss against the reference's glue
restated in torch on the same networks and points (tests/surface_render_scene.py)."""
import warnings

import numpy as np
import pytest
import torch

from oracle import loss_points_oracle as lpo
from recmv_b200 import ops, utils

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SEED = 0x5EED0123456789AB


def _garments(rng, Ms, Vs, frac=0.7):
    out = []
    for M, V in zip(Ms, Vs):
        out.append(dict(P=rng.standard_normal((M, 3)).astype(np.float32), V=rng.standard_normal((V, 3)).astype(np.float32),
                        check=rng.uniform(size=M) < frac, b=rng.integers(0, 4, M), r=rng.integers(0, 64, M),
                        c=rng.integers(0, 64, M), rays=rng.standard_normal((M, 3)).astype(np.float32)))
    return out


def _run(gs, seed, offset):
    t = lambda x, dt=None: torch.from_numpy(np.ascontiguousarray(x)).to(DEV, dt)  # noqa: E731
    return ops.loss_points_sample([t(g["P"]) for g in gs], [t(g["V"]) for g in gs], [t(g["check"]) for g in gs],
                                  [t(g["b"], torch.int64) for g in gs], [t(g["r"], torch.int64) for g in gs],
                                  [t(g["c"], torch.int64) for g in gs], [t(g["rays"]) for g in gs],
                                  4096 // len(gs), seed, offset)


def _same(got, want, flags=None):
    got = got.cpu().numpy()
    assert got.shape == want.shape, (got.shape, want.shape)
    diff = (got.view(np.uint32) != want.view(np.uint32)).any(1)
    if flags is not None:
        diff &= ~flags
    assert not diff.any(), np.flatnonzero(diff)[:10]


S1 = 4096


@pytest.mark.parametrize("Ms,Vs,offset", [
    ((700,), (5000,), 0),
    ((600, 450), (2500, 3100), 123),
    ((300, 0, 90, 1, 257), (900, 820, 819, 818, 1000), 77),         # S = 819: V at S - 1, S and S + 1
    ((0,), (S1 - 1,), 5), ((10,), (S1,), 5), ((10,), (S1 + 1,), 5),
    ((513, 129), (7000, 2049), (1 << 32) - 20000),                  # counters cross into the high word
])
def test_sampler_is_bit_identical_to_the_oracle(Ms, Vs, offset):
    rng = np.random.default_rng(sum(Ms) + sum(Vs))
    gs = _garments(rng, Ms, Vs)
    out = _run(gs, SEED, offset)
    want, nxt = lpo.sample([g["P"] for g in gs], [g["V"] for g in gs], [g["check"] for g in gs], SEED, offset)
    assert nxt == (offset + 5 * (sum(Ms) + sum(Vs))) % (1 << 64)
    for g, (o, w) in enumerate(zip(out, want)):
        X_E, X_D, ps, rays, b, r, c, idx = o
        _same(X_E, w["X_E"], w["flag_e"])
        _same(X_D, w["X_D"], w["flag_d"])
        k = w["checked"]
        assert np.array_equal(idx.cpu().numpy(), k)
        _same(ps, gs[g]["P"][k].reshape(-1, 3))
        _same(rays, gs[g]["rays"][k].reshape(-1, 3))
        for got, src in ((b, "b"), (r, "r"), (c, "c")):
            assert np.array_equal(got.cpu().numpy(), gs[g][src][k])
        gl = X_E[len(X_E) - (Ms[g] + len(w["keep_e"])) // 6:]
        if gl.numel():
            assert float(gl.min()) >= -1.8 and float(gl.max()) < 1.8
    again = _run(gs, SEED, offset)
    for o, a in zip(out, again):
        for x, y in zip(o, a):
            assert torch.equal(x, y)


def test_all_false_check_and_refusals():
    rng = np.random.default_rng(3)
    gs = _garments(rng, (64,), (100,), frac=0.0)
    out = _run(gs, SEED, 0)
    assert all(t.shape[0] == 0 for t in out[0][2:])
    gs[0]["V"] = gs[0]["V"][:0]
    with pytest.raises(RuntimeError):
        _run(gs, SEED, 0)
    g = _garments(rng, (8,), (16,))[0]
    with pytest.raises(RuntimeError):
        ops.loss_points_sample([torch.from_numpy(g["P"])], [torch.from_numpy(g["V"])], [torch.from_numpy(g["check"])],
                               *[[torch.from_numpy(g[k])] for k in ("b", "r", "c")], [torch.from_numpy(g["rays"])], 4096,
                               1, 0)


def test_more_than_2_24_rows():
    M, V = (1 << 24) + 300, 5000
    gen = torch.Generator(device=DEV).manual_seed(4)
    P = torch.randn((M, 3), device=DEV, generator=gen)
    Vt = torch.randn((V, 3), device=DEV, generator=gen)
    check = torch.rand((M,), device=DEV, generator=gen) < 0.5
    ar = torch.arange(M, device=DEV)
    rays = torch.randn((M, 3), device=DEV, generator=gen)
    offset = (1 << 32) - 7 * M
    (X_E, X_D, ps, rays_c, b, r, c, idx), = ops.loss_points_sample([P], [Vt], [check], [ar], [ar], [ar], [rays], 4096,
                                                                    SEED, offset)
    k = torch.nonzero(check)[:, 0]
    assert torch.equal(idx, k) and torch.equal(ps, P[k]) and torch.equal(rays_c, rays[k]) and torch.equal(b, k)
    keep_e = lpo.draw(SEED, offset, 0, lpo.E_DRAW, M + V, V, 4096)
    keep_d = lpo.draw(SEED, offset, 0, lpo.D_DRAW, M + V, V, 4096)
    nE, nD = M + len(keep_e), M + len(keep_d)
    assert X_E.shape[0] == nE + nE // 6 and X_D.shape[0] == 2 * nD
    assert torch.equal(X_D[:M], P) and torch.equal(X_D[M:nD].cpu(), torch.from_numpy(np.asarray(Vt.cpu())[keep_d]))
    Pc = P.cpu().numpy()
    rows = np.array([0, 1, (1 << 24) - 1, 1 << 24, M - 1])
    z, flag = lpo.normals(SEED, lpo.counters(offset, 0, lpo.E_LOCAL, M + V, M)[rows])
    _same(X_E[torch.from_numpy(rows).to(DEV)], lpo.local(Pc[rows], z), flag)
    z, flag = lpo.normals(SEED, lpo.counters(offset, 0, lpo.D_LOCAL, M + V, M)[rows])
    _same(X_D[torch.from_numpy(nD + rows).to(DEV)], lpo.local(Pc[rows], z), flag)
    gi = np.array([0, nE // 6 - 1])
    _same(X_E[torch.from_numpy(nE + gi).to(DEV)], lpo.global_points(SEED, lpo.counters(offset, 0, lpo.E_GLOBAL, M + V,
                                                                                       nE // 6)[gi]))


def _ulp_close(got, want, ulps=1):
    got = np.asarray(got, np.float32).astype(np.float64)
    want = np.asarray(want, np.float64)
    tol = ulps * np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    bad = np.abs(got - want) > tol
    assert not bad.any(), (np.flatnonzero(bad)[:8], got[bad][:8], want[bad][:8])


def _frames(rng, M, N, H=5, W=7):
    b = rng.integers(0, N, M)
    if N > 2:
        b[b == 1] = 0                              # frame 1 empty
    return b, rng.integers(0, H, M), rng.integers(0, W, M), H, W


@pytest.mark.parametrize("N", range(1, 9))
@pytest.mark.parametrize("M", [0, 1, 37, 1025, 5000])
def test_color_frame_mean_against_float64(N, M):
    rng = np.random.default_rng(10 * N + M)
    b, r, c, H, W = _frames(rng, M, N)
    gt = rng.uniform(size=(N, H, W, 3)).astype(np.float32)
    col = rng.uniform(size=(M, 3)).astype(np.float32)
    if M:
        col[: M // 3] = gt[b[: M // 3], r[: M // 3], c[: M // 3]]     # gt == col: sign 0
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(DEV)  # noqa: E731
    colt = t(col).requires_grad_(True)
    L = ops.ColorFrameMeanFunction.apply(colt, t(gt), t(b), t(r), t(c), N)
    L2 = ops.ColorFrameMeanFunction.apply(t(col), t(gt), t(b), t(r), t(c), N)
    assert L.view(1).view(torch.int32).item() == L2.view(1).view(torch.int32).item()
    L.backward(torch.tensor(0.75, device=DEV))
    Lw, dcol = lpo.color_mean(gt, b, r, c, col, N, 0.75)
    _ulp_close(L.item(), Lw)
    _ulp_close(colt.grad.cpu().numpy(), dcol)


@pytest.mark.parametrize("N", range(1, 9))
@pytest.mark.parametrize("M", [0, 1, 37, 1025, 5000])
def test_normal_frame_mean_against_float64(N, M):
    rng = np.random.default_rng(100 * N + M)
    b = _frames(rng, M, N)[0]
    gtn = rng.standard_normal((M, 3)).astype(np.float32)
    gtn[: M // 5] *= 1e-5                                             # invalid normals
    J = (np.eye(3) + 0.3 * rng.standard_normal((M, 3, 3))).astype(np.float32)
    nx = rng.standard_normal((M, 3)).astype(np.float32)
    w = rng.uniform(size=M).astype(np.float32)
    if M > 10:                                                        # |d| = 0 rows
        J[-5:] = np.eye(3, dtype=np.float32)
        gtn[-5:] = np.array([0., 0., 2.], np.float32)
        nx[-5:] = np.array([0., 0., 1.], np.float32)
    if N == 3 and M:
        gtn[:] = 0.                                                   # all invalid
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(DEV)  # noqa: E731
    ins = [t(gtn).requires_grad_(True), t(J).requires_grad_(True), t(nx).requires_grad_(True)]
    L = ops.NormalFrameMeanFunction.apply(*ins, t(w), t(b), N)
    L2 = ops.NormalFrameMeanFunction.apply(t(gtn), t(J), t(nx), t(w), t(b), N)
    assert L.view(1).view(torch.int32).item() == L2.view(1).view(torch.int32).item()
    L.backward(torch.tensor(1.25, device=DEV))
    Lw, dg, dJ, dnx = lpo.normal_mean(gtn, J, nx, w, b, N, 1.25)
    _ulp_close(L.item(), Lw)
    for got, want in zip(ins, (dg, dJ, dnx)):
        _ulp_close(got.grad.cpu().numpy().reshape(want.shape), want)


@pytest.fixture(scope="module")
def nets():
    import surface_render_scene as srs
    return srs.networks(DEV)


def _fresh(nets, **kw):
    import surface_render_scene as srs
    return srs.scene(DEV, nets=nets, **kw)


def _params(self):
    mods = [self.garment_nets[0], self.deformer.defs[0], self.netRender]
    return {f"{type(m).__name__}.{n}": p for m in mods for n, p in m.named_parameters()}


def merr(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def test_drop_in_matches_the_reference_flow_on_the_same_points(nets):
    import surface_render_scene as srs
    fn = utils.make_surface_render_loss()
    s1, a1, (conds, poses, trans) = _fresh(nets)
    for p in _params(s1).values():
        p.grad = None
    loss = fn(s1, *a1)
    loss.backward()
    g1 = {k: p.grad.clone() for k, p in _params(s1).items() if p.grad is not None}
    g1.update({k: t.grad.clone() for k, t in (("poses", poses), ("trans", trans)) if t.grad is not None})
    pts = {}
    seed, off = fn.stream["seed"], fn.stream["offset"]
    # the drop-in's points, re-drawn by the same stream at the same offset
    P = [p.float() for p in a1[7]]
    V = s1.garment_vs
    again = ops.loss_points_sample(P, V, list(a1[5]), list(a1[10]), list(a1[8]), list(a1[9]), list(a1[11]), 2048, seed,
                                   off - 5 * sum(int(p.shape[0]) + int(v.shape[0]) for p, v in zip(P, V)))
    for g, o in enumerate(again):
        pts[g] = (o[0], o[1])
        k = a1[5][g]
        assert torch.equal(s1.TmpPs[g].detach(), a1[7][g][k]) and s1.TmpPs[g].is_leaf and s1.TmpPs[g].requires_grad
        assert torch.equal(s1.rays[g], a1[11][g][k]) and torch.equal(s1.batch_inds[g], a1[10][g][k])
        assert torch.equal(s1.row_inds[g], a1[8][g][k]) and torch.equal(s1.col_inds[g], a1[9][g][k])
        assert s1.TmpPs[g].grad is not None
    s2, a2, (conds2, poses2, trans2) = _fresh(nets)
    for p in _params(s2).values():
        p.grad = None
    ref = srs.reference_flow(s2, *a2, points=lambda g, P, V: pts[g])
    ref.backward()
    g2 = {k: p.grad.clone() for k, p in _params(s2).items() if p.grad is not None}
    g2.update({k: t.grad.clone() for k, t in (("poses", poses2), ("trans", trans2)) if t.grad is not None})
    print("loss", float(loss.detach()), float(ref.detach()))
    assert abs(float(loss) - float(ref)) < 2e-5 * abs(float(ref))
    for key, v in s2.info.items():
        if key.endswith("rayInfo"):
            continue
        assert abs(float(s1.info[key]) - float(v)) <= 2e-5 * max(abs(float(v)), 1e-6), (key, s1.info[key], v)
    assert set(g1) == set(g2)
    worst = max((merr(g1[k], g2[k]), k) for k in g1 if float(g2[k].abs().max()) > 1e-12)
    print("worst parameter gradient", worst)
    assert worst[0] < 1e-2
    # propagateTmpPsGrad (OptimGarmentNetwork.py:2159-2290) on the drop-in's state, as this package runs it: it reads
    # TmpPs[g].grad, rays, batch_inds and the garment's deformer conditions, solves the per-ray algebra
    # (implicit_surface_grad_coeffs), then back-propagates the SDF coefficients through sdf(TmpPs) and the deformation
    # vectors through deformer(TmpPs, ..., batch_inds) into the parameters and conditions
    for p in _params(s1).values():
        p.grad = None
    for g in range(s1.garment_size):
        ps, defconds = s1.TmpPs[g], [conds[g + 1], [poses, trans]]
        assert ps.grad is not None and not s1.rays[g].requires_grad
        coef, vec, rg, ok, d = utils.implicit_surface_grad_coeffs(
            s1.garment_nets[g], s1.deformer, ps, s1.rays[g], ps.grad, defconds, s1.batch_inds[g], a1[4],
            offset_type=s1.garment_names[g])
        assert coef.shape[0] == ps.shape[0] and bool(torch.isfinite(vec).all()) and bool(ok.any())
        p = ps.detach()
        f = s1.garment_nets[g](p, a1[4]).view(-1)
        dd = s1.deformer(p, defconds, s1.batch_inds[g], ratio=a1[4], offset_type=s1.garment_names[g])
        ((f * coef.view(-1)).sum() + (dd * vec).sum()).backward()
    moved = [k for k, p in _params(s1).items() if p.grad is not None and bool(torch.isfinite(p.grad).all())]
    assert any(k.startswith("ImplicitNetwork") for k in moved) and any(k.startswith("MLPTranslator") for k in moved)


def test_drop_in_reads_the_host_once(nets):
    fn = utils.make_surface_render_loss()
    s, a, _ = _fresh(nets)
    fn(s, *a).backward()                                 # warm-up: workspaces, pinned counters
    s, a, _ = _fresh(nets)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            loss = fn(s, *a)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [w for w in rec if str(w.message).startswith("called a synchronizing CUDA operation")]
    assert len(syncs) == 1, [str(w.message) for w in syncs]
    assert s.conf.get_bool("weighted_normal") and s.garment_size == 2
    assert all(isinstance(v, torch.Tensor) for k, v in s.info.items() if k.endswith("_loss"))
    loss.backward()


def test_drop_in_refuses_cpu_tensors_and_offset_weight(nets):
    import surface_render_scene as srs
    fn = utils.make_surface_render_loss()
    s, a, _ = _fresh(nets)
    a = list(a)
    a[7] = [p.cpu() for p in a[7]]
    with pytest.raises(RuntimeError):
        fn(s, *a)
    s, a, _ = _fresh(nets, conf=dict(srs.CONF, offset_weight=0.5))
    with pytest.raises(NotImplementedError):
        fn(s, *a)


def test_drop_in_matches_the_reference_fixture(nets):
    """The drop-in against the reference's own surface_render_loss run on the CPU from the same inputs and the same
    stream (tests/golden/make_golden_surface_render_loss.py): the compacted rows bit for bit, the loss and every info
    term against float64 within the fused second-order path's tolerances (tests/test_gpu_second_order.py: 2e-5 of the
    loss; parameter gradients 1e-2 of each tensor's largest entry), with the float32 reference as the yardstick."""
    import types
    import surface_render_scene as srs
    from conftest import load_golden
    z = load_golden("surface_render_loss_ref.npz")
    t = lambda k, dt=None: torch.from_numpy(np.ascontiguousarray(z[k])).to(DEV, dt)  # noqa: E731
    sdf, deformer, rn = nets
    N = int(z["in/poses"].shape[0])
    poses, trans = t("in/poses").requires_grad_(True), t("in/trans").requires_grad_(True)
    conds = [t("in/conds")[k].clone().requires_grad_(True) for k in range(3)]
    rendcond = torch.zeros((N, 1), device=DEV)
    names = ["upper", "bottom"]
    self = types.SimpleNamespace(
        garment_size=2, garment_names=names, garment_nets=[sdf, sdf], garment_vs=[t(f"in/V_{g}") for g in range(2)],
        deformer=deformer, netRender=rn, info={f"{names[g]}_rayInfo": (int(z[f"in/P_{g}"].shape[0]),
                                                                         int(z[f"in/check_{g}"].sum())) for g in range(2)},
        conf=srs.Conf(dict(srs.CONF)), get_grad_parameters=lambda frame_ids, device: (conds, poses, trans, rendcond))
    cameras = types.SimpleNamespace(R=t("in/R").view(1, 3, 3).expand(N, 3, 3))
    mods = {"sdf": sdf, "translator": deformer.defs[0], "render": rn}
    for m in mods.values():
        m.zero_grad(set_to_none=True)
    fn = utils.make_surface_render_loss()
    fn.stream.update(seed=int(z["seed"]), offset=int(z["offset"]))
    loss = fn(self, {"normal": t("in/normal")}, N, cameras, torch.arange(N, device=DEV), srs.RATIO,
              [t(f"in/check_{g}") for g in range(2)], t("in/gtCs"), [t(f"in/P_{g}") for g in range(2)],
              [t(f"in/row_{g}", torch.int64) for g in range(2)], [t(f"in/col_{g}", torch.int64) for g in range(2)],
              [t(f"in/batch_{g}", torch.int64) for g in range(2)], [t(f"in/rays_{g}") for g in range(2)], DEV)
    loss.backward()
    for g in range(2):
        assert np.array_equal(self.TmpPs[g].detach().cpu().numpy(), z[f"f32/TmpPs_{g}"])
        assert np.array_equal(self.rays[g].cpu().numpy(), z[f"f32/rays_c_{g}"])
        for key, src in (("batch", self.batch_inds), ("row", self.row_inds), ("col", self.col_inds)):
            assert np.array_equal(src[g].cpu().numpy(), z[f"f32/{key}_c_{g}"])
    f64 = float(z["f64/loss"])
    print("loss", float(loss.detach()), "f32 reference", float(z["f32/loss"]), "f64 reference", f64)
    assert abs(float(loss.detach()) - f64) < 2e-5 * abs(f64)
    infos = sorted(k[len("f64/info/"):] for k in z if k.startswith("f64/info/"))
    assert infos == sorted(k for k in self.info if not k.endswith("rayInfo"))
    for k in infos:
        ours, ref, ref32 = float(self.info[k]), float(z[f"f64/info/{k}"]), float(z[f"f32/info/{k}"])
        print(f"{k}: ours {ours:.9g}  f64 {ref:.9g}  f32 reference {ref32:.9g}")
        assert abs(ours - ref) <= max(2e-5 * abs(ref), 4 * abs(ref32 - ref)), k
    grads = {}
    for mname, m in mods.items():
        for pname, p in sorted(m.named_parameters()):
            if p.grad is not None:
                grads[f"grad/{mname}.{pname}"] = p.grad.detach().reshape(-1)[::257]
    for k, x in (("poses", poses), ("trans", trans), ("cond0", conds[0]), ("cond1", conds[1]), ("cond2", conds[2])):
        if x.grad is not None:
            grads[f"grad/{k}"] = x.grad.detach()
    ref_keys = sorted(k[len("f64/"):] for k in z if k.startswith("f64/grad/"))
    nonzero = lambda k: float(np.abs(z["f64/" + k]).max()) > 0  # noqa: E731
    assert [k for k in ref_keys if nonzero(k)] == sorted(k for k in grads if k in ref_keys and nonzero(k))
    assert all(k in grads for k in ref_keys if nonzero(k))
    rows = []
    for k in ref_keys:
        if not nonzero(k):
            continue
        ref = torch.from_numpy(z["f64/" + k]).double()
        ours = grads[k].double().cpu().reshape(ref.shape)
        scale = float(ref.abs().max())
        rows.append((float((ours - ref).abs().max()) / scale,
                     float((torch.from_numpy(z["f32/" + k]).double() - ref).abs().max()) / scale, k))
    for e, e32, k in sorted(rows)[-8:]:
        print(f"{k}: |ours - f64| {e:.2e} of scale, |f32 reference - f64| {e32:.2e}")
    assert max(rows)[0] < 1e-2, max(rows)
