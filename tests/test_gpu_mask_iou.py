"""GPU tests of the mask-IoU kernel (csrc/mask_iou.cu, DESIGN section 1m) and the `mask_loss` drop-in
(utils.make_mask_loss): the dilation against F.max_pool2d bit for bit, I, U, the losses and dL/dm against the float64
oracle (oracle/mask_iou_oracle.py), run-to-run identity, the NaN of an empty frame, the refusals, and the drop-in
against the reference's own `mask_loss` (tests/golden/mask_loss_ref.npz) with its synchronising calls counted."""
import os
import sys
import types
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import mask_iou_oracle as mio
from recmv_b200 import _lib, ops, utils

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
DEV = "cuda"


def _masks(G, N, H, W, soft, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    ms, gts = [], []
    for _ in range(G):
        yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
        blob = ((yy - H * 0.45) / (H * 0.3)) ** 2 + ((xx - W * 0.5) / (W * 0.25)) ** 2 < 1
        m = torch.rand((N, H, W), generator=g) * blob
        if soft:
            gt = torch.rand((N, H, W), generator=g) * (torch.rand((N, H, W), generator=g) < 0.02)
        else:
            gt = (torch.rand((N, H, W), generator=g) < 0.01).float()
        gt[:, 0, :5] = 1.0                                          # touches the border
        gt[:, -1, -1] = 0.75
        ms.append(m.to(DEV))
        gts.append(gt.to(DEV))
    return ms, gts


def _ulps(x, ref):
    """|x - ref| in units of the float32 spacing at ref."""
    ref = np.asarray(ref, np.float64)
    sp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    return np.abs(np.asarray(x, np.float64) - ref) / sp


@pytest.mark.parametrize("shape", [(1080, 1080), (721, 1283)])
@pytest.mark.parametrize("r", [1, 2, 3, 7])
@pytest.mark.parametrize("soft", [False, True])
def test_dilation_is_max_pool2d_bit_for_bit(shape, r, soft):
    H, W = shape
    for G, N in ((1, 1), (2, 2), (1, 3), (2, 4)):
        ms, gts = _masks(G, N, H, W, soft, seed=31 * r + N)
        _, _, _, mgt = ops.mask_iou(ms, gts, r)
        for gt, out in zip(gts, mgt):
            ref = F.max_pool2d(gt, kernel_size=2 * r + 1, stride=1, padding=r)
            assert torch.equal(out.view(torch.int32), ref.view(torch.int32)), (G, N)


@pytest.mark.parametrize("shape,r,G,N", [((1080, 1080), 3, 2, 3), ((1080, 1080), 2, 1, 1), ((721, 1283), 7, 2, 4),
                                         ((33, 47), 1, 2, 2)])
@pytest.mark.parametrize("soft", [False, True])
def test_iou_and_vjp_against_float64(shape, r, G, N, soft):
    H, W = shape
    ms, gts = _masks(G, N, H, W, soft, seed=7 * r + G)
    loss, loss_gn, iu, mgt = ops.mask_iou(ms, gts, r)
    w = torch.tensor([0.75, -1.3][:G], device=DEV)
    dm = ops.mask_iou_backward(ms, mgt, iu, w)
    for g in range(G):
        m64, g64 = ms[g].double().cpu().numpy(), mgt[g].double().cpu().numpy()
        I, U, L, mean = mio.iou(m64, g64)
        assert _ulps(iu[g, :, 0].cpu().numpy(), I).max() <= 1, _ulps(iu[g, :, 0].cpu().numpy(), I)
        assert _ulps(iu[g, :, 1].cpu().numpy(), U).max() <= 1, _ulps(iu[g, :, 1].cpu().numpy(), U)
        assert _ulps(loss_gn[g].cpu().numpy(), L).max() <= 2, _ulps(loss_gn[g].cpu().numpy(), L)
        assert _ulps(loss[g].item(), mean) <= 2, _ulps(loss[g].item(), mean)
        # element-wise against the float64 formula at the kernel's own (I, U), which are checked above
        IU = iu[g].cpu().numpy()
        ref = mio.iou_vjp(m64, g64, float(w[g]), (IU[:, 0], IU[:, 1]))
        ref32 = ref.astype(np.float32).astype(np.float64)                    # the float64 VJP rounded once
        got = dm[g].double().cpu().numpy()
        err = np.abs(got - ref32) / np.spacing(np.abs(ref32).astype(np.float32)).astype(np.float64)
        assert err.max() <= 2, (g, float(err.max()))
        # and against the all-float64 VJP, relative to the size of the two terms that can cancel
        full = mio.iou_vjp(m64, g64, float(w[g]))
        Ib, Ub = I[:, None, None], U[:, None, None]
        scale = abs(float(w[g])) / N * (g64 * Ub + Ib * (1 - g64)) / (Ub * Ub)
        assert np.all(np.abs(got - full) <= 4e-7 * scale + 1e-30)


def test_runs_are_bit_identical():
    ms, gts = _masks(2, 3, 1080, 1080, True, seed=5)
    a = ops.mask_iou(ms, gts, 3)
    b = ops.mask_iou(ms, gts, 3)
    for x, y in zip(a[:3], b[:3]):
        assert torch.equal(x, y)
    da = ops.mask_iou_backward(ms, a[3], a[2], torch.ones(2, device=DEV))
    db = ops.mask_iou_backward(ms, b[3], b[2], torch.ones(2, device=DEV))
    assert all(torch.equal(x, y) for x, y in zip(da, db))


def test_empty_silhouette_and_mask_give_nan():
    z = torch.zeros((2, 40, 50), device=DEV)
    m = z.clone()
    m[1, 10, 10] = 0.5
    loss, loss_gn, iu, _ = ops.mask_iou([m], [z], 2)
    assert torch.isnan(loss_gn[0, 0]) and loss_gn[0, 1].item() == 1.0 and torch.isnan(loss[0])
    assert iu[0, 0].tolist() == [0.0, 0.0]
    mt = m.clone().requires_grad_(True)
    out = ops.MaskIouFunction.apply(2, mt, z)
    assert torch.isnan(out[0]).all()


def test_autograd_function_matches_the_backward_and_makes_no_sync():
    ms, gts = _masks(2, 2, 300, 200, True, seed=3)
    leaves = [m.clone().requires_grad_(True) for m in ms]
    w = torch.tensor([2.0, 0.5], device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = ops.MaskIouFunction.apply(3, *leaves, *gts)
        (out[0] * w).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    loss, _, iu, mgt = ops.mask_iou(ms, gts, 3)
    assert torch.equal(out[0], loss) and all(torch.equal(a, b) for a, b in zip(out[1:], mgt))
    assert not any(t.requires_grad for t in out[1:])
    dm = ops.mask_iou_backward(ms, mgt, iu, w)
    assert all(torch.equal(leaf.grad, d) for leaf, d in zip(leaves, dm))


def test_bad_inputs_are_refused():
    ms, gts = _masks(2, 2, 30, 40, False, seed=1)
    with pytest.raises(_lib.RecmvError):
        ops.mask_iou(ms, gts, 0)
    with pytest.raises(_lib.RecmvError):
        ops.mask_iou(ms, gts, 33)
    with pytest.raises(RuntimeError):
        ops.mask_iou(ms, [gts[0], gts[1][:, :29]], 1)                         # shapes disagree
    with pytest.raises(RuntimeError):
        ops.mask_iou(ms, gts[:1], 1)                                          # G disagrees
    with pytest.raises(RuntimeError):
        ops.mask_iou([ms[0].cpu(), ms[1]], gts, 1)                            # CPU
    with pytest.raises(RuntimeError):
        ops.mask_iou([ms[0].transpose(1, 2).contiguous().transpose(1, 2), ms[1]], gts, 1)   # non-contiguous
    with pytest.raises(RuntimeError):
        ops.mask_iou([ms[0].double(), ms[1]], gts, 1)                         # dtype
    with pytest.raises(RuntimeError):
        ops.MaskIouFunction.apply(1, ms[0], gts[0].clone().requires_grad_(True))


# ---- the drop-in against the reference's own mask_loss (tests/golden/mask_loss_ref.npz) ---------------------------
sys.path.insert(0, HERE)
NAMES = ("upper", "bottom")


def _fixture():
    z = np.load(os.path.join(HERE, "golden", "mask_loss_ref.npz"))
    return {k: z[k] for k in z.files}


def _camera(rows):
    c = torch.as_tensor(rows, dtype=torch.float32, device=DEV)
    return types.SimpleNamespace(focal_length=c[:, 0:2].contiguous(), principal_point=c[:, 2:4].contiguous(),
                                 R=c[:, 4:13].reshape(-1, 3, 3).contiguous(), T=c[:, 13:16].contiguous())


def find_surface_ps(self, meshes):
    """The reference's find_surface_ps (OptimGarmentNetwork.py:742-783) on this package's FindSurfacePs."""
    out = [[] for _ in range(5)]
    with torch.no_grad():
        for mesh, vs, fs in zip(meshes, self.garment_vs, self.garment_fs):
            _, frags = self.maskRender(mesh)
            for lst, x in zip(out, utils.FindSurfacePs(vs.detach(), fs, frags)):
                lst.append(x)
    return out[0], out[0], out[1], out[2], out[3], out[4]


def _scene(d):
    import surface_render_scene as srs
    from recmv_b200.compat.MaskRender import mask_renderer
    from recmv_b200.compat.PointRender import point_renderer
    sdf, deformer, _ = srs.networks(DEV)
    t = lambda k: torch.from_numpy(d[k].copy()).to(DEV)  # noqa: E731
    N, H, W = d["in/gt_0"].shape
    poses, trans = t("in/poses").requires_grad_(True), t("in/trans").requires_grad_(True)
    conds = [t("in/conds")[k].requires_grad_(True) for k in range(3)]
    vs = [t(f"in/V_{g}").requires_grad_(True) for g in range(2)]
    cam = _camera(d["in/cam"])
    conf = srs.Conf({"pc_weight.weight": 60.0, "pc_weight.laplacian_weight": -10.0, "pc_weight.edge_weight": -10.0,
                     "pc_weight.norm_weight": -0.001, "pc_weight.def_consistent.weight": 0.6,
                     "pc_weight.def_consistent.c": 0.01, "pc_weight.curve_aware_weight": 60.0})
    self = types.SimpleNamespace(
        garment_size=2, garment_names=list(NAMES), garment_nets=[sdf, sdf], garment_vs=vs,
        garment_fs=[t(f"in/F_{g}") for g in range(2)], deformer=deformer, conf=conf, info={}, sdfShrinkRadius=0.01,
        pcRender=point_renderer((H, W), float(d["ndc_radius"]), points_per_pixel=int(d["K"]), split=True, cameras=cam),
        maskRender=mask_renderer((H, W), cameras=cam), garment_optimizer=torch.optim.SGD(vs, lr=0.05, momentum=0.9),
        curve_aware_loss=lambda ratio: 0., get_grad_parameters=lambda frame_ids, device: (conds, poses, trans, None))
    self.find_surface_ps = types.MethodType(find_surface_ps, self)
    # fill the deformer's one-time host caches (bone parents, voxel box) before anything is counted
    x = vs[0].detach()[None].expand(N, -1, 3)
    (deformer(x, [conds[1], [poses, trans]], ratio=srs.RATIO, offset_type="warm").sum()
     + deformer.defs[1](x, [poses, trans]).sum()).backward()
    for p in [poses, trans] + conds + list(deformer.parameters()):
        p.grad = None
    deformer.defs[0].offset.pop("warm", None)
    gts = [t(f"in/gt_{g}") for g in range(2)]
    return self, (N, H, W, torch.arange(N, device=DEV), srs.RATIO, gts, DEV), (poses, trans, conds, vs, deformer)


def _close(got, ref, tol, what):
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    scale = max(np.abs(ref).max(), 1e-30)
    err = np.abs(got - ref).max() / scale
    assert err <= tol, (what, err)


def test_drop_in_reproduces_the_reference_mask_loss():
    d = _fixture()
    self, args, (poses, trans, conds, vs, deformer) = _scene(d)
    mask_loss = utils.make_mask_loss()
    syncs = {"renderers": 0}
    rec = []
    syncing = lambda: [w for w in rec if "synchroniz" in str(w.message).lower()]  # noqa: E731
    nsync = lambda: len(syncing())  # noqa: E731
    for name in ("maskRender", "pcRender"):
        inner = getattr(self, name)

        class Counted:
            rasterizer = inner.rasterizer

            def __call__(self_, *a, inner=inner, **k):
                n0 = nsync()
                out = inner(*a, **k)
                syncs["renderers"] += nsync() - n0
                return out

        setattr(self, name, Counted())
    fsp = utils.FindSurfacePs

    def counted_fsp(*a, **k):
        n0 = nsync()
        out = fsp(*a, **k)
        syncs["renderers"] += nsync() - n0
        return out

    utils.FindSurfacePs = counted_fsp
    torch.cuda.synchronize()
    try:
        with warnings.catch_warnings(record=True) as caught:
            rec = caught
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                meshes, masks, mgt, pc_sdf_loss, _ = mask_loss(self, *args)
            finally:
                torch.cuda.set_sync_debug_mode("default")
    finally:
        utils.FindSurfacePs = fsp
    assert nsync() == syncs["renderers"], (nsync(), syncs, [(w.filename, w.lineno) for w in syncing()])

    assert float(d["radius"]) == 2
    for g in range(2):
        assert torch.equal(mgt[g].cpu(), torch.from_numpy(d[f"f32/mgt_{g}"]))
        _close(masks[g][..., -1].detach().cpu(), d[f"f64/masks_{g}"], 2.5e-5, f"masks_{g}")
    info = dict(self.info["pc_loss"])
    info.update({k: v for k, v in self.info.items() if k != "pc_loss"})
    keys = sorted(k[len("f64/info/"):] for k in d if k.startswith("f64/info/"))
    assert sorted(info) == keys
    for k in keys:
        assert isinstance(info[k], torch.Tensor) and info[k].dim() == 0 and not info[k].requires_grad
        ref = float(d[f"f64/info/{k}"])
        # the mask losses are the kernel's: 1e-6 relative.  The template-consistency and SDF terms go through the
        # deformer and the SDF network on the GPU (the latter after the optimiser step): 1e-5 relative, their own
        # float32 / tensor-core error (the float32 reference itself misses 1e-6 on the consistency terms)
        tol = 1e-6 if k.endswith("_mask_loss") else 1e-5
        assert abs(info[k].item() - ref) <= tol * abs(ref), (k, info[k].item(), ref)
    ref = float(d["f64/pc_sdf_loss"])
    assert abs(pc_sdf_loss.item() - ref) <= 1e-5 * abs(ref)
    for g in range(2):
        _close(vs[g].detach().cpu(), d[f"f64/verts_after_{g}"], 2.5e-5, f"verts_after_{g}")
        assert len(meshes[g].verts_list()) == args[0]
    for k, x in (("poses", poses), ("trans", trans), ("cond1", conds[1]), ("cond2", conds[2])):
        _close(x.grad.cpu(), d[f"f64/grad/{k}"], 2.5e-5, k)
    names = [k[len("f64/grad/translator."):] for k in d if k.startswith("f64/grad/translator.")]
    assert names
    params = dict(deformer.defs[0].named_parameters())
    for pname in names:
        stride = 257
        got = params[pname].grad.detach().reshape(-1)[::stride].cpu()
        _close(got, d[f"f64/grad/translator.{pname}"], 2.5e-5, pname)


def test_drop_in_refusals():
    d = _fixture()
    self, args, _ = _scene(d)
    mask_loss = utils.make_mask_loss()
    self.conf.d["pc_weight.edge_weight"] = 1.0
    with pytest.raises(NotImplementedError):
        mask_loss(self, *args)
    self.conf.d["pc_weight.edge_weight"] = -10.0
    cpu_args = args[:5] + ([g.cpu() for g in args[5]],) + args[6:]
    with pytest.raises(RuntimeError):
        mask_loss(self, *cpu_args)
