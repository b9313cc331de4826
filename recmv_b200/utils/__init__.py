"""Mirror of the hot-path helpers of the reference's `utils` package (utils/utils.py:8-18,40-46,133-156,
198-264).  Same names, arguments and return values; the native calls go to librecmv_b200.so."""
import torch

from .. import ops as _ops
from ..model.Embedder import annealing_weights  # noqa: F401  (utils/utils.py:40-46)
from ..ops import FastDiff3x3MinvFunction  # noqa: F401    (utils/utils.py:8-18)
from . import FindSurfacePs as _fsp
from .FindSurfacePs import (FindSurfacePs, FindSurfacePsMesh, FindSurfacePsRays, OptimizeGarmentSurfacePs, OptimizeGarmentSurfaceSinlge,  # noqa: F401
                            OptimizeSurfacePs)


def compute_Jacobian(ps, ds, retain_graph, create_graph, allow_unused=False):
    """J = dD/dp by three autograd passes (utils/utils.py:133-156) -> [N,3,3], row i = grad of D_i."""
    rows = []
    go = torch.ones_like(ds[..., 0])
    for i in range(3):
        keep = True if i < 2 else retain_graph
        with _ops.input_grad_only():   # only d/d ps is asked for: create_graph stays on the tensor-core GEMMs
            g = torch.autograd.grad(ds[..., i], ps, go, retain_graph=keep, create_graph=create_graph,
                                    allow_unused=allow_unused)
        rows.append(g[0].view(-1, 1, 3))
    return torch.cat(rows, dim=1)


def _deform(deformer, ps, defconds, batch_inds, ratio, offset_type):
    return deformer(ps, defconds, batch_inds, ratio=ratio, offset_type=offset_type)


def _value_and_jacobian(deformer, ps, defconds, batch_inds, ratio, offset_type, check):
    """(D(p), J): one forward-mode launch of the fused deformer when no graph is kept (phase != train) and the
    composite is fusable; otherwise the reference's three autograd passes."""
    if not check and hasattr(deformer, "value_and_jacobian") and ps.is_cuda:
        with torch.no_grad():
            res = deformer.value_and_jacobian(ps, defconds, batch_inds, ratio=ratio, offset_type=offset_type)
        if res is not None:
            return res
    ds = _deform(deformer, ps, defconds, batch_inds, ratio, offset_type)
    return ds, compute_Jacobian(ps, ds, check, check)


def compute_cardinal_rays(deformer, ps, rays, defconds, batch_inds, ratio, phase, offset_type=None):
    """crays = normalize(J^-1 v) with the FastMinv singularity fallback (utils/utils.py:232-250)."""
    check = phase in ('train', 'Train')
    ds, J = _value_and_jacobian(deformer, ps, defconds, batch_inds, ratio, offset_type, check)
    Jinv, ok = FastDiff3x3MinvFunction.apply(J)
    crays = Jinv.matmul(rays.view(-1, 3, 1)).view(-1, 3)
    bad = ~ok
    if bad.sum().item() > 0:
        print('unwished error n_inv_mask:(%d:%d)' % (bad.sum().item(), bad.numel()))
        fixed = torch.zeros_like(crays)
        fixed[ok] = crays[ok]
        fixed[bad] = rays[bad].detach()
        crays = fixed
    crays = crays / crays.norm(dim=1, keepdim=True)
    return crays, ds


def compute_deformed_normals(sdf, deformer, ps, defconds, batch_inds, ratio, phase, offset_type):
    """n = normalize(J^-T grad sdf) (utils/utils.py:198-230)."""
    sdfs = sdf(ps, ratio)
    check = phase in ('train', 'Train')
    with _ops.input_grad_only():
        onx = torch.autograd.grad(sdfs, ps, torch.ones_like(sdfs), retain_graph=check, create_graph=check)[0]
    ds, J = _value_and_jacobian(deformer, ps, defconds, batch_inds, ratio, offset_type, check)
    Jinv, ok = FastDiff3x3MinvFunction.apply(J)
    nx = Jinv.transpose(-2, -1).matmul(onx.view(-1, 3, 1)).view(-1, 3)
    bad = ~ok
    if bad.sum().item() > 0:
        print('unwished error n_inv_mask:(%d:%d)' % (bad.sum().item(), bad.numel()))
        fixed = torch.zeros_like(nx)
        fixed[ok] = nx[ok]
        fixed[bad] = J[bad].matmul(onx[bad].unsqueeze(-1)).view(-1, 3)
        nx = fixed
    nx = nx / nx.norm(dim=1, keepdim=True)
    return nx, ds


def compute_netRender_color(net, ps, ds, ns, vs, features, framefeatures, ratio):
    """utils/utils.py:252-264 (the per-frame condition is ignored by the reference as well)."""
    return net(ps, ns, vs, features, ratio)


def implicit_surface_grad_coeffs(sdf, deformer, ps, rays, grad_l_p, defconds, batch_inds, ratio, offset_type=None,
                                 cam_pos=None):
    """The part of `propagateTmpPsGrad` (engineer/networks/OptimNetwork.py:726-879) between the two network
    evaluations, without autograd: grad f and J = dD/dp from the two forward-mode launches, then ONE kernel for the
    per-ray algebra (b = [grad f ; [v]x J], r = dL/dp (b^T b)^-1 b^T, FastMinv singularity rule).
    Returns (sdf_coef [N], def_vec [N,3], ray_grad [N,3] or None, ok [N], d [N,3]): the caller back-propagates
    `sdf_coef` through `sdf(ps)` and `def_vec` through `deformer(ps)` exactly as the reference does (lines 836-858)."""
    from .. import ops
    with torch.no_grad():
        f, gf = sdf.value_and_grad(ps.detach(), ratio.get('sdfRatio') if isinstance(ratio, dict) else ratio)
        d, J = _value_and_jacobian(deformer, ps.detach(), defconds, batch_inds, ratio, offset_type, False)
        dc = (d - cam_pos.view(1, 3)) if cam_pos is not None else None
        coef, vec, rg, ok = ops.surface_grad_coeffs(grad_l_p, gf, J, rays, dc)
    return coef, vec, rg, ok, d


def smooth_weights(weights, times=3):
    """utils/LBSWsmpl.py:2-11: model.Deformer.smooth_weights followed by weights < 5e-3 -> 0 (CUDA only)."""
    if not weights.is_cuda:
        raise RuntimeError("smooth_weights runs on CUDA tensors only (no CPU path)")
    return _ops.lbsw_smooth(_ops.voxel_to_channels_last(weights.float().contiguous()), times, 5e-3)[0]


def compute_lbswField(bmins, bmaxs, resolutions, smpl_verts, smpl_ws, align_corners=False, mean_neighbor=5,
                      smooth_times=30):
    """utils/LBSWsmpl.py:13-51 (exported as utils.compute_lbswField): the model/Deformer.py construction with the final
    5e-3 threshold.  CUDA only."""
    from ..model.Deformer import _lbsw_field
    return _lbsw_field(bmins, bmaxs, resolutions, smpl_verts, smpl_ws, align_corners, mean_neighbor, smooth_times,
                       5e-3)[0]


def GMRobustError(x, c, square=False):
    """Geman-McClure robust error (utils/utils.py:48-52)."""
    if square:
        return 2. * x / (c * c) / (x / (c * c) + 4)
    return 2. * x * x / (c * c) / (x * x / (c * c) + 4)


def eikonal_loss(sdf, pnts, ratio):
    """The eikonal term of the training step (engineer/networks/OptimGarmentNetwork.py:1108-1118;
    OptimNetwork.py's human branch is the same three lines): ((|grad_x sdf| - 1)^2).mean().
    `sdf.gradient` differentiates with create_graph=True; with the fused training path both that reverse chain and the
    backward of THIS loss run on the tensor-core GEMMs (recmv_b200/second_order.py)."""
    pnts.requires_grad_()
    pred = sdf(pnts, ratio)
    grad = sdf.gradient(pnts, pred)
    return ((grad.norm(2, dim=-1) - 1) ** 2).mean()


def deformation_regulariser(translator, pnts, d_cond, ratio, c, offset_type=None):
    """The deformation regulariser (OptimGarmentNetwork.py:1135-1154): Jacobian of the canonical-space deformation by
    three create_graph passes, its singular values, log, Geman-McClure on sum(log^2 s).  The reference copies the
    Jacobians to the host for `torch.svd`; here they stay on the device (ops.svd3x3, csrc/svd3.cu)."""
    pnts.requires_grad_()
    defVs = translator(pnts, d_cond, ratio=ratio, offset_type=offset_type)
    Jacobs = compute_Jacobian(pnts, defVs, True, True)
    _, s, _ = _ops.svd3x3(Jacobs)
    s = torch.log(s)
    return GMRobustError((s * s).sum(1), c, True).mean()
