"""Mirror of the hot-path helpers of the reference's `utils` package (utils/utils.py:8-18,40-46,133-156,
198-264).  Same names, arguments and return values; the native calls go to librecmv_b200.so."""
import torch

from .. import ops as _ops
from .. import raster as _raster
from ..knn import chamfer_distance
from ..model.Embedder import annealing_weights  # noqa: F401  (utils/utils.py:40-46)
from ..ops import FastDiff3x3MinvFunction  # noqa: F401    (utils/utils.py:8-18)
from . import FindSurfacePs as _fsp
from .FindSurfacePs import (FindSurfacePs, FindSurfacePsMesh, FindSurfacePsRays, OptimizeGarmentSurfacePs, OptimizeGarmentSurfaceSinlge,  # noqa: F401
                            OptimizeSurfacePs)


def _pad_points(t, P):
    return t if t.shape[1] == P else torch.cat([t, t.new_zeros((t.shape[0], P - t.shape[1]) + tuple(t.shape[2:]))], 1)


def fl_proj_loss(fl_pts_list, gt_fl_pts_list, fl_masks, proj_fl_weights=None):
    """The feature-curve projection loss (engineer/core/fl_optimizer.py:72-110), batched: C curves with screen points
    fl_pts [N,P_c,>=2] (x, y first), annotations gt [N,M_c,2], per-point visibility fl_masks [N,P_c,3] (the call site
    expands one flag over the coordinates, so [..., 0] is read) and Python-number weights w_c (default 1).
    S_{n,c} = sum-reduced chamfer distance of frame n's visible points and its annotations (0 with none visible),
    V_c = frames with a visible point, Q_c = visible points; L = mean_c w_c sum_n S_{n,c} / (V_c or 1) / (Q_c or 1).
    The C*N clouds go through one nearest-neighbour call per direction; visible points are compacted on the device by
    a stable partition.  No host synchronisation in the forward or the backward."""
    C = len(fl_pts_list)
    N = int(fl_pts_list[0].shape[0])
    dev = fl_pts_list[0].device
    P = max(int(p.shape[1]) for p in fl_pts_list)
    Ms = [int(g.shape[1]) for g in gt_fl_pts_list]
    M = max(Ms)
    x = torch.stack([_pad_points(p[..., :2], P) for p in fl_pts_list]).reshape(C * N, P, 2)
    vis = torch.stack([_pad_points(m[..., 0] != 0, P) for m in fl_masks]).reshape(C * N, P)
    order = torch.argsort((~vis).to(torch.uint8), dim=1, stable=True)     # visible points first, in their order
    xc = torch.gather(x, 1, order[..., None].expand(-1, -1, 2)).contiguous()
    lx = vis.sum(1)
    y = torch.stack([_pad_points(g, M) for g in gt_fl_pts_list]).reshape(C * N, M, 2).contiguous()
    ly = None if min(Ms) == M else torch.cat([torch.full((N,), m, dtype=torch.int64, device=dev) for m in Ms])
    S = chamfer_distance(xc, y, lx, ly, batch_reduction=None, point_reduction="sum")[0].view(C, N).sum(1)
    cnt = lx.view(C, N)
    V, Q = (cnt > 0).sum(1), cnt.sum(1)
    w = [1.0] * C if proj_fl_weights is None else [float(v) for v in proj_fl_weights]
    w = torch.tensor(w, dtype=S.dtype).pin_memory().to(dev, non_blocking=True)
    return (w * S / V.clamp_min(1) / Q.clamp_min(1)).sum() / C


def _curve_index(fl_names, target):
    """The reference's `for fl_idx, name in enumerate(fl_names): if name == target: break`: a missing name falls
    through to the last curve."""
    return next((i for i, n in enumerate(fl_names) if n == target), len(fl_names) - 1)


def make_curve_aware_loss(curve_aware, samples=50000):
    """`OptimGarmentNetwork.curve_aware_loss(self, ratio)` (OptimGarmentNetwork.py:787-839) with the fans sampled on the
    GPU; bind it as `OptimGarmentNetwork.curve_aware_loss = make_curve_aware_loss(CURVE_AWARE)`.
    As the reference: 0. when `pc_weight.curve_aware_weight` is 0; the `upper_bottom` curve's term whenever that curve
    exists, the `curve_aware[garment_type]` curve's term when `isfine` (a missing name falls through to the last
    curve); each term mean |sdf(p) + sdfShrinkRadius| through `garment_nets[-1]` over `samples` area-weighted points of
    the fan (the curve, its centroid, faces (i, i+1, P) and (P-1, 0, P)), times the weight (60 without `pc_weight`).
    The samples are detached, as the reference's host copy is.  Unlike the reference, all fans of a call are sampled
    in one launch (csrc/surface_sample.cu) and evaluated in one SDF forward, `info['pc_<name>_circle_loss_sdf']` holds
    a detached 0-d tensor, and nothing is read back to the host.  The stream's seed is drawn from torch's CPU
    generator at the first call (so `torch.manual_seed` makes a run reproducible) and its offset advances by
    curves * samples per call; both are in the returned function's `stream` dict."""
    stream = {"seed": None, "offset": 0}

    def curve_aware_loss(self, ratio):
        ca_loss = 0.
        if self.conf.get_float('pc_weight.curve_aware_weight') == 0.:
            return ca_loss
        terms = []
        if 'upper_bottom' in self.fl_names:
            terms.append(('upper_bottom', _curve_index(self.fl_names, 'upper_bottom')))
        if self.garment_type in curve_aware and self.isfine:
            target = curve_aware[self.garment_type]
            terms.append((target, _curve_index(self.fl_names, target)))
        if not terms:
            return ca_loss
        curves = self.inter_free_curve.forward()
        pts = torch.stack([curves[i] for _, i in terms]).detach().float()
        if not pts.is_cuda:
            raise RuntimeError("curve_aware_loss runs on CUDA tensors only (no CPU path)")
        M, P = int(pts.shape[0]), int(pts.shape[1])
        verts = torch.cat([pts, pts.mean(1, keepdim=True)], 1).contiguous()
        i = torch.arange(P, device=pts.device)
        faces = torch.stack([i, (i + 1) % P, torch.full_like(i, P)], 1)
        if stream["seed"] is None:
            stream["seed"] = int(torch.empty((), dtype=torch.int64).random_())
        surface_pts = _ops.surface_sample(verts, faces, samples, stream["seed"], stream["offset"])
        stream["offset"] += M * samples
        mnfld_pred = self.garment_nets[-1](surface_pts.view(-1, 3), ratio).view(M, samples)
        circle_sdf_loss = (mnfld_pred + self.sdfShrinkRadius).abs().mean(1)
        for (name, _), v in zip(terms, circle_sdf_loss.detach().unbind(0)):
            self.info['pc_{}_circle_loss_sdf'.format(name)] = v
        weight = self.conf.get_float('pc_weight.curve_aware_weight') if 'pc_weight' in self.conf else 60.
        return (circle_sdf_loss * weight).sum()

    curve_aware_loss.stream = stream
    return curve_aware_loss


def _probe_settings(mask_render):
    """(cameras, (H, W), z_clip, area_eps) of a `maskRender`: its rasterizer's cameras and settings, the image size an
    int or (H, W) as in pytorch3d's RasterizationSettings."""
    r = mask_render.rasterizer
    s = r.raster_settings
    size = s.image_size
    H, W = (int(size), int(size)) if isinstance(size, int) else (int(size[0]), int(size[1]))
    return r.cameras, (H, W), float(getattr(s, "z_clip", 1e-6)), float(getattr(s, "area_eps", 1e-8))


def _cam_z(cameras):
    """cam_pos()[2] of camera 0 (CameraMine.cam_pos, -R T) as a device 0-d tensor."""
    if hasattr(cameras, "cam_pos"):
        return cameras.cam_pos()[2]
    R, T = (torch.as_tensor(x, dtype=torch.float32) for x in (cameras[2], cameras[3]))
    return -R.reshape(-1, 3, 3)[0].matmul(T.reshape(-1, 3)[0].view(-1, 1)).view(-1)[2]


def fl_visible_by_body_zbuff(self, cameras, d_cond_list, poses, ratio, fl_vs_dict, def_fl_vs, cano_smpl_verts_list,
                             fl_names, g_i, garment_name, proj_size, N):
    """`OptimGarmentNetwork.fl_visible_by_body_zbuff` (OptimGarmentNetwork.py:1374-1465) on the sparse z-buffer probe;
    bind it as `OptimGarmentNetwork.fl_visible_by_body_zbuff = fl_visible_by_body_zbuff` (the Large-Pose class inherits
    it).  Returns [N,P,2] = (garment check, body check) for the P curve points, with the reference's formulas: c_z =
    cam_pos()[2] of the renderer's camera 0; garment column z - (s + c_z), s the bilinear sample of the deformed
    garment's zbuf with background filled by max_v(Z - c_z) over the deformed garment vertices; body column the same
    for the skinned canonical-SMPL curve points against the skinned `tmpBodyVs` / `tmpBodyFs`.  The zbuf is the one
    `self.maskRender` would rasterize (its cameras, image size and clip settings); the screen points come from the
    `cameras` argument and are normalised by `proj_size`.  Only the pixels the samples read are rasterized
    (raster.zbuf_probe), nothing is read back to the host, and the deformers run without a graph: the result is
    detached, as the reference's outputs feed only `<` comparisons."""
    rcams, size, z_clip, area_eps = _probe_settings(self.maskRender)
    with torch.no_grad():
        c_z = _cam_z(rcams).detach()
        def_garment_vs = self.deformer(self.garment_vs[g_i][None, :, :].expand(N, -1, 3), [d_cond_list[g_i + 1], poses],
                                       ratio=ratio, offset_type=garment_name)
        fl = torch.cat(def_fl_vs, dim=1).detach()
        fill = (def_garment_vs[..., -1] - c_z).max(-1)[0]
        s = _raster.zbuf_probe(def_garment_vs, self.garment_fs[g_i], rcams, size, _raster.screen_points(fl, cameras),
                               proj_size, fill, z_clip, area_eps)
        garment_check = fl[..., -1] - (s + c_z)
        smpl_fl = torch.cat([self.deformer.defs[1](v.expand(N, -1, 3), poses)
                             for v, _ in zip(cano_smpl_verts_list, fl_names)], dim=1)
        body = self.deformer.defs[1](self.tmpBodyVs.view(1, -1, 3).expand(N, -1, 3), poses)
        fill = (body[..., -1] - c_z).max(-1)[0]
        s = _raster.zbuf_probe(body, self.tmpBodyFs, rcams, size, _raster.screen_points(smpl_fl, cameras), proj_size,
                               fill, z_clip, area_eps)
        smpl_check = smpl_fl[..., -1] - (s + c_z)
    return torch.stack([garment_check, smpl_check], -1)


def check_zbuf_body(smpl_mesh, N, deform_lbs, poses, trans, cameras, mask_render, img_size, screen_pts):
    """`engineer.core.fl_optimizer.check_zbuf_body` (fl_optimizer.py:30-59) on the sparse z-buffer probe; bind it as
    `fl_optimizer.check_zbuf_body = check_zbuf_body`.  Returns [N,Q]: the bilinear sample, at the caller's screen
    points normalised by img_size [N,2] = (w, h), of the skinned body's zbuf with background filled by the raw maximum
    vertex z.  Sets `mask_render.rasterizer.cameras = cameras` as the reference does.  No host read; detached."""
    mask_render.rasterizer.cameras = cameras
    _, size, z_clip, area_eps = _probe_settings(mask_render)
    with torch.no_grad():
        verts = deform_lbs(smpl_mesh.verts_packed()[None].expand(N, -1, 3), [poses, trans])
        fill = verts[..., -1].max(-1)[0]
        return _raster.zbuf_probe(verts, smpl_mesh.faces_packed(), cameras, size, screen_pts, img_size, fill, z_clip,
                                  area_eps)


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
