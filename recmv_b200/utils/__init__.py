"""Mirror of the hot-path helpers of the reference's `utils` package (utils/utils.py:8-18,40-46,133-156,
198-264).  Same names, arguments and return values; the native calls go to librecmv_b200.so."""
import sys

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


def make_sample_train_ray():
    """`OptimGarmentNetwork.sample_train_ray` (OptimGarmentNetwork.py:983-1055) with the selection on the GPU; bind it
    as `OptimGarmentNetwork.sample_train_ray = make_sample_train_ray()` (the Large-Pose class inherits it).
    As the reference: `sample_pix_num` from `self.conf` when present, // `self.garment_size`; per garment the rows whose
    ground-truth mask is > 0 and, when more than T = sample_pix * N of them remain, a Bernoulli draw at fp32(T / pnum);
    a `RectifiedPerspectiveCameras` (looked up in the bound class's module) from `self.dataset.get_camera_parameters`,
    assigned to `self.maskRender.rasterizer.cameras` and to `self.pcRender.rasterizer.cameras` when `pcRender` is set;
    returns (batch, row, col, init points, rays) lists and the cameras.  Unlike the reference, all garments go through
    one launch sequence (csrc/train_rays.cu) with one host read, the G kept counts, and the uniforms come from a
    Philox4x32-10 stream whose seed is drawn from torch's CPU generator at the first call and whose offset advances by
    the garments' input rows per call; both are in the returned function's `stream` dict.  When the camera's
    focal_length, principal_point or R requires grad, the rays are the camera's own `view_rays` of the kept (col, row),
    so the graph is the reference's; otherwise they come from the kernel.  The init points are returned detached (the
    fragment decode that produces them has no graph)."""
    stream = {"seed": None, "offset": 0}

    def sample_train_ray(self, N, sample_pix, gt_garment_masks_list, batch_garment_inds_list, batch_garment_row_list,
                         batch_garment_col_list, batch_garment_init_pts_list, frame_ids, device):
        sample_pix = self.conf.get_int('sample_pix_num') if 'sample_pix_num' in self.conf else sample_pix
        sample_pix = sample_pix // self.garment_size
        for t in list(gt_garment_masks_list) + list(batch_garment_inds_list):
            if not t.is_cuda:
                raise RuntimeError("sample_train_ray runs on CUDA tensors only (no CPU path)")
        focals, princeple_ps, Rs, Ts, H, W = self.dataset.get_camera_parameters(frame_ids.numel(), device)
        cameras_cls = sys.modules[type(self).__module__].RectifiedPerspectiveCameras
        cameras = cameras_cls(focals, princeple_ps, Rs, Ts, image_size=[(W, H)]).to(device)
        self.maskRender.rasterizer.cameras = cameras
        if self.pcRender:
            self.pcRender.rasterizer.cameras = cameras
        if stream["seed"] is None:
            stream["seed"] = int(torch.empty((), dtype=torch.int64).random_())
        masks = [m.float().contiguous() for m in gt_garment_masks_list]
        cam = _raster.camera_rows(cameras, int(cameras.R.reshape(-1, 9).shape[0]), device)[0].detach()
        kept = _ops.train_rays_sample([b.long().contiguous() for b in batch_garment_inds_list],
                                      [r.long().contiguous() for r in batch_garment_row_list],
                                      [c.long().contiguous() for c in batch_garment_col_list],
                                      [p.detach().float().contiguous() for p in batch_garment_init_pts_list], masks,
                                      cam, sample_pix * N, stream["seed"], stream["offset"])
        stream["offset"] += sum(int(b.shape[0]) for b in batch_garment_inds_list)
        out = [list(x) for x in zip(*kept)] if kept else [[] for _ in range(5)]
        if any(t.requires_grad for t in (cameras.focal_length, cameras.principal_point, cameras.R)):
            out[4] = [cameras.view_rays(torch.cat([c.view(-1, 1), r.view(-1, 1), torch.ones_like(c.view(-1, 1))],
                                                  dim=-1).float()) for r, c in zip(out[1], out[2])]
        return out[0], out[1], out[2], out[3], out[4], cameras

    sample_train_ray.stream = stream
    return sample_train_ray


def make_surface_render_loss():
    """`OptimGarmentNetwork.surface_render_loss` (OptimGarmentNetwork.py:1083-1219) with its sampling, compaction and
    per-frame means on the GPU; bind it as `OptimGarmentNetwork.surface_render_loss = make_surface_render_loss()` (the
    Large-Pose class inherits it).  As the reference: the conf lookups and weights, the branch order, per garment the
    eikonal term on cat(init points, vertices kept at rate 4096 // G / V) plus local and global samples, the info-only
    translator forward when `offset_weight` is 0, the regulariser on cat(init points, an independent draw of vertices)
    and their local samples expanded over the N frames, and, when `info['<name>_rayInfo'][1] > 0`, the colour and
    normal terms on the checked rows; `self.TmpPs` (fresh leaves with requires_grad), `self.rays`, `self.batch_inds`,
    `self.row_inds` and `self.col_inds` are set as the reference sets them, for `propagateTmpPsGrad`.
    Unlike the reference: all garments are sampled and compacted in one launch sequence (ops.loss_points_sample,
    csrc/loss_points.cu) with the call's one host read; the draws come from a Philox4x32-10 stream whose seed is drawn
    from torch's CPU generator at the first call and whose offset advances by 5 (M_g + V_g) summed over the garments
    (both in the returned function's `stream` dict); the frame means are ops.ColorFrameMeanFunction and
    ops.NormalFrameMeanFunction, so torch_scatter is not needed; the singular-Jacobian fallbacks are selected with
    `torch.where`, without the reference's host test and print; the info values are detached 0-d tensors (the colour
    default stays -1.0).  `offset_weight > 0` raises NotImplementedError; CPU tensors raise."""
    stream = {"seed": None, "offset": 0}

    def surface_render_loss(self, datas, N, cameras, frame_ids, ratio, check_list, gtCs, init_garment_ps_list,
                            sample_batch_garment_row_list, sample_batch_garment_col_list,
                            sample_batch_garment_inds_list, sample_rays_list, device):
        G = self.garment_size
        self.TmpPs = [None for _ in range(G)]
        self.rays = [None for _ in range(G)]
        self.batch_inds = [None for _ in range(G)]
        self.row_inds = [None for _ in range(G)]
        self.col_inds = [None for _ in range(G)]
        conf = self.conf
        if 'offset_weight' in conf and conf.get_float('offset_weight') > 0.:
            raise NotImplementedError("surface_render_loss: offset_weight > 0 is not supported")
        total_loss = 0.
        d_cond_list, poses, trans, rendcond = self.get_grad_parameters(frame_ids, device)
        inputs = (list(init_garment_ps_list), [self.garment_vs[g] for g in range(len(init_garment_ps_list))],
                  list(check_list), list(sample_batch_garment_inds_list), list(sample_batch_garment_row_list),
                  list(sample_batch_garment_col_list), list(sample_rays_list))
        for t in [t for ts in inputs for t in ts] + [gtCs]:
            if not t.is_cuda:
                raise RuntimeError("surface_render_loss runs on CUDA tensors only (no CPU path)")
        if stream["seed"] is None:
            stream["seed"] = int(torch.empty((), dtype=torch.int64).random_())
        P, V, chk, bi, ri, ci, rays_in = inputs
        samples = _ops.loss_points_sample([p.detach().float().contiguous() for p in P],
                                          [v.detach().float().contiguous() for v in V],
                                          [c.bool().contiguous() for c in chk], [b.long().contiguous() for b in bi],
                                          [r.long().contiguous() for r in ri], [c.long().contiguous() for c in ci],
                                          [r.detach().float().contiguous() for r in rays_in], 4096 // G,
                                          stream["seed"], stream["offset"])
        stream["offset"] += 5 * sum(int(p.shape[0]) + int(v.shape[0]) for p, v in zip(P, V))
        for garment_idx, (X_E, X_D, ps, rays_c, batch_c, row_c, col_c, index) in enumerate(samples):
            garment_name = self.garment_names[garment_idx]
            net = self.garment_nets[garment_idx]
            nonmnfld_pnts = X_E.requires_grad_()
            nonmnfld_grad = net.gradient(nonmnfld_pnts, net(nonmnfld_pnts, ratio))
            grad_loss = ((nonmnfld_grad.norm(2, dim=-1) - 1) ** 2).mean()
            self.info['{}_grad_loss'.format(garment_name)] = grad_loss.detach()
            total_loss += grad_loss * conf.get_float('grad_weight')

            d_cond = d_cond_list[garment_idx + 1]
            if 'offset_weight' in conf and conf.get_float('offset_weight') == 0.:
                with torch.no_grad():
                    self.deformer.defs[0](nonmnfld_pnts.view(1, -1, 3).expand(N, -1, 3), d_cond, ratio=ratio,
                                          offset_type=garment_name)
                    def_offloss = self.deformer.defs[0].offset[garment_name].view(-1, 3).norm(p=2, dim=-1).mean()
                    self.info['{}_offset_loss'.format(garment_name)] = def_offloss.detach()
            nonmnfld_pnts = None
            if 'def_regu' in conf and conf.get_float('def_regu.weight') > 0.:
                def_loss = deformation_regulariser(self.deformer.defs[0], X_D.view(1, -1, 3).expand(N, -1, 3), d_cond,
                                                   ratio, conf.get_float('def_regu.c'), offset_type=garment_name)
                self.info['def_{}_loss'.format(garment_name)] = def_loss.detach()
                total_loss += def_loss * conf.get_float('def_regu.weight')

            self.info['{}_color_loss'.format(garment_name)] = -1.0
            if self.info['{}_rayInfo'.format(garment_name)][1] > 0:
                TmpPs = ps
                TmpPs.requires_grad = True
                self.TmpPs[garment_idx] = TmpPs
                rays = sample_rays_list[garment_idx]
                self.rays[garment_idx] = rays.index_select(0, index) if rays.requires_grad else rays_c
                self.batch_inds[garment_idx] = batch_c
                self.col_inds[garment_idx] = col_c
                self.row_inds[garment_idx] = row_c
                sdfs = net(TmpPs, ratio)
                nx = torch.autograd.grad(sdfs, TmpPs, torch.ones_like(sdfs), retain_graph=True, create_graph=True)[0]
                nx = nx / nx.norm(dim=1, keepdim=True)
                defconds = [d_cond, [poses, trans]]
                crays, defVs = _cardinal_rays_where(self.deformer, TmpPs, self.rays[garment_idx], defconds, batch_c,
                                                    ratio, 'train', offset_type=garment_name)
                if conf.get_float('color_weight') > 0.:
                    colors = compute_netRender_color(self.netRender, TmpPs, defVs, nx, crays, net.rendcond,
                                                     rendcond[batch_c], ratio)
                    color_loss = _ops.ColorFrameMeanFunction.apply(colors, gtCs.float(), batch_c, row_c, col_c, N)
                    self.info['{}_color_loss'.format(garment_name)] = color_loss.detach()
                    total_loss += conf.get_float('color_weight') * color_loss
                if 'normal' in datas and 'normal_weight' in conf and conf.get_float('normal_weight') > 0.:
                    if 'weighted_normal' in conf and conf.get_bool('weighted_normal'):
                        cnx, _ = _deformed_normals_where(net, self.deformer, TmpPs, defconds, batch_c, ratio, 'test',
                                                         garment_name)
                        weights = torch.clamp((-self.rays[garment_idx] * cnx.detach()).sum(1).detach(), max=1.,
                                              min=0.) ** 2
                    else:
                        weights = torch.ones(nx.shape[0], device=device)
                    gtnormals = datas['normal'].to(device)[batch_c, row_c, col_c, :]
                    R0 = cameras.R[0]     # R[0] @ diag(-1, 1, -1), built without a host-to-device copy
                    flipped = torch.stack([-R0[:, 0], R0[:, 1], -R0[:, 2]], 1)
                    gtnormals = (flipped @ gtnormals.view(-1, 3, 1)).view(-1, 3)
                    ds = self.deformer(TmpPs, defconds, batch_c, ratio=ratio, offset_type=garment_name)
                    grad_d_p = compute_Jacobian(TmpPs, ds, True, True)
                    normal_loss = _ops.NormalFrameMeanFunction.apply(gtnormals.float(), grad_d_p.float(), nx.float(),
                                                                     weights.detach().float(), batch_c, N)
                    self.info['{}_normal_loss'.format(garment_name)] = normal_loss.detach()
                    total_loss += conf.get_float('normal_weight') * normal_loss
        return total_loss

    surface_render_loss.stream = stream
    return surface_render_loss


class Meshes:
    """pytorch3d's `Meshes(verts=[...], faces=[...])` for what `mask_loss`'s results feed: `verts_list`, `faces_list`,
    `verts_padded` (meshes of equal size), and `verts_packed` / `faces_packed` (faces offset by the preceding meshes'
    vertex counts, as pytorch3d packs them)."""

    def __init__(self, verts, faces):
        self._v, self._f = list(verts), list(faces)

    def __len__(self):
        return len(self._v)

    def verts_list(self):
        return self._v

    def faces_list(self):
        return self._f

    def verts_padded(self):
        return torch.stack(self._v)

    def verts_packed(self):
        return torch.cat(self._v)

    def faces_packed(self):
        base, out = 0, []
        for v, f in zip(self._v, self._f):
            out.append(f + base)
            base += int(v.shape[0])
        return torch.cat(out)


class _Cloud:
    """The point clouds `pcRender` reads: padded points [N,P,3] and one scalar feature per point."""

    def __init__(self, points, features):
        self._p, self._f = points, features

    def points_padded(self):
        return self._p

    def features_packed(self):
        return self._f


def make_mask_loss():
    """`OptimGarmentNetwork.mask_loss(self, N, H, W, frame_ids, ratio, gt_garment_masks_list, device)`
    (OptimGarmentNetwork.py:621-667, 841-981) with the ground-truth dilation and the soft IoU on the GPU; bind it as
    `OptimGarmentNetwork.mask_loss = make_mask_loss()` (the Large-Pose class inherits it).
    As the reference: per garment the N-expanded deformer call with its offset type and a `Meshes` of the deformed
    copies; `find_surface_ps` through `self.maskRender`; one `self.pcRender` call on the concatenated garment cloud
    with `split_size` and `all_size`; the radius int(round(radius / 2 min(H, W) / 1.2)) of the renderer's NDC radius;
    per garment the mask loss times `pc_weight.mask_weight` (1 without it) and, with `pc_weight.def_consistent`, the
    template-consistency term against `self.deformer.defs[1]` (GM robust error when `c` > 0, else the mean distance);
    `garment_optimizer` zero_grad / backward / step, so the backward also reaches the deformer, the conditions, the
    poses, the translations and any learnable camera; then mean |f + sdfShrinkRadius| per garment times
    `pc_weight.weight` (60 without `pc_weight`) plus `self.curve_aware_loss(ratio)`.  Returns
    (def_garment_meshes, garment_masks_list, mgt_garment_masks_list, pc_sdf_loss, surface_ps_list).
    Unlike the reference: the dilation and the IoU of all garments are one ops.MaskIouFunction (csrc/mask_iou.cu);
    the info values are detached 0-d tensors; nothing is read back to the host beyond the renderers' own reads.  A
    positive `pc_weight.laplacian_weight`, `edge_weight` or `norm_weight` raises NotImplementedError (the reference's
    branches read an undefined template mesh), as do more than two garments and a radius that rounds to 0 pixels
    (where the reference's `raise NotImplemented` fails); CPU tensors raise."""

    def mask_loss(self, N, H, W, frame_ids, ratio, gt_garment_masks_list, device):
        conf = self.conf
        for key in ('laplacian_weight', 'edge_weight', 'norm_weight'):
            if (conf.get_float('pc_weight.' + key) if 'pc_weight' in conf else -1.) > 0.:
                raise NotImplementedError(f"mask_loss: pc_weight.{key} > 0 is not supported")
        G = self.garment_size
        if G > 2:
            raise NotImplementedError('only support less or equal than 2 garment_type')
        for t in list(gt_garment_masks_list) + list(self.garment_vs):
            if not t.is_cuda:
                raise RuntimeError("mask_loss runs on CUDA tensors only (no CPU path)")
        d_cond_list, poses, trans, rendcond = self.get_grad_parameters(frame_ids, device)
        def_garment_vs = [self.deformer(self.garment_vs[g][None, :, :].expand(N, -1, 3),
                                        [d_cond_list[g + 1], [poses, trans]], ratio=ratio, offset_type=name)
                          for g, name in zip(range(G), self.garment_names)]
        def_garment_meshes = [Meshes(verts=[vs.view(int(v.shape[0]), 3) for vs in torch.split(dv, 1)],
                                     faces=[fs for _ in range(N)])
                              for v, fs, dv in zip(self.garment_vs, self.garment_fs, def_garment_vs)]
        self.info['pc_loss'] = {}
        surface_ps_list = self.find_surface_ps(def_garment_meshes)
        points = torch.cat(def_garment_vs, 1)
        P = int(points.shape[1])
        features = torch.ones((N * P, 1), device=points.device)
        garment_masks_list, _ = self.pcRender(_Cloud(points, features), split_size=int(self.garment_vs[0].shape[0]),
                                              all_size=P)
        radius = self.pcRender.rasterizer.raster_settings.radius
        radius = int(round(radius / 2. * float(min(H, W)) / 1.2))
        if radius <= 0:
            raise NotImplementedError("mask_loss: the point radius rounds to 0 pixels")
        out = _ops.MaskIouFunction.apply(radius, *[m[..., -1] for m in garment_masks_list[:G]],
                                         *gt_garment_masks_list[:G])
        mask_losses, mgt_garment_masks_list = out[0], list(out[1:])
        mask_weight = conf.get_float('pc_weight.mask_weight') if 'pc_weight.mask_weight' in conf else 1.
        consistent_weight = (conf.get_float('pc_weight.def_consistent.weight') if 'pc_weight.def_consistent' in conf
                             else -1.)
        garment_loss = 0.
        for g, name in enumerate(self.garment_names[:G]):
            self.info['pc_loss']['{}_mask_loss'.format(name)] = mask_losses[g].detach()
            loss = mask_losses[g] * mask_weight
            if consistent_weight > 0.:
                offset2 = def_garment_vs[g] - self.deformer.defs[1](self.garment_vs[g].view(1, -1, 3).expand(N, -1, 3),
                                                                    [poses, trans])
                offset2 = (offset2 * offset2).sum(-1)
                c = conf.get_float('pc_weight.def_consistent.c')
                consistent_loss = GMRobustError(offset2, c, True).mean() if c > 0. else torch.sqrt(offset2).mean()
                self.info['pc_loss']['garment_{}_defconst_loss'.format(name)] = consistent_loss.detach()
                loss = loss + consistent_loss * consistent_weight
            garment_loss += loss
        self.garment_optimizer.zero_grad()
        garment_loss.backward()
        self.garment_optimizer.step()

        pc_sdf_loss = 0.
        weight = conf.get_float('pc_weight.weight') if 'pc_weight' in conf else 60.
        for g, (garment_vs, name) in enumerate(zip(self.garment_vs, self.garment_names)):
            mnfld_pred = self.garment_nets[g](garment_vs, ratio).view(-1)
            sdf_loss = (mnfld_pred + self.sdfShrinkRadius).abs().mean()
            self.info['pc_{}_loss_sdf'.format(name)] = sdf_loss.detach()
            pc_sdf_loss += sdf_loss * weight
        pc_sdf_loss += self.curve_aware_loss(ratio)
        return def_garment_meshes, garment_masks_list, mgt_garment_masks_list, pc_sdf_loss, surface_ps_list

    return mask_loss


def _repeat_rows(t, G):
    return t.repeat(G, *([1] * (t.dim() - 1)))


def make_propagate_tmp_ps_grad():
    """`propagateTmpPsGrad(self, frame_ids, ratio)` of OptimGarmentNetwork (OptimGarmentNetwork.py:2159-2313) and of
    OptimGarmentNetwork_LargePose (OptimGarmentNetwork_Large_Pose.py:327-473, which drops the SDF term) with the
    implicit-surface algebra on the GPU; bind the returned function on both classes, as the Large-Pose class overrides
    the method.  As the reference: the garments before the first one whose `TmpPs` or `TmpPs.grad` is missing are
    processed and that one gets `info['<name>_invInfo'] = (-1, -1)` (the reference returns there); the cameras are
    rebuilt from `self.dataset.get_camera_parameters` with the bound class's module's `RectifiedPerspectiveCameras` and
    assigned to `self.maskRender.rasterizer.cameras`; v is the camera's `view_rays` of (col, row, 1) when
    `self.rays[g]` requires grad, else `self.rays[g]` detached, c = `cam_pos()`; b = [grad f ; [v]x J] and
    r = TmpPs.grad (b^T b)^-1 b^T with FastMinv's rule; -r0 goes back through the garment's SDF (when it has a
    parameter that requires grad), r[1:4] (-[v]x) through the deformer to its parameters, the garment conditions, the
    poses and the translations, r[1:4] [d - c]x to v when v requires grad and the sum of -r[1:4] (-[v]x) to c when c
    requires grad; gradients accumulate into `.grad`; `deformer.defs[0].offset[<name>]` holds the garment's rows.
    Unlike the reference: grad f comes from each garment net's `value_and_grad`, d and J of all garments from ONE
    forward-mode deformer launch (conditions stacked [G N, 128], poses and translations repeated G times, row frame
    g N + b), the algebra and the per-garment reductions from ONE kernel (ops.implicit_surface_grad), and all VJPs from
    ONE `torch.autograd.backward` (one training forward of the deformer over all rows) instead of the surrogate-loss
    chain: the sums are the same, the floating-point accumulation order differs.  `info['<name>_invInfo']` is
    (rows, ok count) with the count a detached 0-d device tensor; the fixed-camera branch reads `self.rays[g]` (the
    reference's `self.rays.detach()` calls .detach() on the list).  `TmpPs.grad` is left untouched.  No host
    synchronisation; CPU tensors raise."""

    def propagateTmpPsGrad(self, frame_ids, ratio):
        names = self.garment_names
        active = 0
        while active < self.garment_size and self.TmpPs[active] is not None and self.TmpPs[active].grad is not None:
            active += 1
        missing = active < self.garment_size
        if active > 0:
            _propagate(self, frame_ids, ratio, active)
        if missing:
            self.info['{}_invInfo'.format(names[active])] = (-1, -1)

    return propagateTmpPsGrad


def _propagate(self, frame_ids, ratio, G):
    """propagateTmpPsGrad for garments 0 .. G-1, all of which have TmpPs and TmpPs.grad."""
    names = self.garment_names
    ps = [self.TmpPs[g].detach() for g in range(G)]
    device = ps[0].device
    for t in ps + [self.TmpPs[g].grad for g in range(G)] + [self.batch_inds[g] for g in range(G)]:
        if not t.is_cuda:
            raise RuntimeError("propagateTmpPsGrad runs on CUDA tensors only (no CPU path)")
    d_cond_list, poses, trans, _ = self.get_grad_parameters(frame_ids, device)
    focals, princeple_ps, Rs, Ts, H, W = self.dataset.get_camera_parameters(frame_ids.numel(), device)
    cameras_cls = sys.modules[type(self).__module__].RectifiedPerspectiveCameras
    cameras = cameras_cls(focals, princeple_ps, Rs, Ts, image_size=[(W, H)]).to(device)
    self.maskRender.rasterizer.cameras = cameras
    vs = []
    for g in range(G):
        if self.rays[g].requires_grad:
            col, row = self.col_inds[g].view(-1, 1), self.row_inds[g].view(-1, 1)
            vs.append(cameras.view_rays(torch.cat([col, row, torch.ones_like(col)], dim=-1).float()))
        else:
            vs.append(self.rays[g].detach())
    c = cameras.cam_pos()
    offsets = [0]
    for p in ps:
        offsets.append(offsets[-1] + int(p.shape[0]))
    P = torch.cat(ps).float().contiguous()
    gf = torch.cat([self.garment_nets[g].value_and_grad(ps[g], ratio)[1].reshape(-1, 3) for g in range(G)])
    # one deformer over all garments: frame g N + b reads garment g's condition row b and pose / translation b
    N = int(poses.shape[0])
    conds = torch.cat([d_cond_list[1 + g] for g in range(G)])
    defconds = [conds, [_repeat_rows(poses, G), _repeat_rows(trans, G)]]
    binds = torch.cat([self.batch_inds[g].long() + g * N for g in range(G)])
    fixed = [conds.detach(), [t.detach() for t in defconds[1]]]
    d, J = _value_and_jacobian(self.deformer, P.requires_grad_(), fixed, binds, ratio, names[0], False)
    P = P.detach()
    want_ray_grad = any(v.requires_grad for v in vs)
    coef, vec, ray_grad, _, ok_count, cam_grad = _ops.implicit_surface_grad(
        torch.cat([self.TmpPs[g].grad for g in range(G)]).float().contiguous(), gf.float().contiguous(),
        J.detach().float().contiguous(), torch.cat([v.detach() for v in vs]).float().contiguous(),
        d.detach().float().contiguous(), offsets, c.detach().float().reshape(3).contiguous(), want_ray_grad)
    outs, cots = [], []
    for g in range(G):
        net = self.garment_nets[g]
        if any(p.requires_grad for p in net.parameters()):
            f = net(ps[g], ratio)
            outs.append(f)
            cots.append(coef[offsets[g]:offsets[g + 1]].view_as(f).to(f.dtype))
    dtrain = self.deformer(P, defconds, binds, ratio=ratio, offset_type=names[0])
    if dtrain.requires_grad:
        outs.append(dtrain)
        cots.append(vec.to(dtrain.dtype))
    for g, v in enumerate(vs):
        if v.requires_grad:
            outs.append(v)
            cots.append(ray_grad[offsets[g]:offsets[g + 1]].to(v.dtype))
    if c.requires_grad:
        outs.append(c)
        cots.append(cam_grad.sum(0).view_as(c).to(c.dtype))
    if outs:
        torch.autograd.backward(outs, cots)
    tr = self.deformer.defs[0]
    off = getattr(tr, 'offset', {}).get(names[0])
    if off is not None and off.shape[0] == offsets[-1]:
        off = off.detach()
        for g in range(G):
            tr.offset[names[g]] = off[offsets[g]:offsets[g + 1]]
    for g in range(G):
        self.info['{}_invInfo'.format(names[g])] = (offsets[g + 1] - offsets[g], ok_count[g])


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


def _cardinal_rays(deformer, ps, rays, defconds, batch_inds, ratio, phase, offset_type):
    """(J^-1 v, FastMinv's ok flags, D(p)): the formula compute_cardinal_rays shares with the drop-ins."""
    check = phase in ('train', 'Train')
    ds, J = _value_and_jacobian(deformer, ps, defconds, batch_inds, ratio, offset_type, check)
    Jinv, ok = FastDiff3x3MinvFunction.apply(J)
    return Jinv.matmul(rays.view(-1, 3, 1)).view(-1, 3), ok, ds


def _cardinal_rays_where(deformer, ps, rays, defconds, batch_inds, ratio, phase, offset_type=None):
    """compute_cardinal_rays with the singular rows' fallback (the view ray) selected on the device: no host read."""
    crays, ok, ds = _cardinal_rays(deformer, ps, rays, defconds, batch_inds, ratio, phase, offset_type)
    crays = torch.where(ok[:, None], crays, rays.detach())
    return crays / crays.norm(dim=1, keepdim=True), ds


def compute_cardinal_rays(deformer, ps, rays, defconds, batch_inds, ratio, phase, offset_type=None):
    """crays = normalize(J^-1 v) with the FastMinv singularity fallback (utils/utils.py:232-250)."""
    crays, ok, ds = _cardinal_rays(deformer, ps, rays, defconds, batch_inds, ratio, phase, offset_type)
    bad = ~ok
    if bad.sum().item() > 0:
        print('unwished error n_inv_mask:(%d:%d)' % (bad.sum().item(), bad.numel()))
        fixed = torch.zeros_like(crays)
        fixed[ok] = crays[ok]
        fixed[bad] = rays[bad].detach()
        crays = fixed
    crays = crays / crays.norm(dim=1, keepdim=True)
    return crays, ds


def _deformed_normals(sdf, deformer, ps, defconds, batch_inds, ratio, phase, offset_type):
    """(J^-T grad sdf, FastMinv's ok flags, J, grad sdf, D(p)): the formula compute_deformed_normals shares with the
    drop-ins."""
    sdfs = sdf(ps, ratio)
    check = phase in ('train', 'Train')
    with _ops.input_grad_only():
        onx = torch.autograd.grad(sdfs, ps, torch.ones_like(sdfs), retain_graph=check, create_graph=check)[0]
    ds, J = _value_and_jacobian(deformer, ps, defconds, batch_inds, ratio, offset_type, check)
    Jinv, ok = FastDiff3x3MinvFunction.apply(J)
    return Jinv.transpose(-2, -1).matmul(onx.view(-1, 3, 1)).view(-1, 3), ok, J, onx, ds


def _deformed_normals_where(sdf, deformer, ps, defconds, batch_inds, ratio, phase, offset_type):
    """compute_deformed_normals with the singular rows' fallback (J grad sdf) selected on the device: no host read."""
    nx, ok, J, onx, ds = _deformed_normals(sdf, deformer, ps, defconds, batch_inds, ratio, phase, offset_type)
    nx = torch.where(ok[:, None], nx, J.matmul(onx.unsqueeze(-1)).view(-1, 3))
    return nx / nx.norm(dim=1, keepdim=True), ds


def compute_deformed_normals(sdf, deformer, ps, defconds, batch_inds, ratio, phase, offset_type):
    """n = normalize(J^-T grad sdf) (utils/utils.py:198-230)."""
    nx, ok, J, onx, ds = _deformed_normals(sdf, deformer, ps, defconds, batch_inds, ratio, phase, offset_type)
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
