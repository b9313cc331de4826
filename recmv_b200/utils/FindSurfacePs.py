"""Surface-point seeding and the Newton-like surface/ray root solve -- API of utils/FindSurfacePs.py
(:7-60 FindSurfacePs, :145-207 OptimizeSurfacePs, :210-272 OptimizeGarmentSurfaceSinlge, :273-353
OptimizeGarmentSurfacePs).

The three Optimize* functions of the reference are one algorithm copied three times; here they share
`_solve`.  Per iteration on the not-yet-converged subset:
    L = w1 |f(p)| + w2 |(D(p)-c) x v| / |D(p)-c| ,  g = dL/dp ,  p <- p - L g / |g|^2
converged when |f| < dthreshold and asin(|(D-c) x v| / |D-c|) * 180/pi < athreshold.
All no-grad evaluations (the convergence checks) run the fused kernels (one launch for the SDF, one for
the skinning); the gradient step goes through the autograd path of the same modules.
"""
import numpy as np
import torch


def FindSurfacePs(TmpVs, TmpFaces, frags):
    """Rasteriser fragments -> (batch, row, col) of covered pixels, barycentric seed points on the canonical
    mesh and the face ids (utils/FindSurfacePs.py:7-60).  frags: .pix_to_face [N,H,W,K] i64,
    .bary_coords [N,H,W,K,3]."""
    pix_to_face = frags.pix_to_face
    bary = frags.bary_coords
    if pix_to_face.is_cuda and bary.dtype == torch.float32 and not TmpVs.requires_grad:
        from .. import ops      # one ordered compaction on the device (csrc/fragments.cu)
        return ops.fragment_decode(pix_to_face, bary, TmpVs, TmpFaces)
    N, H, W, K = pix_to_face.shape
    inner = (bary > 0.0).all(-1) & (pix_to_face >= 0)                # [N,H,W,K]
    # first valid k per pixel (the reference takes a scatter-min over the nonzero columns, :26-30)
    first = torch.where(inner, torch.arange(K, device=inner.device).view(1, 1, 1, K),
                        torch.full((1, 1, 1, 1), K, device=inner.device)).min(dim=-1).values
    covered = inner.any(dim=-1)
    batch_inds, row_inds, col_inds = covered.nonzero(as_tuple=True)
    k = first[covered].view(-1, 1)
    finds = torch.gather(pix_to_face[covered], 1, k).view(-1)
    finds = finds % TmpFaces.shape[0]                                # packed -> per-mesh face index
    ws = torch.gather(bary[covered], 1, k.view(-1, 1, 1).expand(-1, 1, 3)).view(-1, 3)
    initTmpPs = (TmpVs[TmpFaces[finds].view(-1)].view(-1, 3, 3) * ws[:, :, None]).sum(1)
    return batch_inds, row_inds, col_inds, initTmpPs, finds


def FindSurfacePsRays(TmpVs, TmpFaces, frags, camera, gt_masks=None):
    """FindSurfacePs + the ground-truth mask selection and the per-pixel view rays of sample_train_ray
    (OptimGarmentNetwork.py:1006-1011, 1046-1050; CameraMine.view_rays :146-167) in one device pass.
    camera = (fx, fy, px, py, R) host values of the (shared) RectifiedPerspectiveCameras entry.
    Returns (batch, row, col, init points, face ids, rays)."""
    from .. import ops
    return ops.fragment_decode(frags.pix_to_face, frags.bary_coords, TmpVs, TmpFaces, gt_masks, camera)


def FindSurfacePsMesh(TmpVs, TmpFaces, defVs, cameras, H, W, gt_masks=None):
    """Rasterize the deformed meshes defVs [N,V,3] (faces TmpFaces, one camera per frame, recmv_b200.raster) and decode
    the fragments against the canonical mesh TmpVs with camera 0's view rays and the mask filter (FindSurfacePsRays):
    what `find_surface_ps` + `sample_train_ray` compute with `maskRender` (OptimGarmentNetwork.py:742-783, 1006-1050).
    cameras: reference-camera attributes or (focal_length, principal_point, R, T).  Host reads: the rasterizer's counters
    (which carry camera 0 to the host) and the decode's row count.  Returns (batch, row, col, init points, face ids,
    rays)."""
    from .. import ops
    from ..raster import camera_rows
    if not defVs.is_cuda:
        raise RuntimeError("FindSurfacePsMesh runs on CUDA tensors only (no CPU path)")
    cam = camera_rows(cameras, int(defVs.shape[0]), defVs.device)
    p2f, _, bary, _, counts = ops.rasterize_meshes(defVs.detach().float().contiguous(), TmpFaces.long().contiguous(), cam,
                                                   H, W, want_dists=False, host_camera=True)
    c = counts["camera"]
    return ops.fragment_decode(p2f, bary, TmpVs, TmpFaces, gt_masks, (c[0], c[1], c[2], c[3], c[4:13].view(3, 3)))


# The three Optimize* entry points run the whole loop on the device (one C call) when both networks are on the
# tensor-core engine; set False to force the step-by-step torch loop (`_solve`, which also serves CPU tensors, the
# fp32 SIMT mode and deformers other than [MLPTranslator, LBSkinner]).
DEVICE_SOLVE = True


def _angle_ok(direct, rays, athreshold):
    up = torch.cross(direct, rays, dim=1)
    return torch.arcsin(up.norm(dim=1) / direct.norm(dim=1)) * 180. / np.pi < athreshold


def _solve(cam_pos, rays, initTmpPs, batch_inds, tmpSdf, ratio, deform, dthreshold, athreshold, w1, w2,
           times, deform_jac=None):
    """deform(ps, inds) -> posed points; deform_jac(ps, inds) -> (posed, J [P,3,3]) or None (fused forward-mode
    launch).  Mutates and returns initTmpPs like the reference."""
    cam = cam_pos.view(1, 3)
    with torch.no_grad():
        check = (tmpSdf(initTmpPs, ratio).view(-1).abs() < dthreshold) & \
            _angle_ok(deform(initTmpPs, batch_inds) - cam, rays, athreshold)
        unfinished = ~check
    for _ in range(times):
        sel = unfinished.nonzero(as_tuple=False).view(-1)   # one sync per iteration (reference: several)
        if sel.numel() == 0:
            break
        cur = initTmpPs[sel].detach().clone().requires_grad_(True)
        fused = getattr(tmpSdf, "value_and_grad", None) is not None
        if fused:
            # |f| term analytically from the fused forward-mode launch: d|f|/dp = sign(f) grad f
            f, gf = tmpSdf.value_and_grad(cur.detach(), ratio)
            loss1 = f.abs().view(-1)
        else:
            loss1 = tmpSdf(cur, ratio).abs().view(-1)
        dj = deform_jac(cur.detach(), batch_inds[sel]) if (fused and deform_jac is not None) else None
        if dj is not None:
            # no autograd through the deformer: loss2 depends on p only through D(p), so grad_p = J^T dloss2/dD
            direct = (dj[0] - cam).detach().requires_grad_(True)
        else:
            direct = deform(cur, batch_inds[sel]) - cam
        up = torch.cross(direct, rays[sel], dim=1)
        loss2 = (up.norm(dim=1) / direct.norm(dim=1)).abs()
        loss = w1 * loss1 + w2 * loss2
        if dj is not None:
            gd = torch.autograd.grad((w2 * loss2).sum(), direct)[0]
            grad = torch.bmm(dj[1].transpose(1, 2), gd.unsqueeze(-1)).squeeze(-1) + w1 * torch.sign(f) * gf
            loss = loss.detach()
        elif fused:
            grad = torch.autograd.grad((w2 * loss2).sum(), cur, retain_graph=False, create_graph=False)[0]
            grad = grad + w1 * torch.sign(f) * gf
            loss = loss.detach()
        else:
            grad = torch.autograd.grad(loss.sum(), cur, retain_graph=False, create_graph=False, only_inputs=True)[0]
        t = -loss / (grad * grad).sum(1)
        cur = (cur + t.view(-1, 1) * grad).detach()
        initTmpPs[sel] = cur
        with torch.no_grad():
            ok = (tmpSdf(cur, ratio).view(-1).abs() < dthreshold) & \
                _angle_ok(deform(cur, batch_inds[sel]) - cam, rays[sel], athreshold)
            unfinished[sel[ok]] = False
    return initTmpPs.detach(), ~unfinished


def _solve_device(cam_pos, rays, initTmpPs, batch_inds, tmpSdf, ratio, deformer, defconds, dthreshold, athreshold,
                  w1, w2, times):
    """The whole active-set loop as ONE C call (recmv_surface_solve: times + 1 rounds of two forward-mode launches +
    an update kernel, no host synchronisation) when both networks run on the tensor-core engine; None otherwise."""
    from .. import ops
    if not (initTmpPs.is_cuda and getattr(tmpSdf, "_fusable", False) and hasattr(deformer, "device_solve_args")):
        return None
    if tmpSdf.mlp_mode == ops.MLP_FP32_SIMT:
        return None
    args = deformer.device_solve_args(defconds, ratio)
    if args is None or (args[4] or ops.DEFAULT_MLP_MODE) != (tmpSdf.mlp_mode or ops.DEFAULT_MLP_MODE):
        return None
    tr_packed, tr_pe, conds, skin, mode = args
    sdf_ratio = ratio.get('sdfRatio') if isinstance(ratio, dict) else ratio
    with torch.no_grad():
        ps, ok = ops.surface_solve(cam_pos, rays, initTmpPs, batch_inds, tmpSdf.packed_weights(),
                                   tmpSdf._pe_weights(sdf_ratio), tr_packed, tr_pe, conds, skin, dthreshold,
                                   athreshold, w1, w2, times, mode)
        initTmpPs.copy_(ps)            # the reference mutates and returns its seed tensor
    return initTmpPs.detach(), ok


def _jac_fn(deformer, conds_fn, ratio, offset_type):
    """(ps, inds) -> (D(ps), dD/dps) through the deformer's fused forward-mode launch, or None if it has none."""
    fn = getattr(deformer, "value_and_jacobian", None)
    if fn is None:
        return None

    def deform_jac(ps, inds):
        if not ps.is_cuda:
            return None
        with torch.no_grad():
            return fn(ps, conds_fn(), inds, ratio=ratio, offset_type=offset_type)
    return deform_jac


def OptimizeSurfacePs(cam_pos, rays, initTmpPs, batch_inds, tmpSdf, ratio, deformer, defconds,
                      dthreshold=5.e-5, athreshold=0.02, w1=3.05, w2=1., times=5):
    dev_res = _solve_device(cam_pos, rays, initTmpPs, batch_inds, tmpSdf, ratio, deformer, defconds, dthreshold,
                            athreshold, w1, w2, times) if DEVICE_SOLVE else None
    if dev_res is not None:
        return dev_res

    def deform(ps, inds):
        return deformer(ps, defconds, inds, ratio=ratio)
    return _solve(cam_pos, rays, initTmpPs, batch_inds, tmpSdf, ratio, deform, dthreshold, athreshold, w1, w2, times,
                  _jac_fn(deformer, lambda: defconds, ratio, None))


def OptimizeGarmentSurfaceSinlge(cam_pos, rays, initTmpPs, batch_inds, tmpSdf, ratio, deformer, defconds,
                                 dthreshold=5.e-5, athreshold=0.02, w1=3.05, w2=1., times=5, offset_type=None):
    dev_res = _solve_device(cam_pos, rays, initTmpPs, batch_inds, tmpSdf, ratio, deformer, defconds, dthreshold,
                            athreshold, w1, w2, times) if DEVICE_SOLVE else None
    if dev_res is not None:
        return dev_res

    def deform(ps, inds):
        return deformer(ps, defconds, inds, ratio=ratio, offset_type=offset_type)
    return _solve(cam_pos, rays, initTmpPs, batch_inds, tmpSdf, ratio, deform, dthreshold, athreshold, w1, w2, times,
                  _jac_fn(deformer, lambda: defconds, ratio, offset_type))


def OptimizeGarmentSurfacePs(cam_pos, rays_list, initTmpPs_list, batch_inds_list, tmpSdf_nets, ratio, deformer,
                             defconds_list, garment_names, dthreshold=5.e-5, athreshold=0.02, w1=3.05, w2=1.,
                             times=5):
    smpl_conds = defconds_list[1]
    out_ps, out_ok = [], []
    for gi, (ps, inds, dcond, rays, name) in enumerate(zip(initTmpPs_list, batch_inds_list, defconds_list[0],
                                                            rays_list, garment_names)):
        dev_res = _solve_device(cam_pos, rays, ps, inds, tmpSdf_nets[gi], ratio, deformer, [dcond, smpl_conds],
                                dthreshold, athreshold, w1, w2, times) if DEVICE_SOLVE else None
        if dev_res is not None:
            out_ps.append(dev_res[0])
            out_ok.append(dev_res[1])
            continue

        def deform(p, i, dcond=dcond, name=name):
            return deformer(p, [dcond, smpl_conds], i, ratio=ratio, offset_type=name)
        p, ok = _solve(cam_pos, rays, ps, inds, tmpSdf_nets[gi], ratio, deform, dthreshold, athreshold, w1, w2, times,
                       _jac_fn(deformer, lambda dcond=dcond: [dcond, smpl_conds], ratio, name))
        out_ps.append(p)
        out_ok.append(ok)
    return out_ps, out_ok
