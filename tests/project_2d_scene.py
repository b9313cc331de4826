"""A garment-model stand-in for `project_2d_loss` (OptimGarmentNetwork.py:1772-1883) on this package's networks, and the
reference's method restated in torch.  Shared by tests/test_gpu_project_2d.py and tools/bench_project_2d_loss.py.

`scene` builds a lightweight `self` of the class `Model` (this module carries FL_EXTRACT and ZBUF_THRESHOLD, as the
reference's network modules do): an outfit of `long_sleeve_upper` (4 curves, an ellipsoid) and `long_pants` (2 curves,
an open tube) around an ellipsoid body, the [MLPTranslator, LBSkinner] composite and SDF of the surface scene, a
`Curve` with the reference's Intersect_Free_Curve buffers, forward and regulariser, `fl_optimizer` AdamW(lr=1e-4)
over its scale and nx_scale, the compat `maskRender`, and `utils.fl_visible_by_body_zbuff` bound.
`reference_flow` is the reference's method body with its glue as the reference writes it: one deformer call per
curve, `transform_points_screen` through the composed world-to-NDC matrix with its `(image_size < 1).any()` host
test, the per-curve threshold loop, `utils.fl_proj_loss`, `regularization()` once per garment and `.item()` for every
info value."""
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(HERE, "golden"))

from oracle import zbuf_oracle as zo  # noqa: E402
from recmv_b200 import synth, utils  # noqa: E402

FL_EXTRACT = {'long_sleeve_upper': ['neck', 'left_cuff', 'right_cuff', 'upper_bottom'],
              'long_pants': ['left_pant', 'right_pant']}
ZBUF_THRESHOLD = {'neck': 0.1, 'right_cuff': 0.05, 'left_cuff': 0.05, 'left_pant': 0.05, 'right_pant': 0.05,
                  'upper_bottom': 0.08, 'bottom_curve': 0.1}
GARMENTS = ('long_sleeve_upper', 'long_pants')
FL_NAMES = [n for g in GARMENTS for n in FL_EXTRACT[g]]
RATIO = {"sdfRatio": 0.8, "deformerRatio": 0.6, "renderRatio": 0.9}
FL_WEIGHTS = {'neck': 1.0, 'left_cuff': 0.5, 'right_cuff': 0.75, 'upper_bottom': 1.25, 'left_pant': 0.6,
              'right_pant': 0.9}
# (centre, radius, axis) of each curve's ring: neck and waist horizontal, cuffs and hems vertical
RINGS = {'neck': ((0.0, 0.45, 0.0), 0.09, 1), 'left_cuff': ((0.27, 0.25, 0.0), 0.06, 0),
         'right_cuff': ((-0.27, 0.25, 0.0), 0.06, 0), 'upper_bottom': ((0.0, -0.02, 0.0), 0.26, 1),
         'left_pant': ((0.11, -0.55, 0.0), 0.09, 1), 'right_pant': ((-0.11, -0.55, 0.0), 0.09, 1)}


class Conf:
    def __init__(self, d):
        self.d = dict(d)

    def get_float(self, key):
        return float(self.d[key])

    def get_string(self, key):
        return str(self.d[key])

    def __contains__(self, key):
        return key in self.d or any(k.startswith(key + ".") for k in self.d)


CONF = {"fl_visible_method": "zbuff", "fl_weight.weight": 1.0, "fl_weight.sdf_weight": 60.0,
        "alpha_weight.center_weight": 1.0, "alpha_weight.diff_weight": 1.0}


class Curve(nn.Module):
    """Intersect_Free_Curve (engineer/utils/garment_structure.py:36-145) with the identity canonical-SMPL map: the
    buffers of `initialize_parameters`, `forward`, `regularization` and `query_canosmpl_verts` as the reference
    writes them."""

    def __init__(self, verts, fl_names):
        super().__init__()
        self.fl_names = list(fl_names)
        self.register_buffer('cano_smpl_verts', verts.clone())
        center = verts.mean(1, keepdim=True)
        self.register_buffer('cano_verts_center', center)
        dirs = (verts - center) / ((verts - center).norm(dim=-1, keepdim=True) + 1e-6)
        nx = torch.cross(dirs[:, :-1, :], dirs[:, 1:, :], dim=-1)
        nx = (nx / nx.norm(dim=-1, keepdim=True)).mean(dim=1, keepdim=True)
        self.register_buffer('cano_nx', nx)
        self.register_buffer('cano_v_dirs', dirs)
        self.register_buffer('init_scale', torch.clamp_min(((verts - center) * dirs).sum(-1, keepdim=True), 0.))
        self.scale = nn.Parameter(torch.full(self.init_scale.shape, 1.0, device=verts.device))
        self.nx_scale = nn.Parameter(torch.full(self.init_scale.shape, 0., device=verts.device))

    def query_canosmpl_verts(self, query_names):
        d = {n: v.squeeze(0) for n, v in zip(self.fl_names, torch.split(self.cano_smpl_verts, 1, dim=0))}
        return [d[n] for n in query_names]

    def forward(self):
        return (self.cano_verts_center + self.cano_v_dirs * self.init_scale * F.relu(self.scale)
                + self.nx_scale * self.cano_nx)

    def regularization(self, fl_masks):
        cano_verts = self.forward()
        used_flag = (fl_masks.sum() > 0).float()
        center_loss = used_flag * abs(cano_verts.mean(1, keepdim=True) - self.cano_verts_center).sum()
        diff_a = cano_verts[:, :-1, :] - cano_verts[:, 1:, :]
        diff_b = cano_verts[:, -1:, :] - cano_verts[:, 0:1, :]
        diff_c = cano_verts[:, 0:1, :] - cano_verts[:, 1:2, :]
        diff_a = torch.cat([diff_a, diff_b, diff_c], dim=1)
        diff_a = diff_a / (diff_a.norm(dim=-1, keepdim=True) + 1e-6)
        diff_a_loss = (1 - F.cosine_similarity(diff_a[:, :-1, :], diff_a[:, 1:, :], dim=-1))
        return {'center_offset': 0 * center_loss, 'diff_a_loss': diff_a_loss.sum()}


class Model(types.SimpleNamespace):
    """`self` of the method; the drop-in finds FL_EXTRACT and ZBUF_THRESHOLD in this class's module."""
    fl_visible_by_body_zbuff = utils.fl_visible_by_body_zbuff


def ring(centre, radius, axis, S, phase):
    t = np.linspace(0, 2 * np.pi, S, endpoint=False) + phase
    a, b = radius * np.cos(t), radius * np.sin(t)
    p = np.zeros((S, 3))
    if axis == 1:
        p[:, 0], p[:, 2] = a, b
    else:
        p[:, 1], p[:, 2] = a, b
    return p + np.asarray(centre)


def camera(N, H, W, dev):
    """A pinhole 3 units in front of the outfit, turning by frame; focal length 1.25 min(H, W)."""
    f = 1.25 * min(H, W)
    rows = []
    for n in range(N):
        a = 0.2 * n - 0.1
        R = np.array([[np.cos(a), 0, -np.sin(a)], [0, 1, 0], [np.sin(a), 0, np.cos(a)]])
        rows.append(np.concatenate([[f, f * 1.01, W / 2 + 0.35, H / 2 - 0.4], R.reshape(-1), [0.02, 0.05, 3.0]]))
    c = torch.tensor(np.asarray(rows), dtype=torch.float32, device=dev)
    return zo.Camera(c[:, 0:2].contiguous(), c[:, 2:4].contiguous(), c[:, 4:13].reshape(-1, 3, 3).contiguous(),
                     c[:, 13:16].contiguous(), (W, H))


def scene(dev, N=2, H=96, W=120, S=200, M=160, seed=7, nets=None):
    """(self, args of project_2d_loss) for the two-garment outfit."""
    import surface_render_scene as srs
    from recmv_b200.compat.MaskRender import mask_renderer
    sdf, deformer, _ = nets if nets is not None else srs.networks(dev)
    rng = np.random.default_rng(seed)
    verts = torch.tensor(np.stack([ring(*RINGS[n], S, 0.3 * i) for i, n in enumerate(FL_NAMES)]), dtype=torch.float32,
                         device=dev)
    curve = Curve(verts, FL_NAMES)
    with torch.no_grad():      # a curve part-way through fitting: some scales at or below 0
        curve.scale.copy_(torch.tensor(1.0 + rng.normal(0, 0.05, curve.scale.shape), dtype=torch.float32))
        curve.scale[0, 5:9] = 0.
        curve.scale[3, 40:43] = -0.1
        curve.nx_scale.copy_(torch.tensor(rng.normal(0, 0.01, curve.nx_scale.shape), dtype=torch.float32))
    up_v, up_f = zo.uv_sphere(16, 12, (0.30, 0.26, 0.22), (0.0, 0.22, 0.0))
    lo_v, lo_f = zo.tube(16, 8, 0.24, -0.6, -0.05)
    body_v, body_f = zo.uv_sphere(24, 14, (0.22, 0.62, 0.16), (0.0, -0.05, 0.0))
    d = lambda a, dt=torch.float32: torch.tensor(a, dtype=dt, device=dev)  # noqa: E731
    poses, trans = synth.poses_trans(N, seed=11)
    poses = (poses * 0.3).to(dev).requires_grad_(True)
    trans = (trans * 0.1).to(dev).requires_grad_(True)
    conds = [d(rng.standard_normal((N, 128)) * 0.1).requires_grad_(True) for _ in range(3)]
    cam = camera(N, H, W, dev)
    self = Model(
        garment_size=2, garment_names=list(GARMENTS), garment_nets=[sdf, sdf], fl_names=list(FL_NAMES),
        garment_vs=[d(up_v), d(lo_v)], garment_fs=[d(up_f, torch.int64), d(lo_f, torch.int64)],
        tmpBodyVs=d(body_v), tmpBodyFs=d(body_f, torch.int64), deformer=deformer, conf=Conf(CONF), info={},
        sdfShrinkRadius=0.01, inter_free_curve=curve, maskRender=mask_renderer((H, W), cameras=cam),
        fl_optimizer=torch.optim.AdamW([curve.scale, curve.nx_scale], lr=1e-4),
        dataset=types.SimpleNamespace(fl_weights=dict(FL_WEIGHTS)),
        get_grad_parameters=lambda frame_ids, device: (conds, poses, trans, None))
    fl_masks = torch.ones((N, len(FL_NAMES)), dtype=torch.bool, device=dev)
    fl_masks[:, 2] = False                       # right_cuff unlabelled in every frame
    if N > 1:
        fl_masks[1, 4] = False                   # left_pant unlabelled in frame 1
    gt = []
    with torch.no_grad():
        for n in FL_NAMES:
            c = np.asarray(RINGS[n][0])
            p = torch.tensor(ring(c, RINGS[n][1] * 1.05, RINGS[n][2], M, 0.1), dtype=torch.float32, device=dev)
            gt.append(cam.transform_points_screen(p[None].expand(N, -1, 3),
                                                  torch.tensor([[W, H]] * N, dtype=torch.float32, device=dev))[..., :2])
    gt_fl_pts = torch.cat(gt, 1) + d(rng.normal(0, 0.5, (N, M * len(FL_NAMES), 2)))
    args = (N, H, W, torch.arange(N, device=dev), RATIO, cam, fl_masks, gt_fl_pts.contiguous(), dev)
    return self, args, dict(poses=poses, trans=trans, conds=conds, deformer=deformer, curve=curve, sdf=sdf)


def transform_points_screen(cameras, points, image_size):
    """CameraMine.transform_points_screen: the composed world-to-NDC matrix, the host test of the image size, then
    the screen conversion."""
    if (image_size < 1).any():
        raise ValueError("Provided image size is invalid.")
    return cameras.transform_points_screen(points, image_size)


def reference_flow(self, N, H, W, frame_ids, ratio, cameras, fl_masks, gt_fl_pts, device, sdf_scale=10.,
                   proj_scale=1.):
    """The reference's project_2d_loss (with deform_feature_line and compute_fl_proj_loss), glue as written."""
    project_loss = 0.
    fl_garment_sdf_loss = 0.
    self.info['fl_loss'] = {}
    proj_img_size = torch.Tensor([W, H]).float()[None].expand(N, 2).to(device)
    d_cond_list, poses, trans, _ = self.get_grad_parameters(frame_ids, device)
    offset_fl_verts_list = torch.split(self.inter_free_curve(), 1, dim=0)
    gt_fl_pts_list = torch.split(gt_fl_pts, gt_fl_pts.shape[1] // len(self.fl_names), dim=1)
    gt_fl_masks_list = torch.split(fl_masks, 1, 1)
    fl_vs_dict, gt_dict, mask_dict = {}, {}, {}
    for name, v, g, m in zip(self.fl_names, offset_fl_verts_list, gt_fl_pts_list, gt_fl_masks_list):
        fl_vs_dict[name], gt_dict[name], mask_dict[name] = v, g, m
    visible_mask_list, label_mask_list, drawn = [], [], []
    for g_i, garment_name in enumerate(self.garment_names):
        fl_names = FL_EXTRACT[garment_name]
        def_fl_vs = [self.deformer(fl_vs_dict[n].view(-1, 3).expand(N, -1, 3), [d_cond_list[g_i + 1], [poses, trans]],
                                   ratio=ratio, offset_type=n) for n in fl_names]
        cano_smpl = self.inter_free_curve.query_canosmpl_verts(fl_names)
        nx = self.fl_visible_by_body_zbuff(cameras, d_cond_list, [poses, trans], ratio, fl_vs_dict, def_fl_vs,
                                           cano_smpl, fl_names, g_i, garment_name, proj_img_size, N)
        fl_vs = [fl_vs_dict[n].view(-1, 3) for n in fl_names]
        split = [v.shape[1] for v in def_fl_vs]
        gt_g = torch.cat([gt_dict[n] for n in fl_names], dim=1)
        masks_g = torch.cat([mask_dict[n] for n in fl_names], dim=-1)
        # compute_fl_proj_loss
        screen_pts = transform_points_screen(cameras, torch.cat(def_fl_vs, dim=1), proj_img_size)
        thr = torch.zeros_like(nx)
        end_val = np.cumsum(split)
        start = 0
        for end_ind, n in enumerate(fl_names):
            thr[..., start:end_val[end_ind], :] = ZBUF_THRESHOLD[n]
            start = end_val[end_ind]
        body_visible = (nx < thr)[..., 1]
        gt_list = torch.split(gt_g, [gt_g.shape[1] // len(fl_names)] * len(fl_names), dim=1)
        vis_masks, lab_masks = [], []
        for fl_idx, (pts, cv) in enumerate(zip(torch.split(screen_pts, split, dim=1),
                                               torch.split(body_visible, split, dim=1))):
            fl_mask = masks_g[:, None, fl_idx:fl_idx + 1].expand_as(pts)
            vis_masks.append(torch.logical_and(fl_mask, cv[..., None].expand_as(pts)))
            lab_masks.append(fl_mask)
        w = [self.dataset.fl_weights[n] for n in fl_names]
        fl_loss = utils.fl_proj_loss(list(torch.split(screen_pts, split, dim=1)), gt_list, vis_masks, w) * \
            (self.conf.get_float('fl_weight.weight') if 'fl_weight.weight' in self.conf else 1.)
        self.info['fl_loss']['{}_project loss'.format(garment_name)] = fl_loss.item()
        loss = 0.
        loss += fl_loss
        reg = self.inter_free_curve.regularization(masks_g)
        center = reg['center_offset'] * (self.conf.get_float('alpha_weight.center_weight')
                                         if 'alpha_weight' in self.conf else 1.)
        diff = reg['diff_a_loss'] * (self.conf.get_float('alpha_weight.diff_weight') if 'alpha_weight' in self.conf
                                     else 1.)
        loss += center
        loss += diff
        self.info['fl_loss']['{}_center loss'.format(garment_name)] = center.item()
        self.info['fl_loss']['{}_diff a loss'.format(garment_name)] = diff.item()
        project_loss += loss
        sdf = self.garment_nets[g_i](torch.cat(fl_vs, dim=0), ratio).view(-1)
        sdf_loss = (sdf + self.sdfShrinkRadius).abs().mean()
        self.info['fl_loss']['pc_{}_loss_sdf'.format(garment_name)] = sdf_loss.item()
        fl_garment_sdf_loss += sdf_loss * (self.conf.get_float('fl_weight.sdf_weight') if 'fl_weight' in self.conf
                                           else 60.)
        visible_mask_list.append(vis_masks)
        label_mask_list.append(lab_masks)
        drawn.append((def_fl_vs, split, gt_g))
    self.fl_optimizer.zero_grad()
    loss = sdf_scale * fl_garment_sdf_loss + proj_scale * project_loss
    loss.backward()
    self.fl_optimizer.step()
    with torch.no_grad():
        garment_fl_vs_list, gt_out = [], []
        for def_fl_vs, split, gt_g in drawn:
            screen_pts = transform_points_screen(cameras, torch.cat(def_fl_vs, dim=1), proj_img_size)
            garment_fl_vs_list.append(torch.split(screen_pts, split, dim=1))
            gt_out.append(gt_g)
    return garment_fl_vs_list, visible_mask_list, label_mask_list, gt_out
