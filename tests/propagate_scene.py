"""The state `propagateTmpPsGrad` (OptimGarmentNetwork.py:2159-2313, OptimGarmentNetwork_Large_Pose.py:327-473) runs
on, built on this package's networks, and the reference's method body restated on them.  Shared by
tests/test_gpu_propagate.py, tests/golden/make_golden_propagate.py (the inputs) and tools/bench_propagate_grad.py.

`inputs` draws the seeded arrays of a call: per garment the surface points TmpPs, their loss gradient TmpPs.grad and
their (col, row, frame); a camera; poses, translations and the body and garment conditions.  `state` builds a
lightweight `self` from them as `surface_render_loss` leaves it: TmpPs leaves with .grad set, the rays the camera's
`view_rays` of (col, row, 1) (with a graph when the camera is learnable), batch / row / col indices, `garment_nets`
and `deformer` from tests/surface_render_scene.py's `networks`, `get_grad_parameters`, `dataset.get_camera_parameters`
(focal length, principal point and T requiring grad, as `opt_camera` sets them), `maskRender` and `info`.
`reference_flow` is the reference's method kept as the reference writes it (per garment: autograd for grad f, three
autograd passes for J, the 3x3 algebra in torch with FastMinv, `check.sum().item()`, two VJPs and a surrogate loss),
with `self.rays[g]` in the fixed-camera branch where the reference writes `self.rays`."""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from recmv_b200 import ops, utils  # noqa: E402
from surface_render_scene import RATIO, networks  # noqa: E402

NAMES = ("upper", "bottom", "dress", "skirt", "coat")


class RectifiedPerspectiveCameras:
    """Stands in for the reference's camera class (model/CameraMine.py): its parameters, `view_rays` (:146-167) and
    `cam_pos` (:207-208)."""

    def __init__(self, focal_length, principal_point, R, T, image_size=None):
        self.focal_length, self.principal_point, self.R, self.T = focal_length, principal_point, R, T

    def to(self, device):
        return self

    def view_rays(self, ps, cam_id=0):
        rays = torch.zeros_like(ps)
        rays[:, 0] = -ps[:, 0] / self.focal_length[cam_id, 0] + ps[:, 2] * self.principal_point[cam_id, 0] / self.focal_length[cam_id, 0]
        rays[:, 1] = -ps[:, 1] / self.focal_length[cam_id, 1] + ps[:, 2] * self.principal_point[cam_id, 1] / self.focal_length[cam_id, 1]
        rays[:, 2] = ps[:, 2]
        rays = rays / torch.norm(rays, p=2, dim=1, keepdim=True)
        return rays.matmul(self.R[cam_id].transpose(0, 1))

    def cam_pos(self, cam_id=0):
        return -self.R[cam_id].matmul(self.T[cam_id].view(-1, 1)).view(-1)


class Garment:
    """OptimGarmentNetwork with the drop-in bound."""
    propagateTmpPsGrad = utils.make_propagate_tmp_ps_grad()


class GarmentLargePose(Garment):
    """OptimGarmentNetwork_LargePose with the same drop-in bound (the class overrides the method)."""
    propagateTmpPsGrad = utils.make_propagate_tmp_ps_grad()


def camera(H, W):
    """fx, fy, px, py, R (with the dataset's y / z flips) and T."""
    q = np.array([0.97, 0.05, -0.2, 0.1])
    q /= np.linalg.norm(q)
    w, x, y, z = q
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]) @ np.diag([1., -1., -1.])
    s = W / 64.0
    return (np.array([60.5 * s, 58.25 * s], np.float32), np.array([W * 0.49, H * 0.52], np.float32),
            R.astype(np.float32), np.array([0.02, -0.1, 2.4], np.float32))


def inputs(M=(300, 240), N=3, H=64, W=64, seed=2159):
    """The seeded arrays of one call: P_g, gl_g (TmpPs.grad), col_g / row_g (float32 pixel coordinates), batch_g;
    focal, pp, R, T, H, W; poses, trans, conds [G+1, N, 128]."""
    from recmv_b200 import synth
    rng = np.random.default_rng(seed)
    d = {}
    for g, m in enumerate(M):
        u = rng.standard_normal((m, 3))
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        d[f"P_{g}"] = (u * 0.45 + rng.standard_normal((m, 3)) * 0.02).astype(np.float32)
        d[f"gl_{g}"] = (rng.standard_normal((m, 3)) * 0.01).astype(np.float32)
        d[f"col_{g}"] = rng.integers(0, W, m).astype(np.float32)
        d[f"row_{g}"] = rng.integers(0, H, m).astype(np.float32)
        d[f"batch_{g}"] = rng.integers(0, N, m).astype(np.int64)
    d["focal"], d["pp"], d["R"], d["T"] = camera(H, W)
    d["H"], d["W"], d["N"], d["G"] = np.array(H), np.array(W), np.array(N), np.array(len(M))
    poses, trans = synth.poses_trans(N, seed=11)
    d["poses"], d["trans"] = poses.numpy(), trans.numpy()
    d["conds"] = (rng.standard_normal((len(M) + 1, N, 128)) * 0.1).astype(np.float32)
    return d


def state(dev, d, cls=Garment, learnable_camera=True, nets=None, frozen_sdf=False):
    """(self, leaves) from the arrays of `inputs`: leaves maps focal, pp, T, poses, trans, cond<k> and TmpPs<g> to the
    tensors whose .grad the method fills."""
    sdf, deformer, _ = nets if nets is not None else networks(dev)
    if frozen_sdf:
        sdf.requires_grad_(False)
    G, N, H, W = int(d["G"]), int(d["N"]), int(d["H"]), int(d["W"])
    t = lambda k: torch.from_numpy(np.ascontiguousarray(d[k])).to(dev)  # noqa: E731
    focal, pp, R, T = t("focal"), t("pp"), t("R"), t("T")
    if learnable_camera:
        focal.requires_grad_(True), pp.requires_grad_(True), T.requires_grad_(True)
    poses, trans = t("poses").requires_grad_(True), t("trans").requires_grad_(True)
    conds = [t("conds")[k].clone().requires_grad_(k > 0) for k in range(G + 1)]

    def get_camera_parameters(n, device):
        return (focal.view(1, 2).expand(n, 2), pp.view(1, 2).expand(n, 2), R.view(1, 3, 3).expand(n, 3, 3),
                T.view(1, 3).expand(n, 3), H, W)

    self = cls()
    self.garment_size, self.garment_names = G, list(NAMES[:G])
    self.garment_nets, self.deformer = [sdf] * G, deformer
    self.dataset = types.SimpleNamespace(get_camera_parameters=get_camera_parameters)
    self.maskRender = types.SimpleNamespace(rasterizer=types.SimpleNamespace(cameras=None))
    self.get_grad_parameters = lambda frame_ids, device: (conds, poses, trans, torch.zeros((N, 1), device=dev))
    self.info = {}
    cams = RectifiedPerspectiveCameras(*get_camera_parameters(N, dev)[:4])
    self.TmpPs, self.rays, self.batch_inds, self.row_inds, self.col_inds = ([None] * G for _ in range(5))
    leaves = {"focal": focal, "pp": pp, "T": T, "poses": poses, "trans": trans}
    for k in range(1, G + 1):
        leaves[f"cond{k}"] = conds[k]
    for g in range(G):
        p = t(f"P_{g}").clone().requires_grad_(True)
        p.grad = t(f"gl_{g}").clone()
        self.TmpPs[g] = leaves[f"TmpPs{g}"] = p
        self.col_inds[g], self.row_inds[g], self.batch_inds[g] = t(f"col_{g}"), t(f"row_{g}"), t(f"batch_{g}")
        px = torch.stack([self.col_inds[g], self.row_inds[g], torch.ones_like(self.col_inds[g])], 1).float()
        rays = cams.view_rays(px)
        self.rays[g] = rays if learnable_camera else rays.detach()
    return self, leaves


def reference_flow(self, frame_ids, ratio, large_pose=False):
    """The reference's propagateTmpPsGrad on this package's networks (see the module docstring); `large_pose` drops
    the SDF term as OptimGarmentNetwork_Large_Pose.py does."""
    Fast3x3Minv = ops.minv3x3
    for garment_idx in range(self.garment_size):
        garment_name = self.garment_names[garment_idx]
        if self.TmpPs[garment_idx] is None or self.TmpPs[garment_idx].grad is None:
            self.info['{}_invInfo'.format(garment_name)] = (-1, -1)
            return
        device = self.TmpPs[garment_idx].device
        d_cond_list, poses, trans, _ = self.get_grad_parameters(frame_ids, device)
        defconds = [d_cond_list[1 + garment_idx], [poses, trans]]
        focals, princeple_ps, Rs, Ts, H, W = self.dataset.get_camera_parameters(frame_ids.numel(), device)
        self.maskRender.rasterizer.cameras = RectifiedPerspectiveCameras(focals, princeple_ps, Rs, Ts,
                                                                         image_size=[(W, H)]).to(device)
        grad_l_p = self.TmpPs[garment_idx].grad
        if self.rays[garment_idx].requires_grad:
            v = self.maskRender.rasterizer.cameras.view_rays(torch.cat([self.col_inds[garment_idx].view(-1, 1), self.row_inds[garment_idx].view(-1, 1), torch.ones_like(self.col_inds[garment_idx].view(-1, 1))], dim=-1).float())
        else:
            v = self.rays[garment_idx].detach()
        c = self.maskRender.rasterizer.cameras.cam_pos()
        p = self.TmpPs[garment_idx]
        f = self.garment_nets[garment_idx](p, ratio)
        grad_f_p = torch.autograd.grad(f, p, torch.ones_like(f), retain_graph=False)[0]
        d = self.deformer(p, defconds, self.batch_inds[garment_idx], ratio=ratio, offset_type=garment_name)
        inputs = [p]
        grad_d_p = []
        opt_defconds = []
        for defcond in defconds:
            if type(defcond) is list:
                for defc in defcond:
                    if defc.requires_grad:
                        opt_defconds.append(defc)
            else:
                if defcond.requires_grad:
                    opt_defconds.append(defcond)
        grad_outputs = torch.ones_like(d[..., 0])
        outx = torch.autograd.grad(d[..., 0], inputs, grad_outputs, retain_graph=True)
        grad_d_p.append(outx[0].view(-1, 1, 3))
        outy = torch.autograd.grad(d[..., 1], inputs, grad_outputs, retain_graph=True)
        grad_d_p.append(outy[0].view(-1, 1, 3))
        outz = torch.autograd.grad(d[..., 2], inputs, grad_outputs, retain_graph=False)
        grad_d_p.append(outz[0].view(-1, 1, 3))
        grad_d_p = torch.cat(grad_d_p, dim=1)
        v_cross = torch.zeros_like(grad_d_p)
        v_cross[:, 0, 1] = -v[:, 2]
        v_cross[:, 0, 2] = v[:, 1]
        v_cross[:, 1, 0] = v[:, 2]
        v_cross[:, 1, 2] = -v[:, 0]
        v_cross[:, 2, 0] = -v[:, 1]
        v_cross[:, 2, 1] = v[:, 0]
        v_cross = v_cross.detach()
        a1 = v_cross.matmul(grad_d_p)
        b = torch.cat([grad_f_p.view(-1, 1, 3), a1], dim=1)
        btb = b.permute(0, 2, 1).matmul(b)
        btb_inv, check = Fast3x3Minv(btb.contiguous())
        self.info['{}_invInfo'.format(garment_name)] = (check.numel(), check.sum().item())
        rhs_1 = btb_inv.matmul(b.permute(0, 2, 1))
        rhs_1 = grad_l_p.view(-1, 1, 3).matmul(rhs_1)
        loss = 0.
        if not large_pose:
            params = [param for param in self.garment_nets[garment_idx].parameters() if param.requires_grad]
            params_grads = torch.autograd.grad(self.garment_nets[garment_idx](p, ratio), params, -rhs_1[:, :, 0])
            for param, grad in zip(params, params_grads):
                loss += (param * grad).sum()
        params = [param for param in self.deformer.parameters() if param.requires_grad]
        d = self.deformer(p, defconds, self.batch_inds[garment_idx], ratio=ratio, offset_type=garment_name)
        temp = (rhs_1[:, :, -3:].matmul(-v_cross)).view(-1, 3)
        if len(opt_defconds):
            params_grads = torch.autograd.grad(d, params, temp, retain_graph=True)
        else:
            params_grads = torch.autograd.grad(d, params, temp, retain_graph=False)
        for param, grad in zip(params, params_grads):
            loss += (param * grad).sum()
        if len(opt_defconds):
            params_grads = torch.autograd.grad(d, opt_defconds, temp, retain_graph=False)
            for opt_defcond, grad in zip(opt_defconds, params_grads):
                loss += (opt_defcond * grad).sum()
        if v.requires_grad:
            dc = d.detach() - c.detach().view(1, 3)
            dc_cross = torch.zeros_like(grad_d_p)
            dc_cross[:, 0, 1] = -dc[:, 2]
            dc_cross[:, 0, 2] = dc[:, 1]
            dc_cross[:, 1, 0] = dc[:, 2]
            dc_cross[:, 1, 2] = -dc[:, 0]
            dc_cross[:, 2, 0] = -dc[:, 1]
            dc_cross[:, 2, 1] = dc[:, 0]
            grad = rhs_1[:, :, -3:].matmul(dc_cross).view(-1, 3)
            loss += (v * grad).sum()
        if c.requires_grad:
            grad = -temp.sum(0)
            loss += (c * grad).sum()
        loss.backward()
