"""Drop-in `Laplacian_Optimizer` (engineer/optimizer/lap_deform_optimizer.py:25-186): the feature-curve fit of the
garment templates, solved by the matrix-free PCG of csrc/lap_edit.cu (DESIGN section 1g).

Drop-in `NRICP_Optimizer_AdamW` (engineer/optimizer/nricp_optimizer.py:321-448): the template registration of
`registration` (OptimGarmentNetwork.py:2415-2425) with its inner loop on the fused step of csrc/nricp.cu.

Same constructor, same `__call__(**inputs) -> fitting(inputs) -> (loss, smpl_slice)`, same per-epoch line and the same
`<save_path>/nricp_deform/<garment_name>/<epochs>.obj`.  Per epoch: one warp, one nearest-neighbour query and the inner
steps, with one host read for the epoch's line.  The rules are DESIGN section 1f; the AdamW state restarts every epoch
because the reference builds a new optimizer per epoch.  Not supported (no live caller passes them):
`use_normal=False` and non-empty `static_pts_type`."""
import os
import warnings

import numpy as np
import torch

from . import ops


def _write_obj(path, verts, faces):
    with open(path, "w") as f:
        for v in verts.tolist():
            f.write("v {:.6f} {:.6f} {:.6f}\n".format(*v))
        for t in (faces + 1).tolist():
            f.write("f {:d} {:d} {:d}\n".format(*t))


def _write_ply(path, verts):
    """A vertex-only binary PLY, the form pytorch3d's save_ply(path, verts) writes."""
    v = np.ascontiguousarray(verts.detach().cpu().numpy(), dtype="<f4").reshape(-1, 3)
    with open(path, "wb") as f:
        f.write("ply\nformat binary_little_endian 1.0\nelement vertex {:d}\nproperty float x\nproperty float y\n"
                "property float z\nend_header\n".format(len(v)).encode("ascii"))
        f.write(v.tobytes())


class Laplacian_Optimizer:
    """Laplacian editing of the garment templates onto the feature curves: per epoch and template, the constraints from
    the template's own best_match (and static points), then y = argmin |L y - L x|^2 + c |P y - u|^2 and, with smooth,
    the reference's zero-diagonal Laplacian smoothing.  `stats` keeps the device stats of the last solve."""

    def __init__(self, epoch=3, constrain_weight=1., optimizer_setting=None, smooth=True):
        self.name = "Laplacian_Deform_Optimzier"
        self.optimizier_setting = optimizer_setting
        self.epoch = epoch
        self.constrain_weights = constrain_weight
        self.smooth = smooth
        self.stats = None

    def __call__(self, **inputs):
        return self.fitting(inputs)

    def _collect_data(self, inputs):
        """[(source_idx, target)] per template, the reference's merge_source_target_map of best_match and static points."""
        target_packed = {name: mesh.verts_packed() for mesh, name in zip(inputs["target_meshes"],
                                                                          inputs["target_fl_type"])}
        maps = []
        for template in inputs["source_fl_meshes"]:
            idx, tgt = template.best_match(target_packed, template.device, inputs["outlayer"])
            static = template.static_pts_match()
            if static is not None:
                idx, tgt = torch.cat([idx, static[0]], dim=0), torch.cat([tgt, static[1]], dim=0)
            maps.append((idx, tgt))
        return maps

    @torch.no_grad()
    def fitting(self, inputs):
        templates = inputs["source_fl_meshes"]
        for _ in range(self.epoch):
            maps = self._collect_data(inputs)
            vertices = [template.vertices for template in templates]
            os.makedirs("./debug/register/", exist_ok=True)
            for i, ((idx, tgt), v) in enumerate(zip(maps, vertices)):
                _write_ply("./debug/register/source_{}.ply".format(i), v[idx])
                _write_ply("./debug/register/target_{}.ply".format(i), tgt)
            for template, (idx, tgt), v in zip(templates, maps, vertices):
                dev = v.device
                x = v.to(torch.float32).contiguous()
                faces = template.faces.reshape(-1, 3).to(dev, torch.int64).contiguous()
                adjacency = ops.mesh_adjacency(faces, x.shape[0])
                new_v, stats = ops.laplacian_edit(x, adjacency, idx.to(dev, torch.int64).contiguous(),
                                                  tgt.to(dev, torch.float32).contiguous(), self.constrain_weights,
                                                  self.smooth)
                self.stats = stats
                st = stats.tolist()   # the solve's one host read
                if st[6] != 1.0:
                    warnings.warn("Laplacian_Optimizer: the solve did not converge ({}): iterations {}, relative "
                                  "residuals {}, {} constraints skipped".format(
                                      "non-finite residual" if st[6] < 0 else "max_iter reached",
                                      [int(k) for k in st[:3]], st[3:6], int(st[7])), RuntimeWarning)
                template.update_vertices(new_v)
        return inputs


class NRICP_Optimizer_AdamW:
    """NRICP with a local affine [A | b] per source vertex, fitted by AdamW(lr=1e-4, amsgrad=True) against the nearest
    target points, with a normal-angle gate, an edge stiffness and a uniform Laplacian."""

    def __init__(self, epoch, dense_pcl, use_normal, stiffness_weight=[], mile_stone=[], inner_iter=10,
                 laplacian_weight=0., gamma=1, threshold=0.5, optimizer_setting=None, device="cuda:0"):
        self.name = "NRICP_Optimizer_GPU"
        self.optimizier_setting = optimizer_setting
        self.dense_pcl = int(dense_pcl)
        self.use_normal = use_normal
        self.mile_times = 0
        self.mile_idx = 0
        self.stiffness_weight = stiffness_weight
        self.laplacian_weight = laplacian_weight
        self.inner_iter = inner_iter
        self.mile_stone = mile_stone
        self.epoch = epoch
        self.device = device
        self.gamma = gamma
        self.threshold = threshold
        self.affine = None   # X [V,3,4] of the last fit
        assert len(self.mile_stone) == len(self.stiffness_weight) - 1

    def __call__(self, **inputs):
        return self.fitting(inputs)

    def _collect_data(self, inputs):
        smpl_slice = inputs["smpl_slice"]
        while smpl_slice.vertices.squeeze(0).shape[0] < self.dense_pcl:
            smpl_slice = smpl_slice.dense_pcl(type="edge")
        inputs["smpl_slice"] = smpl_slice
        static_pts_ids = smpl_slice.get_outlayer_idx(*inputs["static_pts_type"])
        if len(static_pts_ids) != 0:
            raise NotImplementedError("NRICP_Optimizer_AdamW: static points are not supported")
        return (smpl_slice, inputs["cano_meshes"], inputs["save_path"], inputs["garment_name"],
                inputs["nricp_masks"])

    def fitting(self, inputs):
        if not self.use_normal:
            raise NotImplementedError("NRICP_Optimizer_AdamW: use_normal=False is not supported")
        self.mile_times = 0
        self.mile_idx = 0
        smpl_slice, cano_meshes, save_path, garment_name, nricp_masks = self._collect_data(inputs)
        if save_path is not None:
            save_path = os.path.join(save_path, "nricp_deform", str(garment_name))
            os.makedirs(save_path, exist_ok=True)
        dev = torch.device(self.device)

        src_v = smpl_slice.vertices.squeeze(0).to(dev, torch.float32).contiguous()
        src_f = smpl_slice.faces.squeeze(0).to(dev, torch.int64).contiguous()
        tgt_v = cano_meshes.verts_packed().to(dev, torch.float32).contiguous()
        tgt_f = cano_meshes.faces_packed().to(dev, torch.int64).contiguous()
        V = int(src_v.shape[0])
        src_n = ops.vertex_normals(src_v[None], src_f)[0]
        tgt_n = ops.vertex_normals(tgt_v[None], tgt_f)[0]
        keep = torch.as_tensor(nricp_masks, device=dev).reshape(-1) > 0
        tgt_v, tgt_n = tgt_v[keep].contiguous(), tgt_n[keep].contiguous()
        if tgt_v.shape[0] == 0:
            raise ValueError("NRICP_Optimizer_AdamW: nricp_masks leaves no target point")

        adjacency = ops.mesh_adjacency(src_f, V)
        X = torch.zeros((V, 3, 4), dtype=torch.float32, device=dev)
        X[:, 0, 0] = X[:, 1, 1] = X[:, 2, 2] = 1.0
        moments = tuple(torch.empty_like(X) for _ in range(3))
        stats = torch.zeros((ops.NRICP_STATS,), dtype=torch.float32, device=dev)

        new_v = ops.nricp_warp(X, src_v)
        for i in range(self.epoch):
            old_v = new_v
            _, idx = ops.knn_nearest(old_v[None], tgt_v[None])
            sw = self.stiffness_weight[self.mile_idx]
            lw = self.laplacian_weight[self.mile_idx]
            iterations = 100 if i == 0 else self.inner_iter
            for t in range(1, iterations + 1):
                ops.nricp_step(src_v, src_n, tgt_v, tgt_n, idx[0], adjacency, X, moments, t, sw, lw,
                               gamma=self.gamma, threshold=self.threshold, stats=stats)
            new_v = ops.nricp_warp(X, src_v)
            distance = (old_v - new_v).norm(dim=1).mean()
            d, s, lap, loss, cnt, dist = torch.cat([stats[:5], distance[None]]).tolist()   # the epoch's one host read
            print("current {:03d} NRICP avg_update:{:.5f} valid{:d}/{:d}: dis:{:.4f}, stiffness:{:.4f}, laplacian:{:.4f}, "
                  "total:{:.4f} laplacian_weight:{:.4f}, stiffness_weight:{:.4f}, static_sum:{:.4f}".format(
                      self.mile_times, dist, int(cnt), V, d, s, lap, loss, lw, sw, 0.0))
            self.mile_times += 1
            if self.mile_times in self.mile_stone:
                self.mile_idx += 1

        if save_path is not None:
            _write_obj(os.path.join(save_path, "{}.obj".format(self.mile_times)), new_v.cpu(), src_f.cpu())
        self.affine = X
        smpl_slice.update_padded(new_v[None].to(smpl_slice.vertices))
        return stats[3].clone(), smpl_slice
