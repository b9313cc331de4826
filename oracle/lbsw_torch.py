"""Restatement of the reference's skinning-voxel construction (model/Deformer.py:533-591, utils/LBSWsmpl.py:2-51) in
plain torch, chunked so it runs at the production size, in fp32 or fp64, on CPU or GPU.  TEST / MEASUREMENT
INFRASTRUCTURE ONLY.

With stable_ties=True the k nearest vertices come from a stable sort, so on exactly equal distances the lower vertex
index wins -- the rule of recmv_lbsw_knn_blend.  stable_ties=False uses torch.topk in 50 000-voxel chunks, which is
the reference's own algorithm (and the one worth timing)."""
import torch


def voxel_centres(bmins, bmaxs, resolutions, align_corners=False, dtype=torch.float32, device="cpu"):
    """[N,3] centres, voxel (z H + y) W + x, in the reference's order of operations (Deformer.py:549-571)."""
    bmins = torch.tensor(bmins, dtype=dtype, device=device).view(1, -1)
    bmaxs = torch.tensor(bmaxs, dtype=dtype, device=device).view(1, -1)
    W, H, D = resolutions
    res = torch.tensor(resolutions, dtype=dtype, device=device).view(-1)
    gz, gy, gx = torch.meshgrid([torch.arange(D, device=device), torch.arange(H, device=device),
                                 torch.arange(W, device=device)], indexing="ij")
    coords = torch.stack([gx, gy, gz]).view(3, -1).t().to(dtype)
    if align_corners:
        c = coords / (res[None, :] - 1)
    else:
        c = coords / res[None, :] + (1.0 / res[None, :]) / 2
    return c * (bmaxs - bmins) + bmins


def knn_blend(bmins, bmaxs, resolutions, verts, vert_ws, k, align_corners=False, dtype=torch.float32,
              stable_ties=True, chunk=None, return_idx=False):
    """Deformer.py:572-585 -> fws [N,24] (and idx [N,k], nearest first, and the chosen distances [N,k])."""
    dev = verts.device
    verts, vert_ws = verts.to(dtype).reshape(-1, 3), vert_ws.to(dtype).reshape(verts.shape[0], -1)
    centres = voxel_centres(bmins, bmaxs, resolutions, align_corners, dtype, dev)
    chunk = chunk or (4096 if stable_ties else 50000)
    fws, idxs, dists = [], [], []
    for tmp in torch.split(centres, chunk):
        d = (tmp[:, None, :] - verts[None, :, :]).norm(dim=-1)
        if stable_ties:
            dk, ik = torch.sort(d, dim=-1, stable=True)
            dk, ik = dk[:, :k], ik[:, :k]
        else:
            dk, ik = d.topk(k, dim=-1, largest=False)
        del d
        ws = 1. / torch.clamp(dk, 0.0001, 1.)
        ws = ws / ws.sum(-1, keepdim=True)
        fws.append((vert_ws[ik.reshape(-1)] * ws.reshape(-1, 1)).reshape(ws.shape[0], k, -1).sum(1))
        if return_idx:
            idxs.append(ik)
            dists.append(dk)
    fws = torch.cat(fws, 0)
    return (fws, torch.cat(idxs, 0), torch.cat(dists, 0)) if return_idx else fws


def smooth_weights(weights, times, zero_below=0.0):
    """Deformer.py:533-544 (zero_below = 5e-3: LBSWsmpl.py:2-11) on a copy of weights [1,24,D,H,W]."""
    weights = weights.clone()
    for _ in range(times):
        mean = (weights[:, :, 2:, 1:-1, 1:-1] + weights[:, :, :-2, 1:-1, 1:-1] +
                weights[:, :, 1:-1, 2:, 1:-1] + weights[:, :, 1:-1, :-2, 1:-1] +
                weights[:, :, 1:-1, 1:-1, 2:] + weights[:, :, 1:-1, 1:-1, :-2]) / 6.0
        weights[:, :, 1:-1, 1:-1, 1:-1] = (weights[:, :, 1:-1, 1:-1, 1:-1] - mean) * 0.7 + mean
        weights = weights / weights.sum(1, keepdim=True)
    if zero_below > 0:
        weights[weights < zero_below] = 0.0
    return weights


def compute_lbswField(bmins, bmaxs, resolutions, verts, vert_ws, align_corners=False, mean_neighbor=5, smooth_times=30,
                      zero_below=0.0, dtype=torch.float32, stable_ties=True):
    """ws [1,24,D,H,W] as Deformer.py:546-591 builds it (LBSWsmpl.py's variant with zero_below = 5e-3)."""
    W, H, D = resolutions
    fws = knn_blend(bmins, bmaxs, resolutions, verts, vert_ws, mean_neighbor, align_corners, dtype, stable_ties)
    return smooth_weights(fws.transpose(0, 1).reshape(1, -1, D, H, W), smooth_times, zero_below)
