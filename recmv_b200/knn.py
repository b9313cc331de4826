"""Drop-in for pytorch3d 0.4's `knn_points`, `knn_gather` and `chamfer_distance` (DESIGN section 1e), on the
deterministic nearest-neighbour kernel of csrc/knn.cu.  K = 1 only (no live caller asks for more); normals, weights
and `return_nn` raise.  There is no CPU path, and nothing here reads the device from the host."""
from collections import namedtuple

import torch

from . import ops

KNN = namedtuple("KNN", ["dists", "idx", "knn"])


def knn_points(p1, p2, lengths1=None, lengths2=None, K=1, return_nn=False, return_sorted=True):
    """KNN(dists [N,P1,1] squared distance, idx [N,P1,1] int64, None) of every p1 point in p2 (float32 CUDA [N,P,D],
    D = 2 or 3; lengths int64 [N] on the device).  On equal distances the lower index wins.  Padded queries, and every
    query of a cloud with lengths2 == 0, get dists 0 and idx -1.  Differentiable in p1 and p2 through dists.  Strided
    inputs are made contiguous first, as pytorch3d accepts them."""
    if int(K) != 1:
        raise NotImplementedError(f"knn_points: only K = 1 is implemented, got K = {K}")
    if return_nn:
        raise NotImplementedError("knn_points: return_nn is not implemented (use knn_gather on idx)")
    dists, idx = ops.KnnNearestFunction.apply(p1.contiguous(), p2.contiguous(), lengths1, lengths2)
    return KNN(dists.unsqueeze(-1), idx.unsqueeze(-1), None)


def knn_gather(x, idx, lengths=None):
    """x [N,M,U] gathered at idx [N,L,K] -> [N,L,K,U] (pytorch3d's signature).  Entries with idx = -1, and neighbours
    k >= lengths[n] when lengths is given, give 0."""
    N, M, U = x.shape
    _N, L, K = idx.shape
    if N != _N:
        raise ValueError("knn_gather: x and idx must have the same batch dimension")
    if M == 0:
        return x.new_zeros((N, L, K, U))
    out = x[:, :, None].expand(-1, -1, K, -1).gather(1, idx.clamp_min(0)[..., None].expand(-1, -1, -1, U))
    drop = idx[..., None] < 0
    if lengths is not None:
        drop = drop | (torch.arange(K, device=idx.device)[None, None, :, None] >= lengths[:, None, None, None])
    return out.masked_fill(drop, 0.0)


def chamfer_distance(x, y, x_lengths=None, y_lengths=None, x_normals=None, y_normals=None, weights=None,
                     batch_reduction="mean", point_reduction="mean"):
    """pytorch3d 0.4's chamfer distance of two padded batches x [N,P1,D], y [N,P2,D] -> (distance, None).
    cham_x[n,i] = squared distance of x_i to its nearest point of y (0 for padded rows and when y is empty), summed
    over i, divided by x_lengths for point_reduction="mean" (an empty cloud gives 0/0 = NaN); the same for y; then
    summed over the batch for batch_reduction "sum" / "mean" (÷N) or kept per cloud for None."""
    if x_normals is not None or y_normals is not None or weights is not None:
        raise NotImplementedError("chamfer_distance: normals and weights are not implemented")
    if batch_reduction not in (None, "sum", "mean"):
        raise ValueError('batch_reduction must be one of ["mean", "sum"] or None')
    if point_reduction not in ("sum", "mean"):
        raise ValueError('point_reduction must be one of ["mean", "sum"]')
    if not (torch.is_tensor(x) and torch.is_tensor(y)):
        raise NotImplementedError("chamfer_distance: only padded tensors are accepted, not Pointclouds")
    N, P1, P2 = x.shape[0], x.shape[1], y.shape[1]
    if y.shape[0] != N or y.shape[2] != x.shape[2]:
        raise ValueError("chamfer_distance: x and y must have the same batch size and dimension")
    x, y = x.contiguous(), y.contiguous()
    cham_x = ops.KnnNearestFunction.apply(x, y, x_lengths, y_lengths)[0].sum(1)
    cham_y = ops.KnnNearestFunction.apply(y, x, y_lengths, x_lengths)[0].sum(1)
    if point_reduction == "mean":
        cham_x = cham_x / (x_lengths if x_lengths is not None else P1)
        cham_y = cham_y / (y_lengths if y_lengths is not None else P2)
    if batch_reduction is not None:
        cham_x, cham_y = cham_x.sum(), cham_y.sum()
        if batch_reduction == "mean":
            cham_x, cham_y = cham_x / N, cham_y / N
    return cham_x + cham_y, None
