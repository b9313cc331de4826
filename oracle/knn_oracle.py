"""TEST INFRASTRUCTURE ONLY -- the nearest-neighbour rules of DESIGN section 1e, restated three ways:

  * nearest_f32        numpy float32: d = (dx*dx + dy*dy) [+ dz*dz], dx = x1 - x2, each operation a separate float32
                       ufunc (correctly rounded, never contracted), first index on equal d (np.argmin).  It reproduces
                       the kernel's dists and idx bit for bit for finite coordinates, by construction.
  * nearest_f64 / nearest_backward_f64
                       float64 brute force, and the backward in closed form:
                       dp1_i = 2 g_i (p1_i - p2_idx_i),  dp2_j = -sum_{i: idx_i = j} 2 g_i (p1_i - p2_j).
  * chamfer_f64 / fl_proj_f64
                       pytorch3d 0.4's chamfer formula and the batched feature-curve loss as float64 torch, so autograd
                       gives the reference gradients.
"""
import numpy as np
import torch


def _lengths(lengths, N, P):
    if lengths is None:
        return np.full(N, P, dtype=np.int64)
    return np.clip(np.asarray(lengths, dtype=np.int64), 0, P)


def dist_f32(q, c):
    """[R,P2] float32 squared distances of query rows q [R,D] to candidates c [P2,D], in the kernel's order."""
    q = np.asarray(q, dtype=np.float32)
    c = np.asarray(c, dtype=np.float32)
    d = None
    for k in range(q.shape[1]):
        dk = q[:, None, k] - c[None, :, k]
        sq = dk * dk
        d = sq if d is None else d + sq
    return d


def nearest_f32(p1, p2, lengths1=None, lengths2=None, rows=None):
    """(dists [N,P1] float32, idx [N,P1] int64) of the kernel.  `rows` restricts the check to those query indices
    (every cloud); the other rows are left as (0, -1)."""
    p1 = np.asarray(p1, dtype=np.float32)
    p2 = np.asarray(p2, dtype=np.float32)
    N, P1, _ = p1.shape
    P2 = p2.shape[1]
    l1, l2 = _lengths(lengths1, N, P1), _lengths(lengths2, N, P2)
    dists = np.zeros((N, P1), dtype=np.float32)
    idx = np.full((N, P1), -1, dtype=np.int64)
    rows = np.arange(P1) if rows is None else np.asarray(rows)
    chunk = max(1, (1 << 24) // max(P2, 1))   # query rows per block of the distance matrix
    for n in range(N):
        if l2[n] == 0:
            continue
        live = rows[rows < l1[n]]
        for s in range(0, len(live), chunk):
            r = live[s:s + chunk]
            d = dist_f32(p1[n, r], p2[n, :l2[n]])
            j = np.argmin(d, axis=1)
            idx[n, r] = j
            dists[n, r] = d[np.arange(len(r)), j]
    return dists, idx


def nearest_f64(p1, p2, lengths1=None, lengths2=None):
    """Float64 brute force of the same rule: (dists [N,P1], idx [N,P1])."""
    p1 = np.asarray(p1, dtype=np.float64)
    p2 = np.asarray(p2, dtype=np.float64)
    N, P1, _ = p1.shape
    l1, l2 = _lengths(lengths1, N, P1), _lengths(lengths2, N, p2.shape[1])
    dists = np.zeros((N, P1))
    idx = np.full((N, P1), -1, dtype=np.int64)
    for n in range(N):
        if l2[n] == 0 or l1[n] == 0:
            continue
        d = ((p1[n, :l1[n], None, :] - p2[n, None, :l2[n], :]) ** 2).sum(-1)
        j = np.argmin(d, axis=1)
        idx[n, :l1[n]] = j
        dists[n, :l1[n]] = d[np.arange(l1[n]), j]
    return dists, idx


def nearest_backward_f64(p1, p2, idx, grad):
    """Closed-form (dp1 [N,P1,D], dp2 [N,P2,D]) in float64 for given idx (-1 = no neighbour, contributes nothing)."""
    p1 = np.asarray(p1, dtype=np.float64)
    p2 = np.asarray(p2, dtype=np.float64)
    idx = np.asarray(idx)
    g = np.asarray(grad, dtype=np.float64)
    N = p1.shape[0]
    dp1 = np.zeros_like(p1)
    dp2 = np.zeros_like(p2)
    for n in range(N):
        ok = idx[n] >= 0
        j = idx[n][ok]
        t = 2.0 * g[n][ok, None] * (p1[n][ok] - p2[n][j])
        dp1[n][ok] = t
        np.add.at(dp2[n], j, -t)
    return dp1, dp2


def _cham_dir(x, y, lx, ly):
    """[N,P1] float64 distance of every x row to its nearest valid y row (0 for padded rows or an empty y)."""
    d = ((x[:, :, None, :] - y[:, None, :, :]) ** 2).sum(-1)
    P2 = y.shape[1]
    bad = torch.arange(P2)[None, None, :] >= ly[:, None, None]
    d = d.masked_fill(bad, float("inf"))
    m = d.min(2).values if P2 > 0 else torch.full(x.shape[:2], float("inf"), dtype=x.dtype)
    keep = (torch.arange(x.shape[1])[None, :] < lx[:, None]) & (ly[:, None] > 0)
    return torch.where(keep, m, torch.zeros_like(m))


def chamfer_f64(x, y, x_lengths=None, y_lengths=None, x_normals=None, y_normals=None, weights=None,
                batch_reduction="mean", point_reduction="mean"):
    """pytorch3d 0.4's chamfer_distance (point-to-point term) in float64 torch -> (distance, None)."""
    assert x_normals is None and y_normals is None and weights is None
    x = torch.as_tensor(x).double()
    y = torch.as_tensor(y).double()
    N, P1, P2 = x.shape[0], x.shape[1], y.shape[1]
    lx = torch.full((N,), P1, dtype=torch.int64) if x_lengths is None else torch.as_tensor(x_lengths).cpu()
    ly = torch.full((N,), P2, dtype=torch.int64) if y_lengths is None else torch.as_tensor(y_lengths).cpu()
    cham_x = _cham_dir(x, y, lx, ly).sum(1)
    cham_y = _cham_dir(y, x, ly, lx).sum(1)
    if point_reduction == "mean":
        cham_x, cham_y = cham_x / lx, cham_y / ly
    if batch_reduction is not None:
        cham_x, cham_y = cham_x.sum(), cham_y.sum()
        if batch_reduction == "mean":
            cham_x, cham_y = cham_x / N, cham_y / N
    return cham_x + cham_y, None


def fl_proj_f64(fl_pts_list, gt_fl_pts_list, fl_masks, proj_fl_weights=None):
    """The batched feature-curve loss of DESIGN section 1e in float64:
    L = (1/C) sum_c w_c sum_n S_{n,c} / (V_c or 1) / (Q_c or 1), S_{n,c} the sum-reduced chamfer distance of frame n's
    visible points (fl_masks[..., 0]) and its annotations."""
    C = len(fl_pts_list)
    w = [1.0] * C if proj_fl_weights is None else list(proj_fl_weights)
    loss = 0.0
    for c in range(C):
        pts, gt, vis = fl_pts_list[c][..., :2].double(), gt_fl_pts_list[c].double(), fl_masks[c][..., 0] != 0
        N, P = vis.shape
        order = torch.argsort((~vis).to(torch.uint8), dim=1, stable=True)
        xc = torch.gather(pts, 1, order[..., None].expand(-1, -1, 2))
        lx = vis.sum(1)
        S = chamfer_f64(xc, gt, lx, None, batch_reduction=None, point_reduction="sum")[0].sum()
        V, Q = int((lx > 0).sum()), int(lx.sum())
        loss = loss + w[c] * S / max(V, 1) / max(Q, 1)
    return loss / C
