"""Float64 oracle of the NRICP rules of DESIGN section 1f, written from the rules: the mesh adjacency and boundary, the
uniform Laplacian built the way pytorch3d 0.4's `laplacian_packed` builds it (COO A over both directions of the edges,
row-sum degrees, D^-1 A - I), the loss of one inner iteration, its closed-form gradient, one AdamW-AMSGrad step and
the fitting loop of `NRICP_Optimizer_AdamW`.  The vertex normals come from oracle/shade_oracle.py.

`Meshes`, `laplacian_smoothing_torch`, `knn_points` and `knn_gather` are float64 torch stand-ins with pytorch3d's
call forms, for running the reference's own loop on the CPU (tests/golden/make_golden_nricp.py) and for checking the
closed-form gradient against autograd."""
import types

import numpy as np
import scipy.sparse as sp
import torch

from oracle import shade_oracle

ADAMW = dict(lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)


def adjacency(faces, V):
    """faces [F,3] over V vertices -> dict(edges [E,2] unique sorted pairs, row_ptr [V+1], col [2E] (neighbours of
    every row ascending, both directions of every edge), deg [V], boundary [V] bool).  Faces with an index outside
    [0, V) are skipped."""
    faces = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    f = faces[np.all((faces >= 0) & (faces < V), axis=1)]
    sides = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1)
    h, cnt = np.unique(sides[:, 0] * V + sides[:, 1], return_counts=True)
    edges = np.stack([h // V, h % V], axis=1)
    boundary = np.zeros(V, dtype=bool)
    once = h[cnt == 1]
    boundary[once // V] = True
    boundary[once % V] = True
    rows = np.concatenate([edges[:, 0], edges[:, 1]])
    cols = np.concatenate([edges[:, 1], edges[:, 0]])
    order = np.lexsort((cols, rows))
    deg = np.bincount(rows, minlength=V).astype(np.int64)
    row_ptr = np.zeros(V + 1, dtype=np.int64)
    row_ptr[1:] = np.cumsum(deg)
    return dict(edges=edges, row_ptr=row_ptr, col=cols[order], deg=deg, boundary=boundary)


def laplacian(edges, V):
    """pytorch3d 0.4's uniform Laplacian: A = COO over (e0, e1) and (e1, e0) with ones, deg = row sums of A,
    L = D^-1 A - I with a zero row scale where deg = 0.  scipy CSR, duplicates summed."""
    e0, e1 = edges[:, 0], edges[:, 1]
    rows, cols = np.concatenate([e0, e1]), np.concatenate([e1, e0])
    A = sp.coo_matrix((np.ones(len(rows)), (rows, cols)), shape=(V, V)).tocsr()
    deg = np.asarray(A.sum(axis=1)).ravel()
    inv = np.where(deg > 0, 1.0 / np.where(deg > 0, deg, 1.0), 0.0)
    vals = np.concatenate([inv[e0], inv[e1]])
    return (sp.coo_matrix((vals, (rows, cols)), shape=(V, V)) - sp.identity(V)).tocsr()


def identity_affine(V):
    X = np.zeros((V, 3, 4))
    X[:, 0, 0] = X[:, 1, 1] = X[:, 2, 2] = 1.0
    return X


def inv3x3(A):
    """FastMinv's rule in float64: inverse by cofactors, zeros and ok = False where |det| < 1e-4."""
    det = np.linalg.det(A)
    ok = np.abs(det) >= 1e-4
    inv = np.zeros_like(A)
    if ok.any():
        inv[ok] = np.linalg.inv(A[ok])
    return inv, ok


def warp(X, x, n=None):
    """v = A x + b; with n also (n' = inv(A)^T n, ok)."""
    v = np.einsum("vij,vj->vi", X[:, :, :3], x) + X[:, :, 3]
    if n is None:
        return v
    inv, ok = inv3x3(X[:, :, :3])
    return v, np.einsum("vji,vj->vi", inv, n), ok


def cosine(a, b):
    """torch 1.10's cosine_similarity: a.b / sqrt(max(|a|^2 |b|^2, 1e-16))."""
    return (a * b).sum(-1) / np.sqrt(np.maximum((a * a).sum(-1) * (b * b).sum(-1), 1e-16))


def gate(X, x, n, m, boundary, threshold):
    _, n2, ok = warp(X, x, n)
    return ~boundary & ok & (cosine(m, n2) > threshold)


def terms(X, x, n, c, m, adj, L, sw, lw, gamma, threshold):
    """Loss terms of one inner iteration: dict(v, w, data, stiff (= sw * the edge sum), lap (= lw * mean |Lv|), S,
    loss, Lv)."""
    v = warp(X, x)
    w = gate(X, x, n, m, adj["boundary"], threshold)
    data = float((w[:, None] * (v - c) ** 2).sum())
    G = np.array([1.0, 1.0, 1.0, gamma])
    e = adj["edges"]
    stiff = sw * float((((X[e[:, 0]] - X[e[:, 1]]) * G) ** 2).sum())
    Lv = L @ v
    lap = lw * float(np.linalg.norm(Lv, axis=1).sum()) / len(x)
    S = data + stiff
    return dict(v=v, w=w, data=data, stiff=stiff, lap=lap, S=S, loss=np.sqrt(S) + lap, Lv=Lv)


def gradient(X, x, n, c, m, adj, L, sw, lw, gamma, threshold):
    """Closed-form dloss/dX [V,3,4] (DESIGN 1f) and the terms."""
    t = terms(X, x, n, c, m, adj, L, sw, lw, gamma, threshold)
    V = len(x)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = 1.0 / (2.0 * np.sqrt(t["S"])) if t["S"] > 0 else np.inf
        nrm = np.linalg.norm(t["Lv"], axis=1, keepdims=True)
        u = np.where(nrm > 0, t["Lv"] / np.where(nrm > 0, nrm, 1.0), 0.0)
        dv = 2 * s * t["w"][:, None] * (t["v"] - c) + (lw / V) * (L.T @ u)
        xh = np.concatenate([x, np.ones((V, 1))], axis=1)
        G2 = np.array([1.0, 1.0, 1.0, gamma * gamma])
        e = adj["edges"]
        d = (X[e[:, 0]] - X[e[:, 1]]) * G2
        K = np.zeros_like(X)
        np.add.at(K, e[:, 0], d)
        np.add.at(K, e[:, 1], -d)
        g = dv[:, :, None] * xh[:, None, :] + 2 * s * sw * K
    return g, t


def adamw_step(X, g, state, step, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2):
    """torch.optim.AdamW(amsgrad=True)'s single-tensor step; state = (exp_avg, exp_avg_sq, max_exp_avg_sq), zeros at
    step 1.  Returns (X, state)."""
    b1, b2 = betas
    m1, m2, mx = state
    X = X * (1 - lr * weight_decay)
    m1 = m1 + (1 - b1) * (g - m1)
    m2 = m2 * b2 + (1 - b2) * g * g
    mx = np.maximum(mx, m2)
    denom = np.sqrt(mx) / np.sqrt(1 - b2 ** step) + eps
    return X - lr / (1 - b1 ** step) * m1 / denom, (m1, m2, mx)


def nearest(q, c):
    """Index of the nearest c for every q; the lower index on ties."""
    d = ((q[:, None, :] - c[None, :, :]) ** 2).sum(-1)
    return np.argmin(d, axis=1)


def fit(src_v, src_f, tgt_v, tgt_f, masks, epoch, inner_iter, stiffness_weight, laplacian_weight, mile_stone,
        gamma=1.0, threshold=0.5):
    """The fitting loop of NRICP_Optimizer_AdamW in float64.  Returns dict(epoch_v [E,V,3] at every epoch start, final_v,
    stats [E,6] = (avg_update, valid, data, stiffness, laplacian, total) of every epoch's last iteration)."""
    src_v, tgt_v = np.asarray(src_v, dtype=np.float64), np.asarray(tgt_v, dtype=np.float64)
    V = len(src_v)
    src_n = shade_oracle.vertex_normals(src_v[None], src_f)[0]
    tgt_n = shade_oracle.vertex_normals(tgt_v[None], tgt_f)[0]
    keep = np.asarray(masks) > 0
    tgt_v, tgt_n = tgt_v[keep], tgt_n[keep]
    adj = adjacency(src_f, V)
    L = laplacian(adj["edges"], V)
    X = identity_affine(V)
    mile_idx, mile_times = 0, 0
    epoch_v, stats = [], []
    new_v = warp(X, src_v)
    for i in range(epoch):
        old_v = new_v
        epoch_v.append(old_v)
        j = nearest(old_v, tgt_v)
        c, m = tgt_v[j], tgt_n[j]
        sw, lw = stiffness_weight[mile_idx], laplacian_weight[mile_idx]
        state = (np.zeros_like(X),) * 3
        for t in range(1, (100 if i == 0 else inner_iter) + 1):
            g, tm = gradient(X, src_v, src_n, c, m, adj, L, sw, lw, gamma, threshold)
            X, state = adamw_step(X, g, state, t)
        new_v = warp(X, src_v)
        stats.append([np.linalg.norm(old_v - new_v, axis=1).mean(), tm["w"].sum(), tm["data"], tm["stiff"],
                      tm["lap"], tm["loss"]])
        mile_times += 1
        if mile_times in mile_stone:
            mile_idx += 1
    return dict(epoch_v=np.stack(epoch_v), final_v=new_v, stats=np.array(stats))


# ---- torch float64 stand-ins with pytorch3d's call forms -----------------------------------------------------------

class Meshes:
    """The two members `mesh_laplacian_smoothing` reads: verts [1,V,3] and faces [1,F,3]."""

    def __init__(self, verts, faces):
        self.verts, self.faces = verts, faces


def laplacian_smoothing_torch(meshes, method="uniform"):
    """pytorch3d 0.4's `mesh_laplacian_smoothing(meshes, 'uniform')` for one mesh: (1/V) sum_i |(L v)_i| with the COO
    Laplacian of `laplacian`, differentiable in the vertices."""
    assert method == "uniform"
    v = meshes.verts[0]
    V = v.shape[0]
    adj = adjacency(meshes.faces[0].detach().cpu().numpy(), V)
    L = laplacian(adj["edges"], V).tocoo()
    Lt = torch.sparse_coo_tensor(np.stack([L.row, L.col]), L.data, (V, V), dtype=torch.float64)
    return torch.sparse.mm(Lt, v).norm(dim=1).sum() / V


def knn_points(p1, p2, K=1):
    """K = 1 `knn_points` of one cloud pair (float64 brute force, lower index on ties)."""
    assert K == 1 and p1.shape[0] == 1
    idx = nearest(p1[0].detach().cpu().numpy(), p2[0].detach().cpu().numpy())
    idx = torch.as_tensor(idx)[None, :, None]
    d = ((p1[0] - p2[0][idx[0, :, 0]]) ** 2).sum(-1)[None, :, None]
    return types.SimpleNamespace(dists=d, idx=idx, knn=None)


def knn_gather(x, idx):
    """x [1,P2,D], idx [1,P1,1] -> [1,P1,1,D]."""
    return x[:, idx[0, :, 0]][:, :, None]


def torch_loss(X, x, n, c, m, faces, boundary, sw, lw, gamma, threshold):
    """The reference's loss in torch float64 with the pytorch3d-form Laplacian, X [V,3,4] requiring grad."""
    A, b = X[:, :, :3], X[:, :, 3]
    v = (A @ x[:, :, None])[:, :, 0] + b
    with torch.no_grad():
        Ai = torch.linalg.inv(A)
        ok = torch.linalg.det(A).abs() >= 1e-4
        n2 = torch.where(ok[:, None], (Ai.transpose(1, 2) @ n[:, :, None])[:, :, 0], torch.zeros_like(n))
        cos = (m * n2).sum(-1) / torch.sqrt(torch.clamp_min((m * m).sum(-1) * (n2 * n2).sum(-1), 1e-16))
        w = ~boundary & ok & (cos > threshold)
    data = (w[:, None] * (v - c) ** 2).sum()
    adj = adjacency(faces.numpy(), len(x))
    e = torch.as_tensor(adj["edges"])
    G = torch.eye(4, dtype=X.dtype)
    G[3, 3] = gamma
    stiff = ((X[e[:, 0]] - X[e[:, 1]]) @ G).pow(2).sum() * sw
    lap = laplacian_smoothing_torch(Meshes(v[None], faces[None])) * lw
    return torch.sqrt(data + stiff) + lap
