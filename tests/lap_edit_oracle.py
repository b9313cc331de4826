"""Float64 oracle of the Laplacian-editing rules of DESIGN section 1g: the solve of `Laplacian_Optimizer`
(engineer/optimizer/lap_deform_optimizer.py:25-186), argmin_y |L y - L x|^2 + c |P y - u|^2, with L pytorch3d 0.4's
uniform Laplacian as tests/nricp_oracle.py builds it.

- `solve`: the normal equations A y = b, A = L^T L + c P^T P, b = L^T L x + c P^T u, by scipy's sparse direct solve on
  every connected component that holds a constraint; a component without one keeps y = x (A is singular there, and
  CG from y0 = x does not move it).
- `dense_reference`: the reference's own formula, inv(L^T W L) L^T W t with L stacked over the COO constraint rows and
  W = diag(1, .., 1, c, .., c), for small meshes where every component is constrained.
- `smooth`: the reference's smoothing, the Laplacian with its diagonal zeroed.
- `pcg`: a NumPy restatement of csrc/lap_edit.cu's Jacobi-preconditioned CG: the same setup, the same per-column
  lockstep iteration, chunked partial sums over 256 vertices and the same stop rule.
- `Template` / `fit`: a garment-template stand-in with what `fitting` reads, and the fitting loop restated on `solve`.
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as sla
import torch
from scipy.optimize import linear_sum_assignment
from scipy.sparse.csgraph import connected_components

import nricp_oracle as no

CHUNK = 256


def laplacian(faces, V):
    """(L scipy CSR [V,V], adjacency dict of nricp_oracle) for faces [F,3] over V vertices."""
    adj = no.adjacency(faces, V)
    return no.laplacian(adj["edges"], V), adj


def constraints(cidx, ctgt, V):
    """Keep the constraints with an index in [0, V): (idx [m], targets [m,3], skipped count)."""
    cidx = np.asarray(cidx, dtype=np.int64).reshape(-1)
    ctgt = np.asarray(ctgt, dtype=np.float64).reshape(-1, 3)
    ok = (cidx >= 0) & (cidx < V)
    return cidx[ok], ctgt[ok], int((~ok).sum())


def normal_equations(x, L, cidx, ctgt, c):
    """(A CSR, b [V,3]) with P the selection rows of the valid constraints, one per entry (duplicates included)."""
    V = L.shape[0]
    idx, u, _ = constraints(cidx, ctgt, V)
    P = sp.csr_matrix((np.ones(len(idx)), (np.arange(len(idx)), idx)), shape=(len(idx), V))
    A = (L.T @ L + c * (P.T @ P)).tocsr()
    b = L.T @ (L @ x) + c * (P.T @ u)
    return A, b


def solve(x, faces, cidx, ctgt, c=1.0, smooth_out=False):
    """y [V,3] float64: the solution on every component with a constraint, x on the others; smoothed when asked."""
    x = np.asarray(x, dtype=np.float64)
    V = len(x)
    L, adj = laplacian(faces, V)
    A, b = normal_equations(x, L, cidx, ctgt, c)
    idx, _, _ = constraints(cidx, ctgt, V)
    rows = np.repeat(np.arange(V), adj["deg"])
    G = sp.csr_matrix((np.ones(len(rows)), (rows, adj["col"])), shape=(V, V))
    _, comp = connected_components(G, directed=False)
    held = np.zeros(comp.max() + 1 if V else 0, dtype=bool)
    held[comp[idx]] = True
    free = held[comp] if V else np.zeros(0, dtype=bool)
    y = x.copy()
    if free.any():
        fi = np.flatnonzero(free)
        fx = np.flatnonzero(~free)
        Aff = A[fi][:, fi].tocsc()
        rhs = b[fi] - A[fi][:, fx] @ x[fx]
        y[fi] = sla.spsolve(Aff, rhs).reshape(-1, 3)
    return smooth(y, L) if smooth_out else y


def dense_reference(x, faces, cidx, ctgt, c=1.0, smooth_out=False):
    """The reference's solver and smoothing, densely in float64 (every index in range)."""
    x = np.asarray(x, dtype=np.float64)
    V = len(x)
    L, _ = laplacian(faces, V)
    Ld = L.toarray()
    cidx = np.asarray(cidx, dtype=np.int64)
    C = np.zeros((len(cidx), V))
    np.add.at(C, (np.arange(len(cidx)), cidx), 1.0)
    Lf = np.concatenate([Ld, C])
    W = np.diag(np.concatenate([np.ones(V), np.full(len(cidx), float(c))]))
    t = np.concatenate([Ld @ x, np.asarray(ctgt, dtype=np.float64)])
    y = np.linalg.inv(Lf.T @ W @ Lf) @ Lf.T @ W @ t
    if smooth_out:
        np.fill_diagonal(Ld, 0.0)
        y = Ld @ y
    return y


def smooth(y, L):
    """The reference's smoothing: L with its diagonal zeroed, times y (an isolated vertex goes to 0)."""
    Z = L.tolil()
    Z.setdiag(0.0)
    return Z.tocsr() @ y


def _csum(v):
    """Column sums of v [V,3] as the kernel forms them: per 256-vertex chunk, then over the chunks in order."""
    V = len(v)
    nc = max((V + CHUNK - 1) // CHUNK, 1)
    pad = np.zeros((nc * CHUNK, 3))
    pad[:V] = v
    return pad.reshape(nc, CHUNK, 3).sum(axis=1).sum(axis=0)


def pcg(x, faces, cidx, ctgt, c=1.0, tol=1e-10, max_iter=50000, smooth_out=False):
    """The kernel's algorithm in NumPy: (y [V,3], stats [8] as recmv_lap_edit_solve writes them)."""
    x = np.asarray(x, dtype=np.float64)
    V = len(x)
    L, _ = laplacian(faces, V)
    idx, u, skipped = constraints(cidx, ctgt, V)
    cnt = np.bincount(idx, minlength=V).astype(np.float64)
    su = np.zeros((V, 3))
    np.add.at(su, idx, u)
    b = L.T @ (L @ x) + c * su
    diag = np.asarray(L.multiply(L).sum(axis=0)).ravel() + c * cnt   # column sums of squares, duplicates summed
    dinv = np.where(diag > 0, 1.0 / np.where(diag > 0, diag, 1.0), 0.0)[:, None]
    y = x.copy()
    r = c * (su - cnt[:, None] * x)
    p = dinv * r
    bb, rz, rr = _csum(b * b), _csum(r * p), _csum(r * r)
    tol2 = tol * tol
    finite = np.isfinite(rr) & np.isfinite(bb)
    nonfinite = not finite.all()
    active = finite & ~(rr <= tol2 * bb)
    iters = np.zeros(3, dtype=np.int64)
    with np.errstate(all="ignore"):
        for _ in range(max_iter):
            if not active.any():
                break
            w = L @ p
            q = L.T @ w + (c * cnt)[:, None] * p
            alpha = rz / _csum(p * q)
            a = active
            y[:, a] += alpha[a] * p[:, a]
            r[:, a] -= alpha[a] * q[:, a]
            z = dinv * r
            rz_new, rr_new = _csum(np.where(a, r * z, 0.0)), _csum(np.where(a, r * r, 0.0))
            iters[a] += 1
            rr[a] = rr_new[a]
            bad = a & ~np.isfinite(rr)
            done = a & np.isfinite(rr) & (rr <= tol2 * bb)
            nonfinite = nonfinite or bad.any()
            active = a & ~bad & ~done
            beta = np.where(active, rz_new / np.where(active, rz, 1.0), 0.0)
            rz = np.where(active, rz_new, rz)
            p[:, active] = z[:, active] + beta[active] * p[:, active]
        rel = np.sqrt(np.where(bb > 0, rr / np.where(bb > 0, bb, 1.0), rr))
    converged = bool((rr <= tol2 * bb).all())
    flag = -1.0 if nonfinite else (1.0 if converged else 0.0)
    stats = np.concatenate([iters, rel, [flag, skipped]]).astype(np.float64)
    return (smooth(y, L) if smooth_out else y), stats


# ---- the fitting loop ------------------------------------------------------------------------------------------------

def subsample(n_target, n_source):
    """The reference's target sub-sampling, torch.arange(0, T, (T - 1) / S).long(), in float64."""
    return torch.arange(0, n_target, (n_target - 1) / n_source, dtype=torch.float64).long().numpy()


def best_match(vertices, fields, targets):
    """The reference's GarmentMesh.best_match (engineer/utils/garment_structure.py:647-723) on plain arrays: per field,
    the sub-sampled target curve, a linear assignment on squared distances and the cosine > 0.5 filter of the centred
    points.  vertices [V,3]; fields {name: vertex indices}; targets {name: [T,3]} -> (source_idx [m], target [m,3])."""
    idx_out, tgt_out = [], []
    for name, fidx in fields.items():
        s = np.asarray(vertices, dtype=np.float64)[fidx]
        t = np.asarray(targets[name], dtype=np.float64)
        t = t[subsample(len(t), len(s))]
        d = ((s[:, None, :] - t[None, :, :]) ** 2).sum(-1)
        si, ti = linear_sum_assignment(d)
        sn = s - s.mean(axis=0)
        tn = (t - t.mean(axis=0))[ti]
        cos = ((sn * tn) / (np.linalg.norm(sn, axis=1, keepdims=True) * np.linalg.norm(tn, axis=1, keepdims=True))).sum(-1)
        keep = cos > 0.5
        idx_out.append(np.asarray(fidx)[si[keep]])
        tgt_out.append(t[ti[keep]])
    return np.concatenate(idx_out), np.concatenate(tgt_out)


class Template:
    """The members of a garment template that `Laplacian_Optimizer.fitting` reads: vertices, faces, device,
    laplacian_packed, best_match, static_pts_match and update_vertices.  `matches` records every best_match call."""

    def __init__(self, vertices, faces, fields, dtype=torch.float64, device="cpu"):
        self.device = torch.device(device)
        self.dtype = dtype
        self.vertices = torch.as_tensor(np.asarray(vertices), dtype=dtype, device=self.device)
        self.faces = torch.as_tensor(np.asarray(faces), dtype=torch.int64, device=self.device)
        self.fields = {k: np.asarray(v, dtype=np.int64) for k, v in fields.items()}
        self.matches = []   # (vertices, source_idx, target) of every best_match call
        self.updates = 0

    def laplacian_packed(self):
        L, _ = laplacian(self.faces.cpu().numpy(), self.vertices.shape[0])
        L = L.tocoo()
        return torch.sparse_coo_tensor(np.stack([L.row, L.col]), L.data, L.shape, dtype=self.dtype, device=self.device)

    def best_match(self, target, device, is_outlayer=False):
        t = {k: v.detach().cpu().numpy() for k, v in target.items()}
        v = self.vertices.detach().cpu().numpy().astype(np.float64)
        idx, tgt = best_match(v, self.fields, t)
        self.matches.append((v, idx, tgt))
        return torch.as_tensor(idx, device=device), torch.as_tensor(tgt, dtype=torch.float32, device=device)

    def static_pts_match(self):
        return None

    def update_vertices(self, new_vertices):
        self.vertices = new_vertices.to(self.vertices)
        self.updates += 1


class Curve:
    """A target feature curve: what `fitting` reads of a pytorch3d Meshes / Pointclouds."""

    def __init__(self, verts):
        self.v = verts

    def verts_packed(self):
        return self.v


def fit(vertices, faces, fields, targets, epoch=3, c=1.0, smooth_out=True):
    """The fitting loop on `solve`: per epoch, match then solve.  Returns dict(epoch_v [E,V,3] at every epoch start,
    idx / tgt lists of every epoch's constraints, final_v)."""
    v = np.asarray(vertices, dtype=np.float64)
    tg = {k: np.asarray(t, dtype=np.float64) for k, t in targets.items()}
    epoch_v, idxs, tgts = [], [], []
    for _ in range(epoch):
        epoch_v.append(v)
        idx, tgt = best_match(v, fields, tg)
        tgt = tgt.astype(np.float32).astype(np.float64)   # the template hands the targets over in fp32
        idxs.append(idx)
        tgts.append(tgt)
        v = solve(v, faces, idx, tgt, c, smooth_out)
    return dict(epoch_v=np.stack(epoch_v), idx=idxs, tgt=tgts, final_v=v)


# ---- scenes ----------------------------------------------------------------------------------------------------------

def tube(nt, nz, radius=0.3, height=1.5, jitter=0.0, seed=0):
    """An open tube of nt x nz vertices (ring-major: vertex i * nz + j is ring position i at height j), its faces, and
    the waist (top) and hem (bottom) loops."""
    g = np.random.default_rng(seed)
    th = np.linspace(0, 2 * np.pi, nt, endpoint=False)
    z = np.linspace(0, height, nz)
    T, Z = np.meshgrid(th, z, indexing="ij")
    if jitter:
        T = T + jitter * (2 * np.pi / nt) * g.uniform(-1, 1, T.shape)
        Z = Z + jitter * (height / nz) * g.uniform(-1, 1, Z.shape) * ((np.arange(nz) > 0) & (np.arange(nz) < nz - 1))
    rad = radius * (1.0 + 0.5 * (1.0 - Z / height))   # wider at the hem: skirt-like
    v = np.stack([(rad * np.cos(T)).ravel(), (rad * np.sin(T)).ravel(), Z.ravel()], 1)
    # quad (i, j) gives faces (a, b, c) and (a, c, d), in i-major then j order
    I, J = np.meshgrid(np.arange(nt), np.arange(nz - 1), indexing="ij")
    a, b = I * nz + J, ((I + 1) % nt) * nz + J
    f = np.stack([np.stack([a, b, b + 1], -1), np.stack([a, b + 1, a + 1], -1)], axis=2).reshape(-1, 3)
    hem = np.arange(nt) * nz
    waist = np.arange(nt) * nz + nz - 1
    return v, f.astype(np.int64), dict(waist=waist, hem=hem)


def loop_targets(v, loops):
    """Displaced and scaled copies of the boundary loops of a tube (the probe scene of tools/bench_lap_edit.py): the hem
    widened by 1.3, the waist raised by 0.1, and a wave in x.  (cidx [m], ctgt [m,3])."""
    waist, hem = loops["waist"], loops["hem"]
    cidx = np.concatenate([hem, waist])
    u = v[cidx].copy()
    n = len(hem)
    u[:n, :2] *= 1.3
    u[n:, 2] += 0.1
    u[:, 0] += 0.05 * np.sin(3 * np.arange(len(cidx)))
    return cidx, u
