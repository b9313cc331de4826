"""Float64 restatement of the point rasterizer and alpha compositor (DESIGN section 1c), written from the definitions:
every point is tested against every pixel centre near its disc.

Points come projected, [N,P,3] = (NDC x, NDC y, view z); pixel (row, col) has its centre at NDC
(1 - (2 col + 1)/W, 1 - (2 row + 1)/H).  A point with z < 0 (or a non-finite coordinate) is skipped; it covers a pixel
when d = (xf - x)^2 + (yf - y)^2 < r^2.  Per pixel the K covering points with the smallest (z, n*P + p) are kept,
sorted.  Composite (pytorch3d's AlphaCompositor, weights 1 - d/r^2): T_0 = 1, image[g] += f alpha T, T *= 1 - alpha,
g = 0 when p < split, else 1.  Backward (pytorch3d's, with the suffix sum):
dL/dalpha_t = sum_g G_g (f_t [g_t = g] T_t - S_{t,g} / (1 - alpha_t + 1e-9)), S_{t,g} = sum_{k>t} [g_k = g] f_k alpha_k T_k,
dL/dx_t += dL/dalpha_t 2 (xf - x_t) / r^2 (y alike); nothing reaches z.

Selections are kept sparse -- flat arrays sorted by (pixel, rank) -- so a 1080 x 1080 frame with K = 50 stays small.
A pixel is AMBIGUOUS at a given precision when some point's d lies within `margin * r^2` of r^2, or its K-th and
(K+1)-th depths differ by a nonzero amount within `ztol` relative (exact ties are decided by the index in any precision).
"""
from types import SimpleNamespace

import numpy as np
import torch


def project(points, cam, H, W):
    """[N,P,3] world points and [N,16] camera rows {fx, fy, px, py, R row-major, T} -> [N,P,3] float64 NDC points."""
    pts = np.asarray(points, dtype=np.float64)
    cam = np.asarray(cam, dtype=np.float64).reshape(-1, 16)
    out = np.empty_like(pts)
    for n in range(pts.shape[0]):
        c = cam[n if cam.shape[0] > 1 else 0]
        v = pts[n] @ c[4:13].reshape(3, 3) + c[13:16]
        with np.errstate(divide="ignore", invalid="ignore"):
            sx, sy = c[2] - c[0] * v[:, 0] / v[:, 2], c[3] - c[1] * v[:, 1] / v[:, 2]
        out[n] = np.stack([1 - (2 * sx + 1) / W, 1 - (2 * sy + 1) / H, v[:, 2]], 1)
    return out


def select(ndc, H, W, radius, K, margin=0.0, ztol=0.0, chunk=4_000_000):
    """Sparse selection of every frame: dict of flat arrays sorted by (pix, rank) -- pix (n*H*W + row*W + col), rank,
    idx (packed n*P + p), z, d -- and per-pixel count [N,H,W], ambiguous [N,H,W], skipped (points)."""
    ndc = np.asarray(ndc, dtype=np.float64)
    N, P = ndc.shape[:2]
    r2 = float(radius) ** 2
    x, y, z = (ndc[..., i].reshape(-1) for i in range(3))
    with np.errstate(invalid="ignore"):
        keep = (z >= 0) & np.isfinite(x) & np.isfinite(y)
    g_all = np.nonzero(keep)[0]
    frame = g_all // max(P, 1)
    # candidate pixels: the disc's bbox plus half a pixel, clipped to the image
    cx, cy = ((1 - x[g_all]) * W - 1) / 2, ((1 - y[g_all]) * H - 1) / 2
    rx, ry = radius * W / 2 + 0.5, radius * H / 2 + 0.5
    x0 = np.clip(np.floor(cx - rx), 0, W).astype(np.int64); x1 = np.clip(np.ceil(cx + rx), -1, W - 1).astype(np.int64)
    y0 = np.clip(np.floor(cy - ry), 0, H).astype(np.int64); y1 = np.clip(np.ceil(cy + ry), -1, H - 1).astype(np.int64)
    nx, ny = np.maximum(x1 - x0 + 1, 0), np.maximum(y1 - y0 + 1, 0)
    cnt = nx * ny
    amb = np.zeros(N * H * W, dtype=bool)
    parts = []
    csum = np.cumsum(cnt)
    start = 0
    while start < len(g_all):
        stop = max(int(np.searchsorted(csum, (csum[start - 1] if start else 0) + chunk, side="right")), start + 1)
        sl = np.arange(start, stop)
        c = cnt[sl]
        e = np.repeat(sl, c)
        k = np.arange(c.sum()) - np.repeat(np.cumsum(c) - c, c)
        col, row = x0[e] + k % nx[e], y0[e] + k // nx[e]
        g = g_all[e]
        d = ((1 - (2 * col + 1) / W) - x[g]) ** 2 + ((1 - (2 * row + 1) / H) - y[g]) ** 2
        pix = (frame[e] * H + row) * W + col
        if margin > 0:
            amb[pix[np.abs(d - r2) <= margin * r2]] = True
        cov = d < r2
        parts.append((pix[cov], z[g[cov]], g[cov], d[cov]))
        start = stop
    pix, zz, g, d = (np.concatenate([p[i] for p in parts]) if parts else np.zeros(0) for i in range(4))
    pix, g = pix.astype(np.int64), g.astype(np.int64)
    o = np.lexsort((g, zz, pix))
    pix, zz, g, d = pix[o], zz[o], g[o], d[o]
    first = np.ones(len(pix), dtype=bool)
    first[1:] = pix[1:] != pix[:-1]
    starts = np.nonzero(first)[0]
    rank = np.arange(len(pix)) - np.repeat(starts, np.diff(np.append(starts, len(pix))))
    # depth ambiguity between the K-th and the (K+1)-th
    nxt = rank == K
    nxt_of = np.nonzero(nxt)[0]
    if len(nxt_of):
        za, zb = zz[nxt_of - 1], zz[nxt_of]
        amb[pix[nxt_of][(zb - za > 0) & (zb - za <= ztol * np.abs(za))]] = True
    sel = rank < K
    count = np.bincount(pix[sel], minlength=N * H * W)
    return dict(pix=pix[sel], rank=rank[sel], idx=g[sel], z=zz[sel], d=d[sel], count=count.reshape(N, H, W),
                ambiguous=amb.reshape(N, H, W), skipped=int(N * P - keep.sum()), N=N, P=P, H=H, W=W, K=K)


def dense(sel):
    """Fragments of a selection in pytorch3d's layout: idx [N,H,W,K] int64, zbuf, dists, padded with -1 (small images
    only)."""
    N, H, W, K = sel["N"], sel["H"], sel["W"], sel["K"]
    idx = -np.ones(N * H * W * K, dtype=np.int64)
    zb, ds = -np.ones(N * H * W * K), -np.ones(N * H * W * K)
    flat = sel["pix"] * K + sel["rank"]
    idx[flat], zb[flat], ds[flat] = sel["idx"], sel["z"], sel["d"]
    return idx.reshape(N, H, W, K), zb.reshape(N, H, W, K), ds.reshape(N, H, W, K)


def _group(sel, split):
    return np.where(sel["idx"] % max(sel["P"], 1) < split, 0, 1)


def _weights(sel, radius, features):
    f = np.ones(len(sel["idx"])) if features is None else np.asarray(features, np.float64).reshape(-1)[sel["idx"]]
    return f, 1 - sel["d"] / float(radius) ** 2


def _transmittance(sel, alpha):
    """T_k of every entry: the product of (1 - alpha) over the entries before it in its pixel."""
    T = np.ones(sel["N"] * sel["H"] * sel["W"])
    Tk = np.empty(len(alpha))
    for k in range(sel["K"]):
        m = sel["rank"] == k
        if not m.any():
            break
        Tk[m] = T[sel["pix"][m]]
        T[sel["pix"][m]] *= 1 - alpha[m]
    return Tk


def composite(sel, radius, features=None, split=None, G=1):
    """images [G,N,H,W] of a selection; split None = every point in image 0."""
    f, alpha = _weights(sel, radius, features)
    Tk = _transmittance(sel, alpha)
    grp = np.zeros(len(f), dtype=np.int64) if split is None else _group(sel, split)
    img = np.zeros((G, sel["N"] * sel["H"] * sel["W"]))
    np.add.at(img, (grp, sel["pix"]), f * alpha * Tk)
    return img.reshape(G, sel["N"], sel["H"], sel["W"])


def composite_grad(sel, ndc, radius, grad_images, features=None, split=None):
    """grad [N,P,3] of sum(grad_images * composite(...)) w.r.t. the NDC points with the selection held fixed, by the
    closed-form backward above (O(K) per pixel)."""
    ndc = np.asarray(ndc, dtype=np.float64)
    N, P, H, W, K = sel["N"], sel["P"], sel["H"], sel["W"], sel["K"]
    r2 = float(radius) ** 2
    Gi = np.asarray(grad_images, dtype=np.float64).reshape(-1, N * H * W)
    G = Gi.shape[0]
    f, alpha = _weights(sel, radius, features)
    Tk = _transmittance(sel, alpha)
    grp = np.zeros(len(f), dtype=np.int64) if split is None else _group(sel, split)
    pix = sel["pix"]
    S = np.zeros((G, N * H * W))
    da = np.zeros(len(f))
    for k in range(K - 1, -1, -1):
        m = np.nonzero(sel["rank"] == k)[0]
        if not len(m):
            continue
        p = pix[m]
        rest = sum(Gi[gg, p] * S[gg, p] for gg in range(G))
        da[m] = Gi[grp[m], p] * f[m] * Tk[m] - rest / (1 - alpha[m] + 1e-9)
        np.add.at(S, (grp[m], p), f[m] * alpha[m] * Tk[m])
    q = pix % (H * W)
    xf, yf = 1 - (2 * (q % W) + 1) / W, 1 - (2 * (q // W) + 1) / H
    pts = ndc.reshape(-1, 3)[sel["idx"]]
    out = np.zeros((N * P, 3))
    np.add.at(out, (sel["idx"], 0), da * 2 * (xf - pts[:, 0]) / r2)
    np.add.at(out, (sel["idx"], 1), da * 2 * (yf - pts[:, 1]) / r2)
    return out.reshape(N, P, 3)


def composite_torch(sel, ndc, radius, features=None, split=None, G=1):
    """composite() as a torch graph of the NDC points (any dtype, e.g. float64 with requires_grad), the selection held
    fixed: for autograd and finite-difference checks of composite_grad."""
    N, H, W, K = sel["N"], sel["H"], sel["W"], sel["K"]
    pix = torch.as_tensor(sel["pix"])
    q = pix % (H * W)
    xf = 1 - (2 * (q % W) + 1).to(ndc.dtype) / W
    yf = 1 - (2 * (q // W) + 1).to(ndc.dtype) / H
    pts = ndc.reshape(-1, 3)[torch.as_tensor(sel["idx"])]
    alpha = 1 - ((xf - pts[:, 0]) ** 2 + (yf - pts[:, 1]) ** 2) / radius ** 2
    f = torch.ones_like(alpha) if features is None else torch.as_tensor(features, dtype=ndc.dtype).reshape(-1)[
        torch.as_tensor(sel["idx"])]
    rank = torch.as_tensor(sel["rank"])
    T = torch.ones(N * H * W, dtype=ndc.dtype)
    grp = torch.zeros(len(pix), dtype=torch.long) if split is None else torch.as_tensor(_group(sel, split))
    img = torch.zeros(G * N * H * W, dtype=ndc.dtype)
    for k in range(K):
        m = torch.nonzero(rank == k)[:, 0]
        if not len(m):
            break
        p = pix[m]
        img = img.index_add(0, grp[m] * N * H * W + p, f[m] * alpha[m] * T[p])
        T = T.index_put((p,), T[p] * (1 - alpha[m]))
    return img.view(G, N, H, W)


def alpha_compositor(pointsidx, alphas, features, **kwargs):
    """pytorch3d's AlphaCompositor (background_color None) in float64 loops over K: pointsidx [N,K,H,W] (-1 = none),
    alphas [N,K,H,W], features [C,P_packed] -> images [N,C,H,W]."""
    idx = pointsidx.long()
    N, K, H, W = idx.shape
    C = features.shape[0]
    out = torch.zeros((N, C, H, W), dtype=torch.float64)
    T = torch.ones((N, H, W), dtype=torch.float64)
    for k in range(K):
        i = idx[:, k]
        valid = i >= 0
        a = torch.where(valid, alphas[:, k].double(), torch.zeros((), dtype=torch.float64))
        f = features.double()[:, i.clamp_min(0)].permute(1, 0, 2, 3)          # [N,C,H,W]
        out = out + f * (a * T)[:, None]
        T = T * (1 - a)
    return out


class Rasterizer:
    """A pytorch3d-style PointsRasterizer over this oracle for already-projected points: __call__(clouds) -> fragments
    with idx / zbuf / dists [N,H,W,K] torch tensors and .raster_settings.radius (what the reference's renderers read)."""

    def __init__(self, H, W, radius, K):
        self.raster_settings = SimpleNamespace(image_size=(H, W), radius=radius, points_per_pixel=K)

    def __call__(self, point_clouds, **kwargs):
        s = self.raster_settings
        ndc = point_clouds.points_padded().double().numpy()
        i, z, d = dense(select(ndc, s.image_size[0], s.image_size[1], s.radius, s.points_per_pixel))
        return SimpleNamespace(idx=torch.as_tensor(i), zbuf=torch.as_tensor(z), dists=torch.as_tensor(d))
