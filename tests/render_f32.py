"""Float32 restatement of the image-space kernels: the mesh rasterizer (csrc/raster_common.cuh, csrc/raster.cu) and the
point rasterizer's forward and backward (csrc/points_raster.cu).

Every operation that decides coverage or produces a value in those kernels is explicitly rounded (__fadd_rn, __fmul_rn,
__fdiv_rn, __fsub_rn), so no contraction can change them.  NumPy float32 arithmetic rounds each ufunc on its own, without
FMA, so restating the kernels' operation order here gives their outputs bit for bit.  Each step below cites the line it
restates.  Written from the documented operation order; no kernel is called.

Also here: running error bounds (class Rb) that carry, next to a float64 value, the bound S of the float32 evaluation
of the same operation order, in units of the float32 unit roundoff u = 2^-24: |fl32(expr) - expr| <= ~S u to first
order.  The float32-vs-float64 tests hold every output to kappa u S entry by entry.
"""
import numpy as np

f32 = np.float32
U = 2.0 ** -24
TINY = 2.0 ** -126          # 2^-150, the largest rounding error of an underflowing float32 result, in units of U
TILE_W, TILE_H = 32, 8


def _f(x):
    return np.asarray(x, dtype=np.float32)


# ---- mesh -----------------------------------------------------------------------------------------------------------
def project_face(verts, faces, cam):
    """raster_common.cuh:26-45 for one frame: verts [V,3] f32, faces [F,3] int64, cam [16] f32 -> (sx, sy, z) [F,3] f32
    and bad [F] (an index outside [0, V))."""
    verts, cam = _f(verts), _f(cam)
    V = verts.shape[0]
    faces = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    bad = ((faces < 0) | (faces >= V)).any(1)
    vi = np.where(faces < 0, 0, np.where(faces >= V, 0, faces))
    p = verts[vi] if V else np.zeros(faces.shape + (3,), np.float32)          # [F,3,3]
    X, Y, Z = p[..., 0], p[..., 1], p[..., 2]
    # :39-40  ((X c[4+j] + Y c[7+j]) + Z c[10+j]) + c[13+j], one rounding each
    v = [((X * cam[4 + j]) + (Y * cam[7 + j]) + (Z * cam[10 + j])) + cam[13 + j] for j in range(3)]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        sx = cam[2] - (cam[0] * v[0]) / v[2]                                   # :42
        sy = cam[3] - (cam[1] * v[1]) / v[2]                                   # :43
    z = v[2]
    zero = f32(0)
    sx, sy, z = (np.where(bad[:, None], zero, a) for a in (sx, sy, z))      # :33
    return sx.astype(np.float32), sy.astype(np.float32), z.astype(np.float32), bad


def edge_fn(ax, ay, bx, by, cx, cy):
    """raster_common.cuh:47-50: (b - a) x (c - a)."""
    return ((bx - ax) * (cy - ay)) - ((by - ay) * (cx - ax))


def make_face_rec(verts, faces, cam, H, W, z_clip, area_eps):
    """raster_common.cuh:70-108 for every face of one frame.  Returns dict of [F] / [F,3] arrays: keep (not skipped),
    x0, x1, y0, y1 (int64, x1 < x0 when no pixel centre is covered), ka, kb, kc, iz, z."""
    sx, sy, z, bad = project_face(verts, faces, cam)
    F = sx.shape[0]
    z_clip, area_eps = f32(z_clip), f32(area_eps)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        keep = ~bad & (z > z_clip).all(1)                                                   # :78
        A = edge_fn(sx[:, 0], sy[:, 0], sx[:, 1], sy[:, 1], sx[:, 2], sy[:, 2])            # :79
        keep &= np.abs(A) > area_eps                                                        # :80
        xmin = np.fmin(np.fmin(sx[:, 0], sx[:, 1]), sx[:, 2])                               # :82-83
        xmax = np.fmax(np.fmax(sx[:, 0], sx[:, 1]), sx[:, 2])
        ymin = np.fmin(np.fmin(sy[:, 0], sy[:, 1]), sy[:, 2])
        ymax = np.fmax(np.fmax(sy[:, 0], sy[:, 1]), sy[:, 2])
        fx0 = np.ceil(np.fmax(xmin, f32(0))); fx1 = np.floor(np.fmin(xmax, f32(W - 1)))     # :85-86
        fy0 = np.ceil(np.fmax(ymin, f32(0))); fy1 = np.floor(np.fmin(ymax, f32(H - 1)))
        vis = keep & (xmax >= 0) & (ymax >= 0) & (xmin <= f32(W - 1)) & (ymin <= f32(H - 1)) & (fx0 <= fx1) \
            & (fy0 <= fy1)                                                                  # :87
    x0 = np.where(vis, np.nan_to_num(fx0), 0).astype(np.int64); x1 = np.where(vis, np.nan_to_num(fx1), -1).astype(np.int64)
    y0 = np.where(vis, np.nan_to_num(fy0), 0).astype(np.int64); y1 = np.where(vis, np.nan_to_num(fy1), -1).astype(np.int64)
    ox, oy = x0.astype(np.float32), y0.astype(np.float32)                                   # :89
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        ex, ey = sx - ox[:, None], sy - oy[:, None]                                         # :92
        Ar = edge_fn(ex[:, 0], ey[:, 0], ex[:, 1], ey[:, 1], ex[:, 2], ey[:, 2])            # :93
        inv = f32(1) / Ar                                                                   # :94
        ka, kb, kc = (np.zeros((F, 3), np.float32) for _ in range(3))
        for i in range(3):                                                                  # :96-105
            a, b = (i + 1) % 3, (i + 2) % 3
            dx, dy = ex[:, b] - ex[:, a], ey[:, b] - ey[:, a]
            ka[:, i] = (-dy) * inv
            kb[:, i] = dx * inv
            kc[:, i] = ((dy * ex[:, a]) - (dx * ey[:, a])) * inv
        iz = f32(1) / z
    return dict(keep=keep, vis=vis, x0=x0, x1=x1, y0=y0, y1=y1, ka=ka, kb=kb, kc=kc, iz=iz, z=z, sx=sx, sy=sy, A=A)


def shade(ka, kb, kc, iz, z, qx, qy):
    """raster_common.cuh:54-65, vectorised over rows: returns (covered, bp [M,3], zb [M])."""
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        b = [((ka[:, i] * qx) + (kb[:, i] * qy)) + kc[:, i] for i in range(3)]             # :57
        cov = (b[0] >= 0) & (b[1] >= 0) & (b[2] >= 0)                                       # :58
        w = [b[i] * iz[:, i] for i in range(3)]                                             # :59
        s = (w[0] + w[1]) + w[2]                                                            # :60
        cov &= s > 0                                                                        # :61
        bp = np.stack([w[i] / s for i in range(3)], 1)                                      # :62
        zb = ((bp[:, 0] * z[:, 0]) + (bp[:, 1] * z[:, 1])) + (bp[:, 2] * z[:, 2])           # :63
    return cov, bp.astype(np.float32), zb.astype(np.float32)


def _enumerate(x0, x1, y0, y1, ids, chunk=4_000_000):
    """Yield (id, col, row) of every pixel in the bboxes of `ids`, row-major per bbox, in chunks."""
    nx, ny = x1[ids] - x0[ids] + 1, y1[ids] - y0[ids] + 1
    cnt = nx * ny
    csum = np.cumsum(cnt)
    start = 0
    while start < len(ids):
        stop = max(int(np.searchsorted(csum, (csum[start - 1] if start else 0) + chunk, side="right")), start + 1)
        c = cnt[start:stop]
        e = np.repeat(np.arange(start, stop), c)
        k = np.arange(int(c.sum())) - np.repeat(np.cumsum(c) - c, c)
        yield ids[e], x0[ids[e]] + k % nx[e], y0[ids[e]] + k // nx[e]
        start = stop


def tiles_of(x0, x1, y0, y1):
    """Tiles a bbox touches (raster.cu:63-66, points_raster.cu:81-82): count per bbox, 0 when x1 < x0."""
    return np.where(x1 >= x0, (x1 // TILE_W - x0 // TILE_W + 1) * (y1 // TILE_H - y0 // TILE_H + 1), 0)


def tile_hist(x0, x1, y0, y1, H, W):
    """Records per tile of one frame [tiles_y, tiles_x] for bboxes x0..y1 (x1 < x0 = none)."""
    ty, tx = (H + TILE_H - 1) // TILE_H, (W + TILE_W - 1) // TILE_W
    hist = np.zeros((ty, tx), np.int64)
    for i in np.nonzero(x1 >= x0)[0]:
        hist[y0[i] // TILE_H:y1[i] // TILE_H + 1, x0[i] // TILE_W:x1[i] // TILE_W + 1] += 1
    return hist


def rasterize_meshes(verts, faces, cams, H, W, z_clip=1e-6, area_eps=1e-8):
    """recmv_rasterize_meshes without dists: verts [N,V,3] f32, faces [F,3], cams [N,16] f32 -> dict of pix_to_face
    [N,H,W] int64 (packed n F + f), zbuf [N,H,W] f32, bary [N,H,W,3] f32 (-1 on background), skipped, pairs, covered
    and the per-frame records (recs)."""
    verts, cams = _f(verts), _f(cams).reshape(-1, 16)
    faces = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    N, F = verts.shape[0], faces.shape[0]
    p2f = np.full((N, H * W), -1, np.int64)
    zbuf = np.full((N, H * W), -1, np.float32)
    bary = np.full((N, H * W, 3), -1, np.float32)
    skipped = pairs = 0
    recs = []
    for n in range(N):
        r = make_face_rec(verts[n], faces, cams[n], H, W, z_clip, area_eps)
        recs.append(r)
        skipped += int((~r["keep"]).sum())
        pairs += int(tiles_of(r["x0"], r["x1"], r["y0"], r["y1"]).sum())
        ids = np.nonzero(r["vis"])[0]
        P_, G_, Z_ = [], [], []
        for f, col, row in _enumerate(r["x0"], r["x1"], r["y0"], r["y1"], ids):
            qx, qy = (col - r["x0"][f]).astype(np.float32), (row - r["y0"][f]).astype(np.float32)   # raster.cu:135
            cov, _, zb = shade(r["ka"][f], r["kb"][f], r["kc"][f], r["iz"][f], r["z"][f], qx, qy)
            cov &= ~np.isnan(zb)          # raster.cu:137: a NaN depth never compares below the running best
            P_.append((row * W + col)[cov]); G_.append(f[cov]); Z_.append(zb[cov])
        if not P_:
            continue
        pix, g, zb = np.concatenate(P_), np.concatenate(G_), np.concatenate(Z_)
        # raster.cu:137: the lexicographic minimum of (zbuf, packed face); -0 == +0 as floats
        o = np.lexsort((g, zb.astype(np.float64) + 0.0, pix))
        pix, g = pix[o], g[o]
        first = np.ones(len(pix), bool)
        first[1:] = pix[1:] != pix[:-1]
        pix, g = pix[first], g[first]
        # raster.cu:161: the winner re-shaded from its record
        col, row = pix % W, pix // W
        _, bp, zw = shade(r["ka"][g], r["kb"][g], r["kc"][g], r["iz"][g], r["z"][g],
                          (col - r["x0"][g]).astype(np.float32), (row - r["y0"][g]).astype(np.float32))
        p2f[n, pix] = n * F + g
        zbuf[n, pix] = zw
        bary[n, pix] = bp
    return dict(pix_to_face=p2f.reshape(N, H, W), zbuf=zbuf.reshape(N, H, W), bary=bary.reshape(N, H, W, 3),
                skipped=skipped, pairs=pairs, covered=int((p2f >= 0).sum()), recs=recs)


# ---- points ---------------------------------------------------------------------------------------------------------
def pixel_ndc(i, size):
    """points_raster.cu:46-48."""
    return f32(1) - (np.asarray(2 * np.asarray(i) + 1).astype(np.float32) / f32(size))


def dist2(xf, yf, x, y):
    """points_raster.cu:50-53."""
    dx, dy = xf - x, yf - y
    return (dx * dx) + (dy * dy)


def alpha_of(d, r2):
    """points_raster.cu:55."""
    return f32(1) - (d / r2)


def fma32(a, b, c):
    """Correctly rounded float32 a * b + c (one rounding, as an FMA).  The product of two float32 values is exact in
    float64; the float64 sum s and its exact error e (TwoSum) give a * b + c = s + e exactly, and rounding s to float32
    is correct except when s lies exactly halfway between two float32 values and e != 0, where e decides."""
    a, b, c = (np.asarray(x, np.float32).astype(np.float64) for x in (a, b, c))
    p = a * b
    s = p + c
    bp = s - c
    e = (p - bp) + (c - (s - bp))                                  # TwoSum: p + c = s + e exactly
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        other = np.nextafter(r, np.where(s > r64, np.float32(np.inf), np.float32(-np.inf))).astype(np.float64)
        half = (s != r64) & (2 * s == r64 + other) & (e != 0)
        toward_other = np.sign(e) == np.sign(other - s)
    return np.where(half & toward_other, other.astype(np.float32), r).astype(np.float32)


def setup_bbox(x, y, H, W, radius, fma_cx=False, fma_rx=False):
    """The setup kernel's disc bbox (points_raster.cu:75-80) with each contractible product-sum evaluated either as two
    roundings or as one (fused multiply-add): returns (x0, x1, y0, y1) int64 and `on` (the bbox meets the image).
    0.5 * t and 0.5 * radius are exact, so these two choices are all a compiler can change."""
    x, y, radius = _f(x), _f(y), f32(radius)

    def prod_sum(a, b, c, fused):
        return fma32(a, b, c) if fused else (a * b) + c

    with np.errstate(invalid="ignore", over="ignore"):
        cx = f32(0.5) * prod_sum(f32(1) - x, f32(W), f32(-1), fma_cx)
        cy = f32(0.5) * prod_sum(f32(1) - y, f32(H), f32(-1), fma_cx)
        rx = prod_sum(f32(0.5) * radius, f32(W), f32(0.01), fma_rx)
        ry = prod_sum(f32(0.5) * radius, f32(H), f32(0.01), fma_rx)
        lx, hx, ly, hy = np.floor(cx - rx), np.ceil(cx + rx), np.floor(cy - ry), np.ceil(cy + ry)
        on = (hx >= 0) & (lx <= W - 1) & (hy >= 0) & (ly <= H - 1)
    x0 = np.where(on, np.fmax(np.nan_to_num(lx), 0), 0).astype(np.int64)
    x1 = np.where(on, np.fmin(np.nan_to_num(hx), W - 1), -1).astype(np.int64)
    y0 = np.where(on, np.fmax(np.nan_to_num(ly), 0), 0).astype(np.int64)
    y1 = np.where(on, np.fmin(np.nan_to_num(hy), H - 1), -1).astype(np.int64)
    return x0, x1, y0, y1, on


def r2_of(radius):
    """The kernels' r^2: radius rounded to float32 (the C ABI's float), squared in float32 (points_raster.cu:410)."""
    return f32(radius) * f32(radius)


def point_cover(points, H, W, radius):
    """Every covering (pixel, point) pair, found on a bbox wider than the setup kernel's by a pixel on each side: the
    exact test (points_raster.cu:176) decides.  Returns dict: keep [NP], pix, g (packed), d (f32), wide bbox."""
    pts = _f(points)
    N, P = pts.shape[:2]
    x, y, z = (pts[..., i].reshape(-1) for i in range(3))
    with np.errstate(invalid="ignore"):
        keep = (z >= 0) & np.isfinite(x) & np.isfinite(y)                                   # :70
    r2 = r2_of(radius)
    g_all = np.nonzero(keep)[0]
    x0, x1, y0, y1, on = setup_bbox(x[g_all], y[g_all], H, W, radius)
    x0, y0 = np.maximum(x0 - 1, 0), np.maximum(y0 - 1, 0)
    x1, y1 = np.where(on, np.minimum(x1 + 1, W - 1), -1), np.where(on, np.minimum(y1 + 1, H - 1), -1)
    P_, G_, D_ = [], [], []
    ids = np.nonzero(on)[0]
    for e, col, row in _enumerate(x0, x1, y0, y1, ids):
        g = g_all[e]
        d = dist2(pixel_ndc(col, W), pixel_ndc(row, H), x[g], y[g])
        c = d < r2
        n = g // P
        P_.append(((n * H + row) * W + col)[c]); G_.append(g[c]); D_.append(d[c])
    cat = (lambda L, dt: np.concatenate(L) if L else np.zeros(0, dt))
    return dict(keep=keep, pix=cat(P_, np.int64), g=cat(G_, np.int64), d=cat(D_, np.float32), r2=r2)


def rasterize_points(points, features, H, W, radius, K, split=None):
    """recmv_rasterize_points: points [N,P,3] f32 NDC, features [N,P] f32 or None -> dict of images [G,N,H,W] f32,
    idx [N,H,W,K] int64, zbuf, dists [N,H,W,K] f32 (-1 padded), count [N,H,W], skipped, covered, and the sparse
    selection (pix, rank, g, d, z) sorted by (pix, rank)."""
    pts = _f(points)
    N, P = pts.shape[:2]
    NP = N * P
    split = P if split is None else int(split)
    c = point_cover(pts, H, W, radius)
    z = (pts[..., 2].reshape(-1) + f32(0)).astype(np.float32)                               # :66, -0 -> +0
    feat = np.ones(NP, np.float32) if features is None else _f(features).reshape(-1)
    zbits = z.view(np.uint32).astype(np.int64)
    pix, g, d = c["pix"], c["g"], c["d"]
    o = np.lexsort((g, zbits[g], pix))                                                      # :177-191: key z_bits | index
    pix, g, d = pix[o], g[o], d[o]
    first = np.ones(len(pix), bool)
    first[1:] = pix[1:] != pix[:-1]
    starts = np.nonzero(first)[0]
    rank = np.arange(len(pix)) - np.repeat(starts, np.diff(np.append(starts, len(pix))))
    s = rank < K
    pix, g, d, rank = pix[s], g[s], d[s], rank[s]
    return dict(pix=pix, g=g, d=d, rank=rank, z=z[g], f=feat[g], grp=np.where(g % max(P, 1) < split, 0, 1),
                count=np.bincount(pix, minlength=N * H * W).reshape(N, H, W), skipped=int(NP - c["keep"].sum()),
                r2=c["r2"], N=N, P=P, H=H, W=W, K=K, split=split, xy=pts.reshape(-1, 3)[:, :2])


def composite(sel, G):
    """points_raster.cu:201-220: acc0, acc1 and T in list order, per pixel."""
    N, H, W, K = sel["N"], sel["H"], sel["W"], sel["K"]
    M = N * H * W
    acc = np.zeros((2, M), np.float32)
    T = np.ones(M, np.float32)
    al = alpha_of(sel["d"], sel["r2"])                                                      # :205-206
    for k in range(K):
        m = np.nonzero(sel["rank"] == k)[0]
        if not len(m):
            break
        p = sel["pix"][m]
        c = (sel["f"][m] * al[m]) * T[p]                                                    # :207
        grp = sel["grp"][m]
        acc[grp, p] = acc[grp, p] + c                                               # :208 (one entry per pixel)
        T[p] = T[p] * (f32(1) - al[m])                                                      # :209
    return acc[:G].reshape(G, N, H, W)


def fragments(sel):
    """points_raster.cu:210-218: idx, zbuf, dists [N,H,W,K], -1 padded."""
    N, H, W, K = sel["N"], sel["H"], sel["W"], sel["K"]
    flat = sel["pix"] * K + sel["rank"]
    idx = np.full(N * H * W * K, -1, np.int64); zb = np.full(N * H * W * K, -1, np.float32)
    ds = np.full(N * H * W * K, -1, np.float32)
    idx[flat], zb[flat], ds[flat] = sel["g"], sel["z"], sel["d"]
    return idx.reshape(N, H, W, K), zb.reshape(N, H, W, K), ds.reshape(N, H, W, K)


def dalpha(sel, grad_images):
    """points_raster.cu:224-250: dL/dalpha of every selected entry."""
    N, H, W, K = sel["N"], sel["H"], sel["W"], sel["K"]
    M = N * H * W
    Gi = _f(grad_images).reshape(-1, M)
    G0 = Gi[0]
    G1 = Gi[1] if Gi.shape[0] == 2 else np.zeros(M, np.float32)                             # :225
    al = alpha_of(sel["d"], sel["r2"])
    Tk = np.empty(len(al), np.float32)
    T = np.ones(M, np.float32)
    by_rank = [np.nonzero(sel["rank"] == k)[0] for k in range(K)]
    for m in by_rank:                                                                       # :227-232
        p = sel["pix"][m]
        Tk[m] = T[p]
        T[p] = T[p] * (f32(1) - al[m])
    S = np.zeros((2, M), np.float32)
    da = np.empty(len(al), np.float32)
    one_eps = f32(1e-9)
    for m in by_rank[::-1]:                                                                 # :236-249
        if not len(m):
            continue
        p = sel["pix"][m]
        first = sel["grp"][m] == 0
        ft = sel["f"][m] * Tk[m]                                                            # :243
        own = np.where(first, G0[p], G1[p]) * ft                                            # :244
        rest = (G0[p] * S[0, p]) + (G1[p] * S[1, p])                                        # :245
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            da[m] = own - (rest / ((f32(1) - al[m]) + one_eps))                             # :246
        grp = sel["grp"][m]
        S[grp, p] = S[grp, p] + (ft * al[m])                                                # :247
    return da


def _seq_segment_sum(vals, seg, nseg):
    """Sequential float32 sums of vals grouped by the sorted segment id `seg`, each from +0 in array order."""
    out = np.zeros(nseg, np.float32)
    if not len(vals):
        return out
    start = np.ones(len(seg), bool)
    start[1:] = seg[1:] != seg[:-1]
    pos = np.arange(len(seg)) - np.repeat(np.nonzero(start)[0], np.diff(np.append(np.nonzero(start)[0], len(seg))))
    with np.errstate(invalid="ignore", over="ignore"):
        for j in range(int(pos.max()) + 1):
            m = pos == j
            out[seg[m]] = out[seg[m]] + vals[m]
    return out


def points_backward(sel, grad_images):
    """recmv_rasterize_points_backward: grad [N,P,3] f32.  Per (tile, point) pair the sum over the tile's pixels in
    row-major order (points_raster.cu:262-279), then per point the sum of its pairs in tile row-major order
    (:280-281, :290-295); every sum is sequential from +0.  Tiles where the point covers no listed pixel add +0, which
    changes no sum (no sum here is ever -0), so the set of tiles visited beyond the covered ones does not matter."""
    N, P, H, W = sel["N"], sel["P"], sel["H"], sel["W"]
    da = dalpha(sel, grad_images)
    inv_r2x2 = f32(2) / sel["r2"]                                                           # :254
    g, pix = sel["g"], sel["pix"]
    q = pix % (H * W)
    col, row = q % W, q // W
    xq, yq = pixel_ndc(col, W), pixel_ndc(row, H)
    dsc = da * inv_r2x2                                                                     # :273
    xy = sel["xy"][g]
    with np.errstate(invalid="ignore", over="ignore"):
        tx_, ty_ = dsc * (xq - xy[:, 0]), dsc * (yq - xy[:, 1])                             # :274-275
    tiles_x = (W + TILE_W - 1) // TILE_W
    tile = (row // TILE_H) * tiles_x + col // TILE_W
    o = np.lexsort((col, row, tile, g))          # per point, per tile (row-major), pixels row-major
    g, tile, tx_, ty_ = g[o], tile[o], tx_[o], ty_[o]
    pair = np.zeros(len(g), np.int64)
    if len(g):
        pair[1:] = np.cumsum((g[1:] != g[:-1]) | (tile[1:] != tile[:-1]))
    npair = int(pair[-1]) + 1 if len(g) else 0
    gx, gy = _seq_segment_sum(tx_, pair, npair), _seq_segment_sum(ty_, pair, npair)
    pg = np.zeros(npair, np.int64)
    pg[pair] = g
    out = np.zeros((N * P, 3), np.float32)
    out[:, 0] = _seq_segment_sum(gx, pg, N * P)
    out[:, 1] = _seq_segment_sum(gy, pg, N * P)
    return out.reshape(N, P, 3)


# ---- running error bounds -------------------------------------------------------------------------------------------
class Rb:
    """A float64 value v with the first-order bound e (in units of u = 2^-24) of the float32 evaluation of the same
    operation order: each rounded operation adds |result| (plus 2^-126, the absolute error 2^-150 of a result that
    underflows), and the operands' bounds propagate through its partial derivatives (a product also carries the
    second-order u e_a e_b).  Constructed from float32 inputs with e = 0 (exact), or from a float64 value with e = |v| (rounded
    once on input)."""
    __array_ufunc__ = None     # an ndarray operand defers to Rb's reflected operators

    def __init__(self, v, e=None, rounded=False):
        self.v = np.asarray(v, dtype=np.float64)
        self.e = np.zeros_like(self.v) if e is None else np.asarray(e, dtype=np.float64)
        if rounded:
            self.e = self.e + np.abs(self.v)

    @staticmethod
    def _w(x):
        return x if isinstance(x, Rb) else Rb(x)

    def __add__(self, o):
        o = Rb._w(o)
        v = self.v + o.v
        return Rb(v, self.e + o.e + np.abs(v) + TINY)

    __radd__ = __add__

    def __sub__(self, o):
        o = Rb._w(o)
        v = self.v - o.v
        return Rb(v, self.e + o.e + np.abs(v) + TINY)

    def __rsub__(self, o):
        return Rb._w(o) - self

    def __mul__(self, o):
        o = Rb._w(o)
        v = self.v * o.v
        # the second-order term u e_a e_b keeps the bound of a square (or product) of two near-zero rounded values
        return Rb(v, np.abs(o.v) * self.e + np.abs(self.v) * o.e + U * self.e * o.e + np.abs(v) + TINY)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = Rb._w(o)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = self.v / o.v
            return Rb(v, (self.e + np.abs(v) * o.e) / np.abs(o.v) + np.abs(v) + TINY)

    def __rtruediv__(self, o):
        return Rb._w(o) / self

    def __neg__(self):
        return Rb(-self.v, self.e)

    def __getitem__(self, i):
        return Rb(self.v[i], self.e[i])


def _project_rb(verts, faces, cam, f):
    """project_face of faces f with running bounds: lists sx, sy, z of 3 Rb each."""
    verts = np.asarray(verts, np.float64)
    cam = [float(c) for c in np.asarray(cam, np.float64).reshape(-1)]
    fa = np.asarray(faces, np.int64).reshape(-1, 3)[f]
    sx, sy, zz = [], [], []
    for k in range(3):
        p = verts[fa[:, k]]
        X, Y, Z = Rb(p[:, 0]), Rb(p[:, 1]), Rb(p[:, 2])
        v = [((X * cam[4 + j]) + (Y * cam[7 + j]) + (Z * cam[10 + j])) + cam[13 + j] for j in range(3)]
        sx.append(cam[2] - (cam[0] * v[0]) / v[2])
        sy.append(cam[3] - (cam[1] * v[1]) / v[2])
        zz.append(v[2])
    return sx, sy, zz


def mesh_dists_bound(verts, faces, cam, f, col, row, H, W):
    """The winner's signed squared NDC edge distance (raster.cu:165-191) of faces f at pixels (col, row) of one frame,
    in float64 with its bound S.  The kernel writes this with plain operations a compiler may contract; a fused
    multiply-add rounds once where the bound counts two roundings, so S bounds every contraction.  The clamp of s to
    [0, 1] and the minimum over edges do not increase the error, so each keeps its operand's bound."""
    sx, sy, _ = _project_rb(verts, faces, cam, f)
    nx = [1.0 - ((2.0 * a + 1.0) / float(W)) for a in sx]
    ny = [1.0 - ((2.0 * a + 1.0) / float(H)) for a in sy]
    qx = 1.0 - Rb(2.0 * np.asarray(col, np.float64) + 1.0) / float(W)
    qy = 1.0 - Rb(2.0 * np.asarray(row, np.float64) + 1.0) / float(H)
    best_v = np.full(len(f), np.inf)
    best_e = np.zeros(len(f))
    for k in range(3):
        ax, ay, bx, by = nx[k], ny[k], nx[(k + 1) % 3], ny[(k + 1) % 3]
        ux, uy, wx, wy = bx - ax, by - ay, qx - ax, qy - ay
        l2 = (ux * ux) + (uy * uy)
        t = ((wx * ux) + (wy * uy)) / l2
        t = Rb(np.where(l2.v > 0, np.clip(np.nan_to_num(t.v), 0.0, 1.0), 0.0), np.where(l2.v > 0, t.e, 0.0))
        dx, dy = wx - (t * ux), wy - (t * uy)
        d = (dx * dx) + (dy * dy)
        best_e = np.maximum(best_e, d.e)        # |min a - min b| <= max |a_i - b_i|
        best_v = np.minimum(best_v, d.v)
    return Rb(-best_v, best_e)


def mesh_bound(verts, faces, cam, f, col, row, origin):
    """The float64 bary [M,3] and zbuf [M] of faces f at pixels (col, row) of one frame, through the kernel's operation
    order (project_face, make_face_rec, shade), each with its bound S.  `origin` [M,2] is the record's integer pixel
    origin (exact in both precisions); verts and cam are float32 inputs (exact)."""
    sx, sy, zz = _project_rb(verts, faces, cam, f)
    ex = [s - origin[:, 0] for s in sx]
    ey = [s - origin[:, 1] for s in sy]
    Ar = ((ex[1] - ex[0]) * (ey[2] - ey[0])) - ((ey[1] - ey[0]) * (ex[2] - ex[0]))
    inv = 1.0 / Ar
    qx, qy = col - origin[:, 0], row - origin[:, 1]
    w = []
    for i in range(3):
        a, b = (i + 1) % 3, (i + 2) % 3
        dx, dy = ex[b] - ex[a], ey[b] - ey[a]
        ka, kb, kc = (-dy) * inv, dx * inv, ((dy * ex[a]) - (dx * ey[a])) * inv
        bi = ((ka * qx) + (kb * qy)) + kc
        w.append(bi * (1.0 / zz[i]))
    s = (w[0] + w[1]) + w[2]
    bp = [wi / s for wi in w]
    zb = ((bp[0] * zz[0]) + (bp[1] * zz[1])) + (bp[2] * zz[2])
    return bp, zb


def points_bound(sel, points, features, radius, grad_images):
    """Bounds S of the point rasterizer's outputs on a float32 selection, in the kernel's operation order: images
    [G,M] (Rb), and grad [NP,2] (Rb).  The radius is rounded to float32 on input (the C ABI's float)."""
    N, P, H, W, K = sel["N"], sel["P"], sel["H"], sel["W"], sel["K"]
    M = N * H * W
    pts = np.asarray(points, np.float64).reshape(-1, 3)
    feat = np.ones(N * P) if features is None else np.asarray(features, np.float64).reshape(-1)
    r = Rb(float(radius), rounded=True)
    r2 = r * r
    g, pix = sel["g"], sel["pix"]
    q = pix % (H * W)
    col, row = q % W, q // W
    xq = 1.0 - Rb(2.0 * col + 1) / float(W)
    yq = 1.0 - Rb(2.0 * row + 1) / float(H)
    dx, dy = xq - Rb(pts[g, 0]), yq - Rb(pts[g, 1])
    d = (dx * dx) + (dy * dy)
    al = 1.0 - d / r2
    f = Rb(feat[g])
    Gi = np.asarray(grad_images, np.float64).reshape(-1, M) if grad_images is not None else np.zeros((1, M))
    G = Gi.shape[0]
    G1 = Gi[1] if G == 2 else np.zeros(M)
    grp = sel["grp"]
    by_rank = [np.nonzero(sel["rank"] == k)[0] for k in range(K)]
    T = Rb(np.ones(M))
    Tk = Rb(np.zeros(len(g)))
    acc = [Rb(np.zeros(M)), Rb(np.zeros(M))]
    for m in by_rank:
        if not len(m):
            continue
        p = pix[m]
        Tk.v[m], Tk.e[m] = T.v[p], T.e[p]
        c = (f[m] * al[m]) * T[p]
        for gg in (0, 1):
            s = grp[m] == gg
            a = acc[gg][p[s]] + c[s]
            acc[gg].v[p[s]], acc[gg].e[p[s]] = a.v, a.e
        t = T[p] * (1.0 - al[m])
        T.v[p], T.e[p] = t.v, t.e
    S = [Rb(np.zeros(M)), Rb(np.zeros(M))]
    da = Rb(np.zeros(len(g)))
    for m in by_rank[::-1]:
        if not len(m):
            continue
        p = pix[m]
        first = grp[m] == 0
        ft = f[m] * Tk[m]
        own = Rb(np.where(first, Gi[0, p], G1[p])) * ft
        rest = (Rb(Gi[0, p]) * S[0][p]) + (Rb(G1[p]) * S[1][p])
        x = own - rest / ((1.0 - al[m]) + Rb(float(f32(1e-9))))
        da.v[m], da.e[m] = x.v, x.e
        for gg in (0, 1):
            s = grp[m] == gg
            a = S[gg][p[s]] + (ft[s] * al[m][s])
            S[gg].v[p[s]], S[gg].e[p[s]] = a.v, a.e
    dsc = da * (2.0 / r2)
    tx_, ty_ = dsc * dx, dsc * dy
    # every sum adds its running magnitude per addition; a sum of n terms in any order is bounded by
    # n * sum |terms| + sum(term bounds), which covers both the per-tile and the per-slot levels
    npp = N * P
    cnt = np.bincount(g, minlength=npp).astype(np.float64)
    out = []
    for t in (tx_, ty_):
        v = np.bincount(g, weights=t.v, minlength=npp)
        e = np.bincount(g, weights=t.e, minlength=npp) + cnt * np.bincount(g, weights=np.abs(t.v), minlength=npp)
        out.append(Rb(v, e))
    return acc[:G], out
