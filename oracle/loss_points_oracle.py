"""TEST INFRASTRUCTURE ONLY -- the NumPy restatement of csrc/loss_points.cu and csrc/frame_loss.cu (DESIGN section 1k),
the sampling, compaction and per-frame means of `surface_render_loss` (OptimGarmentNetwork.py:1083-1219).

`sample` runs the G garments of a call: the E / D vertex draws at fp32(S / V), the eikonal points X_E (local rows
x + fp32(z 0.01f), global rows fp32(fp32(u 3.6f) - 1.8f)), the regulariser points X_D and the check compaction, in
float32 with the kernel's rounding.  The normals are computed in float64 and rounded once; `normals` also flags the
samples whose float64 value lies within a few double ulps of a float32 rounding boundary -- the only ones where the
kernel's libm may round the other way.  `color_mean` and `normal_mean` are the two frame means in float64 with their
analytic VJPs.  Philox4x32-10 is sample_oracle's."""
import numpy as np

from . import sample_oracle

LANES = 5                     # E-draw, D-draw, E-local, E-global, D-local
E_DRAW, D_DRAW, E_LOCAL, E_GLOBAL, D_LOCAL = range(LANES)
FLAG_ULPS = 64                # double ulps around a float32 rounding boundary that flag a normal


def words(seed, counters):
    """[n,4] uint32 Philox4x32-10 words of the 64-bit counters (uint64 array) under `seed`."""
    seed = int(seed) % (1 << 64)
    c = np.asarray(counters, dtype=np.uint64)
    ctr = np.stack([(c & np.uint64(0xFFFFFFFF)).astype(np.uint32), (c >> np.uint64(32)).astype(np.uint32),
                    np.zeros(c.shape, np.uint32), np.zeros(c.shape, np.uint32)], -1)
    return sample_oracle.philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32)).reshape(-1, 4)


def unit24(x):
    """float32 (x >> 8) 2^-24, exact, in [0, 1)."""
    return (np.asarray(x, np.uint32) >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)


def threshold(S, V):
    """fp32(double(S) / double(V)): torch's float32 comparison of a CPU float32 tensor with the Python quotient."""
    if V <= 0:
        raise ValueError("threshold: V must be positive (the reference divides by it)")
    return np.float32(float(S) / float(V))


def counters(offset, base, lane, C, n):
    """uint64 counters offset + base + lane C + i, i < n, modulo 2^64 (base = 5 (C_0 + ... + C_{g-1}))."""
    return np.uint64((int(offset) + int(base) + lane * int(C)) % (1 << 64)) + np.arange(n, dtype=np.uint64)


def _flag(z):
    """z float64 -> True where z lies within FLAG_ULPS double ulps of a float32 rounding boundary."""
    f = z.astype(np.float32)
    lo = np.nextafter(f, np.float32(-np.inf)).astype(np.float64)
    hi = np.nextafter(f, np.float32(np.inf)).astype(np.float64)
    f64 = f.astype(np.float64)
    dist = np.minimum(np.abs(z - (f64 + lo) / 2), np.abs(z - (f64 + hi) / 2))
    return dist <= FLAG_ULPS * np.spacing(np.abs(z))


def normals(seed, ctrs):
    """([n,3] float32 N(0,1) samples, [n] flags) of the counters: Box-Muller of (x0, x1) (cos, sin) and of (x2, x3)
    (cos), ua = ((x >> 8) + 1) 2^-24, ub = (x >> 8) 2^-24, in float64, rounded once."""
    x = words(seed, ctrs).astype(np.uint64)
    s = lambda k: (x[:, k] >> np.uint64(8)).astype(np.float64)  # noqa: E731
    ua, ub, uc, ud = (s(0) + 1) * 2.0 ** -24, s(1) * 2.0 ** -24, (s(2) + 1) * 2.0 ** -24, s(3) * 2.0 ** -24
    two_pi = 6.283185307179586
    r0, r1 = np.sqrt(-2.0 * np.log(ua)), np.sqrt(-2.0 * np.log(uc))
    z = np.stack([r0 * np.cos(two_pi * ub), r0 * np.sin(two_pi * ub), r1 * np.cos(two_pi * ud)], 1)
    return z.astype(np.float32), _flag(z).any(1)


def local(p, z):
    """p + fp32(z 0.01f), each operation rounded in float32."""
    return (np.asarray(p, np.float32) + np.asarray(z, np.float32) * np.float32(0.01)).astype(np.float32)


def global_points(seed, ctrs):
    """[n,3] float32 fp32(fp32(u 3.6f) - 1.8f), u the top 24 bits of words 0, 1, 2."""
    x = words(seed, ctrs)
    return (unit24(x[:, :3]) * np.float32(3.6) - np.float32(1.8)).astype(np.float32)


def draw(seed, offset, base, lane, C, V, S):
    """Kept vertex indices of one lane (E_DRAW or D_DRAW) of a garment."""
    u = unit24(words(seed, counters(offset, base, lane, C, V))[:, 0])
    return np.flatnonzero(u < threshold(S, V))


def garment(P, verts, check, S, seed, offset, base):
    """One garment whose counters start at offset + base: dict with keep_e, keep_d (vertex indices), X_E, X_D,
    flag_e, flag_d (rows whose normal is flagged) and checked (input indices)."""
    P = np.asarray(P, np.float32).reshape(-1, 3)
    verts = np.asarray(verts, np.float32).reshape(-1, 3)
    M, V = P.shape[0], verts.shape[0]
    C = M + V
    keep_e, keep_d = draw(seed, offset, base, E_DRAW, C, V, S), draw(seed, offset, base, D_DRAW, C, V, S)
    B_e, B_d = np.concatenate([P, verts[keep_e]]), np.concatenate([P, verts[keep_d]])
    z_e, flag_e = normals(seed, counters(offset, base, E_LOCAL, C, len(B_e)))
    z_d, flag_d = normals(seed, counters(offset, base, D_LOCAL, C, len(B_d)))
    glob = global_points(seed, counters(offset, base, E_GLOBAL, C, len(B_e) // 6))
    return {"keep_e": keep_e, "keep_d": keep_d,
            "X_E": np.concatenate([local(B_e, z_e), glob]).reshape(-1, 3),
            "X_D": np.concatenate([B_d, local(B_d, z_d)]).reshape(-1, 3),
            "flag_e": np.concatenate([flag_e, np.zeros(len(glob), bool)]),
            "flag_d": np.concatenate([np.zeros(len(B_d), bool), flag_d]),
            "checked": np.flatnonzero(np.asarray(check, bool))}


def sample(P, verts, check, seed, offset=0):
    """G garments of one call (S = 4096 // G): the list of `garment` dicts and the next offset."""
    G = len(P)
    S = 4096 // G
    out, base = [], 0
    for g in range(G):
        out.append(garment(P[g], verts[g], check[g], S, seed, offset, base))
        base += LANES * (len(P[g]) + len(verts[g]))
    return out, (int(offset) + base) % (1 << 64)


def _frame_mean(e, b, ok, N):
    """(L, per-row d L / d e_i) of (1/N) sum_f mean_{ok i in f} e_i, in float64; rows outside [0, N) do not count."""
    e = np.asarray(e, np.float64)
    b = np.asarray(b, np.int64)
    ok = ok & (b >= 0) & (b < N)
    n = np.bincount(b[ok], minlength=N)[:N]
    s = np.bincount(b[ok], weights=e[ok], minlength=N)[:N]
    L = (s / np.maximum(n, 1)).sum() / N
    de = np.zeros(len(e))
    de[ok] = 1.0 / (N * np.maximum(n[b[ok]], 1))
    return L, de


def color_rows(gt, b, r, c, colors):
    """(e [M] float32 with the kernel's channel order, in-range mask, signs [M,3] of gt - colors)."""
    gt = np.asarray(gt, np.float32)
    N, H, W = gt.shape[:3]
    b, r, c = (np.asarray(x, np.int64) for x in (b, r, c))
    ok = (b >= 0) & (b < N) & (r >= 0) & (r < H) & (c >= 0) & (c < W)
    px = gt[np.where(ok, b, 0), np.where(ok, r, 0), np.where(ok, c, 0)]
    diff = (px - np.asarray(colors, np.float32)).astype(np.float32)
    a = np.abs(diff)
    e = ((a[:, 0] + a[:, 1]).astype(np.float32) + a[:, 2]).astype(np.float32)
    return e, ok, np.sign(diff)


def color_mean(gt, b, r, c, colors, N, g=1.0):
    """(L float64, d colors [M,3] float64) of the colour term."""
    e, ok, sgn = color_rows(gt, b, r, c, colors)
    L, de = _frame_mean(e, b, ok, N)
    return L, -sgn * (g * de)[:, None]


def _frame_mean_normal(gtn, J, nx, w, b, N):
    """The normal term's value alone, in float64 from float64 inputs (for finite differences)."""
    n, J, nx, w = (np.asarray(x, np.float64) for x in (gtn, J, nx, w))
    nn = np.sqrt((n * n).sum(1))
    ok = nn > 1e-4
    nh = np.where(ok[:, None], n / np.where(ok, nn, 1.0)[:, None], n)
    d = np.einsum("mab,ma->mb", J, nh) - nx
    return _frame_mean(np.sqrt((d * d).sum(1)) * w, b, ok, N)[0]


def normal_mean(gtn, J, nx, w, b, N, g=1.0):
    """(L, d gtn [M,3], d J [M,3,3], d nx [M,3]) of the normal term in float64."""
    n = np.asarray(gtn, np.float32).astype(np.float64)
    J = np.asarray(J, np.float32).astype(np.float64)
    nx = np.asarray(nx, np.float32).astype(np.float64)
    w = np.asarray(w, np.float32).astype(np.float64)
    nn = np.sqrt((n * n).sum(1))
    ok = nn > 1e-4
    nh = np.where(ok[:, None], n / np.where(ok, nn, 1.0)[:, None], n)
    d = np.einsum("mab,ma->mb", J, nh) - nx
    dn = np.sqrt((d * d).sum(1))
    L, de = _frame_mean(dn * w, b, ok, N)
    gd = np.where((dn > 0)[:, None], (g * de * w / np.where(dn > 0, dn, 1.0))[:, None] * d, 0.0)
    dJ = nh[:, :, None] * gd[:, None, :]
    dnh = np.einsum("mab,mb->ma", J, gd)
    dgtn = (dnh - nh * (nh * dnh).sum(1, keepdims=True)) / np.where(ok, nn, 1.0)[:, None]
    dgtn[~ok] = 0.0
    return L, dgtn, dJ, -gd
