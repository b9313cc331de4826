"""Float32 restatement of the skinning-voxel construction (csrc/lbsw_field.cu): the kNN blend and the smoothing pass.

Every operation of those kernels is explicitly rounded (__fadd_rn, __fsub_rn, __fmul_rn, __fdiv_rn, __frcp_rn,
__fsqrt_rn and the fmaf of the distance), so restating their operation order in NumPy float32 (render_f32.fma32 for
the FMA) gives their outputs bit for bit.  Each step cites the line it restates.  Written from the documented operation
order; no kernel is called.

The neighbour set: the kernel scans the vertices in index order and inserts a candidate when its distance is strictly
below the current k-th, so it keeps the k smallest by (sqrt_rn(d2), index) in lexicographic order.  Its thr2 gate
skips only candidates that insertion would refuse, and a candidate whose d2 is not finite (NaN, or an overflow to inf)
is never offered: a slot no finite candidate fills keeps distance +inf and vertex 0.

The distance scan is the expensive part (every voxel against every vertex), so `neighbours` takes an array module:
NumPy, or torch, whose element-wise float64 and float32 operations round the same way on the CPU and on the GPU.
"""
import numpy as np

from render_f32 import fma32

f32 = np.float32
KCH = 24
KMAX = 32


def voxel_centre(c, res, ac, lo, hi):
    """lbsw_field.cu:23-29 along one axis: c int array, res int, lo / hi float32."""
    r, lo, hi = f32(res), f32(lo), f32(hi)
    c = np.asarray(c).astype(np.float32)
    u = c / (r - f32(1)) if ac else (c / r) + ((f32(1) / r) * f32(0.5))
    return (u * (hi - lo)) + lo


def centres(idx, res, ac, bmin, bmax):
    """Voxel centres [n,3] f32 of flat voxel indices idx ((z H + y) W + x), res = (W, H, D)."""
    W, H, D = res
    idx = np.asarray(idx, np.int64)
    x, y, z = idx % W, (idx // W) % H, idx // (W * H)
    return np.stack([voxel_centre(x, W, ac, bmin[0], bmax[0]), voxel_centre(y, H, ac, bmin[1], bmax[1]),
                     voxel_centre(z, D, ac, bmin[2], bmax[2])], 1)


def _fma32_torch(a, b, c):
    """render_f32.fma32 in torch (float32 tensors in, float32 out)."""
    import torch
    a, b, c = a.double(), b.double(), c.double()
    p = a * b
    s = p + c
    bp = s - c
    e = (p - bp) + (c - (s - bp))
    r = s.float()
    r64 = r.double()
    inf = torch.full_like(r, float("inf"))
    other = torch.nextafter(r, torch.where(s > r64, inf, -inf)).double()
    half = (s != r64) & (2 * s == r64 + other) & (e != 0)
    toward = torch.sign(e) == torch.sign(other - s)
    return torch.where(half & toward, other.float(), r)


def dist2(c, v, xp=np):
    """lbsw_field.cu:33-36: fmaf(dz, dz, fmaf(dy, dy, dx * dx)) of centres c [n,3] against vertices v [V,3] -> [n,V]."""
    fma = fma32 if xp is np else _fma32_torch
    d = [c[:, None, i] - v[None, :, i] for i in range(3)]
    if xp is np:
        with np.errstate(invalid="ignore", over="ignore"):
            return fma(d[2], d[2], fma(d[1], d[1], d[0] * d[0]))
    return fma(d[2], d[2], fma(d[1], d[1], d[0] * d[0]))


def neighbours(c, verts, kmax=KMAX, xp=np, chunk=2048):
    """The kmax nearest vertices of each centre c [n,3] f32, nearest first by (sqrt_rn(d2), index): (s [n,kmax] f32,
    id [n,kmax] int64), +inf / 0 where fewer than kmax vertices have a finite d2.  The neighbours for k <= kmax are the
    first k columns.  xp: numpy (arrays) or torch (tensors on any device; returned as NumPy)."""
    S, I = [], []
    for i in range(0, len(c), chunk):
        cc = c[i:i + chunk]
        d2 = dist2(cc, verts, xp)
        if xp is np:
            sn = np.sqrt(d2.astype(np.float64)).astype(np.float32)     # sqrt_rn: exact through float64
            bits = np.where(np.isfinite(d2), sn.view(np.uint32).astype(np.int64), np.int64(0x7f800000))
            key = (bits << 32) | np.arange(d2.shape[1], dtype=np.int64)[None]
            kk = min(kmax, key.shape[1])
            part = np.argpartition(key, kk - 1, axis=1)[:, :kk]
            ks = np.take_along_axis(key, part, 1)
            o = np.argsort(ks, axis=1)
            ks = np.take_along_axis(ks, o, 1)
        else:
            import torch
            sn = d2.double().sqrt().float()
            bits = torch.where(torch.isfinite(d2), sn.view(torch.int32).long(), torch.tensor(0x7f800000, device=d2.device))
            key = (bits << 32) | torch.arange(d2.shape[1], device=d2.device)[None]
            kk = min(kmax, key.shape[1])
            ks = torch.topk(key, kk, dim=1, largest=False, sorted=True).values.cpu().numpy()
        fin = (ks >> 32) < 0x7f800000
        s = np.where(fin, (ks >> 32).astype(np.uint32).view(np.float32), np.float32(np.inf))
        ids = np.where(fin, ks & 0xffffffff, 0)
        if kk < kmax:
            s = np.concatenate([s, np.full((len(s), kmax - kk), np.inf, np.float32)], 1)
            ids = np.concatenate([ids, np.zeros((len(s), kmax - kk), np.int64)], 1)
        S.append(s)
        I.append(ids)
    return np.concatenate(S), np.concatenate(I)


def blend(s, ids, vert_ws, k):
    """lbsw_field.cu:115-138 for the first k neighbours (s [n,>=k] f32, ids): (out [n,24] f32, idx [n,k])."""
    s, ids = s[:, :k], ids[:, :k]
    vert_ws = np.asarray(vert_ws, np.float32)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        r = f32(1) / np.fmin(np.fmax(s, f32(1e-4)), f32(1))                # :119, __frcp_rn
        tot = np.zeros(len(s), np.float32)
        for i in range(k):                                                # :120, slot order from +0
            tot = tot + r[:, i]
        acc = np.zeros((len(s), KCH), np.float32)
        for i in range(k):                                                # :127-133
            w = r[:, i] / tot
            acc = acc + vert_ws[ids[:, i]] * w[:, None]
    return acc, ids


def smooth(ws_cl, times, zero_below=0.0):
    """recmv_lbsw_smooth on a channels-last [D,H,W,24] f32 voxel (lbsw_field.cu:142-200, 249-262) -> [D,H,W,24]."""
    w = np.array(ws_cl, np.float32, copy=True)
    D, H, W = w.shape[:3]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for _ in range(times):
            if D >= 3 and H >= 3 and W >= 3:                               # :167, interior x, y, z in [1, size - 2]
                c = w[1:-1, 1:-1, 1:-1]
                sum6 = ((((w[2:, 1:-1, 1:-1] + w[:-2, 1:-1, 1:-1]) + w[1:-1, 2:, 1:-1]) + w[1:-1, :-2, 1:-1])
                        + w[1:-1, 1:-1, 2:]) + w[1:-1, 1:-1, :-2]          # :144
                mean = sum6 / f32(6)                                         # :145
                new = w.copy()
                new[1:-1, 1:-1, 1:-1] = ((c - mean) * f32(0.7)) + mean       # :146
                w = new
            tot = np.zeros(w.shape[:3], np.float32)
            for ch in range(KCH):                                          # :183-185, channel order from +0
                tot = tot + w[..., ch]
            w = w / tot[..., None]                                         # :187
        if zero_below > 0:                                                 # :190-193, after the last pass
            w = np.where(w < f32(zero_below), f32(0), w)
    return w
