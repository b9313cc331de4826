"""Float64 restatement of the skinning kernels (csrc/lbs.cu): forward, inverse, backward and the VJP of the backward's
point gradients, each with an absolute twin.

Every function evaluates at the kernels' own fp32 voxel coordinate (`coord32`, bit-equal to what sample_skin24 and
skin_cell compute without fast-math) and with their clamp rule, so the cell, the corner weights' arguments and the
clamping agree with the kernel by construction and only arithmetic error remains.  The derivative chain factor
d i / d s = size / extend follows the sampler: 0 on an axis whose coordinate is clamped (u <= 0 or u >= size - 1) or
NaN.  With the corner weights c_k(s) of the cell, the voxel rows W_k [24] and T_k = sum_b W_kb A_b (rows 0..2):

    forward    out   = sum_k c_k T_k [a;1] + trans             weights = sum_k c_k W_k
    backward   dps   = T3^T g (+ ds without tps)    ds_j = g . sum_k (T_k [a;1]) dc_k/ds_j
               dA_b  = sum_p w_b g [a;1]^T          dtrans = sum_p g
    VJP        phi = g^T T3 u + g^T Jw v' (v' = v with tps, u without), Jw = sum_k T_k [a;1] dc_k^T
               d g = T3 u + Jw v'     d a = sum_k (dc_k . v') T_k3^T g
               d s = sum_k (g^T T_k3 u) dc_k + sum_k (g . T_k [a;1]) H_k v'
               dA_b = g (w_b [u;0] + (sum_k W_kb dc_k . v') [a;1])^T

The absolute twin evaluates the same sums over |inputs| with |dc|, |H|, so each output y = sum t gets its scale
S = sum |t|; an fp32 kernel summing those terms in any order stays within a small multiple of 2^-24 S.  Everything
runs in chunks on the device of its inputs: a per-point gather of A is [P, 24, 12], too large at 1e6 points at once.
"""
import torch

from oracle import oracle_torch as ot

CHUNK = 1 << 16


def coord32(p, size, c, e):
    """u = unnormalize(((p - c) / e) * 2) in fp32, every operation rounded (sample_skin24 / skin_cell)."""
    p = p.float()
    g = ((p - c) / torch.full_like(p, e)) * 2.0     # a tensor divisor: torch divides by a scalar as a * (1 / b)
    return ((g + 1.0) * float(size) - 1.0) * 0.5


def _cell(s, shape, center, extend):
    """Per point: (lin [n,8] corner offsets into the channels-last voxel, cw [n,8] corner weights, dcw [n,8,3] their
    gradients, hcw [n,8,3] their mixed second partials (xy, xz, yz)) in float64, corners in (z, y, x) order, x fastest."""
    D, H, W = shape
    ix, m = [], []
    for a, size in enumerate((W, H, D)):
        u = coord32(s[:, a], size, float(center[a]), float(extend))
        inside = (u > 0) & (u < size - 1)          # NaN: false
        uc = torch.nan_to_num(u, nan=0.0).clamp(0, size - 1)
        ix.append(uc.double())
        m.append(torch.where(inside, float(size) / float(extend), 0.0).double())
    x0 = [torch.floor(i) for i in ix]
    frac = [i - f for i, f in zip(ix, x0)]
    idx = [torch.stack([f.long(), (f.long() + 1).clamp_max(size - 1)], 1) for f, size in zip(x0, (W, H, D))]
    wts = [torch.stack([1 - fr, fr], 1) for fr in frac]                 # [n, 2]
    sl = [torch.stack([-mm, mm], 1) for mm in m]                        # slope of the per-axis weight
    lin, cw, dcw, hcw = [], [], [], []
    for k in range(8):
        dx, dy, dz = k & 1, (k >> 1) & 1, k >> 2
        wx, wy, wz = wts[0][:, dx], wts[1][:, dy], wts[2][:, dz]
        ex, ey, ez = sl[0][:, dx], sl[1][:, dy], sl[2][:, dz]
        lin.append((idx[2][:, dz] * H + idx[1][:, dy]) * W + idx[0][:, dx])
        cw.append(wx * wy * wz)
        dcw.append(torch.stack([ex * wy * wz, ey * wx * wz, ez * wx * wy], 1))
        hcw.append(torch.stack([ex * ey * wz, ex * ez * wy, ey * ez * wx], 1))
    lin, cw, dcw, hcw = torch.stack(lin, 1), torch.stack(cw, 1), torch.stack(dcw, 1), torch.stack(hcw, 1)
    return lin, cw, dcw, hcw


class Skin:
    """The voxel and its normalisation on one device, in float64."""

    def __init__(self, ws_cl, center, extend):
        self.shape = tuple(ws_cl.shape[:3])
        self.flat = ws_cl.reshape(-1, 24).double()
        self.center = [float(x) for x in center]
        self.extend = float(extend)

    def corners(self, s):
        lin, cw, dcw, hcw = _cell(s, self.shape, self.center, self.extend)
        return self.flat[lin], cw, dcw, hcw           # Wc [n,8,24]


def _frames(A, f):
    A64 = A.double()
    Af = A64[f][:, :, :3, :]                          # [n,24,3,4]
    return Af, Af.abs()


def _Tc(Wc, Af):
    """T_k = sum_b W_kb A_b rows 0..2: [n,8,3,4]."""
    return torch.einsum("nkb,nbrc->nkrc", Wc, Af)


def _hv(h, v):
    return torch.stack([h[..., 0] * v[:, None, 1] + h[..., 1] * v[:, None, 2],
                        h[..., 0] * v[:, None, 0] + h[..., 2] * v[:, None, 2],
                        h[..., 1] * v[:, None, 0] + h[..., 2] * v[:, None, 1]], -1)


def _chunks(P):
    for i in range(0, P, CHUNK):
        yield slice(i, min(i + CHUNK, P))


def _a1(a):
    return torch.cat([a, torch.ones_like(a[:, :1])], 1)


def forward(sk, ps, A, trans, f, tps=None):
    """(out, out_S, weights) float64 [P,3], [P,3], [P,24]; f: clamped frame per point."""
    P = ps.shape[0]
    out = torch.empty((P, 3), dtype=torch.float64, device=ps.device)
    S = torch.empty_like(out)
    w = torch.empty((P, 24), dtype=torch.float64, device=ps.device)
    for sl in _chunks(P):
        a = ps[sl].double()
        Wc, cw, _, _ = sk.corners((ps if tps is None else tps)[sl])
        Af, Afa = _frames(A, f[sl])
        wb = (cw[:, :, None] * Wc).sum(1)
        T = torch.einsum("nb,nbrc->nrc", wb, Af)
        Ta = torch.einsum("nb,nbrc->nrc", wb, Afa)
        a1 = _a1(a)
        tr = trans.double()[f[sl]]
        out[sl] = (T * a1[:, None, :]).sum(-1) + tr
        S[sl] = (Ta * a1.abs()[:, None, :]).sum(-1) + tr.abs()
        w[sl] = wb
    return out, S, w


def inverse(sk, x, A, trans, f):
    """(xc, valid, det, det_S, cond, xc_scale): FastMinv rule |det| < 1e-4 -> invalid and xc = 0; a NaN det is valid
    with a NaN xc.  det_S is the permanent of |M|'s twin (the scale of det's rounding error); xc_scale the per-row
    |M^-1| (|x| + |trans| + |t|) and cond the row's float64 condition number |M|_inf |M^-1|_inf."""
    P = x.shape[0]
    dev = x.device
    xc = torch.empty((P, 3), dtype=torch.float64, device=dev)
    ok = torch.empty((P,), dtype=torch.bool, device=dev)
    det = torch.empty((P,), dtype=torch.float64, device=dev)
    detS = torch.empty_like(det)
    cond = torch.empty_like(det)
    scale = torch.empty_like(det)
    for sl in _chunks(P):
        Wc, cw, _, _ = sk.corners(x[sl])
        Af, Afa = _frames(A, f[sl])
        wb = (cw[:, :, None] * Wc).sum(1)
        T = torch.einsum("nb,nbrc->nrc", wb, Af)
        Ta = torch.einsum("nb,nbrc->nrc", wb, Afa)
        M, Ma = T[:, :, :3], Ta[:, :, :3]
        c = torch.stack([M[:, 1, 1] * M[:, 2, 2] - M[:, 1, 2] * M[:, 2, 1],
                         -M[:, 1, 0] * M[:, 2, 2] + M[:, 1, 2] * M[:, 2, 0],
                         M[:, 1, 0] * M[:, 2, 1] - M[:, 1, 1] * M[:, 2, 0]], 1)
        d = (M[:, 0] * c).sum(1)
        ca = torch.stack([Ma[:, 1, 1] * Ma[:, 2, 2] + Ma[:, 1, 2] * Ma[:, 2, 1],
                          Ma[:, 1, 0] * Ma[:, 2, 2] + Ma[:, 1, 2] * Ma[:, 2, 0],
                          Ma[:, 1, 0] * Ma[:, 2, 1] + Ma[:, 1, 1] * Ma[:, 2, 0]], 1)
        detS[sl] = (Ma[:, 0] * ca).sum(1)
        Mi, good = ot.minv3x3_fwd(M.contiguous())      # the cofactor inverse with FastMinv's rule
        tr = trans.double()[f[sl]]
        rhs = x[sl].double() - tr - T[:, :, 3]
        xc[sl] = (Mi @ rhs[:, :, None])[:, :, 0]
        ok[sl] = good
        det[sl] = d
        rs = x[sl].double().abs() + tr.abs() + Ta[:, :, 3]
        scale[sl] = (Mi.abs() @ rs[:, :, None])[:, :, 0].amax(1)
        cond[sl] = M.abs().sum(2).amax(1) * Mi.abs().sum(2).amax(1)
    return xc, ok, det, detS, cond, scale


def backward(sk, ps, A, g, f, F, tps=None):
    """(dps, dtps or None, dA [F,24,4,4], dtrans [F,3]) and their twins, float64."""
    P = ps.shape[0]
    dev = ps.device
    dps = torch.empty((P, 3), dtype=torch.float64, device=dev)
    dpsS = torch.empty_like(dps)
    dtps = torch.empty_like(dps) if tps is not None else None
    dtpsS = torch.empty_like(dps) if tps is not None else None
    dA = torch.zeros((F, 24, 3, 4), dtype=torch.float64, device=dev)
    dAS = torch.zeros_like(dA)
    dtr = torch.zeros((F, 3), dtype=torch.float64, device=dev)
    dtrS = torch.zeros_like(dtr)
    for sl in _chunks(P):
        a = ps[sl].double()
        a1 = _a1(a)
        gg = g[sl].double()
        Wc, cw, dcw, _ = sk.corners((ps if tps is None else tps)[sl])
        Af, Afa = _frames(A, f[sl])
        Tc, Tca = _Tc(Wc, Af), _Tc(Wc, Afa)
        T, Ta = (cw[:, :, None, None] * Tc).sum(1), (cw[:, :, None, None] * Tca).sum(1)
        Y = (Tc * a1[:, None, None, :]).sum(-1)                                # [n,8,3]
        Ya = (Tca * a1.abs()[:, None, None, :]).sum(-1)
        ds = torch.einsum("nki,nkj,ni->nj", Y, dcw, gg)
        dsS = torch.einsum("nki,nkj,ni->nj", Ya, dcw.abs(), gg.abs())
        dT = torch.einsum("nij,ni->nj", T[:, :, :3], gg)
        dTS = torch.einsum("nij,ni->nj", Ta[:, :, :3], gg.abs())
        if tps is None:
            dps[sl], dpsS[sl] = dT + ds, dTS + dsS
        else:
            dps[sl], dpsS[sl] = dT, dTS
            dtps[sl], dtpsS[sl] = ds, dsS
        wb = (cw[:, :, None] * Wc).sum(1)
        fi = f[sl]
        dA.index_add_(0, fi, wb[:, :, None, None] * (gg[:, :, None] * a1[:, None, :])[:, None])
        dAS.index_add_(0, fi, wb[:, :, None, None] * (gg.abs()[:, :, None] * a1.abs()[:, None, :])[:, None])
        dtr.index_add_(0, fi, gg)
        dtrS.index_add_(0, fi, gg.abs())
    pad = lambda t: torch.cat([t, torch.zeros_like(t[:, :, :1])], 2)     # noqa: E731  (row 3 of dA is 0)
    return (dps, dtps, pad(dA), dtr), (dpsS, dtpsS, pad(dAS), dtrS)


def vjp(sk, ps, A, g, u, f, F, tps=None, v=None):
    """(d g, dps, dtps or None, dA [F,24,4,4]) of phi = <dps, u> + <dtps, v> and their twins, float64."""
    P = ps.shape[0]
    dev = ps.device
    z = lambda: torch.empty((P, 3), dtype=torch.float64, device=dev)     # noqa: E731
    dg, dgS, da, daS = z(), z(), z(), z()
    dtps = z() if tps is not None else None
    dtpsS = z() if tps is not None else None
    dA = torch.zeros((F, 24, 3, 4), dtype=torch.float64, device=dev)
    dAS = torch.zeros_like(dA)
    for sl in _chunks(P):
        a = ps[sl].double()
        a1 = _a1(a)
        gg, uu = g[sl].double(), u[sl].double()
        vv = uu if tps is None else v[sl].double()
        Wc, cw, dcw, hcw = sk.corners((ps if tps is None else tps)[sl])
        Af, Afa = _frames(A, f[sl])
        Tc, Tca = _Tc(Wc, Af), _Tc(Wc, Afa)
        Y = (Tc * a1[:, None, None, :]).sum(-1)
        Ya = (Tca * a1.abs()[:, None, None, :]).sum(-1)
        Tu = torch.einsum("nkij,nj->nki", Tc[..., :3], uu)
        Tua = torch.einsum("nkij,nj->nki", Tca[..., :3], uu.abs())
        q = torch.einsum("nkij,ni->nkj", Tc[..., :3], gg)
        qa = torch.einsum("nkij,ni->nkj", Tca[..., :3], gg.abs())
        dv = (dcw * vv[:, None, :]).sum(-1)                                     # [n,8]
        dva = (dcw.abs() * vv.abs()[:, None, :]).sum(-1)
        dg[sl] = (cw[:, :, None] * Tu).sum(1) + (dv[:, :, None] * Y).sum(1)
        dgS[sl] = (cw[:, :, None] * Tua).sum(1) + (dva[:, :, None] * Ya).sum(1)
        d_a = (dv[:, :, None] * q).sum(1)
        d_aS = (dva[:, :, None] * qa).sum(1)
        gTu, gTua = (q * uu[:, None, :]).sum(-1), (qa * uu.abs()[:, None, :]).sum(-1)
        gY, gYa = (Y * gg[:, None, :]).sum(-1), (Ya * gg.abs()[:, None, :]).sum(-1)
        d_s = (gTu[:, :, None] * dcw).sum(1) + (gY[:, :, None] * _hv(hcw, vv)).sum(1)
        d_sS = (gTua[:, :, None] * dcw.abs()).sum(1) + (gYa[:, :, None] * _hv(hcw.abs(), vv.abs())).sum(1)
        if tps is None:
            da[sl], daS[sl] = d_a + d_s, d_aS + d_sS
        else:
            da[sl], daS[sl] = d_a, d_aS
            dtps[sl], dtpsS[sl] = d_s, d_sS
        wb = (cw[:, :, None] * Wc).sum(1)
        gw = (dv[:, :, None] * Wc).sum(1)
        gwa = (dva[:, :, None] * Wc.abs()).sum(1)
        u0 = torch.cat([uu, torch.zeros_like(uu[:, :1])], 1)
        rowv = wb[:, :, None] * u0[:, None, :] + gw[:, :, None] * a1[:, None, :]               # [n,24,4]
        rowa = wb.abs()[:, :, None] * u0.abs()[:, None, :] + gwa[:, :, None] * a1.abs()[:, None, :]
        fi = f[sl]
        dA.index_add_(0, fi, gg[:, None, :, None] * rowv[:, :, None, :])
        dAS.index_add_(0, fi, gg.abs()[:, None, :, None] * rowa[:, :, None, :])
    pad = lambda t: torch.cat([t, torch.zeros_like(t[:, :, :1])], 2)     # noqa: E731
    return (dg, da, dtps, pad(dA)), (dgS, daS, dtpsS, pad(dAS))
