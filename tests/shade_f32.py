"""Float32 restatement of the shading kernels (csrc/shade.cu): the vertex normals and the hard Phong pass.

Every operation of those kernels that produces a value is explicitly rounded (__fadd_rn, __fmul_rn, __fmaf_rn, the
PTX fma.rn), except `powf`, so restating their operation order in NumPy float32 (each ufunc rounds on its own, with
no FMA; render_f32.fma32 is a correctly rounded FMA) gives their outputs bit for bit.  `powf` is the one operation not
restated: `phong` takes the specular term from the caller, either the kernel's own values (read back through a
material that leaves only the specular term, see `spec_only_params`) or a correctly rounded power.  Each step cites
the line it restates.  Written from the documented operation order; no kernel is called.

Also here: the same operation order in float64 with the running error bound S of render_f32.Rb (`normals_bound`,
`phong_bound`), for the float32-vs-float64 tests.
"""
import numpy as np

import render_f32 as rf
from render_f32 import Rb, fma32

f32 = np.float32
EPS = f32(1e-6)
LONG = 256            # segments at least this long are summed with np.add.accumulate, one at a time


def _seq_sums(vals, seg, nseg):
    """Sequential float32 sums from +0 of vals [..., M, 3] grouped by the sorted segment id seg [M], in array order:
    [..., nseg, 3].  Short segments run position by position over all segments at once; long ones (a vertex with 1e5
    faces) run np.add.accumulate, which adds in order."""
    out = np.zeros(vals.shape[:-2] + (nseg, 3), np.float32)
    if not len(seg):
        return out
    start = np.r_[0, np.nonzero(seg[1:] != seg[:-1])[0] + 1]
    length = np.diff(np.r_[start, len(seg)])
    pos = np.arange(len(seg)) - np.repeat(start, length)
    short = np.repeat(length < LONG, length)
    order = np.lexsort((seg, pos))
    order = order[short[order]]
    bounds = np.searchsorted(pos[order], np.arange(LONG + 1))
    with np.errstate(invalid="ignore", over="ignore"):
        for j in range(LONG):
            m = order[bounds[j]:bounds[j + 1]]
            if not len(m):
                break
            out[..., seg[m], :] = out[..., seg[m], :] + vals[..., m, :]
        for s, n in zip(start[length >= LONG], length[length >= LONG]):
            z = np.zeros(vals.shape[:-2] + (1, 3), np.float32)
            out[..., seg[s], :] = np.add.accumulate(np.concatenate([z, vals[..., s:s + n, :]], -2), -2)[..., -1, :]
    return out


def norm2(x, y, z):
    """shade.cu norm2: fma(z, z, fma(x, x, y * y))."""
    with np.errstate(invalid="ignore", over="ignore"):
        return fma32(z, z, fma32(x, x, y * y))


def normalize3(x, y, z):
    """shade.cu normalize3 (and the tail of normals_sum_kernel): v * (1 / max(sqrt(norm2), 1e-6))."""
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        inv = f32(1) / np.fmax(np.sqrt(norm2(x, y, z)), EPS)        # fmaxf returns the non-NaN operand, as np.fmax
        return x * inv, y * inv, z * inv


def _corners(faces, V):
    """The valid (face, corner) entries e = 3 f + k sorted by (vertex, e), as the stable key sort leaves them:
    (e, vertex, b, c) with b, c the corners k + 1 and k + 2."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    ok = ((faces >= 0) & (faces < V)).all(1)                                 # normals_keys_kernel
    e = (3 * np.nonzero(ok)[0][:, None] + np.arange(3)).reshape(-1)
    a = faces.reshape(-1)[e]
    o = np.argsort(a, kind="stable")
    e, a = e[o], a[o]
    f, k = e // 3, e % 3
    return e, a, faces[f, (k + 1) % 3], faces[f, (k + 2) % 3]


def vertex_normals(verts, faces):
    """recmv_vertex_normals: verts [N,V,3] f32, faces [F,3] -> [N,V,3] f32."""
    verts = np.asarray(verts, np.float32)
    N, V = verts.shape[:2]
    _, a, b, c = _corners(faces, V)
    pa, pb, pc = verts[:, a], verts[:, b], verts[:, c]
    with np.errstate(invalid="ignore", over="ignore"):
        u, w = pb - pa, pc - pa                                              # shade.cu:69-70
        cr = np.stack([(u[..., 1] * w[..., 2]) - (u[..., 2] * w[..., 1]),  # :72-74, no contraction
                       (u[..., 2] * w[..., 0]) - (u[..., 0] * w[..., 2]),
                       (u[..., 0] * w[..., 1]) - (u[..., 1] * w[..., 0])], -1)
    s = _seq_sums(cr, a, V)
    return np.stack(normalize3(s[..., 0], s[..., 1], s[..., 2]), -1)


def _rb_sqrt(a):
    with np.errstate(divide="ignore", invalid="ignore"):
        v = np.sqrt(a.v)
        return Rb(v, np.where(v > 0, a.e / (2 * v), 0.0) + v)


def _rb_fmax_eps(a):
    """max(a, 1e-6): the clamp itself is exact; where it applies the value is the constant."""
    c = float(EPS)
    return Rb(np.where(a.v > c, a.v, c), np.where(a.v > c, a.e, 0.0))


def _rb_normalize(x, y, z):
    inv = 1.0 / _rb_fmax_eps(_rb_sqrt(z * z + (x * x + y * y)))   # an FMA rounds once where the bound counts twice
    return x * inv, y * inv, z * inv


def normals_bound(verts, faces):
    """vertex_normals' operation order in float64, with the running bound S of every output: 3 Rb [N,V].  The
    per-vertex sums carry each partial sum's magnitude, so a vertex whose contributions cancel to about 0 gets a
    bound far above its value."""
    verts = np.asarray(verts, np.float64)
    N, V = verts.shape[:2]
    _, a, b, c = _corners(faces, V)
    pa, pb, pc = Rb(verts[:, a]), Rb(verts[:, b]), Rb(verts[:, c])
    u, w = pb - pa, pc - pa
    ux, uy, uz, wx, wy, wz = (t[..., i] for t in (u, w) for i in range(3))
    cr = [(uy * wz) - (uz * wy), (uz * wx) - (ux * wz), (ux * wy) - (uy * wx)]
    # sequential sums: value and bound (bound += e_term + |partial sum|), in the kernel's order
    start = np.r_[0, np.nonzero(a[1:] != a[:-1])[0] + 1] if len(a) else np.zeros(0, np.int64)
    sums = []
    for t in cr:
        v = np.zeros((N, V))
        e = np.zeros((N, V))
        if len(a):
            first = np.repeat(start, np.diff(np.r_[start, len(a)]))         # each entry's segment start
            csum = np.concatenate([np.zeros((N, 1)), np.cumsum(t.v, axis=1)], 1)
            partial = csum[:, 1:] - csum[:, first]                           # the running sum after each entry
            e_run = t.e + np.abs(partial) + rf.TINY
            v[:, a[start]] = np.add.reduceat(t.v, start, axis=1)
            e[:, a[start]] = np.add.reduceat(e_run, start, axis=1)
        sums.append(Rb(v, e))
    return _rb_normalize(*sums)


# ---- Phong ----------------------------------------------------------------------------------------------------------
def _fragments(pix_to_face, faces, N, V, F):
    """The covered pixels and their (frame n of the pixel, frame m of the face, corner vertices) (shade.cu:100-111)."""
    p = np.asarray(pix_to_face, np.int64).reshape(N, -1)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    Fk = F if V > 0 else 0                                  # recmv_shade_phong passes F = 0 when V = 0
    cov = (p >= 0) & (p < N * Fk)
    m, f = np.divmod(np.where(cov, p, 0), max(Fk, 1))
    fi = faces[f] if Fk else np.zeros(p.shape + (3,), np.int64)
    cov &= ((fi >= 0) & (fi < V)).all(-1)
    n_, q_ = np.nonzero(cov)
    return cov, n_, q_, m[cov], fi[cov]


def phong(pix_to_face, bary, verts, normals, colors, faces, params, spec=None):
    """recmv_shade_phong: pix_to_face [N,H,W] int64, bary [N,H,W,3] f32, verts / normals / colors [N,V,3] f32 (colors
    None = 1), faces [F,3], params [N,28] f32 -> (rgba [N,H,W,4] f32, sa [N,H,W] f32 of covered pixels (0 elsewhere)).
    spec [N,H,W] is powf(sa, shininess) per pixel; None takes the correctly rounded power."""
    verts, normals = np.asarray(verts, np.float32), np.asarray(normals, np.float32)
    params = np.asarray(params, np.float32).reshape(-1, 28)
    pix_to_face = np.asarray(pix_to_face, np.int64)
    N, H, W = pix_to_face.shape
    V = verts.shape[1]
    F = np.asarray(faces).reshape(-1, 3).shape[0]
    cov, n_, q_, m, fi = _fragments(pix_to_face, faces, N, V, F)
    out = np.empty((N, H * W, 4), np.float32)
    out[..., :3] = params[:, None, 25:28]                                     # shade.cu:101-103, :109
    out[..., 3] = 1
    sa_out = np.zeros((N, H * W), np.float32)
    b = np.asarray(bary, np.float32).reshape(N, H * W, 3)[n_, q_]
    prm = params[n_]
    col = np.ones_like(verts) if colors is None else np.asarray(colors, np.float32)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        def interp(attr):                                                     # :116-124, fma chain from +0
            acc = np.zeros((len(m), 3), np.float32)
            for k in range(3):
                acc = fma32(b[:, k:k + 1], attr[m, fi[:, k]], acc)
            return acc
        P, Nr, C = interp(verts), interp(normals), interp(col)
        nx, ny, nz = normalize3(Nr[:, 0], Nr[:, 1], Nr[:, 2])                # :125-126
        lx, ly, lz = normalize3(prm[:, 3] - P[:, 0], prm[:, 4] - P[:, 1], prm[:, 5] - P[:, 2])    # :127-128
        vx, vy, vz = normalize3(prm[:, 0] - P[:, 0], prm[:, 1] - P[:, 1], prm[:, 2] - P[:, 2])    # :129-130
        cosl = fma32(nz, lz, fma32(nx, lx, ny * ly))                          # :132
        c2 = f32(2) * cosl
        rx, ry, rz = fma32(nx, c2, -lx), fma32(ny, c2, -ly), fma32(nz, c2, -lz)                  # :133-134
        sa = np.where(cosl > 0, np.fmax(fma32(vz, rz, fma32(vx, rx, vy * ry)), f32(0)), f32(0)).astype(np.float32)  # :135
        if spec is None:
            sp = pow_rn(sa, prm[:, 24])
        else:
            sp = np.asarray(spec, np.float32).reshape(N, H * W)[n_, q_]
        dif = np.fmax(cosl, f32(0))                                           # :137
        for j in range(3):                                                    # :140-145
            d = (prm[:, 18 + j] * prm[:, 9 + j]) * dif
            s = (prm[:, 21 + j] * prm[:, 12 + j]) * sp
            out[n_, q_, j] = fma32(fma32(prm[:, 15 + j], prm[:, 6 + j], d), C[:, j], s)
    sa_out[n_, q_] = sa
    return out.reshape(N, H, W, 4), sa_out.reshape(N, H, W)


def pow_rn(x, y):
    """x^y correctly rounded to float32 (float64 pow is within an ulp of float64, far inside half a float32 ulp except
    next to a float32 tie), with C's powf special cases for x = 0 and y = 0."""
    x64, y64 = np.asarray(x, np.float64), np.asarray(y, np.float64)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        return np.power(x64, y64).astype(np.float32)


def spec_only_params(params):
    """params with ambient and diffuse material colours 0 and specular light and material colours 1: every output
    channel of a covered pixel is then (1 * 1) * powf(sa, shininess) exactly, since fma(0, la, 0 * dif) = 0 and
    fma(0, C, s) = s for finite C."""
    p = np.array(params, np.float32, copy=True).reshape(-1, 28)
    p[:, 12:15] = 1
    p[:, 15:21] = 0
    p[:, 21:24] = 1
    return p


def phong_bound(pix_to_face, bary, verts, normals, colors, faces, params):
    """phong's operation order in float64 with running bounds S: (rgb list of 3 Rb over the covered pixels, covered
    mask [N,H*W], sa Rb).  Inputs are the float32 values (exact).  The power adds its own rounding and carries sa's bound
    through its derivative; an FMA rounds once where the bound counts two roundings, so S bounds it."""
    params = np.asarray(params, np.float64).reshape(-1, 28)
    pix_to_face = np.asarray(pix_to_face, np.int64)
    N, H, W = pix_to_face.shape
    verts, normals = np.asarray(verts, np.float64), np.asarray(normals, np.float64)
    V = verts.shape[1]
    F = np.asarray(faces).reshape(-1, 3).shape[0]
    cov, n_, q_, m, fi = _fragments(pix_to_face, faces, N, V, F)
    b = np.asarray(bary, np.float64).reshape(N, H * W, 3)[n_, q_]
    prm = params[n_]
    col = np.ones_like(verts) if colors is None else np.asarray(colors, np.float64)

    def interp(attr, j):
        acc = Rb(np.zeros(len(m)))
        for k in range(3):
            acc = Rb(b[:, k]) * Rb(attr[m, fi[:, k], j]) + acc
        return acc

    P = [interp(verts, j) for j in range(3)]
    C = [interp(col, j) for j in range(3)]
    nx, ny, nz = _rb_normalize(*[interp(normals, j) for j in range(3)])
    lx, ly, lz = _rb_normalize(*[Rb(prm[:, 3 + j]) - P[j] for j in range(3)])
    vx, vy, vz = _rb_normalize(*[Rb(prm[:, j]) - P[j] for j in range(3)])
    cosl = nz * lz + (nx * lx + ny * ly)
    c2 = 2.0 * cosl
    rx, ry, rz = nx * c2 - lx, ny * c2 - ly, nz * c2 - lz
    dot = vz * rz + (vx * rx + vy * ry)
    on = (cosl.v > 0) & (dot.v > 0)
    sa = Rb(np.where(on, dot.v, 0.0), np.where(on, dot.e, 0.0))
    sh = prm[:, 24]
    with np.errstate(divide="ignore", invalid="ignore"):
        sp_v = np.power(sa.v, sh)
        dsp = np.where(sa.v > 0, sh * sp_v / np.where(sa.v > 0, sa.v, 1.0), 0.0)
    sp = Rb(sp_v, dsp * sa.e + np.abs(sp_v) + rf.TINY)
    dif = Rb(np.maximum(cosl.v, 0.0), np.where(cosl.v > 0, cosl.e, 0.0))
    rgb = []
    for j in range(3):
        d = (Rb(prm[:, 18 + j]) * Rb(prm[:, 9 + j])) * dif
        s = (Rb(prm[:, 21 + j]) * Rb(prm[:, 12 + j])) * sp
        rgb.append((Rb(prm[:, 15 + j]) * Rb(prm[:, 6 + j]) + d) * C[j] + s)
    return rgb, cov, sa
