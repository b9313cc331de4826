"""TEST INFRASTRUCTURE ONLY -- the float64 NumPy restatement of csrc/surface_sample.cu (DESIGN section 1h).

`philox4x32_10` is Random123's Philox4x32 with 10 rounds; `sample_surface` is trimesh's `sample_surface` (inverse CDF
over the face areas, a uniform point in the parallelogram folded back into the triangle) driven by that stream, with
the kernel's pinned summation order, so its output rounded to float32 equals the kernel's bit for bit.  `fan` builds
the curve fan of `curve_aware_loss` (OptimGarmentNetwork.py:800-807)."""
import numpy as np

CHUNK = 256
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)


def philox4x32_10(ctr, key):
    """ctr [..., 4] uint32 counters, key (k0, k1) -> [..., 4] uint32."""
    ctr = np.asarray(ctr, dtype=np.uint32)
    x = [ctr[..., i].astype(np.uint32) for i in range(4)]
    k0, k1 = np.uint32(key[0]), np.uint32(key[1])
    with np.errstate(over="ignore"):
        for r in range(10):
            if r > 0:
                k0, k1 = k0 + _W0, k1 + _W1
            p0 = x[0].astype(np.uint64) * _M0
            p1 = x[2].astype(np.uint64) * _M1
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), p0.astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), p1.astype(np.uint32)
            x = [hi1 ^ x[1] ^ k0, lo1, hi0 ^ x[3] ^ k1, lo0]
    return np.stack(x, -1)


def uniforms(seed, counters):
    """(u, a, b) float64 of the samples with 64-bit counters `counters` (uint64 array) under `seed`."""
    seed = int(seed) % (1 << 64)
    c = np.asarray(counters, dtype=np.uint64)
    ctr = np.stack([(c & np.uint64(0xFFFFFFFF)).astype(np.uint32), (c >> np.uint64(32)).astype(np.uint32),
                    np.zeros(c.shape, np.uint32), np.zeros(c.shape, np.uint32)], -1)
    x = philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32)).astype(np.uint64)
    u = ((x[..., 0] << np.uint64(21)) | (x[..., 1] >> np.uint64(11))).astype(np.float64) * 2.0 ** -53
    a = x[..., 2].astype(np.float64) * 2.0 ** -32
    b = x[..., 3].astype(np.float64) * 2.0 ** -32
    fold = (a + b) > 1.0
    a = np.where(fold, 1.0 - a, a)
    b = np.where(fold, 1.0 - b, b)
    return u, a, b


def face_areas(verts, faces):
    """verts [V,3] float32 values, faces [F,3] -> (area [F] float64 with invalid / non-finite faces 0, valid [F])."""
    v = np.asarray(verts, dtype=np.float32).astype(np.float64)
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    V = v.shape[0]
    valid = ((f >= 0) & (f < V)).all(1)
    fi = np.where(valid[:, None], f, 0)
    if V == 0:
        return np.zeros(len(f)), valid
    v0, v1, v2 = v[fi[:, 0]], v[fi[:, 1]], v[fi[:, 2]]
    e1, e2 = v1 - v0, v2 - v0
    with np.errstate(all="ignore"):
        cx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
        cy = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
        cz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
        area = 0.5 * np.sqrt((cx * cx + cy * cy) + cz * cz)
    area = np.where(valid & np.isfinite(area), area, 0.0)
    return area, valid


def cumulative(area):
    """The kernel's pinned order: sequential inside 256-face chunks, sequential over the chunk totals, then
    prefix + local.  np.cumsum is sequential, so for F <= 256 this is np.cumsum itself."""
    F = len(area)
    nch = (F + CHUNK - 1) // CHUNK
    local = np.empty(F)
    tot = np.empty(nch)
    for c in range(nch):
        seg = np.cumsum(area[c * CHUNK:(c + 1) * CHUNK])
        local[c * CHUNK:c * CHUNK + len(seg)] = seg
        tot[c] = seg[-1]
    pre = np.concatenate([[0.0], np.cumsum(tot)[:-1]]) if nch else tot
    return np.repeat(pre, CHUNK)[:F] + local


def sample_mesh(verts, faces, count, seed, offset):
    """One mesh: verts [V,3], faces [F,3] -> ([count,3] float64 points, face index [count]).  Counters offset + s."""
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    if len(f) == 0:
        raise ValueError("sample_mesh: no faces")
    v = np.asarray(verts, dtype=np.float32).astype(np.float64)
    area, valid = face_areas(verts, f)
    C = cumulative(area)
    ctr = (np.uint64(int(offset) % (1 << 64)) + np.arange(count, dtype=np.uint64)) if count else np.zeros(0, np.uint64)
    u, a, b = uniforms(seed, ctr)
    idx = np.searchsorted(C, u * C[-1], side="left")
    ok = valid[idx]
    fi = np.where(ok[:, None], f[idx], 0)
    if v.shape[0] == 0:
        return np.full((count, 3), np.nan), idx
    v0 = v[fi[:, 0]]
    e1, e2 = v[fi[:, 1]] - v0, v[fi[:, 2]] - v0
    with np.errstate(all="ignore"):
        p = (a[:, None] * e1 + b[:, None] * e2) + v0
    p[~ok] = np.nan
    return p, idx


def sample_surface(verts, faces, count, seed, offset=0):
    """M meshes with one face list: verts [M,V,3] -> [M,count,3] float64; mesh m uses counters offset + m*count + s.
    `.astype(np.float32)` of the result is the kernel's output."""
    verts = np.asarray(verts, dtype=np.float32)
    return np.stack([sample_mesh(verts[m], faces, count, seed, int(offset) + m * count)[0]
                     for m in range(verts.shape[0])])


def fan(curve):
    """curve [P,3] -> (verts [P+1,3] with the centroid appended, faces [P,3] int64: (i, i+1, P) and (P-1, 0, P)).
    The centroid is the float32 mean, as `curve_pts.mean(0)` gives it."""
    c = np.asarray(curve, dtype=np.float32)
    P = c.shape[0]
    i = np.arange(P, dtype=np.int64)
    faces = np.stack([i, (i + 1) % P, np.full(P, P, dtype=np.int64)], 1)
    return np.concatenate([c, c.mean(0, dtype=np.float32, keepdims=True)]), faces
