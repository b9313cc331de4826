"""TEST INFRASTRUCTURE ONLY -- the NumPy restatement of csrc/train_rays.cu (DESIGN section 1j), the training-ray
sub-sampling of `sample_train_ray` (OptimGarmentNetwork.py:983-1055).

`uniforms` is the kernel's u = (x0 >> 8) 2^-24 from sample_oracle's Philox4x32-10; `select` gives the kept input
indices of one garment; `view_rays32` restates the kernel's fp32 view ray (each operation rounded in float32, so it
equals the kernel bit for bit) and raster_oracle.view_rays is the float64 one; `sample` runs G garments of a call."""
import numpy as np

from . import raster_oracle, sample_oracle


def uniforms(seed, counters):
    """float32 u in [0, 1) of the 64-bit counters (uint64 array) under `seed`: the first Philox word's top 24 bits."""
    seed = int(seed) % (1 << 64)
    c = np.asarray(counters, dtype=np.uint64)
    ctr = np.stack([(c & np.uint64(0xFFFFFFFF)).astype(np.uint32), (c >> np.uint64(32)).astype(np.uint32),
                    np.zeros(c.shape, np.uint32), np.zeros(c.shape, np.uint32)], -1)
    x0 = sample_oracle.philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))[..., 0]
    return (x0 >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)


def threshold(target, pnum):
    """fp32(double(target) / double(pnum)): what torch compares a float32 tensor with for the Python float quotient."""
    return np.float32(float(target) / float(pnum))


def counters(offset, base, pnum):
    """uint64 counters offset + base + j of a garment's pnum candidates, modulo 2^64."""
    return np.uint64((int(offset) + int(base)) % (1 << 64)) + np.arange(pnum, dtype=np.uint64)


def candidates(mask, batch, row, col):
    """Input indices with mask[b, r, c] > 0 (NaN fails; an index outside the mask is not a candidate), in order."""
    mask = np.asarray(mask, dtype=np.float32)
    N, H, W = mask.shape
    b, r, c = (np.asarray(x, dtype=np.int64) for x in (batch, row, col))
    inside = (b >= 0) & (b < N) & (r >= 0) & (r < H) & (c >= 0) & (c < W)
    v = np.zeros(len(b), np.float32)
    v[inside] = mask[b[inside], r[inside], c[inside]]
    return np.flatnonzero(inside & (v > 0))


def select(mask, batch, row, col, target, seed, offset, base):
    """Kept input indices of one garment whose list starts at counter offset + base."""
    cand = candidates(mask, batch, row, col)
    pnum = len(cand)
    if pnum <= target:
        return cand
    return cand[uniforms(seed, counters(offset, base, pnum)) < threshold(target, pnum)]


def view_rays32(cols, rows, cam):
    """The kernel's fp32 view rays of pixels (col, row) under cam = {fx, fy, px, py, R row-major, ...} (>= 13 values,
    raster.camera_rows' layout) -> [P,3] float32."""
    c = np.asarray(cam, dtype=np.float32).reshape(-1)
    fx, fy, px, py, R = c[0], c[1], c[2], c[3], c[4:13].reshape(3, 3)
    x = np.asarray(cols).astype(np.float32)
    y = np.asarray(rows).astype(np.float32)
    v0 = -x / fx + px / fx
    v1 = -y / fy + py / fy
    v2 = np.ones_like(v0)
    nrm = np.sqrt((v0 * v0 + v1 * v1) + v2 * v2)
    v = [v0 / nrm, v1 / nrm, v2 / nrm]
    return np.stack([(v[0] * R[i, 0] + v[1] * R[i, 1]) + v[2] * R[i, 2] for i in range(3)], 1).reshape(-1, 3)


def view_rays64(cols, rows, cam):
    """The float64 view rays (raster_oracle.view_rays) under the same camera values."""
    c = np.asarray(cam, dtype=np.float32).reshape(-1)[:13]
    return raster_oracle.view_rays(np.asarray(cols, np.float64), np.asarray(rows, np.float64), c)


def sample(masks, batch, row, col, target, seed, offset, cam=None):
    """G garments of one call: lists of (kept input indices[, fp32 rays]) and the next offset, offset + sum P_g."""
    out, base = [], 0
    for g in range(len(masks)):
        keep = select(masks[g], batch[g], row[g], col[g], target, seed, offset, base)
        rays = view_rays32(np.asarray(col[g])[keep], np.asarray(row[g])[keep], cam) if cam is not None else None
        out.append((keep, rays))
        base += len(batch[g])
    return out, (int(offset) + base) % (1 << 64)
