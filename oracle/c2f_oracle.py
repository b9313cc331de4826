"""Plain-torch restatement of one level of the coarse-to-fine sweep (DESIGN.md section 1, A11;
recmv_b200/MCAcc/seg3d_lossless.py:_forward_torch), cut into the pieces the worklist kernels of csrc/c2f.cu compute, so
each kernel can be checked on its own with any values in place of the network:

    refine        coarse occ / done -> fine occ / done and the SET of voxels to query
    query_points  level voxel indices -> the fp32 points batch_eval hands to the query function
    scatter       queried values -> occ / done / calculated, and the conflicting voxels
    next_round    conflicts -> the not-yet-evaluated 3x3x3 neighbours, each once

Everything is dense masks and whole-array arithmetic (no Python loop over voxels), fp32 with one rounding per operation,
and runs on whichever device its inputs live on.  Sets are returned as sorted flat indices of the level lattice
[D, H, W] (x fastest).  tests/test_c2f_oracle_cpu.py pins the pieces, chained, to Seg3dLossless._forward_torch."""
import torch
import torch.nn.functional as F


def stride(level_whd, final_whd):
    """Level step in final-lattice units per axis (x, y, z)."""
    return tuple((f - 1) // (l - 1) if l > 1 else 1 for l, f in zip(level_whd, final_whd))


def _up(t, dim, pair):
    """2n-1 upsampling along `dim`: even positions copy, odd positions pair(left, right)."""
    n = t.shape[dim]
    shape = list(t.shape)
    shape[dim] = 2 * n - 1
    out = t.new_empty(shape)
    ev = [slice(None)] * t.dim()
    od = list(ev)
    ev[dim], od[dim] = slice(0, None, 2), slice(1, None, 2)
    out[tuple(ev)] = t
    if n > 1:
        out[tuple(od)] = pair(t.narrow(dim, 0, n - 1), t.narrow(dim, 1, n - 1))
    return out


def upsample(occ, balance):
    """occ [D,H,W] f32 -> (values [2D-1,2H-1,2W-1], mixed flag): trilinear with align_corners=True, nested x, y, z
    with weights 1/2 (every product exact, one rounding per addition); the flag is set where the 1, 2, 4 or 8 coarse
    voxels a fine voxel interpolates are not all on one side of `balance` (`>` is inside; NaN counts as not inside)."""
    half = lambda a, b: 0.5 * a + 0.5 * b
    v, inside = occ, occ > balance
    any_in, any_out = inside, ~inside
    for dim in (2, 1, 0):
        v = _up(v, dim, half)
        any_in, any_out = _up(any_in, dim, torch.logical_or), _up(any_out, dim, torch.logical_or)
    return v, any_in & any_out


def dilate(mask):
    """3x3x3 dilation of a bool [D,H,W] lattice, zero padding at the border."""
    return F.max_pool3d(mask[None, None].float(), 3, stride=1, padding=1)[0, 0] > 0


def refine(occ_c, done_c, balance, values=None):
    """One level: (occ_f, done_f bool, todo indices).  `values`: the interpolated lattice when it comes from another
    rounding of the same map (the order-0 upsampler); the flags and sets never depend on it."""
    v, mixed = upsample(occ_c, balance)
    done_f = torch.zeros(v.shape, dtype=torch.bool, device=v.device)
    done_f[::2, ::2, ::2] = done_c.bool()
    todo = dilate(mixed) & ~done_f
    return (v if values is None else values), done_f, todo.view(-1).nonzero().view(-1)


def query_points(idx, level_whd, final_whd, b_min, b_max):
    """fp32 points of the level voxels `idx`: c = coords / res + (1 / res) / 2; p = c (b_max - b_min) + b_min."""
    W, H, _ = level_whd
    dev = idx.device
    s = torch.tensor(stride(level_whd, final_whd), device=dev)
    xyz = torch.stack([idx % W, (idx // W) % H, idx // (W * H)], 1) * s
    res = torch.tensor(final_whd, device=dev)
    step = 1.0 / res.float()
    c = xyz.float() / res + step / 2
    lo, hi = torch.tensor(b_min, dtype=torch.float32, device=dev), torch.tensor(b_max, dtype=torch.float32, device=dev)
    return c * (hi - lo) + lo


def _final_index(idx, level_whd, final_whd):
    W, H, _ = level_whd
    sx, sy, sz = stride(level_whd, final_whd)
    return ((idx // (W * H)) * sz * final_whd[1] + ((idx // W) % H) * sy) * final_whd[0] + (idx % W) * sx


def scatter(idx, vals, occ, done, calculated, balance, level_whd, final_whd):
    """Writes `vals` at `idx` (in place: occ f32 [D,H,W], done bool, calculated bool on the FINAL lattice) and returns
    the conflicting indices, sorted: (interpolated - balance) * (queried - balance) < 0 in fp32."""
    flat = occ.view(-1)
    interp = flat[idx]
    conflict = (interp - balance) * (vals - balance) < 0
    flat[idx] = vals
    done.view(-1)[idx] = True
    calculated.view(-1)[_final_index(idx, level_whd, final_whd)] = True
    return idx[conflict].sort().values


def next_round(conflicts, calculated, level_whd, final_whd):
    """Sorted indices of the 3x3x3 neighbours (level steps, clamped to the lattice) of `conflicts` that were not
    evaluated at any level."""
    W, H, D = level_whd
    sx, sy, sz = stride(level_whd, final_whd)
    m = torch.zeros((D, H, W), dtype=torch.bool, device=calculated.device)
    m.view(-1)[conflicts] = True
    m = dilate(m) & ~calculated[::sz, ::sy, ::sx][:D, :H, :W]
    return m.view(-1).nonzero().view(-1)
