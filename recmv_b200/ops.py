"""Torch-facing wrappers over the C ABI: allocate outputs, pass raw pointers + the current stream,
raise on non-zero status, wire autograd.  PyTorch is plumbing here (device memory, streams,
autograd graph); all arithmetic happens in librecmv_b200.so.
"""
import collections
import contextlib
import ctypes
import functools
import itertools
from ctypes import byref, c_float, c_size_t

import torch

from . import _lib
from ._lib import (F32, F64, LAYOUT_NCDHW, LAYOUT_NDHWC, MLP_FP32_SIMT, MLP_TC_F16X1, MLP_TC_F16X3,
                   RayMarch, Voxel, check)

DEFAULT_MLP_MODE = MLP_TC_F16X3


def _stream(t):
    return ctypes.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _launch(name, like, *args):
    """Call the export `name` with args and the current stream of like's device, under that device's guard; raise on a
    non-zero status."""
    with torch.cuda.device(like.device):
        check(getattr(_lib.load(), name)(*args, _stream(like)), name)


def _size(name, *args, dev=None):
    """Value of a size query (`*_bytes`, `*_workspace`, `*_floats`): returned by the export, or written to a trailing
    size_t* after a status that is checked.  dev: the device the size depends on (SM count, library sort sizes); the
    query then runs under its guard."""
    fn = getattr(_lib.load(), name)
    with torch.cuda.device(dev) if dev is not None else contextlib.nullcontext():
        if fn.restype is c_size_t:
            return int(fn(*args))
        n = c_size_t(0)
        check(fn(*args, byref(n)), name)
    return int(n.value)


# (device index, name) -> what a call keeps on that device for the next one, like the MCGpu singleton
# (MCGpu/CudaKernels.cu:524-604): grow-only buffers, pinned counters, and the rasterizers' pair-list capacities.
# Every caller uses its own names.
_scratch_cache = {}


def _scratch(dev, name, rows, dtype=torch.uint8, tail=()):
    """Grow-only per-device buffer [>= rows, *tail]: reallocated (contents dropped) only when the one kept is smaller."""
    buf = _scratch_cache.get((dev.index, name))
    if buf is None or buf.shape[0] < rows:
        buf = _scratch_cache[(dev.index, name)] = torch.empty((rows,) + tuple(tail), dtype=dtype, device=dev)
    return buf


def _counters(dev, name, n):
    """(int32 [n] device counters, their pinned host copy), zeroed when first made and kept per device."""
    key = (dev.index, name)
    if key not in _scratch_cache:
        _scratch_cache[key] = (torch.zeros((n,), dtype=torch.int32, device=dev),
                               torch.zeros((n,), dtype=torch.int32).pin_memory())
    return _scratch_cache[key]


def _read_counters(ctr, host):
    """Copy the device counters to their pinned host copy and wait for the current stream: the call's one host sync."""
    host.copy_(ctr, non_blocking=True)
    torch.cuda.current_stream(ctr.device).synchronize()
    return host


def _ptr_array(ts):
    """Device pointers of a list of tensors (None for a missing one) as a host void*[len(ts)]."""
    return (ctypes.c_void_p * len(ts))(*[t.data_ptr() if t is not None else None for t in ts])


FLOATS = (torch.float32, torch.float64)    # an operand dtype of the ops that run in either precision


def _dtype_code(dtype):
    return {torch.float32: F32, torch.float64: F64}[dtype]


def _operands(fn, *specs):
    """Refuse (RuntimeError) any operand a kernel of `fn` would misread; return the bound shape symbols.

    A spec is (t, name, dtype, shape).  t: a tensor; None, an absent optional operand, passes; a list of tensors is
    checked element by element as name[i] with the same symbols.  dtype: a torch dtype, or a tuple of accepted dtypes
    that binds like a symbol (key "dtype").  shape entries: an int fixes an extent; a str is a symbol, bound at its first
    use and equal at every later one; None accepts any extent; a callable of the bindings so far gives an extent derived
    from them (row_ptr's V + 1).  A leading ... stands for any number of leading extents whose product binds like a
    symbol (key ...): the point count P of a [..., 3] point tensor that a kernel reads as numel / 3 rows.
    The dtype, extents and contiguity of every operand are checked in argument order, then that all of them sit on one
    CUDA device, so that nothing is allocated, sized or launched for a call that is refused."""
    ops = []
    for t, name, dtype, shape in specs:
        if isinstance(t, (list, tuple)):
            ops += [(x, f"{name}[{i}]", dtype, shape) for i, x in enumerate(t)]
        elif t is not None:
            ops.append((t, name, dtype, shape))
    bound, source = {}, {}
    if not ops:
        return bound
    dev = ops[0][0].get_device()     # -1 for a CPU tensor

    def refuse(t, name, dtype, shape, why="", keys=()):
        label = {Ellipsis: "the product of the leading extents"}
        why += "".join(f" ({label.get(k, k)} is {bound[k]} from {source[k]})" for k in keys)
        want = "|".join(map(str, dtype)) if isinstance(dtype, tuple) else dtype
        dims = ",".join("..." if s is Ellipsis else "*" if s is None else str(s(bound)) if callable(s) else str(s)
                        for s in shape)
        where = f"CUDA device cuda:{dev}" if dev >= 0 else "a CUDA device"
        raise RuntimeError(f"{fn}: {name} must be {want} [{dims}] on {where}, got {t.dtype} {tuple(t.shape)} on "
                           f"{t.device}{why}")

    for t, name, dtype, shape in ops:
        if isinstance(dtype, tuple):
            if t.dtype not in dtype or t.dtype is not bound.setdefault("dtype", t.dtype):
                refuse(t, name, dtype, shape, keys=["dtype"] if "dtype" in source else [])
            source.setdefault("dtype", name)
        elif t.dtype is not dtype:
            refuse(t, name, dtype, shape)
        sizes = t.shape
        if shape and shape[0] is Ellipsis:
            k = len(sizes) - len(shape) + 1
            if k < 0:
                refuse(t, name, dtype, shape)
            sizes = (sizes[:k].numel(),) + tuple(sizes[k:])
        elif len(sizes) != len(shape):
            refuse(t, name, dtype, shape)
        for s, n in zip(shape, sizes):
            if s is None:
                continue
            if isinstance(s, int):
                if n != s:
                    refuse(t, name, dtype, shape)
            elif callable(s):
                if n != s(bound):
                    refuse(t, name, dtype, shape, keys=[b for b in bound if b != "dtype"])
            elif n != bound.setdefault(s, n):
                refuse(t, name, dtype, shape, keys=[s])
            else:
                source.setdefault(s, name)
        if not t.is_contiguous():
            refuse(t, name, dtype, shape, " (not contiguous)")
    for t, name, dtype, shape in ops:
        if not t.is_cuda:
            refuse(t, name, dtype, shape, " (not a CUDA tensor)")
        if t.get_device() != dev:
            refuse(t, name, dtype, shape, f" (not on cuda:{dev}, where {ops[0][1]} is)")
    return bound


# --------------------------------------------------------------------------------------------------
# FastMinv
# --------------------------------------------------------------------------------------------------
def minv3x3(ms):
    """FastMinv.Fast3x3Minv(ms) -> [invs, checks]  (FastMinv/M3x3Inv.cpp:12-37)."""
    d = _operands("minv3x3", (ms, "ms", FLOATS, ("n", 3, 3)))
    n = d["n"]
    invs = torch.empty((n, 3, 3), dtype=ms.dtype, device=ms.device)
    ok = torch.empty((n,), dtype=torch.uint8, device=ms.device)
    _launch("recmv_minv3x3_fwd", ms, _ptr(ms), _ptr(invs), _ptr(ok), n, _dtype_code(d["dtype"]))
    return [invs, ok.view(torch.bool)]


def minv3x3_backward(grads, invs):
    """FastMinv.Fast3x3Minv_backward(grads, invs) -> outs  (FastMinv/M3x3Inv.cpp:39-59)."""
    d = _operands("minv3x3_backward", (grads, "grads", FLOATS, ("n", 3, 3)), (invs, "invs", FLOATS, ("n", 3, 3)))
    n = d["n"]
    outs = torch.empty((n, 3, 3), dtype=invs.dtype, device=invs.device)
    _launch("recmv_minv3x3_bwd", invs, _ptr(grads), _ptr(invs), _ptr(outs), n, _dtype_code(d["dtype"]))
    return outs


class FastDiff3x3MinvFunction(torch.autograd.Function):
    """utils/utils.py:8-18."""

    @staticmethod
    def forward(ctx, input):
        invs, chk = minv3x3(input.contiguous())
        ctx.save_for_backward(invs, chk)
        ctx.mark_non_differentiable(chk)
        return invs, chk

    @staticmethod
    def backward(ctx, grad_input, grad_check):
        invs, _ = ctx.saved_tensors
        return minv3x3_backward(grad_input.contiguous(), invs), None


# --------------------------------------------------------------------------------------------------
# GridSamplerMine
# --------------------------------------------------------------------------------------------------
# the grid sampler's operands: input [N,C,D,H,W] (NCDHW) or [N,D,H,W,C] (NDHWC), grid [N,a,b,c,3] read as [N,P,3]
# with P = a b c, the output cotangent [N,C,a,b,c]
_GS_INPUT = {LAYOUT_NCDHW: ("N", "C", "D", "H", "W"), LAYOUT_NDHWC: ("N", "D", "H", "W", "C")}
_GS_GRID = ("N", "a", "b", "c", 3)
_GS_OUT = ("N", "C", "a", "b", "c")


def _gs_args(d):
    return d["N"], d["C"], d["D"], d["H"], d["W"], d["a"] * d["b"] * d["c"], _dtype_code(d["dtype"])


def grid_sample3d_forward(inp, grid, layout=LAYOUT_NCDHW):
    """GridSamplerMine.forward(input, grid, 0, 1)  (MCAcc/cuda/GridSamplerMine.cpp:75-81)."""
    d = _operands("grid_sample3d_forward", (inp, "input", FLOATS, _GS_INPUT[layout]), (grid, "grid", FLOATS, _GS_GRID))
    out = torch.empty((d["N"], d["C"], d["a"], d["b"], d["c"]), dtype=inp.dtype, device=inp.device)
    _launch("recmv_gridsample3d_fwd", inp, _ptr(inp), _ptr(grid), _ptr(out), *_gs_args(d), layout)
    return out


def grid_sample3d_backward(inp, grid, grad_out, layout=LAYOUT_NCDHW, need_grad_input=True):
    """GridSamplerMine.backward(input, grid, grad_output, 0, 1) -> (grad_input, grad_grid)."""
    grad_out = grad_out.contiguous()
    d = _operands("grid_sample3d_backward", (inp, "input", FLOATS, _GS_INPUT[layout]), (grid, "grid", FLOATS, _GS_GRID),
                  (grad_out, "grad_output", FLOATS, _GS_OUT))
    gi = torch.zeros_like(inp) if need_grad_input else None
    gg = torch.empty_like(grid)
    _launch("recmv_gridsample3d_bwd", inp, _ptr(inp), _ptr(grid), _ptr(grad_out), _ptr(gi), _ptr(gg), *_gs_args(d),
            layout)
    return gi, gg


def grid_sample3d_dbackward(gg_input, gg_grid, inp, grid, grad_out, layout=LAYOUT_NCDHW,
                            need_grad_input=True):
    """GridSamplerMine.dbackward(ggI, ggG, input, grid, grad_output, 0, 1) -> (gI, gG, ggO)."""
    grad_out = grad_out.contiguous()
    gg_grid = gg_grid.contiguous()
    gg_input = gg_input.contiguous() if gg_input is not None else None
    d = _operands("grid_sample3d_dbackward", (gg_input, "gg_input", FLOATS, _GS_INPUT[layout]),
                  (gg_grid, "gg_grid", FLOATS, _GS_GRID), (inp, "input", FLOATS, _GS_INPUT[layout]),
                  (grid, "grid", FLOATS, _GS_GRID), (grad_out, "grad_output", FLOATS, _GS_OUT))
    gi = torch.zeros_like(inp) if need_grad_input else None
    gg = torch.empty_like(grid)
    ggo = torch.empty_like(grad_out)
    _launch("recmv_gridsample3d_bwd2", inp, _ptr(gg_input), _ptr(gg_grid), _ptr(inp), _ptr(grid), _ptr(grad_out),
            _ptr(gi), _ptr(gg), _ptr(ggo), *_gs_args(d), layout)
    return gi, gg, ggo


class GridSamplerMine3dFunction(torch.autograd.Function):
    """MCAcc/grid_sampler_mine.py:8-46 -- twice differentiable trilinear/border sampler."""

    @staticmethod
    def forward(ctx, input, grid, mode="bilinear", padding_mode="border", align_corners=False):
        if align_corners:
            raise NotImplementedError
        input = input.contiguous()
        grid = grid.contiguous()
        ctx.save_for_backward(input, grid)
        return grid_sample3d_forward(input, grid)

    @staticmethod
    def backward(ctx, grad_output):
        input, grid = ctx.saved_tensors
        o0, o1 = GridSamplerMine3dBackwardFunction.apply(input, grid, grad_output)
        return o0, o1, None, None, None


class GridSamplerMine3dBackwardFunction(torch.autograd.Function):
    """MCAcc/grid_sampler_mine.py:48-65.  grad_input is only materialised when the voxel itself
    requires grad (the reference always fills a full zero volume, GridSamplerMineKernel.cu:955)."""

    @staticmethod
    def forward(ctx, input, grid, grad_output):
        ctx.save_for_backward(input, grid, grad_output)
        ctx.need_gi = bool(input.requires_grad)
        gi, gg = grid_sample3d_backward(input, grid, grad_output, need_grad_input=ctx.need_gi)
        if gi is None:
            gi = input.new_zeros(())  # placeholder, never consumed (input does not require grad)
            ctx.mark_non_differentiable(gi)
        return gi, gg

    @staticmethod
    def backward(ctx, grad_output_input, grad_output_grid):
        input, grid, grad_output = ctx.saved_tensors
        ggi = grad_output_input if ctx.need_gi else None
        if grad_output_grid is None:
            grad_output_grid = torch.zeros_like(grid)
        o0, o1, o2 = grid_sample3d_dbackward(ggi, grad_output_grid, input, grid, grad_output,
                                             need_grad_input=ctx.need_gi)
        return o0, o1, o2


class FrozenVoxelSampleFunction(torch.autograd.Function):
    """Twice-differentiable trilinear / border sample of a FROZEN channels-last voxel [1,D,H,W,C] (the cached layout of
    LBSkinner.ws: one corner = C contiguous floats) -- the autograd path of LBSkinner.forward.  Same kernels as
    GridSamplerMine3dFunction (recmv_gridsample3d_{fwd,bwd,bwd2}) with layout NDHWC; the voxel gets no gradient."""

    @staticmethod
    def forward(ctx, voxel_cl, grid):
        grid = grid.contiguous()
        ctx.save_for_backward(voxel_cl, grid)
        return grid_sample3d_forward(voxel_cl, grid, LAYOUT_NDHWC)

    @staticmethod
    def backward(ctx, grad_output):
        voxel_cl, grid = ctx.saved_tensors
        return None, _FrozenVoxelSampleBackward.apply(voxel_cl, grid, grad_output)


class _FrozenVoxelSampleBackward(torch.autograd.Function):
    @staticmethod
    def forward(ctx, voxel_cl, grid, grad_output):
        ctx.save_for_backward(voxel_cl, grid, grad_output)
        return grid_sample3d_backward(voxel_cl, grid, grad_output, LAYOUT_NDHWC, need_grad_input=False)[1]

    @staticmethod
    def backward(ctx, gg_grid):
        voxel_cl, grid, grad_output = ctx.saved_tensors
        _, g_grid, gg_out = grid_sample3d_dbackward(None, gg_grid.contiguous(), voxel_cl, grid, grad_output, LAYOUT_NDHWC,
                                                    need_grad_input=False)
        return None, g_grid, gg_out


def voxel_to_channels_last(ws):
    """[1,C,D,H,W] fp32 -> [D,H,W,C] (private, coalesced copy of LBSkinner.ws)."""
    d = _operands("voxel_to_channels_last", (ws, "ws", torch.float32, (1, "C", "D", "H", "W")))
    C, D, H, W = d["C"], d["D"], d["H"], d["W"]
    out = torch.empty((D, H, W, C), dtype=torch.float32, device=ws.device)
    _launch("recmv_voxel_to_channels_last", ws, _ptr(ws), _ptr(out), C, D, H, W)
    return out


# --------------------------------------------------------------------------------------------------
# skinning-voxel construction (model/Deformer.py:533-591, utils/LBSWsmpl.py)
# --------------------------------------------------------------------------------------------------
def lbsw_knn_blend(verts, vert_ws, bmin, bmax, resolution, k, align_corners=False, want_idx=False):
    """k-nearest-vertex blend of the skinning weights at every voxel centre (recmv_lbsw_knn_blend).
    verts [V,3], vert_ws [V,24] fp32 CUDA; bmin / bmax: 3 host floats; resolution (W,H,D).
    Returns ws_cl [D,H,W,24] (and idx [D*H*W,k] int32, nearest first, when want_idx)."""
    d = _operands("lbsw_knn_blend", (verts, "verts", torch.float32, ("V", 3)),
                  (vert_ws, "vert_ws", torch.float32, ("V", "C")))
    W, H, D = (int(r) for r in resolution)
    V, C = d["V"], d["C"]
    out = torch.empty((D, H, W, C), dtype=torch.float32, device=verts.device)
    idx = torch.empty((D * H * W, k), dtype=torch.int32, device=verts.device) if want_idx else None
    lo, hi = (c_float * 3)(*[float(v) for v in bmin]), (c_float * 3)(*[float(v) for v in bmax])
    _launch("recmv_lbsw_knn_blend", verts, _ptr(verts), _ptr(vert_ws), V, C, lo, hi, W, H, D, int(bool(align_corners)),
            int(k), _ptr(out), _ptr(idx))
    return (out, idx) if want_idx else out


def lbsw_smooth(ws_cl, times, zero_below=0.0):
    """`times` passes of the reference's smooth_weights on a channels-last [D,H,W,24] voxel (recmv_lbsw_smooth), then
    values below zero_below (if > 0) set to 0.  `ws_cl` is consumed (used as the first ping-pong buffer).
    Returns (ws [1,24,D,H,W], ws_cl [D,H,W,24]) -- the second is what LBSkinner samples."""
    d = _operands("lbsw_smooth", (ws_cl, "ws_cl", torch.float32, ("D", "H", "W", 24)))
    D, H, W, C = d["D"], d["H"], d["W"], 24
    spare = torch.empty_like(ws_cl) if times >= 2 else None
    out = torch.empty((1, C, D, H, W), dtype=torch.float32, device=ws_cl.device)
    out_cl = torch.empty_like(ws_cl)
    _launch("recmv_lbsw_smooth", ws_cl, _ptr(ws_cl), _ptr(spare), D, H, W, int(times), float(zero_below), _ptr(out),
            _ptr(out_cl))
    return out, out_cl


# --------------------------------------------------------------------------------------------------
# MCGpu
# --------------------------------------------------------------------------------------------------
def mc_gpu(sdfs, xstep=1.0, ystep=1.0, zstep=1.0, xmin=0.0, ymin=0.0, zmin=0.0, fTargetValue=0.0):
    """MCGpu.mc_gpu(sdfs, steps, mins, iso) -> [verts [V,3] f32, faces [F,3] i64]
    (MCGpu/MCGpu.cpp:20-56).  Wrong dtype returns [] exactly like the reference (:41-42).

    One C call queues every pass (sign mask, count, scan, vertices, faces) into grow-only capacity buffers; the single
    host synchronisation is the read of (V, F) AFTER everything is queued (the reference blocks between its kernels,
    CudaKernels.cu:628).  The results are fresh tensors, as the reference returns (MCGpu.cpp:49-54).  The one-grid case
    of mc_gpu_many."""
    if not (sdfs.is_cuda and sdfs.is_contiguous()):   # CHECK_INPUT (MCGpu/MCGpu.cpp:3-5), before the dtype test
        raise RuntimeError(f"mc_gpu: sdfs must be a contiguous CUDA tensor, got {tuple(sdfs.shape)} on {sdfs.device}")
    if sdfs.dtype != torch.float32 or sdfs.dim() != 3 or min(sdfs.shape) <= 0:
        return []
    return mc_gpu_many([sdfs], [(xstep, ystep, zstep)], [(xmin, ymin, zmin)], fTargetValue)[0]


def mc_gpu_many(grids, steps, origins, iso=0.0, capacity=(4096, 8192)):
    """mc_gpu on every grid with one host synchronisation: grids, float32 CUDA [NX,NY,NZ] on one device; steps and
    origins, one (x, y, z) per grid; one iso value.  Returns [[verts, faces], ...], each bit-identical to mc_gpu on that
    grid.  Every grid's run is queued before the one read of all (V, F, overflow) counters; only the grids whose output
    buffers overflowed are re-run, once, after growing them to their counts.  capacity: the (vertex, face) rows a grid's
    output buffers hold at least at the first run (buffers kept from earlier calls may be larger).

    Grid i writes its mesh into its own cached output buffers, so no later grid overwrites it before the read.  The
    scratch (sign mask, segment sums, packed vertex words) is one buffer of the largest grid's size: each run consumes
    it before the next one on the stream starts, and the counts leave it with the run."""
    if not (len(grids) == len(steps) == len(origins)):
        raise RuntimeError("mc_gpu_many: grids, steps and origins must have the same length")
    if not grids:
        return []
    _operands("mc_gpu_many", (grids, "grids", torch.float32, (None, None, None)))
    if any(min(g.shape) <= 0 for g in grids):
        raise RuntimeError("mc_gpu_many: every grid must be non-empty")
    dev = grids[0].device
    dims = [tuple(int(n) for n in g.shape) for g in grids]
    scratch = _scratch(dev, "mc_scratch", max(_size("recmv_mc_scratch_bytes", *d) for d in dims))
    n = len(grids)
    ctr, host = _counters(dev, ("mc_counters", n), 4 * n)
    caps = [tuple(capacity)] * n
    todo, out = list(range(n)), [None] * n
    for _ in range(2):
        bufs = {}
        for i in todo:
            verts = _scratch(dev, ("mc_verts", i), caps[i][0], torch.float32, (3,))
            faces = _scratch(dev, ("mc_faces", i), caps[i][1], torch.int64, (3,))
            _launch("recmv_mc_run", grids[i], _ptr(grids[i]), *dims[i], float(iso), _ptr(scratch),
                    (c_float * 3)(*steps[i]), (c_float * 3)(*origins[i]), _ptr(verts), verts.shape[0], _ptr(faces),
                    faces.shape[0], _ptr(ctr[4 * i:4 * i + 4]))
            bufs[i] = verts, faces
        h = _read_counters(ctr, host).view(n, 4).tolist()
        again = []
        for i in todo:
            V, F, overflow = h[i][:3]
            if V >= (1 << 25):
                check(_lib.RECMV_E_RANGE, "recmv_mc_run (more than 2^25 vertices)")
            if overflow:
                caps[i] = int(V * 1.25) + 1024, int(F * 1.25) + 2048   # grow once, re-run (buffers are kept)
                again.append(i)
            else:
                out[i] = [bufs[i][0][:V].clone(), bufs[i][1][:F].clone()]
        todo = again
        if not todo:
            return out
    raise _lib.RecmvError("recmv_mc_run: output buffers still too small after growing")


def vertex_faces(faces, V, check_indices=False):
    """The vertex-face incidence of faces [F,3] int64 CUDA over V vertices (recmv_vertex_faces, DESIGN section 1o):
    (fid [3F], vid [3F] int64), one pair per face corner, grouped by ascending vertex and, within a vertex, ascending
    face.  The flattened `TmpFid` / `TmpVid` that OptimGarmentNetwork.marching_cube_update builds from openmesh's
    vertex_face_indices(), in a pinned order.  A face with an index outside [0, V) gives (-1, -1) pairs at the end and
    sets a device flag; check_indices=True reads that flag (one host synchronisation) and raises ValueError when it is
    set.  Otherwise nothing is read back."""
    F = _operands("vertex_faces", (faces, "faces", torch.int64, ("F", 3)))["F"]
    dev, V = faces.device, int(V)
    fid = torch.empty((3 * F,), dtype=torch.int64, device=dev)
    vid = torch.empty((3 * F,), dtype=torch.int64, device=dev)
    flag, host = _counters(dev, "vertex_faces_flag", 1)
    ws = _scratch(dev, "vertex_faces_ws", _size("recmv_vertex_faces_workspace_bytes", F, V, dev=dev))
    _launch("recmv_vertex_faces", faces, _ptr(faces), F, V, _ptr(ws), _ptr(fid), _ptr(vid), _ptr(flag))
    if check_indices and int(_read_counters(flag, host)[0]):
        raise ValueError(f"vertex_faces: a face has an index outside [0, {V})")
    return fid, vid


# --------------------------------------------------------------------------------------------------
# LBS
# --------------------------------------------------------------------------------------------------
# operand shapes shared by the skinning, deformer, render and surface-solve wrappers
_POINTS = (..., 3)              # points the kernels read as P = numel / 3 rows of 3
_BONES = ("F", 24, 4, 4)        # A of F frames; trans is [F,3]
_VOXEL = ("D", "H", "W", 24)    # the channels-last skinning voxel ws_cl


def _voxel(ws_cl, center, extend):
    v = Voxel()
    v.ws_cl = ws_cl.data_ptr()
    v.D, v.H, v.W = int(ws_cl.shape[0]), int(ws_cl.shape[1]), int(ws_cl.shape[2])
    v.center = (c_float * 3)(*[float(x) for x in center])
    v.extend = float(extend)
    return v


def make_voxel(ws_cl, center, extend):
    """The recmv_voxel_t of the channels-last voxel ws_cl [D,H,W,24] f32 (CUDA, contiguous) and its box."""
    _operands("make_voxel", (ws_cl, "ws_cl", torch.float32, _VOXEL))
    return _voxel(ws_cl, center, extend)


def lbs_forward(ps, A, trans, ws_cl, center, extend, batch_inds=None, points_per_frame=0, tps=None,
                want_weights=False):
    ps = ps.contiguous().float()
    A = A.contiguous().float()
    trans = trans.contiguous().float()
    if tps is not None:
        tps = tps.contiguous().float()
    if batch_inds is not None:
        batch_inds = batch_inds.contiguous().long()
    d = _operands("lbs_forward", (ps, "ps", torch.float32, _POINTS), (A, "A", torch.float32, _BONES),
                  (trans, "trans", torch.float32, ("F", 3)), (ws_cl, "ws_cl", torch.float32, _VOXEL),
                  (batch_inds, "batch_inds", torch.int64, (...,)), (tps, "tps", torch.float32, _POINTS))
    P = d[...]
    out = torch.empty_like(ps)
    wout = torch.empty((P, 24), dtype=torch.float32, device=ps.device) if want_weights else None
    _launch("recmv_lbs_fwd", ps, _ptr(ps), _ptr(tps), _ptr(A), _ptr(trans), _ptr(batch_inds), int(points_per_frame),
            d["F"], byref(_voxel(ws_cl, center, extend)), _ptr(out), _ptr(wout), P)
    return (out, wout) if want_weights else out


def lbs_inverse(x_obs, A, trans, ws_cl, center, extend, batch_inds=None, points_per_frame=0):
    x_obs = x_obs.contiguous().float()
    A = A.contiguous().float()
    trans = trans.contiguous().float()
    if batch_inds is not None:
        batch_inds = batch_inds.contiguous().long()
    d = _operands("lbs_inverse", (x_obs, "x_obs", torch.float32, _POINTS), (A, "A", torch.float32, _BONES),
                  (trans, "trans", torch.float32, ("F", 3)), (ws_cl, "ws_cl", torch.float32, _VOXEL),
                  (batch_inds, "batch_inds", torch.int64, (...,)))
    P = d[...]
    xc = torch.empty_like(x_obs)
    valid = torch.empty((P,), dtype=torch.uint8, device=x_obs.device)
    _launch("recmv_lbs_inverse", x_obs, _ptr(x_obs), _ptr(A), _ptr(trans), _ptr(batch_inds), int(points_per_frame),
            d["F"], byref(_voxel(ws_cl, center, extend)), _ptr(xc), _ptr(valid), P)
    return xc, valid.view(torch.bool)


def bone_matrices(poses, Js, parents_i32, init_pose=None, want_A=True):
    """(G [F,24,4,4], A [F,24,4,4] or None): the kinematic chain of LBSkinner in one launch (no autograd)."""
    poses = poses.detach().contiguous().float()
    Js = Js.contiguous().float()
    ip = init_pose.contiguous().float() if init_pose is not None else None
    F_ = _operands("bone_matrices", (poses, "poses", torch.float32, ("F", 24, 3)), (Js, "Js", torch.float32, (24, 3)),
                   (parents_i32, "parents_i32", torch.int32, (24,)), (ip, "init_pose", torch.float32, (24, 4, 4)))["F"]
    dev = poses.device
    G = torch.empty((F_, 24, 4, 4), dtype=torch.float32, device=dev)
    A = torch.empty((F_, 24, 4, 4), dtype=torch.float32, device=dev) if want_A else None
    _launch("recmv_bone_matrices", poses, _ptr(poses), _ptr(Js), _ptr(parents_i32), _ptr(ip), _ptr(G), _ptr(A), F_)
    return G, A


def bone_matrices_backward(poses, Js, parents_i32, init_pose, G, dG=None, dA=None):
    """dposes [F,24,3] = VJP of bone_matrices at `poses` (G: its output); dG / dA: cotangents of G / A or None."""
    poses = poses.detach().contiguous().float()
    Js = Js.contiguous().float()
    ip = init_pose.contiguous().float() if init_pose is not None else None
    G = G.contiguous()
    dG = dG.contiguous().float() if dG is not None else None
    dA = dA.contiguous().float() if dA is not None else None
    F_ = _operands("bone_matrices_backward", (poses, "poses", torch.float32, ("F", 24, 3)),
                   (Js, "Js", torch.float32, (24, 3)), (parents_i32, "parents_i32", torch.int32, (24,)),
                   (ip, "init_pose", torch.float32, (24, 4, 4)), (G, "G", torch.float32, _BONES),
                   (dG, "dG", torch.float32, _BONES), (dA, "dA", torch.float32, _BONES))["F"]
    dposes = torch.empty((F_, 24, 3), dtype=torch.float32, device=poses.device)
    _launch("recmv_bone_matrices_backward", poses, _ptr(poses), _ptr(Js), _ptr(parents_i32), _ptr(ip), _ptr(G), _ptr(dG),
            _ptr(dA), _ptr(dposes), F_)
    return dposes


class BoneMatricesFunction(torch.autograd.Function):
    """(G, A) of the kinematic chain (recmv_bone_matrices) with its VJP on the device (recmv_bone_matrices_backward): the
    autograd path of LBSkinner.bone_matrices / posedSkeleton when the poses are trained.  poses [F,24,3] fp32.
    First order only: nothing in the training step differentiates the skeleton twice."""

    @staticmethod
    def forward(ctx, poses, Js, parents_i32, init_pose):
        G, A = bone_matrices(poses, Js, parents_i32, init_pose)
        ctx.save_for_backward(poses, G)
        ctx.Js, ctx.parents, ctx.init_pose = Js, parents_i32, init_pose
        return G, A

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dG, dA):
        poses, G = ctx.saved_tensors
        if not ctx.needs_input_grad[0]:
            return None, None, None, None
        return bone_matrices_backward(poses, ctx.Js, ctx.parents, ctx.init_pose, G, dG, dA), None, None, None


def lbs_backward(ps, A, grad_out, ws_cl, center, extend, batch_inds=None, points_per_frame=0, tps=None,
                 want_ps=True, want_tps=True, want_A=True, want_trans=True):
    """(dps, dtps, dA, dtrans) of lbs_forward for the cotangent grad_out [P,3] (recmv_lbs_backward); an output that is not
    wanted (or dtps without tps) is None."""
    ps = ps.contiguous().float()
    A = A.contiguous().float()
    g = grad_out.contiguous().float()
    if tps is not None:
        tps = tps.contiguous().float()
    if batch_inds is not None:
        batch_inds = batch_inds.contiguous().long()
    d = _operands("lbs_backward", (ps, "ps", torch.float32, _POINTS), (A, "A", torch.float32, _BONES),
                  (g, "grad_out", torch.float32, _POINTS), (ws_cl, "ws_cl", torch.float32, _VOXEL),
                  (batch_inds, "batch_inds", torch.int64, (...,)), (tps, "tps", torch.float32, _POINTS))
    P, F_, dev = d[...], d["F"], ps.device
    dps = torch.empty((P, 3), dtype=torch.float32, device=dev) if want_ps else None
    dtps = torch.empty((P, 3), dtype=torch.float32, device=dev) if want_tps and tps is not None else None
    dA = torch.empty((F_, 24, 4, 4), dtype=torch.float32, device=dev) if want_A else None
    dtrans = torch.empty((F_, 3), dtype=torch.float32, device=dev) if want_trans else None
    nbytes = _size("recmv_lbs_backward_workspace_bytes", P, F_)
    work = torch.empty((max(nbytes, 16),), dtype=torch.uint8, device=dev) if (want_A or want_trans) else None
    _launch("recmv_lbs_backward", ps, _ptr(ps), _ptr(tps), _ptr(A), None, _ptr(batch_inds), int(points_per_frame), F_,
            byref(_voxel(ws_cl, center, extend)), _ptr(g), _ptr(dps), _ptr(dtps), _ptr(dA), _ptr(dtrans), _ptr(work), P)
    return dps, dtps, dA, dtrans


def lbs_vjp_backward(ps, A, grad_out, ws_cl, center, extend, batch_inds=None, points_per_frame=0, tps=None,
                     cot_ps=None, cot_tps=None, want_grad_out=True, want_ps=True, want_tps=True, want_A=True):
    """(d_grad_out, dps, dtps, dA) of the point outputs (dps, dtps) of lbs_backward, for their cotangents cot_ps /
    cot_tps [P,3] (recmv_lbs_vjp_backward; a missing cotangent is zero, cot_tps needs tps).  An output that is not
    wanted (or dtps without tps) is None."""
    ps = ps.contiguous().float()
    A = A.contiguous().float()
    g = grad_out.contiguous().float()
    if tps is not None:
        tps = tps.contiguous().float()
    else:
        cot_tps = None
    if batch_inds is not None:
        batch_inds = batch_inds.contiguous().long()
    cot_ps = cot_ps.contiguous().float() if cot_ps is not None else None
    cot_tps = cot_tps.contiguous().float() if cot_tps is not None else None
    d = _operands("lbs_vjp_backward", (ps, "ps", torch.float32, _POINTS), (A, "A", torch.float32, _BONES),
                  (g, "grad_out", torch.float32, _POINTS), (ws_cl, "ws_cl", torch.float32, _VOXEL),
                  (batch_inds, "batch_inds", torch.int64, (...,)), (tps, "tps", torch.float32, _POINTS),
                  (cot_ps, "cot_ps", torch.float32, _POINTS), (cot_tps, "cot_tps", torch.float32, _POINTS))
    P, F_, dev = d[...], d["F"], ps.device
    if cot_ps is None and cot_tps is None:
        cot_ps = torch.zeros_like(ps)
    dg = torch.empty((P, 3), dtype=torch.float32, device=dev) if want_grad_out else None
    dps = torch.empty((P, 3), dtype=torch.float32, device=dev) if want_ps else None
    dtps = torch.empty((P, 3), dtype=torch.float32, device=dev) if want_tps and tps is not None else None
    dA = torch.empty((F_, 24, 4, 4), dtype=torch.float32, device=dev) if want_A else None
    work = None
    if want_A:
        work = torch.empty((max(_size("recmv_lbs_backward_workspace_bytes", P, F_), 16),), dtype=torch.uint8, device=dev)
    _launch("recmv_lbs_vjp_backward", ps, _ptr(ps), _ptr(tps), _ptr(A), _ptr(batch_inds), int(points_per_frame), F_,
            byref(_voxel(ws_cl, center, extend)), _ptr(g), _ptr(cot_ps), _ptr(cot_tps), _ptr(dg), _ptr(dps), _ptr(dtps),
            _ptr(dA), _ptr(work), P)
    return dg, dps, dtps, dA


class LbsVjpFunction(torch.autograd.Function):
    """(dps, dtps) = the point gradients of lbs_backward for the cotangent g, as a differentiable op: forward
    recmv_lbs_backward with only dps / dtps, backward recmv_lbs_vjp_backward (d g, d ps, d tps, d A).  ps / tps / g
    [P,3] fp32, A [F,24,4,4]; dtps is None when tps is None.  This is the create_graph backward of LbsTrainFunction for
    input gradients (the train-phase Jacobians); its own backward is first order."""

    @staticmethod
    def forward(ctx, ps, tps, A, g, batch_inds, ppf, skin):
        ws_cl, center, extend = skin
        dps, dtps, _, _ = lbs_backward(ps, A, g, ws_cl, center, extend, batch_inds, ppf, tps, want_ps=True,
                                       want_tps=True, want_A=False, want_trans=False)
        ctx.save_for_backward(ps, tps, A, g, batch_inds)
        ctx.skin, ctx.ppf = skin, ppf
        return dps, dtps

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, u, v):
        ps, tps, A, g, batch_inds = ctx.saved_tensors
        need = ctx.needs_input_grad
        want_tps = need[1] and tps is not None
        if not (need[0] or want_tps or need[2] or need[3]):
            return None, None, None, None, None, None, None
        ws_cl, center, extend = ctx.skin
        dg, dps, dtps, dA = lbs_vjp_backward(ps, A, g, ws_cl, center, extend, batch_inds, ctx.ppf, tps, u,
                                             v if tps is not None else None, want_grad_out=need[3], want_ps=need[0],
                                             want_tps=want_tps, want_A=need[2])
        return dps, dtps, dA, dg, None, None, None


class LbsTrainFunction(torch.autograd.Function):
    """LBSkinner.forward with gradients for the poses / translations (and the points): forward recmv_lbs_fwd, backward
    recmv_lbs_backward (weights resampled, not kept in the graph).  ps [...,3] contiguous fp32 ([N,V,3] with frame = row,
    or [P,3] with batch_inds); tps None or the sampling points of the `[tps, ps]` form; A [F,24,4,4]; trans [F,3].
    `skin` = (ws_cl, center, extend).  A backward under create_graph (the train-phase Jacobians of utils) that asks for
    input gradients only (`input_grad_only()`), with `second_order_fused`, returns LbsVjpFunction's differentiable point
    gradients; any other backward under create_graph evaluates `composite(ps, tps, A, trans)` -- the torch-sampler graph
    of LBSkinner -- on the saved inputs and differentiates it with create_graph=True.  `last_backward` says which branch
    ran."""
    last_backward = None

    @staticmethod
    def forward(ctx, ps, tps, A, trans, batch_inds, skin, composite, second_order_fused=False):
        ws_cl, center, extend = skin
        ppf = 0 if batch_inds is not None else ps.shape[1]
        out = lbs_forward(ps.reshape(-1, 3), A, trans, ws_cl, center, extend, batch_inds, ppf,
                          None if tps is None else tps.reshape(-1, 3))
        ctx.save_for_backward(ps, tps, A, trans, batch_inds)
        ctx.skin, ctx.composite, ctx.ppf = skin, composite, ppf
        ctx.second_order_fused = second_order_fused
        return out.view(ps.shape)

    @staticmethod
    def backward(ctx, g):
        ps, tps, A, trans, batch_inds = ctx.saved_tensors
        need = ctx.needs_input_grad
        if torch.is_grad_enabled() and ctx.second_order_fused and _inputs_only(need[2] or need[3]):
            # create_graph=True for the point gradients only: (dps, dtps) as a differentiable op on the device
            LbsTrainFunction.last_backward = "fused (create_graph, input gradient)"
            dps, dtps = LbsVjpFunction.apply(ps.reshape(-1, 3), None if tps is None else tps.reshape(-1, 3), A,
                                             g.reshape(-1, 3), batch_inds, ctx.ppf, ctx.skin)
            dps = dps.view(ps.shape) if need[0] else None
            dtps = dtps.view(tps.shape) if (dtps is not None and need[1]) else None
            return dps, dtps, None, None, None, None, None, None
        if torch.is_grad_enabled():
            LbsTrainFunction.last_backward = "autograd-composite (create_graph)"
            return (*_composite_grads(ctx.composite, [ps, tps, A, trans], [g]), None, None, None, None)
        LbsTrainFunction.last_backward = "fused"
        ws_cl, center, extend = ctx.skin
        dps, dtps, dA, dtrans = lbs_backward(ps.reshape(-1, 3), A, g.reshape(-1, 3), ws_cl, center, extend, batch_inds,
                                             ctx.ppf, None if tps is None else tps.reshape(-1, 3), want_ps=need[0],
                                             want_tps=need[1], want_A=need[2], want_trans=need[3])
        dps = dps.view(ps.shape) if dps is not None else None
        dtps = dtps.view(tps.shape) if dtps is not None else None
        return dps, dtps, dA, dtrans, None, None, None, None


# --------------------------------------------------------------------------------------------------
# SDF MLP
# --------------------------------------------------------------------------------------------------
SDF_LAYER_SHAPES = [(512, 39), (512, 512), (512, 512), (473, 512), (512, 512), (512, 512), (512, 512),
                    (512, 512), (257, 512)]


def _aligned_blob(nbytes, dev):
    """nbytes of device memory at a 1 KiB boundary (the TMA-visible weight planes need it)."""
    raw = torch.empty((nbytes + 1024,), dtype=torch.uint8, device=dev)
    off = (-raw.data_ptr()) % 1024
    blob = raw[off:off + nbytes]
    blob._keepalive = raw
    return blob


def _pack_weights(net, label, shapes, Ws, bs):
    """Ws[l] [out,in], bs[l] [out] of the layers in `shapes` -> the device blob of recmv_{net}_pack_weights."""
    for (o, i), W, b in zip(shapes, Ws, bs):
        if tuple(W.shape) != (o, i) or tuple(b.shape) != (o,):
            raise RuntimeError(f"unexpected {label} layer shape {tuple(W.shape)} (want {(o, i)})")
    W_all = torch.cat([W.detach().reshape(-1).float() for W in Ws]).contiguous()
    b_all = torch.cat([b.detach().reshape(-1).float() for b in bs]).contiguous()
    _operands(f"{net}_pack_weights", (W_all, "Ws", torch.float32, (None,)), (b_all, "bs", torch.float32, (None,)))
    packed = _aligned_blob(_packed_bytes(net), W_all.device)
    _launch(f"recmv_{net}_pack_weights", W_all, _ptr(W_all), _ptr(b_all), _ptr(packed))
    return packed


@functools.cache
def _packed_bytes(net):
    """Length of a packed weight blob of `net` (recmv_{net}_packed_bytes): the shape its operand checks demand."""
    return _size(f"recmv_{net}_packed_bytes")


def sdf_pack_weights(Ws, bs):
    """Ws[l] [out,in] effective fp32 weights (weight-norm applied), bs[l] [out] -> packed device blob."""
    return _pack_weights("sdf", "SDF", SDF_LAYER_SHAPES, Ws, bs)


def _pe_array(pe_w):
    pe_w = [1.0] * 12 if pe_w is None else [float(w) for w in pe_w]
    if len(pe_w) != 12:
        raise RuntimeError("pe_w must hold 12 annealing weights")
    return (c_float * 12)(*pe_w)


def sdf_mlp_forward(x, packed, pe_w=None, mode=None, want_feat=True):
    """ImplicitNetwork.forward on canonical points x [P,3] -> (sdf [P,1], feat [P,256] or None)."""
    mode = DEFAULT_MLP_MODE if mode is None else mode
    x = x.contiguous().float()
    P = _operands("sdf_mlp_forward", (x, "x", torch.float32, ("P", 3)),
                  (packed, "packed", torch.uint8, (_packed_bytes("sdf"),)))["P"]
    sdf = torch.empty((P, 1), dtype=torch.float32, device=x.device)
    feat = torch.empty((P, 256), dtype=torch.float32, device=x.device) if want_feat else None
    _launch("recmv_sdf_mlp_fwd", x, _ptr(x), _ptr(packed), _pe_array(pe_w), _ptr(sdf), _ptr(feat), P, mode)
    return sdf, feat


def sdf_value_and_grad(x, packed, pe_w=None, mode=None, want_feat=False):
    """(sdf [P,1], d sdf/d x [P,3], feat or None) in ONE forward-mode launch (no graph is recorded)."""
    mode = DEFAULT_MLP_MODE if mode is None else mode
    if mode == MLP_FP32_SIMT:
        raise _lib.RecmvError("the fused value+gradient launch exists for the tensor-core modes only")
    x = x.contiguous().float()
    P = _operands("sdf_value_and_grad", (x, "x", torch.float32, ("P", 3)),
                  (packed, "packed", torch.uint8, (_packed_bytes("sdf"),)))["P"]
    sdf = torch.empty((P, 1), dtype=torch.float32, device=x.device)
    grad = torch.empty((P, 3), dtype=torch.float32, device=x.device)
    feat = torch.empty((P, 256), dtype=torch.float32, device=x.device) if want_feat else None
    _launch("recmv_sdf_mlp_fwd_grad", x, _ptr(x), _ptr(packed), _pe_array(pe_w), _ptr(sdf), _ptr(feat), _ptr(grad), P,
            mode)
    return sdf, grad, feat


# --------------------------------------------------------------------------------------------------
# Training path: layer GEMMs that save their outputs for the backward (csrc/gemm3_tma.cu)
# --------------------------------------------------------------------------------------------------
import os as _os
# create_graph=True input gradients: "1" = differentiable reverse chain on the tensor-core GEMMs (second_order.py), "0" = torch graph
SECOND_ORDER_FUSED = _os.environ.get("RECMV_SECOND_ORDER", "1") != "0"
_INPUT_GRAD_ONLY = [0]


class input_grad_only:
    """`with ops.input_grad_only(): torch.autograd.grad(y, x, ..., create_graph=True)` -- tells the training Functions that
    this differentiation asks for INPUT gradients only (ctx.needs_input_grad cannot: it reflects requires_grad at forward
    time, and the parameters always require grad while training).  The mirrors of the reference's call sites use it
    (ImplicitNetwork.gradient, utils.compute_Jacobian, utils.compute_deformed_normals).  The backward runs on autograd's
    device thread, so the flag is process-wide, not thread-local (one process drives one GPU)."""

    def __enter__(self):
        _INPUT_GRAD_ONLY[0] += 1
        return self

    def __exit__(self, *exc):
        _INPUT_GRAD_ONLY[0] -= 1
        return False


def _inputs_only(need_params):
    return SECOND_ORDER_FUSED and (not need_params or _INPUT_GRAD_ONLY[0] > 0)


def _composite_grads(composite, inputs, cotangents):
    """The create_graph=True backward of a training Function that is not its fused input gradient: differentiate the
    torch composite `composite(*inputs)` (a tensor or a tuple of them) for the output cotangents with a graph.  An input
    may be None; a None cotangent skips its output.  Returns one gradient per input, None where it does not require
    grad."""
    ins = [t if t is None or t.requires_grad else t.detach() for t in inputs]
    with torch.enable_grad():
        outs = composite(*ins)
        outs = outs if isinstance(outs, tuple) else (outs,)
        used = [(o, g) for o, g in zip(outs, cotangents) if g is not None]
        diff = [t for t in ins if t is not None and t.requires_grad]
        gr = iter(torch.autograd.grad([o for o, _ in used], diff, [g for _, g in used], create_graph=True,
                                      allow_unused=True))
    return [next(gr) if t is not None and t.requires_grad else None for t in ins]


_INV_SQRT2 = 0.70710678118654752440


def grad_dyn_scale(*cotangents):
    """Device scalar 2^-floor(log2(max|g|)) (1 for an all-zero cotangent): brings the largest cotangent entry into
    [1, 2) before the fp16 hi/lo split of the backward GEMMs; no host synchronisation."""
    m = torch.stack([c.detach().abs().amax() for c in cotangents if c is not None]).amax().float()
    e = torch.floor(torch.log2(m.clamp_min(1e-30)))
    s = torch.exp2(-e.clamp(-100.0, 100.0))
    return torch.where(m > 0, s, torch.ones_like(s)).reshape(1).contiguous()


def pe_forward(x, pe_w, bands, out, out2=None):
    """out[:, :3 + 6 bands] (and out2) = positional encoding of x [P,3] with annealing weights pe_w.  Callers: the
    translator and colour networks' training forwards build their input rows with it."""
    w = (c_float * (2 * bands))(*[float(v) for v in pe_w[:2 * bands]])
    _launch("recmv_pe_forward", x, _ptr(x), w, int(bands), _ptr(out), out.stride(0), _ptr(out2),
            out2.stride(0) if out2 is not None else 0, x.shape[0])
    return out


def _pad8(n):
    return (int(n) + 7) // 8 * 8


def _plane_pair(rows, cols, dev, zero=False):
    """(hi, lo) fp16 [rows, cols] operand-plane buffers."""
    mk = torch.zeros if zero else torch.empty
    return (mk((rows, cols), dtype=torch.float16, device=dev), mk((rows, cols), dtype=torch.float16, device=dev))


def split_planes(t, rows, cols, scale, scale_dev=None, transpose=False, ldp=None):
    """fp32 [rows, >= cols] -> (hi, lo) fp16 planes of scale (* scale_dev) * t, [rows][ldp] or transposed [cols][ldp]."""
    dev = t.device
    ldp = ldp or _pad8(rows if transpose else cols)
    shape = (cols, ldp) if transpose else (rows, ldp)
    hi = torch.zeros(shape, dtype=torch.float16, device=dev)
    lo = torch.zeros(shape, dtype=torch.float16, device=dev)
    _launch("recmv_split_planes", t, _ptr(t), t.stride(0), int(rows), int(cols), float(scale), _ptr(scale_dev),
            1 if transpose else 0, _ptr(hi), _ptr(lo), ldp)
    return hi, lo


def weight_planes(W, transpose=False):
    """Operand planes of a layer's weight matrix ([out][in], scale 1024; transpose=True: [in][out], the backward-data
    operand), computed once per tensor OBJECT and version: the forward, the reverse chain and the two second-order passes of
    one training step all see the same weight tensor, so three of four splits are cache hits.  The cache lives on the tensor
    (an attribute), so it dies with it -- no address-keyed table that could go stale."""
    if W.is_leaf:
        # a Parameter can be rewritten through `.data` without a version bump: never cache on leaves (weight-normed layers
        # hand over a fresh non-leaf W = g v / |v| every forward, which is the case the cache is for)
        Wd = W.detach().contiguous().float()
        return split_planes(Wd, Wd.shape[0], Wd.shape[1], 1024.0, transpose=transpose)
    ver = W._version
    cache = getattr(W, "_recmv_planes", None)
    if cache is None or cache[0] != ver:
        cache = (ver, {})
        try:
            W._recmv_planes = cache
        except AttributeError:
            pass
    if transpose not in cache[1]:
        Wd = W.detach().contiguous().float()
        cache[1][transpose] = split_planes(Wd, Wd.shape[0], Wd.shape[1], 1024.0, transpose=transpose)
    return cache[1][transpose]


def pe_forward_planes(x, pe_w, bands, out, out_hi, out_lo):
    w = (c_float * (2 * bands))(*[float(v) for v in pe_w[:2 * bands]])
    _launch("recmv_pe_forward_planes", x, _ptr(x), w, int(bands), _ptr(out), out.stride(0) if out is not None else 0,
            _ptr(out_hi), _ptr(out_lo), out_hi.stride(0), x.shape[0])


def mlp_layer_planes(a_planes, b_planes, M, N, K, mode, Y, bias=None, saved_input=None, scale=1.0, dyn=None, a_has_dyn=False,
                     split=0, Y2=None, y_planes=None, planes_with_dyn=False):
    """One TMA-fed layer GEMM on operand planes (recmv_mlp_layer_planes); modes: 4/5/6 forward none/softplus/relu,
    0/1/2 backward-data none/softplus'/relu'."""
    ah, al = a_planes
    bh, bl = b_planes
    yh, yl = y_planes if y_planes is not None else (None, None)
    _launch("recmv_mlp_layer_planes", Y,
            _ptr(ah), _ptr(al), ah.stride(0), _ptr(bh), _ptr(bl), bh.stride(0), int(M), int(N), int(K), int(mode), _ptr(bias),
            _ptr(saved_input), saved_input.stride(0) if saved_input is not None else 0, float(scale), _ptr(dyn),
            1 if a_has_dyn else 0, int(split), _ptr(Y), Y.stride(0), _ptr(Y2), Y2.stride(0) if Y2 is not None else 0, _ptr(yh),
            _ptr(yl), yh.stride(0) if yh is not None else 0, 1 if planes_with_dyn else 0)
    return Y


def _wgrad_workspace(dev):
    """fp32 scratch of the weight gradient: (the GEMM's split partials, sized for dev's SM count; the colsum partials)."""
    return (_scratch(dev, "wgrad", _size("recmv_mlp_wgrad_workspace_floats", dev=dev), torch.float32),
            _scratch(dev, "colsum", 128 * 512, torch.float32))


def mlp_wgrad_planes(g_planes, x_planes, P, out_dim, in_dim, scale=1.0, dyn=None, want_bias=False):
    """dW [out_dim, in_dim] = scale * G^T X from the operand planes the layer GEMMs wrote (recmv_mlp_wgrad_planes); with
    want_bias also db [out_dim] = sum over samples of g (same launch) -> (dW, db)."""
    gh, gl = g_planes
    xh, xl = x_planes
    dev = gh.device
    ws, _ = _wgrad_workspace(dev)
    dW = torch.empty((out_dim, in_dim), dtype=torch.float32, device=dev)
    db = torch.empty((out_dim,), dtype=torch.float32, device=dev) if want_bias else None
    _launch("recmv_mlp_wgrad_planes", gh, _ptr(gh), _ptr(gl), gh.stride(0), _ptr(xh), _ptr(xl), xh.stride(0), int(P),
            int(out_dim), int(in_dim), float(scale), _ptr(dyn), _ptr(ws), _ptr(dW), _ptr(db))
    return (dW, db) if want_bias else dW


def colsum(G, cols):
    """sum over rows of G[:, :cols] (fp32, deterministic two-stage reduction): the bias gradient."""
    _, part = _wgrad_workspace(G.device)
    out = torch.empty((cols,), dtype=torch.float32, device=G.device)
    _launch("recmv_colsum", G, _ptr(G), G.stride(0), G.shape[0], int(cols), _ptr(part), _ptr(out))
    return out


def softplus_tangent_planes(tz, a, h, cols, u, u_planes, inj, plane_scale=64.0):
    """u[:, :cols] = softplus_100'(z) * tz (+ planes), inj[:, :cols] = softplus_100''(z) * (h / softplus') * tz, from the saved
    softplus output a (second_order.py's tangent pass; one launch)."""
    _launch("recmv_softplus_tangent_planes", tz,
            _ptr(tz), tz.stride(0), _ptr(a), a.stride(0), _ptr(h), h.stride(0), tz.shape[0], int(cols), float(plane_scale), _ptr(u),
            u.stride(0), _ptr(u_planes[0]), _ptr(u_planes[1]), u_planes[0].stride(0), _ptr(inj), inj.stride(0))


def add_split_planes(y, addend, cols, y_planes, scale=64.0, scale_dev=None):
    """y[:, :cols] += addend[:, :cols] in place, and the planes of the sum scaled scale (* scale_dev)."""
    _launch("recmv_add_split_planes", y, _ptr(y), y.stride(0), _ptr(addend), addend.stride(0), y.shape[0], int(cols),
            float(scale), _ptr(scale_dev), _ptr(y_planes[0]), _ptr(y_planes[1]), y_planes[0].stride(0))


def pe_backward(x, g, g2, pe_w, bands, dx=None):
    """dx (+)= (d PE/d x)^T (g + g2); g / g2 [P, >= 3 + 6 bands] (row stride free), x [P,3]."""
    P = x.shape[0]
    acc = dx is not None
    if dx is None:
        dx = torch.empty((P, 3), dtype=torch.float32, device=x.device)
    w = (c_float * (2 * bands))(*[float(v) for v in pe_w[:2 * bands]])
    _launch("recmv_pe_backward", x, _ptr(x), _ptr(g), g.stride(0), _ptr(g2), g2.stride(0) if g2 is not None else 0, w,
            int(bands), _ptr(dx), 1 if acc else 0, P)
    return dx


def _pe_torch(x, pe_w, bands):
    outs, f = [x], 1.0
    for k in range(bands):
        outs += [pe_w[2 * k] * torch.sin(x * f), pe_w[2 * k + 1] * torch.cos(x * f)]
        f *= 2.0
    return torch.cat(outs, -1)


def _sdf_composite(x, Ws, bs, pe_w):
    """The same network as a torch graph (model/network.py:89-119) -- the twice-differentiable fallback of the
    training Function's backward when the caller asked for create_graph=True."""
    pe = _pe_torch(x, pe_w, 6)
    h = pe
    for l in range(9):
        if l == 4:
            h = torch.cat([h, pe], 1) * _INV_SQRT2
        h = torch.nn.functional.linear(h, Ws[l], bs[l])
        if l < 8:
            h = torch.nn.functional.softplus(h, beta=100)
    return h[:, :1], h[:, 1:]


class SdfMlpTrainFunction(torch.autograd.Function):
    """ImplicitNetwork.forward with gradients (model/network.py:89-119 inside train.py:317-330), all GEMMs on the tensor cores
    in the engine's fp32-grade arithmetic (fp16 hi/lo split, 3 MMAs per product, fp32 accumulation): TMA-fed GEMMs on
    operand planes (csrc/gemm3_tma.cu).

    forward : PE kernel + 9 layer launches  Y = softplus(X W^T + b)  whose outputs stay in HBM as the next layer's input
              AND as what the backward needs (16 KB per point -- what autograd keeps for the reference's graph); the skip
              concatenation is a column range of layer 4's input buffer, its 1/sqrt2 a scale of that layer's GEMM.
              (The inference engine keeps activations on-chip.)
    backward: first order (`loss.backward()`, parameter VJPs of propagateTmpPsGrad) -> 9 backward-data launches + nine
              weight-gradient launches on the same operand planes (recmv_mlp_wgrad_planes) + the PE Jacobian; weight-norm's
              (g, v) and anything upstream of x stay ordinary autograd.  Called with create_graph=True for the INPUT gradient
              (eikonal / normals, network.py:121-133, inside ops.input_grad_only()) the backward returns the reverse chain as
              a differentiable op on the same GEMMs (recmv_b200/second_order.py); a create_graph call that also wants
              parameter gradients with a graph re-runs the network as a torch graph (cuBLAS); `last_backward` says which ran."""
    last_backward = None

    @staticmethod
    def forward(ctx, x, pe_w, mode, packed, *Wb):
        Ws, bs = Wb[:9], Wb[9:]
        W_in = Ws
        if not (x.is_contiguous() and x.dtype == torch.float32 and x.dim() == 2):
            raise RuntimeError("SdfMlpTrainFunction expects a contiguous float32 [P,3] tensor (convert outside, in the graph)")
        P = x.shape[0]
        dev = x.device
        Ws = [w.detach().contiguous().float() for w in Ws]
        bs = [b.detach().contiguous().float() for b in bs]
        act = [torch.empty((P, 64), dtype=torch.float32, device=dev)] + \
              [torch.empty((P, 512), dtype=torch.float32, device=dev) for _ in range(8)]
        sdf = torch.empty((P, 1), dtype=torch.float32, device=dev)
        feat = torch.empty((P, 256), dtype=torch.float32, device=dev)
        # operands as fp16 hi / lo planes, TMA-fed GEMMs (csrc/gemm3_tma.cu): each layer writes its output in fp32
        # (kept for the backward) AND as the next layer's A planes
        xp = [_plane_pair(P, 64, dev)] + [_plane_pair(P, 512, dev) for _ in range(8)]
        pe_forward_planes(x, pe_w, 6, act[0], xp[0][0], xp[0][1])
        pe_forward_planes(x, pe_w, 6, act[4][:, 473:], xp[4][0][:, 473:], xp[4][1][:, 473:])
        for l in range(9):
            o, i = Ws[l].shape
            wp = weight_planes(W_in[l])
            if l < 8:
                mlp_layer_planes(xp[l], wp, P, o, i, 5, act[l + 1], bias=bs[l], scale=_INV_SQRT2 if l == 4 else 1.0,
                                 y_planes=xp[l + 1])
            else:
                mlp_layer_planes(xp[8], wp, P, 257, 512, 4, sdf, bias=bs[8], split=1, Y2=feat)
        ctx.pe_w, ctx.mode = [float(w) for w in pe_w], mode
        # the layer inputs' operand planes feed the weight gradient too (recmv_mlp_wgrad_planes)
        ctx.save_for_backward(x, *Wb, *act, *[t for pair in xp for t in pair])
        return sdf, feat

    @staticmethod
    def backward(ctx, g_sdf, g_feat):
        saved = ctx.saved_tensors
        x, Ws, bs, act = saved[0], saved[1:10], saved[10:19], saved[19:28]
        P = x.shape[0]
        need_x = ctx.needs_input_grad[0]
        need_w = any(ctx.needs_input_grad[4:])
        if torch.is_grad_enabled() and _inputs_only(need_w):
            # create_graph=True for the INPUT gradient only (ImplicitNetwork.gradient / deformed normals): the reverse
            # chain as a differentiable op whose own backward is tangent + backward GEMMs on the tensor cores (second_order.py)
            from . import second_order
            SdfMlpTrainFunction.last_backward = "fused-tc (create_graph, input gradient)"
            dx = second_order.sdf_input_grad(x, g_sdf, g_feat, ctx.pe_w, act, Ws, bs, saved[28:46]) if need_x else None
            return (dx, None, None, None, *([None] * 18))
        if torch.is_grad_enabled():
            # create_graph=True with parameter gradients in the graph: differentiate a torch graph of the same network
            SdfMlpTrainFunction.last_backward = "autograd-composite (create_graph)"
            g_sdf = g_sdf if g_sdf is not None else x.new_zeros((P, 1))     # the sdf output is always differentiated
            res = _composite_grads(lambda x, *Wb: _sdf_composite(x, Wb[:9], Wb[9:], ctx.pe_w), [x, *Ws, *bs],
                                   [g_sdf, g_feat])
            return (res[0], None, None, None, *res[1:])
        SdfMlpTrainFunction.last_backward = "fused-tc"
        dyn, _, GP, dpe0, dpe4 = sdf_reverse_chain(g_sdf, g_feat, act, Ws, need_x)
        dx = pe_backward(x, dpe0, dpe4, ctx.pe_w, 6) if need_x else None
        dW, db = [None] * 9, [None] * 9
        if need_w:
            # weight gradient straight from the planes both passes wrote (MN-major operands, no transposed copies)
            xpl = saved[28:46]
            for l in range(9):
                o, i = Ws[l].shape
                dW[l], db[l] = mlp_wgrad_planes(GP[l], (xpl[2 * l], xpl[2 * l + 1]), P, o, i,
                                                _INV_SQRT2 if l == 4 else 1.0, dyn, want_bias=True)
        return (dx, None, None, None, *dW, *db)


def sdf_reverse_chain(g_sdf, g_feat, act, Ws, with_layer0=True):
    """Backward-data chain of ImplicitNetwork on the operand-plane GEMMs, from the activations `act` its training forward
    saved: cotangents g_sdf [P,1] / g_feat [P,256] (either may be None) -> (dyn, G, GP, dpe0, dpe4).  G[l] [P, 512] (G[8]
    [P, 264]) is the fp32 cotangent at layer l's output and GP[l] its fp16 planes (carrying 64 * dyn); dpe4 [P, 40] is the
    cotangent of the PE copy in layer 4's skip input, dpe0 [P, 40] that of layer 0's input (None without with_layer0).
    The buffers are not zero-filled, and G[3][:, 473:] and column 39 of dpe0 / dpe4 are never written: layer 3 has 473
    outputs (the skip's cotangent goes to dpe4) and the PE 39 columns, and every result is taken from within those widths."""
    P, dev = act[0].shape[0], act[0].device
    G8 = torch.zeros((P, 264), dtype=torch.float32, device=dev)
    if g_sdf is not None:
        G8[:, 0:1] = g_sdf.detach()
    if g_feat is not None:
        G8[:, 1:257] = g_feat.detach()
    dyn = grad_dyn_scale(G8)
    G, GP = [None] * 9, [None] * 9
    G[8] = G8
    dpe4 = torch.empty((P, 40), dtype=torch.float32, device=dev)
    GP[8] = split_planes(G8, P, 257, 64.0, scale_dev=dyn, ldp=264)       # cotangent planes carry 64 * dyn
    for l in range(8, 0, -1):
        o, i = Ws[l].shape
        G[l - 1] = torch.empty((P, 512), dtype=torch.float32, device=dev)
        GP[l - 1] = _plane_pair(P, 512, dev)
        wtp = weight_planes(Ws[l], transpose=True)                                     # [in][out]: B of backward-data
        mlp_layer_planes(GP[l], wtp, P, i, o, 1, G[l - 1], saved_input=act[l], scale=_INV_SQRT2 if l == 4 else 1.0,
                         dyn=dyn, a_has_dyn=True, split=473 if l == 4 else 0, Y2=dpe4 if l == 4 else None,
                         y_planes=GP[l - 1], planes_with_dyn=True)
    dpe0 = None
    if with_layer0:
        o, i = Ws[0].shape
        dpe0 = torch.empty((P, 40), dtype=torch.float32, device=dev)
        mlp_layer_planes(GP[0], weight_planes(Ws[0], transpose=True), P, i, o, 0, dpe0, dyn=dyn, a_has_dyn=True)
    return dyn, G, GP, dpe0, dpe4


def _plain_mlp_forward(X0, Ws, bs):
    """ReLU MLP on the operand-plane layer GEMMs: returns (output [P, out_last], saved layer inputs [X0, X1, ...], their
    operand planes as a flat hi, lo list)."""
    P, dev = X0.shape[0], X0.device
    Ws = [w.detach().contiguous().float() for w in Ws]
    bs = [b.detach().contiguous().float() for b in bs]
    acts = [X0]
    n = len(Ws)
    xp = split_planes(X0, P, Ws[0].shape[1], 64.0, ldp=_pad8(X0.shape[1]))
    xplanes = []
    for l in range(n):
        o, i = Ws[l].shape
        last = l == n - 1
        Y = torch.empty((P, o if not last else ((o + 3) // 4) * 4), dtype=torch.float32, device=dev)
        yp = None if last else _plane_pair(P, _pad8(o), dev)
        mlp_layer_planes(xp, split_planes(Ws[l], o, i, 1024.0), P, o, i, 4 if last else 6, Y, bias=bs[l], y_planes=yp)
        xplanes += [xp[0], xp[1]]
        xp = yp
        acts.append(Y)
    return acts[-1][:, :Ws[-1].shape[0]], acts[:-1], xplanes


def plain_reverse_chain(g_out, Ws, acts, with_layer0=True):
    """Backward-data chain of a ReLU MLP on the operand-plane GEMMs, from the layer inputs `acts` its training forward
    saved: g_out [P, out_last] -> (dyn, GP, dX0).  GP[l] holds the planes of 64 * dyn * the cotangent at layer l's output
    (after the ReLU derivative), dX0 [P, in_0 rounded up to 4] that of the network input (None without with_layer0)."""
    P, dev = g_out.shape[0], g_out.device
    n = len(Ws)
    o_last = Ws[-1].shape[0]
    G = torch.zeros((P, _pad8(o_last)), dtype=torch.float32, device=dev)
    G[:, :o_last] = g_out
    dyn = grad_dyn_scale(G)
    GP = [None] * n
    GP[n - 1] = split_planes(G, P, o_last, 64.0, scale_dev=dyn, ldp=_pad8(o_last))
    for l in range(n - 1, 0, -1):
        o, i = Ws[l].shape
        G = torch.empty((P, i), dtype=torch.float32, device=dev)
        GP[l - 1] = _plane_pair(P, _pad8(i), dev)
        mlp_layer_planes(GP[l], split_planes(Ws[l].detach(), o, i, 1024.0, transpose=True), P, i, o, 2, G,
                         saved_input=acts[l], dyn=dyn, a_has_dyn=True, y_planes=GP[l - 1], planes_with_dyn=True)
    dX0 = None
    if with_layer0:
        o, i = Ws[0].shape
        dX0 = torch.empty((P, ((i + 3) // 4) * 4), dtype=torch.float32, device=dev)
        mlp_layer_planes(GP[0], split_planes(Ws[0].detach(), o, i, 1024.0, transpose=True), P, i, o, 0, dX0, dyn=dyn,
                         a_has_dyn=True)
    return dyn, GP, dX0


def _plain_mlp_backward(g_out, Ws, acts, need_w, need_x0, xplanes):
    """g_out [P, out_last] -> (dX0 [P, in_0 padded] or None, dW list, db list) for the ReLU MLP.  xplanes: the layer inputs'
    operand planes from the forward (flat hi, lo list), the weight gradient's second operand."""
    P = g_out.shape[0]
    n = len(Ws)
    dyn, GP, dX0 = plain_reverse_chain(g_out, Ws, acts, need_x0)
    dW, db = [None] * n, [None] * n
    if need_w:
        for l in range(n):
            o, i = Ws[l].shape
            dW[l], db[l] = mlp_wgrad_planes(GP[l], (xplanes[2 * l], xplanes[2 * l + 1]), P, o, i, 1.0, dyn, want_bias=True)
    return dX0, dW, db


def _plain_composite(X0, Ws, bs):
    h = X0
    for l in range(len(Ws)):
        h = torch.nn.functional.linear(h, Ws[l], bs[l])
        if l < len(Ws) - 1:
            h = torch.relu(h)
    return h


# One column range of a ReLU network's input row, in column order: "copy" (apply argument `arg`'s `cols` columns as they
# are), "pe" (its positional encoding, 3 + 6 bands columns) or "gather" (arg[apply argument `index`], `cols` columns).
RowSegment = collections.namedtuple("RowSegment", "kind arg cols bands index", defaults=(0, 0, None))


def _relu_mlp_train_function(name, layout, doc):
    """The training Function of a ReLU MLP whose input row is `layout` (RowSegments, zero-padded to a multiple of 4
    columns): apply(*row inputs, pe_w, *Ws, *bs).  Its backward takes SdfMlpTrainFunction's three branches;
    `last_backward` says which ran."""
    ends = list(itertools.accumulate(3 + 6 * s.bands if s.kind == "pe" else s.cols for s in layout))
    spans = list(zip(layout, [0] + ends, ends))                  # (segment, first column, end column)
    width = (ends[-1] + 3) // 4 * 4
    by_arg = sorted(spans, key=lambda sp: sp[0].arg)             # the order of the returned gradients
    n_in = 1 + max(max(s.arg, s.index or 0) for s in layout)     # row inputs; pe_w follows them, then the parameters

    def forward(ctx, *args):
        ins, pe_w, Wb = args[:n_in], args[n_in], args[n_in + 1:]
        n = len(Wb) // 2
        X0 = torch.zeros((ins[0].shape[0], width), dtype=torch.float32, device=ins[0].device)
        for s, a, b in spans:
            t = ins[s.arg].detach()
            if s.kind == "pe":
                pe_forward(t.contiguous(), pe_w, s.bands, X0[:, a:b])
            else:
                X0[:, a:b] = t if s.kind == "copy" else t[ins[s.index]]
        out, acts, xplanes = _plain_mlp_forward(X0, Wb[:n], Wb[n:])
        ctx.pe_w, ctx.n = [float(w) for w in pe_w], n
        ctx.save_for_backward(*ins, *Wb, *acts, *xplanes)
        return out.contiguous()

    def backward(ctx, g_out):
        n, saved, need = ctx.n, ctx.saved_tensors, ctx.needs_input_grad
        ins, Ws, bs = saved[:n_in], saved[n_in:n_in + n], saved[n_in + n:n_in + 2 * n]
        acts, xplanes = saved[n_in + 2 * n:n_in + 3 * n], saved[n_in + 3 * n:]
        wanted = [sp for sp in by_arg if need[sp[0].arg]]
        grads = [None] * n_in
        if torch.is_grad_enabled() and _inputs_only(any(need[n_in + 1:])):
            # create_graph=True for input gradients only (the translator's Jacobian in the deformation regulariser)
            from . import second_order
            fn.last_backward = "fused-tc (create_graph, input gradient)"
            dX0 = second_order.PlainMlpInputGradFunction.apply(g_out.contiguous().float(), n, *acts, *Ws)
            for s, a, b in wanted:
                t, d = ins[s.arg], dX0[:, a:b]
                grads[s.arg] = (d if s.kind == "copy" else
                                second_order.pe_vjp_torch(t, d, ctx.pe_w, s.bands) if s.kind == "pe" else
                                torch.zeros_like(t).index_add(0, ins[s.index], d))      # out of place: stays in the graph
            return (*grads, None, *([None] * (2 * n)))
        if torch.is_grad_enabled():
            fn.last_backward = "autograd-composite (create_graph)"

            def composite(*xs):
                X0 = torch.cat([xs[s.arg] if s.kind == "copy" else _pe_torch(xs[s.arg], ctx.pe_w, s.bands)
                                if s.kind == "pe" else xs[s.arg][xs[s.index]] for s in layout], 1)
                return _plain_composite(X0, xs[n_in:n_in + n], xs[n_in + n:])
            res = _composite_grads(composite, [*ins, *Ws, *bs], [g_out])
            return (*res[:n_in], None, *res[n_in:])
        fn.last_backward = "fused-tc"
        dX0, dW, db = _plain_mlp_backward(g_out.contiguous().float(), Ws, acts, any(need[n_in + 1:]), bool(wanted),
                                          xplanes)
        for s, a, b in wanted:
            t, d = ins[s.arg], dX0[:, a:b]
            grads[s.arg] = (d.contiguous() if s.kind == "copy" else
                            pe_backward(t.detach().contiguous(), d, None, ctx.pe_w, s.bands) if s.kind == "pe" else
                            torch.zeros_like(t).index_add_(0, ins[s.index], d))
        return (*grads, None, *dW, *db)

    fn = type(name, (torch.autograd.Function,), dict(__doc__=doc, row_width=width, last_backward=None,
                                                     forward=staticmethod(forward), backward=staticmethod(backward)))
    return fn


TranslatorTrainFunction = _relu_mlp_train_function("TranslatorTrainFunction", [
    RowSegment("pe", 0, bands=6),                       # PE6(ps)
    RowSegment("gather", 1, cols=128, index=2),         # conds[batch_inds]
], """MLPTranslator offset MLP with gradients (model/Deformer.py:171-206): apply(ps, conds, batch_inds, pe_w, *Ws, *bs),
    input row [PE6(p) 39 | cond[frame] 128] -> 512 x4 ReLU -> 3, forward / backward-data / weight gradient on the tensor
    cores (csrc/gemm3_tma.cu); returns the OFFSET (the caller adds p).""")

RenderNetTrainFunction = _relu_mlp_train_function("RenderNetTrainFunction", [
    RowSegment("copy", 0, cols=3),                      # points
    RowSegment("pe", 2, bands=4),                       # PE4(view_dirs)
    RowSegment("copy", 1, cols=3),                      # normals
    RowSegment("copy", 3, cols=256),                    # feats
], """RenderingNetwork_view_norm ('idr', model/RenderNet.py:59-96) with gradients: apply(points, normals, view_dirs,
    feats, pe_w, *Ws, *bs), input row [p 3 | PE4(v) 27 | n 3 | feat 256] -> 512 x4 ReLU -> 3 (pre-tanh; the caller
    applies tanh), all GEMMs on the tensor cores.""")


TRANSLATOR_LAYER_SHAPES = [(512, 167), (512, 512), (512, 512), (512, 512), (3, 512)]


def translator_pack_weights(Ws, bs):
    """MLPTranslator weights (lin0..lin4, no weight-norm) -> packed fp16 hi/lo panels for the tensor-core engine."""
    return _pack_weights("translator", "translator", TRANSLATOR_LAYER_SHAPES, Ws, bs)


def deformer_forward(ps, conds, packed, pe_w, batch_inds=None, points_per_frame=0, skin=None, mode=None,
                     want_offset=True, want_translated=True, want_jacobian=False):
    """MLPTranslator (+ LBS forward when skin = (A, trans, ws_cl, center, extend)) in one fused launch.
    Returns (translated [P,3] or None, offset [P,3] or None, posed [P,3] or None) -- plus the Jacobian [P,3,3]
    of the last stage w.r.t. ps (forward-mode launch) when want_jacobian."""
    mode = DEFAULT_MLP_MODE if mode is None else mode
    ps = ps.contiguous().float()
    conds = conds.contiguous().float()
    A = trans = ws_cl = vox = posed = None
    if skin is not None:
        A, trans, ws_cl, center, extend = skin
        A, trans = A.contiguous().float(), trans.contiguous().float()
    if batch_inds is not None:
        batch_inds = batch_inds.contiguous().long()
    d = _operands("deformer_forward", (ps, "ps", torch.float32, ("P", 3)), (conds, "conds", torch.float32, ("F", 128)),
                  (packed, "packed", torch.uint8, (_packed_bytes("translator"),)),
                  (batch_inds, "batch_inds", torch.int64, ("P",)), (A, "A", torch.float32, _BONES),
                  (trans, "trans", torch.float32, ("F", 3)), (ws_cl, "ws_cl", torch.float32, _VOXEL))
    P, dev = d["P"], ps.device
    tr = torch.empty((P, 3), dtype=torch.float32, device=dev) if want_translated else None
    off = torch.empty((P, 3), dtype=torch.float32, device=dev) if want_offset else None
    if skin is not None:
        vox = byref(_voxel(ws_cl, center, extend))
        posed = torch.empty((P, 3), dtype=torch.float32, device=dev)
    args = (_ptr(ps), _ptr(conds), _ptr(batch_inds), int(points_per_frame), d["F"], _ptr(packed),
            _pe_array(pe_w), _ptr(A), _ptr(trans), vox, _ptr(tr), _ptr(off), _ptr(posed))
    if want_jacobian:
        jac = torch.empty((P, 3, 3), dtype=torch.float32, device=dev)
        _launch("recmv_deformer_fwd_jac", ps, *args, _ptr(jac), P, mode)
        return tr, off, posed, jac
    _launch("recmv_deformer_fwd", ps, *args, P, mode)
    return tr, off, posed


RENDERNET_LAYER_SHAPES = [(512, 289), (512, 512), (512, 512), (512, 512), (3, 512)]


def rendernet_pack_weights(Ws, bs):
    """Effective colour-network weights (weight norm already applied) -> packed fp16 hi/lo panels."""
    return _pack_weights("rendernet", "colour-network", RENDERNET_LAYER_SHAPES, Ws, bs)


def rendernet_forward(points, normals, view_dirs, feats, packed, pe_w8, mode=None):
    """Fused colour MLP: [P,3] x3 + [P,256] -> rgb [P,3] (tanh)."""
    mode = DEFAULT_MLP_MODE if mode is None else mode
    args = [t.contiguous().float() for t in (points, normals, view_dirs, feats)]
    P = _operands("rendernet_forward", *[(t, n, torch.float32, ("P", 3)) for t, n in
                                         zip(args[:3], ("points", "normals", "view_dirs"))],
                  (args[3], "feature_vectors", torch.float32, ("P", 256)),
                  (packed, "packed", torch.uint8, (_packed_bytes("rendernet"),)))["P"]
    out = torch.empty((P, 3), dtype=torch.float32, device=args[0].device)
    pe = (c_float * 8)(*[float(w) for w in pe_w8])
    _launch("recmv_rendernet_fwd", out, *[_ptr(a) for a in args], _ptr(packed), pe, _ptr(out), P, mode)
    return out


def make_raymarch(cam_pos, t_near, t_far, samples):
    rm = RayMarch()
    rm.cam_pos = (c_float * 3)(*[float(c) for c in cam_pos])
    rm.t_near, rm.t_far, rm.samples_per_ray = float(t_near), float(t_far), int(samples)
    return rm


def render_sdf(ray_dirs, cam_pos, t_near, t_far, samples, A, trans, ws_cl, center, extend, packed,
               pe_w=None, mode=None, frame_of_ray=None, rays_per_frame=0, want_xc=False, want_hit=True,
               out_sdf=None):
    """The fused render path: rays -> samples -> inverse LBS -> PE -> SDF MLP -> sdf [R,S] (+ first hit)."""
    mode = DEFAULT_MLP_MODE if mode is None else mode
    ray_dirs = ray_dirs.contiguous().float()
    A = A.contiguous().float()
    trans = trans.contiguous().float()
    if frame_of_ray is not None:
        frame_of_ray = frame_of_ray.contiguous().to(torch.int32)
    d = _operands("render_sdf", (ray_dirs, "ray_dirs", torch.float32, ("R", 3)), (A, "A", torch.float32, _BONES),
                  (trans, "trans", torch.float32, ("F", 3)), (ws_cl, "ws_cl", torch.float32, _VOXEL),
                  (packed, "packed", torch.uint8, (_packed_bytes("sdf"),)),
                  (frame_of_ray, "frame_of_ray", torch.int32, ("R",)),
                  (out_sdf, "out_sdf", torch.float32, ("R", int(samples))))
    R, dev = d["R"], ray_dirs.device
    sdf = out_sdf if out_sdf is not None else torch.empty((R, samples), dtype=torch.float32, device=dev)
    xc = torch.empty((R, samples, 3), dtype=torch.float32, device=dev) if want_xc else None
    hit_idx = torch.empty((R,), dtype=torch.int32, device=dev) if want_hit else None
    hit_t = torch.empty((R,), dtype=torch.float32, device=dev) if want_hit else None
    rm = make_raymarch(cam_pos, t_near, t_far, samples)
    _launch("recmv_render_sdf", ray_dirs, _ptr(ray_dirs), byref(rm), _ptr(A), _ptr(trans), _ptr(frame_of_ray),
            int(rays_per_frame), d["F"], byref(_voxel(ws_cl, center, extend)), _ptr(packed), _pe_array(pe_w), _ptr(sdf), _ptr(xc),
            _ptr(hit_idx), _ptr(hit_t), R, mode)
    return sdf, xc, hit_idx, hit_t


def interp2x_boundary3d_forward(inp, balance_value, order=0):
    """[N,C,D,H,W] f32 -> (output [N,C,2D-1,2H-1,2W-1] f32, is_boundary bool): the reference's optional
    `interp2x_boundary3d.forward` (order 0: its rounding; order 1: the rounding of F.interpolate(trilinear,
    align_corners=True), the default path of Seg3dLossless)."""
    d = _operands("interp2x_boundary3d_forward", (inp, "input", torch.float32, ("N", "C", "D", "H", "W")))
    N, C, D, H, W = (d[k] for k in "NCDHW")
    out = torch.empty((N, C, 2 * D - 1, 2 * H - 1, 2 * W - 1), dtype=torch.float32, device=inp.device)
    flag = torch.empty(out.shape, dtype=torch.uint8, device=inp.device)
    _launch("recmv_interp2x_boundary3d_fwd", inp, _ptr(inp), _ptr(out), _ptr(flag), N * C, D, H, W, float(balance_value),
            int(order))
    return [out, flag.view(torch.bool)]


def interp2x_boundary3d_backward(grad_output):
    """grad_output [N,C,2D-1,2H-1,2W-1] f32 -> grad_input [N,C,D,H,W] (`interp2x_boundary3d.backward`)."""
    s = _operands("interp2x_boundary3d_backward", (grad_output, "grad_output", torch.float32, ("N", "C", "d", "h", "w")))
    N, C, D, H, W = s["N"], s["C"], (s["d"] + 1) // 2, (s["h"] + 1) // 2, (s["w"] + 1) // 2
    gi = torch.empty((N, C, D, H, W), dtype=torch.float32, device=grad_output.device)
    _launch("recmv_interp2x_boundary3d_bwd", gi, _ptr(grad_output), _ptr(gi), N * C, D, H, W)
    return gi


def c2f_todo_mask(is_boundary, done):
    """(3x3x3 dilation of is_boundary [D,H,W] bool) & ~done [D,H,W] bool -> bool [D,H,W]."""
    d = _operands("c2f_todo_mask", (is_boundary, "is_boundary", torch.bool, ("D", "H", "W")),
                  (done, "done", torch.bool, ("D", "H", "W")))
    D, H, W = d["D"], d["H"], d["W"]
    todo = torch.empty((D, H, W), dtype=torch.uint8, device=done.device)
    _launch("recmv_c2f_todo_mask", todo, _ptr(is_boundary.view(torch.uint8)), _ptr(done.view(torch.uint8)), _ptr(todo),
            D, H, W)
    return todo.view(torch.bool)


def fragment_decode(pix_to_face, bary, verts, faces, mask=None, camera=None):
    """Fragments -> (batch, row, col, seed points, face ids[, rays]) of the covered pixels in (n, row, col) order
    (recmv_fragment_decode).  camera = (fx, fy, px, py, R [3,3]) as host numbers / CPU tensor, or None.
    One host synchronisation: the read of the row count (the reference's `nonzero` has the same one)."""
    pix_to_face = pix_to_face.contiguous().long()
    bary = bary.contiguous().float()
    verts = verts.detach().contiguous().float()
    faces = faces.contiguous().long()
    if mask is not None:
        mask = mask.contiguous().float()
    d = _operands("fragment_decode", (pix_to_face, "pix_to_face", torch.int64, ("N", "H", "W", "K")),
                  (bary, "bary", torch.float32, ("N", "H", "W", "K", 3)), (verts, "verts", torch.float32, (..., 3)),
                  (faces, "faces", torch.int64, ("F", 3)), (mask, "mask", torch.float32, ("N", "H", "W")))
    N, H, W, K = d["N"], d["H"], d["W"], d["K"]
    dev, npix = pix_to_face.device, N * H * W
    scratch = torch.empty((_size("recmv_fragment_decode_scratch_bytes", npix),), dtype=torch.uint8, device=dev)
    ob, orow, ocol, ofi = (torch.empty((npix,), dtype=torch.int64, device=dev) for _ in range(4))
    opts = torch.empty((npix, 3), dtype=torch.float32, device=dev)
    orays = torch.empty((npix, 3), dtype=torch.float32, device=dev) if camera is not None else None
    cam = None
    if camera is not None:
        fx, fy, px, py, R = camera
        cam = (c_float * 13)(float(fx), float(fy), float(px), float(py), *[float(v) for v in torch.as_tensor(R).reshape(-1).tolist()])
    counters = torch.zeros((1,), dtype=torch.int32, device=dev)
    _launch("recmv_fragment_decode", bary, _ptr(pix_to_face), _ptr(bary), N, H, W, K, _ptr(verts), _ptr(faces),
            d["F"], _ptr(mask), cam, _ptr(scratch), _ptr(ob), _ptr(orow), _ptr(ocol), _ptr(opts), _ptr(ofi),
            _ptr(orays), _ptr(counters))
    n = int(counters.item())
    out = (ob[:n], orow[:n], ocol[:n], opts[:n], ofi[:n])
    return out + (orays[:n],) if camera is not None else out


def rasterize_meshes(verts, faces, cameras, H, W, z_clip=1e-6, area_eps=1e-8, want_dists=True, capacity=None,
                     host_camera=False):
    """Single-layer mesh rasterizer (recmv_rasterize_meshes).  verts [N,V,3] f32, faces [F,3] int64, cameras [N,16] f32
    {fx, fy, px, py, R row-major, T}, all CUDA and contiguous.  Returns (pix_to_face [N,H,W,1] int64, zbuf [N,H,W,1],
    bary [N,H,W,1,3], dists [N,H,W,1] or None, counts) with counts = {covered, skipped, pairs} as host ints.

    One host read per call: the counters after the launch.  The (tile, face) pair list lives in a grow-only per-device
    workspace; only when it overflowed is the call re-run, once, with a list of the reported size.  `capacity` sets the
    list size of the first attempt (the retained one when None).  host_camera=True adds cameras[0] as 16 host floats to
    the same read (what the fragment decode's view rays need)."""
    d = _operands("rasterize_meshes", (verts, "verts", torch.float32, ("N", "V", 3)),
                  (faces, "faces", torch.int64, ("F", 3)), (cameras, "cameras", torch.float32, ("N", 16)))
    N, V, F, dev = d["N"], d["V"], d["F"], verts.device
    H, W = int(H), int(W)
    ctr, host = _counters(dev, "raster_counters", 20)       # 4 counters + 16 camera floats
    kept = (dev.index, "raster_pairs")
    cap = int(capacity) if capacity is not None else max(_scratch_cache.get(kept, 0), 2 * N * F + 4096)
    p2f = torch.empty((N, H, W, 1), dtype=torch.int64, device=dev)
    zbuf = torch.empty((N, H, W, 1), dtype=torch.float32, device=dev)
    bary = torch.empty((N, H, W, 1, 3), dtype=torch.float32, device=dev)
    dists = torch.empty((N, H, W, 1), dtype=torch.float32, device=dev) if want_dists else None
    for _ in range(2):
        ws = _scratch(dev, "raster_ws", _size("recmv_raster_workspace_bytes", N, F, H, W, cap))
        _scratch_cache[kept] = max(_scratch_cache.get(kept, 0), cap)
        _launch("recmv_rasterize_meshes", verts, _ptr(verts), V, _ptr(faces), F, N, _ptr(cameras), H, W, float(z_clip),
                float(area_eps), _ptr(ws), cap, _ptr(p2f), _ptr(zbuf), _ptr(bary), _ptr(dists), _ptr(ctr))
        if host_camera and N > 0:
            ctr[4:].copy_(cameras[0].view(torch.int32))
        covered, skipped, pairs, overflow = (int(v) for v in _read_counters(ctr, host)[:4])
        if not overflow:
            break
        if pairs >= 0x7fffffff:
            check(_lib.RECMV_E_RANGE, "recmv_rasterize_meshes (more than 2^31 - 1 tile / face pairs)")
        cap = pairs   # grow once to the exact size, re-run (the workspace is kept for later calls)
    else:
        raise _lib.RecmvError("recmv_rasterize_meshes: pair list still too small after growing")
    counts = {"covered": covered, "skipped": skipped, "pairs": pairs}
    if host_camera:
        counts["camera"] = host[4:].view(torch.float32).clone()
    return p2f, zbuf, bary, dists, counts


def zbuf_probe(verts, faces, cameras, H, W, screen_pts, norm_size, fill, z_clip=1e-6, area_eps=1e-8, return_taps=False):
    """Sparse z-buffer probe (recmv_zbuf_probe, DESIGN section 1i): what grid_sample(align_corners=True) of the filled
    zbuf of rasterize_meshes(verts, faces, cameras, H, W, z_clip, area_eps) returns at the query points, without
    rasterizing the frame.  verts [N,V,3] f32, faces [F,3] int64, cameras [N,16] f32, screen_pts [N,Q,D] f32 (D >= 2;
    x, y read), norm_size [N,2] f32 (w, h) and fill [N] f32, all CUDA and contiguous.  Returns out [N,Q] f32, and with
    return_taps also (tap_zbuf [N,Q,4] f32, tap_face [N,Q,4] int64): the rasterizer's zbuf and packed face at the taps
    nw, ne, sw, se, (-1, -1) on background and outside the image.  Five launches, no host synchronisation."""
    d = _operands("zbuf_probe", (verts, "verts", torch.float32, ("N", "V", 3)), (faces, "faces", torch.int64, ("F", 3)),
                  (cameras, "cameras", torch.float32, ("N", 16)), (screen_pts, "screen_pts", torch.float32, ("N", "Q", "D")),
                  (norm_size, "norm_size", torch.float32, ("N", 2)), (fill, "fill", torch.float32, ("N",)))
    N, V, F, Q, D, dev = d["N"], d["V"], d["F"], d["Q"], d["D"], verts.device
    if D < 2:
        raise RuntimeError(f"zbuf_probe: screen_pts must have at least 2 coordinates, got {D}")
    H, W = int(H), int(W)
    out = torch.empty((N, Q), dtype=torch.float32, device=dev)
    tz = torch.empty((N, Q, 4), dtype=torch.float32, device=dev) if return_taps else None
    tf = torch.empty((N, Q, 4), dtype=torch.int64, device=dev) if return_taps else None
    ws = _scratch(dev, "zbuf_probe_ws", max(_size("recmv_zbuf_probe_workspace_bytes", N, Q, H, W), 1))
    _launch("recmv_zbuf_probe", verts, _ptr(verts), V, _ptr(faces), F, N, _ptr(cameras), H, W, float(z_clip),
            float(area_eps), _ptr(screen_pts), Q, D, _ptr(norm_size), _ptr(fill), _ptr(ws), _ptr(out), _ptr(tz),
            _ptr(tf))
    return (out, tz, tf) if return_taps else out


def rasterize_points(points, features, H, W, radius, K, split_size=None, want_fragments=False, capacity=None):
    """K-nearest point rasterizer + alpha compositor (recmv_rasterize_points).  points [N,P,3] f32 (NDC x, NDC y, view z),
    features [N,P] f32 or None (ones), CUDA and contiguous.  split_size=None renders one image; an int s renders two,
    points p < s into the first.  Returns (images [G,N,H,W], (idx [N,H,W,K] int64, zbuf, dists) or None, counts, ws)
    with counts = {covered, skipped, pairs} as host ints and ws the per-call workspace the backward reads.

    One host read per call: the counters after the launch.  Only when the (tile, point) pair list overflowed is the call
    re-run, once, with a list of the reported size.  `capacity` sets the list size of the first attempt (by default the
    largest pair count this device has seen, at least 8 pairs per point)."""
    d = _operands("rasterize_points", (points, "points", torch.float32, ("N", "P", 3)),
                  (features, "features", torch.float32, ("N", "P")))
    N, P = d["N"], d["P"]
    if not 1 <= int(K) <= 64:
        raise ValueError(f"rasterize_points: points_per_pixel must be in [1, 64], got {K}")
    G, split = (1, P) if split_size is None else (2, int(split_size))
    if not 0 <= split <= P:
        raise ValueError(f"rasterize_points: split_size must be in [0, {P}], got {split_size}")
    H, W, K = int(H), int(W), int(K)
    dev = points.device
    ctr, host = _counters(dev, "points_counters", 4)
    kept = (dev.index, "points_pairs")
    cap = int(capacity) if capacity is not None else max(_scratch_cache.get(kept, 0), 8 * N * P + 4096)
    images = torch.empty((G, N, H, W), dtype=torch.float32, device=dev)
    frags = tuple(torch.empty((N, H, W, K), dtype=dt, device=dev) for dt in (torch.int64, torch.float32, torch.float32)) \
        if want_fragments else None
    for _ in range(2):
        ws = torch.empty((_size("recmv_points_raster_workspace_bytes", N, P, H, W, cap),), dtype=torch.uint8, device=dev)
        _launch("recmv_rasterize_points", points, _ptr(points), _ptr(features), N, P, H, W, float(radius), K, split, G,
                _ptr(ws), cap, _ptr(images), *(_ptr(t) for t in (frags or (None,) * 3)), _ptr(ctr))
        covered, skipped, pairs, overflow = (int(v) for v in _read_counters(ctr, host))
        if overflow and pairs >= 0x7fffffff:
            # before the pair count is kept as the next call's list size: a saturated count would size every later
            # call's workspace at 8 GiB
            check(_lib.RECMV_E_RANGE, "recmv_rasterize_points (more than 2^31 - 1 tile / point pairs)")
        _scratch_cache[kept] = max(_scratch_cache.get(kept, 0), pairs)
        if not overflow:
            break
        cap = pairs   # grow once to the exact size and re-run
    else:
        raise _lib.RecmvError("recmv_rasterize_points: pair list still too small after growing")
    counts = {"covered": covered, "skipped": skipped, "pairs": pairs}
    return images, frags, counts, ws


def rasterize_points_backward(grad_images, ws, pairs, N, P, H, W, radius, K, split_size=None):
    """grad_points [N,P,3] of rasterize_points (recmv_rasterize_points_backward) from the image cotangents
    [G,N,H,W] and the forward's workspace `ws` and pair count; z components are 0."""
    G = 1 if split_size is None else 2
    split = P if split_size is None else int(split_size)
    dev = ws.device
    grad_images = grad_images.contiguous().float()
    _operands("rasterize_points_backward", (grad_images, "grad_images", torch.float32, (G, N, H, W)),
              (ws, "ws", torch.uint8, (None,)))
    grad = torch.empty((N, P, 3), dtype=torch.float32, device=dev)
    scratch = torch.empty((max(int(pairs), 1), 2), dtype=torch.float32, device=dev)
    _launch("recmv_rasterize_points_backward", grad_images, N, P, H, W, float(radius), int(K), split, G, _ptr(ws), int(pairs),
            _ptr(grad_images), _ptr(scratch), _ptr(grad))
    return grad


class RasterizePointsFunction(torch.autograd.Function):
    """images [G,N,H,W] = rasterize_points(points, ...)[0], differentiable in the points' NDC x and y.  The fragments
    (when asked) are returned after the images and carry no gradient; features must not require grad.  The forward's
    binned lists are kept for the backward (no re-binning)."""

    @staticmethod
    def forward(ctx, points, features, H, W, radius, K, split_size=None, want_fragments=False):
        if features is not None and features.requires_grad:
            raise RuntimeError("rasterize_points: features must not require grad (no gradient is computed for them)")
        images, frags, counts, ws = rasterize_points(points, features, H, W, radius, K, split_size, want_fragments)
        ctx.ws, ctx.pairs = ws, counts["pairs"]
        ctx.args = (int(points.shape[0]), int(points.shape[1]), int(H), int(W), float(radius), int(K), split_size)
        if frags is None:
            return images
        ctx.mark_non_differentiable(*frags)
        return (images,) + frags

    @staticmethod
    def backward(ctx, grad_images, *unused):
        g = rasterize_points_backward(grad_images, ctx.ws, ctx.pairs, *ctx.args)
        return g, None, None, None, None, None, None, None


SHADE_PARAMS = 28     # per-frame constants of recmv_shade_phong (include/recmv_b200.h)


def vertex_normals(verts, faces):
    """Area-weighted vertex normals (recmv_vertex_normals): verts [N,V,3] f32, faces [F,3] int64 shared by the N frames,
    CUDA and contiguous -> [N,V,3] f32, n / max(|n|, 1e-6).  Summed in (face, corner) order without float atomics, so
    bit-identical from run to run; no host synchronisation."""
    d = _operands("vertex_normals", (verts, "verts", torch.float32, ("N", "V", 3)), (faces, "faces", torch.int64, ("F", 3)))
    N, V, F, dev = d["N"], d["V"], d["F"], verts.device
    out = torch.empty((N, V, 3), dtype=torch.float32, device=dev)
    ws = _scratch(dev, "normals_ws", max(_size("recmv_vertex_normals_workspace_bytes", V, F, dev=dev), 1))
    _launch("recmv_vertex_normals", verts, _ptr(verts), N, V, _ptr(faces), F, _ptr(ws), _ptr(out))
    return out


def surface_sample(verts, faces, count, seed, offset=0):
    """Area-weighted surface samples (recmv_surface_sample, DESIGN section 1h): verts [M,V,3] f32, faces [F,3] int64
    shared by the M meshes, CUDA and contiguous -> [M,count,3] f32.  Sample s of mesh m is a pure function of (seed,
    offset, m, s) (Philox4x32-10 counter offset + m*count + s), so one call over M meshes equals M calls at offsets
    offset, offset + count, ...  Three launches, bit-identical from run to run, no host synchronisation."""
    d = _operands("surface_sample", (verts, "verts", torch.float32, ("M", "V", 3)), (faces, "faces", torch.int64, ("F", 3)))
    M, V, F, S, dev = d["M"], d["V"], d["F"], int(count), verts.device
    if S < 0:
        raise RuntimeError(f"surface_sample: count must be >= 0, got {S}")
    if F == 0 and M * S > 0:
        raise RuntimeError("surface_sample: faces is empty, there is no surface to sample")
    out = torch.empty((M, S, 3), dtype=torch.float32, device=dev)
    ws = _scratch(dev, "surface_sample_ws", max(_size("recmv_surface_sample_workspace_bytes", M, F), 1))
    _launch("recmv_surface_sample", verts, _ptr(verts), M, V, _ptr(faces), F, S, int(seed) % (1 << 64),
            int(offset) % (1 << 64), _ptr(ws), _ptr(out))
    return out


def train_rays_sample(batch, row, col, init_pts, masks, camera, target, seed, offset=0):
    """sample_train_ray's selection for G garments (recmv_train_rays_sample, DESIGN section 1j).  batch, row, col: G
    int64 [P_g] tensors, init_pts: G f32 [P_g,3], masks: G f32 [N,H,W], camera: f32 [>= 13] or [M,16] (row 0 used,
    raster.camera_rows' layout), all CUDA and on one device.  Rows with mask > 0 are candidates; a garment with more
    than `target` of them keeps candidate j iff its uniform (Philox4x32-10 counter offset + P_0 + ... + P_{g-1} + j)
    is below fp32(target / pnum).  Returns G tuples (batch, row, col, init points, view rays) of the kept rows in input
    order; the stream advances by P_0 + ... + P_{G-1}.  Five launches per 8 garments and one host synchronisation:
    the read of the G kept counts."""
    G = len(batch)
    if not (len(row) == len(col) == len(init_pts) == len(masks) == G):
        raise RuntimeError("train_rays_sample: batch, row, col, init_pts and masks must have one entry per garment")
    if G == 0:
        return []
    rows = [f"P{g}" for g in range(G)]      # garment g's row count
    d = _operands("train_rays_sample", *[(t, f"{name}[{g}]", torch.int64, (f"P{g}",)) for name, ts in
                                         (("batch", batch), ("row", row), ("col", col)) for g, t in enumerate(ts)],
                  *[(t, f"init_pts[{g}]", torch.float32, (f"P{g}", 3)) for g, t in enumerate(init_pts)],
                  (masks, "masks", torch.float32, ("N", "H", "W")), (camera, "camera", torch.float32, (...,)))
    if camera.numel() < 13:
        raise RuntimeError(f"train_rays_sample: camera must hold >= 13 values, got {camera.numel()}")
    dev = camera.device
    lists = [(d[r], tuple(torch.empty((d[r],), dtype=torch.int64, device=dev) for _ in range(3))
              + tuple(torch.empty((d[r], 3), dtype=torch.float32, device=dev) for _ in range(2))) for r in rows]
    lengths = (ctypes.c_int64 * G)(*[d[r] for r in rows])
    ws = _scratch(dev, "train_rays_ws", max(_size("recmv_train_rays_workspace_bytes", G, lengths), 1))
    ctr, host = _counters(dev, f"train_rays_counts_{G}", G)
    _launch("recmv_train_rays_sample", masks[0], G, _ptr_array(batch), _ptr_array(row), _ptr_array(col),
            _ptr_array(init_pts), lengths, _ptr_array(masks), d["N"], d["H"], d["W"], _ptr(camera), int(target),
            int(seed) % (1 << 64), int(offset) % (1 << 64), _ptr(ws), *[_ptr_array([o[k] for _, o in lists])
                                                                         for k in range(5)], _ptr(ctr))
    n = _read_counters(ctr, host).tolist()
    return [tuple(t[:n[g]] for t in o) for g, (_, o) in enumerate(lists)]


def loss_points_sample(init_pts, verts, check, batch, row, col, rays, S, seed, offset=0):
    """surface_render_loss's sample points and check compaction for G garments (recmv_loss_points_count / _emit, DESIGN
    section 1k).  Per garment: init_pts f32 [M,3], verts f32 [V,3] (V >= 1), check bool [M], batch / row / col int64
    [M], rays f32 [M,3], all CUDA and on one device; S = 4096 // G.  Returns G tuples (X_E [|B_E| + |B_E|//6, 3],
    X_D [2|B_D|, 3], points, rays, batch, row, col, index) with B_L = cat(init_pts, the vertices kept by lane L's draw
    at fp32(S / V)); the last six are the rows whose check is true, in order, and their input indices.  The stream
    advances by 5 (C_0 + ... + C_{G-1}), C_g = M_g + V_g.  Three launches per 8 garments and one host
    synchronisation: the read of the 3G counts that size the outputs."""
    G = len(init_pts)
    if not all(len(x) == G for x in (verts, check, batch, row, col, rays)):
        raise RuntimeError("loss_points_sample: every input list must have one entry per garment")
    if G == 0:
        return []
    # garment g has M{g} rows and V{g} vertices
    d = _operands("loss_points_sample", *[(t, f"init_pts[{g}]", torch.float32, (f"M{g}", 3)) for g, t in enumerate(init_pts)],
                  *[(t, f"verts[{g}]", torch.float32, (f"V{g}", 3)) for g, t in enumerate(verts)],
                  *[(t, f"check[{g}]", torch.bool, (f"M{g}",)) for g, t in enumerate(check)],
                  *[(t, f"{name}[{g}]", torch.int64, (f"M{g}",)) for name, ts in
                    (("batch", batch), ("row", row), ("col", col)) for g, t in enumerate(ts)],
                  *[(t, f"rays[{g}]", torch.float32, (f"M{g}", 3)) for g, t in enumerate(rays)])
    Ms, Vs = [d[f"M{g}"] for g in range(G)], [d[f"V{g}"] for g in range(G)]
    if 0 in Vs:
        raise RuntimeError("loss_points_sample: a garment has no vertices (the draw's rate S / V is undefined)")
    dev = verts[0].device
    Mc, Vc = (ctypes.c_int64 * G)(*Ms), (ctypes.c_int64 * G)(*Vs)
    seed, offset = int(seed) % (1 << 64), int(offset) % (1 << 64)
    ws = _scratch(dev, "loss_points_ws", max(_size("recmv_loss_points_workspace_bytes", G, Mc, Vc), 1))
    ctr, host = _counters(dev, f"loss_points_counts_{G}", 3 * G)
    _launch("recmv_loss_points_count", verts[0], G, Mc, Vc, _ptr_array(check), int(S), seed, offset, _ptr(ws), _ptr(ctr))
    n = _read_counters(ctr, host).tolist()
    outs = []
    for g in range(G):
        nE, nD, nc = Ms[g] + n[3 * g], Ms[g] + n[3 * g + 1], n[3 * g + 2]
        f32 = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)  # noqa: E731
        i64 = lambda k: torch.empty((k,), dtype=torch.int64, device=dev)  # noqa: E731
        outs.append((f32(nE + nE // 6, 3), f32(2 * nD, 3), f32(nc, 3), f32(nc, 3), i64(nc), i64(nc), i64(nc), i64(nc)))
    _launch("recmv_loss_points_emit", verts[0], G, _ptr_array(init_pts), Mc, _ptr_array(verts), Vc, _ptr_array(batch),
            _ptr_array(row), _ptr_array(col), _ptr_array(rays), (ctypes.c_int32 * (3 * G))(*n), int(S), seed, offset,
            _ptr(ws), *[_ptr_array([o[k] for o in outs]) for k in range(8)])
    return outs


def _frame_mean_ws(dev, M, N):
    return _scratch(dev, "frame_loss_ws", max(_size("recmv_frame_loss_workspace_bytes", int(M), int(N)), 1))


class ColorFrameMeanFunction(torch.autograd.Function):
    """The colour term of surface_render_loss (OptimGarmentNetwork.py:1186-1188) for one garment:
    apply(colors [M,3] f32, gtCs [N,H,W,3] f32, batch, row, col int64 [M], N) -> 0-d f32
    (1/N) sum_b mean_{i in b} sum_ch |gtCs[b, r, c, ch] - colors[i, ch]|, an empty frame giving 0 (recmv_color_frame_mean,
    DESIGN section 1k).  Deterministic; no host synchronisation.  Differentiable in colors (first order)."""

    @staticmethod
    def forward(ctx, colors, gtCs, batch, row, col, N):
        colors, gtCs = colors.contiguous(), gtCs.contiguous()
        N = int(N)
        d = _operands("color_frame_mean", (colors, "colors", torch.float32, ("M", 3)),
                      (gtCs, "gtCs", torch.float32, (N, "H", "W", 3)),      # the kernel bounds b by N
                      *[(t, name, torch.int64, ("M",)) for t, name in ((batch, "batch"), (row, "row"), (col, "col"))])
        M, H, W, dev = d["M"], d["H"], d["W"], colors.device
        loss = torch.empty((), dtype=torch.float32, device=dev)
        counts = torch.empty((N,), dtype=torch.int32, device=dev)
        _launch("recmv_color_frame_mean", colors, _ptr(gtCs), N, H, W, _ptr(batch), _ptr(row), _ptr(col), _ptr(colors),
                M, _ptr(_frame_mean_ws(dev, M, N)), _ptr(loss), _ptr(counts))
        ctx.save_for_backward(colors, gtCs, batch, row, col, counts)
        ctx.shape = (N, H, W)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        if not ctx.needs_input_grad[0]:
            return None, None, None, None, None, None
        colors, gtCs, batch, row, col, counts = ctx.saved_tensors
        N, H, W = ctx.shape
        g = g.contiguous().float()
        dcol = torch.empty_like(colors)
        _launch("recmv_color_frame_mean_backward", colors, _ptr(gtCs), N, H, W, _ptr(batch), _ptr(row), _ptr(col),
                _ptr(colors), int(colors.shape[0]), _ptr(counts), _ptr(g), _ptr(dcol))
        return dcol, None, None, None, None, None


class NormalFrameMeanFunction(torch.autograd.Function):
    """The normal term of surface_render_loss (OptimGarmentNetwork.py:1206-1215) for one garment:
    apply(gtn [M,3], J [M,3,3], nx [M,3], w [M] f32, batch int64 [M], N) -> 0-d f32: rows with nn = |gtn| > 1e-4 are
    valid, d = J^T (gtn / nn) - nx, and the value is (1/N) sum_b mean_{valid i in b} |d_i| w_i, an empty frame giving 0
    (recmv_normal_frame_mean, computed in double, DESIGN section 1k).  Deterministic; no host synchronisation.
    Differentiable (first order) in gtn, J and nx; w is a constant."""

    @staticmethod
    def forward(ctx, gtn, J, nx, w, batch, N):
        gtn, J, nx, w = (t.contiguous() for t in (gtn, J, nx, w))
        M = _operands("normal_frame_mean", (gtn, "gtn", torch.float32, ("M", 3)), (J, "J", torch.float32, ("M", 3, 3)),
                      (nx, "nx", torch.float32, ("M", 3)), (w, "w", torch.float32, ("M",)),
                      (batch, "batch", torch.int64, ("M",)))["M"]
        N, dev = int(N), gtn.device
        loss = torch.empty((), dtype=torch.float32, device=dev)
        counts = torch.empty((N,), dtype=torch.int32, device=dev)
        _launch("recmv_normal_frame_mean", gtn, _ptr(gtn), _ptr(J), _ptr(nx), _ptr(w), _ptr(batch), M, N,
                _ptr(_frame_mean_ws(dev, M, N)), _ptr(loss), _ptr(counts))
        ctx.save_for_backward(gtn, J, nx, w, batch, counts)
        ctx.N = N
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        need = ctx.needs_input_grad
        if not (need[0] or need[1] or need[2]):
            return None, None, None, None, None, None
        gtn, J, nx, w, batch, counts = ctx.saved_tensors
        g = g.contiguous().float()
        dgtn, dJ, dnx = torch.empty_like(gtn), torch.empty_like(J), torch.empty_like(nx)
        _launch("recmv_normal_frame_mean_backward", gtn, _ptr(gtn), _ptr(J), _ptr(nx), _ptr(w), _ptr(batch),
                int(gtn.shape[0]), ctx.N, _ptr(counts), _ptr(g), _ptr(dgtn), _ptr(dJ), _ptr(dnx))
        return (dgtn if need[0] else None), (dJ if need[1] else None), (dnx if need[2] else None), None, None, None


def mask_iou(masks, gt_masks, r):
    """Dilation and soft IoU of `mask_loss` for G garments (recmv_mask_iou, DESIGN section 1m): masks, gt_masks lists of
    G contiguous f32 [N,H,W] CUDA tensors of one shape, r in 1..32.  Returns (loss [G] f32 = mean_n (1 - I_gn / U_gn), loss_gn [G,N] f32,
    iu [G,N,2] f64 = (I, U), [G dilated masks f32 [N,H,W]]) with the dilation max_pool2d(gt, 2r+1, 1, r) bit for bit,
    I = sum m g', U = sum |m + g' - m g'|.  One pixel launch per 8 garments and one combine launch; deterministic;
    no host synchronisation.  Not differentiable: see MaskIouFunction."""
    G = len(masks)
    if G == 0 or len(gt_masks) != G:
        raise RuntimeError(f"mask_iou: expected the same number (>= 1) of masks and gt_masks, got {G} and "
                           f"{len(gt_masks)}")
    d = _operands("mask_iou", (masks, "masks", torch.float32, ("N", "H", "W")),
                  (gt_masks, "gt_masks", torch.float32, ("N", "H", "W")))
    N, H, W, dev = d["N"], d["H"], d["W"], masks[0].device
    with torch.cuda.device(dev):
        ws = _scratch(dev, "mask_iou_ws", _size("recmv_mask_iou_workspace_bytes", G, N, H, W, int(r)))
    mgt = [torch.empty_like(g) for g in gt_masks]
    iu = torch.empty((G, N, 2), dtype=torch.float64, device=dev)
    loss_gn = torch.empty((G, N), dtype=torch.float32, device=dev)
    loss = torch.empty((G,), dtype=torch.float32, device=dev)
    _launch("recmv_mask_iou", masks[0], G, _ptr_array(masks), _ptr_array(gt_masks), N, H, W, int(r), _ptr(ws),
            _ptr_array(mgt),
            _ptr(iu), _ptr(loss_gn), _ptr(loss))
    return loss, loss_gn, iu, mgt


def mask_iou_backward(masks, mgt, iu, grad_loss):
    """dL/dm of mask_iou for the upstream gradient grad_loss [G] f32 (recmv_mask_iou_backward): G f32 [N,H,W] tensors
    -(w_g / N) (g' U - I s (1 - g')) / U^2, s = sign(m + g' - m g') with sign(0) = 0, from the forward's dilated masks
    and iu.  One launch per 8 garments; no host synchronisation."""
    G = len(masks)
    if G == 0 or len(mgt) != G:
        raise RuntimeError(f"mask_iou_backward: expected the same number (>= 1) of masks and mgt, got {G} and "
                           f"{len(mgt)}")
    grad_loss = grad_loss.contiguous().float().reshape(G)
    d = _operands("mask_iou_backward", (masks, "masks", torch.float32, ("N", "H", "W")),
                  (mgt, "mgt", torch.float32, ("N", "H", "W")), (iu, "iu", torch.float64, (G, "N", 2)),
                  (grad_loss, "grad_loss", torch.float32, (G,)))
    dm = [torch.empty_like(m) for m in masks]
    _launch("recmv_mask_iou_backward", masks[0], G, _ptr_array(masks), _ptr_array(mgt), d["N"], d["H"], d["W"],
            _ptr(iu), _ptr(grad_loss), _ptr_array(dm))
    return dm


class MaskIouFunction(torch.autograd.Function):
    """The per-garment mask loss of `mask_loss` (OptimGarmentNetwork.py:621-629, 941-947) for G garments:
    apply(r, m_0 .. m_{G-1}, gt_0 .. gt_{G-1}) with silhouettes m_g and ground-truth masks gt_g f32 [N,H,W] on one CUDA
    device -> (loss [G] f32, mgt_0 .. mgt_{G-1}): loss_g = mean_n (1 - I / U) against mgt_g = max_pool2d(gt_g, 2r+1,
    1, r) (mask_iou).  Differentiable (first order) in the silhouettes; the ground-truth masks must not require grad
    and the dilated masks carry none.  Saves the dilated masks and (I, U) for the backward.  No host
    synchronisation."""

    @staticmethod
    def forward(ctx, r, *tensors):
        G = len(tensors) // 2
        if len(tensors) != 2 * G or G == 0:
            raise RuntimeError("MaskIouFunction: expected G silhouettes followed by G ground-truth masks")
        masks, gts = tensors[:G], tensors[G:]
        if any(g.requires_grad for g in gts):
            raise RuntimeError("MaskIouFunction: the ground-truth masks get no gradient; pass them detached")
        loss, _, iu, mgt = mask_iou(masks, gts, r)
        ctx.save_for_backward(iu, *masks, *mgt)
        ctx.G = G
        ctx.mark_non_differentiable(*mgt)
        return (loss, *mgt)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss, *grad_mgt):
        G = ctx.G
        saved = ctx.saved_tensors
        iu, masks, mgt = saved[0], saved[1:1 + G], saved[1 + G:]
        nothing = (None,) * (1 + 2 * G)
        if not any(ctx.needs_input_grad[1:1 + G]) or grad_loss is None:
            return nothing
        dm = mask_iou_backward(masks, mgt, iu, grad_loss)
        return (None, *[d if need else None for d, need in zip(dm, ctx.needs_input_grad[1:1 + G])]) + (None,) * G


def _curve_specs(center, dirs, init_scale, nx, scale, nx_scale):
    """Operand specs of the curve tensors: center, nx [C,1,3] or [C,3], dirs [C,S,3], init_scale, scale, nx_scale
    [C,S,1] or [C,S] (a unit axis is checked merged into its neighbour, as the kernels read it)."""
    rows = lambda t: t.view(t.shape[0], -1) if t.dim() == 3 else t  # noqa: E731
    return [(rows(center), "center", torch.float32, ("C", 3)), (dirs, "dirs", torch.float32, ("C", "S", 3)),
            (rows(init_scale), "init_scale", torch.float32, ("C", "S")), (rows(nx), "nx", torch.float32, ("C", 3)),
            (rows(scale), "scale", torch.float32, ("C", "S")), (rows(nx_scale), "nx_scale", torch.float32, ("C", "S"))]


def curve_fit(center, dirs, init_scale, nx, scale, nx_scale):
    """The feature curves and their regulariser (recmv_curve_fit, DESIGN section 1n): Intersect_Free_Curve's buffers
    and parameters (see _curve_specs) -> (v [C,S,3] = center + dirs init_scale relu(scale) + nx_scale nx,
    reg [C,2] = (sum of 1 - cosine of consecutive normalised differences, sum |mean v - center|) per curve).
    Formed in double, rounded once; one launch; deterministic."""
    d = _operands("curve_fit", *_curve_specs(center, dirs, init_scale, nx, scale, nx_scale))
    C, S = d["C"], d["S"]
    v = torch.empty((C, S, 3), dtype=torch.float32, device=dirs.device)
    reg = torch.empty((C, 2), dtype=torch.float32, device=dirs.device)
    _launch("recmv_curve_fit", dirs, C, S, *map(_ptr, (center, dirs, init_scale, nx, scale, nx_scale, v, reg)))
    return v, reg


def curve_fit_backward(center, dirs, init_scale, nx, scale, nx_scale, dv, dreg):
    """(dscale, dnx_scale) [C,S,1] of curve_fit for the upstream dv [C,S,3] (None = 0) and dreg [C,2], with torch's
    rules at relu(0), zero-length differences and the cosine eps clamp (recmv_curve_fit_backward)."""
    dv = dv.float().contiguous() if dv is not None else None
    dreg = dreg.float().contiguous()
    d = _operands("curve_fit_backward", *_curve_specs(center, dirs, init_scale, nx, scale, nx_scale),
                  (dv, "dv", torch.float32, ("C", "S", 3)), (dreg, "dreg", torch.float32, ("C", 2)))
    C, S, dev = d["C"], d["S"], dirs.device
    dscale = torch.empty((C, S, 1), dtype=torch.float32, device=dev)
    dnx = torch.empty((C, S, 1), dtype=torch.float32, device=dev)
    _launch("recmv_curve_fit_backward", dirs, C, S,
            *map(_ptr, (center, dirs, init_scale, nx, scale, nx_scale, dv, dreg, dscale, dnx)))
    return dscale, dnx


class CurveFitFunction(torch.autograd.Function):
    """Intersect_Free_Curve.forward plus its regulariser's terms for all C curves (engineer/utils/
    garment_structure.py:109-145): apply(center, dirs, init_scale, nx, scale, nx_scale) -> (v [C,S,3], reg [C,2])
    as curve_fit.  Differentiable (first order) in scale and nx_scale; the buffers get no gradient.  Deterministic
    backward; no host synchronisation."""

    @staticmethod
    def forward(ctx, center, dirs, init_scale, nx, scale, nx_scale):
        ins = [t.detach().contiguous() for t in (center, dirs, init_scale, nx, scale, nx_scale)]
        v, reg = curve_fit(*ins)
        ctx.save_for_backward(*ins)
        return v, reg

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dv, dreg):
        if not any(ctx.needs_input_grad[4:6]):
            return (None,) * 6
        ins = ctx.saved_tensors
        if dreg is None:
            dreg = torch.zeros((ins[1].shape[0], 2), dtype=torch.float32, device=ins[1].device)
        dscale, dnx = curve_fit_backward(*ins, dv, dreg)
        return (None,) * 4 + (dscale.view_as(ins[4]) if ctx.needs_input_grad[4] else None,
                              dnx.view_as(ins[5]) if ctx.needs_input_grad[5] else None)


def curve_project(X, cams, W, H, curves, thresholds, S, fl_masks, body):
    """Projection, visibility and compaction of the feature-curve rows (recmv_curve_project, DESIGN section 1n).
    X [R,3] f32 rows; cams [N,16] f32 {fx, fy, px, py, R, T} (raster.camera_rows); image W x H; curves a host list
    of K (base, stride, column) and thresholds K floats: curve k owns in frame n the S rows base + n stride + s, reads
    fl_masks [N,M] column `column` and tests body [R] < threshold.  Returns (screen [R,3] (x, y, ndc z), visible [R]
    bool, slot [R] int32, clouds [K N, S, 2], counts [K N] int64).  One launch; no host synchronisation."""
    d = _operands("curve_project", (X, "X", torch.float32, ("R", 3)), (cams, "cams", torch.float32, ("N", 16)),
                  (fl_masks, "fl_masks", torch.float32, ("N", "M")), (body, "body", torch.float32, ("R",)))
    R, N, dev = d["R"], d["N"], X.device
    K = len(curves)
    if K == 0 or len(thresholds) != K:
        raise RuntimeError(f"curve_project: expected K >= 1 curves and K thresholds, got {K} and {len(thresholds)}")
    table = (ctypes.c_int32 * (3 * K))(*[int(x) for c in curves for x in c])
    thr = (c_float * K)(*[float(t) for t in thresholds])
    with torch.cuda.device(dev):
        ws = _scratch(dev, "curve_project_ws", _size("recmv_curve_project_workspace_bytes", K, N, int(S)))
    screen = torch.empty((R, 3), dtype=torch.float32, device=dev)
    visible = torch.empty((R,), dtype=torch.bool, device=dev)
    slot = torch.empty((R,), dtype=torch.int32, device=dev)
    clouds = torch.empty((K * N, int(S), 2), dtype=torch.float32, device=dev)
    counts = torch.empty((K * N,), dtype=torch.int64, device=dev)
    _launch("recmv_curve_project", X, _ptr(X), R, _ptr(cams), N, int(W), int(H), table, thr, K, int(S),
            _ptr(fl_masks), d["M"], _ptr(body), _ptr(ws), _ptr(screen), _ptr(visible), _ptr(slot),
            _ptr(clouds), _ptr(counts))
    return screen, visible, slot, clouds, counts


def curve_project_backward(X, cams, K, S, slot, dclouds):
    """dX [R,3] of curve_project's clouds for dclouds [K N, S, 2]: J^T dclouds[slot] per row, 0 for rows without a
    slot (recmv_curve_project_backward); a gather, no atomics."""
    dclouds = dclouds.float().contiguous()
    d = _operands("curve_project_backward", (X, "X", torch.float32, ("R", 3)), (cams, "cams", torch.float32, ("N", 16)),
                  (slot, "slot", torch.int32, ("R",)), (dclouds, "dclouds", torch.float32, (lambda b: K * b["N"], S, 2)))
    R, N, dev = d["R"], d["N"], X.device
    dX = torch.empty((R, 3), dtype=torch.float32, device=dev)
    _launch("recmv_curve_project_backward", X, _ptr(X), R, _ptr(cams), N, int(K), int(S), _ptr(slot), _ptr(dclouds),
            _ptr(dX))
    return dX


class CurveProjectFunction(torch.autograd.Function):
    """The screen projection, z-buffer visibility and per-(curve, frame) compaction of `project_2d_loss` for every
    garment's curves: apply(X, cams, W, H, curves, thresholds, S, fl_masks, body) -> (screen, visible, counts,
    clouds) as curve_project.  Differentiable (first order) in X through the clouds only; the screen points, flags
    and counts carry no gradient and the cameras are constants.  Deterministic backward; no host synchronisation."""

    @staticmethod
    def forward(ctx, X, cams, W, H, curves, thresholds, S, fl_masks, body):
        X, cams = X.detach().contiguous(), cams.detach().contiguous()
        screen, visible, slot, clouds, counts = curve_project(X, cams, W, H, curves, thresholds, S,
                                                              fl_masks.detach().float().contiguous(),
                                                              body.detach().float().contiguous())
        ctx.save_for_backward(X, cams, slot)
        ctx.K, ctx.S = len(curves), int(S)
        ctx.mark_non_differentiable(screen, visible, counts)
        return screen, visible, counts, clouds

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_screen, d_visible, d_counts, dclouds):
        if not ctx.needs_input_grad[0] or dclouds is None:
            return (None,) * 9
        X, cams, slot = ctx.saved_tensors
        return (curve_project_backward(X, cams, ctx.K, ctx.S, slot, dclouds),) + (None,) * 8


def shade_phong(frags, verts, normals, colors, faces, params):
    """Hard Phong shading of K = 1 mesh fragments (recmv_shade_phong).  frags: an object with pix_to_face [N,H,W,1]
    int64 and bary_coords [N,H,W,1,3] f32 (raster.Fragments), or the tuple of rasterize_meshes; verts, normals [N,V,3]
    f32; colors [N,V,3] f32 or None (= 1); faces [F,3] int64; params [N,28] f32 per-frame constants (camera centre,
    light location and colours, material colours, shininess, background).  All CUDA and contiguous.
    Returns [N,H,W,4] f32 RGBA with alpha 1."""
    p2f, bary = (frags.pix_to_face, frags.bary_coords) if hasattr(frags, "pix_to_face") else (frags[0], frags[2])
    d = _operands("shade_phong", (p2f, "pix_to_face", torch.int64, ("N", "H", "W", 1)),
                  (bary, "bary_coords", torch.float32, ("N", "H", "W", 1, 3)), (verts, "verts", torch.float32, ("N", "V", 3)),
                  (normals, "normals", torch.float32, ("N", "V", 3)), (colors, "colors", torch.float32, ("N", "V", 3)),
                  (faces, "faces", torch.int64, ("F", 3)), (params, "params", torch.float32, ("N", SHADE_PARAMS)))
    N, H, W, V, dev = d["N"], d["H"], d["W"], d["V"], verts.device
    out = torch.empty((N, H, W, 4), dtype=torch.float32, device=dev)
    _launch("recmv_shade_phong", verts, _ptr(p2f), _ptr(bary), N, H, W, _ptr(verts), _ptr(normals), _ptr(colors), V,
            _ptr(faces), d["F"], _ptr(params), _ptr(out))
    return out


def knn_nearest(p1, p2, lengths1=None, lengths2=None):
    """Nearest neighbour of every p1 point in p2 (recmv_knn_nearest): p1 [N,P1,D], p2 [N,P2,D] f32, D = 2 or 3, lengths
    int64 [N] on the device or None, all CUDA and contiguous.  Returns (dists [N,P1] f32 squared distance, idx [N,P1]
    int64); padded rows (i >= lengths1, or lengths2 == 0) get 0 and -1.  Deterministic; no host synchronisation."""
    d = _operands("knn_nearest", (p1, "p1", torch.float32, ("N", "P1", "D")), (p2, "p2", torch.float32, ("N", "P2", "D")),
                  (lengths1, "lengths1", torch.int64, ("N",)), (lengths2, "lengths2", torch.int64, ("N",)))
    N, P1, P2, D, dev = d["N"], d["P1"], d["P2"], d["D"], p1.device
    if D not in (2, 3):
        raise RuntimeError(f"knn_nearest: the points must have 2 or 3 coordinates, got {D}")
    dists = torch.empty((N, P1), dtype=torch.float32, device=dev)
    idx = torch.empty((N, P1), dtype=torch.int64, device=dev)
    ws = _scratch(dev, "knn_ws", max(_size("recmv_knn_workspace_bytes", N, P1, P2, dev=dev), 1))
    _launch("recmv_knn_nearest", p1, _ptr(p1), _ptr(p2), _ptr(lengths1), _ptr(lengths2), N, P1, P2, D, _ptr(ws), _ptr(dists), _ptr(idx))
    return dists, idx


def knn_nearest_backward(p1, p2, idx, grad_dists, need_p2=True):
    """(grad_p1 [N,P1,D], grad_p2 [N,P2,D] or None) of knn_nearest's dists (recmv_knn_nearest_backward), from its idx
    and grad_dists [N,P1].  grad_p2 sums each candidate's queries in increasing index without float atomics."""
    grad_dists = grad_dists.contiguous().float()
    d = _operands("knn_nearest_backward", (p1, "p1", torch.float32, ("N", "P1", "D")),
                  (p2, "p2", torch.float32, ("N", "P2", "D")), (idx, "idx", torch.int64, ("N", "P1")),
                  (grad_dists, "grad_dists", torch.float32, ("N", "P1")))
    N, P1, P2, D, dev = d["N"], d["P1"], d["P2"], d["D"], p1.device
    g1 = torch.empty((N, P1, D), dtype=torch.float32, device=dev)
    g2 = torch.empty((N, P2, D), dtype=torch.float32, device=dev) if need_p2 else None
    ws = _scratch(dev, "knn_ws", max(_size("recmv_knn_workspace_bytes", N, P1, P2, dev=dev), 1))
    _launch("recmv_knn_nearest_backward", p1, _ptr(p1), _ptr(p2), _ptr(idx), _ptr(grad_dists), N, P1, P2, D, _ptr(ws),
            _ptr(g1), _ptr(g2))
    return g1, g2


class KnnNearestFunction(torch.autograd.Function):
    """(dists, idx) = knn_nearest(p1, p2, lengths1, lengths2), differentiable in p1 and p2 through dists; idx carries no
    gradient and the lengths none.  once_differentiable: no double backward."""

    @staticmethod
    def forward(ctx, p1, p2, lengths1=None, lengths2=None):
        dists, idx = knn_nearest(p1, p2, lengths1, lengths2)
        ctx.save_for_backward(p1, p2, idx)
        ctx.mark_non_differentiable(idx)
        return dists, idx

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_dists, unused_idx):
        p1, p2, idx = ctx.saved_tensors
        if grad_dists is None:
            return None, None, None, None
        g1, g2 = knn_nearest_backward(p1, p2, idx, grad_dists, need_p2=ctx.needs_input_grad[1])
        return (g1 if ctx.needs_input_grad[0] else None), g2, None, None


NRICP_STATS = 8   # stats record of recmv_nricp_step (include/recmv_b200.h)


def mesh_adjacency(faces, V):
    """Edges and boundary of a triangle mesh (recmv_mesh_adjacency): faces [F,3] int64, CUDA and contiguous, over V
    vertices -> (row_ptr [V+1] int32, col [6F] int32, deg [V] int32, boundary [V] bool).  row_ptr / col is the symmetric
    CSR of the unique sorted face sides, neighbours ascending; col[row_ptr[V]:] is -1.  A vertex is on the boundary when
    one of its sides occurs once among the 3F sides; faces with an index outside [0, V) are skipped.  No host
    synchronisation."""
    F = _operands("mesh_adjacency", (faces, "faces", torch.int64, ("F", 3)))["F"]
    dev, V = faces.device, int(V)
    row_ptr = torch.empty((V + 1,), dtype=torch.int32, device=dev)
    col = torch.empty((6 * F,), dtype=torch.int32, device=dev)
    deg = torch.empty((V,), dtype=torch.int32, device=dev)
    boundary = torch.empty((V,), dtype=torch.bool, device=dev)
    ws = _scratch(dev, "adjacency_ws", max(_size("recmv_mesh_adjacency_workspace_bytes", V, F, dev=dev), 1))
    _launch("recmv_mesh_adjacency", faces, _ptr(faces), F, V, _ptr(ws), _ptr(row_ptr), _ptr(col), _ptr(deg),
            _ptr(boundary))
    return row_ptr, col, deg, boundary


def nricp_warp(X, x, normals=None):
    """Local affine warp (recmv_nricp_warp): X [V,3,4] f32 = [A | b] per vertex, x [V,3] f32 -> v = A x + b [V,3]; with
    normals [V,3] also (n' = inv(A)^T n [V,3], ok [V] bool), n' = 0 where |det A| < 1e-4.  All CUDA and contiguous."""
    V = _operands("nricp_warp", (X, "X", torch.float32, ("V", 3, 4)), (x, "x", torch.float32, ("V", 3)),
                  (normals, "normals", torch.float32, ("V", 3)))["V"]
    dev = x.device
    v = torch.empty((V, 3), dtype=torch.float32, device=dev)
    n_out = ok = None
    if normals is not None:
        n_out = torch.empty((V, 3), dtype=torch.float32, device=dev)
        ok = torch.empty((V,), dtype=torch.bool, device=dev)
    _launch("recmv_nricp_warp", x, _ptr(X), _ptr(x), _ptr(normals), V, _ptr(v), _ptr(n_out), _ptr(ok))
    return v if normals is None else (v, n_out, ok)


def nricp_step(x, normals, target_v, target_n, corr_idx, adjacency, X, moments, step, stiffness_weight,
               laplacian_weight, gamma=1.0, threshold=0.5, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2,
               stats=None):
    """One NRICP inner iteration (recmv_nricp_step, DESIGN section 1f), in place on X [V,3,4] and moments = (exp_avg,
    exp_avg_sq, max_exp_avg_sq), each [V,3,4] f32: gate, loss, closed-form gradient and torch.optim.AdamW(amsgrad=True)
    with the given hyper-parameters at 1-based `step` (step 1 starts the moments from zero).  x, normals [V,3] f32 are
    the source points and normals; target_v, target_n [T,3] f32; corr_idx [V] int64 the target index of every vertex;
    adjacency = mesh_adjacency(faces, V).  Returns stats [8] f32 on the device (written into `stats` when given):
    {data sum, stiffness term, Laplacian term, loss, gate count, S, 0, 0} before the update.  Two launches, no host
    synchronisation, bit-identical from run to run."""
    row_ptr, col, _deg, boundary = adjacency
    d = _operands("nricp_step", (x, "x", torch.float32, ("V", 3)), (normals, "normals", torch.float32, ("V", 3)),
                  (target_v, "target_v", torch.float32, ("T", 3)), (target_n, "target_n", torch.float32, ("T", 3)),
                  (corr_idx, "corr_idx", torch.int64, ("V",)), (row_ptr, "row_ptr", torch.int32, (lambda b: b["V"] + 1,)),
                  (col, "col", torch.int32, (None,)), (boundary, "boundary", torch.bool, ("V",)),
                  *[(t, name, torch.float32, ("V", 3, 4)) for t, name in
                    ((X, "X"), (moments[0], "exp_avg"), (moments[1], "exp_avg_sq"), (moments[2], "max_exp_avg_sq"))],
                  (stats, "stats", torch.float32, (NRICP_STATS,)))
    V, T, dev = d["V"], d["T"], x.device
    if stats is None:
        stats = torch.empty((NRICP_STATS,), dtype=torch.float32, device=dev)
    prm = _lib.NricpParams(stiffness_weight, laplacian_weight, gamma, threshold, lr, betas[0], betas[1], eps,
                           weight_decay, int(step))
    ws = _scratch(dev, "nricp_ws", max(_size("recmv_nricp_workspace_bytes", V), 1))
    _launch("recmv_nricp_step", x, _ptr(x), _ptr(normals), _ptr(target_v), _ptr(target_n), T, _ptr(corr_idx),
            _ptr(row_ptr), _ptr(col), _ptr(boundary), V, byref(prm), _ptr(X), _ptr(moments[0]), _ptr(moments[1]),
            _ptr(moments[2]), _ptr(ws), _ptr(stats))
    return stats


LAP_EDIT_STATS = 8   # stats record of recmv_lap_edit_solve (include/recmv_b200.h)


def laplacian_edit(verts, adjacency, cidx, ctgt, constrain_weight=1.0, smooth=True, tol=1e-10, max_iter=50000,
                   stats=None, max_blocks=0):
    """Laplacian editing of a template (recmv_lap_edit_solve, DESIGN section 1g): y = argmin |L y - L x|^2 +
    c |P y - u|^2 with x = verts [V,3] f32, adjacency = mesh_adjacency(faces, V), constraints cidx [M] int64 (any order,
    duplicates allowed, indices outside [0, V) skipped and counted) with targets ctgt [M,3] f32 and c =
    constrain_weight, solved in float64 by Jacobi-preconditioned CG from y0 = x; smooth applies the reference's
    zero-diagonal Laplacian afterwards.  Returns (new_verts [V,3] f32, stats [8] f32 on the device, written into `stats`
    when given): {iterations of x, y, z; relative residuals of x, y, z; 1 converged / 0 max_iter reached / -1 non-finite;
    constraints skipped}.  Three launches, no host synchronisation.  max_blocks caps the solver's grid (0: every
    co-resident block); the result does not depend on it."""
    row_ptr, col, deg, _boundary = adjacency
    d = _operands("laplacian_edit", (verts, "verts", torch.float32, ("V", 3)),
                  (row_ptr, "row_ptr", torch.int32, (lambda b: b["V"] + 1,)), (col, "col", torch.int32, (None,)),
                  (deg, "deg", torch.int32, ("V",)), (cidx, "cidx", torch.int64, ("M",)),
                  (ctgt, "ctgt", torch.float32, ("M", 3)), (stats, "stats", torch.float32, (LAP_EDIT_STATS,)))
    V, M, dev = d["V"], d["M"], verts.device
    if stats is None:
        stats = torch.empty((LAP_EDIT_STATS,), dtype=torch.float32, device=dev)
    # the kernel finds each vertex's constraints by binary search: sort them by vertex, keeping duplicates in order
    cidx, order = torch.sort(cidx, stable=True)
    ctgt = ctgt.index_select(0, order)
    out = torch.empty((V, 3), dtype=torch.float32, device=dev)
    ws = _scratch(dev, "lap_edit_ws", _size("recmv_lap_edit_workspace_bytes", V, M))
    _launch("recmv_lap_edit_solve", verts, _ptr(verts), V, _ptr(row_ptr), _ptr(col), _ptr(deg), _ptr(cidx), _ptr(ctgt),
            M, float(constrain_weight), float(tol), int(max_iter), int(bool(smooth)), int(max_blocks), _ptr(ws),
            _ptr(out), _ptr(stats))
    return out, stats


class C2fLevel:
    """Device worklist of one pyramid level (recmv_c2f_refine / recmv_sdf_mlp_fwd_counted / recmv_c2f_scatter_list /
    recmv_c2f_mark_conflicts): one fused full-grid pass builds the level and its worklist, conflict rounds are driven by
    lists; no host round trip inside the level."""

    def __init__(self, coarse_dhw, final_whd, b_min, b_max, device, capacity):
        D, H, W = coarse_dhw
        self.coarse = (int(D), int(H), int(W))
        self.D, self.H, self.W = 2 * D - 1, 2 * H - 1, 2 * W - 1
        self.level = (ctypes.c_int * 3)(self.W, self.H, self.D)
        self.final = (ctypes.c_int * 3)(*[int(v) for v in final_whd])
        self.bmin = (c_float * 3)(*[float(v) for v in b_min])
        self.bmax = (c_float * 3)(*[float(v) for v in b_max])
        self.cap = int(capacity)
        self.dev = device
        self.idx = torch.empty((self.cap,), dtype=torch.int32, device=device)
        self.pts = torch.empty((self.cap, 3), dtype=torch.float32, device=device)
        self.vals = torch.empty((self.cap, 1), dtype=torch.float32, device=device)
        self.clist = [torch.empty((self.cap,), dtype=torch.int32, device=device) for _ in range(2)]
        # [0:2] worklist {count, overflow}; [2], [3] conflict counts of the two lists; [4] queried total
        self.ctr = torch.zeros((8,), dtype=torch.int32, device=device)
        self.claim = torch.zeros((self.D, self.H, self.W), dtype=torch.uint8, device=device)
        self.mixed = torch.empty((max(D - 1, 1) * max(H - 1, 1) * max(W - 1, 1),), dtype=torch.uint8, device=device)
        self.cur = 0     # which conflict list the last scatter filled

    def refine(self, occ_coarse, done_coarse, balance, order):
        occ_f = torch.empty((1, 1, self.D, self.H, self.W), dtype=torch.float32, device=self.dev)
        done_f = torch.empty((self.D, self.H, self.W), dtype=torch.uint8, device=self.dev)
        D, H, W = self.coarse
        _launch("recmv_c2f_refine", occ_f, _ptr(occ_coarse), _ptr(done_coarse), D, H, W, self.final, self.bmin, self.bmax,
                float(balance), int(order), _ptr(self.mixed), _ptr(occ_f), _ptr(done_f), _ptr(self.idx), _ptr(self.pts),
                _ptr(self.ctr), self.cap)
        return occ_f, done_f

    def evaluate(self, packed, pe_w, mode, occ, done_u8, calculated_u8, balance):
        """SDF on the current worklist, scatter, conflicts -> the other conflict list."""
        self.cur ^= 1
        cc = self.ctr[2 + self.cur:3 + self.cur]
        _launch("recmv_sdf_mlp_fwd_counted", occ, _ptr(self.pts), _ptr(packed), _pe_array(pe_w), _ptr(self.vals), None,
                self.cap, _ptr(self.ctr), mode)
        cc.zero_()
        _launch("recmv_c2f_scatter_list", occ, _ptr(self.idx), _ptr(self.vals), _ptr(self.ctr), self.cap, self.level,
                self.final, _ptr(occ), _ptr(done_u8), _ptr(calculated_u8), _ptr(self.claim), float(balance),
                _ptr(self.clist[self.cur]), _ptr(cc), _ptr(self.ctr[4:5]))

    def next_from_conflicts(self, calculated_u8):
        """Worklist of the next round from the conflict list the last evaluate() filled."""
        cc = self.ctr[2 + self.cur:3 + self.cur]
        self.ctr[0:1].zero_()
        _launch("recmv_c2f_mark_conflicts", calculated_u8, _ptr(self.clist[self.cur]), _ptr(cc), self.cap,
                _ptr(calculated_u8), self.level, self.final, self.bmin, self.bmax, _ptr(self.claim), _ptr(self.idx),
                _ptr(self.pts), _ptr(self.ctr), self.cap)

    def read(self):
        """(queried so far, conflicts of the last round, overflow) -- the level's host synchronisation."""
        return self.counts(self.ctr.tolist())

    def counts(self, h):
        """(queried, conflicts, overflow) from a host copy h of the counters."""
        return h[4], h[2 + self.cur], h[1]


def read_c2f_levels(levels):
    """C2fLevel.read of every level in one host synchronisation: the counters of several levels are gathered into one
    tensor and copied back together."""
    if len(levels) == 1:
        return [levels[0].read()]
    h = torch.stack([lvl.ctr for lvl in levels]).tolist()
    return [lvl.counts(r) for lvl, r in zip(levels, h)]


def surface_solve(cam_pos, rays, seeds, batch_inds, sdf_packed, sdf_pe_w, tr_packed, tr_pe_w, conds, skin, dthreshold,
                  athreshold, w1, w2, times, mode=None):
    """Device-resident surface solve (recmv_surface_solve).  skin = (A, trans, ws_cl, center, extend).
    Returns (points [P,3], ok [P] bool); `seeds` is not modified."""
    mode = DEFAULT_MLP_MODE if mode is None else mode
    ps = seeds.detach().contiguous().float().clone()
    rays = rays.contiguous().float()
    A, trans, ws_cl, center, extend = skin
    A, trans, conds = A.contiguous().float(), trans.contiguous().float(), conds.contiguous().float()
    bi = batch_inds.contiguous().long() if batch_inds is not None else None
    d = _operands("surface_solve", (rays, "rays", torch.float32, ("P", 3)), (ps, "seeds", torch.float32, ("P", 3)),
                  (bi, "batch_inds", torch.int64, ("P",)),
                  (sdf_packed, "sdf_packed", torch.uint8, (_packed_bytes("sdf"),)),
                  (tr_packed, "tr_packed", torch.uint8, (_packed_bytes("translator"),)),
                  (conds, "conds", torch.float32, ("F", 128)), (A, "A", torch.float32, _BONES),
                  (trans, "trans", torch.float32, ("F", 3)), (ws_cl, "ws_cl", torch.float32, _VOXEL))
    P, dev = d["P"], ps.device
    wsz = _size("recmv_surface_solve_workspace", P)
    work = torch.empty((max(wsz, 1),), dtype=torch.uint8, device=dev)
    ok = torch.empty((P,), dtype=torch.uint8, device=dev)
    cam = (c_float * 3)(*[float(v) for v in cam_pos.view(-1).tolist()])
    _launch("recmv_surface_solve", ps, cam, _ptr(rays), _ptr(ps), _ptr(bi), _ptr(sdf_packed), _pe_array(sdf_pe_w),
            _ptr(tr_packed), _pe_array(tr_pe_w), _ptr(conds), d["F"], _ptr(A), _ptr(trans),
            byref(_voxel(ws_cl, center, extend)), float(dthreshold), float(athreshold), float(w1), float(w2), int(times),
            mode, _ptr(work), wsz, _ptr(ok), P)
    return ps, ok.view(torch.bool)


def surface_grad_coeffs(grad_l_p, grad_f_p, jac, rays, d_minus_c=None):
    """Per-ray algebra of propagateTmpPsGrad (OptimNetwork.py:788-851) in one launch.
    Returns (sdf_coef [n], def_vec [n,3], ray_grad [n,3] or None, ok [n] bool)."""
    args = [t.contiguous().float() for t in (grad_l_p, grad_f_p, jac, rays)]
    dc = d_minus_c.contiguous().float() if d_minus_c is not None else None
    n = _operands("surface_grad_coeffs", *[(t, name, torch.float32, ("n", 3, 3) if name == "jac" else ("n", 3))
                                           for t, name in zip(args + [dc], ("grad_l_p", "grad_f_p", "jac", "rays",
                                                                             "d_minus_c"))])["n"]
    dev = args[0].device
    coef = torch.empty((n,), dtype=torch.float32, device=dev)
    vec = torch.empty((n, 3), dtype=torch.float32, device=dev)
    rg = torch.empty((n, 3), dtype=torch.float32, device=dev) if dc is not None else None
    ok = torch.empty((n,), dtype=torch.uint8, device=dev)
    _launch("recmv_surface_grad_coeffs", coef, *[_ptr(a) for a in args], _ptr(dc), _ptr(coef), _ptr(vec), _ptr(rg), _ptr(ok),
            n)
    return coef, vec, rg, ok.view(torch.bool)


def implicit_surface_grad(grad_l_p, grad_f_p, jac, rays, d, offsets, cam_pos=None, want_ray_grad=False, _max_ctas=None):
    """The per-row algebra of propagateTmpPsGrad (OptimGarmentNetwork.py:2213-2311) for every garment of a call, and
    its per-garment reductions (recmv_implicit_grad, DESIGN section 1l).  grad_l_p, grad_f_p, rays, d f32 [n,3], jac
    f32 [n,3,3], all CUDA and on one device; offsets: G + 1 host ints, garment g's rows at [offsets[g], offsets[g+1]);
    cam_pos: the camera centre, f32 [3] on the device, or None.  Returns (sdf_coef [n], def_vec [n,3], ray_grad [n,3]
    or None, ok [n] bool, ok_count [G] int32, cam_grad [G,3] or None): ray_grad = r[1:4] [d - c]x when want_ray_grad
    (needs d and cam_pos), cam_grad = -sum of each garment's def_vec rows when cam_pos is given.  Deterministic; no
    host synchronisation (a CUDA `offsets` tensor raises, as reading it would be one)."""
    if torch.is_tensor(offsets):
        if offsets.is_cuda:
            raise RuntimeError("implicit_surface_grad: offsets must be host integers")
        offsets = offsets.tolist()
    offs = [int(o) for o in offsets]
    G = len(offs) - 1
    if G < 0:
        raise RuntimeError("implicit_surface_grad: offsets needs G + 1 >= 1 entries")
    n = _operands("implicit_surface_grad", (grad_l_p, "grad_l_p", torch.float32, ("n", 3)),
                  (grad_f_p, "grad_f_p", torch.float32, ("n", 3)), (jac, "jac", torch.float32, ("n", 3, 3)),
                  (rays, "rays", torch.float32, ("n", 3)), (d, "d", torch.float32, ("n", 3)),
                  (cam_pos, "cam_pos", torch.float32, (3,)))["n"]
    dev = grad_l_p.device
    if offs[0] != 0 or offs[-1] != n or any(b < a for a, b in zip(offs, offs[1:])):
        raise RuntimeError(f"implicit_surface_grad: offsets must run from 0 to n = {n} without decreasing, got {offs}")
    if want_ray_grad and (d is None or cam_pos is None):
        raise RuntimeError("implicit_surface_grad: the ray gradient needs d and cam_pos")
    f32 = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)  # noqa: E731
    coef, vec, ok = f32(n), f32(n, 3), torch.empty((n,), dtype=torch.uint8, device=dev)
    rg = f32(n, 3) if want_ray_grad else None
    cnt = torch.empty((G,), dtype=torch.int32, device=dev)
    camg = f32(G, 3) if cam_pos is not None else None
    ws = _scratch(dev, "implicit_grad_ws", _size("recmv_implicit_grad_workspace_bytes", n, G))
    args = [_ptr(t) for t in (grad_l_p, grad_f_p, jac, rays, d, cam_pos)]
    args += [(ctypes.c_int64 * (G + 1))(*offs), G] + [_ptr(t) for t in (coef, vec, rg, ok, cnt, camg, ws)] + [n]
    if _max_ctas is None:
        _launch("recmv_implicit_grad", coef, *args)
    else:   # the same kernels on a capped grid (include/recmv_b200_diag.h): the results must not change
        _launch("recmv_implicit_grad_grid", coef, *args, int(_max_ctas))
    return coef, vec, rg, ok.view(torch.bool), cnt, camg


class Svd3x3Function(torch.autograd.Function):
    """(U, S, V) = svd(J), J [N,3,3] float32 CUDA, J = U diag(S) V^T with S descending -- torch.svd's contract, computed
    per matrix in registers (csrc/svd3.cu) instead of the reference's round trip through the host
    (`torch.svd(Jacobs.cpu())`, engineer/networks/OptimGarmentNetwork.py:1148).  Differentiable through S (dJ = U diag(dS)
    V^T, one launch); a cotangent on U or V raises (the reference's loss reads the singular values only)."""

    @staticmethod
    def forward(ctx, J):
        if J.dtype != torch.float32 or J.dim() != 3 or tuple(J.shape[1:]) != (3, 3):
            raise TypeError("svd3x3 expects a float32 [N,3,3] tensor")
        N = _operands("svd3x3", (J, "J", torch.float32, ("N", 3, 3)))["N"]
        U = torch.empty((N, 3, 3), dtype=torch.float32, device=J.device)
        V = torch.empty((N, 3, 3), dtype=torch.float32, device=J.device)
        S = torch.empty((N, 3), dtype=torch.float32, device=J.device)
        _launch("recmv_svd3x3", J, _ptr(J), N, _ptr(U), _ptr(S), _ptr(V))
        ctx.save_for_backward(U, V)
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(U, V)
        return U, S, V

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gU, gS, gV):
        if gU is not None or gV is not None:
            raise NotImplementedError("svd3x3 is differentiable through the singular values only")
        if gS is None:
            return None
        U, V = ctx.saved_tensors
        gS = gS.contiguous().float()
        dJ = torch.empty_like(U)
        _launch("recmv_svd3x3_backward_s", U, _ptr(U), _ptr(V), _ptr(gS), U.shape[0], _ptr(dJ))
        return dJ


def svd3x3(J):
    """torch.svd for a batch of 3x3 matrices on the device: returns (U, S, V)."""
    return Svd3x3Function.apply(J.contiguous())


def check_async_errors(clear=False):
    """Raise if a tensor-core launch on the current device aborted on a bounded wait (non-blocking check)."""
    info = (ctypes.c_int * 3)()
    st = _lib.load().recmv_check_async_errors(info, 1 if clear else 0)
    if st != 0:
        if info[0] == 2:
            raise _lib.RecmvError(f"tensor-core operand range exceeded (|activation| >= 1023.5 or |weight| >= 63.97 does not "
                                  f"fit the scaled fp16 operands; results were saturated): site tag={info[1]} block={info[2]}")
        raise _lib.RecmvError(f"tensor-core kernel aborted: code={info[0]} barrier tag={info[1]} block={info[2]}")


def launch_count():
    return int(_lib.load().recmv_launch_count())
