"""The drop-in native ops outside the MLP engines, at production sizes and at their edges:

    grid sampler    csrc/gridsample3d.cu forward / backward / double backward against float64 of
                    oracle_torch.grid_sample3d_{fwd,bwd,bwd2}: f32 and f64, NCDHW and NDHWC (the float4 forward and its
                    scalar fallback), N > 1, size-1 axes, P = 0 / 1 / 255 and one or three grid-stride waves + 77,
                    clipped, lattice, +-inf and NaN coordinates, nullable outputs, output bounds through the C ABI and
                    LBSkinner's composite path (FrozenVoxelSampleFunction under create_graph)
    voxel relayout  ops.voxel_to_channels_last, bit-equal to permute().contiguous()
    marching cubes  csrc/mc.cu bit-exact against oracle/mc_oracle.c: smooth grids at 129^3 and 257^3 (mc_scan_kernel with
                    3 and 17 segment sums per thread), a dense random-sign grid, a quantised grid with values on the iso
                    value
    fragment decode csrc/fragments.cu against the CPU path of FindSurfacePs: one chunk of frag_scan_kernel (1024 block
                    counts = 262 144 pixels), one block into the second chunk, six chunks
    argument checks of ops.py: RuntimeError before any launch

A grid-stride wave of the sampler is SMs x 8 CTAs x 256 threads (stride_grid(N P, 256, 8)); it is derived from the SM
count of the device."""
import numpy as np
import pytest
import torch

from oracle import mc_oracle
from oracle import oracle_torch as ot
from recmv_b200 import _lib, ops, synth
from recmv_b200.utils import FindSurfacePs, FindSurfacePsRays

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NCDHW, NDHWC = _lib.LAYOUT_NCDHW, _lib.LAYOUT_NDHWC
R_TAIL = 77                      # the ragged tail of the multi-wave sizes
GUARD = 256                      # guard elements before and after every output of the bounds test
NAN32 = 0x7FBADBAD               # fp32 NaN bit pattern no kernel writes
NAN64 = 0x7FF8BADBADBADBAD       # fp64 NaN bit pattern no kernel writes
MARGIN = 1e-4                    # random points stay this many cells away from every lattice plane and the border

# Bounds against float64 of the same inputs, max |a - b| / max |b| per tensor.  Float64 kernels: 1e-12.  Float32
# kernels, measured on an H100 80GB HBM3 (700 W power limit), maximum over every case of this file (the inputs are
# seeded):
#   forward out 4.3e-6; backward grad_input 2.2e-6, grad_grid 2.3e-6; double backward g_input 1.3e-6, g_grid 2.0e-6,
#   gg_out 2.1e-6
# (float64 kernels: at most 2.3e-15).  The forward is the loosest because the fp32 unnormalised coordinate itself is off
# by up to half an ulp of the voxel size (4e-6 cells at 65) and the sample moves with it.  Each bound is about 3x its
# maximum.
BOUND = {
    torch.float64: dict(out=1e-12, grad_input=1e-12, grad_grid=1e-12, g_input=1e-12, g_grid=1e-12, gg_out=1e-12),
    torch.float32: dict(out=1.3e-5, grad_input=7e-6, grad_grid=7e-6, g_input=4e-6, g_grid=6e-6, gg_out=6.5e-6),
}
_seen = {}                       # largest error per (dtype, output) over the run, for re-measuring the bounds


@pytest.fixture(autouse=True)
def _no_async_error():
    yield
    torch.cuda.synchronize()
    ops.check_async_errors()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _wave():
    return _sms() * 8 * 256


def merr(a, b):
    a = torch.as_tensor(a).detach().double()
    b = torch.as_tensor(b).detach().double().to(a.device)
    if a.numel() == 0 and b.numel() == 0:
        return 0.0
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


def _close(dtype, name, a, b):
    assert a.shape == b.shape, (name, a.shape, b.shape)
    e = merr(a, b)
    key = (str(dtype), name)
    _seen[key] = max(_seen.get(key, 0.0), e)
    assert e <= BOUND[dtype][name], f"{name} ({dtype}): {e:.3e} > {BOUND[dtype][name]:.1e}"


# ------------------------------------------------------------------------------------------------ grid sampler
def _points(shape, dhw, gen, span=1.3):
    """float64 points uniform in [-span, span]^3, each unnormalised coordinate moved at least MARGIN cells away from
    the nearest integer (lattice planes, border): there the trilinear gradient jumps, and fp32 and fp64 may round to
    different cells."""
    g = (torch.rand(tuple(shape) + (3,), generator=gen, dtype=torch.float64) * 2 - 1) * span
    D, H, W = dhw
    for a, S in enumerate((W, H, D)):
        x = ((g[..., a] + 1) * S - 1) / 2
        r = torch.round(x)
        d = x - r
        x = torch.where(d.abs() < MARGIN, r + torch.where(d < 0, -2 * MARGIN, 2 * MARGIN), x)
        g[..., a] = (2 * x + 1) / S - 1
    return g


def _tensors(N, C, dhw, ohw, dtype, seed, grid=None):
    """Inputs in `dtype` and the same values in float64 for the oracle, both on the device (the oracle is plain torch
    and runs there too).  A different voxel per batch entry."""
    gen = synth.generator(seed)
    inp = torch.randn((N, C) + tuple(dhw), generator=gen, dtype=torch.float64)
    if grid is None:
        grid = _points((N,) + tuple(ohw), dhw, gen)
    go = torch.randn((N, C) + tuple(ohw), generator=gen, dtype=torch.float64)
    ggi = torch.randn(inp.shape, generator=gen, dtype=torch.float64)
    ggg = torch.randn(grid.shape, generator=gen, dtype=torch.float64)
    dev = [t.to(dtype).to(DEV) for t in (inp, grid, go, ggi, ggg)]
    ref = [t.double() for t in dev]
    return dev, ref


def _oracle(inp, grid, go, ggi, ggg):
    """ot.grid_sample3d_fwd, then what ot.grid_sample3d_bwd and ot.grid_sample3d_bwd2 compute, on one autograd graph."""
    i, g, o = (t.detach().requires_grad_(True) for t in (inp, grid, go))
    out = ot.grid_sample3d_fwd(i, g)
    gi, gg = torch.autograd.grad(out, (i, g), o, create_graph=True)
    d = torch.autograd.grad((gi, gg), (i, g, o), (ggi, ggg), allow_unused=True)
    d0, d1, d2 = (torch.zeros_like(t) if x is None else x for x, t in zip(d, (inp, grid, go)))
    return dict(out=out.detach(), grad_input=gi.detach(), grad_grid=gg.detach(), g_input=d0, g_grid=d1, gg_out=d2)


def _to_layout(t, layout):
    return t if layout == NCDHW else t.permute(0, 2, 3, 4, 1).contiguous()


def _from_layout(t, layout):
    return t if layout == NCDHW else t.permute(0, 4, 1, 2, 3)


def _run(inp, grid, go, ggi, ggg, layout, need_grad_input=True):
    x = _to_layout(inp, layout)
    gx = None if ggi is None else _to_layout(ggi, layout)
    out = ops.grid_sample3d_forward(x, grid, layout)
    gi, gg = ops.grid_sample3d_backward(x, grid, go, layout, need_grad_input=need_grad_input)
    d0, d1, d2 = ops.grid_sample3d_dbackward(gx, ggg, x, grid, go, layout, need_grad_input=need_grad_input)
    res = dict(out=out, grad_grid=gg, g_grid=d1, gg_out=d2)
    if need_grad_input:
        res.update(grad_input=_from_layout(gi, layout), g_input=_from_layout(d0, layout))
    return res


def _check_all(dtype, got, ref):
    for name, r in ref.items():
        if name in got:
            _close(dtype, name, got[name], r)


# (N, C, (D, H, W), (Do, Ho, Wo)).  In f32 channels-last, C = 4 and 24 take the float4 forward, C = 1, 5 and 33 the
# scalar fallback.
SHAPES = [
    (1, 1, (1, 9, 7), (1, 1, 255)),
    (3, 5, (17, 33, 21), (4, 5, 7)),
    (3, 24, (17, 33, 21), (1, 1, 1)),
    (2, 33, (9, 1, 16), (3, 1, 11)),
    (3, 4, (6, 5, 1), (2, 9, 13)),
    (1, 24, (65, 17, 33), (5, 1, 255)),
]


@pytest.mark.parametrize("case", SHAPES, ids=lambda c: f"N{c[0]}C{c[1]}-{'x'.join(map(str, c[2]))}-P{'x'.join(map(str, c[3]))}")
@pytest.mark.parametrize("layout", [NCDHW, NDHWC], ids=["ncdhw", "ndhwc"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_gridsample_all_orders_match_float64(dtype, layout, case):
    N, C, dhw, ohw = case
    dev, ref = _tensors(N, C, dhw, ohw, dtype, seed=11 + C)
    _check_all(dtype, _run(*dev, layout), _oracle(*ref))


@pytest.mark.parametrize("waves,dtype,layout", [(1, torch.float32, NCDHW), (1, torch.float64, NDHWC),
                                                (3, torch.float32, NDHWC)],
                         ids=["1wave-f32-ncdhw", "1wave-f64-ndhwc", "3wave-f32-ndhwc"])
def test_gridsample_grid_stride_passes(waves, dtype, layout):
    """N P = waves x (SMs x 8 x 256) + 77: every thread runs `waves` iterations of the grid-stride loop, the first
    77 one more."""
    P = waves * _wave() + R_TAIL
    dev, ref = _tensors(1, 4, (17, 33, 21), (1, 1, P), dtype, seed=20 + waves)
    _check_all(dtype, _run(*dev, layout), _oracle(*ref))


@pytest.mark.parametrize("layout", [NCDHW, NDHWC], ids=["ncdhw", "ndhwc"])
def test_gridsample_no_points(layout):
    inp = _to_layout(torch.randn((2, 24, 5, 6, 7), device=DEV), layout)
    grid = torch.empty((2, 1, 1, 0, 3), device=DEV)
    go = torch.empty((2, 24, 1, 1, 0), device=DEV)
    assert ops.grid_sample3d_forward(inp, grid, layout).shape == (2, 24, 1, 1, 0)
    gi, gg = ops.grid_sample3d_backward(inp, grid, go, layout)
    assert gg.shape == grid.shape and torch.equal(gi, torch.zeros_like(inp))
    d0, d1, d2 = ops.grid_sample3d_dbackward(torch.randn_like(inp), torch.empty_like(grid), inp, grid, go, layout)
    assert torch.equal(d0, torch.zeros_like(inp)) and d1.shape == grid.shape and d2.shape == go.shape


def test_gridsample_float4_and_scalar_forward_agree():
    """C = 24 channels-last at a 16-byte aligned pointer takes gs3d_fwd_cl4_kernel; the same voxel one float into its
    buffer takes the scalar kernel.  Both sum the corners in the same order, so they agree bit for bit."""
    N, C, dhw = 3, 24, (17, 33, 21)
    dev, ref = _tensors(N, C, dhw, (2, 3, 171), torch.float32, seed=5)
    x = _to_layout(dev[0], NDHWC)
    buf = torch.empty(x.numel() + 1, dtype=torch.float32, device=DEV)
    shifted = buf[1:].view(x.shape)
    shifted.copy_(x)
    assert x.data_ptr() % 16 == 0 and shifted.data_ptr() % 16 == 4 and shifted.is_contiguous()
    a = ops.grid_sample3d_forward(x, dev[1], NDHWC)
    b = ops.grid_sample3d_forward(shifted, dev[1], NDHWC)
    assert torch.equal(a, b)
    _close(torch.float32, "out", b, ot.grid_sample3d_fwd(ref[0], ref[1]))
    gi, gg = ops.grid_sample3d_backward(shifted, dev[1], dev[2], NDHWC)
    r = _oracle(*ref)
    _close(torch.float32, "grad_grid", gg, r["grad_grid"])
    _close(torch.float32, "grad_input", _from_layout(gi, NDHWC), r["grad_input"])


def _lattice_points(shape, dhw, gen):
    """Every coordinate is a lattice plane: g = (2k + 1) / S - 1 with S a power of two gives the unnormalised coordinate
    k exactly in fp32 and fp64.  k runs from -2 to S + 1, so points also sit on the border (k = 0, S - 1) and past it."""
    g = torch.empty(tuple(shape) + (3,), dtype=torch.float64)
    for a, S in enumerate(reversed(dhw)):
        k = torch.randint(-2, S + 2, tuple(shape), generator=gen).double()
        g[..., a] = (2 * k + 1) / S - 1
    return g


@pytest.mark.parametrize("layout", [NCDHW, NDHWC], ids=["ncdhw", "ndhwc"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_gridsample_lattice_border_and_infinite_points(dtype, layout):
    N, C, dhw = 2, 8, (8, 16, 4)
    gen = synth.generator(31)
    P = 1000
    grid = _points((N, 1, 1, P), dhw, gen)
    lat = _lattice_points((N, 1, 1, P), dhw, gen)
    pick = torch.rand(grid.shape, generator=gen) < 0.7          # mostly lattice, some axes off it
    grid = torch.where(pick, lat, grid)
    for n in range(N):                                          # all-lattice points and infinities, on every axis
        grid[n, 0, 0, :100] = lat[n, 0, 0, :100]
        for a in range(3):
            grid[n, 0, 0, 100 + 20 * a: 110 + 20 * a, a] = float("inf")
            grid[n, 0, 0, 110 + 20 * a: 120 + 20 * a, a] = float("-inf")
    for a, S in enumerate(reversed(dhw)):                       # exact integers in fp32 as well
        x = ((lat[..., a].float() + 1) * S - 1) / 2
        assert torch.equal(x, torch.round(x))
    dev, ref = _tensors(N, C, dhw, (1, 1, P), dtype, seed=32, grid=grid)
    got = _run(*dev, layout)
    assert all(bool(torch.isfinite(t).all()) for t in got.values())
    _check_all(dtype, got, _oracle(*ref))


@pytest.mark.parametrize("layout", [NCDHW, NDHWC], ids=["ncdhw", "ndhwc"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_gridsample_nan_coordinate_samples_zero_and_has_no_gradient(dtype, layout):
    """A NaN coordinate samples at unnormalised coordinate 0 on its axis and gets no gradient there, as in the fused
    skinning kernels.  So every output equals the oracle's at a coordinate clipped to 0 (here -2), where the
    derivative is zero too."""
    N, C, dhw = 2, 24, (17, 33, 21)
    gen = synth.generator(41)
    P = 300
    grid = _points((N, 1, 1, P), dhw, gen)
    nan = torch.zeros(grid.shape, dtype=torch.bool)
    nan[:, :, :, 0::3, 0] = True
    nan[:, :, :, 1::3, 1] = True
    nan[:, :, :, 2::3, 2] = True
    nan[:, :, :, :30] = True                                    # all three axes
    dev, ref = _tensors(N, C, dhw, (1, 1, P), dtype, seed=42, grid=grid.masked_fill(nan, float("nan")))
    ref[1] = grid.masked_fill(nan, -2.0).to(dtype).double().to(DEV)
    got = _run(*dev, layout)
    for name in ("grad_grid", "g_grid"):
        assert bool(torch.isfinite(got[name]).all())
        assert bool((got[name].cpu()[nan] == 0).all()), f"{name}: a NaN axis has a gradient"
    _check_all(dtype, got, _oracle(*ref))


@pytest.mark.parametrize("layout", [NCDHW, NDHWC], ids=["ncdhw", "ndhwc"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_gridsample_nullable_outputs(dtype, layout):
    """need_grad_input=False skips the atomically accumulated volume and changes no bit of the other outputs;
    gg_input=None is a zero gg_input."""
    dev, ref = _tensors(2, 24, (17, 33, 21), (3, 1, 333), dtype, seed=51)
    full = _run(*dev, layout)
    frozen = _run(*dev, layout, need_grad_input=False)
    for name in ("out", "grad_grid", "g_grid", "gg_out"):
        assert torch.equal(full[name], frozen[name]), name
    inp, grid, go, _, ggg = dev
    x = _to_layout(inp, layout)
    r0, r1, r2 = ot.grid_sample3d_bwd2(torch.zeros_like(ref[0]), ref[4], ref[0], ref[1], ref[2])
    for need in (True, False):
        d0, d1, d2 = ops.grid_sample3d_dbackward(None, ggg, x, grid, go, layout, need_grad_input=need)
        _close(dtype, "g_grid", d1, r1)
        _close(dtype, "gg_out", d2, r2)
        if need:
            _close(dtype, "g_input", _from_layout(d0, layout), r0)
        else:
            assert d0 is None


def _guarded(n, dtype, zero=False):
    """A buffer of n + 2 GUARD elements filled with a NaN bit pattern; returns (buffer, the n-element middle).  With
    zero=True the middle starts at zero (for the atomically accumulated volumes)."""
    itype, pat = (torch.int32, NAN32) if dtype == torch.float32 else (torch.int64, NAN64)
    buf = torch.full((n + 2 * GUARD,), pat, dtype=itype, device=DEV).view(dtype)
    mid = buf[GUARD:GUARD + n]
    if zero:
        mid.zero_()
    return buf, mid


def _guards_intact(buf, n, dtype):
    itype, pat = (torch.int32, NAN32) if dtype == torch.float32 else (torch.int64, NAN64)
    bits = buf.view(itype)
    return bool((bits[:GUARD] == pat).all()) and bool((bits[GUARD + n:] == pat).all())


def _all_written(mid, dtype):
    itype, pat = (torch.int32, NAN32) if dtype == torch.float32 else (torch.int64, NAN64)
    return not bool((mid.view(itype) == pat).any())


@pytest.mark.parametrize("C", [5, 24])
@pytest.mark.parametrize("layout", [NCDHW, NDHWC], ids=["ncdhw", "ndhwc"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
def test_gridsample_c_abi_output_bounds(dtype, layout, C):
    """Every output of recmv_gridsample3d_{fwd,bwd,bwd2} in a NaN-guarded buffer: the guards stay bit-unchanged,
    out / grad_grid / g_grid / gg_out are written in full and equal the ops.py results bit for bit.  grad_input and
    g_input sit zeroed between the guards, so a corner index past the volume changes a guard."""
    N, dhw, P = 2, (17, 33, 21), 1000 + C
    dev, ref = _tensors(N, C, dhw, (1, 1, P), dtype, seed=61 + C)
    inp, grid, go, ggi, ggg = dev
    x, gx = _to_layout(inp, layout), _to_layout(ggi, layout)
    code = _lib.F32 if dtype == torch.float32 else _lib.F64
    lib, st, p = _lib.load(), ops._stream(x), ops._ptr
    D, H, W = dhw
    nout, ngrid, nvox = N * C * P, N * P * 3, x.numel()
    ob, out = _guarded(nout, dtype)
    gib, gi = _guarded(nvox, dtype, zero=True)
    ggb, gg = _guarded(ngrid, dtype)
    d0b, d0 = _guarded(nvox, dtype, zero=True)
    d1b, d1 = _guarded(ngrid, dtype)
    d2b, d2 = _guarded(nout, dtype)
    assert lib.recmv_gridsample3d_fwd(p(x), p(grid), p(out), N, C, D, H, W, P, code, layout, st) == 0
    assert lib.recmv_gridsample3d_bwd(p(x), p(grid), p(go), p(gi), p(gg), N, C, D, H, W, P, code, layout, st) == 0
    assert lib.recmv_gridsample3d_bwd2(p(gx), p(ggg), p(x), p(grid), p(go), p(d0), p(d1), p(d2), N, C, D, H, W, P, code,
                                       layout, st) == 0
    torch.cuda.synchronize()
    for buf, mid, n in ((ob, out, nout), (gib, gi, nvox), (ggb, gg, ngrid), (d0b, d0, nvox), (d1b, d1, ngrid),
                        (d2b, d2, nout)):
        assert _guards_intact(buf, n, dtype)
    for mid in (out, gg, d1, d2):
        assert _all_written(mid, dtype)
    res = _run(*dev, layout)
    assert torch.equal(out, res["out"].reshape(-1)) and torch.equal(gg, res["grad_grid"].reshape(-1))
    assert torch.equal(d1, res["g_grid"].reshape(-1)) and torch.equal(d2, res["gg_out"].reshape(-1))
    r = _oracle(*ref)
    _close(dtype, "grad_input", _from_layout(gi.view(x.shape), layout), r["grad_input"])
    _close(dtype, "g_input", _from_layout(d0.view(x.shape), layout), r["g_input"])


def test_lbskinner_composite_sampler_first_and_second_derivatives():
    """FrozenVoxelSampleFunction on the cached channels-last 24-channel voxel, points also outside the skinning box:
    the sample, its gradient under create_graph and that gradient's derivatives (by the points and by the
    cotangent) against float64 autograd of the oracle on the NCDHW voxel."""
    dhw = (17, 33, 21)
    ws = synth.skinning_voxel(dhw, seed=7)
    ws_cl = ops.voxel_to_channels_last(ws.to(DEV))
    gen = synth.generator(71)
    P = 5003
    grid = _points((1, 1, 1, P), dhw, gen, span=1.5).float()
    assert bool(((grid.abs() > 1).any(-1)).float().mean() > 0.3)
    w = torch.randn((1, 24, 1, 1, P), generator=gen)
    v = torch.randn(grid.shape, generator=gen)
    g_d, w_d = grid.to(DEV).requires_grad_(True), w.to(DEV).requires_grad_(True)
    out = ops.FrozenVoxelSampleFunction.apply(ws_cl.view(1, *ws_cl.shape), g_d)
    (g1,) = torch.autograd.grad(out, g_d, w_d, create_graph=True)
    h, hw = torch.autograd.grad(g1, (g_d, w_d), v.to(DEV))
    g_r, w_r = (t.double().to(DEV).requires_grad_(True) for t in (grid, w))
    out_r = ot.grid_sample3d_fwd(ws.double().to(DEV), g_r)
    (g1_r,) = torch.autograd.grad(out_r, g_r, w_r, create_graph=True)
    h_r, hw_r = torch.autograd.grad(g1_r, (g_r, w_r), v.double().to(DEV))
    f32 = torch.float32
    _close(f32, "out", out, out_r)
    _close(f32, "grad_grid", g1, g1_r)
    _close(f32, "g_grid", h, h_r)
    _close(f32, "gg_out", hw, hw_r)


@pytest.mark.parametrize("C", [1, 24, 32, 33, 64])
@pytest.mark.parametrize("dhw", [(5, 7, 9), (64, 64, 64)], ids=["315", "64cube"])
def test_voxel_to_channels_last_is_a_permute(C, dhw):
    """D H W = 315 is not a multiple of the 32-position tile; 64^3 positions are more than 32 x 8 x SMs, so
    vox_cl_kernel's grid-stride loop takes a second pass."""
    if dhw == (64, 64, 64):
        assert 64 ** 3 > 32 * 8 * _sms()
    ws = torch.randn((1, C) + dhw, generator=synth.generator(C), dtype=torch.float32).to(DEV)
    assert torch.equal(ops.voxel_to_channels_last(ws), ws[0].permute(1, 2, 3, 0).contiguous())


# ------------------------------------------------------------------------------------------------ marching cubes
def _scan_per(shape):
    """Segment sums per thread of mc_scan_kernel: ceil(ceil(N / 1024) / 1024)."""
    nb = -(-int(np.prod(shape)) // 1024)
    return -(-nb // 1024)


def _mc_against_oracle(sdf, iso=0.0):
    n = sdf.shape
    step = tuple(2.0 / (s - 1) for s in n)
    dev = sdf.to(DEV)
    v, f = ops.mc_gpu(dev, *step, -1.0, -1.0, -1.0, iso)
    rv, rf = mc_oracle.marching_cubes(sdf.cpu().numpy(), step, (-1, -1, -1), iso)
    assert v.shape[0] == len(rv) and f.shape[0] == len(rf)
    assert np.array_equal(f.cpu().numpy(), rf)                  # same faces in the same order
    assert len(rv) == 0 or np.abs(v.cpu().numpy() - rv).max() < 1e-6
    return v, f


@pytest.mark.parametrize("res,per", [(129, 3), (257, 17)])
def test_marching_cubes_smooth_grid_matches_oracle(res, per):
    assert _scan_per((res,) * 3) == per
    v, f = _mc_against_oracle(synth.sphere_sdf_grid(res, num=8, seed=3, device=DEV))
    assert f.shape[0] > 10000


def test_marching_cubes_dense_grid_matches_oracle():
    """Random signs at every lattice point: almost every cell is active, segments carry their largest counts, the
    per-warp compaction list runs full, and the one-call path has to grow its buffers."""
    shape = (129, 127, 131)
    sdf = torch.randn(shape, generator=synth.generator(81))
    s = (sdf < 0).numpy()
    corners = [s[i:i + shape[0] - 1, j:j + shape[1] - 1, k:k + shape[2] - 1] for i in (0, 1) for j in (0, 1) for k in (0, 1)]
    active = np.logical_or.reduce(corners) & ~np.logical_and.reduce(corners)
    assert active.mean() > 0.99
    ops._scratch_cache.clear()                                 # start from the smallest buffers: forces a regrowth
    v, f = _mc_against_oracle(sdf)
    assert v.shape[0] > 2_500_000 and f.shape[0] > 2_500_000


@pytest.mark.parametrize("shape", [(301, 203, 2), (37, 29, 31)])
def test_marching_cubes_quantised_grid_on_the_iso_value(shape):
    """Values in {-1, 0, 1} with iso = 0: a third of the lattice sits exactly on the iso value (`v < iso` is strict, so
    those corners count as outside and their vertices land on the corner).  NZ = 2 makes every 32-cell run cross z
    rows; neither shape's point count is a multiple of 1024."""
    assert int(np.prod(shape)) % 1024 != 0
    sdf = torch.randint(-1, 2, shape, generator=synth.generator(91)).float()
    v, f = _mc_against_oracle(sdf)
    assert f.shape[0] > 1000


# ------------------------------------------------------------------------------------------------ fragment decode
class _Frags:
    def __init__(self, p2f, bary):
        self.pix_to_face, self.bary_coords = p2f, bary


def _fragments(N, H, W, K, coverage, seed, V=1000, F=3000):
    """Fragments whose face ids run up to N F - 1 (the `% num_faces` path).  coverage: "all" (every pixel has a valid
    fragment, at a random layer behind invalid ones), "none", or "mix"."""
    gen = synth.generator(seed)
    verts = torch.randn((V, 3), generator=gen) * 0.5             # |seed point| < 8: one fp32 ulp stays below 1e-6
    faces = torch.randint(0, V, (F, 3), generator=gen)
    p2f = torch.randint(0, N * F, (N, H, W, K), generator=gen)
    bary = torch.rand((N, H, W, K, 3), generator=gen) + 1e-3
    invalid = torch.rand((N, H, W, K), generator=gen)
    if coverage == "all":
        first = torch.randint(0, K, (N, H, W, 1), generator=gen)
        invalid = torch.where(torch.arange(K).view(1, 1, 1, K) < first, invalid * 0.6, torch.ones(()))
    elif coverage == "none":
        invalid = invalid * 0.6                                 # every fragment invalid, for one of the two reasons
    p2f[invalid < 0.3] = -1
    bary[(invalid >= 0.3) & (invalid < 0.6)] *= -1.0
    return verts, faces, p2f, bary


FRAG_CASES = [  # (N, H, W, K, coverage); 262 144 pixels = 1024 blocks of 256 = one chunk of frag_scan_kernel
    (1, 512, 512, 1, "mix"),
    (1, 512, 512, 8, "all"),
    (1, 512, 512, 2, "none"),
    (1, 5, 52429, 2, "mix"),        # 262 145 pixels: one block into the second chunk
    (1, 5, 52429, 1, "all"),
    (2, 1024, 768, 1, "all"),       # six chunks
    (2, 1024, 768, 2, "mix"),
    (2, 1024, 768, 8, "mix"),
]


@pytest.mark.parametrize("case", FRAG_CASES, ids=lambda c: f"{c[0]}x{c[1]}x{c[2]}-K{c[3]}-{c[4]}")
def test_fragment_decode_matches_cpu_path(case):
    N, H, W, K, coverage = case
    verts, faces, p2f, bary = _fragments(N, H, W, K, coverage, seed=H + K)
    rb, rr, rc, rp, rf = FindSurfacePs(verts, faces, _Frags(p2f, bary))       # CPU tensors: the torch path
    b, r, c, p, f = ops.fragment_decode(p2f.to(DEV), bary.to(DEV), verts.to(DEV), faces.to(DEV))
    for got, want in ((b, rb), (r, rr), (c, rc), (f, rf)):
        assert got.dtype == torch.int64 and torch.equal(got.cpu(), want)
    assert p.shape == rp.shape and (rp.numel() == 0 or float((p.cpu() - rp).abs().max()) < 1e-6)
    if coverage == "all":
        assert b.numel() == N * H * W
    elif coverage == "none":
        assert b.numel() == 0
    else:
        assert 0 < b.numel() < N * H * W


def test_fragment_decode_mask_and_rays_at_six_chunks():
    N, H, W, K = 2, 1024, 768, 2
    verts, faces, p2f, bary = _fragments(N, H, W, K, "mix", seed=101)
    gen = synth.generator(102)
    mask = (torch.rand((N, H, W), generator=gen) > 0.3).float()
    fx, fy, px, py = 1.2 * W, 1.1 * W, W / 2 - 0.3, H / 2 + 0.2
    R = torch.linalg.qr(torch.randn((3, 3), generator=gen))[0]
    b, r, c, pts, fi = FindSurfacePs(verts, faces, _Frags(p2f, bary))
    sel = mask[b, r, c] > 0.
    ps = torch.stack([c[sel].float(), r[sel].float(), torch.ones_like(c[sel]).float()], 1)
    rays = torch.zeros_like(ps)
    rays[:, 0] = -ps[:, 0] / fx + ps[:, 2] * px / fx
    rays[:, 1] = -ps[:, 1] / fy + ps[:, 2] * py / fy
    rays[:, 2] = ps[:, 2]
    rays = (rays / torch.norm(rays, p=2, dim=1, keepdim=True)).matmul(R.transpose(0, 1))
    fr = _Frags(p2f.to(DEV), bary.to(DEV))
    b2, r2, c2, pts2, fi2, rays2 = FindSurfacePsRays(verts.to(DEV), faces.to(DEV), fr, (fx, fy, px, py, R), mask.to(DEV))
    for got, want in ((b2, b[sel]), (r2, r[sel]), (c2, c[sel]), (fi2, fi[sel])):
        assert torch.equal(got.cpu(), want)
    assert float((pts2.cpu() - pts[sel]).abs().max()) < 1e-6 and float((rays2.cpu() - rays).abs().max()) < 1e-6
    assert b2.numel() > 500_000


# ------------------------------------------------------------------------------------------------ argument checks
def test_gridsample_rejects_mismatched_operands():
    """Each mismatch is at least as large as what the kernel would read, so without the check it reads wrong data,
    never outside an allocation."""
    inp = torch.randn((1, 3, 4, 5, 6), device=DEV)
    grid = torch.rand((1, 1, 1, 10, 3), device=DEV) * 2 - 1
    go = torch.randn((1, 3, 1, 1, 10), device=DEV)
    ggg = torch.randn_like(grid)
    ops.grid_sample3d_backward(inp, grid, go)
    ops.grid_sample3d_dbackward(torch.randn_like(inp), ggg, inp, grid, go)
    with pytest.raises(RuntimeError):
        ops.grid_sample3d_backward(inp, grid, go.double())
    with pytest.raises(RuntimeError):
        ops.grid_sample3d_backward(inp, grid, torch.randn((1, 3, 1, 1, 11), device=DEV))
    with pytest.raises(RuntimeError):
        ops.grid_sample3d_dbackward(None, ggg, inp, grid, go.double())
    with pytest.raises(RuntimeError):
        ops.grid_sample3d_dbackward(None, torch.randn((1, 1, 1, 11, 3), device=DEV), inp, grid, go)
    with pytest.raises(RuntimeError):
        ops.grid_sample3d_dbackward(None, ggg.double(), inp, grid, go)
    with pytest.raises(RuntimeError):
        ops.grid_sample3d_dbackward(torch.randn_like(inp).double(), ggg, inp, grid, go)


def test_voxel_to_channels_last_rejects_other_dtypes_and_batches():
    ws = torch.randn((1, 24, 5, 6, 7), device=DEV)
    with pytest.raises(RuntimeError):
        ops.voxel_to_channels_last(ws.double())
    with pytest.raises(RuntimeError):
        ops.voxel_to_channels_last(torch.cat([ws, ws]))


def test_fragment_decode_rejects_a_mask_of_another_size():
    verts, faces, p2f, bary = _fragments(1, 16, 16, 2, "mix", seed=111)
    args = (p2f.to(DEV), bary.to(DEV), verts.to(DEV), faces.to(DEV))
    ops.fragment_decode(*args, torch.ones((1, 16, 16), device=DEV))
    with pytest.raises(RuntimeError):
        ops.fragment_decode(*args, torch.ones((1, 16, 17), device=DEV))
