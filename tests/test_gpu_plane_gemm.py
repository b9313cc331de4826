"""The TMA-fed training GEMMs on fp16 hi / lo operand planes (csrc/gemm3_tma.cu) against float64, across multi-wave
launches, ragged shapes, the operand planes they emit and their output bounds:

    recmv_mlp_layer_planes   gemm3_tma_kernel: every mode at every shape the training path launches (LAYERS)
    recmv_mlp_wgrad_planes   gemm3_wgrad_kernel + the split-order reductions, and recmv_colsum (WG_SHAPES x WG_SIZES)
    split_planes (plain and transposed), pe_forward_planes, softplus_tangent_planes, add_split_planes, and the fp16 range
    report of the four kernels that split (tags 3500, 3600, 3700, 3710)
    the SDF, translator and colour training steps, the ReLU networks' create_graph input gradient and the eikonal term,
    end to end at multi-wave sizes

gemm3_tma_kernel is persistent with a grid of min(tiles, SMs): CTA b walks tiles b, b + S, ... and carries the ring stage
and parities, the accumulator, the TMA warp's run-ahead into the next tile and the epilogue's tile coordinates from one
tile to the next.  So a CTA reaches a second tile only when a launch has more tiles than the device has SMs.  Row counts
come from the SM count S and the column tiles T_n = ceil(N / 128): 1, 127, 129, one wave floor(S / T_n) 128, one wave + 1,
ceil(3 S / T_n) 128 + r (every CTA runs at least three tiles) and, for the bit-exact checks, ceil(10 S / T_n) 128 + r.

Kinds of checks:
  * accuracy against float64 of the fp32 inputs (merr of test_gpu_train.py, bounds at the top of the file);
  * emitted planes, bit-exact: y_hi / y_lo equal ops.split_planes of the fp32 output (same fp32 scale, same rounding);
  * position invariance, bit-exact: a multi-wave launch equals launches of at most one wave (one tile per CTA), and a
    permuted batch gives the permuted outputs.  Each output element depends only on its own row, its MMAs run in a fixed
    order and the accumulation gain depends only on K, so any difference means that a tile leaked into another;
  * output bounds: outputs are views into buffers with GUARD rows of a NaN bit pattern on each side and guard columns
    past the written width; the guards stay bit-unchanged and every element of the output is written;
  * operand padding is never read: fp16 NaN in the planes' columns >= K and rows >= M / N changes no bit."""
import math

import pytest
import torch

from recmv_b200 import _lib, ops, testing
from recmv_b200.model import getTmpSdf
from recmv_b200.model.Embedder import ratio_to_weights

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GUARD = 128              # guard rows before and after every output (one row tile)
NAN32 = 0x7FBADBAD       # fp32 NaN bit pattern no kernel writes
NAN16 = 0x7E5B           # fp16 NaN bit pattern no kernel writes
R_TAIL = 77              # the ragged r of the multi-wave sizes
F16_MAX = 0x7BFF         # bits of fp16 65504
INV_SQRT2 = ops._INV_SQRT2
OK, E_DTYPE, E_SHAPE, E_UNSUPPORTED, E_DEVICE = 0, -2, -3, -5, -6

# Bounds against float64, max |a - b| / max |b| per tensor (a layer's output is Y and Y2 side by side).  Measured on an
# H100 80GB HBM3 (700 W power limit), maximum over every case of this file (the inputs are seeded):
#   layer GEMM                   1.9e-6 (rgb.bwd0; tangent 1.8e-6 at M = 1); same-sign 2.1e-6, its signed relative bias
#                                -2.1e-6 .. -2.0e-6 at every M
#   weight gradient              dW 4.2e-7 (P <= 10 000), 4.9e-6 (P > 10 000), 6.3e-6 (out_dim 3, P = 131 072);
#                                db (ones tile) 4.4e-6; colsum 9.3e-7
#   softplus_tangent             u 6.7e-8, inj 1.0e-7
#   SDF step                     6.6e-6 (sdf, feat, dx, dW, db at 3wave+r and 131 072 points)
#   translator / colour step     3.6e-6 given our ReLU masks (output, dX0, dW, db); 5 and 7 mask flips, all at |z| < 5e-6
#   their create_graph dX0       5.6e-6 given our ReLU masks (the backward's g_out and dW)
#   eikonal                      loss 3.4e-6, gradient / dx / parameter gradients 1.1e-5
# test_gpu_train.py's 1.5e-6 single-layer bar was measured with cotangents of one scale at M >= 129.  The cotangents
# here have a per-row log-normal scale and the outputs are as narrow as 39 columns or one row, so the largest |b| is a
# single row or column with cancellation in it.  With all products positive the truncating accumulation loses more than
# the fitted gain returns (DESIGN.md section 5c).  Both are above that bar, and LAYER_BOUND is about 3x the larger.
# With out_dim = 3 the largest |dW| is taken over 3 rows instead of hundreds, which puts P = 131 072 above the 6e-6 bar;
# that shape has its own bound.  The weight gradient keeps its 3e-6 / 6e-6 and 5e-6
# bars otherwise, the colsum its 2e-6, the SDF step its 3e-5, the eikonal term test_gpu_second_order.py's 5e-5; the
# other bounds are about 3x the measured maximum.
LAYER_BOUND = 6e-6
WG_BOUND, WG_BOUND_LARGE, WG_BOUND_NARROW, DB_BOUND, COLSUM_BOUND = 3e-6, 6e-6, 2e-5, 5e-6, 2e-6
TANGENT_BOUND = 3e-7
SDF_STEP_BOUND = 3e-5
PLAIN_STEP_BOUND = 1e-5
EIKONAL_BOUND = 5e-5


@pytest.fixture(autouse=True)
def _no_aborted_launch():
    yield
    torch.cuda.synchronize()
    ops.check_async_errors()  # every mbarrier wait of the plane kernels is bounded; none may have timed out


def merr(a, b):
    a = torch.as_tensor(a).detach().double()
    b = torch.as_tensor(b).detach().double().to(a.device)
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tiles_n(N):
    return (N + 127) // 128


def _rows(tag, N):
    S, tn = _sms(), _tiles_n(N)
    wave = (S // tn) * 128
    return {"1": 1, "127": 127, "129": 129, "wave": wave, "wave+1": wave + 1,
            "3wave+r": math.ceil(3 * S / tn) * 128 + R_TAIL, "10wave+r": math.ceil(10 * S / tn) * 128 + R_TAIL}[tag]


def _assert_waves(tag, M, N):
    k = {"3wave+r": 3, "10wave+r": 10}.get(tag)
    if k:   # every CTA of the persistent grid runs at least k tiles
        assert (M + 127) // 128 * _tiles_n(N) >= k * _sms()


def _pad8(n):
    return (int(n) + 7) // 8 * 8


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _softplus_acts(shape, g):
    return torch.nn.functional.softplus(torch.randn(shape, generator=g, device=DEV) * 0.02, beta=100)


def _cotangents(shape, g, scale=1e-4):
    return torch.randn(shape, generator=g, device=DEV) * scale * torch.exp(torch.randn((shape[0], 1), generator=g, device=DEV))


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _pattern(dtype):
    return NAN32 if dtype == torch.float32 else NAN16


class Guarded:
    """A [rows, cols] view (row stride ld, first element `offset` past its row start) into a buffer with GUARD rows of a NaN
    bit pattern before and after and NaN guard columns past cols."""

    def __init__(self, rows, cols, dtype, ld, offset=0):
        assert cols + offset <= ld
        self.buf = torch.empty((rows + 2 * GUARD, ld), dtype=dtype, device=DEV)
        _bits(self.buf).fill_(_pattern(dtype))
        self.view = torch.as_strided(self.buf, (rows, cols), (ld, 1), GUARD * ld + offset)
        self.mask = torch.zeros((rows + 2 * GUARD, ld), dtype=torch.bool, device=DEV)
        torch.as_strided(self.mask, (rows, cols), (ld, 1), GUARD * ld + offset).fill_(True)

    def check(self, what):
        b = _bits(self.buf)
        assert bool((b[~self.mask] == _pattern(self.buf.dtype)).all()), f"{what}: a guard element was written"
        assert not bool((b[self.mask] == _pattern(self.buf.dtype)).any()), f"{what}: an output element was not written"


# ---------------------------------------------------------------------------------------------------------------------
# the layer GEMM: every launch shape of the training path
# ---------------------------------------------------------------------------------------------------------------------
class Layer:
    def __init__(self, name, mode, K, N, split=0, y2=False, scale=1.0, bias=True, positive=False, signed=False):
        self.name, self.mode, self.K, self.N, self.scale = name, mode, K, N, scale
        self.split = split if 0 < split < N else N
        self.y2 = y2
        self.fwd = mode >= 4
        self.bias = bias and self.fwd
        self.dyn = not self.fwd                      # backward-data: cotangent planes carry 64 dyn
        self.planes = mode in (1, 2, 5, 6)           # launches that write the next GEMM's A planes
        self.positive, self.signed = positive, signed

    def __repr__(self):
        return self.name


LAYERS = [
    # SDF forward (ops.SdfMlpTrainFunction.forward)
    Layer("sdf.fwd0", 5, 39, 512), Layer("sdf.fwd1", 5, 512, 512),
    Layer("sdf.fwd3", 5, 512, 473),                               # planes into the 512-wide buffer of layer 4's input
    Layer("sdf.fwd4", 5, 512, 512, scale=INV_SQRT2), Layer("sdf.fwd8", 4, 512, 257, split=1, y2=True),
    # SDF backward-data (ops.SdfMlpTrainFunction.backward, second_order.py)
    Layer("sdf.bwd8", 1, 257, 512), Layer("sdf.bwd4", 1, 512, 512, split=473, y2=True, scale=INV_SQRT2),
    Layer("sdf.bwd3", 1, 473, 512), Layer("sdf.bwd0", 0, 512, 39),
    # translator (ops._plain_mlp_forward / _plain_mlp_backward, 167 -> 512 x4 -> 3)
    Layer("tr.fwd0", 6, 167, 512), Layer("tr.fwd4", 4, 512, 3), Layer("tr.bwd4", 2, 3, 512), Layer("tr.bwd0", 0, 512, 167),
    # colour network (289 -> 512 x4 -> 3)
    Layer("rgb.fwd0", 6, 289, 512), Layer("rgb.bwd0", 0, 512, 289),
    # second-order tangent pass: no bias, signed operands
    Layer("tangent", 4, 512, 512, bias=False, signed=True),
    # geometric-init output layer: every product positive, the accumulation's truncation bias does not average out
    Layer("same-sign", 4, 512, 257, split=1, y2=True, positive=True),
    # the ReLU networks' tangent pass (second_order.PlainMlpInputGradFunction): backward-data modes on the [out][in] weight
    # planes, so K and N are those of the forward layer
    Layer("tr.tan0", 2, 167, 512), Layer("rgb.tan0", 2, 289, 512), Layer("tr.tan4", 0, 512, 3),
]
BY_NAME = {l.name: l for l in LAYERS}
LAYER_SIZES = ["1", "127", "129", "wave", "wave+1", "3wave+r"]


def _layer_inputs(L, M, seed):
    """fp32 operands of one launch and their planes (zero padded, as ops.split_planes writes them)."""
    g = _gen(seed)
    c = {}
    if L.fwd:
        A = torch.randn((M, L.K), generator=g, device=DEV) * 0.05 if L.signed else _softplus_acts((M, L.K), g)
        W = torch.randn((L.N, L.K), generator=g, device=DEV) * 0.05                  # [out][in]
        if L.positive:
            W = W.abs()
        c["bp"] = ops.split_planes(W, L.N, L.K, 1024.0)
        c["bias"] = torch.randn((L.N,), generator=g, device=DEV) * 0.05 if L.bias else None
        c["dyn"] = None
        c["ap"] = ops.split_planes(A, M, L.K, 64.0, ldp=_pad8(L.K))
    else:
        A = _cotangents((M, L.K), g)
        W = torch.randn((L.K, L.N), generator=g, device=DEV) * 0.05                  # [out][in]: the layer's weights
        c["bp"] = ops.split_planes(W, L.K, L.N, 1024.0, transpose=True)              # [in][out]
        c["bias"] = None
        c["dyn"] = ops.grad_dyn_scale(A)
        c["ap"] = ops.split_planes(A, M, L.K, 64.0, scale_dev=c["dyn"], ldp=_pad8(L.K))
    c["E"] = None
    if L.mode == 1:
        c["E"] = _softplus_acts((M, L.N), g)
    elif L.mode == 2:
        c["E"] = torch.relu(torch.randn((M, L.N), generator=g, device=DEV))
    c["A"], c["W"] = A, W
    return c


def _reference(L, c):
    A, W = c["A"].double(), c["W"].double()
    z = (A @ W.T if L.fwd else A @ W) * L.scale
    if L.fwd:
        if c["bias"] is not None:
            z = z + c["bias"].double()
        if L.mode == 5:
            z = torch.nn.functional.softplus(z, beta=100)
        elif L.mode == 6:
            z = torch.relu(z)
        return z[:, :L.split], z[:, L.split:]
    E = c["E"].double() if c["E"] is not None else None
    y = z[:, :L.split]
    if L.mode == 1:
        y = y * (1 - torch.exp(-100 * E[:, :L.split]))
    elif L.mode == 2:
        y = y * (E[:, :L.split] > 0).double()
    return y, z[:, L.split:]


def _launch(L, ap, bp, M, c, Y, Y2=None, yp=None, E=None, mode=None, a_has_dyn=None, planes_with_dyn=None):
    """recmv_mlp_layer_planes through the C entry (status returned, not raised)."""
    yh, yl = yp if yp is not None else (None, None)
    E = c["E"] if E is None else E
    a_has_dyn = L.dyn if a_has_dyn is None else a_has_dyn
    planes_with_dyn = (L.dyn and yp is not None) if planes_with_dyn is None else planes_with_dyn
    with torch.cuda.device(DEV):
        return _lib.load().recmv_mlp_layer_planes(
            ops._ptr(ap[0]), ops._ptr(ap[1]), ap[0].stride(0), ops._ptr(bp[0]), ops._ptr(bp[1]), bp[0].stride(0), int(M),
            L.N, L.K, L.mode if mode is None else mode, ops._ptr(c["bias"]), ops._ptr(E), E.stride(0) if E is not None else 0,
            float(L.scale), ops._ptr(c["dyn"]), 1 if a_has_dyn else 0, L.split if L.split < L.N else 0, ops._ptr(Y),
            Y.stride(0), ops._ptr(Y2), Y2.stride(0) if Y2 is not None else 0, ops._ptr(yh), ops._ptr(yl),
            yh.stride(0) if yh is not None else 0, 1 if planes_with_dyn else 0, ops._stream(Y))


def _plain_outputs(L, M):
    Y = torch.empty((M, L.split), device=DEV)
    Y2 = torch.empty((M, L.N - L.split), device=DEV) if L.y2 else None
    yp = None
    if L.planes:
        yp = tuple(torch.empty((M, _pad8(L.split)), dtype=torch.float16, device=DEV) for _ in range(2))
    return Y, Y2, yp


def _run_plain(L, ap, bp, M, c, E=None):
    Y, Y2, yp = _plain_outputs(L, M)
    assert _launch(L, ap, bp, M, c, Y, Y2, yp, E=E) == OK
    return [Y, Y2] + ([p[:, :L.split] for p in yp] if yp is not None else [])


def _equal_bits(a, b):
    return a is None and b is None or torch.equal(_bits(a.contiguous()), _bits(b.contiguous()))


def _nan_padded(planes, rows, cols):
    """The same operand planes with fp16 NaN in every column >= cols (a whole extra K block of them) and GUARD rows
    of NaN past rows."""
    out = []
    for p in planes:
        q = torch.empty((rows + GUARD, _pad8(cols) + 64), dtype=torch.float16, device=DEV)
        _bits(q).fill_(NAN16)
        q[:rows, :cols] = p[:rows, :cols]
        out.append(q)
    return tuple(out)


@pytest.mark.parametrize("layout", ["paired", "scalar"])
@pytest.mark.parametrize("size", LAYER_SIZES)
@pytest.mark.parametrize("name", [l.name for l in LAYERS])
def test_layer_matches_fp64_and_writes_only_its_outputs(name, size, layout):
    L = BY_NAME[name]
    M = _rows(size, L.N)
    _assert_waves(size, M, L.N)
    c = _layer_inputs(L, M, seed=100 * LAYERS.index(L) + LAYER_SIZES.index(size))
    # "paired": float2 / u32 stores; "scalar": odd row strides and bases one element past alignment (scalar fallback)
    odd = layout == "scalar"
    def ld(cols):
        return (cols + 7) | 1 if odd else _pad8(cols) + 8
    Y = Guarded(M, L.split, torch.float32, ld(L.split), offset=1 if odd else 0)
    Y2 = Guarded(M, L.N - L.split, torch.float32, ld(L.N - L.split), offset=1 if odd else 0) if L.y2 else None
    # plane guard columns reach past 512: sdf.fwd3 writes columns < 473 of a buffer whose columns 473-511 hold PE planes
    ld_p = _pad8(L.split) + (41 if odd else 40)
    YP = [Guarded(M, L.split, torch.float16, ld_p, offset=1 if odd else 0) for _ in range(2)] if L.planes else None
    st = _launch(L, c["ap"], c["bp"], M, c, Y.view, Y2.view if Y2 else None, (YP[0].view, YP[1].view) if YP else None)
    assert st == OK
    torch.cuda.synchronize()
    for what, buf in [("Y", Y), ("Y2", Y2)] + ([("y_hi", YP[0]), ("y_lo", YP[1])] if YP else []):
        if buf is not None:
            buf.check(f"{name}[{size},{layout}] {what}")
    ref = torch.cat(_reference(L, c), 1)
    ours = torch.cat([Y.view, Y2.view], 1) if L.y2 else Y.view
    e = merr(ours, ref)
    msg = f"{name} M={M} {layout}: |Y-f64| {e:.2e}"
    if L.positive:   # the quantity acc_trunc_gain is fitted to (DESIGN.md section 5c)
        msg += f"  signed relative bias {float(((ours.double() - ref) * ref).sum() / (ref * ref).sum()):+.2e}"
    print(msg)
    assert e < LAYER_BOUND, msg
    if YP:   # the emitted planes are the split of the fp32 output, bit for bit
        hi, lo = ops.split_planes(Y.view, M, L.split, 64.0, scale_dev=c["dyn"] if L.dyn else None)
        assert _equal_bits(YP[0].view, hi[:, :L.split]) and _equal_bits(YP[1].view, lo[:, :L.split])
    if layout == "paired":
        # operand padding is never read: NaN in the planes' columns >= K and rows >= M / N changes no bit
        outs = _run_plain(L, _nan_padded(c["ap"], M, L.K), _nan_padded(c["bp"], L.N, L.K), M, c)
        assert _equal_bits(outs[0], Y.view) and (not L.y2 or _equal_bits(outs[1], Y2.view))
        if YP:
            assert _equal_bits(outs[2][:, :L.split], YP[0].view) and _equal_bits(outs[3][:, :L.split], YP[1].view)


@pytest.mark.parametrize("size", ["3wave+r", "10wave+r"])
@pytest.mark.parametrize("name", [l.name for l in LAYERS])
def test_layer_multi_wave_equals_single_wave_launches(name, size):
    L = BY_NAME[name]
    M = _rows(size, L.N)
    _assert_waves(size, M, L.N)
    wave = _rows("wave", L.N)
    c = _layer_inputs(L, M, seed=7 + len(name))
    full = _run_plain(L, c["ap"], c["bp"], M, c)
    for r0 in range(0, M, wave):      # one tile per CTA in every slice
        r1 = min(M, r0 + wave)
        ap = (c["ap"][0][r0:r1], c["ap"][1][r0:r1])
        part = _run_plain(L, ap, c["bp"], r1 - r0, c, E=c["E"][r0:r1] if c["E"] is not None else None)
        for a, b in zip(full, part):
            assert _equal_bits(a[r0:r1] if a is not None else None, b), f"{name}: rows {r0}..{r1}"
    perm = torch.randperm(M, generator=_gen(3), device=DEV)
    ap = (c["ap"][0][perm].contiguous(), c["ap"][1][perm].contiguous())
    outs = _run_plain(L, ap, c["bp"], M, c, E=c["E"][perm].contiguous() if c["E"] is not None else None)
    for a, b in zip(full, outs):
        assert _equal_bits(a[perm] if a is not None else None, b), f"{name}: permuted batch"


def test_layer_empty_batch_and_host_rejections():
    L = BY_NAME["sdf.bwd8"]
    c = _layer_inputs(L, 256, seed=5)
    Y = Guarded(256, 512, torch.float32, 520)
    YP = [Guarded(256, 512, torch.float16, 520) for _ in range(2)]
    yp = (YP[0].view, YP[1].view)
    assert _launch(L, c["ap"], c["bp"], 0, c, Y.view, yp=yp) == OK       # M = 0: nothing to do, nothing written
    torch.cuda.synchronize()
    for b in [Y] + YP:
        assert bool((_bits(b.buf) == _pattern(b.buf.dtype)).all())
    assert _launch(L, c["ap"], c["bp"], 256, c, Y.view, yp=yp, mode=3) == E_DTYPE                 # unknown mode
    assert _launch(L, c["ap"], c["bp"], 256, c, Y.view, yp=yp, a_has_dyn=False, planes_with_dyn=True) == E_UNSUPPORTED
    odd_base = tuple(torch.zeros((256, 272), dtype=torch.float16, device=DEV)[:, 1:] for _ in range(2))
    assert _launch(L, odd_base, c["bp"], 256, c, Y.view, yp=yp) == E_SHAPE                         # base not 16-byte aligned
    odd_ld = tuple(torch.as_strided(torch.zeros((256 * 268,), dtype=torch.float16, device=DEV), (256, 257), (268, 1))
                   for _ in range(2))
    assert _launch(L, odd_ld, c["bp"], 256, c, Y.view, yp=yp) == E_SHAPE                           # ldp % 8 != 0
    torch.cuda.synchronize()
    for b in [Y] + YP:      # the refused launches wrote nothing
        assert bool((_bits(b.buf) == _pattern(b.buf.dtype)).all())


# ---------------------------------------------------------------------------------------------------------------------
# the weight gradient and the column sums
# ---------------------------------------------------------------------------------------------------------------------
WG_SHAPES = [(512, 39), (512, 512), (473, 512), (257, 512), (3, 512), (512, 167), (512, 289)]
WG_SIZES = ["1", "63", "64", "65", "clamped", "32/split", "33/split", "31/split", "131072"]


def _wg_plan(out_dim, in_dim, tag):
    """P for a regime, and the splits the host picks for it (recmv_mlp_wgrad_planes: SMs / tiles, at most nkb)."""
    tiles = _tiles_n(out_dim) * _tiles_n(in_dim)
    base = max(1, _sms() // tiles)
    P = {"1": 1, "63": 63, "64": 64, "65": 65, "clamped": 64 * (base - 1) - 21, "32/split": 64 * 32 * base,
         "33/split": 64 * 33 * base - 13, "31/split": 64 * 31 * base - 13, "131072": 131072}[tag]
    nkb = (P + 63) // 64
    splits = min(base, nkb)
    blocks = [nkb * (s + 1) // splits - nkb * s // splits for s in range(splits)]
    if tag == "clamped":
        assert base >= 2 and splits == nkb < base
    elif tag.endswith("/split"):
        assert splits == base and set(blocks) == {int(tag.split("/")[0])}      # 32: one whole chunk; 31 / 33 around it
    return P, splits


def _wg_inputs(P, out_dim, in_dim, seed):
    g = _gen(seed)
    G = _cotangents((P, out_dim), g, 1e-3)
    X = torch.rand((P, in_dim), generator=g, device=DEV) * 0.3
    dyn = ops.grad_dyn_scale(G)
    return G, X, dyn, ops.split_planes(G, P, out_dim, 64.0, scale_dev=dyn), ops.split_planes(X, P, in_dim, 64.0)


def _wgrad_c(gp, xp, P, out_dim, in_dim, scale, dyn, dW, db):
    ws, _ = ops._wgrad_workspace(torch.device(DEV))
    with torch.cuda.device(DEV):
        return _lib.load().recmv_mlp_wgrad_planes(ops._ptr(gp[0]), ops._ptr(gp[1]), gp[0].stride(0), ops._ptr(xp[0]),
                                                  ops._ptr(xp[1]), xp[0].stride(0), int(P), out_dim, in_dim, float(scale),
                                                  ops._ptr(dyn), ops._ptr(ws), ops._ptr(dW), ops._ptr(db), ops._stream(dW))


@pytest.mark.parametrize("size", WG_SIZES)
@pytest.mark.parametrize("out_dim,in_dim", WG_SHAPES)
def test_wgrad_matches_fp64_at_every_split_regime(out_dim, in_dim, size):
    P, splits = _wg_plan(out_dim, in_dim, size)
    G, X, dyn, gp, xp = _wg_inputs(P, out_dim, in_dim, seed=out_dim + in_dim + P % 101)
    dW, db = ops.mlp_wgrad_planes(gp, xp, P, out_dim, in_dim, 0.5, dyn, want_bias=True)
    ref = 0.5 * G.double().T @ X.double()
    ref_b = G.double().sum(0)
    e, eb, ec = merr(dW, ref), merr(db, ref_b), merr(ops.colsum(G, out_dim), ref_b)
    print(f"wgrad {out_dim}x{in_dim} P={P} splits={splits}: dW {e:.2e}  db {eb:.2e}  colsum {ec:.2e}")
    bound = WG_BOUND if P <= 10000 else (WG_BOUND_NARROW if out_dim < 16 else WG_BOUND_LARGE)
    assert e < bound and eb < DB_BOUND and ec < COLSUM_BOUND
    dW2, db2 = ops.mlp_wgrad_planes(gp, xp, P, out_dim, in_dim, 0.5, dyn, want_bias=True)
    assert torch.equal(dW2, dW) and torch.equal(db2, db)                                   # deterministic
    # NaN in the planes' columns >= out_dim / in_dim and rows >= P changes no bit
    dW3, db3 = ops.mlp_wgrad_planes(_nan_padded(gp, P, out_dim), _nan_padded(xp, P, in_dim), P, out_dim, in_dim, 0.5, dyn,
                                    want_bias=True)
    assert torch.equal(dW3, dW) and torch.equal(db3, db)
    # through the C entry into NaN-guarded outputs: exactly out_dim x in_dim and out_dim elements written
    bw = torch.empty((2 * GUARD + out_dim * in_dim,), device=DEV)
    bb = torch.empty((2 * GUARD + out_dim,), device=DEV)
    _bits(bw).fill_(NAN32)
    _bits(bb).fill_(NAN32)
    assert _wgrad_c(gp, xp, P, out_dim, in_dim, 0.5, dyn, bw[GUARD:GUARD + out_dim * in_dim], bb[GUARD:GUARD + out_dim]) == OK
    torch.cuda.synchronize()
    for b, n in ((bw, out_dim * in_dim), (bb, out_dim)):
        bits = _bits(b)
        assert bool((bits[:GUARD] == NAN32).all()) and bool((bits[GUARD + n:] == NAN32).all())
    assert torch.equal(bw[GUARD:GUARD + out_dim * in_dim].view(out_dim, in_dim), dW) and torch.equal(bb[GUARD:GUARD + out_dim], db)


@pytest.mark.parametrize("out_dim,in_dim", WG_SHAPES)
def test_wgrad_workspace_carries_nothing_between_calls(out_dim, in_dim):
    big = _wg_inputs(131072, out_dim, in_dim, seed=1)
    small = _wg_inputs(65, out_dim, in_dim, seed=2)

    def run(i, P):
        return ops.mlp_wgrad_planes(i[3], i[4], P, out_dim, in_dim, 1.0, i[2], want_bias=True)
    s0 = run(small, 65)
    b1 = run(big, 131072)
    s1 = run(small, 65)
    b2 = run(big, 131072)
    assert all(torch.equal(a, b) for a, b in zip(b1, b2)) and all(torch.equal(a, b) for a, b in zip(s0, s1))


# ---------------------------------------------------------------------------------------------------------------------
# the element-wise plane kernels
# ---------------------------------------------------------------------------------------------------------------------
def _split_ref(v, scale):
    """fp32 v -> the fp16 hi / lo planes of scale * v (round to nearest), scale an fp32 scalar tensor."""
    s = v * scale
    hi = s.half()
    return hi, (s - hi.float()).half()


def _split_c(t, R, C, scale, scale_dev, transpose, hi, lo):
    with torch.cuda.device(DEV):
        return _lib.load().recmv_split_planes(ops._ptr(t), t.stride(0), int(R), int(C), float(scale), ops._ptr(scale_dev),
                                              1 if transpose else 0, ops._ptr(hi), ops._ptr(lo), hi.stride(0), ops._stream(t))


@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("dev_scale", [False, True])
@pytest.mark.parametrize("R,C", [(1, 39), (333, 257), (4099, 473), (70001, 512)])
def test_split_planes_is_bit_exact(R, C, dev_scale, transpose):
    g = _gen(R + C)
    src = torch.randn((R, C + 9), generator=g, device=DEV) * 3.0       # row stride > C
    sd = torch.tensor([0.25 * (1 + dev_scale)], device=DEV) if dev_scale else None
    s = torch.tensor(64.0, device=DEV) * (sd[0] if sd is not None else 1.0)
    rows, cols = (C, R) if transpose else (R, C)
    ld = _pad8(cols) + 8
    hi, lo = Guarded(rows, cols, torch.float16, ld), Guarded(rows, cols, torch.float16, ld)
    assert _split_c(src, R, C, 64.0, sd, transpose, hi.view, lo.view) == OK
    torch.cuda.synchronize()
    hi.check("hi")
    lo.check("lo")
    rh, rl = _split_ref(src[:, :C], s)
    if transpose:
        rh, rl = rh.T, rl.T
    assert _equal_bits(hi.view, rh) and _equal_bits(lo.view, rl)


@pytest.mark.parametrize("P", [1, 129, 70001])
def test_pe_forward_planes_matches_pe_forward_and_writes_only_its_columns(P):
    g = _gen(P)
    x = (torch.rand((P, 3), generator=g, device=DEV) * 2.4 - 1.2).contiguous()
    pe_w = [1.0, 1.0, 0.9, 0.8, 0.6, 0.5, 0.3, 0.2, 0.1, 0.05, 0.0, 0.0]
    ref = torch.zeros((P, 40), device=DEV)
    ops.pe_forward(x, pe_w, 6, ref)
    s = torch.tensor(64.0, device=DEV)
    for width, col in ((64, 0), (512, 473)):      # layer 0's input, and the PE slice of layer 4's input
        out = Guarded(P, width, torch.float32, width)
        planes = [Guarded(P, width, torch.float16, width) for _ in range(2)]
        ops.pe_forward_planes(x, pe_w, 6, out.view[:, col:], planes[0].view[:, col:], planes[1].view[:, col:])
        torch.cuda.synchronize()
        for b in [out] + planes:
            bits = _bits(b.buf)
            written = torch.zeros_like(b.mask)
            written[GUARD:GUARD + P, col:col + 39] = True
            assert bool((bits[~written] == _pattern(b.buf.dtype)).all())         # columns >= 39 of the slice untouched
        got = out.view[:, col:col + 39]
        assert _equal_bits(got, ref[:, :39])                                      # the same sincosf arithmetic
        rh, rl = _split_ref(got, s)
        assert _equal_bits(planes[0].view[:, col:col + 39], rh) and _equal_bits(planes[1].view[:, col:col + 39], rl)


@pytest.mark.parametrize("R,C", [(1, 512), (333, 473), (70001, 512)])
def test_softplus_tangent_planes_matches_fp64(R, C):
    g = _gen(R + 1)
    ld = 520
    tz = torch.randn((R, ld), generator=g, device=DEV) * 0.3
    a = _softplus_acts((R, ld), g)
    h = _cotangents((R, ld), g)
    u = Guarded(R, C, torch.float32, ld)
    inj = Guarded(R, C, torch.float32, ld)
    planes = [Guarded(R, C, torch.float16, ld) for _ in range(2)]
    ops.softplus_tangent_planes(tz, a, h, C, u.view, (planes[0].view, planes[1].view), inj.view)
    torch.cuda.synchronize()
    for b in [u, inj] + planes:
        b.check("softplus_tangent")
    t64, a64, h64 = tz[:, :C].double(), a[:, :C].double(), h[:, :C].double()
    u_ref = (1 - torch.exp(-100 * a64)) * t64
    inj_ref = 100 * torch.exp(-100 * a64) * h64 * t64
    eu, ei = merr(u.view, u_ref), merr(inj.view, inj_ref)
    print(f"softplus_tangent R={R} C={C}: u {eu:.2e}  inj {ei:.2e}")
    assert eu < TANGENT_BOUND and ei < TANGENT_BOUND
    rh, rl = _split_ref(u.view, torch.tensor(64.0, device=DEV))
    assert _equal_bits(planes[0].view, rh) and _equal_bits(planes[1].view, rl)


@pytest.mark.parametrize("dev_scale", [False, True])
@pytest.mark.parametrize("R,C", [(1, 512), (333, 473), (70001, 512)])
def test_add_split_planes_matches_fp64(R, C, dev_scale):
    g = _gen(R + 2)
    ld = 520
    y0 = _cotangents((R, C), g)
    add = _cotangents((R, ld), g)
    y = Guarded(R, C, torch.float32, ld)
    y.view.copy_(y0)
    planes = [Guarded(R, C, torch.float16, ld) for _ in range(2)]
    sd = ops.grad_dyn_scale(y0) if dev_scale else None
    ops.add_split_planes(y.view, add, C, (planes[0].view, planes[1].view), 64.0, sd)
    torch.cuda.synchronize()
    for b in [y] + planes:
        b.check("add_split")
    # the sum of two fp32 numbers is exact in float64, so its fp32 rounding is THE correctly rounded result
    assert _equal_bits(y.view, (y0.double() + add[:, :C].double()).float())
    rh, rl = _split_ref(y.view, torch.tensor(64.0, device=DEV) * (sd[0] if sd is not None else 1.0))
    assert _equal_bits(planes[0].view, rh) and _equal_bits(planes[1].view, rl)


@pytest.mark.parametrize("kernel", ["layer", "split", "softplus_tangent", "add_split"])
def test_fp16_range_is_reported_by_every_splitting_kernel(kernel):
    """One operand whose scaled value is >= 65504: the hi plane saturates, the fp32 output is unaffected, the status record
    says "range" with the kernel's tag, and layer launches are refused until the record is cleared."""
    ops.check_async_errors()
    g = _gen(11)
    R, C = 300, 64
    big = 2000.0     # 64 x 2000 = 128 000 > 65504
    hi, lo = (torch.zeros((R, C), dtype=torch.float16, device=DEV) for _ in range(2))
    if kernel == "layer":
        tag = 3500
        L = Layer("range", 4, 64, C)
        c = _layer_inputs(L, R, seed=3)
        c["bias"] = torch.zeros((C,), device=DEV)
        c["bias"][5] = big
        out = torch.empty((R, C), device=DEV)
        assert _launch(L, c["ap"], c["bp"], R, c, out, yp=(hi, lo)) == OK
        torch.cuda.synchronize()
        clean = torch.empty((R, C), device=DEV)
        pending = _launch(L, c["ap"], c["bp"], R, c, clean)       # made before the clear: refused
        assert bool((out[:, 5] > 1000).all())
    elif kernel == "split":
        tag = 3600
        t = torch.randn((R, C), generator=g, device=DEV)
        t[7, 5] = big
        assert _split_c(t, R, C, 64.0, None, False, hi, lo) == OK
    elif kernel == "softplus_tangent":
        tag = 3700
        tz = torch.randn((R, C), generator=g, device=DEV)
        tz[7, 5] = big
        a = torch.full((R, C), 0.5, device=DEV)       # softplus' = 1 - exp(-50): u = tz
        out, inj = torch.empty((R, C), device=DEV), torch.empty((R, C), device=DEV)
        ops.softplus_tangent_planes(tz, a, torch.ones_like(tz), C, out, (hi, lo), inj)
        assert float(out[7, 5]) == big
    else:
        tag = 3710
        out = torch.zeros((R, C), device=DEV)
        add = torch.randn((R, C), generator=g, device=DEV)
        add[7, 5] = big
        ops.add_split_planes(out, add, C, (hi, lo), 64.0)
        assert torch.equal(out, add)
    torch.cuda.synchronize()
    h = _bits(hi)
    r = slice(None) if kernel == "layer" else 7
    assert bool((h[r, 5] == F16_MAX).all())                          # saturated, not inf
    assert not bool(torch.isinf(hi).any() or torch.isnan(hi).any() or torch.isnan(lo).any())
    if kernel == "layer":
        assert pending == E_DEVICE
    else:   # a layer launch made before the clear is refused
        L = Layer("probe", 4, 64, 64)
        c = _layer_inputs(L, 16, seed=4)
        assert _launch(L, c["ap"], c["bp"], 16, c, torch.empty((16, 64), device=DEV)) == E_DEVICE
    with pytest.raises(_lib.RecmvError, match=f"range.*tag={tag}"):
        ops.check_async_errors(clear=True)
    ops.check_async_errors()                                        # reported once, then cleared
    L = Layer("probe", 4, 64, 64)
    c = _layer_inputs(L, 16, seed=4)
    Y = torch.empty((16, 64), device=DEV)
    assert _launch(L, c["ap"], c["bp"], 16, c, Y) == OK              # after the clear: runs
    if kernel == "layer":   # the fp32 output does not depend on whether (or how) planes were written
        L = Layer("range", 4, 64, C)
        c = _layer_inputs(L, R, seed=3)
        c["bias"] = torch.zeros((C,), device=DEV)
        c["bias"][5] = big
        assert _launch(L, c["ap"], c["bp"], R, c, clean) == OK
        torch.cuda.synchronize()
        assert torch.equal(clean, out)
        ops.check_async_errors()


# ---------------------------------------------------------------------------------------------------------------------
# the training steps end to end at multi-wave sizes
# ---------------------------------------------------------------------------------------------------------------------
def _sdf_params(seed=0):
    net = testing.build_sdf(getTmpSdf, seed=seed, perturb_seed=101).to(DEV)
    with torch.no_grad():
        Ws, bs = net.effective_weights()
        Ws = [w.detach().float().contiguous() for w in Ws]
        bs = [b.detach().float().contiguous() for b in bs]
    return net, Ws, bs


def _points(P, seed):
    return (torch.rand((P, 3), generator=_gen(seed), device=DEV) * 1.2 - 0.6).contiguous()


@pytest.mark.parametrize("size", ["3wave+r", "131072"])
def test_sdf_training_step_matches_fp64_autograd(size):
    P = 131072 if size == "131072" else _rows(size, 512)
    _assert_waves(size, P, 512)
    _, Ws, bs = _sdf_params()
    pe_w = ratio_to_weights(6, 0.7)
    x0 = _points(P, 1)
    g = _gen(2)
    mag = torch.exp(torch.randn((P, 1), generator=g, device=DEV)) / P
    c0 = torch.randn((P, 1), generator=g, device=DEV) * mag
    c1 = torch.randn((P, 256), generator=g, device=DEV) * mag * 0.1
    x = x0.clone().requires_grad_(True)
    Wl = [w.clone().requires_grad_(True) for w in Ws]
    bl = [b.clone().requires_grad_(True) for b in bs]
    sdf, feat = ops.SdfMlpTrainFunction.apply(x, pe_w, ops.DEFAULT_MLP_MODE, None, *Wl, *bl)
    ((sdf * c0).sum() + (feat * c1).sum()).backward()
    assert ops.SdfMlpTrainFunction.last_backward == "fused-tc"
    xd = x0.double().requires_grad_(True)
    Wd = [w.double().requires_grad_(True) for w in Ws]
    bd = [b.double().requires_grad_(True) for b in bs]
    s64, f64 = ops._sdf_composite(xd, Wd, bd, pe_w)
    ((s64 * c0.double()).sum() + (f64 * c1.double()).sum()).backward()
    errs = {"sdf": merr(sdf, s64), "feat": merr(feat, f64), "dx": merr(x.grad, xd.grad)}
    errs.update({f"W{l}": merr(Wl[l].grad, Wd[l].grad) for l in range(9)})
    errs.update({f"b{l}": merr(bl[l].grad, bd[l].grad) for l in range(9)})
    print(f"SDF step P={P}: " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    assert max(errs.values()) < SDF_STEP_BOUND, errs


def test_sdf_forward_multi_wave_equals_single_wave_launches():
    P = _rows("10wave+r", 512)
    _assert_waves("10wave+r", P, 512)
    wave = _rows("wave", 512)
    _, Ws, bs = _sdf_params()
    pe_w = ratio_to_weights(6, 0.7)
    x = _points(P, 3)
    with torch.no_grad():
        sdf, feat = ops.SdfMlpTrainFunction.apply(x, pe_w, ops.DEFAULT_MLP_MODE, None, *Ws, *bs)
        for r0 in range(0, P, wave):
            r1 = min(P, r0 + wave)
            s, f = ops.SdfMlpTrainFunction.apply(x[r0:r1].contiguous(), pe_w, ops.DEFAULT_MLP_MODE, None, *Ws, *bs)
            assert _equal_bits(sdf[r0:r1], s) and _equal_bits(feat[r0:r1], f), (r0, r1)


PLAIN_NETS = {"translator": (167, 3), "colour": (289, 3)}


def _plain_net(net):
    """A ReLU network (d_in -> 512 x4 -> d_out) at 3wave+r rows: (Ws, bs, X0 [P, d_in padded to 8], output cotangent)."""
    d_in, d_out = PLAIN_NETS[net]
    P = _rows("3wave+r", 512)
    _assert_waves("3wave+r", P, 512)
    g = _gen(d_in)
    dims = [d_in, 512, 512, 512, 512, d_out]
    Ws = [torch.randn((dims[l + 1], dims[l]), generator=g, device=DEV) * (2.0 / dims[l]) ** 0.5 for l in range(5)]
    bs = [torch.randn((dims[l + 1],), generator=g, device=DEV) * 0.05 for l in range(5)]
    X0 = torch.zeros((P, _pad8(d_in)), device=DEV)
    X0[:, :d_in] = torch.randn((P, d_in), generator=g, device=DEV) * 0.5
    cot = torch.randn((P, d_out), generator=g, device=DEV) / P
    return Ws, bs, X0, cot


def _plain_f64_given_our_masks(Xd, Wd, bd, acts):
    """The network in float64 with OUR ReLU masks (acts[l + 1] > 0) -> (output, mask flips against float64's own masks,
    flips at |z| > 5e-6).  The masks may differ from float64's only where |z| is at fp32 rounding level."""
    h, flips, amb = Xd, 0, 0
    for l in range(5):
        z = torch.nn.functional.linear(h, Wd[l], bd[l])
        if l < 4:
            ours = acts[l + 1] > 0
            diff = ours != (z > 0)
            flips += int(diff.sum())
            amb += int((diff & (z.abs() > 5e-6)).sum())
            h = z * ours.double()
        else:
            h = z
    return h, flips, amb


@pytest.mark.parametrize("net", list(PLAIN_NETS))
def test_relu_mlp_training_step_matches_fp64_given_our_masks(net):
    """Translator (167 -> 512 x4 -> 3) and colour (289 -> 512 x4 -> 3) networks on the plane GEMMs, through the forward and
    backward the training Functions run (ops._plain_mlp_forward / _plain_mlp_backward)."""
    d_in = PLAIN_NETS[net][0]
    Ws, bs, X0, cot = _plain_net(net)
    P = X0.shape[0]
    out, acts, xplanes = ops._plain_mlp_forward(X0, Ws, bs)
    dX0, dW, db = ops._plain_mlp_backward(cot.contiguous(), Ws, acts, True, True, xplanes)
    Xd = X0[:, :d_in].double().requires_grad_(True)
    Wd = [w.double().requires_grad_(True) for w in Ws]
    bd = [b.double().requires_grad_(True) for b in bs]
    h, flips, amb = _plain_f64_given_our_masks(Xd, Wd, bd, acts)
    assert amb == 0, (flips, amb)
    (h * cot.double()).sum().backward()
    errs = {"out": merr(out, h), "dX0": merr(dX0[:, :d_in], Xd.grad)}
    errs.update({f"W{l}": merr(dW[l], Wd[l].grad) for l in range(5)})
    errs.update({f"b{l}": merr(db[l], bd[l].grad) for l in range(5)})
    print(f"{net} step P={P}: {flips} mask flips (all at |z| < 5e-6); " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    assert max(errs.values()) < PLAIN_STEP_BOUND, errs


@pytest.mark.parametrize("net", list(PLAIN_NETS))
def test_relu_mlp_create_graph_input_grad_matches_fp64_given_our_masks(net):
    """second_order.PlainMlpInputGradFunction, the create_graph input gradient of the translator and colour networks: its
    forward is the first-order chain's dX0 bit for bit, and with the ReLU masks of the saved activations dX0 is linear in
    g_out and in each weight, so the gradients its backward returns must match float64 double autograd under those masks."""
    from recmv_b200 import second_order
    d_in = PLAIN_NETS[net][0]
    Ws, bs, X0, cot = _plain_net(net)
    P = X0.shape[0]
    _, acts, xplanes = ops._plain_mlp_forward(X0, Ws, bs)
    first, _, _ = ops._plain_mlp_backward(cot.contiguous(), Ws, acts, False, True, xplanes)
    q = _cotangents((P, d_in), _gen(d_in + 1), 1.0)
    cot_t = cot.clone().requires_grad_(True)
    Wl = [w.clone().requires_grad_(True) for w in Ws]
    dX0 = second_order.PlainMlpInputGradFunction.apply(cot_t, 5, *acts, *Wl)
    assert _equal_bits(dX0, first[:, :d_in])
    (dX0 * q).sum().backward()
    Xd = X0[:, :d_in].double().requires_grad_(True)
    Wd = [w.double().requires_grad_(True) for w in Ws]
    cd = cot.double().requires_grad_(True)
    h, _, _ = _plain_f64_given_our_masks(Xd, Wd, [b.double() for b in bs], acts)
    (dX64,) = torch.autograd.grad(h, Xd, cd, create_graph=True)
    (dX64 * q.double()).sum().backward()
    errs = {"dX0": merr(dX0, dX64), "g_out": merr(cot_t.grad, cd.grad)}
    errs.update({f"W{l}": merr(Wl[l].grad, Wd[l].grad) for l in range(5)})
    print(f"{net} create_graph input gradient P={P}: " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    assert max(errs.values()) < PLAIN_STEP_BOUND, errs


def test_eikonal_term_matches_fp64_double_backward():
    P = _rows("3wave+r", 512)
    _assert_waves("3wave+r", P, 512)
    net, _, _ = _sdf_params()
    x = _points(P, 4)
    xg = x.clone()
    gr = net.gradient(xg)
    assert net.last_path == "fused-train"
    assert ops.SdfMlpTrainFunction.last_backward == "fused-tc (create_graph, input gradient)"
    loss = ((gr.norm(dim=1) - 1) ** 2).mean()
    loss.backward()
    # float64: the same weight-normed network as a torch graph, differentiated twice
    params = {n: p.detach().double().requires_grad_(True) for n, p in net.named_parameters()}
    Wd, bd = [], []
    for l in range(9):
        gl, vl = params[f"lin{l}.weight_g"], params[f"lin{l}.weight_v"]
        Wd.append(gl * vl / vl.norm(dim=1, keepdim=True))
        bd.append(params[f"lin{l}.bias"])
    xd = x.double().requires_grad_(True)
    s64, _ = ops._sdf_composite(xd, Wd, bd, net._pe_weights(None))
    g64 = torch.autograd.grad(s64.sum(), xd, create_graph=True)[0]
    loss64 = ((g64.norm(dim=1) - 1) ** 2).mean()
    loss64.backward()
    errs = {"loss": abs(float(loss) - float(loss64)) / float(loss64), "gradient": merr(gr, g64), "dx": merr(xg.grad, xd.grad)}
    for n, p in net.named_parameters():
        if n == "lin8.bias":      # the input gradient does not depend on the last bias
            assert p.grad is None
            continue
        errs[n] = merr(p.grad, params[n].grad)
    print(f"eikonal P={P}: " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    assert max(errs.values()) < EIKONAL_BOUND, errs
