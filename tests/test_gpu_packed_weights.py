"""GPU: the packed weight blob of each fused network (recmv_{sdf,translator,rendernet}_pack_weights) equals a NumPy
restatement byte for byte, and a weight outside the tensor-core operand range is reported, not silent.

The restatement, per network:
  * bias planes: [layers][512] fp32 padded with zeros; the SDF adds a second plane of b * 100 log2(e) (fp32 product);
  * SDF only, per layer: the fp32 transposed copy [in][npad] (npad 264 for the last layer, else 512) of w * s, where
    s = 1/sqrt2 for layer 4 (the skip connection's factor) and 1 otherwise;
  * fp16 panels [2 planes][panels][512][64]: v = fp32(w * s) * 1024, hi = fp16(v), lo = fp16(v - hi).  Layer l's K
    inputs are cut into 64-wide panels placed one after another; SDF layer 0 is one panel of the 39 PE inputs, SDF
    layer 4 is 8 panels of its 473 hidden inputs followed by one panel of its 39 PE inputs (the skip connection);
    everything else is zero."""
import ctypes

import numpy as np
import pytest
import torch

from recmv_b200 import _lib, ops

DEV = "cuda:0"
SOFTPLUS_LOG2 = np.float32(144.26950408889634)
INV_SQRT2 = np.float32(0.70710678118654752440)


def _ranges(net, l, n_in):
    """(panel columns, weight columns) slices of layer l's panel matrix"""
    if net == "sdf" and l == 4:
        return [(slice(0, 473), slice(0, 473)), (slice(512, 551), slice(473, 512))]
    return [(slice(0, n_in), slice(0, n_in))]


# net -> (layer shapes [out, in], panels per layer)
NETS = {
    "sdf": (ops.SDF_LAYER_SHAPES, [1, 8, 8, 8, 9, 8, 8, 8, 8]),
    "translator": (ops.TRANSLATOR_LAYER_SHAPES, [3, 8, 8, 8, 8]),
    "rendernet": (ops.RENDERNET_LAYER_SHAPES, [5, 8, 8, 8, 8]),
}
PACK = {"sdf": ops.sdf_pack_weights, "translator": ops.translator_pack_weights,
        "rendernet": ops.rendernet_pack_weights}
TAG = {"sdf": 1201, "translator": 1200, "rendernet": 1200}


def _restate(net, Ws, bs):
    shapes, nkb = NETS[net]
    L = len(shapes)
    sdf = net == "sdf"
    bias = np.zeros((2 if sdf else 1, L, 512), np.float32)
    panels = np.zeros((2, sum(nkb), 512, 64), np.float16)
    w32 = []
    pbase = 0
    for l, ((n_out, n_in), W, b) in enumerate(zip(shapes, Ws, bs)):
        s = INV_SQRT2 if sdf and l == 4 else np.float32(1)
        Ws_ = W * s
        bias[0, l, :n_out] = b
        if sdf:
            bias[1, l, :n_out] = b * SOFTPLUS_LOG2
            t = np.zeros((n_in, 264 if l == 8 else 512), np.float32)
            t[:, :n_out] = Ws_.T
            w32.append(t)
        m = np.zeros((512, nkb[l] * 64), np.float32)
        for cols, src in _ranges(net, l, n_in):
            m[:n_out, cols] = Ws_[:, src] * np.float32(1024)
        m = np.clip(m, -65504, 65504)
        hi = m.astype(np.float16)
        lo = (m - hi.astype(np.float32)).astype(np.float16)
        for plane, x in enumerate((hi, lo)):
            panels[plane, pbase:pbase + nkb[l]] = x.reshape(512, nkb[l], 64).transpose(1, 0, 2)
        pbase += nkb[l]
    return np.concatenate([bias.reshape(-1).view(np.uint8)] + [t.reshape(-1).view(np.uint8) for t in w32]
                          + [panels.reshape(-1).view(np.uint8)])


def _weights(net, seed):
    rng = np.random.default_rng(seed)
    Ws, bs = [], []
    for n_out, n_in in NETS[net][0]:
        W = (rng.standard_normal((n_out, n_in)) * 0.1).astype(np.float32)
        W.flat[rng.integers(0, W.size, 8)] = rng.uniform(-63.9, 63.9, 8).astype(np.float32)   # large, in range
        W.flat[rng.integers(0, W.size, 8)] = rng.uniform(-1e-6, 1e-6, 8).astype(np.float32)   # lo below fp16 normals
        Ws.append(W)
        bs.append((rng.standard_normal(n_out) * 0.5).astype(np.float32))
    return Ws, bs


def _pack(net, Ws, bs):
    packed = PACK[net]([torch.from_numpy(W).to(DEV) for W in Ws], [torch.from_numpy(b).to(DEV) for b in bs])
    torch.cuda.synchronize()
    return packed.cpu().numpy()


def _status(clear):
    info = (ctypes.c_int * 3)()
    with torch.cuda.device(DEV):
        st = _lib.load().recmv_check_async_errors(info, 1 if clear else 0)
    return st, tuple(info)


@pytest.mark.gpu
@pytest.mark.parametrize("net", list(NETS))
@pytest.mark.parametrize("seed", [0, 1])
def test_packed_blob_equals_numpy_restatement(net, seed):
    Ws, bs = _weights(net, seed)
    got = _pack(net, Ws, bs)
    want = _restate(net, Ws, bs)
    assert got.size == want.size == getattr(_lib.load(), f"recmv_{net}_packed_bytes")()
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} bytes differ, first at {bad[:8]}"
    assert _status(clear=False)[0] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("net", list(NETS))
def test_out_of_range_weight_is_reported_and_saturated(net):
    _status(clear=True)
    Ws, bs = _weights(net, 2)
    layer = len(Ws) - 2
    Ws[layer][1, 2] = 64.0    # 1024 * 64 > 65504
    Ws[layer][3, 4] = -1e9
    got = _pack(net, Ws, bs)
    st, info = _status(clear=True)
    assert st == -6 and info[:2] == (2, TAG[net]), (st, info)
    assert _status(clear=False) == (0, (0, 0, 0))                 # cleared
    assert np.array_equal(got, _restate(net, Ws, bs))             # saturated to +-65504, lo plane 0
