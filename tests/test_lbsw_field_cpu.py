"""CPU checks of the skinning-voxel construction: the oracle's restatement against the reference's own
compute_lbswField (tests/golden/lbsw_ref.npz), argument validation of the two C entries before any CUDA call, and the
mirrors' refusal of CPU tensors."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(HERE, "golden"))

from make_golden_lbsw import CASES  # noqa: E402
from oracle import lbsw_torch as lt  # noqa: E402
from recmv_b200 import _lib, synth  # noqa: E402

G = np.load(os.path.join(HERE, "golden", "lbsw_ref.npz"))


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_reproduces_reference(name):
    variant, res, ac, k, times = CASES[name]
    ref = torch.from_numpy(G[name])
    args = (G["bmin"].tolist(), G["bmax"].tolist(), res, torch.from_numpy(G["verts"]), torch.from_numpy(G["vert_ws"]),
            ac, k, times, 5e-3 if variant == "utils" else 0.0)
    f32 = lt.compute_lbswField(*args, dtype=torch.float32)
    # same operations in the same order on CPU: measured bit-identical; the bound leaves room for another CPU's
    # vector paths in norm / sum
    assert (f32 - ref).abs().max().item() <= 1e-6
    f64 = lt.compute_lbswField(*args, dtype=torch.float64)
    # fp32 rounding of the reference itself: measured 1.5e-7 (smoothed) and 8.5e-7 (times = 0)
    assert (f64 - ref.double()).abs().max().item() < 3e-6


def test_body_points_reproducible_and_sparse():
    v, w = synth.body_points()
    v2, w2 = synth.body_points()
    assert v.shape == (6890, 3) and w.shape == (6890, 24) and v.dtype == w.dtype == torch.float32
    assert torch.equal(v, v2) and torch.equal(w, w2)
    assert not torch.equal(v, synth.body_points(seed=6)[0])
    assert torch.allclose(w.sum(1), torch.ones(6890), atol=1e-6)
    assert ((w > 0).sum(1) <= 3).all()


def test_argument_errors_without_gpu():
    lib = _lib.load()
    lo, hi = (ctypes.c_float * 3)(-1, -1, -1), (ctypes.c_float * 3)(1, 1, 1)
    p = ctypes.c_void_p(16)   # never dereferenced: every call below fails validation first

    def knn(V=100, C=24, W=4, H=4, D=4, ac=0, k=5, verts=p, out=p):
        return lib.recmv_lbsw_knn_blend(verts, p, V, C, lo, hi, W, H, D, ac, k, out, None, None)
    assert knn(verts=None) == -1 and knn(out=None) == -1
    assert knn(C=23) == -3 and knn(V=0) == -3 and knn(W=0) == -3 and knn(D=-1) == -3
    assert knn(k=0) == -3 and knn(V=4, k=5) == -3
    assert knn(k=33) == -4 and knn(V=20000) == -4
    assert knn(ac=1, H=1) == -3

    def smooth(a=p, b=ctypes.c_void_p(32), D=4, H=4, W=4, times=3, ncdhw=p, cl=ctypes.c_void_p(48)):
        return lib.recmv_lbsw_smooth(a, b, D, H, W, times, 0.0, ncdhw, cl, None)
    assert smooth(a=None) == -1 and smooth(ncdhw=None) == -1 and smooth(cl=None) == -1 and smooth(b=None) == -1
    assert smooth(D=0) == -3 and smooth(times=-1) == -3
    assert smooth(cl=p) == -3 and smooth(b=p) == -3                       # aliased buffers
    assert smooth(a=ctypes.c_void_p(20)) == -3                            # not 16-byte aligned


def test_mirrors_reject_cpu_tensors():
    from recmv_b200 import utils
    from recmv_b200.model import Deformer, initialLBSkinner  # noqa: F401  (exported like the reference's model package)
    v, w = synth.body_points(200)
    for fn in (Deformer.compute_lbswField, utils.compute_lbswField):
        with pytest.raises(RuntimeError):
            fn([-1, -1, -1], [1, 1, 1], (4, 4, 4), v, w)
    for fn in (Deformer.smooth_weights, utils.smooth_weights):
        with pytest.raises(RuntimeError):
            fn(torch.rand(1, 24, 4, 4, 4), 2)
    Js, parents, init = synth.skeleton()
    with pytest.raises(RuntimeError):
        Deformer.skinner_from_body(v, w, Js, parents, init, (4, 4, 4))
