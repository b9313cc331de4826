"""Without a feature output the fused SDF kernel computes only the last layer's first 128-column tile (the sdf column).
The sdf, and in the forward-mode launch its gradient, must be bit-identical to a launch that also writes the features:
the same MMAs, in the same order, produce column 0 in both."""
import pytest
import torch

from recmv_b200 import _lib, ops, testing
from recmv_b200.model import getTmpSdf

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MODES = [("tc3", _lib.MLP_TC_F16X3), ("tc1", _lib.MLP_TC_F16X1)]
SIZES = [1, 64, 77, 5000]   # one tile, exactly one tile, a ragged tile count, many tiles


@pytest.fixture(scope="module")
def packed():
    net = testing.build_sdf(getTmpSdf, seed=0, perturb_seed=101).to(DEV)
    return net.packed_weights()


def _points(P):
    g = torch.Generator(device="cpu").manual_seed(P)
    return (torch.rand((P, 3), generator=g) * 1.6 - 0.8).to(DEV)


@pytest.mark.parametrize("name,mode", MODES)
@pytest.mark.parametrize("P", SIZES)
def test_sdf_without_features_is_bit_identical(packed, name, mode, P):
    x = _points(P)
    sdf_f, feat = ops.sdf_mlp_forward(x, packed, None, mode, want_feat=True)
    sdf_n, none = ops.sdf_mlp_forward(x, packed, None, mode, want_feat=False)
    torch.cuda.synchronize()
    ops.check_async_errors()
    assert none is None and feat.shape == (P, 256)
    assert torch.equal(sdf_f, sdf_n)


@pytest.mark.parametrize("name,mode", MODES)
@pytest.mark.parametrize("P", SIZES)
def test_value_and_gradient_without_features_is_bit_identical(packed, name, mode, P):
    x = _points(P)
    sdf_f, grad_f, feat = ops.sdf_value_and_grad(x, packed, None, mode, want_feat=True)
    sdf_n, grad_n, none = ops.sdf_value_and_grad(x, packed, None, mode, want_feat=False)
    torch.cuda.synchronize()
    ops.check_async_errors()
    assert none is None and feat.shape == (P, 256)
    assert torch.equal(sdf_f, sdf_n) and torch.equal(grad_f, grad_n)
