"""CPU: the nearest-neighbour oracle (oracle/knn_oracle.py) -- the float32 restatement against the float64 brute force,
the tie and padding rules, the closed-form backward against autograd, the batched feature-curve loss against the
reference's own `fl_proj_loss` (tests/golden/fl_proj_ref.npz) -- and the argument errors of the new C entries and of
the Python layer without a GPU.  The CUDA kernel is compared with this oracle in tests/test_gpu_knn.py."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import knn_oracle as ko
from recmv_b200 import _lib


@pytest.mark.parametrize("D", [2, 3])
def test_f32_restatement_matches_f64_brute_force(D):
    g = np.random.default_rng(D)
    p1 = g.normal(size=(3, 157, D)).astype(np.float32)
    p2 = g.normal(size=(3, 311, D)).astype(np.float32)
    d32, i32 = ko.nearest_f32(p1, p2)
    d64, i64 = ko.nearest_f64(p1, p2)
    # the neighbours agree wherever float64 separates the best two by more than float32 can resolve
    d = np.sort(((p1[:, :, None].astype(np.float64) - p2[:, None].astype(np.float64)) ** 2).sum(-1), axis=2)
    clear = d[..., 1] - d[..., 0] > 1e-5 * d[..., 1]
    assert clear.mean() > 0.99
    assert np.array_equal(i32[clear], i64[clear])
    assert np.abs(d32 - d64).max() <= 1e-6 * np.abs(d64).max()
    assert d32.dtype == np.float32


def test_exact_ties_go_to_the_lower_index():
    p2 = np.array([[[1, 0, 0], [0, 0, 0], [1, 0, 0], [0, 0, 0], [-1, 0, 0]]], dtype=np.float32)
    p1 = np.array([[[0, 0, 0], [1, 0, 0], [0.5, 0, 0], [-0.5, 0, 0], [0, 5, 0]]], dtype=np.float32)
    for fn in (ko.nearest_f32, ko.nearest_f64):
        d, i = fn(p1, p2)
        # 0.5 is equidistant from x = 0 (index 1) and x = 1 (index 0): index 0; -0.5 ties 1 and 4: index 1
        assert i.tolist() == [[1, 0, 0, 1, 1]], fn
        assert np.allclose(d, [[0, 0, 0.25, 0.25, 25]])


def test_padding_rules():
    g = np.random.default_rng(3)
    p1 = g.normal(size=(4, 20, 2)).astype(np.float32)
    p2 = g.normal(size=(4, 30, 2)).astype(np.float32)
    l1, l2 = np.array([20, 0, 7, 1]), np.array([30, 5, 0, 1])
    for fn in (ko.nearest_f32, ko.nearest_f64):
        d, i = fn(p1, p2, l1, l2)
        assert np.all(i[1] == -1) and np.all(d[1] == 0)             # no query
        assert np.all(i[2] == -1) and np.all(d[2] == 0)             # empty candidate cloud
        assert np.all(i[3, 1:] == -1) and i[3, 0] == 0              # one query, one candidate
        assert np.all(i[0] < 30) and np.all(i[0] >= 0)
        full_d, full_i = fn(p1[:1], p2[:1, :30])
        assert np.array_equal(i[:1], full_i)


def test_closed_form_backward_matches_autograd():
    g = np.random.default_rng(5)
    p1 = torch.tensor(g.normal(size=(2, 40, 3)), requires_grad=True)
    p2 = torch.tensor(g.normal(size=(2, 9, 3)), requires_grad=True)
    w = torch.tensor(g.normal(size=(2, 40)))
    _, idx = ko.nearest_f64(p1.detach().numpy(), p2.detach().numpy(), [40, 31], [9, 9])
    it = torch.tensor(idx)
    ok = it >= 0
    nn = torch.gather(p2, 1, it.clamp_min(0)[..., None].expand(-1, -1, 3))
    ((((p1 - nn) ** 2).sum(-1) * w)[ok]).sum().backward()
    dp1, dp2 = ko.nearest_backward_f64(p1.detach().numpy(), p2.detach().numpy(), idx, w.numpy())
    assert np.abs(dp1 - p1.grad.numpy()).max() < 1e-12
    assert np.abs(dp2 - p2.grad.numpy()).max() < 1e-12


def _fixture(golden):
    z = golden("fl_proj_ref.npz")
    C = len(z["weights"])
    pts = [torch.tensor(z[f"pts_{c}"], dtype=torch.float64, requires_grad=True) for c in range(C)]
    gts = [torch.tensor(z[f"gt_{c}"]) for c in range(C)]
    masks = [torch.tensor(z[f"mask_{c}"])[..., None].expand(-1, -1, 3) for c in range(C)]
    return z, pts, gts, masks


def test_fixture_covers_the_edge_cases(golden):
    z, pts, gts, masks = _fixture(golden)
    m = [z[f"mask_{c}"] for c in range(len(z["weights"]))]
    assert len(m) == 6 and pts[0].shape[0] == 3 and gts[0].shape[1] == 100
    assert not m[0][1].any() and not m[3].any()                         # an empty frame, an invisible curve
    assert len({p.shape[1] for p in pts}) > 1                           # curves of unequal length
    assert len({int(x.sum()) for x in m[0]}) > 1                        # unequal visible counts


def test_batched_oracle_equals_the_reference_fl_proj_loss(golden):
    z, pts, gts, masks = _fixture(golden)
    loss = ko.fl_proj_f64(pts, gts, masks, list(z["weights"]))
    grads = torch.autograd.grad(loss, pts)
    assert abs(loss.item() - float(z["loss"])) <= 1e-12 * abs(float(z["loss"]))
    for c, gr in enumerate(grads):
        assert np.abs(gr.numpy() - z[f"grad_{c}"]).max() <= 1e-12 * np.abs(z[f"grad_{c}"]).max() + 1e-300


def test_oracle_chamfer_reductions_and_empty_clouds():
    x = torch.tensor([[[0.0, 0.0], [2.0, 0.0]], [[0.0, 0.0], [9.0, 9.0]]])
    y = torch.tensor([[[1.0, 0.0]], [[0.0, 1.0]]])
    lx = torch.tensor([2, 0])
    s = ko.chamfer_f64(x, y, lx, None, batch_reduction=None, point_reduction="sum")[0]
    assert s.tolist() == [1 + 1 + 1, 0]                 # frame 1: no x points, so both directions give 0
    m = ko.chamfer_f64(x, y, lx, None, batch_reduction=None, point_reduction="mean")[0]
    assert m[0].item() == 1 + 1 and torch.isnan(m[1])   # 0 / 0, as pytorch3d
    assert ko.chamfer_f64(x, y, None, None, batch_reduction="sum", point_reduction="sum")[0].item() == 3 + (1 + 145 + 1)


def test_new_c_entries_check_arguments_without_gpu():
    lib = _lib.load()
    nbytes = ctypes.c_size_t(0)
    assert lib.recmv_knn_workspace_bytes(2, 100, 50, None) == -1
    assert lib.recmv_knn_workspace_bytes(-1, 100, 50, ctypes.byref(nbytes)) == -3
    assert lib.recmv_knn_workspace_bytes(2, -1, 50, ctypes.byref(nbytes)) == -3
    assert lib.recmv_knn_workspace_bytes(1 << 20, 1 << 12, 50, ctypes.byref(nbytes)) == -4
    assert lib.recmv_knn_nearest(None, None, None, None, 1, 10, 10, 4, None, None, None, None) == -3    # D = 4
    assert lib.recmv_knn_nearest(None, None, None, None, 0, 10, 10, 3, None, None, None, None) == 0     # nothing to do
    assert lib.recmv_knn_nearest(None, None, None, None, 1, 10, 10, 3, None, None, None, None) == -1
    assert lib.recmv_knn_nearest_backward(None, None, None, None, 1, 10, 10, 1, None, None, None, None) == -3
    assert lib.recmv_knn_nearest_backward(None, None, None, None, 1, 10, 10, 2, None, None, None, None) == -1
    assert lib.recmv_knn_nearest_backward(None, None, None, None, 0, 10, 10, 2, None, None, None, None) == 0


def test_python_layer_rejects_what_it_does_not_implement():
    from recmv_b200 import knn, ops
    from recmv_b200.utils import fl_proj_loss
    a, b = torch.randn(1, 8, 3), torch.randn(1, 5, 3)
    with pytest.raises(RuntimeError):
        knn.knn_points(a, b)                                    # CPU tensors: no fallback
    with pytest.raises(RuntimeError):
        ops.knn_nearest(a, b)
    with pytest.raises(NotImplementedError):
        knn.knn_points(a, b, K=5)
    with pytest.raises(NotImplementedError):
        knn.knn_points(a, b, return_nn=True)
    with pytest.raises(NotImplementedError):
        knn.chamfer_distance(a, b, x_normals=a)
    with pytest.raises(NotImplementedError):
        knn.chamfer_distance(a, b, weights=torch.ones(1))
    with pytest.raises(ValueError):
        knn.chamfer_distance(a, b, point_reduction=None)
    with pytest.raises(RuntimeError):
        fl_proj_loss([a], [b[..., :2]], [torch.ones(1, 8, 3, dtype=torch.bool)])


def test_knn_gather_masks_missing_neighbours():
    from recmv_b200.knn import knn_gather
    x = torch.arange(12.0).view(1, 4, 3)
    idx = torch.tensor([[[2], [-1], [0]]])
    out = knn_gather(x, idx)
    assert out.shape == (1, 3, 1, 3)
    assert out[0, :, 0].tolist() == [[6, 7, 8], [0, 0, 0], [0, 1, 2]]
    assert knn_gather(x, idx, lengths=torch.tensor([0])).abs().sum() == 0
    assert knn_gather(x[:, :0], torch.full((1, 2, 1), -1)).shape == (1, 2, 1, 3)
