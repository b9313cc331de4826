"""CPU: the float64 point-rasterizer oracle (oracle/points_oracle.py) -- its closed-form composite backward against
torch.autograd and finite differences, its split rule and weights against the reference's own
PointsRendererWithFrags_Split.forward, hand-built selections with known answers -- and the argument errors of the C
entries and of the Python layer without a GPU.  The CUDA kernel is compared with this oracle in
tests/test_gpu_points_raster.py."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import points_oracle as po
from oracle import refload
from recmv_b200 import _lib, ops

H, W, R, K = 24, 32, 0.2, 6


def scene(P=200, N=2, seed=0):
    g = np.random.default_rng(seed)
    ndc = np.stack([g.uniform(-1.1, 1.1, (N, P)), g.uniform(-1.1, 1.1, (N, P)), g.uniform(0.5, 3.0, (N, P))], -1)
    feats = g.uniform(0.3, 1.5, (N, P))
    return ndc, feats


def test_selection_rules_on_a_hand_built_pixel():
    # pixel (row 0, col 0) of a 2 x 2 image is at NDC (0.5, 0.5); five points on it, depths with a tie
    ndc = np.array([[[0.5, 0.5, 2.0], [0.5, 0.5, 1.0], [0.5, 0.5, 1.0], [0.5, 0.5, -1.0], [0.5, 0.5, 0.0]]])
    s = po.select(ndc, 2, 2, 0.1, 3)
    i, z, d = po.dense(s)
    assert i[0, 0, 0].tolist() == [4, 1, 2]              # z = 0 kept, z < 0 skipped, the tie to the lower index
    assert z[0, 0, 0].tolist() == [0.0, 1.0, 1.0] and np.all(d[0, 0, 0] == 0)
    assert s["skipped"] == 1 and np.all(i[0, 1, 1] == -1)
    img = po.composite(s, 0.1)
    assert img[0, 0, 0, 0] == 1.0 and img[0, 0, 1, 1] == 0.0   # alpha = 1 on the centre: nothing behind shows


def test_disc_edge_is_strict():
    # a point exactly r away from a pixel centre does not cover it
    ndc = np.array([[[0.5 + 0.25, 0.5, 1.0]]])
    s = po.select(ndc, 2, 2, 0.25, 4)
    assert s["count"][0, 0, 0] == 0


def test_composite_backward_matches_autograd():
    ndc, feats = scene()
    s = po.select(ndc, H, W, R, K)
    assert s["count"].max() == K and (s["count"] > 0).sum() > 100   # some pixels are full
    gi = np.random.default_rng(1).standard_normal((2, 2, H, W))
    for split, G in ((None, 1), (25, 2)):
        t = torch.tensor(ndc, requires_grad=True)
        img = po.composite_torch(s, t, R, feats, split, G)
        ref = po.composite(s, R, feats, split, G)
        assert np.allclose(img.detach().numpy(), ref, rtol=1e-13, atol=1e-14)
        (img * torch.tensor(gi[:G])).sum().backward()
        got = po.composite_grad(s, ndc, R, gi[:G], feats, split)
        # exact but for the 1e-9 that pytorch3d's backward adds to 1 - alpha
        err = np.abs(got - t.grad.numpy()).max() / np.abs(t.grad.numpy()).max()
        assert err < 1e-6, err
        assert np.all(got[..., 2] == 0) and np.abs(got).max() > 1


def test_composite_backward_matches_finite_differences():
    ndc, feats = scene(seed=3)
    s = po.select(ndc, H, W, R, K, margin=1e-3)
    gi = np.random.default_rng(4).standard_normal((2, 2, H, W)) * ~s["ambiguous"][None]
    grad = po.composite_grad(s, ndc, R, gi, feats, 30)
    v = np.random.default_rng(5).standard_normal(ndc.shape)
    v[..., 2] = 0
    eps = 1e-7

    def loss(p):
        return (po.composite(po.select(p, H, W, R, K), R, feats, 30, 2) * gi).sum()

    fd = (loss(ndc + eps * v) - loss(ndc - eps * v)) / (2 * eps)
    assert abs(fd - (grad * v).sum()) < 1e-6 * max(1.0, abs(fd)), (fd, (grad * v).sum())


@pytest.mark.skipif(not refload.available(), reason="the reference source tree is not present")
def test_reference_split_renderer_over_the_oracle_matches_the_fused_split():
    refload.install()
    import importlib
    cm = importlib.import_module("model.CameraMine")
    ndc, _ = scene(P=80, seed=7)
    N, P = ndc.shape[:2]
    ren = cm.PointsRendererWithFrags_Split(po.Rasterizer(H, W, R, K), po.alpha_compositor)
    clouds = SimpleNamespace(points_padded=lambda: torch.tensor(ndc),
                             features_packed=lambda: torch.ones(N * P, 1, dtype=torch.float64))
    (up, bo), frags = ren(clouds, split_size=35, all_size=P)
    s = po.select(ndc, H, W, R, K)
    fused = po.composite(s, R, None, 35, 2)
    assert up.shape == (N, H, W, 1)
    assert np.allclose(up[..., 0].numpy(), fused[0], atol=1e-14) and np.allclose(bo[..., 0].numpy(), fused[1], atol=1e-14)
    assert up.abs().sum() > 1 and bo.abs().sum() > 1


def test_c_entries_reject_bad_arguments_without_a_gpu():
    lib = _lib.load()
    nb = ctypes.c_size_t(0)
    assert lib.recmv_points_raster_workspace_bytes(3, 1000, 1080, 1080, 5000, None) == -1
    assert lib.recmv_points_raster_workspace_bytes(3, 1000, 0, 1080, 5000, ctypes.byref(nb)) == -3
    assert lib.recmv_points_raster_workspace_bytes(3, 1000, 1080, 1080, 5000, ctypes.byref(nb)) == 0
    assert nb.value >= 3 * 1000 * 32 + 5000 * 4
    p = ctypes.c_void_p(16)   # never dereferenced: validation fails first

    def fwd(N=1, P=10, Hh=8, Ww=8, r=0.1, k=4, split=10, G=1, ctr=p):
        return lib.recmv_rasterize_points(p, None, N, P, Hh, Ww, r, k, split, G, p, 100, p, None, None, None, ctr, None)

    assert fwd(k=65) == _lib.RECMV_E_RANGE
    assert fwd(k=0) == -3 and fwd(r=0.0) == -3 and fwd(r=float("nan")) == -3 and fwd(G=3) == -3
    assert fwd(split=11) == -3 and fwd(split=-1) == -3 and fwd(N=-1) == -3
    assert fwd(N=70000) == _lib.RECMV_E_RANGE and fwd(ctr=None) == -1
    bwd = lib.recmv_rasterize_points_backward
    assert bwd(1, 10, 8, 8, 0.1, 65, 10, 1, p, 5, p, p, p, None) == _lib.RECMV_E_RANGE
    assert bwd(1, 10, 8, 8, 0.1, 4, 10, 1, None, 5, p, p, p, None) == -1
    assert bwd(1, 0, 8, 8, 0.1, 4, 0, 1, None, 0, None, None, None, None) == 0   # nothing to do


def test_python_layer_rejects_cpu_tensors_and_large_k():
    pts = torch.zeros(1, 4, 3)
    with pytest.raises(RuntimeError):
        ops.rasterize_points(pts, None, 8, 8, 0.1, 4)
    from recmv_b200 import raster
    with pytest.raises(RuntimeError):
        raster.rasterize_points(pts, (torch.ones(2), torch.zeros(2), torch.eye(3), torch.zeros(3)), (8, 8), 0.1, 4)
