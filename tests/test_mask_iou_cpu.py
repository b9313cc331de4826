"""CPU tests of the mask-IoU oracle (oracle/mask_iou_oracle.py, DESIGN section 1m), which the GPU tests hold the kernel
to: the dilation equals F.max_pool2d bit for bit, the loss equals the reference's formula, and the VJP matches finite
differences, including the pixels where |m + g' - m g'| has its kink; the Meshes stand-in answers the calls
mask_loss's consumers make; the size query refuses bad extents."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import mask_iou_oracle as mio, refload
from recmv_b200 import _lib


def _masks(rng, N, H, W, soft, border=True):
    if soft:
        gt = rng.uniform(size=(N, H, W)).astype(np.float32) * (rng.uniform(size=(N, H, W)) < 0.3)
    else:
        gt = (rng.uniform(size=(N, H, W)) < 0.05).astype(np.float32)
    if border:
        gt[:, 0, :] = gt[:, :, -1] = 1.0             # the masks touch the image border
    return gt


@pytest.mark.parametrize("H,W", [(17, 23), (16, 24), (21, 20), (1, 9), (9, 1)])
@pytest.mark.parametrize("r", [1, 2, 3, 4])
@pytest.mark.parametrize("soft", [False, True])
def test_dilation_is_max_pool2d_bit_for_bit(H, W, r, soft):
    rng = np.random.default_rng(H * 1000 + W * 10 + r)
    gt = _masks(rng, 3, H, W, soft)
    ref = F.max_pool2d(torch.from_numpy(gt), kernel_size=2 * r + 1, stride=1, padding=r).numpy()
    out = mio.dilate(gt, r)
    assert out.dtype == np.float32
    np.testing.assert_array_equal(out.view(np.uint32), ref.view(np.uint32))


def test_loss_is_the_reference_formula_in_float64():
    rng = np.random.default_rng(7)
    N, H, W = 4, 19, 26
    m = rng.uniform(size=(N, H, W))
    g = mio.dilate(_masks(rng, N, H, W, True).astype(np.float64), 2)
    mt, gt = torch.from_numpy(m), torch.from_numpy(g)
    ref = (1. - (mt * gt).view(N, -1).sum(1) / (mt + gt - mt * gt).abs().view(N, -1).sum(1)).mean()
    I, U, L, loss = mio.iou(m, g)
    assert abs(loss - float(ref)) <= 1e-15
    np.testing.assert_allclose(L, 1 - I / U, rtol=0, atol=0)


def test_empty_silhouette_and_mask_give_nan():
    z = np.zeros((2, 5, 6))
    m = z.copy()
    m[1, 2, 3] = 0.5
    I, U, L, loss = mio.iou(m, z)
    assert np.isnan(L[0]) and L[1] == 1.0 and np.isnan(loss)


def test_vjp_matches_finite_differences_and_autograd():
    rng = np.random.default_rng(11)
    N, H, W = 3, 7, 9
    g = mio.dilate(_masks(rng, N, H, W, True, border=False).astype(np.float64), 1)
    m = rng.uniform(0.05, 0.95, size=(N, H, W))
    m[0, :2] = 0.0                                   # m = 0 where g' = 0 (the kink of |.|) and where g' = 1
    g[0, 0] = 0.0
    g[0, 1] = 1.0
    w = 1.7
    dm = mio.iou_vjp(m, g, w)
    mt = torch.from_numpy(m).requires_grad_(True)
    gt = torch.from_numpy(g)
    loss = (1. - (mt * gt).view(N, -1).sum(1) / (mt + gt - mt * gt).abs().view(N, -1).sum(1)).mean() * w
    loss.backward()
    np.testing.assert_allclose(dm, mt.grad.numpy(), rtol=1e-13, atol=1e-16)
    assert np.all(dm[0, 0] == 0.0)                   # s = 0 and g' = 0: no gradient
    eps = 1e-7
    for n, y, x in [(0, 1, 3), (0, 2, 4), (1, 3, 3), (2, 6, 8)]:     # m = 0, g' = 1 and interior pixels
        mp, mm = m.copy(), m.copy()
        mp[n, y, x] += eps
        mm[n, y, x] -= eps if m[n, y, x] > 0 else 0.0
        fd = (mio.iou(mp, g)[3] - mio.iou(mm, g)[3]) * w / (mp[n, y, x] - mm[n, y, x])
        assert abs(fd - dm[n, y, x]) <= 1e-6 * max(1.0, abs(dm[n, y, x])), (n, y, x, fd, dm[n, y, x])


def test_meshes_stand_in():
    from recmv_b200.utils import Meshes
    v = [torch.randn(5, 3) for _ in range(2)]
    f = torch.tensor([[0, 1, 2], [2, 3, 4]])
    mesh = Meshes(verts=v, faces=[f, f])
    assert mesh.verts_padded().shape == (2, 5, 3) and torch.equal(mesh.verts_packed(), torch.cat(v))
    assert mesh.verts_list()[1] is v[1] and mesh.faces_list()[0] is f and torch.equal(mesh.faces_packed(),
                                                                                    torch.cat([f, f + 5]))
    assert len(mesh) == 2


def test_workspace_query_refuses_bad_extents():
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    assert lib.recmv_mask_iou_workspace_bytes(2, 3, 1080, 1080, 3, ctypes.byref(n)) == 0
    assert n.value == 2 * 3 * 34 * 34 * 16 + (-(2 * 3 * 34 * 34 * 16) % 256)
    assert lib.recmv_mask_iou_workspace_bytes(2, 3, 1080, 1080, 3, None) == -1
    for args, status in [((2, 3, 1080, 1080, 0), -3), ((0, 3, 8, 8, 1), -3), ((1, 0, 8, 8, 1), -3),
                         ((1, 1, 0, 8, 1), -3), ((1, 1, 8, -1, 1), -3), ((1, 1, 8, 8, 33), -4),
                         ((1, 65536, 8, 8, 1), -4)]:
        assert lib.recmv_mask_iou_workspace_bytes(*args, ctypes.byref(n)) == status, args
    assert lib.recmv_mask_iou(1, None, None, 1, 8, 8, 0, None, None, None, None, None, None) == -3
    assert lib.recmv_mask_iou(1, None, None, 1, 8, 8, 1, None, None, None, None, None, None) == -1
    assert lib.recmv_mask_iou_backward(1, None, None, 1, 8, 8, None, None, None, None) == -1
    assert lib.recmv_mask_iou_backward(0, None, None, 1, 8, 8, None, None, None, None) == -3


# ---- the reference's own mask_loss (tests/golden/mask_loss_ref.npz) ------------------------------------------------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _fixture():
    z = np.load(os.path.join(GOLDEN, "mask_loss_ref.npz"))
    return {k: z[k] for k in z.files}


def test_fixture_dilation_and_loss_match_the_oracle():
    d = _fixture()
    for g in range(2):
        mgt = mio.dilate(d[f"in/gt_{g}"], int(d["radius"]))
        np.testing.assert_array_equal(mgt, d[f"f32/mgt_{g}"])
        np.testing.assert_array_equal(mgt.astype(np.float64), d[f"f64/mgt_{g}"])
        loss = mio.iou(d[f"f64/masks_{g}"], d[f"f64/mgt_{g}"])[3]
        assert abs(loss - float(d[f"f64/info/{('upper', 'bottom')[g]}_mask_loss"])) <= 1e-12


@pytest.mark.skipif(not refload.available(), reason="needs the reference source tree")
def test_fixture_regenerates_identically():
    spec = importlib.util.spec_from_file_location("make_golden_mask_loss", os.path.join(GOLDEN,
                                                                                        "make_golden_mask_loss.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    new, old = mod.generate(), _fixture()
    assert set(new) == set(old)
    for k in old:
        np.testing.assert_array_equal(new[k], old[k], err_msg=k)
