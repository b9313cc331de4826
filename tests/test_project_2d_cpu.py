"""CPU: the reference fixture (tests/golden/project_2d_ref.npz) regenerates identically; the projection's table checks
refuse a bad table before any device work; and oracle/curve_oracle.py, the float64 restatement the GPU tests of the
feature-curve kernels compare against, agrees with torch's own float64 autograd of the reference's expressions (Intersect_Free_Curve.forward /
.regularization, CameraMine.transform_points_screen, fl_proj_loss's argsort / gather compaction), including the
kinks: relu at 0, a zero-length segment and collinear points (finite differences away from them)."""
import importlib.util
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import curve_oracle as co, zbuf_oracle as zo  # noqa: E402


def _reference(center, dirs, s0, nx, scale, t):
    v = center[:, None] + dirs * s0[..., None] * F.relu(scale[..., None]) + t[..., None] * nx[:, None]
    d = torch.cat([v[:, :-1] - v[:, 1:], v[:, -1:] - v[:, :1], v[:, :1] - v[:, 1:2]], 1)
    d = d / (d.norm(dim=-1, keepdim=True) + 1e-6)
    diff = (1 - F.cosine_similarity(d[:, :-1], d[:, 1:], dim=-1)).sum(-1)
    return v, diff, (v.mean(1) - center).abs().sum(-1)


def _curves(case, C=3, S=12, seed=0):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, dtype=torch.float64, generator=g)  # noqa: E731
    center, dirs, nx = r(C, 3), r(C, S, 3), r(C, 3)
    s0 = torch.rand(C, S, dtype=torch.float64, generator=g)
    scale, t = r(C, S), r(C, S) * 0.1
    if case == "relu0":
        scale[0, 3] = 0.
    if case == "zero_segment":
        dirs[1, 4], s0[1, 4], scale[1, 4], t[1, 4] = dirs[1, 5], s0[1, 5], scale[1, 5], t[1, 5]
    if case == "collinear":
        t[2] = 0.
        dirs[2] = dirs[2, :1].expand(S, 3)
        s0[2] = torch.linspace(0.1, 2, S, dtype=torch.float64)
        scale[2] = 1.
    return center, dirs, s0, nx, scale, t


@pytest.mark.parametrize("case", ["random", "relu0", "zero_segment", "collinear"])
def test_curve_oracle_matches_torch_autograd(case):
    center, dirs, s0, nx, scale, t = _curves(case)
    scale.requires_grad_()
    t.requires_grad_()
    v, diff, cen = _reference(center, dirs, s0, nx, scale, t)
    g = torch.Generator().manual_seed(1)
    gd, gc = torch.randn(3, dtype=torch.float64, generator=g), torch.randn(3, dtype=torch.float64, generator=g)
    dv = torch.randn(v.shape, dtype=torch.float64, generator=g)
    ((diff * gd).sum() + (cen * gc).sum() + (v * dv).sum()).backward()
    vo = co.curve_points(center, dirs, s0, nx, scale.detach(), t.detach())
    do, ceno = co.regularizer(vo, center)
    np.testing.assert_allclose(vo, v.detach().numpy(), rtol=0, atol=1e-14)
    np.testing.assert_allclose(do, diff.detach().numpy(), rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(ceno, cen.detach().numpy(), rtol=1e-13, atol=1e-13)
    gv = co.regularizer_vjp(vo, center, gd.numpy(), gc.numpy()) + dv.numpy()
    ds, dt = co.curve_vjp(dirs, s0, nx, scale.detach(), gv)
    for got, ref in ((ds, scale.grad.numpy()), (dt, t.grad.numpy())):
        assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()
    if case == "relu0":
        assert ds[0, 3] == 0.0                  # relu'(0) = 0
    if case == "zero_segment":                  # the 1e-8 cosine clamp and the 1e-6 norm offset blow the gradient up
        assert np.abs(ds[1]).max() > 1e6 * np.abs(ds[0]).max()


def test_curve_oracle_matches_finite_differences_away_from_kinks():
    center, dirs, s0, nx, scale, t = _curves("collinear")
    scale = scale.abs() + 0.1
    v = co.curve_points(center, dirs, s0, nx, scale, t)
    rng = np.random.default_rng(3)
    gd, gc = rng.standard_normal(3), rng.standard_normal(3)
    ds, dt = co.curve_vjp(dirs, s0, nx, scale, co.regularizer_vjp(v, center, gd, gc))

    def f(sc, tt):
        d, c = co.regularizer(co.curve_points(center, dirs, s0, nx, sc, tt), center)
        return (d * gd).sum() + (c * gc).sum()

    h = 1e-6
    for (c, s) in ((0, 2), (2, 5), (2, 0), (1, 11)):
        e = np.zeros(scale.shape)
        e[c, s] = h
        fd_s = (f(scale.numpy() + e, t.numpy()) - f(scale.numpy() - e, t.numpy())) / (2 * h)
        fd_t = (f(scale.numpy(), t.numpy() + e) - f(scale.numpy(), t.numpy() - e)) / (2 * h)
        assert abs(fd_s - ds[c, s]) <= 1e-5 * max(1.0, abs(ds[c, s])), (c, s, fd_s, ds[c, s])
        assert abs(fd_t - dt[c, s]) <= 1e-5 * max(1.0, abs(dt[c, s])), (c, s, fd_t, dt[c, s])


def test_projection_oracle_matches_transform_points_screen():
    N, P, W, H = 3, 9, 1283, 721
    g = torch.Generator().manual_seed(5)
    R = torch.linalg.qr(torch.randn(N, 3, 3, dtype=torch.float64, generator=g))[0]
    T = torch.tensor([[0.1, 0.2, 3.0], [0.0, -0.1, 3.5], [0.3, 0.0, 2.5]], dtype=torch.float64)
    f = torch.tensor([[952., 950.], [948., 953.], [900., 910.]], dtype=torch.float64)
    pp = torch.tensor([[640.3, 359.6], [641., 360.5], [630., 350.]], dtype=torch.float64)
    cam = zo.Camera(f, pp, R, T, (W, H))
    X = (torch.randn(N, P, 3, dtype=torch.float64, generator=g) * 0.3).requires_grad_()
    s = cam.transform_points_screen(X, torch.tensor([[W, H]] * N, dtype=torch.float64))
    rows = zo.camera_rows(cam)
    np.testing.assert_allclose(co.screen(X.detach(), rows, W, H), s.detach().numpy(), rtol=1e-12, atol=1e-9)
    dxy = torch.randn(N, P, 2, dtype=torch.float64, generator=g)
    (s[..., :2] * dxy).sum().backward()
    np.testing.assert_allclose(co.screen_vjp(X.detach(), rows, W, H, dxy), X.grad.numpy(), rtol=1e-10, atol=1e-9)


def test_compaction_oracle_equals_fl_proj_loss_argsort_gather():
    g = torch.Generator().manual_seed(9)
    B, P = 12, 37
    x = torch.randn(B, P, 2, generator=g)
    vis = torch.rand(B, P, generator=g) < 0.6
    vis[3] = False
    vis[4] = True
    order = torch.argsort((~vis).to(torch.uint8), dim=1, stable=True)       # utils.fl_proj_loss's compaction
    xc = torch.gather(x, 1, order[..., None].expand(-1, -1, 2))
    clouds, counts = co.compact(x.numpy(), vis.numpy())
    assert (counts == vis.sum(1).numpy()).all()
    for b in range(B):
        assert np.array_equal(clouds[b, :counts[b]], xc[b, :counts[b]].numpy())
        assert not clouds[b, counts[b]:].any()


def test_fixture_regenerates_identically():
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    spec = importlib.util.spec_from_file_location("make_golden_project_2d",
                                                  os.path.join(golden, "make_golden_project_2d.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    z = np.load(os.path.join(golden, "project_2d_ref.npz"))
    old = {k: z[k] for k in z.files}
    new = mod.generate()
    assert set(new) == set(old)
    for k in old:
        np.testing.assert_array_equal(new[k], old[k], err_msg=k)


def test_projection_refuses_bad_tables_before_any_device_work():
    import ctypes
    from recmv_b200 import _lib
    lib = _lib.load()
    K, N, S, M = 3, 2, 4, 3
    R = K * N * S
    fake = ctypes.c_void_p(16)          # never dereferenced: the table is checked first

    def call(table):
        t = (ctypes.c_int32 * (3 * K))(*[x for row in table for x in row])
        thr = (ctypes.c_float * K)(0.1, 0.1, 0.1)
        return lib.recmv_curve_project(fake, R, fake, N, 64, 48, t, thr, K, S, fake, M, fake, fake, fake, fake, fake,
                                       fake, fake, None)

    good = [(0, S, 0), (N * S, S, 1), (2 * N * S, S, 2)]
    assert call([good[0], good[0], good[2]]) == -3                 # overlapping ranges (the total still R)
    assert call([good[0], good[1], (2 * N * S + 1, S, 2)]) == -3   # a range past R
    assert call([good[0], good[1], (2 * N * S, S, 3)]) == -3       # a mask column past M
    interleaved = [(0, K * S, 0), (S, K * S, 1), (2 * S, K * S, 2)]
    assert call([interleaved[0], interleaved[0], interleaved[2]]) == -3
