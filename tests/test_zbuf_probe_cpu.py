"""CPU checks of the sparse z-buffer probe's oracle and fixture, and of its argument checks (DESIGN section 1i):
oracle/zbuf_oracle.py's sampler against F.grid_sample in float64; the oracle against the reference's own visibility
tests (tests/golden/zbuf_ref.npz, tests/golden/make_golden_zbuf.py); the fixture's regeneration; and the C ABI and
Python entry points refusing bad arguments and CPU tensors without a GPU."""
import ctypes
import importlib.util
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from conftest import GOLDEN, load_golden
from oracle import refload
from oracle import zbuf_oracle as zo
from recmv_b200 import _lib, ops, raster
from recmv_b200 import utils as ru

CASES = ("n1_square", "n3_wide")


def _torch_sample(img, uv):
    return Fn.grid_sample(torch.tensor(img)[:, None], torch.tensor(uv)[:, :, None], mode="bilinear",
                          padding_mode="zeros", align_corners=True)[:, 0, :, 0].numpy()


@pytest.mark.parametrize("kind", ["random", "border", "integer", "outside"])
def test_oracle_sampler_matches_grid_sample(kind):
    g = np.random.default_rng(5)
    N, H, W, Q = 3, 7, 11, 500
    img = g.standard_normal((N, H, W))
    if kind == "random":
        uv = g.uniform(-1.2, 1.2, (N, Q, 2))
    elif kind == "border":
        uv = g.uniform(-1, 1, (N, Q, 2))
        uv[:, ::2, 0] = g.choice([-1.0, 1.0], (N, (Q + 1) // 2))
        uv[:, 1::2, 1] = g.choice([-1.0, 1.0], (N, Q // 2))
    elif kind == "integer":   # sample positions exactly on pixel centres
        ix, iy = g.integers(0, W, (N, Q)), g.integers(0, H, (N, Q))
        uv = np.stack([2.0 * ix / (W - 1) - 1, 2.0 * iy / (H - 1) - 1], -1)
    else:
        uv = g.uniform(-3, 3, (N, Q, 2))
        uv[:, :50] = np.where(g.random((N, 50, 2)) < 0.5, -1 - 1e-9, 1 + 1e-9)
    np.testing.assert_allclose(zo.grid_sample(img, uv), _torch_sample(img, uv), rtol=1e-13, atol=1e-13)


def test_oracle_sampler_nonfinite_is_zero():
    img = np.ones((1, 4, 4))
    uv = np.array([[[np.nan, 0.0], [0.0, np.inf], [-np.inf, -np.inf], [1e30, 0.0]]])
    assert (zo.grid_sample(img, uv) == 0).all()


def _case(z, name):
    p = name + "/"
    return {k[len(p):]: v for k, v in z.items() if k.startswith(p)}


def _scene_tensors(s):
    N = int(s["N"])
    cam = zo.Camera(*(torch.tensor(s[k]) for k in ("focal", "pp", "R", "T")), (int(s["W"]), int(s["H"])))
    ps = torch.tensor([[float(s["W"]), float(s["H"])]] * N)
    return N, cam, ps


def oracle_visibility(s):
    """float64 oracle of both fixture functions: (vis [N,P,2], check [N,Q])."""
    N, cam, ps = _scene_tensors(s)
    H, W = int(s["H"]), int(s["W"])
    rows = zo.camera_rows(cam)
    skin, poses = zo.BodySkin(), torch.tensor(s["poses"])
    c_z = float(cam.cam_pos()[2])
    P1 = s["fl1"].shape[0]
    dg = zo.GarmentDeformer()(torch.tensor(s["garm_v"])[None].expand(N, -1, 3), [torch.tensor(s["cond"]), poses])
    fl0 = skin(torch.tensor(s["fl0"])[None].expand(N, -1, 3), poses)
    fl1 = skin(torch.tensor(s["fl1"])[None].expand(N, -1, 3), poses)
    # the border / off-screen points follow the curve points of the second curve unchanged (make_golden_zbuf.inputs)
    nedge = s["vis"].shape[1] - s["fl0"].shape[0] - P1
    gen = _generator()
    edge = torch.tensor(gen.edge_points({k: s[k] for k in ("W", "H", "focal", "pp", "R", "T")}, cam))
    assert edge.shape[0] == nedge
    fl = torch.cat([fl0, fl1, edge[None].expand(N, -1, 3)], 1)
    dgz = dg.double().numpy()
    fill_g = (dgz[..., 2] - c_z).max(-1)
    sg = zo.probe(dgz, s["garm_f"], rows, H, W, cam.transform_points_screen(fl, ps).numpy(), ps.numpy(), fill_g)["out"]
    body = skin(torch.tensor(s["body_v"])[None].expand(N, -1, 3), poses).double().numpy()
    cano = torch.cat([torch.tensor(s["cano0"]), torch.tensor(s["cano1"]), edge])[None].expand(N, -1, 3)
    sfl = skin(cano, poses)
    fill_b = (body[..., 2] - c_z).max(-1)
    sb = zo.probe(body, s["body_f"], rows, H, W, cam.transform_points_screen(sfl, ps).numpy(), ps.numpy(), fill_b)["out"]
    vis = np.stack([fl.double().numpy()[..., 2] - (sg + c_z), sfl.double().numpy()[..., 2] - (sb + c_z)], -1)
    bt = skin(torch.tensor(s["body_v"])[None].expand(N, -1, 3), [poses, torch.tensor(s["trans"])]).double().numpy()
    chk = zo.probe(bt, s["body_f"], rows, H, W, s["check_screen"], ps.numpy(), bt[..., 2].max(-1))["out"]
    return vis, chk


def _generator():
    spec = importlib.util.spec_from_file_location("make_golden_zbuf", os.path.join(GOLDEN, "make_golden_zbuf.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    return gen


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_fixture(name):
    s = _case(load_golden("zbuf_ref.npz"), name)
    vis, chk = oracle_visibility(s)
    # fp32 rounds the sample position by ~1e-5 px; across a depth step of ~1 that moves the value by as much
    ok = ~s["vis_amb"]
    err = np.abs(vis - s["vis"])[ok]
    assert err.max() < 1e-4 and np.median(err) < 1e-6, err.max()
    ok = ~s["check_amb"]
    err = np.abs(chk - s["check"])[ok]
    assert err.max() < 1e-4 and np.median(err) < 1e-6, err.max()
    # the scene holds what the fixture claims: visible and hidden curve points, background and border queries
    assert (s["vis"][..., 1] < 0.08).any() and (s["vis"][..., 1] > 0.08).any()
    H, W = int(s["H"]), int(s["W"])
    cols, rows, w, inside = zo.taps(H, W, s["check_screen"], np.array([[W, H]] * int(s["N"])))
    assert (~inside.any(-1)).any()                                           # entirely off-screen
    assert (inside.any(-1) & ~inside.all(-1)).any()                          # on the border
    assert ok.sum() >= 0.9 * ok.size


@pytest.mark.skipif(not refload.available(), reason="needs the reference source tree")
def test_fixture_regenerates():
    out = _generator().generate()
    z = load_golden("zbuf_ref.npz")
    assert set(out) == set(z)
    for k in z:
        np.testing.assert_array_equal(np.asarray(out[k]), z[k], err_msg=k)


def test_capi_rejects_bad_arguments_without_gpu():
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    assert lib.recmv_zbuf_probe_workspace_bytes(2, 100, 1080, 1080, ctypes.byref(n)) == 0 and n.value > 800 * 8
    assert lib.recmv_zbuf_probe_workspace_bytes(2, 100, 1080, 1080, None) == -1
    assert lib.recmv_zbuf_probe_workspace_bytes(-1, 100, 8, 8, ctypes.byref(n)) == -3
    assert lib.recmv_zbuf_probe_workspace_bytes(1, -1, 8, 8, ctypes.byref(n)) == -3
    assert lib.recmv_zbuf_probe_workspace_bytes(1, 10, 0, 8, ctypes.byref(n)) == -3
    assert lib.recmv_zbuf_probe_workspace_bytes(1, 1 << 30, 8, 8, ctypes.byref(n)) == -4
    assert lib.recmv_zbuf_probe_workspace_bytes(4, 10, 30000, 30000, ctypes.byref(n)) == -4
    args = dict(verts=None, V=4, faces=None, F=2, N=1, cam=None, H=8, W=8, zc=1e-6, ae=1e-8, pts=None, Q=3, D=3,
                ns=None, fill=None, ws=None, out=None, tz=None, tf=None, st=None)

    def call(**kw):
        a = dict(args, **kw)
        return lib.recmv_zbuf_probe(*a.values())

    assert call(D=1) == -3                # x and y at least
    assert call(F=1, V=0) == -3           # faces with no vertices
    assert call(H=0) == -3
    assert call(Q=-1) == -3
    assert call(N=70000, F=40000) == -4   # N * F beyond int32
    assert call(tz=ctypes.c_void_p(16)) == -1   # taps: both or neither
    assert call() == -1                   # NULL operands
    assert call(Q=0) == 0                 # nothing to do: no CUDA call


def test_python_entries_refuse_cpu_tensors():
    v = torch.zeros(1, 3, 3)
    f = torch.tensor([[0, 1, 2]])
    cam = torch.zeros(1, 16)
    pts = torch.zeros(1, 4, 3)
    ns = torch.tensor([[8.0, 8.0]])
    fill = torch.zeros(1)
    with pytest.raises(RuntimeError):
        ops.zbuf_probe(v, f, cam, 8, 8, pts, ns, fill)
    with pytest.raises(RuntimeError):
        raster.zbuf_probe(v, f, (torch.ones(1, 2), torch.zeros(1, 2), torch.eye(3)[None], torch.zeros(1, 3)), (8, 8),
                          pts, ns, fill)
    mr = types.SimpleNamespace(rasterizer=types.SimpleNamespace(
        cameras=None, raster_settings=types.SimpleNamespace(image_size=8)))
    cam_obj = zo.Camera(torch.ones(1, 2), torch.zeros(1, 2), torch.eye(3)[None], torch.tensor([[0.0, 0.0, 2.0]]), (8, 8))
    with pytest.raises(RuntimeError):
        ru.check_zbuf_body(zo.Meshes([v[0]], [f]), 1, zo.BodySkin(), torch.zeros(1, 6), torch.zeros(1, 3), cam_obj, mr,
                           ns, pts)
    assert mr.rasterizer.cameras is cam_obj   # the reference's side effect happens first
    me = types.SimpleNamespace(maskRender=mr, deformer=zo.GarmentDeformer(), garment_vs=[v[0]], garment_fs=[f],
                               tmpBodyVs=v[0], tmpBodyFs=f)
    with pytest.raises(RuntimeError):
        ru.fl_visible_by_body_zbuff(me, cam_obj, [None, torch.zeros(1, 3)], torch.zeros(1, 6), None, {}, [pts],
                                    [pts[:1]], ["neck"], 0, "upper", ns, 1)
