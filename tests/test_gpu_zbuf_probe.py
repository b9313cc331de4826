"""GPU checks of the sparse z-buffer probe (csrc/zbuf_probe.cu, DESIGN section 1i) and of the visibility drop-ins:
  * every tap bit-identical to raster.rasterize_meshes (zbuf and pix_to_face) on a production-size scene and on
    adversarial meshes, for Q from 1 to 1e5;
  * out within 2 ulp of ATen's F.grid_sample(align_corners=True) on the full rasterizer's filled zbuf (which held is
    printed), and within a sample-position ulp of the cuDNN kernel the default dispatch picks;
  * run-to-run bit identity;
  * utils.fl_visible_by_body_zbuff and utils.check_zbuf_body against the reference's own outputs
    (tests/golden/zbuf_ref.npz) and against the reference flow restated on the GPU (compat maskRender, fill,
    grid_sample); no host synchronisation; CPU tensors refused.
"""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from conftest import load_golden
from oracle import zbuf_oracle as zo
from recmv_b200 import raster
from recmv_b200 import utils as ru
from recmv_b200.compat.MaskRender import mask_renderer

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ZBUF_THRESHOLD = {"neck": 0.1, "upper_bottom": 0.08}   # utils/constant.py:219-227 for the fixture's curves


def cameras(N, H, W, seed, dist=2.6):
    g = torch.Generator().manual_seed(seed)
    R = []
    for n in range(N):
        a = 0.3 * torch.randn(3, generator=g, dtype=torch.float64)
        R.append(torch.linalg.matrix_exp(torch.tensor([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])))
    R = torch.stack(R).float()
    T = torch.tensor([[0.01 * n, -0.02, dist + 0.05 * n] for n in range(N)])
    f = 1.1 * max(H, W)
    focal = torch.full((N, 2), f)
    pp = torch.tensor([[W / 2.0 + 0.5, H / 2.0 - 1.0]] * N)
    return tuple(t.to(DEV) for t in (focal, pp, R, T))


def production_scene(N=4, H=1080, W=1080):
    """A garment tube of 159 200 faces around an SMPL-size ellipsoid body (13 776 faces), both jittered."""
    g = np.random.default_rng(7)
    gv, gf = zo.tube(400, 200, 0.27, -0.45, 0.35)
    bv, bf = zo.uv_sphere(84, 83, (0.22, 0.6, 0.16), (0, 0, 0))
    mk = lambda v: torch.tensor(np.stack([v + 0.003 * g.standard_normal(v.shape) for _ in range(N)]),  # noqa: E731
                                dtype=torch.float32, device=DEV)
    return (mk(gv), torch.tensor(gf, device=DEV)), (mk(bv), torch.tensor(bf, device=DEV)), cameras(N, H, W, 1)


def tap_pixels(pts, ns, H, W):
    """The kernel's tap pixels by the same fp32 element-wise formula: (cols, rows) [N,Q,4] int64, in-image [N,Q,4]."""
    u = 2 * pts[..., 0] / ns[:, None, 0] - 1
    v = 2 * pts[..., 1] / ns[:, None, 1] - 1
    ix, iy = ((u + 1) / 2) * (W - 1), ((v + 1) / 2) * (H - 1)
    fin = (ix > -2) & (ix < W + 1) & (iy > -2) & (iy < H + 1)
    x0 = torch.where(fin, ix, torch.full_like(ix, -10)).floor().long()
    y0 = torch.where(fin, iy, torch.full_like(iy, -10)).floor().long()
    cols = torch.stack([x0, x0 + 1, x0, x0 + 1], -1)
    rows = torch.stack([y0, y0, y0 + 1, y0 + 1], -1)
    return cols, rows, (cols >= 0) & (cols < W) & (rows >= 0) & (rows < H)


def ulps(a, b):
    ia, ib = a.view(torch.int32).long(), b.view(torch.int32).long()
    ia = torch.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = torch.where(ib < 0, -(ib & 0x7fffffff), ib)
    return (ia - ib).abs()


def check_probe(verts, faces, cams, H, W, pts, ns, fill, z_clip=1e-6, area_eps=1e-8):
    """Taps bit-identical to the full rasterization, out within 2 ulp of ATen's grid_sample on the filled zbuf;
    returns (max ulp, taps compared, max |out - cuDNN grid_sample|)."""
    fr = raster.rasterize_meshes(verts, faces, cams, (H, W), z_clip=z_clip, area_eps=area_eps, want_dists=False)
    out, tz, tf = raster.zbuf_probe(verts, faces, cams, (H, W), pts, ns, fill, z_clip, area_eps, return_taps=True)
    N = verts.shape[0]
    cols, rows, ok = tap_pixels(pts, ns, H, W)
    n = torch.arange(N, device=DEV)[:, None, None].expand_as(cols)
    zb = fr.zbuf[..., 0][n, rows.clamp(0, H - 1), cols.clamp(0, W - 1)]
    pf = fr.pix_to_face[..., 0][n, rows.clamp(0, H - 1), cols.clamp(0, W - 1)]
    assert torch.equal(tz[ok].view(torch.int32), zb[ok].view(torch.int32))
    assert torch.equal(tf[ok], pf[ok])
    assert (tz[~ok] == -1).all() and (tf[~ok] == -1).all()
    z = fr.zbuf.clone()
    z[z == -1.] = fill[:, None, None, None].expand_as(z)[z == -1.]
    uv = torch.stack([2 * pts[..., 0] / ns[:, None, 0] - 1, 2 * pts[..., 1] / ns[:, None, 1] - 1], -1)
    # a non-finite position, or one with no tap inside the image, gives 0; the rest are compared
    fin = torch.isfinite(uv).all(-1) & ok.any(-1)
    assert (out[~fin] == 0).all()
    # ATen's own kernel (what the probe restates), and the default dispatch, which hands bilinear / zeros /
    # align_corners=True on a 4-D input to cuDNN: its sample position may differ from ATen's by an ulp of ix or iy,
    # which moves the value by up to that much times the spread of the four taps
    with torch.backends.cudnn.flags(enabled=False):
        ref = Fn.grid_sample(z.permute(0, 3, 1, 2), uv[:, :, None], align_corners=True)[:, 0, :, 0]
    d = ulps(out[fin], ref[fin])
    worst = int(d.max()) if d.numel() else 0
    assert worst <= 2, worst
    ref_dnn = Fn.grid_sample(z.permute(0, 3, 1, 2), uv[:, :, None], align_corners=True)[:, 0, :, 0]
    tv = torch.where(tz == -1, fill[:, None, None].expand_as(tz), tz)
    spread = torch.where(ok, tv, torch.zeros_like(tv)).amax(-1) - torch.where(ok, tv, torch.zeros_like(tv)).amin(-1)
    tol = 2.0 ** -22 * (4 * ref_dnn.abs() + spread.abs() * max(H, W))
    dd = (out - ref_dnn).abs()
    assert (dd[fin] <= tol[fin]).all(), float((dd - tol)[fin].max())
    return worst, int(ok.sum()), float(dd[fin].max()) if dd[fin].numel() else 0.0


@pytest.fixture(scope="module")
def prod():
    return production_scene()


@pytest.mark.parametrize("Q", [1, 800, 100_000])
@pytest.mark.parametrize("mesh", ["garment", "body"])
def test_taps_bit_identical_production(prod, Q, mesh):
    (verts, faces) = prod[0] if mesh == "garment" else prod[1]
    cams = prod[2]
    N, H, W = verts.shape[0], 1080, 1080
    g = torch.Generator(device=DEV).manual_seed(Q)
    # half the queries on the mesh's own projected vertices (covered pixels), half anywhere on and around the image
    sp = raster.screen_points(verts, cams)
    idx = torch.randint(0, verts.shape[1], (N, Q), device=DEV, generator=g)
    on = torch.gather(sp, 1, idx[..., None].expand(N, Q, 3))[..., :2]
    anywhere = torch.rand((N, Q, 2), device=DEV, generator=g) * 1200 - 60
    pts = torch.where((torch.arange(Q, device=DEV) % 2 == 0)[None, :, None], on, anywhere).contiguous()
    ns = torch.tensor([[W, H]] * N, dtype=torch.float32, device=DEV)
    fill = torch.rand(N, device=DEV, generator=g) + 3
    ulp, taps, dnn = check_probe(verts, faces, cams, H, W, pts, ns, fill)
    print(f"\n{mesh} Q={Q}: {taps} taps bit-identical to rasterize_meshes; out vs ATen grid_sample max {ulp} ulp "
          f"({'bitwise' if ulp == 0 else 'within 2 ulp'}); vs the cuDNN dispatch max |diff| {dnn:.2e}")


def adversarial_scene(H, W):
    """Faces spanning the whole image, degenerate faces, faces crossing z_clip, off-screen faces, coplanar duplicates
    (ties go to the lower index) and an out-of-range index, on one camera looking down +z from the origin."""
    f = 1.0 * W
    cam = (torch.tensor([[f, f]]), torch.tensor([[W / 2.0, H / 2.0]]), torch.eye(3)[None], torch.zeros(1, 3))
    V, F = [], []

    def tri(a, b, c):
        F.append([len(V), len(V) + 1, len(V) + 2])
        V.extend([a, b, c])

    tri((-30, -30, 5), (30, -30, 5), (0, 40, 5))            # spans the image
    tri((-30, -30, 4), (30, -30, 6), (0, 40, 4.5))          # spans it too, tilted
    tri((0.1, 0.1, 3), (0.2, 0.2, 3), (0.3, 0.3, 3))        # degenerate (collinear)
    tri((0, 0, 2), (0, 0, 2), (0.1, 0, 2))                  # degenerate (repeated vertex)
    tri((-0.5, -0.2, 2), (0.5, -0.2, -1), (0, 0.5, 2))      # crosses z_clip
    tri((50, 50, 3), (60, 50, 3), (55, 60, 3))              # off-screen
    for k in range(3):                                      # coplanar copies: the lowest index wins
        tri((-0.4, -0.4, 3), (0.4, -0.4, 3), (0, 0.4, 3))
    tri((-0.2, 0.0, 2.5), (0.3, -0.3, 3.5), (0.1, 0.4, 2.8))
    verts = torch.tensor([V], dtype=torch.float32)
    faces = torch.tensor(F + [[0, 1, 10 ** 6]], dtype=torch.int64)  # an index outside [0, V): skipped
    return verts.to(DEV), faces.to(DEV), tuple(t.to(DEV) for t in cam)


@pytest.mark.parametrize("HW", [(64, 96), (37, 29)])
def test_taps_bit_identical_adversarial(HW):
    H, W = HW
    verts, faces, cam = adversarial_scene(H, W)
    ns = torch.tensor([[W, H]], dtype=torch.float32, device=DEV)
    # pixel centres (sx = c * W / (W - 1) lands on ix = c up to rounding), tile edges, border, outside, NaN, and
    # 2000 queries in one pixel
    cs = torch.arange(-1, W + 1, dtype=torch.float32)
    rs = torch.arange(-1, H + 1, dtype=torch.float32)
    cc, rr = torch.meshgrid(cs * W / (W - 1), rs * H / (H - 1), indexing="xy")
    centres = torch.stack([cc.reshape(-1), rr.reshape(-1)], -1)
    tiles = torch.tensor([[32 * k - 0.5, 8 * j + 7.5] for k in range(4) for j in range(8)], dtype=torch.float32)
    one = torch.full((2000, 2), 0.0) + torch.tensor([W / 2 + 0.25, H / 2 - 0.3])
    special = torch.tensor([[float("nan"), 3.0], [3.0, float("inf")], [1e30, 1e30], [-1e9, 5.0], [0.0, 0.0],
                            [float(W), float(H)]])
    pts = torch.cat([centres, tiles, one, special])[None].to(DEV).contiguous()
    fill = torch.tensor([7.5], device=DEV)
    for z_clip in (1e-6, 2.5, -2.0):
        ulp, taps, dnn = check_probe(verts, faces, cam, H, W, pts, ns, fill, z_clip=z_clip)
        print(f"\nadversarial {H}x{W} z_clip={z_clip}: {taps} taps bit-identical; out vs ATen max {ulp} ulp, "
              f"vs cuDNN max |diff| {dnn:.2e}")


def test_run_to_run_identity(prod):
    (verts, faces), _, cams = prod
    N = verts.shape[0]
    g = torch.Generator(device=DEV).manual_seed(3)
    pts = (torch.rand((N, 50_000, 3), device=DEV, generator=g) * 1080).contiguous()
    ns = torch.tensor([[1080., 1080.]] * N, device=DEV)
    fill = torch.ones(N, device=DEV)
    a = raster.zbuf_probe(verts, faces, cams, (1080, 1080), pts, ns, fill, return_taps=True)
    b = raster.zbuf_probe(verts, faces, cams, (1080, 1080), pts, ns, fill, return_taps=True)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8))


# ---- the drop-ins on the fixture's inputs --------------------------------------------------------------------------

def _case(name):
    z = load_golden("zbuf_ref.npz")
    p = name + "/"
    return {k[len(p):]: v for k, v in z.items() if k.startswith(p)}


def _fixture_call(s):
    import importlib.util
    import os
    from conftest import GOLDEN
    spec = importlib.util.spec_from_file_location("make_golden_zbuf", os.path.join(GOLDEN, "make_golden_zbuf.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    N, H, W = int(s["N"]), int(s["H"]), int(s["W"])
    cam_cpu, def_fl_vs, cano, check_pts = gen.inputs({k: (int(v) if v.ndim == 0 and k in "NHW" else v)
                                                     for k, v in s.items()})
    cam = cam_cpu.to(DEV)
    d = lambda t: t.to(DEV)  # noqa: E731
    me = types.SimpleNamespace(maskRender=mask_renderer((H, W), cameras=cam), deformer=zo.GarmentDeformer(),
                               garment_vs=[d(torch.tensor(s["garm_v"]))], garment_fs=[d(torch.tensor(s["garm_f"]))],
                               tmpBodyVs=d(torch.tensor(s["body_v"])), tmpBodyFs=d(torch.tensor(s["body_f"])))
    args = (cam, [None, d(torch.tensor(s["cond"]))], d(torch.tensor(s["poses"])), {"sdfRatio": float(s["ratio"])}, {},
            [d(t) for t in def_fl_vs], [d(t) for t in cano], [str(x) for x in s["fl_names"]], 0, str(s["garment"]),
            d(torch.tensor([[float(W), float(H)]] * N)), N)
    chk_args = (zo.Meshes([d(torch.tensor(s["body_v"]))], [d(torch.tensor(s["body_f"]))]), N, zo.BodySkin(),
                d(torch.tensor(s["poses"])), d(torch.tensor(s["trans"])), cam, mask_renderer((H, W)),
                d(torch.tensor([[float(W), float(H)]] * N)), d(torch.tensor(s["check_screen"])))
    return me, args, chk_args


@pytest.mark.parametrize("name", ["n1_square", "n3_wide"])
def test_dropins_match_reference_fixture(name):
    s = _case(name)
    me, args, chk_args = _fixture_call(s)
    vis = ru.fl_visible_by_body_zbuff(me, *args).cpu().numpy()
    chk = ru.check_zbuf_body(*chk_args).cpu().numpy()
    assert "upper" in me.deformer.offset                    # the translator's side effect still happens
    assert chk_args[6].rasterizer.cameras is chk_args[5]    # and check_zbuf_body's camera assignment
    # the screen points differ from the reference camera's NDC round trip in the last bits, which moves a sample
    # across a depth step by up to ~1e-4; ambiguous queries (oracle) are excepted
    ok = ~s["vis_amb"]
    err = np.abs(vis - s["vis"])[ok]
    print(f"\n{name}: visibility max |err| {err.max():.2e} median {np.median(err):.2e} over {ok.sum()} values")
    assert err.max() < 5e-4 and np.median(err) < 1e-6
    ok = ~s["check_amb"]
    err = np.abs(chk - s["check"])[ok]
    print(f"{name}: check_zbuf_body max |err| {err.max():.2e} over {ok.sum()} values")
    assert err.max() < 1e-4 and np.median(err) < 1e-6
    # the masks the call site builds: identical except within the tolerance of the threshold
    P0 = s["fl0"].shape[0]
    thr = np.full(vis.shape[1], ZBUF_THRESHOLD[str(s["fl_names"][1])])
    thr[:P0] = ZBUF_THRESHOLD[str(s["fl_names"][0])]
    near = np.abs(s["vis"] - thr[None, :, None]) < 5e-4
    differ = (vis < thr[None, :, None]) != (s["vis"] < thr[None, :, None])
    assert not (differ & ~near & ~s["vis_amb"]).any()
    excepted = int((near | s["vis_amb"]).sum())
    print(f"{name}: masks identical; {excepted} of {near.size} values excepted (near threshold or ambiguous)")
    assert excepted <= 0.05 * near.size


def _restated_reference(me, cam, def_fl_vs, cano, poses, cond, ps, N):
    """The reference's fl_visible_by_body_zbuff flow on the GPU: full frames through the compat maskRender, fill,
    grid_sample; screen points from raster.screen_points so that only the z-buffer path differs."""
    c_z = cam.cam_pos()[2]
    cols = []
    gv = me.deformer(me.garment_vs[0][None].expand(N, -1, 3), [cond, poses])
    fl = torch.cat(def_fl_vs, 1)
    body = me.deformer.defs[1](me.tmpBodyVs[None].expand(N, -1, 3), poses)
    sfl = torch.cat([me.deformer.defs[1](c.expand(N, -1, 3), poses) for c in cano], 1)
    for verts, faces, q in ((gv, me.garment_fs[0], fl), (body, me.tmpBodyFs, sfl)):
        z = me.maskRender(zo.Meshes(list(verts), [faces] * N))[1].zbuf
        fill = (verts[..., -1] - c_z).max(-1)[0]
        z[z == -1.] = fill[:, None, None, None].expand_as(z)[z == -1.]
        sp = raster.screen_points(q, cam)
        uv = torch.stack([2 * sp[..., 0] / ps[:, None, 0] - 1, 2 * sp[..., 1] / ps[:, None, 1] - 1], -1)
        s = Fn.grid_sample(z.permute(0, 3, 1, 2), uv[:, :, None], align_corners=True)[:, 0, :, 0]
        cols.append(q[..., -1] - (s + c_z))
    return torch.stack(cols, -1)


@pytest.mark.parametrize("name", ["n1_square", "n3_wide"])
def test_dropins_match_restated_flow_without_host_sync(name):
    s = _case(name)
    me, args, chk_args = _fixture_call(s)
    cam, conds, poses, _, _, def_fl_vs, cano, _, _, _, ps, N = args
    ru.fl_visible_by_body_zbuff(me, *args)           # warm: library load and workspaces
    ru.check_zbuf_body(*chk_args)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        vis = ru.fl_visible_by_body_zbuff(me, *args)
        chk = ru.check_zbuf_body(*chk_args)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert not vis.requires_grad and not chk.requires_grad
    ref = _restated_reference(me, cam, def_fl_vs, cano, poses, conds[1], ps, N)
    d = (vis - ref).abs().max().item()
    print(f"\n{name}: drop-in vs restated flow max |diff| {d:.2e}")
    assert d <= 4e-6 * (1 + ref.abs().max().item())
    meshes, N_, skin, poses_, trans, cam_, mr, img, screen = chk_args
    bv = skin(meshes.verts_packed()[None].expand(N_, -1, 3), [poses_, trans])
    z = mr(zo.Meshes(list(bv), [meshes.faces_packed()] * N_))[1].zbuf
    z[z == -1.] = bv[..., -1].max(-1)[0][:, None, None, None].expand_as(z)[z == -1.]
    uv = torch.stack([2 * screen[..., 0] / img[:, None, 0] - 1, 2 * screen[..., 1] / img[:, None, 1] - 1], -1)
    with torch.backends.cudnn.flags(enabled=False):
        ref = Fn.grid_sample(z.permute(0, 3, 1, 2), uv[:, :, None], align_corners=True)[:, 0, :, 0]
    assert int(ulps(chk, ref).max()) <= 2


def test_cpu_tensors_refused():
    v = torch.zeros(1, 3, 3)
    f = torch.tensor([[0, 1, 2]])
    cam = (torch.ones(1, 2), torch.zeros(1, 2), torch.eye(3)[None], torch.zeros(1, 3))
    with pytest.raises(RuntimeError):
        raster.zbuf_probe(v, f, cam, (8, 8), torch.zeros(1, 4, 2), torch.ones(1, 2), torch.zeros(1))
    with pytest.raises(RuntimeError):   # faces on the host with everything else on the device
        raster.zbuf_probe(v.to(DEV), f, cam, (8, 8), torch.zeros(1, 4, 2, device=DEV), torch.ones(1, 2, device=DEV),
                          torch.zeros(1, device=DEV))
