"""The image-space kernels bit for bit against their float32 restatement (tests/render_f32.py), on every pixel.

rasterize_meshes (pix_to_face, zbuf, bary, counts) and rasterize_points (images, idx, zbuf, dists, counts) must equal
the restatement on every pixel of every scene of tests/render_scenes.py, including the pixels the float64 oracles call
ambiguous (edges, rims, depth ties, the K-th / (K+1)-th boundary); rasterize_points_backward must equal it on every
point, with an unmasked random cotangent.  Zeros compare with ==: a +0 / -0 difference is not a finding; every other
value compares by its bits.  The float32 restatement itself is held to float64 by tests/test_render_f32_cpu.py.
"""
import time

import numpy as np
import pytest
import torch

import render_f32 as rf
import render_scenes as rs
from recmv_b200 import _lib, ops, raster, synth
from recmv_b200.model import LBSkinner

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    eq = (a.view(np.uint32) == b.view(np.uint32)) | ((a == 0) & (b == 0))
    return bool(eq.all()), int((~eq).sum())


def first_diff(a, b):
    a, b = np.asarray(a), np.asarray(b)
    eq = (a == b) | (np.isnan(a) & np.isnan(b)) if a.dtype.kind == "f" else (a == b)
    if a.dtype.kind == "f":
        eq &= (a.view(np.uint32) == b.astype(np.float32).view(np.uint32)) | ((a == 0) & (b == 0))
    i = np.argwhere(~eq)
    return None if not len(i) else (tuple(i[0]), a[tuple(i[0])], b[tuple(i[0])])


def t(x, dt=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x)).to(DEV, dt).contiguous()


# ---- mesh -----------------------------------------------------------------------------------------------------------
# The mesh dists are written with plain operations a compiler may contract, so they are held to float64 per entry:
# |d - d64| <= KAPPA_DISTS u S, S the running bound of render_f32.mesh_dists_bound.  About 3x the largest ratio
# measured on an H100 80GB HBM3 at 700 W (0.089, mc sphere N = 7 at 1080^2; printed by each mesh test).
KAPPA_DISTS = 0.3
_kappa = {"dists": 0.0}


def check_dists(dists, ref, verts, faces, cams, H, W):
    """Per-entry bound of the winner's dists on every covered pixel; -1 exactly on background."""
    p2f = ref["pix_to_face"]
    assert (dists[p2f < 0] == -1).all()
    Fn = faces.shape[0]
    worst = 0.0
    for n in range(p2f.shape[0]):
        row, col = np.nonzero(p2f[n] >= 0)
        if not len(row):
            continue
        f = p2f[n, row, col] - n * Fn
        b = rf.mesh_dists_bound(verts[n], faces, cams[n], f, col, row, H, W)
        d = dists[n, row, col].astype(np.float64)
        assert np.array_equal(np.isfinite(d), np.isfinite(b.v))
        m = np.isfinite(d)
        diff = np.abs(d[m] - b.v[m])
        with np.errstate(divide="ignore", invalid="ignore"):
            r = np.where(diff == 0, 0.0, diff / (rf.U * b.e[m]))
        worst = max(worst, float(r.max(initial=0.0)))
    _kappa["dists"] = max(_kappa["dists"], worst)
    return worst


def check_probe_taps(verts, faces, cams, H, W, ref, z_clip, area_eps, seed=0):
    """The sparse z-buffer probe's taps are bit-identical to the full rasterization (as restated) on this scene: queries
    at random positions over and around the image, and at every pixel centre of a small image."""
    from test_gpu_zbuf_probe import tap_pixels
    N = verts.shape[0]
    g = np.random.default_rng(seed)
    Q = min(4000, 4 * H * W)
    pts = np.stack([g.uniform(-1.5, W + 0.5, (N, Q)), g.uniform(-1.5, H + 0.5, (N, Q))], -1)
    pts[:, : min(Q, H * W), 0] = np.arange(min(Q, H * W)) % W
    pts[:, : min(Q, H * W), 1] = np.arange(min(Q, H * W)) // W % H
    ns = np.tile([[max(W - 1, 1), max(H - 1, 1)]], (N, 1))
    pts_t, ns_t = t(pts), t(ns)
    _, tz, tf = ops.zbuf_probe(t(verts), t(faces, torch.int64), t(cams), H, W, pts_t, ns_t,
                               torch.zeros(N, device=DEV), z_clip, area_eps, return_taps=True)
    cols, rows, ok = (a.cpu().numpy() for a in tap_pixels(pts_t, ns_t, H, W))
    n = np.broadcast_to(np.arange(N)[:, None, None], cols.shape)
    cc, rr = np.clip(cols, 0, W - 1), np.clip(rows, 0, H - 1)
    tz, tf = tz.cpu().numpy(), tf.cpu().numpy()
    assert np.array_equal(tf[ok], ref["pix_to_face"][n, rr, cc][ok])
    assert np.array_equal(tz[ok].view(np.uint32), ref["zbuf"][n, rr, cc][ok].view(np.uint32))
    assert (tz[~ok] == -1).all() and (tf[~ok] == -1).all()
    return int(ok.sum())


def check_mesh(verts, faces, cams, H, W, z_clip=1e-6, area_eps=1e-8, label="", capacity=None, probe=True):
    verts, faces, cams = np.asarray(verts, np.float32), np.asarray(faces, np.int64), np.asarray(cams, np.float32)
    t0 = time.time()
    ref = rf.rasterize_meshes(verts, faces, cams, H, W, z_clip, area_eps)
    tr = time.time() - t0
    runs = [None] + ([capacity] if capacity is not None else [])
    kd = 0.0
    taps = 0
    for cap in runs:
        p2f, zbuf, bary, dists, counts = ops.rasterize_meshes(t(verts), t(faces, torch.int64), t(cams), H, W, z_clip,
                                                              area_eps, want_dists=True, capacity=cap)
        p = p2f[..., 0].cpu().numpy()
        z = zbuf[..., 0].cpu().numpy()
        b = bary[..., 0, :].cpu().numpy()
        assert np.array_equal(p, ref["pix_to_face"]), (label, cap, first_diff(p, ref["pix_to_face"]))
        okz, nz = same_bits(z, ref["zbuf"])
        okb, nb = same_bits(b, ref["bary"])
        assert okz and okb, (label, cap, nz, nb, first_diff(z, ref["zbuf"]), first_diff(b, ref["bary"]))
        assert counts["covered"] == ref["covered"] and counts["skipped"] == ref["skipped"], (counts, ref["covered"])
        assert counts["pairs"] == ref["pairs"], (counts, ref["pairs"])
        kd = check_dists(dists[..., 0].cpu().numpy(), ref, verts, faces, cams, H, W)
        assert kd <= KAPPA_DISTS, (label, kd)
    if probe:
        taps = check_probe_taps(verts, faces, cams, H, W, ref, z_clip, area_eps)
    print(f"[mesh {label}] N={verts.shape[0]} {H}x{W} F={faces.shape[0]} covered={ref['covered']} "
          f"skipped={ref['skipped']} pairs={ref['pairs']}: bit-exact (restatement {tr:.1f} s); dists kappa {kd:.3f} "
          f"(bound {KAPPA_DISTS}); probe taps bit-exact ({taps} in the image)")
    return ref


def test_exact_edge_mesh_bit_exact():
    sc = rs.mesh_exact_edges()
    check_mesh(sc["verts"], sc["faces"], sc["cams"], sc["H"], sc["W"], label="exact edges", capacity=1)


def _skinner():
    Js, parents, init = synth.skeleton()
    ws = synth.skinning_voxel((17, 33, 21), seed=7)
    return LBSkinner(ws, [-1.1] * 3, [1.1] * 3, Js, parents, init_pose=init,
                     bbox_extend=torch.tensor(synth.BBOX_EXTEND), bbox_center=torch.tensor(synth.BBOX_CENTER)).to(DEV)


@pytest.fixture(scope="module")
def mc_sphere():
    """The 257^3 marching-cubes sphere of the existing renderer tests."""
    sdf = synth.sphere_sdf_grid(257, num=8, seed=3, device=DEV)
    h = 2.0 / 256
    verts, faces = ops.mc_gpu(sdf, h, h, h, -1.0, -1.0, -1.0, 0.0)
    return verts.float().contiguous(), faces


def deform(verts, N, seed):
    poses, trans = synth.poses_trans(N, seed=seed)
    V = verts.shape[0]
    with torch.no_grad():
        d = _skinner()(verts.repeat(N, 1), [poses.to(DEV), trans.to(DEV)],
                       torch.arange(N, device=DEV).repeat_interleave(V))
    return d.view(N, V, 3).contiguous()


@pytest.mark.parametrize("N,H,W,seed", [(7, 1080, 1080, 1), (64, 45, 77, 2)])
def test_mc_sphere_mesh_bit_exact(mc_sphere, N, H, W, seed):
    verts, faces = mc_sphere
    d = deform(verts, N, seed).cpu().numpy()
    check_mesh(d, faces.cpu().numpy(), rs.cameras(N, H, W, seed), H, W, label=f"mc sphere N={N}")


def test_tile_counts_mesh_bit_exact():
    sc = rs.mesh_tile_counts()
    check_mesh(sc["verts"], sc["faces"], sc["cams"], sc["H"], sc["W"], label="tile counts", capacity=1)


@pytest.mark.parametrize("z_clip", [1e-6, 0.5, -2.0])
def test_adversarial_mesh_bit_exact(z_clip):
    sc = rs.mesh_adversarial(z_clip)
    check_mesh(sc["verts"], sc["faces"], sc["cams"], sc["H"], sc["W"], z_clip=z_clip, label=f"adversarial {z_clip}",
               capacity=1)


def test_many_one_pixel_frames_bit_exact():
    sc = rs.mesh_many_frames()
    check_mesh(sc["verts"], sc["faces"], sc["cams"], sc["H"], sc["W"], label="4096 frames of 1x1")


def test_measured_dists_kappa_printed():
    print(f"[mesh dists] largest measured kappa over the mesh tests run: {_kappa['dists']:.3f} (bound {KAPPA_DISTS})")


# ---- points ---------------------------------------------------------------------------------------------------------
def check_points(points, features, H, W, radius, K, split, label="", seed=0, capacity=None):
    """split None renders one image (every point in it); an int renders two."""
    points = np.asarray(points, np.float32)
    N, P = points.shape[:2]
    G = 1 if split is None else 2
    t0 = time.time()
    sel = rf.rasterize_points(points, features, H, W, radius, K, split)
    img_ref = rf.composite(sel, G)
    idx_ref, zb_ref, ds_ref = rf.fragments(sel)
    cot = np.random.default_rng(seed).normal(size=(G, N, H, W)).astype(np.float32)
    g_ref = rf.points_backward(sel, cot)
    tr = time.time() - t0
    pt = t(points)
    ft = None if features is None else t(features)
    for cap in [None] + ([capacity] if capacity is not None else []):
        images, (idx, zb, ds), counts, ws = ops.rasterize_points(pt, ft, H, W, radius, K, split, want_fragments=True,
                                                                 capacity=cap)
        assert np.array_equal(idx.cpu().numpy(), idx_ref), (label, first_diff(idx.cpu().numpy(), idx_ref))
        for name, a, b in (("images", images.cpu().numpy(), img_ref), ("zbuf", zb.cpu().numpy(), zb_ref),
                           ("dists", ds.cpu().numpy(), ds_ref)):
            ok, nbad = same_bits(a, b)
            assert ok, (label, name, nbad, first_diff(a, b))
        assert counts["skipped"] == sel["skipped"]
        assert counts["covered"] == int((sel["count"] > 0).sum())
        grad = ops.rasterize_points_backward(t(cot), ws, counts["pairs"], N, P, H, W, radius, K, split).cpu().numpy()
        ok, nbad = same_bits(grad, g_ref)
        assert ok, (label, "grad", nbad, first_diff(grad, g_ref))
    print(f"[points {label}] N={N} P={P} {H}x{W} r={radius:.4g} K={K} split={split} entries={len(sel['pix'])} "
          f"pairs={counts['pairs']}: bit-exact forward and backward (restatement {tr:.1f} s)")
    return sel


@pytest.mark.parametrize("K,r", [(1, 0.0015), (8, 0.006), (50, 0.006), (64, 0.015)])
def test_mc_sphere_points_bit_exact(mc_sphere, K, r):
    H = W = 1080
    verts, _ = mc_sphere
    d = deform(verts, 1, 4)
    cam = torch.as_tensor(rs.cameras(1, H, W, 4), device=DEV)
    ndc = raster.project_points(d, cam, H, W).cpu().numpy()
    P = ndc.shape[1]
    check_points(ndc, None, H, W, r, K, P // 2, label=f"mc sphere K={K}")


def test_crowd_points_bit_exact():
    for K in (8, 64):
        sc = rs.points_crowd(K=K)
        check_points(sc["points"], sc["features"], sc["H"], sc["W"], sc["radius"], sc["K"], sc["split"],
                     label=f"crowd K={K}", capacity=1)


def test_edge_points_bit_exact():
    sc = rs.points_edges()
    check_points(sc["points"], sc["features"], sc["H"], sc["W"], sc["radius"], sc["K"], sc["split"], label="edges",
                 capacity=1)


@pytest.mark.parametrize("split", [0, 1, 199, 200])
def test_many_frames_split_bit_exact(split):
    sc = rs.points_frames(split=split)
    check_points(sc["points"], sc["features"], sc["H"], sc["W"], sc["radius"], sc["K"], sc["split"],
                 label=f"64 frames split={split}")


@pytest.mark.parametrize("name", ["edges", "crowd", "frames"])
def test_single_image_path_bit_exact(name):
    sc = {"edges": rs.points_edges, "crowd": lambda: rs.points_crowd(64), "frames": lambda: rs.points_frames()}[name]()
    check_points(sc["points"], sc["features"], sc["H"], sc["W"], sc["radius"], sc["K"], None, label=f"{name} G=1")


def test_big_discs_k64_bit_exact():
    sc = rs.points_big_discs()
    check_points(sc["points"], sc["features"], sc["H"], sc["W"], sc["radius"], sc["K"], sc["split"],
                 label="big discs K=64", capacity=1)


def test_pair_limit_raises_range_and_keeps_the_workspace_small():
    """32768 points whose discs cover all 65536 tiles of a 4096 x 4096 frame: 2^31 (tile, point) pairs, one more than
    the list can index.  The scan saturates the count at 2^31 - 1 and the call raises RECMV_E_RANGE; a later call's
    workspace is sized by its own pairs, not by the saturated count."""
    H = W = 4096
    P = 32768
    g = torch.Generator().manual_seed(0)
    pts = torch.stack([torch.rand(P, generator=g) * 0.1 - 0.05, torch.rand(P, generator=g) * 0.1 - 0.05,
                       torch.rand(P, generator=g) + 0.5], 1)[None].to(DEV).contiguous()
    t0 = time.time()
    with pytest.raises(_lib.RecmvError) as e:
        ops.rasterize_points(pts, None, H, W, 1.6, 4)
    torch.cuda.synchronize()
    dt = time.time() - t0
    small = torch.zeros(1, 8, 3, device=DEV)
    small[..., 2] = 1
    _, _, counts, ws = ops.rasterize_points(small, None, 16, 16, 0.2, 4)
    print(f"[points pair limit] 2^31 pairs -> {e.value} in {dt:.2f} s; next call's workspace {ws.numel()} bytes")
    assert ws.numel() < 1 << 24
