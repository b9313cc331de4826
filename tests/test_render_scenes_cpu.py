"""Each scene of tests/render_scenes.py contains what it claims, in the kernels' own float32 arithmetic
(tests/render_f32.py).  No GPU."""
import numpy as np
import pytest

import render_f32 as rf
import render_scenes as rs


def test_mesh_tile_lists_hold_exactly_the_claimed_record_counts():
    sc = rs.mesh_tile_counts()
    ty, tx = sc["claims"]["tile"]
    seen = set()
    for n, c in enumerate(sc["claims"]["counts"]):
        r = rf.make_face_rec(sc["verts"][n], sc["faces"], sc["cams"][n], sc["H"], sc["W"], sc["z_clip"],
                             sc["area_eps"])
        h = rf.tile_hist(r["x0"], r["x1"], r["y0"], r["y1"], sc["H"], sc["W"])
        assert h[ty, tx] == c, (n, c, h)
        assert h.sum() > h[ty, tx]          # the straddling faces land elsewhere
        seen.add(c % 32)
    assert {0, 1, 31} <= seen
    assert {255, 256, 257, 511, 512, 513} <= set(sc["claims"]["counts"])


def test_adversarial_mesh_reaches_huge_screen_coordinates_slivers_and_full_image_faces():
    sc = rs.mesh_adversarial(1e-6)
    r = rf.make_face_rec(sc["verts"][0], sc["faces"], sc["cams"][0], sc["H"], sc["W"], sc["z_clip"], sc["area_eps"])
    kept = r["keep"]
    big = np.maximum(np.abs(r["sx"]), np.abs(r["sy"])).max(1)
    assert big[kept].max() >= 1e6 and (big[kept] >= 1e6).sum() >= 4, big[kept].max()
    near = (r["z"] <= np.float32(1e-6) * np.float32(1 + 2.0 ** -19)).any(1)
    assert (kept & near).sum() >= 4                        # a vertex within 2^-19 relative above z_clip, still kept
    full = (r["x0"] == 0) & (r["x1"] == sc["W"] - 1) & (r["y0"] == 0) & (r["y1"] == sc["H"] - 1)
    assert full.sum() >= 2
    sx, sy = r["sx"].astype(np.float64), r["sy"].astype(np.float64)
    ln2 = np.max([(sx[:, i] - sx[:, (i + 1) % 3]) ** 2 + (sy[:, i] - sy[:, (i + 1) % 3]) ** 2 for i in range(3)], 0)
    aspect = ln2 / np.abs(r["A"].astype(np.float64))
    assert (kept & (aspect > 1e4)).sum() >= 10
    out = rf.rasterize_meshes(sc["verts"], sc["faces"], sc["cams"], sc["H"], sc["W"], sc["z_clip"], sc["area_eps"])
    assert out["covered"] == sc["H"] * sc["W"]


def test_adversarial_mesh_ties_and_negative_clip():
    sc = rs.mesh_adversarial(-2.0)
    r = rf.make_face_rec(sc["verts"][0], sc["faces"], sc["cams"][0], sc["H"], sc["W"], sc["z_clip"], sc["area_eps"])
    assert (r["keep"] & (r["z"] <= 0).any(1)).sum() >= 3     # faces at and across view depth 0 are not clipped
    assert (r["keep"] & (r["z"] == -1).all(1)).sum() == 1
    # ... but the faces wholly at Z <= 0 win no pixel, and no zbuf <= 0 is produced (sum_j b_j / Z_j > 0 makes zbuf > 0)
    out = rf.rasterize_meshes(sc["verts"], sc["faces"], sc["cams"], sc["H"], sc["W"], sc["z_clip"], sc["area_eps"])
    won = np.unique(out["pix_to_face"][out["pix_to_face"] >= 0])
    assert not (r["z"][won] <= 0).all(1).any() and (out["zbuf"][out["pix_to_face"] >= 0] > 0).all()
    # coincident copies: five faces with the same vertices at the same depth, so the same zbuf where they cover
    sxy = np.concatenate([np.sort(r["sx"], 1), np.sort(r["sy"], 1)], 1)
    _, cnt = np.unique(sxy[r["vis"]], axis=0, return_counts=True)
    assert cnt.max() >= 5


def test_exact_edge_scene_puts_pixel_centres_on_edges():
    """The winners of many pixels have an exactly zero barycentric (the centre lies on one of their edges), and on
    many of those the face across the shared edge also covers the centre, so the coverage rule b >= 0 decides."""
    sc = rs.mesh_exact_edges()
    out = rf.rasterize_meshes(sc["verts"], sc["faces"], sc["cams"], sc["H"], sc["W"], sc["z_clip"], sc["area_eps"])
    hit = out["pix_to_face"] >= 0
    on_edge = (out["bary"] == 0).any(-1)
    assert on_edge.sum() > 0.2 * hit.sum(), on_edge.sum()
    # a pixel covered by two faces at once: restate coverage for every face at every centre of frame 0
    r = out["recs"][0]
    ncov = np.zeros(sc["H"] * sc["W"], np.int64)
    for f, col, row in rf._enumerate(r["x0"], r["x1"], r["y0"], r["y1"], np.nonzero(r["vis"])[0]):
        cov, _, _ = rf.shade(r["ka"][f], r["kb"][f], r["kc"][f], r["iz"][f], r["z"][f],
                             (col - r["x0"][f]).astype(np.float32), (row - r["y0"][f]).astype(np.float32))
        np.add.at(ncov, (row * sc["W"] + col)[cov], 1)
    assert (ncov >= 2).sum() > 0.1 * sc["H"] * sc["W"] and (ncov >= 4).any()
    # frame 1 has shared edges between depths 1 and 2
    assert set(np.unique(out["zbuf"][1])) >= {np.float32(1), np.float32(2)}


def test_many_frames_scene():
    sc = rs.mesh_many_frames()
    assert sc["verts"].shape[0] == 4096 and sc["H"] == sc["W"] == 1
    out = rf.rasterize_meshes(sc["verts"], sc["faces"], sc["cams"], 1, 1)
    assert 0 < out["covered"] < 4096


def test_points_crowd_pixels_have_the_claimed_cover_counts_and_ties_across_k():
    for K in (8, 64):
        sc = rs.points_crowd(K=K)
        H, W = sc["H"], sc["W"]
        c = rf.point_cover(sc["points"], H, W, sc["radius"])
        per = np.bincount(c["pix"], minlength=H * W)
        z = sc["points"][0, :, 2]
        for row, col, n in sc["claims"]["crowd"]:
            p = row * W + col
            assert per[p] == n, (K, row, col, per[p], n)
            if n > K:   # the K-th and (K+1)-th by (z, index) share z
                g = c["g"][c["pix"] == p]
                o = np.lexsort((g, z[g]))
                assert z[g[o[K - 1]]] == z[g[o[K]]], (K, n)
                assert z[g[o[K - 2]]] < z[g[o[K - 1]]]
        x0, x1, y0, y1, _ = rf.setup_bbox(sc["points"][0, :, 0], sc["points"][0, :, 1], H, W, sc["radius"])
        assert rf.tile_hist(x0, x1, y0, y1, H, W)[0, 0] == sum(rs.crowd_counts(K)) > 512
        assert [n for _, _, n in sc["claims"]["crowd"]][:2] == [K, K + 1]


def test_points_edges_scene_has_alpha_one_rim_points_and_special_values():
    sc = rs.points_edges()
    H, W = sc["H"], sc["W"]
    c = rf.point_cover(sc["points"], H, W, sc["radius"])
    r2 = c["r2"]
    assert (c["d"] == 0).sum() >= 12                                      # alpha exactly 1
    x, y = sc["points"][0, :, 0], sc["points"][0, :, 1]
    rim = 0
    for k in range(len(x)):
        cols, rows = np.arange(W), np.arange(H)
        d = rf.dist2(rf.pixel_ndc(cols, W)[None, :], rf.pixel_ndc(rows, H)[:, None], x[k], y[k])
        rim += bool((np.abs(d.astype(np.float64) - r2) <= 1e-6 * r2).any())
    assert rim >= 30
    z = sc["points"][0, :, 2]
    assert (z == np.inf).any() and (np.signbit(z) & (z == 0)).any() and ((z > 0) & (z < 1.2e-38)).any()
    f = sc["features"]
    assert (f == 0).any() and (f < 0).any() and (f == 1e4).any()
    # discs cross tile edges x = 32 k, y = 8 k and the image border
    x0, x1, y0, y1, on = rf.setup_bbox(x, y, H, W, sc["radius"])
    assert ((x0 // 32 != x1 // 32) & on).sum() > 5 and ((y0 // 8 != y1 // 8) & on).sum() > 5
    assert ((x0 == 0) & on).any() and ((x1 == W - 1) & on).any()


SCENES = {
    "sphere": lambda: rs.points_sphere(2, 200, 260, 0.01, 50, 1),
    "sphere_subpixel": lambda: rs.points_sphere(1, 300, 300, 0.002, 1, 2),
    "crowd": lambda: rs.points_crowd(),
    "edges": lambda: rs.points_edges(),
    "frames": lambda: rs.points_frames(),
    "big": lambda: rs.points_big_discs(),
}


@pytest.mark.parametrize("name", sorted(SCENES))
def test_every_covered_pixel_lies_in_the_setup_bbox_with_and_without_fma(name):
    """The setup kernel's disc bbox is computed with plain operations (a compiler may fuse the two product-sums), so
    the restatement enumerates a wider one; no covered pixel may fall outside the kernel's, however it was compiled."""
    sc = SCENES[name]()
    pts = sc["points"]
    N, P = pts.shape[:2]
    H, W = sc["H"], sc["W"]
    c = rf.point_cover(pts, H, W, sc["radius"])
    q = c["pix"] % (H * W)
    col, row = q % W, q // W
    x, y = pts[..., 0].reshape(-1), pts[..., 1].reshape(-1)
    for fc in (False, True):
        for fr in (False, True):
            x0, x1, y0, y1, on = rf.setup_bbox(x, y, H, W, sc["radius"], fc, fr)
            g = c["g"]
            assert on[g].all()
            assert ((col >= x0[g]) & (col <= x1[g]) & (row >= y0[g]) & (row <= y1[g])).all(), (name, fc, fr)
    print(f"[bbox {name}] {len(c['g'])} covering pairs inside the setup bbox in all four contractions")
