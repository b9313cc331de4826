"""CPU: the float64 rasterizer oracle (oracle/raster_oracle.py) on hand-built scenes with known answers, and its tie to
the reference camera: every covered pixel's perspective-correct barycentric point lies on CameraMine.view_rays from
CameraMine.cam_pos.  The CUDA rasterizer is compared with this oracle in tests/test_gpu_raster.py."""
import numpy as np

from oracle import raster_oracle as ro

# fx = fy = 1, principal point 0, R = I, T = 0: at Z = 1 a vertex's screen position is exactly (-X, -Y)
UNIT = np.array([1, 1, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], dtype=np.float64)


def tri(screen, z=1.0):
    """World vertices (R = I, T = 0, unit camera) whose screen positions are `screen` at depth z."""
    s = np.asarray(screen, dtype=np.float64)
    return np.stack([-s[:, 0] * z, -s[:, 1] * z, np.full(len(s), z)], 1)


def run(tris, H=16, W=16, cams=None, **kw):
    verts = np.concatenate(tris)[None]
    faces = np.arange(verts.shape[1]).reshape(-1, 3)
    return ro.rasterize(verts, faces, [UNIT] if cams is None else cams, H, W, **kw)


def test_single_triangle_pixel_count():
    r = run([tri([(0.5, 0.5), (10.5, 0.5), (0.5, 10.5)], 2.0)])
    cov = r["pix_to_face"][0] >= 0
    assert cov.sum() == 55                    # centres (c, r), c, r >= 1, c + r <= 11 (the hypotenuse's centres count)
    rows, cols = np.nonzero(cov)
    assert rows.min() == 1 and cols.min() == 1 and (rows + cols).max() == 11
    assert np.allclose(r["zbuf"][0][cov], 2.0, rtol=1e-14) and np.all(r["zbuf"][0][~cov] == -1)
    assert np.allclose(r["bary"][0][cov].sum(-1), 1, atol=1e-12) and np.all(r["bary"][0][~cov] == -1)
    assert np.all(r["dists"][0][cov] <= 0) and np.all(r["dists"][0][~cov] == -1)
    assert r["skipped"] == 0


def test_winding_does_not_matter():
    a = run([tri([(0.5, 0.5), (10.5, 0.5), (0.5, 10.5)])])
    b = run([tri([(0.5, 0.5), (0.5, 10.5), (10.5, 0.5)])])
    assert np.array_equal(a["pix_to_face"] >= 0, b["pix_to_face"] >= 0)


def test_nearer_of_two_overlapping_triangles_wins():
    far = tri([(-1, -1), (15, -1), (-1, 15)], 3.0)
    near = tri([(4.2, 4.2), (12.3, 4.7), (4.6, 12.1)], 2.0)
    for order in ((far, near), (near, far)):
        r = run(list(order))
        nf = 1 if order[0] is far else 0
        p, z = r["pix_to_face"][0], r["zbuf"][0]
        inner = p == nf
        assert inner.sum() > 20 and np.allclose(z[inner], 2.0)
        assert np.allclose(z[(p >= 0) & ~inner], 3.0, rtol=1e-14)


def test_shared_edge_through_pixel_centres():
    # a square split along its diagonal: the diagonal's centres lie on both faces at equal depth -> the lower index
    a = tri([(2, 2), (12, 2), (2, 12)])
    b = tri([(12, 2), (12, 12), (2, 12)])
    r = run([a, b], ztol=0.0)
    p = r["pix_to_face"][0]
    assert (p >= 0).sum() == 11 * 11                              # no gap, no double count
    diag = np.array([[rr + cc == 14 for cc in range(16)] for rr in range(16)]) & (p >= 0)
    assert diag.sum() == 11 and np.all(p[diag] == 0) and np.all(r["tie"][0][diag])
    assert np.all(r["tie"][0][~diag] == False)  # noqa: E712


def test_exact_z_tie_goes_to_lower_index():
    t = tri([(1.3, 0.7), (13.2, 2.9), (3.1, 14.4)], 1.5)
    r = run([t, t.copy(), t.copy()])
    p = r["pix_to_face"][0]
    assert (p >= 0).sum() > 50 and np.all(p[p >= 0] == 0) and np.all(r["tie"][0][p >= 0])


def test_behind_camera_and_zero_area_faces_are_skipped():
    behind = tri([(1, 1), (14, 1), (1, 14)], 1.0)
    behind[1, 2] = -0.5                                   # one vertex behind the camera
    on_plane = tri([(1, 1), (14, 1), (1, 14)], 1.0)
    on_plane[2, 2] = 0.0                                  # Z = 0 <= z_clip
    flat = tri([(1, 1), (8, 8), (14, 14)], 1.0)           # collinear: zero area
    r = run([behind, on_plane, flat])
    assert r["skipped"] == 3 and np.all(r["pix_to_face"] == -1)


def test_face_straddling_the_image_border():
    r = run([tri([(-20.5, 3.5), (30.5, 3.5), (5.0, 40.0)])], H=8, W=10)
    p = r["pix_to_face"][0]
    # rows 4..7 inside the 8 x 10 image; at row r the face spans x in [-20.5 + (r-3.5)*25.5/36.5, 30.5 - ...]
    assert np.all(p[:4] == -1) and np.all(p[4:] == 0)


def test_off_screen_face_is_not_skipped_but_covers_nothing():
    r = run([tri([(40, 40), (50, 40), (40, 50)])])
    assert r["skipped"] == 0 and np.all(r["pix_to_face"] == -1)


def test_seed_points_lie_on_the_reference_view_rays():
    """CameraMine.view_rays (:146-167) from cam_pos (:207-208) passes through every covered pixel's perspective-correct
    barycentric point: this is what makes the fragments the reference camera's."""
    g = np.random.default_rng(5)
    H, W = 60, 80
    cams, verts = [], []
    for n in range(2):
        Q = np.linalg.qr(g.standard_normal((3, 3)))[0]
        Q *= np.sign(np.linalg.det(Q))
        T = np.array([0.1, -0.2, 3.0]) + 0.1 * g.standard_normal(3)
        cams.append(np.concatenate([[70.0 + 10 * n, 66.0, W / 2 + 1.3, H / 2 - 0.7], Q.reshape(-1), T]))
        # points in front of the camera: view-space samples mapped back to world space, X = (X_v - T) R^T
        Xv = np.stack([g.uniform(-1.2, 1.2, 300), g.uniform(-0.9, 0.9, 300), g.uniform(2.0, 4.0, 300)], 1)
        verts.append((Xv - T) @ Q.T)
    verts = np.stack(verts)
    faces = g.integers(0, 300, (400, 3))
    r = ro.rasterize(verts, faces, cams, H, W)
    pts = ro.seed_points(verts, faces, r["pix_to_face"], r["bary"])
    total = 0
    for n in range(2):
        rows, cols = np.nonzero(r["pix_to_face"][n] >= 0)
        d = ro.view_rays(cols.astype(np.float64), rows.astype(np.float64), cams[n])
        c = ro.cam_pos(cams[n])
        v = pts[n][rows, cols] - c
        off = np.linalg.norm(np.cross(v, d), axis=1) / np.linalg.norm(v, axis=1)
        assert off.max() < 1e-9 and np.all((v * d).sum(1) > 0)        # on the ray, in front of the camera
        # and the depth of that point is the pixel's zbuf
        _, _, _, _, R, T = ro.camera_tuple(cams[n])
        assert np.allclose((pts[n][rows, cols] @ R + T)[:, 2], r["zbuf"][n][rows, cols], rtol=1e-12)
        total += len(rows)
    assert total > 1000


def test_ambiguity_margins_flag_edges_and_near_ties():
    a = tri([(2, 2), (12, 2), (2, 12)])
    b = tri([(12, 2), (12, 12), (2, 12)], 1.0 + 1e-9)
    r = run([a, b], margin_px=1e-3, ztol=1e-6)
    amb = r["ambiguous"][0]
    assert amb.sum() >= 11 + 2 * 11                            # the diagonal and the square's outer edges
    assert not amb[6, 5] and r["pix_to_face"][0][6, 5] == 0    # well inside face 0
