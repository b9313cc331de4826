"""Deterministic scenes for the image-space kernels (mesh rasterizer, point rasterizer), built on the CPU from seeds.

Each builder returns a dict with the kernel's arguments as float32 / int64 NumPy arrays plus `claims`, the properties
tests/test_render_scenes_cpu.py checks the scene really has (tile record counts, ties, rim distances and so on).
A claim holds for the kernel's own float32 arithmetic (tests/render_f32.py), not for an idealised one.
"""
import numpy as np

from render_f32 import pixel_ndc

f32 = np.float32


# ---- shared pieces --------------------------------------------------------------------------------------------------
def uv_sphere(n_lat, n_lon, seed, bumps=0.08):
    """A closed UV sphere of radius ~0.5 with seeded low-frequency bumps: verts [V,3] float64, faces [F,3]."""
    g = np.random.default_rng(seed)
    th = np.linspace(0, np.pi, n_lat + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    T, Pp = np.meshgrid(th, ph, indexing="ij")
    d = np.stack([np.sin(T) * np.cos(Pp), np.sin(T) * np.sin(Pp), np.cos(T)], -1).reshape(-1, 3)
    d = np.concatenate([[[0, 0, 1.0]], d, [[0, 0, -1.0]]])
    c = g.normal(size=(6, 3))
    r = 0.5 * (1 + bumps * np.tanh(np.sin(d @ c.T * 2.0).sum(1)))
    verts = d * r[:, None]
    faces = []
    ring = lambda i, j: 1 + i * n_lon + (j % n_lon)
    for j in range(n_lon):
        faces.append([0, ring(0, j), ring(0, j + 1)])
        faces.append([len(verts) - 1, ring(n_lat - 2, j + 1), ring(n_lat - 2, j)])
    for i in range(n_lat - 2):
        for j in range(n_lon):
            a, b, cc, dd = ring(i, j), ring(i, j + 1), ring(i + 1, j), ring(i + 1, j + 1)
            faces += [[a, cc, b], [b, cc, dd]]
    return verts, np.asarray(faces, np.int64)


def cameras(N, H, W, seed):
    """A camera row per frame {fx, fy, px, py, R row-major, T}: R near diag(-1, -1, 1), the body ~2.6 in front."""
    g = np.random.default_rng(seed)
    rows = []
    for n in range(N):
        a = g.normal(size=3) * 0.15
        Kx = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        Q = np.linalg.qr(np.eye(3) + Kx)[0]
        Q = Q * np.sign(np.diag(Q))
        R = np.diag([-1.0, -1.0, 1.0]) @ Q
        f = 0.9 * min(H, W) * (1 + 0.1 * (n % 8))
        T = np.array([0.02 * (n % 8), -0.03, 2.6 + 0.1 * (n % 8)])
        rows.append(np.concatenate([[f, f * 1.02, W / 2 - 0.5 + n % 8, H / 2 - 0.5 - n % 8], R.reshape(-1), T]))
    return np.stack(rows).astype(np.float32)


def deformed(verts, N, seed, amp=0.05):
    """N smooth, seeded deformations of verts: [N,V,3] float32."""
    g = np.random.default_rng(seed)
    out = []
    for _ in range(N):
        A = g.normal(size=(3, 3)) * amp
        w = g.normal(size=(3, 3)) * 2
        out.append(verts + np.sin(verts @ w) @ A + g.normal(size=3) * 0.02)
    return np.stack(out).astype(np.float32)


# A fixed screen camera for hand-placed screen-space triangles: R = diag(-1, -1, 1), T = 0, so a vertex at view depth
# z and screen (sx, sy) sits at world (-(px - sx) z / fx, -(py - sy) z / fy, z).
def screen_camera(H, W, fx=None):
    fx = float(0.8 * W if fx is None else fx)
    return np.array([fx, fx, W / 2 + 0.25, H / 2 - 0.25, -1, 0, 0, 0, -1, 0, 0, 0, 1, 0, 0, 0], np.float32)


def screen_to_world(s, z, cam):
    s = np.asarray(s, np.float64).reshape(-1, 2)
    z = np.asarray(z, np.float64).reshape(-1)
    fx, fy, px, py = (float(c) for c in cam[:4])
    return np.stack([-(px - s[:, 0]) * z / fx, -(py - s[:, 1]) * z / fy, z], 1)


# ---- mesh scenes ----------------------------------------------------------------------------------------------------
def mesh_sphere(N, H, W, seed, n_lat=60, n_lon=96):
    v, f = uv_sphere(n_lat, n_lon, seed)
    return dict(verts=deformed(v, N, seed), faces=f, cams=cameras(N, H, W, seed), H=H, W=W, z_clip=1e-6,
                area_eps=1e-8, claims={})


MESH_TILE_COUNTS = (255, 256, 257, 511, 512, 513, 1, 31, 32, 33, 63, 64)


def mesh_tile_counts(seed=5):
    """One frame per target count c: tile (1, 1) of a 24 x 96 image holds exactly c face records (small faces, each
    inside that tile's pixel rows and columns), with exact depth ties, coincident copies and faces straddling every
    neighbouring tile.  Frame n, c = MESH_TILE_COUNTS[n]; faces beyond c in a frame sit off-screen."""
    g = np.random.default_rng(seed)
    H, W = 24, 96
    cam = screen_camera(H, W)
    F = max(MESH_TILE_COUNTS) + 40
    verts = []
    for c in MESH_TILE_COUNTS:
        tri = np.empty((F, 3, 2))
        z = np.empty((F, 3))
        # faces around a pixel centre of tile (1, 1) (columns 32..63, rows 8..15), every vertex inside the tile
        cx = g.integers(33, 63, F) + g.uniform(-0.1, 0.1, F)
        cy = g.integers(9, 15, F) + g.uniform(-0.1, 0.1, F)
        ang = g.uniform(0, 2 * np.pi, (F, 1)) + np.array([0, 2.1, 4.2])
        rad = g.uniform(0.6, 0.85, (F, 1))
        tri[..., 0] = cx[:, None] + rad * np.cos(ang)
        tri[..., 1] = cy[:, None] + rad * np.sin(ang)
        z[:] = g.integers(8, 16, (F, 1)) / 4.0                  # a few depth levels: many exact ties
        tri[c // 2:c // 2 + 8] = tri[0]                         # coincident copies of face 0 (same depth)
        z[c // 2:c // 2 + 8] = z[0]
        tri[c:] = tri[c:] + np.array([5000.0, 0.0])             # the rest off-screen
        # 40 faces straddling tile edges away from tile (1, 1): x = 32 and x = 64 in tile rows 0 and 2
        s = slice(F - 40, F)
        tri[s, :, 0] = np.array([30.6, 33.4, 32.0]) + g.integers(0, 2, (40, 1)) * 32
        tri[s, :, 1] = np.array([2.0, 2.0, 5.5]) + g.integers(0, 2, (40, 1)) * 16
        z[s] = 1.0
        verts.append(screen_to_world(tri, z, cam))
    N = len(MESH_TILE_COUNTS)
    return dict(verts=np.stack(verts).astype(np.float32), faces=np.arange(F * 3).reshape(F, 3),
                cams=np.tile(cam, (N, 1)), H=H, W=W, z_clip=1e-6, area_eps=1e-8,
                claims=dict(tile=(1, 1), counts=MESH_TILE_COUNTS))


def mesh_adversarial(z_clip, seed=7):
    """Faces at the edges of the setup's arithmetic, 64 x 96, one frame:
    - a vertex at view depth z_clip (1 + 2^-20) (just kept) whose screen coordinates reach 1e6 .. 1e9,
    - slivers of aspect ratio 1e4, faces over the whole image, coincident copies and exact depth ties,
    - with z_clip < 0: faces at negative and zero-crossing view depth (one at depth exactly -1).  They are kept, but a
      covered pixel needs sum_j b_j / Z_j > 0, and then zbuf = sum_j b_j / sum_j (b_j / Z_j) > 0: the faces wholly at
      Z <= 0 win no pixel, and no zbuf <= 0 can be produced."""
    g = np.random.default_rng(seed)
    H, W = 64, 96
    cam = screen_camera(H, W)
    tris, zs = [], []
    # big faces
    tris += [[[-500, -400], [900, -300], [-200, 1200]], [[-50, -60], [300, 10], [20, 400]]]
    zs += [[2.0, 3.0, 2.5], [2.5, 2.5, 2.5]]
    # slivers: length ~ 60 px, width 6e-3 px
    for k in range(24):
        a = g.uniform(0, np.pi)
        c = g.uniform([10, 10], [W - 10, H - 10])
        u, n = np.array([np.cos(a), np.sin(a)]), np.array([-np.sin(a), np.cos(a)])
        tris.append([c - 30 * u, c + 30 * u, c + 6e-3 * n])
        zs.append(g.uniform(1.0, 3.0, 3))
    # coincident copies and exact ties
    base = [[20.3, 10.7], [60.2, 12.1], [35.5, 50.9]]
    for _ in range(4):
        tris.append(base)
        zs.append([1.5, 1.5, 1.5])
    tris.append([[20.3, 10.7], [35.5, 50.9], [60.2, 12.1]])     # opposite winding, same depth
    zs.append([1.5, 1.5, 1.5])
    verts = screen_to_world(np.asarray(tris, np.float64), np.asarray(zs, np.float64), cam)
    extra = []
    # near-clip vertices: view z = z_clip (1 + 2^-20) for z_clip > 0 (screen coordinates ~ 1e6..1e9)
    zc = float(z_clip)
    znear = zc * (1 + 2.0 ** -20) if zc > 0 else 1e-7
    for k in range(6):
        off = 10.0 ** (1.2 - k * 0.5)
        extra.append([[off, 0.3 * off, znear], [0.0, 0.0, 2.0], [0.1, -0.2, 2.2]])
        extra.append([[-off, 0.2 * off, znear], [0.3, 0.1, 2.0], [-0.1, 0.05, 1.8]])
    if zc < 0:
        # negative depths: the projection mirrors; a zero-crossing face; a face at depth exactly -1 (all kept; only the zero-crossing one can win, with zbuf > 0)
        extra.append([[0.3, 0.2, -0.5], [-0.2, 0.1, -0.6], [0.0, -0.3, -0.4]])
        extra.append([[0.3, 0.2, -0.5], [-0.2, 0.1, 0.6], [0.0, -0.3, 0.4]])
        extra.append([[0.5, 0.5, -1.0], [-0.5, 0.4, -1.0], [0.0, -0.6, -1.0]])
        extra.append([[0.05, 0.05, zc * (1 - 2.0 ** -20)], [-0.3, 0.1, -0.6], [0.1, -0.2, -0.7]])
    # world = view under R = diag(-1, -1, 1), T = 0
    ex = np.asarray(extra, np.float64).reshape(-1, 3) * np.array([-1.0, -1.0, 1.0])
    allv = np.concatenate([verts, ex])
    F = len(allv) // 3
    return dict(verts=allv[None].astype(np.float32), faces=np.arange(F * 3).reshape(F, 3), cams=cam[None],
                H=H, W=W, z_clip=zc, area_eps=1e-8, claims=dict(negative=zc < 0))


def mesh_many_frames(N=4096, seed=11):
    """N frames of a 1 x 1 image, one face each, covering the pixel in most frames (grid.y = N)."""
    g = np.random.default_rng(seed)
    cam = screen_camera(1, 1, fx=1.0)
    verts = []
    for n in range(N):
        c = g.uniform(-0.6, 0.6, 2)
        tri = c + g.uniform(-1.5, 1.5, (3, 2))
        verts.append(screen_to_world(tri, g.uniform(1, 4, 3), cam))
    return dict(verts=np.stack(verts).astype(np.float32), faces=np.array([[0, 1, 2]]), cams=np.tile(cam, (N, 1)),
                H=1, W=1, z_clip=1e-6, area_eps=1e-8, claims={})


def mesh_exact_edges(seed=29):
    """Faces whose edges pass exactly through pixel centres, 40 x 72, two frames.  The camera (fx = fy = 1, p = 0,
    R = I, T = 0) maps a vertex (X, Y, Z) to the screen point (-X / Z, -Y / Z), exactly for Z = 1 and Z = 2, so integer
    screen vertices stay integers.  A grid of unit-multiple quads, each split along a diagonal, puts pixel centres on
    horizontal, vertical and diagonal edges, each shared by two faces, so b = 0 exactly for one face and the winner is
    decided by depth, then by the lower index; frame 1 uses Z = 2 on every other quad, so some shared edges separate
    different depths."""
    g = np.random.default_rng(seed)
    H, W = 40, 72
    cam = np.array([1, 1, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], np.float32)
    frames = []
    for n in range(2):
        tris, zs = [], []
        for y0 in range(-2, H + 2, 6):
            for x0 in range(-3, W + 3, 7):
                w, h = int(g.integers(3, 8)), int(g.integers(3, 7))
                a, b, c, d = (x0, y0), (x0 + w, y0), (x0, y0 + h), (x0 + w, y0 + h)
                z = 2.0 if (n == 1 and (x0 + y0) % 2) else 1.0
                if g.integers(0, 2):
                    tris += [[a, b, d], [a, d, c]]
                else:
                    tris += [[a, b, c], [b, d, c]]
                zs += [z, z]
        tri = np.asarray(tris, np.float64)
        z = np.repeat(np.asarray(zs)[:, None], 3, 1)
        frames.append(np.stack([-tri[..., 0] * z, -tri[..., 1] * z, z], -1).reshape(-1, 3))
    F = len(frames[0]) // 3
    return dict(verts=np.stack(frames).astype(np.float32), faces=np.arange(3 * F).reshape(F, 3),
                cams=np.tile(cam, (2, 1)), H=H, W=W, z_clip=1e-6, area_eps=1e-8, claims={})


# ---- point scenes ---------------------------------------------------------------------------------------------------
def _ndc(col, row, H, W):
    return 1 - (2 * np.asarray(col, np.float64) + 1) / W, 1 - (2 * np.asarray(row, np.float64) + 1) / H


def points_sphere(N, H, W, radius, K, seed, n_lat=80, n_lon=128):
    """The deformed sphere's vertices projected to NDC; split = P // 2."""
    v, _ = uv_sphere(n_lat, n_lon, seed)
    d = deformed(v, N, seed).astype(np.float64)
    cams = cameras(N, H, W, seed).astype(np.float64)
    out = []
    for n in range(N):
        c = cams[n]
        vv = d[n] @ c[4:13].reshape(3, 3) + c[13:16]
        sx, sy = c[2] - c[0] * vv[:, 0] / vv[:, 2], c[3] - c[1] * vv[:, 1] / vv[:, 2]
        out.append(np.stack([1 - (2 * sx + 1) / W, 1 - (2 * sy + 1) / H, vv[:, 2]], 1))
    pts = np.stack(out).astype(np.float32)
    return dict(points=pts, features=None, H=H, W=W, radius=radius, K=K, split=pts.shape[1] // 2, claims={})


def crowd_counts(K):
    return (K, K + 1, 255, 256, 257)


def points_crowd(K=8, seed=13):
    """Pixel (row 3, col 5 + 6 j) of a 16 x 64 image is covered by exactly crowd_counts(K)[j] = K, K + 1, 255, 256 and
    257 points, with a depth tie across the K boundary: the first K - 1 points of a crowd lie in front (z <= 1/2),
    points K - 1 and K share z = 5/8 and the rest lie at z >= 5/8, so the K-th and (K+1)-th by (z, index) are points
    K - 1 and K, tied in z.  Every crowd point sits within 0.3 r of its pixel centre (r = 0.9 px across, 0.225 px down),
    so each crowd covers its own pixel only, and tile (0, 0)'s list holds every record (more than 512)."""
    g = np.random.default_rng(seed)
    H, W = 16, 64
    r = 0.9 * 2 / W
    pts, feats = [], []
    counts = crowd_counts(K)
    for j, c in enumerate(counts):
        x, y = _ndc(5 + 6 * j, 3, H, W)
        z = np.empty(c)
        z[:K - 1] = g.integers(1, 5, K - 1) / 8.0
        z[K - 1:K + 1] = 0.625
        z[K + 1:] = g.integers(5, 9, max(c - K - 1, 0)) / 8.0
        ox = g.uniform(-0.3, 0.3, c) * r
        oy = g.uniform(-0.3, 0.3, c) * r
        pts.append(np.stack([x + ox, y + oy, z], 1))
        feats.append(g.uniform(0.5, 1.5, c))
    pts = np.concatenate(pts)
    P = len(pts)
    return dict(points=pts[None].astype(np.float32), features=np.concatenate(feats)[None].astype(np.float32), H=H, W=W,
                radius=r, K=K, split=P // 3, claims=dict(crowd=[(3, 5 + 6 * j, c) for j, c in enumerate(counts)]))


def points_edges(seed=17):
    """96 x 72 image, r = 2.5 px: points exactly on pixel centres (alpha = 1), points whose squared distance to a pixel
    centre lies within 1e-6 r^2 of r^2 on either side, discs straddling x = 32 k and y = 8 k tile edges and the image
    border, features of 0, negative and 1e4, and z of +0, -0, +inf and a subnormal."""
    g = np.random.default_rng(seed)
    H, W = 72, 96
    r = 2.5 * 2 / W
    r2 = float(np.float32(r) * np.float32(r))
    P_ = []
    # on pixel centres
    for _ in range(12):
        c, rr = g.integers(0, W), g.integers(0, H)
        P_.append([pixel_ndc(c, W), pixel_ndc(rr, H), g.uniform(0.5, 2)])
    # near the rim of some pixel: d = r^2 (1 +- 1e-6 .. 1e-7)
    for k in range(40):
        c, rr = g.integers(2, W - 2), g.integers(2, H - 2)
        xf, yf = float(pixel_ndc(c, W)), float(pixel_ndc(rr, H))
        a = g.uniform(0, 2 * np.pi)
        rho = np.sqrt(r2 * (1 + (-1) ** k * 10.0 ** -g.uniform(6, 7.5)))
        P_.append([xf + rho * np.cos(a), yf + rho * np.sin(a), g.uniform(0.5, 2)])
    # tile edges and the border
    for cx in (31.5, 32.0, 63.7, -0.5, 95.2, 0.0, 96.3):
        for ry in (7.5, 8.0, 15.9, 71.4, -1.0, 35.0):
            P_.append([*_ndc(cx, ry, H, W), g.uniform(0.5, 2)])
    # special depths
    for z in (0.0, -0.0, np.inf, 1e-40, 2e-45):
        P_.append([*_ndc(g.uniform(5, 90), g.uniform(5, 65), H, W), z])
    pts = np.asarray(P_, np.float64)
    P = len(pts)
    feats = g.uniform(0.5, 1.5, P)
    feats[::7] = 0.0
    feats[1::7] = -g.uniform(0.1, 3.0, len(feats[1::7]))
    feats[2::11] = 1e4
    return dict(points=pts[None].astype(np.float32), features=feats[None].astype(np.float32), H=H, W=W, radius=r,
                K=6, split=P // 2, claims=dict(rim=40, centres=12))


def points_frames(N=64, P=200, split=None, seed=19, K=5):
    """N frames of the same small random cloud, 40 x 48, r = 1.6 px; split at `split`."""
    g = np.random.default_rng(seed)
    pts = np.stack([np.stack([g.uniform(-1.1, 1.1, P), g.uniform(-1.1, 1.1, P), g.uniform(0.5, 1.5, P)], 1)
                    for _ in range(N)])
    return dict(points=pts.astype(np.float32), features=g.uniform(0.2, 1.0, (N, P)).astype(np.float32), H=40, W=48,
                radius=1.6 * 2 / 48, K=K, split=P if split is None else split, claims={})


def points_big_discs(seed=23, K=64):
    """24 discs spanning many tiles (r from 0.05 to 0.7 in NDC) over 100 x 140, K = 64 with more than 64 covering
    points on most covered pixels."""
    g = np.random.default_rng(seed)
    P = 90
    pts = np.stack([g.uniform(-1, 1, P), g.uniform(-1, 1, P), g.uniform(0.5, 2.0, P)], 1)
    return dict(points=pts[None].astype(np.float32), features=g.uniform(0.2, 1, (1, P)).astype(np.float32), H=100,
                W=140, radius=0.45, K=K, split=P // 2, claims={})
