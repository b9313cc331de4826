"""Scenes of the shading tests (tests/test_gpu_shade_scale.py, tests/test_shade_f32_cpu.py): meshes with the hard
cases of the vertex normals and hand-built fragments with the hard cases of the Phong pass.  Seeded NumPy only."""
import numpy as np


def fan(K):
    """A [1,K+1,3] fan of K faces around vertex 0 (a vertex summing K contributions)."""
    th = np.linspace(0, 2 * np.pi, K, endpoint=False)
    ring = np.stack([np.cos(th), np.sin(th), 0.1 * np.sin(7 * th)], 1)
    v = np.concatenate([[[0.0, 0.0, 0.3]], ring])[None].astype(np.float32)
    i = np.arange(K)
    return v, np.stack([np.zeros(K, np.int64), 1 + i, 1 + (i + 1) % K], 1)


def uv_sphere(n_lat, n_lon, N, seed):
    """[N,V,3] noisy closed UV spheres with one face list."""
    g = np.random.default_rng(seed)
    th = np.linspace(0, np.pi, n_lat + 2)[1:-1]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    T, P = np.meshgrid(th, ph, indexing="ij")
    pts = np.stack([np.sin(T) * np.cos(P), np.sin(T) * np.sin(P), np.cos(T)], -1).reshape(-1, 3)
    pts = np.concatenate([pts, [[0, 0, 1], [0, 0, -1]]])
    V = len(pts)
    F = []
    for i in range(n_lat - 1):
        for j in range(n_lon):
            a, b = i * n_lon + j, i * n_lon + (j + 1) % n_lon
            F += [[a, b, a + n_lon], [b, b + n_lon, a + n_lon]]
    for j in range(n_lon):
        F += [[V - 2, (j + 1) % n_lon, j], [V - 1, (n_lat - 1) * n_lon + j, (n_lat - 1) * n_lon + (j + 1) % n_lon]]
    v = pts[None] * (1 + 0.05 * g.normal(size=(N, V, 1))) + 0.01 * g.normal(size=(N, V, 3))
    return v.astype(np.float32), np.asarray(F, np.int64)


def adversarial_mesh():
    """One [2,V,3] mesh with every hard case of the normals: a non-manifold edge shared by 4 faces, a face duplicated
    with both orientations (its corners' sums cancel exactly), slivers of aspect 1e4, coordinates around 1e-20
    (subnormal cross products) and 1e18 (the squared norm overflows), a NaN vertex, unreferenced vertices and faces
    with an index -1, V or 2^40."""
    g = np.random.default_rng(11)
    P, F = [], []

    def add(pts, tris):
        base = sum(len(p) for p in P)
        P.append(np.asarray(pts, np.float64))
        F.extend([[base + a, base + b, base + c] for a, b, c in tris])

    add([[0, 0, 0], [1, 0, 0], [0, 1, 0.2], [0, -1, 0.3], [0, 0.3, 1], [0, -0.2, -1]],
        [[0, 1, 2], [1, 0, 3], [0, 1, 4], [1, 0, 5]])                              # edge (0, 1) in 4 faces
    add(g.normal(size=(3, 3)), [[0, 1, 2], [0, 2, 1], [0, 1, 2]])                  # reversed and duplicated
    add(g.normal(size=(3, 3)), [[0, 1, 2], [0, 2, 1]])                             # a pair that cancels exactly
    add([[0, 0, 0], [1, 0, 0], [0.5, 1e-4, 0], [0.5, -1e-4, 1e-4]], [[0, 1, 2], [0, 3, 1]])   # slivers
    add(g.normal(size=(4, 3)) * 1e-20, [[0, 1, 2], [0, 2, 3]])                     # subnormal products
    add(g.normal(size=(4, 3)) * 1e18, [[0, 1, 2], [1, 3, 2]])                      # |n|^2 overflows
    add(g.normal(size=(4, 3)), [[0, 1, 2], [1, 3, 2]])                             # vertex 3 becomes NaN
    nan_v = sum(len(p) for p in P) - 1
    add(g.normal(size=(3, 3)), [])                                                 # unreferenced
    add(g.normal(size=(50, 3)), [[i, (i + 1) % 50, (i + 7) % 50] for i in range(50)])
    V = sum(len(p) for p in P)
    F += [[0, 1, V], [-1, 2, 3], [4, 1 << 40, 5], [V + 3, V + 4, V + 5]]
    v = np.concatenate(P)
    v = np.stack([v, v[::-1].copy() * 0.5 + 0.1])                                  # two frames
    v[0, nan_v, 1] = np.nan
    return v.astype(np.float32), np.asarray(F, np.int64)



def hand_fragments(seed=0):
    """Hand-built fragments over one small mesh, 8 frames of 64 x 64: random faces (some invalid or out of range) and
    barycentrics in [-1, 2] (negative and above 1), a face whose vertex normals cancel at its midpoint, a pixel whose
    point is the light, one whose point is the camera, and one with cos(N, L) exactly 0."""
    g = np.random.default_rng(seed)
    N, H, W, V = 8, 64, 64, 40
    verts = g.normal(size=(N, V, 3)).astype(np.float32)
    normals = g.normal(size=(N, V, 3)).astype(np.float32)
    colors = g.random((N, V, 3)).astype(np.float32)
    faces = g.integers(0, V, size=(30, 3))
    faces[5] = [0, 1, V]
    faces[6] = [-1, 1, 2]
    faces[7] = [3, 4, 5]
    normals[:, 4] = -normals[:, 3]                                     # face 7: normals cancel at b = (.5, .5, 0)
    faces[8] = [6, 7, 8]
    verts[:, 6] = 0
    normals[:, 6] = [0, 0, 1]                                          # face 8 at b = (1, 0, 0): p = 0, n = +z
    F = len(faces)
    p2f = g.integers(-2, N * F + 3, size=(N, H, W))
    bary = g.uniform(-1, 2, size=(N, H, W, 3)).astype(np.float32)
    for n in range(N):
        p2f[n, 0, :4] = n * F + np.array([7, 8, 8, 8])
        bary[n, 0, 0] = [0.5, 0.5, 0]
        bary[n, 0, 1:4] = [1, 0, 0]
    centre = np.tile([0.0, 0.0, 3.0], (N, 1))
    light = np.tile([0.4, -0.8, 1.5], (N, 1))
    centre[1] = 0                                                      # frame 1: camera at the point of (0, 1..3)
    light[2] = 0                                                       # frame 2: light at that point
    light[3] = [1, 0, 0]                                               # frame 3: L = +x, N = +z: cos exactly 0
    return p2f, bary, verts, normals, colors, faces, centre, light
