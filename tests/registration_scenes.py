"""Deterministic NumPy meshes for the registration kernels (csrc/nricp.cu, csrc/lap_edit.cu) at many-block sizes and
with adversarial topology.  Every builder returns float64 vertices (or none, for the sparse mesh) and int64 faces;
tests/test_registration_scenes_cpu.py checks that each scene contains what its docstring claims.

- `sheet(V)`: exactly V vertices on a jittered, bumped height field, 64 per row with a ragged last row, every vertex in
  a face.  With 256 vertices per block of the NRICP step: 257 is two blocks, the second holding one vertex; 8 192 is
  32 blocks, one partial per lane of the cross-block reduction; 8 193 is 33 blocks, lane 0 sums two.
- `big_tube()`: a 1000 x 1000 jittered tube (1e6 vertices, 3 907 blocks, about 122 partials per lane).
- `adversarial()`: a jittered tube plus a 4 096-spoke fan, isolated vertices, a repeated-index face, a duplicated and a
  reversed duplicate face (their sides in three faces), two more non-manifold edges, faces with indices -1 and V, and a
  flat union-jack patch whose float64 (and fp32) uniform Laplacian is exactly 0 at every interior vertex.
- `sparse()`: V = 2^25 + 3 with a few thousand faces on the lowest and highest indices, so that the side keys
  lo * V + hi reach 2^50.
"""
import numpy as np

import lap_edit_oracle as lo

HUB_DEGREE = 4096
N_ISOLATED = 300
SPARSE_V = (1 << 25) + 3


def sheet(V, seed=0, width=64):
    """(v [V,3], faces): vertex k at row k // width, column k % width; quads split into (a, b, d), (b, c, d) wherever
    all three vertices exist."""
    g = np.random.default_rng(seed)
    k = np.arange(V)
    h = 1.0 / width
    px = (k % width + 0.3 * g.uniform(-1, 1, V)) * h
    py = (k // width + 0.3 * g.uniform(-1, 1, V)) * h
    v = np.stack([px, py, 0.1 * np.sin(3 * px) * np.cos(2 * py)], 1)
    rows = (V + width - 1) // width
    R, C = np.meshgrid(np.arange(max(rows - 1, 0)), np.arange(width - 1), indexing="ij")
    a = (R * width + C).ravel()
    b, d = a + 1, a + width
    f = np.concatenate([np.stack([a, b, d], 1), np.stack([b, d + 1, d], 1)])
    return v, f[(f < V).all(axis=1)].astype(np.int64)


def big_tube(seed=0):
    v, f, _ = lo.tube(1000, 1000, jitter=0.3, seed=seed)
    return v, f


def union_jack(m, origin):
    """An m x m flat grid at spacing 1/16 from `origin` (dyadic coordinates), quad (i, j) split along the diagonal
    through (i, j) when i + j is even and through (i + 1, j) otherwise: interior vertices have degree 8 or 4, so
    (1/deg) sum_j v_j - v_i is exactly 0 in float64 and in fp32.  (v [m*m,3], faces, interior vertex indices)."""
    I, J = np.meshgrid(np.arange(m), np.arange(m), indexing="ij")
    v = np.stack([I.ravel() / 16.0, J.ravel() / 16.0, np.zeros(m * m)], 1) + np.asarray(origin, dtype=np.float64)
    f = []
    for i in range(m - 1):
        for j in range(m - 1):
            a, b, c, d = i * m + j, (i + 1) * m + j, (i + 1) * m + j + 1, i * m + j + 1
            f += [[a, b, c], [a, c, d]] if (i + j) % 2 == 0 else [[a, b, d], [b, c, d]]
    interior = ((I > 0) & (I < m - 1) & (J > 0) & (J < m - 1)).ravel()
    return v, np.array(f, dtype=np.int64), np.flatnonzero(interior)


def adversarial(seed=0):
    """(v [V,3], faces, info) with V about 6.3e4; info names the special vertices and faces:
    hub, ring (its spokes), isolated, patch and flat (the flat patch and its interior vertices), self_face, dup_faces,
    nonmanifold_edges, bad_faces, tube (the tube's vertex count), tube_loops (hem and waist of the tube)."""
    g = np.random.default_rng(seed)
    nt = nz = 240
    tv, tf, loops = lo.tube(nt, nz, jitter=0.3, seed=seed)
    verts, faces, info = [tv], [tf], dict(tube=len(tv), tube_loops=loops)
    n = len(tv)
    # a cone fan: the apex has HUB_DEGREE neighbours, every spoke vertex three
    th = 2 * np.pi * np.arange(HUB_DEGREE) / HUB_DEGREE
    ring = np.stack([2.0 + 0.3 * np.cos(th), 0.3 * np.sin(th), np.zeros(HUB_DEGREE)], 1)
    verts += [np.array([[2.0, 0.0, 0.2]]), ring]
    hub, rk = n, n + 1 + np.arange(HUB_DEGREE)
    faces.append(np.stack([np.full(HUB_DEGREE, hub), rk, np.roll(rk, -1)], 1))
    info.update(hub=hub, ring=rk)
    n += 1 + HUB_DEGREE
    # vertices no face references
    verts.append(g.uniform(-1.0, 1.0, (N_ISOLATED, 3)) + [0.0, 0.0, 3.0])
    info["isolated"] = n + np.arange(N_ISOLATED)
    n += N_ISOLATED
    # the flat patch
    pv, pf, interior = union_jack(17, (3.0, 0.0, 0.5))
    verts.append(pv)
    faces.append(pf + n)
    info["flat"], info["patch"] = interior + n, n + np.arange(len(pv))
    n += len(pv)
    # a repeated-index face on an interior tube edge: the self edge (a, a) and (a, b) in four faces
    a = 100 * nz + 100
    faces.append(np.array([[a, a, a + 1]]))
    info["self_face"] = a
    # one interior tube face once more as it is, another once more reversed: their sides in three faces, with every
    # endpoint interior (no side of theirs occurs once)
    k, k2 = 2 * (150 * (nz - 1) + 60), 2 * (30 * (nz - 1) + 200) + 1
    faces.append(np.stack([tf[k], tf[k2][::-1]]))
    info["dup_faces"] = np.stack([tf[k], tf[k2]])
    # non-manifold edges: an interior tube edge with a third face, and an edge shared by three triangles of their own
    e0 = 50 * nz + 170
    verts.append(np.array([[0.0, 0.0, 1.0], [4.0, 0.0, 0.0], [4.0, 0.2, 0.0], [4.1, 0.1, 0.2], [3.9, 0.1, -0.2],
                           [4.0, 0.1, 0.3]]))
    w, p, q = n, n + 1, n + 2
    faces.append(np.array([[e0, e0 + 1, w], [p, q, n + 3], [q, p, n + 4], [p, n + 5, q]]))
    info["nonmanifold_edges"] = [(e0, e0 + 1), (p, q)]
    n += 6
    # faces the adjacency skips
    bad = np.array([[-1, 7, 8], [7, n, 8]])
    faces.append(bad)
    info["bad_faces"] = bad
    return np.concatenate(verts), np.concatenate(faces).astype(np.int64), info


def sparse():
    """(V, faces): two 40 x 40 sheets, one on indices [0, 1600) and one on the last 1600 indices, and faces joining
    vertex 0 and 1 to the last vertices; every other vertex is isolated."""
    _, f = sheet(1600, width=40)
    hi = f + (SPARSE_V - 1600)
    join = np.array([[0, SPARSE_V - 1, SPARSE_V - 2], [1, 0, SPARSE_V - 2], [SPARSE_V - 1, 0, SPARSE_V - 41]])
    return SPARSE_V, np.concatenate([f, hi, join]).astype(np.int64)
