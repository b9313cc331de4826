"""CPU: the scenes of tests/registration_scenes.py contain what they claim -- vertex and block counts around the NRICP
step's 256-vertex blocks and 32-lane partial loop, and the adversarial topology (hub degree, isolated vertices,
repeated-index, duplicated and non-manifold faces, out-of-range faces, an exactly flat patch) -- as the float64
adjacency of tests/nricp_oracle.py sees them."""
import numpy as np
import pytest

import nricp_oracle as no
import registration_scenes as rs


@pytest.mark.parametrize("V,blocks,lane0", [(257, 2, 1), (8192, 32, 1), (8193, 33, 2)])
def test_sheets_have_the_block_counts_and_no_isolated_vertex(V, blocks, lane0):
    v, f = rs.sheet(V)
    assert v.shape == (V, 3) and f.min() >= 0 and f.max() == V - 1
    nb = (V + 255) // 256
    assert nb == blocks and len(range(0, nb, 32)) == lane0   # partials summed by lane 0 of the reduction warp
    a = no.adjacency(f, V)
    assert (a["deg"] > 0).all()
    assert a["boundary"].any() and not a["boundary"].all()


def test_big_tube_reaches_about_120_partials_per_lane():
    v, f = rs.big_tube()
    V = len(v)
    assert V == 10 ** 6 and len(f) == 2 * 1000 * 999
    assert 120 <= ((V + 255) // 256) / 32 <= 125


def test_adversarial_mesh_contains_every_case():
    v, f, info = rs.adversarial()
    V = len(v)
    assert 5.5e4 <= V <= 7e4
    a = no.adjacency(f, V)
    deg, col, row_ptr = a["deg"], a["col"], a["row_ptr"]
    assert deg[info["hub"]] == rs.HUB_DEGREE == deg.max()
    assert (deg[info["ring"]] == 3).all()
    assert (deg[info["isolated"]] == 0).all() and (deg == 0).sum() == rs.N_ISOLATED
    # the repeated-index face: the self edge appears twice in its row, the edge (a, a + 1) in four faces
    s = info["self_face"]
    assert (col[row_ptr[s]:row_ptr[s + 1]] == s).sum() == 2
    g = f[np.all((f >= 0) & (f < V), axis=1)]
    sides = np.sort(np.concatenate([g[:, [0, 1]], g[:, [1, 2]], g[:, [2, 0]]]), axis=1)
    keys, cnt = np.unique(sides[:, 0] * V + sides[:, 1], return_counts=True)
    count = dict(zip(keys.tolist(), cnt.tolist()))
    assert count[s * V + s] == 1 and count[s * V + s + 1] == 4
    # the duplicated face and the reversed duplicate: present twice, their sides in three faces, their vertices interior
    d, d2 = info["dup_faces"]
    assert (f == d).all(1).sum() == 2 and (f == d2).all(1).sum() == 1 and (f == d2[::-1]).all(1).sum() == 1
    dup_sides = [min(p, q) * V + max(p, q) for e in (d, d2) for p, q in ((e[0], e[1]), (e[1], e[2]), (e[2], e[0]))]
    assert not a["boundary"][np.concatenate([d, d2])].any()
    # exactly these and the two non-manifold edges occur three times
    assert sorted(k for k, c in count.items() if c == 3) == sorted(dup_sides + [p * V + q for p, q in
                                                                               info["nonmanifold_edges"]])
    # the faces with -1 and V are present and skipped
    bad = info["bad_faces"]
    assert bad.min() == -1 and bad.max() == V and all((f == b).all(1).any() for b in bad)
    # the flat patch: float64 L v exactly 0 at every interior vertex, whose degree is 4 or 8
    L = no.laplacian(a["edges"], V)
    flat = info["flat"]
    assert len(flat) == 15 * 15 and set(deg[flat].tolist()) == {4, 8}
    assert ((L @ v)[flat] == 0).all()
    assert ((np.float32(1) / deg[flat].astype(np.float32)) * deg[flat] == 1).all()   # 1/deg exact in fp32 too


def test_sparse_mesh_keys_reach_2_to_the_50():
    V, f = rs.sparse()
    assert V == (1 << 25) + 3 and 2000 <= len(f) <= 8000
    assert f.min() == 0 and f.max() == V - 1
    lo_, hi = np.minimum(f[:, 0], f[:, 1]), np.maximum(f[:, 0], f[:, 1])
    assert (lo_ * V + hi).max() >= 2 ** 50 - 2 ** 46 and V * V > 2 ** 50
    # indices in the middle are isolated
    used = np.unique(f)
    assert len(used) == 3200 and used[1599] == 1599 and used[1600] == V - 1600
