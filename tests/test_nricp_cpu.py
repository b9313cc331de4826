"""CPU: the float64 NRICP oracle (tests/nricp_oracle.py, DESIGN section 1f) -- adjacency and boundary on hand-built
meshes, the closed-form gradient against autograd through the pytorch3d-form loss, the AdamW step against
torch.optim.AdamW(amsgrad=True), and the fitting loop against the reference's own loop (tests/golden/nricp_ref.npz)."""
import numpy as np
import pytest
import torch

import nricp_oracle as no


def test_lone_triangle():
    a = no.adjacency([[0, 1, 2]], 3)
    assert a["edges"].tolist() == [[0, 1], [0, 2], [1, 2]]
    assert a["row_ptr"].tolist() == [0, 2, 4, 6]
    assert a["col"].tolist() == [1, 2, 0, 2, 0, 1]
    assert a["deg"].tolist() == [2, 2, 2]
    assert a["boundary"].all()


def test_strip_and_isolated_vertex():
    # two triangles sharing the side (1, 2), and vertex 4 in no face
    a = no.adjacency([[0, 1, 2], [2, 1, 3]], 5)
    assert a["edges"].tolist() == [[0, 1], [0, 2], [1, 2], [1, 3], [2, 3]]
    assert a["deg"].tolist() == [2, 3, 3, 2, 0]
    assert a["col"].tolist() == [1, 2, 0, 2, 3, 0, 1, 3, 1, 2]
    assert a["boundary"].tolist() == [True, True, True, True, False]   # every vertex touches a side used once
    L = no.laplacian(a["edges"], 5).toarray()
    v = np.arange(15, dtype=np.float64).reshape(5, 3)
    assert np.array_equal((L @ v)[4], -v[4])   # D^-1 A - I with a zero row scale at deg 0
    np.testing.assert_allclose((L @ v)[1], (v[0] + v[2] + v[3]) / 3 - v[1])


def test_interior_vertex_of_a_fan():
    # a closed fan of 6 triangles around vertex 0: its sides all occur twice
    faces = [[0, k, k % 6 + 1] for k in range(1, 7)]
    a = no.adjacency(faces, 7)
    assert not a["boundary"][0] and a["boundary"][1:].all()
    assert a["deg"][0] == 6


def test_repeated_index_face():
    # (0, 0, 1): sides (0,0), (0,1), (1,0); (0,1) occurs twice, the self side once -> vertex 0 is on the boundary, and
    # the self edge (0, 0) is in E, twice in row 0 of the adjacency as in pytorch3d's COO A
    a = no.adjacency([[0, 0, 1]], 2)
    assert a["edges"].tolist() == [[0, 0], [0, 1]]
    assert a["col"].tolist() == [0, 0, 1, 0]
    assert a["deg"].tolist() == [3, 1]
    assert a["boundary"].tolist() == [True, False]
    L = no.laplacian(a["edges"], 2).toarray()
    np.testing.assert_allclose(L, [[2 / 3 - 1, 1 / 3], [1.0, -1.0]])


def test_out_of_range_faces_are_skipped():
    a = no.adjacency([[0, 1, 2], [1, 2, 5], [-1, 0, 1]], 4)
    b = no.adjacency([[0, 1, 2]], 4)
    for k in ("edges", "row_ptr", "col", "deg", "boundary"):
        assert np.array_equal(a[k], b[k]), k


def _state(seed, V=None):
    g = np.random.default_rng(seed)
    n = 7
    t = np.linspace(0, 1, n)
    x = np.stack(np.meshgrid(t, t, indexing="ij"), -1).reshape(-1, 2)
    x = np.concatenate([x, 0.1 * g.standard_normal((n * n, 1))], 1)
    faces = []
    for i in range(n - 1):
        for j in range(n - 1):
            a, b, c, d = i * n + j, (i + 1) * n + j, (i + 1) * n + j + 1, i * n + j + 1
            faces += [[a, b, c], [a, c, d]]
    faces = np.array(faces)
    V = n * n
    X = no.identity_affine(V) + 0.05 * g.standard_normal((V, 3, 4))
    nrm = g.standard_normal((V, 3))
    c = x + 0.1 * g.standard_normal((V, 3))
    m = g.standard_normal((V, 3))
    return X, x, nrm, c, m, faces


@pytest.mark.parametrize("gamma", [1.0, 0.5])
def test_closed_form_gradient_matches_autograd(gamma):
    X, x, n, c, m, faces = _state(1)
    adj = no.adjacency(faces, len(x))
    L = no.laplacian(adj["edges"], len(x))
    g, t = no.gradient(X, x, n, c, m, adj, L, 3.0, 7.0, gamma, 0.2)
    assert 0 < t["w"].sum() < len(x)
    Xt = torch.tensor(X, requires_grad=True)
    T = lambda a: torch.tensor(a)  # noqa: E731
    loss = no.torch_loss(Xt, T(x), T(n), T(c), T(m), T(faces), T(adj["boundary"]), 3.0, 7.0, gamma, 0.2)
    (ga,) = torch.autograd.grad(loss, Xt)
    assert abs(loss.item() - t["loss"]) < 1e-13
    np.testing.assert_allclose(g, ga.numpy(), rtol=0, atol=1e-12 * np.abs(g).max())


def test_zero_S_gives_infinite_scale_like_torch():
    # S = 0 (no gated vertex, all X equal): the sqrt backward gives s = +inf, so the gradient is NaN, as in torch
    X, x, n, c, m, faces = _state(2)
    X[:] = no.identity_affine(1)
    adj = no.adjacency(faces, len(x))
    L = no.laplacian(adj["edges"], len(x))
    g, t = no.gradient(X, x, n, c, m, adj, L, 3.0, 7.0, 1.0, 2.0)   # threshold 2: the gate rejects everything
    assert t["S"] == 0.0
    Xt = torch.tensor(X, requires_grad=True)
    T = lambda a: torch.tensor(a)  # noqa: E731
    loss = no.torch_loss(Xt, T(x), T(n), T(c), T(m), T(faces), T(adj["boundary"]), 3.0, 7.0, 1.0, 2.0)
    (ga,) = torch.autograd.grad(loss, Xt)
    assert np.isnan(g).all() and torch.isnan(ga).all()


def test_adamw_matches_torch():
    g = np.random.default_rng(4)
    X0 = g.standard_normal((10, 3, 4))
    p = torch.nn.Parameter(torch.tensor(X0))
    opt = torch.optim.AdamW([p], lr=1e-4, amsgrad=True)
    X, state = X0, (np.zeros_like(X0),) * 3
    for step in range(1, 8):
        grad = g.standard_normal(X0.shape) * 10.0 ** g.uniform(-9, 1)   # also gradients below eps
        p.grad = torch.tensor(grad)
        opt.step()
        X, state = no.adamw_step(X, grad, state, step)
        np.testing.assert_allclose(X, p.detach().numpy(), rtol=0, atol=1e-15)


@pytest.mark.parametrize("case", [0, 1])
def test_fitting_loop_matches_the_reference(golden, case):
    z = golden("nricp_ref.npz")
    r = no.fit(z["src_v"], z["src_f"], z["tgt_v"], z["tgt_f"], z["masks"], int(z["epoch"]), int(z["inner_iter"]),
               list(z["stiffness_weight"]), list(z["laplacian_weight"]), list(z["mile_stone"]),
               gamma=float(z[f"gamma_{case}"]), threshold=float(z[f"threshold_{case}"]))
    scale = np.abs(z[f"final_v_{case}"] - z["src_v"]).max()
    assert np.abs(r["epoch_v"] - z[f"epoch_v_{case}"]).max() < 1e-12 * scale
    assert np.abs(r["final_v"] - z[f"final_v_{case}"]).max() < 1e-12 * scale
    # the printed terms are rounded to 4-5 decimals
    np.testing.assert_allclose(r["stats"], z[f"stats_{case}"], rtol=0, atol=6e-5)
    assert np.array_equal(r["stats"][:, 1], z[f"stats_{case}"][:, 1])


def test_inverse_rule_matches_fastminv_on_non_finite_and_gate_matrices():
    # FastMinv's test is |det| < 1e-4, so a NaN det passes the gate: ok = True and a non-finite inverse
    from oracle import oracle_torch as ot
    g = np.random.default_rng(3)
    A = g.standard_normal((12, 3, 3))
    A[0, 1, 2] = np.nan
    A[1, 0, 0] = np.inf
    A[2, 2, 1] = -np.inf
    A[3] = np.diag([1e-2, 1e-2, 0.99])      # det 9.9e-5: below the gate
    A[4] = np.diag([1e-2, 1e-2, 1.01])      # det 1.01e-4: above it
    A[5, 2] = A[5, 0]                       # exactly singular
    inv, ok = no.inv3x3(A)
    ref_inv, ref_ok = ot.minv3x3_fwd(torch.as_tensor(A))
    assert ok.tolist() == ref_ok.tolist()
    assert ok[0] and ok[1] and ok[2] and not ok[3] and ok[4] and not ok[5]
    assert np.isnan(inv[0]).any() and (inv[3] == 0).all() and (inv[5] == 0).all()
    np.testing.assert_array_equal(np.isnan(inv), torch.isnan(ref_inv).numpy())
    fin = np.isfinite(inv)
    np.testing.assert_allclose(inv[fin], ref_inv.numpy()[fin], rtol=1e-12, atol=0)
    np.testing.assert_allclose(inv[6:], np.linalg.inv(A[6:]), rtol=1e-12, atol=1e-12)
