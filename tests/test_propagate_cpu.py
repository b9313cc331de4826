"""CPU: oracle/implicit_grad_oracle.py against the reference's own propagateTmpPsGrad (tests/golden/propagate_ref.npz,
both garment classes): its float64 coefficients, ok counts and camera sums, its not-ok rows, and the fixture's
regeneration."""
import os

import numpy as np
import pytest

from oracle import implicit_grad_oracle as igo, refload

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURE = os.path.join(GOLDEN, "propagate_ref.npz")
GRAZING = 5


def _z():
    z = np.load(FIXTURE)
    return {k: z[k] for k in z.files}


def _close(a, b, rel):
    scale = max(float(np.abs(b).max(initial=0)), 1e-300)
    return float(np.abs(np.asarray(a, np.float64) - b).max(initial=0)) <= rel * scale


@pytest.mark.parametrize("cls", ["base", "large"])
def test_oracle_reproduces_the_reference_in_float64(cls):
    z = _z()
    G = int(z["in/G"])
    offsets = np.cumsum([0] + [len(z[f"in/P_{g}"]) for g in range(G)])
    per = {k: [] for k in ("sdf_coef", "def_vec", "ray_grad", "ok")}
    for g in range(G):
        k = lambda s: z[f"{cls}/f64/{s}_{g}"]  # noqa: E731
        o = igo.rows(z[f"in/gl_{g}"], k("gf"), k("J"), k("v"), k("d"), k("c"), dc_f32=False)
        assert not o["flags"].any()
        if cls == "base":
            assert _close(o["sdf_coef"], k("sdf_coef"), 1e-12), g
        assert _close(o["def_vec"], k("def_vec"), 1e-12), g
        assert _close(o["ray_grad"], k("ray_grad"), 1e-12), g
        assert np.array_equal(o["ok"], k("ok")), g
        cnt, cam = igo.garments(o, [0, len(o["ok"])])
        assert cnt[0] == k("invInfo")[1] and k("invInfo")[0] == len(o["ok"]), g
        assert _close(cam[0], k("cam_grad"), 1e-12), g
        for key in per:
            per[key].append(o[key])
    # the per-garment reductions over the concatenated rows
    cat = {key: np.concatenate(v) for key, v in per.items()}
    cnt, cam = igo.garments(cat, offsets)
    assert [int(c) for c in cnt] == [int(z[f"{cls}/f64/invInfo_{g}"][1]) for g in range(G)]
    for g in range(G):
        assert _close(cam[g], z[f"{cls}/f64/cam_grad_{g}"], 1e-12)


@pytest.mark.parametrize("tag", ["base/f32", "base/f64", "large/f32", "large/f64"])
def test_grazing_rows_are_exactly_the_rows_the_reference_rejects(tag):
    z = _z()
    for g in range(int(z["in/G"])):
        ok = z[f"{tag}/ok_{g}"]
        assert not ok[:GRAZING].any() and ok[GRAZING:].all(), (tag, g, np.nonzero(~ok)[0])
        assert int(z[f"{tag}/invInfo_{g}"][1]) == len(ok) - GRAZING
        _, m = igo.btb(z[f"{tag}/gf_{g}"], z[f"{tag}/J_{g}"], z[f"{tag}/v_{g}"])
        det = np.abs(np.linalg.det(m))
        assert (det[:GRAZING] < 1e-5).all() and (det[GRAZING:] > 1e-3).all()


def test_oracle_rule_and_reductions_on_edges():
    rng = np.random.default_rng(3)
    n = 40
    gl, gf, v = (rng.standard_normal((n, 3)) for _ in range(3))
    J = rng.standard_normal((n, 3, 3))
    gf[:4] = 0.0                                  # b = [0 ; [v]x J] has rank 2: singular
    o = igo.rows(gl, gf, J, v)
    assert not o["ok"][:4].any()
    assert np.array_equal(o["def_vec"][:4], np.zeros((4, 3))) and np.array_equal(o["sdf_coef"][:4], np.zeros(4))
    cnt, cam = igo.garments(o, [0, 0, 10, 10, n])     # empty garments give 0 and 0
    assert list(cnt) == [0, int(o["ok"][:10].sum()), 0, int(o["ok"][10:].sum())]
    assert np.array_equal(cam[0], np.zeros(3)) and np.array_equal(cam[2], np.zeros(3))
    assert np.allclose(cam[1], -o["def_vec"][:10].sum(0))


@pytest.mark.skipif(not refload.available(), reason="needs the reference source tree")
def test_propagate_generator_reproduces_the_fixture():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_propagate",
                                                  os.path.join(GOLDEN, "make_golden_propagate.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    new = gen.generate()
    z = np.load(FIXTURE)
    assert sorted(new) == sorted(z.files)
    for key in z.files:
        a, b = new[key], z[key]
        if key.startswith("in/") or "/ok_" in key or "/invInfo_" in key:
            assert np.array_equal(a, b), key
        else:
            # CPU torch may split its sums by thread count: float32 values to 1e-4 of the tensor's scale, float64 to 1e-10
            tol = (1e-4 if "/f32/" in key else 1e-10) * max(float(np.abs(b).max(initial=0)), 1e-30)
            assert float(np.abs(a - b).max(initial=0)) <= tol, key
