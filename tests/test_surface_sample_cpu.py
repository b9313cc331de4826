"""CPU tests of the surface sampler's oracle (oracle/sample_oracle.py, DESIGN section 1h), which the GPU tests hold the
kernel to bit for bit: Philox4x32-10 against Random123's published answers, the sampling distribution (face counts
against area fractions, the folded barycentric coordinates), the rules for zero-area, invalid and all-degenerate
faces, the fan builder, the drop-in's early returns, and the curve-aware fixture against its generator."""
import os
import types

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import refload
from oracle import sample_oracle as so
from recmv_b200.utils import make_curve_aware_loss

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(x) for x in so.philox4x32_10(np.array(ctr, dtype=np.uint32), key)) == want


def test_uniforms_use_both_counter_words_and_both_key_words():
    c = np.array([5, 5 + (1 << 32)], dtype=np.uint64)
    u, a, b = so.uniforms(7, c)
    assert u[0] != u[1] and a[0] != a[1]
    u2, _, _ = so.uniforms(7 + (1 << 32), c[:1])
    assert u2[0] != u[0]
    assert np.all((u >= 0) & (u < 1) & (a + b <= 1))


def _mesh(seed, F=60):
    g = np.random.default_rng(seed)
    V = 3 * F
    verts = (g.standard_normal((V, 3)) * g.uniform(0.1, 3.0, size=(V, 1))).astype(np.float32)
    faces = np.arange(V, dtype=np.int64).reshape(F, 3)
    return verts, faces


def test_face_counts_follow_the_area_fractions():
    verts, faces = _mesh(1)
    S = 200_000
    _, idx = so.sample_mesh(verts, faces, S, seed=11, offset=0)
    area, _ = so.face_areas(verts, faces)
    counts = np.bincount(idx, minlength=len(faces))
    chi2, p = stats.chisquare(counts, area / area.sum() * S)
    assert p > 1e-3, (chi2, p)


def test_folded_barycentrics_are_uniform_on_the_triangle():
    # a point uniform on the triangle {a, b >= 0, a + b <= 1} has P(a <= x) = 1 - (1 - x)^2 and P(a + b <= t) = t^2
    _, a, b = so.uniforms(3, np.arange(100_000, dtype=np.uint64))
    assert np.all(a + b <= 1)
    for x in (a, b):
        assert stats.kstest(x, lambda t: 1 - (1 - t) ** 2).pvalue > 1e-3
    assert stats.kstest(a + b, lambda t: t ** 2).pvalue > 1e-3
    # and the point on the unit right triangle reproduces them
    verts = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], dtype=np.float32)
    p, _ = so.sample_mesh(verts, np.array([[0, 1, 2]]), 1000, seed=3, offset=0)
    assert np.array_equal(p[:, :2], np.stack([a[:1000], b[:1000]], 1)) and np.all(p[:, 2] == 0)


def test_zero_area_and_invalid_faces_are_never_drawn():
    verts, faces = _mesh(2, F=40)
    verts[faces[3]] = verts[faces[3, 0]]                 # a point
    faces[10, 1] = -1
    faces[11, 2] = len(verts)
    verts[faces[12, 0]] = np.inf                         # non-finite area
    area, valid = so.face_areas(verts, faces)
    assert area[3] == 0 and area[10] == 0 and area[11] == 0 and area[12] == 0
    assert not valid[10] and not valid[11] and valid[12]
    p, idx = so.sample_mesh(verts, faces, 50_000, seed=5, offset=0)
    assert not np.isin(idx, [3, 10, 11, 12]).any()
    assert np.isfinite(p).all()


def test_all_degenerate_meshes_use_face_zero():
    v = np.zeros((3, 3), dtype=np.float32)
    p, idx = so.sample_mesh(v, np.array([[0, 1, 2], [0, 1, 2]]), 64, seed=1, offset=0)
    assert np.all(idx == 0) and np.all(p == 0)
    # face 0 out of range: every sample is NaN
    p, idx = so.sample_mesh(v, np.array([[0, 1, 3], [0, 1, 2]]), 64, seed=1, offset=0)
    assert np.all(idx == 0) and np.isnan(p).all()


def test_cumulative_order():
    g = np.random.default_rng(4)
    a = g.uniform(0, 1, 256)
    assert np.array_equal(so.cumulative(a), np.cumsum(a))
    b = g.uniform(0, 1, 1000)
    C = so.cumulative(b)
    assert np.all(np.diff(C) >= 0)
    assert np.allclose(C, np.cumsum(b), rtol=1e-13, atol=0)
    ref = np.empty(1000)
    run = 0.0
    for c in range(4):
        loc = np.cumsum(b[256 * c:256 * (c + 1)])
        ref[256 * c:256 * c + len(loc)] = run + loc
        run = run + loc[-1]
    assert np.array_equal(C, ref)


def test_batched_sampling_equals_successive_offsets():
    verts, faces = _mesh(6, F=30)
    vs = np.stack([verts, verts * 2, verts + 1])
    out = so.sample_surface(vs, faces, 500, seed=9, offset=(1 << 32) - 700)
    for m in range(3):
        p, _ = so.sample_mesh(vs[m], faces, 500, seed=9, offset=(1 << 32) - 700 + 500 * m)
        assert np.array_equal(out[m], p)


def test_fan_builder():
    curve = np.random.default_rng(0).standard_normal((200, 3)).astype(np.float32)
    v, f = so.fan(curve)
    assert v.shape == (201, 3) and f.shape == (200, 3)
    assert np.array_equal(v[200], curve.mean(0, dtype=np.float32))
    assert f[0].tolist() == [0, 1, 200] and f[198].tolist() == [198, 199, 200] and f[199].tolist() == [199, 0, 200]


class _Conf:
    def __init__(self, d):
        self.d = d

    def get_float(self, key):
        v = self.d
        for k in key.split("."):
            v = v[k]
        return float(v)

    def __contains__(self, key):
        return key in self.d


def _self(weight, fl_names, garment_type, isfine):
    curves = torch.zeros((len(fl_names), 200, 3))
    return types.SimpleNamespace(conf=_Conf({"pc_weight": {"curve_aware_weight": weight}}), fl_names=fl_names,
                                 garment_type=garment_type, isfine=isfine, sdfShrinkRadius=0.0, info={},
                                 inter_free_curve=types.SimpleNamespace(forward=lambda: curves), garment_nets=[None])


def test_drop_in_returns_zero_without_a_term():
    fn = make_curve_aware_loss({"female_outfit1": "bottom_curve"})
    assert fn(_self(0.0, ["upper_bottom"], "female_outfit1", True), 0.5) == 0.
    assert fn(_self(60.0, ["neck", "bottom_curve"], "female_outfit1", False), 0.5) == 0.   # CURVE_AWARE term: fine only
    assert fn(_self(60.0, ["neck"], "gap_skirt", True), 0.5) == 0.
    assert fn.stream == {"seed": None, "offset": 0}
    with pytest.raises(RuntimeError, match="CUDA"):
        fn(_self(60.0, ["upper_bottom"], "gap_skirt", True), 0.5)


@pytest.mark.skipif(not refload.available(), reason="needs the reference source tree")
def test_generator_reproduces_the_fixture():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_curve_aware",
                                                  os.path.join(GOLDEN, "make_golden_curve_aware.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    new = gen.generate()
    z = np.load(os.path.join(GOLDEN, "curve_aware_ref.npz"), allow_pickle=False)
    assert sorted(new) == sorted(z.files)
    for k in z.files:
        if k.split("/")[1].startswith(("curves", "fan_", "samples_", "offset", "seed", "fl_names", "terms")):
            assert np.array_equal(new[k], z[k]), k       # the stream and the inputs: bit for bit
        elif z[k].dtype.kind == "f":
            # the loss and gradients run through CPU fp32 matmuls whose sums may be split by thread count
            scale = max(float(np.abs(z[k]).max()), 1e-30)
            assert float(np.abs(new[k] - z[k]).max()) <= 1e-5 * scale, k
        else:
            assert np.array_equal(new[k], z[k]), k
