"""CPU tests of the training-ray sampler's oracle (oracle/train_rays_oracle.py, DESIGN section 1j), which the GPU tests
hold the kernel to bit for bit: the oracle against the reference's own `sample_train_ray` (tests/golden/
train_rays_ref.npz), the float32 threshold rule torch applies, the counters of garments and successive calls, and the
drop-in's refusal of CPU tensors."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import refload
from oracle import train_rays_oracle as tro
from recmv_b200.utils import make_sample_train_ray

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ("below", "above", "mixed")


def _case(z, name):
    k = lambda s: z[f"{name}/{s}"]  # noqa: E731
    pix = int(k("conf_pix")) if int(k("conf_pix")) >= 0 else int(k("arg_pix"))
    target = pix // int(k("garment_size")) * int(k("N"))
    cam = np.concatenate([k("focal")[0] if k("focal").ndim > 1 else k("focal"), k("pp"), k("R").reshape(-1)])
    lists = [[k(f"{s}_{g}") for g in range(2)] for s in ("mask", "batch", "row", "col", "pts")]
    return k, target, cam, lists


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_the_reference(name):
    z = np.load(os.path.join(GOLDEN, "train_rays_ref.npz"))
    k, target, cam, (masks, b, r, c, pts) = _case(z, name)
    out, nxt = tro.sample(masks, b, r, c, target, int(k("seed")), int(k("offset")), cam)
    assert nxt == int(k("offset")) + len(b[0]) + len(b[1])
    drew = []
    for g, (keep, rays) in enumerate(out):
        pnum = len(tro.candidates(masks[g], b[g], r[g], c[g]))
        drew.append(pnum > target)
        for key, src in (("batch", b[g]), ("row", r[g]), ("col", c[g]), ("pts", pts[g])):
            assert np.array_equal(src[keep], k(f"ref_{key}_{g}")), (g, key)
        ref = k(f"ref_rays_{g}")
        assert float(np.abs(rays - ref).max(initial=0)) <= 1e-6
        assert float(np.abs(tro.view_rays64(c[g][keep], r[g][keep], cam) - ref).max(initial=0)) <= 1e-6
        assert float(np.abs(tro.view_rays64(c[g][keep], r[g][keep], cam) - rays).max(initial=0)) <= 1e-6
        if pnum > target:
            assert 0 < len(keep) < pnum
    assert drew == {"below": [False, False], "above": [True, True], "mixed": [True, False]}[name]


def test_nan_and_out_of_range_rows_are_not_candidates():
    mask = np.array([[[1, np.nan], [0.5, -1]]], np.float32)
    b = np.array([0, 0, 0, 0, 1, 0, 0, -1])
    r = np.array([0, 0, 1, 1, 0, 2, 0, 0])
    c = np.array([0, 1, 0, 1, 0, 0, -1, 0])
    assert tro.candidates(mask, b, r, c).tolist() == [0, 2]


def test_threshold_is_the_float32_quotient_and_excludes_its_own_value():
    T, pnum = 6144, 700002
    thr = tro.threshold(T, pnum)
    assert float(thr) < T / pnum                                  # rounded below the double quotient
    # torch 2.11 on the CPU compares a float32 tensor with a Python float at float32: u == thr is not kept
    u = torch.tensor([float(thr), float(np.nextafter(thr, np.float32(0)))], dtype=torch.float32)
    assert (u < float(T) / float(pnum)).tolist() == [False, True]
    assert (u.numpy() < thr).tolist() == [False, True]
    # T = 0 keeps nothing once there is a candidate
    assert tro.threshold(0, 5) == 0 and not (tro.uniforms(1, np.arange(1000, dtype=np.uint64)) < 0).any()


def test_uniforms_are_24_bit_and_use_both_counter_and_key_words():
    c = np.array([7, 7 + (1 << 32)], dtype=np.uint64)
    u = tro.uniforms(3, c)
    assert u.dtype == np.float32 and u[0] != u[1]
    assert tro.uniforms(3 + (1 << 32), c[:1])[0] != u[0]
    big = tro.uniforms(11, np.arange(200_000, dtype=np.uint64))
    assert np.all((big >= 0) & (big < 1)) and np.array_equal(big * np.float32(1 << 24), np.floor(big * (1 << 24)))
    assert abs(float(big.mean()) - 0.5) < 0.005


def test_counters_are_disjoint_across_garments_and_calls():
    rng = np.random.default_rng(5)
    N, H, W = 1, 20, 30
    lens = [(300, 0, 451), (17, 600, 2)]
    offset, used = (1 << 64) - 700, []
    for call in lens:
        base = 0
        for P in call:
            pnum = P      # every row a candidate: the most counters a list can use
            used.append(tro.counters(offset, base, pnum))
            base += P
        offset = (offset + base) % (1 << 64)
    flat = np.concatenate(used)
    assert len(np.unique(flat)) == len(flat) == sum(map(sum, lens))
    assert flat.min() == 0 and flat.max() == (1 << 64) - 1           # wrapped modulo 2^64
    # and sample() advances the offset by the input rows, whatever was kept
    masks = [rng.uniform(-1, 1, (N, H, W)).astype(np.float32) for _ in range(2)]
    lists = [np.nonzero(rng.uniform(size=(N, H, W)) < 0.5) for _ in range(2)]
    _, nxt = tro.sample(masks, [x[0] for x in lists], [x[1] for x in lists], [x[2] for x in lists], 10, 1, 40)
    assert nxt == 40 + len(lists[0][0]) + len(lists[1][0])


def test_drop_in_refuses_cpu_tensors():
    fn = make_sample_train_ray()
    self = types.SimpleNamespace(conf=_Conf({"sample_pix_num": 2048}), garment_size=1)
    m = torch.ones((1, 4, 4))
    i = torch.zeros(3, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="CUDA"):
        fn(self, 1, 2048, [m], [i], [i], [i], [torch.zeros((3, 3))], torch.arange(1), "cpu")
    assert fn.stream == {"seed": None, "offset": 0}


class _Conf:
    def __init__(self, d):
        self.d = d

    def get_int(self, key):
        return int(self.d[key])

    def __contains__(self, key):
        return key in self.d


@pytest.mark.skipif(not refload.available(), reason="needs the reference source tree")
def test_generator_reproduces_the_fixture():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_train_rays",
                                                  os.path.join(GOLDEN, "make_golden_train_rays.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    new = gen.generate()
    z = np.load(os.path.join(GOLDEN, "train_rays_ref.npz"))
    assert sorted(new) == sorted(z.files)
    for key in z.files:
        if "/ref_rays" in key:
            # CPU torch's norm and matmul may split their sums by thread count
            assert float(np.abs(new[key] - z[key]).max(initial=0)) <= 1e-6, key
        else:
            assert np.array_equal(new[key], z[key], equal_nan=z[key].dtype.kind == "f"), key
