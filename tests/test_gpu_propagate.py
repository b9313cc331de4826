"""GPU tests of propagateTmpPsGrad on the device (DESIGN section 1l): the batched implicit-gradient kernel
(recmv_implicit_grad, csrc/surface_grad.cu) against oracle/implicit_grad_oracle.py, its rows against
recmv_surface_grad_coeffs bit for bit, and the drop-in utils.make_propagate_tmp_ps_grad against the reference's own
method (tests/golden/propagate_ref.npz) and its torch restatement on the same networks (tests/propagate_scene.py)."""
import warnings

import numpy as np
import pytest
import torch

from oracle import implicit_grad_oracle as igo
from recmv_b200 import ops

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


# ---- the kernel --------------------------------------------------------------------------------------------------
def _rows(rng, n, singular=()):
    """f32 (gl, gf, J, v, d) of n rows; rows in `singular` get v = J t / |J t| with t perpendicular to grad f.  The
    other rows' v is redrawn until the float64 |det b^T b| lies outside [1e-5, 1e-3]: a float32 determinant of these
    matrices is only good to ~1e-5 absolute, so closer to FastMinv's 1e-4 the kernel's flag would be a coin toss."""
    gl = rng.standard_normal((n, 3)) * 0.01
    gf = rng.standard_normal((n, 3))
    J = np.eye(3)[None] + rng.standard_normal((n, 3, 3)) * 0.3
    v = rng.standard_normal((n, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    d = rng.standard_normal((n, 3)) * 0.5
    s = np.asarray(singular, np.int64)
    if len(s):
        t = np.cross(gf[s], np.eye(3)[np.argmin(np.abs(gf[s]), axis=1)])
        w = np.einsum("nij,nj->ni", J[s], t)
        v[s] = w / np.linalg.norm(w, axis=1, keepdims=True)
    free = np.ones(n, bool)
    free[s] = False
    while True:
        v32 = v.astype(np.float32)
        det = np.abs(np.linalg.det(igo.btb(gf.astype(np.float32), J.astype(np.float32), v32)[1])) if n else v[:, 0]
        bad = free & (det >= 1e-5) & (det <= 1e-3)
        if not bad.any():
            break
        w = rng.standard_normal((int(bad.sum()), 3))
        v[bad] = w / np.linalg.norm(w, axis=1, keepdims=True)
    return [x.astype(np.float32) for x in (gl, gf, J, v, d)]


def _run(arrs, offsets, cam, want_ray_grad=True, max_ctas=None):
    t = [torch.from_numpy(x).to(DEV) for x in arrs]
    c = torch.from_numpy(cam).to(DEV) if cam is not None else None
    return ops.implicit_surface_grad(*t[:4], t[4], offsets, c, want_ray_grad, _max_ctas=max_ctas)


def _check_against_oracle(arrs, offsets, cam, out):
    gl, gf, J, v, d = arrs
    o = igo.rows(gl, gf, J, v, d, cam)
    bound = igo.row_bound(gl, gf, J, v, d, cam)
    coef, vec, rg, ok, cnt, camg = (x.cpu().numpy() if x is not None else None for x in out)
    same = ok == o["ok"]
    assert same[~o["flags"]].all(), np.flatnonzero(~same & ~o["flags"])[:10]
    both = ok & o["ok"]
    # per row: |kernel - float64| <= BOUND_K eps32 cond(b^T b) |g| |(b^T b)^-1| |b| max(1, |v|, |d - c|)
    assert (np.abs(coef - o["sdf_coef"]) <= bound)[both].all()
    assert (np.abs(vec - o["def_vec"]).max(1) <= bound)[both].all()
    assert (np.abs(rg - o["ray_grad"]).max(1) <= bound)[both].all()
    assert not vec[~ok].any() and not coef[~ok].any() and not rg[~ok].any()   # FastMinv's zeros
    offs = list(offsets)
    assert [int(x) for x in cnt] == [int(ok[a:b].sum()) for a, b in zip(offs, offs[1:])]   # exact
    want_cnt, want_cam = igo.garments(o, offs)
    for g, (a, b) in enumerate(zip(offs, offs[1:])):
        if same[a:b].all():
            assert int(cnt[g]) == int(want_cnt[g])
            tol = float(bound[a:b].sum()) + 1e-6 * float(np.abs(o["def_vec"][a:b]).sum())
            assert np.abs(camg[g] - want_cam[g]).max() <= tol, (g, camg[g], want_cam[g])
        if b == a:
            assert cnt[g] == 0 and not camg[g].any()


def _bits(x):
    return x.cpu().numpy().view(np.uint8 if x.dtype in (torch.bool, torch.uint8) else np.uint32)


def _deterministic(arrs, offsets, cam, out):
    for max_ctas in (None, 1, 3):        # a second run, and two other grids
        again = _run(arrs, offsets, cam, max_ctas=max_ctas)
        for a, b in zip(out, again):
            assert np.array_equal(_bits(a), _bits(b)), max_ctas


@pytest.mark.parametrize("sizes,singular", [
    ((700,), ()),
    ((300, 1500), ((1500, 1800),)),                        # garment 1: the first 300 rows singular
    ((0, 513, 400, 1, 2100), ((513, 913),)),               # an empty garment, an all-singular one, ragged sizes
    ((1025,), ()), ((1024, 1, 2049), ((0, 7),)),           # just above 1024-row chunk boundaries
])
def test_kernel_matches_the_oracle(sizes, singular):
    rng = np.random.default_rng(sum(sizes) + 7)
    offsets = np.cumsum((0,) + sizes).tolist()
    sing = np.concatenate([np.arange(a, b) for a, b in singular]) if singular else ()
    arrs = _rows(rng, offsets[-1], sing)
    cam = np.array([0.1, -0.2, 2.5], np.float32)
    out = _run(arrs, offsets, cam)
    for a, b in singular:
        assert not out[3][a:b].any()
    _check_against_oracle(arrs, offsets, cam, out)
    _deterministic(arrs, offsets, cam, out)


def test_kernel_rows_are_the_single_garment_kernel_rows():
    rng = np.random.default_rng(11)
    arrs = _rows(rng, 5000, np.arange(0, 5000, 37))
    cam = np.array([0.3, 0.1, -2.0], np.float32)
    out = _run(arrs, [0, 1000, 1000, 5000], cam)
    gl, gf, J, v, d = (torch.from_numpy(x).to(DEV) for x in arrs)
    dc = d - torch.from_numpy(cam).to(DEV).view(1, 3)
    ref = ops.surface_grad_coeffs(gl, gf, J, v, dc)
    for a, b in zip(out[:4], ref):
        assert np.array_equal(_bits(a), _bits(b))


def test_kernel_more_than_2_24_rows():
    """n > 2^24 in three garments: the rows tile a 4099-row pattern, so the float64 expectation is the pattern's."""
    P = 4099
    rng = np.random.default_rng(24)
    pat = _rows(rng, P, np.arange(0, P, 101))
    reps = (1 << 24) // P + 3
    n = reps * P
    offsets = [0, 5 * P, 5 * P + 1 + 1023, n]
    cam = np.array([0.0, 0.2, 2.2], np.float32)
    t = [torch.from_numpy(x).to(DEV).repeat(reps, *([1] * (x.ndim - 1))) for x in pat]
    out = ops.implicit_surface_grad(*t[:4], t[4], offsets, torch.from_numpy(cam).to(DEV), True)
    small = _run(pat, [0, P], cam)
    for a, b in zip(out[:4], small[:4]):                 # every copy of the pattern gives the pattern's rows
        full = a.view(reps, P, -1) if a.dim() > 1 else a.view(reps, P)
        assert torch.equal(full, b.unsqueeze(0).expand_as(full))
    o = igo.rows(*pat, cam)
    ok, vec = small[3].cpu().numpy(), small[1].cpu().numpy().astype(np.float64)
    idx = np.arange(n) % P
    for g, (a, b) in enumerate(zip(offsets, offsets[1:])):
        k = np.bincount(idx[a:b], minlength=P)
        assert int(out[4][g]) == int((k * ok).sum())
        assert int(out[4][g]) == int((k * o["ok"]).sum())
        want = -(k[:, None] * vec).sum(0)                 # the kernel's own float32 rows, summed in float64
        assert np.abs(out[5][g].cpu().numpy() - want).max() <= 1e-6 * np.abs(k[:, None] * vec).sum(0).max()
    again = ops.implicit_surface_grad(*t[:4], t[4], offsets, torch.from_numpy(cam).to(DEV), True, _max_ctas=5)
    assert torch.equal(out[4], again[4]) and np.array_equal(_bits(out[5]), _bits(again[5]))


def test_kernel_arguments():
    rng = np.random.default_rng(1)
    arrs = _rows(rng, 10)
    out = _run(arrs, [0, 10], None, want_ray_grad=False)
    assert out[2] is None and out[5] is None and out[4].shape == (1,)
    with pytest.raises(RuntimeError, match="offsets"):
        _run(arrs, [0, 4, 9], None, want_ray_grad=False)
    with pytest.raises(RuntimeError, match="ray gradient"):
        _run(arrs, [0, 10], None, want_ray_grad=True)
    with pytest.raises(RuntimeError, match="host"):
        t = [torch.from_numpy(x).to(DEV) for x in arrs]
        ops.implicit_surface_grad(*t[:4], t[4], torch.tensor([0, 10], device=DEV))
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.implicit_surface_grad(*[torch.from_numpy(x) for x in arrs[:4]], None, [0, 10])
    e = ops.implicit_surface_grad(*[torch.zeros((0, 3) if k != 2 else (0, 3, 3), device=DEV) for k in range(4)],
                                  None, [0, 0, 0], torch.zeros(3, device=DEV))
    assert e[4].tolist() == [0, 0] and not e[5].any()


# ---- the drop-in -------------------------------------------------------------------------------------------------
def _scene():
    import propagate_scene as ps
    return ps


def _fixture():
    from conftest import load_golden
    z = load_golden("propagate_ref.npz")
    return {k[3:]: v for k, v in z.items() if k.startswith("in/")}, z


def _grads(self, leaves):
    """name -> gradient, as the fixture stores them (weights: every 257th entry; biases whole)."""
    out = {}
    for mname, m in (("sdf", self.garment_nets[0]), ("translator", self.deformer.defs[0])):
        for pname, p in sorted(m.named_parameters()):
            if p.grad is not None:
                step = 257 if p.dim() > 1 else 1
                out[f"{mname}.{pname}"] = p.grad.detach().reshape(-1)[::step].double().cpu().numpy()
    for k, x in leaves.items():
        if not k.startswith("TmpPs") and x.grad is not None:
            out[k] = x.grad.detach().double().cpu().numpy()
    return out


def _err(a, b):
    return float(np.abs(a - b).max(initial=0))


def _run_state(cls_name, flow, learnable_camera=True, d=None):
    ps = _scene()
    d = d if d is not None else _fixture()[0]
    cls = ps.GarmentLargePose if cls_name == "large" else ps.Garment
    self, leaves = ps.state(DEV, d, cls, learnable_camera=learnable_camera, frozen_sdf=cls_name == "large")
    frame_ids = torch.arange(int(d["N"]), device=DEV)
    if flow == "drop-in":
        self.propagateTmpPsGrad(frame_ids, ps.RATIO)
    else:
        ps.reference_flow(self, frame_ids, ps.RATIO, large_pose=cls_name == "large")
    torch.cuda.synchronize()
    return self, leaves


@pytest.mark.parametrize("cls", ["base", "large"])
def test_drop_in_matches_the_reference(cls):
    """Every gradient tensor within 2.5e-5 of its largest entry, or 4x the float32 reference's own error against
    float64, whichever is larger: against the reference's own method (float64), and against its restatement run on the
    GPU from the same state."""
    d, z = _fixture()
    self, leaves = _run_state(cls, "drop-in", d=d)
    got = _grads(self, leaves)
    want = {k[len(f"{cls}/f64/grad/"):]: v for k, v in z.items() if k.startswith(f"{cls}/f64/grad/")}
    assert sorted(got) == sorted(want)
    if cls == "large":
        assert not any(k.startswith("sdf.") for k in got)
    over = {}
    for k, w in want.items():
        own = _err(z[f"{cls}/f32/grad/{k}"], w)
        tol = max(2.5e-5 * float(np.abs(w).max()), 4 * own)
        over[k] = _err(got[k], w) / tol
    assert max(over.values()) <= 1, sorted(over.items(), key=lambda kv: -kv[1])[:8]
    for g in range(int(d["G"])):
        M, cnt = self.info[f"{self.garment_names[g]}_invInfo"]
        assert (M, int(cnt)) == tuple(int(x) for x in z[f"{cls}/f64/invInfo_{g}"])
        assert isinstance(cnt, torch.Tensor) and cnt.dim() == 0 and "%d" % cnt == "%d" % int(cnt)
        off = self.deformer.defs[0].offset[self.garment_names[g]]
        assert off.shape == (len(d[f"P_{g}"]), 3)
    ref_self, ref_leaves = _run_state(cls, "reference", d=d)
    ref = _grads(ref_self, ref_leaves)
    for k, w in want.items():
        own = _err(z[f"{cls}/f32/grad/{k}"], w)
        tol = max(2.5e-5 * float(np.abs(w).max()), 4 * own)
        over[k] = _err(got[k], ref[k]) / tol
    assert max(over.values()) <= 1, sorted(over.items(), key=lambda kv: -kv[1])[:8]
    assert ref_self.info == {k: (v[0], int(v[1])) for k, v in self.info.items()}


def test_drop_in_makes_no_host_synchronisation_and_leaves_tmpps_grad():
    ps = _scene()
    d, _ = _fixture()
    self, leaves = ps.state(DEV, d, ps.Garment)
    frame_ids = torch.arange(int(d["N"]), device=DEV)
    gl = [p.grad.clone() for p in self.TmpPs]
    self.propagateTmpPsGrad(frame_ids, ps.RATIO)          # warm-up: workspaces, packed weights, host caches
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            self.propagateTmpPsGrad(frame_ids, ps.RATIO)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [w for w in rec if str(w.message).startswith("called a synchronizing CUDA operation")]
    assert len(syncs) == 0, [str(w.message) for w in syncs]
    for p, g in zip(self.TmpPs, gl):
        assert torch.equal(p.grad, g)


def test_drop_in_accumulates_into_existing_grads():
    d, _ = _fixture()
    once, lo = _run_state("base", "drop-in", d=d)
    first = _grads(once, lo)
    ps = _scene()
    self, leaves = ps.state(DEV, d, ps.Garment)
    frame_ids = torch.arange(int(d["N"]), device=DEV)
    self.propagateTmpPsGrad(frame_ids, ps.RATIO)
    self.propagateTmpPsGrad(frame_ids, ps.RATIO)
    twice = _grads(self, leaves)
    for k, v in first.items():
        assert _err(twice[k], 2 * v) <= 1e-5 * max(float(np.abs(v).max()), 1e-30), k


def test_drop_in_with_a_fixed_camera():
    d, _ = _fixture()
    self, leaves = _run_state("base", "drop-in", learnable_camera=False, d=d)
    ref_self, ref_leaves = _run_state("base", "reference", learnable_camera=False, d=d)
    got, ref = _grads(self, leaves), _grads(ref_self, ref_leaves)
    assert sorted(got) == sorted(ref) and "focal" not in got
    for k, w in ref.items():
        assert _err(got[k], w) <= 1e-3 * max(float(np.abs(w).max()), 1e-30), k


def test_drop_in_returns_at_the_first_garment_without_tmpps_grad():
    ps = _scene()
    d, _ = _fixture()
    for missing in (0, 1):
        self, leaves = ps.state(DEV, d, ps.Garment)
        self.TmpPs[missing].grad = None
        self.propagateTmpPsGrad(torch.arange(int(d["N"]), device=DEV), ps.RATIO)
        name = self.garment_names[missing]
        assert self.info[f"{name}_invInfo"] == (-1, -1)
        got = _grads(self, leaves)
        if missing == 0:
            assert got == {} and len(self.info) == 1
        else:
            assert f"{self.garment_names[0]}_invInfo" in self.info and "cond1" in got and "cond2" not in got
    self, _ = ps.state(DEV, d, ps.Garment)
    self.TmpPs[0] = self.TmpPs[0].detach().cpu().requires_grad_(True)
    self.TmpPs[0].grad = torch.zeros_like(self.TmpPs[0])
    with pytest.raises(RuntimeError, match="CUDA"):
        self.propagateTmpPsGrad(torch.arange(int(d["N"]), device=DEV), ps.RATIO)
