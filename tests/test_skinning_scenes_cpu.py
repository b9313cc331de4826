"""The skinning scenes (tests/skinning_scenes.py) contain what they claim: voxel shapes and weights, every coordinate
class at the kernels' own fp32 voxel coordinate, the chunk structures the frame layouts give the backward, and the
determinants of the inverse's bone matrices."""
import numpy as np
import pytest
import torch

import skinning_scenes as sc
from oracle import oracle_torch as ot
from recmv_b200 import synth


@pytest.mark.parametrize("name", ["prod", "sharp", "small"])
def test_voxels(name):
    ws = sc.voxel(name)
    assert ws.shape == (1, 24) + sc.SHAPES[name] and ws.dtype == torch.float32
    assert (ws > 0).all() and torch.allclose(ws.sum(1), torch.ones(1), atol=2e-6)
    if name == "sharp":
        # no smoothing: neighbouring cells are independent, so the weights jump between them as much as anywhere
        d = (ws[..., 1:] - ws[..., :-1]).abs().amax(1)
        assert d.mean() > 0.5
        p = sc.voxel("prod")
        assert (p[..., 1:] - p[..., :-1]).abs().amax(1).mean() < 0.1
    if name == "small":
        assert sorted(sc.SHAPES[name])[:2] == [1, 2]
    cl = sc.channels_last(ws)
    assert cl.shape == sc.SHAPES[name] + (24,) and torch.equal(cl[0, 0, 0], ws[0, :, 0, 0, 0])


def test_coords32_is_the_fp32_sampler_coordinate():
    """numpy's fp32 restatement equals ot._unnormalize_clip of the same fp32 g (before its clamp) bit for bit."""
    ps = sc.random_points(4096, seed=1, spread=1.3).numpy()
    shape = sc.SHAPES["prod"]
    u = sc.coords32(ps, shape)
    g = torch.from_numpy(((ps - sc.CENTER) / sc.EXTEND) * np.float32(2))
    for a, size in enumerate(sc.sizes_xyz(shape)):
        ref = ot._unnormalize_clip(g[:, a], int(size))
        inside = (u[:, a] > 0) & (u[:, a] < size - 1)
        assert torch.equal(ref[torch.from_numpy(inside)], torch.from_numpy(u[inside, a]))
        assert torch.equal(ref, torch.from_numpy(u[:, a]).clamp(0, float(size - 1)))


@pytest.mark.parametrize("name", ["prod", "small"])
def test_coordinate_classes(name):
    shape = sc.SHAPES[name]
    size = sc.sizes_xyz(shape)
    ps, cls, axes = sc.classed_points(shape, per_class=64, seed=2)
    u = sc.coords32(ps, shape)
    seen = set()
    for k, cname in enumerate(sc.CLASSES):
        sel = cls == k
        if not sel.any():
            continue
        seen.add(cname)
        uu, ax = u[sel], axes[sel]
        free = ~ax
        # the axes a class does not name are strictly inside (0, size - 1) where that interval is not empty
        for a in range(3):
            if size[a] > 1 and not cname.startswith(("out", "nonfinite")):
                m = free[:, a]
                assert ((uu[m, a] > 0) & (uu[m, a] < size[a] - 1)).all(), (cname, a)
        if cname.startswith("plane"):
            kk = int(cname[-1])
            assert (ax.sum(1) == kk).all()
            assert (uu[ax] == np.round(uu[ax])).all() and (uu[ax] >= 1).all()
            assert all((uu[ax[:, a], a] <= size[a] - 2).all() for a in range(3))
        elif cname in ("last", "last_up", "last_dn", "zero", "zero_dn", "zero_up"):
            assert (ax.sum(1) == 1).all()
            for a in range(3):
                v = uu[ax[:, a], a]
                if not len(v):
                    continue
                t = size[a] - 1 if cname.startswith("last") else 0
                # one step of u near t: an ulp of p moves u by about size / 2 ulps of g
                tol = 64 * np.spacing(np.float32(max(t, 1))) + float(size[a]) * 2.0 ** -20
                if cname == "last":
                    assert (v == t).all()
                elif cname == "zero":
                    assert (v <= 0).all() and (v > -tol).all()
                    if a == 0 and size[0] == 129:
                        assert (v < 0).all()      # no fp32 point reaches u = 0 on this axis: clamped to ix = 0
                elif cname.endswith("_up"):
                    assert (v > t).all() and (v - t <= tol).all()
                else:
                    assert (v < t).all() and (t - v <= tol).all()
        elif cname.startswith("out"):
            kk = int(cname[-1])
            assert (ax.sum(1) == kk).all()
            d = np.abs(ps[sel] - sc.CENTER) - sc.EXTEND / 2
            assert (d[ax] >= 0.9e-3).all() and (d[ax] <= 1.01e3).all() and (d[~ax] < 0).all()
            assert ((uu[ax] <= 0) | (uu[ax] >= np.broadcast_to(size - 1, uu.shape)[ax])).all()
        elif cname.startswith("nonfinite"):
            kk = int(cname[-1])
            p = ps[sel]
            assert (ax.sum(1) == kk).all() and np.isfinite(p[~ax]).all()
            vals = p[ax]
            assert np.isnan(vals).any() and np.isposinf(vals).any() and np.isneginf(vals).any()
            assert (np.abs(vals[np.isfinite(vals)]) == np.float32(1e30)).all()
    expect = set(sc.CLASSES) - ({"plane2", "plane3"} if name == "small" else set())
    assert seen == expect, expect - seen


def test_frame_layouts_reach_every_slot_structure():
    counts = {}
    full, eight_warps = False, False
    for F in sc.FRAME_COUNTS:
        for layout in sc.LAYOUTS:
            for P in (1, 255, 256, 257, 5 * 256 - 3, 32 * 256, 33 * 256):
                f = sc.frames(P, F, layout, seed=F)
                assert f.min() >= 0 and f.max() < F
                d, w = sc.chunk_stats(f)
                counts[len(d)] = True
                full |= bool((d == 256).any())
                eight_warps |= bool((w == 8).any())
    assert full and eight_warps
    assert all(counts.get(n) for n in (5, 32, 33))
    d, w = sc.chunk_stats(sc.frames(10 ** 6 + 77, 3, "random"))      # the largest backward size: 3 907 chunks
    assert len(d) == 3907 and (d == 3).all()
    g = sc.frames(4096, 33, "gap")
    assert (np.bincount(g, minlength=33) == 0).sum() == 1
    o = sc.frames(4096, 31, "random", out_of_range=True)
    assert {-1, 31, 1 << 40} <= set(o.tolist())
    assert (sc.clamp_frames(o, 31) == np.clip(o, 0, 30)).all()


def test_ppf_frames_clamp_the_tail():
    for ppf in sc.PPFS:
        F = 3
        P = ppf * F + 77
        f = sc.ppf_frames(P, ppf, F)
        assert (f[: ppf * F] == np.arange(ppf * F) // ppf).all() and (f[ppf * F:] == F - 1).all()


def test_inverse_bone_matrices_sweep_the_determinant():
    F = 64
    A, trans = sc.inverse_A(F, singular=(5,), nan=(9,))
    dets = sc.inverse_dets(F)
    assert dets.min() < -1 and dets.max() > 1 and np.abs(dets).min() <= 1.01e-7
    M = A[:, :, :3, :3].double()
    for f in range(F):
        if f == 9:
            assert torch.isnan(M[f]).any(1).any(1).all()
            continue
        d = torch.linalg.det(M[f])
        if f == 5:
            assert (d == 0).all() and (A[f, :, 2, :3] == 0).all()
            continue
        # about det M_f, up to the 1e-3 bone spread and the fp32 rounding of M's O(1) entries
        assert ((d - dets[f]).abs() < 5e-3 * abs(dets[f]) + 2e-6).all(), f
        if abs(dets[f]) > 1e-3:
            assert (torch.sign(d) == np.sign(dets[f])).all()
    assert (A[:, :, 3, :3] == 0).all() and (A[:, :, 3, 3] == 1).all() and trans.shape == (F, 3)
    # frames at the FastMinv gate: float64 det within 0.5 % of 1e-4 (1 + offset), on both sides of the gate
    Ag, _ = sc.inverse_A(F, gate=True)
    n = len(sc.GATE_OFFSETS)
    dg = torch.linalg.det(Ag[F - n:, :, :3, :3].double()).abs()
    tgt = torch.tensor([1e-4 * (1 + o) for o in sc.GATE_OFFSETS], dtype=torch.float64)[:, None]
    assert ((dg / tgt - 1).abs() < 5e-3).all()
    assert (dg < 1e-4).any() and (dg >= 1e-4).any()


def test_bone_A_is_the_kinematic_chain():
    A, trans = sc.bone_A(3)
    Js, parents, ip = sc._skeleton()
    poses, tr = synth.poses_trans(3, seed=4)
    ref = ot.bone_matrices(poses, Js, parents, ip)
    assert torch.allclose(A, ref, atol=1e-5) and torch.equal(trans, tr)
