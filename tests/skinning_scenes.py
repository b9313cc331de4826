"""Deterministic scenes for the skinning kernels (csrc/lbs.cu with sample_skin24, skin_cell, lbs_blend_jac and
inverse_lbs_point of csrc/common.cuh) at production sizes and at the voxel border.  Everything is built from seeds on
the CPU; tests/test_skinning_scenes_cpu.py checks that each scene contains what it claims.

- Voxels (`voxel(name)`, [1, 24, D, H, W] fp32): "prod", synth's production stand-in (65, 225, 129); "sharp", the same
  shape with an independent softmax in every cell and no smoothing (the largest weight gradients and Hessians a voxel
  of that shape can have); "small", (1, 2, 7) unsmoothed: an axis of size 1 (always clamped) and one of size 2 (one cell);
  "toy", the (17, 33, 21) voxel of the older tests.
- Coordinate classes (`classed_points`), each defined by the kernel's own fp32 voxel coordinate
  u = unnormalize(((p - c) / e) * 2) before clamping (`coords32` restates it bit for bit): interior points, points
  exactly on 1, 2 or 3 lattice planes, u = size - 1 exactly and the nearest coordinates above and below it, the largest
  u <= 0 (the sampler clamps it to ix = 0 exactly with multiplier 0; no fp32 point reaches u = 0 itself on an axis of
  129, where u steps from -3.6e-6 to 2.4e-7), the largest u < 0 and the smallest u > 0, points 1e-3 to 1e3 outside the box through 1, 2 or 3 faces, and 1e30, +-inf or NaN in 1, 2 or 3
  coordinates.
- Frame layouts (`frames`): sorted, interleaved (p mod F), reversed, random and sorted with one empty frame, with
  out-of-range indices -1, F and 2^40 mixed in on request; `ppf_frames` gives the frames the points-per-frame form
  selects.  `chunk_stats` restates the backward's per-chunk slot numbering (256 points per chunk, slots in order of
  first appearance, 8 warps of 32).
- Bone matrices: `bone_A` from the kinematic chain on synth poses; `inverse_A` builds A directly so that the blended
  3 x 3 part has a chosen determinant (1e-7 to 10 in both signs) per frame, optionally ten frames at |det| = 1e-4 (1 + delta)
  around FastMinv's gate, plus exactly singular and NaN frames.
"""
import functools

import numpy as np
import torch

from oracle import oracle_torch as ot
from recmv_b200 import synth

CENTER = np.array(synth.BBOX_CENTER, dtype=np.float32)
EXTEND = np.float32(synth.BBOX_EXTEND)
SHAPES = {"prod": (65, 225, 129), "sharp": (65, 225, 129), "small": (1, 2, 7), "toy": (17, 33, 21)}
CHUNK = 256                       # points per chunk of the backward (kBwdChunk)
FRAME_COUNTS = (1, 3, 31, 32, 33, 255, 256, 257, 300)
LAYOUTS = ("sorted", "interleaved", "reversed", "random", "gap")
OUT_OF_RANGE = (-1, "F", 1 << 40)
PPFS = (1, 255, 257, 55233)
TEMPLATE_V = 55233                # vertices of the production garment template
CLASSES = ("interior", "plane1", "plane2", "plane3", "last", "last_up", "last_dn", "zero", "zero_dn", "zero_up",
           "out1", "out2", "out3", "nonfinite1", "nonfinite2", "nonfinite3")


@functools.lru_cache(maxsize=None)
def voxel(name):
    shape = SHAPES[name]
    if name == "sharp":
        g = synth.generator(23)
        return torch.softmax(torch.randn((1, 24) + shape, generator=g) * 4.0, dim=1).contiguous()
    if name == "small":
        return synth.skinning_voxel(shape, seed=5, smooth=0)
    return synth.skinning_voxel(shape, seed=7)


def channels_last(ws):
    return ws[0].permute(1, 2, 3, 0).contiguous()


def sizes_xyz(shape):
    """Lattice sizes along x, y, z (W, H, D) of a (D, H, W) voxel."""
    return np.array([shape[2], shape[1], shape[0]])


def coords32(ps, shape):
    """The kernels' voxel coordinate before clamping, in fp32 with every operation rounded as they round it:
    g = ((p - c) / e) * 2, u = (((g + 1) * size) - 1) * 0.5."""
    p = np.asarray(ps, dtype=np.float32)
    size = sizes_xyz(shape).astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        g = ((p - CENTER) / EXTEND) * np.float32(2)
        t = (g + np.float32(1)) * size
        return (t - np.float32(1)) * np.float32(0.5)


def _p_of_u(u, size, axis):
    """float64 position whose exact voxel coordinate on `axis` is u."""
    return float(CENTER[axis]) + float(EXTEND) / 2 * ((2 * u + 1) / size - 1)


def _search(p64, axis, shape, want, pick="near", span=24):
    """For each p64 (float64 [n]), the fp32 point among its neighbours within `span` ulps whose fp32 coordinate u on
    `axis` satisfies want(u): the nearest such point (pick "near"), or the one with the largest or smallest such u
    ("max", "min"); NaN where none does."""
    p32 = np.asarray(p64, dtype=np.float32)
    cands = [p32]
    up, dn = p32.copy(), p32.copy()
    for _ in range(span):
        up = np.nextafter(up, np.float32(np.inf))
        dn = np.nextafter(dn, np.float32(-np.inf))
        cands += [up, dn]
    out = np.full(p32.shape, np.nan, dtype=np.float32)
    best = np.full(p32.shape, np.nan, dtype=np.float32)
    size = np.float32(sizes_xyz(shape)[axis])
    for c in cands:
        g = ((c - CENTER[axis]) / EXTEND) * np.float32(2)
        u = ((g + np.float32(1)) * size - np.float32(1)) * np.float32(0.5)
        hit = want(u)
        if pick == "near":
            hit &= np.isnan(best)
        elif pick == "max":
            hit &= np.isnan(best) | (u > best)
        else:
            hit &= np.isnan(best) | (u < best)
        out[hit] = c[hit]
        best[hit] = u[hit]
    return out


def _interior(n, shape, rng):
    """n points whose coordinate lies strictly inside (0, size - 1) on every axis of size > 1 (the box centre on an
    axis of size 1)."""
    size = sizes_xyz(shape)
    p = np.empty((n, 3), dtype=np.float32)
    for a in range(3):
        if size[a] == 1:
            p[:, a] = CENTER[a]
            continue
        u = rng.uniform(0.02, size[a] - 1.02, n)
        p[:, a] = [_p_of_u(x, size[a], a) for x in u]
    return p


def _on_value(n, axis, shape, rng, target, want, pick="near"):
    """n fp32 coordinates on `axis` found near the float64 solution of u = target (float or array)."""
    size = sizes_xyz(shape)[axis]
    t = np.broadcast_to(np.asarray(target, dtype=np.float64), (n,))
    p64 = np.array([_p_of_u(x, size, axis) for x in t])
    return _search(p64, axis, shape, lambda u: want(u, t), pick)


def classed_points(shape, per_class=64, seed=0):
    """(ps [P,3] fp32, cls [P] int index into CLASSES, axes [P,3] bool: the axes the class applies to)."""
    rng = np.random.default_rng(seed)
    size = sizes_xyz(shape)
    big = [a for a in range(3) if size[a] >= 3]     # axes with an interior lattice plane
    pts, cls, axes = [], [], []

    def add(name, p, ax):
        keep = np.isfinite(p).all(1) | name.startswith("nonfinite")
        pts.append(p[keep])
        cls.append(np.full(keep.sum(), CLASSES.index(name)))
        axes.append(ax[keep])

    n = per_class
    add("interior", _interior(n, shape, rng), np.zeros((n, 3), dtype=bool))
    for k in (1, 2, 3):
        if len(big) < k:
            continue
        p = _interior(n, shape, rng)
        ax = np.zeros((n, 3), dtype=bool)
        for i in range(n):
            ax[i, rng.choice(big, k, replace=False)] = True
        for a in range(3):
            sel = ax[:, a]
            if sel.any():
                tgt = rng.integers(1, size[a] - 1, sel.sum()).astype(np.float64)
                p[sel, a] = _on_value(sel.sum(), a, shape, rng, tgt, lambda u, t: u == t)
        add(f"plane{k}", p, ax)
    for name, target, want, pick in (("last", "hi", lambda u, t: u == t, "near"),
                                     ("last_up", "hi", lambda u, t: u > t, "min"),
                                     ("last_dn", "hi", lambda u, t: u < t, "max"),
                                     ("zero", 0.0, lambda u, t: u <= t, "max"),
                                     ("zero_dn", 0.0, lambda u, t: u < t, "max"),
                                     ("zero_up", 0.0, lambda u, t: u > t, "min")):
        p = _interior(n, shape, rng)
        ax = np.zeros((n, 3), dtype=bool)
        a_of = np.arange(n) % 3
        for a in range(3):
            sel = a_of == a
            if name in ("last_dn", "zero_up") and size[a] == 1:
                continue    # on an axis of size 1 these coincide with zero_dn and last_up
            tgt = float(size[a] - 1) if target == "hi" else target
            p[sel, a] = _on_value(sel.sum(), a, shape, rng, tgt, want, pick)
            ax[sel, a] = True
        keep = ax.any(1)
        add(name, p[keep], ax[keep])
    for k in (1, 2, 3):
        p = _interior(n, shape, rng)
        ax = np.zeros((n, 3), dtype=bool)
        for i in range(n):
            for a in rng.choice(3, k, replace=False):
                ax[i, a] = True
                side = 1.0 if rng.random() < 0.5 else -1.0
                p[i, a] = CENTER[a] + side * (EXTEND / 2 + 10.0 ** rng.uniform(-3, 3))
        add(f"out{k}", p, ax)
    specials = np.array([1e30, np.inf, -np.inf, np.nan], dtype=np.float32)
    for k in (1, 2, 3):
        p = _interior(n, shape, rng)
        ax = np.zeros((n, 3), dtype=bool)
        for i in range(n):
            for j, a in enumerate(rng.choice(3, k, replace=False)):
                ax[i, a] = True
                p[i, a] = specials[(i + j) % 4] * (-1 if (i // 4) % 2 and (i + j) % 4 == 0 else 1)
        add(f"nonfinite{k}", p, ax)
    return np.concatenate(pts), np.concatenate(cls), np.concatenate(axes)


def random_points(P, seed, spread=1.1):
    """P fp32 points, uniform in the box widened by `spread` (about 25 % outside at 1.1)."""
    g = synth.generator(seed)
    return ((torch.rand((P, 3), generator=g) - 0.5) * float(EXTEND) * spread).contiguous()


# ------------------------------------------------------------------ frames
def frames(P, F, layout, seed=0, out_of_range=False):
    """int64 [P] frame indices.  'gap' is 'sorted' with frame F // 2 given no point (F >= 2)."""
    p = np.arange(P, dtype=np.int64)
    if layout == "sorted":
        f = p * F // max(P, 1)
    elif layout == "interleaved":
        f = p % F
    elif layout == "reversed":
        f = F - 1 - p * F // max(P, 1)
    elif layout == "random":
        f = np.random.default_rng(seed).integers(0, F, P)
    elif layout == "gap":
        f = p * F // max(P, 1)
        f[f == F // 2] = min(F // 2 + 1, F - 1)
    else:
        raise ValueError(layout)
    if out_of_range:
        f = f.copy()
        f[1::7] = -1
        f[2::7] = F
        f[3::7] = 1 << 40
    return f


def clamp_frames(f, F):
    return np.clip(f, 0, F - 1)


def ppf_frames(P, ppf, F):
    """The frames the points-per-frame form selects: clamp(p // ppf, 0, F - 1)."""
    return np.minimum(np.arange(P, dtype=np.int64) // ppf, F - 1)


def chunk_stats(f):
    """Per chunk of the backward: (distinct frames, warps in which some point opens a slot) for clamped frames f."""
    P = len(f)
    nch = (P + CHUNK - 1) // CHUNK
    distinct = np.zeros(nch, dtype=np.int64)
    warps = np.zeros(nch, dtype=np.int64)
    for c in range(nch):
        seg = f[c * CHUNK:(c + 1) * CHUNK]
        _, first = np.unique(seg, return_index=True)
        distinct[c] = len(first)
        warps[c] = len(np.unique(first // 32))
    return distinct, warps


# ------------------------------------------------------------------ bone matrices
@functools.lru_cache(maxsize=None)
def _skeleton():
    Js, parents, ip = synth.skeleton()
    R = ot.batch_rodrigues(ip.view(-1, 3).double()).view(24, 3, 3)
    # the init-pose inverse of LBSkinner (model/Deformer.py:280-303), in float64
    Rs, Ts = [R[0]], [Js[0].double()]
    for i in range(1, 24):
        pi = int(parents[i])
        Rs.append(Rs[pi] @ R[i])
        Ts.append(Rs[pi] @ (Js[i] - Js[pi]).double() + Ts[pi])
    inv = torch.zeros(24, 4, 4, dtype=torch.float64)
    inv[:, 3, 3] = 1
    for i in range(24):
        inv[i, :3, :3] = Rs[i].t()
        inv[i, :3, 3] = -(Ts[i] @ Rs[i])
    return Js, parents, inv.float()


def bone_A(F, seed=4):
    """(A [F,24,4,4] fp32, trans [F,3] fp32): the kinematic chain on synth poses, as LBSkinner builds it."""
    Js, parents, ip = _skeleton()
    poses, trans = synth.poses_trans(F, seed=seed)
    A = ot.bone_matrices(poses.double(), Js.double(), parents, ip.double())
    return A.float().contiguous(), trans.contiguous()


# relative offsets from the FastMinv gate |det| = 1e-4 of the frames `inverse_dets(F, gate=True)` ends with: +-10 % and
# +-3 % lie outside fp32's rounding of det, the others straddle or sit inside it (the 1e-3 bone spread moves a row's
# det by up to 0.3 %)
GATE_OFFSETS = (-0.1, -0.03, -0.01, -1e-3, -1e-6, 1e-6, 1e-3, 0.01, 0.03, 0.1)


def inverse_dets(F, gate=False):
    """The target determinant of each frame of `inverse_A`: |det| log-spaced from 1e-7 to 10, alternating sign; with
    `gate`, the last len(GATE_OFFSETS) frames instead get |det| = 1e-4 (1 + offset), alternating sign."""
    mag = np.logspace(-7, 1, F)
    if gate:
        mag[F - len(GATE_OFFSETS):] = 1e-4 * (1 + np.array(GATE_OFFSETS))
    return mag * np.where(np.arange(F) % 2 == 0, 1.0, -1.0)


def inverse_A(F, seed=3, singular=(), nan=(), gate=False):
    """(A [F,24,4,4], trans [F,3]) fp32.  Frame f has A_b[:3,:3] = M_f (1 + 1e-3 r_b) for one random M_f with
    det M_f = inverse_dets(F, gate)[f], so every blended M is M_f times about 1 (and its det about det M_f); bone
    translations are independent.  Frames in `singular` get M_f with an exactly zero last row; frames in `nan` a NaN
    entry in every bone."""
    rng = np.random.default_rng(seed)
    dets = inverse_dets(F, gate)
    A = np.zeros((F, 24, 4, 4))
    for f in range(F):
        Q1, _ = np.linalg.qr(rng.standard_normal((3, 3)))
        Q2, _ = np.linalg.qr(rng.standard_normal((3, 3)))
        s1 = 10.0 ** rng.uniform(-0.3, 0.3)
        s2 = 10.0 ** rng.uniform(-0.3, 0.3)
        d = abs(dets[f])
        M = Q1 @ np.diag([s1, s2, d / (s1 * s2)]) @ Q2
        M *= np.sign(dets[f]) * np.sign(np.linalg.det(M))
        if f in singular:
            M[2] = 0.0
        r = rng.uniform(-1, 1, 24)
        A[f, :, :3, :3] = M[None] * (1 + 1e-3 * r)[:, None, None]
        if f in singular:
            A[f, :, 2, :3] = 0.0
        A[f, :, :3, 3] = rng.uniform(-0.5, 0.5, (24, 3))
        A[f, :, 3, 3] = 1.0
        if f in nan:
            A[f, :, 1, 2] = np.nan
    trans = rng.uniform(-0.05, 0.05, (F, 3))
    return torch.from_numpy(A).float().contiguous(), torch.from_numpy(trans).float().contiguous()
