"""The float32 restatement of the shading kernels (tests/shade_f32.py) against float64.  No GPU.

Every normal and every shaded channel is held, entry by entry, to |v32 - v64| <= kappa u S with u = 2^-24 and S the
running error bound of the kernel's operation order (shade_f32.normals_bound / phong_bound, built on render_f32.Rb).
The normals' S carries the cancellation of each vertex's sum, so a vertex whose contributions cancel to about 0 is
held to its partial sums' scale, not to its value's.  The float64 values of the same operation order also equal the
float64 oracle (oracle/shade_oracle.py) to 1e-12.  Each kappa is about 3x the largest ratio measured on these scenes
(deterministic CPU arithmetic, printed next to it); a ratio above 1 would mean the restatement is wrong or the bound
misses an error source.  Entries whose float64 value leaves the float32 range (the 1e18 mesh, whose squared norm
overflows in float32) or that depend on the NaN vertex are excluded and counted.
"""
import numpy as np
import pytest

import render_f32 as rf
import shade_f32 as sf
import shade_scenes as ss
from oracle import shade_oracle as so

# measured: normals 0.39 (the adversarial mesh; 0.33 the 1e5 fan, 0.21 the sphere), Phong 0.39
KAPPA = dict(normals=1.2, phong=1.2)


def ratio(a, b, S):
    a, b, S = (np.asarray(x, np.float64) for x in (a, b, S))
    d = np.abs(a - b)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(d == 0, 0.0, d / (rf.U * S))
    return float(r.max(initial=0.0))


def unnormalised_norm2(v, f):
    """|sum of the cross products|^2 per vertex in float64."""
    v = v.astype(np.float64)
    V = v.shape[1]
    f = f[((f >= 0) & (f < V)).all(1)]
    acc = np.zeros(v.shape)
    for k in range(3):
        a, b, c = f[:, k], f[:, (k + 1) % 3], f[:, (k + 2) % 3]
        for n in range(v.shape[0]):
            np.add.at(acc[n], a, np.cross(v[n, b] - v[n, a], v[n, c] - v[n, a]))
    return (acc ** 2).sum(-1)


NORMALS = {
    "uv_sphere": lambda: ss.uv_sphere(60, 80, 3, 1),
    "fan_1e5": lambda: ss.fan(100_000),
    "adversarial": ss.adversarial_mesh,
}


@pytest.mark.parametrize("name", sorted(NORMALS))
def test_normals_restatement_against_float64(name):
    v, f = NORMALS[name]()
    n32 = sf.vertex_normals(v, f)
    b = sf.normals_bound(v, f)
    v64 = np.stack([x.v for x in b], -1)
    assert np.nanmax(np.abs(v64 - so.vertex_normals(v.astype(np.float64), f))) < 1e-12
    # float64 intermediates beyond the float32 range, and whatever a NaN reaches, are not comparable
    e = np.stack([x.e for x in b], -1)
    keep = np.isfinite(e).all(-1) & ~np.isnan(v64).any(-1) & ~np.isnan(n32).any(-1)
    keep &= unnormalised_norm2(v, f) < np.finfo(np.float32).max
    k = max(ratio(n32[..., i][keep], b[i].v[keep], b[i].e[keep]) for i in range(3))
    zero = (v64 == 0).all(-1) & keep
    print(f"[f32 normals {name}] V={v.shape[1]} F={len(f)} kappa {k:.3f} (bound {KAPPA['normals']}); "
          f"{int((~keep).sum())} entries excluded; {int(zero.sum())} vertices exactly 0 in float64")
    assert (n32[zero] == 0).all()
    assert k <= KAPPA["normals"], k


def test_phong_restatement_against_float64():
    p2f, bary, verts, normals, colors, faces, centre, light = ss.hand_fragments()
    N = p2f.shape[0]
    worst = 0.0
    for sh in (0.0, 1.0, 10.5, 64.0):
        P = np.zeros((N, 28), np.float32)
        P[:, 0:3], P[:, 3:6] = centre, light
        P[:, 6:9], P[:, 9:12], P[:, 12:15], P[:, 15:24], P[:, 24], P[:, 25:28] = 0.5, 0.3, 0.2, 1.0, sh, 0.3
        img, _ = sf.phong(p2f, bary, verts, normals, colors, faces, P)
        rgb, cov, _ = sf.phong_bound(p2f, bary, verts, normals, colors, faces, P)
        got = img.reshape(-1, 4)[np.flatnonzero(cov.reshape(-1))]
        worst = max([worst] + [ratio(got[:, j], rgb[j].v, rgb[j].e) for j in range(3)])
        ref = so.phong(p2f, bary, verts, normals, colors, faces, P[:, 0:3], P[:, 3:6], P[:, 6:9], P[:, 9:12],
                       P[:, 12:15], P[:, 15:18], P[:, 18:21], P[:, 21:24], P[:, 24:25], P[:, 25:28])
        assert np.array_equal(img[~cov.reshape(img.shape[:3])], ref[~cov.reshape(img.shape[:3])].astype(np.float32))
    print(f"[f32 phong] kappa {worst:.3f} (bound {KAPPA['phong']})")
    assert worst <= KAPPA["phong"], worst
