"""The float32 restatement of the image-space kernels (tests/render_f32.py) against the float64 oracles
(oracle/raster_oracle.py, oracle/points_oracle.py).  No GPU.

Outside the oracles' ambiguous classes (a pixel centre within MARGIN_PX of an edge, a runner-up depth within ZTOL, a
point's d within MARGIN r^2 of r^2, K-th and (K+1)-th depths within ZTOL) coverage, selection and winners must be equal;
the ambiguous count is printed.  Every value is held, entry by entry, to |v32 - v64| <= kappa u S with u = 2^-24 and S
the running error bound of the kernel's operation order (render_f32.Rb), which includes the rounding of the float32
screen coordinates and the cancellation in 1 - alpha near alpha = 1.  Each kappa is about 3x the largest ratio
|v32 - v64| / (u S) measured on these scenes (printed next to it); since S sums every rounding's worst case to first
order, a ratio above 1 means the restatement is wrong or the bound misses an error source.
"""
import numpy as np
import pytest

import render_f32 as rf
import render_scenes as rs
from oracle import points_oracle as po
from oracle import raster_oracle as ro

MARGIN_PX, ZTOL, MARGIN = 2e-3, 1e-6, 2e-4
HUGE_PX = 1e4
# about 3x the largest ratio measured on these scenes (deterministic CPU arithmetic): bary 0.32, zbuf 0.017, images 0.86,
# grad 0.88
KAPPA = dict(bary=1.0, zbuf=0.05, images=2.5, grad=2.5)


def ratio(a, b, S):
    """max |a - b| / (u S) over the entries; inf when a nonzero difference meets S = 0.  The float32 and float64 values
    must be non-finite at the same entries, with the same infinities there."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.array_equal(np.isfinite(a), np.isfinite(b)), "finiteness differs"
    assert np.array_equal(a[np.isinf(a)], b[np.isinf(b)]) and np.array_equal(np.isnan(a), np.isnan(b))
    d = np.abs(a - b)
    S = np.asarray(S, np.float64)
    m = np.isfinite(d)
    if not m.any():
        return 0.0
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(d[m] == 0, 0.0, d[m] / (rf.U * S[m]))
    return float(r.max())


MESH = {
    "sphere": lambda: rs.mesh_sphere(2, 200, 260, 1),
    "tile_counts": rs.mesh_tile_counts,
    "adversarial": lambda: rs.mesh_adversarial(1e-6),
    "adversarial_neg": lambda: rs.mesh_adversarial(-2.0),
    "many_frames": lambda: rs.mesh_many_frames(512),
}


@pytest.mark.parametrize("name", sorted(MESH))
def test_mesh_restatement_against_float64(name):
    sc = MESH[name]()
    V, F, C, H, W = sc["verts"], sc["faces"], sc["cams"], sc["H"], sc["W"]
    r = rf.rasterize_meshes(V, F, C, H, W, sc["z_clip"], sc["area_eps"])
    o = ro.rasterize(V.astype(np.float64), F, C.astype(np.float64), H, W, z_clip=sc["z_clip"], area_eps=sc["area_eps"],
                     margin_px=MARGIN_PX, ztol=ZTOL)
    ok = ~o["ambiguous"]
    # a face whose float32 screen coordinates pass HUGE_PX is placed to a few pixels at best (an ulp of 1e6 is 1/16 px,
    # of 1e9 is 64 px): its whole bbox joins the ambiguous class here
    for n, rec in enumerate(r["recs"]):
        huge = rec["vis"] & (np.maximum(np.abs(rec["sx"]), np.abs(rec["sy"])).max(1) > HUGE_PX)
        for f in np.nonzero(huge)[0]:
            ok[n, rec["y0"][f]:rec["y1"][f] + 1, rec["x0"][f]:rec["x1"][f] + 1] = False
    assert np.array_equal(r["pix_to_face"][ok], o["pix_to_face"][ok])
    assert abs(r["skipped"] - o["skipped"]) <= o["skipped_ambiguous"]
    hit = ok & (o["pix_to_face"] >= 0)
    n_, row, col = np.nonzero(hit)
    Fn = F.shape[0]
    kb = kz = 0.0
    for n in np.unique(n_):
        s = n_ == n
        f = r["pix_to_face"][n, row[s], col[s]] - n * Fn
        rec = r["recs"][n]
        origin = np.stack([rec["x0"][f], rec["y0"][f]], 1).astype(np.float64)
        bp, zb = rf.mesh_bound(V[n], F, C[n], f, col[s].astype(np.float64), row[s].astype(np.float64), origin)
        for i in range(3):
            kb = max(kb, ratio(r["bary"][n, row[s], col[s], i], o["bary"][n, row[s], col[s], i], bp[i].e))
        kz = max(kz, ratio(r["zbuf"][n, row[s], col[s]], o["zbuf"][n, row[s], col[s]], zb.e))
    print(f"[f32 mesh {name}] covered={r['covered']} ambiguous={int((~ok).sum())} kappa bary={kb:.3f} "
          f"(bound {KAPPA['bary']}) zbuf={kz:.3f} (bound {KAPPA['zbuf']})")
    assert kb <= KAPPA["bary"] and kz <= KAPPA["zbuf"], (kb, kz)


POINTS = {
    "sphere_k50": lambda: rs.points_sphere(2, 200, 260, 0.01, 50, 1),
    "sphere_k1_subpixel": lambda: rs.points_sphere(1, 300, 300, 0.002, 1, 2),
    "crowd_k8": lambda: rs.points_crowd(8),
    "crowd_k64": lambda: rs.points_crowd(64),
    "edges": rs.points_edges,
    "frames_split1": lambda: rs.points_frames(split=1),
    "big_k64": rs.points_big_discs,
}


@pytest.mark.parametrize("name", sorted(POINTS))
def test_points_restatement_against_float64(name):
    sc = POINTS[name]()
    pts, feats, H, W, radius, K, split = (sc[k] for k in ("points", "features", "H", "W", "radius", "K", "split"))
    N, P = pts.shape[:2]
    sel = rf.rasterize_points(pts, feats, H, W, radius, K, split)
    r32 = float(np.float32(radius))          # the kernel's radius is the C ABI's float
    ref = po.select(pts.astype(np.float64), H, W, r32, K, margin=MARGIN, ztol=ZTOL)
    amb = ref["ambiguous"].reshape(-1)
    okr, oks = ~amb[ref["pix"]], ~amb[sel["pix"]]
    assert np.array_equal(ref["pix"][okr], sel["pix"][oks]) and np.array_equal(ref["rank"][okr], sel["rank"][oks])
    assert np.array_equal(ref["idx"][okr], sel["g"][oks])
    assert sel["skipped"] == ref["skipped"]
    f64 = None if feats is None else feats.astype(np.float64)
    img = rf.composite(sel, 2).reshape(2, -1)
    iref = po.composite(ref, r32, f64, split, 2).reshape(2, -1)
    # the cotangent is zero on ambiguous pixels here only, where the two selections may differ
    cot = np.random.default_rng(1).normal(size=(2, N, H, W)).astype(np.float32) * ~ref["ambiguous"][None]
    g32 = rf.points_backward(sel, cot).reshape(-1, 3)
    g64 = po.composite_grad(ref, pts.astype(np.float64), r32, cot.astype(np.float64), f64, split).reshape(-1, 3)
    Si, Sg = rf.points_bound(sel, pts, feats, r32, cot)
    ki = max(ratio(img[gg][~amb], iref[gg][~amb], Si[gg].e[~amb]) for gg in range(2))
    kg = max(ratio(g32[:, j], g64[:, j], Sg[j].e) for j in range(2))
    print(f"[f32 points {name}] entries={len(sel['pix'])} ambiguous={int(amb.sum())} kappa images={ki:.3f} "
          f"(bound {KAPPA['images']}) grad={kg:.3f} (bound {KAPPA['grad']})")
    assert (g32[:, 2] == 0).all()
    assert ki <= KAPPA["images"] and kg <= KAPPA["grad"], (ki, kg)
