"""Writes tests/golden/fl_proj_ref.npz: the reference's OWN `fl_proj_loss` (engineer/core/fl_optimizer.py:72-110),
unmodified, run in float64 with autograd, with its pytorch3d `chamfer_distance` rebound to the float64 oracle
(oracle/knn_oracle.chamfer_f64, pytorch3d 0.4's formula).  Needs the reference source tree (oracle/refload.py).

One case with the training shape: N = 3 frames, 4 + 2 curves (a two-garment outfit) of up to 200 screen points against
100 annotation points each, weights != 1, ~70 % of the points visible with unequal counts per frame, one frame of
curve 0 with no visible point, curve 3 invisible in every frame, and curves of unequal length (padding).  Inputs are
float32 values.  Every nearest neighbour is separated from the second-best by more than 1e-3 relative, so float32
and float64 pick the same neighbours (ties are tested separately).

    python tests/golden/make_golden_fl_proj.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import knn_oracle, refload  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "fl_proj_ref.npz")
N, M = 3, 100
P = [200, 200, 170, 200, 200, 150]
WEIGHTS = [1.0, 0.5, 2.0, 1.0, 1.5, 1.0]
GAP = 1e-3


def near_ties(q, c):
    """Rows of q whose best and second-best squared distance to c are within GAP relative."""
    if len(q) == 0 or len(c) < 2:
        return np.zeros(len(q), dtype=bool)
    d = np.sort(((q[:, None, :].astype(np.float64) - c[None].astype(np.float64)) ** 2).sum(-1), axis=1)
    return d[:, 1] - d[:, 0] <= GAP * np.maximum(d[:, 0], 1e-30)


def make_case(seed):
    g = np.random.default_rng(seed)
    pts = [(g.uniform(0, 512, size=(N, p, 3))).astype(np.float32) for p in P]
    gts = [(g.uniform(0, 512, size=(N, M, 2))).astype(np.float32) for _ in P]
    masks = [g.random((N, p)) < 0.7 for p in P]
    masks[0][1] = False
    masks[3][:] = False
    for _ in range(100):
        bad = 0
        for c in range(len(P)):
            for n in range(N):
                v = np.nonzero(masks[c][n])[0]
                bx = v[near_ties(pts[c][n, v, :2], gts[c][n])]
                by = np.nonzero(near_ties(gts[c][n], pts[c][n, v, :2]))[0]
                pts[c][n, bx] = g.uniform(0, 512, size=(len(bx), 3)).astype(np.float32)
                gts[c][n, by] = g.uniform(0, 512, size=(len(by), 2)).astype(np.float32)
                bad += len(bx) + len(by)
        if bad == 0:
            return pts, gts, masks
    raise RuntimeError("could not separate the neighbours")


def main():
    refload.load()
    import engineer.core.fl_optimizer as flo   # after refload.load(): a direct import is circular
    flo.chamfer_distance = knn_oracle.chamfer_f64
    pts, gts, masks = make_case(7)
    fl_pts = [torch.tensor(p, dtype=torch.float64, requires_grad=True) for p in pts]
    gt = [torch.tensor(x, dtype=torch.float64) for x in gts]
    fl_masks = [torch.tensor(m)[..., None].expand(-1, -1, 3) for m in masks]   # per point, as the call site builds it
    loss = flo.fl_proj_loss(fl_pts, gt, fl_masks, WEIGHTS)
    grads = torch.autograd.grad(loss, fl_pts)
    out = {"weights": np.array(WEIGHTS), "loss": np.array(loss.item())}
    for c in range(len(P)):
        out[f"pts_{c}"], out[f"gt_{c}"], out[f"mask_{c}"] = pts[c], gts[c], masks[c]
        out[f"grad_{c}"] = grads[c].numpy()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, "loss", loss.item())


if __name__ == "__main__":
    main()
