"""Writes tests/golden/nricp_ref.npz: the reference's OWN `NRICP_Optimizer_AdamW.fitting`
(engineer/optimizer/nricp_optimizer.py:321-448), unmodified, run on the CPU in float64, with the module's pytorch3d
`Meshes`, `mesh_laplacian_smoothing`, `knn_points` and `knn_gather` rebound to the float64 stand-ins of
tests/nricp_oracle.py (pytorch3d 0.4's forms).  Its `mesh_boundary` and `Local_Affine` are the reference's own, and
FastMinv is oracle/refload.py's restatement.  Needs the reference source tree.

Scene: an open 20 x 20 grid patch (so it has a boundary) fitted onto a bumped, denser copy.  A band of the target has
its faces flipped, so its normals face away and the gate rejects the vertices that land there, and some target points
are masked out by nricp_masks.  Two cases of 3 epochs with a milestone after the first: gamma = 1 and gamma = 2.
Recorded per case: the vertices at every epoch start (what the reference's `knn_points` sees), the final vertices and
the printed per-epoch terms (avg_update, valid count, dis, stiffness, laplacian, total).

    python tests/golden/make_golden_nricp.py
"""
import contextlib
import io
import os
import re
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import nricp_oracle as no  # noqa: E402
from oracle import refload, shade_oracle  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "nricp_ref.npz")
CASES = [dict(gamma=1.0, threshold=0.3), dict(gamma=2.0, threshold=0.5)]
EPOCH, INNER, MILE = 3, 20, [1]
SW, LW = [5.0, 2.0], [25.0, 25.0]


def grid(n, lo, hi):
    t = np.linspace(lo, hi, n)
    X, Y = np.meshgrid(t, t, indexing="ij")
    verts = np.stack([X.ravel(), Y.ravel(), np.zeros(n * n)], axis=1)
    faces = []
    for i in range(n - 1):
        for j in range(n - 1):
            a, b, c, d = i * n + j, (i + 1) * n + j, (i + 1) * n + j + 1, i * n + j + 1
            faces += [[a, b, c], [a, c, d]]
    return verts, np.array(faces, dtype=np.int64)


def scene():
    g = np.random.default_rng(3)
    src_v, src_f = grid(20, -1.0, 1.0)
    src_v[:, :2] += g.uniform(-0.03, 0.03, size=(len(src_v), 2))
    src_v[:, 2] = 0.05 * np.sin(2.0 * src_v[:, 0]) + g.uniform(-0.03, 0.03, size=len(src_v))
    tgt_v, tgt_f = grid(27, -1.15, 1.15)
    x, y = tgt_v[:, 0], tgt_v[:, 1]
    tgt_v[:, 2] = 0.12 * np.exp(-((x - 0.3) ** 2 + (y + 0.2) ** 2) / 0.15) + 0.06 * np.sin(2.5 * y) + 0.03
    tgt_v[:, :2] += g.uniform(-0.01, 0.01, size=(len(tgt_v), 2))
    cx = tgt_v[tgt_f].mean(axis=1)[:, 0]
    band = (cx > -0.75) & (cx < -0.45)                 # these faces face away: their normals point down
    tgt_f[band] = tgt_f[band][:, [0, 2, 1]]
    masks = (g.random(len(tgt_v)) > 0.1).astype(np.float64)
    return src_v, src_f, tgt_v, tgt_f, masks


class Slice:
    """The members of the garment template that `fitting` uses."""

    def __init__(self, v, f):
        self.vertices, self.faces = torch.tensor(v), torch.tensor(f)

    def get_outlayer_idx(self, *types):
        return []

    def verts_normals_packed(self):
        return torch.tensor(shade_oracle.vertex_normals(self.vertices[None].numpy(), self.faces.numpy())[0])

    def edges_packed(self):
        return torch.tensor(no.adjacency(self.faces.numpy(), len(self.vertices))["edges"])

    def update_padded(self, new_verts):
        self.vertices = new_verts[0]


class Target:
    def __init__(self, v, f):
        self.v, self.f = torch.tensor(v), torch.tensor(f)

    def verts_packed(self):
        return self.v

    def faces_packed(self):
        return self.f

    def verts_normals_packed(self):
        return torch.tensor(shade_oracle.vertex_normals(self.v[None].numpy(), self.f.numpy())[0])


LINE = re.compile(r"avg_update:(\S+) valid(\d+)/\d+: dis:(\S+), stiffness:(\S+), laplacian:(\S+), total:(\S+)")


def main():
    torch.set_default_dtype(torch.float64)
    refload.load()
    import engineer.optimizer.nricp_optimizer as nro   # after refload.load(): a direct import is circular
    seen = []

    def knn_points(p1, p2, K=1):
        seen.append(p1[0].detach().numpy().copy())
        return no.knn_points(p1, p2, K)

    nro.Meshes, nro.mesh_laplacian_smoothing = no.Meshes, no.laplacian_smoothing_torch
    nro.knn_points, nro.knn_gather = knn_points, no.knn_gather
    src_v, src_f, tgt_v, tgt_f, masks = scene()
    out = dict(src_v=src_v, src_f=src_f, tgt_v=tgt_v, tgt_f=tgt_f, masks=masks, epoch=EPOCH, inner_iter=INNER,
               mile_stone=np.array(MILE), stiffness_weight=np.array(SW), laplacian_weight=np.array(LW))
    for k, case in enumerate(CASES):
        seen.clear()
        opt = nro.NRICP_Optimizer_AdamW(epoch=EPOCH, dense_pcl=1, use_normal=True, stiffness_weight=list(SW),
                                        mile_stone=list(MILE), inner_iter=INNER, laplacian_weight=list(LW),
                                        gamma=case["gamma"], threshold=case["threshold"], device="cpu")
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            loss, sl = opt(smpl_slice=Slice(src_v, src_f), cano_meshes=Target(tgt_v, tgt_f), save_path=None,
                           garment_name="patch", static_pts_type=[], nricp_masks=torch.tensor(masks))
        lines = [LINE.search(s) for s in buf.getvalue().splitlines()]
        stats = np.array([[float(x) for x in m.groups()] for m in lines if m])
        assert stats.shape == (EPOCH, 6), buf.getvalue()
        out[f"gamma_{k}"], out[f"threshold_{k}"] = case["gamma"], case["threshold"]
        out[f"epoch_v_{k}"] = np.stack(seen)
        out[f"final_v_{k}"] = sl.vertices.detach().numpy()
        out[f"stats_{k}"] = stats
        out[f"loss_{k}"] = float(loss)
        print(buf.getvalue(), end="")
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
