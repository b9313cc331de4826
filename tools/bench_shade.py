"""Time the shading of the rasterized garment meshes: rasterize (recmv_rasterize_meshes), vertex normals
(recmv_vertex_normals) and hard Phong (recmv_shade_phong), each with CUDA events (median of --iters calls), at
1080 x 1080 with N = 1 and 4 frames of the marching-cubes mesh of synth.sphere_sdf_grid at 257^3 (201 548 faces)
deformed by LBSkinner.  Next to them, the same normals and shading written as a torch graph on the same GPU
(index_add normals, gathers and element-wise Phong), the comparison pytorch3d would have been.  The card, power limit
and SM clock come from the same run.

  python tools/bench_shade.py [--iters 30] [--out FILE.json]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as tF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_raster import card, cameras, deform, scene, timed  # noqa: E402
from recmv_b200 import ops, raster  # noqa: E402

DEV = "cuda:0"


def torch_normals(verts, faces):
    v0, v1, v2 = (verts[:, faces[:, k]] for k in range(3))
    n = torch.zeros_like(verts)
    n.index_add_(1, faces[:, 1], torch.linalg.cross(v2 - v1, v0 - v1, dim=-1))
    n.index_add_(1, faces[:, 2], torch.linalg.cross(v0 - v2, v1 - v2, dim=-1))
    n.index_add_(1, faces[:, 0], torch.linalg.cross(v1 - v0, v2 - v0, dim=-1))
    return tF.normalize(n, eps=1e-6, dim=-1)


def torch_phong(p2f, bary, verts, normals, colors, faces, params):
    N, H, W = p2f.shape[:3]
    F, V = faces.shape[0], verts.shape[1]
    p = p2f[..., 0]
    hit = p >= 0
    idx = faces[p.clamp_min(0) % F] + (p.clamp_min(0) // F * V)[..., None]      # [N,H,W,3] packed vertex indices
    b = bary[..., 0, :, None]

    def interp(a):
        return (a.reshape(-1, 3)[idx] * b).sum(-2)
    P, Nr, C = interp(verts), tF.normalize(interp(normals), eps=1e-6, dim=-1), interp(colors)
    pr = params[:, None, None, :]
    L = tF.normalize(pr[..., 3:6] - P, eps=1e-6, dim=-1)
    Vd = tF.normalize(pr[..., 0:3] - P, eps=1e-6, dim=-1)
    cos = (Nr * L).sum(-1)
    R = -L + 2 * cos[..., None] * Nr
    spec = torch.pow(torch.relu((Vd * R).sum(-1)) * (cos > 0), pr[..., 24])
    rgb = (pr[..., 15:18] * pr[..., 6:9] + pr[..., 18:21] * pr[..., 9:12] * torch.relu(cos)[..., None]) * C + \
        pr[..., 21:24] * pr[..., 12:15] * spec[..., None]
    rgb = torch.where(hit[..., None], rgb, pr[..., 25:28].expand_as(rgb))
    return torch.cat([rgb, torch.ones_like(rgb[..., :1])], -1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, q = card()
    verts, faces, sk = scene()
    F, V = faces.shape[0], verts.shape[0]
    res = {"gpu": name, "power_limit,clocks.max.sm,clocks.sm": q, "faces": F, "verts": V, "shapes": []}
    for N in (1, 4):
        H = W = 1080
        d, cam = deform(sk, verts, N), cameras(N, H, W)
        cams = (cam[:, 0:2], cam[:, 2:4], cam[:, 4:13].view(-1, 3, 3), cam[:, 13:16])
        colors = torch.rand((N, V, 3), device=DEV)
        fr = raster.rasterize_meshes(d, faces, cams, (H, W))
        params = raster.shade_params(cams, None, None, (1.0, 1.0, 1.0), N, d.device)
        nrm = ops.vertex_normals(d, faces)
        ours = ops.shade_phong(fr, d, nrm, colors, faces, params)
        ref = torch_phong(fr.pix_to_face, fr.bary_coords, d, torch_normals(d, faces), colors, faces, params)
        row = {"N": N, "H": H, "W": W, "covered": int((fr.pix_to_face >= 0).sum()),
               "max_abs_diff_vs_torch_graph": float((ours - ref).abs().max())}
        for key, fn in (("rasterize_ms", lambda: raster.rasterize_meshes(d, faces, cams, (H, W))),
                        ("normals_ms", lambda: ops.vertex_normals(d, faces)),
                        ("phong_ms", lambda: ops.shade_phong(fr, d, nrm, colors, faces, params)),
                        ("shade_meshes_ms", lambda: raster.shade_meshes(d, faces, fr, cams, colors=colors)),
                        ("torch_normals_ms", lambda: torch_normals(d, faces)),
                        ("torch_phong_ms", lambda: torch_phong(fr.pix_to_face, fr.bary_coords, d, nrm, colors, faces,
                                                               params))):
            row[key] = round(timed(fn, a.iters, a.warmup)[0], 4)
        # algorithmic bytes of the Phong pass: 8 B face index + 12 B bary read, 16 B written per pixel, plus per covered
        # pixel 24 B of face indices and 3 x 36 B of vertex gathers (position, normal, colour)
        nbytes = N * H * W * 36 + row["covered"] * (24 + 3 * 36)
        row["phong_GBps"] = round(nbytes / (row["phong_ms"] * 1e-3) / 1e9, 1)
        res["shapes"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"gpu": name, "power_limit,clocks.max.sm,clocks.sm": q, "faces": F, "verts": V}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
