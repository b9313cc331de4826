"""Time the mesh rasterizer (recmv_rasterize_meshes) at the training and inference shapes: the marching-cubes mesh of
synth.sphere_sdf_grid at 257^3 (201 548 faces) deformed by LBSkinner, N = 1..4 frames at 1080 x 1080 (training:
every garment per step), and one frame per call at 1080 x 1080 and 540 x 960 (inference renders frame by frame).

Reports per shape: median call time (CUDA events around the whole call, including its one counter read), the split
setup+count / scan+emit / tile raster from torch.profiler kernel times (a separate pass: tracing slows the host),
(tile, face) pairs per face, and the output write rate of the tile pass (28 B per pixel).  Also times the composite
LBSkinner deform -> rasterize -> fragment decode (utils.FindSurfacePsMesh).  The card, power limit and SM clock come
from the same run.

  python tools/bench_raster.py [--iters 50] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from recmv_b200 import ops, synth  # noqa: E402
from recmv_b200.model import LBSkinner  # noqa: E402
from recmv_b200.utils import FindSurfacePsMesh  # noqa: E402

DEV = "cuda:0"
PHASES = {"raster_setup_kernel": "setup+count", "raster_scan_kernel": "scan+emit", "raster_emit_kernel": "scan+emit",
          "raster_tile_kernel": "tile raster"}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # report, do not guess
        q = f"unknown ({e})"
    return name, q


def scene():
    sdf = synth.sphere_sdf_grid(257, num=8, seed=3, device=DEV)
    h = 2.0 / 256
    verts, faces = ops.mc_gpu(sdf, h, h, h, -1.0, -1.0, -1.0, 0.0)
    Js, parents, init = synth.skeleton()
    sk = LBSkinner(synth.skinning_voxel((129, 225, 65), seed=7), [-1.1] * 3, [1.1] * 3, Js, parents, init_pose=init,
                   bbox_extend=torch.tensor(synth.BBOX_EXTEND), bbox_center=torch.tensor(synth.BBOX_CENTER)).to(DEV)
    return verts, faces, sk


def deform(sk, verts, N):
    poses, trans = synth.poses_trans(N, seed=2)
    V = verts.shape[0]
    with torch.no_grad():
        d = sk(verts.repeat(N, 1), [poses.to(DEV), trans.to(DEV)], torch.arange(N, device=DEV).repeat_interleave(V))
    return d.view(N, V, 3).contiguous()


def cameras(N, H, W):
    R = torch.diag(torch.tensor([-1.0, -1.0, 1.0]))
    rows = [torch.cat([torch.tensor([0.9 * min(H, W)] * 2 + [W / 2 - 0.5, H / 2 - 0.5]), R.reshape(-1),
                       torch.tensor([0.0, 0.0, 2.6])]) for _ in range(N)]
    return torch.stack(rows).to(DEV).contiguous()


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], ts[0], ts[-1]


def phases(fn, reps):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for k, ph in PHASES.items():
            if k in ev.key:
                out[ph] = out.get(ph, 0.0) + ev.device_time_total / 1000.0 / reps   # ms per call
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, q = card()
    verts, faces, sk = scene()
    F = faces.shape[0]
    res = {"gpu": name, "power_limit,clocks.max.sm,clocks.sm": q, "faces": F, "shapes": []}
    shapes = [("train", N, 1080, 1080) for N in (1, 2, 3, 4)] + [("infer", 1, 1080, 1080), ("infer", 1, 540, 960)]
    for kind, N, H, W in shapes:
        d, cam = deform(sk, verts, N), cameras(N, H, W)
        counts = ops.rasterize_meshes(d, faces, cam, H, W)[4]

        def call():
            ops.rasterize_meshes(d, faces, cam, H, W)
        med, lo, hi = timed(call, a.iters, a.warmup)
        ph = phases(call, 10)
        npix = N * H * W
        row = {"kind": kind, "N": N, "H": H, "W": W, "call_ms_median": round(med, 4), "call_ms_min": round(lo, 4),
               "call_ms_max": round(hi, 4), "phase_ms": {k: round(v, 4) for k, v in ph.items()},
               "pairs_per_face": round(counts["pairs"] / max(N * F, 1), 3), "covered": counts["covered"],
               "output_MB": round(28 * npix / 1e6, 2),
               "tile_pass_GBps": round(28 * npix / (ph.get("tile raster", float("nan")) * 1e-3) / 1e9, 1),
               "call_GBps": round(28 * npix / (med * 1e-3) / 1e9, 1)}
        # composite: LBSkinner deform -> rasterize -> fragment decode (+ rays), one camera row per frame
        mask = torch.ones((N, H, W), device=DEV)
        cam_t = (cam[:, 0:2], cam[:, 2:4], cam[:, 4:13].view(-1, 3, 3), cam[:, 13:16])

        def composite():
            FindSurfacePsMesh(verts, faces, deform(sk, verts, N), cam_t, H, W, mask)
        row["composite_ms_median"] = round(timed(composite, max(a.iters // 2, 5), a.warmup)[0], 4)
        res["shapes"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"gpu": name, "power_limit,clocks.max.sm,clocks.sm": q, "faces": F}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
