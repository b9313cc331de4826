"""Time the point rasterizer + alpha compositor (recmv_rasterize_points, the `pcRender` silhouettes) at the training
shape of mask_loss: the marching-cubes vertices of synth.sphere_sdf_grid at 257^3 split into two groups and deformed by
LBSkinner, N = 1 and 3 frames at 1080 x 1080, r = 0.006, K = 50.

Reports per shape: median forward and forward + backward times (CUDA events around raster.rasterize_points -- the
torch projection, the kernels and the one counter read -- and around that plus .backward() to the deformed points),
the per-kernel split from torch.profiler (a separate pass), the (tile, point) pair count and the peak allocated memory
of the forward + backward.  The card, power limit and SM clock come from the same run.  pytorch3d does not run on
this software stack, so there is no pytorch3d comparison.

  python tools/bench_points_raster.py [--iters 30] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from recmv_b200 import ops, raster, synth  # noqa: E402
from recmv_b200.model import LBSkinner  # noqa: E402

DEV = "cuda:0"
KERNELS = ("points_setup_kernel", "raster_scan_kernel", "points_emit_kernel", "points_tile_kernel<false>",
           "points_tile_kernel<true>", "points_grad_reduce_kernel")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # report, do not guess
        q = f"unknown ({e})"
    return name, q


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


def kernel_ms(fn, reps):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for k in KERNELS:
            if k in ev.key:
                out[k] = out.get(k, 0.0) + ev.device_time_total / 1000.0 / reps   # ms per call
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, q = card()
    sdf = synth.sphere_sdf_grid(257, num=8, seed=3, device=DEV)
    h = 2.0 / 256
    verts, _ = ops.mc_gpu(sdf, h, h, h, -1.0, -1.0, -1.0, 0.0)
    verts = verts.float().contiguous()
    Js, parents, init = synth.skeleton()
    sk = LBSkinner(synth.skinning_voxel((129, 225, 65), seed=7), [-1.1] * 3, [1.1] * 3, Js, parents, init_pose=init,
                   bbox_extend=torch.tensor(synth.BBOX_EXTEND), bbox_center=torch.tensor(synth.BBOX_CENTER)).to(DEV)
    P = verts.shape[0]
    H = W = 1080
    r, K = 0.006, 50
    res = {"gpu": name, "power_limit,clocks.max.sm,clocks.sm": q, "points": P, "H": H, "W": W, "radius": r, "K": K,
           "pytorch3d": "not measured (does not run on this software stack)", "shapes": []}
    for N in (1, 3):
        poses, trans = synth.poses_trans(N, seed=2)
        with torch.no_grad():
            d = sk(verts.repeat(N, 1), [poses.to(DEV), trans.to(DEV)],
                   torch.arange(N, device=DEV).repeat_interleave(P)).view(N, P, 3).contiguous()
        R = torch.diag(torch.tensor([-1.0, -1.0, 1.0]))
        cam = torch.stack([torch.cat([torch.tensor([0.9 * H] * 2 + [W / 2 - 0.5, H / 2 - 0.5]), R.reshape(-1),
                                      torch.tensor([0.0, 0.0, 2.6])]) for _ in range(N)]).to(DEV)
        cam_t = (cam[:, 0:2], cam[:, 2:4], cam[:, 4:13].view(N, 3, 3), cam[:, 13:16])
        pts = d.clone().requires_grad_()
        cot = torch.rand((N, H, W, 1), device=DEV)

        def fwd():
            with torch.no_grad():
                return raster.rasterize_points(d, cam_t, (H, W), r, K, split_size=P // 2)

        def fwd_bwd():
            imgs, _ = raster.rasterize_points(pts, cam_t, (H, W), r, K, split_size=P // 2)
            (imgs[0] * cot + imgs[1] * cot).sum().backward()

        ndc = raster.project_points(d, cam, H, W)
        counts = ops.rasterize_points(ndc, None, H, W, r, K, P // 2)[2]
        f_med, f_lo, f_hi = timed(fwd, a.iters, a.warmup)
        b_med, b_lo, b_hi = timed(fwd_bwd, a.iters, a.warmup)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        fwd_bwd()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        row = {"N": N, "forward_ms_median": round(f_med, 4), "forward_ms_min": round(f_lo, 4),
               "forward_ms_max": round(f_hi, 4), "fwd_bwd_ms_median": round(b_med, 4), "fwd_bwd_ms_min": round(b_lo, 4),
               "fwd_bwd_ms_max": round(b_hi, 4), "pairs": counts["pairs"], "covered": counts["covered"],
               "peak_alloc_MB_fwd_bwd": round(peak / 2 ** 20, 1),
               "kernel_ms_fwd_bwd": {k: round(v, 4) for k, v in kernel_ms(fwd_bwd, 5).items()}}
        res["shapes"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({k: v for k, v in res.items() if k != "shapes"}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
