"""Times the device construction of the skinning voxel (recmv_lbsw_knn_blend + recmv_lbsw_smooth) against the
reference's torch algorithm (oracle/lbsw_torch.py, 50 000-voxel chunks with torch.topk, as model/Deformer.py:546-591)
on the same GPU, at initialLBSkinner's production size.  Prints one JSON line.

    python tools/bench_lbsw_field.py [--res 129 225 65] [--k 30] [--times 30] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import lbsw_torch as lt  # noqa: E402
from recmv_b200 import ops, synth  # noqa: E402


HBM_BYTES_PER_S = 3.35e12   # H100 SXM5 80 GB (HBM3) peak


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return sorted(ms)[len(ms) // 2], out


def smi(field):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={field}", "--format=csv,noheader,nounits", "-i", "0"],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, nargs=3, default=[129, 225, 65])
    ap.add_argument("--k", type=int, default=30)
    ap.add_argument("--times", type=int, default=30)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    v, w = synth.body_points()
    v, w = v.to(dev), w.to(dev)
    bmin, bmax = v.min(0).values.tolist(), v.max(0).values.tolist()
    W, H, D = a.res
    N, V = W * H * D, v.shape[0]

    knn_ms, cl = timed(lambda: ops.lbsw_knn_blend(v, w, bmin, bmax, a.res, a.k), a.reps)
    smooth_ms, (ws, _) = timed(lambda: ops.lbsw_smooth(cl.clone(), a.times), a.reps)
    copy_ms, _ = timed(lambda: cl.clone(), a.reps)       # the clone that feeds each smoothing run, subtracted
    smooth_ms -= copy_ms
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    ops.lbsw_smooth(ops.lbsw_knn_blend(v, w, bmin, bmax, a.res, a.k), a.times)
    torch.cuda.synchronize()
    dev_peak = torch.cuda.max_memory_allocated(dev) - base

    def torch_path():
        return lt.compute_lbswField(bmin, bmax, a.res, v, w, False, a.k, a.times, stable_ties=False)
    torch_ms, ref = timed(torch_path, max(1, a.reps // 2))
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    torch_path()
    torch.cuda.synchronize()
    torch_peak = torch.cuda.max_memory_allocated(dev) - base

    props = torch.cuda.get_device_properties(dev)
    clock_mhz = smi("clocks.max.sm")
    clock = float(clock_mhz) * 1e6 if clock_mhz else 1.98e9
    fp32_lanes = props.multi_processor_count * 128
    # per distance evaluation: 3 subtractions, 1 multiply, 2 FMAs (the reject compare and selection not counted)
    knn_issue = N * V * 6 / (knn_ms * 1e-3) / (fp32_lanes * clock)
    smooth_bytes = a.times * 2 * 24 * 4 * N
    print(json.dumps({
        "gpu": props.name, "power_limit_w": smi("power.limit"), "max_sm_clock_mhz": clock_mhz,
        "res": a.res, "voxels": N, "verts": V, "k": a.k, "times": a.times,
        "knn_ms": round(knn_ms, 3), "smooth_ms": round(smooth_ms, 3), "device_total_ms": round(knn_ms + smooth_ms, 3),
        "torch_ms": round(torch_ms, 1), "speedup": round(torch_ms / (knn_ms + smooth_ms), 1),
        "device_peak_mb": round(dev_peak / 2 ** 20, 1), "torch_peak_mb": round(torch_peak / 2 ** 20, 1),
        "knn_distance_evals": N * V, "knn_share_of_fp32_issue": round(knn_issue, 3),
        "smooth_bytes": smooth_bytes, "smooth_gb_per_s": round(smooth_bytes / (smooth_ms * 1e-3) / 1e9, 1),
        "smooth_share_of_hbm": round(smooth_bytes / (smooth_ms * 1e-3) / HBM_BYTES_PER_S, 3),
        "max_abs_diff_vs_torch": (ws - ref).abs().max().item(),
    }))


if __name__ == "__main__":
    main()
