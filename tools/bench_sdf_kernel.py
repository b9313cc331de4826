"""Times the fused SDF kernel alone at bench.py's frame shape: one render_sdf launch (512 x 512 rays x 64 samples, no
first hit, no x_c) is one sdf_tc_kernel<false, 0, kPasses> launch.  CUDA events around each launch after a warm-up;
prints one JSON line with the card's name and power limit, the per-launch times and their median.

  python tools/bench_sdf_kernel.py [--mode tc3|tc1] [--launches 10] [--warmup 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from recmv_b200 import _lib, ops, synth  # noqa: E402
from recmv_b200.render import SdfRenderer  # noqa: E402

MODES = {"tc3": _lib.MLP_TC_F16X3, "tc1": _lib.MLP_TC_F16X1}
H = W = 512
S = 64


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="tc3", choices=sorted(MODES))
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda", 0)
    ren = SdfRenderer(dev, mode=MODES[args.mode], samples=S)
    poses, trans = synth.poses_trans(1, seed=11, device="cpu")
    A, t = ren.bone_matrices(poses.to(dev), trans.to(dev))
    dirs = synth.pinhole_rays(H, W, device=dev)
    center, extend = ren._bbox()
    out = torch.empty((dirs.shape[0], S), dtype=torch.float32, device=dev)

    def launch():
        ops.render_sdf(dirs, ren.cam_pos, ren.t_near, ren.t_far, S, A, t, ren.ws_cl, center, extend, ren.packed,
                       ren.pe_w, ren.mode, want_xc=False, want_hit=False, out_sdf=out)

    for _ in range(args.warmup):
        launch()
    torch.cuda.synchronize()
    ms = []
    for _ in range(args.launches):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        launch()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    ops.check_async_errors()
    print(json.dumps({"card": card(), "mode": args.mode, "shape": [H * W, S], "launch_ms_median": statistics.median(ms),
                      "launch_ms": [round(m, 3) for m in ms]}))


if __name__ == "__main__":
    main()
