"""Forward + backward time of LBSkinner's training path -- kernel chain + fused skinning backward (train_fused=True)
against the torch chain + composite (train_fused=False) -- at the training shapes, in one process, alternating the two,
timed with CUDA events.  Reports the card and its power limit from the same run.  `--profile` instead counts the
kernel launches of one step of each path with torch.profiler (a separate run: tracing slows the host).

  python tools/bench_lbs_train.py [--iters 50] [--profile]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from recmv_b200 import synth  # noqa: E402
from recmv_b200.model import CompositeDeformer, LBSkinner, MLPTranslator  # noqa: E402

DEV = "cuda:0"
RATIO = {"deformerRatio": 0.6}


def skinner():
    Js, parents, ip = synth.skeleton()
    ws = synth.skinning_voxel((129, 225, 65), seed=7)     # initialLBSkinner's voxel size
    return LBSkinner(ws, [-1.1] * 3, [1.1] * 3, Js, parents, init_pose=ip,
                     bbox_extend=torch.tensor(synth.BBOX_EXTEND), bbox_center=torch.tensor(synth.BBOX_CENTER)).to(DEV)


def workloads():
    sk = skinner()
    gen = synth.generator(1)
    poses3, trans3 = (t.to(DEV) for t in synth.poses_trans(3, seed=2))
    tmpl = ((torch.rand((1, 120000, 3), generator=gen) - 0.5) * 2.0).to(DEV)
    surf = ((torch.rand((6144, 3), generator=gen) - 0.5) * 2.0).to(DEV)
    bi = torch.randint(0, 3, (6144,), generator=gen).to(DEV)
    poses90, trans90 = (t.to(DEV) for t in synth.poses_trans(90, seed=3))
    torch.manual_seed(0)
    tr = MLPTranslator(128, 6)
    deformer = CompositeDeformer([tr, sk]).to(DEV)
    conds = (torch.randn((3, 128), generator=gen) * 0.1).to(DEV)

    def grads(*ts):
        return [t.clone().requires_grad_(True) for t in ts]

    def garment():
        p, t = grads(poses3, trans3)
        sk(tmpl.expand(3, -1, 3), [p, t], None).sum().backward()

    def surface():
        x, p, t = grads(surf, poses3, trans3)
        sk(x, [p, t], bi).sum().backward()

    def skeleton():
        (p,) = grads(poses90)
        sk.posedSkeleton([p, trans90]).sum().backward()

    def full():
        p, t, c = grads(poses3, trans3, conds)
        deformer(tmpl.expand(3, -1, 3), [c, [p, t]], None, ratio=RATIO, offset_type="garment").sum().backward()

    return sk, tr, {"garment 3x120k expanded": garment, "surface 6144 batch_inds": surface,
                    "posedSkeleton 90 frames": skeleton, "deformer [MLPTranslator, LBSkinner] 3x120k": full}


def set_path(sk, tr, fused):
    sk.train_fused = fused
    tr.train_fused = fused


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # report, do not guess
        pl = f"unknown ({e})"
    return name, pl


def time_all(iters, warmup):
    sk, tr, wl = workloads()
    res = {}
    for name, fn in wl.items():
        for fused in (True, False):
            set_path(sk, tr, fused)
            for _ in range(warmup):
                fn()
        torch.cuda.synchronize()
        times = {True: [], False: []}
        for _ in range(iters):
            for fused in (True, False):          # alternate the two paths
                set_path(sk, tr, fused)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn()
                b.record()
                b.synchronize()
                times[fused].append(a.elapsed_time(b))
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        res[name] = {"fused_ms": round(med[True], 4), "composite_ms": round(med[False], 4),
                     "speedup": round(med[False] / med[True], 2),
                     "fused_min_ms": round(min(times[True]), 4), "composite_min_ms": round(min(times[False]), 4)}
        print(name, res[name], flush=True)
    return res


def profile_all():
    from torch.profiler import ProfilerActivity, profile
    sk, tr, wl = workloads()
    res = {}
    for name, fn in wl.items():
        row = {}
        for fused in (True, False):
            set_path(sk, tr, fused)
            fn()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            row["fused_launches" if fused else "composite_launches"] = len(kernels)
        res[name] = row
        print(name, row, flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lbs_train needs a CUDA device")
    name, pl = card()
    result = {"gpu": name, "power_limit": pl}
    result["launches" if a.profile else "timing"] = profile_all() if a.profile else time_all(a.iters, a.warmup)
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
