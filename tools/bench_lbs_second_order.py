"""Time of the train-phase Jacobian block of the skinning -- utils.compute_cardinal_rays(..., 'train'), the normal loss's
utils.compute_Jacobian(ps, ds, True, True) and loss.backward() -- with LBSkinner.second_order_fused on (the point
gradients' VJP kernel) against off (the torch composite under create_graph), alternating the two in one process, timed
with CUDA events.  Shapes: a [MLPTranslator, LBSkinner] deformer and LBSkinner alone, 2048 and 6144 rays over 3 frames
with batch_inds.  Reports the card and its power limit from the same run.  `--profile` instead counts the kernel
launches of one block of each path with torch.profiler (a separate run: tracing slows the host).

  python tools/bench_lbs_second_order.py [--iters 30] [--profile]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from recmv_b200 import synth  # noqa: E402
from recmv_b200.model import CompositeDeformer, LBSkinner, MLPTranslator  # noqa: E402
from recmv_b200.utils import compute_cardinal_rays, compute_Jacobian  # noqa: E402

DEV = "cuda:0"
RATIO = {"deformerRatio": 0.6}


def skinner():
    Js, parents, ip = synth.skeleton()
    ws = synth.skinning_voxel((129, 225, 65), seed=7)     # initialLBSkinner's voxel size
    return LBSkinner(ws, [-1.1] * 3, [1.1] * 3, Js, parents, init_pose=ip,
                     bbox_extend=torch.tensor(synth.BBOX_EXTEND), bbox_center=torch.tensor(synth.BBOX_CENTER)).to(DEV)


def workloads():
    sk = skinner()
    torch.manual_seed(0)
    tr = MLPTranslator(128, 6)
    deformer = CompositeDeformer([tr, sk]).to(DEV)
    gen = synth.generator(1)
    poses, trans = (t.to(DEV) for t in synth.poses_trans(3, seed=2))
    conds = (torch.randn((3, 128), generator=gen) * 0.1).to(DEV)
    wl = {}
    for n in (2048, 6144):                                 # the reference's sample_pix_num values
        x = ((torch.rand((n, 3), generator=gen) - 0.5) * 1.6).to(DEV)
        bi = torch.randint(0, 3, (n,), generator=gen).to(DEV)
        rays = F.normalize(torch.randn((n, 3), generator=gen), dim=1).to(DEV)
        normals = F.normalize(torch.randn((n, 3), generator=gen), dim=1).to(DEV)

        def block(full, x=x, bi=bi, rays=rays, normals=normals):
            ps = x.clone().requires_grad_(True)
            p, t, c = (v.clone().requires_grad_(True) for v in (poses, trans, conds))
            d, defconds = (deformer, [c, [p, t]]) if full else (sk, [p, t])
            crays, ds = compute_cardinal_rays(d, ps, rays, defconds, bi, RATIO, "train", "x")
            J = compute_Jacobian(ps, ds, True, True)       # the normal loss: J^T n
            nx = F.normalize((J.transpose(1, 2) @ normals.unsqueeze(-1)).squeeze(-1), dim=1)
            loss = (crays * rays).sum() + (nx * normals).sum() + (ds * rays).sum()
            loss.backward()
        wl[f"deformer [MLPTranslator, LBSkinner] {n} rays"] = lambda b=block: b(True)
        wl[f"LBSkinner {n} rays"] = lambda b=block: b(False)
    return sk, wl


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # report, do not guess
        pl = f"unknown ({e})"
    return name, pl


def time_all(iters, warmup):
    sk, wl = workloads()
    res = {}
    for name, fn in wl.items():
        for fused in (True, False):
            sk.second_order_fused = fused
            for _ in range(warmup):
                fn()
        torch.cuda.synchronize()
        times = {True: [], False: []}
        for _ in range(iters):
            for fused in (True, False):          # alternate the two paths
                sk.second_order_fused = fused
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
    sk, wl = workloads()
    res = {}
    for name, fn in wl.items():
        row = {}
        for fused in (True, False):
            sk.second_order_fused = fused
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
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lbs_second_order needs a CUDA device")
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
