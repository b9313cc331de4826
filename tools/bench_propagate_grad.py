"""Benchmark of propagateTmpPsGrad on the device (csrc/surface_grad.cu's recmv_implicit_grad, DESIGN section 1l): the
drop-in (recmv_b200.utils.make_propagate_tmp_ps_grad) against the reference's method restated on the same networks
(tests/propagate_scene.reference_flow: per garment an SDF forward and autograd pass for grad f, a deformer forward and
three autograd passes for J, the 3x3 algebra in small torch kernels with FastMinv, `check.sum().item()`, and the VJPs
through a second SDF forward, a second deformer forward and a surrogate `loss.backward()`).  Two garments at
1080 x 1080, with the rows sample_train_ray keeps per garment (3072) at `sample_pix_num` 2048 with a 3-frame batch
and 6144 with 1 frame, a learnable camera, and the shipped weights of configs/people_snapshot/female-3-casual.conf.

Per call: CUDA-event time after a warm-up (the two flows alternated, three rounds, each round's mean over --reps
calls), host synchronisations (torch's sync debug mode), this package's launches (recmv_launch_count) and device work
items (CUDA kernels and memcpy / memset, counted by torch.profiler in a separate run).  The card name, power limit
and SM clocks are read in the same run.

    python tools/bench_propagate_grad.py [--reps 10] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import propagate_scene as ps  # noqa: E402
from recmv_b200 import ops  # noqa: E402

H = W = 1080
SHAPES = [(2048, 3), (6144, 1)]     # (sample_pix_num, frames)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"nvidia-smi unavailable: {e}"
    return q.splitlines()[0] if q else torch.cuda.get_device_name(0)


def events_ms(fn, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def count_syncs(fn):
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            fn()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    return sum("synchroniz" in str(x.message) for x in w)


def count_device_work(fn):
    """(kernels, memcpy + memset) one call puts on the device."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    copies = sum(("memcpy" in e.name.lower() or "memset" in e.name.lower()) for e in evs)
    return len(evs) - copies, copies


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_propagate_grad: needs a CUDA device")
    dev = torch.device("cuda", 0)
    info = dict(card=card(), torch=torch.__version__)
    print(json.dumps(info))
    nets = ps.networks(dev)
    rows = []
    for pix, N in SHAPES:
        m = pix // 2 * N
        d = ps.inputs(M=(m, m), N=N, H=H, W=W, seed=pix + N)
        self, leaves = ps.state(dev, d, ps.Garment, nets=nets)
        frame_ids = torch.arange(N, device=dev)
        params = [p for mod in (nets[0], nets[1].defs[0]) for p in mod.parameters()] + list(leaves.values())
        grads = [p.grad for p in self.TmpPs]

        def run(flow):
            for p in params:
                p.grad = None
            for p, g in zip(self.TmpPs, grads):
                p.grad = g
            flow()

        flows = {"drop_in": lambda: run(lambda: self.propagateTmpPsGrad(frame_ids, ps.RATIO)),
                 "reference_flow": lambda: run(lambda: ps.reference_flow(self, frame_ids, ps.RATIO))}
        for fn in flows.values():
            fn()
        torch.cuda.synchronize()
        row = dict(case=f"sample_pix_num{pix}_N{N}_2garments_1080", rows=[m, m])
        for _ in range(3):
            for name, fn in flows.items():
                row.setdefault(f"{name}_ms", []).append(round(events_ms(fn, a.reps), 3))
        for name, fn in flows.items():
            row[f"{name}_host_syncs"] = count_syncs(fn)
            before = ops.launch_count()
            fn()
            row[f"{name}_recmv_launches"] = ops.launch_count() - before
            row[f"{name}_kernels"], row[f"{name}_copies"] = count_device_work(fn)
        rows.append(row)
        print(json.dumps(row))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(dict(info, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
