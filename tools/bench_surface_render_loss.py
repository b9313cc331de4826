"""Benchmark of surface_render_loss's glue on the device (csrc/loss_points.cu, csrc/frame_loss.cu, DESIGN section 1k):
the drop-in (recmv_b200.utils.make_surface_render_loss) against the reference's flow restated in torch
(tests/surface_render_scene.reference_flow: CPU `torch.rand` and boolean indexing for the draws, `torch.randn_like`
for the local samples, boolean indexing by `check` and `valid_mask`, `.item()` for every info value, the host tests
of the singular-Jacobian fallbacks, and torch_scatter's mean restated with `index_add_`).  Both run on the same fused
networks, so only the glue differs.  Two garments at 1080 x 1080 with about 80 k MC vertices each, at
`sample_pix_num` 2048 with a 3-frame batch and 6144 with 1 frame (3072 rays per garment either way), with the
shipped weights of configs/people_snapshot/female-3-casual.conf.

Per call (forward + `loss.backward()`): CUDA-event time after a warm-up (the two flows alternated, twice), host
synchronisations (torch's sync debug mode) and device work items (CUDA kernels and memcpy / memset, counted by
torch.profiler in a separate run); and the sampler and the two frame means (forward + backward) alone.  The card name,
power limit and SM clocks are read in the same run.

    python tools/bench_surface_render_loss.py [--reps 10] [--out FILE]
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

import surface_render_scene as srs  # noqa: E402
from recmv_b200 import ops  # noqa: E402
from recmv_b200.utils import make_surface_render_loss  # noqa: E402

H = W = 1080
VERTS = 80000
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
        raise SystemExit("bench_surface_render_loss: needs a CUDA device")
    dev = torch.device("cuda", 0)
    info = dict(card=card(), torch=torch.__version__)
    print(json.dumps(info))
    nets = srs.networks(dev)
    torch.manual_seed(0)
    rows = []
    for pix, N in SHAPES:
        rays = pix // 2 * N
        self, args, _ = srs.scene(dev, N=N, H=H, W=W, M=(rays, rays), V=(VERTS, VERTS + 1234), seed=pix + N, nets=nets)
        drop_in = make_surface_render_loss()
        params = [p for m in (nets[0], nets[1].defs[0], nets[2]) for p in m.parameters()]

        def run(flow):
            for p in params:
                p.grad = None
            flow(self, *args).backward()

        flows = {"drop_in": lambda: run(drop_in), "reference_flow": lambda: run(srs.reference_flow)}
        for fn in flows.values():
            fn()
        torch.cuda.synchronize()
        row = dict(case=f"sample_pix_num{pix}_N{N}_2garments_1080", rays=[rays, rays], verts=[VERTS, VERTS + 1234])
        for _ in range(2):
            for name, fn in flows.items():
                row.setdefault(f"{name}_ms", []).append(round(events_ms(fn, a.reps), 3))
        for name, fn in flows.items():
            row[f"{name}_host_syncs"] = count_syncs(fn)
            row[f"{name}_kernels"], row[f"{name}_copies"] = count_device_work(fn)
        # the sampler and the two frame means alone
        P, V = [p.float() for p in args[7]], self.garment_vs
        sample = lambda: ops.loss_points_sample(P, V, list(args[5]), list(args[10]), list(args[8]), list(args[9]),  # noqa: E731
                                                list(args[11]), 2048, 1, 0)
        sample()
        row["sampler_ms"] = round(events_ms(sample, a.reps * 5), 4)
        b, r, c = args[10][0], args[8][0], args[9][0]
        M = int(b.shape[0])
        col = torch.rand((M, 3), device=dev, requires_grad=True)
        gtn, nx = torch.randn((M, 3), device=dev, requires_grad=True), torch.randn((M, 3), device=dev, requires_grad=True)
        J = torch.randn((M, 3, 3), device=dev, requires_grad=True)
        w = torch.rand((M,), device=dev)

        def means():
            (ops.ColorFrameMeanFunction.apply(col, args[6], b, r, c, N)
             + ops.NormalFrameMeanFunction.apply(gtn, J, nx, w, b, N)).backward()

        means()
        row["frame_means_fwd_bwd_ms"] = round(events_ms(means, a.reps * 5), 4)
        rows.append(row)
        print(json.dumps(row))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(dict(info, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
