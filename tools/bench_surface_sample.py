"""Benchmark of the surface sampler (csrc/surface_sample.cu, DESIGN section 1h) and of the curve-aware term.

- the sampler alone, CUDA-event time per call: the call-site shape (M = 2 fans of P = 200 points, S = 5e4) and a
  2e5-face sheet at S = 1e6;
- the whole term, forward and backward through the fused SDF training path, CUDA-event time per step after a warm-up:
  the drop-in (recmv_b200.utils.make_curve_aware_loss, two curves) against the reference's flow restated: per curve,
  read the points to the host, sample the fan with trimesh's algorithm in NumPy (area_faces, cumsum, searchsorted,
  the folded parallelogram, numpy's global RNG), copy the samples back and run one SDF forward; `.item()` per term.
  Host synchronisations per step are counted with torch's sync debug mode.
The card name, power limit and SM clocks are read in the same run.

    python tools/bench_surface_sample.py [--reps 20] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import types
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from recmv_b200 import ops, testing  # noqa: E402
from recmv_b200.model import getTmpSdf  # noqa: E402
from recmv_b200.utils import make_curve_aware_loss  # noqa: E402

CURVE_AWARE = {'female_outfit1': 'bottom_curve'}
S = 50000


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


def curves(C, P=200, seed=0):
    g = np.random.default_rng(seed)
    t = np.linspace(0, 2 * np.pi, P, endpoint=False)
    out = []
    for c in range(C):
        r = 0.55 + 0.08 * np.sin(3 * t + c) + 0.01 * g.standard_normal(P)
        out.append(np.stack([r * np.cos(t), -0.2 + 0.15 * c + 0.05 * np.cos(2 * t), r * np.sin(t)], 1))
    return np.stack(out).astype(np.float32)


class Conf:
    """pyhocon's two calls with pc_weight.curve_aware_weight = 60."""

    def get_float(self, key):
        return 60.0

    def __contains__(self, key):
        return key == "pc_weight"


def fan_faces(P, dev):
    i = torch.arange(P, device=dev)
    return torch.stack([i, (i + 1) % P, torch.full_like(i, P)], 1)


def sheet(n, dev):
    x, y = np.meshgrid(np.linspace(0, 1, n) ** 1.5, np.linspace(0, 2, n))
    v = np.stack([x, y, 0.1 * np.random.default_rng(8).standard_normal((n, n))], -1).reshape(1, -1, 3)
    i = np.arange(n * n).reshape(n, n)
    a, b, c, d = i[:-1, :-1].ravel(), i[:-1, 1:].ravel(), i[1:, :-1].ravel(), i[1:, 1:].ravel()
    f = np.concatenate([np.stack([a, b, c], 1), np.stack([b, d, c], 1)])
    return torch.tensor(v, dtype=torch.float32, device=dev), torch.tensor(f, dtype=torch.int64, device=dev)


def trimesh_sample(v, f, n):
    """trimesh.sample.sample_surface restated in NumPy (float64, numpy's global RNG)."""
    tri = v[f]
    area = np.sqrt((np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]) ** 2).sum(1)) / 2.0
    cum = np.cumsum(area)
    idx = np.searchsorted(cum, np.random.random(n) * cum[-1])
    origins = tri[idx, 0]
    vec = tri[idx, 1:] - origins[:, None]
    lengths = np.random.random((n, 2, 1))
    flip = lengths.sum(axis=1).reshape(-1) > 1.0
    lengths[flip] -= 1.0
    return (vec * np.abs(lengths)).sum(1) + origins


def reference_flow(self, ratio, weight):
    """OptimGarmentNetwork.curve_aware_loss's per-curve flow (two terms), with the fan sampled on the host."""
    loss = 0.
    for idx, name in ((0, 'upper_bottom'), (1, 'bottom_curve')):
        pts = self.inter_free_curve.forward()[idx]
        fan = torch.cat([pts, pts.mean(0, keepdim=True)], 0)
        P = pts.shape[0]
        f = np.stack([np.arange(P), (np.arange(P) + 1) % P, np.full(P, P)], 1)
        sp = torch.from_numpy(trimesh_sample(fan.detach().cpu().numpy().astype(np.float64), f, S)).float().cuda()
        term = (self.garment_nets[-1](sp, ratio).view(-1) + self.sdfShrinkRadius).abs().mean()
        self.info[f'pc_{name}_circle_loss_sdf'] = term.item()
        loss += term * weight
    return loss


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_surface_sample: needs a CUDA device")
    dev = torch.device("cuda", 0)
    info = dict(card=card(), torch=torch.__version__)
    print(json.dumps(info))
    rows = []

    cv = torch.tensor(curves(2), device=dev)
    fan = torch.cat([cv, cv.mean(1, keepdim=True)], 1).contiguous()
    ff = fan_faces(200, dev)
    sv, sf = sheet(317, dev)
    for name, (v, f, n) in {"callsite_M2_P200_S5e4": (fan, ff, S), "sheet_2e5faces_S1e6": (sv, sf, 1_000_000)}.items():
        ops.surface_sample(v, f, n, 1, 0)
        torch.cuda.synchronize()
        l0 = ops.launch_count()
        ms = events_ms(lambda: ops.surface_sample(v, f, n, 1, 0), 10 * a.reps)
        rows.append(dict(case=name, faces=int(f.shape[0]), samples=int(v.shape[0]) * n, sampler_ms=ms,
                         launches=(ops.launch_count() - l0) / (10 * a.reps)))
        print(json.dumps(rows[-1]))

    net = testing.build_sdf(getTmpSdf, seed=0, perturb_seed=101).to(dev)
    self = types.SimpleNamespace(conf=Conf(), fl_names=['upper_bottom', 'bottom_curve'], garment_type='female_outfit1',
                                 isfine=True, inter_free_curve=types.SimpleNamespace(forward=lambda: cv),
                                 garment_nets=[net], sdfShrinkRadius=0.0, info={})
    ratio = {"sdfRatio": 0.7}
    drop_in = make_curve_aware_loss(CURVE_AWARE)
    np.random.seed(0)
    flows = {"drop_in": lambda: drop_in(self, ratio).backward(),
             "reference_flow": lambda: reference_flow(self, ratio, 60.0).backward()}
    for name, fn in flows.items():
        fn()
        torch.cuda.synchronize()
    row = dict(case="term_fwd_bwd_2_curves_S5e4")
    for _ in range(2):   # alternated, twice
        for name, fn in flows.items():
            net.zero_grad(set_to_none=True)
            row.setdefault(f"{name}_ms", []).append(events_ms(fn, a.reps))
    for name, fn in flows.items():
        row[f"{name}_host_syncs"] = count_syncs(fn)
    rows.append(row)
    print(json.dumps(row))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(dict(info, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
