"""Benchmark of project_2d_loss's glue on the device (csrc/curve_fit.cu, csrc/curve_project.cu, DESIGN section 1n):
the drop-in (recmv_b200.utils.make_project_2d_loss) against the reference's method restated in torch
(tests/project_2d_scene.reference_flow: one deformer call per curve, `transform_points_screen` with its host test,
the per-curve threshold loop, `regularization()` per garment and `.item()` for every info value).  Both flows run on
the same fused networks with this package's `fl_visible_by_body_zbuff` and `fl_proj_loss`, so only the glue differs.
The training shape: two garments (4 + 2 curves of 200 points) at 1080 x 1080, N = 3 and N = 1.

Per call (forward, backward and the AdamW step): CUDA-event time after a warm-up (the two flows alternated, twice),
host synchronisations (torch's sync debug mode) and device work items (CUDA kernels and memcpy / memset, counted by
torch.profiler in a separate run); and the two new kernels alone (forward + backward).  The card name, power limit and
SM clocks are read in the same run.

    python tools/bench_project_2d_loss.py [--reps 20] [--out FILE]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import project_2d_scene as ps  # noqa: E402
import surface_render_scene as srs  # noqa: E402
from bench_surface_render_loss import card, count_device_work, count_syncs, events_ms  # noqa: E402
from recmv_b200 import ops  # noqa: E402
from recmv_b200.utils import make_project_2d_loss  # noqa: E402

H = W = 1080
S = 200
FRAMES = [3, 1, 3, 1]               # alternated twice in one run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_project_2d_loss: needs a CUDA device")
    dev = torch.device("cuda", 0)
    print(json.dumps(dict(card=card(), torch=torch.__version__)))
    nets = srs.networks(dev)
    rows = []
    drop_in = make_project_2d_loss()
    for N in FRAMES:
        me, args, _ = ps.scene(dev, N=N, H=H, W=W, S=S, nets=nets)
        flows = {"reference": lambda: ps.reference_flow(me, *args), "drop_in": lambda: drop_in(me, *args)}
        for f in flows.values():
            f()
            f()
        row = dict(N=N, H=H, W=W, curves=6, points=S)
        for name, f in flows.items():
            row[f"{name}_ms"] = round(events_ms(f, a.reps), 4)
        for name, f in flows.items():
            row[f"{name}_ms_again"] = round(events_ms(f, a.reps), 4)
        for name, f in flows.items():
            row[f"{name}_syncs"] = count_syncs(f)
            row[f"{name}_kernels"], row[f"{name}_copies"] = count_device_work(f)
        # the two new kernels alone, forward + backward, at this call's shape
        c = me.inter_free_curve
        fit_in = [t.detach().contiguous() for t in (c.cano_verts_center, c.cano_v_dirs, c.init_scale, c.cano_nx,
                                                   c.scale, c.nx_scale)]
        dv = torch.randn(6, S, 3, device=dev)
        dreg = torch.ones(6, 2, device=dev)
        row["curve_fit_us"] = round(1e3 * events_ms(lambda: (ops.curve_fit(*fit_in),
                                                             ops.curve_fit_backward(*fit_in, dv, dreg)), 200), 2)
        sizes = (4, 2)
        table, base = [], 0
        for Cg in sizes:
            table += [(base + k * S, Cg * S, len(table) + k) for k in range(Cg)]
            base += N * Cg * S
        X = torch.randn(base, 3, device=dev) * 0.3
        cams = torch.tensor([[1350., 1350., 540., 540., 1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 3.]] * N, device=dev)
        masks = torch.ones(N, 6, device=dev)
        body = torch.rand(base, device=dev) * 0.2 - 0.05
        thr = [0.1, 0.05, 0.05, 0.08, 0.05, 0.05]

        def project():
            out = ops.curve_project(X, cams, W, H, table, thr, S, masks, body)
            ops.curve_project_backward(X, cams, 6, S, out[2], out[3])

        row["curve_project_us"] = round(1e3 * events_ms(project, 200), 2)
        print(json.dumps(row))
        rows.append(row)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
