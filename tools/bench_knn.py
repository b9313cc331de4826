"""Time the nearest-neighbour kernel (csrc/knn.cu) at the two shapes its callers use, with CUDA events (median of
--iters calls).  The card, power limit and SM clock come from the same run.

 (a) Training shape: utils.fl_proj_loss forward + backward at N = 3 frames, 4 + 2 curves of 200 screen points against
     100 annotation points, ~70 % visible.  The comparison is the reference's per-frame, per-curve loop
     (engineer/core/fl_optimizer.py:72-110) with a brute-force torch chamfer of the same distance formula, its boolean
     indexing and its host reads.  Reported for each: median time, GPU operations (kernels, copies and memsets seen
     by torch.profiler) and host synchronisations (torch's sync debug mode, counted).
 (b) Registration shape: knn_points on 1e5 x 1e5 points at D = 3 (template registration) and D = 2 (the dataset's
     2-D mask distance), forward and forward + backward (to both clouds).  The comparison is a chunked torch brute
     force (distance matrix of 256 query rows at a time, min over candidates; its backward is autograd through the
     gathered neighbour).  Reported: distance evaluations per second and the FP32 share of peak, counting 3D - 1 FP32
     operations per evaluation (D subtractions, D multiplications, D - 1 additions) against the data-sheet 67 TFLOP/s
     of an H100 SXM.  These are separate add and multiply instructions, not FMAs, so the instruction-issue ceiling
     of this operation is half the data-sheet rate.

  python tools/bench_knn.py [--iters 20] [--out FILE.json]
"""
import argparse
import json
import os
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_raster import card, timed  # noqa: E402
from recmv_b200 import ops  # noqa: E402
from recmv_b200.knn import knn_points  # noqa: E402
from recmv_b200.utils import fl_proj_loss  # noqa: E402

DEV = "cuda:0"
FP32_PEAK = 67e12


def torch_chamfer_sum(x, y):
    """pytorch3d's chamfer_distance(x [1,P,2], y [1,M,2], point_reduction="sum") as a brute-force torch graph."""
    d = ((x[0, :, None, :] - y[0, None, :, :]) ** 2).sum(-1)
    cx = d.min(1).values.sum() if x.shape[1] > 0 else x.new_zeros(())
    cy = d.min(0).values.sum() if x.shape[1] > 0 else x.new_zeros(())
    return cx + cy


def reference_loop(fl_pts_list, gt_fl_pts_list, fl_masks, proj_fl_weights):
    """engineer/core/fl_optimizer.py:72-110 with the torch chamfer above."""
    loss = torch.tensor(0.).to(fl_pts_list[0])
    for fl_pts, gt_fl_pts, fl_mask, w in zip(fl_pts_list, gt_fl_pts_list, fl_masks, proj_fl_weights):
        screen_fl_pts, screen_fl_masks = fl_pts[..., :2], fl_mask[..., :2]
        valid_batch = (fl_mask[..., 0].sum(dim=-1) > 0).float().sum()
        batch_loss = 0.
        for pt, m, gt in zip(screen_fl_pts, screen_fl_masks, gt_fl_pts):
            batch_loss += w * torch_chamfer_sum(pt[m == 1].view(1, -1, 2), gt.view(1, -1, 2))
        if valid_batch != 0:
            batch_loss /= valid_batch
        if screen_fl_masks.sum() != 0.:
            loss += batch_loss / (screen_fl_masks.sum() // 2)
        else:
            loss += batch_loss
    return loss / len(fl_pts_list)


def training_inputs(N=3, C=6, P=200, M=100, seed=0):
    g = torch.Generator().manual_seed(seed)
    pts = [(torch.rand(N, P, 3, generator=g) * 512).to(DEV).requires_grad_() for _ in range(C)]
    gts = [(torch.rand(N, M, 2, generator=g) * 512).to(DEV) for _ in range(C)]
    masks = [(torch.rand(N, P, generator=g) < 0.7).to(DEV)[..., None].expand(-1, -1, 3) for _ in range(C)]
    return pts, gts, masks, [1.0, 0.5, 2.0, 1.0, 1.5, 1.0][:C]


def gpu_ops_and_syncs(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    n_ops = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    n_sync = sum(1 for w in caught if "called a synchronizing" in str(w.message))
    return n_ops, n_sync


def bench_training(iters):
    pts, gts, masks, w = training_inputs()

    def ours():
        fl_proj_loss(pts, gts, masks, w).backward()

    def ref():
        reference_loop(pts, gts, masks, w).backward()

    with torch.no_grad():
        a, b = fl_proj_loss(pts, gts, masks, w), reference_loop(pts, gts, masks, w)
    out = {"shape": "N=3, curves 4+2, 200 points vs 100, ~70% visible",
           "loss_ours": a.item(), "loss_torch_loop": b.item()}
    for name, fn in (("ours", ours), ("torch_loop", ref)):
        med, lo, hi = timed(fn, iters, 5)
        before = ops.launch_count()
        fn()
        lib = ops.launch_count() - before
        n_ops, n_sync = gpu_ops_and_syncs(fn)
        out[name] = {"fwd_bwd_ms_median": med, "min": lo, "max": hi, "gpu_ops": n_ops, "host_syncs": n_sync,
                     "library_launches": lib}
    return out


def brute_idx(p1, p2, rows=256):
    idx = torch.empty(p1.shape[:2], dtype=torch.int64, device=p1.device)
    for s in range(0, p1.shape[1], rows):
        d = ((p1[0, s:s + rows, None, :] - p2[0, None, :, :]) ** 2).sum(-1)
        idx[0, s:s + rows] = d.argmin(1)
    return idx


def bench_registration(iters, P=100000):
    out = {}
    for D in (3, 2):
        g = torch.Generator().manual_seed(D)
        p1 = torch.randn(1, P, D, generator=g).to(DEV).requires_grad_()
        p2 = torch.randn(1, P, D, generator=g).to(DEV).requires_grad_()
        evals = P * P

        def fwd():
            with torch.no_grad():
                knn_points(p1, p2)

        def fwd_bwd():
            knn_points(p1, p2).dists.sum().backward()

        def t_fwd():
            with torch.no_grad():
                brute_idx(p1, p2)

        def t_fwd_bwd():
            with torch.no_grad():
                idx = brute_idx(p1, p2)
            nn = torch.gather(p2, 1, idx[..., None].expand(-1, -1, D))
            ((p1 - nn) ** 2).sum(-1).sum().backward()

        with torch.no_grad():
            same = bool(torch.equal(knn_points(p1, p2).idx[..., 0], brute_idx(p1, p2)))
        r = {"P1": P, "P2": P, "idx_equal_to_torch_brute_force": same}
        for name, fn, n in (("fwd", fwd, iters), ("fwd_bwd", fwd_bwd, iters), ("torch_fwd", t_fwd, 3),
                            ("torch_fwd_bwd", t_fwd_bwd, 3)):
            med, lo, hi = timed(fn, n, 2)
            r[name] = {"ms_median": med, "min": lo, "max": hi, "evals_per_s": evals / (med * 1e-3),
                       "fp32_share_of_peak": evals * (3 * D - 1) / (med * 1e-3) / FP32_PEAK}
        out[f"D{D}"] = r
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_knn: no CUDA device (timings are only meaningful on the GPU)")
    name, q = card()
    res = {"card": name, "power.limit,clocks.max.sm,clocks.sm": q,
           "training": bench_training(a.iters), "registration": bench_registration(a.iters)}
    s = json.dumps(res, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
