"""Benchmark of the Laplacian-editing solve (csrc/lap_edit.cu, DESIGN section 1g) against the reference's dense solve.

Scene: an open tube (tests/lap_edit_oracle.tube) with its hem and waist loops constrained to displaced, scaled copies,
at V = 5 000, 20 000 and 55 440.  Per size:
- ours: ops.laplacian_edit (tol 1e-10, no smoothing), CUDA-event time per solve after a warm-up solve, the iterations
  of each column, launches per solve, and the largest error against scipy's sparse direct solve in float64;
- the reference's dense formula inv(L^T W L) L^T W t restated in torch fp32 on the same card, CUDA-event time and its
  error, or "OOM" where it does not fit;
- scipy's sparse direct solve on the CPU, host time, for scale.

    python tools/bench_lap_edit.py [--sizes 100x50,200x100,330x168] [--reps 3] [--no-dense] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import lap_edit_oracle as lo  # noqa: E402
from recmv_b200 import ops  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"nvidia-smi unavailable: {e}"
    return q.splitlines()[0] if q else torch.cuda.get_device_name(0)


def scene(nt, nz):
    v, f, loops = lo.tube(nt, nz)
    cidx, u = lo.loop_targets(v, loops)
    return v.astype(np.float32).astype(np.float64), f, cidx, u.astype(np.float32).astype(np.float64)


def events_ms(fn, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        out = fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps, out


def dense_reference_torch(x, faces, cidx, u, c, dev):
    """The reference's solver (lap_deform_optimizer.py:160-175) in torch fp32 on the GPU."""
    V = x.shape[0]
    L, _ = lo.laplacian(faces, V)
    L = L.tocoo()
    n, m = V, len(cidx)
    Ld = torch.sparse_coo_tensor(np.stack([L.row, L.col]), L.data, (n, n), dtype=torch.float32, device=dev)
    xt = torch.as_tensor(x, dtype=torch.float32, device=dev)
    ut = torch.as_tensor(u, dtype=torch.float32, device=dev)
    ci = torch.as_tensor(cidx, device=dev)
    C = torch.sparse_coo_tensor(torch.stack([torch.arange(m, device=dev), ci]), torch.ones(m, device=dev), (m, n))
    W = torch.diag(torch.cat([torch.ones(n, device=dev), torch.full((m,), float(c), device=dev)]))
    Lf = torch.cat([Ld, C]).to_dense()
    t = torch.cat([Ld @ xt, ut])
    return torch.linalg.inv(Lf.T @ W @ Lf) @ Lf.T @ W @ t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100x50,200x100,330x168")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-dense", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lap_edit: needs a CUDA device")
    dev = torch.device("cuda", 0)
    info = dict(card=card(), torch=torch.__version__)
    print(json.dumps(info))
    rows = []
    for spec in a.sizes.split(","):
        nt, nz = (int(s) for s in spec.split("x"))
        x, f, cidx, u = scene(nt, nz)
        V = len(x)
        row = dict(V=V, M=len(cidx))
        t0 = time.perf_counter()
        ref = lo.solve(x, f, cidx, u, 1.0)
        row["scipy_spsolve_s"] = time.perf_counter() - t0
        xd = torch.as_tensor(x, dtype=torch.float32, device=dev)
        adj = ops.mesh_adjacency(torch.as_tensor(f, device=dev), V)
        ci = torch.as_tensor(cidx, device=dev)
        ut = torch.as_tensor(u, dtype=torch.float32, device=dev)
        ops.laplacian_edit(xd, adj, ci, ut, 1.0, smooth=False)   # warm-up
        torch.cuda.synchronize()
        l0 = ops.launch_count()
        ms, (y, st) = events_ms(lambda: ops.laplacian_edit(xd, adj, ci, ut, 1.0, smooth=False), a.reps)
        st = st.tolist()
        row.update(ours_ms=ms, launches_per_solve=(ops.launch_count() - l0) / a.reps, iterations=st[:3],
                   rel_residual=st[3:6], converged=st[6], ours_max_err=float(np.abs(y.cpu().numpy() - ref).max()),
                   displacement=float(np.abs(ref - x).max()))
        row["ours_us_per_iteration"] = 1e3 * ms / max(st[:3])
        if not a.no_dense:
            try:
                dense_reference_torch(x[:64], [[0, 1, 2]], [0], u[:1], 1.0, dev)   # warm-up of the libraries
                torch.cuda.synchronize()
                dms, yd = events_ms(lambda: dense_reference_torch(x, f, cidx, u, 1.0, dev), 1)
                row.update(dense_fp32_ms=dms, dense_fp32_max_err=float(np.abs(yd.cpu().numpy() - ref).max()))
                del yd
            except torch.OutOfMemoryError:
                row["dense_fp32_ms"] = "OOM"
            torch.cuda.empty_cache()
        rows.append(row)
        print(json.dumps(row))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(dict(info, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
