"""NRICP template registration on the GPU: the fused inner step (csrc/nricp.cu) against the reference's inner loop
restated in torch, on a production-shaped scene, on the same card in the same run.

Scene: a sphere of radius 0.6 meshed by marching cubes on a 257^3 grid is the target (~1.1e5 vertices); its lower
half, scaled by 0.92 and offset, is the open source template (~5e4 vertices, `dense_pcl = 4e4` as in `registration`).

Fused path: median time of one inner iteration (CUDA events over a block of iterations), the launches and host
syncs per iteration, and the wall time of the whole `fl_fit_registry` schedule (200 epochs, 100 + 199 * 50 = 10 050
inner iterations) through `registration.NRICP_Optimizer_AdamW`.
Baseline: the reference's loop (nricp_optimizer.py:365-423) restated in torch from DESIGN section 1f -- Local_Affine
warp, index_select / einsum stiffness, a new COO Laplacian built per iteration as pytorch3d 0.4 builds it (its edge
list by torch.unique), autograd and torch.optim.AdamW(amsgrad=True) -- timed per iteration over two epochs.
Correspondences come from ops.knn_nearest in both.

    python tools/bench_nricp.py [--quick] [--out results/bench_nricp.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from recmv_b200 import ops  # noqa: E402
from recmv_b200.registration import NRICP_Optimizer_AdamW  # noqa: E402

FIT = dict(epoch=200, dense_pcl=4e4, stiffness_weight=[50, 20, 5, 2, 0.8, 0.5, 0.35, 0.2, 0.1], use_normal=True,
           inner_iter=50, mile_stone=[50, 80, 100, 110, 120, 130, 140, 150], laplacian_weight=[250] * 9,
           threshold=0.3)   # fl_fit_registry (OptimGarmentNetwork.py:2415-2419)


def sphere_scene(dev, res=257, radius=0.6, scale=0.92, offset=(0.03, -0.02, 0.06)):
    """(src_v, src_f, tgt_v, tgt_f) on dev: the target sphere and its lower half, scaled and offset, as the source."""
    ax = torch.linspace(-1.0, 1.0, res, device=dev)
    X, Y, Z = torch.meshgrid(ax, ax, ax, indexing="ij")
    sdf = (torch.sqrt(X * X + Y * Y + Z * Z) - radius).contiguous()
    h = 2.0 / (res - 1)
    tgt_v, tgt_f = ops.mc_gpu(sdf, h, h, h, -1.0, -1.0, -1.0, 0.0)
    lower = tgt_f[(tgt_v[tgt_f][:, :, 2] < 0).all(dim=1)]
    used, src_f = torch.unique(lower, return_inverse=True)
    src_v = tgt_v[used] * scale + torch.tensor(offset, device=dev)
    return src_v.contiguous(), src_f.contiguous(), tgt_v.contiguous(), tgt_f.contiguous()


class Mesh:
    """What NRICP_Optimizer_AdamW reads of the template and the target mesh."""

    def __init__(self, v, f):
        self.vertices, self.faces = v, f

    def verts_packed(self):
        return self.vertices

    def faces_packed(self):
        return self.faces

    def get_outlayer_idx(self, *types):
        return []

    def update_padded(self, new_verts):
        self.vertices = new_verts[0]


# ---- the reference's loop, restated in torch --------------------------------------------------------------------

def edges_packed(faces, V):
    """pytorch3d's edges_packed: unique sorted pairs of the face sides (torch.unique synchronises the host)."""
    e = torch.cat([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]).sort(dim=1).values
    u = torch.unique(e[:, 0] * V + e[:, 1])
    return torch.stack([u // V, u % V], dim=1)


def mesh_boundary(faces, V):
    """engineer/utils/mesh_utils.py's rule: a vertex of a side that occurs once among the 3F sides."""
    e = torch.cat([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]).sort(dim=1).values
    u, cnt = torch.unique(e[:, 0] * V + e[:, 1], return_counts=True)
    b = torch.zeros(V, dtype=torch.bool, device=faces.device)
    once = u[cnt == 1]
    b[once // V] = True
    b[once % V] = True
    return b


def laplacian_smoothing(verts, faces):
    """pytorch3d 0.4's uniform mesh_laplacian_smoothing for one new mesh: edges, COO A over both directions, row-sum
    degrees, D^-1 A - I, then mean |L v|."""
    V = verts.shape[0]
    with torch.no_grad():
        e = edges_packed(faces, V)
        e0, e1 = e[:, 0], e[:, 1]
        idx = torch.cat([torch.stack([e0, e1]), torch.stack([e1, e0])], dim=1)
        A = torch.sparse_coo_tensor(idx, torch.ones(idx.shape[1], device=verts.device), (V, V))
        deg = torch.sparse.sum(A, dim=1).to_dense()
        d0, d1 = deg[e0], deg[e1]
        d0 = torch.where(d0 > 0, 1.0 / d0, d0)
        d1 = torch.where(d1 > 0, 1.0 / d1, d1)
        L = torch.sparse_coo_tensor(idx, torch.cat([d0, d1]), (V, V))
        i = torch.arange(V, device=verts.device)
        L = L - torch.sparse_coo_tensor(torch.stack([i, i]), torch.ones(V, device=verts.device), (V, V))
    return torch.sparse.mm(L, verts).norm(dim=1).sum() / V


def torch_fit(src_v, src_f, tgt_v, tgt_f, epoch, inner_iter, stiffness_weight, laplacian_weight, mile_stone,
              gamma=1.0, threshold=0.5, iter_hook=None):
    """The reference's fitting loop in torch on the GPU.  Returns (final vertices, last gate count).  iter_hook(i, it)
    is called before every inner iteration (timing)."""
    dev = src_v.device
    V = src_v.shape[0]
    src_n = ops.vertex_normals(src_v[None], src_f)[0]
    tgt_n = ops.vertex_normals(tgt_v[None], tgt_f)[0]
    inner = ~mesh_boundary(src_f, V)
    edges = edges_packed(src_f, V)
    A = torch.nn.Parameter(torch.eye(3, device=dev).repeat(V, 1, 1))
    b = torch.nn.Parameter(torch.zeros(V, 3, 1, device=dev))
    G = torch.eye(4, device=dev)
    G[3, 3] = gamma

    def forward():
        v = (A @ src_v[:, :, None] + b)[:, :, 0]
        W = torch.cat([A, b], dim=2)
        d = torch.index_select(W, 0, edges[:, 0]) - torch.index_select(W, 0, edges[:, 1])
        return v, torch.einsum("nhw,nwj->nhj", d, G.repeat(d.shape[0], 1, 1)) ** 2

    def normals():
        inv, ok = ops.minv3x3(A.detach().contiguous())
        return (inv.transpose(1, 2) @ src_n[:, :, None])[:, :, 0], ok

    mile_idx, mile_times, w = 0, 0, None
    for i in range(epoch):
        v, stiff = forward()
        with torch.no_grad():
            n2, ok = normals()
        opt = torch.optim.AdamW([A, b], lr=1e-4, amsgrad=True)
        _, idx = ops.knn_nearest(v.detach()[None].contiguous(), tgt_v[None])
        c, m = tgt_v[idx[0]], tgt_n[idx[0]]
        sw, lw = stiffness_weight[mile_idx], laplacian_weight[mile_idx]
        for it in range(100 if i == 0 else inner_iter):
            if iter_hook is not None:
                iter_hook(i, it)
            opt.zero_grad()
            with torch.no_grad():
                w = inner & ok & (F.cosine_similarity(m, n2, dim=1) > threshold)
            data = (w[:, None] * (v - c) ** 2).sum()
            loss = torch.sqrt(data + stiff.sum() * sw) + laplacian_smoothing(v, src_f) * lw
            loss.backward()
            opt.step()
            v, stiff = forward()
            with torch.no_grad():
                n2, ok = normals()
        mile_times += 1
        if mile_times in mile_stone:
            mile_idx += 1
    return v.detach(), w


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim, sm, smax = (s.strip() for s in q.split(","))
        return dict(name=name, power_limit=plim, sm_clock=sm, sm_clock_max=smax)
    except Exception as e:   # the measurement is still valid; say why the conditions are missing
        return dict(name=torch.cuda.get_device_name(), error=str(e))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="time fewer iterations and skip the full schedule")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nricp needs a CUDA device")
    dev = torch.device("cuda", 0)
    src_v, src_f, tgt_v, tgt_f = sphere_scene(dev)
    V, T = src_v.shape[0], tgt_v.shape[0]
    res = dict(source_vertices=V, target_vertices=T, source_faces=int(src_f.shape[0]))

    # fused: one epoch's state, then blocks of inner steps
    src_n = ops.vertex_normals(src_v[None], src_f)[0]
    tgt_n = ops.vertex_normals(tgt_v[None], tgt_f)[0]
    adj = ops.mesh_adjacency(src_f, V)
    X = torch.zeros((V, 3, 4), device=dev)
    X[:, 0, 0] = X[:, 1, 1] = X[:, 2, 2] = 1.0
    mom = tuple(torch.empty_like(X) for _ in range(3))
    stats = torch.zeros(ops.NRICP_STATS, device=dev)
    v = ops.nricp_warp(X, src_v)
    _, idx = ops.knn_nearest(v[None], tgt_v[None])
    idx = idx[0]
    res["boundary_vertices"] = int(adj[3].sum())
    block = 50 if args.quick else 200
    t = 0

    def steps(k):
        nonlocal t
        for _ in range(k):
            t += 1
            ops.nricp_step(src_v, src_n, tgt_v, tgt_n, idx, adj, X, mom, t, 50.0, 250.0, threshold=0.3, stats=stats)

    steps(20)
    torch.cuda.synchronize()
    l0 = ops.launch_count()
    steps(10)
    res["fused_launches_per_iter"] = (ops.launch_count() - l0) / 10
    torch.cuda.set_sync_debug_mode("warn")
    import warnings
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        steps(10)
    torch.cuda.set_sync_debug_mode(0)
    res["fused_host_syncs_per_iter"] = sum("synchroniz" in str(w.message) for w in caught) / 10
    times = []
    for _ in range(7):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        steps(block)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) / block)
    res["fused_iter_ms_median"] = statistics.median(times)
    res["fused_iter_ms_all"] = times
    # host wall per iteration (the enqueue rate bounds a launch-bound loop)
    torch.cuda.synchronize()
    w0 = time.perf_counter()
    steps(block)
    torch.cuda.synchronize()
    res["fused_iter_wall_ms"] = (time.perf_counter() - w0) * 1e3 / block

    if not args.quick:
        opt = NRICP_Optimizer_AdamW(**FIT)
        import contextlib
        import io
        torch.cuda.synchronize()
        w0 = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            opt(smpl_slice=Mesh(src_v.clone(), src_f), cano_meshes=Mesh(tgt_v, tgt_f), save_path=None,
                garment_name="sphere", static_pts_type=[], nricp_masks=torch.ones(T, device=dev))
        torch.cuda.synchronize()
        res["fused_fl_fit_registry_s"] = time.perf_counter() - w0
        res["fl_fit_registry_inner_iterations"] = 100 + (FIT["epoch"] - 1) * FIT["inner_iter"]

    # baseline: torch restatement, per iteration over epochs 0 and 1
    marks = []

    def hook(i, it):
        torch.cuda.synchronize()
        marks.append((i, it, time.perf_counter()))

    n_inner = 10 if args.quick else 50
    torch_fit(src_v, src_f, tgt_v, tgt_f, 1, n_inner, [50.0], [250.0], [], threshold=0.3)   # warm-up
    torch.cuda.synchronize()
    torch_fit(src_v, src_f, tgt_v, tgt_f, 2, n_inner, [50.0], [250.0], [], threshold=0.3, iter_hook=hook)
    torch.cuda.synchronize()
    marks.append((None, None, time.perf_counter()))
    dts = [(marks[k + 1][2] - marks[k][2]) * 1e3 for k in range(len(marks) - 1)
           if marks[k + 1][0] == marks[k][0]]   # consecutive iterations of one epoch
    res["torch_iter_ms_median"] = statistics.median(dts)
    res["torch_iters_timed"] = len(dts)
    torch.cuda.set_sync_debug_mode("warn")
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch_fit(src_v, src_f, tgt_v, tgt_f, 1, 1, [50.0], [250.0], [], threshold=0.3)
    torch.cuda.set_sync_debug_mode(0)
    res["torch_host_syncs_per_iter"] = sum("synchroniz" in str(w.message) for w in caught) / 100   # epoch 0: 100
    res["speedup_per_iter"] = res["torch_iter_ms_median"] / res["fused_iter_ms_median"]
    res["card"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
