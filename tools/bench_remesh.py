"""Benchmark of the remesh step (OptimGarmentNetwork.marching_cube_update's discretizeSDF and incidence lists, DESIGN
section 1o): the drop-in (recmv_b200.utils.make_discretize_sdf / make_marching_cube_update) against the reference's
method restated on this package's pieces (`reference_remesh` below): the networks' sweeps and marching cubes one after
another (discretize.discretize_all), then per mesh the host copy of vertices and faces, the incidence on the host and
the copy back.  openmesh is not available here, so a vectorised NumPy incidence (a stable argsort of the corners)
stands in for `TriMesh(...).vertex_face_indices()`; the reference's own cost for that step is not measured.

A body and two garment networks (this package's ImplicitNetwork, perturbed geometric inits of three radii) at the
coarse, medium and fine pyramids of train.py.  Per remesh: wall time from the first launch to a final device
synchronise (median of the repetitions, the two flows alternated after a warm-up of each), host synchronisations
(torch's sync debug mode, plus the counter reads of the sweep and marching cubes counted at their helpers),
`recmv_launch_count` launches, and the peak device memory above what was allocated before the call.  The card name,
power limit and SM clocks are read in the same run.

    python tools/bench_remesh.py [--reps 5] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_surface_render_loss import card, count_syncs  # noqa: E402
from recmv_b200 import discretize, ops, testing  # noqa: E402
from recmv_b200 import model as M  # noqa: E402
from recmv_b200 import utils as ru  # noqa: E402
from recmv_b200.MCAcc import Seg3dLossless  # noqa: E402

PYRAMIDS = {   # train.py:47-71
    "coarse": [(15, 21, 9), (29, 41, 17), (57, 81, 33), (113, 161, 65), (225, 321, 129)],
    "medium": [(19, 25, 13), (37, 49, 25), (73, 97, 49), (145, 193, 97), (289, 385, 193)],
    "fine": [(21, 27, 15), (41, 53, 29), (81, 105, 57), (161, 209, 113), (321, 417, 225)],
}
BOX = ([-0.7, -1.0, -0.4], [0.7, 1.0, 0.4])
RATIO = 0.8


class Garment(torch.nn.Module):
    """The attributes the two methods read, on this package's networks."""
    discretizeSDF = ru.make_discretize_sdf()
    marching_cube_update = ru.make_marching_cube_update()

    def __init__(self, nets, engine):
        super().__init__()
        self.sdf, self.garment_nets, self.engine = nets[0], list(nets[1:]), engine
        self.sdfShrinkRadius, self.remesh_time, self.opt_times = 0.01, 0.0, 0.0
        self.inter_free_curve = torch.nn.Linear(4, 4)
        self.visualizer = None

    def update_hierarchical_config(self, device, max_vs, max_fs):
        pass


def numpy_incidence(fs, V):
    """(TmpFid, TmpVid) of faces [F,3] on the host: corners sorted stably by vertex.  A face with an index outside
    [0, V) (marching cubes' -1 where the surface crosses the grid's far boundary) is dropped, as openmesh refuses it."""
    keep = np.nonzero(((fs >= 0) & (fs < V)).all(1))[0]
    corners = fs[keep].reshape(-1)
    order = np.argsort(corners, kind="stable")
    return keep[order // 3], corners[order]


def reference_remesh(m, ratio, device):
    """The reference's discretizeSDF and incidence lists restated on this package's pieces (see the module doc)."""
    vs, fs = discretize.discretize_all(m.sdf, m.garment_nets, m.engine, ratio)
    out = []
    for v, f in zip(vs, fs):
        v.detach().cpu().numpy()                          # the reference builds its TriMesh from both host copies
        fid, vid = numpy_incidence(f.detach().cpu().numpy(), v.shape[0])
        out.append((torch.from_numpy(fid).to(device), torch.from_numpy(vid).to(device)))
    return vs, fs, out


def counted(fn):
    """(result, counter reads at the sweep's and marching cubes' helpers)."""
    n = [0]
    read_levels, read_counters = ops.read_c2f_levels, ops._read_counters

    def levels(*a):
        n[0] += 1
        return read_levels(*a)

    def counters(*a):
        n[0] += 1
        return read_counters(*a)
    ops.read_c2f_levels, ops._read_counters = levels, counters
    try:
        return fn(), n[0]
    finally:
        ops.read_c2f_levels, ops._read_counters = read_levels, read_counters


def measure(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    l0 = ops.launch_count()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    return ms, ops.launch_count() - l0, (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def networks(dev):
    nets = []
    for seed, radius in ((101, 0.6), (202, 0.5), (303, 0.45)):
        nets.append(testing.build_sdf(lambda d, m, b, f: M.getTmpSdf(d, m, radius, f), seed=0, perturb_seed=seed).to(dev))
    return nets


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_remesh: needs a CUDA device")
    dev = torch.device("cuda", 0)
    rows = [dict(card=card(), torch=torch.__version__,
                 note="reference = sequential discretize_all + mc_gpu, host copies and a NumPy incidence in place of "
                      "openmesh (not available); the reference's openmesh time is not measured")]
    print(json.dumps(rows[0]))
    nets = networks(dev)
    root = tempfile.mkdtemp()
    for name, pyramid in PYRAMIDS.items():
        eng = Seg3dLossless(None, b_min=BOX[0], b_max=BOX[1], resolutions=pyramid, align_corners=False,
                            balance_value=0.0).to(dev)
        m = Garment(nets, eng)
        flows = {"drop-in": lambda: m.marching_cube_update([0], RATIO, root, dev),
                 "reference restated": lambda: reference_remesh(m, RATIO, dev)}
        # same meshes and lists from both
        m.marching_cube_update([0], RATIO, root, dev)
        vs, fs, lists = reference_remesh(m, RATIO, dev)
        same = all(torch.equal(x.detach(), y) for x, y in zip([m.body_vs, *m.garment_vs, m.body_fs, *m.garment_fs],
                                                              vs + fs))
        # the drop-in's lists end in (-1, -1) pairs for such faces: compare the valid pairs
        same = same and all(torch.equal(x[x >= 0], y[0]) and torch.equal(z[z >= 0], y[1]) for x, z, y in
                            zip([m.TmpFid, *m.garment_tmpfid], [m.TmpVid, *m.garment_tmpvid], lists))
        times = {k: [] for k in flows}
        stats = {}
        for _ in range(a.reps):
            for k, fn in flows.items():
                ms, launches, peak = measure(fn)
                times[k].append(ms)
                stats[k] = dict(launches=launches, peak_mib=round(peak, 1))
        for k, fn in flows.items():
            _, reads = counted(fn)
            syncs = count_syncs(fn)
            row = dict(pyramid=name, top=pyramid[-1], flow=k, ms_median=round(statistics.median(times[k]), 2),
                       ms_all=[round(t, 2) for t in times[k]], counter_reads=reads, torch_syncs=syncs, **stats[k],
                       verts=[int(v.shape[0]) for v in vs], same_result=same)
            rows.append(row)
            print(json.dumps(row))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
