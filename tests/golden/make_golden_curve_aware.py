"""Writes tests/golden/curve_aware_ref.npz: the reference's OWN `OptimGarmentNetwork.curve_aware_loss`
(engineer/networks/OptimGarmentNetwork.py:787-839), unmodified, run on the CPU in float32 with autograd, with
  * a lightweight `self` (conf, fl_names, garment_type, isfine, inter_free_curve, garment_nets, sdfShrinkRadius, info);
  * the reference `ImplicitNetwork` (getTmpSdf, testing.build_sdf seed 0, perturbed with seed 101);
  * `trimesh` rebound to a stub whose `Trimesh(...).sample(n)` is oracle/sample_oracle.py at successive offsets of one
    (seed, offset) stream, so the drop-in reproduces the reference's points by starting at the same place;
  * `Tensor.cuda` a no-op for the run.
Needs the reference source tree (oracle/refload.py).

Three cases: the `upper_bottom` curve alone; `upper_bottom` and the CURVE_AWARE target in the fine phase; and a
CURVE_AWARE target missing from fl_names, which falls through to the last curve.  The stream of one case starts just
below 2^32, so its counters cross into the high word.  Stored per case: the curves, each term's fan vertices and every
50th sample, the per-term losses, the loss, and the SDF parameters' gradients (biases and weight-norm gains whole,
weight_v on a [::32, ::16] grid).

    python tests/golden/make_golden_curve_aware.py
"""
import contextlib
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import refload, sample_oracle  # noqa: E402
from recmv_b200 import testing  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "curve_aware_ref.npz")
SUB = 50                 # every SUB-th sample is stored
P = 200
RATIO = 0.7
SEED = 0x0123456789ABCDEF
CASES = [  # name, fl_names, garment_type, isfine, weight, sdfShrinkRadius, stream offset
    ("one", ["neck", "upper_bottom"], "gap_skirt", True, 60.0, 0.0, 0),
    ("two", ["upper_bottom", "bottom_curve", "left_cuff"], "female_outfit1", True, 30.0, 0.01, (1 << 32) - 60000),
    ("fallthrough", ["neck", "left_cuff", "right_cuff"], "anran_dance", True, 60.0, 0.005, 12345),
]
WV_GRID = (slice(None, None, 32), slice(None, None, 16))


class Conf:
    """The two pyhocon calls the method makes: get_float('a.b') and `'a' in conf`."""

    def __init__(self, d):
        self.d = d

    def get_float(self, key):
        v = self.d
        for k in key.split("."):
            v = v[k]
        return float(v)

    def __contains__(self, key):
        return key in self.d


class Curves:
    def __init__(self, pts):
        self.pts = pts

    def forward(self):
        return self.pts


class TrimeshStub:
    """`trimesh.Trimesh(vertices, faces, process=False).sample(n)` drawn from the pinned stream; records each call."""

    def __init__(self, seed, offset):
        self.seed, self.offset, self.calls = seed, offset, []
        stub = self

        class Trimesh:
            def __init__(self, vertices, faces, process=True):
                self.v = np.asarray(vertices, dtype=np.float32)
                self.f = np.asarray(faces, dtype=np.int64)

            def sample(self, n):
                pts, _ = sample_oracle.sample_mesh(self.v, self.f, n, stub.seed, stub.offset)
                stub.calls.append((self.v.copy(), stub.offset, pts))
                stub.offset += n
                return pts

        self.Trimesh = Trimesh


def curves(seed, C):
    """C closed 200-point loops around the y axis, crossing the SDF's zero level (radius ~0.6), with wiggles."""
    g = np.random.default_rng(seed)
    t = np.linspace(0, 2 * np.pi, P, endpoint=False)
    out = []
    for c in range(C):
        r = 0.55 + 0.08 * np.sin(3 * t + c) + 0.01 * g.standard_normal(P)
        y = -0.2 + 0.15 * c + 0.05 * np.cos(2 * t) + 0.01 * g.standard_normal(P)
        out.append(np.stack([r * np.cos(t) + 0.03 * c, y, r * np.sin(t)], 1))
    return np.stack(out).astype(np.float32)


@contextlib.contextmanager
def cuda_is_identity():
    old = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        yield
    finally:
        torch.Tensor.cuda = old


def build_net(ns):
    return testing.build_sdf(ns.network.getTmpSdf, seed=0, perturb_seed=101)


def run_case(OGN, ns, k, case):
    name, fl_names, garment_type, isfine, weight, shrink, offset = case
    net = build_net(ns)
    cv = curves(100 + k, len(fl_names))
    stub = TrimeshStub(SEED, offset)
    self = types.SimpleNamespace(conf=Conf({"pc_weight": {"curve_aware_weight": weight}}), fl_names=list(fl_names),
                                 garment_type=garment_type, isfine=isfine, inter_free_curve=Curves(torch.tensor(cv)),
                                 garment_nets=[net], sdfShrinkRadius=shrink, info={})
    OGN.trimesh = types.SimpleNamespace(Trimesh=stub.Trimesh)
    with cuda_is_identity():
        loss = OGN.OptimGarmentNetwork.curve_aware_loss(self, {"sdfRatio": RATIO})
    loss.backward()
    out = {"curves": cv, "fl_names": np.array(fl_names), "garment_type": np.array(garment_type),
           "isfine": np.array(isfine), "weight": np.array(weight), "shrink": np.array(shrink),
           "seed": np.array(SEED, dtype=np.uint64), "offset": np.array(offset, dtype=np.uint64),
           "loss": np.array(loss.item(), dtype=np.float32), "terms": np.array(list(self.info.keys())),
           "term_loss": np.array(list(self.info.values()), dtype=np.float32)}
    for t, (v, off, pts) in enumerate(stub.calls):
        out[f"fan_{t}"] = v
        out[f"offset_{t}"] = np.array(off, dtype=np.uint64)
        out[f"samples_{t}"] = pts[::SUB].astype(np.float32)
    for l in range(9):
        lin = getattr(net, f"lin{l}")
        out[f"lin{l}_bias"] = lin.bias.grad.numpy().copy()
        out[f"lin{l}_weight_g"] = lin.weight_g.grad.numpy().copy()
        out[f"lin{l}_weight_v"] = lin.weight_v.grad[WV_GRID].numpy().copy()
    return {f"{name}/{key}": v for key, v in out.items()}


def generate():
    ns = refload.load()
    import importlib
    OGN = importlib.import_module("engineer.networks.OptimGarmentNetwork")
    old = OGN.trimesh
    try:
        out = {}
        for k, case in enumerate(CASES):
            out.update(run_case(OGN, ns, k, case))
    finally:
        OGN.trimesh = old
    return out


def main():
    out = generate()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, {k: float(v) for k, v in out.items() if k.endswith("/loss")})


if __name__ == "__main__":
    main()
