"""lbsw_ref.npz: the reference's own compute_lbswField -- model/Deformer.py:546-591 and utils/LBSWsmpl.py:13-51 --
run on CPU through oracle/refload.py, on synth.body_points() (stored too, so the tests do not depend on regenerating
them bit for bit).  CASES lists name -> (variant, resolution (W,H,D), align_corners, mean_neighbor, smooth_times)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import refload  # noqa: E402
from recmv_b200 import synth  # noqa: E402

BMIN, BMAX = [-0.85, -0.9, -0.15], [0.85, 0.85, 0.2]
CASES = {
    "model_s30": ("model", (13, 25, 9), False, 30, 30),
    "model_s0": ("model", (13, 25, 9), False, 30, 0),
    "utils_s30": ("utils", (13, 25, 9), False, 30, 30),
    "model_ac": ("model", (7, 11, 5), True, 5, 3),
}


def main():
    ns = refload.load()
    import importlib
    lbsw = importlib.import_module("utils.LBSWsmpl")
    verts, ws = synth.body_points()
    out = {"verts": verts.numpy(), "vert_ws": ws.numpy(), "bmin": np.asarray(BMIN, np.float32),
           "bmax": np.asarray(BMAX, np.float32)}
    for name, (variant, res, ac, k, times) in CASES.items():
        fn = ns.Deformer.compute_lbswField if variant == "model" else lbsw.compute_lbswField
        out[name] = fn(BMIN, BMAX, res, verts, ws, align_corners=ac, mean_neighbor=k, smooth_times=times).numpy()
    np.savez_compressed(os.path.join(HERE, "lbsw_ref.npz"), **out)


if __name__ == "__main__":
    main()
