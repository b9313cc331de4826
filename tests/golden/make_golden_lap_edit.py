"""Writes tests/golden/lap_edit_ref.npz: the reference's OWN `Laplacian_Optimizer.fitting`
(engineer/optimizer/lap_deform_optimizer.py:25-186), unmodified, run on the CPU in float64 and in float32, with its
`save_ply` rebound to capture what it writes.  The garment template is tests/lap_edit_oracle.py's `Template`: the
oracle's COO Laplacian (pytorch3d 0.4's form) and a restatement of the reference's `best_match` (sub-sampled target
curve, linear assignment on squared distances, cosine > 0.5 filter).  Needs the reference source tree
(oracle/refload.py stubs sksparse, ot and pytorch3d).

Scene: an irregular open tube of 288 vertices, wider at the hem (skirt-like), whose waist and hem loops are the two
fields, fitted to a narrower, raised and shifted waist curve and a wider, lowered hem curve over 3 epochs.  Cases:
constrain_weight 1 and 10, each with smooth True and False.  Recorded per case: the vertices at every epoch start
(what best_match sees), every epoch's constraints (indices and fp32 targets) and the final vertices, in float64; the
float32 run's final vertices beside them.

    python tests/golden/make_golden_lap_edit.py
"""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import lap_edit_oracle as lo  # noqa: E402
from oracle import refload  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "lap_edit_ref.npz")
EPOCH = 3
CASES = [dict(c=1.0, smooth=True), dict(c=1.0, smooth=False), dict(c=10.0, smooth=True), dict(c=10.0, smooth=False)]


def curve(n, radius, z, centre):
    th = np.linspace(0, 2 * np.pi, n, endpoint=False) + 0.05
    v = np.stack([centre[0] + radius * np.cos(th), centre[1] + radius * np.sin(th), np.full(n, z)], 1)
    return v.astype(np.float32).astype(np.float64)   # the targets are fp32 values


def scene():
    v, f, fields = lo.tube(24, 12, jitter=0.3, seed=5)
    targets = dict(waist=curve(36, 0.27, 1.58, (0.03, -0.02)), hem=curve(40, 0.54, -0.05, (-0.02, 0.01)))
    return v, f, fields, targets


def run(fit_module, v, f, fields, targets, case, dtype):
    torch.set_default_dtype(dtype)
    written = []
    fit_module.save_ply = lambda path, pts: written.append((os.path.basename(path), pts.detach().cpu().numpy()))
    tmpl = lo.Template(v, f, fields, dtype=dtype)
    opt = fit_module.Laplacian_Optimizer(epoch=EPOCH, constrain_weight=case["c"], smooth=case["smooth"])
    curves = [lo.Curve(torch.tensor(targets[k], dtype=dtype)) for k in ("waist", "hem")]
    opt(source_fl_meshes=[tmpl], target_meshes=curves, source_type=["skirt"], target_fl_type=["waist", "hem"],
        outlayer=True)
    assert tmpl.updates == EPOCH and len(written) == 2 * EPOCH
    for e, (sv, idx, tgt) in enumerate(tmpl.matches):   # what save_ply was given: source points and targets
        assert written[2 * e][0] == "source_0.ply" and written[2 * e + 1][0] == "target_0.ply"
        assert np.array_equal(written[2 * e][1], sv[idx].astype(written[2 * e][1].dtype))
        assert np.array_equal(written[2 * e + 1][1], tgt.astype(np.float32))
    return tmpl


def main():
    refload.load()
    import engineer.optimizer.lap_deform_optimizer as ref   # after refload.load(): a direct import is circular
    v, f, fields, targets = scene()
    out = dict(src_v=v, src_f=f, waist=fields["waist"], hem=fields["hem"], tgt_waist=targets["waist"],
               tgt_hem=targets["hem"], epoch=EPOCH)
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)   # fitting writes ./debug/register/*.ply
        try:
            for k, case in enumerate(CASES):
                t64 = run(ref, v, f, fields, targets, case, torch.float64)
                t32 = run(ref, v, f, fields, targets, case, torch.float32)
                out[f"c_{k}"], out[f"smooth_{k}"] = case["c"], case["smooth"]
                out[f"epoch_v_{k}"] = np.stack([m[0] for m in t64.matches])
                out[f"idx_{k}"] = np.concatenate([m[1] for m in t64.matches])
                out[f"tgt_{k}"] = np.concatenate([m[2] for m in t64.matches])
                out[f"count_{k}"] = np.array([len(m[1]) for m in t64.matches])
                out[f"final_v_{k}"] = t64.vertices.numpy()
                out[f"final_v32_{k}"] = t32.vertices.numpy()
                disp = np.abs(out[f"final_v_{k}"] - v).max()
                err32 = np.abs(out[f"final_v32_{k}"] - out[f"final_v_{k}"]).max()
                print(f"case {k} {case}: constraints per epoch {out[f'count_{k}'].tolist()}, displacement {disp:.4f}, "
                      f"reference fp32 error {err32:.3e} ({err32 / disp:.2e} of the displacement)")
        finally:
            os.chdir(cwd)
            torch.set_default_dtype(torch.float32)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
