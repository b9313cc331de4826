"""lbs_grad.npz: the reference LBSkinner's own autograd gradients -- model/Deformer.py:305-326 (posedSkeleton) and
:359-445 (forward) -- run on CPU through oracle/refload.py, on the scene of lbs.npz (its inputs are read from there).
For each of fp32 and fp64 it stores d/d ps, d/d poses and d/d trans of <forward(ps), cot> in the list form (batch_inds)
and the batch form ([3, 1000, 3]), and d/d poses of <posedSkeleton, cot_J>."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import refload  # noqa: E402
from recmv_b200 import synth  # noqa: E402


def main():
    ns = refload.load()
    g = np.load(os.path.join(HERE, "lbs.npz"))
    Js, parents, init = synth.skeleton()
    ws = synth.skinning_voxel((17, 33, 21), seed=7)
    gen = synth.generator(515)
    cot = torch.randn((3000, 3), generator=gen)
    cot_J = torch.randn((3, 24, 3), generator=gen)
    out = {"cot": cot.numpy(), "cot_J": cot_J.numpy()}
    for tag, dt in (("f32", torch.float32), ("f64", torch.float64)):
        sk = ns.Deformer.LBSkinner(ws, [-1.1] * 3, [1.1] * 3, Js, parents, init_pose=init,
                                   bbox_extend=torch.tensor(synth.BBOX_EXTEND),
                                   bbox_center=torch.tensor(synth.BBOX_CENTER)).to(dt)
        for form in ("list", "batch"):
            ps = torch.from_numpy(g["ps"]).to(dt).requires_grad_(True)
            poses = torch.from_numpy(g["poses"]).to(dt).requires_grad_(True)
            trans = torch.from_numpy(g["trans"]).to(dt).requires_grad_(True)
            if form == "list":
                o = sk(ps, [poses, trans], torch.from_numpy(g["batch_inds"]))
            else:
                o = sk(ps.view(3, 1000, 3), [poses, trans], None).reshape(-1, 3)
            dps, dposes, dtrans = torch.autograd.grad(o, (ps, poses, trans), cot.to(dt))
            out[f"{form}_{tag}_dps"] = dps.numpy()
            out[f"{form}_{tag}_dposes"] = dposes.numpy()
            out[f"{form}_{tag}_dtrans"] = dtrans.numpy()
        poses = torch.from_numpy(g["poses"]).to(dt).requires_grad_(True)
        J = sk.posedSkeleton([poses, torch.from_numpy(g["trans"]).to(dt)])
        out[f"skel_{tag}_dposes"] = torch.autograd.grad(J, poses, cot_J.to(dt))[0].numpy()
    np.savez_compressed(os.path.join(HERE, "lbs_grad.npz"), **out)


if __name__ == "__main__":
    main()
