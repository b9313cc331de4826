"""lbs_grad2.npz: the reference's own second-order gradients of the skinning -- model/Deformer.py:359-445 (LBSkinner
forward) under utils/utils.py:133-156 (compute_Jacobian with create_graph=True) -- run on CPU through oracle/refload.py
on the scene of lbs.npz (its inputs are read from there).  refload's GridSamplerMine shim backs the reference's
GridSamplerMine3dFunction with a twice-differentiable sampler.  For each of fp32 and fp64, in the list form
(batch_inds) and the batch form ([3, 1000, 3]), it stores d/d ps, d/d poses and d/d trans of
<J, cot_J> + <D, cot_D> with D = LBSkinner(ps) and J = compute_Jacobian(ps, D, True, True)."""
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
    gen = synth.generator(616)
    cot_D = torch.randn((3000, 3), generator=gen)
    cot_J = torch.randn((3000, 3, 3), generator=gen)
    out = {"cot_D": cot_D.numpy(), "cot_J": cot_J.numpy()}
    for tag, dt in (("f32", torch.float32), ("f64", torch.float64)):
        sk = ns.Deformer.LBSkinner(ws, [-1.1] * 3, [1.1] * 3, Js, parents, init_pose=init,
                                   bbox_extend=torch.tensor(synth.BBOX_EXTEND),
                                   bbox_center=torch.tensor(synth.BBOX_CENTER)).to(dt)
        for form in ("list", "batch"):
            ps = torch.from_numpy(g["ps"]).to(dt).requires_grad_(True)
            poses = torch.from_numpy(g["poses"]).to(dt).requires_grad_(True)
            trans = torch.from_numpy(g["trans"]).to(dt).requires_grad_(True)
            if form == "list":
                D = sk(ps, [poses, trans], torch.from_numpy(g["batch_inds"]))
            else:
                D = sk(ps.view(3, 1000, 3), [poses, trans], None).reshape(-1, 3)
            J = ns.utils_utils.compute_Jacobian(ps, D, True, True)
            loss = (J * cot_J.to(dt)).sum() + (D * cot_D.to(dt)).sum()
            dps, dposes, dtrans = torch.autograd.grad(loss, (ps, poses, trans))
            out[f"{form}_{tag}_dps"] = dps.numpy()
            out[f"{form}_{tag}_dposes"] = dposes.numpy()
            out[f"{form}_{tag}_dtrans"] = dtrans.numpy()
    np.savez_compressed(os.path.join(HERE, "lbs_grad2.npz"), **out)


if __name__ == "__main__":
    main()
