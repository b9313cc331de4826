"""CPU: host-side behaviour of the second-order skinning entry (recmv_lbs_vjp_backward) -- every rejection happens before
any CUDA call -- and the reference's second-order gradient golden (lbs_grad2.npz) against float64 autograd of the
oracle applied twice."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import oracle_torch as ot
from recmv_b200 import _lib, synth

OK, E_NULL, E_SHAPE = 0, -1, -3
FAKE = 4096


def _vox(ptr=4096, D=4, H=4, W=4):
    v = _lib.Voxel()
    v.ws_cl = ptr
    v.D, v.H, v.W = D, H, W
    v.center = (ctypes.c_float * 3)(0.0, 0.0, 0.0)
    v.extend = 2.0
    return v


def _call(vox="default", nf=3, P=10, ps=FAKE, tps=None, A=FAKE, g=FAKE, u=FAKE, v=None, dg=FAKE, dps=FAKE, dtps=None,
          dA=FAKE, ws=FAKE):
    vox = _vox() if vox == "default" else vox
    return _lib.load().recmv_lbs_vjp_backward(ps, tps, A, None, 0, nf, None if vox is None else ctypes.byref(vox), g, u,
                                              v, dg, dps, dtps, dA, ws, P, None)


def test_lbs_vjp_backward_rejections():
    assert _call(vox=None) == E_NULL
    assert _call(vox=_vox(ptr=0)) == E_NULL
    assert _call(vox=_vox(D=0)) == E_SHAPE
    assert _call(vox=_vox(ptr=4100)) == E_SHAPE            # the voxel is gathered as float4
    assert _call(nf=0) == E_SHAPE
    assert _call(nf=-2) == E_SHAPE
    assert _call(P=-1) == E_SHAPE
    assert _call(ws=None) == E_NULL                        # dA needs the workspace
    assert _call(ws=FAKE + 4) == E_SHAPE                   # 16-byte aligned
    assert _call(ps=None) == E_NULL
    assert _call(A=None) == E_NULL
    for out in ("dps", "dA"):                              # linear in g: g is needed
        kw = {k: None for k in ("dg", "dps", "dA") if k != out}
        assert _call(g=None, **kw) == E_NULL, out
    assert _call(u=None) == E_NULL                         # no cotangent at all
    assert _call(tps=FAKE, u=None, v=None) == E_NULL
    assert _call(v=FAKE) == E_NULL                         # cot_tps without tps
    assert _call(dtps=FAKE) == E_NULL                      # dtps without tps
    assert _call(dtps=FAKE, u=None, v=FAKE) == E_NULL


def test_lbs_vjp_backward_nothing_to_do():
    # nothing requested, or P == 0 without dA: no launch, so fake pointers are never touched
    assert _call(dg=None, dps=None, dA=None, ws=None) == OK
    assert _call(P=0, dA=None, ws=None) == OK
    assert _call(P=0, ps=None, A=None, g=None, u=None, dA=None, ws=None) == OK


def _oracle_second_order(ps, poses, trans, bi, cot_J, cot_D):
    """float64: D by the oracle's bone chain + LBS, J = dD/dps row by row with create_graph, then the gradients of
    <J, cot_J> + <D, cot_D>."""
    Js, parents, _ = synth.skeleton()
    s = load_golden("lbs.npz")
    ws = synth.skinning_voxel((17, 33, 21), seed=7).double()
    center = torch.tensor(synth.BBOX_CENTER).double()
    extend = float(torch.tensor(synth.BBOX_EXTEND))
    A = ot.bone_matrices(poses, Js.double(), parents, torch.from_numpy(s["init_pose"]).double())
    D = ot.lbs_forward(ps, A, trans, ws, center, extend, bi)
    rows = [torch.autograd.grad(D[:, i], ps, torch.ones_like(D[:, 0]), create_graph=True)[0] for i in range(3)]
    J = torch.stack(rows, 1)
    loss = (J * cot_J).sum() + (D * cot_D).sum()
    return torch.autograd.grad(loss, (ps, poses, trans))


def test_golden_precisions_agree_and_match_float64_oracle():
    g = load_golden("lbs_grad2.npz")
    s = load_golden("lbs.npz")
    cot_J = torch.from_numpy(g["cot_J"]).double()
    cot_D = torch.from_numpy(g["cot_D"]).double()
    for form in ("list", "batch"):
        ps = torch.from_numpy(s["ps"]).double().requires_grad_(True)
        poses = torch.from_numpy(s["poses"]).double().requires_grad_(True)
        trans = torch.from_numpy(s["trans"]).double().requires_grad_(True)
        bi = torch.from_numpy(s["batch_inds"]) if form == "list" else torch.arange(3).repeat_interleave(1000)
        ref = _oracle_second_order(ps, poses, trans, bi, cot_J, cot_D)
        for name, r in zip(("dps", "dposes", "dtrans"), ref):
            g64, g32 = g[f"{form}_f64_{name}"], g[f"{form}_f32_{name}"]
            scale = np.abs(g64).max()
            # 1e-6, not 1e-12: the voxel is regenerated in fp32 by torch's CPU kernels, whose last bit may differ
            # between CPUs
            assert np.abs(g64 - r.numpy()).max() / scale < 1e-6, (form, name)
            assert np.abs(g32 - g64).max() / scale < 5e-5, (form, name)
