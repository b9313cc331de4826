"""CPU: host-side behaviour of the skinning training entries (recmv_bone_matrices_backward, recmv_lbs_backward and its
workspace query) -- every rejection happens before any CUDA call -- and the reference gradient golden (lbs_grad.npz)
against float64 autograd of the oracle."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import oracle_torch as ot
from recmv_b200 import _lib, synth

OK, E_NULL, E_SHAPE = 0, -1, -3


def _vox(ptr=4096, D=4, H=4, W=4):
    v = _lib.Voxel()
    v.ws_cl = ptr
    v.D, v.H, v.W = D, H, W
    v.center = (ctypes.c_float * 3)(0.0, 0.0, 0.0)
    v.extend = 2.0
    return v


def _expected_bytes(P, F):
    chunks = (P + 255) // 256
    slots = min(F, 256)
    rec = chunks * slots * 292 * 4
    off_n = (rec + chunks * slots * 4 + 15) // 16 * 16
    return off_n + chunks * 4


@pytest.mark.parametrize("P,F", [(0, 1), (1, 1), (255, 3), (256, 3), (257, 3), (360000, 3), (6144, 90), (1000, 1000)])
def test_workspace_bytes(P, F):
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    assert lib.recmv_lbs_backward_workspace_bytes(P, F, ctypes.byref(n)) == OK
    assert n.value == _expected_bytes(P, F)
    # one record of 291 used floats per (chunk, frame present in the chunk), at most 256 frames per chunk
    assert n.value >= ((P + 255) // 256) * min(F, 256) * 291 * 4


def test_workspace_bytes_rejections():
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    assert lib.recmv_lbs_backward_workspace_bytes(-1, 3, ctypes.byref(n)) == E_SHAPE
    assert lib.recmv_lbs_backward_workspace_bytes(10, 0, ctypes.byref(n)) == E_SHAPE
    assert lib.recmv_lbs_backward_workspace_bytes(10, 3, None) == E_NULL


def test_bone_matrices_backward_rejections():
    lib = _lib.load()
    f = lib.recmv_bone_matrices_backward
    assert f(None, None, None, None, None, None, None, None, -1, None) == E_SHAPE
    assert f(None, None, None, None, None, None, None, None, 0, None) == OK        # nothing to do
    fake = 4096
    assert f(None, fake, fake, None, fake, None, fake, fake, 2, None) == E_NULL    # poses
    assert f(fake, None, fake, None, fake, None, fake, fake, 2, None) == E_NULL    # Js
    assert f(fake, fake, None, None, fake, None, fake, fake, 2, None) == E_NULL    # parents
    assert f(fake, fake, fake, None, None, None, fake, fake, 2, None) == E_NULL    # G
    assert f(fake, fake, fake, None, fake, None, fake, None, 2, None) == E_NULL    # dposes


def test_lbs_backward_rejections():
    lib = _lib.load()
    f = lib.recmv_lbs_backward
    fake = 4096
    v = _vox()

    def call(vox=v, nf=3, P=10, ps=fake, A=fake, g=fake, dps=fake, dA=fake, ws=fake, bi=None):
        return f(ps, None, A, None, bi, 0, nf, vox if vox is None else ctypes.byref(vox), g, dps, None, dA, None, ws, P,
                 None)

    assert call(vox=None) == E_NULL
    assert call(vox=_vox(ptr=0)) == E_NULL
    assert call(vox=_vox(D=0)) == E_SHAPE
    assert call(vox=_vox(ptr=4100)) == E_SHAPE          # the voxel is gathered as float4
    assert call(nf=0) == E_SHAPE
    assert call(P=-1) == E_SHAPE
    assert call(ps=None) == E_NULL
    assert call(A=None) == E_NULL
    assert call(g=None) == E_NULL
    assert call(ws=None) == E_NULL                      # dA needs the workspace
    assert call(ws=fake + 4) == E_SHAPE                 # 16-byte aligned
    assert call(P=0, dps=None, dA=None, ws=None) == OK  # nothing requested, no launch


def test_golden_precisions_agree_and_match_float64_oracle():
    """The reference's own fp32 and fp64 gradients agree with each other, and the fp64 ones with float64 autograd of the
    oracle's restatement (bone chain + LBS with the border-clamped sampler)."""
    g = load_golden("lbs_grad.npz")
    s = load_golden("lbs.npz")
    Js, parents, init = synth.skeleton()
    ws = synth.skinning_voxel((17, 33, 21), seed=7).double()
    # the reference keeps the box in fp32 buffers, so its fp64 run sees their fp32 values
    center = torch.tensor(synth.BBOX_CENTER).double()
    extend = float(torch.tensor(synth.BBOX_EXTEND))
    ip = torch.from_numpy(s["init_pose"]).double()
    bi_list = torch.from_numpy(s["batch_inds"])
    for form in ("list", "batch"):
        ps = torch.from_numpy(s["ps"]).double().requires_grad_(True)
        poses = torch.from_numpy(s["poses"]).double().requires_grad_(True)
        trans = torch.from_numpy(s["trans"]).double().requires_grad_(True)
        bi = bi_list if form == "list" else torch.arange(3).repeat_interleave(1000)
        A = ot.bone_matrices(poses, Js.double(), parents, ip)
        out = ot.lbs_forward(ps, A, trans, ws, center, extend, bi)
        ref = torch.autograd.grad(out, (ps, poses, trans), torch.from_numpy(g["cot"]).double())
        for name, r in zip(("dps", "dposes", "dtrans"), ref):
            g64, g32 = g[f"{form}_f64_{name}"], g[f"{form}_f32_{name}"]
            scale = np.abs(g64).max()
            # 1e-6, not 1e-12: the voxel is regenerated in fp32 by torch's CPU kernels, whose last bit differs between
            # CPUs (measured 8.6e-8 on a machine other than the golden's)
            assert np.abs(g64 - r.numpy()).max() / scale < 1e-6, (form, name)
            assert np.abs(g32 - g64).max() / scale < 1e-5, (form, name)
    poses = torch.from_numpy(s["poses"]).double().requires_grad_(True)
    G = ot.bone_matrices(poses, Js.double(), parents, torch.eye(4, dtype=torch.float64).expand(24, 4, 4))
    r = torch.autograd.grad(G[:, :, :3, 3], poses, torch.from_numpy(g["cot_J"]).double())[0].numpy()
    assert np.abs(g["skel_f64_dposes"] - r).max() / np.abs(r).max() < 1e-12
    assert np.abs(g["skel_f32_dposes"] - r).max() / np.abs(r).max() < 1e-5
