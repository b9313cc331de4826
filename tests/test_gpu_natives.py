"""GPU parity tests of the native ops, called through the C ABI (recmv_b200.ops -> ctypes -> .so),
against the oracle and the committed golden vectors.  Bit-exact for indices; floats within the
stated tolerances."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import mc_oracle
from oracle import oracle_torch as ot
from recmv_b200 import _lib, ops, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


# ------------------------------------------------------------------ FastMinv (A6)
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-5), (torch.float64, 1e-12)])
@pytest.mark.parametrize("n", [1, 255, 10000, 262144])
def test_minv3x3_forward_backward(dtype, tol, n):
    g = synth.generator(n)
    ms = torch.randn((n, 3, 3), generator=g, dtype=dtype)
    ms[::7] *= 0.03  # a good share of near-singular matrices: exercises the 1e-4 determinant gate
    inv, ok = ops.minv3x3(ms.to(DEV))
    ref_inv, ref_ok = ot.minv3x3_fwd(ms)
    # the gate compares a rounded determinant: allow disagreement only within rounding of the threshold
    m = ms.double()
    det = torch.linalg.det(m)
    clear = (det.abs() - 1e-4).abs() > 1e-6 * (1 if dtype == torch.float32 else 1e-6)
    assert bool((ok.cpu() == ref_ok)[clear].all())
    both = ok.cpu() & ref_ok
    if both.any():
        scale = ref_inv[both].abs().amax(dim=(1, 2), keepdim=True).clamp_min(1e-6)
        assert float(((inv.cpu()[both] - ref_inv[both]).abs() / scale).max()) < tol * 50
    assert bool((inv.cpu()[~ok.cpu()] == 0).all())
    gr = torch.randn((n, 3, 3), generator=g, dtype=dtype)
    out = ops.minv3x3_backward(gr.to(DEV), inv)
    ref = ot.minv3x3_bwd(gr, inv.cpu())
    s = ref.abs().amax(dim=(1, 2), keepdim=True).clamp_min(1e-6)
    assert float(((out.cpu() - ref).abs() / s).amax()) < tol * 50


def test_minv3x3_reference_check_script_property():
    # FastMinv/check.py: inv @ m == I on randn(10000,3,3)
    ms = torch.randn((10000, 3, 3), generator=synth.generator(0)).to(DEV)
    inv, ok = ops.minv3x3(ms)
    err = (inv[ok] @ ms[ok] - torch.eye(3, device=DEV)).norm(dim=(1, 2))
    assert ok.sum() > 9900 and err.mean() < 1e-4
    assert ops.minv3x3(torch.empty((0, 3, 3), device=DEV))[0].shape == (0, 3, 3)
    f = ops.FastDiff3x3MinvFunction.apply
    m = (torch.randn(64, 3, 3, dtype=torch.double, device=DEV) + 2 * torch.eye(3, dtype=torch.double, device=DEV)).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda a: f(a)[0], (m,), eps=1e-6, atol=1e-6)
    with pytest.raises(RuntimeError):
        ops.minv3x3(torch.randn(4, 3, 3, device=DEV).transpose(1, 2))  # not contiguous


# ------------------------------------------------------------------ GridSamplerMine (K4-K6)
def test_gridsample_golden_double_all_orders():
    g = load_golden("gridsample.npz")
    t = {k: torch.from_numpy(v).to(DEV) for k, v in g.items()}
    out = ops.grid_sample3d_forward(t["input"], t["grid"])
    assert (out - t["out"]).abs().max() < 1e-12
    gi, gg = ops.grid_sample3d_backward(t["input"], t["grid"], t["grad_out"])
    assert (gi - t["grad_input"]).abs().max() < 1e-11 and (gg - t["grad_grid"]).abs().max() < 1e-10
    d0, d1, d2 = ops.grid_sample3d_dbackward(t["gg_input"], t["gg_grid"], t["input"], t["grid"], t["grad_out"])
    assert (d0 - t["d_input"]).abs().max() < 1e-10
    assert (d1 - t["d_grid"]).abs().max() < 1e-9
    assert (d2 - t["d_gout"]).abs().max() < 1e-10
    # channels-last layout gives the same numbers
    icl = t["input"].permute(0, 2, 3, 4, 1).contiguous()
    assert (ops.grid_sample3d_forward(icl, t["grid"], _lib.LAYOUT_NDHWC) - t["out"]).abs().max() < 1e-12


def test_gridsample_reference_check_script():
    # MCAcc/check_grid_sampler_mine.py: equality with F.grid_sample and gradcheck of fn and of its backward
    gen = synth.generator(3)
    inp = torch.randn((1, 5, 15, 15, 15), generator=gen, dtype=torch.double).to(DEV).requires_grad_(True)
    grid = ((torch.rand((1, 1, 1, 10, 3), generator=gen, dtype=torch.double) - 0.5) * 2.2).to(DEV).requires_grad_(True)
    fn = ops.GridSamplerMine3dFunction.apply
    ref = torch.nn.functional.grid_sample(inp, grid, mode="bilinear", padding_mode="border", align_corners=False)
    assert (fn(inp, grid) - ref).abs().max() < 1e-12
    assert torch.autograd.gradcheck(fn, (inp, grid), eps=1e-6, atol=1e-5)
    go = torch.randn((1, 5, 1, 1, 10), generator=gen, dtype=torch.double).to(DEV).requires_grad_(True)
    assert torch.autograd.gradcheck(ops.GridSamplerMine3dBackwardFunction.apply, (inp, grid, go), eps=1e-6, atol=1e-5)


def test_gridsample_float_large_and_frozen_voxel():
    ws = synth.skinning_voxel((17, 33, 21), seed=7)
    gen = synth.generator(8)
    grid = ((torch.rand((1, 1, 1, 50000, 3), generator=gen) - 0.5) * 2.4)
    ref = torch.nn.functional.grid_sample(ws, grid, mode="bilinear", padding_mode="border", align_corners=False)
    out = ops.grid_sample3d_forward(ws.to(DEV), grid.to(DEV))
    assert (out.cpu() - ref).abs().max() < 2e-6
    # frozen voxel: grad_input skipped, grad_grid identical to the full backward
    go = torch.randn(ref.shape, generator=gen)
    gi, gg = ops.grid_sample3d_backward(ws.to(DEV), grid.to(DEV), go.to(DEV))
    none, gg2 = ops.grid_sample3d_backward(ws.to(DEV), grid.to(DEV), go.to(DEV), need_grad_input=False)
    assert none is None and torch.equal(gg, gg2)
    rgi, rgg = ot.grid_sample3d_bwd(ws, grid, go)
    assert (gg.cpu() - rgg).abs().max() < 1e-4 * rgg.abs().max()
    assert (gi.cpu() - rgi).abs().max() < 1e-4 * rgi.abs().max()
    assert ops.grid_sample3d_forward(ws.to(DEV), torch.empty((1, 1, 1, 0, 3), device=DEV)).shape[-1] == 0


# ------------------------------------------------------------------ MCGpu (A12)
@pytest.mark.parametrize("shape", [41, (21, 37, 13), (33, 17, 50)])
def test_marching_cubes_bit_exact_against_oracle(shape):
    sdf = synth.sphere_sdf_grid(shape, num=4, seed=3)
    n = sdf.shape
    step = (2.0 / (n[0] - 1), 2.0 / (n[1] - 1), 2.0 / (n[2] - 1))
    v, f = ops.mc_gpu(sdf.to(DEV), *step, -1.0, -1.0, -1.0, 0.0)
    rv, rf = mc_oracle.marching_cubes(sdf.numpy(), step, (-1, -1, -1), 0.0)
    assert f.dtype == torch.int64 and v.dtype == torch.float32
    assert v.shape[0] == len(rv) and f.shape[0] == len(rf)
    assert np.array_equal(f.cpu().numpy(), rf)  # triangle indices: bit exact, same order
    assert np.abs(v.cpu().numpy() - rv).max() < 1e-6
    # order-independent form as well (what one would compare against the atomics-ordered reference)
    cv, cf = mc_oracle.canonical(v.cpu().numpy(), f.cpu().numpy())
    ov, of = mc_oracle.canonical(rv, rf)
    assert np.array_equal(cf, of) and np.abs(cv - ov).max() < 1e-6


def _assert_mc_matches_oracle(v, f, sdf, step=(1.0, 1.0, 1.0), origin=(0.0, 0.0, 0.0)):
    rv, rf = mc_oracle.marching_cubes(sdf.cpu().numpy(), step, origin, 0.0)
    assert v.shape[0] == len(rv) and np.array_equal(f.cpu().numpy(), rf)
    assert np.abs(v.cpu().numpy() - rv).max() < 1e-6


def test_marching_cubes_buffer_growth():
    """The one-call path grows its capacity buffers when the first guess is too small, is reproducible afterwards, and
    equals the oracle before and after the growth."""
    ops._scratch_cache.clear()
    big = synth.sphere_sdf_grid(97, num=6, seed=4, device=DEV)        # > 4096 vertices: forces one regrowth
    v1, f1 = ops.mc_gpu(big, 2 / 96, 2 / 96, 2 / 96, -1.0, -1.0, -1.0)
    assert v1.shape[0] > 4096
    v3, f3 = ops.mc_gpu(big, 2 / 96, 2 / 96, 2 / 96, -1.0, -1.0, -1.0)
    assert torch.equal(v1, v3) and torch.equal(f1, f3)
    _assert_mc_matches_oracle(v1, f1, big, (2 / 96,) * 3, (-1.0,) * 3)
    small = synth.sphere_sdf_grid(21, num=2, seed=4, device=DEV)      # smaller than the grown buffers: sliced, not stale
    v4, f4 = ops.mc_gpu(small)
    _assert_mc_matches_oracle(v4, f4, small)
    assert int(f4.max()) == v4.shape[0] - 1


def test_marching_cubes_edge_cases_and_boundary_minus_one():
    assert ops.mc_gpu(torch.ones((5, 6, 7), device=DEV))[0].shape == (0, 3)
    assert ops.mc_gpu(-torch.ones((5, 6, 7), device=DEV))[1].shape == (0, 3)
    assert ops.mc_gpu(torch.ones((5, 6, 7), device=DEV, dtype=torch.float64)) == []  # MCGpu.cpp:41-42
    # a surface that crosses the far boundary planes: -1 indices exactly where the reference emits them
    g = torch.linspace(-1, 1, 17)
    X, Y, Z = torch.meshgrid(g, g, g, indexing="ij")
    sdf = (torch.sqrt((X - 0.9) ** 2 + Y ** 2 + Z ** 2) - 0.5).contiguous()
    v, f = ops.mc_gpu(sdf.to(DEV))
    rv, rf = mc_oracle.marching_cubes(sdf.numpy())
    assert (rf < 0).any() and np.array_equal(f.cpu().numpy(), rf) and np.abs(v.cpu().numpy() - rv).max() < 1e-6
    # non-zero iso value
    v, f = ops.mc_gpu(sdf.to(DEV), fTargetValue=0.1)
    rv, rf = mc_oracle.marching_cubes(sdf.numpy(), iso=0.1)
    assert np.array_equal(f.cpu().numpy(), rf)


def test_marching_cubes_full_size_properties():
    # BASELINE config 3 size (257^3): watertight, deterministic, V - E + F = 2 per component
    sdf = synth.sphere_sdf_grid(257, num=8, seed=3, device=DEV)
    v, f = ops.mc_gpu(sdf, 2 / 256, 2 / 256, 2 / 256, -1.0, -1.0, -1.0)
    v2, f2 = ops.mc_gpu(sdf, 2 / 256, 2 / 256, 2 / 256, -1.0, -1.0, -1.0)
    assert torch.equal(v, v2) and torch.equal(f, f2)
    assert f.min() >= 0 and f.max() == v.shape[0] - 1
    e = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]).sort(dim=1).values
    _, cnt = torch.unique(e, dim=0, return_counts=True)
    assert bool((cnt == 2).all())
    # every vertex lies on its sphere union surface to within half a cell
    assert v.shape[0] > 50000


# ------------------------------------------------------------------ LBS (A5 / A5')
def _skinner():
    from recmv_b200.model import LBSkinner
    Js, parents, init = synth.skeleton()
    ws = synth.skinning_voxel((17, 33, 21), seed=7)
    return LBSkinner(ws, [-1.1] * 3, [1.1] * 3, Js, parents, init_pose=init,
                     bbox_extend=torch.tensor(synth.BBOX_EXTEND), bbox_center=torch.tensor(synth.BBOX_CENTER)).to(DEV)


def test_lbskinner_forward_matches_reference_golden():
    g = load_golden("lbs.npz")
    sk = _skinner()
    assert (sk.init_pose.cpu() - torch.from_numpy(g["init_pose"])).abs().max() < 1e-6
    poses, trans = torch.from_numpy(g["poses"]).to(DEV), torch.from_numpy(g["trans"]).to(DEV)
    ps, bi = torch.from_numpy(g["ps"]).to(DEV), torch.from_numpy(g["batch_inds"]).to(DEV)
    with torch.no_grad():
        o1 = sk(ps, [poses, trans], bi)
        assert sk.last_path == "fused"
        o2 = sk(ps.view(3, 1000, 3), [poses, trans], None)
    assert rel_err(o1, g["out_list"], 1e-2) < 1e-4
    assert rel_err(o2, g["out_batch"], 1e-2) < 1e-4
    # autograd path (CUDA sampler + batched blend) agrees and is differentiable twice
    psg = ps.clone().requires_grad_(True)
    o3 = sk(psg, [poses, trans], bi)
    assert sk.last_path == "autograd-composite" and rel_err(o3, g["out_list"], 1e-2) < 1e-4
    (gr,) = torch.autograd.grad(o3.sum(), psg, create_graph=True)
    gr.pow(2).sum().backward()
    assert torch.isfinite(psg.grad).all()


def test_inverse_warp_matches_oracle_composition():
    g = load_golden("lbs.npz")
    sk = _skinner()
    poses, trans = torch.from_numpy(g["poses"]).to(DEV), torch.from_numpy(g["trans"]).to(DEV)
    xo, bi = torch.from_numpy(g["out_list"]).to(DEV), torch.from_numpy(g["batch_inds"]).to(DEV)
    xc, ok = sk.inverse(xo, [poses, trans], bi)
    assert bool((ok.cpu().numpy() == g["inv_ok"]).all())
    assert rel_err(xc, g["inv_xc"], 1e-2) < 1e-4
