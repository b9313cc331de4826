"""In parity mode (tc3) the plain SDF forward (`sdf_tc_kernel<false, 0, 3>`) computes the sdf column in layer 7's
epilogue, as an fp32 sum of layer 7's outputs times layer 8's packed weights, and runs layer 8 only for the features;
tc1 keeps the sdf on the last layer's first tensor-core tile.  Checked in both modes at sizes where every CTA runs
several tiles and the last tile is partial:
  * the sdf of sdf_mlp_forward and of render_sdf against float64 (the render at the kernel's own x_c), and the render's
    first hit against the sign change of its own sdf;
  * the sdf is bit-identical with and without the feature output;
  * the diagnostics dump of layer 8 still returns its raw accumulator."""
import ctypes

import pytest
import torch

from conftest import norm_err, rel_err
from oracle import oracle_torch as ot
from recmv_b200 import _lib, ops, synth, testing
from recmv_b200.model import getTmpSdf
from recmv_b200.render import SdfRenderer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# mode, passes, bound on max |a-b| / rms(f64), bound on the element-wise |a-b| / max(|f64|, 1e-2)
MODES = [("tc3", _lib.MLP_TC_F16X3, 3, 3e-5, 1.2e-4), ("tc1", _lib.MLP_TC_F16X1, 1, 5e-3, 5e-2)]
IDS = [m[0] for m in MODES]

_cache = {}


@pytest.fixture(autouse=True)
def _no_aborted_launch():
    yield
    torch.cuda.synchronize()
    ops.check_async_errors()


def _net():
    if not _cache:
        net = testing.build_sdf(getTmpSdf, seed=0, perturb_seed=101).to(DEV)
        Ws, bs = net.effective_weights()
        _cache["net"] = net
        _cache["w64"] = ([w.detach().to(DEV, torch.float64) for w in Ws], [b.detach().to(DEV, torch.float64) for b in bs])
    return _cache["net"]


def _truth(x):
    """float64 (sdf [P], feat [P, 256]) of the same effective weights, evaluated on the device."""
    _net()
    sdf, feat = ot.sdf_mlp(x.to(DEV, torch.float64), *_cache["w64"], ot.annealing_weights(6, None))
    return sdf.view(-1), feat


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _points(P, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand((P, 3), generator=g) * 1.6 - 0.8).to(DEV)


@pytest.mark.parametrize("name,mode,passes,ntol,tol", MODES, ids=IDS)
def test_points_sdf_against_float64(name, mode, passes, ntol, tol):
    net = _net()
    P = 3 * _sms() * 64 + 37
    x = _points(P, seed=5)
    sdf, feat = ops.sdf_mlp_forward(x, net.packed_weights(), None, mode, want_feat=False)
    assert feat is None
    truth, _ = _truth(x)
    e_norm, e_el = norm_err(sdf.view(-1), truth), rel_err(sdf.view(-1), truth, 1e-2)
    print(f"{name} points P={P}: |ours-f64| norm {e_norm:.2e} element-wise {e_el:.2e}")
    assert e_norm < ntol and e_el < tol


@pytest.mark.parametrize("name,mode,passes,ntol,tol", MODES, ids=IDS)
def test_render_sdf_against_float64_and_first_hit(name, mode, passes, ntol, tol):
    net = _net()
    ren = SdfRenderer(DEV, sdf_net=net, voxel_shape=(17, 33, 21), mode=mode, samples=64)
    poses, trans = synth.poses_trans(1, seed=11)
    A, t = ren.bone_matrices(poses.to(DEV), trans.to(DEV))
    # 64 samples per ray = one tile per ray: 8 SMs' worth of tiles minus 27, so the last wave is partial; the rays are
    # the middle of a 48 x 48 image, where the body is
    R = 8 * _sms() - 27
    d = synth.pinhole_rays(48, 48, device=DEV)
    dirs = d[(d.shape[0] - R) // 2:(d.shape[0] - R) // 2 + R].contiguous()
    assert dirs.shape[0] == R
    sdf, xc, hit_idx, _ = ren.render(dirs, A, t, want_xc=True)
    valid = sdf != 1e10
    assert valid.float().mean() > 0.9
    truth, _ = _truth(xc.reshape(-1, 3))
    truth = truth.view(R, -1)
    e_norm, e_el = norm_err(sdf[valid], truth[valid]), rel_err(sdf[valid], truth[valid], 1e-2)
    print(f"{name} render R={R}: |ours-f64| norm {e_norm:.2e} element-wise {e_el:.2e}")
    assert e_norm < ntol and e_el < tol
    # first hit: the first sample at or below zero, after at least one sample above it
    s = sdf.cpu()
    neg = s <= 0
    first = torch.where(neg.any(1), neg.long().argmax(1), torch.full((R,), -1))
    first = torch.where(first > 0, first, torch.full_like(first, -1))
    print(f"{name} render: {(first > 0).sum().item()} rays hit")
    assert (first > 0).any()
    assert torch.equal(hit_idx.cpu().long(), first)


@pytest.mark.parametrize("name,mode,passes,ntol,tol", MODES, ids=IDS)
@pytest.mark.parametrize("size", ["1", "63", "65", "wave+1", "3wave+37"])
def test_sdf_is_the_same_with_and_without_features(name, mode, passes, ntol, tol, size):
    net = _net()
    w = _sms() * 64
    P = {"1": 1, "63": 63, "65": 65, "wave+1": w + 1, "3wave+37": 3 * w + 37}[size]
    x = _points(P, seed=P)
    sdf_f, feat = ops.sdf_mlp_forward(x, net.packed_weights(), None, mode, want_feat=True)
    sdf_n, none = ops.sdf_mlp_forward(x, net.packed_weights(), None, mode, want_feat=False)
    assert none is None and feat.shape == (P, 256)
    assert torch.equal(sdf_f, sdf_n)


@pytest.mark.parametrize("name,mode,passes,ntol,tol", MODES, ids=IDS)
def test_layer8_dump_is_the_raw_accumulator(name, mode, passes, ntol, tol):
    """recmv_sdf_mlp_tc_debug with dbg_layer = 8 and no feature output still runs layer 8 and dumps its accumulator
    (before the bias) for the first 64 points; the sdf it stores is that of sdf_mlp_forward."""
    net = _net()
    P = 100
    x = _points(P, seed=3)
    packed = net.packed_weights()
    sdf = torch.full((P,), float("nan"), device=DEV)
    dbg = torch.full((64, 512), float("nan"), device=DEV)
    st = (ctypes.c_int * 4)()
    rc = _lib.load().recmv_sdf_mlp_tc_debug(x.data_ptr(), packed.data_ptr(), ops._pe_array(None), sdf.data_ptr(), None,
                                            P, passes, 8, dbg.data_ptr(), st, None)
    assert rc == 0 and st[0] == 0, (rc, list(st))
    ref, _ = ops.sdf_mlp_forward(x, packed, None, mode, want_feat=False)
    assert torch.equal(sdf, ref.view(-1))
    truth, tfeat = _truth(x[:64])
    b8 = _cache["w64"][1][8]
    raw = torch.cat([truth[:, None], tfeat], 1) - b8[None]
    e = norm_err(dbg[:, :257], raw)
    print(f"{name} layer-8 dump: |raw-f64| norm {e:.2e}")
    assert e < ntol
    assert bool((dbg[:, 257:384] == 0).all())   # zero-padded outputs of the third tile: computed, and exactly zero
