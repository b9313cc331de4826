"""GPU: the remesh path without openmesh.
  * recmv_vertex_faces (ops.vertex_faces) against oracle/vertex_faces_oracle.py, bit for bit in the pinned ascending
    order and per vertex as multisets: marching-cubes meshes of three networks on the coarse production pyramid, a
    1e5-face fan, unreferenced vertices, F = 0, one face, a multi-wave launch, a repeated vertex; the out-of-range flag;
    two runs bit-identical.
  * ops.mc_gpu_many against ops.mc_gpu per grid, bit for bit, with an empty grid among the others and the
    overflow-and-regrow path; one host read, or two with a regrowth.
  * discretize.discretize_many against each network's own device-worklist sweep and the torch-op sweep, bit for bit,
    statistics included, on the coarse pyramid and an isotropic one, with networks whose conflict rounds differ; host
    reads counted at ops.read_c2f_levels: per level, the most trips round the conflict loop any network needs.
  * utils.make_discretize_sdf / make_marching_cube_update on a stand-in garment model built from this package's
    networks: meshes bit-identical to discretize_all, the incidence lists equal to the oracle, the flags and optimizers
    set, no openmesh imported, and a subclass reaching both through inheritance."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import vertex_faces_oracle as vfo  # noqa: E402
from recmv_b200 import discretize, ops, testing  # noqa: E402
from recmv_b200 import model as M  # noqa: E402
from recmv_b200 import utils as ru  # noqa: E402
from recmv_b200.MCAcc import Seg3dLossless  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
COARSE = [(15, 21, 9), (29, 41, 17), (57, 81, 33), (113, 161, 65), (225, 321, 129)]   # train.py's coarse pyramid
ISO = [17, 33, 65, 129, 257]
BOX = ([-0.7, -1.0, -0.4], [0.7, 1.0, 0.4])
RATIO = 0.8


def _engine(resolutions, aniso=True):
    lo, hi = BOX if aniso else ([-1, -1, -1], [1, 1, 1])
    return Seg3dLossless(None, b_min=lo, b_max=hi, resolutions=resolutions, align_corners=False,
                         balance_value=0.0).to(DEV)


def _radius(r):
    return lambda device, multires, bias, width: M.getTmpSdf(device, multires, r, width)


def _nets():
    """A body and two garment-like networks: the committed test network, a plain geometric init with a smaller sphere,
    and another perturbed one."""
    body = testing.build_sdf(M.getTmpSdf, seed=0, perturb_seed=101).to(DEV)
    torch.manual_seed(1)
    plain = M.getTmpSdf("cpu", 6, 0.45, 256).to(DEV)
    garment = testing.build_sdf(_radius(0.5), seed=0, perturb_seed=202).to(DEV)
    return [body, plain, garment]


def _rough():
    """A rough perturbation (scale 0.3) that needs more conflict rounds on the isotropic pyramid than the others."""
    torch.manual_seed(0)
    return testing.perturb_module(M.getTmpSdf("cpu", 6, 0.6, 256), 101, scale=0.3).to(DEV)


@pytest.fixture(scope="module")
def nets():
    return _nets()


@pytest.fixture(scope="module")
def coarse_meshes(nets):
    """The three networks' meshes on the coarse pyramid, one network after another (discretize_all)."""
    return discretize.discretize_all(nets[0], nets[1:], _engine(COARSE), RATIO)


# ------------------------------------------------------------------------------------------------- vertex-face incidence
def _expected(faces, V):
    """The oracle's pairs, then (-1, -1) for each corner of a face with an index outside [0, V), as the kernel
    lists them."""
    efid, evid = vfo.incidence(faces.cpu().numpy(), V)
    tail = np.full(3 * faces.shape[0] - efid.size, -1, dtype=np.int64)
    return torch.from_numpy(np.concatenate([efid, tail])), torch.from_numpy(np.concatenate([evid, tail]))


def _check_incidence(faces, V):
    bad = bool(((faces < 0) | (faces >= V)).any())
    fid, vid = ops.vertex_faces(faces, V, check_indices=not bad)
    efid, evid = _expected(faces, V)
    assert fid.shape == vid.shape == (3 * faces.shape[0],)
    assert torch.equal(fid.cpu(), efid) and torch.equal(vid.cpu(), evid)
    # the same pairs per vertex, as multisets, whatever the order inside a vertex
    F = max(int(faces.shape[0]), 1)
    assert torch.equal(torch.sort(vid * F + fid).values.cpu(), torch.sort(evid * F + efid).values)
    fid2, vid2 = ops.vertex_faces(faces, V)
    assert torch.equal(fid, fid2) and torch.equal(vid, vid2)        # two runs bit-identical
    return fid, vid


def test_incidence_of_marching_cubes_meshes_at_production_size(coarse_meshes):
    for v, f in zip(*coarse_meshes):
        print(f"mesh: {v.shape[0]} vertices, {f.shape[0]} faces, {int((f < 0).any(1).sum())} faces across the far "
              f"boundary (index -1)")
        assert f.shape[0] > 10000
        _check_incidence(f, v.shape[0])


def test_incidence_of_a_1e5_face_fan():
    n = 100000
    i = torch.arange(1, n + 1, device=DEV)
    faces = torch.stack([torch.zeros_like(i), i, i + 1], 1)
    fid, vid = _check_incidence(faces, n + 2)
    assert torch.equal(fid[:n], torch.arange(n, device=DEV)) and bool((vid[:n] == 0).all())


def test_incidence_edges():
    g = torch.Generator(device="cpu").manual_seed(5)
    # unreferenced vertices: indices only in [100, 200) of 300
    _check_incidence(torch.randint(100, 200, (500, 3), generator=g).to(DEV), 300)
    fid, vid = _check_incidence(torch.zeros((0, 3), dtype=torch.int64, device=DEV), 10)      # F = 0
    assert fid.numel() == vid.numel() == 0
    fid, vid = _check_incidence(torch.tensor([[4, 0, 2]], device=DEV), 5)                    # one face
    assert fid.tolist() == [0, 0, 0] and vid.tolist() == [0, 2, 4]
    fid, vid = _check_incidence(torch.tensor([[1, 1, 0], [1, 0, 2]], device=DEV), 3)         # a repeated vertex
    assert fid.tolist() == [0, 1, 0, 0, 1, 1] and vid.tolist() == [0, 0, 1, 1, 1, 2]
    # many waves of blocks: 1.5e6 corners on a 132-SM device
    _check_incidence(torch.randint(0, 50000, (500000, 3), generator=g).to(DEV), 50000)


def test_incidence_flags_an_index_out_of_range():
    faces = torch.tensor([[0, 1, 2], [1, 3, 2], [2, 3, 4]], device=DEV)
    for bad in (5, -1):
        f = faces.clone()
        f[1, 2] = bad
        fid, vid = ops.vertex_faces(f, 5)                 # no read back without check_indices
        with pytest.raises(ValueError, match="outside"):
            ops.vertex_faces(f, 5, check_indices=True)
        # the valid faces keep their pairs; the bad face's three corners are (-1, -1), last
        assert fid.tolist() == [0, 0, 0, 2, 2, 2, -1, -1, -1] and vid.tolist() == [0, 1, 2, 2, 3, 4, -1, -1, -1]
    _check_incidence(faces, 5)                            # the flag is cleared by the next call


# ------------------------------------------------------------------------------------------------------- mc_gpu_many
def _count(monkeypatch, name):
    calls = []
    fn = getattr(ops, name)

    def wrapper(*a, **k):
        calls.append(a)
        return fn(*a, **k)
    monkeypatch.setattr(ops, name, wrapper)
    return calls


def _grids():
    from recmv_b200 import synth
    return [synth.sphere_sdf_grid(97, num=6, seed=4, device=DEV),
            torch.ones((33, 17, 21), device=DEV),                                   # no surface: an empty mesh
            synth.sphere_sdf_grid((41, 57, 29), num=3, seed=7, device=DEV),
            synth.sphere_sdf_grid(65, num=2, seed=9, device=DEV)]


STEPS = [(2 / 96,) * 3, (0.1, 0.2, 0.3), (0.05, 0.04, 0.07), (2 / 64,) * 3]
ORIGINS = [(-1.0,) * 3, (0.5, -0.5, 0.25), (-1.0, -1.1, -0.9), (-1.0,) * 3]


@pytest.mark.parametrize("capacity", [(1 << 20, 1 << 21), (16, 16)], ids=["fits", "regrow"])
def test_mc_gpu_many_equals_mc_gpu_per_grid(monkeypatch, capacity):
    grids = _grids()
    for iso in (0.0, 0.05):
        want = [ops.mc_gpu(g, *s, *o, iso) for g, s, o in zip(grids, STEPS, ORIGINS)]
        ops._scratch_cache.clear()                        # start from the given capacity, not from buffers kept
        reads = _count(monkeypatch, "_read_counters")
        got = ops.mc_gpu_many(grids, STEPS, ORIGINS, iso, capacity=capacity)
        monkeypatch.undo()
        assert len(reads) == (1 if capacity[0] > 16 else 2)
        assert got[1][0].shape == (0, 3) and got[1][1].shape == (0, 3)
        for (v, f), (wv, wf) in zip(got, want):
            assert torch.equal(v, wv) and torch.equal(f, wf)


def test_mc_gpu_many_refuses_bad_grids():
    with pytest.raises(RuntimeError, match="float32"):
        ops.mc_gpu_many([torch.ones((4, 4, 4), device=DEV, dtype=torch.float64)], [(1, 1, 1)], [(0, 0, 0)])
    with pytest.raises(RuntimeError, match="same length"):
        ops.mc_gpu_many([torch.ones((4, 4, 4), device=DEV)], [], [(0, 0, 0)])
    assert ops.mc_gpu_many([], [], []) == []


# -------------------------------------------------------------------------------------------------- discretize_many
def _tagged(net):
    def q(points):
        with torch.no_grad():
            return net.forward(points.reshape(-1, 3), RATIO).reshape(1, 1, -1)
    return q


def _level_reads(monkeypatch):
    """Wrap ops.read_c2f_levels: one entry per host read, the list of levels it served."""
    log = []
    fn = ops.read_c2f_levels

    def wrapper(levels):
        log.append([(lvl.W, lvl.H, lvl.D) for lvl in levels])
        return fn(levels)
    monkeypatch.setattr(ops, "read_c2f_levels", wrapper)
    return log


@pytest.mark.parametrize("pyramid", ["coarse", "isotropic"])
def test_discretize_many_is_bit_identical_per_network_with_shared_reads(monkeypatch, nets, pyramid):
    nets = nets + [_rough()]
    eng = _engine(COARSE) if pyramid == "coarse" else _engine(ISO, aniso=False)
    torch_grids, dev_grids, stats, trips = [], [], [], []
    for net in nets:
        q = _tagged(net)
        eng.query_func = q
        with torch.no_grad():
            torch_grids.append(eng.forward().clone())
        assert eng.last_sweep_path == "fused"
        q.recmv_sdf = (net, RATIO)
        log = _level_reads(monkeypatch)
        with torch.no_grad():
            dev_grids.append(eng.forward().clone())
        monkeypatch.undo()
        assert eng.last_sweep_path == "device-worklist"
        stats.append(list(eng.stats))
        per_level = {}
        for entry in log:
            per_level[entry[0]] = per_level.get(entry[0], 0) + 1
        trips.append(per_level)
    log = _level_reads(monkeypatch)
    grids = discretize.discretize_many(nets, eng, RATIO)
    monkeypatch.undo()
    for g, gd, gt in zip(grids, dev_grids, torch_grids):
        assert torch.equal(g, gd) and torch.equal(g, gt)
    assert eng.stats == stats[-1] and eng.last_sweep_path == "device-worklist" and eng.balance_value == 0.
    # one read per level for all networks, plus one per extra trip any network needs on that level
    levels = sorted(trips[0])
    expect = sum(max(t[lv] for t in trips) for lv in levels)
    print(f"{pyramid}: trips per level per network {trips}; shared reads {len(log)} (one network at a time: "
          f"{sum(sum(t.values()) for t in trips)})")
    assert len(log) == expect
    if pyramid == "isotropic":                  # the rough network takes a second trip round the conflict loop
        assert max(max(t.values()) for t in trips) >= 2
    assert all(len(entry) == len(nets) for entry in log[:1])
    ops.check_async_errors()


def test_discretize_many_falls_back_per_network(monkeypatch, nets):
    """A network that cannot use the worklist (here: the SIMT engine) takes the torch-op sweep; the others keep theirs."""
    eng = _engine(COARSE[:4])
    want = []
    for net in nets:
        eng.query_func = _tagged(net)
        with torch.no_grad():
            want.append(eng.forward().clone())
    nets[1].mlp_mode = ops.MLP_FP32_SIMT
    try:
        eng.query_func = _tagged(nets[1])
        with torch.no_grad():
            want[1] = eng.forward().clone()
        grids = discretize.discretize_many(nets, eng, RATIO)
    finally:
        nets[1].mlp_mode = None
    for g, w in zip(grids, want):
        assert torch.equal(g, w)


# ------------------------------------------------------------------------------------------------------------ drop-ins
class _Curve(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.scale = torch.nn.Parameter(torch.ones(4, 8, device=DEV))
        self.nx = torch.nn.Parameter(torch.zeros(4, 8, device=DEV))


class _Garment(torch.nn.Module):
    """The attributes OptimGarmentNetwork.discretizeSDF / marching_cube_update read, on this package's networks."""
    discretizeSDF = ru.make_discretize_sdf()
    marching_cube_update = ru.make_marching_cube_update()

    def __init__(self, nets, engine):
        super().__init__()
        self.sdf, self.garment_nets, self.engine = nets[0], list(nets[1:]), engine
        self.sdfShrinkRadius, self.remesh_time, self.opt_times = 0.01, 0.5, 3.0
        self.inter_free_curve = _Curve()
        self.visualizer, self.config = None, []

    def update_hierarchical_config(self, device, max_vs, max_fs):
        self.config.append((device, max_vs, max_fs))


class _LargePose(_Garment):
    """A subclass that, like OptimGarmentNetwork_LargePose, does not override the two methods."""


@pytest.mark.parametrize("cls", [_Garment, _LargePose])
def test_marching_cube_update_drop_in(monkeypatch, tmp_path, nets, coarse_meshes, cls):
    m = cls(nets, _engine(COARSE))
    m.marching_cube_update([0], RATIO, str(tmp_path), torch.device(DEV))   # a first remesh grows the output buffers
    m.remesh_time, m.config = 0.5, []
    reads = _count(monkeypatch, "_read_counters")
    level_reads = _level_reads(monkeypatch)
    m.marching_cube_update([0], RATIO, str(tmp_path), torch.device(DEV))
    monkeypatch.undo()
    assert len(reads) == 1 and len(level_reads) >= len(COARSE) - 1       # marching cubes: one read for all meshes
    assert "openmesh" not in sys.modules
    ref_vs, ref_fs = coarse_meshes
    for a, b in zip([m.body_vs, *m.garment_vs, m.body_fs, *m.garment_fs], ref_vs + ref_fs):
        assert torch.equal(a.detach(), b)
    assert all(v.requires_grad and v.is_leaf for v in [m.body_vs, *m.garment_vs])
    assert m.config == [(torch.device(DEV), max(v.shape[0] for v in ref_vs[1:]), max(f.shape[0] for f in ref_fs[1:]))]
    assert m.remesh_time == 1.0 and m.root == str(tmp_path) and os.path.isdir(tmp_path / "fl_mesh_show")
    for fid, vid, v, f in zip([m.TmpFid, *m.garment_tmpfid], [m.TmpVid, *m.garment_tmpvid], ref_vs, ref_fs):
        efid, evid = _expected(f, v.shape[0])
        assert torch.equal(fid.cpu(), efid) and torch.equal(vid.cpu(), evid)
    assert type(m.TmpOptimizer) is torch.optim.SGD and type(m.garment_optimizer) is torch.optim.SGD
    assert type(m.fl_optimizer) is torch.optim.AdamW
    assert [p is q for p, q in zip(m.TmpOptimizer.param_groups[0]["params"], [m.body_vs, *m.garment_vs])] == [True] * 3
    assert [p is q for p, q in zip(m.garment_optimizer.param_groups[0]["params"], m.garment_vs)] == [True] * 2
    assert len(m.garment_optimizer.param_groups[0]["params"]) == 2
    assert [p is q for p, q in zip(m.fl_optimizer.param_groups[0]["params"], m.inter_free_curve.parameters())] == [True] * 2
    for opt, lr, mom in ((m.TmpOptimizer, 0.05, 0.9), (m.garment_optimizer, 0.05, 0.9)):
        assert opt.param_groups[0]["lr"] == lr and opt.param_groups[0]["momentum"] == mom
    assert m.fl_optimizer.param_groups[0]["lr"] == 1e-4 and m.fl_optimizer.param_groups[0]["weight_decay"] == 0.01


def test_discretize_sdf_drop_in_quirks(nets):
    eng = _engine(COARSE[:4])
    m = _Garment(nets, eng)
    for ratio in (-1, RATIO):
        want = discretize.discretize_all(nets[0], nets[1:], _engine(COARSE[:4]), ratio)
        other = _engine(COARSE[:3])
        got = m.discretizeSDF(ratio, other, 0.3)                 # engine and balance_value are ignored
        assert other.query_func is None
        for a, b in zip(got[0] + got[1], want[0] + want[1]):
            assert torch.equal(a, b)
        assert eng.balance_value == 0. and eng.query_func.recmv_sdf == (nets[2], ratio)
    again = m.discretizeSDF(RATIO)
    assert all(a.data_ptr() != b.data_ptr() for a, b in zip(again[0] + again[1], got[0] + got[1]))  # fresh tensors
