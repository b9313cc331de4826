"""CPU: the remesh drop-ins (utils.make_discretize_sdf / make_marching_cube_update) keep the bookkeeping of the
reference's own OptimGarmentNetwork.discretizeSDF / marching_cube_update (OptimGarmentNetwork.py:581-618, 678-740), run
unmodified through oracle/refload.py.  Both sides get the same fake stages: the sweep returns a grid that names its
network, marching cubes (the reference's MCGpu.mc_gpu, our ops.mc_gpu_many) turns it into that network's fake mesh,
and the incidence (openmesh's vertex_face_indices on the reference side, our ops.vertex_faces) is
oracle/vertex_faces_oracle.py.  Compared: the mesh lists, the incidence lists, remesh_time, the
update_hierarchical_config arguments, the three optimizers, the printed lines, the vanished-mesh assertion, and that
the `engine` / `balance_value` arguments are ignored.  Also the NumPy incidence oracle on a hand-worked mesh."""
import importlib
import os
import sys
import types

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import refload, vertex_faces_oracle as vfo  # noqa: E402
from recmv_b200 import discretize, ops  # noqa: E402
from recmv_b200 import utils as ru  # noqa: E402


def test_incidence_oracle_on_a_hand_worked_mesh():
    # a square split along 0-2, a third triangle on 2-3, vertex 5 unreferenced
    faces = [[0, 1, 2], [0, 2, 3], [3, 2, 4]]
    fi = vfo.vertex_face_indices(faces, 6)
    assert fi.tolist() == [[0, 1, -1], [0, -1, -1], [0, 1, 2], [1, 2, -1], [2, -1, -1], [-1, -1, -1]]
    fid, vid = vfo.incidence(faces, 6)
    assert fid.tolist() == [0, 1, 0, 0, 1, 2, 1, 2, 2]
    assert vid.tolist() == [0, 0, 1, 2, 2, 2, 3, 3, 4]
    # a repeated vertex gives one pair per corner; no faces give empty lists
    assert vfo.incidence([[1, 1, 0]], 2)[0].tolist() == [0, 0, 0]
    assert vfo.incidence([[1, 1, 0]], 2)[1].tolist() == [0, 1, 1]
    assert [a.size for a in vfo.incidence(np.zeros((0, 3), np.int64), 3)] == [0, 0]


def _mesh(V, faces):
    g = torch.Generator().manual_seed(V)
    return torch.randn(V, 3, generator=g), torch.tensor(faces, dtype=torch.int64).view(-1, 3)


MESHES = [_mesh(4, [[0, 1, 2], [0, 3, 1], [1, 3, 2], [0, 2, 3]]),            # body: a tetrahedron
          _mesh(5, [[0, 1, 2], [0, 2, 3]]),                                 # garment 1: vertex 4 unreferenced
          _mesh(3, [[0, 1, 2]])]                                            # garment 2
EMPTY = (torch.zeros(0, 3), torch.zeros(0, 3, dtype=torch.int64))


class _Net(torch.nn.Module):
    def __init__(self, k):
        super().__init__()
        self.k = k
        self.seen = []

    def forward(self, points, ratio):
        self.seen.append((ratio, torch.is_grad_enabled()))
        return torch.full((points.reshape(-1, 3).shape[0],), float(self.k))


class _Engine:
    spacing_x, spacing_y, spacing_z = 0.1, 0.2, 0.3
    bx, by, bz = -1.0, -2.0, -3.0

    def __init__(self):
        self.balance_value, self.query_func, self.calls = 0.7, None, []

    def forward(self):        # the sweep: a grid that names the network the query function evaluates
        self.calls.append(self.balance_value)
        return self.query_func(torch.zeros(1, 1, 3)).reshape(1, 1, 1, 1, 1).expand(1, 1, 2, 2, 2)


def _fake_mesh(grid, meshes):
    v, f = meshes[int(grid.reshape(-1)[0])]
    return [v.clone(), f.clone()]


class _Curve(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.a, self.b = torch.nn.Parameter(torch.zeros(3)), torch.nn.Parameter(torch.ones(2))


def _model(cls, meshes):
    m = object.__new__(cls)
    torch.nn.Module.__init__(m)
    m.sdf = _Net(0)
    m.garment_nets = [_Net(1), _Net(2)][:len(meshes) - 1]
    m.engine = _Engine()
    m.sdfShrinkRadius = 0.01
    m.remesh_time = 2.4
    m.inter_free_curve = _Curve()
    m.opt_times = 7.0
    m.log = []
    m.update_hierarchical_config = lambda device, V, F: m.log.append(("config", device, V, F))
    m.visualizer = object()
    m.visualize_curve_mesh = lambda path, times, device: m.log.append(("vis", path, times, device))
    return m


@pytest.fixture(scope="module")
def ref():
    if not refload.available():
        pytest.skip("needs the reference source tree")
    refload.load()
    return (importlib.import_module("engineer.networks.OptimGarmentNetwork"),
            importlib.import_module("engineer.networks.OptimGarmentNetwork_Large_Pose"))


def _run_pair(ref, monkeypatch, tmp_path, meshes, large=False):
    """(reference model, our model) after marching_cube_update(...) on both, and what the fake stages saw."""
    OGN, OGNL = ref
    mc_seen, sweep_seen, mc_many_seen = [], [], []

    def mc_gpu(grid, sx, sy, sz, x0, y0, z0, iso):
        mc_seen.append(((sx, sy, sz), (x0, y0, z0), iso))
        return _fake_mesh(grid, meshes)

    def vertex_face_indices(vs, fs):
        assert isinstance(vs, np.ndarray) and isinstance(fs, np.ndarray)
        return vfo.vertex_face_indices(fs, vs.shape[0])
    monkeypatch.setattr(OGN, "MCGpu", types.SimpleNamespace(mc_gpu=mc_gpu))
    monkeypatch.setattr(OGN, "om", types.SimpleNamespace(
        TriMesh=lambda vs, fs: types.SimpleNamespace(vertex_face_indices=lambda: vertex_face_indices(vs, fs))))
    # the reference's own methods, taken before the drop-ins are bound on the class
    Ref = type("Ref", (OGN.OptimGarmentNetwork,), {k: OGN.OptimGarmentNetwork.__dict__[k]
                                                   for k in ("discretizeSDF", "marching_cube_update")})
    reference = _model(Ref, meshes)

    def discretize_many(nets, engine, ratio):
        sweep_seen.append(([n.k for n in nets], engine, ratio))
        return [torch.full((1, 1, 2, 2, 2), float(n.k)) for n in nets]

    def mc_gpu_many(grids, steps, origins, iso):
        mc_many_seen.append((steps, origins, iso))
        return [_fake_mesh(g, meshes) for g in grids]

    def vertex_faces(faces, V):
        fid, vid = vfo.incidence(faces.numpy(), V)
        return torch.from_numpy(fid), torch.from_numpy(vid)
    monkeypatch.setattr(discretize, "discretize_many", discretize_many)
    monkeypatch.setattr(ops, "mc_gpu_many", mc_gpu_many)
    monkeypatch.setattr(ops, "vertex_faces", vertex_faces)
    monkeypatch.setattr(OGN.OptimGarmentNetwork, "discretizeSDF", ru.make_discretize_sdf())
    monkeypatch.setattr(OGN.OptimGarmentNetwork, "marching_cube_update", ru.make_marching_cube_update())
    ours = _model(OGNL.OptimGarmentNetwork_LargePose if large else OGN.OptimGarmentNetwork, meshes)
    out = []
    for m in (reference, ours):
        try:
            m.marching_cube_update([0, 1], 0.5, str(tmp_path / type(m).__name__), "cpu")
            out.append(None)
        except AssertionError as e:
            out.append(e)
    return reference, ours, out, mc_seen, sweep_seen, mc_many_seen


def _params(opt):
    return [[p for p in g["params"]] for g in opt.param_groups]


def _hyper(opt):
    return [{k: v for k, v in g.items() if k != "params"} for g in opt.param_groups]


@pytest.mark.parametrize("large", [False, True], ids=["OptimGarmentNetwork", "LargePose"])
def test_marching_cube_update_bookkeeping_matches_the_reference(ref, monkeypatch, tmp_path, capsys, large):
    r, o, err, mc_seen, sweep_seen, mc_many_seen = _run_pair(ref, monkeypatch, tmp_path, MESHES, large)
    printed = capsys.readouterr().out.splitlines()
    assert err == [None, None]
    assert printed == ["tmp sdf generate"] * 2
    # the sweeps: our engine, iso 0 and the ratio; the reference's marching cubes at the engine's spacing and origin
    assert sweep_seen == [([0, 1, 2], o.engine, 0.5)]
    assert mc_seen == [((0.1, 0.2, 0.3), (-1.0, -2.0, -3.0), 0.)] * 3
    assert mc_many_seen == [([(0.1, 0.2, 0.3)] * 3, [(-1.0, -2.0, -3.0)] * 3, 0.)]
    assert [n.seen for n in [r.sdf, *r.garment_nets]] == [[(0.5, False)]] * 3
    assert r.engine.calls == [0.] * 3 and r.engine.balance_value == 0.
    # the meshes and their flags
    for m in (r, o):
        assert [m.body_vs, *m.garment_vs] is not None and all(v.requires_grad for v in [m.body_vs, *m.garment_vs])
    for a, b in zip([r.body_vs, *r.garment_vs, r.body_fs, *r.garment_fs],
                    [o.body_vs, *o.garment_vs, o.body_fs, *o.garment_fs]):
        assert a.dtype == b.dtype and torch.equal(a.detach(), b.detach())
    assert len(r.garment_vs) == len(o.garment_vs) == 2
    # incidence lists
    for a, b in zip([r.TmpFid, r.TmpVid, *r.garment_tmpfid, *r.garment_tmpvid],
                    [o.TmpFid, o.TmpVid, *o.garment_tmpfid, *o.garment_tmpvid]):
        assert a.dtype == b.dtype == torch.int64 and torch.equal(a, b)
    assert len(r.garment_tmpfid) == len(o.garment_tmpfid) == 2
    # remesh_time, config, visualizer
    assert r.remesh_time == o.remesh_time == 3.0 and type(r.remesh_time) is type(o.remesh_time)
    assert [e[0] for e in r.log] == [e[0] for e in o.log] == ["config", "vis"]
    assert r.log[0] == o.log[0] == ("config", "cpu", 5, 2)
    assert r.log[1][2:] == o.log[1][2:] == (7, "cpu")
    assert os.path.isdir(o.log[1][1]) and o.log[1][1] == os.path.join(o.root, "fl_mesh_show")
    assert r.root.endswith("Ref") and o.root.endswith(type(o).__name__)
    # the optimizers: types, hyperparameters, parameter identity and order
    for name in ("TmpOptimizer", "garment_optimizer", "fl_optimizer"):
        a, b = getattr(r, name), getattr(o, name)
        assert type(a) is type(b) and _hyper(a) == _hyper(b), name
    for m in (r, o):
        assert [[id(p) for p in g] for g in _params(m.TmpOptimizer)] == [[id(v) for v in [m.body_vs, *m.garment_vs]]]
        assert [[id(p) for p in g] for g in _params(m.garment_optimizer)] == [[id(v) for v in m.garment_vs]]
        assert [[id(p) for p in g] for g in _params(m.fl_optimizer)] == [[id(p) for p in m.inter_free_curve.parameters()]]
    assert type(o.TmpOptimizer) is torch.optim.SGD and _hyper(o.TmpOptimizer)[0]["lr"] == 0.05
    assert _hyper(o.TmpOptimizer)[0]["momentum"] == 0.9
    assert type(o.fl_optimizer) is torch.optim.AdamW and _hyper(o.fl_optimizer)[0]["lr"] == 1e-4


def test_vanished_body_mesh_asserts_after_the_config_call(ref, monkeypatch, tmp_path, capsys):
    r, o, err, *_ = _run_pair(ref, monkeypatch, tmp_path, [EMPTY] + MESHES[1:])
    assert all(isinstance(e, AssertionError) for e in err)
    assert capsys.readouterr().out.splitlines() == ["tmp sdf generate", "tmp sdf vanished..."] * 2
    assert r.log == o.log == [("config", "cpu", 5, 2)]
    assert r.remesh_time == o.remesh_time == 2.4
    for m in (r, o):
        assert not hasattr(m, "TmpOptimizer") and not hasattr(m, "TmpFid")


def test_discretize_sdf_ignores_engine_and_balance_value(ref, monkeypatch, tmp_path):
    r, o, *_ = _run_pair(ref, monkeypatch, tmp_path, MESHES)
    seen = []
    monkeypatch.setattr(discretize, "discretize_many",
                        lambda nets, engine, ratio: seen.append((engine, ratio)) or
                        [torch.full((1, 1, 2, 2, 2), float(n.k)) for n in nets])
    other_r, other_o = _Engine(), _Engine()
    r.engine.calls.clear()
    vs_r, fs_r = r.discretizeSDF(-1, other_r, 0.3)
    vs_o, fs_o = o.discretizeSDF(-1, other_o, 0.3)
    assert other_r.calls == [] and other_o.calls == [] and other_r.query_func is None
    assert r.engine.calls == [0.] * 3 and [n.seen[-1] for n in [r.sdf, *r.garment_nets]] == [(-1, False)] * 3
    assert seen == [(o.engine, -1)]
    assert len(vs_r) == len(vs_o) == 3
    for a, b, ref_mesh in zip(vs_r + fs_r, vs_o + fs_o, [m[0] for m in MESHES] + [m[1] for m in MESHES]):
        assert torch.equal(a, b) and torch.equal(a, ref_mesh)
        assert b.data_ptr() != ref_mesh.data_ptr()                    # fresh tensors
