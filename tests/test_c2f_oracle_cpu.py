"""CPU: oracle/c2f_oracle.py, the per-kernel restatement of one sweep level, chained into a whole sweep equals
Seg3dLossless._forward_torch (itself bit-identical to the reference class, tests/test_c2f_cpu.py) query by query: the
same set of points in every call of the query function, bit for bit, the same statistics and the same final grid."""
import pytest
import torch
import torch.nn.functional as F

from oracle import c2f_oracle as co
from recmv_b200.MCAcc import Seg3dLossless, create_grid3D
from test_c2f_cpu import KW, sphere_query


def _rows(p):
    """The rows of a point batch as a sorted list of bit patterns (the sweep's order inside a batch is not the oracle's)."""
    return sorted(map(tuple, p.reshape(-1, 3).contiguous().view(torch.int32).tolist()))


def oracle_sweep(query, b_min, b_max, resolutions, balance):
    """The sweep from the oracle's pieces; returns (grid [D,H,W], stats, list of queried point batches)."""
    final = tuple(resolutions[-1])
    calculated = torch.zeros(final[::-1], dtype=torch.bool)
    calls, stats = [], []
    occ = done = None
    for li, level in enumerate(resolutions):
        W, H, D = level
        if li == 0:
            idx = torch.arange(W * H * D)
            pts = co.query_points(idx, level, final, b_min, b_max)
            calls.append(pts)
            occ = query(pts).view(D, H, W).float()
            done = torch.ones((D, H, W), dtype=torch.bool)
            sx, sy, sz = co.stride(level, final)
            calculated[::sz, ::sy, ::sx] = True
            stats.append((W, H, D, W * H * D))
            continue
        occ, done, idx = co.refine(occ, done, balance)
        queried = 0
        while idx.numel():
            pts = co.query_points(idx, level, final, b_min, b_max)
            calls.append(pts)
            queried += idx.numel()
            conflicts = co.scatter(idx, query(pts).view(-1), occ, done, calculated, balance, level, final)
            idx = co.next_round(conflicts, calculated, level, final)
        stats.append((W, H, D, queried))
    return occ, stats, calls


def wavy_query(points):
    """A field with detail below the coarse cell, so levels run several conflict rounds."""
    p = points.reshape(-1, 3)
    return (p.norm(dim=1) - 0.55 + 0.3 * torch.sin(31 * p[:, 0]) * torch.sin(27 * p[:, 1]) * torch.cos(37 * p[:, 2])).reshape(1, 1, -1)


ANISO = dict(KW, b_min=[-0.7, -1.0, -0.4], b_max=[0.7, 1.0, 0.4], resolutions=[(15, 21, 9), (29, 41, 17), (57, 81, 33)])


@pytest.mark.parametrize("kw,query", [(KW, sphere_query), (ANISO, wavy_query)], ids=["sphere", "aniso-wavy"])
def test_oracle_sweep_equals_forward_torch_query_by_query(kw, query):
    calls = []

    def recording(points):
        # contiguous rows: the sweep hands nonzero()'s column-major points over, and a vectorised norm rounds differently
        # on another memory layout; that belongs to the query function, not to the sweep
        calls.append(points.detach().reshape(-1, 3).contiguous())
        return query(calls[-1])
    eng = Seg3dLossless(recording, **kw)
    grid = eng._forward_torch()[0, 0]
    o_grid, o_stats, o_calls = oracle_sweep(query, kw["b_min"], kw["b_max"], [tuple(r) for r in kw["resolutions"]], 0.0)
    assert o_stats == list(eng.stats)
    assert len(o_calls) == len(calls)
    for ours, theirs in zip(o_calls, calls):
        assert _rows(ours) == _rows(theirs)
    assert torch.equal(o_grid, grid)
    if query is wavy_query:       # the conflict loop ran: more query calls than levels
        assert len(calls) > len(kw["resolutions"]) + 2


def test_oracle_pieces_against_torch_ops():
    """upsample == F.interpolate on the values and on the 0/1 flags (the sweep's definition), with values on the
    balance value and axes of size 1 and 2; the level-0 points equal batch_eval's."""
    g = torch.Generator().manual_seed(3)
    for shape in ((5, 6, 7), (1, 4, 2), (2, 2, 2), (3, 1, 1)):
        x = torch.randn(shape, generator=g).mul(2).round()           # many values equal to the balance value 0
        v, mixed = co.upsample(x, 0.0)
        size = tuple(2 * s - 1 for s in shape)
        ref = F.interpolate(x[None, None], size=size, mode="trilinear", align_corners=True)[0, 0]
        valid = F.interpolate((x > 0.0).float()[None, None], size=size, mode="trilinear", align_corners=True)[0, 0]
        assert torch.equal(v, ref) and torch.equal(mixed, (valid > 0) & (valid < 1))
    eng = Seg3dLossless(sphere_query, **KW)
    seen = []
    eng.query_func = lambda points: seen.append(points) or sphere_query(points)
    final, level = KW["resolutions"][-1], KW["resolutions"][0]
    coords = create_grid3D(0, torch.tensor(final) - 1, steps=torch.tensor(level), device="cpu")
    eng.batch_eval(coords.unsqueeze(0))
    pts = co.query_points(torch.arange(level[0] * level[1] * level[2]), level, final, KW["b_min"], KW["b_max"])
    assert torch.equal(seen[0].view(-1, 3), pts)
