"""SDF network -> triangle mesh: coarse-to-fine grid sweep + marching cubes.
Mirrors OptimNetwork.discretizeSDF (engineer/networks/OptimNetwork.py:207-220) and the per-garment
override (engineer/networks/OptimGarmentNetwork.py:581-618)."""
import torch

from . import ops


def _query_func(sdf_net, ratio):
    def query_func(points):
        with torch.no_grad():   # fused no-grad forward: one launch per query batch
            return sdf_net.forward(points.reshape(-1, 3), ratio).reshape(1, 1, -1)
    # declares the query as "this recmv_b200 network under no_grad": the sweep may then run as a device worklist
    # (Seg3dLossless._forward_device); any other query function takes the torch-op path
    query_func.recmv_sdf = (sdf_net, ratio)
    return query_func


def discretize_sdf(sdf_net, engine, ratio, balance_value=0.):
    """engine: recmv_b200.MCAcc.Seg3dLossless.  Returns (verts [V,3] f32, faces [F,3] i64)."""
    engine.balance_value = balance_value
    engine.query_func = _query_func(sdf_net, ratio)
    with torch.no_grad():
        sdfs = engine.forward()
    verts, faces = ops.mc_gpu(sdfs[0, 0].permute(2, 1, 0).contiguous(), engine.spacing_x, engine.spacing_y,
                              engine.spacing_z, engine.bx, engine.by, engine.bz, balance_value)
    return verts, faces


def discretize_all(body_sdf, garment_nets, engine, ratio):
    """Body + every garment net (OptimGarmentNetwork.py:600-618) -> ([verts...], [faces...])."""
    pts, fcs = [], []
    for net in [body_sdf] + list(garment_nets):
        v, f = discretize_sdf(net, engine, ratio, 0.)
        pts.append(v)
        fcs.append(f)
    return pts, fcs


def discretize_many(nets, engine, ratio):
    """The coarse-to-fine grids of several networks on one engine at iso 0 (Seg3dLossless.forward_many): one [1,1,D,H,W]
    grid per network, each bit-identical to that network's own sweep, with one host read per pyramid level for all of
    them instead of one per level per network."""
    engine.balance_value = 0.
    with torch.no_grad():
        return engine.forward_many([_query_func(net, ratio) for net in nets])


def mesh_many(nets, engine, ratio):
    """discretize_all for any list of networks: discretize_many, then marching cubes on every grid with one host read
    (ops.mc_gpu_many).  Returns ([verts...], [faces...]), each mesh bit-identical to discretize_sdf's for its network."""
    grids = discretize_many(nets, engine, ratio)
    step, origin = (engine.spacing_x, engine.spacing_y, engine.spacing_z), (engine.bx, engine.by, engine.bz)
    meshes = ops.mc_gpu_many([g[0, 0].permute(2, 1, 0).contiguous() for g in grids], [step] * len(grids),
                             [origin] * len(grids), 0.)
    return [m[0] for m in meshes], [m[1] for m in meshes]
