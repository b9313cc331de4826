"""A garment-model stand-in for `surface_render_loss` (OptimGarmentNetwork.py:1083-1219) on this package's networks, and
the reference's glue restated in torch.  Shared by tests/test_gpu_loss_points.py and tools/bench_surface_render_loss.py.

`scene` builds a lightweight `self` (conf with the shipped weights of configs/people_snapshot/female-3-casual.conf,
garment nets, the [MLPTranslator, LBSkinner] composite, the colour network, garment vertices, info with rayInfo) and
the method's arguments.  `reference_flow` is the reference's method body with its glue kept as the reference writes
it: boolean indexing by `check` and `valid_mask`, `.item()` for every info value, the host tests of the
singular-Jacobian fallbacks (utils.compute_cardinal_rays / compute_deformed_normals) and torch_scatter's mean
restated with `index_add_`.  Its points come from `points(g, P, V)`: `torch_points` draws them as the reference does
(CPU `torch.rand`, `torch.randn_like`), or a caller passes the drop-in's own to compare the two on the same points."""
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

from recmv_b200 import synth, testing, utils  # noqa: E402

CONF = {"grad_weight": 1.0, "offset_weight": 0.0, "def_regu.weight": 0.1, "def_regu.c": 0.5, "color_weight": 0.5,
        "normal_weight": 0.1, "weighted_normal": True}
RATIO = {"sdfRatio": 0.8, "deformerRatio": 0.6, "renderRatio": 0.9}


class Conf:
    def __init__(self, d):
        self.d = dict(d)

    def get_float(self, key):
        return float(self.d[key])

    def get_bool(self, key):
        return bool(self.d[key])

    def __contains__(self, key):
        return key in self.d or any(k.startswith(key + ".") for k in self.d)


def networks(dev):
    """(sdf, deformer, colour network) of tests/golden/make_golden.py's surface scene, the colour network built as
    tests/golden/make_golden_surface_render_loss.py builds the reference's (seed 2, perturbed with seed 303)."""
    import make_golden as mg
    import recmv_b200.model as M

    class _Mods:
        getTmpSdf = staticmethod(M.getTmpSdf)
        MLPTranslator, LBSkinner, CompositeDeformer = M.MLPTranslator, M.LBSkinner, M.CompositeDeformer

    sdf, deformer = mg.surface_scene(_Mods, _Mods, device="cpu")
    torch.manual_seed(2)
    rn = M.RenderingNetwork_view_norm(256, d_in=9, d_out=3, dims=[512] * 4, mode="idr", weight_norm=True, multires_v=4,
                                      multires_n=0)
    testing.perturb_module(rn, 303)
    return sdf.to(dev), deformer.to(dev), rn.to(dev)


def scene(dev, N=2, H=64, W=64, M=(600, 500), V=(2500, 3100), seed=5, conf=None, nets=None):
    """(self, args of surface_render_loss) for len(M) garments with M[g] surface points and V[g] vertices."""
    gen = synth.generator(seed)
    sdf, deformer, rn = nets if nets is not None else networks(dev)
    G = len(M)
    poses, trans = synth.poses_trans(N, seed=11)
    poses, trans = poses.to(dev).requires_grad_(True), trans.to(dev).requires_grad_(True)
    conds = [(torch.randn((N, 128), generator=gen) * 0.1).to(dev).requires_grad_(True) for _ in range(G + 1)]
    rendcond = torch.zeros((N, 1), device=dev)
    names = ["upper", "bottom", "dress", "skirt", "coat"][:G]

    def unit(n):
        return torch.nn.functional.normalize(torch.randn((n, 3), generator=gen), dim=1)

    init, check, rows, cols, binds, rays, verts, info = [], [], [], [], [], [], [], {}
    for g in range(G):
        init.append((unit(M[g]) * 0.45 + torch.randn((M[g], 3), generator=gen) * 0.02).to(dev))
        verts.append((unit(V[g]) * 0.45).to(dev))
        c = torch.rand((M[g],), generator=gen) < 0.8
        check.append(c.to(dev))
        rows.append(torch.randint(0, H, (M[g],), generator=gen).to(dev))
        cols.append(torch.randint(0, W, (M[g],), generator=gen).to(dev))
        binds.append(torch.randint(0, N, (M[g],), generator=gen).to(dev))
        rays.append(unit(M[g]).to(dev))
        info[f"{names[g]}_rayInfo"] = (M[g], int(c.sum()))
    gtCs = torch.rand((N, H, W, 3), generator=gen).to(dev)
    normal = torch.nn.functional.normalize(torch.randn((N, H, W, 3), generator=gen), dim=-1)
    normal[:, : H // 4] = 0.                       # background rows: invalid normals
    q = torch.nn.functional.normalize(torch.tensor([0.97, 0.05, -0.2, 0.1]), dim=0)
    w_, x, y, z = q.tolist()
    R = torch.tensor([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w_), 2 * (x * z + y * w_)],
                      [2 * (x * y + z * w_), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w_)],
                      [2 * (x * z - y * w_), 2 * (y * z + x * w_), 1 - 2 * (x * x + y * y)]])
    cameras = types.SimpleNamespace(R=R.view(1, 3, 3).expand(N, 3, 3).contiguous().to(dev))

    self = types.SimpleNamespace(
        garment_size=G, garment_names=names, garment_nets=[sdf] * G, garment_vs=verts, deformer=deformer,
        netRender=rn, conf=Conf(CONF if conf is None else conf), info=info,
        get_grad_parameters=lambda frame_ids, device: (conds, poses, trans, rendcond))
    args = ({"normal": normal.to(dev)}, N, cameras, torch.arange(N, device=dev), RATIO, check, gtCs, init, rows, cols,
            binds, rays, dev)
    return self, args, (conds, poses, trans)


def torch_points(g, P, V, S):
    """The reference's draws (OptimGarmentNetwork.py:1108, 1139-1141): CPU torch.rand, boolean indexing,
    utils.sample_points with torch.randn_like / torch.rand."""
    def sample_points(x, ratio):
        local = x + torch.randn_like(x) * 0.01
        if ratio > 0:
            return torch.cat([local, torch.rand(x.shape[0] // ratio, 3, device=x.device) * 3.6 - 1.8])
        return local

    n = V.shape[0]
    X_E = sample_points(torch.cat([P, V[torch.rand(n) < float(S) / float(n)].detach()]), 6)
    B_D = torch.cat([P, V[torch.rand(n) < float(S) / float(n)].detach()])
    return X_E, torch.cat([B_D, sample_points(B_D, 0)])


def _scatter_mean(e, b, N):
    s = torch.zeros(N, dtype=e.dtype, device=e.device).index_add_(0, b, e)
    n = torch.zeros(N, dtype=e.dtype, device=e.device).index_add_(0, b, torch.ones_like(e))
    return s / n.clamp_min(1)


def reference_flow(self, datas, N, cameras, frame_ids, ratio, check_list, gtCs, init_garment_ps_list,
                   sample_batch_garment_row_list, sample_batch_garment_col_list, sample_batch_garment_inds_list,
                   sample_rays_list, device, points=None):
    """The reference's surface_render_loss restated in torch on this package's networks (see the module docstring)."""
    G = self.garment_size
    S = 4096 // G
    points = points or (lambda g, P, V: torch_points(g, P, V, S))
    self.TmpPs, self.rays, self.batch_inds, self.row_inds, self.col_inds = ([None] * G for _ in range(5))
    conf = self.conf
    total_loss = 0.
    d_cond_list, poses, trans, rendcond = self.get_grad_parameters(frame_ids, device)
    for g, (init, rows, cols, binds) in enumerate(zip(init_garment_ps_list, sample_batch_garment_row_list,
                                                      sample_batch_garment_col_list, sample_batch_garment_inds_list)):
        name, net = self.garment_names[g], self.garment_nets[g]
        X_E, X_D = points(g, init, self.garment_vs[g])
        pn = X_E.detach().requires_grad_()
        grad = net.gradient(pn, net(pn, ratio))
        grad_loss = ((grad.norm(2, dim=-1) - 1) ** 2).mean()
        self.info[f"{name}_grad_loss"] = grad_loss.item()
        total_loss += grad_loss * conf.get_float("grad_weight")
        d_cond = d_cond_list[g + 1]
        with torch.no_grad():
            self.deformer.defs[0](pn.view(1, -1, 3).expand(N, -1, 3), d_cond, ratio=ratio, offset_type=name)
            self.info[f"{name}_offset_loss"] = self.deformer.defs[0].offset[name].view(-1, 3).norm(dim=-1).mean().item()
        def_loss = utils.deformation_regulariser(self.deformer.defs[0], X_D.detach().view(1, -1, 3).expand(N, -1, 3),
                                                 d_cond, ratio, conf.get_float("def_regu.c"), offset_type=name)
        self.info[f"def_{name}_loss"] = def_loss.item()
        total_loss += def_loss * conf.get_float("def_regu.weight")
        self.info[f"{name}_color_loss"] = -1.0
        check = check_list[g]
        if self.info[f"{name}_rayInfo"][1] > 0:
            self.TmpPs[g] = init[check]
            self.TmpPs[g].requires_grad = True
            self.rays[g] = sample_rays_list[g][check]
            self.batch_inds[g], self.col_inds[g], self.row_inds[g] = binds[check], cols[check], rows[check]
            ps, b = self.TmpPs[g], self.batch_inds[g]
            sdfs = net(ps, ratio)
            nx = torch.autograd.grad(sdfs, ps, torch.ones_like(sdfs), retain_graph=True, create_graph=True)[0]
            nx = nx / nx.norm(dim=1, keepdim=True)
            defconds = [d_cond, [poses, trans]]
            crays, defVs = utils.compute_cardinal_rays(self.deformer, ps, self.rays[g], defconds, b, ratio, "train",
                                                       offset_type=name)
            colors = utils.compute_netRender_color(self.netRender, ps, defVs, nx, crays, net.rendcond, rendcond[b],
                                                   ratio)
            color_loss = (gtCs[b, self.row_inds[g], self.col_inds[g], :] - colors).abs().sum(1)
            color_loss = _scatter_mean(color_loss, b, N).mean()
            self.info[f"{name}_color_loss"] = color_loss.item()
            total_loss += conf.get_float("color_weight") * color_loss
            cnx, _ = utils.compute_deformed_normals(net, self.deformer, ps, defconds, b, ratio, "test", name)
            weights = torch.clamp((-self.rays[g] * cnx.detach()).sum(1).detach(), max=1., min=0.) ** 2
            gtn = datas["normal"].to(device)[b, self.row_inds[g], self.col_inds[g], :]
            flip = torch.tensor([[-1., 0., 0.], [0., 1., 0.], [0., 0., -1.]], device=device)
            gtn = ((cameras.R[0] @ flip) @ gtn.view(-1, 3, 1)).view(-1, 3)
            nrm = gtn.norm(dim=1, keepdim=True)
            valid = (nrm > 0.0001)[..., 0]
            gtn[valid] = gtn[valid] / nrm[valid]
            ds = self.deformer(ps, defconds, b, ratio=ratio, offset_type=name)
            J = utils.compute_Jacobian(ps, ds, True, True)
            gtn = (J.transpose(-2, -1) @ gtn.view(-1, 3, 1)).view(-1, 3)
            normal_loss = (gtn - nx).norm(2, dim=1) * weights
            normal_loss = _scatter_mean(normal_loss[valid], b[valid], N).mean()
            self.info[f"{name}_normal_loss"] = normal_loss.item()
            total_loss += conf.get_float("normal_weight") * normal_loss
    return total_loss
