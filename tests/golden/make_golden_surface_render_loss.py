"""Writes tests/golden/surface_render_loss_ref.npz: the reference's OWN `OptimGarmentNetwork.surface_render_loss`
(engineer/networks/OptimGarmentNetwork.py:1083-1219), unmodified, run on the CPU in float32 and float64 with
  * a lightweight `self`: conf with the shipped weights of configs/people_snapshot/female-3-casual.conf (grad 1,
    offset 0, def_regu 0.1 / c 0.5, colour 0.5, normal 0.1, weighted_normal), two garments sharing the reference's
    `ImplicitNetwork` (testing.build_sdf seed 0, perturbed with seed 101), `CompositeDeformer(MLPTranslator,
    LBSkinner)` of tests/golden/make_golden.py's surface scene and `RenderingNetwork_view_norm` (seed 2, perturbed
    with seed 303), the garment vertices, and `info` with each garment's rayInfo;
  * the module's `torch.rand` answering with oracle/loss_points_oracle.py's E / D uniforms, in the reference's call
    order (E then D, garment by garment), so the reference's own `< float(S)/float(V)` comparison decides what is kept;
  * the module's `utils.sample_points` answering with the oracle's lane values (x + z 0.01 at the E-local / D-local
    counters, the global rows at the E-global counters);
  * the module's `scatter` rebound to a mean restatement (torch_scatter is not on this stack);
  * in float64, torch's default dtype set to float64 for the call, so the constants the method builds match.
Needs the reference source tree (oracle/refload.py).

Stored: the inputs, the stream, the points the reference drew with (its own B_E / B_D), its compacted rows, the loss
and every info term, and the gradients of the loss to the three networks' parameters (every 257th entry of each,
flattened) and to poses, trans and the garment conditions, in float32 and float64.

    python tests/golden/make_golden_surface_render_loss.py
"""
import importlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from oracle import loss_points_oracle as lpo, refload  # noqa: E402
from recmv_b200 import synth, testing  # noqa: E402

OUT = os.path.join(HERE, "surface_render_loss_ref.npz")
SEED = 0x0123456789ABCDEF
OFFSET = (1 << 32) - 9000          # the counters cross into Philox's high counter word
N, H, W = 2, 24, 24
M = (160, 120)                      # surface-solve points per garment
V = (2300, 2600)                    # MC vertices: above S = 4096 // 2, so the draws thin
NAMES = ("upper", "bottom")
CONF = {"grad_weight": 1.0, "offset_weight": 0.0, "def_regu": {"weight": 0.1, "c": 0.5}, "color_weight": 0.5,
        "normal_weight": 0.1, "weighted_normal": True}
RATIO = {"sdfRatio": 0.8, "deformerRatio": 0.6, "renderRatio": 0.9}
GRAD_STRIDE = 257


class Conf:
    """The pyhocon calls the method makes: get_float('a.b'), get_bool and `'a' in conf`."""

    def __init__(self, d):
        self.d = d

    def _get(self, key):
        v = self.d
        for k in key.split("."):
            v = v[k]
        return v

    def get_float(self, key):
        return float(self._get(key))

    def get_bool(self, key):
        return bool(self._get(key))

    def __contains__(self, key):
        return key in self.d


def inputs():
    """The call's arrays, seeded: per garment init points, vertices, check, batch, row, col, rays; gtCs, normals,
    camera R, poses, trans and the N x 128 conditions of the body and the two garments."""
    rng = np.random.default_rng(1083)

    def unit(n):
        x = rng.standard_normal((n, 3))
        return x / np.linalg.norm(x, axis=1, keepdims=True)

    d = {}
    for g in range(2):
        d[f"P_{g}"] = (unit(M[g]) * 0.45 + rng.standard_normal((M[g], 3)) * 0.02).astype(np.float32)
        d[f"V_{g}"] = (unit(V[g]) * 0.45).astype(np.float32)
        d[f"check_{g}"] = rng.uniform(size=M[g]) < 0.8
        d[f"batch_{g}"] = rng.integers(0, N, M[g])
        d[f"row_{g}"] = rng.integers(0, H, M[g])
        d[f"col_{g}"] = rng.integers(0, W, M[g])
        d[f"rays_{g}"] = unit(M[g]).astype(np.float32)
    d["gtCs"] = rng.uniform(size=(N, H, W, 3)).astype(np.float32)
    nrm = rng.standard_normal((N, H, W, 3))
    nrm /= np.linalg.norm(nrm, axis=-1, keepdims=True)
    nrm[:, : H // 4] = 0.                                            # background rows: invalid normals
    d["normal"] = nrm.astype(np.float32)
    q = np.array([0.97, 0.05, -0.2, 0.1])
    q /= np.linalg.norm(q)
    w, x, y, z = q
    d["R"] = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                       [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                       [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], np.float32)
    poses, trans = synth.poses_trans(N, seed=11)
    d["poses"], d["trans"] = poses.numpy(), trans.numpy()
    d["conds"] = (rng.standard_normal((3, N, 128)) * 0.1).astype(np.float32)
    return d


def stream(d):
    """The oracle's draws in the reference's call order: the uniforms of torch.rand and the sample_points answers."""
    rands, samples, base = [], [], 0
    for g in range(2):
        Mg, Vg = M[g], V[g]
        C = Mg + Vg
        for lane in (lpo.E_DRAW, lpo.D_DRAW):
            rands.append(lpo.unit24(lpo.words(SEED, lpo.counters(OFFSET, base, lane, C, Vg))[:, 0]))
        keep_e = lpo.draw(SEED, OFFSET, base, lpo.E_DRAW, C, Vg, 2048)
        keep_d = lpo.draw(SEED, OFFSET, base, lpo.D_DRAW, C, Vg, 2048)
        nE, nD = Mg + len(keep_e), Mg + len(keep_d)
        z_e = lpo.normals(SEED, lpo.counters(OFFSET, base, lpo.E_LOCAL, C, nE))[0]
        glob = lpo.global_points(SEED, lpo.counters(OFFSET, base, lpo.E_GLOBAL, C, nE // 6))
        z_d = lpo.normals(SEED, lpo.counters(OFFSET, base, lpo.D_LOCAL, C, nD))[0]
        samples += [(z_e, glob), (z_d, None)]
        base += lpo.LANES * C
    return rands, samples


class TorchWithRand(types.ModuleType):
    """The torch module with `rand(n)` answered from a queue of prepared float32 uniforms."""

    def __init__(self, draws):
        super().__init__("torch")
        self.draws = list(draws)

    def __getattr__(self, name):
        return getattr(torch, name)

    def rand(self, n):
        u = self.draws.pop(0)
        assert len(u) == n, (len(u), n)
        return torch.from_numpy(u.copy())


class UtilsWithSamples(types.ModuleType):
    """The reference's `utils` package with `sample_points` answered from the oracle; records each call's input."""

    def __init__(self, utils, samples):
        super().__init__("utils")
        self.utils, self.samples, self.seen = utils, list(samples), []

    def __getattr__(self, name):
        return getattr(self.utils, name)

    def sample_points(self, x, global_sigma, local_sigma, ratio=6):
        z, glob = self.samples.pop(0)
        assert (global_sigma, local_sigma) == (1.8, 0.01) and len(z) == x.shape[0] and (ratio > 0) == (glob is not None)
        self.seen.append(x.detach().clone())
        local = x + torch.from_numpy(z).to(x.dtype) * 0.01
        return torch.cat([local, torch.from_numpy(glob).to(x.dtype)]) if ratio > 0 else local


def scatter_mean(src, index, reduce="mean", dim_size=None):
    assert reduce == "mean"
    s = torch.zeros(dim_size, dtype=src.dtype).index_add_(0, index, src)
    n = torch.zeros(dim_size, dtype=src.dtype).index_add_(0, index, torch.ones_like(src))
    return s / n.clamp_min(1)


def networks(ns):
    import make_golden as mg
    sdf, deformer = mg.surface_scene(ns.network, ns.Deformer)
    torch.manual_seed(2)
    rn = ns.RenderNet.RenderingNetwork_view_norm(256, d_in=9, d_out=3, dims=[512] * 4, mode="idr", weight_norm=True,
                                                 multires_v=4, multires_n=0)
    testing.perturb_module(rn, 303)
    return sdf, deformer, rn


def run(OGN, ns, d, dt):
    sdf, deformer, rn = (m.to(dt) for m in networks(ns))
    t = lambda k: torch.from_numpy(d[k])  # noqa: E731
    poses, trans = t("poses").to(dt).requires_grad_(True), t("trans").to(dt).requires_grad_(True)
    conds = [t("conds")[k].to(dt).requires_grad_(True) for k in range(3)]
    rendcond = torch.zeros((N, 1), dtype=dt)
    info = {f"{NAMES[g]}_rayInfo": (M[g], int(d[f"check_{g}"].sum())) for g in range(2)}
    self = types.SimpleNamespace(
        garment_size=2, garment_names=list(NAMES), garment_nets=[sdf, sdf],
        garment_vs=[t(f"V_{g}").to(dt) for g in range(2)], deformer=deformer, netRender=rn, conf=Conf(CONF), info=info,
        get_grad_parameters=lambda frame_ids, device: (conds, poses, trans, rendcond))
    cameras = types.SimpleNamespace(R=t("R").to(dt).view(1, 3, 3).expand(N, 3, 3))
    rands, samples = stream(d)
    old = OGN.torch, OGN.utils, OGN.scatter
    OGN.torch, OGN.utils, OGN.scatter = TorchWithRand(rands), UtilsWithSamples(ns.utils, samples), scatter_mean
    prev = torch.get_default_dtype()
    torch.set_default_dtype(dt)
    try:
        loss = OGN.OptimGarmentNetwork.surface_render_loss(
            self, {"normal": t("normal").to(dt)}, N, cameras, torch.arange(N), RATIO,
            [t(f"check_{g}") for g in range(2)], t("gtCs").to(dt), [t(f"P_{g}").to(dt) for g in range(2)],
            [t(f"row_{g}") for g in range(2)], [t(f"col_{g}") for g in range(2)], [t(f"batch_{g}") for g in range(2)],
            [t(f"rays_{g}").to(dt) for g in range(2)], "cpu")
        seen = OGN.utils.seen
        assert not OGN.torch.draws and not OGN.utils.samples
    finally:
        torch.set_default_dtype(prev)
        OGN.torch, OGN.utils, OGN.scatter = old
    loss.backward()
    tag = "f32" if dt == torch.float32 else "f64"
    out = {f"{tag}/loss": np.array(float(loss.detach()))}
    for k, v in self.info.items():
        if not k.endswith("rayInfo"):
            out[f"{tag}/info/{k}"] = np.array(float(v))
    for g in range(2):
        out[f"{tag}/B_E_{g}"] = seen[2 * g].numpy()
        out[f"{tag}/B_D_{g}"] = seen[2 * g + 1].numpy()
        out[f"{tag}/TmpPs_{g}"] = self.TmpPs[g].detach().numpy()
        out[f"{tag}/rays_c_{g}"] = self.rays[g].detach().numpy()
        for k, src in (("batch", self.batch_inds), ("row", self.row_inds), ("col", self.col_inds)):
            out[f"{tag}/{k}_c_{g}"] = src[g].numpy()
    mods = {"sdf": sdf, "translator": deformer.defs[0], "render": rn}
    for mname, m in mods.items():
        for pname, p in sorted(m.named_parameters()):
            if p.grad is not None:
                out[f"{tag}/grad/{mname}.{pname}"] = p.grad.detach().reshape(-1)[::GRAD_STRIDE].numpy()
    for k, x in (("poses", poses), ("trans", trans), ("cond0", conds[0]), ("cond1", conds[1]), ("cond2", conds[2])):
        if x.grad is not None:
            out[f"{tag}/grad/{k}"] = x.grad.detach().numpy()
    return out


def generate():
    ns = refload.load()
    OGN = importlib.import_module("engineer.networks.OptimGarmentNetwork")
    d = inputs()
    out = {f"in/{k}": v for k, v in d.items()}
    out["seed"] = np.array(SEED, dtype=np.uint64)
    out["offset"] = np.array(OFFSET, dtype=np.uint64)
    for dt in (torch.float32, torch.float64):
        out.update(run(OGN, ns, d, dt))
    return out


def main():
    out = generate()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out), "arrays;", {k: float(v) for k, v in out.items() if k.endswith("/loss")})


if __name__ == "__main__":
    main()
