"""Writes tests/golden/mask_loss_ref.npz: the reference's OWN `OptimGarmentNetwork.mask_loss`
(engineer/networks/OptimGarmentNetwork.py:841-981, with compute_garment_pc_loss :621-667 and find_surface_ps
:742-783), unmodified, run on the CPU in float32 and float64 with
  * a lightweight `self`: conf with the coarse `pc_weight` of configs/people_snapshot/female-3-casual.conf (weight 60,
    laplacian / edge / norm weights negative, def_consistent 0.6 / c 0.01, curve_aware 60), two garments (an
    ellipsoid and an open tube) sharing the reference's `ImplicitNetwork` and the `CompositeDeformer(MLPTranslator,
    LBSkinner)` of tests/golden/make_golden.py's surface scene, the garment optimiser SGD(lr 0.05, momentum 0.9) and
    `curve_aware_loss` returning 0 (it has its own fixture);
  * `pcRender` backed by oracle/points_oracle.py (the selection of the projected points, then its differentiable
    composite) and `maskRender` by oracle/raster_oracle.py, both through the camera of `camera()`;
  * `Meshes` and `Pointclouds` stand-ins in the module namespace;
  * in float64, torch's default dtype set to float64 for the call, so the constants the method builds match.
The scene is checked so that no pixel centre lies within 1e-4 r^2 of a disc boundary and no two depths that decide a
pixel's order are within 1e-5 relative, so float32 and float64 select the same points.
Needs the reference source tree (oracle/refload.py).

Stored: the inputs, the radius, per precision the silhouettes, the dilated masks, the loss terms and every info term,
the garment vertices after the optimiser step and the gradients to poses, trans, the conditions and the translator's
parameters (every 257th entry of each, flattened).

    python tests/golden/make_golden_mask_loss.py
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

from oracle import points_oracle as po, raster_oracle as ro, refload, zbuf_oracle as zo  # noqa: E402
from recmv_b200 import synth  # noqa: E402

OUT = os.path.join(HERE, "mask_loss_ref.npz")
N, H, W = 2, 40, 44
RADIUS = 0.12                       # NDC; int(round(0.12 / 2 * 40 / 1.2)) = 2 pixels of dilation
K = 32
NAMES = ("upper", "bottom")
PC_WEIGHT = {"weight": 60.0, "laplacian_weight": -10.0, "edge_weight": -10.0, "norm_weight": -0.001,
             "def_consistent": {"weight": 0.6, "c": 0.01}, "curve_aware_weight": 60.0}
RATIO = {"sdfRatio": 0.8, "deformerRatio": 0.6, "renderRatio": 0.9}
SHRINK = 0.01
GRAD_STRIDE = 257
MARGIN, ZTOL = 1e-4, 1e-5


class Conf:
    """The pyhocon calls the method makes: get_float('a.b') and `'a.b' in conf`."""

    def __init__(self, d):
        self.d = d

    def _get(self, key):
        v = self.d
        for k in key.split("."):
            v = v[k]
        return v

    def get_float(self, key):
        return float(self._get(key))

    def __contains__(self, key):
        try:
            self._get(key)
            return True
        except (KeyError, TypeError):
            return False


CONF = {"pc_weight": PC_WEIGHT}


def camera():
    """[N,16] float64 camera rows {fx, fy, px, py, R, T}: a pinhole 3 units in front of the scene, turning by frame."""
    rows = []
    for n in range(N):
        a = 0.15 * n - 0.05
        R = np.array([[np.cos(a), 0, -np.sin(a)], [0, 1, 0], [np.sin(a), 0, np.cos(a)]])
        rows.append(np.concatenate([[52.0, 52.0, W / 2 + 0.35, H / 2 - 0.4], R.reshape(-1), [0.02, 0.05, 3.0]]))
    return np.asarray(rows)


def inputs():
    """Garment templates, ground-truth masks, poses, trans and the N x 128 conditions of the body and two garments."""
    rng = np.random.default_rng(841)
    up_v, up_f = zo.uv_sphere(10, 8, (0.30, 0.26, 0.22), (0.0, 0.22, 0.0))
    lo_v, lo_f = zo.tube(10, 5, 0.24, -0.55, -0.08)
    d = {"V_0": (up_v + rng.normal(0, 0.004, up_v.shape)).astype(np.float32), "F_0": up_f,
         "V_1": (lo_v + rng.normal(0, 0.004, lo_v.shape)).astype(np.float32), "F_1": lo_f}
    yy, xx = np.mgrid[0:H, 0:W]
    for g, (cy, cx, ry, rx) in enumerate(((14, 22, 8, 9), (28, 21, 9, 7))):
        ell = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1
        gt = np.stack([np.roll(ell, n, axis=1) for n in range(N)]).astype(np.float32)
        gt[:, 0, :3] = 1.0                                           # touches the border
        d[f"gt_{g}"] = gt
    poses, trans = synth.poses_trans(N, seed=11)
    d["poses"], d["trans"] = (poses * 0.3).numpy(), (trans * 0.1).numpy()
    d["conds"] = (rng.standard_normal((3, N, 128)) * 0.1).astype(np.float32)
    d["cam"] = camera()
    return d


def project_torch(pts, cam):
    """points_oracle.project as a torch graph of the world points [N,P,3] (any dtype)."""
    c = torch.as_tensor(cam, dtype=pts.dtype)
    v = pts @ c[:, 4:13].reshape(-1, 3, 3) + c[:, None, 13:16]
    sx = c[:, None, 2] - c[:, None, 0] * v[..., 0] / v[..., 2]
    sy = c[:, None, 3] - c[:, None, 1] * v[..., 1] / v[..., 2]
    return torch.stack([1 - (2 * sx + 1) / W, 1 - (2 * sy + 1) / H, v[..., 2]], -1)


class Pointclouds:
    def __init__(self, points, features):
        self._p, self._f = list(points), list(features)

    def points_list(self):
        return self._p


class OraclePointRender:
    """`pcRender` (PointsRendererWithFrags_Split) on points_oracle: select on the detached projection, composite as a
    torch graph of it.  Records each call's selection."""

    def __init__(self, cam):
        self.cam = cam
        self.rasterizer = types.SimpleNamespace(
            cameras=None, raster_settings=types.SimpleNamespace(image_size=(H, W), radius=RADIUS, points_per_pixel=K))
        self.seen = []

    def __call__(self, clouds, split_size, all_size):
        pts = torch.stack(clouds.points_list())
        assert pts.shape[1] == all_size
        ndc = project_torch(pts, self.cam)
        sel = po.select(ndc.detach().double().numpy(), H, W, RADIUS, K)
        self.seen.append(po.project(pts.detach().double().numpy(), self.cam, H, W))
        img = po.composite_torch(sel, ndc, RADIUS, split=split_size, G=2)
        return [img[0][..., None], img[1][..., None]], None


class OracleMaskRender:
    """`maskRender` on raster_oracle: fragments pix_to_face, zbuf and bary_coords [N,H,W,1(,3)]."""

    def __init__(self, cam):
        self.cam = cam

    def __call__(self, meshes):
        v = torch.stack(meshes.verts_list()).detach().double().numpy()
        fr = ro.rasterize(v, meshes.faces_list()[0].numpy(), self.cam, H, W)
        dt = torch.get_default_dtype()
        frags = types.SimpleNamespace(pix_to_face=torch.tensor(fr["pix_to_face"])[..., None],
                                      zbuf=torch.tensor(fr["zbuf"], dtype=dt)[..., None],
                                      bary_coords=torch.tensor(fr["bary"], dtype=dt)[..., None, :])
        return None, frags


def networks(ns):
    import make_golden as mg
    return mg.surface_scene(ns.network, ns.Deformer)


def run(OGN, ns, d, dt):
    sdf, deformer = (m.to(dt) for m in networks(ns))
    t = lambda k: torch.from_numpy(d[k].copy())  # noqa: E731  (the optimiser steps the vertices in place)
    poses, trans = t("poses").to(dt).requires_grad_(True), t("trans").to(dt).requires_grad_(True)
    conds = [t("conds")[k].to(dt).requires_grad_(True) for k in range(3)]
    vs = [t(f"V_{g}").to(dt).requires_grad_(True) for g in range(2)]
    pc = OraclePointRender(d["cam"])
    self = types.SimpleNamespace(
        garment_size=2, garment_names=list(NAMES), garment_nets=[sdf, sdf], garment_vs=vs,
        garment_fs=[t(f"F_{g}") for g in range(2)], body_vs=torch.zeros((5, 3), dtype=dt), deformer=deformer,
        conf=Conf(CONF), info={}, sdfShrinkRadius=SHRINK, pcRender=pc, maskRender=OracleMaskRender(d["cam"]),
        garment_optimizer=torch.optim.SGD(vs, lr=0.05, momentum=0.9), curve_aware_loss=lambda ratio: 0.,
        get_grad_parameters=lambda frame_ids, device: (conds, poses, trans, None))
    for name in ("find_surface_ps", "compute_garment_pc_loss"):
        setattr(self, name, types.MethodType(getattr(OGN.OptimGarmentNetwork, name), self))
    old = OGN.Meshes, OGN.Pointclouds
    OGN.Meshes, OGN.Pointclouds = zo.Meshes, Pointclouds
    prev = torch.get_default_dtype()
    torch.set_default_dtype(dt)
    try:
        meshes, masks, mgt, pc_sdf_loss, _ = OGN.OptimGarmentNetwork.mask_loss(
            self, N, H, W, torch.arange(N), RATIO, [t(f"gt_{g}").to(dt) for g in range(2)], "cpu")
    finally:
        torch.set_default_dtype(prev)
        OGN.Meshes, OGN.Pointclouds = old
    tag = "f32" if dt == torch.float32 else "f64"
    out = {f"{tag}/pc_sdf_loss": np.array(float(pc_sdf_loss.detach()))}
    for k, v in self.info["pc_loss"].items():
        out[f"{tag}/info/{k}"] = np.array(float(v))
    for k, v in self.info.items():
        if k != "pc_loss":
            out[f"{tag}/info/{k}"] = np.array(float(v))
    for g in range(2):
        out[f"{tag}/masks_{g}"] = masks[g][..., -1].detach().numpy()
        out[f"{tag}/mgt_{g}"] = mgt[g].detach().numpy()
        out[f"{tag}/def_verts_{g}"] = meshes[g].verts_padded().detach().numpy()
        out[f"{tag}/verts_after_{g}"] = vs[g].detach().numpy()
    for pname, p in sorted(deformer.defs[0].named_parameters()):
        if p.grad is not None:
            out[f"{tag}/grad/translator.{pname}"] = p.grad.detach().reshape(-1)[::GRAD_STRIDE].numpy()
    for k, x in (("poses", poses), ("trans", trans), ("cond1", conds[1]), ("cond2", conds[2])):
        out[f"{tag}/grad/{k}"] = x.grad.detach().numpy()
    return out, pc.seen[0]


def check_margins(ndc):
    """No pixel centre within MARGIN r^2 of a disc boundary, no deciding depth pair within ZTOL, and K not reached."""
    sel = po.select(ndc, H, W, RADIUS, K, margin=MARGIN, ztol=ZTOL)
    assert not sel["ambiguous"].any(), int(sel["ambiguous"].sum())
    assert sel["count"].max() < K and sel["skipped"] == 0
    return sel


def generate():
    ns = refload.load()
    OGN = importlib.import_module("engineer.networks.OptimGarmentNetwork")
    d = inputs()
    out = {f"in/{k}": v for k, v in d.items()}
    out["radius"] = np.array(int(np.round(RADIUS / 2. * float(min(H, W)) / 1.2)))
    out["K"] = np.array(K)
    out["ndc_radius"] = np.array(RADIUS)
    for dt in (torch.float32, torch.float64):
        o, ndc = run(OGN, ns, d, dt)
        out.update(o)
        if dt == torch.float64:
            check_margins(ndc)
    out["margin"] = np.array(MARGIN)
    return out


def main():
    out = generate()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out), "arrays;", {k: float(v) for k, v in out.items() if "/info/" in k})


if __name__ == "__main__":
    main()
