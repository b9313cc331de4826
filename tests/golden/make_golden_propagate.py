"""Writes tests/golden/propagate_ref.npz: the reference's OWN `propagateTmpPsGrad` of OptimGarmentNetwork
(engineer/networks/OptimGarmentNetwork.py:2159-2313) and of OptimGarmentNetwork_LargePose
(OptimGarmentNetwork_Large_Pose.py:327-473), unmodified, run on the CPU in float32 and float64 with
  * a lightweight `self` built from tests/propagate_scene.py's `inputs`: two garments (300 and 240 rows, N = 3)
    sharing the reference's `ImplicitNetwork` and `CompositeDeformer(MLPTranslator, LBSkinner)` of
    tests/golden/make_golden.py's surface scene; a learnable camera (focal length, principal point and T require
    grad, as female-3-casual.conf's `opt_camera` sets them); poses, translations and garment conditions that require
    grad; seeded TmpPs.grad; for the Large-Pose class the garment net frozen;
  * `RectifiedPerspectiveCameras` rebound to a subclass of the reference's own class (model/CameraMine.py) that only
    stores its parameters, so `view_rays` and `cam_pos` are the reference's own;
  * `Fast3x3Minv` answering with oracle/implicit_grad_oracle.py's rule (the extension is CUDA-only);
  * GRAZING rows per garment: the first rows get v = J t / |J t| with t perpendicular to grad f (in float64 on these
    networks), expressed as the sub-pixel (col, row) whose view ray is v, so b^T b is singular.  Every other row's
    float64 |det b^T b| is asserted to lie more than a factor of 10 away from 1e-4.
  * in float64, torch's default dtype set to float64 for the call, and `view_rays` given the pixel coordinates in
    float64 (the method's `.float()` would mix float32 rays with the float64 rotation; the coordinates are float32
    values, so nothing is rounded).
Tensor hooks record what the method feeds its backward passes: -r0 (the SDF cotangent), r[1:4] (-[v]x) (the deformer
cotangent), the ray and camera-centre gradients; grad f, J, v, d and c are recomputed by the same expressions.
Stored per class and dtype: those, FastMinv's ok flags, invInfo, and the gradients of the SDF and translator
parameters (weights: every 257th entry, flattened; biases whole), focal length, principal point, T, poses, translations and the garment
conditions.  Needs the reference source tree (oracle/refload.py).

    python tests/golden/make_golden_propagate.py
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
sys.path.insert(0, os.path.dirname(HERE))

from oracle import implicit_grad_oracle as igo, refload  # noqa: E402

OUT = os.path.join(HERE, "propagate_ref.npz")
GRAZING = 5
GRAD_STRIDE = 257
RATIO = {"sdfRatio": 0.8, "deformerRatio": 0.6, "renderRatio": 0.9}


def networks(ns, dt):
    import make_golden as mg
    sdf, deformer = mg.surface_scene(ns.network, ns.Deformer)
    return sdf.to(dt), deformer.to(dt)


def grad_f_and_jac(sdf, deformer, p, cond, poses, trans, batch, name):
    """grad f [n,3] and J [n,3,3] (row i = gradient of D_i) by the method's own expressions, and D(p)."""
    p = p.detach().clone().requires_grad_(True)
    f = sdf(p, RATIO)
    gf = torch.autograd.grad(f, p, torch.ones_like(f))[0]
    d = deformer(p, [cond, [poses, trans]], batch, ratio=RATIO, offset_type=name)
    rows = [torch.autograd.grad(d[..., i], p, torch.ones_like(d[..., 0]), retain_graph=True)[0] for i in range(3)]
    return gf.detach(), torch.stack(rows, 1).detach(), d.detach()


def add_grazing(ns, d):
    """Make the first GRAZING rows of each garment singular (see the module docstring); returns d."""
    sdf, deformer = networks(ns, torch.float64)
    R = d["R"].astype(np.float64)
    for g in range(int(d["G"])):
        p = torch.from_numpy(d[f"P_{g}"][:GRAZING].astype(np.float64))
        b = torch.from_numpy(d[f"batch_{g}"][:GRAZING])
        cond = torch.from_numpy(d["conds"][g + 1].astype(np.float64))
        gf, J, _ = grad_f_and_jac(sdf, deformer, p, cond, torch.from_numpy(d["poses"]).double(),
                                  torch.from_numpy(d["trans"]).double(), b, "x")
        gf, J = gf.numpy(), J.numpy()
        e = np.eye(3)[np.argmin(np.abs(gf), axis=1)]
        t = np.cross(gf, e)
        v = np.einsum("nij,nj->ni", J, t)
        v /= np.linalg.norm(v, axis=1, keepdims=True)
        u = v @ R                                       # camera-frame ray R^T v
        v = np.where(u[:, 2:3] < 0, -v, v)
        u = v @ R
        fx, fy = d["focal"].astype(np.float64)
        px, py = d["pp"].astype(np.float64)
        d[f"col_{g}"][:GRAZING] = (px - fx * u[:, 0] / u[:, 2]).astype(np.float32)
        d[f"row_{g}"][:GRAZING] = (py - fy * u[:, 1] / u[:, 2]).astype(np.float32)
        # every other row: redraw its pixel until |det| > 1e-3 (a factor of 10 above 1e-4)
        gf, J, _ = grad_f_and_jac(sdf, deformer, torch.from_numpy(d[f"P_{g}"].astype(np.float64)),
                                  cond, torch.from_numpy(d["poses"]).double(), torch.from_numpy(d["trans"]).double(),
                                  torch.from_numpy(d[f"batch_{g}"]), "x")
        rng = np.random.default_rng(2313 + g)
        for _ in range(200):
            cam = np.stack([(px - d[f"col_{g}"]) / fx, (py - d[f"row_{g}"]) / fy, np.ones(len(gf))], 1)
            v = (cam / np.linalg.norm(cam, axis=1, keepdims=True)) @ R.T
            det = np.abs(np.linalg.det(igo.btb(gf.numpy(), J.numpy(), v)[1]))
            bad = det <= 1e-3
            bad[:GRAZING] = False
            if not bad.any():
                break
            d[f"col_{g}"][bad] = rng.integers(0, int(d["W"]), int(bad.sum()))
            d[f"row_{g}"][bad] = rng.integers(0, int(d["H"]), int(bad.sum()))
    return d


class Hooked:
    """A module stand-in recording, for every call, the output and the gradients its backward passes deliver."""

    def __init__(self, mod):
        self.mod, self.calls = mod, []

    def __call__(self, *a, **k):
        out = self.mod(*a, **k)
        rec = {"out": out.detach().clone(), "grads": []}
        self.calls.append(rec)
        if out.requires_grad:
            out.register_hook(lambda gr: rec["grads"].append(gr.detach().clone()))
        return out

    def parameters(self):
        return self.mod.parameters()

    def __getattr__(self, name):
        return getattr(self.mod, name)


def run(mod, cls, ns, d, dt, large_pose):
    import propagate_scene as ps
    sdf, deformer = networks(ns, dt)
    if large_pose:
        sdf.requires_grad_(False)
    G, N, H, W = int(d["G"]), int(d["N"]), int(d["H"]), int(d["W"])
    t = lambda k: torch.from_numpy(np.ascontiguousarray(d[k]))  # noqa: E731
    focal, pp, R, T = (t(k).to(dt) for k in ("focal", "pp", "R", "T"))
    focal.requires_grad_(True), pp.requires_grad_(True), T.requires_grad_(True)
    poses, trans = t("poses").to(dt).requires_grad_(True), t("trans").to(dt).requires_grad_(True)
    conds = [t("conds")[k].to(dt).clone().requires_grad_(k > 0) for k in range(G + 1)]
    CameraMine = importlib.import_module("model.CameraMine")
    cam_rec = {"v": [], "c": []}

    class Cam(CameraMine.RectifiedPerspectiveCameras):
        def __init__(self, focal_length, principal_point, R, T, image_size=None):
            self.focal_length, self.principal_point, self.R, self.T = focal_length, principal_point, R, T

        def to(self, device):
            return self

        def view_rays(self, ps_, cam_id=0):
            out = super().view_rays(ps_.to(dt), cam_id)
            rec = {"out": out.detach().clone(), "grads": []}
            cam_rec["v"].append(rec)
            out.register_hook(lambda gr: rec["grads"].append(gr.detach().clone()))
            return out

        def cam_pos(self, cam_id=0):
            out = super().cam_pos(cam_id)
            rec = {"out": out.detach().clone(), "grads": []}
            cam_rec["c"].append(rec)
            out.register_hook(lambda gr: rec["grads"].append(gr.detach().clone()))
            return out

    def get_camera_parameters(n, device):
        return (focal.view(1, 2).expand(n, 2), pp.view(1, 2).expand(n, 2), R.view(1, 3, 3).expand(n, 3, 3),
                T.view(1, 3).expand(n, 3), H, W)

    minv_ok = []

    def fast3x3minv(m):
        inv, ok = igo.minv_rule(m.detach().numpy())
        minv_ok.append(ok)
        return torch.from_numpy(inv), torch.from_numpy(ok)

    hnet, hdef = Hooked(sdf), Hooked(deformer)
    self = types.SimpleNamespace(
        garment_size=G, garment_names=list(ps.NAMES[:G]), garment_nets=[hnet] * G, deformer=hdef,
        dataset=types.SimpleNamespace(get_camera_parameters=get_camera_parameters),
        maskRender=types.SimpleNamespace(rasterizer=types.SimpleNamespace(cameras=None)), info={},
        get_grad_parameters=lambda frame_ids, device: (conds, poses, trans, None))
    cams = Cam(*get_camera_parameters(N, "cpu")[:4])
    self.TmpPs, self.rays, self.batch_inds, self.row_inds, self.col_inds = ([None] * G for _ in range(5))
    for g in range(G):
        p = t(f"P_{g}").to(dt).clone().requires_grad_(True)
        p.grad = t(f"gl_{g}").to(dt).clone()
        self.TmpPs[g] = p
        self.col_inds[g], self.row_inds[g], self.batch_inds[g] = t(f"col_{g}"), t(f"row_{g}"), t(f"batch_{g}")
        self.rays[g] = cams.view_rays(torch.stack([self.col_inds[g], self.row_inds[g], torch.ones_like(self.col_inds[g])], 1).float())
    cam_rec["v"].clear()
    gl0 = [p.grad.clone() for p in self.TmpPs]
    old = mod.Fast3x3Minv, mod.RectifiedPerspectiveCameras
    mod.Fast3x3Minv, mod.RectifiedPerspectiveCameras = fast3x3minv, Cam
    prev = torch.get_default_dtype()
    torch.set_default_dtype(dt)
    try:
        cls.propagateTmpPsGrad(self, torch.arange(N), RATIO)
    finally:
        torch.set_default_dtype(prev)
        mod.Fast3x3Minv, mod.RectifiedPerspectiveCameras = old
    for g in range(G):
        assert torch.equal(self.TmpPs[g].grad, gl0[g])
    tag = ("large" if large_pose else "base") + ("/f32" if dt == torch.float32 else "/f64")
    out = {}
    for g in range(G):
        name = self.garment_names[g]
        out[f"{tag}/invInfo_{g}"] = np.array(self.info[f"{name}_invInfo"], np.int64)
        out[f"{tag}/ok_{g}"] = minv_ok[g]
        gf, J, _ = grad_f_and_jac(sdf, deformer, self.TmpPs[g], conds[g + 1].detach(), poses.detach(),
                                  trans.detach(), self.batch_inds[g], name)
        out[f"{tag}/gf_{g}"], out[f"{tag}/J_{g}"] = gf.numpy(), J.numpy()
        vjp_call = hdef.calls[2 * g + 1]
        out[f"{tag}/d_{g}"] = vjp_call["out"].numpy()
        out[f"{tag}/def_vec_{g}"] = vjp_call["grads"][0].numpy()
        out[f"{tag}/v_{g}"] = cam_rec["v"][g]["out"].numpy()
        out[f"{tag}/ray_grad_{g}"] = cam_rec["v"][g]["grads"][0].numpy()
        out[f"{tag}/c_{g}"] = cam_rec["c"][g]["out"].numpy()
        out[f"{tag}/cam_grad_{g}"] = cam_rec["c"][g]["grads"][0].numpy()
        if not large_pose:
            out[f"{tag}/sdf_coef_{g}"] = hnet.calls[2 * g + 1]["grads"][0].reshape(-1).numpy()
    mods = {"sdf": sdf, "translator": deformer.defs[0]}
    for mname, m in mods.items():
        for pname, p in sorted(m.named_parameters()):
            if p.grad is not None:
                step = GRAD_STRIDE if p.dim() > 1 else 1
                out[f"{tag}/grad/{mname}.{pname}"] = p.grad.detach().reshape(-1)[::step].numpy()
    leaves = {"focal": focal, "pp": pp, "T": T, "poses": poses, "trans": trans}
    leaves.update({f"cond{k}": conds[k] for k in range(1, G + 1)})
    for k, x in leaves.items():
        if x.grad is not None:
            out[f"{tag}/grad/{k}"] = x.grad.detach().numpy()
    return out


def check_dets(d, out):
    """Every non-grazing row's float64 |det| lies more than a factor of 10 from 1e-4; the grazing rows are singular."""
    for g in range(int(d["G"])):
        _, m = igo.btb(out[f"base/f64/gf_{g}"], out[f"base/f64/J_{g}"], out[f"base/f64/v_{g}"])
        det = np.abs(np.linalg.det(m))
        assert (det[:GRAZING] < 1e-4 / 10).all(), det[:GRAZING]
        rest = det[GRAZING:]
        assert ((rest > 1e-4 * 10) | (rest < 1e-4 / 10)).all(), rest.min()


def generate():
    import propagate_scene as ps
    ns = refload.load()
    OGN = importlib.import_module("engineer.networks.OptimGarmentNetwork")
    OGNL = importlib.import_module("engineer.networks.OptimGarmentNetwork_Large_Pose")
    d = add_grazing(ns, ps.inputs())
    out = {f"in/{k}": v for k, v in d.items()}
    for large, mod, cls in ((False, OGN, OGN.OptimGarmentNetwork), (True, OGNL, OGNL.OptimGarmentNetwork_LargePose)):
        for dt in (torch.float32, torch.float64):
            out.update(run(mod, cls, ns, d, dt, large))
    check_dets(d, out)
    return out


def main():
    out = generate()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out), "arrays;", {k: v.tolist() for k, v in out.items() if "invInfo" in k})


if __name__ == "__main__":
    main()
