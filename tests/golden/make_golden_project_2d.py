"""Writes tests/golden/project_2d_ref.npz: the reference's OWN `project_2d_loss` of both garment classes
(engineer/networks/OptimGarmentNetwork.py:1772-1883 with deform_feature_line :1516-1602, compute_fl_proj_loss
:1604-1712 and fl_visible_by_body_zbuff :1374-1465; OptimGarmentNetwork_Large_Pose.py:139-239), unmodified, run on
the CPU in float32 and float64 with
  * a lightweight `self`: the outfit of tests/project_2d_scene.py (`long_sleeve_upper` with 4 curves, `long_pants` with
    2, S = 200 points each, ellipsoid / tube garments around an ellipsoid body), the reference's `ImplicitNetwork` and
    `CompositeDeformer(MLPTranslator, LBSkinner)` of tests/golden/make_golden.py's surface scene, the reference's
    `Intersect_Free_Curve` built with object.__new__ + `initialize_parameters` (identity canonical-SMPL map, so
    trimesh is not needed) and `fl_optimizer` AdamW(lr=1e-4) over its scale and nx_scale;
  * `chamfer_distance` of engineer.core.fl_optimizer rebound to oracle/knn_oracle.chamfer_f64, `maskRender` on
    oracle/raster_oracle.py and the camera of oracle/zbuf_oracle.py (CameraMine's `transform_points_screen` through
    pytorch3d's composed world-to-NDC matrix, built for the same (W, H) as the method's image size);
  * in float64, torch's default dtype set to float64 for the call.
N = 1 and N = 3 on a 120 x 96 image.  The curve buffers are made once in float64 and rounded to float32, so every run
starts from the same values.  The scene is checked so that every body check lies more than 1e-4 from its threshold and
every nearest neighbour of the chamfer terms (both directions) is more than 1e-3 relative closer than the second best,
so float32, float64 and the drop-in's own z-buffer select the same points; annotation points that break the margin are
moved and the run repeated.

Stored per class (base, large) in float64: the info values, the returned screen points, visible masks and annotations
(the label masks are checked to be fl_masks' columns), the body checks, the curve-parameter gradients, the post-step
scale / nx_scale, the deformer offsets of every curve, and the gradients of poses, trans, the garment conditions, the
translator and the SDF (every 257th entry of each weight); in float32 the info values and the curve gradients.

    python tests/golden/make_golden_project_2d.py
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

from oracle import knn_oracle, refload, zbuf_oracle as zo  # noqa: E402
from recmv_b200 import synth  # noqa: E402

import project_2d_scene as ps  # noqa: E402

OUT = os.path.join(HERE, "project_2d_ref.npz")
H, W, S, M = 96, 120, 200, 160
FRAMES = (1, 3)
GRAD_STRIDE = 257
BODY_MARGIN, NN_MARGIN = 1e-4, 1e-3


def inputs(N, seed):
    """Every input of one case as float32 / int64 / bool numpy arrays (curve buffers from the reference's own
    initialize_parameters in float64, rounded)."""
    rng = np.random.default_rng(seed)
    d = {}
    verts = np.stack([ps.ring(*ps.RINGS[n], S, 0.3 * i) for i, n in enumerate(ps.FL_NAMES)])
    d["curve_verts"] = verts.astype(np.float32)
    scale = 1.0 + rng.normal(0, 0.05, (6, S, 1))
    scale[0, 5:9] = 0.
    scale[3, 40:43] = -0.1
    d["scale"], d["nx_scale"] = scale.astype(np.float32), rng.normal(0, 0.01, (6, S, 1)).astype(np.float32)
    up_v, up_f = zo.uv_sphere(16, 12, (0.30, 0.26, 0.22), (0.0, 0.22, 0.0))
    lo_v, lo_f = zo.tube(16, 8, 0.24, -0.6, -0.05)
    body_v, body_f = zo.uv_sphere(24, 14, (0.22, 0.62, 0.16), (0.0, -0.05, 0.0))
    d.update(V_0=up_v, F_0=up_f, V_1=lo_v, F_1=lo_f, body_v=body_v, body_f=body_f)
    poses, trans = synth.poses_trans(N, seed=11)
    d["poses"], d["trans"] = (poses * 0.3).numpy(), (trans * 0.1).numpy()
    d["conds"] = (rng.standard_normal((3, N, 128)) * 0.1).astype(np.float32)
    cam = ps.camera(N, H, W, "cpu")
    d["cam"] = zo.camera_rows(cam).astype(np.float32)
    masks = np.ones((N, 6), bool)
    masks[:, 2] = False                          # right_cuff unlabelled in every frame
    if N > 1:
        masks[1, 4] = False                      # left_pant unlabelled in frame 1
    d["fl_masks"] = masks
    gt = []
    size = torch.tensor([[W, H]] * N, dtype=torch.float64)
    cam64 = camera(d, torch.float64)
    for n in ps.FL_NAMES:
        p = torch.tensor(ps.ring(np.asarray(ps.RINGS[n][0]), ps.RINGS[n][1] * 1.05, ps.RINGS[n][2], M, 0.1))
        gt.append(cam64.transform_points_screen(p[None].expand(N, -1, 3), size)[..., :2])
    d["gt_fl_pts"] = (torch.cat(gt, 1).numpy() + rng.normal(0, 0.5, (N, 6 * M, 2))).astype(np.float32)
    return d


class MaskRender(zo.OracleMaskRender):
    """raster_oracle's fragments with the zbuf in torch's default dtype (float32-rounded in the float32 run)."""

    def __call__(self, meshes):
        _, frags = super().__call__(meshes)
        frags.zbuf = frags.zbuf.to(torch.get_default_dtype())
        return None, frags


class Camera(zo.Camera):
    """zbuf_oracle's camera with CameraMine's own `view_rays` (whose output the zbuff branch does not use)."""

    def view_rays(self, ps_, cam_id=0):
        CameraMine = importlib.import_module("model.CameraMine")
        return CameraMine.RectifiedPerspectiveCameras.view_rays(self, ps_, cam_id)


def camera(d, dt):
    c = torch.tensor(d["cam"], dtype=dt)
    return Camera(c[:, 0:2], c[:, 2:4], c[:, 4:13].reshape(-1, 3, 3), c[:, 13:16], (W, H))


def curve_buffers(IFC, d):
    """The reference's initialize_parameters in float64 on the rings: its buffers, rounded to float32."""
    curve = make_curve(IFC, torch.tensor(d["curve_verts"], dtype=torch.float64))
    return {k: getattr(curve, k).detach().float().numpy() for k in
            ("cano_smpl_verts", "cano_verts_center", "cano_v_dirs", "cano_nx", "init_scale")}


def make_curve(IFC, verts):
    curve = object.__new__(IFC)
    torch.nn.Module.__init__(curve)
    curve.fl_names = list(ps.FL_NAMES)
    curve.sample_num = S
    curve.cano2canosmpl = lambda vs, names: [v.clone() for v in vs]
    curve.initialize_parameters(list(verts))
    return curve


def run(cls, OGN, ns, d, dt, weights_tag):
    import make_golden as mg
    sdf, deformer = (m.to(dt) for m in mg.surface_scene(ns.network, ns.Deformer))
    t = lambda k: torch.from_numpy(np.ascontiguousarray(d[k]))  # noqa: E731
    N = int(d["poses"].shape[0])
    IFC = importlib.import_module("engineer.utils.garment_structure").Intersect_Free_Curve
    curve = make_curve(IFC, t("curve_verts").to(dt))
    with torch.no_grad():
        for k in ("cano_smpl_verts", "cano_verts_center", "cano_v_dirs", "cano_nx", "init_scale"):
            getattr(curve, k).copy_(t("buf_" + k).to(dt))
        curve.scale.copy_(t("scale").to(dt))
        curve.nx_scale.copy_(t("nx_scale").to(dt))
    poses, trans = t("poses").to(dt).requires_grad_(True), t("trans").to(dt).requires_grad_(True)
    conds = [t("conds")[k].to(dt).requires_grad_(True) for k in range(3)]
    cam = camera(d, dt)
    checks = []
    self = types.SimpleNamespace(
        garment_size=2, garment_names=list(ps.GARMENTS), garment_nets=[sdf, sdf], fl_names=list(ps.FL_NAMES),
        garment_vs=[t("V_0").to(dt), t("V_1").to(dt)], garment_fs=[t("F_0"), t("F_1")], tmpBodyVs=t("body_v").to(dt),
        tmpBodyFs=t("body_f"), deformer=deformer, conf=ps.Conf(ps.CONF), info={}, sdfShrinkRadius=0.01,
        inter_free_curve=curve, maskRender=MaskRender(H, W, cam),
        fl_optimizer=torch.optim.AdamW([curve.scale, curve.nx_scale], lr=1e-4),
        dataset=types.SimpleNamespace(fl_weights=dict(ps.FL_WEIGHTS)),
        get_grad_parameters=lambda frame_ids, device: (conds, poses, trans, None))
    for name in ("deform_feature_line", "compute_fl_proj_loss"):
        setattr(self, name, types.MethodType(getattr(cls, name), self))
    zbuff = types.MethodType(cls.fl_visible_by_body_zbuff, self)

    def recorded_zbuff(*a, **k):
        out = zbuff(*a, **k)
        checks.append(out.detach().clone())
        return out

    self.fl_visible_by_body_zbuff = recorded_zbuff
    prev = torch.get_default_dtype()
    torch.set_default_dtype(dt)
    try:
        fl_vs, vis, lab, gts = cls.project_2d_loss(self, N, H, W, torch.arange(N), ps.RATIO, cam, t("fl_masks"),
                                                   t("gt_fl_pts").to(dt), "cpu")
    finally:
        torch.set_default_dtype(prev)
    tag = f"{weights_tag}/{'f32' if dt == torch.float32 else 'f64'}"
    out = {f"{tag}/info/{k}": np.array(float(v)) for k, v in self.info["fl_loss"].items()}
    for g in range(2):
        for c in range(len(fl_vs[g])):
            out[f"{tag}/screen_{g}_{c}"] = fl_vs[g][c].detach().numpy()
            out[f"{tag}/visible_{g}_{c}"] = vis[g][c].numpy()
            col = ps.FL_NAMES.index(ps.FL_EXTRACT[ps.GARMENTS[g]][c])
            assert torch.equal(lab[g][c], t("fl_masks")[:, None, col:col + 1].expand(N, S, 3))
        out[f"{tag}/gt_{g}"] = gts[g].detach().numpy()
        out[f"{tag}/body_check_{g}"] = checks[g][..., 1].numpy()
    out[f"{tag}/grad/scale"] = curve.scale.grad.detach().numpy()
    out[f"{tag}/grad/nx_scale"] = curve.nx_scale.grad.detach().numpy()
    out[f"{tag}/scale_after"] = curve.scale.detach().numpy()
    out[f"{tag}/nx_scale_after"] = curve.nx_scale.detach().numpy()
    for n in ps.FL_NAMES:
        out[f"{tag}/offset/{n}"] = deformer.defs[0].offset[n].detach().numpy()
    for mname, m in (("translator", deformer.defs[0]), ("sdf", sdf)):
        for pname, p in sorted(m.named_parameters()):
            if p.grad is not None:
                out[f"{tag}/grad/{mname}.{pname}"] = p.grad.detach().reshape(-1)[::GRAD_STRIDE].numpy()
    for k, x in (("poses", poses), ("trans", trans), ("cond1", conds[1]), ("cond2", conds[2])):
        if x.grad is not None:
            out[f"{tag}/grad/{k}"] = x.grad.detach().numpy()
    return out


def nn_violations(out, tag, d):
    """Annotation indices [(n, column)] whose chamfer nearest neighbours (either direction) are within NN_MARGIN."""
    bad = set()
    for g, garment in enumerate(ps.GARMENTS):
        for c, name in enumerate(ps.FL_EXTRACT[garment]):
            col = ps.FL_NAMES.index(name)
            x = out[f"{tag}/screen_{g}_{c}"][..., :2]
            v = out[f"{tag}/visible_{g}_{c}"][..., 0]
            for n in range(x.shape[0]):
                y = d["gt_fl_pts"][n, col * M:(col + 1) * M].astype(np.float64)
                q = x[n][v[n]]
                if len(q) < 2:
                    continue
                dist = ((q[:, None, :] - y[None]) ** 2).sum(-1)
                for axis in (1, 0):
                    srt = np.sort(dist, axis=axis)
                    d1, d2 = np.take(srt, 0, axis=axis), np.take(srt, 1, axis=axis)
                    amb = d2 - d1 <= NN_MARGIN * d1
                    if axis == 1:       # a curve point between two annotations: move its nearest annotation
                        for i in np.nonzero(amb)[0]:
                            bad.add((n, col * M + int(np.argmin(dist[i]))))
                    else:
                        for j in np.nonzero(amb)[0]:
                            bad.add((n, col * M + j))
    return sorted(bad)


def body_violations(out, tag):
    """Curve points [(curve column, point)] whose body check lies within BODY_MARGIN of the curve's threshold."""
    bad = set()
    for g, garment in enumerate(ps.GARMENTS):
        chk = out[f"{tag}/body_check_{g}"]
        thr = np.concatenate([np.full(S, ps.ZBUF_THRESHOLD[n]) for n in ps.FL_EXTRACT[garment]])
        for i in np.nonzero((np.abs(chk - thr[None]) <= BODY_MARGIN).any(0))[0]:
            bad.add((ps.FL_NAMES.index(ps.FL_EXTRACT[garment][i // S]), int(i % S)))
    return sorted(bad)


def generate():
    ns = refload.load()
    OGN = importlib.import_module("engineer.networks.OptimGarmentNetwork")
    OGNL = importlib.import_module("engineer.networks.OptimGarmentNetwork_Large_Pose")
    flo = importlib.import_module("engineer.core.fl_optimizer")
    IFC = importlib.import_module("engineer.utils.garment_structure").Intersect_Free_Curve
    old = flo.chamfer_distance, OGN.Meshes
    flo.chamfer_distance, OGN.Meshes = knn_oracle.chamfer_f64, zo.Meshes
    classes = (("base", OGN.OptimGarmentNetwork), ("large", OGNL.OptimGarmentNetwork_LargePose))
    out = {}
    try:
        for N in FRAMES:
            d = inputs(N, 1772 + N)
            d.update({"buf_" + k: v for k, v in curve_buffers(IFC, d).items()})
            rng = np.random.default_rng(N)
            for _ in range(20):
                o = run(classes[0][1], OGN, ns, d, torch.float64, "base")
                bad_nn, bad_body = nn_violations(o, "base/f64", d), body_violations(o, "base/f64")
                if not bad_nn and not bad_body:
                    break
                for n, j in bad_nn:             # move the annotation
                    d["gt_fl_pts"][n, j] += rng.normal(0, 0.3, 2).astype(np.float32)
                for c, i in bad_body:           # move the canonical-body point in depth
                    d["buf_cano_smpl_verts"][c, i, 2] += np.float32(0.003)
            assert not bad_nn and not bad_body, (bad_nn, bad_body)
            case = {f"in/{k}": v for k, v in d.items()}
            for tag, cls in classes:
                for dt in (torch.float32, torch.float64):
                    o = run(cls, OGN, ns, d, dt, tag)
                    if dt == torch.float32:         # float32: the loss terms and the curve gradients
                        o = {k: v for k, v in o.items() if "/info/" in k or k.endswith(("grad/scale", "grad/nx_scale"))}
                    case.update(o)
            out.update({f"n{N}/{k}": v for k, v in case.items()})
    finally:
        flo.chamfer_distance, OGN.Meshes = old
    return out


def main():
    out = generate()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out), "arrays;", {k: float(v) for k, v in out.items() if "/info/" in k and "f64" in k})


if __name__ == "__main__":
    main()
