"""Writes tests/golden/zbuf_ref.npz: the reference's OWN visibility tests, unmodified, run on the CPU in float32:
`OptimGarmentNetwork.fl_visible_by_body_zbuff` (engineer/networks/OptimGarmentNetwork.py:1374-1465) and
`check_zbuf_body` (engineer/core/fl_optimizer.py:30-59), with three stand-ins from oracle/zbuf_oracle.py:
  * `maskRender` returns raster_oracle's fragments (its float64 zbuf rounded to float32), and `Meshes` is a plain
    container of the vertex and face lists;
  * the camera is CameraMine's `transform_points_screen` (pytorch3d's composed world-to-NDC matrix, then the screen
    conversion) and `cam_pos`, restated in torch;
  * the deformers are small element-wise maps (GarmentDeformer, BodySkin).
Needs the reference source tree (oracle/refload.py).

Cases: N = 1 on a square image and N = 3 on a non-square one.  The body is an ellipsoid, the garment an open tube
around it; the curve points are rings on the garment (in front of and behind the body), rings near the body surface,
a wide ring off the silhouette (background, so the fill rule applies), points off-screen, and points on the image
border.  Stored per case: the inputs, both functions' outputs, and the oracle's per-query ambiguity flags.

    python tests/golden/make_golden_zbuf.py
"""
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import refload  # noqa: E402
from oracle import zbuf_oracle as zo  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "zbuf_ref.npz")
CASES = [  # name, N, H, W
    ("n1_square", 1, 160, 160),
    ("n3_wide", 3, 120, 200),
]
FL_NAMES = ["upper_bottom", "neck"]
GARMENT = "upper"
RATIO = 0.7


def scene(N, H, W, seed):
    """Every input of one case as float32 / int64 numpy arrays."""
    g = np.random.default_rng(seed)
    body_v, body_f = zo.uv_sphere(24, 14, (0.22, 0.55, 0.16), (0.0, 0.0, 0.0))
    garm_v, garm_f = zo.tube(32, 10, 0.27, -0.35, 0.3)
    ang = 0.25 * g.standard_normal((N, 3))
    R = np.stack([_rot(a) for a in ang]).astype(np.float32)
    T = np.stack([np.array([0.02 * n, -0.03, 2.6 + 0.1 * n]) for n in range(N)]).astype(np.float32)
    f = 1.1 * max(H, W)
    focal = np.full((N, 2), f, dtype=np.float32)
    pp = np.stack([np.full(N, W / 2.0 + 1.5), np.full(N, H / 2.0 - 2.0)], 1).astype(np.float32)
    poses = (0.3 * g.standard_normal((N, 6))).astype(np.float32)
    cond = g.standard_normal((N, 3)).astype(np.float32)
    trans = (0.02 * g.standard_normal((N, 3))).astype(np.float32)
    # curve points: rings on the garment (front visible, back hidden by the body), a ring far off the silhouette
    fl0 = np.concatenate([zo.rings(0.27, (-0.3, 0.0, 0.25), 40), zo.rings(1.4, (0.1,), 24)])
    fl1 = zo.rings(0.25, (0.28,), 32, phase=0.1)
    # their canonical-body counterparts, one per curve point
    cano0 = np.concatenate([zo.rings(0.2, (-0.2, 0.1, 0.3), 40), zo.rings(1.3, (0.0,), 24)])
    cano1 = zo.rings(0.12, (0.45,), 32, phase=0.1)
    return dict(N=N, H=H, W=W, body_v=body_v, body_f=body_f, garm_v=garm_v, garm_f=garm_f, R=R, T=T, focal=focal,
                pp=pp, poses=poses, cond=cond, trans=trans, fl0=fl0, fl1=fl1, cano0=cano0, cano1=cano1)


def _rot(a):
    cx, cy, cz = np.cos(a)
    sx, sy, sz = np.sin(a)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def camera(s, device="cpu"):
    t = lambda k: torch.tensor(s[k], device=device)  # noqa: E731
    return zo.Camera(t("focal"), t("pp"), t("R"), t("T"), (s["W"], s["H"]))


def proj_size(s, device="cpu"):
    return torch.tensor([[float(s["W"]), float(s["H"])]] * s["N"], device=device)


def edge_points(s, cam, n_each=6):
    """World points that project to the image border (sx = 0, sx = W, sy = 0, sy = H) and off-screen, on frame 0's
    camera, at depth 2.6: [k,3] float32."""
    W, H = s["W"], s["H"]
    fx, fy = s["focal"][0]
    px, py = s["pp"][0]
    R, T = s["R"][0].astype(np.float64), s["T"][0].astype(np.float64)
    ts = np.linspace(0.1, 0.9, n_each)
    scr = [(0.0, t * H) for t in ts] + [(float(W), t * H) for t in ts] + [(t * W, 0.0) for t in ts]
    scr += [(t * W, float(H)) for t in ts] + [(-40.0, 0.5 * H), (W + 40.0, 0.3 * H), (0.5 * W, -1e3)]
    Z = 2.6
    out = []
    for sx, sy in scr:
        xv = np.array([(px - sx) * Z / fx, (py - sy) * Z / fy, Z])
        out.append((xv - T) @ R.T)
    return np.asarray(out, dtype=np.float32)


def inputs(s):
    """The reference call's tensors: (cameras, def_fl_vs list, cano list, check-body screen points, ...)."""
    cam = camera(s)
    skin = zo.BodySkin()
    N = s["N"]
    poses = torch.tensor(s["poses"])
    edge = torch.tensor(edge_points(s, cam))
    def_fl_vs = [skin(torch.tensor(s["fl0"])[None].expand(N, -1, 3), poses),
                 torch.cat([skin(torch.tensor(s["fl1"])[None].expand(N, -1, 3), poses), edge[None].expand(N, -1, 3)], 1)]
    cano = [torch.tensor(s["cano0"])[None], torch.cat([torch.tensor(s["cano1"]), edge])[None]]
    q = torch.cat([torch.tensor(s["fl0"]), torch.tensor(s["cano0"])])[None].expand(N, -1, 3)
    check_pts = skin(q, [poses, torch.tensor(s["trans"])])
    check_pts = torch.cat([check_pts, edge[None].expand(N, -1, 3)], 1)
    return cam, def_fl_vs, cano, check_pts


def make_self(s, mask_render):
    from types import SimpleNamespace
    return SimpleNamespace(maskRender=mask_render, deformer=zo.GarmentDeformer(), garment_vs=[torch.tensor(s["garm_v"])],
                           garment_fs=[torch.tensor(s["garm_f"])], tmpBodyVs=torch.tensor(s["body_v"]),
                           tmpBodyFs=torch.tensor(s["body_f"]))


def oracle_flags(s, cam, def_fl_vs, cano, check_pts):
    """The oracle's ambiguity flags of both visibility columns [N,P,2] and of check_zbuf_body [N,Q]."""
    N, H, W = s["N"], s["H"], s["W"]
    rows = zo.camera_rows(cam)
    ps = proj_size(s)
    skin = zo.BodySkin()
    poses = torch.tensor(s["poses"])
    dg = zo.GarmentDeformer()(torch.tensor(s["garm_v"])[None].expand(N, -1, 3), [torch.tensor(s["cond"]), poses])
    fl = torch.cat(def_fl_vs, 1)
    a0 = zo.probe(dg.numpy(), s["garm_f"], rows, H, W, cam.transform_points_screen(fl, ps).numpy(), ps.numpy(),
                  np.zeros(N))["ambiguous"]
    body = skin(torch.tensor(s["body_v"])[None].expand(N, -1, 3), poses)
    sfl = torch.cat([skin(c.expand(N, -1, 3), poses) for c in cano], 1)
    a1 = zo.probe(body.numpy(), s["body_f"], rows, H, W, cam.transform_points_screen(sfl, ps).numpy(), ps.numpy(),
                  np.zeros(N))["ambiguous"]
    bt = skin(torch.tensor(s["body_v"])[None].expand(N, -1, 3), [poses, torch.tensor(s["trans"])])
    a2 = zo.probe(bt.numpy(), s["body_f"], rows, H, W, cam.transform_points_screen(check_pts, ps).numpy(), ps.numpy(),
                  np.zeros(N))["ambiguous"]
    return np.stack([a0, a1], -1), a2


def run_case(OGN, flo, k, case):
    name, N, H, W = case
    s = scene(N, H, W, 300 + k)
    cam, def_fl_vs, cano, check_pts = inputs(s)
    ps = proj_size(s)
    me = make_self(s, zo.OracleMaskRender(H, W, cam))
    with torch.no_grad():
        vis = OGN.OptimGarmentNetwork.fl_visible_by_body_zbuff(
            me, cam, [None, torch.tensor(s["cond"])], torch.tensor(s["poses"]), {"sdfRatio": RATIO}, {}, def_fl_vs,
            cano, FL_NAMES, 0, GARMENT, ps, N)
        screen = cam.transform_points_screen(check_pts, ps)
        mr = zo.OracleMaskRender(H, W, None)
        chk = flo.check_zbuf_body(zo.Meshes([torch.tensor(s["body_v"])], [torch.tensor(s["body_f"])]), N,
                                  zo.BodySkin(), torch.tensor(s["poses"]), torch.tensor(s["trans"]), cam, mr, ps,
                                  screen)
    vis_amb, chk_amb = oracle_flags(s, cam, def_fl_vs, cano, check_pts)
    out = {k2: np.asarray(v) for k2, v in s.items()}
    out.update(vis=vis.numpy(), vis_amb=vis_amb, check=chk.numpy(), check_screen=screen.numpy(), check_amb=chk_amb,
               fl_names=np.array(FL_NAMES), garment=np.array(GARMENT), ratio=np.array(RATIO))
    return {f"{name}/{key}": v for key, v in out.items()}


def generate():
    refload.load()
    OGN = importlib.import_module("engineer.networks.OptimGarmentNetwork")
    flo = importlib.import_module("engineer.core.fl_optimizer")
    old = OGN.Meshes, flo.Meshes
    try:
        OGN.Meshes = flo.Meshes = zo.Meshes
        out = {}
        for k, case in enumerate(CASES):
            out.update(run_case(OGN, flo, k, case))
    finally:
        OGN.Meshes, flo.Meshes = old
    return out


def main():
    out = generate()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, {k: int(v.sum()) for k, v in out.items() if k.endswith("_amb")})


if __name__ == "__main__":
    main()
