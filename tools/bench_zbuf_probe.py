"""Benchmark of the sparse z-buffer probe (csrc/zbuf_probe.cu, DESIGN section 1i) at the training shape: N = 3 frames
of 1080 x 1080, a garment of 159 200 faces, a 13 776-face body, Q = 800 curve points.

- the probe alone against full rasterization + fill + grid_sample (compat maskRender), CUDA-event time per call;
- the whole drop-in (utils.fl_visible_by_body_zbuff) against the reference's flow restated with the compat renderer
  (two full frames, fill, grid_sample, the camera's transform_points_screen), with element-wise deformer stand-ins.
Host synchronisations per call are counted with torch's sync debug mode.  The card name, power limit and SM clocks
are read in the same run.

    python tools/bench_zbuf_probe.py [--reps 50] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import types
import warnings

import numpy as np
import torch
import torch.nn.functional as Fn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import zbuf_oracle as zo  # noqa: E402
from recmv_b200 import raster  # noqa: E402
from recmv_b200 import utils as ru  # noqa: E402
from recmv_b200.compat.MaskRender import mask_renderer  # noqa: E402

N, H, W, Q = 3, 1080, 1080, 800


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def events_ms(fn, reps):
    for _ in range(5):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def count_syncs(fn):
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            fn()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    return sum("synchroniz" in str(x.message) for x in w)


def scene(dev):
    g = np.random.default_rng(0)
    gv, gf = zo.tube(400, 200, 0.27, -0.45, 0.35)
    bv, bf = zo.uv_sphere(84, 83, (0.22, 0.6, 0.16), (0, 0, 0))
    assert gf.shape[0] == 159200 and bf.shape[0] == 13776
    t = lambda a: torch.tensor(a, device=dev)  # noqa: E731
    R = torch.eye(3)[None].repeat(N, 1, 1)
    cam = zo.Camera(torch.full((N, 2), 1.1 * W), torch.tensor([[W / 2.0, H / 2.0]] * N), R,
                    torch.tensor([[0.0, 0.0, 2.6]] * N), (W, H)).to(dev)
    fl = [t(zo.rings(0.27, (-0.3, 0.0, 0.25), 200)), t(zo.rings(0.25, (0.28,), 200))]
    cano = [t(zo.rings(0.2, (-0.2, 0.1, 0.3), 200))[None], t(zo.rings(0.12, (0.45,), 200))[None]]
    poses, cond = t(0.2 * g.standard_normal((N, 6)).astype(np.float32)), t(g.standard_normal((N, 3)).astype(np.float32))
    me = types.SimpleNamespace(maskRender=mask_renderer((H, W), cameras=cam), deformer=zo.GarmentDeformer(),
                               garment_vs=[t(gv)], garment_fs=[t(gf)], tmpBodyVs=t(bv), tmpBodyFs=t(bf))
    skin = me.deformer.defs[1]
    def_fl = [skin(c[None].expand(N, -1, 3), poses) for c in fl]
    ps = torch.tensor([[float(W), float(H)]] * N, device=dev)
    args = (cam, [None, cond], poses, {}, {}, def_fl, cano, ["upper_bottom", "neck"], 0, "upper", ps, N)
    return me, args


def reference_flow(me, cam, d_cond_list, poses, ratio, fl_vs_dict, def_fl_vs, cano, fl_names, g_i, garment_name, ps, N):
    """OptimGarmentNetwork.fl_visible_by_body_zbuff (:1374-1465) restated on the compat renderer."""
    def sample(zbuf, pts):
        u = 2 * pts[..., 0] / ps[:, 0].view(-1, 1) - 1
        v = 2 * pts[..., 1] / ps[:, 1].view(-1, 1) - 1
        uv = torch.cat([u[..., None], v[..., None]], -1)
        return Fn.grid_sample(zbuf.permute(0, 3, 1, 2), uv.unsqueeze(2), align_corners=True)[:, 0, :, 0]

    c_z = me.maskRender.rasterizer.cameras.cam_pos()[None, None].detach().clone()[..., -1]
    gv = me.deformer(me.garment_vs[g_i][None].expand(N, -1, 3), [d_cond_list[g_i + 1], poses], ratio=ratio,
                     offset_type=garment_name)
    fl = torch.cat(def_fl_vs, 1)
    z = me.maskRender(zo.Meshes(list(gv), [me.garment_fs[g_i]] * N))[1].zbuf
    zm = (gv[..., -1].detach() - c_z).max(-1)[0][:, None, None, None].expand_as(z)
    z[z == -1.] = zm[z == -1.]
    gc = fl[..., -1] - (sample(z, cam.transform_points_screen(fl, ps)) + c_z)
    sfl = torch.cat([me.deformer.defs[1](c.expand(N, -1, 3), poses) for c, _ in zip(cano, fl_names)], 1)
    body = me.deformer.defs[1](me.tmpBodyVs.view(1, -1, 3).expand(N, -1, 3), poses)
    z = me.maskRender(zo.Meshes(list(body), [me.tmpBodyFs] * N))[1].zbuf
    zm = (body[..., -1].detach() - c_z).max(-1)[0][:, None, None, None].expand_as(z)
    z[z == -1.] = zm[z == -1.]
    bc = sfl[..., -1] - (sample(z, cam.transform_points_screen(sfl, ps)) + c_z)
    return torch.cat([gc[..., None], bc[..., None]], -1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_zbuf_probe: needs a CUDA device")
    dev = torch.device("cuda", 0)
    me, args = scene(dev)
    cam, ps = args[0], args[10]
    gv = me.deformer(me.garment_vs[0][None].expand(N, -1, 3), [args[1][1], args[2]])
    fl = torch.cat(args[5], 1)[:, :Q].contiguous()
    sp = raster.screen_points(fl, cam)
    fill = torch.ones(N, device=dev)
    faces = me.garment_fs[0]

    def probe():
        return raster.zbuf_probe(gv, faces, cam, (H, W), sp, ps, fill)

    def full():
        z = me.maskRender(zo.Meshes(list(gv), [faces] * N))[1].zbuf
        z[z == -1.] = fill[:, None, None, None].expand_as(z)[z == -1.]
        uv = torch.stack([2 * sp[..., 0] / ps[:, None, 0] - 1, 2 * sp[..., 1] / ps[:, None, 1] - 1], -1)
        return Fn.grid_sample(z.permute(0, 3, 1, 2), uv[:, :, None], align_corners=True)[:, 0, :, 0]

    def drop_in():
        return ru.fl_visible_by_body_zbuff(me, *args)

    def reference():
        with torch.no_grad():
            return reference_flow(me, *args)

    d = (probe() - full()).abs().max().item()
    dv = (drop_in() - reference()).abs().max().item()
    row = {"card": card(), "N": N, "H": H, "W": W, "Q": Q, "garment_faces": int(faces.shape[0]),
           "body_faces": int(me.tmpBodyFs.shape[0]), "curve_points": int(fl.shape[1]),
           "probe_vs_full_max_abs": d, "dropin_vs_reference_max_abs": dv}
    for name, fn in (("probe", probe), ("full_raster_fill_grid_sample", full), ("dropin", drop_in),
                     ("reference_flow", reference)):
        row[f"{name}_ms"] = round(events_ms(fn, a.reps), 4)
        row[f"{name}_host_syncs"] = count_syncs(fn)
    print(json.dumps(row))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(row, f, indent=1)


if __name__ == "__main__":
    main()
