"""Benchmark of mask_loss's dilation and soft IoU on the device (csrc/mask_iou.cu, DESIGN section 1m): the drop-in
(recmv_b200.utils.make_mask_loss) against the reference's method restated in torch on the same renderers and networks
(`reference_mask_loss` below: `F.max_pool2d` of each ground-truth mask, the IoU as the reference's element-wise chain,
`.item()` for every info value), and the dilation and IoU forward + backward alone against the torch chain.  Two
garments, the marching-cubes vertices of synth.sphere_sdf_grid at 257^3 split in two (as tools/bench_points_raster.py),
at 1080 x 1080: N = 3 frames with r = 3 (coarse stage) and N = 1 with r = 2 (fine stage).

Per call: CUDA-event time after a warm-up (the flows alternated, twice), host synchronisations (torch's sync debug
mode) and device work items (kernels and memcpy / memset, torch.profiler in a separate run).  The IoU alone is also
reported as achieved bytes per second against its ~12 B per pixel per direction.  The card name, power limit and SM
clocks are read in the same run.

    python tools/bench_mask_loss.py [--reps 10] [--out FILE]
"""
import argparse
import json
import os
import sys
import types

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import surface_render_scene as srs  # noqa: E402
from bench_surface_render_loss import card, count_device_work, count_syncs, events_ms  # noqa: E402
from recmv_b200 import ops, synth, utils  # noqa: E402
from recmv_b200.compat.MaskRender import mask_renderer  # noqa: E402
from recmv_b200.compat.PointRender import point_renderer  # noqa: E402

H = W = 1080
SHAPES = [(3, 3), (1, 2)]            # (frames, dilation radius in pixels)


def reference_mask_loss(self, N, H, W, frame_ids, ratio, gt_garment_masks_list, device):
    """The reference's mask_loss (OptimGarmentNetwork.py:621-667, 841-981) restated in torch on the same renderers."""
    conf = self.conf
    G = self.garment_size
    d_cond_list, poses, trans, _ = self.get_grad_parameters(frame_ids, device)
    def_vs = [self.deformer(self.garment_vs[g][None].expand(N, -1, 3), [d_cond_list[g + 1], [poses, trans]],
                            ratio=ratio, offset_type=name) for g, name in zip(range(G), self.garment_names)]
    meshes = [utils.Meshes(verts=[v.view(-1, 3) for v in torch.split(dv, 1)], faces=[fs] * N)
              for fs, dv in zip(self.garment_fs, def_vs)]
    self.info['pc_loss'] = {}
    surface_ps = self.find_surface_ps(meshes)
    whole = [torch.cat([a, b], 0) for a, b in zip(meshes[0].verts_list(), meshes[1].verts_list())]
    P = int(whole[0].shape[0])
    feats = torch.ones((N * P, 1), device=device)
    masks, _ = self.pcRender(utils._Cloud(torch.stack(whole), feats), split_size=int(self.garment_vs[0].shape[0]),
                             all_size=P)
    radius = int(round(self.pcRender.rasterizer.raster_settings.radius / 2. * float(min(H, W)) / 1.2))
    mgt = [F.max_pool2d(gt, kernel_size=2 * radius + 1, stride=1, padding=radius) for gt in gt_garment_masks_list]
    garment_loss = 0.
    for g, name in enumerate(self.garment_names):
        m, gm = masks[g][..., -1], mgt[g]
        mask_loss = (1. - (m * gm).view(N, -1).sum(1) / (m + gm - m * gm).abs().view(N, -1).sum(1)).mean()
        self.info['pc_loss']['{}_mask_loss'.format(name)] = mask_loss.item()
        loss = mask_loss
        off = def_vs[g] - self.deformer.defs[1](self.garment_vs[g].view(1, -1, 3).expand(N, -1, 3), [poses, trans])
        off = (off * off).sum(-1)
        c = conf.get_float('pc_weight.def_consistent.c')
        cl = utils.GMRobustError(off, c, True).mean()
        self.info['pc_loss']['garment_{}_defconst_loss'.format(name)] = cl.item()
        garment_loss += loss + cl * conf.get_float('pc_weight.def_consistent.weight')
    self.garment_optimizer.zero_grad()
    garment_loss.backward()
    self.garment_optimizer.step()
    pc_sdf_loss = 0.
    for g, (vs, name) in enumerate(zip(self.garment_vs, self.garment_names)):
        sdf_loss = (self.garment_nets[g](vs, ratio).view(-1) + self.sdfShrinkRadius).abs().mean()
        self.info['pc_{}_loss_sdf'.format(name)] = sdf_loss.item()
        pc_sdf_loss += sdf_loss * conf.get_float('pc_weight.weight')
    return meshes, masks, mgt, pc_sdf_loss, surface_ps


def find_surface_ps(self, meshes):
    out = [[] for _ in range(5)]
    with torch.no_grad():
        for mesh, vs, fs in zip(meshes, self.garment_vs, self.garment_fs):
            _, frags = self.maskRender(mesh)
            for lst, x in zip(out, utils.FindSurfacePs(vs.detach(), fs, frags)):
                lst.append(x)
    return out[0], out[0], out[1], out[2], out[3], out[4]


def garments(dev):
    """The sphere grid's marching-cubes mesh split by vertex index into two garments: (verts, faces) each."""
    sdf = synth.sphere_sdf_grid(257, num=8, seed=3, device=dev)
    h = 2.0 / 256
    verts, faces = ops.mc_gpu(sdf, h, h, h, -1.0, -1.0, -1.0, 0.0)
    verts, faces = verts.float() * 0.9, faces.long()
    half = int(verts.shape[0]) // 2
    out = []
    for lo, hi in ((0, half), (half, int(verts.shape[0]))):
        keep = ((faces >= lo) & (faces < hi)).all(1)
        out.append((verts[lo:hi].contiguous(), (faces[keep] - lo).contiguous()))
    return out


def scene(dev, N, r, nets, parts):
    sdf, deformer, _ = nets
    radius = r * 1.2 * 2. / min(H, W)
    conf = srs.Conf({"pc_weight.weight": 60.0, "pc_weight.laplacian_weight": -10.0, "pc_weight.edge_weight": -10.0,
                     "pc_weight.norm_weight": -0.001, "pc_weight.def_consistent.weight": 0.6,
                     "pc_weight.def_consistent.c": 0.01, "pc_weight.curve_aware_weight": 0.0})
    poses, trans = (x.to(dev).requires_grad_(True) for x in synth.poses_trans(N, seed=2))
    conds = [(torch.randn((N, 128), device=dev) * 0.1).requires_grad_(True) for _ in range(3)]
    R = torch.diag(torch.tensor([-1.0, -1.0, 1.0]))
    cam = types.SimpleNamespace(focal_length=torch.full((N, 2), 0.9 * H, device=dev),
                                principal_point=torch.tensor([[W / 2 - 0.5, H / 2 - 0.5]] * N, device=dev),
                                R=R.expand(N, 3, 3).contiguous().to(dev), T=torch.tensor([[0.0, 0.0, 2.6]] * N,
                                                                                         device=dev))
    vs = [v.clone().requires_grad_(True) for v, _ in parts]
    self = types.SimpleNamespace(
        garment_size=2, garment_names=["upper", "bottom"], garment_nets=[sdf, sdf], garment_vs=vs,
        garment_fs=[f for _, f in parts], deformer=deformer, conf=conf, info={}, sdfShrinkRadius=0.01,
        pcRender=point_renderer((H, W), radius, points_per_pixel=50, split=True, cameras=cam),
        maskRender=mask_renderer((H, W), cameras=cam), garment_optimizer=torch.optim.SGD(vs, lr=0.0, momentum=0.9),
        curve_aware_loss=lambda ratio: 0., get_grad_parameters=lambda frame_ids, device: (conds, poses, trans, None))
    self.find_surface_ps = types.MethodType(find_surface_ps, self)
    g = torch.Generator(device="cpu").manual_seed(N)
    gts = [(torch.rand((N, H, W), generator=g) < 0.3).float().to(dev) for _ in range(2)]
    return self, (N, H, W, torch.arange(N, device=dev), srs.RATIO, gts, dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mask_loss: needs a CUDA device")
    dev = torch.device("cuda", 0)
    info = dict(card=card(), torch=torch.__version__)
    print(json.dumps(info))
    nets = srs.networks(dev)
    parts = garments(dev)
    torch.manual_seed(0)
    rows = []
    for N, r in SHAPES:
        self, args = scene(dev, N, r, nets, parts)
        drop_in = utils.make_mask_loss()
        flows = {"drop_in": lambda: drop_in(self, *args), "reference_flow": lambda: reference_mask_loss(self, *args)}
        for fn in flows.values():
            fn()
        torch.cuda.synchronize()
        row = dict(case=f"N{N}_r{r}_2garments_1080", verts=[int(v.shape[0]) for v, _ in parts])
        for _ in range(2):
            for name, fn in flows.items():
                row.setdefault(f"{name}_ms", []).append(round(events_ms(fn, a.reps), 3))
        for name, fn in flows.items():
            row[f"{name}_host_syncs"] = count_syncs(fn)
            row[f"{name}_kernels"], row[f"{name}_copies"] = count_device_work(fn)
        # the dilation and IoU alone, forward + backward
        ms = [torch.rand((N, H, W), device=dev, requires_grad=True) for _ in range(2)]
        gts = args[5]

        def kernel():
            out = ops.MaskIouFunction.apply(r, *ms, *gts)
            out[0].sum().backward()

        def chain():
            tot = 0.
            for m, gt in zip(ms, gts):
                gm = F.max_pool2d(gt, kernel_size=2 * r + 1, stride=1, padding=r)
                tot = tot + (1. - (m * gm).view(N, -1).sum(1) / (m + gm - m * gm).abs().view(N, -1).sum(1)).mean()
            tot.backward()

        fwd = lambda: ops.mask_iou(ms, gts, r)  # noqa: E731
        loss, _, iu, mgt = fwd()
        bwd = lambda: ops.mask_iou_backward(ms, mgt, iu, torch.ones(2, device=dev))  # noqa: E731
        for name, fn in (("iou_kernel_fwd_bwd", kernel), ("iou_torch_chain_fwd_bwd", chain), ("iou_fwd", fwd),
                         ("iou_bwd", bwd)):
            fn()
            row[f"{name}_ms"] = round(events_ms(fn, a.reps * 5), 4)
        for name, fn in (("iou_kernel_fwd_bwd", kernel), ("iou_torch_chain_fwd_bwd", chain)):
            row[f"{name}_kernels"], row[f"{name}_copies"] = count_device_work(fn)
        pix = 2 * N * H * W
        row["iou_fwd_GBps_at_12B_per_px"] = round(12 * pix / row["iou_fwd_ms"] / 1e6, 1)
        row["iou_bwd_GBps_at_12B_per_px"] = round(12 * pix / row["iou_bwd_ms"] / 1e6, 1)
        rows.append(row)
        print(json.dumps(row))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(dict(info, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
