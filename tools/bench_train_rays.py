"""Benchmark of the training-ray sub-sampling (csrc/train_rays.cu, DESIGN section 1j): the `sample_train_ray` drop-in
(recmv_b200.utils.make_sample_train_ray) against the reference's flow restated in torch on the same device
(OptimGarmentNetwork.py:983-1055: per garment the mask gather, four boolean selections, a CPU `torch.rand` copied to
the device, four more selections; then `view_rays` per garment), at the training shapes: two garments at 1080 x 1080,
`sample_pix_num` 2048 with a 3-frame batch and 6144 with 1- and 2-frame batches (configs/people_snapshot/*.conf),
each garment's list the pixels of a 15 %-of-frame silhouette, 90 % of them inside its ground-truth mask.

Per call: CUDA-event time after a warm-up (the two flows alternated, twice), host synchronisations (torch's sync
debug mode) and device work items (CUDA kernels and memcpy / memset, counted by torch.profiler in a separate run).
The card name, power limit and SM clocks are read in the same run.

    python tools/bench_train_rays.py [--reps 50] [--out FILE]
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from recmv_b200.utils import make_sample_train_ray  # noqa: E402

H = W = 1080
SHAPES = [(2048, 3), (6144, 1), (6144, 2)]     # (sample_pix_num, frames)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"nvidia-smi unavailable: {e}"
    return q.splitlines()[0] if q else torch.cuda.get_device_name(0)


def events_ms(fn, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
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


def count_device_work(fn):
    """(kernels, memcpy + memset) one call puts on the device."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    copies = sum(("memcpy" in e.name.lower() or "memset" in e.name.lower()) for e in evs)
    return len(evs) - copies, copies


class RectifiedPerspectiveCameras:
    """The reference camera's parameters and `view_rays` (model/CameraMine.py:146-167)."""

    def __init__(self, focal_length, principal_point, R, T, image_size=None):
        self.focal_length, self.principal_point, self.R, self.T = focal_length, principal_point, R, T

    def to(self, device):
        return self

    def view_rays(self, ps, cam_id=0):
        rays = torch.zeros_like(ps)
        f, p = self.focal_length, self.principal_point
        rays[:, 0] = -ps[:, 0] / f[cam_id, 0] + ps[:, 2] * p[cam_id, 0] / f[cam_id, 0]
        rays[:, 1] = -ps[:, 1] / f[cam_id, 1] + ps[:, 2] * p[cam_id, 1] / f[cam_id, 1]
        rays[:, 2] = ps[:, 2]
        rays = rays / torch.norm(rays, p=2, dim=1, keepdim=True)
        return rays.matmul(self.R[cam_id].transpose(0, 1))


class Conf:
    def __init__(self, pix):
        self.pix = pix

    def get_int(self, key):
        return self.pix

    def __contains__(self, key):
        return key == "sample_pix_num"


class Net:
    sample_train_ray = make_sample_train_ray()

    def reference_flow(self, N, sample_pix, gt_garment_masks_list, batch_garment_inds_list, batch_garment_row_list,
                       batch_garment_col_list, batch_garment_init_pts_list, frame_ids, device):
        """OptimGarmentNetwork.sample_train_ray as the reference writes it."""
        sample_pix = self.conf.get_int('sample_pix_num') if 'sample_pix_num' in self.conf else sample_pix
        sample_pix = sample_pix // self.garment_size
        lists = [[], [], [], []]
        for gt_garment_masks, batch_inds, row_inds, col_inds, init_pts in zip(
                gt_garment_masks_list, batch_garment_inds_list, batch_garment_row_list, batch_garment_col_list,
                batch_garment_init_pts_list):
            sel = gt_garment_masks[batch_inds, row_inds, col_inds] > 0.
            batch_inds, row_inds, col_inds, init_pts = batch_inds[sel], row_inds[sel], col_inds[sel], init_pts[sel]
            pnum = batch_inds.shape[0]
            if pnum > sample_pix * N:
                sel = torch.rand(pnum) < float(sample_pix * N) / float(pnum)
                sel = sel.to(batch_inds.device)
                batch_inds, row_inds, col_inds, init_pts = batch_inds[sel], row_inds[sel], col_inds[sel], init_pts[sel]
            for lst, t in zip(lists, (batch_inds, row_inds, col_inds, init_pts)):
                lst.append(t)
        focals, princeple_ps, Rs, Ts, H, W = self.dataset.get_camera_parameters(frame_ids.numel(), device)
        cameras = RectifiedPerspectiveCameras(focals, princeple_ps, Rs, Ts, image_size=[(W, H)]).to(device)
        self.maskRender.rasterizer.cameras = cameras
        if self.pcRender:
            self.pcRender.rasterizer.cameras = cameras
        rays = [cameras.view_rays(torch.cat([c.view(-1, 1), r.view(-1, 1), torch.ones_like(c.view(-1, 1))], dim=-1).float())
                for r, c in zip(lists[1], lists[2])]
        return lists[0], lists[1], lists[2], lists[3], rays, cameras


def scene(N, dev, seed):
    """Two garments: silhouettes (15 % of each frame, a disc per frame), lists in (n, row, col) order, masks keeping
    90 % of each list."""
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[:H, :W]
    args = [[], [], [], [], []]
    for k in range(2):
        cover = np.zeros((N, H, W), bool)
        for n in range(N):
            cy, cx = H * (0.4 + 0.2 * k), W * (0.45 + 0.05 * n)
            cover[n] = (yy - cy) ** 2 + (xx - cx) ** 2 < 0.15 * H * W / np.pi
        mask = (cover & (g.uniform(size=cover.shape) < 0.9)).astype(np.float32)
        b, r, c = np.nonzero(cover)
        for lst, t in zip(args, (mask, b, r, c, g.standard_normal((len(b), 3)).astype(np.float32))):
            lst.append(torch.from_numpy(t).to(dev))
    return args


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_rays: needs a CUDA device")
    dev = torch.device("cuda", 0)
    info = dict(card=card(), torch=torch.__version__)
    print(json.dumps(info))
    f = torch.tensor([[1100.0, 1100.0]], device=dev)
    pp = torch.tensor([[540.0, 540.0]], device=dev)
    R = torch.tensor([[[1.0, 0.0, 0.0], [0.0, -1.0, 0.0], [0.0, 0.0, -1.0]]], device=dev)
    T = torch.tensor([[0.0, 0.3, 2.5]], device=dev)
    torch.manual_seed(0)
    rows = []
    for pix, N in SHAPES:
        net = Net()
        net.conf, net.garment_size = Conf(pix), 2
        net.dataset = types.SimpleNamespace(get_camera_parameters=lambda n, d: (
            f.expand(n, 2), pp.expand(n, 2), R.expand(n, 3, 3), T.expand(n, 3), H, W))
        net.maskRender = types.SimpleNamespace(rasterizer=types.SimpleNamespace(cameras=None))
        net.pcRender = types.SimpleNamespace(rasterizer=types.SimpleNamespace(cameras=None))
        masks, b, r, c, pts = scene(N, dev, pix + N)
        call = (N, pix, masks, b, r, c, pts, torch.arange(N, device=dev), dev)
        flows = {"drop_in": lambda: net.sample_train_ray(*call), "reference_flow": lambda: net.reference_flow(*call)}
        for fn in flows.values():
            fn()
        torch.cuda.synchronize()
        row = dict(case=f"sample_pix_num{pix}_N{N}_2garments_1080", rows_in=[int(x.shape[0]) for x in b],
                   kept=[int(x.shape[0]) for x in net.sample_train_ray(*call)[0]])
        for _ in range(2):
            for name, fn in flows.items():
                row.setdefault(f"{name}_ms", []).append(round(events_ms(fn, a.reps), 4))
        for name, fn in flows.items():
            row[f"{name}_host_syncs"] = count_syncs(fn)
            row[f"{name}_kernels"], row[f"{name}_copies"] = count_device_work(fn)
        rows.append(row)
        print(json.dumps(row))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(dict(info, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
