"""Writes tests/golden/train_rays_ref.npz: the reference's OWN `OptimGarmentNetwork.sample_train_ray`
(engineer/networks/OptimGarmentNetwork.py:983-1055), unmodified, run on the CPU with
  * a lightweight `self` (conf, garment_size, dataset.get_camera_parameters, maskRender, pcRender);
  * `RectifiedPerspectiveCameras` rebound to a subclass of the reference's own class (model/CameraMine.py) that only
    stores focal_length, principal_point, R and T, so the rays are the reference's own `view_rays`;
  * the module's `torch.rand` answering with oracle/train_rays_oracle.py's uniforms at the counters the kernel uses
    (offset + the earlier garments' input rows + j), so the reference's own selection code decides what is kept.
Needs the reference source tree (oracle/refload.py).

Three cases of two garments on seeded masks (values 0, 1, 0.5, -1 and NaN) and decode-ordered lists:
  below  every garment has pnum <= T (no draw);
  above  both garments draw, from an offset just below 2^32 so the counters cross into the high word;
  mixed  one garment draws and the other does not; `sample_pix_num` is absent from conf, so the argument is used.
Stored per case: the inputs, the camera, T's parts, the stream, and the reference's outputs.

    python tests/golden/make_golden_train_rays.py
"""
import importlib
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import refload, train_rays_oracle as tro  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "train_rays_ref.npz")
SEED = 0x0123456789ABCDEF
N, H, W = 2, 32, 36
CASES = [  # name, conf sample_pix_num (None = absent), sample_pix argument, garment_size, stream offset, coverage
    ("below", 8192, 64, 2, 0, (0.5, 0.3)),
    ("above", 512, 64, 2, (1 << 32) - 1000, (0.8, 0.6)),
    ("mixed", None, 600, 2, 12345, (0.9, 0.1)),
]


class Conf:
    def __init__(self, d):
        self.d = d

    def get_int(self, key):
        return int(self.d[key])

    def __contains__(self, key):
        return key in self.d


def camera():
    """fx, fy, px, py and a rotation with the reference's y / z flips, as the dataset's get_camera_parameters gives."""
    q = np.array([0.97, 0.05, -0.2, 0.1])
    q /= np.linalg.norm(q)
    w, x, y, z = q
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]) @ np.diag([1., -1., -1.])
    return (np.array([52.5, 49.75], np.float32), np.array([19.3, 24.6], np.float32), R.astype(np.float32),
            np.array([0.02, -0.1, 2.4], np.float32))


def garment(rng, cover):
    """(mask [N,H,W], batch, row, col, init pts) of one garment: the list is the covered pixels in (n, row, col)
    order, as the fragment decode emits them."""
    mask = rng.choice(np.array([0., 1., 0.5, -1., np.nan], np.float32), size=(N, H, W), p=[0.3, 0.5, 0.1, 0.05, 0.05])
    b, r, c = np.nonzero(rng.uniform(size=(N, H, W)) < cover)
    pts = (rng.integers(-128, 128, size=(len(b), 3)) / 64).astype(np.float32)
    return mask.astype(np.float32), b.astype(np.int64), r.astype(np.int64), c.astype(np.int64), pts


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


def run_case(OGN, Cam, k, case):
    name, conf_pix, arg_pix, gsize, offset, covers = case
    rng = np.random.default_rng(200 + k)
    lists = [garment(rng, c) for c in covers]
    focal, pp, R, T = camera()
    sample_pix = (conf_pix if conf_pix is not None else arg_pix) // gsize
    target = sample_pix * N
    # the uniforms the kernel draws for each garment that draws, in call order
    draws, base = [], 0
    for mask, b, r, c, _ in lists:
        pnum = len(tro.candidates(mask, b, r, c))
        if pnum > target:
            draws.append(tro.uniforms(SEED, tro.counters(offset, base, pnum)))
        base += len(b)
    dataset = types.SimpleNamespace(get_camera_parameters=lambda n, dev: (
        torch.tensor(focal).view(1, 2).expand(n, 2), torch.tensor(pp).view(1, 2).expand(n, 2),
        torch.tensor(R).view(1, 3, 3).expand(n, 3, 3), torch.tensor(T).view(1, 3).expand(n, 3), H, W))
    self = types.SimpleNamespace(conf=Conf({} if conf_pix is None else {"sample_pix_num": conf_pix}),
                                 garment_size=gsize, dataset=dataset,
                                 maskRender=types.SimpleNamespace(rasterizer=types.SimpleNamespace(cameras=None)),
                                 pcRender=types.SimpleNamespace(rasterizer=types.SimpleNamespace(cameras=None)))
    old_torch, old_cam = OGN.torch, OGN.RectifiedPerspectiveCameras
    OGN.torch, OGN.RectifiedPerspectiveCameras = TorchWithRand(draws), Cam
    try:
        res = OGN.OptimGarmentNetwork.sample_train_ray(
            self, N, arg_pix, [torch.tensor(m) for m, *_ in lists], [torch.tensor(x[1]) for x in lists],
            [torch.tensor(x[2]) for x in lists], [torch.tensor(x[3]) for x in lists], [torch.tensor(x[4]) for x in lists],
            torch.arange(N), "cpu")
        assert not OGN.torch.draws
    finally:
        OGN.torch, OGN.RectifiedPerspectiveCameras = old_torch, old_cam
    assert self.maskRender.rasterizer.cameras is res[5] and self.pcRender.rasterizer.cameras is res[5]
    out = {"seed": np.array(SEED, dtype=np.uint64), "offset": np.array(offset, dtype=np.uint64),
           "conf_pix": np.array(-1 if conf_pix is None else conf_pix), "arg_pix": np.array(arg_pix),
           "garment_size": np.array(gsize), "N": np.array(N), "focal": focal, "pp": pp, "R": R, "T": T}
    for g, (mask, b, r, c, pts) in enumerate(lists):
        out.update({f"mask_{g}": mask, f"batch_{g}": b, f"row_{g}": r, f"col_{g}": c, f"pts_{g}": pts})
        for j, key in enumerate(("batch", "row", "col", "pts", "rays")):
            out[f"ref_{key}_{g}"] = res[j][g].detach().numpy()
    return {f"{name}/{key}": v for key, v in out.items()}


def generate():
    refload.load()
    OGN = importlib.import_module("engineer.networks.OptimGarmentNetwork")
    CameraMine = importlib.import_module("model.CameraMine")

    class Cam(CameraMine.RectifiedPerspectiveCameras):
        """The reference camera class without pytorch3d's base: its own view_rays on the stored parameters."""

        def __init__(self, focal_length, principal_point, R, T, image_size=None):
            self.focal_length, self.principal_point, self.R, self.T = focal_length, principal_point, R, T

        def to(self, device):
            return self

    out = {}
    for k, case in enumerate(CASES):
        out.update(run_case(OGN, Cam, k, case))
    return out


def main():
    out = generate()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, {k: v.shape for k, v in out.items() if "/ref_batch" in k})


if __name__ == "__main__":
    main()
