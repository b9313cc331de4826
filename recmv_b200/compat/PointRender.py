"""Drop-in for the reference's `pcRender`: PointsRendererWithFrags_Split(PointsRasterizer, AlphaCompositor) built in
`update_hierarchical_config` (OptimNetwork.py:87-100; model/CameraMine.py:347-415), and PointsRendererWithFrags
(OptimNetwork.py:444) with split=False, on recmv_b200.raster.rasterize_points.

The reference assigns the frame cameras through `renderer.rasterizer.cameras` and reads
`renderer.rasterizer.raster_settings.radius` (OptimGarmentNetwork.py:887, 940); both are plain attributes here.
`renderer(point_clouds, split_size=s, all_size=P)` returns `([upper, bottom], fragments)` with each image [N,H,W,1]
(so `imgs[..., -1]` works); without split, `(images, fragments)`.  Point clouds are any object with `points_padded()`
(or `points_list()`) and `features_packed()` (or `features_list()`), all clouds of one size.  Fragments are None unless
the renderer was built with return_fragments=True; they carry no gradient.
"""
from types import SimpleNamespace

import torch

from recmv_b200.raster import rasterize_points


def PointsRasterizationSettings(image_size, radius=0.01, points_per_pixel=8, **ignored):
    """image_size = (H, W), radius in NDC; the pytorch3d-only options (bin_size, max_points_per_bin) are accepted and
    ignored -- there is no per-bin cap to size."""
    return SimpleNamespace(image_size=tuple(image_size), radius=float(radius), points_per_pixel=int(points_per_pixel))


class PointsRasterizer:
    def __init__(self, cameras=None, raster_settings=None):
        self.cameras = cameras
        self.raster_settings = raster_settings

    def to(self, device):
        return self


class PointsRendererWithFrags:
    """Renders one silhouette per cloud; `split=True` (PointsRendererWithFrags_Split) renders two."""

    def __init__(self, rasterizer, compositor=None, split=False, return_fragments=False):
        self.rasterizer = rasterizer
        self.compositor = compositor
        self.split = split
        self.return_fragments = return_fragments

    def to(self, device):
        return self

    def __call__(self, point_clouds, **kwargs):
        cameras = kwargs.get("cameras", self.rasterizer.cameras)
        if cameras is None:
            raise RuntimeError("PointsRenderer: no cameras (assign renderer.rasterizer.cameras first)")
        if hasattr(point_clouds, "points_padded"):
            points = point_clouds.points_padded()
        else:
            points = torch.stack(point_clouds.points_list())
        N, P = int(points.shape[0]), int(points.shape[1])
        if hasattr(point_clouds, "features_packed"):
            feats = point_clouds.features_packed()
        else:
            feats = torch.cat(point_clouds.features_list())
        if feats is None or feats.numel() != N * P:
            raise NotImplementedError("PointsRenderer: one scalar feature per point is supported")
        split_size = None
        if self.split:
            split_size = int(kwargs["split_size"])
            if int(kwargs["all_size"]) != P:
                raise NotImplementedError(f"PointsRenderer: all_size {kwargs['all_size']} must equal the cloud size {P}")
        s = self.rasterizer.raster_settings
        images, frags = rasterize_points(points, cameras, s.image_size, s.radius, s.points_per_pixel,
                                         split_size=split_size, features=feats, want_fragments=self.return_fragments)
        return (images if self.split else images[0]), frags


def point_renderer(image_size, radius, points_per_pixel=50, split=True, cameras=None, return_fragments=False):
    """The `pcRender` of OptimNetwork.py:87-100 (split=True) or :444 (split=False) for an image of (H, W) pixels."""
    settings = PointsRasterizationSettings(image_size, radius=radius, points_per_pixel=points_per_pixel)
    return PointsRendererWithFrags(PointsRasterizer(cameras, settings), split=split, return_fragments=return_fragments)
