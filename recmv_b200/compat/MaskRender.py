"""Drop-in for the reference's `maskRender`: the pytorch3d MeshRendererWithFragments(MeshRasterizer,
SoftSilhouetteShader) built at model/network.py:307-322 (faces_per_pixel 1, blur_radius 0, perspective-correct,
unclipped barycentrics, no back-face culling), on recmv_b200.raster.

The reference assigns the frame cameras through `renderer.rasterizer.cameras` (OptimGarmentNetwork.py:1043, 3029) and
reads `renderer.rasterizer.raster_settings.image_size`; both are plain attributes here.  `renderer(meshes)` returns
`(images, fragments)` with images = None: `find_surface_ps` (the training call site, OptimGarmentNetwork.py:742-783)
discards them, and the shaded previews `infer_garment` saves (`imgs[..., :3]`) are not produced.  Meshes are any object
with `verts_padded()` (or `verts_list()`) and `faces_list()`, one mesh per camera, all with the same faces (the deformed
copies of one marching-cubes mesh).
"""
from types import SimpleNamespace

import torch

from recmv_b200.raster import rasterize_meshes


def RasterizationSettings(image_size, z_clip=1e-6, area_eps=1e-8, want_dists=True, **ignored):
    """image_size = (H, W) as in the reference's settings; the pytorch3d-only options (blur_radius, bin_size,
    faces_per_pixel=1, ...) are accepted and ignored -- there is no per-bin cap to size."""
    return SimpleNamespace(image_size=tuple(image_size), z_clip=z_clip, area_eps=area_eps, want_dists=want_dists)


class MeshRasterizer:
    def __init__(self, cameras=None, raster_settings=None):
        self.cameras = cameras
        self.raster_settings = raster_settings

    def __call__(self, meshes, **kwargs):
        cameras = kwargs.get("cameras", self.cameras)
        if cameras is None:
            raise RuntimeError("MeshRasterizer: no cameras (assign renderer.rasterizer.cameras first)")
        fl = meshes.faces_list()
        faces = fl[0]
        for f in fl[1:]:
            if f.shape != faces.shape or (f.data_ptr() != faces.data_ptr() and not torch.equal(f, faces)):
                raise NotImplementedError("MeshRasterizer: all meshes must share one face list")
        if hasattr(meshes, "verts_padded"):
            verts = meshes.verts_padded()
        else:
            verts = torch.stack(meshes.verts_list())
        s = self.raster_settings
        return rasterize_meshes(verts.detach().float().contiguous(), faces.long().contiguous(), cameras, s.image_size,
                                z_clip=s.z_clip, area_eps=s.area_eps, want_dists=s.want_dists)


class MeshRendererWithFragments:
    def __init__(self, rasterizer, shader=None):
        self.rasterizer = rasterizer
        self.shader = shader

    def __call__(self, meshes, **kwargs):
        return None, self.rasterizer(meshes, **kwargs)


def mask_renderer(image_size, cameras=None):
    """The `maskRender` of model/network.py:307-322 for an image of (H, W) pixels."""
    return MeshRendererWithFragments(MeshRasterizer(cameras, RasterizationSettings(image_size)))
