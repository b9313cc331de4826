"""Drop-in for the reference's `maskRender`: the pytorch3d MeshRendererWithFragments(MeshRasterizer,
SoftSilhouetteShader) built at model/network.py:307-322 (faces_per_pixel 1, blur_radius 0, perspective-correct,
unclipped barycentrics, no back-face culling), on recmv_b200.raster.

The reference assigns the frame cameras through `renderer.rasterizer.cameras` (OptimGarmentNetwork.py:1043, 3029) and
reads `renderer.rasterizer.raster_settings.image_size`; both are plain attributes here.  `renderer(meshes)` returns
`(images, fragments)`.  Without a shader (what `mask_renderer` builds, and all `find_surface_ps` needs) images is None.
With `renderer.shader = HardPhongShader(device, cameras)` (infer_fl.py:167) the images are the Phong-shaded RGBA renders
`infer_garment` saves (`imgs[..., :3]`), and with a SoftSilhouetteShader the silhouettes (DESIGN section 1d).  Meshes
are any object with `verts_padded()` (or `verts_list()`) and `faces_list()`, one mesh per camera, all with the same
faces (the deformed copies of one marching-cubes mesh), and optionally `textures` with `verts_features_padded()` or
`verts_features_list()`.  Shaders, lights, materials and blend parameters are read by attribute, so pytorch3d's own
objects of these names work too.
"""
from types import SimpleNamespace

import torch

from recmv_b200.raster import rasterize_meshes, shade_meshes


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


def _rows3(x):
    return torch.as_tensor(x, dtype=torch.float32).reshape(-1, 3)


class PointLights:
    """pytorch3d's PointLights: one point light per row (1 row = every frame)."""

    def __init__(self, ambient_color=((0.5, 0.5, 0.5),), diffuse_color=((0.3, 0.3, 0.3),),
                 specular_color=((0.2, 0.2, 0.2),), location=((0, 1, 0),), device="cpu"):
        self.ambient_color, self.diffuse_color, self.specular_color, self.location = (
            _rows3(x).to(device) for x in (ambient_color, diffuse_color, specular_color, location))


class Materials:
    """pytorch3d's Materials: reflectance colours per row and a shininess exponent."""

    def __init__(self, ambient_color=((1, 1, 1),), diffuse_color=((1, 1, 1),), specular_color=((1, 1, 1),),
                 shininess=64, device="cpu"):
        self.ambient_color, self.diffuse_color, self.specular_color = (
            _rows3(x).to(device) for x in (ambient_color, diffuse_color, specular_color))
        self.shininess = torch.as_tensor(shininess, dtype=torch.float32).reshape(-1).to(device)


def BlendParams(sigma=1e-4, gamma=1e-4, background_color=(1.0, 1.0, 1.0)):
    return SimpleNamespace(sigma=sigma, gamma=gamma, background_color=background_color)


class TexturesVertex:
    """pytorch3d's TexturesVertex for meshes of equal size: per-vertex features, a list of [V,C] or a [N,V,C] tensor."""

    def __init__(self, verts_features):
        self._f = verts_features

    def verts_features_list(self):
        return list(self._f)

    def verts_features_padded(self):
        return self._f if torch.is_tensor(self._f) else torch.stack(list(self._f))


class HardPhongShader:
    """pytorch3d's HardPhongShader: Phong lighting of the K = 1 fragments with hard blending (alpha 1)."""

    def __init__(self, device="cpu", cameras=None, lights=None, materials=None, blend_params=None):
        self.cameras = cameras
        self.lights = lights if lights is not None else PointLights(device=device)
        self.materials = materials if materials is not None else Materials(device=device)
        self.blend_params = blend_params if blend_params is not None else BlendParams()


class SoftSilhouetteShader:
    """pytorch3d's SoftSilhouetteShader with K = 1: rgb 1, alpha sigmoid(-dists / sigma) on covered pixels."""

    def __init__(self, blend_params=None):
        self.blend_params = blend_params if blend_params is not None else BlendParams()


def _verts(meshes):
    return meshes.verts_padded() if hasattr(meshes, "verts_padded") else torch.stack(meshes.verts_list())


def _vertex_colors(meshes):
    tex = getattr(meshes, "textures", None)
    if tex is None:
        return None
    if hasattr(tex, "verts_features_padded"):
        return tex.verts_features_padded()
    return torch.stack(list(tex.verts_features_list()))


def _phong(shader, fragments, meshes, kwargs):
    cameras = kwargs.get("cameras", shader.cameras)
    if cameras is None:
        raise RuntimeError("HardPhongShader: no cameras (pass cameras= or build the shader with them)")
    lights = kwargs.get("lights", shader.lights)
    materials = kwargs.get("materials", shader.materials)
    blend = kwargs.get("blend_params", shader.blend_params)
    colors = _vertex_colors(meshes)
    if colors is not None and colors.shape[-1] != 3:
        raise NotImplementedError(f"HardPhongShader: vertex textures must have 3 channels, got {colors.shape[-1]}")
    return shade_meshes(_verts(meshes), meshes.faces_list()[0], fragments, cameras, colors=colors, lights=lights,
                        materials=materials, background=blend.background_color)


def _silhouette(shader, fragments, kwargs):
    if fragments.dists is None:
        raise RuntimeError("SoftSilhouetteShader: the rasterizer must compute dists (want_dists=True)")
    sigma = kwargs.get("blend_params", shader.blend_params).sigma
    d = fragments.dists[..., 0]
    alpha = torch.where(fragments.pix_to_face[..., 0] >= 0, torch.sigmoid(-d / sigma), torch.zeros_like(d))
    return torch.cat([torch.ones(d.shape + (3,), dtype=d.dtype, device=d.device), alpha[..., None]], -1)


class MeshRendererWithFragments:
    def __init__(self, rasterizer, shader=None):
        self.rasterizer = rasterizer
        self.shader = shader

    def __call__(self, meshes, **kwargs):
        fragments = self.rasterizer(meshes, **kwargs)
        shader = self.shader
        if shader is None:
            return None, fragments
        kind = type(shader).__name__
        with torch.no_grad():
            if kind == "HardPhongShader":
                return _phong(shader, fragments, meshes, kwargs), fragments
            if kind == "SoftSilhouetteShader":
                return _silhouette(shader, fragments, kwargs), fragments
        raise NotImplementedError(f"MeshRendererWithFragments: shader {kind} is not supported "
                                  "(HardPhongShader, SoftSilhouetteShader or None)")


def mask_renderer(image_size, cameras=None):
    """The `maskRender` of model/network.py:307-322 for an image of (H, W) pixels."""
    return MeshRendererWithFragments(MeshRasterizer(cameras, RasterizationSettings(image_size)))
