"""Mesh rasterizer that produces the fragments `FindSurfacePs` reads, in pytorch3d's `Fragments` layout with one face
per pixel (csrc/raster.cu).  It replaces the MeshRasterizer of the reference's `maskRender` (model/network.py:307-322)
in the reference camera's own screen space (model/CameraMine.py): view X R + T, screen (px - fx X/Z, py - fy Y/Z),
pixel (row, col) centred at (col, row).  Forward only; there is no CPU path.

Also the differentiable point-cloud silhouettes of the reference's `pcRender` (csrc/points_raster.cu): the points are
projected to NDC by a small torch graph, then rasterized and alpha-composited in one CUDA pass.
"""
from collections import namedtuple

import torch

from . import ops

Fragments = namedtuple("Fragments", ["pix_to_face", "zbuf", "bary_coords", "dists"])


def camera_rows(cameras, N, device):
    """[N,16] f32 {fx, fy, px, py, R row-major, T} on `device` from a camera with the reference camera's attributes
    (focal_length [N,2], principal_point [N,2], R [N,3,3], T [N,3]) or a tuple (focal_length, principal_point, R, T).
    A single camera is shared by all N frames."""
    if isinstance(cameras, (tuple, list)):
        focal, pp, R, T = cameras
    else:
        focal, pp, R, T = cameras.focal_length, cameras.principal_point, cameras.R, cameras.T
    focal, pp, R, T = (torch.as_tensor(x, dtype=torch.float32).to(device) for x in (focal, pp, R, T))
    M = R.reshape(-1, 9).shape[0]
    rows = torch.cat([focal.reshape(M, -1).expand(M, 2), pp.reshape(M, 2), R.reshape(M, 9), T.reshape(M, 3)], 1)
    if M == 1 and N != 1:
        rows = rows.expand(N, 16)
    elif M != N:
        raise RuntimeError(f"rasterize_meshes: {M} cameras for {N} frames")
    return rows.contiguous()


def rasterize_meshes(verts, faces, cameras, image_size, z_clip=1e-6, area_eps=1e-8, want_dists=True):
    """verts [N,V,3] f32 (one mesh per frame, shared topology), faces [F,3] int64 -> Fragments(pix_to_face [N,H,W,1]
    int64 packed n*F + f, zbuf [N,H,W,1], bary_coords [N,H,W,1,3] perspective-corrected and unclipped, dists [N,H,W,1]
    signed squared NDC distance to the nearest edge, or None when want_dists=False).  Background pixels are -1 in every
    output.  The nearest face wins; equal depths go to the lower face index, so the result is deterministic.
    Faces with a vertex at view depth <= z_clip or a doubled screen area <= area_eps are skipped."""
    H, W = (int(s) for s in image_size)
    if not verts.is_cuda:
        raise RuntimeError("rasterize_meshes runs on CUDA tensors only (no CPU path)")
    cam = camera_rows(cameras, int(verts.shape[0]), verts.device)
    p2f, zbuf, bary, dists, _ = ops.rasterize_meshes(verts, faces, cam, H, W, z_clip, area_eps, want_dists)
    return Fragments(p2f, zbuf, bary, dists)


def vertex_normals(verts, faces):
    """Per-vertex normals of N meshes with one face list (pytorch3d's `Meshes.verts_normals_padded` for meshes of equal
    size): verts [N,V,3], faces [F,3] -> [N,V,3] f32, area-weighted, unit length (0 for an unreferenced vertex).
    Deterministic (csrc/shade.cu, DESIGN section 1d).  Forward only; the inputs are used detached."""
    if not verts.is_cuda:
        raise RuntimeError("vertex_normals runs on CUDA tensors only (no CPU path)")
    return ops.vertex_normals(verts.detach().float().contiguous(), faces.detach().long().contiguous())


def sample_surface(verts, faces, count, seed=0, offset=0):
    """Area-weighted surface samples of N meshes with one face list (trimesh's `sample_surface` with a pinned stream):
    verts [N,V,3], faces [F,3] -> [N,count,3] f32.  Sample s of mesh n is a pure function of (seed, offset, n, s), so
    advancing `offset` by N*count per call continues the stream (csrc/surface_sample.cu, DESIGN section 1h).  Faces
    with an index outside [0, V) have area 0.  Forward only; the inputs are used detached."""
    if not verts.is_cuda:
        raise RuntimeError("sample_surface runs on CUDA tensors only (no CPU path)")
    return ops.surface_sample(verts.detach().float().contiguous(), faces.detach().long().contiguous(), count, seed,
                              offset)


# pytorch3d's PointLights and Materials defaults
DEFAULT_LIGHTS = {"location": (0.0, 1.0, 0.0), "ambient_color": (0.5,) * 3, "diffuse_color": (0.3,) * 3,
                  "specular_color": (0.2,) * 3}
DEFAULT_MATERIALS = {"ambient_color": (1.0,) * 3, "diffuse_color": (1.0,) * 3, "specular_color": (1.0,) * 3,
                     "shininess": 64.0}


def _rows(x, N, width, device, what):
    """x (1 or N rows of `width` values) -> [N,width] f32 on `device`, one row broadcast to all frames."""
    t = torch.as_tensor(x, dtype=torch.float32).detach().to(device).reshape(-1, width)
    if t.shape[0] == 1:
        return t.expand(N, width)
    if t.shape[0] != N:
        raise RuntimeError(f"shade_meshes: {t.shape[0]} rows of {what} for {N} frames")
    return t


def shade_params(cameras, lights, materials, background, N, device):
    """[N,28] per-frame constants of ops.shade_phong, built on `device` without a host read: camera centre -R T,
    light location and colours, material colours, shininess, background.  lights / materials are objects with
    pytorch3d's attribute names (or None for its defaults)."""
    cam = camera_rows(cameras, N, device)
    R, T = cam[:, 4:13].view(N, 3, 3), cam[:, 13:16]
    # element-wise, so one broadcast camera and N equal rows give the same bits
    centre = -(R[:, :, 0] * T[:, 0:1] + R[:, :, 1] * T[:, 1:2] + R[:, :, 2] * T[:, 2:3])
    lt = {k: getattr(lights, k) if lights is not None else v for k, v in DEFAULT_LIGHTS.items()}
    mt = {k: getattr(materials, k) if materials is not None else v for k, v in DEFAULT_MATERIALS.items()}
    parts = [centre] + [_rows(lt[k], N, 3, device, k) for k in ("location", "ambient_color", "diffuse_color",
                                                                   "specular_color")]
    parts += [_rows(mt[k], N, 3, device, k) for k in ("ambient_color", "diffuse_color", "specular_color")]
    parts += [_rows(mt["shininess"], N, 1, device, "shininess"), _rows(background, N, 3, device, "background")]
    return torch.cat(parts, 1).contiguous()


def shade_meshes(verts, faces, fragments, cameras, colors=None, lights=None, materials=None, background=(1.0, 1.0, 1.0)):
    """pytorch3d's HardPhongShader on the K = 1 fragments of rasterize_meshes (DESIGN section 1d): verts [N,V,3] world,
    faces [F,3], colors [N,V,3] or [1,V,3] per-vertex colours (None = 1), cameras as for rasterize_meshes (the camera
    centre -R T is the eye of the specular term), lights / materials with pytorch3d's attributes (None = its
    defaults), each with 1 or N rows.  Returns [N,H,W,4]: rgb = (ambient + diffuse) * colour + specular, unclamped,
    `background` where no face was hit, alpha 1.  Forward only; the inputs are used detached."""
    if not verts.is_cuda:
        raise RuntimeError("shade_meshes runs on CUDA tensors only (no CPU path)")
    verts = verts.detach().float().contiguous()
    faces = faces.detach().long().contiguous()
    N, V = int(verts.shape[0]), int(verts.shape[1])
    if colors is not None:
        colors = torch.as_tensor(colors).detach().to(device=verts.device, dtype=torch.float32).reshape(-1, V, 3)
        colors = colors.expand(N, V, 3).contiguous() if colors.shape[0] == 1 else colors.contiguous()
    params = shade_params(cameras, lights, materials, background, N, verts.device)
    return ops.shade_phong(fragments, verts, ops.vertex_normals(verts, faces), colors, faces, params)


PointFragments = namedtuple("PointFragments", ["idx", "zbuf", "dists"])


def project_points(points, cam, H, W):
    """[N,P,3] world points -> [N,P,3] (NDC x, NDC y, view z) under the camera rows of `camera_rows`: view X R + T,
    screen (px - fx X/Z, py - fy Y/Z), NDC x = 1 - (2 sx + 1) / W, y = 1 - (2 sy + 1) / H.  A torch graph, so the
    gradient reaches the points and any camera parameter that requires grad."""
    R = cam[:, 4:13].view(-1, 3, 3)
    v = torch.bmm(points, R) + cam[:, None, 13:16]
    sx = cam[:, None, 2] - cam[:, None, 0] * v[..., 0] / v[..., 2]
    sy = cam[:, None, 3] - cam[:, None, 1] * v[..., 1] / v[..., 2]
    return torch.stack([1 - (2 * sx + 1) / W, 1 - (2 * sy + 1) / H, v[..., 2]], -1).contiguous()


def rasterize_points(points, cameras, image_size, radius, points_per_pixel, split_size=None, features=None,
                     want_fragments=False):
    """Silhouettes of point clouds: pytorch3d's PointsRasterizer + AlphaCompositor as the reference's `pcRender` uses
    them (csrc/points_raster.cu, DESIGN section 1c).  points [N,P,3] f32 world (one cloud per frame, all of size P),
    features [N,P] or [N*P,1] (default ones; must not require grad), radius in NDC.  Returns (images, fragments):
    images is a list of [N,H,W,1] tensors -- one, or two when split_size is an int (points p < split_size go to the
    first, the rest to the second; the transmittance runs over both, so one group occludes the other) --
    differentiable in the points and the camera; fragments = PointFragments(idx [N,H,W,K] packed n*P + p, zbuf, dists)
    padded with -1 and without gradient when want_fragments, else None.  Ties in z go to the lower packed index."""
    H, W = (int(s) for s in image_size)
    if not points.is_cuda:
        raise RuntimeError("rasterize_points runs on CUDA tensors only (no CPU path)")
    N, P = int(points.shape[0]), int(points.shape[1])
    cam = camera_rows(cameras, N, points.device)
    ndc = project_points(points.float(), cam, H, W)
    if features is not None:
        if features.requires_grad:
            raise RuntimeError("rasterize_points: features must not require grad (no gradient is computed for them)")
        features = features.detach().float().reshape(N, P).contiguous()
    out = ops.RasterizePointsFunction.apply(ndc, features, H, W, float(radius), int(points_per_pixel), split_size,
                                            bool(want_fragments))
    images, frags = (out[0], PointFragments(*out[1:])) if want_fragments else (out, None)
    return [im[..., None] for im in images.unbind(0)], frags
