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
