"""Mesh rasterizer that produces the fragments `FindSurfacePs` reads, in pytorch3d's `Fragments` layout with one face
per pixel (csrc/raster.cu).  It replaces the MeshRasterizer of the reference's `maskRender` (model/network.py:307-322)
in the reference camera's own screen space (model/CameraMine.py): view X R + T, screen (px - fx X/Z, py - fy Y/Z),
pixel (row, col) centred at (col, row).  Forward only; there is no CPU path.
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
