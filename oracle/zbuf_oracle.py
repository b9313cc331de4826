"""Float64 restatement of the sparse z-buffer probe (DESIGN section 1i), written from the definitions: the full frame
from `raster_oracle.rasterize`, its background (zbuf == -1) replaced by a per-frame fill, then sampled at the query
points as ATen's `grid_sample(mode='bilinear', padding_mode='zeros', align_corners=True)` samples it.  Also the
pieces the fixture generator and the tests share to drive the reference's visibility tests: a camera with CameraMine's
`transform_points_screen` and `cam_pos` restated in torch, a `Meshes` stand-in, a `maskRender` that returns the
oracle's fragments, small element-wise deformers and the scenes.
"""
from types import SimpleNamespace

import numpy as np
import torch

from . import raster_oracle


def grid_sample(img, uv):
    """ATen's bilinear, zeros-padding, align_corners=True sampling of img [N,H,W] at uv [N,Q,2] (x, y in [-1, 1]) in
    float64 -> [N,Q].  ix = ((u + 1) / 2) (W - 1); taps nw, ne, sw, se at floor(ix) + {0, 1}; a tap outside the image
    contributes 0; terms summed in the order nw, ne, sw, se.  A non-finite coordinate gives 0."""
    img = np.asarray(img, dtype=np.float64)
    uv = np.asarray(uv, dtype=np.float64)
    N, H, W = img.shape
    with np.errstate(invalid="ignore"):
        ix = ((uv[..., 0] + 1) / 2) * (W - 1)
        iy = ((uv[..., 1] + 1) / 2) * (H - 1)
    fin = np.isfinite(ix) & np.isfinite(iy) & (np.abs(ix) < 2 ** 30) & (np.abs(iy) < 2 ** 30)
    ix, iy = np.where(fin, ix, -10.0), np.where(fin, iy, -10.0)
    x0, y0 = np.floor(ix), np.floor(iy)
    out = np.zeros(ix.shape)
    n = np.broadcast_to(np.arange(N)[:, None], ix.shape)
    for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1)):
        cx, cy = x0 + dx, y0 + dy
        w = (1 - np.abs(ix - cx)) * (1 - np.abs(iy - cy))
        ok = (cx >= 0) & (cx < W) & (cy >= 0) & (cy < H)
        v = img[n, np.clip(cy, 0, H - 1).astype(np.int64), np.clip(cx, 0, W - 1).astype(np.int64)]
        out += np.where(ok, v * w, 0.0)
    return out


def taps(H, W, screen_pts, norm_size):
    """(cols, rows, weights, in-image) [N,Q,4] of the four taps nw, ne, sw, se in float64."""
    p = np.asarray(screen_pts, dtype=np.float64)
    ns = np.asarray(norm_size, dtype=np.float64).reshape(-1, 1, 2)
    u, v = 2 * p[..., 0] / ns[..., 0] - 1, 2 * p[..., 1] / ns[..., 1] - 1
    with np.errstate(invalid="ignore"):
        ix, iy = ((u + 1) / 2) * (W - 1), ((v + 1) / 2) * (H - 1)
    fin = np.isfinite(ix) & np.isfinite(iy) & (np.abs(ix) < 2 ** 30) & (np.abs(iy) < 2 ** 30)
    ix, iy = np.where(fin, ix, -10.0), np.where(fin, iy, -10.0)
    x0, y0 = np.floor(ix), np.floor(iy)
    cols = np.stack([x0, x0 + 1, x0, x0 + 1], -1)
    rows = np.stack([y0, y0, y0 + 1, y0 + 1], -1)
    w = (1 - np.abs(ix[..., None] - cols)) * (1 - np.abs(iy[..., None] - rows))
    ok = (cols >= 0) & (cols < W) & (rows >= 0) & (rows < H)
    return cols.astype(np.int64), rows.astype(np.int64), w, ok


def probe(verts, faces, cams, H, W, screen_pts, norm_size, fill, z_clip=1e-6, area_eps=1e-8, margin_px=1e-3,
          ztol=1e-5):
    """verts [N,V,3], faces [F,3], cams [N,16], screen_pts [N,Q,>=2], norm_size [N,2] (w, h), fill [N] -> dict:
    out [N,Q] float64; tap_zbuf / tap_face [N,Q,4] (the oracle's zbuf and packed face, -1 on background and outside);
    ambiguous [N,Q]: a tap of non-zero weight at a pixel whose coverage or depth order fp32 could decide differently
    (raster_oracle's margins margin_px and ztol, or an exact depth tie); frags: the full rasterization."""
    fr = raster_oracle.rasterize(verts, faces, cams, H, W, z_clip, area_eps, margin_px=margin_px, ztol=ztol)
    z = fr["zbuf"].copy()
    fill = np.asarray(fill, dtype=np.float64).reshape(-1)
    for n in range(z.shape[0]):
        z[n][z[n] == -1.0] = fill[n]
    p = np.asarray(screen_pts, dtype=np.float64)
    ns = np.asarray(norm_size, dtype=np.float64).reshape(-1, 1, 2)
    uv = np.stack([2 * p[..., 0] / ns[..., 0] - 1, 2 * p[..., 1] / ns[..., 1] - 1], -1)
    out = grid_sample(z, uv)
    cols, rows, w, ok = taps(H, W, p, norm_size)
    n = np.broadcast_to(np.arange(z.shape[0])[:, None, None], cols.shape)
    cc, rr = np.clip(cols, 0, W - 1), np.clip(rows, 0, H - 1)
    tz = np.where(ok, fr["zbuf"][n, rr, cc], -1.0)
    tf = np.where(ok, fr["pix_to_face"][n, rr, cc], -1)
    amb = ((fr["ambiguous"] | fr["tie"])[n, rr, cc] & ok & (w > 0)).any(-1)
    return dict(out=out, tap_zbuf=tz, tap_face=tf, ambiguous=amb, frags=fr)


# ---- the reference's collaborators, restated for the fixture and the tests ---------------------------------------

class Camera:
    """CameraMine (model/CameraMine.py) as the visibility tests use it: focal_length [N,2], principal_point [N,2],
    R [N,3,3], T [N,3]; `transform_points_screen` through pytorch3d's composed world-to-NDC matrix (SfM perspective K
    built for image_size (W, H), :265-300) and the screen conversion of :104-142; `cam_pos` = -R[0] T[0] (:207-208)."""

    def __init__(self, focal_length, principal_point, R, T, image_size):
        self.focal_length, self.principal_point, self.R, self.T = focal_length, principal_point, R, T
        self.image_size = image_size   # (W, H)

    def to(self, device):
        return Camera(*(t.to(device) for t in (self.focal_length, self.principal_point, self.R, self.T)),
                      self.image_size)

    def cam_pos(self, cam_id=0):
        return -self.R[cam_id].matmul(self.T[cam_id].view(-1, 1)).view(-1)

    def full_matrix(self):
        N = self.R.shape[0]
        W, H = self.image_size
        fx, fy = self.focal_length.unbind(1)
        px, py = self.principal_point.unbind(1)
        fx, fy = fx / (W / 2.0), fy / (H / 2.0)
        px, py = 1. - 1. / W - px / (W / 2.0), 1. - 1. / H - py / (H / 2.0)
        K = fx.new_zeros(N, 4, 4)
        K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2] = fx, fy, px, py
        K[:, 3, 2], K[:, 2, 3] = 1.0, 1.0
        W2V = self.R.new_zeros(N, 4, 4)
        W2V[:, :3, :3], W2V[:, 3, :3], W2V[:, 3, 3] = self.R, self.T, 1.0
        return W2V.bmm(K.transpose(1, 2))

    def transform_points_screen(self, points, image_size, eps=None):
        M = self.full_matrix()
        ph = torch.cat([points, torch.ones_like(points[..., :1])], -1)
        o = ph.bmm(M)
        ndc = o[..., :3] / o[..., 3:]
        w, h = image_size.unbind(1)
        w, h = w.view(-1, 1), h.view(-1, 1)
        return torch.stack(((w - 1.) / 2. - w * ndc[..., 0] / 2., (h - 1.) / 2. - h * ndc[..., 1] / 2., ndc[..., 2]), 2)


class Meshes:
    """pytorch3d's Meshes for meshes of equal size: verts / faces lists."""

    def __init__(self, verts, faces):
        self._v, self._f = list(verts), list(faces)

    def verts_list(self):
        return self._v

    def faces_list(self):
        return self._f

    def verts_padded(self):
        return torch.stack(self._v)

    def verts_packed(self):
        return torch.cat(self._v)

    def faces_packed(self):
        return self._f[0]


def camera_rows(cam):
    """[N,16] float64 {fx, fy, px, py, R, T} of a Camera."""
    N = cam.R.shape[0]
    return torch.cat([cam.focal_length.reshape(N, 2), cam.principal_point.reshape(N, 2), cam.R.reshape(N, 9),
                      cam.T.reshape(N, 3)], 1).double().cpu().numpy()


class OracleMaskRender:
    """`maskRender` whose fragments are raster_oracle's (zbuf rounded to float32), one call per mesh batch."""

    def __init__(self, H, W, cameras):
        self.rasterizer = SimpleNamespace(cameras=cameras, raster_settings=SimpleNamespace(image_size=(H, W)))
        self.H, self.W = H, W

    def __call__(self, meshes):
        v = torch.stack(meshes.verts_list()).detach().double().numpy()
        f = meshes.faces_list()[0].numpy()
        fr = raster_oracle.rasterize(v, f, camera_rows(self.rasterizer.cameras), self.H, self.W)
        zbuf = torch.tensor(fr["zbuf"], dtype=torch.float32)[..., None]
        return None, SimpleNamespace(zbuf=zbuf, pix_to_face=torch.tensor(fr["pix_to_face"])[..., None])


class BodySkin:
    """Stand-in for `deformer.defs[1](x, poses)` and `deform_lbs(x, [poses, trans])`: an element-wise per-frame
    stretch and shift from poses [N,>=6] (and trans [N,3] when given)."""

    def __call__(self, x, poses):
        trans = None
        if isinstance(poses, (list, tuple)):
            poses, trans = poses
        y = x * (1.0 + 0.05 * poses[:, None, 0:3]) + 0.1 * poses[:, None, 3:6]
        return y if trans is None else y + trans[:, None, :]


class GarmentDeformer:
    """Stand-in for `self.deformer(x, [cond, poses], ratio=..., offset_type=...)`: a cond-driven element-wise offset,
    then BodySkin; records the offset_type of each call, like the translator's `offset[garment_name]`."""

    def __init__(self):
        self.defs = [None, BodySkin()]
        self.offset = {}

    def __call__(self, x, conds, ratio=None, offset_type=None):
        cond, poses = conds
        y = x + 0.02 * cond[:, None, 0:3] * x[..., 1:2]
        self.offset[offset_type] = y - x
        return self.defs[1](y, poses)


def uv_sphere(nu, nv, radii, centre):
    """A closed ellipsoid with nu x nv quads split into triangles: (verts [V,3] float32, faces [F,3] int64)."""
    th = np.linspace(0, np.pi, nv + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, nu, endpoint=False)
    t, p = np.meshgrid(th, ph, indexing="ij")
    v = np.stack([np.sin(t) * np.cos(p), np.cos(t), np.sin(t) * np.sin(p)], -1).reshape(-1, 3)
    v = np.concatenate([[[0, 1, 0]], v, [[0, -1, 0]]]) * np.asarray(radii) + np.asarray(centre)
    f = []
    for i in range(nu):
        j = (i + 1) % nu
        f.append([0, 1 + j, 1 + i])
        for r in range(nv - 2):
            a, b, c, d = 1 + r * nu + i, 1 + r * nu + j, 1 + (r + 1) * nu + i, 1 + (r + 1) * nu + j
            f += [[a, b, c], [b, d, c]]
        last = len(v) - 1
        f.append([1 + (nv - 2) * nu + i, 1 + (nv - 2) * nu + j, last])
    return v.astype(np.float32), np.asarray(f, dtype=np.int64)


def tube(nu, nv, radius, y0, y1):
    """An open cylinder around the y axis: (verts, faces)."""
    ys = np.linspace(y0, y1, nv)
    ph = np.linspace(0, 2 * np.pi, nu, endpoint=False)
    y, p = np.meshgrid(ys, ph, indexing="ij")
    v = np.stack([radius * np.cos(p), y, radius * np.sin(p)], -1).reshape(-1, 3)
    f = []
    for r in range(nv - 1):
        for i in range(nu):
            j = (i + 1) % nu
            a, b, c, d = r * nu + i, r * nu + j, (r + 1) * nu + i, (r + 1) * nu + j
            f += [[a, b, c], [b, d, c]]
    return v.astype(np.float32), np.asarray(f, dtype=np.int64)


def rings(radius, ys, P, phase=0.0):
    """Curve points: len(ys) horizontal rings of P points each around the y axis -> [len(ys) * P, 3] float32."""
    ph = np.linspace(0, 2 * np.pi, P, endpoint=False) + phase
    return np.concatenate([np.stack([radius * np.cos(ph), np.full(P, y), radius * np.sin(ph)], 1) for y in ys]
                          ).astype(np.float32)
