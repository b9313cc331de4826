"""Float64 brute-force restatement of the mesh rasterizer's semantics (DESIGN section 1b), written from the definitions,
not from any rasterizer's code: every face is tested against every pixel centre in its screen bbox.

Camera (model/CameraMine.py): view X_v = X R + T (:169-173), screen (sx, sy) = (px - fx X_v/Z_v, py - fy Y_v/Z_v)
(:104-142, :273-287), pixel (row, col) centred at (col, row).  A face is skipped when a vertex has Z_v <= z_clip or its
doubled screen area |A| <= area_eps; it covers a pixel when its three barycentrics (edge functions over A) are >= 0
and the perspective denominator sum_j b_j / Z_j is > 0 (the interpolated point lies in front of the camera plane; only
a face with a vertex at Z <= 0, which needs z_clip < 0, can fail this);
b'_i = (b_i/Z_i) / sum_j (b_j/Z_j), zbuf = sum_i b'_i Z_i; the smallest zbuf wins, ties to the lower packed index
n*F + f; dists = -(squared distance to the nearest edge) in NDC x = 1 - (2 sx + 1)/W, y = 1 - (2 sy + 1)/H.

Besides the fragments it reports, per pixel, whether the decision is AMBIGUOUS at a given precision: some face's pixel
centre lies within `margin_px` pixels of one of its edges (inside or out), or the runner-up's zbuf is within
`ztol * zbuf` of the winner's; and whether there was an exact z-tie.
"""
import numpy as np


def camera_tuple(cam):
    """(fx, fy, px, py, R [3,3], T [3]) as float64 numpy from a 16-vector or a tuple."""
    c = np.asarray(cam, dtype=np.float64).reshape(-1)
    return c[0], c[1], c[2], c[3], c[4:13].reshape(3, 3), c[13:16]


def project(verts, cam):
    fx, fy, px, py, R, T = camera_tuple(cam)
    v = np.asarray(verts, dtype=np.float64) @ R + T
    with np.errstate(divide="ignore", invalid="ignore"):
        return px - fx * v[:, 0] / v[:, 2], py - fy * v[:, 1] / v[:, 2], v[:, 2]


def cam_pos(cam):
    """CameraMine.cam_pos (:207-208): -R T."""
    _, _, _, _, R, T = camera_tuple(cam)
    return -R @ T


def view_rays(cols, rows, cam):
    """CameraMine.view_rays (:146-167) with ps = (col, row, 1), in float64."""
    fx, fy, px, py, R, _ = camera_tuple(cam)
    r = np.stack([-cols / fx + px / fx, -rows / fy + py / fy, np.ones_like(cols, dtype=np.float64)], 1)
    r = r / np.linalg.norm(r, axis=1, keepdims=True)
    return r @ R.T


def _frame(verts, faces, cam, H, W, z_clip, area_eps, margin_px, ztol, face_base, chunk=4_000_000):
    sx, sy, z = project(verts, cam)
    F = faces.shape[0]
    x = sx[faces]; y = sy[faces]; zz = z[faces]                          # [F,3]
    with np.errstate(invalid="ignore"):
        A = (x[:, 1] - x[:, 0]) * (y[:, 2] - y[:, 0]) - (y[:, 1] - y[:, 0]) * (x[:, 2] - x[:, 0])
        keep = (zz > z_clip).all(1) & (np.abs(A) > area_eps)
    skipped = int(F - keep.sum())
    # faces whose skip decision fp32 could flip: screen positions good to ~4 units in the last place of an fp32
    # coordinate, which moves the area by that much times the perimeter; depths good to a relative 1e-6
    with np.errstate(invalid="ignore"):
        per = sum(np.hypot(x[:, i] - x[:, (i + 1) % 3], y[:, i] - y[:, (i + 1) % 3]) for i in range(3))
        cp = 4 * 2.0 ** -24 * np.maximum(np.abs(x).max(1), np.abs(y).max(1)) + 1e-9
        skip_amb = int(((np.abs(np.abs(A) - area_eps) <= 2 * cp * per)
                        | (np.abs(zz - z_clip) <= 1e-6 * np.abs(zz)).any(1)).sum())
    lo_x = np.ceil(np.clip(np.nan_to_num(x.min(1), nan=1e30), -1, W)).astype(np.int64)
    hi_x = np.floor(np.clip(np.nan_to_num(x.max(1), nan=-1e30), -1, W)).astype(np.int64)
    lo_y = np.ceil(np.clip(np.nan_to_num(y.min(1), nan=1e30), -1, H)).astype(np.int64)
    hi_y = np.floor(np.clip(np.nan_to_num(y.max(1), nan=-1e30), -1, H)).astype(np.int64)
    lo_x = np.maximum(lo_x, 0); lo_y = np.maximum(lo_y, 0)
    hi_x = np.minimum(hi_x, W - 1); hi_y = np.minimum(hi_y, H - 1)
    # the margin band reaches one pixel beyond the bbox at most (margin_px < 1)
    bx0, bx1 = np.maximum(lo_x - 1, 0), np.minimum(hi_x + 1, W - 1)
    by0, by1 = np.maximum(lo_y - 1, 0), np.minimum(hi_y + 1, H - 1)
    nx, ny = np.maximum(bx1 - bx0 + 1, 0), np.maximum(by1 - by0 + 1, 0)
    cnt = np.where(keep, nx * ny, 0)
    npix = H * W
    best_z = np.full(npix, np.inf)
    best_f = np.full(npix, -1, dtype=np.int64)
    second_z = np.full(npix, np.inf)
    tie = np.zeros(npix, dtype=bool)
    amb = np.zeros(npix, dtype=bool)
    cover_list = []
    fids = np.nonzero(cnt)[0]
    csum = np.cumsum(cnt[fids])
    start = 0
    while start < len(fids):
        stop = int(np.searchsorted(csum, (csum[start - 1] if start else 0) + chunk, side="right"))
        stop = max(stop, start + 1)
        fs = fids[start:stop]
        c = cnt[fs]
        f = np.repeat(fs, c)
        k = np.arange(c.sum()) - np.repeat(np.cumsum(c) - c, c)
        col = bx0[f] + k % nx[f]
        row = by0[f] + k // nx[f]
        X, Y = x[f], y[f]
        b = np.empty((len(f), 3))
        d = np.empty((len(f), 3))
        for i in range(3):
            a, bb = (i + 1) % 3, (i + 2) % 3
            e = (X[:, bb] - X[:, a]) * (row - Y[:, a]) - (Y[:, bb] - Y[:, a]) * (col - X[:, a])
            b[:, i] = e / A[f]
            d[:, i] = b[:, i] * np.abs(A[f]) / np.hypot(X[:, bb] - X[:, a], Y[:, bb] - Y[:, a])   # signed px distance
        pix = row * W + col
        inb = (col >= lo_x[f]) & (col <= hi_x[f]) & (row >= lo_y[f]) & (row <= hi_y[f])
        with np.errstate(divide="ignore", invalid="ignore"):
            covered = (b >= 0).all(1) & inb & ((b / zz[f]).sum(1) > 0)
        dmin = d.min(1)
        amb[pix[(d > -margin_px).all(1) & (dmin < margin_px)]] = True   # coverage could flip
        f, pix, b = f[covered], pix[covered], b[covered]
        w = b / zz[f]
        bp = w / w.sum(1, keepdims=True)
        zb = (bp * zz[f]).sum(1)
        cover_list.append((pix, f, zb))
        start = stop
    if cover_list:
        pix = np.concatenate([c[0] for c in cover_list])
        f = np.concatenate([c[1] for c in cover_list])
        zb = np.concatenate([c[2] for c in cover_list])
        o = np.lexsort((f, zb, pix))
        pix, f, zb = pix[o], f[o], zb[o]
        first = np.ones(len(pix), dtype=bool)
        first[1:] = pix[1:] != pix[:-1]
        best_z[pix[first]] = zb[first]
        best_f[pix[first]] = f[first]
        sec = np.zeros(len(pix), dtype=bool)
        sec[1:] = (~first[1:]) & first[:-1]
        second_z[pix[sec]] = zb[sec]
    hit = best_f >= 0
    with np.errstate(invalid="ignore"):
        tie = hit & (second_z == best_z)
        amb_z = hit & (second_z - best_z <= ztol * np.abs(best_z))
    amb |= amb_z
    # outputs of the winners
    p2f = np.where(hit, best_f + face_base, -1)
    zbuf = np.where(hit, best_z, -1.0)
    bary = -np.ones((npix, 3))
    dists = -np.ones(npix)
    hp = np.nonzero(hit)[0]
    if len(hp):
        f = best_f[hp]
        col, row = (hp % W).astype(np.float64), (hp // W).astype(np.float64)
        X, Y = x[f], y[f]
        b = np.empty((len(f), 3))
        for i in range(3):
            a, bb = (i + 1) % 3, (i + 2) % 3
            b[:, i] = ((X[:, bb] - X[:, a]) * (row - Y[:, a]) - (Y[:, bb] - Y[:, a]) * (col - X[:, a])) / A[f]
        w = b / zz[f]
        bary[hp] = w / w.sum(1, keepdims=True)
        nxv, nyv = 1 - (2 * X + 1) / W, 1 - (2 * Y + 1) / H
        qx, qy = 1 - (2 * col + 1) / W, 1 - (2 * row + 1) / H
        dm = np.full(len(f), np.inf)
        for i in range(3):
            ax, ay, bx, by = nxv[:, i], nyv[:, i], nxv[:, (i + 1) % 3], nyv[:, (i + 1) % 3]
            ux, uy, wx, wy = bx - ax, by - ay, qx - ax, qy - ay
            l2 = ux * ux + uy * uy
            s = np.clip(np.where(l2 > 0, (wx * ux + wy * uy) / np.where(l2 > 0, l2, 1), 0), 0, 1)
            dm = np.minimum(dm, (wx - s * ux) ** 2 + (wy - s * uy) ** 2)
        dists[hp] = -dm
    return dict(pix_to_face=p2f.reshape(H, W), zbuf=zbuf.reshape(H, W), bary=bary.reshape(H, W, 3),
                dists=dists.reshape(H, W), ambiguous=amb.reshape(H, W), ambiguous_z=amb_z.reshape(H, W), tie=tie.reshape(H, W), skipped=skipped,
                skipped_ambiguous=skip_amb)


def rasterize(verts, faces, cams, H, W, z_clip=1e-6, area_eps=1e-8, margin_px=0.0, ztol=0.0):
    """verts [N,V,3], faces [F,3], cams [N,16] (or N tuples) -> dict of numpy arrays: pix_to_face [N,H,W] int64 (packed),
    zbuf [N,H,W], bary [N,H,W,3], dists [N,H,W], ambiguous [N,H,W] bool, tie [N,H,W] bool, skipped (int, all frames),
    skipped_ambiguous (faces whose skip decision lies within the margins)."""
    verts = np.asarray(verts, dtype=np.float64)
    faces = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    N, F = verts.shape[0], faces.shape[0]
    outs = [_frame(verts[n], faces, cams[n], H, W, z_clip, area_eps, margin_px, ztol, n * F) for n in range(N)]
    res = {k: np.stack([o[k] for o in outs]) for k in outs[0] if not k.startswith("skipped")} if N else {}
    res["skipped"] = sum(o["skipped"] for o in outs)
    res["skipped_ambiguous"] = sum(o["skipped_ambiguous"] for o in outs)
    return res


def seed_points(verts, faces, p2f, bary):
    """World-space barycentric point sum_i b'_i X_i of every covered pixel: [N,H,W,3] (NaN on background)."""
    verts = np.asarray(verts, dtype=np.float64)
    faces = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    N, F = verts.shape[0], max(faces.shape[0], 1)
    out = np.full(p2f.shape + (3,), np.nan)
    for n in range(N):
        m = p2f[n] >= 0
        f = p2f[n][m] % F
        out[n][m] = (verts[n][faces[f]] * bary[n][m][:, :, None]).sum(1)
    return out
