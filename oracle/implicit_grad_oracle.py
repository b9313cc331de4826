"""TEST INFRASTRUCTURE ONLY -- the float64 NumPy restatement of csrc/surface_grad.cu's recmv_implicit_grad (DESIGN
section 1l), the per-row algebra of `propagateTmpPsGrad` (OptimGarmentNetwork.py:2213-2311) and its per-garment
reductions.

Per row: b = [grad f ; [v]x J] (4 x 3), btb = b^T b, FastMinv's rule (|det btb| < 1e-4: inverse 0, ok False),
r = g btb^-1 b^T (1 x 4), sdf_coef = -r0, def_vec = r[1:4] (-[v]x), ray_grad = r[1:4] [d - c]x.  Per garment: the ok
count and cam_grad = -sum def_vec.  The kernel decides `ok` on a float32 determinant, so `flags` marks the rows whose
float64 |det| lies within FLAG_REL of 1e-4: only there may the two disagree.  `row_bound` is the per-row error bound
the GPU test allows a float32 result: a multiple of float32's unit roundoff times the condition number of btb times
the size of the row's terms."""
import numpy as np

DET_MIN = 1e-4                 # FastMinv/Matrix3x3InvKernels.cu:29-60
FLAG_REL = 1e-3                # |det| within this relative distance of DET_MIN: ok may differ
EPS32 = 2.0 ** -24
BOUND_K = 64.0                 # safety factor of row_bound over cond * eps32 * size


def cross_matrix(v):
    """[n,3] -> [n,3,3] with [v]x w = v x w."""
    v = np.asarray(v, np.float64)
    z = np.zeros(v.shape[0])
    return np.stack([np.stack([z, -v[:, 2], v[:, 1]], 1), np.stack([v[:, 2], z, -v[:, 0]], 1),
                     np.stack([-v[:, 1], v[:, 0], z], 1)], 1)


def minv_rule(m):
    """FastMinv's cofactor inverse in m's own precision: ([n,3,3] inverse, [n] ok); |det| < 1e-4 -> zeros, False."""
    m = np.asarray(m).reshape(-1, 3, 3)
    c = np.empty_like(m)
    c[:, 0, 0] = m[:, 1, 1] * m[:, 2, 2] - m[:, 1, 2] * m[:, 2, 1]
    c[:, 0, 1] = -m[:, 1, 0] * m[:, 2, 2] + m[:, 1, 2] * m[:, 2, 0]
    c[:, 0, 2] = m[:, 1, 0] * m[:, 2, 1] - m[:, 1, 1] * m[:, 2, 0]
    c[:, 1, 0] = -m[:, 0, 1] * m[:, 2, 2] + m[:, 0, 2] * m[:, 2, 1]
    c[:, 1, 1] = m[:, 0, 0] * m[:, 2, 2] - m[:, 0, 2] * m[:, 2, 0]
    c[:, 1, 2] = -m[:, 0, 0] * m[:, 2, 1] + m[:, 0, 1] * m[:, 2, 0]
    c[:, 2, 0] = m[:, 0, 1] * m[:, 1, 2] - m[:, 0, 2] * m[:, 1, 1]
    c[:, 2, 1] = -m[:, 0, 0] * m[:, 1, 2] + m[:, 0, 2] * m[:, 1, 0]
    c[:, 2, 2] = m[:, 0, 0] * m[:, 1, 1] - m[:, 0, 1] * m[:, 1, 0]
    det = m[:, 0, 0] * c[:, 0, 0] + m[:, 0, 1] * c[:, 0, 1] + m[:, 0, 2] * c[:, 0, 2]
    ok = ~(np.abs(det) < DET_MIN)
    safe = np.where(ok, det, np.ones_like(det))
    inv = np.where(ok[:, None, None], np.transpose(c, (0, 2, 1)) / safe[:, None, None], 0)
    return inv.astype(m.dtype), ok


def btb(grad_f_p, jac, rays):
    """(b [n,4,3], b^T b [n,3,3]) in float64."""
    gf = np.asarray(grad_f_p, np.float64)
    a = cross_matrix(rays) @ np.asarray(jac, np.float64).reshape(-1, 3, 3)
    b = np.concatenate([gf[:, None, :], a], 1)
    return b, np.transpose(b, (0, 2, 1)) @ b


def rows(grad_l_p, grad_f_p, jac, rays, d=None, cam_pos=None, dc_f32=True):
    """Per row in float64: dict(sdf_coef [n], def_vec [n,3], ray_grad [n,3] or None, ok [n], det [n], flags [n]).
    d - c is rounded to float32 first, as the kernel forms it (dc_f32=False: in float64, as the reference's float64
    run forms it)."""
    b, m = btb(grad_f_p, jac, rays)
    inv, ok = minv_rule(m)
    det = np.linalg.det(m) if len(m) else np.zeros(0)
    r = (np.asarray(grad_l_p, np.float64)[:, None, :] @ inv @ np.transpose(b, (0, 2, 1)))[:, 0, :]   # [n,4]
    vx = cross_matrix(rays)
    out = {"sdf_coef": -r[:, 0], "def_vec": (r[:, None, 1:] @ -vx)[:, 0, :], "ok": ok, "det": det,
           "flags": np.abs(np.abs(det) - DET_MIN) <= FLAG_REL * DET_MIN, "ray_grad": None}
    if d is not None and cam_pos is not None:
        ft = np.float32 if dc_f32 else np.float64
        dc = (np.asarray(d, ft) - np.asarray(cam_pos, ft).reshape(1, 3)).astype(np.float64)
        out["ray_grad"] = (r[:, None, 1:] @ cross_matrix(dc))[:, 0, :]
    return out


def garments(per_row, offsets):
    """(ok_count [G] int64, cam_grad [G,3] float64) of the rows' ok and def_vec, garment g at [offsets[g], offsets[g+1])."""
    offs = [int(o) for o in offsets]
    cnt = np.array([int(per_row["ok"][a:b].sum()) for a, b in zip(offs, offs[1:])], np.int64)
    cam = np.array([-per_row["def_vec"][a:b].sum(0) if b > a else np.zeros(3) for a, b in zip(offs, offs[1:])])
    return cnt, cam.reshape(-1, 3)


def row_bound(grad_l_p, grad_f_p, jac, rays, d=None, cam_pos=None):
    """Per-row bound ([n]) on the float32 kernel's error in sdf_coef, def_vec and ray_grad of a row that is ok in both:
    BOUND_K eps32 cond(btb) |g| |btb^-1| |b| max(1, |v|, |d - c|), cond = lambda_max / lambda_min of the symmetric
    btb.  Forming btb in float32 perturbs it by ~eps32 |b|^2 relative; the solve amplifies that by cond; |g| |btb^-1|
    |b| bounds |r|; the cross products scale by |v| or |d - c|."""
    b, m = btb(grad_f_p, jac, rays)
    lam = np.linalg.eigvalsh(m) if len(m) else np.zeros((0, 3))
    with np.errstate(over="ignore", divide="ignore"):    # singular rows: an infinite bound (they are not compared)
        lmin = np.maximum(lam[:, 0], 1e-300)
        cond = lam[:, 2] / lmin
        size = np.linalg.norm(np.asarray(grad_l_p, np.float64), axis=1) / lmin * np.sqrt(np.maximum(lam[:, 2], 0))
        scale = np.maximum(1.0, np.linalg.norm(np.asarray(rays, np.float64), axis=1))
        if d is not None and cam_pos is not None:
            dc = np.asarray(d, np.float64) - np.asarray(cam_pos, np.float64).reshape(1, 3)
            scale = np.maximum(scale, np.linalg.norm(dc, axis=1))
        return BOUND_K * EPS32 * cond * size * scale + 1e-30
