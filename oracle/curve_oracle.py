"""Float64 NumPy restatement of the feature-curve pieces of `project_2d_loss` (DESIGN section 1n):
  * the learnable curve and its regulariser (Intersect_Free_Curve.forward / regularization,
    engineer/utils/garment_structure.py:109-145) with torch's derivative rules at the kinks;
  * CameraMine's `transform_points_screen` with its Jacobian in the world point;
  * the per-(curve, frame) stable compaction of the visible screen points that `utils.fl_proj_loss` builds.

Curve: v = c + d * s0 * relu(scale) + t * nx, per curve c [3], d [S,3], s0 [S], nx [3], scale, t [S].
Regulariser per curve: e_i = v_a(i) - v_b(i) for i = 0..S (i < S-1: (i, i+1); S-1: (S-1, 0); S: (0, 1)),
u_i = e_i / (|e_i| + 1e-6); diff_c = sum_{i<S} (1 - cos(u_i, u_{i+1})) with torch's cosine_similarity
(each side divided by its norm clamped at 1e-8, the clamp invisible to autograd); centre_c = sum_j |mean_s v_sj - c_j|.
Derivatives as torch takes them: relu'(0) = 0, d|e|/de = 0 at e = 0, sign(0) = 0 for |.|."""
import numpy as np

EPS_NORM = 1e-6
EPS_COS = 1e-8


def curve_points(center, dirs, init_scale, nx, scale, nx_scale):
    """[C,S,3] curve points from center [C,3], dirs [C,S,3], init_scale [C,S], nx [C,3], scale, nx_scale [C,S]."""
    center, dirs, init_scale, nx, scale, nx_scale = (np.asarray(a, dtype=np.float64) for a in
                                                     (center, dirs, init_scale, nx, scale, nx_scale))
    return (center[:, None, :] + dirs * (init_scale * np.maximum(scale, 0.0))[..., None]
            + nx_scale[..., None] * nx[:, None, :])


def _edges(v):
    e = np.concatenate([v[:, :-1] - v[:, 1:], v[:, -1:] - v[:, :1], v[:, :1] - v[:, 1:2]], 1)   # [C,S+1,3]
    n = np.linalg.norm(e, axis=-1, keepdims=True)
    return e, n


def regularizer(v, center):
    """(diff [C], centre [C]) of the curve points v [C,S,3] and the centres [C,3]."""
    v = np.asarray(v, dtype=np.float64)
    e, n = _edges(v)
    u = e / (n + EPS_NORM)
    a, b = u[:, :-1], u[:, 1:]
    na = np.maximum(np.linalg.norm(a, axis=-1, keepdims=True), EPS_COS)
    nb = np.maximum(np.linalg.norm(b, axis=-1, keepdims=True), EPS_COS)
    cos = ((a / na) * (b / nb)).sum(-1)
    centre = np.abs(v.mean(1) - np.asarray(center, dtype=np.float64)).sum(-1)
    return (1.0 - cos).sum(-1), centre


def regularizer_vjp(v, center, g_diff, g_centre):
    """dv [C,S,3] of g_diff [C] . diff + g_centre [C] . centre under torch's rules."""
    v = np.asarray(v, dtype=np.float64)
    C, S, _ = v.shape
    e, n = _edges(v)
    q = n + EPS_NORM
    u = e / q
    a, b = u[:, :-1], u[:, 1:]
    na_raw = np.linalg.norm(a, axis=-1, keepdims=True)
    nb_raw = np.linalg.norm(b, axis=-1, keepdims=True)
    na, nb = np.maximum(na_raw, EPS_COS), np.maximum(nb_raw, EPS_COS)
    dot = (a * b).sum(-1, keepdims=True)
    gcos = -np.asarray(g_diff, dtype=np.float64)[:, None, None]
    # cos = (a / na) . (b / nb): direct terms, then through the (unclamped) norms; d|x|/dx = 0 at x = 0
    ua = np.where(na_raw > 0, a / np.where(na_raw > 0, na_raw, 1.0), 0.0)
    ub = np.where(nb_raw > 0, b / np.where(nb_raw > 0, nb_raw, 1.0), 0.0)
    ga = gcos * (b / (na * nb) - dot / (na * na * nb) * ua)
    gb = gcos * (a / (na * nb) - dot / (na * nb * nb) * ub)
    gu = np.zeros_like(u)
    gu[:, :-1] += ga
    gu[:, 1:] += gb
    ue = np.where(n > 0, e / np.where(n > 0, n, 1.0), 0.0)
    ge = gu / q - (gu * e).sum(-1, keepdims=True) / (q * q) * ue
    gv = np.zeros_like(v)
    gv[:, :-1] += ge[:, :S - 1]
    gv[:, 1:] -= ge[:, :S - 1]
    gv[:, S - 1] += ge[:, S - 1]
    gv[:, 0] -= ge[:, S - 1]
    gv[:, 0] += ge[:, S]
    gv[:, 1] -= ge[:, S]
    sgn = np.sign(v.mean(1) - np.asarray(center, dtype=np.float64))
    gv += (np.asarray(g_centre, dtype=np.float64)[:, None] * sgn / S)[:, None, :]
    return gv


def curve_vjp(dirs, init_scale, nx, scale, dv):
    """(dscale, dnx_scale) [C,S] of the total upstream dv [C,S,3] through curve_points."""
    dirs, init_scale, nx, scale, dv = (np.asarray(x, dtype=np.float64) for x in (dirs, init_scale, nx, scale, dv))
    dscale = np.where(scale > 0, init_scale * (dirs * dv).sum(-1), 0.0)
    return dscale, (nx[:, None, :] * dv).sum(-1)


def screen(points, cams, W, H):
    """transform_points_screen of points [N,P,3] under camera rows cams [N,16] {fx, fy, px, py, R, T} (pixels) for an
    image W x H: pytorch3d's SfM K for image_size (W, H), ndc = (fx' X/Z + px', fy' Y/Z + py', 1/Z) with view
    (X, Y, Z) = p R + T, then ((W-1)/2 - W ndc_x / 2, (H-1)/2 - H ndc_y / 2, ndc_z).  Returns [N,P,3]."""
    p = np.asarray(points, dtype=np.float64)
    c = np.asarray(cams, dtype=np.float64)
    R, T = c[:, 4:13].reshape(-1, 3, 3), c[:, 13:16]
    v = np.einsum("npk,nkj->npj", p, R) + T[:, None]
    fx, fy = c[:, 0:1] / (W / 2.0), c[:, 1:2] / (H / 2.0)
    px, py = 1.0 - 1.0 / W - c[:, 2:3] / (W / 2.0), 1.0 - 1.0 / H - c[:, 3:4] / (H / 2.0)
    ndc = np.stack([fx * v[..., 0] / v[..., 2] + px, fy * v[..., 1] / v[..., 2] + py, 1.0 / v[..., 2]], -1)
    return np.stack([(W - 1.0) / 2.0 - W * ndc[..., 0] / 2.0, (H - 1.0) / 2.0 - H * ndc[..., 1] / 2.0, ndc[..., 2]],
                    -1)


def screen_vjp(points, cams, W, H, dxy):
    """d points [N,P,3] of dxy [N,P,2] . (screen x, screen y)."""
    p = np.asarray(points, dtype=np.float64)
    c = np.asarray(cams, dtype=np.float64)
    R, T = c[:, 4:13].reshape(-1, 3, 3), c[:, 13:16]
    v = np.einsum("npk,nkj->npj", p, R) + T[:, None]
    fx, fy = c[:, 0:1], c[:, 1:2]          # (W/2) fx' = fx: the screen scale of the NDC focal length
    dxy = np.asarray(dxy, dtype=np.float64)
    z = v[..., 2]
    gv = np.stack([-fx * dxy[..., 0] / z, -fy * dxy[..., 1] / z,
                   (fx * v[..., 0] * dxy[..., 0] + fy * v[..., 1] * dxy[..., 1]) / (z * z)], -1)
    return np.einsum("npj,nkj->npk", gv, R)


def compact(xy, visible):
    """fl_proj_loss's compaction: xy [B,P,2], visible [B,P] bool -> (clouds [B,P,2] with each cloud's visible points
    first in their order and zeros after, counts [B])."""
    xy = np.asarray(xy)
    visible = np.asarray(visible, dtype=bool)
    out = np.zeros_like(xy)
    counts = visible.sum(1)
    for b in range(xy.shape[0]):
        out[b, :counts[b]] = xy[b, visible[b]]
    return out, counts
