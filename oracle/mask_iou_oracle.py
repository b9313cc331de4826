"""Float64 restatement of `mask_loss`'s ground-truth dilation and soft silhouette IoU (DESIGN section 1m), written from
the definitions (engineer/networks/OptimGarmentNetwork.py:621-629, 941-947):

  g'     = max over the (2r+1)^2 window of gt centred on the pixel, taps outside the image ignored
           (F.max_pool2d(gt, 2r+1, stride 1, padding r));
  I_n    = sum m g',  U_n = sum |m + g' - m g'|  over frame n's pixels;
  L_n    = 1 - I_n / U_n (NaN at U_n = 0, as 0 / 0),  loss = mean_n L_n;
  dL/dm  = -(w / N) (g' U - I s (1 - g')) / U^2,  s = sign(m + g' - m g'), sign(0) = 0 (torch's abs gradient).

Arrays are [N,H,W]; everything is computed in float64.
"""
import numpy as np


def dilate(gt, r):
    """max_pool2d(gt, 2r+1, 1, r) of gt [N,H,W]: every window tap compared directly (no separable shortcut), in the
    input's dtype, so the result can be compared bit for bit."""
    gt = np.asarray(gt)
    N, H, W = gt.shape
    pad = np.full((N, H + 2 * r, W + 2 * r), -np.inf, dtype=gt.dtype)
    pad[:, r:r + H, r:r + W] = gt
    out = np.full_like(gt, -np.inf)
    for dy in range(2 * r + 1):
        for dx in range(2 * r + 1):
            out = np.maximum(out, pad[:, dy:dy + H, dx:dx + W])
    return out


def iou(m, mgt):
    """(I [N], U [N], L [N], loss) in float64 of silhouettes m and dilated masks mgt [N,H,W]."""
    m, g = np.asarray(m, np.float64), np.asarray(mgt, np.float64)
    N = m.shape[0]
    I = (m * g).reshape(N, -1).sum(1)
    U = np.abs(m + g - m * g).reshape(N, -1).sum(1)
    with np.errstate(invalid="ignore", divide="ignore"):
        L = 1.0 - I / U
    return I, U, L, L.mean()


def iou_vjp(m, mgt, w=1.0, IU=None):
    """dL/dm [N,H,W] in float64 of w * loss (the mean over frames of 1 - I / U); IU = (I [N], U [N]) evaluates the
    formula at given sums instead of the float64 ones (where g' U and I s (1 - g') nearly cancel, the result is only
    as good as the sums)."""
    m, g = np.asarray(m, np.float64), np.asarray(mgt, np.float64)
    N = m.shape[0]
    I, U = iou(m, g)[:2] if IU is None else (np.asarray(IU[0], np.float64), np.asarray(IU[1], np.float64))
    s = np.sign(m + g - m * g)
    I, U = I[:, None, None], U[:, None, None]
    with np.errstate(invalid="ignore", divide="ignore"):
        return -(float(w) / N) * (g * U - I * s * (1.0 - g)) / (U * U)
