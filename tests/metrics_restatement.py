"""Float64 numpy / scipy restatement of the validation metric PSNR_SSIM (reference network/metrics.py:13-79 and
color_map_backward, utils/base_utils.py:496-499), the yardstick of neuray_b200.metrics.

The reference scores SSIM with skimage's structural_similarity(win_size=11, multichannel=True, data_range=255), and skimage
is not installed where these tests run, so no golden could be generated from the unmodified reference.  This module
restates what that call computes: per channel in float64, 11x11 uniform means of x, y, x^2, y^2 and xy
(scipy.ndimage.uniform_filter, as skimage uses), the sample covariance (cov_norm = 121/120), C1 = (0.01*255)^2,
C2 = (0.03*255)^2, the SSIM map averaged with 5 pixels cropped from every side, then the mean over the channels.
PSNR is compute_psnr's: per-channel mean squared error, averaged over the channels, 10 log10(255^2 / mse) (here in
float64; the reference evaluates it in float32).
"""
import math

import numpy as np
from scipy.ndimage import uniform_filter

WIN = 11


def color_map_backward(rgb):
    """reference utils/base_utils.py:496-499 on float32 input."""
    rgb = np.asarray(rgb, np.float32) * np.float32(255)
    return np.clip(rgb, 0, 255).astype(np.uint8)


def margins(h, w, margin_ratio):
    """reference metrics.py:50-51."""
    return int(h * (1 - margin_ratio)) // 2, int(w * (1 - margin_ratio)) // 2


def crop(img, margin_ratio):
    """reference metrics.py:52-53 on an [h,w,3] image."""
    h, w = img.shape[:2]
    mh, mw = margins(h, w, margin_ratio)
    return img[mh:h - mh, mw:w - mw]


def psnr(gt, pr):
    d = gt.reshape(-1, 3).astype(np.float64) - pr.reshape(-1, 3).astype(np.float64)
    mse = float(np.mean(np.mean(d * d, 0)))
    return math.inf if mse == 0 else 10 * math.log10(255 * 255 / mse)


def ssim(gt, pr):
    if gt.shape[0] < WIN or gt.shape[1] < WIN:
        raise ValueError("win_size exceeds image extent")
    cov_norm = WIN * WIN / (WIN * WIN - 1)
    C1, C2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2
    pad = (WIN - 1) // 2
    out = []
    for c in range(3):
        x, y = gt[..., c].astype(np.float64), pr[..., c].astype(np.float64)
        ux, uy = uniform_filter(x, WIN), uniform_filter(y, WIN)
        uxx, uyy, uxy = uniform_filter(x * x, WIN), uniform_filter(y * y, WIN), uniform_filter(x * y, WIN)
        vx, vy, vxy = cov_norm * (uxx - ux * ux), cov_norm * (uyy - uy * uy), cov_norm * (uxy - ux * uy)
        S = ((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux ** 2 + uy ** 2 + C1) * (vx + vy + C2))
        out.append(S[pad:-pad, pad:-pad].mean(dtype=np.float64))
    return float(np.mean(out))


def psnr_ssim(gt, pr, h, w, margin_ratio=1.0):
    """(psnr, ssim) of one prediction; gt and pr hold h*w*3 float32 values in raster order ([1,h*w,3] or [h,w,3])."""
    g = crop(color_map_backward(np.asarray(gt).reshape(h, w, 3)), margin_ratio)
    p = crop(color_map_backward(np.asarray(pr).reshape(h, w, 3)), margin_ratio)
    return psnr(g, p), ssim(g, p)
