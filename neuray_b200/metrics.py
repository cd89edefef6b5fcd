"""Validation metrics on the GPU: reference network/metrics.py:13-79 (PSNR_SSIM, compute_psnr) with skimage's
structural_similarity(win_size=11, multichannel=True, data_range=255).

    psnr_ssim(gt, preds, h, w, margin_ratio)   one ground truth against several predictions in one launch
    image_metrics(...)                          the same on the device, without the copy to the host
    PSNR_SSIM, name2metrics                     the reference's metric class and table, same cfg and output keys

`train/trainer.py` picks `model_best.pth` by `psnr_nr_fine`, so the values follow the reference's definition exactly:
inputs quantised like color_map_backward, the eval_margin_ratio crop, PSNR over the crop, SSIM with uniform 11x11 windows
and the sample covariance.  The arithmetic runs in libneuray_b200.so (csrc/nr_metrics.cu); each call copies one [n,4]
fp64 result to the host.  CUDA tensors only; there is no CPU path.
"""
import ctypes as C
import math

import torch

from . import _lib
from .losses import Loss

MAX_PRED = 8      # NR_METRICS_MAX_PRED


def margins(h, w, margin_ratio):
    """Rows / columns cropped from each side (reference metrics.py:50-51)."""
    return int(h * (1 - margin_ratio)) // 2, int(w * (1 - margin_ratio)) // 2


def _image(t, h, w):
    t = t.detach()
    if t.numel() != h * w * 3:
        raise ValueError(f"an image of {h}x{w}x3 values was expected, got shape {tuple(t.shape)}")
    return t.float().contiguous()


def image_metrics(gt, preds, h, w, margin_h, margin_w):
    """nr_image_metrics, stream-ordered: a CUDA fp64 tensor [len(preds), 4] holding, per prediction, the three per-channel
    sums of squared errors over the crop and the SSIM.  gt and every prediction hold an h x w RGB image in raster order
    ([1,h*w,3] as the renderer returns it, or [h,w,3]) on one CUDA device.  A crop smaller than 11 x 11 raises."""
    preds = list(preds)
    if not 1 <= len(preds) <= MAX_PRED:
        raise ValueError(f"1..{MAX_PRED} predictions per call, got {len(preds)}")
    g = _image(gt, h, w)
    ps = [_image(p, h, w) for p in preds]
    if any(p.device != g.device for p in ps):
        raise ValueError("the ground truth and the predictions must be on one device")
    with _lib.on_device(g):
        ws = torch.empty(max(_lib.lib().nr_image_metrics_workspace(len(ps), h, w, margin_h, margin_w), 1), dtype=torch.uint8, device=g.device)
        out = torch.empty(len(ps), 4, dtype=torch.float64, device=g.device)
        arr = (C.c_void_p * len(ps))(*[_lib.ptr(p) for p in ps])
        _lib.check(_lib.lib().nr_image_metrics(_lib.ptr(g), arr, len(ps), h, w, margin_h, margin_w, _lib.ptr(out), _lib.ptr(ws), ws.numel(),
                                               _lib.stream_of(g)), "nr_image_metrics")
    _lib.count_launches(2)
    return out


def psnr_ssim(gt, preds, h, w, margin_ratio=1.0):
    """PSNR and SSIM of each prediction against `gt`, after the eval_margin_ratio crop: a list of (psnr, ssim) floats in the
    order of `preds` (inputs as for image_metrics).  PSNR is inf for identical images.  One device-to-host copy."""
    mh, mw = margins(h, w, margin_ratio)
    npix = (h - 2 * mh) * (w - 2 * mw)
    scores = []
    for sse_r, sse_g, sse_b, ssim in image_metrics(gt, preds, h, w, mh, mw).cpu().tolist():
        mse = (sse_r / npix + sse_g / npix + sse_b / npix) / 3
        scores.append((math.inf if mse == 0 else 10 * math.log10(255 * 255 / mse), ssim))
    return scores


class PSNR_SSIM(Loss):
    """reference metrics.py:29-79.  Returns psnr_nr / ssim_nr and, for each of the dr, nr_fine and dr_fine renderings
    present in data_pr, psnr_* / ssim_*: CPU float32 tensors of shape [1].  Every prediction gets the eval_margin_ratio
    crop; the reference crops only the ground truth and pixel_colors_nr, so for a ratio below 1 its other renderings
    fail on mismatched shapes."""
    default_cfg = {"eval_margin_ratio": 1.0}

    def __init__(self, cfg):
        super().__init__([])
        self.cfg = {**self.default_cfg, **cfg}

    def __call__(self, data_pr, data_gt, step, **kwargs):
        info = data_gt["que_imgs_info"] if "que_imgs_info" in data_gt else data_pr["que_imgs_info"]
        h, w = info["imgs"].shape[2:]
        suffixes = ["nr"] + [s for s in ("dr", "nr_fine", "dr_fine") if f"pixel_colors_{s}" in data_pr]
        scores = psnr_ssim(data_pr["pixel_colors_gt"], [data_pr[f"pixel_colors_{s}"] for s in suffixes], h, w,
                           self.cfg["eval_margin_ratio"])
        outputs = {}
        for s, (psnr, ssim) in zip(suffixes, scores):
            outputs[f"psnr_{s}"] = torch.tensor([psnr], dtype=torch.float32)
            outputs[f"ssim_{s}"] = torch.tensor([ssim], dtype=torch.float32)
        return outputs


name2metrics = {"psnr_ssim": PSNR_SSIM}
