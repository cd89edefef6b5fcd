"""Restatements of the reference eval.py's scores, the yardsticks of neuray_b200.eval_metrics.

eval.py scores PSNR and SSIM with TensorFlow (tf.image.psnr / tf.image.ssim, max_val 1) and LPIPS with the lpips package
(LPIPS(net='vgg'), version 0.1).  Neither TensorFlow nor lpips is installed where these tests run, so this module restates
what those calls compute:

* psnr_tf / ssim_tf: float64 numpy / scipy.  Inputs are converted like color_map_forward (float32(v) / 255).  PSNR =
  10 log10(1 / mse) over all h*w*3 values.  SSIM: 11x11 Gaussian window g (x) g (sigma 1.5, g normalised to sum 1), VALID
  region, weighted means, population covariance, c1 = 0.01^2, c2 = 0.03^2, luminance * cs averaged over the region and the
  channels.
* lpips_torch: torch, with torchvision.models.vgg16(weights=None).features[0:30] and lin weights given by the caller, run
  with TF32 off.
"""
import math

import numpy as np
from scipy.ndimage import correlate1d

WIN, SIGMA = 11, 1.5


def color_map_forward(img):
    """reference utils/base_utils.py:492-493."""
    return np.asarray(img).astype(np.float32) / np.float32(255)


def gauss_window():
    i = np.arange(WIN, dtype=np.float64) - (WIN - 1) / 2
    g = np.exp(-i * i / (2 * SIGMA * SIGMA))
    return g / g.sum()


def psnr_tf(gt_u8, pr_u8):
    a, b = color_map_forward(gt_u8).astype(np.float64), color_map_forward(pr_u8).astype(np.float64)
    mse = float(np.mean((a - b) ** 2))
    return math.inf if mse == 0 else 10 * math.log10(1 / mse)


def _valid_filter(x, g):
    """Gaussian-weighted window means over the VALID region of a [h,w,3] float64 image."""
    h = (WIN - 1) // 2
    y = correlate1d(x, g, axis=0, mode="constant")[h:-h]
    return correlate1d(y, g, axis=1, mode="constant")[:, h:-h]


def ssim_tf(gt_u8, pr_u8):
    x, y = color_map_forward(gt_u8).astype(np.float64), color_map_forward(pr_u8).astype(np.float64)
    if x.shape[0] < WIN or x.shape[1] < WIN:
        raise ValueError("images smaller than the 11x11 window")
    g = gauss_window()
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    ux, uy = _valid_filter(x, g), _valid_filter(y, g)
    exy, exxyy = _valid_filter(x * y, g), _valid_filter(x * x + y * y, g)
    num0, den0 = 2 * ux * uy, ux * ux + uy * uy
    luminance = (num0 + c1) / (den0 + c1)
    cs = (2 * exy - num0 + c2) / (exxyy - den0 + c2)
    return float(np.mean(luminance * cs))


# ---- LPIPS-VGG --------------------------------------------------------------------------------------------------------

TAP_ENDS = (4, 9, 16, 23, 30)     # vgg16.features slices ending after relu1_2, relu2_2, relu3_3, relu4_3, relu5_3
SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)


def seeded_weights(seed):
    """A state dict with LpipsVGG's names: torchvision's vgg16(weights=None).features (its own init, biases made non-zero)
    and lin weights, all from `seed`."""
    import torch
    import torchvision
    torch.manual_seed(seed)
    feats = torchvision.models.vgg16(weights=None).features
    sd = {}
    for k, v in feats.state_dict().items():
        sd[f"features.{k}"] = v.clone() if k.endswith("weight") else torch.empty_like(v).uniform_(-0.1, 0.1)
    for k, c in enumerate((64, 128, 256, 512, 512)):
        sd[f"lin{k}.model.1.weight"] = torch.rand(1, c, 1, 1) / c * 4
    return sd


def lpips_torch(sd, gt_u8, pr_u8, device):
    """LPIPS-VGG of one pair or a batch ([n,h,w,3] uint8) in torch with TF32 off: a float64 numpy array [n]."""
    import torch
    import torchvision
    feats = torchvision.models.vgg16(weights=None).features[:30]
    feats.load_state_dict({k[len("features."):]: v for k, v in sd.items() if k.startswith("features.")})
    feats = feats.to(device).eval()
    lins = [sd[f"lin{k}.model.1.weight"].to(device) for k in range(5)]
    shift = torch.tensor(SHIFT, device=device)[None, :, None, None]
    scale = torch.tensor(SCALE, device=device)[None, :, None, None]

    def prep(u8):
        x = torch.from_numpy(color_map_forward(u8)).to(device)
        x = x.reshape(-1, *x.shape[-3:]).permute(0, 3, 1, 2) * 2 - 1
        return (x - shift) / scale

    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            a, b = prep(gt_u8), prep(pr_u8)
            total = 0
            start = 0
            for t, end in enumerate(TAP_ENDS):
                a, b = feats[start:end](a), feats[start:end](b)
                start = end
                na = a / (torch.sqrt((a * a).sum(1, keepdim=True)) + 1e-10)
                nb = b / (torch.sqrt((b * b).sum(1, keepdim=True)) + 1e-10)
                d = torch.nn.functional.conv2d((na - nb) ** 2, lins[t])
                total = total + d.mean([2, 3])[:, 0]
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    return total.double().cpu().numpy()
