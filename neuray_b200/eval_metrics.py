"""The scores of the reference's eval.py on the GPU: PSNR and SSIM as TensorFlow defines them, and LPIPS-VGG.

    psnr_ssim_tf(gt_u8, pr_u8)     tf.image.psnr / tf.image.ssim (max_val 1) of uint8 pairs, one launch for all pairs
    eval_metrics(gt_u8, pr_u8)     the same on the device: a CUDA fp64 tensor [n, 2] (psnr, ssim)
    LpipsVGG                       lpips.LPIPS(net='vgg') (version 0.1), state dict named like torchvision's vgg16().features.*
                                   and lpips's lin{0..4}.model.1.weight; LpipsVGG.from_files loads both from local files
    lpips(gt_u8, pr_u8, net)       LPIPS-VGG of uint8 pairs, called as eval.py calls it (on color_map_forward(x) * 2 - 1)

Images are uint8 [h,w,3] (one pair) or [n,h,w,3] (n pairs of one size), torch tensors or numpy arrays; host inputs are
copied to the GPU.  The arithmetic runs in libneuray_b200.so (csrc/nr_metrics.cu): PSNR / SSIM in fp64 with Gaussian 11x11
windows over the VALID region and the population covariance, LPIPS's 13 convolutions on nr_conv2d_nhwc with the encoders'
precision (encoders.set_precision).  These are eval.py's conventions, not the skimage ones of neuray_b200.metrics.
"""
import ctypes as C

import numpy as np
import torch
from torch import nn

from . import _lib, encoders

VGG_CONVS = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)     # torchvision vgg16().features indices of features[0:30]'s convs
VGG_CHANNELS = ((3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 512), (512, 512), (512, 512),
                (512, 512), (512, 512), (512, 512))
TAP_CHANNELS = (64, 128, 256, 512, 512)
LPIPS_LAUNCHES = 1 + 34 + 13 + 5 + 4 + 1       # input, conv slices, ReLUs, taps, pools, finish
WORKSPACE_BUDGET = 2 << 30                     # bytes of LPIPS workspace one call may take; larger batches are split


def _pairs(gt, pr, device=None):
    """gt, pr -> two contiguous CUDA uint8 [n,h,w,3] tensors on `device` (default: the current CUDA device)."""
    gt, pr = torch.as_tensor(gt), torch.as_tensor(pr)
    if gt.dtype != torch.uint8 or pr.dtype != torch.uint8:
        raise ValueError(f"uint8 images expected, got {gt.dtype} and {pr.dtype}")
    if gt.shape != pr.shape or gt.dim() not in (3, 4) or gt.shape[-1] != 3:
        raise ValueError(f"pairs of [h,w,3] or [n,h,w,3] images of one shape expected, got {tuple(gt.shape)} and {tuple(pr.shape)}")
    if gt.dim() == 3:
        gt, pr = gt[None], pr[None]
    if device is None:
        device = gt.device if gt.is_cuda else torch.device("cuda", torch.cuda.current_device())
    return gt.to(device).contiguous(), pr.to(device).contiguous()


def eval_metrics(gt_u8, pr_u8):
    """nr_eval_metrics, stream-ordered: a CUDA fp64 tensor [n, 2] of (psnr, ssim) per pair.  Images smaller than 11 x 11
    raise."""
    g, p = _pairs(gt_u8, pr_u8)
    n, h, w, _ = g.shape
    with _lib.on_device(g):
        nbytes = _lib.lib().nr_eval_metrics_workspace(n, h, w)
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=g.device)
        out = torch.empty(n, 2, dtype=torch.float64, device=g.device)
        _lib.check(_lib.lib().nr_eval_metrics(_lib.ptr(g), _lib.ptr(p), n, h, w, _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream_of(g)),
                   "nr_eval_metrics")
    _lib.count_launches(2)
    return out


def psnr_ssim_tf(gt_u8, pr_u8):
    """[(psnr, ssim)] per pair, as eval.py computes them with tf.image.psnr / tf.image.ssim (max_val 1) on
    color_map_forward'ed images.  PSNR is inf for identical images.  One device-to-host copy."""
    return [tuple(r) for r in eval_metrics(gt_u8, pr_u8).cpu().tolist()]


class _Node(nn.Module):
    pass


class LpipsVGG(nn.Module):
    """lpips.LPIPS(net='vgg', version='0.1') in inference.  Parameters: features.{i}.weight / bias for the 13 convolutions of
    torchvision's vgg16().features[0:30] and lin{k}.model.1.weight ([1,C,1,1], no bias) for the five taps.  Move it to a CUDA
    device before scoring; the forward runs in libneuray_b200.so."""

    def __init__(self):
        super().__init__()
        self.features = _Node()
        for i, (cin, cout) in zip(VGG_CONVS, VGG_CHANNELS):
            conv = _Node()
            conv.weight = nn.Parameter(torch.zeros(cout, cin, 3, 3), requires_grad=False)
            conv.bias = nn.Parameter(torch.zeros(cout), requires_grad=False)
            self.features.add_module(str(i), conv)
        for k, c in enumerate(TAP_CHANNELS):
            lin, model, conv = _Node(), _Node(), _Node()
            conv.weight = nn.Parameter(torch.zeros(1, c, 1, 1), requires_grad=False)
            model.add_module("1", conv)
            lin.add_module("model", model)
            self.add_module(f"lin{k}", lin)

    @classmethod
    def from_files(cls, vgg16_path, lin_path):
        """Weights the user already has: torchvision's vgg16 state dict (its features.* entries are used, the classifier is
        ignored) and lpips's weights/v0.1/vgg.pth.  Nothing is downloaded."""
        net = cls()
        vgg = torch.load(vgg16_path, map_location="cpu", weights_only=True)
        lin = torch.load(lin_path, map_location="cpu", weights_only=True)
        sd = {k: v for k, v in vgg.items() if k.startswith("features.")}
        sd.update({k: v for k, v in lin.items() if k.startswith("lin")})
        net.load_state_dict(sd, strict=True)
        return net

    def param_names(self):
        return [f"features.{i}.{s}" for i in VGG_CONVS for s in ("weight", "bias")] + [f"lin{k}.model.1.weight" for k in range(5)]

    def _packed(self, dev):
        sd = dict(self.named_parameters())
        params = [sd[n] for n in self.param_names()]
        stamp = tuple((p.data_ptr(), p._version) for p in params) + (str(dev),)
        hit = self.__dict__.get("_nr_pack")
        if hit is None or hit[0] != stamp:
            n_tensors, n_floats = C.c_int(), C.c_longlong()
            _lib.check(_lib.lib().nr_lpips_vgg_layout(C.byref(n_tensors), C.byref(n_floats)), "nr_lpips_vgg_layout")
            keep = [p.detach().contiguous().float() for p in params]
            ptrs = (C.c_void_p * len(keep))(*[t.data_ptr() for t in keep])
            out = torch.empty(n_floats.value, dtype=torch.float32, device=dev)
            with torch.cuda.device(dev):
                _lib.check(_lib.lib().nr_lpips_vgg_pack(ptrs, len(keep), _lib.ptr(out), torch.cuda.current_stream(dev).cuda_stream),
                           "nr_lpips_vgg_pack")
            _lib.count_launches(1)
            hit = (stamp, out)
            self.__dict__["_nr_pack"] = hit
        return hit[1]

    @torch.no_grad()
    def forward(self, gt_u8, pr_u8):
        """A CUDA fp64 tensor [n] of LPIPS per pair (stream-ordered).  Pairs are scored in batches whose workspace stays
        under WORKSPACE_BUDGET bytes."""
        dev = self.features._modules["0"].weight.device
        if dev.type != "cuda":
            raise _lib.NeurayB200Error("LpipsVGG runs on the GPU: move the module to a CUDA device first (no CPU fallback)")
        g, p = _pairs(gt_u8, pr_u8, dev)
        n, h, w, _ = g.shape
        packed = self._packed(dev)
        per_pair = _lib.lib().nr_lpips_vgg_workspace(1, h, w)
        if per_pair <= 0:
            raise _lib.NeurayB200Error(f"LPIPS-VGG needs images of at least 32 x 32, got {h} x {w}")
        batch = max(1, min(n, WORKSPACE_BUDGET // per_pair))
        out = torch.empty(n, dtype=torch.float64, device=dev)
        nbytes = _lib.lib().nr_lpips_vgg_workspace(batch, h, w)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        tf32x1 = int(encoders.PRECISION == "tf32")
        with _lib.on_device(g):
            for i in range(0, n, batch):
                b = min(batch, n - i)
                _lib.check(_lib.lib().nr_lpips_vgg_fwd(_lib.ptr(packed), _lib.ptr(g[i:i + b]), _lib.ptr(p[i:i + b]), b, h, w, _lib.ptr(out[i:i + b]),
                                                       tf32x1, _lib.ptr(ws), nbytes, _lib.stream_of(g)), "nr_lpips_vgg_fwd")
                _lib.count_launches(LPIPS_LAUNCHES)
        return out


def lpips(gt_u8, pr_u8, net):
    """[lpips] per pair: `net` (an LpipsVGG on a CUDA device) on color_map_forward(x) * 2 - 1 of both images, as eval.py
    scores them.  One device-to-host copy."""
    return net(gt_u8, pr_u8).cpu().tolist()


def read_rgb(path):
    """An image file as uint8 [h,w,3] RGB, as skimage.io.imread gives a colour JPEG."""
    from PIL import Image
    with Image.open(path) as im:
        return np.asarray(im.convert("RGB"), dtype=np.uint8)
