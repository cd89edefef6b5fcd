"""Timing of eval.py's scores for a folder of 800x800 test views (uint8 ground truths and predictions already decoded).
GPU: psnr_ssim_tf over all pairs in one call and LPIPS-VGG (fp32 = 3xTF32 and tf32 = one TF32 pass), CUDA events around the
calls after warm-up, plus the whole psnr_ssim_tf call with its copy to the host.  CPU: the float64 numpy / scipy restatement
of tests/eval_restatement.py, standing in for eval.py's TensorFlow-on-CPU PSNR / SSIM.  GPU reference point: the torch
restatement of LPIPS-VGG (cuDNN, TF32 off and on).  LPIPS weights are seeded (timing does not depend on their values).
Prints the card name and power limit with the numbers, one JSON line.
usage: python tools/eval_time.py [views] [iters]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torchvision

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import eval_restatement as er  # noqa: E402
from neuray_b200 import encoders, eval_metrics  # noqa: E402

views = int(sys.argv[1]) if len(sys.argv) > 1 else 8
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 5
h = w = 800
rs = np.random.RandomState(0)
yy, xx = np.meshgrid(np.linspace(0, 4, h), np.linspace(0, 4, w), indexing="ij")
base = 127.5 + 110 * np.sin(xx[..., None] + 1.3 * yy[..., None] + np.arange(3))
gt = np.stack([np.clip(base + rs.normal(0, 4, base.shape), 0, 255) for _ in range(views)]).astype(np.uint8)
pr = np.clip(gt + rs.normal(0, 10, gt.shape), 0, 255).astype(np.uint8)

t0 = time.perf_counter()
cpu_scores = [(er.psnr_tf(a, b), er.ssim_tf(a, b)) for a, b in zip(gt, pr)]
cpu_ms = (time.perf_counter() - t0) * 1e3

assert torch.cuda.is_available(), "eval_time.py measures on a GPU"
g, p = torch.from_numpy(gt).cuda(), torch.from_numpy(pr).cuda()
sd = er.seeded_weights(0)
net = eval_metrics.LpipsVGG()
net.load_state_dict(sd)
net.cuda()


def device_ms(fn, n):
    for _ in range(2):
        fn()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(n):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / n


psnr_ssim_ms = device_ms(lambda: eval_metrics.eval_metrics(g, p), 20 * iters)
torch.cuda.synchronize()
t0 = time.perf_counter()
for _ in range(20 * iters):
    gpu_scores = eval_metrics.psnr_ssim_tf(g, p)
call_ms = (time.perf_counter() - t0) * 1e3 / (20 * iters)
lpips_ms = {}
for mode in ("fp32", "tf32"):
    encoders.set_precision(mode)
    lpips_ms[mode] = device_ms(lambda: net(g, p), iters)
encoders.set_precision("fp32")
lp = net(g, p).cpu().numpy()
torch_ms = {}
for tf32 in (False, True):
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = tf32
    feats = torchvision.models.vgg16(weights=None).features[:30].cuda().eval()
    x = torch.rand(2 * views, 3, h, w, device="cuda")
    with torch.no_grad():
        torch_ms["tf32" if tf32 else "fp32"] = device_ms(lambda: feats(x), iters)
    torch.backends.cudnn.allow_tf32 = old
want = er.lpips_torch(sd, gt, pr, "cuda")

try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, check=True).stdout.strip()
except (OSError, subprocess.CalledProcessError):
    power = "unknown"
print(json.dumps({"gpu": torch.cuda.get_device_name(), "power_limit": power, "image": f"{h}x{w}", "views": views,
                  "gpu_psnr_ssim_ms": round(psnr_ssim_ms, 4), "gpu_psnr_ssim_call_ms": round(call_ms, 4),
                  "cpu_restatement_psnr_ssim_ms": round(cpu_ms, 1),
                  "gpu_lpips_ms": {k: round(v, 2) for k, v in lpips_ms.items()},
                  "torch_cudnn_vgg_features_ms": {k: round(v, 2) for k, v in torch_ms.items()},
                  "max_ssim_diff": max(abs(a[1] - b[1]) for a, b in zip(gpu_scores, cpu_scores)),
                  "max_psnr_diff_db": max(abs(a[0] - b[0]) for a, b in zip(gpu_scores, cpu_scores)),
                  "max_lpips_rel_diff": float(np.max(np.abs(lp - want) / np.abs(want)))}))
