"""Validation-metric timing: PSNR_SSIM of one 800x800 frame with two predictions (nr and nr_fine), as every shipped training
config scores each validation image.  GPU: nr_image_metrics (CUDA events around back-to-back launches after warm-up) and the
whole psnr_ssim call including its copy to the host.  CPU: the float64 numpy / scipy restatement of tests/metrics_restatement.py,
standing in for the reference's skimage call.  Prints the card name and power limit with the numbers, one JSON line.
usage: python tools/metrics_time.py [iters]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import metrics_restatement as mr  # noqa: E402
from neuray_b200 import metrics  # noqa: E402

iters = int(sys.argv[1]) if len(sys.argv) > 1 else 200
h = w = 800
rs = np.random.RandomState(0)
yy, xx = np.meshgrid(np.linspace(0, 4, h), np.linspace(0, 4, w), indexing="ij")
gt = (0.5 + 0.45 * np.sin(xx[..., None] + 1.3 * yy[..., None] + np.arange(3))).astype(np.float32)
preds = [(gt + rs.normal(0, s, gt.shape)).astype(np.float32) for s in (0.05, 0.03)]

t0 = time.perf_counter()
cpu_scores = [mr.psnr_ssim(gt, p, h, w) for p in preds]
cpu_ms = (time.perf_counter() - t0) * 1e3

assert torch.cuda.is_available(), "metrics_time.py measures on a GPU"
g = torch.from_numpy(gt).reshape(1, -1, 3).cuda()
ps = [torch.from_numpy(p).reshape(1, -1, 3).cuda() for p in preds]
for _ in range(20):
    metrics.psnr_ssim(g, ps, h, w)
start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
start.record()
for _ in range(iters):
    metrics.image_metrics(g, ps, h, w, 0, 0)
stop.record()
torch.cuda.synchronize()
kernel_ms = start.elapsed_time(stop) / iters
torch.cuda.synchronize()
t0 = time.perf_counter()
for _ in range(iters):
    gpu_scores = metrics.psnr_ssim(g, ps, h, w)
call_ms = (time.perf_counter() - t0) * 1e3 / iters

try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, check=True).stdout.strip()
except (OSError, subprocess.CalledProcessError):
    power = "unknown"
print(json.dumps({"gpu": torch.cuda.get_device_name(), "power_limit": power, "image": f"{h}x{w}", "predictions": len(preds),
                  "gpu_launches_ms": round(kernel_ms, 4), "gpu_psnr_ssim_call_ms": round(call_ms, 4),
                  "cpu_restatement_ms": round(cpu_ms, 1),
                  "max_ssim_diff": max(abs(a[1] - b[1]) for a, b in zip(gpu_scores, cpu_scores)),
                  "max_psnr_diff_db": max(abs(a[0] - b[0]) for a, b in zip(gpu_scores, cpu_scores))}))
