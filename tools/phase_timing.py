"""Per-phase critical-path timing of the tensor-core point kernel (clock64 stamps, CTA 0, thread 0 of each of the two
compute warp groups).  usage: phase_timing.py [rays]"""
import ctypes as C
import os
import sys

import torch

torch.set_grad_enabled(False)      # inference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from neuray_b200 import _lib, renderer, synthetic  # noqa: E402
from neuray_b200.weights import camera_blocks  # noqa: E402

rays = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
wl = bench.WORKLOADS["black_800"]
w, rfn, (dn_c, dn_f) = wl["scene"]["w"], wl["rfn"], wl["dn"]
cfg = bench.model_cfg(dn_c, dn_f)
que, ref = bench.make_workload("black_800", seed=0)
n = que["coords"].shape[1]
start = (n // 2 // w) * w
que = synthetic.slice_rays(que, start, start + rays)
W = synthetic.make_weights(cfg, seed=0)
net = renderer.NeuralRayRenderPath(cfg)
net.load_state_dict(W, strict=True)
net.cuda()
dq, dr = synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda")
out = net.render_impl(dq, dr, False)          # warm-up, builds caches
depth = renderer.sample_depth(dq["depth_range"], dq["coords"], dn_c, False)[0]
pack = renderer.frame_pack(dr)
wp, wr, pe, wt = renderer.pass_weights(net, False, dn_c, depth.device)
cam, _ = camera_blocks(dq, None)
rec = torch.empty(rays * dn_c * 20, device="cuda")
timing = torch.zeros(64 * 2 * 32, dtype=torch.int64, device="cuda")
p = _lib.NrPassParams()
coords = dq["coords"][0].contiguous()
p.coords, p.que_depth, p.que_cam, p.rn, p.dn = coords.data_ptr(), depth.data_ptr(), cam.data_ptr(), rays, dn_c
p.feat, p.rgb, p.view_params = pack.feat.data_ptr(), pack.rgb.data_ptr(), pack.view_params.data_ptr()
p.rfn, p.h, p.w, p.fh, p.fw = pack.rfn, pack.h, pack.w, pack.fh, pack.fw
p.w_point, p.w_ray, p.pos_enc, p.w_tc = wp.data_ptr(), wr.data_ptr(), pe.data_ptr(), wt.data_ptr()
p.use_vis, p.var_bias, p.point_rec = 0, 0.05, rec.data_ptr()
_lib.check(_lib.lib().nr_point_kernel_timing(C.byref(p), timing.data_ptr(), None), "timing")
torch.cuda.synchronize()
t = timing.cpu().reshape(64, 2, 32)
nm = ["geom+proj", "gather", "RF->A", "dd heads", "hit/vis+pe0", "pe1+nf+raydir", "pool1+base0 per point", "base0 epilogue",
      "base1 (chain entry)", "vis0", "vis2+vis1", "v20+v21", "rgb0+exit", "pool2+geo0 per point", "geo2 (wg0) / blend (wg1) + rec"]
for wg in (0, 1):
    d = (t[4:40, wg, 1:16] - t[4:40, wg, 0:15]).double().mean(0)
    tot = (t[4:40, wg, 15] - t[4:40, wg, 0]).double().mean()
    print(f"warp group {wg}: tile (16 points x 8 views = 128 rows) total {tot:.0f} cycles")
    print("  " + "  ".join(f"{nm[i]}:{d[i]:.0f}" for i in range(15)))
