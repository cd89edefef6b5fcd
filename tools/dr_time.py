"""Cost of direct rendering (cfg use_dr_prediction) per frame: the bench's black_800 frame (800x800 query, 8 views, 64+64
samples, bench.model_cfg, seeded weights) rendered in eval with DR off and on, alternating, CUDA events around each whole
render after warm-up.  DR on is run with the SH fit (use_nr_color_for_dr off) and with the NR colours (on).  Prints the card
name and power limit with the median times, one JSON line.
usage: python tools/dr_time.py [frames]"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from neuray_b200 import renderer, synthetic  # noqa: E402

frames = int(sys.argv[1]) if len(sys.argv) > 1 else 5
assert torch.cuda.is_available(), "dr_time.py measures on a GPU"
dev = torch.device("cuda")
wl = bench.WORKLOADS["black_800"]
que, ref = bench.make_workload("black_800")
dq, dr = synthetic.to_device(que, dev), synthetic.to_device(ref, dev)
cfg = bench.model_cfg(*wl["dn"])
W = synthetic.make_weights(cfg, seed=0)
arms = {"dr_off": {}, "dr_sh": {"use_dr_prediction": True}, "dr_nr_color": {"use_dr_prediction": True, "use_nr_color_for_dr": True}}
nets = {}
for name, over in arms.items():
    net = renderer.NeuralRayRenderPath(dict(cfg, **over))
    net.load_state_dict(W, strict=True)
    nets[name] = net.to(dev)


def render(net):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    with torch.no_grad():
        out = net.render(dict(dq), dict(dr), False)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


for net in nets.values():      # warm-up: module loads, workspaces, weight packing
    render(net)
times = {name: [] for name in nets}
for _ in range(frames):
    for name, net in nets.items():
        times[name].append(render(net)[0])
_, out = render(nets["dr_sh"])
assert torch.isfinite(out["pixel_colors_dr"]).all() and torch.isfinite(out["pixel_colors_dr_fine"]).all()
try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    power = "unknown"
med = {name: sorted(t)[len(t) // 2] for name, t in times.items()}
print(json.dumps({"gpu": torch.cuda.get_device_name(), "power_limit": power, "workload": "black_800", "frames": frames,
                  "frame_ms_median": {k: round(v, 1) for k, v in med.items()},
                  "dr_cost_ms": {k: round(med[k] - med["dr_off"], 1) for k in ("dr_sh", "dr_nr_color")},
                  "frame_ms_all": {k: [round(x, 1) for x in v] for k, v in times.items()}}))
