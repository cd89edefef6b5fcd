"""Cost of the per-view visibility output (cfg render_visibility) per frame: the bench's black_800 and fern_high frames
(bench.WORKLOADS, bench.model_cfg, seeded weights) rendered in eval with the option off and on, alternating frame by
frame, CUDA events around each whole render after warm-up.  Prints one JSON line: the card name, power limit and SM clocks
read in the same run, and per workload the median frame times (with their range) and the median cost of the option.
usage: python tools/visibility_time.py [frames]"""
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
assert torch.cuda.is_available(), "visibility_time.py measures on a GPU"
dev = torch.device("cuda")


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def render(net, dq, dr):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    with torch.no_grad():
        out = net.render(dict(dq), dict(dr), False)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def spread(v):
    s = sorted(v)
    return {"median": round(s[len(s) // 2], 1), "min": round(s[0], 1), "max": round(s[-1], 1)}


result = {"gpu": torch.cuda.get_device_name(), "power_limit": smi("power.limit"), "sm_clock_max": smi("clocks.max.sm"),
          "frames": frames, "workloads": {}}
for name in ("black_800", "fern_high"):
    wl = bench.WORKLOADS[name]
    que, ref = bench.make_workload(name)
    dq, dr = synthetic.to_device(que, dev), synthetic.to_device(ref, dev)
    cfg = bench.model_cfg(*wl["dn"])
    W = synthetic.make_weights(cfg, seed=0)
    nets = {}
    for arm, on in (("off", False), ("on", True)):
        nets[arm] = renderer.NeuralRayRenderPath(dict(cfg, render_visibility=on))
        nets[arm].load_state_dict(W, strict=True)
        nets[arm].to(dev)
    for net in nets.values():          # warm-up: module loads, workspaces, weight packing
        render(net, dq, dr)
    ms = {arm: [] for arm in nets}
    for _ in range(frames):
        for arm, net in nets.items():
            ms[arm].append(render(net, dq, dr)[0])
    _, out = render(nets["on"], dq, dr)
    assert torch.isfinite(out["visibility_nr"]).all() and torch.isfinite(out["visibility_nr_fine"]).all()
    med = {arm: sorted(t)[len(t) // 2] for arm, t in ms.items()}
    result["workloads"][name] = {"rays": que["coords"].shape[1], "views": wl["rfn"], "samples": list(wl["dn"]),
                                 "sm_clock_now": smi("clocks.sm"),
                                 "frame_ms": {arm: spread(t) for arm, t in ms.items()},
                                 "visibility_cost_ms_median": round(med["on"] - med["off"], 1)}
print(json.dumps(result))
