"""Speed of the point kernel's TF32 render mode (renderer.set_precision("tf32")) against the default fp32 (3xTF32) mode:
the bench's black_800 and fern_high frames (bench.WORKLOADS, bench.model_cfg, seeded weights) rendered in eval, the two
modes alternating frame by frame, CUDA events around each whole render after warm-up.  Prints one JSON line: the card
name, power limit and SM clocks read in the same run, and per workload and mode the median ray-samples/s with its range.
With --point-kernel, _lib.PROFILE also times the point kernel alone (events around each point-kernel launch).
usage: python tools/tf32_time.py [frames] [--point-kernel]"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from neuray_b200 import _lib, renderer, synthetic  # noqa: E402

args = [a for a in sys.argv[1:] if not a.startswith("--")]
frames = int(args[0]) if args else 5
point_kernel = "--point-kernel" in sys.argv
assert torch.cuda.is_available(), "tf32_time.py measures on a GPU"
dev = torch.device("cuda")


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def render(net, dq, dr, mode):
    renderer.set_precision(mode)
    if point_kernel:
        _lib.PROFILE = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    with torch.no_grad():
        out = net.render(dict(dq), dict(dr), False)
    e1.record()
    torch.cuda.synchronize()
    pk = sum(a.elapsed_time(b) for a, b, _, _ in _lib.PROFILE) if point_kernel else None
    _lib.PROFILE = None
    return e0.elapsed_time(e1), pk, out


def spread(v):
    s = sorted(v)
    return {"median": round(s[len(s) // 2], 1), "min": round(s[0], 1), "max": round(s[-1], 1)}


result = {"gpu": torch.cuda.get_device_name(), "power_limit": smi("power.limit"), "sm_clock_max": smi("clocks.max.sm"),
          "frames": frames, "workloads": {}}
try:
    for name in ("black_800", "fern_high"):
        wl = bench.WORKLOADS[name]
        que, ref = bench.make_workload(name)
        dq, dr = synthetic.to_device(que, dev), synthetic.to_device(ref, dev)
        cfg = bench.model_cfg(*wl["dn"])
        net = renderer.NeuralRayRenderPath(cfg)
        net.load_state_dict(synthetic.make_weights(cfg, seed=0), strict=True)
        net.to(dev)
        samples = que["coords"].shape[1] * sum(wl["dn"])
        for mode in ("fp32", "tf32"):          # warm-up: module loads, workspaces, both weight packs
            render(net, dq, dr, mode)
        ms = {"fp32": [], "tf32": []}
        pk = {"fp32": [], "tf32": []}
        for _ in range(frames):
            for mode in ("fp32", "tf32"):
                t, p, _ = render(net, dq, dr, mode)
                ms[mode].append(t)
                pk[mode].append(p)
        outs = {mode: render(net, dq, dr, mode)[2] for mode in ("fp32", "tf32")}
        err = float((outs["tf32"]["pixel_colors_nr_fine"] - outs["fp32"]["pixel_colors_nr_fine"]).abs().max())
        entry = {"ray_samples": samples, "sm_clock_now": smi("clocks.sm"),
                 "max_abs_diff_pixel_colors_nr_fine": err}
        for mode in ("fp32", "tf32"):
            entry[mode] = {"ray_samples_per_s": spread([samples / (t * 1e-3) for t in ms[mode]]), "frame_ms": spread(ms[mode])}
            if point_kernel:
                entry[mode]["point_kernel_ms"] = spread(pk[mode])
        entry["speedup_median"] = round(entry["tf32"]["ray_samples_per_s"]["median"] / entry["fp32"]["ray_samples_per_s"]["median"], 3)
        result["workloads"][name] = entry
finally:
    renderer.set_precision("fp32")
print(json.dumps(result))
