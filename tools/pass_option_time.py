"""Cost or speed of one render-pass option per frame: the bench's frames (bench.WORKLOADS, bench.model_cfg, seeded
weights) rendered in eval under each arm of the option, the arms alternating frame by frame, CUDA events around each whole
render after warm-up.

    dr          black_800: direct rendering off, with the SH fit, with the NR colours (cfg use_dr_prediction,
                use_nr_color_for_dr)
    tf32        black_800 and fern_high: renderer.set_precision "fp32" (3xTF32) and "tf32"
    visibility  black_800 and fern_high: cfg render_visibility off and on
    blend       black_800 and fern_high: cfg render_blend_weights off and on
    agg         black_800 and fern_high: cfg render_agg_weights off, on, and on together with render_blend_weights
    view        black_800 and fern_high: cfg render_view_depth off, on, and on together with render_agg_weights and
                render_blend_weights
    colors      black_800 and fern_high: cfg render_view_colors off, on, and on together with render_view_depth,
                render_agg_weights and render_blend_weights

Prints one JSON line: the card name, power limit and SM clocks read in the same run; per workload and arm the median
frame time and ray-samples/s with their ranges; and the option's summary (dr_cost_ms, speedup_median and
max_abs_diff_pixel_colors_nr_fine, visibility_cost_ms_median, blend_cost_ms_median, agg_cost_ms_median with
agg_blend_cost_ms_median, view_cost_ms_median with view_agg_blend_cost_ms_median, colors_cost_ms_median with
colors_all_cost_ms_median and all_cost_ms_median, the cost of the three other exports alone).  With --point-kernel,
_lib.PROFILE also times the point kernel alone (events around each point-kernel launch); the blend, agg and view exports
and the per-view colours have no such timing.
usage: python tools/pass_option_time.py {dr,tf32,visibility,blend,agg,view,colors} [frames] [--point-kernel]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from neuray_b200 import _lib, renderer, synthetic  # noqa: E402


def finite(*ts):
    return all(bool(torch.isfinite(t).all()) for t in ts)


def dr_summary(entry, outs):
    for arm in ("dr_sh", "dr_nr_color"):
        assert finite(outs[arm]["pixel_colors_dr"], outs[arm]["pixel_colors_dr_fine"]), arm
    off = entry["dr_off"]["frame_ms"]["median"]
    return {"dr_cost_ms": {arm: round(entry[arm]["frame_ms"]["median"] - off, 1) for arm in ("dr_sh", "dr_nr_color")}}


def tf32_summary(entry, outs):
    err = float((outs["tf32"]["pixel_colors_nr_fine"] - outs["fp32"]["pixel_colors_nr_fine"]).abs().max())
    rate = {mode: entry[mode]["ray_samples_per_s"]["median"] for mode in ("fp32", "tf32")}
    return {"max_abs_diff_pixel_colors_nr_fine": err, "speedup_median": round(rate["tf32"] / rate["fp32"], 3)}


def visibility_summary(entry, outs):
    assert finite(outs["on"]["visibility_nr"], outs["on"]["visibility_nr_fine"])
    return {"visibility_cost_ms_median": round(entry["on"]["frame_ms"]["median"] - entry["off"]["frame_ms"]["median"], 1)}


def blend_summary(entry, outs):
    assert finite(outs["on"]["blend_weights_nr"], outs["on"]["blend_weights_nr_fine"])
    return {"blend_cost_ms_median": round(entry["on"]["frame_ms"]["median"] - entry["off"]["frame_ms"]["median"], 1)}


def agg_summary(entry, outs):
    for arm in ("on", "on_blend"):
        assert finite(*(outs[arm][k + sfx] for k in ("neuray_weights_nr", "geometry_weights_nr") for sfx in ("", "_fine")))
    off = entry["off"]["frame_ms"]["median"]
    return {"agg_cost_ms_median": round(entry["on"]["frame_ms"]["median"] - off, 1),
            "agg_blend_cost_ms_median": round(entry["on_blend"]["frame_ms"]["median"] - off, 1)}


def view_summary(entry, outs):
    for arm in ("on", "on_agg_blend"):
        assert finite(*(outs[arm][k + sfx] for k in ("view_hit_nr", "view_depth_nr") for sfx in ("", "_fine")))
    off = entry["off"]["frame_ms"]["median"]
    return {"view_cost_ms_median": round(entry["on"]["frame_ms"]["median"] - off, 1),
            "view_agg_blend_cost_ms_median": round(entry["on_agg_blend"]["frame_ms"]["median"] - off, 1)}


def colors_summary(entry, outs):
    for arm in ("on", "on_all"):
        assert finite(*(outs[arm]["view_colors_nr" + sfx] for sfx in ("", "_fine")))
    off = entry["off"]["frame_ms"]["median"]
    return {"colors_cost_ms_median": round(entry["on"]["frame_ms"]["median"] - off, 1),
            "colors_all_cost_ms_median": round(entry["on_all"]["frame_ms"]["median"] - off, 1),
            "all_cost_ms_median": round(entry["all"]["frame_ms"]["median"] - off, 1)}


_ALL = {"render_view_depth": True, "render_agg_weights": True, "render_blend_weights": True}
# option -> (workloads, {arm: (cfg overrides, render precision)}, summary)
OPTIONS = {
    "dr": (("black_800",), {"dr_off": ({}, "fp32"), "dr_sh": ({"use_dr_prediction": True}, "fp32"),
                            "dr_nr_color": ({"use_dr_prediction": True, "use_nr_color_for_dr": True}, "fp32")}, dr_summary),
    "tf32": (("black_800", "fern_high"), {"fp32": ({}, "fp32"), "tf32": ({}, "tf32")}, tf32_summary),
    "visibility": (("black_800", "fern_high"), {"off": ({}, "fp32"), "on": ({"render_visibility": True}, "fp32")}, visibility_summary),
    "blend": (("black_800", "fern_high"), {"off": ({}, "fp32"), "on": ({"render_blend_weights": True}, "fp32")}, blend_summary),
    "agg": (("black_800", "fern_high"), {"off": ({}, "fp32"), "on": ({"render_agg_weights": True}, "fp32"),
                                         "on_blend": ({"render_agg_weights": True, "render_blend_weights": True}, "fp32")}, agg_summary),
    "view": (("black_800", "fern_high"), {"off": ({}, "fp32"), "on": ({"render_view_depth": True}, "fp32"),
                                          "on_agg_blend": ({"render_view_depth": True, "render_agg_weights": True,
                                                            "render_blend_weights": True}, "fp32")}, view_summary),
    "colors": (("black_800", "fern_high"), {"off": ({}, "fp32"), "on": ({"render_view_colors": True}, "fp32"),
                                            "all": (_ALL, "fp32"), "on_all": (dict(_ALL, render_view_colors=True), "fp32")},
               colors_summary),
}

ap = argparse.ArgumentParser(description="per-frame cost of a render-pass option")
ap.add_argument("option", choices=OPTIONS)
ap.add_argument("frames", nargs="?", type=int, default=5)
ap.add_argument("--point-kernel", action="store_true", help="also time the point kernel alone")
args = ap.parse_args()
if args.option in ("blend", "agg", "view", "colors") and args.point_kernel:
    ap.error(f"the point kernel with the {args.option} export is not timed alone")
assert torch.cuda.is_available(), "pass_option_time.py measures on a GPU"
dev = torch.device("cuda")


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def render(net, mode, dq, dr):
    renderer.set_precision(mode)
    if args.point_kernel:
        _lib.PROFILE = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    with torch.no_grad():
        out = net.render(dict(dq), dict(dr), False)
    e1.record()
    torch.cuda.synchronize()
    pk = sum(a.elapsed_time(b) for a, b, _, _ in _lib.PROFILE) if args.point_kernel else None
    _lib.PROFILE = None
    return e0.elapsed_time(e1), pk, out


def spread(v):
    s = sorted(v)
    return {"median": round(s[len(s) // 2], 1), "min": round(s[0], 1), "max": round(s[-1], 1)}


workloads, arms, summary = OPTIONS[args.option]
result = {"option": args.option, "gpu": torch.cuda.get_device_name(), "power_limit": smi("power.limit"),
          "sm_clock_max": smi("clocks.max.sm"), "frames": args.frames, "workloads": {}}
try:
    for name in workloads:
        wl = bench.WORKLOADS[name]
        que, ref = bench.make_workload(name)
        dq, dr = synthetic.to_device(que, dev), synthetic.to_device(ref, dev)
        cfg = bench.model_cfg(*wl["dn"])
        W = synthetic.make_weights(cfg, seed=0)
        nets = {}
        for arm, (over, _) in arms.items():
            nets[arm] = renderer.NeuralRayRenderPath(dict(cfg, **over))
            nets[arm].load_state_dict(W, strict=True)
            nets[arm].to(dev)
        for arm, (_, mode) in arms.items():          # warm-up: module loads, workspaces, weight packing
            render(nets[arm], mode, dq, dr)
        ms, pk, outs = {arm: [] for arm in arms}, {arm: [] for arm in arms}, {}
        for _ in range(args.frames):
            for arm, (_, mode) in arms.items():
                t, p, outs[arm] = render(nets[arm], mode, dq, dr)
                ms[arm].append(t)
                pk[arm].append(p)
        rays = que["coords"].shape[1]
        samples = rays * sum(wl["dn"])
        entry = {"rays": rays, "views": wl["rfn"], "samples": list(wl["dn"]), "ray_samples": samples, "sm_clock_now": smi("clocks.sm")}
        for arm in arms:
            entry[arm] = {"ray_samples_per_s": spread([samples / (t * 1e-3) for t in ms[arm]]), "frame_ms": spread(ms[arm])}
            if args.point_kernel:
                entry[arm]["point_kernel_ms"] = spread(pk[arm])
        entry.update(summary(entry, outs))
        result["workloads"][name] = entry
finally:
    renderer.set_precision("fp32")
print(json.dumps(result))
