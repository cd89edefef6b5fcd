"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/dr.npz by executing the UNMODIFIED reference's render_impl
(network/renderer.py:217-226) with use_dr_prediction on seeded synthetic scenes: direct rendering (renderer.py:85-125,
181-185) with the SH fit (use_nr_color_for_dr off) and with the NR colours (on), each with the dist decoder's vis head on
and off.  Run where the reference tree exists:

    python oracle/gen_golden_dr.py            # writes tests/golden/dr.npz

Per case <c> the file holds the case spec as json (c_spec_json: scene, ray slice, weight seed, cfg), from which
neuray_b200.synthetic regenerates the inputs deterministically, the float64 sums of every input tensor (c_input_sums, in
input_tensors() order: a check that the regeneration still gives the same inputs), the fine-pass depths the reference
resampled (c_que_depth_fine) and the reference's colour and hit-probability outputs (c_out_*).  Only data goes into the
repository.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import ref_import  # noqa: E402
from neuray_b200 import synthetic  # noqa: E402

_BASE = {"use_hierarchical_sampling": True, "use_dr_prediction": True, "depth_sample_num": 16, "fine_depth_sample_num": 16,
         "agg_net_cfg": {"sample_num": 16}, "fine_agg_net_cfg": {"sample_num": 16}, "ray_batch_num": 4096}
CASES = {
    "sh_novis": dict(scene=dict(h=40, w=48, rfn=3, seed=31, smooth=1), rays=(300, 396), seed=21,
                     cfg={**_BASE, "dist_decoder_cfg": {"use_vis": False}, "fine_dist_decoder_cfg": {"use_vis": False}}),
    "sh_vis": dict(scene=dict(h=40, w=52, rfn=8, seed=32, smooth=2, depth_range=(2.5, 5.5), arc_deg=80.0), rays=(200, 296), seed=22,
                   cfg=dict(_BASE)),
    "nrc_novis": dict(scene=dict(h=40, w=48, rfn=3, seed=33, smooth=1), rays=(300, 396), seed=23,
                      cfg={**_BASE, "use_nr_color_for_dr": True, "dist_decoder_cfg": {"use_vis": False},
                           "fine_dist_decoder_cfg": {"use_vis": False}}),
    "nrc_vis": dict(scene=dict(h=48, w=64, rfn=10, seed=34, smooth=2, depth_range=(1.2, 12.0), arc_deg=100.0), rays=(150, 246), seed=24,
                    cfg={**_BASE, "use_nr_color_for_dr": True}),
}


def make_inputs(spec):
    """(que, ref, W) of a case, regenerated from its spec."""
    que, ref = synthetic.make_scene(**spec["scene"])
    return synthetic.slice_rays(que, *spec["rays"]), ref, synthetic.make_weights(spec["cfg"], seed=spec["seed"])


def input_tensors(que, ref, W):
    return [que[k] for k in sorted(que)] + [ref[k] for k in sorted(ref)] + [W[k] for k in sorted(W)]


def run_case(name, spec, mod, blob):
    que, ref, W = make_inputs(spec)
    net = mod.NeuralRayBaseRenderer(spec["cfg"])
    missing, unexpected = net.load_state_dict(W, strict=False)
    assert not unexpected and all(k.split(".")[0] in ("image_encoder", "vis_encoder", "sph_fitter") for k in missing), missing
    net.eval()
    with torch.no_grad():
        q = {k: v.clone() for k, v in que.items()}
        r = {k: v.clone() for k, v in ref.items()}
        res = net.render_impl(q, r, False)
        que_depth, _ = mod.sample_depth(q["depth_range"], q["coords"], spec["cfg"]["depth_sample_num"], False)
        fd = mod.sample_fine_depth(que_depth, res["hit_prob_nr"], q["depth_range"], spec["cfg"]["fine_depth_sample_num"], False)
    for k, v in res.items():
        if k.startswith(("pixel_colors_dr", "hit_prob_dr", "pixel_colors_nr")):
            blob[f"{name}_out_{k}"] = v.numpy()
    blob[f"{name}_que_depth_fine"] = torch.sort(fd, -1)[0].numpy()
    blob[f"{name}_input_sums"] = np.array([float(t.double().sum()) for t in input_tensors(que, ref, W)])
    blob[f"{name}_spec_json"] = np.frombuffer(json.dumps(spec).encode(), dtype=np.uint8)
    print(name, {k: tuple(v.shape) for k, v in res.items() if "_dr" in k})


def main():
    mod = ref_import.load_reference()
    blob = {"sph_regs": mod.NeuralRayBaseRenderer(dict(_BASE)).sph_fitter.regs.numpy()}
    for name, spec in CASES.items():
        run_case(name, spec, mod, blob)
    path = os.path.join(ROOT, "tests", "golden", "dr.npz")
    np.savez_compressed(path, **blob)
    print("->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
