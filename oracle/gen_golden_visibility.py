"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/visibility.npz by executing the UNMODIFIED reference's render_impl
(network/renderer.py:217-226) on seeded synthetic scenes and recording, for both passes, what the per-view visibility
output is made of: prj_dict['vis'] and prj_dict['mask'] as predict_proj_ray_prob (renderer.py:67-83) leaves them, and
hit_prob_nr.  The cases cover 3 and 8 views, the coarse decoder's vis head on and off, and rays along the image border
whose points fall outside some views.  Run where the reference tree exists:

    python oracle/gen_golden_visibility.py            # writes tests/golden/visibility.npz

Per case <c> the file holds the case spec as json (c_spec_json), the float64 sums of every input tensor (c_input_sums,
in input_tensors() order), the fine-pass depths the reference resampled (c_que_depth_fine) and, per pass (suffix '' or
'_fine'), c_prj_vis / c_prj_mask [rfn,1,rn,dn,1] and c_hit_prob_nr [1,rn,dn].  Only data goes into the repository.
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

from neuray_b200 import synthetic  # noqa: E402

_BASE = {"use_hierarchical_sampling": True, "depth_sample_num": 16, "fine_depth_sample_num": 16,
         "agg_net_cfg": {"sample_num": 16}, "fine_agg_net_cfg": {"sample_num": 16}, "ray_batch_num": 4096}
_NOVIS = {"dist_decoder_cfg": {"use_vis": False}, "fine_dist_decoder_cfg": {"use_vis": False}}
# rays: the first rows of the query image (points near its border fall outside some views) and a band through the centre
CASES = {
    "v3_novis": dict(scene=dict(h=40, w=48, rfn=3, seed=41, smooth=1), rays=(0, 96), seed=51, cfg={**_BASE, **_NOVIS}),
    "v3_vis": dict(scene=dict(h=40, w=48, rfn=3, seed=42, smooth=2), rays=(900, 996), seed=52, cfg=dict(_BASE)),
    "v8_novis": dict(scene=dict(h=40, w=52, rfn=8, seed=43, smooth=2, depth_range=(2.5, 5.5), arc_deg=80.0), rays=(0, 104), seed=53,
                     cfg={**_BASE, **_NOVIS}),
    "v8_vis": dict(scene=dict(h=48, w=64, rfn=8, seed=44, smooth=2, depth_range=(1.2, 12.0), arc_deg=100.0), rays=(1500, 1596), seed=54,
                   cfg=dict(_BASE)),
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
    seen = []
    own = net.predict_proj_ray_prob

    def record(prj_dict, *args):            # the reference's own method; its result is only copied out
        out = own(prj_dict, *args)
        seen.append((out["vis"].clone(), out["mask"].clone()))
        return out
    net.predict_proj_ray_prob = record
    with torch.no_grad():
        q = {k: v.clone() for k, v in que.items()}
        r = {k: v.clone() for k, v in ref.items()}
        res = net.render_impl(q, r, False)
        que_depth, _ = mod.sample_depth(q["depth_range"], q["coords"], spec["cfg"]["depth_sample_num"], False)
        fd = mod.sample_fine_depth(que_depth, res["hit_prob_nr"], q["depth_range"], spec["cfg"]["fine_depth_sample_num"], False)
    assert len(seen) == 2
    for sfx, (vis, mask) in zip(("", "_fine"), seen):
        blob[f"{name}_prj_vis{sfx}"] = vis.numpy()
        blob[f"{name}_prj_mask{sfx}"] = mask.numpy()
        blob[f"{name}_hit_prob_nr{sfx}"] = res["hit_prob_nr" + sfx].numpy()
    blob[f"{name}_que_depth_fine"] = torch.sort(fd, -1)[0].numpy()
    blob[f"{name}_input_sums"] = np.array([float(t.double().sum()) for t in input_tensors(que, ref, W)])
    blob[f"{name}_spec_json"] = np.frombuffer(json.dumps(spec).encode(), dtype=np.uint8)
    m = seen[0][1][..., 0]
    print(name, tuple(seen[0][0].shape), "points outside a view: %.1f %%" % (100.0 * float((m == 0).float().mean())),
          "(view, ray) pairs with no sample in the view: %d" % int((m.sum(-1) == 0).sum()))


def main():
    import ref_import
    mod = ref_import.load_reference()
    blob = {}
    for name, spec in CASES.items():
        run_case(name, spec, mod, blob)
    path = os.path.join(ROOT, "tests", "golden", "visibility.npz")
    np.savez_compressed(path, **blob)
    print("->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
