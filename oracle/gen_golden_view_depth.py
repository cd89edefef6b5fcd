"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/view_depth.npz by executing the UNMODIFIED reference's render_impl
(network/renderer.py:217-226) on the scenes of gen_golden_blend.CASES (3, 5 and 8 views, the vis head on and off, points
outside some views and points that no view sees) and recording, for both passes, each view's masked hit probability
prj_dict['hit_prob'] (network/renderer.py:75-82: the coarse dist decoder's compute_prob(is_ref=True) on the pass'
decoder outputs, times the projection mask) together with prj_dict['mask'] and hit_prob_nr.  Run where the reference
tree exists:

    python oracle/gen_golden_view_depth.py            # writes tests/golden/view_depth.npz

Both fields are copied out of the dict that the reference's predict_proj_ray_prob returns.  Per case <c> the file holds
the case spec as json (c_spec_json), the float64 sums of every input tensor (c_input_sums, in
gen_golden_visibility.input_tensors() order), the fine-pass depths the reference resampled (c_que_depth_fine) and, per
pass (suffix '' or '_fine'), c_prj_hit_prob and c_prj_mask [rfn,1,rn,dn,1] and c_hit_prob_nr [1,rn,dn].  Only data goes
into the repository.
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

import gen_golden_blend as ggb  # noqa: E402
import gen_golden_visibility as ggv  # noqa: E402

CASES = dict(ggb.CASES)


def run_case(name, spec, mod, blob):
    que, ref, W = ggv.make_inputs(spec)
    net = mod.NeuralRayBaseRenderer(spec["cfg"])
    missing, unexpected = net.load_state_dict(W, strict=False)
    assert not unexpected and all(k.split(".")[0] in ("image_encoder", "vis_encoder", "sph_fitter") for k in missing), missing
    net.eval()
    recorded = []
    own_prob = net.predict_proj_ray_prob

    def record(prj_dict, *args):                 # the reference's own prediction; its fields are only copied out
        out = own_prob(prj_dict, *args)
        recorded.append((out["hit_prob"].clone(), out["mask"].clone()))
        return out
    net.predict_proj_ray_prob = record
    with torch.no_grad():
        q = {k: v.clone() for k, v in que.items()}
        r = {k: v.clone() for k, v in ref.items()}
        res = net.render_impl(q, r, False)
        que_depth, _ = mod.sample_depth(q["depth_range"], q["coords"], spec["cfg"]["depth_sample_num"], False)
        fd = mod.sample_fine_depth(que_depth, res["hit_prob_nr"], q["depth_range"], spec["cfg"]["fine_depth_sample_num"], False)
    assert len(recorded) == 2, len(recorded)
    for sfx, (hit, mask) in zip(("", "_fine"), recorded):
        blob[f"{name}_prj_hit_prob{sfx}"] = hit.numpy()
        blob[f"{name}_prj_mask{sfx}"] = mask.numpy()
        blob[f"{name}_hit_prob_nr{sfx}"] = res["hit_prob_nr" + sfx].numpy()
    blob[f"{name}_que_depth_fine"] = torch.sort(fd, -1)[0].numpy()
    blob[f"{name}_input_sums"] = np.array([float(t.double().sum()) for t in ggv.input_tensors(que, ref, W)])
    blob[f"{name}_spec_json"] = np.frombuffer(json.dumps(spec).encode(), dtype=np.uint8)
    hit = recorded[0][0][..., 0]
    print(name, tuple(hit.shape), "max Σ_d hit_v: %.3f (coarse), %.3f (fine)" % tuple(float(h[..., 0].sum(-1).max()) for h, _ in recorded),
          "points no view sees: %d (coarse), %d (fine)" % tuple(int((mk[..., 0].sum(0) == 0).sum()) for _, mk in recorded))


def main():
    import ref_import
    mod = ref_import.load_reference()
    blob = {}
    for name, spec in CASES.items():
        run_case(name, spec, mod, blob)
    path = os.path.join(ROOT, "tests", "golden", "view_depth.npz")
    np.savez_compressed(path, **blob)
    print("->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
