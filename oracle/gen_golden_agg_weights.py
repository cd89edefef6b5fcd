"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/agg_weights.npz by executing the UNMODIFIED reference's render_impl
(network/renderer.py:217-226) on the scenes of gen_golden_blend.CASES (3, 5 and 8 views, the vis head on and off, points
outside some views and points that no view sees) and recording, for both passes, the aggregation net's two per-view
pooling weights: the NeuRay weight weight0 (network/ibrnet.py:334-337: sigmoid(neuray_fc(neuray_feat)) · mask / (Σ_v mask
+ 1e-8)) and the geometry weight (network/ibrnet.py:349-350: vis / (Σ_v vis + 1e-8), vis = vis_fc2(x · vis) · mask),
together with prj_dict['mask'] and hit_prob_nr.  Run where the reference tree exists:

    python oracle/gen_golden_agg_weights.py            # writes tests/golden/agg_weights.npz

The weights are copied out of the reference's fused_mean_variance (network/ibrnet.py:113-116), which
IBRNetWithNeuRay.forward calls three times per pass in a fixed order: with weight0 (:338), with the mask weight (:339)
and with the geometry weight (:352).  Per case <c> the file holds the case spec as json (c_spec_json), the float64 sums
of every input tensor (c_input_sums, in gen_golden_visibility.input_tensors() order), the fine-pass depths the reference
resampled (c_que_depth_fine) and, per pass (suffix '' or '_fine'), c_weight0 and c_weight [rn,dn,rfn,1] as the reference
forms them, c_prj_mask [rfn,1,rn,dn,1] and c_hit_prob_nr [1,rn,dn].  Only data goes into the repository.
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
    ibr = sys.modules["network.ibrnet"]
    pooled, masks = [], []
    own_fmv = ibr.fused_mean_variance

    def fused_mean_variance(x, weight):          # the reference's own pooling; its weight is only copied out
        pooled.append(weight.clone())
        return own_fmv(x, weight)
    ibr.fused_mean_variance = fused_mean_variance
    own_prob = net.predict_proj_ray_prob

    def record(prj_dict, *args):
        out = own_prob(prj_dict, *args)
        masks.append(out["mask"].clone())
        return out
    net.predict_proj_ray_prob = record
    try:
        with torch.no_grad():
            q = {k: v.clone() for k, v in que.items()}
            r = {k: v.clone() for k, v in ref.items()}
            res = net.render_impl(q, r, False)
            que_depth, _ = mod.sample_depth(q["depth_range"], q["coords"], spec["cfg"]["depth_sample_num"], False)
            fd = mod.sample_fine_depth(que_depth, res["hit_prob_nr"], q["depth_range"], spec["cfg"]["fine_depth_sample_num"], False)
    finally:
        ibr.fused_mean_variance = own_fmv
    assert len(pooled) == 6 and len(masks) == 2, (len(pooled), len(masks))
    for k, (sfx, mask) in enumerate(zip(("", "_fine"), masks)):
        weight0, _, weight = pooled[3 * k: 3 * k + 3]             # weight0 (:338), mask weight (:339), geometry weight (:352)
        blob[f"{name}_weight0{sfx}"] = weight0.numpy()
        blob[f"{name}_weight{sfx}"] = weight.numpy()
        blob[f"{name}_prj_mask{sfx}"] = mask.numpy()
        blob[f"{name}_hit_prob_nr{sfx}"] = res["hit_prob_nr" + sfx].numpy()
    blob[f"{name}_que_depth_fine"] = torch.sort(fd, -1)[0].numpy()
    blob[f"{name}_input_sums"] = np.array([float(t.double().sum()) for t in ggv.input_tensors(que, ref, W)])
    blob[f"{name}_spec_json"] = np.frombuffer(json.dumps(spec).encode(), dtype=np.uint8)
    m = masks[0][..., 0]
    print(name, tuple(pooled[0].shape), "points outside a view: %.1f %%" % (100.0 * float((m == 0).float().mean())),
          "points no view sees: %d (coarse), %d (fine)" % tuple(int((mk[..., 0].sum(0) == 0).sum()) for mk in masks))


def main():
    import ref_import
    mod = ref_import.load_reference()
    blob = {}
    for name, spec in CASES.items():
        run_case(name, spec, mod, blob)
    path = os.path.join(ROOT, "tests", "golden", "agg_weights.npz")
    np.savez_compressed(path, **blob)
    print("->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
