"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/blend_weights.npz by executing the UNMODIFIED reference's render_impl
(network/renderer.py:217-226) on seeded synthetic scenes and recording, for both passes, the aggregation net's colour-blend
weights blending_weights_valid (network/ibrnet.py:362-366: softmax over the views of rgb_fc's logit, -1e9 where the
projection mask is 0) together with prj_dict['mask'] and hit_prob_nr.  The scenes are those of gen_golden_visibility.py
(3 and 8 views, the vis head on and off, rays whose points fall outside some views) plus one whose top rows hold points
that no view sees.  Run where the reference tree exists:

    python oracle/gen_golden_blend.py            # writes tests/golden/blend_weights.npz

Per case <c> the file holds the case spec as json (c_spec_json), the float64 sums of every input tensor (c_input_sums, in
gen_golden_visibility.input_tensors() order), the fine-pass depths the reference resampled (c_que_depth_fine) and, per
pass (suffix '' or '_fine'), c_blend [rn,dn,rfn,1] as the reference forms it, c_prj_mask [rfn,1,rn,dn,1] and c_hit_prob_nr
[1,rn,dn].  Only data goes into the repository.
"""
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import gen_golden_visibility as ggv  # noqa: E402

_WIDE = dict(ggv._BASE, dist_decoder_cfg={"use_vis": False}, fine_dist_decoder_cfg={"use_vis": False})
CASES = dict(ggv.CASES)
# 5 views on a wide arc, depths out to 3x the scene: the far samples of the top rows leave every view
CASES["v5_unseen"] = dict(scene=dict(h=40, w=48, rfn=5, seed=45, smooth=2, depth_range=(1.0, 14.0), arc_deg=120.0), rays=(0, 96), seed=55,
                          cfg=_WIDE)


def run_case(name, spec, mod, blob):
    que, ref, W = ggv.make_inputs(spec)
    net = mod.NeuralRayBaseRenderer(spec["cfg"])
    missing, unexpected = net.load_state_dict(W, strict=False)
    assert not unexpected and all(k.split(".")[0] in ("image_encoder", "vis_encoder", "sph_fitter") for k in missing), missing
    net.eval()
    ibr = sys.modules["network.ibrnet"]
    blends, masks = [], []
    own_F = ibr.F

    def softmax(x, dim=None, **kw):            # the reference's own F.softmax; the colour blend's result is only copied out
        y = own_F.softmax(x, dim=dim, **kw)
        if dim == 2:
            blends.append(y.clone())
        return y
    ibr.F = types.SimpleNamespace(**{k: getattr(own_F, k) for k in dir(own_F) if not k.startswith("__")})
    ibr.F.softmax = softmax
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
        ibr.F = own_F
    assert len(blends) == 2 and len(masks) == 2, (len(blends), len(masks))
    for sfx, blend, mask in zip(("", "_fine"), blends, masks):
        blob[f"{name}_blend{sfx}"] = blend.numpy()
        blob[f"{name}_prj_mask{sfx}"] = mask.numpy()
        blob[f"{name}_hit_prob_nr{sfx}"] = res["hit_prob_nr" + sfx].numpy()
    blob[f"{name}_que_depth_fine"] = torch.sort(fd, -1)[0].numpy()
    blob[f"{name}_input_sums"] = np.array([float(t.double().sum()) for t in ggv.input_tensors(que, ref, W)])
    blob[f"{name}_spec_json"] = np.frombuffer(json.dumps(spec).encode(), dtype=np.uint8)
    m = masks[0][..., 0]
    print(name, tuple(blends[0].shape), "points outside a view: %.1f %%" % (100.0 * float((m == 0).float().mean())),
          "points no view sees: %d (coarse), %d (fine)" % tuple(int((mk[..., 0].sum(0) == 0).sum()) for mk in masks))


def main():
    import ref_import
    mod = ref_import.load_reference()
    blob = {}
    for name, spec in CASES.items():
        run_case(name, spec, mod, blob)
    path = os.path.join(ROOT, "tests", "golden", "blend_weights.npz")
    np.savez_compressed(path, **blob)
    print("->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
