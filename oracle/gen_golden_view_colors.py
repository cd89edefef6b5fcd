"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/view_colors.npz by executing the UNMODIFIED reference's render_impl
(network/renderer.py:217-226) on the scenes of gen_golden_blend.CASES (3, 5 and 8 views, the vis head on and off, points
outside some views and points that no view sees) and recording, for both passes, the aggregation net's per-view colour
terms rgb_in * blending_weights_valid (network/ibrnet.py:366-367: each view's masked prj_dict['rgb'] times its colour-blend
weight, the terms whose sum over the views is the point's colour) together with prj_dict['mask'], hit_prob_nr and
pixel_colors_nr.  Run where the reference tree exists:

    python oracle/gen_golden_view_colors.py            # writes tests/golden/view_colors.npz

The product is copied out of the reference's own torch.sum over the views.  Per case <c> the file holds the case spec as
json (c_spec_json), the float64 sums of every input tensor (c_input_sums, in gen_golden_visibility.input_tensors() order),
the fine-pass depths the reference resampled (c_que_depth_fine) and, per pass (suffix '' or '_fine'), c_rgb_blend
[rn,dn,rfn,3] as the reference forms it, c_prj_mask [rfn,1,rn,dn,1], c_hit_prob_nr [1,rn,dn] and c_pixel_colors_nr
[1,rn,3].  Only data goes into the repository.
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
    products, masks = [], []
    own_torch = ibr.torch

    def view_sum(x, dim=None, **kw):           # the reference's own torch.sum; the colour blend's operand is only copied out
        if dim == 2 and not kw.get("keepdim", False) and x.shape[-1] == 3:
            products.append(x.clone())
        return own_torch.sum(x, dim=dim, **kw) if dim is not None else own_torch.sum(x, **kw)
    ibr.torch = types.SimpleNamespace(**{k: getattr(own_torch, k) for k in dir(own_torch) if not k.startswith("__")})
    ibr.torch.sum = view_sum
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
        ibr.torch = own_torch
    assert len(products) == 2 and len(masks) == 2, (len(products), len(masks))
    for sfx, prod, mask in zip(("", "_fine"), products, masks):
        blob[f"{name}_rgb_blend{sfx}"] = prod.numpy()
        blob[f"{name}_prj_mask{sfx}"] = mask.numpy()
        blob[f"{name}_hit_prob_nr{sfx}"] = res["hit_prob_nr" + sfx].numpy()
        blob[f"{name}_pixel_colors_nr{sfx}"] = res["pixel_colors_nr" + sfx].numpy()
    blob[f"{name}_que_depth_fine"] = torch.sort(fd, -1)[0].numpy()
    blob[f"{name}_input_sums"] = np.array([float(t.double().sum()) for t in ggv.input_tensors(que, ref, W)])
    blob[f"{name}_spec_json"] = np.frombuffer(json.dumps(spec).encode(), dtype=np.uint8)
    print(name, tuple(products[0].shape),
          "points no view sees: %d (coarse), %d (fine)" % tuple(int((mk[..., 0].sum(0) == 0).sum()) for mk in masks))


def main():
    import ref_import
    mod = ref_import.load_reference()
    blob = {}
    for name, spec in CASES.items():
        run_case(name, spec, mod, blob)
    path = os.path.join(ROOT, "tests", "golden", "view_colors.npz")
    np.savez_compressed(path, **blob)
    print("->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
