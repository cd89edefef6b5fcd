"""Golden vectors of the UNMODIFIED reference's whole NeuralRayGenRenderer (init net 'depth', both encoders, coarse + fine
render, depth-loss means) for tests/test_reference_gpu.py:

    python oracle/gen_golden_reference_net.py      # needs the reference tree (oracle/ref_import.py) -> tests/golden/reference_net.npz

  * eval_*   : forward() in eval mode on make_data()
  * train_*  : forward() in training mode (self-hit prob on) on make_data(self_feats=True): what the three training losses read
  * loss_* / dloss_* : network.loss.name2loss['render' | 'depth' | 'consist'] on those outputs, the values and the gradients of
               sum_i (i + 1) * loss_i with respect to every output tensor the losses read
Weights: synthetic.make_weights for the path modules, the encoder and init-net test weights of encoders.npz / depth_init_net.npz.
make_data() and net_weights() are what the test rebuilds the same inputs and weights with.
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

from neuray_b200 import synthetic  # noqa: E402
import neuray_oracle as orc  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_net.npz")
DN = 24
CFG = {"init_net_type": "depth", "use_hierarchical_sampling": True, "use_depth_loss": True, "dist_decoder_cfg": {"use_vis": False},
       "depth_sample_num": DN, "fine_depth_sample_num": DN, "agg_net_cfg": {"sample_num": DN}, "fine_agg_net_cfg": {"sample_num": DN},
       "ray_batch_num": 192, "render_depth": True, "depth_loss_coords_num": 256}
LOSS_READS = ("pixel_colors_nr", "pixel_colors_nr_fine", "depth_mean", "depth_mean_fine", "hit_prob_self", "hit_prob_self_fine")
LOSS_CFGS = {"render": {"use_nr_fine_loss": True}, "depth": {"depth_loss_type": "smooth_l1"}, "consist": {}}


def _smooth(rs, shape, lo, hi, cells=8):
    """Low-frequency random field (bilinear upsampling of a coarse grid): images and depth maps of real scenes are smooth at
    the pixel scale; white noise would make every bilinear lookup hypersensitive to the last bit of its coordinates."""
    n, c, h, w = shape
    coarse = torch.from_numpy(rs.uniform(lo, hi, (n, c, max(2, h // cells), max(2, w // cells))).astype(np.float32))
    return torch.nn.functional.interpolate(coarse, size=(h, w), mode="bilinear", align_corners=True)


def make_data(rfn=6, rays=384, self_feats=False, seed=3):
    que, ref = synthetic.make_scene(64, 80, rfn, seed=seed, smooth=2)
    ref = dict(ref)
    ref.pop("ray_feats"), ref.pop("img_feats")
    rs = np.random.RandomState(seed)
    ref["imgs"] = _smooth(rs, tuple(ref["imgs"].shape), 0.0, 1.0)
    que = dict(que, imgs=_smooth(rs, tuple(que["imgs"].shape), 0.0, 1.0))
    ref["depth"] = _smooth(rs, (rfn, 1, 64, 80), 2.5, 5.0)
    ref["true_depth"] = ref["depth"]
    n = que["coords"].shape[1]
    idx = torch.from_numpy(rs.permutation(n)[:rays])
    que = dict(que, coords=que["coords"][:, idx].contiguous())
    if self_feats:
        que["ray_feats"] = torch.from_numpy(rs.standard_normal((1, 32, 16, 20)).astype(np.float32))
    return que, ref


def net_weights(cfg, seed=0):
    """Every parameter of NeuralRayGenRenderer(cfg) under the reference's state-dict names."""
    W = dict(synthetic.make_weights(cfg, seed=seed, sigma_gain=1.0, sigma_bias=0.02))
    z = np.load(os.path.join(ROOT, "tests", "golden", "encoders.npz"))
    W.update({"image_encoder." + k: v for k, v in orc.encoder_test_weights(json.loads(str(z["image_shapes"])), 11).items()})
    W.update({"vis_encoder." + k: v for k, v in orc.encoder_test_weights(json.loads(str(z["vis_shapes"])), 12).items()})
    z = np.load(os.path.join(ROOT, "tests", "golden", "depth_init_net.npz"))
    W.update({"init_net." + k: v for k, v in orc.encoder_test_weights(json.loads(str(z["shapes"])), 13).items()})
    return W


def main():
    import ref_import
    mod = ref_import.load_reference()
    import network.loss as ref_loss
    blob = {}
    torch.backends.cudnn.allow_tf32 = False

    def build(cfg):
        torch.manual_seed(0)
        net = mod.NeuralRayGenRenderer(cfg)
        missing, unexpected = net.load_state_dict(net_weights(cfg), strict=False)
        assert not unexpected and all(k.startswith("sph_fitter.") for k in missing), (missing, unexpected)
        return net

    def run(net, que, ref, is_train):
        data = {"que_imgs_info": {k: v.clone() for k, v in que.items()}, "ref_imgs_info": {k: v.clone() for k, v in ref.items()}}
        if not is_train:
            data["eval"] = True
        torch.manual_seed(77)            # randperm of the depth-loss coordinates, torch.rand of the fine quantiles
        return net(data)

    que, ref = make_data()
    with torch.no_grad():
        out = run(build(CFG).eval(), que, ref, False)
    blob.update({"eval_" + k: v.numpy() for k, v in out.items()})

    cfg = dict(CFG, use_self_hit_prob=True)
    que, ref = make_data(self_feats=True)
    with torch.no_grad():
        out = run(build(cfg).train(), que, ref, True)
    blob.update({"train_" + k: v.numpy() for k, v in out.items()})
    data_gt = {"ref_imgs_info": ref, "scene_name": "dtu_train/scan1"}
    data_pr = {k: (v.clone().requires_grad_(True) if k in LOSS_READS else v) for k, v in out.items()}
    res = {}
    for name, c in LOSS_CFGS.items():
        res.update(ref_loss.name2loss[name](c)(data_pr, data_gt, 0))
    sum((i + 1.0) * v.sum() for i, v in enumerate(res.values())).backward()
    blob["loss_names"] = np.array(json.dumps(list(res)))
    blob.update({"loss_" + k: v.detach().numpy() for k, v in res.items()})
    blob.update({"dloss_" + k: data_pr[k].grad.numpy() for k in LOSS_READS})
    np.savez_compressed(GOLDEN, **blob)
    print(GOLDEN, "%.1f KB" % (os.path.getsize(GOLDEN) / 1024), sorted(blob))


if __name__ == "__main__":
    main()
