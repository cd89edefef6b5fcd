"""GPU: direct rendering (cfg use_dr_prediction; nr_direct_render) against the oracle's restatement, whose SH fit runs in
fp64 (oracle/dr_oracle.py), and its contract with the NR path: NR outputs and gradients bit-identical
with DR on and off, hit_prob_dr* dropped in eval, empty and multi-chunk renders, a loss on the DR outputs refused.

Tolerance: 1e-4 abs / 1e-3 rel.  Points whose SH normal matrix has a 2-norm condition number above COND_MAX (fp64,
computed by the oracle) cannot be solved to that tolerance in fp32; rays with such a point are left out of the colour
comparison and the excluded fraction is printed (DESIGN.md, direct rendering)."""
import os
import sys

import numpy as np
import pytest
import torch

import dr_oracle as dro
import neuray_oracle as orc
from gen_golden import CASES as GOLDEN_CASES
from gen_golden import flat_cfg
from neuray_b200 import _lib, metrics, renderer, synthetic

pytestmark = pytest.mark.gpu
ATOL, RTOL = 1e-4, 1e-3
COND_MAX = 1e6
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DR = {"use_dr_prediction": True}
SPREAD = dict(sigma_gain=1.0, sigma_bias=0.02)


def ocfg(cfg):
    out = flat_cfg({**renderer.base_cfg, **cfg})
    out["alpha_value_ground_state"] = cfg.get("alpha_value_ground_state", -15)
    out["use_nr_color_for_dr"] = cfg.get("use_nr_color_for_dr", False)
    return out


def close(a, b, what, keep=None):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    assert a.shape == b.shape, (what, a.shape, b.shape)
    err = (a - b).abs()
    bad = (err > ATOL + RTOL * b.abs()) | torch.isnan(a)
    if keep is not None:
        bad = bad & keep.reshape(keep.shape + (1,) * (bad.dim() - keep.dim()))
    print(f"{what}: max abs err {err.max().item():.3e}, {int(bad.sum())}/{err.numel()} outside tol")
    assert int(bad.sum()) == 0, f"{what}: {int(bad.sum())} values outside tolerance"


def well_conditioned(cond):
    """[qn,rn] rays whose every point's normal matrix is solvable in fp32 to the tolerance (all rays with NR colours)."""
    if cond is None:
        return None
    keep = (cond <= COND_MAX).all(-1)
    print(f"condition numbers: median {cond.median().item():.3g}, max {cond.max().item():.3g}; "
          f"{100.0 * (1 - keep.float().mean().item()):.3f} % of rays excluded")
    return keep


def check(que, ref, cfg, W):
    """coarse pass end to end and the fine pass on the oracle's fine depths, DR outputs against the oracle."""
    oc = ocfg(cfg)
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
    info = {}
    with torch.no_grad():
        gold = dro.render_impl_dr(W, oc, que, ref, False, info=info)
    net = renderer.NeuralRayRenderPath(cfg)
    net.load_state_dict(W, strict=True)
    net.cuda()
    dq, dr = synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda")
    with torch.no_grad():
        out = net.render_impl(dq, dr, False)
        out_f = net.render_by_depth(gold["que_depth_fine"].cuda(), dq, dr, False, True)
    torch.cuda.synchronize()
    close(out["hit_prob_dr"], gold["hit_prob_dr"], "hit_prob_dr")
    close(out["pixel_colors_dr"], gold["pixel_colors_dr"], "pixel_colors_dr", well_conditioned(info["cond"]))
    close(out_f["hit_prob_dr"], gold["hit_prob_dr_fine"], "hit_prob_dr_fine (oracle's fine depths)")
    close(out_f["pixel_colors_dr"], gold["pixel_colors_dr_fine"], "pixel_colors_dr_fine (oracle's fine depths)",
          well_conditioned(info["cond_fine"]))
    return net, out, gold


def pick_rays(que, w, h, n=48):
    """n rays through the image centre + n rays along the top-left edge region (most views masked there)."""
    centre = (h // 2) * w + w // 2 - n // 2
    idx = torch.cat([torch.arange(centre, centre + n), torch.arange(2 * w + 1, 2 * w + 1 + n)])
    return dict(que, coords=que["coords"][:, idx].contiguous())


GEN_DEPTH = {"use_hierarchical_sampling": True, "dist_decoder_cfg": {"use_vis": False}}


@pytest.mark.parametrize("nr_color", [False, True])
def test_cfg1_3_views(nr_color):
    spec = GOLDEN_CASES["cfg1"]
    cfg = dict(spec["cfg"], **DR, use_nr_color_for_dr=nr_color)
    que, ref = synthetic.make_scene(**spec["scene"])
    check(synthetic.slice_rays(que, 1900, 2100), ref, cfg, synthetic.make_weights(cfg, seed=spec["seed"], **SPREAD))


@pytest.mark.parametrize("use_vis", [False, True])
def test_black_400_8_views(use_vis):
    cfg = dict(GEN_DEPTH, **DR, dist_decoder_cfg={"use_vis": use_vis})
    que, ref = synthetic.make_scene(h=400, w=400, rfn=8, seed=0, smooth=2, with_que_imgs=False)
    check(pick_rays(que, 400, 400), ref, cfg, synthetic.make_weights(cfg, seed=0, **SPREAD))


@pytest.mark.parametrize("nr_color", [False, True])
def test_benched_black_800(nr_color):
    sys.path.insert(0, ROOT)
    import bench
    wl = bench.WORKLOADS["black_800"]
    cfg = dict(bench.model_cfg(*wl["dn"]), **DR, use_nr_color_for_dr=nr_color)
    que, ref = synthetic.make_scene(**dict(wl["scene"], rfn=wl["rfn"], seed=0, smooth=2, with_que_imgs=False))
    check(pick_rays(que, 800, 800), ref, cfg, synthetic.make_weights(cfg, seed=0))


@pytest.mark.parametrize("use_vis", [False, True])
def test_10_views_fern_geometry(use_vis):
    cfg = dict(GEN_DEPTH, **DR, dist_decoder_cfg={"use_vis": use_vis}, fine_dist_decoder_cfg={"use_vis": True})
    que, ref = synthetic.make_scene(h=189, w=252, rfn=10, seed=7, smooth=2, depth_range=(1.2, 12.0), arc_deg=100.0,
                                    focal=0.83 * 252, with_que_imgs=False)
    check(pick_rays(que, 252, 189), ref, cfg, synthetic.make_weights(cfg, seed=5, **SPREAD))


SMALL = {"use_hierarchical_sampling": True, "depth_sample_num": 16, "fine_depth_sample_num": 16, "agg_net_cfg": {"sample_num": 16},
         "fine_agg_net_cfg": {"sample_num": 16}, "render_depth": True}


def small_setup(cfg, rays=(300, 428), grad=False):
    que, ref = synthetic.make_scene(40, 48, 4, seed=3, smooth=2)
    que = synthetic.slice_rays(que, *rays)
    W = synthetic.make_weights(cfg, seed=3, **SPREAD)
    nets = []
    for dr in (False, True):
        net = renderer.NeuralRayRenderPath(dict(cfg, use_dr_prediction=dr))
        net.load_state_dict(W, strict=True)
        nets.append(net.cuda())
    return que, ref, nets


@pytest.mark.parametrize("nr_color", [False, True])
def test_nr_outputs_identical_with_dr_on_and_off_in_eval(nr_color):
    que, ref, (off, on) = small_setup(dict(SMALL, use_nr_color_for_dr=nr_color))
    outs = []
    for net in (off, on):
        with torch.no_grad():
            outs.append(net.render(synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda"), False))
    torch.cuda.synchronize()
    a, b = outs
    assert set(b) - set(a) == {"pixel_colors_dr", "pixel_colors_dr_fine"}      # eval drops hit_prob_dr*
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_nr_outputs_and_gradients_unchanged_by_dr_in_training():
    que, ref, nets = small_setup(dict(SMALL))
    results = []
    for net in nets:
        dq, dr = synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda")
        dr["ray_feats"].requires_grad_(True)
        dr["img_feats"].requires_grad_(True)
        torch.manual_seed(7)
        out = net.render(dq, dr, True)
        loss = ((out["pixel_colors_nr"] - out["pixel_colors_gt"]) ** 2).mean() + (out["pixel_colors_nr_fine"] ** 2).mean() + \
            out["hit_prob_nr"].square().mean() + out["render_depth"].mean()
        loss.backward()
        torch.cuda.synchronize()
        grads = {k: p.grad.clone() for k, p in net.named_parameters() if p.grad is not None}
        grads.update({k: dr[k].grad.clone() for k in ("ray_feats", "img_feats")})
        results.append((out, grads))
    (a, ga), (b, gb) = results
    assert {"pixel_colors_dr", "hit_prob_dr", "pixel_colors_dr_fine", "hit_prob_dr_fine"} <= set(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    # the weight-gradient GEMMs and the map gradients accumulate with atomics, so two runs differ in the last bits whatever
    # the cfg (rgb_fc.4.bias, whose true gradient is zero under the softmax, is pure rounding): equal up to that reordering
    assert set(ga) == set(gb) and len(ga) > 100
    for k in ga:
        torch.testing.assert_close(ga[k], gb[k], atol=1e-5 * float(ga[k].abs().max()) + 1e-8, rtol=0, msg=k)


def test_loss_on_dr_outputs_raises():
    que, ref, (_, net) = small_setup(dict(SMALL))
    dq, dr = synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda")
    out = net.render(dq, dr, True)
    assert out["pixel_colors_dr"].requires_grad
    with pytest.raises(_lib.NeurayB200Error, match="use_dr_loss"):
        ((out["pixel_colors_dr"] - out["pixel_colors_gt"]) ** 2).mean().backward()


def test_empty_and_chunked_renders():
    cfg = dict(SMALL, ray_batch_num=128)
    que, ref, (_, net) = small_setup(cfg, rays=(300, 700))
    dq, dr = synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda")
    whole = renderer.NeuralRayRenderPath(dict(cfg, use_dr_prediction=True, ray_batch_num=4096))
    whole.load_state_dict(net.state_dict(), strict=True)
    whole.cuda()
    with torch.no_grad():
        # eval: the fine quantiles are fixed, so four chunks and one chunk render the same rays bit for bit
        a, b = net.render(dq, dr, False), whole.render(dq, dr, False)
        # training: the coarse pass has no random draw (the fine quantiles are drawn per chunk)
        at, bt = net.render(dq, dr, True), whole.render(dq, dr, True)
        empty = net.render(dict(dq, coords=dq["coords"][:, :0]), dr, True)
    torch.cuda.synchronize()
    for k in ("pixel_colors_dr", "pixel_colors_dr_fine"):
        assert torch.equal(a[k], b[k]), k
    for k in ("pixel_colors_dr", "hit_prob_dr"):
        assert torch.equal(at[k], bt[k]), k
    for k in ("pixel_colors_dr", "hit_prob_dr", "pixel_colors_dr_fine", "hit_prob_dr_fine"):
        assert empty[k].shape[:2] == (1, 0), (k, empty[k].shape)
    assert at["hit_prob_dr"].shape == (1, 400, 16)


def test_psnr_ssim_scores_the_dr_renderings():
    que, ref, (_, net) = small_setup(dict(SMALL), rays=(0, 40 * 48))
    dq, dr = synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda")
    with torch.no_grad():
        out = net.render(dq, dr, False)
    out["que_imgs_info"] = dq
    scores = metrics.PSNR_SSIM({})(out, {}, 0)
    for s in ("nr", "dr", "nr_fine", "dr_fine"):
        assert np.isfinite(float(scores[f"psnr_{s}"])) and np.isfinite(float(scores[f"ssim_{s}"])), s


def test_gen_frame_renderer_with_dr_matches_the_oracle():
    """NeuralRayGenFrameRenderer.forward in eval with use_dr_prediction: init net -> encoders -> render, against the
    oracle's stages (encoder outputs carry ~1e-5 differences into the fit, hence the quantile bounds)."""
    from test_encoders_gpu import _smooth_depth, depth_init_golden, golden
    cfg = {"use_hierarchical_sampling": True, "dist_decoder_cfg": {"use_vis": False}, "depth_sample_num": 32, "fine_depth_sample_num": 32,
           "agg_net_cfg": {"sample_num": 32}, "fine_agg_net_cfg": {"sample_num": 32}, "ray_batch_num": 160, **DR}
    _, img_w, vis_w = golden()
    _, _, init_w = depth_init_golden()
    que, ref = synthetic.make_scene(64, 80, 4, seed=6, smooth=2)
    que = synthetic.slice_rays(que, 1500, 1900)
    ref = {k: ref[k] for k in ("imgs", "poses", "Ks", "depth_range")}
    ref["depth"] = _smooth_depth(np.random.RandomState(6), 4, 64, 80, 2.5, 5.0)
    W = synthetic.make_weights(cfg, seed=6)
    full = dict(W)
    full.update({"image_encoder." + k: v for k, v in img_w.items()})
    full.update({"vis_encoder." + k: v for k, v in vis_w.items()})
    full.update({"init_net." + k: v for k, v in init_w.items()})
    net = renderer.NeuralRayGenFrameRenderer(cfg)
    net.load_state_dict(full, strict=True)
    net.cuda().eval()
    with torch.no_grad():
        out = net({"que_imgs_info": synthetic.to_device(que, "cuda"), "ref_imgs_info": synthetic.to_device(ref, "cuda"), "eval": True})
    torch.cuda.synchronize()
    assert not any(k.startswith("hit_prob") for k in out)
    img_feats = orc.res_unet_light(img_w, "", ref["imgs"])
    ray_feats = orc.vis_encoder(vis_w, "", orc.depth_init_net(init_w, "", ref), img_feats)
    gold = dro.render_impl_dr(W, ocfg(cfg), que, dict(ref, ray_feats=ray_feats, img_feats=img_feats), False)
    err = (out["pixel_colors_dr"].cpu() - gold["pixel_colors_dr"]).abs()
    print(f"pixel_colors_dr: max {err.max().item():.2e}, q99 {torch.quantile(err.flatten(), 0.99).item():.2e}")
    assert float(torch.quantile(err.flatten(), 0.99)) < 3e-4 and float(err.max()) < 3e-3
    fine = (out["pixel_colors_dr_fine"].cpu() - gold["pixel_colors_dr_fine"]).abs()
    print(f"pixel_colors_dr_fine: max {fine.max().item():.2e}, q99 {torch.quantile(fine.flatten(), 0.99).item():.2e}")
    assert float(torch.quantile(fine.flatten(), 0.99)) < 1e-3 and float((fine > 1e-3).float().mean()) < 0.01
