"""GPU: the validation metric PSNR_SSIM (csrc/nr_metrics.cu through neuray_b200.metrics) against the float64 restatement of
the reference's definition (tests/metrics_restatement.py), at evaluation image sizes and at the smallest legal crops."""
import math

import numpy as np
import pytest
import torch

import metrics_restatement as mr
from neuray_b200 import _lib

SHAPES = [(800, 800), (400, 400), (300, 400), (756, 1008), (11, 11), (13, 17)]


def frame(h, w, seed):
    """A ground truth and three predictions as float32 [h,w,3]: a noisy copy of a smooth image, independent uniform noise,
    and values well outside [0, 1] (the clip matters)."""
    rs = np.random.RandomState(seed)
    yy, xx = np.meshgrid(np.linspace(0, 4, h), np.linspace(0, 4, w), indexing="ij")
    gt = 0.5 + 0.45 * np.sin(xx[..., None] + 1.3 * yy[..., None] + np.arange(3))
    preds = [gt + rs.normal(0, 0.04, gt.shape), rs.uniform(0, 1, gt.shape), rs.uniform(-0.5, 1.5, gt.shape)]
    return gt.astype(np.float32), [p.astype(np.float32) for p in preds]


def cuda(a):
    return torch.from_numpy(a).reshape(1, -1, 3).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("ratio", [1.0, 0.8])
@pytest.mark.parametrize("h,w", SHAPES)
def test_gpu_matches_the_restatement(h, w, ratio):
    from neuray_b200 import metrics
    gt, preds = frame(h, w, seed=h + w)
    mh, mw = metrics.margins(h, w, ratio)
    if min(h - 2 * mh, w - 2 * mw) < 11:
        with pytest.raises(_lib.NeurayB200Error):
            metrics.psnr_ssim(cuda(gt), [cuda(p) for p in preds], h, w, ratio)
        return
    got = metrics.psnr_ssim(cuda(gt), [cuda(p) for p in preds], h, w, ratio)
    sse = metrics.image_metrics(cuda(gt), [cuda(p) for p in preds], h, w, mh, mw).cpu()[:, :3]
    g = mr.crop(mr.color_map_backward(gt), ratio).astype(np.int64)
    for k, p in enumerate(preds):
        want_psnr, want_ssim = mr.psnr_ssim(gt, p, h, w, ratio)
        assert abs(got[k][1] - want_ssim) < 1e-9, (k, got[k][1], want_ssim)
        assert abs(got[k][0] - want_psnr) < 1e-4, (k, got[k][0], want_psnr)
        d = g - mr.crop(mr.color_map_backward(p), ratio).astype(np.int64)
        assert sse[k].tolist() == (d * d).reshape(-1, 3).sum(0).astype(np.float64).tolist()


@pytest.mark.gpu
def test_quantisation_matches_numpy_on_edge_values():
    """Every quantised value shows in the exact squared error against an all-zero prediction."""
    from neuray_b200 import metrics
    from test_metrics import quantisation_edge_values
    x = quantisation_edge_values()
    h, w = 11, -(-x.size // 33)
    img = np.zeros(h * w * 3, np.float32)
    img[:x.size] = x
    zero = np.zeros_like(img)
    out = metrics.image_metrics(cuda(img), [cuda(zero)], h, w, 0, 0).cpu()
    q = ((img * 255).clip(0, 255).astype(np.uint8)).astype(np.int64).reshape(-1, 3)
    assert out[0, :3].tolist() == (q * q).sum(0).astype(np.float64).tolist()


@pytest.mark.gpu
def test_identical_images_and_too_small_crops():
    from neuray_b200 import metrics
    gt, preds = frame(64, 48, seed=1)
    assert metrics.psnr_ssim(cuda(gt), [cuda(gt.copy())], 64, 48) == [(math.inf, 1.0)]
    with pytest.raises(_lib.NeurayB200Error):
        metrics.psnr_ssim(cuda(gt[:10]), [cuda(preds[0][:10])], 10, 48)
    with pytest.raises(_lib.NeurayB200Error):
        metrics.image_metrics(cuda(gt), [cuda(preds[0])], 64, 48, 0, 19)      # 48 - 38 = 10 columns
    with pytest.raises(ValueError):
        metrics.psnr_ssim(cuda(gt), [cuda(preds[0])] * (metrics.MAX_PRED + 1), 64, 48)


@pytest.mark.gpu
def test_repeatable_and_batched_equals_single():
    """Bit-identical from run to run, and N predictions in one launch give exactly what N single launches give."""
    from neuray_b200 import metrics
    h, w = 756, 1008
    gt, preds = frame(h, w, seed=4)
    g, ps = cuda(gt), [cuda(p) for p in preds]
    a = metrics.image_metrics(g, ps, h, w, 75, 100)
    b = metrics.image_metrics(g, ps, h, w, 75, 100)
    assert torch.equal(a, b)
    singles = torch.cat([metrics.image_metrics(g, [p], h, w, 75, 100) for p in ps])
    assert torch.equal(a, singles)


@pytest.mark.gpu
def test_metric_class_on_a_rendered_frame():
    """PSNR_SSIM on a full-raster coarse + fine render of a synthetic frame: the reference's keys, the restatement's values."""
    from neuray_b200 import metrics, renderer, synthetic
    cfg = {"use_hierarchical_sampling": True, "dist_decoder_cfg": {"use_vis": False}, "depth_sample_num": 32,
           "fine_depth_sample_num": 32, "agg_net_cfg": {"sample_num": 32}, "fine_agg_net_cfg": {"sample_num": 32}}
    h, w = 48, 64
    que, ref = synthetic.make_scene(h, w, 4, seed=3, smooth=2)
    net = renderer.NeuralRayRenderPath(cfg)
    net.load_state_dict(synthetic.make_weights(cfg, seed=3), strict=True)
    net.cuda()
    dq, dr = synthetic.to_device(que, "cuda:0"), synthetic.to_device(ref, "cuda:0")
    with torch.no_grad():
        out = net.render(dq, dr, False)
    assert out["pixel_colors_nr"].shape == (1, h * w, 3)
    res = metrics.PSNR_SSIM({})(out, {"que_imgs_info": dq}, 0)
    assert list(res) == ["psnr_nr", "ssim_nr", "psnr_nr_fine", "ssim_nr_fine"]
    gt = out["pixel_colors_gt"].cpu().numpy()
    for s in ("nr", "nr_fine"):
        want_psnr, want_ssim = mr.psnr_ssim(gt, out[f"pixel_colors_{s}"].cpu().numpy(), h, w)
        for key, want in ((f"psnr_{s}", want_psnr), (f"ssim_{s}", want_ssim)):
            assert res[key].dtype == torch.float32 and res[key].shape == (1,) and res[key].device.type == "cpu"
            assert res[key].item() == pytest.approx(want, rel=1e-6), key
    res8 = metrics.PSNR_SSIM({"eval_margin_ratio": 0.8})({**out, "que_imgs_info": dq}, {}, 0)    # h, w from data_pr
    want = mr.psnr_ssim(gt, out["pixel_colors_nr_fine"].cpu().numpy(), h, w, 0.8)
    assert res8["ssim_nr_fine"].item() == pytest.approx(want[1], rel=1e-6)
