"""GPU: eval.py's scores (csrc/nr_metrics.cu through neuray_b200.eval_metrics and the neuray_b200.eval CLI) against the
restatements of tests/eval_restatement.py, at test-view sizes."""
import math

import numpy as np
import pytest
import torch

import eval_restatement as er
from neuray_b200 import _lib
from test_eval_metrics import pair, write_folder

KINDS = ("random", "smooth", "identical")


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(64, 80), (800, 800), (756, 1008)])
def test_psnr_ssim_match_the_restatement(h, w):
    from neuray_b200 import eval_metrics
    pairs = [pair(k, h, w, seed=h + w + i) for i, k in enumerate(KINDS)]
    gt, pr = np.stack([a for a, _ in pairs]), np.stack([b for _, b in pairs])
    got = eval_metrics.psnr_ssim_tf(gt, pr)
    for kind, (a, b), (psnr, ssim) in zip(KINDS, pairs, got):
        if kind == "identical":
            assert (psnr, ssim) == (math.inf, 1.0)
            continue
        assert abs(ssim - er.ssim_tf(a, b)) < 1e-6, (kind, ssim, er.ssim_tf(a, b))
        assert abs(psnr - er.psnr_tf(a, b)) < 1e-6, (kind, psnr, er.psnr_tf(a, b))


@pytest.mark.gpu
def test_psnr_ssim_batched_equals_single_and_repeats():
    from neuray_b200 import eval_metrics
    h, w = 756, 1008
    pairs = [pair(k, h, w, seed=40 + i) for i, k in enumerate(KINDS + ("random", "smooth"))]
    gt = torch.from_numpy(np.stack([a for a, _ in pairs])).cuda()
    pr = torch.from_numpy(np.stack([b for _, b in pairs])).cuda()
    a = eval_metrics.eval_metrics(gt, pr)
    b = eval_metrics.eval_metrics(gt, pr)
    assert torch.equal(a, b)
    singles = torch.cat([eval_metrics.eval_metrics(gt[i], pr[i]) for i in range(len(pairs))])
    assert torch.equal(a, singles)


@pytest.mark.gpu
def test_psnr_ssim_refuse_bad_input():
    from neuray_b200 import eval_metrics
    a, b = pair("random", 10, 40, seed=1)
    with pytest.raises(_lib.NeurayB200Error):
        eval_metrics.psnr_ssim_tf(a, b)
    a, b = pair("random", 16, 16, seed=1)
    with pytest.raises(ValueError):
        eval_metrics.psnr_ssim_tf(a, b[:, :15])
    with pytest.raises(ValueError):
        eval_metrics.psnr_ssim_tf(a.astype(np.float32), b.astype(np.float32))


def lpips_net(seed=5):
    from neuray_b200.eval_metrics import LpipsVGG
    sd = er.seeded_weights(seed)
    net = LpipsVGG()
    net.load_state_dict(sd, strict=True)
    return net.cuda(), sd


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(64, 64), (800, 800)])
def test_lpips_matches_torch(h, w):
    from neuray_b200 import eval_metrics
    net, sd = lpips_net()
    pairs = [pair(k, h, w, seed=h + i) for i, k in enumerate(KINDS)]
    gt, pr = np.stack([a for a, _ in pairs]), np.stack([b for _, b in pairs])
    got = eval_metrics.lpips(gt, pr, net)
    want = er.lpips_torch(sd, gt, pr, "cuda")
    for kind, g, wv in zip(KINDS, got, want):
        if kind == "identical":
            assert g == 0.0 and wv == 0.0
        else:
            assert abs(g - wv) <= 1e-4 * abs(wv), (kind, g, wv)


@pytest.mark.gpu
def test_lpips_tf32_batches_and_repeats():
    """One TF32 pass per product (encoders.set_precision('tf32')) stays near the fp32 result; a batch of pairs gives what
    single pairs give, bit for bit, and so does a second run."""
    from neuray_b200 import encoders, eval_metrics
    net, sd = lpips_net(seed=6)
    h, w = 96, 128
    pairs = [pair(k, h, w, seed=90 + i) for i, k in enumerate(("random", "smooth", "smooth"))]
    gt = torch.from_numpy(np.stack([a for a, _ in pairs])).cuda()
    pr = torch.from_numpy(np.stack([b for _, b in pairs])).cuda()
    full = net(gt, pr)
    assert torch.equal(full, net(gt, pr))
    assert torch.equal(full, torch.cat([net(gt[i], pr[i]) for i in range(len(pairs))]))
    try:
        encoders.set_precision("tf32")
        fast = net(gt, pr)
    finally:
        encoders.set_precision("fp32")
    assert not torch.equal(fast, full)
    assert ((fast - full).abs() / full.abs()).max().item() < 2e-2
    with pytest.raises(_lib.NeurayB200Error):
        eval_metrics.lpips(gt[:, :31], pr[:, :31], net)


@pytest.mark.gpu
def test_cli_scores_a_folder(tmp_path, capsys):
    from neuray_b200 import eval as nr_eval
    from neuray_b200.eval_metrics import read_rgb
    gt_dir, pr_dir = write_folder(tmp_path, 5)
    imgs = [(read_rgb(g), read_rgb(p)) for g, p in nr_eval.frame_paths(gt_dir, pr_dir)]
    want = np.mean([(er.psnr_tf(a, b), er.ssim_tf(a, b)) for a, b in imgs], 0)

    assert nr_eval.main(["--dir_gt", gt_dir, "--dir_pr", pr_dir]) == 0
    out = capsys.readouterr().out.splitlines()
    assert len(out) == 2 and out[1] == "lpips not computed: pass --vgg16 and --lpips-lin"
    words = out[0].split()
    assert words[0::2] == ["psnr", "ssim"]
    assert np.abs(np.array([float(v) for v in words[1::2]]) - want).max() < 6e-5

    _, sd = lpips_net()
    torch.save({k: v for k, v in sd.items() if k.startswith("features.")}, tmp_path / "vgg16.pth")
    torch.save({k: v for k, v in sd.items() if k.startswith("lin")}, tmp_path / "vgg.pth")
    lp = er.lpips_torch(sd, np.stack([a for a, _ in imgs]), np.stack([b for _, b in imgs]), "cuda").mean()
    assert nr_eval.main(["--dir_gt", gt_dir, "--dir_pr", pr_dir, "--vgg16", str(tmp_path / "vgg16.pth"),
                         "--lpips-lin", str(tmp_path / "vgg.pth")]) == 0
    words = capsys.readouterr().out.split()
    assert words[0::2] == ["psnr", "ssim", "lpips"]
    got = np.array([float(v) for v in words[1::2]])
    assert np.abs(got - [want[0], want[1], lp]).max() < 6e-5
