"""Score a folder of rendered test views the way the reference's eval.py does, on the GPU, without TensorFlow or lpips.

    python -m neuray_b200.eval --dir_gt D --dir_pr P [--vgg16 PATH --lpips-lin PATH]

For k in range(len(os.listdir(D))) it reads D/{k}.jpg and P/{k}-nr_fine.jpg (PIL, RGB uint8), scores each pair with
tf.image.psnr / tf.image.ssim (max_val 1) and, given the weights, LPIPS-VGG, and prints the means as
`psnr %.4f ssim %.4f lpips %.4f`.  --vgg16 is torchvision's vgg16 state dict (vgg16-397923af.pth), --lpips-lin lpips's
weights/v0.1/vgg.pth; without them PSNR and SSIM are printed and LPIPS is reported as not computed.
"""
import argparse
import os
import sys

import numpy as np

BATCH = 16       # pairs decoded and scored per GPU call


def frame_paths(dir_gt, dir_pr):
    """[(gt_path, pr_path)] in eval.py's order; FileNotFoundError naming the first missing file and how many are missing."""
    pairs = [(os.path.join(dir_gt, f"{k}.jpg"), os.path.join(dir_pr, f"{k}-nr_fine.jpg")) for k in range(len(os.listdir(dir_gt)))]
    missing = [p for pair in pairs for p in pair if not os.path.isfile(p)]
    if missing:
        raise FileNotFoundError(f"{missing[0]} not found ({len(missing)} of the {2 * len(pairs)} expected files are missing: "
                                f"{{k}}.jpg in --dir_gt and {{k}}-nr_fine.jpg in --dir_pr for k < {len(pairs)}, the number of "
                                f"entries in --dir_gt)")
    return pairs


def evaluate(dir_gt, dir_pr, net=None):
    """Per-view scores as a float64 array [views, 2 or 3]: psnr, ssim and, with an LpipsVGG `net`, lpips."""
    import torch

    from . import eval_metrics
    pairs = frame_paths(dir_gt, dir_pr)
    dev = net.features._modules["0"].weight.device if net is not None else torch.device("cuda", torch.cuda.current_device())
    rows = []
    for i in range(0, len(pairs), BATCH):
        chunk = [(eval_metrics.read_rgb(g), eval_metrics.read_rgb(p)) for g, p in pairs[i:i + BATCH]]
        for g, p in chunk:
            if g.shape != p.shape:
                raise ValueError(f"ground truth {g.shape} and prediction {p.shape} differ in size")
        groups = {}            # pairs of one size are scored in one call
        for j, (g, _) in enumerate(chunk):
            groups.setdefault(g.shape, []).append(j)
        scores = [None] * len(chunk)
        for idx in groups.values():
            gt = torch.from_numpy(np.stack([chunk[j][0] for j in idx])).to(dev)     # one upload for both scores
            pr = torch.from_numpy(np.stack([chunk[j][1] for j in idx])).to(dev)
            ps = eval_metrics.psnr_ssim_tf(gt, pr)
            lp = eval_metrics.lpips(gt, pr, net) if net is not None else [None] * len(idx)
            for j, (psnr, ssim), l in zip(idx, ps, lp):
                scores[j] = (psnr, ssim) if l is None else (psnr, ssim, l)
        rows.extend(scores)
    return np.asarray(rows, dtype=np.float64)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--dir_gt", default="data/render/fern/gt")
    ap.add_argument("--dir_pr", default="data/render/fern/neuray_gen_depth-pretrain-eval")
    ap.add_argument("--vgg16", help="torchvision vgg16 state dict (features.* are used)")
    ap.add_argument("--lpips-lin", dest="lpips_lin", help="lpips v0.1 vgg.pth (lin0..4.model.1.weight)")
    args = ap.parse_args(argv)
    if (args.vgg16 is None) != (args.lpips_lin is None):
        ap.error("LPIPS needs both --vgg16 and --lpips-lin")
    try:
        pairs = frame_paths(args.dir_gt, args.dir_pr)
    except FileNotFoundError as e:
        print(f"eval: {e}", file=sys.stderr)
        return 2
    if not pairs:
        print(f"eval: no views in {args.dir_gt}", file=sys.stderr)
        return 2
    net = None
    if args.vgg16 is not None:
        from .eval_metrics import LpipsVGG
        net = LpipsVGG.from_files(args.vgg16, args.lpips_lin).cuda()
    means = evaluate(args.dir_gt, args.dir_pr, net).mean(0)
    if net is not None:
        print(f"psnr {means[0]:.4f} ssim {means[1]:.4f} lpips {means[2]:.4f}")
    else:
        print(f"psnr {means[0]:.4f} ssim {means[1]:.4f}")
        print("lpips not computed: pass --vgg16 and --lpips-lin")
    return 0


if __name__ == "__main__":
    sys.exit(main())
