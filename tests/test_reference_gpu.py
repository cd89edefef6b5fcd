"""GPU: the native path against stored outputs of the UNMODIFIED reference's whole network (tests/golden/reference_net.npz,
oracle/gen_golden_reference_net.py).  The reference's NeuralRayGenRenderer (init net 'depth', both encoders, coarse + fine
render, depth-loss means) was run on seeded inputs and weights that make_data() / net_weights() rebuild here:
  * eval mode: every output key of forward(), against NeuralRayGenFrameRenderer, every stage native;
  * training mode: the three training losses of network.loss (what train/trainer.py builds its losses from) on the
    reference's training-mode outputs, values and gradients with respect to every output tensor they read, against
    neuray_b200.losses.
"""
import json
import os

import numpy as np
import pytest
import torch

from gen_golden_reference_net import CFG, LOSS_CFGS, LOSS_READS, make_data, net_weights
from neuray_b200 import synthetic

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_net.npz")


@pytest.fixture(autouse=True)
def fp32_convolutions():
    """cuDNN runs fp32 convolutions through TF32 by default; the encoders are compared at fp32 accuracy."""
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


def golden(prefix):
    z = np.load(GOLDEN)
    return {k[len(prefix):]: torch.from_numpy(np.ascontiguousarray(z[k])) for k in z.files if k.startswith(prefix) and z[k].dtype.kind in "biuf"}

def compare_outputs(a, b, fine_bad_frac):
    assert set(a) == set(b), set(a) ^ set(b)
    for k in a:
        x, y = a[k].detach().float().cpu(), b[k].detach().float().cpu()
        assert x.shape == y.shape, k
        if a[k].dtype == torch.bool:
            assert (x != y).float().mean().item() <= (fine_bad_frac if k.endswith("_fine") else 0.0), k
            continue
        bad = ((x - y).abs() > 1e-4 + 1e-3 * y.abs()).float().mean().item()
        # fine-pass quantities sit behind searchsorted (SURVEY.md section 7): isolated samples may move by a bin
        allowed = fine_bad_frac if ("fine" in k) else 0.0
        assert bad <= allowed, (k, bad, float((x - y).abs().max()))


def test_eval_forward_matches_the_reference_golden():
    from neuray_b200 import renderer
    que, ref = make_data()
    net = renderer.NeuralRayGenFrameRenderer(CFG)
    net.load_state_dict(net_weights(CFG), strict=True)
    net.cuda().eval()
    data = {"que_imgs_info": synthetic.to_device(que, "cuda"), "ref_imgs_info": synthetic.to_device(ref, "cuda"), "eval": True}
    torch.manual_seed(77)            # randperm of the depth-loss coordinates (CPU generator, like the reference)
    with torch.no_grad():
        got = net(data)
    torch.cuda.synchronize()
    compare_outputs(got, golden("eval_"), fine_bad_frac=0.01)


def test_render_ops_refuse_to_cut_a_graph():
    """A drop-in without a backward raises when handed an input that requires grad (instead of silently detaching)."""
    from neuray_b200 import _lib, render_ops
    d = torch.rand(1, 8, 16, device="cuda", requires_grad=True)
    with pytest.raises(_lib.NeurayB200Error):
        render_ops.depth2dists(d)
    with torch.no_grad():
        render_ops.depth2dists(d)
    fm = torch.randn(2, 32, 12, 16, device="cuda", requires_grad=True)
    pts = torch.rand(2, 50, 2, device="cuda") * torch.tensor([60.0, 44.0], device="cuda")
    mask = (torch.rand(2, 50, device="cuda") > 0.2).float()
    out = render_ops.interpolate_feature_map(fm, pts, mask, 48, 64)
    out.square().sum().backward()
    import neuray_oracle as orc                   # the torch restatement pinned to the reference's goldens
    fm2 = fm.detach().cpu().requires_grad_(True)
    want = orc.interpolate_feature_map(fm2, pts.cpu(), mask.cpu(), 48, 64)
    want.square().sum().backward()
    assert torch.allclose(out.cpu(), want, atol=1e-5) and torch.allclose(fm.grad.cpu(), fm2.grad, atol=1e-4, rtol=1e-4)


def test_losses_match_the_reference_golden():
    """neuray_b200.losses.name2loss on the reference's training-mode outputs: values and the gradients of
    sum_i (i + 1) * loss_i with respect to every output tensor the losses read, against the reference's."""
    from neuray_b200 import losses
    _, ref = make_data(self_feats=True)
    out = {k: v.cuda() for k, v in golden("train_").items()}
    data_gt = {"ref_imgs_info": synthetic.to_device(ref, "cuda"), "scene_name": "dtu_train/scan1"}
    data_pr = {k: (v.detach().clone().requires_grad_(True) if k in LOSS_READS else v) for k, v in out.items()}
    res = {}
    for name, c in LOSS_CFGS.items():
        res.update(losses.name2loss[name](c)(data_pr, data_gt, 0))
    names = json.loads(str(np.load(GOLDEN)["loss_names"]))
    assert list(res) == names, (list(res), names)
    sum((i + 1.0) * v.sum() for i, v in enumerate(res.values())).backward()
    want, gwant = golden("loss_"), golden("dloss_")
    for k in names:
        assert torch.allclose(res[k].detach().cpu(), want[k], rtol=2e-5, atol=1e-6), (k, res[k], want[k])
    for k in LOSS_READS:
        g = data_pr[k].grad
        assert g is not None, k
        err, scale = float((g.cpu() - gwant[k]).abs().max()), float(gwant[k].abs().max())
        assert err <= 1e-4 * scale + 1e-9, (k, err, scale)
