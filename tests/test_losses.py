"""Training extras next to the ray path (SURVEY.md 8f row 3): predict_mean_for_depth_loss (reference renderer.py:280-316)
and RenderLoss / DepthLoss / ConsistencyLoss (network/loss.py:17-132).

CPU: the oracle's restatement and the host build of the product routines (csrc/nr_loss_math.cuh through
tests/cpu_harness/loss_cpu_harness.cu) against tests/golden/losses.npz -- values AND input / parameter gradients produced by
the UNMODIFIED reference (oracle/gen_golden_losses.py).  GPU: the CUDA path through neuray_b200.losses against the same
golden and against the oracle at training sizes."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import neuray_oracle as orc
import ref_packers
from golden_io import GOLDEN_DIR
from neuray_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")


def golden():
    z = np.load(os.path.join(GOLDEN_DIR, "losses.npz"))
    return {k: torch.from_numpy(np.ascontiguousarray(z[k])) for k in z.files}


DEPTH_CASES = [("l2", "l2", False), ("smooth", "smooth_l1", False), ("gso", "l2", True)]


def close(a, b, rtol=2e-5, atol=2e-6):
    assert a.shape == b.shape, (a.shape, b.shape)
    assert torch.allclose(a, b, rtol=rtol, atol=atol), float((a - b).abs().max())


def test_oracle_matches_the_reference():
    G = golden()
    for tag, mask in (("masked", G["render_mask"]), ("plain", None)):
        pr = G["render_pr"].clone().requires_grad_(True)
        loss = orc.render_loss(pr, G["render_gt"], mask)
        close(loss.detach(), G[f"render_{tag}_loss"])
        close(torch.autograd.grad(loss.sum() * 1.7, pr)[0], G[f"render_{tag}_grad"])
    for tag, kind, gso in DEPTH_CASES:
        dp = G["depth_pr"].clone().requires_grad_(True)
        loss = orc.depth_loss(dp, G["depth_coords"], G["true_depth"], G["depth_range"], kind, 0.05, G["aug_depth"] if gso else None)
        close(loss.detach(), G[f"depth_{tag}_loss"])
        close(torch.autograd.grad((loss * G["depth_gscale"]).sum(), dp)[0], G[f"depth_{tag}_grad"])
    p1 = G["consist_p1"].clone().requires_grad_(True)
    loss = orc.consistency_loss(G["consist_p0"], p1)
    close(loss.detach(), G["consist_loss"])
    close(torch.autograd.grad(loss.sum() * 0.3, p1)[0], G["consist_grad"], rtol=1e-4)
    W = {"d." + k[7:]: v.clone().requires_grad_(True) for k, v in G.items() if k.startswith("mean_w_")}
    rf = G["mean_ray_feats"].clone().requires_grad_(True)
    mean = orc.predict_mean(W, "d", rf, G["depth_coords"], 24, 32)
    close(mean.detach(), G["mean_out"])
    (mean * G["mean_gout"]).sum().backward()
    close(rf.grad, G["mean_d_ray_feats"], rtol=1e-4, atol=1e-6)
    for k, v in G.items():
        if k.startswith("mean_g_"):
            close(W["d." + k[7:]].grad, v, rtol=1e-4, atol=1e-6)


@pytest.fixture(scope="module")
def harness():
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    os.makedirs(BUILD, exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpu_harness", "loss_cpu_harness.cu")
    lib = os.path.join(BUILD, "libloss_cpu_harness.so")
    deps = [src] + [os.path.join(ROOT, "neuray_b200", "csrc", f) for f in ("nr_loss_math.cuh", "nr_train_math.cuh", "nr_common.cuh")]
    if not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in deps):
        subprocess.run(["nvcc", "-shared", "-Xcompiler", "-fPIC", "-O1", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                        src, "-o", lib], check=True)
    return C.CDLL(lib)


def vp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def decoder_state(G, prefix="dist_decoder"):
    """The golden's decoder (use_vis False) as a full pass state dict for the packers: mean head from the golden, rest random."""
    from neuray_b200 import synthetic
    cfg = {"depth_sample_num": 8, "agg_net_cfg": {"sample_num": 8}, "dist_decoder_cfg": {"use_vis": False}}
    W = synthetic.make_weights(cfg, seed=1)
    for k, v in G.items():
        if k.startswith("mean_w_"):
            W[f"{prefix}.{k[7:]}"] = v.clone()
    return {k: v for k, v in W.items() if k.startswith("dist_decoder.") or k.startswith("agg_net.")}


def test_host_build_matches_the_reference(harness):
    G = golden()
    f = lambda t: t.contiguous().float()
    # RenderLoss
    pr, gt, mask = f(G["render_pr"]), f(G["render_gt"]), G["render_mask"].to(torch.uint8).contiguous()
    for tag, m in (("masked", mask), ("plain", None)):
        loss, d, g = torch.empty(1), torch.empty_like(pr), torch.tensor([1.7])
        assert harness.nr_cpu_render_loss(vp(pr), vp(gt), vp(m), 1, 50, vp(loss), None, None) == 0
        assert harness.nr_cpu_render_loss(vp(pr), vp(gt), vp(m), 1, 50, None, vp(g), vp(d)) == 0
        close(loss, G[f"render_{tag}_loss"])
        close(d, G[f"render_{tag}_grad"])
    # DepthLoss
    coords, dp, td, ad, rng = f(G["depth_coords"]), f(G["depth_pr"]), f(G["true_depth"]), f(G["aug_depth"]), f(G["depth_range"])
    for tag, kind, gso in DEPTH_CASES:
        p = _lib.NrDepthLossParams()
        loss, d, g = torch.empty(3), torch.empty_like(dp), f(G["depth_gscale"])
        p.depth_pr, p.coords, p.true_depth, p.aug_depth, p.depth_range = dp.data_ptr(), coords.data_ptr(), td.data_ptr(), ad.data_ptr() if gso else None, rng.data_ptr()
        p.rfn, p.pn, p.h, p.w, p.loss_type, p.beta, p.correct_thresh = 3, 40, 24, 32, 0 if kind == "l2" else 1, 0.05, 0.02
        p.loss = loss.data_ptr()
        assert harness.nr_cpu_depth_loss(C.byref(p)) == 0
        p.g, p.d_depth_pr = g.data_ptr(), d.data_ptr()
        assert harness.nr_cpu_depth_loss(C.byref(p)) == 0
        close(loss, G[f"depth_{tag}_loss"])
        close(d, G[f"depth_{tag}_grad"])
    # ConsistencyLoss
    p0, p1 = f(G["consist_p0"]), f(G["consist_p1"])
    loss, d, g = torch.empty(1), torch.empty_like(p1), torch.tensor([0.3])
    assert harness.nr_cpu_consistency_loss(vp(p0), vp(p1), 1, 50, 8, vp(loss), None, None) == 0
    assert harness.nr_cpu_consistency_loss(vp(p0), vp(p1), 1, 50, 8, None, vp(g), vp(d)) == 0
    close(loss, G["consist_loss"])
    close(d, G["consist_grad"], rtol=1e-4)
    # predict_mean: values, mean-head parameter gradients through the packed layout, map gradient
    from neuray_b200 import backward
    params = decoder_state(G)
    wp = ref_packers.pack_pass_weights(params, "dist_decoder", "agg_net", torch.device("cpu"))[0]
    plan = ref_packers.point_index_map_cpu(params, "dist_decoder", "agg_net")
    rf, gm = f(G["mean_ray_feats"]), f(G["mean_gout"])
    mean, d_w, d_map = torch.empty(3, 40, 2), torch.zeros_like(wp), torch.zeros_like(rf)
    q = _lib.NrDepthMeanParams()
    q.map, q.coords, q.rfn, q.pn, q.h, q.w, q.fh, q.fw = rf.data_ptr(), coords.data_ptr(), 3, 40, 24, 32, 6, 8
    q.w_point[0], q.mean[0] = wp.data_ptr(), mean.data_ptr()
    assert harness.nr_cpu_depth_mean(C.byref(q)) == 0
    close(mean, G["mean_out"])
    q.d_mean[0], q.d_w_point[0], q.d_map = gm.data_ptr(), d_w.data_ptr(), d_map.data_ptr()
    assert harness.nr_cpu_depth_mean(C.byref(q)) == 0
    close(d_map, G["mean_d_ray_feats"], rtol=1e-4, atol=1e-6)
    grads = backward.unpack_point_grads(plan, d_w)
    for k, v in G.items():
        if k.startswith("mean_g_"):
            close(grads["dist_decoder." + k[7:]], v, rtol=1e-4, atol=1e-6)
    others = [k for k in grads if ".mean_decoder." not in k]
    assert others and all(float(grads[k].abs().max()) == 0.0 for k in others)


# ---- GPU ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_cuda_losses_match_the_reference_golden():
    from neuray_b200 import losses
    G = {k: v.cuda() for k, v in golden().items()}
    for tag, use in (("masked", True), ("plain", False)):
        pr = G["render_pr"].clone().requires_grad_(True)
        out = losses.RenderLoss({"use_ray_mask": use})({"pixel_colors_gt": G["render_gt"], "pixel_colors_nr": pr, "ray_mask": G["render_mask"]}, {}, 0)
        assert set(out) == {"loss_rgb_nr"}
        close(out["loss_rgb_nr"].detach(), G[f"render_{tag}_loss"])
        close(torch.autograd.grad(out["loss_rgb_nr"].sum() * 1.7, pr)[0], G[f"render_{tag}_grad"])
    for tag, kind, gso in DEPTH_CASES:
        dp = G["depth_pr"].clone().requires_grad_(True)
        data_gt = {"ref_imgs_info": {"true_depth": G["true_depth"], "depth": G["aug_depth"], "depth_range": G["depth_range"]},
                   "scene_name": "gso/x" if gso else "dtu_train/scan1"}
        out = losses.DepthLoss({"depth_loss_type": kind})({"depth_coords": G["depth_coords"], "depth_mean": dp, "depth_mean_fine": dp,
                                                          "pixel_colors_nr": G["render_pr"]}, data_gt, 0)
        assert set(out) == {"loss_depth", "loss_depth_fine"}
        close(out["loss_depth"].detach(), G[f"depth_{tag}_loss"])
        close(torch.autograd.grad((out["loss_depth"] * G["depth_gscale"]).sum(), dp)[0], G[f"depth_{tag}_grad"])
    p1 = G["consist_p1"].clone().requires_grad_(True)
    out = losses.ConsistencyLoss({})({"hit_prob_nr": G["consist_p0"], "hit_prob_self": p1}, {}, 0)
    close(out["loss_prob"].detach(), G["consist_loss"])
    close(torch.autograd.grad(out["loss_prob"].sum() * 0.3, p1)[0], G["consist_grad"], rtol=1e-4)
    assert losses.ConsistencyLoss({})({"hit_prob_nr": G["consist_p0"]}, {}, 0) == {}
    assert float(losses.DepthLoss({})({"pixel_colors_nr": G["render_pr"]}, {"ref_imgs_info": {}}, 0)["loss_depth"]) == 0.0


@pytest.mark.gpu
def test_cuda_predict_mean_for_depth_loss_matches_the_oracle():
    """Training shape (cfg5: 8 views 304x400, 8192 coordinates, coarse + fine decoder): values, the gradients of both mean
    heads and of ray_feats, against the oracle's autograd; the coordinates are drawn like the reference does (randperm)."""
    from neuray_b200 import losses, renderer, synthetic
    cfg = {"use_hierarchical_sampling": True, "dist_decoder_cfg": {"use_vis": False}, "depth_sample_num": 64, "fine_depth_sample_num": 64,
           "agg_net_cfg": {"sample_num": 64}, "fine_agg_net_cfg": {"sample_num": 64}, "depth_loss_coords_num": 8192}
    W = synthetic.make_weights(cfg, seed=6)
    net = renderer.NeuralRayRenderPath(cfg)
    net.load_state_dict(W, strict=True)
    net.cuda()
    rs = np.random.RandomState(8)
    rfn, h, w = 8, 304, 400
    ray_feats = torch.from_numpy(rs.standard_normal((rfn, 32, h // 4, w // 4)).astype(np.float32))
    ref = {"imgs": torch.zeros(rfn, 3, h, w, device="cuda"), "ray_feats": ray_feats.cuda().requires_grad_(True)}
    torch.manual_seed(5)
    out = losses.predict_mean_for_depth_loss(net, ref)
    assert set(out) == {"depth_mean", "depth_coords", "depth_mean_2", "depth_mean_fine", "depth_mean_fine_2"}
    assert out["depth_coords"].shape == (rfn, 8192, 2) and out["depth_coords"].dtype == torch.int64
    coords = out["depth_coords"].cpu()
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    rf = ray_feats.clone().requires_grad_(True)
    want_c = orc.predict_mean(Wg, "dist_decoder", rf, coords, h, w)
    want_f = orc.predict_mean(Wg, "fine_dist_decoder", rf, coords, h, w)
    close(out["depth_mean"].detach().cpu(), want_c[..., 0].detach(), rtol=1e-4, atol=1e-5)
    close(out["depth_mean_2"].detach().cpu(), want_c[..., 1].detach(), rtol=1e-4, atol=1e-5)
    close(out["depth_mean_fine"].detach().cpu(), want_f[..., 0].detach(), rtol=1e-4, atol=1e-5)
    g1 = torch.from_numpy(rs.standard_normal((rfn, 8192)).astype(np.float32))
    g2 = torch.from_numpy(rs.standard_normal((rfn, 8192)).astype(np.float32))
    ((out["depth_mean"] * g1.cuda()).sum() + (out["depth_mean_fine"] * g2.cuda()).sum() + 0.5 * out["depth_mean_2"].sum()).backward()
    ((want_c[..., 0] * g1).sum() + (want_f[..., 0] * g2).sum() + 0.5 * want_c[..., 1].sum()).backward()
    torch.cuda.synchronize()
    rel = lambda a, b: float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))
    assert rel(ref["ray_feats"].grad.cpu(), rf.grad) < 1e-3
    named = dict(net.named_parameters())
    checked = 0
    for k, v in Wg.items():
        if ".mean_decoder." in k:
            assert rel(named[k].grad.cpu(), v.grad) < 2e-3, k       # 65 536 atomically accumulated terms per element
            checked += 1
        else:
            assert named[k].grad is None and v.grad is None, k
    assert checked == 12
