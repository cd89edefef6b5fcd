"""CostVolumeInitNet's frozen MVSNet (SURVEY.md 8f row 4; reference network/init_net.py:113-168, network/mvsnet/): the softmaxed
cost volume and the regressed depth of construct_cost_volume_with_src.

CPU: the oracle's restatement and the product's graph + per-voxel routines (csrc/nr_mvs_graph.cuh, csrc/nr_mvs.cuh) executed on
the host by tests/cpu_harness/mvs_cpu_harness.cu, against tests/golden/mvsnet.npz = outputs of the UNMODIFIED reference
(oracle/gen_golden_mvsnet.py).  GPU: the CUDA path through neuray_b200.init_nets against the same golden and the oracle."""
import ctypes as C
import json
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import neuray_oracle as orc
from golden_io import GOLDEN_DIR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")


def golden():
    z = np.load(os.path.join(GOLDEN_DIR, "mvsnet.npz"))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    ref = {k[4:]: t(z[k]) for k in z.files if k.startswith("ref_")}
    src = {k[4:]: t(z[k]) for k in z.files if k.startswith("src_")}
    W = orc.mvs_test_weights(json.loads(str(z["shapes"])), 31)
    out = {k: t(z[k]) for k in ("train_cost", "train_depth", "eval_cost", "eval_depth")}
    return ref, src, W, int(z["dn"]), out


@pytest.mark.parametrize("tag", ["train", "eval"])
def test_oracle_matches_the_reference(tag):
    ref, src, W, dn, out = golden()
    cost, depth = orc.mvs_cost_volume(W, "", ref, src, dn, tag == "train")
    assert cost.shape == out[f"{tag}_cost"].shape
    assert torch.allclose(cost, out[f"{tag}_cost"], atol=2e-5), float((cost - out[f"{tag}_cost"]).abs().max())
    assert torch.allclose(depth, out[f"{tag}_depth"], atol=1e-4), float((depth - out[f"{tag}_depth"]).abs().max())


@pytest.fixture(scope="module")
def harness():
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    os.makedirs(BUILD, exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpu_harness", "mvs_cpu_harness.cu")
    lib = os.path.join(BUILD, "libmvs_cpu_harness.so")
    deps = [src] + [os.path.join(ROOT, "neuray_b200", "csrc", f) for f in ("nr_mvs.cuh", "nr_mvs_graph.cuh", "nr_encoder_graph.cuh", "nr_conv.cuh")]
    if not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in deps):
        subprocess.run(["nvcc", "-shared", "-Xcompiler", "-fPIC", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                        src, "-o", lib], check=True)
    return C.CDLL(lib)


def test_graph_on_the_host_matches_the_reference(harness):
    ref, src, W, dn, out = golden()
    assert harness.nr_cpu_mvsnet_tensors() == len(W)
    params = [t.contiguous() for t in W.values()]
    arr = (C.c_void_p * len(params))(*[t.data_ptr() for t in params])
    rfn, _, h, w = ref["imgs"].shape
    sn, nn = src["imgs"].shape[0], ref["nn_ids"].shape[1]
    f = lambda t: t.contiguous().float()
    keep = [f(ref["imgs"]), f(src["imgs"]), f(ref["Ks"]), f(ref["poses"]), f(src["Ks"]), f(src["poses"]), f(ref["depth_range"]),
            ref["nn_ids"].to(torch.int32).contiguous()]
    prob, depth = torch.full((rfn, h // 4, w // 4, dn), 7.0), torch.full((rfn, h // 4, w // 4), 7.0)
    rc = harness.nr_cpu_mvsnet(arr, len(params), *[C.c_void_p(t.data_ptr()) for t in keep], rfn, sn, nn, h, w, dn, 1,
                               C.c_void_p(prob.data_ptr()), C.c_void_p(depth.data_ptr()))
    assert rc == 0
    e1 = float((prob.permute(0, 3, 1, 2) - out["train_cost"]).abs().max())
    e2 = float((depth - out["train_depth"]).abs().max())
    assert e1 < 5e-5 and e2 < 3e-4, (e1, e2)


# ---- the whole CostVolumeInitNet (init_net.py:205-254) ---------------------------------------------------------------------------

def cv_golden():
    z = np.load(os.path.join(GOLDEN_DIR, "cost_volume_init_net.npz"))
    shapes = json.loads(str(z["shapes"]))
    mv = {k[7:]: v for k, v in shapes.items() if k.startswith("mvsnet.")}
    rest = {k: v for k, v in shapes.items() if not k.startswith("mvsnet.") and not k.startswith("imagenet_")}
    W = {"mvsnet." + k: v for k, v in orc.mvs_test_weights(mv, 31).items()}
    W.update(orc.encoder_test_weights(rest, 32))
    return W, {k: torch.from_numpy(np.ascontiguousarray(z[k])) for k in ("train", "eval")}


def test_cost_volume_init_net_oracle_matches_the_reference():
    ref, src, _, _, _ = golden()
    W, out = cv_golden()
    got = orc.cost_volume_init_net(W, "", ref, src, True, sn=16)
    assert got.shape == out["train"].shape
    assert float((got - out["train"]).abs().max()) < 1e-4 * float(out["train"].abs().max())


@pytest.fixture(scope="module")
def conv_harness():
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    os.makedirs(BUILD, exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpu_harness", "conv_cpu_harness.cu")
    lib = os.path.join(BUILD, "libconv_cpu_harness.so")
    deps = [src] + [os.path.join(ROOT, "neuray_b200", "csrc", f) for f in ("nr_conv.cuh", "nr_encoder_graph.cuh", "nr_common.cuh")]
    if not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in deps):
        subprocess.run(["nvcc", "-shared", "-Xcompiler", "-fPIC", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                        src, "-o", lib], check=True)
    return C.CDLL(lib)


def test_cost_volume_init_net_graphs_on_the_host_match_the_reference(harness, conv_harness):
    """MVSNet graph -> nr_extract_depth's arithmetic -> the head's graph (ResUNetLight 3->32 with stages [2,3,6], volume_conv2d,
    depth_conv with its single channel packed into 16, out_conv on 96 channels), all on the host, against the unmodified module."""
    ref, src, _, dn, _ = golden()
    W, out = cv_golden()
    rfn, _, h, w = ref["imgs"].shape
    sn_views, nn = src["imgs"].shape[0], ref["nn_ids"].shape[1]
    f = lambda t: t.contiguous().float()
    mv = [W[k].contiguous() for k in W if k.startswith("mvsnet.")]
    arr = (C.c_void_p * len(mv))(*[t.data_ptr() for t in mv])
    keep = [f(ref["imgs"]), f(src["imgs"]), f(ref["Ks"]), f(ref["poses"]), f(src["Ks"]), f(src["poses"]), f(ref["depth_range"]),
            ref["nn_ids"].to(torch.int32).contiguous()]
    prob, depth = torch.empty(rfn, h // 4, w // 4, dn), torch.empty(rfn, h // 4, w // 4)
    assert harness.nr_cpu_mvsnet(arr, len(mv), *[C.c_void_p(t.data_ptr()) for t in keep], rfn, sn_views, nn, h, w, dn, 1,
                                 C.c_void_p(prob.data_ptr()), C.c_void_p(depth.data_ptr())) == 0
    depth_norm = orc.extract_depth_for_init(ref["depth_range"], depth[:, None])[:, 0].contiguous()
    head = [W[k].contiguous() for k in W if not k.startswith("mvsnet.")]
    assert conv_harness.nr_cpu_cost_volume_head_tensors(dn) == len(head)
    harr = (C.c_void_p * len(head))(*[t.data_ptr() for t in head])
    buf = torch.full((rfn, h // 4, w // 4, 64), 5.0)
    rc = conv_harness.nr_cpu_cost_volume_head(dn, harr, len(head), C.c_void_p(keep[0].data_ptr()), C.c_void_p(prob.data_ptr()),
                                              C.c_void_p(depth_norm.data_ptr()), rfn, h, w, C.c_void_p(buf.data_ptr()), 64, 0)
    assert rc == 0
    got = buf[..., :32].permute(0, 3, 1, 2)
    err = float((got - out["train"]).abs().max())
    assert err < 2e-4 * float(out["train"].abs().max()), err
    assert bool(torch.all(buf[..., 32:] == 5.0))


# ---- GPU -------------------------------------------------------------------------------------------------------------------------

def _module(W, sn):
    from neuray_b200 import init_nets
    net = init_nets.CostVolumeInitNet({"cost_volume_sn": sn})
    missing, unexpected = net.load_state_dict(W, strict=False)
    assert not unexpected and set(missing) == {"imagenet_mean", "imagenet_std"}
    return net.cuda().eval()


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["train", "eval"])
def test_cuda_cost_volume_init_net_matches_the_reference_golden(tag):
    from neuray_b200 import init_nets, synthetic
    ref, src, _, dn, mv_out = golden()
    W, out = cv_golden()
    net = _module(W, dn)
    dref, dsrc = synthetic.to_device(ref, "cuda"), synthetic.to_device(src, "cuda")
    with torch.no_grad():
        prob, depth = init_nets.mvsnet_cost_volume(net, dref, dsrc, tag == "train")
        got = net(dref, dsrc, tag == "train")
    torch.cuda.synchronize()
    e1 = float((prob.permute(0, 3, 1, 2).cpu() - mv_out[f"{tag}_cost"]).abs().max())
    e2 = float((depth.cpu() - mv_out[f"{tag}_depth"]).abs().max())
    assert e1 < 5e-5 and e2 < 3e-4, (e1, e2)
    err = float((got.cpu() - out[tag]).abs().max())
    assert err < 2e-4 * float(out[tag].abs().max()), err


@pytest.mark.gpu
def test_cuda_cost_volume_init_net_matches_the_oracle_with_the_evaluation_resize():
    """800x800 in eval mode: MVSNet runs at 640x640 and the cost volume is resized back to 200x200 (init_net.py:120-139,155);
    cost_volume_sn = 64 as in the shipped configs."""
    from neuray_b200 import init_nets, synthetic
    _, ref = synthetic.make_scene(800, 800, 1, seed=41, smooth=2, pad=32, depth_range=(2.0, 6.0), arc_deg=25.0)
    _, src = synthetic.make_scene(800, 800, 2, seed=42, smooth=2, pad=32, depth_range=(2.0, 6.0), arc_deg=30.0)
    ref = {k: ref[k] for k in ("imgs", "poses", "Ks", "depth_range")}
    src = {k: src[k] for k in ("imgs", "poses", "Ks")}
    ref["nn_ids"] = torch.tensor([[1, 0]])
    shapes = {k: list(v.shape) for k, v in init_nets.CostVolumeInitNet({"cost_volume_sn": 64}).state_dict().items()}
    mv = {k[7:]: v for k, v in shapes.items() if k.startswith("mvsnet.")}
    rest = {k: v for k, v in shapes.items() if not k.startswith("mvsnet.") and not k.startswith("imagenet_")}
    W = {"mvsnet." + k: v for k, v in orc.mvs_test_weights(mv, 33).items()}
    W.update(orc.encoder_test_weights(rest, 34))
    net = _module(W, 64)
    with torch.no_grad():
        prob, depth = init_nets.mvsnet_cost_volume(net, synthetic.to_device(ref, "cuda"), synthetic.to_device(src, "cuda"), False)
        got = net(synthetic.to_device(ref, "cuda"), synthetic.to_device(src, "cuda"), False)
    torch.cuda.synchronize()
    cost_o, depth_o = orc.mvs_cost_volume(W, "mvsnet.", ref, src, 64, False)
    assert prob.shape == (1, 200, 200, 64)
    e1 = (prob.permute(0, 3, 1, 2).cpu() - cost_o).abs()
    e2 = (depth.cpu() - depth_o).abs()
    assert float(e1.max()) < 2e-4 and float(e2.max()) < 2e-3, (float(e1.max()), float(e2.max()))
    want = orc.cost_volume_init_net(W, "", ref, src, False, sn=64)
    err = (got.cpu() - want).abs()
    assert float(err.max()) < 5e-4 * float(want.abs().max()) and float(err.mean()) < 1e-5 * float(want.abs().max()), (float(err.max()), float(err.mean()), float(want.abs().max()))      # measured 6.7e-4 / 5.6e-5 at |out| <= 31


@pytest.mark.gpu
def test_gen_frame_renderer_with_the_cost_volume_init_net():
    """NeuralRayGenFrameRenderer(init_net_type='cost_volume'): MVSNet + head -> encoders -> render against the oracle's stages."""
    from gen_golden import flat_cfg
    from neuray_b200 import renderer, synthetic
    import test_encoders_gpu as teg
    cfg = {"init_net_type": "cost_volume", "init_net_cfg": {"cost_volume_sn": 16}, "use_hierarchical_sampling": True, "dist_decoder_cfg": {"use_vis": False},
           "depth_sample_num": 32, "fine_depth_sample_num": 32, "agg_net_cfg": {"sample_num": 32}, "fine_agg_net_cfg": {"sample_num": 32},
           "render_depth": True, "ray_batch_num": 200, "depth_loss_coords_num": 32}
    ref, src, _, dn, _ = golden()
    Wi, _ = cv_golden()
    _, img_w, vis_w = teg.golden()
    que, _ = synthetic.make_scene(64, 96, 2, seed=23, smooth=2, pad=32, depth_range=(2.0, 6.0), arc_deg=30.0)
    que = synthetic.slice_rays(que, 1000, 1400)
    W = synthetic.make_weights(cfg, seed=8)
    full = dict(W)
    full.update({"image_encoder." + k: v for k, v in img_w.items()})
    full.update({"vis_encoder." + k: v for k, v in vis_w.items()})
    full.update({"init_net." + k: v for k, v in Wi.items()})
    net = renderer.NeuralRayGenFrameRenderer(cfg)
    missing, unexpected = net.load_state_dict(full, strict=False)
    assert not unexpected and set(missing) == {"init_net.imagenet_mean", "init_net.imagenet_std"}
    net.cuda().eval()
    data = {"que_imgs_info": synthetic.to_device(que, "cuda"), "ref_imgs_info": synthetic.to_device(ref, "cuda"),
            "src_imgs_info": synthetic.to_device(src, "cuda"), "eval": True}
    torch.manual_seed(2)
    with torch.no_grad():
        out = net(data)
    torch.cuda.synchronize()
    ray_in = orc.cost_volume_init_net(Wi, "", ref, src, False, sn=dn)
    img_feats = orc.res_unet_light(img_w, "", ref["imgs"])
    ray_feats = orc.vis_encoder(vis_w, "", ray_in, img_feats)
    rr = {k: ref[k] for k in ("imgs", "poses", "Ks", "depth_range")}
    gold = orc.render(W, flat_cfg({**renderer.base_cfg, **cfg}), que, dict(rr, ray_feats=ray_feats, img_feats=img_feats), False, ray_batch_num=200)
    err = float((out["pixel_colors_nr"].cpu() - gold["pixel_colors_nr"]).abs().max())
    assert err < 5e-4, err
    assert torch.equal(out["ray_mask"].cpu(), gold["ray_mask"])
    assert "depth_mean" in out


def test_evaluation_resize_path_on_the_host(harness):
    """800x800 in eval mode (init_net.py:120-139,155): images resized to 640x640, MVSNet at 160x160, the cost volume resized back to
    200x200 before the softmax -- the product's graph on the host against the oracle (8 depth planes, one neighbour)."""
    from neuray_b200 import synthetic
    _, ref = synthetic.make_scene(800, 800, 1, seed=51, smooth=2, pad=32, depth_range=(2.0, 6.0), arc_deg=20.0)
    _, src = synthetic.make_scene(800, 800, 1, seed=52, smooth=2, pad=32, depth_range=(2.0, 6.0), arc_deg=26.0)
    ref = {k: ref[k] for k in ("imgs", "poses", "Ks", "depth_range")}
    src = {k: src[k] for k in ("imgs", "poses", "Ks")}
    ref["nn_ids"] = torch.tensor([[0]])
    _, _, W, _, _ = golden()
    dn = 8
    cost_o, depth_o = orc.mvs_cost_volume(W, "", ref, src, dn, False)
    assert cost_o.shape == (1, dn, 200, 200)
    params = [t.contiguous() for t in W.values()]
    arr = (C.c_void_p * len(params))(*[t.data_ptr() for t in params])
    f = lambda t: t.contiguous().float()
    keep = [f(ref["imgs"]), f(src["imgs"]), f(ref["Ks"]), f(ref["poses"]), f(src["Ks"]), f(src["poses"]), f(ref["depth_range"]),
            ref["nn_ids"].to(torch.int32).contiguous()]
    prob, depth = torch.empty(1, 200, 200, dn), torch.empty(1, 200, 200)
    rc = harness.nr_cpu_mvsnet(arr, len(params), *[C.c_void_p(t.data_ptr()) for t in keep], 1, 1, 1, 800, 800, dn, 0,
                               C.c_void_p(prob.data_ptr()), C.c_void_p(depth.data_ptr()))
    assert rc == 0
    e1 = float((prob.permute(0, 3, 1, 2) - cost_o).abs().max())
    e2 = float((depth - depth_o).abs().max())
    assert e1 < 1e-4 and e2 < 1e-3, (e1, e2)
