"""CPU: the hand-written backward of a render pass (csrc/nr_train_math.cuh, the code the CUDA kernels run per point /
sample / ray) compiled as HOST code and checked against PyTorch autograd over the same pass.  No GPU needed: nvcc
compiles the __host__ __device__ routines for the CPU (tests/cpu_harness/train_cpu_harness.cu)."""
import ctypes as C
import os
import shutil
import subprocess

import pytest
import torch

import ref_packers as weights
import torch_restatement as autograd_path
from neuray_b200 import _lib, backward, renderer, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")


@pytest.fixture(scope="module")
def harness():
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    os.makedirs(BUILD, exist_ok=True)
    so = os.path.join(BUILD, "libnr_train_cpu.so")
    src = os.path.join(ROOT, "tests", "cpu_harness", "train_cpu_harness.cu")
    deps = [src, os.path.join(ROOT, "neuray_b200", "csrc", "nr_train_math.cuh"), os.path.join(ROOT, "neuray_b200", "csrc", "nr_common.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.run(["nvcc", "-shared", "-Xcompiler", "-fPIC", "-O1", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                        "-o", so, src], check=True, capture_output=True)
    lib = C.CDLL(so)
    lib.nr_train_cpu.restype = C.c_int
    lib.nr_train_cpu.argtypes = [C.c_void_p, C.c_void_p]
    return lib


def native_pass(harness, params, dec, agg, use_vis, que, ref, coords, que_depth, g_pix, g_hit, g_dep, var_bias=0.05):
    """Runs the hand-written backward of one pass on the host.  params: {name: tensor} of the pass' modules; coords
    [1,rn,2], que_depth [1,rn,dn]; upstream gradients [1,rn,3] / [1,rn,dn] / [1,rn] (None = zero).
    Returns (tape buffers, d_feat [rfn,fh,fw,64], {name: grad})."""
    names = list(params)
    rfn = ref["imgs"].shape[0]
    rays, dn = que_depth.shape[1:]
    pos_enc = weights.posenc_table(dn)
    wp, wr = weights.pack_pass_weights(params, dec, agg, torch.device("cpu"))
    feat = torch.cat([ref["ray_feats"], ref["img_feats"]], 1).permute(0, 2, 3, 1).contiguous()
    rgb = torch.cat([ref["imgs"], torch.zeros_like(ref["imgs"][:, :1])], 1).permute(0, 2, 3, 1).contiguous()
    vp = weights.view_param_block(ref["poses"], ref["Ks"], ref["depth_range"])
    cam = weights.camera_block(que["poses"][0], que["Ks"][0], que["depth_range"][0])
    cc, qd = coords[0].contiguous().float(), que_depth[0].contiguous().float()
    p = _lib.NrPassParams()
    p.coords, p.que_depth, p.que_cam, p.rn, p.dn = cc.data_ptr(), qd.data_ptr(), cam.data_ptr(), rays, dn
    p.feat, p.rgb, p.view_params = feat.data_ptr(), rgb.data_ptr(), vp.data_ptr()
    p.rfn, p.h, p.w, p.fh, p.fw = rfn, ref["imgs"].shape[2], ref["imgs"].shape[3], ref["ray_feats"].shape[2], ref["ray_feats"].shape[3]
    p.w_point, p.w_ray, p.pos_enc = wp.data_ptr(), wr.data_ptr(), pos_enc.data_ptr()
    p.use_vis, p.var_bias = int(use_vis), var_bias
    shapes = backward.tape_shapes(rfn, rays * dn)
    bufs = {k: torch.full(sh, float("nan")) for k, sh in shapes.items()}
    d_feat = torch.zeros_like(feat)
    b = _lib.NrBwdParams()
    keep = [t[0].contiguous().float() if t is not None else None for t in (g_pix, g_hit, g_dep)]
    b.d_pixel_colors, b.d_hit_prob, b.d_render_depth = (t.data_ptr() if t is not None else None for t in keep)
    b.tape_row, b.grad_row = bufs["tape_row"].data_ptr(), bufs["grad_row"].data_ptr()
    b.tape_point, b.grad_point = bufs["tape_point"].data_ptr(), bufs["grad_point"].data_ptr()
    b.d_feat = d_feat.data_ptr()
    assert harness.nr_train_cpu(C.addressof(p), C.addressof(b)) == 0
    grads = backward.assemble_param_grads(names, dec, agg, 4 if use_vis else 3, bufs["tape_row"], bufs["grad_row"], bufs["tape_point"],
                                          bufs["grad_point"], rfn * rays * dn, rays * dn)
    return bufs, d_feat, grads


def run_case(harness, rfn, use_vis, dn=8, rays=5, seed=0, with_hit=True, full_res=False):
    torch.manual_seed(seed)
    cfg = {"depth_sample_num": dn, "agg_net_cfg": {"sample_num": dn}, "dist_decoder_cfg": {"use_vis": use_vis}, "render_depth": True}
    que, ref = synthetic.make_scene(40, 48, rfn, seed=20 + seed, smooth=2)
    if full_res:      # feature maps at image resolution: the align_corners sampling path (ops.py:14-34)
        ph, pw = ref["imgs"].shape[-2:]
        ref["ray_feats"], ref["img_feats"] = torch.randn(rfn, 32, ph, pw), torch.randn(rfn, 32, ph, pw)
    n = que["coords"].shape[1]
    idx = torch.randperm(n)[:rays]
    # push one ray outside most views so that masks / padding paths are exercised
    coords = que["coords"][:, idx].clone()
    W = synthetic.make_weights(cfg, seed=seed)
    dec, agg = "dist_decoder", "agg_net"
    names = [k for k in W if k.startswith(dec + ".") or k.startswith(agg + ".")]
    import neuray_oracle as orc
    que_depth, _ = orc.sample_depth(que["depth_range"], coords, dn, False)            # [1,rays,dn]
    pos_enc = weights.posenc_table(dn)
    g_pix, g_hit, g_dep = torch.randn(1, rays, 3), torch.randn(1, rays, dn) * 0.5, torch.randn(1, rays) * 0.3

    # ---- autograd reference ----
    P = {k: W[k].clone().requires_grad_(True) for k in names}
    rref = {k: ref[k] for k in ("poses", "Ks", "depth_range", "imgs")}
    rref["ray_feats"] = ref["ray_feats"].clone().requires_grad_(True)
    rref["img_feats"] = ref["img_feats"].clone().requires_grad_(True)
    cfgv = {"use_vis_prob": use_vis, "var_bias": 0.05}
    pix, hit, dep = autograd_path.render_pass_torch(P, dec, agg, cfgv, que_depth, coords, que["poses"], que["Ks"], que["depth_range"],
                                                    rref, pos_enc)
    loss = (pix * g_pix).sum() + (dep * g_dep).sum() + ((hit * g_hit).sum() if with_hit else 0.0)
    loss.backward()

    # ---- hand-written backward on the host ----
    bufs, d_feat, grads = native_pass(harness, {k: W[k] for k in names}, dec, agg, use_vis, que, ref, coords, que_depth,
                                      g_pix, g_hit if with_hit else None, g_dep)
    s = _lib.bwd_slot
    # recomputed forward agrees with the reference pass
    alpha = backward._slots(bufs["tape_point"], s("P_ALPHA"), 1, rays * dn).reshape(rays, dn)
    T = torch.cumprod(torch.cat([torch.ones(rays, 1), 1 - alpha + 1e-10], 1), 1)[:, :-1]
    assert torch.allclose(alpha * T, hit[0].detach(), atol=2e-5), (alpha * T - hit[0].detach()).abs().max()
    worst = {}
    for k in names:
        ga, gn = P[k].grad, grads[k]
        if ga is None:
            assert gn is None or float(gn.abs().max()) == 0.0, k
            continue
        assert gn is not None, k
        assert gn.shape == ga.shape, (k, gn.shape, ga.shape)
        err = (gn - ga).abs().max().item()
        scale = ga.abs().max().item()
        worst[k] = (err, scale)
        assert err <= 2e-4 * max(scale, 1e-3) + 2e-6, (k, err, scale)
    drf, dimf = backward.feat_grads_to_nchw(d_feat)
    for name, gn, ga in (("ray_feats", drf, rref["ray_feats"].grad), ("img_feats", dimf, rref["img_feats"].grad)):
        err, scale = (gn - ga).abs().max().item(), ga.abs().max().item()
        assert err <= 2e-4 * max(scale, 1e-3) + 2e-6, (name, err, scale)
    return worst


@pytest.mark.parametrize("rfn,use_vis", [(3, False), (5, True), (8, False)])
def test_hand_written_backward_matches_autograd(harness, rfn, use_vis):
    worst = run_case(harness, rfn, use_vis, seed=rfn)
    assert len(worst) > 60


def test_backward_without_hit_prob_gradient(harness):
    run_case(harness, 4, True, dn=6, rays=3, seed=9, with_hit=False)


@pytest.mark.parametrize("use_vis", [False, True])
def test_self_hit_prob_forward_and_backward(harness, use_vis):
    """nr_self_hit_prob's routine (host build) against the PyTorch restatement of predict_self_hit_prob
    (reference renderer.py:137-155) and autograd over it: values, every decoder parameter gradient (through the packed
    layout and the position -> parameter index map) and the gradient of the query feature map."""
    torch.manual_seed(3)
    dn, rays = 12, 9
    cfg = {"depth_sample_num": dn, "agg_net_cfg": {"sample_num": dn}, "dist_decoder_cfg": {"use_vis": use_vis}}
    que, ref = synthetic.make_scene(40, 48, 3, seed=31, smooth=2)
    coords = que["coords"][:, torch.randperm(que["coords"].shape[1])[:rays]].clone()
    fmap = torch.randn(1, 32, 10, 12)
    W = synthetic.make_weights(cfg, seed=5)
    dec, agg = "dist_decoder", "agg_net"
    names = [k for k in W if k.startswith(dec + ".") or k.startswith(agg + ".")]
    import neuray_oracle as orc
    que_depth, _ = orc.sample_depth(que["depth_range"], coords, dn, False)
    g_hit = torch.randn(1, rays, dn)
    P = {k: W[k].clone().requires_grad_(True) for k in names}
    fm = fmap.clone().requires_grad_(True)
    ref_hit = autograd_path.self_hit_prob_torch(P, dec, use_vis, 0.05, fm, coords, 40, 48, que_depth, que["depth_range"])
    (ref_hit * g_hit).sum().backward()

    params = {k: W[k] for k in names}
    plan = weights.point_index_map_cpu(params, dec, agg)
    wp = weights.pack_pass_weights(params, dec, agg, torch.device("cpu"))[0]
    cc, qd, m0, gh = coords[0].contiguous(), que_depth[0].contiguous(), fmap[0].contiguous(), g_hit[0].contiguous()
    hit, d_w, d_map = torch.empty(rays, dn), torch.zeros_like(wp), torch.zeros_like(m0)
    p = _lib.NrSelfParams()
    p.map, p.coords, p.que_depth, p.w_point = m0.data_ptr(), cc.data_ptr(), qd.data_ptr(), wp.data_ptr()
    p.rn, p.dn, p.h, p.w, p.fh, p.fw, p.use_vis = rays, dn, 40, 48, 10, 12, int(use_vis)
    rng = que["depth_range"][0].contiguous().float()
    p.depth_range, p.var_bias = rng.data_ptr(), 0.05
    p.hit, p.d_hit, p.d_w_point, p.d_map = hit.data_ptr(), gh.data_ptr(), d_w.data_ptr(), d_map.data_ptr()
    harness.nr_self_cpu.restype = C.c_int
    harness.nr_self_cpu.argtypes = [C.c_void_p]
    assert harness.nr_self_cpu(C.addressof(p)) == 0
    assert torch.allclose(hit, ref_hit[0].detach(), atol=2e-6), (hit - ref_hit[0].detach()).abs().max()
    grads = backward.unpack_point_grads(plan, d_w)
    checked = 0
    for k in names:
        ga = P[k].grad
        if ga is None or not k.startswith(dec + "."):
            assert float(grads[k].abs().max()) == 0.0, k
            continue
        err, scale = float((grads[k] - ga).abs().max()), float(ga.abs().max())
        assert err <= 2e-4 * max(scale, 1e-3) + 2e-6, (k, err, scale)
        checked += 1
    assert checked == (24 if use_vis else 18)
    assert float((d_map - fm.grad[0]).abs().max()) <= 2e-4 * float(fm.grad.abs().max()) + 2e-6


def test_backward_single_view_and_full_resolution_maps(harness):
    """One reference view (every pool degenerates to its single element) and feature maps at image resolution."""
    run_case(harness, 1, False, dn=5, rays=4, seed=2)
    run_case(harness, 4, True, dn=6, rays=4, seed=4, full_res=True)


@pytest.mark.parametrize("name", ["train8", "views10"])
def test_hand_written_backward_matches_the_reference_gradients(harness, name):
    """The gradients the UNMODIFIED reference's autograd produces (tests/golden/grads_*.npz, oracle/gen_golden_grads.py:
    coarse + fine render_by_depth on the golden case's stage rays, fixed linear loss) against the hand-written backward:
    every parameter of both passes' modules and the gradients of ray_feats / img_feats (sum of both passes)."""
    import numpy as np
    from golden_io import GOLDEN_DIR, GoldenCase
    g = GoldenCase(name)
    z = np.load(os.path.join(GOLDEN_DIR, f"grads_{name}.npz"))
    lw = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("lw_")}
    gold = {k[5:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("grad_")}
    sel = g.stage_sel
    coords = g.que["coords"][:, sel].contiguous()
    use_vis = g.cfg.get("dist_decoder_cfg", {}).get("use_vis", True)      # compute_prob follows the COARSE decoder (renderer.py:75)
    total_feat = None
    checked = 0
    for dec, agg, depth, gp, gh, gd in (("dist_decoder", "agg_net", g.que_depth[:, sel], lw["gw_c"], lw["gh_c"], None),
                                        ("fine_dist_decoder", "fine_agg_net", g.que_depth_fine[:, sel], lw["gw_f"], None, lw["gd_f"])):
        params = {k: v for k, v in g.W.items() if k.startswith(dec + ".") or k.startswith(agg + ".")}
        bias = g.cfg.get(dec + "_cfg", {}).get("bias_val", 0.05)
        _, d_feat, grads = native_pass(harness, params, dec, agg, use_vis, g.que, g.ref, coords, depth.contiguous(), gp, gh, gd, bias)
        total_feat = d_feat if total_feat is None else total_feat + d_feat
        for k in params:
            if k not in gold:
                assert grads[k] is None or float(grads[k].abs().max()) == 0.0, k
                continue
            err, scale = float((grads[k] - gold[k]).abs().max()), float(gold[k].abs().max())
            assert err <= 3e-4 * max(scale, 1e-3) + 3e-6, (k, err, scale)
            checked += 1
    assert checked == len([k for k in gold if not k.startswith("ref_")])
    drf, dimf = backward.feat_grads_to_nchw(total_feat)
    for got, ref_g in ((drf, gold["ref_ray_feats"]), (dimf, gold["ref_img_feats"])):
        assert float((got - ref_g).abs().max()) <= 3e-4 * float(ref_g.abs().max()) + 3e-6


@pytest.mark.parametrize("name", ["train8", "views10"])
def test_float64_restatement_matches_the_reference_gradients(name):
    """The float64 restatement (tests/torch_restatement.py, autograd, every input cast to double) -- the reference the GPU
    backward is judged by in tests/test_backward_gpu.py -- against the unmodified reference's gradients on the golden
    case's stage rays, at the tolerance of the test above."""
    import numpy as np
    from golden_io import GOLDEN_DIR, GoldenCase
    g = GoldenCase(name)
    z = np.load(os.path.join(GOLDEN_DIR, f"grads_{name}.npz"))
    lw = {k[3:]: torch.from_numpy(z[k]).double() for k in z.files if k.startswith("lw_")}
    gold = {k[5:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("grad_")}
    sel = g.stage_sel
    d = lambda t: t.double()
    coords = d(g.que["coords"][:, sel])
    use_vis = g.cfg.get("dist_decoder_cfg", {}).get("use_vis", True)
    ref = {k: d(g.ref[k]) for k in ("poses", "Ks", "depth_range", "imgs")}
    ref["ray_feats"] = d(g.ref["ray_feats"]).requires_grad_(True)
    ref["img_feats"] = d(g.ref["img_feats"]).requires_grad_(True)
    checked = 0
    for dec, agg, depth, gp, gh, gd in (("dist_decoder", "agg_net", g.que_depth[:, sel], lw["gw_c"], lw["gh_c"], None),
                                        ("fine_dist_decoder", "fine_agg_net", g.que_depth_fine[:, sel], lw["gw_f"], None, lw["gd_f"])):
        P = {k: d(v).requires_grad_(True) for k, v in g.W.items() if k.startswith(dec + ".") or k.startswith(agg + ".")}
        cfgv = {"use_vis_prob": use_vis, "var_bias": g.cfg.get(dec + "_cfg", {}).get("bias_val", 0.05)}
        pix, hit, dep = autograd_path.render_pass_torch(P, dec, agg, cfgv, d(depth), coords, d(g.que["poses"]), d(g.que["Ks"]),
                                                        d(g.que["depth_range"]), ref, d(weights.posenc_table(depth.shape[-1])))
        loss = (pix * gp).sum() + ((hit * gh).sum() if gh is not None else 0.0) + ((dep * gd).sum() if gd is not None else 0.0)
        loss.backward()
        for k, p in P.items():
            if k not in gold:
                assert p.grad is None or float(p.grad.abs().max()) == 0.0, k
                continue
            err, scale = float((p.grad - gold[k].double()).abs().max()), float(gold[k].abs().max())
            assert err <= 3e-4 * max(scale, 1e-3) + 3e-6, (k, err, scale)
            checked += 1
    assert checked == len([k for k in gold if not k.startswith("ref_")])
    for got, ref_g in ((ref["ray_feats"].grad, gold["ref_ray_feats"]), (ref["img_feats"].grad, gold["ref_img_feats"])):
        assert float((got - ref_g.double()).abs().max()) <= 3e-4 * float(ref_g.abs().max()) + 3e-6


@pytest.mark.parametrize("name", ["train8", "views10"])
def test_self_hit_prob_matches_the_reference(harness, name):
    """predict_self_hit_prob as the unmodified reference computes it (values and autograd gradients stored in
    tests/golden/grads_*.npz) against nr_self_hit_prob's routine (host build) and against the oracle."""
    import numpy as np
    import neuray_oracle as orc
    from golden_io import GOLDEN_DIR, GoldenCase
    g = GoldenCase(name)
    z = np.load(os.path.join(GOLDEN_DIR, f"grads_{name}.npz"))
    t = lambda k: torch.from_numpy(z[k])
    sel = g.stage_sel
    coords, depth = g.que["coords"][:, sel].contiguous(), g.que_depth[:, sel].contiguous()
    use_vis = g.cfg.get("dist_decoder_cfg", {}).get("use_vis", True)
    # oracle
    q = dict(g.stage_que(), ray_feats=t("self_map"))
    o = orc.predict_self_hit_prob(g.W, g.flat_cfg(), q, depth, orc.depth2inv_dists(depth, g.que["depth_range"]), False)
    assert torch.allclose(o, t("self_hit"), atol=2e-6)
    # hand-written routine
    dec, agg = "dist_decoder", "agg_net"
    params = {k: v for k, v in g.W.items() if k.startswith(dec + ".") or k.startswith(agg + ".")}
    plan = weights.point_index_map_cpu(params, dec, agg)
    wp = weights.pack_pass_weights(params, dec, agg, torch.device("cpu"))[0]
    rays, dn = depth.shape[1:]
    m0, cc, qd, gh = t("self_map")[0].contiguous(), coords[0].contiguous(), depth[0].contiguous(), t("self_gs")[0].contiguous()
    hit, d_w, d_map = torch.empty(rays, dn), torch.zeros_like(wp), torch.zeros_like(m0)
    p = _lib.NrSelfParams()
    p.map, p.coords, p.que_depth, p.w_point = m0.data_ptr(), cc.data_ptr(), qd.data_ptr(), wp.data_ptr()
    p.rn, p.dn, p.h, p.w, p.fh, p.fw, p.use_vis = rays, dn, g.que["imgs"].shape[2], g.que["imgs"].shape[3], m0.shape[1], m0.shape[2], int(use_vis)
    rng = g.que["depth_range"][0].contiguous().float()
    p.depth_range, p.var_bias = rng.data_ptr(), 0.05
    p.hit, p.d_hit, p.d_w_point, p.d_map = hit.data_ptr(), gh.data_ptr(), d_w.data_ptr(), d_map.data_ptr()
    harness.nr_self_cpu.restype = C.c_int
    harness.nr_self_cpu.argtypes = [C.c_void_p]
    assert harness.nr_self_cpu(C.addressof(p)) == 0
    assert torch.allclose(hit, t("self_hit")[0], atol=2e-6), (hit - t("self_hit")[0]).abs().max()
    grads = backward.unpack_point_grads(plan, d_w)
    checked = 0
    for k in z.files:
        if not k.startswith("selfgrad_"):
            continue
        ga = t(k)
        err, scale = float((grads[k[9:]] - ga).abs().max()), float(ga.abs().max())
        assert err <= 3e-4 * max(scale, 1e-3) + 3e-6, (k, err, scale)
        checked += 1
    assert checked >= 18
    gm = t("self_grad_map")[0]
    assert float((d_map - gm).abs().max()) <= 3e-4 * float(gm.abs().max()) + 3e-6
