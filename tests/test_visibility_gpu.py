"""GPU: the per-view visibility output (cfg render_visibility; nr_view_visibility) against the fp64 oracle
(visibility_nr[r, v] = Σ_d hit_nr[r, d] · prj_vis[v, r, d] of neuray_oracle.render_by_depth), and its contract with the
rest of the render path: exact zeros for a view that sees none of a ray's samples, every pre-existing output bit-identical
with the option on and off, NR gradients unchanged, chunked = whole, empty renders, the TF32 mode, the frame renderers,
a reference-style cfg and a host that only knows the header.  Tolerance: 1e-4 abs / 1e-3 rel."""
import ctypes as C
import os
import sys

import pytest
import torch

import neuray_oracle as orc
from gen_golden import flat_cfg
from neuray_b200 import _lib, renderer, synthetic
from test_dr_gpu import pick_rays
from test_pack_gpu import nr_posenc, weight_struct
from test_visibility_cpu import f64, oracle_visibility

pytestmark = pytest.mark.gpu
ATOL, RTOL = 1e-4, 1e-3
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VIS = {"render_visibility": True}
SPREAD = dict(sigma_gain=1.0, sigma_bias=0.02)


@pytest.fixture(autouse=True)
def _fp32_after():
    yield
    renderer.set_precision("fp32")


def close(a, b, what):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    assert a.shape == b.shape, (what, a.shape, b.shape)
    err = (a - b).abs()
    bad = (err > ATOL + RTOL * b.abs()) | torch.isnan(a)
    print(f"{what}: max abs err {err.max().item():.3e}, {int(bad.sum())}/{err.numel()} outside tol")
    assert int(bad.sum()) == 0, f"{what}: {int(bad.sum())} values outside tolerance"


def oracle_pass(W, oc, que, ref, depth, is_fine):
    keep = {}
    with torch.no_grad():
        out = orc.render_by_depth(f64(W), oc, depth.double(), f64(que), f64(ref), False, is_fine, keep)
    return keep, out


def make_net(cfg, W):
    net = renderer.NeuralRayRenderPath(cfg)
    net.load_state_dict(W, strict=True)
    return net.cuda()


def check(que, ref, cfg, W, mode="fp32"):
    """Coarse pass end to end and the fine pass on the oracle's fine depths, against the fp64 oracle.  In TF32 mode the
    oracle's prj_vis is weighted by the TF32 pass' own hit_prob."""
    oc = flat_cfg({**renderer.base_cfg, **cfg})
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
    depth, _ = orc.sample_depth(que["depth_range"], que["coords"], oc["depth_sample_num"])
    keep_c, gold_c = oracle_pass(W, oc, que, ref, depth, False)
    fd = orc.sample_fine_depth(depth.double(), gold_c["hit_prob_nr"], que["depth_range"].double(), oc["fine_depth_sample_num"], False)
    fd = torch.sort(fd, -1)[0].float()
    keep_f, gold_f = oracle_pass(W, oc, que, ref, fd, True)
    net = make_net(cfg, W)
    renderer.set_precision(mode)
    dq, dr = synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda")
    with torch.no_grad():
        out = net.render_impl(dq, dr, False)
        out_f = net.render_by_depth(fd.cuda(), dq, dr, False, True)
    torch.cuda.synchronize()
    rfn = ref["imgs"].shape[0]
    assert out["visibility_nr"].shape == (1, que["coords"].shape[1], rfn)
    hits = (gold_c["hit_prob_nr"], gold_f["hit_prob_nr"]) if mode == "fp32" else \
        (out["hit_prob_nr"].cpu().double(), out_f["hit_prob_nr"].cpu().double())
    close(out["visibility_nr"], oracle_visibility(keep_c, hits[0]), f"visibility_nr ({mode})")
    close(out_f["visibility_nr"], oracle_visibility(keep_f, hits[1]), f"visibility_nr, fine pass on the oracle's depths ({mode})")
    return out, out_f, keep_c


def small_cfg(dn, use_vis, **over):
    return {"use_hierarchical_sampling": True, "depth_sample_num": dn, "fine_depth_sample_num": dn, "agg_net_cfg": {"sample_num": dn},
            "fine_agg_net_cfg": {"sample_num": dn}, "dist_decoder_cfg": {"use_vis": use_vis},
            "fine_dist_decoder_cfg": {"use_vis": use_vis}, **VIS, **over}


@pytest.mark.parametrize("use_vis", [False, True])
@pytest.mark.parametrize("rfn", [3, 5, 6, 8, 9, 13, 20])
def test_matches_the_fp64_oracle_at_every_lane_group(rfn, use_vis):
    cfg = small_cfg(32, use_vis)
    que, ref = synthetic.make_scene(h=40, w=48, rfn=rfn, seed=rfn, smooth=2, arc_deg=90.0, with_que_imgs=False)
    check(pick_rays(que, 48, 40, n=40), ref, cfg, synthetic.make_weights(cfg, seed=rfn, **SPREAD))


@pytest.mark.parametrize("dn", [16, 48, 200])
def test_matches_the_fp64_oracle_at_every_ray_split(dn):
    """dn 16: eight rays per CTA; 48: 64 lanes, some idle; 200: two samples per lane."""
    cfg = small_cfg(dn, True)
    que, ref = synthetic.make_scene(h=40, w=48, rfn=5, seed=3, smooth=2, with_que_imgs=False)
    check(pick_rays(que, 48, 40, n=24), ref, cfg, synthetic.make_weights(cfg, seed=4, **SPREAD))


def test_benched_black_800_on_a_ray_slice():
    sys.path.insert(0, ROOT)
    import bench
    wl = bench.WORKLOADS["black_800"]
    cfg = dict(bench.model_cfg(*wl["dn"]), **VIS)
    que, ref = synthetic.make_scene(**dict(wl["scene"], rfn=wl["rfn"], seed=0, smooth=2, with_que_imgs=False))
    check(pick_rays(que, 800, 800), ref, cfg, synthetic.make_weights(cfg, seed=0))


@pytest.mark.parametrize("use_vis", [False, True])
def test_tf32_mode_uses_the_tf32_pass_hit_prob(use_vis):
    cfg = small_cfg(32, use_vis)
    que, ref = synthetic.make_scene(h=40, w=48, rfn=8, seed=9, smooth=2, with_que_imgs=False)
    que, W = pick_rays(que, 48, 40, n=40), synthetic.make_weights(cfg, seed=9, **SPREAD)
    out, _, _ = check(que, ref, cfg, W, mode="tf32")
    renderer.set_precision("fp32")
    with torch.no_grad():
        fp32 = make_net(cfg, W).render_impl(synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda"), False)
    assert not torch.equal(out["hit_prob_nr"], fp32["hit_prob_nr"])          # the TF32 kernels ran


def test_unseen_views_give_exact_zeros_and_visibility_is_bounded():
    cfg = small_cfg(32, False)
    que, ref = synthetic.make_scene(h=40, w=52, rfn=8, seed=43, smooth=2, depth_range=(2.5, 5.5), arc_deg=80.0, with_que_imgs=False)
    que = synthetic.slice_rays(que, 0, 156)               # the top rows: many points fall outside some views
    out, out_f, keep = check(que, ref, cfg, synthetic.make_weights(cfg, seed=43, **SPREAD))
    unseen = (keep["prj_mask"][..., 0].sum(-1) == 0).permute(1, 2, 0).cuda()       # [1,rn,rfn]
    assert int(unseen.sum()) > 0
    vis = out["visibility_nr"]
    assert torch.equal(vis[unseen], torch.zeros_like(vis[unseen]))
    for o in (out, out_f):
        assert bool((o["visibility_nr"] >= 0).all())
        assert bool((o["visibility_nr"] <= o["hit_prob_nr"].sum(-1, keepdim=True) + 1e-6).all())


SMALL = {"use_hierarchical_sampling": True, "depth_sample_num": 16, "fine_depth_sample_num": 16, "agg_net_cfg": {"sample_num": 16},
         "fine_agg_net_cfg": {"sample_num": 16}, "render_depth": True}


def small_setup(cfg, rays=(300, 428)):
    que, ref = synthetic.make_scene(40, 48, 4, seed=3, smooth=2)
    que = synthetic.slice_rays(que, *rays)
    W = synthetic.make_weights(cfg, seed=3, **SPREAD)
    return que, ref, [make_net(dict(cfg, render_visibility=on), W) for on in (False, True)]


@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_existing_outputs_identical_with_the_option_on_and_off_in_eval(mode):
    que, ref, (off, on) = small_setup(dict(SMALL, use_dr_prediction=True))
    renderer.set_precision(mode)
    outs = []
    for net in (off, on):
        with torch.no_grad():
            outs.append(net.render(synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda"), False))
    torch.cuda.synchronize()
    a, b = outs
    assert set(b) - set(a) == {"visibility_nr", "visibility_nr_fine"}
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert b["visibility_nr_fine"].shape == (1, 128, 4)


def test_nr_outputs_and_gradients_unchanged_in_training():
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
    assert set(b) - set(a) == {"visibility_nr", "visibility_nr_fine"}
    assert not b["visibility_nr"].requires_grad and not b["visibility_nr_fine"].requires_grad
    for k in a:
        assert torch.equal(a[k], b[k]), k
    # the weight-gradient GEMMs and the map gradients accumulate with atomics: two runs differ in the last bits whatever
    # the cfg, so the gradients are equal up to that reordering
    assert set(ga) == set(gb) and len(ga) > 100
    for k in ga:
        torch.testing.assert_close(ga[k], gb[k], atol=1e-5 * float(ga[k].abs().max()) + 1e-8, rtol=0, msg=k)


def test_chunked_equals_whole_and_empty_renders():
    cfg = dict(SMALL, ray_batch_num=96)
    que, ref, (_, net) = small_setup(cfg, rays=(300, 700))
    dq, dr = synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda")
    whole = make_net(dict(cfg, **VIS, ray_batch_num=4096), {k: v.cpu() for k, v in net.state_dict().items()})
    with torch.no_grad():
        a, b = net.render(dq, dr, False), whole.render(dq, dr, False)
        empty = net.render(dict(dq, coords=dq["coords"][:, :0]), dr, False)
        empty_t = net.render(dict(dq, coords=dq["coords"][:, :0]), dr, True)
    torch.cuda.synchronize()
    for k in ("visibility_nr", "visibility_nr_fine"):
        assert torch.equal(a[k], b[k]), k
        assert empty[k].shape == (1, 0, 4) and empty_t[k].shape == (1, 0, 4), k
    assert a["visibility_nr"].shape == (1, 400, 4)


def test_a_reference_style_cfg_without_the_key_renders_as_before():
    """patch.install() runs these functions on the reference's own renderer, whose cfg has the key only if the user set it."""
    que, ref, (off, on) = small_setup(dict(SMALL))
    del off.cfg["render_visibility"]
    with torch.no_grad():
        a = off.render(synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda"), False)
        b = on.render(synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda"), False)
    assert "visibility_nr" not in a and "visibility_nr" in b


def test_gen_frame_renderer_carries_the_output():
    from test_encoders_gpu import _smooth_depth, depth_init_golden, golden
    import numpy as np
    cfg = {"use_hierarchical_sampling": True, "dist_decoder_cfg": {"use_vis": False}, "depth_sample_num": 32, "fine_depth_sample_num": 32,
           "agg_net_cfg": {"sample_num": 32}, "fine_agg_net_cfg": {"sample_num": 32}, "ray_batch_num": 160}
    _, img_w, vis_w = golden()
    _, _, init_w = depth_init_golden()
    que, ref = synthetic.make_scene(64, 80, 4, seed=6, smooth=2)
    que = synthetic.slice_rays(que, 1500, 1900)
    ref = {k: ref[k] for k in ("imgs", "poses", "Ks", "depth_range")}
    ref["depth"] = _smooth_depth(np.random.RandomState(6), 4, 64, 80, 2.5, 5.0)
    full = dict(synthetic.make_weights(cfg, seed=6))
    full.update({"image_encoder." + k: v for k, v in img_w.items()})
    full.update({"vis_encoder." + k: v for k, v in vis_w.items()})
    full.update({"init_net." + k: v for k, v in init_w.items()})
    outs = []
    for on in (False, True):
        net = renderer.NeuralRayGenFrameRenderer(dict(cfg, render_visibility=on))
        net.load_state_dict(full, strict=True)
        net.cuda().eval()
        torch.manual_seed(0)           # predict_mean_for_depth_loss draws its pixels at random
        with torch.no_grad():
            outs.append(net({"que_imgs_info": synthetic.to_device(que, "cuda"), "ref_imgs_info": synthetic.to_device(ref, "cuda"), "eval": True}))
    torch.cuda.synchronize()
    a, b = outs
    assert set(b) - set(a) == {"visibility_nr", "visibility_nr_fine"}
    for k in a:
        assert torch.equal(a[k], b[k]), k
    for k in ("visibility_nr", "visibility_nr_fine"):
        assert b[k].shape == (1, 400, 4) and bool((b[k] >= 0).all()) and float(b[k].max()) > 0, k


class HeaderVisParams(C.Structure):      # field for field as NrVisParams in include/neuray_b200.h
    _fields_ = [("hit_prob", C.c_void_p), ("visibility", C.c_void_p)]


def test_header_only_host_drives_nr_view_visibility():
    """A coarse pass (+ fused resampling) and a fine pass through ctypes calls only, each followed by nr_view_visibility
    on a handle without the package's argtypes, equal the Python path bit for bit."""
    cfg = {"use_hierarchical_sampling": True, "dist_decoder_cfg": {"use_vis": False}, "depth_sample_num": 32, "fine_depth_sample_num": 32,
           "agg_net_cfg": {"sample_num": 32}, "fine_agg_net_cfg": {"sample_num": 32}, **VIS}
    que, ref = synthetic.make_scene(48, 64, 5, seed=12, smooth=2, with_que_imgs=False)
    que = synthetic.slice_rays(que, 900, 1100)
    W = synthetic.make_weights(cfg, seed=2)
    dev = torch.device("cuda", 0)
    lib, ck = _lib.lib(), _lib.check
    raw = C.CDLL(_lib.LIB_PATH)
    f32 = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream().cuda_stream
        P = {k: v.to(dev).contiguous() for k, v in W.items()}
        q = {k: v.to(dev).contiguous() for k, v in que.items()}
        r = {k: v.to(dev).contiguous() for k, v in ref.items()}
        L, T = _lib.weight_layout(), _lib.tc_layout()
        rfn, _, h, w = r["imgs"].shape
        fh, fw = r["ray_feats"].shape[-2:]
        rn, dn, fdn = q["coords"].shape[1], cfg["depth_sample_num"], cfg["fine_depth_sample_num"]
        feat, rgb = f32(rfn, fh, fw, 64), f32(rfn, h, w, 4)
        ck(lib.nr_pack_feature_maps(r["ray_feats"].data_ptr(), r["img_feats"].data_ptr(), r["imgs"].data_ptr(), rfn, h, w, fh, fw,
                                    feat.data_ptr(), rgb.data_ptr(), stream), "pack maps")
        cam, vp = f32(24), f32(rfn, 20)
        ck(lib.nr_camera_blocks(q["poses"].data_ptr(), q["Ks"].data_ptr(), q["depth_range"].data_ptr(), r["poses"].data_ptr(),
                                r["Ks"].data_ptr(), r["depth_range"].data_ptr(), rfn, cam.data_ptr(), vp.data_ptr(), stream), "camera blocks")
        packed = {}
        for tag, dec, agg in (("c", "dist_decoder", "agg_net"), ("f", "fine_dist_decoder", "fine_agg_net")):
            bufs = (f32(L.total_point), f32(L.total_ray), f32(T.total))
            ck(lib.nr_pack_weights(C.byref(weight_struct(P, dec, agg)), bufs[0].data_ptr(), bufs[1].data_ptr(), bufs[2].data_ptr(), stream),
               "pack weights")
            packed[tag] = bufs
        depth = f32(rn, dn)
        ck(lib.nr_sample_depth(q["depth_range"].data_ptr(), rn, dn, None, depth.data_ptr(), None, stream), "sample_depth")
        u = (0.5 * (1 / fdn) + torch.arange(fdn) * (1 / fdn)).to(dev).contiguous()
        fine_depth = f32(rn, fdn)
        vis = {}
        for tag, qd, sample_num in (("c", depth, dn), ("f", fine_depth, fdn)):
            pe = nr_posenc(sample_num).to(dev)
            rec = f32(rn * sample_num * _lib.NR_POINT_REC)
            o = {"pixel_colors": f32(rn, 3), "hit_prob": f32(rn, sample_num), "render_depth": f32(rn),
                 "ray_mask": torch.empty(rn, dtype=torch.uint8, device=dev)}
            p = _lib.NrPassParams()
            p.coords, p.que_depth, p.que_cam, p.rn, p.dn = q["coords"].data_ptr(), qd.data_ptr(), cam.data_ptr(), rn, sample_num
            p.feat, p.rgb, p.view_params = feat.data_ptr(), rgb.data_ptr(), vp.data_ptr()
            p.rfn, p.h, p.w, p.fh, p.fw = rfn, h, w, fh, fw
            p.w_point, p.w_ray, p.w_tc = (b.data_ptr() for b in packed[tag])
            p.pos_enc = pe.data_ptr()
            p.use_vis, p.var_bias = 0, 0.05
            p.ray_mask_view_num, p.ray_mask_point_num = 2, 8
            p.point_rec = rec.data_ptr()
            p.pixel_colors, p.hit_prob = o["pixel_colors"].data_ptr(), o["hit_prob"].data_ptr()
            p.render_depth, p.ray_mask = o["render_depth"].data_ptr(), o["ray_mask"].data_ptr()
            if tag == "c":
                p.fine_dn, p.fine_use_all, p.fine_u, p.fine_u_stride, p.fine_depth = fdn, 0, u.data_ptr(), 0, fine_depth.data_ptr()
            ck(lib.nr_render_pass_fwd(C.byref(p), stream), "render pass")
            vis[tag] = f32(rn, rfn)
            hv = HeaderVisParams(o["hit_prob"].data_ptr(), vis[tag].data_ptr())
            assert raw.nr_view_visibility(C.byref(p), C.byref(hv), C.c_void_p(stream)) == 0
        torch.cuda.synchronize()
    with torch.no_grad():
        want = make_net(cfg, W).render_impl(synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda"), False)
    torch.cuda.synchronize()
    assert torch.equal(vis["c"][None], want["visibility_nr"])
    assert torch.equal(vis["f"][None], want["visibility_nr_fine"])
