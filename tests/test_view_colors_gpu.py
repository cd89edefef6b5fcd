"""GPU: what colour each working view puts into a pixel (cfg render_view_colors; nr_view_colors behind
nr_render_pass_fwd_blend, _agg or _view) against the fp64 oracle (view_colors_nr[r, v] = Σ_d hit_nr[r, d] · w[v, r, d] ·
rgb_v[r, d], w the blend weights render_by_depth_with_blend records and rgb_v the prj_rgb of neuray_oracle.render_by_depth),
and its contract with the rest of the render path: Σ_v view_colors equals the pass' pixel_colors_nr to fp32 rounding, a
view that sees none of a ray's samples gives 0, every other output bit-identical with the option on and off through each
launch path, NR gradients unchanged, chunked = whole, empty renders, the TF32 mode, the generalising frame renderer and a
host that only knows the header.  Tolerance: 1e-4 abs / 1e-3 rel."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

import neuray_oracle as orc
from gen_golden import flat_cfg
from neuray_b200 import _lib, renderer, synthetic
from test_agg_weights_cpu import f64
from test_blend_weights_cpu import render_by_depth_with_blend
from test_dr_gpu import pick_rays
from test_pack_gpu import nr_posenc, weight_struct
from test_tf32_gpu import _lin_tf32
from test_view_colors_cpu import oracle_view_colors

pytestmark = pytest.mark.gpu
ATOL, RTOL = 1e-4, 1e-3
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COLORS = {"render_view_colors": True}
SPREAD = dict(sigma_gain=1.0, sigma_bias=0.02)
KEYS = {"view_colors_nr", "view_colors_nr_fine"}


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
        out = render_by_depth_with_blend(f64(W), oc, depth.double(), f64(que), f64(ref), False, is_fine, keep)
    return keep, out


def oracle_passes(W, oc, que, ref):
    """The fp64 coarse pass on render_impl's depths and the fine pass on the oracle's own resampling: (gold view colours of
    the coarse pass [1,rn,rfn,3], of the fine pass, the coarse keep, the fine depths)."""
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
    depth, _ = orc.sample_depth(que["depth_range"], que["coords"], oc["depth_sample_num"])
    keep_c, gold_c = oracle_pass(W, oc, que, ref, depth, False)
    fd = orc.sample_fine_depth(depth.double(), gold_c["hit_prob_nr"], que["depth_range"].double(), oc["fine_depth_sample_num"], False)
    fd = torch.sort(fd, -1)[0].float()
    keep_f, gold_f = oracle_pass(W, oc, que, ref, fd, True)
    return oracle_view_colors(keep_c, gold_c["hit_prob_nr"]), oracle_view_colors(keep_f, gold_f["hit_prob_nr"]), keep_c, fd


def make_net(cfg, W):
    net = renderer.NeuralRayRenderPath(cfg)
    net.load_state_dict(W, strict=True)
    return net.cuda()


def native(net, que, ref, fd, mode):
    renderer.set_precision(mode)
    dq, dr = synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda")
    with torch.no_grad():
        out = net.render_impl(dq, dr, False)
        out_f = net.render_by_depth(fd.cuda(), dq, dr, False, True)
    torch.cuda.synchronize()
    return out, out_f


def check_sum(colors, pixel, dn, what):
    """Σ_v view_colors = pixel_colors_nr of the same pass.  Both sum the same dn · rfn products hit · w · rgb, whose
    absolute values add up to at most 1 (Σ_d hit <= 1, Σ_v w = 1, rgb in [0, 1]), in different orders: the point kernel adds
    the views, then the ray kernel the samples; nr_view_colors adds the samples, then the views.  So they differ by at most
    (dn + rfn + 8) fp32 roundings of 1, the 8 covering the products and the lanes' butterfly."""
    rfn = colors.shape[2]
    err = float((colors.sum(2).double() - pixel.double()).abs().max()) if colors.numel() else 0.0
    bound = (dn + rfn + 8) * 2.0 ** -24
    print(f"{what}: max |Σ_v view_colors - pixel_colors_nr| {err:.2e} (bound {bound:.2e})")
    assert err <= bound, (what, err, bound)


def check(que, ref, cfg, W):
    """Coarse pass end to end and the fine pass on the oracle's fine depths, against the fp64 oracle; both passes' Σ_v."""
    assert float(ref["imgs"].min()) >= 0 and float(ref["imgs"].max()) <= 1
    oc = flat_cfg({**renderer.base_cfg, **cfg})
    gold_c, gold_f, keep_c, fd = oracle_passes(W, oc, que, ref)
    out, out_f = native(make_net(cfg, W), que, ref, fd, "fp32")
    rfn = ref["imgs"].shape[0]
    assert out["view_colors_nr"].shape == (1, que["coords"].shape[1], rfn, 3)
    close(out["view_colors_nr"], gold_c, "view_colors_nr")
    close(out_f["view_colors_nr"], gold_f, "view_colors_nr, fine pass on the oracle's depths")
    check_sum(out["view_colors_nr"], out["pixel_colors_nr"], oc["depth_sample_num"], "coarse")
    check_sum(out_f["view_colors_nr"], out_f["pixel_colors_nr"], oc["fine_depth_sample_num"], "fine")
    return out, out_f, keep_c


def small_cfg(dn, use_vis, **over):
    return {"use_hierarchical_sampling": True, "depth_sample_num": dn, "fine_depth_sample_num": dn, "agg_net_cfg": {"sample_num": dn},
            "fine_agg_net_cfg": {"sample_num": dn}, "dist_decoder_cfg": {"use_vis": use_vis},
            "fine_dist_decoder_cfg": {"use_vis": use_vis}, **COLORS, **over}


# one rfn per lane-group instantiation of the point kernel (G 4, 5, 6, 8, 10, 16, 32)
@pytest.mark.parametrize("use_vis", [False, True])
@pytest.mark.parametrize("rfn", [3, 5, 6, 8, 9, 13, 20])
def test_matches_the_fp64_oracle_at_every_lane_group(rfn, use_vis):
    cfg = small_cfg(32, use_vis)
    que, ref = synthetic.make_scene(h=40, w=48, rfn=rfn, seed=rfn, smooth=2, arc_deg=90.0, with_que_imgs=False)
    check(pick_rays(que, 48, 40, n=40), ref, cfg, synthetic.make_weights(cfg, seed=rfn, **SPREAD))


@pytest.mark.parametrize("dn", [16, 32, 48, 64, 200])
def test_matches_the_fp64_oracle_at_every_sample_count(dn):
    """dn 16: half the lanes of a ray idle; 48: the second pass over the lanes partly idle; 200: seven samples per lane."""
    cfg = small_cfg(dn, True)
    que, ref = synthetic.make_scene(h=40, w=48, rfn=5, seed=3, smooth=2, with_que_imgs=False)
    check(pick_rays(que, 48, 40, n=24), ref, cfg, synthetic.make_weights(cfg, seed=4, **SPREAD))


def test_benched_black_800_on_a_ray_slice():
    sys.path.insert(0, ROOT)
    import bench
    wl = bench.WORKLOADS["black_800"]
    cfg = dict(bench.model_cfg(*wl["dn"]), **COLORS)
    que, ref = synthetic.make_scene(**dict(wl["scene"], rfn=wl["rfn"], seed=0, smooth=2, with_que_imgs=False))
    check(pick_rays(que, 800, 800), ref, cfg, synthetic.make_weights(cfg, seed=0))


@pytest.mark.parametrize("use_vis", [False, True])
def test_tf32_mode_against_the_tf32_restatement(use_vis, monkeypatch):
    """The TF32 pass' output against the fp64 oracle: its max and 99th-percentile abs errors stay within 2x those of the
    oracle's TF32 restatement (every Linear's input and weight rounded to tf32, test_tf32_gpu.py) -- the criterion of the
    TF32 mode.  Σ_v view_colors equals the TF32 pass' own pixel_colors_nr to fp32 rounding."""
    cfg = small_cfg(32, use_vis)
    que, ref = synthetic.make_scene(h=40, w=48, rfn=8, seed=9, smooth=2, with_que_imgs=False)
    que, W = pick_rays(que, 48, 40, n=40), synthetic.make_weights(cfg, seed=9, **SPREAD)
    oc = flat_cfg({**renderer.base_cfg, **cfg})
    gold_c, gold_f, _, fd = oracle_passes(W, oc, que, ref)
    with monkeypatch.context() as m:
        m.setattr(orc, "_lin", _lin_tf32)
        emu_c, _, _, _ = oracle_passes(W, oc, que, ref)
        keep, out = oracle_pass(W, oc, que, ref, fd, True)
        emu_f = oracle_view_colors(keep, out["hit_prob_nr"])
    net = make_net(cfg, W)
    f32 = native(net, que, ref, fd, "fp32")
    t32 = native(net, que, ref, fd, "tf32")
    assert not torch.equal(t32[0]["view_colors_nr"], f32[0]["view_colors_nr"])      # the TF32 kernels ran
    for tag, gold, emu, out in (("coarse", gold_c, emu_c, t32[0]), ("fine", gold_f, emu_f, t32[1])):
        err = (out["view_colors_nr"].cpu().double() - gold).abs().flatten()
        ref_err = (emu - gold).abs().flatten()
        mx, q99 = float(err.max()), float(torch.quantile(err, 0.99))
        emx, eq99 = float(ref_err.max()), float(torch.quantile(ref_err, 0.99))
        print(f"{tag} view_colors_nr (tf32): max abs err {mx:.3e} restatement {emx:.3e} (ratio {mx / max(emx, 1e-30):.2f}); "
              f"q99 {q99:.3e} restatement {eq99:.3e} (ratio {q99 / max(eq99, 1e-30):.2f})")
        assert mx <= 2 * emx and q99 <= 2 * eq99, (tag, mx, emx, q99, eq99)
        check_sum(out["view_colors_nr"], out["pixel_colors_nr"], 32, f"{tag} (tf32)")


def test_unseen_views_give_zero():
    """Far samples of the top rows leave every view, and rays aimed far off the image leave every view with all their
    samples.  A view that sees none of a ray's samples gives exactly 0, also where its blend weight is 1/rfn."""
    cfg = small_cfg(32, False)
    rfn = 5
    que, ref = synthetic.make_scene(h=40, w=48, rfn=rfn, seed=45, smooth=2, depth_range=(1.0, 14.0), arc_deg=120.0, with_que_imgs=False)
    que = synthetic.slice_rays(que, 0, 96)
    off = torch.tensor([[-4000.0, -4000.0], [5000.0, -4000.0], [-4000.0, 5000.0], [5000.0, 5000.0]])
    que = dict(que, coords=torch.cat([que["coords"], off[None]], 1).contiguous())
    W = synthetic.make_weights(cfg, seed=55, **SPREAD)
    out, _, keep = check(que, ref, cfg, W)
    mask = keep["prj_mask"][:, 0, :, :, 0]                                           # [rfn,rn,dn]
    blind = (mask.sum(-1) == 0).t()                                                  # [rn,rfn]: the view sees no sample
    assert int(blind.all(-1).sum()) >= 4 and int(blind.sum()) > int(blind.all(-1).sum()) * rfn
    assert bool((out["view_colors_nr"][0].cpu()[blind] == 0).all())
    assert float(out["view_colors_nr"].abs().max()) > 0


SMALL = {"use_hierarchical_sampling": True, "depth_sample_num": 16, "fine_depth_sample_num": 16, "agg_net_cfg": {"sample_num": 16},
         "fine_agg_net_cfg": {"sample_num": 16}, "render_depth": True}
# the three launch paths nr_view_colors runs behind: _blend (without its reduction when alone, or with it), _agg, _view
OTHERS = {"alone": {}, "blend": {"render_blend_weights": True}, "agg": {"render_agg_weights": True},
          "view": {"render_view_depth": True}}


def small_setup(cfg, rays=(300, 428)):
    que, ref = synthetic.make_scene(40, 48, 4, seed=3, smooth=2)
    que = synthetic.slice_rays(que, *rays)
    W = synthetic.make_weights(cfg, seed=3, **SPREAD)
    return que, ref, [make_net(dict(cfg, render_view_colors=on), W) for on in (False, True)]


@pytest.mark.parametrize("others", list(OTHERS.values()), ids=list(OTHERS))
@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_existing_outputs_identical_with_the_option_on_and_off_in_eval(mode, others):
    """With direct rendering and visibility on, and the blend, agg or view outputs on or off: every other output is the same
    with the option on and off, and the option adds only its two outputs."""
    que, ref, (off, on) = small_setup(dict(SMALL, use_dr_prediction=True, render_visibility=True, **others))
    renderer.set_precision(mode)
    outs = []
    for net in (off, on):
        with torch.no_grad():
            outs.append(net.render(synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda"), False))
    torch.cuda.synchronize()
    a, b = outs
    assert set(b) - set(a) == KEYS
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert b["view_colors_nr_fine"].shape == (1, 128, 4, 3) and b["view_colors_nr"].shape == (1, 128, 4, 3)


@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_every_launch_path_gives_the_same_colours(mode):
    """The blend row is plane 0 of each export's workspace and the same for every export set, so the colours are the same
    bit for bit whichever launch nr_view_colors runs behind."""
    que, ref = synthetic.make_scene(40, 48, 4, seed=3, smooth=2)
    que = synthetic.slice_rays(que, 300, 428)
    W = synthetic.make_weights(SMALL, seed=3, **SPREAD)
    renderer.set_precision(mode)
    res = {}
    for tag, others in OTHERS.items():
        with torch.no_grad():
            res[tag] = make_net(dict(SMALL, **COLORS, **others), W).render(synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda"), False)
    torch.cuda.synchronize()
    for tag in OTHERS:
        for k in KEYS:
            assert torch.equal(res[tag][k], res["alone"][k]), (tag, k)


def test_launch_count():
    """Off: the launches of the render as before.  On: one more kernel per pass."""
    que, ref, (off, on) = small_setup(dict(SMALL))
    counts = []
    for net in (off, on):
        before = _lib.LAUNCHES
        with torch.no_grad():
            net.render(synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda"), False)
        counts.append(_lib.LAUNCHES - before)
    torch.cuda.synchronize()
    assert counts[1] == counts[0] + 2, counts


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
    assert set(b) - set(a) == KEYS
    assert not any(b[k].requires_grad for k in KEYS)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    # the weight-gradient GEMMs and the map gradients accumulate with atomics: two runs differ in the last bits whatever
    # the cfg, so the gradients are equal up to that reordering
    assert set(ga) == set(gb) and len(ga) > 100
    for k in ga:
        torch.testing.assert_close(ga[k], gb[k], atol=1e-5 * float(ga[k].abs().max()) + 1e-8, rtol=0, msg=k)


def test_chunked_equals_whole_and_empty_renders():
    cfg = dict(SMALL, ray_batch_num=128)
    que, ref, (_, net) = small_setup(cfg, rays=(300, 700))
    dq, dr = synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda")
    whole = make_net(dict(cfg, **COLORS, ray_batch_num=4096), {k: v.cpu() for k, v in net.state_dict().items()})
    with torch.no_grad():
        a, b = net.render(dq, dr, False), whole.render(dq, dr, False)
        empty = net.render(dict(dq, coords=dq["coords"][:, :0]), dr, False)
        empty_t = net.render(dict(dq, coords=dq["coords"][:, :0]), dr, True)
    torch.cuda.synchronize()
    for k in KEYS:
        assert torch.equal(a[k], b[k]), k
        assert not a[k].requires_grad, k
        assert empty[k].shape == (1, 0, 4, 3) and empty_t[k].shape == (1, 0, 4, 3), k
    assert a["view_colors_nr"].shape == (1, 400, 4, 3)


def test_a_reference_style_cfg_without_the_key_renders_as_before():
    """patch.install() runs these functions on the reference's own renderer, whose cfg has the key only if the user set it."""
    que, ref, (off, on) = small_setup(dict(SMALL))
    del off.cfg["render_view_colors"]
    with torch.no_grad():
        a = off.render(synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda"), False)
        b = on.render(synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda"), False)
    assert not KEYS & set(a) and KEYS <= set(b)


FRAME_CFG = {"use_hierarchical_sampling": True, "dist_decoder_cfg": {"use_vis": False}, "depth_sample_num": 32, "fine_depth_sample_num": 32,
             "agg_net_cfg": {"sample_num": 32}, "fine_agg_net_cfg": {"sample_num": 32}, "ray_batch_num": 160}


def test_gen_frame_renderer_with_the_option_matches_the_oracle():
    """NeuralRayGenFrameRenderer.forward in eval: init net -> encoders -> render.  Every other output bit-identical with the
    option off; both passes against the oracle's stages (encoder outputs carry ~1e-5 differences into the passes, hence
    the quantile bounds of test_dr_gpu.py for this path)."""
    from test_encoders_gpu import _smooth_depth, depth_init_golden, golden
    cfg = dict(FRAME_CFG)
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
    outs = []
    for on in (False, True):
        net = renderer.NeuralRayGenFrameRenderer(dict(cfg, render_view_colors=on))
        net.load_state_dict(full, strict=True)
        net.cuda().eval()
        torch.manual_seed(0)           # predict_mean_for_depth_loss draws its pixels at random
        with torch.no_grad():
            outs.append(net({"que_imgs_info": synthetic.to_device(que, "cuda"), "ref_imgs_info": synthetic.to_device(ref, "cuda"), "eval": True}))
    torch.cuda.synchronize()
    a, out = outs
    assert set(out) - set(a) == KEYS
    for k in a:
        assert torch.equal(a[k], out[k]), k
    img_feats = orc.res_unet_light(img_w, "", ref["imgs"])
    ray_feats = orc.vis_encoder(vis_w, "", orc.depth_init_net(init_w, "", ref), img_feats)
    oc = flat_cfg({**renderer.base_cfg, **cfg})
    gold_c, gold_f, _, _ = oracle_passes(W, oc, que, dict(ref, ray_feats=ray_feats, img_feats=img_feats))
    err = (out["view_colors_nr"].cpu().double() - gold_c).abs()
    print(f"view_colors_nr: max {err.max().item():.2e}, q99 {torch.quantile(err.flatten(), 0.99).item():.2e}")
    assert float(torch.quantile(err.flatten(), 0.99)) < 3e-4 and float(err.max()) < 3e-3
    # the fine pass resamples from the native coarse hit_prob, whose inverse-CDF knots are ill-conditioned
    fine = (out["view_colors_nr_fine"].cpu().double() - gold_f).abs()
    print(f"view_colors_nr_fine: max {fine.max().item():.2e}, q99 {torch.quantile(fine.flatten(), 0.99).item():.2e}")
    assert float(torch.quantile(fine.flatten(), 0.99)) < 1e-3 and float((fine > 1e-3).float().mean()) < 0.01
    check_sum(out["view_colors_nr"], out["pixel_colors_nr"], 32, "frame, coarse")
    check_sum(out["view_colors_nr_fine"], out["pixel_colors_nr_fine"], 32, "frame, fine")


class HeaderBlendParams(C.Structure):       # field for field as NrBlendParams in include/neuray_b200.h
    _fields_ = [("row_blend", C.c_void_p), ("blend_weights", C.c_void_p)]


class HeaderColorParams(C.Structure):       # field for field as NrColorParams in include/neuray_b200.h
    _fields_ = [("row_blend", C.c_void_p), ("hit_prob", C.c_void_p), ("view_colors", C.c_void_p)]


def test_header_only_host_drives_nr_view_colors():
    """A coarse pass (+ fused resampling) and a fine pass through ctypes calls only, each by nr_render_pass_fwd_blend with
    blend_weights NULL followed by nr_view_colors on a handle without the package's argtypes, equal the Python path bit
    for bit: the per-view colours and every pass output."""
    cfg = {"use_hierarchical_sampling": True, "dist_decoder_cfg": {"use_vis": False}, "depth_sample_num": 32, "fine_depth_sample_num": 32,
           "agg_net_cfg": {"sample_num": 32}, "fine_agg_net_cfg": {"sample_num": 32}, "render_depth": True, **COLORS}
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
        outs = {}
        for tag, qd, sample_num in (("c", depth, dn), ("f", fine_depth, fdn)):
            pe = nr_posenc(sample_num).to(dev)
            rec = f32(rn * sample_num * _lib.NR_POINT_REC)
            o = {"pixel_colors": f32(rn, 3), "hit_prob": f32(rn, sample_num), "render_depth": f32(rn),
                 "ray_mask": torch.empty(rn, dtype=torch.uint8, device=dev), "view_colors": f32(rn, rfn, 3)}
            p = _lib.NrPassParams()
            p.coords, p.que_depth, p.que_cam, p.rn, p.dn = q["coords"].data_ptr(), qd.data_ptr(), cam.data_ptr(), rn, sample_num
            p.feat, p.rgb, p.view_params = feat.data_ptr(), rgb.data_ptr(), vp.data_ptr()
            p.rfn, p.h, p.w, p.fh, p.fw = rfn, h, w, fh, fw
            p.w_point, p.w_ray, p.w_tc = (b.data_ptr() for b in packed[tag])
            p.pos_enc = pe.data_ptr()
            p.use_vis, p.var_bias = 0, 0.05
            p.ray_mask_view_num, p.ray_mask_point_num = 2, 8
            p.point_rec = rec.data_ptr()
            p.pixel_colors, p.render_depth, p.ray_mask = o["pixel_colors"].data_ptr(), o["render_depth"].data_ptr(), o["ray_mask"].data_ptr()
            if tag == "c":
                p.fine_dn, p.fine_use_all, p.fine_u, p.fine_u_stride, p.fine_depth = fdn, 0, u.data_ptr(), 0, fine_depth.data_ptr()
            p.hit_prob = o["hit_prob"].data_ptr()
            row = f32(rfn, rn * sample_num)
            assert raw.nr_render_pass_fwd_blend(C.byref(p), C.byref(HeaderBlendParams(row.data_ptr(), None)), C.c_void_p(stream)) == 0
            hc = HeaderColorParams(row.data_ptr(), o["hit_prob"].data_ptr(), o["view_colors"].data_ptr())
            assert raw.nr_view_colors(C.byref(p), C.byref(hc), C.c_void_p(stream)) == 0
            outs[tag] = o
        torch.cuda.synchronize()
    with torch.no_grad():
        want = make_net(cfg, W).render_impl(synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda"), False)
    torch.cuda.synchronize()
    for tag, sfx in (("c", ""), ("f", "_fine")):
        assert torch.equal(outs[tag]["view_colors"][None], want["view_colors_nr" + sfx]), tag
        assert torch.equal(outs[tag]["pixel_colors"][None], want["pixel_colors_nr" + sfx])
        assert torch.equal(outs[tag]["hit_prob"][None], want["hit_prob_nr" + sfx])
        assert torch.equal(outs[tag]["render_depth"][None], want["render_depth" + sfx])
