"""GPU: the point kernel's TF32 render mode (renderer.set_precision("tf32"), nr_render_pass_fwd_tf32).

Accuracy.  The reference pins torch 1.7.1, which ran nn.Linear in TF32 on Ampere and later GPUs by default, so its own GPU
arithmetic is restated here: the oracle evaluated in fp64 with every Linear's input and weight rounded to nearest tf32
(tf32_rne, ties to even) and the products and sums in fp64 -- without the accumulation-order noise of a real GEMM.  The
TF32 mode's max and 99th-percentile abs errors against the plain fp64 oracle must each stay within 2x the restatement's,
for pixel_colors, hit_prob and render_depth of the coarse pass end to end and of the fine pass on the oracle's fine depths
(inverse-CDF knots make end-to-end fine outputs ill-conditioned).  ray_mask is geometry only, so it is bit-identical to
the fp32 mode; the other outputs are not, which shows the TF32 kernels ran.

Contract.  A pass that records a gradient runs in fp32 whatever the switch says; the switch can be flipped back and forth;
an optimizer step re-packs the TF32 weights; empty and chunked renders, direct rendering with NR colours, the profiling
launch path and a host that only knows the header all work in TF32 mode.
"""
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
from test_tf32_cpu import tf32_rne

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUTS = ("pixel_colors_nr", "hit_prob_nr", "render_depth")


@pytest.fixture(autouse=True)
def _fp32_after():
    yield
    renderer.set_precision("fp32")


def _lin_tf32(W, name, x):
    """Linear as torch 1.7.1 ran it on the GPU: input and weight rounded to tf32, products and sums (here) in fp64."""
    y = tf32_rne(x).double() @ tf32_rne(W[name + ".weight"]).double().t()
    b = W.get(name + ".bias")
    return y if b is None else y + b.double()


def f64(d):
    return {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in d.items()}


def oracle_passes(W, oc, que, ref, fine_depth=None):
    """fp64 coarse pass (render_impl's sample_depth) and the fine pass on `fine_depth` (default: the coarse pass'
    own resampling, render_impl's way).  Returns (coarse, fine, fine depths)."""
    Wd, qd, rd = f64(W), f64(que), f64(ref)
    with torch.no_grad():
        depth, _ = orc.sample_depth(qd["depth_range"], qd["coords"], oc["depth_sample_num"], False)
        coarse = orc.render_by_depth(Wd, oc, depth, qd, rd, False, False)
        if fine_depth is None:
            fd = orc.sample_fine_depth(depth, coarse["hit_prob_nr"], qd["depth_range"], oc["fine_depth_sample_num"], False)
            if oc["fine_depth_use_all"]:
                fd = torch.cat([depth, fd], -1)
            fine_depth = torch.sort(fd, -1)[0].float()
        fine = orc.render_by_depth(Wd, oc, fine_depth.double(), qd, rd, False, True)
    return coarse, fine, fine_depth


def native(net, que, ref, fine_depth, mode):
    renderer.set_precision(mode)
    dq, dr = synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda")
    with torch.no_grad():
        coarse = net.render_impl(dq, dr, False)
        fine = net.render_by_depth(fine_depth.cuda(), dq, dr, False, True)
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in coarse.items()}, {k: v.cpu() for k, v in fine.items()}


def check_accuracy(que, ref, cfg, W, monkeypatch):
    oc = flat_cfg({**renderer.base_cfg, **cfg})
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
    gold_c, gold_f, fd = oracle_passes(W, oc, que, ref)
    with monkeypatch.context() as m:
        m.setattr(orc, "_lin", _lin_tf32)
        emu_c, emu_f, _ = oracle_passes(W, oc, que, ref, fd)
    net = renderer.NeuralRayRenderPath(cfg)
    net.load_state_dict(W, strict=True)
    net.cuda()
    f32_c, f32_f = native(net, que, ref, fd, "fp32")
    t32_c, t32_f = native(net, que, ref, fd, "tf32")
    assert torch.equal(t32_c["ray_mask"], f32_c["ray_mask"]) and torch.equal(t32_f["ray_mask"], f32_f["ray_mask"])
    assert not torch.equal(t32_c["pixel_colors_nr"], f32_c["pixel_colors_nr"]), "TF32 mode gave the fp32 mode's bits"
    for tag, gold, emu, f32, t32 in (("coarse", gold_c, emu_c, f32_c, t32_c), ("fine", gold_f, emu_f, f32_f, t32_f)):
        for k in OUTS:
            g = gold[k]
            e = {"tf32": (t32[k].double() - g).abs().flatten(), "emulated": (emu[k] - g).abs().flatten(),
                 "fp32": (f32[k].double() - g).abs().flatten()}
            mx = {n: float(v.max()) for n, v in e.items()}
            q99 = {n: float(torch.quantile(v, 0.99)) for n, v in e.items()}
            r_max, r_q99 = mx["tf32"] / max(mx["emulated"], 1e-30), q99["tf32"] / max(q99["emulated"], 1e-30)
            print(f"{tag} {k}: max abs err tf32 {mx['tf32']:.3e} emulated {mx['emulated']:.3e} fp32 {mx['fp32']:.3e} "
                  f"(ratio {r_max:.2f}); q99 tf32 {q99['tf32']:.3e} emulated {q99['emulated']:.3e} fp32 {q99['fp32']:.3e} "
                  f"(ratio {r_q99:.2f})")
            assert mx["tf32"] <= 2 * mx["emulated"], f"{tag} {k}: max abs err {mx['tf32']:.3e} > 2 x {mx['emulated']:.3e}"
            assert q99["tf32"] <= 2 * q99["emulated"], f"{tag} {k}: q99 abs err {q99['tf32']:.3e} > 2 x {q99['emulated']:.3e}"


def small_cfg(dn, use_vis, fine_vis=None):
    return {"use_hierarchical_sampling": True, "dist_decoder_cfg": {"use_vis": use_vis},
            "fine_dist_decoder_cfg": {"use_vis": use_vis if fine_vis is None else fine_vis}, "depth_sample_num": dn,
            "fine_depth_sample_num": dn, "agg_net_cfg": {"sample_num": dn}, "fine_agg_net_cfg": {"sample_num": dn},
            "render_depth": True}


# one rfn per lane-group instantiation of nr_point_kernel.cu (rfn <= 4: G 4, 5, 6, 7..8: G 8, 9..10: G 10, 11..16: G 16,
# 17..32: G 32), the vis head on and off
@pytest.mark.parametrize("rfn,use_vis", [(3, False), (5, True), (6, False), (8, True), (9, False), (13, True), (20, False)])
def test_accuracy_at_every_lane_group(rfn, use_vis, monkeypatch):
    cfg = small_cfg(32, use_vis)
    que, ref = synthetic.make_scene(48, 64, rfn, seed=20 + rfn, smooth=2, with_que_imgs=False)
    que = synthetic.slice_rays(que, 24 * 64 + 20, 24 * 64 + 44)
    check_accuracy(que, ref, cfg, synthetic.make_weights(cfg, seed=rfn, sigma_gain=1.0, sigma_bias=0.02), monkeypatch)


def test_accuracy_benched_black_800(monkeypatch):
    sys.path.insert(0, ROOT)
    import bench
    wl = bench.WORKLOADS["black_800"]
    cfg = bench.model_cfg(*wl["dn"])
    que, ref = bench.make_workload("black_800")
    check_accuracy(pick_rays(que, 800, 800), ref, cfg, synthetic.make_weights(cfg, seed=0), monkeypatch)


SMALL = {"use_hierarchical_sampling": True, "depth_sample_num": 16, "fine_depth_sample_num": 16, "agg_net_cfg": {"sample_num": 16},
         "fine_agg_net_cfg": {"sample_num": 16}, "render_depth": True}


def small_setup(cfg, rays=(300, 428)):
    que, ref = synthetic.make_scene(40, 48, 4, seed=3, smooth=2)
    que = synthetic.slice_rays(que, *rays)
    W = synthetic.make_weights(cfg, seed=3)
    net = renderer.NeuralRayRenderPath(cfg)
    net.load_state_dict(W, strict=True)
    return synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda"), net.cuda()


def render_eval(net, dq, dr, mode):
    renderer.set_precision(mode)
    with torch.no_grad():
        out = net.render(dict(dq), dict(dr), False)
    torch.cuda.synchronize()
    return out


def test_passes_with_gradients_run_in_fp32():
    """Under autograd the switch does not apply: outputs bit-identical to the fp32 mode, gradients equal up to the
    reordering of the backward's atomics (the tolerance of test_dr_gpu's training contract)."""
    dq, dr, net = small_setup(dict(SMALL))
    results = []
    for mode in ("fp32", "tf32"):
        renderer.set_precision(mode)
        net.zero_grad(set_to_none=True)
        q, r = dict(dq), {k: (v.clone() if torch.is_tensor(v) else v) for k, v in dr.items()}
        r["ray_feats"].requires_grad_(True)
        r["img_feats"].requires_grad_(True)
        torch.manual_seed(7)
        out = net.render(q, r, True)
        loss = ((out["pixel_colors_nr"] - out["pixel_colors_gt"]) ** 2).mean() + (out["pixel_colors_nr_fine"] ** 2).mean() + \
            out["hit_prob_nr"].square().mean() + out["render_depth"].mean()
        loss.backward()
        torch.cuda.synchronize()
        grads = {k: p.grad.clone() for k, p in net.named_parameters() if p.grad is not None}
        grads.update({k: r[k].grad.clone() for k in ("ray_feats", "img_feats")})
        results.append((out, grads))
    (a, ga), (b, gb) = results
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert set(ga) == set(gb) and len(ga) > 100
    for k in ga:
        torch.testing.assert_close(ga[k], gb[k], atol=1e-5 * float(ga[k].abs().max()) + 1e-8, rtol=0, msg=k)


def test_switching_back_and_forth():
    dq, dr, net = small_setup(dict(SMALL))
    outs = [render_eval(net, dq, dr, m) for m in ("tf32", "fp32", "tf32", "fp32")]
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[2][k]) and torch.equal(outs[1][k], outs[3][k]), k
    assert not torch.equal(outs[0]["pixel_colors_nr"], outs[1]["pixel_colors_nr"])


def test_optimizer_step_repacks_the_tf32_weights():
    dq, dr, net = small_setup(dict(SMALL))
    before = render_eval(net, dq, dr, "tf32")
    renderer.set_precision("fp32")
    opt = torch.optim.SGD(net.parameters(), lr=0.05)
    torch.manual_seed(7)
    out = net.render(dict(dq), dict(dr), True)
    ((out["pixel_colors_nr"] - out["pixel_colors_gt"]) ** 2).mean().backward()
    opt.step()
    after = render_eval(net, dq, dr, "tf32")
    fresh = renderer.NeuralRayRenderPath(dict(SMALL))
    fresh.load_state_dict(net.state_dict(), strict=True)
    want = render_eval(fresh.cuda(), dq, dr, "tf32")
    assert not torch.equal(before["pixel_colors_nr"], after["pixel_colors_nr"])
    for k in want:
        assert torch.equal(after[k], want[k]), k


def test_empty_and_chunked_renders():
    dq, dr, net = small_setup(dict(SMALL, ray_batch_num=128), rays=(300, 700))
    whole = renderer.NeuralRayRenderPath(dict(SMALL, ray_batch_num=4096))
    whole.load_state_dict(net.state_dict(), strict=True)
    whole.cuda()
    a, b = render_eval(net, dq, dr, "tf32"), render_eval(whole, dq, dr, "tf32")
    for k in a:
        assert torch.equal(a[k], b[k]), k
    empty = render_eval(net, dict(dq, coords=dq["coords"][:, :0]), dr, "tf32")
    for k in ("pixel_colors_nr", "pixel_colors_nr_fine", "render_depth_fine"):
        assert empty[k].shape[:2] == (1, 0), (k, empty[k].shape)


def test_direct_rendering_with_nr_colours():
    cfg = dict(SMALL, use_dr_prediction=True, use_nr_color_for_dr=True)
    dq, dr, net = small_setup(cfg)
    plain = renderer.NeuralRayRenderPath(dict(SMALL))
    plain.load_state_dict(net.state_dict(), strict=True)
    plain.cuda()
    t32, f32, nr_only = render_eval(net, dq, dr, "tf32"), render_eval(net, dq, dr, "fp32"), render_eval(plain, dq, dr, "tf32")
    for k in nr_only:
        assert torch.equal(t32[k], nr_only[k]), k                         # DR leaves the TF32 NR outputs alone
    for k in ("pixel_colors_dr", "pixel_colors_dr_fine"):
        assert torch.isfinite(t32[k]).all(), k
        err = float((t32[k] - f32[k]).abs().max())
        print(f"{k}: tf32 vs fp32 mode max abs diff {err:.3e}")
        # the fine pass samples where each mode's coarse pass put its inverse-CDF knots: compared in the coarse pass only
        assert err > 0 and (k.endswith("_fine") or err < 2e-2), (k, err)


def test_point_kernel_alone_matches_the_fused_pass():
    """The _lib.PROFILE launch path (nr_point_kernel_tf32 + nr_ray_kernel) gives the fused pass' bits."""
    dq, dr, net = small_setup(dict(SMALL))
    a = render_eval(net, dq, dr, "tf32")
    _lib.PROFILE = []
    try:
        b = render_eval(net, dq, dr, "tf32")
        assert len(_lib.PROFILE) == 2
    finally:
        _lib.PROFILE = None
    for k in a:
        assert torch.equal(a[k], b[k]), k


def rna_bits(x):
    """x rounded to tf32 the way cvt.rna.tf32.f32 does (ties away from zero), on the bit pattern"""
    b = x.view(torch.int32).long() & 0xffffffff
    r = (b + 0x1000) & 0xffffe000
    return torch.where(r >= 2 ** 31, r - 2 ** 32, r).to(torch.int32).view(torch.float32)


def test_tf32_pack_is_the_fp32_pack_of_the_rounded_weights():
    """nr_pack_weights_tf32(W) == the tensor-core buffer nr_pack_weights makes of rna(W) (whose lo parts are zero), bit for
    bit -- except the composed neuray_fc.0 @ prob_embed.2 rows, which are rounded after composing: there the hi slots hold
    rna of the fp32 pack's hi + lo (48-row tile: hi 0..1536, lo 1536..3072)."""
    from neuray_b200 import weights as nr_weights
    cfg = {"use_hierarchical_sampling": True, "dist_decoder_cfg": {"use_vis": True}}
    W = {k: v.cuda() for k, v in synthetic.make_weights(cfg, seed=4).items()}
    T = _lib.tc_layout()
    for dec, agg in (("dist_decoder", "agg_net"), ("fine_dist_decoder", "fine_agg_net")):
        params = {k: v for k, v in W.items() if k.startswith(dec + ".") or k.startswith(agg + ".")}
        rounded = {k: rna_bits(v.cpu()).cuda() for k, v in params.items()}
        want = nr_weights.pack_pass(rounded, dec, agg)[2].cpu()
        full = nr_weights.pack_pass(params, dec, agg)[2].cpu()
        got = nr_weights.pack_pass_tf32(params, dec, agg).cpu()
        torch.cuda.synchronize()
        assert got.numel() == T.total
        pe1 = slice(T.pe1, T.pe1 + 3072)
        keep = torch.ones(T.total, dtype=torch.bool)
        keep[pe1] = False
        assert torch.equal(got[keep], want[keep]), (got[keep] != want[keep]).nonzero()[:5]
        tile = full[pe1]
        assert torch.equal(got[pe1][:1536], rna_bits(tile[:1536] + tile[1536:]))
        assert float(got[pe1][1536:].abs().sum()) == 0.0


def test_header_only_host_drives_the_tf32_entry_points():
    """A coarse pass (+ fused resampling) and a fine pass through ctypes calls only, with nr_pack_weights_tf32 and
    nr_render_pass_fwd_tf32, equal the Python path in TF32 mode bit for bit."""
    cfg = {"use_hierarchical_sampling": True, "dist_decoder_cfg": {"use_vis": False}, "depth_sample_num": 32, "fine_depth_sample_num": 32,
           "agg_net_cfg": {"sample_num": 32}, "fine_agg_net_cfg": {"sample_num": 32}, "render_depth": True}
    que, ref = synthetic.make_scene(48, 64, 5, seed=12, smooth=2, with_que_imgs=False)
    que = synthetic.slice_rays(que, 900, 1100)
    W = synthetic.make_weights(cfg, seed=2)
    dev = torch.device("cuda", 0)
    lib, ck = _lib.lib(), _lib.check
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
            bufs = (f32(L.total_point), f32(L.total_ray), f32(T.total), f32(T.total))
            ws = weight_struct(P, dec, agg)
            ck(lib.nr_pack_weights(C.byref(ws), bufs[0].data_ptr(), bufs[1].data_ptr(), bufs[2].data_ptr(), stream), "pack weights")
            ck(lib.nr_pack_weights_tf32(C.byref(ws), bufs[3].data_ptr(), stream), "pack weights tf32")
            packed[tag] = bufs
        depth = f32(rn, dn)
        ck(lib.nr_sample_depth(q["depth_range"].data_ptr(), rn, dn, None, depth.data_ptr(), None, stream), "sample_depth")
        u = (0.5 * (1 / fdn) + torch.arange(fdn) * (1 / fdn)).to(dev).contiguous()
        fine_depth = f32(rn, fdn)
        out = {}
        for tag, qd, sample_num in (("c", depth, dn), ("f", fine_depth, fdn)):
            pe = nr_posenc(sample_num).to(dev)
            rec = f32(rn * sample_num * _lib.NR_POINT_REC)
            o = {"pixel_colors": f32(rn, 3), "hit_prob": f32(rn, sample_num), "render_depth": f32(rn),
                 "ray_mask": torch.empty(rn, dtype=torch.uint8, device=dev)}
            p = _lib.NrPassParams()
            p.coords, p.que_depth, p.que_cam, p.rn, p.dn = q["coords"].data_ptr(), qd.data_ptr(), cam.data_ptr(), rn, sample_num
            p.feat, p.rgb, p.view_params = feat.data_ptr(), rgb.data_ptr(), vp.data_ptr()
            p.rfn, p.h, p.w, p.fh, p.fw = rfn, h, w, fh, fw
            p.w_point, p.w_ray, p.w_tc = packed[tag][0].data_ptr(), packed[tag][1].data_ptr(), packed[tag][3].data_ptr()
            p.pos_enc = pe.data_ptr()
            p.use_vis, p.var_bias = 0, 0.05
            p.ray_mask_view_num, p.ray_mask_point_num = 2, 8
            p.point_rec = rec.data_ptr()
            p.pixel_colors, p.hit_prob = o["pixel_colors"].data_ptr(), o["hit_prob"].data_ptr()
            p.render_depth, p.ray_mask = o["render_depth"].data_ptr(), o["ray_mask"].data_ptr()
            if tag == "c":
                p.fine_dn, p.fine_use_all, p.fine_u, p.fine_u_stride, p.fine_depth = fdn, 0, u.data_ptr(), 0, fine_depth.data_ptr()
            ck(lib.nr_render_pass_fwd_tf32(C.byref(p), stream), "render pass tf32")
            out[tag] = o
        torch.cuda.synchronize()
    net = renderer.NeuralRayRenderPath(cfg)
    net.load_state_dict(W, strict=True)
    net.cuda()
    want = render_eval(net, synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda"), "tf32")
    fp32 = render_eval(net, synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda"), "fp32")
    assert torch.equal(out["c"]["pixel_colors"][None], want["pixel_colors_nr"])
    assert torch.equal(out["f"]["pixel_colors"][None], want["pixel_colors_nr_fine"])
    assert torch.equal(out["f"]["render_depth"][None], want["render_depth_fine"])
    assert torch.equal(out["f"]["ray_mask"][None].bool(), want["ray_mask_fine"])
    assert not torch.equal(want["pixel_colors_nr"], fp32["pixel_colors_nr"])
