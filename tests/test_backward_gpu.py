"""GPU: the native training backward of a render pass (nr_render_pass_bwd + nr_tape_gemms through backward.RenderPassFn)
against float64 autograd over the PyTorch restatement of the same pass (tests/torch_restatement.py), at the benchmark's
training shape and at ragged shapes, with the fp32 restatement as the calibration of what fp32 can reach.

Gates, per parameter and per feature map, with g64 the fp64 gradient and rel(a) = |a - g64| / |g64| (Frobenius):
  * rel(native) <= 4 rel(torch fp32), floor REL_FLOOR: the native backward is as accurate as fp32 autograd;
  * max |native - g64| <= 1e-3 max |g64|; for the feature-map gradients a fraction of at most 1e-4 of the elements may be
    outside (a projection within rounding of an image border may flip its mask between fp32 and fp64).
Before every backward the tape workspace holds NaN: a kernel that reads a slot or row the pass did not write produces a
NaN gradient.  Also: the GPU tapes against the host build of the same routines, slot by slot, and two properties at sizes
where fp64 is too heavy (the grid-stride loop above the launch cap, several autograd nodes in one backward).
"""
import ctypes as C
import time

import pytest
import torch

import bench
import neuray_oracle as orc
import ref_packers as packers
import torch_restatement as tr
from neuray_b200 import _lib, backward, render_ops, renderer, synthetic
from neuray_b200.weights import posenc_table
from test_backward_cpu import harness, native_pass as host_pass  # noqa: F401  (harness is a pytest fixture)

pytestmark = pytest.mark.gpu

CHANNELS = {"pix": ("pix",), "hit": ("hit",), "depth": ("depth",), "all": ("pix", "hit", "depth")}
FEAT_BAD_FRAC = 1e-4
# Floor of the calibrated gate.  Bias gradients are sums of dz over all rows with heavy cancellation; the native path
# sums them per 64-row chunk on the tensor cores and then sequentially per CTA, autograd reduces in a tree.  Measured on
# H100: worst rel(native) 5.9e-5 ((5, 37, 11) fine pass, fine_agg_net.agg_impl.neuray_fc.0.bias, fp32 autograd 1.0e-5).
REL_FLOOR = 1e-4
# A gradient fp32 cannot resolve (rel(fp32) > 0.1) is rounding noise in both fp32 computations; measured noise ratio
# native / autograd up to 10.2 (one view, vis_fc2.2.bias, rel 28.6 vs 2.8).
UNRESOLVED = 16


def cfg_for(dn, use_vis=True, bias_val=None):
    dd = {"use_vis": use_vis}
    if bias_val is not None:
        dd["bias_val"] = bias_val
    return {"use_hierarchical_sampling": True, "depth_sample_num": dn, "fine_depth_sample_num": dn, "agg_net_cfg": {"sample_num": dn},
            "fine_agg_net_cfg": {"sample_num": dn}, "render_depth": True, "dist_decoder_cfg": dd, "fine_dist_decoder_cfg": dict(dd)}


def pass_names(is_fine):
    return ("fine_dist_decoder", "fine_agg_net") if is_fine else ("dist_decoder", "agg_net")


def nan_tapes(rfn, n_points):
    """NaN in the backward's tape workspace, exactly the size this pass needs."""
    for k, sh in backward.tape_shapes(rfn, n_points).items():
        backward._WS[(k, "cuda:0")] = torch.full((sh[0] * sh[1] * sh[2],), float("nan"), device="cuda")


def upstream(rn, dn, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return {"pix": torch.randn(1, rn, 3, generator=g, device="cuda"), "hit": torch.randn(1, rn, dn, generator=g, device="cuda") * 0.3,
            "depth": torch.randn(1, rn, generator=g, device="cuda") * 0.2}


def loss_of(pix, hit, dep, up, channels):
    terms = {"pix": lambda: (pix * up["pix"].to(pix.dtype)).sum(), "hit": lambda: (hit * up["hit"].to(hit.dtype)).sum(),
             "depth": lambda: (dep * up["depth"].to(dep.dtype)).sum()}
    return sum(terms[c]() for c in channels)


def native_grads(net, is_fine, depth, dq, dr, up, channels):
    dec, agg = pass_names(is_fine)
    net.zero_grad(set_to_none=True)
    for k in ("ray_feats", "img_feats"):
        dr[k].grad = None
    nan_tapes(dr["imgs"].shape[0], depth.shape[1] * depth.shape[2])
    out = net.render_by_depth(depth, dq, dr, True, is_fine)
    loss_of(out["pixel_colors_nr"], out["hit_prob_nr"], out["render_depth"], up, channels).backward()
    torch.cuda.synchronize()
    g = {k: (p.grad.detach().clone() if p.grad is not None else None) for k, p in net.named_parameters() if k.startswith((dec + ".", agg + "."))}
    g["ray_feats"], g["img_feats"] = dr["ray_feats"].grad.detach().clone(), dr["img_feats"].grad.detach().clone()
    return g


def torch_grads(net, is_fine, depth, dq, dr, up, channels, dtype):
    """Autograd over the restatement with every input cast to dtype."""
    dec, agg = pass_names(is_fine)
    P = {k: v.detach().to(dtype).requires_grad_(True) for k, v in net.named_parameters() if k.startswith((dec + ".", agg + "."))}
    ref = {k: dr[k].detach().to(dtype) for k in ("poses", "Ks", "depth_range", "imgs")}
    for k in ("ray_feats", "img_feats"):
        ref[k] = dr[k].detach().to(dtype).requires_grad_(True)
    cfgv = {"use_vis_prob": bool(net.dist_decoder.cfg["use_vis"]), "var_bias": float(getattr(net, dec).cfg["bias_val"])}
    c = lambda k: dq[k].detach().to(dtype)
    pix, hit, dep = tr.render_pass_torch(P, dec, agg, cfgv, depth.to(dtype), c("coords"), c("poses"), c("Ks"), c("depth_range"), ref,
                                         posenc_table(depth.shape[-1]).to(depth.device, dtype))
    loss_of(pix, hit, dep, up, channels).backward()
    torch.cuda.synchronize()
    g = {k: (v.grad if v.grad is not None else None) for k, v in P.items()}
    g["ray_feats"], g["img_feats"] = ref["ray_feats"].grad, ref["img_feats"].grad
    return g


def compare(label, gn, g32, g64):
    """The gates of the module docstring.  Returns (worst rel(native) / rel(fp32), feature-map elements outside, tensors
    checked); every violation of the case is listed in the failure.

    A gradient that fp32 cannot resolve at all (rel(fp32) > 0.1) only has its noise compared (UNRESOLVED): the bias of rgb_fc.4
    feeds a softmax over the views and is zero analytically (fp64 gives ~1e-17, fp32 ~1e-8), and with one view the
    vis_fc2 weights cancel in weight / sum(weight) (measured rel(fp32) ~ 1 and above).  Max-abs against such a g64 only
    measures rounding noise.  Where fp32 autograd itself is off by more than 1e-3 max|g64| the max-abs gate is 4x its
    error: agg_impl.vis_fc2.2.bias at train_dtu is one sum over 262 144 rows; measured native error 3.8e-5 of 1.9e-2, and
    it passes the calibrated gate."""
    worst, bad_feat, checked, fails = 0.0, 0, 0, []
    for k, b in g64.items():
        a = gn[k]
        if a is not None and not bool(torch.isfinite(a).all()):
            fails.append((k, "non-finite native gradient"))
            continue
        if b is None or float(b.abs().max()) == 0.0:
            if a is not None and float(a.abs().max()) != 0.0:
                fails.append((k, "gradient where fp64 has none", float(a.abs().max())))
            continue
        if a is None:
            fails.append((k, "no native gradient"))
            continue
        a64, c64 = a.double(), g32[k].double()
        nb = float(b.norm())
        rel_n, rel_32 = float((a64 - b).norm()) / nb, float((c64 - b).norm()) / nb
        checked += 1
        if rel_32 > 0.1:          # fp32 cannot resolve it: only the size of the noise is compared
            if rel_n > UNRESOLVED * rel_32:
                fails.append((k, "unresolved", rel_n, rel_32))
            continue
        if rel_n > max(4 * rel_32, REL_FLOOR):
            fails.append((k, "rel", rel_n, rel_32))
        worst = max(worst, rel_n / max(rel_32, 1e-12))
        bad = int(((a64 - b).abs() > max(1e-3 * float(b.abs().max()), 4 * float((c64 - b).abs().max()))).sum())
        if k in ("ray_feats", "img_feats"):
            bad_feat += bad
            if bad > FEAT_BAD_FRAC * b.numel():
                fails.append((k, "max-abs", bad, b.numel()))
        elif bad:
            fails.append((k, "max-abs", float((a64 - b).abs().max()), float(b.abs().max())))
    assert not fails, (label, fails)
    return worst, bad_feat, checked


def check_pass(label, net, is_fine, depth, dq, dr, up, channels):
    gn = native_grads(net, is_fine, depth, dq, dr, up, channels)
    g32 = torch_grads(net, is_fine, depth, dq, dr, up, channels, torch.float32)
    g64 = torch_grads(net, is_fine, depth, dq, dr, up, channels, torch.float64)
    worst, bad_feat, checked = compare(label, gn, g32, g64)
    print(f"backward {label}: worst rel(native)/rel(fp32) = {worst:.3f}, d_feat outside = {bad_feat}, tensors checked = {checked}")
    return checked


def scene(rfn, rays, dn, seed, cfg, full_res=False, look_away=False, h=40, w=48):
    que, ref = synthetic.make_scene(h, w, rfn, seed=50 + seed, smooth=2)
    idx = torch.randperm(que["coords"].shape[1], generator=torch.Generator().manual_seed(seed))[:rays]
    que = dict(que, coords=que["coords"][:, idx].contiguous())
    if look_away:      # the query camera turned around: every sample projects behind / outside every reference view
        que["poses"] = que["poses"].clone()
        que["poses"][:, :, :3] = que["poses"][:, :, :3] * torch.tensor([1.0, 1.0, -1.0])[None, :, None]
    if full_res:       # feature maps at image resolution: the align_corners gather
        g = torch.Generator().manual_seed(seed)
        ref["ray_feats"] = torch.randn(rfn, 32, *ref["imgs"].shape[-2:], generator=g)
        ref["img_feats"] = torch.randn(rfn, 32, *ref["imgs"].shape[-2:], generator=g)
    net = renderer.NeuralRayRenderPath(cfg)
    net.load_state_dict(synthetic.make_weights(cfg, seed=seed), strict=True)
    net.cuda()
    dq, dr = synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda")
    dr["ray_feats"].requires_grad_(True)
    dr["img_feats"].requires_grad_(True)
    return net, dq, dr


def depths(net, dq, dr, dn_c, dn_f):
    """Coarse depths from sample_depth, fine depths resampled from the native coarse pass: the same for all three."""
    depth = renderer.sample_depth(dq["depth_range"], dq["coords"], dn_c, False)[0]
    with torch.no_grad():
        hit = net.render_by_depth(depth, dq, dr, False, False)["hit_prob_nr"]
    fd = torch.sort(render_ops.sample_fine_depth(depth, hit, dq["depth_range"], dn_f, False), -1)[0]
    return depth, fd.contiguous()


# (views, rays, samples): no row count rfn * rays * dn is a multiple of 64; rows or points end in both halves of a tile
RAGGED = [(3, 7, 5), (1, 13, 9), (5, 37, 11), (32, 9, 7), (2, 3, 200), (4, 50, 3)]


@pytest.mark.parametrize("rfn,rays,dn", RAGGED)
def test_ragged_shapes_against_fp64(rfn, rays, dn):
    """Both passes, each upstream gradient alone and all three together; use_vis alternates between the shapes."""
    t0 = time.time()
    use_vis = (rfn + dn) % 2 == 0
    net, dq, dr = scene(rfn, rays, dn, rfn * 100 + dn, cfg_for(dn, use_vis))
    depth, fd = depths(net, dq, dr, dn, dn)
    checked, fails = 0, []
    for is_fine, d in ((False, depth), (True, fd)):
        up = upstream(rays, dn, 7 + int(is_fine))
        for ch, channels in CHANNELS.items():
            try:
                checked += check_pass(f"({rfn},{rays},{dn}) {'fine' if is_fine else 'coarse'} {ch}", net, is_fine, d, dq, dr, up, channels)
            except AssertionError as e:
                fails.append(str(e))
    assert not fails, "\n".join(fails)
    assert checked > 200       # 244 with 32 views (many views see none of the 9 rays: fewer non-zero gradients)
    print(f"backward ({rfn},{rays},{dn}): {time.time() - t0:.1f} s")


@pytest.mark.parametrize("variant", ["no_vis", "bias_val", "full_res"])
def test_configuration_variants_against_fp64(variant):
    rfn, rays, dn = 4, 21, 13
    cfg = cfg_for(dn, use_vis=variant != "no_vis", bias_val=0.3 if variant == "bias_val" else None)
    net, dq, dr = scene(rfn, rays, dn, 11, cfg, full_res=variant == "full_res")
    if variant == "full_res":
        assert dr["ray_feats"].shape[-2:] == dr["imgs"].shape[-2:]
    depth, fd = depths(net, dq, dr, dn, dn)
    for is_fine, d in ((False, depth), (True, fd)):
        check_pass(f"{variant} {'fine' if is_fine else 'coarse'}", net, is_fine, d, dq, dr, upstream(rays, dn, 3), CHANNELS["all"])


def test_look_away_camera():
    """The query camera turned around: most samples project behind / outside every view."""
    rfn, rays, dn = 3, 7, 5
    net, dq, dr = scene(rfn, rays, dn, 4, cfg_for(dn, False), look_away=True, h=48, w=64)
    depth, fd = depths(net, dq, dr, dn, dn)
    for is_fine, d in ((False, depth), (True, fd)):
        check_pass(f"look-away {'fine' if is_fine else 'coarse'}", net, is_fine, d, dq, dr, upstream(rays, dn, 5), CHANNELS["all"])


def test_train_dtu_against_fp64():
    """bench.py's train_dtu step shape exactly: 8 views 304x400, 512 rays, 64 + 64 samples (262 144 rows per pass), the
    fine decoder with a vis head; both passes, the fp64 reference run and freed per pass."""
    t0 = time.time()
    wl = bench.WORKLOADS["train_dtu"]
    cfg = dict(bench.model_cfg(*wl["dn"]), fine_dist_decoder_cfg={"use_vis": True}, ray_batch_num=bench.TRAIN_RAYS)
    que, ref = bench.make_workload("train_dtu", seed=5)
    idx = torch.randperm(que["coords"].shape[1], generator=torch.Generator().manual_seed(100))[:bench.TRAIN_RAYS]
    que = dict(que, coords=que["coords"][:, idx].contiguous())
    net = renderer.NeuralRayRenderPath(cfg)
    net.load_state_dict(synthetic.make_weights(cfg, seed=1), strict=True)
    net.cuda()
    dq, dr = synthetic.to_device(que, "cuda"), synthetic.to_device(ref, "cuda")
    dr["ray_feats"].requires_grad_(True)
    dr["img_feats"].requires_grad_(True)
    depth, fd = depths(net, dq, dr, *wl["dn"])
    assert dr["imgs"].shape[0] * depth.shape[1] * depth.shape[2] == 262144
    torch.cuda.reset_peak_memory_stats()
    for is_fine, d in ((False, depth), (True, fd)):
        check_pass(f"train_dtu {'fine' if is_fine else 'coarse'}", net, is_fine, d, dq, dr, upstream(512, 64, 9 + int(is_fine)), CHANNELS["all"])
        torch.cuda.empty_cache()
    print(f"backward train_dtu: peak memory {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB, {time.time() - t0:.1f} s")


# ---- GPU tapes against the host build of the same routines ----------------------------------------------------------

SLOT_NAMES = ("R_RF R_DD R_H1 R_H2 R_P1 R_RGBF R_NF R_Q8 R_R16 R_B1 R_U R_VH R_X2 R_U2 R_WH R_CH1 R_CH2 R_MASK R_HITN R_VISN R_BLEND "
              "R_TCODE G_DD0 G_DD1 G_DD2 G_PE0 G_PE1 G_NF0 G_NF1 G_RD0 G_RD1 G_B0 G_B1 G_V0 G_V1 G_V20 G_V21 G_C0 G_C1 G_C2 P_GLOB "
              "P_GIN P_GH P_G16 P_RGBO P_AX P_O P_XH P_Y P_T16 P_SIG P_ALPHA GP_B0SUM GP_GEO0 GP_GEO1 GP_DQ GP_DK GP_DV GP_DFC "
              "GP_DLNY GP_OG0 GP_OG1").split()
TAPE_PREFIX = {"tape_row": "R_", "grad_row": "G_", "tape_point": "P_", "grad_point": "GP_"}


def slot_name(tape, slot):
    """Nearest named slot at or below `slot` on that tape, e.g. R_H1+5."""
    pre = TAPE_PREFIX[tape]
    named = [(_lib.bwd_slot(n), n) for n in SLOT_NAMES if n.split("_")[0] + "_" == pre]
    start, name = max([s for s in named if s[0] <= slot], default=(0, pre + "?"))
    return f"{name}+{slot - start}"


def device_tapes(params, dec, agg, use_vis, que, ref, coords, que_depth, g_pix, g_hit, g_dep, var_bias=0.05):
    """nr_render_pass_bwd on the GPU with the inputs host_pass builds (packed on the host, copied to the device)."""
    rfn = ref["imgs"].shape[0]
    rays, dn = que_depth.shape[1:]
    d = lambda t: t.contiguous().float().cuda()
    wp, wr = (d(t) for t in packers.pack_pass_weights(params, dec, agg, torch.device("cpu")))
    feat = d(torch.cat([ref["ray_feats"], ref["img_feats"]], 1).permute(0, 2, 3, 1))
    rgb = d(torch.cat([ref["imgs"], torch.zeros_like(ref["imgs"][:, :1])], 1).permute(0, 2, 3, 1))
    vp = d(packers.view_param_block(ref["poses"], ref["Ks"], ref["depth_range"]))
    cam = d(packers.camera_block(que["poses"][0], que["Ks"][0], que["depth_range"][0]))
    cc, qd, pe = d(coords[0]), d(que_depth[0]), d(packers.posenc_table(dn))
    p = _lib.NrPassParams()
    p.coords, p.que_depth, p.que_cam, p.rn, p.dn = cc.data_ptr(), qd.data_ptr(), cam.data_ptr(), rays, dn
    p.feat, p.rgb, p.view_params = feat.data_ptr(), rgb.data_ptr(), vp.data_ptr()
    p.rfn, p.h, p.w, p.fh, p.fw = rfn, ref["imgs"].shape[2], ref["imgs"].shape[3], ref["ray_feats"].shape[2], ref["ray_feats"].shape[3]
    p.w_point, p.w_ray, p.pos_enc = wp.data_ptr(), wr.data_ptr(), pe.data_ptr()
    p.use_vis, p.var_bias = int(use_vis), var_bias
    bufs = {k: torch.full(sh, float("nan"), device="cuda") for k, sh in backward.tape_shapes(rfn, rays * dn).items()}
    d_feat = torch.zeros_like(feat)
    b = _lib.NrBwdParams()
    keep = [d(t[0]) for t in (g_pix, g_hit, g_dep)]
    b.d_pixel_colors, b.d_hit_prob, b.d_render_depth = (t.data_ptr() for t in keep)
    b.tape_row, b.grad_row = bufs["tape_row"].data_ptr(), bufs["grad_row"].data_ptr()
    b.tape_point, b.grad_point = bufs["tape_point"].data_ptr(), bufs["grad_point"].data_ptr()
    b.d_feat = d_feat.data_ptr()
    _lib.check(_lib.lib().nr_render_pass_bwd(C.byref(p), C.byref(b), torch.cuda.current_stream().cuda_stream), "nr_render_pass_bwd")
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in bufs.items()}, d_feat.cpu()


@pytest.mark.parametrize("rfn,rays,dn,use_vis", [(3, 7, 5, False), (5, 37, 11, True), (2, 3, 200, True)])
def test_device_tapes_match_host_build(harness, rfn, rays, dn, use_vis):  # noqa: F811
    """The host build runs the eleven phases one after another; the GPU runs each phase's items concurrently.  Same
    elements written (NaN pattern), the feature-map tap codes bit for bit, every other value within 1e-4 (1 + |host|)."""
    torch.manual_seed(rfn)
    cfg = cfg_for(dn, use_vis)
    que, ref = synthetic.make_scene(40, 48, rfn, seed=60 + rfn, smooth=2)
    coords = que["coords"][:, torch.randperm(que["coords"].shape[1])[:rays]].contiguous()
    W = synthetic.make_weights(cfg, seed=rfn)
    dec, agg = "dist_decoder", "agg_net"
    params = {k: v for k, v in W.items() if k.startswith((dec + ".", agg + "."))}
    que_depth = orc.sample_depth(que["depth_range"], coords, dn, False)[0].contiguous()
    g_pix, g_hit, g_dep = torch.randn(1, rays, 3), torch.randn(1, rays, dn) * 0.5, torch.randn(1, rays) * 0.3
    host, host_feat, _ = host_pass(harness, params, dec, agg, use_vis, que, ref, coords, que_depth, g_pix, g_hit, g_dep)
    dev, dev_feat = device_tapes(params, dec, agg, use_vis, que, ref, coords, que_depth, g_pix, g_hit, g_dep)
    tcode = _lib.bwd_slot("R_TCODE")
    for k in host:
        h, g = host[k], dev[k]
        if k == "tape_row":       # integer bits stored as float: compare the bits, then leave the slot out
            assert torch.equal(h[:, tcode].view(torch.int32), g[:, tcode].view(torch.int32)), "R_TCODE differs"
            keep = torch.ones(h.shape[1], dtype=torch.bool)
            keep[tcode] = False
            h, g = h[:, keep], g[:, keep]
            names = [s for s in range(host[k].shape[1]) if s != tcode]
        else:
            names = list(range(h.shape[1]))
        nh, ng = torch.isnan(h), torch.isnan(g)
        if not torch.equal(nh, ng):
            per_slot = (nh != ng).sum((0, 2))
            s = int(per_slot.argmax())
            raise AssertionError(f"{k}: written elements differ, worst slot {slot_name(k, names[s])} ({int(per_slot[s])} elements)")
        err = torch.where(nh, torch.zeros_like(h), (g - h).abs() / (1 + h.abs()))
        per_slot = err.amax((0, 2))
        s = int(per_slot.argmax())
        assert float(per_slot[s]) <= 1e-4, f"{k}: worst slot {slot_name(k, names[s])}, error {float(per_slot[s]):.3e}"
    assert float(((dev_feat - host_feat).abs() / (1 + host_feat.abs())).max()) <= 1e-4


# ---- properties at sizes where fp64 is too heavy --------------------------------------------------------------------

def _grads(net, dr, prefixes):
    g = {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None and k.startswith(prefixes)}
    g["ray_feats"], g["img_feats"] = dr["ray_feats"].grad.detach().clone(), dr["img_feats"].grad.detach().clone()
    return g


def _same(label, a, b, tol=1e-5):
    assert set(a) == set(b), (label, set(a) ^ set(b))
    worst, fails = 0.0, []
    top = max(float(v.norm()) for v in b.values())
    for k in b:
        assert bool(torch.isfinite(a[k]).all()), (label, k)
        nb = float(b[k].norm())
        if nb < 1e-5 * top:       # rounding noise only: rgb_fc.4.bias feeds a softmax over the views, zero analytically
            continue
        r = float((a[k] - b[k]).norm()) / nb if nb > 0 else float(a[k].norm())
        worst = max(worst, r)
        if r > tol:
            fails.append((k, r))
    print(f"backward {label}: worst norm-relative difference {worst:.2e} over {len(b)} tensors")
    assert not fails, (label, fails)


def test_grid_stride_loop_above_the_launch_cap():
    """8 views x 1 100 rays x 64 samples = 563 200 rows: above the 132 * 32 * 128 = 540 672 threads of a row launch, so
    every row kernel takes a second grid-stride iteration.  The backward of the whole pass equals the sum of the backwards
    of its two 550-ray halves (each under the cap); only the order of the sums differs."""
    rfn, rays, dn = 8, 1100, 64
    cfg = cfg_for(dn, False)
    net, dq, dr = scene(rfn, rays, dn, 12, cfg, h=64, w=80)
    assert rfn * rays * dn > 132 * 32 * 128
    depth = renderer.sample_depth(dq["depth_range"], dq["coords"], dn, False)[0]
    up = upstream(rays, dn, 13)
    native_grads(net, False, depth, dq, dr, up, CHANNELS["all"])
    whole = _grads(net, dr, ("dist_decoder.", "agg_net."))
    net.zero_grad(set_to_none=True)
    for k in ("ray_feats", "img_feats"):
        dr[k].grad = None
    for a, b in ((0, 550), (550, 1100)):       # gradients accumulate over the two halves
        q = dict(dq, coords=dq["coords"][:, a:b])
        out = net.render_by_depth(depth[:, a:b].contiguous(), q, dr, True, False)
        part = {k: v[:, a:b] for k, v in up.items()}
        loss_of(out["pixel_colors_nr"], out["hit_prob_nr"], out["render_depth"], part, CHANNELS["all"]).backward()
    torch.cuda.synchronize()
    _same("grid-stride: whole vs halves", whole, _grads(net, dr, ("dist_decoder.", "agg_net.")))


def test_several_render_pass_nodes_in_one_backward():
    """A batch chunked 200 + 200 + 112 rays, coarse then fine per chunk (as render_chunks interleaves them), on fixed
    depths: one loss.backward() runs six RenderPassFn nodes that share the tape workspace and accumulate into the same
    .grad.  Same gradients as the batch in one chunk."""
    rfn, rays, dn = 6, 512, 24
    net, dq, dr = scene(rfn, rays, dn, 14, cfg_for(dn, True), h=48, w=64)
    depth, fd = depths(net, dq, dr, dn, dn)
    up_c, up_f = upstream(rays, dn, 15), upstream(rays, dn, 16)
    res = {}
    for name, bounds in (("one chunk", [(0, 512)]), ("three chunks", [(0, 200), (200, 400), (400, 512)])):
        net.zero_grad(set_to_none=True)
        for k in ("ray_feats", "img_feats"):
            dr[k].grad = None
        nan_tapes(rfn, 512 * dn)
        loss = 0.0
        for a, b in bounds:
            q = dict(dq, coords=dq["coords"][:, a:b])
            for is_fine, d, up in ((False, depth, up_c), (True, fd, up_f)):
                out = net.render_by_depth(d[:, a:b].contiguous(), q, dr, True, is_fine)
                loss = loss + loss_of(out["pixel_colors_nr"], out["hit_prob_nr"], out["render_depth"], {k: v[:, a:b] for k, v in up.items()},
                                      CHANNELS["all"])
        loss.backward()
        torch.cuda.synchronize()
        res[name] = _grads(net, dr, ("dist_decoder.", "agg_net.", "fine_dist_decoder.", "fine_agg_net."))
    _same("three chunks vs one", res["three chunks"], res["one chunk"])
