"""Encoders upstream of the ray path (SURVEY.md 8f row 1) without a GPU:
  * the oracle's functional restatement against the golden outputs of the UNMODIFIED reference modules
    (tests/golden/encoders.npz, oracle/gen_golden_encoders.py);
  * the product's layer graphs + index math (csrc/nr_encoder_graph.cuh, csrc/nr_conv.cuh) executed on the host by
    tests/cpu_harness/conv_cpu_harness.cu -- the tensor-core convolution is emulated CTA by CTA through the same staging /
    fragment / epilogue routines the kernel calls -- against the same goldens and against torch's conv2d."""
import ctypes as C
import json
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import neuray_oracle as orc
from golden_io import GOLDEN_DIR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")


def golden():
    z = np.load(os.path.join(GOLDEN_DIR, "encoders.npz"))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    cases = {tag: {k[2:]: t(z[k]) for k in z.files if k.startswith(tag + "_")} for tag in ("a", "b")}
    img_w = orc.encoder_test_weights(json.loads(str(z["image_shapes"])), 11)
    vis_w = orc.encoder_test_weights(json.loads(str(z["vis_shapes"])), 12)
    return cases, img_w, vis_w


@pytest.mark.parametrize("tag", ["a", "b"])
def test_oracle_matches_the_reference(tag):
    cases, img_w, vis_w = golden()
    c = cases[tag]
    got = orc.res_unet_light(img_w, "", c["imgs"])
    assert got.shape == c["img_feats"].shape
    assert torch.allclose(got, c["img_feats"], atol=2e-5, rtol=1e-5), float((got - c["img_feats"]).abs().max())
    got = orc.vis_encoder(vis_w, "", c["ray_in"], c["img_feats"])
    assert torch.allclose(got, c["ray_feats"], atol=2e-5, rtol=1e-5), float((got - c["ray_feats"]).abs().max())


@pytest.fixture(scope="module")
def harness():
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


def _ptrs(tensors):
    arr = (C.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr()
    return arr


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("tag", ["a", "b"])
def test_layer_graphs_on_the_host_match_the_reference(harness, tag):
    cases, img_w, vis_w = golden()
    c = cases[tag]
    n, _, h, w = c["imgs"].shape
    fh, fw = C.c_int(), C.c_int()
    harness.nr_cpu_image_dims(h, w, C.byref(fh), C.byref(fw))
    assert (fh.value, fw.value) == tuple(c["img_feats"].shape[-2:])
    n_img, n_vis = C.c_int(), C.c_int()
    harness.nr_cpu_encoder_counts(C.byref(n_img), C.byref(n_vis))
    assert n_img.value == len(img_w) and n_vis.value == len(vis_w)
    # frame pack: ray_feats slot 0..31 (input: the init net's ray_feats), img_feats slot 32..63
    feat = torch.zeros(n, fh.value, fw.value, 64)
    feat[..., :32] = _nhwc(c["ray_in"])
    imgs = c["imgs"].contiguous()
    params = [t.contiguous() for t in img_w.values()]
    rc = harness.nr_cpu_image_encoder(_ptrs(params), len(params), C.c_void_p(imgs.data_ptr()), n, h, w, C.c_void_p(feat.data_ptr()), 64, 32)
    assert rc == 0
    got = feat[..., 32:].permute(0, 3, 1, 2)
    err = float((got - c["img_feats"]).abs().max())
    assert err < 5e-5, err
    vparams = [t.contiguous() for t in vis_w.values()]
    rc = harness.nr_cpu_vis_encoder(_ptrs(vparams), len(vparams), C.c_void_p(feat.data_ptr()), n, fh.value, fw.value)
    assert rc == 0
    got = feat[..., :32].permute(0, 3, 1, 2)
    err = float((got - c["ray_feats"]).abs().max())
    assert err < 1e-4, err
    # the img_feats slot is untouched by the vis encoder
    assert float((feat[..., 32:].permute(0, 3, 1, 2) - c["img_feats"]).abs().max()) < 5e-5


@pytest.mark.parametrize("n,h,w,cin,cout,ks,stride,reflect,rot,pad,cin_ref,bm", [
    (2, 9, 11, 16, 32, 3, 2, 1, 0, -1, 0, 128),      # Cin 16 (KC 16), stride 2, odd sizes, images share a CTA
    (3, 7, 9, 32, 64, 3, 1, 0, 0, -1, 0, 128),       # zero padding, a warp's rows straddle two images
    (1, 12, 13, 64, 128, 3, 1, 1, 32, -1, 0, 128),   # 128 outputs (4 m-tiles per warp), rotated input channels
    (2, 8, 8, 32, 32, 1, 2, 1, 0, -1, 0, 128),       # 1x1 stride 2 (the downsample branch)
    (1, 20, 20, 128, 64, 3, 1, 1, 0, -1, 0, 128),    # 4 CTAs, the last one partial
    (2, 22, 26, 16, 32, 8, 2, 1, 0, 2, 12, 0),       # ResEncoder.conv1: 8x8 stride 2 padding 2, 12 reference channels packed into 16
    (1, 10, 12, 48, 32, 1, 1, 1, 0, -1, 0, 0),       # DepthInitNet.conv_out: 48 inputs (three K steps of 16)
    (3, 9, 10, 64, 128, 3, 1, 1, 0, -1, 0, 64),      # 64-pixel tiles, 128 outputs (two m-tiles per warp), images straddle CTAs and warps
    (2, 7, 11, 32, 64, 3, 2, 1, 0, -1, 0, 64),       # 64-pixel tiles, 64 outputs (one m-tile per warp)
    (3, 13, 15, 32, 32, 3, 1, 1, 0, -1, 0, 256),     # 256-pixel tiles, 32 outputs (two m-tiles per warp, two pipeline stages)
    (2, 18, 20, 16, 32, 3, 2, 0, 0, -1, 0, 256),     # 256-pixel tiles, Cin 16, zero padding, stride 2
])
def test_emulated_tensor_core_conv_matches_conv2d(harness, n, h, w, cin, cout, ks, stride, reflect, rot, pad, cin_ref, bm):
    g = torch.Generator().manual_seed(cin * 1000 + cout + ks)
    cr = cin_ref or cin
    x = torch.randn(n, cin, h, w, generator=g)
    x[:, cr:] = 0.0 if cr < cin else x[:, cr:]
    wt = torch.randn(cout, cr, ks, ks, generator=g) / (cin * ks * ks) ** 0.5
    bias = torch.randn(cout, generator=g)
    p = (ks - 1) // 2 if pad < 0 else pad
    xin = x if rot == 0 else torch.roll(x, rot, 1)       # packed channel c reads reference channel (c + rot) % cin
    xp = F.pad(x[:, :cr], (p, p, p, p), mode="reflect") if (reflect and p) else x[:, :cr]
    want = F.conv2d(xp, wt, bias, stride=stride, padding=0 if (reflect or not p) else p)
    res = torch.randn(n, want.shape[2], want.shape[3], cout, generator=g)
    want = want + res.permute(0, 3, 1, 2)
    # channel-last input with slack channels on both sides, output into a slot of a wider buffer
    xs, xo, ys, yo = cin + 8, 4, cout + 8, 4
    xbuf = torch.full((n, h, w, xs), 7.0)
    xbuf[..., xo:xo + cin] = _nhwc(xin if rot == 0 else torch.roll(x, -rot, 1))
    if cr < cin:
        xbuf[..., xo + cr:xo + cin] = 5.0        # the padding channels meet zero weight rows: their content must not matter
    ybuf = torch.full((n, want.shape[2], want.shape[3], ys), -3.0)
    stats = torch.zeros(n, cout, 2, dtype=torch.float64)
    wt_c, b_c, r_c = wt.contiguous(), bias.contiguous(), res.contiguous()
    rc = harness.nr_cpu_conv2d(C.c_void_p(xbuf.data_ptr()), C.c_void_p(wt_c.data_ptr()), C.c_void_p(b_c.data_ptr()), C.c_void_p(r_c.data_ptr()),
                               C.c_void_p(ybuf.data_ptr()), C.c_void_p(stats.data_ptr()), n, h, w, cin, cout, ks, stride, reflect, rot, xs, xo, ys, yo, pad, cin_ref, bm)
    assert rc == 0
    got = ybuf[..., yo:yo + cout].permute(0, 3, 1, 2)
    assert float((got - want).abs().max()) < 2e-5
    assert torch.all(ybuf[..., :yo] == -3.0) and torch.all(ybuf[..., yo + cout:] == -3.0)       # nothing outside the slot
    assert torch.allclose(stats[..., 0], want.double().sum((2, 3)), atol=1e-4)
    assert torch.allclose(stats[..., 1], (want.double() ** 2).sum((2, 3)), rtol=1e-5, atol=1e-4)


def depth_init_golden():
    z = np.load(os.path.join(GOLDEN_DIR, "depth_init_net.npz"))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    ref = {k[4:]: t(z[k]) for k in z.files if k.startswith("ref_")}
    return ref, t(z["out"]), orc.encoder_test_weights(json.loads(str(z["shapes"])), 13)


def test_depth_init_net_oracle_matches_the_reference():
    ref, out, W = depth_init_golden()
    got = orc.depth_init_net(W, "", ref)
    assert got.shape == out.shape
    assert torch.allclose(got, out, atol=3e-5, rtol=1e-5), float((got - out).abs().max())


def test_depth_init_net_graph_on_the_host_matches_the_reference(harness):
    """DepthInitNet (init_net.py:76-101) after extract_depth / get_diff_feats: ResEncoder (8x8 first conv on 12 channels packed
    into 16), depth_skip, conv_out -- the product's graph + packing on the host against the unmodified module's output."""
    ref, out, W = depth_init_golden()
    n, _, h, w = ref["imgs"].shape
    depth = orc.extract_depth_for_init(ref["depth_range"], ref["depth"]).contiguous()
    diff = orc.get_diff_feats(ref, depth).contiguous()
    fh, fw, nt = C.c_int(), C.c_int(), C.c_int()
    harness.nr_cpu_depth_init_dims(h, w, C.byref(fh), C.byref(fw), C.byref(nt))
    assert (fh.value, fw.value) == tuple(out.shape[-2:]) and nt.value == len(W)
    params = [t.contiguous() for t in W.values()]
    buf = torch.full((n, fh.value, fw.value, 64), 9.0)
    imgs = ref["imgs"].contiguous()
    rc = harness.nr_cpu_depth_init(_ptrs(params), len(params), C.c_void_p(imgs.data_ptr()), C.c_void_p(depth.data_ptr()), C.c_void_p(diff.data_ptr()),
                                   n, h, w, C.c_void_p(buf.data_ptr()), 64, 0)
    assert rc == 0
    got = buf[..., :32].permute(0, 3, 1, 2)
    err = float((got - out).abs().max())
    assert err < 1e-4, err
    assert bool(torch.all(buf[..., 32:] == 9.0))


def test_parameter_containers_carry_the_reference_state_dicts():
    """encoders.ImageEncoder / VisEncoder / init_nets.DepthInitNet: names, order and shapes of state_dict() equal the unmodified
    reference modules' (recorded in the goldens), so a reference checkpoint loads strict=True; the library's layer tables have
    the same tensor counts; and there is no CPU path."""
    from neuray_b200 import _lib, encoders, init_nets
    z = np.load(os.path.join(GOLDEN_DIR, "encoders.npz"))
    zi = np.load(os.path.join(GOLDEN_DIR, "depth_init_net.npz"))
    want = {"image": json.loads(str(z["image_shapes"])), "vis": json.loads(str(z["vis_shapes"])), "depth_init": json.loads(str(zi["shapes"]))}
    mods = {"image": encoders.ImageEncoder(), "vis": encoders.VisEncoder(), "depth_init": init_nets.DepthInitNet()}
    names = {"image": encoders.image_param_names(), "vis": encoders.vis_param_names(), "depth_init": init_nets.param_names()}
    for k, m in mods.items():
        sd = m.state_dict()
        assert list(sd) == list(want[k]) == names[k], k
        assert {n: list(v.shape) for n, v in sd.items()} == want[k], k
        m.load_state_dict(orc.encoder_test_weights(want[k], 1), strict=True)
    lay = _lib.NrEncoderLayout()
    _lib.check(_lib.lib().nr_encoder_layout(C.byref(lay)), "nr_encoder_layout")
    assert (lay.image_tensors, lay.vis_tensors, lay.depth_init_tensors) == (len(want["image"]), len(want["vis"]), len(want["depth_init"]))
    # conv weights keep their element count in the packed buffers, except ResEncoder.conv1 (12 -> 16 input channels)
    n_img = sum(int(np.prod(s)) for s in want["image"].values())
    assert n_img <= lay.image_packed_floats <= n_img + 4 * len(want["image"])
    n_di = sum(int(np.prod(s)) for s in want["depth_init"].values()) + 32 * 4 * 64
    assert n_di <= lay.depth_init_packed_floats <= n_di + 4 * len(want["depth_init"])
    with pytest.raises(_lib.NeurayB200Error):
        with torch.no_grad():
            mods["image"](torch.zeros(1, 3, 32, 32))
    assert encoders.image_dims(800, 800) == (200, 200) and init_nets.dims(768, 1008) == (192, 252) and encoders.image_dims(40, 52) == (12, 16)
    fh, fw = C.c_int(), C.c_int()
    assert _lib.lib().nr_image_encoder_dims(16, 16, C.byref(fh), C.byref(fw)) != 0          # below the smallest supported image
    assert _lib.lib().nr_image_encoder_workspace(8, 800, 800) > 0 and _lib.lib().nr_depth_init_workspace(8, 800, 800) > 0
