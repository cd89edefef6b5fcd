"""CPU: the validation metric PSNR_SSIM (reference network/metrics.py:13-79).

The float64 restatement (tests/metrics_restatement.py) against explicit 11x11 windows; the host build of the product's
per-pixel routines (csrc/nr_metrics_math.cuh through tests/cpu_harness/metrics_cpu_harness.cu) against numpy's
quantisation and against the restatement; patch.install() rebinding the reference's metric."""
import ctypes as C
import math
import os
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest

import metrics_restatement as mr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")


def images(kind, h, w, seed):
    """Two float32 [h,w,3] images: 'random' (independent uniform), 'smooth' (a smooth field and a noisy copy) or 'range'
    (values well outside [0, 1], so the clip matters)."""
    rs = np.random.RandomState(seed)
    if kind == "random":
        a, b = rs.uniform(0, 1, (h, w, 3)), rs.uniform(0, 1, (h, w, 3))
    elif kind == "smooth":
        yy, xx = np.meshgrid(np.linspace(0, 3, h), np.linspace(0, 3, w), indexing="ij")
        a = 0.5 + 0.4 * np.sin(xx[..., None] + 1.7 * yy[..., None] + np.arange(3))
        b = a + rs.normal(0, 0.03, a.shape)
    else:
        a, b = rs.uniform(-0.5, 1.5, (h, w, 3)), rs.uniform(-0.5, 1.5, (h, w, 3))
    return a.astype(np.float32), b.astype(np.float32)


def brute_force(g, p):
    """(psnr, ssim) of two uint8 [h,w,3] images with every 11x11 window summed explicitly."""
    g, p = g.astype(np.float64), p.astype(np.float64)
    h, w, _ = g.shape
    mse = np.mean([np.mean((g[..., c] - p[..., c]) ** 2) for c in range(3)])
    C1, C2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2
    per_channel = []
    for c in range(3):
        s = []
        for i in range(5, h - 5):
            for j in range(5, w - 5):
                x, y = g[i - 5:i + 6, j - 5:j + 6, c], p[i - 5:i + 6, j - 5:j + 6, c]
                ux, uy = x.mean(), y.mean()
                vx, vy = ((x - ux) ** 2).sum() / 120, ((y - uy) ** 2).sum() / 120
                vxy = ((x - ux) * (y - uy)).sum() / 120
                s.append((2 * ux * uy + C1) * (2 * vxy + C2) / ((ux * ux + uy * uy + C1) * (vx + vy + C2)))
        per_channel.append(np.mean(s))
    return (math.inf if mse == 0 else 10 * math.log10(255 * 255 / mse)), float(np.mean(per_channel))


SHAPES = [(11, 11), (13, 17), (24, 20)]


@pytest.mark.parametrize("kind", ["random", "smooth", "range"])
@pytest.mark.parametrize("h,w", SHAPES)
def test_restatement_matches_explicit_windows(kind, h, w):
    a, b = images(kind, h, w, seed=h * w)
    g, p = mr.color_map_backward(a), mr.color_map_backward(b)
    want_psnr, want_ssim = brute_force(g, p)
    got_psnr, got_ssim = mr.psnr_ssim(a, b, h, w)
    assert abs(got_ssim - want_ssim) < 1e-12
    assert abs(got_psnr - want_psnr) < 1e-12


def test_restatement_crop_and_identical_images():
    a, b = images("smooth", 40, 30, seed=3)
    g, p = mr.color_map_backward(a), mr.color_map_backward(b)
    # ratio 0.8: 1 - 0.8 is just below 0.2 in float64, so int(40 * 0.2) // 2 = 3 rows and int(30 * 0.2) // 2 = 2 columns
    assert mr.margins(40, 30, 0.8) == (3, 2)
    assert mr.psnr_ssim(a, b, 40, 30, 0.8) == pytest.approx(brute_force(g[3:37, 2:28], p[3:37, 2:28]), abs=1e-12)
    assert mr.psnr_ssim(a, a, 40, 30) == (math.inf, 1.0)
    with pytest.raises(ValueError):
        mr.psnr_ssim(a[:10], b[:10], 10, 30)


@pytest.fixture(scope="module")
def harness():
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    os.makedirs(BUILD, exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpu_harness", "metrics_cpu_harness.cu")
    lib = os.path.join(BUILD, "libmetrics_cpu_harness.so")
    deps = [src] + [os.path.join(ROOT, "neuray_b200", "csrc", f) for f in ("nr_metrics_math.cuh", "nr_common.cuh")]
    if not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in deps):
        subprocess.run(["nvcc", "-shared", "-Xcompiler", "-fPIC", "-O1", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                        src, "-o", lib], check=True)
    return C.CDLL(lib)


def quantisation_edge_values():
    k = np.arange(256, dtype=np.float32) / np.float32(255)
    edges = [k, np.nextafter(k, np.float32(-1)), np.nextafter(k, np.float32(2)),
             np.array([-0.0, -1e-30, -0.5, -1.0, -1e30, -np.inf, 1.0 + 1e-7, 1.5, 2.0, 1e30, np.inf, 0.5, 1e-30], np.float32)]
    return np.concatenate(edges).astype(np.float32)


def test_host_quantisation_matches_numpy(harness):
    x = quantisation_edge_values()
    q = np.empty(x.shape, np.uint8)
    assert harness.nr_cpu_quantise(x.ctypes.data_as(C.c_void_p), C.c_longlong(x.size), q.ctypes.data_as(C.c_void_p)) == 0
    want = (x * 255).clip(0, 255).astype(np.uint8)
    assert np.array_equal(q, want), np.nonzero(q != want)
    # astype truncates: one ulp below k/255 lands below k for most k, which must give k - 1, not k
    assert np.array_equal(want[257:512], np.arange(255))


@pytest.mark.parametrize("ratio", [1.0, 0.8])
@pytest.mark.parametrize("kind", ["random", "smooth", "range"])
def test_host_build_matches_the_restatement(harness, kind, ratio):
    h, w = 37, 29
    a, b = images(kind, h, w, seed=7)
    out = np.empty(4, np.float64)
    assert harness.nr_cpu_image_metrics(a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), h, w, *mr.margins(h, w, ratio),
                                        out.ctypes.data_as(C.c_void_p)) == 0
    mh, mw = mr.margins(h, w, ratio)
    g, p = mr.color_map_backward(a)[mh:h - mh, mw:w - mw], mr.color_map_backward(b)[mh:h - mh, mw:w - mw]
    d = g.astype(np.int64) - p.astype(np.int64)
    assert out[:3].tolist() == (d * d).reshape(-1, 3).sum(0).astype(np.float64).tolist()
    assert abs(out[3] - mr.psnr_ssim(a, b, h, w, ratio)[1]) < 1e-12


def test_patch_rebinds_and_restores_the_metric(monkeypatch):
    """patch.install() on stand-in network.* modules (a trimmed tree: no init_net, no loss) swaps PSNR_SSIM in both places
    the reference's trainer can look it up; uninstall() puts the reference's back."""
    from neuray_b200 import metrics, patch

    class RefPSNR_SSIM:
        pass

    class RefVisualizeImage:
        pass

    base = type("NeuralRayBaseRenderer", (), {n: (lambda self: None) for n in ("render_by_depth", "fine_render_impl", "render_impl", "render")})
    gen = type("NeuralRayGenRenderer", (base,), {"predict_mean_for_depth_loss": lambda self: None})
    net = types.ModuleType("network")
    net.__path__ = []
    mods = {"network": net, "network.render_ops": types.ModuleType("network.render_ops"),
            "network.renderer": types.ModuleType("network.renderer"), "network.metrics": types.ModuleType("network.metrics")}
    mods["network.renderer"].NeuralRayBaseRenderer, mods["network.renderer"].NeuralRayGenRenderer = base, gen
    ref_metrics = mods["network.metrics"]
    ref_metrics.PSNR_SSIM = RefPSNR_SSIM
    ref_metrics.name2metrics = {"psnr_ssim": RefPSNR_SSIM, "vis_img": RefVisualizeImage}
    for k, v in mods.items():
        monkeypatch.setitem(sys.modules, k, v)
    assert not patch._ORIGINALS
    try:
        patch.install()
        assert ref_metrics.PSNR_SSIM is metrics.PSNR_SSIM
        assert ref_metrics.name2metrics == {"psnr_ssim": metrics.PSNR_SSIM, "vis_img": RefVisualizeImage}
    finally:
        patch.uninstall()
    assert ref_metrics.PSNR_SSIM is RefPSNR_SSIM
    assert ref_metrics.name2metrics == {"psnr_ssim": RefPSNR_SSIM, "vis_img": RefVisualizeImage}


def test_metric_class_keeps_the_reference_interface():
    from neuray_b200 import metrics
    assert metrics.PSNR_SSIM.default_cfg == {"eval_margin_ratio": 1.0}
    assert metrics.PSNR_SSIM({}).cfg == {"eval_margin_ratio": 1.0}
    assert set(metrics.name2metrics) == {"psnr_ssim"}
    assert metrics.margins(800, 800, 1.0) == (0, 0) and metrics.margins(756, 1008, 0.8) == (75, 100)
