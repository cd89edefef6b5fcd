"""CPU: eval.py's scores (neuray_b200.eval_metrics, neuray_b200.eval).

The float64 restatement of tf.image.psnr / tf.image.ssim (tests/eval_restatement.py) against explicit 11x11 Gaussian
windows; the host build of the product's per-pixel routines (csrc/nr_metrics_math.cuh through
tests/cpu_harness/eval_cpu_harness.cu) against the restatement; LpipsVGG's parameter names and file loading; the CLI's file
enumeration and its message for missing files."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import eval_restatement as er

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")


def pair(kind, h, w, seed):
    """Two uint8 [h,w,3] images: 'random' (independent), 'smooth' (a smooth field and a noisy copy) or 'identical'."""
    rs = np.random.RandomState(seed)
    if kind == "random":
        return rs.randint(0, 256, (h, w, 3)).astype(np.uint8), rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    yy, xx = np.meshgrid(np.linspace(0, 3, h), np.linspace(0, 3, w), indexing="ij")
    a = np.clip(127.5 + 110 * np.sin(xx[..., None] + 1.7 * yy[..., None] + np.arange(3)), 0, 255)
    if kind == "identical":
        return a.astype(np.uint8), a.astype(np.uint8)
    b = np.clip(a + rs.normal(0, 8, a.shape), 0, 255)
    return a.astype(np.uint8), b.astype(np.uint8)


def brute_force(g_u8, p_u8):
    """(psnr, ssim) with every 11x11 Gaussian window summed explicitly."""
    x, y = er.color_map_forward(g_u8).astype(np.float64), er.color_map_forward(p_u8).astype(np.float64)
    h, w, _ = x.shape
    mse = np.mean((x - y) ** 2)
    win = np.outer(er.gauss_window(), er.gauss_window())
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    s = []
    for c in range(3):
        for i in range(h - 10):
            for j in range(w - 10):
                a, b = x[i:i + 11, j:j + 11, c], y[i:i + 11, j:j + 11, c]
                ux, uy = (win * a).sum(), (win * b).sum()
                vx, vy = (win * a * a).sum() - ux * ux, (win * b * b).sum() - uy * uy
                vxy = (win * a * b).sum() - ux * uy
                s.append((2 * ux * uy + c1) * (2 * vxy + c2) / ((ux * ux + uy * uy + c1) * (vx + vy + c2)))
    return (math.inf if mse == 0 else 10 * math.log10(1 / mse)), float(np.mean(s))


SHAPES = [(11, 11), (13, 17), (24, 20)]


def test_gauss_window_is_tensorflows():
    """tf.image.ssim's _fspecial_gauss: softmax over -(i^2 + j^2) / (2 sigma^2), i.e. the outer product of g with itself."""
    i = np.arange(11) - 5.0
    e = -(i[:, None] ** 2 + i[None, :] ** 2) / (2 * 1.5 ** 2)
    soft = np.exp(e) / np.exp(e).sum()
    g = er.gauss_window()
    assert abs(g.sum() - 1) < 1e-15
    assert np.abs(np.outer(g, g) - soft).max() < 1e-16


@pytest.mark.parametrize("kind", ["random", "smooth", "identical"])
@pytest.mark.parametrize("h,w", SHAPES)
def test_restatement_matches_explicit_windows(kind, h, w):
    a, b = pair(kind, h, w, seed=h * w)
    want_psnr, want_ssim = brute_force(a, b)
    assert abs(er.ssim_tf(a, b) - want_ssim) < 1e-12
    got_psnr = er.psnr_tf(a, b)
    assert got_psnr == want_psnr if kind == "identical" else abs(got_psnr - want_psnr) < 1e-12
    if kind == "identical":
        assert got_psnr == math.inf and abs(er.ssim_tf(a, b) - 1) < 1e-12


def test_restatement_refuses_small_images():
    a, b = pair("random", 10, 30, seed=1)
    with pytest.raises(ValueError):
        er.ssim_tf(a, b)


@pytest.fixture(scope="module")
def harness():
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    os.makedirs(BUILD, exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpu_harness", "eval_cpu_harness.cu")
    lib = os.path.join(BUILD, "libeval_cpu_harness.so")
    deps = [src] + [os.path.join(ROOT, "neuray_b200", "csrc", f) for f in ("nr_metrics_math.cuh", "nr_common.cuh")]
    if not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in deps):
        subprocess.run(["nvcc", "-shared", "-Xcompiler", "-fPIC", "-O1", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                        src, "-o", lib], check=True)
    return C.CDLL(lib)


def test_host_unit_and_window(harness):
    v = np.arange(256, dtype=np.uint8)
    out = np.empty(256, np.float32)
    assert harness.nr_cpu_unit(v.ctypes.data_as(C.c_void_p), C.c_longlong(256), out.ctypes.data_as(C.c_void_p)) == 0
    assert np.array_equal(out, er.color_map_forward(v))
    g = np.empty(11, np.float64)
    assert harness.nr_cpu_gauss_window(g.ctypes.data_as(C.c_void_p)) == 0
    assert np.abs(g - er.gauss_window()).max() < 1e-17


@pytest.mark.parametrize("kind", ["random", "smooth", "identical"])
def test_host_build_matches_the_restatement(harness, kind):
    h, w = 37, 29
    a, b = pair(kind, h, w, seed=7)
    out = np.empty(2, np.float64)
    assert harness.nr_cpu_eval_metrics(a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), h, w, out.ctypes.data_as(C.c_void_p)) == 0
    if kind == "identical":
        assert out.tolist() == [math.inf, 1.0]
        return
    assert abs(out[0] - er.psnr_tf(a, b)) < 1e-12
    assert abs(out[1] - er.ssim_tf(a, b)) < 1e-12


def test_lpips_module_names_follow_torchvision_and_lpips():
    import torchvision
    from neuray_b200.eval_metrics import LpipsVGG
    net = LpipsVGG()
    want = {f"features.{k}": v.shape for k, v in torchvision.models.vgg16(weights=None).features[:30].state_dict().items()}
    want.update({f"lin{k}.model.1.weight": torch.Size([1, c, 1, 1]) for k, c in enumerate((64, 128, 256, 512, 512))})
    got = {k: v.shape for k, v in net.state_dict().items()}
    assert got == want
    assert net.param_names() == list(net.state_dict())


def test_lpips_weights_load_from_local_files(tmp_path):
    """A full torchvision vgg16 state dict (classifier included) and an lpips lin file load without a download."""
    import torchvision
    from neuray_b200.eval_metrics import LpipsVGG
    sd = er.seeded_weights(3)
    full = torchvision.models.vgg16(weights=None).state_dict()
    full.update({k: v for k, v in sd.items() if k.startswith("features.")})
    torch.save(full, tmp_path / "vgg16.pth")
    torch.save({k: v for k, v in sd.items() if k.startswith("lin")}, tmp_path / "vgg.pth")
    net = LpipsVGG.from_files(tmp_path / "vgg16.pth", tmp_path / "vgg.pth")
    for k, v in net.state_dict().items():
        assert torch.equal(v, sd[k]), k
    with pytest.raises(Exception):
        net.forward(*pair("random", 32, 32, seed=0))         # a CPU module does not score


def write_folder(tmp_path, n, missing=()):
    from PIL import Image
    gt, pr = tmp_path / "gt", tmp_path / "pr"
    gt.mkdir()
    pr.mkdir()
    for k in range(n):
        a, b = pair("smooth", 40, 48, seed=k)
        if f"{k}.jpg" not in missing:
            Image.fromarray(a).save(gt / f"{k}.jpg")
        if f"{k}-nr_fine.jpg" not in missing:
            Image.fromarray(b).save(pr / f"{k}-nr_fine.jpg")
    return str(gt), str(pr)


def test_cli_enumerates_views_like_eval_py(tmp_path):
    from neuray_b200 import eval as nr_eval
    gt, pr = write_folder(tmp_path, 3)
    (tmp_path / "pr" / "3-nr_coarse.jpg").write_bytes(b"")       # other files in dir_pr are not read
    assert nr_eval.frame_paths(gt, pr) == [(os.path.join(gt, f"{k}.jpg"), os.path.join(pr, f"{k}-nr_fine.jpg")) for k in range(3)]
    from neuray_b200.eval_metrics import read_rgb
    a = read_rgb(os.path.join(gt, "0.jpg"))
    assert a.dtype == np.uint8 and a.shape == (40, 48, 3)


def test_cli_names_the_missing_files(tmp_path, capsys):
    from neuray_b200 import eval as nr_eval
    gt, pr = write_folder(tmp_path, 3, missing=("1-nr_fine.jpg",))
    with pytest.raises(FileNotFoundError, match="1-nr_fine.jpg not found"):
        nr_eval.frame_paths(gt, pr)
    assert nr_eval.main(["--dir_gt", gt, "--dir_pr", pr]) == 2
    err = capsys.readouterr().err
    assert "1-nr_fine.jpg not found" in err and "1 of the 6 expected files" in err
    # eval.py counts every entry of dir_gt: a stray file there asks for one view more
    from PIL import Image
    Image.fromarray(pair("smooth", 40, 48, seed=1)[1]).save(os.path.join(pr, "1-nr_fine.jpg"))
    (tmp_path / "gt" / "notes.txt").write_text("x")
    with pytest.raises(FileNotFoundError, match="3.jpg not found"):
        nr_eval.frame_paths(gt, pr)
    with pytest.raises(SystemExit):
        nr_eval.main(["--dir_gt", gt, "--dir_pr", pr, "--vgg16", "x.pth"])        # --lpips-lin missing
