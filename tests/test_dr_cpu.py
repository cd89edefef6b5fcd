"""CPU: direct rendering (cfg use_dr_prediction, reference renderer.py:85-125 and sph_solver.py).

  * the oracle's restatement (oracle/dr_oracle.py) against the unmodified reference's outputs stored in
    tests/golden/dr.npz (oracle/gen_golden_dr.py);
  * the per-point / per-ray routines of csrc/nr_dr_math.cuh, compiled as HOST code (tests/cpu_harness/dr_cpu_harness.cu),
    against the oracle;
  * the fp32 Cholesky SH solve against an fp64 solve, including the near-singular cases: one valid view, all hit ~ 0 (the
    insufficient-weight branch) and points no view sees."""
import ctypes as C
import json
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import dr_oracle as dro
import gen_golden_dr
import neuray_oracle as orc
from gen_golden import flat_cfg as golden_flat_cfg
import ref_packers as weights
from neuray_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
GOLDEN = os.path.join(ROOT, "tests", "golden", "dr.npz")
CASES = ("sh_novis", "sh_vis", "nrc_novis", "nrc_vis")


def flat_cfg(cfg):
    """gen_golden.flat_cfg plus the two direct-rendering keys the oracle reads."""
    out = golden_flat_cfg(cfg)
    out["alpha_value_ground_state"] = cfg.get("alpha_value_ground_state", -15)
    out["use_nr_color_for_dr"] = cfg.get("use_nr_color_for_dr", False)
    return out


def load_case(name):
    """cfg, inputs regenerated from the case's spec, the reference's outputs and fine-pass depths."""
    z = np.load(GOLDEN)
    pre = name + "_"
    spec = json.loads(bytes(z[pre + "spec_json"]).decode())
    que, ref, W = gen_golden_dr.make_inputs(spec)
    sums = torch.tensor([float(t.double().sum()) for t in gen_golden_dr.input_tensors(que, ref, W)], dtype=torch.float64)
    torch.testing.assert_close(sums, torch.from_numpy(z[pre + "input_sums"]), rtol=1e-9, atol=1e-9)
    out = {k[len(pre) + 4:]: torch.from_numpy(z[k].copy()) for k in z.files if k.startswith(pre + "out_")}
    return spec["cfg"], que, ref, W, out, torch.from_numpy(z[pre + "que_depth_fine"].copy())


def test_golden_regs_are_the_solver_defaults():
    z = np.load(GOLDEN)
    assert np.array_equal(z["sph_regs"], np.array(dro.SH_REGS, dtype=np.float32))


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference(name):
    cfg, que, ref, W, gold, fd = load_case(name)
    out = dro.render_impl_dr(W, flat_cfg(cfg), que, ref, False, fine_depth_override=fd)
    for k in ("pixel_colors_dr", "hit_prob_dr", "pixel_colors_dr_fine", "hit_prob_dr_fine"):
        # the reference inverts the normal matrix in fp32 (torch.inverse), the oracle solves in fp64
        torch.testing.assert_close(out[k].float(), gold[k], atol=2e-4, rtol=1e-3, msg=lambda m: f"{name} {k}: {m}")
    for k in ("pixel_colors_nr", "pixel_colors_nr_fine"):
        torch.testing.assert_close(out[k], gold[k], atol=1e-5, rtol=1e-4)


@pytest.fixture(scope="module")
def harness():
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    os.makedirs(BUILD, exist_ok=True)
    so = os.path.join(BUILD, "libnr_dr_cpu.so")
    src = os.path.join(ROOT, "tests", "cpu_harness", "dr_cpu_harness.cu")
    csrc = os.path.join(ROOT, "neuray_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in ("nr_dr_math.cuh", "nr_train_math.cuh", "nr_common.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.run(["nvcc", "-shared", "-Xcompiler", "-fPIC", "-O1", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                        "-o", so, src], check=True, capture_output=True)
    lib = C.CDLL(so)
    lib.nr_dr_cpu.argtypes = [C.c_void_p, C.c_void_p]
    lib.nr_sh_fit_cpu.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 5
    return lib


def host_direct_render(harness, cfg, W, que, ref, que_depth, is_fine, nr_colors=None):
    """nr_direct_render's routines on the host for one pass: (pixel_colors_dr [1,rn,3], hit_prob_dr [1,rn,dn])."""
    dec, agg = ("fine_dist_decoder", "fine_agg_net") if is_fine else ("dist_decoder", "agg_net")
    params = {k: v for k, v in W.items() if k.split(".")[0] in (dec, agg)}
    rfn = ref["imgs"].shape[0]
    rn, dn = que_depth.shape[1:]
    wp, _ = weights.pack_pass_weights(params, dec, agg, torch.device("cpu"))
    feat = torch.cat([ref["ray_feats"], ref["img_feats"]], 1).permute(0, 2, 3, 1).contiguous()
    rgb = torch.cat([ref["imgs"], torch.zeros_like(ref["imgs"][:, :1])], 1).permute(0, 2, 3, 1).contiguous()
    vp = weights.view_param_block(ref["poses"], ref["Ks"], ref["depth_range"])
    cam = weights.camera_block(que["poses"][0], que["Ks"][0], que["depth_range"][0])
    cc, qd = que["coords"][0].contiguous().float(), que_depth[0].contiguous().float()
    rec = torch.zeros(rn * dn, _lib.NR_POINT_REC)
    if nr_colors is not None:
        rec[:, 16:19] = nr_colors.reshape(-1, 3)
    p = _lib.NrPassParams()
    p.coords, p.que_depth, p.que_cam, p.rn, p.dn = cc.data_ptr(), qd.data_ptr(), cam.data_ptr(), rn, dn
    p.feat, p.rgb, p.view_params = feat.data_ptr(), rgb.data_ptr(), vp.data_ptr()
    p.rfn, p.h, p.w, p.fh, p.fw = rfn, ref["imgs"].shape[2], ref["imgs"].shape[3], ref["ray_feats"].shape[2], ref["ray_feats"].shape[3]
    p.w_point, p.point_rec = wp.data_ptr(), rec.data_ptr()
    p.use_vis, p.var_bias = int(cfg["dist_decoder_use_vis"]), float(cfg[dec + "_bias_val"])
    pix, hit, colors = torch.empty(rn, 3), torch.empty(rn, dn), torch.empty(rn * dn * 3)
    d = _lib.NrDrParams()
    d.regs[:] = dro.SH_REGS
    d.alpha_ground_state, d.use_nr_color = float(cfg["alpha_value_ground_state"]), int(cfg["use_nr_color_for_dr"])
    d.point_colors, d.pixel_colors_dr, d.hit_prob_dr = colors.data_ptr(), pix.data_ptr(), hit.data_ptr()
    assert harness.nr_dr_cpu(C.addressof(p), C.addressof(d)) == 0
    return pix[None], hit[None]


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("is_fine", [False, True])
def test_host_routine_matches_oracle(harness, name, is_fine):
    cfg, que, ref, W, _, fd = load_case(name)
    cfg = flat_cfg(cfg)
    que_depth = fd if is_fine else orc.sample_depth(que["depth_range"], que["coords"], cfg["depth_sample_num"])[0]
    keep = {}
    orc.render_by_depth(W, cfg, que_depth, que, ref, False, is_fine, keep)
    pix_o, hit_o = dro.direct_rendering(cfg, keep)
    pix, hit = host_direct_render(harness, cfg, W, que, ref, que_depth, is_fine, keep["colors"])
    torch.testing.assert_close(hit.double(), hit_o, atol=1e-4, rtol=1e-3)
    torch.testing.assert_close(pix.double(), pix_o, atol=1e-4, rtol=1e-3)


def _sh_case(npts, rfn, seed, kind):
    g = torch.Generator().manual_seed(seed)
    dirs = torch.nn.functional.normalize(torch.randn(npts, rfn, 3, generator=g), dim=-1)
    rgb = torch.rand(npts, rfn, 3, generator=g)
    hit = torch.rand(npts, rfn, generator=g)
    if kind == "one_view":          # a single view sees the point
        hit[:, 1:] = 0
        rgb[:, 1:] = 0
    elif kind == "no_hit":          # the insufficient-weight branch: every weight + 1e-4
        hit = hit * 1e-9
    elif kind == "unseen":          # no view sees the point: zero hit and colour
        hit.zero_()
        rgb.zero_()
    qdir = torch.nn.functional.normalize(torch.randn(npts, 3, generator=g), dim=-1)
    return dirs, rgb, hit, qdir


@pytest.mark.parametrize("kind", ["random", "one_view", "no_hit", "unseen"])
@pytest.mark.parametrize("rfn", [1, 3, 8, 32])
def test_sh_solve_against_fp64(harness, kind, rfn):
    npts = 256
    dirs, rgb, hit, qdir = _sh_case(npts, rfn, seed=rfn * 7 + len(kind), kind=kind)
    rows = torch.cat([hit[..., None], rgb, dirs], -1).contiguous()
    hsum = hit.sum(1).contiguous()
    color = torch.empty(npts, 3)
    regs = torch.tensor(dro.SH_REGS)
    harness.nr_sh_fit_cpu(npts, rfn, rows.data_ptr(), hsum.data_ptr(), regs.data_ptr(), qdir.contiguous().data_ptr(), color.data_ptr())
    w = hit.double() / (hit.double().sum(1, keepdim=True) + 1e-3)
    M, rhs = dro.sh_normal_equations(dirs.double(), rgb.double(), w, regs.double())
    ref = (dro.sh_basis(qdir.double()[:, None]) @ torch.linalg.solve(M, rhs))[:, 0]
    assert torch.isfinite(color).all()
    # fp32 against fp64: the error scales with the normal matrix's condition number
    tol = 1e-6 * torch.linalg.cond(M).clamp_min(1.0) * ref.abs().amax(-1).clamp_min(1.0)
    err = (color.double() - ref).abs().amax(-1)
    assert (err <= tol).all(), (err / tol).max()
    if kind == "unseen":
        assert color.abs().max() == 0
