"""CPU: the per-view visibility output (cfg render_visibility, visibility_nr[r, v] = Σ_d hit_nr[r, d] · vis_v[r, d]).

  * the fp64 oracle's intermediates (neuray_oracle.render_by_depth(..., keep): prj_vis, prj_mask, hit_prob_nr) against the
    unmodified reference's, stored in tests/golden/visibility.npz (oracle/gen_golden_visibility.py), for both passes;
  * the routines of csrc/nr_visibility_math.cuh, compiled as HOST code (tests/cpu_harness/vis_cpu_harness.cu) and run
    the way the kernel splits each ray, against the fp64 oracle: the values, exact zeros for a view that sees none of a
    ray's samples, and visibility <= Σ_d hit."""
import ctypes as C
import json
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import gen_golden_visibility as ggv
import neuray_oracle as orc
import ref_packers as weights
from gen_golden import flat_cfg
from neuray_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "_build")
GOLDEN = os.path.join(ROOT, "tests", "golden", "visibility.npz")
CASES = tuple(ggv.CASES)
ATOL, RTOL = 1e-4, 1e-3


def f64(d):
    return {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in d.items()}


def oracle_visibility(keep, hit):
    """Σ_d hit[q, r, d] · prj_vis[v, q, r, d] -> [qn, rn, rfn], in the dtype of the inputs."""
    return (keep["prj_vis"][..., 0] * hit[None]).sum(-1).permute(1, 2, 0)


def load_case(name):
    """cfg, inputs regenerated from the case's spec, the reference's recorded tensors and fine-pass depths."""
    z = np.load(GOLDEN)
    pre = name + "_"
    spec = json.loads(bytes(z[pre + "spec_json"]).decode())
    que, ref, W = ggv.make_inputs(spec)
    sums = torch.tensor([float(t.double().sum()) for t in ggv.input_tensors(que, ref, W)], dtype=torch.float64)
    torch.testing.assert_close(sums, torch.from_numpy(z[pre + "input_sums"]), rtol=1e-9, atol=1e-9)
    gold = {k[len(pre):]: torch.from_numpy(z[k].copy()) for k in z.files if k.startswith(pre) and not k.endswith(("spec_json", "input_sums"))}
    return spec["cfg"], que, ref, W, gold


def oracle_pass(cfg, W, que, ref, is_fine, fine_depth):
    """fp64 render_by_depth of one pass (the coarse pass on render_impl's depths): (keep, hit_prob_nr, que_depth)."""
    oc = flat_cfg(cfg)
    depth = fine_depth if is_fine else orc.sample_depth(que["depth_range"], que["coords"], oc["depth_sample_num"])[0]
    keep = {}
    with torch.no_grad():
        out = orc.render_by_depth(f64(W), oc, depth.double(), f64(que), f64(ref), False, is_fine, keep)
    return keep, out["hit_prob_nr"], depth


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("is_fine", [False, True])
def test_oracle_matches_reference(name, is_fine):
    cfg, que, ref, W, gold = load_case(name)
    sfx = "_fine" if is_fine else ""
    keep, hit, _ = oracle_pass(cfg, W, que, ref, is_fine, gold["que_depth_fine"])
    assert torch.equal(keep["prj_mask"].float(), gold["prj_mask" + sfx])
    torch.testing.assert_close(keep["prj_vis"].float(), gold["prj_vis" + sfx], atol=1e-5, rtol=1e-4)
    # hit_prob_nr comes out of the whole aggregation network, which the reference runs in fp32
    torch.testing.assert_close(hit.float(), gold["hit_prob_nr" + sfx], atol=ATOL, rtol=RTOL)
    want = oracle_visibility({"prj_vis": gold["prj_vis" + sfx].double()}, gold["hit_prob_nr" + sfx].double())
    torch.testing.assert_close(oracle_visibility(keep, hit), want, atol=ATOL, rtol=RTOL)
    # the cases reach the masked branch: some points lie outside some views
    assert 0 < float(gold["prj_mask" + sfx].mean()) < 1


@pytest.fixture(scope="module")
def harness():
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not available")
    os.makedirs(BUILD, exist_ok=True)
    so = os.path.join(BUILD, "libnr_vis_cpu.so")
    src = os.path.join(ROOT, "tests", "cpu_harness", "vis_cpu_harness.cu")
    csrc = os.path.join(ROOT, "neuray_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in ("nr_visibility_math.cuh", "nr_train_math.cuh", "nr_common.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.run(["nvcc", "-shared", "-Xcompiler", "-fPIC", "-O1", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                        "-o", so, src], check=True, capture_output=True)
    lib = C.CDLL(so)
    lib.nr_vis_cpu.argtypes = [C.c_void_p, C.c_void_p]
    return lib


def host_visibility(harness, cfg, W, que, ref, que_depth, hit, is_fine):
    """nr_view_visibility's routines on the host for one pass with the given hit_prob [1,rn,dn]: [1,rn,rfn]."""
    oc = flat_cfg(cfg)
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
    hp = hit[0].contiguous().float()
    p = _lib.NrPassParams()
    p.coords, p.que_depth, p.que_cam, p.rn, p.dn = cc.data_ptr(), qd.data_ptr(), cam.data_ptr(), rn, dn
    p.feat, p.rgb, p.view_params = feat.data_ptr(), rgb.data_ptr(), vp.data_ptr()
    p.rfn, p.h, p.w, p.fh, p.fw = rfn, ref["imgs"].shape[2], ref["imgs"].shape[3], ref["ray_feats"].shape[2], ref["ray_feats"].shape[3]
    p.w_point = wp.data_ptr()
    p.use_vis, p.var_bias = int(oc["dist_decoder_use_vis"]), float(oc[dec + "_bias_val"])
    out = torch.full((rn, rfn), float("nan"))
    q = _lib.NrVisParams()
    q.hit_prob, q.visibility = hp.data_ptr(), out.data_ptr()
    assert harness.nr_vis_cpu(C.addressof(p), C.addressof(q)) == 0
    return out[None]


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("is_fine", [False, True])
def test_host_routine_matches_oracle(harness, name, is_fine):
    cfg, que, ref, W, gold = load_case(name)
    keep, hit, depth = oracle_pass(cfg, W, que, ref, is_fine, gold["que_depth_fine"])
    hit32 = hit.float()
    want = oracle_visibility(keep, hit32.double())
    got = host_visibility(harness, cfg, W, que, ref, depth, hit32, is_fine)
    torch.testing.assert_close(got.double(), want, atol=ATOL, rtol=RTOL)
    unseen = (keep["prj_mask"][..., 0].sum(-1) == 0).permute(1, 2, 0)            # [qn,rn,rfn]: no sample in the view
    assert torch.equal(got[unseen], torch.zeros(int(unseen.sum())))
    assert bool((got <= hit32.sum(-1, keepdim=True) + 1e-6).all())
    if name.startswith("v8_novis") and not is_fine:
        assert int(unseen.sum()) > 0
