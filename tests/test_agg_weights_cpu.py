"""CPU: the per-view weights inside the aggregation net (cfg render_agg_weights):
neuray_weights_nr[r, v] = Σ_d hit_nr[r, d] · weight0[v, r, d] and geometry_weights_nr[r, v] = Σ_d hit_nr[r, d] · weight[v, r, d],
weight0 the reference's NeuRay weight (ibrnet.py:334-337) and weight its geometry weight (ibrnet.py:349-350).

  * the oracle's two weights (recorded from ibrnet_forward's view poolings by render_by_depth_with_agg), in fp32 and fp64,
    against the unmodified reference's, stored in tests/golden/agg_weights.npz (oracle/gen_golden_agg_weights.py), for
    both passes;
  * the contract: Σ_v weight = Σ_v vis / (Σ_v vis + 1e-8), weight0 <= mask / (Σ_v mask + 1e-8) (so Σ_v weight0 <= 1),
    and a point that no view sees has exactly 0 in both;
  * the binding: the two entry points and NrAggParams match the header, and the ABI version;
  * the SASS of the built library: the export kernels issue their wgmma in whole batches."""
import json
import os
import re

import numpy as np
import pytest
import torch

import gen_golden_agg_weights as gga
import gen_golden_visibility as ggv
import neuray_oracle as orc
from gen_golden import flat_cfg
from neuray_b200 import _lib
from test_point_kernel_sass import _batches, sass  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "agg_weights.npz")
CASES = tuple(gga.CASES)


def f64(d):
    return {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in d.items()}


def render_by_depth_with_agg(W, cfg, que_depth, que, ref, is_train, is_fine, keep):
    """neuray_oracle.render_by_depth(..., keep) that also leaves the oracle's two pooling weights in keep["weight0"] and
    keep["weight"], and the geometry pooling's unmasked vis_fc2 output in keep["vis2"], in the layout of its prj fields:
    [rfn, qn, rn, dn, 1].  ibrnet_forward pools three times in a fixed order, with weight0, the mask weight and the
    geometry weight (ibrnet.py:338, 339, 352); vis_fc2's sigmoid is its last sigmoid before the third pooling."""
    pooled, sig = [], []
    own_pool, own_sig = orc.weighted_mean_var, orc._sigmoid

    def pool(x, w):
        pooled.append((w, sig[-1] if sig else None))
        return own_pool(x, w)

    def sigmoid(x):
        y = own_sig(x)
        sig.append(y)
        return y
    orc.weighted_mean_var, orc._sigmoid = pool, sigmoid
    try:
        out = orc.render_by_depth(W, cfg, que_depth, que, ref, is_train, is_fine, keep)
    finally:
        orc.weighted_mean_var, orc._sigmoid = own_pool, own_sig
    assert len(pooled) == 3, len(pooled)
    rfn, qn, rn, dn, _ = keep["prj_mask"].shape
    to_prj = lambda t: t.permute(2, 0, 1, 3).reshape(rfn, qn, rn, dn, 1)            # [qn*rn, dn, rfn, 1] -> prj layout
    keep["weight0"], keep["weight"], keep["vis2"] = to_prj(pooled[0][0]), to_prj(pooled[2][0]), to_prj(pooled[2][1])
    return out


def oracle_view_sums(w, hit):
    """Σ_d hit[q, r, d] · w[v, q, r, d] -> [qn, rn, rfn], in the dtype of the inputs."""
    return (w[..., 0] * hit[None]).sum(-1).permute(1, 2, 0)


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


def oracle_pass(cfg, W, que, ref, is_fine, fine_depth, dtype=torch.float64):
    """The oracle's render_by_depth of one pass (the coarse pass on render_impl's depths), in fp64 unless dtype says
    otherwise: (keep, outputs)."""
    oc = flat_cfg(cfg)
    depth = fine_depth if is_fine else orc.sample_depth(que["depth_range"], que["coords"], oc["depth_sample_num"])[0]
    cast = f64 if dtype == torch.float64 else (lambda d: d)
    keep = {}
    with torch.no_grad():
        out = render_by_depth_with_agg(cast(W), oc, depth.to(dtype), cast(que), cast(ref), False, is_fine, keep)
    return keep, out


def prj(t):
    """The reference's [rn, dn, rfn, 1] in the oracle's layout of prj fields [rfn, 1, rn, dn, 1]."""
    return t.permute(2, 0, 1, 3)[:, None]


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("is_fine", [False, True])
def test_oracle_matches_reference(name, is_fine):
    """Run in fp32, the reference's own precision, the oracle's weights equal the reference's within 1e-6.  In fp64 they
    differ from the reference by its own fp32 rounding through the aggregation net, within 1e-5."""
    cfg, que, ref, W, gold = load_case(name)
    sfx = "_fine" if is_fine else ""
    for dtype, tol in ((torch.float32, 1e-6), (torch.float64, 1e-5)):
        keep, out = oracle_pass(cfg, W, que, ref, is_fine, gold["que_depth_fine"], dtype)
        assert torch.equal(keep["prj_mask"].float(), gold["prj_mask" + sfx])
        for k in ("weight0", "weight"):
            err = float((keep[k].double() - prj(gold[k + sfx]).double()).abs().max())
            print(f"{name}{sfx} {k} {dtype}: max |oracle - reference| {err:.2e}")
            assert err <= tol, (k, dtype, err)
        torch.testing.assert_close(out["hit_prob_nr"].float(), gold["hit_prob_nr" + sfx], atol=1e-4, rtol=1e-3)


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("is_fine", [False, True])
def test_the_contract_of_the_two_weights(name, is_fine):
    """In the fp64 oracle: Σ_v weight = Σ_v vis / (Σ_v vis + 1e-8), weight0 <= mask / (Σ_v mask + 1e-8) and so Σ_v weight0
    <= 1.  In the reference's fp32 golden the bound on weight0 holds exactly too (a sigmoid is at most 1 in fp32)."""
    cfg, que, ref, W, gold = load_case(name)
    keep, out = oracle_pass(cfg, W, que, ref, is_fine, gold["que_depth_fine"])
    mask = keep["prj_mask"].double()
    vis = keep["vis2"] * mask
    s = vis.sum(0)
    torch.testing.assert_close(keep["weight"].sum(0), s / (s + 1e-8), atol=1e-12, rtol=0)
    assert bool((keep["weight"] >= 0).all())
    bound = mask / (mask.sum(0, keepdim=True) + 1e-8)
    assert bool((keep["weight0"] <= bound).all()) and bool((keep["weight0"] >= 0).all())
    assert bool((keep["weight0"].sum(0) <= 1).all())
    sfx = "_fine" if is_fine else ""
    m32 = gold["prj_mask" + sfx]
    assert bool((prj(gold["weight0" + sfx]) <= m32 / (m32.sum(0, keepdim=True) + 1e-8)).all())
    # unnormalised like render_depth: Σ_v of the view sums is Σ_d hit · (Σ_v of the weight)
    hit = out["hit_prob_nr"]
    torch.testing.assert_close(oracle_view_sums(keep["weight"], hit).sum(-1), (hit * (s / (s + 1e-8))[..., 0]).sum(-1), atol=1e-12, rtol=0)


@pytest.mark.parametrize("is_fine", [False, True])
def test_a_point_no_view_sees_gets_zero(is_fine):
    cfg, que, ref, W, gold = load_case("v5_unseen")
    keep, _ = oracle_pass(cfg, W, que, ref, is_fine, gold["que_depth_fine"])
    unseen = keep["prj_mask"][..., 0].sum(0) == 0                            # [qn,rn,dn]
    assert int(unseen.sum()) > 0
    sfx = "_fine" if is_fine else ""
    for k in ("weight0", "weight"):
        for w in (keep[k][..., 0], prj(gold[k + sfx])[..., 0]):
            assert bool((w[:, unseen] == 0).all()), k


def test_entry_points_and_params_match_the_header():
    src = open(os.path.join(ROOT, "include", "neuray_b200.h")).read()
    body = re.search(r"typedef struct NrAggParams \{(.*?)\} NrAggParams;", src, re.S).group(1)
    fields = re.findall(r"float\*\s+(\w+);", body)
    assert fields == [n for n, _ in _lib.NrAggParams._fields_] == ["rows", "neuray_weights", "geometry_weights", "blend_weights"]
    for name in ("nr_render_pass_fwd_agg", "nr_render_pass_fwd_tf32_agg"):
        assert re.search(rf"int {name}\(const NrPassParams\* p, const NrAggParams\* a, void\* stream\);", src), name
        assert name in _lib.SIGNATURES


def test_abi_version_matches_the_header():
    src = open(os.path.join(ROOT, "include", "neuray_b200.h")).read()
    assert int(re.search(r"#define NR_ABI_VERSION (\d+)", src).group(1)) == _lib.ABI_VERSION == 13


def test_export_kernels_issue_whole_batches(sass):  # noqa: F811
    """The point kernel with the blend and pooling-weight exports (point_kernel_agg<G, NP>: both precisions, every lane
    group) keeps the wgmma batch structure of the kernels without them."""
    names = [n for n in sass if "point_kernel_agg" in n]
    assert len(names) == 14, names
    for n in names:
        lines = sass[n]
        hgmma = [ln for ln in lines if "HGMMA" in ln]
        assert hgmma and (len(lines) - len(hgmma)) * 2 <= len(hgmma), n
        for i, batch in enumerate(_batches(lines)):
            gsb = [j for j, ln in enumerate(batch) if "gsb0" in ln.split(";")[0]]
            assert len(batch) >= 2 and gsb == [len(batch) - 1], (n, i, len(batch), gsb)
