"""CPU: where each working view puts the surface along a pixel's ray (cfg render_view_depth):
view_hit_nr[r, v] = Σ_d hit_v[r, d] and view_depth_nr[r, v] = Σ_d hit_v[r, d] · que_depth[r, d], hit_v the reference's
masked prj_dict['hit_prob'] of the pass (renderer.py:75-82).

  * the oracle's prj_hit_prob (neuray_oracle.render_by_depth's keep), in fp32 and fp64, against the unmodified
    reference's, stored in tests/golden/view_depth.npz (oracle/gen_golden_view_depth.py), for both passes;
  * the contract: view_depth lies in [near · view_hit, far · view_hit], and a view that sees none of a ray's samples has
    exactly 0 in both;
  * the binding: the two entry points and NrViewParams match the header, and the ABI version is still 13;
  * the SASS of the built library: the view-export kernels issue their wgmma in whole batches."""
import json
import os
import re

import numpy as np
import pytest
import torch

import gen_golden_view_depth as ggd
import gen_golden_visibility as ggv
import neuray_oracle as orc
from gen_golden import flat_cfg
from neuray_b200 import _lib
from test_agg_weights_cpu import f64
from test_point_kernel_sass import _batches, sass  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "view_depth.npz")
CASES = tuple(ggd.CASES)
# max |oracle - reference| of prj_hit_prob over every case and pass: 1.2e-7 in fp32 (the reference's own precision),
# 2.1e-7 in fp64 (the reference's fp32 rounding through the dist decoder); the bounds leave about 4x of headroom
TOL = {torch.float32: 5e-7, torch.float64: 1e-6}


def view_sums(hit, depth):
    """hit [rfn, qn, rn, dn, 1] (prj layout), depth [qn, rn, dn] -> (Σ_d hit, Σ_d hit · depth) [qn, rn, rfn] each, in the
    dtype of the inputs."""
    h = hit[..., 0]
    return h.sum(-1).permute(1, 2, 0), (h * depth[None]).sum(-1).permute(1, 2, 0)


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
    otherwise: (keep, outputs, depths)."""
    oc = flat_cfg(cfg)
    depth = fine_depth if is_fine else orc.sample_depth(que["depth_range"], que["coords"], oc["depth_sample_num"])[0]
    cast = f64 if dtype == torch.float64 else (lambda d: d)
    keep = {}
    with torch.no_grad():
        out = orc.render_by_depth(cast(W), oc, depth.to(dtype), cast(que), cast(ref), False, is_fine, keep)
    return keep, out, depth.to(dtype)


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("is_fine", [False, True])
def test_oracle_matches_reference(name, is_fine):
    """Run in fp32, the reference's own precision, the oracle's masked hit probabilities equal the reference's within
    5e-7.  In fp64 they differ from the reference by its own fp32 rounding through the dist decoder, within 1e-6."""
    cfg, que, ref, W, gold = load_case(name)
    sfx = "_fine" if is_fine else ""
    for dtype in (torch.float32, torch.float64):
        keep, out, _ = oracle_pass(cfg, W, que, ref, is_fine, gold["que_depth_fine"], dtype)
        assert torch.equal(keep["prj_mask"].float(), gold["prj_mask" + sfx])
        err = float((keep["prj_hit_prob"].double() - gold["prj_hit_prob" + sfx].double()).abs().max())
        print(f"{name}{sfx} prj_hit_prob {dtype}: max |oracle - reference| {err:.2e}")
        assert err <= TOL[dtype], (dtype, err)
        torch.testing.assert_close(out["hit_prob_nr"].float(), gold["hit_prob_nr" + sfx], atol=1e-4, rtol=1e-3)


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("is_fine", [False, True])
def test_view_depth_lies_between_near_and_far_times_view_hit(name, is_fine):
    """Every sample depth lies in the query's [near, far], and hit_v >= 0, so near · view_hit <= view_depth <= far ·
    view_hit: view_depth / view_hit is a depth inside the query's range.  In the fp64 oracle and in the reference's fp32
    golden."""
    cfg, que, ref, W, gold = load_case(name)
    sfx = "_fine" if is_fine else ""
    keep, _, depth = oracle_pass(cfg, W, que, ref, is_fine, gold["que_depth_fine"])
    near, far = (float(x) for x in que["depth_range"][0])
    assert float(depth.min()) >= near * (1 - 1e-6) and float(depth.max()) <= far * (1 + 1e-6)
    for hit, d in ((keep["prj_hit_prob"], depth), (gold["prj_hit_prob" + sfx].double(), depth)):
        assert bool((hit >= 0).all())
        vh, vd = view_sums(hit, d)
        assert bool((vd >= near * vh * (1 - 1e-6)).all()) and bool((vd <= far * vh * (1 + 1e-6)).all())
        assert float(vh.max()) > 0


@pytest.mark.parametrize("is_fine", [False, True])
def test_a_view_that_sees_none_of_a_rays_samples_gives_zero(is_fine):
    """hit_v carries the projection mask, so a view with no valid sample on a ray adds exactly 0 to both sums, in the
    oracle and in the reference."""
    cfg, que, ref, W, gold = load_case("v5_unseen")
    sfx = "_fine" if is_fine else ""
    keep, _, depth = oracle_pass(cfg, W, que, ref, is_fine, gold["que_depth_fine"])
    blind = keep["prj_mask"][..., 0].sum(-1) == 0                                   # [rfn,qn,rn]: the view sees no sample
    assert int(blind.sum()) > 0
    for hit in (keep["prj_hit_prob"], gold["prj_hit_prob" + sfx].double()):
        for s in view_sums(hit, depth):
            assert bool((s[blind.permute(1, 2, 0)] == 0).all())


def test_view_hit_follows_the_references_bins():
    """The reference's definition, which the outputs reproduce: each bin is centred on the sample's inverse depth in the
    view's own range but is as wide as the query's interval, and the last interval is 1e6.  So a view whose surface lies
    beyond the last sample puts all its mass on that sample (it reads as far), and a view that sees the ray end-on, its
    samples crowded in its own inverse depth, has overlapping bins and Σ_d hit_v above 1."""
    depth = torch.tensor([[[2.0, 3.0, 4.0]]], dtype=torch.float64)
    rng = torch.tensor([[1.0, 5.0]], dtype=torch.float64)
    dists = orc.depth2inv_dists(depth, rng)
    assert float(dists[..., -1]) == 1e6
    mean = torch.full((1, 1, 1, 3, 2), 3.0, dtype=torch.float64)                 # beyond far (t = 1) in the view's range
    var = torch.full((1, 1, 1, 3, 2), 20.0, dtype=torch.float64)
    vis, aw = torch.zeros(1, 1, 1, 3, 2, dtype=torch.float64), torch.full((1, 1, 1, 3, 1), 0.5, dtype=torch.float64)
    _, _, hit = orc.compute_prob(depth[None], dists[None], mean, var, vis, aw, True, rng, False)
    vh, vd = view_sums(hit[..., None], depth)
    print(f"surface beyond the last sample: hit {hit.flatten().tolist()}, view_depth / view_hit {float(vd / vh):.4f}")
    assert float(hit[..., :2].max()) < 1e-12 and abs(float(vh) - 1) < 1e-12 and abs(float(vd / vh) - 4.0) < 1e-9
    mean = torch.full((1, 1, 1, 3, 2), 0.95, dtype=torch.float64)
    crowded = torch.tensor([[[[4.4, 4.5, 4.6]]]], dtype=torch.float64)           # the view's depths of the three samples
    _, _, hit = orc.compute_prob(crowded, dists[None], mean, var, vis, aw, True, rng, False)
    print(f"samples crowded in the view: Σ_d hit_v {float(hit.sum()):.3f}")
    assert float(hit.sum()) > 1.0


def test_entry_points_and_params_match_the_header():
    src = open(os.path.join(ROOT, "include", "neuray_b200.h")).read()
    body = re.search(r"typedef struct NrViewParams \{(.*?)\} NrViewParams;", src, re.S).group(1)
    fields = re.findall(r"float\*\s+(\w+);", body)
    assert fields == [n for n, _ in _lib.NrViewParams._fields_] == ["rows", "view_hit", "view_depth", "blend_weights",
                                                                    "neuray_weights", "geometry_weights"]
    for name in ("nr_render_pass_fwd_view", "nr_render_pass_fwd_tf32_view"):
        assert re.search(rf"int {name}\(const NrPassParams\* p, const NrViewParams\* w, void\* stream\);", src), name
        assert name in _lib.SIGNATURES


def test_abi_version_is_still_13():
    src = open(os.path.join(ROOT, "include", "neuray_b200.h")).read()
    assert int(re.search(r"#define NR_ABI_VERSION (\d+)", src).group(1)) == _lib.ABI_VERSION == 13


def test_output_names_survive_the_eval_chunk_loop():
    """The chunk loop drops keys that start with hit_prob in eval; the two outputs must not."""
    from neuray_b200 import renderer
    keys = [key for switch, _, key in renderer._OPTIONAL_OUTPUTS if switch == "render_view_depth"]
    assert keys == ["view_hit_nr", "view_depth_nr"]
    assert not any(k.startswith("hit_prob") for k in keys)
    assert renderer.base_cfg["render_view_depth"] is False


def test_view_kernels_issue_whole_batches(sass):  # noqa: F811
    """The point kernel with the hit-row export (point_kernel_view<G, NP>: both precisions, every lane group) keeps the
    wgmma batch structure of the kernels without it."""
    names = [n for n in sass if "point_kernel_view" in n]
    assert len(names) == 14, names
    for n in names:
        lines = sass[n]
        hgmma = [ln for ln in lines if "HGMMA" in ln]
        assert hgmma and (len(lines) - len(hgmma)) * 2 <= len(hgmma), n
        for i, batch in enumerate(_batches(lines)):
            gsb = [j for j, ln in enumerate(batch) if "gsb0" in ln.split(";")[0]]
            assert len(batch) >= 2 and gsb == [len(batch) - 1], (n, i, len(batch), gsb)
