"""CPU: the per-view colour-blend weight output (cfg render_blend_weights, blend_weights_nr[r, v] = Σ_d hit_nr[r, d] · w[v, r, d],
w the reference's blending_weights_valid, ibrnet.py:362-366).

  * the oracle's blend weights (the softmax over the views of ibrnet_forward, recorded by render_by_depth_with_blend), in
    fp32 and fp64, against the unmodified reference's, stored in tests/golden/blend_weights.npz (oracle/gen_golden_blend.py),
    for both passes;
  * what the weights are: they sum to 1 over the views, blending the views' colours with them gives the oracle's NR
    colours, and a point that no view sees gets 1/rfn from every view;
  * the binding: the two entry points and NrBlendParams match the header;
  * the SASS of the built library: the export kernels issue their wgmma in whole batches."""
import json
import os
import re

import numpy as np
import pytest
import torch

import gen_golden_blend as ggb
import gen_golden_visibility as ggv
import neuray_oracle as orc
from gen_golden import flat_cfg
from neuray_b200 import _lib
from test_point_kernel_sass import _batches, sass  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "blend_weights.npz")
CASES = tuple(ggb.CASES)


def f64(d):
    return {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in d.items()}


class _SoftmaxRecorder:
    """Stands in for the oracle module's `torch`: every attribute is torch's, and softmax over dim 2 (ibrnet_forward's colour
    blend, ibrnet.py:362-366; its ray attention takes the softmax over dim -1) is also appended to `seen`."""

    def __init__(self, seen):
        self.seen = seen

    def __getattr__(self, name):
        return getattr(torch, name)

    def softmax(self, x, dim=None, **kw):
        y = torch.softmax(x, dim, **kw)
        if dim == 2:
            self.seen.append(y)
        return y


def render_by_depth_with_blend(W, cfg, que_depth, que, ref, is_train, is_fine, keep):
    """neuray_oracle.render_by_depth(..., keep) that also leaves the oracle's colour-blend weights in keep["blend"], in the
    layout of its prj fields: [rfn, qn, rn, dn, 1].  The oracle forms them and only returns their blend of the colours."""
    seen = []
    own = orc.torch
    orc.torch = _SoftmaxRecorder(seen)
    try:
        out = orc.render_by_depth(W, cfg, que_depth, que, ref, is_train, is_fine, keep)
    finally:
        orc.torch = own
    assert len(seen) == 1, len(seen)
    rfn, qn, rn, dn, _ = keep["prj_mask"].shape
    keep["blend"] = seen[0].permute(2, 0, 1, 3).reshape(rfn, qn, rn, dn, 1)       # [qn*rn, dn, rfn, 1] -> prj layout
    return out


def oracle_blend_weights(keep, hit):
    """Σ_d hit[q, r, d] · blend[v, q, r, d] -> [qn, rn, rfn], in the dtype of the inputs."""
    return (keep["blend"][..., 0] * hit[None]).sum(-1).permute(1, 2, 0)


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
        out = render_by_depth_with_blend(cast(W), oc, depth.to(dtype), cast(que), cast(ref), False, is_fine, keep)
    return keep, out


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("is_fine", [False, True])
def test_oracle_matches_reference(name, is_fine):
    """Run in fp32, the reference's own precision, the oracle's blend weights equal the reference's within 1e-6 (measured:
    at most 7.8e-7).  In fp64 they differ from the reference by its own fp32 rounding through the aggregation net
    (measured: at most 4.6e-6)."""
    cfg, que, ref, W, gold = load_case(name)
    sfx = "_fine" if is_fine else ""
    # the reference's [rn, dn, rfn, 1] in the oracle's layout of prj fields [rfn, 1, rn, dn, 1]
    want = gold["blend" + sfx].permute(2, 0, 1, 3)[:, None].double()
    for dtype, tol in ((torch.float32, 1e-6), (torch.float64, 1e-5)):
        keep, out = oracle_pass(cfg, W, que, ref, is_fine, gold["que_depth_fine"], dtype)
        assert torch.equal(keep["prj_mask"].float(), gold["prj_mask" + sfx])
        err = float((keep["blend"].double() - want).abs().max())
        print(f"{name}{sfx} {dtype}: max |oracle - reference| {err:.2e}")
        assert err <= tol, (dtype, err)
        torch.testing.assert_close(out["hit_prob_nr"].float(), gold["hit_prob_nr" + sfx], atol=1e-4, rtol=1e-3)


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("is_fine", [False, True])
def test_weights_sum_to_one_and_blend_the_nr_colour(name, is_fine):
    cfg, que, ref, W, gold = load_case(name)
    keep, out = oracle_pass(cfg, W, que, ref, is_fine, gold["que_depth_fine"])
    w = keep["blend"]                                                        # [rfn,qn,rn,dn,1]
    torch.testing.assert_close(w.sum(0), torch.ones_like(w[0]), atol=1e-12, rtol=0)
    colors = (w * keep["prj_rgb"]).sum(0)                                    # [qn,rn,dn,3]
    torch.testing.assert_close(colors, keep["colors"], atol=1e-12, rtol=0)
    hit = out["hit_prob_nr"]
    torch.testing.assert_close((hit[..., None] * colors).sum(2), out["pixel_colors_nr"], atol=1e-12, rtol=0)
    # unnormalised like render_depth: Σ_v B = Σ_d hit
    torch.testing.assert_close(oracle_blend_weights(keep, hit).sum(-1), hit.sum(-1), atol=1e-12, rtol=0)


@pytest.mark.parametrize("is_fine", [False, True])
def test_a_point_no_view_sees_gets_one_over_rfn(is_fine):
    cfg, que, ref, W, gold = load_case("v5_unseen")
    keep, _ = oracle_pass(cfg, W, que, ref, is_fine, gold["que_depth_fine"])
    unseen = keep["prj_mask"][..., 0].sum(0) == 0                            # [qn,rn,dn]
    assert int(unseen.sum()) > 0
    rfn = keep["blend"].shape[0]
    for w in (keep["blend"][..., 0], gold["blend" + ("_fine" if is_fine else "")][..., 0].permute(2, 0, 1)[:, None]):
        assert torch.equal(w[:, unseen].float(), torch.full((rfn, int(unseen.sum())), 1.0 / rfn))


def test_entry_points_and_params_match_the_header():
    src = open(os.path.join(ROOT, "include", "neuray_b200.h")).read()
    body = re.search(r"typedef struct NrBlendParams \{(.*?)\} NrBlendParams;", src, re.S).group(1)
    fields = re.findall(r"float\*\s+(\w+);", body)
    assert fields == [n for n, _ in _lib.NrBlendParams._fields_] == ["row_blend", "blend_weights"]
    for name in ("nr_render_pass_fwd_blend", "nr_render_pass_fwd_tf32_blend"):
        assert re.search(rf"int {name}\(const NrPassParams\* p, const NrBlendParams\* b, void\* stream\);", src), name
        assert name in _lib.SIGNATURES
    assert int(re.search(r"#define NR_ABI_VERSION (\d+)", src).group(1)) == _lib.ABI_VERSION


def test_export_kernels_issue_whole_batches(sass):  # noqa: F811
    """The point kernel with the blend export (point_kernel_blend<G, NP>: both precisions, every lane group) keeps the
    wgmma batch structure of the kernels without it."""
    names = [n for n in sass if "point_kernel_blend" in n]
    assert len(names) == 14, names
    for n in names:
        lines = sass[n]
        hgmma = [ln for ln in lines if "HGMMA" in ln]
        assert hgmma and (len(lines) - len(hgmma)) * 2 <= len(hgmma), n
        for i, batch in enumerate(_batches(lines)):
            gsb = [j for j, ln in enumerate(batch) if "gsb0" in ln.split(";")[0]]
            assert len(batch) >= 2 and gsb == [len(batch) - 1], (n, i, len(batch), gsb)
