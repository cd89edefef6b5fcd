"""CPU: what colour each working view puts into a pixel (cfg render_view_colors): view_colors_nr[r, v] = Σ_d hit_nr[r, d] ·
w[v, r, d] · rgb_v[r, d], w the reference's blending_weights_valid (ibrnet.py:362-366) and rgb_v its masked
prj_dict['rgb'] (render_ops.py:132-139).

  * the oracle's per-view colours (its prj_rgb times the blend weights that render_by_depth_with_blend records), in fp32
    and fp64, against the unmodified reference's, formed from the per-view colour terms rgb_in * blending_weights_valid
    stored in tests/golden/view_colors.npz (oracle/gen_golden_view_colors.py), for both passes;
  * the contract: Σ_v view_colors equals the reference's pixel_colors_nr, and a view that sees none of a ray's samples
    gives exactly 0;
  * the binding: nr_view_colors and NrColorParams match the header, and the ABI version is still 13;
  * dist.render_sharded carries a [1, rn, rfn, 3] output bit for bit."""
import json
import os
import re
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import gen_golden_view_colors as ggc
import gen_golden_visibility as ggv
from neuray_b200 import _lib
from neuray_b200 import dist as nrd
from test_blend_weights_cpu import oracle_pass

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "view_colors.npz")
CASES = tuple(ggc.CASES)
# max |oracle - reference| of view_colors over every case and pass (colours up to 0.92): 1.2e-6 in fp32, 1.7e-5 in fp64
# (the reference's fp32 rounding through the aggregation net and the compositing weights); the bounds leave about 2.5x
# of headroom
TOL = {torch.float32: 3e-6, torch.float64: 4e-5}


def oracle_view_colors(keep, hit):
    """Σ_d hit[q, r, d] · blend[v, q, r, d] · prj_rgb[v, q, r, d, :] -> [qn, rn, rfn, 3], in the dtype of the inputs."""
    return (hit[None, ..., None] * keep["blend"] * keep["prj_rgb"]).sum(-2).permute(1, 2, 0, 3)


def reference_view_colors(gold, sfx):
    """The same sum from the reference's own terms: rgb_blend [rn, dn, rfn, 3] and hit_prob_nr [1, rn, dn], in fp64."""
    prod, hit = gold["rgb_blend" + sfx].double(), gold["hit_prob_nr" + sfx].double()
    return (hit[0][:, :, None, None] * prod).sum(1)[None]


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


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("is_fine", [False, True])
def test_oracle_matches_reference(name, is_fine):
    """Run in fp32, the reference's own precision, the oracle's per-view colours equal the reference's within 3e-6.  In
    fp64 they differ from the reference by its own fp32 rounding through the aggregation net, within 4e-5."""
    cfg, que, ref, W, gold = load_case(name)
    sfx = "_fine" if is_fine else ""
    want = reference_view_colors(gold, sfx)
    for dtype in (torch.float32, torch.float64):
        keep, out = oracle_pass(cfg, W, que, ref, is_fine, gold["que_depth_fine"], dtype)
        assert torch.equal(keep["prj_mask"].float(), gold["prj_mask" + sfx])
        err = float((oracle_view_colors(keep, out["hit_prob_nr"]).double() - want).abs().max())
        print(f"{name}{sfx} view_colors {dtype}: max |oracle - reference| {err:.2e}")
        assert err <= TOL[dtype], (dtype, err)


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("is_fine", [False, True])
def test_views_sum_to_the_pixel_colour(name, is_fine):
    """Σ_v view_colors = pixel_colors_nr: in the reference's own terms to its fp32 rounding (the reference sums the views
    first, then the samples; the bound is a few ulps of colours below 1), and in the fp64 oracle to fp64 rounding."""
    cfg, que, ref, W, gold = load_case(name)
    sfx = "_fine" if is_fine else ""
    err = float((reference_view_colors(gold, sfx).sum(2) - gold["pixel_colors_nr" + sfx].double()).abs().max())
    print(f"{name}{sfx}: max |Σ_v C - pixel_colors_nr| in the reference {err:.2e}")
    assert err <= 1e-6
    keep, out = oracle_pass(cfg, W, que, ref, is_fine, gold["que_depth_fine"])
    torch.testing.assert_close(oracle_view_colors(keep, out["hit_prob_nr"]).sum(2), out["pixel_colors_nr"], atol=1e-12, rtol=0)


@pytest.mark.parametrize("is_fine", [False, True])
def test_a_view_that_sees_none_of_a_rays_samples_gives_zero(is_fine):
    """rgb_v carries the projection mask, so a view with no valid sample on a ray adds exactly 0, in the oracle and in the
    reference; this holds although such a view's blend weight is 1/rfn at a point that no view sees."""
    cfg, que, ref, W, gold = load_case("v5_unseen")
    sfx = "_fine" if is_fine else ""
    keep, out = oracle_pass(cfg, W, que, ref, is_fine, gold["que_depth_fine"])
    blind = (keep["prj_mask"][..., 0].sum(-1) == 0).permute(1, 2, 0)                  # [qn,rn,rfn]: the view sees no sample
    assert int(blind.sum()) > 0
    unseen = keep["prj_mask"][..., 0].sum(0) == 0                                       # [qn,rn,dn]: no view sees the point
    assert int(unseen.sum()) > 0 and bool((keep["blend"][:, unseen] > 0).all())
    for c in (oracle_view_colors(keep, out["hit_prob_nr"]), reference_view_colors(gold, sfx)):
        assert bool((c[blind] == 0).all())
        assert float(c.abs().max()) > 0


def test_entry_point_and_params_match_the_header():
    src = open(os.path.join(ROOT, "include", "neuray_b200.h")).read()
    body = re.search(r"typedef struct NrColorParams \{(.*?)\} NrColorParams;", src, re.S).group(1)
    fields = re.findall(r"float\*\s+(\w+);", body)
    assert fields == [n for n, _ in _lib.NrColorParams._fields_] == ["row_blend", "hit_prob", "view_colors"]
    assert re.search(r"int nr_view_colors\(const NrPassParams\* p, const NrColorParams\* c, void\* stream\);", src)
    assert _lib.SIGNATURES["nr_view_colors"][1][1]._type_ is _lib.NrColorParams
    # the blend launch it runs behind with no blend output keeps its struct
    body = re.search(r"typedef struct NrBlendParams \{(.*?)\} NrBlendParams;", src, re.S).group(1)
    assert re.findall(r"float\*\s+(\w+);", body) == [n for n, _ in _lib.NrBlendParams._fields_] == ["row_blend", "blend_weights"]


def test_abi_version_is_still_13():
    src = open(os.path.join(ROOT, "include", "neuray_b200.h")).read()
    assert int(re.search(r"#define NR_ABI_VERSION (\d+)", src).group(1)) == _lib.ABI_VERSION == 13


def test_output_name_survives_the_eval_chunk_loop():
    """The chunk loop drops keys that start with hit_prob in eval; the output must not."""
    from neuray_b200 import renderer
    keys = [key for switch, _, key in renderer._OPTIONAL_OUTPUTS if switch == "render_view_colors"]
    assert keys == ["view_colors_nr"]
    assert renderer.base_cfg["render_view_colors"] is False


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _colour_render(que, ref, is_train):
    """A stand-in for renderer.render with a [1, rn, rfn, 3] output that every bit of the coordinates reaches."""
    c = que["coords"]
    v = torch.arange(5, dtype=torch.float32)
    col = torch.stack([c[..., 0, None] * 0.37 + v, c[..., 1, None] / 7.0 - v, torch.sin(c[..., 0, None] * v)], -1)
    return {"view_colors_nr": col, "pixel_colors_nr": col.sum(2)}


def _worker(rank, world, port, n_rays, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    coords = torch.stack([torch.arange(n_rays, dtype=torch.float32) * 1.3, torch.arange(n_rays, dtype=torch.float32) * 3], -1)[None]
    que = {"coords": coords}
    full = nrd.render_sharded(_colour_render, que, {}, False)
    single = _colour_render(que, {}, False)
    ret[rank] = all(full[k].shape == single[k].shape and torch.equal(full[k], single[k]) for k in single) and \
        full["view_colors_nr"].shape == (1, n_rays, 5, 3)
    dist.destroy_process_group()


@pytest.mark.parametrize("n_rays", [37, 1])
def test_sharded_render_carries_the_per_view_colours_gloo(n_rays):
    """Two ranks over gloo (37 rays: a ragged split; 1 ray: rank 1's shard is empty): the gathered [1, rn, rfn, 3] output
    equals a single render bit for bit."""
    world = 2
    with mp.Manager() as m:
        ret = m.dict()
        mp.spawn(_worker, args=(world, _free_port(), n_rays, ret), nprocs=world, join=True)
        assert dict(ret) == {0: True, 1: True}
