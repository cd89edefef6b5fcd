"""GPU: nr_tape_gemms (csrc/nr_tape_gemm.cu) on its own, the weight-gradient GEMMs dW = dz x^T of the training backward.

The tapes are [tiles, slots, 128] as nr_render_pass_bwd writes them.  Every padding row (index >= M in the last tile) and
every slot that no descriptor reads holds NaN, so a read of anything the kernel should not touch poisons the result.

* exact: integer-valued tapes (x in {0, 1, 2}, dz in {-3 .. 3}).  Every product and partial sum is an integer below 2^24,
  exact in the TF32 hi/lo split and in fp32 atomics, so the result must equal the fp64 reference bit for bit: a dropped,
  duplicated or shifted row, chunk, half tile or slot fails however large K is.
* accuracy: N(0,1) tapes and their absolute values, against the fp64 product, elementwise relative to B = |dz| |x|^T.
* row counts that end in both halves of a 128-row tile (the partial-chunk branch), layers with more CTAs than chunks,
  and K = 262 144 (+ 77), the training shape.
"""
import ctypes as C
import itertools

import pytest
import torch

from neuray_b200 import _lib, backward, renderer

pytestmark = pytest.mark.gpu

NAN = float("nan")
SENTINEL = 7.0          # fills the gaps between the output blocks: the kernel must never write there
GAP = 5
NOUT = (1, 2, 8, 15, 16, 17, 33, 35, 64)
NIN = (1, 4, 7, 8, 9, 16, 32, 67, 140)
# (rows, points): every count of the set on both tapes; 63/65 and 127/129/191 end in the first and second half of a tile
COUNTS = [(1, 63), (5, 64), (63, 1000), (64, 5), (65, 127), (127, 129), (128, 191), (129, 192), (191, 65), (192, 128),
          (1000, 1), (9216, 1000), (262144, 9216), (262144 + 77, 192), (0, 129), (129, 0)]


def slot_counts():
    return [_lib.bwd_slot(n) for n in ("R_SLOTS", "G_SLOTS", "P_SLOTS", "GP_SLOTS")]


def synthetic_layers():
    """Every (n_out, n_in) of NOUT x NIN (81 layers: ksplit 1, 2, 4 and 8, up to the 64 x 141 maximum), alternately on the
    row and the point tapes, at slot offsets that vary the alignment."""
    S = slot_counts()
    out = []
    for i, (no, ni) in enumerate(itertools.product(NOUT, NIN)):
        xt, gt = (2, 3) if i % 2 else (0, 1)
        out.append((gt, (53 * i + 11) % (S[gt] - no + 1), no, xt, (37 * i) % (S[xt] - ni + 1), ni))
    return out


def real_table(n_heads):
    net = renderer.NeuralRayRenderPath({"dist_decoder_cfg": {"use_vis": True}})
    names = [k for k, _ in net.named_parameters() if k.startswith(("dist_decoder.", "agg_net."))]
    return names, backward.layer_table(names, "dist_decoder", "agg_net", n_heads)


def make_tapes(layers, rows, points, kind, seed):
    """Four NaN tapes; the slots the layers read get values over their first M rows.  kind: int / normal / nonneg."""
    S = slot_counts()
    count = (rows, rows, points, points)
    read = [set() for _ in range(4)]
    for gt, gs, no, xt, xs, ni, *_ in layers:
        read[gt].update(range(gs, gs + no))
        read[xt].update(range(xs, xs + ni))
    gen = torch.Generator(device="cuda").manual_seed(seed)
    tapes = []
    for tp in range(4):
        m = count[tp]
        tiles = max(1, (m + 127) // 128)          # one tile at least: a zero-row tape is still a valid pointer
        buf = torch.full((tiles, S[tp], 128), NAN, device="cuda")
        slots = sorted(read[tp])
        for j in range(0, len(slots), 64):
            sl = torch.tensor(slots[j:j + 64], device="cuda")
            n = sl.numel()
            if kind == "int":
                v = torch.randint(0, 3, (n, m), generator=gen, device="cuda") if tp in (0, 2) else \
                    torch.randint(-3, 4, (n, m), generator=gen, device="cuda")
                v = v.float()
            else:
                v = torch.randn(n, m, generator=gen, device="cuda")
                if kind == "nonneg":
                    v = v.abs()
            pad = torch.full((n, tiles * 128), NAN, device="cuda")
            pad[:, :m] = v
            buf[:, sl, :] = pad.view(n, tiles, 128).permute(1, 0, 2)
        tapes.append(buf)
    return tapes


def layout(layers):
    """Output offsets with a GAP-float sentinel gap before every block."""
    offs, off = [], GAP
    for gt, gs, no, xt, xs, ni, *_ in layers:
        offs.append(off)
        off += no * (ni + 1) + GAP
    return offs, off


def launch(layers, offs, tapes, rows, points, out, n_desc=None):
    arr = (_lib.NrGemmDesc * max(1, len(layers)))()
    for i, ((gt, gs, no, xt, xs, ni, *_), o) in enumerate(zip(layers, offs)):
        arr[i].g_tape, arr[i].g_slot, arr[i].n_out, arr[i].x_tape, arr[i].x_slot, arr[i].n_in, arr[i].out_off = gt, gs, no, xt, xs, ni, o
    p = [None if t is None else t.data_ptr() for t in tapes]
    rc = _lib.lib().nr_tape_gemms(arr, len(layers) if n_desc is None else n_desc, p[0], p[1], rows, p[2], p[3], points,
                                  out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc


def reference(layers, tapes, rows, points):
    """fp64 [n_out, n_in + 1] blocks (dW | db) and their bounds B = |dz| |x|^T (| sum |dz|)."""
    count = (rows, rows, points, points)
    blocks, bounds = [], []
    for gt, gs, no, xt, xs, ni, *_ in layers:
        dz = backward._slots(tapes[gt], gs, no, count[gt]).double()
        x = backward._slots(tapes[xt], xs, ni, count[xt]).double()
        blocks.append(torch.cat([dz @ x.t(), dz.sum(1, keepdim=True)], 1))
        bounds.append(torch.cat([dz.abs() @ x.abs().t(), dz.abs().sum(1, keepdim=True)], 1))
    return blocks, bounds


def run(layers, rows, points, kind, seed, out_init=0.0):
    """-> (blocks the kernel added to out, fp64 blocks, bounds); checks the sentinel gaps."""
    tapes = make_tapes(layers, rows, points, kind, seed)
    offs, total = layout(layers)
    out = torch.full((total,), SENTINEL, device="cuda")
    for (gt, gs, no, xt, xs, ni, *_), o in zip(layers, offs):
        out[o:o + no * (ni + 1)] = out_init
    assert launch(layers, offs, tapes, rows, points, out) == 0, _lib.lib().nr_last_error()
    blocks, bounds = reference(layers, tapes, rows, points)
    got = [out[o:o + b.numel()].view(b.shape) for o, b in zip(offs, blocks)]
    gaps = torch.ones(total, dtype=torch.bool, device="cuda")
    for o, b in zip(offs, blocks):
        gaps[o:o + b.numel()] = False
    assert bool((out[gaps] == SENTINEL).all()), "nr_tape_gemms wrote outside its output blocks"
    return got, blocks, bounds


def check_exact(layers, rows, points, seed, out_init=0.0):
    got, blocks, _ = run(layers, rows, points, "int", seed, out_init)
    bad = [(i, layers[i][:6], float((g.double() - out_init - b).abs().max())) for i, (g, b) in enumerate(zip(got, blocks))
           if not torch.equal(g.double(), b + out_init)]
    assert not bad, f"rows={rows} points={points}: {len(bad)} layers not exact, first {bad[:4]}"


# A 3xTF32 product with the truncating split is good to about 3 * 2^-20 of |dz||x|; the fp32 accumulation in the MMA
# accumulators adds at most (additions per accumulator) * 2^-24 of B.  Each 64-row chunk goes through at most 24 MMA
# accumulations before it is added to the running fp32 sum; measured on H100: worst max(err/B) 2.4e-6 (non-negative
# tapes, K = 262 221), 2.3e-4 when the whole CTA range went through the MMA accumulators.
ACC_GATE = 1e-5
WORST = {}


def check_accuracy(layers, rows, points, kind, seed, label):
    got, blocks, bounds = run(layers, rows, points, kind, seed)
    worst, where = 0.0, None
    for i, (g, b, B) in enumerate(zip(got, blocks, bounds)):
        assert bool(torch.isfinite(g).all()), (label, layers[i][:6], "non-finite output")
        err = (g.double() - b).abs()
        assert bool((err[B == 0] == 0).all()), (label, layers[i][:6])
        r = float((err / B.clamp_min(1e-300)).max())
        if r > worst:
            worst, where = r, layers[i][:6]
    WORST[label] = worst
    print(f"tape_gemm {label}: max(err/B) = {worst:.3e} at layer {where}")
    assert worst <= ACC_GATE, (label, worst, where)


@pytest.mark.parametrize("rows,points", COUNTS)
def test_exact_integer_tapes(rows, points):
    """81 synthetic layers in a 48-descriptor and a 33-descriptor launch, bit-exact against fp64."""
    layers = synthetic_layers()
    for part, seed in ((layers[:48], 1), (layers[48:], 2)):
        check_exact(part, rows, points, seed + rows)


@pytest.mark.parametrize("rows,points", COUNTS)
@pytest.mark.parametrize("kind", ["normal", "nonneg"])
def test_accuracy_against_fp64(rows, points, kind):
    if rows == 0 and points == 0:
        pytest.skip("nothing to multiply")
    layers = synthetic_layers()
    for j, part in enumerate((layers[:48], layers[48:])):
        check_accuracy(part, rows, points, kind, 10 + j, f"synthetic[{j}] {kind} rows={rows} points={points}")


@pytest.mark.parametrize("n_heads", [3, 4])
@pytest.mark.parametrize("rfn,points", [(8, 32768), (5, 407), (3, 35)])
def test_real_layer_table(n_heads, rfn, points):
    """The layers of a pass (backward.layer_table: 34 with three decoder heads, 37 with four) at the training shape
    (8 views x 32 768 points = 262 144 rows) and at ragged sizes: exact on integer tapes and accurate on N(0,1) tapes."""
    _, table = real_table(n_heads)
    assert len(table) == (34 if n_heads == 3 else 37)
    check_exact(table, rfn * points, points, 3)
    for kind in ("normal", "nonneg"):
        check_accuracy(table, rfn * points, points, kind, 4, f"layer_table h{n_heads} {kind} rows={rfn * points} points={points}")


@pytest.mark.parametrize("n_heads", [3, 4])
def test_fused_matches_torch_assembly(n_heads):
    """assemble_param_grads_fused (one nr_tape_gemms launch, then _finish) against assemble_param_grads over the same tapes
    in fp64: covers the LayerNorm diagonal and the base_fc.0 weight assembled from its pooled and per-row halves."""
    names, table = real_table(n_heads)
    rows, points = 5 * 407, 407
    tapes = make_tapes(table, rows, points, "normal", 5)
    fused = backward.assemble_param_grads_fused(names, "dist_decoder", "agg_net", n_heads, *tapes, rows, points,
                                                torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ref = backward.assemble_param_grads(names, "dist_decoder", "agg_net", n_heads, *[t.double() for t in tapes], rows, points)
    bound = backward.assemble_param_grads(names, "dist_decoder", "agg_net", n_heads, *[t.double().abs() for t in tapes], rows, points)
    checked = 0
    for k in names:
        if ref[k] is None:
            assert fused[k] is None, k
            continue
        assert fused[k].shape == ref[k].shape, k
        err = (fused[k].double() - ref[k]).abs()
        assert bool((err <= ACC_GATE * bound[k]).all()), (k, float((err / bound[k]).max()))
        checked += 1
    assert checked == len([k for k in names if ref[k] is not None]) and checked > 60


def test_out_is_accumulated():
    """out is added to: a pre-filled out comes back as the old value plus the gradient (exactly, on integer tapes)."""
    layers = synthetic_layers()[:48]
    check_exact(layers, 1000, 129, 6, out_init=-250.0)


def test_zero_rows_leave_out_unchanged():
    layers = synthetic_layers()[:48]
    tapes = make_tapes(layers, 0, 0, "int", 7)
    offs, total = layout(layers)
    out = torch.randn(total, device="cuda")
    before = out.clone()
    assert launch(layers, offs, tapes, 0, 0, out) == 0
    assert torch.equal(out, before)


def _bad_cases():
    ok = (1, 3, 16, 0, 5, 16)
    return {
        "n_desc 0": ([ok], 0, None),
        "n_desc 49": ([ok] * 49, None, None),
        "n_out 65": ([(1, 3, 65, 0, 5, 16)], None, None),
        "n_out 0": ([(1, 3, 0, 0, 5, 16)], None, None),
        "n_in 141": ([(1, 3, 16, 0, 5, 141)], None, None),
        "n_in 0": ([(1, 3, 16, 0, 5, 0)], None, None),
        "x tape 4": ([(1, 3, 16, 4, 5, 16)], None, None),
        "dz tape 4": ([(4, 3, 16, 0, 5, 16)], None, None),
        "dz tape -1": ([(-1, 3, 16, 0, 5, 16)], None, None),
        "null tape": ([ok], None, 2),
        "row x with point dz": ([(3, 3, 16, 0, 5, 16)], None, None),
        "point x with row dz": ([(1, 3, 16, 2, 5, 16)], None, None),
        "negative out_off": ([ok], None, None, -1),
    }


@pytest.mark.parametrize("case", list(_bad_cases()))
def test_bad_arguments_are_rejected(case):
    """NR_E_INVALID and out untouched; nothing is launched for such a descriptor."""
    layers, n_desc, null_tape, *neg = _bad_cases()[case]
    good = [(1, 3, 16, 0, 5, 16)]
    tapes = make_tapes(good, 300, 70, "int", 8)
    if null_tape is not None:
        tapes[null_tape] = None
    out = torch.randn(4096, device="cuda")
    before = out.clone()
    offs = [neg[0] if neg else 0] * len(layers)
    assert launch(layers, offs, tapes, 300, 70, out, n_desc=n_desc) == -1       # NR_E_INVALID
    assert torch.equal(out, before)
