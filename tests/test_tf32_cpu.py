"""CPU: the pieces of the point kernel's TF32 render mode that need no GPU.

  * tf32_rne, the rounding the emulated-TF32 restatement of test_tf32_gpu.py applies to every Linear's input and weight:
    round to nearest, ties to even, at tf32's 10 mantissa bits
  * the SASS of the built library: each of the seven point_kernel_tf32 instantiations issues its wgmma in whole batches
    (one pass per product, so a batch can be as short as its K steps: 2), and the fourteen point_kernel_pm3 ones are
    still there
  * renderer.set_precision takes "fp32" or "tf32" and leaves the encoders' switch alone
"""
import pytest
import torch

from test_point_kernel_sass import _batches, sass  # noqa: F401  (the module's SASS fixture)


def tf32_rne(x):
    """x rounded to the nearest tf32 value (1 + 10 significant bits, fp32's exponent range), ties to even; same dtype.
    Evaluated in fp64, so fp64 inputs are rounded once."""
    m, e = torch.frexp(x.double())                    # x = m 2^e, 0.5 <= |m| < 1: 11 significant bits = round(m 2^11)
    return torch.ldexp(torch.round(m * 2048.0), e - 11).to(x.dtype)


def test_tf32_rne_ties_go_to_even():
    u = 2.0 ** -10                                    # tf32 ulp at 1
    cases = [
        (1.0 + u / 2, 1.0),                           # tie, even neighbour below
        (1.0 + 3 * u / 2, 1.0 + 2 * u),               # tie, even neighbour above
        (1.0 + u / 2 + 2.0 ** -23, 1.0 + u),          # just above a tie
        (1.0 + 3 * u / 2 - 2.0 ** -23, 1.0 + u),      # just below a tie
        (-(1.0 + u / 2), -1.0),
        (-(1.0 + 3 * u / 2), -(1.0 + 2 * u)),
        (2.0 ** -19 * (1.5 + u / 2), 2.0 ** -19 * 1.5),     # tie at another exponent, even neighbour below
        (2.0 ** 19 * (1.5 + 3 * u / 2), 2.0 ** 19 * (1.5 + 2 * u)),
    ]
    x = torch.tensor([c[0] for c in cases], dtype=torch.float32)
    want = torch.tensor([c[1] for c in cases], dtype=torch.float32)
    assert torch.equal(tf32_rne(x), want)


def test_tf32_rne_carries_into_the_exponent():
    u = 2.0 ** -10
    x = torch.tensor([2.0 - u / 2, 2.0 - u / 2 - 2.0 ** -23, -(2.0 - u / 2), 1024.0 * (2.0 - u / 2), 1.0 - u / 4],
                     dtype=torch.float32)
    want = torch.tensor([2.0, 2.0 - u, -2.0, 2048.0, 1.0], dtype=torch.float32)
    assert torch.equal(tf32_rne(x), want)
    assert torch.equal(tf32_rne(torch.tensor([0.0, -0.0, 1.0, 2.0 - u])), torch.tensor([0.0, -0.0, 1.0, 2.0 - u]))


def test_tf32_rne_matches_integer_rounding():
    """On random fp32 values: the classic bit formula, add 0xfff plus the kept lowest bit, clear the 13 low bits."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(100000, generator=g) * torch.exp2(torch.randint(-20, 20, (100000,), generator=g).float())
    b = x.view(torch.int32).long() & 0xffffffff
    r = ((b + 0xfff + ((b >> 13) & 1)) & 0xffffe000)
    want = torch.where(r >= 2 ** 31, r - 2 ** 32, r).to(torch.int32).view(torch.float32)
    assert torch.equal(tf32_rne(x), want)
    assert torch.equal(tf32_rne(x.double()), want.double())


def test_tf32_point_kernels_issue_whole_batches(sass):  # noqa: F811
    tf32 = [n for n in sass if "point_kernel_tf32" in n]
    assert len(tf32) == 7, tf32                     # G in {4, 5, 6, 8, 10, 16, 32}, release only
    assert len([n for n in sass if "point_kernel_pm3" in n]) == 14
    for name in tf32:
        lines = sass[name]
        hgmma = [ln for ln in lines if "HGMMA" in ln]
        depbar = len(lines) - len(hgmma)
        assert hgmma, f"{name}: no HGMMA"
        # the shortest batch is ray_dir_fc.2 (K 16: 2 MMAs); a serialised function has one DEPBAR per HGMMA
        assert depbar * 2 <= len(hgmma), f"{name}: {depbar} WARPGROUP.DEPBAR for {len(hgmma)} HGMMA (wgmma serialised)"
        for i, batch in enumerate(_batches(lines)):
            gsb = [j for j, ln in enumerate(batch) if "gsb0" in ln.split(";")[0]]
            assert len(batch) >= 2 and gsb == [len(batch) - 1], (
                f"{name}: batch {i} has {len(batch)} HGMMA, gsb0 on {gsb} (only the last one may carry it)")


def test_set_precision():
    from neuray_b200 import encoders, renderer
    assert renderer.PRECISION == "fp32" and encoders.PRECISION == "fp32"
    try:
        renderer.set_precision("tf32")
        assert renderer.PRECISION == "tf32" and encoders.PRECISION == "fp32"
        with pytest.raises(ValueError):
            renderer.set_precision("bf16")
        assert renderer.PRECISION == "tf32"
        renderer.set_precision("fp32")
        assert renderer.PRECISION == "fp32"
    finally:
        renderer.set_precision("fp32")
