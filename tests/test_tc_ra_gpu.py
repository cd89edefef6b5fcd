"""GPU: the register-A wgmma primitive (tc::wgmma_tf32_ra, A fragments in registers, W in swizzled smem, 3xTF32) against
fp64 matmul, at the two output widths the point kernel uses it at."""
import pytest
import torch

from neuray_b200 import _lib

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,k", [(32, 32), (16, 64)])
def test_tc_layer_a_from_registers(n, k):
    torch.manual_seed(n * 100 + k + 2)
    A = torch.randn(128, k, device="cuda")
    W = torch.randn(n, k, device="cuda") * 0.3
    D = torch.full((128, n), float("nan"), device="cuda")
    _lib.check(_lib.lib().nr_tc_selftest(A.data_ptr(), W.data_ptr(), D.data_ptr(), n, k, 2, None), "selftest")
    torch.cuda.synchronize()
    ref = (A.double() @ W.double().t())
    err = (D.double() - ref).abs().max().item()
    print(f"n={n} k={k} A from registers: max abs err {err:.3e} (|ref| max {ref.abs().max().item():.2f})")
    assert err < 2e-5, err
    # the same products in the same order as with A in shared memory: the accumulators agree bit for bit
    Ds = torch.full_like(D, float("nan"))
    _lib.check(_lib.lib().nr_tc_selftest(A.data_ptr(), W.data_ptr(), Ds.data_ptr(), n, k, 1, None), "selftest")
    torch.cuda.synchronize()
    assert torch.equal(D, Ds)
