"""GPU: the wgmma layer primitive (A in the shared-memory activation tile, W in swizzled smem, fp32 accumulate) against fp64 matmul."""
import pytest
import torch

from neuray_b200 import _lib

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,k", [(32, 32), (64, 64), (16, 64)])
@pytest.mark.parametrize("mode", [0, 1])
def test_tc_layer(n, k, mode):
    torch.manual_seed(n * 100 + k + mode)
    A = torch.randn(128, k, device="cuda")
    W = torch.randn(n, k, device="cuda") * 0.3
    D = torch.full((128, n), float("nan"), device="cuda")
    _lib.check(_lib.lib().nr_tc_selftest(A.data_ptr(), W.data_ptr(), D.data_ptr(), n, k, mode, None), "selftest")
    torch.cuda.synchronize()
    ref = (A.double() @ W.double().t())
    err = (D.double() - ref).abs().max().item()
    print(f"n={n} k={k} mode={mode}: max abs err {err:.3e} (|ref| max {ref.abs().max().item():.2f})")
    assert err < (2e-2 if mode == 0 else 2e-5), err
