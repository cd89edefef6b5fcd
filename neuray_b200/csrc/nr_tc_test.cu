// Self-test of the wgmma layer primitive in nr_tc.cuh: D[128 x N] = A[128 x K] * W[N x K]^T with A in the shared-memory
// activation tile, W in shared memory (K-major, 128B swizzle), fp32 accumulators in registers written back into the tile.
// mode 0: single TF32 pass, mode 1: 3xTF32, mode 2: 3xTF32 with A from registers (tc::wgmma_tf32_ra, N = 16 and 32).
// tests/test_tc_gpu.py and tests/test_tc_ra_gpu.py compare against an fp64 reference.
#include "nr_common.cuh"
#include "nr_tc.cuh"

namespace nr {

template <int N, int K, int MODE>
__global__ void __launch_bounds__(128, 1) tc_selftest_kernel(const float* __restrict__ A, const float* __restrict__ W,
                                                           float* __restrict__ D) {
  static_assert(K % 32 == 0 && N % 16 == 0, "shape");
  constexpr int PASSES = MODE == 0 ? 1 : 3;
  constexpr int KS = K / 32;                       // 32-wide K slabs of the B tile
  constexpr int SLAB = N * 32;                     // floats per slab
  constexpr int COLS = 2 * K + 64;                 // activation tile: A_hi K | A_lo K | D N (<= 64)
  __shared__ __align__(1024) float sBhi[KS * SLAB];
  __shared__ __align__(1024) float sBlo[KS * SLAB];
  extern __shared__ __align__(1024) float act[];   // COLS / 32 slabs of 4096 floats
  const int tid = threadIdx.x;
  const int cA_hi = 0, cA_lo = K, cD = 2 * K;

  // weights -> swizzled smem tiles (hi / lo)
  for (int i = tid; i < N * K; i += 128) {
    const int n = i / K, k = i % K;
    uint32_t hi, lo;
    tc::split_tf32(W[i], hi, lo);
    const int idx = (k >> 5) * SLAB + tc::sw128_index(n, k & 31);
    sBhi[idx] = __uint_as_float(hi);
    sBlo[idx] = __uint_as_float(lo);
  }
  // this thread's row of A -> the activation tile (hi and lo)
  {
    const float* __restrict__ row = A + size_t(tid) * K;
#pragma unroll
    for (int c = 0; c < K; ++c) {
      uint32_t hi, lo;
      tc::split_tf32(row[c], hi, lo);
      act[tc::act_index(tid, cA_hi + c)] = __uint_as_float(hi);
      act[tc::act_index(tid, cA_lo + c)] = __uint_as_float(lo);
    }
  }
  tc::fence_proxy_async_smem();
  __syncthreads();

  {
    const uint32_t sa = tc::smem_u32(act);
    float d[2][N / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < N / 2; ++j) d[h][j] = 0.f;
    tc::wgmma_fence_operand(d[0]);
    tc::wgmma_fence_operand(d[1]);
    if constexpr (MODE == 2) {
      // A fragments straight from global memory: row 64 h + 16 (tid / 32) + g (+ 8), column 8 s + q (+ 4) of half h, K step s
      const int g = (tid & 31) >> 2, q = tid & 3;
      uint32_t ah[2][K / 8][4], al[2][K / 8][4];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int s = 0; s < K / 8; ++s)
#pragma unroll
          for (int i = 0; i < 4; ++i)
            tc::split_tf32(A[size_t(64 * h + 16 * (tid >> 5) + g + 8 * (i & 1)) * K + 8 * s + q + 4 * (i >> 1)], ah[h][s][i], al[h][s][i]);
      tc::wgmma_fence_operand(ah[0]); tc::wgmma_fence_operand(ah[1]);
      tc::wgmma_fence_operand(al[0]); tc::wgmma_fence_operand(al[1]);
      tc::wgmma_fence();
#pragma unroll
      for (int ps = 0; ps < 3; ++ps) {
        const float* b_s = (ps == 2) ? sBlo : sBhi;
#pragma unroll
        for (int s = 0; s < K / 8; ++s) {
          const uint64_t bd = tc::smem_desc_sw128(tc::smem_u32(b_s + (s >> 2) * SLAB) + (s & 3) * 32);
          tc::wgmma_tf32_ra<N>(d[0], ps == 1 ? al[0][s] : ah[0][s], bd);
          tc::wgmma_tf32_ra<N>(d[1], ps == 1 ? al[1][s] : ah[1][s], bd);
        }
      }
      tc::wgmma_commit();
      tc::wgmma_wait_all();
      tc::wgmma_fence_operand(ah[0]); tc::wgmma_fence_operand(ah[1]);
      tc::wgmma_fence_operand(al[0]); tc::wgmma_fence_operand(al[1]);
    } else {
      tc::wgmma_fence();
#pragma unroll
      for (int ps = 0; ps < PASSES; ++ps) {
        const int a_c = (ps == 1) ? cA_lo : cA_hi;
        const float* b_s = (ps == 2) ? sBlo : sBhi;
#pragma unroll
        for (int s = 0; s < K / 8; ++s) {
          const uint64_t bd = tc::smem_desc_sw128(tc::smem_u32(b_s + (s >> 2) * SLAB) + (s & 3) * 32);
          tc::wgmma_tf32<N>(d[0], tc::act_desc(sa, a_c + 8 * s, 0), bd);
          tc::wgmma_tf32<N>(d[1], tc::act_desc(sa, a_c + 8 * s, 1), bd);
        }
      }
      tc::wgmma_commit();
      tc::wgmma_wait_all();
    }
    tc::wgmma_fence_operand(d[0]);
    tc::wgmma_fence_operand(d[1]);
    tc::acc_store<N>(act, cD, tid, d);
  }
  __syncthreads();
  for (int c = 0; c < N; ++c) D[size_t(tid) * N + c] = act[tc::act_index(tid, cD + c)];
}

}  // namespace nr

extern "C" int nr_tc_selftest(const float* A, const float* W, float* D, int n, int k, int mode, void* stream) {
  NR_CHECK_ARG(A && W && D, "null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  NR_CHECK_ARG(mode >= 0 && mode <= 2, "mode");
  auto run = [&](auto* fn, int k_) {
    const int smem = (2 * k_ + 64) / 32 * 4096 * 4;
    if (nr::opt_in_smem((const void*)fn, smem, "nr_tc_selftest") != NR_OK) return NR_E_CUDA;
    fn<<<1, 128, smem, s>>>(A, W, D);
    NR_CHECK_LAUNCH("tc_selftest");
    return NR_OK;
  };
  // the mode is a template argument: a runtime loop around the wgmma batch makes ptxas serialise it
  if (n == 32 && k == 32) {
    if (mode == 0) return run(nr::tc_selftest_kernel<32, 32, 0>, 32);
    if (mode == 1) return run(nr::tc_selftest_kernel<32, 32, 1>, 32);
    return run(nr::tc_selftest_kernel<32, 32, 2>, 32);
  }
  if (n == 64 && k == 64 && mode < 2) {
    if (mode == 0) return run(nr::tc_selftest_kernel<64, 64, 0>, 64);
    return run(nr::tc_selftest_kernel<64, 64, 1>, 64);
  }
  if (n == 16 && k == 64) {
    if (mode == 0) return run(nr::tc_selftest_kernel<16, 64, 0>, 64);
    if (mode == 1) return run(nr::tc_selftest_kernel<16, 64, 1>, 64);
    return run(nr::tc_selftest_kernel<16, 64, 2>, 64);
  }
  nr::set_error("nr_tc_selftest: unsupported shape n=%d k=%d mode=%d", n, k, mode);
  return NR_E_UNSUPPORTED;
}
