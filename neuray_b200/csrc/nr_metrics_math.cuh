// Validation metrics (reference network/metrics.py:13-79): the per-pixel routines shared by the CUDA kernels
// (csrc/nr_metrics.cu) and the host build of tests/cpu_harness/metrics_cpu_harness.cu.
#pragma once
#include <math.h>

#include "nr_common.cuh"

#ifndef NR_HD
#define NR_HD __host__ __device__ __forceinline__
#endif

namespace nr {
namespace mt {

constexpr int HALF = 5;    // 11x11 window

// color_map_backward (reference utils/base_utils.py:496-499): v * 255 in fp32, clip to [0, 255], truncate
NR_HD int quantise(float v) {
#ifdef __CUDA_ARCH__
  const float s = __fmul_rn(v, 255.f);
#else
  const float s = v * 255.f;
#endif
  return (int)fminf(fmaxf(s, 0.f), 255.f);
}

// S of one window from its integer sums.  With N = 121: ux = sx/N and vx = (N sxx - sx^2) / (N (N-1)) (skimage's sample
// covariance), likewise for y and xy.  The luminance factors of S share the denominator N^2 and the contrast factors
// N (N-1), so those cancel and every term but C1, C2 is an exact integer.
NR_HD double ssim_term(int sx, int sy, int sxx, int syy, int sxy) {
  constexpr double N = 121.0;
  constexpr double C1 = (0.01 * 255) * (0.01 * 255) * N * N;
  constexpr double C2 = (0.03 * 255) * (0.03 * 255) * N * (N - 1);
  const long long xx = (long long)sx * sx, yy = (long long)sy * sy, xy = (long long)sx * sy;
  const long long a1 = 2 * xy, b1 = xx + yy;
  const long long a2 = 2 * (121LL * sxy - xy), b2 = 121LL * (sxx + syy) - xx - yy;
  return ((double(a1) + C1) * (double(a2) + C2)) / ((double(b1) + C1) * (double(b2) + C2));
}

}  // namespace mt
}  // namespace nr
