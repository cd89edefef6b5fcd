// Validation metrics (reference network/metrics.py:13-79) and eval.py's PSNR / SSIM: the per-pixel routines shared by the
// CUDA kernels (csrc/nr_metrics.cu) and the host builds of tests/cpu_harness/{metrics,eval}_cpu_harness.cu.
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

// ---- eval.py's scores (tf.image.psnr / tf.image.ssim with max_val 1, filter 11, sigma 1.5, k1 0.01, k2 0.03) ----------

// color_map_forward (reference utils/base_utils.py:492-493): float32(v) / 255, rounded in fp32
NR_HD float unit(int v) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(float(v), 255.f);
#else
  return float(v) / 255.f;
#endif
}

// products and sums that must not be contracted into an FMA: with x == y, 2 E[xy] must equal E[x^2 + y^2] and 2 ux uy must
// equal ux^2 + uy^2 bit for bit, so that identical images give SSIM 1 exactly
NR_HD double mul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}

// the 1-D factor of the 11x11 Gaussian window: g[i] = exp(-(i-5)^2 / (2 1.5^2)), normalised to sum 1; the window is g (x) g
inline void gauss_window(double (&g)[2 * HALF + 1]) {
  double s = 0.0;
  for (int i = 0; i <= 2 * HALF; ++i) {
    g[i] = exp(-double((i - HALF) * (i - HALF)) / (2.0 * 1.5 * 1.5));
    s += g[i];
  }
  for (int i = 0; i <= 2 * HALF; ++i) g[i] /= s;
}

// luminance * cs of one window from its weighted means ux, uy, E[xy] and E[x^2 + y^2] (tf.image.ssim: population covariance,
// c1 = 0.01^2, c2 = 0.03^2)
NR_HD double tf_ssim_term(double ux, double uy, double exy, double exxyy) {
  constexpr double C1 = 0.01 * 0.01, C2 = 0.03 * 0.03;
  const double num0 = 2.0 * mul_rn(ux, uy), den0 = mul_rn(ux, ux) + mul_rn(uy, uy);
  return ((num0 + C1) / (den0 + C1)) * ((2.0 * exy - num0 + C2) / (exxyy - den0 + C2));
}

}  // namespace mt
}  // namespace nr
