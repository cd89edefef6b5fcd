// Inverse-CDF resampling of one ray by one warp (reference render_ops.py:172-229 with inv_mode=True, followed by
// the sort of renderer.py:210-213).  Shared by the ray kernel (fused) and nr_sample_fine_depth (stand-alone).
#pragma once
#include "nr_common.cuh"

namespace nr {

// hit: [dn] hit probabilities (shared or global); qd: [dn] depths of the current samples (global)
// sT [dn], sCdf [dn+1], sSort [sort_n] are per-warp shared scratch.  out: [fine_dn (+dn)] global.
// inv: resample in normalised inverse depth (inv_mode=True, the renderer's mode); otherwise directly in depth.
__device__ __forceinline__ void resample_ray(const float* hit, const float* __restrict__ qd, int dn, bool inv, float near, float far,
                                             const float* __restrict__ u_row, int fdn, int use_all, int do_sort, int sort_n,
                                             float* sT, float* sCdf, float* sSort, float* __restrict__ out, int lane) {
  const float a = -1.f / near, b = -1.f / far;
  float psum = 0.f;
  for (int s = lane; s < dn; s += 32) {
    sT[s] = inv ? (-1.f / __ldg(qd + s) - a) / (b - a) : __ldg(qd + s);
    psum += hit[s] + 1e-5f;
  }
  psum = warp_sum(psum);
  __syncwarp();
  if (lane == 0) {   // torch.cumsum on the CPU accumulates float inputs in double
    double acc = 0.0;
    sCdf[0] = 0.f;
    for (int s = 0; s < dn; ++s) {
      acc += double((hit[s] + 1e-5f) / psum);
      sCdf[s + 1] = float(acc);
    }
  }
  __syncwarp();
  const int base = use_all ? dn : 0;
  for (int k = lane; k < fdn; k += 32) {
    const float u = __ldg(u_row + k);
    // searchsorted(cdf, u, right=True): first index with cdf[i] > u, in [0, dn+1]
    int lo = 0, hi = dn + 1;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (sCdf[mid] > u) hi = mid; else lo = mid + 1;
    }
    const int below = max(lo - 1, 0), above = min(lo, dn);
    const float c0 = sCdf[below], c1 = sCdf[above];
    // bin edges: e_0 = t_0, e_i = (t_i + t_{i-1})/2, e_dn = t_{dn-1}
    const float e0 = below == 0 ? sT[0] : (below == dn ? sT[dn - 1] : (sT[below] + sT[below - 1]) / 2.f);
    const float e1 = above == 0 ? sT[0] : (above == dn ? sT[dn - 1] : (sT[above] + sT[above - 1]) / 2.f);
    float den = c1 - c0;
    if (den < 1e-5f) den = 1.f;
    const float tt = (u - c0) / den;
    const float fd = e0 + tt * (e1 - e0);
    sSort[base + k] = inv ? -1.f / (fd * (b - a) + a) : fd;
  }
  if (use_all)
    for (int s = lane; s < dn; s += 32) sSort[s] = __ldg(qd + s);
  const int M = base + fdn;
  __syncwarp();
  if (do_sort) {
    for (int i = M + lane; i < sort_n; i += 32) sSort[i] = __int_as_float(0x7f800000);
    __syncwarp();
    for (int size = 2; size <= sort_n; size <<= 1) {   // bitonic, ascending
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        for (int i = lane; i < sort_n / 2; i += 32) {
          const int lo_i = 2 * i - (i & (stride - 1));
          const int hi_i = lo_i + stride;
          const bool up = (lo_i & size) == 0;
          const float x0 = sSort[lo_i], x1 = sSort[hi_i];
          if ((x0 > x1) == up) { sSort[lo_i] = x1; sSort[hi_i] = x0; }
        }
        __syncwarp();
      }
    }
  }
  for (int i = lane; i < M; i += 32) out[i] = sSort[i];
}

inline int sort_size_for(int M) {
  int n = 2;
  while (n < M) n <<= 1;
  return n;
}

}  // namespace nr
