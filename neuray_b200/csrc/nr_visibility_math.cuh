// Per-view visibility of each rendered pixel (nr_view_visibility, include/neuray_b200.h), as plain routines.  The device
// kernel of nr_visibility.cu runs them, and tests/cpu_harness/vis_cpu_harness.cu runs the same code on the host.
//
//   visibility[r, v] = Σ_d hit_nr[r, d] · vis_v[r, d]
//
// vis_v is the reference's masked prj_dict['vis'] (network/renderer.py:79-82): compute_prob's visibility of the active
// pass' dist decoder (the mixture-weighted 1 - cdf0, times the vis head with the coarse decoder's use_vis), times the
// projection mask; each row comes from tr::row_front, the one copy of the gather and dist-decoder math.
//
// A ray's samples are split over `lanes` lanes (ray_lanes): lane l sums its samples l, l + lanes, ... in order, and the
// lanes are then added by a fixed binary tree (tree_level, half = lanes / 2, ..., 1).  The order depends only on dn, so
// a ray's result is the same whichever chunk, shard or CTA renders it.
#pragma once
#include "nr_train_math.cuh"

namespace nr {
namespace vis {

constexpr int THREADS = 128;

// Lanes per ray: the least power of two >= dn, at most THREADS.
NR_HD int ray_lanes(int dn) {
  int l = 1;
  while (l < dn && l < THREADS) l <<= 1;
  return l;
}

// One lane's share of ray `ray`: acc[v * stride] = Σ over samples d = lane, lane + lanes, ... of hit[d] · vis_v[d].
// A sample with hit exactly 0 adds exactly 0, so its rows are skipped.
NR_HD void lane_sum(const NrPassParams& pp, const float* __restrict__ W, const float* __restrict__ hit_prob, long long ray,
                    int lane, int lanes, float* acc, int stride) {
  const int n_heads = pp.use_vis ? 4 : 3;
  for (int v = 0; v < pp.rfn; ++v) acc[v * stride] = 0.f;
  for (int d = lane; d < pp.dn; d += lanes) {
    const long long n = ray * pp.dn + d;
    const float hit = hit_prob[n];
    if (hit == 0.f) continue;
    const PointGeo g = point_geometry(pp.que_cam, pp.coords, pp.que_depth, pp.dn, n);
    for (int v = 0; v < pp.rfn; ++v) {
      tr::RowFront f;
      tr::row_front(pp, W, n_heads, g, v, f, nullptr, 0);
      acc[v * stride] = fmaf(hit, f.visb * f.mask, acc[v * stride]);
    }
  }
}

// One level of the per-ray tree, for a lane below `half`: adds the partial sums of lane + half to its own.
NR_HD void tree_level(float* acc, int stride, int rfn, int half) {
  for (int v = 0; v < rfn; ++v) acc[v * stride] += acc[v * stride + half];
}

}  // namespace vis
}  // namespace nr
