// Per-view colour-blend weight of each rendered pixel (nr_render_pass_fwd_blend, include/neuray_b200.h): the reduction
// behind the pass.  The point kernel exports each valid (view, point) row's blend weight w (the reference's
// blending_weights_valid, ibrnet.py:362-366) into row_blend [rfn][rn*dn]; this kernel forms
//
//   blend_weights[r, v] = Σ_d hit_nr[r, d] · row_blend[v, r*dn + d]
//
//   blend_weights_kernel  one warp per ray, 256 threads per CTA.  Lane l holds the ray's hit_prob at d = l, l + 32, ...
//                         in registers; per view it sums its samples in increasing d, reading the view's row of the ray
//                         (dn consecutive floats) coalesced, and a fixed xor butterfly (16, 8, 4, 2, 1) adds the 32
//                         lanes.  The order depends on dn alone and no atomics are used, so a ray's weights are the same
//                         whichever chunk, shard or CTA renders it.  Lane v keeps view v's sum; the ray's rfn values
//                         leave in one store.
//
// nr_render_pass_fwd_view runs the same kernel on the exported hit rows with the query depths as the per-sample weight
// (view_depth) and, in its UNIT form, with a weight of 1 (view_hit: the per-sample weight is not read).
#include "../../include/neuray_b200.h"
#include "nr_common.cuh"

namespace nr {
namespace blend {

constexpr int THREADS = 256;
constexpr int PER_LANE = NR_MAX_SAMPLES / 32;     // a ray's samples held by one lane

// UNIT: every sample weighs 1 and hit_prob is not read
template <bool UNIT>
__global__ void __launch_bounds__(THREADS) blend_weights_kernel(const float* __restrict__ hit_prob, const float* __restrict__ row_blend,
                                                                 float* __restrict__ blend_weights, int rn, int dn, int rfn) {
  const int lane = threadIdx.x & 31;
  const long long ray = (long long)blockIdx.x * (THREADS / 32) + (threadIdx.x >> 5);
  if (ray >= rn) return;                          // whole warps leave together
  const long long N = (long long)rn * dn;
  float hit[PER_LANE];
#pragma unroll
  for (int j = 0; j < PER_LANE; ++j) {
    const int d = lane + 32 * j;
    hit[j] = d < dn ? (UNIT ? 1.f : __ldg(hit_prob + ray * dn + d)) : 0.f;
  }
  float mine = 0.f;
  for (int v = 0; v < rfn; ++v) {
    const float* __restrict__ w = row_blend + v * N + ray * dn;
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < PER_LANE; ++j) {
      const int d = lane + 32 * j;
      if (d < dn) acc = fmaf(hit[j], __ldg(w + d), acc);
    }
    acc = warp_sum(acc);
    if (lane == v) mine = acc;
  }
  if (lane < rfn) blend_weights[ray * rfn + lane] = mine;
}

}  // namespace blend

// The reduction of nr_render_pass_fwd_blend / _tf32_blend, enqueued behind the pass that filled b->row_blend and
// p->hit_prob.  nr_render_pass_fwd_agg / _tf32_agg and _view / _tf32_view run it once per output, each on its
// [rfn][rn*dn] row of the export.  weight: the per-sample weight [rn, dn] (p->hit_prob, or p->que_depth for
// view_depth), NULL for a weight of 1 (view_hit).
int launch_blend_weights(const NrPassParams* p, const NrBlendParams* b, const float* weight, cudaStream_t stream) {
  if (p->rn == 0) return NR_OK;
  const long long blocks = ((long long)p->rn + blend::THREADS / 32 - 1) / (blend::THREADS / 32);
  if (weight != nullptr)
    blend::blend_weights_kernel<false><<<unsigned(blocks), blend::THREADS, 0, stream>>>(weight, b->row_blend, b->blend_weights, p->rn,
                                                                                        p->dn, p->rfn);
  else
    blend::blend_weights_kernel<true><<<unsigned(blocks), blend::THREADS, 0, stream>>>(nullptr, b->row_blend, b->blend_weights, p->rn,
                                                                                       p->dn, p->rfn);
  NR_CHECK_LAUNCH("blend_weights");
  return NR_OK;
}

}  // namespace nr
