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
//
// nr_view_colors weights each view's colour with the same blend row:
//
//   view_colors[r, v, c] = Σ_d hit_nr[r, d] · row_blend[v, r*dn + d] · rgb_v[r, d, c]
//
//   view_colors_kernel    the same layout: one warp per ray, lane l owns d = l, l + 32, ...  Each lane forms its samples'
//                         world points once (point_geometry) and keeps them with hit_prob in registers.  Per view it reads
//                         the ray's blend row coalesced; a sample whose hit · w is exactly 0 adds exactly 0 and is
//                         skipped, the others are projected into the view and, where the projection is valid, take the
//                         RGB taps of the point kernel (rgb_tap) into three sums in increasing d.  The same butterfly
//                         adds the lanes, and lane v stores view v's three sums.
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

__global__ void __launch_bounds__(THREADS) view_colors_kernel(const NrPassParams p, const NrColorParams c) {
  const int lane = threadIdx.x & 31, dn = p.dn, rfn = p.rfn;
  const long long ray = (long long)blockIdx.x * (THREADS / 32) + (threadIdx.x >> 5);
  if (ray >= p.rn) return;                        // whole warps leave together
  const long long N = (long long)p.rn * dn;
  float hit[PER_LANE], X[PER_LANE], Y[PER_LANE], Z[PER_LANE];
#pragma unroll
  for (int j = 0; j < PER_LANE; ++j) {
    const int d = lane + 32 * j;
    hit[j] = 0.f; X[j] = 0.f; Y[j] = 0.f; Z[j] = 0.f;
    if (d < dn) {
      hit[j] = __ldg(c.hit_prob + ray * dn + d);
      if (hit[j] != 0.f) {
        const PointGeo g = point_geometry(p.que_cam, p.coords, p.que_depth, dn, ray * dn + d);
        X[j] = g.X; Y[j] = g.Y; Z[j] = g.Z;
      }
    }
  }
  float mine[3] = {0.f, 0.f, 0.f};
  for (int v = 0; v < rfn; ++v) {
    const float* __restrict__ w = c.row_blend + v * N + ray * dn;
    float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < PER_LANE; ++j) {
      const int d = lane + 32 * j;
      if (d >= dn) continue;
      const float hw = hit[j] * __ldg(w + d);
      if (hw == 0.f) continue;
      const Proj pj = project(p.view_params + 20 * v, X[j], Y[j], Z[j], p.h, p.w);
      if (!pj.valid) continue;
      float rgb[3];
      rgb_tap(p.rgb, v, pj.ux, pj.uy, p.h, p.w, rgb);
#pragma unroll
      for (int k = 0; k < 3; ++k) acc[k] = fmaf(hw, rgb[k], acc[k]);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      acc[k] = warp_sum(acc[k]);
      if (lane == v) mine[k] = acc[k];
    }
  }
  if (lane < rfn) {
    float* o = c.view_colors + (ray * rfn + lane) * 3;
    o[0] = mine[0]; o[1] = mine[1]; o[2] = mine[2];
  }
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

extern "C" int nr_view_colors(const NrPassParams* p, const NrColorParams* c, void* stream) {
  using namespace nr;
  NR_CHECK_ARG(p != nullptr && c != nullptr, "params");
  if (p->rn == 0) return NR_OK;
  NR_CHECK_ARG(p->coords && p->que_depth && p->que_cam && p->rgb && p->view_params, "null device pointer");
  NR_CHECK_ARG(c->row_blend && c->hit_prob && c->view_colors, "null blend row, hit_prob or view_colors");
  NR_CHECK_ARG(p->rn > 0 && p->rfn >= 1 && p->rfn <= NR_MAX_VIEWS && p->dn >= 1 && p->dn <= NR_MAX_SAMPLES && p->h > 1 && p->w > 1,
               "shape");
  static_assert(NR_MAX_VIEWS <= 32, "lane v keeps view v's sums");
  const long long blocks = ((long long)p->rn + blend::THREADS / 32 - 1) / (blend::THREADS / 32);
  blend::view_colors_kernel<<<unsigned(blocks), blend::THREADS, 0, (cudaStream_t)stream>>>(*p, *c);
  NR_CHECK_LAUNCH("nr_view_colors");
  return NR_OK;
}
