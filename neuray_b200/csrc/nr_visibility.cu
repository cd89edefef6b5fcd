// Per-view visibility of each rendered pixel (nr_view_visibility, include/neuray_b200.h): the routines of
// nr_visibility_math.cuh on the device.
//   view_visibility_kernel  128 threads per CTA, THREADS / lanes rays at a time, one lane per thread.  The dist-decoder
//                           heads (26 KB, 35 KB with the vis head) sit in shared memory, where every thread of the CTA
//                           reads the same address; each thread's per-view partial sums sit in a shared-memory slab,
//                           view-major ([rfn][128]), so that a warp's lanes hit 32 consecutive words.  A persistent grid
//                           stages the heads once per CTA.
#include "../../include/neuray_b200.h"
#include "nr_visibility_math.cuh"

namespace nr {
namespace vis {

__global__ void __launch_bounds__(THREADS) view_visibility_kernel(const NrPassParams p, const NrVisParams q, int w_floats, int lanes,
                                                                  long long groups) {
  extern __shared__ float4 smem4[];
  float* sw = reinterpret_cast<float*>(smem4);
  float* slab = sw + w_floats;
  for (int i = threadIdx.x; i < w_floats / 4; i += THREADS)
    reinterpret_cast<float4*>(sw)[i] = __ldg(reinterpret_cast<const float4*>(p.w_point) + i);
  __syncthreads();
  const int lane = threadIdx.x & (lanes - 1), slot = threadIdx.x / lanes;
  float* acc = slab + threadIdx.x;
  for (long long grp = blockIdx.x; grp < groups; grp += gridDim.x) {
    const long long ray = grp * (THREADS / lanes) + slot;
    const bool live = ray < p.rn;
    if (live) lane_sum(p, sw, q.hit_prob, ray, lane, lanes, acc, THREADS);
    __syncthreads();
    for (int half = lanes >> 1; half > 0; half >>= 1) {       // the same number of levels in every thread of the CTA
      if (live && lane < half) tree_level(acc, THREADS, p.rfn, half);
      __syncthreads();
    }
    if (live)
      for (int v = lane; v < p.rfn; v += lanes) q.visibility[ray * p.rfn + v] = slab[v * THREADS + slot * lanes];
    __syncthreads();                                           // the slab is read before the next group overwrites it
  }
}

}  // namespace vis
}  // namespace nr

extern "C" int nr_view_visibility(const NrPassParams* p, const NrVisParams* q, void* stream) {
  using namespace nr;
  NR_CHECK_ARG(p != nullptr && q != nullptr, "params");
  if (p->rn == 0) return NR_OK;
  NR_CHECK_ARG(p->coords && p->que_depth && p->que_cam && p->feat && p->rgb && p->view_params && p->w_point, "null device pointer");
  NR_CHECK_ARG(q->hit_prob && q->visibility, "null visibility input or output");
  NR_CHECK_ARG(p->rfn >= 1 && p->rfn <= NR_MAX_VIEWS && p->dn >= 1 && p->dn <= NR_MAX_SAMPLES, "shape");
  const int w_floats = (p->use_vis ? 4 : 3) * lay::DD_HEAD_STRIDE;
  const size_t smem = sizeof(float) * (w_floats + size_t(vis::THREADS) * p->rfn);
  static_assert(lay::DD_HEAD == 0 && lay::DD_HEAD_STRIDE % 4 == 0, "the decoder heads are staged as float4 from offset 0");
  if (opt_in_smem((const void*)vis::view_visibility_kernel, smem, "nr_view_visibility") != NR_OK) return NR_E_CUDA;
  int sms = 0, per_sm = 0;
  if (sm_count(&sms, "nr_view_visibility") != NR_OK) return NR_E_CUDA;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, vis::view_visibility_kernel, vis::THREADS, smem) != cudaSuccess || per_sm == 0) {
    set_error("nr_view_visibility: no occupancy for %zu bytes of shared memory", smem);
    return NR_E_CUDA;
  }
  const int lanes = vis::ray_lanes(p->dn);
  const int rays_per_cta = vis::THREADS / lanes;
  const long long groups = (p->rn + rays_per_cta - 1) / rays_per_cta;
  const long long grid = groups < (long long)sms * per_sm ? groups : (long long)sms * per_sm;
  vis::view_visibility_kernel<<<unsigned(grid), vis::THREADS, smem, (cudaStream_t)stream>>>(*p, *q, w_floats, lanes, groups);
  NR_CHECK_LAUNCH("nr_view_visibility");
  return NR_OK;
}
