// Direct rendering of one pass (nr_direct_render, include/neuray_b200.h): the routines of nr_dr_math.cuh on the device.
//   dr_point_kernel  one thread per point, 64 per CTA.  The dist-decoder heads (35 KB) sit in shared memory, where every
//                    thread of the CTA reads the same address; each thread keeps its views' SH-fit rows in a shared-memory
//                    slab, slot-major so that the 64 threads of a slot hit 64 consecutive words.  The packed normal
//                    matrix, the right-hand sides and the Cholesky solve live in registers.
//   dr_ray_kernel    one thread per ray: cumprod of the transmittance and the colour sum.
#include "../../include/neuray_b200.h"
#include "nr_dr_math.cuh"

namespace nr {
namespace dr {

constexpr int THREADS = 64;

__global__ void __launch_bounds__(THREADS) dr_point_kernel(const NrPassParams p, const NrDrParams d, int w_floats) {
  extern __shared__ float4 smem4[];
  float* sw = reinterpret_cast<float*>(smem4);
  float* rows = sw + w_floats;
  for (int i = threadIdx.x; i < w_floats / 4; i += THREADS)
    reinterpret_cast<float4*>(sw)[i] = __ldg(reinterpret_cast<const float4*>(p.w_point) + i);
  __syncthreads();
  const long long N = (long long)p.rn * p.dn;
  const long long n = blockIdx.x * (long long)THREADS + threadIdx.x;
  if (n < N) dr_point(p, d, sw, n, rows + threadIdx.x, THREADS, d.hit_prob_dr, d.point_colors);
}

__global__ void __launch_bounds__(128) dr_ray_kernel(const NrPassParams p, const NrDrParams d) {
  const long long ray = blockIdx.x * 128LL + threadIdx.x;
  if (ray < p.rn) dr_ray(p, d, ray, d.point_colors);
}

}  // namespace dr
}  // namespace nr

extern "C" int nr_direct_render(const NrPassParams* p, const NrDrParams* d, void* stream) {
  using namespace nr;
  NR_CHECK_ARG(p != nullptr && d != nullptr, "params");
  if (p->rn == 0) return NR_OK;
  NR_CHECK_ARG(p->coords && p->que_depth && p->que_cam && p->feat && p->rgb && p->view_params && p->w_point, "null device pointer");
  NR_CHECK_ARG(d->point_colors && d->pixel_colors_dr && d->hit_prob_dr, "null DR output");
  NR_CHECK_ARG(!d->use_nr_color || p->point_rec, "use_nr_color needs the pass' point record");
  NR_CHECK_ARG(p->rfn >= 1 && p->rfn <= NR_MAX_VIEWS && p->dn >= 1 && p->dn <= NR_MAX_SAMPLES, "shape");
  const int w_floats = (p->use_vis ? 4 : 3) * lay::DD_HEAD_STRIDE;
  const size_t smem = sizeof(float) * (w_floats + (d->use_nr_color ? 0 : size_t(dr::THREADS) * p->rfn * dr::ROW));
  static_assert(lay::DD_HEAD == 0 && lay::DD_HEAD_STRIDE % 4 == 0, "the decoder heads are staged as float4 from offset 0");
  if (opt_in_smem((const void*)dr::dr_point_kernel, smem, "nr_direct_render") != NR_OK) return NR_E_CUDA;
  const long long N = (long long)p->rn * p->dn;
  cudaStream_t s = (cudaStream_t)stream;
  dr::dr_point_kernel<<<unsigned((N + dr::THREADS - 1) / dr::THREADS), dr::THREADS, smem, s>>>(*p, *d, w_floats);
  dr::dr_ray_kernel<<<unsigned((p->rn + 127) / 128), 128, 0, s>>>(*p, *d);
  NR_CHECK_LAUNCH("nr_direct_render");
  return NR_OK;
}
