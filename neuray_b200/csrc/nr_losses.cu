// Training extras next to the ray path (SURVEY.md 8(f) row f3): kernels and C-ABI entry points over the routines of
// nr_loss_math.cuh -- predict_mean_for_depth_loss (renderer.py:280-316) and the three losses of network/loss.py.
// The reductions are one block per output element (512 .. 65 536 terms each): deterministic, no atomics.
#include "nr_loss_math.cuh"

namespace nr {
namespace ls {

__global__ void __launch_bounds__(64) depth_mean_kernel(const __grid_constant__ DepthMeanP p) {
  const long long i = (long long)blockIdx.x * 64 + threadIdx.x;
  if (i < (long long)p.rfn * p.pn) depth_mean_point(p, i);
}

// sum of (a, b) over the block's threads; result valid in thread 0
__device__ __forceinline__ void block_sum2(double& a, double& b) {
  __shared__ double sa[32], sb[32];
  a = warp_sum(a);
  b = warp_sum(b);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { sa[warp] = a; sb[warp] = b; }
  __syncthreads();
  if (warp == 0) {
    a = lane < (blockDim.x >> 5) ? sa[lane] : 0.0;
    b = lane < (blockDim.x >> 5) ? sb[lane] : 0.0;
    a = warp_sum(a);
    b = warp_sum(b);
  }
}

__global__ void __launch_bounds__(1024) render_loss_kernel(const float* pr, const float* gt, const uint8_t* mask, int rn, float* loss) {
  const int q = blockIdx.x;
  double num = 0.0, den = 0.0;
  for (int r = threadIdx.x; r < rn; r += blockDim.x) {
    const long long i = (long long)q * rn + r;
    const float m = mask != nullptr ? float(mask[i] != 0) : 1.f;
    num += double(render_loss_term(pr, gt, i) * m);
    den += double(m);
  }
  block_sum2(num, den);
  if (threadIdx.x == 0) loss[q] = mask != nullptr ? float(num) / (float(den) + 1e-3f) : float(num / rn);
}
__global__ void __launch_bounds__(1024) render_loss_bwd_kernel(const float* pr, const float* gt, const uint8_t* mask, int rn, const float* g, float* d_pr) {
  const int q = blockIdx.x;
  double den = 0.0, unused = 0.0;
  if (mask != nullptr)
    for (int r = threadIdx.x; r < rn; r += blockDim.x) den += double(mask[(long long)q * rn + r] != 0);
  block_sum2(den, unused);
  __shared__ float scale;
  if (threadIdx.x == 0) scale = g[q] * 2.f / (mask != nullptr ? float(den) + 1e-3f : float(rn));
  __syncthreads();
  for (int r = threadIdx.x; r < rn; r += blockDim.x) {
    const long long i = (long long)q * rn + r;
    const float m = mask != nullptr ? float(mask[i] != 0) : 1.f;
    for (int c = 0; c < 3; ++c) d_pr[3 * i + c] = scale * m * (pr[3 * i + c] - gt[3 * i + c]);
  }
}

__global__ void __launch_bounds__(1024) depth_loss_kernel(const __grid_constant__ DepthLossP p) {
  const int view = blockIdx.x;
  double num = 0.0, den = 0.0;
  for (int j = threadIdx.x; j < p.pn; j += blockDim.x) {
    float term, dterm, m;
    depth_loss_term(p, (long long)view * p.pn + j, p.depth_pr, term, dterm, m);
    num += double(term * m);
    den += double(m);
  }
  block_sum2(num, den);
  __shared__ float scale;
  if (threadIdx.x == 0) {
    const float d = p.aug_depth != nullptr ? float(den) + 1e-4f : float(p.pn);
    if (p.g == nullptr) p.loss[view] = float(num) / d;
    else scale = p.g[view] / d;
  }
  if (p.g == nullptr) return;
  __syncthreads();
  for (int j = threadIdx.x; j < p.pn; j += blockDim.x) {
    const long long i = (long long)view * p.pn + j;
    float term, dterm, m;
    depth_loss_term(p, i, p.depth_pr, term, dterm, m);
    p.d_depth_pr[i] = scale * m * dterm;
  }
}

__global__ void __launch_bounds__(1024) consistency_loss_kernel(const float* p0, const float* p1, int rn, int dn, float* loss, const float* g, float* d_p1) {
  const int q = blockIdx.x;
  const long long n = (long long)rn * dn, base = (long long)q * n;
  if (g == nullptr) {
    double num = 0.0, unused = 0.0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) num += double(consist_term(p0[base + i], p1[base + i]));
    block_sum2(num, unused);
    if (threadIdx.x == 0) loss[q] = float(num / double(n));
  } else {
    const float scale = g[q] / float(n);
    for (long long i = threadIdx.x; i < n; i += blockDim.x) d_p1[base + i] = scale * consist_dterm(p0[base + i], p1[base + i]);
  }
}

}  // namespace ls
}  // namespace nr

using namespace nr;

extern "C" int nr_depth_mean(const NrDepthMeanParams* p, void* stream) {
  NR_CHECK_ARG(p != nullptr, "params");
  if (p->rfn == 0 || p->pn == 0) return NR_OK;
  NR_CHECK_ARG(p->map && p->coords && p->w_point[0], "depth_mean: null device pointer");
  NR_CHECK_ARG(p->rfn >= 1 && p->pn >= 1 && p->h > 1 && p->w > 1 && p->fh >= 1 && p->fw >= 1, "depth_mean: shape");
  for (int d = 0; d < 2; ++d) {
    NR_CHECK_ARG(p->d_mean[d] == nullptr || (p->w_point[d] != nullptr && p->d_w_point[d] != nullptr), "depth_mean: d_w_point required for the backward");
    NR_CHECK_ARG(p->w_point[d] == nullptr || p->mean[d] != nullptr || p->d_mean[d] != nullptr, "depth_mean: an evaluated decoder needs mean or d_mean");
  }
  const long long n = (long long)p->rfn * p->pn;
  ls::depth_mean_kernel<<<unsigned((n + 63) / 64), 64, 0, (cudaStream_t)stream>>>(*p);
  NR_CHECK_LAUNCH("depth_mean_kernel");
  return NR_OK;
}

extern "C" int nr_render_loss(const float* pr, const float* gt, const uint8_t* ray_mask, int qn, int rn, float* loss, const float* g, float* d_pr,
                              void* stream) {
  if (qn == 0) return NR_OK;
  NR_CHECK_ARG(pr && gt && qn >= 1 && rn >= 0, "render_loss: arguments");
  NR_CHECK_ARG(g == nullptr ? loss != nullptr : d_pr != nullptr, "render_loss: output pointer");
  if (g == nullptr) ls::render_loss_kernel<<<qn, 1024, 0, (cudaStream_t)stream>>>(pr, gt, ray_mask, rn, loss);
  else ls::render_loss_bwd_kernel<<<qn, 1024, 0, (cudaStream_t)stream>>>(pr, gt, ray_mask, rn, g, d_pr);
  NR_CHECK_LAUNCH("render_loss");
  return NR_OK;
}

extern "C" int nr_depth_loss(const NrDepthLossParams* p, void* stream) {
  NR_CHECK_ARG(p != nullptr, "params");
  if (p->rfn == 0) return NR_OK;
  NR_CHECK_ARG(p->depth_pr && p->coords && p->true_depth && p->depth_range, "depth_loss: null device pointer");
  NR_CHECK_ARG(p->rfn >= 1 && p->pn >= 1 && p->h > 1 && p->w > 1 && (p->loss_type == 0 || (p->loss_type == 1 && p->beta > 0.f)), "depth_loss: arguments");
  NR_CHECK_ARG(p->g == nullptr ? p->loss != nullptr : p->d_depth_pr != nullptr, "depth_loss: output pointer");
  ls::depth_loss_kernel<<<p->rfn, 1024, 0, (cudaStream_t)stream>>>(*p);
  NR_CHECK_LAUNCH("depth_loss_kernel");
  return NR_OK;
}

extern "C" int nr_consistency_loss(const float* prob0, const float* prob1, int qn, int rn, int dn, float* loss, const float* g, float* d_prob1,
                                   void* stream) {
  if (qn == 0) return NR_OK;
  NR_CHECK_ARG(prob0 && prob1 && qn >= 1 && rn >= 1 && dn >= 1, "consistency_loss: arguments");
  NR_CHECK_ARG(g == nullptr ? loss != nullptr : d_prob1 != nullptr, "consistency_loss: output pointer");
  ls::consistency_loss_kernel<<<qn, 1024, 0, (cudaStream_t)stream>>>(prob0, prob1, rn, dn, loss, g, d_prob1);
  NR_CHECK_LAUNCH("consistency_loss_kernel");
  return NR_OK;
}
