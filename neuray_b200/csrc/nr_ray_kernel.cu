// Ray kernel: the per-ray tail of one render_by_depth pass, one warp per ray.
//   + pos_encoding, 4-head self-attention over the ray's samples, LayerNorm (ibrnet.py:356-358, 52-102, 7-27)
//   out_geometry_fc -> sigma, invalid points zeroed (ibrnet.py:359-360)
//   alpha = 1-exp(-relu(sigma)), transmittance product, hit_prob, pixel colour (renderer.py:163-165, render_ops.py:72-80)
//   ray_mask, render_depth (renderer.py:195-202)
//   optional hierarchical resampling: sample_fine_depth + sort (render_ops.py:172-229, renderer.py:205-213)
// Input: the point kernel's 20-float record per point.
#include "nr_common.cuh"
#include "nr_resample.cuh"

namespace nr {
namespace rk {

constexpr int REC = NR_POINT_REC;
constexpr int ROW = 20;   // padded stride of the 16-float per-sample rows in shared memory: the lanes' float4 accesses
                          // (lane = sample) then fall into 8 distinct bank groups instead of 2

struct KParams {
  NrPassParams p;
  int warps;          // warps per CTA
  int per_warp;       // floats of shared memory per warp
  int sort_n;         // power of two >= number of output fine samples (0 if no resampling)
};

__global__ void __launch_bounds__(512) ray_kernel(const KParams kp) {
  extern __shared__ __align__(16) float smem[];
  const NrPassParams& pp = kp.p;
  const int dn = pp.dn, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // CTA-wide: weights + positional table
  float* const sW = smem;                                   // lay::TOTAL_RAY
  float* const sPE = sW + lay::TOTAL_RAY;                   // [dn][ROW]
  float* const wbase = sPE + dn * ROW + size_t(warp) * kp.per_warp;
  // per warp: K and V rows of the ray's samples.  The attention input x = g + pos_enc is NOT kept: a lane re-reads its own
  // sample's 64 bytes (L2 hit) when it needs them again, which brings a warp's footprint from 16.4 KB to 11.3 KB at dn = 64
  // and lets 16 warps share an SM instead of 8 (the kernel is latency bound: ncu short_scoreboard 2.2 per issue at 12 % occupancy)
  float* const sK = wbase;                                  // [dn][ROW]
  float* const sV = sK + dn * ROW;
  float* const sHit = sV + dn * ROW;                        // [dn]
  float* const sT = sHit + dn;                              // [dn]   normalised inverse depth
  float* const sCdf = sT + dn;                              // [dn+1]
  float* const sSort = sCdf + dn + 4;                       // [sort_n]

  for (int i = threadIdx.x; i < lay::TOTAL_RAY; i += blockDim.x) sW[i] = __ldg(pp.w_ray + i);
  for (int i = threadIdx.x; i < dn * 16; i += blockDim.x) sPE[(i >> 4) * ROW + (i & 15)] = __ldg(pp.pos_enc + i);
  __syncthreads();

  const int n_chunks = (dn + 31) / 32;
  for (int ray = blockIdx.x * kp.warps + warp; ray < pp.rn; ray += gridDim.x * kp.warps) {
    const float* __restrict__ rec = pp.point_rec + size_t(ray) * dn * REC;
    const float* __restrict__ qd = pp.que_depth + size_t(ray) * dn;

    // ---- A: x = g + pos_enc ; K, V projections ----
    for (int s = lane; s < dn; s += 32) {
      float x[16];
#pragma unroll
      for (int q4 = 0; q4 < 4; ++q4) {
        const float4 g = __ldg(reinterpret_cast<const float4*>(rec + s * REC) + q4);
        const float4 pe = *reinterpret_cast<const float4*>(sPE + s * ROW + 4 * q4);
        x[4 * q4 + 0] = g.x + pe.x; x[4 * q4 + 1] = g.y + pe.y; x[4 * q4 + 2] = g.z + pe.z; x[4 * q4 + 3] = g.w + pe.w;
      }
      float kk[16], vv[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) { kk[j] = 0.f; vv[j] = 0.f; }
#pragma unroll
      for (int k = 0; k < 16; ++k) {
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          kk[j] = fmaf(sW[lay::WK + k * 16 + j], x[k], kk[j]);
          vv[j] = fmaf(sW[lay::WV + k * 16 + j], x[k], vv[j]);
        }
      }
#pragma unroll
      for (int q4 = 0; q4 < 4; ++q4) {
        *reinterpret_cast<float4*>(sK + s * ROW + 4 * q4) = make_float4(kk[4 * q4], kk[4 * q4 + 1], kk[4 * q4 + 2], kk[4 * q4 + 3]);
        *reinterpret_cast<float4*>(sV + s * ROW + 4 * q4) = make_float4(vv[4 * q4], vv[4 * q4 + 1], vv[4 * q4 + 2], vv[4 * q4 + 3]);
      }
    }
    __syncwarp();

    // ---- B: attention + LayerNorm + out_geometry_fc per owned sample -> alpha ----
    for (int s = lane; s < dn; s += 32) {
      {
        float x[16], q[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) q[j] = 0.f;
#pragma unroll
        for (int q4 = 0; q4 < 4; ++q4) {      // the same expression as in phase A: bit-identical x
          const float4 g = __ldg(reinterpret_cast<const float4*>(rec + s * REC) + q4);
          const float4 pe = *reinterpret_cast<const float4*>(sPE + s * ROW + 4 * q4);
          x[4 * q4 + 0] = g.x + pe.x; x[4 * q4 + 1] = g.y + pe.y; x[4 * q4 + 2] = g.z + pe.z; x[4 * q4 + 3] = g.w + pe.w;
        }
#pragma unroll
        for (int k = 0; k < 16; ++k)
#pragma unroll
          for (int j = 0; j < 16; ++j) q[j] = fmaf(sW[lay::WQ + k * 16 + j], x[k], q[j]);
#pragma unroll
        for (int j = 0; j < 16; ++j) q[j] = (q[j] / 2.f) * 1.4426950408889634f;   // temperature = d_k ** 0.5 = 2; logits in log2 units (softmax via ex2)
        const float nvalid = __ldg(rec + s * REC + 19);
        float o[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) o[j] = 0.f;
        if (nvalid > 1.f) {
          // single pass, blockwise online softmax: 8 keys at a time -- logits of the block, block maximum, ONE rescale of the
          // running sums per block (instead of a separate max pass over all keys: half the K loads and dot products)
          float mx[4] = {-3.4e38f, -3.4e38f, -3.4e38f, -3.4e38f};
          float den[4] = {0.f, 0.f, 0.f, 0.f};
          for (int t0 = 0; t0 < dn; t0 += 8) {
            const int tn = min(8, dn - t0);
#pragma unroll
            for (int hh = 0; hh < 4; ++hh) {
              float l[8];
              float bm = -3.4e38f;
#pragma unroll
              for (int u = 0; u < 8; ++u) {
                if (u < tn) {
                  const float4 k4 = *reinterpret_cast<const float4*>(sK + (t0 + u) * ROW + 4 * hh);
                  l[u] = fmaf(q[4 * hh + 3], k4.w, fmaf(q[4 * hh + 2], k4.z, fmaf(q[4 * hh + 1], k4.y, q[4 * hh] * k4.x)));
                  bm = fmaxf(bm, l[u]);
                } else l[u] = -3.4e38f;
              }
              const float m_new = fmaxf(mx[hh], bm);
              const float scale = ex2_ftz(mx[hh] - m_new);          // first block: ex2(-huge) = 0 on zero sums
              mx[hh] = m_new;
              den[hh] *= scale;
              o[4 * hh + 0] *= scale; o[4 * hh + 1] *= scale; o[4 * hh + 2] *= scale; o[4 * hh + 3] *= scale;
#pragma unroll
              for (int u = 0; u < 8; ++u) {
                if (u < tn) {
                  const float4 v4 = *reinterpret_cast<const float4*>(sV + (t0 + u) * ROW + 4 * hh);
                  const float e = ex2_ftz(l[u] - m_new);
                  den[hh] += e;
                  o[4 * hh + 0] = fmaf(e, v4.x, o[4 * hh + 0]); o[4 * hh + 1] = fmaf(e, v4.y, o[4 * hh + 1]);
                  o[4 * hh + 2] = fmaf(e, v4.z, o[4 * hh + 2]); o[4 * hh + 3] = fmaf(e, v4.w, o[4 * hh + 3]);
                }
              }
            }
          }
#pragma unroll
          for (int j = 0; j < 16; ++j) o[j] /= den[j >> 2];
        } else {
          // masked query row: every logit is -1e9 -> uniform attention over all samples (ibrnet.py:20)
          for (int t = 0; t < dn; ++t) {
#pragma unroll
            for (int j4 = 0; j4 < 4; ++j4) {
              const float4 v4 = *reinterpret_cast<const float4*>(sV + t * ROW + 4 * j4);
              o[4 * j4 + 0] += v4.x; o[4 * j4 + 1] += v4.y; o[4 * j4 + 2] += v4.z; o[4 * j4 + 3] += v4.w;
            }
          }
          const float inv = 1.f / float(dn);
#pragma unroll
          for (int j = 0; j < 16; ++j) o[j] *= inv;
        }
        // fc + residual + LayerNorm(eps 1e-6)
        float y[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) y[j] = x[j];
#pragma unroll
        for (int k = 0; k < 16; ++k)
#pragma unroll
          for (int j = 0; j < 16; ++j) y[j] = fmaf(sW[lay::WFC + k * 16 + j], o[k], y[j]);
        float mean = 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j) mean += y[j];
        mean *= (1.f / 16.f);
        float var = 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j) var = fmaf(y[j] - mean, y[j] - mean, var);
        const float rstd = rsqrtf(var * (1.f / 16.f) + 1e-6f);
#pragma unroll
        for (int j = 0; j < 16; ++j) y[j] = (y[j] - mean) * rstd * sW[lay::LN_W + j] + sW[lay::LN_B + j];
        // out_geometry_fc: 16 -> 16 (ELU) -> 1 (ReLU)
        float hmid[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) hmid[j] = sW[lay::OG0_B + j];
#pragma unroll
        for (int k = 0; k < 16; ++k)
#pragma unroll
          for (int j = 0; j < 16; ++j) hmid[j] = fmaf(sW[lay::OG0_W + k * 16 + j], y[k], hmid[j]);
        float sg = sW[lay::OG1_B];
#pragma unroll
        for (int j = 0; j < 16; ++j) sg = fmaf(sW[lay::OG1_W + j], elu(hmid[j]), sg);
        sg = fmaxf(sg, 0.f);
        if (nvalid < 1.f) sg = 0.f;
        sHit[s] = 1.f - expf(-sg);   // alpha; turned into hit_prob below
      }
    }
    __syncwarp();

    // ---- C: compositing ----
    float carry = 1.f, px = 0.f, py = 0.f, pz = 0.f, pd = 0.f;
    int seen = 0;
    for (int c = 0; c < n_chunks; ++c) {
      {
        const int s = c * 32 + lane;
        const bool in = s < dn;
        const float a = in ? sHit[s] : 0.f;
        const float f = in ? (1.f - a + 1e-10f) : 1.f;
        float incl = f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const float t = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl *= t;
        }
        float excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = 1.f;
        const float hit = a * (carry * excl);
        carry *= __shfl_sync(0xffffffffu, incl, 31);
        if (in) {
          sHit[s] = hit;
          if (pp.hit_prob) pp.hit_prob[size_t(ray) * dn + s] = hit;
          const float4 tail = __ldg(reinterpret_cast<const float4*>(rec + s * REC) + 4);   // rgb, nvalid
          px = fmaf(hit, tail.x, px); py = fmaf(hit, tail.y, py); pz = fmaf(hit, tail.z, pz);
          pd = fmaf(hit, __ldg(qd + s), pd);
          seen += (tail.w > float(pp.ray_mask_view_num)) ? 1 : 0;
        }
      }
    }
    px = warp_sum(px); py = warp_sum(py); pz = warp_sum(pz); pd = warp_sum(pd);
    seen = __reduce_add_sync(0xffffffffu, seen);
    if (lane == 0) {
      if (pp.pixel_colors) { pp.pixel_colors[ray * 3 + 0] = px; pp.pixel_colors[ray * 3 + 1] = py; pp.pixel_colors[ray * 3 + 2] = pz; }
      if (pp.render_depth) pp.render_depth[ray] = pd;
      if (pp.ray_mask) pp.ray_mask[ray] = seen > pp.ray_mask_point_num ? 1 : 0;
    }

    // ---- D: inverse-CDF resampling of the next pass' depths ----
    if (pp.fine_dn > 0) {
      const int M = pp.fine_dn + (pp.fine_use_all ? dn : 0);
      resample_ray(sHit, qd, dn, true, pp.que_cam[21], pp.que_cam[22], pp.fine_u + size_t(ray) * pp.fine_u_stride, pp.fine_dn,
                   pp.fine_use_all, 1, kp.sort_n, sT, sCdf, sSort, pp.fine_depth + size_t(ray) * M, lane);
    }
    __syncwarp();
  }
}

}  // namespace rk

int launch_ray_kernel(const NrPassParams* p, cudaStream_t stream) {
  NR_CHECK_ARG(p != nullptr, "params");
  NR_CHECK_ARG(p->point_rec && p->que_depth && p->que_cam && p->w_ray && p->pos_enc, "null device pointer");
  NR_CHECK_ARG(p->dn >= 3 && p->dn <= NR_MAX_SAMPLES, "dn out of range");
  if (p->fine_dn > 0) {
    NR_CHECK_ARG(p->fine_u && p->fine_depth, "fine_u / fine_depth required when fine_dn > 0");
    NR_CHECK_ARG(p->fine_dn + (p->fine_use_all ? p->dn : 0) <= 2 * NR_MAX_SAMPLES, "too many fine samples");
  }
  if (p->rn == 0) return NR_OK;
  rk::KParams kp;
  kp.p = *p;
  kp.sort_n = 0;
  if (p->fine_dn > 0) {
    kp.sort_n = sort_size_for(p->fine_dn + (p->fine_use_all ? p->dn : 0));
  }
  kp.per_warp = p->dn * 2 * rk::ROW + p->dn * 3 + 8 + kp.sort_n;
  kp.per_warp = (kp.per_warp + 3) & ~3;
  const int shared_common = lay::TOTAL_RAY + p->dn * rk::ROW;
  int warps = 16;
  while (warps > 1 && size_t(shared_common + warps * kp.per_warp) * 4 > 216 * 1024) warps >>= 1;
  kp.warps = warps;
  const size_t smem = size_t(shared_common + warps * kp.per_warp) * 4;
  NR_CHECK_ARG(smem <= 227 * 1024, "ray kernel shared memory");
  if (opt_in_smem((const void*)rk::ray_kernel, smem, "ray_kernel") != NR_OK) return NR_E_CUDA;
  int sms;
  if (sm_count(&sms, "ray_kernel") != NR_OK) return NR_E_CUDA;
  int grid = (p->rn + warps - 1) / warps;
  const int cap = sms * 4;
  if (grid > cap) grid = cap;
  rk::ray_kernel<<<grid, warps * 32, smem, stream>>>(kp);
  NR_CHECK_LAUNCH("ray_kernel");
  return NR_OK;
}

}  // namespace nr
