// Per-checkpoint / per-optimizer-step and per-frame packing done by the library itself, so that a host in any language
// can drive the kernels from the reference's own tensors:
//
//   nr_pack_weights   parameters of one pass in PyTorch's [out][in] layout -> the three flat buffers the kernels read
//                     (w_point, w_ray: NrWeightLayout; w_tc: NrTcLayout = hi/lo tf32 parts in K-major SWIZZLE_128B tiles)
//   nr_pack_weights_tf32  the same pass -> w_tc of the point kernel's TF32 mode: the same layout, each weight rounded
//                     to the nearest tf32 value in its hi slot, the lo slots zero
//   nr_camera_blocks  poses / intrinsics / depth ranges -> que_cam [24] and view_params [rfn,20]
//
// Both are single launches with no host synchronisation and no library-side state.
#include "nr_common.cuh"
#include "nr_tc.cuh"

namespace nr {
namespace pack {

struct Job {
  const float* w;
  const float* b;
  int n_out, n_in;
};
constexpr int NJOBS = 38;
struct Jobs {
  Job j[NJOBS];
};
// job numbers
enum { J_DD = 0 /* + 3*head + layer */, J_PE0 = 12, J_PE1, J_RD0, J_RD1, J_NF0, J_NF1, J_B0, J_B1, J_V0, J_V1, J_V20, J_V21,
       J_C0, J_C1, J_C2, J_G0, J_G1, J_OG0, J_OG1, J_WQ, J_WK, J_WV, J_WFC, J_LNW, J_LNB, J_COMP };
static_assert(J_COMP == NJOBS - 1, "job table");

struct Out {
  float* wp;
  float* wr;
  float* wt;
};

// element (row n, column k) of the tensor-core tile at `off` with layout t: slab k/32, swizzled inside.  TF32: rna(v) in
// the hi slot and nothing in the lo slot (the TF32 point kernel reads only hi)
template <bool TF32>
__device__ __forceinline__ void put_tc(float* wt, int off, tcl::Tile t, int n, int k, float v) {
  const int pos = off + (k >> 5) * t.slab + tc::sw128_index(n, k & 31);
  if constexpr (TF32) {
    wt[pos + t.hi] = __uint_as_float(tc::tf32_rna(v));
  } else {
    const float hi = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
    wt[pos + t.hi] = hi;
    wt[pos + t.lo] = v - hi;
  }
}
// an entry of w_point / w_ray (the TF32 pack writes neither)
template <bool TF32>
__device__ __forceinline__ void put_w(float* buf, int i, float v) {
  if constexpr (!TF32) buf[i] = v;
}

template <bool TF32>
__global__ void pack_weights_kernel(const Jobs jobs, const Out out) {
  const int job = blockIdx.x;
  const Job J = jobs.j[job];
  if (J.w == nullptr) return;
  float* __restrict__ wp = out.wp;
  float* __restrict__ wr = out.wr;
  float* __restrict__ wt = out.wt;
  const int nw = J.n_out * J.n_in;
  if (job == J_COMP) {
    // rows 32..39 of the prob_embed.2 tile: neuray_fc.0 applied to prob_embed.2's (linear) output, W_nf0 @ W_pe2 in fp64
    const float* __restrict__ nf0 = J.w;      // [8,32]
    const float* __restrict__ pe1 = J.b;      // [32,32]
    for (int e = threadIdx.x; e < 8 * 32; e += blockDim.x) {
      const int r = e >> 5, k = e & 31;
      double acc = 0.0;
      for (int j = 0; j < 32; ++j) acc = fma(double(nf0[r * 32 + j]), double(pe1[j * 32 + k]), acc);
      put_tc<TF32>(wt, tcl::PE1, tcl::PE1_L, 32 + r, k, float(acc));
    }
    return;
  }
  // weights, element e = o * n_in + i  (PyTorch Linear layout [out][in])
  for (int e = threadIdx.x; e < nw; e += blockDim.x) {
    const int o = e / J.n_in, i = e - o * J.n_in;
    const float v = J.w[e];
    if (job < 12) {
      const int h = job / 3, l = job - 3 * h;
      const int base = lay::DD_HEAD + h * lay::DD_HEAD_STRIDE;
      if (l == 0) { put_w<TF32>(wp, base + lay::DD_L0_W + i * 32 + o, v); put_tc<TF32>(wt, tcl::HEAD0 + h * tcl::STAGE, tcl::HEAD_L0, o, i, v); }
      else if (l == 1) { put_w<TF32>(wp, base + lay::DD_L1_W + i * 32 + o, v); put_tc<TF32>(wt, tcl::HEAD0 + h * tcl::STAGE, tcl::HEAD_L1, o, i, v); }
      else put_w<TF32>(wp, base + lay::DD_L2_W + o * 32 + i, v);
      continue;
    }
    switch (job) {
      case J_PE0: put_w<TF32>(wp, lay::GRP_B + lay::PE0_W + i * 32 + o, v); put_tc<TF32>(wt, tcl::PE0, tcl::PE0_L, o, i, v); break;
      case J_PE1: put_w<TF32>(wp, lay::GRP_B + lay::PE1_W + i * 32 + o, v); put_tc<TF32>(wt, tcl::PE1, tcl::PE1_L, o, i, v); break;
      case J_RD0: put_w<TF32>(wp, lay::GRP_B + lay::RD0_W + i * 16 + o, v); break;
      case J_RD1: put_w<TF32>(wp, lay::GRP_B + lay::RD1_W + i * 36 + o, v); put_tc<TF32>(wt, tcl::RD1, tcl::RD1_L, o, i, v); break;
      case J_NF0: put_w<TF32>(wp, lay::GRP_B + lay::NF0_W + i * 8 + o, v); break;
      case J_NF1: put_w<TF32>(wp, lay::GRP_B + lay::NF1_W + i, v); break;
      case J_B0: {   // base_fc.0 [64,207] = [view-pooled 140 | rgb_feat 35 | neuray_feat 32]
        if (i < 140) {
          put_w<TF32>(wp, lay::HOIST_W + i * 64 + o, v);
          const int s = i / 35, f = i - 35 * s, r = f >> 3, q = f & 7;        // stat, feature -> K = 32 r + 8 s + q
          put_tc<TF32>(wt, tcl::HST, tcl::HST_L, o, 32 * r + 8 * s + q, v);
        } else {
          put_w<TF32>(wp, lay::BASE0_W + (i - 140) * 64 + o, v);
          const int k = i < 175 ? i - 140 : 40 + (i - 175);                    // rgb_feat 35 | bias | 4 zeros | neuray_feat 32
          put_tc<TF32>(wt, tcl::B0, tcl::B0_L, o, k, v);
        }
        break;
      }
      case J_B1: put_w<TF32>(wp, lay::BASE1_W + i * 32 + o, v); put_tc<TF32>(wt, tcl::B1, tcl::B1_L, o, i, v); break;
      case J_V0: put_w<TF32>(wp, lay::GRP_D1 + lay::VIS0_W + i * 32 + o, v); put_tc<TF32>(wt, tcl::V01, tcl::VIS0_L, o, i, v); break;
      case J_V1:
        if (o < 32) { put_w<TF32>(wp, lay::GRP_D1 + lay::VIS1_W + i * 32 + o, v); put_tc<TF32>(wt, tcl::V01, tcl::VIS2_L, o, i, v); }
        else put_w<TF32>(wp, lay::GRP_D1 + lay::VIS1L_W + i, v);
        break;
      case J_V20: put_w<TF32>(wp, lay::GRP_D1 + lay::V20_W + i * 32 + o, v); put_tc<TF32>(wt, tcl::V2R, tcl::V20_L, o, i, v); break;
      case J_V21: put_w<TF32>(wp, lay::GRP_D1 + lay::V21_W + i, v); break;
      case J_C0: put_w<TF32>(wp, lay::GRP_D1 + lay::RGB0_W + i * 16 + o, v); put_tc<TF32>(wt, tcl::V2R, tcl::RGB0_L, o, i, v); break;
      case J_C1: put_w<TF32>(wp, lay::GRP_D1 + lay::RGB1_W + i * 8 + o, v); break;
      case J_C2: put_w<TF32>(wp, lay::GRP_D1 + lay::RGB2_W + i, v); break;
      case J_G0: {   // geometry_fc.0 [64,65] = [mean 32 | var 32 | mean weight]
        put_w<TF32>(wp, lay::GRP_D2 + lay::GEO0_W + i * 64 + o, v);
        int k;
        if (i < 64) { const int s = i >> 5, f = i & 31, r = f >> 4, q = f & 15; k = 32 * r + 16 * s + q; }
        else k = 64;
        put_tc<TF32>(wt, tcl::G0, tcl::G0_L, o, k, v);
        break;
      }
      case J_G1: put_w<TF32>(wp, lay::GRP_D2 + lay::GEO1_W + i * 16 + o, v); break;
      case J_OG0: put_w<TF32>(wr, lay::OG0_W + i * 16 + o, v); break;
      case J_OG1: put_w<TF32>(wr, lay::OG1_W + i, v); break;
      case J_WQ: put_w<TF32>(wr, lay::WQ + i * 16 + o, v); break;
      case J_WK: put_w<TF32>(wr, lay::WK + i * 16 + o, v); break;
      case J_WV: put_w<TF32>(wr, lay::WV + i * 16 + o, v); break;
      case J_WFC: put_w<TF32>(wr, lay::WFC + i * 16 + o, v); break;
      case J_LNW: put_w<TF32>(wr, lay::LN_W + e, v); break;
      case J_LNB: put_w<TF32>(wr, lay::LN_B + e, v); break;
      default: break;
    }
  }
  // biases
  if (J.b == nullptr) return;
  for (int o = threadIdx.x; o < J.n_out; o += blockDim.x) {
    const float v = J.b[o];
    if (job < 12) {
      const int h = job / 3, l = job - 3 * h;
      const int base = lay::DD_HEAD + h * lay::DD_HEAD_STRIDE;
      put_w<TF32>(wp, base + (l == 0 ? lay::DD_L0_B : l == 1 ? lay::DD_L1_B : lay::DD_L2_B) + o, v);
      continue;
    }
    switch (job) {
      case J_PE0: put_w<TF32>(wp, lay::GRP_B + lay::PE0_B + o, v); break;
      case J_PE1: put_w<TF32>(wp, lay::GRP_B + lay::PE1_B + o, v); break;
      case J_RD0: put_w<TF32>(wp, lay::GRP_B + lay::RD0_B + o, v); break;
      case J_RD1: put_w<TF32>(wp, lay::GRP_B + lay::RD1_B + o, v); break;
      case J_NF0: put_w<TF32>(wp, lay::GRP_B + lay::NF0_B + o, v); break;
      case J_NF1: put_w<TF32>(wp, lay::GRP_B + lay::NF1_B + o, v); break;
      case J_B0: put_w<TF32>(wp, lay::HOIST_B + o, v); put_tc<TF32>(wt, tcl::B0, tcl::B0_L, o, 35, v); break;   // bias = column 35 (constant-1 input)
      case J_B1: put_w<TF32>(wp, lay::BASE1_B + o, v); break;
      case J_V0: put_w<TF32>(wp, lay::GRP_D1 + lay::VIS0_B + o, v); break;
      case J_V1: put_w<TF32>(wp, lay::GRP_D1 + (o < 32 ? lay::VIS1_B + o : lay::VIS1L_B), v); break;
      case J_V20: put_w<TF32>(wp, lay::GRP_D1 + lay::V20_B + o, v); break;
      case J_V21: put_w<TF32>(wp, lay::GRP_D1 + lay::V21_B + o, v); break;
      case J_C0: put_w<TF32>(wp, lay::GRP_D1 + lay::RGB0_B + o, v); break;
      case J_C1: put_w<TF32>(wp, lay::GRP_D1 + lay::RGB1_B + o, v); break;
      case J_C2: put_w<TF32>(wp, lay::GRP_D1 + lay::RGB2_B + o, v); break;
      case J_G0: put_w<TF32>(wp, lay::GRP_D2 + lay::GEO0_B + o, v); put_tc<TF32>(wt, tcl::G0, tcl::G0_L, o, 65, v); break;   // bias = column 65
      case J_G1: put_w<TF32>(wp, lay::GRP_D2 + lay::GEO1_B + o, v); break;
      case J_OG0: put_w<TF32>(wr, lay::OG0_B + o, v); break;
      case J_OG1: put_w<TF32>(wr, lay::OG1_B + o, v); break;
      default: break;
    }
  }
}

// ---- camera blocks ---------------------------------------------------------------------------------------------
// que_cam [24] = R^T (9) | centre (3) | K^-1 (9) | near, far, 0   (reference render_ops.py:14-20)
// view_params [rfn,20] = K@Rt (12) | centre (3) | -1/near, -1/far | pad (3)   (render_ops.py:95,112; dist_decoder.py:17-20)
// The small matrix products and the 3x3 inverse are evaluated in fp64 and rounded once to fp32: within half an ulp of the
// exact value, i.e. at least as close to it as the reference's own fp32 matmul / LU inverse are.
__device__ void centre_of(const float* __restrict__ pose, double* c) {   // -R^T t
  for (int i = 0; i < 3; ++i)
    c[i] = -(double(pose[0 * 4 + i]) * double(pose[3]) + double(pose[1 * 4 + i]) * double(pose[7]) + double(pose[2 * 4 + i]) * double(pose[11]));
}

__global__ void camera_blocks_kernel(const float* __restrict__ que_pose, const float* __restrict__ que_K, const float* __restrict__ que_range,
                                     const float* __restrict__ ref_poses, const float* __restrict__ ref_Ks, const float* __restrict__ ref_range,
                                     int rfn, float* __restrict__ que_cam, float* __restrict__ view_params) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t == 0 && que_cam != nullptr) {
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) que_cam[3 * i + j] = que_pose[4 * j + i];
    double c[3];
    centre_of(que_pose, c);
    for (int i = 0; i < 3; ++i) que_cam[9 + i] = float(c[i]);
    double k[9], inv[9];
    for (int i = 0; i < 9; ++i) k[i] = double(que_K[i]);
    const double det = k[0] * (k[4] * k[8] - k[5] * k[7]) - k[1] * (k[3] * k[8] - k[5] * k[6]) + k[2] * (k[3] * k[7] - k[4] * k[6]);
    inv[0] = (k[4] * k[8] - k[5] * k[7]) / det; inv[1] = (k[2] * k[7] - k[1] * k[8]) / det; inv[2] = (k[1] * k[5] - k[2] * k[4]) / det;
    inv[3] = (k[5] * k[6] - k[3] * k[8]) / det; inv[4] = (k[0] * k[8] - k[2] * k[6]) / det; inv[5] = (k[2] * k[3] - k[0] * k[5]) / det;
    inv[6] = (k[3] * k[7] - k[4] * k[6]) / det; inv[7] = (k[1] * k[6] - k[0] * k[7]) / det; inv[8] = (k[0] * k[4] - k[1] * k[3]) / det;
    for (int i = 0; i < 9; ++i) que_cam[12 + i] = float(inv[i]);
    que_cam[21] = que_range ? que_range[0] : 0.f;
    que_cam[22] = que_range ? que_range[1] : 0.f;
    que_cam[23] = 0.f;
  }
  if (t < rfn && view_params != nullptr) {
    const float* __restrict__ P = ref_poses + 12 * t;
    const float* __restrict__ K = ref_Ks + 9 * t;
    float* __restrict__ o = view_params + 20 * t;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 4; ++j)
        o[4 * i + j] = float(double(K[3 * i]) * double(P[j]) + double(K[3 * i + 1]) * double(P[4 + j]) + double(K[3 * i + 2]) * double(P[8 + j]));
    double c[3];
    centre_of(P, c);
    for (int i = 0; i < 3; ++i) o[12 + i] = float(c[i]);
    o[15] = ref_range ? -1.f / ref_range[2 * t] : 0.f;
    o[16] = ref_range ? -1.f / ref_range[2 * t + 1] : 0.f;
    o[17] = o[18] = o[19] = 0.f;
  }
}

}  // namespace pack
}  // namespace nr

using namespace nr;

// The job table of a pass, checked; tf32: only w_tc, for the TF32 point kernel
static int pack_pass(const NrPassWeights* w, float* w_point, float* w_ray, float* w_tc, bool tf32, cudaStream_t s) {
  pack::Jobs jobs;
  auto set = [&](int j, const NrLinear& l, int n_out, int n_in) { jobs.j[j] = pack::Job{l.w, l.b, n_out, n_in}; };
  for (int h = 0; h < 4; ++h) {
    const int outs = h < 2 ? 2 : 1;
    set(pack::J_DD + 3 * h + 0, w->dist_decoder[h][0], 32, 32);
    set(pack::J_DD + 3 * h + 1, w->dist_decoder[h][1], 32, 32);
    set(pack::J_DD + 3 * h + 2, w->dist_decoder[h][2], outs, 32);
    const bool any = w->dist_decoder[h][0].w || w->dist_decoder[h][1].w || w->dist_decoder[h][2].w;
    for (int l = 0; l < 3; ++l)
      NR_CHECK_ARG(!any || (w->dist_decoder[h][l].w && w->dist_decoder[h][l].b), "dist decoder head: all three layers (weight and bias) or none");
    NR_CHECK_ARG(h == 3 || any, "mean / var / aw decoder heads are required");
  }
  set(pack::J_PE0, w->prob_embed[0], 32, 34);
  set(pack::J_PE1, w->prob_embed[1], 32, 32);
  set(pack::J_RD0, w->ray_dir_fc[0], 16, 4);
  set(pack::J_RD1, w->ray_dir_fc[1], 35, 16);
  set(pack::J_NF0, w->neuray_fc[0], 8, 32);
  set(pack::J_NF1, w->neuray_fc[1], 1, 8);
  set(pack::J_B0, w->base_fc[0], 64, 207);
  set(pack::J_B1, w->base_fc[1], 32, 64);
  set(pack::J_V0, w->vis_fc[0], 32, 32);
  set(pack::J_V1, w->vis_fc[1], 33, 32);
  set(pack::J_V20, w->vis_fc2[0], 32, 32);
  set(pack::J_V21, w->vis_fc2[1], 1, 32);
  set(pack::J_C0, w->rgb_fc[0], 16, 37);
  set(pack::J_C1, w->rgb_fc[1], 8, 16);
  set(pack::J_C2, w->rgb_fc[2], 1, 8);
  set(pack::J_G0, w->geometry_fc[0], 64, 65);
  set(pack::J_G1, w->geometry_fc[1], 16, 64);
  set(pack::J_OG0, w->out_geometry_fc[0], 16, 16);
  set(pack::J_OG1, w->out_geometry_fc[1], 1, 16);
  for (int j = pack::J_PE0; j <= pack::J_OG1; ++j) NR_CHECK_ARG(jobs.j[j].w && jobs.j[j].b, "aggregation net: every Linear needs weight and bias");
  NR_CHECK_ARG(w->w_qs && w->w_ks && w->w_vs && w->attn_fc && w->layer_norm_w && w->layer_norm_b, "ray attention parameters");
  jobs.j[pack::J_WQ] = pack::Job{w->w_qs, nullptr, 16, 16};
  jobs.j[pack::J_WK] = pack::Job{w->w_ks, nullptr, 16, 16};
  jobs.j[pack::J_WV] = pack::Job{w->w_vs, nullptr, 16, 16};
  jobs.j[pack::J_WFC] = pack::Job{w->attn_fc, nullptr, 16, 16};
  jobs.j[pack::J_LNW] = pack::Job{w->layer_norm_w, nullptr, 16, 1};
  jobs.j[pack::J_LNB] = pack::Job{w->layer_norm_b, nullptr, 16, 1};
  jobs.j[pack::J_COMP] = pack::Job{w->neuray_fc[0].w, w->prob_embed[1].w, 8, 32};
  if (tf32) {
    cudaMemsetAsync(w_tc, 0, sizeof(float) * tcl::TOTAL, s);
    pack::pack_weights_kernel<true><<<pack::NJOBS, 256, 0, s>>>(jobs, pack::Out{nullptr, nullptr, w_tc});
    NR_CHECK_LAUNCH("pack_weights_tf32");
    return NR_OK;
  }
  cudaMemsetAsync(w_point, 0, sizeof(float) * lay::TOTAL_POINT, s);
  cudaMemsetAsync(w_ray, 0, sizeof(float) * lay::TOTAL_RAY, s);
  cudaMemsetAsync(w_tc, 0, sizeof(float) * tcl::TOTAL, s);
  pack::pack_weights_kernel<false><<<pack::NJOBS, 256, 0, s>>>(jobs, pack::Out{w_point, w_ray, w_tc});
  NR_CHECK_LAUNCH("pack_weights");
  return NR_OK;
}

extern "C" {

int nr_pack_weights(const NrPassWeights* w, float* w_point, float* w_ray, float* w_tc, void* stream) {
  NR_CHECK_ARG(w != nullptr && w_point != nullptr && w_ray != nullptr && w_tc != nullptr, "null pointer");
  return pack_pass(w, w_point, w_ray, w_tc, false, (cudaStream_t)stream);
}

int nr_pack_weights_tf32(const NrPassWeights* w, float* w_tc, void* stream) {
  NR_CHECK_ARG(w != nullptr && w_tc != nullptr, "null pointer");
  return pack_pass(w, nullptr, nullptr, w_tc, true, (cudaStream_t)stream);
}

int nr_camera_blocks(const float* que_pose, const float* que_K, const float* que_range, const float* ref_poses, const float* ref_Ks,
                     const float* ref_range, int rfn, float* que_cam, float* view_params, void* stream) {
  NR_CHECK_ARG(que_cam == nullptr || (que_pose && que_K), "query pose / intrinsics");
  NR_CHECK_ARG(view_params == nullptr || (ref_poses && ref_Ks && rfn >= 1 && rfn <= (1 << 20)), "reference poses / intrinsics");
  NR_CHECK_ARG(que_cam || view_params, "nothing to do");
  const int n = view_params ? rfn : 1;
  pack::camera_blocks_kernel<<<(n + 63) / 64, 64, 0, (cudaStream_t)stream>>>(que_pose, que_K, que_range, ref_poses, ref_Ks, ref_range,
                                                                          view_params ? rfn : 0, que_cam, view_params);
  NR_CHECK_LAUNCH("camera_blocks");
  return NR_OK;
}

}  // extern "C"
