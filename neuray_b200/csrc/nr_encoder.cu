// Encoders upstream of the ray path on the GPU (SURVEY.md 8(f) row f1): kernels for the building blocks of nr_conv.cuh, the
// stream backend of the layer graphs of nr_encoder_graph.cuh, and the C-ABI entry points (include/neuray_b200.h).
#include "nr_encoder_graph.cuh"
#include "nr_tc.cuh"

namespace nr {
namespace cv {

// FAST = one TF32 pass per product (operands rounded to TF32: ~1e-3 relative, torch's default for cuDNN convolutions);
// otherwise the 3xTF32 split (fp32 accuracy, what the parity tests run)
template <int BM, int BN, int KC, bool FAST>
__global__ void __launch_bounds__(THREADS, BN >= 128 ? 1 : 2) conv_mma_kernel(const __grid_constant__ ConvP p) {
  extern __shared__ __align__(16) float sm[];
  constexpr int MT = mt_of(BM, BN), WN = BN / 32, STAGES = stages_of(BM);
  static_assert(MT >= 1 && MT <= 4 && MT * 16 * (8 / WN) == BM, "tile shape");
  constexpr int A_ST = BM * (KC + 4), B_ST = KC * (BN + 8), ST = A_ST + B_ST;
  constexpr int A_ROWS = THREADS / (KC / 4);      // rows of the A tile one pass of the 256 threads covers
  constexpr int A_PASSES = BM / A_ROWS;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int warp_m = warp / WN, warp_n = warp - warp_m * WN;
  const long long m0 = (long long)blockIdx.x * BM;
  const int nk = p.ks * p.ks * (p.Cin / KC);
  const int a_row = tid / (KC / 4), a_c4 = (tid - a_row * (KC / 4)) * 4;
  RowInfo ri[A_PASSES];
#pragma unroll
  for (int j = 0; j < A_PASSES; ++j) ri[j] = row_info(p, m0 + a_row + j * A_ROWS);

  auto stage = [&](int kt, int slot) {
    float* A = sm + slot * ST;
    float* B = A + A_ST;
#pragma unroll
    for (int j = 0; j < A_PASSES; ++j) {
      int dst;
      const float* src;
      a_chunk<KC>(p, ri[j], a_row + j * A_ROWS, a_c4, kt, dst, src);
      tc::cp_async16_zfill(A + dst, src != nullptr ? src : p.x, src != nullptr);
    }
    for (int idx = tid; idx < KC * BN / 4; idx += THREADS) {
      int dst;
      const float* src;
      b_chunk<BN, KC>(p, idx, kt, dst, src);
      tc::cp_async16_zfill(B + dst, src, true);
    }
  };

  float acc[MT][4][4];
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < nk) stage(s, s);
    tc::cp_async_commit();
  }
  for (int kt = 0; kt < nk; ++kt) {
    tc::cp_async_wait<STAGES - 2>();  // this thread's copies of step kt have landed ...
    __syncthreads();                  // ... and everybody's; everybody is also done with the slot refilled next
    if (kt + STAGES - 1 < nk) stage(kt + STAGES - 1, (kt + STAGES - 1) % STAGES);
    tc::cp_async_commit();
    const float* A = sm + (kt % STAGES) * ST;
    const float* B = A + A_ST;
    // The tensor cores add into their fp32 accumulator with truncation (measured: 1e-7 of the running sum per MMA, always
    // toward zero, i.e. 4e-5 after the 432 chained MMAs of a K = 1152 layer).  A K step therefore accumulates from zero
    // (12 MMAs on a partial sum ~1/sqrt(steps) of the total) and is added to the running sum with a rounding FADD.
    float part[MT][4][4];
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) part[i][j][e] = 0.f;
#pragma unroll
    for (int k8 = 0; k8 < KC / 8; ++k8) {
      uint32_t ah[MT][4], al[FAST ? 1 : MT][4], bh[4][2], bl[FAST ? 1 : 4][2];
#pragma unroll
      for (int i = 0; i < MT; ++i) {
        int off[4];
        a_frag<KC>(warp_m * (16 * MT) + 16 * i, lane, k8, off);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if constexpr (FAST) ah[i][e] = tc::tf32_rna(A[off[e]]);
          else tc::split_tf32(A[off[e]], ah[i][e], al[i][e]);
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int off[2];
        b_frag<BN>(warp_n * 32 + 8 * j, lane, k8, off);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          if constexpr (FAST) bh[j][e] = tc::tf32_rna(B[off[e]]);
          else tc::split_tf32(B[off[e]], bh[j][e], bl[j][e]);
        }
      }
#pragma unroll
      for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if constexpr (!FAST) {
            tc::mma_tf32_m16n8k8(part[i][j], al[i], bh[j]);      // small terms first
            tc::mma_tf32_m16n8k8(part[i][j], ah[i], bl[j]);
          }
          tc::mma_tf32_m16n8k8(part[i][j], ah[i], bh[j]);
        }
    }
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[i][j][e] += part[i][j][e];
  }
  tc::cp_async_wait<0>();

  // InstanceNorm sums: thread partials -> the 8 row lanes of a warp (shuffles) -> the CTA (shared memory) -> ONE fp64 atomic
  // per (column, sum) and CTA.  Thousands of CTAs adding to the same 2 x Cout addresses of an image serialise in L2: with one
  // atomic per warp the large-CTA-count layers spent most of their time on them.
  __shared__ double cta_sums[2 * 128];
  const long long M = (long long)p.N * p.Ho * p.Wo;
  const long long plane = (long long)p.Ho * p.Wo;
  const long long last_row = m0 + BM - 1 < M ? m0 + BM - 1 : M - 1;
  const bool cta_uniform = p.stats != nullptr && m0 / plane == last_row / plane;      // all rows of the CTA in one image
  if (cta_uniform) {
    for (int i = tid; i < 2 * BN; i += THREADS) cta_sums[i] = 0.0;
    __syncthreads();
  }
  const bool uniform = warp_rows_uniform<BM, BN>(p, m0, warp);
  float s[4][2], q[4][2];
  epilogue_thread<BM, BN>(p, m0, warp, lane, acc, uniform, s, q);
  if (p.stats != nullptr && uniform) {
    const long long first = m0 + warp_m * (16 * MT);
    if (first < M) {                  // warp-uniform
      const int n = int(first / plane);
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          double sd = double(s[j][b]), qd = double(q[j][b]);
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {      // over the 8 row lanes g (lane = 4 g + t4)
            sd += __shfl_xor_sync(0xffffffffu, sd, o);
            qd += __shfl_xor_sync(0xffffffffu, qd, o);
          }
          if ((lane >> 2) == 0) {
            const int col = warp_n * 32 + 8 * j + 2 * (lane & 3) + b;
            if (cta_uniform) {
              atomicAdd(&cta_sums[2 * col], sd);
              atomicAdd(&cta_sums[2 * col + 1], qd);
            } else {
              double* st = p.stats + ((long long)n * BN + col) * 2;
              atomicAdd(st, sd);
              atomicAdd(st + 1, qd);
            }
          }
        }
    }
  }
  if (cta_uniform) {
    __syncthreads();
    const int n = int(m0 / plane);
    for (int i = tid; i < 2 * BN; i += THREADS) atomicAdd(p.stats + (long long)n * BN * 2 + i, cta_sums[i]);
  }
}

template <int COUT>
__global__ void __launch_bounds__(256) conv7_kernel(const __grid_constant__ Conv7P p) {
  __shared__ __align__(16) float w[147 * COUT];
  for (int i = threadIdx.x; i < 147 * COUT; i += 256) w[i] = p.w[i];
  __syncthreads();
  const int n = blockIdx.y, pix = blockIdx.x * 256 + threadIdx.x;
  const bool valid = pix < p.Ho * p.Wo;
  float out[COUT];
#pragma unroll
  for (int c = 0; c < COUT; ++c) out[c] = 0.f;
  if (valid) {
    conv7_pixel<COUT>(p, w, n, pix, out);
    float4* o = reinterpret_cast<float4*>(p.y + ((long long)n * p.Ho * p.Wo + pix) * COUT);
#pragma unroll
    for (int c = 0; c < COUT / 4; ++c) o[c] = make_float4(out[4 * c], out[4 * c + 1], out[4 * c + 2], out[4 * c + 3]);
  }
  // InstanceNorm sums of the block's pixels (one image per blockIdx.y): warp sums in fp32 -> block sums in shared memory ->
  // one fp64 atomic per channel, sum and block
  __shared__ double cta_sums[2 * COUT];
  if (threadIdx.x < 2 * COUT) cta_sums[threadIdx.x] = 0.0;
  __syncthreads();
#pragma unroll
  for (int c = 0; c < COUT; ++c) {
    float sv = out[c], qv = out[c] * out[c];
    sv = warp_sum(sv);
    qv = warp_sum(qv);
    if ((threadIdx.x & 31) == 0) {
      atomicAdd(&cta_sums[2 * c], double(sv));
      atomicAdd(&cta_sums[2 * c + 1], double(qv));
    }
  }
  __syncthreads();
  if (threadIdx.x < 2 * COUT) atomicAdd(p.stats + (long long)n * 2 * COUT + threadIdx.x, cta_sums[threadIdx.x]);
}

__global__ void __launch_bounds__(256) norm_act_kernel(const __grid_constant__ NormP p) {
  __shared__ float sc[128], sh[128], rsc[128], rsh[128];
  const int n = blockIdx.y;
  for (int c = threadIdx.x; c < p.C; c += 256) {
    if (p.stats != nullptr) norm_coeffs(p.stats, p.gamma, p.beta, n, c, p.C, p.HW, p.eps, sc[c], sh[c]);
    else { sc[c] = 1.f; sh[c] = 0.f; }
    if (p.res != nullptr && p.res_stats != nullptr) norm_coeffs(p.res_stats, p.res_gamma, p.res_beta, n, c, p.C, p.HW, p.eps, rsc[c], rsh[c]);
    else { rsc[c] = 1.f; rsh[c] = 0.f; }
  }
  __syncthreads();
  const int c4n = p.C / 4;
  const long long total = (long long)p.HW * c4n;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long pix = i / c4n;
    const int c = int(i - pix * c4n) * 4;
    const long long m = (long long)n * p.HW + pix;
    const float4 v = *reinterpret_cast<const float4*>(p.x + m * p.x_stride + p.x_off + c);
    float o[4] = {v.x * sc[c] + sh[c], v.y * sc[c + 1] + sh[c + 1], v.z * sc[c + 2] + sh[c + 2], v.w * sc[c + 3] + sh[c + 3]};
    if (p.res != nullptr) {
      const float4 r = *reinterpret_cast<const float4*>(p.res + m * p.res_stride + p.res_off + c);
      o[0] += r.x * rsc[c] + rsh[c]; o[1] += r.y * rsc[c + 1] + rsh[c + 1]; o[2] += r.z * rsc[c + 2] + rsh[c + 2]; o[3] += r.w * rsc[c + 3] + rsh[c + 3];
    }
    *reinterpret_cast<float4*>(p.y + m * p.y_stride + p.y_off + c) =
        make_float4(act_f(o[0], p.act), act_f(o[1], p.act), act_f(o[2], p.act), act_f(o[3], p.act));
  }
}

__global__ void __launch_bounds__(256) upsample_kernel(const __grid_constant__ UpP p) {
  const int c4n = p.C / 4;
  const long long total = (long long)p.N * p.Ho * p.Wo * c4n;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long pix = i / c4n;
    const int c = int(i - pix * c4n) * 4;
    const int xo = int(pix % p.Wo);
    const long long t = pix / p.Wo;
    const int yo = int(t % p.Ho), n = int(t / p.Ho);
    int y0, y1, x0, x1;
    float ly0, ly1, lx0, lx1;
    up_taps(yo, p.H, p.Ho, y0, y1, ly0, ly1);
    up_taps(xo, p.W, p.Wo, x0, x1, lx0, lx1);
    const float* base = p.x + (long long)n * p.H * p.W * p.x_stride + p.x_off + c;
    const float4 a = *reinterpret_cast<const float4*>(base + ((long long)y0 * p.W + x0) * p.x_stride);
    const float4 b = *reinterpret_cast<const float4*>(base + ((long long)y0 * p.W + x1) * p.x_stride);
    const float4 cc = *reinterpret_cast<const float4*>(base + ((long long)y1 * p.W + x0) * p.x_stride);
    const float4 d = *reinterpret_cast<const float4*>(base + ((long long)y1 * p.W + x1) * p.x_stride);
    float4 o;
    o.x = ly0 * (lx0 * a.x + lx1 * b.x) + ly1 * (lx0 * cc.x + lx1 * d.x);
    o.y = ly0 * (lx0 * a.y + lx1 * b.y) + ly1 * (lx0 * cc.y + lx1 * d.y);
    o.z = ly0 * (lx0 * a.z + lx1 * b.z) + ly1 * (lx0 * cc.z + lx1 * d.z);
    o.w = ly0 * (lx0 * a.w + lx1 * b.w) + ly1 * (lx0 * cc.w + lx1 * d.w);
    *reinterpret_cast<float4*>(p.y + pix * p.y_stride + p.y_off + c) = o;
  }
}

__global__ void __launch_bounds__(256) copy_pad_kernel(const __grid_constant__ enc::CopyP p) {
  const int c4n = p.C / 4;
  const long long total = (long long)p.N * p.Ho * p.Wo * c4n;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long pix = i / c4n;
    const int c = int(i - pix * c4n) * 4;
    const int xo = int(pix % p.Wo);
    const long long t = pix / p.Wo;
    const int yo = int(t % p.Ho), n = int(t / p.Ho);
    const int yi = yo - p.py, xi = xo - p.px;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (yi >= 0 && yi < p.H && xi >= 0 && xi < p.W)
      v = *reinterpret_cast<const float4*>(p.x + (((long long)n * p.H + yi) * p.W + xi) * p.x_stride + p.x_off + c);
    *reinterpret_cast<float4*>(p.y + pix * p.y_stride + p.y_off + c) = v;
  }
}

// [N,C,H,W] -> channels [y_off, y_off + C) of a channel-last buffer
__global__ void __launch_bounds__(256) nchw_to_nhwc_kernel(const float* __restrict__ x, float* __restrict__ y, int N, int C, long long HW, int y_stride,
                                                           int y_off) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z, c0 = blockIdx.y * 32;
  const long long p0 = (long long)blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;     // 32 x 8
  for (int r = ty; r < 32; r += 8) {
    const int c = c0 + r;
    const long long pix = p0 + tx;
    tile[r][tx] = (c < C && pix < HW) ? x[((long long)n * C + c) * HW + pix] : 0.f;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const long long pix = p0 + r;
    const int c = c0 + tx;
    if (c < C && pix < HW) y[((long long)n * HW + pix) * y_stride + y_off + c] = tile[tx][r];
  }
}
// channels [x_off, x_off + C) of a channel-last buffer -> [N,C,H,W]
__global__ void __launch_bounds__(256) nhwc_to_nchw_kernel(const float* __restrict__ x, float* __restrict__ y, int N, int C, long long HW, int x_stride,
                                                           int x_off) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z, c0 = blockIdx.y * 32;
  const long long p0 = (long long)blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int r = ty; r < 32; r += 8) {
    const long long pix = p0 + r;
    const int c = c0 + tx;
    tile[r][tx] = (c < C && pix < HW) ? x[((long long)n * HW + pix) * x_stride + x_off + c] : 0.f;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int c = c0 + r;
    const long long pix = p0 + tx;
    if (c < C && pix < HW) y[((long long)n * C + c) * HW + pix] = tile[tx][r];
  }
}

__global__ void __launch_bounds__(256) depth_skip_kernel(const __grid_constant__ DepthSkipP p) {
  const long long total = (long long)p.N * p.Ho * p.Wo;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int xo = int(i % p.Wo);
    const long long t = i / p.Wo;
    const int yo = int(t % p.Ho), n = int(t / p.Ho);
    float out[16];
    depth_skip_pixel(p, n, yo, xo, out);
    float4* o = reinterpret_cast<float4*>(p.y + i * p.y_stride + p.y_off);
#pragma unroll
    for (int c = 0; c < 4; ++c) o[c] = make_float4(out[4 * c], out[4 * c + 1], out[4 * c + 2], out[4 * c + 3]);
  }
}

// extract_depth_for_init_impl (init_net.py:63-74): metric depth -> normalised inverse depth in [0, 1], per view
__global__ void __launch_bounds__(256) extract_depth_kernel(const float* __restrict__ depth, const float* __restrict__ range, int N, long long HW,
                                                            float* __restrict__ out) {
  const long long total = (long long)N * HW;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int n = int(i / HW);
    const float a = -1.f / range[2 * n], b = -1.f / range[2 * n + 1];
    const float d = -1.f / fmaxf(depth[i], 1e-5f);
    out[i] = fminf(fmaxf((d - a) / (b - a), 0.f), 1.f);
  }
}

struct PackJob {
  enc::TensorSpec spec;
  const float* src;
};
struct PackArgs {
  PackJob job[160];
  int count;
  float* out;
};
__global__ void __launch_bounds__(256) pack_params_kernel(const __grid_constant__ PackArgs a) {
  const PackJob& j = a.job[blockIdx.y];
  for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < j.spec.n; e += (long long)gridDim.x * 256)
  {
    const long long src = enc::pack_source(j.spec, e);
    a.out[j.spec.off + e] = src >= 0 ? j.src[src] : 0.f;
  }
}

template <int BM, int BN, int KC, bool FAST>
int launch_conv_f(const ConvP& p, cudaStream_t st) {
  constexpr size_t smem = size_t(stages_of(BM)) * (BM * (KC + 4) + KC * (BN + 8)) * sizeof(float);
  if (opt_in_smem((const void*)conv_mma_kernel<BM, BN, KC, FAST>, smem, "conv_mma_kernel") != NR_OK) return NR_E_CUDA;
  const long long M = (long long)p.N * p.Ho * p.Wo;
  conv_mma_kernel<BM, BN, KC, FAST><<<unsigned((M + BM - 1) / BM), THREADS, smem, st>>>(p);
  NR_CHECK_LAUNCH("conv_mma_kernel");
  return NR_OK;
}
template <int BM, int BN, int KC>
int launch_conv_t(const ConvP& p, cudaStream_t st) {
  return p.tf32x1 ? launch_conv_f<BM, BN, KC, true>(p, st) : launch_conv_f<BM, BN, KC, false>(p, st);
}
template <int BM, int BN>
int launch_conv_k(const ConvP& p, cudaStream_t st) {
  return p.Cin % 32 == 0 ? launch_conv_t<BM, BN, 32>(p, st) : launch_conv_t<BM, BN, 16>(p, st);
}

int check_conv(const ConvP& p) {
  NR_CHECK_ARG(p.x != nullptr && p.w != nullptr && p.y != nullptr, "conv: null pointer");
  NR_CHECK_ARG(p.Cout == 32 || p.Cout == 64 || p.Cout == 128, "conv: Cout must be 32, 64 or 128");
  NR_CHECK_ARG(p.Cin >= 16 && p.Cin % 16 == 0, "conv: Cin must be a multiple of 16");
  NR_CHECK_ARG(p.ks >= 1 && p.ks <= 8, "conv: kernel size 1 .. 8");
  NR_CHECK_ARG(p.stride == 1 || p.stride == 2, "conv: stride 1 or 2");
  NR_CHECK_ARG(p.pad >= 0 && p.pad < p.ks && p.pad < p.H && p.pad < p.W, "conv: padding (one reflection: pad < H, W)");
  NR_CHECK_ARG(p.N >= 1 && p.H >= 2 && p.W >= 2 && p.Ho >= 1 && p.Wo >= 1, "conv: empty input");
  NR_CHECK_ARG(p.x_stride % 4 == 0 && p.x_off % 4 == 0 && p.y_stride % 2 == 0 && p.y_off % 2 == 0, "conv: channel strides / offsets must keep 16-byte alignment");
  NR_CHECK_ARG(p.res == nullptr || (p.res_stride % 2 == 0 && p.res_off % 2 == 0), "conv: residual alignment");
  return NR_OK;
}

int launch_conv(const ConvP& p, cudaStream_t st) {
  const int rc = check_conv(p);
  if (rc != NR_OK) return rc;
  int sms = 0;
  if (p.bm == 0 && sm_count(&sms, "conv") != NR_OK) return NR_E_CUDA;
  const int bm = p.bm != 0 ? p.bm : pick_bm(p.Cout, (long long)p.N * p.Ho * p.Wo, sms);
  switch (p.Cout) {
    case 32:
      NR_CHECK_ARG(bm == 128 || bm == 256, "conv: 128 or 256 pixels per CTA for 32 outputs");
      return bm == 256 ? launch_conv_k<256, 32>(p, st) : launch_conv_k<128, 32>(p, st);
    case 64:
      NR_CHECK_ARG(bm == 64 || bm == 128, "conv: 64 or 128 pixels per CTA for 64 outputs");
      return bm == 64 ? launch_conv_k<64, 64>(p, st) : launch_conv_k<128, 64>(p, st);
    default:
      NR_CHECK_ARG(bm == 64 || bm == 128, "conv: 64 or 128 pixels per CTA for 128 outputs");
      return bm == 64 ? launch_conv_k<64, 128>(p, st) : launch_conv_k<128, 128>(p, st);
  }
}

inline unsigned grid_for(long long items, int cap) {
  long long g = (items + 255) / 256;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return unsigned(g);
}

// stream backend of the layer graphs
struct StreamOps {
  cudaStream_t st;
  int sms;
  int rc;
  int tf32x1;
  void conv(const ConvP& p) {
    if (rc != NR_OK) return;
    ConvP q = p;
    q.tf32x1 = tf32x1;
    q.bm = 0;
    rc = launch_conv(q, st);
  }
  void conv7(const Conv7P& p) {
    if (rc != NR_OK) return;
    const dim3 grid(unsigned((p.Ho * p.Wo + 255) / 256), p.N);
    if (p.Cout == 16) conv7_kernel<16><<<grid, 256, 0, st>>>(p);
    else conv7_kernel<32><<<grid, 256, 0, st>>>(p);
  }
  void norm(const NormP& p) {
    if (rc != NR_OK) return;
    norm_act_kernel<<<dim3(grid_for((long long)p.HW * (p.C / 4), (8 * sms + p.N - 1) / p.N), p.N), 256, 0, st>>>(p);
  }
  void upsample(const UpP& p) {
    if (rc != NR_OK) return;
    upsample_kernel<<<grid_for((long long)p.N * p.Ho * p.Wo * (p.C / 4), 16 * sms), 256, 0, st>>>(p);
  }
  void copy_pad(const enc::CopyP& p) {
    if (rc != NR_OK) return;
    copy_pad_kernel<<<grid_for((long long)p.N * p.Ho * p.Wo * (p.C / 4), 16 * sms), 256, 0, st>>>(p);
  }
  void depth_skip(const DepthSkipP& p) {
    if (rc != NR_OK) return;
    depth_skip_kernel<<<grid_for((long long)p.N * p.Ho * p.Wo, 16 * sms), 256, 0, st>>>(p);
  }
  void zero(void* ptr, size_t bytes) {
    if (rc != NR_OK) return;
    cudaMemsetAsync(ptr, 0, bytes, st);
  }
};

int pack_params(const enc::NetSpec& spec, const float* const* params, int n_params, float* packed, cudaStream_t st) {
  NR_CHECK_ARG(params != nullptr && packed != nullptr, "pack: null pointer");
  NR_CHECK_ARG(n_params == spec.count, "pack: wrong number of parameter tensors (state_dict order, see include/neuray_b200.h)");
  PackArgs a;
  a.count = spec.count;
  a.out = packed;
  long long biggest = 0;
  for (int i = 0; i < spec.count; ++i) {
    NR_CHECK_ARG(params[i] != nullptr, "pack: null parameter tensor");
    a.job[i].spec = spec.t[i];
    a.job[i].src = params[i];
    if (spec.t[i].n > biggest) biggest = spec.t[i].n;
  }
  cudaMemsetAsync(packed, 0, size_t(spec.total) * sizeof(float), st);
  pack_params_kernel<<<dim3(grid_for(biggest, 64), spec.count), 256, 0, st>>>(a);
  NR_CHECK_LAUNCH("pack_params_kernel");
  return NR_OK;
}

}  // namespace cv
}  // namespace nr

using namespace nr;

extern "C" int nr_encoder_layout(NrEncoderLayout* out) {
  NR_CHECK_ARG(out != nullptr, "null layout");
  enc::ImageNet in;
  enc::VisNet vn;
  enc::build_image_net(in);
  enc::build_vis_net(vn);
  out->image_tensors = in.spec.count;
  out->image_packed_floats = in.spec.total;
  out->vis_tensors = vn.spec.count;
  out->vis_packed_floats = vn.spec.total;
  enc::DepthInitNet* dn = new enc::DepthInitNet;
  enc::build_depth_init_net(*dn);
  out->depth_init_tensors = dn->res.spec.count;
  out->depth_init_packed_floats = dn->res.spec.total;
  delete dn;
  return NR_OK;
}

extern "C" int nr_image_encoder_dims(int h, int w, int* fh, int* fw) {
  NR_CHECK_ARG(h >= 32 && w >= 32 && fh != nullptr && fw != nullptr, "image_encoder_dims");
  const enc::ImageDims d = enc::image_dims(h, w);
  *fh = d.u2h;
  *fw = d.u2w;
  return NR_OK;
}

extern "C" long long nr_image_encoder_workspace(int n, int h, int w) {
  if (n < 1 || h < 32 || w < 32) return 0;
  enc::ImageNet net;
  enc::build_image_net(net);
  return (long long)enc::image_workspace_bytes(net, n, h, w);
}
extern "C" long long nr_vis_encoder_workspace(int n, int fh, int fw) {
  if (n < 1 || fh < 2 || fw < 2) return 0;
  enc::VisNet net;
  enc::build_vis_net(net);
  return (long long)enc::vis_workspace_bytes(net, n, fh, fw);
}

extern "C" int nr_image_encoder_pack(const float* const* params, int n_params, float* packed, void* stream) {
  enc::ImageNet net;
  enc::build_image_net(net);
  return cv::pack_params(net.spec, params, n_params, packed, (cudaStream_t)stream);
}
extern "C" int nr_vis_encoder_pack(const float* const* params, int n_params, float* packed, void* stream) {
  enc::VisNet net;
  enc::build_vis_net(net);
  return cv::pack_params(net.spec, params, n_params, packed, (cudaStream_t)stream);
}

extern "C" int nr_image_encoder_fwd(const float* packed, const float* imgs, int n, int h, int w, float* out, int out_stride, int out_off,
                                    int tf32x1, void* workspace, long long workspace_bytes, void* stream) {
  if (n == 0) return NR_OK;
  NR_CHECK_ARG(packed != nullptr && imgs != nullptr && out != nullptr && workspace != nullptr, "image_encoder: null pointer");
  NR_CHECK_ARG(n >= 1 && h >= 32 && w >= 32, "image_encoder: images must be at least 32 x 32");
  NR_CHECK_ARG(out_stride >= 32 && out_stride % 4 == 0 && out_off % 4 == 0 && out_off + 32 <= out_stride, "image_encoder: output channel slot");
  enc::ImageNet net;
  enc::build_image_net(net);
  const long long stats = enc::image_stats_doubles(net, n, h, w);
  NR_CHECK_ARG(stats > 0, "image_encoder: image size the decoder's skip connections cannot take (ops.py:199-208)");
  int sms;
  if (sm_count(&sms, "image_encoder") != NR_OK) return NR_E_CUDA;
  enc::Arena ar{(char*)workspace, size_t(workspace_bytes), 0, true};
  cv::StreamOps ops{(cudaStream_t)stream, sms, NR_OK, tf32x1 != 0};
  const bool ok = enc::image_encoder_graph(ops, ar, net, packed, imgs, n, h, w, out, out_stride, out_off, stats, nullptr);
  if (ops.rc != NR_OK) return ops.rc;
  NR_CHECK_ARG(ok, "image_encoder: workspace too small (nr_image_encoder_workspace)");
  NR_CHECK_LAUNCH("image_encoder");
  return NR_OK;
}

extern "C" int nr_vis_encoder_fwd(const float* packed, float* feat, int n, int fh, int fw, int tf32x1, void* workspace, long long workspace_bytes,
                                  void* stream) {
  if (n == 0) return NR_OK;
  NR_CHECK_ARG(packed != nullptr && feat != nullptr && workspace != nullptr, "vis_encoder: null pointer");
  NR_CHECK_ARG(n >= 1 && fh >= 2 && fw >= 2, "vis_encoder: empty maps");
  enc::VisNet net;
  enc::build_vis_net(net);
  const long long stats = enc::vis_stats_doubles(net, n, fh, fw);
  int sms;
  if (sm_count(&sms, "vis_encoder") != NR_OK) return NR_E_CUDA;
  enc::Arena ar{(char*)workspace, size_t(workspace_bytes), 0, true};
  cv::StreamOps ops{(cudaStream_t)stream, sms, NR_OK, tf32x1 != 0};
  const bool ok = enc::vis_encoder_graph(ops, ar, net, packed, feat, n, fh, fw, stats, nullptr);
  if (ops.rc != NR_OK) return ops.rc;
  NR_CHECK_ARG(ok, "vis_encoder: workspace too small (nr_vis_encoder_workspace)");
  NR_CHECK_LAUNCH("vis_encoder");
  return NR_OK;
}

extern "C" int nr_extract_depth(const float* depth, const float* depth_range, int n, int h, int w, float* out, void* stream) {
  if (n == 0) return NR_OK;
  NR_CHECK_ARG(depth && depth_range && out && n >= 1 && h >= 1 && w >= 1, "extract_depth");
  int sms;
  if (sm_count(&sms, "extract_depth") != NR_OK) return NR_E_CUDA;
  const long long hw = (long long)h * w;
  cv::extract_depth_kernel<<<cv::grid_for((long long)n * hw, 16 * sms), 256, 0, (cudaStream_t)stream>>>(depth, depth_range, n, hw, out);
  NR_CHECK_LAUNCH("extract_depth_kernel");
  return NR_OK;
}

extern "C" int nr_depth_init_dims(int h, int w, int* fh, int* fw) {
  NR_CHECK_ARG(h >= 32 && w >= 32 && fh != nullptr && fw != nullptr, "depth_init_dims");
  const enc::ImageDims d = enc::depth_init_dims(h, w);
  *fh = d.u2h;
  *fw = d.u2w;
  return NR_OK;
}
extern "C" long long nr_depth_init_workspace(int n, int h, int w) {
  if (n < 1 || h < 32 || w < 32) return 0;
  enc::DepthInitNet* net = new enc::DepthInitNet;
  enc::build_depth_init_net(*net);
  const long long bytes = (long long)enc::depth_init_workspace_bytes(*net, n, h, w) + ((long long)n * h * w * 16 * 4 + 256);   // + the 16-channel input
  delete net;
  return bytes;
}
extern "C" int nr_depth_init_pack(const float* const* params, int n_params, float* packed, void* stream) {
  enc::DepthInitNet* net = new enc::DepthInitNet;
  enc::build_depth_init_net(*net);
  const int rc = cv::pack_params(net->res.spec, params, n_params, packed, (cudaStream_t)stream);
  delete net;
  return rc;
}
extern "C" int nr_depth_init_fwd(const float* packed, const float* imgs, const float* depth_norm, const float* diff_feats, int n, int h, int w,
                                 float* out, int out_stride, int out_off, int tf32x1, void* workspace, long long workspace_bytes, void* stream) {
  if (n == 0) return NR_OK;
  NR_CHECK_ARG(packed && imgs && depth_norm && diff_feats && out && workspace, "depth_init: null pointer");
  NR_CHECK_ARG(n >= 1 && h >= 32 && w >= 32, "depth_init: images must be at least 32 x 32");
  NR_CHECK_ARG(out_stride >= 32 && out_stride % 4 == 0 && out_off % 4 == 0 && out_off + 32 <= out_stride, "depth_init: output channel slot");
  int sms;
  if (sm_count(&sms, "depth_init") != NR_OK) return NR_E_CUDA;
  enc::DepthInitNet* net = new enc::DepthInitNet;
  enc::build_depth_init_net(*net);
  const long long stats = enc::depth_init_stats_doubles(*net, n, h, w);
  int rc = NR_OK;
  bool ok = false;
  if (stats > 0) {
    enc::Arena ar{(char*)workspace, size_t(workspace_bytes), 0, true};
    cudaStream_t st = (cudaStream_t)stream;
    // the 12 input channels of ResEncoder.conv1 (init_net.py:98: cat([imgs, depth, diff_feats])) channel-last, padded to 16
    const long long hw = (long long)h * w;
    float* x16 = ar.floats((long long)n * hw * 16);
    if (ar.ok) {
      cudaMemsetAsync(x16, 0, size_t(n) * hw * 16 * sizeof(float), st);
      cv::nchw_to_nhwc_kernel<<<dim3(unsigned((hw + 31) / 32), 1, n), 256, 0, st>>>(imgs, x16, n, 3, hw, 16, 0);
      cv::nchw_to_nhwc_kernel<<<dim3(unsigned((hw + 31) / 32), 1, n), 256, 0, st>>>(depth_norm, x16, n, 1, hw, 16, 3);
      cv::nchw_to_nhwc_kernel<<<dim3(unsigned((hw + 31) / 32), 1, n), 256, 0, st>>>(diff_feats, x16, n, 8, hw, 16, 4);
      cv::StreamOps ops{st, sms, NR_OK, tf32x1 != 0};
      ok = enc::depth_init_graph(ops, ar, *net, packed, x16, depth_norm, n, h, w, out, out_stride, out_off, stats, nullptr);
      rc = ops.rc;
    }
  }
  delete net;
  if (rc != NR_OK) return rc;
  NR_CHECK_ARG(stats > 0, "depth_init: image size whose depth_skip and ResEncoder outputs differ (init_net.py:101 would fail too)");
  NR_CHECK_ARG(ok, "depth_init: workspace too small (nr_depth_init_workspace)");
  NR_CHECK_LAUNCH("depth_init");
  return NR_OK;
}

extern "C" int nr_cost_volume_head_layout(int cost_volume_sn, int* n_tensors, long long* packed_floats) {
  NR_CHECK_ARG(n_tensors && packed_floats && cost_volume_sn >= 16 && cost_volume_sn % 16 == 0, "cost_volume_head_layout");
  enc::CostVolumeHead* net = new enc::CostVolumeHead;
  enc::build_cost_volume_head(*net, cost_volume_sn);
  *n_tensors = net->res.spec.count;
  *packed_floats = net->res.spec.total;
  delete net;
  return NR_OK;
}
extern "C" int nr_cost_volume_head_pack(int cost_volume_sn, const float* const* params, int n_params, float* packed, void* stream) {
  NR_CHECK_ARG(cost_volume_sn >= 16 && cost_volume_sn % 16 == 0, "cost_volume_head_pack: cost_volume_sn must be a multiple of 16");
  enc::CostVolumeHead* net = new enc::CostVolumeHead;
  enc::build_cost_volume_head(*net, cost_volume_sn);
  const int rc = cv::pack_params(net->res.spec, params, n_params, packed, (cudaStream_t)stream);
  delete net;
  return rc;
}
extern "C" long long nr_cost_volume_head_workspace(int cost_volume_sn, int n, int h, int w) {
  if (n < 1 || h < 32 || w < 32 || cost_volume_sn < 16 || cost_volume_sn % 16 != 0) return 0;
  enc::CostVolumeHead* net = new enc::CostVolumeHead;
  enc::build_cost_volume_head(*net, cost_volume_sn);
  const enc::ImageDims d = enc::image_dims(h, w);
  const long long bytes = (long long)enc::cv_head_workspace_bytes(*net, n, h, w, d.u2h, d.u2w) + ((long long)n * d.u2h * d.u2w * 16 * 4 + 256);
  delete net;
  return bytes;
}
extern "C" int nr_cost_volume_head_fwd(int cost_volume_sn, const float* packed, const float* imgs, const float* prob, const float* depth_norm, int n,
                                       int h, int w, float* out, int out_stride, int out_off, int tf32x1, void* workspace, long long workspace_bytes,
                                       void* stream) {
  if (n == 0) return NR_OK;
  NR_CHECK_ARG(packed && imgs && prob && depth_norm && out && workspace, "cost_volume_head: null pointer");
  NR_CHECK_ARG(n >= 1 && h >= 32 && w >= 32 && cost_volume_sn >= 16 && cost_volume_sn % 16 == 0, "cost_volume_head: shape");
  NR_CHECK_ARG(out_stride >= 32 && out_stride % 4 == 0 && out_off % 4 == 0 && out_off + 32 <= out_stride, "cost_volume_head: output channel slot");
  int sms;
  if (sm_count(&sms, "cost_volume_head") != NR_OK) return NR_E_CUDA;
  enc::CostVolumeHead* net = new enc::CostVolumeHead;
  enc::build_cost_volume_head(*net, cost_volume_sn);
  const enc::ImageDims d = enc::image_dims(h, w);
  const long long stats = enc::cv_head_stats_doubles(*net, n, h, w, d.u2h, d.u2w);
  int rc = NR_OK;
  bool ok = false;
  if (stats > 0) {
    enc::Arena ar{(char*)workspace, size_t(workspace_bytes), 0, true};
    cudaStream_t st = (cudaStream_t)stream;
    const long long hw = (long long)d.u2h * d.u2w;
    float* d16 = ar.floats((long long)n * hw * 16);          // depth_conv's single input channel packed into 16 (zero weight rows for the rest)
    if (ar.ok) {
      cudaMemsetAsync(d16, 0, size_t(n) * hw * 16 * sizeof(float), st);
      cv::nchw_to_nhwc_kernel<<<dim3(unsigned((hw + 31) / 32), 1, n), 256, 0, st>>>(depth_norm, d16, n, 1, hw, 16, 0);
      cv::StreamOps ops{st, sms, NR_OK, tf32x1 != 0};
      ok = enc::cost_volume_head_graph(ops, ar, *net, packed, imgs, prob, cost_volume_sn, d16, n, h, w, d.u2h, d.u2w, out, out_stride, out_off, stats, nullptr);
      rc = ops.rc;
    }
  }
  delete net;
  if (rc != NR_OK) return rc;
  NR_CHECK_ARG(stats > 0, "cost_volume_head: image size the decoder's skip connections cannot take");
  NR_CHECK_ARG(ok, "cost_volume_head: workspace too small (nr_cost_volume_head_workspace)");
  NR_CHECK_LAUNCH("cost_volume_head");
  return NR_OK;
}

/* ---- single building blocks (tests, and hosts that run other conv stacks) ---- */
extern "C" int nr_conv2d_nhwc(const NrConv2d* c, void* stream) {
  NR_CHECK_ARG(c != nullptr, "null conv descriptor");
  cv::ConvP p;
  p.x = c->x; p.w = c->w_packed; p.bias = c->bias; p.res = c->res; p.y = c->y; p.stats = c->stats;
  p.N = c->n; p.H = c->h; p.W = c->w; p.Cin = c->cin; p.Cout = c->cout; p.ks = c->ks; p.stride = c->stride; p.reflect = c->reflect;
  NR_CHECK_ARG(p.ks >= 1 && p.ks <= 8, "conv: kernel size 1 .. 8");
  NR_CHECK_ARG(p.stride == 1 || p.stride == 2, "conv: stride 1 or 2");
  p.pad = c->pad >= 0 ? c->pad : (p.ks - 1) / 2;
  p.Ho = enc::conv_out(p.H, p.ks, p.stride, p.pad); p.Wo = enc::conv_out(p.W, p.ks, p.stride, p.pad);
  p.x_stride = c->x_stride; p.x_off = c->x_off; p.y_stride = c->y_stride; p.y_off = c->y_off; p.res_stride = c->res_stride; p.res_off = c->res_off;
  p.tf32x1 = c->tf32x1 != 0;
  p.bm = c->bm;
  if (p.N == 0) return NR_OK;
  return cv::launch_conv(p, (cudaStream_t)stream);
}

extern "C" int nr_conv_pack_weight(const float* w, int cout, int cin, int ks, int cin_rot, float* packed, void* stream) {
  NR_CHECK_ARG(w != nullptr && packed != nullptr && cout >= 1 && cin >= 1 && ks >= 1 && ks <= 7 && cin_rot >= 0, "conv_pack_weight");
  enc::NetSpec* spec = new enc::NetSpec;
  spec->count = 0; spec->total = 0;
  spec->conv(cout, cin, ks, cin_rot, 0);
  const float* params[1] = {w};
  const int rc = cv::pack_params(*spec, params, 1, packed, (cudaStream_t)stream);
  delete spec;
  return rc;
}

extern "C" int nr_instance_norm_act(const float* x, const double* stats, const float* gamma, const float* beta, const float* res,
                                    const double* res_stats, const float* res_gamma, const float* res_beta, int n, int hw, int c, int act, float* y,
                                    void* stream) {
  if (n == 0) return NR_OK;
  NR_CHECK_ARG(x != nullptr && y != nullptr && stats != nullptr, "instance_norm_act: null pointer");
  NR_CHECK_ARG(c >= 4 && c <= 128 && c % 4 == 0 && hw >= 1 && act >= 0 && act <= 2, "instance_norm_act: C must be a multiple of 4, at most 128");
  cv::NormP p;
  p.x = x; p.stats = stats; p.gamma = gamma; p.beta = beta; p.res = res; p.res_stats = res_stats; p.res_gamma = res_gamma; p.res_beta = res_beta;
  p.y = y; p.N = n; p.HW = hw; p.C = c; p.act = act; p.x_stride = c; p.x_off = 0; p.res_stride = c; p.res_off = 0; p.y_stride = c; p.y_off = 0;
  p.eps = 1e-5f;
  int sms;
  if (sm_count(&sms, "instance_norm_act") != NR_OK) return NR_E_CUDA;
  cv::StreamOps ops{(cudaStream_t)stream, sms, NR_OK, 0};
  ops.norm(p);
  NR_CHECK_LAUNCH("norm_act_kernel");
  return NR_OK;
}

extern "C" int nr_nchw_to_nhwc(const float* x, int n, int c, int h, int w, float* y, int y_stride, int y_off, void* stream) {
  if (n == 0) return NR_OK;
  NR_CHECK_ARG(x != nullptr && y != nullptr && c >= 1 && h >= 1 && w >= 1 && y_stride >= c + y_off && y_off >= 0, "nchw_to_nhwc");
  const long long hw = (long long)h * w;
  cv::nchw_to_nhwc_kernel<<<dim3(unsigned((hw + 31) / 32), (c + 31) / 32, n), 256, 0, (cudaStream_t)stream>>>(x, y, n, c, hw, y_stride, y_off);
  NR_CHECK_LAUNCH("nchw_to_nhwc_kernel");
  return NR_OK;
}
extern "C" int nr_nhwc_to_nchw(const float* x, int n, int c, int h, int w, int x_stride, int x_off, float* y, void* stream) {
  if (n == 0) return NR_OK;
  NR_CHECK_ARG(x != nullptr && y != nullptr && c >= 1 && h >= 1 && w >= 1 && x_stride >= c + x_off && x_off >= 0, "nhwc_to_nchw");
  const long long hw = (long long)h * w;
  cv::nhwc_to_nchw_kernel<<<dim3(unsigned((hw + 31) / 32), (c + 31) / 32, n), 256, 0, (cudaStream_t)stream>>>(x, y, n, c, hw, x_stride, x_off);
  NR_CHECK_LAUNCH("nhwc_to_nchw_kernel");
  return NR_OK;
}
