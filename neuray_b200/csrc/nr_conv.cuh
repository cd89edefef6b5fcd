// Convolution building blocks of the encoders upstream of the ray path (SURVEY.md 8(f) row f1):
//   image_encoder = ResUNetLight(3, [1,2,6,4], 32, inplanes=16)   reference network/ops.py:150-230, renderer.py:59
//   vis_encoder   = DefaultVisEncoder                              reference network/vis_encoder.py:6-21
// Everything is channel-last (NHWC) so that the last layers write straight into the [rfn,fh,fw,64] frame pack the point
// kernel gathers from (no NCHW -> NHWC repack, no 148 MB upload in a frame loop).
//
// conv_mma_kernel: implicit GEMM, M = output pixels (linear over n, y, x), N = Cout (whole, 32 / 64 / 128), K = taps x Cin,
// walked in (tap, KC-channel) steps.  A step's A tile (128 pixels x KC channels, each pixel's chunk one contiguous
// 4*KC-byte read of the NHWC input, reflect / zero padding resolved per row) and B tile (KC x Cout of the packed
// [tap][cin][cout] weights) arrive through a 3-stage cp.async ring; the product runs on the tensor cores as warp-level
// m16n8k8 TF32 MMAs with the 3xTF32 split (hi*hi + lo*hi + hi*lo), i.e. fp32 accuracy: the oracle is the fp32 reference.
// The epilogue adds bias / a residual, stores the raw output and accumulates the InstanceNorm statistics (sum, sum of
// squares per (image, channel)) in fp64 atomics, so a normalisation never re-reads its input for the statistics.
//
// The index math lives in __host__ __device__ helpers: tests/cpu_harness/conv_cpu_harness.cu emulates a CTA on the host
// (staging, fragment gathers, the documented m16n8k8 fragment layout, epilogue) and checks it against torch's conv2d.
#pragma once
#include <math.h>

#include "nr_common.cuh"

#ifndef NR_HD
#define NR_HD __host__ __device__ __forceinline__
#endif

namespace nr {
namespace cv {

constexpr int THREADS = 256;   // 8 warps: WM = 8 / WN along M x WN = Cout / 32 along N; a warp owns 16*MT pixels x 32 channels
// Output pixels per CTA: BM in {64, 128, 256}, MT = BM / (16 WM) m16 tiles per warp.  128 is the default; 64 for Cout = 128 when
// 128-pixel tiles would leave a nearly empty last wave (layer3 of an 800x800 frame: 157 tiles on 132 SMs); 256 for Cout = 32,
// where a warp otherwise owns a single m16 tile and re-reads / re-splits the whole weight tile for 12 MMAs (2 pipeline stages
// instead of 3, so that two CTAs still fit an SM).
__host__ __device__ constexpr int mt_of(int BM, int BN) { return BM / (16 * (8 / (BN / 32))); }
__host__ __device__ constexpr int stages_of(int BM) { return BM > 128 ? 2 : 3; }

struct ConvP {
  const float* x;       // input: pixel (n, y, x) channel c at x[((n*H + y)*W + x) * x_stride + x_off + c]
  const float* w;       // packed [ks*ks][Cin][Cout]
  const float* bias;    // [Cout] or null
  const float* res;     // residual added before the store / the statistics, output geometry, or null
  float* y;             // output: pixel m (linear) channel c at y[m * y_stride + y_off + c]
  double* stats;        // [N][Cout][2]: sum, sum of squares (accumulated; the caller zeroes it) or null
  int N, H, W, Ho, Wo, Cin, Cout, ks, stride, pad, reflect;
  int x_stride, x_off, y_stride, y_off, res_stride, res_off;
  int bm;               // output pixels per CTA: 0 = chosen by the launcher, else 64 / 128 / 256 (tests force every variant)
  int tf32x1;           // 0: 3xTF32 (fp32 accuracy, the default); 1: one TF32 pass, what cuDNN does under torch's default allow_tf32
};

// tile height the launcher uses when p.bm == 0: slots = CTAs the device runs at once for this Cout
NR_HD int pick_bm(int Cout, long long M, int sms) {
  if (Cout == 32) return M >= 2LL * 256 * sms ? 256 : 128;
  if (Cout == 128) {
    const long long w128 = (M + 128LL * sms - 1) / (128LL * sms), w64 = (M + 64LL * sms - 1) / (64LL * sms);
    return w64 * 64 < w128 * 128 ? 64 : 128;          // rows an SM works through, one CTA per SM either way
  }
  return 128;
}

struct RowInfo {
  int n, y0, x0;        // image (-1: row beyond the last pixel), input coordinates of tap (0, 0)
};

NR_HD RowInfo row_info(const ConvP& p, long long m) {
  RowInfo r;
  const long long M = (long long)p.N * p.Ho * p.Wo;
  if (m >= M) { r.n = -1; r.y0 = 0; r.x0 = 0; return r; }
  const int plane = p.Ho * p.Wo;
  r.n = int(m / plane);
  const int rem = int(m - (long long)r.n * plane);
  const int yo = rem / p.Wo, xo = rem - yo * p.Wo;
  r.y0 = yo * p.stride - p.pad;
  r.x0 = xo * p.stride - p.pad;
  return r;
}

// linear input pixel of a row for one tap, -1 = zeros (zero padding or a row beyond the end)
NR_HD long long src_pixel(const ConvP& p, const RowInfo& r, int tap) {
  if (r.n < 0) return -1;
  const int dy = tap / p.ks, dx = tap - dy * p.ks;
  int yi = r.y0 + dy, xi = r.x0 + dx;
  if (p.reflect) {   // padding_mode='reflect': -1 -> 1, H -> H-2 (one reflection: pad < H)
    yi = yi < 0 ? -yi : (yi >= p.H ? 2 * (p.H - 1) - yi : yi);
    xi = xi < 0 ? -xi : (xi >= p.W ? 2 * (p.W - 1) - xi : xi);
  } else if (yi < 0 || yi >= p.H || xi < 0 || xi >= p.W) {
    return -1;
  }
  return ((long long)r.n * p.H + yi) * p.W + xi;
}

// 16-byte chunk idx of the A tile of K step kt: destination (floats inside the A stage) and source (null = zero fill)
template <int KC>
NR_HD void a_chunk(const ConvP& p, const RowInfo& r, int row, int c4, int kt, int& dst, const float*& src) {
  const int kchunks = p.Cin / KC;
  const int tap = kt / kchunks, c0 = (kt - tap * kchunks) * KC;
  const long long pix = src_pixel(p, r, tap);
  dst = row * (KC + 4) + c4;
  src = pix < 0 ? nullptr : p.x + pix * p.x_stride + p.x_off + c0 + c4;
}
// 16-byte chunk idx of the B tile: row k (channel c0 + k of the tap), columns n4..n4+3
template <int BN, int KC>
NR_HD void b_chunk(const ConvP& p, int idx, int kt, int& dst, const float*& src) {
  const int kchunks = p.Cin / KC;
  const int tap = kt / kchunks, c0 = (kt - tap * kchunks) * KC;
  const int k = idx / (BN / 4), n4 = (idx - k * (BN / 4)) * 4;
  dst = k * (BN + 8) + n4;
  src = p.w + ((long long)(tap * p.Cin + c0 + k)) * BN + n4;
}

// fragment element offsets (floats) of mma.m16n8k8: lane = 4 g + t4
//   A (16 x 8, row):  a0 (g, t4)  a1 (g + 8, t4)  a2 (g, t4 + 4)  a3 (g + 8, t4 + 4)       banks (KC+4) g + t4: distinct
//   B (8 x 8, col):   b0 (k = t4, n = g)  b1 (k = t4 + 4, n = g)                            banks 8 t4 + g: distinct
//   C (16 x 8):       c0 (g, 2 t4)  c1 (g, 2 t4 + 1)  c2 (g + 8, 2 t4)  c3 (g + 8, 2 t4 + 1)
template <int KC>
NR_HD void a_frag(int row0, int lane, int k8, int (&off)[4]) {
  const int g = lane >> 2, t4 = lane & 3;
  off[0] = (row0 + g) * (KC + 4) + 8 * k8 + t4;
  off[1] = (row0 + g + 8) * (KC + 4) + 8 * k8 + t4;
  off[2] = off[0] + 4;
  off[3] = off[1] + 4;
}
template <int BN>
NR_HD void b_frag(int col0, int lane, int k8, int (&off)[2]) {
  const int g = lane >> 2, t4 = lane & 3;
  off[0] = (8 * k8 + t4) * (BN + 8) + col0 + g;
  off[1] = (8 * k8 + t4 + 4) * (BN + 8) + col0 + g;
}

NR_HD void atomic_add_f64(double* p, double v) {
#ifdef __CUDA_ARCH__
  atomicAdd(p, v);
#else
  *p += v;
#endif
}

// Epilogue of one thread: its accumulators (MT m-tiles x 4 n-tiles x 4) -> y (+ bias, + residual), and the thread's share of
// the InstanceNorm sums.  When all rows of the warp lie in one image (`uniform`), the per-column partial sums come back in
// s / q (the caller reduces them over the 8 row lanes and issues one atomic per column); otherwise every element is added
// on its own.
template <int BM, int BN>
NR_HD void epilogue_thread(const ConvP& p, long long m0, int warp, int lane, const float (&acc)[mt_of(BM, BN)][4][4], bool uniform,
                           float (&s)[4][2], float (&q)[4][2]) {
  constexpr int MT = mt_of(BM, BN), WN = BN / 32;
  const int g = lane >> 2, t4 = lane & 3;
  const int warp_m = warp / WN, warp_n = warp - warp_m * WN;
  const long long M = (long long)p.N * p.Ho * p.Wo;
  const int plane = p.Ho * p.Wo;
#pragma unroll
  for (int j = 0; j < 4; ++j) { s[j][0] = s[j][1] = q[j][0] = q[j][1] = 0.f; }
#pragma unroll
  for (int i = 0; i < MT; ++i) {
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const long long m = m0 + warp_m * (16 * MT) + 16 * i + g + 8 * hf;
      if (m >= M) continue;
      const int n = int(m / plane);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = warp_n * 32 + 8 * j + 2 * t4;
        float v0 = acc[i][j][2 * hf], v1 = acc[i][j][2 * hf + 1];
        if (p.bias != nullptr) { v0 += p.bias[col]; v1 += p.bias[col + 1]; }
        if (p.res != nullptr) {
          const float* r = p.res + m * p.res_stride + p.res_off + col;
          v0 += r[0]; v1 += r[1];
        }
        float* o = p.y + m * p.y_stride + p.y_off + col;
        o[0] = v0; o[1] = v1;
        if (p.stats != nullptr) {
          if (uniform) {
            s[j][0] += v0; s[j][1] += v1; q[j][0] += v0 * v0; q[j][1] += v1 * v1;
          } else {
            double* st = p.stats + ((long long)n * BN + col) * 2;
            atomic_add_f64(st, v0); atomic_add_f64(st + 1, double(v0) * v0);
            atomic_add_f64(st + 2, v1); atomic_add_f64(st + 3, double(v1) * v1);
          }
        }
      }
    }
  }
}

// all valid rows of the warp's 16*MT rows in one image?
template <int BM, int BN>
NR_HD bool warp_rows_uniform(const ConvP& p, long long m0, int warp) {
  constexpr int MT = mt_of(BM, BN), WN = BN / 32;
  const long long M = (long long)p.N * p.Ho * p.Wo;
  const long long first = m0 + (warp / WN) * (16 * MT);
  long long last = first + 16 * MT - 1;
  if (last >= M) last = M - 1;
  if (first >= M) return true;
  const int plane = p.Ho * p.Wo;
  return first / plane == last / plane;
}

// ---- first layer: 7x7 stride-2 reflect conv of the NCHW image (Cin 3 -> COUT = 16 | 32), one thread per output pixel -----
struct Conv7P {
  const float* img;     // [N,3,H,W] (the reference's layout, read as is)
  const float* w;       // packed [147][Cout]  (tap-major: (c*7 + dy)*7 + dx)
  float* y;             // [N,Ho,Wo,Cout]
  double* stats;        // [N][Cout][2]
  int N, H, W, Ho, Wo, Cout;
};
NR_HD int reflect_idx(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * (n - 1) - i : i); }

template <int COUT>
NR_HD void conv7_pixel(const Conv7P& p, const float* w, int n, int pix, float (&out)[COUT]) {
  const int yo = pix / p.Wo, xo = pix - yo * p.Wo;
#pragma unroll
  for (int c = 0; c < COUT; ++c) out[c] = 0.f;
  for (int c = 0; c < 3; ++c) {
    const float* im = p.img + ((long long)n * 3 + c) * p.H * p.W;
    for (int dy = 0; dy < 7; ++dy) {
      const int yi = reflect_idx(2 * yo - 3 + dy, p.H);
      for (int dx = 0; dx < 7; ++dx) {
        const int xi = reflect_idx(2 * xo - 3 + dx, p.W);
        const float v = im[(long long)yi * p.W + xi];
        const float* wr = w + ((c * 7 + dy) * 7 + dx) * COUT;
#pragma unroll
        for (int o = 0; o < COUT; ++o) out[o] = fmaf(v, wr[o], out[o]);
      }
    }
  }
}

// ---- InstanceNorm (+ residual, + activation) over a raw conv output ------------------------------------------------
// y = act( IN(x) * gamma + beta  [+ res | + IN(res) * res_gamma + res_beta] ),  reference ops.py:104-124 (BasicBlock),
// :137 (conv: ELU), ResidualBlock :47-53.  act: 0 none, 1 ReLU, 2 ELU.
struct NormP {
  const float* x; const double* stats; const float* gamma; const float* beta;
  const float* res; const double* res_stats; const float* res_gamma; const float* res_beta;
  float* y;
  int N, HW, C, act;
  int x_stride, x_off, res_stride, res_off, y_stride, y_off;
  float eps;
};
// scale / shift of channel c of image n: IN(x) * gamma + beta = x * scale + shift  (biased variance, like F.instance_norm)
NR_HD void norm_coeffs(const double* stats, const float* gamma, const float* beta, int n, int c, int C, int HW, float eps, float& scale,
                       float& shift) {
  const double* st = stats + ((long long)n * C + c) * 2;
  const double mean = st[0] / HW;
  double var = st[1] / HW - mean * mean;
  if (var < 0.0) var = 0.0;
  const double rstd = 1.0 / sqrt(var + double(eps));
  const double g = gamma != nullptr ? double(gamma[c]) : 1.0, b = beta != nullptr ? double(beta[c]) : 0.0;
  scale = float(rstd * g);
  shift = float(b - mean * rstd * g);
}
NR_HD float act_f(float v, int act) {
  if (act == 1) return v > 0.f ? v : 0.f;
  if (act == 2) return v > 0.f ? v : expm1f(v);
  return v;
}

// ---- DepthInitNet.depth_skip (init_net.py:85-89): Conv2d(1,8,2,2) ReLU Conv2d(8,16,2,2) on the normalised depth map -----------
struct DepthSkipP {
  const float* depth;   // [N,H,W]
  const float* w0; const float* b0;   // [8][1][2][2], [8]
  const float* w1; const float* b1;   // [16][8][2][2], [16]
  float* y;             // channels [y_off, y_off + 16) of [N,Ho,Wo,y_stride], Ho = (H/2)/2
  int N, H, W, Ho, Wo, y_stride, y_off;
};
NR_HD void depth_skip_pixel(const DepthSkipP& p, int n, int yo, int xo, float (&out)[16]) {
  for (int o = 0; o < 16; ++o) out[o] = p.b1[o];
  const float* d = p.depth + (long long)n * p.H * p.W;
  for (int py = 0; py < 2; ++py)
    for (int px = 0; px < 2; ++px) {          // the four outputs of the first conv under this output pixel
      const int y1 = 2 * yo + py, x1 = 2 * xo + px;
      float h[8];
      for (int c = 0; c < 8; ++c) {
        float a = p.b0[c];
        for (int ky = 0; ky < 2; ++ky)
          for (int kx = 0; kx < 2; ++kx) a = fmaf(p.w0[(c * 2 + ky) * 2 + kx], d[(long long)(2 * y1 + ky) * p.W + 2 * x1 + kx], a);
        h[c] = a > 0.f ? a : 0.f;
      }
      for (int o = 0; o < 16; ++o)
        for (int c = 0; c < 8; ++c) out[o] = fmaf(p.w1[((o * 8 + c) * 2 + py) * 2 + px], h[c], out[o]);
    }
}

// ---- bilinear x2 upsampling, align_corners=True (reference ops.py:147, nn.functional.interpolate) ----------------
struct UpP {
  const float* x; float* y;
  int N, H, W, Ho, Wo, C, x_stride, x_off, y_stride, y_off;
};
NR_HD void up_taps(int o, int n_in, int n_out, int& i0, int& i1, float& l0, float& l1) {
  const float scale = n_out > 1 ? float(n_in - 1) / float(n_out - 1) : 0.f;
  const float r = scale * float(o);
  i0 = int(r);
  if (i0 > n_in - 1) i0 = n_in - 1;
  i1 = i0 + (i0 < n_in - 1 ? 1 : 0);
  l1 = r - float(i0);
  l0 = 1.f - l1;
}

}  // namespace cv
}  // namespace nr
