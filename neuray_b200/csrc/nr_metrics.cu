// Validation image metrics (reference network/metrics.py:13-79, PSNR_SSIM with skimage's structural_similarity(win_size=11,
// data_range=255) and compute_psnr): one ground truth against up to NR_METRICS_MAX_PRED predictions per call.
//
// Every input is quantised to an integer 0..255 first (color_map_backward), so the 11x11 window sums of x, y, x^2, y^2 and xy
// are exact in int32 (at most 121 * 65025) and the squared errors are exact integers.  Only the SSIM term itself is floating
// point (fp64).  Its per-block sums are written to the workspace and added up by a second kernel in a fixed order: the result
// is the same bit for bit from run to run, with no floating-point atomics.
//
// The reference's eval.py scores rendered frames with its own definitions, also here: tf.image.psnr / tf.image.ssim on
// color_map_forward'ed uint8 pairs (nr_eval_metrics: Gaussian windows, VALID region, fp64) and LPIPS-VGG (nr_lpips_vgg_*:
// vgg16 on the nr_conv2d_nhwc building block, one fused kernel per tap).  Both reduce in a fixed order as well.
#include <utility>

#include "nr_metrics_math.cuh"

namespace nr {
namespace mt {

constexpr int TW = 32, TH = 32;                            // SSIM-map pixels per block
constexpr int LW = TW + 2 * HALF, LH = TH + 2 * HALF;      // the block's input tile with its halo
constexpr int THREADS = 256;

struct Partial {
  double ssim[3];        // sum of the SSIM map over the block's pixels, per channel
  long long sse[3];      // sum of squared errors over the pixels the block owns, per channel
};

struct Args {
  const float* gt;
  const float* pred[NR_METRICS_MAX_PRED];
  int w;                 // row stride of the [h,w,3] images
  int y0, x0;            // top-left corner of the crop
  int ch, cw;            // cropped size
  int tiles_x, tiles_y;
  Partial* part;         // [n_pred][tiles_y * tiles_x]
};

// sum over the block in a fixed order; the result is valid in thread 0
template <class T>
__device__ __forceinline__ T block_sum(T v, T* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int k = 1; k < THREADS / 32; ++k) v += red[k];
  return v;
}

// One block: a TH x TW tile of the SSIM map of one prediction (blockIdx.z), all three channels, plus the squared errors of
// the pixels it owns.  The SSIM map covers the cropped image less 5 pixels on every side, so every window lies inside
// the crop; pixel (y, x) of the crop is owned by the tile whose map rows / columns contain it, the 5-pixel border
// strips by the first / last tile.
__global__ void __launch_bounds__(THREADS) ssim_tile_kernel(const __grid_constant__ Args a) {
  __shared__ uint8_t px[2][3][LH][LW];     // quantised ground truth / prediction
  __shared__ int hs[5][LH][TW];            // horizontal 11-sums of x, y, x^2, y^2, xy
  __shared__ double red_d[THREADS / 32];
  __shared__ long long red_l[THREADS / 32];
  const float* pr = a.pred[blockIdx.z];
  const int ty0 = blockIdx.y * TH, tx0 = blockIdx.x * TW;   // crop coordinates of the tile's first input pixel
  int sse[3] = {0, 0, 0};
  for (int i = threadIdx.x; i < LH * LW; i += THREADS) {
    const int r = i / LW, c = i - r * LW, y = ty0 + r, x = tx0 + c;
    const bool in = y < a.ch && x < a.cw;
    const bool own = in && min(max(y - HALF, 0) / TH, a.tiles_y - 1) == (int)blockIdx.y &&
                     min(max(x - HALF, 0) / TW, a.tiles_x - 1) == (int)blockIdx.x;
    const long long o = in ? 3 * ((long long)(a.y0 + y) * a.w + a.x0 + x) : 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int g = in ? quantise(a.gt[o + k]) : 0, p = in ? quantise(pr[o + k]) : 0;
      px[0][k][r][c] = (uint8_t)g;
      px[1][k][r][c] = (uint8_t)p;
      if (own) sse[k] += (g - p) * (g - p);
    }
  }
  const int rows = min(TH, a.ch - 2 * HALF - ty0), cols = min(TW, a.cw - 2 * HALF - tx0);   // map pixels of this tile
  double ssim[3] = {0.0, 0.0, 0.0};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    __syncthreads();
    for (int i = threadIdx.x; i < LH * TW; i += THREADS) {
      const int r = i / TW, c = i - r * TW;
      int sx = 0, sy = 0, sxx = 0, syy = 0, sxy = 0;
#pragma unroll
      for (int d = 0; d <= 2 * HALF; ++d) {
        const int x = px[0][k][r][c + d], y = px[1][k][r][c + d];
        sx += x; sy += y; sxx += x * x; syy += y * y; sxy += x * y;
      }
      hs[0][r][c] = sx; hs[1][r][c] = sy; hs[2][r][c] = sxx; hs[3][r][c] = syy; hs[4][r][c] = sxy;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < TH * TW; i += THREADS) {
      const int r = i / TW, c = i - r * TW;
      if (r >= rows || c >= cols) continue;
      int s[5] = {0, 0, 0, 0, 0};
#pragma unroll
      for (int d = 0; d <= 2 * HALF; ++d)
#pragma unroll
        for (int q = 0; q < 5; ++q) s[q] += hs[q][r + d][c];
      ssim[k] += ssim_term(s[0], s[1], s[2], s[3], s[4]);
    }
  }
  Partial out;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    out.ssim[k] = block_sum(ssim[k], red_d);
    out.sse[k] = block_sum((long long)sse[k], red_l);
  }
  if (threadIdx.x == 0) a.part[(blockIdx.z * a.tiles_y + blockIdx.y) * a.tiles_x + blockIdx.x] = out;
}

// One block per prediction: out[n] = {sse_r, sse_g, sse_b, ssim}, the SSIM as skimage averages it (per channel over the
// map, then over the channels).
__global__ void __launch_bounds__(THREADS) finish_kernel(const Partial* part, int tiles, long long map_pixels, double* out) {
  __shared__ double red_d[THREADS / 32];
  __shared__ long long red_l[THREADS / 32];
  const Partial* p = part + (long long)blockIdx.x * tiles;
  double s[3] = {0.0, 0.0, 0.0};
  long long e[3] = {0, 0, 0};
  for (int t = threadIdx.x; t < tiles; t += THREADS)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      s[k] += p[t].ssim[k];
      e[k] += p[t].sse[k];
    }
  double mean[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    mean[k] = block_sum(s[k], red_d) / double(map_pixels);
    e[k] = block_sum(e[k], red_l);
  }
  if (threadIdx.x == 0) {
    double* o = out + 4 * blockIdx.x;
    o[0] = double(e[0]);
    o[1] = double(e[1]);
    o[2] = double(e[2]);
    o[3] = (mean[0] + mean[1] + mean[2]) / 3.0;
  }
}

inline int tiles_of(int n, int t) { return n > 2 * HALF ? (n - 2 * HALF + t - 1) / t : 0; }

// ---- eval.py: tf.image.psnr and tf.image.ssim of uint8 pairs ------------------------------------------------------------

constexpr int ETW = 32, ETH = 16;                           // SSIM-map pixels per block
constexpr int ELW = ETW + 2 * HALF, ELH = ETH + 2 * HALF;

struct EvalPartial {
  double ssim;           // sum of luminance * cs over the block's map pixels and the three channels
  double sse;            // sum of squared errors over the pixels the block owns, all channels
};

struct EvalArgs {
  const uint8_t* gt;     // [n,h,w,3]
  const uint8_t* pr;
  int h, w;
  int tiles_x, tiles_y;
  double g[2 * HALF + 1];   // gauss_window
  EvalPartial* part;     // [n][tiles_y * tiles_x]
};

// One block: an ETH x ETW tile of the VALID SSIM map of one pair (blockIdx.z), all three channels, plus the squared errors
// of the pixels it owns (the same ownership as ssim_tile_kernel).  Window sums are separable: horizontal 11-tap Gaussian
// sums of x, y, xy and x^2 + y^2 in shared memory, then vertical ones, all in fp64.
__global__ void __launch_bounds__(THREADS) eval_tile_kernel(const __grid_constant__ EvalArgs a) {
  __shared__ uint8_t px[2][3][ELH][ELW];
  __shared__ double hs[4][ELH][ETW];
  __shared__ double lut[256];                // color_map_forward of every byte value
  __shared__ double red[THREADS / 32];
  const long long img = (long long)blockIdx.z * a.h * a.w * 3;
  const int ty0 = blockIdx.y * ETH, tx0 = blockIdx.x * ETW;
  lut[threadIdx.x] = double(unit(threadIdx.x));
  __syncthreads();
  double sse = 0.0;
  for (int i = threadIdx.x; i < ELH * ELW; i += THREADS) {
    const int r = i / ELW, c = i - r * ELW, y = ty0 + r, x = tx0 + c;
    const bool in = y < a.h && x < a.w;
    const bool own = in && min(max(y - HALF, 0) / ETH, a.tiles_y - 1) == (int)blockIdx.y &&
                     min(max(x - HALF, 0) / ETW, a.tiles_x - 1) == (int)blockIdx.x;
    const long long o = in ? img + 3 * ((long long)y * a.w + x) : 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int g = in ? a.gt[o + k] : 0, p = in ? a.pr[o + k] : 0;
      px[0][k][r][c] = (uint8_t)g;
      px[1][k][r][c] = (uint8_t)p;
      const double d = lut[g] - lut[p];
      if (own) sse += d * d;
    }
  }
  const int rows = min(ETH, a.h - 2 * HALF - ty0), cols = min(ETW, a.w - 2 * HALF - tx0);
  double ssim = 0.0;
#pragma unroll 1
  for (int k = 0; k < 3; ++k) {
    __syncthreads();
    for (int i = threadIdx.x; i < ELH * ETW; i += THREADS) {
      const int r = i / ETW, c = i - r * ETW;
      double s[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int d = 0; d <= 2 * HALF; ++d) {
        const double x = lut[px[0][k][r][c + d]], y = lut[px[1][k][r][c + d]];
        s[0] += a.g[d] * x;
        s[1] += a.g[d] * y;
        s[2] += a.g[d] * mul_rn(x, y);
        s[3] += a.g[d] * (mul_rn(x, x) + mul_rn(y, y));
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) hs[q][r][c] = s[q];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < ETH * ETW; i += THREADS) {
      const int r = i / ETW, c = i - r * ETW;
      if (r >= rows || c >= cols) continue;
      double s[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int d = 0; d <= 2 * HALF; ++d)
#pragma unroll
        for (int q = 0; q < 4; ++q) s[q] += a.g[d] * hs[q][r + d][c];
      ssim += tf_ssim_term(s[0], s[1], s[2], s[3]);
    }
  }
  EvalPartial out;
  out.ssim = block_sum(ssim, red);
  out.sse = block_sum(sse, red);
  if (threadIdx.x == 0) a.part[(blockIdx.z * a.tiles_y + blockIdx.y) * a.tiles_x + blockIdx.x] = out;
}

// One block per pair: out[n] = {psnr, ssim}
__global__ void __launch_bounds__(THREADS) eval_finish_kernel(const EvalPartial* part, int tiles, long long pixels, long long map_pixels,
                                                              double* out) {
  __shared__ double red[THREADS / 32];
  const EvalPartial* p = part + (long long)blockIdx.x * tiles;
  double s = 0.0, e = 0.0;
  for (int t = threadIdx.x; t < tiles; t += THREADS) {
    s += p[t].ssim;
    e += p[t].sse;
  }
  s = block_sum(s, red);
  e = block_sum(e, red);
  if (threadIdx.x == 0) {
    const double mse = e / double(3 * pixels);
    out[2 * blockIdx.x] = mse == 0.0 ? INFINITY : 10.0 * log10(1.0 / mse);
    out[2 * blockIdx.x + 1] = s / double(3 * map_pixels);
  }
}

}  // namespace mt

// ---- eval.py: LPIPS-VGG (lpips.LPIPS(net='vgg'), version 0.1) --------------------------------------------------------------
// A pair batch runs as one 2n-image batch (ground truths first, predictions after them) through torchvision's
// vgg16.features[0:30] on nr_conv2d_nhwc; at each of the five taps a fused kernel scores every pixel of every pair.
namespace lp {

constexpr int CONVS = 13, TAPS = 5, PARAMS = 2 * CONVS + TAPS;
constexpr int CIN0 = 16;       // the first layer's 3 input channels, zero-padded to what nr_conv2d_nhwc takes
constexpr int SLICE = 128;     // output channels per convolution launch: nr_conv2d_nhwc takes at most 128
constexpr int TAP_PIX = 512;   // pixels of one pair per tap_kernel block
constexpr int THREADS = 256;

struct Conv {
  int cin, cout;
  int tap;                     // tap taken after this conv's ReLU (relu1_2 .. relu5_3), -1: none
  int pool;                    // 2x2 max-pool after it
};
constexpr Conv NET[CONVS] = {{3, 64, -1, 0},    {64, 64, 0, 1},     {64, 128, -1, 0},   {128, 128, 1, 1},   {128, 256, -1, 0},
                             {256, 256, -1, 0}, {256, 256, 2, 1},   {256, 512, -1, 0},  {512, 512, -1, 0},  {512, 512, 3, 1},
                             {512, 512, -1, 0}, {512, 512, -1, 0},  {512, 512, 4, 0}};
constexpr int TAP_C[TAPS] = {64, 128, 256, 512, 512};

inline int cin_packed(int l) { return l == 0 ? CIN0 : NET[l].cin; }
inline int slice_of(int l) { return NET[l].cout < SLICE ? NET[l].cout : SLICE; }

// packed buffer: per conv its weights as cout / slice blocks of [9 taps][cin_packed][slice], then its bias; then the five
// lin weights.  Every block starts on a 16-byte boundary (the convolution stages its weights with 16-byte copies).
struct Layout {
  long long w[CONVS], b[CONVS], lin[TAPS], total;
};
inline Layout layout() {
  Layout L;
  long long o = 0;
  auto take = [&o](long long n) {
    const long long r = o;
    o += (n + 3) & ~3LL;
    return r;
  };
  for (int l = 0; l < CONVS; ++l) {
    L.w[l] = take(9LL * cin_packed(l) * NET[l].cout);
    L.b[l] = take(NET[l].cout);
  }
  for (int t = 0; t < TAPS; ++t) L.lin[t] = take(TAP_C[t]);
  L.total = o;
  return L;
}

inline long long tap_blocks(long long hw) { return (hw + TAP_PIX - 1) / TAP_PIX; }

struct PackJob {
  const float* src;
  long long off, n;
  int cin, cinp, slice;        // cin == 0: copied as is (bias, lin)
};
struct PackArgs {
  PackJob job[PARAMS];
  float* out;
};

__global__ void __launch_bounds__(THREADS) pack_kernel(const __grid_constant__ PackArgs a) {
  const PackJob& j = a.job[blockIdx.y];
  for (long long e = (long long)blockIdx.x * THREADS + threadIdx.x; e < j.n; e += (long long)gridDim.x * THREADS) {
    float v;
    if (j.cin == 0) {
      v = j.src[e];
    } else {                   // [cout][cin][3][3] -> slice s, tap, packed input channel c, output o of the slice
      const long long per_slice = 9LL * j.cinp * j.slice;
      const int s = int(e / per_slice);
      long long r = e - s * per_slice;
      const int tap = int(r / ((long long)j.cinp * j.slice));
      r -= (long long)tap * j.cinp * j.slice;
      const int c = int(r / j.slice), o = int(r - (long long)c * j.slice);
      v = c < j.cin ? j.src[((long long)(s * j.slice + o) * j.cin + c) * 9 + tap] : 0.f;
    }
    a.out[j.off + e] = v;
  }
}

__constant__ float SHIFT[3] = {(float)-.030, (float)-.088, (float)-.188};
__constant__ float SCALE[3] = {(float).458, (float).448, (float).450};

// x[(i, y, x)][16]: image i < n is gt[i], image n + i is pr[i]; channels 0..2 = the scaling layer of color_map_forward(v) * 2 - 1
__global__ void __launch_bounds__(THREADS) input_kernel(const uint8_t* __restrict__ gt, const uint8_t* __restrict__ pr, long long px, float* x) {
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < 2 * px; i += (long long)gridDim.x * THREADS) {
    const uint8_t* src = i < px ? gt + 3 * i : pr + 3 * (i - px);
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = __fdiv_rn(__fsub_rn(__fsub_rn(__fmul_rn(mt::unit(src[c]), 2.f), 1.f), SHIFT[c]), SCALE[c]);
    float4* o = reinterpret_cast<float4*>(x + 16 * i);
    o[0] = make_float4(v[0], v[1], v[2], 0.f);
    o[1] = o[2] = o[3] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

__global__ void __launch_bounds__(THREADS) relu_kernel(float4* x, long long n4) {
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < n4; i += (long long)gridDim.x * THREADS) {
    float4 v = x[i];
    v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    x[i] = v;
  }
}

// MaxPool2d(2, 2): [N,H,W,C] -> [N,H/2,W/2,C]
__global__ void __launch_bounds__(THREADS) pool_kernel(const float4* __restrict__ x, float4* __restrict__ y, int N, int H, int W, int C4) {
  const int Ho = H / 2, Wo = W / 2;
  const long long total = (long long)N * Ho * Wo * C4;
  for (long long i = (long long)blockIdx.x * THREADS + threadIdx.x; i < total; i += (long long)gridDim.x * THREADS) {
    const int c = int(i % C4);
    const long long q = i / C4;
    const int xo = int(q % Wo), yo = int((q / Wo) % Ho);
    const long long img = q / ((long long)Wo * Ho);
    const float4* s = x + ((img * H + 2 * yo) * W + 2 * xo) * C4 + c;
    const float4 a = s[0], b = s[C4], d = s[(long long)W * C4], e = s[(long long)W * C4 + C4];
    y[i] = make_float4(fmaxf(fmaxf(a.x, b.x), fmaxf(d.x, e.x)), fmaxf(fmaxf(a.y, b.y), fmaxf(d.y, e.y)),
                       fmaxf(fmaxf(a.z, b.z), fmaxf(d.z, e.z)), fmaxf(fmaxf(a.w, b.w), fmaxf(d.w, e.w)));
  }
}

// sum of squares of a float4 with every product and sum rounded on its own: both images of a pair go through these same
// operations, so identical features give bit-identical norms (a free FMA contraction may pair the terms differently)
__device__ __forceinline__ float sum_sq(float4 v) {
  return __fadd_rn(__fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)), __fadd_rn(__fmul_rn(v.z, v.z), __fmul_rn(v.w, v.w)));
}

// One tap, steps 3-4 of LPIPS for TAP_PIX pixels of one pair (blockIdx.y): per pixel, each image's features divided by
// (their channel norm + 1e-10), the squared difference weighted by lin and summed over the channels.  A group of L lanes
// holds one pixel's C channels.  part[pair * stride + block] = the sum over the block's pixels, added in a fixed order.
template <int C>
__global__ void __launch_bounds__(THREADS) tap_kernel(const float* __restrict__ f, const float* __restrict__ lin, int n, long long hw,
                                                      double* part, long long stride) {
  constexpr int L = C / 4 < 32 ? C / 4 : 32, V = C / (4 * L), G = THREADS / L;
  static_assert(TAP_PIX % G == 0, "whole iterations");
  __shared__ double red[THREADS / 32];
  const int pair = blockIdx.y, grp = threadIdx.x / L, sub = threadIdx.x - grp * L;
  const float4* f0 = reinterpret_cast<const float4*>(f) + (long long)pair * hw * (C / 4);
  const float4* f1 = reinterpret_cast<const float4*>(f) + ((long long)n + pair) * hw * (C / 4);
  float4 wl[V];
#pragma unroll
  for (int v = 0; v < V; ++v) wl[v] = reinterpret_cast<const float4*>(lin)[sub + v * L];
  const long long p0 = (long long)blockIdx.x * TAP_PIX;
  double acc = 0.0;
  for (int it = 0; it < TAP_PIX / G; ++it) {         // the same trip count in every lane: the shuffles see whole warps
    const long long p = p0 + it * G + grp;
    const bool valid = p < hw;
    float4 a[V], b[V];
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      a[v] = valid ? f0[p * (C / 4) + sub + v * L] : z;
      b[v] = valid ? f1[p * (C / 4) + sub + v * L] : z;
      s0 = __fadd_rn(s0, sum_sq(a[v]));
      s1 = __fadd_rn(s1, sum_sq(b[v]));
    }
    const float n0 = sqrtf(warp_sum<L>(s0)) + 1e-10f, n1 = sqrtf(warp_sum<L>(s1)) + 1e-10f;
    float t = 0.f;
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const float dx = a[v].x / n0 - b[v].x / n1, dy = a[v].y / n0 - b[v].y / n1;
      const float dz = a[v].z / n0 - b[v].z / n1, dw = a[v].w / n0 - b[v].w / n1;
      t += wl[v].x * dx * dx + wl[v].y * dy * dy + wl[v].z * dz * dz + wl[v].w * dw * dw;
    }
    t = warp_sum<L>(t);
    if (valid && sub == 0) acc += t;
  }
  acc = mt::block_sum(acc, red);
  if (threadIdx.x == 0) part[pair * stride + blockIdx.x] = acc;
}

struct FinishArgs {
  const double* part;          // [TAPS][n][stride]
  long long stride;
  int n;
  long long blocks[TAPS], hw[TAPS];
  double* out;
};

// One block per pair: out[pair] = the sum over the taps of the spatial mean
__global__ void __launch_bounds__(THREADS) finish_kernel(const __grid_constant__ FinishArgs a) {
  __shared__ double red[THREADS / 32];
  double total = 0.0;
  for (int t = 0; t < TAPS; ++t) {
    const double* p = a.part + ((long long)t * a.n + blockIdx.x) * a.stride;
    double s = 0.0;
    for (long long b = threadIdx.x; b < a.blocks[t]; b += THREADS) s += p[b];
    s = mt::block_sum(s, red);
    total += s / double(a.hw[t]);
  }
  if (threadIdx.x == 0) a.out[blockIdx.x] = total;
}

inline unsigned grid_for(long long items) {
  const long long g = (items + THREADS - 1) / THREADS;
  return unsigned(g < 1 ? 1 : (g > 8192 ? 8192 : g));
}

int tap(int t, const float* f, const float* lin, int n, long long hw, double* part, long long stride, cudaStream_t st) {
  const dim3 grid(unsigned(tap_blocks(hw)), n);
  switch (TAP_C[t]) {
    case 64: tap_kernel<64><<<grid, THREADS, 0, st>>>(f, lin, n, hw, part, stride); break;
    case 128: tap_kernel<128><<<grid, THREADS, 0, st>>>(f, lin, n, hw, part, stride); break;
    case 256: tap_kernel<256><<<grid, THREADS, 0, st>>>(f, lin, n, hw, part, stride); break;
    default: tap_kernel<512><<<grid, THREADS, 0, st>>>(f, lin, n, hw, part, stride); break;
  }
  NR_CHECK_LAUNCH("lpips tap_kernel");
  return NR_OK;
}

}  // namespace lp
}  // namespace nr

using namespace nr;

extern "C" long long nr_image_metrics_workspace(int n_pred, int h, int w, int margin_h, int margin_w) {
  if (n_pred < 1 || margin_h < 0 || margin_w < 0) return 0;
  const long long tiles = (long long)mt::tiles_of(h - 2 * margin_h, mt::TH) * mt::tiles_of(w - 2 * margin_w, mt::TW);
  return n_pred * tiles * (long long)sizeof(mt::Partial);
}

extern "C" int nr_image_metrics(const float* gt, const float* const* preds, int n_pred, int h, int w, int margin_h, int margin_w,
                                double* out, void* workspace, long long workspace_bytes, void* stream) {
  NR_CHECK_ARG(gt != nullptr && preds != nullptr && out != nullptr, "image_metrics: null pointer");
  NR_CHECK_ARG(n_pred >= 1 && n_pred <= NR_METRICS_MAX_PRED, "image_metrics: n_pred must be 1..NR_METRICS_MAX_PRED");
  NR_CHECK_ARG(h >= 1 && w >= 1 && margin_h >= 0 && margin_w >= 0, "image_metrics: shape");
  const int ch = h - 2 * margin_h, cw = w - 2 * margin_w;
  NR_CHECK_ARG(ch >= 11 && cw >= 11, "image_metrics: the cropped image is smaller than the 11x11 SSIM window");
  NR_CHECK_ARG(workspace != nullptr && workspace_bytes >= nr_image_metrics_workspace(n_pred, h, w, margin_h, margin_w),
               "image_metrics: workspace too small");
  mt::Args a;
  a.gt = gt;
  for (int n = 0; n < NR_METRICS_MAX_PRED; ++n) a.pred[n] = n < n_pred ? preds[n] : nullptr;
  for (int n = 0; n < n_pred; ++n) NR_CHECK_ARG(a.pred[n] != nullptr, "image_metrics: null prediction");
  a.w = w;
  a.y0 = margin_h;
  a.x0 = margin_w;
  a.ch = ch;
  a.cw = cw;
  a.tiles_x = mt::tiles_of(cw, mt::TW);
  a.tiles_y = mt::tiles_of(ch, mt::TH);
  NR_CHECK_ARG(a.tiles_y <= 65535, "image_metrics: image too tall");
  a.part = (mt::Partial*)workspace;
  mt::ssim_tile_kernel<<<dim3(a.tiles_x, a.tiles_y, n_pred), mt::THREADS, 0, (cudaStream_t)stream>>>(a);
  NR_CHECK_LAUNCH("ssim_tile_kernel");
  mt::finish_kernel<<<n_pred, mt::THREADS, 0, (cudaStream_t)stream>>>(a.part, a.tiles_x * a.tiles_y, (long long)(ch - 10) * (cw - 10), out);
  NR_CHECK_LAUNCH("finish_kernel");
  return NR_OK;
}

extern "C" long long nr_eval_metrics_workspace(int n, int h, int w) {
  if (n < 1) return 0;
  return n * (long long)mt::tiles_of(h, mt::ETH) * mt::tiles_of(w, mt::ETW) * (long long)sizeof(mt::EvalPartial);
}

extern "C" int nr_eval_metrics(const uint8_t* gt, const uint8_t* pr, int n, int h, int w, double* out, void* workspace, long long workspace_bytes,
                               void* stream) {
  NR_CHECK_ARG(gt != nullptr && pr != nullptr && out != nullptr, "eval_metrics: null pointer");
  NR_CHECK_ARG(n >= 1 && n <= 65535, "eval_metrics: n must be 1..65535");
  NR_CHECK_ARG(h >= 11 && w >= 11, "eval_metrics: images smaller than the 11x11 SSIM window");
  NR_CHECK_ARG(workspace != nullptr && workspace_bytes >= nr_eval_metrics_workspace(n, h, w), "eval_metrics: workspace too small");
  mt::EvalArgs a;
  a.gt = gt;
  a.pr = pr;
  a.h = h;
  a.w = w;
  a.tiles_x = mt::tiles_of(w, mt::ETW);
  a.tiles_y = mt::tiles_of(h, mt::ETH);
  NR_CHECK_ARG(a.tiles_y <= 65535, "eval_metrics: image too tall");
  mt::gauss_window(a.g);
  a.part = (mt::EvalPartial*)workspace;
  mt::eval_tile_kernel<<<dim3(a.tiles_x, a.tiles_y, n), mt::THREADS, 0, (cudaStream_t)stream>>>(a);
  NR_CHECK_LAUNCH("eval_tile_kernel");
  mt::eval_finish_kernel<<<n, mt::THREADS, 0, (cudaStream_t)stream>>>(a.part, a.tiles_x * a.tiles_y, (long long)h * w,
                                                                       (long long)(h - 2 * mt::HALF) * (w - 2 * mt::HALF), out);
  NR_CHECK_LAUNCH("eval_finish_kernel");
  return NR_OK;
}

extern "C" int nr_lpips_vgg_layout(int* n_tensors, long long* packed_floats) {
  NR_CHECK_ARG(n_tensors != nullptr && packed_floats != nullptr, "lpips_vgg_layout: null pointer");
  *n_tensors = lp::PARAMS;
  *packed_floats = lp::layout().total;
  return NR_OK;
}

extern "C" int nr_lpips_vgg_pack(const float* const* params, int n_params, float* packed, void* stream) {
  NR_CHECK_ARG(params != nullptr && packed != nullptr, "lpips_vgg_pack: null pointer");
  NR_CHECK_ARG(n_params == lp::PARAMS, "lpips_vgg_pack: 31 tensors expected (features.*.weight / bias, then lin0..4)");
  const lp::Layout L = lp::layout();
  lp::PackArgs a;
  a.out = packed;
  long long biggest = 0;
  for (int i = 0; i < lp::PARAMS; ++i) {
    NR_CHECK_ARG(params[i] != nullptr, "lpips_vgg_pack: null parameter tensor");
    lp::PackJob& j = a.job[i];
    j.src = params[i];
    j.cin = j.cinp = j.slice = 0;
    if (i < 2 * lp::CONVS) {
      const int l = i / 2;
      if (i % 2 == 0) {
        j.off = L.w[l];
        j.n = 9LL * lp::cin_packed(l) * lp::NET[l].cout;
        j.cin = lp::NET[l].cin;
        j.cinp = lp::cin_packed(l);
        j.slice = lp::slice_of(l);
      } else {
        j.off = L.b[l];
        j.n = lp::NET[l].cout;
      }
    } else {
      const int t = i - 2 * lp::CONVS;
      j.off = L.lin[t];
      j.n = lp::TAP_C[t];
    }
    if (j.n > biggest) biggest = j.n;
  }
  lp::pack_kernel<<<dim3(unsigned((biggest + lp::THREADS - 1) / lp::THREADS < 64 ? (biggest + lp::THREADS - 1) / lp::THREADS : 64), lp::PARAMS),
                    lp::THREADS, 0, (cudaStream_t)stream>>>(a);
  NR_CHECK_LAUNCH("lpips pack_kernel");
  return NR_OK;
}

extern "C" long long nr_lpips_vgg_workspace(int n, int h, int w) {
  if (n < 1 || h < 32 || w < 32) return 0;
  const long long hw = (long long)h * w;
  return 2 * (2LL * n * hw * 64) * (long long)sizeof(float) + lp::TAPS * n * lp::tap_blocks(hw) * (long long)sizeof(double);
}

extern "C" int nr_lpips_vgg_fwd(const float* packed, const uint8_t* gt, const uint8_t* pr, int n, int h, int w, double* out, int tf32x1,
                                void* workspace, long long workspace_bytes, void* stream) {
  NR_CHECK_ARG(packed != nullptr && gt != nullptr && pr != nullptr && out != nullptr, "lpips_vgg: null pointer");
  NR_CHECK_ARG(n >= 1 && n <= 65535, "lpips_vgg: n must be 1..65535");
  NR_CHECK_ARG(h >= 32 && w >= 32, "lpips_vgg: images must be at least 32 x 32 (nr_conv2d_nhwc needs 2 x 2 for conv5, after four 2x2 pools)");
  NR_CHECK_ARG(workspace != nullptr && workspace_bytes >= nr_lpips_vgg_workspace(n, h, w), "lpips_vgg: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const lp::Layout L = lp::layout();
  const long long N = 2LL * n, hw = (long long)h * w, stride = lp::tap_blocks(hw);
  float* cur = (float*)workspace;               // two ping-pong buffers of the largest activation, [2n,h,w,64]
  float* nxt = cur + N * hw * 64;
  double* part = (double*)(nxt + N * hw * 64);
  lp::input_kernel<<<lp::grid_for(N * hw), lp::THREADS, 0, st>>>(gt, pr, n * hw, cur);
  NR_CHECK_LAUNCH("lpips input_kernel");
  lp::FinishArgs fa;
  fa.part = part;
  fa.stride = stride;
  fa.n = n;
  fa.out = out;
  int H = h, W = w;
  for (int l = 0; l < lp::CONVS; ++l) {
    const int cinp = lp::cin_packed(l), cout = lp::NET[l].cout, S = lp::slice_of(l);
    for (int s = 0; s < cout / S; ++s) {
      NrConv2d c = {};
      c.x = cur;
      c.w_packed = packed + L.w[l] + 9LL * cinp * S * s;
      c.bias = packed + L.b[l] + S * s;
      c.y = nxt;
      c.n = int(N); c.h = H; c.w = W; c.cin = cinp; c.cout = S; c.ks = 3; c.stride = 1; c.reflect = 0; c.pad = 1;
      c.x_stride = cinp; c.y_stride = cout; c.y_off = S * s;
      c.tf32x1 = tf32x1 != 0;
      const int rc = nr_conv2d_nhwc(&c, stream);
      if (rc != NR_OK) return rc;
    }
    std::swap(cur, nxt);
    lp::relu_kernel<<<lp::grid_for(N * H * W * cout / 4), lp::THREADS, 0, st>>>((float4*)cur, N * H * W * cout / 4);
    NR_CHECK_LAUNCH("lpips relu_kernel");
    const int t = lp::NET[l].tap;
    if (t >= 0) {
      const int rc = lp::tap(t, cur, packed + L.lin[t], n, (long long)H * W, part + (long long)t * n * stride, stride, st);
      if (rc != NR_OK) return rc;
      fa.blocks[t] = lp::tap_blocks((long long)H * W);
      fa.hw[t] = (long long)H * W;
    }
    if (lp::NET[l].pool) {
      lp::pool_kernel<<<lp::grid_for(N * (H / 2) * (W / 2) * cout / 4), lp::THREADS, 0, st>>>((const float4*)cur, (float4*)nxt, int(N), H, W, cout / 4);
      NR_CHECK_LAUNCH("lpips pool_kernel");
      std::swap(cur, nxt);
      H /= 2;
      W /= 2;
    }
  }
  lp::finish_kernel<<<n, lp::THREADS, 0, st>>>(fa);
  NR_CHECK_LAUNCH("lpips finish_kernel");
  return NR_OK;
}
