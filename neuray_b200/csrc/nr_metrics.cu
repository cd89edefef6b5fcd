// Validation image metrics (reference network/metrics.py:13-79, PSNR_SSIM with skimage's structural_similarity(win_size=11,
// data_range=255) and compute_psnr): one ground truth against up to NR_METRICS_MAX_PRED predictions per call.
//
// Every input is quantised to an integer 0..255 first (color_map_backward), so the 11x11 window sums of x, y, x^2, y^2 and xy
// are exact in int32 (at most 121 * 65025) and the squared errors are exact integers.  Only the SSIM term itself is floating
// point (fp64).  Its per-block sums are written to the workspace and added up by a second kernel in a fixed order: the result
// is the same bit for bit from run to run, with no floating-point atomics.
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
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
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

}  // namespace mt
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
