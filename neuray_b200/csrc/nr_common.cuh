// Shared device helpers + the packed weight layout (single source of truth for host and kernels).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/neuray_b200.h"

#define NR_HD __host__ __device__ __forceinline__

namespace nr {

void set_error(const char* fmt, ...);

// Launch helpers (nr_ops.cu).  On a failed CUDA call both set an error naming `who` and return NR_E_CUDA.
// The SM count of the current device.
int sm_count(int* sms, const char* who);
// The dynamic shared-memory opt-in of kernel `fn` for a launch with `bytes` of it (nothing to do at or below 48 KB).  It
// is a per-device function attribute and is set on every launch, so that the library keeps no per-process state: a
// process may render on any number of devices from any number of threads.
int opt_in_smem(const void* fn, size_t bytes, const char* who);

// The point kernel's optional per-(view, point) exports (launch_point_kernel's `exports`, point_body's EXPORTS), stored
// into a [k][rfn][rn*dn] workspace: EXPORT_BLEND the colour-blend weight (row 0), EXPORT_AGG the aggregation net's
// pooling weights w0 and w2 (rows 1 and 2; only together with EXPORT_BLEND), EXPORT_VIEW the dist decoder's masked hit
// probability (row 3; only together with both).  The sets nest, so one request is served by the smallest that covers it.
constexpr int EXPORT_BLEND = 1, EXPORT_AGG = 2, EXPORT_VIEW = 4;

#define NR_CHECK_ARG(cond, msg)                    \
  do {                                             \
    if (!(cond)) {                                 \
      nr::set_error("invalid argument: %s", msg);  \
      return NR_E_INVALID;                         \
    }                                              \
  } while (0)

#define NR_CHECK_LAUNCH(name)                                                   \
  do {                                                                          \
    cudaError_t e_ = cudaGetLastError();                                        \
    if (e_ != cudaSuccess) {                                                    \
      nr::set_error("%s: CUDA error %s", name, cudaGetErrorString(e_));         \
      return NR_E_CUDA;                                                         \
    }                                                                           \
  } while (0)

// ------------------------------------------------------------------------------------------------------------
// Packed weight layout (floats).  Every block starts on a multiple of 4 floats so it can be staged to shared
// memory with 128-bit copies.  "WT" = weight stored transposed, [in][out] row-major (out contiguous).
namespace lay {
constexpr int pad4(int x) { return (x + 3) & ~3; }

// dist-decoder head block (reference dist_decoder.py:64-97): Linear(32,32) ELU Linear(32,32) ELU Linear(32,{2,1})
constexpr int DD_L0_W = 0;                  // WT[32][32]
constexpr int DD_L0_B = DD_L0_W + 1024;     // [32]
constexpr int DD_L1_W = DD_L0_B + 32;       // WT[32][32]
constexpr int DD_L1_B = DD_L1_W + 1024;     // [32]
constexpr int DD_L2_W = DD_L1_B + 32;       // W[2][32] row-major (second row zero for 1-output heads)
constexpr int DD_L2_B = DD_L2_W + 64;       // [4]
constexpr int DD_HEAD_STRIDE = DD_L2_B + 4; // 2180
constexpr int DD_HEAD = 0;                  // heads: 0 mean, 1 var, 2 aw, 3 vis

// group B: prob_embed (aggregate_net.py:28-32), ray_dir_fc, neuray_fc (ibrnet.py:248-251,286-290)
constexpr int GRP_B = DD_HEAD + 4 * DD_HEAD_STRIDE;
constexpr int PE0_W = 0;                    // WT[34][32]
constexpr int PE0_B = PE0_W + 34 * 32;      // [32]
constexpr int PE1_W = PE0_B + 32;           // WT[32][32]
constexpr int PE1_B = PE1_W + 1024;         // [32]
constexpr int RD0_W = PE1_B + 32;           // WT[4][16]
constexpr int RD0_B = RD0_W + 64;           // [16]
constexpr int RD1_W = RD0_B + 16;           // WT[16][36] (35 used)
constexpr int RD1_B = RD1_W + 16 * 36;      // [36]
constexpr int NF0_W = RD1_B + 36;           // WT[32][8]
constexpr int NF0_B = NF0_W + 256;          // [8]
constexpr int NF1_W = NF0_B + 8;            // [8]
constexpr int NF1_B = NF1_W + 8;            // [4]
constexpr int GRP_B_SIZE = NF1_B + 4;

// group C: base_fc (ibrnet.py:253-256).  Layer 0 is split into the 140 view-invariant inputs ("hoist", applied
// once per point) and the 67 per-view inputs.
constexpr int HOIST_W = GRP_B + GRP_B_SIZE; // WT[140][64]
constexpr int HOIST_B = HOIST_W + 140 * 64; // [64]
constexpr int BASE0_W = HOIST_B + 64;       // WT[67][64]  (rgb_feat 35 | neuray_feat 32)
constexpr int BASE1_W = BASE0_W + 67 * 64;  // WT[64][32]
constexpr int BASE1_B = BASE1_W + 64 * 32;  // [32]

// group D1: vis_fc, vis_fc2, rgb_fc (ibrnet.py:258-284)
constexpr int GRP_D1 = BASE1_B + 32;
constexpr int VIS0_W = 0;                   // WT[32][32]
constexpr int VIS0_B = VIS0_W + 1024;
constexpr int VIS1_W = VIS0_B + 32;         // WT[32][32]  (x_res outputs 0..31)
constexpr int VIS1_B = VIS1_W + 1024;
constexpr int VIS1L_W = VIS1_B + 32;        // [32]        (33rd output: visibility logit)
constexpr int VIS1L_B = VIS1L_W + 32;       // [4]
constexpr int V20_W = VIS1L_B + 4;          // WT[32][32]
constexpr int V20_B = V20_W + 1024;
constexpr int V21_W = V20_B + 32;           // [32]
constexpr int V21_B = V21_W + 32;           // [4]
constexpr int RGB0_W = V21_B + 4;           // WT[37][16]
constexpr int RGB0_B = RGB0_W + 37 * 16;    // [16]
constexpr int RGB1_W = RGB0_B + 16;         // WT[16][8]
constexpr int RGB1_B = RGB1_W + 128;        // [8]
constexpr int RGB2_W = RGB1_B + 8;          // [8]
constexpr int RGB2_B = RGB2_W + 8;          // [4]
constexpr int GRP_D1_SIZE = RGB2_B + 4;

// group D2: geometry_fc (ibrnet.py:271-274)
constexpr int GRP_D2 = GRP_D1 + GRP_D1_SIZE;
constexpr int GEO0_W = 0;                   // WT[65][64]
constexpr int GEO0_B = GEO0_W + 65 * 64;    // [64]
constexpr int GEO1_W = GEO0_B + 64;         // WT[64][16]
constexpr int GEO1_B = GEO1_W + 64 * 16;    // [16]
constexpr int GRP_D2_SIZE = GEO1_B + 16;

constexpr int TOTAL_POINT = GRP_D2 + GRP_D2_SIZE;

// ray kernel: MultiHeadAttention(4,16,4,4) + out_geometry_fc (ibrnet.py:52-102,276-279)
constexpr int WQ = 0;        // WT[16][16]
constexpr int WK = 256;
constexpr int WV = 512;
constexpr int WFC = 768;
constexpr int LN_W = 1024;   // [16]
constexpr int LN_B = 1040;   // [16]
constexpr int OG0_W = 1056;  // WT[16][16]
constexpr int OG0_B = 1312;  // [16]
constexpr int OG1_W = 1328;  // [16]
constexpr int OG1_B = 1344;  // [4]
constexpr int TOTAL_RAY = 1348;

static_assert(GRP_B % 4 == 0 && HOIST_W % 4 == 0 && BASE0_W % 4 == 0 && BASE1_W % 4 == 0 && GRP_D1 % 4 == 0 &&
                  GRP_D2 % 4 == 0 && RD1_W % 4 == 0 && NF0_W % 4 == 0 && RGB0_W % 4 == 0 && GEO1_W % 4 == 0,
              "weight blocks must be 16-byte aligned");
}  // namespace lay

// ------------------------------------------------------------------------------------------------------------
// Tensor-core weight buffer (w_tc): every tensor-core layer's W^T as hi / lo tf32 parts, K padded and re-ordered to the
// kernel's A-column order, pre-swizzled into K-major SWIZZLE_128B tiles of 32-wide K slabs (N rows x 32 floats), grouped
// into the 16 KB ring stages the producer warp streams (offsets in floats).  Where a layer's parts sit inside its stage
// or tile is a Tile below; the packer, the stage table and the kernel all read it from there.
namespace tcl {
// hi part at `hi`, lo part at `lo`, K slab s of either part s * slab floats further
struct Tile {
  int hi, lo, slab;
};
constexpr int STAGE = 4096;
constexpr int HEAD0 = 0;            // head h: stage h
constexpr Tile HEAD_L0 = {0, 1024, 1024}, HEAD_L1 = {2048, 3072, 1024};   // N 32, K 32 each
constexpr int PE0 = 4 * STAGE;
constexpr Tile PE0_L = {0, 2048, 1024};                                    // N 32, K 34 -> 40
constexpr int PE1 = PE0 + STAGE;
constexpr Tile PE1_L = {0, 1536, 1536};                                    // N 48 (prob_embed.2 + neuray_fc.0 behind it), K 32
constexpr int PE1_SIZE = 3072;
constexpr int B0 = PE1 + STAGE;     // base_fc.0's per-view inputs (rgb_feat 35 + bias + 4 zeros | neuray_feat 32): stage s holds slab s
constexpr Tile B0_L = {0, 2048, STAGE};                                    // N 64, K 67 -> 72
constexpr int B1 = B0 + 3 * STAGE;
constexpr Tile B1_L = {0, 2048, 1024};                                     // N 32, K 64
constexpr int V01 = B1 + STAGE;
constexpr Tile VIS0_L = {0, 1024, 1024}, VIS2_L = {2048, 3072, 1024};      // vis_fc.0, vis_fc.2[:32]: N 32, K 32
constexpr int V2R = V01 + STAGE;
constexpr Tile V20_L = {0, 1024, 1024}, RGB0_L = {2048, 3072, 512};        // vis_fc2.0: N 32, K 32; rgb_fc.0: N 16, K 37 -> 40
constexpr int RD1 = V2R + STAGE;    // ray_dir_fc.2, resident in shared memory
constexpr Tile RD1_L = {0, 1536, 1536};                                    // N 48 (35 used), K 16
constexpr int RD1_SIZE = 3072;
constexpr int HST = RD1 + RD1_SIZE; // the 140 view-pooled inputs of base_fc.0: K index = 32*round + 8*stat + i (feature 8*round + i;
                                    //   stat = mean0, var0, mean1, var1)
constexpr Tile HST_L = {0, 10240, 2048};                                   // N 64, K 140 -> 160: hi 5 slabs | lo 5 slabs
constexpr int HST_SIZE = 2 * HST_L.lo;
constexpr Tile HST_STAGE = {0, 2048, 2048};   // HST streams through the ring a slab per stage: hi slab | lo slab right behind it
constexpr int G0 = HST + HST_SIZE;  // geometry_fc.0 on the view-pooled statistics, stage s holds slab s: K index = 32*round +
                                    //   16*stat + i (feature 16*round + i; stat = mean, var); K 64 = mean weight, K 65 = bias
constexpr Tile G0_L = {0, 2048, STAGE};                                    // N 64, K 66 -> 96
constexpr int TOTAL = G0 + 3 * STAGE;
static_assert(HST_STAGE.lo == HST_L.slab, "stage_source lands a HST lo slab right behind its hi slab");
}  // namespace tcl

// ------------------------------------------------------------------------------------------------------------
// math used by both kernels

// ELU = x > 0 ? x : exp(x) - 1, five instructions and no branch:
//   * exp through ex2.approx.ftz (FMUL + MUFU; __expf's non-ftz path adds a compare and two predicated multiplies per
//     call for denormal results, which only matter below exp(-87) where ELU is -1 either way); abs error ~1e-7
//   * the select is a selp on a setp, never a divergent branch around the MUFU (the ternary form compiled to one and
//     serialised the 32-wide epilogues)
__device__ __forceinline__ float ex2_ftz(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float elu(float x) {
  const float e = ex2_ftz(x * 1.4426950408889634f) - 1.f;
  float y;
  asm("{\n\t.reg .pred p;\n\tsetp.gt.f32 p, %1, 0f00000000;\n\tselp.f32 %0, %1, %2, p;\n\t}" : "=f"(y) : "f"(x), "f"(e));
  return y;
}
__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }
// softplus(x) = max(x, 0) + log(1 + exp(-|x|)): the exponential is in (0, 1], so the fast ex2/lg2 paths are accurate to ~2e-7
// absolute here (log1pf(expf(x)) costs two slow-path libm calls per value)
__device__ __forceinline__ float softplusf_(float x) { return x > 20.f ? x : fmaxf(x, 0.f) + __logf(1.f + __expf(-fabsf(x))); }
// 0.5 + 0.5 tanh(x), accurate to ~1e-7 absolute (tanh.approx is only ~5e-4)
__device__ __forceinline__ float logistic_cdf(float x) {
  // 0.5 + 0.5*tanh(x) = 1/(1+exp(-2x))
  return 1.f / (1.f + __expf(-2.f * x));
}

// sum over each aligned group of L lanes (a power of two), xor butterfly L/2, ..., 1; every lane of the group gets the sum
template <int L = 32, class T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = L / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// read-only input: the non-coherent load path on the device
NR_HD float ld_ro(const float* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}

// four consecutive read-only floats (16-byte aligned on the device)
NR_HD float4 ld_ro4(const float* p) {
#ifdef __CUDA_ARCH__
  return __ldg(reinterpret_cast<const float4*>(p));
#else
  return make_float4(p[0], p[1], p[2], p[3]);
#endif
}

// ---- geometry of one query point (render_ops.py coords2rays / depth2points, dist_decoder.py get_near_far_points) ---------
// Point n = ray * dn + s: its world position on ray `ray` at que_depth[n], the unit query direction (camera -> point,
// negated) and the half widths of its bin towards the previous / next sample in normalised inverse depth.  cam: the query
// camera block of NrPassParams::que_cam, wherever the caller keeps it.
struct PointGeo { float X, Y, Z, qx, qy, qz, ihp, ihc; };
template <typename I>
NR_HD PointGeo point_geometry(const float* cam, const float* coords, const float* que_depth, int dn, I n) {
  PointGeo g;
  const I ray = n / dn;
  const int s = int(n - ray * dn);
  const float cx = ld_ro(coords + 2 * ray), cy = ld_ro(coords + 2 * ray + 1);
  float cm[3], d[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) cm[i] = fmaf(cam[12 + 3 * i + 1], cy, cam[12 + 3 * i] * cx) + cam[12 + 3 * i + 2];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float wld = fmaf(cam[3 * i + 2], cm[2], fmaf(cam[3 * i + 1], cm[1], cam[3 * i] * cm[0])) + cam[9 + i];
    d[i] = wld - cam[9 + i];   // the reference adds the centre and subtracts it again (render_ops.py:22-23)
  }
  const float z = ld_ro(que_depth + n);
  g.X = fmaf(d[0], z, cam[9]); g.Y = fmaf(d[1], z, cam[10]); g.Z = fmaf(d[2], z, cam[11]);
  const float nrm = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  g.qx = -d[0] / nrm; g.qy = -d[1] / nrm; g.qz = -d[2] / nrm;
  const float a = -1.f / cam[21], bb = -1.f / cam[22];
  const float tcur = (-1.f / z - a) / (bb - a);
  float dc = 1e6f;
  if (s + 1 < dn) dc = (-1.f / ld_ro(que_depth + n + 1) - a) / (bb - a) - tcur;
  float dp = dc;
  if (s > 0) dp = tcur - (-1.f / ld_ro(que_depth + n - 1) - a) / (bb - a);
  g.ihc = dc * 0.5f; g.ihp = dp * 0.5f;
  return g;
}

// ---- projection of a point into a view of an h x w image (render_ops.py project_points_dict) ----------------------------
// vp: the view's 20-float row of NrPassParams::view_params.  zh is the projected depth after the fix-up of a point on the
// camera plane; valid_z is false for such a point, valid also for one outside the image.  dir: the unit vector view centre
// -> point, negated (project_points_directions).
struct Proj {
  float ux, uy, zh, dir[3];
  bool valid, valid_z;
};
NR_HD Proj project(const float* vp, float X, float Y, float Z, int h, int w) {
  Proj p;
  const float xh = fmaf(vp[2], Z, fmaf(vp[1], Y, vp[0] * X)) + vp[3];
  const float yh = fmaf(vp[6], Z, fmaf(vp[5], Y, vp[4] * X)) + vp[7];
  float zh = fmaf(vp[10], Z, fmaf(vp[9], Y, vp[8] * X)) + vp[11];
  const bool degenerate = fabsf(zh) < 1e-4f;
  if (degenerate) zh = 1e-3f;
  p.ux = xh / zh; p.uy = yh / zh; p.zh = zh;
  const bool outside = (p.ux < -0.5f) || (p.ux >= float(w) - 0.5f) || (p.uy < -0.5f) || (p.uy >= float(h) - 0.5f);
  p.valid_z = !degenerate;
  p.valid = !degenerate && !outside;
  const float dx = X - vp[12], dy = Y - vp[13], dz = Z - vp[14];
  const float inv = -1.f / fmaxf(sqrtf(dx * dx + dy * dy + dz * dz), 1e-5f);
  p.dir[0] = dx * inv; p.dir[1] = dy * inv; p.dir[2] = dz * inv;
  return p;
}

// ---- bilinear taps of interpolate_feats (ops.py:14-34) with padding_mode='border' ---------------------------------------
// Coordinates (x, y) in pixels of an h x w image, sampled from an fh x fw map; align_corners when the map is full
// resolution (render_ops.py:54-70).  Texel columns x0 <= x1 and rows y0 <= y1, weights of (y0,x0), (y0,x1), (y1,x0), (y1,x1).
struct Taps {
  int x0, x1, y0, y1;
  float w[4];
};
NR_HD Taps border_taps(float x, float y, int h, int w, int fh, int fw, bool align) {
  const float gx = x / float(w - 1) * 2.f - 1.f, gy = y / float(h - 1) * 2.f - 1.f;
  float fx = align ? (gx + 1.f) / 2.f * float(fw - 1) : ((gx + 1.f) * float(fw) - 1.f) / 2.f;
  float fy = align ? (gy + 1.f) / 2.f * float(fh - 1) : ((gy + 1.f) * float(fh) - 1.f) / 2.f;
  fx = fminf(fmaxf(fx, 0.f), float(fw - 1));
  fy = fminf(fmaxf(fy, 0.f), float(fh - 1));
  const float x0f = floorf(fx), y0f = floorf(fy);
  Taps t;
  t.x0 = int(x0f); t.y0 = int(y0f);
  t.x1 = t.x0 + 1 < fw ? t.x0 + 1 : fw - 1; t.y1 = t.y0 + 1 < fh ? t.y0 + 1 : fh - 1;
  const float we = fx - x0f, ww = (x0f + 1.f) - fx, ws = fy - y0f, wn = (y0f + 1.f) - fy;
  t.w[0] = ww * wn; t.w[1] = we * wn; t.w[2] = ww * ws; t.w[3] = we * ws;
  return t;
}
// the taps applied to one fw-wide plane
NR_HD float bilinear(const float* plane, int fw, const Taps& t) {
  return plane[t.y0 * fw + t.x0] * t.w[0] + plane[t.y0 * fw + t.x1] * t.w[1] + plane[t.y1 * fw + t.x0] * t.w[2] +
         plane[t.y1 * fw + t.x1] * t.w[3];
}
// the taps in view v of the channel-last [rfn, fh, fw, 64] feature maps: element offset of the (y0,x0) texel (a multiple
// of 64) with "x1 > x0" / "y1 > y0" in its two low bits
NR_HD int tap_code(const Taps& t, int v, int fh, int fw) {
  return (((v * fh + t.y0) * fw + t.x0) << 6) | (t.x1 > t.x0 ? 1 : 0) | (t.y1 > t.y0 ? 2 : 0);
}
// the colour of view v at a valid projection (x, y): the reference's prj_dict['rgb'] (render_ops.py:132-139, the full-
// resolution border taps with align_corners) from the [rfn, h, w, 4] RGB pack of NrPassParams::rgb.  The point kernel
// blends this colour and nr_view_colors weights it, so both read it here.
NR_HD void rgb_tap(const float* rgb, int v, float x, float y, int h, int w, float* out) {
  const Taps rt = border_taps(x, y, h, w, h, w, true);
  const float* base = rgb + size_t(v) * h * w * 4;
  const float4 t00 = ld_ro4(base + (size_t(rt.y0) * w + rt.x0) * 4), t01 = ld_ro4(base + (size_t(rt.y0) * w + rt.x1) * 4);
  const float4 t10 = ld_ro4(base + (size_t(rt.y1) * w + rt.x0) * 4), t11 = ld_ro4(base + (size_t(rt.y1) * w + rt.x1) * 4);
  const float w00 = rt.w[0], w01 = rt.w[1], w10 = rt.w[2], w11 = rt.w[3];
  out[0] = t00.x * w00 + t01.x * w01 + t10.x * w10 + t11.x * w11;
  out[1] = t00.y * w00 + t01.y * w01 + t10.y * w10 + t11.y * w11;
  out[2] = t00.z * w00 + t01.z * w01 + t10.z * w10 + t11.z * w11;
}

}  // namespace nr
