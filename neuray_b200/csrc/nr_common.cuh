// Shared device helpers + the packed weight layout (single source of truth for host and kernels).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/neuray_b200.h"

namespace nr {

void set_error(const char* fmt, ...);

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

}  // namespace nr
