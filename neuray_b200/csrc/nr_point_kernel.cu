// Point kernel (namespace nr::pkt): everything of a render pass that is per (point, view) row, the cross-view pooling and
// the per-point layers -- reference renderer.py:171-178 up to geometry_fc, ibrnet.py:315-354.  One kernel
// (nr_point_kernel_pm3.cuh, one 128-row block per SM); this file holds what its pieces share and the launcher:
//
//   * thread r of each of the block's two compute warp groups works on (point,view) row r of the 128-row block = row r
//     of its shared-memory activation tile, row = point * G + view (G = lanes per point); the two warp groups split the
//     row's columns between them (nr_point_kernel_pm3.cuh)
//   * a layer  D[128 x N] += A[128 x K] * W^T :  A (hi and lo parts of the 3xTF32 split) is written into the activation
//     tile by the row owners, W^T (hi / lo, pre-split and pre-swizzled by nr_pack_weights) sits in shared memory, the warp
//     group multiplies them with wgmma and writes D back into the tile for the bias / activation epilogue, whose result
//     goes back into the tile as the next A; warp group c issues the MMAs of rows 64c .. 64c + 63
//   * weights stream through a 4 x 16 KB shared-memory ring filled by TMA bulk copies (cp.async.bulk) in the order of
//     stage_source; full/empty mbarriers, the "empty" barrier takes one arrival from thread 0 of each compute warp group
//     once that warp group's consuming wgmma have completed (Ring: the compute threads' side)
//   * where each layer's B sits inside its ring stage is a tcl::Tile (nr_common.cuh), shared with the weight packer
//   * TF32 mode (point_kernel_tf32, inference): the same body with one tensor-core pass per product instead of three, A
//     rounded to nearest where the 3xTF32 body splits it, B from nr_pack_weights_tf32 (rna(W) in the hi slots)
#include <type_traits>

#include "nr_common.cuh"
#include "nr_tc.cuh"

namespace nr {
namespace pkt {

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

constexpr int REC = NR_POINT_REC;
constexpr int RING_STAGE = 4096;    // 16 KB
constexpr int NBUF = 4;             // depth of the shared weight ring (the three base_fc.0 stages are held at once, so at least 3)
constexpr int SW = 2048;

// ---- small resident weights (floats inside `sw`) ----
constexpr int SW_HEAD = 0, SW_HEAD_STRIDE = 136;   // per head: L0 bias 32 | L1 bias 32 | L2 W[2][32] | L2 bias 4
constexpr int SW_PE0B = 544, SW_PE1B = 576, SW_RD0W = 608, SW_RD0B = 672, SW_RD1W = 688, SW_RD1B = 1264, SW_NF0W = 1300,
              SW_NF0B = 1556, SW_NF1W = 1564, SW_NF1B = 1572, SW_B1B = 1576, SW_V0B = 1608, SW_V1B = 1640, SW_V1LW = 1672,
              SW_V1LB = 1704, SW_V20B = 1708, SW_V21W = 1740, SW_V21B = 1772, SW_RGB0B = 1776, SW_RGB1W = 1792, SW_RGB1B = 1920,
              SW_RGB2W = 1928, SW_RGB2B = 1936,
              SW_NF0C = 1944;   // neuray_fc.0 bias seen through prob_embed.2: W_nf0 @ b_pe2 + b_nf0 (pm3 kernel)
static_assert(SW_NF0C + 8 <= SW, "small weights overflow");

struct KParams {
  NrPassParams p;
  float* dbg;
  long long* timing;   // optional: clock64() at phase boundaries, CTA 0, thread 0 of each compute warp group: [tile][2][32]
  float* rows;         // optional per-row exports, [k][rfn][rn*dn]: the colour-blend weight, then (EXPORT_AGG) w0, w2,
                       // then (EXPORT_VIEW) hit
  int P, n_tiles, n_heads;
};

// One ring stage from w_tc: up to two bulk copies (source offset in floats, bytes) x2, the second landing right behind the first
__device__ __forceinline__ void load_stage(float* slot, const float* w_tc, int4 e, uint64_t* full) {
  tc::mbar_arrive_expect_tx(full, uint32_t(e.y + e.w));
  tc::bulk_g2s(slot, w_tc + e.x, e.y, full);
  if (e.w) tc::bulk_g2s(slot + e.y / 4, w_tc + e.z, e.w, full);
}

// copies of stage s of a tile: heads, prob_embed x2, base_fc.0 x3, the view-pooled base_fc.0 inputs x5 (hi slab | lo slab
// of HST: tcl::HST_STAGE), base_fc.2, vis, vis2+rgb, geometry_fc.0 x3
__device__ __forceinline__ int4 stage_source(int s, int n_heads) {
  if (s < n_heads) return make_int4(tcl::HEAD0 + s * RING_STAGE, RING_STAGE * 4, 0, 0);
  const int t = s - n_heads;
  if (t >= 5 && t < 10) {
    const int slab = (t - 5) * tcl::HST_L.slab;
    return make_int4(tcl::HST + tcl::HST_L.hi + slab, tcl::HST_L.slab * 4, tcl::HST + tcl::HST_L.lo + slab, tcl::HST_L.slab * 4);
  }
  const int src = t == 0 ? tcl::PE0 : t == 1 ? tcl::PE1 : t <= 4 ? tcl::B0 + (t - 2) * RING_STAGE : t == 10 ? tcl::B1 : t == 11 ? tcl::V01
                : t == 12 ? tcl::V2R : tcl::G0 + (t - 13) * RING_STAGE;
  return make_int4(src, t == 1 ? tcl::PE1_SIZE * 4 : RING_STAGE * 4, 0, 0);
}

// The compute threads' side of the weight ring.  Stage i of the stream sits in slot i % NBUF, and a slot's barriers
// complete once per trip round the ring, so stage i waits on parity (i / NBUF) & 1.  wi advances by the same amount in
// every compute thread; only the leader arrives on `empty`, which counts one arrival per compute warp group.
struct Ring {
  struct Slot {
    float* p;
    uint32_t addr;              // shared-space byte address
  };
  float* base;                  // slot 0
  uint32_t base_addr;
  uint64_t *full, *empty;       // [NBUF] each
  uint32_t wi;                  // stages consumed so far
  bool leader;                  // thread 0 of the warp group: releases the stages for it
  __device__ static uint32_t slot_of(uint32_t i) { return i % NBUF; }
  __device__ static uint32_t parity(uint32_t i) { return (i / NBUF) & 1; }
  // slot of stage wi + s
  __device__ uint32_t slot_at(int s) const { return (slot_of(wi) + s) % NBUF; }
  // where stage wi + s sits (without waiting for it)
  __device__ Slot slot(int s) const {
    const uint32_t k = slot_at(s);
    return Slot{base + k * RING_STAGE, base_addr + k * (RING_STAGE * 4)};
  }
  // stage wi + s, once it has landed
  __device__ Slot wait(int s) const {
    tc::mbar_wait(full + slot_at(s), parity(wi + s));
    return slot(s);
  }
  // this warp group is done with stage wi + s: its slot may be refilled
  __device__ void release(int s) const {
    if (leader) tc::mbar_arrive(empty + slot_at(s));
  }
  __device__ void advance(int n) { wi += n; }
};

// Everything a compute thread needs to drive its block's tensor-core layers.
struct Blk {
  float* act;                   // the block's activation tile (tc::act_index)
  uint32_t act_addr;            // its shared-space byte address
  int row;                      // this thread's row of the tile = its index in its warp group
  int wg;                       // compute warp group (0, 1): issues the MMAs of rows 64 wg .. 64 wg + 63, owns columns 4 wg + [0,4) of every 8
  int rbase, key;               // act_index(row, c + 4 wg) = (c >> 5) * 4096 + rbase + ((((c & 31) >> 2) ^ key) << 2) for c % 8 == 0
};

namespace pm {
template <int G>
__device__ __forceinline__ float bmax(float x) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, o));
  return x;
}

// N independent butterflies advanced together: the N shuffles of a step are independent, so they pipeline instead of
// forming one latency chain per value (the scalar form ran the 140 pooled statistics at ~80 cycles each).
template <int G, int N>
__device__ __forceinline__ void bsum_vec(float (&x)[N]) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) {
    float t[N];
#pragma unroll
    for (int i = 0; i < N; ++i) t[i] = __shfl_xor_sync(0xffffffffu, x[i], o);
#pragma unroll
    for (int i = 0; i < N; ++i) x[i] += t[i];
  }
}

// Sum of N (16 or 32) per-row values over the G rows (views) of each point, result in every lane of the point -- through
// the warp-private transposition buffer instead of N butterflies (3 shuffles + 3 adds per value at G = 8):
//   every lane stores its row [N] (128-bit stores, row stride 36 floats: conflict-free), lane v of a point then adds up its
//   N/G columns over the point's G rows (the G lanes of a point read one contiguous N*4-byte stretch per row), writes the
//   partial row into the point's first row, and every lane reads the N sums back (broadcast reads).  ~57 instructions for
//   32 values at G = 8 against 192.  `stg`: this warp's [32][36] buffer; lane0: first lane of the point.
template <int G, int N>
__device__ __forceinline__ void pool_rows(float* stg, int lane, int lane0, int v, const float (&in)[N], float (&out)[N]) {
  static_assert(N == 16 || N == 32, "row length");
  constexpr int C = N / G > 0 ? N / G : 1;          // columns per lane (G = 32, N = 16: lanes >= 16 idle)
  constexpr int ROW = 36;
#pragma unroll
  for (int q = 0; q < N / 4; ++q) *reinterpret_cast<float4*>(stg + lane * ROW + 4 * q) = make_float4(in[4 * q], in[4 * q + 1], in[4 * q + 2], in[4 * q + 3]);
  __syncwarp();
  float acc[C];
#pragma unroll
  for (int j = 0; j < C; ++j) acc[j] = 0.f;
  const bool active = v * C < N;
  if (active) {
#pragma unroll
    for (int t = 0; t < G; ++t) {
      const float* __restrict__ src = stg + (lane0 + t) * ROW + v * C;
      if constexpr (C >= 4) {
#pragma unroll
        for (int j = 0; j < C; j += 4) {
          const float4 x = *reinterpret_cast<const float4*>(src + j);
          acc[j] += x.x; acc[j + 1] += x.y; acc[j + 2] += x.z; acc[j + 3] += x.w;
        }
      } else if constexpr (C == 2) {
        const float2 x = *reinterpret_cast<const float2*>(src);
        acc[0] += x.x; acc[1] += x.y;
      } else {
        acc[0] += src[0];
      }
    }
  }
  __syncwarp();
  if (active) {
#pragma unroll
    for (int j = 0; j < C; ++j) stg[lane0 * ROW + v * C + j] = acc[j];
  }
  __syncwarp();
#pragma unroll
  for (int q = 0; q < N / 4; ++q) {
    const float4 x = *reinterpret_cast<const float4*>(stg + lane0 * ROW + 4 * q);
    out[4 * q] = x.x; out[4 * q + 1] = x.y; out[4 * q + 2] = x.z; out[4 * q + 3] = x.w;
  }
  __syncwarp();
}

// ---- lane groups that are not a power of two (G = 5, 6, 10: PPW = 32 / G points per warp, the last 32 - PPW * G lanes idle) ----
// Butterflies do not exist for them; a group's scalars are summed through columns 32..35 of the group's rows in the same
// warp-private buffer (pool_rows only touches columns 0..31).  `idle` lanes take part in the warp syncs only.
template <int G>
__device__ __forceinline__ float gsum_np2(float* stg, int lane, int lane0, bool idle, float x) {
  stg[lane * 36 + 32] = x;
  __syncwarp();
  float s = 0.f;
  if (!idle) {
#pragma unroll
    for (int t = 0; t < G; ++t) s += stg[(lane0 + t) * 36 + 32];
  }
  __syncwarp();
  return s;
}
template <int G>
__device__ __forceinline__ float gmax_np2(float* stg, int lane, int lane0, bool idle, float x) {
  stg[lane * 36 + 32] = x;
  __syncwarp();
  float s = x;
  if (!idle) {
#pragma unroll
    for (int t = 0; t < G; ++t) s = fmaxf(s, stg[(lane0 + t) * 36 + 32]);
  }
  __syncwarp();
  return s;
}
template <int G>
__device__ __forceinline__ void gsum4_np2(float* stg, int lane, int lane0, bool idle, float (&x)[4]) {
  *reinterpret_cast<float4*>(stg + lane * 36 + 32) = make_float4(x[0], x[1], x[2], x[3]);
  __syncwarp();
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!idle) {
#pragma unroll
    for (int t = 0; t < G; ++t) {
      const float4 y = *reinterpret_cast<const float4*>(stg + (lane0 + t) * 36 + 32);
      s.x += y.x; s.y += y.y; s.z += y.z; s.w += y.w;
    }
  }
  __syncwarp();
  x[0] = s.x; x[1] = s.y; x[2] = s.z; x[3] = s.w;
}
// pool_rows for such a group: lane v adds up columns v, v + G, v + 2G, ... of the group's G rows
template <int G, int N>
__device__ __forceinline__ void pool_rows_np2(float* stg, int lane, int lane0, int v, bool idle, const float (&in)[N], float (&out)[N]) {
  constexpr int ROW = 36;
  constexpr int C = (N + G - 1) / G;
#pragma unroll
  for (int q = 0; q < N / 4; ++q) *reinterpret_cast<float4*>(stg + lane * ROW + 4 * q) = make_float4(in[4 * q], in[4 * q + 1], in[4 * q + 2], in[4 * q + 3]);
  __syncwarp();
  float acc[C];
#pragma unroll
  for (int j = 0; j < C; ++j) acc[j] = 0.f;
  if (!idle) {
#pragma unroll
    for (int t = 0; t < G; ++t) {
#pragma unroll
      for (int j = 0; j < C; ++j)
        if (v + G * j < N) acc[j] += stg[(lane0 + t) * ROW + v + G * j];
    }
  }
  __syncwarp();
  if (!idle) {
#pragma unroll
    for (int j = 0; j < C; ++j)
      if (v + G * j < N) stg[lane0 * ROW + v + G * j] = acc[j];
  }
  __syncwarp();
  if (!idle) {
#pragma unroll
    for (int q = 0; q < N / 4; ++q) {
      const float4 x = *reinterpret_cast<const float4*>(stg + lane0 * ROW + 4 * q);
      out[4 * q] = x.x; out[4 * q + 1] = x.y; out[4 * q + 2] = x.z; out[4 * q + 3] = x.w;
    }
  } else {
#pragma unroll
    for (int q = 0; q < N; ++q) out[q] = 0.f;
  }
  __syncwarp();
}

// The 64/G output columns a lane owns in the streamed per-point layers.  Lane v takes, for q = 0..CPL/4-1, the float4
// at columns q*4G + 4v: the G lanes of a point then read G consecutive 16-byte chunks (one conflict-free wavefront) for
// every q, instead of 32-byte chunks whose second halves collide in the banks.  (G = 32: two columns 2v, 2v+1.)
template <int G>
__device__ __forceinline__ int own_col(int v, int j) {
  constexpr int CPL = 64 / G;
  if constexpr (CPL == 2) return 2 * v + j;
  else return (j >> 2) * 4 * G + 4 * v + (j & 3);
}
// this lane's CPL values of a 64-wide row at `row`
template <int G>
__device__ __forceinline__ void ld_cols(const float* __restrict__ row, int v, float* w) {
  constexpr int CPL = 64 / G;
  if constexpr (CPL == 2) {
    const float2 t = *reinterpret_cast<const float2*>(row + 2 * v);
    w[0] = t.x; w[1] = t.y;
  } else {
#pragma unroll
    for (int q = 0; q < CPL / 4; ++q) {
      const float4 t = *reinterpret_cast<const float4*>(row + q * 4 * G + 4 * v);
      w[4 * q] = t.x; w[4 * q + 1] = t.y; w[4 * q + 2] = t.z; w[4 * q + 3] = t.w;
    }
  }
}

}  // namespace pm

#include "nr_point_kernel_pm3.cuh"

}  // namespace pkt

// TF32: the TF32-mode kernel (release form only), else the 3xTF32 one; EXPORTS: the release form with that export set
// (kp.rows): EXPORT_BLEND alone, with EXPORT_AGG, or with EXPORT_AGG and EXPORT_VIEW
template <int G, bool DEBUG, bool TF32, int EXPORTS = 0>
static int launch_pm3_inst(const pkt::KParams& kp, int grid, cudaStream_t stream) {
  static_assert(!(TF32 && DEBUG) && !(EXPORTS && DEBUG), "the TF32 mode and the exports have no debug form");
  static_assert(EXPORTS == 0 || EXPORTS == EXPORT_BLEND || EXPORTS == (EXPORT_BLEND | EXPORT_AGG) ||
                    EXPORTS == (EXPORT_BLEND | EXPORT_AGG | EXPORT_VIEW),
                "export sets");
  void (*fn)(const pkt::KParams);
  if constexpr (EXPORTS & EXPORT_VIEW) fn = pkt::pm3::point_kernel_view<G, TF32 ? 1 : 3>;
  else if constexpr (EXPORTS == (EXPORT_BLEND | EXPORT_AGG)) fn = pkt::pm3::point_kernel_agg<G, TF32 ? 1 : 3>;
  else if constexpr (EXPORTS == EXPORT_BLEND) fn = pkt::pm3::point_kernel_blend<G, TF32 ? 1 : 3>;
  else if constexpr (TF32) fn = pkt::pm3::point_kernel_tf32<G>;
  else fn = pkt::pm3::point_kernel_pm3<G, DEBUG>;
  if (opt_in_smem((const void*)fn, pkt::pm3::SMEM_BYTES, "point kernel") != NR_OK) return NR_E_CUDA;
  fn<<<grid, pkt::pm3::NTHR, pkt::pm3::SMEM_BYTES, stream>>>(kp);
  NR_CHECK_LAUNCH(EXPORTS & EXPORT_VIEW  ? "point_kernel_view"
                  : EXPORTS & EXPORT_AGG ? "point_kernel_agg"
                  : EXPORTS              ? "point_kernel_blend"
                  : TF32                 ? "point_kernel_tf32"
                                         : "point_kernel_pm3");
  return NR_OK;
}

template <int G>
static int launch_pm3(pkt::KParams kp, int exports, bool tf32, cudaStream_t stream) {
  constexpr int PB = 4 * (32 / G);       // points per 128-row block: 32 / G per warp (G not a power of two leaves 32 % G lanes idle)
  const long long N = (long long)kp.p.rn * kp.p.dn;
  kp.P = PB;
  kp.n_tiles = int((N + PB - 1) / PB);
  int sms;
  if (sm_count(&sms, "point kernel") != NR_OK) return NR_E_CUDA;
  const int grid = kp.n_tiles < sms ? kp.n_tiles : sms;
  constexpr int AGG = EXPORT_BLEND | EXPORT_AGG, VIEW = EXPORT_BLEND | EXPORT_AGG | EXPORT_VIEW;
  if (exports & EXPORT_VIEW)
    return tf32 ? launch_pm3_inst<G, false, true, VIEW>(kp, grid, stream) : launch_pm3_inst<G, false, false, VIEW>(kp, grid, stream);
  if (exports & EXPORT_AGG)
    return tf32 ? launch_pm3_inst<G, false, true, AGG>(kp, grid, stream) : launch_pm3_inst<G, false, false, AGG>(kp, grid, stream);
  if (exports)
    return tf32 ? launch_pm3_inst<G, false, true, EXPORT_BLEND>(kp, grid, stream) : launch_pm3_inst<G, false, false, EXPORT_BLEND>(kp, grid, stream);
  if (tf32) return launch_pm3_inst<G, false, true>(kp, grid, stream);
  return (kp.dbg || kp.timing) ? launch_pm3_inst<G, true, false>(kp, grid, stream) : launch_pm3_inst<G, false, false>(kp, grid, stream);
}

// `timing`: optional clock64() stamps at the phase boundaries (nr_point_kernel_timing), passed per call.  tf32: the TF32
// mode (p->w_tc from nr_pack_weights_tf32), which has neither the debug tap nor the stamps.  exports: 0, EXPORT_BLEND
// ([rfn][rn*dn] colour-blend weights in rows: nr_render_pass_fwd_blend / _tf32_blend) or EXPORT_BLEND | EXPORT_AGG
// ([3][rfn][rn*dn]: those, then w0 and w2: nr_render_pass_fwd_agg / _tf32_agg) or all three with EXPORT_VIEW
// ([4][rfn][rn*dn]: those, then the masked hit probability: nr_render_pass_fwd_view / _tf32_view), in either mode.
int launch_point_kernel(const NrPassParams* p, float* dbg, long long* timing, float* rows, int exports, bool tf32, cudaStream_t stream) {
  NR_CHECK_ARG(p != nullptr, "params");
  NR_CHECK_ARG(!tf32 || (dbg == nullptr && timing == nullptr), "the TF32 point kernel has no debug tap or phase stamps");
  NR_CHECK_ARG(exports == 0 || exports == EXPORT_BLEND || exports == (EXPORT_BLEND | EXPORT_AGG) ||
                   exports == (EXPORT_BLEND | EXPORT_AGG | EXPORT_VIEW),
               "export set");
  NR_CHECK_ARG(!exports || (dbg == nullptr && timing == nullptr), "the exports have no debug tap or phase stamps");
  NR_CHECK_ARG(p->coords && p->que_depth && p->que_cam && p->feat && p->rgb && p->view_params && p->w_point && p->point_rec,
               "null device pointer");
  NR_CHECK_ARG(p->w_tc != nullptr, "w_tc (tensor-core weight buffer, nr_pack_weights) is required");
  NR_CHECK_ARG(p->rfn >= 1 && p->rfn <= NR_MAX_VIEWS, "rfn out of range");
  NR_CHECK_ARG(p->dn >= 3 && p->dn <= NR_MAX_SAMPLES, "dn out of range");
  NR_CHECK_ARG(p->rn >= 0, "rn");
  NR_CHECK_ARG(p->h > 1 && p->w > 1 && p->fh > 0 && p->fw > 0, "map shape");
  NR_CHECK_ARG((long long)p->rn * p->dn < (1ll << 31) / NR_POINT_REC, "too many points for one call; chunk the rays");
  NR_CHECK_ARG((long long)p->rfn * p->fh * p->fw * 64 < (1ll << 31), "feature maps too large for 32-bit texel offsets");
  if (p->rn == 0) return NR_OK;
  pkt::KParams kp;
  kp.p = *p;
  kp.dbg = dbg;
  kp.timing = timing;
  kp.rows = rows;
  kp.n_heads = p->use_vis ? 4 : 3;
  // lanes per point: the smallest group size that holds the views and wastes the fewest of a warp's 32 lanes
  if (p->rfn <= 4) return launch_pm3<4>(kp, exports, tf32, stream);
  if (p->rfn == 5) return launch_pm3<5>(kp, exports, tf32, stream);      // 6 points per warp (30 lanes) instead of 4 groups of 8
  if (p->rfn == 6) return launch_pm3<6>(kp, exports, tf32, stream);      // 5 points per warp
  if (p->rfn <= 8) return launch_pm3<8>(kp, exports, tf32, stream);
  if (p->rfn <= 10) return launch_pm3<10>(kp, exports, tf32, stream);    // 3 points per warp instead of 2 groups of 16 (cfg4: 10 views)
  if (p->rfn <= 16) return launch_pm3<16>(kp, exports, tf32, stream);
  return launch_pm3<32>(kp, exports, tf32, stream);
}

}  // namespace nr
