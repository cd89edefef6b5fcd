// Point kernel (namespace nr::pkt::pm3): point-major rows, wgmma layers, one 128-row block per SM.
//
// Row = point * G + view inside a block (G lanes per point: 4, 5, 6, 8, 10, 16 or 32), thread r of the block's warp group =
// row r of the activation tile; a thread keeps its row in registers from the gather to the output record.  Resource plan
// (one CTA per SM: 128 compute threads + a 128-thread producer group whose lane 0 feeds the weight ring, see
// NR_PRODUCER_WARP below):
//   * activation tile (80 KB of shared memory, 160 columns x 128 rows, tc::act_index): hi parts at columns [0,64), lo parts
//     at [64,128), accumulator at [128,160).  base_fc.0 (N = 64) is issued in K rounds into one accumulator at [96,160):
//     round A (the 32 neuray_feat inputs) right after prob_embed.2 while they are still the only live A operand, round B
//     (the 40 rgb_feat inputs, lo parts at [48,88)) after ray_dir_fc, then five rounds of view-pooled statistics (K 32
//     each).  Its epilogue reads the accumulator half by half and writes base_fc.2's operand over the columns it has
//     already consumed.
//   * the rest of shared memory: 4 x 16 KB weight ring (TMA bulk copies, fed by the producer group; the view-pooled
//     base_fc.0 inputs stream through it as five more stages), the resident tile of ray_dir_fc.2, small weights, camera
//     blocks, and one [32][36] transposition buffer per warp: gather (two channel passes: ray_feats, then img_feats, which
//     stay there until ray_dir_fc needs them), the cross-view pooling (pm::pool_rows) and the lane-group sums of the
//     non-power-of-two groups all go through it.
//   * a layer is one wgmma round trip of the warp group (issue, wait, accumulator back into the tile): the 227 KB of shared
//     memory hold one activation tile next to the ring, so a second block per SM would have to give up the ring.
#pragma once

namespace pm3 {

using pm::bsum;
using pm::bmax;
using pm::bsum_vec;
using pm::own_col;
using pm::ld_cols;
using pm::pool_rows;
using pm::pool_rows_np2;
using pm::gsum_np2;
using pm::gmax_np2;
using pm::gsum4_np2;

#ifndef NR_GATHER_BATCH
#define NR_GATHER_BATCH 2     // 4 (16 loads in flight per lane) spills
#endif
constexpr int GB = NR_GATHER_BATCH;                           // rows whose 4 taps a quarter-warp keeps in flight at once (4 x GB 128-bit loads per lane)
#ifndef NR_GATHER_OVERLAP
#define NR_GATHER_OVERLAP 1
#endif
constexpr int NBLK = 1;
#ifndef NR_PRODUCER_WARP
#define NR_PRODUCER_WARP 1
#endif
constexpr int NCOMP = NBLK * 128;
// + one warp group whose lane 0 does nothing but keep the weight ring full
constexpr int NTHR = NCOMP + (NR_PRODUCER_WARP ? 128 : 0);
constexpr int TCOLS = 160;                                    // activation-tile columns per block
constexpr int ACT = (TCOLS / 32) * 4096;                      // floats per activation tile

// ---- shared memory map (floats) ----
constexpr int OFF_RING = 0;                                   // NBUF x RING_STAGE
constexpr int OFF_ACT = OFF_RING + NBUF * RING_STAGE;         // NBLK activation tiles (1024-byte aligned)
constexpr int OFF_RD1 = OFF_ACT + NBLK * ACT;                 // ray_dir_fc.2 tensor-core tile (resident, 1024-byte aligned)
constexpr int OFF_WG1 = OFF_RD1 + tcl::RD1_SIZE;              // geometry_fc.2: [16][64] (output-major, columns in own_col order) | bias[16]
constexpr int WG1 = 64 * 16 + 16;
constexpr int OFF_SW = OFF_WG1 + WG1;                         // small resident weights (offsets SW_*, nr_point_kernel.cu)
constexpr int OFF_STG = OFF_SW + SW;                          // gather transposition: per warp [32 rows][36]
constexpr int STG_ROW = 36;
constexpr int STG = (NCOMP / 32) * 32 * STG_ROW;
constexpr int OFF_CAM = OFF_STG + STG;                        // que_cam [24] (padded to 32) | view_params [NR_MAX_VIEWS][20]
constexpr int CAM = 32 + NR_MAX_VIEWS * 20;
constexpr int OFF_STAB = OFF_CAM + CAM;                       // Producer::table: int4 per stage of a tile (at most 4 + 16)
constexpr int OFF_BAR = OFF_STAB + 80;
constexpr int SMEM_FLOATS = OFF_BAR + 32;
constexpr size_t SMEM_BYTES = size_t(SMEM_FLOATS) * 4;
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");
static_assert(OFF_STAB % 4 == 0, "alignment");
static_assert((OFF_ACT * 4) % 1024 == 0 && (OFF_RD1 * 4) % 1024 == 0 && OFF_WG1 % 4 == 0 && OFF_SW % 4 == 0 && OFF_STG % 4 == 0, "alignment");

// Layer issue, executed by all 128 threads of the block after they wrote their A columns.  K chunk c (of NCH) reads A
// columns AHI + 8c (c < NLIN) or TAILHI + 8(c - NLIN), lo parts LOOFF columns further, and B chunk CB0 + c of the layer's
// tiles (slab (CB0+c)/4; one ring stage per slab when NSTG > 1); ACC: the first MMA accumulates onto what is already in the
// accumulator columns [DCOL, DCOL + N).  Returns with the outputs in the activation tile, visible to every row owner.
template <int N, int NCH, int AHI, int LOOFF, int NLIN, int TAILHI, int DCOL, int CB0, int NSTG, uint32_t OFF_HI, uint32_t OFF_LO,
          uint32_t SLAB, bool WAIT_FULL, bool RELEASE, bool ACC>
__device__ __forceinline__ void issue_layer(Blk& b) {
  // b.tk: diagnostics of ONE layer's round trip (debug instantiation only; a compile-time null otherwise)
  if (b.tk) b.tk[0] = clock64();
  tc::fence_proxy_async_smem();              // this thread's A columns -> visible to the tensor cores
  if (b.tk) b.tk[1] = clock64();
  tc::named_sync(2 + b.blk, 128);
  if (b.tk) b.tk[2] = clock64();
  const uint32_t st0 = b.wi % NBUF;
  if (WAIT_FULL && b.prod != nullptr) b.prod->feed(b.wi + NSTG - 1);
  if (WAIT_FULL) {
#pragma unroll
    for (int s = 0; s < NSTG; ++s) tc::mbar_wait(b.wfull + ((st0 + s) % NBUF), ((b.wi + s) / NBUF) & 1);
  }
  if (b.tk) b.tk[3] = clock64();
  float d[2][N / 2];
  if (ACC) tc::acc_load<N>(b.act, DCOL, b.row, d);
  else {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < N / 2; ++j) d[h][j] = 0.f;
  }
  uint64_t dhi[NSTG], dlo[NSTG];
#pragma unroll
  for (int s = 0; s < NSTG; ++s) {
    const uint32_t base = b.ring_addr + ((st0 + s) % NBUF) * (RING_STAGE * 4);
    dhi[s] = tc::smem_desc_sw128(base + OFF_HI);
    dlo[s] = tc::smem_desc_sw128(base + OFF_LO);
  }
  tc::wgmma_fence_operand(d[0]);
  tc::wgmma_fence_operand(d[1]);
  tc::wgmma_fence();
#pragma unroll
  for (int ps = 0; ps < 3; ++ps) {
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int acol = (c < NLIN ? AHI + 8 * c : TAILHI + 8 * (c - NLIN)) + (ps == 1 ? LOOFF : 0);
      const int cb = CB0 + c;
      const int slab = cb >> 2;
      const int stg = NSTG == 1 ? 0 : slab;
      const uint32_t inc = ((NSTG == 1 ? slab * SLAB : 0u) + (cb & 3) * 32) >> 4;
      const uint64_t bd = (ps == 2 ? dlo[stg] : dhi[stg]) + inc;
      tc::wgmma_tf32<N>(d[0], tc::act_desc(b.act_addr, acol, 0), bd);
      tc::wgmma_tf32<N>(d[1], tc::act_desc(b.act_addr, acol, 1), bd);
    }
  }
  tc::wgmma_commit();
  if (b.tk) b.tk[4] = clock64();
  tc::wgmma_wait_all();
  tc::wgmma_fence_operand(d[0]);
  tc::wgmma_fence_operand(d[1]);
  if (b.tk) b.tk[5] = clock64();
  tc::acc_store<N>(b.act, DCOL, b.row, d);
  tc::named_sync(2 + b.blk, 128);            // outputs in the tile; every warp's reads of the stages have completed
  if (RELEASE) {
    if (b.leader) {
#pragma unroll
      for (int s = 0; s < NSTG; ++s) tc::mbar_arrive(b.wempty + ((st0 + s) % NBUF));
    }
    b.wi += NSTG;
  }
  if (b.tk) b.tk[6] = clock64();
}
// Same, B operand = a resident shared-memory tile at byte address `base` (hi slabs first, SLAB bytes apart; lo parts
// OFF_LO bytes further): no ring accounting.
template <int N, int NCH, int AHI, int LOOFF, int DCOL, int CB0, uint32_t OFF_LO, uint32_t SLAB, bool ACC>
__device__ __forceinline__ void issue_layer_resident(Blk& b, uint32_t base) {
  tc::fence_proxy_async_smem();
  tc::named_sync(2 + b.blk, 128);
  float d[2][N / 2];
  if (ACC) tc::acc_load<N>(b.act, DCOL, b.row, d);
  else {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < N / 2; ++j) d[h][j] = 0.f;
  }
  const uint64_t dhi = tc::smem_desc_sw128(base), dlo = tc::smem_desc_sw128(base + OFF_LO);
  tc::wgmma_fence_operand(d[0]);
  tc::wgmma_fence_operand(d[1]);
  tc::wgmma_fence();
#pragma unroll
  for (int ps = 0; ps < 3; ++ps) {
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int acol = AHI + 8 * c + (ps == 1 ? LOOFF : 0);
      const int cb = CB0 + c;
      const uint32_t inc = ((cb >> 2) * SLAB + (cb & 3) * 32) >> 4;
      const uint64_t bd = (ps == 2 ? dlo : dhi) + inc;
      tc::wgmma_tf32<N>(d[0], tc::act_desc(b.act_addr, acol, 0), bd);
      tc::wgmma_tf32<N>(d[1], tc::act_desc(b.act_addr, acol, 1), bd);
    }
  }
  tc::wgmma_commit();
  tc::wgmma_wait_all();
  tc::wgmma_fence_operand(d[0]);
  tc::wgmma_fence_operand(d[1]);
  tc::acc_store<N>(b.act, DCOL, b.row, d);
  tc::named_sync(2 + b.blk, 128);
}
// the common case: activations hi [0,64) / lo [64,128), accumulator at 128, one ring stage
template <int N, int NCH, int AHI, int NLIN, int TAILHI, uint32_t OFF_HI, uint32_t OFF_LO, uint32_t SLAB, bool WAIT_FULL, bool RELEASE>
__device__ __forceinline__ void run_layer(Blk& b) {
  issue_layer<N, NCH, AHI, 64, NLIN, TAILHI, 128, 0, 1, OFF_HI, OFF_LO, SLAB, WAIT_FULL, RELEASE, false>(b);
}

// this thread's row of the activation tile: columns [col, col + 4Q), col a multiple of 4
template <int Q>
__device__ __forceinline__ void ld_row(const Blk& b, int col, float* v) {
#pragma unroll
  for (int q = 0; q < Q; ++q) {
    const float4 t = *reinterpret_cast<const float4*>(b.act + tc::act_index(b.row, col + 4 * q));
    v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
  }
}
template <int Q>
__device__ __forceinline__ void st_split(const Blk& b, int hi, int lo, const float* v) {
#pragma unroll
  for (int q = 0; q < Q; ++q) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) tc::split_tf32(v[4 * q + j], h[j], l[j]);
    *reinterpret_cast<uint4*>(b.act + tc::act_index(b.row, hi + 4 * q)) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(b.act + tc::act_index(b.row, lo + 4 * q)) = make_uint4(l[0], l[1], l[2], l[3]);
  }
}
__device__ __forceinline__ void ld32(const Blk& b, int col, float* v) { ld_row<8>(b, col, v); }
__device__ __forceinline__ void ld16(const Blk& b, int col, float* v) { ld_row<4>(b, col, v); }
// 16 / 32 / 8 activations -> hi parts at `hi`, lo parts at `lo`
__device__ __forceinline__ void st16(const Blk& b, int hi, int lo, const float* v) { st_split<4>(b, hi, lo, v); }
__device__ __forceinline__ void st32(const Blk& b, int hi, int lo, const float* v) { st_split<8>(b, hi, lo, v); }
__device__ __forceinline__ void st8(const Blk& b, int hi, int lo, const float* v) { st_split<2>(b, hi, lo, v); }

template <int G, bool DEBUG>
__global__ void __launch_bounds__(NTHR, 1) point_kernel_pm3(const KParams kp) {
  extern __shared__ __align__(1024) float smem[];
  constexpr bool P2 = (G & (G - 1)) == 0;      // power-of-two lane groups reduce with butterflies, the others through shared memory
  constexpr int PPW = 32 / G;                   // points per warp (G = 10: 3, two lanes idle)
  constexpr int PB = 4 * PPW;                   // points per block
  constexpr int GE = G >= 32 ? 32 : G >= 16 ? 16 : G >= 8 ? 8 : 4;   // lanes of a point that share geometry_fc's 64 hidden units
  constexpr int CPL = 64 / GE;                  // geometry_fc.0 output columns per such lane
  static_assert(G == 4 || G == 5 || G == 6 || G == 8 || G == 10 || G == 16 || G == 32, "lanes per point");
  const NrPassParams& pp = kp.p;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  float* const ring = smem + OFF_RING;
  float* const sWg1 = smem + OFF_WG1;
  float* const sw = smem + OFF_SW;
  uint64_t* const bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* const wfull = bars;
  uint64_t* const wempty = bars + NBUF;
  uint64_t* const res_bar = bars + 2 * NBUF;                  // resident tensor-core tile has landed

  const int rfn = pp.rfn, dn = pp.dn;
  const int N = pp.rn * dn;
  const int n_heads = kp.n_heads;
  const int stages_per_tile = n_heads + 16;                    // Producer::stage_source
  const int n_tiles = kp.n_tiles;                              // tiles of PB points
  const int iters = (n_tiles + int(gridDim.x) * NBLK - 1) / (int(gridDim.x) * NBLK);
  const float* __restrict__ W = pp.w_point;

  // ---------------- one-time setup ----------------
  if (tid == 0) {
    for (int i = 0; i < NBUF; ++i) { tc::mbar_init(wfull + i, 1); tc::mbar_init(wempty + i, NBLK); }
    tc::mbar_init(res_bar, 1);
    tc::fence_mbar_init();
    tc::mbar_arrive_expect_tx(res_bar, tcl::RD1_SIZE * 4);
    tc::bulk_g2s(smem + OFF_RD1, pp.w_tc + tcl::RD1, tcl::RD1_SIZE * 4, res_bar);
  }
  if (tid < NCOMP) {
    auto cp = [&](float* dst, int src, int n) { for (int i = tid; i < n; i += NCOMP) dst[i] = __ldg(W + src + i); };
    for (int hh = 0; hh < 4; ++hh) {
      const int g = lay::DD_HEAD + hh * lay::DD_HEAD_STRIDE;
      float* d = sw + SW_HEAD + hh * SW_HEAD_STRIDE;
      cp(d, g + lay::DD_L0_B, 32); cp(d + 32, g + lay::DD_L1_B, 32); cp(d + 64, g + lay::DD_L2_W, 64); cp(d + 128, g + lay::DD_L2_B, 4);
    }
    const int gb = lay::GRP_B, gd = lay::GRP_D1;
    cp(sw + SW_PE0B, gb + lay::PE0_B, 32); cp(sw + SW_PE1B, gb + lay::PE1_B, 32); cp(sw + SW_RD0W, gb + lay::RD0_W, 64);
    cp(sw + SW_RD0B, gb + lay::RD0_B, 16); cp(sw + SW_RD1W, gb + lay::RD1_W, 576); cp(sw + SW_RD1B, gb + lay::RD1_B, 36);
    cp(sw + SW_NF0W, gb + lay::NF0_W, 256); cp(sw + SW_NF0B, gb + lay::NF0_B, 8); cp(sw + SW_NF1W, gb + lay::NF1_W, 8);
    cp(sw + SW_NF1B, gb + lay::NF1_B, 4); cp(sw + SW_B1B, lay::BASE1_B, 32);
    cp(sw + SW_V0B, gd + lay::VIS0_B, 32); cp(sw + SW_V1B, gd + lay::VIS1_B, 32); cp(sw + SW_V1LW, gd + lay::VIS1L_W, 32);
    cp(sw + SW_V1LB, gd + lay::VIS1L_B, 4); cp(sw + SW_V20B, gd + lay::V20_B, 32); cp(sw + SW_V21W, gd + lay::V21_W, 32);
    cp(sw + SW_V21B, gd + lay::V21_B, 4); cp(sw + SW_RGB0B, gd + lay::RGB0_B, 16); cp(sw + SW_RGB1W, gd + lay::RGB1_W, 128);
    cp(sw + SW_RGB1B, gd + lay::RGB1_B, 8); cp(sw + SW_RGB2W, gd + lay::RGB2_W, 8); cp(sw + SW_RGB2B, gd + lay::RGB2_B, 4);
    // WT[64][16] -> [16][64]; hidden unit c = v*CPL + j sits where lane v's j-th own column is (conflict-free ld_cols)
    for (int i = tid; i < 64 * 16; i += NCOMP)
      sWg1[(i & 15) * 64 + own_col<GE>((i >> 4) / CPL, (i >> 4) % CPL)] = __ldg(W + lay::GRP_D2 + lay::GEO1_W + i);
    cp(sWg1 + 64 * 16, lay::GRP_D2 + lay::GEO1_B, 16);
    if (tid < stages_per_tile) reinterpret_cast<int4*>(smem + OFF_STAB)[tid] = Producer::stage_source(tid, n_heads);
    for (int i = tid; i < 24; i += NCOMP) smem[OFF_CAM + i] = __ldg(pp.que_cam + i);
    for (int i = tid; i < pp.rfn * 20; i += NCOMP) smem[OFF_CAM + 32 + i] = __ldg(pp.view_params + i);
  }
  __syncthreads();
  tc::mbar_wait(res_bar, 0);
  if (tid < 8) {   // neuray_fc.0 rides on prob_embed.2's MMA (8 extra output rows): its bias as seen through that layer
    float acc = sw[SW_NF0B + tid];
    for (int j = 0; j < 32; ++j) acc = fmaf(sw[SW_NF0W + j * 8 + tid], sw[SW_PE1B + j], acc);
    sw[SW_NF0C + tid] = acc;
  }
  __syncthreads();

#if NR_PRODUCER_WARP
  if (tid >= NCOMP) {
    // ---------------- producer warp: a stage goes out the moment its ring slot is free ----------------
    // (fed from a compute thread's issue path, a load only started at that thread's next layer: ~500-850 cycles of every
    // layer's round trip were the issuing lane waiting for weights)
    if (tid == NCOMP) {
      const int4* table = reinterpret_cast<const int4*>(smem + OFF_STAB);
      const uint32_t total = uint32_t(iters) * uint32_t(stages_per_tile);
      int s = 0;
      for (uint32_t n = 0; n < total; ++n) {
        const uint32_t buf = n % NBUF;
        if (n >= NBUF) tc::mbar_wait(wempty + buf, ((n / NBUF) - 1) & 1);
        load_stage(ring + buf * RING_STAGE, pp.w_tc, table[s], wfull + buf);
        if (++s == stages_per_tile) s = 0;
      }
    }
    __syncwarp();
  } else
#endif
  {
    // ---------------- compute warps ----------------
    const int fh = pp.fh, fw = pp.fw, h = pp.h, w = pp.w;
    const bool feat_align = (fh == h && fw == w);
    const int grp = lane / G;                       // point of this lane inside the warp (>= PPW: idle lane)
    const bool idle = P2 ? false : grp >= PPW;     // a compile-time false for the power-of-two groups
    const int v = P2 ? lane % G : lane - grp * G;   // view of this row (>= rfn: padding lane)
    const int pl = P2 ? (tid & 127) / G : (warp & 3) * PPW + grp;   // point inside the block
    const int lane0 = lane - v;                     // first lane of this point's group
    float* const stg = smem + OFF_STG + warp * 32 * STG_ROW;
    // sums / maxima over the lanes of a point
    auto gsum = [&](float x) { if constexpr (P2) return bsum<G>(x); else return gsum_np2<G>(stg, lane, lane0, idle, x); };
    auto gmax = [&](float x) { if constexpr (P2) return bmax<G>(x); else return gmax_np2<G>(stg, lane, lane0, idle, x); };
    auto gpool32 = [&](const float (&in)[32], float (&out)[32]) {
      if constexpr (P2) pool_rows<G, 32>(stg, lane, lane0, v, in, out); else pool_rows_np2<G, 32>(stg, lane, lane0, v, idle, in, out);
    };

    Blk b;
    b.blk = warp >> 2;
    b.leader = (tid & 127) == 0;
    b.act = smem + OFF_ACT + ACT * b.blk;
    b.act_addr = tc::smem_u32(b.act);
    b.row = tid & 127;
    b.wfull = wfull; b.wempty = wempty;
    b.ring_addr = tc::smem_u32(ring);
    b.wi = 0;
    b.tk = nullptr;
    Producer prod;
    prod.w_tc = pp.w_tc; prod.ring = ring; prod.wfull = wfull; prod.wempty = wempty;
    prod.next = 0; prod.total = uint32_t(iters) * uint32_t(stages_per_tile);
    prod.stages_per_tile = stages_per_tile; prod.s = 0; prod.table = reinterpret_cast<const int4*>(smem + OFF_STAB);
#if NR_PRODUCER_WARP
    b.prod = nullptr;
    (void)prod;
#else
    b.prod = tid == 0 ? &prod : nullptr;                       // thread 0 feeds the ring from inside its own issue path
    if (tid == 0) prod.feed(0);
#endif

  // phase stamps exist only in the DEBUG instantiation (nr_point_kernel_timing / nr_point_kernel_debug)
#define PM_TICK(id)                                                                                      \
  if constexpr (DEBUG) {                                                                                 \
    if (kp.timing != nullptr && blockIdx.x == 0 && b.leader && b.blk < 2 && it < 64) kp.timing[(it * 2 + b.blk) * 32 + (id)] = clock64(); \
  }
    for (int it = 0; it < iters; ++it) {
      const int tile = (it * int(gridDim.x) + int(blockIdx.x)) * NBLK + b.blk;
      if (tile >= n_tiles) {
        // nothing to render in this iteration: still take part in the weight-ring accounting
        for (int s = 0; s < stages_per_tile; ++s) {
          if (b.leader) {
            const uint32_t i = b.wi + s;
            if (b.prod) b.prod->feed(i);
            tc::mbar_wait(wfull + (i % NBUF), (i / NBUF) & 1);
            tc::mbar_arrive(wempty + (i % NBUF));
          }
        }
        b.wi += stages_per_tile;
        continue;
      }
      const int n = tile * PB + pl;
      const bool pt_ok = P2 ? n < N : (n < N && !idle);
      const bool row_ok = pt_ok && v < rfn;

      PM_TICK(0)
      // ---------------- ray geometry of this row's point (every lane of the group computes the same values) ----------------
      float X = 0.f, Y = 0.f, Z = 0.f, qx = 0.f, qy = 0.f, qz = 0.f, ihp = 0.f, ihc = 0.f;
      if (pt_ok) {
        const float* cam = smem + OFF_CAM;
        const int ray = n / dn, s = n - ray * dn;
        const float cx = __ldg(pp.coords + 2 * ray), cy = __ldg(pp.coords + 2 * ray + 1);
        float cm[3], d[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) cm[i] = fmaf(cam[12 + 3 * i + 1], cy, cam[12 + 3 * i] * cx) + cam[12 + 3 * i + 2];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const float wld = fmaf(cam[3 * i + 2], cm[2], fmaf(cam[3 * i + 1], cm[1], cam[3 * i] * cm[0])) + cam[9 + i];
          d[i] = wld - cam[9 + i];   // the reference adds the centre and subtracts it again (render_ops.py:22-23)
        }
        const float z = __ldg(pp.que_depth + n);
        X = fmaf(d[0], z, cam[9]); Y = fmaf(d[1], z, cam[10]); Z = fmaf(d[2], z, cam[11]);
        const float nrm = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        qx = -d[0] / nrm; qy = -d[1] / nrm; qz = -d[2] / nrm;
        const float a = -1.f / cam[21], bb = -1.f / cam[22];
        const float tcur = (-1.f / z - a) / (bb - a);
        float dc = 1e6f;
        if (s + 1 < dn) dc = (-1.f / __ldg(pp.que_depth + n + 1) - a) / (bb - a) - tcur;
        float dp = dc;
        if (s > 0) dp = tcur - (-1.f / __ldg(pp.que_depth + n - 1) - a) / (bb - a);
        ihc = dc * 0.5f; ihp = dp * 0.5f;
      }

      // ---------------- projection into this row's view + rgb taps ----------------
      float mrow = 0.f, zrow = 1.f, dd[4] = {0.f, 0.f, 0.f, 0.f}, fxr = 0.f, fyr = 0.f, rgbin[3] = {0.f, 0.f, 0.f};
      float dbg_px = 0.f, dbg_py = 0.f, dbg_dir[3] = {0.f, 0.f, 0.f};
      int tcode = -1;
      float tw[4] = {0.f, 0.f, 0.f, 0.f};
      if (row_ok) {
        const float* vp = smem + OFF_CAM + 32 + v * 20;
        const float xh = fmaf(vp[2], Z, fmaf(vp[1], Y, vp[0] * X)) + vp[3];
        const float yh = fmaf(vp[6], Z, fmaf(vp[5], Y, vp[4] * X)) + vp[7];
        float zh = fmaf(vp[10], Z, fmaf(vp[9], Y, vp[8] * X)) + vp[11];
        const bool degenerate = fabsf(zh) < 1e-4f;
        if (degenerate) zh = 1e-3f;
        const float ux = xh / zh, uy = yh / zh;
        const bool outside = (ux < -0.5f) || (ux >= float(w) - 0.5f) || (uy < -0.5f) || (uy >= float(h) - 0.5f);
        const bool valid = !degenerate && !outside;
        mrow = valid ? 1.f : 0.f;
        zrow = zh;
        const float dx = X - vp[12], dy = Y - vp[13], dz = Z - vp[14];
        const float inv = -1.f / fmaxf(sqrtf(dx * dx + dy * dy + dz * dz), 1e-5f);
        const float ex = dx * inv, ey = dy * inv, ez = dz * inv;
        dd[0] = ex - qx; dd[1] = ey - qy; dd[2] = ez - qz; dd[3] = ex * qx + ey * qy + ez * qz;
        if (DEBUG) { dbg_px = ux; dbg_py = uy; dbg_dir[0] = ex; dbg_dir[1] = ey; dbg_dir[2] = ez; }
        const float gx = ux / float(w - 1) * 2.f - 1.f, gy = uy / float(h - 1) * 2.f - 1.f;
        fxr = feat_align ? (gx + 1.f) / 2.f * float(fw - 1) : ((gx + 1.f) * float(fw) - 1.f) / 2.f;
        fyr = feat_align ? (gy + 1.f) / 2.f * float(fh - 1) : ((gy + 1.f) * float(fh) - 1.f) / 2.f;
        fxr = fminf(fmaxf(fxr, 0.f), float(fw - 1)); fyr = fminf(fmaxf(fyr, 0.f), float(fh - 1));
        if (valid) {
          // feature-map taps of this row, worked out once here instead of by each of the gathering lanes: element offset
          // of the (y0,x0) texel (a multiple of 64) with "x1 > x0" / "y1 > y0" in its two low bits, and the four weights
          const float x0f = floorf(fxr), y0f = floorf(fyr);
          const int x0 = int(x0f), y0 = int(y0f);
          const float we = fxr - x0f, ww = (x0f + 1.f) - fxr, ws = fyr - y0f, wn = (y0f + 1.f) - fyr;
          tcode = (((v * fh + y0) * fw + x0) << 6) | (x0 + 1 <= fw - 1 ? 1 : 0) | (y0 + 1 <= fh - 1 ? 2 : 0);
          tw[0] = ww * wn; tw[1] = we * wn; tw[2] = ww * ws; tw[3] = we * ws;
        }
        if (valid) {
          float ix = (gx + 1.f) / 2.f * float(w - 1), iy = (gy + 1.f) / 2.f * float(h - 1);
          ix = fminf(fmaxf(ix, 0.f), float(w - 1)); iy = fminf(fmaxf(iy, 0.f), float(h - 1));
          const float x0f = floorf(ix), y0f = floorf(iy);
          const int x0 = int(x0f), y0 = int(y0f);
          const int x1 = min(x0 + 1, w - 1), y1 = min(y0 + 1, h - 1);
          const float we = ix - x0f, ww = (x0f + 1.f) - ix, ws = iy - y0f, wn = (y0f + 1.f) - iy;
          const float* __restrict__ base = pp.rgb + size_t(v) * h * w * 4;
          const float4 t00 = ldg4(base + (size_t(y0) * w + x0) * 4), t01 = ldg4(base + (size_t(y0) * w + x1) * 4);
          const float4 t10 = ldg4(base + (size_t(y1) * w + x0) * 4), t11 = ldg4(base + (size_t(y1) * w + x1) * 4);
          const float w00 = ww * wn, w01 = we * wn, w10 = ww * ws, w11 = we * ws;
          rgbin[0] = t00.x * w00 + t01.x * w01 + t10.x * w10 + t11.x * w11;
          rgbin[1] = t00.y * w00 + t01.y * w01 + t10.y * w10 + t11.y * w11;
          rgbin[2] = t00.z * w00 + t01.z * w01 + t10.z * w10 + t11.z * w11;
        }
      }

      PM_TICK(1)
      // ---------------- bilinear gather of this warp's 32 rows, ray_feats (channels 0..31): 8 lanes x float4 per texel ----------------
      // The gathering quarter-warp and the row owner are different lanes: the row's coordinates come over by shuffle,
      // the channels go back through the warp-private transposition buffer.
      auto gather32 = [&](const int ch0) {
        const int qw = lane >> 3, l = lane & 7;
        __syncwarp();
#pragma unroll 1
        for (int rb = 0; rb < 32; rb += 4 * GB) {
          float4 t[GB][4];
          float wq[GB][4];
          bool on[GB];
#pragma unroll
          for (int u = 0; u < GB; ++u) {
            const int j = rb + 4 * u + qw;                                   // row (= lane) whose texels this quarter-warp fetches
            const int code = __shfl_sync(0xffffffffu, tcode, j);
#pragma unroll
            for (int k = 0; k < 4; ++k) wq[u][k] = __shfl_sync(0xffffffffu, tw[k], j);
            on[u] = code >= 0;
            if (on[u]) {
              const float* __restrict__ base = pp.feat + (code & ~63) + ch0 + 4 * l;
              const int dx = (code & 1) << 6, dy = (code & 2) ? fw * 64 : 0;
              t[u][0] = ldg4(base); t[u][1] = ldg4(base + dx);
              t[u][2] = ldg4(base + dy); t[u][3] = ldg4(base + dy + dx);
            }
          }
#pragma unroll
          for (int u = 0; u < GB; ++u) {
            const int j = rb + 4 * u + qw;
            float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
            if (on[u]) {
              o.x = t[u][0].x * wq[u][0] + t[u][1].x * wq[u][1] + t[u][2].x * wq[u][2] + t[u][3].x * wq[u][3];
              o.y = t[u][0].y * wq[u][0] + t[u][1].y * wq[u][1] + t[u][2].y * wq[u][2] + t[u][3].y * wq[u][3];
              o.z = t[u][0].z * wq[u][0] + t[u][1].z * wq[u][1] + t[u][2].z * wq[u][2] + t[u][3].z * wq[u][3];
              o.w = t[u][0].w * wq[u][0] + t[u][1].w * wq[u][1] + t[u][2].w * wq[u][2] + t[u][3].w * wq[u][3];
            }
            *reinterpret_cast<float4*>(stg + j * STG_ROW + 4 * l) = o;
          }
        }
        __syncwarp();
      };
      // The same gather split into "issue the loads of rows [rb, rb + 4 GB)" and "blend them and store": the img_feats half is
      // fetched underneath the dist decoder's first MMA round trips instead of in front of them (NR_GATHER_OVERLAP).
      float4 gt[GB][4];
      float gwq[GB][4];
      bool gon[GB];
      auto g_issue = [&](const int rb, const int ch0) {
        const int qw = lane >> 3, l = lane & 7;
#pragma unroll
        for (int u = 0; u < GB; ++u) {
          const int j = rb + 4 * u + qw;
          const int code = __shfl_sync(0xffffffffu, tcode, j);
#pragma unroll
          for (int k = 0; k < 4; ++k) gwq[u][k] = __shfl_sync(0xffffffffu, tw[k], j);
          gon[u] = code >= 0;
          if (gon[u]) {
            const float* __restrict__ base = pp.feat + (code & ~63) + ch0 + 4 * l;
            const int dx = (code & 1) << 6, dy = (code & 2) ? fw * 64 : 0;
            gt[u][0] = ldg4(base); gt[u][1] = ldg4(base + dx);
            gt[u][2] = ldg4(base + dy); gt[u][3] = ldg4(base + dy + dx);
          }
        }
      };
      auto g_consume = [&](const int rb) {
        const int qw = lane >> 3, l = lane & 7;
#pragma unroll
        for (int u = 0; u < GB; ++u) {
          const int j = rb + 4 * u + qw;
          float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
          if (gon[u]) {
            o.x = gt[u][0].x * gwq[u][0] + gt[u][1].x * gwq[u][1] + gt[u][2].x * gwq[u][2] + gt[u][3].x * gwq[u][3];
            o.y = gt[u][0].y * gwq[u][0] + gt[u][1].y * gwq[u][1] + gt[u][2].y * gwq[u][2] + gt[u][3].y * gwq[u][3];
            o.z = gt[u][0].z * gwq[u][0] + gt[u][1].z * gwq[u][1] + gt[u][2].z * gwq[u][2] + gt[u][3].z * gwq[u][3];
            o.w = gt[u][0].w * gwq[u][0] + gt[u][1].w * gwq[u][1] + gt[u][2].w * gwq[u][2] + gt[u][3].w * gwq[u][3];
          }
          *reinterpret_cast<float4*>(stg + j * STG_ROW + 4 * l) = o;
        }
      };
      constexpr int GSTEP = 4 * GB;                  // rows per issue/consume step; 32 / GSTEP steps per half
      static_assert(!NR_GATHER_OVERLAP || GB == 2, "the overlapped gather is written for four steps of eight rows");
      gather32(0);

      PM_TICK(2)
      // ---------------- dist decoder on the tensor cores: A[0:32] <- this row's ray_feats ----------------
      {
        float x[32];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 t4 = *reinterpret_cast<const float4*>(stg + lane * STG_ROW + 4 * q);
          x[4 * q] = t4.x; x[4 * q + 1] = t4.y; x[4 * q + 2] = t4.z; x[4 * q + 3] = t4.w;
        }
        st32(b, 0, 64, x);
        if (DEBUG && kp.dbg != nullptr && row_ok) {
          float* __restrict__ o = kp.dbg + (size_t(v) * N + n) * 76;
          for (int k = 0; k < 32; ++k) o[12 + k] = x[k];
        }
      }
#if NR_GATHER_OVERLAP
      __syncwarp();                                                                  // every lane has read its ray_feats row
      g_issue(0, 32);                                                                // img_feats, step 0: in flight under head 0
#else
      gather32(32);                                                                  // img_feats: stay in the buffer until ray_dir_fc
#endif
      PM_TICK(3)
      float hv[4][2] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}};
#pragma unroll 1
      for (int hd = 0; hd < n_heads; ++hd) {
        const float* __restrict__ hw_ = sw + SW_HEAD + hd * SW_HEAD_STRIDE;
#if NR_GATHER_OVERLAP
        issue_layer<32, 4, 0, 64, 4, 0, 128, 0, 1, 0, 1024 * 4, 0, true, false, false>(b);          // L0: A[0:32]
        if (hd < 2) { g_consume(2 * GSTEP * hd); g_issue(2 * GSTEP * hd + GSTEP, 32); }
#else
        run_layer<32, 4, 0, 4, 0, 0, 1024 * 4, 0, true, false>(b);              // L0: A[0:32]
#endif
        {
          float x[32];
          ld32(b, 128, x);
          add_bias32(x, hw_);
#pragma unroll
          for (int j = 0; j < 32; ++j) x[j] = elu(x[j]);
          st32(b, 32, 96, x);
        }
#if NR_GATHER_OVERLAP
        issue_layer<32, 4, 32, 64, 4, 0, 128, 0, 1, 2048 * 4, 3072 * 4, 0, false, true, false>(b);  // L1: A[32:64]
        if (hd < 2) {
          g_consume(2 * GSTEP * hd + GSTEP);
          if (hd == 0) g_issue(2 * GSTEP, 32);
          else __syncwarp();                                                         // img_feats complete in the buffer
        }
#else
        run_layer<32, 4, 32, 4, 0, 2048 * 4, 3072 * 4, 0, false, true>(b);      // L1: A[32:64]
#endif
        float o0 = hw_[128], o1 = hw_[129];
        {
          float x[32];
          ld32(b, 128, x);
          add_bias32(x, hw_ + 32);
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const float4 wa = *reinterpret_cast<const float4*>(hw_ + 64 + 4 * q);
            const float4 wb = *reinterpret_cast<const float4*>(hw_ + 96 + 4 * q);
            const float a0 = elu(x[4 * q]), a1 = elu(x[4 * q + 1]), a2 = elu(x[4 * q + 2]), a3 = elu(x[4 * q + 3]);
            o0 = fmaf(wa.w, a3, fmaf(wa.z, a2, fmaf(wa.y, a1, fmaf(wa.x, a0, o0))));
            o1 = fmaf(wb.w, a3, fmaf(wb.z, a2, fmaf(wb.y, a1, fmaf(wb.x, a0, o1))));
          }
        }
        if (hd == 0) { hv[0][0] = o0; hv[0][1] = o1; }
        else if (hd == 1) { hv[1][0] = o0; hv[1][1] = o1; }
        else if (hd == 2) { hv[2][0] = o0; hv[2][1] = o1; }
        else { hv[3][0] = o0; hv[3][1] = o1; }
      }
      PM_TICK(4)
      float hit = 0.f, visib = 0.f;
      {
        const float* vp = smem + OFF_CAM + 32 + (v < rfn ? v : 0) * 20;
        const float zc = fmaxf(zrow, 1e-5f);
        const float a = vp[15], bb = vp[16];
        const float tz = (-1.f / zc - a) / (bb - a);
        const float lo = tz - ihp, hi = tz + ihc;
        const float aw = sigmoidf_(hv[2][0]);
        const float vd = pp.use_vis ? sigmoidf_(hv[3][0]) : 1.f;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float mean = softplusf_(hv[0][i]);
          const float var = softplusf_(hv[1][i]) + pp.var_bias;
          const float c0 = logistic_cdf((lo - mean) * var) * vd, c1 = logistic_cdf((hi - mean) * var) * vd;
          const float mix = i == 0 ? aw : 1.f - aw;
          visib = fmaf(1.f - c0, mix, visib);
          hit = fmaf(c1 - c0, mix, hit);
        }
        visib *= mrow; hit *= mrow;
      }

      // ---------------- prob_embed (tensor cores), neuray_fc, ray_dir_fc ----------------
      {
        float x[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = 0.f;
        x[0] = (hit - 0.5f) * 2.f; x[1] = (visib - 0.5f) * 2.f;
        st8(b, 32, 96, x);                                                           // A[32:40] = hit', vis', 0... (the heads' hidden layer is dead)
      }
      run_layer<32, 5, 0, 4, 32, 0, 2048 * 4, 4096, true, true>(b);                 // prob_embed.0: K = 32 + 8
      {
        float x[32];
        ld32(b, 128, x);
        add_bias32(x, sw + SW_PE0B);
#pragma unroll
        for (int j = 0; j < 32; ++j) x[j] = fmaxf(x[j], 0.f);
        st32(b, 0, 64, x);                                                           // over ray_feats: their last reader has completed
      }
      PM_TICK(5)
      // prob_embed.2 with neuray_fc.0 behind it: N = 48, accumulator columns [96,144)
      issue_layer<48, 4, 0, 64, 4, 0, 96, 0, 1, 0, 1536 * 4, 0, true, true, false>(b);
      float gate;
      {
        float x[32];
        ld32(b, 96, x);
        add_bias32(x, sw + SW_PE1B);                                                 // neuray_feat
        st32(b, 0, 64, x);
        float h8[16];
        ld16(b, 128, h8);                                                            // neuray_fc.0 pre-activations (8 used)
        gate = sw[SW_NF1B];
#pragma unroll
        for (int j = 0; j < 8; ++j) gate = fmaf(sw[SW_NF1W + j], elu(h8[j] + sw[SW_NF0C + j]), gate);
      }
      // base_fc.0, K round A: the neuray_feat inputs (B chunks 5..8), accumulator columns [96,160)
      issue_layer<64, 4, 0, 64, 4, 0, 96, 5, 3, 0, 2048 * 4, 0, true, false, false>(b);
      float rf[40];                                                                  // rgb_feat (35) + zero padding
      {
        {
          float h16[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const float* __restrict__ w0 = sw + SW_RD0W;
            h16[j] = elu(fmaf(w0[48 + j], dd[3], fmaf(w0[32 + j], dd[2], fmaf(w0[16 + j], dd[1], fmaf(w0[j], dd[0], sw[SW_RD0B + j])))));
          }
          st16(b, 48, 64, h16);                                                      // ray_dir_fc.2 operand: hi [48,64), lo [64,80)
        }
        issue_layer_resident<48, 2, 48, 16, 0, 0, 1536 * 4, 0, false>(b, tc::smem_u32(smem + OFF_RD1));   // ray_dir_fc.2: K = 16, accumulator [0,48)
        ld32(b, 0, rf);
        {
          float t16[16];
          ld16(b, 32, t16);
#pragma unroll
          for (int j = 0; j < 8; ++j) rf[32 + j] = t16[j];
        }
#pragma unroll
        for (int j4 = 0; j4 < 36; j4 += 4) {
          const float4 bb = *reinterpret_cast<const float4*>(sw + SW_RD1B + j4);
          rf[j4] = elu(rf[j4] + bb.x); rf[j4 + 1] = elu(rf[j4 + 1] + bb.y); rf[j4 + 2] = elu(rf[j4 + 2] + bb.z); rf[j4 + 3] = elu(rf[j4 + 3] + bb.w);
        }
        // + [rgb | img_feats] of this row (img_feats come back from the transposition buffer)
        rf[0] += rgbin[0]; rf[1] += rgbin[1]; rf[2] += rgbin[2];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 t4 = *reinterpret_cast<const float4*>(stg + lane * STG_ROW + 4 * q);
          rf[3 + 4 * q] += t4.x; rf[4 + 4 * q] += t4.y; rf[5 + 4 * q] += t4.z; rf[6 + 4 * q] += t4.w;
          if (DEBUG && kp.dbg != nullptr && row_ok) {
            float* __restrict__ o = kp.dbg + (size_t(v) * N + n) * 76;
            o[44 + 4 * q] = t4.x; o[45 + 4 * q] = t4.y; o[46 + 4 * q] = t4.z; o[47 + 4 * q] = t4.w;
          }
        }
        rf[35] = 1.f;                                                                // constant input: base_fc.0's bias is column 35 of its tile
#pragma unroll
        for (int j = 36; j < 40; ++j) rf[j] = 0.f;
        st32(b, 0, 48, rf);                                                          // rgb_feat: hi [0,40), lo [48,88)
        st8(b, 32, 80, rf + 32);
      }
      // base_fc.0, K round B: rgb_feat (B chunks 0..4)
      issue_layer<64, 5, 0, 48, 5, 0, 96, 0, 3, 0, 2048 * 4, 0, false, true, true>(b);
      if (DEBUG && kp.dbg != nullptr && row_ok) {
        float* __restrict__ o = kp.dbg + (size_t(v) * N + n) * 76;
        o[0] = mrow; o[1] = zrow; o[2] = hit; o[3] = visib; o[4] = dbg_px; o[5] = dbg_py;
        o[6] = dbg_dir[0]; o[7] = dbg_dir[1]; o[8] = dbg_dir[2]; o[9] = rgbin[0]; o[10] = rgbin[1]; o[11] = rgbin[2];
      }

      PM_TICK(6)
      // ---------------- view pooling #1 (ibrnet.py:336-339) -> five more K rounds of base_fc.0 ----------------
      // Every lane of a point ends a round with the point's statistics, which is exactly its row of the view-invariant
      // operand: 8 features x (mean0, var0, mean1, var1) = K 32 per round go to A[0:32) and are multiplied into the same
      // accumulator, B from one ring stage per round.  The sums over the views go through the
      // warp's transposition buffer (pool_rows); the variance comes from the weighted second moment:
      //   sum_v w (x - mu)^2 = sum_v w x^2 - mu^2 (2 - sum_v w),  mu = sum_v w x   (the reference's mean is NOT normalised)
      const float msum = gsum(mrow);
      const float w1 = mrow / (msum + 1e-8f);
      const float w0 = sigmoidf_(gate) * w1;
      {
        const float c1 = 2.f - gsum(w1), c0 = 2.f - gsum(w0);
        auto round = [&](auto rc) {
          constexpr int R = decltype(rc)::value;
          float in[32], st[32];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float x = (8 * R + i < 35) ? rf[8 * R + i] : 0.f;
            const float p0 = x * w0, p1 = x * w1;
            in[i] = p0; in[8 + i] = p0 * x; in[16 + i] = p1; in[24 + i] = p1 * x;
          }
          gpool32(in, st);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            st[8 + i] = fmaf(-st[i] * st[i], c0, st[8 + i]);
            st[24 + i] = fmaf(-st[16 + i] * st[16 + i], c1, st[24 + i]);
          }
          st32(b, 0, 32, st);
          issue_layer<64, 4, 0, 32, 4, 0, 96, 0, 1, 0, 2048 * 4, 0, true, true, true>(b);
        };
        round(std::integral_constant<int, 0>{}); round(std::integral_constant<int, 1>{}); round(std::integral_constant<int, 2>{});
        round(std::integral_constant<int, 3>{}); round(std::integral_constant<int, 4>{});
      }

      PM_TICK(7)
      // ---------------- base_fc on the tensor cores ----------------
#pragma unroll
      for (int c0 = 0; c0 < 64; c0 += 32) {
        float x[32];
        ld32(b, 96 + c0, x);
#pragma unroll
        for (int j = 0; j < 32; ++j) x[j] = elu(x[j]);
        st32(b, c0, 64 + c0, x);                                                     // lo half 1 lands on accumulator columns already consumed
      }
      PM_TICK(8)
      run_layer<32, 8, 0, 8, 0, 0, 2048 * 4, 4096, true, true>(b);                  // base_fc.2: K = 64
      float xr[32];
      ld32(b, 128, xr);
      add_bias32(xr, sw + SW_B1B);
#pragma unroll
      for (int j = 0; j < 32; ++j) xr[j] = elu(xr[j]);
      st32(b, 0, 64, xr);

      PM_TICK(9)
      // ---------------- vis_fc, vis_fc2, rgb_fc ----------------
      if constexpr (DEBUG) {
        if (kp.timing != nullptr && blockIdx.x == 0 && b.leader && b.blk < 2 && it < 64) b.tk = kp.timing + (it * 2 + b.blk) * 32 + 16;
      }
      run_layer<32, 4, 0, 4, 0, 0, 1024 * 4, 0, true, false>(b);                     // vis_fc.0 (row scale folded into the epilogue)
      float lg = sw[SW_V1LB];
      {
        float x[32];
        ld32(b, 128, x);
        if (b.tk) b.tk[7] = clock64();
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 bb = *reinterpret_cast<const float4*>(sw + SW_V0B + 4 * q);
          const float4 wl = *reinterpret_cast<const float4*>(sw + SW_V1LW + 4 * q);
          x[4 * q] = elu(fmaf(w1, x[4 * q], bb.x)); x[4 * q + 1] = elu(fmaf(w1, x[4 * q + 1], bb.y));
          x[4 * q + 2] = elu(fmaf(w1, x[4 * q + 2], bb.z)); x[4 * q + 3] = elu(fmaf(w1, x[4 * q + 3], bb.w));
          lg = fmaf(wl.w, x[4 * q + 3], fmaf(wl.z, x[4 * q + 2], fmaf(wl.y, x[4 * q + 1], fmaf(wl.x, x[4 * q], lg))));
        }
        if (b.tk) b.tk[8] = clock64();
        st32(b, 32, 96, x);
        if (b.tk) { b.tk[9] = clock64(); b.tk = nullptr; }
      }
      PM_TICK(10)
      const float visa = sigmoidf_(elu(lg)) * mrow;
      run_layer<32, 4, 32, 4, 0, 2048 * 4, 3072 * 4, 0, false, true>(b);             // vis_fc.2 outputs 0..31 (residual)
      {
        float x[32];
        ld32(b, 128, x);
        add_bias32(x, sw + SW_V1B);
#pragma unroll
        for (int j = 0; j < 32; ++j) xr[j] += elu(x[j]);
        st32(b, 0, 64, xr);
      }
      PM_TICK(11)
      run_layer<32, 4, 0, 4, 0, 0, 1024 * 4, 0, true, false>(b);                     // vis_fc2.0
      float vis2;
      {
        float l2 = sw[SW_V21B];
        float x[32];
        ld32(b, 128, x);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 bb = *reinterpret_cast<const float4*>(sw + SW_V20B + 4 * q);
          const float4 wl = *reinterpret_cast<const float4*>(sw + SW_V21W + 4 * q);
          l2 = fmaf(wl.x, elu(fmaf(visa, x[4 * q], bb.x)), l2); l2 = fmaf(wl.y, elu(fmaf(visa, x[4 * q + 1], bb.y)), l2);
          l2 = fmaf(wl.z, elu(fmaf(visa, x[4 * q + 2], bb.z)), l2); l2 = fmaf(wl.w, elu(fmaf(visa, x[4 * q + 3], bb.w)), l2);
        }
        vis2 = sigmoidf_(l2) * mrow;
        float y[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) y[j] = 0.f;
        y[0] = vis2; y[1] = dd[0]; y[2] = dd[1]; y[3] = dd[2]; y[4] = dd[3];
        st8(b, 32, 96, y);                                                           // A[32:40] = vis, ray_diff, 0
      }
      PM_TICK(12)
      run_layer<16, 5, 0, 4, 32, 2048 * 4, 3072 * 4, 2048, false, true>(b);          // rgb_fc.0: K = 32 + 8, N = 16
      float logit;
      {
        float x[16];
        ld16(b, 128, x);
        float h8[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) h8[j] = sw[SW_RGB1B + j];
#pragma unroll
        for (int k = 0; k < 16; ++k) {
          const float a = elu(x[k] + sw[SW_RGB0B + k]);
          const float4 wa = *reinterpret_cast<const float4*>(sw + SW_RGB1W + k * 8);
          const float4 wb = *reinterpret_cast<const float4*>(sw + SW_RGB1W + k * 8 + 4);
          h8[0] = fmaf(wa.x, a, h8[0]); h8[1] = fmaf(wa.y, a, h8[1]); h8[2] = fmaf(wa.z, a, h8[2]); h8[3] = fmaf(wa.w, a, h8[3]);
          h8[4] = fmaf(wb.x, a, h8[4]); h8[5] = fmaf(wb.y, a, h8[5]); h8[6] = fmaf(wb.z, a, h8[6]); h8[7] = fmaf(wb.w, a, h8[7]);
        }
        float l3 = sw[SW_RGB2B];
#pragma unroll
        for (int j = 0; j < 8; ++j) l3 = fmaf(sw[SW_RGB2W + j], elu(h8[j]), l3);
        // masked views get -1e9 like the reference; padding lanes must not take part at all
        logit = v >= rfn ? -3.0e38f : (mrow == 0.f ? -1e9f : l3);
      }

      PM_TICK(13)
      // ---------------- softmax colour blend over the views (ibrnet.py:365-367) ----------------
      float rgbo[3];
      {
        const float mx = gmax(logit);
        const float e = v >= rfn ? 0.f : expf(logit - mx);
        float acc[4] = {e, e * rgbin[0], e * rgbin[1], e * rgbin[2]};
        if constexpr (P2) bsum_vec<G, 4>(acc); else gsum4_np2<G>(stg, lane, lane0, idle, acc);
#pragma unroll
        for (int cc = 0; cc < 3; ++cc) rgbo[cc] = acc[1 + cc] / acc[0];
      }

      PM_TICK(14)
      // ---------------- view pooling #2 (ibrnet.py:352-353) -> geometry_fc.0 on the tensor cores, geometry_fc.2 across the lanes ----------------
      {
        const float vs = gsum(vis2);
        const float w2 = vis2 / (vs + 1e-8f);
        const float sw2 = gsum(w2);
        const float wmean = sw2 / float(rfn);
        // two K rounds of 16 features x (mean, var) and a third with the mean weight and the constant that multiplies the
        // bias column, one ring stage each; sums over the views through pool_rows, variance from the second moment (above)
        const float c2 = 2.f - sw2;
        auto ground = [&](auto rc) {
          constexpr int R = decltype(rc)::value;
          float in[32], st[32];
#pragma unroll
          for (int i = 0; i < 16; ++i) { const float p = xr[16 * R + i] * w2; in[i] = p; in[16 + i] = p * xr[16 * R + i]; }
          gpool32(in, st);
#pragma unroll
          for (int i = 0; i < 16; ++i) st[16 + i] = fmaf(-st[i] * st[i], c2, st[16 + i]);
          st32(b, 0, 32, st);
          issue_layer<64, 4, 0, 32, 4, 0, 96, 0, 1, 0, 2048 * 4, 0, true, true, (R > 0)>(b);
        };
        ground(std::integral_constant<int, 0>{}); ground(std::integral_constant<int, 1>{});
        {
          float st[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) st[i] = 0.f;
          st[0] = wmean; st[1] = 1.f;
          st8(b, 0, 32, st);
          issue_layer<64, 1, 0, 32, 1, 0, 96, 0, 1, 0, 2048 * 4, 0, true, true, true>(b);
        }
        // all G rows of a point hold the same 64 hidden pre-activations; lane v keeps columns [v*CPL, (v+1)*CPL)
        float hh[CPL];
        {
          float d[64];
          ld32(b, 96, d);
          ld32(b, 128, d + 32);
          // GE = the lanes of the point that take part (all G of a power-of-two group, else the first 8 / 4)
#pragma unroll
          for (int m = GE >> 1, len = 32; m >= 1; m >>= 1, len >>= 1) {
#pragma unroll
            for (int k = 0; k < len; ++k) d[k] = (v & m) ? d[len + k] : d[k];
          }
#pragma unroll
          for (int j = 0; j < CPL; ++j) hh[j] = (P2 || v < GE) ? elu(d[j]) : 0.f;
        }
        float out[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) out[k] = 0.f;
#pragma unroll
        for (int k = 0; k < 16; ++k) {                                               // sWg1 is stored output-major: [16][64]
          float wk[CPL];
          ld_cols<GE>(sWg1 + k * 64, (P2 || v < GE) ? v : 0, wk);
#pragma unroll
          for (int j = 0; j < CPL; ++j) out[k] = fmaf(wk[j], hh[j], out[k]);
        }
        {
          float sum[16];
          if constexpr (P2) pool_rows<G, 16>(stg, lane, lane0, v, out, sum); else pool_rows_np2<G, 16>(stg, lane, lane0, v, idle, out, sum);
#pragma unroll
          for (int k = 0; k < 16; ++k) out[k] = elu(sum[k] + sWg1[64 * 16 + k]);
        }
        if (v == 0 && pt_ok) {
          float4* __restrict__ dst = reinterpret_cast<float4*>(pp.point_rec + size_t(n) * REC);
          dst[0] = make_float4(out[0], out[1], out[2], out[3]); dst[1] = make_float4(out[4], out[5], out[6], out[7]);
          dst[2] = make_float4(out[8], out[9], out[10], out[11]); dst[3] = make_float4(out[12], out[13], out[14], out[15]);
          dst[4] = make_float4(rgbo[0], rgbo[1], rgbo[2], msum);
        }
      }
      PM_TICK(15)
    }
  }

}

}  // namespace pm3
