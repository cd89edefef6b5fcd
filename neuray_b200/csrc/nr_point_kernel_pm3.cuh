// Point kernel (namespace nr::pkt::pm3): point-major rows, wgmma layers, one 128-row block per SM.
//
// Row = point * G + view inside a block (G lanes per point: 4, 5, 6, 8, 10, 16 or 32).  Two compute warp groups work on
// the same rows: thread r of either one is row r of the activation tile, and each warp group keeps half of the row's
// columns in registers from the gather to the output record.  Resource plan (one CTA per SM: 2 x 128 compute threads at
// 240 registers + a 128-thread producer group at 24 registers whose lane 0 feeds the weight ring):
//   * column ownership (own_index): every operand and every output of a layer starts on a multiple of 8 columns, and in
//     every 8-column group warp group c owns columns [4c, 4c + 4).  A warp group writes the hi/lo parts of its columns,
//     reads its accumulator columns and runs their epilogue; its registers hold its 16 of 32 (20 of 40) values.  The
//     view-pooled statistics keep this split, because both pooled operands put one feature's statistics 8 or 16 columns
//     apart.  rgb_fc.1/.2 and the colour blend run in warp group 1 only, geometry_fc.2 in warp group 0 only, each from the
//     whole row in the tile.
//   * MMAs: warp group c issues the m64 wgmma of rows 64c .. 64c + 63 of every layer; both warp groups meet at a
//     256-thread barrier before a layer (its A columns come from both) and after the accumulator store.  The dist-decoder
//     heads (run_head) and the per-view tail base_fc.2 .. rgb_fc.0 (run_chain) are the exception: nothing in them is
//     pooled or needs the row-owner layout, so each warp group runs them for its own 64 rows in the accumulator fragment
//     (A from registers after the first layer, row sums over the 4 lanes that hold a row) and hands the results to the
//     row owners through the tile and a small shared array (xch).  The ring's "empty" barriers count one arrival per
//     compute warp group, so each releases those stages on its own.
//   * activation tile (80 KB of shared memory, 160 columns x 128 rows, tc::act_index): hi parts at columns [0,64), lo parts
//     at [64,128), accumulator at [128,160).  base_fc.0 (N = 64) has its per-view inputs issued in two K rounds into one
//     accumulator at [96,160): round A (the 32 neuray_feat inputs) right after prob_embed.2 while they are still the only
//     live A operand, round B (the 40 rgb_feat inputs, lo parts at [48,88)) after ray_dir_fc.  Its epilogue reads the
//     accumulator half by half, adds the point's view-pooled part and writes base_fc.2's operand over the columns it has
//     already consumed (the same warp group owns column c and c + 32, so no other warp group reads them).  run_chain
//     leaves x2 at [96,128) and rgb_fc.0's pre-activations at [128,144).
//   * per-point layers: the view-pooled part of base_fc.0 (K 140 -> 160) and geometry_fc.0 have the same inputs for every
//     view of a point, so they are multiplied once per point, not once per row: the pooled statistics go into a compact
//     operand of PB rows (one per point, in tile columns [0,96) while those are dead), the eight compute warps multiply
//     it with warp-level mma.sync (3xTF32, B read straight from the weight ring stages, warp w computes outputs
//     8w .. 8w + 7) into a [PB][64] result in shared memory (OFF_PT), and every row of the point reads it from there.
//   * the rest of shared memory: 4 x 16 KB weight ring (TMA bulk copies, fed by the producer group; the view-pooled
//     base_fc.0 weights stream through it as five more stages), the resident tile of ray_dir_fc.2, small weights, camera
//     blocks, the row-scalar exchange, the per-point result, and one [32][36] transposition buffer per warp: gather (16
//     channels per warp group in two passes: ray_feats, then img_feats, which stay there until ray_dir_fc needs them), the
//     cross-view pooling (pm::pool_rows) and the lane-group sums of the non-power-of-two groups all go through it.
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
#define NR_GATHER_BATCH 2
#endif
constexpr int GB = NR_GATHER_BATCH;                           // rows whose 4 taps an eighth of a warp keeps in flight at once (4 x GB 128-bit loads per lane)
constexpr int NCOMP = 256;                                    // two compute warp groups
constexpr int NTHR = NCOMP + 128;                             // + a producer warp group whose lane 0 does nothing but keep the weight ring full
// __launch_bounds__(NTHR, 1) starts every thread at 168 registers; the producer group gives all but REG_PROD back and the
// compute groups take them: 128 x 24 + 256 x 240 = 64512 of the SM's 65536
constexpr int REG_PROD = 24, REG_COMP = 240;
static_assert(128 * REG_PROD + NCOMP * REG_COMP <= 65536, "register file");
constexpr int BAR_LAYER = 1;                                  // named barrier of the compute warp groups: around every layer
constexpr int TCOLS = 160;                                    // activation-tile columns
constexpr int ACT = (TCOLS / 32) * 4096;                      // floats per activation tile

// ---- shared memory map (floats) ----
constexpr int OFF_RING = 0;                                   // NBUF x RING_STAGE
constexpr int OFF_ACT = OFF_RING + NBUF * RING_STAGE;         // activation tile (1024-byte aligned)
constexpr int OFF_RD1 = OFF_ACT + ACT;                        // ray_dir_fc.2 tensor-core tile (resident, 1024-byte aligned)
constexpr int OFF_WG1 = OFF_RD1 + tcl::RD1_SIZE;              // geometry_fc.2: [16][64] (output-major, columns in own_col order) | bias[16]
constexpr int WG1 = 64 * 16 + 16;
constexpr int OFF_SW = OFF_WG1 + WG1;                         // small resident weights (offsets SW_*, nr_point_kernel.cu)
constexpr int OFF_STG = OFF_SW + SW;                          // gather transposition: per warp [32 rows][36]
constexpr int STG_ROW = 36;
constexpr int STG = (NCOMP / 32) * 32 * STG_ROW;
constexpr int OFF_XCH = OFF_STG + STG;                        // row scalars handed between the warp groups: [slot][128 rows], slots XCH_*
// (o0, o1) of the 4 heads; once the heads' outputs are read, the chain's row scalars w1, mrow, dd[0..3] | vis_fc2 visibility
constexpr int XCH_HEAD = 0, XCH_ROW = 0, XCH_L2 = 8, XCH = 9 * 128;
constexpr int OFF_PT = OFF_XCH + XCH;                         // per-point layer outputs: [point][PT_ROW] (64 used), at most 32 points
constexpr int PT_ROW = 72;
constexpr int PT = 32 * PT_ROW;
constexpr int OFF_CAM = OFF_PT + PT;                          // que_cam [24] (padded to 32) | view_params [NR_MAX_VIEWS][20]
constexpr int CAM = 32 + NR_MAX_VIEWS * 20;
constexpr int OFF_STAB = OFF_CAM + CAM;                       // stage_source: int4 per stage of a tile (at most 4 + 16)
constexpr int OFF_BAR = OFF_STAB + 80;
constexpr int SMEM_FLOATS = OFF_BAR + 32;
constexpr size_t SMEM_BYTES = size_t(SMEM_FLOATS) * 4;
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");
static_assert(OFF_STAB % 4 == 0, "alignment");
static_assert((OFF_ACT * 4) % 1024 == 0 && (OFF_RD1 * 4) % 1024 == 0 && OFF_WG1 % 4 == 0 && OFF_SW % 4 == 0 && OFF_STG % 4 == 0 &&
                  OFF_PT % 4 == 0, "alignment");
// the per-point operand of a per-point layer: [point][OP_ROW] (K 160 used) in activation-tile columns [0,96), which are
// dead while it is used (after base_fc.0's round B until its epilogue; after rgb_fc.0 until the next tile's gather)
constexpr int OP_ROW = 164;                                   // = 4 mod 32: the 32 lanes of an A-fragment load hit 32 banks
static_assert(32 * OP_ROW <= 3 * 4096, "per-point operand");

// ---- per-point layers: [points x K] x [K x 64] on warp-level mma.sync, 3xTF32 ----
// Compute warp w (of 8) computes outputs 8w .. 8w + 7 for all PB points of the tile: MT m16 tiles of points, and one
// accumulator per 3xTF32 pass (hi*hi, lo*hi, hi*lo) so that the three MMAs of a K step do not wait for each other.
template <int PB>
struct PtAcc {
  static constexpr int MT = (PB + 15) / 16;
  float d[MT][3][4];
};
// acc += op[points][kcol + k] * W[8w + n][k], k < 8 KS: B from a weight ring stage `w` (64 rows x K32, K-major 128-byte
// swizzle, hi slab | lo slab 2048 floats further, K steps 0 .. KS - 1).  Operand rows at or past PB read as 0.
template <int PB, int KS>
__device__ __forceinline__ void point_mma(PtAcc<PB>& acc, const float* __restrict__ op, int kcol, const float* __restrict__ w, int warp, int lane) {
  const int g = lane >> 2, t = lane & 3;
  const float* __restrict__ bw = w + warp * 256 + g * 32 + t;             // tc::sw128_index(8 warp + g, 8 j + t) = bw[((2j) ^ g) << 2]
  const float* __restrict__ aw = op + g * OP_ROW + kcol + t;
#pragma unroll
  for (int j = 0; j < KS; ++j) {
    const uint32_t bh[2] = {__float_as_uint(bw[((2 * j) ^ g) << 2]), __float_as_uint(bw[((2 * j + 1) ^ g) << 2])};
    const uint32_t bl[2] = {__float_as_uint(bw[2048 + (((2 * j) ^ g) << 2)]), __float_as_uint(bw[2048 + (((2 * j + 1) ^ g) << 2)])};
#pragma unroll
    for (int m = 0; m < PtAcc<PB>::MT; ++m) {
      const bool ok0 = 16 * m + 8 <= PB || 16 * m + g < PB, ok1 = 16 * m + 16 <= PB || 16 * m + 8 + g < PB;
      const float* __restrict__ a = aw + 16 * m * OP_ROW + 8 * j;
      const float x[4] = {ok0 ? a[0] : 0.f, ok1 ? a[8 * OP_ROW] : 0.f, ok0 ? a[4] : 0.f, ok1 ? a[8 * OP_ROW + 4] : 0.f};
      uint32_t ah[4], al[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) tc::split_tf32(x[i], ah[i], al[i]);
      tc::mma_tf32_m16n8k8(acc.d[m][0], ah, bh);
      tc::mma_tf32_m16n8k8(acc.d[m][1], al, bh);
      tc::mma_tf32_m16n8k8(acc.d[m][2], ah, bl);
    }
  }
}
// the accumulated outputs -> pt[point][8w .. 8w + 7] (points < PB)
template <int PB>
__device__ __forceinline__ void point_store(const PtAcc<PB>& acc, float* __restrict__ pt, int warp, int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int m = 0; m < PtAcc<PB>::MT; ++m) {
    float o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = acc.d[m][0][i] + (acc.d[m][1][i] + acc.d[m][2][i]);
    float* __restrict__ p = pt + (16 * m + g) * PT_ROW + 8 * warp + 2 * t;
    if (16 * m + 8 <= PB || 16 * m + g < PB) *reinterpret_cast<float2*>(p) = make_float2(o[0], o[1]);
    if (16 * m + 16 <= PB || 16 * m + 8 + g < PB) *reinterpret_cast<float2*>(p + 8 * PT_ROW) = make_float2(o[2], o[3]);
  }
}

// Layer issue, executed by both compute warp groups after they wrote their A columns; warp group c multiplies rows
// 64c .. 64c + 63.  K chunk c (of NCH) reads A columns AHI + 8c (c < NLIN) or TAILHI + 8(c - NLIN), lo parts LOOFF
// columns further, and B chunk CB0 + c of the layer's tiles (slab (CB0+c)/4; one ring stage per slab when NSTG > 1); ACC:
// the first MMA accumulates onto what is already in the accumulator columns [DCOL, DCOL + N).  Returns with the outputs in
// the activation tile, visible to every row owner of both warp groups.
template <int N, int NCH, int AHI, int LOOFF, int NLIN, int TAILHI, int DCOL, int CB0, int NSTG, uint32_t OFF_HI, uint32_t OFF_LO,
          uint32_t SLAB, bool WAIT_FULL, bool RELEASE, bool ACC>
__device__ __forceinline__ void issue_layer(Blk& b) {
  tc::fence_proxy_async_smem();              // this thread's A columns -> visible to the tensor cores
  tc::named_sync(BAR_LAYER, NCOMP);
  const uint32_t st0 = b.wi % NBUF;
  if (WAIT_FULL) {
#pragma unroll
    for (int s = 0; s < NSTG; ++s) tc::mbar_wait(b.wfull + ((st0 + s) % NBUF), ((b.wi + s) / NBUF) & 1);
  }
  float d[N / 2];
  if (ACC) tc::acc_load_half<N>(b.act, DCOL, b.row, b.wg, d);
  else {
#pragma unroll
    for (int j = 0; j < N / 2; ++j) d[j] = 0.f;
  }
  uint64_t dhi[NSTG], dlo[NSTG];
#pragma unroll
  for (int s = 0; s < NSTG; ++s) {
    const uint32_t base = b.ring_addr + ((st0 + s) % NBUF) * (RING_STAGE * 4);
    dhi[s] = tc::smem_desc_sw128(base + OFF_HI);
    dlo[s] = tc::smem_desc_sw128(base + OFF_LO);
  }
  tc::wgmma_fence_operand(d);
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
      tc::wgmma_tf32<N>(d, tc::act_desc(b.act_addr, acol, b.wg), bd);
    }
  }
  tc::wgmma_commit();
  tc::wgmma_wait_all();
  tc::wgmma_fence_operand(d);
  tc::acc_store_half<N>(b.act, DCOL, b.row, b.wg, d);
  tc::named_sync(BAR_LAYER, NCOMP);          // outputs in the tile; both warp groups' reads of the stages have completed
  if (RELEASE) {
    if (b.leader) {
#pragma unroll
      for (int s = 0; s < NSTG; ++s) tc::mbar_arrive(b.wempty + ((st0 + s) % NBUF));
    }
    b.wi += NSTG;
  }
}
// Same, B operand = a resident shared-memory tile at byte address `base` (hi slabs first, SLAB bytes apart; lo parts
// OFF_LO bytes further): no ring accounting.
template <int N, int NCH, int AHI, int LOOFF, int DCOL, int CB0, uint32_t OFF_LO, uint32_t SLAB, bool ACC>
__device__ __forceinline__ void issue_layer_resident(Blk& b, uint32_t base) {
  tc::fence_proxy_async_smem();
  tc::named_sync(BAR_LAYER, NCOMP);
  float d[N / 2];
  if (ACC) tc::acc_load_half<N>(b.act, DCOL, b.row, b.wg, d);
  else {
#pragma unroll
    for (int j = 0; j < N / 2; ++j) d[j] = 0.f;
  }
  const uint64_t dhi = tc::smem_desc_sw128(base), dlo = tc::smem_desc_sw128(base + OFF_LO);
  tc::wgmma_fence_operand(d);
  tc::wgmma_fence();
#pragma unroll
  for (int ps = 0; ps < 3; ++ps) {
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int acol = AHI + 8 * c + (ps == 1 ? LOOFF : 0);
      const int cb = CB0 + c;
      const uint32_t inc = ((cb >> 2) * SLAB + (cb & 3) * 32) >> 4;
      const uint64_t bd = (ps == 2 ? dlo : dhi) + inc;
      tc::wgmma_tf32<N>(d, tc::act_desc(b.act_addr, acol, b.wg), bd);
    }
  }
  tc::wgmma_commit();
  tc::wgmma_wait_all();
  tc::wgmma_fence_operand(d);
  tc::acc_store_half<N>(b.act, DCOL, b.row, b.wg, d);
  tc::named_sync(BAR_LAYER, NCOMP);
}
// the common case: activations hi [0,64) / lo [64,128), accumulator at 128, one ring stage
template <int N, int NCH, int AHI, int NLIN, int TAILHI, uint32_t OFF_HI, uint32_t OFF_LO, uint32_t SLAB, bool WAIT_FULL, bool RELEASE>
__device__ __forceinline__ void run_layer(Blk& b) {
  issue_layer<N, NCH, AHI, 64, NLIN, TAILHI, 128, 0, 1, OFF_HI, OFF_LO, SLAB, WAIT_FULL, RELEASE, false>(b);
}

// ---- layers in the accumulator fragment of the warp group that issues them (the heads and the per-view chain) ----
// This thread holds columns 8j + 2q + {0, 1} of fragment rows fr and fr + 8 (q = t % 4, tc::acc_load_half):
// d[4j + 2r + e] is column 8j + 2q + e of row fr + 8r.  B of K step c sits at descriptor + (c >> 2) SLAB16 + 2 (c & 3)
// of the hi (passes 0, 1) or lo (pass 2) descriptor; the passes and K steps go in issue_layer's order, so the
// accumulators get the same products in the same order as a round trip through the tile.
// d = A x B, A = tile columns [0, 8 KS) (hi) / [64, 64 + 8 KS) (lo) of this warp group's 64 rows.  Committed, not waited for.
template <int KS, int SLAB16>
__device__ __forceinline__ void issue_frag_ss(const Blk& b, float (&d)[16], uint64_t dhi, uint64_t dlo) {
#pragma unroll
  for (int j = 0; j < 16; ++j) d[j] = 0.f;
  tc::wgmma_fence_operand(d);
  tc::wgmma_fence();
#pragma unroll
  for (int ps = 0; ps < 3; ++ps) {
#pragma unroll
    for (int c = 0; c < KS; ++c)
      tc::wgmma_tf32<32>(d, tc::act_desc(b.act_addr, 8 * c + (ps == 1 ? 64 : 0), b.wg), (ps == 2 ? dlo : dhi) + (c >> 2) * SLAB16 + 2 * (c & 3));
  }
  tc::wgmma_commit();
}
// d = A x B, A from registers: K step c from ah[c] / al[c] (c < KS <= KA).  Committed, not waited for: the A registers and
// d stay pinned until wait_frag.
template <int N, int KS, int SLAB16, int KA>
__device__ __forceinline__ void issue_frag_ra(float (&d)[N / 2], uint32_t (&ah)[KA][4], uint32_t (&al)[KA][4], uint64_t dhi, uint64_t dlo) {
#pragma unroll
  for (int j = 0; j < N / 2; ++j) d[j] = 0.f;
  tc::wgmma_fence_operand(d);
#pragma unroll
  for (int c = 0; c < KS; ++c)
#pragma unroll
    for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(ah[c][i]), "+r"(al[c][i])::"memory");
  tc::wgmma_fence();
#pragma unroll
  for (int ps = 0; ps < 3; ++ps) {
#pragma unroll
    for (int c = 0; c < KS; ++c) tc::wgmma_tf32_ra<N>(d, ps == 1 ? al[c] : ah[c], (ps == 2 ? dlo : dhi) + (c >> 2) * SLAB16 + 2 * (c & 3));
  }
  tc::wgmma_commit();
}
template <int N, int KS, int KA>
__device__ __forceinline__ void wait_frag_ra(float (&d)[N / 2], uint32_t (&ah)[KA][4], uint32_t (&al)[KA][4]) {
  tc::wgmma_wait_all();
  tc::wgmma_fence_operand(d);
#pragma unroll
  for (int c = 0; c < KS; ++c)
#pragma unroll
    for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(ah[c][i]), "+r"(al[c][i])::"memory");
}
__device__ __forceinline__ void wait_frag(float (&d)[16]) {
  tc::wgmma_wait_all();
  tc::wgmma_fence_operand(d);
}
// An N = 32 fragment x (after its epilogue) -> the A fragments of the next layer's 4 K steps, split into hi / lo
// (ah[j], al[j], j < 4).  A K step wants columns 8j + q and 8j + q + 4 of rows fr, fr + 8 (tc::wgmma_tf32_ra): lane q of
// a quad reads lane s = 2 (q & 1) + (q >> 1) in the first shuffle and lane s ^ 2 in the second; a lane offers column
// 2q + (q >> 1) in the first and its other column in the second, and what arrives is column q and q + 4 (in that order
// for even q, swapped for odd q).
template <int KA>
__device__ __forceinline__ void frag_to_a(const float (&x)[16], int lane, uint32_t (&ah)[KA][4], uint32_t (&al)[KA][4]) {
  const int q = lane & 3, s1 = (lane & ~3) | ((q & 1) << 1) | (q >> 1);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float x0 = x[4 * j + 2 * r], x1 = x[4 * j + 2 * r + 1];
      const float r1 = __shfl_sync(0xffffffffu, q >> 1 ? x1 : x0, s1);
      const float r2 = __shfl_sync(0xffffffffu, q >> 1 ? x0 : x1, s1 ^ 2);
      tc::split_tf32(q & 1 ? r2 : r1, ah[j][r], al[j][r]);              // column 8j + q of row fr + 8r
      tc::split_tf32(q & 1 ? r1 : r2, ah[j][2 + r], al[j][2 + r]);      // column 8j + q + 4
    }
  }
}
// s[r] = bias + sum_c w[c] z(row fr + 8r, column c) over the 32 columns of an N = 32 fragment z, one fmaf per column in
// column order (the order the training recompute and a single row owner use), in every lane of the quad: column
// 8j + 2q' + e comes over from lane q' of the quad
__device__ __forceinline__ void row_dot(const float (&z)[16], const float* __restrict__ w, float bias, int lane, float (&s)[2]) {
  s[0] = s[1] = bias;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
#pragma unroll
    for (int qs = 0; qs < 4; ++qs) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
#pragma unroll
        for (int r = 0; r < 2; ++r) s[r] = fmaf(w[8 * j + 2 * qs + e], __shfl_sync(0xffffffffu, z[4 * j + 2 * r + e], (lane & ~3) | qs), s[r]);
      }
    }
  }
}

// One dist-decoder head (two K 32, N 32 layers and the (o0, o1) outputs) for the 64 rows whose MMAs this warp group
// issues, without leaving its registers and without meeting the other warp group: L0 reads A[0:32] from the tile (both
// warp groups wrote it before the barrier in front of the heads), its epilogue runs on the accumulator fragment, L1 takes
// A from registers, and the outputs go to xch slots XCH_HEAD + 2 hd + {0, 1}.  Releases the head's ring stage on its own
// (wempty counts one arrival per compute warp group).
__device__ __forceinline__ void run_head(Blk& b, const float* __restrict__ hw, float* __restrict__ xo, int fr) {
  const int lane = b.row & 31, q = lane & 3;
  const uint32_t st = b.wi % NBUF;
  tc::mbar_wait(b.wfull + st, (b.wi / NBUF) & 1);
  const uint32_t base = b.ring_addr + st * (RING_STAGE * 4);
  // L0: B hi / lo at stage floats 0 / 1024
  float d[16];
  issue_frag_ss<4, 0>(b, d, tc::smem_desc_sw128(base), tc::smem_desc_sw128(base + 1024 * 4));
  wait_frag(d);
  // bias + ELU, then into L1's A layout
  uint32_t ah[4][4], al[4][4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 bb = *reinterpret_cast<const float2*>(hw + 8 * j + 2 * q);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      d[4 * j + 2 * r] = elu(d[4 * j + 2 * r] + bb.x);
      d[4 * j + 2 * r + 1] = elu(d[4 * j + 2 * r + 1] + bb.y);
    }
  }
  frag_to_a(d, lane, ah, al);
  // L1: B hi / lo at stage floats 2048 / 3072
  float e[16];
  issue_frag_ra<32, 4, 0>(e, ah, al, tc::smem_desc_sw128(base + 2048 * 4), tc::smem_desc_sw128(base + 3072 * 4));
  wait_frag_ra<32, 4>(e, ah, al);
  if (b.leader) tc::mbar_arrive(b.wempty + st);
  b.wi += 1;
  // (o0, o1) of rows fr, fr + 8: this thread's 8 columns, then the quad's sum; lane q stores output q & 1 of row fr + 8 (q >> 1)
  float p[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = 8 * j + 2 * q;
    const float2 bb = *reinterpret_cast<const float2*>(hw + 32 + c);
    const float2 wa = *reinterpret_cast<const float2*>(hw + 64 + c), wb = *reinterpret_cast<const float2*>(hw + 96 + c);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float h0 = elu(e[4 * j + 2 * r] + bb.x), h1 = elu(e[4 * j + 2 * r + 1] + bb.y);
      p[2 * r] = fmaf(wa.y, h1, fmaf(wa.x, h0, p[2 * r]));
      p[2 * r + 1] = fmaf(wb.y, h1, fmaf(wb.x, h0, p[2 * r + 1]));
    }
  }
#pragma unroll
  for (int o = 1; o < 4; o <<= 1) {
#pragma unroll
    for (int i = 0; i < 4; ++i) p[i] += __shfl_xor_sync(0xffffffffu, p[i], o);
  }
  const float mine = q == 0 ? p[0] : q == 1 ? p[1] : q == 2 ? p[2] : p[3];
  xo[(q & 1) * 128 + fr + 8 * (q >> 1)] = mine + hw[128 + (q & 1)];
}

// The per-view tail base_fc.2 -> vis_fc.0 -> vis_fc.2 -> vis_fc2.0 -> rgb_fc.0 for the 64 rows whose MMAs this warp
// group issues, in its accumulator fragment and without meeting the other warp group: nothing in it pools across views.
// base_fc.2 reads its A (K 64) from the tile, where both warp groups' row owners wrote it before the barrier in front of
// the chain, together with the row scalars w1, mrow and dd[0..3] in xch slots XCH_ROW + [0,6); every later layer takes
// A from registers.  vis_fc.1 and vis_fc2.1 are summed by the quad that holds a row, in column order (row_dot), so every
// value is bit-identical to a round trip through the row owners.  Leaves x2 (base_fc.2's output +
// the vis_fc residual) in tile columns [96,128), rgb_fc.0's pre-activations in [128,144) and vis2 in xch slot XCH_L2.
// Ring stages (each warp group waits and releases on its own): base_fc.2 | vis_fc.0 (B hi / lo at stage floats
// 0 / 1024) + vis_fc.2 (2048 / 3072) | vis_fc2.0 (0 / 1024) + rgb_fc.0 (2048 / 3072, K step 4 512 floats further).
// tk: where the phase stamps after base_fc.2, vis_fc.0, vis_fc.2 and vis_fc2.0 go (nullptr: none).
__device__ __forceinline__ void run_chain(Blk& b, const float* __restrict__ sw, float* __restrict__ xch, int fr, long long* tk) {
  const int lane = b.row & 31, q = lane & 3;
  auto stage = [&](int s) {
    const uint32_t i = b.wi + s;
    tc::mbar_wait(b.wfull + i % NBUF, (i / NBUF) & 1);
    return b.ring_addr + (i % NBUF) * (RING_STAGE * 4);
  };
  auto release = [&](int s) {
    if (b.leader) tc::mbar_arrive(b.wempty + (b.wi + s) % NBUF);
  };
  // base_fc.2: K = 64 from the tile; the row scalars load under its MMAs
  uint32_t base = stage(0);
  float d[16];
  issue_frag_ss<8, 256>(b, d, tc::smem_desc_sw128(base), tc::smem_desc_sw128(base + 2048 * 4));
  float w1[2], mr[2], t0[2], t1[2];                 // t0, t1: rgb_fc.0's K tail, columns 32 + q and 36 + q (t0 of lane 0 is vis2)
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const float* __restrict__ x = xch + XCH_ROW * 128 + fr + 8 * r;
    w1[r] = x[0];
    mr[r] = x[128];
    t0[r] = q == 0 ? 0.f : x[(1 + q) * 128];
    t1[r] = q == 0 ? x[5 * 128] : 0.f;
  }
  wait_frag(d);
  release(0);
  float xr[16];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 bb = *reinterpret_cast<const float2*>(sw + SW_B1B + 8 * j + 2 * q);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      xr[4 * j + 2 * r] = elu(d[4 * j + 2 * r] + bb.x);
      xr[4 * j + 2 * r + 1] = elu(d[4 * j + 2 * r + 1] + bb.y);
    }
  }
  uint32_t ah[4][4], al[4][4];
  frag_to_a(xr, lane, ah, al);
  if (tk) tk[0] = clock64();
  // vis_fc.0 (row scale w1 in the epilogue)
  base = stage(1);
  issue_frag_ra<32, 4, 0>(d, ah, al, tc::smem_desc_sw128(base), tc::smem_desc_sw128(base + 1024 * 4));
  wait_frag_ra<32, 4>(d, ah, al);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 bb = *reinterpret_cast<const float2*>(sw + SW_V0B + 8 * j + 2 * q);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      d[4 * j + 2 * r] = elu(fmaf(w1[r], d[4 * j + 2 * r], bb.x));
      d[4 * j + 2 * r + 1] = elu(fmaf(w1[r], d[4 * j + 2 * r + 1], bb.y));
    }
  }
  frag_to_a(d, lane, ah, al);
  if (tk) tk[1] = clock64();
  // vis_fc.2, then vis_fc.1 (the vis_fc.0 outputs' dot product; under the MMAs, with their A registers pinned, it spills)
  float e[16];
  issue_frag_ra<32, 4, 0>(e, ah, al, tc::smem_desc_sw128(base + 2048 * 4), tc::smem_desc_sw128(base + 3072 * 4));
  wait_frag_ra<32, 4>(e, ah, al);
  release(1);
  float visa[2];
  {
    float lg[2];
    row_dot(d, sw + SW_V1LW, sw[SW_V1LB], lane, lg);
#pragma unroll
    for (int r = 0; r < 2; ++r) visa[r] = sigmoidf_(elu(lg[r])) * mr[r];
  }
  // x2 = xr + vis_fc.2's outputs: A of vis_fc2.0 and of rgb_fc.0's first 4 K steps
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 bb = *reinterpret_cast<const float2*>(sw + SW_V1B + 8 * j + 2 * q);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      xr[4 * j + 2 * r] += elu(e[4 * j + 2 * r] + bb.x);
      xr[4 * j + 2 * r + 1] += elu(e[4 * j + 2 * r + 1] + bb.y);
    }
  }
  uint32_t a2h[5][4], a2l[5][4];
  frag_to_a(xr, lane, a2h, a2l);
  if (tk) tk[2] = clock64();
  // vis_fc2.0; x2 goes to the tile under its MMAs
  base = stage(2);
  issue_frag_ra<32, 4, 0>(d, a2h, a2l, tc::smem_desc_sw128(base), tc::smem_desc_sw128(base + 1024 * 4));
  tc::acc_store_half<32>(b.act, 96, b.row, b.wg, xr);
  wait_frag_ra<32, 4>(d, a2h, a2l);
  float vis2[2];
  {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 bb = *reinterpret_cast<const float2*>(sw + SW_V20B + 8 * j + 2 * q);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        d[4 * j + 2 * r] = elu(fmaf(visa[r], d[4 * j + 2 * r], bb.x));
        d[4 * j + 2 * r + 1] = elu(fmaf(visa[r], d[4 * j + 2 * r + 1], bb.y));
      }
    }
    float l2[2];
    row_dot(d, sw + SW_V21W, sw[SW_V21B], lane, l2);
#pragma unroll
    for (int r = 0; r < 2; ++r) vis2[r] = sigmoidf_(l2[r]) * mr[r];
  }
  if (tk) tk[3] = clock64();
  // rgb_fc.0: K = 32 (x2) + the tail (vis2, dd0, dd1, dd2 | dd3, 0, 0, 0), N = 16
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    tc::split_tf32(q == 0 ? vis2[r] : t0[r], a2h[4][r], a2l[4][r]);
    tc::split_tf32(t1[r], a2h[4][2 + r], a2l[4][2 + r]);
  }
  float g[8];
  issue_frag_ra<16, 5, 128>(g, a2h, a2l, tc::smem_desc_sw128(base + 2048 * 4), tc::smem_desc_sw128(base + 3072 * 4));
  if (q < 2) xch[XCH_L2 * 128 + fr + 8 * q] = q ? vis2[1] : vis2[0];
  wait_frag_ra<16, 5>(g, a2h, a2l);
  release(2);
  b.wi += 3;
  tc::acc_store_half<16>(b.act, 128, b.row, b.wg, g);
}

// ---- this thread's columns of its row ----
// own_index(b, c): the float index of column c + 4 wg of this row, c a multiple of 8 (= tc::act_index(row, c + 4 wg))
__device__ __forceinline__ int own_index(const Blk& b, int c) { return (c >> 5) * 4096 + b.rbase + ((((c & 31) >> 2) ^ b.key) << 2); }
// the Q 4-column groups this warp group owns in columns [col, col + 8Q): v[4q + i] = column col + 8q + 4 wg + i
template <int Q>
__device__ __forceinline__ void ld_own(const Blk& b, int col, float* v) {
#pragma unroll
  for (int q = 0; q < Q; ++q) {
    const float4 t = *reinterpret_cast<const float4*>(b.act + own_index(b, col + 8 * q));
    v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
  }
}
// the same columns of a row of activations -> hi parts from `hi`, lo parts from `lo`
template <int Q>
__device__ __forceinline__ void st_own(const Blk& b, int hi, int lo, const float* v) {
#pragma unroll
  for (int q = 0; q < Q; ++q) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) tc::split_tf32(v[4 * q + j], h[j], l[j]);
    *reinterpret_cast<uint4*>(b.act + own_index(b, hi + 8 * q)) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(b.act + own_index(b, lo + 8 * q)) = make_uint4(l[0], l[1], l[2], l[3]);
  }
}
// entries 8q + 4 wg + [0,4) of a weight or bias vector (shared memory, 16-byte aligned)
__device__ __forceinline__ float4 own4(const Blk& b, const float* __restrict__ w, int q) {
  return *reinterpret_cast<const float4*>(w + 8 * q + 4 * b.wg);
}
// + the matching entries of a bias vector
template <int Q>
__device__ __forceinline__ void add_bias_own(const Blk& b, float* x, const float* __restrict__ bias) {
#pragma unroll
  for (int q = 0; q < Q; ++q) {
    const float4 t = own4(b, bias, q);
    x[4 * q] += t.x; x[4 * q + 1] += t.y; x[4 * q + 2] += t.z; x[4 * q + 3] += t.w;
  }
}
// this thread's row of the activation tile, all columns [col, col + 4Q), col a multiple of 4
template <int Q>
__device__ __forceinline__ void ld_row(const Blk& b, int col, float* v) {
#pragma unroll
  for (int q = 0; q < Q; ++q) {
    const float4 t = *reinterpret_cast<const float4*>(b.act + tc::act_index(b.row, col + 4 * q));
    v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
  }
}

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
  const int stages_per_tile = n_heads + 16;                    // stage_source
  const int n_tiles = kp.n_tiles;                              // tiles of PB points
  const int iters = (n_tiles + int(gridDim.x) - 1) / int(gridDim.x);
  const float* __restrict__ W = pp.w_point;

  // ---------------- one-time setup ----------------
  if (tid == 0) {
    for (int i = 0; i < NBUF; ++i) { tc::mbar_init(wfull + i, 1); tc::mbar_init(wempty + i, 2); }   // empty: one arrival per compute warp group
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
    if (tid < stages_per_tile) reinterpret_cast<int4*>(smem + OFF_STAB)[tid] = stage_source(tid, n_heads);
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

  if (tid >= NCOMP) {
    // ---------------- producer warp group: a stage goes out the moment its ring slot is free ----------------
    tc::setmaxnreg_dec<REG_PROD>();
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
    return;
  }

  // ---------------- compute warp groups ----------------
  tc::setmaxnreg_inc<REG_COMP>();
  const int fh = pp.fh, fw = pp.fw, h = pp.h, w = pp.w;
  const bool feat_align = (fh == h && fw == w);
  const int grp = lane / G;                       // point of this lane inside the warp (>= PPW: idle lane)
  const bool idle = P2 ? false : grp >= PPW;     // a compile-time false for the power-of-two groups
  const int v = P2 ? lane % G : lane - grp * G;   // view of this row (>= rfn: padding lane)
  const int pl = P2 ? (tid & 127) / G : (warp & 3) * PPW + grp;   // point inside the block
  const int pq = P2 ? pl : (idle ? 0 : pl);       // the same, < PB for idle lanes too: the per-point row this row reads
  const int lane0 = lane - v;                     // first lane of this point's group
  float* const stg = smem + OFF_STG + warp * 32 * STG_ROW;
  float* const xch = smem + OFF_XCH;
  // sums / maxima over the lanes of a point
  auto gsum = [&](float x) { if constexpr (P2) return bsum<G>(x); else return gsum_np2<G>(stg, lane, lane0, idle, x); };
  auto gmax = [&](float x) { if constexpr (P2) return bmax<G>(x); else return gmax_np2<G>(stg, lane, lane0, idle, x); };
  auto gpool16 = [&](const float (&in)[16], float (&out)[16]) {
    if constexpr (P2) pool_rows<G, 16>(stg, lane, lane0, v, in, out); else pool_rows_np2<G, 16>(stg, lane, lane0, v, idle, in, out);
  };

  Blk b;
  b.act = smem + OFF_ACT;
  b.act_addr = tc::smem_u32(b.act);
  b.row = tid & 127;
  b.wg = tid >> 7;
  b.rbase = (b.row >> 3) * 256 + (b.row & 7) * 32;
  b.key = (b.row & 7) ^ b.wg;
  b.leader = b.row == 0;
  b.wfull = wfull; b.wempty = wempty;
  b.ring_addr = tc::smem_u32(ring);
  b.wi = 0;
  const int row = b.row, wg = b.wg;
  const int fr = 64 * wg + 16 * (row >> 5) + ((row & 31) >> 2);           // this thread's accumulator fragment rows: fr, fr + 8
  // a point's 16 pooled values (which every lane of the point holds) -> its row of the per-point operand: value 4q + i at
  // column col + 8q + 4 wg + i, the layout st_own gives a row of the tile; lane v < 4 of the point stores q = v
  auto put_point = [&](float* op, int col, const float (&st)[16]) {
    if (v < 4 && !idle) {
      float4 o = make_float4(st[0], st[1], st[2], st[3]);
      if (v == 1) o = make_float4(st[4], st[5], st[6], st[7]);
      else if (v == 2) o = make_float4(st[8], st[9], st[10], st[11]);
      else if (v == 3) o = make_float4(st[12], st[13], st[14], st[15]);
      *reinterpret_cast<float4*>(op + pl * OP_ROW + col + 8 * v + 4 * wg) = o;
    }
  };

  // phase stamps exist only in the DEBUG instantiation (nr_point_kernel_timing / nr_point_kernel_debug): [tile][warp group][32]
#define PM_TICK(id)                                                                                      \
  if constexpr (DEBUG) {                                                                                 \
    if (kp.timing != nullptr && blockIdx.x == 0 && row == 0 && it < 64) kp.timing[(it * 2 + wg) * 32 + (id)] = clock64(); \
  }
  for (int it = 0; it < iters; ++it) {
    const int tile = it * int(gridDim.x) + int(blockIdx.x);
    if (tile >= n_tiles) {
      // nothing to render in this iteration: still take part in the weight-ring accounting
      for (int s = 0; s < stages_per_tile; ++s) {
        if (b.leader) {
          const uint32_t i = b.wi + s;
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
    // ---------------- ray geometry of this row's point (every lane of the group, in both warp groups, computes the same values) ----------------
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
    // ---------------- bilinear gather of this warp's 32 rows, this warp group's 16 of the 32 channels: 4 lanes x float4 per texel ----------------
    // The gathering lanes and the row owner are different lanes: the row's coordinates come over by shuffle, the channels
    // go back through the warp-private transposition buffer.  Lane l of a texel fetches channels ch0 + 8l + 4wg + [0,4)
    // (the warp group's own columns) and puts them at buffer columns 4l + [0,4).
    const int gch = 8 * (lane & 3) + 4 * wg;
    auto gather16 = [&](const int ch0) {
      const int qw = lane >> 2, l = lane & 3;
      __syncwarp();
#pragma unroll 1
      for (int rb = 0; rb < 32; rb += 8 * GB) {
        float4 t[GB][4];
        float wq[GB][4];
        bool on[GB];
#pragma unroll
        for (int u = 0; u < GB; ++u) {
          const int j = rb + 8 * u + qw;                                   // row (= lane) whose texels these 4 lanes fetch
          const int code = __shfl_sync(0xffffffffu, tcode, j);
#pragma unroll
          for (int k = 0; k < 4; ++k) wq[u][k] = __shfl_sync(0xffffffffu, tw[k], j);
          on[u] = code >= 0;
          if (on[u]) {
            const float* __restrict__ base = pp.feat + (code & ~63) + ch0 + gch;
            const int dx = (code & 1) << 6, dy = (code & 2) ? fw * 64 : 0;
            t[u][0] = ldg4(base); t[u][1] = ldg4(base + dx);
            t[u][2] = ldg4(base + dy); t[u][3] = ldg4(base + dy + dx);
          }
        }
#pragma unroll
        for (int u = 0; u < GB; ++u) {
          const int j = rb + 8 * u + qw;
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
    gather16(0);

    PM_TICK(2)
    // ---------------- dist decoder on the tensor cores: A[0:32] <- this row's ray_feats ----------------
    {
      float x[16];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 t4 = *reinterpret_cast<const float4*>(stg + lane * STG_ROW + 4 * q);
        x[4 * q] = t4.x; x[4 * q + 1] = t4.y; x[4 * q + 2] = t4.z; x[4 * q + 3] = t4.w;
      }
      st_own<4>(b, 0, 64, x);
      if (DEBUG && kp.dbg != nullptr && row_ok) {
        float* __restrict__ o = kp.dbg + (size_t(v) * N + n) * 76;
        for (int k = 0; k < 16; ++k) o[12 + 8 * (k >> 2) + 4 * wg + (k & 3)] = x[k];
      }
    }
    gather16(32);                                                                  // img_feats: stay in the buffer until ray_dir_fc
    PM_TICK(3)
    // the heads: each warp group runs them for the 64 rows whose MMAs it issues (run_head); A[0:32] comes from both
    tc::fence_proxy_async_smem();
    tc::named_sync(BAR_LAYER, NCOMP);
#pragma unroll 1
    for (int hd = 0; hd < n_heads; ++hd) run_head(b, sw + SW_HEAD + hd * SW_HEAD_STRIDE, xch + (XCH_HEAD + 2 * hd) * 128, fr);
    PM_TICK(4)
    tc::named_sync(BAR_LAYER, NCOMP);                                              // head outputs -> the row owners
    // hit and visibility go into warp group 0's columns
    float hit = 0.f, visib = 0.f;
    if (wg == 0) {
      float hv[4][2];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        hv[k][0] = k < n_heads ? xch[(XCH_HEAD + 2 * k) * 128 + row] : 0.f;
        hv[k][1] = k < n_heads ? xch[(XCH_HEAD + 2 * k + 1) * 128 + row] : 0.f;
      }
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
      float x[4] = {0.f, 0.f, 0.f, 0.f};
      if (wg == 0) { x[0] = (hit - 0.5f) * 2.f; x[1] = (visib - 0.5f) * 2.f; }
      st_own<1>(b, 32, 96, x);                                                     // A[32:40] = hit', vis', 0... (the heads' hidden layer is dead)
    }
    run_layer<32, 5, 0, 4, 32, 0, 2048 * 4, 4096, true, true>(b);                 // prob_embed.0: K = 32 + 8
    {
      float x[16];
      ld_own<4>(b, 128, x);
      add_bias_own<4>(b, x, sw + SW_PE0B);
#pragma unroll
      for (int j = 0; j < 16; ++j) x[j] = fmaxf(x[j], 0.f);
      st_own<4>(b, 0, 64, x);                                                      // over ray_feats: their last reader has completed
    }
    PM_TICK(5)
    // prob_embed.2 with neuray_fc.0 behind it: N = 48, accumulator columns [96,144)
    issue_layer<48, 4, 0, 64, 4, 0, 96, 0, 1, 0, 1536 * 4, 0, true, true, false>(b);
    float gate;
    {
      float x[16];
      ld_own<4>(b, 96, x);
      add_bias_own<4>(b, x, sw + SW_PE1B);                                         // neuray_feat
      st_own<4>(b, 0, 64, x);
      float h8[8];
      ld_row<2>(b, 128, h8);                                                       // neuray_fc.0 pre-activations (both warp groups: the whole row)
      gate = sw[SW_NF1B];
#pragma unroll
      for (int j = 0; j < 8; ++j) gate = fmaf(sw[SW_NF1W + j], elu(h8[j] + sw[SW_NF0C + j]), gate);
    }
    // base_fc.0, K round A: the neuray_feat inputs (B chunks 5..8), accumulator columns [96,160)
    issue_layer<64, 4, 0, 64, 4, 0, 96, 5, 3, 0, 2048 * 4, 0, true, false, false>(b);
    // rgb_feat (35) + zero padding: rf[4q + i] = column 8q + 4wg + i
    float rf[20];
    {
      {
        float h8[8];
        const float* __restrict__ w0 = sw + SW_RD0W;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const float4 b4 = own4(b, sw + SW_RD0B, q), k0 = own4(b, w0, q), k1 = own4(b, w0 + 16, q), k2 = own4(b, w0 + 32, q), k3 = own4(b, w0 + 48, q);
          h8[4 * q] = elu(fmaf(k3.x, dd[3], fmaf(k2.x, dd[2], fmaf(k1.x, dd[1], fmaf(k0.x, dd[0], b4.x)))));
          h8[4 * q + 1] = elu(fmaf(k3.y, dd[3], fmaf(k2.y, dd[2], fmaf(k1.y, dd[1], fmaf(k0.y, dd[0], b4.y)))));
          h8[4 * q + 2] = elu(fmaf(k3.z, dd[3], fmaf(k2.z, dd[2], fmaf(k1.z, dd[1], fmaf(k0.z, dd[0], b4.z)))));
          h8[4 * q + 3] = elu(fmaf(k3.w, dd[3], fmaf(k2.w, dd[2], fmaf(k1.w, dd[1], fmaf(k0.w, dd[0], b4.w)))));
        }
        st_own<2>(b, 48, 64, h8);                                                  // ray_dir_fc.2 operand: hi [48,64), lo [64,80)
      }
      issue_layer_resident<48, 2, 48, 16, 0, 0, 1536 * 4, 0, false>(b, tc::smem_u32(smem + OFF_RD1));   // ray_dir_fc.2: K = 16, accumulator [0,48)
      ld_own<5>(b, 0, rf);
      // + [rgb | img_feats]: column c holds img_feats channel c - 3, which warp group ((c - 3) >> 2) & 1 gathered into
      // its buffer column 4 ((c - 3) >> 3) + ((c - 3) & 3).  Of this warp group's columns 8q + 4wg + i, i = 3 is in its own
      // buffer (column 4q), i < 3 in the other warp group's (column 4(q - 1 + wg) + 1 + i).
      const float* __restrict__ mine = stg + lane * STG_ROW;
      const float* __restrict__ other = smem + OFF_STG + (warp ^ 4) * 32 * STG_ROW + lane * STG_ROW;
#pragma unroll
      for (int q = 0; q < 5; ++q) {
        const float4 bb = own4(b, sw + SW_RD1B, q);                                // (q = 4, wg = 1: past the 36 biases, unused)
        float* r = rf + 4 * q;
        r[0] = elu(r[0] + bb.x); r[1] = elu(r[1] + bb.y); r[2] = elu(r[2] + bb.z); r[3] = elu(r[3] + bb.w);
        if (q == 0 && wg == 0) {
          r[0] += rgbin[0]; r[1] += rgbin[1]; r[2] += rgbin[2];
        } else if (q < 4 || wg == 0) {
#pragma unroll
          for (int i = 0; i < 3; ++i) r[i] += other[4 * (q - 1 + wg) + 1 + i];
        }
        if (q < 4) r[3] += mine[4 * q];
        if (q == 4) {
          if (wg == 0) r[3] = 1.f;                                                 // constant input: base_fc.0's bias is column 35 of its tile
          else r[0] = r[1] = r[2] = r[3] = 0.f;
        }
      }
      if (DEBUG && kp.dbg != nullptr && row_ok) {
        float* __restrict__ o = kp.dbg + (size_t(v) * N + n) * 76;
        for (int k = 0; k < 16; ++k) o[44 + 8 * (k >> 2) + 4 * wg + (k & 3)] = mine[k];
      }
      st_own<5>(b, 0, 48, rf);                                                     // rgb_feat: hi [0,40), lo [48,88)
    }
    // base_fc.0, K round B: rgb_feat (B chunks 0..4)
    issue_layer<64, 5, 0, 48, 5, 0, 96, 0, 3, 0, 2048 * 4, 0, false, true, true>(b);
    if (DEBUG && kp.dbg != nullptr && row_ok && wg == 0) {
      float* __restrict__ o = kp.dbg + (size_t(v) * N + n) * 76;
      o[0] = mrow; o[1] = zrow; o[2] = hit; o[3] = visib; o[4] = dbg_px; o[5] = dbg_py;
      o[6] = dbg_dir[0]; o[7] = dbg_dir[1]; o[8] = dbg_dir[2]; o[9] = rgbin[0]; o[10] = rgbin[1]; o[11] = rgbin[2];
    }

    PM_TICK(6)
    // ---------------- view pooling #1 (ibrnet.py:336-339) -> the view-pooled part of base_fc.0, once per point ----------------
    // Every lane of a point ends a round with the point's statistics: 8 features x (mean0, var0, mean1, var1) = K 32 per
    // round (statistic t of feature i at column 32 R + 8t + i, so warp group c pools features 4c .. 4c + 3 of the round).
    // They go into the point's row of the per-point operand (PB rows, K 160) and each round's K 32 is multiplied as soon
    // as it is complete, B from the round's ring stage, into a per-point [PB][64] result that the epilogue adds to every
    // view's row.  One barrier per round: it publishes the round's operand columns and tells the leaders (b.leader) that every
    // warp is done with the previous round's stage (the fifth stage can only load into the first one's ring slot).  The sums over
    // the views go through the warp's transposition buffer (pool_rows); the variance comes from the weighted second moment:
    //   sum_v w (x - mu)^2 = sum_v w x^2 - mu^2 (2 - sum_v w),  mu = sum_v w x   (the reference's mean is NOT normalised)
    const float msum = gsum(mrow);
    const float w1 = mrow / (msum + 1e-8f);
    const float w0 = sigmoidf_(gate) * w1;
    {
      const float c1 = 2.f - gsum(w1), c0 = 2.f - gsum(w0);
      float* const op = b.act;
      const uint32_t s0 = b.wi;
      PtAcc<PB> acc = {};
      auto round = [&](auto rc) {
        constexpr int R = decltype(rc)::value;
        float in[16], st[16];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float x = (R == 4 && i == 3) ? 0.f : rf[4 * R + i];                // features 35.. (the constant, padding) pool to 0
          const float p0 = x * w0, p1 = x * w1;
          in[i] = p0; in[4 + i] = p0 * x; in[8 + i] = p1; in[12 + i] = p1 * x;
        }
        gpool16(in, st);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          st[4 + i] = fmaf(-st[i] * st[i], c0, st[4 + i]);
          st[12 + i] = fmaf(-st[8 + i] * st[8 + i], c1, st[12 + i]);
        }
        put_point(op, 32 * R, st);
        tc::named_sync(BAR_LAYER, NCOMP);
        if (R > 0 && b.leader) tc::mbar_arrive(wempty + (s0 + R - 1) % NBUF);
        tc::mbar_wait(wfull + (s0 + R) % NBUF, ((s0 + R) / NBUF) & 1);
        point_mma<PB, 4>(acc, op, 32 * R, ring + ((s0 + R) % NBUF) * RING_STAGE, warp, lane);
      };
      round(std::integral_constant<int, 0>{}); round(std::integral_constant<int, 1>{}); round(std::integral_constant<int, 2>{});
      round(std::integral_constant<int, 3>{}); round(std::integral_constant<int, 4>{});
      point_store(acc, smem + OFF_PT, warp, lane);
      tc::named_sync(BAR_LAYER, NCOMP);                                            // per-point result visible; the last stage read
      if (b.leader) tc::mbar_arrive(wempty + (s0 + 4) % NBUF);
      b.wi += 5;
    }

    PM_TICK(7)
    // ---------------- base_fc on the tensor cores ----------------
    // base_fc.0 = the per-view rounds A and B (accumulator [96,160), bias included) + the point's view-pooled part
#pragma unroll
    for (int c0 = 0; c0 < 64; c0 += 32) {
      float x[16];
      ld_own<4>(b, 96 + c0, x);
      add_bias_own<4>(b, x, smem + OFF_PT + pq * PT_ROW + c0);
#pragma unroll
      for (int j = 0; j < 16; ++j) x[j] = elu(x[j]);
      st_own<4>(b, c0, 64 + c0, x);                                                // lo half 1 lands on accumulator columns already consumed
    }
    {
      // the row scalars of the chain's fragment rows, into the heads' exchange slots (dead since the heads' outputs were
      // read): w1, mrow, dd[0] from warp group 0, dd[1..3] from warp group 1
      const float rs[6] = {w1, mrow, dd[0], dd[1], dd[2], dd[3]};
#pragma unroll
      for (int k = 0; k < 3; ++k) xch[(XCH_ROW + 3 * wg + k) * 128 + row] = wg ? rs[3 + k] : rs[k];
    }
    PM_TICK(8)
    // ---------------- base_fc.2, vis_fc, vis_fc2, rgb_fc.0: each warp group for its own 64 rows (run_chain) ----------------
    tc::fence_proxy_async_smem();
    tc::named_sync(BAR_LAYER, NCOMP);
    {
      long long* tk = nullptr;                                                     // phase stamps 9 .. 12 inside the chain
      if constexpr (DEBUG) {
        if (kp.timing != nullptr && blockIdx.x == 0 && row == 0 && it < 64) tk = kp.timing + (it * 2 + wg) * 32 + 9;
      }
      run_chain(b, sw, xch, fr, tk);
    }
    tc::named_sync(BAR_LAYER, NCOMP);                                              // x2, rgb_fc.0 and vis2 -> the row owners
    float xr[16];
    ld_own<4>(b, 96, xr);
    const float vis2 = xch[XCH_L2 * 128 + row];
    float xg[16];                                                                  // warp group 1: rgb_fc.0 outputs, for the colour blend at the end
    if (wg == 1) ld_row<4>(b, 128, xg);

    PM_TICK(13)
    // ---------------- view pooling #2 (ibrnet.py:352-353) -> geometry_fc.0 on the tensor cores ----------------
    const float vs = gsum(vis2);
    const float w2 = vis2 / (vs + 1e-8f);
    const float sw2 = gsum(w2);
    const float wmean = sw2 / float(rfn);
    {
      // geometry_fc.0, once per point: per-point operand (PB rows) = two K rounds of 16 features x (mean, var) (feature i
      // of round R at columns 32R + i and 32R + 16 + i: warp group c pools features 16R + 8q + 4c + [0,4), its
      // xr[8R + 4q + i]), then the mean weight and the constant that multiplies the bias column at columns 64, 65; B from
      // three ring stages, all in the ring at once; sums over the views through pool_rows, variance from the second
      // moment (above)
      const float c2 = 2.f - sw2;
      float* const op = b.act;
      auto ground = [&](auto rc) {
        constexpr int R = decltype(rc)::value;
        float in[16], st[16];
#pragma unroll
        for (int i = 0; i < 8; ++i) { const float p = xr[8 * R + i] * w2; in[i] = p; in[8 + i] = p * xr[8 * R + i]; }
        gpool16(in, st);
#pragma unroll
        for (int i = 0; i < 8; ++i) st[8 + i] = fmaf(-st[i] * st[i], c2, st[8 + i]);
        put_point(op, 32 * R, st);
      };
      ground(std::integral_constant<int, 0>{}); ground(std::integral_constant<int, 1>{});
      if (wg == 0 && v == 0 && !idle) {
        *reinterpret_cast<float4*>(op + pl * OP_ROW + 64) = make_float4(wmean, 1.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(op + pl * OP_ROW + 68) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      tc::named_sync(BAR_LAYER, NCOMP);
      const uint32_t s0 = b.wi;
      PtAcc<PB> acc = {};
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        tc::mbar_wait(wfull + (s0 + s) % NBUF, ((s0 + s) / NBUF) & 1);
        const float* w = ring + ((s0 + s) % NBUF) * RING_STAGE;
        if (s < 2) point_mma<PB, 4>(acc, op, 32 * s, w, warp, lane);
        else point_mma<PB, 1>(acc, op, 64, w, warp, lane);
      }
      point_store(acc, smem + OFF_PT, warp, lane);
      tc::named_sync(BAR_LAYER, NCOMP);                                            // per-point result visible; the stages read
      if (b.leader) {
#pragma unroll
        for (int s = 0; s < 3; ++s) tc::mbar_arrive(wempty + (s0 + s) % NBUF);
      }
      b.wi += 3;
    }

    PM_TICK(14)
    if (wg == 0) {
      // ---------------- geometry_fc.2 across the lanes of a point ----------------
      // the point's 64 hidden pre-activations are its row of the per-point result; lane v takes [v*CPL, (v+1)*CPL)
      // (GE = the lanes of the point that take part: all G of a power-of-two group, else the first 8 / 4)
      const int vg = (P2 || v < GE) ? v : 0;
      float hh[CPL];
      const float* __restrict__ hp = smem + OFF_PT + pq * PT_ROW + vg * CPL;
      if constexpr (CPL >= 4) {
#pragma unroll
        for (int q = 0; q < CPL / 4; ++q) {
          const float4 t = *reinterpret_cast<const float4*>(hp + 4 * q);
          hh[4 * q] = t.x; hh[4 * q + 1] = t.y; hh[4 * q + 2] = t.z; hh[4 * q + 3] = t.w;
        }
      } else {
        const float2 t = *reinterpret_cast<const float2*>(hp);
        hh[0] = t.x; hh[1] = t.y;
      }
#pragma unroll
      for (int j = 0; j < CPL; ++j) hh[j] = (P2 || v < GE) ? elu(hh[j]) : 0.f;
      float out[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) out[k] = 0.f;
#pragma unroll
      for (int k = 0; k < 16; ++k) {                                               // sWg1 is stored output-major: [16][64]
        float wk[CPL];
        ld_cols<GE>(sWg1 + k * 64, vg, wk);
#pragma unroll
        for (int j = 0; j < CPL; ++j) out[k] = fmaf(wk[j], hh[j], out[k]);
      }
      float sum[16];
      if constexpr (P2) pool_rows<G, 16>(stg, lane, lane0, v, out, sum); else pool_rows_np2<G, 16>(stg, lane, lane0, v, idle, out, sum);
#pragma unroll
      for (int k = 0; k < 16; ++k) out[k] = elu(sum[k] + sWg1[64 * 16 + k]);
      if (v == 0 && pt_ok) {
        float4* __restrict__ dst = reinterpret_cast<float4*>(pp.point_rec + size_t(n) * REC);
        dst[0] = make_float4(out[0], out[1], out[2], out[3]); dst[1] = make_float4(out[4], out[5], out[6], out[7]);
        dst[2] = make_float4(out[8], out[9], out[10], out[11]); dst[3] = make_float4(out[12], out[13], out[14], out[15]);
      }
    } else {
      // ---------------- rgb_fc.1 / .2 and the softmax colour blend over the views (ibrnet.py:365-367) ----------------
      float h8[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) h8[j] = sw[SW_RGB1B + j];
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const float a = elu(xg[k] + sw[SW_RGB0B + k]);
        const float4 wa = *reinterpret_cast<const float4*>(sw + SW_RGB1W + k * 8);
        const float4 wb = *reinterpret_cast<const float4*>(sw + SW_RGB1W + k * 8 + 4);
        h8[0] = fmaf(wa.x, a, h8[0]); h8[1] = fmaf(wa.y, a, h8[1]); h8[2] = fmaf(wa.z, a, h8[2]); h8[3] = fmaf(wa.w, a, h8[3]);
        h8[4] = fmaf(wb.x, a, h8[4]); h8[5] = fmaf(wb.y, a, h8[5]); h8[6] = fmaf(wb.z, a, h8[6]); h8[7] = fmaf(wb.w, a, h8[7]);
      }
      float l3 = sw[SW_RGB2B];
#pragma unroll
      for (int j = 0; j < 8; ++j) l3 = fmaf(sw[SW_RGB2W + j], elu(h8[j]), l3);
      // masked views get -1e9 like the reference; padding lanes must not take part at all
      const float logit = v >= rfn ? -3.0e38f : (mrow == 0.f ? -1e9f : l3);
      const float mx = gmax(logit);
      const float e = v >= rfn ? 0.f : expf(logit - mx);
      float acc[4] = {e, e * rgbin[0], e * rgbin[1], e * rgbin[2]};
      if constexpr (P2) bsum_vec<G, 4>(acc); else gsum4_np2<G>(stg, lane, lane0, idle, acc);
      if (v == 0 && pt_ok) {
        float4* __restrict__ dst = reinterpret_cast<float4*>(pp.point_rec + size_t(n) * REC);
        dst[4] = make_float4(acc[1] / acc[0], acc[2] / acc[0], acc[3] / acc[0], msum);
      }
    }
    PM_TICK(15)
  }
#undef PM_TICK
}

}  // namespace pm3
