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
//   * MMAs: warp group c issues the m64 wgmma of rows 64c .. 64c + 63 of every layer, each layer as one 3xTF32 batch
//     (mma_batch; the TF32 mode, point_kernel_tf32, issues the hi*hi pass alone: NP = 1).  Every per-view layer runs in the accumulator fragment of the warp group that issues it, for its own
//     64 rows: the dist-decoder heads (run_head), the front hit/vis .. base_fc.0 (in the kernel body) and the tail
//     base_fc.2 .. rgb_fc.0 (run_chain).  Nothing in them is pooled or needs the row-owner layout; A comes from registers
//     after each stretch's first layer, row sums run over the 4 lanes that hold a row, and the results go to the row
//     owners through the tile and a small shared array (xch) at one 256-thread barrier per stretch.  The ring's "empty"
//     barriers count one arrival per compute warp group, so each releases those stages on its own.
//   * activation tile (80 KB of shared memory, 160 columns x 128 rows, tc::act_index): hi parts at columns [0,64), lo parts
//     at [64,128), accumulator at [128,160).  base_fc.0 (N = 64) has its per-view inputs issued in two K rounds into one
//     accumulator, round A (the 32 neuray_feat inputs) and round B (the 40 rgb_feat inputs) with A from registers; the
//     front stores it at [96,160).  Its epilogue reads the accumulator half by half, adds the point's view-pooled part and
//     writes base_fc.2's operand over the columns it has already consumed (the same warp group owns column c and c + 32,
//     so no other warp group reads them).  run_chain leaves x2 at [96,128) and rgb_fc.0's pre-activations at [128,144).
//   * per-point layers: the view-pooled part of base_fc.0 (K 140 -> 160) and geometry_fc.0 have the same inputs for every
//     view of a point, so they are multiplied once per point, not once per row: the pooled statistics go into a compact
//     operand of PB rows (one per point, in tile columns [0,64) while those are dead), the eight compute warps multiply
//     it with warp-level mma.sync (3xTF32, B read straight from the weight ring stages, warp w computes outputs
//     8w .. 8w + 7) into a [PB][64] result in shared memory (OFF_PT), and every row of the point reads it from there.
//   * the rest of shared memory: 4 x 16 KB weight ring (TMA bulk copies, fed by the producer group; the view-pooled
//     base_fc.0 weights stream through it as five more stages), the resident tile of ray_dir_fc.2, small weights, camera
//     blocks, the row-scalar exchange, the per-point result, and one [32][36] transposition buffer per warp: gather (16
//     channels per warp group in two passes: ray_feats, then img_feats, which stay there until rgb_feat is built), the
//     cross-view pooling (pm::pool_rows) and the lane-group sums of the non-power-of-two groups all go through it.
#pragma once

namespace pm3 {

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
constexpr int BAR_LAYER = 1;                                  // named barrier of both compute warp groups
constexpr int BAR_WG = 2;                                     // + wg: named barrier of one compute warp group's 128 threads
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
// (o0, o1) of the 4 heads | the row scalars zrow, ihp, ihc, mrow, dd[0..3], rgbin[0..2] (XCH_FRONT + k, written before the
// heads; mrow, dd and rgbin stay there for the chain and the colour blend).  Once a warp group has read its rows' head
// outputs, the front's outputs over them: the neuray_fc gate and rgb_feat columns 32..34.  After pooling #1 the chain's
// w1 over the gate, and its vis_fc2 visibility over zrow.
constexpr int XCH_HEAD = 0, XCH_FRONT = 8, XCH_GATE = 0, XCH_RF = 1, XCH_W1 = 0, XCH_L2 = 8, XCH = 19 * 128;
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
// the per-point operand of a per-point layer: [point][OP_ROW] (K 160 used) in the first two slabs of the activation tile
// (columns [0,64)), which are dead while it is used (after base_fc.0's round B until its epilogue; after rgb_fc.0 until the
// next tile's gather).  Pooling #1 reads rgb_feat from the third slab (columns [64,96)) while its operand fills up.
constexpr int OP_ROW = 164;                                   // = 4 mod 32: the 32 lanes of an A-fragment load hit 32 banks
static_assert(32 * OP_ROW <= 2 * 4096, "per-point operand");
// rgb_feat columns 0..31 on their way from the front to pooling #1, in fp32, in tile slab 2 (columns [64,96)): row r,
// column c at RF_SLAB + rf_slab_index(r, c).  Rows 64c .. 64c + 63 keep to the half of the slab that holds those rows in
// the tile's own layout (floats 2048c .. 2048c + 2047), so the front of warp group c writes only its own rows: the other
// warp group may still be reading its half of the slab (ray_feats' lo part, A of its heads and of its prob_embed.0).
constexpr int RF_SLAB = 2 * 4096;
__host__ __device__ constexpr int rf_slab_index(int r, int c) { return (r >> 6) * 2048 + (c >> 2) * 256 + (r & 63) * 4 + (c & 3); }
static_assert(rf_slab_index(63, 31) < 2048 && rf_slab_index(64, 0) == 2048 && rf_slab_index(127, 31) < 4096 &&
                  tc::act_index(64, 64) - RF_SLAB == 2048, "rgb_feat: each warp group's rows in its own half of slab 2");

// ---- passes per product: NP = 3 (3xTF32, fp32 accuracy) or 1 (TF32 mode: the hi*hi pass alone) ----
// An A operand value -> its hi part and, for NP = 3, its lo part.  NP = 1 rounds to nearest (tc::tf32_rna) and leaves
// lo unwritten: no pass reads it.
template <int NP>
__device__ __forceinline__ void split(float x, uint32_t& hi, uint32_t& lo) {
  static_assert(NP == 1 || NP == 3, "passes per product");
  if constexpr (NP == 3) tc::split_tf32(x, hi, lo);
  else hi = tc::tf32_rna(x);
}

// ---- per-point layers: [points x K] x [K x 64] on warp-level mma.sync, NP passes ----
// Compute warp w (of 8) computes outputs 8w .. 8w + 7 for all PB points of the tile: MT m16 tiles of points, and one
// accumulator per pass (hi*hi, lo*hi, hi*lo) so that the MMAs of a K step do not wait for each other.
template <int PB, int NP>
struct PtAcc {
  static constexpr int MT = (PB + 15) / 16;
  float d[MT][NP][4];
};
// acc += op[points][kcol + k] * W[8w + n][k], k < 8 KS: B from a weight ring stage `w` that holds one K32 slab of a 64-row
// tile with layout L (K steps 0 .. KS - 1).  Operand rows at or past PB read as 0.
template <int PB, int KS, int NP>
__device__ __forceinline__ void point_mma(PtAcc<PB, NP>& acc, const float* __restrict__ op, int kcol, const float* __restrict__ w, tcl::Tile L, int warp,
                                          int lane) {
  const int g = lane >> 2, t = lane & 3;
  const float* __restrict__ bw = w + L.hi + warp * 256 + g * 32 + t;      // tc::sw128_index(8 warp + g, 8 j + t) = bw[((2j) ^ g) << 2]
  const float* __restrict__ aw = op + g * OP_ROW + kcol + t;
#pragma unroll
  for (int j = 0; j < KS; ++j) {
    const uint32_t bh[2] = {__float_as_uint(bw[((2 * j) ^ g) << 2]), __float_as_uint(bw[((2 * j + 1) ^ g) << 2])};
    uint32_t bl[2];
    if constexpr (NP == 3) {
      bl[0] = __float_as_uint(bw[L.lo - L.hi + (((2 * j) ^ g) << 2)]);
      bl[1] = __float_as_uint(bw[L.lo - L.hi + (((2 * j + 1) ^ g) << 2)]);
    }
#pragma unroll
    for (int m = 0; m < PtAcc<PB, NP>::MT; ++m) {
      const bool ok0 = 16 * m + 8 <= PB || 16 * m + g < PB, ok1 = 16 * m + 16 <= PB || 16 * m + 8 + g < PB;
      const float* __restrict__ a = aw + 16 * m * OP_ROW + 8 * j;
      const float x[4] = {ok0 ? a[0] : 0.f, ok1 ? a[8 * OP_ROW] : 0.f, ok0 ? a[4] : 0.f, ok1 ? a[8 * OP_ROW + 4] : 0.f};
      uint32_t ah[4], al[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) split<NP>(x[i], ah[i], al[i]);
      tc::mma_tf32_m16n8k8(acc.d[m][0], ah, bh);
      if constexpr (NP == 3) {
        tc::mma_tf32_m16n8k8(acc.d[m][1], al, bh);
        tc::mma_tf32_m16n8k8(acc.d[m][2], ah, bl);
      }
    }
  }
}
// the accumulated outputs -> pt[point][8w .. 8w + 7] (points < PB)
template <int PB, int NP>
__device__ __forceinline__ void point_store(const PtAcc<PB, NP>& acc, float* __restrict__ pt, int warp, int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int m = 0; m < PtAcc<PB, NP>::MT; ++m) {
    float o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if constexpr (NP == 3) o[i] = acc.d[m][0][i] + (acc.d[m][1][i] + acc.d[m][2][i]);
      else o[i] = acc.d[m][0][i];
    }
    float* __restrict__ p = pt + (16 * m + g) * PT_ROW + 8 * warp + 2 * t;
    if (16 * m + 8 <= PB || 16 * m + g < PB) *reinterpret_cast<float2*>(p) = make_float2(o[0], o[1]);
    if (16 * m + 16 <= PB || 16 * m + 8 + g < PB) *reinterpret_cast<float2*>(p + 8 * PT_ROW) = make_float2(o[2], o[3]);
  }
}

// ---- tensor-core layers: one wgmma batch of NP passes each ----
// A operand of a batch from the activation tile: K step c at column col + 8c, its lo part lo_off columns further, rows
// 64 wg .. 64 wg + 63
struct TileA {
  uint32_t act_addr;
  int wg, col, lo_off;
  template <int KS>
  __device__ void pin() const {}
  __device__ uint64_t operator()(int c, bool lo) const { return tc::act_desc(act_addr, col + 8 * c + (lo ? lo_off : 0), wg); }
};
__device__ __forceinline__ TileA tile_a(const Blk& b, int col, int lo_off) { return TileA{b.act_addr, b.wg, col, lo_off}; }
// A from registers (tc::wgmma_tf32_ra): K step c from h[c] / l[c] (l only for NP = 3).  The K steps a batch reads stay
// pinned until it has completed.
template <int KA, int NP>
struct RegA {
  uint32_t (&h)[KA][4];
  uint32_t (&l)[KA][4];
  template <int KS>
  __device__ void pin() const {
    tc::wgmma_fence_operand<KS>(h);
    if constexpr (NP == 3) tc::wgmma_fence_operand<KS>(l);
  }
  __device__ const uint32_t (&operator()(int c, bool lo) const)[4] { return lo ? l[c] : h[c]; }
};
template <int N>
__device__ __forceinline__ void wgmma(float (&d)[N / 2], uint64_t a, uint64_t b) { tc::wgmma_tf32<N>(d, a, b); }
template <int N>
__device__ __forceinline__ void wgmma(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b) { tc::wgmma_tf32_ra<N>(d, a, b); }
// B operand of a batch in a tensor-core tile (tcl::Tile t) at shared byte address `addr`: K step c is step c & 3 of slab c >> 2
struct TileB {
  uint64_t hi, lo;
  int slab16;                   // slab stride in 16-byte descriptor units
  __device__ uint64_t operator()(int c, bool l) const { return (l ? lo : hi) + (c >> 2) * slab16 + 2 * (c & 3); }
};
__device__ __forceinline__ TileB tile_b(uint32_t addr, tcl::Tile t) {
  return TileB{tc::smem_desc_sw128(addr + t.hi * 4), tc::smem_desc_sw128(addr + t.lo * 4), t.slab / 4};
}
// B of base_fc.0's per-view inputs from its K step k0 on: slab s of tcl::B0_L is ring stage wi + s
__device__ __forceinline__ auto base0_b(const Ring& ring, int k0) {
  return [=](int c, bool lo) {
    const int k = k0 + c;
    return tc::smem_desc_sw128(ring.slot(k >> 2).addr + (lo ? tcl::B0_L.lo : tcl::B0_L.hi) * 4) + 2 * (k & 3);
  };
}

// d (+)= A x B over K steps c < KS, issued by this warp group as one wgmma batch and waited for; `under` runs between the
// commit and the wait.  Every batch of the kernel goes through here, so every accumulator gets its products in the same
// order: pass hi*hi, lo*hi, hi*lo (the first NP of them), the K steps inside each pass.  a(c, lo) (TileA or RegA) and
// bd(c, lo): the A operand and the B descriptor of K step c, hi or lo part.  ACC: onto what d holds, else from 0.
template <int NP, int N, int KS, bool ACC = false, class A, class B, class U>
__device__ __forceinline__ void mma_batch(float (&d)[N / 2], const A& a, const B& bd, U&& under) {
  if (!ACC) {
#pragma unroll
    for (int j = 0; j < N / 2; ++j) d[j] = 0.f;
  }
  tc::wgmma_fence_operand(d);
  a.template pin<KS>();
  tc::wgmma_fence();
#pragma unroll
  for (int ps = 0; ps < NP; ++ps) {
#pragma unroll
    for (int c = 0; c < KS; ++c) wgmma<N>(d, a(c, ps == 1), bd(c, ps == 2));
  }
  tc::wgmma_commit();
  under();
  tc::wgmma_wait_all();
  tc::wgmma_fence_operand(d);
  a.template pin<KS>();
}

// ---- layers in the accumulator fragment of the warp group that issues them (the heads, the front and the chain) ----
// This thread holds columns 8j + 2q + {0, 1} of fragment rows fr and fr + 8 (q = t % 4, tc::acc_load_half):
// d[4j + 2r + e] is column 8j + 2q + e of row fr + 8r.
// An A fragment (tc::wgmma_tf32_ra) wants columns 8j + q and 8j + q + 4 of rows fr, fr + 8 instead.  frag_cols turns one
// row's pair of group j (x0, x1 = columns 8j + 2q, 8j + 2q + 1) into those two columns (c0 = 8j + q, c4 = 8j + q + 4):
// lane q of a quad reads lane s = 2 (q & 1) + (q >> 1) in the first shuffle and lane s ^ 2 in the second; a lane offers
// column 2q + (q >> 1) in the first and its other column in the second, and what arrives is column q and q + 4 (in that
// order for even q, swapped for odd q).
__device__ __forceinline__ void frag_cols(float x0, float x1, int lane, float& c0, float& c4) {
  const int q = lane & 3, s1 = (lane & ~3) | ((q & 1) << 1) | (q >> 1);
  const float r1 = __shfl_sync(0xffffffffu, q >> 1 ? x1 : x0, s1);
  const float r2 = __shfl_sync(0xffffffffu, q >> 1 ? x0 : x1, s1 ^ 2);
  c0 = q & 1 ? r2 : r1;
  c4 = q & 1 ? r1 : r2;
}
// An N = 32 fragment x (after its epilogue) -> the A fragments of the next layer's 4 K steps, split into hi / lo
// (ah[j], al[j], j < 4)
template <int NP, int KA>
__device__ __forceinline__ void frag_to_a(const float (&x)[16], int lane, uint32_t (&ah)[KA][4], uint32_t (&al)[KA][4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float c0, c4;
      frag_cols(x[4 * j + 2 * r], x[4 * j + 2 * r + 1], lane, c0, c4);
      split<NP>(c0, ah[j][r], al[j][r]);                               // column 8j + q of row fr + 8r
      split<NP>(c4, ah[j][2 + r], al[j][2 + r]);                       // column 8j + q + 4
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
// the same over one 8-column group: z[2r + e] is its column 2q + e of row fr + 8r
__device__ __forceinline__ void row_dot8(const float (&z)[4], const float* __restrict__ w, float bias, int lane, float (&s)[2]) {
  s[0] = s[1] = bias;
#pragma unroll
  for (int qs = 0; qs < 4; ++qs) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
#pragma unroll
      for (int r = 0; r < 2; ++r) s[r] = fmaf(w[2 * qs + e], __shfl_sync(0xffffffffu, z[2 * r + e], (lane & ~3) | qs), s[r]);
    }
  }
}

// One dist-decoder head (two K 32, N 32 layers and the (o0, o1) outputs) for the 64 rows whose MMAs this warp group
// issues, without leaving its registers and without meeting the other warp group: L0 reads A[0:32] from the tile (both
// warp groups wrote it before the barrier in front of the heads), its epilogue runs on the accumulator fragment, L1 takes
// A from registers, and the outputs go to xch slots XCH_HEAD + 2 hd + {0, 1}.  Releases the head's ring stage on its own.
template <int NP>
__device__ __forceinline__ void run_head(const Blk& b, Ring& ring, const float* __restrict__ hw, float* __restrict__ xo, int fr) {
  const int lane = b.row & 31, q = lane & 3;
  const uint32_t w = ring.wait(0).addr;
  float d[16];
  mma_batch<NP, 32, 4>(d, tile_a(b, 0, 64), tile_b(w, tcl::HEAD_L0), [] {});
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
  frag_to_a<NP>(d, lane, ah, al);
  float e[16];
  mma_batch<NP, 32, 4>(e, RegA<4, NP>{ah, al}, tile_b(w, tcl::HEAD_L1), [] {});
  ring.release(0);
  ring.advance(1);
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
// the chain, together with w1 in xch slot XCH_W1 (mrow and dd[0..3] are still in XCH_FRONT + 3 .. 7); every later layer takes
// A from registers.  vis_fc.1 and vis_fc2.1 are summed by the quad that holds a row, in column order (row_dot), so every
// value is bit-identical to a round trip through the row owners.  Leaves x2 (base_fc.2's output +
// the vis_fc residual) in tile columns [96,128), rgb_fc.0's pre-activations in [128,144) and vis2 in xch slot XCH_L2.
// Ring stages (each warp group waits and releases on its own): base_fc.2 (tcl::B1_L) | vis_fc.0 + vis_fc.2 (tcl::VIS0_L,
// VIS2_L) | vis_fc2.0 + rgb_fc.0 (tcl::V20_L, RGB0_L).
// tk: where the phase stamps after base_fc.2, vis_fc.0, vis_fc.2 and vis_fc2.0 go (nullptr: none).
template <int NP>
__device__ __forceinline__ void run_chain(const Blk& b, Ring& ring, const float* __restrict__ sw, float* __restrict__ xch, int fr, long long* tk) {
  const int lane = b.row & 31, q = lane & 3;
  // base_fc.2: K = 64 from the tile; the row scalars load under its MMAs
  uint32_t w = ring.wait(0).addr;
  float d[16];
  float w1[2], mr[2], t0[2], t1[2];                 // t0, t1: rgb_fc.0's K tail, columns 32 + q and 36 + q (t0 of lane 0 is vis2)
  mma_batch<NP, 32, 8>(d, tile_a(b, 0, 64), tile_b(w, tcl::B1_L), [&] {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float* __restrict__ x = xch + XCH_FRONT * 128 + fr + 8 * r;
      w1[r] = xch[XCH_W1 * 128 + fr + 8 * r];
      mr[r] = x[3 * 128];
      t0[r] = q == 0 ? 0.f : x[(3 + q) * 128];
      t1[r] = q == 0 ? x[7 * 128] : 0.f;
    }
  });
  ring.release(0);
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
  frag_to_a<NP>(xr, lane, ah, al);
  if (tk) tk[0] = clock64();
  // vis_fc.0 (row scale w1 in the epilogue)
  w = ring.wait(1).addr;
  mma_batch<NP, 32, 4>(d, RegA<4, NP>{ah, al}, tile_b(w, tcl::VIS0_L), [] {});
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 bb = *reinterpret_cast<const float2*>(sw + SW_V0B + 8 * j + 2 * q);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      d[4 * j + 2 * r] = elu(fmaf(w1[r], d[4 * j + 2 * r], bb.x));
      d[4 * j + 2 * r + 1] = elu(fmaf(w1[r], d[4 * j + 2 * r + 1], bb.y));
    }
  }
  frag_to_a<NP>(d, lane, ah, al);
  if (tk) tk[1] = clock64();
  // vis_fc.2, then vis_fc.1 (the vis_fc.0 outputs' dot product; under the MMAs, with their A registers pinned, it spills)
  float e[16];
  mma_batch<NP, 32, 4>(e, RegA<4, NP>{ah, al}, tile_b(w, tcl::VIS2_L), [] {});
  ring.release(1);
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
  frag_to_a<NP>(xr, lane, a2h, a2l);
  if (tk) tk[2] = clock64();
  // vis_fc2.0; x2 goes to the tile under its MMAs
  w = ring.wait(2).addr;
  mma_batch<NP, 32, 4>(d, RegA<5, NP>{a2h, a2l}, tile_b(w, tcl::V20_L), [&] { tc::acc_store_half<32>(b.act, 96, b.row, b.wg, xr); });
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
    split<NP>(q == 0 ? vis2[r] : t0[r], a2h[4][r], a2l[4][r]);
    split<NP>(t1[r], a2h[4][2 + r], a2l[4][2 + r]);
  }
  float g[8];
  mma_batch<NP, 16, 5>(g, RegA<5, NP>{a2h, a2l}, tile_b(w, tcl::RGB0_L), [&] {
    if (q < 2) xch[XCH_L2 * 128 + fr + 8 * q] = q ? vis2[1] : vis2[0];
  });
  ring.release(2);
  ring.advance(3);
  tc::acc_store_half<16>(b.act, 128, b.row, b.wg, g);
}

// x as a value the compiler cannot see through: what is computed from it is not hoisted out of a loop
__device__ __forceinline__ int opaque(int x) {
  int y;
  asm volatile("mov.b32 %0, %1;" : "=r"(y) : "r"(x));
  return y;
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
// the same columns of a row of activations -> hi parts from `hi`, lo parts from `lo` (NP = 3 only)
template <int NP, int Q>
__device__ __forceinline__ void st_own(const Blk& b, int hi, int lo, const float* v) {
#pragma unroll
  for (int q = 0; q < Q; ++q) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) split<NP>(v[4 * q + j], h[j], l[j]);
    *reinterpret_cast<uint4*>(b.act + own_index(b, hi + 8 * q)) = make_uint4(h[0], h[1], h[2], h[3]);
    if constexpr (NP == 3) *reinterpret_cast<uint4*>(b.act + own_index(b, lo + 8 * q)) = make_uint4(l[0], l[1], l[2], l[3]);
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

// The kernel body, NP passes per tensor-core product (point_kernel_pm3: 3, point_kernel_tf32: 1).  EXPORTS: the per-row
// weights it also stores into kp.rows, a compile-time set so that the kernels without an export are the same code as
// before it existed.  EXPORT_BLEND: warp group 1 stores each valid row's colour-blend weight into kp.rows[0]
// (point_kernel_blend).  EXPORT_AGG: warp group 1 also stores the row's pooling weights, the NeuRay weight w0 into
// kp.rows[1] and the geometry weight w2 into kp.rows[2] (point_kernel_agg, which carries EXPORT_BLEND as well); all at
// the end of the tile.  EXPORT_VIEW: the front's fragment lanes also store each valid row's masked hit probability into
// kp.rows[3] where they form it (point_kernel_view, which carries EXPORT_BLEND and EXPORT_AGG as well).
template <int G, bool DEBUG, int NP, int EXPORTS = 0>
__device__ __forceinline__ void point_body(const KParams& kp) {
  constexpr bool BLEND = (EXPORTS & EXPORT_BLEND) != 0, AGG = (EXPORTS & EXPORT_AGG) != 0, VIEW = (EXPORTS & EXPORT_VIEW) != 0;
  extern __shared__ __align__(1024) float smem[];
  constexpr bool P2 = (G & (G - 1)) == 0;      // power-of-two lane groups reduce with butterflies, the others through shared memory
  constexpr int PPW = 32 / G;                   // points per warp (G = 10: 3, two lanes idle)
  constexpr int PB = 4 * PPW;                   // points per block
  constexpr int GE = G >= 32 ? 32 : G >= 16 ? 16 : G >= 8 ? 8 : 4;   // lanes of a point that share geometry_fc's 64 hidden units
  constexpr int CPL = 64 / GE;                  // geometry_fc.0 output columns per such lane
  static_assert(G == 4 || G == 5 || G == 6 || G == 8 || G == 10 || G == 16 || G == 32, "lanes per point");
  const NrPassParams& pp = kp.p;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  float* const ring_smem = smem + OFF_RING;
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
        const uint32_t buf = Ring::slot_of(n);
        if (n >= NBUF) tc::mbar_wait(wempty + buf, Ring::parity(n - NBUF));   // both compute warp groups released stage n - NBUF
        load_stage(ring_smem + buf * RING_STAGE, pp.w_tc, table[s], wfull + buf);
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
  auto gsum = [&](float x) { if constexpr (P2) return warp_sum<G>(x); else return gsum_np2<G>(stg, lane, lane0, idle, x); };
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
  Ring ring{ring_smem, tc::smem_u32(ring_smem), wfull, wempty, 0, b.row == 0};
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
        if (ring.leader) ring.wait(s);
        ring.release(s);
      }
      ring.advance(stages_per_tile);
      continue;
    }
    const int n = tile * PB + pl;
    const bool pt_ok = P2 ? n < N : (n < N && !idle);
    const bool row_ok = pt_ok && v < rfn;

    PM_TICK(0)
    // ---------------- ray geometry of this row's point (every lane of the group, in both warp groups, computes the same values) ----------------
    PointGeo geo = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (pt_ok) geo = point_geometry(smem + OFF_CAM, pp.coords, pp.que_depth, dn, n);

    // ---------------- projection into this row's view + feature and rgb taps ----------------
    float mrow = 0.f, zrow = 1.f, dd[4] = {0.f, 0.f, 0.f, 0.f}, rgbin[3] = {0.f, 0.f, 0.f};
    float dbg_px = 0.f, dbg_py = 0.f, dbg_dir[3] = {0.f, 0.f, 0.f};
    int tcode = -1;
    float tw[4] = {0.f, 0.f, 0.f, 0.f};
    if (row_ok) {
      const Proj pj = project(smem + OFF_CAM + 32 + v * 20, geo.X, geo.Y, geo.Z, h, w);
      mrow = pj.valid ? 1.f : 0.f;
      zrow = pj.zh;
      const float ex = pj.dir[0], ey = pj.dir[1], ez = pj.dir[2];
      dd[0] = ex - geo.qx; dd[1] = ey - geo.qy; dd[2] = ez - geo.qz; dd[3] = ex * geo.qx + ey * geo.qy + ez * geo.qz;
      if (DEBUG) { dbg_px = pj.ux; dbg_py = pj.uy; dbg_dir[0] = ex; dbg_dir[1] = ey; dbg_dir[2] = ez; }
      if (pj.valid) {
        // feature-map taps of this row, worked out once here instead of by each of the gathering lanes
        const Taps ft = border_taps(pj.ux, pj.uy, h, w, fh, fw, feat_align);
        tcode = tap_code(ft, v, fh, fw);
        tw[0] = ft.w[0]; tw[1] = ft.w[1]; tw[2] = ft.w[2]; tw[3] = ft.w[3];
        rgb_tap(pp.rgb, v, pj.ux, pj.uy, h, w, rgbin);
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
      st_own<NP, 4>(b, 0, 64, x);
      if (DEBUG && kp.dbg != nullptr && row_ok) {
        float* __restrict__ o = kp.dbg + (size_t(v) * N + n) * 76;
        for (int k = 0; k < 16; ++k) o[12 + 8 * (k >> 2) + 4 * wg + (k & 3)] = x[k];
      }
    }
    gather16(32);                                                                  // img_feats: stay in the buffer until rgb_feat is built
    {
      // the row scalars of the front's fragment rows, read after the heads: zrow, ihp, ihc, mrow, dd[0..1] from warp
      // group 0, dd[2..3], rgbin[0..2] from warp group 1
      const float rs[11] = {zrow, geo.ihp, geo.ihc, mrow, dd[0], dd[1], dd[2], dd[3], rgbin[0], rgbin[1], rgbin[2]};
#pragma unroll
      for (int k = 0; k < 5; ++k) xch[(XCH_FRONT + 6 * wg + k) * 128 + row] = wg ? rs[6 + k] : rs[k];
      if (wg == 0) xch[(XCH_FRONT + 5) * 128 + row] = rs[5];
    }
    if (DEBUG && kp.dbg != nullptr && row_ok) {                                   // the row scalars and img_feats (hit, vis: in the front)
      float* __restrict__ o = kp.dbg + (size_t(v) * N + n) * 76;
      const float* __restrict__ mine = stg + lane * STG_ROW;
      for (int k = 0; k < 16; ++k) o[44 + 8 * (k >> 2) + 4 * wg + (k & 3)] = mine[k];
      if (wg == 0) {
        o[0] = mrow; o[1] = zrow; o[4] = dbg_px; o[5] = dbg_py;
        o[6] = dbg_dir[0]; o[7] = dbg_dir[1]; o[8] = dbg_dir[2]; o[9] = rgbin[0]; o[10] = rgbin[1]; o[11] = rgbin[2];
      }
    }
    PM_TICK(3)
    // the heads: each warp group runs them for the 64 rows whose MMAs it issues (run_head); A[0:32] comes from both
    tc::fence_proxy_async_smem();
    tc::named_sync(BAR_LAYER, NCOMP);
#pragma unroll 1
    for (int hd = 0; hd < n_heads; ++hd) run_head<NP>(b, ring, sw + SW_HEAD + hd * SW_HEAD_STRIDE, xch + (XCH_HEAD + 2 * hd) * 128, fr);
    PM_TICK(4)

    // ---------------- the front, hit/vis through base_fc.0: each warp group for its own 64 rows, in its accumulator fragment ----------------
    // Nothing in it pools across views, so it needs no barrier with the other warp group until its outputs go to the row
    // owners: every shared-memory write in it lands in this warp group's own rows (of the tile, RF_SLAB and xch), which
    // only it reads before the hand-off barrier.  Every accumulator gets the products and every row sum the order the row owners gave them, so every value
    // is bit-identical to a round trip through them.  Ring stages (each warp group waits and releases on its own):
    // prob_embed.0 (tcl::PE0_L) | prob_embed.2 + neuray_fc.0 (tcl::PE1_L) | base_fc.0 x3 (tcl::B0_L); ray_dir_fc.2 is resident.
    {
      // fr_f, lane_f: fr and the lane as values the compiler cannot see through.  The front's per-thread addresses are
      // then worked out here in every tile instead of being hoisted out of the tile loop and held in registers across the
      // chain (which made the DEBUG instantiations spill).  In the comments below, fr stands for fr_f.
      const int fr_f = opaque(fr), lane_f = opaque(lane);
      const int q = lane_f & 3;
      const float* __restrict__ xf = xch + XCH_FRONT * 128;                       // xf[k * 128 + r]: row scalar k of row r
      // hit and visibility of row fr + 8 (q >> 1) (lanes q and q ^ 1 both compute it) from its heads' outputs
      float hv01;                                                                  // hit' (even q) or vis' (odd q)
      {
        const int rr = fr_f + 8 * (q >> 1);
        __syncwarp();                                                              // run_head: this warp's lanes wrote rows fr, fr + 8
        float hv[4][2];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          hv[k][0] = k < n_heads ? xch[(XCH_HEAD + 2 * k) * 128 + rr] : 0.f;
          hv[k][1] = k < n_heads ? xch[(XCH_HEAD + 2 * k + 1) * 128 + rr] : 0.f;
        }
        // (point, view) of row rr, as the row owners get theirs
        const int l = rr & 31, g = l / G;
        const int rv = P2 ? l % G : l - g * G;
        const float* vp = smem + OFF_CAM + 32 + (rv < rfn ? rv : 0) * 20;
        const float zc = fmaxf(xf[rr], 1e-5f);
        const float a = vp[15], bb = vp[16];
        const float tz = (-1.f / zc - a) / (bb - a);
        const float lo = tz - xf[128 + rr], hi = tz + xf[2 * 128 + rr];
        const float aw = sigmoidf_(hv[2][0]);
        const float vd = pp.use_vis ? sigmoidf_(hv[3][0]) : 1.f;
        float hit = 0.f, visib = 0.f;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float mean = softplusf_(hv[0][i]);
          const float var = softplusf_(hv[1][i]) + pp.var_bias;
          const float c0 = logistic_cdf((lo - mean) * var) * vd, c1 = logistic_cdf((hi - mean) * var) * vd;
          const float mix = i == 0 ? aw : 1.f - aw;
          visib = fmaf(1.f - c0, mix, visib);
          hit = fmaf(c1 - c0, mix, hit);
        }
        const float mr = xf[3 * 128 + rr];
        visib *= mr; hit *= mr;
        if (DEBUG && kp.dbg != nullptr && (q & 1) == 0) {
          const int rn_ = n - pl + (P2 ? rr / G : (rr >> 5) * PPW + g);            // n - pl: the block's first point
          if ((P2 ? rn_ < N : (rn_ < N && g < PPW)) && rv < rfn) {
            float* __restrict__ o = kp.dbg + (size_t(rv) * N + rn_) * 76;
            o[2] = hit; o[3] = visib;
          }
        }
        // the masked hit probability of row rr (nr_render_pass_fwd_view): the reference's prj_dict['hit_prob']
        // (renderer.py:75-82); the even lane of the pair stores it, once per valid (view, point) row
        if constexpr (VIEW) {
          if ((q & 1) == 0) {
            const int rn_ = n - pl + (P2 ? rr / G : (rr >> 5) * PPW + g);
            if ((P2 ? rn_ < N : (rn_ < N && g < PPW)) && rv < rfn) kp.rows[size_t(3 * rfn + rv) * N + rn_] = hit;
          }
        }
        hv01 = q & 1 ? (visib - 0.5f) * 2.f : (hit - 0.5f) * 2.f;
      }
      // prob_embed.0's K step 4 of rows fr, fr + 8 (columns 32, 33 = hit', vis', the rest 0) -> this warp group's rows of
      // the tile (the heads' hidden layer is dead); lanes 0 and 1 have their row fr values, lanes 2 and 3 the row fr + 8 ones
      {
        const float other = __shfl_xor_sync(0xffffffffu, hv01, 2);
        uint32_t* const at = reinterpret_cast<uint32_t*>(b.act);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          uint32_t h, l;
          split<NP>(q < 2 ? (r ? other : hv01) : 0.f, h, l);
          const int rr = fr_f + 8 * r;
          at[tc::act_index(rr, 32 + q)] = h;
          at[tc::act_index(rr, 36 + q)] = 0u;
          if constexpr (NP == 3) {
            at[tc::act_index(rr, 96 + q)] = l;
            at[tc::act_index(rr, 100 + q)] = 0u;
          }
        }
      }
      tc::fence_proxy_async_smem();
      tc::named_sync(BAR_WG + wg, 128);
      // prob_embed.0: K = 32 + 8 (ray_feats, hit' and vis'), A from the tile; ReLU, then into prob_embed.2's A layout
      uint32_t ah[4][4], al[4][4];
      {
        float d[16];
        mma_batch<NP, 32, 5>(d, tile_a(b, 0, 64), tile_b(ring.wait(0).addr, tcl::PE0_L), [] {});
        ring.release(0);
        ring.advance(1);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 bb = *reinterpret_cast<const float2*>(sw + SW_PE0B + 8 * j + 2 * q);
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            d[4 * j + 2 * r] = fmaxf(d[4 * j + 2 * r] + bb.x, 0.f);
            d[4 * j + 2 * r + 1] = fmaxf(d[4 * j + 2 * r + 1] + bb.y, 0.f);
          }
        }
        frag_to_a<NP>(d, lane_f, ah, al);
      }
      PM_TICK(5)
      // prob_embed.2 with neuray_fc.0 behind it (N = 48): neuray_feat = columns [0,32) + bias, the gate from columns [32,40)
      float gate[2];
      {
        float d[24];
        mma_batch<NP, 48, 4>(d, RegA<4, NP>{ah, al}, tile_b(ring.wait(0).addr, tcl::PE1_L), [] {});
        ring.release(0);
        ring.advance(1);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 bb = *reinterpret_cast<const float2*>(sw + SW_PE1B + 8 * j + 2 * q);
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            d[4 * j + 2 * r] += bb.x;
            d[4 * j + 2 * r + 1] += bb.y;
          }
        }
        // neuray_fc.0's ELU in the lane that holds the column, neuray_fc.1 over the quad in column order
        float y[4];
        const float2 c = *reinterpret_cast<const float2*>(sw + SW_NF0C + 2 * q);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          y[2 * r] = elu(d[16 + 2 * r] + c.x);
          y[2 * r + 1] = elu(d[16 + 2 * r + 1] + c.y);
        }
        row_dot8(y, sw + SW_NF1W, sw[SW_NF1B], lane_f, gate);
        float nf[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) nf[j] = d[j];
        frag_to_a<NP>(nf, lane_f, ah, al);
      }
      // base_fc.0, K round A: the neuray_feat inputs (its K steps 5..8).  Waits for all three of its stages, which round B
      // reads too.  Under its MMAs: the gate goes to the row owners' slot, and ray_dir_fc.0 (K 4, N 16) runs on the CUDA
      // cores straight into ray_dir_fc.2's A fragments (column u = hidden unit u)
      ring.wait(0);
      ring.wait(1);
      ring.wait(2);
      float acc[32];
      uint32_t rh[2][4], rl[2][4];
      mma_batch<NP, 64, 4>(acc, RegA<4, NP>{ah, al}, base0_b(ring, 5), [&] {
        if (q < 2) xch[XCH_GATE * 128 + fr_f + 8 * q] = q ? gate[1] : gate[0];
        const float* __restrict__ w0 = sw + SW_RD0W;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int rr = fr_f + 8 * r;
          const float d0 = xf[4 * 128 + rr], d1 = xf[5 * 128 + rr], d2 = xf[6 * 128 + rr], d3 = xf[7 * 128 + rr];
#pragma unroll
          for (int s = 0; s < 2; ++s) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int u = 8 * s + 4 * h + q;
              const float x = elu(fmaf(w0[48 + u], d3, fmaf(w0[32 + u], d2, fmaf(w0[16 + u], d1, fmaf(w0[u], d0, sw[SW_RD0B + u])))));
              split<NP>(x, rh[s][2 * h + r], rl[s][2 * h + r]);
            }
          }
        }
      });
      // ray_dir_fc.2: K = 16, N = 48 (35 used)
      float e[24];
      mma_batch<NP, 48, 2>(e, RegA<2, NP>{rh, rl}, tile_b(tc::smem_u32(smem + OFF_RD1), tcl::RD1_L), [] {});
      // rgb_feat (35) + the constant 1 (column 35: base_fc.0's bias) + zero padding, in round B's A fragments.  Column c < 35
      // is elu(ray_dir_fc.2 + bias) + rgbin[c] (c < 3) or img_feats channel c - 3, which warp group ((c - 3) >> 2) & 1
      // gathered into its buffer column 4 ((c - 3) >> 3) + ((c - 3) & 3), row rr at lane rr & 31 of its warp rr >> 5.
      // Columns < 35 also go to the row owners in fp32 for pooling #1: [0,32) to tile slab 2 (RF_SLAB), [32,35) to xch.
      // Of K step s, column 8s + 4h + q: img_feats channel 8s + 4h + q - 3 of row fr is at im[h] + 4s (h = 0: own buffer
      // for q = 3, the other's column 4 (s - 1) + q + 1 for q < 3; h = 1: own buffer column 4s + q + 1 for q < 3, the
      // other's column 4s for q = 3); row fr + 8 is 8 buffer rows further.
      uint32_t bh[5][4], bl[5][4];
      {
        const float* __restrict__ img0 = smem + OFF_STG + ((fr_f >> 5) * 32 + (fr_f & 31)) * STG_ROW;
        const float* __restrict__ img1 = img0 + 4 * 32 * STG_ROW;
        const float* __restrict__ im[2] = {q == 3 ? img0 : img1 + q - 3, q < 3 ? img0 + q + 1 : img1};
        float* __restrict__ rfo = b.act + RF_SLAB + rf_slab_index(fr_f, q);          // column 8s + 4h + q of row fr + 8r: rfo[(2s + h) * 256 + 32r]
#pragma unroll
        for (int r = 0; r < 2; ++r) {
#pragma unroll
          for (int s = 0; s < 5; ++s) {
            float x[2];
            frag_cols(e[4 * s + 2 * r], e[4 * s + 2 * r + 1], lane_f, x[0], x[1]);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int c = 8 * s + 4 * h + q;
              float f = c == 35 ? 1.f : 0.f;
              if (c < 35) {
                f = elu(x[h] + sw[SW_RD1B + c]);
                if (c < 3) f += xf[(8 + q) * 128 + fr_f + 8 * r];
                else f += im[h][4 * s + 8 * r * STG_ROW];
                if (s < 4) rfo[(2 * s + h) * 256 + 32 * r] = f;
                else xch[(XCH_RF + q) * 128 + fr_f + 8 * r] = f;
              }
              split<NP>(f, bh[s][2 * h + r], bl[s][2 * h + r]);
            }
          }
        }
      }
      // base_fc.0, K round B: rgb_feat (its K steps 0..4), onto round A's accumulators
      mma_batch<NP, 64, 5, true>(acc, RegA<5, NP>{bh, bl}, base0_b(ring, 0), [] {});
#pragma unroll
      for (int s = 0; s < 3; ++s) ring.release(s);
      ring.advance(3);
      tc::acc_store_half<64>(b.act, 96, b.row, b.wg, acc);
    }
    // Hand-off to the row owners.  Live in the tile: base_fc.0's per-view accumulator (bias included) in columns [96,160)
    // and rgb_feat columns 0..31 in fp32 in slab 2 (columns [64,96), RF_SLAB); [0,64) is dead (pooling #1's per-point
    // operand goes there).  In xch: the gate and rgb_feat columns 32..34.
    tc::named_sync(BAR_LAYER, NCOMP);
    // rgb_feat: rf[4q + i] = column 8q + 4wg + i (columns 35.. are the constant and padding, which pool to 0)
    float rf[20];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float4 t = *reinterpret_cast<const float4*>(b.act + RF_SLAB + rf_slab_index(row, 8 * k + 4 * wg));
      rf[4 * k] = t.x; rf[4 * k + 1] = t.y; rf[4 * k + 2] = t.z; rf[4 * k + 3] = t.w;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) rf[16 + i] = wg == 0 && i < 3 ? xch[(XCH_RF + i) * 128 + row] : 0.f;
    const float gate = xch[XCH_GATE * 128 + row];

    PM_TICK(6)
    // ---------------- view pooling #1 (ibrnet.py:336-339) -> the view-pooled part of base_fc.0, once per point ----------------
    // Every lane of a point ends a round with the point's statistics: 8 features x (mean0, var0, mean1, var1) = K 32 per
    // round (statistic t of feature i at column 32 R + 8t + i, so warp group c pools features 4c .. 4c + 3 of the round).
    // They go into the point's row of the per-point operand (PB rows, K 160) and each round's K 32 is multiplied as soon
    // as it is complete, B from the round's ring stage, into a per-point [PB][64] result that the epilogue adds to every
    // view's row.  One barrier per round: it publishes the round's operand columns and tells the leaders (Ring::leader) that every
    // warp is done with the previous round's stage (the fifth stage can only load into the first one's ring slot).  The sums over
    // the views go through the warp's transposition buffer (pool_rows); the variance comes from the weighted second moment:
    //   sum_v w (x - mu)^2 = sum_v w x^2 - mu^2 (2 - sum_v w),  mu = sum_v w x   (the reference's mean is NOT normalised)
    const float msum = gsum(mrow);
    const float w1 = mrow / (msum + 1e-8f);
    const float w0 = sigmoidf_(gate) * w1;
    {
      const float c1 = 2.f - gsum(w1), c0 = 2.f - gsum(w0);
      float* const op = b.act;
      PtAcc<PB, NP> acc = {};
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
        if (R > 0) ring.release(R - 1);
        point_mma<PB, 4, NP>(acc, op, 32 * R, ring.wait(R).p, tcl::HST_STAGE, warp, lane);
      };
      round(std::integral_constant<int, 0>{}); round(std::integral_constant<int, 1>{}); round(std::integral_constant<int, 2>{});
      round(std::integral_constant<int, 3>{}); round(std::integral_constant<int, 4>{});
      point_store(acc, smem + OFF_PT, warp, lane);
      tc::named_sync(BAR_LAYER, NCOMP);                                            // per-point result visible; the last stage read
      ring.release(4);
      ring.advance(5);
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
      st_own<NP, 4>(b, c0, 64 + c0, x);                                                // lo half 1 lands on accumulator columns already consumed
    }
    if (wg == 0) xch[XCH_W1 * 128 + row] = w1;                                     // w1 of the chain's fragment rows
    PM_TICK(8)
    // ---------------- base_fc.2, vis_fc, vis_fc2, rgb_fc.0: each warp group for its own 64 rows (run_chain) ----------------
    tc::fence_proxy_async_smem();
    tc::named_sync(BAR_LAYER, NCOMP);
    {
      long long* tk = nullptr;                                                     // phase stamps 9 .. 12 inside the chain
      if constexpr (DEBUG) {
        if (kp.timing != nullptr && blockIdx.x == 0 && row == 0 && it < 64) tk = kp.timing + (it * 2 + wg) * 32 + 9;
      }
      run_chain<NP>(b, ring, sw, xch, fr, tk);
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
      PtAcc<PB, NP> acc = {};
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const float* w = ring.wait(s).p;
        if (s < 2) point_mma<PB, 4, NP>(acc, op, 32 * s, w, tcl::G0_L, warp, lane);
        else point_mma<PB, 1, NP>(acc, op, 64, w, tcl::G0_L, warp, lane);
      }
      point_store(acc, smem + OFF_PT, warp, lane);
      tc::named_sync(BAR_LAYER, NCOMP);                                            // per-point result visible; the stages read
#pragma unroll
      for (int s = 0; s < 3; ++s) ring.release(s);
      ring.advance(3);
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
      const float* __restrict__ rgbin_x = xch + (XCH_FRONT + 8) * 128 + row;       // this row's rgbin, as the front read it
      float acc[4] = {e, e * rgbin_x[0], e * rgbin_x[128], e * rgbin_x[256]};
      if constexpr (P2) bsum_vec<G, 4>(acc); else gsum4_np2<G>(stg, lane, lane0, idle, acc);
      if (v == 0 && pt_ok) {
        float4* __restrict__ dst = reinterpret_cast<float4*>(pp.point_rec + size_t(n) * REC);
        dst[4] = make_float4(acc[1] / acc[0], acc[2] / acc[0], acc[3] / acc[0], msum);
      }
      // the blend weight of this (view, point) row (nr_render_pass_fwd_blend): the reference's blending_weights_valid
      if constexpr (BLEND) {
        if (row_ok) kp.rows[size_t(v) * N + n] = e / acc[0];
      }
      // the pooling weights of this row (nr_render_pass_fwd_agg): the reference's weight0 (ibrnet.py:334-337) and its
      // weight from vis (ibrnet.py:349-350).  Both warp groups hold them; stored here, off the pooling rounds' barriers.
      if constexpr (AGG) {
        if (row_ok) {
          kp.rows[size_t(rfn + v) * N + n] = w0;
          kp.rows[size_t(2 * rfn + v) * N + n] = w2;
        }
      }
    }
    PM_TICK(15)
  }
#undef PM_TICK
}

template <int G, bool DEBUG>
__global__ void __launch_bounds__(NTHR, 1) point_kernel_pm3(const KParams kp) { point_body<G, DEBUG, 3>(kp); }
// TF32 mode (release form only): one tensor-core pass per product, operands rounded to nearest, B from a pack with
// rna(W) in the hi slots (nr_pack_weights_tf32)
template <int G>
__global__ void __launch_bounds__(NTHR, 1) point_kernel_tf32(const KParams kp) { point_body<G, false, 1>(kp); }
// Either release form (NP = 3: 3xTF32, 1: TF32 mode) with the colour-blend export (kp.rows [rfn][rn*dn])
template <int G, int NP>
__global__ void __launch_bounds__(NTHR, 1) point_kernel_blend(const KParams kp) { point_body<G, false, NP, EXPORT_BLEND>(kp); }
// Either release form with the colour-blend and the pooling-weight exports (kp.rows [3][rfn][rn*dn]: blend, w0, w2)
template <int G, int NP>
__global__ void __launch_bounds__(NTHR, 1) point_kernel_agg(const KParams kp) { point_body<G, false, NP, EXPORT_BLEND | EXPORT_AGG>(kp); }
// Either release form with those exports and the masked hit probability (kp.rows [4][rfn][rn*dn]: blend, w0, w2, hit)
template <int G, int NP>
__global__ void __launch_bounds__(NTHR, 1) point_kernel_view(const KParams kp) {
  point_body<G, false, NP, EXPORT_BLEND | EXPORT_AGG | EXPORT_VIEW>(kp);
}

}  // namespace pm3
