// wgmma / TMA / mbarrier primitives for the tensor-core MLP layers (sm_90a).
//
// Layer shape used throughout:  D[128 x N] (fp32) += A[128 x K] (tf32, smem) * B[N x K]^T (tf32, smem), issued as one
// m64nNk8 wgmma per K = 8 step for each row half (rows 0..63 and 64..127): by two warp groups, one half each (point
// kernel), or both halves by one warp group (self-test)
//   * A lives in a per-block shared-memory activation tile: row r = the row thread r of the warp group owns, one fp32 column
//     per k, 32-column slabs of 128 rows in the K-major SWIZZLE_128B layout (act_index).  A thread writes and reads its own
//     row with 128-bit accesses, which are conflict-free in that layout.  The accumulator of a layer is written back into
//     columns of the same tile, so the row owners read their outputs the way they read their inputs.
//   * B lives in shared memory, K-major, 128-byte swizzle: row n = 32 consecutive k (128 B), 8-row atoms of
//     1024 B; a K = 8 step advances the descriptor start address by 32 B inside the atom
//   * fp32 accuracy comes from the 3xTF32 split: x = hi + lo with hi = x & 0xffffe000 (exactly representable in
//     tf32, so it does not matter whether the tensor core truncates or rounds), lo = x - hi (exact);
//     D = A_hi*B_hi + A_lo*B_hi + A_hi*B_lo
//   * the point kernel's TF32 mode issues only the first of these passes, on operands rounded to nearest (tf32_rna)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nr {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// generic-proxy shared-memory writes -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }

// ---- mbarrier ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// bounded spin: a protocol bug traps instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  for (uint32_t it = 0; !mbar_try_wait(bar, parity); ++it)
    if (it > (1u << 26)) __trap();
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// TMA 1-D bulk copy global -> shared, completion counted in bytes on `bar` (size and addresses multiples of 16)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// named barrier among `count` threads (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_sync(int id, int count) { asm volatile("bar.sync %0, %1;\n" ::"r"(id), "r"(count) : "memory"); }

// per-thread register budget of the executing warp group (all of its warps execute it): give registers back to the CTA's
// pool / take them from it
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(R)); }
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(R)); }

// ---- descriptors ----
// shared-memory matrix descriptor, K-major, SWIZZLE_128B, 8-row atoms 1024 B apart (sm_90 GMMA descriptor)
__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= uint64_t((saddr & 0x3ffff) >> 4);          // start address, bits [0,14)
  d |= uint64_t(1) << 16;                         // leading byte offset (unused for swizzled K-major), bits [16,30)
  d |= uint64_t(1024 >> 4) << 32;                 // stride byte offset = 1024 B between 8-row atoms, bits [32,46)
  d |= uint64_t(1) << 62;                         // layout type SWIZZLE_128B, bits [62,64)
  return d;
}

// float index inside a K-major SWIZZLE_128B tile of 32-wide fp32 rows: element (row n, k in [0,32))
__host__ __device__ constexpr int sw128_index(int n, int k) { return (n >> 3) * 256 + (n & 7) * 32 + ((((k >> 2) ^ (n & 7)) << 2) | (k & 3)); }

// ---- the activation tile: 128 rows, 32-column slabs of 4096 floats (16 KB, 1024-byte aligned) ----
__host__ __device__ constexpr int act_index(int r, int c) { return (c >> 5) * 4096 + sw128_index(r, c & 31); }
// A operand of the K = 8 step that starts at column `col` (a multiple of 8), rows 64 * half .. 64 * half + 63
__device__ __forceinline__ uint64_t act_desc(uint32_t act_saddr, int col, int half) {
  return smem_desc_sw128(act_saddr + uint32_t((col >> 5) * 16384 + half * 8192 + (col & 31) * 4));
}

// ---- wgmma (one warp group) ----
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory"); }
// Operand fence on an accumulator fragment: every register of `d` is defined before this point and read after it.  Put
// before wgmma_fence() and after the wait that completes the batch.  Without it the compiler may sink the moves that
// build the accumulators (zeroing, acc_load_half) past wgmma_fence(), in between the wgmmas; ptxas then injects a
// warpgroup.arrive there and serialises every wgmma of the function (C7520: each one issued alone and waited for).
template <int M>
__device__ __forceinline__ void wgmma_fence_operand(float (&d)[M]) {
#pragma unroll
  for (int i = 0; i < M; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// the same for the A fragments of register-A wgmmas (wgmma_tf32_ra): they must stay put until the batch has completed.
// R > 0: only rows [0, R) of `a`, the K steps a batch reads.
template <int R = 0, int M, int K>
__device__ __forceinline__ void wgmma_fence_operand(uint32_t (&a)[M][K]) {
  static_assert(R <= M, "rows");
#pragma unroll
  for (int i = 0; i < (R > 0 ? R : M); ++i)
#pragma unroll
    for (int k = 0; k < K; ++k) asm volatile("" : "+r"(a[i][k])::"memory");
}

// d[N/2] (this thread's part of a 64 x N fp32 accumulator) += A[64 x 8] * B[N x 8]^T, both operands in shared memory
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], uint64_t a, uint64_t b);

#define NR_WGMMA_D8(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
template <>
__device__ __forceinline__ void wgmma_tf32<16>(float (&d)[8], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1;\n}\n"
      : NR_WGMMA_D8(0)
      : "l"(a), "l"(b), "r"(1)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<32>(float (&d)[16], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1;\n}\n"
      : NR_WGMMA_D8(0), NR_WGMMA_D8(8)
      : "l"(a), "l"(b), "r"(1)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<48>(float (&d)[24], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p, 1, 1;\n}\n"
      : NR_WGMMA_D8(0), NR_WGMMA_D8(8), NR_WGMMA_D8(16)
      : "l"(a), "l"(b), "r"(1)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32<64>(float (&d)[32], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
      "%32, %33, p, 1, 1;\n}\n"
      : NR_WGMMA_D8(0), NR_WGMMA_D8(8), NR_WGMMA_D8(16), NR_WGMMA_D8(24)
      : "l"(a), "l"(b), "r"(1)
      : "memory");
}
// d[N/2] += A[64 x 8] * B[N x 8]^T with A in registers: the mma.sync m16n8k8 A layout within each warp's 16 rows
// (rows 16 (t / 32) .. + 15 of the warp group's 64; with g = (t % 32) / 4, q = t % 4: a = A(g, q), A(g + 8, q),
// A(g, q + 4), A(g + 8, q + 4)), B in shared memory
template <int N>
__device__ __forceinline__ void wgmma_tf32_ra(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b);
template <>
__device__ __forceinline__ void wgmma_tf32_ra<16>(float (&d)[8], const uint32_t (&a)[4], uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %13, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1;\n}\n"
      : NR_WGMMA_D8(0)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32_ra<32>(float (&d)[16], const uint32_t (&a)[4], uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1;\n}\n"
      : NR_WGMMA_D8(0), NR_WGMMA_D8(8)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32_ra<48>(float (&d)[24], const uint32_t (&a)[4], uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %29, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, {%24,%25,%26,%27}, %28, p, 1, 1;\n}\n"
      : NR_WGMMA_D8(0), NR_WGMMA_D8(8), NR_WGMMA_D8(16)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_tf32_ra<64>(float (&d)[32], const uint32_t (&a)[4], uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
      "{%32,%33,%34,%35}, %36, p, 1, 1;\n}\n"
      : NR_WGMMA_D8(0), NR_WGMMA_D8(8), NR_WGMMA_D8(16), NR_WGMMA_D8(24)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1)
      : "memory");
}
#undef NR_WGMMA_D8

// The accumulator fragment of thread t of the warp group that issued the rows 64 * half .. 64 * half + 63 <-> the
// activation tile: for 8-column group j, d[4j + {0,1}] = (row 64 half + 16 (t / 32) + (t % 32) / 4, columns
// dcol + 8j + 2 (t % 4) + {0,1}), d[4j + {2,3}] = 8 rows lower.
template <int N>
__device__ __forceinline__ void acc_load_half(const float* act, int dcol, int t, int half, float (&d)[N / 2]) {
  const int r = 64 * half + 16 * (t >> 5) + ((t & 31) >> 2);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const int c = dcol + 8 * j + 2 * (t & 3);
    const float2 x = *reinterpret_cast<const float2*>(act + act_index(r, c));
    const float2 y = *reinterpret_cast<const float2*>(act + act_index(r + 8, c));
    d[4 * j] = x.x; d[4 * j + 1] = x.y; d[4 * j + 2] = y.x; d[4 * j + 3] = y.y;
  }
}
template <int N>
__device__ __forceinline__ void acc_store_half(float* act, int dcol, int t, int half, const float (&d)[N / 2]) {
  const int r = 64 * half + 16 * (t >> 5) + ((t & 31) >> 2);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const int c = dcol + 8 * j + 2 * (t & 3);
    *reinterpret_cast<float2*>(act + act_index(r, c)) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(act + act_index(r + 8, c)) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}
// both row halves issued by one warp group: d[h] is the fragment of half h
template <int N>
__device__ __forceinline__ void acc_store(float* act, int dcol, int t, const float (&d)[2][N / 2]) {
  acc_store_half<N>(act, dcol, t, 0, d[0]);
  acc_store_half<N>(act, dcol, t, 1, d[1]);
}

// 3xTF32 split
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(x) & 0xffffe000u;
  lo = __float_as_uint(x - __uint_as_float(hi));
}
// one-pass TF32 operand: x rounded to the nearest tf32 value (ties away from zero; the low 13 bits come out zero).  A
// truncated operand would bias every product of a K-long sum the same way.
__device__ __forceinline__ uint32_t tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(x));
  return r;
}

// ---- mma.sync (one warp) ----
// d (16x8, fp32) += A (16x8, tf32, row) * B (8x8, tf32, col).  With g = lane / 4, t = lane % 4: a = A(g, t), A(g + 8, t),
// A(g, t + 4), A(g + 8, t + 4); b = B(k t, n g), B(k t + 4, n g); d = D(g, 2t), D(g, 2t + 1), D(g + 8, 2t), D(g + 8, 2t + 1)
__device__ __forceinline__ void mma_tf32_m16n8k8(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

}  // namespace tc
}  // namespace nr
