// bdiff_tc.cuh — wgmma / shared-memory-descriptor helpers and the accumulator scratch of the tensor-core path (sm_90a).
//
// Conventions used by every wgmma operand in this library (bf16, K-major):
//   A: an operand "K-block" is [rows][64 bf16] = rows x 128 B, 1024-byte aligned, 128-byte swizzle; element (r, k) lives at
//       r*128 + (((k >> 3) ^ (r & 7)) << 4) + (k & 7)*2            (the TMA SWIZZLE_128B pattern)
//     the descriptor points at the block (plus 32 B per K=16 step, plus r0*128 for a row offset that is a multiple of 8),
//     SBO = 1024 B (8 rows), layout SWIZZLE_128B.  A warpgroup's M=64 rows start 64*128 = 8 KiB further on.
//   B: un-swizzled K=16 slabs (see bdiff_slab.cuh), descriptor with explicit LBO / SBO.
//   Accumulators: registers of the issuing warpgroup, stored at the end of a GEMM phase to a per-CTA scratch of 128 rows
//   x 512 columns (column-major) that the epilogue threads read by row (scratch_ld / scratch_st).
//   Elementwise epilogues instead run on the registers themselves (frag_row / frag_col give each register's place).
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

#include "bdiff_common.cuh"

namespace bdiff {

__device__ __forceinline__ uint32_t sw128_offset(int r, int k) {   // byte offset inside a K-block
  return (uint32_t)(r * 128 + ((((k >> 3) ^ (r & 7)) & 7) << 4) + (k & 7) * 2);
}

// 64-bit wgmma shared-memory descriptor for a K-major SWIZZLE_128B operand at byte address `saddr`.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);          // start address  [0,14)
  d |= (uint64_t)1 << 16;                          // leading byte offset [16,30): unused for a swizzled K-major operand
  d |= (uint64_t)((1024 >> 4) & 0x3FFF) << 32;     // stride byte offset  [32,46): 8 rows * 128 B
  d |= (uint64_t)1 << 62;                          // layout type [62,64): SWIZZLE_128B
  return d;
}

// 64-bit wgmma descriptor for a K-major operand WITHOUT swizzle: core matrices of 8 rows x 16 bytes are contiguous
// (128 B); consecutive 8-row groups are `sbo` bytes apart, the two 16-byte K chunks of one K=16 step `lbo` bytes apart.
__device__ __forceinline__ uint64_t gmma_desc_k16(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo >> 4) & 0x3FFF) << 32;
  return d;
}

// D[64 x N] += (SA * A[64 x 16]) . B[N x 16]^T, bf16 operands from shared memory, fp32 accumulators in registers
// (fragment of thread t of the warpgroup: see acc_store).  SA = -1 negates the product.
template <int SA>
__device__ __forceinline__ void wgmma_n128(float* d, uint64_t ad, uint64_t bd) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, %67, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(ad), "l"(bd), "r"(1), "n"(SA));
}

template <int SA>
__device__ __forceinline__ void wgmma_n32(float* d, uint64_t ad, uint64_t bd) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, %19, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(ad), "l"(bd), "r"(1), "n"(SA));
}

template <int SA>
__device__ __forceinline__ void wgmma_n16(float* d, uint64_t ad, uint64_t bd) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, %11, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(ad), "l"(bd), "r"(1), "n"(SA));
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma
template <int R>
__device__ __forceinline__ void acc_fence(float* d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrive by the threads with `pred` set, as a predicated instruction rather than a branch (no divergent path between wgmmas)
__device__ __forceinline__ void mbar_arrive_if(uint64_t* bar, bool pred) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %1, 0;\n@p mbarrier.arrive.shared::cta.b64 _, [%0];\n}\n" ::"r"(smem_u32(bar)),
               "r"((int)pred) : "memory");
}

// ------------------------------------------------------------------------------------------ accumulator scratch
// Base of this CTA's [512 columns][128 rows] fp32 scratch; set by the kernel before its first barrier.
__shared__ float* acc_scratch;
// wgmma fragment of an M=64 x N tile issued by warpgroup wg: register j of this thread holds the element at row
// frag_row(wg, j) of the 128-row tile and column frag_col(j) of the tile's N columns.  Registers j and j + 1 (j even)
// are two adjacent columns of one row.
__device__ __forceinline__ int frag_row(int wg, int j) {
  return 64 * wg + 16 * ((threadIdx.x >> 5) & 3) + ((threadIdx.x & 31) >> 2) + 8 * ((j >> 1) & 1);
}
__device__ __forceinline__ int frag_col(int j) { return 8 * (j >> 2) + 2 * (threadIdx.x & 3) + (j & 1); }
// fragment (columns col0 ..) <-> scratch
template <int N>
__device__ __forceinline__ void acc_store(const float* d, int col0, int wg) {
  float* const base = acc_scratch;     // one read of the pointer (a store through float* could alias it)
#pragma unroll
  for (int j = 0; j < N / 2; ++j) base[(size_t)(col0 + frag_col(j)) * 128 + frag_row(wg, j)] = d[j];
}
template <int N>
__device__ __forceinline__ void acc_load(float* d, int col0, int wg) {
  const float* const base = acc_scratch;
#pragma unroll
  for (int j = 0; j < N / 2; ++j) d[j] = base[(size_t)(col0 + frag_col(j)) * 128 + frag_row(wg, j)];
}

// This thread's row of the scratch: row 32 * (warp % 4) + lane, columns col .. col + N - 1.  Nothing here orders the
// accesses of different threads: that is the job of the CTA barriers around them.
__device__ __forceinline__ float* scratch_row() { return acc_scratch + (threadIdx.x & 127); }
template <int N>
__device__ __forceinline__ void scratch_ld(int col, float* v) {
  const float* p = scratch_row() + (size_t)col * 128;
#pragma unroll
  for (int i = 0; i < N; ++i) v[i] = p[i * 128];
}
template <int N>
__device__ __forceinline__ void scratch_st(int col, const float* v) {
  float* p = scratch_row() + (size_t)col * 128;
#pragma unroll
  for (int i = 0; i < N; ++i) p[i * 128] = v[i];
}

// Two-lane fp32 arithmetic, one instruction per lane.  The names are those of the toolkit's packed fp32x2 intrinsics,
// which exist for device code from sm_100 on only (the host pass sees the toolkit's declarations); sm_90 device code gets
// these definitions.
#if defined(__CUDA_ARCH__) && __CUDA_ARCH__ < 1000
__device__ __forceinline__ float2 __fmul2_rn(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
__device__ __forceinline__ float2 __fadd2_rn(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 __ffma2_rn(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
#endif

// ------------------------------------------------------------------------------------- split-bf16 operands
// Every GEMM operand of the tensor path is the pair (hi, lo) of bf16 numbers with hi = RN_bf16(value)
// and lo = RN_bf16(value - hi): hi + lo carries >= 16 significant bits (relative error
// <= 2^-18) and is exactly representable in fp32.  A product is evaluated as A_hi.W_hi + A_lo.W_hi + A_hi.W_lo
// (three wgmma products accumulating into the same fp32 registers; the dropped A_lo.W_lo term is 2^-18 relative).
__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  hi = *reinterpret_cast<uint32_t*>(&h);
  const float ra = a - __uint_as_float(hi << 16), rb = b - __uint_as_float(hi & 0xffff0000u);
  __nv_bfloat162 l = __floats2bfloat162_rn(ra, rb);
  lo = *reinterpret_cast<uint32_t*>(&l);
}
__device__ __forceinline__ float2 join_bf16x2(uint32_t hi, uint32_t lo) {
  return make_float2(__uint_as_float(hi << 16) + __uint_as_float(lo << 16),
                     __uint_as_float(hi & 0xffff0000u) + __uint_as_float(lo & 0xffff0000u));
}
__device__ __forceinline__ void split_bf16(float a, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(a);
  lo = __float2bfloat16_rn(a - __bfloat162float(hi));
}

// fp32-class activations for the tensor path: ex2.approx / rcp.approx are accurate to ~2 ulp.
// sigmoid(x) = 1 / (1 + 2^(-x log2 e)).
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float sigmoid_acc(float x) { return rcp_approx(1.0f + ex2_approx(-1.4426950408889634f * x)); }
__device__ __forceinline__ float silu_acc(float x) { return x * sigmoid_acc(x); }
__device__ __forceinline__ float2 sigmoid_acc2(float2 x) {
  const float2 t = __fmul2_rn(x, make_float2(-1.4426950408889634f, -1.4426950408889634f));
  const float2 d = __fadd2_rn(make_float2(ex2_approx(t.x), ex2_approx(t.y)), make_float2(1.0f, 1.0f));
  return make_float2(rcp_approx(d.x), rcp_approx(d.y));
}
__device__ __forceinline__ float2 silu_acc2(float2 x) { return __fmul2_rn(x, sigmoid_acc2(x)); }

// A-operand tile: 128 rows x 64 bf16 per K-block (16 KiB), K-blocks consecutive.
constexpr int X_BLOCK = 128 * 128;

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

}  // namespace bdiff
