// bdiff_slab.cuh — split-bf16 (hi, lo) operand layouts of the tensor path.
//
// A operand (activations, written by the compute warps): K-major 128B-swizzled bf16 blocks as in bdiff_tc.cuh, one
// set of blocks for the hi parts and one for the lo parts.
//   edge tile  : 9 blocks of [128 rows][64]: hi of columns 0..255 in blocks 0..3, lo in blocks 4..7; block 8 holds the
//                32 "extra" columns [vector norms | scalarised frames]: hi at k 0..31, lo at k 32..63.
//   node tile  : 5 blocks of [160 rows][64] ("R5"): node l of the 32-node tile is stored as hi in rows l, l+64, l+128
//                and as lo in rows l+32, l+96.  The MMA reads the block through two 128-row views (row 0: hi lo hi lo,
//                row 32: lo hi lo hi); view0.W_hi + view32.W_hi + view0.W_lo + view32.W_lo leaves the complete
//                (hi+lo)(W_hi+W_lo) product in all four row quarters of the accumulator, so the 8 compute warps share the 32
//                nodes: each reads its accumulator columns from its own row quarter.
// B operand (weights, packed once per weight update): "slabs" of one K=16 step:
//                [hi plane | lo plane], plane = [2 K-chunks][N rows][16 bytes], un-swizzled (SWIZZLE_NONE, LBO = N*16,
//                SBO = 128).  A slab plane is one contiguous TMA bulk copy of N*32 bytes (<= 10 KiB for N = 320), which
//                lets the weight ring work in 10 KiB slots.
#pragma once
#include "bdiff_tc.cuh"

namespace bdiff {

// element (row n, k in [0,16)) of a K-step slab whose planes have N rows; writes the hi and the lo plane
__device__ __forceinline__ void slab_store(unsigned char* slab, int N, int n, int kk, float v) {
  __nv_bfloat16 hi, lo;
  split_bf16(v, hi, lo);
  unsigned char* p = slab + (size_t)(kk >> 3) * N * 16 + (size_t)n * 16 + (kk & 7) * 2;
  *reinterpret_cast<__nv_bfloat16*>(p) = hi;
  *reinterpret_cast<__nv_bfloat16*>(p + (size_t)N * 32) = lo;
}

// ---- generic [128 rows] hi/lo blocks: hi block (kk>>6), lo block lo0 + (kk>>6)
__device__ __forceinline__ void x_store8_hl(unsigned char* X, int lo0, int r, int kk, const float* v) {   // kk % 8 == 0
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) split_bf16x2(v[2 * i], v[2 * i + 1], h[i], l[i]);
  const uint32_t off = sw128_offset(r, kk & 63);
  *reinterpret_cast<uint4*>(X + (kk >> 6) * X_BLOCK + off) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(X + (lo0 + (kk >> 6)) * X_BLOCK + off) = make_uint4(l[0], l[1], l[2], l[3]);
}

// ---- edge tile (9 blocks)
constexpr int XE_LO = 4, XE_EXTRA = 8, XE_BLOCKS = 9;
__device__ __forceinline__ void xe_store4(unsigned char* X, int r, int kk, float a, float b, float c, float d) {   // kk % 4 == 0
  uint32_t h0, l0, h1, l1;
  split_bf16x2(a, b, h0, l0);
  split_bf16x2(c, d, h1, l1);
  const uint32_t off = sw128_offset(r, kk & 63);
  *reinterpret_cast<uint2*>(X + (kk >> 6) * X_BLOCK + off) = make_uint2(h0, h1);
  *reinterpret_cast<uint2*>(X + (XE_LO + (kk >> 6)) * X_BLOCK + off) = make_uint2(l0, l1);
}
__device__ __forceinline__ void xe_store1(unsigned char* X, int r, int kk, float v) {   // kk < 256
  __nv_bfloat16 hi, lo;
  split_bf16(v, hi, lo);
  const uint32_t off = sw128_offset(r, kk & 63);
  *reinterpret_cast<__nv_bfloat16*>(X + (kk >> 6) * X_BLOCK + off) = hi;
  *reinterpret_cast<__nv_bfloat16*>(X + (XE_LO + (kk >> 6)) * X_BLOCK + off) = lo;
}
// extra block: column c in [0,32): hi at k = c, lo at k = 32 + c
__device__ __forceinline__ void xe_store8_extra(unsigned char* X, int r, int c, const float* v) {   // c % 8 == 0
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) split_bf16x2(v[2 * i], v[2 * i + 1], h[i], l[i]);
  unsigned char* B8 = X + XE_EXTRA * X_BLOCK;
  *reinterpret_cast<uint4*>(B8 + sw128_offset(r, c)) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(B8 + sw128_offset(r, 32 + c)) = make_uint4(l[0], l[1], l[2], l[3]);
}

// ---- node tile "R5" (5 blocks of 160 rows)
constexpr int R5_ROWS = 160;
constexpr int R5_BLOCK = R5_ROWS * 128;      // 20 KiB
constexpr int R5_BLOCKS = 5;
__device__ __forceinline__ void x_store8_r5(unsigned char* X, int l, int kk, const float* v) {   // kk % 8 == 0
  uint32_t h[4], lo[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) split_bf16x2(v[2 * i], v[2 * i + 1], h[i], lo[i]);
  const uint4 uh = make_uint4(h[0], h[1], h[2], h[3]), ul = make_uint4(lo[0], lo[1], lo[2], lo[3]);
  unsigned char* q = X + (kk >> 6) * R5_BLOCK + sw128_offset(l, kk & 63);      // rows l + 32 i keep the swizzle phase
  *reinterpret_cast<uint4*>(q) = uh;
  *reinterpret_cast<uint4*>(q + 4096) = ul;
  *reinterpret_cast<uint4*>(q + 8192) = uh;
  *reinterpret_cast<uint4*>(q + 12288) = ul;
  *reinterpret_cast<uint4*>(q + 16384) = uh;
}
__device__ __forceinline__ void x_store4_r5(unsigned char* X, int l, int kk, float a, float b, float c, float d) {   // kk % 4 == 0
  uint32_t h0, l0, h1, l1;
  split_bf16x2(a, b, h0, l0);
  split_bf16x2(c, d, h1, l1);
  const uint2 uh = make_uint2(h0, h1), ul = make_uint2(l0, l1);
  unsigned char* q = X + (kk >> 6) * R5_BLOCK + sw128_offset(l, kk & 63);
  *reinterpret_cast<uint2*>(q) = uh;
  *reinterpret_cast<uint2*>(q + 4096) = ul;
  *reinterpret_cast<uint2*>(q + 8192) = uh;
  *reinterpret_cast<uint2*>(q + 12288) = ul;
  *reinterpret_cast<uint2*>(q + 16384) = uh;
}
__device__ __forceinline__ void x_store1_r5(unsigned char* X, int l, int kk, float v) {
  __nv_bfloat16 hi, lo;
  split_bf16(v, hi, lo);
  unsigned char* q = X + (kk >> 6) * R5_BLOCK + sw128_offset(l, kk & 63);
  *reinterpret_cast<__nv_bfloat16*>(q) = hi;
  *reinterpret_cast<__nv_bfloat16*>(q + 4096) = lo;
  *reinterpret_cast<__nv_bfloat16*>(q + 8192) = hi;
  *reinterpret_cast<__nv_bfloat16*>(q + 12288) = lo;
  *reinterpret_cast<__nv_bfloat16*>(q + 16384) = hi;
}

}  // namespace bdiff
