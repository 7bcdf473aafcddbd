// bdiff_selftest.cu — hardware self test of the split-bf16 wgmma machinery used by the layer megakernel:
//   * A operand: 128B-swizzled K-major bf16 blocks, hi and lo blocks written by threads (x_store8_hl);
//   * B operand: un-swizzled K=16 slabs [2 chunks][N rows][16 B] (hi plane, lo plane) fetched by TMA bulk copies
//     and addressed with the SWIZZLE_NONE descriptor (gmma_desc_k16);
//   * three products per K step (A_hi.W_hi + A_lo.W_hi + A_hi.W_lo), N = 128 | 128 | 32 | 32 (the last one negated),
//     each of the two warpgroups on its 64 rows;
//   * variant bit 1: the node-tile "R5" layout (32 distinct rows stored as hi, lo, hi, lo, hi in 160-row blocks;
//     two row views 0 / +32 and four products leave the complete sum in every row quarter);
//   * the accumulator scratch: fragment stores, and a round trip between the two threads that share a row (the pair
//     exchange of the edge tile).
// tests/test_gpu_tc.py compares C with an fp64 matmul at 3e-5 relative before the fused kernel is trusted.
#include "bdiff_kernels.h"
#include "bdiff_tc.cuh"
#include "bdiff_slab.cuh"

namespace bdiff {

constexpr int ST_K = 128, ST_N = 320, ST_STEPS = ST_K / 16;
constexpr int ST_SLAB = ST_N * 32;                       // bytes of one plane of one K step
constexpr size_t ST_SMEM = 4 * (size_t)X_BLOCK + (size_t)ST_STEPS * 2 * ST_SLAB + 64 + 1024;
constexpr size_t ST_IMG = (size_t)ST_STEPS * 2 * ST_SLAB;   // packed weights, followed by the accumulator scratch

__global__ void k_selftest_pack_slabs(const float* __restrict__ W, unsigned char* __restrict__ img) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= ST_N * ST_K) return;
  const int n = idx / ST_K, k = idx - n * ST_K;
  slab_store(img + (size_t)(k >> 4) * 2 * ST_SLAB, ST_N, n, k & 15, W[idx]);
}

// columns [n0, n0 + N) of A . W^T (SA = -1: negated) for this warpgroup's 64 rows -> accumulator scratch
template <int N, int SA>
__device__ __forceinline__ void selftest_gemm(uint32_t xa, uint32_t wb, bool r5, int n0) {
  float d[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  wgmma_fence();
  for (int ks = 0; ks < ST_STEPS; ++ks) {
    const uint32_t bh = wb + (uint32_t)ks * 2 * ST_SLAB + n0 * 16, bl = bh + ST_SLAB;
    const int j = ks >> 2, s = ks & 3;
    uint64_t a0, a1;
    if (!r5) {
      a0 = gmma_desc_sw128(xa + j * X_BLOCK + s * 32);            // A_hi
      a1 = gmma_desc_sw128(xa + (2 + j) * X_BLOCK + s * 32);      // A_lo
    } else {
      a0 = gmma_desc_sw128(xa + j * R5_BLOCK + s * 32);           // view 0:  hi lo hi lo
      a1 = gmma_desc_sw128(xa + j * R5_BLOCK + 4096 + s * 32);    // view 32: lo hi lo hi
    }
    const uint64_t dh = gmma_desc_k16(bh, ST_N * 16, 128), dl = gmma_desc_k16(bl, ST_N * 16, 128);
    // products: edge layout (A_hi,W_hi) (A_lo,W_hi) (A_hi,W_lo);  R5: (v0,W_hi) (v32,W_hi) (v0,W_lo) (v32,W_lo)
    if (N == 128) {
      wgmma_n128<SA>(d, a0, dh); wgmma_n128<SA>(d, a1, dh); wgmma_n128<SA>(d, a0, dl);
      if (r5) wgmma_n128<SA>(d, a1, dl);
    } else {
      wgmma_n32<SA>(d, a0, dh); wgmma_n32<SA>(d, a1, dh); wgmma_n32<SA>(d, a0, dl);
      if (r5) wgmma_n32<SA>(d, a1, dl);
    }
  }
  wgmma_commit();
  wgmma_wait<0>();
  acc_fence<N / 2>(d);
  acc_store<N>(d, n0, threadIdx.x >> 7);
}

__global__ void __launch_bounds__(320, 1) k_wgmma_selftest_split(const float* __restrict__ A,
                                                                 const unsigned char* __restrict__ wimg,
                                                                 float* __restrict__ scratch, float* __restrict__ C,
                                                                 int variant) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* X = smem;                           // edge layout: hi blocks 0,1 | lo blocks 2,3;  R5 layout: 2 blocks x 20 KiB
  unsigned char* Wb = smem + 4 * X_BLOCK;
  uint64_t* bars = reinterpret_cast<uint64_t*>(Wb + (size_t)ST_STEPS * 2 * ST_SLAB);
  const int tid = threadIdx.x;
  const bool r5 = variant & 2;
  if (tid == 0) {
    mbar_init(&bars[0], 1);
    mbar_fence_init();
    acc_scratch = scratch;
  }
  __syncthreads();
  if (tid < 128) {
    if (!r5) {
      for (int k8 = 0; k8 < ST_K / 8; ++k8) {
        float v[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) v[q] = A[(size_t)tid * ST_K + k8 * 8 + q];
        x_store8_hl(X, 2, tid, k8 * 8, v);
      }
    } else if (tid < 32) {
      for (int k8 = 0; k8 < ST_K / 8; ++k8) {
        float v[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) v[q] = A[(size_t)tid * ST_K + k8 * 8 + q];
        x_store8_r5(X, tid, k8 * 8, v);
      }
    }
    fence_proxy_async();
  }
  if (tid == 256) {
    mbar_expect_tx(&bars[0], ST_STEPS * 2 * ST_SLAB);
    for (int s = 0; s < ST_STEPS * 2; ++s) bulk_g2s(Wb + (size_t)s * ST_SLAB, wimg + (size_t)s * ST_SLAB, ST_SLAB, &bars[0]);
  }
  __syncthreads();
  if (tid < 256) {
    mbar_wait(&bars[0], 0);
    const uint32_t xa = smem_u32(X) + (uint32_t)(tid >> 7) * 8192u, wb = smem_u32(Wb);
    selftest_gemm<128, 1>(xa, wb, r5, 0);
    selftest_gemm<128, 1>(xa, wb, r5, 128);
    selftest_gemm<32, 1>(xa, wb, r5, 256);
    selftest_gemm<32, -1>(xa, wb, r5, 288);
    named_bar_sync(3, 256);
    const int half = tid >> 7, r = tid & 127;
    // pair exchange through the scratch: each half writes 8 values into its own columns, reads the partner's
    float mine[8], theirs[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) mine[i] = (float)(1000 * half + r * 8 + i);
    scratch_st<8>(320 + half * 8, mine);
    named_bar_sync(3, 256);
    scratch_ld<8>(320 + (half ^ 1) * 8, theirs);
    for (int c0 = half * 160; c0 < half * 160 + 160; c0 += 32) {
      float v[32];
      scratch_ld<32>(c0, v);
#pragma unroll
      for (int i = 0; i < 32; ++i) C[(size_t)r * 336 + c0 + i] = v[i];
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) C[(size_t)r * 336 + 320 + half * 8 + i] = theirs[i];
  }
}


cudaError_t selftest_configure() {
  return cudaFuncSetAttribute(k_wgmma_selftest_split, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ST_SMEM);
}

void launch_wgmma_selftest_split(cudaStream_t st, const float* A, const float* W, unsigned char* img_scratch, float* C,
                                int variant) {
  k_selftest_pack_slabs<<<(ST_N * ST_K + 255) / 256, 256, 0, st>>>(W, img_scratch);
  k_wgmma_selftest_split<<<1, 320, ST_SMEM, st>>>(A, img_scratch, reinterpret_cast<float*>(img_scratch + ST_IMG), C, variant);
}

size_t selftest_img_bytes() { return ST_IMG + (size_t)TM_COLS * 128 * sizeof(float); }

}  // namespace bdiff
