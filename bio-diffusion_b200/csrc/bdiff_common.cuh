// bdiff_common.cuh — shared definitions for libbdiff_sm90.so (sm_90a only).
//
// Layout conventions (all fp32 unless noted):
//   node tensors  h [N,256], chi [N,32*3] (channel-major, xyz-minor == ScalarVector.flatten order,
//                 reference components/__init__.py:702-710), x [N,3]
//   edge tensors  e [E,Ed], xi [E,Xd*3], frames [E,9] rows (d, c, d x c); edges are the implicit
//                 (row, col)-sorted block-diagonal list of gcpnet.py:1054-1066 — never materialised
//   weights       K-major: W[k][o] = torch_weight[o][k]; big matrices have leading dim 256
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bdiff {

constexpr int kThreads = 256;
constexpr int kH = 256;       // node scalar hidden dim (model_cfg.h_hidden_dim)
constexpr int kC = 32;        // node vector hidden channels (model_cfg.chi_hidden_dim)
constexpr int kMsg = kH + 3 * kC;   // 352: flattened message / aggregate width
constexpr int kHidM = 8;      // hidden vector dim of G1..G3 / POS: 32 / bottleneck 4
constexpr int kHidFF = 16;    // hidden vector dim of the feed-forward GCP: 64 / 4
constexpr int kKM = 280;      // padded fan-in of G1..G3 / POS scalar_out: 256 + 8 + 9 = 273 -> 280
constexpr int kKFF = 540;     // padded fan-in of FF scalar_out.0: 512 + 16 + 9 = 537 -> 540
constexpr int TM_COLS = 512;  // columns of the per-CTA accumulator scratch of the tensor path (bdiff_tc.cuh)
constexpr int kPStride = 328; // per-node projection record: 256 + hid0*3 (<=60) + 9 -> 328
constexpr int kKC = 16;       // K rows of a weight chunk staged in shared memory (16 x 256 x 4 B = 16 KiB)

// Topology plan (device arrays), built once per (batch_index, mask) by bdiff_plan_topology (host part: bdiff_plan.h).
struct Plan {
  int B;                 // molecules
  int N;                 // nodes (masked ones included)
  long long E;           // edges = sum nact^2
  const int* mol_off;    // [B+1] node offsets
  const int* act_off;    // [B+1] offsets into act_idx
  const int* act_idx;    // [M]   global ids of unmasked nodes, ascending
  const long long* edge_off;  // [B+1] prefix of nact^2
  const int* node_mol;   // [N]   molecule of each node
  const unsigned char* mask;  // [N]
  const int4* edge_rc;   // [128*ceil(E/128)] per edge {row, col, b, nact} (row = -1 past E): b = position in the row segment
  const int2* node_mid;  // [32*ceil(N/32)] per node {first, count} of the 128-edge tiles that lie strictly inside its row (count > 0 only for n >= 130)
};

// Per-layer packed weights (device pointers, K-major).
struct LayerW {
  // message GCP 0 in split form: S0 = [e | vn | q] W0e + (h_row Wsi + b0) + (h_col Wsj)
  const float *W0e, *Wsi, *Wsj, *b0;
  const float *Wd0i, *Wd0x, *Wd0j;   // [32][hid0], [Xd][hid0], [32][hid0]
  const float *Wf0i, *Wf0x, *Wf0j;   // [32][3], [Xd][3], [32][3]
  const float *Wu0, *Wg0, *bg0;      // [hid0][32], [256][32], [32]
  // message GCPs 1..3
  const float *Wk[3], *bk[3], *Wdk[3], *Wfk[3], *Wuk[3], *Wgk[3], *bgk[3];
  const float *wa, *ba;              // scalar message attention [256], [1]
  // feed-forward GCP
  const float *W1, *b1, *W2, *b2, *Wdf, *Wff, *Wuf, *Wgf, *bgf;
  // node position update GCP
  const float *Wp, *bp, *Wdp, *Wfp, *Wup, *Wgp, *bgp;
};

struct EmbedW {
  // edge embedding GCP (1,1)->(Ed,Xd): Ws [Ke][Ed], wd [Xd], wf [3], Wu [Xd][Xd], Wg [Ed][Xd]
  const float *eWs, *ebs, *ewd, *ewf, *eWu, *eWg, *ebg;
  // node embedding GCP (Hin,2)->(256,32): Ws [Kn][256], Wd [2][32], Wf [2][3], Wu [32][32], Wg [256][32]
  const float *nWs, *nbs, *nWd, *nWf, *nWu, *nWg, *nbg;
  // projection GCP (256,32)->(Hin,0): Ws [300][Hin], Wd [32][32], Wf [32][3]
  const float *pWs, *pbs, *pWd, *pWf;
};

struct Dims {
  int F;       // node scalar features in xh
  int C;       // context columns
  int Hin;     // F + 1 + C
  int Ed, Xd;  // edge hidden dims
  int hid0;    // (2*32 + Xd) / 4
  int K0;      // padded fan-in of the edge part of G0: Ed + hid0 + 9 -> multiple of 4
  int Ke;      // padded fan-in of the edge embedding: 1 + Xd + 9 -> multiple of 4
  int Kn;      // padded fan-in of the node embedding: Hin + 32 + 9 -> multiple of 4
  int L;
};

// ------------------------------------------------------------------------------------------ math
// parity-mode activations: full-precision expf (the reference uses torch's fp32 sigmoid / silu)
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float siluf_(float x) { return x / (1.0f + expf(-x)); }
// safe_norm of the reference (components/__init__.py:276-286): sqrt(sum + 1e-8) + 1e-8
__device__ __forceinline__ float safe_norm3(float a, float b, float c) {
  return sqrtf(a * a + b * b + c * c + 1e-8f) + 1e-8f;
}

// --------------------------------------------------------------------------- mbarrier + bulk copy
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// for the single helper threads (TMA producer, MMA issuer): mbarrier.try_wait already suspends the warp in hardware
// and wakes ~60 cycles after the arrive, so no software back-off (a __nanosleep here only adds hand-off latency)
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// TMA bulk copy global -> shared (SASS: UBLKCP), completion signalled on an mbarrier.
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// Double-buffered weight streamer state: two 16 KiB buffers + two mbarriers; parity bits persist
// across calls (each barrier completes one phase per chunk it receives).
struct WStream {
  float* buf;        // [2][kKC*256]
  uint64_t* bar;     // [2]
  uint32_t parity;   // bit i = parity to wait for on bar[i]
};

// acc[RT][4] += A[r][0..Kpad) . W[0..Kpad)[c..c+3]   for rows r = ty*RT + i, cols c = tx*4
//   A: shared memory, row stride lda (multiple of 4 floats, 16 B aligned rows), Kpad multiple of 4
//   W: global, K-major [Kpad][256]; streamed through shared memory in kKC-row chunks by TMA bulk copies
// All kThreads threads must call this together.  Thread layout: tx = tid % 64, ty = tid / 64 (warp-uniform).
template <int RT>
__device__ __forceinline__ void gemm256(const float* __restrict__ sA, int lda, int Kpad,
                                        const float* __restrict__ gW, WStream& ws, float (&acc)[RT][4]) {
  const int tid = threadIdx.x;
  const int tx = tid & 63, ty = tid >> 6;
  const int nchunks = (Kpad + kKC - 1) / kKC;
  // prologue: fill both buffers
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      if (s < nchunks) {
        int rows = min(kKC, Kpad - s * kKC);
        uint32_t bytes = rows * 256 * 4;
        mbar_expect_tx(&ws.bar[s], bytes);
        bulk_g2s(ws.buf + s * kKC * 256, gW + (size_t)s * kKC * 256, bytes, &ws.bar[s]);
      }
    }
  }
  const float* arow = sA + (ty * RT) * lda;
  for (int ch = 0; ch < nchunks; ++ch) {
    const int s = ch & 1;
    mbar_wait(&ws.bar[s], (ws.parity >> s) & 1u);
    ws.parity ^= (1u << s);
    const float* wb = ws.buf + s * kKC * 256 + tx * 4;
    const int k0 = ch * kKC;
    const int rows = min(kKC, Kpad - k0);
    for (int kk = 0; kk < rows; kk += 4) {
      float4 a[RT];
#pragma unroll
      for (int i = 0; i < RT; ++i) a[i] = *reinterpret_cast<const float4*>(arow + i * lda + k0 + kk);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float4 w = *reinterpret_cast<const float4*>(wb + (kk + j) * 256);
#pragma unroll
        for (int i = 0; i < RT; ++i) {
          const float av = j == 0 ? a[i].x : (j == 1 ? a[i].y : (j == 2 ? a[i].z : a[i].w));
          acc[i][0] = fmaf(av, w.x, acc[i][0]);
          acc[i][1] = fmaf(av, w.y, acc[i][1]);
          acc[i][2] = fmaf(av, w.z, acc[i][2]);
          acc[i][3] = fmaf(av, w.w, acc[i][3]);
        }
      }
    }
    __syncthreads();   // everyone is done with buffer s
    if (tid == 0 && ch + 2 < nchunks) {
      int rows2 = min(kKC, Kpad - (ch + 2) * kKC);
      uint32_t bytes = rows2 * 256 * 4;
      mbar_expect_tx(&ws.bar[s], bytes);
      bulk_g2s(ws.buf + s * kKC * 256, gW + (size_t)(ch + 2) * kKC * 256, bytes, &ws.bar[s]);
    }
  }
}

// out[r][o] = f( sum_k A[r][k] W[k][o] + b[o] )  for r < TM, o < NO (NO <= 64), K multiple of 4.
//   A shared (lda), W global K-major [K][NO] (read through L1), out shared (ldo).  act: 0 none, 1 silu, 2 sigmoid
template <int TM>
__device__ __forceinline__ void small_linear(const float* __restrict__ sA, int lda, int K,
                                             const float* __restrict__ W, const float* __restrict__ b, int NO,
                                             float* __restrict__ sOut, int ldo, int act) {
  for (int idx = threadIdx.x; idx < TM * NO; idx += kThreads) {
    const int r = idx / NO, o = idx - r * NO;
    const float* a = sA + r * lda;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    for (int k = 0; k < K; k += 4) {
      const float4 av = *reinterpret_cast<const float4*>(a + k);
      s0 = fmaf(av.x, __ldg(W + (k + 0) * NO + o), s0);
      s1 = fmaf(av.y, __ldg(W + (k + 1) * NO + o), s1);
      s2 = fmaf(av.z, __ldg(W + (k + 2) * NO + o), s2);
      s3 = fmaf(av.w, __ldg(W + (k + 3) * NO + o), s3);
    }
    float v = (s0 + s1) + (s2 + s3) + (b ? __ldg(b + o) : 0.f);
    if (act == 1) v = siluf_(v);
    else if (act == 2) v = sigmoidf_(v);
    sOut[r * ldo + o] = v;
  }
}

// out[r] = f( sum_k A[r][k] w[k] + b ) with one warp per row (lanes stride k, butterfly reduce).
template <int TM>
__device__ __forceinline__ void row_dot(const float* __restrict__ sA, int lda, int K, const float* __restrict__ w,
                                        float b, float* __restrict__ sOut, int act) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < TM; r += kThreads / 32) {
    float s = 0.f;
    for (int k = lane; k < K; k += 32) s = fmaf(sA[r * lda + k], __ldg(w + k), s);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
    if (lane == 0) {
      float v = s + b;
      if (act == 2) v = sigmoidf_(v);
      sOut[r] = v;
    }
  }
}

// out[r][h*3+x] (=|+=) sum_{c<nch} W[c*hid + h] * V[r][(c)*3 + x]      (vector_down / vector_down_frames)
template <int TM>
__device__ __forceinline__ void vec_down(float* __restrict__ out, int ldo, const float* __restrict__ V, int ldv,
                                         int nch, const float* __restrict__ W, int hid, bool accumulate) {
  const int per = hid * 3;
  for (int idx = threadIdx.x; idx < TM * per; idx += kThreads) {
    const int r = idx / per, hx = idx - r * per;
    const int h = hx / 3, x = hx - h * 3;
    const float* v = V + r * ldv + x;
    float s = 0.f;
    for (int c = 0; c < nch; ++c) s = fmaf(__ldg(W + c * hid + h), v[c * 3], s);
    if (accumulate) out[r * ldo + hx] += s;
    else out[r * ldo + hx] = s;
  }
}

// dst[r][hid_off + h] = safe_norm_xyz(VD[r][h][:]);  dst[r][hid_off + hid + ch*3 + a] = sum_x F[r][a*3+x] VDF[r][ch*3+x];
// then zero-fill dst[r][hid_off + hid + 9 .. kend).          (gcpnet.py:445-459, components/__init__.py:175-219)
template <int TM>
__device__ __forceinline__ void norms_and_q(float* __restrict__ dst, int ldd, int hid_off, int kend,
                                            const float* __restrict__ VD, int ldvd, int hid,
                                            const float* __restrict__ VDF, int ldvdf, const float* __restrict__ Fr,
                                            int ldf) {
  const int per = kend - hid_off;
  for (int idx = threadIdx.x; idx < TM * per; idx += kThreads) {
    const int r = idx / per, j = idx - r * per;
    float v = 0.f;
    if (j < hid) {
      const float* p = VD + r * ldvd + j * 3;
      v = safe_norm3(p[0], p[1], p[2]);
    } else if (j < hid + 9) {
      const int ch = (j - hid) / 3, a = (j - hid) - ch * 3;
      const float* f = Fr + r * ldf + a * 3;
      const float* p = VDF + r * ldvdf + ch * 3;
      v = f[0] * p[0] + f[1] * p[1] + f[2] * p[2];
    }
    dst[r * ldd + hid_off + j] = v;
  }
}

// Vout[r][o*3+x] = (accumulate ? Vout : 0) + (sum_{h<hid} Wu[h*vout + o] * VD[r][h*3+x]) * gate[r][o]
template <int TM>
__device__ __forceinline__ void vec_up_gate(float* __restrict__ Vout, int ldv, const float* __restrict__ VD,
                                            int ldvd, int hid, const float* __restrict__ Wu, int vout,
                                            const float* __restrict__ gate, int ldg, bool accumulate) {
  const int per = vout * 3;
  for (int idx = threadIdx.x; idx < TM * per; idx += kThreads) {
    const int r = idx / per, ox = idx - r * per;
    const int o = ox / 3, x = ox - o * 3;
    const float* vd = VD + r * ldvd + x;
    float s = 0.f;
    for (int h = 0; h < hid; ++h) s = fmaf(__ldg(Wu + h * vout + o), vd[h * 3], s);
    s *= gate[r * ldg + o];
    if (accumulate) Vout[r * ldv + ox] += s;
    else Vout[r * ldv + ox] = s;
  }
}

// Edge id -> (molecule, local row a, local col b) by binary search over the per-molecule edge offsets.
__device__ __forceinline__ int find_mol(const long long* __restrict__ edge_off, int B, long long g) {
  int lo = 0, hi = B;   // invariant: edge_off[lo] <= g < edge_off[hi]
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (__ldg(edge_off + mid) <= g) lo = mid;
    else hi = mid;
  }
  return lo;
}

}  // namespace bdiff
