// bdiff_classifier.cu — the EGNN property classifier of EDM (reference: src/__init__.py:233-419, E_GCL / E_GCL_mask /
// EGNN), inference only, on packed molecules (real atoms only, no n_max padding).  Padding does not couple molecules in
// the reference (every pair with a padded atom is masked), so the packed forward differs from it only in the order of
// the fp32 sums.
//
// Per layer l (E_GCL_mask.forward, :352-360; coordinates never move, coord_mlp is deleted):
//   edge kernel  m_ij = silu(W2 a_ij + b2) * sigmoid(w_att . m + b_att) * [i != j],  a_ij = silu(P_i + Q_j + w_r |x_i - x_j|^2)
//                with P = W1[:, :H] h + b1 and Q = W1[:, H:2H] h computed once per node (the edge_mlp.0 split);
//                agg_i = sum_j m_ij, a deterministic segmented row sum.
//   node kernel  h_i += W4 silu(W3 [h_i | agg_i (| h0_i)] + b3) + b4, then P / Q of layer l + 1 (or node_dec after the last
//                layer); readout kernel: pred_k = graph_dec(sum_{i in k} node_dec(h_i)) (:410-419).
//
// The edge kernel's K = 128 product a . W2^T runs on wgmma with split-bf16 operands (bdiff_tc.cuh): three products per
// K step, fp32 accumulation.  The node-level GEMMs (~20 % of the FLOPs at QM9 sizes, M = the few thousand atoms of a
// batch) are fp32 FFMA: exact fp32 products, and a 32-node tile reads each weight once from L2.
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <map>
#include <string>
#include <vector>

#include "../../include/bdiff.h"
#include "bdiff_slab.cuh"

namespace bdiff {

constexpr int CH = 128;               // hidden_nf
constexpr int CIN = 5;                // in_node_nf: the QM9 one-hot (H, C, N, O, F)
constexpr int CT = 128;               // edges per tile
constexpr int CLF_MAX_ATOMS = 128;    // a row of pairs is then cut by at most one tile border
constexpr int K3_MAX = 2 * CH + 8;    // node_mlp.0 fan-in 2H (+ 5 with node_attr), padded to a multiple of 4
constexpr int W2_STEP = 2 * CH * 32;  // one K = 16 slab of W2: [hi plane | lo plane] of 128 rows (bdiff_slab.cuh)
constexpr int W2_BYTES = (CH / 16) * W2_STEP;       // 64 KiB
constexpr int A_BYTES = 4 * X_BLOCK;                // a_ij: hi in blocks 0-1, lo in blocks 2-3 (64 KiB)
constexpr int EDGE_THREADS = 256;                   // two warpgroups: tile rows [64 wg, 64 wg + 64)
constexpr int NT = 32;                              // nodes per node-kernel tile
constexpr int NODE_THREADS = 256;

struct ClfLayer {
  float *Pt, *Qt, *wr, *b1;     // W1 split: [128 in][128 out] x 2, radial column, bias
  float *b2, *watt, *batt;      // edge_mlp.2 bias, att_mlp.0 weight / bias
  float *W3t, *b3, *W4t, *b4;   // node_mlp: [K3 pad][128], [128][128]
  unsigned char* W2s;           // edge_mlp.2 weight as split-bf16 slabs
};

struct ClfWeights {
  float *embWt, *embB;                       // [8][128] (rows 5..7 zero), [128]
  float *nd1t, *nd1b, *nd2t, *nd2b;          // node_dec
  float *gd1t, *gd1b, *gd2, *gd2b;           // graph_dec: [128][128], [128], [128], [1]
};

// ---------------------------------------------------------------------------------------------------- packing
// dst[k][o] (leading dim 128) = src[o][col0 + k] (torch nn.Linear layout [out][in], row length ld)
__global__ void k_clf_transpose(const float* __restrict__ src, int ld, int col0, int ncols, int nout, float* __restrict__ dst) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= ncols * nout) return;
  const int k = idx / nout, o = idx - k * nout;
  dst[(size_t)k * CH + o] = src[(size_t)o * ld + col0 + k];
}
__global__ void k_clf_pack_w2(const float* __restrict__ W, unsigned char* __restrict__ slab) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= CH * CH) return;
  const int n = idx / CH, k = idx - n * CH;
  slab_store(slab + (size_t)(k >> 4) * W2_STEP, CH, n, k & 15, W[idx]);
}
// the slabs of W2^T (B operand of the reverse sweep's da = dz2 . W2)
__global__ void k_clf_pack_w2t(const float* __restrict__ W, unsigned char* __restrict__ slab) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= CH * CH) return;
  const int n = idx / CH, k = idx - n * CH;
  slab_store(slab + (size_t)(k >> 4) * W2_STEP, CH, n, k & 15, W[(size_t)k * CH + n]);
}

// ---------------------------------------------------------------------------------------------------- edge kernel
struct ClfEdgeArgs {
  const float *x, *P, *Q;
  const int* mol_off;            // [B+1]
  const long long* pair_off;     // [B+1]: exclusive prefix sum of n_k^2
  int B;
  long long E;
  int ntiles;
  ClfLayer w;
  int attention;
  float* agg;                    // [N][128]: rows cut by a tile border must be zero on entry
};

struct ClfEdgeSmall {
  float b2[CH], watt[CH];
  int row[CT];                   // global source atom of each tile row (-1 past E)
  int keep[CT];                  // 1 for a pair i != j
  int cutL, cutR;                // tile row 0 continues a row of the previous tile / row 127 continues in the next
  float tail[CH];                // half 0's partial sum of the row that crosses tile row 63 | 64
};
constexpr size_t EDGE_SMEM = A_BYTES + W2_BYTES + sizeof(ClfEdgeSmall) + 1024;

// fp32 view [128 rows][128 cols] of the message tile (over the A blocks once the wgmmas are done); the column is
// xor-swizzled with the row so that fragment stores spread over the banks and row reads stay conflict-free
__device__ __forceinline__ int mt_idx(int r, int c) { return r * CH + (c ^ ((r & 7) << 3)); }

__global__ void __launch_bounds__(EDGE_THREADS, 1) k_clf_edge(ClfEdgeArgs a) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* X = smem;
  unsigned char* W2 = smem + A_BYTES;
  ClfEdgeSmall& S = *reinterpret_cast<ClfEdgeSmall*>(smem + A_BYTES + W2_BYTES);
  float* M = reinterpret_cast<float*>(X);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // W2's hi / lo slabs stay resident for the whole launch
  {
    const uint4* src = reinterpret_cast<const uint4*>(a.w.W2s);
    uint4* dst = reinterpret_cast<uint4*>(W2);
    for (int i = tid; i < W2_BYTES / 16; i += EDGE_THREADS) dst[i] = src[i];
    for (int i = tid; i < CH; i += EDGE_THREADS) { S.b2[i] = a.w.b2[i]; S.watt[i] = a.attention ? a.w.watt[i] : 0.f; }
  }
  const float batt = a.attention ? a.w.batt[0] : 0.f;
  const int wg = tid >> 7;
  const uint32_t xa = smem_u32(X) + (uint32_t)wg * 8192u, wb = smem_u32(W2);

  for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
    // ---- a_ij = silu(P_i + Q_j + w_r radial_ij) -> split-bf16 A tile.  A half warp per pair, 8 columns per lane.
    {
      const int cb = (lane & 15) * 8;
      float wr[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) wr[q] = __ldg(a.w.wr + cb + q);
      for (int it = 0; it < 8; ++it) {
        const int r = warp * 16 + 2 * it + (lane >> 4);
        const long long e = (long long)tile * CT + r;
        float v[8];
        int gi = -1, keep = 0, cut_l = 0, cut_r = 0;
        if (e < a.E) {
          const int k = find_mol(a.pair_off, a.B, e);
          const int n0 = __ldg(a.mol_off + k), n = __ldg(a.mol_off + k + 1) - n0;
          const int loc = (int)(e - __ldg(a.pair_off + k));
          const int i = loc / n, j = loc - i * n;
          gi = n0 + i;
          const int gj = n0 + j;
          keep = i != j;
          cut_l = j != 0;
          cut_r = j != n - 1;
          const float dx = a.x[gi * 3] - a.x[gj * 3], dy = a.x[gi * 3 + 1] - a.x[gj * 3 + 1], dz = a.x[gi * 3 + 2] - a.x[gj * 3 + 2];
          const float rad = dx * dx + dy * dy + dz * dz;
          const float4* pi = reinterpret_cast<const float4*>(a.P + (size_t)gi * CH + cb);
          const float4* qj = reinterpret_cast<const float4*>(a.Q + (size_t)gj * CH + cb);
          const float4 p0 = pi[0], p1 = pi[1], q0 = qj[0], q1 = qj[1];
          const float p[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
          const float q[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
          for (int c = 0; c < 8; ++c) v[c] = silu_acc(fmaf(wr[c], rad, p[c] + q[c]));
        } else {
#pragma unroll
          for (int c = 0; c < 8; ++c) v[c] = 0.f;
        }
        x_store8_hl(X, 2, r, cb, v);
        if ((lane & 15) == 0) {
          S.row[r] = gi;
          S.keep[r] = keep;
          if (r == 0) S.cutL = gi >= 0 && cut_l;
          if (r == CT - 1) S.cutR = gi >= 0 && cut_r;
        }
      }
    }
    fence_proxy_async();
    __syncthreads();

    // ---- m = a . W2^T on the tensor cores: 8 K steps x (A_hi W_hi + A_lo W_hi + A_hi W_lo), one wait
    float d[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < CH / 16; ++ks) {
      const uint64_t ah = gmma_desc_sw128(xa + (ks >> 2) * X_BLOCK + (ks & 3) * 32);
      const uint64_t al = gmma_desc_sw128(xa + (2 + (ks >> 2)) * X_BLOCK + (ks & 3) * 32);
      const uint64_t bh = gmma_desc_k16(wb + ks * W2_STEP, CH * 16, 128);
      const uint64_t bl = gmma_desc_k16(wb + ks * W2_STEP + CH * 32, CH * 16, 128);
      wgmma_n128<1>(d, ah, bh);
      wgmma_n128<1>(d, al, bh);
      wgmma_n128<1>(d, ah, bl);
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence<64>(d);

    // ---- epilogue on the fragments: bias + SiLU, attention gate, pair mask.  Rows frag_row(wg, 0) / (wg, 2) of this thread.
    float att[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 64; ++j) {
      const int c = frag_col(j);
      d[j] = silu_acc(d[j] + S.b2[c]);
      att[(j >> 1) & 1] = fmaf(S.watt[c], d[j], att[(j >> 1) & 1]);
    }
    // the 4 lanes of a quad hold the row's 128 columns: butterfly sum (commutative adds: every lane gets the same bits)
#pragma unroll
    for (int r8 = 0; r8 < 2; ++r8) {
      att[r8] += __shfl_xor_sync(0xffffffffu, att[r8], 1);
      att[r8] += __shfl_xor_sync(0xffffffffu, att[r8], 2);
    }
    float g[2];
#pragma unroll
    for (int r8 = 0; r8 < 2; ++r8) {
      const int rr = frag_row(wg, 2 * r8);
      g[r8] = S.keep[rr] ? (a.attention ? sigmoid_acc(att[r8] + batt) : 1.f) : 0.f;
    }
    __syncthreads();     // both warpgroups' wgmmas have read the A tile: it becomes the fp32 message tile
#pragma unroll
    for (int j = 0; j < 64; j += 2) {
      const int rr = frag_row(wg, j), c = frag_col(j), r8 = (j >> 1) & 1;
      *reinterpret_cast<float2*>(M + mt_idx(rr, c)) = make_float2(d[j] * g[r8], d[j + 1] * g[r8]);
    }
    __syncthreads();

    // ---- agg_i = sum_j m_ij, deterministic: thread (half, column c) scans tile rows [64 half, 64 half + 64) in order.
    // One value per (tile, source atom, column) leaves the tile: a plain store if the atom's whole row of pairs lies in
    // the tile, else a red.add into a word that is zero on entry; a row has <= 128 pairs, so it is cut by at most one tile
    // border and such a word receives exactly two addends (commutative: the result does not depend on their order).  The
    // row that crosses tile row 63 | 64 is summed as (half 0's part) + (half 1's part).
    {
      const int c = tid & (CH - 1), half = tid >> 7, r0 = half * 64;
      const int row0 = S.row[0], rowL = S.row[CT - 1];
      auto emit = [&](int row, float v) {
        if (row < 0) return;
        float* dst = a.agg + (size_t)row * CH + c;
        if ((S.cutL && row == row0) || (S.cutR && row == rowL)) atomicAdd(dst, v);
        else *dst = v;
      };
      const bool joined = S.row[63] >= 0 && S.row[63] == S.row[64];
      int cur = S.row[r0];
      float acc = 0.f, head = 0.f;
      bool first = true;
      for (int r = r0; r < r0 + 64; ++r) {
        const int row = S.row[r];
        if (row != cur) {
          if (half == 1 && first && joined) head = acc;
          else emit(cur, acc);
          first = false;
          cur = row;
          acc = 0.f;
        }
        acc += M[mt_idx(r, c)];
      }
      if (half == 0 && joined) S.tail[c] = acc;
      else if (half == 1 && first && joined) head = acc;
      else emit(cur, acc);
      __syncthreads();
      if (half == 1 && joined) emit(S.row[64], S.tail[c] + head);
    }
    __syncthreads();     // message tile, row records and tail free for the next tile
  }
}

// ---------------------------------------------------------------------------------------------------- node kernels
// acc[4 nodes][4 columns] (+)= sIn[NT][ld] . Wt[K][128]: thread (warp w, lane l) owns nodes 4w..4w+3 and columns 4l..4l+3;
// K is a multiple of 4 (zero-padded in both operands).  Every output is one fp32 FMA chain in k order.
__device__ __forceinline__ void tile_gemm(const float* __restrict__ sIn, int ld, int K, const float* __restrict__ Wt,
                                          float (&acc)[4][4]) {
  const int n0 = (threadIdx.x >> 5) * 4, c0 = (threadIdx.x & 31) * 4;
  for (int k = 0; k < K; k += 4) {
    float4 w[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) w[q] = __ldg(reinterpret_cast<const float4*>(Wt + (size_t)(k + q) * CH + c0));
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      const float4 s = *reinterpret_cast<const float4*>(sIn + (n0 + n) * ld + k);
      const float sv[4] = {s.x, s.y, s.z, s.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        acc[n][0] = fmaf(sv[q], w[q].x, acc[n][0]);
        acc[n][1] = fmaf(sv[q], w[q].y, acc[n][1]);
        acc[n][2] = fmaf(sv[q], w[q].z, acc[n][2]);
        acc[n][3] = fmaf(sv[q], w[q].w, acc[n][3]);
      }
    }
  }
}
__device__ __forceinline__ void acc_init(float (&acc)[4][4], const float* bias) {
  const int c0 = (threadIdx.x & 31) * 4;
#pragma unroll
  for (int n = 0; n < 4; ++n)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[n][q] = bias ? __ldg(bias + c0 + q) : 0.f;
}
// rows of acc -> sOut (leading dim K3_MAX; optionally SiLU) and / or global rows (nodes past N are not written)
__device__ __forceinline__ void acc_out(const float (&acc)[4][4], float* sOut, bool silu, float* g, int node0, int N) {
  const int n0 = (threadIdx.x >> 5) * 4, c0 = (threadIdx.x & 31) * 4;
#pragma unroll
  for (int n = 0; n < 4; ++n) {
    float4 v = make_float4(acc[n][0], acc[n][1], acc[n][2], acc[n][3]);
    if (silu) v = make_float4(silu_acc(v.x), silu_acc(v.y), silu_acc(v.z), silu_acc(v.w));
    if (sOut) *reinterpret_cast<float4*>(sOut + (n0 + n) * K3_MAX + c0) = v;
    if (g && node0 + n0 + n < N) *reinterpret_cast<float4*>(g + (size_t)(node0 + n0 + n) * CH + c0) = v;
  }
}

struct ClfNodeArgs {
  const float* one_hot;   // [N][5]
  float *h, *agg, *P, *Q, *nodeout;
  int N, layer, L, node_attr;
  ClfLayer cur, nxt;
  ClfWeights g;
  // training pass only (TAPE = true): h_out receives the layer's output (h is its input and is not overwritten), agg is
  // the layer's own tape slice (read, not zeroed), and the pre-activations / SiLU outputs the reverse sweep reads
  float *h_out, *v, *u, *q, *qs;
};

// layer < 0: embedding (EGNN.forward :407), then P / Q of layer 0.
// layer l:   h += node_mlp([h | agg (| h0)]) (E_GCL.node_model :318-328), agg rows zeroed after reading (the next edge
//            kernel's red.add words); then P / Q of layer l + 1, or node_dec after the last layer (:415).
// One [NT][K3_MAX] tile in shared memory: columns 0..127 hold h, 128..255 agg and then the hidden activation u,
// 256..263 the one-hot h0 (node_attr).
// TAPE = false is the inference kernel; TAPE = true (the training pass) runs the same arithmetic and also writes the tape
// (ClfNodeArgs: h_out, v / u = node_mlp.0 pre-activation / SiLU, q / qs = node_dec.0 pre-activation / SiLU).
template <bool TAPE>
__global__ void __launch_bounds__(NODE_THREADS) k_clf_node(ClfNodeArgs a) {
  __shared__ __align__(16) float sIn[NT * K3_MAX];
  float* const sH = sIn;
  float* const sU = sIn + CH;
  const int node0 = blockIdx.x * NT, tid = threadIdx.x;
  float acc[4][4];
  auto load_h0 = [&](float* dst) {
    for (int i = tid; i < NT * 8; i += NODE_THREADS) {
      const int n = i >> 3, k = i & 7;
      dst[n * K3_MAX + k] = (k < CIN && node0 + n < a.N) ? a.one_hot[(size_t)(node0 + n) * CIN + k] : 0.f;
    }
  };
  if (a.layer < 0) {
    load_h0(sU);
    __syncthreads();
    acc_init(acc, a.g.embB);
    tile_gemm(sU, K3_MAX, 8, a.g.embWt, acc);
    acc_out(acc, sH, false, TAPE ? a.h_out : a.h, node0, a.N);
  } else {
    for (int i = tid; i < NT * (CH / 4); i += NODE_THREADS) {
      const int n = i / (CH / 4), c = (i % (CH / 4)) * 4;
      float4 hv = make_float4(0.f, 0.f, 0.f, 0.f), gv = hv;
      if (node0 + n < a.N) {
        float4* ag = reinterpret_cast<float4*>(a.agg + (size_t)(node0 + n) * CH + c);
        hv = *reinterpret_cast<const float4*>(a.h + (size_t)(node0 + n) * CH + c);
        gv = *ag;
        if constexpr (!TAPE) *ag = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      *reinterpret_cast<float4*>(sH + n * K3_MAX + c) = hv;
      *reinterpret_cast<float4*>(sU + n * K3_MAX + c) = gv;
    }
    if (a.node_attr) load_h0(sIn + 2 * CH);
    __syncthreads();
    acc_init(acc, a.cur.b3);
    tile_gemm(sIn, K3_MAX, a.node_attr ? 2 * CH + 8 : 2 * CH, a.cur.W3t, acc);
    __syncthreads();     // agg is read: u takes its columns
    if constexpr (TAPE) acc_out(acc, nullptr, false, a.v, node0, a.N);
    acc_out(acc, sU, true, TAPE ? a.u : nullptr, node0, a.N);
    __syncthreads();
    acc_init(acc, a.cur.b4);
    tile_gemm(sU, K3_MAX, CH, a.cur.W4t, acc);
    {
      const int n0 = (tid >> 5) * 4, c0 = (tid & 31) * 4;
#pragma unroll
      for (int n = 0; n < 4; ++n)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[n][q] = sH[(n0 + n) * K3_MAX + c0 + q] + acc[n][q];
    }
    __syncthreads();     // every thread has read its h entries before they are overwritten
    acc_out(acc, sH, false, TAPE ? a.h_out : a.h, node0, a.N);
  }
  __syncthreads();
  if (a.layer < a.L - 1) {
    acc_init(acc, a.nxt.b1);
    tile_gemm(sH, K3_MAX, CH, a.nxt.Pt, acc);
    acc_out(acc, nullptr, false, a.P, node0, a.N);
    acc_init(acc, nullptr);
    tile_gemm(sH, K3_MAX, CH, a.nxt.Qt, acc);
    acc_out(acc, nullptr, false, a.Q, node0, a.N);
  } else {
    acc_init(acc, a.g.nd1b);
    tile_gemm(sH, K3_MAX, CH, a.g.nd1t, acc);
    if constexpr (TAPE) acc_out(acc, nullptr, false, a.q, node0, a.N);
    acc_out(acc, sU, true, TAPE ? a.qs : nullptr, node0, a.N);
    __syncthreads();
    acc_init(acc, a.g.nd2b);
    tile_gemm(sU, K3_MAX, CH, a.g.nd2t, acc);
    acc_out(acc, nullptr, false, a.nodeout, node0, a.N);
  }
}

// pred_k = graph_dec(sum_{i in k} node_dec(h_i)): one CTA per molecule, the atom sum in atom order per column.
// TAPE: also the molecule sums s, the graph_dec.0 pre-activation w and its SiLU ws, [B][128] each.
template <bool TAPE>
__global__ void __launch_bounds__(CH) k_clf_readout(const float* __restrict__ nodeout, const int* __restrict__ mol_off,
                                                    ClfWeights g, float* __restrict__ pred, float* __restrict__ s_t = nullptr,
                                                    float* __restrict__ w_t = nullptr, float* __restrict__ ws_t = nullptr) {
  __shared__ float s[CH], u[CH];
  const int k = blockIdx.x, c = threadIdx.x;
  const int a0 = mol_off[k], a1 = mol_off[k + 1];
  float acc = 0.f;
  for (int i = a0; i < a1; ++i) acc += nodeout[(size_t)i * CH + c];
  s[c] = acc;
  __syncthreads();
  float v = g.gd1b[c];
  for (int q = 0; q < CH; ++q) v = fmaf(s[q], __ldg(g.gd1t + (size_t)q * CH + c), v);
  if constexpr (TAPE) {
    s_t[(size_t)k * CH + c] = acc;
    w_t[(size_t)k * CH + c] = v;
    ws_t[(size_t)k * CH + c] = silu_acc(v);
  }
  u[c] = silu_acc(v) * g.gd2[c];
  __syncthreads();
  if (c == 0) {
    float p = g.gd2b[0];
    for (int q = 0; q < CH; ++q) p += u[q];
    pred[k] = p;
  }
}

}  // namespace bdiff

#include "bdiff_classifier_train.cuh"

// ---------------------------------------------------------------------------------------------------- C ABI
using namespace bdiff;

struct bdiff_classifier {
  bdiff_classifier_config cfg;
  float* wbuf = nullptr;
  unsigned char* w2buf = nullptr;
  std::vector<ClfLayer> layers;
  ClfWeights g{};
  std::map<std::string, bool> seen;
  // workspace (grown on demand)
  void* ws = nullptr;
  size_t ws_bytes = 0;
  // training pass: W2^T slabs, the canonical flat layout (name -> offset, count), one tape and the reverse sweep's scratch
  unsigned char* w2tbuf = nullptr;
  std::map<std::string, std::pair<int64_t, int64_t>> playout;
  int64_t pfloats = 0;
  void* tape = nullptr;
  size_t tape_bytes = 0;
  void* bws = nullptr;
  size_t bws_bytes = 0;
  bool tape_valid = false;
  uint64_t weights_gen = 0, tape_weights_gen = 0;
  int tape_B = 0, tape_N = 0;
  long long tape_E = 0;
  int num_sms = 0;
  std::string err;
  int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    err = buf;
    return code;
  }
};

namespace {
thread_local std::string g_clf_create_error;

int k3_pad(const bdiff_classifier_config& c) { return c.node_attr ? 2 * CH + 8 : 2 * CH; }

size_t layout(bdiff_classifier* h, bool assign) {
  size_t used = 0;
  auto A = [&](size_t n) -> float* {
    float* r = assign ? h->wbuf + used : nullptr;
    used += (n + 63) / 64 * 64;
    return r;
  };
  ClfWeights& g = h->g;
  g.embWt = A(8 * CH); g.embB = A(CH);
  g.nd1t = A(CH * CH); g.nd1b = A(CH); g.nd2t = A(CH * CH); g.nd2b = A(CH);
  g.gd1t = A(CH * CH); g.gd1b = A(CH); g.gd2 = A(CH); g.gd2b = A(1);
  h->layers.assign(h->cfg.n_layers, ClfLayer{});
  for (int l = 0; l < h->cfg.n_layers; ++l) {
    ClfLayer& w = h->layers[l];
    w.Pt = A(CH * CH); w.Qt = A(CH * CH); w.wr = A(CH); w.b1 = A(CH);
    w.b2 = A(CH); w.watt = A(CH); w.batt = A(1);
    w.W3t = A((size_t)k3_pad(h->cfg) * CH); w.b3 = A(CH); w.W4t = A(CH * CH); w.b4 = A(CH);
    w.W2s = assign ? h->w2buf + (size_t)l * W2_BYTES : nullptr;
  }
  return used;
}

// one repack step: transposed columns [col0, col0 + ncols) of a [rows][cols] tensor, or a plain copy (transpose of a
// [n][1] bias is a copy), or the W2 slab
struct ClfOp { float* dst; int col0, ncols; unsigned char* slab; bool tr = false; };

bool resolve(bdiff_classifier* h, const std::string& name, std::vector<ClfOp>& ops, int64_t& rows, int64_t& cols) {
  const int in3 = 2 * CH + (h->cfg.node_attr ? CIN : 0);
  auto lin = [&](float* wt, float* b, int fan_in, int nout, const std::string& leaf) -> bool {
    if (leaf == "weight") { rows = nout; cols = fan_in; ops.push_back({wt, 0, fan_in, nullptr}); return true; }
    if (leaf == "bias") { rows = nout; cols = 1; ops.push_back({b, 0, 1, nullptr}); return true; }
    return false;
  };
  ClfWeights& g = h->g;
  if (name.rfind("embedding.", 0) == 0) return lin(g.embWt, g.embB, CIN, CH, name.substr(10));
  if (name.rfind("node_dec.0.", 0) == 0) return lin(g.nd1t, g.nd1b, CH, CH, name.substr(11));
  if (name.rfind("node_dec.2.", 0) == 0) return lin(g.nd2t, g.nd2b, CH, CH, name.substr(11));
  if (name.rfind("graph_dec.0.", 0) == 0) return lin(g.gd1t, g.gd1b, CH, CH, name.substr(12));
  if (name == "graph_dec.2.weight") { rows = 1; cols = CH; ops.push_back({g.gd2, 0, CH, nullptr}); return true; }
  if (name == "graph_dec.2.bias") { rows = 1; cols = 1; ops.push_back({g.gd2b, 0, 1, nullptr}); return true; }
  int l = -1, used = 0;
  if (sscanf(name.c_str(), "gcl_%d.%n", &l, &used) != 1 || used == 0 || l < 0 || l >= h->cfg.n_layers) return false;
  const std::string rest = name.substr(used);
  ClfLayer& w = h->layers[l];
  if (rest == "edge_mlp.0.weight") {
    rows = CH; cols = 2 * CH + 1;
    ops.push_back({w.Pt, 0, CH, nullptr});
    ops.push_back({w.Qt, CH, CH, nullptr});
    ops.push_back({w.wr, 2 * CH, 1, nullptr});
    return true;
  }
  if (rest == "edge_mlp.0.bias") { rows = CH; cols = 1; ops.push_back({w.b1, 0, 1, nullptr}); return true; }
  if (rest == "edge_mlp.2.weight") {
    rows = CH; cols = CH;
    ops.push_back({nullptr, 0, 0, w.W2s});
    if (h->w2tbuf) ops.push_back({nullptr, 0, 0, h->w2tbuf + (size_t)l * W2_BYTES, true});
    return true;
  }
  if (rest == "edge_mlp.2.bias") { rows = CH; cols = 1; ops.push_back({w.b2, 0, 1, nullptr}); return true; }
  if (rest.rfind("node_mlp.0.", 0) == 0) return lin(w.W3t, w.b3, in3, CH, rest.substr(11));
  if (rest.rfind("node_mlp.2.", 0) == 0) return lin(w.W4t, w.b4, CH, CH, rest.substr(11));
  if (h->cfg.attention && rest == "att_mlp.0.weight") { rows = 1; cols = CH; ops.push_back({w.watt, 0, CH, nullptr}); return true; }
  if (h->cfg.attention && rest == "att_mlp.0.bias") { rows = 1; cols = 1; ops.push_back({w.batt, 0, 1, nullptr}); return true; }
  return false;
}

cudaError_t grow_buf(void*& buf, size_t& have, size_t bytes) {
  if (bytes <= have) return cudaSuccess;
  if (buf) cudaFree(buf);
  buf = nullptr;
  have = 0;
  cudaError_t e = cudaMalloc(&buf, bytes);
  if (e == cudaSuccess) have = bytes;
  return e;
}
cudaError_t grow(bdiff_classifier* h, size_t bytes) { return grow_buf(h->ws, h->ws_bytes, bytes); }

// Bump allocator over one device buffer: 256-byte aligned float slices.
struct Carve {
  unsigned char* base;
  size_t used = 0;
  float* f(size_t n) {
    float* r = base ? reinterpret_cast<float*>(base + used) : nullptr;
    used += (n * sizeof(float) + 255) / 256 * 256;
    return r;
  }
};

// The tape of one training forward (B molecules, N atoms, L layers).  Per layer l: h[l] its input (h[L] the last output),
// P / Q (edge_mlp.0 node halves), agg, v / u (node_mlp.0 pre-activation / SiLU); node_dec's q / qs; readout s / w / ws;
// copies of x, one_hot and the offsets (the reverse sweep must not depend on the caller's buffers).
struct ClfTape {
  float *h, *P, *Q, *agg, *v, *u, *q, *qs, *nodeout, *s, *w, *ws, *x, *oh;
  int* mol_off;
  long long* pair_off;
};
size_t tape_carve(unsigned char* base, int L, int N, int B, ClfTape& t) {
  Carve c{base};
  const size_t nc = (size_t)N * CH, lnc = (size_t)L * nc, bc = (size_t)B * CH;
  t.h = c.f(lnc + nc); t.P = c.f(lnc); t.Q = c.f(lnc); t.agg = c.f(lnc); t.v = c.f(lnc); t.u = c.f(lnc);
  t.q = c.f(nc); t.qs = c.f(nc); t.nodeout = c.f(nc); t.s = c.f(bc); t.w = c.f(bc); t.ws = c.f(bc);
  t.x = c.f((size_t)N * 3); t.oh = c.f((size_t)N * CIN);
  t.mol_off = reinterpret_cast<int*>(c.f(B + 1));
  t.pair_off = reinterpret_cast<long long*>(c.f(2 * (size_t)(B + 1)));
  return c.used;
}
// Scratch of the reverse sweep.  Per atom: two dh buffers (ping-pong over layers), dv, dagg, dP, dQ, R, dy, dq; per
// molecule dw, dS; per pair a, s, dz2, dz1 and dt; the weight-gradient chunk partials.
constexpr long long WG_MAX_CHUNKS = 256;
struct ClfBwdScratch {
  float *dHa, *dHb, *dV, *dAgg, *dP, *dQ, *R, *dY, *dQd, *dWk, *dS, *A, *S, *DZ2, *DZ1, *DT, *part;
};
size_t bws_carve(unsigned char* base, int N, int B, long long E, ClfBwdScratch& t) {
  Carve c{base};
  const size_t nc = (size_t)N * CH, ec = (size_t)E * CH;
  t.dHa = c.f(nc); t.dHb = c.f(nc); t.dV = c.f(nc); t.dAgg = c.f(nc); t.dP = c.f(nc); t.dQ = c.f(nc); t.R = c.f(nc);
  t.dY = c.f(nc); t.dQd = c.f(nc); t.dWk = c.f((size_t)B * CH); t.dS = c.f((size_t)B * CH);
  t.A = c.f(ec); t.S = c.f(ec); t.DZ2 = c.f(ec); t.DZ1 = c.f(ec); t.DT = c.f(E);
  t.part = c.f((size_t)WG_MAX_CHUNKS * CH * (CH + 1));
  return c.used;
}

// dW[o][col0 + k] = sum_rows G[row][o] X[row][k] (k < K), db[o * dbs] = sum_rows G[row][o]: fixed chunks of rows, then
// the chunks in index order — the summation order depends on `rows` only.
void wgrad(cudaStream_t st, float* part, const float* G, int ldg, const float* X, int ldx, int O, int K, long long rows,
           float* dW, int ldw, int col0, float* db, int dbs) {
  long long nchunks = std::max(1ll, std::min(WG_MAX_CHUNKS, (rows + 255) / 256));
  const long long chunk = ((rows + nchunks - 1) / nchunks + 31) / 32 * 32;
  nchunks = std::max(1ll, (rows + chunk - 1) / chunk);
  ClfWgradArgs a{G, X, ldg, ldx, O, K, rows, chunk, part};
  k_clf_wgrad<<<dim3((O + 31) / 32, (K + 1 + 31) / 32, (unsigned)nchunks), 256, 0, st>>>(a);
  k_clf_wgrad_sum<<<(O * (K + 1) + 255) / 256, 256, 0, st>>>(part, (int)nchunks, O, K, dW, ldw, col0, db, dbs);
}

// host checks of a packed batch shared by the inference and the training forward: pair offsets, or an error message
int check_batch(bdiff_classifier* h, int32_t num_mols, const int32_t* mol_off_host, std::vector<long long>& pair_off) {
  for (const auto& kv : h->seen)
    if (!kv.second) return h->fail(BDIFF_ESTATE, "parameter '%s' was never set", kv.first.c_str());
  if (mol_off_host[0] != 0) return h->fail(BDIFF_EINVAL, "mol_off[0] must be 0");
  pair_off.assign(num_mols + 1, 0);
  for (int k = 0; k < num_mols; ++k) {
    const int n = mol_off_host[k + 1] - mol_off_host[k];
    if (n < 1 || n > CLF_MAX_ATOMS)
      return h->fail(BDIFF_EINVAL, "molecule %d has %d atoms: the classifier takes 1..%d atoms per molecule", k, n, CLF_MAX_ATOMS);
    pair_off[k + 1] = pair_off[k] + (long long)n * n;
  }
  if ((pair_off[num_mols] + CT - 1) / CT > (1ll << 30)) return h->fail(BDIFF_EINVAL, "batch too large");
  return BDIFF_OK;
}

}  // namespace

extern "C" {

int32_t bdiff_classifier_create(const bdiff_classifier_config* cfg, bdiff_classifier** out) {
  if (!cfg || !out) { g_clf_create_error = "null argument"; return BDIFF_EINVAL; }
  *out = nullptr;
  if (cfg->in_node_nf != CIN) { g_clf_create_error = "in_node_nf must be 5"; return BDIFF_EINVAL; }
  if (cfg->in_edge_nf != 0) { g_clf_create_error = "in_edge_nf must be 0 (edge attributes are not supported)"; return BDIFF_EINVAL; }
  if (cfg->hidden_nf != CH) { g_clf_create_error = "hidden_nf must be 128"; return BDIFF_EINVAL; }
  if (cfg->n_layers < 1 || cfg->n_layers > 64) { g_clf_create_error = "n_layers out of range [1, 64]"; return BDIFF_EINVAL; }
  if ((cfg->attention != 0 && cfg->attention != 1) || (cfg->node_attr != 0 && cfg->node_attr != 1)) {
    g_clf_create_error = "attention and node_attr must be 0 or 1";
    return BDIFF_EINVAL;
  }
  int dev_count = 0;
  if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count == 0) {
    g_clf_create_error = "no CUDA device: libbdiff_sm90 has no CPU fallback";
    return BDIFF_ECUDA;
  }
  cudaDeviceProp prop{};
  int dev = 0;
  cudaGetDevice(&dev);
  cudaGetDeviceProperties(&prop, dev);
  if (prop.major != 9 || prop.minor != 0) {
    g_clf_create_error = "libbdiff_sm90 is built for sm_90a (H100) only";
    return BDIFF_ECUDA;
  }
  bdiff_classifier* h = new bdiff_classifier();
  h->cfg = *cfg;
  h->num_sms = prop.multiProcessorCount;
  const size_t nf = layout(h, false);
  cudaError_t e = cudaMalloc(&h->wbuf, nf * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->w2buf, (size_t)cfg->n_layers * W2_BYTES);
  if (e == cudaSuccess) e = cudaMalloc(&h->w2tbuf, (size_t)cfg->n_layers * W2_BYTES);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_clf_bwd_edge, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BWD_EDGE_SMEM);
  if (e == cudaSuccess) e = cudaMemset(h->wbuf, 0, nf * sizeof(float));
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_clf_edge, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)EDGE_SMEM);
  if (e != cudaSuccess) {
    g_clf_create_error = std::string("bdiff_classifier_create: ") + cudaGetErrorString(e);
    if (h->wbuf) cudaFree(h->wbuf);
    if (h->w2buf) cudaFree(h->w2buf);
    if (h->w2tbuf) cudaFree(h->w2tbuf);
    delete h;
    return BDIFF_ECUDA;
  }
  layout(h, true);
  auto lin = [&](const std::string& p) { h->seen[p + ".weight"] = false; h->seen[p + ".bias"] = false; };
  lin("embedding");
  for (int l = 0; l < cfg->n_layers; ++l) {
    const std::string p = "gcl_" + std::to_string(l) + ".";
    lin(p + "edge_mlp.0"); lin(p + "edge_mlp.2"); lin(p + "node_mlp.0"); lin(p + "node_mlp.2");
    if (cfg->attention) lin(p + "att_mlp.0");
  }
  lin("node_dec.0"); lin("node_dec.2"); lin("graph_dec.0"); lin("graph_dec.2");
  // canonical flat layout of the parameters / gradients: ascending name order, each tensor at a multiple of 64 floats
  for (const auto& kv : h->seen) {
    std::vector<ClfOp> ops;
    int64_t rows = 0, cols = 0;
    resolve(h, kv.first, ops, rows, cols);
    h->playout[kv.first] = {h->pfloats, rows * cols};
    h->pfloats += (rows * cols + 63) / 64 * 64;
  }
  *out = h;
  return BDIFF_OK;
}

void bdiff_classifier_destroy(bdiff_classifier* h) {
  if (!h) return;
  if (h->wbuf) cudaFree(h->wbuf);
  if (h->w2buf) cudaFree(h->w2buf);
  if (h->w2tbuf) cudaFree(h->w2tbuf);
  if (h->ws) cudaFree(h->ws);
  if (h->tape) cudaFree(h->tape);
  if (h->bws) cudaFree(h->bws);
  delete h;
}

const char* bdiff_classifier_last_error(const bdiff_classifier* h) { return h ? h->err.c_str() : g_clf_create_error.c_str(); }

int32_t bdiff_classifier_set_weight(bdiff_classifier* h, void* stream, const char* name, const float* data,
                                    const int64_t* shape, int32_t ndim) {
  if (!h || !name || !data || !shape || ndim < 1 || ndim > 2) return h ? h->fail(BDIFF_EINVAL, "bad argument") : BDIFF_EINVAL;
  auto it = h->seen.find(name);
  std::vector<ClfOp> ops;
  int64_t rows = 0, cols = 0;
  if (it == h->seen.end() || !resolve(h, name, ops, rows, cols)) return h->fail(BDIFF_EINVAL, "unknown parameter name '%s'", name);
  const int64_t got_rows = shape[0], got_cols = ndim == 2 ? shape[1] : 1;
  if (got_rows != rows || got_cols != cols)
    return h->fail(BDIFF_EINVAL, "parameter '%s': expected shape [%lld,%lld], got [%lld,%lld]", name, (long long)rows,
                   (long long)cols, (long long)got_rows, (long long)got_cols);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (const ClfOp& op : ops) {
    if (op.slab && op.tr) {
      k_clf_pack_w2t<<<(CH * CH + 255) / 256, 256, 0, st>>>(data, op.slab);
    } else if (op.slab) {
      k_clf_pack_w2<<<(CH * CH + 255) / 256, 256, 0, st>>>(data, op.slab);
    } else if (cols == 1 || rows == 1) {      // bias or single-row weight: a copy
      cudaMemcpyAsync(op.dst, data, (size_t)rows * cols * sizeof(float), cudaMemcpyDeviceToDevice, st);
    } else {
      const int n = op.ncols * (int)rows;
      k_clf_transpose<<<(n + 255) / 256, 256, 0, st>>>(data, (int)cols, op.col0, op.ncols, (int)rows, op.dst);
    }
  }
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "set_weight(%s): %s", name, cudaGetErrorString(e));
  it->second = true;
  ++h->weights_gen;
  return BDIFF_OK;
}

int32_t bdiff_classifier_forward(bdiff_classifier* h, void* stream, int32_t num_mols, const int32_t* mol_off_host,
                                 const float* x, const float* one_hot, float* pred) {
  if (!h) return BDIFF_EINVAL;
  if (num_mols < 1 || !mol_off_host || !x || !one_hot || !pred) return h->fail(BDIFF_EINVAL, "bad argument");
  std::vector<long long> pair_off;
  if (const int rc = check_batch(h, num_mols, mol_off_host, pair_off)) return rc;
  const int N = mol_off_host[num_mols];
  const long long E = pair_off[num_mols];
  const long long ntiles = (E + CT - 1) / CT;
  // workspace: h, P, Q, agg, nodeout [N][128] fp32 | mol_off int32 [B+1] | pair_off int64 [B+1]
  const size_t node_bytes = (size_t)N * CH * sizeof(float);
  const size_t off_i = 5 * node_bytes, off_p = off_i + ((size_t)(num_mols + 1) * 4 + 15) / 16 * 16;
  cudaError_t e = grow(h, off_p + (size_t)(num_mols + 1) * 8);
  if (e != cudaSuccess) return h->fail(BDIFF_ENOMEM, "workspace: %s", cudaGetErrorString(e));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  unsigned char* ws = static_cast<unsigned char*>(h->ws);
  float* hb = reinterpret_cast<float*>(ws);
  float* P = reinterpret_cast<float*>(ws + node_bytes);
  float* Q = reinterpret_cast<float*>(ws + 2 * node_bytes);
  float* agg = reinterpret_cast<float*>(ws + 3 * node_bytes);
  float* nodeout = reinterpret_cast<float*>(ws + 4 * node_bytes);
  int* mol_off = reinterpret_cast<int*>(ws + off_i);
  long long* poff = reinterpret_cast<long long*>(ws + off_p);
  cudaMemcpyAsync(mol_off, mol_off_host, (size_t)(num_mols + 1) * 4, cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(poff, pair_off.data(), (size_t)(num_mols + 1) * 8, cudaMemcpyHostToDevice, st);
  cudaMemsetAsync(agg, 0, node_bytes, st);

  const int L = h->cfg.n_layers;
  ClfNodeArgs na{};
  na.one_hot = one_hot; na.h = hb; na.agg = agg; na.P = P; na.Q = Q; na.nodeout = nodeout;
  na.N = N; na.L = L; na.node_attr = h->cfg.node_attr; na.g = h->g;
  const int node_grid = (N + NT - 1) / NT;
  ClfEdgeArgs ea{};
  ea.x = x; ea.P = P; ea.Q = Q; ea.mol_off = mol_off; ea.pair_off = poff; ea.B = num_mols; ea.E = E;
  ea.ntiles = (int)ntiles; ea.attention = h->cfg.attention; ea.agg = agg;
  const int edge_grid = (int)std::min<long long>(ntiles, h->num_sms);
  for (int l = -1; l < L; ++l) {
    if (l >= 0) {
      ea.w = h->layers[l];
      k_clf_edge<<<edge_grid, EDGE_THREADS, EDGE_SMEM, st>>>(ea);
    }
    na.layer = l;
    if (l >= 0) na.cur = h->layers[l];
    if (l + 1 < L) na.nxt = h->layers[l + 1];
    k_clf_node<false><<<node_grid, NODE_THREADS, 0, st>>>(na);
  }
  k_clf_readout<false><<<num_mols, CH, 0, st>>>(nodeout, mol_off, h->g, pred);
  e = cudaGetLastError();
  if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "classifier forward: %s", cudaGetErrorString(e));
  return BDIFF_OK;
}

int64_t bdiff_classifier_param_floats(const bdiff_classifier* h) { return h ? h->pfloats : 0; }

int32_t bdiff_classifier_param_layout(bdiff_classifier* h, const char* name, int64_t* offset, int64_t* count) {
  if (!h || !name || !offset || !count) return h ? h->fail(BDIFF_EINVAL, "bad argument") : BDIFF_EINVAL;
  auto it = h->playout.find(name);
  if (it == h->playout.end()) return h->fail(BDIFF_EINVAL, "unknown parameter name '%s'", name);
  *offset = it->second.first;
  *count = it->second.second;
  return BDIFF_OK;
}

int32_t bdiff_classifier_train_forward(bdiff_classifier* h, void* stream, int32_t num_mols, const int32_t* mol_off_host,
                                       const float* x, const float* one_hot, float* pred) {
  if (!h) return BDIFF_EINVAL;
  if (num_mols < 1 || !mol_off_host || !x || !one_hot || !pred) return h->fail(BDIFF_EINVAL, "bad argument");
  std::vector<long long> pair_off;
  if (const int rc = check_batch(h, num_mols, mol_off_host, pair_off)) return rc;
  const int N = mol_off_host[num_mols], L = h->cfg.n_layers;
  const long long E = pair_off[num_mols];
  const long long ntiles = (E + CT - 1) / CT;
  h->tape_valid = false;
  ClfTape t{};
  cudaError_t e = grow_buf(h->tape, h->tape_bytes, tape_carve(nullptr, L, N, num_mols, t));
  if (e != cudaSuccess) return h->fail(BDIFF_ENOMEM, "tape: %s", cudaGetErrorString(e));
  tape_carve(static_cast<unsigned char*>(h->tape), L, N, num_mols, t);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t nc = (size_t)N * CH;
  cudaMemcpyAsync(t.mol_off, mol_off_host, (size_t)(num_mols + 1) * 4, cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(t.pair_off, pair_off.data(), (size_t)(num_mols + 1) * 8, cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(t.x, x, (size_t)N * 3 * sizeof(float), cudaMemcpyDeviceToDevice, st);
  cudaMemcpyAsync(t.oh, one_hot, (size_t)N * CIN * sizeof(float), cudaMemcpyDeviceToDevice, st);
  cudaMemsetAsync(t.agg, 0, (size_t)L * nc * sizeof(float), st);    // every layer's agg: the edge kernel's red.add words

  // the inference kernels' schedule; TAPE = true node / readout kernels keep what the reverse sweep reads
  ClfNodeArgs na{};
  na.one_hot = t.oh; na.nodeout = t.nodeout; na.N = N; na.L = L; na.node_attr = h->cfg.node_attr; na.g = h->g;
  na.q = t.q; na.qs = t.qs;
  const int node_grid = (N + NT - 1) / NT;
  ClfEdgeArgs ea{};
  ea.x = t.x; ea.mol_off = t.mol_off; ea.pair_off = t.pair_off; ea.B = num_mols; ea.E = E;
  ea.ntiles = (int)ntiles; ea.attention = h->cfg.attention;
  const int edge_grid = (int)std::min<long long>(ntiles, h->num_sms);
  for (int l = -1; l < L; ++l) {
    if (l >= 0) {
      ea.w = h->layers[l];
      ea.P = t.P + l * nc; ea.Q = t.Q + l * nc; ea.agg = t.agg + l * nc;
      k_clf_edge<<<edge_grid, EDGE_THREADS, EDGE_SMEM, st>>>(ea);
    }
    na.layer = l;
    na.h = l >= 0 ? t.h + l * nc : nullptr;
    na.h_out = t.h + (l + 1) * nc;
    if (l >= 0) {
      na.cur = h->layers[l];
      na.agg = t.agg + l * nc; na.v = t.v + l * nc; na.u = t.u + l * nc;
    }
    if (l + 1 < L) { na.nxt = h->layers[l + 1]; na.P = t.P + (l + 1) * nc; na.Q = t.Q + (l + 1) * nc; }
    k_clf_node<true><<<node_grid, NODE_THREADS, 0, st>>>(na);
  }
  k_clf_readout<true><<<num_mols, CH, 0, st>>>(t.nodeout, t.mol_off, h->g, pred, t.s, t.w, t.ws);
  e = cudaGetLastError();
  if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "classifier training forward: %s", cudaGetErrorString(e));
  h->tape_valid = true;
  h->tape_weights_gen = h->weights_gen;
  h->tape_B = num_mols; h->tape_N = N; h->tape_E = E;
  return BDIFF_OK;
}

int32_t bdiff_classifier_train_backward(bdiff_classifier* h, void* stream, const float* d_pred, float* grad_flat) {
  if (!h) return BDIFF_EINVAL;
  if (!d_pred || !grad_flat) return h->fail(BDIFF_EINVAL, "bad argument");
  if (!h->tape_valid) return h->fail(BDIFF_ESTATE, "no tape: run bdiff_classifier_train_forward first");
  if (h->tape_weights_gen != h->weights_gen)
    return h->fail(BDIFF_ESTATE, "the weights changed after the training forward: its tape is stale");
  const int B = h->tape_B, N = h->tape_N, L = h->cfg.n_layers;
  const long long E = h->tape_E, ntiles = (E + CT - 1) / CT;
  ClfTape t{};
  tape_carve(static_cast<unsigned char*>(h->tape), L, N, B, t);
  ClfBwdScratch b{};
  cudaError_t e = grow_buf(h->bws, h->bws_bytes, bws_carve(nullptr, N, B, E, b));
  if (e != cudaSuccess) return h->fail(BDIFF_ENOMEM, "backward scratch: %s", cudaGetErrorString(e));
  bws_carve(static_cast<unsigned char*>(h->bws), N, B, E, b);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t nc = (size_t)N * CH;
  const int in3 = 2 * CH + (h->cfg.node_attr ? CIN : 0);
  auto G = [&](const std::string& name) { return grad_flat + h->playout.at(name).first; };
  cudaMemsetAsync(grad_flat, 0, (size_t)h->pfloats * sizeof(float), st);     // the alignment gaps

  // readout: graph_dec, the molecule sum, node_dec (EGNN.forward :415-419)
  k_clf_bwd_readout<<<B, CH, 0, st>>>(d_pred, t.w, h->g, b.dWk, b.dS);
  wgrad(st, b.part, d_pred, 1, t.ws, CH, 1, CH, B, G("graph_dec.2.weight"), CH, 0, G("graph_dec.2.bias"), 1);
  wgrad(st, b.part, b.dWk, CH, t.s, CH, CH, CH, B, G("graph_dec.0.weight"), CH, 0, G("graph_dec.0.bias"), 1);
  const int node_grid = (N + NT - 1) / NT;
  ClfBwdDecArgs da{b.dS, t.q, t.mol_off, B, N, h->g, b.dY, b.dQd, b.dHa};
  k_clf_bwd_nodedec<<<node_grid, NODE_THREADS, 0, st>>>(da);
  wgrad(st, b.part, b.dY, CH, t.qs, CH, CH, CH, N, G("node_dec.2.weight"), CH, 0, G("node_dec.2.bias"), 1);
  wgrad(st, b.part, b.dQd, CH, t.h + L * nc, CH, CH, CH, N, G("node_dec.0.weight"), CH, 0, G("node_dec.0.bias"), 1);

  float *dHo = b.dHa, *dH = b.dHb;
  ClfBwdEdgeArgs ea{};
  ea.x = t.x; ea.dAgg = b.dAgg; ea.mol_off = t.mol_off; ea.pair_off = t.pair_off; ea.B = B; ea.E = E;
  ea.ntiles = (int)ntiles; ea.attention = h->cfg.attention;
  ea.A = b.A; ea.S = b.S; ea.DZ2 = b.DZ2; ea.DT = b.DT; ea.DZ1 = b.DZ1;
  const int edge_grid = (int)std::min<long long>(ntiles, h->num_sms);
  for (int l = L - 1; l >= 0; --l) {
    const std::string p = "gcl_" + std::to_string(l) + ".";
    const float* hl = t.h + l * nc;
    // node_mlp (E_GCL.node_model :318-328)
    ClfBwdNodeArgs nb{dHo, t.v + l * nc, N, h->layers[l], b.dV, dH, b.dAgg};
    k_clf_bwd_node<<<node_grid, NODE_THREADS, 0, st>>>(nb);
    wgrad(st, b.part, dHo, CH, t.u + l * nc, CH, CH, CH, N, G(p + "node_mlp.2.weight"), CH, 0, G(p + "node_mlp.2.bias"), 1);
    wgrad(st, b.part, b.dV, CH, hl, CH, CH, CH, N, G(p + "node_mlp.0.weight"), in3, 0, G(p + "node_mlp.0.bias"), 1);
    wgrad(st, b.part, b.dV, CH, t.agg + l * nc, CH, CH, CH, N, G(p + "node_mlp.0.weight"), in3, CH, nullptr, 1);
    if (h->cfg.node_attr)
      wgrad(st, b.part, b.dV, CH, t.oh, CIN, CH, CIN, N, G(p + "node_mlp.0.weight"), in3, 2 * CH, nullptr, 1);
    // edge side (E_GCL.edge_model :306-316, the mask of E_GCL_mask.forward :357)
    ea.P = t.P + l * nc; ea.Q = t.Q + l * nc; ea.w = h->layers[l]; ea.W2Ts = h->w2tbuf + (size_t)l * W2_BYTES;
    k_clf_bwd_edge<<<edge_grid, EDGE_THREADS, BWD_EDGE_SMEM, st>>>(ea);
    if (h->cfg.attention)
      wgrad(st, b.part, b.DT, 1, b.S, CH, 1, CH, E, G(p + "att_mlp.0.weight"), CH, 0, G(p + "att_mlp.0.bias"), 1);
    wgrad(st, b.part, b.DZ2, CH, b.A, CH, CH, CH, E, G(p + "edge_mlp.2.weight"), CH, 0, G(p + "edge_mlp.2.bias"), 1);
    k_clf_bwd_pairs<<<N, CH, 0, st>>>(b.DZ1, t.x, t.mol_off, t.pair_off, B, b.dP, b.dQ, b.R);
    float* w1 = G(p + "edge_mlp.0.weight");
    wgrad(st, b.part, b.dP, CH, hl, CH, CH, CH, N, w1, 2 * CH + 1, 0, G(p + "edge_mlp.0.bias"), 1);
    wgrad(st, b.part, b.dQ, CH, hl, CH, CH, CH, N, w1, 2 * CH + 1, CH, nullptr, 1);
    wgrad(st, b.part, b.R, CH, nullptr, 0, CH, 0, N, nullptr, 0, 0, w1 + 2 * CH, 2 * CH + 1);
    k_clf_bwd_dh_edge<<<node_grid, NODE_THREADS, 0, st>>>(b.dP, b.dQ, N, h->layers[l], dH);
    std::swap(dHo, dH);
  }
  // embedding (EGNN.forward :407); h0 and x are data: no input gradient
  wgrad(st, b.part, dHo, CH, t.oh, CIN, CH, CIN, N, G("embedding.weight"), CIN, 0, G("embedding.bias"), 1);
  e = cudaGetLastError();
  if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "classifier training backward: %s", cudaGetErrorString(e));
  return BDIFF_OK;
}

}  // extern "C"
