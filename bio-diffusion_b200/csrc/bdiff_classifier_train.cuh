// bdiff_classifier_train.cuh — reverse sweep of the EGNN property classifier (the training pass; DESIGN §4d).
// Included by bdiff_classifier.cu after the forward kernels, whose constants, weight structs and tile helpers it reuses.
// The float64 formula sheet of every step is tests/classifier_backward.py:packed_backward.
//
// Per layer l, last to first (h' = h + W4 u + b4, u = silu(v), v = W3 [h | agg (| h0)] + b3):
//   k_clf_bwd_node    du = W4^T dh', dv = du * silu'(v), dh = dh' + W3h^T dv, dagg = W3a^T dv
//   k_clf_bwd_edge    per 128-pair tile: a = silu(z1) and z2 = W2 a + b2 recomputed (wgmma, as the forward), dm = dagg_i [i != j],
//                     back through the gate m = s g, g = sigmoid(w_att . s + b_att), s = silu(z2) -> dz2; da = W2^T dz2 on wgmma
//                     (split-bf16, W2^T slabs); dz1 = da * silu'(z1)
//   k_clf_bwd_pairs   dP_i = sum_j dz1_ij (row), dQ_j = sum_i dz1_ij (column), R_i = sum_j dz1_ij r_ij
//   k_clf_bwd_dh_edge dh += W1a^T dP + W1b^T dQ
// Every weight gradient is a sum over atoms or pairs of an outer product: k_clf_wgrad (fixed row chunks) + k_clf_wgrad_sum
// (chunks added in index order).  No atomics anywhere: the gradients are bit-reproducible.
#pragma once

namespace bdiff {

__device__ __forceinline__ float dsilu_acc(float z) {
  const float s = sigmoid_acc(z);
  return s * fmaf(z, 1.f - s, 1.f);
}

// acc[4 nodes][4 columns] += sIn[NT][ld] . Wt^T, i.e. acc[n][c] += sum_o sIn[n][o] Wt[c][o] (Wt [128][128], the forward's
// transposed weight read by rows): the product with the untransposed nn.Linear weight, W^T x.  One FMA chain in o order.
__device__ __forceinline__ void tile_gemm_t(const float* __restrict__ sIn, int ld, const float* __restrict__ Wt,
                                            float (&acc)[4][4]) {
  const int n0 = (threadIdx.x >> 5) * 4, c0 = (threadIdx.x & 31) * 4;
  for (int o = 0; o < CH; o += 4) {
    float4 w[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) w[q] = __ldg(reinterpret_cast<const float4*>(Wt + (size_t)(c0 + q) * CH + o));
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      const float4 s = *reinterpret_cast<const float4*>(sIn + (n0 + n) * ld + o);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        acc[n][q] = fmaf(s.x, w[q].x, acc[n][q]);
        acc[n][q] = fmaf(s.y, w[q].y, acc[n][q]);
        acc[n][q] = fmaf(s.z, w[q].z, acc[n][q]);
        acc[n][q] = fmaf(s.w, w[q].w, acc[n][q]);
      }
    }
  }
}
// global rows [node0, node0 + NT) of src (leading dim 128) -> sDst (leading dim K3_MAX); rows past N are zero
__device__ __forceinline__ void tile_load(const float* __restrict__ src, float* sDst, int node0, int N) {
  for (int i = threadIdx.x; i < NT * (CH / 4); i += NODE_THREADS) {
    const int n = i / (CH / 4), c = (i % (CH / 4)) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (node0 + n < N) v = *reinterpret_cast<const float4*>(src + (size_t)(node0 + n) * CH + c);
    *reinterpret_cast<float4*>(sDst + n * K3_MAX + c) = v;
  }
}
// acc[n][q] *= silu'(z) with z the global pre-activation tape
__device__ __forceinline__ void acc_dsilu(float (&acc)[4][4], const float* __restrict__ z, int node0, int N) {
  const int n0 = (threadIdx.x >> 5) * 4, c0 = (threadIdx.x & 31) * 4;
#pragma unroll
  for (int n = 0; n < 4; ++n) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (node0 + n0 + n < N) v = *reinterpret_cast<const float4*>(z + (size_t)(node0 + n0 + n) * CH + c0);
    acc[n][0] *= dsilu_acc(v.x);
    acc[n][1] *= dsilu_acc(v.y);
    acc[n][2] *= dsilu_acc(v.z);
    acc[n][3] *= dsilu_acc(v.w);
  }
}
__device__ __forceinline__ int atom_mol(const int* __restrict__ mol_off, int B, int i) {   // mol_off[k] <= i < mol_off[k+1]
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(mol_off + mid) <= i) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// ---------------------------------------------------------------------------------------------------- readout
// One CTA per molecule, thread c: dw = d_pred gd2 * silu'(w) (graph_dec.0 pre-activation), dS = gd1^T dw.
__global__ void __launch_bounds__(CH) k_clf_bwd_readout(const float* __restrict__ d_pred, const float* __restrict__ w_t,
                                                        ClfWeights g, float* __restrict__ dW, float* __restrict__ dS) {
  __shared__ float sw[CH];
  const int k = blockIdx.x, c = threadIdx.x;
  const float dw = d_pred[k] * g.gd2[c] * dsilu_acc(w_t[(size_t)k * CH + c]);
  dW[(size_t)k * CH + c] = dw;
  sw[c] = dw;
  __syncthreads();
  float s = 0.f;
  for (int o = 0; o < CH; ++o) s = fmaf(sw[o], __ldg(g.gd1t + (size_t)c * CH + o), s);
  dS[(size_t)k * CH + c] = s;
}

// node_dec: dy_i = dS_k(i) -> dY; dq = (nd2^T dy) * silu'(q) -> dQd; dh_L = nd1^T dq -> dH.
struct ClfBwdDecArgs {
  const float *dS, *q;
  const int* mol_off;
  int B, N;
  ClfWeights g;
  float *dY, *dQd, *dH;
};
__global__ void __launch_bounds__(NODE_THREADS) k_clf_bwd_nodedec(ClfBwdDecArgs a) {
  __shared__ __align__(16) float sIn[NT * K3_MAX];
  const int node0 = blockIdx.x * NT;
  for (int i = threadIdx.x; i < NT * (CH / 4); i += NODE_THREADS) {
    const int n = i / (CH / 4), c = (i % (CH / 4)) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (node0 + n < a.N) {
      v = *reinterpret_cast<const float4*>(a.dS + (size_t)atom_mol(a.mol_off, a.B, node0 + n) * CH + c);
      *reinterpret_cast<float4*>(a.dY + (size_t)(node0 + n) * CH + c) = v;
    }
    *reinterpret_cast<float4*>(sIn + n * K3_MAX + c) = v;
  }
  __syncthreads();
  float acc[4][4];
  acc_init(acc, nullptr);
  tile_gemm_t(sIn, K3_MAX, a.g.nd2t, acc);
  acc_dsilu(acc, a.q, node0, a.N);
  acc_out(acc, sIn + CH, false, a.dQd, node0, a.N);
  __syncthreads();
  acc_init(acc, nullptr);
  tile_gemm_t(sIn + CH, K3_MAX, a.g.nd1t, acc);
  acc_out(acc, nullptr, false, a.dH, node0, a.N);
}

// ---------------------------------------------------------------------------------------------------- node_mlp
struct ClfBwdNodeArgs {
  const float *dHo, *v;     // grad of the layer's output h', node_mlp.0 pre-activation
  int N;
  ClfLayer w;
  float *dV, *dH, *dAgg;    // dv; dh (before the edge terms); dagg
};
__global__ void __launch_bounds__(NODE_THREADS) k_clf_bwd_node(ClfBwdNodeArgs a) {
  __shared__ __align__(16) float sIn[NT * K3_MAX];
  const int node0 = blockIdx.x * NT;
  tile_load(a.dHo, sIn, node0, a.N);
  __syncthreads();
  float acc[4][4];
  acc_init(acc, nullptr);
  tile_gemm_t(sIn, K3_MAX, a.w.W4t, acc);
  acc_dsilu(acc, a.v, node0, a.N);
  acc_out(acc, sIn + CH, false, a.dV, node0, a.N);
  __syncthreads();
  {
    const int n0 = (threadIdx.x >> 5) * 4, c0 = (threadIdx.x & 31) * 4;
#pragma unroll
    for (int n = 0; n < 4; ++n)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[n][q] = sIn[(n0 + n) * K3_MAX + c0 + q];     // the residual: dh = dh' + ...
  }
  tile_gemm_t(sIn + CH, K3_MAX, a.w.W3t, acc);
  acc_out(acc, nullptr, false, a.dH, node0, a.N);
  acc_init(acc, nullptr);
  tile_gemm_t(sIn + CH, K3_MAX, a.w.W3t + (size_t)CH * CH, acc);
  acc_out(acc, nullptr, false, a.dAgg, node0, a.N);
}

// dH += W1a^T dP + W1b^T dQ (the node-level products of edge_mlp.0's h_i / h_j blocks)
__global__ void __launch_bounds__(NODE_THREADS) k_clf_bwd_dh_edge(const float* __restrict__ dP, const float* __restrict__ dQ,
                                                                  int N, ClfLayer w, float* __restrict__ dH) {
  __shared__ __align__(16) float sIn[NT * K3_MAX];
  const int node0 = blockIdx.x * NT;
  tile_load(dP, sIn, node0, N);
  tile_load(dQ, sIn + CH, node0, N);
  __syncthreads();
  float acc[4][4];
  {
    const int n0 = (threadIdx.x >> 5) * 4, c0 = (threadIdx.x & 31) * 4;
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (node0 + n0 + n < N) v = *reinterpret_cast<const float4*>(dH + (size_t)(node0 + n0 + n) * CH + c0);
      acc[n][0] = v.x; acc[n][1] = v.y; acc[n][2] = v.z; acc[n][3] = v.w;
    }
  }
  tile_gemm_t(sIn, K3_MAX, w.Pt, acc);
  tile_gemm_t(sIn + CH, K3_MAX, w.Qt, acc);
  acc_out(acc, nullptr, false, dH, node0, N);
}

// ---------------------------------------------------------------------------------------------------- edge tile
struct ClfBwdEdgeArgs {
  const float *x, *P, *Q, *dAgg;
  const int* mol_off;
  const long long* pair_off;
  int B;
  long long E;
  int ntiles;
  ClfLayer w;
  const unsigned char* W2Ts;     // W2^T as split-bf16 slabs
  int attention;
  float *A, *S, *DZ2, *DT, *DZ1; // per pair: a, s (attention only), dz2, the gate's dt (attention only), dz1
};
struct ClfBwdEdgeSmall {
  float b2[CH], watt[CH], wr[CH];
  int row[CT], col[CT], keep[CT];
  float rad[CT];
};
constexpr size_t BWD_EDGE_SMEM = A_BYTES + 2 * W2_BYTES + sizeof(ClfBwdEdgeSmall) + 1024;

// fragment pair (row r, columns c, c + 1; c even) -> split-bf16 A tile
__device__ __forceinline__ void x_store2_hl(unsigned char* X, int r, int c, float v0, float v1) {
  uint32_t hi, lo;
  split_bf16x2(v0, v1, hi, lo);
  const uint32_t off = sw128_offset(r, c & 63);
  *reinterpret_cast<uint32_t*>(X + (c >> 6) * X_BLOCK + off) = hi;
  *reinterpret_cast<uint32_t*>(X + (2 + (c >> 6)) * X_BLOCK + off) = lo;
}

// d (+)= A . B^T over K = 128: A the split-bf16 tile X (this warpgroup's 64 rows), B the slabs at wb
__device__ __forceinline__ void clf_gemm128(float (&d)[64], uint32_t xa, uint32_t wb) {
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
}

__global__ void __launch_bounds__(EDGE_THREADS, 1) k_clf_bwd_edge(ClfBwdEdgeArgs a) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* X = smem;
  unsigned char* W2 = smem + A_BYTES;
  unsigned char* W2T = W2 + W2_BYTES;
  ClfBwdEdgeSmall& S = *reinterpret_cast<ClfBwdEdgeSmall*>(W2T + W2_BYTES);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  {
    const uint4* s0 = reinterpret_cast<const uint4*>(a.w.W2s);
    const uint4* s1 = reinterpret_cast<const uint4*>(a.W2Ts);
    uint4* d0 = reinterpret_cast<uint4*>(W2);
    uint4* d1 = reinterpret_cast<uint4*>(W2T);
    for (int i = tid; i < W2_BYTES / 16; i += EDGE_THREADS) { d0[i] = s0[i]; d1[i] = s1[i]; }
    for (int i = tid; i < CH; i += EDGE_THREADS) {
      S.b2[i] = a.w.b2[i];
      S.watt[i] = a.attention ? a.w.watt[i] : 0.f;
      S.wr[i] = a.w.wr[i];
    }
  }
  const float batt = a.attention ? a.w.batt[0] : 0.f;
  const int wg = tid >> 7;
  const uint32_t xa = smem_u32(X) + (uint32_t)wg * 8192u;
  __syncthreads();

  for (int tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
    // ---- a_ij = silu(z1), exactly the forward's arithmetic -> A tile and the per-pair record a
    {
      const int cb = (lane & 15) * 8;
      for (int it = 0; it < 8; ++it) {
        const int r = warp * 16 + 2 * it + (lane >> 4);
        const long long e = (long long)tile * CT + r;
        float v[8];
        int gi = -1, gj = -1, keep = 0;
        float rad = 0.f;
        if (e < a.E) {
          const int k = find_mol(a.pair_off, a.B, e);
          const int n0 = __ldg(a.mol_off + k), n = __ldg(a.mol_off + k + 1) - n0;
          const int loc = (int)(e - __ldg(a.pair_off + k));
          const int i = loc / n, j = loc - i * n;
          gi = n0 + i;
          gj = n0 + j;
          keep = i != j;
          const float dx = a.x[gi * 3] - a.x[gj * 3], dy = a.x[gi * 3 + 1] - a.x[gj * 3 + 1], dz = a.x[gi * 3 + 2] - a.x[gj * 3 + 2];
          rad = dx * dx + dy * dy + dz * dz;
          const float4* pi = reinterpret_cast<const float4*>(a.P + (size_t)gi * CH + cb);
          const float4* qj = reinterpret_cast<const float4*>(a.Q + (size_t)gj * CH + cb);
          const float4 p0 = pi[0], p1 = pi[1], q0 = qj[0], q1 = qj[1];
          const float p[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
          const float q[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
          for (int c = 0; c < 8; ++c) v[c] = silu_acc(fmaf(S.wr[cb + c], rad, p[c] + q[c]));
          float4* ad = reinterpret_cast<float4*>(a.A + (size_t)e * CH + cb);
          ad[0] = make_float4(v[0], v[1], v[2], v[3]);
          ad[1] = make_float4(v[4], v[5], v[6], v[7]);
        } else {
#pragma unroll
          for (int c = 0; c < 8; ++c) v[c] = 0.f;
        }
        x_store8_hl(X, 2, r, cb, v);
        if ((lane & 15) == 0) {
          S.row[r] = gi;
          S.col[r] = gj;
          S.keep[r] = keep;
          S.rad[r] = rad;
        }
      }
    }
    fence_proxy_async();
    __syncthreads();

    // ---- z2 = a . W2^T + b2; back through m = s g to dz2
    float d[64];
    clf_gemm128(d, xa, smem_u32(W2));
    int rows[2];
    long long es[2];
#pragma unroll
    for (int r8 = 0; r8 < 2; ++r8) {
      rows[r8] = frag_row(wg, 2 * r8);
      es[r8] = (long long)tile * CT + rows[r8];
    }
    float att[2] = {0.f, 0.f}, sd[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 64; j += 2) {
      const int c = frag_col(j), r8 = (j >> 1) & 1;
      const int gi = S.row[rows[r8]];
      float2 dm = make_float2(0.f, 0.f);
      if (gi >= 0 && S.keep[rows[r8]]) dm = *reinterpret_cast<const float2*>(a.dAgg + (size_t)gi * CH + c);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float z = d[j + h] + S.b2[c + h];
        const float s = silu_acc(z);
        att[r8] = fmaf(S.watt[c + h], s, att[r8]);
        sd[r8] = fmaf(h ? dm.y : dm.x, s, sd[r8]);
      }
    }
#pragma unroll
    for (int r8 = 0; r8 < 2; ++r8) {
      att[r8] += __shfl_xor_sync(0xffffffffu, att[r8], 1);
      att[r8] += __shfl_xor_sync(0xffffffffu, att[r8], 2);
      sd[r8] += __shfl_xor_sync(0xffffffffu, sd[r8], 1);
      sd[r8] += __shfl_xor_sync(0xffffffffu, sd[r8], 2);
    }
    float gate[2], dt[2];
#pragma unroll
    for (int r8 = 0; r8 < 2; ++r8) {
      const int rr = rows[r8];
      const bool keep = S.row[rr] >= 0 && S.keep[rr];
      gate[r8] = keep ? (a.attention ? sigmoid_acc(att[r8] + batt) : 1.f) : 0.f;
      dt[r8] = keep && a.attention ? sd[r8] * gate[r8] * (1.f - gate[r8]) : 0.f;
      if (a.attention && (lane & 3) == 0 && es[r8] < a.E) a.DT[es[r8]] = dt[r8];
    }
    __syncthreads();     // both warpgroups' wgmmas have read the A tile: it takes dz2
#pragma unroll
    for (int j = 0; j < 64; j += 2) {
      const int c = frag_col(j), r8 = (j >> 1) & 1, rr = rows[r8];
      const int gi = S.row[rr];
      float2 dm = make_float2(0.f, 0.f);
      if (gi >= 0 && S.keep[rr]) dm = *reinterpret_cast<const float2*>(a.dAgg + (size_t)gi * CH + c);
      float z[2], s[2], g2[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        z[h] = d[j + h] + S.b2[c + h];
        s[h] = silu_acc(z[h]);
        const float ds = fmaf(h ? dm.y : dm.x, gate[r8], dt[r8] * S.watt[c + h]);
        g2[h] = ds * dsilu_acc(z[h]);
      }
      if (es[r8] < a.E) {
        *reinterpret_cast<float2*>(a.DZ2 + (size_t)es[r8] * CH + c) = make_float2(g2[0], g2[1]);
        if (a.attention) *reinterpret_cast<float2*>(a.S + (size_t)es[r8] * CH + c) = make_float2(s[0], s[1]);
      }
      x_store2_hl(X, rr, c, g2[0], g2[1]);
    }
    fence_proxy_async();
    __syncthreads();

    // ---- da = dz2 . W2 on the tensor cores; dz1 = da * silu'(z1)
    clf_gemm128(d, xa, smem_u32(W2T));
#pragma unroll
    for (int j = 0; j < 64; j += 2) {
      const int c = frag_col(j), r8 = (j >> 1) & 1, rr = rows[r8];
      const int gi = S.row[rr], gj = S.col[rr];
      if (gi < 0) continue;
      const float2 p = *reinterpret_cast<const float2*>(a.P + (size_t)gi * CH + c);
      const float2 q = *reinterpret_cast<const float2*>(a.Q + (size_t)gj * CH + c);
      const float rad = S.rad[rr];
      const float z0 = fmaf(S.wr[c], rad, p.x + q.x), z1 = fmaf(S.wr[c + 1], rad, p.y + q.y);
      *reinterpret_cast<float2*>(a.DZ1 + (size_t)es[r8] * CH + c) = make_float2(d[j] * dsilu_acc(z0), d[j + 1] * dsilu_acc(z1));
    }
    __syncthreads();     // A tile and row records free for the next tile
  }
}

// One CTA per atom i of molecule k, thread c: dP_i = sum_j dz1_ij, dQ_i = sum_j dz1_ji, R_i = sum_j dz1_ij r_ij (j in order).
__global__ void __launch_bounds__(CH) k_clf_bwd_pairs(const float* __restrict__ DZ1, const float* __restrict__ x,
                                                      const int* __restrict__ mol_off, const long long* __restrict__ pair_off,
                                                      int B, float* __restrict__ dP, float* __restrict__ dQ,
                                                      float* __restrict__ R) {
  const int gi = blockIdx.x, c = threadIdx.x;
  const int k = atom_mol(mol_off, B, gi);
  const int n0 = mol_off[k], n = mol_off[k + 1] - n0, i = gi - n0;
  const float* base = DZ1 + (size_t)pair_off[k] * CH + c;
  float p = 0.f, q = 0.f, r = 0.f;
  for (int j = 0; j < n; ++j) {
    const int gj = n0 + j;
    const float dx = x[gi * 3] - x[gj * 3], dy = x[gi * 3 + 1] - x[gj * 3 + 1], dz = x[gi * 3 + 2] - x[gj * 3 + 2];
    const float rad = dx * dx + dy * dy + dz * dz;
    const float v = base[(size_t)(i * n + j) * CH];
    p += v;
    r = fmaf(v, rad, r);
    q += base[(size_t)(j * n + i) * CH];
  }
  dP[(size_t)gi * CH + c] = p;
  dQ[(size_t)gi * CH + c] = q;
  R[(size_t)gi * CH + c] = r;
}

// ---------------------------------------------------------------------------------------------------- weight gradients
// part[chunk][o][k] = sum over rows of the chunk (in order) of G[row][o] X[row][k], with column k = K of X read as 1 (the
// bias).  CTA tile 32 o x 32 k, 4 k per thread; rows staged 32 at a time.
struct ClfWgradArgs {
  const float* G;
  const float* X;
  int ldg, ldx, O, K;
  long long rows, chunk;
  float* part;
};
__global__ void __launch_bounds__(256) k_clf_wgrad(ClfWgradArgs a) {
  __shared__ float sG[32][33], sX[32][33];
  const int o0 = blockIdx.x * 32, k0 = blockIdx.y * 32, tid = threadIdx.x;
  const int ol = tid >> 3, kl = (tid & 7) * 4;
  const long long r0 = (long long)blockIdx.z * a.chunk, r1 = min(a.rows, r0 + a.chunk);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (long long rb = r0; rb < r1; rb += 32) {
    for (int i = tid; i < 32 * 32; i += 256) {
      const int rr = i >> 5, cc = i & 31;
      const long long row = rb + rr;
      const bool ok = row < r1;
      const int o = o0 + cc, k = k0 + cc;
      sG[rr][cc] = ok && o < a.O ? a.G[row * a.ldg + o] : 0.f;
      sX[rr][cc] = ok && k < a.K ? a.X[row * a.ldx + k] : (ok && k == a.K ? 1.f : 0.f);
    }
    __syncthreads();
#pragma unroll 8
    for (int rr = 0; rr < 32; ++rr) {
      const float gv = sG[rr][ol];
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[q] = fmaf(gv, sX[rr][kl + q], acc[q]);
    }
    __syncthreads();
  }
  const int o = o0 + ol;
  if (o >= a.O) return;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int k = k0 + kl + q;
    if (k <= a.K) a.part[((size_t)blockIdx.z * a.O + o) * (a.K + 1) + k] = acc[q];
  }
}
// dW[o * ldw + col0 + k] (k < K) and db[o * dbs] (k = K, if db) = sum over chunks in index order
__global__ void k_clf_wgrad_sum(const float* __restrict__ part, int nchunks, int O, int K, float* __restrict__ dW, int ldw,
                                int col0, float* __restrict__ db, int dbs) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= O * (K + 1)) return;
  const int o = idx / (K + 1), k = idx - o * (K + 1);
  float s = 0.f;
  for (int c = 0; c < nchunks; ++c) s += part[((size_t)c * O + o) * (K + 1) + k];
  if (k < K) dW[(size_t)o * ldw + col0 + k] = s;
  else if (db) db[(size_t)o * dbs] = s;
}

}  // namespace bdiff
