// bdiff_kernels_fp32.cu — parity-mode (fp32 FFMA) kernels of the GCPNet denoiser hot path.
//
// One forward = prep_nodes -> node_frames -> edge_embed -> node_embed -> L x (edge_message, node_update)
// -> finalize.  The edge list is implicit (Plan): edge g of molecule k is (act[a], act[b]) with
// a = (g - edge_off[k]) / nact, b = (g - edge_off[k]) % nact — the (row, col)-sorted order of
// gcpnet.py:1054-1066.  Reference citations are relative to /root/reference/src/.
#include "bdiff_common.cuh"
#include "bdiff_kernels.h"
#include "bdiff_philox.cuh"

namespace bdiff {

// ============================================================================================ geometry
__device__ __forceinline__ void cross3(const float* a, const float* b, float* o) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}

// Frame of edge (r -> c) from CENTRED positions: rows (d, c, d x c), both normalised by (|.| + 1).
// models/components/__init__.py:123-171 (localize, norm_x_diff=True).
__device__ __forceinline__ void edge_frame(const float* xr, const float* xc, float* f) {
  float d[3] = {xr[0] - xc[0], xr[1] - xc[1], xr[2] - xc[2]};
  float c[3];
  cross3(xr, xc, c);
  const float dn = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]) + 1.0f;
  const float cn = sqrtf(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]) + 1.0f;
  d[0] /= dn; d[1] /= dn; d[2] /= dn;
  c[0] /= cn; c[1] /= cn; c[2] /= cn;
  f[0] = d[0]; f[1] = d[1]; f[2] = d[2];
  f[3] = c[0]; f[4] = c[1]; f[5] = c[2];
  cross3(d, c, f + 6);
}

// v / |v| with 0/0 -> 0 (datamodules/components/helper.py:15-24).
__device__ __forceinline__ void unit3(const float* v, float* o) {
  const float n = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  if (n > 0.f) { o[0] = v[0] / n; o[1] = v[1] / n; o[2] = v[2] / n; }
  else { o[0] = 0.f; o[1] = 0.f; o[2] = 0.f; }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}

// Block-wide sum of up to 4 values with a fixed reduction tree (deterministic). blockDim = 128.
__device__ __forceinline__ void block_sum4(float* v, float (*red)[4]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = warp_sum(v[i]);
  __syncthreads();
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < 4; ++i) red[warp][i] = v[i];
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = (red[0][i] + red[1][i]) + (red[2][i] + red[3][i]);
}

// One CTA per molecule: mask xh, split, centroid, centred x, orientations, time/context columns.
// gcpnet.py:1081-1166; edm_dataset.py:42-76; protein_graph_dataset.py:217-225; __init__.py:46-98.
__global__ void __launch_bounds__(128) k_prep_nodes(Plan p, Dims d, const float* __restrict__ xh,
                                                    const float* __restrict__ t_nodes,
                                                    const float* __restrict__ coef_table,
                                                    const int* __restrict__ step_ptr,
                                                    const float* __restrict__ ctx, Work w) {
  __shared__ float red[4][4];
  const int k = blockIdx.x;
  const int n0 = p.mol_off[k], n1 = p.mol_off[k + 1];
  const int ld = 3 + d.F;
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    const float m = p.mask[i] ? 1.f : 0.f;
    s[0] += xh[(size_t)i * ld + 0] * m;
    s[1] += xh[(size_t)i * ld + 1] * m;
    s[2] += xh[(size_t)i * ld + 2] * m;
    s[3] += m;
  }
  block_sum4(s, red);
  const float cx = s[3] > 0.f ? s[0] / s[3] : 0.f;
  const float cy = s[3] > 0.f ? s[1] / s[3] : 0.f;
  const float cz = s[3] > 0.f ? s[2] / s[3] : 0.f;
  // uniform time of a sampler step: coef_table[4*step + 3]
  const float tu = t_nodes ? 0.f : __ldg(coef_table + 4 * (step_ptr ? __ldg(step_ptr) : 0) + 3);
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    const float m = p.mask[i] ? 1.f : 0.f;
    float x0[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) x0[a] = xh[(size_t)i * ld + a] * m;
    w.x_init[i * 3 + 0] = x0[0]; w.x_init[i * 3 + 1] = x0[1]; w.x_init[i * 3 + 2] = x0[2];
    w.x[i * 3 + 0] = x0[0] - cx * m;
    w.x[i * 3 + 1] = x0[1] - cy * m;
    w.x[i * 3 + 2] = x0[2] - cz * m;
    float* hi = w.h_in + (size_t)i * d.Hin;
    for (int f = 0; f < d.F; ++f) hi[f] = xh[(size_t)i * ld + 3 + f] * m;
    hi[d.F] = t_nodes ? t_nodes[i] : tu;
    for (int c = 0; c < d.C; ++c) hi[d.F + 1 + c] = ctx[(size_t)i * d.C + c];
    // orientations over the CONCATENATED atom list (neighbour may belong to another molecule)
    float fw[3] = {0.f, 0.f, 0.f}, bw[3] = {0.f, 0.f, 0.f};
    if (i + 1 < p.N) {
      const float mn = p.mask[i + 1] ? 1.f : 0.f;
      float dv[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) dv[a] = xh[(size_t)(i + 1) * ld + a] * mn - x0[a];
      unit3(dv, fw);
    }
    if (i > 0) {
      const float mn = p.mask[i - 1] ? 1.f : 0.f;
      float dv[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) dv[a] = xh[(size_t)(i - 1) * ld + a] * mn - x0[a];
      unit3(dv, bw);
    }
    float* ci = w.chi_in + (size_t)i * 6;
    ci[0] = fw[0]; ci[1] = fw[1]; ci[2] = fw[2];
    ci[3] = bw[0]; ci[4] = bw[1]; ci[5] = bw[2];
  }
  // reset the aggregate rows of this molecule (edge_message accumulates into them) and the NaN flag
  for (size_t j = (size_t)n0 * kMsg + threadIdx.x; j < (size_t)n1 * kMsg; j += 128) w.agg[j] = 0.f;
  if (k == 0 && threadIdx.x == 0) *w.nan_flag = 0;
}

// One warp per node: mean over the row's edges of the edge frames (node-side scalarize commutes with the
// mean because frames are frozen across layers: __init__.py:187,208-217; gcpnet.py:1169-1174).
__global__ void __launch_bounds__(256) k_node_frames(Plan p, Work w) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * 8 + warp;
  if (i >= p.N) return;
  float acc[9];
#pragma unroll
  for (int q = 0; q < 9; ++q) acc[q] = 0.f;
  int na = 0;
  if (p.mask[i]) {
    const int k = p.node_mol[i];
    const int a0 = p.act_off[k];
    na = p.act_off[k + 1] - a0;
    const float xi[3] = {w.x[i * 3], w.x[i * 3 + 1], w.x[i * 3 + 2]};
    for (int j = lane; j < na; j += 32) {
      const int c = p.act_idx[a0 + j];
      const float xj[3] = {w.x[c * 3], w.x[c * 3 + 1], w.x[c * 3 + 2]};
      float f[9];
      edge_frame(xi, xj, f);
#pragma unroll
      for (int q = 0; q < 9; ++q) acc[q] += f[q];
    }
  }
#pragma unroll
  for (int q = 0; q < 9; ++q) acc[q] = warp_sum(acc[q]);
  if (lane == 0) {
    const float inv = na > 0 ? 1.0f / (float)na : 0.f;
    float* o = w.fbar + (size_t)i * 12;
#pragma unroll
    for (int q = 0; q < 9; ++q) o[q] = na > 0 ? acc[q] / (float)na : 0.f;
    o[9] = 0.f; o[10] = 0.f; o[11] = 0.f;
    (void)inv;
  }
}

// ====================================================================================== edge embedding
constexpr int TME = 32;   // edges per CTA tile

struct EmbedSmem {
  float sA[TME][28];      // merged scalar input [e_raw | vnorm(Xd) | q(9)] padded
  float sO[TME][64];      // silu(scalar_out)  == embedded e
  float sVD[TME][48];     // vector_down output [Xd][3]
  float sGate[TME][16];
  float sXo[TME][48];     // embedded xi
  float sF[TME][12];
};

// Per tile of 32 edges: e_raw, xi_raw (un-centred x_init; edm_dataset.py:22-38), frames (centred x), then the
// edge embedding GCP2 (1,1)->(Ed,Xd) (gcpnet.py:584-590 with :418-491).  Writes e, xi, frames.
__global__ void __launch_bounds__(kThreads) k_edge_embed(Plan p, Dims d, EmbedW ew, Work w) {
  __shared__ EmbedSmem S;
  const int tid = threadIdx.x;
  const long long g0 = (long long)blockIdx.x * TME;
  if (tid < TME) {
    const long long g = g0 + tid;
    float xiraw[3] = {0.f, 0.f, 0.f}, eraw = 0.f;
    float f[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) f[q] = 0.f;
    if (g < p.E) {
      const int k = find_mol(p.edge_off, p.B, g);
      const int loc = (int)(g - p.edge_off[k]);
      const int a0 = p.act_off[k], na = p.act_off[k + 1] - a0;
      const int a = loc / na, b = loc - a * na;
      const int row = p.act_idx[a0 + a], col = p.act_idx[a0 + b];
      float dv[3];
#pragma unroll
      for (int q = 0; q < 3; ++q) dv[q] = w.x_init[row * 3 + q] - w.x_init[col * 3 + q];
      eraw = dv[0] * dv[0] + dv[1] * dv[1] + dv[2] * dv[2];
      unit3(dv, xiraw);
      const float xr[3] = {w.x[row * 3], w.x[row * 3 + 1], w.x[row * 3 + 2]};
      const float xc[3] = {w.x[col * 3], w.x[col * 3 + 1], w.x[col * 3 + 2]};
      edge_frame(xr, xc, f);
    }
#pragma unroll
    for (int q = 0; q < 9; ++q) S.sF[tid][q] = f[q];
    S.sA[tid][0] = eraw;
    for (int h = 0; h < d.Xd; ++h) {
      const float wd = __ldg(ew.ewd + h);
      const float v0 = wd * xiraw[0], v1 = wd * xiraw[1], v2 = wd * xiraw[2];
      S.sVD[tid][h * 3 + 0] = v0; S.sVD[tid][h * 3 + 1] = v1; S.sVD[tid][h * 3 + 2] = v2;
      S.sA[tid][1 + h] = safe_norm3(v0, v1, v2);
    }
    for (int ch = 0; ch < 3; ++ch) {
      const float wf = __ldg(ew.ewf + ch);
      const float v0 = wf * xiraw[0], v1 = wf * xiraw[1], v2 = wf * xiraw[2];
      for (int a = 0; a < 3; ++a)
        S.sA[tid][1 + d.Xd + ch * 3 + a] = f[a * 3] * v0 + f[a * 3 + 1] * v1 + f[a * 3 + 2] * v2;
    }
    for (int j = 1 + d.Xd + 9; j < d.Ke; ++j) S.sA[tid][j] = 0.f;
  }
  __syncthreads();
  small_linear<TME>(&S.sA[0][0], 28, d.Ke, ew.eWs, ew.ebs, d.Ed, &S.sO[0][0], 64, 1);
  __syncthreads();
  small_linear<TME>(&S.sO[0][0], 64, d.Ed, ew.eWg, ew.ebg, d.Xd, &S.sGate[0][0], 16, 2);
  __syncthreads();
  vec_up_gate<TME>(&S.sXo[0][0], 48, &S.sVD[0][0], 48, d.Xd, ew.eWu, d.Xd, &S.sGate[0][0], 16, false);
  __syncthreads();
  // coalesced tile stores (buffers are padded to whole tiles)
  for (int idx = tid; idx < TME * d.Ed; idx += kThreads) {
    const int r = idx / d.Ed, c = idx - r * d.Ed;
    w.e[(size_t)(g0 + r) * d.Ed + c] = S.sO[r][c];
  }
  const int xw = d.Xd * 3;
  for (int idx = tid; idx < TME * xw; idx += kThreads) {
    const int r = idx / xw, c = idx - r * xw;
    w.xi[(size_t)(g0 + r) * xw + c] = S.sXo[r][c];
  }
  for (int idx = tid; idx < TME * 9; idx += kThreads) {
    const int r = idx / 9, c = idx - r * 9;
    w.frames[(size_t)(g0 + r) * 9 + c] = S.sF[r][c];
  }
}

// Thread-per-edge variant for the shipped dims (everything in registers, weights broadcast from shared memory).
// Uses  vector_up(vector_down(xi))[o][x] = (sum_h Wu[h][o] wd[h]) * xi[x]  (the input has a single vector channel).
template <int ED, int XD>
__global__ void __launch_bounds__(128) k_edge_embed_tpe(Plan p, EmbedW ew, Work w) {
  constexpr int KE = 1 + XD + 9;
  __shared__ float sWs[KE * ED], sbs[ED], swd[XD], swf[4], sWg[ED * XD], sbg[XD], sUd[XD];
  const int tid = threadIdx.x;
  for (int i = tid; i < KE * ED; i += 128) sWs[i] = ew.eWs[i];
  for (int i = tid; i < ED; i += 128) sbs[i] = ew.ebs[i];
  for (int i = tid; i < ED * XD; i += 128) sWg[i] = ew.eWg[i];
  if (tid < XD) {
    swd[tid] = ew.ewd[tid];
    sbg[tid] = ew.ebg[tid];
    float a = 0.f;
    for (int h = 0; h < XD; ++h) a = fmaf(ew.eWu[h * XD + tid], ew.ewd[h], a);
    sUd[tid] = a;
  }
  if (tid < 3) swf[tid] = ew.ewf[tid];
  __syncthreads();
  const long long g = (long long)blockIdx.x * 128 + tid;
  float xiraw[3] = {0.f, 0.f, 0.f}, eraw = 0.f, f[9];
#pragma unroll
  for (int q = 0; q < 9; ++q) f[q] = 0.f;
  if (g < p.E) {
    const int k = find_mol(p.edge_off, p.B, g);
    const int loc = (int)(g - p.edge_off[k]);
    const int a0 = p.act_off[k], na = p.act_off[k + 1] - a0;
    const int a = loc / na, b = loc - a * na;
    const int row = p.act_idx[a0 + a], col = p.act_idx[a0 + b];
    float dv[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) dv[q] = w.x_init[row * 3 + q] - w.x_init[col * 3 + q];
    eraw = dv[0] * dv[0] + dv[1] * dv[1] + dv[2] * dv[2];
    unit3(dv, xiraw);
    const float xr[3] = {w.x[row * 3], w.x[row * 3 + 1], w.x[row * 3 + 2]};
    const float xc[3] = {w.x[col * 3], w.x[col * 3 + 1], w.x[col * 3 + 2]};
    edge_frame(xr, xc, f);
  }
  float mg[KE];
  mg[0] = eraw;
#pragma unroll
  for (int h = 0; h < XD; ++h) {
    const float wd = swd[h];
    mg[1 + h] = safe_norm3(wd * xiraw[0], wd * xiraw[1], wd * xiraw[2]);
  }
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float wf = swf[ch];
    const float v0 = wf * xiraw[0], v1 = wf * xiraw[1], v2 = wf * xiraw[2];
#pragma unroll
    for (int a = 0; a < 3; ++a) mg[1 + XD + ch * 3 + a] = f[a * 3] * v0 + f[a * 3 + 1] * v1 + f[a * 3 + 2] * v2;
  }
  float S[ED];
#pragma unroll
  for (int o = 0; o < ED; ++o) S[o] = sbs[o];
#pragma unroll
  for (int k = 0; k < KE; ++k) {
#pragma unroll
    for (int o4 = 0; o4 < ED; o4 += 4) {
      const float4 wv = *reinterpret_cast<const float4*>(&sWs[k * ED + o4]);
      S[o4 + 0] = fmaf(mg[k], wv.x, S[o4 + 0]);
      S[o4 + 1] = fmaf(mg[k], wv.y, S[o4 + 1]);
      S[o4 + 2] = fmaf(mg[k], wv.z, S[o4 + 2]);
      S[o4 + 3] = fmaf(mg[k], wv.w, S[o4 + 3]);
    }
  }
  float gate[XD];
#pragma unroll
  for (int j = 0; j < XD; ++j) gate[j] = sbg[j];
  float* eo = w.e + (size_t)g * ED;
#pragma unroll
  for (int o4 = 0; o4 < ED; o4 += 4) {
    float4 sv;
    sv.x = siluf_(S[o4 + 0]); sv.y = siluf_(S[o4 + 1]); sv.z = siluf_(S[o4 + 2]); sv.w = siluf_(S[o4 + 3]);
    *reinterpret_cast<float4*>(eo + o4) = sv;
    const float se[4] = {sv.x, sv.y, sv.z, sv.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j4 = 0; j4 < XD; j4 += 4) {
        const float4 wg = *reinterpret_cast<const float4*>(&sWg[(o4 + i) * XD + j4]);
        gate[j4 + 0] = fmaf(se[i], wg.x, gate[j4 + 0]);
        gate[j4 + 1] = fmaf(se[i], wg.y, gate[j4 + 1]);
        gate[j4 + 2] = fmaf(se[i], wg.z, gate[j4 + 2]);
        gate[j4 + 3] = fmaf(se[i], wg.w, gate[j4 + 3]);
      }
  }
  float xo[XD * 3];
#pragma unroll
  for (int j = 0; j < XD; ++j) {
    const float s = sUd[j] * sigmoidf_(gate[j]);
    xo[j * 3 + 0] = s * xiraw[0]; xo[j * 3 + 1] = s * xiraw[1]; xo[j * 3 + 2] = s * xiraw[2];
  }
  float* xop = w.xi + (size_t)g * (XD * 3);
#pragma unroll
  for (int c4 = 0; c4 < XD * 3; c4 += 4) *reinterpret_cast<float4*>(xop + c4) = make_float4(xo[c4], xo[c4 + 1], xo[c4 + 2], xo[c4 + 3]);
  float* fo = w.frames + (size_t)g * 9;
#pragma unroll
  for (int q = 0; q < 9; ++q) fo[q] = f[q];
}

// ================================================================================= fused edge message
struct EdgeSmem {
  float sA[TME][284];     // A operand: stage 0 [e | vn | q], stages 1..3 [m.s(256) | vn(8) | q(9) | pad]
  float sO[TME][260];     // silu(scalar_out) of the current GCP (input of the vector gate)
  float sMV[TME][96];     // running vector message m.v [32][3]
  float sVD[TME][60];     // vector_down output [hid][3]
  float sVDF[TME][12];    // vector_down_frames output [3][3]
  float sXi[TME][48];
  float sF[TME][12];
  float sGate[TME][32];
  float sAttn[TME];
  int sRow[TME], sCol[TME], sB[TME], sNa[TME];
  float sW[2][kKC * 256];
  uint64_t bar[2];
};

// Fused per-edge message MLP (4 residual GCP2s) + attention gate + segmented row-sum.
// gcpnet.py:676-737 (GCPMessagePassing.message/aggregate) with GCP2.forward :418-491 per stage.
__global__ void __launch_bounds__(kThreads, 1) k_edge_message(Plan p, Dims d, LayerW lw, Work w) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  EdgeSmem& S = *reinterpret_cast<EdgeSmem*>(smem_raw);
  const int tid = threadIdx.x;
  const int tx = tid & 63, ty = tid >> 6;
  const long long g0 = (long long)blockIdx.x * TME;
  if (tid == 0) {
    mbar_init(&S.bar[0], 1);
    mbar_init(&S.bar[1], 1);
    mbar_fence_init();
  }
  if (tid < TME) {
    const long long g = g0 + tid;
    int row = -1, col = -1, b = 0, na = 0;
    if (g < p.E) {
      const int k = find_mol(p.edge_off, p.B, g);
      const int loc = (int)(g - p.edge_off[k]);
      const int a0 = p.act_off[k];
      na = p.act_off[k + 1] - a0;
      const int a = loc / na;
      b = loc - a * na;
      row = p.act_idx[a0 + a];
      col = p.act_idx[a0 + b];
    }
    S.sRow[tid] = row; S.sCol[tid] = col; S.sB[tid] = b; S.sNa[tid] = na;
  }
  // tile loads (buffers are padded to whole tiles and zero-initialised, so no bounds checks)
  for (int idx = tid; idx < TME * d.Ed; idx += kThreads) {
    const int r = idx / d.Ed, c = idx - r * d.Ed;
    S.sA[r][c] = w.e[(size_t)(g0 + r) * d.Ed + c];
  }
  const int xw = d.Xd * 3;
  for (int idx = tid; idx < TME * xw; idx += kThreads) {
    const int r = idx / xw, c = idx - r * xw;
    S.sXi[r][c] = w.xi[(size_t)(g0 + r) * xw + c];
  }
  for (int idx = tid; idx < TME * 9; idx += kThreads) {
    const int r = idx / 9, c = idx - r * 9;
    S.sF[r][c] = w.frames[(size_t)(g0 + r) * 9 + c];
  }
  __syncthreads();
  WStream ws{&S.sW[0][0], S.bar, 0u};

  // ---- stage 0: vector_down / vector_down_frames of [chi_row | xi | chi_col] in split form
  const int hid0 = d.hid0, per0 = hid0 * 3;
  for (int idx = tid; idx < TME * per0; idx += kThreads) {
    const int r = idx / per0, hx = idx - r * per0;
    const int h = hx / 3, x = hx - h * 3;
    const int row = S.sRow[r];
    float v = 0.f;
    if (row >= 0) v = w.PI[(size_t)row * kPStride + kH + hx] + w.PJ[(size_t)S.sCol[r] * kPStride + kH + hx];
    for (int c = 0; c < d.Xd; ++c) v = fmaf(__ldg(lw.Wd0x + c * hid0 + h), S.sXi[r][c * 3 + x], v);
    S.sVD[r][hx] = v;
  }
  for (int idx = tid; idx < TME * 9; idx += kThreads) {
    const int r = idx / 9, cx = idx - r * 9;
    const int ch = cx / 3, x = cx - ch * 3;
    const int row = S.sRow[r];
    float v = 0.f;
    if (row >= 0)
      v = w.PI[(size_t)row * kPStride + kH + per0 + cx] + w.PJ[(size_t)S.sCol[r] * kPStride + kH + per0 + cx];
    for (int c = 0; c < d.Xd; ++c) v = fmaf(__ldg(lw.Wf0x + c * 3 + ch), S.sXi[r][c * 3 + x], v);
    S.sVDF[r][cx] = v;
  }
  __syncthreads();
  norms_and_q<TME>(&S.sA[0][0], 284, d.Ed, d.K0, &S.sVD[0][0], 60, hid0, &S.sVDF[0][0], 12, &S.sF[0][0], 12);
  __syncthreads();
  {
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
    gemm256<8>(&S.sA[0][0], 284, d.K0, lw.W0e, ws, acc);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = ty * 8 + i;
      const int row = S.sRow[r];
      float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row >= 0) {
        const float4 pi = *reinterpret_cast<const float4*>(w.PI + (size_t)row * kPStride + tx * 4);
        const float4 pj = *reinterpret_cast<const float4*>(w.PJ + (size_t)S.sCol[r] * kPStride + tx * 4);
        o.x = siluf_(acc[i][0] + pi.x + pj.x);
        o.y = siluf_(acc[i][1] + pi.y + pj.y);
        o.z = siluf_(acc[i][2] + pi.z + pj.z);
        o.w = siluf_(acc[i][3] + pi.w + pj.w);
      }
      *reinterpret_cast<float4*>(&S.sO[r][tx * 4]) = o;
      *reinterpret_cast<float4*>(&S.sA[r][tx * 4]) = o;   // m.s = silu(S0)
    }
  }
  __syncthreads();
  small_linear<TME>(&S.sO[0][0], 260, kH, lw.Wg0, lw.bg0, kC, &S.sGate[0][0], 32, 2);
  __syncthreads();
  vec_up_gate<TME>(&S.sMV[0][0], 96, &S.sVD[0][0], 60, hid0, lw.Wu0, kC, &S.sGate[0][0], 32, false);
  __syncthreads();

  // ---- stages 1..3: residual GCP2s on the running message
  for (int k = 0; k < 3; ++k) {
    vec_down<TME>(&S.sVD[0][0], 60, &S.sMV[0][0], 96, kC, lw.Wdk[k], kHidM, false);
    vec_down<TME>(&S.sVDF[0][0], 12, &S.sMV[0][0], 96, kC, lw.Wfk[k], 3, false);
    __syncthreads();
    norms_and_q<TME>(&S.sA[0][0], 284, kH, kKM, &S.sVD[0][0], 60, kHidM, &S.sVDF[0][0], 12, &S.sF[0][0], 12);
    __syncthreads();
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
    gemm256<8>(&S.sA[0][0], 284, kKM, lw.Wk[k], ws, acc);
    const float4 bb = *reinterpret_cast<const float4*>(lw.bk[k] + tx * 4);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = ty * 8 + i;
      float4 o;
      o.x = siluf_(acc[i][0] + bb.x);
      o.y = siluf_(acc[i][1] + bb.y);
      o.z = siluf_(acc[i][2] + bb.z);
      o.w = siluf_(acc[i][3] + bb.w);
      *reinterpret_cast<float4*>(&S.sO[r][tx * 4]) = o;
      float4 m = *reinterpret_cast<float4*>(&S.sA[r][tx * 4]);
      m.x += o.x; m.y += o.y; m.z += o.z; m.w += o.w;
      *reinterpret_cast<float4*>(&S.sA[r][tx * 4]) = m;   // m.s += new.s
    }
    __syncthreads();
    small_linear<TME>(&S.sO[0][0], 260, kH, lw.Wgk[k], lw.bgk[k], kC, &S.sGate[0][0], 32, 2);
    __syncthreads();
    vec_up_gate<TME>(&S.sMV[0][0], 96, &S.sVD[0][0], 60, kHidM, lw.Wuk[k], kC, &S.sGate[0][0], 32, true);
    __syncthreads();
  }

  // ---- scalar message attention (gcpnet.py:709-711)
  row_dot<TME>(&S.sA[0][0], 284, kH, lw.wa, __ldg(lw.ba), S.sAttn, 2);
  __syncthreads();

  // ---- segmented sum over the source node (gcpnet.py:716-724).  Rows wholly inside the tile are stored,
  // rows cut by a tile boundary are accumulated with atomics (agg rows are zeroed beforehand).
  for (int c = tid; c < kMsg; c += kThreads) {
    float acc = 0.f;
    int cur = -1;
    bool first_ok = false;
    for (int r = 0; r < TME; ++r) {
      const int row = S.sRow[r];
      if (row < 0) break;
      if (row != cur) { cur = row; acc = 0.f; first_ok = (S.sB[r] == 0); }
      acc += (c < kH) ? S.sA[r][c] * S.sAttn[r] : S.sMV[r][c - kH];
      const bool last = (r == TME - 1) || (S.sRow[r + 1] != row);
      if (last) {
        float* dst = w.agg + (size_t)row * kMsg + c;
        if (first_ok && S.sB[r] == S.sNa[r] - 1) *dst = acc;
        else atomicAdd(dst, acc);
      }
    }
  }
}

// ======================================================================================== node kernels
constexpr int TMN = 16;   // nodes per CTA tile

struct NodeSmem {
  float sA[TMN][544];     // A operand (FF: [agg_s | h | vn | q]); later h_new in cols 0..255
  float sO[TMN][260];
  float sV[TMN][196];     // vectors [agg_v(96) | chi(96)]; later chi_new in cols 0..95
  float sVD[TMN][96];
  float sVDF[TMN][12];
  float sF[TMN][12];      // mean frame of the node's row
  float sGate[TMN][32];
  float sG1[TMN];
  float sMask[TMN];
  float sW[2][kKC * 256];
  uint64_t bar[2];
};

// Projections of the NEXT layer's message GCP 0 that only depend on one endpoint (split form of
// scalar_out / vector_down / vector_down_frames over [h_row | e | h_col], gcpnet.py:694,444-464).
__device__ __forceinline__ void stage_next(NodeSmem& S, const Dims& d, const LayerW& wn, Work& w, int n0,
                                           WStream& ws) {
  const int tid = threadIdx.x, tx = tid & 63, ty = tid >> 6;
  {
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
    gemm256<4>(&S.sA[0][0], 544, kH, wn.Wsi, ws, acc);
    const float4 bb = *reinterpret_cast<const float4*>(wn.b0 + tx * 4);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float4 o = make_float4(acc[i][0] + bb.x, acc[i][1] + bb.y, acc[i][2] + bb.z, acc[i][3] + bb.w);
      *reinterpret_cast<float4*>(w.PI + (size_t)(n0 + ty * 4 + i) * kPStride + tx * 4) = o;
    }
  }
  {
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
    gemm256<4>(&S.sA[0][0], 544, kH, wn.Wsj, ws, acc);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float4 o = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
      *reinterpret_cast<float4*>(w.PJ + (size_t)(n0 + ty * 4 + i) * kPStride + tx * 4) = o;
    }
  }
  const int per0 = d.hid0 * 3;
  vec_down<TMN>(w.PI + (size_t)n0 * kPStride + kH, kPStride, &S.sV[0][0], 196, kC, wn.Wd0i, d.hid0, false);
  vec_down<TMN>(w.PJ + (size_t)n0 * kPStride + kH, kPStride, &S.sV[0][0], 196, kC, wn.Wd0j, d.hid0, false);
  vec_down<TMN>(w.PI + (size_t)n0 * kPStride + kH + per0, kPStride, &S.sV[0][0], 196, kC, wn.Wf0i, 3, false);
  vec_down<TMN>(w.PJ + (size_t)n0 * kPStride + kH + per0, kPStride, &S.sV[0][0], 196, kC, wn.Wf0j, 3, false);
}

// Final scalar projection GCP2 (256,32)->(Hin,0), no activation (gcpnet.py:1025-1039,1191-1197).
__device__ __forceinline__ void stage_proj(NodeSmem& S, const Dims& d, const EmbedW& ew, Work& w, int n0) {
  vec_down<TMN>(&S.sVD[0][0], 96, &S.sV[0][0], 196, kC, ew.pWd, 32, false);
  vec_down<TMN>(&S.sVDF[0][0], 12, &S.sV[0][0], 196, kC, ew.pWf, 3, false);
  __syncthreads();
  norms_and_q<TMN>(&S.sA[0][0], 544, kH, 300, &S.sVD[0][0], 96, 32, &S.sVDF[0][0], 12, &S.sF[0][0], 12);
  __syncthreads();
  small_linear<TMN>(&S.sA[0][0], 544, 300, ew.pWs, ew.pbs, d.Hin, &S.sO[0][0], 260, 0);
  __syncthreads();
  for (int idx = threadIdx.x; idx < TMN * d.Hin; idx += kThreads) {
    const int r = idx / d.Hin, c = idx - r * d.Hin;
    w.hproj[(size_t)(n0 + r) * 32 + c] = S.sO[r][c];
  }
}

__device__ __forceinline__ void node_smem_init(NodeSmem& S) {
  if (threadIdx.x == 0) {
    mbar_init(&S.bar[0], 1);
    mbar_init(&S.bar[1], 1);
    mbar_fence_init();
  }
}

// Node embedding GCP2 (Hin,2)->(256,32), no activation, node_inputs=True (gcpnet.py:591-597), followed by the
// endpoint projections of layer 0.
__global__ void __launch_bounds__(kThreads, 2) k_node_embed(Plan p, Dims d, EmbedW ew, LayerW wn, Work w) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  NodeSmem& S = *reinterpret_cast<NodeSmem*>(smem_raw);
  const int tid = threadIdx.x, tx = tid & 63, ty = tid >> 6;
  const int n0 = blockIdx.x * TMN;
  node_smem_init(S);
  for (int idx = tid; idx < TMN * d.Hin; idx += kThreads) {
    const int r = idx / d.Hin, c = idx - r * d.Hin;
    S.sA[r][c] = w.h_in[(size_t)(n0 + r) * d.Hin + c];
  }
  for (int idx = tid; idx < TMN * 6; idx += kThreads) {
    const int r = idx / 6, c = idx - r * 6;
    S.sV[r][c] = w.chi_in[(size_t)(n0 + r) * 6 + c];
  }
  for (int idx = tid; idx < TMN * 12; idx += kThreads) {
    const int r = idx / 12, c = idx - r * 12;
    S.sF[r][c] = w.fbar[(size_t)(n0 + r) * 12 + c];
  }
  __syncthreads();
  WStream ws{&S.sW[0][0], S.bar, 0u};
  vec_down<TMN>(&S.sVD[0][0], 96, &S.sV[0][0], 196, 2, ew.nWd, 32, false);
  vec_down<TMN>(&S.sVDF[0][0], 12, &S.sV[0][0], 196, 2, ew.nWf, 3, false);
  __syncthreads();
  norms_and_q<TMN>(&S.sA[0][0], 544, d.Hin, d.Kn, &S.sVD[0][0], 96, 32, &S.sVDF[0][0], 12, &S.sF[0][0], 12);
  __syncthreads();
  {
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
    gemm256<4>(&S.sA[0][0], 544, d.Kn, ew.nWs, ws, acc);
    const float4 bb = *reinterpret_cast<const float4*>(ew.nbs + tx * 4);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = ty * 4 + i;
      float4 o = make_float4(acc[i][0] + bb.x, acc[i][1] + bb.y, acc[i][2] + bb.z, acc[i][3] + bb.w);
      *reinterpret_cast<float4*>(&S.sO[r][tx * 4]) = o;
      *reinterpret_cast<float4*>(&S.sA[r][tx * 4]) = o;
      *reinterpret_cast<float4*>(w.h + (size_t)(n0 + r) * kH + tx * 4) = o;
    }
  }
  __syncthreads();
  small_linear<TMN>(&S.sO[0][0], 260, kH, ew.nWg, ew.nbg, kC, &S.sGate[0][0], 32, 2);
  __syncthreads();
  vec_up_gate<TMN>(&S.sV[0][0], 196, &S.sVD[0][0], 96, 32, ew.nWu, kC, &S.sGate[0][0], 32, false);
  __syncthreads();
  for (int idx = tid; idx < TMN * 96; idx += kThreads) {
    const int r = idx / 96, c = idx - r * 96;
    w.chi[(size_t)(n0 + r) * 96 + c] = S.sV[r][c];
  }
  stage_next(S, d, wn, w, n0, ws);
  if (w.PJT) {     // tensor mode: the edge pass gathers the scalar part of P_j column-major (see Work::PJT)
    __syncthreads();
    for (int idx = tid; idx < TMN * kH; idx += kThreads) {
      const int c = idx / TMN, r = idx - c * TMN;
      const int n = n0 + r;
      w.PJT[((size_t)(n >> 5) * 256 + c) * 32 + (n & 31)] = w.PJ[(size_t)n * kPStride + c];
    }
  }
}

// Per layer, per node tile: feed-forward GCP2 on [aggregate | node], residual, mask, position-update GCP2,
// x += v, then either the next layer's endpoint projections or the final scalar projection.
// gcpnet.py:893-930 (GCPInteractions.forward), :834-857 (derive_x_update).
__global__ void __launch_bounds__(kThreads, 2) k_node_update(Plan p, Dims d, LayerW lw, LayerW wn, EmbedW ew,
                                                             Work w, int last) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  NodeSmem& S = *reinterpret_cast<NodeSmem*>(smem_raw);
  const int tid = threadIdx.x, tx = tid & 63, ty = tid >> 6;
  const int n0 = blockIdx.x * TMN;
  node_smem_init(S);
  for (int idx = tid; idx < TMN * 64; idx += kThreads) {       // 64 float4 per 256-wide row
    const int r = idx >> 6, c4 = (idx & 63) * 4;
    float* ag = w.agg + (size_t)(n0 + r) * kMsg + c4;
    *reinterpret_cast<float4*>(&S.sA[r][c4]) = *reinterpret_cast<const float4*>(ag);
    *reinterpret_cast<float4*>(ag) = make_float4(0.f, 0.f, 0.f, 0.f);    // reset for the next layer
    *reinterpret_cast<float4*>(&S.sA[r][kH + c4]) =
        *reinterpret_cast<const float4*>(w.h + (size_t)(n0 + r) * kH + c4);
  }
  for (int idx = tid; idx < TMN * 24; idx += kThreads) {       // 24 float4 per 96-wide row
    const int r = idx / 24, c4 = (idx - r * 24) * 4;
    float* ag = w.agg + (size_t)(n0 + r) * kMsg + kH + c4;
    *reinterpret_cast<float4*>(&S.sV[r][c4]) = *reinterpret_cast<const float4*>(ag);
    *reinterpret_cast<float4*>(ag) = make_float4(0.f, 0.f, 0.f, 0.f);
    *reinterpret_cast<float4*>(&S.sV[r][96 + c4]) =
        *reinterpret_cast<const float4*>(w.chi + (size_t)(n0 + r) * 96 + c4);
  }
  for (int idx = tid; idx < TMN * 12; idx += kThreads) {
    const int r = idx / 12, c = idx - r * 12;
    S.sF[r][c] = w.fbar[(size_t)(n0 + r) * 12 + c];
  }
  if (tid < TMN) S.sMask[tid] = (n0 + tid < p.N && p.mask[n0 + tid]) ? 1.f : 0.f;
  __syncthreads();
  WStream ws{&S.sW[0][0], S.bar, 0u};

  // ---- feed-forward GCP2 (512,64)->(256,32), feedforward_out, no activation, node_inputs
  vec_down<TMN>(&S.sVD[0][0], 96, &S.sV[0][0], 196, 2 * kC, lw.Wdf, kHidFF, false);
  vec_down<TMN>(&S.sVDF[0][0], 12, &S.sV[0][0], 196, 2 * kC, lw.Wff, 3, false);
  __syncthreads();
  norms_and_q<TMN>(&S.sA[0][0], 544, 2 * kH, kKFF, &S.sVD[0][0], 96, kHidFF, &S.sVDF[0][0], 12, &S.sF[0][0], 12);
  __syncthreads();
  {
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
    gemm256<4>(&S.sA[0][0], 544, kKFF, lw.W1, ws, acc);
    const float4 bb = *reinterpret_cast<const float4*>(lw.b1 + tx * 4);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = ty * 4 + i;
      float4 o = make_float4(siluf_(acc[i][0] + bb.x), siluf_(acc[i][1] + bb.y), siluf_(acc[i][2] + bb.z),
                             siluf_(acc[i][3] + bb.w));
      *reinterpret_cast<float4*>(&S.sO[r][tx * 4]) = o;
    }
  }
  __syncthreads();
  {
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
    gemm256<4>(&S.sO[0][0], 260, kH, lw.W2, ws, acc);
    const float4 bb = *reinterpret_cast<const float4*>(lw.b2 + tx * 4);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = ty * 4 + i;
      const float m = S.sMask[r];
      float4 z = make_float4(acc[i][0] + bb.x, acc[i][1] + bb.y, acc[i][2] + bb.z, acc[i][3] + bb.w);
      *reinterpret_cast<float4*>(&S.sO[r][tx * 4]) = z;              // gate input (identity nonlinearity)
      const float4 ho = *reinterpret_cast<const float4*>(&S.sA[r][kH + tx * 4]);
      float4 hn = make_float4((ho.x + z.x) * m, (ho.y + z.y) * m, (ho.z + z.z) * m, (ho.w + z.w) * m);
      *reinterpret_cast<float4*>(&S.sA[r][tx * 4]) = hn;             // residual + mask (gcpnet.py:907,914)
      *reinterpret_cast<float4*>(w.h + (size_t)(n0 + r) * kH + tx * 4) = hn;
    }
  }
  __syncthreads();
  small_linear<TMN>(&S.sO[0][0], 260, kH, lw.Wgf, lw.bgf, kC, &S.sGate[0][0], 32, 2);
  __syncthreads();
  for (int idx = tid; idx < TMN * 96; idx += kThreads) {
    const int r = idx / 96, ox = idx - r * 96;
    const int o = ox / 3, x = ox - o * 3;
    float s = 0.f;
    for (int h = 0; h < kHidFF; ++h) s = fmaf(__ldg(lw.Wuf + h * kC + o), S.sVD[r][h * 3 + x], s);
    const float cn = (S.sV[r][96 + ox] + s * S.sGate[r][o]) * S.sMask[r];
    S.sV[r][ox] = cn;
    w.chi[(size_t)(n0 + r) * 96 + ox] = cn;
  }
  __syncthreads();

  // ---- node position update GCP2 (256,32)->(256,1), silu/silu (gcpnet.py:828-857)
  vec_down<TMN>(&S.sVD[0][0], 96, &S.sV[0][0], 196, kC, lw.Wdp, kHidM, false);
  vec_down<TMN>(&S.sVDF[0][0], 12, &S.sV[0][0], 196, kC, lw.Wfp, 3, false);
  __syncthreads();
  norms_and_q<TMN>(&S.sA[0][0], 544, kH, kKM, &S.sVD[0][0], 96, kHidM, &S.sVDF[0][0], 12, &S.sF[0][0], 12);
  __syncthreads();
  {
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
    gemm256<4>(&S.sA[0][0], 544, kKM, lw.Wp, ws, acc);
    const float4 bb = *reinterpret_cast<const float4*>(lw.bp + tx * 4);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = ty * 4 + i;
      float4 o = make_float4(siluf_(acc[i][0] + bb.x), siluf_(acc[i][1] + bb.y), siluf_(acc[i][2] + bb.z),
                             siluf_(acc[i][3] + bb.w));
      *reinterpret_cast<float4*>(&S.sO[r][tx * 4]) = o;
    }
  }
  __syncthreads();
  row_dot<TMN>(&S.sO[0][0], 260, kH, lw.Wgp, __ldg(lw.bgp), S.sG1, 2);
  __syncthreads();
  if (tid < TMN * 3) {
    const int r = tid / 3, x = tid - r * 3;
    float s = 0.f;
    for (int h = 0; h < kHidM; ++h) s = fmaf(__ldg(lw.Wup + h), S.sVD[r][h * 3 + x], s);
    const int node = n0 + r;
    const float xn = (w.x[(size_t)node * 3 + x] + s * S.sG1[r]) * S.sMask[r];
    w.x[(size_t)node * 3 + x] = xn;
    if (xn != xn) atomicExch(w.nan_flag, 1);
  }
  __syncthreads();
  if (!last) stage_next(S, d, wn, w, n0, ws);
  else stage_proj(S, d, ew, w, n0);
}

// One CTA per molecule: vel = (x - x_init) * mask, NaN guard, centre, assemble net_out (gcpnet.py:1204-1230).
__global__ void __launch_bounds__(128) k_finalize(Plan p, Dims d, Work w, float* __restrict__ out) {
  __shared__ float red[4][4];
  const int k = blockIdx.x;
  const int n0 = p.mol_off[k], n1 = p.mol_off[k + 1];
  const bool bad = (*w.nan_flag) != 0;
  if (bad && k == 0 && threadIdx.x == 0) atomicAdd(w.nan_flag + 1, 1);     // cumulative NaN-guard hits (bdiff_nan_guard_count)
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    const float m = p.mask[i] ? 1.f : 0.f;
    if (!bad) {
      s[0] += (w.x[i * 3 + 0] - w.x_init[i * 3 + 0]) * m;
      s[1] += (w.x[i * 3 + 1] - w.x_init[i * 3 + 1]) * m;
      s[2] += (w.x[i * 3 + 2] - w.x_init[i * 3 + 2]) * m;
    }
    s[3] += m;
  }
  block_sum4(s, red);
  const float cx = s[3] > 0.f ? s[0] / s[3] : 0.f;
  const float cy = s[3] > 0.f ? s[1] / s[3] : 0.f;
  const float cz = s[3] > 0.f ? s[2] / s[3] : 0.f;
  const int ld = 3 + d.F;
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    const float m = p.mask[i] ? 1.f : 0.f;
    float v0 = 0.f, v1 = 0.f, v2 = 0.f;
    if (!bad) {
      v0 = (w.x[i * 3 + 0] - w.x_init[i * 3 + 0]) * m;
      v1 = (w.x[i * 3 + 1] - w.x_init[i * 3 + 1]) * m;
      v2 = (w.x[i * 3 + 2] - w.x_init[i * 3 + 2]) * m;
    }
    out[(size_t)i * ld + 0] = v0 - cx * m;
    out[(size_t)i * ld + 1] = v1 - cy * m;
    out[(size_t)i * ld + 2] = v2 - cz * m;
    for (int f = 0; f < d.F; ++f) out[(size_t)i * ld + 3 + f] = w.hproj[(size_t)i * 32 + f];
  }
}

// ============================================================================================ sampler
// One CTA per molecule.  mode 0 (reverse step, variational_diffusion.py:1247-1277):
//   z' = z / alpha_ts - c_eps * eps + sigma * noise_mc ; x-part of z' re-centred.          coef = {alpha_ts, c_eps, sigma, t}
// mode 1 (decode, :559-577,880-885): out = inv_alpha0 * (z - sigma0 * eps) + sigma_x * noise_mc.  coef = {inv_alpha0, sigma0, sigma_x, 0}
// mode 2: out = noise_mc (z_T).   noise_mc = raw randn masked, x-part centred per molecule (:795-819).
// mode 3 (jump back of inpaint, sample_p_zt_given_zs :1163-1201 indexing alpha_t|s by batch_index):
//   z' = alpha_t|s * z + sigma_t|s * noise_mc ; x-part of z' re-centred.                coef = {alpha_t|s, sigma_t|s, s, t}
__global__ void __launch_bounds__(128) k_step(Plan p, Dims d, int mode, const float* __restrict__ z,
                                              const float* __restrict__ eps, const float* __restrict__ noise_x,
                                              const float* __restrict__ noise_h,
                                              const float* __restrict__ coef_table,
                                              const int* __restrict__ step_ptr, float* __restrict__ out) {
  const float* coef = coef_table ? coef_table + 4 * (step_ptr ? __ldg(step_ptr) : 0) : nullptr;
  __shared__ float red[4][4];
  const int k = blockIdx.x;
  const int n0 = p.mol_off[k], n1 = p.mol_off[k + 1];
  const int ld = 3 + d.F;
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    const float m = p.mask[i] ? 1.f : 0.f;
    s[0] += noise_x[(size_t)i * 3 + 0] * m;
    s[1] += noise_x[(size_t)i * 3 + 1] * m;
    s[2] += noise_x[(size_t)i * 3 + 2] * m;
    s[3] += m;
  }
  block_sum4(s, red);
  const float cnt = s[3];
  const float ncx = cnt > 0.f ? s[0] / cnt : 0.f, ncy = cnt > 0.f ? s[1] / cnt : 0.f,
              ncz = cnt > 0.f ? s[2] / cnt : 0.f;
  const float c0 = mode == 2 ? 0.f : __ldg(coef + 0), c1 = mode == 2 ? 0.f : __ldg(coef + 1),
              c2 = mode == 2 ? 1.f : __ldg(coef + 2);
  float t[4] = {0.f, 0.f, 0.f, 0.f};
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    const float m = p.mask[i] ? 1.f : 0.f;
    const float nc[3] = {ncx, ncy, ncz};
    for (int c = 0; c < ld; ++c) {
      float nz = (c < 3 ? noise_x[(size_t)i * 3 + c] : noise_h[(size_t)i * d.F + (c - 3)]) * m;
      if (c < 3) nz -= nc[c] * m;
      float v;
      if (mode == 0) v = z[(size_t)i * ld + c] / c0 - c1 * eps[(size_t)i * ld + c] + c2 * nz;
      else if (mode == 1) v = c0 * (z[(size_t)i * ld + c] - c1 * eps[(size_t)i * ld + c]) + c2 * nz;
      else if (mode == 3) v = c0 * z[(size_t)i * ld + c] + c1 * nz;
      else v = nz;
      out[(size_t)i * ld + c] = v;
      if (c < 3) t[c] += v;
    }
  }
  if (mode == 1 || mode == 2) return;
  block_sum4(t, red);
  const float zx = cnt > 0.f ? t[0] / cnt : 0.f, zy = cnt > 0.f ? t[1] / cnt : 0.f, zz = cnt > 0.f ? t[2] / cnt : 0.f;
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    const float m = p.mask[i] ? 1.f : 0.f;
    out[(size_t)i * ld + 0] -= zx * m;
    out[(size_t)i * ld + 1] -= zy * m;
    out[(size_t)i * ld + 2] -= zz * m;
  }
}

// One CTA per molecule: the RePaint combination of inpaint (variational_diffusion.py:1659-1667, 1694-1713), applied after
// the reverse step has written z_unknown into z.  known = {alpha_s, sigma_s} = known_table[2 * *op_ptr]:
//   z_known = alpha_s * xh0 + sigma_s * noise_mc                      (compute_noised_representation, :910-931)
//   z_known.x += mean_fixed(z_unknown.x) - mean_fixed(z_known.x)      (per molecule)
//   z[fixed rows] = z_known                                           (z[free rows] stays z_unknown)
// A molecule without fixed atoms is left untouched.  Fixed-order reductions: the result is bit-reproducible.
__global__ void __launch_bounds__(128) k_repaint_combine(Plan p, Dims d, float* __restrict__ z,
                                                         const float* __restrict__ xh0,
                                                         const uint8_t* __restrict__ fixed,
                                                         const float* __restrict__ noise_x,
                                                         const float* __restrict__ noise_h,
                                                         const float* __restrict__ known_table,
                                                         const int* __restrict__ op_ptr) {
  __shared__ float red[4][4];
  const int k = blockIdx.x;
  const int n0 = p.mol_off[k], n1 = p.mol_off[k + 1];
  const int ld = 3 + d.F;
  const int op = __ldg(op_ptr);
  const float alpha = __ldg(known_table + 2 * op), sigma = __ldg(known_table + 2 * op + 1);
  // 1) centre of the raw x noise over the molecule's present atoms
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    const float m = p.mask[i] ? 1.f : 0.f;
    s[0] += noise_x[(size_t)i * 3 + 0] * m;
    s[1] += noise_x[(size_t)i * 3 + 1] * m;
    s[2] += noise_x[(size_t)i * 3 + 2] * m;
    s[3] += m;
  }
  block_sum4(s, red);
  const float cnt = s[3];
  const float nc[3] = {cnt > 0.f ? s[0] / cnt : 0.f, cnt > 0.f ? s[1] / cnt : 0.f, cnt > 0.f ? s[2] / cnt : 0.f};
  // 2) sums over the fixed atoms of z_unknown.x and of z_known.x
  float u[4] = {0.f, 0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f};
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    if (!fixed[i]) continue;
    const float m = p.mask[i] ? 1.f : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      u[c] += z[(size_t)i * ld + c];
      q[c] += alpha * xh0[(size_t)i * ld + c] + sigma * ((noise_x[(size_t)i * 3 + c] - nc[c] * m) * m);
    }
    u[3] += 1.f;
  }
  block_sum4(u, red);
  block_sum4(q, red);
  const float nf = u[3];
  if (nf == 0.f) return;                                 // no fixed atom: the molecule is sampled freely
  const float sh[3] = {u[0] / nf - q[0] / nf, u[1] / nf - q[1] / nf, u[2] / nf - q[2] / nf};
  // 3) overwrite the fixed rows
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    if (!fixed[i]) continue;
    const float m = p.mask[i] ? 1.f : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c)
      z[(size_t)i * ld + c] = (alpha * xh0[(size_t)i * ld + c] + sigma * ((noise_x[(size_t)i * 3 + c] - nc[c] * m) * m)) + sh[c];
    for (int f = 0; f < d.F; ++f)
      z[(size_t)i * ld + 3 + f] = alpha * xh0[(size_t)i * ld + 3 + f] + sigma * (noise_h[(size_t)i * d.F + f] * m);
  }
}

// ------------------------------------------------------------------------------- native chain (bdiff_sample)
// The last CTA of a grid to get here (every CTA has read *ctr by then) stores value into *ctr and re-arms *done, so a
// counter a kernel reads is advanced without another launch.
__device__ __forceinline__ void advance_counter(int* ctr, int* done, int value) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(done, 1) == (int)gridDim.x - 1) {
      *done = 0;
      *ctr = value;
    }
  }
}

// k_step with the noise computed in place: noise_x = draw dx, noise_h = draw dx + 1 of `seed` (bdiff_philox.cuh), where
// dx = draw0 + draw_table[*step_ptr] when a draw table is given (RePaint programs), else draw0 + 2 * *step_ptr in mode 0
// and draw0 otherwise ({seed, draw0} = seed_draw[0..1] when seed_draw is given).  Masking, centring and every arithmetic
// step are k_step's, mode 3 included.  Modes 0 and 3 advance the step counter when `done` is given.
__global__ void __launch_bounds__(128) k_step_philox(Plan p, Dims d, int mode, const float* __restrict__ z,
                                                     const float* __restrict__ eps, const float* __restrict__ coef_table,
                                                     int* step_ptr, int* done, unsigned long long seed,
                                                     unsigned long long draw0, const unsigned long long* seed_draw,
                                                     const unsigned long long* __restrict__ draw_table,
                                                     float* __restrict__ out) {
  const int step = step_ptr ? *step_ptr : 0;
  if (seed_draw) {            // a captured step reads {seed, draw0} from the device, so one graph serves every seed
    seed = seed_draw[0];
    draw0 = seed_draw[1];
  }
  const float* coef = coef_table ? coef_table + 4 * step : nullptr;
  const unsigned long long dx = draw0 + (draw_table ? draw_table[step] : mode == 0 ? 2ull * (unsigned)step : 0ull),
                           dh = dx + 1;
  __shared__ float red[4][4];
  const int k = blockIdx.x;
  const int n0 = p.mol_off[k], n1 = p.mol_off[k + 1];
  const int ld = 3 + d.F;
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    const float m = p.mask[i] ? 1.f : 0.f;
    s[0] += philox_normal(seed, dx, (unsigned long long)i * 3 + 0) * m;
    s[1] += philox_normal(seed, dx, (unsigned long long)i * 3 + 1) * m;
    s[2] += philox_normal(seed, dx, (unsigned long long)i * 3 + 2) * m;
    s[3] += m;
  }
  block_sum4(s, red);
  const float cnt = s[3];
  const float ncx = cnt > 0.f ? s[0] / cnt : 0.f, ncy = cnt > 0.f ? s[1] / cnt : 0.f,
              ncz = cnt > 0.f ? s[2] / cnt : 0.f;
  const float c0 = mode == 2 ? 0.f : __ldg(coef + 0), c1 = mode == 2 ? 0.f : __ldg(coef + 1),
              c2 = mode == 2 ? 1.f : __ldg(coef + 2);
  float t[4] = {0.f, 0.f, 0.f, 0.f};
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    const float m = p.mask[i] ? 1.f : 0.f;
    const float nc[3] = {ncx, ncy, ncz};
    for (int c = 0; c < ld; ++c) {
      float nz = (c < 3 ? philox_normal(seed, dx, (unsigned long long)i * 3 + c)
                        : philox_normal(seed, dh, (unsigned long long)i * d.F + (c - 3))) * m;
      if (c < 3) nz -= nc[c] * m;
      float v;
      if (mode == 0) v = z[(size_t)i * ld + c] / c0 - c1 * eps[(size_t)i * ld + c] + c2 * nz;
      else if (mode == 1) v = c0 * (z[(size_t)i * ld + c] - c1 * eps[(size_t)i * ld + c]) + c2 * nz;
      else if (mode == 3) v = c0 * z[(size_t)i * ld + c] + c1 * nz;
      else v = nz;
      out[(size_t)i * ld + c] = v;
      if (c < 3) t[c] += v;
    }
  }
  if (mode == 1 || mode == 2) return;
  block_sum4(t, red);
  const float zx = cnt > 0.f ? t[0] / cnt : 0.f, zy = cnt > 0.f ? t[1] / cnt : 0.f, zz = cnt > 0.f ? t[2] / cnt : 0.f;
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    const float m = p.mask[i] ? 1.f : 0.f;
    out[(size_t)i * ld + 0] -= zx * m;
    out[(size_t)i * ld + 1] -= zy * m;
    out[(size_t)i * ld + 2] -= zz * m;
  }
  if (done) advance_counter(step_ptr, done, step + 1);
}

// k_repaint_combine with the known part's noise computed in place: noise_x = draw dk, noise_h = draw dk + 1 of the seed,
// dk = seed_draw[1] + draw_table[*op_ptr], element layouts as in k_step_philox.  Advances the op counter when `done` is
// given.
__global__ void __launch_bounds__(128) k_repaint_combine_philox(Plan p, Dims d, float* __restrict__ z,
                                                                const float* __restrict__ xh0,
                                                                const uint8_t* __restrict__ fixed,
                                                                const float* __restrict__ known_table, int* op_ptr,
                                                                int* done, const unsigned long long* seed_draw,
                                                                const unsigned long long* __restrict__ draw_table) {
  __shared__ float red[4][4];
  const int k = blockIdx.x;
  const int n0 = p.mol_off[k], n1 = p.mol_off[k + 1];
  const int ld = 3 + d.F;
  const int op = *op_ptr;
  const unsigned long long seed = seed_draw[0], dk = seed_draw[1] + draw_table[op], dkh = dk + 1;
  const float alpha = __ldg(known_table + 2 * op), sigma = __ldg(known_table + 2 * op + 1);
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    const float m = p.mask[i] ? 1.f : 0.f;
    s[0] += philox_normal(seed, dk, (unsigned long long)i * 3 + 0) * m;
    s[1] += philox_normal(seed, dk, (unsigned long long)i * 3 + 1) * m;
    s[2] += philox_normal(seed, dk, (unsigned long long)i * 3 + 2) * m;
    s[3] += m;
  }
  block_sum4(s, red);
  const float cnt = s[3];
  const float nc[3] = {cnt > 0.f ? s[0] / cnt : 0.f, cnt > 0.f ? s[1] / cnt : 0.f, cnt > 0.f ? s[2] / cnt : 0.f};
  float u[4] = {0.f, 0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f};
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    if (!fixed[i]) continue;
    const float m = p.mask[i] ? 1.f : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      u[c] += z[(size_t)i * ld + c];
      q[c] += alpha * xh0[(size_t)i * ld + c] + sigma * ((philox_normal(seed, dk, (unsigned long long)i * 3 + c) - nc[c] * m) * m);
    }
    u[3] += 1.f;
  }
  block_sum4(u, red);
  block_sum4(q, red);
  const float nf = u[3];
  if (nf != 0.f) {                                       // no fixed atom: the molecule is sampled freely
    const float sh[3] = {u[0] / nf - q[0] / nf, u[1] / nf - q[1] / nf, u[2] / nf - q[2] / nf};
    for (int i = n0 + threadIdx.x; i < n1; i += 128) {
      if (!fixed[i]) continue;
      const float m = p.mask[i] ? 1.f : 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c)
        z[(size_t)i * ld + c] =
            (alpha * xh0[(size_t)i * ld + c] + sigma * ((philox_normal(seed, dk, (unsigned long long)i * 3 + c) - nc[c] * m) * m)) + sh[c];
      for (int f = 0; f < d.F; ++f)
        z[(size_t)i * ld + 3 + f] =
            alpha * xh0[(size_t)i * ld + 3 + f] + sigma * (philox_normal(seed, dkh, (unsigned long long)i * d.F + f) * m);
    }
  }
  if (done) advance_counter(op_ptr, done, op + 1);
}

// frames[slot[*step_ptr]] = unnormalize_z(z) (sampler.py _write_frame; every atom present, so the mask factor is 1), with
// torch's rounding: each multiply and add rounded on its own.  Then advances the step counter.
__global__ void __launch_bounds__(128) k_write_frame(Plan p, Dims d, int A, float nv0, float nv1, float nb1, float nv2,
                                                     float nb2, const float* __restrict__ z,
                                                     const int* __restrict__ slot, int* step_ptr, int* done,
                                                     float* __restrict__ frames) {
  const int step = *step_ptr;
  const int k = blockIdx.x;
  const int n0 = p.mol_off[k], n1 = p.mol_off[k + 1];
  const int ld = 3 + d.F;
  float* fr = frames + (size_t)slot[step] * p.N * ld;
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    const float* row = z + (size_t)i * ld;
    float* o = fr + (size_t)i * ld;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = __fmul_rn(row[c], nv0);
    for (int a = 0; a < A; ++a) o[3 + a] = __fadd_rn(__fmul_rn(row[3 + a], nv1), nb1);
    if (ld > 3 + A) o[3 + A] = __fadd_rn(__fmul_rn(row[3 + A], nv2), nb2);
  }
  advance_counter(step_ptr, done, step + 1);
}

__global__ void k_noise_fill(unsigned long long seed, unsigned long long draw, long long n, float* __restrict__ out) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) out[e] = philox_normal(seed, draw, (unsigned long long)e);
}

__global__ void k_philox_fill(unsigned long long seed, unsigned long long draw, long long blocks, uint32_t* __restrict__ out) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= blocks) return;
  const Philox4 r = philox_block(seed, draw, (unsigned long long)b);
  reinterpret_cast<uint4*>(out)[b] = make_uint4(r.w[0], r.w[1], r.w[2], r.w[3]);
}

// ctx[n, :] = context[molecule of n, :] (sampler.py's context[batch_index] * node_mask, every atom present)
__global__ void k_gather_context(Plan p, int C, const float* __restrict__ context, float* __restrict__ ctx) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)p.N * C) return;
  const int n = (int)(g / C), c = (int)(g - (long long)n * C);
  ctx[g] = context[(size_t)p.node_mol[n] * C + c];
}

// One CTA per molecule: the unnormalise / discretise tail of mol_gen_sample (sampler.py _finish, variational_diffusion.py
// :892-907): x = xh.x * nv0; one_hot = argmax of (xh.h_cat * nv1 + nb1) (first maximum, NaN counts as the maximum);
// charge = round-half-even(xh.h_int * nv2 + nb2) through int64.  Writes tot[k] = the molecule's coordinate sums.
__global__ void __launch_bounds__(128) k_sample_finish(Plan p, Dims d, int A, float nv0, float nv1, float nb1, float nv2,
                                                       float nb2, const float* __restrict__ xhn, float* __restrict__ out,
                                                       float* __restrict__ tot) {
  __shared__ float red[4][4];
  const int k = blockIdx.x;
  const int n0 = p.mol_off[k], n1 = p.mol_off[k + 1];
  const int ld = 3 + d.F;
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  for (int i = n0 + threadIdx.x; i < n1; i += 128) {
    const float* row = xhn + (size_t)i * ld;
    float* o = out + (size_t)i * ld;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      o[c] = __fmul_rn(row[c], nv0);
      s[c] += o[c];
    }
    int best = 0;
    float bv = 0.f;
    for (int a = 0; a < A; ++a) {
      const float v = __fadd_rn(__fmul_rn(row[3 + a], nv1), nb1);
      if (a == 0 || (!(bv != bv) && (v > bv || v != v))) { best = a; bv = v; }
    }
    for (int a = 0; a < A; ++a) o[3 + a] = a == best ? 1.f : 0.f;
    if (ld > 3 + A) o[3 + A] = (float)(long long)rintf(__fadd_rn(__fmul_rn(row[3 + A], nv2), nb2));
  }
  block_sum4(s, red);
  if (threadIdx.x == 0) {
    tot[3 * k + 0] = s[0];
    tot[3 * k + 1] = s[1];
    tot[3 * k + 2] = s[2];
  }
}

// CoG drift fix (variational_diffusion.py:1391-1402): when max |tot| over the batch exceeds 5e-2, x -= tot[k] / n_k.
__global__ void __launch_bounds__(128) k_sample_cog_fix(Plan p, Dims d, const float* __restrict__ tot, float* __restrict__ out) {
  __shared__ int fire;
  if (threadIdx.x == 0) fire = 0;
  __syncthreads();
  for (int j = threadIdx.x; j < 3 * p.B; j += 128)
    if (fabsf(tot[j]) > 5e-2f) fire = 1;
  __syncthreads();
  if (!fire) return;
  const int k = blockIdx.x;
  const int n0 = p.mol_off[k], n1 = p.mol_off[k + 1];
  const float cnt = (float)(n1 - n0);
  const int ld = 3 + d.F;
  for (int i = n0 + threadIdx.x; i < n1; i += 128)
#pragma unroll
    for (int c = 0; c < 3; ++c) out[(size_t)i * ld + c] = __fsub_rn(out[(size_t)i * ld + c], __fdiv_rn(tot[3 * k + c], cnt));
}

// edge_index int64 [2, E] from the plan (gcpnet.py:1054-1066) — only when a caller asks for it.
__global__ void k_edge_index(Plan p, long long* __restrict__ out) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= p.E) return;
  const int k = find_mol(p.edge_off, p.B, g);
  const int loc = (int)(g - p.edge_off[k]);
  const int a0 = p.act_off[k], na = p.act_off[k + 1] - a0;
  const int a = loc / na, b = loc - a * na;
  out[g] = p.act_idx[a0 + a];
  out[p.E + g] = p.act_idx[a0 + b];
}

// Per-edge record used by the tensor-core edge pass: one coalesced 16-byte load instead of a chain of dependent
// lookups (edge_off -> act_off -> act_idx) at the top of every tile.
__global__ void k_edge_rc(Plan p, int4* __restrict__ out, long long n) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n) return;
  int4 v = make_int4(-1, -1, 0, 0);
  if (g < p.E) {
    const int k = find_mol(p.edge_off, p.B, g);
    const int loc = (int)(g - p.edge_off[k]);
    const int a0 = p.act_off[k], na = p.act_off[k + 1] - a0;
    const int a = loc / na, b = loc - a * na;
    v = make_int4(p.act_idx[a0 + a], p.act_idx[a0 + b], b, na);
  }
  out[g] = v;
}

// dst[k*dst_ld + o] = k < ncols ? src[o*src_ld + col0 + k] : 0   (torch [out,in] weight -> K-major, padded), for a whole
// table of slices in ONE launch (a reference checkpoint is 432 tensors / ~950 slices): block b works on the job whose
// [block0, block0 + blocks) range contains it.
__global__ void k_pack_multi(const PackJob* __restrict__ jobs, int njobs) {
  int lo = 0, hi = njobs - 1;
  while (lo < hi) {                       // last job with block0 <= blockIdx.x
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].block0 <= (int)blockIdx.x) lo = mid;
    else hi = mid - 1;
  }
  const PackJob j = jobs[lo];
  const int idx = ((int)blockIdx.x - j.block0) * blockDim.x + threadIdx.x;
  if (idx >= j.kpad * j.nout) return;
  const int k = idx / j.nout, o = idx - k * j.nout;
  j.dst[(size_t)k * j.dst_ld + o] = k < j.ncols ? j.src[(size_t)o * j.src_ld + j.col0 + k] : 0.f;
}

// ============================================================================================ launchers
size_t edge_smem_bytes() { return sizeof(EdgeSmem); }
size_t node_smem_bytes() { return sizeof(NodeSmem); }

cudaError_t configure_kernels() {
  cudaError_t e;
  e = cudaFuncSetAttribute(k_edge_message, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(EdgeSmem));
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(k_node_embed, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(NodeSmem));
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(k_node_update, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(NodeSmem));
  return e;
}

void launch_prep(cudaStream_t st, const Plan& p, const Dims& d, const float* xh, const float* t_nodes,
                 const float* coef_table, const int* step_ptr, const float* ctx, const Work& w) {
  k_prep_nodes<<<p.B, 128, 0, st>>>(p, d, xh, t_nodes, coef_table, step_ptr, ctx, w);
  k_node_frames<<<(p.N + 7) / 8, 256, 0, st>>>(p, w);
}
void launch_edge_embed(cudaStream_t st, const Plan& p, const Dims& d, const EmbedW& ew, const Work& w) {
  const unsigned tiles = (unsigned)((p.E + TME - 1) / TME);
  if (!tiles) return;
  const unsigned blocks = (unsigned)((p.E + 127) / 128);
  if (d.Ed == 64 && d.Xd == 16) k_edge_embed_tpe<64, 16><<<blocks, 128, 0, st>>>(p, ew, w);
  else if (d.Ed == 16 && d.Xd == 8) k_edge_embed_tpe<16, 8><<<blocks, 128, 0, st>>>(p, ew, w);
  else k_edge_embed<<<tiles, kThreads, 0, st>>>(p, d, ew, w);
}
void launch_node_embed(cudaStream_t st, const Plan& p, const Dims& d, const EmbedW& ew, const LayerW& l0,
                       const Work& w) {
  k_node_embed<<<(p.N + TMN - 1) / TMN, kThreads, sizeof(NodeSmem), st>>>(p, d, ew, l0, w);
}
void launch_edge_message(cudaStream_t st, const Plan& p, const Dims& d, const LayerW& lw, const Work& w) {
  const unsigned tiles = (unsigned)((p.E + TME - 1) / TME);
  if (tiles) k_edge_message<<<tiles, kThreads, sizeof(EdgeSmem), st>>>(p, d, lw, w);
}
void launch_node_update(cudaStream_t st, const Plan& p, const Dims& d, const LayerW& lw, const LayerW& wn,
                        const EmbedW& ew, const Work& w, int last) {
  k_node_update<<<(p.N + TMN - 1) / TMN, kThreads, sizeof(NodeSmem), st>>>(p, d, lw, wn, ew, w, last);
}
void launch_finalize(cudaStream_t st, const Plan& p, const Dims& d, const Work& w, float* out) {
  k_finalize<<<p.B, 128, 0, st>>>(p, d, w, out);
}
void launch_step(cudaStream_t st, const Plan& p, const Dims& d, int mode, const float* z, const float* eps,
                 const float* noise_x, const float* noise_h, const float* coef_table, const int* step_ptr,
                 float* out) {
  k_step<<<p.B, 128, 0, st>>>(p, d, mode, z, eps, noise_x, noise_h, coef_table, step_ptr, out);
}
void launch_repaint_combine(cudaStream_t st, const Plan& p, const Dims& d, float* z, const float* xh0,
                            const uint8_t* fixed, const float* noise_x, const float* noise_h,
                            const float* known_table, const int* op_ptr) {
  k_repaint_combine<<<p.B, 128, 0, st>>>(p, d, z, xh0, fixed, noise_x, noise_h, known_table, op_ptr);
}
void launch_step_philox(cudaStream_t st, const Plan& p, const Dims& d, int mode, const float* z, const float* eps,
                        const float* coef_table, int* step_ptr, int* done, unsigned long long seed,
                        unsigned long long draw0, const unsigned long long* seed_draw,
                        const unsigned long long* draw_table, float* out) {
  k_step_philox<<<p.B, 128, 0, st>>>(p, d, mode, z, eps, coef_table, step_ptr, done, seed, draw0, seed_draw, draw_table,
                                     out);
}
void launch_repaint_combine_philox(cudaStream_t st, const Plan& p, const Dims& d, float* z, const float* xh0,
                                   const uint8_t* fixed, const float* known_table, int* op_ptr, int* done,
                                   const unsigned long long* seed_draw, const unsigned long long* draw_table) {
  k_repaint_combine_philox<<<p.B, 128, 0, st>>>(p, d, z, xh0, fixed, known_table, op_ptr, done, seed_draw, draw_table);
}
void launch_write_frame(cudaStream_t st, const Plan& p, const Dims& d, int A, const float* nv, const float* nb,
                        const float* z, const int* slot, int* step_ptr, int* done, float* frames) {
  k_write_frame<<<p.B, 128, 0, st>>>(p, d, A, nv[0], nv[1], nb[1], nv[2], nb[2], z, slot, step_ptr, done, frames);
}
void launch_noise_fill(cudaStream_t st, unsigned long long seed, unsigned long long draw, long long n, float* out) {
  if (n > 0) k_noise_fill<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(seed, draw, n, out);
}
void launch_philox_fill(cudaStream_t st, unsigned long long seed, unsigned long long draw, long long blocks, uint32_t* out) {
  if (blocks > 0) k_philox_fill<<<(unsigned)((blocks + 255) / 256), 256, 0, st>>>(seed, draw, blocks, out);
}
void launch_gather_context(cudaStream_t st, const Plan& p, int C, const float* context, float* ctx) {
  const long long n = (long long)p.N * C;
  if (n > 0) k_gather_context<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p, C, context, ctx);
}
void launch_sample_finish(cudaStream_t st, const Plan& p, const Dims& d, int A, const float* nv, const float* nb,
                          const float* xhn, float* out, float* tot, bool cog_fix) {
  k_sample_finish<<<p.B, 128, 0, st>>>(p, d, A, nv[0], nv[1], nb[1], nv[2], nb[2], xhn, out, tot);
  if (cog_fix) k_sample_cog_fix<<<p.B, 128, 0, st>>>(p, d, tot, out);
}
void launch_edge_index(cudaStream_t st, const Plan& p, long long* out) {
  if (p.E > 0) k_edge_index<<<(unsigned)((p.E + 255) / 256), 256, 0, st>>>(p, out);
}
void launch_edge_rc(cudaStream_t st, const Plan& p, int4* out, long long n) {
  if (n > 0) k_edge_rc<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p, out, n);
}
void launch_pack_multi(cudaStream_t st, const PackJob* jobs_dev, int njobs, int total_blocks) {
  if (njobs > 0 && total_blocks > 0) k_pack_multi<<<total_blocks, 256, 0, st>>>(jobs_dev, njobs);
}

}  // namespace bdiff
