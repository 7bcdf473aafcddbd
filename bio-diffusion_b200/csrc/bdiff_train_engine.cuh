// bdiff_train_engine.cuh — the training pass of the GCPNet denoiser: forward with a tape, then the hand-derived reverse
// sweep that yields the gradient of  sum(net_out * d_net_out)  with respect to every parameter tensor (SURVEY.md §8
// a20; reference: loss.backward() through GCPNetDynamics.forward, src/models/components/gcpnet.py:1069-1232, driven by
// EquivariantVariationalDiffusion.forward in .train() mode, variational_diffusion.py:955-1160).
//
// Unlike the sampler's fused kernels this pass keeps every intermediate a derivative needs, so it is organised as the
// reference's operator graph: per geometry-complete perceptron (gcpnet.py:418-491) a handful of plain row-major GEMMs
// (vector_down / vector_down_frames / scalar_out / vector_up / vector_out_scale and their two transposes) with small
// element-wise kernels between them, plus gather / segmented-sum kernels that use the implicit edge plan (edges of a
// molecule are its nact x nact block, row-major), so no scatter ever needs an atomic: every sum runs in a fixed order.
// Two departures from the graph, same mathematics: message GCP 0 runs in the sampler's split form (the endpoint blocks
// of scalar_out are node-level GEMMs PI = h.Wsi^T, PJ = h.Wsj^T, gathered per edge, instead of an [E, 512+Ed] gather
// and GEMM), and the backward writes every input gradient straight into its consumer (beta = 1 into the residual
// stream) with the activations act1(z) and silu(z1) read from the tape.
//
// The file is written against a small `Backend` concept  { run(n, functor); gemm(...); }  so that the very same
// functors and the very same orchestration compile twice: with the CUDA backend of bdiff_train.cu (kernels + cuBLAS
// SGEMM; the only one the product library contains) and with the host backend of oracle/hostcheck/train_hostcheck.cpp,
// a TEST-ONLY build that lets the CPU test-suite check this code against the autograd oracle without a GPU.
//
// Layouts: scalars [M, ld] row-major; vectors "xyz-major" [M*3, ld] (row m*3+x, column = channel), which turns every
// vector linear map of a GCP into one GEMM with M*3 rows.  Parameters and their gradients stay in the reference's
// layout (nn.Linear weight [out, in]), addressed through the same offsets as the raw staging copy of bdiff_set_weight.
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

#if defined(__CUDACC__)
#define BDT_HD __host__ __device__ __forceinline__
#else
#define BDT_HD inline
#endif

namespace bdiff {
namespace train {

struct EdgeRc { int row, col, b, nact; };   // same 16 bytes as the int4 records of Plan::edge_rc

struct Topo {
  int B = 0, N = 0;
  long long E = 0;
  const int* mol_off = nullptr;         // [B+1]
  const int* act_off = nullptr;         // [B+1]
  const int* act_idx = nullptr;         // [M]
  const long long* edge_off = nullptr;  // [B+1]
  const int* node_mol = nullptr;        // [N]
  const unsigned char* mask = nullptr;  // [N]
  const EdgeRc* edge_rc = nullptr;      // [E]
  int Mact = 0;                         // unmasked nodes = length of act_idx
};

struct NetDims { int F, C, Hin, Ed, Xd, L; };

BDT_HD float t_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }
BDT_HD float t_act(int a, float z) { return a ? z / (1.0f + expf(-z)) : z; }
BDT_HD float t_dact(int a, float z) {
  if (!a) return 1.0f;
  const float s = t_sigmoid(z);
  return s * (1.0f + z * (1.0f - s));
}
BDT_HD float t_nan0(float v) {   // torch.nan_to_num
  if (v != v) return 0.0f;
  if (v > 3.4028234663852886e38f) return 3.4028234663852886e38f;
  if (v < -3.4028234663852886e38f) return -3.4028234663852886e38f;
  return v;
}

// ------------------------------------------------------------------------------------------------ functors: inputs
struct FPrepNodes {     // xh*mask -> x_init, h_in = [h*mask | t | context]          (gcpnet.py:1081, 1142-1150)
  const float *xh, *t, *ctx; const unsigned char* mask; float *x_init, *h_in; int F, C, Hin, ldh;
  BDT_HD void operator()(long long i) const {
    const float m = mask[i] ? 1.0f : 0.0f;
    const float* r = xh + i * (3 + F);
    for (int j = 0; j < 3; ++j) x_init[i * 3 + j] = r[j] * m;
    float* o = h_in + i * ldh;
    for (int j = 0; j < F; ++j) o[j] = r[3 + j] * m;
    o[F] = t[i];
    for (int c = 0; c < C; ++c) o[F + 1 + c] = ctx[i * C + c];
  }
};
struct FCentre {        // x = x_init - mask * mean_mol(x_init)                       (components/__init__.py:46-98)
  Topo tp; const float* x_init; float* x;
  BDT_HD void operator()(long long i) const {
    const int k = tp.node_mol[i];
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, cnt = 0.f;
    for (int j = tp.mol_off[k]; j < tp.mol_off[k + 1]; ++j) {
      s0 += x_init[j * 3 + 0]; s1 += x_init[j * 3 + 1]; s2 += x_init[j * 3 + 2];
      cnt += tp.mask[j] ? 1.0f : 0.0f;
    }
    const float m = tp.mask[i] ? 1.0f : 0.0f;
    x[i * 3 + 0] = x_init[i * 3 + 0] - (s0 / cnt) * m;
    x[i * 3 + 1] = x_init[i * 3 + 1] - (s1 / cnt) * m;
    x[i * 3 + 2] = x_init[i * 3 + 2] - (s2 / cnt) * m;
  }
};
struct FOrient {        // chi_in over the concatenated atom list                      (protein_graph_dataset.py:217-225)
  const float* x_init; float* chi_t; int N;     // chi_t [N*3, 2]
  BDT_HD void operator()(long long i) const {
    float f[3] = {0.f, 0.f, 0.f}, b[3] = {0.f, 0.f, 0.f};
    if (i + 1 < N) {
      float d[3], n2 = 0.f;
      for (int x = 0; x < 3; ++x) { d[x] = x_init[(i + 1) * 3 + x] - x_init[i * 3 + x]; n2 += d[x] * d[x]; }
      const float n = sqrtf(n2);
      for (int x = 0; x < 3; ++x) f[x] = t_nan0(t_nan0(d[x] / n));
    }
    if (i > 0) {
      float d[3], n2 = 0.f;
      for (int x = 0; x < 3; ++x) { d[x] = x_init[(i - 1) * 3 + x] - x_init[i * 3 + x]; n2 += d[x] * d[x]; }
      const float n = sqrtf(n2);
      for (int x = 0; x < 3; ++x) b[x] = t_nan0(t_nan0(d[x] / n));
    }
    for (int x = 0; x < 3; ++x) { chi_t[(i * 3 + x) * 2 + 0] = f[x]; chi_t[(i * 3 + x) * 2 + 1] = b[x]; }
  }
};
struct FEdgeGeom {      // e_in, xi_in (un-centred x), frames (centred x)             (edm_dataset.py:22-38, components/__init__.py:123-171)
  const EdgeRc* rc; const float *x_init, *x; float *e_in, *xi_t, *frames; int ld_e;
  BDT_HD void operator()(long long e) const {
    const int r = rc[e].row, c = rc[e].col;
    float d[3], n2 = 0.f;
    for (int k = 0; k < 3; ++k) { d[k] = x_init[r * 3 + k] - x_init[c * 3 + k]; n2 += d[k] * d[k]; }
    e_in[e * ld_e] = t_nan0(n2);
    const float n = sqrtf(n2);
    for (int k = 0; k < 3; ++k) xi_t[e * 3 + k] = t_nan0(t_nan0(d[k] / n));
    float a[3], b[3], dd[3], cr[3], v[3];
    for (int k = 0; k < 3; ++k) { a[k] = x[r * 3 + k]; b[k] = x[c * 3 + k]; dd[k] = a[k] - b[k]; }
    cr[0] = a[1] * b[2] - a[2] * b[1]; cr[1] = a[2] * b[0] - a[0] * b[2]; cr[2] = a[0] * b[1] - a[1] * b[0];
    const float nd = sqrtf(dd[0] * dd[0] + dd[1] * dd[1] + dd[2] * dd[2]) + 1.0f;
    const float nc = sqrtf(cr[0] * cr[0] + cr[1] * cr[1] + cr[2] * cr[2]) + 1.0f;
    for (int k = 0; k < 3; ++k) { dd[k] = dd[k] / nd; cr[k] = cr[k] / nc; }
    v[0] = dd[1] * cr[2] - dd[2] * cr[1]; v[1] = dd[2] * cr[0] - dd[0] * cr[2]; v[2] = dd[0] * cr[1] - dd[1] * cr[0];
    float* f = frames + e * 9;
    for (int k = 0; k < 3; ++k) { f[k] = dd[k]; f[3 + k] = cr[k]; f[6 + k] = v[k]; }
  }
};
// first edge and edge count of node n's row (count 0 for masked nodes)
BDT_HD void row_span(const Topo& tp, const int* apos, long long n, long long& e0, int& na) {
  const int a = apos[n];
  if (a < 0) { e0 = 0; na = 0; return; }
  const int k = tp.node_mol[n];
  na = tp.act_off[k + 1] - tp.act_off[k];
  e0 = tp.edge_off[k] + (long long)a * na;
}
struct FApos {          // position of each unmasked node inside its molecule's active list
  Topo tp; int* apos;
  BDT_HD void operator()(long long j) const {      // j over act_idx
    const int n = tp.act_idx[j];
    apos[n] = (int)j - tp.act_off[tp.node_mol[n]];
  }
};
struct FFillInt { int* p; int v; BDT_HD void operator()(long long i) const { p[i] = v; } };
struct FFill { float* p; float v; BDT_HD void operator()(long long i) const { p[i] = v; } };
struct FNodeFbar {      // mean frame of a node's row (node-side scalarize, components/__init__.py:175-219)
  Topo tp; const int* apos; const float* frames; float* fbar;
  BDT_HD void operator()(long long idx) const {
    const long long n = idx / 9; const int j = (int)(idx % 9);
    long long e0; int na;
    row_span(tp, apos, n, e0, na);
    float s = 0.f;
    for (int b = 0; b < na; ++b) s += frames[(e0 + b) * 9 + j];
    fbar[idx] = s / (float)(na > 1 ? na : 1);
  }
};

// ------------------------------------------------------------------------------------------------ functors: GCP forward
struct FMerge {         // merged[:, S_in : S_in+H+9] = [safe_norm(hid) | scalarize(vdf, frames)]   (gcpnet.py:444-459)
  const float *hid, *vdf, *frames; float* merged; int S_in, H, fan;
  BDT_HD void operator()(long long idx) const {
    const int w = H + 9;
    const long long m = idx / w; const int j = (int)(idx % w);
    float out;
    if (j < H) {
      const float a = hid[(m * 3 + 0) * H + j], b = hid[(m * 3 + 1) * H + j], c = hid[(m * 3 + 2) * H + j];
      out = sqrtf(a * a + b * b + c * c + 1e-8f) + 1e-8f;
    } else {
      const int c = (j - H) / 3, a = (j - H) % 3;
      const float* f = frames + m * 9 + a * 3;
      out = f[0] * vdf[(m * 3 + 0) * 3 + c] + f[1] * vdf[(m * 3 + 1) * 3 + c] + f[2] * vdf[(m * 3 + 2) * 3 + c];
    }
    merged[m * fan + S_in + j] = out;
  }
};
struct FBiasSilu {      // feed-forward scalar_out: z1 += b0 (kept), a = silu(z1)
  float* z1; const float* b; float* a; int n;
  BDT_HD void operator()(long long idx) const {
    const float z = z1[idx] + b[idx % n];
    z1[idx] = z;
    a[idx] = t_act(1, z);
  }
};
struct FScalarOut {     // z += bias (kept on the tape); s_out = (act0(z) + residual) * mask; a1 = act1(z)
  float* z; const float* b; int n, act0, act1;
  float* s_out; int ld_so; const float* res; int ld_res; const unsigned char* mask; float* a1;
  const float *pi, *pj; const EdgeRc* rc;     // split message GCP 0: z += PI[row] + PJ[col] (node-level h.Wsi^T, h.Wsj^T)
  BDT_HD void operator()(long long idx) const {
    const long long m = idx / n; const int j = (int)(idx % n);
    float zz = z[idx] + b[j];
    if (pi) zz += pi[(long long)rc[m].row * n + j] + pj[(long long)rc[m].col * n + j];
    z[idx] = zz;
    if (a1) a1[idx] = t_act(act1, zz);
    if (s_out) {
      float v = t_act(act0, zz);
      if (res) v += res[m * ld_res + j];
      if (mask) v *= mask[m] ? 1.0f : 0.0f;
      s_out[m * ld_so + j] = v;
    }
  }
};
struct FVecOut {        // sg = sigmoid(gate + bg) (kept); v_out = (up * sg + residual) * mask      (gcpnet.py:388-411)
  float* sg; const float* bg; const float* up; int V;
  float* v_out; int ld_vo; const float* res; int ld_res; const unsigned char* mask;
  BDT_HD void operator()(long long idx) const {
    const long long m = idx / V; const int o = (int)(idx % V);
    const float g = t_sigmoid(sg[idx] + bg[o]);
    sg[idx] = g;
    const float mk = mask ? (mask[m] ? 1.0f : 0.0f) : 1.0f;
    for (int x = 0; x < 3; ++x) {
      float v = up[(m * 3 + x) * V + o] * g;
      if (res) v += res[(m * 3 + x) * ld_res + o];
      v_out[(m * 3 + x) * ld_vo + o] = v * mk;
    }
  }
};

// ------------------------------------------------------------------------------------------------ functors: GCP backward
struct FDVecOut {       // d gate (pre-sigmoid) and d up from d v_out
  const float *dv, *up, *sg; int ld_dv, V; float *dgate, *dup;
  BDT_HD void operator()(long long idx) const {
    const long long m = idx / V; const int o = (int)(idx % V);
    const float g = sg[idx];
    float acc = 0.f;
    for (int x = 0; x < 3; ++x) {
      const float d = dv[(m * 3 + x) * ld_dv + o];
      acc += d * up[(m * 3 + x) * V + o];
      dup[(m * 3 + x) * V + o] = d * g;
    }
    dgate[idx] = acc * g * (1.0f - g);
  }
};
struct FDZ {            // dz = ds_out * act0'(z) + dgz * act1'(z)
  const float* ds; int ld_ds; const float* dgz; const float* z; int n, act0, act1; float* dz;
  BDT_HD void operator()(long long idx) const {
    const long long m = idx / n; const int j = (int)(idx % n);
    const float zz = z[idx];
    float v = 0.f;
    if (ds) v = ds[m * ld_ds + j] * t_dact(act0, zz);
    if (dgz) v += dgz[idx] * t_dact(act1, zz);
    dz[idx] = v;
  }
};
struct FMulDSilu { float* d; const float* z; BDT_HD void operator()(long long i) const { d[i] *= t_dact(1, z[i]); } };
struct FDNorm {         // dhid (+)= dvnorm / sqrt(sum hid^2 + 1e-8) * hid
  const float* dvq; int ld, H; const float* hid; float* dhid; int accumulate;
  BDT_HD void operator()(long long idx) const {
    const long long m = idx / H; const int h = (int)(idx % H);
    const float a = hid[(m * 3 + 0) * H + h], b = hid[(m * 3 + 1) * H + h], c = hid[(m * 3 + 2) * H + h];
    const float s = dvq[m * ld + h] / sqrtf(a * a + b * b + c * c + 1e-8f);
    if (accumulate) {
      dhid[(m * 3 + 0) * H + h] += s * a; dhid[(m * 3 + 1) * H + h] += s * b; dhid[(m * 3 + 2) * H + h] += s * c;
    } else {
      dhid[(m * 3 + 0) * H + h] = s * a; dhid[(m * 3 + 1) * H + h] = s * b; dhid[(m * 3 + 2) * H + h] = s * c;
    }
  }
};
struct FDQ {            // dvdf[m,x,c] = sum_a dq[m,c,a] * frames[m,a,x]
  const float* dvq; int ld, off; const float* frames; float* dvdf;
  BDT_HD void operator()(long long idx) const {
    const long long m = idx / 9; const int x = (int)(idx % 9) / 3, c = (int)(idx % 3);
    const float* dq = dvq + m * ld + off + c * 3;
    const float* f = frames + m * 9;
    dvdf[idx] = dq[0] * f[0 + x] + dq[1] * f[3 + x] + dq[2] * f[6 + x];
  }
};
// column sums in a fixed order: partial[j][c] = sum of rows [j*R, (j+1)*R), then out[c] += sum_j partial[j][c]
constexpr int kColsumRows = 512;
struct FColsum1 {
  const float* A; long long M; int N, lda; float* part;
  BDT_HD void operator()(long long idx) const {
    const long long j = idx / N; const int c = (int)(idx % N);
    const long long r0 = j * kColsumRows, r1 = (r0 + kColsumRows < M) ? r0 + kColsumRows : M;
    float s = 0.f;
    for (long long r = r0; r < r1; ++r) s += A[r * lda + c];
    part[idx] = s;
  }
};
struct FColsum2 {
  const float* part; long long J; int N; float* out;
  BDT_HD void operator()(long long c) const {
    float s = 0.f;
    for (long long j = 0; j < J; ++j) s += part[j * N + c];
    out[c] += s;
  }
};

// ------------------------------------------------------------------------------------------------ functors: message passing
struct FGatherV {       // mv_t = [chi[row] | xi | chi[col]]
  const EdgeRc* rc; const float* chi; int ld_c; const float* xi; int Xd; float* out;
  BDT_HD void operator()(long long idx) const {
    const int w = 64 + Xd;
    const long long rx = idx / w; const int i = (int)(idx % w);
    const long long ed = rx / 3; const int x = (int)(rx % 3);
    float v;
    if (i < 32) v = chi[((long long)rc[ed].row * 3 + x) * ld_c + i];
    else if (i < 32 + Xd) v = xi[rx * Xd + (i - 32)];
    else v = chi[((long long)rc[ed].col * 3 + x) * ld_c + (i - 32 - Xd)];
    out[idx] = v;
  }
};
struct FSigmoidBias { float* p; const float* b; BDT_HD void operator()(long long i) const { p[i] = t_sigmoid(p[i] + b[0]); } };
struct FAggS {          // a_s[n] = sum over the row's edges of s * attn                (gcpnet.py:709-723)
  Topo tp; const int* apos; const float *s, *attn; float* out; int ld_o;
  BDT_HD void operator()(long long idx) const {
    const long long n = idx / 256; const int j = (int)(idx % 256);
    long long e0; int na;
    row_span(tp, apos, n, e0, na);
    float acc = 0.f;
    for (int b = 0; b < na; ++b) acc += s[(e0 + b) * 256 + j] * attn[e0 + b];
    out[n * ld_o + j] = acc;
  }
};
struct FAggV {
  Topo tp; const int* apos; const float* v; float* out; int ld_o;
  BDT_HD void operator()(long long idx) const {
    const long long nx = idx / 32; const int o = (int)(idx % 32);
    const long long n = nx / 3; const int x = (int)(nx % 3);
    long long e0; int na;
    row_span(tp, apos, n, e0, na);
    float acc = 0.f;
    for (int b = 0; b < na; ++b) acc += v[((e0 + b) * 3 + x) * 32 + o];
    out[nx * ld_o + o] = acc;
  }
};
struct FCopy2D {        // dst[r, c] = src[r, c] for c < cols
  const float* src; int ld_s; float* dst; int ld_d, cols;
  BDT_HD void operator()(long long idx) const {
    const long long r = idx / cols; const int c = (int)(idx % cols);
    dst[r * ld_d + c] = src[r * ld_s + c];
  }
};
struct FAdd2D {         // dst[r, c] += src[r, c]
  const float* src; int ld_s; float* dst; int ld_d, cols;
  BDT_HD void operator()(long long idx) const {
    const long long r = idx / cols; const int c = (int)(idx % cols);
    dst[r * ld_d + c] += src[r * ld_s + c];
  }
};
struct FDAttnPre {      // dpre = <d(s*attn), s> * attn (1 - attn)
  const EdgeRc* rc; const float* da; int ld_da; const float *s, *attn; float* dpre;
  BDT_HD void operator()(long long e) const {
    const float* d = da + (long long)rc[e].row * ld_da;
    const float* ss = s + e * 256;
    float acc = 0.f;
    for (int j = 0; j < 256; ++j) acc += d[j] * ss[j];
    const float a = attn[e];
    dpre[e] = acc * a * (1.0f - a);
  }
};
struct FDAttnS {        // ds = da[row] * attn + dpre * wa
  const EdgeRc* rc; const float* da; int ld_da; const float *attn, *dpre, *wa; float* ds;
  BDT_HD void operator()(long long idx) const {
    const long long e = idx / 256; const int j = (int)(idx % 256);
    ds[idx] = da[(long long)rc[e].row * ld_da + j] * attn[e] + dpre[e] * wa[j];
  }
};
struct FGatherRowV {    // dv[e] = da_v[row]
  const EdgeRc* rc; const float* dav; int ld; float* dv;
  BDT_HD void operator()(long long idx) const {
    const long long ex = idx / 32; const int o = (int)(idx % 32);
    const long long e = ex / 3; const int x = (int)(ex % 3);
    dv[idx] = dav[((long long)rc[e].row * 3 + x) * ld + o];
  }
};
struct FScatterV {
  Topo tp; const int* apos; const float* dmv; int w, Xd; float* dchi; int ld;
  BDT_HD void operator()(long long idx) const {
    const long long nx = idx / 32; const int o = (int)(idx % 32);
    const long long n = nx / 3; const int x = (int)(nx % 3);
    long long e0; int na;
    row_span(tp, apos, n, e0, na);
    if (na == 0) return;
    float acc = 0.f;
    for (int b = 0; b < na; ++b) acc += dmv[((e0 + b) * 3 + x) * w + o];
    const int a = apos[n];
    const long long base = e0 - (long long)a * na;
    for (int r = 0; r < na; ++r) acc += dmv[((base + (long long)r * na + a) * 3 + x) * w + 32 + Xd + o];
    dchi[nx * ld + o] += acc;
  }
};
struct FScatterDZ {     // split message GCP 0: dPI[n] = sum over row n of dz, dPJ[n] = sum over column n of dz
  Topo tp; const int* apos; const float* dz; float *dpi, *dpj;
  BDT_HD void operator()(long long idx) const {
    const long long n = idx / 256; const int j = (int)(idx % 256);
    long long e0; int na;
    row_span(tp, apos, n, e0, na);
    float a0 = 0.f, a1 = 0.f;
    if (na) {
      for (int b = 0; b < na; ++b) a0 += dz[(e0 + b) * 256 + j];
      const int a = apos[n];
      const long long base = e0 - (long long)a * na;
      for (int r = 0; r < na; ++r) a1 += dz[(base + (long long)r * na + a) * 256 + j];
    }
    dpi[idx] = a0; dpj[idx] = a1;
  }
};
struct FMaskAdd {       // dst[m, c] = (dst[m, c] + add[m_row, c]) * mask[m]; rows_per = 1 (scalars) or 3 (vectors)
  float* dst; int ld_d; const float* add; int ld_a, cols, rows_per; const unsigned char* mask;
  BDT_HD void operator()(long long idx) const {
    const long long r = idx / cols; const int c = (int)(idx % cols);
    const float mk = mask[r / rows_per] ? 1.0f : 0.0f;
    dst[r * ld_d + c] = (dst[r * ld_d + c] + add[r * ld_a + c]) * mk;
  }
};

// ------------------------------------------------------------------------------------------------ functors: output
struct FFinal {         // net_out = [centralize((x_L - x_init) * mask) | hp[:, :F]]   (gcpnet.py:1204-1230)
  Topo tp; const float *xL, *x_init, *hp; int ld_hp, F; float* out;
  BDT_HD void operator()(long long i) const {
    const int k = tp.node_mol[i];
    float s[3] = {0.f, 0.f, 0.f}, cnt = 0.f;
    for (int j = tp.mol_off[k]; j < tp.mol_off[k + 1]; ++j) {
      const float m = tp.mask[j] ? 1.0f : 0.0f;
      for (int x = 0; x < 3; ++x) s[x] += (xL[j * 3 + x] - x_init[j * 3 + x]) * m;
      cnt += m;
    }
    const float m = tp.mask[i] ? 1.0f : 0.0f;
    float* o = out + i * (3 + F);
    for (int x = 0; x < 3; ++x) o[x] = (xL[i * 3 + x] - x_init[i * 3 + x]) * m - (s[x] / cnt) * m;
    for (int j = 0; j < F; ++j) o[3 + j] = hp[i * ld_hp + j];
  }
};
struct FDFinal {        // d x_L and d hp from d net_out
  Topo tp; const float* dout; int F, Hin; float *dx, *dhp;
  BDT_HD void operator()(long long i) const {
    const int k = tp.node_mol[i];
    float s[3] = {0.f, 0.f, 0.f}, cnt = 0.f;
    for (int j = tp.mol_off[k]; j < tp.mol_off[k + 1]; ++j) {
      const float m = tp.mask[j] ? 1.0f : 0.0f;
      for (int x = 0; x < 3; ++x) s[x] += dout[(long long)j * (3 + F) + x] * m;
      cnt += m;
    }
    const float m = tp.mask[i] ? 1.0f : 0.0f;
    for (int x = 0; x < 3; ++x) dx[i * 3 + x] = (dout[i * (3 + F) + x] - s[x] / cnt) * m;
    for (int j = 0; j < Hin; ++j) dhp[i * Hin + j] = j < F ? dout[i * (3 + F) + 3 + j] : 0.0f;
  }
};

// ------------------------------------------------------------------------------------------------ one GCP
struct Gcp {
  int S_in = 0, V_in = 0, H = 0, S_out = 0, V_out = 0, ff = 0, act0 = 0, act1 = 0;
  long long M = 0;
  const float *Wd = nullptr, *Wf = nullptr, *Ws = nullptr, *bs = nullptr, *W2 = nullptr, *b2 = nullptr, *Wu = nullptr,
              *Wg = nullptr, *bg = nullptr;
  float *gWd = nullptr, *gWf = nullptr, *gWs = nullptr, *gbs = nullptr, *gW2 = nullptr, *gb2 = nullptr, *gWu = nullptr,
        *gWg = nullptr, *gbg = nullptr;
  float* vt = nullptr; int ldv = 0;    // input vectors [M*3, ldv]
  float* merged = nullptr; int fan = 0; // [M, fan] = [s | vnorm | q]; the scalar_out weight block that multiplies it starts at
  int fanW = 0, wcol = 0;               // column wcol of Ws, whose rows are fanW long (fanW = fan, wcol = 0 unless split)
  // split form of message GCP 0: merged = [vnorm | q] only; z also gets e.We^T (a second GEMM) and the node-level
  // projections PI[row] + PJ[col] (gathered in FScalarOut)
  int split = 0, Ed = 0;
  const float *ee = nullptr, *pi = nullptr, *pj = nullptr; const EdgeRc* rc = nullptr;
  float *a1t = nullptr, *aff = nullptr;  // act1(z) (if V_out) and silu(z1) (if ff), kept on the tape for the backward
  float *hid = nullptr, *vdf = nullptr, *z1 = nullptr, *z = nullptr, *up = nullptr, *sg = nullptr;
  const float* frames = nullptr;        // [M, 9]: edge frames or the nodes' mean row frames
};

struct Scratch {        // sized for the largest entity count; used inside one GCP forward / backward only
  float *dz, *dgz, *dg, *dup, *dhid, *dvdf, *part;
};

struct ParamRef { const float* w; float* g; };

// Where a GCP's backward puts its input gradients: d s into `ds_dst` [M, ld_ds] and d v into `dvt` [M*3, ld_dvt], each
// as C = grad + beta * C (so beta = 1 accumulates into a residual stream) and skipped when null.  d[vnorm | q] only
// passes through the engine's DVQ scratch.
struct BwdOut {
  float* ds_dst = nullptr; int ld_ds = 0; float beta_ds = 0.f;
  float* dvt = nullptr; int ld_dvt = 0; float beta_dvt = 0.f;
};

// Everything below is host code (both backends).
template <class Backend>
struct Engine {
  Backend& be;
  NetDims d{};
  Topo tp{};
  explicit Engine(Backend& b) : be(b) {}

  // arena
  float* arena = nullptr;
  size_t used = 0;
  bool assign = false;
  float* take(size_t n) {
    n = (n + 63) / 64 * 64;
    float* r = assign ? arena + used : nullptr;
    used += n;
    return r;
  }

  // network
  Gcp g_edge, g_node, g_proj;
  struct Layer {
    Gcp msg[4], ff, pos;
    const float *wa, *ba; float *gwa, *gba;
    float *V[4], *S3, *attn, *FV, *CHI2, *Xn;
  };
  std::vector<Layer> layers;
  // inputs / shared
  int* apos = nullptr;
  float *x_init = nullptr, *x0 = nullptr, *chi_in = nullptr, *xi_in = nullptr, *frames = nullptr, *fbar = nullptr,
        *EE = nullptr, *XI = nullptr, *HP = nullptr;
  // backward state
  float *DX = nullptr, *DHP = nullptr, *DH = nullptr, *DCHI = nullptr, *DMN = nullptr, *DFV = nullptr, *DMV = nullptr,
        *DS = nullptr, *DV = nullptr, *DPRE = nullptr, *DE = nullptr, *DXI = nullptr;
  Scratch sc{};
  float *PI = nullptr, *PJ = nullptr, *DVQ = nullptr;
  float* grad_base = nullptr;   // flat gradient buffer (reference layout), zeroed at the start of backward()
  size_t grad_count = 0;
  bool have_tape = false;

  static int hid_of(int v_in, int v_out, int bottleneck) { return bottleneck > 1 ? v_in / bottleneck : (v_in > v_out ? v_in : v_out); }

  template <class Lookup>
  void shape_gcp(Gcp& g, const std::string& p, long long M, int S_in, int V_in, int S_out, int V_out, int bott, int ff,
                 int act, const float* fr, Lookup& look, int split = 0) {
    g.M = M; g.S_in = S_in; g.V_in = V_in; g.S_out = S_out; g.V_out = V_out; g.ff = ff; g.act0 = act; g.act1 = act;
    g.H = hid_of(V_in, V_out, bott);
    g.fan = S_in + g.H + 9;
    g.fanW = g.fan; g.wcol = 0; g.split = split;
    if (split) { g.wcol = S_in; g.S_in = 0; g.fan = g.H + 9; }
    g.frames = fr;
    auto P = [&](const char* leaf, const float*& w, float*& gr) { ParamRef r = look(p + leaf); w = r.w; gr = r.g; };
    P("vector_down.weight", g.Wd, g.gWd);
    P("vector_down_frames.weight", g.Wf, g.gWf);
    if (ff) {
      P("scalar_out.0.weight", g.Ws, g.gWs); P("scalar_out.0.bias", g.bs, g.gbs);
      P("scalar_out.2.weight", g.W2, g.gW2); P("scalar_out.2.bias", g.b2, g.gb2);
    } else {
      P("scalar_out.weight", g.Ws, g.gWs); P("scalar_out.bias", g.bs, g.gbs);
    }
    if (V_out) {
      P("vector_up.weight", g.Wu, g.gWu);
      P("vector_out_scale.weight", g.Wg, g.gWg); P("vector_out_scale.bias", g.bg, g.gbg);
    }
    g.merged = take((size_t)M * g.fan);
    g.hid = take((size_t)M * 3 * g.H);
    g.vdf = take((size_t)M * 9);
    g.z1 = ff ? take((size_t)M * S_out) : nullptr;
    g.z = take((size_t)M * S_out);
    g.up = V_out ? take((size_t)M * 3 * V_out) : nullptr;
    g.sg = V_out ? take((size_t)M * V_out) : nullptr;
    g.a1t = V_out ? take((size_t)M * S_out) : nullptr;
    g.aff = ff ? take((size_t)M * S_out) : nullptr;
  }

  // Lays out the tape for (dims, topology sizes).  Call with assign=false to size the arena, then with the arena.
  template <class Lookup>
  size_t layout(const NetDims& dims, const Topo& topo, float* arena_ptr, Lookup look) {
    d = dims; tp = topo;
    arena = arena_ptr; assign = arena_ptr != nullptr; used = 0;
    const long long N = tp.N, E = tp.E;
    const long long Mx = E > N ? E : N;
    apos = reinterpret_cast<int*>(take((size_t)N));
    x_init = take((size_t)N * 3); x0 = take((size_t)N * 3); chi_in = take((size_t)N * 6);
    xi_in = take((size_t)E * 3); frames = take((size_t)E * 9); fbar = take((size_t)N * 9);
    EE = take((size_t)E * d.Ed); XI = take((size_t)E * 3 * d.Xd); HP = take((size_t)N * d.Hin);
    shape_gcp(g_edge, "gcp_embedding.edge_embedding.", E, 1, 1, d.Ed, d.Xd, 1, 0, 1, frames, look);
    g_edge.vt = xi_in; g_edge.ldv = 1;
    shape_gcp(g_node, "gcp_embedding.node_embedding.", N, d.Hin, 2, 256, 32, 1, 0, 0, fbar, look);
    g_node.vt = chi_in; g_node.ldv = 2;
    layers.assign(d.L, Layer{});
    for (int l = 0; l < d.L; ++l) {
      Layer& y = layers[l];
      const std::string p = "interaction_layers." + std::to_string(l) + ".";
      shape_gcp(y.msg[0], p + "interaction.message_fusion.0.", E, 512 + d.Ed, 64 + d.Xd, 256, 32, 4, 0, 1, frames, look, 1);
      y.msg[0].vt = take((size_t)E * 3 * (64 + d.Xd)); y.msg[0].ldv = 64 + d.Xd;
      y.msg[0].Ed = d.Ed; y.msg[0].ee = EE; y.msg[0].rc = tp.edge_rc;
      for (int k = 0; k < 4; ++k) y.V[k] = take((size_t)E * 96);
      for (int k = 1; k < 4; ++k) {
        shape_gcp(y.msg[k], p + "interaction.message_fusion." + std::to_string(k) + ".", E, 256, 32, 256, 32, 4, 0, 1, frames, look);
        y.msg[k].vt = y.V[k - 1]; y.msg[k].ldv = 32;
      }
      y.S3 = take((size_t)E * 256); y.attn = take((size_t)E);
      ParamRef a = look(p + "interaction.scalar_message_attention.0.weight"), b = look(p + "interaction.scalar_message_attention.0.bias");
      y.wa = a.w; y.gwa = a.g; y.ba = b.w; y.gba = b.g;
      shape_gcp(y.ff, p + "feedforward_network.0.", N, 512, 64, 256, 32, 4, 1, 0, fbar, look);
      y.FV = take((size_t)N * 3 * 64); y.ff.vt = y.FV; y.ff.ldv = 64;
      shape_gcp(y.pos, p + "node_position_update_gcp.", N, 256, 32, 256, 1, 4, 0, 1, fbar, look);
      y.CHI2 = take((size_t)N * 96); y.pos.vt = y.CHI2; y.pos.ldv = 32;
      y.Xn = take((size_t)N * 3);
    }
    shape_gcp(g_proj, "scalar_node_projection_gcp.", N, 256, 32, d.Hin, 0, 1, 0, 0, fbar, look);
    g_proj.vt = d.L ? layers[d.L - 1].CHI2 : nullptr; g_proj.ldv = 32;
    // scratch + backward state
    sc.dz = take((size_t)Mx * 256); sc.dgz = take((size_t)Mx * 256);
    sc.dg = take((size_t)Mx * 32); sc.dup = take((size_t)Mx * 96); sc.dhid = take((size_t)Mx * 96); sc.dvdf = take((size_t)Mx * 9);
    sc.part = take((size_t)((Mx * 3 + kColsumRows - 1) / kColsumRows + 1) * 640);
    DX = take((size_t)N * 3); DHP = take((size_t)N * d.Hin); DH = take((size_t)N * 256); DCHI = take((size_t)N * 96);
    // DMN: d s of the position GCP [N, 256], then d[agg_s | h] of the feed-forward GCP [N, 512]
    DMN = take((size_t)N * 512); DFV = take((size_t)N * 3 * 64);
    DMV = take((size_t)E * 3 * (64 + d.Xd));
    DS = take((size_t)E * 256); DV = take((size_t)E * 96); DPRE = take((size_t)E);
    DE = take((size_t)E * d.Ed); DXI = take((size_t)E * 3 * d.Xd);
    PI = take((size_t)N * 256); PJ = take((size_t)N * 256); DVQ = take((size_t)Mx * 48);
    for (int l = 0; l < d.L; ++l) { layers[l].msg[0].pi = PI; layers[l].msg[0].pj = PJ; }
    have_tape = false;
    return used;
  }

  void colsum(const float* A, long long M, int N, int lda, float* out) {
    const long long J = (M + kColsumRows - 1) / kColsumRows;
    be.run(J * N, FColsum1{A, M, N, lda, sc.part});
    be.run(N, FColsum2{sc.part, J, N, out});
  }

  // ---------------------------------------------------------------------------------------------- GCP forward
  void gcp_forward(Gcp& g, float* s_out, int ld_so, const float* res_s, int ld_rs, float* v_out, int ld_vo,
                   const float* res_v, int ld_rv, const unsigned char* mask) {
    const long long M = g.M;
    if (M == 0) return;
    be.gemm(false, true, M * 3, g.H, g.V_in, g.vt, g.ldv, g.Wd, g.V_in, g.hid, g.H, 0.f);          // vector_down
    be.gemm(false, true, M * 3, 3, g.V_in, g.vt, g.ldv, g.Wf, g.V_in, g.vdf, 3, 0.f);              // vector_down_frames
    be.run(M * (g.H + 9), FMerge{g.hid, g.vdf, g.frames, g.merged, g.S_in, g.H, g.fan});
    const float* bias = g.bs;
    const float* Wm = g.Ws + g.wcol;      // the block of scalar_out's weight that multiplies `merged`
    if (g.ff) {
      be.gemm(false, true, M, g.S_out, g.fan, g.merged, g.fan, Wm, g.fanW, g.z1, g.S_out, 0.f);
      be.run(M * g.S_out, FBiasSilu{g.z1, g.bs, g.aff, g.S_out});
      be.gemm(false, true, M, g.S_out, g.S_out, g.aff, g.S_out, g.W2, g.S_out, g.z, g.S_out, 0.f);
      bias = g.b2;
    } else {
      be.gemm(false, true, M, g.S_out, g.fan, g.merged, g.fan, Wm, g.fanW, g.z, g.S_out, 0.f);
      if (g.split) be.gemm(false, true, M, g.S_out, g.Ed, g.ee, g.Ed, g.Ws + 256, g.fanW, g.z, g.S_out, 1.f);   // + e.We^T
    }
    be.run(M * g.S_out, FScalarOut{g.z, bias, g.S_out, g.act0, g.act1, s_out, ld_so, res_s, ld_rs, mask,
                                   g.a1t, g.split ? g.pi : nullptr, g.pj, g.rc});
    if (!g.V_out) return;
    be.gemm(false, true, M * 3, g.V_out, g.H, g.hid, g.H, g.Wu, g.H, g.up, g.V_out, 0.f);           // vector_up
    be.gemm(false, true, M, g.V_out, g.S_out, g.a1t, g.S_out, g.Wg, g.S_out, g.sg, g.V_out, 0.f);   // vector_out_scale
    be.run(M * g.V_out, FVecOut{g.sg, g.bg, g.up, g.V_out, v_out, ld_vo, res_v, ld_rv, mask});
  }

  // ---------------------------------------------------------------------------------------------- GCP backward
  // (d s_out [M, ld_ds] or null, d v_out [M*3, ld_dv] or null) -> input gradients as `o` says (see BwdOut).  Parameter
  // gradients are accumulated.  On return sc.dz (ff: sc.dgz) still holds d z of the scalar_out linear map.
  void gcp_backward(Gcp& g, const float* ds_out, int ld_ds, const float* dv_out, int ld_dv, const BwdOut& o) {
    const long long M = g.M;
    if (M == 0) return;
    const float* dgz = nullptr;
    if (g.V_out) {
      be.run(M * g.V_out, FDVecOut{dv_out, g.up, g.sg, ld_dv, g.V_out, sc.dg, sc.dup});
      be.gemm(true, false, g.V_out, g.S_out, M, sc.dg, g.V_out, g.a1t, g.S_out, g.gWg, g.S_out, 1.f);
      colsum(sc.dg, M, g.V_out, g.V_out, g.gbg);
      be.gemm(false, false, M, g.S_out, g.V_out, sc.dg, g.V_out, g.Wg, g.S_out, sc.dgz, g.S_out, 0.f);
      be.gemm(true, false, g.V_out, g.H, M * 3, sc.dup, g.V_out, g.hid, g.H, g.gWu, g.H, 1.f);
      be.gemm(false, false, M * 3, g.H, g.V_out, sc.dup, g.V_out, g.Wu, g.H, sc.dhid, g.H, 0.f);
      dgz = sc.dgz;
    }
    be.run(M * g.S_out, FDZ{ds_out, ld_ds, dgz, g.z, g.S_out, g.act0, g.act1, sc.dz});
    const float* dzz = sc.dz;             // gradient at the output of the linear map that reads `merged`
    if (g.ff) {
      be.gemm(true, false, g.S_out, g.S_out, M, sc.dz, g.S_out, g.aff, g.S_out, g.gW2, g.S_out, 1.f);
      colsum(sc.dz, M, g.S_out, g.S_out, g.gb2);
      be.gemm(false, false, M, g.S_out, g.S_out, sc.dz, g.S_out, g.W2, g.S_out, sc.dgz, g.S_out, 0.f);
      be.run(M * g.S_out, FMulDSilu{sc.dgz, g.z1});
      dzz = sc.dgz;
    }
    be.gemm(true, false, g.S_out, g.fan, M, dzz, g.S_out, g.merged, g.fan, g.gWs + g.wcol, g.fanW, 1.f);
    colsum(dzz, M, g.S_out, g.S_out, g.gbs);
    if (o.ds_dst && g.S_in)
      be.gemm(false, false, M, g.S_in, g.S_out, dzz, g.S_out, g.Ws + g.wcol, g.fanW, o.ds_dst, o.ld_ds, o.beta_ds);
    be.gemm(false, false, M, g.H + 9, g.S_out, dzz, g.S_out, g.Ws + g.wcol + g.S_in, g.fanW, DVQ, g.H + 9, 0.f);
    be.run(M * g.H, FDNorm{DVQ, g.H + 9, g.H, g.hid, sc.dhid, g.V_out ? 1 : 0});
    be.run(M * 9, FDQ{DVQ, g.H + 9, g.H, g.frames, sc.dvdf});
    be.gemm(true, false, 3, g.V_in, M * 3, sc.dvdf, 3, g.vt, g.ldv, g.gWf, g.V_in, 1.f);
    be.gemm(true, false, g.H, g.V_in, M * 3, sc.dhid, g.H, g.vt, g.ldv, g.gWd, g.V_in, 1.f);
    if (o.dvt) {
      be.gemm(false, false, M * 3, g.V_in, 3, sc.dvdf, 3, g.Wf, g.V_in, o.dvt, o.ld_dvt, o.beta_dvt);
      be.gemm(false, false, M * 3, g.V_in, g.H, sc.dhid, g.H, g.Wd, g.V_in, o.dvt, o.ld_dvt, 1.f);
    }
  }

  // ---------------------------------------------------------------------------------------------- network forward
  // GCPNetDynamics.atom_types_and_coords_forward (gcpnet.py:1069-1232); keeps the tape for backward().
  void forward(const float* xh, const float* t, const float* ctx, float* net_out) {
    const long long N = tp.N, E = tp.E;
    const EdgeRc* rc = tp.edge_rc;
    be.run(N, FFillInt{apos, -1});
    be.run(tp.Mact, FApos{tp, apos});
    be.run(N, FPrepNodes{xh, t, ctx, tp.mask, x_init, g_node.merged, d.F, d.C, d.Hin, g_node.fan});
    be.run(N, FCentre{tp, x_init, x0});
    be.run(N, FOrient{x_init, chi_in, (int)N});
    be.run(E, FEdgeGeom{rc, x_init, x0, g_edge.merged, xi_in, frames, g_edge.fan});
    be.run(N * 9, FNodeFbar{tp, apos, frames, fbar});
    gcp_forward(g_edge, EE, d.Ed, nullptr, 0, XI, d.Xd, nullptr, 0, nullptr);
    gcp_forward(g_node, layers[0].ff.merged + 256, layers[0].ff.fan, nullptr, 0, layers[0].FV + 32, 64, nullptr, 0, nullptr);
    const float* xcur = x0;
    for (int l = 0; l < d.L; ++l) {
      Layer& y = layers[l];
      const float* h = y.ff.merged + 256; const int ldh = y.ff.fan;      // this layer's input (h, chi) lives inside the
      const float* chi = y.FV + 32; const int ldc = 64;                   // feed-forward GCP's concatenated inputs
      Gcp& m0 = y.msg[0];
      // split form: the endpoint parts of scalar_out are node-level GEMMs, gathered in FScalarOut
      be.gemm(false, true, N, 256, 256, h, ldh, m0.Ws, m0.fanW, PI, 256, 0.f);
      be.gemm(false, true, N, 256, 256, h, ldh, m0.Ws + 256 + d.Ed, m0.fanW, PJ, 256, 0.f);
      be.run(E * 3 * (64 + d.Xd), FGatherV{rc, chi, ldc, XI, d.Xd, m0.vt});
      gcp_forward(m0, y.msg[1].merged, y.msg[1].fan, nullptr, 0, y.V[0], 32, nullptr, 0, nullptr);
      for (int k = 1; k < 4; ++k) {                                       // residual message GCPs (gcpnet.py:698-701)
        Gcp& mk = y.msg[k];
        float* so = k < 3 ? y.msg[k + 1].merged : y.S3;
        const int ldo = k < 3 ? y.msg[k + 1].fan : 256;
        gcp_forward(mk, so, ldo, mk.merged, mk.fan, y.V[k], 32, y.V[k - 1], 32, nullptr);
      }
      be.gemm(false, true, E, 1, 256, y.S3, 256, y.wa, 256, y.attn, 1, 0.f);  // scalar message attention (:709-711)
      be.run(E, FSigmoidBias{y.attn, y.ba});
      be.run(N * 256, FAggS{tp, apos, y.S3, y.attn, y.ff.merged, y.ff.fan});
      be.run(N * 96, FAggV{tp, apos, y.V[3], y.FV, 64});
      gcp_forward(y.ff, y.pos.merged, y.pos.fan, h, ldh, y.CHI2, 32, chi, ldc, tp.mask);   // (:897-915)
      gcp_forward(y.pos, nullptr, 0, nullptr, 0, y.Xn, 1, xcur, 1, tp.mask);               // (:852, 922-928)
      xcur = y.Xn;
      if (l + 1 < d.L) {
        Layer& nx = layers[l + 1];
        be.run(N * 256, FCopy2D{y.pos.merged, y.pos.fan, nx.ff.merged + 256, nx.ff.fan, 256});
        be.run(N * 96, FCopy2D{y.CHI2, 32, nx.FV + 32, 64, 32});
      } else {
        be.run(N * 256, FCopy2D{y.pos.merged, y.pos.fan, g_proj.merged, g_proj.fan, 256});
      }
    }
    gcp_forward(g_proj, HP, d.Hin, nullptr, 0, nullptr, 0, nullptr, 0, nullptr);
    be.run(N, FFinal{tp, xcur, x_init, HP, d.Hin, d.F, net_out});
    have_tape = true;
  }

  // ---------------------------------------------------------------------------------------------- network backward
  // Accumulates d/dtheta sum(net_out * d_out) into the gradient slots (zeroed here first).
  void backward(const float* d_out) {
    const long long N = tp.N, E = tp.E;
    const EdgeRc* rc = tp.edge_rc;
    if (grad_count) be.run((long long)grad_count, FFill{grad_base, 0.f});
    be.run(N, FDFinal{tp, d_out, d.F, d.Hin, DX, DHP});
    gcp_backward(g_proj, DHP, d.Hin, nullptr, 0, BwdOut{DH, 256, 0.f, DCHI, 32, 0.f});
    if (E) { be.run(E * d.Ed, FFill{DE, 0.f}); be.run(E * 3 * d.Xd, FFill{DXI, 0.f}); }
    for (int l = d.L - 1; l >= 0; --l) {
      Layer& y = layers[l];
      Gcp& m0 = y.msg[0];
      const float* h = y.ff.merged + 256; const int ldh = y.ff.fan;
      // x_{l+1} = (x_l + pv) * mask and the frames are frozen: d x is the same masked vector at every layer
      gcp_backward(y.pos, nullptr, 0, DX, 1, BwdOut{DMN, 256, 0.f, DFV, 32, 0.f});
      be.run(N * 256, FMaskAdd{DH, 256, DMN, 256, 256, 1, tp.mask});
      be.run(N * 96, FMaskAdd{DCHI, 32, DFV, 32, 32, 3, tp.mask});
      // feed-forward GCP: d[agg_s | h] -> DMN [N, 512], d[agg_v | chi] -> DFV [N*3, 64]
      gcp_backward(y.ff, DH, 256, DCHI, 32, BwdOut{DMN, 512, 0.f, DFV, 64, 0.f});
      // message passing: d agg_s = DMN[:, :256], d agg_v = DFV[:, :32]
      if (E) {
        be.run(E, FDAttnPre{rc, DMN, 512, y.S3, y.attn, DPRE});
        be.gemm(true, false, 1, 256, E, DPRE, 1, y.S3, 256, y.gwa, 256, 1.f);
        colsum(DPRE, E, 1, 1, y.gba);
        be.run(E * 256, FDAttnS{rc, DMN, 512, y.attn, DPRE, y.wa, DS});
        be.run(E * 96, FGatherRowV{rc, DFV, 64, DV});
        for (int k = 3; k >= 1; --k)
          gcp_backward(y.msg[k], DS, 256, DV, 32, BwdOut{DS, 256, 1.f, DV, 32, 1.f});    // residual: += in place
        gcp_backward(m0, DS, 256, DV, 32, BwdOut{nullptr, 0, 0.f, DMV, 64 + d.Xd, 0.f});
      }
      be.run(N * 256, FAdd2D{DMN + 256, 512, DH, 256, 256});
      be.run(N * 96, FAdd2D{DFV + 32, 64, DCHI, 32, 32});
      if (E) {
        // split message GCP 0: sc.dz is d z0 [E, 256].  e block of the weight, then the node-level endpoint blocks
        be.gemm(true, false, 256, d.Ed, E, sc.dz, 256, EE, d.Ed, m0.gWs + 256, m0.fanW, 1.f);
        be.gemm(false, false, E, d.Ed, 256, sc.dz, 256, m0.Ws + 256, m0.fanW, DE, d.Ed, 1.f);
        be.run(N * 256, FScatterDZ{tp, apos, sc.dz, PI, PJ});        // PI / PJ reused as d PI / d PJ
        be.gemm(true, false, 256, 256, N, PI, 256, h, ldh, m0.gWs, m0.fanW, 1.f);
        be.gemm(true, false, 256, 256, N, PJ, 256, h, ldh, m0.gWs + 256 + d.Ed, m0.fanW, 1.f);
        be.gemm(false, false, N, 256, 256, PI, 256, m0.Ws, m0.fanW, DH, 256, 1.f);
        be.gemm(false, false, N, 256, 256, PJ, 256, m0.Ws + 256 + d.Ed, m0.fanW, DH, 256, 1.f);
        be.run(N * 96, FScatterV{tp, apos, DMV, 64 + d.Xd, d.Xd, DCHI, 32});
        be.run(E * 3 * d.Xd, FAdd2D{DMV + 32, 64 + d.Xd, DXI, d.Xd, d.Xd});
      }
    }
    // embedding inputs are data: no input gradient
    gcp_backward(g_node, DH, 256, DCHI, 32, BwdOut{});
    gcp_backward(g_edge, DE, d.Ed, DXI, d.Xd, BwdOut{});
  }
};

}  // namespace train
}  // namespace bdiff
