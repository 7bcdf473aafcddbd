// bdiff_train.cu — CUDA backend + C ABI of the denoiser's training pass (forward with tape, backward): the functors of
// bdiff_train_engine.cuh run as grid-stride-free element kernels (one thread per output element, coalesced along the
// fastest index), the GEMMs between them are cuBLAS SGEMM calls (plain library GEMMs in the reference's row-major
// layout; fp32 by default, TF32 tensor cores on request).  Everything runs on the caller's stream, no host
// synchronisation, no atomics: gradients are bit-reproducible from run to run.
#include <cublas_v2.h>
#include <cxxabi.h>

#include <algorithm>
#include <typeinfo>

#include <cstring>

#include "bdiff_handle.h"
#include "bdiff_train_engine.cuh"

namespace bdiff {

template <class F>
__global__ void __launch_bounds__(256) k_train(long long n, F f) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i < n) f(i);
}

// Optional per-operation timing (bdiff_train_timing): a CUDA event pair around every kernel / GEMM on the launch stream.
struct OpTimer {
  bool on = false;
  std::vector<cudaEvent_t> ev;
  size_t used = 0;
  std::vector<std::pair<std::string, size_t>> recs;     // (operation, index of its first event)
  long long E = 0, N = 0;                              // to print GEMM shapes symbolically
  cudaEvent_t next() {
    if (used == ev.size()) {
      cudaEvent_t e;
      cudaEventCreate(&e);
      ev.push_back(e);
    }
    return ev[used++];
  }
  std::string dim(long long x) const {
    if (E > 0 && x == E) return "E";
    if (E > 0 && x == 3 * E) return "3E";
    if (N > 0 && x == N) return "N";
    if (N > 0 && x == 3 * N) return "3N";
    return std::to_string(x);
  }
};

struct CudaBackend {
  cudaStream_t st = nullptr;
  cublasHandle_t cb = nullptr;
  cublasStatus_t blas_err = CUBLAS_STATUS_SUCCESS;
  int64_t launches = 0, gemms = 0;
  OpTimer tm;
  template <class F>
  void run(long long n, const F& f) {
    if (n <= 0) return;
    cudaEvent_t e1 = nullptr;
    if (tm.on) {
      int status = 0;
      char* dn = abi::__cxa_demangle(typeid(F).name(), nullptr, nullptr, &status);
      std::string name = (status == 0 && dn) ? dn : typeid(F).name();
      if (dn) free(dn);
      const size_t pos = name.rfind("::");
      tm.recs.emplace_back("k_train<" + (pos == std::string::npos ? name : name.substr(pos + 2)) + ">", tm.used);
      cudaEventRecord(tm.next(), st);
      e1 = tm.next();
    }
    k_train<F><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, f);
    if (e1) cudaEventRecord(e1, st);
    ++launches;
  }
  // row-major C[M,N] = op(A)[M,K] * op(B)[K,N] + beta*C  ==  column-major C^T[N,M] = op(B)^T * op(A)^T
  void gemm(bool ta, bool tb, long long M, int N, long long K, const float* A, int lda, const float* B, int ldb, float* C,
            int ldc, float beta) {
    if (M <= 0 || N <= 0 || K <= 0) return;
    const float alpha = 1.0f;
    cudaEvent_t e1 = nullptr;
    if (tm.on) {
      tm.recs.emplace_back(std::string("cublasSgemm ") + (ta ? "T" : "N") + (tb ? "T" : "N") + " m=" + tm.dim(M) + " n=" +
                           std::to_string(N) + " k=" + tm.dim(K), tm.used);
      cudaEventRecord(tm.next(), st);
      e1 = tm.next();
    }
    cublasStatus_t s = cublasSgemm(cb, tb ? CUBLAS_OP_T : CUBLAS_OP_N, ta ? CUBLAS_OP_T : CUBLAS_OP_N, N, (int)M, (int)K, &alpha,
                                   B, ldb, A, lda, &beta, C, ldc);
    if (e1) cudaEventRecord(e1, st);
    if (s != CUBLAS_STATUS_SUCCESS && blas_err == CUBLAS_STATUS_SUCCESS) blas_err = s;
    ++gemms;
  }
};

struct TrainState {
  CudaBackend be;
  train::Engine<CudaBackend> eng{be};
  DevBuf arena;
  // what the current tape layout was built for
  int plan_epoch = -1;
  const float* params = nullptr;
  float* grads = nullptr;
  bool tf32 = false;
};

void train_destroy(TrainState* t) {
  if (!t) return;
  for (cudaEvent_t e : t->be.tm.ev) cudaEventDestroy(e);
  if (t->be.cb) cublasDestroy(t->be.cb);
  t->arena.release();
  delete t;
}

}  // namespace bdiff

namespace {

int32_t ensure_train(bdiff_handle* h, cudaStream_t st, const float* params, float* grads) {
  if (!h->have_plan) return h->fail(BDIFF_ESTATE, "bdiff_plan_topology has not been called");
  if (h->plan.E >= (1ll << 31) / 3) return h->fail(BDIFF_EINVAL, "too many edges for the training pass");
  if (!h->train) h->train = new TrainState();
  TrainState* t = h->train;
  if (!t->be.cb) {
    if (cublasCreate(&t->be.cb) != CUBLAS_STATUS_SUCCESS) { t->be.cb = nullptr; return h->fail(BDIFF_ECUDA, "cublasCreate failed"); }
    cublasSetMathMode(t->be.cb, t->tf32 ? CUBLAS_TF32_TENSOR_OP_MATH : CUBLAS_DEFAULT_MATH);
  }
  cublasSetStream(t->be.cb, st);
  t->be.st = st;
  if (t->plan_epoch == h->plan_epoch && t->params == params && (grads == nullptr || t->grads == grads)) return BDIFF_OK;
  train::NetDims d{h->d.F, h->d.C, h->d.Hin, h->d.Ed, h->d.Xd, h->d.L};
  train::Topo tp;
  const Plan& p = h->plan;
  tp.B = p.B; tp.N = p.N; tp.E = p.E; tp.Mact = h->Mact;
  tp.mol_off = p.mol_off; tp.act_off = p.act_off; tp.act_idx = p.act_idx; tp.edge_off = p.edge_off; tp.node_mol = p.node_mol;
  tp.mask = p.mask; tp.edge_rc = reinterpret_cast<const train::EdgeRc*>(p.edge_rc);
  int missing = 0;
  float* g = grads ? grads : t->grads;
  auto look = [&](const std::string& name) -> train::ParamRef {
    auto it = h->param_layout.find(name);
    if (it == h->param_layout.end()) { ++missing; return train::ParamRef{params, g}; }
    return train::ParamRef{params + it->second.first, g ? g + it->second.first : nullptr};
  };
  const bool same_shape = t->plan_epoch == h->plan_epoch;
  if (!same_shape) {
    const size_t need = t->eng.layout(d, tp, nullptr, look);
    if (missing) return h->fail(BDIFF_ESTATE, "internal: %d parameter names unknown to the training pass", missing);
    if (need * sizeof(float) > t->arena.bytes) {
      cudaError_t e = t->arena.ensure((need + need / 4) * sizeof(float));     // headroom: batches differ in size
      if (e != cudaSuccess) return h->fail(BDIFF_ENOMEM, "training tape (%.1f MiB): %s", need * 4.0 / 1048576.0, cudaGetErrorString(e));
    }
  }
  t->eng.layout(d, tp, static_cast<float*>(t->arena.p), look);
  t->eng.grad_base = g;
  t->eng.grad_count = g ? h->param_floats : 0;
  t->eng.have_tape = same_shape && t->params == params && t->eng.have_tape;
  t->plan_epoch = h->plan_epoch;
  t->params = params;
  t->grads = g;
  return BDIFF_OK;
}

int32_t finish(bdiff_handle* h, const char* what) {
  TrainState* t = h->train;
  h->launches += t->be.launches;
  t->be.launches = 0;
  if (t->be.blas_err != CUBLAS_STATUS_SUCCESS) {
    const int code = (int)t->be.blas_err;
    t->be.blas_err = CUBLAS_STATUS_SUCCESS;
    return h->fail(BDIFF_ECUDA, "%s: cuBLAS status %d", what, code);
  }
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? BDIFF_OK : h->fail(BDIFF_ECUDA, "%s: %s", what, cudaGetErrorString(e));
}

}  // namespace

extern "C" {

int64_t bdiff_param_floats(const bdiff_handle* h) { return h ? (int64_t)h->param_floats : 0; }

int32_t bdiff_param_layout(bdiff_handle* h, const char* name, int64_t* offset, int64_t* count) {
  if (!h || !name || !offset || !count) return h ? h->fail(BDIFF_EINVAL, "null argument") : BDIFF_EINVAL;
  auto it = h->param_layout.find(name);
  if (it == h->param_layout.end()) return h->fail(BDIFF_EINVAL, "unknown parameter name '%s'", name);
  *offset = (int64_t)it->second.first;
  *count = (int64_t)it->second.second;
  return BDIFF_OK;
}

int32_t bdiff_train_precision(bdiff_handle* h, int32_t tf32) {
  if (!h) return BDIFF_EINVAL;
  if (!h->train) h->train = new TrainState();
  h->train->tf32 = tf32 != 0;
  if (h->train->be.cb) cublasSetMathMode(h->train->be.cb, tf32 ? CUBLAS_TF32_TENSOR_OP_MATH : CUBLAS_DEFAULT_MATH);
  return BDIFF_OK;
}

int32_t bdiff_train_timing(bdiff_handle* h, void* stream, int32_t enable, char* report, int64_t report_bytes) {
  if (!h) return BDIFF_EINVAL;
  if (!h->train) h->train = new TrainState();
  OpTimer& tm = h->train->be.tm;
  if (enable) {
    tm.on = true;
    tm.used = 0;
    tm.recs.clear();
    tm.E = h->have_plan ? h->plan.E : 0;
    tm.N = h->have_plan ? h->plan.N : 0;
    return BDIFF_OK;
  }
  tm.on = false;
  cudaError_t e = cudaStreamSynchronize(static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "train_timing: %s", cudaGetErrorString(e));
  std::map<std::string, std::pair<int, double>> agg;
  double total = 0.0;
  for (auto& r : tm.recs) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, tm.ev[r.second], tm.ev[r.second + 1]) != cudaSuccess) continue;
    auto& a = agg[r.first];
    a.first += 1;
    a.second += ms;
    total += ms;
  }
  std::vector<std::pair<std::string, std::pair<int, double>>> rows(agg.begin(), agg.end());
  std::sort(rows.begin(), rows.end(), [](const auto& a, const auto& b) { return a.second.second > b.second.second; });
  std::string out;
  char line[256];
  snprintf(line, sizeof line, "%-44s %6s %10s %8s\n", "operation (E=%lld edges, N=%lld nodes)", "calls", "total_ms", "share");
  char hdr[256];
  snprintf(hdr, sizeof hdr, line, tm.E, tm.N);
  out += hdr;
  for (auto& r : rows) {
    snprintf(line, sizeof line, "%-44s %6d %10.3f %7.1f%%\n", r.first.c_str(), r.second.first, r.second.second,
             total > 0 ? 100.0 * r.second.second / total : 0.0);
    out += line;
  }
  snprintf(line, sizeof line, "%-44s %6zu %10.3f\n", "sum of the per-operation times", tm.recs.size(), total);
  out += line;
  if (report && report_bytes > 0) {
    const size_t n = std::min<size_t>(out.size(), (size_t)report_bytes - 1);
    memcpy(report, out.data(), n);
    report[n] = 0;
  }
  return BDIFF_OK;
}

int32_t bdiff_train_forward(bdiff_handle* h, void* stream, const float* params_flat, const float* xh, const float* t,
                            const float* context, float* net_out) {
  if (!h || !params_flat || !xh || !t || !net_out) return h ? h->fail(BDIFF_EINVAL, "null argument") : BDIFF_EINVAL;
  if (h->d.C > 0 && !context) return h->fail(BDIFF_EINVAL, "context required (num_context=%d)", h->d.C);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int32_t rc = ensure_train(h, st, params_flat, nullptr);
  if (rc != BDIFF_OK) return rc;
  h->train->eng.forward(xh, t, context, net_out);
  return finish(h, "train_forward");
}

int32_t bdiff_train_backward(bdiff_handle* h, void* stream, const float* d_net_out, float* grads_flat) {
  if (!h || !d_net_out || !grads_flat) return h ? h->fail(BDIFF_EINVAL, "null argument") : BDIFF_EINVAL;
  if (!h->train || !h->train->eng.have_tape || h->train->plan_epoch != h->plan_epoch)
    return h->fail(BDIFF_ESTATE, "bdiff_train_backward needs the tape of a bdiff_train_forward on the current plan");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  TrainState* t = h->train;
  if (t->grads != grads_flat) {
    // re-point the gradient slots (pointer arithmetic only; the tape itself does not move)
    const bool tape = t->eng.have_tape;
    int32_t rc = ensure_train(h, st, t->params, grads_flat);
    if (rc != BDIFF_OK) return rc;
    t->eng.have_tape = tape;
  } else {
    cublasSetStream(t->be.cb, st);
    t->be.st = st;
  }
  t->eng.backward(d_net_out);
  return finish(h, "train_backward");
}

}  // extern "C"
