// train_hostcheck.cpp — TEST INFRASTRUCTURE ONLY (never linked into libbdiff_sm90.so, never on the product path).
//
// Compiles the product's training pass (bio-diffusion_b200/csrc/bdiff_train_engine.cuh: the functors every CUDA kernel
// of bdiff_train.cu executes and the orchestration of the GEMMs between them) against a host backend — plain loops and
// a naive GEMM — so that tests/test_train_hostcheck.py can compare it with torch.autograd through the oracle on the
// CPU-only build container.  What this does NOT cover is the CUDA backend itself (kernel launch wrapper, the cuBLAS
// row-major adapter): tests/test_gpu_train.py checks those on the device against the reference's gradient fixtures.
#include <cstring>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "../../bio-diffusion_b200/csrc/bdiff_train_engine.cuh"

using namespace bdiff::train;

namespace {
struct HostBackend {
  template <class F>
  void run(long long n, const F& f) {      // every functor writes only its own output elements: any order / parallelism is valid
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < n; ++i) f(i);
  }
  // row-major  C[M,N] = op(A)[M,K] * op(B)[K,N] + beta * C
  // (the leading-dimension rules of cuBLAS are enforced so that an illegal call fails here, not on the GPU)
  int bad_ld = 0;
  void gemm(bool ta, bool tb, long long M, int N, long long K, const float* A, int lda, const float* B, int ldb, float* C,
            int ldc, float beta) {
    if (lda < (ta ? M : K) || ldb < (tb ? K : N) || ldc < N || lda < 1 || ldb < 1) ++bad_ld;
#pragma omp parallel for collapse(2) schedule(static)
    for (long long m = 0; m < M; ++m)
      for (int n = 0; n < N; ++n) {
        double acc = 0.0;
        for (long long k = 0; k < K; ++k) {
          const float a = ta ? A[k * lda + m] : A[m * lda + k];
          const float b = tb ? B[(long long)n * ldb + k] : B[k * ldb + n];
          acc += (double)a * (double)b;
        }
        C[m * ldc + n] = (float)(acc + (beta != 0.f ? (double)beta * C[m * ldc + n] : 0.0));
      }
  }
};
}  // namespace

extern "C" int hostcheck_train(const int* dims, int B, int N, long long E, int Mact, const int* mol_off, const int* act_off,
                               const int* act_idx, const long long* edge_off, const int* node_mol, const unsigned char* mask,
                               const int* edge_rc, const char* names, const long long* offsets, int nparams,
                               const float* params, float* grads, long long nfloats, const float* xh, const float* t,
                               const float* ctx, const float* d_out, float* net_out) {
  NetDims d{dims[0], dims[1], dims[2], dims[3], dims[4], dims[5]};
  Topo tp;
  tp.B = B; tp.N = N; tp.E = E; tp.Mact = Mact;
  tp.mol_off = mol_off; tp.act_off = act_off; tp.act_idx = act_idx; tp.edge_off = edge_off; tp.node_mol = node_mol;
  tp.mask = mask; tp.edge_rc = reinterpret_cast<const EdgeRc*>(edge_rc);
  std::map<std::string, long long> off;
  {
    std::stringstream ss(names);
    std::string line;
    int i = 0;
    while (std::getline(ss, line, '\n') && i < nparams) off[line] = offsets[i++];
  }
  int missing = 0;
  auto look = [&](const std::string& name) -> ParamRef {
    auto it = off.find(name);
    if (it == off.end()) { ++missing; return ParamRef{params, grads}; }
    return ParamRef{params + it->second, grads + it->second};
  };
  HostBackend be;
  Engine<HostBackend> eng(be);
  const size_t need = eng.layout(d, tp, nullptr, look);
  if (missing) return -missing;
  std::vector<float> arena(need, 0.f);
  missing = 0;
  eng.layout(d, tp, arena.data(), look);
  eng.grad_base = grads;
  eng.grad_count = (size_t)nfloats;
  eng.forward(xh, t, ctx, net_out);
  eng.backward(d_out);
  return be.bad_ld ? 1000000 + be.bad_ld : 0;
}
