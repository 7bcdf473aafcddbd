// bdiff_handle.h — the state behind the opaque `bdiff_handle` of include/bdiff.h (internal; shared by bdiff_api.cu and
// bdiff_train.cu).
#pragma once
#include <cstdarg>
#include <cstdio>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "../../include/bdiff.h"
#include "bdiff_kernels.h"

namespace bdiff {

struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  cudaError_t ensure(size_t need) {
    if (need <= bytes) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    bytes = 0;
    cudaError_t e = cudaMalloc(&p, need);
    if (e != cudaSuccess) return e;
    bytes = need;
    return cudaMemset(p, 0, need);
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    bytes = 0;
  }
};

inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

struct TrainState;     // bdiff_train.cu
void train_destroy(TrainState*);

}  // namespace bdiff

using namespace bdiff;

struct bdiff_handle {
  bdiff_config cfg{};
  Dims d{};
  std::string err;
  int64_t launches = 0;

  // packed weights
  float* wbuf = nullptr;
  size_t wfloats = 0, wused = 0;
  std::vector<LayerW> layers;
  EmbedW embed{};
  std::map<std::string, bool> seen;   // reference parameter name -> set?
  // raw copies of the reference tensors + the slice table: all slices are repacked by ONE kernel in bdiff_prepare
  DevBuf stage_buf, jobs_dev;
  size_t stage_used = 0;
  std::map<std::string, size_t> stage_off;      // parameter name -> offset (floats) of its raw copy
  std::vector<PackJob> jobs;
  int pack_blocks = 0;
  bool pack_dirty = false, jobs_uploaded = false;

  // canonical flat layout of the reference parameter tensors (name -> {offset, count} in floats, names ascending):
  // the training pass reads parameters from / writes gradients to flat buffers of `param_floats` floats in this layout
  std::map<std::string, std::pair<size_t, size_t>> param_layout;
  size_t param_floats = 0;
  TrainState* train = nullptr;
  int plan_epoch = 0;    // bumped by every bdiff_plan_topology that builds a plan or, failing, drops one
  int Mact = 0;          // unmasked nodes of the current plan

  // plan
  bool have_plan = false;
  Plan plan{};
  DevBuf plan_buf, rc_buf, layers_dev, sched_buf;
  LayerSched sched{};

  // workspace
  DevBuf work_buf;
  Work work{};
  DevBuf eps_buf;      // [N,3+F] denoiser output inside reverse_step / decode
  DevBuf dbg_buf;      // clock64 stamps (BDIFF_TIMING=1)
  DevBuf tu_buf;       // uniform t scalar

  // tensor-core path state (bdiff_edge_tc.cu): per-layer pre-swizzled bf16 weight blobs
  DevBuf tc_blob, tc_node_blob;
  size_t tc_layer_bytes = 0, tc_node_layer_bytes = 0;
  bool tc_dirty = true;
  int num_sms = 132;
  cudaStream_t side = nullptr;          // fork/join stream: the edge embedding runs next to the node embedding
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;

  // bdiff_sample: sampling constants, the chain's buffers, and the captured reverse step with the key it was built for
  int weights_epoch = 0;                // bumped by every bdiff_set_weight
  bool have_sample_cfg = false;
  bdiff_sample_config scfg{};
  DevBuf smp_buf;                       // batch_index, mask, z, decoded xh, ctx, coef table, decode row, counters, CoG sums
  std::vector<int32_t> smp_counts;      // the batch of the handle's plan when bdiff_sample built it ...
  int smp_plan_epoch = -1;              // ... and the plan epoch that plan got
  cudaStream_t smp_stream = nullptr;    // the chain runs here when the caller passes the legacy stream (not capturable)
  cudaEvent_t smp_ev = nullptr;
  cudaGraphExec_t smp_graph = nullptr;
  std::vector<long long> smp_graph_key;
  int64_t smp_step_launches = 0;        // kernels in one captured reverse step
  int64_t smp_graph_builds = 0;
  DevBuf smp_slot, smp_frames;          // bdiff_sample_frames: frame slot per step, frame rows (+ the dummy slot)
  // bdiff_inpaint: the chain's per-atom buffers, the program's tables, and the captured op and jump bodies
  DevBuf inp_buf, inp_rev, inp_known, inp_slot, inp_draw, inp_jump, inp_jdraw;
  std::vector<int32_t> inp_counts;
  int inp_plan_epoch = -1;
  cudaGraphExec_t inp_op_graph = nullptr, inp_jump_graph = nullptr;
  std::vector<long long> inp_graph_key;
  int64_t inp_op_launches = 0, inp_jump_launches = 0, inp_graph_builds = 0;

  int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    err = buf;
    return code;
  }
  float* walloc(size_t n) {
    n = (n + 63) / 64 * 64;   // 256-byte granularity keeps every matrix 16 B aligned for bulk copies
    float* r = wbuf + wused;
    wused += n;
    return r;
  }
};

