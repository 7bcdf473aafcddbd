// bdiff_api.cu — the C ABI declared in include/bdiff.h: handle, weight repacking, topology plan, forward,
// reverse step.  Host-side logic only; kernels live in bdiff_kernels_fp32.cu / bdiff_edge_tc.cu.
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "../../include/bdiff.h"
#include "bdiff_handle.h"
#include "bdiff_plan.h"
#include "bdiff_schedule.h"

using namespace bdiff;

namespace {

thread_local std::string g_create_error;


}  // namespace

namespace {

// ------------------------------------------------------------------------------------------ weight layout
void gcp_names(std::map<std::string, bool>& seen, const std::string& p, bool ff, bool vout) {
  seen[p + "vector_down.weight"] = false;
  seen[p + "vector_down_frames.weight"] = false;
  if (ff) {
    seen[p + "scalar_out.0.weight"] = false; seen[p + "scalar_out.0.bias"] = false;
    seen[p + "scalar_out.2.weight"] = false; seen[p + "scalar_out.2.bias"] = false;
  } else {
    seen[p + "scalar_out.weight"] = false; seen[p + "scalar_out.bias"] = false;
  }
  if (vout) {
    seen[p + "vector_up.weight"] = false;
    seen[p + "vector_out_scale.weight"] = false; seen[p + "vector_out_scale.bias"] = false;
  }
}

size_t layout_weights(bdiff_handle* h, bool assign) {
  // When !assign only the size is computed (wbuf is null); offsets are deterministic so a second pass assigns.
  const Dims& d = h->d;
  h->wused = 0;
  auto A = [&](size_t n) -> float* { float* r = h->walloc(n); return assign ? r : nullptr; };
  EmbedW& e = h->embed;
  e.eWs = A((size_t)d.Ke * d.Ed); e.ebs = A(d.Ed); e.ewd = A(d.Xd); e.ewf = A(4);
  e.eWu = A((size_t)d.Xd * d.Xd); e.eWg = A((size_t)d.Ed * d.Xd); e.ebg = A(d.Xd);
  e.nWs = A((size_t)d.Kn * 256); e.nbs = A(256); e.nWd = A(2 * 32); e.nWf = A(2 * 3 + 2);
  e.nWu = A(32 * 32); e.nWg = A(256 * 32); e.nbg = A(32);
  e.pWs = A((size_t)300 * d.Hin); e.pbs = A(d.Hin); e.pWd = A(32 * 32); e.pWf = A(32 * 3);
  h->layers.assign(d.L, LayerW{});
  for (int l = 0; l < d.L; ++l) {
    LayerW& w = h->layers[l];
    w.W0e = A((size_t)d.K0 * 256); w.Wsi = A(256 * 256); w.Wsj = A(256 * 256); w.b0 = A(256);
    w.Wd0i = A(32 * d.hid0); w.Wd0x = A((size_t)d.Xd * d.hid0); w.Wd0j = A(32 * d.hid0);
    w.Wf0i = A(32 * 3); w.Wf0x = A(d.Xd * 3); w.Wf0j = A(32 * 3);
    w.Wu0 = A(d.hid0 * 32); w.Wg0 = A(256 * 32); w.bg0 = A(32);
    for (int k = 0; k < 3; ++k) {
      w.Wk[k] = A((size_t)kKM * 256); w.bk[k] = A(256); w.Wdk[k] = A(32 * kHidM); w.Wfk[k] = A(32 * 3);
      w.Wuk[k] = A(kHidM * 32); w.Wgk[k] = A(256 * 32); w.bgk[k] = A(32);
    }
    w.wa = A(256); w.ba = A(4);
    w.W1 = A((size_t)kKFF * 256); w.b1 = A(256); w.W2 = A(256 * 256); w.b2 = A(256);
    w.Wdf = A(64 * kHidFF); w.Wff = A(64 * 3); w.Wuf = A(kHidFF * 32); w.Wgf = A(256 * 32); w.bgf = A(32);
    w.Wp = A((size_t)kKM * 256); w.bp = A(256); w.Wdp = A(32 * kHidM); w.Wfp = A(32 * 3);
    w.Wup = A(kHidM); w.Wgp = A(256); w.bgp = A(4);
  }
  return h->wused;
}

struct PackOp {
  const float* dst; int dst_ld; int col0; int ncols; int kpad; int nout;
};

// Resolve a reference parameter name to its pack operations + expected shape.
bool resolve(bdiff_handle* h, const std::string& name, std::vector<PackOp>& ops, int64_t& rows, int64_t& cols) {
  const Dims& d = h->d;
  auto W = [&](const float* dst, int dst_ld, int col0, int ncols, int kpad, int nout) {
    ops.push_back(PackOp{dst, dst_ld, col0, ncols, kpad, nout});
  };
  auto gcp = [&](const std::string& leaf, const float* Ws, int s_in, int kpad_s, int nout_s, const float* bs,
                 const float* Wd, int v_in, int hid, const float* Wf, const float* Wu, int v_out,
                 const float* Wg, const float* bg) -> bool {
    const int fan = s_in + hid + 9;
    if (leaf == "scalar_out.weight") { rows = nout_s; cols = fan; W(Ws, nout_s, 0, fan, kpad_s, nout_s); return true; }
    if (leaf == "scalar_out.bias") { rows = nout_s; cols = 1; W(bs, nout_s, 0, 1, 1, nout_s); return true; }
    if (leaf == "vector_down.weight") { rows = hid; cols = v_in; W(Wd, hid, 0, v_in, v_in, hid); return true; }
    if (leaf == "vector_down_frames.weight") { rows = 3; cols = v_in; W(Wf, 3, 0, v_in, v_in, 3); return true; }
    if (Wu && leaf == "vector_up.weight") { rows = v_out; cols = hid; W(Wu, v_out, 0, hid, hid, v_out); return true; }
    if (Wg && leaf == "vector_out_scale.weight") { rows = v_out; cols = nout_s; W(Wg, v_out, 0, nout_s, nout_s, v_out); return true; }
    if (bg && leaf == "vector_out_scale.bias") { rows = v_out; cols = 1; W(bg, v_out, 0, 1, 1, v_out); return true; }
    return false;
  };
  const EmbedW& e = h->embed;
  const std::string pe = "gcp_embedding.edge_embedding.", pn = "gcp_embedding.node_embedding.",
                    pp = "scalar_node_projection_gcp.";
  if (name.rfind(pe, 0) == 0)
    return gcp(name.substr(pe.size()), e.eWs, 1, d.Ke, d.Ed, e.ebs, e.ewd, 1, d.Xd, e.ewf, e.eWu, d.Xd, e.eWg, e.ebg);
  if (name.rfind(pn, 0) == 0)
    return gcp(name.substr(pn.size()), e.nWs, d.Hin, d.Kn, 256, e.nbs, e.nWd, 2, 32, e.nWf, e.nWu, 32, e.nWg, e.nbg);
  if (name.rfind(pp, 0) == 0)
    return gcp(name.substr(pp.size()), e.pWs, 256, 300, d.Hin, e.pbs, e.pWd, 32, 32, e.pWf, nullptr, 0, nullptr, nullptr);
  int l = -1, consumed = 0;
  if (sscanf(name.c_str(), "interaction_layers.%d.%n", &l, &consumed) != 1 || l < 0 || l >= d.L) return false;
  const std::string rest = name.substr(consumed);
  const LayerW& w = h->layers[l];
  const std::string pm = "interaction.message_fusion.", pa = "interaction.scalar_message_attention.0.",
                    pf = "feedforward_network.0.", px = "node_position_update_gcp.";
  if (rest.rfind(pm, 0) == 0) {
    int k = -1, c2 = 0;
    if (sscanf(rest.c_str() + pm.size(), "%d.%n", &k, &c2) != 1 || k < 0 || k > 3) return false;
    const std::string leaf = rest.substr(pm.size() + c2);
    if (k > 0)
      return gcp(leaf, w.Wk[k - 1], 256, kKM, 256, w.bk[k - 1], w.Wdk[k - 1], 32, kHidM, w.Wfk[k - 1], w.Wuk[k - 1],
                 32, w.Wgk[k - 1], w.bgk[k - 1]);
    // k == 0: split form.  Torch columns of scalar_out: [h_row(256) | e(Ed) | h_col(256) | vn(hid0) | q(9)],
    // of vector_down / vector_down_frames: [chi_row(32) | xi(Xd) | chi_col(32)]   (gcpnet.py:694)
    const int fan = 512 + d.Ed + d.hid0 + 9, vin = 64 + d.Xd;
    if (leaf == "scalar_out.weight") {
      rows = 256; cols = fan;
      W(w.Wsi, 256, 0, 256, 256, 256);
      W(w.Wsj, 256, 256 + d.Ed, 256, 256, 256);
      W(w.W0e, 256, 256, d.Ed, d.Ed, 256);                                             // e rows
      W(w.W0e + (size_t)d.Ed * 256, 256, 512 + d.Ed, d.hid0 + 9, d.K0 - d.Ed, 256);     // vn, q rows + zero pad
      return true;
    }
    if (leaf == "scalar_out.bias") { rows = 256; cols = 1; W(w.b0, 256, 0, 1, 1, 256); return true; }
    if (leaf == "vector_down.weight") {
      rows = d.hid0; cols = vin;
      W(w.Wd0i, d.hid0, 0, 32, 32, d.hid0); W(w.Wd0x, d.hid0, 32, d.Xd, d.Xd, d.hid0);
      W(w.Wd0j, d.hid0, 32 + d.Xd, 32, 32, d.hid0);
      return true;
    }
    if (leaf == "vector_down_frames.weight") {
      rows = 3; cols = vin;
      W(w.Wf0i, 3, 0, 32, 32, 3); W(w.Wf0x, 3, 32, d.Xd, d.Xd, 3); W(w.Wf0j, 3, 32 + d.Xd, 32, 32, 3);
      return true;
    }
    if (leaf == "vector_up.weight") { rows = 32; cols = d.hid0; W(w.Wu0, 32, 0, d.hid0, d.hid0, 32); return true; }
    if (leaf == "vector_out_scale.weight") { rows = 32; cols = 256; W(w.Wg0, 32, 0, 256, 256, 32); return true; }
    if (leaf == "vector_out_scale.bias") { rows = 32; cols = 1; W(w.bg0, 32, 0, 1, 1, 32); return true; }
    return false;
  }
  if (rest.rfind(pa, 0) == 0) {
    const std::string leaf = rest.substr(pa.size());
    if (leaf == "weight") { rows = 1; cols = 256; W(w.wa, 1, 0, 256, 256, 1); return true; }
    if (leaf == "bias") { rows = 1; cols = 1; W(w.ba, 1, 0, 1, 1, 1); return true; }
    return false;
  }
  if (rest.rfind(pf, 0) == 0) {
    const std::string leaf = rest.substr(pf.size());
    if (leaf == "scalar_out.0.weight") { rows = 256; cols = 537; W(w.W1, 256, 0, 537, kKFF, 256); return true; }
    if (leaf == "scalar_out.0.bias") { rows = 256; cols = 1; W(w.b1, 256, 0, 1, 1, 256); return true; }
    if (leaf == "scalar_out.2.weight") { rows = 256; cols = 256; W(w.W2, 256, 0, 256, 256, 256); return true; }
    if (leaf == "scalar_out.2.bias") { rows = 256; cols = 1; W(w.b2, 256, 0, 1, 1, 256); return true; }
    return gcp(leaf, nullptr, 512, 0, 256, nullptr, w.Wdf, 64, kHidFF, w.Wff, w.Wuf, 32, w.Wgf, w.bgf);
  }
  if (rest.rfind(px, 0) == 0)
    return gcp(rest.substr(px.size()), w.Wp, 256, kKM, 256, w.bp, w.Wdp, 32, kHidM, w.Wfp, w.Wup, 1, w.Wgp, w.bgp);
  return false;
}

// Np / Ep: rows of the node / edge buffers
cudaError_t ensure_work(bdiff_handle* h, size_t Np, size_t Ep) {
  const Dims& d = h->d;
  size_t off = 0;
  auto take = [&](size_t n) { size_t o = off; off += (n + 63) / 64 * 64; return o; };
  const size_t o_xi = take(Np * 3), o_x = take(Np * 3), o_hin = take(Np * d.Hin), o_chin = take(Np * 6),
               o_fbar = take(Np * 12), o_h = take(Np * 256), o_chi = take(Np * 96), o_PI = take(Np * kPStride),
               o_PJ = take(Np * kPStride), o_agg = take(Np * kMsg), o_hp = take(Np * 32),
               o_e = take(Ep * d.Ed), o_xie = take(Ep * d.Xd * 3), o_fr = take(Ep * 9), o_pjt = take(Np * 256),
               o_mid = take(h->cfg.mode == BDIFF_MODE_TENSOR ? (Ep / 128) * kMsg : 0),
               o_acc = take(h->cfg.mode == BDIFF_MODE_TENSOR ? (size_t)h->num_sms * TM_COLS * 128 : 0),
               o_flag = take(64);
  cudaError_t e = h->work_buf.ensure(off * sizeof(float));
  if (e != cudaSuccess) return e;
  float* b = static_cast<float*>(h->work_buf.p);
  Work& w = h->work;
  w.x_init = b + o_xi; w.x = b + o_x; w.h_in = b + o_hin; w.chi_in = b + o_chin; w.fbar = b + o_fbar;
  w.h = b + o_h; w.chi = b + o_chi; w.PI = b + o_PI; w.PJ = b + o_PJ; w.agg = b + o_agg; w.hproj = b + o_hp;
  w.e = b + o_e; w.xi = b + o_xie; w.frames = b + o_fr;
  w.PJT = h->cfg.mode == BDIFF_MODE_TENSOR ? b + o_pjt : nullptr;
  w.mid = h->cfg.mode == BDIFF_MODE_TENSOR ? b + o_mid : nullptr;
  w.acc = h->cfg.mode == BDIFF_MODE_TENSOR ? b + o_acc : nullptr;
  w.npad = (int)Np;
  w.nan_flag = reinterpret_cast<int*>(b + o_flag);
  w.dbg = nullptr;
  if (getenv("BDIFF_TIMING")) {
    e = h->dbg_buf.ensure(2 * 256 * 64 * sizeof(long long));
    if (e != cudaSuccess) return e;
    w.dbg = static_cast<long long*>(h->dbg_buf.p);
  }
  e = h->eps_buf.ensure(Np * (3 + d.F) * sizeof(float));
  if (e != cudaSuccess) return e;
  return h->tu_buf.ensure(256);
}

}  // namespace

extern "C" {

int32_t bdiff_abi_version(void) { return BDIFF_ABI_VERSION; }

const char* bdiff_last_error(const bdiff_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int32_t bdiff_create(const bdiff_config* cfg, bdiff_handle** out) {
  if (!cfg || !out) { g_create_error = "null argument"; return BDIFF_EINVAL; }
  *out = nullptr;
  if (cfg->h_hidden != 256 || cfg->chi_hidden != 32) { g_create_error = "h_hidden must be 256 and chi_hidden 32"; return BDIFF_EINVAL; }
  if (cfg->e_hidden < 4 || cfg->e_hidden > 64 || cfg->e_hidden % 4) { g_create_error = "e_hidden must be a multiple of 4 in [4,64]"; return BDIFF_EINVAL; }
  if (cfg->xi_hidden < 4 || cfg->xi_hidden > 16 || cfg->xi_hidden % 4) { g_create_error = "xi_hidden must be a multiple of 4 in [4,16]"; return BDIFF_EINVAL; }
  if (cfg->num_h < 1 || cfg->num_context < 0 || cfg->num_h + 1 + cfg->num_context > 28) { g_create_error = "num_h + 1 + num_context must be in [2,28]"; return BDIFF_EINVAL; }
  if (cfg->num_layers < 1 || cfg->num_layers > 64) { g_create_error = "num_layers out of range"; return BDIFF_EINVAL; }
  if (cfg->mode != BDIFF_MODE_PARITY_FP32 && cfg->mode != BDIFF_MODE_TENSOR) { g_create_error = "unknown mode"; return BDIFF_EINVAL; }
  if (cfg->mode == BDIFF_MODE_TENSOR && !tc_supported(cfg->e_hidden, cfg->xi_hidden)) {
    g_create_error = "tensor mode supports (e_hidden, xi_hidden) in {(64,16), (16,8)} only";
    return BDIFF_EINVAL;
  }
  int dev_count = 0;
  if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count == 0) {
    g_create_error = "no CUDA device: libbdiff_sm90 has no CPU fallback";
    return BDIFF_ECUDA;
  }
  cudaDeviceProp prop{};
  int dev = 0;
  cudaGetDevice(&dev);
  cudaGetDeviceProperties(&prop, dev);
  if (prop.major != 9 || prop.minor != 0) {
    g_create_error = "libbdiff_sm90 is built for sm_90a (H100) only; found compute capability " +
                     std::to_string(prop.major) + "." + std::to_string(prop.minor);
    return BDIFF_ECUDA;
  }
  bdiff_handle* h = new bdiff_handle();
  h->cfg = *cfg;
  Dims& d = h->d;
  d.F = cfg->num_h; d.C = cfg->num_context; d.Hin = d.F + 1 + d.C; d.Ed = cfg->e_hidden; d.Xd = cfg->xi_hidden;
  d.hid0 = (64 + d.Xd) / 4;
  d.K0 = round_up(d.Ed + d.hid0 + 9, 4);
  d.Ke = round_up(1 + d.Xd + 9, 4);
  d.Kn = round_up(d.Hin + 32 + 9, 4);
  d.L = cfg->num_layers;
  if ((64 + d.Xd) % 4) { g_create_error = "2*chi_hidden + xi_hidden must be divisible by the bottleneck 4"; delete h; return BDIFF_EINVAL; }
  const size_t need = layout_weights(h, false);
  if (cudaMalloc(&h->wbuf, need * sizeof(float)) != cudaSuccess) { g_create_error = "cudaMalloc(weights) failed"; delete h; return BDIFF_ENOMEM; }
  cudaMemset(h->wbuf, 0, need * sizeof(float));
  h->wfloats = need;
  layout_weights(h, true);
  // the set of reference parameter names this configuration must receive
  gcp_names(h->seen, "gcp_embedding.edge_embedding.", false, true);
  gcp_names(h->seen, "gcp_embedding.node_embedding.", false, true);
  gcp_names(h->seen, "scalar_node_projection_gcp.", false, false);
  for (int l = 0; l < d.L; ++l) {
    const std::string p = "interaction_layers." + std::to_string(l) + ".";
    for (int k = 0; k < 4; ++k) gcp_names(h->seen, p + "interaction.message_fusion." + std::to_string(k) + ".", false, true);
    h->seen[p + "interaction.scalar_message_attention.0.weight"] = false;
    h->seen[p + "interaction.scalar_message_attention.0.bias"] = false;
    gcp_names(h->seen, p + "feedforward_network.0.", true, true);
    gcp_names(h->seen, p + "node_position_update_gcp.", false, true);
  }
  for (auto& kv : h->seen) {
    std::vector<PackOp> ops;
    int64_t rows = 0, cols = 0;
    if (!resolve(h, kv.first, ops, rows, cols)) { g_create_error = "internal: cannot place " + kv.first; cudaFree(h->wbuf); delete h; return BDIFF_EINVAL; }
    const size_t count = (size_t)rows * (size_t)cols;
    h->param_layout[kv.first] = {h->param_floats, count};
    h->param_floats += (count + 63) / 64 * 64;
  }
  h->num_sms = prop.multiProcessorCount;
  if (cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming) != cudaSuccess) {
    h->side = nullptr;               // fall back to a single stream
  }
  cudaError_t e = configure_kernels();
  if (e == cudaSuccess && cfg->mode == BDIFF_MODE_TENSOR) {
    e = tc_layers_configure();
    h->tc_layer_bytes = tc_blob_bytes(d.Ed, d.Xd);
    h->tc_node_layer_bytes = tc_node_blob_bytes();
    if (e == cudaSuccess) e = h->tc_blob.ensure(h->tc_layer_bytes * d.L);
    if (e == cudaSuccess) e = h->tc_node_blob.ensure(h->tc_node_layer_bytes * d.L);
  }
  if (e != cudaSuccess) {
    g_create_error = std::string("configure_kernels: ") + cudaGetErrorString(e);
    cudaFree(h->wbuf);
    delete h;
    return BDIFF_ECUDA;
  }
  *out = h;
  return BDIFF_OK;
}

void bdiff_destroy(bdiff_handle* h) {
  if (!h) return;
  if (h->wbuf) cudaFree(h->wbuf);
  if (h->train) train_destroy(h->train);
  if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  if (h->ev_join) cudaEventDestroy(h->ev_join);
  if (h->side) cudaStreamDestroy(h->side);
  if (h->smp_graph) cudaGraphExecDestroy(h->smp_graph);
  if (h->smp_ev) cudaEventDestroy(h->smp_ev);
  if (h->smp_stream) cudaStreamDestroy(h->smp_stream);
  if (h->inp_op_graph) cudaGraphExecDestroy(h->inp_op_graph);
  if (h->inp_jump_graph) cudaGraphExecDestroy(h->inp_jump_graph);
  h->smp_buf.release(); h->smp_slot.release(); h->smp_frames.release();
  for (DevBuf* b : {&h->inp_buf, &h->inp_rev, &h->inp_known, &h->inp_slot, &h->inp_draw, &h->inp_jump, &h->inp_jdraw})
    b->release();
  h->plan_buf.release(); h->rc_buf.release(); h->layers_dev.release(); h->sched_buf.release(); h->work_buf.release(); h->eps_buf.release(); h->tu_buf.release(); h->tc_blob.release(); h->tc_node_blob.release(); h->stage_buf.release(); h->jobs_dev.release();
  delete h;
}

int32_t bdiff_set_weight(bdiff_handle* h, void* stream, const char* name, const float* data, const int64_t* shape,
                         int32_t ndim) {
  if (!h || !name || !data || !shape || ndim < 1 || ndim > 2) return h ? h->fail(BDIFF_EINVAL, "bad argument") : BDIFF_EINVAL;
  auto it = h->seen.find(name);
  if (it == h->seen.end()) return h->fail(BDIFF_EINVAL, "unknown parameter name '%s'", name);
  std::vector<PackOp> ops;
  int64_t rows = 0, cols = 0;
  if (!resolve(h, name, ops, rows, cols)) return h->fail(BDIFF_EINVAL, "cannot place parameter '%s'", name);
  const int64_t got_rows = shape[0], got_cols = ndim == 2 ? shape[1] : 1;
  if (got_rows != rows || got_cols != cols)
    return h->fail(BDIFF_EINVAL, "parameter '%s': expected shape [%lld,%lld], got [%lld,%lld]", name, (long long)rows,
                   (long long)cols, (long long)got_rows, (long long)got_cols);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // raw copy into the staging area (device-to-device, stream ordered); the repack of all slices is one kernel in bdiff_prepare
  const size_t count = (size_t)rows * (size_t)cols;
  cudaError_t e = h->stage_buf.p ? cudaSuccess : h->stage_buf.ensure((h->wfloats + 64 * h->seen.size()) * sizeof(float));
  if (e != cudaSuccess) return h->fail(BDIFF_ENOMEM, "weight staging: %s", cudaGetErrorString(e));
  auto so = h->stage_off.find(name);
  size_t off;
  if (so == h->stage_off.end()) {
    off = h->stage_used;
    h->stage_used += (count + 63) / 64 * 64;
    if (h->stage_used * sizeof(float) > h->stage_buf.bytes) return h->fail(BDIFF_ENOMEM, "weight staging overflow");
    h->stage_off[name] = off;
    const float* src = static_cast<const float*>(h->stage_buf.p) + off;
    for (const PackOp& op : ops) {
      PackJob j{const_cast<float*>(op.dst), src, op.dst_ld, (int)cols, op.col0, op.ncols, op.kpad, op.nout, h->pack_blocks};
      h->pack_blocks += (op.kpad * op.nout + 255) / 256;
      h->jobs.push_back(j);
    }
    h->jobs_uploaded = false;
  } else {
    off = so->second;
  }
  e = cudaMemcpyAsync(static_cast<float*>(h->stage_buf.p) + off, data, count * sizeof(float), cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "stage '%s': %s", name, cudaGetErrorString(e));
  it->second = true;
  h->weights_epoch++;
  h->pack_dirty = true;
  h->tc_dirty = true;
  return BDIFF_OK;
}

static void tc_prepare(bdiff_handle* h, cudaStream_t st) {
  if (h->pack_dirty) {
    if (!h->jobs_uploaded && h->jobs_dev.ensure(h->jobs.size() * sizeof(PackJob)) == cudaSuccess) {
      cudaMemcpyAsync(h->jobs_dev.p, h->jobs.data(), h->jobs.size() * sizeof(PackJob), cudaMemcpyHostToDevice, st);
      cudaStreamSynchronize(st);    // pageable source; once per slice-table change, never inside a graph capture
      h->jobs_uploaded = true;
    }
    launch_pack_multi(st, static_cast<const PackJob*>(h->jobs_dev.p), (int)h->jobs.size(), h->pack_blocks);
    h->launches++;
    h->pack_dirty = false;
  }
  if (h->cfg.mode != BDIFF_MODE_TENSOR || !h->tc_dirty) return;
  for (int l = 0; l < h->d.L; ++l) {
    launch_tc_pack(st, h->layers[l], h->d, static_cast<unsigned char*>(h->tc_blob.p) + (size_t)l * h->tc_layer_bytes);
    const int last = (l == h->d.L - 1);
    unsigned char* nb = static_cast<unsigned char*>(h->tc_node_blob.p) + (size_t)l * h->tc_node_layer_bytes;
    launch_tc_pack_node(st, h->layers[l], h->layers[last ? l : l + 1], h->embed, h->d, last, nb);
    h->launches += 2;
  }
  if (h->layers_dev.ensure(h->layers.size() * sizeof(LayerW)) == cudaSuccess) {
    cudaMemcpyAsync(h->layers_dev.p, h->layers.data(), h->layers.size() * sizeof(LayerW), cudaMemcpyHostToDevice, st);
    cudaStreamSynchronize(st);      // pageable source; runs once per weight update, never inside a graph capture
  }
  h->tc_dirty = false;
}

int32_t bdiff_prepare(bdiff_handle* h, void* stream) {
  if (!h) return BDIFF_EINVAL;
  if (bdiff_weights_missing(h) != 0) return h->fail(BDIFF_ESTATE, "%d parameters not set", bdiff_weights_missing(h));
  tc_prepare(h, static_cast<cudaStream_t>(stream));
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? BDIFF_OK : h->fail(BDIFF_ECUDA, "prepare: %s", cudaGetErrorString(e));
}

int32_t bdiff_selftest_split(void* stream, int32_t variant, const float* A, const float* W, float* C) {
  if (!A || !W || !C) return BDIFF_EINVAL;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (selftest_configure() != cudaSuccess) return BDIFF_ECUDA;
  void* img = nullptr;
  if (cudaMalloc(&img, selftest_img_bytes()) != cudaSuccess) return BDIFF_ENOMEM;
  launch_wgmma_selftest_split(st, A, W, static_cast<unsigned char*>(img), C, variant);
  cudaError_t e = cudaStreamSynchronize(st);
  cudaFree(img);
  return e == cudaSuccess ? BDIFF_OK : BDIFF_ECUDA;
}

int32_t bdiff_weights_missing(const bdiff_handle* h) {
  if (!h) return BDIFF_EINVAL;
  int n = 0;
  for (auto& kv : h->seen) n += kv.second ? 0 : 1;
  return n;
}

int32_t bdiff_plan_topology(bdiff_handle* h, void* stream, int32_t num_mols, int64_t num_nodes,
                            const int64_t* batch_index, const uint8_t* mask, int64_t* num_edges_host) {
  if (!h) return BDIFF_EINVAL;
  if (!batch_index || !mask) return h->fail(BDIFF_EINVAL, "bad plan arguments");
  if (const char* why = plan_args_error(num_mols, num_nodes)) return h->fail(BDIFF_EINVAL, "%s", why);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int N = (int)num_nodes;
  std::vector<int64_t> bi(N);
  std::vector<uint8_t> mk(N);
  cudaError_t e = cudaMemcpyAsync(bi.data(), batch_index, N * sizeof(int64_t), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(mk.data(), mask, N, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "plan D2H: %s", cudaGetErrorString(e));
  HostPlan hp;
  const std::string why = plan_host(num_mols, num_nodes, bi.data(), mk.data(), h->d.L, h->num_sms, hp);
  if (!why.empty()) return h->fail(BDIFF_EINVAL, "%s", why.c_str());

  // From here on the buffers of the previous plan may be freed: a failure leaves no plan.
  auto lose = [&](int code, const char* what, cudaError_t err) {
    h->have_plan = false;
    h->plan_epoch++;
    return h->fail(code, "%s: %s", what, cudaGetErrorString(err));
  };
  const long long nrc = (long long)hp.TE * 128;
  const size_t nsched = 1 + (size_t)hp.nitems;       // queue head + one completion flag per item
  e = h->plan_buf.ensure(hp.at.bytes);
  if (e == cudaSuccess) e = h->rc_buf.ensure((size_t)std::max(nrc, 1ll) * sizeof(int4));
  if (e == cudaSuccess) e = h->sched_buf.ensure((nsched + 1) * sizeof(int));
  if (e != cudaSuccess) return lose(BDIFF_ENOMEM, "plan buffers", e);
  e = cudaMemcpyAsync(h->plan_buf.p, hp.block.data(), hp.at.bytes, cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return lose(BDIFF_ECUDA, "plan H2D", e);
  unsigned char* base = static_cast<unsigned char*>(h->plan_buf.p);
  Plan p{};
  p.B = hp.B; p.N = hp.N; p.E = hp.E;
  p.mol_off = reinterpret_cast<const int*>(base + hp.at.mol_off);
  p.act_off = reinterpret_cast<const int*>(base + hp.at.act_off);
  p.act_idx = reinterpret_cast<const int*>(base + hp.at.act_idx);
  p.node_mol = reinterpret_cast<const int*>(base + hp.at.node_mol);
  p.edge_off = reinterpret_cast<const long long*>(base + hp.at.edge_off);
  p.mask = base + hp.at.mask;
  p.node_mid = reinterpret_cast<const int2*>(base + hp.at.node_mid);
  launch_edge_rc(st, p, static_cast<int4*>(h->rc_buf.p), nrc);
  p.edge_rc = static_cast<const int4*>(h->rc_buf.p);
  e = cudaGetLastError();
  LayerSched q = h->sched;
  q.TE = hp.TE; q.TN = hp.TN; q.nitems = hp.nitems;
  q.edge_dep = reinterpret_cast<const int2*>(base + hp.at.edge_dep);
  q.node_dep = reinterpret_cast<const int2*>(base + hp.at.node_dep);
  q.items = reinterpret_cast<const int*>(base + hp.at.items);
  q.sched = static_cast<int*>(h->sched_buf.p);
  q.err = q.sched + nsched;
  if (e == cudaSuccess) e = cudaMemsetAsync(q.err, 0, sizeof(int), st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return lose(BDIFF_ECUDA, "plan upload", e);
  // node buffers carry one spare 128-row block, edge buffers one spare 128-edge tile
  e = ensure_work(h, round_up(hp.N, 128) + 128, (size_t)hp.TE * 128 + 128);
  if (e != cudaSuccess) return lose(BDIFF_ENOMEM, "workspace", e);
  h->plan = p;
  h->sched = q;
  h->Mact = hp.Mact;
  h->have_plan = true;
  h->plan_epoch++;
  if (num_edges_host) *num_edges_host = hp.E;
  return BDIFF_OK;
}

int32_t bdiff_edge_index(bdiff_handle* h, void* stream, int64_t* edge_index) {
  if (!h || !edge_index) return BDIFF_EINVAL;
  if (!h->have_plan) return h->fail(BDIFF_ESTATE, "no topology plan");
  launch_edge_index(static_cast<cudaStream_t>(stream), h->plan, reinterpret_cast<long long*>(edge_index));
  h->launches++;
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? BDIFF_OK : h->fail(BDIFF_ECUDA, "edge_index: %s", cudaGetErrorString(e));
}

static int32_t forward_impl(bdiff_handle* h, cudaStream_t st, const float* xh, const float* t_nodes,
                            const float* coef_table, const int* step_ptr, const float* context, float* net_out,
                            std::vector<cudaEvent_t>* ev = nullptr) {
  if (!h->have_plan) return h->fail(BDIFF_ESTATE, "bdiff_plan_topology has not been called");
  if (bdiff_weights_missing(h) != 0) {
    for (auto& kv : h->seen)
      if (!kv.second) return h->fail(BDIFF_ESTATE, "%d parameters not set, first missing: %s", bdiff_weights_missing(h), kv.first.c_str());
  }
  if (h->d.C > 0 && !context) return h->fail(BDIFF_EINVAL, "context required (num_context=%d)", h->d.C);
  const Plan& p = h->plan;
  const Dims& d = h->d;
  const Work& w = h->work;
  auto mark = [&]() {
    if (!ev) return;
    cudaEvent_t e;
    cudaEventCreate(&e);
    cudaEventRecord(e, st);
    ev->push_back(e);
  };
  tc_prepare(h, st);
  const bool tensor = h->cfg.mode == BDIFF_MODE_TENSOR;
  mark();
  launch_prep(st, p, d, xh, t_nodes, coef_table, step_ptr, context, w);
  mark();
  // the edge embedding (e, xi, frames) and the node embedding (+ layer-0 endpoint projections) are independent and
  // neither fills the chip: run them side by side (fork/join through events; also valid under stream capture).
  // With per-kernel timing marks requested they stay in order on one stream.
  const bool fork = h->side != nullptr && ev == nullptr;
  if (fork) {
    cudaEventRecord(h->ev_fork, st);
    cudaStreamWaitEvent(h->side, h->ev_fork, 0);
    launch_edge_embed(h->side, p, d, h->embed, w);
    cudaEventRecord(h->ev_join, h->side);
  } else {
    launch_edge_embed(st, p, d, h->embed, w);
  }
  mark();
  launch_node_embed(st, p, d, h->embed, h->layers[0], w);
  if (fork) cudaStreamWaitEvent(st, h->ev_join, 0);
  mark();
  h->launches += 4;
  const bool fused = tensor;
  if (fused) {
    // all L layers in one persistent kernel (bdiff_layers_tc.cu); its queue head + completion flags are zeroed first
    LayerSched& q = h->sched;
    q.layers = static_cast<const LayerW*>(h->layers_dev.p);
    q.edge_blob = static_cast<const unsigned char*>(h->tc_blob.p);
    q.edge_blob_stride = h->tc_layer_bytes;
    q.node_blob = static_cast<const unsigned char*>(h->tc_node_blob.p);
    q.node_blob_stride = h->tc_node_layer_bytes;
    q.L = d.L;
    cudaMemsetAsync(q.sched, 0, (1 + (size_t)q.nitems) * sizeof(int), st);
    launch_layers_tc(st, p, d, h->embed, q, w, h->num_sms);
    mark();
    h->launches += 1;
  }
  for (int l = 0; l < d.L && !fused; ++l) {
    launch_edge_message(st, p, d, h->layers[l], w);
    mark();
    const bool last = (l == d.L - 1);
    launch_node_update(st, p, d, h->layers[l], h->layers[last ? l : l + 1], h->embed, w, last ? 1 : 0);
    mark();
    h->launches += 2;
  }
  launch_finalize(st, p, d, w, net_out);
  mark();
  h->launches += 1;
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? BDIFF_OK : h->fail(BDIFF_ECUDA, "forward: %s", cudaGetErrorString(e));
}

int32_t bdiff_profile_forward(bdiff_handle* h, void* stream, const float* xh, const float* t, const float* context,
                              float* net_out, float* ms_host) {
  if (!h || !xh || !t || !net_out || !ms_host) return h ? h->fail(BDIFF_EINVAL, "null argument") : BDIFF_EINVAL;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  std::vector<cudaEvent_t> ev;
  int32_t rc = forward_impl(h, st, xh, t, nullptr, nullptr, context, net_out, &ev);
  cudaError_t e = cudaStreamSynchronize(st);
  if (rc == BDIFF_OK && e != cudaSuccess) rc = h->fail(BDIFF_ECUDA, "profile sync: %s", cudaGetErrorString(e));
  if (rc == BDIFF_OK && h->cfg.mode == BDIFF_MODE_TENSOR && h->sched_buf.p) {
    int flag = 0;
    cudaMemcpy(&flag, h->sched.err, sizeof(int), cudaMemcpyDeviceToHost);
    if (flag) { cudaMemset(h->sched.err, 0, sizeof(int)); rc = h->fail(BDIFF_ECUDA, "layer megakernel: a tile dependency wait timed out"); }
  }
  for (int i = 0; i < 8; ++i) ms_host[i] = 0.f;
  if (rc == BDIFF_OK) {
    auto dt = [&](size_t a, size_t b) { float ms = 0.f; cudaEventElapsedTime(&ms, ev[a], ev[b]); return ms; };
    const int L = h->d.L;
    ms_host[0] = dt(0, 1); ms_host[1] = dt(1, 2); ms_host[2] = dt(2, 3);
    if (ev.size() == 6) {          // fused layers: [prep | edge_embed | node_embed | k_layers_tc | finalize]
      ms_host[3] = dt(3, 4);       // reported in the edge_message slot; ms_host[7] < 0 marks the fusion
      ms_host[5] = dt(4, 5);
      ms_host[6] = dt(0, 5);
      ms_host[7] = -(float)L;
    } else {
      for (int l = 0; l < L; ++l) { ms_host[3] += dt(3 + 2 * l, 4 + 2 * l); ms_host[4] += dt(4 + 2 * l, 5 + 2 * l); }
      ms_host[5] = dt(3 + 2 * L, 4 + 2 * L);
      ms_host[6] = dt(0, 4 + 2 * L);
      ms_host[7] = (float)L;
    }
  }
  for (cudaEvent_t x : ev) cudaEventDestroy(x);
  return rc;
}

int32_t bdiff_denoise_forward(bdiff_handle* h, void* stream, const float* xh, const float* t, const float* context,
                              float* net_out) {
  if (!h || !xh || !t || !net_out) return h ? h->fail(BDIFF_EINVAL, "null argument") : BDIFF_EINVAL;
  return forward_impl(h, static_cast<cudaStream_t>(stream), xh, t, nullptr, nullptr, context, net_out);
}

int32_t bdiff_debug_tap(bdiff_handle* h, void* stream, const char* which, float* dst, int64_t* rows, int64_t* cols) {
  if (!h || !which || !rows || !cols) return BDIFF_EINVAL;
  if (!h->have_plan) return h->fail(BDIFF_ESTATE, "no topology plan");
  const std::string s = which;
  const Work& w = h->work;
  const Dims& d = h->d;
  const int64_t N = h->plan.N, E = h->plan.E;
  const float* src = nullptr;
  if (s == "f_ij") { src = w.frames; *rows = E; *cols = 9; }
  else if (s == "e") { src = w.e; *rows = E; *cols = d.Ed; }
  else if (s == "xi") { src = w.xi; *rows = E; *cols = d.Xd * 3; }
  else if (s == "h") { src = w.h; *rows = N; *cols = 256; }
  else if (s == "chi") { src = w.chi; *rows = N; *cols = 96; }
  else if (s == "x") { src = w.x; *rows = N; *cols = 3; }
  else if (s == "fbar") { src = w.fbar; *rows = N; *cols = 12; }
  else if (s == "chi_in") { src = w.chi_in; *rows = N; *cols = 6; }
  else if (s == "dbg" && w.dbg) { src = reinterpret_cast<const float*>(w.dbg); *rows = 512; *cols = 128; }
  else return h->fail(BDIFF_EINVAL, "unknown tap '%s'", which);
  if (dst && *rows * *cols > 0) {
    cudaError_t e = cudaMemcpyAsync(dst, src, (size_t)(*rows) * (*cols) * sizeof(float), cudaMemcpyDeviceToDevice,
                                    static_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "tap copy: %s", cudaGetErrorString(e));
  }
  return BDIFF_OK;
}

int32_t bdiff_reverse_step(bdiff_handle* h, void* stream, float* z, const float* context, const float* noise_x,
                           const float* noise_h, const float* coef_table, const int32_t* step_index) {
  if (!h || !z || !noise_x || !noise_h || !coef_table) return h ? h->fail(BDIFF_EINVAL, "null argument") : BDIFF_EINVAL;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* eps = static_cast<float*>(h->eps_buf.p);
  int32_t rc = forward_impl(h, st, z, nullptr, coef_table, step_index, context, eps);
  if (rc != BDIFF_OK) return rc;
  launch_step(st, h->plan, h->d, 0, z, eps, noise_x, noise_h, coef_table, step_index, z);
  h->launches++;
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? BDIFF_OK : h->fail(BDIFF_ECUDA, "reverse_step: %s", cudaGetErrorString(e));
}

int32_t bdiff_decode_z0(bdiff_handle* h, void* stream, const float* z0, const float* context, const float* noise_x,
                        const float* noise_h, const float* coef, float* xh) {
  if (!h || !z0 || !noise_x || !noise_h || !coef || !xh) return h ? h->fail(BDIFF_EINVAL, "null argument") : BDIFF_EINVAL;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* eps = static_cast<float*>(h->eps_buf.p);
  int32_t rc = forward_impl(h, st, z0, nullptr, coef, nullptr, context, eps);
  if (rc != BDIFF_OK) return rc;
  launch_step(st, h->plan, h->d, 1, z0, eps, noise_x, noise_h, coef, nullptr, xh);
  h->launches++;
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? BDIFF_OK : h->fail(BDIFF_ECUDA, "decode_z0: %s", cudaGetErrorString(e));
}

int32_t bdiff_center_noise(bdiff_handle* h, void* stream, const float* noise_x, const float* noise_h, float* z) {
  if (!h || !noise_x || !noise_h || !z) return h ? h->fail(BDIFF_EINVAL, "null argument") : BDIFF_EINVAL;
  if (!h->have_plan) return h->fail(BDIFF_ESTATE, "no topology plan");
  launch_step(static_cast<cudaStream_t>(stream), h->plan, h->d, 2, nullptr, nullptr, noise_x, noise_h, nullptr, nullptr, z);
  h->launches++;
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? BDIFF_OK : h->fail(BDIFF_ECUDA, "center_noise: %s", cudaGetErrorString(e));
}

int32_t bdiff_repaint_combine(bdiff_handle* h, void* stream, float* z, const float* xh0, const uint8_t* fixed,
                              const float* noise_x, const float* noise_h, const float* known_table,
                              const int32_t* op_index) {
  if (!h || !z || !xh0 || !fixed || !noise_x || !noise_h || !known_table || !op_index)
    return h ? h->fail(BDIFF_EINVAL, "null argument") : BDIFF_EINVAL;
  if (!h->have_plan) return h->fail(BDIFF_ESTATE, "no topology plan");
  launch_repaint_combine(static_cast<cudaStream_t>(stream), h->plan, h->d, z, xh0, fixed, noise_x, noise_h, known_table,
                         op_index);
  h->launches++;
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? BDIFF_OK : h->fail(BDIFF_ECUDA, "repaint_combine: %s", cudaGetErrorString(e));
}

int32_t bdiff_renoise(bdiff_handle* h, void* stream, float* z, const float* noise_x, const float* noise_h,
                      const float* jump_table, const int32_t* jump_index) {
  if (!h || !z || !noise_x || !noise_h || !jump_table || !jump_index)
    return h ? h->fail(BDIFF_EINVAL, "null argument") : BDIFF_EINVAL;
  if (!h->have_plan) return h->fail(BDIFF_ESTATE, "no topology plan");
  launch_step(static_cast<cudaStream_t>(stream), h->plan, h->d, 3, z, nullptr, noise_x, noise_h, jump_table, jump_index, z);
  h->launches++;
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? BDIFF_OK : h->fail(BDIFF_ECUDA, "renoise: %s", cudaGetErrorString(e));
}

int32_t bdiff_check(bdiff_handle* h, void* stream) {
  if (!h) return BDIFF_EINVAL;
  cudaError_t e = cudaStreamSynchronize(static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "check: %s", cudaGetErrorString(e));
  if (h->cfg.mode == BDIFF_MODE_TENSOR && h->sched_buf.p && h->have_plan) {
    int flag = 0;
    e = cudaMemcpy(&flag, h->sched.err, sizeof(int), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "check: %s", cudaGetErrorString(e));
    if (flag) { cudaMemset(h->sched.err, 0, sizeof(int)); return h->fail(BDIFF_ECUDA, "layer megakernel: a tile dependency wait timed out"); }
  }
  return BDIFF_OK;
}

int32_t bdiff_nan_guard_count(bdiff_handle* h, void* stream, int64_t* count_host, int32_t reset) {
  if (!h || !count_host) return h ? h->fail(BDIFF_EINVAL, "null argument") : BDIFF_EINVAL;
  *count_host = 0;
  if (!h->have_plan) return BDIFF_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int v = 0;
  cudaError_t e = cudaMemcpyAsync(&v, h->work.nan_flag + 1, sizeof(int), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && reset) e = cudaMemsetAsync(h->work.nan_flag + 1, 0, sizeof(int), st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "nan_guard_count: %s", cudaGetErrorString(e));
  *count_host = v;
  return BDIFF_OK;
}

int64_t bdiff_launch_count(const bdiff_handle* h) { return h ? h->launches : 0; }

// ------------------------------------------------------------------------------------------ native chain
int32_t bdiff_schedule_tables(const bdiff_sample_config* cfg, int32_t num_timesteps, float* coef_out, float* decode_out) {
  if (!cfg || !coef_out || !decode_out || num_timesteps < 1) return BDIFF_EINVAL;
  if (sample_config_error(*cfg)) return BDIFF_EINVAL;
  schedule_tables(schedule_gamma(cfg->model_timesteps, cfg->schedule_power, cfg->noise_precision), num_timesteps,
                  coef_out, decode_out);
  return BDIFF_OK;
}

int32_t bdiff_sample_setup(bdiff_handle* h, const bdiff_sample_config* cfg) {
  if (!h || !cfg) return h ? h->fail(BDIFF_EINVAL, "null argument") : BDIFF_EINVAL;
  if (const char* why = sample_config_error(*cfg)) return h->fail(BDIFF_EINVAL, "%s", why);
  if (cfg->num_atom_types + cfg->include_charges != h->d.F)
    return h->fail(BDIFF_EINVAL, "num_atom_types + include_charges = %d, but the handle's num_h is %d",
                   cfg->num_atom_types + cfg->include_charges, h->d.F);
  h->scfg = *cfg;
  h->have_sample_cfg = true;
  return BDIFF_OK;
}

int32_t bdiff_noise_fill(void* stream, uint64_t seed, uint64_t draw_index, int64_t rows, int64_t cols, float* out) {
  if (!out || rows < 0 || cols < 0) return BDIFF_EINVAL;
  launch_noise_fill(static_cast<cudaStream_t>(stream), seed, draw_index, rows * cols, out);
  return cudaGetLastError() == cudaSuccess ? BDIFF_OK : BDIFF_ECUDA;
}

int32_t bdiff_philox_fill(void* stream, uint64_t seed, uint64_t draw_index, int64_t blocks, uint32_t* out) {
  if (!out || blocks < 0) return BDIFF_EINVAL;
  launch_philox_fill(static_cast<cudaStream_t>(stream), seed, draw_index, blocks, out);
  return cudaGetLastError() == cudaSuccess ? BDIFF_OK : BDIFF_ECUDA;
}

int64_t bdiff_sample_graph_builds(const bdiff_handle* h) { return h ? h->smp_graph_builds : 0; }
int64_t bdiff_inpaint_graph_builds(const bdiff_handle* h) { return h ? h->inp_graph_builds : 0; }

// The stream a native chain runs on: the caller's, or, for the legacy default stream (which cannot be captured), the
// handle's own stream ordered after it.
static int32_t chain_stream(bdiff_handle* h, void* stream, cudaStream_t* run) {
  *run = static_cast<cudaStream_t>(stream);
  if (*run) return BDIFF_OK;
  cudaError_t e = cudaSuccess;
  if (!h->smp_stream) {
    e = cudaStreamCreateWithFlags(&h->smp_stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->smp_ev, cudaEventDisableTiming);
    if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "sample stream: %s", cudaGetErrorString(e));
  }
  *run = h->smp_stream;
  e = cudaEventRecord(h->smp_ev, cudaStreamLegacy);
  if (e == cudaSuccess) e = cudaStreamWaitEvent(*run, h->smp_ev, 0);
  return e == cudaSuccess ? BDIFF_OK : h->fail(BDIFF_ECUDA, "sample stream: %s", cudaGetErrorString(e));
}

// Writes the batch's batch_index and mask into the chain's buffers (on every call: a grown buffer is a zeroed allocation
// even when the plan is reused) and plans the topology when the batch changed or another plan replaced the chain's.
static int32_t chain_batch(bdiff_handle* h, cudaStream_t run, const std::vector<int32_t>& counts, int64_t* bi_dev,
                           uint8_t* mask_dev, std::vector<int32_t>* last_counts, int* last_epoch) {
  std::vector<int64_t> bi;
  for (size_t k = 0; k < counts.size(); ++k) bi.insert(bi.end(), (size_t)counts[k], (int64_t)k);
  const long long N = (long long)bi.size();
  cudaError_t e = cudaMemcpyAsync(bi_dev, bi.data(), N * 8, cudaMemcpyHostToDevice, run);
  if (e == cudaSuccess) e = cudaMemsetAsync(mask_dev, 1, N, run);
  if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "sample batch: %s", cudaGetErrorString(e));
  if (h->have_plan && counts == *last_counts && h->plan_epoch == *last_epoch) return BDIFF_OK;
  last_counts->clear();
  int32_t rc = bdiff_plan_topology(h, run, (int32_t)counts.size(), N, bi_dev, mask_dev, nullptr);
  if (rc != BDIFF_OK) return rc;
  *last_counts = counts;
  *last_epoch = h->plan_epoch;
  return BDIFF_OK;
}

// What every captured chain body bakes in besides its own buffers: the plan, the workspace, the weights and their
// tensor-core streams, next to the plan and weights epochs.  A buffer that moved for any reason changes the key, so it
// forces a new capture instead of a replay through a freed pointer.
static std::vector<long long> chain_key(const bdiff_handle* h, std::initializer_list<long long> own) {
  auto addr = [](const void* q) { return (long long)(uintptr_t)q; };
  std::vector<long long> key = {h->plan_epoch, h->weights_epoch, addr(h->eps_buf.p), addr(h->work_buf.p),
                                addr(h->plan_buf.p), addr(h->rc_buf.p), addr(h->sched_buf.p), addr(h->wbuf),
                                addr(h->tc_blob.p), addr(h->tc_node_blob.p), addr(h->layers_dev.p)};
  key.insert(key.end(), own);
  return key;
}

// Captures body() on `run` into *graph (replacing the old one); *launches receives the kernels one replay runs.
static int32_t chain_capture(bdiff_handle* h, cudaStream_t run, const std::function<int32_t()>& body,
                             cudaGraphExec_t* graph, int64_t* launches) {
  if (*graph) cudaGraphExecDestroy(*graph);
  *graph = nullptr;
  const int64_t before = h->launches;
  cudaGraph_t g = nullptr;
  cudaError_t e = cudaStreamBeginCapture(run, cudaStreamCaptureModeThreadLocal);
  if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "chain capture: %s", cudaGetErrorString(e));
  const int32_t rc = body();
  e = cudaStreamEndCapture(run, &g);
  *launches = h->launches - before;
  h->launches = before;
  if (rc != BDIFF_OK) { if (g) cudaGraphDestroy(g); return rc; }
  if (e == cudaSuccess) e = cudaGraphInstantiate(graph, g, 0);
  if (g) cudaGraphDestroy(g);
  if (e != cudaSuccess) { *graph = nullptr; return h->fail(BDIFF_ECUDA, "chain graph: %s", cudaGetErrorString(e)); }
  return BDIFF_OK;
}

// p(x, h | z_0) with draws decode_draw and decode_draw + 1, the discretising tail of mol_gen_sample into out[0 .. N), and
// for F > 1 frames 1 .. F-1 behind it; ends with bdiff_check.
static int32_t chain_tail(bdiff_handle* h, cudaStream_t run, float* z, const float* ctx, const float* dec,
                          unsigned long long seed, unsigned long long decode_draw, float* xhn, float* tot,
                          const float* frames, int F, const int64_t* bi_dev, float* out, int64_t* batch_index) {
  const Plan& p = h->plan;
  const size_t rows = (size_t)p.N * (3 + h->d.F);
  float* eps = static_cast<float*>(h->eps_buf.p);
  int32_t rc = forward_impl(h, run, z, nullptr, dec, nullptr, ctx, eps);
  if (rc != BDIFF_OK) return rc;
  launch_step_philox(run, p, h->d, 1, z, eps, dec, nullptr, nullptr, seed, decode_draw, nullptr, nullptr, xhn);
  launch_sample_finish(run, p, h->d, h->scfg.num_atom_types, h->scfg.norm_values, h->scfg.norm_biases, xhn, out, tot,
                       F == 1);
  h->launches += F == 1 ? 3 : 2;
  cudaError_t e = cudaSuccess;
  if (F > 1) e = cudaMemcpyAsync(out + rows, frames + rows, (F - 1) * rows * 4, cudaMemcpyDeviceToDevice, run);
  if (e == cudaSuccess && batch_index) e = cudaMemcpyAsync(batch_index, bi_dev, p.N * 8, cudaMemcpyDeviceToDevice, run);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "chain tail: %s", cudaGetErrorString(e));
  return bdiff_check(h, run);
}

int32_t bdiff_sample(bdiff_handle* h, void* stream, int32_t num_mols, const int32_t* num_nodes_host, const float* context,
                     int32_t num_timesteps, uint64_t seed, const float* z_init, const int64_t* z_init_shape,
                     const float* tables_host, float* xh, int64_t* batch_index) {
  return bdiff_sample_frames(h, stream, num_mols, num_nodes_host, context, num_timesteps, seed, z_init, z_init_shape, 1,
                             tables_host, xh, batch_index);
}

int32_t bdiff_sample_frames(bdiff_handle* h, void* stream, int32_t num_mols, const int32_t* num_nodes_host,
                            const float* context, int32_t num_timesteps, uint64_t seed, const float* z_init,
                            const int64_t* z_init_shape, int32_t return_frames, const float* tables_host, float* out,
                            int64_t* batch_index) {
  if (!h) return BDIFF_EINVAL;
  if (!h->have_sample_cfg) return h->fail(BDIFF_ESTATE, "bdiff_sample_setup has not been called");
  std::string why = sample_args_error(h->d.F, h->d.C, h->scfg, num_mols, num_nodes_host, context, num_timesteps,
                                      z_init, z_init_shape, out);
  if (why.empty()) why = frames_args_error(num_timesteps, return_frames);
  if (!why.empty()) return h->fail(BDIFF_EINVAL, "bdiff_sample: %s", why.c_str());
  if (bdiff_weights_missing(h) != 0) return h->fail(BDIFF_ESTATE, "%d parameters not set", bdiff_weights_missing(h));
  const int B = num_mols, T = num_timesteps, F = return_frames, C = h->d.C, ld = 3 + h->d.F;
  std::vector<int32_t> counts(num_nodes_host, num_nodes_host + B);
  long long N = 0;
  for (int32_t c : counts) N += c;
  cudaStream_t run;
  int32_t rc = chain_stream(h, stream, &run);
  if (rc != BDIFF_OK) return rc;

  // chain buffers: batch_index, mask, z, decoded xh, per-atom context, {step, done, seed, draw0}, CoG sums, decode row,
  // and last the coefficient table, so that no buffer the captured step reads moves with the chain length
  size_t at = 0;
  auto take = [&](size_t bytes) { const size_t o = at; at += (bytes + 255) / 256 * 256; return o; };
  const size_t o_bi = take(N * 8), o_mask = take(N), o_z = take(N * ld * 4), o_xhn = take(N * ld * 4),
               o_ctx = take(N * C * 4), o_ctr = take(24), o_tot = take((size_t)B * 12), o_dec = take(16),
               o_coef = take((size_t)T * 16);
  cudaError_t e = h->smp_buf.ensure(at);
  if (e == cudaSuccess && F > 1) e = h->smp_slot.ensure((size_t)T * 4);
  if (e == cudaSuccess && F > 1) e = h->smp_frames.ensure((size_t)(F + 1) * N * ld * 4);
  if (e != cudaSuccess) return h->fail(BDIFF_ENOMEM, "sample buffers: %s", cudaGetErrorString(e));
  unsigned char* base = static_cast<unsigned char*>(h->smp_buf.p);
  int64_t* bi_dev = reinterpret_cast<int64_t*>(base + o_bi);
  float* z = reinterpret_cast<float*>(base + o_z);
  float* xhn = reinterpret_cast<float*>(base + o_xhn);
  float* ctx = C ? reinterpret_cast<float*>(base + o_ctx) : nullptr;
  float* coef = reinterpret_cast<float*>(base + o_coef);
  float* dec = reinterpret_cast<float*>(base + o_dec);
  int* ctr = reinterpret_cast<int*>(base + o_ctr);                                   // {step, done}
  unsigned long long* seed_draw = reinterpret_cast<unsigned long long*>(base + o_ctr + 8);   // {seed, draw0}
  float* tot = reinterpret_cast<float*>(base + o_tot);
  int* slot = static_cast<int*>(h->smp_slot.p);
  float* frames = static_cast<float*>(h->smp_frames.p);

  rc = chain_batch(h, run, counts, bi_dev, base + o_mask, &h->smp_counts, &h->smp_plan_epoch);
  if (rc != BDIFF_OK) return rc;

  std::vector<float> tables((size_t)T * 4 + 4);
  if (tables_host) {
    std::copy(tables_host, tables_host + tables.size(), tables.begin());
  } else {
    schedule_tables(schedule_gamma(h->scfg.model_timesteps, h->scfg.schedule_power, h->scfg.noise_precision), T,
                    tables.data(), tables.data() + (size_t)T * 4);
  }
  e = cudaMemcpyAsync(coef, tables.data(), (size_t)T * 16, cudaMemcpyHostToDevice, run);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dec, tables.data() + (size_t)T * 4, 16, cudaMemcpyHostToDevice, run);
  // z_T = draws 0, 1 (masked, x centred), or the caller's start; the reverse steps' draws follow
  const unsigned long long draw0 = z_init ? 0 : 2, sd[2] = {seed, draw0};
  if (e == cudaSuccess) e = cudaMemsetAsync(ctr, 0, 8, run);
  if (e == cudaSuccess) e = cudaMemcpyAsync(seed_draw, sd, 16, cudaMemcpyHostToDevice, run);
  std::vector<int32_t> slots;
  if (F > 1) {            // reverse step r lands on s = T-1-r; the steps between frames write the dummy slot F
    for (int r = 0; r < T; ++r) {
      const int v = frame_slot(T - 1 - r, T, F);
      slots.push_back(v < 0 ? F : v);
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(slot, slots.data(), (size_t)T * 4, cudaMemcpyHostToDevice, run);
    if (e == cudaSuccess) e = cudaMemsetAsync(frames, 0, (size_t)(F + 1) * N * ld * 4, run);
  }
  if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "sample tables: %s", cudaGetErrorString(e));
  tc_prepare(h, run);
  const Plan& p = h->plan;
  if (C) {
    launch_gather_context(run, p, C, context, ctx);
    h->launches++;
  }
  if (z_init) {
    e = cudaMemcpyAsync(z, z_init, N * ld * 4, cudaMemcpyDeviceToDevice, run);
    if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "z_init copy: %s", cudaGetErrorString(e));
  } else {
    launch_step_philox(run, p, h->d, 2, nullptr, nullptr, nullptr, nullptr, nullptr, seed, 0, nullptr, nullptr, z);
    h->launches++;
  }

  // one reverse step (and, with frames, the frame write), captured once and replayed T times; it reads the step, the seed
  // and the first draw index from the device, and the coefficient table at a fixed address
  float* eps = static_cast<float*>(h->eps_buf.p);
  auto addr = [](const void* q) { return (long long)(uintptr_t)q; };
  const std::vector<long long> key = chain_key(h, {N, B, F > 1, addr(h->smp_buf.p), addr(slot), addr(frames)});
  if (!h->smp_graph || key != h->smp_graph_key) {
    h->smp_graph_key.clear();
    rc = chain_capture(h, run, [&]() {
      const int32_t r = forward_impl(h, run, z, nullptr, coef, ctr, ctx, eps);
      if (r != BDIFF_OK) return r;
      launch_step_philox(run, p, h->d, 0, z, eps, coef, ctr, F > 1 ? nullptr : ctr + 1, 0, 0, seed_draw, nullptr, z);
      h->launches++;
      if (F > 1) {
        launch_write_frame(run, p, h->d, h->scfg.num_atom_types, h->scfg.norm_values, h->scfg.norm_biases, z, slot, ctr,
                           ctr + 1, frames);
        h->launches++;
      }
      return BDIFF_OK;
    }, &h->smp_graph, &h->smp_step_launches);
    if (rc != BDIFF_OK) return rc;
    h->smp_graph_key = key;
    h->smp_graph_builds++;
  }
  for (int r = 0; r < T && e == cudaSuccess; ++r) {
    e = cudaGraphLaunch(h->smp_graph, run);
    h->launches += h->smp_step_launches;
  }
  if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "sample replay: %s", cudaGetErrorString(e));
  return chain_tail(h, run, z, ctx, dec, seed, draw0 + 2ull * T, xhn, tot, frames, F, bi_dev, out, batch_index);
}

int32_t bdiff_repaint_tables(const bdiff_sample_config* cfg, int32_t num_timesteps, int32_t num_resamplings,
                             int32_t jump_length, int32_t return_frames, int32_t* num_ops, int32_t* num_jumps,
                             float* rev_out, float* known_out, float* jump_out, float* decode_out, int32_t* op_s_out,
                             int32_t* slot_out, uint8_t* jump_after_out, uint64_t* op_draw_out, uint64_t* jump_draw_out,
                             uint64_t* decode_draw_out) {
  if (!cfg || !num_ops || !num_jumps || sample_config_error(*cfg)) return BDIFF_EINVAL;
  if (!repaint_args_error(num_timesteps, num_resamplings, jump_length, return_frames).empty()) return BDIFF_EINVAL;
  const RepaintProgram g = repaint_program(schedule_gamma(cfg->model_timesteps, cfg->schedule_power, cfg->noise_precision),
                                           num_resamplings, jump_length, num_timesteps, return_frames);
  *num_ops = (int32_t)g.op_s.size();
  *num_jumps = (int32_t)g.jump_draw.size();
  if (rev_out) std::copy(g.rev.begin(), g.rev.end(), rev_out);
  if (known_out) std::copy(g.known.begin(), g.known.end(), known_out);
  if (jump_out) std::copy(g.jump.begin(), g.jump.end(), jump_out);
  if (decode_out) std::copy(g.dec, g.dec + 4, decode_out);
  if (op_s_out) std::copy(g.op_s.begin(), g.op_s.end(), op_s_out);
  if (slot_out) std::copy(g.slot.begin(), g.slot.end(), slot_out);
  if (jump_after_out) std::copy(g.jump_after.begin(), g.jump_after.end(), jump_after_out);
  if (op_draw_out) std::copy(g.op_draw.begin(), g.op_draw.end(), op_draw_out);
  if (jump_draw_out) std::copy(g.jump_draw.begin(), g.jump_draw.end(), jump_draw_out);
  if (decode_draw_out) *decode_draw_out = g.decode_draw;
  return BDIFF_OK;
}

int32_t bdiff_inpaint(bdiff_handle* h, void* stream, int32_t num_mols, const int32_t* num_nodes_host, const float* context,
                      int32_t num_timesteps, int32_t num_resamplings, int32_t jump_length, uint64_t seed,
                      const float* xh0_host, const uint8_t* fixed_host, int32_t return_frames, const float* tables_host,
                      float* out, int64_t* batch_index) {
  if (!h) return BDIFF_EINVAL;
  if (!h->have_sample_cfg) return h->fail(BDIFF_ESTATE, "bdiff_sample_setup has not been called");
  const std::string why = inpaint_args_error(h->d.F, h->d.C, h->scfg, num_mols, num_nodes_host, context, num_timesteps,
                                             num_resamplings, jump_length, return_frames, xh0_host, fixed_host, out);
  if (!why.empty()) return h->fail(BDIFF_EINVAL, "bdiff_inpaint: %s", why.c_str());
  if (bdiff_weights_missing(h) != 0) return h->fail(BDIFF_ESTATE, "%d parameters not set", bdiff_weights_missing(h));
  const int B = num_mols, T = num_timesteps, F = return_frames, C = h->d.C, ld = 3 + h->d.F;
  std::vector<int32_t> counts(num_nodes_host, num_nodes_host + B);
  long long N = 0;
  for (int32_t c : counts) N += c;
  RepaintProgram g = repaint_program(schedule_gamma(h->scfg.model_timesteps, h->scfg.schedule_power,
                                                    h->scfg.noise_precision),
                                     num_resamplings, jump_length, T, F);
  const size_t ops = g.op_s.size(), jumps = g.jump_draw.size();
  if (tables_host) {      // the caller's rows, in bdiff_repaint_tables' order
    const float* q = tables_host;
    g.rev.assign(q, q + ops * 4);
    q += ops * 4;
    g.known.assign(q, q + ops * 2);
    q += ops * 2;
    g.jump.assign(q, q + jumps * 4);
    q += jumps * 4;
    std::copy(q, q + 4, g.dec);
  }
  std::vector<float> xh0(xh0_host, xh0_host + N * ld);
  center_on_fixed(B, num_nodes_host, ld, fixed_host, xh0.data());
  cudaStream_t run;
  int32_t rc = chain_stream(h, stream, &run);
  if (rc != BDIFF_OK) return rc;

  // per-atom buffers (their layout depends on the batch only) and the frames last; the program's tables each in a buffer
  // of its own, so that a shorter program reuses every address the captured bodies read
  size_t at = 0;
  auto take = [&](size_t bytes) { const size_t o = at; at += (bytes + 255) / 256 * 256; return o; };
  const size_t o_bi = take(N * 8), o_mask = take(N), o_z = take(N * ld * 4), o_xhn = take(N * ld * 4),
               o_ctx = take(N * C * 4), o_xh0 = take(N * ld * 4), o_fixed = take(N), o_ctr = take(48),
               o_tot = take((size_t)B * 12), o_dec = take(16), o_frames = take(F > 1 ? (size_t)(F + 1) * N * ld * 4 : 0);
  cudaError_t e = h->inp_buf.ensure(at);
  if (e == cudaSuccess) e = h->inp_rev.ensure(ops * 16);
  if (e == cudaSuccess) e = h->inp_known.ensure(ops * 8);
  if (e == cudaSuccess) e = h->inp_slot.ensure(ops * 4);
  if (e == cudaSuccess) e = h->inp_draw.ensure(ops * 8);
  if (e == cudaSuccess) e = h->inp_jump.ensure(std::max<size_t>(jumps, 1) * 16);
  if (e == cudaSuccess) e = h->inp_jdraw.ensure(std::max<size_t>(jumps, 1) * 8);
  if (e != cudaSuccess) return h->fail(BDIFF_ENOMEM, "inpaint buffers: %s", cudaGetErrorString(e));
  unsigned char* base = static_cast<unsigned char*>(h->inp_buf.p);
  int64_t* bi_dev = reinterpret_cast<int64_t*>(base + o_bi);
  float* z = reinterpret_cast<float*>(base + o_z);
  float* xhn = reinterpret_cast<float*>(base + o_xhn);
  float* ctx = C ? reinterpret_cast<float*>(base + o_ctx) : nullptr;
  float* xh0_dev = reinterpret_cast<float*>(base + o_xh0);
  uint8_t* fixed = base + o_fixed;
  int* ctr = reinterpret_cast<int*>(base + o_ctr);                                   // {op, op done, jump, jump done}
  // {seed, 0}: the known part's and the jump's draws are the table's; {seed, 2}: the unknown part's follow the known's
  unsigned long long* seed_draw = reinterpret_cast<unsigned long long*>(base + o_ctr + 16);
  float* tot = reinterpret_cast<float*>(base + o_tot);
  float* dec = reinterpret_cast<float*>(base + o_dec);
  float* frames = F > 1 ? reinterpret_cast<float*>(base + o_frames) : nullptr;
  float* rev = static_cast<float*>(h->inp_rev.p);
  float* known = static_cast<float*>(h->inp_known.p);
  int* slot = static_cast<int*>(h->inp_slot.p);
  unsigned long long* draw = static_cast<unsigned long long*>(h->inp_draw.p);
  float* jump = static_cast<float*>(h->inp_jump.p);
  unsigned long long* jdraw = static_cast<unsigned long long*>(h->inp_jdraw.p);

  rc = chain_batch(h, run, counts, bi_dev, base + o_mask, &h->inp_counts, &h->inp_plan_epoch);
  if (rc != BDIFF_OK) return rc;
  const unsigned long long sd[4] = {seed, 0, seed, 2};
  e = cudaMemcpyAsync(rev, g.rev.data(), ops * 16, cudaMemcpyHostToDevice, run);
  if (e == cudaSuccess) e = cudaMemcpyAsync(known, g.known.data(), ops * 8, cudaMemcpyHostToDevice, run);
  if (e == cudaSuccess) e = cudaMemcpyAsync(slot, g.slot.data(), ops * 4, cudaMemcpyHostToDevice, run);
  if (e == cudaSuccess) e = cudaMemcpyAsync(draw, g.op_draw.data(), ops * 8, cudaMemcpyHostToDevice, run);
  if (e == cudaSuccess && jumps) e = cudaMemcpyAsync(jump, g.jump.data(), jumps * 16, cudaMemcpyHostToDevice, run);
  if (e == cudaSuccess && jumps) e = cudaMemcpyAsync(jdraw, g.jump_draw.data(), jumps * 8, cudaMemcpyHostToDevice, run);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dec, g.dec, 16, cudaMemcpyHostToDevice, run);
  if (e == cudaSuccess) e = cudaMemcpyAsync(xh0_dev, xh0.data(), N * ld * 4, cudaMemcpyHostToDevice, run);
  if (e == cudaSuccess) e = cudaMemcpyAsync(fixed, fixed_host, N, cudaMemcpyHostToDevice, run);
  if (e == cudaSuccess) e = cudaMemsetAsync(ctr, 0, 16, run);
  if (e == cudaSuccess) e = cudaMemcpyAsync(seed_draw, sd, 32, cudaMemcpyHostToDevice, run);
  if (e == cudaSuccess && frames) e = cudaMemsetAsync(frames, 0, (size_t)(F + 1) * N * ld * 4, run);
  if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "inpaint tables: %s", cudaGetErrorString(e));
  tc_prepare(h, run);
  const Plan& p = h->plan;
  if (C) {
    launch_gather_context(run, p, C, context, ctx);
    h->launches++;
  }
  launch_step_philox(run, p, h->d, 2, nullptr, nullptr, nullptr, nullptr, nullptr, seed, 0, nullptr, nullptr, z);
  h->launches++;

  // the op body: reverse step to s, combination with the known part, frame write; it advances the op counter.  The jump
  // body: the jump back at the jump counter, which it advances.
  float* eps = static_cast<float*>(h->eps_buf.p);
  auto addr = [](const void* q) { return (long long)(uintptr_t)q; };
  const std::vector<long long> key = chain_key(h, {N, B, F > 1, addr(h->inp_buf.p), addr(rev), addr(known), addr(slot),
                                                  addr(draw), addr(jump), addr(jdraw)});
  if (!h->inp_op_graph || !h->inp_jump_graph || key != h->inp_graph_key) {
    h->inp_graph_key.clear();
    rc = chain_capture(h, run, [&]() {
      const int32_t r = forward_impl(h, run, z, nullptr, rev, ctr, ctx, eps);
      if (r != BDIFF_OK) return r;
      launch_step_philox(run, p, h->d, 0, z, eps, rev, ctr, nullptr, 0, 0, seed_draw + 2, draw, z);
      launch_repaint_combine_philox(run, p, h->d, z, xh0_dev, fixed, known, ctr, frames ? nullptr : ctr + 1, seed_draw,
                                    draw);
      h->launches += 2;
      if (frames) {
        launch_write_frame(run, p, h->d, h->scfg.num_atom_types, h->scfg.norm_values, h->scfg.norm_biases, z, slot, ctr,
                           ctr + 1, frames);
        h->launches++;
      }
      return BDIFF_OK;
    }, &h->inp_op_graph, &h->inp_op_launches);
    if (rc == BDIFF_OK)
      rc = chain_capture(h, run, [&]() {
        launch_step_philox(run, p, h->d, 3, z, nullptr, jump, ctr + 2, ctr + 3, 0, 0, seed_draw, jdraw, z);
        h->launches++;
        return BDIFF_OK;
      }, &h->inp_jump_graph, &h->inp_jump_launches);
    if (rc != BDIFF_OK) return rc;
    h->inp_graph_key = key;
    h->inp_graph_builds++;
  }
  for (size_t i = 0; i < ops && e == cudaSuccess; ++i) {
    e = cudaGraphLaunch(h->inp_op_graph, run);
    h->launches += h->inp_op_launches;
    if (e == cudaSuccess && g.jump_after[i]) {
      e = cudaGraphLaunch(h->inp_jump_graph, run);
      h->launches += h->inp_jump_launches;
    }
  }
  if (e != cudaSuccess) return h->fail(BDIFF_ECUDA, "inpaint replay: %s", cudaGetErrorString(e));
  return chain_tail(h, run, z, ctx, dec, seed, g.decode_draw, xhn, tot, frames, F, bi_dev, out, batch_index);
}

}  // extern "C"
