// plan_hostcheck.cpp — TEST INFRASTRUCTURE ONLY (never linked into libbdiff_sm90.so, never on the product path).
//
// Exposes the host planner of bdiff_plan_topology (bio-diffusion_b200/csrc/bdiff_plan.h) through a C ABI so that
// tests/test_plan_cpu.py can check the staging block it builds — the plan arrays, the dependency tables and the layer
// megakernel's work list — on the CPU-only build container.
#include <cstring>

#include "../../bio-diffusion_b200/csrc/bdiff_plan.h"

namespace {
bdiff::HostPlan g_plan;
}

extern "C" {

// Runs the planner.  On success returns 0 and fills info[18] = {B, N, E, Mact, TE, TN, nitems, bytes, then the byte
// offsets of mol_off, act_off, act_idx, node_mol, edge_off, mask, edge_dep, node_dep, node_mid, items}; the block is then
// read with plan_hostcheck_block.  On a rejection returns 1 and copies the message into err.
int plan_hostcheck(int num_mols, long long num_nodes, const long long* batch_index, const unsigned char* mask, int L,
                   int num_sms, long long* info, char* err, int err_len) {
  const std::string why = bdiff::plan_host(num_mols, num_nodes, reinterpret_cast<const int64_t*>(batch_index), mask, L,
                                           num_sms, g_plan);
  if (!why.empty()) {
    snprintf(err, err_len, "%s", why.c_str());
    return 1;
  }
  const bdiff::HostPlan& p = g_plan;
  const bdiff::PlanLayout& a = p.at;
  const long long v[18] = {p.B, p.N, p.E, p.Mact, p.TE, p.TN, p.nitems, (long long)a.bytes,
                           (long long)a.mol_off, (long long)a.act_off, (long long)a.act_idx, (long long)a.node_mol,
                           (long long)a.edge_off, (long long)a.mask, (long long)a.edge_dep, (long long)a.node_dep,
                           (long long)a.node_mid, (long long)a.items};
  memcpy(info, v, sizeof v);
  return 0;
}

void plan_hostcheck_block(unsigned char* dst) { memcpy(dst, g_plan.block.data(), g_plan.block.size()); }

}  // extern "C"
