// bdiff_plan.h — the host half of bdiff_plan_topology: it validates a batch and builds the topology plan, the layer
// megakernel's dependency tables and work list, all packed into the one staging block that is copied to the device.
// Plain C++17 without CUDA headers, so that the CPU suite compiles it with g++ (oracle/hostcheck/plan_hostcheck.cpp).
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

namespace bdiff {

// Byte offsets of the arrays in the staging block (256-byte aligned), and the block's size.
struct PlanLayout {
  size_t mol_off, act_off, act_idx, node_mol, edge_off, mask, edge_dep, node_dep, node_mid, items, bytes;
};

struct HostPlan {
  int B = 0, N = 0, Mact = 0;     // molecules, nodes, unmasked nodes
  long long E = 0;                // edges = sum nact^2
  int TE = 0, TN = 0;             // 128-edge tiles, 32-node tiles
  int nitems = 0;                 // work items: L * (TE + TN)
  PlanLayout at{};
  std::vector<unsigned char> block;
};

// A work item of the layer megakernel: type (0 edge tile, 1 node tile) << 30 | layer << 24 | tile.
inline int work_item(int type, int layer, int tile) { return type << 30 | layer << 24 | tile; }

// The checks that need no host copy of batch_index (so they also run before it is copied).
inline const char* plan_args_error(int num_mols, int64_t num_nodes) {
  if (num_mols < 1 || num_nodes < 1) return "bad plan arguments";
  if (num_nodes > (1ll << 30)) return "too many nodes";
  return nullptr;
}

// Builds `out` from host copies of batch_index and mask for L layers on num_sms SMs.  Returns "" on success, else why the
// batch is rejected (then `out` is unspecified).
inline std::string plan_host(int num_mols, int64_t num_nodes, const int64_t* batch_index, const uint8_t* mask, int L,
                             int num_sms, HostPlan& out) {
  if (const char* m = plan_args_error(num_mols, num_nodes)) return m;
  char msg[128];
  const int N = (int)num_nodes, B = num_mols;
  std::vector<int> mol_off(B + 1, 0), act_off(B + 1, 0), act_idx, node_mol(N);
  std::vector<long long> edge_off(B + 1, 0);
  act_idx.reserve(N);
  int64_t prev = 0;
  for (int i = 0; i < N; ++i) {
    const int64_t m = batch_index[i];
    if (m < 0 || m >= B) {
      snprintf(msg, sizeof msg, "batch_index[%d]=%lld outside [0,%d)", i, (long long)m, B);
      return msg;
    }
    if (m < prev) {
      snprintf(msg, sizeof msg, "batch_index must be sorted (node %d)", i);
      return msg;
    }
    prev = m;
    mol_off[m + 1]++;
    node_mol[i] = (int)m;
  }
  for (int k = 0; k < B; ++k) mol_off[k + 1] += mol_off[k];
  for (int k = 0; k < B; ++k) {
    for (int i = mol_off[k]; i < mol_off[k + 1]; ++i)
      if (mask[i]) act_idx.push_back(i);
    act_off[k + 1] = (int)act_idx.size();
    const long long na = act_off[k + 1] - act_off[k];
    edge_off[k + 1] = edge_off[k] + na * na;
  }
  const long long E = edge_off[B];
  if (E >= (1ll << 36)) return "too many edges";
  // an item holds the layer in bits 24..29 (up to the 64 layers bdiff_create accepts) and the tile in bits 0..23; the
  // queue head counts past the last item by up to one claim per CTA
  const long long TE = (E + 127) / 128, TN = (N + 31) / 32;
  if (L > 64 || TE >= (1 << 24) || TN >= (1 << 24) || L * (TE + TN) >= (1ll << 30))
    return "problem too large for the tile scheduler";

  // dependency tables: edge tile -> inclusive range of the 32-node tiles of its molecules, node tile -> inclusive range of
  // the edge tiles of its molecules ({0, -1}: none)
  std::vector<int> edge_dep(2 * TE), node_dep(2 * TN);
  for (long long t = 0, k0 = 0; t < TE; ++t) {
    const long long g0 = t * 128, g1 = std::min(E, g0 + 128) - 1;
    while (edge_off[k0 + 1] <= g0) ++k0;       // the molecule of edge g0 (g0 < E = edge_off[B] ends the scan)
    long long k1 = k0;
    while (edge_off[k1 + 1] <= g1) ++k1;
    edge_dep[2 * t] = mol_off[k0] / 32;
    edge_dep[2 * t + 1] = (mol_off[k1 + 1] - 1) / 32;
  }
  for (int u = 0; u < TN; ++u) {
    const int n1 = std::min(N, u * 32 + 32) - 1;
    const int k0 = node_mol[u * 32], k1 = node_mol[n1];
    const long long e0 = edge_off[k0], e1 = edge_off[k1 + 1] - 1;
    node_dep[2 * u] = e1 >= e0 ? (int)(e0 / 128) : 0;
    node_dep[2 * u + 1] = e1 >= e0 ? (int)(e1 / 128) : -1;
  }
  // per node of the node tiles: {first, count} of the edge tiles strictly inside its row (their sums go through Work::mid,
  // see edge_tile_epilogue.inc)
  std::vector<int> node_mid(2 * 32 * TN, 0);
  for (int k = 0; k < B; ++k) {
    const long long na = act_off[k + 1] - act_off[k];
    for (long long a = 0; a < na; ++a) {
      const long long g0 = edge_off[k] + a * na, g1 = g0 + na - 1;
      const long long t0 = g0 / 128, t1 = g1 / 128;
      if (t1 - t0 >= 2) {
        const int i = act_idx[act_off[k] + a];
        node_mid[2 * (size_t)i] = (int)(t0 + 1);
        node_mid[2 * (size_t)i + 1] = (int)(t1 - t0 - 1);
      }
    }
  }

  // Claim order (DESIGN §4 "Scheduling"): edge tile (l, t) at time l*TE + t; node tile (l, u) at l*TE + th(u) + lag, where
  // th(u) = node_dep[u].y is the last edge tile it reads (at l*TE if it reads none); ties go to the edge tile.  The
  // megakernel cannot deadlock when every dependency precedes its consumer: node (l, u) follows its edge tiles since
  // lag >= 0, and edge tile (l+1, t), which reads node tiles up to u = edge_dep[t].y, follows them when
  // lag <= TE - 1 + t - th(u).  Within that bound lag is one wave of claims (num_sms): by then the node tile's inputs
  // have normally finished, so the CTA that claims it waits little.  tests/test_plan_cpu.py checks the order.
  long long lag = num_sms;
  for (long long t = 0; t < TE; ++t) {
    const int th = node_dep[2 * edge_dep[2 * t + 1] + 1];
    if (th >= 0) lag = std::min(lag, TE - 1 + t - th);
  }
  std::vector<std::pair<long long, int>> order;        // (2 * time + type, item)
  order.reserve(L * (TE + TN));
  for (int l = 0; l < L; ++l) {
    for (int t = 0; t < TE; ++t) order.emplace_back(2 * (l * TE + t), work_item(0, l, t));
    for (int u = 0; u < TN; ++u) {
      const int th = node_dep[2 * u + 1];
      order.emplace_back(2 * (l * TE + (th >= 0 ? th + lag : 0)) + 1, work_item(1, l, u));
    }
  }
  std::stable_sort(order.begin(), order.end(),
                   [](const std::pair<long long, int>& a, const std::pair<long long, int>& b) { return a.first < b.first; });

  PlanLayout& at = out.at;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) / 256 * 256; return o; };
  at.mol_off = take((B + 1) * 4);
  at.act_off = take((B + 1) * 4);
  at.act_idx = take(act_idx.size() * 4);
  at.node_mol = take((size_t)N * 4);
  at.edge_off = take((B + 1) * 8);
  at.mask = take(N);
  at.edge_dep = take(edge_dep.size() * 4);
  at.node_dep = take(node_dep.size() * 4);
  at.node_mid = take(node_mid.size() * 4);
  at.items = take(order.size() * 4);
  at.bytes = off;
  out.block.assign(off, 0);
  unsigned char* b = out.block.data();
  auto put = [&](size_t o, const void* src, size_t bytes) { if (bytes) memcpy(b + o, src, bytes); };
  put(at.mol_off, mol_off.data(), (B + 1) * 4);
  put(at.act_off, act_off.data(), (B + 1) * 4);
  put(at.act_idx, act_idx.data(), act_idx.size() * 4);
  put(at.node_mol, node_mol.data(), (size_t)N * 4);
  put(at.edge_off, edge_off.data(), (B + 1) * 8);
  put(at.mask, mask, N);
  put(at.edge_dep, edge_dep.data(), edge_dep.size() * 4);
  put(at.node_dep, node_dep.data(), node_dep.size() * 4);
  put(at.node_mid, node_mid.data(), node_mid.size() * 4);
  int* items = reinterpret_cast<int*>(b + at.items);
  for (size_t i = 0; i < order.size(); ++i) items[i] = order[i].second;

  out.B = B; out.N = N; out.E = E; out.Mact = (int)act_idx.size();
  out.TE = (int)TE; out.TN = (int)TN; out.nitems = (int)order.size();
  return "";
}

}  // namespace bdiff
