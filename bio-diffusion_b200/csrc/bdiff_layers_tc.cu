// bdiff_layers_tc.cu — all L interaction layers of one denoiser forward in ONE persistent tensor-core kernel (sm_90a).
//
// Why: with one kernel per pass the forward is quantised twice per layer (the edge tiles of a batch fill the SMs in a
// few rounds with an idle tail, and the node pass has work for fewer SMs) and pays ~18 launch / prologue /
// pipeline-ramp gaps.  Nothing in the network couples molecules inside a
// layer (gcpnet.py:676-737, 893-930: messages, aggregation and node updates are per molecule), so layer l+1 of
// a molecule only needs layer l of the same molecule.  This kernel therefore runs the edge-tile and node-tile bodies
// (edge_tile_*.inc, node_r4_tile_*.inc) from a global work list of tiles (built by plan_host, bdiff_plan.h)
//     for l in 0..L-1:  edge tiles (l, 0..TE-1) in order, node tile (l, u) inserted ~one wave of claims after the last
//                       edge tile it depends on (so its wait is short and the CTA that claims it does not idle)
// claimed with one atomicAdd per tile, with per-tile completion flags as dependencies:
//     edge (l, t)  waits for node (l-1, u) of every 32-node tile u that intersects the molecules of edge tile t;
//     node (l, u)  waits for edge (l, t) of every edge tile t that intersects the molecules of node tile u.
// Every dependency has a smaller queue index and a CTA only claims a tile once it is running, so the smallest unfinished
// tile can always run: no deadlock.  A dependency wait beyond 2^32 cycles can only mean a broken schedule: it traps (sticky
// launch failure + error word read by bdiff_check) instead of computing on stale data.
// Flags are released with fence + st.release after a CTA barrier and acquired with ld.acquire + a gpu-scope fence
// in every consumer thread (mutable activations are re-read from L2, not from a stale L1 line).
//
// The TMA-producer lane also claims the tiles (so the next tile's weights stream while the current tile computes) and hands
// them to the flag lane and the 8 compute warps through a two-slot mbarrier ring.
#include "bdiff_node_tc.cuh"

namespace bdiff {

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Shared memory: [A region: 9 x 16 KiB (edge tile: hi blocks 0-3, lo blocks 4-7, extra block 8; node tile: 5 R5 blocks
// of 20 KiB + NodeScratch)] [weight ring: TC_NSLOT x 10 KiB] [tail: barriers + per-tile small weights / buffers].
union LayersTail {
  TcBars bars;
  EdgeTail edge;
  NodeTail node;
};
constexpr size_t LAYERS_SMEM_BYTES = XE_BLOCKS * (size_t)X_BLOCK + TC_NSLOT * (size_t)TC_SLOT + sizeof(LayersTail) + 1024;
static_assert(LAYERS_SMEM_BYTES + 64 <= 232448, "shared memory budget of the layer megakernel (227 KiB per block)");

// 12 warps: 0-7 compute (two warpgroups: epilogue and wgmma issue), 8 scheduler + TMA producer, 9 completion-flag lane,
// 10-11 padding so that the service warps form a complete third warpgroup for setmaxnreg.  The CTA is launched with
// 168 registers/thread (384 threads -> a pool of 64512); the service warpgroup shrinks to 40 and the two compute
// warpgroups grow to 232 (256*232 + 128*40 = 64512 — a request the pool cannot satisfy would block forever).
constexpr int LAYERS_THREADS = 384;
constexpr int LAYERS_REG_COMPUTE = 232, LAYERS_REG_SERVICE = 40;
static_assert(256 * LAYERS_REG_COMPUTE + 128 * LAYERS_REG_SERVICE <= 168 * LAYERS_THREADS, "setmaxnreg pool");
constexpr int RING_CONSUMERS = TC_EPI / 32;       // one arrival per compute warp frees a ring slot

template <int ED, int XD>
__global__ void __launch_bounds__(LAYERS_THREADS, 1) k_layers_tc(Plan p, Dims d, EmbedW ew, LayerSched q, Work w) {
  constexpr int HID0 = (64 + XD) / 4;
  constexpr int H2 = HID0 / 2;
  constexpr int K0RAW = ED + HID0 + 9;
  constexpr int K0S = (K0RAW + 15) / 16;
  static_assert(HID0 % 2 == 0 && H2 * 3 <= 32 && HID0 + 9 <= 32 && ED % 16 == 0, "layout");

  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  unsigned char* X = smem;
  unsigned char* ring = smem + XE_BLOCKS * X_BLOCK;
  unsigned char* tail = ring + TC_NSLOT * TC_SLOT;
  TcBars& B = *reinterpret_cast<TcBars*>(tail);
  // warp role and claimed item are broadcast with __shfl_sync so that ptxas can prove them warp-uniform: a wgmma on a
  // path it cannot prove convergent serializes all of them (each waits for its own completion, ptxas C7520; see gemm)
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  const int hid0 = d.hid0;
  const int per_layer = q.TE + q.TN;
  int* const flags = q.sched + 1;

  if (tid == 0) {
    for (int i = 0; i < TC_NSLOT; ++i) { mbar_init(&B.full[i], 1); mbar_init(&B.empty[i], RING_CONSUMERS); }
    for (int i = 0; i < 2; ++i) { mbar_init(&B.item_full[i], 1); mbar_init(&B.item_empty[i], TC_EPI + 1); }
    mbar_init(&B.tile_done, TC_EPI);
    mbar_init(&B.wbar, 1);
    mbar_fence_init();
    acc_scratch = w.acc + (size_t)blockIdx.x * TM_COLS * 128;
  }
  __syncthreads();

  if (warp == 8) {
    // ============================================================ scheduler + TMA producer (one lane)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(LAYERS_REG_SERVICE));
    if (lane == 0) {
      uint32_t ci = 0;
      for (uint32_t k = 0;; ++k) {
        const uint32_t slot = k & 1;
        mbar_wait_backoff(&B.item_empty[slot], ((k >> 1) & 1) ^ 1);
        int type = -1, layer = 0, tile = 0;
        const int qi = atomicAdd(q.sched, 1);
        if (qi < q.nitems) {
          const int it = __ldg(q.items + qi);
          type = (it >> 30) & 1; layer = (it >> 24) & 63; tile = it & 0xffffff;
        }
        B.item[slot][0] = type; B.item[slot][1] = layer; B.item[slot][2] = tile;
        mbar_arrive(&B.item_full[slot]);
        if (type < 0) break;
        // the layer's weight stream (tc_edge_stream / tc_node_stream): per segment, the chunks of N half 0, then of half 1
        const size_t stride = type == 0 ? q.edge_blob_stride : q.node_blob_stride;
        const unsigned char* blob = (type == 0 ? q.edge_blob : q.node_blob) + (size_t)layer * stride;
        const Stream S = type == 0 ? tc_edge_stream(K0S) : tc_node_stream(layer == q.L - 1);
        size_t off = 0;
        for (int i = 0; i < S.n; ++i) {
          const StreamSeg g = S.seg[i];
          const uint32_t step = seg_step_bytes(g);
          for (int h = 0; h < 2; ++h)
            for (int c = 0; c < seg_chunks(g); ++c) {
              const int steps = min(g.group, g.steps - c * g.group);
              const uint32_t s = ci % TC_NSLOT;
              mbar_wait_backoff(&B.empty[s], ((ci / TC_NSLOT) & 1) ^ 1);
              mbar_expect_tx(&B.full[s], steps * step);
              bulk_g2s(ring + s * TC_SLOT, blob + h * (stride / 2) + off + (size_t)c * g.group * step, steps * step, &B.full[s]);
              ++ci;
            }
          off += (size_t)g.steps * step;
        }
      }
    }
  } else if (warp == 9) {
    // ============================================================ completion-flag lane
    // every compute thread arrives (release) on tile_done after its last global write; this lane acquires it, makes the
    // writes visible gpu-wide and raises the flag, so the ~1 us fence is off the compute warps' critical path
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(LAYERS_REG_SERVICE));
    if (lane == 0) {
      for (uint32_t k = 0;; ++k) {
        const uint32_t slot = k & 1;
        mbar_wait(&B.item_full[slot], (k >> 1) & 1);
        const int type = B.item[slot][0], layer = B.item[slot][1], tile = B.item[slot][2];
        if (type < 0) break;
        mbar_wait_backoff(&B.tile_done, k & 1);
        __threadfence();
        st_release_gpu(flags + (size_t)layer * per_layer + (type == 0 ? tile : q.TE + tile), 1);
        mbar_arrive(&B.item_empty[slot]);
      }
    }
  } else if (warp >= 10) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(LAYERS_REG_SERVICE));     // padding warps of the service warpgroup
  } else {
    // ============================================================================ compute / epilogue warps
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(LAYERS_REG_COMPUTE));
    uint32_t pw = 0, ci = 0;
    int cur_type = -1, cur_layer = -1;
    const uint32_t xa = smem_u32(X) + (uint32_t)(tid >> 7) * 8192u;     // this warpgroup's 64 A rows
    const uint32_t raddr = smem_u32(ring);
    // BDIFF_TIMING: phase stamps (clock64) of the first edge / node item with k >= 2 of every CTA: [128 + 0..31] edge,
    // [128 + 32..63] node — one stamp before and after every GEMM phase, one at every accumulator read
    int es = 0;
    long long* stamp = nullptr;
    auto PH = [&]() __attribute__((always_inline)) { if (stamp && tid == 0 && es < 32) stamp[es] = clock64(); ++es; };
    bool stamped[2] = {false, false};
    auto sz = [](int n) { return (uint32_t)((n * 4 + 15) & ~15); };
    for (uint32_t k = 0;; ++k) {
      const uint32_t slot = k & 1;
      mbar_wait(&B.item_full[slot], (k >> 1) & 1);
      const int type = __shfl_sync(0xffffffffu, B.item[slot][0], 0);
      const int layer = __shfl_sync(0xffffffffu, B.item[slot][1], 0);
      const int tile = __shfl_sync(0xffffffffu, B.item[slot][2], 0);
      if (type < 0) break;
      if (tid == 0 && w.dbg && k < 16) {      // BDIFF_TIMING: {item code, t_fetch, t_start, t_end} for the first 16 items
        w.dbg[(size_t)blockIdx.x * 64 + 4 * k] = (type << 30) | (layer << 24) | tile;
        w.dbg[(size_t)blockIdx.x * 64 + 4 * k + 1] = clock64();
      }
      // ---- small (vector-channel) weights of this (pass, layer): reload only when they change
      if (type != cur_type || layer != cur_layer) {
        named_bar_sync(3, TC_EPI);             // everybody is done with the previous set
        if (tid == 0) {
          const LayerW lw = q.layers[layer];       // by value: the pointer loads go out together, not one per copy
          // every (destination, source, count) is listed once and visited twice: for the byte total, then for the copies
          auto stage = [&](auto&& list) {
            uint32_t total = 0;
            list([&](float*, const float*, int n) { total += sz(n); });
            mbar_expect_tx(&B.wbar, total);
            list([&](float* dst, const float* src, int n) { bulk_g2s(dst, src, sz(n), &B.wbar); });
          };
          if (type == 0) {
            stage([&](auto&& cp) { small_w_copies<XD>(reinterpret_cast<EdgeTail*>(tail)->sw, lw, cp); });
          } else {
            const int last = layer == q.L - 1;
            const LayerW wn = q.layers[last ? layer : layer + 1];
            stage([&](auto&& cp) { small_wr4_copies(reinterpret_cast<NodeTail*>(tail)->sw, lw, wn, ew, hid0, d.Hin, last, cp); });
          }
        }
        mbar_wait(&B.wbar, pw);
        pw ^= 1;
        cur_type = type; cur_layer = layer;
      }
      // ---- dependencies: completion flags of the producer tiles (bounded spin), then a gpu-scope acquire in
      //      every thread before it reads activations written by other SMs
      if (tid == 0) {
        int lo = 0, hi = -1;
        const int* fbase = flags;
        if (type == 0) {
          if (layer > 0) {
            const int2 dep = q.edge_dep[tile];
            lo = dep.x; hi = dep.y;
            fbase = flags + (size_t)(layer - 1) * per_layer + q.TE;
          }
        } else {
          const int2 dep = q.node_dep[tile];
          lo = dep.x; hi = dep.y;
          fbase = flags + (size_t)layer * per_layer;
        }
        const long long t0 = clock64();
        for (int u = lo; u <= hi; ++u) {
          while (ld_acquire_gpu(fbase + u) == 0) {
            // every producer precedes its consumer in the claim order and all CTAs are resident, so this wait is bounded
            // by a few tile times; > 2^32 cycles (~2 s) can only mean a broken schedule: record it and abort the kernel
            // HERE (sticky launch failure) rather than computing on stale data
            if (clock64() - t0 > (1ll << 32)) { atomicExch(q.err, 1); __threadfence_system(); __trap(); }
          }
        }
      }
      named_bar_sync(3, TC_EPI);
      __threadfence();
      if (tid == 0 && w.dbg && k < 16) w.dbg[(size_t)blockIdx.x * 64 + 4 * k + 2] = clock64();
      es = 0;
      stamp = nullptr;
      if (w.dbg && k >= 2 && !stamped[type]) { stamp = w.dbg + 256 * 64 + (size_t)blockIdx.x * 64 + type * 32; stamped[type] = true; }
      PH();
      // GEMM phases run where the epilogue publishes an operand: both warpgroups issue their wgmmas and leave the
      // accumulators in the scratch, which the epilogue reads after the closing barrier, or hand them to an elementwise
      // epilogue in registers (edge tile: E0, E(k)b).
      // The lambdas are always inlined: compiled as a called subroutine, a GEMM phase is a path that ptxas cannot prove
      // warp-uniform, and then it serializes EVERY wgmma of the kernel (C7520; tests/test_layers_sass.py).  Inlined, each
      // publish site sees a constant phase, and a ring chunk's wgmmas issue back to back with one wait at its end.
      const int last = type == 1 && layer == q.L - 1;
      int ph = 0;
      auto gemm = [&](int phase) __attribute__((always_inline)) {
        if (type == 0) {
          const int ph = phase;
#include "edge_tile_mma.inc"
        } else {
          const int ph = phase;
#include "node_r4_tile_mma.inc"
        }
      };
      // run: a GEMM phase whose epilogue runs inside it (writes the A tile, nothing to read back from the scratch), so the
      // next publish follows directly; publish: a GEMM phase whose accumulators the epilogue reads after the barrier
      auto run = [&]() __attribute__((always_inline)) { fence_proxy_async(); named_bar_sync(3, TC_EPI); PH(); gemm(ph++); };
      auto publish = [&]() __attribute__((always_inline)) { run(); named_bar_sync(3, TC_EPI); PH(); };
      // node tile: U has been read (E3a), so G4 may overwrite its columns
      auto release_u = [&]() __attribute__((always_inline)) { named_bar_sync(3, TC_EPI); gemm(-1); named_bar_sync(3, TC_EPI); };
      if (type == 0) {
        EdgeTail& T = *reinterpret_cast<EdgeTail*>(tail);
        const int half = tid >> 7, r = tid & 127;
        const SmallW& sw = T.sw;
#include "edge_tile_epilogue.inc"
      } else {
        NodeTail& T = *reinterpret_cast<NodeTail*>(tail);
        NodeScratch& SC = *reinterpret_cast<NodeScratch*>(X + R5_BLOCKS * R5_BLOCK);
        const int l = lane, s = warp, c0 = warp * 32;
        const SmallWR4& sw = T.sw;
#include "node_r4_tile_epilogue.inc"
      }
      PH();
      if (tid == 0 && w.dbg && k < 16) w.dbg[(size_t)blockIdx.x * 64 + 4 * k + 3] = clock64();
      mbar_arrive(&B.tile_done);
      mbar_arrive(&B.item_empty[slot]);
    }
  }
  __syncthreads();
}

bool tc_supported(int Ed, int Xd) { return (Ed == 64 && Xd == 16) || (Ed == 16 && Xd == 8); }

cudaError_t tc_layers_configure() {
  cudaError_t e = cudaFuncSetAttribute(k_layers_tc<64, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)LAYERS_SMEM_BYTES);
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(k_layers_tc<16, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LAYERS_SMEM_BYTES);
}

// one CTA per SM at most (the accumulator scratch holds `num_sms` CTAs)
void launch_layers_tc(cudaStream_t st, const Plan& p, const Dims& d, const EmbedW& ew, const LayerSched& q,
                      const Work& w, int num_sms) {
  const int grid = q.nitems < num_sms ? q.nitems : num_sms;
  if (d.Ed == 64) k_layers_tc<64, 16><<<grid, LAYERS_THREADS, LAYERS_SMEM_BYTES, st>>>(p, d, ew, q, w);
  else k_layers_tc<16, 8><<<grid, LAYERS_THREADS, LAYERS_SMEM_BYTES, st>>>(p, d, ew, q, w);
}

}  // namespace bdiff
