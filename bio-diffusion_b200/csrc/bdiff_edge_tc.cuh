// bdiff_edge_tc.cuh — declarations of the tensor-core edge tile of the layer megakernel (bdiff_layers_tc.cu):
// tile / accumulator-scratch constants, shared-memory layout, weight-slab stream, the ring consumer that the GEMM phases of
// both tiles use (run_seg), the small-weight copy list, the per-thread vector-channel update.
#pragma once
#include <type_traits>

#include "bdiff_kernels.h"
#include "bdiff_slab.cuh"

namespace bdiff {

constexpr int TMT = 128;                 // edges per tile
// weight ring: TC_NSLOT slots of TC_SLOT bytes; a chunk is always a single contiguous TMA bulk copy
constexpr int TC_SLOT = 2 * 160 * 32;    // 10 KiB: one N half of the widest K step (checked against the stream tables)
constexpr int TC_NSLOT = 5;
// accumulator-scratch column map of an edge tile (512 columns; S never leaves the registers, so columns 0..255 are unused)
constexpr int TM_U0 = 256, TM_U1 = 288, TM_MV = 320, TM_VD0 = 416;
constexpr int TM_EX = 416, TM_EX_STRIDE = 40;     // pair-exchange scratch (over VD0, which is dead by then): 2 x 40 columns

// ---- The weight stream of one (pass, layer), defined here and nowhere else: the pack kernels (bdiff_tc_pack.cu), the
// TMA lane and the GEMM phases of the megakernel all walk these tables.
// A stream is [N half 0 | N half 1]: every weight plane is split in two, and the megakernel multiplies one half at a
// time.  A half is a sequence of segments.  A segment is `steps` K=16 steps; a step is [hi plane | lo plane] of `rows`
// local rows each (slab layout of bdiff_slab.cuh, 2 * rows * 32 bytes).  `group` steps travel as one ring chunk (the
// last chunk of a segment may be short).  The consumer takes all chunks of a segment for half 0, then for half 1.
// The 2 * rows plane rows of a step are, in order: [128 product rows of half 0 | of half 1 | gate rows of half 0 | of
// half 1] (planes of fewer than 128 rows have no gate rows); a half's local rows are its product rows, then its gate rows.
struct StreamSeg { int steps, rows, group; };
struct Stream { StreamSeg seg[8]; int n; };
__host__ __device__ constexpr int seg_step_bytes(StreamSeg g) { return 2 * g.rows * 32; }
__host__ __device__ constexpr int seg_chunks(StreamSeg g) { return (g.steps + g.group - 1) / g.group; }
__host__ __device__ constexpr size_t stream_bytes(const Stream& s) {        // both halves
  size_t b = 0;
  for (int i = 0; i < s.n; ++i) b += (size_t)s.seg[i].steps * 2 * seg_step_bytes(s.seg[i]);
  return b;
}
__host__ __device__ constexpr long long stream_plane_rows(const Stream& s) {      // plane rows of both halves, all steps
  long long r = 0;
  for (int i = 0; i < s.n; ++i) r += (long long)s.seg[i].steps * 2 * s.seg[i].rows;
  return r;
}
__host__ __device__ constexpr int stream_max_chunk(const Stream& s) {
  int m = 0;
  for (int i = 0; i < s.n; ++i) {
    const int c = s.seg[i].group * seg_step_bytes(s.seg[i]);
    m = c > m ? c : m;
  }
  return m;
}

__host__ __device__ constexpr int tc_k0_steps(int Ed, int Xd) {     // K=16 steps of message GCP 0's edge part
  return (Ed + (64 + Xd) / 4 + 9 + 15) / 16;
}
// Edge pass: entry i is GEMM phase i of edge_tile_mma.inc.
//   G0: W0e, zero-padded to k0s * 16 K rows;  G(k)u, k = 1..3: 32 gate rows of m_{k-1} (half 0 -> U0, half 1 -> U1),
//   four K steps per chunk;  G(k)s: all K rows of W_k ([m_{k-1} | vn_k | q_k], zero-padded to 288);  G4: Wg_3, four K
//   steps per chunk.
__host__ __device__ constexpr Stream tc_edge_stream(int k0s) {
  constexpr StreamSeg Gu{16, 32, 4}, Gs{18, 128, 1};
  return {{{k0s, 128, 1}, Gu, Gs, Gu, Gs, Gu, Gs, {16, 16, 4}}, 8};
}
static_assert(stream_max_chunk(tc_edge_stream(8)) <= TC_SLOT, "an edge-pass chunk must fit a ring slot");

// mbarriers / bookkeeping of the megakernel; first member (base class) of both tile tails
struct TcBars {
  uint64_t full[TC_NSLOT], empty[TC_NSLOT], wbar;
  uint64_t item_full[2], item_empty[2], tile_done;
  alignas(16) int item[2][4];   // work items {type, layer, tile, -}
};

// Thread roles: warps 0-7 epilogue/compute — edge r of the tile is owned by the thread PAIR (r, r+128): "half" 0
// works on accumulator columns [0,128) and vector channels [0,16), half 1 on columns [128,256) and channels
// [16,32) (both warps of a pair address the same scratch rows: row quarter = warp % 4).  The two compute warpgroups
// also issue the wgmmas (warpgroup g: tile rows [64 g, 64 g + 64)).  Warp 8 = scheduler + TMA producer, warp 9 =
// completion-flag lane.
constexpr int TC_EPI = 256;

// One ring chunk c of a GEMM phase: issue(ts, tu, chunk address, c) issues its wgmmas into fresh register tiles (ts: NS
// columns; tu: TU tiles of NU columns, for chunks that carry TU K steps whose products must stay apart), one wait, the
// slot is released, and the tiles are added to the running sums s / u with round-to-nearest fp32 adds, tile after tile:
// the tensor core's own fp32 accumulation truncates, and over a 1000-step chain (where |h| grows by ~17 decades) that
// bias towards zero compounds into a visible drift from the fp32 path.
template <int NS, int NU, int TU, class Issue>
__device__ __forceinline__ void seg_chunk(TcBars& B, uint32_t raddr, uint32_t& ci, int c, float* s, float* u, Issue& issue) {
  constexpr int RS = NS ? NS / 2 : 1, RU = NU ? NU / 2 : 1;
  const uint32_t slot = ci % TC_NSLOT;
  float ts[RS], tu[TU * RU];
#pragma unroll
  for (int i = 0; i < RS; ++i) ts[i] = 0.f;
#pragma unroll
  for (int i = 0; i < TU * RU; ++i) tu[i] = 0.f;
  mbar_wait(&B.full[slot], (ci / TC_NSLOT) & 1);
  wgmma_fence();
  issue(ts, tu, raddr + slot * TC_SLOT, c);
  wgmma_commit();
  wgmma_wait<0>();
  acc_fence<RS>(ts);
  acc_fence<TU * RU>(tu);
  mbar_arrive_if(&B.empty[slot], (threadIdx.x & 31) == 0);
  ++ci;
  if (NS) {
#pragma unroll
    for (int i = 0; i < RS; ++i) s[i] += ts[i];
  }
  if (NU) {
#pragma unroll
    for (int t = 0; t < TU; ++t)
#pragma unroll
      for (int i = 0; i < RU; ++i) u[i] += tu[t * RU + i];
  }
}

// One weight-stream segment of a GEMM phase, run by both compute warpgroups (warpgroup wg: tile rows [64 wg, 64 wg + 64)).
// For each N half h of the weight planes, `nch` = seg_chunks(stream-table entry) ring chunks (seg_chunk) into the
// accumulators s (NS columns, scratch columns scol + h NS) and u (NU columns at ucol + h NU), which start at zero (s:
// sfresh; u: bit h of ufresh) or from the scratch.  A finished half goes to the scratch, or, when an epilogue
// `epi(s, u, h, wg)` is given, to that functor (fragment layout: frag_row / frag_col), which then runs between the
// halves' wgmmas: it must be always_inline and free of divergent branches (see the kernel's note on C7520).
struct AccToScratch {};
template <int NS, int NU, int TU = 1, class Issue, class Epi = AccToScratch>
__device__ __forceinline__ void run_seg(TcBars& B, uint32_t raddr, uint32_t& ci, int nch, int scol, bool sfresh, int ucol,
                                        int ufresh, Issue&& issue, Epi&& epi = Epi{}) {
  constexpr int RS = NS ? NS / 2 : 1, RU = NU ? NU / 2 : 1;
  const int wg = threadIdx.x >> 7;
  for (int h = 0; h < 2; ++h) {
    float s[RS], u[RU];
    if (NS) {
      if (sfresh) {
#pragma unroll
        for (int i = 0; i < RS; ++i) s[i] = 0.f;
      } else {
        acc_load<NS>(s, scol + h * NS, wg);
      }
    }
    if (NU) {
      if ((ufresh >> h) & 1) {
#pragma unroll
        for (int i = 0; i < RU; ++i) u[i] = 0.f;
      } else {
        acc_load<NU>(u, ucol + h * NU, wg);
      }
    }
    for (int c = 0; c < nch; ++c) seg_chunk<NS, NU, TU>(B, raddr, ci, c, s, u, issue);
    if constexpr (std::is_same_v<std::decay_t<Epi>, AccToScratch>) {
      if (NS) acc_store<NS>(s, scol + h * NS, wg);
      if (NU) acc_store<NU>(u, ucol + h * NU, wg);
    } else {
      epi(s, u, h, wg);
    }
  }
}

// A segment of N = 2 x 128 columns that starts at zero and whose epilogue overwrites part of its own A operand: N half
// 0's epilogue writes A columns that half 1's chunks 0..hold still read.  Half 0's finished accumulators therefore wait
// in registers until this warpgroup has retired half 1's chunk `hold`; then epi(s, nullptr, 0, wg) runs, then the rest of
// half 1 and epi(s, nullptr, 1, wg).  Same products and adds in the same order as run_seg<128, 0>.
template <class Issue, class Epi>
__device__ __forceinline__ void run_seg_held(TcBars& B, uint32_t raddr, uint32_t& ci, int nch, int hold, Issue&& issue,
                                             Epi&& epi) {
  const int wg = threadIdx.x >> 7;
  float s0[64], s1[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) s0[i] = 0.f;
  for (int c = 0; c < nch; ++c) seg_chunk<128, 0, 1>(B, raddr, ci, c, s0, nullptr, issue);
#pragma unroll
  for (int i = 0; i < 64; ++i) s1[i] = 0.f;
  for (int c = 0; c <= hold; ++c) seg_chunk<128, 0, 1>(B, raddr, ci, c, s1, nullptr, issue);
  epi(s0, nullptr, 0, wg);
  for (int c = hold + 1; c < nch; ++c) seg_chunk<128, 0, 1>(B, raddr, ci, c, s1, nullptr, issue);
  epi(s1, nullptr, 1, wg);
}

struct alignas(16) SmallW {   // fp32 copies of the thread-local (vector channel) weights, broadcast-read
  float Wd0x[16 * 20];     // [Xd][hid0]
  float Wf0x[16 * 3];      // [Xd][3]
  float Wu0[20 * 32];      // [hid0][32]
  float Wdk[3][32 * 8];    // [32][8]
  float Wfk[3][32 * 3];    // [32][3]
  float Wuk[3][8 * 32];    // [8][32]
  float bg[4][32];
  float bk[3][256];
  float wa[256];
  float ba[4];
};
// every (destination, source, float count) that fills SmallW from the layer's weights lw, as cp(dst, src, n)
template <int XD, class Copy>
__device__ __forceinline__ void small_w_copies(SmallW& s, const LayerW& lw, Copy&& cp) {
  constexpr int HID0 = (64 + XD) / 4;
  cp(s.Wd0x, lw.Wd0x, XD * HID0); cp(s.Wf0x, lw.Wf0x, XD * 3); cp(s.Wu0, lw.Wu0, HID0 * 32);
  for (int kk = 0; kk < 3; ++kk) {
    cp(s.Wdk[kk], lw.Wdk[kk], 256); cp(s.Wuk[kk], lw.Wuk[kk], 256); cp(s.bk[kk], lw.bk[kk], 256);
    cp(s.Wfk[kk], lw.Wfk[kk], 96); cp(s.bg[kk + 1], lw.bgk[kk], 32);
  }
  cp(s.bg[0], lw.bg0, 32); cp(s.wa, lw.wa, 256); cp(s.ba, lw.ba, 1);
}

struct EdgeTail : TcBars {
  float2 wbuf[2][8][2][32];   // [round parity][16-row window]: [0] head piece (segment entered from the previous window), [1] tail / whole piece
  SmallW sw;
  float sAttn[2][TMT];
  int sRow[TMT], sCol[TMT], sB[TMT], sNa[TMT];
  uint32_t winfo[8];       // per window: start mask | end mask << 16
};

// Gate of the previous GCP from the scratch (U), vector-message update in the scratch for this thread's 16 channels,
// and this thread's partial vector_down / vector_down_frames sums of the NEXT GCP.
// HP = hidden dim of the previous GCP; vdp = its vector_down output (full, [HP][3]).
template <int HP, bool FIRST, bool LAST>
__device__ __forceinline__ void gate_update(int half, int ucol, const float* __restrict__ vdp,
                                            const float* __restrict__ Wu, const float* __restrict__ bgp,
                                            const float* __restrict__ Wdn, const float* __restrict__ Wfn,
                                            float* __restrict__ part) {   // part[33]: partial VD_next(24)+VDF_next(9)
  float2 p2[4][3];                 // VD_next accumulators, pairs of hidden rows (h = 2hp, 2hp+1) per component
  if (!LAST) {
#pragma unroll
    for (int i = 0; i < 33; ++i) part[i] = 0.f;
#pragma unroll
    for (int hp = 0; hp < 4; ++hp) { p2[hp][0] = make_float2(0.f, 0.f); p2[hp][1] = p2[hp][0]; p2[hp][2] = p2[hp][0]; }
  }
  for (int oc = half * 2; oc < half * 2 + 2; ++oc) {
    float u[8], mv[24];
    scratch_ld<8>(ucol + oc * 8, u);
    if (!FIRST) scratch_ld<24>(TM_MV + oc * 24, mv);
#pragma unroll
    for (int jp = 0; jp < 4; ++jp) {          // two output channels (j = 2jp, 2jp+1) per packed instruction
      const int o = oc * 8 + 2 * jp;
      const float2 g = sigmoid_acc2(__fadd2_rn(make_float2(u[2 * jp], u[2 * jp + 1]),
                                               *reinterpret_cast<const float2*>(bgp + o)));
      float2 s0 = make_float2(0.f, 0.f), s1 = s0, s2 = s0;
#pragma unroll
      for (int h = 0; h < HP; ++h) {
        const float2 wu = *reinterpret_cast<const float2*>(Wu + h * 32 + o);
        s0 = __ffma2_rn(wu, make_float2(vdp[h * 3 + 0], vdp[h * 3 + 0]), s0);
        s1 = __ffma2_rn(wu, make_float2(vdp[h * 3 + 1], vdp[h * 3 + 1]), s1);
        s2 = __ffma2_rn(wu, make_float2(vdp[h * 3 + 2], vdp[h * 3 + 2]), s2);
      }
      const int ja = 2 * jp * 3, jb = (2 * jp + 1) * 3;
      float2 r0, r1, r2;
      if (FIRST) { r0 = __fmul2_rn(s0, g); r1 = __fmul2_rn(s1, g); r2 = __fmul2_rn(s2, g); }
      else {
        r0 = __ffma2_rn(s0, g, make_float2(mv[ja + 0], mv[jb + 0]));
        r1 = __ffma2_rn(s1, g, make_float2(mv[ja + 1], mv[jb + 1]));
        r2 = __ffma2_rn(s2, g, make_float2(mv[ja + 2], mv[jb + 2]));
      }
      mv[ja + 0] = r0.x; mv[jb + 0] = r0.y; mv[ja + 1] = r1.x; mv[jb + 1] = r1.y; mv[ja + 2] = r2.x; mv[jb + 2] = r2.y;
    }
    scratch_st<24>(TM_MV + oc * 24, mv);
    if (!LAST) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = oc * 8 + j;
        const float4 wd0 = *reinterpret_cast<const float4*>(Wdn + c * 8), wd1 = *reinterpret_cast<const float4*>(Wdn + c * 8 + 4);
        const float2 wdp[4] = {make_float2(wd0.x, wd0.y), make_float2(wd0.z, wd0.w), make_float2(wd1.x, wd1.y),
                               make_float2(wd1.z, wd1.w)};
#pragma unroll
        for (int x = 0; x < 3; ++x) {
          const float2 mb = make_float2(mv[j * 3 + x], mv[j * 3 + x]);
#pragma unroll
          for (int hp = 0; hp < 4; ++hp) p2[hp][x] = __ffma2_rn(wdp[hp], mb, p2[hp][x]);
        }
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
          const float wf = Wfn[c * 3 + ch];
          part[24 + ch * 3 + 0] = fmaf(wf, mv[j * 3 + 0], part[24 + ch * 3 + 0]);
          part[24 + ch * 3 + 1] = fmaf(wf, mv[j * 3 + 1], part[24 + ch * 3 + 1]);
          part[24 + ch * 3 + 2] = fmaf(wf, mv[j * 3 + 2], part[24 + ch * 3 + 2]);
        }
      }
    }
  }
  if (!LAST) {
#pragma unroll
    for (int hp = 0; hp < 4; ++hp)
#pragma unroll
      for (int x = 0; x < 3; ++x) { part[(2 * hp) * 3 + x] = p2[hp][x].x; part[(2 * hp + 1) * 3 + x] = p2[hp][x].y; }
  }
}

// The two threads of a pair (same scratch row) swap their 33 partial sums through scratch columns.
// Callers guarantee that nobody still reads the columns (VD0) being overwritten.
__device__ __forceinline__ void pair_exchange33(int half, const float* __restrict__ mine, float* __restrict__ theirs) {
  float pad[40];
#pragma unroll
  for (int i = 0; i < 33; ++i) pad[i] = mine[i];
#pragma unroll
  for (int i = 33; i < 40; ++i) pad[i] = 0.f;
  scratch_st<40>(TM_EX + half * TM_EX_STRIDE, pad);
  named_bar_sync(3, TC_EPI);
  float got[40];
  scratch_ld<40>(TM_EX + (half ^ 1) * TM_EX_STRIDE, got);
#pragma unroll
  for (int i = 0; i < 33; ++i) theirs[i] = got[i];
}

}  // namespace bdiff
