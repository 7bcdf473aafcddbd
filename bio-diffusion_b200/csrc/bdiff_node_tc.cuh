// bdiff_node_tc.cuh — declarations of the tensor-core node tile of the layer megakernel (bdiff_layers_tc.cu).
//
// Tile = 32 nodes.  The A operand uses the "R5" split-bf16 layout of bdiff_slab.cuh (each node row stored as
// hi, lo, hi, lo, hi; two 128-row views and four products per K step), which leaves node l's complete accumulator row
// in all four row quarters of the accumulator scratch: the 8 compute warps share the same 32 nodes, warp s owns
// accumulator columns [32 s, 32 s + 32) (read from its own row quarter) and 1/8 of the vector-channel work.
#pragma once
#include "bdiff_edge_tc.cuh"

namespace bdiff {

constexpr int NT_EPI = 256;
constexpr int NM_S = 0, NM_U = 256;
constexpr int R4M = 32;
constexpr int NM_S1 = 256;        // second accumulator (overlaps U, see G4)

// Node pass weight stream (StreamSeg / Stream: bdiff_edge_tc.cuh), in issue order; the last layer has no next layer to
// prepare (G4, G5) and ends with the projection instead.
//   G1a: W1[0:256]   G1b: W1[256:512] + 16 gate rows of -Wg_ff   G1c: W1[512:544]   G2: W2   G3a: Wp[0:256] + 16 gate rows of Wg_ff
//   G4: next.Wsi   G3b: Wp[256:288]   G5: next.Wsj   Gp: projection scalar_out (K = 300 -> 19 steps, Hin -> 32 rows, zero padded)
enum { NG_1A, NG_1B, NG_1C, NG_2, NG_3A, NG_4, NG_3B, NG_5, NGL_3B = 5, NGL_P = 6 };     // NGL_*: the last layer's tail
__host__ __device__ constexpr Stream tc_node_stream(bool last) {
  constexpr StreamSeg G{16, 128, 1}, Gg{16, 144, 1}, Gx{2, 128, 1};
  return last ? Stream{{G, Gg, Gx, G, Gg, Gx, {19, 16, 4}}, 7} : Stream{{G, Gg, Gx, G, Gg, G, Gx, G}, 8};
}
static_assert(stream_max_chunk(tc_node_stream(false)) <= TC_SLOT && stream_max_chunk(tc_node_stream(true)) <= TC_SLOT,
              "a node-pass chunk must fit a ring slot");

// the small weights with the (mutually exclusive) next-layer / projection sets overlaid
struct alignas(16) SmallWR4 {
  float Wdf[64 * 16], Wff[64 * 3], Wuf[16 * 32], bgf[32];
  float b1[256], b2[256];
  float Wdp[32 * 8], Wfp[32 * 3], Wup[8], bp[256], wgp[256], bgp[4];
  union {
    struct { float b0[256], Wd0i[32 * 20], Wd0j[32 * 20], Wf0i[32 * 3], Wf0j[32 * 3]; } nx;
    struct { float pWd[32 * 32], pWf[32 * 3], pbs[32]; } pj;
  } u;
};
// every (destination, source, float count) that fills SmallWR4 for a node tile of the layer lw, as cp(dst, src, n):
// the next layer's set from wn, or in the last layer (wn unused) the projection set from ew
template <class Copy>
__device__ __forceinline__ void small_wr4_copies(SmallWR4& s, const LayerW& lw, const LayerW& wn, const EmbedW& ew, int hid0,
                                                 int hin, bool last, Copy&& cp) {
  cp(s.Wdf, lw.Wdf, 64 * 16); cp(s.Wff, lw.Wff, 64 * 3); cp(s.Wuf, lw.Wuf, 16 * 32); cp(s.bgf, lw.bgf, 32);
  cp(s.b1, lw.b1, 256); cp(s.b2, lw.b2, 256);
  cp(s.Wdp, lw.Wdp, 32 * 8); cp(s.Wfp, lw.Wfp, 32 * 3); cp(s.Wup, lw.Wup, 8); cp(s.bp, lw.bp, 256);
  cp(s.wgp, lw.Wgp, 256); cp(s.bgp, lw.bgp, 1);
  if (!last) {
    cp(s.u.nx.b0, wn.b0, 256);
    cp(s.u.nx.Wd0i, wn.Wd0i, 32 * hid0); cp(s.u.nx.Wd0j, wn.Wd0j, 32 * hid0);
    cp(s.u.nx.Wf0i, wn.Wf0i, 96); cp(s.u.nx.Wf0j, wn.Wf0j, 96);
  } else {
    cp(s.u.pj.pWd, ew.pWd, 32 * 32); cp(s.u.pj.pWf, ew.pWf, 96); cp(s.u.pj.pbs, ew.pbs, hin);
  }
}

struct NodeTail : TcBars {
  SmallWR4 sw;
};

// scratch of a node tile; lives behind the 5 R5 blocks inside the (larger) A region of the edge tile
struct NodeScratch {
  float4 sT[8][8 * 8];     // per-warp 8 x 32 fp32 transposition scratch (xor-swizzled 16-byte chunks)
  float sV[R4M][193];      // per node [agg_v (32x3) | chi (32x3)]; chi is replaced by chi_new in E3a
  float sVD[R4M][49];      // vector_down of the feed-forward GCP (16 x 3)
  float sVP[R4M][25];      // vector_down of the position GCP (8 x 3)
  float sDot[8][R4M];
};
static_assert(R5_BLOCKS * (size_t)R5_BLOCK + sizeof(NodeScratch) <= XE_BLOCKS * (size_t)X_BLOCK, "node scratch must fit behind the R5 blocks");

// Global <-> "lane = row" register tiles through the per-warp scratch, so that every global instruction touches 4
// rows x 128 contiguous bytes instead of 32 rows x 16 bytes (the L1 processes one line tag per cycle).
// v[32] = this lane's row (32 consecutive floats); gbase -> (row 0, first column) of the warp's 32 x 32 block.
__device__ __forceinline__ void warp_store_rows(float4* sc, const float* v, float* gbase, int ld, int lane) {
#pragma unroll
  for (int pass = 0; pass < 4; ++pass) {          // 8 rows per pass (1 KiB of scratch per warp)
    if ((lane >> 3) == pass) {
      const int r = lane & 7;
#pragma unroll
      for (int j = 0; j < 8; ++j) sc[r * 8 + (j ^ r)] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = 4 * i + (lane >> 3);
      const float4 t = sc[r * 8 + ((lane & 7) ^ r)];
      *reinterpret_cast<float4*>(gbase + (size_t)(pass * 8 + r) * ld + (lane & 7) * 4) = t;
    }
    __syncwarp();
  }
}
// t[8]: t[i] = float4 #(lane & 7) of row 4i + (lane >> 3) of the block (see the caller's loads)
__device__ __forceinline__ void warp_load_rows(float4* sc, float* v, const float4* t, int lane) {
#pragma unroll
  for (int pass = 0; pass < 4; ++pass) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = 4 * i + (lane >> 3);
      sc[r * 8 + ((lane & 7) ^ r)] = t[pass * 2 + i];
    }
    __syncwarp();
    if ((lane >> 3) == pass) {
      const int r = lane & 7;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 x = sc[r * 8 + (j ^ r)];
        v[4 * j] = x.x; v[4 * j + 1] = x.y; v[4 * j + 2] = x.z; v[4 * j + 3] = x.w;
      }
    }
    __syncwarp();
  }
}

}  // namespace bdiff
