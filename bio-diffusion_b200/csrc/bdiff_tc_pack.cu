// bdiff_tc_pack.cu — per-layer weight streams of the tensor path: split-bf16 K=16 slabs (bdiff_slab.cuh) laid out as the
// stream tables say (tc_edge_stream / tc_node_stream), which is how the megakernel's TMA lane streams them.  Runs once
// per weight update (bdiff_prepare).
#include "bdiff_node_tc.cuh"

namespace bdiff {

size_t tc_blob_bytes(int Ed, int Xd) { return stream_bytes(tc_edge_stream(tc_k0_steps(Ed, Xd))); }
size_t tc_node_blob_bytes() { return stream_bytes(tc_node_stream(false)); }      // the last layer's stream is shorter

// Where global plane row `row` of a stream (counting the 2 * rows plane rows of every step, segment after segment) lives.
struct SlabPos {
  int seg, rows;      // segment index, its plane height
  int k0, n;          // first K row of the step inside the segment's weight matrix; row inside the step's 2 * rows
  int half, local;    // N half and local plane row that row n goes to
  size_t base;        // byte offset of the step inside an N half's stream
};
__device__ bool stream_find(const Stream& S, long long row, SlabPos& p) {
  size_t base = 0;
  for (int i = 0; i < S.n; ++i) {
    const StreamSeg g = S.seg[i];
    const long long seg_rows = (long long)g.steps * 2 * g.rows;
    if (row >= seg_rows) {
      row -= seg_rows;
      base += (size_t)g.steps * seg_step_bytes(g);
      continue;
    }
    const int step = (int)(row / (2 * g.rows)), n = (int)(row % (2 * g.rows));
    const int body = g.rows < 128 ? g.rows : 128, gate = g.rows - body;      // product rows | gate rows of one half
    p.seg = i; p.rows = g.rows; p.k0 = step * 16; p.n = n;
    p.base = base + (size_t)step * seg_step_bytes(g);
    if (n < 2 * body) { p.half = n / body; p.local = n % body; }
    else { p.half = (n - 2 * body) / gate; p.local = body + (n - 2 * body) % gate; }
    return true;
  }
  return false;
}

// Edge pass (tc_edge_stream).  Gate rows of G(k)u: GCP k adds +Wg_{k-1} m_{k-1} to U[(k-1) & 1] and starts
// U[k & 1] = -Wg_k m_{k-1} (sign folded into the packed weights so that U0 | U1 is one N=64 accumulator range).
// one thread per (global plane row, k in [0,16)); writes the hi and the lo plane element
__global__ void k_pack_edge_slabs(LayerW lw, Dims d, unsigned char* __restrict__ blob, size_t half_bytes) {
  const Stream S = tc_edge_stream(tc_k0_steps(d.Ed, d.Xd));
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int kk = (int)(idx & 15);
  SlabPos p;
  if (!stream_find(S, idx >> 4, p)) return;
  const int n = p.n, k = p.k0 + kk;
  float v;
  if (p.seg == 0) {
    v = k < d.K0 ? lw.W0e[(size_t)k * 256 + n] : 0.f;
  } else if (p.seg == 7) {
    v = lw.Wgk[2][(size_t)k * 32 + n];
  } else {
    const int gi = (p.seg - 1) >> 1;        // GCP gi + 1
    if (!(p.seg & 1)) {                     // G(k)s
      v = k < kKM ? lw.Wk[gi][(size_t)k * 256 + n] : 0.f;
    } else {                                // G(k)u
      const float* wprev = gi == 0 ? lw.Wg0 : lw.Wgk[gi - 1];
      const float* wthis = lw.Wgk[gi];
      const bool odd = ((gi + 1) & 1) != 0;           // GCP odd: U0 <- +prev, U1 <- -this;  even: U0 <- -this, U1 <- +prev
      const int c = n & 31;
      v = (p.half == 0) == odd ? wprev[(size_t)k * 32 + c] : -wthis[(size_t)k * 32 + c];
    }
  }
  slab_store(blob + (size_t)p.half * half_bytes + p.base, p.rows, p.local, kk, v);
}

// Node pass (tc_node_stream)
__global__ void k_pack_node_slabs(LayerW lw, LayerW wn, EmbedW ew, Dims d, int last, unsigned char* __restrict__ blob,
                                  size_t half_bytes) {
  const Stream S = tc_node_stream(last);
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int kk = (int)(idx & 15);
  SlabPos p;
  if (!stream_find(S, idx >> 4, p)) return;
  const int n = p.n, k = p.k0 + kk;
  float v;
  switch (p.seg) {
    case NG_1A: v = lw.W1[(size_t)k * 256 + n]; break;
    case NG_1B: v = n < 256 ? lw.W1[(size_t)(256 + k) * 256 + n] : -lw.Wgf[(size_t)k * 32 + (n - 256)]; break;   // U = -Wg h_old
    case NG_1C: v = 512 + k < kKFF ? lw.W1[(size_t)(512 + k) * 256 + n] : 0.f; break;
    case NG_2: v = lw.W2[(size_t)k * 256 + n]; break;
    case NG_3A: v = n < 256 ? lw.Wp[(size_t)k * 256 + n] : lw.Wgf[(size_t)k * 32 + (n - 256)]; break;
    default:
      if (p.seg == (last ? NGL_3B : NG_3B)) v = 256 + k < kKM ? lw.Wp[(size_t)(256 + k) * 256 + n] : 0.f;
      else if (last) v = (k < 300 && n < d.Hin) ? ew.pWs[(size_t)k * d.Hin + n] : 0.f;      // NGL_P
      else v = (p.seg == NG_4 ? wn.Wsi : wn.Wsj)[(size_t)k * 256 + n];
  }
  slab_store(blob + (size_t)p.half * half_bytes + p.base, p.rows, p.local, kk, v);
}

void launch_tc_pack(cudaStream_t st, const LayerW& lw, const Dims& d, unsigned char* blob) {
  const long long total = stream_plane_rows(tc_edge_stream(tc_k0_steps(d.Ed, d.Xd))) * 16;
  k_pack_edge_slabs<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(lw, d, blob, tc_blob_bytes(d.Ed, d.Xd) / 2);
}

void launch_tc_pack_node(cudaStream_t st, const LayerW& lw, const LayerW& wn, const EmbedW& ew, const Dims& d, int last,
                         unsigned char* blob) {
  const long long total = stream_plane_rows(tc_node_stream(last)) * 16;
  k_pack_node_slabs<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(lw, wn, ew, d, last, blob, tc_node_blob_bytes() / 2);
}

}  // namespace bdiff
