// LSTM time step with the cell update fused into the recurrent GEMM's epilogue (DESIGN.md 9, item 1).
//
//   pre[:, g*H + u] = h_{t-1} W_hh^T  (wgmma, 3xTF32 or TF32)  + P_obs[trace] + P_step[segment] + smp_emb W_smp
//   i,f,o = sigmoid, g = tanh;  c_t = f c_{t-1} + i g;  h_t = o tanh(c_t)          (torch.nn.LSTM, gate order i,f,g,o)
//
// replaces, for t >= 1, the pair (tcg::k_grouped<X3,0> writing fp32 gate pre-activations, k_cell_fwd re-reading
// them): pyprob/nn/inference_network_lstm.py:186-188.  The trick is the weight layout: W_hh is packed with
// GATE-INTERLEAVED rows — packed row ub*128 + g*32 + j  <-  original row g*H + ub*32 + j — so that the 128 output
// columns of one tile are the four gates of the SAME 32 hidden units, and epilogue warp (q, cb) holds gate cb of rows
// 32q..32q+31.  Each warp finishes its gate (adds the projections, applies the activation, stores it for the
// backward pass, keeps it in its staging block); after a 128-thread named barrier per row quadrant the four warps
// each complete 8 rows of the cell: c, h, and the K-/MN-format tile images of h that the next step, the heads and
// the weight-gradient GEMMs read.
//
// Mainloop, pipeline, descriptors and the 3xTF32 scheme are those of tc_grouped.cuh.
//
// The default step runs k_lstm_step, one launch per time step, whenever pick_cluster (net_tc.inc) finds no cluster split
// worth making: H < 128 (K too short to split) or more than SMs / 2 tiles (two CTAs per tile would not fit one wave).
// Otherwise the step runs tcc::k_lstm_cluster (tc_cluster.cuh), which shares the step list, CellIO and the W_hh layout.
#pragma once
#include "tc_grouped.cuh"

namespace tcl {

using namespace tc;

struct CellIO {               // element-wise operands of the cell update, shared by all steps of a launch
  const float* p_obs;         // [traces, 4H]  observation projection, original gate-major columns
  const float* p_step;        // [steps, 4H]   step-embedding projection + both biases
  const float* smp_emb;       // [rows, S]     previous-sample embedding of every row
  const float* w_smp_t;       // [S, 4H]       W_ih columns of the sample embedding, transposed
  const int* row_trace;       // [rows] trace of a row, -1 for padding rows
  const int* row_step;        // [rows] step (segment) id of a row
  const int* row_prev;        // [rows] row of the same trace at step t-1
  float* gates;               // [rows, 4H] activated gates (i,f,g,o), gate-major columns — read by the backward pass
  float* c;                   // [rows, H]
  float* h;                   // [rows, H]
  float* hk_hi; float* hk_lo; float* hmn_hi; float* hmn_lo;   // tile images of h (both formats)
  int hkb;                    // column blocks of the h images (H / 32)
  int H, S;                   // hidden size (reduction length; N = 4H), sample-embedding width (<= 8)
};

struct Step {                 // one (time step t >= 1, sub-batch) segment: one launch per time step
  tcg::Operand a;             // h image, rows of the segment at step t-1 (K-major, row0 = previous row origin)
  tcg::Operand b;             // gate-interleaved W_hh image (K-major, 4H rows, H columns)
  int M;                      // segment rows, padded to 128
  int row0;                   // first global row of the segment at step t (multiple of 128)
  int tile_start, tiles_m, tiles_n;
  CellIO io;
};

struct __align__(1024) Smem {
  float a_hi[tcg::kStages][kTileFloats];
  float a_lo[tcg::kStages][kTileFloats];
  float b_hi[tcg::kStages][kTileFloats];
  float b_lo[tcg::kStages][kTileFloats];
  uint64_t full[tcg::kStages];
  uint64_t empty[tcg::kStages];
  Step step;
};
static_assert(tcg::kEpiWarps * 32 * 33 * 4 <= 2 * tcg::kStages * kTileBytes, "staging blocks must fit in the A stages");

__device__ __forceinline__ void quad_barrier(int q) {  // the four epilogue warps of 32-row block q
  asm volatile("bar.sync %0, %1;" ::"r"(1 + q), "r"(128) : "memory");
}

// Epilogue of one 128-row x 32-unit tile: gate activations (phase 1), then the cell update (phase 2).
// `staging` = base of the idle A stages, `ctile` = the step's result tile (tcg::kCPitch, in the B stages);
// `tile_row0` = global row of the tile's first row.  Called by the 16 consumer warps only, after the result tile is complete.
__device__ __forceinline__ void cell_epilogue(float* staging, const float* ctile, const CellIO& io, int warp, int lane, int nt,
                                              int64_t tile_row0) {
  const int q = warp & 3;              // 32-row block of the tile
  const int g = warp >> 2;             // 32-column chunk of the tile = gate (i, f, g, o)
  const int qi = q;                    // position of this quadrant's warp inside every group of four staging blocks
  float (*stg)[33] = reinterpret_cast<float (*)[33]>(staging + warp * 32 * 33);
  const int H = io.H, H4 = 4 * io.H, S = io.S;
  const int u = nt * 32 + lane;        // hidden unit owned by this lane
  const int col = g * H + u;           // its column in the gate-major [.., 4H] arrays
#pragma unroll
  for (int r = 0; r < 32; ++r) stg[r][lane] = ctile[(q * 32 + r) * tcg::kCPitch + g * 32 + lane];
  __syncwarp();
  float wsmp[8];
#pragma unroll
  for (int s = 0; s < 8; ++s) wsmp[s] = (s < S) ? __ldg(io.w_smp_t + (int64_t)s * H4 + col) : 0.0f;
  const int64_t row_base = tile_row0 + q * 32;
  // ---- phase 1: this warp's gate for its 32 rows ------------------------------------------------------------------
  for (int r = 0; r < 32; ++r) {
    const int64_t row = row_base + r;
    const int tr = __ldg(io.row_trace + row);
    float act = 0.0f;
    if (tr >= 0) {   // warp-uniform
      const int st = __ldg(io.row_step + row);
      // same order of additions as k_cell_fwd: (P_obs + P_step) + recurrent, then the sample-embedding FMAs
      float x = __ldg(io.p_obs + (int64_t)tr * H4 + col) + __ldg(io.p_step + (int64_t)st * H4 + col);
      x += stg[r][lane];
#pragma unroll
      for (int s = 0; s < 8; ++s)
        if (s < S) x = fmaf(__ldg(io.smp_emb + row * S + s), wsmp[s], x);
      act = (g == 2) ? ppb_cell_tanh(x) : ppb_cell_sigmoid(x);
    }
    tcg::st_global(io.gates + row * H4 + col, act);
    stg[r][lane] = act;
  }
  quad_barrier(q);
  // ---- phase 2: cell update, 8 rows per warp; the four gates come from the four staging blocks of the quadrant --------
  float (*sg_i)[33] = reinterpret_cast<float (*)[33]>(staging + (0 * 4 + qi) * 32 * 33);
  float (*sg_f)[33] = reinterpret_cast<float (*)[33]>(staging + (1 * 4 + qi) * 32 * 33);
  float (*sg_g)[33] = reinterpret_cast<float (*)[33]>(staging + (2 * 4 + qi) * 32 * 33);
  float (*sg_o)[33] = reinterpret_cast<float (*)[33]>(staging + (3 * 4 + qi) * 32 * 33);
  const int64_t hkb = io.hkb;
#pragma unroll
  for (int rr = 0; rr < 8; ++rr) {
    const int r = g * 8 + rr;
    const int64_t row = row_base + r;
    const int tr = __ldg(io.row_trace + row);
    float cn = 0.0f, hn = 0.0f;
    if (tr >= 0) {
      const int64_t rp = __ldg(io.row_prev + row);
      const float cp = tcg::ld_global(io.c + rp * H + u);
      cn = sg_f[r][lane] * cp + sg_i[r][lane] * sg_g[r][lane];
      hn = sg_o[r][lane] * ppb_cell_tanh(cn);
    }
    tcg::st_global(io.c + row * H + u, cn);
    tcg::st_global(io.h + row * H + u, hn);
    // image position of (row, u): column lane of block nt
    const int64_t span = img_span(row, nt, hkb);
    float hh, hl;
    split_tf32(hn, hh, hl);
    const int64_t pos_k = k_swz(row, lane, span);
    tcg::st_global(io.hk_hi + pos_k, hh);
    tcg::st_global(io.hk_lo + pos_k, hl);
    const int64_t pos_mn = mn_swz(row, lane, span);
    tcg::st_global(io.hmn_hi + pos_mn, hh);
    tcg::st_global(io.hmn_lo + pos_mn, hl);
  }
}

template <bool X3>
__global__ void __launch_bounds__(tcg::kThreads, 1) k_lstm_step(const Step* __restrict__ steps, int n_steps) {
  extern __shared__ uint8_t smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x;
  int lo_i = 0, hi_i = n_steps - 1;
  while (lo_i < hi_i) {
    int mid = (lo_i + hi_i + 1) >> 1;
    if (steps[mid].tile_start <= tile) lo_i = mid; else hi_i = mid - 1;
  }
  for (int i = threadIdx.x; i < (int)(sizeof(Step) / 4); i += blockDim.x)
    reinterpret_cast<uint32_t*>(&sm.step)[i] = reinterpret_cast<const uint32_t*>(steps + lo_i)[i];
  __syncthreads();
  const Step& P = sm.step;
  const int local = tile - P.tile_start;
  const int mt = local / P.tiles_n, nt = local % P.tiles_n;   // nt = block of 32 hidden units
  const int KC = (P.io.H + 31) / 32;

  if (warp == tcg::kProducerWarp && lane == 0) {
    for (int s = 0; s < tcg::kStages; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], tcg::kEpiWarps); }
    fence_barrier_init();
  }
  __syncthreads();
  const tcg::Ring R{sm.a_hi[0], sm.a_lo[0], sm.b_hi[0], sm.b_lo[0], kTileFloats, tcg::kStages, sm.full, sm.empty};

  if (warp == tcg::kProducerWarp) {
    if (lane == 0) tcg::produce<X3>(R, P.a, P.b, mt, nt, 0, KC, 0);
  } else {
    float acc[32];
    tcg::mma_mainloop<X3>(R, 0, KC, false, false, warp, lane, acc);
    float* const ctile = sm.b_hi[0];
    tcg::consumer_sync();
    tcg::store_acc(acc, warp, lane, [&](int r, int c) { return ctile + r * tcg::kCPitch + c; });
    tcg::consumer_sync();
    cell_epilogue(reinterpret_cast<float*>(sm.a_hi), ctile, P.io, warp, lane, nt, (int64_t)P.row0 + mt * 128);
  }
  __syncthreads();
}

inline size_t smem_bytes() { return sizeof(Smem) + 1024; }

// W_hh [4H, H] (row-major, gate-major rows) -> K-format hi / lo tile image with gate-interleaved rows
static __global__ void __launch_bounds__(256) k_pack_whh_interleaved(const float* __restrict__ w_hh, int H,
                                                               float* __restrict__ img_hi, float* __restrict__ img_lo) {
  const int rt = blockIdx.x;             // packed row tile = block of 32 hidden units
  pack_tile<Parts::k>(rt, H / 32, img_hi, img_lo, nullptr, nullptr, [&](int row, int k0, float (&x)[4]) {
    const int r = row - rt * 128;        // packed row inside the tile = gate * 32 + j
    const int src_row = (r >> 5) * H + rt * 32 + (r & 31);
#pragma unroll
    for (int j = 0; j < 4; ++j) x[j] = __ldg(w_hh + (int64_t)src_row * H + k0 + j);
  });
}

}  // namespace tcl
