// Cluster split-K wgmma GEMM: small-M problems spread over the SMs without atomics.
//
// The proposal network's per-time-step GEMMs have few rows (one minibatch: M = 256 .. 512) and a deep reduction
// (K = 512 forward, K = 2048 in BPTT).  One 128 x 128 tile per CTA leaves most SMs idle and makes one CTA walk the whole
// reduction at the per-SM operand-ingest rate (measured ~100 GB/s: 0.64 us per 32-element chunk in 3xTF32); global
// split-K (tc_grouped.cuh) fixes the parallelism but pays one fp32 red.add per element per split (measured 33 us for the
// 512 x 512 x 2048 BPTT GEMM, 9.4 MB of atomics).  Here the CS splits of one output tile form a thread-block CLUSTER:
// every CTA accumulates its K-slice in registers, parks the fp32 partial tile in its own shared memory (the operand stages
// are idle by then), and after a cluster barrier each CTA reduces 128 / CS rows of the tile over all partials through
// distributed shared memory (ld.shared::cluster) and runs the epilogue for those rows only.  No atomics, no zero-fill,
// fixed summation order, and the epilogue work is spread over the cluster too.
//
// Epilogues (reduce phase; one thread owns one row x four columns {lane, lane+32, lane+64, lane+96} of the tile):
//   k_cluster<X3, CS, 0>   fp32 store (+bias, ReLU, zero-invalid rows)           head dX
//   k_cluster<X3, CS, 2>   tile images (+fp32, ReLU-mask from an image)          head hidden layer and its gradient
//   k_cluster<X3, CS, 3, RE> whole-row epilogue of a caller type RE (N <= 128: one warp holds a whole output row): what
//                          re.load(row) returns is fetched before the mainloop; the bias-added row goes to a per-warp
//                          shared-memory buffer and re.row(state, loaded, x, row, lane) reads it as one warp; then EVERY
//                          thread calls re.finish(state, lane) (it may hold CTA barriers)
//                                                                                head output layer + NLL
//   k_cluster<X3, CS, 4, RE> element epilogue: re.cells(row, col0, v) gets a thread's four sums (columns col0 + 32 g)
//                                                                                T = 1 dh + LSTM cell backward
//   No fp32 store in 3 and 4: the caller's routine writes what its consumers read.
//   k_lstm_cluster<X3, CS> LSTM cell: with gate-interleaved W_hh the four columns of a thread are the gates i, f, g, o
//                          of ONE hidden unit, so the cell update is thread-local (tc_lstm.cuh has the layout)
// Mainloop, descriptors, the 3xTF32 scheme: tc_grouped.cuh.
#pragma once
#include "tc_grouped.cuh"
#include "tc_lstm.cuh"

namespace tcc {

using namespace tc;

// Parked partial tile: 128 rows x 128 floats, row r at byte 512 r, the eight 16-byte chunks of every 128-byte segment permuted
// by (chunk ^ (r & 7)), so that a reduce-phase warp reads one whole, 128-byte ALIGNED segment of one row per request (an odd
// pitch would make every remote read straddle two segments of distributed shared memory).
constexpr int kPitch = 128;
constexpr int kPartFloats = 128 * kPitch;    // 64 KB, aliases the operand stages
static_assert(kPartFloats * 4 <= 2 * tcg::kStages * kTileBytes, "partial tile must fit in the A stages");

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {   // every thread of every CTA of the cluster
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t map_to_rank(uint32_t local_smem_addr, uint32_t rank) {
  uint32_t ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local_smem_addr), "r"(rank));
  return ra;
}
__device__ __forceinline__ float ld_cluster(uint32_t cluster_addr) {
  float v;
  // volatile keeps it behind the cluster barrier (volatile + memory clobber); no clobber of its own, so that independent global
  // loads may be scheduled around it — nothing writes the parked tiles between the two cluster barriers
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(cluster_addr));
  return v;
}

struct __align__(1024) Smem {
  float a_hi[tcg::kStages][kTileFloats];
  float a_lo[tcg::kStages][kTileFloats];
  float b_hi[tcg::kStages][kTileFloats];
  float b_lo[tcg::kStages][kTileFloats];
  uint64_t full[tcg::kStages];
  uint64_t empty[tcg::kStages];
  union { tcg::Problem prob; tcl::Step step; };
};
inline size_t smem_bytes() { return sizeof(Smem) + 1024; }

// optional phase clock (ppb_debug_trace): CTA 0 stamps %globaltimer at the phase boundaries; slots as in tcg::k_grouped plus
// 7 = partials of the whole cluster visible
#define TCC_TRACE(slot)                                                                                   \
  do {                                                                                                    \
    if (trace && blockIdx.x == 0) {                                                                       \
      unsigned long long _t;                                                                              \
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(_t));                                              \
      trace[slot] = _t;                                                                                   \
    }                                                                                                     \
  } while (0)

// Mainloop over this CTA's K-slice [c0, c1) of output tile (mt, nt), then the partial tile parked in shared memory.
// Called by all threads; returns after the first cluster barrier (every partial of the cluster is readable).
template <bool X3>
__device__ __forceinline__ void mainloop_and_park(Smem& sm, const tcg::Operand& A, const tcg::Operand& B, int mt, int nt,
                                                  int c0, int c1, int warp, int lane,
                                                  unsigned long long* trace = nullptr, int b_prefetched = 0) {
  const tcg::Ring R{sm.a_hi[0], sm.a_lo[0], sm.b_hi[0], sm.b_lo[0], kTileFloats, tcg::kStages, sm.full, sm.empty};
  if (warp == tcg::kProducerWarp) {
    if (lane == 0) {
      const uint32_t bytes = (tcg::stage_bytes(A, mt) + tcg::stage_bytes(B, nt)) * (X3 ? 2u : 1u);
      for (int c = c0; c < c1; ++c) {
        int s = (c - c0) % tcg::kStages;
        uint32_t ph = ((c - c0) / tcg::kStages) & 1;
        mbar_wait(&sm.empty[s], ph ^ 1);
        const bool b_there = c - c0 < b_prefetched;   // B tile (and the expect-tx) of this stage issued before the PDL wait
        if (!b_there) mbar_expect_tx(&sm.full[s], bytes);
        tcg::load_operand(A, mt, c, sm.a_hi[s], sm.a_lo[s], X3, &sm.full[s]);
        if (!b_there) tcg::load_operand(B, nt, c, sm.b_hi[s], sm.b_lo[s], X3, &sm.full[s]);
      }
    }
  } else {
    float acc[32];
    tcg::mma_mainloop<X3>(R, 0, c1 - c0, A.mn != 0, B.mn != 0, warp, lane, acc);
    if (threadIdx.x == 0) TCC_TRACE(3);
    float* part = reinterpret_cast<float*>(sm.a_hi);
    tcg::consumer_sync();   // every warpgroup is done reading the A stages
    if (threadIdx.x == 64) TCC_TRACE(4);
    tcg::store_acc(acc, warp, lane, [&](int r, int c) {
      return part + r * kPitch + (c & ~31) + ((((c >> 2) & 7) ^ (r & 7)) << 2) + (c & 3);
    });
  }
  cluster_sync_all();
  if (threadIdx.x == 64) TCC_TRACE(7);
}

// sum of the CS partials at (row, lane + 32 g), g = 0..3, in fixed split order
template <int CS>
__device__ __forceinline__ void reduce_row(const Smem& sm, int row, int lane, float (&v)[4]) {
  const uint32_t local = smem_u32(reinterpret_cast<const float*>(sm.a_hi) + row * kPitch + ((((lane >> 2) ^ (row & 7))) << 2) +
                                  (lane & 3));
#pragma unroll
  for (int g = 0; g < 4; ++g) v[g] = 0.0f;
#pragma unroll
  for (int s = 0; s < CS; ++s) {
    const uint32_t base = map_to_rank(local, (uint32_t)s);
#pragma unroll
    for (int g = 0; g < 4; ++g) v[g] += ld_cluster(base + g * 32 * 4);
  }
}

__device__ __forceinline__ void common_setup(Smem& sm, int warp, int lane, bool pdl_wait = true) {
  if (warp == tcg::kProducerWarp && lane == 0) {
    for (int s = 0; s < tcg::kStages; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], tcg::kEpiWarps); }
    fence_barrier_init();
  }
  __syncthreads();
  // PDL (common.cuh): up to here only the host-uploaded descriptor table and shared memory were touched
  ppb_pdl_trigger();
  if (pdl_wait) ppb_pdl_wait();
}

// ---- generic flavours -------------------------------------------------------------------------------------------------
// grid = (sum of tiles) * CS, cluster (CS, 1, 1): blockIdx.x / CS = tile, %cluster_ctarank = K-split.
struct NoRowEpi {};   // RE of the epilogues 0 and 2
template <typename RE, int EPI> struct RowInOf { struct type {}; };
template <typename RE> struct RowInOf<RE, 3> { using type = typename RE::RowIn; };
template <bool X3, int CS, int EPI, typename RE = NoRowEpi>
__global__ void __launch_bounds__(tcg::kThreads, 1) k_cluster(const tcg::Problem* __restrict__ probs, int n_probs,
                                                                 unsigned long long* __restrict__ trace, const RE re) {
  if (threadIdx.x == 0) TCC_TRACE(0);
  extern __shared__ uint8_t smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x / CS;
  const int split = (int)cluster_ctarank();
  int lo_i = 0, hi_i = n_probs - 1;
  while (lo_i < hi_i) {
    int mid = (lo_i + hi_i + 1) >> 1;
    if (probs[mid].tile_start <= tile) lo_i = mid; else hi_i = mid - 1;
  }
  for (int i = threadIdx.x; i < (int)(sizeof(tcg::Problem) / 4); i += blockDim.x)
    reinterpret_cast<uint32_t*>(&sm.prob)[i] = reinterpret_cast<const uint32_t*>(probs + lo_i)[i];
  __syncthreads();
  const tcg::Problem& P = sm.prob;
  const int local = tile - P.tile_start;
  const int mt = local / P.tiles_n, nt = local % P.tiles_n;
  const int KC = (P.K + 31) / 32;
  const int c0 = (int)((int64_t)KC * split / CS), c1 = (int)((int64_t)KC * (split + 1) / CS);
  common_setup(sm, warp, lane);
  if (threadIdx.x == 0) TCC_TRACE(1);
  constexpr int kRowsPerCta = 128 / CS, kRowsPerWarp = kRowsPerCta / tcg::kEpiWarps;
  // epilogue 3: the inputs of the row routine that do not depend on the product are loaded while the operands stream in
  typename RowInOf<RE, EPI>::type rin[kRowsPerWarp];
  if constexpr (EPI == 3) {
    if (warp < tcg::kEpiWarps) {
#pragma unroll
      for (int rr = 0; rr < kRowsPerWarp; ++rr)   // every row of a tile exists (M is a multiple of 128)
        rin[rr] = re.load(P.o_row0 + mt * 128 + split * kRowsPerCta + warp * kRowsPerWarp + rr);
    }
  }
  mainloop_and_park<X3>(sm, P.a, P.b, mt, nt, c0, c1, warp, lane, trace);

  if constexpr (EPI == 3) {
    // the sums of all rows of the warp first (their remote loads overlap), then one row at a time through the buffer: the
    // B stages are idle once the mainloop is through, and the parked partials live in the A stages
    typename RE::State rs{};
    if (warp < tcg::kEpiWarps) {
      const int pM = P.M, pN = P.N;
      const int64_t orow0 = P.o_row0;
      float bias[4];
#pragma unroll
      for (int g = 0; g < 4; ++g) bias[g] = (P.bias && g * 32 + lane < pN) ? __ldg(P.bias + g * 32 + lane) : 0.0f;
      float r_x[kRowsPerWarp][4];
#pragma unroll
      for (int rr = 0; rr < kRowsPerWarp; ++rr) {
        float v[4];
        reduce_row<CS>(sm, split * kRowsPerCta + warp * kRowsPerWarp + rr, lane, v);
#pragma unroll
        for (int g = 0; g < 4; ++g) r_x[rr][g] = g * 32 + lane < pN ? v[g] + bias[g] : 0.0f;
      }
      float* const xrow = sm.b_hi[0] + warp * 128;
#pragma unroll
      for (int rr = 0; rr < kRowsPerWarp; ++rr) {
        const int m = mt * 128 + split * kRowsPerCta + warp * kRowsPerWarp + rr;
        if (m >= pM) continue;   // warp-uniform
#pragma unroll
        for (int g = 0; g < 4; ++g) xrow[g * 32 + lane] = r_x[rr][g];
        __syncwarp();
        re.row(rs, rin[rr], xrow, orow0 + m, lane);
        __syncwarp();
      }
    }
    re.finish(rs, lane);
  } else if constexpr (EPI == 4) {
    if (warp < tcg::kEpiWarps) {
      const int pM = P.M;
      const int64_t orow0 = P.o_row0;
      float r_v[kRowsPerWarp][4];
#pragma unroll
      for (int rr = 0; rr < kRowsPerWarp; ++rr) reduce_row<CS>(sm, split * kRowsPerCta + warp * kRowsPerWarp + rr, lane, r_v[rr]);
#pragma unroll
      for (int rr = 0; rr < kRowsPerWarp; ++rr) {
        const int m = mt * 128 + split * kRowsPerCta + warp * kRowsPerWarp + rr;
        if (m < pM) re.cells(orow0 + m, nt * 128 + lane, r_v[rr]);
      }
    }
  }
  if (EPI <= 2 && warp < tcg::kEpiWarps) {
    const int ew = warp;
    const bool do_relu = (P.flags & tcg::kRelu) != 0, do_mask = (P.flags & tcg::kMaskImg) != 0;
    const int m_valid = (P.flags & tcg::kZeroInvalid) ? P.m_valid : P.M;
    float bias[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const int n = nt * 128 + g * 32 + lane;
      bias[g] = (P.bias && n < P.N) ? __ldg(P.bias + n) : 0.0f;
    }
    // descriptor fields in registers: the explicit stores below are compiler barriers, every P.x after one is a reload
    const int pM = P.M, pN = P.N;
    const int64_t ldc = P.ldc, o_kb = P.o_kb, orow0 = P.o_row0, ocb0 = P.o_col0 / 32 + nt * 4;
    float* const c_p = P.c;
    float* const ok_hi = P.o_k_hi; float* const ok_lo = P.o_k_lo;
    float* const omn_hi = P.o_mn_hi; float* const omn_lo = P.o_mn_lo;
    const float* const mask_p = P.mask_hi;
    const int n_blocks = (pN - nt * 128 + 31) >> 5;     // 32-column blocks of this tile inside the (padded) width
    // pass 1 (no stores): partial sums from the peers' shared memory and the ReLU-mask words of all rows in flight together
    float r_x[kRowsPerWarp][4];
#pragma unroll
    for (int rr = 0; rr < kRowsPerWarp; ++rr) {
      const int row = split * kRowsPerCta + ew * kRowsPerWarp + rr;   // row of the tile
      const int m = mt * 128 + row;
      const bool live = m < pM;   // no per-row branch: the rows of a warp form one basic block, their loads overlap
      float v[4];
      reduce_row<CS>(sm, row, lane, v);
      const int64_t orow = orow0 + m;
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        const int n = nt * 128 + g * 32 + lane;
        float x = v[g] + bias[g];
        x = do_relu ? fmaxf(x, 0.0f) : x;
        x = (n < pN && m < m_valid) ? x : 0.0f;
        if (EPI == 2) {
          const int64_t span = ((orow >> 7) * o_kb + (ocb0 + g)) * kTileFloats + (orow & 127) * 32;
          const int64_t pos_k = span + ((((lane >> 2) ^ (int)(orow & 7))) << 2) + (lane & 3);
          const float mk = (do_mask && live && g < n_blocks) ? __ldg(mask_p + pos_k) : 1.0f;
          x = (mk > 0.0f) ? x : 0.0f;
        }
        r_x[rr][g] = x;
      }
    }
    if (threadIdx.x == 64) TCC_TRACE(14);
    // pass 2: stores
#pragma unroll
    for (int rr = 0; rr < kRowsPerWarp; ++rr) {
      const int row = split * kRowsPerCta + ew * kRowsPerWarp + rr;
      const int m = mt * 128 + row;
      if (m >= pM) continue;   // warp-uniform
      const int64_t orow = orow0 + m;
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        const int n = nt * 128 + g * 32 + lane;
        if (g >= n_blocks) continue;   // warp-uniform: column block beyond the (padded) width
        const float x = r_x[rr][g];
        if (c_p && n < pN) tcg::st_global(c_p + (int64_t)m * ldc + n, x);
        if (EPI == 2) {
          const int64_t span = ((orow >> 7) * o_kb + (ocb0 + g)) * kTileFloats + (orow & 127) * 32;
          const int64_t pos_k = span + ((((lane >> 2) ^ (int)(orow & 7))) << 2) + (lane & 3);
          float h, l;
          split_tf32(x, h, l);
          if (ok_hi) { tcg::st_global(ok_hi + pos_k, h); tcg::st_global(ok_lo + pos_k, l); }
          if (omn_hi) {
            const int64_t pos_mn = span + ((((lane >> 3) ^ (int)(orow & 3))) << 3) + (lane & 7);
            tcg::st_global(omn_hi + pos_mn, h);
            tcg::st_global(omn_lo + pos_mn, l);
          }
        }
      }
    }
  }
  if (threadIdx.x == 64) TCC_TRACE(5);
  cluster_sync_all();
  if (threadIdx.x == 0) TCC_TRACE(6);
  if (threadIdx.x == 0 && trace && blockIdx.x == 0) {
    const int dm[3] = {P.M, P.N, P.K};
    trace[13] = 1ull + CS * 16;
    trace[8] = (unsigned long long)dm[0]; trace[9] = (unsigned long long)dm[1]; trace[10] = (unsigned long long)dm[2];
    trace[11] = (unsigned long long)gridDim.x; trace[12] = (unsigned long long)(c1 - c0);
  }
}

// ---- LSTM time step: recurrent GEMM + cell in the reduce phase --------------------------------------------------------------
// Step list and CellIO as in tc_lstm.cuh (gate-interleaved W_hh: tile column g * 32 + j = gate g of unit nt * 32 + j).
// SMAX: compile-time bound of the sample-embedding width S (4 = pyprob's default sample_embedding_dim, 8 = the general case)
template <bool X3, int CS, int SMAX>
__global__ void __launch_bounds__(tcg::kThreads, 1) k_lstm_cluster(const tcl::Step* __restrict__ steps, int n_steps,
                                                                      unsigned long long* __restrict__ trace) {
  if (threadIdx.x == 0) TCC_TRACE(0);
  extern __shared__ uint8_t smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x / CS;
  const int split = (int)cluster_ctarank();
  int lo_i = 0, hi_i = n_steps - 1;
  while (lo_i < hi_i) {
    int mid = (lo_i + hi_i + 1) >> 1;
    if (steps[mid].tile_start <= tile) lo_i = mid; else hi_i = mid - 1;
  }
  for (int i = threadIdx.x; i < (int)(sizeof(tcl::Step) / 4); i += blockDim.x)
    reinterpret_cast<uint32_t*>(&sm.step)[i] = reinterpret_cast<const uint32_t*>(steps + lo_i)[i];
  __syncthreads();
  const tcl::Step& P = sm.step;
  const tcl::CellIO& io = P.io;
  const int local = tile - P.tile_start;
  const int mt = local / P.tiles_n, nt = local % P.tiles_n;   // nt = block of 32 hidden units
  const int KC = (io.H + 31) / 32;
  const int c0 = (int)((int64_t)KC * split / CS), c1 = (int)((int64_t)KC * (split + 1) / CS);
  common_setup(sm, warp, lane, false);
  if (threadIdx.x == 0) TCC_TRACE(1);
  // The W_hh tiles of the first stages do not depend on the previous time step (the images are packed once per training step,
  // before the chain of step kernels starts): the producer requests them BEFORE the PDL wait, so that only the h_{t-1} tiles
  // remain to be fetched once the previous step's kernel has finished.
  int b_pre = 0;
  if (warp == tcg::kProducerWarp && lane == 0) {
    const uint32_t bytes = (tcg::stage_bytes(P.a, mt) + tcg::stage_bytes(P.b, nt)) * (X3 ? 2u : 1u);
    b_pre = (c1 - c0) < tcg::kStages ? (c1 - c0) : tcg::kStages;
    for (int i = 0; i < b_pre; ++i) {
      mbar_expect_tx(&sm.full[i], bytes);
      tcg::load_operand(P.b, nt, c0 + i, sm.b_hi[i], sm.b_lo[i], X3, &sm.full[i]);
    }
  }
  ppb_pdl_wait();
  // Row metadata of this warp's rows (trace, step, previous row): it heads the dependency chain of the whole epilogue, so the
  // epilogue warps fetch it while the mainloop runs instead of after the cluster barrier.
  constexpr int kRowsPerCta = 128 / CS, kRowsPerWarp = kRowsPerCta / tcg::kEpiWarps;
  int m_tr[kRowsPerWarp], m_st[kRowsPerWarp], m_rp[kRowsPerWarp];
  if (warp < tcg::kEpiWarps) {
#pragma unroll
    for (int rr = 0; rr < kRowsPerWarp; ++rr) {
      const int64_t row = (int64_t)P.row0 + mt * 128 + split * kRowsPerCta + warp * kRowsPerWarp + rr;
      m_tr[rr] = __ldg(io.row_trace + row);
      m_st[rr] = __ldg(io.row_step + row);
      m_rp[rr] = (int)__ldg(io.row_prev + row);
    }
  }
  mainloop_and_park<X3>(sm, P.a, P.b, mt, nt, c0, c1, warp, lane, trace, b_pre);

  if (warp < tcg::kEpiWarps) {
    const int ew = warp;
    const int H = io.H, H4 = 4 * io.H, S = io.S;
    const int u = nt * 32 + lane;     // hidden unit of this lane
    float wsmp[4][SMAX];
#pragma unroll
    for (int g = 0; g < 4; ++g)
#pragma unroll
      for (int s = 0; s < SMAX; ++s) wsmp[g][s] = (s < S) ? __ldg(io.w_smp_t + (int64_t)s * H4 + g * H + u) : 0.0f;
    const int64_t hkb = io.hkb;
    // Two passes over the warp's rows.  Pass 1 holds no stores (and no compiler barrier), so the loads of all rows — partial
    // sums from the peers' shared memory, P_obs / P_step / c_{t-1} from L2 — are in flight together instead of one row's
    // latency chain after the other; pass 2 writes the results.
    // Pass 1 is ONE basic block (padding rows read row 0 of the segment and are zeroed afterwards — no per-row branch), with
    // the pointers of the descriptor in registers (P lives in shared memory behind a generic pointer: every io.x is a load).
    float r_act[kRowsPerWarp][4], r_c[kRowsPerWarp], r_h[kRowsPerWarp];
    {
      const float* const g_pobs = io.p_obs; const float* const g_pstep = io.p_step;
      const float* const g_c = io.c; const float* const g_smp = io.smp_emb;
      const int64_t seg_row0 = (int64_t)P.row0;
#pragma unroll
      for (int rr = 0; rr < kRowsPerWarp; ++rr) {
        const int trow = split * kRowsPerCta + ew * kRowsPerWarp + rr;
        const bool live = m_tr[rr] >= 0;
        const int64_t row = live ? seg_row0 + mt * 128 + trow : seg_row0;     // global row of the step (a valid one)
        const int tr = live ? m_tr[rr] : 0, st = live ? m_st[rr] : 0;
        const int64_t rp = (live && m_rp[rr] >= 0) ? (int64_t)m_rp[rr] : 0;
        float v[4];
        reduce_row<CS>(sm, trow, lane, v);
        float sm_e[SMAX];
#pragma unroll
        for (int s = 0; s < SMAX; ++s) sm_e[s] = (s < S) ? __ldg(g_smp + row * S + s) : 0.0f;
        const float cp = __ldcg(g_c + rp * H + u);
        float act[4];
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const int col = g * H + u;
          // same order of additions as k_cell_fwd: (P_obs + P_step) + recurrent, then the sample-embedding FMAs
          float x = __ldg(g_pobs + (int64_t)tr * H4 + col) + __ldg(g_pstep + (int64_t)st * H4 + col);
          x += v[g];
#pragma unroll
          for (int s = 0; s < SMAX; ++s)
            if (s < S) x = fmaf(sm_e[s], wsmp[g][s], x);
          act[g] = (g == 2) ? ppb_cell_tanh(x) : ppb_cell_sigmoid(x);
        }
        const float cn = act[1] * cp + act[0] * act[2];
        const float hn = act[3] * ppb_cell_tanh(cn);
#pragma unroll
        for (int g = 0; g < 4; ++g) r_act[rr][g] = live ? act[g] : 0.0f;
        r_c[rr] = live ? cn : 0.0f;
        r_h[rr] = live ? hn : 0.0f;
      }
    }
    if (threadIdx.x == 64) TCC_TRACE(14);
    {
      float* const g_gates = io.gates; float* const g_c = io.c; float* const g_h = io.h;
      float* const g_hk_hi = io.hk_hi; float* const g_hk_lo = io.hk_lo;
      float* const g_hmn_hi = io.hmn_hi; float* const g_hmn_lo = io.hmn_lo;
      const int64_t row_first = (int64_t)P.row0 + mt * 128 + split * kRowsPerCta + ew * kRowsPerWarp;
#pragma unroll
      for (int rr = 0; rr < kRowsPerWarp; ++rr) {
        const int64_t row = row_first + rr;
#pragma unroll
        for (int g = 0; g < 4; ++g) tcg::st_global(g_gates + row * H4 + g * H + u, r_act[rr][g]);
        tcg::st_global(g_c + row * H + u, r_c[rr]);
        tcg::st_global(g_h + row * H + u, r_h[rr]);
        const int64_t span = ((row >> 7) * hkb + nt) * kTileFloats + (row & 127) * 32;
        float hh, hl;
        split_tf32(r_h[rr], hh, hl);
        const int64_t pos_k = span + ((((lane >> 2) ^ (int)(row & 7))) << 2) + (lane & 3);
        tcg::st_global(g_hk_hi + pos_k, hh);
        tcg::st_global(g_hk_lo + pos_k, hl);
        const int64_t pos_mn = span + ((((lane >> 3) ^ (int)(row & 3))) << 3) + (lane & 7);
        tcg::st_global(g_hmn_hi + pos_mn, hh);
        tcg::st_global(g_hmn_lo + pos_mn, hl);
      }
    }
  }
  if (threadIdx.x == 64) TCC_TRACE(5);
  cluster_sync_all();
  if (threadIdx.x == 0) TCC_TRACE(6);
  if (threadIdx.x == 0 && trace && blockIdx.x == 0) {
    const int dm[3] = {P.M, 4 * io.H, io.H};
    trace[13] = 2ull + CS * 16;
    trace[8] = (unsigned long long)dm[0]; trace[9] = (unsigned long long)dm[1]; trace[10] = (unsigned long long)dm[2];
    trace[11] = (unsigned long long)gridDim.x; trace[12] = (unsigned long long)(c1 - c0);
  }
}

}  // namespace tcc
