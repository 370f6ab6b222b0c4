// Persistent form of the grouped wgmma GEMM (tc_grouped.cuh): one CTA per SM walks output tiles blockIdx.x, + gridDim.x, ...
//
// Why: with one tile per CTA every tile pays the prologue (barrier init, descriptor fetch, first operand latency) and an
// epilogue during which no operands are in flight.  Here the producer runs free of the consumers across tiles: it streams
// operand chunks of tile after tile into the stage ring (full/empty mbarriers, one running chunk counter), so the next tile's
// first stages are loaded while the consumer warps run the previous tile's epilogue out of a DEDICATED result tile.
// 128 KB of operand stages (2 x 64 KB in 3xTF32, 4 x 32 KB single-pass) + 66 KB result tile.
// Same Problem descriptors, same arithmetic and the same epilogue flavours as tcg::k_grouped; results are identical.
#pragma once
#include "tc_grouped.cuh"

namespace tcp {

using namespace tc;

// 128 KB of operand stages either way: 3xTF32 moves 64 KB per 32-element chunk (A/B x hi/lo) -> 2 stages; single-pass TF32
// moves 32 KB -> 4 stages (with two, a CTA kept ~58 GB/s of loads in flight and the mainloop waited on latency)
template <bool X3> struct StageCfg { static constexpr int kStages = X3 ? 2 : 4; static constexpr int kFloats = (X3 ? 4 : 2) * kTileFloats; };

constexpr int kMaxStages = 4;
struct __align__(1024) Smem {
  float ring[8 * kTileFloats];            // 128 KB: stage s at s * kFloats: [a_hi | b_hi | a_lo | b_lo] (lo parts: 3xTF32 only)
  float ctile[tcg::kCFloats];
  uint64_t full[kMaxStages];
  uint64_t empty[kMaxStages];
};
inline size_t smem_bytes() { return sizeof(Smem) + 1024; }

// index of the problem that owns `tile` (tile_start is ascending)
__device__ __forceinline__ int find_problem(const tcg::Problem* __restrict__ probs, int n_probs, int tile) {
  int lo = 0, hi = n_probs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (probs[mid].tile_start <= tile) lo = mid; else hi = mid - 1;
  }
  return lo;
}

struct TileGeom { int mt, nt, c0, c1; };
__device__ __forceinline__ TileGeom tile_geom(const tcg::Problem& P, int tile) {
  const int local = tile - P.tile_start;
  const int tiles_mn = P.tiles_m * P.tiles_n;
  const int split = local / tiles_mn, rem = local % tiles_mn;
  const int KC = (P.K + 31) / 32;
  const int nsplit = P.k_splits > 1 ? P.k_splits : 1;
  TileGeom g;
  g.mt = rem / P.tiles_n; g.nt = rem % P.tiles_n;
  g.c0 = (int)((int64_t)KC * split / nsplit); g.c1 = (int)((int64_t)KC * (split + 1) / nsplit);
  return g;
}

template <bool X3, int EPI>
__global__ void __launch_bounds__(tcg::kThreads, 1) k_grouped_persistent(const tcg::Problem* __restrict__ probs, int n_probs,
                                                                          int total_tiles) {
  extern __shared__ uint8_t smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kStages = StageCfg<X3>::kStages, kStageFloats = StageCfg<X3>::kFloats;
  const tcg::Ring R{sm.ring, sm.ring + 2 * kTileFloats, sm.ring + kTileFloats, sm.ring + 3 * kTileFloats, kStageFloats, kStages,
                    sm.full, sm.empty};   // lo parts: 3xTF32 only
  if (warp == tcg::kProducerWarp && lane == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], tcg::kEpiWarps); }
    fence_barrier_init();
  }
  __syncthreads();
  ppb_pdl_trigger();
  ppb_pdl_wait();

  if (warp == tcg::kProducerWarp) {
    if (lane == 0) {
      uint32_t kc = 0;   // chunks issued so far (all tiles)
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const tcg::Problem& P = probs[find_problem(probs, n_probs, tile)];
        const TileGeom g = tile_geom(P, tile);
        tcg::produce<X3>(R, P.a, P.b, g.mt, g.nt, g.c0, g.c1 - g.c0, kc);
        kc += (uint32_t)(g.c1 - g.c0);
      }
    }
  } else {
    const int q = warp & 3;                 // 32-row block of the tile
    const int cb = warp >> 2;               // 32-column chunk of the tile
    const float* stg = sm.ctile + (q * 32) * tcg::kCPitch + cb * 32;
    uint32_t kc = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      int pi = 0;
      if (lane == 0) pi = find_problem(probs, n_probs, tile);
      pi = __shfl_sync(0xffffffffu, pi, 0);
      const tcg::Problem& P = probs[pi];
      const TileGeom g = tile_geom(P, tile);
      float acc[32];
      tcg::mma_mainloop<X3>(R, kc, g.c1 - g.c0, P.a.mn != 0, P.b.mn != 0, warp, lane, acc);
      kc += (uint32_t)(g.c1 - g.c0);
      tcg::consumer_sync();   // the previous tile's epilogue is done with the result tile
      tcg::store_acc(acc, warp, lane, [&](int r, int c) { return sm.ctile + r * tcg::kCPitch + c; });
      tcg::consumer_sync();
      const int pM = P.M, pN = P.N, flags = P.flags;
      const int m_base = g.mt * 128 + q * 32;
      const bool do_relu = (flags & tcg::kRelu) != 0, do_mask = (flags & tcg::kMaskImg) != 0;
      const int rows = (pM - m_base) < 32 ? (pM - m_base) : 32;
      const int valid_rows = (flags & tcg::kZeroInvalid) ? (P.m_valid - m_base) : 32;
      const float* bias_p = P.bias;
      const float* mask_p = P.mask_hi;
      float* c_p = P.c;
      float* ok_hi = P.o_k_hi; float* ok_lo = P.o_k_lo; float* omn_hi = P.o_mn_hi; float* omn_lo = P.o_mn_lo;
      const int64_t ldc = P.ldc, o_kb = P.o_kb, orow0 = (int64_t)P.o_row0 + m_base, ocb0 = P.o_col0 / 32 + g.nt * 4;
      const int n0 = g.nt * tcg::kBN + cb * 32;
      const bool work = n0 < ((pN + 31) & ~31) && m_base < pM;   // warp-uniform
      if (!work) continue;
      const int n = n0 + lane;
      const bool col_ok = n < pN;
      const float bias = (bias_p && col_ok) ? __ldg(bias_p + n) : 0.0f;
      const int64_t span0 = img_span(orow0, ocb0 + cb, o_kb);
      float* cp = c_p ? c_p + (int64_t)m_base * ldc + n : nullptr;
      const bool c_ok = cp != nullptr && col_ok;
#pragma unroll
      for (int rb = 0; rb < 32; rb += 8) {
        float mk[8];
        if (EPI == 2) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int r = rb + j;
            const int64_t pos_k = k_swz(r, lane, span0 + r * 32);
            mk[j] = 1.0f;
            if (do_mask && r < rows) asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(mk[j]) : "l"(mask_p + pos_k));
          }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int r = rb + j;
          float x = stg[r * tcg::kCPitch + lane] + bias;
          x = do_relu ? fmaxf(x, 0.0f) : x;
          const bool live = r < rows;
          x = (col_ok && r < valid_rows) ? x : 0.0f;
          if (EPI == 0) {
            if (live && c_ok) tcg::st_global(cp + (int64_t)r * ldc, x);
          } else if (EPI == 1) {
            if (live && c_ok && x != 0.0f) tcg::red_add_global(cp + (int64_t)r * ldc, x);
          } else {
            const int64_t pos_k = k_swz(r, lane, span0 + r * 32);
            if (do_mask && live) x = (mk[j] > 0.0f) ? x : 0.0f;
            if (live && c_ok) tcg::st_global(cp + (int64_t)r * ldc, x);
            float h, l;
            split_tf32(x, h, l);
            if (live && ok_hi) { tcg::st_global(ok_hi + pos_k, h); tcg::st_global(ok_lo + pos_k, l); }
            if (live && omn_hi) {
              const int64_t pos_mn = mn_swz(r, lane, span0 + r * 32);
              tcg::st_global(omn_hi + pos_mn, h);
              tcg::st_global(omn_lo + pos_mn, l);
            }
          }
        }
      }
    }
  }
  __syncthreads();
}

}  // namespace tcp
