// Grouped wgmma GEMM over packed tile images (the tensor-core workhorse of the proposal network).
//
//   C[m, n] (op)= epi( sum_k A(m, k) * B(n, k) )      fp32-faithful 3xTF32 or single-pass TF32
//
// Every operand is a tile image (tc.cuh): 128-row x 32-column tiles, tf32 hi / lo parts.  An operand is read
//   * K-major  when the reduction runs along the image COLUMNS (image rows = M or N index)        [fmt K]
//   * MN-major when the reduction runs along the image ROWS    (image columns = M or N index)      [fmt MN]
// so forward GEMMs, input-gradient GEMMs and weight-gradient GEMMs all read the same row-major tensors
// without transposed copies (a tensor that is read both ways keeps one image per format).
// One pipeline stage = 32 reduction elements: a 16 KB tile (K-major) or 4 x 4 KB row pieces (MN-major, rewritten into
// the K-major image in shared memory before the MMAs).
// Warp roles (544 threads): warps 0-15 = four warpgroups, each issuing the wgmma of one 64 x 64 quadrant and then running
// the epilogue of a 32 x 32 block; warp 16 bulk-TMA producer.  One 128 x 128 output tile per CTA.
#pragma once
#include "common.cuh"
#include "tc.cuh"

namespace tcg {

using namespace tc;

// explicit global-space accesses: pointers fetched from the on-chip descriptor are generic to the compiler
__device__ __forceinline__ void st_global(float* p, float v) { asm volatile("st.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory"); }
__device__ __forceinline__ void red_add_global(float* p, float v) { asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory"); }
__device__ __forceinline__ float ld_global(const float* p) { float v; asm volatile("ld.global.f32 %0, [%1];" : "=f"(v) : "l"(p)); return v; }

enum : int {
  kRelu = 1,        // max(x, 0)
  kMaskImg = 4,     // result = mask_img(m, n) > 0 ? result : 0   (mask image: K-format hi part, output geometry)
  kZeroInvalid = 8, // rows m >= m_valid produce zeros (padding rows of a segment)
};
// Epilogue 1 always adds into C (red.add), so the caller zero-initialises C or accumulates into it.
// Split-K: when k_splits > 1 the reduction is divided over k_splits CTAs per output tile and the fp32 result is combined
// that way (epilogue 1 only; no images, bias, ReLU, mask or zero-invalid rows).

struct Operand {
  const float* hi;
  const float* lo;
  const int* k_rows;  // MN-major: image row origin of each 32-row reduction chunk (null: row0 + 32 c)
                      // K-major, read only by the chunk-table instantiation (KTAB): pairs (first M/N row [mult of
                      // 128], column block) of each 32-column reduction chunk — a reduction over column ranges of
                      // different row blocks of one image (null: row0, col0 / 32 + c)
  int kb;             // column blocks of the image
  int mn;             // 0 = K-major, 1 = MN-major
  int row0, col0;     // K-major: (first M/N row [mult of 128], first reduction col [mult of 32])
                      // MN-major: (first reduction row [mult of 32], first M/N col [mult of 32])
};

struct Problem {
  Operand a, b;
  int M, N, K;        // logical dims (K = reduction length)
  int m_valid;        // rows >= m_valid are padding (kZeroInvalid)
  int flags;
  float* c;           // fp32 output or null
  int64_t ldc;
  const float* bias;  // [N] or null
  float* o_k_hi; float* o_k_lo;    // K-format output image (or null)
  float* o_mn_hi; float* o_mn_lo;  // MN-format output image (or null)
  const float* mask_hi;            // K-format image with the geometry of the output
  int o_kb;           // column blocks of the output / mask images
  int o_row0, o_col0; // origin of C(0,0) inside the output images (mult of 128 / 32)
  int tile_start, tiles_m, tiles_n;
  int k_splits;
};

constexpr int kStages = 3;
constexpr int kEpiWarps = 16;                     // = the MMA warps: four warpgroups, one 64 x 64 quadrant of the tile each
constexpr int kProducerWarp = kEpiWarps;          // bulk-TMA producer
constexpr int kThreads = 32 * (kEpiWarps + 1);
constexpr int kConsumerThreads = 32 * kEpiWarps;
constexpr int kBN = 128;
constexpr int kPiece = 32 * 128;  // bytes: 32 rows x 128 B
constexpr int kCPitch = 129;      // fp32 result tile in shared memory: row r at float r * 129 (row and column reads conflict-free)
constexpr int kCFloats = 128 * kCPitch;

struct __align__(1024) Smem {
  float a_hi[kStages][kTileFloats];
  float a_lo[kStages][kTileFloats];
  float b_hi[kStages][kTileFloats];
  float b_lo[kStages][kTileFloats];
  uint64_t full[kStages];
  uint64_t empty[kStages];
  Problem prob;  // on-chip copy of the descriptor
};
// The result tile is parked in the B stages, which are idle once the last MMA has completed.
static_assert(kCFloats * 4 <= 2 * kStages * kTileBytes, "result tile must fit in the B stages");

__device__ __forceinline__ uint32_t stage_bytes(const Operand& o, int tile_idx) {
  if (!o.mn) return kTileBytes;
  int n = 0;
  for (int j = 0; j < 4; ++j) n += (o.col0 / 32 + tile_idx * 4 + j < o.kb);
  return (uint32_t)n * kPiece;
}

template <bool KTAB = false>
__device__ __forceinline__ void load_operand(const Operand& o, int tile_idx, int chunk, float* s_hi, float* s_lo,
                                             bool x3, uint64_t* bar) {
  if (!o.mn) {
    int64_t rt = o.row0 / 128 + tile_idx, cb = o.col0 / 32 + chunk;
    if (KTAB && o.k_rows) { rt = o.k_rows[2 * chunk] / 128 + tile_idx; cb = o.k_rows[2 * chunk + 1]; }
    int64_t off = (rt * o.kb + cb) * kTileFloats;
    bulk_g2s(s_hi, o.hi + off, kTileBytes, bar);
    if (x3) bulk_g2s(s_lo, o.lo + off, kTileBytes, bar);
  } else {
    int r0 = o.k_rows ? o.k_rows[chunk] : o.row0 + 32 * chunk;
    int64_t rt = r0 >> 7, sub = (r0 & 127) >> 3;
    for (int j = 0; j < 4; ++j) {
      int cb = o.col0 / 32 + tile_idx * 4 + j;
      if (cb < o.kb) {
        int64_t off = (rt * o.kb + cb) * kTileFloats + sub * 256;
        bulk_g2s(s_hi + j * (kPiece / 4), o.hi + off, kPiece, bar);
        if (x3) bulk_g2s(s_lo + j * (kPiece / 4), o.lo + off, kPiece, bar);
      }
    }
  }
}

// named barrier of the 16 MMA / epilogue warps (ids 1-4 are the LSTM epilogue's quadrant barriers)
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 5, %0;" ::"n"(kConsumerThreads) : "memory"); }

// An MN-major stage (four pieces of 32 reduction rows x 32 M/N columns, chunks permuted by (c32 ^ (k & 3))) is rewritten in
// place into the K-major SWIZZLE_128B image of its 128 M/N rows, which is what tf32 wgmma reads.  Consecutive threads walk
// along M/N, so the reads are conflict-free and the writes 4-way.
__device__ __forceinline__ void stage_to_kmajor(float* const (&t)[4], int n, int tid) {
  float v[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (i < n)
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int idx = tid + kConsumerThreads * e, r = idx & 127, k = idx >> 7;
        v[i][e] = t[i][(r >> 5) * 1024 + k * 32 + ((((r & 31) >> 3) ^ (k & 3)) << 3) + (r & 7)];
      }
  consumer_sync();
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (i < n)
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int idx = tid + kConsumerThreads * e, r = idx & 127, k = idx >> 7;
        t[i][r * 32 + (((k >> 2) ^ (r & 7)) << 2) + (k & 3)] = v[i][e];
      }
  fence_proxy_async();   // generic-proxy writes, read next by wgmma (async proxy)
  consumer_sync();
}

// Operand stage ring: stage s of operand X at X + s * stride.
struct Ring {
  float* a_hi; float* a_lo; float* b_hi; float* b_lo;
  int stride, stages;
  uint64_t* full; uint64_t* empty;
};

// Mainloop of the 16 consumer warps over n chunks (ring positions kc0 .. kc0 + n - 1) of one 128 x 128 output tile.
// Warpgroup g computes the quadrant rows 64 (g & 1), columns 64 (g >> 1) into acc (fragment layout of
// wgmma_tf32_m64n64k8).  Each 32-element chunk is accumulated by the tensor core into a zeroed register tile and then added
// to acc in fp32 with round-to-nearest, so the tensor core's truncating accumulation only ever spans 4 (TF32) or 12
// (3xTF32: cross terms first, then hi * hi) products of one chunk.  The empty barrier of a stage expects one arrival per
// consumer warp.
template <bool X3>
__device__ __forceinline__ void mma_mainloop(const Ring& R, uint32_t kc0, int n, bool amn, bool bmn, int warp, int lane,
                                             float (&acc)[32]) {
  const int tid = warp * 32 + lane;
  const uint32_t a_off = (uint32_t)((warp >> 2) & 1) * 8192u, b_off = (uint32_t)(warp >> 3) * 8192u;
#pragma unroll
  for (int j = 0; j < 32; ++j) acc[j] = 0.0f;
  for (int i = 0; i < n; ++i) {
    const uint32_t kc = kc0 + (uint32_t)i;
    const int s = (int)(kc % (uint32_t)R.stages);
    const uint32_t ph = (kc / (uint32_t)R.stages) & 1;
    float* const ah_p = R.a_hi + s * R.stride; float* const al_p = R.a_lo + s * R.stride;
    float* const bh_p = R.b_hi + s * R.stride; float* const bl_p = R.b_lo + s * R.stride;
    mbar_wait(&R.full[s], ph);
    if (amn || bmn) {
      float* t[4] = {nullptr, nullptr, nullptr, nullptr};
      int nt = 0;
      if (amn) { t[nt++] = ah_p; if (X3) t[nt++] = al_p; }
      if (bmn) { t[nt++] = bh_p; if (X3) t[nt++] = bl_p; }
      stage_to_kmajor(t, nt, tid);
    }
    float d[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) d[j] = 0.0f;
    const uint64_t ah = smem_desc_sw128(smem_u32(ah_p) + a_off), bh = smem_desc_sw128(smem_u32(bh_p) + b_off);
    const uint64_t al = smem_desc_sw128(smem_u32(al_p) + a_off), bl = smem_desc_sw128(smem_u32(bl_p) + b_off);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      if (X3) {
        wgmma_tf32_m64n64k8(d, al + 2 * ks, bh + 2 * ks);
        wgmma_tf32_m64n64k8(d, ah + 2 * ks, bl + 2 * ks);
      }
      wgmma_tf32_m64n64k8(d, ah + 2 * ks, bh + 2 * ks);
    }
    wgmma_commit();
    wgmma_wait0();
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] += d[j];
    __syncwarp();
    if (lane == 0) mbar_arrive(&R.empty[s]);
  }
}

// Write the accumulator fragment of this thread to at(row, col) of the 128 x 128 tile.
template <class At>
__device__ __forceinline__ void store_acc(const float (&acc)[32], int warp, int lane, At at) {
  const int r0 = ((warp >> 2) & 1) * 64 + (warp & 3) * 16 + (lane >> 2), c0 = (warp >> 3) * 64 + 2 * (lane & 3);
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) *at(r0 + 8 * (j >> 1), c0 + 8 * i + (j & 1)) = acc[4 * i + j];
}

// Bulk-TMA producer: streams n chunks (c0 .. c0 + n - 1, ring positions kc0 ..) of tile (mt, nt) into the ring.
template <bool X3, bool KTAB = false>
__device__ __forceinline__ void produce(const Ring& R, const Operand& A, const Operand& B, int mt, int nt, int c0, int n,
                                        uint32_t kc0) {
  const uint32_t bytes = (stage_bytes(A, mt) + stage_bytes(B, nt)) * (X3 ? 2u : 1u);
  for (int i = 0; i < n; ++i) {
    const uint32_t kc = kc0 + (uint32_t)i;
    const int s = (int)(kc % (uint32_t)R.stages);
    const uint32_t ph = (kc / (uint32_t)R.stages) & 1;
    mbar_wait(&R.empty[s], ph ^ 1);
    mbar_expect_tx(&R.full[s], bytes);
    load_operand<KTAB>(A, mt, c0 + i, R.a_hi + s * R.stride, R.a_lo + s * R.stride, X3, &R.full[s]);
    load_operand(B, nt, c0 + i, R.b_hi + s * R.stride, R.b_lo + s * R.stride, X3, &R.full[s]);
  }
}

__device__ __forceinline__ Ring ring_of(Smem& sm) {
  return Ring{sm.a_hi[0], sm.a_lo[0], sm.b_hi[0], sm.b_lo[0], kTileFloats, kStages, sm.full, sm.empty};
}

// EPI selects the (compile-time) epilogue flavour so that the row loop is straight-line code:
//   0 = fp32 store (+bias, relu)   1 = fp32 reduction (red.add: weight gradients, split-K)   2 = tile images (+fp32)
// KTAB: the A operand may be K-major with a chunk table (Operand::k_rows); a separate instantiation, so that the other
// kernels keep their loader unchanged.
template <bool X3, int EPI, bool KTAB = false>
__global__ void __launch_bounds__(kThreads, 1) k_grouped(const Problem* __restrict__ probs, int n_probs,
                                                          unsigned long long* __restrict__ trace) {
#define TCG_TRACE(slot)                                                                                   \
  do {                                                                                                    \
    if (trace && blockIdx.x == 0) {                                                                       \
      unsigned long long _t;                                                                              \
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(_t));                                              \
      trace[slot] = _t;                                                                                   \
    }                                                                                                     \
  } while (0)
  if (threadIdx.x == 0) TCG_TRACE(0);
  extern __shared__ uint8_t smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x;
  int lo_i = 0, hi_i = n_probs - 1;
  while (lo_i < hi_i) {
    int mid = (lo_i + hi_i + 1) >> 1;
    if (probs[mid].tile_start <= tile) lo_i = mid; else hi_i = mid - 1;
  }
  for (int i = threadIdx.x; i < (int)(sizeof(Problem) / 4); i += blockDim.x)
    reinterpret_cast<uint32_t*>(&sm.prob)[i] = reinterpret_cast<const uint32_t*>(probs + lo_i)[i];
  __syncthreads();
  const Problem& P = sm.prob;
  const int local = tile - P.tile_start;
  const int tiles_mn = P.tiles_m * P.tiles_n;
  const int split = local / tiles_mn, rem = local % tiles_mn;
  const int mt = rem / P.tiles_n, nt = rem % P.tiles_n;
  const int KC = (P.K + 31) / 32;
  const int nsplit = P.k_splits > 1 ? P.k_splits : 1;
  const int c0 = (int)((int64_t)KC * split / nsplit), c1 = (int)((int64_t)KC * (split + 1) / nsplit);

  if (warp == kProducerWarp && lane == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], kEpiWarps); }
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) TCG_TRACE(1);
  // PDL (common.cuh): everything above touched only the host-uploaded descriptor table and shared memory
  ppb_pdl_trigger();
  ppb_pdl_wait();
  const Ring R = ring_of(sm);

  if (warp == kProducerWarp) {
    if (lane == 0) produce<X3, KTAB>(R, P.a, P.b, mt, nt, c0, c1 - c0, 0);
  } else {
    float acc[32];
    mma_mainloop<X3>(R, 0, c1 - c0, P.a.mn != 0, P.b.mn != 0, warp, lane, acc);
    if (threadIdx.x == 0) TCG_TRACE(3);
    float* const ctile = sm.b_hi[0];
    consumer_sync();   // every warpgroup is done reading the B stages
    store_acc(acc, warp, lane, [&](int r, int c) { return ctile + r * kCPitch + c; });
    consumer_sync();
    if (threadIdx.x == 0) TCG_TRACE(4);
    // Epilogue: warp (q, cb) owns rows 32q..32q+31, columns 32cb..32cb+31 of the tile and emits whole 128-byte row spans
    // (lane = column).
    const int q = warp & 3;
    const int cb = warp >> 2;
    const float* stg = ctile + (q * 32) * kCPitch + cb * 32;
    const int m_base = mt * 128 + q * 32;  // first row of C handled by this warp
    // hoist everything that does not depend on the row out of the (fully unrolled) row loop
    const bool do_relu = (P.flags & kRelu) != 0, do_mask = (P.flags & kMaskImg) != 0;
    const int rows = (P.M - m_base) < 32 ? (P.M - m_base) : 32;
    const int valid_rows = (P.flags & kZeroInvalid) ? (P.m_valid - m_base) : 32;
    const float* bias_p = P.bias;
    const float* mask_p = P.mask_hi;
    float* c_p = P.c;
    float* ok_hi = P.o_k_hi; float* ok_lo = P.o_k_lo; float* omn_hi = P.o_mn_hi; float* omn_lo = P.o_mn_lo;
    const int64_t ldc = P.ldc, o_kb = P.o_kb, orow0 = (int64_t)P.o_row0 + m_base, ocb0 = P.o_col0 / 32 + nt * 4;
    {
      const int n0 = nt * kBN + cb * 32;
      if (n0 < ((P.N + 31) & ~31) && m_base < P.M) {  // warp-uniform
      const int n = n0 + lane;
      const bool col_ok = n < P.N;
      const float bias = (bias_p && col_ok) ? __ldg(bias_p + n) : 0.0f;
      // the warp's 32 rows sit inside one 128-row image tile (m_base % 32 == 0, o_row0 % 128 == 0): row r of the block is
      // image row (orow0 + r), so (orow & 7) == (r & 7) and the span offset advances by 32 floats per row
      const int64_t span0 = img_span(orow0, ocb0 + cb, o_kb);
      float* cp = c_p ? c_p + (int64_t)m_base * ldc + n : nullptr;
      const bool c_ok = cp != nullptr && col_ok;
      // rows in batches of eight: the ReLU-mask loads of a batch are issued together (one L2 round trip per batch instead of
      // one per row)
#pragma unroll
      for (int rb = 0; rb < 32; rb += 8) {
        float mk[8];
        if (EPI == 2) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int r = rb + j;
            const int64_t pos_k = k_swz(r, lane, span0 + r * 32);
            // explicit loads into distinct registers, issued back to back (the compiler folded the predicated __ldg's into
            // one register and serialised them)
            mk[j] = 1.0f;
            if (do_mask && r < rows) asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(mk[j]) : "l"(mask_p + pos_k));
          }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int r = rb + j;
          float x = stg[r * kCPitch + lane] + bias;
          x = do_relu ? fmaxf(x, 0.0f) : x;
          const bool live = r < rows;                        // row exists in C
          x = (col_ok && r < valid_rows) ? x : 0.0f;
          if (EPI == 0) {
            if (live && c_ok) st_global(cp + (int64_t)r * ldc, x);
          } else if (EPI == 1) {
            if (live && c_ok && x != 0.0f) red_add_global(cp + (int64_t)r * ldc, x);
          } else {
            const int64_t pos_k = k_swz(r, lane, span0 + r * 32);
            if (do_mask && live) x = (mk[j] > 0.0f) ? x : 0.0f;
            if (live && c_ok) st_global(cp + (int64_t)r * ldc, x);
            float h, l;
            split_tf32(x, h, l);
            if (live && ok_hi) { st_global(ok_hi + pos_k, h); st_global(ok_lo + pos_k, l); }
            if (live && omn_hi) {
              const int64_t pos_mn = mn_swz(r, lane, span0 + r * 32);
              st_global(omn_hi + pos_mn, h);
              st_global(omn_lo + pos_mn, l);
            }
          }
        }
      }
      }
    }
  }
  if (threadIdx.x == 0) TCG_TRACE(5);
  __syncthreads();
  if (threadIdx.x == 0) TCG_TRACE(6);
  if (threadIdx.x == 0 && trace && blockIdx.x == 0) { trace[8] = (unsigned long long)P.M; trace[9] = (unsigned long long)P.N; trace[10] = (unsigned long long)P.K; trace[11] = (unsigned long long)gridDim.x; trace[12] = (unsigned long long)(c1 - c0); }
}

inline size_t smem_bytes() { return sizeof(Smem) + 1024; }

// image element writers for element-wise kernels (one value at logical (row, col) of an image with KB blocks)
__device__ __forceinline__ void img_store(float* k_hi, float* k_lo, float* mn_hi, float* mn_lo, int64_t row,
                                          int64_t col, int64_t KB, float x) {
  float h, l;
  split_tf32(x, h, l);
  if (k_hi) {
    int64_t o = packed_offset(row, col, KB);
    k_hi[o] = h;
    if (k_lo) k_lo[o] = l;
  }
  if (mn_hi) {
    int64_t o = packed_offset_mn(row, col, KB);
    mn_hi[o] = h;
    if (mn_lo) mn_lo[o] = l;
  }
}

}  // namespace tcg
