// wgmma / mbarrier / bulk-TMA primitives for sm_90a (inline PTX; no CUTLASS dependency).
// Bit layouts follow the PTX ISA "wgmma" shared-memory matrix descriptor.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace tc {

// ---- packed operand image (tile image): K-major, SWIZZLE_128B ------------------------------------
// A matrix X[rows, K] is stored as tiles of 128 rows x 32 fp32 (one 128-byte swizzle span along K):
//   tile(rt, kb) at float offset (rt * KB + kb) * 4096, KB = ceil(K/32); row r of a tile is the 32-float span at r * 32
//   inside a span the eight 16-byte chunks sit at chunk position (c16 ^ (r & 7))  -> exactly the shared-memory image
//   wgmma expects, so a tile moves HBM -> SMEM with one linear cp.async.bulk (no tensor map needed).
// MN-major flavour of the same tile (for tensors whose reduction runs along the image ROWS): same spans, but the four
// 32-byte chunks of a span are permuted by (c32 ^ (r & 3)).  tf32 wgmma reads K-major operands only, so the GEMM kernels
// rewrite an MN-major stage into the K-major image in shared memory before the MMAs (tcg::stage_to_kmajor).
// Every writer of an image places its values through img_span + k_swz / mn_swz.
constexpr int kTileRows = 128;
constexpr int kTileK = 32;                       // fp32 elements per 128-byte swizzle span
constexpr int kTileFloats = kTileRows * kTileK;  // 4096 floats = 16 KB
constexpr int kTileBytes = kTileFloats * 4;

// floats of one image (one part: hi or lo, one flavour) of a [rows, cols] matrix, padded to whole tiles
__host__ __device__ __forceinline__ int64_t img_floats(int64_t rows, int64_t cols) {
  return ((rows + 127) / 128) * ((cols + 31) / 32) * kTileFloats;
}

// float offset of the 32-float span of row r (0..127) of row tile rt in column block cb
template <class R>
__host__ __device__ __forceinline__ int64_t img_span(int64_t rt, R r, int64_t cb, int64_t KB) {
  return (rt * KB + cb) * kTileFloats + r * 32;
}
// the same for image row `row`
__host__ __device__ __forceinline__ int64_t img_span(int64_t row, int64_t cb, int64_t KB) {
  return img_span(row >> 7, row & 127, cb, KB);
}

// position of column c (0..31) of a block inside the span of image row `row`, K-major / MN-major, plus `span` (the span's
// offset, when the caller passes it).  The chunk index is swizzled in the column's type and added to the span before the
// column's low bits, so that callers keep their index widths.
template <class R, class C, class S = C>
__host__ __device__ __forceinline__ S k_swz(R row, C c, S span = 0) {
  return span + (((c >> 2) ^ (C)(row & 7)) << 2) + (c & 3);
}
template <class R, class C, class S = C>
__host__ __device__ __forceinline__ S mn_swz(R row, C c, S span = 0) {
  return span + (((c >> 3) ^ (C)(row & 3)) << 3) + (c & 7);
}

__host__ __device__ __forceinline__ int64_t packed_offset(int64_t row, int64_t k, int64_t KB) {
  return k_swz(row, k & 31, img_span(row, k >> 5, KB));
}
__host__ __device__ __forceinline__ int64_t packed_offset_mn(int64_t row, int64_t k, int64_t KB) {
  return mn_swz(row, k & 31, img_span(row, k >> 5, KB));
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t addr = smem_u32(bar), done;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!done);
}

// ---- bulk TMA (linear): global -> shared, completion on an mbarrier ----------------------------------
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---- wgmma (sm_90a warpgroup MMA) --------------------------------------------------------------------
// Shared-memory matrix descriptor, K-major, SWIZZLE_128B, dense 8-row atoms (SBO = 1024 B; LBO unused for SW128 K-major).
// The swizzle is applied to absolute address bits, so a descriptor may start 32/64/96 B into a 1024-aligned atom row:
// that is how the four k8 steps of a 32-element chunk are addressed (+2 in the 16-byte start-address field per step).
__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);  // start address   bits [0,14)
  d |= (uint64_t)1 << 16;                        // leading byte offset (16 B >> 4), unused for SW128 K-major
  d |= (uint64_t)(1024 >> 4) << 32;              // stride byte offset: next 8-row atom
  d |= (uint64_t)1 << 62;                        // layout type SWIZZLE_128B
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x 64] += A[64 x 8] B[64 x 8]^T, tf32 operands K-major in shared memory, fp32 accumulators in registers.
// Fragment: thread (warp w of the warpgroup, lane l) holds d[4 i + j] = D(16 w + l / 4 + 8 (j >> 1), 8 i + 2 (l % 4) + (j & 1)).
__device__ __forceinline__ void wgmma_tf32_m64n64k8(float (&d)[32], uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, 1, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a_desc), "l"(b_desc)
      : "memory");
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "elect.sync _|P, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// round-to-nearest TF32 split: x = hi + lo (+ O(2^-22 |x|))
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  uint32_t h;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(x));
  hi = __uint_as_float(h);
  float rest = x - hi;
  uint32_t l;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"(rest));
  lo = __uint_as_float(l);
}

// Which images pack_tile stores: the K-major pair, both flavours, or each flavour whose hi pointer is set (checked at run time)
enum class Parts { k, both, present };

// Packs row tile rt of an image with kb column blocks, one 16-byte chunk per thread and iteration; the CTAs along blockIdx.y
// share the tile.  load(row, k0, x) fills x[0..3] with columns k0..k0+3 of image row `row` (zero outside the source).
template <Parts P, class Load>
__device__ __forceinline__ void pack_tile(int rt, int kb, float* k_hi, float* k_lo, float* mn_hi, float* mn_lo, Load load) {
  for (int q = threadIdx.x + blockIdx.y * blockDim.x; q < 128 * kb * 8; q += blockDim.x * gridDim.y) {
    const int c16 = q & 7, t = q >> 3;
    const int cb = t % kb, r = t / kb;  // consecutive threads walk along a row: coalesced reads
    float x[4], h[4], l[4];
    load(rt * 128 + r, cb * 32 + c16 * 4, x);
#pragma unroll
    for (int j = 0; j < 4; ++j) split_tf32(x[j], h[j], l[j]);
    const int64_t span = img_span((int64_t)rt, r, cb, kb);
    if (P != Parts::present || k_hi) {
      const int64_t o = k_swz(r, c16 * 4, span);
      *reinterpret_cast<float4*>(k_hi + o) = make_float4(h[0], h[1], h[2], h[3]);
      *reinterpret_cast<float4*>(k_lo + o) = make_float4(l[0], l[1], l[2], l[3]);
    }
    if (P == Parts::both || (P == Parts::present && mn_hi)) {
      const int64_t o = mn_swz(r, c16 * 4, span);
      *reinterpret_cast<float4*>(mn_hi + o) = make_float4(h[0], h[1], h[2], h[3]);
      *reinterpret_cast<float4*>(mn_lo + o) = make_float4(l[0], l[1], l[2], l[3]);
    }
  }
}

}  // namespace tc
