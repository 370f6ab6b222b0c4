// Grouped fp32 SIMT GEMM: one launch runs a list of heterogeneous problems
//   C[gm(m), n] (op)= act( sum_k A(gm(m), ka(k)) * B(n, kb(k)) + bias[n] )
// with arbitrary strides (so NT / NN / TN forms share one kernel), optional row gather on M and
// independent gathers on K for A and B.  Exact-fp32 cross-check path and the workhorse for the small
// / ragged GEMMs of the proposal network; the large GEMMs run on wgmma (tc_*.cuh).
#pragma once
#include "common.cuh"

namespace gemm {

enum : int {
  kRelu = 1,        // apply max(x,0)
  kAccumulate = 2,  // C += result (exclusive owner; no atomics)
  kMaskAux = 4,     // result = aux(gm(m), n) > 0 ? result : 0      (ReLU backward)
  kScale = 8,       // result *= alpha
};

struct Problem {
  const float* A;
  const float* B;
  float* C;
  const float* bias;   // [N] or null
  const float* aux;    // mask source, same indexing as C (ld_aux)
  const int* m_gather; // logical row -> physical row (A rows, C rows, aux rows) or null
  const int* ka_gather;  // k -> physical k index for A, or null
  const int* kb_gather;  // k -> physical k index for B, or null
  int64_t sam, sak;    // A(m,k) = A[m*sam + k*sak]
  int64_t sbn, sbk;    // B(n,k) = B[n*sbn + k*sbk]
  int64_t ldc, ld_aux;
  int M, N, K;
  int flags;
  float alpha;
  int tile_start;      // first global tile index of this problem
  int tiles_m, tiles_n;
  int pad_;
};

constexpr int BM = 64, BN = 64, BK = 16, kThreads = 256;

__global__ void __launch_bounds__(kThreads) k_grouped(const Problem* __restrict__ probs, int n_probs, int total_tiles) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  __shared__ Problem sP;  // the descriptor is read hundreds of times per tile: keep it on chip
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    // binary search the owning problem
    int lo = 0, hi = n_probs - 1;
    while (lo < hi) {
      int mid = (lo + hi + 1) >> 1;
      if (probs[mid].tile_start <= tile) lo = mid; else hi = mid - 1;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < (int)(sizeof(Problem) / 4); i += blockDim.x)
      reinterpret_cast<uint32_t*>(&sP)[i] = reinterpret_cast<const uint32_t*>(probs + lo)[i];
    __syncthreads();
    const Problem& P = sP;
    const int local = tile - P.tile_start;
    const int tm = local / P.tiles_n, tn = local % P.tiles_n;
    const int m0 = tm * BM, n0 = tn * BN;
    const int tid = threadIdx.x;
    const int ty = tid / 16, tx = tid % 16;  // 16x16 threads, 4x4 outputs each

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;

    // loader mapping: make the unit-stride dimension the fastest-varying one
    const bool a_k_fast = (P.sak == 1) || (P.ka_gather == nullptr && P.sak < P.sam);
    const bool b_k_fast = (P.sbk == 1) || (P.kb_gather == nullptr && P.sbk < P.sbn);

    // register-staged software pipeline: the global loads of chunk k+1 are in flight while chunk k is multiplied
    float ra[4], rb[4];
    auto fetch = [&](int k0) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        int e = tid + i * kThreads;  // 0..1023
        int mm, kk;
        if (a_k_fast) { kk = e % BK; mm = e / BK; } else { mm = e % BM; kk = e / BM; }
        int m = m0 + mm, k = k0 + kk;
        float v = 0.0f;
        if (m < P.M && k < P.K) {
          int64_t pm = P.m_gather ? P.m_gather[m] : m;
          int64_t pk = P.ka_gather ? P.ka_gather[k] : k;
          v = __ldg(P.A + pm * P.sam + pk * P.sak);
        }
        ra[i] = v;
        int nn;
        if (b_k_fast) { kk = e % BK; nn = e / BK; } else { nn = e % BN; kk = e / BN; }
        int n = n0 + nn;
        k = k0 + kk;
        v = 0.0f;
        if (n < P.N && k < P.K) {
          int64_t pk = P.kb_gather ? P.kb_gather[k] : k;
          v = __ldg(P.B + (int64_t)n * P.sbn + pk * P.sbk);
        }
        rb[i] = v;
      }
    };
    fetch(0);
    for (int k0 = 0; k0 < P.K; k0 += BK) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        int e = tid + i * kThreads;
        int mm, kk, nn;
        if (a_k_fast) { kk = e % BK; mm = e / BK; } else { mm = e % BM; kk = e / BM; }
        As[kk][mm] = ra[i];
        if (b_k_fast) { kk = e % BK; nn = e / BK; } else { nn = e % BN; kk = e / BN; }
        Bs[kk][nn] = rb[i];
      }
      __syncthreads();
      if (k0 + BK < P.K) fetch(k0 + BK);
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
        float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
        float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
      __syncthreads();
    }

#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int m = m0 + ty * 4 + i;
      if (m >= P.M) continue;
      int64_t pm = P.m_gather ? P.m_gather[m] : m;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int n = n0 + tx * 4 + j;
        if (n >= P.N) continue;
        float v = acc[i][j];
        if (P.bias) v += __ldg(P.bias + n);
        if (P.flags & kScale) v *= P.alpha;
        if (P.flags & kRelu) v = fmaxf(v, 0.0f);
        if (P.flags & kMaskAux) v = (P.aux[pm * P.ld_aux + n] > 0.0f) ? v : 0.0f;
        float* c = P.C + pm * P.ldc + n;
        if (P.flags & kAccumulate) v += *c;
        *c = v;
      }
    }
  }
}

}  // namespace gemm
