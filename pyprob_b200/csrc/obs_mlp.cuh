// Fused observation-embedding MLP (pyprob/nn/inference_network.py:132-139 + embedding_feedforward.py:35-48):
// per-observable Linear+ReLU chains -> concat -> final Linear+ReLU chain, all layers in ONE kernel per direction.
// Used in the small-batch regime where a GEMM launch per layer is latency-bound (each layer is a few MFLOP);
// wide / large-batch cases fall back to the grouped GEMM path.
//
// Both kernels work on a chunk of up to kMT traces at a time, with all 256 threads on one layer: thread = (output row,
// k-slice), 32 rows x 8 slices per pass, so a layer costs in_dim / 8 FMAs per trace plus a three-step shuffle reduction
// instead of an in_dim-long FMA chain.  Every weight matrix is staged once per CTA with 16-byte cp.async.  The forward grid
// spreads the traces over all SMs.  The backward kernel runs the input-gradient chain the same way and then reduces the
// weight / bias gradients over its traces in shared memory; the CTAs of a thread-block cluster combine their partial sums
// through distributed shared memory and each gradient entry gets one red.add per cluster.
#pragma once
#include "common.cuh"
#include "tc.cuh"
#include "tc_cluster.cuh"

namespace obsmlp {

constexpr int W2 = 96;          // widest activation on this path (obs_fused_ok)
constexpr int kThreads = 256;
constexpr int kSlices = 8;      // k-slices per output row (lanes of one 8-lane group)
constexpr int kRows = kThreads / kSlices;
constexpr int kMT = 4;          // traces per chunk (per-thread accumulators)
constexpr int kCluster = 8;     // backward: CTAs whose partial weight gradients meet in distributed shared memory
constexpr int kMaxLayers = PPB_MAX_OBS * PPB_MAX_FF_LAYERS + PPB_MAX_FF_LAYERS;
constexpr size_t kMaxSmem = 227 * 1024;

// One Linear+ReLU layer of the whole MLP (observable chains first, then the final chain), with the places its operands
// live: shared-memory offsets are in floats; "act" is a trace's vector of every layer input plus the embedding, "dz" its
// vector of every layer's d(pre-activation).
struct Layer {
  int in_dim, out_dim;
  int sw, pitch;          // staged weight rows (sw + n * pitch), bias at sw + out_dim * pitch
  int xoff, yoff;         // input / output in act
  int dzoff, dxoff;       // d(pre-activation) of the output / of the input in dz (dxoff < 0: the input is the observation)
  int part;               // first entry of this layer's W (then b) gradient in the partial-sum area
  int64_t w_off, b_off;
  float* y; int ldy;      // global copy of the output (read by the GEMM path's consumers and by the backward kernel)
  const float* x; int ldx;  // global input rows
};

struct Plan {
  int n_layers;
  int A, Dz;              // floats per trace of act / dz
  int w_floats, part_floats;
  int E;
  Layer L[kMaxLayers];
  // optional: tf32 tile images of obs_emb (tc.cuh), written by k_fwd itself so that no packing kernel sits between the
  // embedding and the P_obs GEMM on the critical path (only when B % 128 == 0 and E % 32 == 0: no padding to zero-fill)
  float* emb_k_hi; float* emb_k_lo; float* emb_mn_hi; float* emb_mn_lo;
  long long emb_kb;
  // optional (G > 0, LSTM network): k_bwd forms d obs_emb = d_pobs W_ih[:, :E] itself (form_d_emb) instead of reading it.
  // Rank r of a cluster reduces over gates [r G / kCluster, (r + 1) G / kCluster) in chunks of kg gates.
  int G, kg;
  int64_t wih_off, ld_wih; int wih_vec;   // W_ih row g at arena + wih_off + g * ld_wih; wih_vec: rows copied 16 bytes at a time
  const float* dp; int64_t ld_dp;         // d_pobs rows
  // non-null: dp holds batch rows (the T = 1 dgates), and trace tr's row is its sub-batch's first t = 0 row plus its place
  // in the sub-batch (whose first trace is row_trace of that row); null: dp holds one row per trace
  const int* trace_sub; const int* step_row0; const int* row_trace;
};

inline size_t smem_fwd(const Plan& p) { return (size_t)(p.w_floats + kMT * p.A) * sizeof(float); }
inline size_t smem_bwd(const Plan& p) { return (size_t)(p.w_floats + p.part_floats + kMT * (p.A + p.Dz)) * sizeof(float); }
// form_d_emb's buffers, from the end of the staged weights (over act / dz / part, which it runs before): a chunk of the
// W_ih[:, :E] slice (kg x emb_wp), the d_pobs chunk of the cluster's kCluster * kMT traces of a round (pitch kg + 4) and
// their partial sums (x emb_wp).  Overlaid rather than appended: the kernel is slower with the larger allocation.
constexpr int kRoundTraces = kCluster * kMT;
__host__ __device__ inline int emb_wp(int E) { return (E + 3) & ~3; }
inline size_t smem_emb(const Plan& p, int kg) {
  const int wp = emb_wp(p.E);
  return (size_t)(p.w_floats + kg * wp + kRoundTraces * (kg + 4) + kRoundTraces * wp) * sizeof(float);
}

__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src)
               : "memory");
}
__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gmem_src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src)
               : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// Issue the copies of one layer (the caller waits once for all layers).  Rows whose length is a multiple of four floats
// go as 16-byte copies into a pitch of 4 mod 8 floats, which keeps both the forward (lanes along k) and the backward
// (lanes along n) reads free of bank conflicts; other widths (the first layer of a scalar observable) are copied as they lie.
// Descriptor fields are read into registers before the loops (here and below): the copies' memory clobber and the stores
// would otherwise make the compiler fetch them from parameter memory again on every iteration.
__device__ __forceinline__ void stage_layer(float* smem, const float* __restrict__ arena, const Layer& L) {
  const int in_dim = L.in_dim, out_dim = L.out_dim, pitch = L.pitch;
  float* dst = smem + L.sw;
  const float* src = arena + L.w_off;
  const float* bsrc = arena + L.b_off;
  if ((in_dim & 3) == 0) {
    const int q = in_dim >> 2, nq = out_dim * q;
    for (int c = threadIdx.x; c < nq; c += kThreads) {
      const int n = c / q, k4 = c - n * q;
      cp_async16(dst + n * pitch + 4 * k4, src + 4 * c);
    }
  } else {
    const int nw = out_dim * in_dim;
    for (int c = threadIdx.x; c < nw; c += kThreads) cp_async4(dst + c, src + c);
  }
  float* bias = dst + out_dim * pitch;
  for (int n = threadIdx.x; n < out_dim; n += kThreads) cp_async4(bias + n, bsrc + n);
}
// rows [tr0, tr0 + nt) x [0, width) of a global matrix (ld floats) -> dst[t * pitch + k], as 4-byte asynchronous copies
__device__ __forceinline__ void load_rows(float* dst, int pitch, const float* src, int64_t ld, int tr0, int nt, int width) {
  for (int idx = threadIdx.x; idx < nt * width; idx += kThreads) {
    const int t = idx / width, k = idx - t * width;
    cp_async4(dst + t * pitch + k, src + (int64_t)(tr0 + t) * ld + k);
  }
}

// sum over the 8 lanes of a k-slice group (every lane ends with the total)
__device__ __forceinline__ float group_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v;
}
__device__ __forceinline__ float pick(const float (&a)[kMT], int i) {
  float r = a[0];
#pragma unroll
  for (int t = 1; t < kMT; ++t) r = i == t ? a[t] : r;
  return r;
}

// y[t][n] = relu(b[n] + sum_k x[t][k] W[n][k]) for the chunk's nt traces; lane s of a group stores trace s
__device__ __forceinline__ void layer_fwd(const Plan& P, const Layer& L, const float* smem, float* act, int tr0, int nt,
                                          bool last) {
  const int g = threadIdx.x / kSlices, s = threadIdx.x % kSlices;
  const int in_dim = L.in_dim, out_dim = L.out_dim, pitch = L.pitch, A = P.A, ldy = L.ldy;
  const float* w = smem + L.sw;
  const float* bias = w + out_dim * pitch;
  const float* xr = act + L.xoff;
  float* yr = act + L.yoff;
  float* y = L.y;
  float* ek_hi = last ? P.emb_k_hi : nullptr;
  float* ek_lo = P.emb_k_lo;
  float* em_hi = P.emb_mn_hi;
  float* em_lo = P.emb_mn_lo;
  const long long kb = P.emb_kb;
  // the bound is that of the warp's first group: every lane of a warp takes part in every shuffle
  for (int n = g; n - (g & 3) < out_dim; n += kRows) {
    float acc[kMT];
#pragma unroll
    for (int t = 0; t < kMT; ++t) acc[t] = 0.f;
    const float* wr = w + n * pitch;
    const int kend = n < out_dim ? in_dim : 0;
    for (int k = s; k < kend; k += kSlices) {
      const float wv = wr[k];
#pragma unroll
      for (int t = 0; t < kMT; ++t) acc[t] = fmaf(wv, xr[t * A + k], acc[t]);
    }
#pragma unroll
    for (int t = 0; t < kMT; ++t) acc[t] = group_sum(acc[t]);
    if (s < nt && n < out_dim) {
      const float v = fmaxf(pick(acc, s) + bias[n], 0.f);
      const int tr = tr0 + s;
      yr[s * A + n] = v;
      y[(int64_t)tr * ldy + n] = v;
      if (ek_hi) {
        float hi, lo;
        tc::split_tf32(v, hi, lo);
        const int64_t ok = tc::packed_offset(tr, n, kb);
        ek_hi[ok] = hi;
        if (ek_lo) ek_lo[ok] = lo;
        if (em_hi) {
          const int64_t om = tc::packed_offset_mn(tr, n, kb);
          em_hi[om] = hi;
          if (em_lo) em_lo[om] = lo;
        }
      }
    }
  }
}

// grid = ceil(B / traces_per_cta); every CTA walks its traces in chunks of kMT
__global__ void __launch_bounds__(kThreads) k_fwd(const __grid_constant__ Plan P, const float* __restrict__ arena, int B,
                                                  int traces_per_cta) {
  // Launched with PDL: its CTAs are placed while the predecessor drains, ahead of the side-stream kernels that start beside
  // it.  It waits before its first read AND before it lets its own dependents launch, so every later kernel of the step
  // starts after whatever ran before this one (the optimiser that wrote the weights) has finished: kernels further down the
  // chain may read the weights before their own wait (k_bwd does).
  ppb_pdl_wait();
  ppb_pdl_trigger();   // the P_obs GEMM that follows is launched with the PDL attribute: its prologue overlaps this kernel
  extern __shared__ __align__(16) float smem[];
  const int n_layers = P.n_layers, A = P.A;
  float* act = smem + P.w_floats;
  for (int i = 0; i < n_layers; ++i) stage_layer(smem, arena, P.L[i]);
  const int t_begin = blockIdx.x * traces_per_cta;
  const int t_end = min(B, t_begin + traces_per_cta);
  for (int c0 = t_begin; c0 < t_end; c0 += kMT) {
    const int nt = min(kMT, t_end - c0);
    for (int i = 0; i < n_layers; ++i) {   // observations: the inputs of the first layer of every chain
      const Layer& L = P.L[i];
      if (L.dxoff < 0) load_rows(act + L.xoff, A, L.x, L.ldx, c0, nt, L.in_dim);
    }
    cp_async_wait_all();
    __syncthreads();
    for (int i = 0; i < n_layers; ++i) {
      layer_fwd(P, P.L[i], smem, act, c0, nt, i == n_layers - 1);
      __syncthreads();
    }
  }
}

// dx[t][k] = (x[t][k] > 0) * sum_n dz[t][n] W[n][k]
__device__ __forceinline__ void layer_dx(const Plan& P, const Layer& L, const float* smem, const float* act, float* dz,
                                         int nt) {
  const int g = threadIdx.x / kSlices, s = threadIdx.x % kSlices;
  const int in_dim = L.in_dim, out_dim = L.out_dim, pitch = L.pitch, A = P.A, Dz = P.Dz;
  const float* w = smem + L.sw;
  const float* dr = dz + L.dzoff;
  const float* xr = act + L.xoff;
  float* dxr = dz + L.dxoff;
  for (int k = g; k - (g & 3) < in_dim; k += kRows) {   // warp-uniform bound, as in layer_fwd
    float acc[kMT];
#pragma unroll
    for (int t = 0; t < kMT; ++t) acc[t] = 0.f;
    const int nend = k < in_dim ? out_dim : 0;
    for (int n = s; n < nend; n += kSlices) {
      const float wv = w[n * pitch + k];
#pragma unroll
      for (int t = 0; t < kMT; ++t) acc[t] = fmaf(wv, dr[t * Dz + n], acc[t]);
    }
#pragma unroll
    for (int t = 0; t < kMT; ++t) acc[t] = group_sum(acc[t]);
    if (s < nt && k < in_dim) dxr[s * Dz + k] = xr[s * A + k] > 0.f ? pick(acc, s) : 0.f;
  }
}

// this chunk's share of dW[n][k] = sum_t dz[t][n] x[t][k] and db[n] = sum_t dz[t][n], added to part.  A thread takes four
// of its entries at a time and loads all their operands before the first read-modify-write of part: one entry after the
// other, every sum was a chain of dependent shared-memory loads, and eight warps per SM could not hide it.  Traces t >= nt
// enter as zeros (selected, not branched around), which keeps the sums those of the nt traces in the same order.
__device__ __forceinline__ void layer_partial(const Plan& P, const Layer& L, const float* act, const float* dz, float* part,
                                              int nt) {
  constexpr int kBatch = 4;
  const int in_dim = L.in_dim, out_dim = L.out_dim, A = P.A, Dz = P.Dz;
  const int nw = out_dim * in_dim;
  const float* dr = dz + L.dzoff;
  const float* xr = act + L.xoff;
  float* pr = part + L.part;
  const int dn = kThreads / in_dim, dk = kThreads - dn * in_dim;   // (n, k) of entry e + kThreads from those of e
  int n = threadIdx.x / in_dim, k = threadIdx.x - n * in_dim;
  for (int e = threadIdx.x; e < nw; e += kBatch * kThreads) {
    float v[kBatch];
#pragma unroll
    for (int j = 0; j < kBatch; ++j) {
      v[j] = 0.f;
      const bool in = e + j * kThreads < nw;
#pragma unroll
      for (int t = 0; t < kMT; ++t) {
        const bool on = in && t < nt;
        const float d = on ? dr[t * Dz + n] : 0.f, x = on ? xr[t * A + k] : 0.f;
        v[j] = fmaf(d, x, v[j]);
      }
      n += dn; k += dk;
      if (k >= in_dim) { k -= in_dim; ++n; }
    }
#pragma unroll
    for (int j = 0; j < kBatch; ++j)
      if (e + j * kThreads < nw) pr[e + j * kThreads] += v[j];
  }
  for (int o = threadIdx.x; o < out_dim; o += kThreads) {
    float v = 0.f;
#pragma unroll
    for (int t = 0; t < kMT; ++t) v += t < nt ? dr[t * Dz + o] : 0.f;
    pr[nw + o] += v;
  }
}

// rows [g0, g0 + kg) of W_ih[:, :E] -> wsl[g * emb_wp + e]
__device__ __forceinline__ void stage_wih(const Plan& P, const float* __restrict__ arena, float* wsl, int g0, int kg) {
  const int E = P.E, wp = emb_wp(E);
  const int64_t ld = P.ld_wih;
  const float* src = arena + P.wih_off + (int64_t)g0 * ld;
  if (P.wih_vec) {
    const int q = E >> 2;
    for (int c = threadIdx.x; c < kg * q; c += kThreads) {
      const int g = c / q, k4 = c - g * q;
      cp_async16(wsl + g * wp + 4 * k4, src + g * ld + 4 * k4);
    }
  } else {
    for (int c = threadIdx.x; c < kg * E; c += kThreads) {
      const int g = c / E, e = c - g * E;
      cp_async4(wsl + g * wp + e, src + g * ld + e);
    }
  }
}

// d_emb[tr] = d_pobs[tr] W_ih[:, :E] for the traces of this CTA, exact fp32.  Round c takes the c-th chunk of kMT traces of
// every rank of the cluster (kRoundTraces in all): each rank forms their partial sums over its gate slice, and the partials
// meet in distributed shared memory, where rank r adds those of its own kMT traces in rank order (deterministic, no
// atomics) and stores them to d_emb.  The first W_ih chunk is staged by the caller before the PDL wait.
__device__ __forceinline__ void form_d_emb(const Plan& P, const float* __restrict__ arena, float* buf, float* d_emb, int B,
                                           int traces_per_cta) {
  const int E = P.E, wp = emb_wp(E), KG = P.kg, dpp = KG + 4, gs = P.G / kCluster;
  float* wsl = buf;
  float* dps = wsl + KG * wp;
  float* pb = dps + kRoundTraces * dpp;
  const uint32_t rank = tcc::cluster_ctarank();
  const int cbase = (int)(blockIdx.x - rank) * traces_per_cta;   // first trace of the cluster
  const int g_first = (int)rank * gs;
  const int nch = (gs + KG - 1) / KG, rounds = (traces_per_cta + kMT - 1) / kMT;
  const int np = (E + 1) >> 1;                                   // (trace quad, column pair) work items: 8 * np <= 2 * kThreads
  const float* dp = P.dp;
  const int64_t ld_dp = P.ld_dp;
  const int* trace_sub = P.trace_sub; const int* step_row0 = P.step_row0; const int* row_trace = P.row_trace;
  const uint32_t pb_addr = (uint32_t)__cvta_generic_to_shared(pb);
  for (int c = 0; c < rounds; ++c) {
    float acc[2][kMT][2];
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int t = 0; t < kMT; ++t) acc[k][t][0] = acc[k][t][1] = 0.f;
    for (int ch = 0; ch < nch; ++ch) {
      const int g0 = ch * KG, kg = min(KG, gs - g0);
      if (c > 0 || ch > 0) {
        __syncthreads();   // every thread is through the previous chunk
        if (nch > 1) stage_wih(P, arena, wsl, g_first + g0, kg);
      }
      const int q4 = kg >> 2;
      for (int idx = threadIdx.x; idx < kRoundTraces * q4; idx += kThreads) {
        const int j = idx / q4, k4 = idx - j * q4;
        const int i = c * kMT + (j % kMT);
        const int tr = cbase + (j / kMT) * traces_per_cta + i;
        if (i >= traces_per_cta || tr >= B) continue;   // a slot without a trace: its sums are never stored
        int row = tr;
        if (trace_sub) {
          const int r0 = __ldg(step_row0 + __ldg(trace_sub + tr));
          row = r0 + tr - __ldg(row_trace + r0);
        }
        cp_async16(dps + j * dpp + 4 * k4, dp + (int64_t)row * ld_dp + g_first + g0 + 4 * k4);
      }
      cp_async_wait_all();
      __syncthreads();
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int it = threadIdx.x + k * kThreads;
        if (it >= kRoundTraces / kMT * np) continue;
        const int q = it / np, p = it - q * np;
        const float* dr = dps + q * kMT * dpp;
        const float* wr = wsl + 2 * p;
#pragma unroll 2
        for (int g = 0; g < kg; g += 4) {
          float d[kMT][4];
#pragma unroll
          for (int t = 0; t < kMT; ++t) {
            const float4 v = *reinterpret_cast<const float4*>(dr + t * dpp + g);
            d[t][0] = v.x; d[t][1] = v.y; d[t][2] = v.z; d[t][3] = v.w;
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const float2 w = *reinterpret_cast<const float2*>(wr + (g + u) * wp);
#pragma unroll
            for (int t = 0; t < kMT; ++t) {
              acc[k][t][0] = fmaf(d[t][u], w.x, acc[k][t][0]);
              acc[k][t][1] = fmaf(d[t][u], w.y, acc[k][t][1]);
            }
          }
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int it = threadIdx.x + k * kThreads;
      if (it >= kRoundTraces / kMT * np) continue;
      const int q = it / np, p = it - q * np;
#pragma unroll
      for (int t = 0; t < kMT; ++t) {
        pb[(q * kMT + t) * wp + 2 * p] = acc[k][t][0];
        pb[(q * kMT + t) * wp + 2 * p + 1] = acc[k][t][1];
      }
    }
    tcc::cluster_sync_all();
    for (int idx = threadIdx.x; idx < kMT * E; idx += kThreads) {
      const int t = idx / E, e = idx - t * E;
      const int i = c * kMT + t, tr = cbase + (int)rank * traces_per_cta + i;
      if (i >= traces_per_cta || tr >= B) continue;
      const uint32_t a = pb_addr + 4u * (uint32_t)(((int)rank * kMT + t) * wp + e);
      float v = 0.f;
#pragma unroll
      for (int r = 0; r < kCluster; ++r) v += tcc::ld_cluster(tcc::map_to_rank(a, (uint32_t)r));
      d_emb[(int64_t)tr * E + e] = v;
    }
    tcc::cluster_sync_all();   // the partial sums stay readable until every rank is through
  }
}

// d_emb holds d(loss)/d(obs_emb), or (P.G > 0) is written with it by form_d_emb.  grad += dW, db of every layer.  grid = a
// multiple of kCluster CTAs (some may own no trace: they still take part in the cluster reductions).
__global__ void __launch_bounds__(kThreads) k_bwd(const __grid_constant__ Plan P, const float* __restrict__ arena,
                                                  float* __restrict__ d_emb, float* __restrict__ grad, int B,
                                                  int traces_per_cta) {
  ppb_pdl_trigger();
  extern __shared__ __align__(16) float smem[];
  const int n_layers = P.n_layers, A = P.A, Dz = P.Dz, E = P.E, part_floats = P.part_floats;
  float* act = smem + P.w_floats;
  float* dz = act + kMT * A;
  float* part = dz + kMT * Dz;
  // Staged before the wait: the weights (arena), the first chunk of W_ih[:, :E] included.  Only the optimiser writes them,
  // and no kernel of a training step can start before the previous step's optimiser has finished: k_fwd waits before it
  // lets its dependents launch.  The first layer of a chain never propagates further down: it is not staged.
  for (int i = 0; i < n_layers; ++i)
    if (P.L[i].dxoff >= 0) stage_layer(smem, arena, P.L[i]);
  const bool form = P.G > 0;
  if (form) stage_wih(P, arena, act, (int)tcc::cluster_ctarank() * (P.G / kCluster), min(P.kg, P.G / kCluster));
  else for (int i = threadIdx.x; i < part_floats; i += kThreads) part[i] = 0.f;
  // Everything else after it: the forward activations and the embedding are written by k_fwd of this same step, which a
  // chain of programmatic edges does not order before this point (each kernel of the chain triggers before its own wait);
  // d_pobs by the kernel right before this one
  ppb_pdl_wait();
  if (form) {
    form_d_emb(P, arena, act, d_emb, B, traces_per_cta);   // its buffers overlay act, dz and part
    for (int i = threadIdx.x; i < part_floats; i += kThreads) part[i] = 0.f;
    __syncthreads();
  }
  const int t_begin = blockIdx.x * traces_per_cta;
  const int t_end = min(B, t_begin + traces_per_cta);
  const int zoff = P.L[n_layers - 1].dzoff, eoff = P.L[n_layers - 1].yoff;
  const float* emb = P.L[n_layers - 1].y;
  for (int c0 = t_begin; c0 < t_end; c0 += kMT) {
    const int nt = min(kMT, t_end - c0);
    for (int i = 0; i < n_layers; ++i) {   // every layer's input, and the embedding
      const Layer& L = P.L[i];
      load_rows(act + L.xoff, A, L.x, L.ldx, c0, nt, L.in_dim);
    }
    load_rows(act + eoff, A, emb, E, c0, nt, E);
    load_rows(dz + zoff, Dz, d_emb, E, c0, nt, E);
    cp_async_wait_all();
    __syncthreads();
    // d(pre-activation) of the last layer: the incoming gradient masked by the (post-ReLU) embedding
    for (int idx = threadIdx.x; idx < nt * E; idx += kThreads) {
      const int t = idx / E, k = idx - t * E;
      if (!(act[t * A + eoff + k] > 0.f)) dz[t * Dz + zoff + k] = 0.f;
    }
    __syncthreads();
    for (int i = n_layers - 1; i >= 0; --i) {
      if (P.L[i].dxoff < 0) continue;
      layer_dx(P, P.L[i], smem, act, dz, nt);
      __syncthreads();
    }
    for (int i = 0; i < n_layers; ++i) layer_partial(P, P.L[i], act, dz, part, nt);
    __syncthreads();
  }
  cp_async_wait_all();   // a CTA without traces still has its staging copies in flight: none may stay past the exit
  // cluster reduction: rank r sums entries r*256 + tid (stride kCluster*256) over the cluster and adds them to the arena
  tcc::cluster_sync_all();
  const uint32_t rank = tcc::cluster_ctarank();
  const uint32_t part_addr = (uint32_t)__cvta_generic_to_shared(part);
  int li = 0, lpart = P.L[0].part, lnext = n_layers > 1 ? P.L[1].part : part_floats, lnw = P.L[0].out_dim * P.L[0].in_dim;
  int64_t lw = P.L[0].w_off, lb = P.L[0].b_off;
  for (int e = rank * kThreads + threadIdx.x; e < part_floats; e += kCluster * kThreads) {
    float v = 0.f;
#pragma unroll
    for (int r = 0; r < kCluster; ++r) v += tcc::ld_cluster(tcc::map_to_rank(part_addr + 4u * (uint32_t)e, (uint32_t)r));
    while (e >= lnext) {
      ++li;
      const Layer& L = P.L[li];
      lpart = L.part; lnw = L.out_dim * L.in_dim; lw = L.w_off; lb = L.b_off;
      lnext = li + 1 < n_layers ? P.L[li + 1].part : part_floats;
    }
    const int le = e - lpart;
    if (v != 0.f) atomicAdd(grad + (le < lnw ? lw + le : lb + (le - lnw)), v);
  }
  tcc::cluster_sync_all();   // the partial sums stay readable until every rank is through
}

}  // namespace obsmlp
