// Fused observation-embedding MLP (pyprob/nn/inference_network.py:132-139 + embedding_feedforward.py:35-48):
// per-observable Linear+ReLU chains -> concat -> final Linear+ReLU chain, all layers in ONE kernel per direction.
// Used in the small-batch regime where a GEMM launch per layer is latency-bound (each layer is a few MFLOP);
// wide / large-batch cases fall back to the grouped GEMM path.
#pragma once
#include "common.cuh"
#include "tc.cuh"

namespace obsmlp {

constexpr int TB = 4;        // traces per CTA: the chain is latency-bound, so favour CTAs in flight (64 at B=256)
constexpr int WMAX = 256;    // widest activation handled on chip
constexpr int LD = WMAX + 1;
constexpr int NC = 64;       // output columns per staged weight chunk
constexpr int kThreads = 256;

struct Bufs {  // global activation buffers (forward writes, backward reads) — same layout as the GEMM path
  float* obs_act[PPB_MAX_OBS][PPB_MAX_FF_LAYERS];
  float* obs_cat;
  float* fin_act[PPB_MAX_FF_LAYERS];
  float* obs_emb;
  // optional: tf32 tile images of obs_emb (tc.cuh), written by k_fwd2 itself so that no packing kernel sits between the
  // embedding and the P_obs GEMM on the critical path (only when B % 128 == 0 and E % 32 == 0: no padding to zero-fill)
  float* emb_k_hi = nullptr; float* emb_k_lo = nullptr; float* emb_mn_hi = nullptr; float* emb_mn_lo = nullptr;
  long long emb_kb = 0;
};

struct Net {
  int num_obs, obs_in_total, E;
  ppb_ff_desc obs_ff[PPB_MAX_OBS];
  ppb_ff_desc obs_final;
};

inline size_t smem_bytes() { return (size_t)(3 * TB * LD + WMAX * (NC + 1)) * sizeof(float); }

// out_s[r][n] = relu(b[n] + sum_k in_s[r][k] W[n][k]) for the CTA's TB rows; also streamed to global (ldg)
__device__ __forceinline__ void dense_fwd(const float (*in_s)[LD], int in_dim, const float* __restrict__ W,
                                          const float* __restrict__ b, int out_dim, float (*out_s)[LD], int out_col0,
                                          float* ws, float* gout, int64_t ldg, int gcol0, int r0, int B) {
  const int tid = threadIdx.x;
  for (int n0 = 0; n0 < out_dim; n0 += NC) {
    const int nc = out_dim - n0 < NC ? out_dim - n0 : NC;
    for (int idx = tid; idx < nc * in_dim; idx += kThreads) {  // k fastest: coalesced read of W rows
      int nn = idx / in_dim, k = idx - nn * in_dim;
      ws[k * (NC + 1) + nn] = __ldg(W + (int64_t)(n0 + nn) * in_dim + k);
    }
    __syncthreads();
    for (int o = tid; o < TB * NC; o += kThreads) {
      int r = o / NC, nn = o % NC;
      if (nn < nc) {
        float acc = __ldg(b + n0 + nn);
#pragma unroll 4
        for (int k = 0; k < in_dim; ++k) acc = fmaf(in_s[r][k], ws[k * (NC + 1) + nn], acc);
        acc = fmaxf(acc, 0.0f);
        out_s[r][out_col0 + n0 + nn] = acc;
        if (r0 + r < B) gout[(int64_t)(r0 + r) * ldg + gcol0 + n0 + nn] = acc;
      }
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kThreads) k_fwd(Net net, const float* __restrict__ arena, const float* __restrict__ obs,
                                                   int B, Bufs bufs) {
  extern __shared__ float smem[];
  float (*cat)[LD] = reinterpret_cast<float (*)[LD]>(smem);
  float (*pa)[LD] = reinterpret_cast<float (*)[LD]>(smem + TB * LD);
  float (*pb)[LD] = reinterpret_cast<float (*)[LD]>(smem + 2 * TB * LD);
  float* ws = smem + 3 * TB * LD;
  const int r0 = blockIdx.x * TB, tid = threadIdx.x;
  int in_off = 0, out_off = 0;
  for (int j = 0; j < net.num_obs; ++j) {
    const ppb_ff_desc& ff = net.obs_ff[j];
    for (int idx = tid; idx < TB * ff.in_dim; idx += kThreads) {
      int r = idx / ff.in_dim, k = idx % ff.in_dim;
      pa[r][k] = (r0 + r < B) ? __ldg(obs + (int64_t)(r0 + r) * net.obs_in_total + in_off + k) : 0.0f;
    }
    __syncthreads();
    float (*cur)[LD] = pa;
    float (*nxt)[LD] = pb;
    for (int l = 0; l < ff.num_layers; ++l) {
      const ppb_linear_desc& L = ff.layers[l];
      const bool last = l == ff.num_layers - 1;
      if (last) dense_fwd(cur, L.in_dim, arena + L.w_off, arena + L.b_off, L.out_dim, cat, out_off, ws, bufs.obs_cat, net.E, out_off, r0, B);
      else dense_fwd(cur, L.in_dim, arena + L.w_off, arena + L.b_off, L.out_dim, nxt, 0, ws, bufs.obs_act[j][l], L.out_dim, 0, r0, B);
      float (*t)[LD] = cur; cur = nxt; nxt = t;
    }
    in_off += ff.in_dim;
    out_off += ff.out_dim;
  }
  float (*cur)[LD] = cat;
  float (*nxt)[LD] = pa;
  for (int l = 0; l < net.obs_final.num_layers; ++l) {
    const ppb_linear_desc& L = net.obs_final.layers[l];
    const bool last = l == net.obs_final.num_layers - 1;
    dense_fwd(cur, L.in_dim, arena + L.w_off, arena + L.b_off, L.out_dim, nxt, 0, ws, last ? bufs.obs_emb : bufs.fin_act[l],
              L.out_dim, 0, r0, B);
    cur = nxt;
    nxt = (nxt == pa) ? pb : pa;
  }
}

// One layer of the backward chain for the CTA's TB rows.
//   dy_s : d(loss)/d(pre-activation) of this layer  [TB][out]      (already ReLU-masked)
//   x    : the layer's input rows (global, ld)       -> staged in x_s [TB][in]
//   dW += dy^T x, db += colsum(dy) (atomics), dx_s[r][k] = (x[r][k] > 0) * sum_n dy[r][n] W[n][k]  (if want_dx)
__device__ __forceinline__ void dense_bwd(const float (*dy_s)[LD], int dy_col0, int out_dim, const float* __restrict__ x,
                                          int64_t ldx, int xcol0, int in_dim, const float* __restrict__ W,
                                          float* __restrict__ dW, float* __restrict__ db, float (*x_s)[LD],
                                          float (*dx_s)[LD], bool want_dx, int r0, int B) {
  const int tid = threadIdx.x;
  for (int idx = tid; idx < TB * in_dim; idx += kThreads) {
    int r = idx / in_dim, k = idx % in_dim;
    x_s[r][k] = (r0 + r < B) ? __ldg(x + (int64_t)(r0 + r) * ldx + xcol0 + k) : 0.0f;
  }
  __syncthreads();
  for (int idx = tid; idx < out_dim * in_dim; idx += kThreads) {  // weight gradient: one atomic per (n, k) per CTA
    int n = idx / in_dim, k = idx - n * in_dim;
    float s = 0.0f;
#pragma unroll
    for (int r = 0; r < TB; ++r) s = fmaf(dy_s[r][dy_col0 + n], x_s[r][k], s);
    if (s != 0.0f) atomicAdd(dW + idx, s);
  }
  for (int n = tid; n < out_dim; n += kThreads) {
    float s = 0.0f;
#pragma unroll
    for (int r = 0; r < TB; ++r) s += dy_s[r][dy_col0 + n];
    if (s != 0.0f) atomicAdd(db + n, s);
  }
  if (want_dx) {
    for (int idx = tid; idx < TB * in_dim; idx += kThreads) {  // lanes along k: coalesced reads of W rows
      int r = idx / in_dim, k = idx - r * in_dim;
      float s = 0.0f;
      for (int n = 0; n < out_dim; ++n) s = fmaf(dy_s[r][dy_col0 + n], __ldg(W + (int64_t)n * in_dim + k), s);
      dx_s[r][k] = x_s[r][k] > 0.0f ? s : 0.0f;
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads) k_bwd(Net net, const float* __restrict__ arena, float* __restrict__ grad,
                                                   const float* __restrict__ obs, const float* __restrict__ d_obs_emb,
                                                   int B, Bufs bufs) {
  extern __shared__ float smem[];
  float (*da)[LD] = reinterpret_cast<float (*)[LD]>(smem);
  float (*dbuf)[LD] = reinterpret_cast<float (*)[LD]>(smem + TB * LD);
  float (*xs)[LD] = reinterpret_cast<float (*)[LD]>(smem + 2 * TB * LD);
  const int r0 = blockIdx.x * TB, tid = threadIdx.x, E = net.E;
  // gradient w.r.t. the pre-activation of the last final layer: mask by its (post-ReLU) output
  for (int idx = tid; idx < TB * E; idx += kThreads) {
    int r = idx / E, k = idx % E;
    float g = 0.0f;
    if (r0 + r < B) {
      int64_t o = (int64_t)(r0 + r) * E + k;
      g = bufs.obs_emb[o] > 0.0f ? d_obs_emb[o] : 0.0f;
    }
    da[r][k] = g;
  }
  __syncthreads();
  float (*cur)[LD] = da;
  float (*nxt)[LD] = dbuf;
  for (int l = net.obs_final.num_layers - 1; l >= 0; --l) {
    const ppb_linear_desc& L = net.obs_final.layers[l];
    const float* x = l == 0 ? bufs.obs_cat : bufs.fin_act[l - 1];
    dense_bwd(cur, 0, L.out_dim, x, L.in_dim, 0, L.in_dim, arena + L.w_off, grad + L.w_off, grad + L.b_off, xs, nxt, true, r0, B);
    float (*t)[LD] = cur; cur = nxt; nxt = t;
  }
  // cur now holds d(obs_cat pre-activations) [TB][E]; keep it and walk every observable's chain
  float (*dcat)[LD] = cur;
  float (*tmp)[LD] = nxt;
  // a third scratch is needed for ping-pong inside a chain: reuse xs' neighbour region is not available, so chains
  // alternate between `tmp` and the tail of the shared allocation
  float (*tmp2)[LD] = reinterpret_cast<float (*)[LD]>(smem + 3 * TB * LD);
  int in_off = 0, out_off = 0;
  for (int j = 0; j < net.num_obs; ++j) {
    const ppb_ff_desc& ff = net.obs_ff[j];
    const float (*dy)[LD] = dcat;
    int dy_col0 = out_off;
    float (*o1)[LD] = tmp;
    float (*o2)[LD] = tmp2;
    for (int l = ff.num_layers - 1; l >= 0; --l) {
      const ppb_linear_desc& L = ff.layers[l];
      const float* x = l == 0 ? obs : bufs.obs_act[j][l - 1];
      int64_t ldx = l == 0 ? net.obs_in_total : ff.layers[l - 1].out_dim;
      int xcol0 = l == 0 ? in_off : 0;
      dense_bwd(dy, dy_col0, L.out_dim, x, ldx, xcol0, L.in_dim, arena + L.w_off, grad + L.w_off, grad + L.b_off, xs, o1,
                l > 0, r0, B);
      dy = o1; dy_col0 = 0;
      float (*t)[LD] = o1; o1 = o2; o2 = t;
    }
    in_off += ff.in_dim;
    out_off += ff.out_dim;
  }
}

inline size_t smem_bytes_bwd() { return (size_t)(4 * TB * LD) * sizeof(float); }

// =====================================================================================================================
// Warp-per-trace variant (default for narrow layers).  The kernels above synchronise the whole CTA twice per layer and
// pay one global atomic per weight per 4-trace CTA in the backward pass.  Here every weight matrix is staged ONCE per CTA in shared memory, each warp walks the
// whole layer chain of its traces with warp-level synchronisation only, and the weight gradients are a separate,
// atomic-free reduction over traces (k_dw): dW[n][k] = sum_b dy[b][n] x[b][k].
// =====================================================================================================================
constexpr int W2 = 96;          // widest activation on this path (obs_fused_ok)
constexpr int TPW = 1;          // traces per warp per pass
constexpr int kWarps = 8;

struct DBufs {  // d(loss)/d(pre-activation) of every layer's output, stored for the weight-gradient reduction
  float* d_obs_act[PPB_MAX_OBS][PPB_MAX_FF_LAYERS];
  float* d_obs_cat;
  float* d_fin_act[PPB_MAX_FF_LAYERS];
  float* d_obs_emb;   // masked in place
};

__host__ __device__ inline int layer_floats(const ppb_linear_desc& L) { return L.out_dim * (L.in_dim | 1) + L.out_dim; }
__host__ __device__ inline int weights_floats(const Net& net) {
  int n = 0;
  for (int j = 0; j < net.num_obs; ++j)
    for (int l = 0; l < net.obs_ff[j].num_layers; ++l) n += layer_floats(net.obs_ff[j].layers[l]);
  for (int l = 0; l < net.obs_final.num_layers; ++l) n += layer_floats(net.obs_final.layers[l]);
  return n;
}
inline size_t smem_bytes2(const Net& net) { return (size_t)(weights_floats(net) + kWarps * 3 * W2) * sizeof(float); }

__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gmem_src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src)
               : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
}
// Stage one layer with asynchronous 4-byte copies (all of a CTA's copies are in flight at once; the caller waits once):
// row n of W at pitch (in_dim | 1) floats — odd, so "lane = output row" (forward) and "lane = input column" (backward)
// both read conflict-free — followed by the bias.
__device__ __forceinline__ float* stage_layer(float* dst, const float* __restrict__ arena, const ppb_linear_desc& L) {
  const int pitch = L.in_dim | 1, nw = L.out_dim * L.in_dim;
  for (int idx = threadIdx.x; idx < nw; idx += blockDim.x) {
    int n = idx / L.in_dim, k = idx - n * L.in_dim;
    cp_async4(dst + n * pitch + k, arena + L.w_off + idx);
  }
  float* bias = dst + L.out_dim * pitch;
  for (int n = threadIdx.x; n < L.out_dim; n += blockDim.x) cp_async4(bias + n, arena + L.b_off + n);
  return bias + L.out_dim;
}

// out[n] = relu(b[n] + sum_k in[k] W[n][k]); lanes own outputs n, n + 32, n + 64
__device__ __forceinline__ void warp_dense_fwd(const float* in, int in_dim, const float* w, int out_dim, float* out,
                                               int out_col0, float* gout, int lane) {
  const int pitch = in_dim | 1;
  const float* bias = w + out_dim * pitch;
  const bool p0 = lane < out_dim, p1 = lane + 32 < out_dim, p2 = lane + 64 < out_dim;
  const float* r0 = w + (p0 ? lane : 0) * pitch;
  const float* r1 = w + (p1 ? lane + 32 : 0) * pitch;
  const float* r2 = w + (p2 ? lane + 64 : 0) * pitch;
  float a0 = p0 ? bias[lane] : 0.f, a1 = p1 ? bias[lane + 32] : 0.f, a2 = p2 ? bias[lane + 64] : 0.f;
  if (out_dim <= 32) {
#pragma unroll 4
    for (int k = 0; k < in_dim; ++k) a0 = fmaf(in[k], r0[k], a0);
  } else if (out_dim <= 64) {
#pragma unroll 4
    for (int k = 0; k < in_dim; ++k) { const float x = in[k]; a0 = fmaf(x, r0[k], a0); a1 = fmaf(x, r1[k], a1); }
  } else {
#pragma unroll 4
    for (int k = 0; k < in_dim; ++k) { const float x = in[k]; a0 = fmaf(x, r0[k], a0); a1 = fmaf(x, r1[k], a1); a2 = fmaf(x, r2[k], a2); }
  }
  a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); a2 = fmaxf(a2, 0.f);
  if (p0) { out[out_col0 + lane] = a0; gout[lane] = a0; }
  if (p1) { out[out_col0 + lane + 32] = a1; gout[lane + 32] = a1; }
  if (p2) { out[out_col0 + lane + 64] = a2; gout[lane + 64] = a2; }
  __syncwarp();
}

__global__ void __launch_bounds__(kWarps * 32) k_fwd2(Net net, const float* __restrict__ arena,
                                                      const float* __restrict__ obs, int B, int traces_per_cta, Bufs bufs) {
  ppb_pdl_trigger();   // the P_obs GEMM that follows is launched with the PDL attribute: its prologue overlaps this kernel
  extern __shared__ float smem[];
  // stage every layer once per CTA
  float* p = smem;
  const float* w_obs[PPB_MAX_OBS][PPB_MAX_FF_LAYERS];
  const float* w_fin[PPB_MAX_FF_LAYERS];
  for (int j = 0; j < net.num_obs; ++j)
    for (int l = 0; l < net.obs_ff[j].num_layers; ++l) { w_obs[j][l] = p; p = stage_layer(p, arena, net.obs_ff[j].layers[l]); }
  for (int l = 0; l < net.obs_final.num_layers; ++l) { w_fin[l] = p; p = stage_layer(p, arena, net.obs_final.layers[l]); }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* cat = p + warp * 3 * W2;   // per warp: the concatenated per-observable outputs + two ping-pong vectors
  float* va = cat + W2;
  float* vb = va + W2;
  cp_async_wait_all();
  __syncthreads();
  const int t0 = blockIdx.x * traces_per_cta;
  for (int tr = t0 + warp; tr < t0 + traces_per_cta && tr < B; tr += kWarps) {
    int in_off = 0, out_off = 0;
    for (int j = 0; j < net.num_obs; ++j) {
      const ppb_ff_desc& ff = net.obs_ff[j];
      float* cur = va;
      float* nxt = vb;
      for (int k = lane; k < ff.in_dim; k += 32) cur[k] = __ldg(obs + (int64_t)tr * net.obs_in_total + in_off + k);
      __syncwarp();
      for (int l = 0; l < ff.num_layers; ++l) {
        const ppb_linear_desc& L = ff.layers[l];
        const bool last = l == ff.num_layers - 1;
        if (last) warp_dense_fwd(cur, L.in_dim, w_obs[j][l], L.out_dim, cat, out_off, bufs.obs_cat + (int64_t)tr * net.E + out_off, lane);
        else warp_dense_fwd(cur, L.in_dim, w_obs[j][l], L.out_dim, nxt, 0, bufs.obs_act[j][l] + (int64_t)tr * L.out_dim, lane);
        float* t = cur; cur = nxt; nxt = t;
      }
      in_off += ff.in_dim;
      out_off += ff.out_dim;
    }
    float* cur = cat;
    float* nxt = va;
    for (int l = 0; l < net.obs_final.num_layers; ++l) {
      const ppb_linear_desc& L = net.obs_final.layers[l];
      const bool last = l == net.obs_final.num_layers - 1;
      warp_dense_fwd(cur, L.in_dim, w_fin[l], L.out_dim, nxt, 0,
                     (last ? bufs.obs_emb : bufs.fin_act[l]) + (int64_t)tr * L.out_dim, lane);
      float* t = cur; cur = nxt; nxt = (t == cat) ? vb : t;
    }
    if (bufs.emb_k_hi) {   // cur = the embedding of this trace (warp-private shared memory)
      for (int k = lane; k < net.E; k += 32) {
        float hi, lo;
        tc::split_tf32(cur[k], hi, lo);
        const int64_t ok = tc::packed_offset(tr, k, bufs.emb_kb);
        bufs.emb_k_hi[ok] = hi;
        if (bufs.emb_k_lo) bufs.emb_k_lo[ok] = lo;
        if (bufs.emb_mn_hi) {
          const int64_t om = tc::packed_offset_mn(tr, k, bufs.emb_kb);
          bufs.emb_mn_hi[om] = hi;
          if (bufs.emb_mn_lo) bufs.emb_mn_lo[om] = lo;
        }
      }
    }
    __syncwarp();
  }
}

// dx[k] = (x[k] > 0) * sum_n dy[n] W[n][k]; lanes own inputs k, k + 32, k + 64; x read from the stored activations
__device__ __forceinline__ void warp_dense_dx(const float* dy, int out_dim, const float* w, int in_dim,
                                              const float* __restrict__ x, float* dx, float* gdx, int lane) {
  const int pitch = in_dim | 1;
  const bool p0 = lane < in_dim, p1 = lane + 32 < in_dim, p2 = lane + 64 < in_dim;
  const float x0 = p0 ? __ldg(x + lane) : 0.f, x1 = p1 ? __ldg(x + lane + 32) : 0.f, x2 = p2 ? __ldg(x + lane + 64) : 0.f;
  const float* c0 = w + (p0 ? lane : 0);
  const float* c1 = w + (p1 ? lane + 32 : 0);
  const float* c2 = w + (p2 ? lane + 64 : 0);
  float a0 = 0.f, a1 = 0.f, a2 = 0.f;
  if (in_dim <= 32) {
#pragma unroll 4
    for (int n = 0; n < out_dim; ++n) a0 = fmaf(dy[n], c0[n * pitch], a0);
  } else if (in_dim <= 64) {
#pragma unroll 4
    for (int n = 0; n < out_dim; ++n) { const float g = dy[n]; a0 = fmaf(g, c0[n * pitch], a0); a1 = fmaf(g, c1[n * pitch], a1); }
  } else {
#pragma unroll 4
    for (int n = 0; n < out_dim; ++n) { const float g = dy[n]; a0 = fmaf(g, c0[n * pitch], a0); a1 = fmaf(g, c1[n * pitch], a1); a2 = fmaf(g, c2[n * pitch], a2); }
  }
  if (p0) { a0 = x0 > 0.f ? a0 : 0.f; dx[lane] = a0; gdx[lane] = a0; }
  if (p1) { a1 = x1 > 0.f ? a1 : 0.f; dx[lane + 32] = a1; gdx[lane + 32] = a1; }
  if (p2) { a2 = x2 > 0.f ? a2 : 0.f; dx[lane + 64] = a2; gdx[lane + 64] = a2; }
  __syncwarp();
}

// backward chain per trace: fills the d(pre-activation) buffers of every layer (no weight gradients here)
__global__ void __launch_bounds__(kWarps * 32) k_bwd2_dx(Net net, const float* __restrict__ arena, int B, int traces_per_cta,
                                                         Bufs bufs, DBufs dbufs) {
  ppb_pdl_trigger();
  ppb_pdl_wait();
  extern __shared__ float smem[];
  float* p = smem;
  const float* w_obs[PPB_MAX_OBS][PPB_MAX_FF_LAYERS];
  const float* w_fin[PPB_MAX_FF_LAYERS];
  for (int j = 0; j < net.num_obs; ++j)
    for (int l = 0; l < net.obs_ff[j].num_layers; ++l) {
      w_obs[j][l] = p;
      // the first layer of a chain never propagates further down: no need to stage it
      if (l > 0) p = stage_layer(p, arena, net.obs_ff[j].layers[l]);
    }
  for (int l = 0; l < net.obs_final.num_layers; ++l) { w_fin[l] = p; p = stage_layer(p, arena, net.obs_final.layers[l]); }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, E = net.E;
  float* va = p + warp * 3 * W2;
  float* vb = va + W2;
  float* vc = vb + W2;
  cp_async_wait_all();
  __syncthreads();
  const int t0 = blockIdx.x * traces_per_cta;
  for (int tr = t0 + warp; tr < t0 + traces_per_cta && tr < B; tr += kWarps) {
    // d(pre-activation) of the last final layer: mask the incoming gradient by the (post-ReLU) output, in place
    for (int k = lane; k < E; k += 32) {
      int64_t o = (int64_t)tr * E + k;
      float g = bufs.obs_emb[o] > 0.f ? dbufs.d_obs_emb[o] : 0.f;
      va[k] = g;
      dbufs.d_obs_emb[o] = g;
    }
    __syncwarp();
    float* cur = va;
    float* nxt = vb;
    for (int l = net.obs_final.num_layers - 1; l >= 0; --l) {
      const ppb_linear_desc& L = net.obs_final.layers[l];
      const float* x = (l == 0 ? bufs.obs_cat : bufs.fin_act[l - 1]) + (int64_t)tr * L.in_dim;
      float* gdx = (l == 0 ? dbufs.d_obs_cat : dbufs.d_fin_act[l - 1]) + (int64_t)tr * L.in_dim;
      warp_dense_dx(cur, L.out_dim, w_fin[l], L.in_dim, x, nxt, gdx, lane);
      float* t = cur; cur = nxt; nxt = t;
    }
    // cur = d(obs_cat pre-activations) [E]; walk every observable's chain from its slice
    float* dcat = cur;
    float* scratch = nxt;
    int out_off = 0;
    for (int j = 0; j < net.num_obs; ++j) {
      const ppb_ff_desc& ff = net.obs_ff[j];
      const float* dy = dcat + out_off;
      float* o1 = scratch;
      float* o2 = vc;
      for (int l = ff.num_layers - 1; l >= 1; --l) {
        const ppb_linear_desc& L = ff.layers[l];
        const float* x = bufs.obs_act[j][l - 1] + (int64_t)tr * L.in_dim;
        warp_dense_dx(dy, L.out_dim, w_obs[j][l], L.in_dim, x, o1, dbufs.d_obs_act[j][l - 1] + (int64_t)tr * L.in_dim, lane);
        dy = o1;
        float* t = o1; o1 = o2; o2 = t;
      }
      out_off += ff.out_dim;
    }
    __syncwarp();
  }
}

// weight / bias gradients of every layer: one thread per weight, an atomic-free reduction over the traces of its slice
struct DwLayer { const float* dy; const float* x; int ldy, ldx, out_dim, in_dim, start, pad_; int64_t w_off, b_off; };
struct DwTable { int n_layers, total; DwLayer layer[PPB_MAX_OBS * PPB_MAX_FF_LAYERS + PPB_MAX_FF_LAYERS]; };

// block = 8 warps x 32 consecutive gradient entries: lane = entry, the warps stride over the traces of the block's slice,
// partial sums meet in shared memory (every thread runs B / 8 iterations, not B)
__global__ void __launch_bounds__(256) k_dw(DwTable tab, int B, int b_chunk, float* __restrict__ grad) {
  ppb_pdl_trigger();
  ppb_pdl_wait();
  __shared__ float part[8][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int idx = blockIdx.x * 32 + lane;
  float s = 0.f;
  int li = 0, e = 0, nw = 0;
  const bool live = idx < tab.total;
  if (live) {
    while (li + 1 < tab.n_layers && tab.layer[li + 1].start <= idx) ++li;
    const DwLayer& L = tab.layer[li];
    e = idx - L.start;
    nw = L.out_dim * L.in_dim;
    const int b0 = blockIdx.y * b_chunk, b1 = min(B, b0 + b_chunk);
    if (e < nw) {
      const int n = e / L.in_dim, k = e - n * L.in_dim;
      const float* dy = L.dy + n;
      const float* x = L.x + k;
#pragma unroll 8
      for (int b = b0 + warp; b < b1; b += 8) s = fmaf(__ldg(dy + (int64_t)b * L.ldy), __ldg(x + (int64_t)b * L.ldx), s);
    } else {
      const float* dy = L.dy + (e - nw);
#pragma unroll 8
      for (int b = b0 + warp; b < b1; b += 8) s += __ldg(dy + (int64_t)b * L.ldy);
    }
  }
  part[warp][lane] = s;
  __syncthreads();
  if (warp == 0 && live) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += part[w][lane];
    const DwLayer& L = tab.layer[li];
    if (t != 0.f) atomicAdd(grad + (e < nw ? L.w_off + e : L.b_off + (e - nw)), t);
  }
}

}  // namespace obsmlp
