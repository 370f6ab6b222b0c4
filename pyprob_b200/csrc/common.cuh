// Shared helpers for the pyprob_b200 CUDA sources (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <math.h>

#include "../../include/pyprob_b200.h"

#define PPB_NUM_SMS 132  // H100 SXM; grids are sized in multiples of this

void ppb_set_error(const char* fmt, ...);

#define PPB_CHECK_ARG(cond, msg)                               \
  do {                                                         \
    if (!(cond)) {                                             \
      ppb_set_error("%s: %s", __func__, msg);                  \
      return PPB_EINVAL;                                       \
    }                                                          \
  } while (0)

#define PPB_CUDA(call)                                                              \
  do {                                                                              \
    cudaError_t _e = (call);                                                        \
    if (_e != cudaSuccess) {                                                        \
      ppb_set_error("%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
      return (int)_e;                                                               \
    }                                                                               \
  } while (0)

extern unsigned long long g_ppb_launches;  // kernels launched by this library (bench.py reports it)

#define PPB_LAUNCH_CHECK()                                                          \
  do {                                                                              \
    ++g_ppb_launches;                                                               \
    cudaError_t _e = cudaGetLastError();                                            \
    if (_e != cudaSuccess) {                                                        \
      ppb_set_error("%s:%d launch: %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return (int)_e;                                                               \
    }                                                                               \
  } while (0)

// ---- programmatic dependent launch (PDL) -----------------------------------------------------------------------------------
// A kernel launched with the programmatic-stream-serialisation attribute may START (block scheduling, shared-memory carve-out,
// its own prologue) while its predecessor in the stream is still running; ppb_pdl_wait() then blocks until the predecessor
// grid has completed and its writes are visible.  The launch gap between two dependent kernels and the tensor-core
// kernels' prologue (barrier init, descriptor fetch) are hidden behind the predecessor's tail this way.
// Rules kept by every converted kernel: before ppb_pdl_wait() it reads nothing but its host-uploaded descriptor table and
// writes nothing to global memory; ppb_pdl_trigger() comes first so that the successor can be scheduled as early as possible
// (the hardware launches it only after EVERY block of this grid has started, so it cannot starve this grid of SMs).
// Both instructions are no-ops in a kernel launched without the attribute.
__device__ __forceinline__ void ppb_pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void ppb_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

bool ppb_pdl_enabled();          // default on; PPB_PDL=0 disables (lib.cu)
bool ppb_persistent_enabled();   // default on; PPB_PERSISTENT=0 disables the persistent grouped GEMM (lib.cu)

// <<<grid, block, smem, st>>> with optional PDL attribute (pdl, unless PPB_PDL=0) and optional (cluster, 1, 1)
// thread-block cluster
template <typename... KArgs, typename... Args>
inline cudaError_t ppb_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl,
                              int cluster, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = (unsigned)cluster;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  if (pdl && ppb_pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = (unsigned)n;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}

static inline int ppb_grid_for(int64_t n, int threads, int items_per_thread, int max_waves = 8) {
  int64_t blocks = (n + (int64_t)threads * items_per_thread - 1) / ((int64_t)threads * items_per_thread);
  if (blocks < 1) blocks = 1;
  // cap at a multiple of the SM count; kernels are grid-stride
  int64_t cap = (int64_t)PPB_NUM_SMS * max_waves;
  if (blocks > cap) blocks = cap;
  return (int)blocks;
}

// Bias corrections of Adam step t (1-based) from the betas of a device hyper vector (PPB_HYPER_* slots), computed in
// double and rounded once to fp32: bc1 = 1 - b1^t (the update's step is lr / bc1) and bc2_sqrt = sqrt(1 - b2^t).
// beta2 is read after the first pow(), so that it does not hold a register across it.
__device__ __forceinline__ void ppb_adam_bias_corrections(const float* hyper, long long t, float& bc1, float& bc2_sqrt) {
  bc1 = (float)(1.0 - pow((double)hyper[PPB_HYPER_BETA1], (double)t));
  bc2_sqrt = (float)sqrt(1.0 - pow((double)hyper[PPB_HYPER_BETA2], (double)t));
}

// One Adam update (torch.optim.Adam without amsgrad) with every rounding spelled out, so that the flat, the
// segmented and the data-parallel fused optimiser kernels produce the same bits:
//   g' = g*gscale + wd*p;  m = b1 m + (1-b1) g';  v = b2 v + (1-b2) g'^2;  p -= step * m / (sqrt(v)/bc2_sqrt + eps)
__device__ __forceinline__ void ppb_adam_update(float& p, float g, float& m, float& v, float b1, float b2, float eps,
                                                float wd, float gscale, float step, float bc2_sqrt) {
  float gr = __fmaf_rn(g, gscale, __fmul_rn(wd, p));
  m = __fmaf_rn(b1, m, __fmul_rn(1.0f - b1, gr));
  v = __fmaf_rn(b2, v, __fmul_rn(__fmul_rn(1.0f - b2, gr), gr));
  float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), eps);
  p = __fsub_rn(p, __fdiv_rn(__fmul_rn(step, m), denom));
}

// ---- math constants (fp32, written the way torch.distributions writes them) -------------------
#define PPB_LOG_SQRT_2PI 0.9189385332046727f  // math.log(math.sqrt(2*math.pi))
#define PPB_LOG2E 1.4426950408889634f
#define PPB_LN2 0.6931471805599453f
#define PPB_INV_SQRT2 0.7071067811865476f
#define PPB_EPS32 1.1920928955078125e-07f     // torch.finfo(torch.float32).eps
#define PPB_LOG_EPSILON (-18.420680743952367f) // pyprob/util.py:35 log(1e-8)

__device__ __forceinline__ float ppb_normal_lp(float v, float mu, float sigma) {
  // torch/distributions/normal.py log_prob: -((v-mu)^2)/(2 var) - log(scale) - log(sqrt(2 pi))
  float var = sigma * sigma;
  float d = v - mu;
  return -(d * d) / (2.0f * var) - logf(sigma) - PPB_LOG_SQRT_2PI;
}

// LSTM cell activations, branch-free (the libm forms carry a slow-path branch each — division, tanhf's range split — which cut
// the epilogue of the fused LSTM kernels into one basic block per gate and kept the loads of different rows from overlapping;
// they were also a third of its instructions).  EX2 / RCP approximations, measured against fp64 on an H100: sigmoid within
// 1.5e-7 relative for x >= -1; below, x * log2(e) is rounded to fp32 before ex2, so the relative error grows with |x|
// (1.7e-6 at x = -25, 3.8e-6 at x = -84), and below x = -87.3 the result is flushed to zero.  tanh within 3.7e-7 relative
// (odd Taylor polynomial to x^9 below 0.25, 1 - 2 / (1 + exp(2|x|)) above, worst just above 0.25).  Every cell kernel, fused or not,
// forward or backward, goes through these two, so all variants agree to the last bit of the activation.
__device__ __forceinline__ float ppb_cell_sigmoid(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -PPB_LOG2E));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return r;
}
__device__ __forceinline__ float ppb_cell_tanh(float x) {
  const float ax = fabsf(x);
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(ax * (2.0f * PPB_LOG2E)));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  const float big = fmaf(-2.0f, r, 1.0f);
  const float x2 = ax * ax;
  float p = fmaf(x2, 62.0f / 2835.0f, -17.0f / 315.0f);
  p = fmaf(x2, p, 2.0f / 15.0f);
  p = fmaf(x2, p, -1.0f / 3.0f);
  const float small = fmaf(ax * x2, p, ax);
  return copysignf(ax < 0.25f ? small : big, x);
}

__device__ __forceinline__ float ppb_std_normal_cdf(float x) {
  // torch Normal(0,1).cdf: 0.5 * (1 + erf(x / sqrt(2)))
  return 0.5f * (1.0f + erff(x * PPB_INV_SQRT2));
}

__device__ __forceinline__ float ppb_clamp_prob(float p) {
  // pyprob/util.py:393-395 clamp_probs
  return fminf(fmaxf(p, PPB_EPS32), 1.0f - PPB_EPS32);
}

__device__ __forceinline__ float ppb_truncnormal_lp(float v, float mu, float sigma, float lo, float hi) {
  // pyprob/distributions/truncated_normal.py:24-30, :40-45
  float alpha = (lo - mu) / sigma;
  float beta = (hi - mu) / sigma;
  float Z = ppb_std_normal_cdf(beta) - ppb_std_normal_cdf(alpha);
  float log_sz = logf(sigma * Z);
  float z = (v - mu) / sigma;
  float inside = (v >= lo && v <= hi) ? 0.0f : -INFINITY;  // log(lb*ub)
  return inside + (-(z * z) / 2.0f - PPB_LOG_SQRT_2PI) - log_sz;
}

// inverse-CDF draw (truncated_normal.py:104): icdf(Phi(alpha) + u (Phi(beta)-Phi(alpha))) * sigma + mu; shared by the
// truncated mixture sampler (sampling.cu) and the RMH Uniform kernel (mcmc.cu)
__device__ __forceinline__ float ppb_truncnormal_draw(float mu, float sg, float lo, float hi, float u) {
  float ca = ppb_std_normal_cdf((lo - mu) / sg), cb = ppb_std_normal_cdf((hi - mu) / sg);
  float q = ca + u * (cb - ca);
  q = fminf(fmaxf(q, 1e-7f), 1.0f - 6e-8f);
  float v = normcdfinvf(q) * sg + mu;
  // keep the draw inside [lo, hi): the reference retries until lo <= v < hi, and a Uniform prior that this mixture proposes
  // for scores v = hi as -inf
  return fminf(fmaxf(v, lo), nextafterf(hi, lo));
}

__device__ __forceinline__ float ppb_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double ppb_warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float ppb_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- Philox4x32-10 (counter-based; D. E. Shaw Research "Random123" published algorithm) --------
struct ppb_philox {
  uint32_t c[4];
};
__device__ __forceinline__ ppb_philox ppb_philox4x32_10(uint64_t seed, uint64_t idx, uint64_t offset) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  uint32_t c0 = (uint32_t)idx, c1 = (uint32_t)(idx >> 32), c2 = (uint32_t)offset, c3 = (uint32_t)(offset >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  ppb_philox out; out.c[0] = c0; out.c[1] = c1; out.c[2] = c2; out.c[3] = c3;
  return out;
}
// uniform in [0,1): 24 random bits
__device__ __forceinline__ float ppb_u01(uint32_t x) { return (float)(x >> 8) * (1.0f / 16777216.0f); }
// uniform in (0,1]: for logs
__device__ __forceinline__ float ppb_u01_open0(uint32_t x) { return ((float)(x >> 8) + 1.0f) * (1.0f / 16777216.0f); }
__device__ __forceinline__ float ppb_std_normal_from(uint32_t a, uint32_t b) {
  // Box-Muller
  float u1 = ppb_u01_open0(a), u2 = ppb_u01(b);
  return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
}
