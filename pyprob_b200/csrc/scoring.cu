// Per-family log_prob over the particle axis — warp-coalesced, 128-bit vectorised, HBM-bound.
// Replaces pyprob/distributions/distribution.py:38-43 as driven per particle by pyprob/state.py.
// Algorithmic bytes per element (SURVEY §8d): Normal/Uniform 16 B, Poisson/Bernoulli 12 B, Categorical 4C+12 B,
// Mixture-Normal (3K+2)*4 B, Mixture-TruncatedNormal (3K+4)*4 B; Exponential 12 B, Gamma/LogNormal/Weibull/Binomial/
// VonMises 16 B, Beta 24 B with per-particle parameters (value + lp_out + 4 B per per-particle parameter).
// Event sites (k_event, pyprob/state.py:147 with a tensor value): 4 B per element of each per-particle-event operand, a
// shared event row once, 16 B per particle for the fp64 accumulator (+ 4 B per element for lp_out).
#include "common.cuh"
#include "families.cuh"

namespace {

constexpr int kThreads = 256;

__host__ __device__ __forceinline__ bool aligned16(const void* p) { return (((uintptr_t)p) & 15u) == 0; }

// Streaming 128-bit load that bypasses L1 (each element is touched once).
__device__ __forceinline__ float4 ldg_stream4(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}

struct Param {
  const float* p;
  int stride;  // 0 = scalar broadcast, 1 = per particle
  __device__ __forceinline__ float at(int64_t i) const { return stride ? __ldg(p + i) : __ldg(p); }
  __device__ __forceinline__ void load4(int64_t i, float (&o)[4]) const {
    if (stride) {
      float4 v = ldg_stream4(p + i);
      o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
    } else {
      float s = __ldg(p);
      o[0] = o[1] = o[2] = o[3] = s;
    }
  }
  bool vec_ok() const { return stride == 0 || ((((uintptr_t)p) & 15u) == 0); }
};

struct Sink {
  float* lp;
  double* acc;
  double scale;
  __device__ __forceinline__ void put(int64_t i, float v) const {
    if (lp) lp[i] = v;
    if (acc) acc[i] += scale * (double)v;
  }
  __device__ __forceinline__ void put4(int64_t i, const float (&v)[4]) const {
    if (lp) *reinterpret_cast<float4*>(lp + i) = make_float4(v[0], v[1], v[2], v[3]);
    if (acc) {
      double2 a0 = *reinterpret_cast<double2*>(acc + i);
      double2 a1 = *reinterpret_cast<double2*>(acc + i + 2);
      a0.x += scale * (double)v[0]; a0.y += scale * (double)v[1];
      a1.x += scale * (double)v[2]; a1.y += scale * (double)v[3];
      *reinterpret_cast<double2*>(acc + i) = a0;
      *reinterpret_cast<double2*>(acc + i + 2) = a1;
    }
  }
  bool vec_ok() const { return (!lp || ((((uintptr_t)lp) & 15u) == 0)) && (!acc || ((((uintptr_t)acc) & 15u) == 0)); }
};

// ---- two-parameter families ---------------------------------------------------------------------
// MUFU approximations (<= 2 ulp): the scoring kernels are bound by instruction issue, not HBM, as soon as they carry an IEEE
// division or a libm logf/expf; results stay within 1e-6 relative of the libm forms.
__device__ __forceinline__ float fast_rcp(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float fast_ex2(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float fast_lg2(float x) { float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

struct NormalOp {
  static constexpr bool kTable = false;
  // torch/distributions/normal.py log_prob: -((v - mu)^2) / (2 var) - log(sigma) - log(sqrt(2 pi))
  __device__ __forceinline__ float operator()(float v, float mu, float sigma, const float*) const {
    const float z = (v - mu) * fast_rcp(sigma);
    return fmaf(-0.5f * z, z, -fast_lg2(sigma) * PPB_LN2) - PPB_LOG_SQRT_2PI;
  }
};
struct UniformOp {
  // torch/distributions/uniform.py log_prob: log(lb*ub) - log(high-low), lb = low<=v, ub = high>v
  static constexpr bool kTable = false;
  __device__ __forceinline__ float operator()(float v, float lo, float hi, const float*) const {
    float inside = (lo <= v && hi > v) ? 0.0f : -INFINITY;
    return inside - logf(hi - lo);
  }
};
// log(k!) for the counts that actually occur (k < 64), correctly rounded from the double-precision lgamma: lgammaf costs
// ~40 instructions per particle and made the Poisson kernel ALU-bound at 39 % of HBM; other values take lgammaf.
// The table is copied to shared memory by every CTA: the lanes of a warp hold different counts, and a constant-bank read
// with divergent indices is replayed once per distinct address (63 % of HBM), shared memory serves them in one pass.
__constant__ float c_log_factorial[64];
struct PoissonOp {
  static constexpr bool kTable = true;
  // torch/distributions/poisson.py log_prob: xlogy(v, rate) - rate - lgamma(v+1)
  __device__ __forceinline__ float operator()(float v, float rate, float, const float* tab) const {
    float xl = (v == 0.0f) ? 0.0f : v * (fast_lg2(rate) * PPB_LN2);
    const int k = (int)v;
    const float lg = (v >= 0.0f && v < 64.0f && (float)k == v) ? tab[k] : lgammaf(v + 1.0f);
    return xl - rate - lg;
  }
};
struct BernoulliOp {
  static constexpr bool kTable = false;
  // torch/distributions/bernoulli.py log_prob: -BCEWithLogits(log pc - log1p(-pc), v) = v log pc + (1 - v) log(1 - pc),
  // pc = clamp_probs(p); values outside {0, 1} are rejected by the reference's argument validation: NaN here
  __device__ __forceinline__ float operator()(float v, float p, float, const float*) const {
    const float pc = ppb_clamp_prob(p);
    return (v == 1.0f) ? logf(pc) : (v == 0.0f) ? log1pf(-pc) : NAN;
  }
};

// Exponential .. VonMises (families.cuh).  An Op whose log_prob has a term that depends on the parameters only keeps it
// in the thread together with the parameters it was computed for, and recomputes it only when they change: with shared
// (stride-0) parameters that is once per thread instead of once per particle (lgammaf alone is ~40 instructions).
struct ExponentialOp {
  static constexpr bool kTable = false;
  __device__ __forceinline__ float operator()(float v, float rate, float, const float*) const {
    return fam::exponential_lp(v, rate);
  }
};
struct GammaOp {
  static constexpr bool kTable = false;
  float c_ = NAN, r_ = NAN, k_ = NAN;
  __device__ __forceinline__ float operator()(float v, float c, float r, const float*) {
    if (!(c == c_ && r == r_)) { c_ = c; r_ = r; k_ = fam::gamma_const(c, r); }
    return fam::gamma_lp(v, c, r, k_);
  }
};
struct LogNormalOp {
  static constexpr bool kTable = false;
  __device__ __forceinline__ float operator()(float v, float mu, float s, const float*) const {
    return fam::lognormal_lp(v, mu, s);
  }
};
struct WeibullOp {
  static constexpr bool kTable = false;
  __device__ __forceinline__ float operator()(float v, float scale, float k, const float*) const {
    return fam::weibull_lp(v, scale, k);
  }
};
struct BinomialOp {
  static constexpr bool kTable = false;
  float n_ = NAN, p_ = NAN;
  fam::BinomialConst k_{NAN, NAN};
  __device__ __forceinline__ float operator()(float v, float n, float p, const float*) {
    if (!(n == n_ && p == p_)) { n_ = n; p_ = p; k_ = fam::binomial_const(n, p); }
    return fam::binomial_lp(v, n, p, k_);
  }
};
struct VonMisesOp {
  static constexpr bool kTable = false;
  float kappa_ = NAN, k_ = NAN;
  __device__ __forceinline__ float operator()(float v, float loc, float kappa, const float*) {
    if (!(kappa == kappa_)) { kappa_ = kappa; k_ = fam::von_mises_const(kappa); }
    return fam::von_mises_lp(v, loc, kappa, k_);
  }
};

template <class Op, bool VEC>
__global__ void __launch_bounds__(kThreads) k_score2(const float* __restrict__ value, Param a, Param b, Sink out,
                                                      int64_t n, Op op) {
  __shared__ float tab[Op::kTable ? 64 : 1];
  if (Op::kTable) {
    if (threadIdx.x < 64) tab[threadIdx.x] = c_log_factorial[threadIdx.x];
    __syncthreads();
  }
  int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t nth = (int64_t)gridDim.x * blockDim.x;
  if (VEC) {
    int64_t n4 = n >> 2;
    for (int64_t q = tid; q < n4; q += nth) {
      int64_t i = q << 2;
      float4 vv = ldg_stream4(value + i);
      float v[4] = {vv.x, vv.y, vv.z, vv.w};
      float pa[4], pb[4], r[4];
      a.load4(i, pa);
      b.load4(i, pb);
#pragma unroll
      for (int j = 0; j < 4; ++j) r[j] = op(v[j], pa[j], pb[j], tab);
      out.put4(i, r);
    }
    for (int64_t i = (n4 << 2) + tid; i < n; i += nth) out.put(i, op(__ldg(value + i), a.at(i), b.at(i), tab));
  } else {
    for (int64_t i = tid; i < n; i += nth) out.put(i, op(__ldg(value + i), a.at(i), b.at(i), tab));
  }
}

template <class Op>
int launch_score2(const float* value, Param a, Param b, Sink out, int64_t n, void* stream, Op op) {
  if (n == 0) return PPB_OK;
  bool vec = aligned16(value) && a.vec_ok() && b.vec_ok() && out.vec_ok();
  cudaStream_t st = (cudaStream_t)stream;
  int grid = ppb_grid_for(n, kThreads, 4);
  if (vec)
    k_score2<Op, true><<<grid, kThreads, 0, st>>>(value, a, b, out, n, op);
  else
    k_score2<Op, false><<<grid, kThreads, 0, st>>>(value, a, b, out, n, op);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

// ---- beta (four parameters) ----------------------------------------------------------------------------------------------
// lbeta(c1, c0) is kept per thread while (c1, c0) repeat, as in the Ops above
template <bool VEC>
__global__ void __launch_bounds__(kThreads) k_beta(const float* __restrict__ value, Param c1, Param c0, Param low,
                                                    Param high, Sink out, int64_t n) {
  int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t nth = (int64_t)gridDim.x * blockDim.x;
  float a_ = NAN, b_ = NAN, k_ = NAN;
  auto lp = [&](float v, float a, float b, float lo, float hi) {
    if (!(a == a_ && b == b_)) { a_ = a; b_ = b; k_ = fam::beta_const(a, b); }
    return fam::beta_lp(v, a, b, lo, hi, k_);
  };
  int64_t i0 = 0;
  if (VEC) {
    int64_t n4 = n >> 2;
    for (int64_t q = tid; q < n4; q += nth) {
      int64_t i = q << 2;
      float4 vv = ldg_stream4(value + i);
      float v[4] = {vv.x, vv.y, vv.z, vv.w};
      float pa[4], pb[4], pl[4], ph[4], r[4];
      c1.load4(i, pa);
      c0.load4(i, pb);
      low.load4(i, pl);
      high.load4(i, ph);
#pragma unroll
      for (int j = 0; j < 4; ++j) r[j] = lp(v[j], pa[j], pb[j], pl[j], ph[j]);
      out.put4(i, r);
    }
    i0 = n4 << 2;
  }
  for (int64_t i = i0 + tid; i < n; i += nth) out.put(i, lp(__ldg(value + i), c1.at(i), c0.at(i), low.at(i), high.at(i)));
}

// ---- categorical --------------------------------------------------------------------------------
// log_prob = log(clamp(p[v] / sum(p))) (torch Categorical(probs=...): normalise, probs_to_logits clamps)
__global__ void __launch_bounds__(kThreads) k_categorical(const float* __restrict__ value,
                                                           const float* __restrict__ probs, int64_t row_stride,
                                                           int C, Sink out, int64_t n) {
  int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t nth = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = tid; i < n; i += nth) {
    const float* p = probs + i * row_stride;
    int v = (int)__ldg(value + i);
    float s = 0.0f, pv = 0.0f;
    bool vec = (C % 4 == 0) && aligned16(p);
    if (vec) {
      for (int c = 0; c < C; c += 4) {
        float4 q = __ldg(reinterpret_cast<const float4*>(p + c));
        s += q.x; s += q.y; s += q.z; s += q.w;
        if (v >= c && v < c + 4) pv = (v == c) ? q.x : (v == c + 1) ? q.y : (v == c + 2) ? q.z : q.w;
      }
    } else {
      for (int c = 0; c < C; ++c) {
        float q = __ldg(p + c);
        s += q;
        if (c == v) pv = q;
      }
    }
    float lp = (v >= 0 && v < C) ? logf(ppb_clamp_prob(pv / s)) : NAN;
    out.put(i, lp);
  }
}

// ---- mixtures ------------------------------------------------------------------------------------
// Mixture.log_prob (pyprob/distributions/mixture.py:15-16, :38-45):
//   w = probs / sum(probs); lw = log(clamp(w)); lp = logsumexp_k(lw_k + lp_k(v))
// Arithmetic: with w_k = clamp(p_k / sum p) and z_k = (v - mu_k) / sigma_k,
//   logsumexp_k(log w_k + log N(v; mu_k, sigma_k)) = max_k(-z_k^2 / 2) + log sum_k (w_k / sigma_k) exp(-z_k^2 / 2 - max) - log sqrt(2 pi)
// (truncated components: sigma_k -> sigma_k Z_k, and -inf outside [low, high]): one exp and one reciprocal per component and
// ONE log per particle instead of two logs, an exp and two divisions per component — these kernels are bound by the
// transcendental/ALU rate, not by HBM.  Same value as the reference's formula up to fp32 rounding.
// EXACT: K == KMAX is known at compile time (the component loops carry no k < K predicates)
template <int KMAX, bool TRUNC, bool EXACT = false>
__device__ __forceinline__ float mixture_row(float v, const float* __restrict__ m, const float* __restrict__ s,
                                             const float* __restrict__ p, int K_rt, float lo, float hi) {
  const int K = EXACT ? KMAX : K_rt;
  // Reciprocals, the exponentials and the final log use the hardware approximations (MUFU.RCP / EX2 / LG2: <= 2 ulp on the
  // terms that matter — exp arguments are <= 0 and the largest term is exp(0) = 1 exactly): IEEE divisions and expf make the
  // kernel issue-bound well below HBM bandwidth.
  float pk[KMAX], a[KMAX], scale[KMAX];
  float psum = 0.0f;
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    pk[k] = (k < K) ? p[k] : 0.0f;
    psum += pk[k];
  }
  const float inv_psum = fast_rcp(psum);
  float mx = -INFINITY;
  bool bad = false;
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    if (k < K) {
      const float mu = m[k], sg = s[k];
      const float inv_sg = fast_rcp(sg);
      const float z = (v - mu) * inv_sg;
      float inv_norm = inv_sg;               // 1 / (sigma * truncated mass)
      bool neg = !(sg >= 0.0f);
      if (TRUNC) {
        const float alpha = (lo - mu) * inv_sg, beta = (hi - mu) * inv_sg;
        const float mass = ppb_std_normal_cdf(beta) - ppb_std_normal_cdf(alpha);
        inv_norm = inv_sg * fast_rcp(mass);
        neg = neg || !(mass >= 0.0f);
      }
      a[k] = (-0.5f * PPB_LOG2E) * z * z;   // exponent in base 2
      scale[k] = ppb_clamp_prob(pk[k] * inv_psum) * inv_norm;
      bad = bad || neg || (a[k] != a[k]) || (scale[k] != scale[k]);
      mx = fmaxf(mx, a[k]);
    }
  }
  if (bad) return NAN;                       // log of a negative / NaN parameter poisons the row like the reference
  if (TRUNC && !(v >= lo && v <= hi)) return -INFINITY;   // log(lb * ub) = -inf in every component
  if (mx == -INFINITY) return -INFINITY;     // torch.logsumexp of all -inf
  float acc = 0.0f;
#pragma unroll
  for (int k = 0; k < KMAX; ++k)
    if (k < K) acc = fmaf(scale[k], fast_ex2(a[k] - mx), acc);
  return (mx + fast_lg2(acc)) * PPB_LN2 - PPB_LOG_SQRT_2PI;
}

template <int KMAX, bool TRUNC, bool EXACT = false>
__global__ void __launch_bounds__(kThreads) k_mixture(const float* __restrict__ value,
                                                       const float* __restrict__ means,
                                                       const float* __restrict__ stddevs,
                                                       const float* __restrict__ probs, int64_t row_stride, int K,
                                                       Param low, Param high, Sink out, int64_t n) {
  int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t nth = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = tid; i < n; i += nth) {
    float lo = 0.f, hi = 0.f;
    if (TRUNC) { lo = low.at(i); hi = high.at(i); }
    out.put(i, mixture_row<KMAX, TRUNC, EXACT>(__ldg(value + i), means + i * row_stride, stddevs + i * row_stride,
                                               probs + i * row_stride, K, lo, hi));
  }
}

template <bool TRUNC>
int launch_mixture(const float* value, const float* means, const float* stddevs, const float* probs,
                   int64_t row_stride, int K, Param low, Param high, Sink out, int64_t n, void* stream) {
  if (n == 0) return PPB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int grid = ppb_grid_for(n, kThreads, 1);
  if (K <= 4)
    k_mixture<4, TRUNC><<<grid, kThreads, 0, st>>>(value, means, stddevs, probs, row_stride, K, low, high, out, n);
  else if (K == 10)   // the proposal heads' component count (pyprob/nn/proposal_normal_mixture.py: mixture_components = 10)
    k_mixture<10, TRUNC, true><<<grid, kThreads, 0, st>>>(value, means, stddevs, probs, row_stride, K, low, high, out, n);
  else if (K <= 10)
    k_mixture<10, TRUNC><<<grid, kThreads, 0, st>>>(value, means, stddevs, probs, row_stride, K, low, high, out, n);
  else if (K <= 32)
    k_mixture<32, TRUNC><<<grid, kThreads, 0, st>>>(value, means, stddevs, probs, row_stride, K, low, high, out, n);
  else {
    ppb_set_error("mixture log_prob: K=%d > 32 not supported", K);
    return PPB_ENOTSUP;
  }
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

// ---- event-shaped sites: sum_j log p(v_ij) per particle ----------------------------------------------------------------
// One kernel template over the Ops above for every family with an element-wise log_prob.  An operand is (pointer,
// particle stride ps, element stride es): element j of particle i is p[i ps + j es], with (ps, es) one of (0, 0) scalar,
// (1, 0) one per particle, (0, 1) shared event, (D, 1) event per particle.
// Thread mapping: G lanes (a power of two, 1 .. 32) share a row; lane l of a group owns the 4-element chunks
// l, l + G, l + 2G, ... of the row, and G is the smallest power of two >= ceil(D / 4) (capped at 32), so small D puts
// several rows in a warp and large D a warp on each row.  A chunk is one 128-bit load where its address is 16-byte
// aligned (every chunk of an aligned row; D is generally not a multiple of 4, so which rows are aligned depends on i) and
// four 32-bit loads elsewhere.  Per-particle rows stream past L1; a shared event row is read through L1 / L2.
// Each lane sums its elements in fp64 in element order, and the group combines its lanes with a fixed butterfly: the
// order depends on (n, D) only (G is a function of D; the load width does not change what is summed), so a call is
// bit-reproducible, and with D = 1 the sum is the single term, exactly k_score2's accumulator update.
struct EvOperand {
  const float* p;
  int64_t ps, es;
  // elements j0 .. j0 + 3 of row i (elements at or past D read as 0 and are never used)
  __device__ __forceinline__ void load4(int64_t i, int64_t j0, int64_t D, float (&o)[4]) const {
    const float* r = p + i * ps;
    if (es == 0) {
      const float s = __ldg(r);
      o[0] = o[1] = o[2] = o[3] = s;
      return;
    }
    r += j0;
    if (j0 + 4 <= D && aligned16(r)) {
      const float4 v = ps ? ldg_stream4(r) : __ldg(reinterpret_cast<const float4*>(r));
      o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) o[k] = (j0 + k < D) ? __ldg(r + k) : 0.0f;
    }
  }
};

struct EvArgs {
  EvOperand v, p[4];
  float* lp;       // nullable [n, D] element-wise log-densities
  float* row_lp;   // nullable [n] fp32 row sums (the samplers' lp_out)
  double* acc;     // nullable [n] acc[i] += scale * row sum
  double scale;
  int64_t n, D;
};

// (value, parameter vector) -> log-density, over the two-parameter Ops (one-parameter families ignore p[1])
template <class Op>
struct EvFamily {
  static constexpr bool kTable = Op::kTable;
  Op op;
  __device__ __forceinline__ float operator()(float v, const float (&p)[4], const float* tab) {
    return op(v, p[0], p[1], tab);
  }
};
struct EvBeta {
  static constexpr bool kTable = false;
  float a_ = NAN, b_ = NAN, k_ = NAN;
  __device__ __forceinline__ float operator()(float v, const float (&p)[4], const float*) {
    if (!(p[0] == a_ && p[1] == b_)) { a_ = p[0]; b_ = p[1]; k_ = fam::beta_const(p[0], p[1]); }
    return fam::beta_lp(v, p[0], p[1], p[2], p[3], k_);
  }
};

template <class F, int NP, int G>
__global__ void __launch_bounds__(kThreads) k_event(EvArgs a, F f) {
  __shared__ float tab[F::kTable ? 64 : 1];
  if (F::kTable) {
    if (threadIdx.x < 64) tab[threadIdx.x] = c_log_factorial[threadIdx.x];
    __syncthreads();
  }
  constexpr int kRowsPerWarp = 32 / G;
  const int lane = threadIdx.x & 31, sub = lane % G;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t D = a.D, chunks = (D + 3) >> 2;
  for (int64_t base = warp * kRowsPerWarp; base < a.n; base += nwarps * kRowsPerWarp) {   // warp-uniform
    const int64_t i = base + lane / G;
    double s = 0.0;
    if (i < a.n) {
      for (int64_t c = sub; c < chunks; c += G) {
        const int64_t j0 = c << 2;
        float v[4], p[NP][4], r[4];
        a.v.load4(i, j0, D, v);
#pragma unroll
        for (int k = 0; k < NP; ++k) a.p[k].load4(i, j0, D, p[k]);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float pe[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) pe[k] = p[k < NP ? k : 0][e];
          r[e] = f(v[e], pe, tab);
        }
        const int m = (D - j0 < 4) ? (int)(D - j0) : 4;
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (e < m) s += (double)r[e];
        if (a.lp) {
          float* o = a.lp + i * D + j0;
          if (m == 4 && aligned16(o)) {
            *reinterpret_cast<float4*>(o) = make_float4(r[0], r[1], r[2], r[3]);
          } else {
#pragma unroll
            for (int e = 0; e < 4; ++e)
              if (e < m) o[e] = r[e];
          }
        }
      }
    }
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (i < a.n && sub == 0) {
      if (a.acc) a.acc[i] += a.scale * s;
      if (a.row_lp) a.row_lp[i] = (float)s;
    }
  }
}

template <class F, int NP>
int launch_event(const EvArgs& a, cudaStream_t st, F f) {
  const int64_t chunks = (a.D + 3) >> 2;
  int g = 1;
  while (g < chunks && g < 32) g <<= 1;
  const int grid = ppb_grid_for(a.n, kThreads / g, 1);
  switch (g) {
    case 1: k_event<F, NP, 1><<<grid, kThreads, 0, st>>>(a, f); break;
    case 2: k_event<F, NP, 2><<<grid, kThreads, 0, st>>>(a, f); break;
    case 4: k_event<F, NP, 4><<<grid, kThreads, 0, st>>>(a, f); break;
    case 8: k_event<F, NP, 8><<<grid, kThreads, 0, st>>>(a, f); break;
    case 16: k_event<F, NP, 16><<<grid, kThreads, 0, st>>>(a, f); break;
    default: k_event<F, NP, 32><<<grid, kThreads, 0, st>>>(a, f); break;
  }
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

// c_log_factorial, uploaded once per process by the first Poisson log_prob call (per-particle or event)
int upload_log_factorial() {
  static bool table_ready = false;
  if (!table_ready) {
    float t[64];
    for (int k = 0; k < 64; ++k) t[k] = (float)lgamma((double)k + 1.0);
    PPB_CUDA(cudaMemcpyToSymbol(c_log_factorial, t, sizeof(t)));
    table_ready = true;
  }
  return PPB_OK;
}

bool ev_layout_ok(const void* p, int64_t ps, int64_t es, int64_t D) {
  return p && ((ps == 0 && es == 0) || (ps == 1 && es == 0) || (ps == 0 && es == 1) || (ps == D && es == 1));
}

}  // namespace

int ppb_event_num_params(int family) {
  switch (family) {
    case PPB_EVENT_POISSON: case PPB_EVENT_BERNOULLI: case PPB_EVENT_EXPONENTIAL: return 1;
    case PPB_EVENT_BETA: return 4;
    case PPB_EVENT_NORMAL: case PPB_EVENT_UNIFORM: case PPB_EVENT_GAMMA: case PPB_EVENT_LOGNORMAL:
    case PPB_EVENT_WEIBULL: case PPB_EVENT_BINOMIAL: case PPB_EVENT_VON_MISES: return 2;
    default: return -1;
  }
}

int ppb_event_score(int family, const float* value, int64_t value_ps, int64_t value_es, const float* const* params,
                    const int64_t* params_ps, const int64_t* params_es, int64_t n, int64_t D, float* lp_out,
                    float* row_lp, double* acc, double acc_scale, void* stream) {
  const int np = ppb_event_num_params(family);
  PPB_CHECK_ARG(np > 0, "unknown family id");
  PPB_CHECK_ARG(n >= 0 && D > 0, "n must be >= 0 and D > 0");
  PPB_CHECK_ARG(ev_layout_ok(value, value_ps, value_es, D),
                "value: null pointer, or strides not one of (0, 0), (1, 0), (0, 1), (D, 1)");
  EvArgs a;
  a.v = EvOperand{value, value_ps, value_es};
  for (int k = 0; k < 4; ++k) {
    if (k < np) {
      PPB_CHECK_ARG(ev_layout_ok(params[k], params_ps[k], params_es[k], D),
                    "parameter: null pointer, or strides not one of (0, 0), (1, 0), (0, 1), (D, 1)");
      a.p[k] = EvOperand{params[k], params_ps[k], params_es[k]};
    } else {
      a.p[k] = EvOperand{nullptr, 0, 0};
    }
  }
  if (n == 0) return PPB_OK;
  a.lp = lp_out;
  a.row_lp = row_lp;
  a.acc = acc;
  a.scale = acc_scale;
  a.n = n;
  a.D = D;
  cudaStream_t st = (cudaStream_t)stream;
  switch (family) {
    case PPB_EVENT_NORMAL: return launch_event<EvFamily<NormalOp>, 2>(a, st, {});
    case PPB_EVENT_UNIFORM: return launch_event<EvFamily<UniformOp>, 2>(a, st, {});
    case PPB_EVENT_POISSON: {
      const int e = upload_log_factorial();
      if (e != PPB_OK) return e;
      return launch_event<EvFamily<PoissonOp>, 1>(a, st, {});
    }
    case PPB_EVENT_BERNOULLI: return launch_event<EvFamily<BernoulliOp>, 1>(a, st, {});
    case PPB_EVENT_EXPONENTIAL: return launch_event<EvFamily<ExponentialOp>, 1>(a, st, {});
    case PPB_EVENT_GAMMA: return launch_event<EvFamily<GammaOp>, 2>(a, st, {});
    case PPB_EVENT_LOGNORMAL: return launch_event<EvFamily<LogNormalOp>, 2>(a, st, {});
    case PPB_EVENT_WEIBULL: return launch_event<EvFamily<WeibullOp>, 2>(a, st, {});
    case PPB_EVENT_BETA: return launch_event<EvBeta, 4>(a, st, {});
    case PPB_EVENT_BINOMIAL: return launch_event<EvFamily<BinomialOp>, 2>(a, st, {});
    default: return launch_event<EvFamily<VonMisesOp>, 2>(a, st, {});
  }
}

extern "C" {

int ppb_event_log_prob(int family, const float* value, int64_t value_ps, int64_t value_es, const float* p0,
                       int64_t p0_ps, int64_t p0_es, const float* p1, int64_t p1_ps, int64_t p1_es, const float* p2,
                       int64_t p2_ps, int64_t p2_es, const float* p3, int64_t p3_ps, int64_t p3_es, int64_t n,
                       int64_t D, float* lp_out, double* acc, double acc_scale, void* stream) {
  const float* p[4] = {p0, p1, p2, p3};
  const int64_t ps[4] = {p0_ps, p1_ps, p2_ps, p3_ps}, es[4] = {p0_es, p1_es, p2_es, p3_es};
  return ppb_event_score(family, value, value_ps, value_es, p, ps, es, n, D, lp_out, nullptr, acc, acc_scale, stream);
}

int ppb_normal_log_prob(const float* value, const float* mean, int mean_stride, const float* stddev,
                        int stddev_stride, float* lp_out, double* acc, double acc_scale, int64_t n, void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && value && mean && stddev, "null pointer or negative n");
  PPB_CHECK_ARG((mean_stride | 1) == 1 && (stddev_stride | 1) == 1, "strides must be 0 or 1");
  return launch_score2(value, Param{mean, mean_stride}, Param{stddev, stddev_stride}, Sink{lp_out, acc, acc_scale}, n,
                       stream, NormalOp{});
}

int ppb_uniform_log_prob(const float* value, const float* low, int low_stride, const float* high, int high_stride,
                         float* lp_out, double* acc, double acc_scale, int64_t n, void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && value && low && high, "null pointer or negative n");
  PPB_CHECK_ARG((low_stride | 1) == 1 && (high_stride | 1) == 1, "strides must be 0 or 1");
  return launch_score2(value, Param{low, low_stride}, Param{high, high_stride}, Sink{lp_out, acc, acc_scale}, n, stream,
                       UniformOp{});
}

int ppb_poisson_log_prob(const float* value, const float* rate, int rate_stride, float* lp_out, double* acc,
                         double acc_scale, int64_t n, void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && value && rate, "null pointer or negative n");
  PPB_CHECK_ARG((rate_stride | 1) == 1, "strides must be 0 or 1");
  const int e = upload_log_factorial();
  if (e != PPB_OK) return e;
  return launch_score2(value, Param{rate, rate_stride}, Param{rate, 0}, Sink{lp_out, acc, acc_scale}, n, stream,
                       PoissonOp{});
}

int ppb_bernoulli_log_prob(const float* value, const float* probs, int probs_stride, float* lp_out, double* acc,
                           double acc_scale, int64_t n, void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && value && probs, "null pointer or negative n");
  PPB_CHECK_ARG((probs_stride | 1) == 1, "strides must be 0 or 1");
  return launch_score2(value, Param{probs, probs_stride}, Param{probs, 0}, Sink{lp_out, acc, acc_scale}, n, stream,
                       BernoulliOp{});
}

int ppb_exponential_log_prob(const float* value, const float* rate, int rate_stride, float* lp_out, double* acc,
                             double acc_scale, int64_t n, void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && value && rate, "null pointer or negative n");
  PPB_CHECK_ARG((rate_stride | 1) == 1, "strides must be 0 or 1");
  return launch_score2(value, Param{rate, rate_stride}, Param{rate, 0}, Sink{lp_out, acc, acc_scale}, n, stream,
                       ExponentialOp{});
}

int ppb_gamma_log_prob(const float* value, const float* concentration, int concentration_stride, const float* rate,
                       int rate_stride, float* lp_out, double* acc, double acc_scale, int64_t n, void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && value && concentration && rate, "null pointer or negative n");
  PPB_CHECK_ARG((concentration_stride | 1) == 1 && (rate_stride | 1) == 1, "strides must be 0 or 1");
  return launch_score2(value, Param{concentration, concentration_stride}, Param{rate, rate_stride},
                       Sink{lp_out, acc, acc_scale}, n, stream, GammaOp{});
}

int ppb_lognormal_log_prob(const float* value, const float* loc, int loc_stride, const float* scale, int scale_stride,
                           float* lp_out, double* acc, double acc_scale, int64_t n, void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && value && loc && scale, "null pointer or negative n");
  PPB_CHECK_ARG((loc_stride | 1) == 1 && (scale_stride | 1) == 1, "strides must be 0 or 1");
  return launch_score2(value, Param{loc, loc_stride}, Param{scale, scale_stride}, Sink{lp_out, acc, acc_scale}, n,
                       stream, LogNormalOp{});
}

int ppb_weibull_log_prob(const float* value, const float* scale, int scale_stride, const float* concentration,
                         int concentration_stride, float* lp_out, double* acc, double acc_scale, int64_t n,
                         void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && value && scale && concentration, "null pointer or negative n");
  PPB_CHECK_ARG((scale_stride | 1) == 1 && (concentration_stride | 1) == 1, "strides must be 0 or 1");
  return launch_score2(value, Param{scale, scale_stride}, Param{concentration, concentration_stride},
                       Sink{lp_out, acc, acc_scale}, n, stream, WeibullOp{});
}

int ppb_beta_log_prob(const float* value, const float* concentration1, int concentration1_stride,
                      const float* concentration0, int concentration0_stride, const float* low, int low_stride,
                      const float* high, int high_stride, float* lp_out, double* acc, double acc_scale, int64_t n,
                      void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && value && concentration1 && concentration0 && low && high, "null pointer or negative n");
  PPB_CHECK_ARG((concentration1_stride | 1) == 1 && (concentration0_stride | 1) == 1 && (low_stride | 1) == 1 &&
                    (high_stride | 1) == 1,
                "strides must be 0 or 1");
  Param a{concentration1, concentration1_stride}, b{concentration0, concentration0_stride}, lo{low, low_stride},
      hi{high, high_stride};
  Sink out{lp_out, acc, acc_scale};
  const bool vec = aligned16(value) && a.vec_ok() && b.vec_ok() && lo.vec_ok() && hi.vec_ok() && out.vec_ok();
  const int grid = ppb_grid_for(n, kThreads, 4);
  if (vec)
    k_beta<true><<<grid, kThreads, 0, (cudaStream_t)stream>>>(value, a, b, lo, hi, out, n);
  else
    k_beta<false><<<grid, kThreads, 0, (cudaStream_t)stream>>>(value, a, b, lo, hi, out, n);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int ppb_binomial_log_prob(const float* value, const float* total_count, int total_count_stride, const float* probs,
                          int probs_stride, float* lp_out, double* acc, double acc_scale, int64_t n, void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && value && total_count && probs, "null pointer or negative n");
  PPB_CHECK_ARG((total_count_stride | 1) == 1 && (probs_stride | 1) == 1, "strides must be 0 or 1");
  return launch_score2(value, Param{total_count, total_count_stride}, Param{probs, probs_stride},
                       Sink{lp_out, acc, acc_scale}, n, stream, BinomialOp{});
}

int ppb_von_mises_log_prob(const float* value, const float* loc, int loc_stride, const float* concentration,
                           int concentration_stride, float* lp_out, double* acc, double acc_scale, int64_t n,
                           void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && value && loc && concentration, "null pointer or negative n");
  PPB_CHECK_ARG((loc_stride | 1) == 1 && (concentration_stride | 1) == 1, "strides must be 0 or 1");
  return launch_score2(value, Param{loc, loc_stride}, Param{concentration, concentration_stride},
                       Sink{lp_out, acc, acc_scale}, n, stream, VonMisesOp{});
}

int ppb_categorical_log_prob(const float* value, const float* probs, int64_t probs_row_stride, int num_categories,
                             float* lp_out, double* acc, double acc_scale, int64_t n, void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && value && probs && num_categories > 0, "bad arguments");
  PPB_CHECK_ARG(probs_row_stride == 0 || probs_row_stride >= num_categories, "row stride < num_categories");
  if (n == 0) return PPB_OK;
  int grid = ppb_grid_for(n, kThreads, 1);
  k_categorical<<<grid, kThreads, 0, (cudaStream_t)stream>>>(value, probs, probs_row_stride, num_categories,
                                                             Sink{lp_out, acc, acc_scale}, n);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int ppb_mixture_normal_log_prob(const float* value, const float* means, const float* stddevs, const float* probs,
                                int64_t row_stride, int K, float* lp_out, double* acc, double acc_scale, int64_t n,
                                void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && value && means && stddevs && probs && K > 0, "bad arguments");
  return launch_mixture<false>(value, means, stddevs, probs, row_stride, K, Param{nullptr, 0}, Param{nullptr, 0},
                               Sink{lp_out, acc, acc_scale}, n, stream);
}

int ppb_mixture_truncated_normal_log_prob(const float* value, const float* means, const float* stddevs,
                                          const float* probs, int64_t row_stride, int K, const float* low,
                                          int low_stride, const float* high, int high_stride, float* lp_out,
                                          double* acc, double acc_scale, int64_t n, void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && value && means && stddevs && probs && low && high && K > 0, "bad arguments");
  return launch_mixture<true>(value, means, stddevs, probs, row_stride, K, Param{low, low_stride},
                              Param{high, high_stride}, Sink{lp_out, acc, acc_scale}, n, stream);
}

}  // extern "C"
