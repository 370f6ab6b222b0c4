// Log-densities of the eleven families with an element-wise log_prob (PPB_EVENT_*), shared by the scoring kernels
// (scoring.cu) and the fused sample+score samplers (sampling.cu), so that a sampler's lp_out is the log_prob kernel's
// value at the drawn value.
// The reference wraps torch.distributions (pyprob/distributions/{exponential,gamma,log_normal,weibull,beta,binomial,
// von_mises}.py); every function below follows torch's log_prob term by term, in fp32.  A value outside the support or
// an invalid parameter gives NaN: the reference's argument validation raises there, and ppb_weights_cast then marks
// the particle invalid.
// Terms that depend on the parameters only (lgamma(c), lbeta, log I0(kappa), the Binomial normaliser) are split out as
// *_const so that a kernel can keep them per thread while the parameters repeat.
#pragma once
#include "common.cuh"

#define PPB_FLT_TINY 1.17549435e-38f     // torch.finfo(torch.float32).tiny
#define PPB_LOG_2PI 1.8378770664093453f  // math.log(2 * math.pi)

// MUFU approximations (<= 2 ulp): the scoring kernels are bound by instruction issue, not HBM, as soon as they carry an IEEE
// division or a libm logf/expf; results stay within 1e-6 relative of the libm forms.
__device__ __forceinline__ float fast_rcp(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float fast_ex2(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float fast_lg2(float x) { float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

// log(k!) for the counts that actually occur (k < 64), correctly rounded from the double-precision lgamma: lgammaf costs
// ~40 instructions per particle and made the Poisson kernel ALU-bound at 39 % of HBM; other values take lgammaf.
// A kernel whose Op has kTable copies the table to shared memory in every CTA: the lanes of a warp hold different counts,
// and a constant-bank read with divergent indices is replayed once per distinct address (63 % of HBM), shared memory
// serves them in one pass.  The library is built without relocatable device code, so every translation unit has its own
// copy of the table and uploads it once, on its first launch that needs it.
static __constant__ float c_log_factorial[64];
static inline int ppb_upload_log_factorial() {
  static bool table_ready = false;
  if (!table_ready) {
    float t[64];
    for (int k = 0; k < 64; ++k) t[k] = (float)lgamma((double)k + 1.0);
    PPB_CUDA(cudaMemcpyToSymbol(c_log_factorial, t, sizeof(t)));
    table_ready = true;
  }
  return PPB_OK;
}

namespace fam {

// torch.xlogy: 0 where x == 0, x * log(y) elsewhere
__device__ __forceinline__ float xlogy(float x, float y) { return x == 0.0f ? 0.0f : x * logf(y); }

// ---- Exponential(rate): log r - r x, x >= 0 ---------------------------------------------------------------------------
__device__ __forceinline__ float exponential_lp(float v, float r) {
  if (!(r > 0.0f) || !(v >= 0.0f)) return NAN;
  return logf(r) - r * v;
}

// ---- Gamma(concentration, rate): xlogy(c, r) + xlogy(c - 1, x) - r x - lgamma(c), x >= 0 ------------------------------
__device__ __forceinline__ float gamma_const(float c, float r) { return xlogy(c, r) - lgammaf(c); }
__device__ __forceinline__ float gamma_lp(float v, float c, float r, float k) {
  if (!(c > 0.0f) || !(r > 0.0f) || !(v >= 0.0f)) return NAN;
  return k + xlogy(c - 1.0f, v) - r * v;     // x = 0: +inf for c < 1, -inf for c > 1, as torch
}

// ---- LogNormal(loc, scale): Normal(loc, scale).log_prob(log x) - log x, x > 0 ------------------------------------------
__device__ __forceinline__ float lognormal_lp(float v, float mu, float s) {
  if (!(s > 0.0f) || !(v > 0.0f)) return NAN;
  const float x = logf(v);
  const float d = x - mu;
  return -(d * d) / (2.0f * (s * s)) - logf(s) - PPB_LOG_SQRT_2PI - x;
}

// ---- Weibull(scale, concentration), x > 0 --------------------------------------------------------------------------------
// torch's TransformedDistribution(Exponential(1), [PowerTransform(1/k), AffineTransform(0, scale)]) step by step:
// x1 = x / scale, x0 = x1^(1 / (1/k)), log_prob = -log(scale) - log|(1/k) x1 / x0| - x0.  Kept in that form (rather than
// log k - log scale + (k - 1) log x1 - x0) because torch's value differs from the closed form where x1^k under- or
// overflows, and the reference's value is torch's.
__device__ __forceinline__ float weibull_lp(float v, float lam, float k) {
  if (!(lam > 0.0f) || !(k > 0.0f) || !(v > 0.0f)) return NAN;
  const float e = 1.0f / k;
  const float x1 = v / lam;
  const float x0 = powf(x1, 1.0f / e);
  return (-logf(lam) - logf(fabsf(e * x1 / x0))) - x0;
}

// ---- Beta(c1, c0, low, high): torch Beta(c1, c0).log_prob(u), u = (x - low) / (high - low), u in [0, 1] ---------------
// torch Beta scores through Dirichlet: xlogy(c1 - 1, u) + xlogy(c0 - 1, 1 - u) + lgamma(c1 + c0) - lgamma(c1) - lgamma(c0).
// No -log(high - low) term: pyprob/distributions/beta.py:38-40 has none.
__device__ __forceinline__ float beta_const(float c1, float c0) { return lgammaf(c1 + c0) - (lgammaf(c1) + lgammaf(c0)); }
__device__ __forceinline__ float beta_lp(float v, float c1, float c0, float lo, float hi, float k) {
  const float u = (v - lo) / (hi - lo);
  if (!(c1 > 0.0f) || !(c0 > 0.0f) || !(u >= 0.0f && u <= 1.0f)) return NAN;
  return (xlogy(c1 - 1.0f, u) + xlogy(c0 - 1.0f, 1.0f - u)) + k;
}

// ---- Binomial(total_count, probs), k in {0, ..., n} ----------------------------------------------------------------------
// torch's logits form: logit = log(pc) - log1p(-pc) with pc = clamp_probs(p) (probs_to_logits, is_binary=True);
// log_prob = k logit - lgamma(k + 1) - lgamma(n - k + 1) - (n max(logit, 0) + n log1p(exp(-|logit|)) - lgamma(n + 1)).
struct BinomialConst {
  float logit, norm;
};
__device__ __forceinline__ BinomialConst binomial_const(float n, float p) {
  const float pc = ppb_clamp_prob(p);
  const float logit = logf(pc) - log1pf(-pc);
  return BinomialConst{logit, (n * fmaxf(logit, 0.0f) + n * log1pf(expf(-fabsf(logit)))) - lgammaf(n + 1.0f)};
}
__device__ __forceinline__ bool binomial_args_ok(float n, float p) {
  return n >= 0.0f && isfinite(n) && floorf(n) == n && p >= 0.0f && p <= 1.0f;
}
__device__ __forceinline__ float binomial_lp(float v, float n, float p, BinomialConst k) {
  if (!binomial_args_ok(n, p) || !(v >= 0.0f && v <= n && floorf(v) == v)) return NAN;
  return ((v * k.logit - lgammaf(v + 1.0f)) - lgammaf(n - v + 1.0f)) - k.norm;
}

// ---- VonMises(loc, concentration): kappa cos(x - loc) - log(2 pi) - log I0(kappa), x real --------------------------------
// log I0 as torch.distributions.von_mises._log_modified_bessel_fn(kappa, order=0) computes it: the Abramowitz & Stegun
// 9.8.1 polynomial below 3.75, and kappa - log(kappa) / 2 + log(9.8.2 polynomial) above, which does not overflow at large
// kappa the way log(I0) computed directly does past kappa = 88.
__device__ __forceinline__ float von_mises_const(float kappa) {
  if (kappa < 3.75f) {
    float y = kappa / 3.75f;
    y = y * y;
    float s = 0.45813e-2f;
    s = 0.360768e-1f + y * s;
    s = 0.2659732f + y * s;
    s = 1.2067492f + y * s;
    s = 3.0899424f + y * s;
    s = 3.5156229f + y * s;
    s = 1.0f + y * s;
    return logf(s);
  }
  const float y = 3.75f / kappa;
  float l = 0.392377e-2f;
  l = -0.1647633e-1f + y * l;
  l = 0.2635537e-1f + y * l;
  l = -0.2057706e-1f + y * l;
  l = 0.916281e-2f + y * l;
  l = -0.157565e-2f + y * l;
  l = 0.225319e-2f + y * l;
  l = 0.1328592e-1f + y * l;
  l = 0.39894228f + y * l;
  return kappa - 0.5f * logf(kappa) + logf(l);
}
__device__ __forceinline__ float von_mises_lp(float v, float loc, float kappa, float li0) {
  if (!(kappa > 0.0f)) return NAN;
  return (kappa * cosf(v - loc) - PPB_LOG_2PI) - li0;
}

}  // namespace fam

// ---- one log-density functor per family ---------------------------------------------------------------------------------
// op(v, p, tab): log p(v) under parameters p[0 .. kParams - 1] (the PPB_EVENT_* order; later slots are unused), with tab
// the shared-memory copy of c_log_factorial when kTable.  An Op whose log_prob has a term that depends on the parameters
// only keeps it in the thread together with the parameters it was computed for, and recomputes it only when they change:
// with shared (stride-0) parameters that is once per thread instead of once per particle (lgammaf alone is ~40
// instructions).  A kernel keeps one Op per thread for its whole grid-stride loop.
struct NormalOp {
  static constexpr int kFamily = PPB_EVENT_NORMAL, kParams = 2;
  static constexpr bool kTable = false;
  // torch/distributions/normal.py log_prob: -((v - mu)^2) / (2 var) - log(sigma) - log(sqrt(2 pi))
  __device__ __forceinline__ float operator()(float v, const float (&p)[4], const float*) const {
    const float z = (v - p[0]) * fast_rcp(p[1]);
    return fmaf(-0.5f * z, z, -fast_lg2(p[1]) * PPB_LN2) - PPB_LOG_SQRT_2PI;
  }
};
struct UniformOp {
  static constexpr int kFamily = PPB_EVENT_UNIFORM, kParams = 2;
  static constexpr bool kTable = false;
  // torch/distributions/uniform.py log_prob: log(lb*ub) - log(high-low), lb = low<=v, ub = high>v
  __device__ __forceinline__ float operator()(float v, const float (&p)[4], const float*) const {
    float inside = (p[0] <= v && p[1] > v) ? 0.0f : -INFINITY;
    return inside - logf(p[1] - p[0]);
  }
};
struct PoissonOp {
  static constexpr int kFamily = PPB_EVENT_POISSON, kParams = 1;
  static constexpr bool kTable = true;
  // torch/distributions/poisson.py log_prob: xlogy(v, rate) - rate - lgamma(v+1)
  __device__ __forceinline__ float operator()(float v, const float (&p)[4], const float* tab) const {
    float xl = (v == 0.0f) ? 0.0f : v * (fast_lg2(p[0]) * PPB_LN2);
    const int k = (int)v;
    const float lg = (v >= 0.0f && v < 64.0f && (float)k == v) ? tab[k] : lgammaf(v + 1.0f);
    return xl - p[0] - lg;
  }
};
struct BernoulliOp {
  static constexpr int kFamily = PPB_EVENT_BERNOULLI, kParams = 1;
  static constexpr bool kTable = false;
  // torch/distributions/bernoulli.py log_prob: -BCEWithLogits(log pc - log1p(-pc), v) = v log pc + (1 - v) log(1 - pc),
  // pc = clamp_probs(p); values outside {0, 1} are rejected by the reference's argument validation: NaN here
  __device__ __forceinline__ float operator()(float v, const float (&p)[4], const float*) const {
    const float pc = ppb_clamp_prob(p[0]);
    return (v == 1.0f) ? logf(pc) : (v == 0.0f) ? log1pf(-pc) : NAN;
  }
};
struct ExponentialOp {
  static constexpr int kFamily = PPB_EVENT_EXPONENTIAL, kParams = 1;
  static constexpr bool kTable = false;
  __device__ __forceinline__ float operator()(float v, const float (&p)[4], const float*) const {
    return fam::exponential_lp(v, p[0]);
  }
};
struct GammaOp {
  static constexpr int kFamily = PPB_EVENT_GAMMA, kParams = 2;
  static constexpr bool kTable = false;
  float c_ = NAN, r_ = NAN, k_ = NAN;
  __device__ __forceinline__ float operator()(float v, const float (&p)[4], const float*) {
    if (!(p[0] == c_ && p[1] == r_)) { c_ = p[0]; r_ = p[1]; k_ = fam::gamma_const(p[0], p[1]); }
    return fam::gamma_lp(v, p[0], p[1], k_);
  }
};
struct LogNormalOp {
  static constexpr int kFamily = PPB_EVENT_LOGNORMAL, kParams = 2;
  static constexpr bool kTable = false;
  __device__ __forceinline__ float operator()(float v, const float (&p)[4], const float*) const {
    return fam::lognormal_lp(v, p[0], p[1]);
  }
};
struct WeibullOp {
  static constexpr int kFamily = PPB_EVENT_WEIBULL, kParams = 2;
  static constexpr bool kTable = false;
  __device__ __forceinline__ float operator()(float v, const float (&p)[4], const float*) const {
    return fam::weibull_lp(v, p[0], p[1]);
  }
};
struct BetaOp {
  static constexpr int kFamily = PPB_EVENT_BETA, kParams = 4;
  static constexpr bool kTable = false;
  float a_ = NAN, b_ = NAN, k_ = NAN;
  __device__ __forceinline__ float operator()(float v, const float (&p)[4], const float*) {
    if (!(p[0] == a_ && p[1] == b_)) { a_ = p[0]; b_ = p[1]; k_ = fam::beta_const(p[0], p[1]); }
    return fam::beta_lp(v, p[0], p[1], p[2], p[3], k_);
  }
};
struct BinomialOp {
  static constexpr int kFamily = PPB_EVENT_BINOMIAL, kParams = 2;
  static constexpr bool kTable = false;
  float n_ = NAN, p_ = NAN;
  fam::BinomialConst k_{NAN, NAN};
  __device__ __forceinline__ float operator()(float v, const float (&p)[4], const float*) {
    if (!(p[0] == n_ && p[1] == p_)) { n_ = p[0]; p_ = p[1]; k_ = fam::binomial_const(p[0], p[1]); }
    return fam::binomial_lp(v, p[0], p[1], k_);
  }
};
struct VonMisesOp {
  static constexpr int kFamily = PPB_EVENT_VON_MISES, kParams = 2;
  static constexpr bool kTable = false;
  float kappa_ = NAN, k_ = NAN;
  __device__ __forceinline__ float operator()(float v, const float (&p)[4], const float*) {
    if (!(p[1] == kappa_)) { kappa_ = p[1]; k_ = fam::von_mises_const(p[1]); }
    return fam::von_mises_lp(v, p[0], p[1], k_);
  }
};

// fn(Op{}) for the Op of a PPB_EVENT_* id; -1 for an unknown id
template <class Fn>
int ppb_with_family(int family, Fn&& fn) {
  switch (family) {
    case PPB_EVENT_NORMAL: return fn(NormalOp{});
    case PPB_EVENT_UNIFORM: return fn(UniformOp{});
    case PPB_EVENT_POISSON: return fn(PoissonOp{});
    case PPB_EVENT_BERNOULLI: return fn(BernoulliOp{});
    case PPB_EVENT_EXPONENTIAL: return fn(ExponentialOp{});
    case PPB_EVENT_GAMMA: return fn(GammaOp{});
    case PPB_EVENT_LOGNORMAL: return fn(LogNormalOp{});
    case PPB_EVENT_WEIBULL: return fn(WeibullOp{});
    case PPB_EVENT_BETA: return fn(BetaOp{});
    case PPB_EVENT_BINOMIAL: return fn(BinomialOp{});
    case PPB_EVENT_VON_MISES: return fn(VonMisesOp{});
    default: return -1;
  }
}

// number of parameters of a family; -1 for an unknown id
inline int ppb_event_num_params(int family) {
  return ppb_with_family(family, [](auto op) { return decltype(op)::kParams; });
}

// Event-summed log_prob (scoring.cu), shared with the event sampler (sampling.cu), whose lp_out at D > 1 is this
// kernel's fp32 row sum of the drawn rows (row_lp; at D = 1 a row is its one element, lp_out).  params / params_ps /
// params_es hold ppb_event_num_params(family) operands.
int ppb_event_score(int family, const float* value, int64_t value_ps, int64_t value_es, const float* const* params,
                    const int64_t* params_ps, const int64_t* params_es, int64_t n, int64_t D, float* lp_out,
                    float* row_lp, double* acc, double acc_scale, void* stream);
