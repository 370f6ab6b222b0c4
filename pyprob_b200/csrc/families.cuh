// Log-densities of the Exponential, Gamma, LogNormal, Weibull, Beta, Binomial and VonMises families, shared by the
// scoring kernels (scoring.cu) and the fused sample+score samplers (sampling.cu), so that a sampler's lp_out is the
// log_prob kernel's value at the drawn value.
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

// Event-summed log_prob (scoring.cu), shared with the event samplers (sampling.cu), whose lp_out is this kernel's fp32
// row sum of the drawn rows.  params / params_ps / params_es hold ppb_event_num_params(family) operands.
int ppb_event_num_params(int family);
int ppb_event_score(int family, const float* value, int64_t value_ps, int64_t value_es, const float* const* params,
                    const int64_t* params_ps, const int64_t* params_es, int64_t n, int64_t D, float* lp_out,
                    float* row_lp, double* acc, double acc_scale, void* stream);
