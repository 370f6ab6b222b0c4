// Proposal-head parameter transforms, log-probabilities and their hand-derived gradients.
// Mirrors pyprob/nn/proposal_normal_normal_mixture.py:18-35, proposal_uniform_truncated_normal_mixture.py:18-36,
// proposal_poisson_truncated_normal_mixture.py:20-36, proposal_categorical_categorical.py:16-20,
// proposal_bernoulli_bernoulli.py:16-20 and the distributions they build (mixture.py:8-45, truncated_normal.py:11-54,
// torch Categorical(probs), torch Bernoulli(probs)).
#pragma once
#include "common.cuh"

namespace heads {

constexpr int KMAX = 32;    // mixture components supported per head
constexpr int CMAX = 128;   // categories supported per categorical head
#define PPB_INV_SQRT_2PI 0.3989422804014327f
#define PPB_UTIL_EPSILON 1e-8f  // pyprob/util.py:34

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float std_normal_pdf(float x) { return PPB_INV_SQRT_2PI * expf(-0.5f * x * x); }

// x[0..3K): raw head output.  Writes means/stddevs/probs (each K) as the reference's Mixture receives them.
// family NORMAL: p0 = prior mean, p1 = prior stddev; UNIFORM: p0 = low, p1 = high; POISSON: ignored (0, 40).
__device__ __forceinline__ void mixture_params(int family, const float* x, int K, float p0, float p1, float* mean,
                                               float* sd, float* prob, float* lo_out, float* hi_out) {
  float mx = -INFINITY;
  for (int k = 0; k < K; ++k) mx = fmaxf(mx, x[2 * K + k]);
  float s = 0.0f;
  for (int k = 0; k < K; ++k) { prob[k] = expf(x[2 * K + k] - mx); s += prob[k]; }
  for (int k = 0; k < K; ++k) prob[k] /= s;
  if (family == PPB_FAMILY_NORMAL) {
    for (int k = 0; k < K; ++k) { mean[k] = p0 + x[k] * p1; sd[k] = expf(x[K + k]) * p1; }
    *lo_out = 0.0f; *hi_out = 0.0f;
  } else if (family == PPB_FAMILY_UNIFORM) {
    float range = p1 - p0;
    for (int k = 0; k < K; ++k) {
      mean[k] = p0 + sigmoidf_(x[k]) * range;
      sd[k] = range / 1000.0f + sigmoidf_(x[K + k]) * range * 10.0f;
    }
    *lo_out = p0; *hi_out = p1;
  } else {  // POISSON: fixed truncation [0, 40]
    for (int k = 0; k < K; ++k) { mean[k] = 0.0f + sigmoidf_(x[k]) * (40.0f - 0.0f); sd[k] = expf(x[K + k]); }
    *lo_out = 0.0f; *hi_out = 40.0f;
  }
}

// log q(v) for a mixture head and d(-log q)/dx into gx[0..3K).  Returns log q (may be -inf / nan).
__device__ __forceinline__ float mixture_nll(int family, const float* x, int K, float p0, float p1, float v,
                                             float* gx, bool want_grad) {
  float mean[KMAX], sd[KMAX], prob[KMAX];
  float lo, hi;
  mixture_params(family, x, K, p0, p1, mean, sd, prob, &lo, &hi);
  const bool trunc = family != PPB_FAMILY_NORMAL;
  // Mixture.__init__: renormalise, clamp, log
  float S = 0.0f;
  for (int k = 0; k < K; ++k) S += prob[k];
  float t[KMAX];
  bool clamped[KMAX];
  float mxt = -INFINITY;
  for (int k = 0; k < K; ++k) {
    float ph = prob[k] / S;
    clamped[k] = (ph < PPB_EPS32) || (ph > 1.0f - PPB_EPS32);
    float lw = logf(ppb_clamp_prob(ph));
    float lpk = trunc ? ppb_truncnormal_lp(v, mean[k], sd[k], lo, hi) : ppb_normal_lp(v, mean[k], sd[k]);
    t[k] = lw + lpk;
    mxt = fmaxf(mxt, t[k]);
  }
  float lp;
  if (mxt == -INFINITY) {
    lp = -INFINITY;
  } else {
    float acc = 0.0f;
    for (int k = 0; k < K; ++k) acc += expf(t[k] - mxt);
    lp = mxt + logf(acc);
  }
  if (!want_grad) return lp;
  if (!(lp > -INFINITY) || !(lp < INFINITY)) {  // -inf is repaired with a constant (zero gradient); nan/inf abort
    for (int j = 0; j < 3 * K; ++j) gx[j] = 0.0f;
    return lp;
  }
  // responsibilities r_k = exp(t_k - lp)
  float g_prob[KMAX];  // d lp / d prob_k (before softmax)
  float sum_r_unclamped = 0.0f;
  float r[KMAX];
  for (int k = 0; k < K; ++k) {
    r[k] = expf(t[k] - lp);
    if (!clamped[k]) sum_r_unclamped += r[k];
  }
  for (int k = 0; k < K; ++k) {
    float ph = prob[k] / S;
    float direct = clamped[k] ? 0.0f : r[k] / ph;   // d lp / d phat_k
    g_prob[k] = (direct - sum_r_unclamped) / S;      // through phat = prob / S
  }
  // softmax backward: d lp / d z_j = prob_j * (g_j - sum_m prob_m g_m)
  float dot = 0.0f;
  for (int k = 0; k < K; ++k) dot += prob[k] * g_prob[k];
  for (int k = 0; k < K; ++k) gx[2 * K + k] = -(prob[k] * (g_prob[k] - dot));
  for (int k = 0; k < K; ++k) {
    float z = (v - mean[k]) / sd[k];
    float dmu, dsd;
    if (!trunc) {
      dmu = z / sd[k];
      dsd = (z * z - 1.0f) / sd[k];
    } else {
      float alpha = (lo - mean[k]) / sd[k], beta = (hi - mean[k]) / sd[k];
      float Z = ppb_std_normal_cdf(beta) - ppb_std_normal_cdf(alpha);
      float pa = std_normal_pdf(alpha), pb = std_normal_pdf(beta);
      dmu = z / sd[k] - (pa - pb) / (sd[k] * Z);
      dsd = (z * z - 1.0f) / sd[k] - (alpha * pa - beta * pb) / (sd[k] * Z);
    }
    dmu *= r[k];
    dsd *= r[k];
    float dxm, dxs;
    if (family == PPB_FAMILY_NORMAL) {
      dxm = dmu * p1;
      dxs = dsd * sd[k];
    } else if (family == PPB_FAMILY_UNIFORM) {
      float range = p1 - p0;
      float sm = sigmoidf_(x[k]), ss = sigmoidf_(x[K + k]);
      dxm = dmu * sm * (1.0f - sm) * range;
      dxs = dsd * ss * (1.0f - ss) * range * 10.0f;
    } else {
      float sm = sigmoidf_(x[k]);
      dxm = dmu * sm * (1.0f - sm) * 40.0f;
      dxs = dsd * sd[k];
    }
    gx[k] = -dxm;
    gx[K + k] = -dxs;
  }
  return lp;
}

// Categorical head: probs = softmax(x) + 1e-8; torch Categorical(probs) normalises and clamps.
__device__ __forceinline__ void categorical_probs(const float* x, int C, float* prob) {
  float mx = -INFINITY;
  for (int c = 0; c < C; ++c) mx = fmaxf(mx, x[c]);
  float s = 0.0f;
  for (int c = 0; c < C; ++c) { prob[c] = expf(x[c] - mx); s += prob[c]; }
  for (int c = 0; c < C; ++c) prob[c] = prob[c] / s + PPB_UTIL_EPSILON;
}

// Bernoulli head (proposal_bernoulli_bernoulli.py): probs = sigmoid(x) + 1e-8; torch Bernoulli(probs) clamps.
__device__ __forceinline__ float bernoulli_prob(float x) { return sigmoidf_(x) + PPB_UTIL_EPSILON; }

__device__ __forceinline__ float categorical_nll(const float* x, int C, float v, float* gx, bool want_grad) {
  float q[CMAX];
  categorical_probs(x, C, q);
  float S = 0.0f;
  for (int c = 0; c < C; ++c) S += q[c];
  int iv = (int)v;
  if (iv < 0 || iv >= C) {
    if (want_grad) for (int c = 0; c < C; ++c) gx[c] = 0.0f;
    return NAN;
  }
  float ph = q[iv] / S;
  bool clamped = (ph < PPB_EPS32) || (ph > 1.0f - PPB_EPS32);
  float lp = logf(ppb_clamp_prob(ph));
  if (!want_grad) return lp;
  if (clamped || !(lp > -INFINITY)) {
    for (int c = 0; c < C; ++c) gx[c] = 0.0f;
    return lp;
  }
  // d lp / d q_j = delta_jv / q_v - 1 / S ; softmax part of q_j is sm_j = q_j - eps
  float dot = 0.0f;
  for (int c = 0; c < C; ++c) {
    float g = ((c == iv) ? 1.0f / q[iv] : 0.0f) - 1.0f / S;
    dot += (q[c] - PPB_UTIL_EPSILON) * g;
  }
  for (int c = 0; c < C; ++c) {
    float g = ((c == iv) ? 1.0f / q[iv] : 0.0f) - 1.0f / S;
    gx[c] = -((q[c] - PPB_UTIL_EPSILON) * (g - dot));
  }
  return lp;
}

}  // namespace heads
