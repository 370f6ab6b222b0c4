// Proposal-head parameter transforms (the IC proposal step; net.cu: nll_row restates them lane-parallel for the loss).
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

}  // namespace heads
