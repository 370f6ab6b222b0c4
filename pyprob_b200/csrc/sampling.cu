// Samplers over the particle axis (Philox4x32-10, counter = (global particle index, offset)).
// Replaces pyprob/distributions/distribution.py:31-36, mixture.py:47-63, truncated_normal.py:94-112.
// Fused sample+score: lp_out (nullable) gets log_prob of the drawn value (pyprob/state.py:196-197).
#include "common.cuh"

namespace {

constexpr int kThreads = 256;

struct P {
  const float* p;
  int stride;
  __device__ __forceinline__ float at(int64_t i) const { return stride ? __ldg(p + i) : __ldg(p); }
};

__global__ void __launch_bounds__(kThreads) k_normal(P mean, P sd, float* __restrict__ out, float* __restrict__ lp,
                                                      int64_t n, uint64_t seed, uint64_t offset, int64_t first) {
  int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = tid; i < n; i += nth) {
    ppb_philox r = ppb_philox4x32_10(seed, (uint64_t)(first + i), offset);
    float z = ppb_std_normal_from(r.c[0], r.c[1]);
    float mu = mean.at(i), s = sd.at(i);
    float v = mu + s * z;
    out[i] = v;
    if (lp) lp[i] = ppb_normal_lp(v, mu, s);
  }
}

__global__ void __launch_bounds__(kThreads) k_uniform(P low, P high, float* __restrict__ out, float* __restrict__ lp,
                                                       int64_t n, uint64_t seed, uint64_t offset, int64_t first) {
  int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = tid; i < n; i += nth) {
    ppb_philox r = ppb_philox4x32_10(seed, (uint64_t)(first + i), offset);
    float lo = low.at(i), hi = high.at(i);
    float v = lo + ppb_u01(r.c[0]) * (hi - lo);
    out[i] = v;
    if (lp) lp[i] = ((lo <= v && hi > v) ? 0.0f : -INFINITY) - logf(hi - lo);
  }
}

// Poisson: inversion by sequential search for rate < 10 (Devroye), PTRS transformed rejection
// (W. Hoermann 1993) for rate >= 10; the rejection loop draws fresh Philox words with a bumped counter.
__device__ float poisson_draw(float rate, uint64_t seed, uint64_t idx, uint64_t offset) {
  if (!(rate > 0.0f)) return 0.0f;
  if (rate < 10.0f) {
    float L = expf(-rate);
    float k = 0.0f, p = 1.0f;
    uint64_t sub = 0;
    while (true) {
      ppb_philox r = ppb_philox4x32_10(seed, idx, offset + (sub << 40));
      ++sub;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        p *= ppb_u01_open0(r.c[j]);
        if (p <= L) return k;
        k += 1.0f;
      }
      if (sub > 64) return k;
    }
  }
  float slam = sqrtf(rate), loglam = logf(rate);
  float b = 0.931f + 2.53f * slam;
  float a = -0.059f + 0.02483f * b;
  float invalpha = 1.1239f + 1.1328f / (b - 3.4f);
  float vr = 0.9277f - 3.6224f / (b - 2.0f);
  for (uint64_t sub = 0; sub < 64; ++sub) {
    ppb_philox r = ppb_philox4x32_10(seed, idx, offset + (sub << 40));
    for (int j = 0; j < 4; j += 2) {
      float U = ppb_u01(r.c[j]) - 0.5f;
      float V = ppb_u01_open0(r.c[j + 1]);
      float us = 0.5f - fabsf(U);
      float k = floorf((2.0f * a / us + b) * U + rate + 0.43f);
      if (us >= 0.07f && V <= vr) return k;
      if (k < 0.0f || (us < 0.013f && V > us)) continue;
      if (logf(V) + logf(invalpha) - logf(a / (us * us) + b) <= -rate + k * loglam - lgammaf(k + 1.0f)) return k;
    }
  }
  return floorf(rate);
}

__global__ void __launch_bounds__(kThreads) k_poisson(P rate, float* __restrict__ out, float* __restrict__ lp,
                                                       int64_t n, uint64_t seed, uint64_t offset, int64_t first) {
  int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = tid; i < n; i += nth) {
    float lam = rate.at(i);
    float v = poisson_draw(lam, seed, (uint64_t)(first + i), offset);
    out[i] = v;
    if (lp) lp[i] = ((v == 0.0f) ? 0.0f : v * logf(lam)) - lam - lgammaf(v + 1.0f);
  }
}

// Bernoulli: 1 if u < p (u uniform in [0, 1) from word 0), so p = 0 never and p = 1 always draws 1
__global__ void __launch_bounds__(kThreads) k_bernoulli(P probs, float* __restrict__ out, float* __restrict__ lp,
                                                         int64_t n, uint64_t seed, uint64_t offset, int64_t first) {
  int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = tid; i < n; i += nth) {
    ppb_philox r = ppb_philox4x32_10(seed, (uint64_t)(first + i), offset);
    const float p = probs.at(i);
    const bool one = ppb_u01(r.c[0]) < p;
    out[i] = one ? 1.0f : 0.0f;
    if (lp) {
      const float pc = ppb_clamp_prob(p);
      lp[i] = one ? logf(pc) : log1pf(-pc);
    }
  }
}

__device__ __forceinline__ int pick_category(const float* __restrict__ p, int C, float u, float* p_sel, float* p_sum) {
  float s = 0.0f;
  for (int c = 0; c < C; ++c) s += __ldg(p + c);
  float target = u * s, run = 0.0f;
  int sel = C - 1;
  for (int c = 0; c < C; ++c) {
    run += __ldg(p + c);
    if (target < run) { sel = c; break; }
  }
  // never return a zero-probability tail category because of rounding
  while (sel > 0 && __ldg(p + sel) <= 0.0f) --sel;
  *p_sel = __ldg(p + sel);
  *p_sum = s;
  return sel;
}

__global__ void __launch_bounds__(kThreads) k_categorical(const float* __restrict__ probs, int64_t row_stride, int C,
                                                           float* __restrict__ out, float* __restrict__ lp, int64_t n,
                                                           uint64_t seed, uint64_t offset, int64_t first) {
  int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = tid; i < n; i += nth) {
    ppb_philox r = ppb_philox4x32_10(seed, (uint64_t)(first + i), offset);
    float ps, sum;
    int sel = pick_category(probs + i * row_stride, C, ppb_u01(r.c[0]), &ps, &sum);
    out[i] = (float)sel;
    if (lp) lp[i] = logf(ppb_clamp_prob(ps / sum));
  }
}

__device__ __forceinline__ float truncnormal_draw(float mu, float sg, float lo, float hi, float u) {
  // inverse-CDF draw (truncated_normal.py:104): icdf(Phi(alpha) + u (Phi(beta)-Phi(alpha))) * sigma + mu
  float ca = ppb_std_normal_cdf((lo - mu) / sg), cb = ppb_std_normal_cdf((hi - mu) / sg);
  float q = ca + u * (cb - ca);
  q = fminf(fmaxf(q, 1e-7f), 1.0f - 6e-8f);
  float v = normcdfinvf(q) * sg + mu;
  // keep the draw inside the truncation domain (the reference retries until it is)
  return fminf(fmaxf(v, lo), hi);
}

template <bool TRUNC>
__global__ void __launch_bounds__(kThreads) k_mixture(const float* __restrict__ means,
                                                       const float* __restrict__ stddevs,
                                                       const float* __restrict__ probs, int64_t row_stride, int K,
                                                       P low, P high, float* __restrict__ out,
                                                       float* __restrict__ lp, int64_t n, uint64_t seed,
                                                       uint64_t offset, int64_t first) {
  int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = tid; i < n; i += nth) {
    ppb_philox r = ppb_philox4x32_10(seed, (uint64_t)(first + i), offset);
    const float* m = means + i * row_stride;
    const float* s = stddevs + i * row_stride;
    const float* p = probs + i * row_stride;
    float ps, psum;
    int k = pick_category(p, K, ppb_u01(r.c[0]), &ps, &psum);
    float mu = __ldg(m + k), sg = __ldg(s + k);
    float lo = 0.f, hi = 0.f, v;
    if (TRUNC) {
      lo = low.at(i); hi = high.at(i);
      v = truncnormal_draw(mu, sg, lo, hi, ppb_u01(r.c[1]));
    } else {
      v = mu + sg * ppb_std_normal_from(r.c[1], r.c[2]);
    }
    out[i] = v;
    if (lp) {
      float mx = -INFINITY, t[32];
      for (int j = 0; j < K; ++j) {
        float lw = logf(ppb_clamp_prob(__ldg(p + j) / psum));
        float mj = __ldg(m + j), sj = __ldg(s + j);
        t[j] = lw + (TRUNC ? ppb_truncnormal_lp(v, mj, sj, lo, hi) : ppb_normal_lp(v, mj, sj));
        mx = fmaxf(mx, t[j]);
      }
      float acc = 0.0f;
      for (int j = 0; j < K; ++j) acc += expf(t[j] - mx);
      lp[i] = (mx == -INFINITY) ? -INFINITY : mx + logf(acc);
    }
  }
}

}  // namespace

extern "C" {

int ppb_normal_sample(const float* mean, int mean_stride, const float* stddev, int stddev_stride, float* value_out,
                      float* lp_out, int64_t n, uint64_t seed, uint64_t offset, int64_t first_index, void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && mean && stddev && value_out, "bad arguments");
  if (n == 0) return PPB_OK;
  k_normal<<<ppb_grid_for(n, kThreads, 1), kThreads, 0, (cudaStream_t)stream>>>(
      P{mean, mean_stride}, P{stddev, stddev_stride}, value_out, lp_out, n, seed, offset, first_index);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int ppb_uniform_sample(const float* low, int low_stride, const float* high, int high_stride, float* value_out,
                       float* lp_out, int64_t n, uint64_t seed, uint64_t offset, int64_t first_index, void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && low && high && value_out, "bad arguments");
  if (n == 0) return PPB_OK;
  k_uniform<<<ppb_grid_for(n, kThreads, 1), kThreads, 0, (cudaStream_t)stream>>>(
      P{low, low_stride}, P{high, high_stride}, value_out, lp_out, n, seed, offset, first_index);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int ppb_poisson_sample(const float* rate, int rate_stride, float* value_out, float* lp_out, int64_t n, uint64_t seed,
                       uint64_t offset, int64_t first_index, void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && rate && value_out, "bad arguments");
  if (n == 0) return PPB_OK;
  k_poisson<<<ppb_grid_for(n, kThreads, 1), kThreads, 0, (cudaStream_t)stream>>>(P{rate, rate_stride}, value_out,
                                                                                 lp_out, n, seed, offset, first_index);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int ppb_bernoulli_sample(const float* probs, int probs_stride, float* value_out, float* lp_out, int64_t n, uint64_t seed,
                         uint64_t offset, int64_t first_index, void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && probs && value_out, "bad arguments");
  PPB_CHECK_ARG((probs_stride | 1) == 1, "strides must be 0 or 1");
  k_bernoulli<<<ppb_grid_for(n, kThreads, 1), kThreads, 0, (cudaStream_t)stream>>>(P{probs, probs_stride}, value_out,
                                                                                   lp_out, n, seed, offset, first_index);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int ppb_categorical_sample(const float* probs, int64_t probs_row_stride, int num_categories, float* value_out,
                           float* lp_out, int64_t n, uint64_t seed, uint64_t offset, int64_t first_index,
                           void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && probs && value_out && num_categories > 0, "bad arguments");
  if (n == 0) return PPB_OK;
  k_categorical<<<ppb_grid_for(n, kThreads, 1), kThreads, 0, (cudaStream_t)stream>>>(
      probs, probs_row_stride, num_categories, value_out, lp_out, n, seed, offset, first_index);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int ppb_mixture_normal_sample(const float* means, const float* stddevs, const float* probs, int64_t row_stride, int K,
                              float* value_out, float* lp_out, int64_t n, uint64_t seed, uint64_t offset,
                              int64_t first_index, void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && means && stddevs && probs && value_out && K > 0 && K <= 32, "bad arguments (K<=32)");
  if (n == 0) return PPB_OK;
  k_mixture<false><<<ppb_grid_for(n, kThreads, 1), kThreads, 0, (cudaStream_t)stream>>>(
      means, stddevs, probs, row_stride, K, P{nullptr, 0}, P{nullptr, 0}, value_out, lp_out, n, seed, offset,
      first_index);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int ppb_mixture_truncated_normal_sample(const float* means, const float* stddevs, const float* probs,
                                        int64_t row_stride, int K, const float* low, int low_stride,
                                        const float* high, int high_stride, float* value_out, float* lp_out,
                                        int64_t n, uint64_t seed, uint64_t offset, int64_t first_index, void* stream) {
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(n >= 0 && means && stddevs && probs && low && high && value_out && K > 0 && K <= 32,
                "bad arguments (K<=32)");
  if (n == 0) return PPB_OK;
  k_mixture<true><<<ppb_grid_for(n, kThreads, 1), kThreads, 0, (cudaStream_t)stream>>>(
      means, stddevs, probs, row_stride, K, P{low, low_stride}, P{high, high_stride}, value_out, lp_out, n, seed,
      offset, first_index);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

}  // extern "C"
