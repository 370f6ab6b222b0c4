// Samplers over the particle axis (Philox4x32-10, counter = (global particle index, offset)).
// Replaces pyprob/distributions/distribution.py:31-36, mixture.py:47-63, truncated_normal.py:94-112.
// Fused sample+score: lp_out (nullable) gets log_prob of the drawn value (pyprob/state.py:196-197); for the eleven
// element-wise families that is the scoring kernels' value, through the Ops of families.cuh.
// Event draws (k_event_sample, [n, D]): element j of particle i uses Philox index (first + i) | (j << 40) and the usual
// offset + (round << 40) for rejection rounds, so particle indices must stay below 2^40 and D at most 2^24 (checked
// before launch); element 0 is the per-particle draw, and a shard of the particles draws the full run's rows.
#include "common.cuh"
#include "families.cuh"

namespace {

constexpr int kThreads = 256;

struct P {
  const float* p;
  int stride;
  __device__ __forceinline__ float at(int64_t i) const { return stride ? __ldg(p + i) : __ldg(p); }
};

// The draw of each family from Philox counter (idx, offset [+ (round << 40)]), shared by the per-particle sampler (k_sample)
// and the event sampler (k_event_sample), so that element 0 of an event row is the per-particle draw bit for bit.
// The single-counter families take the Philox words of (idx, offset).
__device__ __forceinline__ float normal_draw(const ppb_philox& r, float mu, float s) {
  float z = ppb_std_normal_from(r.c[0], r.c[1]);
  return mu + s * z;
}

__device__ __forceinline__ float uniform_draw(const ppb_philox& r, float lo, float hi) {
  float v = lo + ppb_u01(r.c[0]) * (hi - lo);
  // u < 1, but the fp32 sum can round up onto hi (Uniform(1000, 1001): every u above 1 - 3.05e-5), which log_prob
  // scores -inf: step such a draw to the largest float below hi
  if (v >= hi) v = nextafterf(hi, lo);
  return v;
}

// Poisson: inversion by sequential search for rate < 10 (Devroye), PTRS transformed rejection
// (W. Hoermann 1993) for rate >= 10; the rejection loop draws fresh Philox words with a bumped counter.
// PTRS runs in double, as torch's CPU sampler does: its log acceptance ratio -rate + k log(rate) - lgamma(k + 1) is a
// difference of terms near rate log(rate), and in fp32 (spacing 0.125 at 1e6) it is off by tenths from rate 1e5 up, which
// skews the distribution (variance 1.05 rate at 1e6).  The draw is returned as a float: exact integers up to 2^24, so rates
// much above 1e7 are not supported.
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
  const double lam = rate, slam = sqrt(lam), loglam = log(lam);
  const double b = 0.931 + 2.53 * slam;
  const double a = -0.059 + 0.02483 * b;
  const double invalpha = 1.1239 + 1.1328 / (b - 3.4);
  const double vr = 0.9277 - 3.6224 / (b - 2.0);
  for (uint64_t sub = 0; sub < 64; ++sub) {
    ppb_philox r = ppb_philox4x32_10(seed, idx, offset + (sub << 40));
    for (int j = 0; j < 4; j += 2) {
      const double U = (double)ppb_u01(r.c[j]) - 0.5;
      const double V = ppb_u01_open0(r.c[j + 1]);
      const double us = 0.5 - fabs(U);
      const double k = floor((2.0 * a / us + b) * U + lam + 0.43);
      if (us >= 0.07 && V <= vr) return (float)k;
      if (k < 0.0 || (us < 0.013 && V > us)) continue;
      if (log(V * invalpha / (a / (us * us) + b)) <= -lam + k * loglam - lgamma(k + 1.0)) return (float)k;
    }
  }
  return floorf(rate);
}

// Bernoulli: 1 if u < p (u uniform in [0, 1) from word 0), so p = 0 never and p = 1 always draws 1
__device__ __forceinline__ bool bernoulli_one(const ppb_philox& r, float p) {
  return ppb_u01(r.c[0]) < p;
}

// uniform in (0, 1), open at both ends: the inversions below take logs of u and of 1 - u
__device__ __forceinline__ float u01_open(uint32_t x) { return ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f); }
// uniform in [0, 1) with 53 random bits from two words
__device__ __forceinline__ double u01_double(uint32_t a, uint32_t b) {
  return (double)((((uint64_t)a << 32) | b) >> 11) * (1.0 / 9007199254740992.0);
}
__device__ __forceinline__ ppb_philox philox_sub(uint64_t seed, uint64_t idx, uint64_t offset, uint64_t sub) {
  return ppb_philox4x32_10(seed, idx, offset + (sub << 40));   // fresh words for rejection rounds, as poisson_draw
}

// Exponential: inversion, -log(u) / rate
__device__ __forceinline__ float exponential_draw(const ppb_philox& r, float lam) {
  return (lam > 0.0f) ? -logf(u01_open(r.c[0])) / lam : NAN;
}

// log of a standard Gamma(c) draw.  Marsaglia & Tsang (2000) for c >= 1; c < 1 as G(c + 1) U^(1/c), with the power
// taken in log space.  Sub-counters sub0 .. sub0 + kGammaCalls - 1 feed the rounds, sub0 + kGammaCalls the boost uniform.
// Each Philox call gives two attempts (Box-Muller's cosine and sine normals, two uniforms).  The acceptance rate is
// lowest at c = 1, 0.952, so all 2 * kGammaCalls = 16 attempts fail with probability below 0.048^16 < 1e-20 per draw;
// the draw then falls back to log(d), deterministically.
constexpr uint64_t kGammaCalls = 8;
__device__ float std_gamma_log(float c, uint64_t seed, uint64_t idx, uint64_t offset, uint64_t sub0) {
  const bool boost = c < 1.0f;
  const float d = (boost ? c + 1.0f : c) - 1.0f / 3.0f;
  const float cc = 1.0f / sqrtf(9.0f * d);
  float lg = logf(d);
  bool done = false;
  for (uint64_t k = 0; k < kGammaCalls && !done; ++k) {
    const ppb_philox r = philox_sub(seed, idx, offset, sub0 + k);
    const float rad = sqrtf(-2.0f * logf(ppb_u01_open0(r.c[0])));
    float sn, cs;
    sincospif(2.0f * ppb_u01(r.c[1]), &sn, &cs);
    const float z[2] = {rad * cs, rad * sn};
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const float t = 1.0f + cc * z[j];
      if (done || t <= 0.0f) continue;
      const float v = t * t * t, x2 = z[j] * z[j], u = ppb_u01_open0(r.c[2 + j]);
      if (u < 1.0f - 0.0331f * x2 * x2 || logf(u) < 0.5f * x2 + d * (1.0f - v + logf(v))) {
        lg = logf(d * v);
        done = true;
      }
    }
  }
  if (boost) lg += logf(ppb_u01_open0(philox_sub(seed, idx, offset, sub0 + kGammaCalls).c[0])) / c;
  return lg;
}

// Gamma: standard draw / rate, clamped below at the smallest normal float as torch's Gamma.rsample does (no draw is 0)
__device__ __forceinline__ float gamma_draw(float c, float rt, uint64_t seed, uint64_t idx, uint64_t offset) {
  float v = NAN;
  if (c > 0.0f && rt > 0.0f)
    v = fmaxf(expf(std_gamma_log(c, seed, idx, offset, 0) - logf(rt)), PPB_FLT_TINY);
  return v;
}

// LogNormal: exp of the Box-Muller normal that normal_draw draws
__device__ __forceinline__ float lognormal_draw(const ppb_philox& r, float mu, float s) {
  return (s > 0.0f) ? expf(mu + s * ppb_std_normal_from(r.c[0], r.c[1])) : NAN;
}

// Weibull: scale (-log u)^(1/k), kept above 0 (the support) where the power underflows
__device__ __forceinline__ float weibull_draw(const ppb_philox& r, float lam, float k) {
  return (lam > 0.0f && k > 0.0f) ? fmaxf(lam * powf(-logf(u01_open(r.c[0])), 1.0f / k), PPB_FLT_TINY) : NAN;
}

// Beta: Ga / (Ga + Gb) from two standard Gamma draws on disjoint sub-counters, as 1 / (1 + exp(log Gb - log Ga)) so that
// neither draw underflows; clamped to [tiny, 1 - eps] as torch's Dirichlet sampler clamps; then low + u (high - low)
__device__ __forceinline__ float beta_draw(float a, float b, float lo, float hi, uint64_t seed, uint64_t idx,
                                           uint64_t offset) {
  float v = NAN;
  if (a > 0.0f && b > 0.0f) {
    const float la = std_gamma_log(a, seed, idx, offset, 0);
    const float lb = std_gamma_log(b, seed, idx, offset, kGammaCalls + 1);
    const float u = fminf(fmaxf(1.0f / (1.0f + expf(lb - la)), PPB_FLT_TINY), 1.0f - PPB_EPS32);
    v = lo + u * (hi - lo);
  }
  return v;
}

// Binomial, drawn for q = min(p, 1 - p) and mirrored (n - k) for p > 1/2.
//  * n q < 10: inversion by sequential search from k = 0 with one 53-bit uniform.  The mean is below 10, so
//    P(X > 110) < 1e-60: the search stops there (and at n).
//  * n q >= 10: BTRS, transformed rejection with squeeze (W. Hoermann 1993, "The generation of binomial random variates"),
//    the acceptance test on exact log-factorials in double precision.  Two attempts per Philox call.  The acceptance
//    rate is lowest at n q = 10, q = 1/2: 0.71, so all 2 * kBtrsCalls = 32 attempts fail with probability below
//    0.29^32 < 1e-17 per draw; the draw then falls back to the mode, deterministically.
constexpr uint64_t kBtrsCalls = 16;
__device__ float binomial_draw(float nf, float p, uint64_t seed, uint64_t idx, uint64_t offset) {
  if (!fam::binomial_args_ok(nf, p)) return NAN;
  if (nf == 0.0f || p == 0.0f) return 0.0f;
  if (p == 1.0f) return nf;
  const bool flip = p > 0.5f;
  const double n = nf, q = flip ? 1.0 - (double)p : (double)p;
  double k;
  if (n * q < 10.0) {
    const ppb_philox r = ppb_philox4x32_10(seed, idx, offset);
    double u = u01_double(r.c[0], r.c[1]);
    double f = exp(n * log1p(-q));    // P(X = 0)
    const double s = q / (1.0 - q), kmax = fmin(n, 110.0);
    k = 0.0;
    while (u >= f && k < kmax) {
      u -= f;
      f *= (n - k) / (k + 1.0) * s;
      k += 1.0;
    }
  } else {
    const double spq = sqrt(n * q * (1.0 - q));
    const double b = 1.15 + 2.53 * spq, a = -0.0873 + 0.0248 * b + 0.01 * q, c = n * q + 0.5;
    const double alpha = (2.83 + 5.1 / b) * spq, vr = 0.92 - 4.2 / b;
    const double m = floor((n + 1.0) * q), lpq = log(q / (1.0 - q));
    const double h = lgamma(m + 1.0) + lgamma(n - m + 1.0);
    k = m;
    bool done = false;
    for (uint64_t call = 0; call < kBtrsCalls && !done; ++call) {
      const ppb_philox r = philox_sub(seed, idx, offset, call);
#pragma unroll
      for (int j = 0; j < 4; j += 2) {
        if (done) continue;
        const double U = (double)ppb_u01(r.c[j]) - 0.5, V = ppb_u01(r.c[j + 1]);
        const double us = 0.5 - fabs(U);
        const double kk = floor((2.0 * a / us + b) * U + c);
        if (!(kk >= 0.0 && kk <= n)) continue;
        if ((us >= 0.07 && V <= vr) ||
            log(V * alpha / (a / (us * us) + b)) <= h - lgamma(kk + 1.0) - lgamma(n - kk + 1.0) + (kk - m) * lpq) {
          k = kk;
          done = true;
        }
      }
    }
  }
  return (float)(flip ? n - k : k);
}

// VonMises: Best & Fisher (1979) rejection, in double precision as torch's VonMises.sample runs it (kappa (r - f)
// cancels in fp32 at large kappa), then wrapped as torch does: (x + pi + loc) mod 2 pi - pi.  One round per Philox call.
// The acceptance rate falls with kappa towards 0.658, so all kVonMisesCalls = 32 rounds fail with probability below
// 0.343^32 < 1e-14 per draw; the draw then falls back to loc, deterministically.
constexpr uint64_t kVonMisesCalls = 32;
__device__ __forceinline__ float von_mises_draw(float locf, float kf, uint64_t seed, uint64_t idx, uint64_t offset) {
  const double kPi = 3.14159265358979323846;
  float v = NAN;
  if (kf > 0.0f) {
    const double kappa = kf;
    const double tau = 1.0 + sqrt(1.0 + 4.0 * kappa * kappa);
    const double rho = (tau - sqrt(2.0 * tau)) / (2.0 * kappa);
    const double pr = (kappa < 1e-5) ? 1.0 / kappa + kappa : (1.0 + rho * rho) / (2.0 * rho);
    double x = 0.0;
    for (uint64_t call = 0; call < kVonMisesCalls; ++call) {
      const ppb_philox r = philox_sub(seed, idx, offset, call);
      const double u1 = ppb_u01(r.c[0]), u2 = ppb_u01(r.c[1]), u3 = ppb_u01(r.c[2]);
      const double z = cospi(u1);
      const double f = fmin(fmax((1.0 + pr * z) / (pr + z), -1.0), 1.0);
      const double c = kappa * (pr - f);
      if (c * (2.0 - c) - u2 > 0.0 || log(c / u2) + 1.0 - c >= 0.0) {
        x = (u3 > 0.5 ? 1.0 : u3 < 0.5 ? -1.0 : 0.0) * acos(f);
        break;
      }
    }
    const double y = x + kPi + (double)locf, two_pi = 2.0 * kPi;
    v = (float)(y - two_pi * floor(y / two_pi) - kPi);
  }
  return v;
}

// The draw of family FAMILY with parameters p (the PPB_EVENT_* order) from Philox index idx
template <int FAMILY>
__device__ __forceinline__ float family_draw(const float (&p)[4], uint64_t seed, uint64_t idx, uint64_t offset) {
  switch (FAMILY) {
    case PPB_EVENT_NORMAL: return normal_draw(ppb_philox4x32_10(seed, idx, offset), p[0], p[1]);
    case PPB_EVENT_UNIFORM: return uniform_draw(ppb_philox4x32_10(seed, idx, offset), p[0], p[1]);
    case PPB_EVENT_POISSON: return poisson_draw(p[0], seed, idx, offset);
    case PPB_EVENT_BERNOULLI: return bernoulli_one(ppb_philox4x32_10(seed, idx, offset), p[0]) ? 1.0f : 0.0f;
    case PPB_EVENT_EXPONENTIAL: return exponential_draw(ppb_philox4x32_10(seed, idx, offset), p[0]);
    case PPB_EVENT_GAMMA: return gamma_draw(p[0], p[1], seed, idx, offset);
    case PPB_EVENT_LOGNORMAL: return lognormal_draw(ppb_philox4x32_10(seed, idx, offset), p[0], p[1]);
    case PPB_EVENT_WEIBULL: return weibull_draw(ppb_philox4x32_10(seed, idx, offset), p[0], p[1]);
    case PPB_EVENT_BETA: return beta_draw(p[0], p[1], p[2], p[3], seed, idx, offset);
    case PPB_EVENT_BINOMIAL: return binomial_draw(p[0], p[1], seed, idx, offset);
    default: return von_mises_draw(p[0], p[1], seed, idx, offset);
  }
}

// The eleven element-wise families at D = 1: particle i draws from Philox index first + i, and lp_out is the Op's value.
struct Operands {
  P p[4];
};

template <class Op>
__global__ void __launch_bounds__(kThreads) k_sample(Operands q, float* __restrict__ out, float* __restrict__ lp,
                                                      int64_t n, uint64_t seed, uint64_t offset, int64_t first) {
  __shared__ float tab[Op::kTable ? 64 : 1];
  if (Op::kTable) {
    if (threadIdx.x < 64) tab[threadIdx.x] = c_log_factorial[threadIdx.x];
    __syncthreads();
  }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float p[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) p[k] = q.p[k < Op::kParams ? k : 0].at(i);
    const float v = family_draw<Op::kFamily>(p, seed, (uint64_t)(first + i), offset);
    out[i] = v;
    if (lp) lp[i] = Op{}(v, p, tab);   // a fresh Op: the draw dominates, and a parameter-only term kept across
                                       // particles would only hold registers
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
      v = ppb_truncnormal_draw(mu, sg, lo, hi, ppb_u01(r.c[1]));
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

// ---- event sampler: [n, D] draws ------------------------------------------------------------------------------------------
// Philox counter layout.  Element j of particle i (global index g = first + i) draws from idx = g | (j << 40), with the
// family's rejection rounds in offset + (round << 40) as above:
//   * idx bits 0 .. 39 hold the particle (g < 2^40) and bits 40 .. 63 the element (j < 2^24), so no (particle, element)
//     pair shares idx, and the rounds of one pair differ in offset: no (particle, element, round) triple shares a counter;
//   * element 0 has idx = g, the per-particle samplers' counter, so it is their draw bit for bit;
//   * the counter depends on the global index only, so a shard [a, b) of the particles draws the full run's rows.
// ppb_event_sample rejects D > 2^24 and first_index + n > 2^40 before launch.
struct EvP {
  const float* p;
  int64_t ps, es;
  __device__ __forceinline__ float at(int64_t i, int64_t j) const { return p ? __ldg(p + i * ps + j * es) : 0.0f; }
};

template <class Op>
__global__ void __launch_bounds__(kThreads) k_event_sample(EvP p0, EvP p1, EvP p2, EvP p3, float* __restrict__ out,
                                                            int64_t n, int64_t D, uint64_t seed, uint64_t offset,
                                                            int64_t first) {
  const int64_t total = n * D;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / D, j = e - i * D;
    const uint64_t idx = (uint64_t)(first + i) | ((uint64_t)j << 40);
    const float p[4] = {p0.at(i, j), p1.at(i, j), Op::kParams > 2 ? p2.at(i, j) : 0.0f,
                        Op::kParams > 2 ? p3.at(i, j) : 0.0f};
    out[e] = family_draw<Op::kFamily>(p, seed, idx, offset);
  }
}

}  // namespace

extern "C" {

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

namespace {

int event_sample(int family, const float* const* p, const int64_t* ps, const int64_t* es, float* value_out,
                 float* lp_out, int64_t n, int64_t D, uint64_t seed, uint64_t offset, int64_t first_index,
                 void* stream) {
  const int np = ppb_event_num_params(family);
  PPB_CHECK_ARG(np > 0, "unknown family id");
  PPB_CHECK_ARG(n >= 0 && D > 0, "n must be >= 0 and D > 0");
  PPB_CHECK_ARG(D <= ((int64_t)1 << 24), "D > 2^24: the element index does not fit Philox counter bits 40 .. 63");
  PPB_CHECK_ARG(first_index >= 0 && first_index + n <= ((int64_t)1 << 40),
                "first_index + n > 2^40: the particle index does not fit Philox counter bits 0 .. 39");
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(value_out, "value_out is null");
  EvP q[4] = {};
  for (int k = 0; k < np; ++k) {
    PPB_CHECK_ARG(p[k] && ((ps[k] == 0 && es[k] == 0) || (ps[k] == 1 && es[k] == 0) || (ps[k] == 0 && es[k] == 1) ||
                           (ps[k] == D && es[k] == 1)),
                  "parameter: null pointer, or strides not one of (0, 0), (1, 0), (0, 1), (D, 1)");
    q[k] = EvP{p[k], ps[k], es[k]};
  }
  cudaStream_t st = (cudaStream_t)stream;
  return ppb_with_family(family, [&](auto op) {
    using Op = decltype(op);
    if (D == 1) {   // one draw per particle, its log_prob fused (every operand is flat with stride ps, 0 or 1)
      if (Op::kTable && lp_out) {
        const int e = ppb_upload_log_factorial();
        if (e != PPB_OK) return e;
      }
      Operands f;
      for (int k = 0; k < 4; ++k) f.p[k] = P{q[k].p, (int)q[k].ps};
      k_sample<Op><<<ppb_grid_for(n, kThreads, 1), kThreads, 0, st>>>(f, value_out, lp_out, n, seed, offset,
                                                                        first_index);
      PPB_LAUNCH_CHECK();
      return PPB_OK;
    }
    k_event_sample<Op><<<ppb_grid_for(n * D, kThreads, 1), kThreads, 0, st>>>(q[0], q[1], q[2], q[3], value_out, n, D,
                                                                                seed, offset, first_index);
    PPB_LAUNCH_CHECK();
    if (!lp_out) return PPB_OK;
    // lp_out: the scoring kernel's row sums over the drawn rows (value operand (D, 1))
    return ppb_event_score(family, value_out, D, 1, p, ps, es, n, D, nullptr, lp_out, nullptr, 0.0, stream);
  });
}

}  // namespace

extern "C" {

int ppb_event_sample(int family, const float* p0, int64_t p0_ps, int64_t p0_es, const float* p1, int64_t p1_ps,
                     int64_t p1_es, const float* p2, int64_t p2_ps, int64_t p2_es, const float* p3, int64_t p3_ps,
                     int64_t p3_es, float* value_out, float* lp_out, int64_t n, int64_t D, uint64_t seed,
                     uint64_t offset, int64_t first_index, void* stream) {
  const float* p[4] = {p0, p1, p2, p3};
  const int64_t ps[4] = {p0_ps, p1_ps, p2_ps, p3_ps}, es[4] = {p0_es, p1_es, p2_es, p3_es};
  return event_sample(family, p, ps, es, value_out, lp_out, n, D, seed, offset, first_index, stream);
}

int ppb_event_sample_d1(int family, const float* p0, const float* p1, const float* p2, const float* p3,
                        int param_strides, float* value_out, float* lp_out, int64_t n, uint64_t seed, uint64_t offset,
                        int64_t first_index, void* stream) {
  const float* p[4] = {p0, p1, p2, p3};
  const int64_t ps[4] = {param_strides & 1, (param_strides >> 1) & 1, (param_strides >> 2) & 1,
                         (param_strides >> 3) & 1};
  const int64_t es[4] = {0, 0, 0, 0};
  return event_sample(family, p, ps, es, value_out, lp_out, n, 1, seed, offset, first_index, stream);
}

}  // extern "C"
