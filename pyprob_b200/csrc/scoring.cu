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

// ---- the eleven element-wise families at D = 1: one particle-flat kernel over the Ops of families.cuh ---------------------
// The value and each of the Op::kParams parameters is a scalar (stride 0) or one per particle (stride 1).
struct Operands {
  Param p[4];
};

template <class Op, bool VEC>
__global__ void __launch_bounds__(kThreads) k_score2(Param value, Operands q, Sink out, int64_t n, Op op) {
  __shared__ float tab[Op::kTable ? 64 : 1];
  if (Op::kTable) {
    if (threadIdx.x < 64) tab[threadIdx.x] = c_log_factorial[threadIdx.x];
    __syncthreads();
  }
  int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t nth = (int64_t)gridDim.x * blockDim.x;
  int64_t i0 = 0;
  if (VEC) {
    int64_t n4 = n >> 2;
    for (int64_t q4 = tid; q4 < n4; q4 += nth) {
      int64_t i = q4 << 2;
      const float4 vv = ldg_stream4(value.p + i);   // VEC: the value is one per particle
      const float v[4] = {vv.x, vv.y, vv.z, vv.w};
      float p[Op::kParams][4], r[4];
#pragma unroll
      for (int k = 0; k < Op::kParams; ++k) q.p[k].load4(i, p[k]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float pj[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) pj[k] = p[k < Op::kParams ? k : 0][j];
        r[j] = op(v[j], pj, tab);
      }
      out.put4(i, r);
    }
    i0 = n4 << 2;
  }
  for (int64_t i = i0 + tid; i < n; i += nth) {
    float p[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) p[k] = q.p[k < Op::kParams ? k : 0].at(i);
    out.put(i, op(value.at(i), p, tab));
  }
}

template <class Op>
int launch_score2(Param value, const Operands& q, Sink out, int64_t n, cudaStream_t st) {
  bool vec = value.stride == 1 && value.vec_ok() && out.vec_ok();
  for (int k = 0; k < Op::kParams; ++k) vec = vec && q.p[k].vec_ok();
  const int grid = ppb_grid_for(n, kThreads, 4);
  if (vec)
    k_score2<Op, true><<<grid, kThreads, 0, st>>>(value, q, out, n, Op{});
  else
    k_score2<Op, false><<<grid, kThreads, 0, st>>>(value, q, out, n, Op{});
  PPB_LAUNCH_CHECK();
  return PPB_OK;
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
// bit-reproducible.  Each element is the Op's value, as k_score2 gives it for a particle; ppb_event_score runs D = 1 on
// k_score2, whose accumulator update is this kernel's at D = 1 (the fp64 sum of a single term).
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

template <class Op, int G>
__global__ void __launch_bounds__(kThreads) k_event(EvArgs a, Op op) {
  constexpr int NP = Op::kParams;
  __shared__ float tab[Op::kTable ? 64 : 1];
  if (Op::kTable) {
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
          r[e] = op(v[e], pe, tab);
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

template <class Op>
int launch_event(const EvArgs& a, cudaStream_t st) {
  const int64_t chunks = (a.D + 3) >> 2;
  int g = 1;
  while (g < chunks && g < 32) g <<= 1;
  const int grid = ppb_grid_for(a.n, kThreads / g, 1);
  switch (g) {
    case 1: k_event<Op, 1><<<grid, kThreads, 0, st>>>(a, Op{}); break;
    case 2: k_event<Op, 2><<<grid, kThreads, 0, st>>>(a, Op{}); break;
    case 4: k_event<Op, 4><<<grid, kThreads, 0, st>>>(a, Op{}); break;
    case 8: k_event<Op, 8><<<grid, kThreads, 0, st>>>(a, Op{}); break;
    case 16: k_event<Op, 16><<<grid, kThreads, 0, st>>>(a, Op{}); break;
    default: k_event<Op, 32><<<grid, kThreads, 0, st>>>(a, Op{}); break;
  }
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

bool ev_layout_ok(const void* p, int64_t ps, int64_t es, int64_t D) {
  return p && ((ps == 0 && es == 0) || (ps == 1 && es == 0) || (ps == 0 && es == 1) || (ps == D && es == 1));
}

}  // namespace

int ppb_event_score(int family, const float* value, int64_t value_ps, int64_t value_es, const float* const* params,
                    const int64_t* params_ps, const int64_t* params_es, int64_t n, int64_t D, float* lp_out,
                    float* row_lp, double* acc, double acc_scale, void* stream) {
  const int np = ppb_event_num_params(family);
  PPB_CHECK_ARG(np > 0, "unknown family id");
  PPB_CHECK_ARG(n >= 0 && D > 0, "n must be >= 0 and D > 0");
  PPB_CHECK_ARG(D > 1 || !row_lp, "row_lp at D = 1: a row's sum is its one element, lp_out");
  if (n == 0) return PPB_OK;
  PPB_CHECK_ARG(ev_layout_ok(value, value_ps, value_es, D),
                "value: null pointer, or strides not one of (0, 0), (1, 0), (0, 1), (D, 1)");
  EvArgs a{EvOperand{value, value_ps, value_es}, {}, lp_out, row_lp, acc, acc_scale, n, D};
  for (int k = 0; k < np; ++k) {
    PPB_CHECK_ARG(ev_layout_ok(params[k], params_ps[k], params_es[k], D),
                  "parameter: null pointer, or strides not one of (0, 0), (1, 0), (0, 1), (D, 1)");
    a.p[k] = EvOperand{params[k], params_ps[k], params_es[k]};
  }
  cudaStream_t st = (cudaStream_t)stream;
  return ppb_with_family(family, [&](auto op) {
    using Op = decltype(op);
    if (Op::kTable) {
      const int e = ppb_upload_log_factorial();
      if (e != PPB_OK) return e;
    }
    if (D > 1) return launch_event<Op>(a, st);
    // D = 1: every operand is flat with stride ps (0 or 1), and each row one particle's element
    Operands q;
    for (int k = 0; k < 4; ++k) q.p[k] = Param{a.p[k].p, (int)a.p[k].ps};
    return launch_score2<Op>(Param{value, (int)value_ps}, q, Sink{lp_out, acc, acc_scale}, n, st);
  });
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

int ppb_event_log_prob_d1(int family, const float* value, const float* p0, const float* p1, const float* p2,
                          const float* p3, int param_strides, float* lp_out, double* acc, double acc_scale, int64_t n,
                          void* stream) {
  const float* p[4] = {p0, p1, p2, p3};
  const int64_t ps[4] = {param_strides & 1, (param_strides >> 1) & 1, (param_strides >> 2) & 1,
                         (param_strides >> 3) & 1};
  const int64_t es[4] = {0, 0, 0, 0};
  return ppb_event_score(family, value, 1, 0, p, ps, es, n, 1, lp_out, nullptr, acc, acc_scale, stream);
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
