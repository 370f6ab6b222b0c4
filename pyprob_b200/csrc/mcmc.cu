// Metropolis-Hastings chains (LMH / RMH), C chains in lock-step: reference pyprob/model.py:118-178 and
// pyprob/state.py:225-276, :328-336.  One chain is one lane of the lock-step interpreter; its current and candidate traces
// are two rows of per-chain trace tables (value, prior log-prob, step stamp and reuse flag per address column,
// [2, C, lda]).  See include/pyprob_b200.h section 7 for the table format and the Philox rules.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;

struct P {
  const float* p;
  int stride;
  __device__ __forceinline__ float at(int64_t i) const { return stride ? __ldg(p + i) : __ldg(p); }
};

__device__ __forceinline__ int64_t cell(int b, int64_t c, int64_t C, int64_t lda, int col) {
  return ((int64_t)b * C + c) * lda + col;
}

// log(a e^x + (1 - a) e^y) in double, -inf when both terms are -inf
__device__ __forceinline__ double log_mix(double la, double x, double l1a, double y) {
  const double p = la + x, q = l1a + y;
  const double m = fmax(p, q);
  if (m == -INFINITY) return -INFINITY;
  return m + log(exp(p - m) + exp(q - m));
}

// One warp per chain: reset the candidate accumulators and, unless this is the initial step, pick the MH site.
__global__ void __launch_bounds__(kThreads) k_mh_select(const int32_t* __restrict__ stamp,
                                                         const int32_t* __restrict__ buf,
                                                         const int32_t* __restrict__ cur_stamp, int64_t C, int64_t lda,
                                                         int ncols, int32_t* __restrict__ choice,
                                                         int32_t* __restrict__ cand_n, double* __restrict__ cand_lpo,
                                                         double* __restrict__ reuse, double* __restrict__ trans,
                                                         int initial, uint64_t seed, uint64_t offset) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < C; c += warps) {
    int sel = -1;
    if (!initial) {
      const int b = buf[c];
      const int32_t s = cur_stamp[c];
      const int32_t* row = stamp + cell(b, c, C, lda, 0);
      int count = 0;
      for (int a0 = 0; a0 < ncols; a0 += 32) {
        const int a = a0 + lane;
        count += __popc(__ballot_sync(0xffffffffu, a < ncols && row[a] == s));
      }
      if (count > 0) {
        const float u = ppb_u01(ppb_philox4x32_10(seed, (uint64_t)c, offset).c[0]);
        int k = min((int)(u * (float)count), count - 1);
        for (int a0 = 0; a0 < ncols && sel < 0; a0 += 32) {
          const int a = a0 + lane;
          const unsigned m = __ballot_sync(0xffffffffu, a < ncols && row[a] == s);
          const int pc = __popc(m);
          if (k < pc) {
            // the k-th set bit of m: the lane whose prefix count is k
            const bool mine = ((m >> lane) & 1u) && __popc(m & ((1u << lane) - 1u)) == k;
            const unsigned who = __ballot_sync(0xffffffffu, mine);
            sel = a0 + __ffs(who) - 1;
          } else {
            k -= pc;
          }
        }
      }
    }
    if (lane == 0) {
      choice[c] = sel;
      cand_n[c] = 0;
      cand_lpo[c] = 0.0;
      reuse[c] = 0.0;
      trans[c] = 0.0;
    }
  }
}

// Per lane of one executed sample statement: the value the current trace holds at this column, if it has it.
__global__ void __launch_bounds__(kThreads) k_mh_fetch(const float* __restrict__ val, const float* __restrict__ lp,
                                                        const int32_t* __restrict__ stamp,
                                                        const int32_t* __restrict__ buf,
                                                        const int32_t* __restrict__ cur_stamp, int64_t C, int64_t lda,
                                                        int col, const uint8_t* __restrict__ mask, int64_t n,
                                                        int64_t first, float* __restrict__ old_v,
                                                        float* __restrict__ old_lp, uint8_t* __restrict__ has) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t c = first + i;
    const int64_t x = cell(buf[c], c, C, lda, col);
    const bool h = (!mask || mask[i]) && stamp[x] == cur_stamp[c];
    has[i] = h ? 1 : 0;
    old_v[i] = h ? val[x] : 0.0f;
    old_lp[i] = h ? lp[x] : 0.0f;
  }
}

// KIND: 0 = the chosen site draws from the prior (LMH, and RMH for every family but Normal and Uniform);
// 1 = RMH Normal kernel Normal(x_old, prior stddev); 2 = RMH Uniform kernel TruncatedNormal(x_old, 0.1 (high - low),
// low, high).  For KIND 1 / 2, p0 / p1 are the prior's (loc, scale) / (low, high).
template <int KIND>
__global__ void __launch_bounds__(kThreads) k_mh_site(
    int col, const uint8_t* __restrict__ mask, int64_t n, int64_t first, const float* __restrict__ fresh_v,
    const float* __restrict__ fresh_lp, const float* __restrict__ old_v, const float* __restrict__ old_lp,
    const uint8_t* __restrict__ has, const float* __restrict__ rescored, P p0, P p1, float* __restrict__ val,
    float* __restrict__ lp, int32_t* __restrict__ stamp, uint8_t* __restrict__ reused_flag,
    const int32_t* __restrict__ buf, const int32_t* __restrict__ choice, int32_t step, int64_t C, int64_t lda,
    int32_t* __restrict__ cand_n, double* __restrict__ reuse, double* __restrict__ trans,
    int64_t* __restrict__ reused_cnt, float* __restrict__ value_out, uint64_t seed, uint64_t offset) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = fresh_v[i];
    if (mask && !mask[i]) {   // the lane does not execute the statement: the program discards its value
      value_out[i] = v;
      continue;
    }
    const int64_t c = first + i;
    float l = fresh_lp[i];
    bool reused = false;
    if (choice[c] == col) {
      if (KIND != 0) {
        const float xo = old_v[i], lo_old = old_lp[i];
        const ppb_philox r = ppb_philox4x32_10(seed, (uint64_t)c, offset);
        const double la = log(0.5), l1a = log(0.5);
        double q_rev, q_fwd;
        if (KIND == 1) {
          const float mu = p0.at(i), sd = p1.at(i);
          if (ppb_u01(r.c[0]) < 0.5f) v = xo + sd * ppb_std_normal_from(r.c[1], r.c[2]);
          l = ppb_normal_lp(v, mu, sd);
          q_rev = ppb_normal_lp(xo, v, sd);
          q_fwd = ppb_normal_lp(v, xo, sd);
        } else {
          const float a = p0.at(i), b = p1.at(i), s = 0.1f * (b - a);
          if (ppb_u01(r.c[0]) < 0.5f) v = ppb_truncnormal_draw(xo, s, a, b, ppb_u01(r.c[1]));
          l = ((a <= v && b > v) ? 0.0f : -INFINITY) - logf(b - a);
          q_rev = ppb_truncnormal_lp(xo, v, s, a, b);
          q_fwd = ppb_truncnormal_lp(v, xo, s, a, b);
        }
        trans[c] = log_mix(la, q_rev, l1a, (double)lo_old) + (double)l - log_mix(la, q_fwd, l1a, (double)l) -
                   (double)lo_old;
      }
    } else if (has[i] && rescored[i] > -INFINITY) {   // reuse; -inf or NaN (outside the new support) draws fresh
      v = old_v[i];
      l = rescored[i];
      reused = true;
      reuse[c] += (double)l - (double)old_lp[i];
      reused_cnt[c] += 1;
    }
    const int64_t x = cell(1 - buf[c], c, C, lda, col);
    val[x] = v;
    lp[x] = l;
    stamp[x] = step;
    reused_flag[x] = reused ? 1 : 0;
    cand_n[c] += 1;
    value_out[i] = v;
  }
}

// Per chain: log alpha, the accept draw, the buffer flip and the recorded map_func row.
__global__ void __launch_bounds__(kThreads) k_mh_accept(
    int64_t C, int initial, int32_t step, int32_t* __restrict__ buf, int32_t* __restrict__ cur_stamp,
    int32_t* __restrict__ cur_n, double* __restrict__ cur_lpo, const int32_t* __restrict__ cand_n,
    const double* __restrict__ cand_lpo, const double* __restrict__ reuse, const double* __restrict__ trans,
    double* __restrict__ log_alpha, int64_t* __restrict__ accepted, int64_t* __restrict__ sites_all,
    const int32_t* __restrict__ cand_map, int32_t* __restrict__ cur_map, int map_words, int32_t* __restrict__ out,
    int64_t slot, uint64_t seed, uint64_t offset) {
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < C; c += (int64_t)gridDim.x * blockDim.x) {
    const int cn = cand_n[c];
    bool acc;
    if (initial) {
      acc = true;
      log_alpha[c] = 0.0;
    } else {
      double la = -INFINITY;   // a candidate without controlled sites is rejected
      if (cn > 0)
        la = log((double)cur_n[c]) - log((double)cn) + cand_lpo[c] - cur_lpo[c] + reuse[c] + trans[c];
      const float u = ppb_u01_open0(ppb_philox4x32_10(seed, (uint64_t)c, offset).c[0]);
      acc = log((double)u) < la;
      log_alpha[c] = la;
      sites_all[c] += cn;
      if (acc) accepted[c] += 1;
    }
    if (acc) {
      buf[c] ^= 1;
      cur_stamp[c] = step;
      cur_n[c] = cn;
      cur_lpo[c] = cand_lpo[c];
      for (int w = 0; w < map_words; ++w) cur_map[c * map_words + w] = cand_map[c * map_words + w];
    }
    if (slot >= 0)
      for (int w = 0; w < map_words; ++w) out[(slot * C + c) * map_words + w] = cur_map[c * map_words + w];
  }
}

}  // namespace

extern "C" {

int ppb_mh_select(const int32_t* stamp, const int32_t* buf, const int32_t* cur_stamp, int64_t C, int64_t lda, int ncols,
                  int32_t* choice, int32_t* cand_n, double* cand_lpo, double* reuse, double* trans, int initial,
                  uint64_t seed, uint64_t offset, void* stream) {
  PPB_CHECK_ARG(C > 0 && stamp && buf && cur_stamp && choice && cand_n && cand_lpo && reuse && trans, "bad arguments");
  PPB_CHECK_ARG(ncols >= 0 && ncols <= lda, "ncols must be in [0, lda]");
  k_mh_select<<<ppb_grid_for(C * 32, kThreads, 1), kThreads, 0, (cudaStream_t)stream>>>(
      stamp, buf, cur_stamp, C, lda, ncols, choice, cand_n, cand_lpo, reuse, trans, initial, seed, offset);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int ppb_mh_fetch(const float* val, const float* lp, const int32_t* stamp, const int32_t* buf, const int32_t* cur_stamp,
                 int64_t C, int64_t lda, int col, const uint8_t* mask, int64_t n, int64_t first, float* old_v,
                 float* old_lp, uint8_t* has, void* stream) {
  PPB_CHECK_ARG(n > 0 && val && lp && stamp && buf && cur_stamp && old_v && old_lp && has, "bad arguments");
  PPB_CHECK_ARG(col >= 0 && col < lda && first >= 0 && first + n <= C, "column or rows out of range");
  k_mh_fetch<<<ppb_grid_for(n, kThreads, 1), kThreads, 0, (cudaStream_t)stream>>>(
      val, lp, stamp, buf, cur_stamp, C, lda, col, mask, n, first, old_v, old_lp, has);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int ppb_mh_site(int kind, int col, const uint8_t* mask, int64_t n, int64_t first, const float* fresh_v,
                const float* fresh_lp, const float* old_v, const float* old_lp, const uint8_t* has,
                const float* rescored, const float* p0, int p0_stride, const float* p1, int p1_stride, float* val,
                float* lp, int32_t* stamp, uint8_t* reused_flag, const int32_t* buf, const int32_t* choice,
                int32_t step, int64_t C, int64_t lda, int32_t* cand_n, double* reuse, double* trans,
                int64_t* reused_cnt, float* value_out, uint64_t seed, uint64_t offset, void* stream) {
  PPB_CHECK_ARG(n > 0 && fresh_v && fresh_lp && old_v && old_lp && has && rescored && val && lp && stamp &&
                    reused_flag && buf && choice && cand_n && reuse && trans && reused_cnt && value_out,
                "bad arguments");
  PPB_CHECK_ARG(col >= 0 && col < lda && first >= 0 && first + n <= C, "column or rows out of range");
  PPB_CHECK_ARG(kind == 0 || (p0 && p1 && (p0_stride | 1) == 1 && (p1_stride | 1) == 1),
                "RMH kernels need the prior's two parameters (stride 0 or 1)");
  const int grid = ppb_grid_for(n, kThreads, 1);
#define PPB_MH_SITE(K)                                                                                              \
  k_mh_site<K><<<grid, kThreads, 0, (cudaStream_t)stream>>>(                                                        \
      col, mask, n, first, fresh_v, fresh_lp, old_v, old_lp, has, rescored, P{p0, p0_stride}, P{p1, p1_stride}, val, \
      lp, stamp, reused_flag, buf, choice, step, C, lda, cand_n, reuse, trans, reused_cnt, value_out, seed, offset)
  if (kind == PPB_MH_KERNEL_NORMAL) PPB_MH_SITE(1);
  else if (kind == PPB_MH_KERNEL_UNIFORM) PPB_MH_SITE(2);
  else PPB_MH_SITE(0);
#undef PPB_MH_SITE
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int ppb_mh_accept(int64_t C, int initial, int32_t step, int32_t* buf, int32_t* cur_stamp, int32_t* cur_n,
                  double* cur_lpo, const int32_t* cand_n, const double* cand_lpo, const double* reuse,
                  const double* trans, double* log_alpha, int64_t* accepted, int64_t* sites_all,
                  const int32_t* cand_map, int32_t* cur_map, int map_words, int32_t* out, int64_t slot, uint64_t seed,
                  uint64_t offset, void* stream) {
  PPB_CHECK_ARG(C > 0 && buf && cur_stamp && cur_n && cur_lpo && cand_n && cand_lpo && reuse && trans && log_alpha &&
                    accepted && sites_all && cand_map && cur_map && map_words > 0,
                "bad arguments");
  PPB_CHECK_ARG(slot < 0 || out, "a recorded step needs the output buffer");
  k_mh_accept<<<ppb_grid_for(C, kThreads, 1), kThreads, 0, (cudaStream_t)stream>>>(
      C, initial, step, buf, cur_stamp, cur_n, cur_lpo, cand_n, cand_lpo, reuse, trans, log_alpha, accepted, sites_all,
      cand_map, cur_map, map_words, out, slot, seed, offset);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

}  // extern "C"
