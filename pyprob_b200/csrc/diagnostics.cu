// MCMC convergence diagnostics over C chains of S steps and V variables: Gelman-Rubin R-hat against the prefix length and
// per-chain autocorrelation (reference pyprob/diagnostics.py:714-873).  See include/pyprob_b200.h section 8 and DESIGN.md
// sections 4 and 8.
//
// The values are x[s, c, v] at s * stride_s + c * stride_c + v * stride_v, fp32 or fp64; column j = c * V + v is one
// chain of one variable.  Everything is fp64 and reduced in a fixed order (no atomics), so two calls give the same bits.
// Means and variances are never formed as sum(x^2) - sum(x)^2 / n: a segment's (count, mean, M2) is built from chunks of
// 8 steps centred on their first value, and statistics meet through Chan's parallel formula.  A constant chain therefore
// has mean exactly its value and M2 exactly 0.
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kFinThreads = 128;
constexpr int kChunk = 8;           // steps per Welford chunk in the segment kernel
constexpr int kTile = 128;          // steps per shared-memory tile in the autocorrelation kernel
constexpr int kLagWarps = kThreads / 32;
constexpr int64_t kTargetThreads = 1 << 17;   // segment-kernel threads to aim for when there are few chains
constexpr int64_t kMaxSegments = 1024;        // uniform segments per column at most
constexpr int64_t kMinSegment = 64;           // steps per uniform segment at least
constexpr int64_t kRhatStatBudget = int64_t(256) << 20;     // bytes of R-hat segment statistics cut at boundaries
constexpr int64_t kAcfTargetBlocks = 8 * PPB_NUM_SMS;
constexpr int64_t kAcfResident = (2048 / kThreads) * PPB_NUM_SMS;   // autocorrelation blocks resident at once, at most
constexpr int64_t kAcfL2Budget = int64_t(24) << 20;          // bytes of series the resident column tiles may span
constexpr int64_t kAcfPartialBudget = int64_t(1) << 30;      // bytes of per-chunk autocorrelation partials at most
constexpr double kEpsilon = 1e-8;   // pyprob/util.py:34 _epsilon, the reference's autocorrelation denominator floor

__constant__ double kRcp[kChunk + 1] = {0.0, 1.0, 1.0 / 2, 1.0 / 3, 1.0 / 4, 1.0 / 5, 1.0 / 6, 1.0 / 7, 1.0 / 8};

struct Stat {
  double n, mean, m2;
};

// Chan et al.: the statistics of the union of two disjoint sets.  Exact passthrough when either side is empty, and the
// mean does not move when both means are equal.
__device__ __forceinline__ Stat chan(Stat a, Stat b) {
  if (b.n == 0.0) return a;
  if (a.n == 0.0) return b;
  const double n = a.n + b.n, d = b.mean - a.mean;
  return Stat{n, a.mean + d * (b.n / n), a.m2 + b.m2 + d * d * (a.n * (b.n / n))};
}

template <typename T>
__device__ __forceinline__ double ld(const T* x, int64_t i) {
  return (double)__ldg(x + i);
}

struct Geom {
  int64_t S, C, V, ss, sc, sv;
  __device__ __forceinline__ int64_t base(int64_t j) const { return (j / V) * sc + (j % V) * sv; }
};

// (count, mean, M2) of x[a .. b) of one column (p = its first element, ss = the step stride), from chunks of 8 steps
// centred on their first value: a constant chunk has mean v[0] and M2 0 exactly.
template <typename T>
__device__ __forceinline__ Stat range_stat(const T* p, int64_t ss, int64_t a, int64_t b) {
  Stat s{0.0, 0.0, 0.0};
  for (int64_t i0 = a; i0 < b; i0 += kChunk) {
    const int cnt = (int)min((int64_t)kChunk, b - i0);
    double v[kChunk];
#pragma unroll
    for (int u = 0; u < kChunk; ++u) v[u] = u < cnt ? ld(p, (i0 + u) * ss) : 0.0;
    double sum = 0.0;
#pragma unroll
    for (int u = 1; u < kChunk; ++u) sum += u < cnt ? v[u] - v[0] : 0.0;
    const double mc = v[0] + sum * kRcp[cnt];
    double q = 0.0;
#pragma unroll
    for (int u = 0; u < kChunk; ++u) {
      const double d = v[u] - mc;
      q += u < cnt ? d * d : 0.0;
    }
    s = chan(s, Stat{(double)cnt, mc, q});
  }
  return s;
}

// One thread per (column j, segment g), j fastest: (count, mean, M2) of x[seg_begin .. seg_end) of column j, written to
// mean[g * cols + j], m2[g * cols + j].  Threads of a warp read adjacent columns of the same step.
template <typename T>
__global__ void __launch_bounds__(kThreads) k_seg_stats(const T* __restrict__ x, Geom gm,
                                                         const int64_t* __restrict__ seg_end, int64_t G,
                                                         double* __restrict__ mean, double* __restrict__ m2) {
  const int64_t cols = gm.C * gm.V;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < G * cols; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t g = t / cols, j = t - g * cols;
    const Stat s = range_stat(x + gm.base(j), gm.ss, g ? seg_end[g - 1] : 0, seg_end[g]);
    mean[g * cols + j] = s.mean;
    m2[g * cols + j] = s.m2;
  }
}

__device__ __forceinline__ Stat seg_stat(const int64_t* seg_end, const double* mean, const double* m2, int64_t g,
                                         int64_t cols, int64_t j) {
  const int64_t a = g ? seg_end[g - 1] : 0;
  return Stat{(double)(seg_end[g] - a), mean[g * cols + j], m2[g * cols + j]};
}

// Cross-chain partial of one boundary: the chain means' (count, mean, M2) and the sum of the chain variances.
struct Part {
  Stat m;
  double sv;
};

__device__ __forceinline__ Part part_combine(Part a, Part b) { return Part{chan(a.m, b.m), a.sv + b.sv}; }

__device__ __forceinline__ Part shfl_down(Part p, int off) {
  return Part{Stat{__shfl_down_sync(0xffffffffu, p.m.n, off), __shfl_down_sync(0xffffffffu, p.m.mean, off),
                   __shfl_down_sync(0xffffffffu, p.m.m2, off)},
              __shfl_down_sync(0xffffffffu, p.sv, off)};
}

// Fixed-shape block reduction (shuffle tree per warp, then warp 0 over the warps); the result is valid in thread 0.
template <int NT>
__device__ __forceinline__ Part block_reduce(Part p, Part* sh) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) p = part_combine(p, shfl_down(p, off));
  if (lane == 0) sh[w] = p;
  __syncthreads();
  if (w == 0) {
    p = lane < NT / 32 ? sh[lane] : Part{Stat{0.0, 0.0, 0.0}, 0.0};
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) p = part_combine(p, shfl_down(p, off));
  }
  __syncthreads();
  return p;
}

// The block's chains at iteration boundary k: reduce (prefix mean, prefix variance ddof 1) into
// part[(k * V + v) * nblk + blk].
__device__ __forceinline__ void reduce_boundary(Stat run, bool valid, int k, int64_t V, int64_t v, int64_t nblk,
                                                Part* sh, double* part) {
  // numpy var(ddof=1): 0 / 0 = NaN for a one-step prefix
  Part q = valid ? Part{Stat{1.0, run.mean, 0.0}, run.m2 / (run.n - 1.0)} : Part{Stat{0.0, 0.0, 0.0}, 0.0};
  q = block_reduce<kThreads>(q, sh);
  if (threadIdx.x == 0) {
    double* o = part + (((int64_t)k * V + v) * nblk + blockIdx.x) * 4;
    o[0] = q.m.n;
    o[1] = q.m.mean;
    o[2] = q.m.m2;
    o[3] = q.sv;
  }
}

// R-hat stage 2.  Block (chain tile, variable v), one thread per chain: walk the segments in order, Chan-combining the
// chain's prefix from the stage-1 statistics, and reduce over the block's chains at every iteration boundary.  The plan
// ends segments on the boundaries when their statistics fit kRhatStatBudget; otherwise (e.g. a per-iteration curve over
// many chains) the boundaries bnd[seg_kb[g] .. seg_kb[g + 1]) inside a segment are reached by reading that segment again
// from x piece by piece: at most the values once more, and a workspace that does not grow per (chain, iteration).
template <typename T>
__global__ void __launch_bounds__(kThreads, 1) k_rhat_prefix(const T* __restrict__ x, Geom gm,
                                                           const int64_t* __restrict__ seg_end,
                                                           const int32_t* __restrict__ seg_kb, int64_t G,
                                                           const int64_t* __restrict__ bnd,
                                                           const double* __restrict__ mean,
                                                           const double* __restrict__ m2, double* __restrict__ part) {
  __shared__ Part sh[kThreads / 32];
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x, v = blockIdx.y;
  const int64_t cols = gm.C * gm.V, nblk = gridDim.x;
  const bool valid = c < gm.C;
  const int64_t j = (valid ? c : 0) * gm.V + v;
  const T* p = x + gm.base(j);
  Stat run{0.0, 0.0, 0.0};
  for (int64_t g = 0; g < G; ++g) {
    const int k0 = seg_kb[g], k1 = seg_kb[g + 1];
    const bool ends = k1 > k0 && bnd[k1 - 1] == seg_end[g];   // a boundary at the segment's end needs no re-read
    if (k1 - k0 == (ends ? 1 : 0)) {
      if (valid) run = chan(run, seg_stat(seg_end, mean, m2, g, cols, j));
      if (ends) reduce_boundary(run, valid, k1 - 1, gm.V, v, nblk, sh, part);
      continue;
    }
    int64_t pos = g ? seg_end[g - 1] : 0;
    for (int k = k0; k < k1; ++k) {
      const int64_t n = bnd[k];
      if (valid) run = chan(run, range_stat(p, gm.ss, pos, n));
      pos = n;
      reduce_boundary(run, valid, k, gm.V, v, nblk, sh, part);
    }
    if (valid && pos < seg_end[g]) run = chan(run, range_stat(p, gm.ss, pos, seg_end[g]));
  }
}

// R-hat stage 3.  Block (requested iteration i, variable v): combine the chain tiles' partials in order and apply
// pyprob/diagnostics.py:792-795 with n the prefix length and m the number of chains.
__global__ void __launch_bounds__(kFinThreads) k_rhat_final(const int32_t* __restrict__ iter_bound,
                                                             const int64_t* __restrict__ iter_n, int n_iters, int64_t V,
                                                             int64_t nblk, const double* __restrict__ part,
                                                             double* __restrict__ out) {
  __shared__ Part sh[kFinThreads / 32];
  const int i = blockIdx.x;
  const int64_t v = blockIdx.y;
  const double* src = part + ((int64_t)iter_bound[i] * V + v) * nblk * 4;
  Part p{Stat{0.0, 0.0, 0.0}, 0.0};
  for (int64_t b = threadIdx.x; b < nblk; b += kFinThreads)
    p = part_combine(p, Part{Stat{src[4 * b], src[4 * b + 1], src[4 * b + 2]}, src[4 * b + 3]});
  p = block_reduce<kFinThreads>(p, sh);
  if (threadIdx.x == 0) {
    const double n = (double)iter_n[i], m = p.m.n;
    const double b = n * (p.m.m2 / (m - 1.0));   // n var(chain means, ddof 1)
    const double w = p.sv / m;                   // mean(chain variances, ddof 1)
    const double v_hat = ((n - 1.0) / n) * w + b / n;
    out[v * n_iters + i] = sqrt(v_hat / w);
  }
}

// Autocorrelation stage 2: per column, the mean over all S steps and the reference's denominator 1e-8 + M2.
__global__ void __launch_bounds__(kThreads) k_col_stats(int64_t cols, const int64_t* __restrict__ seg_end, int64_t G,
                                                         const double* __restrict__ mean,
                                                         const double* __restrict__ m2, double* __restrict__ mu,
                                                         double* __restrict__ den) {
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < cols; j += (int64_t)gridDim.x * blockDim.x) {
    Stat s{0.0, 0.0, 0.0};
    for (int64_t g = 0; g < G; ++g) s = chan(s, seg_stat(seg_end, mean, m2, g, cols, j));
    mu[j] = s.mean;
    den[j] = kEpsilon + s.m2;
  }
}

// Autocorrelation stage 3.  Block (32-column tile, group of 8 lags, step chunk): 32 lanes = 32 columns, warp w owns
// lag lags[8 * group + w].  The chunk's steps pass through shared memory as centred values d_i = x_i - mu in tiles of
// kTile; each thread accumulates sum_{i in chunk, i + lag < S} d_i d_{i+lag} in a register, the partner d_{i+lag} read
// through the read-only cache, and writes it once to part[(chunk * n_lags + l) * cols + j]: no atomics.
// A partner window is a different stretch of the same series for every lag, so the series would come from HBM once per
// lag if it left the L2 in between.  The blocks of one column tile are adjacent in launch order (all lag groups and step
// chunks of the tile, then the next tile), and the plan (acf_plan) makes enough of them per tile that the series of the
// column tiles resident at one time fit in the L2: each value is then read from HBM about once, and the partner reads
// are L2 hits.
template <typename T>
__global__ void __launch_bounds__(kThreads) k_acf(const T* __restrict__ x, Geom gm, const int64_t* __restrict__ lags,
                                                   int n_lags, int64_t n_groups, int64_t chunk, int64_t n_chunks,
                                                   const double* __restrict__ mu, double* __restrict__ part) {
  __shared__ double d_s[kTile][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t cols = gm.C * gm.V;
  const int64_t ch = blockIdx.x % n_chunks, tg = blockIdx.x / n_chunks;
  const int64_t grp = tg % n_groups, ct = tg / n_groups;
  const int64_t j = ct * 32 + lane;
  const int64_t l = grp * kLagWarps + w;
  const bool valid = j < cols, mine = valid && l < n_lags;
  const T* p = x + gm.base(valid ? j : 0);
  const double m = valid ? mu[j] : 0.0;
  const int64_t lag = l < n_lags ? lags[l] : 0;
  const int64_t a = ch * chunk, b = min(a + chunk, gm.S);
  const T* q = p + lag * gm.ss;
  double acc = 0.0;
  for (int64_t t0 = a; t0 < b; t0 += kTile) {
    const int rows = (int)min((int64_t)kTile, b - t0);
    __syncthreads();
    for (int r = w; r < rows; r += kLagWarps) d_s[r][lane] = valid ? ld(p, (t0 + r) * gm.ss) - m : 0.0;
    __syncthreads();
    if (!mine) continue;
    const int n = (int)max((int64_t)0, min((int64_t)rows, gm.S - lag - t0));
#pragma unroll 4
    for (int r = 0; r < n; ++r) acc = fma(d_s[r][lane], ld(q, (t0 + r) * gm.ss) - m, acc);
  }
  if (mine) part[(ch * n_lags + l) * cols + j] = acc;
}

// Autocorrelation stage 4: numerator summed over the chunks in order, divided by the denominator; out[(v * C + c) *
// n_lags + l].
__global__ void __launch_bounds__(kThreads) k_acf_final(Geom gm, int n_lags, int64_t n_chunks,
                                                         const double* __restrict__ part,
                                                         const double* __restrict__ den, double* __restrict__ out) {
  const int64_t cols = gm.C * gm.V;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < (int64_t)n_lags * cols;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t l = t / cols, j = t - l * cols;
    double num = 0.0;
    for (int64_t ch = 0; ch < n_chunks; ++ch) num += part[(ch * n_lags + l) * cols + j];
    const int64_t c = j / gm.V, v = j - c * gm.V;
    out[(v * gm.C + c) * n_lags + l] = num / den[j];
  }
}

// ---- host-side plans --------------------------------------------------------------------------------------------------

int64_t align_up(int64_t b) { return (b + 255) & ~int64_t(255); }

// Uniform segment length for columns of n steps: enough (column, segment) threads when there are few columns.
int64_t segment_length(int64_t n, int64_t cols) {
  int64_t nseg = (kTargetThreads + cols - 1) / cols;
  nseg = nseg < 1 ? 1 : (nseg > kMaxSegments ? kMaxSegments : nseg);
  int64_t len = (n + nseg - 1) / nseg;
  return len < kMinSegment ? kMinSegment : len;
}

// R-hat plan: segments of at most `len` steps up to the largest clamped iteration, also ended on every boundary when
// that keeps the segment statistics within kRhatStatBudget; seg_kb[g] .. seg_kb[g + 1] are the distinct boundaries bnd[]
// in segment g's (start, end].  The workspace is at most max(kRhatStatBudget, (2^17 + C V) x 16 B) of segment
// statistics plus 32 B per (distinct iteration, variable, 256 chains), whatever the number of iterations.
struct RhatPlan {
  int64_t G = 0, K = 0, nblk = 0;
  std::vector<int64_t> seg_end, bnd, iter_n;
  std::vector<int32_t> seg_kb, iter_bound;
  int64_t off_seg_end, off_bnd, off_iter_n, off_seg_kb, off_iter_bound, off_mean, off_m2, off_part, bytes, table_bytes;
};

bool rhat_plan(RhatPlan& p, int64_t S, int64_t C, int64_t V, const int64_t* iters, int n_iters) {
  if (S < 1 || C < 2 || V < 1 || !iters || n_iters < 1) return false;
  for (int i = 0; i < n_iters; ++i) {
    if (iters[i] < 1) return false;
    p.bnd.push_back(iters[i] < S ? iters[i] : S);
  }
  std::sort(p.bnd.begin(), p.bnd.end());
  p.bnd.erase(std::unique(p.bnd.begin(), p.bnd.end()), p.bnd.end());
  p.K = (int64_t)p.bnd.size();
  const int64_t nmax = p.bnd.back(), len = segment_length(nmax, C * V);
  const int64_t uniform = (nmax + len - 1) / len;
  const bool cut = (uniform + p.K) * C * V * 16 <= kRhatStatBudget;   // end segments on the boundaries too
  for (int64_t a = 0; a < nmax;) {
    int64_t e = std::min(a + len, nmax);
    if (cut) e = std::min(e, *std::upper_bound(p.bnd.begin(), p.bnd.end(), a));
    p.seg_end.push_back(e);
    p.seg_kb.push_back((int32_t)(std::upper_bound(p.bnd.begin(), p.bnd.end(), a) - p.bnd.begin()));
    a = e;
  }
  p.seg_kb.push_back((int32_t)p.K);
  p.G = (int64_t)p.seg_end.size();
  for (int i = 0; i < n_iters; ++i) {
    const int64_t n = iters[i] < S ? iters[i] : S;
    p.iter_n.push_back(n);
    p.iter_bound.push_back((int32_t)(std::lower_bound(p.bnd.begin(), p.bnd.end(), n) - p.bnd.begin()));
  }
  p.nblk = (C + kThreads - 1) / kThreads;
  const int64_t cols = C * V;
  p.off_seg_end = 0;
  p.off_bnd = p.off_seg_end + align_up(8 * p.G);
  p.off_iter_n = p.off_bnd + align_up(8 * p.K);
  p.off_seg_kb = p.off_iter_n + align_up(8 * (int64_t)n_iters);
  p.off_iter_bound = p.off_seg_kb + align_up(4 * (p.G + 1));
  p.table_bytes = p.off_iter_bound + align_up(4 * (int64_t)n_iters);
  p.off_mean = p.table_bytes;
  p.off_m2 = p.off_mean + align_up(8 * p.G * cols);
  p.off_part = p.off_m2 + align_up(8 * p.G * cols);
  p.bytes = p.off_part + align_up(8 * 4 * p.K * V * p.nblk);
  return true;
}

// Autocorrelation plan.  Uniform segments for the column statistics, then the step chunks of k_acf: enough blocks in
// all (kAcfTargetBlocks), and enough blocks per column tile that the column tiles resident at one time hold at most
// kAcfL2Budget bytes of series, so that the partner reads of every lag hit the L2 (at most kAcfResident blocks are
// resident: 8 per SM, the thread limit), within kAcfPartialBudget bytes of per-chunk partials.
struct AcfPlan {
  int64_t G, len, n_groups, chunk, n_chunks;
  std::vector<int64_t> seg_end;
  int64_t off_seg_end, off_lags, off_mean, off_m2, off_mu, off_den, off_part, bytes, table_bytes;
};

bool acf_plan(AcfPlan& p, int dtype, int64_t S, int64_t C, int64_t V, const int64_t* lags, int n_lags) {
  if (S < 1 || C < 1 || V < 1 || n_lags < 1 || (dtype != PPB_DIAG_F32 && dtype != PPB_DIAG_F64)) return false;
  if (lags)
    for (int i = 0; i < n_lags; ++i)
      if (lags[i] < 0 || lags[i] > S) return false;
  const int64_t cols = C * V;
  p.len = segment_length(S, cols);
  for (int64_t e = p.len; ; e += p.len) {
    p.seg_end.push_back(std::min(e, S));
    if (e >= S) break;
  }
  p.G = (int64_t)p.seg_end.size();
  p.n_groups = (n_lags + kLagWarps - 1) / kLagWarps;
  const int64_t tiles = (cols + 31) / 32, step_tiles = (S + kTile - 1) / kTile;
  const int64_t elem = dtype == PPB_DIAG_F32 ? 4 : 8;
  const int64_t tile_bytes = S * std::max<int64_t>(32, std::min<int64_t>(cols, 32) * elem);
  const int64_t fit = std::max<int64_t>(1, kAcfL2Budget / tile_bytes);
  const int64_t per_tile = p.n_groups;   // blocks per column tile per step chunk
  int64_t nc = (kAcfTargetBlocks + tiles * per_tile - 1) / (tiles * per_tile);
  if (tiles > fit) nc = std::max(nc, (kAcfResident + fit * per_tile - 1) / (fit * per_tile));
  const int64_t cap = std::max<int64_t>(1, kAcfPartialBudget / (8 * (int64_t)n_lags * cols));
  nc = std::max<int64_t>(1, std::min(std::min(nc, step_tiles), cap));
  p.chunk = (step_tiles + nc - 1) / nc * kTile;
  p.n_chunks = (S + p.chunk - 1) / p.chunk;
  p.off_seg_end = 0;
  p.off_lags = align_up(8 * p.G);
  p.table_bytes = p.off_lags + align_up(8 * (int64_t)n_lags);
  p.off_mean = p.table_bytes;
  p.off_m2 = p.off_mean + align_up(8 * p.G * cols);
  p.off_mu = p.off_m2 + align_up(8 * p.G * cols);
  p.off_den = p.off_mu + align_up(8 * cols);
  p.off_part = p.off_den + align_up(8 * cols);
  p.bytes = p.off_part + align_up(8 * p.n_chunks * (int64_t)n_lags * cols);
  return true;
}

template <typename V>
void put(std::vector<char>& host, int64_t off, const std::vector<V>& v) {
  if (!v.empty()) memcpy(host.data() + off, v.data(), v.size() * sizeof(V));
}

template <typename T>
int launch_seg_stats(const void* x, Geom gm, const int64_t* seg_end, int64_t G, double* mean, double* m2,
                     cudaStream_t st) {
  k_seg_stats<T><<<ppb_grid_for(G * gm.C * gm.V, kThreads, 1), kThreads, 0, st>>>((const T*)x, gm, seg_end, G, mean,
                                                                                   m2);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

}  // namespace

extern "C" {

int64_t ppb_diag_rhat_workspace_bytes(int64_t S, int64_t C, int64_t V, const int64_t* iters, int n_iters) {
  RhatPlan p;
  return rhat_plan(p, S, C, V, iters, n_iters) ? p.bytes : -1;
}

int ppb_diag_rhat(const void* x, int dtype, int64_t S, int64_t C, int64_t V, int64_t stride_s, int64_t stride_c,
                  int64_t stride_v, const int64_t* iters, int n_iters, double* out, void* workspace,
                  int64_t workspace_bytes, void* stream) {
  PPB_CHECK_ARG(x && out && workspace && (dtype == PPB_DIAG_F32 || dtype == PPB_DIAG_F64), "bad arguments");
  PPB_CHECK_ARG(C >= 2, "Gelman-Rubin diagnostic requires at least two chains");
  RhatPlan p;
  PPB_CHECK_ARG(rhat_plan(p, S, C, V, iters, n_iters), "need S >= 1, V >= 1 and at least one iteration, all >= 1");
  PPB_CHECK_ARG(workspace_bytes >= p.bytes, "workspace too small (ppb_diag_rhat_workspace_bytes)");
  PPB_CHECK_ARG(p.nblk <= 65535 * 256 && V <= 65535 && n_iters <= 0x7fffffff, "too many chains or variables");
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  std::vector<char> host(p.table_bytes);
  put(host, p.off_seg_end, p.seg_end);
  put(host, p.off_bnd, p.bnd);
  put(host, p.off_iter_n, p.iter_n);
  put(host, p.off_seg_kb, p.seg_kb);
  put(host, p.off_iter_bound, p.iter_bound);
  PPB_CUDA(cudaMemcpyAsync(ws, host.data(), p.table_bytes, cudaMemcpyHostToDevice, st));
  const int64_t* seg_end = (const int64_t*)(ws + p.off_seg_end);
  double* mean = (double*)(ws + p.off_mean);
  double* m2 = (double*)(ws + p.off_m2);
  double* part = (double*)(ws + p.off_part);
  const Geom gm{S, C, V, stride_s, stride_c, stride_v};
  const int rc = dtype == PPB_DIAG_F32 ? launch_seg_stats<float>(x, gm, seg_end, p.G, mean, m2, st)
                                       : launch_seg_stats<double>(x, gm, seg_end, p.G, mean, m2, st);
  if (rc != PPB_OK) return rc;
  const dim3 grid2((unsigned)p.nblk, (unsigned)V);
  const int32_t* seg_kb = (const int32_t*)(ws + p.off_seg_kb);
  const int64_t* bnd = (const int64_t*)(ws + p.off_bnd);
  if (dtype == PPB_DIAG_F32)
    k_rhat_prefix<float><<<grid2, kThreads, 0, st>>>((const float*)x, gm, seg_end, seg_kb, p.G, bnd, mean, m2, part);
  else
    k_rhat_prefix<double><<<grid2, kThreads, 0, st>>>((const double*)x, gm, seg_end, seg_kb, p.G, bnd, mean, m2, part);
  PPB_LAUNCH_CHECK();
  k_rhat_final<<<dim3((unsigned)n_iters, (unsigned)V), kFinThreads, 0, st>>>(
      (const int32_t*)(ws + p.off_iter_bound), (const int64_t*)(ws + p.off_iter_n), n_iters, V, p.nblk, part, out);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int64_t ppb_diag_autocorr_workspace_bytes(int dtype, int64_t S, int64_t C, int64_t V, int n_lags) {
  AcfPlan p;
  return acf_plan(p, dtype, S, C, V, nullptr, n_lags) ? p.bytes : -1;
}

int ppb_diag_autocorr(const void* x, int dtype, int64_t S, int64_t C, int64_t V, int64_t stride_s, int64_t stride_c,
                      int64_t stride_v, const int64_t* lags, int n_lags, double* out, void* workspace,
                      int64_t workspace_bytes, void* stream) {
  PPB_CHECK_ARG(x && out && workspace && lags && (dtype == PPB_DIAG_F32 || dtype == PPB_DIAG_F64), "bad arguments");
  AcfPlan p;
  PPB_CHECK_ARG(acf_plan(p, dtype, S, C, V, lags, n_lags), "need S, C, V >= 1 and at least one lag, all in [0, S]");
  PPB_CHECK_ARG(workspace_bytes >= p.bytes, "workspace too small (ppb_diag_autocorr_workspace_bytes)");
  const int64_t cols = C * V, tiles = (cols + 31) / 32;
  PPB_CHECK_ARG(tiles * p.n_groups * p.n_chunks <= 0x7fffffff, "too many chains or lags");
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  std::vector<char> host(p.table_bytes);
  put(host, p.off_seg_end, p.seg_end);
  memcpy(host.data() + p.off_lags, lags, 8 * (size_t)n_lags);
  PPB_CUDA(cudaMemcpyAsync(ws, host.data(), p.table_bytes, cudaMemcpyHostToDevice, st));
  const int64_t* seg_end = (const int64_t*)(ws + p.off_seg_end);
  const int64_t* lags_dev = (const int64_t*)(ws + p.off_lags);
  double* mean = (double*)(ws + p.off_mean);
  double* m2 = (double*)(ws + p.off_m2);
  double* mu = (double*)(ws + p.off_mu);
  double* den = (double*)(ws + p.off_den);
  double* part = (double*)(ws + p.off_part);
  const Geom gm{S, C, V, stride_s, stride_c, stride_v};
  int rc = dtype == PPB_DIAG_F32 ? launch_seg_stats<float>(x, gm, seg_end, p.G, mean, m2, st)
                                 : launch_seg_stats<double>(x, gm, seg_end, p.G, mean, m2, st);
  if (rc != PPB_OK) return rc;
  k_col_stats<<<ppb_grid_for(cols, kThreads, 1), kThreads, 0, st>>>(cols, seg_end, p.G, mean, m2, mu, den);
  PPB_LAUNCH_CHECK();
  const unsigned grid = (unsigned)(tiles * p.n_groups * p.n_chunks);
  if (dtype == PPB_DIAG_F32)
    k_acf<float><<<grid, kThreads, 0, st>>>((const float*)x, gm, lags_dev, n_lags, p.n_groups, p.chunk, p.n_chunks, mu,
                                            part);
  else
    k_acf<double><<<grid, kThreads, 0, st>>>((const double*)x, gm, lags_dev, n_lags, p.n_groups, p.chunk, p.n_chunks,
                                             mu, part);
  PPB_LAUNCH_CHECK();
  k_acf_final<<<ppb_grid_for(cols * n_lags, kThreads, 1), kThreads, 0, st>>>(gm, n_lags, p.n_chunks, part, den, out);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

}  // extern "C"
