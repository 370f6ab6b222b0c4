/*
 * pyprob_b200 — C-ABI of the H100-native inference-compilation hot path.
 *
 * This header is the drop-in boundary (SURVEY.md §8b).  pyprob has no FFI of its own: the
 * reference reaches its arithmetic through Python calls into torch.  Every entry point below
 * names the reference call site (file:line under the pyprob tree) whose arithmetic it replaces;
 * INTEGRATION.md shows the ctypes stub a pyprob maintainer would add at that call site.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes only.  No torch types.
 *   - Unless a parameter is suffixed `_host`, pointers are DEVICE pointers (cudaMalloc / torch
 *     allocations on the current device).  `stream` is a cudaStream_t passed as void*.
 *   - All functions return 0 on success, a negative PPB_E* code on argument errors, or a positive
 *     cudaError_t.  ppb_last_error() returns a human-readable message for the calling thread.
 *   - There is NO CPU fallback anywhere in this library.
 */
#ifndef PYPROB_B200_H
#define PYPROB_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PPB_OK 0
#define PPB_EINVAL (-1)
#define PPB_ENOTSUP (-2)
#define PPB_ENOMEM (-3)

/* distribution families (value of ppb_addr_desc.family; order mirrors north_star's list) */
#define PPB_FAMILY_NORMAL 0      /* prior Normal      -> proposal mixture of K Normals            */
#define PPB_FAMILY_UNIFORM 1     /* prior Uniform     -> proposal mixture of K TruncatedNormals   */
#define PPB_FAMILY_POISSON 2     /* prior Poisson     -> proposal mixture of K TruncatedNormals   */
#define PPB_FAMILY_CATEGORICAL 3 /* prior Categorical -> proposal Categorical                     */
#define PPB_FAMILY_BERNOULLI 4   /* prior Bernoulli   -> proposal Bernoulli, head_out = 1, smp_in = 1 */

const char* ppb_last_error(void);
int ppb_version(void);
/* Compute capability major*10+minor of the current device (90 on an H100; the kernels are built for sm_90a only). */
int ppb_device_arch(void);
/* Number of kernels this library has launched in the calling process (bench.py's gpu_launches). */
int64_t ppb_launch_count(void);
/* Kernel-level profiling for bench.py's roofline: when enabled, the library brackets every launch of the
 * LSTM gate GEMM class (input projections + recurrent GEMMs, forward and backward) with CUDA events on the
 * launching stream; ppb_prof_read sums their durations.  Off by default (events perturb the step). */
int ppb_prof_enable(int on);
int ppb_prof_read(double* total_ms_out, int64_t* launches_out, double* flops_out);

/* ------------------------------------------------------------------------------------------------
 * 1. Trace scoring: per-family log_prob over the particle axis  (SURVEY §8a rows a6, a12)
 *
 * Replaces  pyprob/distributions/distribution.py:38-43  (Distribution.log_prob -> torch_dist.log_prob)
 * as called from pyprob/state.py:147,181,196-217,282-288, one particle at a time.
 * Here `n` particles are scored per call.  A parameter pointer with stride 0 is a scalar broadcast
 * over particles, stride 1 is per-particle.
 *   lp_out   (nullable) fp32[n]   log_prob of each particle
 *   acc      (nullable) fp64[n]   per-particle running log importance weight; acc[i] += acc_scale*lp
 *                                 (Trace.end's double-precision sum of fp32 terms, pyprob/trace.py:123-125;
 *                                  acc_scale = likelihood_importance for observes, -1 for a proposal term)
 * The eleven families with an element-wise log_prob (Normal .. VonMises) are scored by ppb_event_log_prob_d1
 * (section 2b); this section holds the families whose parameters are rows.
 * ---------------------------------------------------------------------------------------------- */
/* probs: [n, C] (probs_row_stride = C) or [C] shared (probs_row_stride = 0); unnormalised, as given to
 * pyprob/distributions/categorical.py:8-21.  value holds category indices stored as fp32. */
int ppb_categorical_log_prob(const float* value, const float* probs, int64_t probs_row_stride,
                             int num_categories, float* lp_out, double* acc, double acc_scale,
                             int64_t n, void* stream);
/* Mixture of K Normals (pyprob/distributions/mixture.py:8-45 over normal.py:8-11).
 * means/stddevs/probs: [n, K] row-major (row stride K) or [K] shared (row stride 0). */
int ppb_mixture_normal_log_prob(const float* value, const float* means, const float* stddevs,
                                const float* probs, int64_t row_stride, int K, float* lp_out,
                                double* acc, double acc_scale, int64_t n, void* stream);
/* Mixture of K TruncatedNormals (mixture.py:38-45 over truncated_normal.py:11-54); low/high per
 * particle (stride 1) or scalar (stride 0). */
int ppb_mixture_truncated_normal_log_prob(const float* value, const float* means,
                                          const float* stddevs, const float* probs,
                                          int64_t row_stride, int K, const float* low, int low_stride,
                                          const float* high, int high_stride, float* lp_out,
                                          double* acc, double acc_scale, int64_t n, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 2. Samplers over the particle axis (SURVEY §8a row a13)
 *
 * Replace  pyprob/distributions/distribution.py:31-36  (torch normal/rand/multinomial/poisson),
 * pyprob/distributions/mixture.py:47-63, pyprob/distributions/truncated_normal.py:94-112.
 * Counter-based Philox4x32-10: particle i of call (seed, offset) uses counter (i, offset), so results
 * are independent of the launch geometry and of the number of GPUs (rank r shards the index range).
 * `first_index` is the global index of element 0 (for sharded particle ranges).
 * lp_out (nullable): log_prob of the drawn value under the sampled distribution (fused sample+score).
 * The eleven families with an element-wise log_prob are drawn by ppb_event_sample_d1 (section 2b).
 * ---------------------------------------------------------------------------------------------- */
int ppb_categorical_sample(const float* probs, int64_t probs_row_stride, int num_categories,
                           float* value_out, float* lp_out, int64_t n, uint64_t seed, uint64_t offset,
                           int64_t first_index, void* stream);
int ppb_mixture_normal_sample(const float* means, const float* stddevs, const float* probs,
                              int64_t row_stride, int K, float* value_out, float* lp_out, int64_t n,
                              uint64_t seed, uint64_t offset, int64_t first_index, void* stream);
int ppb_mixture_truncated_normal_sample(const float* means, const float* stddevs, const float* probs,
                                        int64_t row_stride, int K, const float* low, int low_stride,
                                        const float* high, int high_stride, float* value_out,
                                        float* lp_out, int64_t n, uint64_t seed, uint64_t offset,
                                        int64_t first_index, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 2b. The families with an element-wise log_prob: scalar sites, and sites whose value is a vector or an image
 *
 * Replace  pyprob/distributions/distribution.py:31-43 for these families as pyprob/state.py drives them, one
 * particle at a time, and pyprob/state.py:118-155 with a tensor value: distribution.log_prob(value, sum=True)
 * (torch broadcasts the value against the parameters and the element-wise log-densities are summed), and
 * pyprob/state.py:136-137, which draws the observed value from the likelihood for a training trace.
 * A site has D = prod(event shape) elements per particle; D = 1 is the per-particle (scalar) site.
 * Every operand is (pointer, particle stride ps, element stride es): element j of particle i is p[i ps + j es], and
 * (ps, es) must be one of (0, 0) scalar, (1, 0) one per particle, (0, 1) shared event, (D, 1) event per particle
 * (at D = 1 all four are a scalar or one per particle).
 * Families and their parameters p0 .. p3 (unused slots are ignored).  log_prob follows torch.distributions, which the
 * reference wraps; a value outside the support or an invalid parameter scores NaN (the reference's argument
 * validation raises) and draws NaN:
 *   NORMAL (loc, scale), UNIFORM (low, high), POISSON (rate)
 *   BERNOULLI (probs): v log(pc) + (1 - v) log(1 - pc), pc = clamp_probs(p), v in {0, 1}; draws 1 if u < p
 *   EXPONENTIAL (rate): log r - r x, x >= 0
 *   GAMMA (concentration, rate): xlogy(c, r) + xlogy(c - 1, x) - r x - lgamma(c), x >= 0
 *   LOGNORMAL (loc, scale): Normal(loc, scale).log_prob(log x) - log x, x > 0
 *   WEIBULL (scale, concentration): torch's Exponential(1) through PowerTransform(1/k), AffineTransform(0, scale)
 *   BETA (concentration1, concentration0, low, high): torch Beta(c1, c0).log_prob((x - low) / (high - low)), with no
 *     -log(high - low) term, as pyprob/distributions/beta.py:38-40
 *   BINOMIAL (total_count, probs): torch's logits form, logits = log(pc) - log1p(-pc); x an integer in [0, total_count]
 *   VON_MISES (loc, concentration): kappa cos(x - loc) - log(2 pi) - log I0(kappa), log I0 as torch's
 *     _log_modified_bessel_fn computes it (finite at any kappa)
 * Draws: Normal and LogNormal by Box-Muller, Uniform, Exponential and Weibull by inversion, Poisson by inversion below
 * rate 10 and PTRS above; Gamma by Marsaglia-Tsang (c < 1 as G(c + 1) u^(1/c)), clamped below at FLT_MIN as torch;
 * Beta as low + (high - low) Ga / (Ga + Gb), the ratio clamped to [FLT_MIN, 1 - eps] as torch's Dirichlet; Binomial by
 * inversion for n min(p, 1 - p) < 10 and BTRS (Hoermann 1993) otherwise; VonMises by Best-Fisher rejection in double
 * precision, wrapped into [-pi, pi) as torch.  The rejection samplers draw each round from the counter
 * (index, offset + (round << 40)) and stop after a fixed number of rounds (failure probability below 1e-12 per draw),
 * so every draw takes bounded time.
 * ---------------------------------------------------------------------------------------------- */
#define PPB_EVENT_NORMAL 0
#define PPB_EVENT_UNIFORM 1
#define PPB_EVENT_POISSON 2
#define PPB_EVENT_BERNOULLI 3
#define PPB_EVENT_EXPONENTIAL 4
#define PPB_EVENT_GAMMA 5
#define PPB_EVENT_LOGNORMAL 6
#define PPB_EVENT_WEIBULL 7
#define PPB_EVENT_BETA 8
#define PPB_EVENT_BINOMIAL 9
#define PPB_EVENT_VON_MISES 10
/* acc (nullable) fp64[n]: acc[i] += acc_scale * sum_j lp_ij, summed in fp64 in an order that depends on (n, D) only,
 * without atomics (repeated calls give identical bits).
 * lp_out (nullable) fp32[n, D], row-major: the element-wise log-densities.  PPB_EINVAL for an unknown family, n < 0 or
 * D < 1, and with n > 0 for a null operand the family needs or strides not of the four forms; n = 0 does nothing. */
int ppb_event_log_prob(int family, const float* value, int64_t value_ps, int64_t value_es, const float* p0,
                       int64_t p0_ps, int64_t p0_es, const float* p1, int64_t p1_ps, int64_t p1_es,
                       const float* p2, int64_t p2_ps, int64_t p2_es, const float* p3, int64_t p3_ps,
                       int64_t p3_es, int64_t n, int64_t D, float* lp_out, double* acc, double acc_scale,
                       void* stream);
/* value_out fp32[n, D] row-major; lp_out (nullable) fp32[n]: the row's event-summed log-density, as
 * ppb_event_log_prob sums it.  Element j of particle i draws from the Philox counter
 * ((first_index + i) | (j << 40), offset + (round << 40)): element 0 is the D = 1 draw bit for bit, and a shard of
 * the particles draws the rows the full run draws.  PPB_EINVAL, besides the cases above, for D > 2^24, a negative
 * first_index or first_index + n > 2^40 (the counter fields would overlap), at any D, and for a null value_out with
 * n > 0. */
int ppb_event_sample(int family, const float* p0, int64_t p0_ps, int64_t p0_es, const float* p1, int64_t p1_ps,
                     int64_t p1_es, const float* p2, int64_t p2_ps, int64_t p2_es, const float* p3, int64_t p3_ps,
                     int64_t p3_es, float* value_out, float* lp_out, int64_t n, int64_t D, uint64_t seed,
                     uint64_t offset, int64_t first_index, void* stream);
/* The same two entry points at D = 1, the per-particle site, with a shorter argument list for the calls that score or
 * draw one scalar site at a time: value is fp32[n]; parameter k is one per particle where bit k of param_strides is set
 * and a scalar where it is clear (unused slots are ignored).  Results, checks and draws are ppb_event_log_prob's and
 * ppb_event_sample's with D = 1. */
int ppb_event_log_prob_d1(int family, const float* value, const float* p0, const float* p1, const float* p2,
                          const float* p3, int param_strides, float* lp_out, double* acc, double acc_scale, int64_t n,
                          void* stream);
int ppb_event_sample_d1(int family, const float* p0, const float* p1, const float* p2, const float* p3,
                        int param_strides, float* value_out, float* lp_out, int64_t n, uint64_t seed, uint64_t offset,
                        int64_t first_index, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 3. Importance-weight normalisation (SURVEY §8a rows a14, a15)
 *
 * Replaces  pyprob/distributions/empirical.py:298-302 (Categorical(logits=log_weights.double()))
 * and :759-766 (ESS = 1/sum p^2), pyprob/util.py:398-399.
 *   ppb_weights_cast     : fp64 accumulators -> fp32 log weights (empirical.py:326 stores fp32),
 *                          invalid[i]=1 where the weight is NaN/+-inf (pyprob/model.py:65-68 discards).
 *   ppb_weights_partials : per-block online (max, sum exp, sum exp^2) in fp64 -> partials[3*nblocks]
 *                          (the 3-scalar-per-block form that multi-GPU runs all-gather, SURVEY §8e).
 *   ppb_weights_finalize : combines `npartials` triples (from any number of ranks), writes
 *                          stats[0]=logsumexp, stats[1]=ESS, stats[2]=max, stats[3]=sum exp(w-max),
 *                          and (if logits_out != NULL) logits_out[i] = w[i] - logsumexp in fp64.
 * ---------------------------------------------------------------------------------------------- */
int ppb_weights_cast(const double* acc, float* log_w_out, uint8_t* invalid_out, int64_t n,
                     void* stream);
int ppb_weights_num_partials(int64_t n);
int ppb_weights_partials(const float* log_w, int64_t n, double* partials, void* stream);
int ppb_weights_finalize(const float* log_w, int64_t n, const double* partials, int npartials,
                         double* stats4, double* logits_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 4. Proposal network (SURVEY §8a rows a2-a8, a10, a11)
 *
 * Replaces  pyprob/nn/inference_network_lstm.py:136-220 (_loss), :82-134 (_infer_step),
 *           pyprob/nn/inference_network.py:132-139 (_embed_observe), :493 (loss.backward()),
 *           :496 (optimizer.step(), Adam), pyprob/nn/embedding_feedforward.py:35-48,
 *           pyprob/nn/proposal_*.py forward, pyprob/distributions/mixture.py:38-45.
 *
 * Parameters live in ONE flat fp32 arena owned by the caller (torch allocation); the arena layout is
 * described by offsets (in floats).  All weight matrices are row-major [out, in] exactly like
 * nn.Linear / nn.LSTM (gate order i,f,g,o), so a reference state_dict copies in verbatim.
 * ---------------------------------------------------------------------------------------------- */
#define PPB_MAX_OBS 8
#define PPB_MAX_FF_LAYERS 4

typedef struct {
  int32_t in_dim, out_dim;
  int64_t w_off, b_off; /* W[out,in], b[out] */
} ppb_linear_desc;

typedef struct {
  int32_t num_layers; /* EmbeddingFeedForward: Linear+ReLU per layer (ReLU on the last one too) */
  int32_t in_dim, out_dim;
  ppb_linear_desc layers[PPB_MAX_FF_LAYERS];
} ppb_ff_desc;

typedef struct {
  int32_t lstm_dim;       /* H   (inference_network_lstm.py:13 lstm_dim)                    */
  int32_t obs_dim;        /* E   (inference_network.py:127 _observe_embedding_dim)          */
  int32_t sample_dim;     /* 4   sample_embedding_dim                                       */
  int32_t addr_dim;       /* 64  address_embedding_dim                                      */
  int32_t type_dim;       /* 8   distribution_type_embedding_dim                            */
  int32_t mixture_k;      /* K   proposal_mixture_components                                */
  int32_t num_obs;        /* observables, concatenated in observe_embeddings dict order     */
  int32_t obs_in_total;   /* sum of flattened observable sizes (row width of `obs` input)   */
  ppb_ff_desc obs_ff[PPB_MAX_OBS]; /* per-observable embedding (inference_network.py:117)   */
  ppb_ff_desc obs_final;  /* _layers_observe_embedding_final, E->E->E (:129)                */
  int64_t w_ih_off, w_hh_off, b_ih_off, b_hh_off; /* nn.LSTM(I,H,1): [4H,I],[4H,H],[4H],[4H]   */
  int32_t network_type;   /* PPB_NET_*; 0 (zero-initialised callers) = the LSTM network         */
  int32_t reserved_;
} ppb_net_desc;

/* ppb_net_desc.network_type.  PPB_NET_FEEDFORWARD is InferenceNetworkFeedForward
 * (pyprob/nn/inference_network_feedforward.py:13-98): every proposal head reads the observation embedding directly, so
 * lstm_dim, sample_dim, addr_dim and type_dim are 0, the LSTM offsets are ignored, and a head's first layer is
 * Linear(E -> head_hidden) with head_hidden = int((E + out) / 2). */
#define PPB_NET_LSTM 0
#define PPB_NET_FEEDFORWARD 1

typedef struct {
  int32_t family;         /* PPB_FAMILY_*                                                    */
  int32_t num_categories; /* C for categorical, else 0                                       */
  int32_t head_hidden;    /* int((H+out)/2), embedding_feedforward.py:26                     */
  int32_t head_out;       /* 3K or C                                                         */
  int32_t smp_in;         /* sample-embedding input width: 1, or C (one-hot)                 */
  int32_t type_id;        /* index into the distribution-type embedding table               */
  int64_t addr_emb_off;   /* [addr_dim]                                                      */
  int64_t smp_w_off, smp_b_off;   /* Linear(smp_in -> sample_dim)                            */
  int64_t w1_off, b1_off, w2_off, b2_off; /* head trunk Linear(H->hidden), Linear(hidden->out) */
} ppb_addr_desc;

typedef struct ppb_net ppb_net; /* opaque: device copies of the tables above */

int ppb_net_create(ppb_net** out, const ppb_net_desc* desc_host);
/* (Re)load the address table and the type-embedding offsets after _polymorph grew the network
 * (inference_network_lstm.py:34-80, inference_network_feedforward.py:21-51).  type_emb_off_host[n_types] are arena
 * offsets of [type_dim].  A feed-forward net takes n_types = 0 (type_emb_off_host may be NULL) and ignores
 * addr_emb_off, smp_* and type_id; its w1 is [head_hidden, E]. */
int ppb_net_set_tables(ppb_net* net, const ppb_addr_desc* addrs_host, int32_t n_addrs,
                       const int64_t* type_emb_off_host, int32_t n_types, int64_t arena_floats);
int ppb_net_destroy(ppb_net* net);

/* Encoded trace minibatch = what pyprob/nn/dataset.py:21-37 (Batch) + the Python loops of
 * inference_network_lstm.py:146-182 compute, as index tensors ("address/index tensors bit-exact").
 * Traces are ordered by sub-batch, sub-batches by decreasing length T (stable w.r.t. the reference's
 * dict-insertion order); rows are time-major: row(t,i) = row_off[t] + i for the n_active[t] traces whose
 * length exceeds t (always a prefix of the trace order).  A "step" is one (t, sub-batch) pair.
 * The whole batch travels as ONE contiguous image (header + arrays, built by
 * pyprob_b200.encoding.pack_batch) so it moves host->device in a single copy; ppb_batch is the decoded
 * view: `_host` fields point into the host image (planning), the rest into the device copy. */
typedef struct {
  int32_t n_traces;       /* B: batch.size                                                   */
  int32_t n_sub;          /* S: len(batch.sub_batches)                                       */
  int32_t t_max;          /* longest controlled length                                       */
  int32_t n_rows;         /* R = sum_s B_s*T_s                                               */
  int32_t n_steps;        /* sum_t (#sub-batches active at t)                                */
  int32_t n_groups;       /* distinct addresses present in the batch                         */
  int32_t obs_in_total;   /* row width of obs                                                */
  int32_t reserved_;
  /* host planning arrays */
  const int32_t* row_off_host;     /* [t_max+1]                                              */
  const int32_t* group_addr_host;  /* [n_groups]   address id of each group                  */
  const int32_t* group_start_host; /* [n_groups+1] offsets into head_rows                    */
  /* device arrays */
  const int32_t* trace_sub;      /* [B]   sub-batch of trace i                                */
  const int32_t* step_addr;      /* [n_steps] address id at (t, s)                            */
  const int32_t* step_prev_addr; /* [n_steps] address id at (t-1, s), -1 at t = 0            */
  const int32_t* step_row0;      /* [n_steps] first row of the step                           */
  const int32_t* step_nrows;     /* [n_steps] B_s                                             */
  const int32_t* row_step;       /* [R]   step index of each row                              */
  const int32_t* row_prev;       /* [R]   row of the same trace at t-1, -1 at t = 0          */
  const float* values;           /* [R]   sampled value at (t,i) (category index as float)    */
  const float* prior0;           /* [R]   prior mean | low                                    */
  const float* prior1;           /* [R]   prior stddev | high                                 */
  const float* obs;              /* [B, obs_in_total] flattened observed values               */
  const int32_t* head_rows;      /* [valid rows] row ids grouped by address                   */
  const int32_t* row_trace;      /* [R]   trace index of the row, -1 for padding rows             */
  const int32_t* row_next;       /* [R]   row of the same trace at t+1, -1 if the trace ends      */
  const int32_t* step_t;         /* [n_steps] time index of the step                              */
  const int32_t* step_prev_row0; /* [n_steps] first row of the same sub-batch at t-1 (-1 at t=0)  */
  const int32_t* group_addr;     /* [n_groups]   device copy of group_addr_host                   */
  const int32_t* group_start;    /* [n_groups+1] device copy of group_start_host                  */
  /* host copies of the per-step arrays, used to plan launches: required at every precision */
  const int32_t* step_addr_host;
  const int32_t* step_row0_host;
  const int32_t* step_nrows_host;
  const int32_t* step_t_host;
  const int32_t* step_prev_row0_host;
  int32_t row_align;             /* 1 = compact rows, 128 = every (t, sub-batch) segment padded to 128 rows */
  int32_t reserved2_;
} ppb_batch;

/* Batch image header: int64[PPB_IMAGE_HEADER_WORDS]; word 0 = magic, 1..7 = the seven int32 fields
 * above in order, 8 = total bytes, 9.. = byte offsets of the arrays in the order they are declared
 * above (row_off, group_addr, group_start, trace_sub, step_addr, step_prev_addr, step_row0, step_nrows,
 * row_step, row_prev, values, prior0, prior1, obs, head_rows, row_trace, row_next, step_t, step_prev_row0);
 * word 28 = row_align.  Every array is 16-byte aligned. */
#define PPB_IMAGE_MAGIC 0x5050423230304231LL
#define PPB_IMAGE_HEADER_WORDS 32
int ppb_batch_from_image(const void* image_host, const void* image_dev, int64_t image_bytes,
                         ppb_batch* out);
/* sizeof() of the ABI structs, for binding self-checks: 0 = ppb_net_desc, 1 = ppb_addr_desc,
 * 2 = ppb_batch, 3 = ppb_ff_desc, 4 = ppb_linear_desc, 5 = tcg::Problem (ppb_tc_run_problems) */
int64_t ppb_sizeof(int which);

/* precision of the tensor-core GEMMs: 0 = 3xTF32 split (fp32-faithful, parity mode, default),
 * 1 = single-pass TF32, 2 = fp32 SIMT everywhere (bring-up / cross-check). */
#define PPB_PREC_TF32X3 0
#define PPB_PREC_TF32 1
#define PPB_PREC_FP32_SIMT 2

int64_t ppb_ic_workspace_bytes(const ppb_net* net, int32_t n_traces, int32_t n_rows, int32_t t_max,
                               int32_t n_steps, int32_t n_groups);
/* Both calls dispatch on the net's network_type; a feed-forward net's workspace holds no LSTM buffers.
 * loss = sum over rows of -log q(value | h_row) / n_traces  (inference_network_lstm.py:218-220; feed-forward:
 * inference_network_feedforward.py:68-98, h_row = the observation embedding of the row's trace);
 * -inf log-probs are replaced by log(1e-8) with zero gradient (:207-217, util.py:278-284).
 * status_out[0] = number of rows whose log-prob is NaN/+inf after the repair (reference returns
 * (False, 0) when that is non-zero).  row_lp_out (nullable) fp32[R] per-row log q. */
int ppb_ic_loss_forward(ppb_net* net, const float* arena, const ppb_batch* batch_host_struct,
                        void* workspace, int64_t workspace_bytes, int precision, float* loss_out,
                        int32_t* status_out, float* row_lp_out, int want_grad, void* stream);
/* grad_arena += d(loss*grad_scale)/d(arena); must follow ppb_ic_loss_forward on the same workspace. */
int ppb_ic_loss_backward(ppb_net* net, const float* arena, float* grad_arena,
                         const ppb_batch* batch_host_struct, void* workspace, int64_t workspace_bytes,
                         int precision, float grad_scale, void* stream);

/* Slots of the device hyper-parameter vector (float) read by the optimiser steps.  The Adam steps
 * (ppb_adam_step_dev, ppb_dp_adam_step) read the first PPB_HYPER_ADAM_COUNT; the segmented step
 * (ppb_optimizer_step_segmented) reads all PPB_HYPER_COUNT. */
enum {
  PPB_HYPER_LR = 0,
  PPB_HYPER_BETA1,
  PPB_HYPER_BETA2,
  PPB_HYPER_EPS,
  PPB_HYPER_WEIGHT_DECAY,
  PPB_HYPER_GRAD_SCALE,      /* multiplies the gradient first (1/world for data-parallel averaging, :324-325) */
  PPB_HYPER_ADAM_COUNT,
  PPB_HYPER_MOMENTUM = PPB_HYPER_ADAM_COUNT,
  PPB_HYPER_LARC_TRUST,      /* LARC trust coefficient (0.002) */
  PPB_HYPER_LARC_EPS,        /* LARC eps (1e-8) */
  PPB_HYPER_LARC_EPSILON,    /* LARC epsilon (1/16000) */
  PPB_HYPER_COUNT
};

/* Adam state block (16 bytes of device memory, zero-initialised), shared by ppb_adam_step_dev and
 * ppb_dp_adam_step:
 *   byte 0   int64   step counter: the number of steps taken; each call advances it by one
 *   byte 8   float   1 - beta1^t of the last step (written, read by nothing in this library)
 *   byte 12  uint32  finished-block count of ppb_adam_step_dev: zero between calls
 * A caller that resumes from a checkpoint writes its step count at byte 0. */

/* Fused flat-arena Adam (torch.optim.Adam semantics: pyprob/nn/inference_network.py:348, :496) with the step
 * counter and hyper-parameters in device memory, so that a whole training step (forward, backward, optimiser) can be
 * captured once in a CUDA graph and replayed.  Any alignment of the four arrays is accepted.
 *   hyper_dev: float[PPB_HYPER_ADAM_COUNT]
 *   state_dev: the Adam state block */
int ppb_adam_step_dev(float* arena, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n,
                      const float* hyper_dev, void* state_dev, void* stream);

/* Segment-aware optimiser step (pyprob/nn/inference_network.py:343-355, pyprob/nn/optimizer_larc.py:74-107):
 * Adam or Nesterov SGD (dampening 0), optionally under LARC (clip mode), over a flat arena whose parameter
 * tensors ("segments") may be absent from the minibatch.  An absent segment is skipped exactly as torch skips a
 * parameter whose .grad is None: no moment decay, no step-count increment, no LARC scaling.
 *   kind            0 Adam, 1 Adam+LARC, 2 SGD, 3 SGD+LARC
 *   n               arena length in floats; segments start on multiples of 4 (16-byte aligned regions)
 *   seg_of_block    int32[ceil(n/4)] device: segment id of floats [4i, 4i+4), -1 for padding
 *   present         int32[n_segs] device: 1 if the segment received a gradient this step
 *   seg_steps       int64[n_segs] device: per-segment step counts (incremented for present segments)
 *   state0/state1   Adam: exp_avg / exp_avg_sq;  SGD: momentum buffer / unused (may be NULL)
 *   hyper_dev       float[PPB_HYPER_COUNT] device
 *   scratch         ppb_optimizer_scratch_bytes(n_segs) bytes of device memory
 * Graph-capturable (all step-dependent state lives in device memory). */
int64_t ppb_optimizer_scratch_bytes(int32_t n_segs);
int ppb_optimizer_step_segmented(float* arena, const float* grad, float* state0, float* state1, int64_t n,
                                 const int32_t* seg_of_block_dev, int32_t n_segs, const int32_t* present_dev,
                                 int64_t* seg_steps_dev, void* scratch_dev, int64_t scratch_bytes, int kind,
                                 const float* hyper_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Data-parallel optimiser step fused with its collective (replaces the per-parameter gradient
 * all-reduce + optimizer.step() of pyprob/nn/inference_network.py:296-333, :496).
 *
 * Every rank owns one "peer block" of device memory that all ranks of the node map over NVLink
 * (CUDA IPC).  Block layout (byte offsets chosen by the caller, 16-byte aligned, identical on all ranks):
 *   param_off : float[n]            parameter arena (replicated)
 *   grad_off  : float[n + n_extra]  this rank's gradient, then n_extra piggy-backed scalars (loss ...)
 *   flag_off  : uint32[64]          barrier words, zero before the first step
 * ppb_dp_adam_step is ONE kernel: cross-rank barrier -> each rank sums ITS 1/world slice of the gradient
 * over all peers in fixed rank order (reduce-scatter by peer loads) -> Adam on that slice (exp_avg /
 * exp_avg_sq are local, only the slice is touched) -> the updated parameters are stored into every peer's
 * arena (all-gather by peer stores) -> cross-rank barrier.  The n_extra scalars are summed by rank 0 and
 * written back to every rank's gradient tail.  Replicas stay bit-identical: every element is reduced by
 * exactly one rank.  hyper_dev/state_dev as for ppb_adam_step_dev (grad_scale = 1/world); the step leaves
 * byte 12 of the state block untouched.  The call is
 * CUDA-graph capturable; all ranks must issue it the same number of times. */
int ppb_dp_alloc(int64_t bytes, void** ptr_out, void* ipc_handle_out /* 64 bytes */);
int ppb_dp_open(const void* ipc_handle /* 64 bytes, from another process */, void** ptr_out);
int ppb_dp_close(void* mapped_ptr);
int ppb_dp_free(void* ptr);
/* Stream-ordered cross-rank rendezvous over the same peer blocks (one tiny kernel: each rank releases a flag word in
 * every peer's block and waits for all of its own): work enqueued after it starts on all ranks at the same time.
 * Replaces the host-side dist.barrier() of the reference's training loop where only stream order matters; bench.py
 * uses it to start every timed step simultaneously on all ranks (the L2 flush before it is not part of the step). */
int ppb_dp_rendezvous(int world, int rank, void* const* peer_blocks, int64_t flag_off, void* stream);
int ppb_dp_adam_step(int world, int rank, void* const* peer_blocks /* host array [world], own block at [rank] */,
                     int64_t param_off, int64_t grad_off, int64_t flag_off, float* exp_avg,
                     float* exp_avg_sq, int64_t n, int64_t n_extra, const float* hyper_dev, void* state_dev,
                     void* stream);

/* Batched proposal step for IC posterior sampling (inference_network_lstm.py:82-134 for n particles in
 * lock-step at the same address).  h/c: fp32[n,H] LSTM state, updated in place (zeros at t=0).
 * prev_addr < 0 means first step.  Writes the proposal parameters:
 *   mixtures: params_out[n, 3K] = (means | stddevs | probs), categorical: params_out[n, C] = probs,
 *   bernoulli: params_out[n, 1] = probs.
 * Feed-forward net (inference_network_feedforward.py:53-66): prev_addr and prev_value are ignored, h and c may be NULL;
 * the head runs on the one shared observation row and its output is expanded over the n particles (only the priors
 * differ per particle). */
int ppb_ic_infer_step(ppb_net* net, const float* arena, const float* obs_emb /*[n or 1, E]*/,
                      int obs_emb_row_stride, int32_t prev_addr, const float* prev_value,
                      int32_t cur_addr, const float* prior0, int prior0_stride, const float* prior1,
                      int prior1_stride, float* h, float* c, float* params_out, int64_t n,
                      void* workspace, int64_t workspace_bytes, int precision, void* stream);
/* Observation embedding alone (inference_network.py:141-148 _infer_init): obs[n, obs_in_total] -> [n,E] */
int ppb_ic_embed_observe(ppb_net* net, const float* arena, const float* obs, float* obs_emb_out,
                         int64_t n, void* workspace, int64_t workspace_bytes, void* stream);
int64_t ppb_ic_infer_workspace_bytes(const ppb_net* net, int64_t n);
/* Rebuild the packed tf32 tile images of all GEMM weights from the arena (done automatically by
 * ppb_ic_loss_forward and ppb_ic_embed_observe; call it if the arena was modified by other means before
 * ppb_ic_infer_step). */
int ppb_net_refresh_weights(ppb_net* net, const float* arena, void* stream);
/* The loss and infer calls keep their problem and chunk lists in the caller's workspace and do not send a list again
 * while the same content already lives at the same address.  A caller that writes a workspace between two calls of one
 * net, or hands the net memory that held another workspace, calls this first: the next calls upload every list. */
int ppb_net_forget_uploads(ppb_net* net);

/* ------------------------------------------------------------------------------------------------
 * 5. Host-buffer convenience entry (the end-to-end call bench.py times as `e2e`)
 *    One IC training step from an encoded batch in HOST memory: H2D of the batch image,
 *    forward, backward, Adam, D2H of the loss.  batch_image_host is the packed layout produced by
 *    pyprob_b200.encoding.pack_batch (header ints + arrays); see DESIGN.md §3.
 *    The call returns when the step has finished (loss_host / status_host are valid).  After the first call
 *    with a given batch STRUCTURE the whole step — including both copies, staged through an internal pinned
 *    buffer, so batch_image_host need not be pinned — replays from one CUDA graph (PPB_HOST_STEP_GRAPH=0:
 *    the same launches, issued without capture).  Adam runs as ppb_adam_step_dev on a state block the net owns;
 *    `step` is the 1-based count after this step, and the block's counter is rewritten when it disagrees.
 * ---------------------------------------------------------------------------------------------- */
int ppb_ic_train_step_host(ppb_net* net, float* arena, float* grad_arena, float* exp_avg,
                           float* exp_avg_sq, int64_t arena_floats, const void* batch_image_host,
                           int64_t batch_image_bytes, void* batch_image_dev, void* workspace,
                           int64_t workspace_bytes, int precision, float lr, float beta1, float beta2,
                           float eps, float weight_decay, int64_t step, float* loss_host,
                           int32_t* status_host, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 6. Tensor-core building blocks exposed for tests (wgmma / bulk-TMA; sm_90a only)
 *    pack : row-major fp32 X[rows, K] (leading dim ldx) -> wgmma-ready K-major SWIZZLE_128B tile
 *           images (tf32 hi and lo parts), see DESIGN.md §4.
 *    gemm : C[M,N] (ldc) = A[M,K] * B[N,K]^T (+ bias[N]) (relu) from packed images, 3xTF32 or TF32.
 * ---------------------------------------------------------------------------------------------- */
int64_t ppb_packed_floats(int64_t rows, int64_t K);
int ppb_pack_tf32(const float* X, int64_t rows, int64_t K, int64_t ldx, float* hi_out, float* lo_out,
                  void* stream);
/* Same geometry, MN-major swizzle pattern (32-byte chunks permuted by (c ^ (row & 3))): the operand form whose reduction
 * runs along the image rows (weight-gradient and input-gradient GEMMs; the GEMM kernels rewrite it K-major in shared memory).  See DESIGN.md section 4. */
int ppb_pack_tf32_mn(const float* X, int64_t rows, int64_t K, int64_t ldx, float* hi_out, float* lo_out,
                     void* stream);
int ppb_gemm_packed(const float* A_hi, const float* A_lo, const float* B_hi, const float* B_lo,
                    float* C, int64_t M, int64_t N, int64_t K, int64_t ldc, const float* bias,
                    int relu, int precision, void* stream);
/* Same GEMM with the reduction of every 128 x 128 output tile split over a thread-block cluster of cluster_size (2, 4, 8)
 * CTAs whose partial tiles are combined through distributed shared memory (csrc/tc_cluster.cuh): the form the network
 * uses for its few-row, deep-K GEMMs — nn.LSTM's recurrent product h W_hh^T and its BPTT mirror
 * (pyprob/nn/inference_network_lstm.py:186-188), the proposal heads at small minibatches. */
int ppb_gemm_packed_cluster(const float* A_hi, const float* A_lo, const float* B_hi, const float* B_lo,
                            float* C, int64_t M, int64_t N, int64_t K, int64_t ldc, const float* bias,
                            int relu, int precision, int cluster_size, void* stream);

/* Phase-trace buffer for the tensor-core grouped GEMM: 64 launches x 16 int64 slots of globaltimer stamps written by
 * CTA 0 of each launch (setup, first data, last MMA commit, accumulators ready, epilogue done); NULL disables. */
int ppb_debug_trace(void* buf16_dev);
/* TN form over the same images: C[M,N] = sum_r X[r,m] * Y[r,n], X packed from [R,M], Y from [R,N]
 * (both operands MN-major; used by every weight-gradient GEMM: no transposed copies in HBM). */
int ppb_gemm_packed_tn(const float* X_hi, const float* X_lo, const float* Y_hi, const float* Y_lo,
                       float* C, int64_t M, int64_t N, int64_t R, int64_t ldc, int precision,
                       void* stream);
/* Runs n tensor-core GEMM descriptors (host array of tcg::Problem, csrc/tc_grouped.cuh; ppb_sizeof(5) bytes each) as one
 * launch of the kernel the network would use: cluster_size 1 = the grouped kernel, or its persistent form when the problems
 * have more tiles than SMs (PPB_PERSISTENT=0 keeps the grouped one); 2, 4, 8 = cluster split-K; chunk_table != 0 = the
 * grouped kernel that reads the K-major A through its chunk table.  epi: 0 = fp32 store, 1 = fp32 red.add, 2 = tile images
 * (+ fp32).  The tile bookkeeping (tiles_m, tiles_n, tile_start, k_splits >= 1) is filled in here.  Combinations the kernels
 * do not implement are refused before anything is uploaded or launched.  The K padding of the last 32-element reduction
 * chunk must be zero in both operands. */
int ppb_tc_run_problems(const void* problems_host, int n, int epi, int cluster_size, int chunk_table, int precision,
                        void* stream);

/* ------------------------------------------------------------------------------------------------
 * 7. Metropolis-Hastings chains (LMH / RMH), csrc/mcmc.cu.  C chains run as the C lanes of one lock-step execution.
 *    Trace tables, column = address (assigned in order of first appearance, pyprob_b200/mcmc.py), row = (buffer, chain):
 *      val[2, C, lda] fp32, lp[2, C, lda] fp32 prior log-prob, stamp[2, C, lda] int32, reused[2, C, lda] uint8.
 *    buf[c] (0 / 1) is the buffer of chain c's current trace, 1 - buf[c] its candidate's; accepting flips buf[c].  A cell
 *    belongs to the current trace iff its stamp equals cur_stamp[c] (the step that made the trace), to the candidate iff
 *    it equals the running step: nothing is ever cleared.
 *    Philox key = seed, counter = (chain index c, offset):
 *      site choice (ppb_mh_select): m present columns of the current row, u = (w0 >> 8) 2^-24 from word 0,
 *        k = min(floor(u m), m - 1) in fp32, the chosen column is the k-th present one in increasing column order.
 *      accept (ppb_mh_accept): u = ((w0 >> 8) + 1) 2^-24 from word 0; accept iff log(u) < log alpha (fp64), where
 *        log alpha = log cur_n - log cand_n + cand_lpo - cur_lpo + reuse + trans, and -inf when cand_n = 0.
 *      RMH kernel at the chosen site (ppb_mh_site, kind 1 / 2): the kernel draws iff (w0 >> 8) 2^-24 < 0.5, from
 *        words 1, 2 (Normal: Box-Muller, as the Normal sampler) or word 1 (Uniform: inverse-CDF truncated normal).
 * ---------------------------------------------------------------------------------------------- */
#define PPB_MH_KERNEL_PRIOR 0
#define PPB_MH_KERNEL_NORMAL 1
#define PPB_MH_KERNEL_UNIFORM 2
/* Start a step: reset the candidate accumulators (cand_n, cand_lpo, reuse, trans) and, unless initial, write each chain's
 * chosen column into choice (-1 when its current trace has no site, and always for the initial step). */
int ppb_mh_select(const int32_t* stamp, const int32_t* buf, const int32_t* cur_stamp, int64_t C, int64_t lda, int ncols,
                  int32_t* choice, int32_t* cand_n, double* cand_lpo, double* reuse, double* trans, int initial,
                  uint64_t seed, uint64_t offset, void* stream);
/* Rows first .. first + n - 1: the current trace's value and log-prob at column col (has = 0 where it has none or the
 * lane is masked out). */
int ppb_mh_fetch(const float* val, const float* lp, const int32_t* stamp, const int32_t* buf, const int32_t* cur_stamp,
                 int64_t C, int64_t lda, int col, const uint8_t* mask, int64_t n, int64_t first, float* old_v,
                 float* old_lp, uint8_t* has, void* stream);
/* One executed sample statement: per executing lane, the chosen site takes the fresh prior draw (kind 0) or the RMH
 * kernel mixture (writing trans); otherwise the current value is reused where has and rescored > -inf (reuse +=
 * rescored - old_lp), else the fresh draw is taken.  Writes the candidate cell, cand_n += 1 and value_out. */
int ppb_mh_site(int kind, int col, const uint8_t* mask, int64_t n, int64_t first, const float* fresh_v,
                const float* fresh_lp, const float* old_v, const float* old_lp, const uint8_t* has,
                const float* rescored, const float* p0, int p0_stride, const float* p1, int p1_stride, float* val,
                float* lp, int32_t* stamp, uint8_t* reused_flag, const int32_t* buf, const int32_t* choice,
                int32_t step, int64_t C, int64_t lda, int32_t* cand_n, double* reuse, double* trans,
                int64_t* reused_cnt, float* value_out, uint64_t seed, uint64_t offset, void* stream);
/* End a step: log alpha and the accept draw per chain (initial: accept always), flip and count, then copy the current
 * map_func row (map_words 32-bit words) into out[slot] when slot >= 0. */
int ppb_mh_accept(int64_t C, int initial, int32_t step, int32_t* buf, int32_t* cur_stamp, int32_t* cur_n,
                  double* cur_lpo, const int32_t* cand_n, const double* cand_lpo, const double* reuse,
                  const double* trans, double* log_alpha, int64_t* accepted, int64_t* sites_all,
                  const int32_t* cand_map, int32_t* cur_map, int map_words, int32_t* out, int64_t slot, uint64_t seed,
                  uint64_t offset, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 8. MCMC diagnostics, csrc/diagnostics.cu: Gelman-Rubin R-hat against the prefix length and per-chain autocorrelation
 *    (replaces pyprob/diagnostics.py:714-873, the reference's python loops over traces, lags and steps).
 *    x holds S steps of C chains of V variables: x[s, c, v] at element s * stride_s + c * stride_c + v * stride_v, fp32
 *    (PPB_DIAG_F32) or fp64 (PPB_DIAG_F64).  iters / lags are HOST int64 arrays; out is device fp64.  Every statistic is
 *    accumulated in fp64 in a fixed order (two calls give the same bits); means and variances are Welford / Chan
 *    combinations, never sum(x^2) - sum(x)^2 / n.  The caller allocates the device workspace of the size the
 *    *_workspace_bytes function returns for the same arguments (-1: invalid arguments).  R-hat's workspace is
 *    at most max(256 MiB, (2^17 + C V) * 16 B) + n_distinct_iters * V * ceil(C / 256) * 32 B, so a per-iteration curve
 *    (iters = 1 .. S) costs 32 B per (iteration, variable, 256 chains), not per chain; autocorrelation's is at most about 1 GiB of per-chunk
 *    partials plus 16 B per value column.
 *    R-hat (diagnostics.py:788-796), for every iters[i] (any order, >= 1; values above S mean S) with n = min(iters[i], S)
 *    and m = C: b = n var(chain means of x[:n], ddof 1), w = mean(chain variances of x[:n], ddof 1),
 *    out[v * n_iters + i] = sqrt(((n - 1) / n w + b / n) / w) -- NaN at n = 1, inf / NaN where w = 0, as numpy.  C >= 2.
 *    Autocorrelation (diagnostics.py:720-736), for every lags[l] in [0, S]: with mu the chain's mean over all S steps,
 *    out[(v * C + c) * n_lags + l] = sum_{i < S - lag} (x_i - mu)(x_{i+lag} - mu) / (1e-8 + sum_i (x_i - mu)^2).
 * ---------------------------------------------------------------------------------------------- */
#define PPB_DIAG_F32 0
#define PPB_DIAG_F64 1
int64_t ppb_diag_rhat_workspace_bytes(int64_t S, int64_t C, int64_t V, const int64_t* iters, int n_iters);
int ppb_diag_rhat(const void* x, int dtype, int64_t S, int64_t C, int64_t V, int64_t stride_s, int64_t stride_c,
                  int64_t stride_v, const int64_t* iters, int n_iters, double* out, void* workspace,
                  int64_t workspace_bytes, void* stream);
int64_t ppb_diag_autocorr_workspace_bytes(int dtype, int64_t S, int64_t C, int64_t V, int n_lags);
int ppb_diag_autocorr(const void* x, int dtype, int64_t S, int64_t C, int64_t V, int64_t stride_s, int64_t stride_c,
                      int64_t stride_v, const int64_t* lags, int n_lags, double* out, void* workspace,
                      int64_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PYPROB_B200_H */
