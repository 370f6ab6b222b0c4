// Proposal network: observe embedding -> LSTM -> per-address heads -> NLL, forward and the
// hand-differentiated backward, over an encoded trace minibatch (include/pyprob_b200.h section 4).
// Replaces pyprob/nn/inference_network_lstm.py:136-220 (_loss) + autograd (inference_network.py:493).
//
// Algorithmic restructuring relative to the reference's per-(t,b) concatenation (:146-182): the LSTM
// input GEMM x_t W_ih^T is split by the block structure of x_t = [obs_emb(b) | smp_emb(t,b) | step_emb(t,s)]:
//   P_obs[b]    = obs_emb[b]  W_ih[:, :E]^T           once per trace          (GEMM, K = E)
//   P_step[t,s] = step_emb    W_ih[:, E+S:]^T + b_ih + b_hh   once per (step, sub-batch) (k_pstep_fwd, K = 2(td+ad))
//   smp term    = sum_j smp_emb[t,b,j] W_ih[:, E+j]   S FMAs per gate element, fused in the cell kernel
// which removes the T-fold recomputation of the observation block.
#include <vector>
#include <string.h>
#include <stdlib.h>
#include <stdint.h>

#include "common.cuh"
#include "gemm_simt.cuh"
#include "heads.cuh"
#include "tc_grouped.cuh"
#include "tc_lstm.cuh"
#include "tc_cluster.cuh"
#include "tc_persist.cuh"
#include "tc_launch.cuh"
#include "obs_mlp.cuh"

using gemm::Problem;

// tile images of one tensor (either format may be absent); passed by value to element-wise kernels
struct HImg {
  float* k_hi = nullptr; float* k_lo = nullptr; float* mn_hi = nullptr; float* mn_lo = nullptr;
  int64_t kb = 0;
};

struct WImg {  // tile images of one weight matrix (float offsets into ppb_net::wimg)
  int64_t k_hi = 0, k_lo = 0, mn_hi = 0, mn_lo = 0;
  int kb = 0;
};
struct PackEntry {  // one matrix of the weight-packing table
  int64_t src_off;  // floats from the arena base
  int rows, cols, ld, kb;
  int64_t k_hi, k_lo, mn_hi, mn_lo;
  int tile_start, pad_;
};

// how the tensor-core pipeline runs the observe embedding (obs_embed.inc)
enum class ObsForm { fused, tensor_core, simt };

// The device regions whose last upload ppb_net remembers (upload_cached): the problem lists of a loss call (SIMT and tensor
// core, forward in the first half of a region and backward in the second, and the tensor-core backward's reduction chunks),
// those of an inference call, and the fused LSTM step list, which lives in memory the net owns.  forget_on_new_layout
// forgets the lists of one kind of call: a contiguous range.
enum UploadSlot {
  kSlotSimtFwd, kSlotSimtBwd, kSlotTcFwd, kSlotTcBwd, kSlotChunks,  // loss calls (ws_layout)
  kSlotInferSimt, kSlotInferTc,                                       // observe embedding and infer step (infer_layout)
  kSlotLstmSteps,
  kNumUploadSlots
};

struct ppb_net {
  // tensor-core path: packed tf32 images of every GEMM weight, refreshed from the arena each forward
  float* wimg = nullptr;
  int64_t wimg_floats = 0;
  std::vector<PackEntry> pack;
  PackEntry* d_pack = nullptr;
  int pack_tiles = 0;
  WImg w_ihE, w_hh;
  std::vector<WImg> w1, w2;
  ObsForm obs_form = ObsForm::simt;   // chosen when the tables are set
  // tensor-core form of the observe embedding: layers >= 1 of every observable chain, the final chain
  WImg w_obs[PPB_MAX_OBS][PPB_MAX_FF_LAYERS];
  WImg w_fin[PPB_MAX_FF_LAYERS];
  // content hashes of the problem lists last uploaded to each device region: identical lists are not re-sent,
  // which also makes a repeated step capturable in a CUDA graph (no host->device copy inside the capture)
  uint64_t slot_hash[kNumUploadSlots] = {};
  const void* slot_dev[kNumUploadSlots] = {};
  uint64_t ws_layout = 0;      // workspace address, batch dims and precision of the last loss call (forget_on_new_layout)
  uint64_t infer_layout = 0;   // workspace address, particle count and entry of the last inference call
  void* h_blob[2] = {nullptr, nullptr};
  cudaEvent_t ev_blob[2] = {nullptr, nullptr};
  size_t blob_cap = 0;
  int blob_idx = 0;
  ppb_net_desc desc;
  std::vector<ppb_addr_desc> addrs;
  std::vector<int64_t> type_off;
  ppb_addr_desc* d_addrs = nullptr;
  int64_t* d_type_off = nullptr;
  int64_t arena_floats = 0;
  int I = 0;        // LSTM input width  E + S + 2 (td + ad)
  int dh_pad = 4;   // max head hidden width, padded to 4
  int out_pad = 4;  // max head output width, padded to 4
  // LSTM cell fused into the recurrent GEMM (tc_lstm.cuh, tc_cluster.cuh); PPB_FUSED_CELL=0: GEMM and cell kernels
  bool fused_cell = true;
  float* whh_il = nullptr;          // gate-interleaved K-format image of W_hh: hi part, then lo part
  int64_t whh_il_floats = 0;        // floats per part
  void* d_lstm_steps = nullptr;     // device list of tcl::Step
  size_t lstm_steps_cap = 0;        // bytes
  // side streams: independent branches of the step run beside the critical path (captured into the same CUDA graph)
  cudaStream_t side[2] = {nullptr, nullptr};
  cudaEvent_t fork_ev[16] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                             nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  int fork_next = 0;
  int pack_tiles_no_hh = 0;         // weight-image tiles without W_hh (a T = 1 step never reads it)
  // ppb_ic_train_step_host: the whole step cached as an instantiated CUDA graph per batch structure
  int host_graph = 1;               // PPB_HOST_STEP_GRAPH=0 disables
  cudaStream_t host_stream = nullptr;
  cudaGraphExec_t host_exec = nullptr;
  uint64_t host_key = 0;
  int host_seen = 0;
  float* host_hyper_dev = nullptr;  // [PPB_HYPER_ADAM_COUNT] (include/pyprob_b200.h)
  void* host_state_dev = nullptr;   // Adam state block (include/pyprob_b200.h)
  float host_hyper[PPB_HYPER_ADAM_COUNT] = {0, 0, 0, 0, 0, 0};
  int64_t host_step_dev = -1;       // value of the device step counter
  char* host_pin = nullptr;         // pinned staging: [image bytes | 8 B loss + status]; both copies are nodes of the step graph
  int64_t host_pin_cap = 0;
  // pinned staging ring for problem lists
  Problem* h_stage[2] = {nullptr, nullptr};
  cudaEvent_t ev_stage[2] = {nullptr, nullptr};
  size_t stage_cap = 0;
  int stage_idx = 0;
};

namespace {

inline int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

// ---------------------------------------------------------------------------------------------------
// workspace carving
// ---------------------------------------------------------------------------------------------------
struct Ws {
  // forward
  float* obs_act[PPB_MAX_OBS][PPB_MAX_FF_LAYERS];
  float* obs_cat; float* fin_act[PPB_MAX_FF_LAYERS]; float* obs_emb;
  float* p_obs; float* emb_cat; float* p_step; float* w_smp_t; float* smp_emb;
  float* gates; float* c; float* h; float* hid; float* out_raw; float* row_lp; float* d_out;
  float* loss_acc;  // [0] = sum of -lp ; int status at [1]
  // backward
  float* d_hid; float* dh; float* dh_rec; float* dc; float* d_pobs; float* d_pstep;
  float* d_obs_emb; float* d_fin_act[PPB_MAX_FF_LAYERS]; float* d_obs_cat; float* d_obs_act[PPB_MAX_OBS][PPB_MAX_FF_LAYERS];
  Problem* problems; // device problem list
  int64_t max_problems;
  int64_t total_bytes;
};

struct Dims {
  int B, R, T, NS, G;
};

Ws carve(const ppb_net* net, Dims d, void* base) {
  const ppb_net_desc& D = net->desc;
  Ws w;
  memset(&w, 0, sizeof(w));
  char* p = (char*)base;
  int64_t off = 0;
  auto take = [&](int64_t floats) {
    float* r = (float*)(p + off);
    off += align_up(floats * 4, 256);
    return r;
  };
  const int H = D.lstm_dim, E = D.obs_dim, S = D.sample_dim, C2 = 2 * (D.type_dim + D.addr_dim);
  // h / dh: the rows the heads read and their gradient — the LSTM output, or (feed-forward, fp32 path) the observation
  // embedding of each row's trace.  A feed-forward net has H = S = C2 = 0: none of the LSTM buffers take space.
  const int HX = D.network_type == PPB_NET_FEEDFORWARD ? E : H;
  for (int j = 0; j < D.num_obs; ++j)
    for (int l = 0; l + 1 < D.obs_ff[j].num_layers; ++l) w.obs_act[j][l] = take((int64_t)d.B * D.obs_ff[j].layers[l].out_dim);
  w.obs_cat = take((int64_t)d.B * E);
  for (int l = 0; l + 1 < D.obs_final.num_layers; ++l) w.fin_act[l] = take((int64_t)d.B * D.obs_final.layers[l].out_dim);
  w.obs_emb = take((int64_t)d.B * E);
  w.p_obs = take((int64_t)d.B * 4 * H);
  w.emb_cat = take((int64_t)d.NS * C2);
  w.p_step = take((int64_t)d.NS * 4 * H);
  w.w_smp_t = take((int64_t)S * 4 * H);
  w.smp_emb = take((int64_t)d.R * S);
  w.gates = take((int64_t)d.R * 4 * H);
  w.c = take((int64_t)d.R * H);
  w.h = take((int64_t)d.R * HX);
  w.hid = take((int64_t)d.R * net->dh_pad);
  w.out_raw = take((int64_t)d.R * net->out_pad);
  w.row_lp = take(d.R);
  w.d_out = take((int64_t)d.R * net->out_pad);
  w.loss_acc = take(64);
  w.d_hid = take((int64_t)d.R * net->dh_pad);
  w.dh = take((int64_t)d.R * HX);
  w.dh_rec = take((int64_t)d.R * H);
  w.dc = take((int64_t)d.R * H);
  w.d_pobs = take((int64_t)d.B * 4 * H);
  w.d_pstep = take((int64_t)d.NS * 4 * H);   // d_pstep and d_obs_emb are adjacent: the tensor-core backward zeroes both at once
  w.d_obs_emb = take((int64_t)d.B * E);
  for (int l = 0; l + 1 < D.obs_final.num_layers; ++l) w.d_fin_act[l] = take((int64_t)d.B * D.obs_final.layers[l].out_dim);
  w.d_obs_cat = take((int64_t)d.B * E);
  for (int j = 0; j < D.num_obs; ++j)
    for (int l = 0; l + 1 < D.obs_ff[j].num_layers; ++l) w.d_obs_act[j][l] = take((int64_t)d.B * D.obs_ff[j].layers[l].out_dim);
  // dgates reuses `gates`?  No: backward needs the activations; keep a separate buffer.
  w.max_problems = 2 * (64 + 4LL * PPB_MAX_OBS * PPB_MAX_FF_LAYERS + 8LL * d.G + 4LL * d.T);  // fwd | bwd halves
  w.problems = (Problem*)take(w.max_problems * (int64_t)(sizeof(Problem) / 4));
  w.total_bytes = off;
  return w;
}

// dgates lives after the carved region (largest buffer; only needed by backward)
inline float* dgates_ptr(const Ws& w, void* base) { return (float*)((char*)base + w.total_bytes); }
inline int64_t dgates_bytes(const ppb_net* net, Dims d) { return align_up((int64_t)d.R * 4 * net->desc.lstm_dim * 4, 256); }

// ---------------------------------------------------------------------------------------------------
// problem-list builder
// ---------------------------------------------------------------------------------------------------
struct Builder {
  std::vector<Problem> probs;
  std::vector<gemm::Phase> phases;
  void begin() { gemm::Phase ph; ph.first = (int)probs.size(); phases.push_back(ph); }
  void add(Problem p) {
    gemm::Phase& ph = phases.back();
    p.tiles_m = (p.M + gemm::BM - 1) / gemm::BM;
    p.tiles_n = (p.N + gemm::BN - 1) / gemm::BN;
    p.tile_start = ph.tiles;
    if (p.M <= 0 || p.N <= 0) return;
    ph.tiles += p.tiles_m * p.tiles_n;
    ph.count += 1;
    probs.push_back(p);
  }
};

inline Problem P0() {
  Problem p;
  memset(&p, 0, sizeof(p));
  p.alpha = 1.0f;
  return p;
}

// Y[M, N] (ldy) = act(X[M,K] (ldx) W[N,K]^T (ldw) + b)
inline Problem linear_fwd(const float* X, int64_t ldx, const float* W, int64_t ldw, const float* b, float* Y,
                          int64_t ldy, int M, int N, int K, int flags) {
  Problem p = P0();
  p.A = X; p.sam = ldx; p.sak = 1;
  p.B = W; p.sbn = ldw; p.sbk = 1;
  p.C = Y; p.ldc = ldy; p.bias = b;
  p.M = M; p.N = N; p.K = K; p.flags = flags;
  return p;
}
// dX[M,K] (lddx) = dY[M,N] (lddy) W[N,K] (ldw)
inline Problem linear_dx(const float* dY, int64_t lddy, const float* W, int64_t ldw, float* dX, int64_t lddx, int M,
                         int N, int K, int flags) {
  Problem p = P0();
  p.A = dY; p.sam = lddy; p.sak = 1;   // reduction index = n
  p.B = W; p.sbn = 1; p.sbk = ldw;     // B(k_out, n) = W[n*ldw + k_out]
  p.C = dX; p.ldc = lddx;
  p.M = M; p.N = K; p.K = N; p.flags = flags;
  return p;
}
// dW[N,K] (ldw) += dY[M,N]^T X[M,K]   (reduction over rows m)
inline Problem linear_dw(const float* dY, int64_t lddy, const float* X, int64_t ldx, float* dW, int64_t ldw, int M,
                         int N, int K) {
  Problem p = P0();
  p.A = dY; p.sam = 1; p.sak = lddy;   // A(n_out, m) = dY[m*lddy + n_out]
  p.B = X; p.sbn = 1; p.sbk = ldx;     // B(k_in, m)  = X[m*ldx + k_in]
  p.C = dW; p.ldc = ldw;
  p.M = N; p.N = K; p.K = M; p.flags = gemm::kAccumulate;
  return p;
}

inline uint64_t fnv1a(const void* data, size_t n, uint64_t h = 1469598103934665603ULL) {
  const unsigned char* p = (const unsigned char*)data;
  for (size_t i = 0; i < n; ++i) { h ^= p[i]; h *= 1099511628211ULL; }
  return h;
}

// Send `bytes` of host data to `dev` through the pinned staging ring unless the same content already lives there.
int upload_cached(ppb_net* net, UploadSlot slot, const void* src, size_t bytes, void* dev, cudaStream_t st) {
  if (bytes == 0) return PPB_OK;
  uint64_t h = fnv1a(src, bytes, 1469598103934665603ULL ^ (uint64_t)bytes);
  if (net->slot_hash[slot] == h && net->slot_dev[slot] == dev) return PPB_OK;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(st, &cap);
  if (cap != cudaStreamCaptureStatusNone) {
    ppb_set_error("the batch structure changed inside a CUDA-graph capture: run the step once eagerly first");
    return PPB_EINVAL;
  }
  if (net->blob_cap < bytes) {
    for (int i = 0; i < 2; ++i) {
      if (net->h_blob[i]) cudaFreeHost(net->h_blob[i]);
      PPB_CUDA(cudaMallocHost(&net->h_blob[i], bytes * 2));
      if (!net->ev_blob[i]) PPB_CUDA(cudaEventCreateWithFlags(&net->ev_blob[i], cudaEventDisableTiming));
    }
    net->blob_cap = bytes * 2;
  }
  int i = net->blob_idx;
  net->blob_idx ^= 1;
  PPB_CUDA(cudaEventSynchronize(net->ev_blob[i]));
  memcpy(net->h_blob[i], src, bytes);
  PPB_CUDA(cudaMemcpyAsync(dev, net->h_blob[i], bytes, cudaMemcpyHostToDevice, st));
  PPB_CUDA(cudaEventRecord(net->ev_blob[i], st));
  net->slot_hash[slot] = h;
  net->slot_dev[slot] = dev;
  return PPB_OK;
}

// Send a SIMT problem list of at most `cap` problems to `dev`, tracked as `slot` (UploadSlot)
int upload_and_get(ppb_net* net, const Builder& b, Problem* dev, int64_t cap, cudaStream_t st, UploadSlot slot) {
  size_t n = b.probs.size();
  if ((int64_t)n > cap) { ppb_set_error("problem list overflow (%zu > %lld)", n, (long long)cap); return PPB_ENOMEM; }
  return upload_cached(net, slot, b.probs.data(), n * sizeof(Problem), dev, st);
}

// ---- side streams -------------------------------------------------------------------------------------
// `to` continues after everything enqueued on `from` so far (event record + wait: both are graph-capturable, the
// side stream joins the capture and must be joined back before the capture ends).
int stream_after(ppb_net* net, cudaStream_t from, cudaStream_t to) {
  if (from == to) return PPB_OK;
  cudaEvent_t& ev = net->fork_ev[net->fork_next];
  net->fork_next = (net->fork_next + 1) & 15;
  if (!ev) PPB_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  PPB_CUDA(cudaEventRecord(ev, from));
  PPB_CUDA(cudaStreamWaitEvent(to, ev, 0));
  return PPB_OK;
}
// ---- optional kernel-level profiling of the LSTM gate GEMM class (bench.py roofline) ---------------
struct Prof {
  bool on = false;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> spans;
  double flops = 0.0;
  int64_t launches = 0;
} g_prof;

// The profiling argument of a phase runner for phase `i` of a problem list (Builder, TcBuilder): the phase's FLOPs, or 0 (not
// profiled) while profiling is off
template <typename B>
double profile(const B& bl, int i) {
  if (!g_prof.on) return 0.0;
  const gemm::Phase& ph = bl.phases[i];
  double f = 0.0;
  for (int j = 0; j < ph.count; ++j) { const auto& p = bl.probs[ph.first + j]; f += 2.0 * p.M * p.N * p.K; }
  return f;
}

int run_phase(const gemm::Phase& ph, const Problem* dev, cudaStream_t st, double prof_flops = 0.0) {
  if (ph.count == 0) return PPB_OK;
  int grid = ph.tiles < 8 * PPB_NUM_SMS ? ph.tiles : 8 * PPB_NUM_SMS;
  return profiled(prof_flops, st, [&] {
    gemm::k_grouped<<<grid, gemm::kThreads, 0, st>>>(dev + ph.first, ph.count, ph.tiles);
    PPB_LAUNCH_CHECK();
    return PPB_OK;
  });
}

// ---------------------------------------------------------------------------------------------------
// element-wise / fused kernels
// ---------------------------------------------------------------------------------------------------
// Arena offset of column j of a step-embedding row [prev_type | prev_addr | cur_type | cur_addr]
// (inference_network_lstm.py:175-180), or -1 in the previous half when there is no previous site (t = 0).
// desc(is_prev, a) points a at the descriptor of that half and returns false when there is no site; only the half that
// column j needs is looked up.
template <typename Desc>
__device__ __forceinline__ int64_t step_embed_off(const int64_t* __restrict__ type_off, int td, int ad, int j, Desc desc) {
  const bool is_prev = j < td + ad;
  const ppb_addr_desc* a;
  if (!desc(is_prev, a)) return -1;
  const int jj = is_prev ? j : j - (td + ad);
  return jj < td ? type_off[a->type_id] + jj : a->addr_emb_off + (jj - td);
}

// Pre-activation of unit j of an address's sample embedding at value x: b[j] + W[j] . x, with x one-hot for a Categorical
// address (inference_network_lstm.py:168-169, embedding_feedforward.py:35-48)
__device__ __forceinline__ float smp_embed_pre(const float* __restrict__ arena, const ppb_addr_desc& a, float x, int j) {
  const float* W = arena + a.smp_w_off + (int64_t)j * a.smp_in;
  float pre = arena[a.smp_b_off + j];
  if (a.family == PPB_FAMILY_CATEGORICAL) {
    const int c = (int)x;
    if (c >= 0 && c < a.smp_in) pre += W[c];
  } else {
    pre += W[0] * x;
  }
  return pre;
}

// step embedding rows, one per (step, sub-batch)
__global__ void k_step_embed(const float* __restrict__ arena, const ppb_addr_desc* __restrict__ addrs,
                             const int64_t* __restrict__ type_off, const int* __restrict__ step_addr,
                             const int* __restrict__ step_prev, int n_steps, int td, int ad,
                             float* __restrict__ emb_cat) {
  int C2 = 2 * (td + ad);
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < (int64_t)n_steps * C2;
       e += (int64_t)gridDim.x * blockDim.x) {
    int st = (int)(e / C2), j = (int)(e % C2);
    const int64_t o = step_embed_off(type_off, td, ad, j, [&](bool is_prev, const ppb_addr_desc*& a) {
      const int which = is_prev ? step_prev[st] : step_addr[st];
      a = addrs + which;
      return which >= 0;
    });
    emb_cat[e] = o >= 0 ? arena[o] : 0.0f;
  }
}

// transposed copy of the sample-embedding columns of W_ih: w_smp_t[j][col] = W_ih[col, E + j]
__global__ void k_wsmp_transpose(const float* __restrict__ w_ih, int I, int E, int S, int H4,
                                 float* __restrict__ w_smp_t) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < S * H4; e += gridDim.x * blockDim.x) {
    int j = e / H4, col = e % H4;
    w_smp_t[e] = w_ih[(int64_t)col * I + E + j];
  }
}

// previous-sample embedding per row: relu of the previous address's sample-embedding layer; zeros at t = 0 (:157)
__global__ void k_smp_embed(const float* __restrict__ arena, const ppb_addr_desc* __restrict__ addrs,
                            const int* __restrict__ row_step, const int* __restrict__ step_prev,
                            const int* __restrict__ row_prev, const float* __restrict__ values, int R, int S,
                            float* __restrict__ smp_emb) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < (int64_t)R * S;
       e += (int64_t)gridDim.x * blockDim.x) {
    int row = (int)(e / S), j = (int)(e % S);
    int pa = step_prev[row_step[row]];
    smp_emb[e] = pa >= 0 ? fmaxf(smp_embed_pre(arena, addrs[pa], values[row_prev[row]], j), 0.0f) : 0.0f;
  }
}

// LSTM cell forward of one (row, unit) from its gate pre-activations (torch.nn.LSTM gate order i, f, g, o): the activations,
// c_t and h_t.  c_prev() returns c_{t-1}; it is called after the activations, where both cell kernels issue that load.
struct CellFwd { float i, f, g, o, c, h; };
template <typename CPrev>
__device__ __forceinline__ CellFwd cell_fwd_unit(const float (&pre)[4], CPrev c_prev) {
  const float i = ppb_cell_sigmoid(pre[0]), f = ppb_cell_sigmoid(pre[1]);
  const float g = ppb_cell_tanh(pre[2]), o = ppb_cell_sigmoid(pre[3]);
  const float c = f * c_prev() + i * g;
  return {i, f, g, o, c, o * ppb_cell_tanh(c)};
}

// LSTM cell, one time step, all active rows (h0 = c0 = 0, :186-187)
__global__ void __launch_bounds__(256) k_cell_fwd(float* __restrict__ gates, const float* __restrict__ p_obs,
                                                   const float* __restrict__ p_step, const float* __restrict__ w_smp_t,
                                                   const float* __restrict__ smp_emb, const int* __restrict__ row_step,
                                                   const int* __restrict__ row_prev, const int* __restrict__ row_trace,
                                                   float* __restrict__ c, float* __restrict__ h, HImg himg, int row0,
                                                   int n_rows, int H, int S, int t) {
  ppb_pdl_trigger();
  ppb_pdl_wait();
  int64_t total = (int64_t)n_rows * H;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    int i = (int)(e / H), j = (int)(e % H);
    int row = row0 + i;
    int st = row_step[row];
    int tr = row_trace[row];
    if (tr < 0) {  // padding row of a 128-row segment: keep every consumer's reduction clean
      gates[(int64_t)row * 4 * H + j] = 0.f; gates[(int64_t)row * 4 * H + H + j] = 0.f;
      gates[(int64_t)row * 4 * H + 2 * H + j] = 0.f; gates[(int64_t)row * 4 * H + 3 * H + j] = 0.f;
      c[(int64_t)row * H + j] = 0.f; h[(int64_t)row * H + j] = 0.f;
      if (himg.k_hi) tcg::img_store(himg.k_hi, himg.k_lo, himg.mn_hi, himg.mn_lo, row, j, himg.kb, 0.0f);
      continue;
    }
    float pre[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      int col = g * H + j;
      float v = p_obs[(int64_t)tr * 4 * H + col] + p_step[(int64_t)st * 4 * H + col];
      if (t > 0) {
        v += gates[(int64_t)row * 4 * H + col];  // recurrent part written by the GEMM
        for (int s = 0; s < S; ++s) v = fmaf(smp_emb[(int64_t)row * S + s], w_smp_t[(int64_t)s * 4 * H + col], v);
      }
      pre[g] = v;
    }
    const CellFwd u = cell_fwd_unit(pre, [&] { return (t > 0) ? c[(int64_t)row_prev[row] * H + j] : 0.0f; });
    gates[(int64_t)row * 4 * H + j] = u.i;
    gates[(int64_t)row * 4 * H + H + j] = u.f;
    gates[(int64_t)row * 4 * H + 2 * H + j] = u.g;
    gates[(int64_t)row * 4 * H + 3 * H + j] = u.o;
    c[(int64_t)row * H + j] = u.c;
    h[(int64_t)row * H + j] = u.h;
    if (himg.k_hi) tcg::img_store(himg.k_hi, himg.k_lo, himg.mn_hi, himg.mn_lo, row, j, himg.kb, u.h);
  }
}

// heads: family transform + log q(value) + d(-log q)/d out, loss reduction (:199-218).
// One WARP per row: lane k owns mixture component k (or categories k, k+32, ...), reductions are shuffles;
// the transforms are those of heads.cuh and the log q those of the reference's Mixture / TruncatedNormal / Categorical /
// Bernoulli, with d(-log q)/d out derived by hand (tests/heads_fp64.py states the same formulas in fp64 with autograd).
// nll_row is the per-row routine (x = the row's raw head outputs, global or shared memory); two callers:
// k_head_nll (x read from the output of the h2 GEMM) and NllRowEpi (x parked in shared memory by the h2 cluster GEMM, below).
struct NllArgs {
  const ppb_addr_desc* addrs;
  const int* row_step; const int* step_addr;
  const float* values; const float* prior0; const float* prior1;
  const int* row_trace;
  int K; float inv_batch;
  float* row_lp; float* d_out; int out_pad;
  HImg dimg;
};
// what the NLL of a row reads besides its head outputs: a chain of dependent loads (row -> step -> address), which a caller
// may issue long before the outputs exist (NllRowEpi: before the GEMM mainloop)
struct NllRowIn {
  bool valid;
  int O, family, C;
  float v, p0, p1;
};
__device__ __forceinline__ NllRowIn nll_row_in(const NllArgs& A, int row) {
  NllRowIn in;
  in.valid = A.row_trace[row] >= 0;
  in.O = 0; in.family = 0; in.C = 0; in.v = 0.f; in.p0 = 0.f; in.p1 = 0.f;
  if (in.valid) {
    const ppb_addr_desc& a = A.addrs[A.step_addr[A.row_step[row]]];
    in.O = a.head_out; in.family = a.family; in.C = a.num_categories;
    in.v = A.values[row]; in.p0 = A.prior0[row]; in.p1 = A.prior1[row];
  }
  return in;
}
__device__ __forceinline__ void nll_row(const NllArgs& A, const NllRowIn& in, const float* x, int row, int lane, float& local,
                                        int& bad) {
  const int K = A.K, out_pad = A.out_pad;
  const float inv_batch = A.inv_batch;
  float* row_lp = A.row_lp; float* d_out = A.d_out;
  const HImg dimg = A.dimg;
  const int img_cols = (int)dimg.kb * 32;
  const bool valid = in.valid;
  float g0 = 0.f, g1 = 0.f, g2 = 0.f, g3 = 0.f;  // this lane's gradient entries (mixture: m,s,p ; categorical: 4 cats)
  float lp = 0.0f;
  int O = 0;
  bool is_cat = false, is_bern = false;
  if (valid) {
    const float v = in.v;
    O = in.O;
    is_cat = in.family == PPB_FAMILY_CATEGORICAL;
    is_bern = in.family == PPB_FAMILY_BERNOULLI;
    if (is_bern) {
      // one output: p = sigmoid(x) + 1e-8, lp = v log pc + (1 - v) log(1 - pc); every lane computes it, lane 0's counts.
      // d(-lp)/dx = -(v / pc - (1 - v) / (1 - pc)) sigma (1 - sigma), zero where the clamp is active
      if (v != 0.0f && v != 1.0f) {
        lp = NAN;
      } else {
        const float sg = heads::sigmoidf_(x[0]);
        const float p = sg + PPB_UTIL_EPSILON;
        const float pc = ppb_clamp_prob(p);
        lp = (v == 1.0f) ? logf(pc) : log1pf(-pc);
        const bool clamped = (p < PPB_EPS32) || (p > 1.0f - PPB_EPS32);
        if (!clamped) g0 = -((v == 1.0f) ? 1.0f / pc : -1.0f / (1.0f - pc)) * (sg * (1.0f - sg));
      }
    } else if (is_cat) {
      const int C = in.C;
      float q[4], xs[4];
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 4; ++i) { int c = lane + 32 * i; xs[i] = c < C ? x[c] : -INFINITY; mx = fmaxf(mx, xs[i]); }
      mx = ppb_warp_max(mx);
      float s = 0.0f;
#pragma unroll
      for (int i = 0; i < 4; ++i) { q[i] = (lane + 32 * i < C) ? expf(xs[i] - mx) : 0.0f; s += q[i]; }
      s = ppb_warp_sum(s);
      float S = 0.0f;
      // sm = the softmax, q = sm + 1e-8 (the probs the reference's Categorical receives); the gradient goes through sm
      // itself, not q - 1e-8, which loses the digits of a softmax entry far below 1e-8
      float sm[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        sm[i] = (lane + 32 * i < C) ? q[i] / s : 0.0f;
        q[i] = (lane + 32 * i < C) ? sm[i] + PPB_UTIL_EPSILON : 0.0f;
        S += q[i];
      }
      S = ppb_warp_sum(S);
      const int iv = (int)v;
      if (iv < 0 || iv >= C) {
        lp = NAN;
      } else {
        float qv = 0.0f;
#pragma unroll
        for (int i = 0; i < 4; ++i) if (lane + 32 * i == iv) qv = q[i];
        qv = ppb_warp_sum(qv);
        float ph = qv / S;
        bool clamped = (ph < PPB_EPS32) || (ph > 1.0f - PPB_EPS32);
        lp = logf(ppb_clamp_prob(ph));
        if (!clamped && lp > -INFINITY) {
          float dot = 0.0f, g[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            int c = lane + 32 * i;
            g[i] = c < C ? ((c == iv) ? 1.0f / qv : 0.0f) - 1.0f / S : 0.0f;
            dot += c < C ? sm[i] * g[i] : 0.0f;
          }
          dot = ppb_warp_sum(dot);
          g0 = -(sm[0] * (g[0] - dot));
          g1 = (lane + 32 < C) ? -(sm[1] * (g[1] - dot)) : 0.f;
          g2 = (lane + 64 < C) ? -(sm[2] * (g[2] - dot)) : 0.f;
          g3 = (lane + 96 < C) ? -(sm[3] * (g[3] - dot)) : 0.f;
          if (lane >= C) g0 = 0.f;
        }
      }
    } else {
      const bool on = lane < K;
      const int fam = in.family;
      const float p0 = in.p0, p1 = in.p1;
      const float xm = on ? x[lane] : 0.f, xsd = on ? x[K + lane] : 0.f, xp = on ? x[2 * K + lane] : -INFINITY;
      float mx = ppb_warp_max(xp);
      float e = on ? expf(xp - mx) : 0.0f;
      float prob = e / ppb_warp_sum(e);
      float mean, sd, lo = 0.f, hi = 0.f;
      if (fam == PPB_FAMILY_NORMAL) { mean = p0 + xm * p1; sd = expf(xsd) * p1; }
      else if (fam == PPB_FAMILY_UNIFORM) {
        float range = p1 - p0;
        mean = p0 + heads::sigmoidf_(xm) * range;
        sd = range / 1000.0f + heads::sigmoidf_(xsd) * range * 10.0f;
        lo = p0; hi = p1;
      } else { mean = heads::sigmoidf_(xm) * 40.0f; sd = expf(xsd); lo = 0.f; hi = 40.f; }
      const bool trunc = fam != PPB_FAMILY_NORMAL;
      float S = ppb_warp_sum(on ? prob : 0.0f);
      float ph = prob / S;
      bool clamped = (ph < PPB_EPS32) || (ph > 1.0f - PPB_EPS32);
      float lw = logf(ppb_clamp_prob(ph));
      float lpk = trunc ? ppb_truncnormal_lp(v, mean, sd, lo, hi) : ppb_normal_lp(v, mean, sd);
      float t = on ? lw + lpk : -INFINITY;
      if (on && isnan(t)) t = NAN;
      float mxt = ppb_warp_max(t);
      // NaN anywhere poisons the row (reference: has_nan_or_inf on the log_prob)
      bool any_nan = __any_sync(0xffffffffu, on && isnan(t));
      if (any_nan) lp = NAN;
      else if (mxt == -INFINITY) lp = -INFINITY;
      else lp = mxt + logf(ppb_warp_sum(on ? expf(t - mxt) : 0.0f));
      if (lp > -INFINITY && lp < INFINITY) {
        float r = on ? expf(t - lp) : 0.0f;
        float sum_r_unc = ppb_warp_sum((on && !clamped) ? r : 0.0f);
        float direct = (on && !clamped) ? r / ph : 0.0f;
        float g_prob = (direct - sum_r_unc) / S;
        float dot = ppb_warp_sum(on ? prob * g_prob : 0.0f);
        // dmu = sd d lp_k / d mean and dls = sd d lp_k / d sd, then the transform's factor over sd: nothing overflows where
        // the exact gradient fits fp32 (z / sd and (z^2 - 1) / sd alone do from sd ~ 1e-13 on)
        float z = (v - mean) / sd, dmu, dls;
        if (!trunc) { dmu = z; dls = z * z - 1.0f; }
        else {
          float alpha = (lo - mean) / sd, beta = (hi - mean) / sd;
          float Z = ppb_std_normal_cdf(beta) - ppb_std_normal_cdf(alpha);
          float pa = heads::std_normal_pdf(alpha), pb = heads::std_normal_pdf(beta);
          dmu = z - (pa - pb) / Z;
          dls = z * z - 1.0f - (alpha * pa - beta * pb) / Z;
        }
        float dxm, dxs;
        if (fam == PPB_FAMILY_NORMAL) { dxm = (dmu * p1) / sd; dxs = dls; }
        else if (fam == PPB_FAMILY_UNIFORM) {
          float range = p1 - p0, sm = heads::sigmoidf_(xm), ss = heads::sigmoidf_(xsd);
          dxm = (dmu * (sm * (1.0f - sm) * range)) / sd;
          dxs = (dls * (ss * (1.0f - ss) * range * 10.0f)) / sd;
        } else { float sm = heads::sigmoidf_(xm); dxm = (dmu * (sm * (1.0f - sm) * 40.0f)) / sd; dxs = dls; }
        // a component with responsibility 0 contributes nothing: its derivatives may overflow (a tiny sd far from v) and
        // 0 * inf would put NaN into d_out with the status still 0 (DESIGN.md §8)
        dxm = r > 0.0f ? dxm * r : 0.0f; dxs = r > 0.0f ? dxs * r : 0.0f;
        if (on) { g0 = -dxm; g1 = -dxs; g2 = -(prob * (g_prob - dot)); }
      }
    }
    if (lp == -INFINITY) { lp = PPB_LOG_EPSILON; g0 = g1 = g2 = g3 = 0.f; }  // util.replace_negative_inf (:213)
    // a finite log q whose gradient does not fit fp32 (a component with sd ~ 1e-20 that explains v from 0.3 away:
    // d(-log q)/d out ~ 1e38 and beyond) fails the batch like a NaN log q, so that no inf reaches the optimiser (DESIGN.md §8)
    const bool g_bad = __any_sync(0xffffffffu, !(isfinite(g0) && isfinite(g1) && isfinite(g2) && isfinite(g3)));
    if (isnan(lp) || isinf(lp) || g_bad) { if (lane == 0) bad += 1; lp = 0.0f; g0 = g1 = g2 = g3 = 0.f; }
    if (lane == 0) local += -lp;
  }
  if (row_lp && lane == 0) row_lp[row] = lp;
  // scatter this lane's entries; everything else in the (padded) row is zero
  if (d_out) {
    const int ncols = (dimg.k_hi && img_cols > out_pad) ? img_cols : out_pad;
    auto put = [&](int j, float gv) {
      gv *= inv_batch;
      if (j < out_pad) d_out[(int64_t)row * out_pad + j] = gv;
      if (dimg.k_hi && j < img_cols) tcg::img_store(dimg.k_hi, dimg.k_lo, dimg.mn_hi, dimg.mn_lo, row, j, dimg.kb, gv);
    };
    if (valid) {
      if (is_cat) {
        if (lane < O) put(lane, g0);
        if (lane + 32 < O) put(lane + 32, g1);
        if (lane + 64 < O) put(lane + 64, g2);
        if (lane + 96 < O) put(lane + 96, g3);
      } else if (is_bern) {
        if (lane == 0) put(0, g0);
      } else if (lane < K) {
        put(lane, g0); put(K + lane, g1); put(2 * K + lane, g2);
      }
    }
    for (int j = (valid ? O : 0) + lane; j < ncols; j += 32) put(j, 0.0f);
  }
  }

__device__ __forceinline__ void nll_row(const NllArgs& A, const float* x, int row, int lane, float& local, int& bad) {
  nll_row(A, nll_row_in(A, row), x, row, lane, local, bad);
}

// sum of -log q and count of failed rows -> loss accumulators; the last block to finish publishes the totals
// (loss_acc[2] counts finished blocks; zeroed with the accumulators)
__device__ __forceinline__ void nll_finish(float local, int bad, int lane, float inv_batch, unsigned int n_blocks,
                                           float* __restrict__ loss_acc, float* __restrict__ loss_out,
                                           int* __restrict__ status_out) {
  if (lane == 0) {
    if (local != 0.0f) atomicAdd(loss_acc, local * inv_batch);
    if (bad) atomicAdd(reinterpret_cast<int*>(loss_acc + 1), bad);
  }
  __shared__ int s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    s_last = atomicAdd(reinterpret_cast<unsigned int*>(loss_acc + 2), 1u) == n_blocks - 1;
  }
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    __threadfence();
    if (loss_out) *loss_out = atomicAdd(loss_acc, 0.0f);
    if (status_out) *status_out = atomicAdd(reinterpret_cast<int*>(loss_acc + 1), 0);
  }
}

// Epilogue 3 of tcc::k_cluster (tc_cluster.cuh) for the h2 phase when it runs as a cluster: each output row goes through
// nll_row as soon as the cluster has reduced it, and the grid publishes the loss as k_head_nll does — the output layer and
// the NLL in one launch.  The row's other inputs (nll_row_in) are loaded before the mainloop, so that only the arithmetic
// of the row follows the reduction.  No row-major copy of the outputs is written: in a training step nothing else reads it.
struct NllRowEpi {
  NllArgs A;
  float* loss_acc; float* loss_out; int* status_out;
  struct State { float local; int bad; };
  using RowIn = NllRowIn;
  __device__ __forceinline__ RowIn load(int64_t row) const { return nll_row_in(A, (int)row); }
  __device__ __forceinline__ void row(State& s, const RowIn& in, const float* x, int64_t row, int lane) const {
    nll_row(A, in, x, (int)row, lane, s.local, s.bad);
  }
  __device__ __forceinline__ void finish(const State& s, int lane) const {
    nll_finish(s.local, s.bad, lane, A.inv_batch, gridDim.x, loss_acc, loss_out, status_out);
  }
};

__global__ void __launch_bounds__(256) k_head_nll(const float* __restrict__ out_raw, NllArgs A, int R,
                                                   float* __restrict__ loss_acc, float* __restrict__ loss_out,
                                                   int* __restrict__ status_out) {
  ppb_pdl_trigger();
  ppb_pdl_wait();
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  float local = 0.0f;
  int bad = 0;
  for (int row = warp; row < R; row += nwarps) nll_row(A, out_raw + (int64_t)row * A.out_pad, row, lane, local, bad);
  nll_finish(local, bad, lane, A.inv_batch, gridDim.x, loss_acc, loss_out, status_out);
}

// LSTM cell backward of one (row, unit) (torch.nn.LSTM gate order i, f, g, o): dht = dL/dh_t, dc_next = dL/dc_t carried back
// from step t + 1 (0 without a successor), cp = c_{t-1}.  dv = dL/d(gate pre-activations); returns dL/dc_t.
__device__ __forceinline__ float cell_bwd_unit(float ig, float fg, float gg, float og, float cn, float cp, float dht,
                                               float dc_next, float (&dv)[4]) {
  const float tc_ = ppb_cell_tanh(cn);
  const float dct = dc_next + dht * og * (1.0f - tc_ * tc_);
  dv[0] = dct * gg * ig * (1.0f - ig);
  dv[1] = dct * cp * fg * (1.0f - fg);
  dv[2] = dct * ig * (1.0f - gg * gg);
  dv[3] = dht * tc_ * og * (1.0f - og);
  return dct;
}

// tile-image stores of the four gate entries of unit j in image row `row`: with H % 32 == 0 the columns j + q H sit
// gate_stride = (H / 32) column blocks apart in the image as well
__device__ __forceinline__ void img_store_gates(const HImg& img, int64_t row, int j, int64_t gate_stride, const float (&v)[4]) {
  const int64_t ok = tc::packed_offset(row, j, img.kb), omn = tc::packed_offset_mn(row, j, img.kb);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    float hi, lo;
    tc::split_tf32(v[q], hi, lo);
    img.k_hi[ok + q * gate_stride] = hi;
    if (img.k_lo) img.k_lo[ok + q * gate_stride] = lo;
    if (img.mn_hi) {
      img.mn_hi[omn + q * gate_stride] = hi;
      if (img.mn_lo) img.mn_lo[omn + q * gate_stride] = lo;
    }
  }
}

// Epilogue 4 of tcc::k_cluster (tc_cluster.cuh) for the dh phase of a T = 1 step: the cell backward of (row, unit j) where the
// cluster has reduced dh[row, j], so that neither dh nor a k_cell_bwd launch sits on the chain.  At T = 1 no row has a
// successor (no dh_rec, no carried dc) and the trace's d_pobs is its one row's dgates; of d_pobs only the tile images are
// read (the W_ih[:, :E] gradient and d obs_emb GEMMs), of dgates the fp32 rows (k_dgates_reduce).  H % 32 == 0, B % 128 == 0.
struct CellBwdT1Epi {
  const float* gates; const float* c; const int* row_trace;
  float* dgates; HImg pimg; int H;
  __device__ __forceinline__ void cells(int64_t row, int j0, const float (&dh)[4]) const {
    const int tr = __ldg(row_trace + row);
    const int64_t gate_stride = (int64_t)(H >> 5) * tc::kTileFloats;
    float gv[4][4], cv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {   // loads of all four units first
      const int j = min(j0 + 32 * u, H - 1);   // columns >= H are loaded in range and not stored
#pragma unroll
      for (int q = 0; q < 4; ++q) gv[u][q] = __ldg(gates + row * 4 * H + q * H + j);
      cv[u] = __ldg(c + row * H + j);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = j0 + 32 * u;
      if (j >= H) continue;   // warp-uniform (H % 32 == 0)
      float dv[4] = {0.f, 0.f, 0.f, 0.f};
      if (tr >= 0) cell_bwd_unit(gv[u][0], gv[u][1], gv[u][2], gv[u][3], cv[u], 0.0f, dh[u], 0.0f, dv);
#pragma unroll
      for (int q = 0; q < 4; ++q) dgates[row * 4 * H + q * H + j] = dv[q];
      if (tr >= 0) img_store_gates(pimg, tr, j, gate_stride, dv);
    }
  }
};

// LSTM cell backward, one time step (reverse order).  dgates rows of this step are produced here;
// dh_rec = dgates[t+1] W_hh (prefix of this step's rows), dc carries d c_t across steps (dc == nullptr: not written, T = 1).
// 8 blocks of 256 threads per SM: the 1024 blocks of a 512-row, H = 512 step are ONE wave (at 40 registers it was 6 per SM,
// a second wave of 136 blocks, and the kernel went from 9.2 to 10.7 us)
// FINAL (the t = 0 launch, which ends every trace's sum): the per-trace gradient d_pobs is also written as tile images
// (pimg), so that no packing kernel sits between BPTT and the weight-gradient GEMMs.
template <bool FINAL>
__global__ void __launch_bounds__(256, FINAL ? 4 : 8) k_cell_bwd(const float* __restrict__ gates, const float* __restrict__ c,
                                                   const float* __restrict__ dh, const float* __restrict__ dh_rec,
                                                   float* __restrict__ dc, float* __restrict__ dgates,
                                                   float* __restrict__ d_pobs, const int* __restrict__ row_prev,
                                                   const int* __restrict__ row_next, const int* __restrict__ row_trace,
                                                   HImg gimg, int row0, int n_rows, int H, int t, HImg pimg) {
  ppb_pdl_trigger();
  ppb_pdl_wait();
  // Index arithmetic once per (row, unit): the four gate columns j, H + j, 2H + j, 3H + j sit H / 32 column blocks apart
  // (H % 32 == 0 on this path), so their image positions differ by a constant; the kernel used to spend most of its
  // instructions on four independent 64-bit offset computations per format.
  const int64_t total = (int64_t)n_rows * H;
  const int64_t gate_stride = (int64_t)(H >> 5) * tc::kTileFloats;
  const bool h32 = (H & 31) == 0;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(e / H), j = (int)(e - (int64_t)i * H);
    const int row = row0 + i;
    const int tr = __ldg(row_trace + row);
    const int64_t rH = (int64_t)row * H + j;       // position in [R, H] tensors
    float* dgr = dgates + (int64_t)row * 4 * H + j;
    float dv[4] = {0.f, 0.f, 0.f, 0.f};
    if (tr >= 0) {
      const int nx = __ldg(row_next + row);
      const float* g = gates + (int64_t)row * 4 * H + j;
      const float ig = g[0], fg = g[H], gg = g[2 * H], og = g[3 * H];
      const float cn = c[rH];
      const float cp = (t > 0) ? c[(int64_t)__ldg(row_prev + row) * H + j] : 0.0f;
      const bool has_next = nx >= 0;
      const float dht = dh[rH] + (has_next ? dh_rec[rH] : 0.0f);
      const float dct = cell_bwd_unit(ig, fg, gg, og, cn, cp, dht, has_next ? dc[(int64_t)nx * H + j] : 0.0f, dv);
      if (dc) dc[rH] = dct * fg;
      float* dp = d_pobs + (int64_t)tr * 4 * H + j;
      float tot[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        tot[q] = has_next ? dp[q * H] + dv[q] : dv[q];
        dp[q * H] = tot[q];
      }
      if (FINAL && pimg.k_hi) img_store_gates(pimg, tr, j, gate_stride, tot);   // H % 32 == 0 on this path
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) dgr[q * H] = dv[q];
    if (gimg.k_hi) {
      if (h32) {
        img_store_gates(gimg, row, j, gate_stride, dv);
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q)
          tcg::img_store(gimg.k_hi, gimg.k_lo, gimg.mn_hi, gimg.mn_lo, row, q * H + j, gimg.kb, dv[q]);
      }
    }
  }
}

// d_pstep[st, col] = sum over the rows of step st (contiguous range) of dgates[row, col]
__global__ void __launch_bounds__(256) k_step_colsum(const float* __restrict__ dgates, const int* __restrict__ step_row0,
                                                      const int* __restrict__ step_nrows, int H4,
                                                      float* __restrict__ d_pstep) {
  __shared__ float part[8][33];
  const int st = blockIdx.y;
  const int r0 = step_row0[st], n = step_nrows[st];
  const int lane = threadIdx.x & 31, slice = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + lane;
  float s = 0.0f;
  if (col < H4)
    for (int r = slice; r < n; r += 8) s += dgates[(int64_t)(r0 + r) * H4 + col];
  part[slice][lane] = s;
  __syncthreads();
  if (slice == 0 && col < H4) {
    float t = 0.0f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += part[k][lane];
    d_pstep[(int64_t)st * H4 + col] = t;
  }
}

// d smp_emb[row, j] = sum_col dgates[row, col] * w_smp_t[j][col], masked by relu; then the per-address sample-embedding layer
// gradients.  All rows of a (step, sub-batch) segment share their previous address, so a block owns a slab of ONE segment,
// accumulates the tiny [S x smp_in] weight and [S] bias gradients of that address in shared memory and issues one global
// atomic per entry per block (one global atomic per row took 0.38 ms at T = 50, B = 512: 200 k atomics on ~500 addresses).
__global__ void __launch_bounds__(128) k_smp_bwd_seg(const float* __restrict__ dgates, const float* __restrict__ w_smp_t,
                                                      const float* __restrict__ smp_emb, const float* __restrict__ values,
                                                      const int* __restrict__ step_prev, const int* __restrict__ step_row0,
                                                      const int* __restrict__ step_nrows, const int* __restrict__ row_prev,
                                                      const ppb_addr_desc* __restrict__ addrs, int H4, int S,
                                                      int rows_per_block, float* __restrict__ grad) {
  __shared__ float acc_b[8];
  __shared__ float acc_w[8][heads::CMAX];
  const int st = blockIdx.y;
  const int pa = step_prev[st];
  if (pa < 0) return;
  const int seg0 = step_row0[st], r0 = seg0 + blockIdx.x * rows_per_block;
  int r1 = r0 + rows_per_block;
  if (r1 > seg0 + step_nrows[st]) r1 = seg0 + step_nrows[st];
  if (r0 >= r1) return;
  const ppb_addr_desc a = addrs[pa];
  const bool is_cat = a.family == PPB_FAMILY_CATEGORICAL;
  const int width = is_cat ? a.smp_in : 1;
  for (int i = threadIdx.x; i < 8 * heads::CMAX; i += blockDim.x) (&acc_w[0][0])[i] = 0.0f;
  if (threadIdx.x < 8) acc_b[threadIdx.x] = 0.0f;
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int row = r0 + warp; row < r1; row += 4) {
    float s[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = 0.0f;
    for (int col = lane; col < H4; col += 32) {
      const float d = dgates[(int64_t)row * H4 + col];
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (j < S) s[j] = fmaf(d, __ldg(w_smp_t + (int64_t)j * H4 + col), s[j]);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (j < S) s[j] = ppb_warp_sum(s[j]);
    if (lane == 0) {
      const float x = values[row_prev[row]];
      const int cidx = (int)x;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (j < S && smp_emb[(int64_t)row * S + j] > 0.0f && s[j] != 0.0f) {
          atomicAdd(&acc_b[j], s[j]);
          if (is_cat) { if (cidx >= 0 && cidx < a.smp_in) atomicAdd(&acc_w[j][cidx], s[j]); }
          else atomicAdd(&acc_w[j][0], s[j] * x);
        }
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < S * (width + 1); i += blockDim.x) {
    const int j = i / (width + 1), c = i % (width + 1);
    if (c == width) { if (acc_b[j] != 0.0f) atomicAdd(grad + a.smp_b_off + j, acc_b[j]); }
    else if (acc_w[j][c] != 0.0f) atomicAdd(grad + a.smp_w_off + (int64_t)j * a.smp_in + c, acc_w[j][c]);
  }
}

// ONE pass over dgates for everything that reduces it over rows (T = 50, B = 512: dgates is 210 MB; the three kernels it
// replaces — k_step_colsum, k_smp_bwd_seg, k_wsmp_grad — each streamed it again):
//   d_pstep[st, col]        += sum over the rows of segment st of dgates[row, col]                 (atomics; zeroed before)
//   dW_ih[col, E + j]       += sum_rows dgates[row, col] * smp_emb[row, j]
//   d smp_emb[row, j]        = sum_col dgates[row, col] * W_ih[col, E + j]  -> ReLU mask -> the previous address's
//                              sample-embedding layer gradients (shared-memory accumulation per block, see k_smp_bwd_seg)
// A block owns a slab of rows of one (step, sub-batch) segment; a thread owns NC = 4H / 256 columns.
constexpr int kRedSlab = 64;
template <int NC>
__global__ void __launch_bounds__(256) k_dgates_reduce(const float* __restrict__ dgates, const float* __restrict__ w_smp_t,
                                                        const float* __restrict__ smp_emb, const float* __restrict__ values,
                                                        const int* __restrict__ step_prev, const int* __restrict__ step_row0,
                                                        const int* __restrict__ step_nrows, const int* __restrict__ row_prev,
                                                        const ppb_addr_desc* __restrict__ addrs, int H4, int S, int I, int E,
                                                        float* __restrict__ d_pstep, float* __restrict__ grad,
                                                        int64_t w_ih_off, int slab) {
  __shared__ float s_emb[kRedSlab][8];
  __shared__ float s_dot[kRedSlab][8];
  __shared__ float acc_b[8];
  __shared__ float acc_w[8][heads::CMAX];
  const int st = blockIdx.y;
  const int seg0 = step_row0[st], r0 = seg0 + blockIdx.x * slab;   // slab <= kRedSlab rows per block
  int r1 = r0 + slab;
  if (r1 > seg0 + step_nrows[st]) r1 = seg0 + step_nrows[st];
  if (r0 >= r1) return;
  const int pa = step_prev[st];
  const bool smp = pa >= 0;
  const int tid = threadIdx.x, lane = tid & 31;
  if (smp) {
    for (int i = tid; i < kRedSlab * 8; i += 256) {
      const int rr = i >> 3, j = i & 7;
      s_emb[rr][j] = (r0 + rr < r1 && j < S) ? smp_emb[(int64_t)(r0 + rr) * S + j] : 0.0f;
      s_dot[rr][j] = 0.0f;
    }
    for (int i = tid; i < 8 * heads::CMAX; i += 256) (&acc_w[0][0])[i] = 0.0f;
    if (tid < 8) acc_b[tid] = 0.0f;
  }
  __syncthreads();
  float colsum[NC], w[NC][4], wg[NC][4];
#pragma unroll
  for (int i = 0; i < NC; ++i) {
    colsum[i] = 0.0f;
    const int col = tid + 256 * i;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      w[i][j] = (smp && j < S && col < H4) ? __ldg(w_smp_t + (int64_t)j * H4 + col) : 0.0f;
      wg[i][j] = 0.0f;
    }
  }
  float dn[NC];   // next row's values: two rows of loads in flight (the row loop is latency-bound otherwise)
#pragma unroll
  for (int i = 0; i < NC; ++i) {
    const int col = tid + 256 * i;
    dn[i] = col < H4 ? __ldg(dgates + (int64_t)r0 * H4 + col) : 0.0f;
  }
  for (int r = r0; r < r1; ++r) {
    const int rr = r - r0;
    float d[NC];
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const int col = tid + 256 * i;
      d[i] = dn[i];
      dn[i] = (r + 1 < r1 && col < H4) ? __ldg(dgates + (int64_t)(r + 1) * H4 + col) : 0.0f;
      colsum[i] += d[i];
    }
    if (smp) {
      float p[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float e = s_emb[rr][j];
#pragma unroll
        for (int i = 0; i < NC; ++i) {
          wg[i][j] = fmaf(d[i], e, wg[i][j]);
          p[j] = fmaf(d[i], w[i][j], p[j]);
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float t = ppb_warp_sum(p[j]);
        if (lane == 0 && j < S) atomicAdd(&s_dot[rr][j], t);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NC; ++i) {
    const int col = tid + 256 * i;
    if (col < H4) {
      if (colsum[i] != 0.0f) atomicAdd(d_pstep + (int64_t)st * H4 + col, colsum[i]);
      if (smp) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (j < S && wg[i][j] != 0.0f) atomicAdd(grad + w_ih_off + (int64_t)col * I + E + j, wg[i][j]);
      }
    }
  }
  if (!smp) return;
  __syncthreads();
  const ppb_addr_desc a = addrs[pa];
  const bool is_cat = a.family == PPB_FAMILY_CATEGORICAL;
  if (tid < r1 - r0) {
    const float x = values[row_prev[r0 + tid]];
    const int cidx = (int)x;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float sj = s_dot[tid][j];
      if (j < S && s_emb[tid][j] > 0.0f && sj != 0.0f) {
        atomicAdd(&acc_b[j], sj);
        if (is_cat) { if (cidx >= 0 && cidx < a.smp_in) atomicAdd(&acc_w[j][cidx], sj); }
        else atomicAdd(&acc_w[j][0], sj * x);
      }
    }
  }
  __syncthreads();
  const int width = is_cat ? a.smp_in : 1;
  for (int i = tid; i < S * (width + 1); i += 256) {
    const int j = i / (width + 1), c = i % (width + 1);
    if (c == width) { if (acc_b[j] != 0.0f) atomicAdd(grad + a.smp_b_off + j, acc_b[j]); }
    else if (acc_w[j][c] != 0.0f) atomicAdd(grad + a.smp_w_off + (int64_t)j * a.smp_in + c, acc_w[j][c]);
  }
}

// dW_ih[:, E + j] += sum_rows dgates[row, col] * smp_emb[row, j]
__global__ void k_wsmp_grad(const float* __restrict__ dgates, const float* __restrict__ smp_emb, int R, int H4, int S,
                            int I, int E, float* __restrict__ dw_ih, int rows_per_block) {
  int r0 = blockIdx.y * rows_per_block;
  int r1 = r0 + rows_per_block < R ? r0 + rows_per_block : R;
  for (int col = blockIdx.x * blockDim.x + threadIdx.x; col < H4; col += gridDim.x * blockDim.x) {
    float acc[8];
    for (int j = 0; j < S; ++j) acc[j] = 0.0f;
    for (int r = r0; r < r1; ++r) {
      float d = dgates[(int64_t)r * H4 + col];
      for (int j = 0; j < S; ++j) acc[j] = fmaf(d, smp_emb[(int64_t)r * S + j], acc[j]);
    }
    for (int j = 0; j < S; ++j)
      if (acc[j] != 0.0f) atomicAdd(dw_ih + (int64_t)col * I + E + j, acc[j]);
  }
}

// p_step[st, col] = b_ih[col] + b_hh[col] + sum_j emb_cat[st, j] W_ih[col, E + S + j]   (one warp per output)
__global__ void __launch_bounds__(256) k_pstep_fwd(const float* __restrict__ emb_cat, const float* __restrict__ w_ih,
                                                    const float* __restrict__ b_ih, const float* __restrict__ b_hh,
                                                    int NS, int H4, int I, int off, int C2, float* __restrict__ p_step) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  int nw = (gridDim.x * blockDim.x) >> 5;
  for (int o = warp; o < NS * H4; o += nw) {
    int st = o / H4, col = o % H4;
    float s = 0.0f;
    for (int j = lane; j < C2; j += 32) s = fmaf(emb_cat[(int64_t)st * C2 + j], w_ih[(int64_t)col * I + off + j], s);
    s = ppb_warp_sum(s);
    if (lane == 0) p_step[o] = s + b_ih[col] + b_hh[col];
  }
}
// Every gradient that follows from d_pstep, in ONE launch (T = 50: NS = 50 step segments):
//   blocks [0, nx)  : d emb_cat[st, j] = sum_col d_pstep[st, col] W_ih[col, off + j], lanes over j, warps and blockIdx over
//                     column slices; each block's partial sum goes straight into the type / address embedding it came from
//   blocks [nx, ...): dW_ih[col, off + j] += sum_st d_pstep[st, col] emb_cat[st, j] (one thread per entry), then
//                     db_ih[col] = db_hh[col] += sum_st d_pstep[st, col]
__global__ void __launch_bounds__(256) k_pstep_bwd(const float* __restrict__ d_pstep, const float* __restrict__ w_ih,
                                                    const float* __restrict__ emb_cat, const ppb_addr_desc* __restrict__ addrs,
                                                    const int64_t* __restrict__ type_off, const int* __restrict__ step_addr,
                                                    const int* __restrict__ step_prev, int NS, int H4, int I, int off, int td,
                                                    int ad, int zsplit, int nx, float* __restrict__ grad, int64_t w_ih_off,
                                                    int64_t b_ih_off, int64_t b_hh_off) {
  const int C2 = 2 * (td + ad);
  if ((int)blockIdx.x < nx) {
    __shared__ float part[8][33];
    const int jbs = (C2 + 31) / 32;
    const int jb = blockIdx.x % jbs, st = (blockIdx.x / jbs) % NS, z = blockIdx.x / (jbs * NS);
    const int lane = threadIdx.x & 31, slice = threadIdx.x >> 5;
    const int j = jb * 32 + lane;
    float s = 0.0f;
    if (j < C2)
      for (int col = z * 8 + slice; col < H4; col += 8 * zsplit)
        s = fmaf(d_pstep[(int64_t)st * H4 + col], __ldg(w_ih + (int64_t)col * I + off + j), s);
    part[slice][lane] = s;
    __syncthreads();
    if (slice == 0 && j < C2) {
      float t = 0.0f;
#pragma unroll
      for (int k = 0; k < 8; ++k) t += part[k][lane];
      const int64_t o = step_embed_off(type_off, td, ad, j, [&](bool is_prev, const ppb_addr_desc*& a) {
        const int which = is_prev ? step_prev[st] : step_addr[st];
        a = addrs + which;
        return which >= 0;
      });
      if (o >= 0 && t != 0.0f) atomicAdd(grad + o, t);
    }
    return;
  }
  const int64_t nwe = (int64_t)H4 * C2;
  for (int64_t e = (int64_t)(blockIdx.x - nx) * blockDim.x + threadIdx.x; e < nwe + H4;
       e += (int64_t)(gridDim.x - nx) * blockDim.x) {
    if (e < nwe) {
      const int col = (int)(e / C2), j = (int)(e % C2);
      float s = 0.0f;
      for (int st = 0; st < NS; ++st) s = fmaf(d_pstep[(int64_t)st * H4 + col], emb_cat[(int64_t)st * C2 + j], s);
      grad[w_ih_off + (int64_t)col * I + off + j] += s;
    } else {
      const int col = (int)(e - nwe);
      float s = 0.0f;
      for (int st = 0; st < NS; ++st) s += d_pstep[(int64_t)st * H4 + col];
      grad[b_ih_off + col] += s;
      grad[b_hh_off + col] += s;
    }
  }
}

// db2[a] += colsum(d_out rows of a), db1[a] += colsum(d_hid rows of a) for every address group in ONE launch:
// blockIdx.y = group, blockIdx.x = 32-column block (first the hidden columns, then the output columns)
__global__ void __launch_bounds__(256) k_head_bias_grad(const float* __restrict__ d_out, int out_pad,
                                                         const float* __restrict__ d_hid, int dh_pad,
                                                         const int* __restrict__ head_rows, const int* __restrict__ group_start,
                                                         const int* __restrict__ group_addr,
                                                         const ppb_addr_desc* __restrict__ addrs, float* __restrict__ grad) {
  __shared__ float part[8][33];
  const int g = blockIdx.y;
  const ppb_addr_desc a = addrs[group_addr[g]];
  const int hid_blocks = (dh_pad + 31) / 32;
  const bool is_hid = (int)blockIdx.x < hid_blocks;
  const int lane = threadIdx.x & 31, slice = threadIdx.x >> 5;
  const int n = (is_hid ? blockIdx.x : blockIdx.x - hid_blocks) * 32 + lane;
  const int width = is_hid ? a.head_hidden : a.head_out;
  const float* src = is_hid ? d_hid : d_out;
  const int ld = is_hid ? dh_pad : out_pad;
  const int s0 = group_start[g], cnt = group_start[g + 1] - s0;
  float s = 0.0f;
  if (n < width)   // blockIdx.z splits the rows of the group
    for (int m = blockIdx.z * 8 + slice; m < cnt; m += 8 * gridDim.z) s += src[(int64_t)head_rows[s0 + m] * ld + n];
  part[slice][lane] = s;
  __syncthreads();
  if (slice == 0 && n < width) {
    float t = 0.0f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += part[k][lane];
    if (t != 0.0f) atomicAdd(grad + (is_hid ? a.b1_off : a.b2_off) + n, t);
  }
}
// bias gradient of a Linear: db[n] += sum_m dY[gm(m), n].  Block = 32 columns x 8 row-slices; rows are
// strided over the slices and blockIdx.y, partial sums meet in shared memory / one atomic per block column.
__global__ void __launch_bounds__(256) k_colsum_gather(const float* __restrict__ dY, int64_t ld,
                                                        const int* __restrict__ m_gather, int M, int N,
                                                        float* __restrict__ db) {
  __shared__ float part[8][33];
  const int lane = threadIdx.x & 31, slice = threadIdx.x >> 5;
  const int n = blockIdx.x * 32 + lane;
  float s = 0.0f;
  if (n < N)
    for (int m = blockIdx.y * 8 + slice; m < M; m += 8 * gridDim.y) {
      int64_t pm = m_gather ? m_gather[m] : m;
      s += dY[pm * ld + n];
    }
  part[slice][lane] = s;
  __syncthreads();
  if (slice == 0 && n < N) {
    float t = 0.0f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += part[k][lane];
    if (t != 0.0f) atomicAdd(db + n, t);
  }
}
__global__ void k_scale(float* __restrict__ x, int64_t n, float a) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) x[i] *= a;
}

// ReLU backward at the top of a chain: d[i] = y[i] > 0 ? d[i] : 0
__global__ void k_mask_nonpos(float* __restrict__ d, const float* __restrict__ y, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (!(y[i] > 0.0f)) d[i] = 0.0f;
}

inline int ew_grid(int64_t n, int threads = 256) { return ppb_grid_for(n, threads, 1); }

Dims dims_of(const ppb_batch* b) {
  Dims d; d.B = b->n_traces; d.R = b->n_rows; d.T = b->t_max; d.NS = b->n_steps; d.G = b->n_groups;
  return d;
}

int check_batch(const ppb_net* net, const ppb_batch* b) {
  PPB_CHECK_ARG(net && b, "null net or batch");
  PPB_CHECK_ARG(b->n_traces > 0 && b->n_rows > 0 && b->t_max > 0 && b->n_steps > 0 && b->n_groups > 0, "empty batch");
  PPB_CHECK_ARG(b->row_off_host && b->group_addr_host && b->group_start_host, "missing host arrays");
  PPB_CHECK_ARG(b->row_off_host[0] == 0 && b->row_off_host[b->t_max] == b->n_rows, "row_off inconsistent");
  for (int g = 0; g < b->n_groups; ++g)
    PPB_CHECK_ARG(b->group_addr_host[g] >= 0 && b->group_addr_host[g] < (int)net->addrs.size(), "address id out of range");
  return PPB_OK;
}

// ---- proposal heads on the fp32 path, shared by the LSTM and the feed-forward networks ------------------------------------
// The heads read w.h [R, kx]: the LSTM output, or the observation embedding of each row's trace.
// Forward phases: hid = relu(h W1^T + b1), out_raw = hid W2^T + b2 (one problem per address group)
void simt_head_fwd(Builder& bl, const ppb_net* net, const float* arena, const ppb_batch* b, const Ws& w, int kx, int& ph_h1,
                   int& ph_h2) {
  const int G = b->n_groups;
  ph_h1 = (int)bl.phases.size();
  bl.begin();
  for (int g = 0; g < G; ++g) {
    const ppb_addr_desc& a = net->addrs[b->group_addr_host[g]];
    int s0 = b->group_start_host[g], cnt = b->group_start_host[g + 1] - s0;
    Problem p = linear_fwd(w.h, kx, arena + a.w1_off, kx, arena + a.b1_off, w.hid, net->dh_pad, cnt, a.head_hidden, kx, gemm::kRelu);
    p.m_gather = b->head_rows + s0;
    bl.add(p);
  }
  ph_h2 = (int)bl.phases.size();
  bl.begin();
  for (int g = 0; g < G; ++g) {
    const ppb_addr_desc& a = net->addrs[b->group_addr_host[g]];
    int s0 = b->group_start_host[g], cnt = b->group_start_host[g + 1] - s0;
    Problem p = linear_fwd(w.hid, net->dh_pad, arena + a.w2_off, a.head_hidden, arena + a.b2_off, w.out_raw, net->out_pad, cnt, a.head_out, a.head_hidden, 0);
    p.m_gather = b->head_rows + s0;
    bl.add(p);
  }
}

// Runs the two head phases (uploaded to w.problems) and the NLL
int simt_head_nll(const ppb_net* net, const ppb_batch* b, const Ws& w, const Builder& bl, int ph_h1, int ph_h2, float* loss_out,
                  int32_t* status_out, float* row_lp_out, int want_grad, cudaStream_t st) {
  int rc = run_phase(bl.phases[ph_h1], w.problems, st); if (rc) return rc;
  rc = run_phase(bl.phases[ph_h2], w.problems, st); if (rc) return rc;
  NllArgs na;
  na.addrs = net->d_addrs; na.row_step = b->row_step; na.step_addr = b->step_addr;
  na.values = b->values; na.prior0 = b->prior0; na.prior1 = b->prior1; na.row_trace = b->row_trace;
  na.K = net->desc.mixture_k; na.inv_batch = 1.0f / (float)b->n_traces;
  na.row_lp = row_lp_out ? row_lp_out : w.row_lp; na.d_out = want_grad ? w.d_out : nullptr; na.out_pad = net->out_pad;
  na.dimg = HImg();
  k_head_nll<<<ew_grid((int64_t)b->n_rows * 32, 256), 256, 0, st>>>(w.out_raw, na, b->n_rows, w.loss_acc, loss_out, status_out);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

// Backward phases: d_hid = (d_out W2) * relu'(hid) ; then dW2 += d_out^T hid ; dW1 += d_hid^T h ; dh = d_hid W1
void simt_head_bwd(Builder& bl, const ppb_net* net, const float* arena, float* grad, const ppb_batch* b, const Ws& w, int kx) {
  const int G = b->n_groups;
  bl.begin();
  for (int g = 0; g < G; ++g) {
    const ppb_addr_desc& a = net->addrs[b->group_addr_host[g]];
    int s0 = b->group_start_host[g], cnt = b->group_start_host[g + 1] - s0;
    Problem p = linear_dx(w.d_out, net->out_pad, arena + a.w2_off, a.head_hidden, w.d_hid, net->dh_pad, cnt, a.head_out, a.head_hidden, gemm::kMaskAux);
    p.aux = w.hid; p.ld_aux = net->dh_pad; p.m_gather = b->head_rows + s0;
    bl.add(p);
  }
  bl.begin();
  for (int g = 0; g < G; ++g) {
    const ppb_addr_desc& a = net->addrs[b->group_addr_host[g]];
    int s0 = b->group_start_host[g], cnt = b->group_start_host[g + 1] - s0;
    Problem p2 = linear_dw(w.d_out, net->out_pad, w.hid, net->dh_pad, grad + a.w2_off, a.head_hidden, cnt, a.head_out, a.head_hidden);
    p2.ka_gather = b->head_rows + s0; p2.kb_gather = b->head_rows + s0;
    bl.add(p2);
    Problem p1 = linear_dw(w.d_hid, net->dh_pad, w.h, kx, grad + a.w1_off, kx, cnt, a.head_hidden, kx);
    p1.ka_gather = b->head_rows + s0; p1.kb_gather = b->head_rows + s0;
    bl.add(p1);
    Problem px = linear_dx(w.d_hid, net->dh_pad, arena + a.w1_off, kx, w.dh, kx, cnt, a.head_hidden, kx, 0);
    px.m_gather = b->head_rows + s0;
    bl.add(px);
  }
}

// ---- CUDA-core side jobs of the training step, shared by every precision -------------------------------------------------
// db2[a] += colsum(d_out rows of a), db1[a] += colsum(d_hid rows of a), every address group in one launch
int launch_head_bias_grad(const ppb_net* net, const ppb_batch* b, const Ws& w, float* grad, cudaStream_t st) {
  // a row split that brings the grid to about one block per SM (T = 1: 10 column blocks, one address group) and leaves
  // each warp at least eight rows
  const int G = b->n_groups;
  const int cb = (net->dh_pad + 31) / 32 + (net->out_pad + 31) / 32;
  int max_rows = 0;
  for (int g = 0; g < G; ++g) max_rows = b->group_start_host[g + 1] - b->group_start_host[g] > max_rows ? b->group_start_host[g + 1] - b->group_start_host[g] : max_rows;
  int zs = PPB_NUM_SMS / (cb * G);
  const int zmax = (max_rows + 63) / 64;
  zs = zs > zmax ? zmax : zs;
  zs = zs < 1 ? 1 : zs;
  k_head_bias_grad<<<dim3(cb, G, zs), 256, 0, st>>>(w.d_out, net->out_pad, w.d_hid, net->dh_pad, b->head_rows, b->group_start,
                                                     b->group_addr, net->d_addrs, grad);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

// The LSTM inputs that do not depend on the observation: step embeddings -> P_step (both biases folded in), and at T > 1 the
// transposed sample-embedding columns of W_ih and the previous-sample embeddings (they only enter at t >= 1)
int launch_step_inputs_fwd(const ppb_net* net, const float* arena, const ppb_batch* b, const Ws& w, cudaStream_t st) {
  const ppb_net_desc& D = net->desc;
  const Dims d = dims_of(b);
  const int H4 = 4 * D.lstm_dim, E = D.obs_dim, S = D.sample_dim, I = net->I;
  const int C2 = 2 * (D.type_dim + D.addr_dim);
  k_step_embed<<<ew_grid((int64_t)d.NS * C2), 256, 0, st>>>(arena, net->d_addrs, net->d_type_off, b->step_addr,
                                                            b->step_prev_addr, d.NS, D.type_dim, D.addr_dim, w.emb_cat);
  PPB_LAUNCH_CHECK();
  k_pstep_fwd<<<ew_grid((int64_t)d.NS * H4 * 32), 256, 0, st>>>(w.emb_cat, arena + D.w_ih_off, arena + D.b_ih_off,
                                                                arena + D.b_hh_off, d.NS, H4, I, E + S, C2, w.p_step);
  PPB_LAUNCH_CHECK();
  if (d.T > 1) {
    k_wsmp_transpose<<<ew_grid(S * H4), 256, 0, st>>>(arena + D.w_ih_off, I, E, S, H4, w.w_smp_t);
    PPB_LAUNCH_CHECK();
    k_smp_embed<<<ew_grid((int64_t)d.R * S), 256, 0, st>>>(arena, net->d_addrs, b->row_step, b->step_prev_addr,
                                                           b->row_prev, b->values, d.R, S, w.smp_emb);
    PPB_LAUNCH_CHECK();
  }
  return PPB_OK;
}

// Every gradient that reduces dgates over the rows of a step, and every one that follows from d_pstep: d_pstep (an atomic
// target, zeroed before the call), dW_ih[:, E:], db_ih, db_hh, the type / address embeddings and the sample-embedding layers
int launch_step_inputs_bwd(const ppb_net* net, const float* arena, float* grad, const ppb_batch* b, const Ws& w,
                           const float* dgates, cudaStream_t st) {
  const ppb_net_desc& D = net->desc;
  const Dims d = dims_of(b);
  const int H4 = 4 * D.lstm_dim, E = D.obs_dim, S = D.sample_dim, I = net->I;
  const int C2 = 2 * (D.type_dim + D.addr_dim);
  // one pass over dgates: step column sums + sample-embedding gradients (S <= 4, 4H <= 2048); otherwise separate kernels
  const bool one_pass = S <= 4 && H4 <= 2048;
  int max_rows = 0;
  for (int s = 0; s < d.NS; ++s) max_rows = b->step_nrows_host[s] > max_rows ? b->step_nrows_host[s] : max_rows;
  if (one_pass) {
    // rows per block: enough blocks to fill the SMs twice (a T = 1 minibatch of 256 rows used to be FOUR blocks walking
    // 64 rows each: 44 us on the side branch that then bounded the step), at most kRedSlab
    int slab = (d.R + 2 * PPB_NUM_SMS - 1) / (2 * PPB_NUM_SMS);
    slab = slab < 4 ? 4 : (slab > kRedSlab ? kRedSlab : slab);
    const dim3 g((max_rows + slab - 1) / slab, d.NS);
    const float* wt = d.T > 1 ? w.w_smp_t : w.p_step;   // T = 1: no row has a previous site, the pointers are never read
    if (H4 <= 1024)
      k_dgates_reduce<4><<<g, 256, 0, st>>>(dgates, wt, w.smp_emb, b->values, b->step_prev_addr, b->step_row0, b->step_nrows,
                                            b->row_prev, net->d_addrs, H4, S, I, E, w.d_pstep, grad, D.w_ih_off, slab);
    else
      k_dgates_reduce<8><<<g, 256, 0, st>>>(dgates, wt, w.smp_emb, b->values, b->step_prev_addr, b->step_row0, b->step_nrows,
                                            b->row_prev, net->d_addrs, H4, S, I, E, w.d_pstep, grad, D.w_ih_off, slab);
    PPB_LAUNCH_CHECK();
  } else {
    dim3 g((H4 + 31) / 32, d.NS);
    k_step_colsum<<<g, 256, 0, st>>>(dgates, b->step_row0, b->step_nrows, H4, w.d_pstep);
    PPB_LAUNCH_CHECK();
  }
  {
    // about half an SM's worth of blocks split the d emb_cat columns (T = 1: one step segment, 5 column blocks); the weight
    // and bias entries get one thread each
    const int jbs = (C2 + 31) / 32;
    int zsplit = PPB_NUM_SMS / 2 / (jbs * d.NS);
    zsplit = zsplit < 1 ? 1 : (zsplit > 16 ? 16 : zsplit);
    const int nx = jbs * d.NS * zsplit;
    const int nw = (int)(((int64_t)H4 * C2 + H4 + 255) / 256);
    k_pstep_bwd<<<nx + nw, 256, 0, st>>>(w.d_pstep, arena + D.w_ih_off, w.emb_cat, net->d_addrs, net->d_type_off, b->step_addr,
                                         b->step_prev_addr, d.NS, H4, I, E + S, D.type_dim, D.addr_dim, zsplit, nx, grad,
                                         D.w_ih_off, D.b_ih_off, D.b_hh_off);
    PPB_LAUNCH_CHECK();
  }
  if (d.T > 1 && !one_pass) {
    const int slab = 64;
    k_smp_bwd_seg<<<dim3((max_rows + slab - 1) / slab, d.NS), 128, 0, st>>>(dgates, w.w_smp_t, w.smp_emb, b->values,
                                                                           b->step_prev_addr, b->step_row0, b->step_nrows,
                                                                           b->row_prev, net->d_addrs, H4, S, slab, grad);
    PPB_LAUNCH_CHECK();
    int rpb = 1024;
    dim3 g((H4 + 255) / 256, (d.R + rpb - 1) / rpb);
    k_wsmp_grad<<<g, 256, 0, st>>>(dgates, w.smp_emb, d.R, H4, S, I, E, grad + D.w_ih_off, rpb);
    PPB_LAUNCH_CHECK();
  }
  return PPB_OK;
}

}  // namespace

#include "net_tc.inc"
#include "net_ff.inc"

namespace {

// ---- LSTM network, fp32 SIMT path (precision 2) ------------------------------------------------------------------------
int simt_loss_forward(ppb_net* net, const float* arena, const ppb_batch* b, void* workspace, float* loss_out,
                      int32_t* status_out, float* row_lp_out, int want_grad, cudaStream_t st) {
  PPB_CHECK_ARG(b->row_align == 1, "the SIMT path needs a batch encoded with row_align = 1");
  const ppb_net_desc& D = net->desc;
  Dims d = dims_of(b);
  Ws w = carve(net, d, workspace);
  const int H = D.lstm_dim, H4 = 4 * H, E = D.obs_dim, S = D.sample_dim, I = net->I;

  // ---- problem lists for all forward GEMM phases -------------------------------------------------
  Builder bl;
  obs_fp32_plan_fwd(bl, D, arena, b->obs, d.B, w, w.obs_emb);
  const int ph_p = (int)bl.phases.size();
  bl.begin();
  bl.add(linear_fwd(w.obs_emb, E, arena + D.w_ih_off, I, nullptr, w.p_obs, H4, d.B, H4, E, 0));
  // recurrent GEMMs: gates[rows of t] = h[rows of t-1 (prefix)] W_hh^T
  const int ph_rec0 = (int)bl.phases.size();
  for (int t = 1; t < d.T; ++t) {
    bl.begin();
    int r0 = b->row_off_host[t], n = b->row_off_host[t + 1] - r0, rp = b->row_off_host[t - 1];
    bl.add(linear_fwd(w.h + (int64_t)rp * H, H, arena + D.w_hh_off, H, nullptr, w.gates + (int64_t)r0 * H4, H4, n, H4, H, 0));
  }
  int ph_h1, ph_h2;
  simt_head_fwd(bl, net, arena, b, w, H, ph_h1, ph_h2);
  int rc = upload_and_get(net, bl, w.problems, w.max_problems / 2, st, kSlotSimtFwd);
  if (rc) return rc;

  // ---- launches -----------------------------------------------------------------------------------
  PPB_CUDA(cudaMemsetAsync(w.loss_acc, 0, 256, st));
  for (int l = 0; l < ph_p; ++l) { rc = run_phase(bl.phases[l], w.problems, st); if (rc) return rc; }
  rc = launch_step_inputs_fwd(net, arena, b, w, st); if (rc) return rc;
  rc = run_phase(bl.phases[ph_p], w.problems, st, profile(bl, ph_p)); if (rc) return rc;
  for (int t = 0; t < d.T; ++t) {
    int r0 = b->row_off_host[t], n = b->row_off_host[t + 1] - r0;
    if (t > 0) { rc = run_phase(bl.phases[ph_rec0 + t - 1], w.problems, st, profile(bl, ph_rec0 + t - 1)); if (rc) return rc; }
    k_cell_fwd<<<ew_grid((int64_t)n * H), 256, 0, st>>>(w.gates, w.p_obs, w.p_step, w.w_smp_t, w.smp_emb, b->row_step,
                                                       b->row_prev, b->row_trace, w.c, w.h, HImg(), r0, n, H, S, t);
    PPB_LAUNCH_CHECK();
  }
  return simt_head_nll(net, b, w, bl, ph_h1, ph_h2, loss_out, status_out, row_lp_out, want_grad, st);
}

int simt_loss_backward(ppb_net* net, const float* arena, float* grad, const ppb_batch* b, void* workspace, float grad_scale,
                       cudaStream_t st) {
  PPB_CHECK_ARG(b->step_nrows_host, "missing per-step host arrays");
  const ppb_net_desc& D = net->desc;
  Dims d = dims_of(b);
  Ws w = carve(net, d, workspace);
  float* dgates = dgates_ptr(w, workspace);
  const int H = D.lstm_dim, H4 = 4 * H, E = D.obs_dim, I = net->I;

  // d_pstep: atomic target of k_dgates_reduce
  PPB_CUDA(cudaMemsetAsync(w.d_pstep, 0, (size_t)d.NS * H4 * sizeof(float), st));
  if (grad_scale != 1.0f) {
    k_scale<<<ew_grid((int64_t)d.R * net->out_pad), 256, 0, st>>>(w.d_out, (int64_t)d.R * net->out_pad, grad_scale);
    PPB_LAUNCH_CHECK();
  }

  Builder bl;
  const int ph_dhid = 0, ph_hw = 1;
  simt_head_bwd(bl, net, arena, grad, b, w, H);
  // BPTT recurrent: dh_rec[prefix rows of t-1] = dgates[rows of t] W_hh
  const int ph_rec0 = 2;
  for (int t = d.T - 1; t >= 1; --t) {
    bl.begin();
    int r0 = b->row_off_host[t], n = b->row_off_host[t + 1] - r0;
    bl.add(linear_dx(dgates + (int64_t)r0 * H4, H4, arena + D.w_hh_off, H, w.dh_rec + (int64_t)b->row_off_host[t - 1] * H, H, n, H4, H, 0));
  }
  const int ph_lstm_w = (int)bl.phases.size();
  bl.begin();
  {
    // dW_hh += sum_{rows t>=1} dgates[row]^T h[row_prev[row]]
    int r1 = b->row_off_host[1 < d.T ? 1 : d.T];
    int n1 = d.R - r1;
    if (n1 > 0) {
      Problem p = linear_dw(dgates + (int64_t)r1 * H4, H4, w.h, H, grad + D.w_hh_off, H, n1, H4, H);
      p.kb_gather = b->row_prev + r1;  // h row of the previous step
      bl.add(p);
    }
    // dW_ih[:, :E] += d_pobs^T obs_emb ; d obs_emb = d_pobs W_ih[:, :E]
    bl.add(linear_dw(w.d_pobs, H4, w.obs_emb, E, grad + D.w_ih_off, I, d.B, H4, E));
    bl.add(linear_dx(w.d_pobs, H4, arena + D.w_ih_off, I, w.d_obs_emb, E, d.B, H4, E, 0));
  }
  const int ph_obs = obs_fp32_plan_bwd(bl, D, arena, grad, b->obs, d.B, w);
  Problem* dprobs = w.problems + w.max_problems / 2;
  int rc = upload_and_get(net, bl, dprobs, w.max_problems / 2, st, kSlotSimtBwd);
  if (rc) return rc;

  // ---- launches -----------------------------------------------------------------------------------
  rc = run_phase(bl.phases[ph_dhid], dprobs, st); if (rc) return rc;
  rc = run_phase(bl.phases[ph_hw], dprobs, st); if (rc) return rc;
  rc = launch_head_bias_grad(net, b, w, grad, st); if (rc) return rc;
  // BPTT
  for (int t = d.T - 1; t >= 0; --t) {
    int r0 = b->row_off_host[t], n = b->row_off_host[t + 1] - r0;
    int n_next = (t + 1 < d.T) ? b->row_off_host[t + 2] - b->row_off_host[t + 1] : 0;
    const int ph = ph_rec0 + (d.T - 2 - t);
    if (n_next > 0) { rc = run_phase(bl.phases[ph], dprobs, st, profile(bl, ph)); if (rc) return rc; }
    k_cell_bwd<false><<<ew_grid((int64_t)n * H), 256, 0, st>>>(w.gates, w.c, w.dh, w.dh_rec, w.dc, dgates, w.d_pobs, b->row_prev,
                                                       b->row_next, b->row_trace, HImg(), r0, n, H, t, HImg());
    PPB_LAUNCH_CHECK();
  }
  rc = launch_step_inputs_bwd(net, arena, grad, b, w, dgates, st); if (rc) return rc;
  rc = run_phase(bl.phases[ph_lstm_w], dprobs, st, profile(bl, ph_lstm_w)); if (rc) return rc;
  return obs_fp32_bwd(bl, ph_obs, dprobs, D, grad, d.B, w, st);
}

}  // namespace

// =====================================================================================================
extern "C" {

int ppb_net_create(ppb_net** out, const ppb_net_desc* d) {
  PPB_CHECK_ARG(out && d, "null argument");
  PPB_CHECK_ARG(d->network_type == PPB_NET_LSTM || d->network_type == PPB_NET_FEEDFORWARD, "unknown network type");
  if (d->network_type == PPB_NET_FEEDFORWARD)
    PPB_CHECK_ARG(d->obs_dim > 0 && d->lstm_dim == 0 && d->sample_dim == 0 && d->addr_dim == 0 && d->type_dim == 0,
                  "bad dims (a feed-forward net has obs_dim > 0 and no LSTM, sample, address or type embedding)");
  else
    PPB_CHECK_ARG(d->lstm_dim > 0 && d->obs_dim > 0 && d->sample_dim > 0 && d->sample_dim <= 8, "bad dims");
  PPB_CHECK_ARG(d->num_obs > 0 && d->num_obs <= PPB_MAX_OBS, "bad observable count");
  PPB_CHECK_ARG(d->mixture_k > 0 && d->mixture_k <= heads::KMAX, "mixture components must be in [1,32]");
  ppb_net* n = new ppb_net();
  n->desc = *d;
  n->I = d->obs_dim + d->sample_dim + 2 * (d->type_dim + d->addr_dim);
  const char* fc = getenv("PPB_FUSED_CELL");
  // LSTM steps t >= 1: recurrent GEMM + cell in one kernel per step, cluster split-K when the step has few tiles
  // (tc_cluster.cuh); PPB_FUSED_CELL=0 = GEMM and cell kernels, the reference the fused step is tested against
  n->fused_cell = !(fc && fc[0] == '0');
  const char* hg = getenv("PPB_HOST_STEP_GRAPH");
  n->host_graph = (hg && hg[0] == '0') ? 0 : 1;   // on by default (PPB_HOST_STEP_GRAPH=0: always launch eagerly)
  // created up front: a training step must be capturable in a CUDA graph right after its first eager run
  for (int i = 0; i < 16; ++i) PPB_CUDA(cudaEventCreateWithFlags(&n->fork_ev[i], cudaEventDisableTiming));
  for (int i = 0; i < 2; ++i) PPB_CUDA(cudaStreamCreateWithFlags(&n->side[i], cudaStreamNonBlocking));
  *out = n;
  return PPB_OK;
}

int ppb_net_set_tables(ppb_net* net, const ppb_addr_desc* addrs, int32_t n_addrs, const int64_t* type_off,
                       int32_t n_types, int64_t arena_floats) {
  const bool ff = net && net->desc.network_type == PPB_NET_FEEDFORWARD;
  PPB_CHECK_ARG(net && addrs && n_addrs > 0 && (ff ? n_types == 0 : (type_off && n_types > 0)), "bad arguments");
  net->addrs.assign(addrs, addrs + n_addrs);
  net->type_off.assign(type_off, type_off + n_types);
  net->arena_floats = arena_floats;
  int dh = 4, op = 4;
  for (auto& a : net->addrs) {
    PPB_CHECK_ARG(a.family >= 0 && a.family <= PPB_FAMILY_BERNOULLI, "unknown family");
    PPB_CHECK_ARG(a.family != PPB_FAMILY_CATEGORICAL || (a.num_categories > 0 && a.num_categories <= heads::CMAX),
                  "categorical head: 1..128 categories supported");
    PPB_CHECK_ARG(a.family != PPB_FAMILY_BERNOULLI || (a.head_out == 1 && a.smp_in == 1 && a.num_categories == 0),
                  "bernoulli head: head_out = 1, smp_in = 1, num_categories = 0");
    PPB_CHECK_ARG(ff || (a.type_id >= 0 && a.type_id < n_types), "type id out of range");
    if (a.head_hidden > dh) dh = a.head_hidden;
    if (a.head_out > op) op = a.head_out;
  }
  net->dh_pad = (int)align_up(dh, 4);
  net->out_pad = (int)align_up(op, 4);
  if (net->d_addrs) cudaFree(net->d_addrs);
  if (net->d_type_off) cudaFree(net->d_type_off);
  net->d_type_off = nullptr;
  PPB_CUDA(cudaMalloc((void**)&net->d_addrs, sizeof(ppb_addr_desc) * n_addrs));
  PPB_CUDA(cudaMemcpy(net->d_addrs, addrs, sizeof(ppb_addr_desc) * n_addrs, cudaMemcpyHostToDevice));
  if (n_types > 0) {
    PPB_CUDA(cudaMalloc((void**)&net->d_type_off, sizeof(int64_t) * n_types));
    PPB_CUDA(cudaMemcpy(net->d_type_off, type_off, sizeof(int64_t) * n_types, cudaMemcpyHostToDevice));
  }
  return build_weight_images(net);
}

int ppb_net_destroy(ppb_net* net) {
  if (!net) return PPB_OK;
  if (net->d_addrs) cudaFree(net->d_addrs);
  if (net->d_type_off) cudaFree(net->d_type_off);
  for (int i = 0; i < 2; ++i) {
    if (net->h_stage[i]) cudaFreeHost(net->h_stage[i]);
    if (net->ev_stage[i]) cudaEventDestroy(net->ev_stage[i]);
    if (net->h_blob[i]) cudaFreeHost(net->h_blob[i]);
    if (net->ev_blob[i]) cudaEventDestroy(net->ev_blob[i]);
  }
  for (int i = 0; i < 2; ++i) if (net->side[i]) cudaStreamDestroy(net->side[i]);
  for (int i = 0; i < 16; ++i) if (net->fork_ev[i]) cudaEventDestroy(net->fork_ev[i]);
  if (net->wimg) cudaFree(net->wimg);
  if (net->d_pack) cudaFree(net->d_pack);
  if (net->whh_il) cudaFree(net->whh_il);
  if (net->d_lstm_steps) cudaFree(net->d_lstm_steps);
  if (net->host_exec) cudaGraphExecDestroy(net->host_exec);
  if (net->host_stream) cudaStreamDestroy(net->host_stream);
  if (net->host_hyper_dev) cudaFree(net->host_hyper_dev);
  if (net->host_state_dev) cudaFree(net->host_state_dev);
  if (net->host_pin) cudaFreeHost(net->host_pin);
  delete net;
  return PPB_OK;
}

int64_t ppb_ic_workspace_bytes(const ppb_net* net, int32_t n_traces, int32_t n_rows, int32_t t_max, int32_t n_steps,
                               int32_t n_groups) {
  if (!net || n_traces <= 0 || n_rows <= 0) return -1;
  Dims d; d.B = n_traces; d.R = n_rows; d.T = t_max; d.NS = n_steps; d.G = n_groups;
  // SIMT region (fp32 activations + dgates) followed by the tensor-core tail (tile images, problem lists)
  return simt_region_bytes(net, d) + carve_tc(net, d, nullptr).total_bytes + 1024;
}

// The workspace regions move with the batch dims (carve, carve_tc; carve_infer with n), so a call with another layout may
// write its buffers over a list an earlier call uploaded (a no-grad forward of a larger batch over the last step's backward
// lists, _infer_init's embedding over the infer step's list): when the workspace address or the layout key changes, the
// lists of slots [first, last] are sent again.  kSlotLstmSteps (the fused LSTM step list) lives in memory the net owns.
static void forget_on_new_layout(ppb_net* net, uint64_t& last_key, const void* key, size_t key_bytes, const void* workspace,
                                 UploadSlot first, UploadSlot last) {
  const uint64_t h = fnv1a(&workspace, sizeof(workspace), fnv1a(key, key_bytes));
  if (h == last_key) return;
  for (int i = first; i <= last; ++i) net->slot_hash[i] = 0;
  last_key = h;
}

int ppb_ic_loss_forward(ppb_net* net, const float* arena, const ppb_batch* b, void* workspace,
                        int64_t workspace_bytes, int precision, float* loss_out, int32_t* status_out,
                        float* row_lp_out, int want_grad, void* stream) {
  int rc = check_batch(net, b);
  if (rc) return rc;
  PPB_CHECK_ARG(arena && workspace, "null arena/workspace");
  PPB_CHECK_ARG(!net->addrs.empty(), "address tables not set");
  PPB_CHECK_ARG(precision >= 0 && precision <= 2, "unknown precision mode");
  Dims d = dims_of(b);
  PPB_CHECK_ARG(workspace_bytes >= ppb_ic_workspace_bytes(net, d.B, d.R, d.T, d.NS, d.G), "workspace too small");
  {
    const int key[6] = {d.B, d.R, d.T, d.NS, d.G, precision};
    forget_on_new_layout(net, net->ws_layout, key, sizeof(key), workspace, kSlotSimtFwd, kSlotChunks);
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (net->desc.network_type == PPB_NET_FEEDFORWARD)
    return ff_loss_forward(net, arena, b, workspace, precision, loss_out, status_out, row_lp_out, want_grad, st);
  if (precision != PPB_PREC_FP32_SIMT)
    return tc_loss_forward(net, arena, b, workspace, precision, loss_out, status_out, row_lp_out, want_grad, st);
  return simt_loss_forward(net, arena, b, workspace, loss_out, status_out, row_lp_out, want_grad, st);
}

int ppb_ic_loss_backward(ppb_net* net, const float* arena, float* grad, const ppb_batch* b, void* workspace,
                         int64_t workspace_bytes, int precision, float grad_scale, void* stream) {
  int rc = check_batch(net, b);
  if (rc) return rc;
  PPB_CHECK_ARG(arena && grad && workspace, "null arena/grad/workspace");
  Dims d = dims_of(b);
  PPB_CHECK_ARG(workspace_bytes >= ppb_ic_workspace_bytes(net, d.B, d.R, d.T, d.NS, d.G), "workspace too small");
  {
    const int key[6] = {d.B, d.R, d.T, d.NS, d.G, precision};
    forget_on_new_layout(net, net->ws_layout, key, sizeof(key), workspace, kSlotSimtFwd, kSlotChunks);
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (net->desc.network_type == PPB_NET_FEEDFORWARD)
    return ff_loss_backward(net, arena, grad, b, workspace, precision, grad_scale, st);
  if (precision != PPB_PREC_FP32_SIMT) return tc_loss_backward(net, arena, grad, b, workspace, precision, grad_scale, st);
  return simt_loss_backward(net, arena, grad, b, workspace, grad_scale, st);
}

}  // extern "C"

// =====================================================================================================
// batch image decoding, Adam, inference-time entry points, host-buffer training step
// =====================================================================================================
namespace {

// Graph-replayable Adam: step counter and hyper-parameters live in device memory.  Every block derives the bias
// corrections of step t+1 itself; the last block to finish advances the counter (the Adam state block of
// include/pyprob_b200.h).
__global__ void __launch_bounds__(256) k_adam_dev(float* __restrict__ p, const float* __restrict__ g,
                                                   float* __restrict__ m, float* __restrict__ v, int64_t n, int vec,
                                                   const float* __restrict__ hyper, long long* __restrict__ step_ctr,
                                                   float* __restrict__ bc1_out, unsigned int* __restrict__ done_ctr) {
  ppb_pdl_trigger();
  ppb_pdl_wait();
  __shared__ float s_bc[2];
  __shared__ long long s_t;
  // the gradient / moment loads of the first pass are issued BEFORE the block waits for thread 0's two double-precision
  // pow() calls (the bias corrections used to sit in front of every block's first load)
  const int64_t n4 = vec ? (n >> 2) : 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 gg = z4, mm = z4, vv = z4;
  if (q < n4) {
    gg = reinterpret_cast<const float4*>(g)[q];
    mm = reinterpret_cast<float4*>(m)[q];
    vv = reinterpret_cast<float4*>(v)[q];
  }
  if (threadIdx.x == 0) {
    long long t = *step_ctr + 1;
    s_t = t;
    ppb_adam_bias_corrections(hyper, t, s_bc[0], s_bc[1]);
  }
  __syncthreads();
  const float lr = hyper[PPB_HYPER_LR], b1 = hyper[PPB_HYPER_BETA1], b2 = hyper[PPB_HYPER_BETA2];
  const float eps = hyper[PPB_HYPER_EPS], wd = hyper[PPB_HYPER_WEIGHT_DECAY], gscale = hyper[PPB_HYPER_GRAD_SCALE];
  const float step = lr / s_bc[0], bc2_sqrt = s_bc[1];
  while (q < n4) {
    // a tensor that has never seen a gradient (g = m = v = 0) and no weight decay: the update is exactly zero — skip
    // the parameter read and all three writes (T = 1 models never touch W_hh: 64 % of the configs[1] arena)
    const bool zero = wd == 0.0f && gg.x == 0.0f && gg.y == 0.0f && gg.z == 0.0f && gg.w == 0.0f && mm.x == 0.0f &&
                      mm.y == 0.0f && mm.z == 0.0f && mm.w == 0.0f && vv.x == 0.0f && vv.y == 0.0f && vv.z == 0.0f &&
                      vv.w == 0.0f;
    if (!zero) {
      float4 pp = reinterpret_cast<float4*>(p)[q];
      ppb_adam_update(pp.x, gg.x, mm.x, vv.x, b1, b2, eps, wd, gscale, step, bc2_sqrt);
      ppb_adam_update(pp.y, gg.y, mm.y, vv.y, b1, b2, eps, wd, gscale, step, bc2_sqrt);
      ppb_adam_update(pp.z, gg.z, mm.z, vv.z, b1, b2, eps, wd, gscale, step, bc2_sqrt);
      ppb_adam_update(pp.w, gg.w, mm.w, vv.w, b1, b2, eps, wd, gscale, step, bc2_sqrt);
      reinterpret_cast<float4*>(p)[q] = pp;
      reinterpret_cast<float4*>(m)[q] = mm;
      reinterpret_cast<float4*>(v)[q] = vv;
    }
    q += stride;
    if (q < n4) {
      gg = reinterpret_cast<const float4*>(g)[q];
      mm = reinterpret_cast<float4*>(m)[q];
      vv = reinterpret_cast<float4*>(v)[q];
    }
  }
  for (int64_t i = (n4 << 2) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    float pi = p[i], mi = m[i], vi = v[i];
    ppb_adam_update(pi, g[i], mi, vi, b1, b2, eps, wd, gscale, step, bc2_sqrt);
    m[i] = mi; v[i] = vi; p[i] = pi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(done_ctr, 1u) == gridDim.x - 1) {   // every block has read the counter by now
      *step_ctr = s_t;
      *bc1_out = s_bc[0];
      *done_ctr = 0u;
    }
  }
}

// inference-time cell: n particles in lock-step at one address; state updated in place.
// p_row = step projection + biases + (shared) observation projection, identical for all particles.
__global__ void __launch_bounds__(256) k_cell_infer(const float* __restrict__ rec, const float* __restrict__ p_row,
                                                     const float* __restrict__ w_smp_t,
                                                     const float* __restrict__ smp_emb, float* __restrict__ c,
                                                     float* __restrict__ h, int64_t n, int H, int S, int first) {
  int64_t total = n * H;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    int64_t i = e / H;
    int j = (int)(e % H);
    float pre[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      int col = g * H + j;
      float v = p_row[col];
      if (!first) {
        v += rec[i * 4 * H + col];
        for (int s = 0; s < S; ++s) v = fmaf(smp_emb[i * S + s], w_smp_t[(int64_t)s * 4 * H + col], v);
      }
      pre[g] = v;
    }
    const CellFwd u = cell_fwd_unit(pre, [&] { return first ? 0.0f : c[i * H + j]; });
    c[i * H + j] = u.c;
    h[i * H + j] = u.h;
  }
}

__global__ void k_smp_embed_infer(const float* __restrict__ arena, ppb_addr_desc a, const float* __restrict__ value,
                                  int64_t n, int S, float* __restrict__ smp_emb) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n * S; e += (int64_t)gridDim.x * blockDim.x) {
    int64_t i = e / S;
    int j = (int)(e % S);
    smp_emb[e] = fmaxf(smp_embed_pre(arena, a, value[i], j), 0.0f);
  }
}

__global__ void k_step_row_infer(const float* __restrict__ arena, ppb_addr_desc prev, int has_prev, ppb_addr_desc cur,
                                 const int64_t* __restrict__ type_off, int td, int ad, float* __restrict__ row) {
  int C2 = 2 * (td + ad);
  for (int j = threadIdx.x; j < C2; j += blockDim.x) {
    const int64_t o = step_embed_off(type_off, td, ad, j, [&](bool is_prev, const ppb_addr_desc*& a) {
      a = is_prev ? &prev : &cur;
      return !is_prev || has_prev;
    });
    row[j] = o >= 0 ? arena[o] : 0.0f;
  }
}

// raw head output -> distribution parameters as the reference's proposal layers return them
__global__ void __launch_bounds__(128) k_head_params(const float* __restrict__ out_raw, int out_pad, ppb_addr_desc a,
                                                      int K, const float* __restrict__ prior0, int s0,
                                                      const float* __restrict__ prior1, int s1,
                                                      float* __restrict__ params, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float* x = out_raw + i * out_pad;
    if (a.family == PPB_FAMILY_BERNOULLI) {
      params[i] = heads::bernoulli_prob(x[0]);
    } else if (a.family == PPB_FAMILY_CATEGORICAL) {
      float xs[heads::CMAX], q[heads::CMAX];
      for (int c = 0; c < a.num_categories; ++c) xs[c] = x[c];
      heads::categorical_probs(xs, a.num_categories, q);
      for (int c = 0; c < a.num_categories; ++c) params[i * a.num_categories + c] = q[c];
    } else {
      float xs[3 * heads::KMAX], mean[heads::KMAX], sd[heads::KMAX], pr[heads::KMAX], lo, hi;
      for (int j = 0; j < 3 * K; ++j) xs[j] = x[j];
      float p0 = prior0 ? prior0[i * s0] : 0.0f, p1 = prior1 ? prior1[i * s1] : 0.0f;
      heads::mixture_params(a.family, xs, K, p0, p1, mean, sd, pr, &lo, &hi);
      for (int k = 0; k < K; ++k) {
        params[i * 3 * K + k] = mean[k];
        params[i * 3 * K + K + k] = sd[k];
        params[i * 3 * K + 2 * K + k] = pr[k];
      }
    }
  }
}

struct InferWs {
  HImg h_img, hid_img;        // tensor-core operands (K-format)
  tcg::Problem* tprobs;
  float *gates, *hid, *out_raw, *smp_emb, *p_row, *emb_row, *w_smp_t;
  float* obs_act[PPB_MAX_OBS][PPB_MAX_FF_LAYERS];
  float* obs_cat;
  float* fin_act[PPB_MAX_FF_LAYERS];
  Problem* problems;
  int64_t max_problems, total_bytes;
};

InferWs carve_infer(const ppb_net* net, int64_t n, void* base) {
  const ppb_net_desc& D = net->desc;
  InferWs w;
  memset(&w, 0, sizeof(w));
  char* p = (char*)base;
  int64_t off = 0;
  auto take = [&](int64_t floats) { float* r = (float*)(p + off); off += align_up(floats * 4, 256); return r; };
  const int H4 = 4 * D.lstm_dim;
  w.gates = take(n * H4);
  w.hid = take(n * net->dh_pad);
  w.out_raw = take(n * net->out_pad);
  w.smp_emb = take(n * D.sample_dim);
  w.p_row = take(H4);
  w.emb_row = take(2 * (D.type_dim + D.addr_dim));
  w.w_smp_t = take((int64_t)D.sample_dim * H4);
  for (int j = 0; j < D.num_obs; ++j)
    for (int l = 0; l + 1 < D.obs_ff[j].num_layers; ++l) w.obs_act[j][l] = take(n * D.obs_ff[j].layers[l].out_dim);
  w.obs_cat = take(n * D.obs_dim);
  for (int l = 0; l + 1 < D.obs_final.num_layers; ++l) w.fin_act[l] = take(n * D.obs_final.layers[l].out_dim);
  w.max_problems = 64 + 2LL * PPB_MAX_OBS * PPB_MAX_FF_LAYERS;
  w.problems = (Problem*)take(w.max_problems * (int64_t)(sizeof(Problem) / 4));
  auto img_k = [&](int64_t rows, int64_t cols) {
    HImg im;
    int64_t nfl = tc::img_floats(rows, cols);
    off = align_up(off, 1024);
    im.kb = (cols + 31) / 32;
    im.k_hi = take(nfl); im.k_lo = take(nfl);
    return im;
  };
  w.h_img = img_k(n, D.lstm_dim);
  w.hid_img = img_k(n, net->dh_pad);
  w.tprobs = (tcg::Problem*)take(8 * (int64_t)(sizeof(tcg::Problem) / 4));
  w.total_bytes = off;
  return w;
}

}  // namespace

int prof_begin(double flops, cudaStream_t st, cudaEvent_t& e0) {
  e0 = nullptr;
  if (flops <= 0.0 || !g_prof.on) return PPB_OK;
  PPB_CUDA(cudaEventCreate(&e0));
  PPB_CUDA(cudaEventRecord(e0, st));
  return PPB_OK;
}
int prof_end(cudaEvent_t e0, cudaStream_t st, double flops) {
  if (!e0) return PPB_OK;
  cudaEvent_t e1;
  PPB_CUDA(cudaEventCreate(&e1));
  PPB_CUDA(cudaEventRecord(e1, st));
  g_prof.spans.push_back({e0, e1});
  g_prof.launches += 1;
  g_prof.flops += flops;
  return PPB_OK;
}

extern "C" {

int ppb_prof_enable(int on) {
  for (auto& sp : g_prof.spans) { cudaEventDestroy(sp.first); cudaEventDestroy(sp.second); }
  g_prof.spans.clear();
  g_prof.flops = 0.0;
  g_prof.launches = 0;
  g_prof.on = on != 0;
  return PPB_OK;
}

int ppb_prof_read(double* total_ms_out, int64_t* launches_out, double* flops_out) {
  double total = 0.0;
  for (auto& sp : g_prof.spans) {
    PPB_CUDA(cudaEventSynchronize(sp.second));
    float ms = 0.0f;
    PPB_CUDA(cudaEventElapsedTime(&ms, sp.first, sp.second));
    total += ms;
  }
  if (total_ms_out) *total_ms_out = total;
  if (launches_out) *launches_out = g_prof.launches;
  if (flops_out) *flops_out = g_prof.flops;
  return PPB_OK;
}

int64_t ppb_sizeof(int which) {
  switch (which) {
    case 0: return sizeof(ppb_net_desc);
    case 1: return sizeof(ppb_addr_desc);
    case 2: return sizeof(ppb_batch);
    case 3: return sizeof(ppb_ff_desc);
    case 4: return sizeof(ppb_linear_desc);
    case 5: return sizeof(tcg::Problem);
    default: return -1;
  }
}

int ppb_batch_from_image(const void* image_host, const void* image_dev, int64_t image_bytes, ppb_batch* out) {
  PPB_CHECK_ARG(image_host && out, "null image");
  const int64_t* hd = (const int64_t*)image_host;
  PPB_CHECK_ARG(image_bytes >= (int64_t)(PPB_IMAGE_HEADER_WORDS * 8), "image too small");
  PPB_CHECK_ARG(hd[0] == PPB_IMAGE_MAGIC, "bad batch image magic");
  PPB_CHECK_ARG(hd[8] == image_bytes, "image size mismatch");
  memset(out, 0, sizeof(*out));
  out->n_traces = (int32_t)hd[1]; out->n_sub = (int32_t)hd[2]; out->t_max = (int32_t)hd[3];
  out->n_rows = (int32_t)hd[4]; out->n_steps = (int32_t)hd[5]; out->n_groups = (int32_t)hd[6];
  out->obs_in_total = (int32_t)hd[7];
  for (int k = 9; k < 9 + 19; ++k)
    PPB_CHECK_ARG(hd[k] >= PPB_IMAGE_HEADER_WORDS * 8 && hd[k] < image_bytes && (hd[k] & 15) == 0, "bad array offset");
  out->row_align = (int32_t)hd[28];
  PPB_CHECK_ARG(out->row_align == 1 || out->row_align == 128, "row_align must be 1 or 128");
  const char* Hh = (const char*)image_host;
  const char* Dv = (const char*)image_dev;
  out->row_off_host = (const int32_t*)(Hh + hd[9]);
  out->group_addr_host = (const int32_t*)(Hh + hd[10]);
  out->group_start_host = (const int32_t*)(Hh + hd[11]);
  out->step_addr_host = (const int32_t*)(Hh + hd[13]);
  out->step_row0_host = (const int32_t*)(Hh + hd[15]);
  out->step_nrows_host = (const int32_t*)(Hh + hd[16]);
  out->step_t_host = (const int32_t*)(Hh + hd[26]);
  out->step_prev_row0_host = (const int32_t*)(Hh + hd[27]);
  if (Dv) {
    out->trace_sub = (const int32_t*)(Dv + hd[12]);
    out->step_addr = (const int32_t*)(Dv + hd[13]);
    out->step_prev_addr = (const int32_t*)(Dv + hd[14]);
    out->step_row0 = (const int32_t*)(Dv + hd[15]);
    out->step_nrows = (const int32_t*)(Dv + hd[16]);
    out->row_step = (const int32_t*)(Dv + hd[17]);
    out->row_prev = (const int32_t*)(Dv + hd[18]);
    out->values = (const float*)(Dv + hd[19]);
    out->prior0 = (const float*)(Dv + hd[20]);
    out->prior1 = (const float*)(Dv + hd[21]);
    out->obs = (const float*)(Dv + hd[22]);
    out->head_rows = (const int32_t*)(Dv + hd[23]);
    out->row_trace = (const int32_t*)(Dv + hd[24]);
    out->row_next = (const int32_t*)(Dv + hd[25]);
    out->step_t = (const int32_t*)(Dv + hd[26]);
    out->step_prev_row0 = (const int32_t*)(Dv + hd[27]);
    out->group_addr = (const int32_t*)(Dv + hd[10]);
    out->group_start = (const int32_t*)(Dv + hd[11]);
  }
  return PPB_OK;
}

// Graph-replayable Adam: the step counter and the hyper-parameters live in device memory, so a captured
// training step stays valid while the count advances and the learning rate follows its schedule.  The float4 path
// needs all four arrays 16-byte aligned; otherwise every element takes the scalar loop.
int ppb_adam_step_dev(float* arena, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n,
                      const float* hyper_dev, void* state_dev, void* stream) {
  PPB_CHECK_ARG(arena && grad && exp_avg && exp_avg_sq && hyper_dev && state_dev && n > 0, "bad arguments");
  const int vec = ((((uintptr_t)arena | (uintptr_t)grad | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15) == 0) ? 1 : 0;
  PPB_CUDA(ppb_launch(k_adam_dev, dim3(ppb_grid_for(n, 256, 4)), dim3(256), 0, (cudaStream_t)stream, 0, 0, arena, grad,
                      exp_avg, exp_avg_sq, n, vec, hyper_dev, (long long*)state_dev, (float*)((char*)state_dev + 8),
                      (unsigned int*)((char*)state_dev + 12)));
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int ppb_net_forget_uploads(ppb_net* net) {
  PPB_CHECK_ARG(net, "bad arguments");
  for (int i = 0; i < kNumUploadSlots; ++i) net->slot_hash[i] = 0;
  return PPB_OK;
}

int ppb_net_refresh_weights(ppb_net* net, const float* arena, void* stream) {
  PPB_CHECK_ARG(net && arena && net->wimg, "bad arguments (tables not set?)");
  k_pack_table<<<dim3(net->pack_tiles, 8), 256, 0, (cudaStream_t)stream>>>(arena, net->d_pack, (int)net->pack.size(), net->wimg);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int64_t ppb_ic_infer_workspace_bytes(const ppb_net* net, int64_t n) {
  if (!net || n <= 0) return -1;
  return carve_infer(net, n, nullptr).total_bytes + 1024;
}

int ppb_ic_embed_observe(ppb_net* net, const float* arena, const float* obs, float* obs_emb_out, int64_t n,
                         void* workspace, int64_t workspace_bytes, void* stream) {
  PPB_CHECK_ARG(net && arena && obs && obs_emb_out && workspace && n > 0, "bad arguments");
  PPB_CHECK_ARG(workspace_bytes >= ppb_ic_infer_workspace_bytes(net, n), "workspace too small");
  {
    const int64_t key[2] = {n, 0};
    forget_on_new_layout(net, net->infer_layout, key, sizeof(key), workspace, kSlotInferSimt, kSlotInferTc);
  }
  cudaStream_t st = (cudaStream_t)stream;
  InferWs w = carve_infer(net, n, workspace);
  if (net->wimg) {  // inference starts here (_infer_init): bring the tensor-core weight images up to date
    int rcw = ppb_net_refresh_weights(net, arena, stream);
    if (rcw) return rcw;
  }
  Builder bl;
  obs_fp32_plan_fwd(bl, net->desc, arena, obs, (int)n, w, obs_emb_out);
  int rc = upload_and_get(net, bl, w.problems, w.max_problems, st, kSlotInferSimt);
  if (rc) return rc;
  for (auto& ph : bl.phases) { rc = run_phase(ph, w.problems, st); if (rc) return rc; }
  return PPB_OK;
}

int ppb_ic_infer_step(ppb_net* net, const float* arena, const float* obs_emb, int obs_emb_row_stride, int32_t prev_addr,
                      const float* prev_value, int32_t cur_addr, const float* prior0, int prior0_stride,
                      const float* prior1, int prior1_stride, float* h, float* c, float* params_out, int64_t n,
                      void* workspace, int64_t workspace_bytes, int precision, void* stream) {
  PPB_CHECK_ARG(net && arena && obs_emb && params_out && workspace && n > 0, "bad arguments");
  PPB_CHECK_ARG(cur_addr >= 0 && cur_addr < (int)net->addrs.size(), "unknown current address");
  PPB_CHECK_ARG(workspace_bytes >= ppb_ic_infer_workspace_bytes(net, n), "workspace too small");
  if (obs_emb_row_stride != 0) {
    ppb_set_error("ppb_ic_infer_step: per-particle observation embeddings are not supported yet (stride must be 0)");
    return PPB_ENOTSUP;
  }
  const bool lstm = net->desc.network_type != PPB_NET_FEEDFORWARD;
  if (lstm) {
    PPB_CHECK_ARG(h && c, "bad arguments");
    PPB_CHECK_ARG(prev_addr < (int)net->addrs.size(), "unknown previous address");
    PPB_CHECK_ARG(prev_addr < 0 || prev_value, "previous value missing");
  }
  {
    const int64_t key[2] = {n, 1};
    forget_on_new_layout(net, net->infer_layout, key, sizeof(key), workspace, kSlotInferSimt, kSlotInferTc);
  }
  const ppb_net_desc& D = net->desc;
  cudaStream_t st = (cudaStream_t)stream;
  InferWs w = carve_infer(net, n, workspace);
  const int H = D.lstm_dim, H4 = 4 * H, E = D.obs_dim, S = D.sample_dim, I = net->I, C2 = 2 * (D.type_dim + D.addr_dim);
  const ppb_addr_desc cur = net->addrs[cur_addr];
  const bool first = prev_addr < 0;
  // The head reads the LSTM output h after the cell update, n rows.  The feed-forward head reads the observation embedding
  // (inference_network_feedforward.py:53-66); with one shared observation every particle's head output is the same, so it
  // runs on ONE row and k_head_params expands it over the particles (row stride 0), applying each particle's prior.
  const float* x = lstm ? h : obs_emb;
  const int x_dim = lstm ? H : E, head_rows = lstm ? (int)n : 1, out_stride = lstm ? net->out_pad : 0;
  // large LSTM GEMMs on the tensor cores (weight images must be current: ppb_net_refresh_weights / ppb_ic_embed_observe)
  const bool use_tc = lstm && precision != PPB_PREC_FP32_SIMT && (H % 32 == 0) && net->wimg != nullptr;

  // One phase per GEMM, at the same index in both problem lists.  The p_row GEMMs run on the CUDA cores; the recurrent and
  // head GEMMs go to the tensor-core list when use_tc, else to the SIMT list.
  enum { kPRowStep, kPRowObs, kRecurrent, kHeadHidden, kHeadOut };
  Builder bl;
  bl.begin();  // kPRowStep: p_row = step_emb W_ih[:, E+S:]^T + b_ih
  if (lstm) bl.add(linear_fwd(w.emb_row, C2, arena + D.w_ih_off + E + S, I, arena + D.b_ih_off, w.p_row, H4, 1, H4, C2, 0));
  bl.begin();  // kPRowObs: p_row += obs_emb W_ih[:, :E]^T + b_hh   (one shared observation row)
  if (lstm) bl.add(linear_fwd(obs_emb, E, arena + D.w_ih_off, I, arena + D.b_hh_off, w.p_row, H4, 1, H4, E, gemm::kAccumulate));
  bl.begin();  // kRecurrent
  if (lstm && !first && !use_tc) bl.add(linear_fwd(h, H, arena + D.w_hh_off, H, nullptr, w.gates, H4, (int)n, H4, H, 0));
  bl.begin();  // kHeadHidden
  if (!use_tc)
    bl.add(linear_fwd(x, x_dim, arena + cur.w1_off, x_dim, arena + cur.b1_off, w.hid, net->dh_pad, head_rows, cur.head_hidden,
                      x_dim, gemm::kRelu));
  bl.begin();  // kHeadOut
  if (!use_tc)
    bl.add(linear_fwd(w.hid, net->dh_pad, arena + cur.w2_off, cur.head_hidden, arena + cur.b2_off, w.out_raw, net->out_pad,
                      head_rows, cur.head_out, cur.head_hidden, 0));
  int rc = upload_and_get(net, bl, w.problems, w.max_problems, st, kSlotInferSimt);
  if (rc) return rc;
  TcBuilder tb;
  if (use_tc) {
    tb.begin(); tb.begin();  // kPRowStep, kPRowObs: SIMT list only
    tb.begin();  // kRecurrent
    if (!first) {
      tcg::Problem p = TP0();
      p.a = op_k(w.h_img.k_hi, w.h_img.k_lo, (int)w.h_img.kb, 0, 0);
      p.b = wk(net, net->w_hh);
      p.M = (int)n; p.N = H4; p.K = H; p.c = w.gates; p.ldc = H4;
      tb.add(p);
    }
    tb.begin();  // kHeadHidden: head trunk -> hid image
    {
      tcg::Problem p = TP0();
      p.a = op_k(w.h_img.k_hi, w.h_img.k_lo, (int)w.h_img.kb, 0, 0);
      p.b = wk(net, net->w1[cur_addr]);
      p.M = (int)n; p.N = cur.head_hidden; p.K = H;
      p.flags = tcg::kRelu; p.bias = arena + cur.b1_off;
      p.o_k_hi = w.hid_img.k_hi; p.o_k_lo = w.hid_img.k_lo; p.o_kb = (int)w.hid_img.kb;
      tb.add(p);
    }
    tb.begin();  // kHeadOut
    {
      tcg::Problem p = TP0();
      p.a = op_k(w.hid_img.k_hi, w.hid_img.k_lo, (int)w.hid_img.kb, 0, 0);
      p.b = wk(net, net->w2[cur_addr]);
      p.M = (int)n; p.N = cur.head_out; p.K = cur.head_hidden;
      p.bias = arena + cur.b2_off; p.c = w.out_raw; p.ldc = net->out_pad;
      tb.add(p);
    }
    rc = upload_cached(net, kSlotInferTc, tb.probs.data(), tb.probs.size() * sizeof(tcg::Problem), w.tprobs, st);
    if (rc) return rc;
  }
  const dim3 pack_grid((unsigned)((n + 127) / 128), 4);
  if (lstm) {
    const ppb_addr_desc prev = first ? cur : net->addrs[prev_addr];
    k_step_row_infer<<<1, 128, 0, st>>>(arena, prev, first ? 0 : 1, cur, net->d_type_off, D.type_dim, D.addr_dim, w.emb_row);
    PPB_LAUNCH_CHECK();
    rc = run_phase(bl.phases[kPRowStep], w.problems, st); if (rc) return rc;
    rc = run_phase(bl.phases[kPRowObs], w.problems, st); if (rc) return rc;
    if (!first) {
      k_wsmp_transpose<<<ew_grid(S * H4), 256, 0, st>>>(arena + D.w_ih_off, I, E, S, H4, w.w_smp_t);
      PPB_LAUNCH_CHECK();
      k_smp_embed_infer<<<ew_grid(n * S), 256, 0, st>>>(arena, prev, prev_value, n, S, w.smp_emb);
      PPB_LAUNCH_CHECK();
      if (use_tc) {
        k_pack_rows<<<pack_grid, 256, 0, st>>>(h, (int)n, H, H, w.h_img);
        PPB_LAUNCH_CHECK();
        rc = run_tc_phase<0>(tb.phases[kRecurrent], w.tprobs, precision, st); if (rc) return rc;
      } else {
        rc = run_phase(bl.phases[kRecurrent], w.problems, st); if (rc) return rc;
      }
    }
    k_cell_infer<<<ew_grid(n * H), 256, 0, st>>>(w.gates, w.p_row, w.w_smp_t, w.smp_emb, c, h, n, H, S, first ? 1 : 0);
    PPB_LAUNCH_CHECK();
  }
  if (use_tc) {
    k_pack_rows<<<pack_grid, 256, 0, st>>>(h, (int)n, H, H, w.h_img);
    PPB_LAUNCH_CHECK();
    rc = run_tc_phase<2>(tb.phases[kHeadHidden], w.tprobs, precision, st); if (rc) return rc;
    rc = run_tc_phase<0>(tb.phases[kHeadOut], w.tprobs, precision, st); if (rc) return rc;
  } else {
    rc = run_phase(bl.phases[kHeadHidden], w.problems, st); if (rc) return rc;
    rc = run_phase(bl.phases[kHeadOut], w.problems, st); if (rc) return rc;
  }
  k_head_params<<<ew_grid(n, 128), 128, 0, st>>>(w.out_raw, out_stride, cur, D.mixture_k, prior0, prior0_stride, prior1,
                                                 prior1_stride, params_out, n);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int ppb_ic_train_step_host(ppb_net* net, float* arena, float* grad_arena, float* exp_avg, float* exp_avg_sq,
                           int64_t arena_floats, const void* batch_image_host, int64_t batch_image_bytes,
                           void* batch_image_dev, void* workspace, int64_t workspace_bytes, int precision, float lr,
                           float beta1, float beta2, float eps, float weight_decay, int64_t step, float* loss_host,
                           int32_t* status_host, void* stream) {
  PPB_CHECK_ARG(net && arena && grad_arena && exp_avg && exp_avg_sq && batch_image_host && batch_image_dev && workspace,
                "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  ppb_batch b;
  int rc = ppb_batch_from_image(batch_image_host, batch_image_dev, batch_image_bytes, &b);
  if (rc) return rc;
  Dims d = dims_of(&b);
  int64_t need = ppb_ic_workspace_bytes(net, d.B, d.R, d.T, d.NS, d.G);
  PPB_CHECK_ARG(workspace_bytes >= need + 256, "workspace too small (need ppb_ic_workspace_bytes + 256)");
  float* loss_dev = (float*)((char*)workspace + need);  // loss scalar + status live after the carved region
  int32_t* status_dev = (int32_t*)(loss_dev + 1);

  // The launches of a step depend only on the batch STRUCTURE (host index arrays) and on the buffers: the first call with a
  // structure runs eagerly (and uploads the problem lists), the second captures the step into a graph on an internal
  // stream, later calls replay it.  With PPB_HOST_STEP_GRAPH=0 or kernel profiling on, every call runs eagerly on that
  // stream.  Adam's step count and hyper-parameters live in device memory.
  if (!net->host_stream) {
    PPB_CUDA(cudaStreamCreateWithFlags(&net->host_stream, cudaStreamNonBlocking));
    PPB_CUDA(cudaMalloc((void**)&net->host_hyper_dev, sizeof(net->host_hyper)));
    PPB_CUDA(cudaMalloc(&net->host_state_dev, 16));
    PPB_CUDA(cudaMemset(net->host_state_dev, 0, 16));
    net->host_step_dev = 0;
  }
  cudaStream_t hs = net->host_stream;
  // The host->device copy of the batch image and the device->host read of (loss, status) are NODES of the step graph, out of
  // and into an internal pinned staging buffer: one cudaGraphLaunch + one synchronise per step instead of five stream calls,
  // and the copies start without a stream round trip.
  if (net->host_pin_cap < batch_image_bytes + 16) {
    PPB_CUDA(cudaStreamSynchronize(hs));
    if (net->host_pin) cudaFreeHost(net->host_pin);
    net->host_pin_cap = 2 * batch_image_bytes + 16;
    PPB_CUDA(cudaHostAlloc((void**)&net->host_pin, (size_t)net->host_pin_cap, cudaHostAllocDefault));
  }
  char* const pin_img = net->host_pin;
  char* const pin_res = net->host_pin + (net->host_pin_cap - 16);
  uint64_t key = fnv1a(&d, sizeof(d));
  key = fnv1a(&batch_image_bytes, sizeof(batch_image_bytes), key);
  key = fnv1a(&pin_img, sizeof(pin_img), key);
  key = fnv1a(b.row_off_host, sizeof(int32_t) * (d.T + 1), key);
  key = fnv1a(b.group_addr_host, sizeof(int32_t) * d.G, key);
  key = fnv1a(b.group_start_host, sizeof(int32_t) * (d.G + 1), key);
  key = fnv1a(b.step_addr_host, sizeof(int32_t) * d.NS, key);
  key = fnv1a(b.step_row0_host, sizeof(int32_t) * d.NS, key);
  key = fnv1a(b.step_nrows_host, sizeof(int32_t) * d.NS, key);
  key = fnv1a(b.step_t_host, sizeof(int32_t) * d.NS, key);
  key = fnv1a(b.step_prev_row0_host, sizeof(int32_t) * d.NS, key);
  const void* ptrs[8] = {arena, grad_arena, exp_avg, exp_avg_sq, batch_image_dev, workspace, (const void*)(intptr_t)precision,
                         (const void*)(intptr_t)arena_floats};
  key = fnv1a(ptrs, sizeof(ptrs), key);
  key = fnv1a(&net->arena_floats, sizeof(net->arena_floats), key);
  if (key != net->host_key) {
    if (net->host_exec) { cudaGraphExecDestroy(net->host_exec); net->host_exec = nullptr; }
    net->host_key = key;
    net->host_seen = 0;
  }
  // order after whatever the caller queued on its stream
  rc = stream_after(net, st, hs);
  if (rc) return rc;
  memcpy(pin_img, batch_image_host, (size_t)batch_image_bytes);
  const float hyper[PPB_HYPER_ADAM_COUNT] = {lr, beta1, beta2, eps, weight_decay, 1.0f};
  if (memcmp(hyper, net->host_hyper, sizeof(hyper)) != 0) {
    memcpy(net->host_hyper, hyper, sizeof(hyper));
    PPB_CUDA(cudaMemcpyAsync(net->host_hyper_dev, net->host_hyper, sizeof(hyper), cudaMemcpyHostToDevice, hs));
  }
  if (net->host_step_dev != step - 1) {
    const int64_t prev = step - 1;
    PPB_CUDA(cudaMemcpyAsync(net->host_state_dev, &prev, sizeof(prev), cudaMemcpyHostToDevice, hs));
    PPB_CUDA(cudaStreamSynchronize(hs));   // `prev` lives on this frame
  }
  auto enqueue = [&](cudaStream_t q) -> int {
    PPB_CUDA(cudaMemcpyAsync(batch_image_dev, pin_img, batch_image_bytes, cudaMemcpyHostToDevice, q));
    PPB_CUDA(cudaMemsetAsync(grad_arena, 0, arena_floats * sizeof(float), q));
    int r = ppb_ic_loss_forward(net, arena, &b, workspace, need, precision, loss_dev, status_dev, nullptr, 1, (void*)q);
    if (r) return r;
    r = ppb_ic_loss_backward(net, arena, grad_arena, &b, workspace, need, precision, 1.0f, (void*)q);
    if (r) return r;
    r = ppb_adam_step_dev(arena, grad_arena, exp_avg, exp_avg_sq, arena_floats, net->host_hyper_dev, net->host_state_dev,
                          (void*)q);
    if (r) return r;
    PPB_CUDA(cudaMemcpyAsync(pin_res, loss_dev, 8, cudaMemcpyDeviceToHost, q));   // loss (float) + status (int32), adjacent
    return PPB_OK;
  };
  const bool use_graph = net->host_graph && !g_prof.on;
  if (use_graph && net->host_exec) {
    PPB_CUDA(cudaGraphLaunch(net->host_exec, hs));
  } else if (use_graph && net->host_seen >= 1) {
    cudaGraph_t graph = nullptr;
    PPB_CUDA(cudaStreamBeginCapture(hs, cudaStreamCaptureModeThreadLocal));
    rc = enqueue(hs);
    cudaError_t ce = cudaStreamEndCapture(hs, &graph);
    if (rc || ce != cudaSuccess || !graph) {
      if (graph) cudaGraphDestroy(graph);
      cudaGetLastError();
      if (rc) return rc;
      ppb_set_error("ppb_ic_train_step_host: graph capture failed: %s", cudaGetErrorString(ce));
      return (int)ce;
    }
    ce = cudaGraphInstantiate(&net->host_exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce != cudaSuccess) {
      net->host_exec = nullptr;
      ppb_set_error("ppb_ic_train_step_host: cudaGraphInstantiate: %s", cudaGetErrorString(ce));
      return (int)ce;
    }
    PPB_CUDA(cudaGraphLaunch(net->host_exec, hs));
  } else {
    rc = enqueue(hs);
    if (rc) return rc;
  }
  net->host_seen += 1;
  net->host_step_dev = step;
  PPB_CUDA(cudaStreamSynchronize(hs));
  if (loss_host) memcpy(loss_host, pin_res, sizeof(float));
  if (status_host) memcpy(status_host, pin_res + sizeof(float), sizeof(int32_t));
  return PPB_OK;
}

}  // extern "C"
