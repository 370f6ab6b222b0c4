// Segment-aware optimiser step on the flat parameter arena: Adam / Nesterov SGD, optionally under LARC, with the
// reference's treatment of parameter tensors whose gradient is absent from the minibatch.
//
// Reference: pyprob/nn/inference_network.py:343-355 (optim.Adam / optim.SGD(nesterov) built over self.parameters(),
// optionally wrapped in LARC) and pyprob/nn/optimizer_larc.py:74-107.  torch skips a parameter whose .grad is None —
// no moment decay, no step-count increment — and LARC leaves it alone; a "segment" here is one such parameter tensor
// (one region of the arena).  With thousands of per-address tensors the reference launches a handful of kernels per
// tensor; here the whole arena is three launches: per-segment norms (LARC only), a per-segment table (step counts,
// bias corrections, LARC ratios), and one element-wise update.  HBM-bound: 16 B read + 12 B written per parameter
// (+8 B read for the norms pass under LARC).
#include "common.cuh"

namespace {

enum { kAdam = 0, kAdamLarc = 1, kSgd = 2, kSgdLarc = 3 };
// per-segment table written by k_seg_table
struct SegEntry {
  float step_size;  // Adam: lr / (1 - b1^t); SGD: lr
  float bc2_sqrt;   // Adam: sqrt(1 - b2^t)
  float adaptive;   // LARC factor applied to (g + wd p); 1 without LARC
  int first;        // SGD: 1 on the tensor's first step (momentum buffer := gradient)
};

// float4 block i of an array of n floats; the last block may be ragged (n need not be a multiple of 4)
__device__ __forceinline__ float4 load4(const float* a, int64_t i, int64_t n) {
  if (4 * i + 4 <= n) return reinterpret_cast<const float4*>(a)[i];
  float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
  const int64_t b = 4 * i;
  if (b < n) r.x = a[b];
  if (b + 1 < n) r.y = a[b + 1];
  if (b + 2 < n) r.z = a[b + 2];
  return r;
}
__device__ __forceinline__ void store4(float* a, int64_t i, int64_t n, float4 x) {
  if (4 * i + 4 <= n) {
    reinterpret_cast<float4*>(a)[i] = x;
    return;
  }
  const int64_t b = 4 * i;
  if (b < n) a[b] = x.x;
  if (b + 1 < n) a[b + 1] = x.y;
  if (b + 2 < n) a[b + 2] = x.z;
}

__global__ void __launch_bounds__(256) k_seg_norms(const float* __restrict__ p, const float* __restrict__ g,
                                                    int64_t n, int64_t n_blocks,
                                                    const int32_t* __restrict__ seg_of_block,
                                                    const int32_t* __restrict__ present, const float* __restrict__ hyper,
                                                    float* __restrict__ norms /* [2*S] zeroed */) {
  const float gscale = hyper[PPB_HYPER_GRAD_SCALE];
  const unsigned lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t rounds = (n_blocks + stride - 1) / stride;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (int64_t r = 0; r < rounds; ++r, i += stride) {  // every lane runs every round: the shuffles below need the full warp
    int seg = -1;
    float sp = 0.f, sg = 0.f;
    if (i < n_blocks) {
      seg = seg_of_block[i];
      if (seg >= 0 && present[seg]) {
        float4 a = load4(p, i, n), b = load4(g, i, n);
        b.x *= gscale; b.y *= gscale; b.z *= gscale; b.w *= gscale;
        sp = a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
        sg = b.x * b.x + b.y * b.y + b.z * b.z + b.w * b.w;
      } else {
        seg = -1;
      }
    }
    // one atomic per warp when the whole warp sits in one segment (the common case: big weight matrices)
    const int seg0 = __shfl_sync(0xffffffffu, seg, 0);
    if (__all_sync(0xffffffffu, seg == seg0)) {
      if (seg0 >= 0) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          sp += __shfl_xor_sync(0xffffffffu, sp, o);
          sg += __shfl_xor_sync(0xffffffffu, sg, o);
        }
        if (lane == 0) {
          atomicAdd(norms + 2 * seg0, sp);
          atomicAdd(norms + 2 * seg0 + 1, sg);
        }
      }
    } else if (seg >= 0) {
      atomicAdd(norms + 2 * seg, sp);
      atomicAdd(norms + 2 * seg + 1, sg);
    }
  }
}

__global__ void k_seg_table(int n_segs, const int32_t* __restrict__ present, long long* __restrict__ steps,
                            const float* __restrict__ norms, const float* __restrict__ hyper, int kind,
                            SegEntry* __restrict__ table) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_segs || !present[k]) return;
  const float lr = hyper[PPB_HYPER_LR], wd = hyper[PPB_HYPER_WEIGHT_DECAY];
  long long t = steps[k] + 1;
  steps[k] = t;
  SegEntry e;
  e.first = (t == 1);
  if (kind == kAdam || kind == kAdamLarc) {
    float bc1;
    ppb_adam_bias_corrections(hyper, t, bc1, e.bc2_sqrt);
    e.step_size = lr / bc1;
  } else {
    e.step_size = lr;
    e.bc2_sqrt = 1.0f;
  }
  e.adaptive = 1.0f;
  if (kind == kAdamLarc || kind == kSgdLarc) {
    // optimizer_larc.py:87-99, clip mode: min(local_lr / lr, 1)
    float pn = sqrtf(norms[2 * k]), gn = sqrtf(norms[2 * k + 1]);
    float local = (pn != 0.0f && gn != 0.0f)
                      ? hyper[PPB_HYPER_LARC_TRUST] * pn / (gn + pn * wd + hyper[PPB_HYPER_LARC_EPS])
                      : hyper[PPB_HYPER_LARC_EPSILON];
    e.adaptive = fminf(local / lr, 1.0f);
  }
  table[k] = e;
}

__global__ void __launch_bounds__(256) k_seg_update(float* __restrict__ p, const float* __restrict__ g,
                                                     float* __restrict__ m, float* __restrict__ v, int64_t n,
                                                     int64_t n_blocks, const int32_t* __restrict__ seg_of_block,
                                                     const int32_t* __restrict__ present,
                                                     const SegEntry* __restrict__ table,
                                                     const float* __restrict__ hyper, int kind) {
  const float b1 = hyper[PPB_HYPER_BETA1], b2 = hyper[PPB_HYPER_BETA2], eps = hyper[PPB_HYPER_EPS];
  const float wd = hyper[PPB_HYPER_WEIGHT_DECAY], gscale = hyper[PPB_HYPER_GRAD_SCALE];
  const float momentum = hyper[PPB_HYPER_MOMENTUM];
  const bool larc = kind == kAdamLarc || kind == kSgdLarc;
  const bool adam = kind == kAdam || kind == kAdamLarc;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_blocks; i += (int64_t)gridDim.x * blockDim.x) {
    const int seg = seg_of_block[i];
    if (seg < 0 || !present[seg]) continue;
    const SegEntry e = table[seg];
    float4 pp = load4(p, i, n), gg = load4(g, i, n), mm = load4(m, i, n);
    float pa[4] = {pp.x, pp.y, pp.z, pp.w}, ga[4] = {gg.x, gg.y, gg.z, gg.w}, ma[4] = {mm.x, mm.y, mm.z, mm.w};
    if (adam) {
      float4 vv = load4(v, i, n);
      float va[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (larc) {
          // LARC folds the weight decay into the gradient, scales it, and runs the wrapped optimiser with wd = 0
          float gr = __fmul_rn(__fmaf_rn(ga[j], gscale, __fmul_rn(wd, pa[j])), e.adaptive);
          ppb_adam_update(pa[j], gr, ma[j], va[j], b1, b2, eps, 0.0f, 1.0f, e.step_size, e.bc2_sqrt);
        } else {
          ppb_adam_update(pa[j], ga[j], ma[j], va[j], b1, b2, eps, wd, gscale, e.step_size, e.bc2_sqrt);
        }
      }
      store4(v, i, n, make_float4(va[0], va[1], va[2], va[3]));
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float gr = __fmaf_rn(ga[j], gscale, __fmul_rn(wd, pa[j]));
        if (larc) gr = __fmul_rn(gr, e.adaptive);
        // torch.optim.SGD, dampening 0, nesterov: buf = g (first step) | momentum*buf + g; p -= lr*(g + momentum*buf)
        ma[j] = e.first ? gr : __fmaf_rn(momentum, ma[j], gr);
        pa[j] = __fsub_rn(pa[j], __fmul_rn(e.step_size, __fmaf_rn(momentum, ma[j], gr)));
      }
    }
    store4(p, i, n, make_float4(pa[0], pa[1], pa[2], pa[3]));
    store4(m, i, n, make_float4(ma[0], ma[1], ma[2], ma[3]));
  }
}

}  // namespace

extern "C" {

int64_t ppb_optimizer_scratch_bytes(int32_t n_segs) {
  // [2*S] float norms, then S SegEntry records (16 B each)
  return n_segs <= 0 ? 0 : (int64_t)((2 * (int64_t)n_segs * 4 + 15) / 16 * 16 + (int64_t)n_segs * (int64_t)sizeof(SegEntry));
}

int ppb_optimizer_step_segmented(float* arena, const float* grad, float* state0, float* state1, int64_t n,
                                 const int32_t* seg_of_block_dev, int32_t n_segs, const int32_t* present_dev,
                                 int64_t* seg_steps_dev, void* scratch_dev, int64_t scratch_bytes, int kind,
                                 const float* hyper_dev, void* stream) {
  PPB_CHECK_ARG(arena && grad && state0 && seg_of_block_dev && present_dev && seg_steps_dev && scratch_dev && hyper_dev,
                "null argument");
  PPB_CHECK_ARG(n > 0 && n_segs > 0, "empty arena");
  PPB_CHECK_ARG(kind >= kAdam && kind <= kSgdLarc, "unknown optimiser kind");
  PPB_CHECK_ARG(kind >= kSgd || state1 != nullptr, "Adam needs the second-moment arena");
  PPB_CHECK_ARG(scratch_bytes >= ppb_optimizer_scratch_bytes(n_segs), "scratch too small");
  static_assert(sizeof(SegEntry) == 16, "SegEntry layout");
  cudaStream_t st = (cudaStream_t)stream;
  float* norms = (float*)scratch_dev;
  SegEntry* table = (SegEntry*)((char*)scratch_dev + (2 * (int64_t)n_segs * 4 + 15) / 16 * 16);
  const int64_t n_blocks = (n + 3) >> 2;
  const bool larc = kind == kAdamLarc || kind == kSgdLarc;
  if (larc) {
    PPB_CUDA(cudaMemsetAsync(norms, 0, 2 * (size_t)n_segs * sizeof(float), st));
    k_seg_norms<<<ppb_grid_for(n_blocks, 256, 2), 256, 0, st>>>(arena, grad, n, n_blocks, seg_of_block_dev, present_dev,
                                                              hyper_dev, norms);
    PPB_LAUNCH_CHECK();
  }
  k_seg_table<<<(n_segs + 127) / 128, 128, 0, st>>>(n_segs, present_dev, (long long*)seg_steps_dev, norms, hyper_dev, kind,
                                                    table);
  PPB_LAUNCH_CHECK();
  k_seg_update<<<ppb_grid_for(n_blocks, 256, 2), 256, 0, st>>>(arena, grad, state0, state1, n, n_blocks, seg_of_block_dev,
                                                             present_dev, table, hyper_dev, kind);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

}  // extern "C"
