// Data-parallel optimiser step fused with its collective, over NVLink peer memory (see include/pyprob_b200.h).
//
//   barrier A | reduce-scatter (peer loads, fixed rank order) | Adam on the local 1/world slice |
//   all-gather of the new parameters (peer stores) | barrier B            -- one kernel, graph-capturable.
//
// Reference semantics: pyprob/nn/inference_network.py:296-333 (gradients summed over ranks, divided by the world
// size) followed by optimizer.step() (:496).  The reference sends one message per parameter tensor through
// dist.all_reduce; here every element crosses NVLink twice (once as a gradient into its owner, once as a
// parameter out of it) and the optimiser state of an element is only ever touched on its owner.
#include <string.h>

#include "common.cuh"

namespace {

constexpr int kMaxWorld = 16;
constexpr int kFlagB = 16;       // barrier-B words start here
constexpr int kFlagEpoch = 32;   // launches completed by this rank
constexpr int kFlagDone = 33;    // blocks of the running launch that finished their slice
constexpr int kFlagTimeout = 34; // set if a barrier wait gave up
constexpr int kFlagRvEpoch = 35; // rendezvous launches completed by this rank (ppb_dp_rendezvous)
constexpr int kFlagTrace = 40;   // low 32 bits of %globaltimer at: kernel start, after barrier A, slice done, after barrier B
constexpr int kFlagAccum = 44;   // running sums (ns, low 32 bits) of the three phase durations, then the launch count
constexpr int kFlagRv = 48;      // rendezvous words, one per peer rank (kMaxWorld of them); block needs flag_off + 256 bytes
constexpr unsigned long long kSpinLimitNs = 4000000000ull;

struct Peers {
  float* param[kMaxWorld];
  float* grad[kMaxWorld];
  uint32_t* flags[kMaxWorld];
};

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float4 ld_peer4(const float* p) {
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ float ld_peer1(const float* p) {
  float v;
  asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_peer4(float* p, float4 v) {
  asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
__device__ __forceinline__ void st_peer1(float* p, float v) {
  asm volatile("st.relaxed.sys.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
__device__ __forceinline__ unsigned long long now_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// wait until flag word >= epoch (wrap-safe); gives up after kSpinLimitNs so that a missing rank cannot wedge the GPU
__device__ __forceinline__ void wait_flag(const uint32_t* p, uint32_t epoch, uint32_t* timeout_word) {
  unsigned long long t0 = now_ns();
  while ((int32_t)(ld_acquire_sys(p) - epoch) < 0) {
    if (now_ns() - t0 > kSpinLimitNs) {
      *timeout_word = 1u;
      break;
    }
  }
}

__global__ void __launch_bounds__(256) k_dp_adam(Peers P, int world, int rank, float* __restrict__ m,
                                                  float* __restrict__ v, int64_t n, int n_extra,
                                                  const float* __restrict__ hyper, long long* __restrict__ step_ctr,
                                                  float* __restrict__ bc_out) {
  uint32_t* my = P.flags[rank];
  __shared__ uint32_t s_epoch;
  __shared__ float s_bc[2];
  __shared__ int s_last;
  if (threadIdx.x == 0) {
    s_epoch = my[kFlagEpoch] + 1u;  // written only by the last block of the previous launch
    ppb_adam_bias_corrections(hyper, *step_ctr + 1, s_bc[0], s_bc[1]);
  }
  __syncthreads();
  const uint32_t epoch = s_epoch;
  if (blockIdx.x == 0 && threadIdx.x == 0) my[kFlagTrace] = (uint32_t)now_ns();

  // ---- barrier A: every rank's backward pass is complete (kernel boundary) and its gradient may be read;
  //      nobody is still reading the parameters of the previous step
  if (blockIdx.x == 0 && threadIdx.x < world) st_release_sys(P.flags[threadIdx.x] + rank, epoch);
  if (threadIdx.x < world) wait_flag(my + threadIdx.x, epoch, my + kFlagTimeout);
  __syncthreads();
  if (blockIdx.x == 0 && threadIdx.x == 0) my[kFlagTrace + 1] = (uint32_t)now_ns();

  const float lr = hyper[PPB_HYPER_LR], b1 = hyper[PPB_HYPER_BETA1], b2 = hyper[PPB_HYPER_BETA2];
  const float eps = hyper[PPB_HYPER_EPS], wd = hyper[PPB_HYPER_WEIGHT_DECAY], gscale = hyper[PPB_HYPER_GRAD_SCALE];
  const float step = lr / s_bc[0], bc2_sqrt = s_bc[1];

  // ---- this rank's slice: [lo, hi), boundaries on float4
  int64_t per = ((n + (int64_t)world * 4 - 1) / ((int64_t)world * 4)) * 4;
  int64_t lo = (int64_t)rank * per, hi = lo + per;
  if (lo > n) lo = n;
  if (hi > n) hi = n;
  float* p_own = P.param[rank];
  for (int64_t i = lo + 4 * ((int64_t)blockIdx.x * blockDim.x + threadIdx.x); i < hi;
       i += 4 * (int64_t)gridDim.x * blockDim.x) {
    if (i + 4 <= hi) {
      float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
      for (int r = 0; r < world; ++r) {  // fixed order: the sum does not depend on which rank owns the element
        float4 x = ld_peer4(P.grad[r] + i);
        g.x += x.x; g.y += x.y; g.z += x.z; g.w += x.w;
      }
      float4 pp = *reinterpret_cast<const float4*>(p_own + i);
      float4 mm = *reinterpret_cast<const float4*>(m + i), vv = *reinterpret_cast<const float4*>(v + i);
      ppb_adam_update(pp.x, g.x, mm.x, vv.x, b1, b2, eps, wd, gscale, step, bc2_sqrt);
      ppb_adam_update(pp.y, g.y, mm.y, vv.y, b1, b2, eps, wd, gscale, step, bc2_sqrt);
      ppb_adam_update(pp.z, g.z, mm.z, vv.z, b1, b2, eps, wd, gscale, step, bc2_sqrt);
      ppb_adam_update(pp.w, g.w, mm.w, vv.w, b1, b2, eps, wd, gscale, step, bc2_sqrt);
      *reinterpret_cast<float4*>(m + i) = mm;
      *reinterpret_cast<float4*>(v + i) = vv;
#pragma unroll 4
      for (int r = 0; r < world; ++r) st_peer4(P.param[r] + i, pp);
    } else {
      for (int64_t j = i; j < hi; ++j) {
        float g = 0.f;
        for (int r = 0; r < world; ++r) g += ld_peer1(P.grad[r] + j);
        float pj = p_own[j], mj = m[j], vj = v[j];
        ppb_adam_update(pj, g, mj, vj, b1, b2, eps, wd, gscale, step, bc2_sqrt);
        m[j] = mj; v[j] = vj;
        for (int r = 0; r < world; ++r) st_peer1(P.param[r] + j, pj);
      }
    }
  }
  // piggy-backed scalars (loss): summed by rank 0, handed back to everyone's gradient tail
  if (rank == 0 && blockIdx.x == 0 && (int)threadIdx.x < n_extra) {
    float s = 0.f;
    for (int r = 0; r < world; ++r) s += ld_peer1(P.grad[r] + n + threadIdx.x);
    for (int r = 0; r < world; ++r) st_peer1(P.grad[r] + n + threadIdx.x, s);
  }

  // ---- barrier B: all of this rank's peer stores are performed before any rank starts its next forward pass
  __threadfence_system();
  __syncthreads();
  if (blockIdx.x == 0 && threadIdx.x == 0) my[kFlagTrace + 2] = (uint32_t)now_ns();
  if (threadIdx.x == 0) s_last = (atomicAdd(my + kFlagDone, 1u) == gridDim.x - 1) ? 1 : 0;
  __syncthreads();
  if (s_last) {
    __threadfence_system();
    if (threadIdx.x < world) {
      st_release_sys(P.flags[threadIdx.x] + kFlagB + rank, epoch);
      wait_flag(my + kFlagB + threadIdx.x, epoch, my + kFlagTimeout);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      my[kFlagTrace + 3] = (uint32_t)now_ns();
      my[kFlagAccum + 0] += my[kFlagTrace + 1] - my[kFlagTrace + 0];
      my[kFlagAccum + 1] += my[kFlagTrace + 2] - my[kFlagTrace + 1];
      my[kFlagAccum + 2] += my[kFlagTrace + 3] - my[kFlagTrace + 2];
      my[kFlagAccum + 3] += 1u;
      my[kFlagDone] = 0u;
      my[kFlagEpoch] = epoch;
      *step_ctr = *step_ctr + 1;
      bc_out[0] = s_bc[0];   // byte 8 of the Adam state block (include/pyprob_b200.h); byte 12 is left untouched
    }
  }
}

// cross-rank rendezvous on the stream: returns once every rank's stream has reached its matching call
__global__ void k_dp_rendezvous(Peers P, int world, int rank) {
  uint32_t* my = P.flags[rank];
  __shared__ uint32_t s_epoch;
  if (threadIdx.x == 0) s_epoch = my[kFlagRvEpoch] + 1u;
  __syncthreads();
  const uint32_t epoch = s_epoch;
  if ((int)threadIdx.x < world) {
    st_release_sys(P.flags[threadIdx.x] + kFlagRv + rank, epoch);
    wait_flag(my + kFlagRv + threadIdx.x, epoch, my + kFlagTimeout);
  }
  __syncthreads();
  if (threadIdx.x == 0) my[kFlagRvEpoch] = epoch;
}

}  // namespace

extern "C" {

int ppb_dp_rendezvous(int world, int rank, void* const* peer_blocks, int64_t flag_off, void* stream) {
  PPB_CHECK_ARG(world >= 1 && world <= kMaxWorld && rank >= 0 && rank < world && peer_blocks, "bad world/rank");
  Peers P;
  memset(&P, 0, sizeof(P));
  for (int r = 0; r < world; ++r) {
    PPB_CHECK_ARG(peer_blocks[r] != nullptr, "null peer block");
    P.flags[r] = (uint32_t*)((char*)peer_blocks[r] + flag_off);
  }
  k_dp_rendezvous<<<1, 32, 0, (cudaStream_t)stream>>>(P, world, rank);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int ppb_dp_alloc(int64_t bytes, void** ptr_out, void* ipc_handle_out) {
  PPB_CHECK_ARG(bytes > 0 && ptr_out && ipc_handle_out, "bad arguments");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  void* p = nullptr;
  PPB_CUDA(cudaMalloc(&p, (size_t)bytes));
  PPB_CUDA(cudaMemset(p, 0, (size_t)bytes));
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) {
    cudaFree(p);
    ppb_set_error("ppb_dp_alloc: cudaIpcGetMemHandle: %s", cudaGetErrorString(e));
    return (int)e;
  }
  memcpy(ipc_handle_out, &h, sizeof(h));
  *ptr_out = p;
  return PPB_OK;
}

int ppb_dp_open(const void* ipc_handle, void** ptr_out) {
  PPB_CHECK_ARG(ipc_handle && ptr_out, "bad arguments");
  cudaIpcMemHandle_t h;
  memcpy(&h, ipc_handle, sizeof(h));
  PPB_CUDA(cudaIpcOpenMemHandle(ptr_out, h, cudaIpcMemLazyEnablePeerAccess));
  return PPB_OK;
}

int ppb_dp_close(void* mapped_ptr) {
  PPB_CHECK_ARG(mapped_ptr, "bad arguments");
  PPB_CUDA(cudaIpcCloseMemHandle(mapped_ptr));
  return PPB_OK;
}

int ppb_dp_free(void* ptr) {
  PPB_CHECK_ARG(ptr, "bad arguments");
  PPB_CUDA(cudaFree(ptr));
  return PPB_OK;
}

int ppb_dp_adam_step(int world, int rank, void* const* peer_blocks, int64_t param_off, int64_t grad_off,
                     int64_t flag_off, float* exp_avg, float* exp_avg_sq, int64_t n, int64_t n_extra,
                     const float* hyper_dev, void* state_dev, void* stream) {
  PPB_CHECK_ARG(world >= 1 && world <= kMaxWorld && rank >= 0 && rank < world && peer_blocks, "bad world/rank");
  PPB_CHECK_ARG(exp_avg && exp_avg_sq && hyper_dev && state_dev && n > 0 && n_extra >= 0 && n_extra <= 32,
                "bad arguments");
  PPB_CHECK_ARG(((param_off | grad_off | flag_off) & 15) == 0, "offsets must be 16-byte aligned");
  Peers P;
  for (int r = 0; r < world; ++r) {
    PPB_CHECK_ARG(peer_blocks[r] != nullptr, "null peer block");
    char* base = (char*)peer_blocks[r];
    P.param[r] = (float*)(base + param_off);
    P.grad[r] = (float*)(base + grad_off);
    P.flags[r] = (uint32_t*)(base + flag_off);
  }
  int64_t per = ((n + (int64_t)world * 4 - 1) / ((int64_t)world * 4)) * 4;
  int64_t blocks = (per / 4 + 255) / 256;
  if (blocks < 1) blocks = 1;
  // one float4 per thread keeps every peer load of the slice in flight at once; blocks beyond the first wave are
  // harmless (barrier A is signalled by block 0, barrier B by whichever block finishes last)
  if (blocks > 8 * PPB_NUM_SMS) blocks = 8 * PPB_NUM_SMS;
  k_dp_adam<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(P, world, rank, exp_avg, exp_avg_sq, n, (int)n_extra,
                                                           hyper_dev, (long long*)state_dev,
                                                           (float*)((char*)state_dev + 8));
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

}  // extern "C"
