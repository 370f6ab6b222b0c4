// Launch code of the tensor-core kernels, shared by the networks (net.cu) and the standalone GEMM entry points (tc_gemm.cu):
// the shared-memory opt-in, one counted launch, the runtime-to-template dispatch and the phase runners built on them.  Which
// kernel form a phase runs (cluster size, fused or not) is decided by the callers.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "tc_grouped.cuh"
#include "tc_persist.cuh"
#include "tc_cluster.cuh"

extern unsigned long long* g_trace;  // phase-trace buffer of ppb_debug_trace (tc_gemm.cu), 16 slots per launch
extern int g_trace_launch;

// Kernel-level profiling (ppb_prof_enable / ppb_prof_read, net.cu): prof_begin records a start event on st when profiling is
// on and the launch is profiled (flops > 0), else leaves e0 null; prof_end books the span and its FLOPs after a non-null e0.
int prof_begin(double flops, cudaStream_t st, cudaEvent_t& e0);
int prof_end(cudaEvent_t e0, cudaStream_t st, double flops);

namespace {

// Raises a kernel's dynamic shared-memory limit to `bytes`, once per kernel: eager launches pay no host call after the first
template <auto Kernel>
int smem_opt_in(size_t bytes) {
  static bool done = false;
  if (!done) {
    PPB_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    done = true;
  }
  return PPB_OK;
}

// The next launch's slot of the phase-trace buffer, or null when tracing is off or the buffer is full
inline unsigned long long* trace_slot() {
  if (!g_trace || g_trace_launch >= 256) return nullptr;
  return g_trace + 16 * g_trace_launch++;
}

// One counted launch of a tensor-core kernel (tcg::kThreads per CTA) with `smem` bytes of dynamic shared memory, a
// (cluster, 1, 1) thread-block cluster when cluster > 1 and the PDL attribute when pdl (common.cuh: ppb_launch)
template <auto Kernel, typename... Args>
int tc_launch(int grid, size_t smem, int cluster, bool pdl, cudaStream_t st, Args... args) {
  int rc = smem_opt_in<Kernel>(smem);
  if (rc) return rc;
  PPB_CUDA(ppb_launch(Kernel, dim3((unsigned)grid), dim3(tcg::kThreads), smem, st, pdl, cluster, args...));
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

// Runtime value -> template argument: f(std::integral_constant<int, V>()) for the first V of the list with v <= V, the last
// V when there is none
template <int V, int... Vs, typename F>
int pick(int v, F&& f) {
  if constexpr (sizeof...(Vs) == 0) return f(std::integral_constant<int, V>());
  else return v <= V ? f(std::integral_constant<int, V>()) : pick<Vs...>(v, f);
}
// precision -> the X3 template argument (3xTF32 or 1xTF32)
template <typename F>
int with_x3(int precision, F&& f) {
  return precision == PPB_PREC_TF32X3 ? f(std::true_type()) : f(std::false_type());
}

// launch() inside a profiling span of `prof_flops` FLOPs (0: not profiled)
template <typename F>
int profiled(double prof_flops, cudaStream_t st, F&& launch) {
  cudaEvent_t e0;
  int rc = prof_begin(prof_flops, st, e0);
  if (rc) return rc;
  rc = launch();
  if (rc) return rc;
  return prof_end(e0, st, prof_flops);
}

// A phase of tcg::k_grouped with epilogue EPI: 0 = fp32 store, 1 = fp32 reduction (weight gradients / split-K), 2 = tile images
// (+ fp32).  With more tiles than SMs it runs the persistent form (tc_persist.cuh), which overlaps every tile's epilogue with
// the next tile's mainloop, unless the launch is traced.
template <int EPI>
int run_tc_phase(const gemm::Phase& ph, const tcg::Problem* dev, int precision, cudaStream_t st, double prof_flops = 0.0,
                 bool pdl = true) {
  if (ph.count == 0) return PPB_OK;
  return profiled(prof_flops, st, [&] {
    unsigned long long* tr = trace_slot();
    return with_x3(precision, [&](auto x3) {
      if (ppb_persistent_enabled() && ph.tiles > PPB_NUM_SMS && tr == nullptr)
        return tc_launch<tcp::k_grouped_persistent<x3, EPI>>(PPB_NUM_SMS, tcp::smem_bytes(), 1, pdl, st, dev + ph.first,
                                                             ph.count, ph.tiles);
      return tc_launch<tcg::k_grouped<x3, EPI>>(ph.tiles, tcg::smem_bytes(), 1, pdl, st, dev + ph.first, ph.count, tr);
    });
  });
}

// A phase of tcc::k_cluster: the reduction of every output tile split over a cluster of cs CTAs (2, 4 or 8), epilogue EPI
// (tc_cluster.cuh; 3 and 4 run the row routine re in the reduce phase)
template <int EPI, typename RE = tcc::NoRowEpi>
int run_tc_phase_cluster(int cs, const gemm::Phase& ph, const tcg::Problem* dev, int precision, cudaStream_t st,
                         const RE& re = RE()) {
  return with_x3(precision, [&](auto x3) {
    return pick<2, 4, 8>(cs, [&](auto c) {
      return tc_launch<tcc::k_cluster<x3, c, EPI, RE>>(ph.tiles * c, tcc::smem_bytes(), c, true, st, dev + ph.first, ph.count,
                                                       trace_slot(), re);
    });
  });
}

}  // namespace
