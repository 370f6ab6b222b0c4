// Tensor-core building blocks exposed through the C-ABI: operand packing (K- and MN-format tile images) and
// standalone GEMM entry points over packed images, implemented on the production grouped kernel
// (tc_grouped.cuh):  C[M,N] = A[M,K] * B[N,K]^T (+bias) (relu)  and  C[M,N] = X[R,M]^T Y[R,N].
#include <string.h>

#include "common.cuh"
#include "tc.cuh"
#include "tc_launch.cuh"

namespace {

using namespace tc;

// ---- pack: row-major fp32 -> swizzled tile image(s) ------------------------------------------------
template <bool MN>
__global__ void __launch_bounds__(256) k_pack(const float* __restrict__ X, int64_t rows, int64_t K, int64_t ldx,
                                               float* __restrict__ hi, float* __restrict__ lo) {
  const int64_t KB = (K + kTileK - 1) / kTileK;
  const int64_t RT = (rows + kTileRows - 1) / kTileRows;
  const int64_t chunks = RT * kTileRows * KB * 8;  // 16-byte chunks in the padded image
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < chunks; q += (int64_t)gridDim.x * blockDim.x) {
    int64_t c = q & 7, t = q >> 3;
    int64_t row = t / KB, kb = t % KB;  // consecutive threads walk along K of one row: coalesced reads
    int64_t k0 = kb * kTileK + c * 4;
    float x[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) x[j] = (row < rows && k0 + j < K) ? __ldg(X + row * ldx + k0 + j) : 0.0f;
    float h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) split_tf32(x[j], h[j], l[j]);
    int64_t off = MN ? packed_offset_mn(row, k0, KB) : packed_offset(row, k0, KB);
    *reinterpret_cast<float4*>(hi + off) = make_float4(h[0], h[1], h[2], h[3]);
    if (lo) *reinterpret_cast<float4*>(lo + off) = make_float4(l[0], l[1], l[2], l[3]);
  }
}

}  // namespace

unsigned long long* g_trace = nullptr;  // optional phase-trace buffer for the grouped tensor-core GEMM (ppb_debug_trace)
int g_trace_launch = 0;

namespace {

// one-problem launch of the production kernels — the standalone GEMM entry points below are thin wrappers around the
// network's phase runners (tc_launch.cuh), so that tests and micro-benchmarks exercise exactly the kernels and the launch code
// the network uses
tcg::Problem* g_dev_problem = nullptr;

// cs = 1: grouped or persistent form, launched without PDL (the benchmarks time these launches as such); else the cluster
// split-K form over cs CTAs
int run_single(tcg::Problem& hp, int precision, int cs, cudaStream_t st) {
  hp.tiles_m = (hp.M + 127) / 128; hp.tiles_n = (hp.N + 127) / 128; hp.k_splits = 1;
  if (!g_dev_problem) PPB_CUDA(cudaMalloc((void**)&g_dev_problem, sizeof(tcg::Problem)));
  PPB_CUDA(cudaMemcpyAsync(g_dev_problem, &hp, sizeof(hp), cudaMemcpyHostToDevice, st));
  gemm::Phase ph;
  ph.count = 1;
  ph.tiles = hp.tiles_m * hp.tiles_n;
  if (cs == 1) return run_tc_phase<0>(ph, g_dev_problem, precision, st, 0.0, false);
  return run_tc_phase_cluster<0>(cs, ph, g_dev_problem, precision, st);
}

}  // namespace

extern "C" {

// Phase-trace buffer (64 launches x 16 slots of globaltimer stamps) for the tensor-core grouped GEMM; NULL disables.
int ppb_debug_trace(void* buf_dev) { g_trace = (unsigned long long*)buf_dev; g_trace_launch = 0; return PPB_OK; }

int64_t ppb_packed_floats(int64_t rows, int64_t K) {
  int64_t RT = (rows + tc::kTileRows - 1) / tc::kTileRows, KB = (K + tc::kTileK - 1) / tc::kTileK;
  return RT * KB * tc::kTileFloats;
}

int ppb_pack_tf32(const float* X, int64_t rows, int64_t K, int64_t ldx, float* hi_out, float* lo_out, void* stream) {
  PPB_CHECK_ARG(X && hi_out && rows > 0 && K > 0 && ldx >= K, "bad arguments");
  int64_t chunks = ppb_packed_floats(rows, K) / 4;
  k_pack<false><<<ppb_grid_for(chunks, 256, 1), 256, 0, (cudaStream_t)stream>>>(X, rows, K, ldx, hi_out, lo_out);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int ppb_pack_tf32_mn(const float* X, int64_t rows, int64_t K, int64_t ldx, float* hi_out, float* lo_out, void* stream) {
  PPB_CHECK_ARG(X && hi_out && rows > 0 && K > 0 && ldx >= K, "bad arguments");
  int64_t chunks = ppb_packed_floats(rows, K) / 4;
  k_pack<true><<<ppb_grid_for(chunks, 256, 1), 256, 0, (cudaStream_t)stream>>>(X, rows, K, ldx, hi_out, lo_out);
  PPB_LAUNCH_CHECK();
  return PPB_OK;
}

int ppb_gemm_packed(const float* A_hi, const float* A_lo, const float* B_hi, const float* B_lo, float* C, int64_t M,
                    int64_t N, int64_t K, int64_t ldc, const float* bias, int relu, int precision, void* stream) {
  PPB_CHECK_ARG(A_hi && B_hi && C && M > 0 && N > 0 && K > 0 && ldc >= N, "bad arguments");
  PPB_CHECK_ARG(precision == PPB_PREC_TF32X3 || precision == PPB_PREC_TF32, "precision must be TF32X3 or TF32");
  PPB_CHECK_ARG(precision == PPB_PREC_TF32 || (A_lo && B_lo), "3xTF32 needs the lo images");
  tcg::Problem p;
  memset(&p, 0, sizeof(p));
  const int kb = (int)((K + 31) / 32);
  p.a.hi = A_hi; p.a.lo = A_lo; p.a.kb = kb;
  p.b.hi = B_hi; p.b.lo = B_lo; p.b.kb = kb;
  p.M = (int)M; p.N = (int)N; p.K = (int)K;
  p.c = C; p.ldc = ldc; p.bias = bias; p.flags = relu ? tcg::kRelu : 0;
  return run_single(p, precision, 1, (cudaStream_t)stream);
}

// Same GEMM with the reduction split over a thread-block cluster of `cluster_size` CTAs per output tile (2, 4 or 8):
// partial tiles are combined through distributed shared memory (tc_cluster.cuh) — the kernel the network uses for its
// few-row, deep-K GEMMs (LSTM recurrence, BPTT, proposal heads at small minibatches).
int ppb_gemm_packed_cluster(const float* A_hi, const float* A_lo, const float* B_hi, const float* B_lo, float* C, int64_t M,
                            int64_t N, int64_t K, int64_t ldc, const float* bias, int relu, int precision, int cluster_size,
                            void* stream) {
  PPB_CHECK_ARG(A_hi && B_hi && C && M > 0 && N > 0 && K > 0 && ldc >= N, "bad arguments");
  PPB_CHECK_ARG(precision == PPB_PREC_TF32X3 || precision == PPB_PREC_TF32, "precision must be TF32X3 or TF32");
  PPB_CHECK_ARG(precision == PPB_PREC_TF32 || (A_lo && B_lo), "3xTF32 needs the lo images");
  PPB_CHECK_ARG(cluster_size == 2 || cluster_size == 4 || cluster_size == 8, "cluster size must be 2, 4 or 8");
  tcg::Problem p;
  memset(&p, 0, sizeof(p));
  const int kb = (int)((K + 31) / 32);
  p.a.hi = A_hi; p.a.lo = A_lo; p.a.kb = kb;
  p.b.hi = B_hi; p.b.lo = B_lo; p.b.kb = kb;
  p.M = (int)M; p.N = (int)N; p.K = (int)K;
  p.c = C; p.ldc = ldc; p.bias = bias; p.flags = relu ? tcg::kRelu : 0;
  return run_single(p, precision, cluster_size, (cudaStream_t)stream);
}

int ppb_gemm_packed_tn(const float* X_hi, const float* X_lo, const float* Y_hi, const float* Y_lo, float* C, int64_t M,
                       int64_t N, int64_t R, int64_t ldc, int precision, void* stream) {
  PPB_CHECK_ARG(X_hi && Y_hi && C && M > 0 && N > 0 && R > 0 && ldc >= N, "bad arguments");
  PPB_CHECK_ARG(precision == PPB_PREC_TF32X3 || precision == PPB_PREC_TF32, "precision must be TF32X3 or TF32");
  PPB_CHECK_ARG(precision == PPB_PREC_TF32 || (X_lo && Y_lo), "3xTF32 needs the lo images");
  tcg::Problem p;
  memset(&p, 0, sizeof(p));
  p.a.hi = X_hi; p.a.lo = X_lo; p.a.kb = (int)((M + 31) / 32); p.a.mn = 1;
  p.b.hi = Y_hi; p.b.lo = Y_lo; p.b.kb = (int)((N + 31) / 32); p.b.mn = 1;
  p.M = (int)M; p.N = (int)N; p.K = (int)((R + 31) / 32 * 32);  // image rows beyond R are zero padding
  p.c = C; p.ldc = ldc;
  return run_single(p, precision, 1, (cudaStream_t)stream);
}

}  // extern "C"
