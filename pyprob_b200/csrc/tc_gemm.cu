// Tensor-core building blocks exposed through the C-ABI: operand packing (K- and MN-format tile images) and
// standalone GEMM entry points over packed images, implemented on the production grouped kernel
// (tc_grouped.cuh):  C[M,N] = A[M,K] * B[N,K]^T (+bias) (relu)  and  C[M,N] = X[R,M]^T Y[R,N].
#include <string.h>

#include <vector>

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

// Descriptor-level launch of the production kernels: the standalone GEMM entry points below and ppb_tc_run_problems fill
// tcg::Problem descriptors and run them as one phase through the network's phase runners (tc_launch.cuh), so that tests and
// micro-benchmarks exercise exactly the kernels and the launch code the network uses.
tcg::Problem* g_dev_problems = nullptr;
int g_dev_capacity = 0;

bool k_aligned(const tcg::Operand& o) { return o.mn ? (o.row0 % 32 == 0 && o.col0 % 32 == 0) : (o.row0 % 128 == 0 && o.col0 % 32 == 0); }

// Every descriptor of the phase against what the kernels implement; nothing is uploaded or launched when one fails
int check_problems(const tcg::Problem* p, int n, int epi, int cs, bool ktab, int precision) {
  PPB_CHECK_ARG(p && n > 0, "no problems");
  PPB_CHECK_ARG(epi >= 0 && epi <= 2, "epilogue must be 0 (fp32 store), 1 (fp32 red.add) or 2 (tile images)");
  PPB_CHECK_ARG(precision == PPB_PREC_TF32X3 || precision == PPB_PREC_TF32, "precision must be TF32X3 or TF32");
  PPB_CHECK_ARG(cs == 1 || cs == 2 || cs == 4 || cs == 8, "cluster size must be 1, 2, 4 or 8");
  PPB_CHECK_ARG(cs == 1 || (epi != 1 && !ktab), "the cluster form has no red.add epilogue and no chunk table");
  PPB_CHECK_ARG(!ktab || epi == 0, "the chunk table runs with epilogue 0 only");
  const bool x3 = precision == PPB_PREC_TF32X3;
  for (int i = 0; i < n; ++i) {
    const tcg::Problem& q = p[i];
    const bool img = q.o_k_hi || q.o_k_lo || q.o_mn_hi || q.o_mn_lo;
    PPB_CHECK_ARG(q.M > 0 && q.N > 0 && q.K > 0, "M, N and K must be positive");
    PPB_CHECK_ARG(q.a.hi && q.b.hi && q.a.kb > 0 && q.b.kb > 0, "operand without an image");
    PPB_CHECK_ARG(!x3 || (q.a.lo && q.b.lo), "3xTF32 needs the operand lo parts");
    PPB_CHECK_ARG(k_aligned(q.a) && k_aligned(q.b),
                  "operand offset off the layout: K-major row0 % 128, col0 % 32; MN-major row0 % 32, col0 % 32");
    PPB_CHECK_ARG(!ktab || (!q.a.mn && q.a.k_rows), "the chunk table needs a K-major A with k_rows");
    PPB_CHECK_ARG(ktab || q.a.mn || !q.a.k_rows, "a K-major k_rows is read by the chunk table only");
    PPB_CHECK_ARG(q.b.mn || !q.b.k_rows, "a K-major B has no chunk table");
    PPB_CHECK_ARG((q.flags & ~(tcg::kRelu | tcg::kMaskImg | tcg::kZeroInvalid)) == 0, "unknown flags");
    PPB_CHECK_ARG(q.k_splits <= 1 || cs == 1, "the cluster form splits the reduction itself (k_splits must be 1)");
    PPB_CHECK_ARG(q.k_splits <= 1 || (epi == 1 && !q.bias && (q.flags & (tcg::kRelu | tcg::kMaskImg | tcg::kZeroInvalid)) == 0),
                  "k_splits > 1 adds partial sums: epilogue 1 without bias, ReLU, mask or zero-invalid rows");
    PPB_CHECK_ARG(epi == 2 || q.c, "epilogues 0 and 1 need c");
    PPB_CHECK_ARG(epi != 2 || q.c || q.o_k_hi || q.o_mn_hi, "epilogue 2 without any output");
    PPB_CHECK_ARG(!q.c || q.ldc >= q.N, "ldc < N");
    PPB_CHECK_ARG(epi == 2 || (!img && !(q.flags & tcg::kMaskImg)), "images and the mask need epilogue 2");
    PPB_CHECK_ARG(!q.o_k_hi == !q.o_k_lo && !q.o_mn_hi == !q.o_mn_lo, "an output image needs both its hi and lo parts");
    PPB_CHECK_ARG(!(q.flags & tcg::kMaskImg) || q.mask_hi, "kMaskImg without a mask image");
    PPB_CHECK_ARG(!(img || (q.flags & tcg::kMaskImg)) || (q.o_kb > 0 && q.o_row0 % 128 == 0 && q.o_col0 % 32 == 0),
                  "output image geometry off the layout: o_kb > 0, o_row0 % 128, o_col0 % 32");
  }
  return PPB_OK;
}

// Uploads n problems (tile bookkeeping filled in here) and runs them as one phase: cs = 1 the grouped or persistent form
// (launched without PDL: the benchmarks time these launches as such), the chunk-table form when ktab, else the cluster split-K
// form over cs CTAs
int run_problems(const tcg::Problem* hp, int n, int epi, int cs, bool ktab, int precision, cudaStream_t st) {
  int rc = check_problems(hp, n, epi, cs, ktab, precision);
  if (rc) return rc;
  std::vector<tcg::Problem> probs(hp, hp + n);
  gemm::Phase ph;
  for (tcg::Problem& q : probs) phase_add(ph, q);
  if (n > g_dev_capacity) {
    if (g_dev_problems) PPB_CUDA(cudaFree(g_dev_problems));
    g_dev_problems = nullptr;
    g_dev_capacity = 0;
    PPB_CUDA(cudaMalloc((void**)&g_dev_problems, (size_t)n * sizeof(tcg::Problem)));
    g_dev_capacity = n;
  }
  PPB_CUDA(cudaMemcpyAsync(g_dev_problems, probs.data(), (size_t)n * sizeof(tcg::Problem), cudaMemcpyHostToDevice, st));
  if (ktab) return run_tc_phase_ktab(ph, g_dev_problems, precision, st, false);
  if (cs == 1) {
    if (epi == 0) return run_tc_phase<0>(ph, g_dev_problems, precision, st, 0.0, false);
    if (epi == 1) return run_tc_phase<1>(ph, g_dev_problems, precision, st, 0.0, false);
    return run_tc_phase<2>(ph, g_dev_problems, precision, st, 0.0, false);
  }
  if (epi == 0) return run_tc_phase_cluster<0>(cs, ph, g_dev_problems, precision, st);
  return run_tc_phase_cluster<2>(cs, ph, g_dev_problems, precision, st);
}

}  // namespace

extern "C" {

// Phase-trace buffer (64 launches x 16 slots of globaltimer stamps) for the tensor-core grouped GEMM; NULL disables.
int ppb_debug_trace(void* buf_dev) { g_trace = (unsigned long long*)buf_dev; g_trace_launch = 0; return PPB_OK; }

int64_t ppb_packed_floats(int64_t rows, int64_t K) { return img_floats(rows, K); }

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
  return run_problems(&p, 1, 0, 1, false, precision, (cudaStream_t)stream);
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
  return run_problems(&p, 1, 0, cluster_size, false, precision, (cudaStream_t)stream);
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
  return run_problems(&p, 1, 0, 1, false, precision, (cudaStream_t)stream);
}

int ppb_tc_run_problems(const void* problems_host, int n, int epi, int cluster_size, int chunk_table, int precision,
                        void* stream) {
  return run_problems((const tcg::Problem*)problems_host, n, epi, cluster_size, chunk_table != 0, precision,
                      (cudaStream_t)stream);
}

}  // extern "C"
