// Generic fp32 Dense kernels for ARBITRARY layer shapes (hidden_size=(10,2,10), the GLM-shaped
// hidden_size=(), ragged gene counts ...).  64x64x16 register-tiled CUDA-core GEMM with optional
// transposes, row gather on A, split-K (atomic accumulate) and the fused output activations of
// dca/network.py:38-39,369-381.  The gene-wide layers of the flagship shape (hidden 64) run on
// the tensor-core kernels in dense_tc.cu instead; this file is the shape-general path.
#include "dca_internal.cuh"

namespace dca {
namespace {

constexpr int BM = 64, BN = 64, BK = 16, TM = 4, TN = 4;
constexpr int kThreads = (BM / TM) * (BN / TN);   // 256

__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }

__device__ __forceinline__ float softplus_f(float x) { return x > 20.f ? x : log1pf(expf(x)); }
__device__ __forceinline__ float sigmoid_f(float x) {
  return x >= 0.f ? 1.0f / (1.0f + expf(-x)) : expf(x) / (1.0f + expf(x));
}

template <typename AT, bool TA, bool TB>
__global__ void __launch_bounds__(kThreads)
gemm_kernel(const AT* __restrict__ A, int64_t lda, const int32_t* __restrict__ a_rows,
            const float* __restrict__ B, int64_t ldb, float* C, int64_t ldc, int M, int N, int K,
            const float* __restrict__ bias, const float* __restrict__ row_scale, int epilogue, int k_per_split) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kbeg = blockIdx.z * k_per_split;
  const int kend = min(K, kbeg + k_per_split);
  const int ty = tid / (BN / TN), tx = tid % (BN / TN);
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int k0 = kbeg; k0 < kend; k0 += BK) {
    // ---- stage A tile (BM x BK) into As[k][m]
#pragma unroll
    for (int i = 0; i < (BM * BK) / kThreads; ++i) {
      const int e = tid + i * kThreads;
      int m, k;
      if (TA) { m = e % BM; k = e / BM; }        // storage rows are k: consecutive threads along m (contiguous)
      else    { k = e % BK; m = e / BK; }        // storage rows are m: consecutive threads along k (contiguous)
      const int gm = m0 + m, gk = k0 + k;
      float v = 0.f;
      if (gm < M && gk < kend) {
        if (TA) { const int64_t r = a_rows ? (int64_t)a_rows[gk] : (int64_t)gk; v = to_f(A[r * lda + gm]); }
        else    { const int64_t r = a_rows ? (int64_t)a_rows[gm] : (int64_t)gm; v = to_f(A[r * lda + gk]); }
      }
      As[k][m] = v;
    }
    // ---- stage B tile (BK x BN) into Bs[k][n]
#pragma unroll
    for (int i = 0; i < (BK * BN) / kThreads; ++i) {
      const int e = tid + i * kThreads;
      int n, k;
      if (TB) { k = e % BK; n = e / BK; }        // B stored [n][k]
      else    { n = e % BN; k = e / BN; }        // B stored [k][n]
      const int gn = n0 + n, gk = k0 + k;
      float v = 0.f;
      if (gn < N && gk < kend) v = TB ? B[(int64_t)gn * ldb + gk] : B[(int64_t)gk * ldb + gn];
      Bs[k][n] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = As[k][ty * TM + i];
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = Bs[k][tx * TN + j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

  const bool split = gridDim.z > 1;
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int gm = m0 + ty * TM + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int gn = n0 + tx * TN + j;
      if (gn >= N) continue;
      float v = acc[i][j];
      float* c = C + (int64_t)gm * ldc + gn;
      if (split) { atomicAdd(c, v); continue; }
      if (bias) v += bias[gn];
      switch (epilogue) {
        case EPI_ACCUM: *c += v; break;
        case EPI_MEAN_ACT: {
          v = fminf(fmaxf(expf(v), 1e-5f), 1e6f);                  // MeanAct  dca/network.py:38
          if (row_scale) v *= row_scale[gm];                       // mean * sf dca/layers.py:85
          *c = v; break; }
        case EPI_DISP_ACT: *c = fminf(fmaxf(softplus_f(v), 1e-4f), 1e4f); break;   // DispAct dca/network.py:39
        case EPI_SIGMOID: *c = sigmoid_f(v); break;                // dca/network.py:369
        case EPI_LINEAR_SCALE: *c = row_scale ? v * row_scale[gm] : v; break;
        default: *c = v; break;
      }
    }
  }
}

}  // namespace

int gemm_generic(const GemmArgs& g, cudaStream_t s) {
  if (g.M <= 0 || g.N <= 0) return DCA_OK;
  if (g.K < 0) { set_error("gemm_generic: negative K"); return DCA_ERR_BAD_ARG; }
  int splits = g.splits < 1 ? 1 : g.splits;
  if (splits > 1 && !(g.epilogue == EPI_ACCUM)) { set_error("gemm_generic: split-K needs EPI_ACCUM"); return DCA_ERR_BAD_ARG; }
  int kps = cdiv(cdiv(g.K, splits), BK) * BK;
  if (kps <= 0) kps = BK;
  splits = g.K > 0 ? cdiv(g.K, kps) : 1;
  dim3 grid(cdiv(g.N, BN), cdiv(g.M, BM), splits), block(kThreads);
#define DCA_GEMM(AT, TA_, TB_)                                                                         \
  gemm_kernel<AT, TA_, TB_><<<grid, block, 0, s>>>((const AT*)g.A, g.lda, g.a_rows, g.B, g.ldb, g.C,   \
                                                   g.ldc, g.M, g.N, g.K, g.bias, g.row_scale, g.epilogue, kps)
  if (g.a_bf16) {
    if (g.transA) { if (g.transB) DCA_GEMM(__nv_bfloat16, true, true); else DCA_GEMM(__nv_bfloat16, true, false); }
    else          { if (g.transB) DCA_GEMM(__nv_bfloat16, false, true); else DCA_GEMM(__nv_bfloat16, false, false); }
  } else {
    if (g.transA) { if (g.transB) DCA_GEMM(float, true, true); else DCA_GEMM(float, true, false); }
    else          { if (g.transB) DCA_GEMM(float, false, true); else DCA_GEMM(float, false, false); }
  }
#undef DCA_GEMM
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

}  // namespace dca

// Stand-alone head layer entry point (generic path; dense_tc.cu overrides for qualifying shapes).
using namespace dca;
extern "C" int dca_dense_heads_fwd(const float* H, int64_t ldh, int32_t batch, int32_t K, int32_t genes,
                                   const float* w_mean, const float* b_mean, const float* w_disp,
                                   const float* b_disp, const float* w_pi, const float* b_pi,
                                   const float* row_scale, float* m_out, float* d_out, float* pi_out,
                                   int64_t ld_out, void* stream) {
  if (!H || batch <= 0 || K <= 0 || genes <= 0) { set_error("dca_dense_heads_fwd: bad argument"); return DCA_ERR_BAD_ARG; }
  cudaStream_t s = (cudaStream_t)stream;
  struct { const float* w; const float* b; float* out; int epi; const float* rs; } heads[3] = {
      {w_mean, b_mean, m_out, EPI_MEAN_ACT, row_scale},
      {w_disp, b_disp, d_out, EPI_DISP_ACT, nullptr},
      {w_pi, b_pi, pi_out, EPI_SIGMOID, nullptr}};
  for (auto& hd : heads) {
    if (!hd.w || !hd.out) continue;
    GemmArgs g{};
    g.A = H; g.lda = ldh; g.a_bf16 = 0; g.transA = 0; g.a_rows = nullptr;
    g.B = hd.w; g.ldb = genes; g.transB = 0;
    g.C = hd.out; g.ldc = ld_out; g.M = batch; g.N = genes; g.K = K;
    g.bias = hd.b; g.row_scale = hd.rs; g.epilogue = hd.epi; g.splits = 1;
    DCA_TRY(gemm_generic(g, s));
  }
  return DCA_OK;
}
