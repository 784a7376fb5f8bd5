// Internal declarations shared by the translation units of libdca_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stddef.h>
#include <atomic>
#include "../../include/dca_b200.h"

namespace dca {

// ---------------------------------------------------------------- errors / launch count
void set_error(const char* fmt, ...);
extern std::atomic<long long> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define DCA_CUDA_OK(expr)                                                              \
  do {                                                                                 \
    cudaError_t _e = (expr);                                                           \
    if (_e != cudaSuccess) {                                                           \
      ::dca::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return DCA_ERR_CUDA;                                                             \
    }                                                                                  \
  } while (0)

#define DCA_LAUNCH_CHECK()                                                             \
  do {                                                                                 \
    ::dca::count_launch();                                                             \
    cudaError_t _e = cudaGetLastError();                                               \
    if (_e != cudaSuccess) {                                                           \
      ::dca::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
      return DCA_ERR_CUDA;                                                             \
    }                                                                                  \
  } while (0)

#define DCA_TRY(expr)                \
  do {                               \
    int _s = (expr);                 \
    if (_s != DCA_OK) return _s;     \
  } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// ---------------------------------------------------------------- generic fp32 GEMM (dense_generic.cu)
enum Epilogue : int {
  EPI_STORE = 0,        // C = acc (+bias)
  EPI_ACCUM = 1,        // C += acc             (atomic when split-K)
  EPI_MEAN_ACT = 2,     // C = clip(exp(acc+bias),1e-5,1e6) [* row_scale]
  EPI_DISP_ACT = 3,     // C = clip(softplus(acc+bias),1e-4,1e4)
  EPI_SIGMOID = 4,      // C = sigmoid(acc+bias)
  EPI_LINEAR_SCALE = 5  // C = (acc+bias) [* row_scale]     ('normal' type: linear mean head, dca/network.py:147-150)
};

struct GemmArgs {
  const void* A; int64_t lda; int a_bf16; int transA;   // A(m,k) = transA ? A[k*lda+m] : A[m*lda+k]
  const int32_t* a_rows;                                 // optional gather on A's STORAGE rows
  const float* B; int64_t ldb; int transB;              // B(k,n) = transB ? B[n*ldb+k] : B[k*ldb+n]
  float* C; int64_t ldc;
  int M, N, K;
  const float* bias;                                     // per column n (only with splits == 1)
  const float* row_scale;                                // per row m, EPI_MEAN_ACT only
  int epilogue;
  int splits;                                            // split-K factor (>1 => atomicAdd into C)
};
int gemm_generic(const GemmArgs& g, cudaStream_t s);

// ---------------------------------------------------------------- small element-wise / BN kernels (layers.cu)
int fill_rows_with_bias(float* C, int64_t ldc, int M, int N, const float* bias, cudaStream_t s);
// column statistics over rows: sum(a) and sum(a*b) (b == nullptr -> sum(a*a)); results in double
int col_sums(const float* a, const float* b, int64_t ld, int M, int N, double* out_sum, double* out_prod,
             double* scratch, cudaStream_t s);
int col_sums_scratch_elems(int M, int N);
int bn_train_finalize(const double* sum, const double* sq, int M, int N, float eps, float momentum,
                      float* mean, float* inv_std, float* moving_mean, float* moving_var, cudaStream_t s);
int bn_relu_fwd(const float* a, int64_t ld, int M, int N, const float* mean, const float* inv_std,
                const float* beta, float* xhat, float* h, __nv_bfloat16* h_bf16, cudaStream_t s);
int bn_infer_prepare(const float* moving_mean, const float* moving_var, int N, float eps,
                     float* mean, float* inv_std, cudaStream_t s);
int bias_relu_fwd(const float* a, int64_t ld, int M, int N, float* h, __nv_bfloat16* h_bf16, cudaStream_t s);
// g = dh * (h > 0), in place on dh
int relu_bwd(float* dh, const float* h, int64_t ld, int M, int N, cudaStream_t s);
// da = inv*(g - mean(g) - xhat*mean(g*xhat)); dbeta = sum(g);  sums provided in double; stat_rows: rows behind the
// sums when they cover more than the M local rows (sync_bn: global batch), 0 = M
int bn_bwd_apply(float* g_inout, const float* xhat, int64_t ld, int M, int N, const float* inv_std,
                 const double* sum_g, const double* sum_gx, float* dbeta, cudaStream_t s, int stat_rows = 0);
int col_sum_to_float(const double* sum, int N, float* out, cudaStream_t s);
int theta_prepare(const float* theta_raw, int G, float* theta, float* chain, cudaStream_t s);
int theta_grad_finish(const float* dtheta, const float* chain, int G, float scale, float* grad_out, cudaStream_t s);
int add_reg_grad(const float* w, float* g, int64_t n, float l1, float l2, cudaStream_t s);
int reg_penalty(const float* w, int64_t n, float l1, float l2, double* acc, cudaStream_t s);
int rmsprop_update(float* params, const float* grads, float* rms, int64_t n, float lr, float clip,
                   float rho, float eps, float grad_scale, __nv_bfloat16* shadow, float* loss_out, cudaStream_t s);
// Keras 2.x update rules other than RMSprop (SGD, Adagrad, Adadelta, Adam, Adamax, Nadam); c[] are the per-step scalars
// the host derives from the iteration count (bias corrections, Nadam's momentum schedule)
struct OptScalars { int kind; float lr, clip, gs, c0, c1, c2, c3, c4; };
int optimizer_update(float* params, const float* grads, float* s1, float* s2, int64_t n, OptScalars o, __nv_bfloat16* shadow,
                     float* loss_out, cudaStream_t s);
int glorot_fill(float* w, int64_t n, int fan_in, int fan_out, uint64_t seed, uint64_t stream_id, cudaStream_t s);
int fill_value(float* p, int64_t n, float v, cudaStream_t s);
int cast_to_bf16(const float* in, __nv_bfloat16* out, int64_t n, cudaStream_t s);
int expand_counts(const void* cnt, int bits, const float* sf_in, int M, int n, const float* mean, const float* inv_std, int use_sf,
                  int use_log1p, float* Yout, void* Xout, int x_bf16, float* sf_out, const int64_t* ovf_indptr,
                  const void* ovf_entries, cudaStream_t s);
int expand_sparse(const void* bitmap, const int64_t* nib_indptr, const void* nibbles, const float* sf_in, int M, int n,
                  const float* mean, const float* inv_std, int use_sf, int use_log1p, float* Yout, void* Xout, int x_bf16,
                  float* sf_out, const int64_t* ovf_indptr, const void* ovf_entries, int max_row_nibble_bytes, cudaStream_t s);
int gather_rows_bf16(const void* X, int x_bf16, int64_t ldx, const int32_t* rows, int M, int n, __nv_bfloat16* out,
                     cudaStream_t s);

// ---------------------------------------------------------------- tensor-core kernels (dense_tc.cu, gene_gemm_tc.cu)
namespace tc {
int heads_fwd_tc(const __nv_bfloat16* Hb, int B, const __nv_bfloat16* const W[3], const float* const bias[3], int G,
                 int n_heads, const int kind[3], const float* row_scale, float* const out[3], int64_t ld_out, int sm_count,
                 cudaStream_t s);
int gene_gemm_tc(int mode, const __nv_bfloat16* const Z[3], int64_t ldz, int B, int G, int n_heads,
                 const __nv_bfloat16* H, const __nv_bfloat16* const W[3], float* out_b, float* const dW[3], int64_t dW_ld,
                 int dW_transposed, float* const db[3], void* ws, size_t ws_bytes, int sm_count, cudaStream_t s);
size_t gene_gemm_workspace_bytes(int B);
int flash_zinb_tc(const __nv_bfloat16* H3, int B, int G, const __nv_bfloat16* const W[3], const float* const bias[3],
                  const float* Y, int64_t ldy, const int32_t* rows, const float* sf, float ridge, float inv_n,
                  float* dH3, float* const dW[3], float* const db[3], void* ws, size_t ws_bytes, double* loss_sum,
                  const double* penalty, float* loss_slot, double* epoch_acc, int batch, const float* lf_dev, int sm_count,
                  cudaStream_t s);
}  // namespace tc

// ---------------------------------------------------------------- ZINB loss (zinb_loss.cu)
struct LossArgs {
  const float* Y; int64_t ldy; const int32_t* rows; const float* sf;
  const float* m; const float* d; const float* pi; int64_t ld;
  int B, G; int ae_type; float ridge; float inv_n;
  void* dzm; void* dzd; void* dzp; int grad_bf16;
  float* dtheta;            // const-disp: [G] summed d/dtheta
  double* loss_sum;         // device scalar, overwritten (fwd_bwd) or accumulated (fwd)
  void* ws; size_t ws_bytes;
  // optional fused finalize (engine): loss_slot[0] = loss_sum*inv_n (+penalty), [1] = non-finite flag, epoch acc update
  int counter_ready = 0;      // the self-resetting block counter inside `ws` is known to be zero (engine-owned workspace)
  float* fin_loss_slot = nullptr; double* fin_epoch_acc = nullptr; const double* fin_penalty = nullptr; int fin_batch = 0;
};
size_t loss_workspace_bytes(int B, int G);
extern int g_fused_heads_default;       // dca_set_tunable("fused_heads", 0 | 1)
const float* loss_log_fact_table();      // device table of log(k!), k < 64 (filled on first use)
int zinb_loss_fwd_bwd(const LossArgs& a, cudaStream_t s);
int zinb_loss_fwd(const LossArgs& a, cudaStream_t s);
// writes grads[P] = loss_sum*inv_n + penalty, grads[P+1] = nonfinite flag, epoch acc update

}  // namespace dca
