/* dca_b200.h -- C ABI of libdca_b200.so: the H100-native DCA training hot path.
 *
 * The reference (theislab/dca @ 6abd124) has no FFI: its boundary is the Python API, and the
 * arithmetic runs inside Keras/TensorFlow.  Each entry point below names the reference call
 * site(s) whose work it replaces (paths relative to the reference repository root).  The
 * Python binding a maintainer would add is shown in INTEGRATION.md; ours is dca_b200/_lib.py.
 *
 * Conventions
 *   - every function returns 0 on success or a negative dca_status; a thread-local message
 *     is available from dca_last_error().
 *   - all data pointers are DEVICE pointers unless the name ends in _host.
 *   - the caller owns every data buffer; a handle owns only what lives in its arena
 *     (parameters, gradients, optimizer state, BatchNorm state, fixed workspace).  No
 *     allocation happens inside step / predict calls.
 *   - all work is enqueued on the caller's stream (a cudaStream_t passed as void*); no
 *     hidden synchronisation except in the *_host entry points and dca_read_*.
 *   - a handle is bound to the device that was current at dca_create and is not thread safe.
 *   - matrices are row-major (cells x genes), leading dimensions in ELEMENTS.
 */
#ifndef DCA_B200_H
#define DCA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DCA_B200_VERSION 100          /* major*10000 + minor*100 + patch */
#define DCA_MAX_HIDDEN 8
#define DCA_NAME_LEN 48

typedef enum dca_status {
  DCA_OK = 0,
  DCA_ERR_BAD_ARG = -1,
  DCA_ERR_CUDA = -2,
  DCA_ERR_UNSUPPORTED = -3,
  DCA_ERR_NONFINITE = -4,
  DCA_ERR_NO_DEVICE = -5
} dca_status;

/* dca/network.py:763-768 AE_types keys on the accelerated path */
typedef enum dca_ae_type {
  DCA_AE_ZINB_CONDDISP = 0,   /* 'zinb-conddisp' ZINBAutoencoder              dca/network.py:366-393 */
  DCA_AE_ZINB = 1,            /* 'zinb'          ZINBConstantDispAutoencoder  dca/network.py:496-522 */
  DCA_AE_NB_CONDDISP = 2,     /* 'nb-conddisp'   NBAutoencoder                dca/network.py:293-316 */
  DCA_AE_NB = 3,              /* 'nb'            NBConstantDispAutoencoder    dca/network.py:249-269 */
  /* the remaining registry keys (SURVEY.md 8f-4): shape-general fp32 path, same loss kernel (extra_types.cu) */
  DCA_AE_POISSON = 4,         /* 'poisson'       PoissonAutoencoder           dca/network.py:233-246, dca/loss.py:33-48 */
  DCA_AE_NORMAL = 5,          /* 'normal'        Autoencoder (MSE, linear mean) dca/network.py:143-156 */
  DCA_AE_NB_SHARED = 6,       /* 'nb-shared'     NBSharedAutoencoder          dca/network.py:341-363 (dispersion per cell) */
  DCA_AE_ZINB_SHARED = 7,     /* 'zinb-shared'   ZINBSharedAutoencoder        dca/network.py:465-493 (pi, dispersion per cell) */
  DCA_AE_ZINB_ELEMPI = 8,     /* 'zinb-elempi'   ZINBAutoencoderElemPi        dca/network.py:424-462, dca/layers.py:50-81 */
  DCA_AE_NB_FORK = 9,         /* 'nb-fork'       NBForkAutoencoder            dca/network.py:664-760 */
  DCA_AE_ZINB_FORK = 10       /* 'zinb-fork'     ZINBForkAutoencoder          dca/network.py:553-661 */
} dca_ae_type;

/* Hidden-layer activation: Keras `Activation(name)` or, for the two names in `advanced_activations`
 * (dca/network.py:41,132-135), the Keras layer of that name with its default arguments.  Anything but
 * relu, and any dropout rate > 0, runs the per-layer hidden path (the one-launch hidden-stack kernel is
 * relu-only). */
typedef enum dca_activation {
  DCA_ACT_RELU = 0,
  DCA_ACT_LINEAR = 1,
  DCA_ACT_ELU = 2,            /* alpha = 1 */
  DCA_ACT_SELU = 3,
  DCA_ACT_TANH = 4,
  DCA_ACT_SIGMOID = 5,
  DCA_ACT_HARD_SIGMOID = 6,   /* clip(0.2 x + 0.5, 0, 1) */
  DCA_ACT_SOFTPLUS = 7,
  DCA_ACT_SOFTSIGN = 8,
  DCA_ACT_EXPONENTIAL = 9,
  DCA_ACT_LEAKY_RELU = 10,    /* keras.layers.LeakyReLU(): alpha = 0.3 */
  DCA_ACT_PRELU = 11          /* keras.layers.PReLU(): one trainable alpha per unit, zero-initialised ("<layer>_act/alpha") */
} dca_activation;

typedef enum dca_dtype { DCA_F32 = 0, DCA_BF16 = 1 } dca_dtype;

typedef enum dca_gemm_path {
  DCA_GEMM_AUTO = 0,          /* tensor-core (wgmma) tiles whenever the shape qualifies, else generic */
  DCA_GEMM_GENERIC = 1,       /* fp32 CUDA-core tiles for every layer (arbitrary shapes)  */
  DCA_GEMM_TCGEN05 = 2        /* require the tensor-core path; create fails if shape unsupported */
} dca_gemm_path;

typedef enum dca_region_id {
  DCA_REGION_PARAMS = 0,      /* float[P]   trainable parameters, Keras layouts (see dca_param_info) */
  DCA_REGION_GRADS = 1,       /* float[P+2] gradient of the mean loss; [P] = batch loss, [P+1] = non-finite flag */
  DCA_REGION_RMS = 2,         /* float[P]   first optimizer accumulator (RMSprop / Adagrad / Adadelta: mean square; Adam family: m) */
  DCA_REGION_BN_STATE = 3,    /* float[S]   BatchNorm moving_mean / moving_variance, see dca_state_info */
  DCA_REGION_EPOCH_ACC = 4    /* double[4]  {sum(loss*batch), sum(batch), sum(val_loss_elem), n_val_elem} */
} dca_region_id;

/* Mirrors the constructor of dca/network.py:44-59 (Autoencoder.__init__) plus the optimizer
 * constants of dca/train.py:54-57 and the Keras defaults they imply (SURVEY.md Appendix B). */
typedef struct dca_config {
  int32_t struct_bytes;       /* sizeof(dca_config), ABI guard */
  int32_t n_in;               /* input_size  (genes)           */
  int32_t n_out;              /* output_size (genes)           */
  int32_t n_hidden;           /* len(hidden_size), 0..DCA_MAX_HIDDEN */
  int32_t hidden[DCA_MAX_HIDDEN];
  int32_t ae_type;            /* dca_ae_type */
  int32_t batchnorm;          /* BatchNormalization(center=True, scale=False) after each hidden Dense */
  int32_t max_batch;          /* largest batch any step/predict call will pass */
  int32_t x_dtype;            /* dca_dtype of the network input matrix X */
  int32_t gemm_path;          /* dca_gemm_path */
  float ridge;                /* ZINB ridge_lambda, dca/loss.py:139 */
  float l1, l2, l1_enc, l2_enc;   /* kernel regularisers, dca/network.py:113-125 */
  float bn_momentum, bn_eps;  /* 0.99, 1e-3 */
  float rms_rho, rms_eps;     /* 0.9, 1e-7 */
  int32_t elempi_shared;      /* zinb-elempi: network_kwds sharedpi (scalar pi kernel / bias), dca/network.py:425-427,441 */
  int32_t sync_bn;            /* data-parallel runs (dca_comm_init): BatchNorm statistics over the GLOBAL batch (sum all-reduce of
                               * the column sums, forward and backward) -- exactly the single-GPU model at the global batch size.
                               * 0 (default): per-rank batch statistics, no extra collective (SURVEY.md 8e). */
  int32_t activation;         /* dca_activation of every hidden layer (dca/network.py:58,129-135; CLI --activation); 0 = relu */
  float input_dropout;        /* Dropout(rate) on the network input, training only (dca/network.py:98-99); 0 = off */
  float hidden_dropout[DCA_MAX_HIDDEN];   /* Dropout(rate) after each hidden activation (dca/network.py:137-138) */
  uint64_t dropout_seed;      /* stream of the counter-based mask generator (dca_dropout_mask_host reproduces a mask) */
} dca_config;

typedef struct dca_handle dca_handle;

typedef struct dca_tensor_info {
  char name[DCA_NAME_LEN];    /* e.g. "enc0/kernel", "center/bn_beta", "mean/bias", "dispersion/theta", "dec1_last_mean/kernel", "mean_no_act/kernel" */
  int64_t offset;             /* element offset into the region */
  int32_t rows, cols;         /* kernel: (in, out) as in Keras; vectors: rows = 1 */
} dca_tensor_info;

int dca_version(void);
const char* dca_last_error(void);
void dca_config_default(dca_config* cfg);

/* ---- lifetime ------------------------------------------------------------------------- */
/* Bytes of device memory a handle needs. */
int dca_arena_bytes(const dca_config* cfg, size_t* bytes);
/* Build the engine.  `arena` is caller-allocated device memory of at least dca_arena_bytes
 * (256-byte aligned), or NULL to let the library cudaMalloc it.
 * Replaces: AE_types[type](...).build() + model.compile(...)  (dca/api.py:183-188,
 * dca/network.py:92-156, dca/train.py:54-59). Parameters are zero until dca_init_params /
 * a write through DCA_REGION_PARAMS. */
int dca_create(const dca_config* cfg, void* arena, size_t arena_bytes, dca_handle** out);
int dca_destroy(dca_handle* h);

int dca_param_count(const dca_handle* h, int64_t* n_params, int32_t* n_tensors);
int dca_param_info(const dca_handle* h, int32_t index, dca_tensor_info* info);
int dca_state_count(const dca_handle* h, int64_t* n_state, int32_t* n_tensors);
int dca_state_info(const dca_handle* h, int32_t index, dca_tensor_info* info);
int dca_region(dca_handle* h, int32_t region_id, void** dev_ptr, int64_t* count);

/* Glorot-uniform kernels, zero biases/beta/theta, moving_mean 0, moving_var 1, rms 0
 * (Keras initialisers named at dca/network.py:124-126, dca/layers.py:17-20). */
int dca_init_params(dca_handle* h, uint64_t seed, void* stream);
/* Call after writing DCA_REGION_PARAMS directly (refreshes operand-layout shadow copies). */
int dca_params_changed(dca_handle* h, void* stream);

/* ---- the hot path --------------------------------------------------------------------- */
/* One training batch: forward (training-mode BatchNorm, moving statistics updated), loss,
 * backward into DCA_REGION_GRADS (gradient of the batch-mean loss; grads[P] = loss).
 * X: network input (dataset base pointer, dtype cfg.x_dtype, leading dim ldx);
 * Y: raw counts float32 (leading dim ldy); sf: size factors, one per dataset row;
 * rows: int32[batch] dataset row indices of this batch, or NULL for rows 0..batch-1.
 * Replaces one iteration of Keras Model.fit's batch loop up to (excluding) the optimizer
 * update: dca/train.py:91-98 executing dca/network.py:124-139,369-381 and dca/loss.py:122-148. */
int dca_train_step(dca_handle* h, const void* X, int64_t ldx, const float* Y, int64_t ldy,
                   const float* sf, const int32_t* rows, int32_t batch, void* stream);

/* The same step in two halves, for overlapping the gradient all-reduce with the tail of the backward pass:
 * phase 1 = forward + loss + head backward (afterwards grads[head_bucket_offset : P+2] -- the head kernels and
 * biases, ~98 % of the parameters, plus the loss slot -- are final), phase 2 = hidden-stack / encoder backward
 * (fills grads[0 : head_bucket_offset]).  Same arguments for both calls. */
int dca_train_step_phase(dca_handle* h, const void* X, int64_t ldx, const float* Y, int64_t ldy,
                         const float* sf, const int32_t* rows, int32_t batch, int32_t phase, void* stream);
int dca_grad_buckets(const dca_handle* h, int64_t* head_bucket_offset);

/* Data-parallel exchange inside the library (SURVEY.md 8b/8e; the reference is single-process: dca/train.py:91-98 has no
 * counterpart).  One NCCL communicator per engine: rank 0 calls dca_comm_unique_id, the 128 bytes travel to the other
 * ranks by any means (torch.distributed broadcast in dca_b200/engine.py), every rank calls dca_comm_init.  libnccl.so.2
 * is resolved with dlopen at the first call (DCA_ERR_UNSUPPORTED when absent).
 *   dca_allreduce      sum all-reduce of DCA_REGION_GRADS (P + 2 floats: gradients, loss slot, non-finite flag) in place.
 *   dca_train_step_dp  dca_train_step with the exchange fused into the launch sequence: phase 1 -> all-reduce(head bucket)
 *                      on an internal high-priority stream || phase 2 -> all-reduce(rest) -> join; captured and replayed
 *                      as ONE CUDA graph like dca_train_step.  Follow with dca_apply_update(grad_scale = 1 / world). */
int dca_comm_unique_id(void* id128);
int dca_comm_init(dca_handle* h, const void* id128, int32_t rank, int32_t world);
int dca_comm_destroy(dca_handle* h);
int dca_allreduce(dca_handle* h, void* stream);
int dca_train_step_dp(dca_handle* h, const void* X, int64_t ldx, const float* Y, int64_t ldy,
                      const float* sf, const int32_t* rows, int32_t batch, void* stream);

/* Optimizer of dca_apply_update: `opt.__dict__[optimizer](clipvalue=clip_grad[, lr=learning_rate])` of dca/train.py:54-57
 * (CLI --optimizer).  Every hyper-parameter except the learning rate and the clip value is the Keras 2.x default of that
 * class (keras/optimizers.py -- a dependency of the reference, not vendored in it): SGD (no momentum), RMSprop (rho 0.9),
 * Adagrad, Adadelta (rho 0.95), Adam / Adamax (beta 0.9 / 0.999), Nadam (schedule_decay 0.004); epsilon 1e-7, decay 0.
 * dca_set_optimizer selects the rule and clears its state (accumulators, iteration count); dca_reset_optimizer only
 * clears the state.  RMSprop is the default of a new handle. */
typedef enum dca_optimizer {
  DCA_OPT_RMSPROP = 0, DCA_OPT_SGD = 1, DCA_OPT_ADAGRAD = 2, DCA_OPT_ADADELTA = 3, DCA_OPT_ADAM = 4, DCA_OPT_ADAMAX = 5,
  DCA_OPT_NADAM = 6
} dca_optimizer;
int dca_set_optimizer(dca_handle* h, int32_t optimizer, void* stream);
int dca_reset_optimizer(dca_handle* h, void* stream);

/* clip(g*grad_scale, +-clip) -> the selected optimizer (RMSprop unless dca_set_optimizer chose another) -> parameters.
 * Replaces keras RMSprop(clipvalue=clip_grad[, lr]) applied by model.fit: dca/train.py:54-57.
 * grad_scale = 1/world_size after a sum all-reduce of DCA_REGION_GRADS, else 1. */
int dca_apply_update(dca_handle* h, float lr, float clip, float grad_scale, void* stream);

/* Inference-mode forward + summed element loss, accumulated into DCA_REGION_EPOCH_ACC[2..3].
 * Replaces the validation pass of Model.fit (validation_split, dca/train.py:96). */
int dca_eval_step(dca_handle* h, const void* X, int64_t ldx, const float* Y, int64_t ldy,
                  const float* sf, const int32_t* rows, int32_t batch, void* stream);

/* Inference forward producing every output of the four Keras predict() passes in one:
 * mean_out = MeanAct(.)*sf  (model.predict, dca/network.py:202-203),
 * disp_out (B x G; for const-disp types G values, the per-gene theta)  (dca/network.py:400, 530),
 * pi_out (dca/network.py:401), latent_out = 'center' Dense output before BN (dca/network.py:184-185,197).
 * Any output pointer may be NULL.  ld_out is the leading dim of the B x G outputs. */
int dca_predict(dca_handle* h, const void* X, int64_t ldx, const float* sf, const int32_t* rows,
                int32_t batch, float* mean_out, float* disp_out, float* pi_out, int64_t ld_out,
                float* latent_out, void* stream);

/* Blocking helpers: copy the last batch loss / epoch accumulators to the host. */
int dca_read_loss(dca_handle* h, float* loss_host, int32_t* nonfinite_host, void* stream);
int dca_read_epoch_acc(dca_handle* h, double acc_host[4], int32_t reset, void* stream);

/* Mirror every step's loss into pinned (mapped) HOST memory without a copy in the stream: the k-th
 * dca_apply_update after this call stores grads[P] * grad_scale (the batch loss, averaged over ranks once the
 * gradient buffer was all-reduced) into host_ring[k % n_slots] from inside the update kernel.  The host reads a
 * slot after synchronising on a later event.  NULL / 0 switches it off. */
int dca_set_loss_ring(dca_handle* h, float* host_ring, int32_t n_slots);

/* End-to-end variant with HOST buffers (pinned recommended): copies the batch
 * (x_host: batch x n_in of cfg.x_dtype, y_host: batch x n_out float, sf_host: batch float)
 * to the device, runs dca_train_step + dca_apply_update, copies the loss back and waits. */
int dca_train_step_host(dca_handle* h, const void* x_host, const float* y_host,
                        const float* sf_host, int32_t batch, float lr, float clip,
                        float* loss_host, void* stream);

/* ---- streaming from host memory (out-of-core / end-to-end path) ----------------------------- */
/* On-device restatement of dca/io.py:99-109 for one batch: X = ((log1p)(y / sf) - mean_g) * inv_std_g.
 * gene_mean_host / gene_inv_std_host: float[n_in] HOST arrays (copied), or NULL for no centring/scaling. */
int dca_set_input_transform(dca_handle* h, const float* gene_mean_host, const float* gene_inv_std_host,
                            int32_t use_size_factors, int32_t use_log1p, void* stream);
/* Train from a HOST-resident raw count matrix (uint16 counts [n_rows x n_in], leading dim ld_counts, pinned
 * memory recommended; size factors float[n_rows]).  dca_stream_step(i, next) waits for batch i (rows
 * [i*batch, min(n_rows,(i+1)*batch))) to arrive, starts the copy of batch `next` on an internal copy stream
 * (double-buffered staging), expands the counts on the device into the fp32 target Y and the normalised
 * network input X, and runs dca_train_step on them; the caller then all-reduces / calls dca_apply_update
 * exactly as for the resident path.  Requires n_in == n_out. */
int dca_stream_begin(dca_handle* h, const uint16_t* counts_host, int64_t ld_counts, const float* sf_host,
                     int64_t n_rows, int32_t batch, void* stream);
/* Same, from a bit-PACKED count matrix (fewer PCIe bytes per step): `bits` = 4, 8 or 16 per entry, row-major,
 * row stride `row_bytes` (a 4-bit row keeps gene c in byte c/2, low nibble = even c).  Counts >= 2^bits-1 are
 * stored as the escape value 2^bits-1 and listed in a CSR overflow list over ALL rows: ovf_indptr_host
 * int64[n_rows+1], ovf_entries_host {int32 gene; float count}[ovf_indptr[n_rows]] sorted by row; each step
 * copies its batch's segment with the tile and patches the escapes on the device.  Both NULL: no escapes
 * (2^bits-1 is a literal count).  A batch may carry at most max_batch*n_in/32 (>= 4096) overflow entries.
 * dca_b200/io.py:pack_counts builds the format; dca_stream_begin(...) == bits 16 without an overflow list. */
int dca_stream_begin_packed(dca_handle* h, const void* packed_host, int32_t bits, int64_t row_bytes,
                            const int64_t* ovf_indptr_host, const void* ovf_entries_host, const float* sf_host,
                            int64_t n_rows, int32_t batch, void* stream);
/* Sparse host format for matrices with <= 50 % non-zero entries (scRNA-seq: ~10-20 %): bitmap_host = one bit per entry
 * (row-major, n_in/8 bytes per row, bit g%8 of byte g/8 set when the count is non-zero), nibbles_host = the non-zero counts
 * of every row as consecutive 4-bit codes in gene order (low nibble first; 1..14 literal, 15 = escape into the overflow
 * list above), each row starting on a byte boundary at nib_indptr_host[row] (int64[n_rows+1], byte offsets).  ~0.2 bytes
 * per entry cross PCIe per step instead of 0.5 (4-bit dense) or the reference's 8 (float32 X + Y, dca/train.py:78-98).
 * dca_b200/io.py:pack_counts(..., bits='sparse' | 'auto') builds it. */
int dca_stream_begin_sparse(dca_handle* h, const void* bitmap_host, const int64_t* nib_indptr_host, const void* nibbles_host,
                            const int64_t* ovf_indptr_host, const void* ovf_entries_host, const float* sf_host,
                            int64_t n_rows, int32_t batch, void* stream);
int dca_stream_step(dca_handle* h, int64_t batch_index, int64_t next_batch_index /* -1: none */, void* stream);
int dca_stream_end(dca_handle* h, void* stream);

/* ---- stand-alone kernels (parity tests, profiling) -------------------------------------- */
/* ZINB / NB negative log-likelihood forward + backward, one pass (dca/loss.py:72-156 and its
 * autodiff).  Inputs are POST-activation head outputs: m = MeanAct(zm) (not yet multiplied by
 * sf), d = DispAct(zd) (B x G) or, for const-disp types, theta (G values, ld ignored), pi.
 * Outputs (may alias the inputs): gradients of the mean loss w.r.t. the PRE-activations
 * dzm, dzd, dzp scaled by inv_n; for const-disp types dzd receives nothing and
 * dtheta (G floats) receives d(loss)/d(theta) (before the exp/clip chain) summed over rows.
 * loss_sum: device double, receives the SUM of element losses (not the mean).
 * grad_dtype selects float32 or bfloat16 storage for dz*. */
int dca_zinb_loss_fwd_bwd(const float* Y, int64_t ldy, const int32_t* rows, const float* sf,
                          const float* m, const float* d, const float* pi, int64_t ld,
                          int32_t batch, int32_t genes, int32_t ae_type, float ridge, float inv_n,
                          void* dzm, void* dzd, void* dzp, int32_t grad_dtype,
                          float* dtheta, double* loss_sum, void* workspace, size_t workspace_bytes,
                          void* stream);
int dca_zinb_loss_workspace_bytes(int32_t batch, int32_t genes, size_t* bytes);
/* Forward only (validation): loss_sum += sum of element losses. */
int dca_zinb_loss_fwd(const float* Y, int64_t ldy, const int32_t* rows, const float* sf,
                      const float* m, const float* d, const float* pi, int64_t ld,
                      int32_t batch, int32_t genes, int32_t ae_type, float ridge,
                      double* loss_sum, void* workspace, size_t workspace_bytes, void* stream);

/* HOST mirror of the per-element device arithmetic of the loss kernel (same source compiled for
 * the CPU); a testing aid so the formulas can be checked against the oracle without a GPU.
 * out = {element loss, dL/dzm, dL/dzd (or raw dL/dtheta for const-disp types), dL/dzp}, not / N.
 * ae_type | 0x100 (ZINB types) evaluates the formulations the staged / fused kernels execute instead: the
 * branch-free zero branch and the NB branch computed from mu = m * sf with the MeanAct mask applied afterwards. */
int dca_zinb_elem_host(int32_t ae_type, float y, float m, float sf, float d, float pi, float ridge,
                       float out[4]);

/* HOST mirrors of the hidden-layer pieces the per-layer path adds (same source as the device code):
 * dca_dropout_mask_host writes the keep mask (1 = kept) the device applies at training step `step` (1 for the first
 * dca_train_step after dca_create) to elements [0, n) of `layer` (hidden layer index; -1 = the input; fork branches
 * use DCA_MAX_HIDDEN + branch); kept values are scaled by 1 / (1 - rate) as keras.layers.Dropout does.
 * dca_activation_host evaluates activation `act` (value and derivative; PReLU with slope `alpha`). */
int dca_dropout_mask_host(uint64_t seed, uint64_t step, int32_t layer, int64_t n, float rate, uint8_t* keep);
int dca_activation_host(int32_t act, float x, float alpha, float out[2]);

/* Head Dense layers with fused output activations (dca/network.py:369-381, :38-39,
 * dca/layers.py:85): H (B x K float32, ld ldh) times the Keras-layout kernels (K x G) plus bias,
 * then MeanAct / DispAct / sigmoid.  Any of the three heads may be NULL.  row_scale (B floats,
 * or NULL) multiplies the mean head (mean*sf, used by predict). */
int dca_dense_heads_fwd(const float* H, int64_t ldh, int32_t batch, int32_t K, int32_t genes,
                        const float* w_mean, const float* b_mean,
                        const float* w_disp, const float* b_disp,
                        const float* w_pi, const float* b_pi,
                        const float* row_scale,
                        float* m_out, float* d_out, float* pi_out, int64_t ld_out, void* stream);

/* tensor-core head layer: Hb = bf16 [batch x 64] (decoder output), Wk = bf16 [n_heads][64][genes] (the Keras
 * kernels, read in place as MN-major operands), bias = float [n_heads*genes]; kind[i] in {2 MeanAct,
 * 3 DispAct, 4 sigmoid} per head slot.  Same arithmetic as dca_dense_heads_fwd with bf16-rounded operands
 * and fp32 accumulation. */
int dca_tc_heads_fwd(const void* Hb, int32_t batch, const void* Wk, const float* bias, int32_t genes,
                     int32_t n_heads, const int32_t kind[3], const float* row_scale,
                     float* out0, float* out1, float* out2, int64_t ld_out, void* stream);

/* The gene-wide tensor-core product kernel (one smem tile of Z = X or dZ feeds both products):
 * mode 1: out_b[B x 64] += Z . W (W = bf16 [genes x 64], Keras layout)             -- encoder forward
 * mode 2: dW += Z^T . H (H = bf16 [B x 64])                                       -- encoder backward
 * mode 3: both (W = bf16 [n_heads][64][genes]), plus db = column sums of Z         -- head backward
 * Z0..Z2: bf16 [B x genes] per head (leading dim ldz); dW per head: float, dW[f*dW_ld + g] when
 * dW_transposed (Keras [64 x genes]) else dW[g*dW_ld + f].  All outputs are accumulated (+=). */
int dca_tc_gene_gemm(int32_t mode, const void* Z0, const void* Z1, const void* Z2, int64_t ldz, int32_t batch,
                     int32_t genes, int32_t n_heads, const void* H, const void* W, float* out_b,
                     float* dW0, float* dW1, float* dW2, int64_t dW_ld, int32_t dW_transposed,
                     float* db0, float* db1, float* db2, void* stream);

/* Single-tile wgmma probe used by the tests to pin the operand descriptor conventions: D[128 x N] =
 * A . B with bf16 operands; a K-major operand is stored [MN x K], an MN-major one [K x MN].
 * *_lbo / *_sbo < 0 select the library's defaults for that layout. */
int dca_tc_probe(const void* A, int32_t a_rows, int32_t a_cols, const void* B, int32_t b_rows, int32_t b_cols,
                 int32_t a_mn_major, int32_t b_mn_major, int32_t M, int32_t N, int32_t K,
                 int32_t a_lbo, int32_t a_sbo, int32_t b_lbo, int32_t b_sbo, float* D, void* stream);

/* Optional per-phase device timing (CUDA events on the caller's stream around each phase of
 * dca_train_step / dca_apply_update).  Off by default; bench.py turns it on for a separate
 * profiled pass.  Phases: 0 hidden forward, 1 head Dense + activations, 2 ZINB loss fwd+bwd,
 * 3 head backward, 4 hidden backward, 5 optimizer update. */
#define DCA_N_PHASES 6
int dca_profile_enable(dca_handle* h, int32_t on);
int dca_profile_read(dca_handle* h, double ms[DCA_N_PHASES], int64_t counts[DCA_N_PHASES], int32_t reset);

/* Which code paths an engine selected: info = {tensor-core heads (K2/K4), tensor-core encoder (K1/K5),
 * fused hidden stack, head slots, SM count, bytes per loss-gradient element (4 fp32 | 2 bf16),
 * instantiated step graphs, graphs enabled}. */
int dca_engine_info(const dca_handle* h, int32_t info[8]);

/* Number of kernels this library has launched in this process (all handles, all streams). */
/* ---- host-side output writer ------------------------------------------------------------------- */
/* Replaces write_text_matrix (dca/io.py:120-129: pandas to_csv(sep='\t', float_format='%.6f')) byte for byte:
 * optional header line of column labels (preceded by an empty cell when row labels are given), one line per
 * row "label\tv\tv...", NaN as an empty field, labels quoted only when they contain a tab, quote or newline.
 * matrix: HOST float32 (is_float64 = 0) or float64 rows x cols, leading dimension ld; transpose != 0 writes the
 * transposed matrix (labels swap roles) without materialising it.  threads <= 0: up to 16 hardware threads. */
int dca_write_text_matrix(const char* path, const void* matrix, int32_t is_float64, int64_t rows, int64_t cols,
                          int64_t ld, const char* const* row_names, const char* const* col_names,
                          int32_t transpose, int32_t threads);

/* Host-side packer for dca_stream_begin_packed (multi-threaded counterpart of dca_b200/io.py:pack_counts; no
 * reference counterpart).  counts: HOST matrix rows x cols (ld elements per row) of dtype 0 float32, 1 float64,
 * 2 uint16, 3 int32, 4 int64 holding non-negative integers.  dca_count_escapes fills per_row[w*rows + r] with the
 * number of entries of row r that need the overflow list at width w (0: 4 bits, 1: 8 bits, 2: 16 bits);
 * dca_pack_counts writes the packed matrix and the overflow entries given indptr = exclusive prefix sum of the
 * chosen width's per-row counts (int64[rows+1]). */
int dca_count_escapes(const void* counts, int32_t dtype, int64_t rows, int64_t cols, int64_t ld, int64_t* per_row,
                      int32_t threads);
int dca_pack_counts(const void* counts, int32_t dtype, int64_t rows, int64_t cols, int64_t ld, int32_t bits,
                    void* packed, const int64_t* indptr, void* entries, int32_t threads);

/* Host-side packer of the sparse format (dca_stream_begin_sparse): dca_sparse_counts fills nnz[r] (non-zero entries of row r)
 * and esc[r] (entries >= 15); with nib_indptr = cumsum((nnz + 1) / 2) (bytes) and ovf_indptr = cumsum(esc) dca_pack_sparse
 * writes the bitmap [rows x cols/8], the 4-bit codes and the overflow entries.  Multi-threaded, no reference counterpart. */
int dca_sparse_counts(const void* counts, int32_t dtype, int64_t rows, int64_t cols, int64_t ld, int64_t* nnz, int64_t* esc,
                      int32_t threads);
int dca_pack_sparse(const void* counts, int32_t dtype, int64_t rows, int64_t cols, int64_t ld, void* bitmap,
                    const int64_t* nib_indptr, void* nibbles, const int64_t* ovf_indptr, void* entries, int32_t threads);

int64_t dca_launch_count(void);
/* Launch tunables of the loss kernel (process-wide; set them BEFORE the first training step of an engine,
 * a captured step graph keeps the values it was recorded with): "loss_target_blocks",
 * "loss_producer_sleep_ns", "loss_consumer_sleep_ns", "loss_branch_free" (0 | 1, default 1); "fused_heads" (0 | 1, default 0): engines created afterwards
 * run head forward + loss + head backward of a zinb-conddisp training step as one fused kernel (flash_zinb.cu)
 * instead of three (environment override DCA_FUSED_HEADS).  Profiling aid -- no reference counterpart. */
int dca_set_tunable(const char* name, int64_t value);

#ifdef __cplusplus
}
#endif
#endif /* DCA_B200_H */
