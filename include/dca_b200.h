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
 *     hidden synchronisation except in the *_host entry points, dca_read_* and dca_write_text_device.
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

/* ---- initializers: the `kernel_initializer` of every Dense / ElementwiseDense kernel (dca/network.py:124-126,
 * CLI --init), Keras 2 / tf.keras 2.x semantics.  Fans (Keras _compute_fans): a 2-D kernel (in, out) has fan_in = in,
 * fan_out = out; a 1-D kernel of length n (zinb-elempi's "pi/kernel") has fan_in = fan_out = n.  In the types other
 * than the four flagship ones, a 2-D kernel with one input row (n_in or a hidden width of 1) also takes fan_in = out,
 * as glorot_uniform has always drawn it there (Keras: 1); it is still 2-D for ORTHOGONAL and IDENTITY.
 *   VARIANCE_SCALING(scale > 0, mode, distribution): n = fan_in, fan_out or (fan_in + fan_out) / 2 by mode,
 *     s = scale / max(1, n); uniform: U(-sqrt(3 s), sqrt(3 s)) (limit computed in float); untruncated normal:
 *     N(0, sqrt(s)); truncated normal: N(0, sqrt(s) / 0.87962566103423978) re-drawn beyond 2 sigma.
 *   RANDOM_NORMAL(stddev): N(0, stddev).  TRUNCATED_NORMAL(stddev): the same re-drawn beyond 2 stddev.
 *   RANDOM_UNIFORM(minval, maxval): U(minval, maxval).  CONSTANT(value).
 *   ORTHOGONAL(gain): A = (max(rows, cols) x min(rows, cols)) standard normals, Q R = A (reduced), Q <- Q sign(diag R),
 *     W = gain Q, transposed when rows < cols; an fp64 Householder QR on the device, one CTA per kernel.
 *   IDENTITY(gain): gain * eye(rows, cols).  ORTHOGONAL and IDENTITY need 2-D kernels.
 * Draws are counter-based: element i of the kernel with stream id sid is a function of (seed, sid, i) alone.
 *   uniform: u = (h >> 40) 2^-24 from a 64-bit hash h of (seed, sid, i); w = fmaf(2u - 1, half, center).
 *   normal: Box-Muller in fp64 from two 53-bit uniforms of draw a (0, 1, ...) of the element, rounded once to float;
 *     a truncated normal takes the first draw with |z| < 2, and 0 if 16 draws all fail (probability < 4e-22).
 * Kernel stream ids: the four flagship types (zinb-conddisp, zinb, nb-conddisp, nb) number their hidden layers 0, 1,
 * ... and the head kernels 100 (mean), 101 (dispersion), 102 (pi); the other types number every kernel in the order
 * of dca_param_info. */
typedef enum dca_init_kind {
  DCA_INIT_VARIANCE_SCALING = 0, DCA_INIT_RANDOM_NORMAL = 1, DCA_INIT_RANDOM_UNIFORM = 2, DCA_INIT_TRUNCATED_NORMAL = 3,
  DCA_INIT_CONSTANT = 4, DCA_INIT_ORTHOGONAL = 5, DCA_INIT_IDENTITY = 6
} dca_init_kind;
typedef enum dca_fan_mode { DCA_FAN_IN = 0, DCA_FAN_OUT = 1, DCA_FAN_AVG = 2 } dca_fan_mode;
typedef enum dca_distribution {
  DCA_DIST_TRUNCATED_NORMAL = 0, DCA_DIST_UNTRUNCATED_NORMAL = 1, DCA_DIST_UNIFORM = 2
} dca_distribution;
typedef struct dca_initializer {
  int32_t struct_bytes;       /* sizeof(dca_initializer), ABI guard */
  int32_t kind;               /* dca_init_kind */
  float scale;                /* VARIANCE_SCALING */
  int32_t mode;               /* VARIANCE_SCALING: dca_fan_mode */
  int32_t distribution;       /* VARIANCE_SCALING: dca_distribution */
  float stddev;               /* RANDOM_NORMAL, TRUNCATED_NORMAL */
  float minval, maxval;       /* RANDOM_UNIFORM */
  float value;                /* CONSTANT */
  float gain;                 /* ORTHOGONAL, IDENTITY */
} dca_initializer;
/* dca_init_params with `init` for every kernel (biases, BatchNorm, PReLU slopes, theta and the optimizer state as
 * there).  glorot_uniform is VARIANCE_SCALING(1, FAN_AVG, UNIFORM): the same bits as dca_init_params.  An invalid
 * spec, or ORTHOGONAL / IDENTITY on a model with a 1-D kernel, returns DCA_ERR_BAD_ARG and changes nothing. */
int dca_init_params_ex(dca_handle* h, uint64_t seed, const dca_initializer* init, void* stream);
/* HOST restatement of the draws (same source as the device code): the rows x cols elements (ndim 1: rows = 1) of the
 * kernel with stream id sid into out, row-major.  ORTHOGONAL writes its matrix A instead (max(rows, cols) x
 * min(rows, cols), row-major), whose QR the device takes. */
int dca_init_fill_host(const dca_initializer* init, uint64_t seed, uint64_t sid, int32_t ndim, int32_t rows, int32_t cols,
                       float* out);
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

/* Debug checks (--debug, dca/loss.py:87-100): with `on`, every training step (dca_train_step*, the streamed and packed
 * steps) and every dca_eval_step* evaluates the reference's NB terms of every element of the batch, in float32 and in
 * the reference's form -- theta' = min(theta, 1e6), eps = 1e-10, y_pred = mean * sf,
 * t1 = lgamma(theta' + eps) + lgamma(y + 1) - lgamma(y + theta' + eps),
 * t2 = (theta' + y) log(1 + y_pred / (theta' + eps)) + y (log(theta' + eps) - log(y_pred + eps)) -- and records which
 * are not finite in a report the step clears first.  Types whose reference loss has no such check (nb, poisson,
 * normal) always report nothing.  The checks are a kernel of their own, launched ahead of the loss kernel on the
 * operands it reads (on the tensor-core heads + loss path, the head-forward kernel first writes the head outputs for
 * them), so the loss, the gradients and every accumulator have the same bits with the checks on.  Toggling drops the
 * captured step graphs; the fused flash_zinb path is not taken while the checks are on.  Off (the default), every
 * kernel, launch and graph is the one without checks. */
int dca_set_debug_checks(dca_handle* h, int32_t on);
typedef struct dca_debug_report {
  int32_t struct_bytes;      /* sizeof(dca_debug_report), set by the caller: ABI guard */
  int32_t reserved;
  int64_t count[3];          /* non-finite y_pred, t1, t2 elements of the last step */
  int32_t first_row[3];      /* per term: batch row of its first non-finite element in row-major order, -1 if none */
  int32_t first_gene[3];     /* ... and its gene (output column), -1 if none */
} dca_debug_report;
/* Blocking: copies the report of the last step on `stream` to *out.  The same report on every run of the same step. */
int dca_read_debug_report(dca_handle* h, dca_debug_report* out, void* stream);
/* The checks of one batch on their own (the kernel the steps run ahead of their loss kernel): counts Y (device, row
 * rows[r] for batch row r, rows NULL: r; leading dim ldy), size factors sf (indexed like Y's rows; NULL: 1), mean m
 * (before the size factor, [batch x genes], leading dim ldm), dispersion theta (leading dim ld_theta; 0: one theta per
 * gene).  workspace: 48 bytes of device memory.  Blocking; writes *out (struct_bytes set by the caller). */
int dca_debug_check(const float* Y, int64_t ldy, const int32_t* rows, const float* sf, const float* m, int64_t ldm,
                    const float* theta, int64_t ld_theta, int32_t batch, int32_t genes, void* workspace,
                    dca_debug_report* out, void* stream);

/* Mirror every step's loss into pinned (mapped) HOST memory without a copy in the stream: the k-th
 * dca_apply_update after this call stores grads[P] * grad_scale (the batch loss, averaged over ranks once the
 * gradient buffer was all-reduced) into host_ring[k % n_slots] from inside the update kernel.  The host reads a
 * slot after synchronising on a later event.  NULL / 0 switches it off. */
int dca_set_loss_ring(dca_handle* h, float* host_ring, int32_t n_slots);

/* End-to-end variant with HOST buffers (pinned recommended): copies the batch
 * (x_host: batch x n_in of cfg.x_dtype, y_host: batch x n_out float, sf_host: batch float)
 * to the device, runs dca_train_step + dca_apply_update, copies the loss back and waits.  Its staging buffers are
 * those of the streaming path below: between dca_stream_begin* and dca_stream_end it returns DCA_ERR_BAD_ARG. */
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
 * dca_b200/io.py:pack_counts builds the format; dca_stream_begin(...) == bits 16 without an overflow list.
 * Ragged gene counts: the rows are Gp = n_in rounded up to a multiple of 8 entries wide, the Gp - n_in pad genes
 * zero counts (io.pack_rows(..., pad_genes=True)).  Batches are expanded Gp wide and the step reads their first n_in
 * columns; the pad genes never reach the model, its loss or its outputs.  Such an engine streams only with the exact
 * transform (dca_set_input_transform_exact), which gives the pad genes mean 0 and std 1. */
int dca_stream_begin_packed(dca_handle* h, const void* packed_host, int32_t bits, int64_t row_bytes,
                            const int64_t* ovf_indptr_host, const void* ovf_entries_host, const float* sf_host,
                            int64_t n_rows, int32_t batch, void* stream);
/* Sparse host format for matrices with <= 50 % non-zero entries (scRNA-seq: ~10-20 %): bitmap_host = one bit per entry
 * (row-major, Gp/8 bytes per row, bit g%8 of byte g/8 set when the count is non-zero), nibbles_host = the non-zero counts
 * of every row as consecutive 4-bit codes in gene order (low nibble first; 1..14 literal, 15 = escape into the overflow
 * list above), each row starting on a byte boundary at nib_indptr_host[row] (int64[n_rows+1], byte offsets).  ~0.2 bytes
 * per entry cross PCIe per step instead of 0.5 (4-bit dense) or the reference's 8 (float32 X + Y, dca/train.py:78-98).
 * dca_b200/io.py:pack_counts(..., bits='sparse' | 'auto') builds it. */
int dca_stream_begin_sparse(dca_handle* h, const void* bitmap_host, const int64_t* nib_indptr_host, const void* nibbles_host,
                            const int64_t* ovf_indptr_host, const void* ovf_entries_host, const float* sf_host,
                            int64_t n_rows, int32_t batch, void* stream);
int dca_stream_step(dca_handle* h, int64_t batch_index, int64_t next_batch_index /* -1: none */, void* stream);
int dca_stream_end(dca_handle* h, void* stream);
/* The exact transform of the device preprocessing (see "preprocessing" below; dca/io.py:88-111) for streamed batches,
 * instead of the float one of dca_set_input_transform: sf = float(n_counts[r] / median), X = float(((double)l -
 * mean_g) / std_g) with l = float(log1p((double)float((double)y / sf64))) per the DCA_PRE_* flags -- the bits
 * dca_normalize_write stores for the same cell.  gene_mean_host / gene_std_host: HOST fp64 [n_in] (copied; mean 0
 * and std 1 without DCA_PRE_SCALE).  With DCA_PRE_SIZE_FACTORS every stream needs its per-row fp64 totals:
 * dca_stream_row_totals(h, n_counts_host [n_rows], pinned, kept until dca_stream_end), called between
 * dca_stream_begin* and the first step; sf_host is then not read.  dca_set_input_transform switches back. */
int dca_set_input_transform_exact(dca_handle* h, const double* gene_mean_host, const double* gene_std_host, double median,
                                  int32_t flags, void* stream);
int dca_stream_row_totals(dca_handle* h, const double* n_counts_host);
/* Inference on the host stream (dca/network.py:188-211 on data that does not fit the GPU): dca_predict on batch
 * batch_index (outputs as there, batch rows), while the copy and expansion of next_batch_index overlap it -- the
 * batch bookkeeping of dca_stream_step, which it may follow or precede within one stream. */
int dca_stream_predict(dca_handle* h, int64_t batch_index, int64_t next_batch_index, float* mean_out, float* disp_out,
                       float* pi_out, int64_t ld_out, float* latent_out, void* stream);
/* The validation pass of fit (dca/train.py:96) on the host stream: dca_eval_step on batch batch_index, with the batch
 * bookkeeping of dca_stream_step. */
int dca_stream_eval(dca_handle* h, int64_t batch_index, int64_t next_batch_index, void* stream);
/* What one streamed batch may carry (fixed by max_batch and n_in at dca_create): overflow entries (dca_stream_begin_packed)
 * and bytes of non-zero codes (dca_stream_begin_sparse).  dca_stream_begin* rejects a dataset with a batch above either. */
int dca_stream_capacity(const dca_handle* h, int64_t* ovf_entries, int64_t* nibble_bytes);
/* The expansion of one streamed batch on its own (parity tests): the same kernels dca_stream_step runs, on DEVICE
 * arrays of n_rows contiguous rows in the formats above (overflow indptr int64[n_rows+1] and nib_indptr int64[n_rows+1]
 * are offsets relative to their first entry).  Writes Y (float [n_rows x genes]), X = ((log1p)(y / sf) - mean_g) *
 * inv_std_g in x_dtype (DCA_F32 | DCA_BF16, row stride genes) and sf_out[r] = sf[r] (1 when sf is NULL; sf_out may be
 * NULL).  y / sf is taken only when use_size_factors is set and sf is given; gene_mean / gene_inv_std: device
 * float[genes] or both NULL.  Sparse: max_row_nibble_bytes sizes the shared-memory copy of a row's codes; longer rows
 * read them from global memory.  Returns DCA_ERR_BAD_ARG when genes % 8 != 0, bits is not 4, 8 or 16, or the counts,
 * Y or X are not 16-byte aligned; DCA_ERR_UNSUPPORTED for a sparse matrix of more than 65536 genes; DCA_ERR_NO_DEVICE
 * without a CUDA device. */
int dca_expand_packed_counts(const void* packed, int32_t bits, const int64_t* ovf_indptr, const void* ovf_entries,
                             const float* sf, int32_t n_rows, int32_t genes, const float* gene_mean,
                             const float* gene_inv_std, int32_t use_size_factors, int32_t use_log1p,
                             float* Y, void* X, int32_t x_dtype, float* sf_out, void* stream);
int dca_expand_sparse_counts(const void* bitmap, const int64_t* nib_indptr, const void* nibbles,
                             int32_t max_row_nibble_bytes, const int64_t* ovf_indptr, const void* ovf_entries,
                             const float* sf, int32_t n_rows, int32_t genes, const float* gene_mean,
                             const float* gene_inv_std, int32_t use_size_factors, int32_t use_log1p,
                             float* Y, void* X, int32_t x_dtype, float* sf_out, void* stream);
/* The same with the exact transform of dca_set_input_transform_exact (dca/io.py:99-109 as dca_normalize_write computes
 * it): n_counts = device fp64 [n_rows] totals of these rows (needed with DCA_PRE_SIZE_FACTORS), gene_mean / gene_std =
 * device fp64 [genes].  sf_out[r] = float(n_counts[r] / median) (1 without DCA_PRE_SIZE_FACTORS). */
int dca_expand_packed_counts_exact(const void* packed, int32_t bits, const int64_t* ovf_indptr, const void* ovf_entries,
                                   const double* n_counts, int32_t n_rows, int32_t genes, double median, int32_t flags,
                                   const double* gene_mean, const double* gene_std, float* Y, void* X, int32_t x_dtype,
                                   float* sf_out, void* stream);
int dca_expand_sparse_counts_exact(const void* bitmap, const int64_t* nib_indptr, const void* nibbles,
                                   int32_t max_row_nibble_bytes, const int64_t* ovf_indptr, const void* ovf_entries,
                                   const double* n_counts, int32_t n_rows, int32_t genes, double median, int32_t flags,
                                   const double* gene_mean, const double* gene_std, float* Y, void* X, int32_t x_dtype,
                                   float* sf_out, void* stream);

/* ---- packed counts resident in device memory -------------------------------------------------------------------
 * The formats of dca_stream_begin_packed / dca_stream_begin_sparse, held whole in DEVICE memory with absolute offsets:
 * a dataset several times larger than the fp32 Y + X of the resident path, with no host traffic per step.  The rows of
 * a batch are named by index and expanded into the engine's expanded-batch staging with the exact transform
 * (dca_set_input_transform_exact), so every X, Y and size factor is the one dca_normalize_write stores for that cell. */
typedef struct dca_packed_counts {
  int32_t struct_bytes;           /* sizeof(dca_packed_counts), ABI guard */
  int32_t bits;                   /* 1 (sparse: bitmap + 4-bit codes of the non-zeros), 4, 8 or 16 bits per entry */
  int64_t n_rows;
  int32_t genes;                  /* the stored width, a multiple of 8: an engine's n_in rounded up (pad genes are zero) */
  int32_t max_row_nibble_bytes;   /* sparse: the longest row's code bytes (sizes the expansion's shared memory) */
  const void* packed;             /* [n_rows x genes*bits/8] bytes, 16-byte aligned (sparse: the bitmap) */
  const int64_t* ovf_indptr;      /* int64 [n_rows + 1], absolute offsets into ovf_entries; NULL: no overflow entries */
  const void* ovf_entries;        /* {int32 gene; float count} sorted by row, then gene */
  const int64_t* nib_indptr;      /* sparse: int64 [n_rows + 1], absolute byte offsets into nibbles */
  const void* nibbles;            /* sparse: the codes, each row on a byte boundary, 16 readable bytes of slack */
  const double* n_counts;         /* fp64 [n_rows] row totals (needed with DCA_PRE_SIZE_FACTORS) */
} dca_packed_counts;

/* The GPU packer.  Count pass: for n_rows rows of fp32 counts Y (device, leading dim ldy) stats[k * ld_stats + r]
 * (device int64) receives, per row r: k = 0 the non-zero entries, 1..3 the entries >= 15, >= 255 and >= 65535 (the
 * overflow entries of the 4, 8 and 16-bit widths, dca_count_escapes), 4 the entries that are negative, not an
 * integer or not finite.  Pack pass: rows [0, n_rows) of Y become rows row0 .. row0 + n_rows of the arrays of `dst`
 * (its pointers are the whole matrix's, its ovf_indptr / nib_indptr the exclusive prefix sums of the chosen width's
 * per-row escapes / (non-zeros + 1) / 2 over all rows): the bytes dca_pack_counts / dca_pack_sparse write for the same
 * counts.  dst->n_counts is not read.  No atomics: the output is a function of the counts. */
int dca_pack_count_rows(const float* Y, int64_t ldy, int64_t n_rows, int32_t genes, int64_t* stats, int64_t ld_stats,
                        void* stream);
int dca_pack_rows_device(const float* Y, int64_t ldy, int64_t n_rows, int64_t row0, const dca_packed_counts* dst,
                         void* stream);
/* Y [n x genes] (fp32), X (x_dtype, row stride genes) and sf_out [n] of rows rows[0..n) of src (device int32, each
 * < src->n_rows; NULL: rows 0..n-1) with the exact transform: the rows dca_normalize_write and the resident dataset
 * hold for the same cells.  gene_mean / gene_std: device fp64 [genes]. */
int dca_expand_rows_exact(const dca_packed_counts* src, const int32_t* rows, int32_t n, double median, int32_t flags,
                          const double* gene_mean, const double* gene_std, float* Y, void* X, int32_t x_dtype,
                          float* sf_out, void* stream);
/* dca_train_step / dca_eval_step / dca_predict on the batch rows[0..batch) of src: the rows are expanded with the
 * transform of dca_set_input_transform_exact (which must come first) into the engine's expanded-batch staging (bf16 X
 * for the tensor-core encoder) on `stream`, then the step runs on that contiguous batch.  The same bits as the step on
 * a resident dataset of the same cells.  DCA_ERR_BAD_ARG while a host stream is active (dca_stream_begin*);
 * DCA_ERR_UNSUPPORTED when n_in != n_out; DCA_ERR_BAD_ARG when src->genes is not n_in rounded up to a multiple of 8
 * (the pad genes of a ragged n_in are expanded with the batch and never reach the model). */
int dca_packed_train_step(dca_handle* h, const dca_packed_counts* src, const int32_t* rows, int32_t batch, void* stream);
int dca_packed_eval_step(dca_handle* h, const dca_packed_counts* src, const int32_t* rows, int32_t batch, void* stream);
int dca_packed_predict(dca_handle* h, const dca_packed_counts* src, const int32_t* rows, int32_t batch, float* mean_out,
                       float* disp_out, float* pi_out, int64_t ld_out, float* latent_out, void* stream);

/* ---- stand-alone kernels (parity tests, profiling) -------------------------------------- */
/* ZINB / NB negative log-likelihood forward + backward, one pass (dca/loss.py:72-156 and its
 * autodiff).  Inputs are POST-activation head outputs: m = MeanAct(zm) (not yet multiplied by
 * sf), d = DispAct(zd) (B x G) or, for const-disp types, theta (G values, ld ignored), pi.
 * Outputs (may alias the inputs): gradients of the mean loss w.r.t. the PRE-activations
 * dzm, dzd, dzp scaled by inv_n; for const-disp types dzd receives nothing and
 * dtheta (G floats) receives d(loss)/d(theta) (before the exp/clip chain) summed over rows: per row chunk of the
 * launch plan into the workspace, then the chunks in row order, so the result is the same bits on every run.
 * workspace_bytes: at least dca_zinb_loss_workspace_bytes(batch, genes), which does not shrink as batch grows, so the
 * size for a larger batch serves too; a plan that does not fit (e.g. after raising the "loss_target_blocks" tunable)
 * is refused with DCA_ERR_BAD_ARG.
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
 * ae_type | 0x200 (ZINB types) evaluates the formulation the ring and heads + loss kernels execute instead: the
 * f32x2 zero branch and the raw NB derivatives, chained through the activations by shared finishing factors. */
int dca_zinb_elem_host(int32_t ae_type, float y, float m, float sf, float d, float pi, float ridge,
                       float out[4]);

/* HOST mirrors of the hidden-layer pieces the per-layer path adds (same source as the device code):
 * dca_dropout_mask_host writes the keep mask (1 = kept) the device applies at training step `step` (1 for the first
 * dca_train_step after dca_create) to elements [0, n) of `layer` (hidden layer index; -1 = the input; fork branches
 * use DCA_MAX_HIDDEN + branch); kept values are scaled by 1 / (1 - rate) as keras.layers.Dropout does.
 * dca_activation_host evaluates activation `act` (value and derivative; PReLU with slope `alpha`).
 * dca_activation_bwd_host runs one element of a training step through activation + dropout at `rate` (0: none) with
 * keep flag `kept`: out[0] = the stored layer output, out[1] = the gradient w.r.t. the activation's input x given the
 * gradient g w.r.t. the layer's output. */
int dca_dropout_mask_host(uint64_t seed, uint64_t step, int32_t layer, int64_t n, float rate, uint8_t* keep);
int dca_activation_host(int32_t act, float x, float alpha, float out[2]);
int dca_activation_bwd_host(int32_t act, float x, float alpha, float rate, int32_t kept, float g, float out[2]);

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

/* Heads forward + zinb-conddisp loss forward/backward in one kernel (the training step's path): Hb, Wk (3 heads:
 * mean, dispersion, pi) and bias as in dca_tc_heads_fwd; Y, rows, sf, ridge, inv_n as in dca_zinb_loss_fwd_bwd.
 * Writes the bf16 gradients dzm / dzd / dzp (leading dim ldz) and *loss_sum, bit-identical in dZ to
 * dca_tc_heads_fwd (no row scale) followed by dca_zinb_loss_fwd_bwd with bf16 gradients; the fp32 head outputs are
 * never stored.  Needs genes % 8 == 0, Y 16-byte aligned with ldy % 4 == 0, ldz % 4 == 0.  Workspace: as for
 * dca_zinb_loss_fwd_bwd. */
int dca_tc_heads_loss(const void* Hb, int32_t batch, const void* Wk, const float* bias, int32_t genes,
                      const float* Y, int64_t ldy, const int32_t* rows, const float* sf, float ridge, float inv_n,
                      void* dzm, void* dzd, void* dzp, int64_t ldz, double* loss_sum, void* workspace,
                      size_t workspace_bytes, void* stream);

/* The gene-wide tensor-core product kernel (one smem tile of Z = X or dZ feeds both products):
 * mode 1: out_b[B x 64] += Z . W (W = bf16 [genes x 64], Keras layout)             -- encoder forward
 * mode 2: dW += Z^T . H (H = bf16 [B x 64])                                       -- encoder backward
 * mode 3: both (W = bf16 [n_heads][64][genes]), plus db = column sums of Z         -- head backward
 * Z0..Z2: bf16 [B x genes] per head (leading dim ldz); dW per head: float, dW[f*dW_ld + g] when
 * dW_transposed (Keras [64 x genes]) else dW[g*dW_ld + f].  All outputs are accumulated (+=).
 * The grid is at most the device's SM count. */
int dca_tc_gene_gemm(int32_t mode, const void* Z0, const void* Z1, const void* Z2, int64_t ldz, int32_t batch,
                     int32_t genes, int32_t n_heads, const void* H, const void* W, float* out_b,
                     float* dW0, float* dW1, float* dW2, int64_t dW_ld, int32_t dW_transposed,
                     float* db0, float* db1, float* db2, void* stream);
/* The same with the grid capped at sm_count CTAs (what the engine does when SMs are left to a collective): the CTAs
 * then stride over the items.  sm_count <= 0 uses the device's SM count. */
int dca_tc_gene_gemm_sms(int32_t mode, const void* Z0, const void* Z1, const void* Z2, int64_t ldz, int32_t batch,
                         int32_t genes, int32_t n_heads, const void* H, const void* W, float* out_b,
                         float* dW0, float* dW1, float* dW2, int64_t dW_ld, int32_t dW_transposed,
                         float* db0, float* db1, float* db2, void* stream, int32_t sm_count);
/* The same for modes 1 and 2 with the batch named by row index: cell i is row rows[i] of Z0 (leading dim ldz, a
 * multiple of 8; 16-byte aligned base), which may hold more rows than the batch.  Every index must be a row of Z0.
 * Computes the same bits as dca_tc_gene_gemm_sms on the gathered contiguous Z0[rows].  rows == NULL: row i. */
int dca_tc_gene_gemm_rows(int32_t mode, const void* Z0, const void* Z1, const void* Z2, int64_t ldz, const int32_t* rows,
                          int32_t batch, int32_t genes, int32_t n_heads, const void* H, const void* W, float* out_b,
                          float* dW0, float* dW1, float* dW2, int64_t dW_ld, int32_t dW_transposed,
                          float* db0, float* db1, float* db2, void* stream, int32_t sm_count);
/* The item schedule of mode 3 (host only, no device needed) for a batch of `batch` cells, `genes` genes, n_heads heads
 * and a grid of at most sm_count CTAs.  banded = 1: the one band-ordered launch (tunable "head_bwd_banded" = 1);
 * 0: the dW / db launch, then the dH launch.  Writes *n_items and grid[0..1] (CTAs of launch 0 and 1; 0 = no launch);
 * items (may be NULL) receives min(*n_items, cap) rows of 8 int32 in launch order: (launch, kind, head, first gene
 * block, gene blocks, first cell block, cell blocks, partial slot).  kind 0: dW / db over the item's 128-gene blocks and
 * all cells (slot -1); kind 1: dH over the item's gene blocks into its partial slot.  CTA c of a launch runs the
 * launch's items c, c + grid, c + 2 grid, ... */
int dca_head_bwd_schedule(int32_t batch, int32_t genes, int32_t n_heads, int32_t sm_count, int32_t banded,
                          int32_t* items, int64_t cap, int64_t* n_items, int32_t* grid);
/* The schedule of mode 2 (host only, no device needed) for `genes` genes and a grid of at most sm_count CTAs.  The
 * genes are cut into blocks of 64 (the last may be shorter); CTA c owns blocks first[c] .. first[c + 1] - 1, a
 * contiguous run, and the runs differ in length by at most one.  Writes *ctas and min(*ctas + 1, cap) entries of first
 * (may be NULL).  Each block's dW rows are summed over all cells by one warpgroup, in cell order, so the schedule does
 * not change the bits of dW. */
int dca_enc_bwd_schedule(int32_t genes, int32_t sm_count, int32_t* first, int64_t cap, int32_t* ctas);

/* ---- preprocessing of raw counts in HBM (csrc/preprocess.cu) ------------------------------------------------------
 * dca/io.py:88-111 -- scanpy's pp.filter_genes / pp.filter_cells(min_counts=1), pp.normalize_per_cell, pp.log1p and
 * pp.scale, restated on the host by dca_b200/io.py:normalize -- computed from the fp32 count matrix Y [n_cells x genes,
 * leading dimension ldy] the training step reads.  No atomics: reductions over cells fold per-CTA workspace slots in
 * slot order, so two calls are bit-identical.  The workspace of dca_count_totals / dca_log_moments is
 * dca_preprocess_workspace_bytes(n_cells, genes).  Without a CUDA device every entry point returns DCA_ERR_NO_DEVICE.
 *
 * Arithmetic, per cell r and gene g (flags: DCA_PRE_*; a step whose flag is clear is skipped):
 *   sf64 = n_counts[r] / median (fp64)                          normalize_per_cell (median of the fp64 totals)
 *   q    = float((double)y / sf64)
 *   l    = float(log1p((double)q))  -- rounded from double      pp.log1p
 *   mean = sum_r l / N, std = sqrt(sum_r (l - mean)^2 / (N - 1)), fp64 sums, two passes as NumPy's var;
 *          std = 1 for N = 1 and where it is 0                  pp.scale(zero_center=True), no clipping
 *   X    = float(((double)l - mean) / std); a bf16 X is __float2bfloat16_rn of that float. */
#define DCA_PRE_SIZE_FACTORS 1
#define DCA_PRE_LOG1P 2
#define DCA_PRE_SCALE 4
int dca_preprocess_workspace_bytes(int64_t n_cells, int32_t genes, size_t* bytes);
/* Y (zeros included) from a canonical CSR matrix (rows sorted, no duplicate entries, every index in [0, genes)):
 * int64 indptr [n_cells + 1], int32 indices, float32 data. */
int dca_counts_csr_to_dense(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_cells,
                            int32_t genes, float* Y, int64_t ldy, void* stream);
/* fp64 totals per cell (obs n_counts) and per gene (filter_genes' counts); either may be NULL.  *n_bad (device int64, or
 * NULL) receives the number of entries that are negative, non-integer or not finite; they are not an error. */
int dca_count_totals(const float* Y, int64_t ldy, int64_t n_cells, int32_t genes, double* cell_totals,
                     double* gene_totals, int64_t* n_bad, void* workspace, size_t workspace_bytes, void* stream);
/* out[i][j] = Y[rows[i]][cols[j]] (leading dimension ldo); rows / cols NULL: the identity.  Subsetting of AnnData's
 * _inplace_subset_obs / _inplace_subset_var (filter_genes, filter_cells) and of the output genes of --denoisesubset. */
int dca_gather_counts(const float* Y, int64_t ldy, const int32_t* rows, int64_t n_rows, const int32_t* cols,
                      int32_t n_cols, float* out, int64_t ldo, void* stream);
/* Gene mean and std of l (fp64, genes each).  Without DCA_PRE_SCALE: mean = 0, std = 1 and Y is not read.  n_counts
 * (device fp64) and median are needed with DCA_PRE_SIZE_FACTORS only. */
int dca_log_moments(const float* Y, int64_t ldy, int64_t n_cells, int32_t genes, const double* n_counts, double median,
                    int32_t flags, double* mean, double* std, void* workspace, size_t workspace_bytes, void* stream);
/* X [n_cells x genes, leading dimension ldx] in x_dtype (DCA_F32 | DCA_BF16); mean / std NULL: X = l. */
int dca_normalize_write(const float* Y, int64_t ldy, int64_t n_cells, int32_t genes, const double* n_counts,
                        double median, int32_t flags, const double* mean, const double* std, void* X, int32_t x_dtype,
                        int64_t ldx, void* stream);
/* The statistics of dca_count_totals and dca_log_moments over an n_cells-row matrix fed in row chunks (out-of-core
 * preprocessing of dca/io.py:88-111: the matrix never exists whole in device memory).  Every chunking gives the same
 * bits as the whole-matrix call: the chunk kernels run the CTA plan of the whole matrix and carry each warp's fp64
 * sums in the workspace from one chunk to the next.  A pass is dca_stats_begin, then the *_rows call for rows
 * [row0, row0 + n_rows) of every chunk -- in row order, without gaps or overlaps, Y holding those rows -- then the
 * *_finish call.  Pass 0 (totals): cell_totals (device fp64 [n_cells], or NULL) receives the chunk's per-cell totals
 * at [row0, row0 + n_rows); the finish writes gene_totals and *n_bad (either may be NULL).  Passes 1 and 2 (moments):
 * n_counts (device fp64 [n_cells], indexed by row) and median with DCA_PRE_SIZE_FACTORS; pass 2 reads the mean pass 1
 * finished; finish(1) writes the mean, finish(2) the std (without DCA_PRE_SCALE: 0 and 1; the rows calls then do
 * nothing).  The workspace (dca_stats_workspace_bytes; about slices x 8 x genes doubles, 18 MB at 20000 genes, plus
 * 8 bytes per gene block and row of the largest chunk) belongs to one pass at a time.  No atomics. */
int dca_stats_workspace_bytes(int64_t n_cells, int32_t genes, int64_t max_chunk_rows, size_t* bytes);
int dca_stats_begin(int64_t n_cells, int32_t genes, void* workspace, size_t workspace_bytes, void* stream);
int dca_count_totals_rows(const float* Y, int64_t ldy, int64_t row0, int64_t n_rows, int64_t n_cells, int32_t genes,
                          double* cell_totals, void* workspace, size_t workspace_bytes, void* stream);
int dca_count_totals_finish(int64_t n_cells, int32_t genes, double* gene_totals, int64_t* n_bad, void* workspace,
                            size_t workspace_bytes, void* stream);
int dca_log_moments_rows(int32_t pass, const float* Y, int64_t ldy, int64_t row0, int64_t n_rows, int64_t n_cells,
                         int32_t genes, const double* n_counts, double median, int32_t flags, const double* mean,
                         void* workspace, size_t workspace_bytes, void* stream);
int dca_log_moments_finish(int32_t pass, int64_t n_cells, int32_t genes, int32_t flags, double* out, void* workspace,
                           size_t workspace_bytes, void* stream);

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
 * fused hidden stack at a batch of max_batch (larger than 8192 rows: the per-layer kernels), head slots, SM count, bytes per loss-gradient element (4 fp32 | 2 bf16),
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

/* GPU writer of the same bytes (dca_b200/io.py:write_text_matrix_device) from a DEVICE float32 matrix rows x cols,
 * leading dimension ld (rows, cols >= 1): output line i holds row i, or column i with transpose != 0.  The file is
 * created (append == 0) or appended to; header_len bytes of `header` are written first as given (the caller quotes the
 * labels).  label_offsets: NULL for lines without labels, else HOST int64[out_lines + 1] into the HOST bytes `labels`
 * (already quoted): line i starts with labels[label_offsets[i] .. label_offsets[i + 1]) and a tab.  Values are
 * printf's '%.6f' of the float32 value (correctly rounded, ties to even, the sign of -0.0 and of negatives that round to
 * zero kept), NaN an empty field, infinities "inf" / "-inf", all formatted with integer arithmetic on `device`.
 * Whole lines are formatted in groups on `stream` (a length pass, one fixed-order scan, a write pass), so the bytes
 * do not depend on scheduling; the text goes to the file in pieces of at most chunk_bytes (0 = 16 MB) through two
 * pinned buffers, the write of one piece overlapping the formatting and copy of the next by a helper thread that is
 * joined before the call returns.  info (NULL or int64[4]): bytes written, line groups, microseconds of the
 * formatting kernels, microseconds spent waiting for the file writes.  Without a CUDA device it returns
 * DCA_ERR_NO_DEVICE. */
int dca_write_text_device(const char* path, int32_t append, const float* matrix, int64_t rows, int64_t cols, int64_t ld,
                          int32_t transpose, const char* header, int64_t header_len, const char* labels,
                          const int64_t* label_offsets, int64_t chunk_bytes, int32_t device, void* stream,
                          int64_t* info);
/* dca_write_text_device writing one gzip member (RFC 1952) of the same text instead: the same parameters, and the
 * file holds one more member per call with append != 0, so a matrix written in blocks of lines is a multi-member
 * gzip file whose decompressed bytes are those dca_write_text_device writes.  The header and every formatted group
 * of lines are compressed on `device` (dca_gzip_device's encoder; a group's matches do not reach into the group
 * before) before the pinned copy, so only compressed bytes cross to the host.  info[0] is the compressed bytes
 * written; the formatting microseconds in info[2] include the compression's. */
int dca_write_text_device_gz(const char* path, int32_t append, const float* matrix, int64_t rows, int64_t cols,
                             int64_t ld, int32_t transpose, const char* header, int64_t header_len, const char* labels,
                             const int64_t* label_offsets, int64_t chunk_bytes, int32_t device, void* stream,
                             int64_t* info);
/* The number formatter of dca_write_text_device run on the CPU, for tests: the '%.6f' text of the float32 bit patterns
 * bits[0..n) back to back in out (at least 47 * n bytes), that of bits[i] at out[offsets[i] .. offsets[i + 1]). */
int dca_format_fixed6_host(const uint32_t* bits, int64_t n, char* out, int64_t* offsets);

/* GPU reader of a count table in text form (dca_b200/io.py:read_counts_text): a header line, then one line per gene
 * whose first field is its label and whose other fields are counts, separated by `sep` (',' or '\t').  It gives the
 * matrix pandas.read_csv(path, sep=sep, index_col=0).values.astype(numpy.float32) gives, bit for bit, for exactly the
 * files whose
 *   - header line has as many fields as every data line, and no quote, NUL or carriage return before its line end;
 *   - lines end in '\n' or "\r\n" (the final one may have no line end), none is blank and none holds a quote or NUL;
 *   - value fields are non-empty [0-9]+ or [0-9]+\.0* with at most 18 digits (and no value above 2^53 when some
 *     field has a '.'), at most 64 bytes long;
 *   - data lines each fit in chunk_bytes.
 * Any other file returns DCA_ERR_UNSUPPORTED with the first reason in file order in dca_last_error(), and nothing is
 * returned.  Two calls with the same arguments:
 *   1. out == NULL: reads and checks the file; info[0..3] = data lines, value columns, total label bytes, device bytes
 *      the chunk buffers of the second call take besides `out`.
 *   2. out: device float32 [rows x cols] (row = data line), or [cols x rows] with transpose != 0; info as the first
 *      call returned it; label_offsets: host int64 [rows + 1]; label_bytes: host char [info[2]]: the first field of data
 *      line r is label_bytes[label_offsets[r] .. label_offsets[r + 1]), raw bytes.
 * Each call reads the file once through two pinned chunk buffers (chunk_bytes each, 0 = 64 MB), overlapping the disk
 * read with the copy and the kernels on `stream` (of `device`), and returns when they are done.  Without a CUDA
 * device it returns DCA_ERR_NO_DEVICE. */
int dca_read_text_counts(const char* path, int32_t sep, int32_t transpose, int64_t chunk_bytes, int32_t device,
                         void* stream, float* out, int64_t out_elems, int64_t* label_offsets, char* label_bytes,
                         int64_t label_cap, int64_t* info);

/* GPU reader of a Matrix Market coordinate file of counts (dca_b200/io.py:read_counts_mtx).  It gives the CSR arrays of
 * scipy.sparse.csr_matrix(scipy.io.mmread(path).astype(numpy.float32)) (of its .T.tocsr() with transpose != 0), bit for
 * bit, for exactly the files whose
 *   - first line is "%%MatrixMarket matrix coordinate integer general" or "... real general", followed by zero or more
 *     lines starting with '%' and the size line "M N NNZ" (single spaces, digits only, 1 <= M, N < 2^31);
 *   - NNZ entry lines follow, each "i j v": single spaces, 1 <= i <= M, 1 <= j <= N, v = [0-9]+ of at most 18 digits
 *     (integer) or 15 digits (real); lines end in '\n' or "\r\n", the last one may have no line end;
 *   - entries are in strictly increasing (row, column) order of the output, whose entry (row, column) is (i, j), or
 *     (j, i) with transpose: the CSR order, so there are no duplicates.  Cell Ranger's genes x cells matrix.mtx read
 *     with transpose, and scipy.io.mmwrite of a CSR cells x genes matrix read without, are in this order;
 *   - lines each fit in chunk_bytes.
 * Explicit zeros are kept.  Any other file returns DCA_ERR_UNSUPPORTED with the first reason in file order in
 * dca_last_error(), and the outputs hold nothing defined.  Two calls with the same arguments:
 *   1. indptr == NULL: reads the header only; info[0..3] = output rows, output columns, NNZ, device bytes the chunk
 *      buffers of the second call take besides the outputs.
 *   2. info as the first call returned it; device int64 indptr[rows + 1], int32 indices[NNZ], float32 data[NNZ]:
 *      one pass over the entries through two pinned chunk buffers (chunk_bytes each, 0 = 64 MB), overlapping the disk
 *      read with the copy and the kernels on `stream` (of `device`); it returns when they are done, and stops at the
 *      first chunk with a problem.  Entry k of the file goes to slot k; indptr is written without atomics.
 * File offsets, entry ordinals and indptr are 64-bit.  Without a CUDA device it returns DCA_ERR_NO_DEVICE. */
int dca_read_mtx_counts(const char* path, int32_t transpose, int64_t chunk_bytes, int32_t device, void* stream,
                        int64_t* indptr, int32_t* indices, float* data, int64_t* info);

/* The same readers over the inflated bytes of a gzip file (dca_b200/io.py:read_counts_gzip): the parameters, outputs,
 * accepted files and two calls of dca_read_text_counts and dca_read_mtx_counts, with the file inflated on `device` as
 * dca_gunzip does (each call inflates it again; info[3] includes the inflate's device memory).  A file dca_gunzip
 * declines returns DCA_ERR_UNSUPPORTED.  The entry points above keep reading compressed files as bytes. */
int dca_read_text_counts_gz(const char* path, int32_t sep, int32_t transpose, int64_t chunk_bytes, int32_t device,
                            void* stream, float* out, int64_t out_elems, int64_t* label_offsets, char* label_bytes,
                            int64_t label_cap, int64_t* info);
int dca_read_mtx_counts_gz(const char* path, int32_t transpose, int64_t chunk_bytes, int32_t device, void* stream,
                           int64_t* indptr, int32_t* indices, float* data, int64_t* info);

/* dca_read_mtx_counts and dca_read_mtx_counts_gz keeping only some features, the file's rows (dca_b200/io.py:
 * read_counts_10x drops the rows of a Cell Ranger matrix whose feature type is not "Gene Expression").  The same
 * parameters, accepted files and two calls, plus host int32 feature_map[map_len] with map_len = M (the file's rows):
 * feature_map[i - 1] is -1 to drop the entries of file row i, or the output index of its feature, which must be the
 * number of features kept before it (0, 1, 2, ... over the kept rows, so the kept entries stay in CSR order; any other
 * map returns DCA_ERR_BAD_ARG).  The output is the input's output with the dropped features taken out: with transpose
 * the map renumbers the output's columns, without it its rows.  feature_map NULL keeps every feature, with the bytes
 * of dca_read_mtx_counts / dca_read_mtx_counts_gz.
 *   1. indptr == NULL: info[0..3] = output rows, output columns (after the map), NNZ of the file (an upper bound of
 *      the kept entries, which the outputs must hold), device bytes besides the outputs.
 *   2. as before, and info[2] = the kept NNZ on return.  Kept entry k goes to slot k (a scan over the entries, carried
 *      across chunks; no atomics), and the order check applies to the kept entries only.
 * Entries of dropped rows are parsed and checked like the others. */
int dca_read_mtx_counts_map(const char* path, int32_t transpose, int64_t chunk_bytes, int32_t device, void* stream,
                            int64_t* indptr, int32_t* indices, float* data, int64_t* info, const int32_t* feature_map,
                            int64_t map_len);
int dca_read_mtx_counts_gz_map(const char* path, int32_t transpose, int64_t chunk_bytes, int32_t device, void* stream,
                               int64_t* indptr, int32_t* indices, float* data, int64_t* info,
                               const int32_t* feature_map, int64_t map_len);

/* GPU inflate of a gzip file (RFC 1952: one or more members of DEFLATE data, RFC 1951) into DEVICE memory, with no
 * zlib: the host reads the compressed file in 64 MB segments and the device decodes each segment in spans of about
 * 32 KB in parallel, speculatively from block starts it finds, then checks the chain of spans, the CRC-32 and the
 * ISIZE of every member.  Headers may have FTEXT, FEXTRA, FNAME, FCOMMENT and FHCRC (checked).  It declines
 * (DCA_ERR_UNSUPPORTED, the reason in dca_last_error()) a file that is not one or more such members back to back:
 * CM != 8, reserved flag bits, a bad FHCRC, invalid DEFLATE data, a distance before the member's start, a CRC-32 or
 * ISIZE mismatch, truncation or trailing bytes; and a file whose chain of spans needs more than 16 rounds in a segment
 * or a block longer than a segment.  Device memory does not depend on the file's size (at most about 1 GB besides
 * `out`).  Two calls with the same arguments:
 *   1. out == NULL: inflates and checks the file; info[0..3] = output bytes, device bytes this call took (the
 *      second call takes 256 MB less: it has no scratch output window), the most rounds of span decoding any segment
 *      needed (1: every speculative span was right), members.
 *   2. out: device bytes [out_bytes], out_bytes = info[0] of the first call: the same, into out.
 * Work runs on `stream` (of `device`); it returns when it is done.  Without a CUDA device: DCA_ERR_NO_DEVICE. */
int dca_gunzip(const char* path, int32_t device, void* stream, void* out, int64_t out_bytes, int64_t* info);
/* The span decoder of dca_gunzip run on the CPU, for tests: decodes in[0, n) (eof != 0: n is the end of the file) from
 * bit `start` to the first block boundary at or beyond bit `stop`, or to the end of the file's last member.  out: NULL
 * to count, else 16-bit symbols: a byte (< 0x8000), or 0x8000 | k for the byte k + 1 positions before the span's first
 * output byte.  info[0..5] = status (0 stopped at a boundary, 1 end of the file, 2 input ran out, 3 invalid), the bit
 * where it stopped, output bytes, the lowest output position a back-reference reached in the span's first member
 * (< 0 before the span), the output position of the last member starting in the span (-1: none), member trailers. */
int dca_inflate_span_host(const uint8_t* in, int64_t n, int32_t eof, int64_t start, int64_t stop, uint16_t* out,
                          int64_t out_cap, int64_t* info);
/* The block-start test of dca_gunzip on the CPU: *found = the first bit in [first_bit, end_bit) of in[0, n) where a
 * dynamic block with a fully valid header or a stored block with LEN = ~NLEN and zero padding could start, or -1. */
int dca_inflate_find_host(const uint8_t* in, int64_t n, int64_t first_bit, int64_t end_bit, int64_t* found);

/* GPU gzip compressor: one gzip member (RFC 1952; header 1f 8b 08 00, MTIME 0, XFL 0, OS 255) of the n DEVICE bytes
 * at `in`, written to DEVICE memory `out` (out_cap bytes), with no zlib.  The input is cut into blocks of 32 KB, each
 * compressed by one CTA: greedy LZ77 whose matches reach up to 32 KB back (into the blocks before), then the smallest
 * of a dynamic Huffman block (codes limited to 15 bits), a fixed Huffman block and a stored block; a non-final block
 * ends with an empty stored block so that the blocks concatenate at byte offsets.  The bytes depend on the input
 * alone, never on scheduling, and equal dca_gzip_host's.  Sizes and offsets are 64-bit (ISIZE is n mod 2^32).
 *   out == NULL: info[0] = the most bytes the member can take (18 + n + 5 per block; 20 for n = 0).
 *   out: out_cap must be at least that bound; info[0..2] = the member's bytes, blocks, stored blocks.
 * Work runs on `stream` (of `device`); it returns when it is done.  Without a CUDA device: DCA_ERR_NO_DEVICE. */
int dca_gzip_device(const void* in, int64_t n, void* out, int64_t out_cap, int32_t device, void* stream, int64_t* info);
/* The same encoder on the CPU, for tests: the same bytes from HOST in[0, n) into HOST out; out == NULL: *out_len = the
 * bound, else out_cap must be at least the bound and *out_len = the member's bytes. */
int dca_gzip_host(const void* in, int64_t n, void* out, int64_t out_cap, int64_t* out_len);

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
 * a captured step graph keeps the values it was recorded with): "loss_target_blocks" (blocks per launch of the
 * loss kernel, default 0 = auto); "fused_heads" (0 | 1, default 0): engines created afterwards
 * run head forward + loss + head backward of a zinb-conddisp training step as one fused kernel (flash_zinb.cu)
 * instead of three (environment override DCA_FUSED_HEADS); "head_bwd_banded" (0 | 1, default 1): the head backward
 * as one band-ordered launch instead of two (same bits); "head_bwd_stagger" (SM cycles, default 1300): the start delay
 * of that launch's CTAs per position in their band.  Profiling aid -- no reference counterpart. */
int dca_set_tunable(const char* name, int64_t value);

#ifdef __cplusplus
}
#endif
#endif /* DCA_B200_H */
