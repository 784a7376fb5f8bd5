// Engine: arena layout + kernel sequencing (see engine.cu).
#pragma once
#include <functional>
#include <string>
#include <vector>
#include "dca_internal.cuh"
#include "mid_stack.h"

namespace dca {

struct Layer {
  int in = 0, out = 0;
  int64_t W = -1, b = -1, beta = -1;     // element offsets into params / grads
  int64_t mm = -1, mv = -1;              // element offsets into the BN state region
  size_t o_a = 0, o_xhat = 0, o_h = 0, o_mean = 0, o_inv = 0;   // byte offsets into the arena
  int64_t alpha = -1;                    // PReLU slopes ("<layer>_act/alpha"), element offset into params / grads
  float drop = 0.f; int id = 0;          // dropout rate after the activation; mask-stream id (dca_dropout_mask_host)
};


struct Engine {
  dca_config cfg{};
  int L = 0, maxh = 1, K_head = 0;
  bool has_pi = false, cond = false;
  int64_t P = 0, S = 0;
  std::vector<dca_tensor_info> params, states;
  Layer lay[DCA_MAX_HIDDEN];
  int64_t head_W[3], head_b[3], theta_off = -1;
  // arena
  char* base = nullptr;
  size_t arena_bytes = 0;
  size_t o_params = 0, o_grads = 0, o_rms = 0, o_state = 0, o_acc = 0;
  size_t o_head[3] = {0, 0, 0}, o_dh[2] = {0, 0}, o_dsum = 0, o_dprod = 0, o_scratch = 0;
  size_t o_theta = 0, o_chain = 0, o_dtheta = 0, o_sfb = 0, o_lossws = 0, loss_ws_bytes = 0;
  size_t o_stage_x = 0, o_stage_y = 0, o_stage_sf = 0;       // == o_sx[0], o_sy[0], o_ssf[0]
  static constexpr int kExpBufs = 3;                           // expanded batches in flight (streaming path)
  size_t o_sx[kExpBufs] = {0, 0, 0}, o_sy[kExpBufs] = {0, 0, 0}, o_ssf[kExpBufs] = {0, 0, 0};
  // head input of the current forward (set by forward())
  const void* head_in = nullptr; int64_t head_ld = 0; int head_bf16 = 0; const int32_t* head_rows = nullptr;
  // CUDA-graph replay of the training step (captured from the same launch sequence on the 2nd call with a key)
  struct StepGraph {
    const void* X; int64_t ldx; const void* Y; int64_t ldy; const void* sf; int Bn; int has_rows; int phase;
    cudaGraphExec_t exec; long long launches; int seen;
  };
  std::vector<StepGraph> graphs;
  bool graphs_enabled = true;
  size_t o_rowsbuf = 0;
  int train_step_body(const void* X, int64_t ldx, const float* Y, int64_t ldy, const float* sf, const int32_t* rows, int Bn,
                      cudaStream_t s, int phase);
  // streaming from host counts
  size_t o_cnt[2] = {0, 0}, o_sfst[2] = {0, 0}, o_gmean = 0, o_ginv = 0;
  size_t o_ovp[2] = {0, 0}, o_ove[2] = {0, 0};     // overflow list of a staged batch: indptr[B+1] (int64), entries (8 B each)
  int64_t ovf_cap = 0;                              // entries per staging buffer
  size_t o_nibp[2] = {0, 0}, o_nib[2] = {0, 0}; int64_t nib_cap = 0;   // sparse format: nibble indptr (int64[B+1]) + nibble bytes per staging buffer
  int tf_use_sf = 1, tf_use_log1p = 1, tf_set = 0, x_override_bf16 = 0;
  // exact transform (dca_set_input_transform_exact): fp64 gene mean / std, X of a zero count, per-row fp64 totals of
  // each staged batch
  size_t o_gmean64 = 0, o_gstd64 = 0, o_gx0 = 0, o_ncst[2] = {0, 0};
  bool tf_exact = false; int tf_flags = 0; double tf_median = 1.0;
  float* loss_ring = nullptr; int ring_n = 0; int64_t ring_pos = 0;   // mapped host mirror of the per-step loss
  struct HostStream {
    const unsigned char* counts = nullptr; int64_t row_bytes = 0; int bits = 16;       // packed host count matrix
    const int64_t* ovf_indptr = nullptr; const unsigned char* ovf_entries = nullptr;   // host CSR overflow list (or null)
    const int64_t* nib_indptr = nullptr; const unsigned char* nibbles = nullptr;       // bits == 1: sparse format (bitmap in `counts`)
    const float* sf = nullptr; int64_t n_rows = 0; int batch = 0;
    const double* n_counts = nullptr;                 // per-row fp64 totals of the exact transform (dca_stream_row_totals)
    cudaStream_t copy = nullptr;                     // host->device copies of the next batch
    cudaStream_t expand = nullptr;                    // its expansion kernel (lowest priority: yields SMs to the step)
    cudaEvent_t h2d_done[2] = {nullptr, nullptr};     // copy stream: raw staging buffer b has arrived
    cudaEvent_t cnt_free[2] = {nullptr, nullptr};     // expand stream: raw staging buffer b has been consumed
    cudaEvent_t ready[3] = {nullptr, nullptr, nullptr};        // expand stream: batch in expanded buffer e is ready (Y, X, sf)
    cudaEvent_t step_done[3] = {nullptr, nullptr, nullptr};    // compute stream: the step that read expanded buffer e has finished
    int exp_bufs = 3;                                 // 3: the expansion of batch k+1 may run under step k-1 (2: only after it)
    int64_t pref_idx = -1, step_no = 0; bool active = false;
    // DCA_STREAM_DIAG=2: device-side timeline (events) of the first steps, printed by dca_stream_end
    std::vector<cudaEvent_t> tl; cudaEvent_t tl_base = nullptr;
    void tl_mark(cudaStream_t st) { cudaEvent_t e; if (cudaEventCreate(&e) == cudaSuccess) { cudaEventRecord(e, st); tl.push_back(e); } }
  } hs;
  int stream_prefetch(int64_t i, int raw_buf, int exp_buf);
  // element type of an expanded batch (host stream, packed counts): bf16 when X is stored in bf16, or when the
  // tensor-core encoder can read it in place.  fp32 X with input dropout stays fp32, so that the mask scales the fp32 value
  // and the encoder's gather rounds it once, bf16(x * inv_keep), as on a resident fp32 X
  int expand_bf16() const { return cfg.x_dtype == DCA_BF16 || (tc_enc && !(cfg.input_dropout > 0.f)); }
  // stored width of packed rows and of the expanded batches: n_in rounded up to a multiple of 8.  The step reads the
  // first n_in columns of an expanded batch at leading dimension g_store; the g_store - n_in pad genes are zero counts
  // that never reach the model (their mean / std entries of the exact transform are 0 / 1)
  int g_store = 0;
  // optional phase timing
  struct Prof {
    bool on = false;
    std::vector<cudaEvent_t> ev; std::vector<int> phase; size_t n = 0;
    double ms[DCA_N_PHASES] = {0, 0, 0, 0, 0, 0}; long long cnt[DCA_N_PHASES] = {0, 0, 0, 0, 0, 0};
  } prof;
  void mark(int phase, cudaStream_t s);
  int prof_collect();
  // fused hidden stack (mid_stack.cu)
  bool mid_ok = false; size_t o_bar = 0, o_midpart = 0, o_midgpart = 0;
  bool use_mid(int Bn) const { return mid_ok && !bn_synced() && Bn <= mid::kMaxRows * mid::kMaxCtas; }
  void mid_params(mid::Params& p, int Bn, bool training);
  // activations other than relu, PReLU slopes, dropout (activations.cu): per-layer hidden path only
  size_t o_step = 0, o_actscr = 0, o_xdrop = 0;       // device step counter (mask stream), PReLU scratch, dropped input batch
  bool plain_hidden() const;                          // relu and no dropout anywhere: the default model
  int bump_step(cudaStream_t s);
  int act_fwd(Layer& l, int Bn, bool training, __nv_bfloat16* hb, cudaStream_t s);
  int act_bwd(Layer& l, float* dh, int Bn, cudaStream_t s);
  int drop_input(const void* X, int in_bf16, int64_t ldx, const int32_t* rows, int Bn, cudaStream_t s);
  // tensor-core path: flags + operand-layout shadows / bf16 activations in the arena
  bool tc_heads = false, tc_enc = false;
  bool fused_heads = false;       // flash_zinb.cu replaces K2 + K3 + K4 of the training step (zinb-conddisp only)
  int sm_count = 132, n_slots = 1;
  int slot_head[3] = {0, -1, -1};          // packed head slot -> head index (0 mean, 1 dispersion, 2 pi)
  int slot_kind[3] = {0, 0, 0};
  size_t o_pbf = 0, o_h3b = 0, o_da1b = 0, o_xb = 0, o_dzb[3] = {0, 0, 0}, o_ggws = 0, ggws_bytes = 0;
  // bf16 encoder input of the current step (set by forward(), read again by the encoder backward): cell i of the batch
  // is row rows[i] of base (row i when rows is null); base == null: the encoder runs on the generic path
  struct XOperand { const __nv_bfloat16* base = nullptr; int64_t ld = 0; const int32_t* rows = nullptr; } cur_x;
  __nv_bfloat16* bf(size_t byte_off) const { return reinterpret_cast<__nv_bfloat16*>(base + byte_off); }

  // ---- remaining AE types (extra_types.cu): shape-general fp32 path, cfg.ae_type >= DCA_AE_POISSON
  int x_kind = 0;                 // 0: one of the four flagship types; else the dca_ae_type
  int n_branch = 0, trunk_L = 0;  // forks: parallel copies of the last decoder layer (mean, disp[, pi]); layers in the trunk
  Layer brlay[3];
  int head_N[3] = {0, 0, 0}, head_K[3] = {0, 0, 0};   // output width (G or 1) / input width per head (0 mean, 1 dispersion, 2 pi)
  int64_t epi_k = -1, epi_c = -1; int epi_n = 0;      // zinb-elempi: element-wise pi kernel / bias offsets, length (G or 1)
  size_t o_zraw = 0, o_small[4] = {0, 0, 0, 0}, o_xacc = 0;
  struct RegItem { int64_t off, n; bool enc; };
  std::vector<RegItem> reg_items;                     // kernels with a regulariser (dca/network.py:113-125)
  int x_plan_params(const dca_config& c, int64_t& off, int64_t& soff);
  void x_plan_arena(size_t B, const std::function<size_t(size_t)>& take);
  int x_layer_fwd(Layer& l, const void* hin, int64_t ldin, int in_bf16, const int32_t* gather, int Bn, bool training, cudaStream_t s);
  int x_layer_bwd(Layer& l, float* dh, const void* hin, int64_t ldin, int in_bf16, const int32_t* gather, int Bn, float* din,
                  bool din_accumulate, cudaStream_t s);
  const float* x_head_in(int k) const;
  int x_forward(const void* X, int64_t ldx, const int32_t* rows, int Bn, bool training, cudaStream_t s);
  int x_head_gemm(int k, int Bn, float* out, int64_t ld_out, int epi, const float* row_scale, cudaStream_t s);
  int x_heads_forward(int Bn, float* Mb, float* Db, float* Pb, const float* row_scale, cudaStream_t s);
  int x_penalty(cudaStream_t s, bool& any);
  int x_train_step_body(const void* X, int64_t ldx, const float* Y, int64_t ldy, const float* sf, const int32_t* rows, int Bn,
                        cudaStream_t s);
  int x_eval_step(const void* X, int64_t ldx, const float* Y, int64_t ldy, const float* sf, const int32_t* rows, int Bn, cudaStream_t s);
  int x_predict(const void* X, int64_t ldx, const float* sf, const int32_t* rows, int Bn, float* mean_out, float* disp_out,
                float* pi_out, int64_t ld_out, float* latent_out, cudaStream_t s);
  int x_gather_sf(const float* sf, const int32_t* rows, int Bn, cudaStream_t s);

  // data-parallel gradient exchange (comm.cu): NCCL communicator owned by the engine, resolved with dlopen
  void* comm = nullptr; int comm_world = 1, comm_rank = 0;
  int dp_reserve_sms = 0;          // phase 2 of dca_train_step_dp: SMs the hidden-stack / encoder backward leave to the collective
  bool dp_split_heads = false;     // set around phase 1 of dca_train_step_dp: head backward per head + per-head all-reduce
  cudaStream_t comm_stream = nullptr; cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  int comm_init(const void* id128, int rank, int world);
  int comm_destroy();
  static bool split_heads_enabled();       // DCA_DP_SPLIT_HEADS=1: head backward per head + per-head all-reduce (opt-in)
  int allreduce_range(int64_t lo, int64_t hi, cudaStream_t s);
  // sync_bn: sum the BatchNorm column sums (one or two double vectors) over the ranks; bn_rows(Bn) = rows behind the sums
  bool bn_synced() const { return cfg.sync_bn && comm && comm_world > 1; }
  int bn_rows(int Bn) const { return bn_synced() ? Bn * comm_world : Bn; }
  int bn_allreduce(double* a, double* b, int n, cudaStream_t s);
  int train_step_dp_body(const void* X, int64_t ldx, const float* Y, int64_t ldy, const float* sf, const int32_t* rows, int Bn,
                         cudaStream_t s);

  ~Engine();
  int plan(const dca_config& c);
  void bind(void* base_);
  float* f(size_t byte_off) const { return reinterpret_cast<float*>(base + byte_off); }
  double* d(size_t byte_off) const { return reinterpret_cast<double*>(base + byte_off); }
  float* pp(int64_t elem) const { return reinterpret_cast<float*>(base + o_params) + elem; }
  float* gp(int64_t elem) const { return reinterpret_cast<float*>(base + o_grads) + elem; }
  float* st(int64_t elem) const { return reinterpret_cast<float*>(base + o_state) + elem; }

  int gemm_auto(GemmArgs g, cudaStream_t s);
  int forward(const void* X, int64_t ldx, const int32_t* rows, int Bn, bool training, cudaStream_t s);
  int heads_forward(int Bn, float* m_out, float* d_out, float* p_out, int64_t ld_out, const float* row_scale,
                    cudaStream_t s);
  int penalty(cudaStream_t s, bool& any);
  int train_step(const void* X, int64_t ldx, const float* Y, int64_t ldy, const float* sf, const int32_t* rows, int Bn,
                 cudaStream_t s, int phase = 0);
  int apply_update(float lr, float clip, float grad_scale, cudaStream_t s);
  // optimizer of apply_update (dca_set_optimizer): Keras 2.x rules, state in o_rms (+ o_opt2), iteration count on the host
  int opt_kind = DCA_OPT_RMSPROP; long long opt_iter = 0; double nadam_sched = 1.0; size_t o_opt2 = 0;
  int reset_optimizer(cudaStream_t s);
  int eval_step(const void* X, int64_t ldx, const float* Y, int64_t ldy, const float* sf, const int32_t* rows, int Bn,
                cudaStream_t s);
  int predict(const void* X, int64_t ldx, const float* sf, const int32_t* rows, int Bn, float* mean_out, float* disp_out,
              float* pi_out, int64_t ld_out, float* latent_out, cudaStream_t s);
  int init_params(uint64_t seed, const dca_initializer& init, cudaStream_t s);

  // --debug (dca_set_debug_checks): debug_check_kernel (zinb_loss.cu) checks the reference's NB terms of every element
  // into a 48-byte report at o_dbg, cleared at the start of every training / validation step, from the operands of the
  // loss kernel, just before it.  The types whose reference loss has no such check (nb, poisson, normal) get no report
  // pointer: their report stays zero.
  bool debug_checks = false;
  size_t o_dbg = 0;
  void* debug_report() const {
    const int t = cfg.ae_type;
    return debug_checks && t != DCA_AE_NB && t != DCA_AE_POISSON && t != DCA_AE_NORMAL ? base + o_dbg : nullptr;
  }
  int debug_reset(cudaStream_t s) {
    if (void* r = debug_report()) DCA_CUDA_OK(cudaMemsetAsync(r, 0, kDebugReportBytes, s));
    return DCA_OK;
  }
  // the checks of the loss operands a loss kernel is about to read (no-op with the checks off)
  int debug_check_loss(const LossArgs& la, cudaStream_t s) {
    void* r = debug_report();
    if (!r) return DCA_OK;
    return debug_check(DebugCheckArgs{la.Y, la.ldy, la.rows, la.sf, la.m, la.ld, la.d,
                                      (la.ae_type == DCA_AE_ZINB || la.ae_type == DCA_AE_NB) ? 0 : la.ld, la.B, la.G, r}, s);
  }

  // tensor-core path hooks (dense_tc.cu)
  bool tc_supported() const;
  const char* tc_reason() const;
  int setup_tc();
  int refresh_shadows(cudaStream_t s);
};

}  // namespace dca

// the opaque handle of the C ABI (include/dca_b200.h)
struct dca_handle { dca::Engine e; void* owned = nullptr; int device = 0; };
