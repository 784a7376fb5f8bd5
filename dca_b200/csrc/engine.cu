// The engine behind the C ABI: owns the arena layout (parameters, gradients, RMSprop and
// BatchNorm state, fixed workspace) and sequences the kernels of one training / validation /
// predict batch.  Replaces what Keras Model.fit / Model.predict execute for
// dca/train.py:91-98, dca/network.py:92-141,366-393 (see include/dca_b200.h per entry point).
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <string>
#include <vector>
#include "dca_internal.cuh"
#include "engine.h"

namespace dca {

std::atomic<long long> g_launches{0};
static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

namespace {

inline size_t align_up(size_t v, size_t a = 256) { return (v + a - 1) / a * a; }

__global__ void add_double_kernel(double* p, double v) { *p += v; }
__global__ void gather_sf_kernel(const float* __restrict__ sf, const int32_t* __restrict__ rows, int n,
                                 float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = sf ? sf[rows ? rows[i] : i] : 1.0f;
}
__global__ void copy_strided_kernel(const float* __restrict__ in, int64_t ldi, float* __restrict__ out, int64_t ldo,
                                    int M, int N) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)M * N) return;
  const int r = (int)(i / N), c = (int)(i % N);
  out[(int64_t)r * ldo + c] = in[(int64_t)r * ldi + c];
}

int validate(const dca_config* c) {
  if (!c) { set_error("config is NULL"); return DCA_ERR_BAD_ARG; }
  if (c->struct_bytes != (int32_t)sizeof(dca_config)) {
    set_error("dca_config.struct_bytes=%d does not match library (%zu): header/library mismatch", c->struct_bytes,
              sizeof(dca_config));
    return DCA_ERR_BAD_ARG;
  }
  if (c->n_in <= 0 || c->n_out <= 0) { set_error("n_in/n_out must be positive (got %d, %d)", c->n_in, c->n_out); return DCA_ERR_BAD_ARG; }
  if (c->n_hidden < 0 || c->n_hidden > DCA_MAX_HIDDEN) { set_error("n_hidden must be in [0,%d]", DCA_MAX_HIDDEN); return DCA_ERR_BAD_ARG; }
  for (int i = 0; i < c->n_hidden; ++i)
    if (c->hidden[i] <= 0) { set_error("hidden[%d] must be positive", i); return DCA_ERR_BAD_ARG; }
  if (c->ae_type < 0 || c->ae_type > DCA_AE_ZINB_FORK) { set_error("autoencoder type not supported (ae_type=%d)", c->ae_type); return DCA_ERR_UNSUPPORTED; }
  if (c->max_batch <= 0) { set_error("max_batch must be positive"); return DCA_ERR_BAD_ARG; }
  if (c->x_dtype != DCA_F32 && c->x_dtype != DCA_BF16) { set_error("x_dtype must be DCA_F32 or DCA_BF16"); return DCA_ERR_BAD_ARG; }
  if (c->gemm_path < 0 || c->gemm_path > 2) { set_error("unknown gemm_path %d", c->gemm_path); return DCA_ERR_BAD_ARG; }
  if (c->activation < DCA_ACT_RELU || c->activation > DCA_ACT_PRELU) { set_error("unknown activation %d", c->activation); return DCA_ERR_BAD_ARG; }
  if (c->activation == DCA_ACT_PRELU && c->ae_type >= DCA_AE_NB_FORK) {
    // dca/network.py:711-712: the fork branches wrap the name in Activation(), which has no 'PReLU'
    set_error("activation PReLU is not available for the fork types"); return DCA_ERR_UNSUPPORTED;
  }
  if (!(c->input_dropout >= 0.f && c->input_dropout < 1.f)) { set_error("input_dropout must be in [0, 1)"); return DCA_ERR_BAD_ARG; }
  for (int i = 0; i < c->n_hidden; ++i)
    if (!(c->hidden_dropout[i] >= 0.f && c->hidden_dropout[i] < 1.f)) { set_error("hidden_dropout[%d] must be in [0, 1)", i); return DCA_ERR_BAD_ARG; }
  return DCA_OK;
}

void add_tensor(std::vector<dca_tensor_info>& v, int64_t& off, const std::string& name, int rows, int cols) {
  dca_tensor_info t;
  memset(&t, 0, sizeof(t));
  snprintf(t.name, sizeof(t.name), "%s", name.c_str());
  t.offset = off; t.rows = rows; t.cols = cols;
  off += (int64_t)rows * cols;
  v.push_back(t);
}

std::string layer_name(int i, int n) {   // dca/network.py:102-111
  const int center = n / 2;
  if (i == center) return "center";
  if (i < center) return "enc" + std::to_string(i);
  return "dec" + std::to_string(i - center);
}

}  // namespace

// ------------------------------------------------------------------------------------ layout
int Engine::plan(const dca_config& c) {
  cfg = c;
  L = c.n_hidden;
  has_pi = (c.ae_type == DCA_AE_ZINB_CONDDISP || c.ae_type == DCA_AE_ZINB);
  cond = (c.ae_type == DCA_AE_ZINB_CONDDISP || c.ae_type == DCA_AE_NB_CONDDISP);
  params.clear(); states.clear(); reg_items.clear();
  int64_t off = 0, soff = 0;
  x_kind = 0; n_branch = 0; trunk_L = L;
  if (c.ae_type >= DCA_AE_POISSON) {
    DCA_TRY(x_plan_params(c, off, soff));
  } else {
  int prev = c.n_in;
  maxh = 1;
  for (int i = 0; i < L; ++i) {
    const std::string nm = layer_name(i, L);
    const int h = c.hidden[i];
    lay[i].in = prev; lay[i].out = h;
    lay[i].W = off; add_tensor(params, off, nm + "/kernel", prev, h);
    lay[i].b = off; add_tensor(params, off, nm + "/bias", 1, h);
    if (c.batchnorm) {
      lay[i].beta = off; add_tensor(params, off, nm + "/bn_beta", 1, h);
      lay[i].mm = soff; add_tensor(states, soff, nm + "/bn_moving_mean", 1, h);
      lay[i].mv = soff; add_tensor(states, soff, nm + "/bn_moving_var", 1, h);
    }
    if (c.activation == DCA_ACT_PRELU) { lay[i].alpha = off; add_tensor(params, off, nm + "_act/alpha", 1, h); }
    lay[i].drop = c.hidden_dropout[i]; lay[i].id = i;
    prev = h;
    if (h > maxh) maxh = h;
  }
  K_head = prev;
  head_W[0] = off; add_tensor(params, off, "mean/kernel", prev, c.n_out);
  head_b[0] = off; add_tensor(params, off, "mean/bias", 1, c.n_out);
  head_W[1] = head_b[1] = head_W[2] = head_b[2] = theta_off = -1;
  if (cond) {
    head_W[1] = off; add_tensor(params, off, "dispersion/kernel", prev, c.n_out);
    head_b[1] = off; add_tensor(params, off, "dispersion/bias", 1, c.n_out);
  }
  if (has_pi) {
    head_W[2] = off; add_tensor(params, off, "pi/kernel", prev, c.n_out);
    head_b[2] = off; add_tensor(params, off, "pi/bias", 1, c.n_out);
  }
  if (!cond) { theta_off = off; add_tensor(params, off, "dispersion/theta", 1, c.n_out); }
  }
  P = off; S = soff;

  // ---- arena carve-up
  const int G = c.n_out;
  const size_t B = (size_t)c.max_batch;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t at = o; o = align_up(o + bytes); return at; };
  o_params = take(sizeof(float) * (size_t)P);
  o_grads = take(sizeof(float) * (size_t)(P + 2));
  o_rms = take(sizeof(float) * (size_t)P);
  o_opt2 = take(sizeof(float) * (size_t)P);   // second accumulator of Adadelta / Adam / Adamax / Nadam (12 MB at 20k genes)
  o_state = take(sizeof(float) * (size_t)(S > 0 ? S : 1));
  o_acc = take(sizeof(double) * 8);          // epoch acc[4], loss_sum, penalty
  for (int i = 0; i < L; ++i) {
    const size_t h = (size_t)c.hidden[i];
    lay[i].o_a = take(sizeof(float) * B * h);
    lay[i].o_xhat = take(sizeof(float) * B * h);
    lay[i].o_h = take(sizeof(float) * B * h);
    lay[i].o_mean = take(sizeof(float) * h);
    lay[i].o_inv = take(sizeof(float) * h);
  }
  for (int k = 0; k < 3; ++k) o_head[k] = take(sizeof(float) * B * (size_t)G);
  o_dh[0] = take(sizeof(float) * B * (size_t)maxh);
  o_dh[1] = take(sizeof(float) * B * (size_t)maxh);
  const size_t statw = (size_t)(maxh > G ? maxh : G);
  o_dsum = take(sizeof(double) * statw);
  o_dprod = take(sizeof(double) * statw);
  o_scratch = take(sizeof(double) * (size_t)col_sums_scratch_elems((int)B, (int)statw));
  o_theta = take(sizeof(float) * (size_t)G);
  o_chain = take(sizeof(float) * (size_t)G);
  o_dtheta = take(sizeof(float) * (size_t)G);
  o_sfb = take(sizeof(float) * B);
  loss_ws_bytes = loss_workspace_bytes((int)B, G);
  o_lossws = take(loss_ws_bytes);
  o_rowsbuf = take(sizeof(int32_t) * B);
  o_step = take(256);
  if (c.activation == DCA_ACT_PRELU) o_actscr = take(sizeof(float) * B * (size_t)maxh);
  if (c.input_dropout > 0.f) o_xdrop = take((c.x_dtype == DCA_BF16 ? sizeof(__nv_bfloat16) : sizeof(float)) * B * (size_t)c.n_in);
  mid_ok = !x_kind && plain_hidden() && mid_supported(c.hidden, L);     // the one-launch hidden stack is relu-only, no dropout
  o_bar = take(256);
  o_midpart = take(sizeof(double) * mid_partial_doubles());
  o_midgpart = take(sizeof(float) * mid_grad_partial_floats(L));
  // tensor-core path (flagship shape): gene-wide layers with a 64-wide partner dimension
  n_slots = 0;
  slot_head[0] = 0; slot_kind[0] = EPI_MEAN_ACT; n_slots = 1;
  if (cond) { slot_head[n_slots] = 1; slot_kind[n_slots] = EPI_DISP_ACT; ++n_slots; }
  if (has_pi) { slot_head[n_slots] = 2; slot_kind[n_slots] = EPI_SIGMOID; ++n_slots; }
  const bool want_tc = c.gemm_path != DCA_GEMM_GENERIC && !x_kind;     // the extra AE types run the shape-general fp32 path
  tc_heads = want_tc && L >= 1 && K_head == 64 && (G % 8 == 0);
  tc_enc = want_tc && L >= 1 && c.hidden[0] == 64 && (c.n_in % 8 == 0);
  // the tensor-core kernels read the kernels in place from the flat bf16 parameter copy: TMA needs 16-byte aligned bases
  if (tc_heads) for (int k = 0; k < 3; ++k) if (head_W[k] >= 0 && (head_W[k] % 8) != 0) tc_heads = false;
  {
    const char* ev = getenv("DCA_FUSED_HEADS");
    const bool want = ev ? atoi(ev) != 0 : g_fused_heads_default != 0;
    fused_heads = want && tc_heads && cond && has_pi && L >= 1 && (G % 8 == 0);
  }
  if (tc_enc && (lay[0].W % 8) != 0) tc_enc = false;
  if (tc_heads || tc_enc) o_pbf = take(2 * (size_t)P);       // bf16 copy of the parameters, same flat layout
  if (tc_heads || tc_enc) { ggws_bytes = tc::gene_gemm_workspace_bytes((int)B); o_ggws = take(ggws_bytes); }
  if (tc_heads) {
    o_h3b = take(2 * B * 64);
    for (int k = 0; k < n_slots; ++k) o_dzb[k] = take(2 * B * (size_t)G);
  }
  if (tc_enc) {
    o_da1b = take(2 * B * 64);
    o_xb = take(2 * B * (size_t)c.n_in);
  }
  // double-buffered staging of raw uint16 counts streamed from the host + the input transform
  for (int k = 0; k < 2; ++k) { o_cnt[k] = take(sizeof(uint16_t) * B * (size_t)c.n_in); o_sfst[k] = take(sizeof(float) * B); }
  ovf_cap = (int64_t)(B * (size_t)c.n_in / 32); if (ovf_cap < 4096) ovf_cap = 4096;
  for (int k = 0; k < 2; ++k) { o_ovp[k] = take(sizeof(int64_t) * (B + 1)); o_ove[k] = take(8 * (size_t)ovf_cap); }
  nib_cap = (int64_t)(B * (size_t)c.n_in / 4) + 64;       // sparse format: up to 50 % non-zero entries per batch
  for (int k = 0; k < 2; ++k) { o_nibp[k] = take(sizeof(int64_t) * (B + 1)); o_nib[k] = take((size_t)nib_cap); }
  o_gmean = take(sizeof(float) * (size_t)c.n_in); o_ginv = take(sizeof(float) * (size_t)c.n_in);
  // staging for the host-buffer entry point
  const size_t xb = (c.x_dtype == DCA_BF16) ? 2 : 4;
  for (int k = 0; k < kExpBufs; ++k) {
    o_sx[k] = take(xb * B * (size_t)c.n_in);
    o_sy[k] = take(sizeof(float) * B * (size_t)G);
    o_ssf[k] = take(sizeof(float) * B);
  }
  o_stage_x = o_sx[0]; o_stage_y = o_sy[0]; o_stage_sf = o_ssf[0];
  if (x_kind) x_plan_arena(B, take);
  arena_bytes = o;
  return DCA_OK;
}

void Engine::mark(int phase, cudaStream_t s) {
  if (!prof.on) return;
  if (prof.n == prof.ev.size()) {
    cudaEvent_t e;
    if (cudaEventCreate(&e) != cudaSuccess) return;
    prof.ev.push_back(e); prof.phase.push_back(-1);
  }
  prof.phase[prof.n] = phase;
  cudaEventRecord(prof.ev[prof.n], s);
  ++prof.n;
}

int Engine::prof_collect() {
  if (prof.n == 0) return DCA_OK;
  DCA_CUDA_OK(cudaEventSynchronize(prof.ev[prof.n - 1]));
  for (size_t i = 0; i + 1 < prof.n; ++i) {
    const int ph = prof.phase[i];
    if (ph < 0 || ph >= DCA_N_PHASES) continue;
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, prof.ev[i], prof.ev[i + 1]) == cudaSuccess) { prof.ms[ph] += ms; prof.cnt[ph] += 1; }
  }
  prof.n = 0;
  return DCA_OK;
}

void Engine::bind(void* base_) {
  base = reinterpret_cast<char*>(base_);
}

// ------------------------------------------------------------------------------------ forward
int Engine::gemm_auto(GemmArgs g, cudaStream_t s) {
  // split-K so that skinny outputs still fill the SMs: at least two tiles per SM
  const long long tiles = (long long)cdiv(g.M, 64) * cdiv(g.N, 64), target = 2ll * sm_count;
  int splits = 1;
  if (g.epilogue == EPI_ACCUM && tiles < target && g.K >= 256) {
    splits = (int)((target + tiles - 1) / tiles);
    const int maxs = g.K / 128;
    if (splits > maxs) splits = maxs;
    if (splits < 1) splits = 1;
  }
  g.splits = splits;
  return gemm_generic(g, s);
}

int Engine::forward(const void* X, int64_t ldx, const int32_t* rows, int Bn, bool training, cudaStream_t s) {
  const void* hin = X; int64_t ldin = ldx; int in_bf16 = x_override_bf16 ? 1 : (cfg.x_dtype == DCA_BF16); const int32_t* gather = rows;
  // tensor-core encoder: needs a contiguous bf16 batch (gathered / converted once, reused by the backward pass)
  cur_xb = nullptr;
  if (tc_enc) {
    const bool direct = in_bf16 && !rows && (ldx % 8 == 0) && ((reinterpret_cast<uintptr_t>(X) & 15) == 0);
    const bool can_gather = (ldx % (in_bf16 ? 8 : 4) == 0) && ((reinterpret_cast<uintptr_t>(X) & 15) == 0);
    if (direct) { cur_xb = reinterpret_cast<const __nv_bfloat16*>(X); cur_ldxb = ldx; }
    else if (can_gather) {
      DCA_TRY(gather_rows_bf16(X, in_bf16, ldx, rows, Bn, cfg.n_in, bf(o_xb), s));
      cur_xb = bf(o_xb); cur_ldxb = cfg.n_in;
    }
  }
  const bool fused = use_mid(Bn);
  for (int i = 0; i < (fused ? 1 : L); ++i) {
    Layer& l = lay[i];
    float* a = f(l.o_a);
    DCA_TRY(fill_rows_with_bias(a, l.out, Bn, l.out, pp(l.b), s));
    if (i == 0 && cur_xb) {
      const __nv_bfloat16* Z[3] = {cur_xb, cur_xb, cur_xb};
      const __nv_bfloat16* W1[3] = {bf(o_pbf) + lay[0].W, bf(o_pbf) + lay[0].W, bf(o_pbf) + lay[0].W};
      DCA_TRY(tc::gene_gemm_tc(1, Z, cur_ldxb, Bn, cfg.n_in, 1, nullptr, W1, a, nullptr, 0, 0, nullptr, base + o_ggws, ggws_bytes, sm_count, s));
    } else {
    GemmArgs g{};
    g.A = hin; g.lda = ldin; g.a_bf16 = in_bf16; g.transA = 0; g.a_rows = gather;
    g.B = pp(l.W); g.ldb = l.out; g.transB = 0;
    g.C = a; g.ldc = l.out; g.M = Bn; g.N = l.out; g.K = l.in; g.epilogue = EPI_ACCUM;
    DCA_TRY(gemm_auto(g, s));
    }
    if (fused) break;                 // BN / relu / inner layers: one fused launch below
    if (cfg.batchnorm) {
      if (training) {
        DCA_TRY(col_sums(a, nullptr, l.out, Bn, l.out, d(o_dsum), d(o_dprod), d(o_scratch), s));
        DCA_TRY(bn_allreduce(d(o_dsum), d(o_dprod), l.out, s));                  // sync_bn: statistics of the global batch
        DCA_TRY(bn_train_finalize(d(o_dsum), d(o_dprod), bn_rows(Bn), l.out, cfg.bn_eps, cfg.bn_momentum, f(l.o_mean),
                                  f(l.o_inv), st(l.mm), st(l.mv), s));
      } else {
        DCA_TRY(bn_infer_prepare(st(l.mm), st(l.mv), l.out, cfg.bn_eps, f(l.o_mean), f(l.o_inv), s));
      }
    }
    DCA_TRY(act_fwd(l, Bn, training, (tc_heads && i == L - 1) ? bf(o_h3b) : nullptr, s));
    hin = f(l.o_h); ldin = l.out; in_bf16 = 0; gather = nullptr;
  }
  if (fused) {
    mid::Params mp;
    mid_params(mp, Bn, training);
    DCA_TRY(mid_forward(mp, s));
    hin = f(lay[L - 1].o_h); ldin = lay[L - 1].out; in_bf16 = 0; gather = nullptr;
  }
  head_in = hin; head_ld = ldin; head_bf16 = in_bf16; head_rows = gather;
  return DCA_OK;
}

int Engine::x_gather_sf(const float* sf, const int32_t* rows, int Bn, cudaStream_t s) {
  gather_sf_kernel<<<cdiv(Bn, 256), 256, 0, s>>>(sf, rows, Bn, f(o_sfb));
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

void Engine::mid_params(mid::Params& p, int Bn, bool training) {
  memset(&p, 0, sizeof(p));
  p.L = L; p.B = Bn; p.training = training ? 1 : 0; p.batchnorm = cfg.batchnorm; p.center = L / 2;
  for (int i = 0; i < L; ++i) {
    Layer& l = lay[i];
    p.w[i] = l.out; p.W[i] = pp(l.W); p.b[i] = pp(l.b);
    p.beta[i] = cfg.batchnorm ? pp(l.beta) : nullptr;
    p.mm[i] = cfg.batchnorm ? st(l.mm) : nullptr; p.mv[i] = cfg.batchnorm ? st(l.mv) : nullptr;
    p.mean[i] = f(l.o_mean); p.inv[i] = f(l.o_inv); p.xhat[i] = f(l.o_xhat); p.h[i] = f(l.o_h);
    p.gW[i] = gp(l.W); p.gb[i] = gp(l.b); p.gbeta[i] = cfg.batchnorm ? gp(l.beta) : nullptr;
  }
  p.a0 = f(lay[0].o_a); p.a_center = f(lay[L / 2].o_a);
  p.h_last_bf16 = tc_heads ? bf(o_h3b) : nullptr;
  p.partial = d(o_midpart); p.gpart = f(o_midgpart); p.bar = reinterpret_cast<unsigned*>(base + o_bar);
  p.eps = cfg.bn_eps; p.momentum = cfg.bn_momentum;
}

int Engine::heads_forward(int Bn, float* m_out, float* d_out, float* p_out, int64_t ld_out, const float* row_scale,
                          cudaStream_t s) {
  const int G = cfg.n_out;
  if (tc_heads && (ld_out % 4 == 0)) {
    float* outs_by_head[3] = {m_out, d_out, p_out};
    bool all = true;
    for (int k = 0; k < n_slots; ++k) all = all && outs_by_head[slot_head[k]] && ((reinterpret_cast<uintptr_t>(outs_by_head[slot_head[k]]) & 15) == 0);
    if (all) {
      float* outs[3] = {nullptr, nullptr, nullptr};
      for (int k = 0; k < n_slots; ++k) outs[k] = outs_by_head[slot_head[k]];
      for (int k = n_slots; k < 3; ++k) outs[k] = outs[0];
      const __nv_bfloat16* Wk[3]; const float* bk[3];
      for (int k = 0; k < 3; ++k) { const int kk = k < n_slots ? k : 0; Wk[k] = bf(o_pbf) + head_W[slot_head[kk]]; bk[k] = pp(head_b[slot_head[kk]]); }
      return tc::heads_fwd_tc(bf(o_h3b), Bn, Wk, bk, G, n_slots, slot_kind, row_scale, outs, ld_out, sm_count, s);
    }
  }
  struct H { int k; float* out; int epi; const float* rs; } hs[3] = {
      {0, m_out, EPI_MEAN_ACT, row_scale}, {1, d_out, EPI_DISP_ACT, nullptr}, {2, p_out, EPI_SIGMOID, nullptr}};
  for (auto& h : hs) {
    if (head_W[h.k] < 0 || !h.out) continue;
    GemmArgs g{};
    g.A = head_in; g.lda = head_ld; g.a_bf16 = head_bf16; g.transA = 0; g.a_rows = head_rows;
    g.B = pp(head_W[h.k]); g.ldb = G; g.transB = 0;
    g.C = h.out; g.ldc = ld_out; g.M = Bn; g.N = G; g.K = K_head;
    g.bias = pp(head_b[h.k]); g.row_scale = h.rs; g.epilogue = h.epi; g.splits = 1;
    DCA_TRY(gemm_generic(g, s));
  }
  return DCA_OK;
}

int Engine::penalty(cudaStream_t s, bool& any) {
  any = false;
  auto coeff = [&](int i, float& l1, float& l2) {   // dca/network.py:113-122
    const int center = L / 2;
    const bool enc = (i >= 0 && i <= center);
    l1 = (enc && cfg.l1_enc != 0.f) ? cfg.l1_enc : cfg.l1;
    l2 = (enc && cfg.l2_enc != 0.f) ? cfg.l2_enc : cfg.l2;
  };
  for (int i = 0; i < L; ++i) {
    float l1, l2; coeff(i, l1, l2);
    if (l1 != 0.f || l2 != 0.f) any = true;
  }
  if (cfg.l1 != 0.f || cfg.l2 != 0.f) any = true;
  if (!any) return DCA_OK;
  DCA_CUDA_OK(cudaMemsetAsync(d(o_acc) + 5, 0, sizeof(double), s));
  for (int i = 0; i < L; ++i) {
    float l1, l2; coeff(i, l1, l2);
    if (l1 == 0.f && l2 == 0.f) continue;
    const int64_t n = (int64_t)lay[i].in * lay[i].out;
    DCA_TRY(reg_penalty(pp(lay[i].W), n, l1, l2, d(o_acc) + 5, s));
    DCA_TRY(add_reg_grad(pp(lay[i].W), gp(lay[i].W), n, l1, l2, s));
  }
  if (cfg.l1 != 0.f || cfg.l2 != 0.f) {
    for (int k = 0; k < 3; ++k) {
      if (head_W[k] < 0) continue;
      const int64_t n = (int64_t)K_head * cfg.n_out;
      DCA_TRY(reg_penalty(pp(head_W[k]), n, cfg.l1, cfg.l2, d(o_acc) + 5, s));
      DCA_TRY(add_reg_grad(pp(head_W[k]), gp(head_W[k]), n, cfg.l1, cfg.l2, s));
    }
  }
  return DCA_OK;
}

// ------------------------------------------------------------------------------------ train step
int Engine::train_step(const void* X, int64_t ldx, const float* Y, int64_t ldy, const float* sf, const int32_t* rows,
                       int Bn, cudaStream_t s, int phase) {
  if (phase < 0 || phase > 3) { set_error("dca_train_step: phase must be 0, 1, 2 or 3"); return DCA_ERR_BAD_ARG; }
  if (!X || !Y) { set_error("dca_train_step: X and Y must not be NULL"); return DCA_ERR_BAD_ARG; }
  if (Bn <= 0 || Bn > cfg.max_batch) { set_error("dca_train_step: batch %d outside (0, max_batch=%d]", Bn, cfg.max_batch); return DCA_ERR_BAD_ARG; }
  // the legacy default stream (handle 0) cannot be captured: stay on the direct path there
  if (!graphs_enabled || prof.on || s == nullptr || s == cudaStreamLegacy || s == cudaStreamPerThread)
    return phase == 3 ? train_step_dp_body(X, ldx, Y, ldy, sf, rows, Bn, s) : train_step_body(X, ldx, Y, ldy, sf, rows, Bn, s, phase);
  // ---- CUDA-graph replay: the launch sequence only depends on (pointers, leading dims, batch); the batch's row
  // indices are copied into a fixed buffer so that the captured kernels read them from a stable address.
  StepGraph* g = nullptr;
  for (auto& c : graphs)
    if (c.X == X && c.ldx == ldx && c.Y == Y && c.ldy == ldy && c.sf == sf && c.Bn == Bn && c.has_rows == (rows != nullptr) && c.phase == phase) { g = &c; break; }
  if (!g) {
    if (graphs.size() >= 16) { for (auto& c : graphs) if (c.exec) cudaGraphExecDestroy(c.exec); graphs.clear(); }
    graphs.push_back(StepGraph{X, ldx, Y, ldy, sf, Bn, rows != nullptr, phase, nullptr, 0, 0});
    g = &graphs.back();
  }
  int32_t* rbuf = reinterpret_cast<int32_t*>(base + o_rowsbuf);
  if (!g->exec && g->seen >= 1 && g->seen < 1000) {
    // capture on the second call with this key (the first, direct call has done every one-time initialisation)
    const long long l0 = g_launches.load();
    if (cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
      const int st = phase == 3 ? train_step_dp_body(X, ldx, Y, ldy, sf, rows ? rbuf : nullptr, Bn, s)
                                : train_step_body(X, ldx, Y, ldy, sf, rows ? rbuf : nullptr, Bn, s, phase);
      cudaGraph_t graph = nullptr;
      const cudaError_t ce = cudaStreamEndCapture(s, &graph);
      if (st == DCA_OK && ce == cudaSuccess && graph && cudaGraphInstantiate(&g->exec, graph, 0) == cudaSuccess) {
        g->launches = g_launches.load() - l0;
        g_launches.store(l0);                      // the capture itself launched nothing
      } else {
        if (getenv("DCA_GRAPH_DEBUG"))
          fprintf(stderr, "[dca_b200] graph capture failed: body status %d (%s), end-capture %s\n", st, g_err,
                  cudaGetErrorString(ce));
        g->exec = nullptr; g->seen = 1000;         // not capturable: stay on the direct path for this key
        (void)cudaGetLastError();
      }
      if (graph) cudaGraphDestroy(graph);
    } else {
      if (getenv("DCA_GRAPH_DEBUG")) fprintf(stderr, "[dca_b200] cudaStreamBeginCapture failed: %s\n", cudaGetErrorString(cudaGetLastError()));
      (void)cudaGetLastError(); g->seen = 1000;
    }
  }
  if (g->exec) {
    if (rows && phase != 2) DCA_CUDA_OK(cudaMemcpyAsync(rbuf, rows, sizeof(int32_t) * (size_t)Bn, cudaMemcpyDeviceToDevice, s));
    DCA_CUDA_OK(cudaGraphLaunch(g->exec, s));
    count_launch((int)g->launches);
    return DCA_OK;
  }
  if (g->seen < 1000) ++g->seen;
  return phase == 3 ? train_step_dp_body(X, ldx, Y, ldy, sf, rows, Bn, s) : train_step_body(X, ldx, Y, ldy, sf, rows, Bn, s, phase);
}

// phase 0: whole step; 1: forward + loss + head backward (the head gradients -- 98 % of the parameters -- are then
// final, so their all-reduce can overlap phase 2); 2: hidden-stack / encoder backward.
int Engine::train_step_body(const void* X, int64_t ldx, const float* Y, int64_t ldy, const float* sf, const int32_t* rows,
                            int Bn, cudaStream_t s, int phase) {
  if (x_kind) return phase == 2 ? DCA_OK : x_train_step_body(X, ldx, Y, ldy, sf, rows, Bn, s);   // whole step in phase 1
  const int G = cfg.n_out;
  float* dh = f(o_dh[0]); float* dh2 = f(o_dh[1]);
  // input dropout: the network reads a masked, gathered copy of the batch (forward and encoder backward); Y keeps `rows`
  const int32_t* xrows = rows;
  if (cfg.input_dropout > 0.f) {
    if (phase != 2) {
      DCA_TRY(bump_step(s));
      DCA_TRY(drop_input(X, x_override_bf16 ? 1 : (cfg.x_dtype == DCA_BF16), ldx, rows, Bn, s));
    }
    X = base + o_xdrop; ldx = cfg.n_in; xrows = nullptr;
  } else if (phase != 2 && !plain_hidden()) DCA_TRY(bump_step(s));
  if (phase != 2) {
  DCA_CUDA_OK(cudaMemsetAsync(gp(0), 0, sizeof(float) * (size_t)(P + 2), s));
  bool any_pen = false;
  mark(0, s);
  DCA_TRY(penalty(s, any_pen));
  DCA_TRY(forward(X, ldx, xrows, Bn, true, s));
  mark(1, s);
  float* Mb = f(o_head[0]); float* Db = f(o_head[1]); float* Pb = f(o_head[2]);
  const float inv_n = 1.0f / ((float)Bn * (float)G);
  const bool fuse = fused_heads && (ldy % 4 == 0) && ((reinterpret_cast<uintptr_t>(Y) & 15) == 0);
  if (fuse) {
    // heads forward + loss + head backward in ONE kernel (flash_zinb.cu): no B x G tensor reaches HBM
    mark(2, s);
    DCA_CUDA_OK(cudaMemsetAsync(dh, 0, sizeof(float) * (size_t)Bn * K_head, s));
    const float* lf_dev = loss_log_fact_table();
    if (!lf_dev) return DCA_ERR_CUDA;
    const __nv_bfloat16* Wk[3]; const float* bk[3]; float* dWp[3]; float* dbp[3];
    for (int k = 0; k < 3; ++k) { Wk[k] = bf(o_pbf) + head_W[k]; bk[k] = pp(head_b[k]); dWp[k] = gp(head_W[k]); dbp[k] = gp(head_b[k]); }
    DCA_TRY(tc::flash_zinb_tc(bf(o_h3b), Bn, G, Wk, bk, Y, ldy, rows, sf, cfg.ridge, inv_n, dh, dWp, dbp, base + o_lossws,
                              loss_ws_bytes, d(o_acc) + 4, any_pen ? d(o_acc) + 5 : nullptr, gp(P), d(o_acc), Bn, lf_dev,
                              sm_count, s));
  } else {
  DCA_TRY(heads_forward(Bn, Mb, cond ? Db : nullptr, has_pi ? Pb : nullptr, G, nullptr, s));
  if (!cond) DCA_TRY(theta_prepare(pp(theta_off), G, f(o_theta), f(o_chain), s));
  mark(2, s);

  LossArgs la{};
  la.Y = Y; la.ldy = ldy; la.rows = rows; la.sf = sf;
  la.m = Mb; la.d = cond ? Db : f(o_theta); la.pi = has_pi ? Pb : nullptr; la.ld = G;
  la.B = Bn; la.G = G; la.ae_type = cfg.ae_type; la.ridge = cfg.ridge; la.inv_n = inv_n;
  la.dzm = Mb; la.dzd = cond ? Db : nullptr; la.dzp = has_pi ? Pb : nullptr; la.grad_bf16 = 0;
  if (tc_heads) {          // bf16 gradients for the tensor-core head-backward kernel, packed-slot order
    void* slot_buf[3] = {nullptr, nullptr, nullptr};
    for (int k = 0; k < n_slots; ++k) slot_buf[slot_head[k]] = bf(o_dzb[k]);
    la.dzm = slot_buf[0]; la.dzd = cond ? slot_buf[1] : nullptr; la.dzp = has_pi ? slot_buf[2] : nullptr; la.grad_bf16 = 1;
  }
  la.dtheta = cond ? nullptr : f(o_dtheta);
  la.loss_sum = d(o_acc) + 4; la.ws = base + o_lossws; la.ws_bytes = loss_ws_bytes;
  la.counter_ready = 1;
  la.fin_loss_slot = gp(P); la.fin_epoch_acc = d(o_acc); la.fin_penalty = any_pen ? d(o_acc) + 5 : nullptr; la.fin_batch = Bn;
  DCA_TRY(zinb_loss_fwd_bwd(la, s));
  if (!cond) {
    // dtheta currently holds sum over rows of dL/dtheta (not / N)
    DCA_TRY(theta_grad_finish(f(o_dtheta), f(o_chain), G, inv_n, gp(theta_off), s));
  }

  // ---- head backward
  mark(3, s);
  if (L > 0) DCA_CUDA_OK(cudaMemsetAsync(dh, 0, sizeof(float) * (size_t)Bn * K_head, s));
  float* dz[3] = {Mb, cond ? Db : nullptr, has_pi ? Pb : nullptr};
  if (tc_heads) {
    const __nv_bfloat16* Z[3]; const __nv_bfloat16* Wk[3]; float* dWp[3]; float* dbp[3];
    for (int k = 0; k < 3; ++k) {
      const int kk = k < n_slots ? k : 0;
      Z[k] = bf(o_dzb[kk]); Wk[k] = bf(o_pbf) + head_W[slot_head[kk]];
      dWp[k] = gp(head_W[slot_head[kk]]); dbp[k] = gp(head_b[slot_head[kk]]);
    }
    if (dp_split_heads && comm && n_slots > 1) {
      // data-parallel step: one head-backward launch PER HEAD, each followed by the all-reduce of that head's kernel + bias
      // gradients on the communicator stream -- two thirds of the gradient bytes travel under the remaining head-backward
      // launches, the last third under the hidden-stack / encoder backward (comm.cu: train_step_dp_body)
      for (int k = 0; k < n_slots; ++k) {
        const __nv_bfloat16* Z1[3] = {Z[k], Z[k], Z[k]}; const __nv_bfloat16* W1[3] = {Wk[k], Wk[k], Wk[k]};
        float* dW1[3] = {dWp[k], dWp[k], dWp[k]}; float* db1[3] = {dbp[k], dbp[k], dbp[k]};
        DCA_TRY(tc::gene_gemm_tc(3, Z1, G, Bn, G, 1, bf(o_h3b), W1, dh, dW1, G, 1, db1, base + o_ggws, ggws_bytes, sm_count, s));
        const int h = slot_head[k];
        DCA_CUDA_OK(cudaEventRecord(ev_fork, s));
        DCA_CUDA_OK(cudaStreamWaitEvent(comm_stream, ev_fork, 0));
        DCA_TRY(allreduce_range(head_W[h], head_b[h] + G, comm_stream));
      }
    } else
    DCA_TRY(tc::gene_gemm_tc(3, Z, G, Bn, G, n_slots, bf(o_h3b), Wk, dh, dWp, G, 1, dbp, base + o_ggws, ggws_bytes, sm_count, s));
  } else
  for (int k = 0; k < 3; ++k) {
    if (head_W[k] < 0 || !dz[k]) continue;
    GemmArgs g{};
    g.A = head_in; g.lda = head_ld; g.a_bf16 = head_bf16; g.transA = 1; g.a_rows = head_rows;
    g.B = dz[k]; g.ldb = G; g.transB = 0;
    g.C = gp(head_W[k]); g.ldc = G; g.M = K_head; g.N = G; g.K = Bn; g.epilogue = EPI_ACCUM;
    DCA_TRY(gemm_auto(g, s));
    DCA_TRY(col_sums(dz[k], nullptr, G, Bn, G, d(o_dsum), nullptr, d(o_scratch), s));
    DCA_TRY(col_sum_to_float(d(o_dsum), G, gp(head_b[k]), s));
    if (L > 0) {
      GemmArgs b{};
      b.A = dz[k]; b.lda = G; b.a_bf16 = 0; b.transA = 0; b.a_rows = nullptr;
      b.B = pp(head_W[k]); b.ldb = G; b.transB = 1;
      b.C = dh; b.ldc = K_head; b.M = Bn; b.N = K_head; b.K = G; b.epilogue = EPI_ACCUM;
      DCA_TRY(gemm_auto(b, s));
    }
  }
  }  // !fuse
  }  // phase != 2
  if (phase == 1) { mark(-1, s); return DCA_OK; }
  // ---- hidden stack backward
  mark(4, s);
  if (L > 0 && use_mid(Bn)) {
    mid::Params mp;
    mid_params(mp, Bn, true);
    mp.dh_last = dh; mp.da0 = dh2; mp.da0_bf16 = cur_xb ? bf(o_da1b) : nullptr;
    mp.max_ctas = dp_reserve_sms ? (sm_count - dp_reserve_sms) : 0;
    DCA_TRY(mid_backward(mp, s));
    Layer& l = lay[0];
    if (cur_xb) {
      const __nv_bfloat16* Z[3] = {cur_xb, cur_xb, cur_xb};
      float* dWp[3] = {gp(l.W), gp(l.W), gp(l.W)};
      DCA_TRY(tc::gene_gemm_tc(2, Z, cur_ldxb, Bn, cfg.n_in, 1, bf(o_da1b), nullptr, nullptr, dWp, l.out, 0, nullptr, nullptr, 0, sm_count - dp_reserve_sms, s));
    } else {
      GemmArgs g{};
      g.A = X; g.lda = ldx; g.a_bf16 = x_override_bf16 ? 1 : (cfg.x_dtype == DCA_BF16); g.transA = 1; g.a_rows = xrows;
      g.B = dh2; g.ldb = l.out; g.transB = 0;
      g.C = gp(l.W); g.ldc = l.out; g.M = l.in; g.N = l.out; g.K = Bn; g.epilogue = EPI_ACCUM;
      DCA_TRY(gemm_auto(g, s));
    }
  } else
  for (int i = L - 1; i >= 0; --i) {
    Layer& l = lay[i];
    DCA_TRY(act_bwd(l, dh, Bn, s));
    if (cfg.batchnorm) {
      DCA_TRY(col_sums(dh, f(l.o_xhat), l.out, Bn, l.out, d(o_dsum), d(o_dprod), d(o_scratch), s));
      if (bn_synced()) {          // d beta is this rank's share (the gradient all-reduce sums it); the means are global
        DCA_TRY(col_sum_to_float(d(o_dsum), l.out, gp(l.beta), s));
        DCA_TRY(bn_allreduce(d(o_dsum), d(o_dprod), l.out, s));
        DCA_TRY(bn_bwd_apply(dh, f(l.o_xhat), l.out, Bn, l.out, f(l.o_inv), d(o_dsum), d(o_dprod), nullptr, s, bn_rows(Bn)));
      } else
      DCA_TRY(bn_bwd_apply(dh, f(l.o_xhat), l.out, Bn, l.out, f(l.o_inv), d(o_dsum), d(o_dprod), gp(l.beta), s));
    }
    if (i == 0 && cur_xb) {
      DCA_TRY(cast_to_bf16(dh, bf(o_da1b), (int64_t)Bn * l.out, s));
      const __nv_bfloat16* Z[3] = {cur_xb, cur_xb, cur_xb};
      float* dWp[3] = {gp(l.W), gp(l.W), gp(l.W)};
      DCA_TRY(tc::gene_gemm_tc(2, Z, cur_ldxb, Bn, cfg.n_in, 1, bf(o_da1b), nullptr, nullptr, dWp, l.out, 0, nullptr, nullptr, 0, sm_count, s));
      DCA_TRY(col_sums(dh, nullptr, l.out, Bn, l.out, d(o_dsum), nullptr, d(o_scratch), s));
      DCA_TRY(col_sum_to_float(d(o_dsum), l.out, gp(l.b), s));
      continue;
    }
    const void* ain = (i == 0) ? X : (const void*)f(lay[i - 1].o_h);
    GemmArgs g{};
    g.A = ain; g.lda = (i == 0) ? ldx : lay[i - 1].out; g.a_bf16 = (i == 0) ? (x_override_bf16 ? 1 : (cfg.x_dtype == DCA_BF16)) : 0;
    g.transA = 1; g.a_rows = (i == 0) ? xrows : nullptr;
    g.B = dh; g.ldb = l.out; g.transB = 0;
    g.C = gp(l.W); g.ldc = l.out; g.M = l.in; g.N = l.out; g.K = Bn; g.epilogue = EPI_ACCUM;
    DCA_TRY(gemm_auto(g, s));
    DCA_TRY(col_sums(dh, nullptr, l.out, Bn, l.out, d(o_dsum), nullptr, d(o_scratch), s));
    DCA_TRY(col_sum_to_float(d(o_dsum), l.out, gp(l.b), s));
    if (i > 0) {
      GemmArgs b{};
      b.A = dh; b.lda = l.out; b.transA = 0;
      b.B = pp(l.W); b.ldb = l.out; b.transB = 1;
      b.C = dh2; b.ldc = l.in; b.M = Bn; b.N = l.in; b.K = l.out; b.epilogue = EPI_STORE; b.splits = 1;
      DCA_TRY(gemm_generic(b, s));
      float* t = dh; dh = dh2; dh2 = t;
    }
  }
  mark(-1, s);
  return DCA_OK;
}

int Engine::apply_update(float lr, float clip, float grad_scale, cudaStream_t s) {
  mark(5, s);
  float* ring_slot = loss_ring ? loss_ring + (ring_pos++ % ring_n) : nullptr;
  if (opt_kind != DCA_OPT_RMSPROP) {
    // per-step scalars of keras/optimizers.py get_updates (t = iterations + 1), evaluated in double on the host
    OptScalars o{}; o.kind = opt_kind; o.lr = lr; o.clip = clip; o.gs = grad_scale;
    const double t = (double)(++opt_iter), b1 = 0.9, b2 = 0.999;
    if (opt_kind == DCA_OPT_ADAM) o.c0 = (float)((double)lr * sqrt(1.0 - pow(b2, t)) / (1.0 - pow(b1, t)));
    else if (opt_kind == DCA_OPT_ADAMAX) o.c0 = (float)((double)lr / (1.0 - pow(b1, t)));
    else if (opt_kind == DCA_OPT_NADAM) {
      const double sd = 0.004;
      const double mu_t = b1 * (1.0 - 0.5 * pow(0.96, t * sd)), mu_t1 = b1 * (1.0 - 0.5 * pow(0.96, (t + 1.0) * sd));
      const double sched_new = nadam_sched * mu_t, sched_next = sched_new * mu_t1;
      nadam_sched = sched_new;
      o.c0 = (float)(1.0 / (1.0 - sched_new)); o.c1 = (float)(1.0 / (1.0 - sched_next)); o.c2 = (float)(1.0 / (1.0 - pow(b2, t)));
      o.c3 = (float)mu_t; o.c4 = (float)mu_t1;
    }
    DCA_TRY(optimizer_update(pp(0), gp(0), f(o_rms), f(o_opt2), P, o, (tc_heads || tc_enc) ? bf(o_pbf) : nullptr, ring_slot, s));
    mark(-1, s);
    return DCA_OK;
  }
  DCA_TRY(rmsprop_update(pp(0), gp(0), f(o_rms), P, lr, clip, cfg.rms_rho, cfg.rms_eps, grad_scale,
                         (tc_heads || tc_enc) ? bf(o_pbf) : nullptr, ring_slot, s));   // also refreshes the bf16 operand copy
  mark(-1, s);
  return DCA_OK;
}

int Engine::reset_optimizer(cudaStream_t s) {
  DCA_CUDA_OK(cudaMemsetAsync(f(o_rms), 0, sizeof(float) * (size_t)P, s));
  DCA_CUDA_OK(cudaMemsetAsync(f(o_opt2), 0, sizeof(float) * (size_t)P, s));
  opt_iter = 0; nadam_sched = 1.0;
  return DCA_OK;
}

int Engine::eval_step(const void* X, int64_t ldx, const float* Y, int64_t ldy, const float* sf, const int32_t* rows,
                      int Bn, cudaStream_t s) {
  if (!X || !Y) { set_error("dca_eval_step: X and Y must not be NULL"); return DCA_ERR_BAD_ARG; }
  if (Bn <= 0 || Bn > cfg.max_batch) { set_error("dca_eval_step: batch %d outside (0, max_batch=%d]", Bn, cfg.max_batch); return DCA_ERR_BAD_ARG; }
  if (x_kind) return x_eval_step(X, ldx, Y, ldy, sf, rows, Bn, s);
  const int G = cfg.n_out;
  DCA_TRY(forward(X, ldx, rows, Bn, false, s));
  float* Mb = f(o_head[0]); float* Db = f(o_head[1]); float* Pb = f(o_head[2]);
  DCA_TRY(heads_forward(Bn, Mb, cond ? Db : nullptr, has_pi ? Pb : nullptr, G, nullptr, s));
  if (!cond) DCA_TRY(theta_prepare(pp(theta_off), G, f(o_theta), f(o_chain), s));
  LossArgs la{};
  la.Y = Y; la.ldy = ldy; la.rows = rows; la.sf = sf;
  la.m = Mb; la.d = cond ? Db : f(o_theta); la.pi = has_pi ? Pb : nullptr; la.ld = G;
  la.B = Bn; la.G = G; la.ae_type = cfg.ae_type; la.ridge = cfg.ridge; la.inv_n = 1.f;
  la.loss_sum = d(o_acc) + 2; la.ws = base + o_lossws; la.ws_bytes = loss_ws_bytes;
  DCA_TRY(zinb_loss_fwd(la, s));
  add_double_kernel<<<1, 1, 0, s>>>(d(o_acc) + 3, (double)Bn * (double)G);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int Engine::predict(const void* X, int64_t ldx, const float* sf, const int32_t* rows, int Bn, float* mean_out,
                    float* disp_out, float* pi_out, int64_t ld_out, float* latent_out, cudaStream_t s) {
  if (!X) { set_error("dca_predict: X must not be NULL"); return DCA_ERR_BAD_ARG; }
  if (Bn <= 0 || Bn > cfg.max_batch) { set_error("dca_predict: batch %d outside (0, max_batch=%d]", Bn, cfg.max_batch); return DCA_ERR_BAD_ARG; }
  if (x_kind) return x_predict(X, ldx, sf, rows, Bn, mean_out, disp_out, pi_out, ld_out, latent_out, s);
  const int G = cfg.n_out;
  DCA_TRY(forward(X, ldx, rows, Bn, false, s));
  if (latent_out) {
    if (L == 0) { set_error("dca_predict: no hidden layer -> no latent output"); return DCA_ERR_BAD_ARG; }
    const int c = L / 2;
    copy_strided_kernel<<<cdiv((int64_t)Bn * lay[c].out, 256), 256, 0, s>>>(f(lay[c].o_a), lay[c].out, latent_out,
                                                                            lay[c].out, Bn, lay[c].out);
    DCA_LAUNCH_CHECK();
  }
  const bool want_heads = mean_out || (cond && disp_out) || (has_pi && pi_out);
  if (want_heads) {
    gather_sf_kernel<<<cdiv(Bn, 256), 256, 0, s>>>(sf, rows, Bn, f(o_sfb));
    DCA_LAUNCH_CHECK();
    DCA_TRY(heads_forward(Bn, mean_out, cond ? disp_out : nullptr, has_pi ? pi_out : nullptr, ld_out, f(o_sfb), s));
  }
  if (!cond && disp_out) {
    DCA_TRY(theta_prepare(pp(theta_off), G, disp_out, f(o_chain), s));
  }
  return DCA_OK;
}

bool Engine::tc_supported() const { return tc_heads && tc_enc; }
const char* Engine::tc_reason() const {
  return "tensor-core path needs hidden_size[0] == hidden_size[-1] == 64, n_in % 8 == 0 and n_out % 8 == 0";
}
int Engine::setup_tc() {
  if (const char* e = getenv("DCA_GRAPH")) graphs_enabled = !(e[0] == '0');
  int dev = 0;
  DCA_CUDA_OK(cudaGetDevice(&dev));
  DCA_CUDA_OK(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
  if (mid_ok && !mid_device_ok()) mid_ok = false;   // grid-barrier kernels need a cooperative launch of <= 128 CTAs: else per-layer path
  if (tc_heads || tc_enc) {
    int major = 0;
    DCA_CUDA_OK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    if (major != 9) { set_error("libdca_b200 is built for sm_90a only (device compute capability %d.x)", major); return DCA_ERR_UNSUPPORTED; }
  }
  return DCA_OK;
}
// Re-derive the bf16 copy of the parameters (the tensor-core kernels read every kernel in its Keras layout, so the
// "shadow" is a plain element-wise cast; after an optimizer step the RMSprop kernel writes it directly).
int Engine::refresh_shadows(cudaStream_t s) {
  if (!tc_heads && !tc_enc) return DCA_OK;
  return cast_to_bf16(pp(0), bf(o_pbf), P, s);
}

int Engine::init_params(uint64_t seed, cudaStream_t s) {
  DCA_CUDA_OK(cudaMemsetAsync(pp(0), 0, sizeof(float) * (size_t)P, s));
  DCA_TRY(reset_optimizer(s));
  DCA_CUDA_OK(cudaMemsetAsync(gp(0), 0, sizeof(float) * (size_t)(P + 2), s));
  DCA_CUDA_OK(cudaMemsetAsync(d(o_acc), 0, sizeof(double) * 8, s));
  uint64_t sid = 0;
  if (x_kind) {
    // Glorot-uniform for every kernel of the tensor table (1-D element-wise kernels: fan_in = fan_out = length, like Keras)
    for (auto& t : params) {
      const std::string nm(t.name);
      if (nm.size() < 7 || nm.compare(nm.size() - 7, 7, "/kernel") != 0) continue;
      const int fi = t.rows == 1 ? t.cols : t.rows, fo = t.cols;
      DCA_TRY(glorot_fill(pp(t.offset), (int64_t)t.rows * t.cols, fi, fo, seed, sid++, s));
    }
    if (cfg.batchnorm)
      for (auto& t : states) {
        const std::string nm(t.name);
        DCA_TRY(fill_value(st(t.offset), t.cols, nm.find("moving_var") != std::string::npos ? 1.f : 0.f, s));
      }
    return DCA_OK;
  }
  for (int i = 0; i < L; ++i)
    DCA_TRY(glorot_fill(pp(lay[i].W), (int64_t)lay[i].in * lay[i].out, lay[i].in, lay[i].out, seed, sid++, s));
  for (int k = 0; k < 3; ++k)
    if (head_W[k] >= 0) DCA_TRY(glorot_fill(pp(head_W[k]), (int64_t)K_head * cfg.n_out, K_head, cfg.n_out, seed, 100 + k, s));
  if (cfg.batchnorm)
    for (int i = 0; i < L; ++i) {
      DCA_TRY(fill_value(st(lay[i].mm), lay[i].out, 0.f, s));
      DCA_TRY(fill_value(st(lay[i].mv), lay[i].out, 1.f, s));
    }
  return DCA_OK;
}

}  // namespace dca

// ==================================================================================== C ABI
using namespace dca;


extern "C" int dca_version(void) { return DCA_B200_VERSION; }
extern "C" const char* dca_last_error(void) { return g_err; }
extern "C" int64_t dca_launch_count(void) { return (int64_t)g_launches.load(); }

extern "C" void dca_config_default(dca_config* c) {
  if (!c) return;
  memset(c, 0, sizeof(*c));
  c->struct_bytes = (int32_t)sizeof(dca_config);
  c->n_hidden = 3; c->hidden[0] = 64; c->hidden[1] = 32; c->hidden[2] = 64;   // dca/network.py:47
  c->ae_type = DCA_AE_ZINB_CONDDISP;
  c->batchnorm = 1; c->max_batch = 32; c->x_dtype = DCA_F32; c->gemm_path = DCA_GEMM_AUTO;
  c->bn_momentum = 0.99f; c->bn_eps = 1e-3f; c->rms_rho = 0.9f; c->rms_eps = 1e-7f;
}

extern "C" int dca_arena_bytes(const dca_config* cfg, size_t* bytes) {
  DCA_TRY(validate(cfg));
  if (!bytes) { set_error("dca_arena_bytes: bytes is NULL"); return DCA_ERR_BAD_ARG; }
  Engine e;
  DCA_TRY(e.plan(*cfg));
  *bytes = e.arena_bytes;
  return DCA_OK;
}

extern "C" int dca_create(const dca_config* cfg, void* arena, size_t arena_bytes, dca_handle** out) {
  if (!out) { set_error("dca_create: out is NULL"); return DCA_ERR_BAD_ARG; }
  *out = nullptr;
  DCA_TRY(validate(cfg));
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    (void)cudaGetLastError();
    set_error("dca_create: no CUDA device available (this library has no CPU fallback)");
    return DCA_ERR_NO_DEVICE;
  }
  dca_handle* h = new dca_handle();
  int st = h->e.plan(*cfg);
  if (st != DCA_OK) { delete h; return st; }
  if (cfg->gemm_path == DCA_GEMM_TCGEN05 && !h->e.tc_supported()) {
    set_error("dca_create: gemm_path=TCGEN05 requested but the layer shapes do not qualify (%s)", h->e.tc_reason());
    delete h; return DCA_ERR_UNSUPPORTED;
  }
  cudaGetDevice(&h->device);
  if (arena) {
    if (arena_bytes < h->e.arena_bytes) {
      set_error("dca_create: arena too small (%zu < %zu)", arena_bytes, h->e.arena_bytes);
      delete h; return DCA_ERR_BAD_ARG;
    }
    if (reinterpret_cast<uintptr_t>(arena) & 255) { set_error("dca_create: arena must be 256-byte aligned"); delete h; return DCA_ERR_BAD_ARG; }
    h->e.bind(arena);
  } else {
    void* p = nullptr;
    cudaError_t ce = cudaMalloc(&p, h->e.arena_bytes);
    if (ce != cudaSuccess) { set_error("dca_create: cudaMalloc(%zu) failed: %s", h->e.arena_bytes, cudaGetErrorString(ce)); delete h; return DCA_ERR_CUDA; }
    h->owned = p;
    h->e.bind(p);
  }
  cudaError_t ce = cudaMemset(h->e.base, 0, h->e.arena_bytes);
  if (ce != cudaSuccess) { set_error("dca_create: cudaMemset failed: %s", cudaGetErrorString(ce)); if (h->owned) cudaFree(h->owned); delete h; return DCA_ERR_CUDA; }
  st = h->e.setup_tc();
  if (st != DCA_OK) { if (h->owned) cudaFree(h->owned); delete h; return st; }
  *out = h;
  return DCA_OK;
}

extern "C" int dca_destroy(dca_handle* h) {
  if (!h) return DCA_OK;
  if (h->owned) cudaFree(h->owned);
  delete h;
  return DCA_OK;
}

#define DCA_NEED_HANDLE(h) \
  if (!(h)) { set_error("%s: handle is NULL", __func__); return DCA_ERR_BAD_ARG; }

extern "C" int dca_param_count(const dca_handle* h, int64_t* n, int32_t* nt) {
  DCA_NEED_HANDLE(h);
  if (n) *n = h->e.P;
  if (nt) *nt = (int32_t)h->e.params.size();
  return DCA_OK;
}
extern "C" int dca_param_info(const dca_handle* h, int32_t i, dca_tensor_info* info) {
  DCA_NEED_HANDLE(h);
  if (!info || i < 0 || i >= (int32_t)h->e.params.size()) { set_error("dca_param_info: index out of range"); return DCA_ERR_BAD_ARG; }
  *info = h->e.params[i];
  return DCA_OK;
}
extern "C" int dca_state_count(const dca_handle* h, int64_t* n, int32_t* nt) {
  DCA_NEED_HANDLE(h);
  if (n) *n = h->e.S;
  if (nt) *nt = (int32_t)h->e.states.size();
  return DCA_OK;
}
extern "C" int dca_state_info(const dca_handle* h, int32_t i, dca_tensor_info* info) {
  DCA_NEED_HANDLE(h);
  if (!info || i < 0 || i >= (int32_t)h->e.states.size()) { set_error("dca_state_info: index out of range"); return DCA_ERR_BAD_ARG; }
  *info = h->e.states[i];
  return DCA_OK;
}
extern "C" int dca_region(dca_handle* h, int32_t id, void** ptr, int64_t* count) {
  DCA_NEED_HANDLE(h);
  Engine& e = h->e;
  void* p = nullptr; int64_t n = 0;
  switch (id) {
    case DCA_REGION_PARAMS: p = e.base + e.o_params; n = e.P; break;
    case DCA_REGION_GRADS: p = e.base + e.o_grads; n = e.P + 2; break;
    case DCA_REGION_RMS: p = e.base + e.o_rms; n = e.P; break;
    case DCA_REGION_BN_STATE: p = e.base + e.o_state; n = e.S; break;
    case DCA_REGION_EPOCH_ACC: p = e.base + e.o_acc; n = 4; break;
    default: set_error("dca_region: unknown region %d", id); return DCA_ERR_BAD_ARG;
  }
  if (ptr) *ptr = p;
  if (count) *count = n;
  return DCA_OK;
}

extern "C" int dca_init_params(dca_handle* h, uint64_t seed, void* stream) {
  DCA_NEED_HANDLE(h);
  DCA_TRY(h->e.init_params(seed, (cudaStream_t)stream));
  return h->e.refresh_shadows((cudaStream_t)stream);
}
extern "C" int dca_params_changed(dca_handle* h, void* stream) {
  DCA_NEED_HANDLE(h);
  return h->e.refresh_shadows((cudaStream_t)stream);
}

extern "C" int dca_train_step(dca_handle* h, const void* X, int64_t ldx, const float* Y, int64_t ldy, const float* sf,
                              const int32_t* rows, int32_t batch, void* stream) {
  DCA_NEED_HANDLE(h);
  return h->e.train_step(X, ldx, Y, ldy, sf, rows, batch, (cudaStream_t)stream, 0);
}
extern "C" int dca_train_step_phase(dca_handle* h, const void* X, int64_t ldx, const float* Y, int64_t ldy, const float* sf,
                                    const int32_t* rows, int32_t batch, int32_t phase, void* stream) {
  DCA_NEED_HANDLE(h);
  if (phase != 1 && phase != 2) { set_error("dca_train_step_phase: phase must be 1 or 2"); return DCA_ERR_BAD_ARG; }
  return h->e.train_step(X, ldx, Y, ldy, sf, rows, batch, (cudaStream_t)stream, phase);
}
extern "C" int dca_grad_buckets(const dca_handle* h, int64_t* head_bucket_offset) {
  DCA_NEED_HANDLE(h);
  if (!head_bucket_offset) { set_error("dca_grad_buckets: NULL"); return DCA_ERR_BAD_ARG; }
  *head_bucket_offset = h->e.x_kind ? 0 : h->e.head_W[0];      // grads[offset : P+2] are final after phase 1
  return DCA_OK;
}
extern "C" int dca_set_optimizer(dca_handle* h, int32_t optimizer, void* stream) {
  if (!h) { set_error("dca_set_optimizer: handle is NULL"); return DCA_ERR_BAD_ARG; }
  if (optimizer < DCA_OPT_RMSPROP || optimizer > DCA_OPT_NADAM) { set_error("dca_set_optimizer: unknown optimizer %d", optimizer); return DCA_ERR_BAD_ARG; }
  h->e.opt_kind = optimizer;
  return h->e.reset_optimizer((cudaStream_t)stream);
}

extern "C" int dca_reset_optimizer(dca_handle* h, void* stream) {
  if (!h) { set_error("dca_reset_optimizer: handle is NULL"); return DCA_ERR_BAD_ARG; }
  return h->e.reset_optimizer((cudaStream_t)stream);
}

extern "C" int dca_apply_update(dca_handle* h, float lr, float clip, float grad_scale, void* stream) {
  DCA_NEED_HANDLE(h);
  return h->e.apply_update(lr, clip, grad_scale, (cudaStream_t)stream);
}
extern "C" int dca_eval_step(dca_handle* h, const void* X, int64_t ldx, const float* Y, int64_t ldy, const float* sf,
                             const int32_t* rows, int32_t batch, void* stream) {
  DCA_NEED_HANDLE(h);
  return h->e.eval_step(X, ldx, Y, ldy, sf, rows, batch, (cudaStream_t)stream);
}
extern "C" int dca_predict(dca_handle* h, const void* X, int64_t ldx, const float* sf, const int32_t* rows,
                           int32_t batch, float* mean_out, float* disp_out, float* pi_out, int64_t ld_out,
                           float* latent_out, void* stream) {
  DCA_NEED_HANDLE(h);
  return h->e.predict(X, ldx, sf, rows, batch, mean_out, disp_out, pi_out, ld_out, latent_out, (cudaStream_t)stream);
}

extern "C" int dca_read_loss(dca_handle* h, float* loss_host, int32_t* nonfinite_host, void* stream) {
  DCA_NEED_HANDLE(h);
  float v[2] = {0.f, 0.f};
  cudaStream_t s = (cudaStream_t)stream;
  DCA_CUDA_OK(cudaMemcpyAsync(v, h->e.gp(h->e.P), sizeof(v), cudaMemcpyDeviceToHost, s));
  DCA_CUDA_OK(cudaStreamSynchronize(s));
  if (loss_host) *loss_host = v[0];
  if (nonfinite_host) *nonfinite_host = v[1] != 0.f;
  return DCA_OK;
}
extern "C" int dca_read_epoch_acc(dca_handle* h, double acc_host[4], int32_t reset, void* stream) {
  DCA_NEED_HANDLE(h);
  cudaStream_t s = (cudaStream_t)stream;
  DCA_CUDA_OK(cudaMemcpyAsync(acc_host, h->e.d(h->e.o_acc), 4 * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (reset) DCA_CUDA_OK(cudaMemsetAsync(h->e.d(h->e.o_acc), 0, 4 * sizeof(double), s));
  DCA_CUDA_OK(cudaStreamSynchronize(s));
  return DCA_OK;
}

extern "C" int dca_train_step_host(dca_handle* h, const void* x_host, const float* y_host, const float* sf_host,
                                   int32_t batch, float lr, float clip, float* loss_host, void* stream) {
  DCA_NEED_HANDLE(h);
  Engine& e = h->e;
  if (!x_host || !y_host) { set_error("dca_train_step_host: NULL host buffer"); return DCA_ERR_BAD_ARG; }
  if (batch <= 0 || batch > e.cfg.max_batch) { set_error("dca_train_step_host: batch %d outside (0, max_batch=%d]", batch, e.cfg.max_batch); return DCA_ERR_BAD_ARG; }
  cudaStream_t s = (cudaStream_t)stream;
  const size_t xb = (e.cfg.x_dtype == DCA_BF16) ? 2 : 4;
  DCA_CUDA_OK(cudaMemcpyAsync(e.base + e.o_stage_x, x_host, xb * (size_t)batch * e.cfg.n_in, cudaMemcpyHostToDevice, s));
  DCA_CUDA_OK(cudaMemcpyAsync(e.base + e.o_stage_y, y_host, sizeof(float) * (size_t)batch * e.cfg.n_out, cudaMemcpyHostToDevice, s));
  const float* sfd = nullptr;
  if (sf_host) {
    DCA_CUDA_OK(cudaMemcpyAsync(e.base + e.o_stage_sf, sf_host, sizeof(float) * (size_t)batch, cudaMemcpyHostToDevice, s));
    sfd = e.f(e.o_stage_sf);
  }
  DCA_TRY(e.train_step(e.base + e.o_stage_x, e.cfg.n_in, e.f(e.o_stage_y), e.cfg.n_out, sfd, nullptr, batch, s, 0));
  DCA_TRY(e.apply_update(lr, clip, 1.0f, s));
  return dca_read_loss(h, loss_host, nullptr, stream);
}

extern "C" int dca_profile_enable(dca_handle* h, int32_t on) {
  DCA_NEED_HANDLE(h);
  if (!on && h->e.prof.on) DCA_TRY(h->e.prof_collect());
  h->e.prof.on = on != 0;
  return DCA_OK;
}
extern "C" int dca_profile_read(dca_handle* h, double ms[DCA_N_PHASES], int64_t counts[DCA_N_PHASES], int32_t reset) {
  DCA_NEED_HANDLE(h);
  DCA_TRY(h->e.prof_collect());
  for (int i = 0; i < DCA_N_PHASES; ++i) {
    if (ms) ms[i] = h->e.prof.ms[i];
    if (counts) counts[i] = h->e.prof.cnt[i];
    if (reset) { h->e.prof.ms[i] = 0; h->e.prof.cnt[i] = 0; }
  }
  return DCA_OK;
}

extern "C" int dca_engine_info(const dca_handle* h, int32_t info[8]) {
  DCA_NEED_HANDLE(h);
  if (!info) { set_error("dca_engine_info: info is NULL"); return DCA_ERR_BAD_ARG; }
  const Engine& e = h->e;
  info[0] = e.tc_heads; info[1] = e.tc_enc; info[2] = e.mid_ok; info[3] = e.n_slots; info[4] = e.sm_count;
  info[5] = e.tc_heads ? 2 : 4;
  int ng = 0; for (auto& g : e.graphs) if (g.exec) ++ng;
  info[6] = ng; info[7] = e.graphs_enabled;
  return DCA_OK;
}

// ------------------------------------------------------------------------------------ streaming from host counts
// copy batch `i` of the host dataset into staging buffer `b` (copy stream) and expand it (counts -> Y fp32, X
// normalised; low-priority expand stream): both overlap the training step of the previous batch, which works on the
// other buffer pair, and the copy of batch i+1 does not wait for the expansion of batch i
// raw staging buffer b (packed counts as they arrive: two of them) and expanded buffer e (Y, X, sf of the batch: hs.exp_bufs)
int Engine::stream_prefetch(int64_t i, int b, int e) {
  const int64_t r0 = i * hs.batch;
  const int64_t nb = (hs.n_rows - r0 < hs.batch) ? (hs.n_rows - r0) : hs.batch;
  const bool sparse = hs.bits == 1;
  const size_t tight = (size_t)cfg.n_in * (size_t)hs.bits / 8;             // bytes of one packed row (sparse: its bitmap)
  DCA_CUDA_OK(cudaStreamWaitEvent(hs.copy, hs.cnt_free[b], 0));          // the expansion two batches ago has consumed staging b
  if (hs.tl_base && hs.tl.size() < 400) hs.tl_mark(hs.copy);
  if ((size_t)hs.row_bytes == tight)  // contiguous rows: one linear copy (faster than the pitched path)
    DCA_CUDA_OK(cudaMemcpyAsync(base + o_cnt[b], hs.counts + r0 * hs.row_bytes, tight * (size_t)nb, cudaMemcpyHostToDevice, hs.copy));
  else
    DCA_CUDA_OK(cudaMemcpy2DAsync(base + o_cnt[b], tight, hs.counts + r0 * hs.row_bytes, (size_t)hs.row_bytes, tight, (size_t)nb,
                                  cudaMemcpyHostToDevice, hs.copy));
  if (hs.sf) DCA_CUDA_OK(cudaMemcpyAsync(base + o_sfst[b], hs.sf + r0, sizeof(float) * (size_t)nb, cudaMemcpyHostToDevice, hs.copy));
  if (sparse) {
    const int64_t n0 = hs.nib_indptr[r0], n1 = hs.nib_indptr[r0 + nb];
    DCA_CUDA_OK(cudaMemcpyAsync(base + o_nibp[b], hs.nib_indptr + r0, sizeof(int64_t) * (size_t)(nb + 1), cudaMemcpyHostToDevice, hs.copy));
    if (n1 > n0) DCA_CUDA_OK(cudaMemcpyAsync(base + o_nib[b], hs.nibbles + n0, (size_t)(n1 - n0), cudaMemcpyHostToDevice, hs.copy));
  }
  bool has_ovf = false;
  if (hs.ovf_indptr) {
    const int64_t e0 = hs.ovf_indptr[r0], e1 = hs.ovf_indptr[r0 + nb];
    has_ovf = e1 > e0;
    if (has_ovf) {
      DCA_CUDA_OK(cudaMemcpyAsync(base + o_ovp[b], hs.ovf_indptr + r0, sizeof(int64_t) * (size_t)(nb + 1), cudaMemcpyHostToDevice, hs.copy));
      DCA_CUDA_OK(cudaMemcpyAsync(base + o_ove[b], hs.ovf_entries + 8 * e0, 8 * (size_t)(e1 - e0), cudaMemcpyHostToDevice, hs.copy));
    }
  }
  DCA_CUDA_OK(cudaEventRecord(hs.h2d_done[b], hs.copy));
  if (hs.tl_base && hs.tl.size() < 400) hs.tl_mark(hs.copy);
  // expansion on its own low-priority stream: the next copy does not queue behind it, the step's kernels go first
  DCA_CUDA_OK(cudaStreamWaitEvent(hs.expand, hs.h2d_done[b], 0));
  DCA_CUDA_OK(cudaStreamWaitEvent(hs.expand, hs.step_done[e], 0));       // the step that read the expanded buffers b has finished
  const int x_bf16 = tc_enc ? 1 : (cfg.x_dtype == DCA_BF16);
  int max_nib = 0;                       // longest nibble run of a row of this batch (host CSR): sizes the expansion's smem
  if (sparse) for (int64_t r = r0; r < r0 + nb; ++r) { const int len = (int)(hs.nib_indptr[r + 1] - hs.nib_indptr[r]); if (len > max_nib) max_nib = len; }
  if (sparse)
    DCA_TRY(expand_sparse(base + o_cnt[b], reinterpret_cast<const int64_t*>(base + o_nibp[b]), base + o_nib[b],
                          hs.sf ? f(o_sfst[b]) : nullptr, (int)nb, cfg.n_in, tf_set == 2 ? f(o_gmean) : nullptr,
                          tf_set == 2 ? f(o_ginv) : nullptr, tf_use_sf && hs.sf, tf_use_log1p, f(o_sy[e]), base + o_sx[e], x_bf16,
                          f(o_ssf[e]), has_ovf ? reinterpret_cast<const int64_t*>(base + o_ovp[b]) : nullptr,
                          has_ovf ? (const void*)(base + o_ove[b]) : nullptr, max_nib, hs.expand));
  else
  DCA_TRY(expand_counts(base + o_cnt[b], hs.bits, hs.sf ? f(o_sfst[b]) : nullptr, (int)nb, cfg.n_in,
                        tf_set == 2 ? f(o_gmean) : nullptr, tf_set == 2 ? f(o_ginv) : nullptr, tf_use_sf && hs.sf,
                        tf_use_log1p, f(o_sy[e]), base + o_sx[e], x_bf16, f(o_ssf[e]),
                        has_ovf ? reinterpret_cast<const int64_t*>(base + o_ovp[b]) : nullptr,
                        has_ovf ? (const void*)(base + o_ove[b]) : nullptr, hs.expand));
  DCA_CUDA_OK(cudaEventRecord(hs.cnt_free[b], hs.expand));
  DCA_CUDA_OK(cudaEventRecord(hs.ready[e], hs.expand));
  if (hs.tl_base && hs.tl.size() < 400) hs.tl_mark(hs.expand);
  hs.pref_idx = i;
  return DCA_OK;
}

extern "C" int dca_set_loss_ring(dca_handle* h, float* host_ring, int32_t n_slots) {
  DCA_NEED_HANDLE(h);
  Engine& e = h->e;
  if (!host_ring || n_slots <= 0) { e.loss_ring = nullptr; e.ring_n = 0; e.ring_pos = 0; return DCA_OK; }
  void* dptr = nullptr;
  if (cudaHostGetDevicePointer(&dptr, host_ring, 0) != cudaSuccess || !dptr) {
    cudaGetLastError();
    set_error("dca_set_loss_ring: the buffer is not pinned (mapped) host memory");
    return DCA_ERR_BAD_ARG;
  }
  e.loss_ring = reinterpret_cast<float*>(dptr); e.ring_n = n_slots; e.ring_pos = 0;
  return DCA_OK;
}

extern "C" int dca_set_input_transform(dca_handle* h, const float* gene_mean_host, const float* gene_inv_std_host,
                                       int32_t use_size_factors, int32_t use_log1p, void* stream) {
  DCA_NEED_HANDLE(h);
  Engine& e = h->e;
  cudaStream_t s = (cudaStream_t)stream;
  if ((gene_mean_host == nullptr) != (gene_inv_std_host == nullptr)) { set_error("dca_set_input_transform: give both mean and inv_std or neither"); return DCA_ERR_BAD_ARG; }
  if (gene_mean_host) {
    DCA_CUDA_OK(cudaMemcpyAsync(e.base + e.o_gmean, gene_mean_host, sizeof(float) * (size_t)e.cfg.n_in, cudaMemcpyHostToDevice, s));
    DCA_CUDA_OK(cudaMemcpyAsync(e.base + e.o_ginv, gene_inv_std_host, sizeof(float) * (size_t)e.cfg.n_in, cudaMemcpyHostToDevice, s));
    DCA_CUDA_OK(cudaStreamSynchronize(s));
  }
  e.tf_set = gene_mean_host ? 2 : 1; e.tf_use_sf = use_size_factors != 0; e.tf_use_log1p = use_log1p != 0;
  return DCA_OK;
}

extern "C" int dca_stream_begin_packed(dca_handle* h, const void* packed_host, int32_t bits, int64_t row_bytes,
                                       const int64_t* ovf_indptr_host, const void* ovf_entries_host, const float* sf_host,
                                       int64_t n_rows, int32_t batch, void* stream) {
  DCA_NEED_HANDLE(h);
  Engine& e = h->e;
  if (!packed_host || n_rows <= 0 || batch <= 0 || batch > e.cfg.max_batch) { set_error("dca_stream_begin: bad argument"); return DCA_ERR_BAD_ARG; }
  if (bits != 1 && bits != 4 && bits != 8 && bits != 16) { set_error("dca_stream_begin: bits must be 4, 8 or 16 (got %d)", bits); return DCA_ERR_BAD_ARG; }
  if (row_bytes < (int64_t)e.cfg.n_in * bits / 8) { set_error("dca_stream_begin: row stride smaller than a packed row"); return DCA_ERR_BAD_ARG; }
  if (bits == 1 && !e.hs.nib_indptr) { set_error("dca_stream_begin: the sparse format starts with dca_stream_begin_sparse"); return DCA_ERR_BAD_ARG; }
  if ((ovf_indptr_host == nullptr) != (ovf_entries_host == nullptr)) { set_error("dca_stream_begin: give both overflow arrays or neither"); return DCA_ERR_BAD_ARG; }
  if (e.cfg.n_in != e.cfg.n_out) { set_error("dca_stream_begin: needs n_in == n_out"); return DCA_ERR_UNSUPPORTED; }
  if (e.cfg.n_in % 8 != 0) { set_error("dca_stream_begin: n_in must be a multiple of 8"); return DCA_ERR_UNSUPPORTED; }
  if (!e.tf_set) { set_error("dca_stream_begin: call dca_set_input_transform first"); return DCA_ERR_BAD_ARG; }
  if (ovf_indptr_host) {
    for (int64_t r0 = 0; r0 < n_rows; r0 += batch) {
      const int64_t r1 = (r0 + batch < n_rows) ? r0 + batch : n_rows;
      const int64_t cnt = ovf_indptr_host[r1] - ovf_indptr_host[r0];
      if (cnt < 0 || cnt > e.ovf_cap) {
        set_error("dca_stream_begin: batch starting at row %lld has %lld overflow entries (capacity %lld): pack with more bits",
                  (long long)r0, (long long)cnt, (long long)e.ovf_cap);
        return DCA_ERR_BAD_ARG;
      }
    }
  }
  auto& hs = e.hs;
  if (!hs.copy) {
    int least = 0, greatest = 0;
    DCA_CUDA_OK(cudaDeviceGetStreamPriorityRange(&least, &greatest));
    DCA_CUDA_OK(cudaStreamCreateWithFlags(&hs.copy, cudaStreamNonBlocking));
    // expansion stream: HIGHEST priority.  Its blocks only find room between the kernels of the step; at the lowest
    // priority the expansion of batch i+1 can run after step i instead of under it.  DCA_EXPAND_PRIO=low selects the
    // lowest priority
    const char* pe = getenv("DCA_EXPAND_PRIO");
    DCA_CUDA_OK(cudaStreamCreateWithPriority(&hs.expand, cudaStreamNonBlocking, (pe && pe[0] == 'l') ? least : greatest));
    for (int k = 0; k < 2; ++k) {
      DCA_CUDA_OK(cudaEventCreateWithFlags(&hs.h2d_done[k], cudaEventDisableTiming));
      DCA_CUDA_OK(cudaEventCreateWithFlags(&hs.cnt_free[k], cudaEventDisableTiming));
    }
    for (int k = 0; k < 3; ++k) {
      DCA_CUDA_OK(cudaEventCreateWithFlags(&hs.ready[k], cudaEventDisableTiming));
      DCA_CUDA_OK(cudaEventCreateWithFlags(&hs.step_done[k], cudaEventDisableTiming));
    }
    if (const char* eb = getenv("DCA_STREAM_BUFS")) hs.exp_bufs = (atoi(eb) == 2) ? 2 : 3;
  }
  cudaStream_t s = (cudaStream_t)stream;
  for (int k = 0; k < 2; ++k) DCA_CUDA_OK(cudaEventRecord(hs.cnt_free[k], s));     // every staging buffer starts free
  for (int k = 0; k < 3; ++k) DCA_CUDA_OK(cudaEventRecord(hs.step_done[k], s));
  hs.counts = reinterpret_cast<const unsigned char*>(packed_host); hs.row_bytes = row_bytes; hs.bits = bits;
  hs.ovf_indptr = ovf_indptr_host; hs.ovf_entries = reinterpret_cast<const unsigned char*>(ovf_entries_host);
  hs.sf = sf_host; hs.n_rows = n_rows; hs.batch = batch;
  if (bits != 1) { hs.nib_indptr = nullptr; hs.nibbles = nullptr; }
  hs.pref_idx = -1; hs.step_no = 0; hs.active = true;
  { const char* v = getenv("DCA_STREAM_DIAG");
    if (v && atoi(v) == 2) { hs.tl.clear(); if (!hs.tl_base) cudaEventCreate(&hs.tl_base); cudaEventRecord(hs.tl_base, s); } }
  return DCA_OK;
}

extern "C" int dca_stream_begin_sparse(dca_handle* h, const void* bitmap_host, const int64_t* nib_indptr_host,
                                       const void* nibbles_host, const int64_t* ovf_indptr_host, const void* ovf_entries_host,
                                       const float* sf_host, int64_t n_rows, int32_t batch, void* stream) {
  DCA_NEED_HANDLE(h);
  Engine& e = h->e;
  if (!bitmap_host || !nib_indptr_host || !nibbles_host || n_rows <= 0 || batch <= 0) { set_error("dca_stream_begin_sparse: bad argument"); return DCA_ERR_BAD_ARG; }
  for (int64_t r0 = 0; r0 < n_rows; r0 += batch) {
    const int64_t r1 = (r0 + batch < n_rows) ? r0 + batch : n_rows;
    const int64_t nbytes = nib_indptr_host[r1] - nib_indptr_host[r0];
    if (nbytes < 0 || nbytes > e.nib_cap) {
      set_error("dca_stream_begin_sparse: batch starting at row %lld has %lld bytes of non-zero codes (capacity %lld = 50 %% non-zeros): "
                "use the dense 4-bit format", (long long)r0, (long long)nbytes, (long long)e.nib_cap);
      return DCA_ERR_BAD_ARG;
    }
  }
  e.hs.nib_indptr = nib_indptr_host; e.hs.nibbles = reinterpret_cast<const unsigned char*>(nibbles_host);
  return dca_stream_begin_packed(h, bitmap_host, 1, (int64_t)e.cfg.n_in / 8, ovf_indptr_host, ovf_entries_host, sf_host, n_rows,
                                 batch, stream);
}

extern "C" int dca_stream_begin(dca_handle* h, const uint16_t* counts_host, int64_t ld_counts, const float* sf_host,
                                int64_t n_rows, int32_t batch, void* stream) {
  return dca_stream_begin_packed(h, counts_host, 16, ld_counts * (int64_t)sizeof(uint16_t), nullptr, nullptr, sf_host, n_rows,
                                 batch, stream);
}

extern "C" int dca_stream_step(dca_handle* h, int64_t i, int64_t next, void* stream) {
  DCA_NEED_HANDLE(h);
  Engine& e = h->e; auto& hs = e.hs;
  if (!hs.active) { set_error("dca_stream_step: no active stream (dca_stream_begin)"); return DCA_ERR_BAD_ARG; }
  if (i < 0 || i * (int64_t)hs.batch >= hs.n_rows || next * (int64_t)hs.batch >= hs.n_rows) {
    set_error("dca_stream_step: batch index out of range (%lld, next %lld)", (long long)i, (long long)next); return DCA_ERR_BAD_ARG;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const int b = (int)(hs.step_no & 1), xb = (int)(hs.step_no % hs.exp_bufs);
  const int nb_raw = b ^ 1, nxb = (int)((hs.step_no + 1) % hs.exp_bufs);
  if (hs.pref_idx != i) DCA_TRY(e.stream_prefetch(i, b, xb));       // not prefetched by the previous step: fetch now
  const int64_t r0 = i * hs.batch;
  const int nb = (int)((hs.n_rows - r0 < hs.batch) ? (hs.n_rows - r0) : hs.batch);
  ++hs.step_no;
  hs.pref_idx = -1;
  if (next >= 0) DCA_TRY(e.stream_prefetch(next, nb_raw, nxb));     // next batch: copy + expansion overlap this step
  DCA_CUDA_OK(cudaStreamWaitEvent(s, hs.ready[xb], 0));
  const bool tl_on = hs.tl_base && hs.tl.size() < 400;
  if (tl_on) hs.tl_mark(s);
  static const int diag = [] { const char* v = getenv("DCA_STREAM_DIAG"); return v ? atoi(v) : 0; }();
  int st = DCA_OK;
  if (diag != 1) {                                  // (1 = diagnosis: copies + expansion only)
    e.x_override_bf16 = e.tc_enc ? 1 : 0;           // the tensor-core encoder reads the expanded bf16 batch in place
    st = e.train_step(e.base + e.o_sx[xb], e.cfg.n_in, e.f(e.o_sy[xb]), e.cfg.n_out, e.f(e.o_ssf[xb]), nullptr, nb, s, 0);
    e.x_override_bf16 = 0;
  }
  DCA_CUDA_OK(cudaEventRecord(hs.step_done[xb], s));
  if (tl_on) hs.tl_mark(s);
  return st;
}

extern "C" int dca_stream_end(dca_handle* h, void* stream) {
  DCA_NEED_HANDLE(h);
  auto& hs = h->e.hs;
  if (hs.copy) DCA_CUDA_OK(cudaStreamSynchronize(hs.copy));
  if (hs.expand) DCA_CUDA_OK(cudaStreamSynchronize(hs.expand));
  DCA_CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream));
  if (hs.tl_base && !hs.tl.empty()) {   // order of marks per step: [copy0 c0 c1 (first step only)] x0 x1 | copy-next c0 c1 | step-end
    fprintf(stderr, "[dca stream timeline, ms since stream_begin; first 3 marks: copy/expand of batch 0; then per step: "
                    "next_copy_start next_copy_end next_expand_end step_start step_end]\n");
    std::vector<float> t(hs.tl.size());
    for (size_t k = 0; k < hs.tl.size(); ++k) { t[k] = -1.f; cudaEventElapsedTime(&t[k], hs.tl_base, hs.tl[k]); cudaEventDestroy(hs.tl[k]); }
    for (size_t k = 0; k < t.size(); ++k) fprintf(stderr, "%.3f%s", t[k], ((k + 1 - 3) % 5 == 0 && k >= 3) ? "\n" : " ");
    fprintf(stderr, "\n");
    hs.tl.clear();
  }
  hs.active = false; hs.counts = nullptr; hs.ovf_indptr = nullptr; hs.ovf_entries = nullptr; hs.nib_indptr = nullptr; hs.nibbles = nullptr;
  return DCA_OK;
}
