// The remaining registry keys of dca/network.py:763-768 (SURVEY.md 8f-4) on the shape-general fp32 path:
//   poisson      dca/network.py:233-246   mean head (MeanAct), poisson_loss (dca/loss.py:33-48)
//   normal       dca/network.py:143-156   LINEAR mean head, keras mean_squared_error
//   nb-shared    dca/network.py:341-363   dispersion = Dense(1, DispAct): one theta per CELL
//   zinb-shared  dca/network.py:465-493   pi = Dense(1, sigmoid), dispersion = Dense(1, DispAct) per cell
//   zinb-elempi  dca/network.py:424-462   t = -Dense(G)(h); mean = MeanAct(t); pi = sigmoid(t * k + c)
//                                         (ElementwiseDense dca/layers.py:50-81; network_kwds sharedpi: scalar k, c)
//   nb-fork / zinb-fork  dca/network.py:553-760   the decoder layer after 'center' exists once PER HEAD
// Every one is a re-parameterisation of the heads around the SAME NB / ZINB loss kernel (zinb_loss.cu): per-cell
// parameters are broadcast to the B x G operand the kernel reads and their gradients summed back along the genes,
// the element-wise pi of zinb-elempi is an element-wise kernel before / after it, fork branches are ordinary
// Dense -> BatchNorm -> relu layers that read the trunk.  Generic CUDA-core GEMMs (dense_generic.cu) throughout:
// these types are outside the benchmarked path, correctness against the autograd oracle is the bar.
#include "dca_internal.cuh"
#include "engine.h"
#include <cstring>
#include <string>

namespace dca {

namespace {

__global__ void bcast_rows_kernel(const float* __restrict__ v, int B, int G, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < (int64_t)B * G) out[i] = v[i / G];
}
// out[r] = sum_g a[r, g]   (one warp per row, fp64 accumulation)
__global__ void row_sums_kernel(const float* __restrict__ a, int B, int G, float* __restrict__ out) {
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= B) return;
  double acc = 0.0;
  for (int g = lane; g < G; g += 32) acc += (double)a[(int64_t)r * G + g];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) out[r] = (float)acc;
}
// zinb-elempi forward: z (linear Dense output) -> m = MeanAct(-z) [* row_scale], pi = sigmoid(-z * k + c)
__global__ void elempi_fwd_kernel(const float* __restrict__ z, int B, int G, const float* __restrict__ k, const float* __restrict__ c,
                                  int nk, const float* __restrict__ row_scale, float* __restrict__ m, float* __restrict__ pi) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * G) return;
  const int g = (int)(i % G), r = (int)(i / G);
  const float t = -z[i];
  float mv = fminf(fmaxf(expf(t), 1e-5f), 1e6f);                       // MeanAct  dca/network.py:38,447
  if (row_scale) mv *= row_scale[r];
  if (m) m[i] = mv;
  if (pi) {
    const float u = t * k[nk == 1 ? 0 : g] + c[nk == 1 ? 0 : g];      // ElementwiseDense  dca/layers.py:74-81
    pi[i] = u >= 0.f ? 1.0f / (1.0f + expf(-u)) : expf(u) / (1.0f + expf(u));
  }
}
// zinb-elempi backward: dz = -(dzm + dzp * k)  (in place over dzm);  dzp, z stay for the column sums of dk, dc
__global__ void elempi_bwd_kernel(float* __restrict__ dzm, const float* __restrict__ dzp, int B, int G,
                                  const float* __restrict__ k, int nk) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * G) return;
  const int g = (int)(i % G);
  dzm[i] = -(dzm[i] + dzp[i] * k[nk == 1 ? 0 : g]);
}
// dk = -sum(dzp * z), dc = sum(dzp) from the fp64 column sums; nk == 1 folds the genes as well
__global__ void elempi_param_grad_kernel(const double* __restrict__ sum_p, const double* __restrict__ sum_pz, int G, int nk,
                                         float* __restrict__ dk, float* __restrict__ dc) {
  if (nk == 1) {
    if (blockIdx.x || threadIdx.x) return;
    double a = 0.0, b = 0.0;
    for (int g = 0; g < G; ++g) { a += sum_p[g]; b += sum_pz[g]; }
    dc[0] += (float)a; dk[0] += (float)(-b);
    return;
  }
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < G) { dc[g] += (float)sum_p[g]; dk[g] += (float)(-sum_pz[g]); }
}

// poisson_loss (dca/loss.py:33-48) and keras mean_squared_error on mu = m * sf.
//   KIND 0: poisson, m = MeanAct output;  elem = mu - y log(mu + 1e-10) + lgamma(y + 1), NaN targets count as 0 and are
//           left out of the element count (nelem);  dzm = (1 - y / (mu + eps)) * mu * [clip mask] / nelem
//   KIND 1: normal,  m = linear output;   elem = (mu - y)^2;  dz = 2 (mu - y) sf / (B G)
// pass 0 accumulates {loss sum, element count} (double atomics per block), pass 1 writes the gradients in place.
template <int KIND>
__global__ void simple_loss_kernel(const float* __restrict__ Y, int64_t ldy, const int32_t* __restrict__ rows,
                                   const float* __restrict__ sf, float* m, int B, int G, double* __restrict__ acc /* [2] */, int pass) {
  __shared__ double red[2][8];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double l = 0.0, n = 0.0;
  if (i < (int64_t)B * G) {
    const int r = (int)(i / G), g = (int)(i % G);
    const int64_t yr = rows ? (int64_t)rows[r] : (int64_t)r;
    const float s = sf ? sf[yr] : 1.0f;
    float y = Y[yr * ldy + g];
    const float mv = m[i], mu = mv * s;
    if (KIND == 0) {
      const bool ok = !(y != y);
      if (!ok) y = 0.f;
      if (pass == 0) { l = (double)(mu - y * logf(mu + 1e-10f) + lgammaf(y + 1.0f)); n = ok ? 1.0 : 0.0; }
      else {
        const float inv = 1.0f / (float)fmax(acc[1], 1.0);
        const bool pass_m = (mv > 1e-5f) && (mv < 1e6f);
        m[i] = pass_m ? (1.0f - y / (mu + 1e-10f)) * mu * inv : 0.f;
      }
    } else {
      const float dlt = mu - y;
      if (pass == 0) { l = (double)dlt * (double)dlt; n = 1.0; }
      else m[i] = 2.0f * dlt * s / ((float)B * (float)G);
    }
  }
  if (pass == 0) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { l += __shfl_xor_sync(0xffffffffu, l, o); n += __shfl_xor_sync(0xffffffffu, n, o); }
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { red[0][w] = l; red[1][w] = n; }
    __syncthreads();
    if (threadIdx.x == 0) {
      double a = 0.0, b = 0.0;
      for (int k = 0; k < (int)(blockDim.x >> 5); ++k) { a += red[0][k]; b += red[1][k]; }
      atomicAdd(&acc[0], a); atomicAdd(&acc[1], b);
    }
  }
}
// loss slot / epoch accumulators from {sum, count}: training (slot != null) or validation (val_acc != null)
__global__ void simple_loss_finish_kernel(const double* __restrict__ acc, const double* penalty, float* slot, double* epoch_acc,
                                          double* val_acc, int batch) {
  const double cnt = fmax(acc[1], 1.0);
  if (slot) {
    double l = acc[0] / cnt;
    if (l != l) l = INFINITY;
    if (penalty) l += *penalty;
    slot[0] = (float)l; slot[1] = isfinite((float)l) ? 0.f : 1.f;
    if (epoch_acc) { epoch_acc[0] += l * (double)batch; epoch_acc[1] += (double)batch; }
  }
  if (val_acc) { val_acc[0] += acc[0]; val_acc[1] += cnt; }
}

__global__ void x_add_double_kernel(double* p, double v) { *p += v; }

inline int nblk(int64_t n, int t = 256) { return (int)((n + t - 1) / t); }

}  // namespace

// ------------------------------------------------------------------------------------ layout
static void x_add_tensor(std::vector<dca_tensor_info>& v, int64_t& off, const std::string& name, int rows, int cols) {
  dca_tensor_info t;
  memset(&t, 0, sizeof(t));
  snprintf(t.name, sizeof(t.name), "%s", name.c_str());
  t.offset = off; t.rows = rows; t.cols = cols;
  off += (int64_t)rows * cols;
  v.push_back(t);
}

static std::string x_layer_name(int i, int n) {   // dca/network.py:102-111
  const int center = n / 2;
  if (i == center) return "center";
  if (i < center) return "enc" + std::to_string(i);
  return "dec" + std::to_string(i - center);
}

int Engine::x_plan_params(const dca_config& c, int64_t& off, int64_t& soff) {
  const int t = c.ae_type;
  x_kind = t;
  const bool fork = (t == DCA_AE_NB_FORK || t == DCA_AE_ZINB_FORK);
  has_pi = (t == DCA_AE_ZINB_SHARED || t == DCA_AE_ZINB_ELEMPI || t == DCA_AE_ZINB_FORK);
  cond = !(t == DCA_AE_POISSON || t == DCA_AE_NORMAL);           // a dispersion head exists
  const int center = L / 2;
  if (fork && L - 1 != center + 1) {
    set_error("fork types need exactly one decoder layer after 'center' (hidden_size like (64, 32, 64)); got %d hidden layers", L);
    return DCA_ERR_UNSUPPORTED;
  }
  trunk_L = fork ? center + 1 : L;
  int prev = c.n_in;
  maxh = 1;
  auto add_layer = [&](Layer& l, const std::string& nm, int in, int out, bool enc, int id, float drop) {
    l.id = id; l.drop = drop;
    l.in = in; l.out = out;
    l.W = off; x_add_tensor(params, off, nm + "/kernel", in, out);
    reg_items.push_back({l.W, (int64_t)in * out, enc});
    l.b = off; x_add_tensor(params, off, nm + "/bias", 1, out);
    if (c.batchnorm) {
      l.beta = off; x_add_tensor(params, off, nm + "/bn_beta", 1, out);
      l.mm = soff; x_add_tensor(states, soff, nm + "/bn_moving_mean", 1, out);
      l.mv = soff; x_add_tensor(states, soff, nm + "/bn_moving_var", 1, out);
    }
    if (c.activation == DCA_ACT_PRELU) { l.alpha = off; x_add_tensor(params, off, nm + "_act/alpha", 1, out); }
    if (out > maxh) maxh = out;
  };
  for (int i = 0; i < trunk_L; ++i) { add_layer(lay[i], x_layer_name(i, L), prev, c.hidden[i], i <= center, i, c.hidden_dropout[i]); prev = c.hidden[i]; }
  n_branch = 0;
  if (fork) {
    static const char* br[3] = {"mean", "disp", "pi"};
    n_branch = (t == DCA_AE_ZINB_FORK) ? 3 : 2;
    const std::string nm = x_layer_name(L - 1, L);
    for (int b = 0; b < n_branch; ++b) add_layer(brlay[b], nm + "_last_" + br[b], prev, c.hidden[L - 1], false, DCA_MAX_HIDDEN + b,
                                                c.hidden_dropout[L - 1]);
  }
  const int G = c.n_out;
  for (int k = 0; k < 3; ++k) { head_W[k] = head_b[k] = -1; head_N[k] = 0; head_K[k] = fork && k < n_branch ? c.hidden[L - 1] : prev; }
  theta_off = -1; epi_k = epi_c = -1; epi_n = 0;
  auto add_head = [&](int k, const char* nm, int N) {
    head_N[k] = N;
    head_W[k] = off; x_add_tensor(params, off, std::string(nm) + "/kernel", head_K[k], N);
    reg_items.push_back({head_W[k], (int64_t)head_K[k] * N, false});
    head_b[k] = off; x_add_tensor(params, off, std::string(nm) + "/bias", 1, N);
  };
  const bool shared = (t == DCA_AE_NB_SHARED || t == DCA_AE_ZINB_SHARED);
  // creation order of the reference's build_output (pi, dispersion, mean); names are what matters
  if (t == DCA_AE_ZINB_SHARED || t == DCA_AE_ZINB_FORK) add_head(2, "pi", shared ? 1 : G);
  if (cond) add_head(1, "dispersion", shared ? 1 : G);
  add_head(0, t == DCA_AE_ZINB_ELEMPI ? "mean_no_act" : "mean", G);
  if (t == DCA_AE_ZINB_ELEMPI) {
    epi_n = c.elempi_shared ? 1 : G;
    epi_k = off; x_add_tensor(params, off, "pi/kernel", 1, epi_n);
    reg_items.push_back({epi_k, (int64_t)epi_n, false});
    epi_c = off; x_add_tensor(params, off, "pi/bias", 1, epi_n);
  }
  K_head = head_K[0];
  return DCA_OK;
}

void Engine::x_plan_arena(size_t B, const std::function<size_t(size_t)>& take) {
  const size_t G = (size_t)cfg.n_out;
  for (int b = 0; b < n_branch; ++b) {
    const size_t h = (size_t)brlay[b].out;
    brlay[b].o_a = take(sizeof(float) * B * h); brlay[b].o_xhat = take(sizeof(float) * B * h); brlay[b].o_h = take(sizeof(float) * B * h);
    brlay[b].o_mean = take(sizeof(float) * h); brlay[b].o_inv = take(sizeof(float) * h);
  }
  if (x_kind == DCA_AE_ZINB_ELEMPI) o_zraw = take(sizeof(float) * B * G);
  for (int k = 0; k < 4; ++k) o_small[k] = take(sizeof(float) * B);
  o_xacc = take(sizeof(double) * 4);
}

// ------------------------------------------------------------------------------------ layers
int Engine::x_layer_fwd(Layer& l, const void* hin, int64_t ldin, int in_bf16, const int32_t* gather, int Bn, bool training,
                        cudaStream_t s) {
  float* a = f(l.o_a);
  DCA_TRY(fill_rows_with_bias(a, l.out, Bn, l.out, pp(l.b), s));
  GemmArgs g{};
  g.A = hin; g.lda = ldin; g.a_bf16 = in_bf16; g.transA = 0; g.a_rows = gather;
  g.B = pp(l.W); g.ldb = l.out; g.transB = 0;
  g.C = a; g.ldc = l.out; g.M = Bn; g.N = l.out; g.K = l.in; g.epilogue = EPI_ACCUM;
  DCA_TRY(gemm_auto(g, s));
  if (cfg.batchnorm) {
    if (training) {
      DCA_TRY(col_sums(a, nullptr, l.out, Bn, l.out, d(o_dsum), d(o_dprod), d(o_scratch), s));
      DCA_TRY(bn_allreduce(d(o_dsum), d(o_dprod), l.out, s));                    // sync_bn: statistics of the global batch
      DCA_TRY(bn_train_finalize(d(o_dsum), d(o_dprod), bn_rows(Bn), l.out, cfg.bn_eps, cfg.bn_momentum, f(l.o_mean), f(l.o_inv),
                                st(l.mm), st(l.mv), s));
    } else {
      DCA_TRY(bn_infer_prepare(st(l.mm), st(l.mv), l.out, cfg.bn_eps, f(l.o_mean), f(l.o_inv), s));
    }
  }
  return act_fwd(l, Bn, training, nullptr, s);
}

// dh [Bn x l.out] (overwritten) -> parameter gradients of the layer; din (nullable) += or = dh * W^T
int Engine::x_layer_bwd(Layer& l, float* dh, const void* hin, int64_t ldin, int in_bf16, const int32_t* gather, int Bn,
                        float* din, bool din_accumulate, cudaStream_t s) {
  DCA_TRY(act_bwd(l, dh, Bn, s));
  if (cfg.batchnorm) {
    DCA_TRY(col_sums(dh, f(l.o_xhat), l.out, Bn, l.out, d(o_dsum), d(o_dprod), d(o_scratch), s));
    if (bn_synced()) {
      DCA_TRY(col_sum_to_float(d(o_dsum), l.out, gp(l.beta), s));
      DCA_TRY(bn_allreduce(d(o_dsum), d(o_dprod), l.out, s));
      DCA_TRY(bn_bwd_apply(dh, f(l.o_xhat), l.out, Bn, l.out, f(l.o_inv), d(o_dsum), d(o_dprod), nullptr, s, bn_rows(Bn)));
    } else
    DCA_TRY(bn_bwd_apply(dh, f(l.o_xhat), l.out, Bn, l.out, f(l.o_inv), d(o_dsum), d(o_dprod), gp(l.beta), s));
  }
  GemmArgs g{};
  g.A = hin; g.lda = ldin; g.a_bf16 = in_bf16; g.transA = 1; g.a_rows = gather;
  g.B = dh; g.ldb = l.out; g.transB = 0;
  g.C = gp(l.W); g.ldc = l.out; g.M = l.in; g.N = l.out; g.K = Bn; g.epilogue = EPI_ACCUM;
  DCA_TRY(gemm_auto(g, s));
  DCA_TRY(col_sums(dh, nullptr, l.out, Bn, l.out, d(o_dsum), nullptr, d(o_scratch), s));
  DCA_TRY(col_sum_to_float(d(o_dsum), l.out, gp(l.b), s));
  if (din) {
    GemmArgs b{};
    b.A = dh; b.lda = l.out; b.transA = 0;
    b.B = pp(l.W); b.ldb = l.out; b.transB = 1;
    b.C = din; b.ldc = l.in; b.M = Bn; b.N = l.in; b.K = l.out; b.epilogue = din_accumulate ? EPI_ACCUM : EPI_STORE; b.splits = 1;
    DCA_TRY(gemm_generic(b, s));
  }
  return DCA_OK;
}

const float* Engine::x_head_in(int k) const { return n_branch && k < n_branch ? f(brlay[k].o_h) : (trunk_L ? f(lay[trunk_L - 1].o_h) : nullptr); }

// trunk + fork branches; afterwards x_head_in(k) is the input of head k (or X itself when there is no hidden layer)
int Engine::x_forward(const void* X, int64_t ldx, const int32_t* rows, int Bn, bool training, cudaStream_t s) {
  const void* hin = X; int64_t ldin = ldx; int in_bf16 = (cfg.x_dtype == DCA_BF16); const int32_t* gather = rows;
  for (int i = 0; i < trunk_L; ++i) {
    DCA_TRY(x_layer_fwd(lay[i], hin, ldin, in_bf16, gather, Bn, training, s));
    hin = f(lay[i].o_h); ldin = lay[i].out; in_bf16 = 0; gather = nullptr;
  }
  for (int b = 0; b < n_branch; ++b) DCA_TRY(x_layer_fwd(brlay[b], hin, ldin, in_bf16, gather, Bn, training, s));
  head_in = hin; head_ld = ldin; head_bf16 = in_bf16; head_rows = gather;      // trunk output (heads without a branch)
  return DCA_OK;
}

// head k: out[Bn x head_N[k]] = act(h_k W_k + b_k)
int Engine::x_head_gemm(int k, int Bn, float* out, int64_t ld_out, int epi, const float* row_scale, cudaStream_t s) {
  GemmArgs g{};
  if (n_branch && k < n_branch) { g.A = f(brlay[k].o_h); g.lda = brlay[k].out; g.a_bf16 = 0; g.a_rows = nullptr; }
  else { g.A = head_in; g.lda = head_ld; g.a_bf16 = head_bf16; g.a_rows = head_rows; }
  g.transA = 0;
  g.B = pp(head_W[k]); g.ldb = head_N[k]; g.transB = 0;
  g.C = out; g.ldc = ld_out; g.M = Bn; g.N = head_N[k]; g.K = head_K[k];
  g.bias = pp(head_b[k]); g.row_scale = row_scale; g.epilogue = epi; g.splits = 1;
  return gemm_generic(g, s);
}

// Post-activation head outputs as FULL B x G operands of the loss kernel: Mb (un-scaled mean; normal: linear output),
// Db, Pb.  row_scale (predict): the mean is multiplied by the size factor.
int Engine::x_heads_forward(int Bn, float* Mb, float* Db, float* Pb, const float* row_scale, cudaStream_t s) {
  const int G = cfg.n_out;
  const int64_t n = (int64_t)Bn * G;
  if (x_kind == DCA_AE_ZINB_ELEMPI) {
    DCA_TRY(x_head_gemm(0, Bn, f(o_zraw), G, EPI_STORE, nullptr, s));
    elempi_fwd_kernel<<<nblk(n), 256, 0, s>>>(f(o_zraw), Bn, G, pp(epi_k), pp(epi_c), epi_n, row_scale, Mb, Pb);
    DCA_LAUNCH_CHECK();
    if (Db) DCA_TRY(x_head_gemm(1, Bn, Db, G, EPI_DISP_ACT, nullptr, s));
    return DCA_OK;
  }
  if (Mb) DCA_TRY(x_head_gemm(0, Bn, Mb, G, x_kind == DCA_AE_NORMAL ? EPI_LINEAR_SCALE : EPI_MEAN_ACT, row_scale, s));
  const bool shared = (x_kind == DCA_AE_NB_SHARED || x_kind == DCA_AE_ZINB_SHARED);
  if (cond && Db) {
    if (shared) {
      DCA_TRY(x_head_gemm(1, Bn, f(o_small[0]), 1, EPI_DISP_ACT, nullptr, s));
      bcast_rows_kernel<<<nblk(n), 256, 0, s>>>(f(o_small[0]), Bn, G, Db);
      DCA_LAUNCH_CHECK();
    } else {
      DCA_TRY(x_head_gemm(1, Bn, Db, G, EPI_DISP_ACT, nullptr, s));
    }
  }
  if (has_pi && Pb) {
    if (shared) {
      DCA_TRY(x_head_gemm(2, Bn, f(o_small[1]), 1, EPI_SIGMOID, nullptr, s));
      bcast_rows_kernel<<<nblk(n), 256, 0, s>>>(f(o_small[1]), Bn, G, Pb);
      DCA_LAUNCH_CHECK();
    } else {
      DCA_TRY(x_head_gemm(2, Bn, Pb, G, EPI_SIGMOID, nullptr, s));
    }
  }
  return DCA_OK;
}

int Engine::x_penalty(cudaStream_t s, bool& any) {
  any = false;
  auto coeff = [&](const RegItem& r, float& l1, float& l2) {   // dca/network.py:113-122
    l1 = (r.enc && cfg.l1_enc != 0.f) ? cfg.l1_enc : cfg.l1;
    l2 = (r.enc && cfg.l2_enc != 0.f) ? cfg.l2_enc : cfg.l2;
  };
  for (auto& r : reg_items) { float l1, l2; coeff(r, l1, l2); if (l1 != 0.f || l2 != 0.f) any = true; }
  if (!any) return DCA_OK;
  DCA_CUDA_OK(cudaMemsetAsync(d(o_acc) + 5, 0, sizeof(double), s));
  for (auto& r : reg_items) {
    float l1, l2; coeff(r, l1, l2);
    if (l1 == 0.f && l2 == 0.f) continue;
    DCA_TRY(reg_penalty(pp(r.off), r.n, l1, l2, d(o_acc) + 5, s));
    DCA_TRY(add_reg_grad(pp(r.off), gp(r.off), r.n, l1, l2, s));
  }
  return DCA_OK;
}

// ------------------------------------------------------------------------------------ one training step
int Engine::x_train_step_body(const void* X, int64_t ldx, const float* Y, int64_t ldy, const float* sf, const int32_t* rows,
                              int Bn, cudaStream_t s) {
  const int G = cfg.n_out;
  const int64_t n = (int64_t)Bn * G;
  DCA_TRY(debug_reset(s));
  DCA_CUDA_OK(cudaMemsetAsync(gp(0), 0, sizeof(float) * (size_t)(P + 2), s));
  bool any_pen = false;
  mark(0, s);
  DCA_TRY(x_penalty(s, any_pen));
  // input dropout: the network reads a masked, gathered copy of the batch; Y keeps `rows`
  const int32_t* xrows = rows;
  if (!plain_hidden()) DCA_TRY(bump_step(s));
  if (cfg.input_dropout > 0.f) {
    DCA_TRY(drop_input(X, cfg.x_dtype == DCA_BF16, ldx, rows, Bn, s));
    X = base + o_xdrop; ldx = cfg.n_in; xrows = nullptr;
  }
  DCA_TRY(x_forward(X, ldx, xrows, Bn, true, s));
  mark(1, s);
  float* Mb = f(o_head[0]); float* Db = f(o_head[1]); float* Pb = f(o_head[2]);
  DCA_TRY(x_heads_forward(Bn, Mb, cond ? Db : nullptr, has_pi ? Pb : nullptr, nullptr, s));
  mark(2, s);
  const float inv_n = 1.0f / ((float)Bn * (float)G);
  if (x_kind == DCA_AE_POISSON || x_kind == DCA_AE_NORMAL) {
    double* acc = d(o_xacc);
    DCA_CUDA_OK(cudaMemsetAsync(acc, 0, 2 * sizeof(double), s));
    for (int pass = 0; pass < 2; ++pass) {
      if (x_kind == DCA_AE_POISSON) simple_loss_kernel<0><<<nblk(n), 256, 0, s>>>(Y, ldy, rows, sf, Mb, Bn, G, acc, pass);
      else simple_loss_kernel<1><<<nblk(n), 256, 0, s>>>(Y, ldy, rows, sf, Mb, Bn, G, acc, pass);
      DCA_LAUNCH_CHECK();
    }
    simple_loss_finish_kernel<<<1, 1, 0, s>>>(acc, any_pen ? d(o_acc) + 5 : nullptr, gp(P), d(o_acc), nullptr, Bn);
    DCA_LAUNCH_CHECK();
  } else {
    LossArgs la{};
    la.Y = Y; la.ldy = ldy; la.rows = rows; la.sf = sf;
    la.m = Mb; la.d = Db; la.pi = has_pi ? Pb : nullptr; la.ld = G;
    la.B = Bn; la.G = G; la.ae_type = has_pi ? DCA_AE_ZINB_CONDDISP : DCA_AE_NB_CONDDISP; la.ridge = cfg.ridge; la.inv_n = inv_n;
    la.dzm = Mb; la.dzd = Db; la.dzp = has_pi ? Pb : nullptr; la.grad_bf16 = 0;       // gradients in place
    la.loss_sum = d(o_acc) + 4; la.ws = base + o_lossws; la.ws_bytes = loss_ws_bytes; la.counter_ready = 1;
    la.fin_loss_slot = gp(P); la.fin_epoch_acc = d(o_acc); la.fin_penalty = any_pen ? d(o_acc) + 5 : nullptr; la.fin_batch = Bn;
    DCA_TRY(debug_check_loss(la, s));
    DCA_TRY(zinb_loss_fwd_bwd(la, s));
  }
  mark(3, s);
  // ---- back through the head parameterisations
  if (x_kind == DCA_AE_ZINB_ELEMPI) {
    // dk = sum_b dzp * t = -sum_b dzp * z,  dc = sum_b dzp;  then dz = -(dzm + dzp * k) in place over Mb
    DCA_TRY(col_sums(Pb, f(o_zraw), G, Bn, G, d(o_dsum), d(o_dprod), d(o_scratch), s));
    elempi_param_grad_kernel<<<epi_n == 1 ? 1 : nblk(G), epi_n == 1 ? 1 : 256, 0, s>>>(d(o_dsum), d(o_dprod), G, epi_n, gp(epi_k), gp(epi_c));
    DCA_LAUNCH_CHECK();
    elempi_bwd_kernel<<<nblk(n), 256, 0, s>>>(Mb, Pb, Bn, G, pp(epi_k), epi_n);
    DCA_LAUNCH_CHECK();
  }
  const bool shared = (x_kind == DCA_AE_NB_SHARED || x_kind == DCA_AE_ZINB_SHARED);
  // per head: gradient operand dz_k [Bn x head_N[k]]
  const float* dz[3] = {Mb, nullptr, nullptr};
  if (cond) {
    if (shared) { row_sums_kernel<<<nblk((int64_t)Bn * 32), 256, 0, s>>>(Db, Bn, G, f(o_small[2])); DCA_LAUNCH_CHECK(); dz[1] = f(o_small[2]); }
    else dz[1] = Db;
  }
  if (has_pi && x_kind != DCA_AE_ZINB_ELEMPI) {
    if (shared) { row_sums_kernel<<<nblk((int64_t)Bn * 32), 256, 0, s>>>(Pb, Bn, G, f(o_small[3])); DCA_LAUNCH_CHECK(); dz[2] = f(o_small[3]); }
    else dz[2] = Pb;
  }
  const bool have_hidden = trunk_L > 0;
  float* dh_trunk = f(o_dh[0]);          // gradient w.r.t. the trunk output
  float* dh_tmp = f(o_dh[1]);
  if (have_hidden) DCA_CUDA_OK(cudaMemsetAsync(dh_trunk, 0, sizeof(float) * (size_t)Bn * lay[trunk_L - 1].out, s));
  for (int k = 0; k < 3; ++k) {
    if (!dz[k] || head_W[k] < 0) continue;
    const int N = head_N[k];
    const bool br = n_branch && k < n_branch;
    GemmArgs g{};
    if (br) { g.A = f(brlay[k].o_h); g.lda = brlay[k].out; g.a_bf16 = 0; g.a_rows = nullptr; }
    else { g.A = head_in; g.lda = head_ld; g.a_bf16 = head_bf16; g.a_rows = head_rows; }
    g.transA = 1;
    g.B = dz[k]; g.ldb = N; g.transB = 0;
    g.C = gp(head_W[k]); g.ldc = N; g.M = head_K[k]; g.N = N; g.K = Bn; g.epilogue = EPI_ACCUM;
    DCA_TRY(gemm_auto(g, s));
    DCA_TRY(col_sums(dz[k], nullptr, N, Bn, N, d(o_dsum), nullptr, d(o_scratch), s));
    DCA_TRY(col_sum_to_float(d(o_dsum), N, gp(head_b[k]), s));
    if (!have_hidden) continue;
    // d(head input) = dz W^T: into the branch's own buffer (fork) or accumulated into the trunk gradient
    GemmArgs b{};
    b.A = dz[k]; b.lda = N; b.a_bf16 = 0; b.transA = 0; b.a_rows = nullptr;
    b.B = pp(head_W[k]); b.ldb = N; b.transB = 1;
    b.M = Bn; b.N = head_K[k]; b.K = N;
    if (br) {
      b.C = dh_tmp; b.ldc = head_K[k]; b.epilogue = EPI_STORE; b.splits = 1;
      DCA_TRY(gemm_generic(b, s));
      // branch layer backward; its input gradient accumulates into the trunk gradient
      DCA_TRY(x_layer_bwd(brlay[k], dh_tmp, f(lay[trunk_L - 1].o_h), lay[trunk_L - 1].out, 0, nullptr, Bn, dh_trunk, true, s));
    } else {
      b.C = dh_trunk; b.ldc = head_K[k]; b.epilogue = EPI_ACCUM;
      DCA_TRY(gemm_auto(b, s));
    }
  }
  mark(4, s);
  // ---- trunk backward
  float* dh = dh_trunk; float* dh2 = dh_tmp;
  for (int i = trunk_L - 1; i >= 0; --i) {
    const void* ain = (i == 0) ? X : (const void*)f(lay[i - 1].o_h);
    DCA_TRY(x_layer_bwd(lay[i], dh, ain, (i == 0) ? ldx : lay[i - 1].out, (i == 0) ? (cfg.x_dtype == DCA_BF16) : 0,
                        (i == 0) ? xrows : nullptr, Bn, i > 0 ? dh2 : nullptr, false, s));
    float* t = dh; dh = dh2; dh2 = t;
  }
  mark(-1, s);
  return DCA_OK;
}

int Engine::x_eval_step(const void* X, int64_t ldx, const float* Y, int64_t ldy, const float* sf, const int32_t* rows, int Bn,
                        cudaStream_t s) {
  const int G = cfg.n_out;
  DCA_TRY(x_forward(X, ldx, rows, Bn, false, s));
  float* Mb = f(o_head[0]); float* Db = f(o_head[1]); float* Pb = f(o_head[2]);
  DCA_TRY(x_heads_forward(Bn, Mb, cond ? Db : nullptr, has_pi ? Pb : nullptr, nullptr, s));
  if (x_kind == DCA_AE_POISSON || x_kind == DCA_AE_NORMAL) {
    double* acc = d(o_xacc);
    const int64_t n = (int64_t)Bn * G;
    DCA_CUDA_OK(cudaMemsetAsync(acc, 0, 2 * sizeof(double), s));
    if (x_kind == DCA_AE_POISSON) simple_loss_kernel<0><<<nblk(n), 256, 0, s>>>(Y, ldy, rows, sf, Mb, Bn, G, acc, 0);
    else simple_loss_kernel<1><<<nblk(n), 256, 0, s>>>(Y, ldy, rows, sf, Mb, Bn, G, acc, 0);
    DCA_LAUNCH_CHECK();
    simple_loss_finish_kernel<<<1, 1, 0, s>>>(acc, nullptr, nullptr, nullptr, d(o_acc) + 2, Bn);
    DCA_LAUNCH_CHECK();
    return DCA_OK;
  }
  LossArgs la{};
  la.Y = Y; la.ldy = ldy; la.rows = rows; la.sf = sf;
  la.m = Mb; la.d = Db; la.pi = has_pi ? Pb : nullptr; la.ld = G;
  la.B = Bn; la.G = G; la.ae_type = has_pi ? DCA_AE_ZINB_CONDDISP : DCA_AE_NB_CONDDISP; la.ridge = cfg.ridge; la.inv_n = 1.f;
  la.loss_sum = d(o_acc) + 2; la.ws = base + o_lossws; la.ws_bytes = loss_ws_bytes;
  DCA_TRY(debug_check_loss(la, s));
  DCA_TRY(zinb_loss_fwd(la, s));
  x_add_double_kernel<<<1, 1, 0, s>>>(d(o_acc) + 3, (double)Bn * (double)G);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

// predict: mean * sf [B x G], dispersion / pi [B x G] -- or [B] for the per-cell heads of the shared types -- and the
// pre-BN 'center' latent (dca/network.py:188-211, 318-339, 395-405)
int Engine::x_predict(const void* X, int64_t ldx, const float* sf, const int32_t* rows, int Bn, float* mean_out, float* disp_out,
                      float* pi_out, int64_t ld_out, float* latent_out, cudaStream_t s) {
  const int G = cfg.n_out;
  if (ld_out != G && (mean_out || !(x_kind == DCA_AE_NB_SHARED || x_kind == DCA_AE_ZINB_SHARED))) {
    set_error("dca_predict: this autoencoder type needs contiguous outputs (ld_out == n_out)"); return DCA_ERR_UNSUPPORTED;
  }
  DCA_TRY(x_forward(X, ldx, rows, Bn, false, s));
  if (latent_out) {
    if (L == 0) { set_error("dca_predict: no hidden layer -> no latent output"); return DCA_ERR_BAD_ARG; }
    const int c = L / 2;
    DCA_CUDA_OK(cudaMemcpyAsync(latent_out, f(lay[c].o_a), sizeof(float) * (size_t)Bn * lay[c].out, cudaMemcpyDeviceToDevice, s));
  }
  DCA_TRY(x_gather_sf(sf, rows, Bn, s));
  const bool shared = (x_kind == DCA_AE_NB_SHARED || x_kind == DCA_AE_ZINB_SHARED);
  if (shared) {
    if (mean_out) DCA_TRY(x_head_gemm(0, Bn, mean_out, G, EPI_MEAN_ACT, f(o_sfb), s));
    if (disp_out) DCA_TRY(x_head_gemm(1, Bn, disp_out, 1, EPI_DISP_ACT, nullptr, s));
    if (pi_out && has_pi) DCA_TRY(x_head_gemm(2, Bn, pi_out, 1, EPI_SIGMOID, nullptr, s));
    return DCA_OK;
  }
  if (x_kind == DCA_AE_ZINB_ELEMPI) {
    if (mean_out || pi_out) {
      DCA_TRY(x_head_gemm(0, Bn, f(o_zraw), G, EPI_STORE, nullptr, s));
      elempi_fwd_kernel<<<nblk((int64_t)Bn * G), 256, 0, s>>>(f(o_zraw), Bn, G, pp(epi_k), pp(epi_c), epi_n, f(o_sfb), mean_out, pi_out);
      DCA_LAUNCH_CHECK();
    }
    if (disp_out) DCA_TRY(x_head_gemm(1, Bn, disp_out, G, EPI_DISP_ACT, nullptr, s));
    return DCA_OK;
  }
  return x_heads_forward(Bn, mean_out, cond ? disp_out : nullptr, has_pi ? pi_out : nullptr, f(o_sfb), s);
}

}  // namespace dca
