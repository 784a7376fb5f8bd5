// Hidden-layer activations other than relu, PReLU's trainable slopes, and dropout (input + hidden) for the per-layer
// hidden path.  Reference: dca/network.py:98-99 (input dropout), :129-138 (activation layer, hidden dropout),
// :41 (advanced_activations), CLI flags --activation / --dropoutrate / --inputdropout (dca/__main__.py:76-84).
//
// Masks come from a counter-based generator keyed by (cfg.dropout_seed, layer, training step): the step counter lives
// in device memory and is bumped by a one-thread kernel at the start of each training step, so a captured CUDA graph
// replays with fresh masks.  The backward pass regenerates the mask instead of storing it.
#include "engine.h"
#include "activations.cuh"

namespace dca {

namespace {

struct ActSpec {
  int kind; float rate, keep, inv_keep; uint32_t thr; uint64_t seed; const unsigned long long* step; int layer;
  const float* alpha;
};

__global__ void bump_step_kernel(unsigned long long* step) { *step += 1ull; }

// h = dropout(act(BN(a)));  mean == nullptr: no BatchNorm (a already holds Dense + bias)
__global__ void act_fwd_kernel(const float* __restrict__ a, int64_t ld, int M, int N, const float* __restrict__ mean,
                               const float* __restrict__ inv_std, const float* __restrict__ beta, float* __restrict__ xhat,
                               float* __restrict__ h, __nv_bfloat16* __restrict__ hb, ActSpec sp) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)M * N) return;
  const int r = (int)(i / N), c = (int)(i % N);
  float x = a[(int64_t)r * ld + c];
  if (mean) {
    const float xh = (x - mean[c]) * inv_std[c];
    if (xhat) xhat[i] = xh;
    x = xh + beta[c];
  }
  float v = act::value(sp.kind, x, sp.alpha ? sp.alpha[c] : 0.f);
  if (sp.rate > 0.f) {
    const uint64_t key = act::drop_key(sp.seed, *sp.step, sp.layer);
    v = act::drop_keep(key, (uint64_t)i, sp.thr) ? v * sp.inv_keep : 0.f;
  }
  h[i] = v;
  if (hb) hb[i] = __float2bfloat16_rn(v);
}

// stage 0: dh <- dropout'(dh) [and, PReLU, scr <- min(x, 0) for the slope gradient]; stage 1 (or the only stage for
// parameter-free activations): dh <- dh * act'(.)
__global__ void act_bwd_kernel(float* __restrict__ dh, const float* __restrict__ h, const float* __restrict__ xhat,
                               const float* __restrict__ beta, const float* __restrict__ a, int64_t ld, int M, int N,
                               ActSpec sp, float* __restrict__ scr, int stage) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)M * N) return;
  const int r = (int)(i / N), c = (int)(i % N);
  const float g = dh[i];
  const float rate = stage == 0 ? sp.rate : 0.f;
  bool kept = true;
  if (rate > 0.f) kept = act::drop_keep(act::drop_key(sp.seed, *sp.step, sp.layer), (uint64_t)i, sp.thr);
  if (sp.kind == DCA_ACT_PRELU) {
    const float x = xhat ? xhat[i] + beta[c] : a[(int64_t)r * ld + c];
    if (stage == 0) {                                        // dropout only: the slope gradient reads this dh
      dh[i] = act::bwd_elem(DCA_ACT_LINEAR, g, 0.f, 0.f, 0.f, rate, sp.keep, sp.inv_keep, kept);
      scr[i] = fminf(x, 0.f);
      return;
    }
    dh[i] = act::bwd_elem(DCA_ACT_PRELU, g, 0.f, x, sp.alpha[c], 0.f, 1.f, 1.f, true);
    return;
  }
  // hard_sigmoid takes its derivative from the pre-activation, not from the rescaled stored h (act::bwd_elem)
  const float x = sp.kind != DCA_ACT_HARD_SIGMOID ? 0.f : xhat ? xhat[i] + beta[c] : a[(int64_t)r * ld + c];
  dh[i] = act::bwd_elem(sp.kind, g, h[i], x, 0.f, rate, sp.keep, sp.inv_keep, kept);
}

__device__ __forceinline__ float elem_to_f(float v) { return v; }
__device__ __forceinline__ float elem_to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ void elem_from_f(float& o, float v) { o = v; }
__device__ __forceinline__ void elem_from_f(__nv_bfloat16& o, float v) { o = __float2bfloat16_rn(v); }

// out[r][:] = dropout(X[rows[r]][:]) in X's own element type (bf16 or fp32), contiguous rows
template <typename T>
__global__ void drop_rows_kernel(const T* __restrict__ X, int64_t ldx, const int32_t* __restrict__ rows, int M, int n,
                                 T* __restrict__ out, ActSpec sp) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)M * n) return;
  const int r = (int)(i / n), c = (int)(i % n);
  const int64_t sr = rows ? (int64_t)rows[r] : (int64_t)r;
  const uint64_t key = act::drop_key(sp.seed, *sp.step, sp.layer);
  const float v = act::drop_keep(key, (uint64_t)i, sp.thr) ? elem_to_f(X[sr * ldx + c]) * sp.inv_keep : 0.f;
  elem_from_f(out[i], v);
}

inline unsigned blocks_of(int64_t n) { return (unsigned)((n + 255) / 256); }

}  // namespace

bool Engine::plain_hidden() const {
  if (cfg.activation != DCA_ACT_RELU || cfg.input_dropout > 0.f) return false;
  for (int i = 0; i < cfg.n_hidden; ++i) if (cfg.hidden_dropout[i] > 0.f) return false;
  return true;
}

static ActSpec make_spec(const Engine& e, const Layer& l, bool training) {
  ActSpec sp{};
  sp.kind = e.cfg.activation;
  sp.rate = training ? l.drop : 0.f;
  sp.keep = 1.f - sp.rate; sp.inv_keep = 1.f / sp.keep; sp.thr = act::drop_threshold(sp.rate);
  sp.seed = e.cfg.dropout_seed; sp.step = reinterpret_cast<const unsigned long long*>(e.base + e.o_step); sp.layer = l.id;
  sp.alpha = l.alpha >= 0 ? e.pp(l.alpha) : nullptr;
  return sp;
}

int Engine::bump_step(cudaStream_t s) {
  bump_step_kernel<<<1, 1, 0, s>>>(reinterpret_cast<unsigned long long*>(base + o_step));
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

// BatchNorm normalisation (statistics already in o_mean / o_inv) + activation + dropout of one hidden layer
int Engine::act_fwd(Layer& l, int Bn, bool training, __nv_bfloat16* hb, cudaStream_t s) {
  float* a = f(l.o_a);
  if (cfg.activation == DCA_ACT_RELU && !(training && l.drop > 0.f)) {       // the relu-only kernels of the default model
    if (cfg.batchnorm)
      return bn_relu_fwd(a, l.out, Bn, l.out, f(l.o_mean), f(l.o_inv), pp(l.beta), training ? f(l.o_xhat) : nullptr, f(l.o_h), hb, s);
    return bias_relu_fwd(a, l.out, Bn, l.out, f(l.o_h), hb, s);
  }
  const ActSpec sp = make_spec(*this, l, training);
  act_fwd_kernel<<<blocks_of((int64_t)Bn * l.out), 256, 0, s>>>(
      a, l.out, Bn, l.out, cfg.batchnorm ? f(l.o_mean) : nullptr, cfg.batchnorm ? f(l.o_inv) : nullptr,
      cfg.batchnorm ? pp(l.beta) : nullptr, (cfg.batchnorm && training) ? f(l.o_xhat) : nullptr, f(l.o_h), hb, sp);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

// dh (gradient w.r.t. the layer's output, after dropout) -> gradient w.r.t. the activation's input, in place;
// PReLU: also the slope gradient
int Engine::act_bwd(Layer& l, float* dh, int Bn, cudaStream_t s) {
  if (cfg.activation == DCA_ACT_RELU && !(l.drop > 0.f)) return relu_bwd(dh, f(l.o_h), l.out, Bn, l.out, s);
  const ActSpec sp = make_spec(*this, l, true);
  const float* xhat = cfg.batchnorm ? f(l.o_xhat) : nullptr;
  const float* beta = cfg.batchnorm ? pp(l.beta) : nullptr;
  const unsigned nb = blocks_of((int64_t)Bn * l.out);
  if (cfg.activation == DCA_ACT_PRELU) {
    float* scr = f(o_actscr);
    act_bwd_kernel<<<nb, 256, 0, s>>>(dh, f(l.o_h), xhat, beta, f(l.o_a), l.out, Bn, l.out, sp, scr, 0);
    DCA_LAUNCH_CHECK();
    DCA_TRY(col_sums(dh, scr, l.out, Bn, l.out, d(o_dsum), d(o_dprod), d(o_scratch), s));
    DCA_TRY(col_sum_to_float(d(o_dprod), l.out, gp(l.alpha), s));
    act_bwd_kernel<<<nb, 256, 0, s>>>(dh, f(l.o_h), xhat, beta, f(l.o_a), l.out, Bn, l.out, sp, scr, 1);
    DCA_LAUNCH_CHECK();
    return DCA_OK;
  }
  act_bwd_kernel<<<nb, 256, 0, s>>>(dh, f(l.o_h), xhat, beta, f(l.o_a), l.out, Bn, l.out, sp, nullptr, 0);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

// Input dropout: the batch's rows, gathered and masked, as a contiguous matrix in X's element type (arena: o_xdrop)
int Engine::drop_input(const void* X, int in_bf16, int64_t ldx, const int32_t* rows, int Bn, cudaStream_t s) {
  Layer in{}; in.drop = cfg.input_dropout; in.id = -1;
  ActSpec sp = make_spec(*this, in, true);
  const int64_t n = (int64_t)Bn * cfg.n_in;
  if (in_bf16)
    drop_rows_kernel<__nv_bfloat16><<<blocks_of(n), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(X), ldx, rows, Bn, cfg.n_in,
                                                                 bf(o_xdrop), sp);
  else
    drop_rows_kernel<float><<<blocks_of(n), 256, 0, s>>>(reinterpret_cast<const float*>(X), ldx, rows, Bn, cfg.n_in, f(o_xdrop), sp);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

}  // namespace dca

// ---- host mirrors (include/dca_b200.h)
extern "C" int dca_dropout_mask_host(uint64_t seed, uint64_t step, int32_t layer, int64_t n, float rate, uint8_t* keep) {
  if (!keep || n < 0 || !(rate >= 0.f && rate < 1.f)) return DCA_ERR_BAD_ARG;
  const uint64_t key = dca::act::drop_key(seed, step, layer);
  const uint32_t thr = dca::act::drop_threshold(rate);
  for (int64_t i = 0; i < n; ++i) keep[i] = dca::act::drop_keep(key, (uint64_t)i, thr) ? 1 : 0;
  return DCA_OK;
}

extern "C" int dca_activation_host(int32_t act, float x, float alpha, float out[2]) {
  if (!out || act < DCA_ACT_RELU || act > DCA_ACT_PRELU) return DCA_ERR_BAD_ARG;
  out[0] = dca::act::value(act, x, alpha);
  out[1] = dca::act::deriv(act, out[0], x, alpha);
  return DCA_OK;
}

extern "C" int dca_activation_bwd_host(int32_t act, float x, float alpha, float rate, int32_t kept, float g, float out[2]) {
  if (!out || act < DCA_ACT_RELU || act > DCA_ACT_PRELU || !(rate >= 0.f && rate < 1.f)) return DCA_ERR_BAD_ARG;
  const float keep = 1.f - rate, inv_keep = 1.f / keep;
  const float v = dca::act::value(act, x, alpha);
  out[0] = rate > 0.f ? (kept ? v * inv_keep : 0.f) : v;                    // the stored output, as act_fwd_kernel writes it
  out[1] = dca::act::bwd_elem(act, g, out[0], x, alpha, rate, keep, inv_keep, rate <= 0.f || kept != 0);
  return DCA_OK;
}
