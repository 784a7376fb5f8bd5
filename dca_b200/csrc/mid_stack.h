// Parameters of the fused hidden-stack kernels (mid_stack.cu).
#pragma once
#include "dca_internal.cuh"

namespace dca {
namespace mid {

constexpr int kMaxW = 64;          // widest hidden layer handled by the fused kernels
constexpr int kMaxCtas = 128;      // co-resident CTAs (one per SM, cooperative launch)
constexpr int kMaxRows = 64;       // rows per CTA strip  (=> batch <= 8192; larger batches use the per-layer kernels)
constexpr int kGradSlots = kMaxW + kMaxW * kMaxW;   // per layer: bias gradient, then the kernel gradient [w_in x w]

struct Params {
  int L, B, training, batchnorm, center, rows_per_cta, n_ctas;
  int max_ctas;                       // 0: as many as the batch wants (<= kMaxCtas); else an upper bound (SMs left to a collective)
  int w[DCA_MAX_HIDDEN];
  const float* W[DCA_MAX_HIDDEN];      // W[i], i >= 1: [w[i-1] x w[i]] (Keras)
  const float* b[DCA_MAX_HIDDEN];
  const float* beta[DCA_MAX_HIDDEN];
  float* mm[DCA_MAX_HIDDEN]; float* mv[DCA_MAX_HIDDEN];      // moving statistics
  float* mean[DCA_MAX_HIDDEN]; float* inv[DCA_MAX_HIDDEN];   // batch (or moving) statistics used
  float* xhat[DCA_MAX_HIDDEN]; float* h[DCA_MAX_HIDDEN];     // [B x w[i]] saved activations
  float* a0;                          // [B x w[0]]  in: first layer pre-activation
  float* a_center;                    // [B x w[center]] out (may equal a0 when center == 0)
  __nv_bfloat16* h_last_bf16;         // optional
  // backward
  float* dh_last;                     // [B x w[L-1]] in
  float* gW[DCA_MAX_HIDDEN]; float* gb[DCA_MAX_HIDDEN]; float* gbeta[DCA_MAX_HIDDEN];
  float* da0; __nv_bfloat16* da0_bf16;
  double* partial;                    // [n_ctas][2][kMaxW] scratch per barrier round
  float* gpart;                       // [L][kGradSlots][kMaxCtas]: per-CTA bias / kernel gradients, folded in CTA order
  unsigned* bar;                      // {count, generation}
  float eps, momentum;
  long long* dbg;                     // gg_profile: clock64 stamps of CTA 0 at the phase boundaries (nullptr = off)
};

}  // namespace mid

bool mid_supported(const int* widths, int L);
bool mid_device_ok();   // cooperative launch available and the largest grid fits the device
size_t mid_partial_doubles();
size_t mid_grad_partial_floats(int L);
int mid_forward(mid::Params& p, cudaStream_t s);
int mid_backward(mid::Params& p, cudaStream_t s);

}  // namespace dca
