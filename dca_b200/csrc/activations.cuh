// Hidden-layer activation and dropout arithmetic, shared by the device kernels (activations.cu) and their host
// mirrors (dca_activation_host / dca_dropout_mask_host).
//
// Reference behaviour: dca/network.py:129-138 -- after each hidden Dense (+ BatchNormalization) comes
// `Activation(self.activation)` or, for 'PReLU' / 'LeakyReLU' (network.py:41), the Keras layer of that name with default
// arguments, then `Dropout(hid_drop)` when the rate is > 0; network.py:98-99 puts `Dropout(input_dropout)` on the input.
// Keras Dropout in training mode: x * mask / (1 - rate), mask ~ Bernoulli(1 - rate); identity at inference.
#pragma once
#include <stdint.h>
#include <math.h>
#include "../../include/dca_b200.h"

#if defined(__CUDACC__)
#define DCA_HD __host__ __device__ __forceinline__
#else
#define DCA_HD inline
#endif

namespace dca {
namespace act {

constexpr float kSeluScale = 1.0507009873554805f;
constexpr float kSeluAlpha = 1.6732632423543772f;
constexpr float kLeakySlope = 0.3f;                 // keras.layers.LeakyReLU() default

DCA_HD float value(int kind, float x, float alpha) {
  switch (kind) {
    case DCA_ACT_RELU: return fmaxf(x, 0.f);
    case DCA_ACT_LINEAR: return x;
    case DCA_ACT_ELU: return x > 0.f ? x : expm1f(x);
    case DCA_ACT_SELU: return kSeluScale * (x > 0.f ? x : kSeluAlpha * expm1f(x));
    case DCA_ACT_TANH: return tanhf(x);
    case DCA_ACT_SIGMOID: return 1.f / (1.f + expf(-x));
    case DCA_ACT_HARD_SIGMOID: return fminf(fmaxf(0.2f * x + 0.5f, 0.f), 1.f);
    case DCA_ACT_SOFTPLUS: return x > 20.f ? x : log1pf(expf(x));
    case DCA_ACT_SOFTSIGN: return x / (1.f + fabsf(x));
    case DCA_ACT_EXPONENTIAL: return expf(x);
    case DCA_ACT_LEAKY_RELU: return x > 0.f ? x : kLeakySlope * x;
    case DCA_ACT_PRELU: return x > 0.f ? x : alpha * x;
    default: return x;
  }
}

// d value / d x from the activation's OUTPUT h (what the forward pass keeps); PReLU needs the input x as well
DCA_HD float deriv(int kind, float h, float x, float alpha) {
  switch (kind) {
    case DCA_ACT_RELU: return h > 0.f ? 1.f : 0.f;
    case DCA_ACT_LINEAR: return 1.f;
    case DCA_ACT_ELU: return h > 0.f ? 1.f : h + 1.f;
    case DCA_ACT_SELU: return h > 0.f ? kSeluScale : h + kSeluScale * kSeluAlpha;
    case DCA_ACT_TANH: return 1.f - h * h;
    case DCA_ACT_SIGMOID: return h * (1.f - h);
    case DCA_ACT_HARD_SIGMOID: return (h > 0.f && h < 1.f) ? 0.2f : 0.f;
    case DCA_ACT_SOFTPLUS: return -expm1f(-h);                       // sigmoid(x) = 1 - exp(-softplus(x))
    case DCA_ACT_SOFTSIGN: { const float t = 1.f - fabsf(h); return t * t; }
    case DCA_ACT_EXPONENTIAL: return h;
    case DCA_ACT_LEAKY_RELU: return h > 0.f ? 1.f : kLeakySlope;
    case DCA_ACT_PRELU: return x > 0.f ? 1.f : (x < 0.f ? alpha : 0.f);
    default: return 1.f;
  }
}

// One element of the backward pass through activation + dropout (rate 0: no dropout): the gradient w.r.t. the
// activation's input x from the gradient g w.r.t. the layer's output, the stored output h (the activation times
// inv_keep where kept) and the keep flag.  The activation is recovered as h * keep, which is off by an ulp: harmless for
// the continuous derivatives, but a saturated hard_sigmoid unit (value 1) comes back as 1 - 2^-24 at rates such as 0.01,
// 0.11, 0.15, 0.23 and 0.77 and would get slope 0.2.  hard_sigmoid and PReLU take their derivative from x instead.
DCA_HD float bwd_elem(int kind, float g, float h, float x, float alpha, float rate, float keep, float inv_keep, bool kept) {
  if (rate > 0.f) {
    if (!kept) return 0.f;
    g = g * inv_keep;
  }
  if (kind == DCA_ACT_HARD_SIGMOID) return g * deriv(kind, value(kind, x, 0.f), x, 0.f);
  if (kind == DCA_ACT_PRELU) return g * deriv(kind, 0.f, x, alpha);
  return g * deriv(kind, rate > 0.f ? h * keep : h, x, alpha);
}

// ---- counter-based dropout masks: one 64-bit mix per element, keyed by (seed, layer, training step)
DCA_HD uint64_t mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
DCA_HD uint64_t drop_key(uint64_t seed, uint64_t step, int layer) {
  return mix64(seed ^ mix64(step * 1024ull + (uint64_t)(layer + 8)));
}
DCA_HD bool drop_keep(uint64_t key, uint64_t idx, uint32_t thr) {       // thr = keep probability in 2^-24 units
  return (uint32_t)(mix64(key + idx) >> 40) < thr;
}
inline uint32_t drop_threshold(float rate) { return (uint32_t)((1.0 - (double)rate) * 16777216.0); }

}  // namespace act
}  // namespace dca
