// Output activations of the three heads as evaluated in the tensor-core epilogues (dca/network.py:38-39,369):
// MeanAct = clip(exp(z), 1e-5, 1e6), DispAct = clip(softplus(z), 1e-4, 1e4), sigmoid.  One definition shared by
// the head-forward kernel (dense_tc.cu) and the fused head/loss/backward kernel (flash_zinb.cu) so that both
// produce bit-identical head outputs.
#pragma once
#include "tc_common.cuh"

namespace dca {
namespace tc {

__device__ __forceinline__ float act_mean(float z) { return fminf(fmaxf(ex2f(z * 1.442695041f), 1e-5f), 1e6f); }
// softplus(z) = max(z,0) + log1p(exp(-|z|)), branch-free; log1p by series when exp(-|z|) is small
__device__ __forceinline__ float act_disp(float z) {
  const float e = ex2f(-fabsf(z) * 1.442695041f);                       // (0, 1]
  const float l_series = e * fmaf(e, fmaf(e, 0.333333333f, -0.5f), 1.0f);
  const float l_log = 0.693147181f * lg2f(1.0f + e);
  const float sp = fmaxf(z, 0.f) + (e < 0.01f ? l_series : l_log);
  return fminf(fmaxf(sp, 1e-4f), 1e4f);
}
__device__ __forceinline__ float act_sigmoid(float z) { return rcpf(1.0f + ex2f(-z * 1.442695041f)); }

}  // namespace tc
}  // namespace dca
