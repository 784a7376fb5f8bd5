// Output activations of the three heads as evaluated in the tensor-core epilogues (dca/network.py:38-39,369):
// MeanAct = clip(exp(z), 1e-5, 1e6), DispAct = clip(softplus(z), 1e-4, 1e4), sigmoid.  One definition shared by
// the head-forward kernel (dense_tc.cu) and the fused head/loss/backward kernel (flash_zinb.cu) so that both
// produce bit-identical head outputs.
#pragma once
#include "dca_internal.cuh"
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

// Pre-activations of one 64-cell x 128-gene head tile, issued by one warpgroup: H (K-major, 64 rows of 128 B, SWIZZLE_128B,
// 32 B per k16 step) times W (MN-major, the Keras [64 k][genes] layout as two 64-gene boxes 8 KB apart, 2 KB per k16 step),
// four k16 steps from a zero accumulator.  The head-forward kernel's product (dense_tc.cu); the heads + loss kernel
// (zinb_loss.cu) computes the same products gene-major with head_piece_mma.
__device__ __forceinline__ void head_tile_mma(float (&acc)[64], uint32_t h_smem, uint32_t w_smem) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k)
    wgmma_m64n128k16<0, 1>(acc, make_smem_desc(h_smem + k * 32, 0, 1024), make_smem_desc(w_smem + k * 2048, 8192, 1024), k > 0);
  wgmma_commit();
  wgmma_wait<0>();
  acc_fence(acc);
}

// Gene-major pre-activations of one head for 16 cells, issued by one warpgroup: D[128 genes x 16 cells] = Wᵀ . Hᵀ as two
// m64n16 m-blocks (genes 0-63 | 64-127, acc[0] | acc[1]) of four k16 steps from a zero accumulator.  A = W, MN-major (the
// same two 64-gene boxes as head_tile_mma's B operand, one box per m-block); B = 16 consecutive rows of H (K-major,
// h_smem 1024-byte aligned, i.e. a multiple of 8 rows into the swizzled block).  Commits one wgmma group and does not
// wait: the caller waits (wgmma_wait) and fences the accumulators before reading them.  Thread t holds acc[mb][i] at
// gene 64 mb + 16 (t/32 % 4) + (t%32)/4 + 8 ((i/2)%2), cell 8 (i/4) + 2 (t%4) + i%2.
__device__ __forceinline__ void head_piece_mma(float (&acc)[2][8], uint32_t h_smem, uint32_t w_smem) {
  wgmma_fence();
#pragma unroll
  for (int mb = 0; mb < 2; ++mb)
#pragma unroll
    for (int k = 0; k < 4; ++k)
      wgmma_m64n16k16<1, 0>(acc[mb], make_smem_desc(w_smem + mb * 8192 + k * 2048, 8192, 1024),
                            make_smem_desc(h_smem + k * 32, 0, 1024), k > 0);
  wgmma_commit();
}

// Epilogue of one head output: activation of (accumulator + bias), MeanAct scaled by the row's scale (1 in training).
// KIND: EPI_MEAN_ACT / EPI_DISP_ACT / EPI_SIGMOID.
template <int KIND>
__device__ __forceinline__ float head_out(float acc, float bias, float row_scale) {
  const float z = acc + bias;
  if (KIND == EPI_MEAN_ACT) return act_mean(z) * row_scale;
  if (KIND == EPI_DISP_ACT) return act_disp(z);
  return act_sigmoid(z);
}

}  // namespace tc
}  // namespace dca
