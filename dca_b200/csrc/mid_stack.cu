// Fused hidden stack ("K7"): everything between the first Dense layer's pre-activation and the last
// hidden activation, forward and backward, in ONE launch each (dca/network.py:124-139 for every hidden
// layer: [Dense ->] BatchNormalization(center, no scale) -> relu).  The tensors are tiny (B x <=64), the
// work is latency-bound, and training-mode BatchNorm needs full-batch column statistics before it can
// normalise -- so the kernel runs as <= 128 co-resident CTAs that own a strip of rows each, keep the
// strip in shared memory across layers, and meet at a grid-wide barrier once per BatchNorm layer.
//
//   forward : a_0 (given, bias included) -> BN/relu -> [Dense -> BN/relu]* -> h_last (fp32 + bf16)
//             saves x_hat_i, h_i (training) for the backward pass, the pre-BN 'center' output (latent,
//             dca/network.py:184-185) and updates the moving statistics (momentum 0.99).
//   backward: dh_last -> for each layer: relu mask, BN backward (two column sums -> barrier), bias / beta /
//             kernel gradients of the inner layers (per-CTA partials, added to the flat gradient buffer in CTA
//             order after a last barrier), dh of the previous layer; ends with da_0 (fp32 + bf16) for the first
//             layer's weight gradient.
#include "dca_internal.cuh"
#include "mid_stack.h"
#include <cstdio>
#include <cstdlib>

namespace dca {
namespace mid {

constexpr int kThreads = 256;
#define MID_STAMP(i) do { if (p.dbg && blockIdx.x == 0 && threadIdx.x == 0) p.dbg[i] = clock64(); } while (0)
constexpr int kGenWord = 32;       // generation counter lives 128 bytes after the arrival counter
constexpr int kStripStride = kMaxW + 4;   // activation strips: rows 16-byte aligned (float4 broadcasts along k)
typedef float Strip[kStripStride];        // lanes always differ in the COLUMN of a strip -> no bank conflicts
typedef float WRow[kMaxW + 1];            // weights: lanes differ in the ROW -> odd stride

// Self-resetting sense-reversal barrier over the whole (co-resident) grid.
__device__ __forceinline__ void grid_barrier(unsigned* bar, unsigned n, unsigned& gen) {
  __syncthreads();
  if (threadIdx.x == 0) {
    // release this CTA's writes (made visible to thread 0 by the block barrier) / acquire the others': an acq_rel fence at
    // gpu scope is what the pattern needs; __threadfence() is the sequentially consistent MEMBAR.SC
    asm volatile("fence.acq_rel.gpu;" ::: "memory");
    // bar[0] = arrival count, bar[kGenWord] = generation (separate 128-byte lines: pollers do not slow arrivals)
    const unsigned arrived = atomicAdd(&bar[0], 1u);
    if (arrived == n - 1) {
      bar[0] = 0;
      asm volatile("fence.acq_rel.gpu;" ::: "memory");
      atomicAdd(&bar[kGenWord], 1u);
    } else {
      // bounded: the kernels are launched cooperatively (co-residency is guaranteed by the driver), so a barrier that
      // does not open within seconds means a lost participant -- trap (kernel error) instead of hanging the GPU
      unsigned cur, polls = 0;
      long long t0 = 0;
      for (;;) {
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(cur) : "l"(&bar[kGenWord]) : "memory");
        if (cur != gen) break;
        __nanosleep(40);
        if ((++polls & 0xFFF) == 0) {
          const long long now = clock64();
          if (t0 == 0) t0 = now;
          else if (now - t0 > 8000000000ll) __trap();
        }
      }
    }
    asm volatile("fence.acq_rel.gpu;" ::: "memory");
  }
  ++gen;
  __syncthreads();
}

// column sums over this CTA's rows of s1 = sum(x) and s2 = sum(x*y) (double), x,y in smem [rows][kMaxW]
__device__ __forceinline__ void cta_col_sums(Strip* x, Strip* y, int rows, int w,
                                             double* out /* [2][kMaxW] global */, double (*red)[kMaxW]) {
  // 256 threads: 4 row-groups x 64 columns
  const int c = threadIdx.x & 63, g = threadIdx.x >> 6;
  double s1 = 0.0, s2 = 0.0;
  if (c < w)
    for (int r = g; r < rows; r += 4) { const double a = x[r][c]; s1 += a; s2 += a * (double)y[r][c]; }
  red[g][c] = s1; red[4 + g][c] = s2;
  __syncthreads();
  // partial layout: [stat k][column c][cta]  (so that the fold reads contiguous CTAs per column)
  if (threadIdx.x < 64 && c < w) {
    out[(size_t)c * kMaxCtas] = red[0][c] + red[1][c] + red[2][c] + red[3][c];
    out[(size_t)(kMaxW + c) * kMaxCtas] = red[4][c] + red[5][c] + red[6][c] + red[7][c];
  }
}

// tot[k][c] = sum over CTAs in a fixed order (deterministic).  A warp owns 16 of the 128 (stat, column) pairs; its lanes read
// CONSECUTIVE CTAs of a pair (one coalesced 256-byte request per 32 CTAs -- the first version gave every thread its own
// 256-byte run: 32 sectors per warp instruction, 9 k cycles per fold, gg_profile), then a shuffle tree joins the lanes.
__device__ __forceinline__ void fold_partials(const double* partial, int n_ctas, int w, double* tot /* smem [2][kMaxW] */) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kPairsPerWarp = 2 * kMaxW / (kThreads / 32), kPer = kMaxCtas / 32;
  // every load first (64 independent 8-byte loads per thread, ONE round trip to L2), then the adds: written pair by pair
  // the compiler emitted load-load-load-load-add-add-add-add per pair and the in-order issue serialised 16 round trips
  double x[kPairsPerWarp][kPer];
#pragma unroll
  for (int i = 0; i < kPairsPerWarp; ++i) {
    const int pair = warp + i * (kThreads / 32), c = pair & (kMaxW - 1);
    const double* src = partial + (size_t)pair * kMaxCtas;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int cta = j * 32 + lane;
      x[i][j] = (c < w && cta < n_ctas) ? __ldcg(src + cta) : 0.0;
    }
  }
#pragma unroll
  for (int i = 0; i < kPairsPerWarp; ++i) {
    double sacc = x[i][0];
#pragma unroll
    for (int j = 1; j < kPer; ++j) sacc += x[i][j];
    x[i][0] = sacc;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
#pragma unroll
    for (int i = 0; i < kPairsPerWarp; ++i) x[i][0] += __shfl_xor_sync(0xffffffffu, x[i][0], o);
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < kPairsPerWarp; ++i) tot[warp + i * (kThreads / 32)] = x[i][0];
  }
  __syncthreads();
}

// out[r][c] = sum_k in[r][k] * W[k][c] (+ bias[c]).  Thread = column c, 4 rows at a time; k in groups of 4 with
// one 128-bit broadcast load per row: 8 shared loads per 16 FMA.  Padded rows / columns of `in` are zero.
__device__ __forceinline__ void strip_gemm(Strip* in, WRow* Ws, const float* bias, int rows, int w_in, int w_out, Strip* out) {
  const int c = threadIdx.x & 63, g = threadIdx.x >> 6;      // 4 row groups
  if (c < w_out) {
    const float bv = bias ? bias[c] : 0.f;
    for (int r0 = g * 4; r0 < rows; r0 += 16) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
      for (int k = 0; k < w_in; k += 4) {
        const float w0 = Ws[k][c], w1 = Ws[k + 1][c], w2 = Ws[k + 2][c], w3 = Ws[k + 3][c];   // rows >= w_in are zero
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float4 x = *reinterpret_cast<const float4*>(&in[r0 + j][k]);
          acc[j] = fmaf(x.x, w0, fmaf(x.y, w1, fmaf(x.z, w2, fmaf(x.w, w3, acc[j]))));
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (r0 + j < rows) out[r0 + j][c] = acc[j] + bv;
    }
  }
}

constexpr size_t kStripFloats = (size_t)(kMaxRows + 4) * kStripStride;
constexpr size_t kWsFloats = (size_t)kMaxW * (kMaxW + 1);
constexpr int kWSlots = DCA_MAX_HIDDEN - 1;      // forward: every inner kernel resident at once
constexpr size_t kSmemBytes = sizeof(double) * (8 * kMaxW + 2 * kMaxW) + sizeof(float) * (2 * kStripFloats + kWSlots * kWsFloats + 2 * kMaxW) + 16;

__global__ void __launch_bounds__(kThreads, 1) mid_forward_kernel(const Params p) {
  extern __shared__ __align__(16) unsigned char smem_mid[];
  double (*red)[kMaxW] = reinterpret_cast<double (*)[kMaxW]>(smem_mid);
  double* tot = reinterpret_cast<double*>(smem_mid) + 8 * kMaxW;
  float* fbase = reinterpret_cast<float*>(tot + 2 * kMaxW);
  Strip* cur = reinterpret_cast<Strip*>(fbase);                       // current layer pre-activation / activation strip
  Strip* nxt = reinterpret_cast<Strip*>(fbase + kStripFloats);
  WRow* Ws = reinterpret_cast<WRow*>(fbase + 2 * kStripFloats);
  float* s_mean = fbase + 2 * kStripFloats + kWSlots * kWsFloats;
  float* s_inv = s_mean + kMaxW;
  __shared__ unsigned s_gen;
  if (threadIdx.x == 0) s_gen = *reinterpret_cast<volatile unsigned*>(&p.bar[kGenWord]);
  __syncthreads();
  unsigned gen = s_gen;
  MID_STAMP(0);

  const int row0 = blockIdx.x * p.rows_per_cta;
  const int rows = max(0, min(p.rows_per_cta, p.B - row0));
  for (int i = threadIdx.x; i < (int)kStripFloats; i += kThreads) { (&cur[0][0])[i] = 0.f; (&nxt[0][0])[i] = 0.f; }
  __syncthreads();
  // thread -> (column tc, row lane tr): no integer divisions in the element loops (widths <= 64)
  const int tc = threadIdx.x & 63, tr = threadIdx.x >> 6;
  // Prologue loads, ALL issued before the first dependent shared-memory store (in-order issue: a store that waits for its
  // load blocks the loads behind it): the a_0 strip and every inner kernel (slot l - 1, zero-padded) -- the layer loop then
  // never waits for a global load between two grid barriers.
  constexpr int kRowIters = kMaxRows / 4, kKIters = kMaxW / 4;
  float a0r[kRowIters];
#pragma unroll
  for (int i = 0; i < kRowIters; ++i) {
    const int r = tr + 4 * i;
    a0r[i] = (tc < p.w[0] && r < rows) ? p.a0[(size_t)(row0 + r) * p.w[0] + tc] : 0.f;
  }
  for (int l0 = 1; l0 < p.L; l0 += 2) {
    float wr[2][kKIters];
#pragma unroll
    for (int d = 0; d < 2; ++d) {
      const int l = l0 + d;
      const int win = l < p.L ? p.w[l - 1] : 0, w = l < p.L ? p.w[l] : 0;
#pragma unroll
      for (int i = 0; i < kKIters; ++i) { const int k = tr + 4 * i; wr[d][i] = (k < win && tc < w) ? p.W[l][(size_t)k * w + tc] : 0.f; }
    }
#pragma unroll
    for (int d = 0; d < 2; ++d) {
      if (l0 + d >= p.L) break;
      WRow* Wl = Ws + (size_t)(l0 + d - 1) * kMaxW;
#pragma unroll
      for (int i = 0; i < kKIters; ++i) Wl[tr + 4 * i][tc] = wr[d][i];
    }
  }
  // CTA 0 updates the moving statistics: their old values are fetched here, not between the barriers
  float mm_old[DCA_MAX_HIDDEN], mv_old[DCA_MAX_HIDDEN];
#pragma unroll
  for (int l = 0; l < DCA_MAX_HIDDEN; ++l) {
    const bool mine = p.batchnorm && p.training && blockIdx.x == 0 && l < p.L && (int)threadIdx.x < p.w[l];
    mm_old[l] = mine ? p.mm[l][threadIdx.x] : 0.f; mv_old[l] = mine ? p.mv[l][threadIdx.x] : 0.f;
  }
  float beta_r[DCA_MAX_HIDDEN];                 // this thread's column of every layer's beta (same reason)
#pragma unroll
  for (int l = 0; l < DCA_MAX_HIDDEN; ++l) beta_r[l] = (p.batchnorm && l < p.L && tc < p.w[l]) ? p.beta[l][tc] : 0.f;
  if (tc < p.w[0]) {
#pragma unroll
    for (int i = 0; i < kRowIters; ++i) { const int r = tr + 4 * i; if (r < rows) cur[r][tc] = a0r[i]; }
  }
  __syncthreads();
  MID_STAMP(1);
  Strip* a = cur;
  Strip* o = nxt;
  for (int l = 0; l < p.L; ++l) {
    const int w = p.w[l];
    if (l > 0) {
      const int win = p.w[l - 1];
      strip_gemm(a, Ws + (size_t)(l - 1) * kMaxW, p.b[l], rows, win, w, o);
      __syncthreads();
      Strip* t = a; a = o; o = t;
      MID_STAMP(2 + l * 5);
    }
    if (l == p.center && p.a_center && !(l == 0 && p.a_center == p.a0) && tc < w)
      for (int r = tr; r < rows; r += 4) p.a_center[(size_t)(row0 + r) * w + tc] = a[r][tc];
    if (p.batchnorm) {
      if (p.training) {
        double* part = p.partial + (size_t)(l & 1) * kMaxCtas * 2 * kMaxW;       // double-buffered across layers
        cta_col_sums(a, a, rows, w, part + blockIdx.x, red);
        MID_STAMP(3 + l * 5);
        grid_barrier(p.bar, gridDim.x, gen);
        MID_STAMP(4 + l * 5);
        fold_partials(part, gridDim.x, w, tot);
        MID_STAMP(5 + l * 5);
        if (threadIdx.x < w) {
          const int c = threadIdx.x;
          const double inv_b = 1.0 / (double)p.B;                    // (one division; B is a launch constant)
          const double mu = tot[c] * inv_b;
          double var = tot[kMaxW + c] * inv_b - mu * mu;             // biased batch variance
          if (var < 0.0) var = 0.0;
          s_mean[c] = (float)mu;
          // 1 / sqrt(var + eps): float rsqrt + one Newton step (2e-7 relative) instead of a double sqrt and division
          const float vf = (float)(var + (double)p.eps);
          float r = rsqrtf(vf);
          r = r * (1.5f - 0.5f * vf * r * r);
          s_inv[c] = r;
          if (blockIdx.x == 0) {
            p.mean[l][c] = s_mean[c]; p.inv[l][c] = r;
#pragma unroll
            for (int q = 0; q < DCA_MAX_HIDDEN; ++q)
              if (q == l) {
                p.mm[l][c] = p.momentum * mm_old[q] + (1.0f - p.momentum) * (float)mu;
                p.mv[l][c] = p.momentum * mv_old[q] + (1.0f - p.momentum) * (float)var;
              }
          }
        }
        __syncthreads();
      } else {
        if (threadIdx.x < w) { s_mean[threadIdx.x] = p.mm[l][threadIdx.x]; s_inv[threadIdx.x] = rsqrtf(p.mv[l][threadIdx.x] + p.eps); }
        __syncthreads();
      }
    }
    const bool last = (l == p.L - 1);
    if (tc < w) {
      const float mean_c = p.batchnorm ? s_mean[tc] : 0.f, inv_c = p.batchnorm ? s_inv[tc] : 1.f;
      float beta_c = 0.f;
#pragma unroll
      for (int q = 0; q < DCA_MAX_HIDDEN; ++q) if (q == l) beta_c = beta_r[q];
      for (int r = tr; r < rows; r += 4) {
        const size_t gi = (size_t)(row0 + r) * w + tc;
        float v = a[r][tc];
        if (p.batchnorm) {
          const float xh = (v - mean_c) * inv_c;
          if (p.training) p.xhat[l][gi] = xh;
          v = xh + beta_c;
        }
        v = fmaxf(v, 0.f);
        a[r][tc] = v;
        p.h[l][gi] = v;
        if (last && p.h_last_bf16) p.h_last_bf16[gi] = __float2bfloat16_rn(v);
      }
    }
    __syncthreads();
    MID_STAMP(6 + l * 5);
  }
  MID_STAMP(31);
}

__global__ void __launch_bounds__(kThreads, 1) mid_backward_kernel(const Params p) {
  extern __shared__ __align__(16) unsigned char smem_mid[];
  double (*red)[kMaxW] = reinterpret_cast<double (*)[kMaxW]>(smem_mid);
  double* tot = reinterpret_cast<double*>(smem_mid) + 8 * kMaxW;
  float* fbase = reinterpret_cast<float*>(tot + 2 * kMaxW);
  Strip* g = reinterpret_cast<Strip*>(fbase);                         // gradient strip of the current layer
  Strip* xh = reinterpret_cast<Strip*>(fbase + kStripFloats);         // x_hat strip / previous activation strip
  WRow* Ws = reinterpret_cast<WRow*>(fbase + 2 * kStripFloats);
  __shared__ unsigned s_gen;
  if (threadIdx.x == 0) s_gen = *reinterpret_cast<volatile unsigned*>(&p.bar[kGenWord]);
  __syncthreads();
  unsigned gen = s_gen;
  MID_STAMP(0);

  const int row0 = blockIdx.x * p.rows_per_cta;
  const int rows = max(0, min(p.rows_per_cta, p.B - row0));
  for (int i = threadIdx.x; i < (int)kStripFloats; i += kThreads) { (&g[0][0])[i] = 0.f; (&xh[0][0])[i] = 0.f; }
  for (int i = threadIdx.x; i < (int)kWsFloats; i += kThreads) (&Ws[0][0])[i] = 0.f;
  __syncthreads();
  const int tc = threadIdx.x & 63, tr = threadIdx.x >> 6;
  float* s_mg = reinterpret_cast<float*>(Ws);          // per-column means of the BN backward (Ws is free at that point)
  {
    const int w = p.w[p.L - 1];
    if (tc < w)
      for (int r = tr; r < rows; r += 4) g[r][tc] = p.dh_last[(size_t)(row0 + r) * w + tc];
  }
  __syncthreads();
  MID_STAMP(1);
  for (int l = p.L - 1; l >= 0; --l) {
    const int w = p.w[l];
    float* gpart_l = p.gpart + (size_t)l * kGradSlots * kMaxCtas + blockIdx.x;   // this CTA's column of the layer's slots
    // relu mask (+ load x_hat): loads first, then the dependent shared-memory traffic
    {
      constexpr int kRowIters = kMaxRows / 4;
      float hr[kRowIters], xr[kRowIters];
#pragma unroll
      for (int i = 0; i < kRowIters; ++i) {
        const int r = tr + 4 * i;
        const bool ok = tc < w && r < rows;
        const size_t gi = (size_t)(row0 + r) * w + tc;
        hr[i] = ok ? p.h[l][gi] : 0.f;
        xr[i] = (ok && p.batchnorm) ? p.xhat[l][gi] : 0.f;
      }
      if (tc < w) {
#pragma unroll
        for (int i = 0; i < kRowIters; ++i) {
          const int r = tr + 4 * i;
          if (r < rows) { if (!(hr[i] > 0.f)) g[r][tc] = 0.f; xh[r][tc] = xr[i]; }
        }
      }
    }
    __syncthreads();
    MID_STAMP(2 + (p.L - 1 - l) * 8);
    if (p.batchnorm) {
      double* part = p.partial + (size_t)(l & 1) * kMaxCtas * 2 * kMaxW;
      cta_col_sums(g, xh, rows, w, part + blockIdx.x, red);
      MID_STAMP(3 + (p.L - 1 - l) * 8);
      grid_barrier(p.bar, gridDim.x, gen);
      MID_STAMP(4 + (p.L - 1 - l) * 8);
      fold_partials(part, gridDim.x, w, tot);
      MID_STAMP(5 + (p.L - 1 - l) * 8);
      if (blockIdx.x == 0 && threadIdx.x < w) p.gbeta[l][threadIdx.x] = (float)tot[threadIdx.x];   // d beta = sum(g)
      if (threadIdx.x < w) {
        s_mg[threadIdx.x] = (float)(tot[threadIdx.x] / (double)p.B);
        s_mg[kMaxW + threadIdx.x] = (float)(tot[kMaxW + threadIdx.x] / (double)p.B);
        s_mg[2 * kMaxW + threadIdx.x] = p.inv[l][threadIdx.x];
      }
      __syncthreads();
      if (tc < w) {
        const float mg = s_mg[tc], mgx = s_mg[kMaxW + tc], inv_c = s_mg[2 * kMaxW + tc];
        for (int r = tr; r < rows; r += 4) g[r][tc] = inv_c * (g[r][tc] - mg - xh[r][tc] * mgx);
      }
      __syncthreads();
    }
    // bias gradient: column sums of da over my rows
    {
      const int c = threadIdx.x & 63, q = threadIdx.x >> 6;
      float s = 0.f;
      if (c < w) for (int r = q; r < rows; r += 4) s += g[r][c];
      red[q][c] = (double)s;
      __syncthreads();
      if (threadIdx.x < w) gpart_l[(size_t)threadIdx.x * kMaxCtas] = (float)(red[0][c] + red[1][c] + red[2][c] + red[3][c]);
      __syncthreads();
    }
    MID_STAMP(6 + (p.L - 1 - l) * 8);
    if (l == 0) {
      if (tc < w)
        for (int r = tr; r < rows; r += 4) {
          const size_t gi = (size_t)(row0 + r) * w + tc;
          if (p.da0) p.da0[gi] = g[r][tc];
          if (p.da0_bf16) p.da0_bf16[gi] = __float2bfloat16_rn(g[r][tc]);
        }
      break;
    }
    // ---- inner layer l >= 1: dW_l += h_{l-1}^T . da ;  dh_{l-1} = da . W_l^T
    const int win = p.w[l - 1];
    {
      constexpr int kRowIters = kMaxRows / 4, kKIters = kMaxW / 4;
      float hr[kRowIters], wr[kKIters];
#pragma unroll
      for (int i = 0; i < kRowIters; ++i) { const int r = tr + 4 * i; hr[i] = (tc < win && r < rows) ? p.h[l - 1][(size_t)(row0 + r) * win + tc] : 0.f; }
#pragma unroll
      for (int i = 0; i < kKIters; ++i) { const int k = tr + 4 * i; wr[i] = (k < win && tc < w) ? p.W[l][(size_t)k * w + tc] : 0.f; }
      if (tc < win) {
#pragma unroll
        for (int i = 0; i < kRowIters; ++i) { const int r = tr + 4 * i; if (r < rows) xh[r][tc] = hr[i]; }
      }
#pragma unroll
      for (int i = 0; i < kKIters; ++i) Ws[tr + 4 * i][tc] = wr[i];
    }
    __syncthreads();
    MID_STAMP(24 + (p.L - 1 - l) * 3);
    // dW[k][c] = sum_r h[r][k] * da[r][c]: thread = column c and a group of 4 consecutive k (128-bit broadcast of h)
    if (tc < w)
      for (int k0 = tr * 4; k0 < win; k0 += 16) {
        float s[4] = {0.f, 0.f, 0.f, 0.f};
        // four rows per trip, loads ahead of the FMAs (one row per trip exposed two shared-memory latencies per 4 FMAs: 37
        // cycles per row, gg_profile); rows beyond `rows` are zero in both strips and the strip height is a multiple of 4
        for (int r = 0; r < rows; r += 4) {
          float gv[4]; float4 hv[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) { gv[j] = g[r + j][tc]; hv[j] = *reinterpret_cast<const float4*>(&xh[r + j][k0]); }
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            s[0] = fmaf(hv[j].x, gv[j], s[0]); s[1] = fmaf(hv[j].y, gv[j], s[1]);
            s[2] = fmaf(hv[j].z, gv[j], s[2]); s[3] = fmaf(hv[j].w, gv[j], s[3]);
          }
        }
        if (k0 == tr * 4) MID_STAMP(25 + (p.L - 1 - l) * 3);
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (k0 + j < win) gpart_l[(size_t)(kMaxW + (k0 + j) * w + tc) * kMaxCtas] = s[j];
        if (k0 == tr * 4) MID_STAMP(26 + (p.L - 1 - l) * 3);
      }
    __syncthreads();
    MID_STAMP(7 + (p.L - 1 - l) * 8);
    // dh_{l-1}[r][k] = sum_c da[r][c] * W[k][c]: thread = k (= tc), 4 rows at a time, c in groups of 4
    constexpr int kRowGroups = kMaxRows / 16;
    float dhv[kRowGroups][4];                                          // [row group][row in group]
    if (tc < win) {
#pragma unroll
      for (int q = 0; q < kRowGroups; ++q) {
        const int r0 = tr * 4 + q * 16;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        if (r0 < rows)
#pragma unroll 4
          for (int c = 0; c < w; c += 4) {                             // padded columns of g / Ws are zero
            const float w0 = Ws[tc][c], w1 = Ws[tc][c + 1], w2 = Ws[tc][c + 2], w3 = Ws[tc][c + 3];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float4 x = *reinterpret_cast<const float4*>(&g[r0 + j][c]);
              acc[j] = fmaf(x.x, w0, fmaf(x.y, w1, fmaf(x.z, w2, fmaf(x.w, w3, acc[j]))));
            }
          }
#pragma unroll
        for (int j = 0; j < 4; ++j) dhv[q][j] = acc[j];
      }
    }
    __syncthreads();                                                   // all reads of xh (as h_{l-1}) and g are done
    if (tc < win) {
#pragma unroll
      for (int q = 0; q < kRowGroups; ++q)
#pragma unroll
        for (int j = 0; j < 4; ++j) { const int r = tr * 4 + q * 16 + j; if (r < rows) xh[r][tc] = dhv[q][j]; }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < (int)kStripFloats; i += kThreads) (&g[0][0])[i] = 0.f;
    __syncthreads();
    if (tc < win)
      for (int r = tr; r < rows; r += 4) g[r][tc] = xh[r][tc];
    __syncthreads();
    MID_STAMP(8 + (p.L - 1 - l) * 8);
  }
  // bias / kernel gradients: every CTA has written its partial of every slot; one thread per slot adds the partials in
  // CTA order, so the sum does not depend on which CTA finished first
  grid_barrier(p.bar, gridDim.x, gen);
  for (int e = blockIdx.x * kThreads + threadIdx.x; e < p.L * kGradSlots; e += gridDim.x * kThreads) {
    const int l = e / kGradSlots, o = e % kGradSlots, w = p.w[l];
    float* dst;
    if (o < kMaxW) { if (o >= w) continue; dst = p.gb[l] + o; }
    else { if (l == 0 || o - kMaxW >= p.w[l - 1] * w) continue; dst = p.gW[l] + (o - kMaxW); }
    const float* src = p.gpart + (size_t)e * kMaxCtas;
    float sum = 0.f;
    for (int c = 0; c < (int)gridDim.x; ++c) sum += __ldcg(src + c);
    *dst += sum;
  }
  MID_STAMP(31);
}

}  // namespace mid

bool mid_supported(const int* widths, int L) {
  if (L < 1) return false;
  for (int i = 0; i < L; ++i) if (widths[i] > mid::kMaxW) return false;
  return true;
}

static int mid_fill(mid::Params& p, int B) {
  static const int rows_target = [] { const char* e = getenv("DCA_MID_ROWS"); int v = e ? atoi(e) : 32; return (v >= 16 && v <= mid::kMaxRows) ? v : 32; }();
  int ctas = cdiv(B, rows_target);
  if (ctas > mid::kMaxCtas) ctas = mid::kMaxCtas;
  if (p.max_ctas > 0 && ctas > p.max_ctas) { ctas = p.max_ctas; if ((long long)ctas * mid::kMaxRows < B) ctas = cdiv(B, mid::kMaxRows); }
  if ((long long)ctas * mid::kMaxRows < B) { set_error("mid_stack: batch %d exceeds %d rows", B, mid::kMaxRows * mid::kMaxCtas); return DCA_ERR_UNSUPPORTED; }
  // spread rows evenly, at least 16 rows per CTA so tiny batches do not pay for 64 barriers participants
  int rpc = cdiv(B, ctas);
  if (rpc < 16) rpc = 16;
  rpc = (rpc + 3) & ~3;
  if (rpc > mid::kMaxRows) rpc = mid::kMaxRows;
  while ((long long)rpc * mid::kMaxCtas < B) rpc += 4;
  p.rows_per_cta = rpc; p.n_ctas = cdiv(B, rpc);
  return DCA_OK;
}

size_t mid_partial_doubles() { return (size_t)2 * mid::kMaxCtas * 2 * mid::kMaxW; }
size_t mid_grad_partial_floats(int L) { return (size_t)L * mid::kGradSlots * mid::kMaxCtas; }

static int mid_attr() {
  static bool done = false;
  if (!done) {
    DCA_CUDA_OK(cudaFuncSetAttribute(mid::mid_forward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mid::kSmemBytes));
    DCA_CUDA_OK(cudaFuncSetAttribute(mid::mid_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mid::kSmemBytes));
    done = true;
  }
  return DCA_OK;
}

// The grid barrier needs every CTA resident at once: the kernels are launched COOPERATIVELY (the driver then either
// guarantees co-residency or fails the launch; capturable into CUDA graphs), and mid_device_ok() checks once per
// device that max-active-blocks x SM count covers the largest grid, so that the engine can fall back to the per-layer
// kernels (MIG slice, tiny part) instead of failing at launch time.
bool mid_device_ok() {
  static thread_local int ok_dev = -1, ok = 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { (void)cudaGetLastError(); return false; }
  if (ok_dev == dev) return ok != 0;
  ok_dev = dev; ok = 0;
  if (mid_attr() != DCA_OK) return false;
  int coop = 0, sms = 0, nf = 0, nb = 0;
  if (cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev) != cudaSuccess || !coop) return false;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return false;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nf, mid::mid_forward_kernel, mid::kThreads, mid::kSmemBytes) != cudaSuccess) return false;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, mid::mid_backward_kernel, mid::kThreads, mid::kSmemBytes) != cudaSuccess) return false;
  ok = ((long long)nf * sms >= mid::kMaxCtas && (long long)nb * sms >= mid::kMaxCtas) ? 1 : 0;
  return ok != 0;
}

template <class K>
static int mid_launch(K kernel, mid::Params& p, cudaStream_t s) {
  cudaLaunchConfig_t lc{};
  lc.gridDim = dim3((unsigned)p.n_ctas); lc.blockDim = dim3(mid::kThreads); lc.dynamicSmemBytes = mid::kSmemBytes; lc.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative; at[0].val.cooperative = 1;
  lc.attrs = at; lc.numAttrs = 1;
  DCA_CUDA_OK(cudaLaunchKernelEx(&lc, kernel, p));
  count_launch(1);
  return DCA_OK;
}

namespace tc { extern int g_gg_profile; }

// gg_profile: phase timeline of CTA 0 (clock64 stamps), printed after the launch (synchronises; DCA_GRAPH=0)
static int mid_profiled(const char* name, int (*launch)(mid::Params&, cudaStream_t), mid::Params& p, cudaStream_t s) {
  static long long* dbg_buf = nullptr;
  if (!dbg_buf) DCA_CUDA_OK(cudaMalloc(&dbg_buf, sizeof(long long) * 32));
  DCA_CUDA_OK(cudaMemsetAsync(dbg_buf, 0, sizeof(long long) * 32, s));
  p.dbg = dbg_buf;
  DCA_TRY(launch(p, s));
  long long h[32];
  DCA_CUDA_OK(cudaStreamSynchronize(s));
  DCA_CUDA_OK(cudaMemcpy(h, dbg_buf, sizeof(h), cudaMemcpyDeviceToHost));
  fprintf(stderr, "[gg_profile %s ctas %d rows %d] cycles since start:", name, p.n_ctas, p.rows_per_cta);
  for (int i = 1; i < 32; ++i) if (h[i]) fprintf(stderr, " s%d=%lld", i, h[i] - h[0]);
  fprintf(stderr, "\n");
  return DCA_OK;
}
static int mid_forward_launch(mid::Params& p, cudaStream_t s) { return mid_launch(mid::mid_forward_kernel, p, s); }
static int mid_backward_launch(mid::Params& p, cudaStream_t s) { return mid_launch(mid::mid_backward_kernel, p, s); }

int mid_forward(mid::Params& p, cudaStream_t s) {
  DCA_TRY(mid_fill(p, p.B));
  DCA_TRY(mid_attr());
  p.dbg = nullptr;
  if (tc::g_gg_profile) return mid_profiled("mid_forward", mid_forward_launch, p, s);
  return mid_forward_launch(p, s);
}

int mid_backward(mid::Params& p, cudaStream_t s) {
  DCA_TRY(mid_fill(p, p.B));
  DCA_TRY(mid_attr());
  p.dbg = nullptr;
  if (tc::g_gg_profile) return mid_profiled("mid_backward", mid_backward_launch, p, s);
  return mid_backward_launch(p, s);
}

}  // namespace dca
