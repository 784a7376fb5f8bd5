// Small element-wise / column-reduction kernels of the hidden stack and the optimizer:
//   BatchNormalization(center=True, scale=False) train / inference / backward  (dca/network.py:127-128)
//   relu forward / backward                                                    (dca/network.py:135)
//   ConstantDispersionLayer theta = clip(exp(theta_raw), 1e-3, 1e4)             (dca/layers.py:17-21)
//   l1_l2 kernel regulariser gradient + penalty                                (dca/network.py:125)
//   clipvalue + RMSprop                                                        (dca/train.py:54-57)
//   kernel initialisers: Keras' VarianceScaling family, normal, uniform, constant,
//   identity and orthogonal (fp64 Householder QR)                              (dca/network.py:124-126)
#include "dca_internal.cuh"

namespace dca {
namespace {

constexpr int kColChunks = 64;   // row chunks for column statistics

__global__ void fill_rows_kernel(float* C, int64_t ldc, int M, int N, const float* __restrict__ bias) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)M * N) return;
  const int r = (int)(i / N), c = (int)(i % N);
  C[(int64_t)r * ldc + c] = bias ? bias[c] : 0.f;
}

// partial column sums over a chunk of rows: block (32 cols, 8 row lanes)
__global__ void col_sums_partial_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t ld,
                                        int M, int N, int rows_per_chunk, double* __restrict__ psum,
                                        double* __restrict__ pprod) {
  __shared__ double s1[8][33], s2[8][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  const int r0 = blockIdx.y * rows_per_chunk;
  const int r1 = min(M, r0 + rows_per_chunk);
  double t1 = 0.0, t2 = 0.0;
  if (col < N) {
    for (int r = r0 + threadIdx.y; r < r1; r += 8) {
      const float x = a[(int64_t)r * ld + col];
      const float y = b ? b[(int64_t)r * ld + col] : x;
      t1 += (double)x;
      t2 += (double)x * (double)y;
    }
  }
  s1[threadIdx.y][threadIdx.x] = t1;
  s2[threadIdx.y][threadIdx.x] = t2;
  __syncthreads();
  if (threadIdx.y == 0 && col < N) {
#pragma unroll
    for (int i = 1; i < 8; ++i) { t1 += s1[i][threadIdx.x]; t2 += s2[i][threadIdx.x]; }
    psum[(int64_t)blockIdx.y * N + col] = t1;
    pprod[(int64_t)blockIdx.y * N + col] = t2;
  }
}

__global__ void col_sums_fold_kernel(const double* __restrict__ psum, const double* __restrict__ pprod, int chunks,
                                     int N, double* __restrict__ out_sum, double* __restrict__ out_prod) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= N) return;
  double a = 0.0, b = 0.0;
  for (int k = 0; k < chunks; ++k) { a += psum[(int64_t)k * N + c]; b += pprod[(int64_t)k * N + c]; }
  out_sum[c] = a;
  if (out_prod) out_prod[c] = b;
}

__global__ void bn_train_finalize_kernel(const double* __restrict__ sum, const double* __restrict__ sq, int M, int N,
                                         float eps, float momentum, float* __restrict__ mean,
                                         float* __restrict__ inv_std, float* __restrict__ mmean,
                                         float* __restrict__ mvar) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= N) return;
  const double mu = sum[c] / (double)M;
  double var = sq[c] / (double)M - mu * mu;          // biased batch variance (Keras non-fused BN)
  if (var < 0.0) var = 0.0;
  mean[c] = (float)mu;
  inv_std[c] = (float)(1.0 / sqrt(var + (double)eps));
  mmean[c] = momentum * mmean[c] + (1.0f - momentum) * (float)mu;
  mvar[c] = momentum * mvar[c] + (1.0f - momentum) * (float)var;
}

__global__ void bn_relu_fwd_kernel(const float* __restrict__ a, int64_t ld, int M, int N,
                                   const float* __restrict__ mean, const float* __restrict__ inv_std,
                                   const float* __restrict__ beta, float* __restrict__ xhat,
                                   float* __restrict__ h, __nv_bfloat16* __restrict__ hb) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)M * N) return;
  const int r = (int)(i / N), c = (int)(i % N);
  const float xh = (a[(int64_t)r * ld + c] - mean[c]) * inv_std[c];
  if (xhat) xhat[i] = xh;
  const float v = fmaxf(xh + beta[c], 0.f);
  h[i] = v;
  if (hb) hb[i] = __float2bfloat16_rn(v);
}

__global__ void bn_infer_prepare_kernel(const float* __restrict__ mm, const float* __restrict__ mv, int N, float eps,
                                        float* __restrict__ mean, float* __restrict__ inv_std) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= N) return;
  mean[c] = mm[c];
  inv_std[c] = rsqrtf(mv[c] + eps);
}

__global__ void relu_fwd_kernel(const float* __restrict__ a, int64_t ld, int M, int N, float* __restrict__ h,
                                __nv_bfloat16* __restrict__ hb) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)M * N) return;
  const int r = (int)(i / N), c = (int)(i % N);
  const float v = fmaxf(a[(int64_t)r * ld + c], 0.f);
  h[i] = v;
  if (hb) hb[i] = __float2bfloat16_rn(v);
}



// out[r][0..n) = bf16(X[rows[r]][0..n)), 8 elements per thread (n % 8 == 0, 16-byte aligned rows)
template <typename T>
__global__ void gather_rows_bf16_kernel(const T* __restrict__ X, int64_t ldx, const int32_t* __restrict__ rows, int M,
                                        int n, __nv_bfloat16* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int per_row = n / 8;
  if (i >= (int64_t)M * per_row) return;
  const int r = (int)(i / per_row), c = (int)(i % per_row) * 8;
  const int64_t sr = rows ? (int64_t)rows[r] : (int64_t)r;
  uint4 o;
  if (sizeof(T) == 2) {
    o = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(X) + sr * ldx + c);
  } else {
    const float* s = reinterpret_cast<const float*>(X) + sr * ldx + c;
    const float4 a = *reinterpret_cast<const float4*>(s), bq = *reinterpret_cast<const float4*>(s + 4);
    __nv_bfloat162 p0 = __floats2bfloat162_rn(a.x, a.y), p1 = __floats2bfloat162_rn(a.z, a.w);
    __nv_bfloat162 p2 = __floats2bfloat162_rn(bq.x, bq.y), p3 = __floats2bfloat162_rn(bq.z, bq.w);
    o.x = *reinterpret_cast<uint32_t*>(&p0); o.y = *reinterpret_cast<uint32_t*>(&p1);
    o.z = *reinterpret_cast<uint32_t*>(&p2); o.w = *reinterpret_cast<uint32_t*>(&p3);
  }
  *reinterpret_cast<uint4*>(out + (int64_t)r * n + c) = o;
}

__global__ void relu_bwd_kernel(float* __restrict__ dh, const float* __restrict__ h, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (!(h[i] > 0.f)) dh[i] = 0.f;
}

__global__ void bn_bwd_apply_kernel(float* __restrict__ g, const float* __restrict__ xhat, int M, int N,
                                    const float* __restrict__ inv_std, const double* __restrict__ sum_g,
                                    const double* __restrict__ sum_gx, float* __restrict__ dbeta, int stat_rows) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)M * N) return;
  const int c = (int)(i % N);
  const float mg = (float)(sum_g[c] / (double)stat_rows), mgx = (float)(sum_gx[c] / (double)stat_rows);
  g[i] = inv_std[c] * (g[i] - mg - xhat[i] * mgx);
  if (i < N && dbeta) dbeta[c] = (float)sum_g[c];
}

__global__ void double_to_float_kernel(const double* __restrict__ in, int n, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (float)in[i];
}

__global__ void theta_prepare_kernel(const float* __restrict__ raw, int G, float* __restrict__ theta,
                                     float* __restrict__ chain) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const float e = expf(raw[g]);
  const float t = fminf(fmaxf(e, 1e-3f), 1e4f);        // dca/layers.py:21
  theta[g] = t;
  chain[g] = (e >= 1e-3f && e <= 1e4f) ? t : 0.f;       // d theta / d raw, clip_by_value gradient
}

__global__ void theta_grad_finish_kernel(const float* __restrict__ dth, const float* __restrict__ chain, int G,
                                         float scale, float* __restrict__ out) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < G) out[g] = dth[g] * chain[g] * scale;
}

__global__ void add_reg_grad_kernel(const float* __restrict__ w, float* __restrict__ g, int64_t n, float l1, float l2) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = w[i];
  const float sg = (v > 0.f) ? 1.f : ((v < 0.f) ? -1.f : 0.f);
  g[i] += l1 * sg + 2.f * l2 * v;
}

__global__ void reg_penalty_kernel(const float* __restrict__ w, int64_t n, float l1, float l2, double* acc) {
  __shared__ double sm[8];
  double t = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double v = w[i];
    t += l1 * fabs(v) + l2 * v * v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) a += sm[i];
    atomicAdd(acc, a);
  }
}

__device__ __forceinline__ float rmsprop_one(float p, float g, float& r, float lr, float clip, float rho, float eps, float gs) {
  float gi = g * gs;
  if (clip > 0.f) gi = fminf(fmaxf(gi, -clip), clip);       // clipvalue
  r = rho * r + (1.0f - rho) * gi * gi;
  return p - lr * gi / (sqrtf(r) + eps);                     // epsilon outside the sqrt (Keras RMSprop)
}

// four parameters per thread (128-bit loads / stores; the three regions are 256-byte aligned), scalar tail
__global__ void rmsprop_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ r, int64_t n,
                               float lr, float clip, float rho, float eps, float gs, __nv_bfloat16* __restrict__ shadow,
                               float* loss_out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t == 0 && loss_out) {             // the step's (all-reduced) mean loss, mirrored into mapped HOST memory
    *loss_out = g[n] * gs;              // grads[P] is the loss slot
    __threadfence_system();
  }
  const int64_t i = t * 4;
  if (i >= n) return;
  if (i + 3 < n) {
    const float4 pv = *reinterpret_cast<const float4*>(p + i), gv = *reinterpret_cast<const float4*>(g + i);
    float4 rv = *reinterpret_cast<const float4*>(r + i);
    float4 o;
    o.x = rmsprop_one(pv.x, gv.x, rv.x, lr, clip, rho, eps, gs); o.y = rmsprop_one(pv.y, gv.y, rv.y, lr, clip, rho, eps, gs);
    o.z = rmsprop_one(pv.z, gv.z, rv.z, lr, clip, rho, eps, gs); o.w = rmsprop_one(pv.w, gv.w, rv.w, lr, clip, rho, eps, gs);
    *reinterpret_cast<float4*>(r + i) = rv;
    *reinterpret_cast<float4*>(p + i) = o;
    if (shadow) {                        // bf16 operand copy for the tensor-core kernels (same layout)
      __nv_bfloat162 a = __floats2bfloat162_rn(o.x, o.y), b = __floats2bfloat162_rn(o.z, o.w);
      uint2 w; w.x = *reinterpret_cast<uint32_t*>(&a); w.y = *reinterpret_cast<uint32_t*>(&b);
      *reinterpret_cast<uint2*>(shadow + i) = w;
    }
  } else {
    for (int64_t k = i; k < n; ++k) {
      float rk = r[k];
      const float pn = rmsprop_one(p[k], g[k], rk, lr, clip, rho, eps, gs);
      r[k] = rk; p[k] = pn;
      if (shadow) shadow[k] = __float2bfloat16_rn(pn);
    }
  }
}

// keras/optimizers.py (Keras 2.x) get_updates of SGD / Adagrad / Adadelta / Adam / Adamax / Nadam, clipvalue first
__global__ void optimizer_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ s1,
                                 float* __restrict__ s2, int64_t n, OptScalars o, __nv_bfloat16* __restrict__ shadow,
                                 float* loss_out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (i == 0 && loss_out) { *loss_out = g[n] * o.gs; __threadfence_system(); }
  float gi = g[i] * o.gs;
  if (o.clip > 0.f) gi = fminf(fmaxf(gi, -o.clip), o.clip);
  const float eps = 1e-7f;
  float pn = p[i];
  switch (o.kind) {
    case DCA_OPT_SGD: pn -= o.lr * gi; break;
    case DCA_OPT_ADAGRAD: { const float a = s1[i] + gi * gi; s1[i] = a; pn -= o.lr * gi / (sqrtf(a) + eps); break; }
    case DCA_OPT_ADADELTA: {
      const float rho = 0.95f;
      const float a = rho * s1[i] + (1.f - rho) * gi * gi; s1[i] = a;
      const float d = s2[i];
      const float u = gi * sqrtf(d + eps) / sqrtf(a + eps);
      pn -= o.lr * u;
      s2[i] = rho * d + (1.f - rho) * u * u;
      break;
    }
    case DCA_OPT_ADAM: {          // c0 = lr * sqrt(1 - b2^t) / (1 - b1^t)
      const float m = 0.9f * s1[i] + 0.1f * gi, v = 0.999f * s2[i] + 0.001f * gi * gi;
      s1[i] = m; s2[i] = v;
      pn -= o.c0 * m / (sqrtf(v) + eps);
      break;
    }
    case DCA_OPT_ADAMAX: {        // c0 = lr / (1 - b1^t)
      const float m = 0.9f * s1[i] + 0.1f * gi, u = fmaxf(0.999f * s2[i], fabsf(gi));
      s1[i] = m; s2[i] = u;
      pn -= o.c0 * m / (u + eps);
      break;
    }
    case DCA_OPT_NADAM: {         // c0 = 1/(1 - m_schedule_new), c1 = 1/(1 - m_schedule_next), c2 = 1/(1 - b2^t), c3 = mu_t, c4 = mu_{t+1}
      const float m = 0.9f * s1[i] + 0.1f * gi, v = 0.999f * s2[i] + 0.001f * gi * gi;
      s1[i] = m; s2[i] = v;
      const float mbar = (1.f - o.c3) * (gi * o.c0) + o.c4 * (m * o.c1);
      pn -= o.lr * mbar / (sqrtf(v * o.c2) + eps);
      break;
    }
    default: break;
  }
  p[i] = pn;
  if (shadow) shadow[i] = __float2bfloat16_rn(pn);
}

// ---- weight initialisers (include/dca_b200.h, "initializers").  Every element is a function of (seed, sid, i): sid
// numbers the kernel tensor, i is the element's flat index.  The same source runs on the host (dca_init_fill_host).
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__host__ __device__ __forceinline__ uint64_t init_hash(uint64_t seed, uint64_t sid, int64_t i) {
  return splitmix64(splitmix64(seed ^ (sid * 0xD1B54A32D192ED03ull)) + (uint64_t)i);
}

enum InitFill : int { FILL_UNIFORM = 0, FILL_NORMAL = 1, FILL_TRUNC_NORMAL = 2, FILL_CONST = 3, FILL_IDENTITY = 4 };
// One kernel tensor's element rule, derived on the host from a dca_initializer and the tensor's fans
struct InitDraw {
  int kind;             // InitFill
  float center, half;   // uniform: center + (2u - 1) * half, one fused multiply-add in float
  double sigma;         // normal kinds: float(z * sigma), z a standard normal in fp64
  float value;          // constant; identity: the diagonal
  int cols;             // identity
};
// Re-draws of a truncated normal before the element is set to 0: all 16 fail with probability 0.0455^16 < 4e-22
constexpr int kTruncAttempts = 16;

// Box-Muller in fp64 on two 53-bit uniforms of draw `attempt` of the element with hash h
__host__ __device__ __forceinline__ double init_std_normal(uint64_t h, uint32_t attempt) {
  const uint64_t h1 = splitmix64(h ^ (0x632BE59BD9B4E019ull * (2ull * attempt + 1)));
  const uint64_t h2 = splitmix64(h ^ (0x632BE59BD9B4E019ull * (2ull * attempt + 2)));
  const double u1 = (double)((h1 >> 11) + 1) * 0x1p-53;     // (0, 1]
  const double u2 = (double)(h2 >> 11) * 0x1p-53;           // [0, 1)
  return sqrt(-2.0 * log(u1)) * cos(6.283185307179586476925 * u2);
}

__host__ __device__ __forceinline__ float init_draw(const InitDraw& d, uint64_t seed, uint64_t sid, int64_t i) {
  if (d.kind == FILL_CONST) return d.value;
  if (d.kind == FILL_IDENTITY) return i / d.cols == i % d.cols ? d.value : 0.f;
  const uint64_t h = init_hash(seed, sid, i);
  if (d.kind == FILL_UNIFORM) {
    const float u = (float)(h >> 40) * (1.0f / 16777216.0f);   // [0,1)
    return fmaf(2.0f * u - 1.0f, d.half, d.center);
  }
  double z = 0.0;
  if (d.kind == FILL_NORMAL) {
    z = init_std_normal(h, 0);
  } else {
    for (int a = 0; a < kTruncAttempts; ++a) {
      const double t = init_std_normal(h, (uint32_t)a);
      if (fabs(t) < 2.0) { z = t; break; }
    }
  }
  return (float)(z * d.sigma);
}

__global__ void init_fill_kernel(float* __restrict__ w, int64_t n, InitDraw d, uint64_t seed, uint64_t sid) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) w[i] = init_draw(d, seed, sid, i);
}

// Orthogonal: A (m x n, m = max(rows, cols), n = min) of standard normals rounded to float, Householder QR of A in
// fp64, Q <- Q sign(diag R), W = gain Q (rows >= cols) or gain Q^T.  One CTA per tensor; A, tau and the signs live in a
// fp64 workspace.  Every reduction runs in a fixed order, so the result is the same bits on every run.
constexpr int kMaxOrthoJobs = 2 * DCA_MAX_HIDDEN + 4;
struct OrthoJob { float* w; double* a; int rows, cols; uint64_t sid; };
struct OrthoJobs { OrthoJob job[kMaxOrthoJobs]; uint64_t seed; float gain; };
constexpr int kQrWarps = 16;

// sum over the CTA of v, in a fixed order; every thread gets the result
__device__ double qr_block_sum(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double t = 0.0;
  for (int k = 0; k < kQrWarps; ++k) t += red[k];
  return t;
}

// A(i:m, i+1:n) <- (I - tau v v^T) A(i:m, i+1:n), v = A(i:m, i) with v_i = 1.  Lanes own columns, warps stride rows:
// each pass reads a row's 64 trailing columns as one coalesced piece.
__device__ void qr_reflect(double* A, int m, int n, int i, double tau, double* red, double* wsum) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int c0 = i + 1; c0 < n; c0 += 64) {
    const int ca = c0 + lane, cb = c0 + 32 + lane;
    double sa = 0.0, sb = 0.0;
    for (int r = i + warp; r < m; r += kQrWarps) {
      const double* row = A + (int64_t)r * n;
      const double v = r == i ? 1.0 : row[i];
      if (ca < n) sa += v * row[ca];
      if (cb < n) sb += v * row[cb];
    }
    red[warp * 64 + lane] = sa;
    red[warp * 64 + 32 + lane] = sb;
    __syncthreads();
    if (threadIdx.x < 64) {
      double t = 0.0;
      for (int k = 0; k < kQrWarps; ++k) t += red[k * 64 + threadIdx.x];
      wsum[threadIdx.x] = tau * t;
    }
    __syncthreads();
    const double wa = wsum[lane], wb = wsum[32 + lane];
    for (int r = i + warp; r < m; r += kQrWarps) {
      double* row = A + (int64_t)r * n;
      const double v = r == i ? 1.0 : row[i];
      if (ca < n) row[ca] -= v * wa;
      if (cb < n) row[cb] -= v * wb;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kQrWarps * 32) orthogonal_kernel(OrthoJobs jobs) {
  __shared__ double red[kQrWarps * 64], wsum[64];
  const OrthoJob jb = jobs.job[blockIdx.x];
  const bool tall = jb.rows >= jb.cols;
  const int m = tall ? jb.rows : jb.cols, n = tall ? jb.cols : jb.rows;
  double* A = jb.a;
  double* tau = A + (int64_t)m * n;
  double* sgn = tau + n;
  const InitDraw nd{FILL_NORMAL, 0.f, 0.f, 1.0, 0.f, 0};
  for (int64_t e = threadIdx.x; e < (int64_t)m * n; e += blockDim.x) A[e] = (double)init_draw(nd, jobs.seed, jb.sid, e);
  __syncthreads();
  // A = QR: reflectors below the diagonal (LAPACK dgeqr2 / dlarfg)
  for (int i = 0; i < n; ++i) {
    double t = 0.0;
    for (int r = i + 1 + threadIdx.x; r < m; r += blockDim.x) { const double x = A[(int64_t)r * n + i]; t += x * x; }
    const double xnorm2 = qr_block_sum(t, red);
    const double alpha = A[(int64_t)i * n + i];
    double beta = alpha, ti = 0.0;
    if (xnorm2 > 0.0) {
      beta = -copysign(sqrt(alpha * alpha + xnorm2), alpha);
      ti = (beta - alpha) / beta;
      const double sc = 1.0 / (alpha - beta);
      for (int r = i + 1 + threadIdx.x; r < m; r += blockDim.x) A[(int64_t)r * n + i] *= sc;
    }
    __syncthreads();
    if (threadIdx.x == 0) { A[(int64_t)i * n + i] = beta; tau[i] = ti; sgn[i] = beta < 0.0 ? -1.0 : 1.0; }
    // qr_reflect has no barrier when no column is left (i = n - 1): without this one, the first step of the Q
    // formation below could read tau[n - 1] and write A(n-1, n-1) before thread 0's stores
    __syncthreads();
    qr_reflect(A, m, n, i, ti, red, wsum);
  }
  // Q (m x n) in place of the reflectors (LAPACK dorg2r)
  for (int i = n - 1; i >= 0; --i) {
    const double ti = tau[i];
    if (i < n - 1) qr_reflect(A, m, n, i, ti, red, wsum);
    for (int r = threadIdx.x; r < m; r += blockDim.x) {
      double* p = A + (int64_t)r * n + i;
      *p = r > i ? -ti * *p : (r == i ? 1.0 - ti : 0.0);
    }
    __syncthreads();
  }
  const double g = (double)jobs.gain;
  for (int64_t e = threadIdx.x; e < (int64_t)jb.rows * jb.cols; e += blockDim.x) {
    const int r = (int)(e / jb.cols), c = (int)(e % jb.cols);
    const int qrow = tall ? r : c, qcol = tall ? c : r;
    jb.w[e] = (float)(g * sgn[qcol] * A[(int64_t)qrow * n + qcol]);
  }
}

__global__ void fill_kernel(float* __restrict__ p, int64_t n, float v) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

__global__ void cast_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __float2bfloat16_rn(in[i]);
}

// packed counts (BITS = 4 / 8 / 16 per entry, row-major, gene c of a 4-bit row in byte c/2, low nibble = even c)
// -> Y (fp32 target) and X = ((log1p)(y/sf) - mean_g) * inv_std_g (network input), 8 genes per thread.
// With an overflow list the value 2^BITS-1 is an escape: the true count is looked up in the row's (short,
// gene-sorted) segment of the CSR list.  log1p uses MUFU lg2: with its bound (2^-22 absolute on [0.5, 2], 2 ulp
// elsewhere) and the roundings of y/sf, 1 + v and the ln2 product, |l - log1p(y/sf)| < 4e-7 + 4e-7 l, and
// |X - X_exact| <= inv_std (4e-7 + 4e-7 l) + 2^-23 |X| (derived and checked in tests/test_gpu_stream.py), far below
// the bf16 rounding of the encoder input.
__device__ __forceinline__ float normalise_count(float y, float inv_s, int use_log1p, const float* mean,
                                                 const float* inv_std, int c) {
  float v = y * inv_s;                                    // sc.pp.normalize_per_cell   dca/io.py:99-100
  if (use_log1p) v = 0.6931471805599453f * __log2f(1.0f + v);   // sc.pp.log1p (MUFU lg2)   dca/io.py:105-106
  return mean ? (v - mean[c]) * inv_std[c] : v;           // sc.pp.scale                dca/io.py:108-109
}

// r: the source row; absolute: the offsets of indptr index `entries` directly (a row-indexed expansion of a whole packed
// matrix), else they are relative to indptr[0] (a contiguous batch whose entries start at `entries`)
__device__ __forceinline__ float overflow_find(const int64_t* __restrict__ indptr, const int2* __restrict__ entries, int64_t r,
                                               int c, float fallback, bool absolute = false) {
  const int64_t base = absolute ? 0 : indptr[0];
  int64_t lo = indptr[r] - base, hi = indptr[r + 1] - base;
  while (lo < hi) {                                       // entries of a row are sorted by gene
    const int64_t mid = (lo + hi) >> 1;
    const int g = entries[mid].x;
    if (g == c) return __int_as_float(entries[mid].y);
    if (g < c) lo = mid + 1; else hi = mid;
  }
  return fallback;
}
// out of line for the float transform (keeps its registers); the exact kernels inline it: a call there costs a spill
__device__ __noinline__ float overflow_lookup(const int64_t* __restrict__ indptr, const int2* __restrict__ entries, int64_t r,
                                              int c, float fallback, bool absolute) {
  return overflow_find(indptr, entries, r, c, fallback, absolute);
}

// The exact variant (EXACT = true, preprocess.cu's arithmetic): sf64 = n_counts[r] / median, X =
// float(((double)l - mean_g) / std_g) with l = pre_log_value(y, sf64, flags).  Zero counts take the per-gene constant
// x_zero, so the fp64 division and log1p run on non-zero entries only.
__device__ __forceinline__ double exact_row_sf(const ExactXform& ex, int64_t r) {
  return (ex.flags & DCA_PRE_SIZE_FACTORS) ? ex.n_counts[r] / ex.median : 1.0;
}
__device__ __forceinline__ float exact_count(float y, double sf64, const ExactXform& ex, int c) {
  if (y == 0.f) return ex.x_zero ? ex.x_zero[c] : (float)((0.0 - ex.mean[c]) / ex.std[c]);
  return (float)(((double)pre_log_value(y, sf64, ex.flags) - ex.mean[c]) / ex.std[c]);
}

__global__ void exact_zero_kernel(const double* __restrict__ mean, const double* __restrict__ std, int n, float* __restrict__ out) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n) out[g] = (float)((0.0 - mean[g]) / std[g]);
}

template <int BITS, typename XT, bool EXACT>
__global__ void expand_counts_kernel(const unsigned char* __restrict__ cnt, const float* __restrict__ sf_in, int M, int n,
                                     const float* __restrict__ mean, const float* __restrict__ inv_std, int use_sf,
                                     int use_log1p, float* __restrict__ Yout, XT* __restrict__ Xout, float* __restrict__ sf_out,
                                     const int64_t* __restrict__ ovf_indptr, const int2* __restrict__ ovf_entries,
                                     ExactXform ex, const int32_t* __restrict__ rows) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int per_row = n / 8;
  if (i >= (int64_t)M * per_row) return;
  const int r = (int)(i / per_row), c = (int)(i % per_row) * 8;
  const int64_t sr = rows ? (int64_t)rows[r] : (int64_t)r;        // source row (ROWS: any row of the whole matrix)
  const double sf64 = EXACT ? exact_row_sf(ex, sr) : 1.0;
  const float s = EXACT ? (float)sf64 : (sf_in ? sf_in[sr] : 1.0f);
  if (c == 0 && sf_out) sf_out[r] = s;
  const float inv_s = use_sf ? 1.0f / s : 1.0f;
  uint32_t q[8];
  const unsigned char* src = cnt + (sr * n + c) * BITS / 8;
  if (BITS == 16) {
    const uint4 raw = *reinterpret_cast<const uint4*>(src);
    const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) { q[2 * k] = w[k] & 0xffffu; q[2 * k + 1] = w[k] >> 16; }
  } else if (BITS == 8) {
    const uint2 raw = *reinterpret_cast<const uint2*>(src);
    const uint32_t w[2] = {raw.x, raw.y};
#pragma unroll
    for (int k = 0; k < 8; ++k) q[k] = (w[k >> 2] >> (8 * (k & 3))) & 0xffu;
  } else {
    const uint32_t w = *reinterpret_cast<const uint32_t*>(src);
#pragma unroll
    for (int k = 0; k < 8; ++k) q[k] = (w >> (4 * k)) & 0xfu;
  }
  constexpr uint32_t kEsc = (1u << BITS) - 1u;
  float y[8], x[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    y[k] = (float)q[k];
    if (ovf_indptr && q[k] == kEsc)
      y[k] = EXACT ? overflow_find(ovf_indptr, ovf_entries, sr, c + k, y[k], rows != nullptr)
                   : overflow_lookup(ovf_indptr, ovf_entries, sr, c + k, y[k], rows != nullptr);
    x[k] = EXACT ? exact_count(y[k], sf64, ex, c + k) : normalise_count(y[k], inv_s, use_log1p, mean, inv_std, c + k);
  }
  float* yo = Yout + (int64_t)r * n + c;
  *reinterpret_cast<float4*>(yo) = make_float4(y[0], y[1], y[2], y[3]);
  *reinterpret_cast<float4*>(yo + 4) = make_float4(y[4], y[5], y[6], y[7]);
  if (sizeof(XT) == 2) {
    __nv_bfloat162 p0 = __floats2bfloat162_rn(x[0], x[1]), p1 = __floats2bfloat162_rn(x[2], x[3]);
    __nv_bfloat162 p2 = __floats2bfloat162_rn(x[4], x[5]), p3 = __floats2bfloat162_rn(x[6], x[7]);
    uint4 o;
    o.x = *reinterpret_cast<uint32_t*>(&p0); o.y = *reinterpret_cast<uint32_t*>(&p1);
    o.z = *reinterpret_cast<uint32_t*>(&p2); o.w = *reinterpret_cast<uint32_t*>(&p3);
    *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(Xout) + (int64_t)r * n + c) = o;
  } else {
    float* xo = reinterpret_cast<float*>(Xout) + (int64_t)r * n + c;
    *reinterpret_cast<float4*>(xo) = make_float4(x[0], x[1], x[2], x[3]);
    *reinterpret_cast<float4*>(xo + 4) = make_float4(x[4], x[5], x[6], x[7]);
  }
}

// Sparse host format (dca_stream_begin_sparse): one bit per (cell, gene) entry -- "non-zero" -- plus the non-zero
// counts of a row as consecutive 4-bit codes in gene order (1..14 literal, 15 = escape into the same CSR overflow list
// as above).  scRNA-seq matrices are > 80 % zeros, so this is ~0.2 bytes per entry over PCIe instead of 0.5 (4-bit
// dense) or 8 (the reference's float32 X + Y).  One block per row: the threads popcount their bitmap words, a block
// scan gives every word the position of its first code in the row's nibble stream, then each thread expands its 32
// genes (Y fp32, X normalised) with 128-bit stores.
constexpr int kSparseMaxBytes = 8192;                    // bitmap bytes per row the kernel supports (65536 genes)
template <typename XT, bool EXACT>
__global__ void __launch_bounds__(256)
expand_sparse_kernel(const uint32_t* __restrict__ bitmap, const int64_t* __restrict__ nib_indptr,
                     const unsigned char* __restrict__ nibbles, const float* __restrict__ sf_in, int M, int n,
                     const float* __restrict__ mean, const float* __restrict__ inv_std, int use_sf, int use_log1p,
                     float* __restrict__ Yout, XT* __restrict__ Xout, float* __restrict__ sf_out,
                     const int64_t* __restrict__ ovf_indptr, const int2* __restrict__ ovf_entries, int nib_cap,
                     ExactXform ex, const int32_t* __restrict__ rows) {
  // One block per row.  Phase 0: the row's bitmap and its nibble bytes go to shared memory with thread-strided loads (all in
  // flight at once; the first version chased them from global memory, one dependent byte load after another: 0.25 ms per
  // 4096 x 20000 batch, 3 x what its 0.5 GB of stores need).  Phase 1: thread t popcounts S consecutive bitmap bytes and
  // records, per byte, the number of non-zero genes before it inside its own span; a block scan over the 256 span totals
  // gives every span its base.  Phase 2: thread = one bitmap byte = 8 consecutive genes, bytes taken in order b = tid,
  // tid + 256, ... so that a warp writes 1 KB of Y and 512 B of X contiguously; the position of a byte's first code in the
  // row's nibble stream is pre[b] + tbase[b / S].
  extern __shared__ __align__(16) unsigned char sp_dyn[];
  __shared__ int tbase[256];
  __shared__ int warp_tot[8];
  const int r = blockIdx.x;
  if (r >= M) return;
  // source row: rows[r] of the whole matrix (offsets absolute), else row r of a contiguous batch (offsets relative to
  // its first row)
  const int64_t sr = rows ? (int64_t)rows[r] : (int64_t)r;
  const int nbytes = n / 8;
  unsigned short* pre = reinterpret_cast<unsigned short*>(sp_dyn);
  unsigned char* s_bm = sp_dyn + ((2 * nbytes + 15) & ~15);
  unsigned char* s_nib = s_bm + ((nbytes + 15) & ~15);
  const unsigned char* bmg = reinterpret_cast<const unsigned char*>(bitmap) + sr * nbytes;
  const int64_t nib0 = nib_indptr[sr] - (rows ? 0 : nib_indptr[0]);
  const int nib_len = (int)(nib_indptr[sr + 1] - nib_indptr[sr]);
  const unsigned char* nibg = nibbles + nib0;
  for (int i = threadIdx.x; i < nbytes; i += 256) s_bm[i] = bmg[i];
  const bool nib_smem = nib_len <= nib_cap;                 // (always, when the host sized the launch from this batch)
  if (nib_smem) for (int i = threadIdx.x; i < nib_len; i += 256) s_nib[i] = nibg[i];
  const unsigned char* bmb = s_bm;
  const unsigned char* nib = nib_smem ? s_nib : nibg;
  const double sf64 = EXACT ? exact_row_sf(ex, sr) : 1.0;
  const float s = EXACT ? (float)sf64 : (sf_in ? sf_in[sr] : 1.0f);
  if (threadIdx.x == 0 && sf_out) sf_out[r] = s;
  const float inv_s = use_sf ? 1.0f / s : 1.0f;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int S = (nbytes + 255) / 256;
  __syncthreads();
  int cnt = 0;
  for (int k = 0; k < S; ++k) {
    const int b = threadIdx.x * S + k;
    if (b < nbytes) { pre[b] = (unsigned short)cnt; cnt += __popc((unsigned)bmb[b]); }
  }
  int incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  int before = 0;
  for (int k = 0; k < warp; ++k) before += warp_tot[k];
  tbase[threadIdx.x] = before + incl - cnt;
  __syncthreads();
  for (int b = threadIdx.x; b < nbytes; b += 256) {
    const unsigned bits = bmb[b];
    int pos = (int)pre[b] + tbase[b / S];
    const int c0 = b * 8;
    float y[8], x[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      float yv = 0.f;
      if ((bits >> k) & 1u) {
        const unsigned code = (nib[pos >> 1] >> ((pos & 1) * 4)) & 0xfu;
        ++pos;
        yv = (float)code;
        if (ovf_indptr && code == 15u)
          yv = EXACT ? overflow_find(ovf_indptr, ovf_entries, sr, c0 + k, yv, rows != nullptr)
                     : overflow_lookup(ovf_indptr, ovf_entries, sr, c0 + k, yv, rows != nullptr);
      }
      y[k] = yv;
      x[k] = EXACT ? exact_count(yv, sf64, ex, c0 + k) : normalise_count(yv, inv_s, use_log1p, mean, inv_std, c0 + k);
    }
    float* yo = Yout + (int64_t)r * n + c0;
    *reinterpret_cast<float4*>(yo) = make_float4(y[0], y[1], y[2], y[3]);
    *reinterpret_cast<float4*>(yo + 4) = make_float4(y[4], y[5], y[6], y[7]);
    if (sizeof(XT) == 2) {
      __nv_bfloat162 p0 = __floats2bfloat162_rn(x[0], x[1]), p1 = __floats2bfloat162_rn(x[2], x[3]);
      __nv_bfloat162 p2 = __floats2bfloat162_rn(x[4], x[5]), p3 = __floats2bfloat162_rn(x[6], x[7]);
      uint4 o;
      o.x = *reinterpret_cast<uint32_t*>(&p0); o.y = *reinterpret_cast<uint32_t*>(&p1);
      o.z = *reinterpret_cast<uint32_t*>(&p2); o.w = *reinterpret_cast<uint32_t*>(&p3);
      *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(Xout) + (int64_t)r * n + c0) = o;
    } else {
      float* xo = reinterpret_cast<float*>(Xout) + (int64_t)r * n + c0;
      *reinterpret_cast<float4*>(xo) = make_float4(x[0], x[1], x[2], x[3]);
      *reinterpret_cast<float4*>(xo + 4) = make_float4(x[4], x[5], x[6], x[7]);
    }
  }
}

inline int blocks_for(int64_t n, int t = 256) { return (int)((n + t - 1) / t); }

}  // namespace

int expand_sparse(const void* bitmap, const int64_t* nib_indptr, const void* nibbles, const float* sf_in, int M, int n,
                  const float* mean, const float* inv_std, int use_sf, int use_log1p, float* Yout, void* Xout, int x_bf16,
                  float* sf_out, const int64_t* ovf_indptr, const void* ovf_entries, int max_row_nibble_bytes, cudaStream_t s,
                  const ExactXform* ex, const int32_t* rows) {
  if (M <= 0) return DCA_OK;
  if (n / 8 > kSparseMaxBytes) { set_error("expand_sparse: at most %d genes in the sparse format (got %d)", kSparseMaxBytes * 8, n); return DCA_ERR_UNSUPPORTED; }
  const int2* oe = ovf_indptr ? reinterpret_cast<const int2*>(ovf_entries) : nullptr;
  if (!oe) ovf_indptr = nullptr;
  // dynamic shared memory: prefix table (2 B per bitmap byte) + the row's bitmap + the longest row's nibble bytes of THIS
  // batch (rows above the cap -- none when the caller passes the batch maximum -- read their nibbles from global memory)
  const int nbytes = n / 8;
  int nib_cap = max_row_nibble_bytes < 0 ? 0 : max_row_nibble_bytes;
  if (nib_cap > n / 2) nib_cap = n / 2;
  nib_cap = (nib_cap + 15) & ~15;
  const size_t dyn = (size_t)((2 * nbytes + 15) & ~15) + (size_t)((nbytes + 15) & ~15) + (size_t)nib_cap;
  // one attribute value per instantiation (index: x_bf16 + 2 * exact)
  static size_t attr[4] = {48 * 1024, 48 * 1024, 48 * 1024, 48 * 1024};
  const int inst = (x_bf16 ? 1 : 0) + (ex ? 2 : 0);
  const ExactXform e = ex ? *ex : ExactXform{};
#define DCA_SPARSE_LAUNCH(XT, EX)                                                                                      \
  do {                                                                                                                 \
    if (dyn > attr[inst]) {                                                                                            \
      DCA_CUDA_OK(cudaFuncSetAttribute(expand_sparse_kernel<XT, EX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn)); \
      attr[inst] = dyn;                                                                                                \
    }                                                                                                                  \
    expand_sparse_kernel<XT, EX><<<M, 256, dyn, s>>>((const uint32_t*)bitmap, nib_indptr, (const unsigned char*)nibbles, \
        sf_in, M, n, mean, inv_std, use_sf, use_log1p, Yout, (XT*)Xout, sf_out, ovf_indptr, oe, nib_cap, e, rows);    \
  } while (0)
  if (x_bf16) { if (ex) DCA_SPARSE_LAUNCH(__nv_bfloat16, true); else DCA_SPARSE_LAUNCH(__nv_bfloat16, false); }
  else { if (ex) DCA_SPARSE_LAUNCH(float, true); else DCA_SPARSE_LAUNCH(float, false); }
#undef DCA_SPARSE_LAUNCH
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int exact_zero_inputs(const double* mean, const double* std, int n, float* x_zero, cudaStream_t s) {
  exact_zero_kernel<<<blocks_for(n), 256, 0, s>>>(mean, std, n, x_zero);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int fill_rows_with_bias(float* C, int64_t ldc, int M, int N, const float* bias, cudaStream_t s) {
  if (M <= 0 || N <= 0) return DCA_OK;
  fill_rows_kernel<<<blocks_for((int64_t)M * N), 256, 0, s>>>(C, ldc, M, N, bias);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int col_sums_scratch_elems(int M, int N) { (void)M; return 2 * kColChunks * N; }

int col_sums(const float* a, const float* b, int64_t ld, int M, int N, double* out_sum, double* out_prod,
             double* scratch, cudaStream_t s) {
  if (M <= 0 || N <= 0) return DCA_OK;
  int rpc = cdiv(M, kColChunks);
  if (rpc < 8) rpc = 8;
  const int chunks = cdiv(M, rpc);
  double* psum = scratch;
  double* pprod = scratch + (size_t)kColChunks * N;
  col_sums_partial_kernel<<<dim3(cdiv(N, 32), chunks), dim3(32, 8), 0, s>>>(a, b, ld, M, N, rpc, psum, pprod);
  DCA_LAUNCH_CHECK();
  col_sums_fold_kernel<<<cdiv(N, 128), 128, 0, s>>>(psum, pprod, chunks, N, out_sum, out_prod);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int bn_train_finalize(const double* sum, const double* sq, int M, int N, float eps, float momentum, float* mean,
                      float* inv_std, float* moving_mean, float* moving_var, cudaStream_t s) {
  bn_train_finalize_kernel<<<cdiv(N, 128), 128, 0, s>>>(sum, sq, M, N, eps, momentum, mean, inv_std, moving_mean,
                                                        moving_var);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int bn_relu_fwd(const float* a, int64_t ld, int M, int N, const float* mean, const float* inv_std, const float* beta,
                float* xhat, float* h, __nv_bfloat16* h_bf16, cudaStream_t s) {
  bn_relu_fwd_kernel<<<blocks_for((int64_t)M * N), 256, 0, s>>>(a, ld, M, N, mean, inv_std, beta, xhat, h, h_bf16);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int bn_infer_prepare(const float* mm, const float* mv, int N, float eps, float* mean, float* inv_std, cudaStream_t s) {
  bn_infer_prepare_kernel<<<cdiv(N, 128), 128, 0, s>>>(mm, mv, N, eps, mean, inv_std);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int bias_relu_fwd(const float* a, int64_t ld, int M, int N, float* h, __nv_bfloat16* h_bf16, cudaStream_t s) {
  relu_fwd_kernel<<<blocks_for((int64_t)M * N), 256, 0, s>>>(a, ld, M, N, h, h_bf16);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int relu_bwd(float* dh, const float* h, int64_t ld, int M, int N, cudaStream_t s) {
  (void)ld;
  relu_bwd_kernel<<<blocks_for((int64_t)M * N), 256, 0, s>>>(dh, h, (int64_t)M * N);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int bn_bwd_apply(float* g, const float* xhat, int64_t ld, int M, int N, const float* inv_std, const double* sum_g,
                 const double* sum_gx, float* dbeta, cudaStream_t s, int stat_rows) {
  (void)ld;
  bn_bwd_apply_kernel<<<blocks_for((int64_t)M * N), 256, 0, s>>>(g, xhat, M, N, inv_std, sum_g, sum_gx, dbeta,
                                                                 stat_rows > 0 ? stat_rows : M);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int col_sum_to_float(const double* sum, int N, float* out, cudaStream_t s) {
  double_to_float_kernel<<<cdiv(N, 128), 128, 0, s>>>(sum, N, out);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int theta_prepare(const float* raw, int G, float* theta, float* chain, cudaStream_t s) {
  theta_prepare_kernel<<<cdiv(G, 256), 256, 0, s>>>(raw, G, theta, chain);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int theta_grad_finish(const float* dth, const float* chain, int G, float scale, float* out, cudaStream_t s) {
  theta_grad_finish_kernel<<<cdiv(G, 256), 256, 0, s>>>(dth, chain, G, scale, out);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int add_reg_grad(const float* w, float* g, int64_t n, float l1, float l2, cudaStream_t s) {
  add_reg_grad_kernel<<<blocks_for(n), 256, 0, s>>>(w, g, n, l1, l2);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int reg_penalty(const float* w, int64_t n, float l1, float l2, double* acc, cudaStream_t s) {
  int blocks = blocks_for(n);
  if (blocks > 296) blocks = 296;
  reg_penalty_kernel<<<blocks, 256, 0, s>>>(w, n, l1, l2, acc);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int rmsprop_update(float* params, const float* grads, float* rms, int64_t n, float lr, float clip, float rho,
                   float eps, float grad_scale, __nv_bfloat16* shadow, float* loss_out, cudaStream_t s) {
  rmsprop_kernel<<<blocks_for((n + 3) / 4), 256, 0, s>>>(params, grads, rms, n, lr, clip, rho, eps, grad_scale, shadow, loss_out);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int optimizer_update(float* params, const float* grads, float* s1, float* s2, int64_t n, OptScalars o, __nv_bfloat16* shadow,
                     float* loss_out, cudaStream_t s) {
  optimizer_kernel<<<blocks_for(n), 256, 0, s>>>(params, grads, s1, s2, n, o, shadow, loss_out);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

// The element rule of `ini` on one kernel tensor (fans: t.fan_in and fan_out = cols).  Orthogonal gives no rule (its elements come from the QR); DCA_ERR_BAD_ARG with the
// message set for an invalid spec or a kind the tensor's rank does not allow.
static int init_rule(const dca_initializer& ini, const InitTensor& t, InitDraw& d) {
  d = InitDraw{FILL_CONST, 0.f, 0.f, 0.0, 0.f, t.cols};
  if (t.ndim != 1 && t.ndim != 2) { set_error("initializer: %s has rank %d (1 or 2 expected)", t.name, t.ndim); return DCA_ERR_BAD_ARG; }
  if (t.rows < 1 || t.cols < 1 || (t.ndim == 1 && t.rows != 1)) {
    set_error("initializer: %s has shape (%d, %d) at rank %d", t.name, t.rows, t.cols, t.ndim); return DCA_ERR_BAD_ARG;
  }
  const int fan_in = t.fan_in, fan_out = t.cols;
  switch (ini.kind) {
    case DCA_INIT_VARIANCE_SCALING: {
      if (!(ini.scale > 0.f)) { set_error("initializer: variance_scaling needs scale > 0 (got %g)", ini.scale); return DCA_ERR_BAD_ARG; }
      if (ini.mode < DCA_FAN_IN || ini.mode > DCA_FAN_AVG) { set_error("initializer: unknown fan mode %d", ini.mode); return DCA_ERR_BAD_ARG; }
      if (ini.distribution == DCA_DIST_UNIFORM) {
        // in float, as glorot_uniform has always been drawn: limit = sqrt(3 scale / n) (= sqrt(6 / (in + out)) for it)
        const float n = ini.mode == DCA_FAN_IN ? (float)fan_in : ini.mode == DCA_FAN_OUT ? (float)fan_out
                                                                                      : 0.5f * (float)(fan_in + fan_out);
        d.kind = FILL_UNIFORM; d.center = 0.f; d.half = sqrtf(3.0f * ini.scale / fmaxf(1.0f, n));
        return DCA_OK;
      }
      if (ini.distribution != DCA_DIST_TRUNCATED_NORMAL && ini.distribution != DCA_DIST_UNTRUNCATED_NORMAL) {
        set_error("initializer: unknown distribution %d", ini.distribution); return DCA_ERR_BAD_ARG;
      }
      const double n = ini.mode == DCA_FAN_IN ? (double)fan_in : ini.mode == DCA_FAN_OUT ? (double)fan_out
                                                                                       : 0.5 * ((double)fan_in + fan_out);
      const double sd = sqrt((double)ini.scale / (n > 1.0 ? n : 1.0));
      // 0.8796...: the standard deviation of a standard normal truncated to [-2, 2]
      if (ini.distribution == DCA_DIST_TRUNCATED_NORMAL) { d.kind = FILL_TRUNC_NORMAL; d.sigma = sd / 0.87962566103423978; }
      else { d.kind = FILL_NORMAL; d.sigma = sd; }
      return DCA_OK;
    }
    case DCA_INIT_RANDOM_NORMAL:
    case DCA_INIT_TRUNCATED_NORMAL:
      if (!(ini.stddev >= 0.f)) { set_error("initializer: stddev must be >= 0 (got %g)", ini.stddev); return DCA_ERR_BAD_ARG; }
      d.kind = ini.kind == DCA_INIT_RANDOM_NORMAL ? FILL_NORMAL : FILL_TRUNC_NORMAL;
      d.sigma = (double)ini.stddev;
      return DCA_OK;
    case DCA_INIT_RANDOM_UNIFORM:
      if (!(ini.maxval >= ini.minval)) { set_error("initializer: needs minval <= maxval (got %g, %g)", ini.minval, ini.maxval); return DCA_ERR_BAD_ARG; }
      d.kind = FILL_UNIFORM; d.center = 0.5f * (ini.minval + ini.maxval); d.half = 0.5f * (ini.maxval - ini.minval);
      return DCA_OK;
    case DCA_INIT_CONSTANT:
      d.value = ini.value;
      return DCA_OK;
    case DCA_INIT_ORTHOGONAL:
    case DCA_INIT_IDENTITY:
      if (t.ndim != 2) {
        set_error("initializer: %s needs a 2-D kernel; %s is 1-D", ini.kind == DCA_INIT_ORTHOGONAL ? "orthogonal" : "identity", t.name);
        return DCA_ERR_BAD_ARG;
      }
      d.kind = FILL_IDENTITY; d.value = ini.gain;
      return DCA_OK;
    default:
      set_error("initializer: unknown kind %d", ini.kind);
      return DCA_ERR_BAD_ARG;
  }
}

int check_initializer(const dca_initializer* ini) {
  if (!ini) { set_error("initializer is NULL"); return DCA_ERR_BAD_ARG; }
  if (ini->struct_bytes != (int32_t)sizeof(dca_initializer)) {
    set_error("initializer: struct_bytes %d != sizeof(dca_initializer) %d", ini->struct_bytes, (int)sizeof(dca_initializer));
    return DCA_ERR_BAD_ARG;
  }
  return DCA_OK;
}

int check_init_tensors(const dca_initializer& ini, const InitTensor* t, int n) {
  InitDraw d;
  for (int k = 0; k < n; ++k) DCA_TRY(init_rule(ini, t[k], d));
  if (ini.kind == DCA_INIT_ORTHOGONAL && n > kMaxOrthoJobs) {
    set_error("initializer: orthogonal supports at most %d kernels (got %d)", kMaxOrthoJobs, n); return DCA_ERR_BAD_ARG;
  }
  return DCA_OK;
}

int init_kernels(const dca_initializer& ini, const InitTensor* t, int n, uint64_t seed, cudaStream_t s) {
  DCA_TRY(check_init_tensors(ini, t, n));
  InitDraw d;
  if (ini.kind != DCA_INIT_ORTHOGONAL) {
    for (int k = 0; k < n; ++k) {
      init_rule(ini, t[k], d);
      init_fill_kernel<<<blocks_for((int64_t)t[k].rows * t[k].cols), 256, 0, s>>>(t[k].w, (int64_t)t[k].rows * t[k].cols, d, seed, t[k].sid);
      DCA_LAUNCH_CHECK();
    }
    return DCA_OK;
  }
  if (n == 0) return DCA_OK;
  OrthoJobs jobs{};
  jobs.seed = seed; jobs.gain = ini.gain;
  size_t bytes = 0;
  for (int k = 0; k < n; ++k) {
    const int mn = t[k].rows < t[k].cols ? t[k].rows : t[k].cols;
    bytes += sizeof(double) * ((size_t)t[k].rows * t[k].cols + 2 * (size_t)mn);
  }
  void* ws = nullptr;
  DCA_CUDA_OK(cudaMallocAsync(&ws, bytes, s));
  size_t at = 0;
  for (int k = 0; k < n; ++k) {
    const int mn = t[k].rows < t[k].cols ? t[k].rows : t[k].cols;
    jobs.job[k] = OrthoJob{t[k].w, reinterpret_cast<double*>(static_cast<char*>(ws) + at), t[k].rows, t[k].cols, t[k].sid};
    at += sizeof(double) * ((size_t)t[k].rows * t[k].cols + 2 * (size_t)mn);
  }
  orthogonal_kernel<<<n, kQrWarps * 32, 0, s>>>(jobs);
  const cudaError_t le = cudaGetLastError();
  count_launch();
  DCA_CUDA_OK(cudaFreeAsync(ws, s));
  if (le != cudaSuccess) { set_error("orthogonal_kernel launch failed: %s", cudaGetErrorString(le)); return DCA_ERR_CUDA; }
  return DCA_OK;
}

int fill_value(float* p, int64_t n, float v, cudaStream_t s) {
  if (n <= 0) return DCA_OK;
  fill_kernel<<<blocks_for(n), 256, 0, s>>>(p, n, v);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int gather_rows_bf16(const void* X, int x_bf16, int64_t ldx, const int32_t* rows, int M, int n, __nv_bfloat16* out,
                     cudaStream_t s) {
  const int64_t tot = (int64_t)M * (n / 8);
  if (x_bf16) gather_rows_bf16_kernel<__nv_bfloat16><<<blocks_for(tot), 256, 0, s>>>((const __nv_bfloat16*)X, ldx, rows, M, n, out);
  else gather_rows_bf16_kernel<float><<<blocks_for(tot), 256, 0, s>>>((const float*)X, ldx, rows, M, n, out);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int expand_counts(const void* cnt, int bits, const float* sf_in, int M, int n, const float* mean, const float* inv_std, int use_sf,
                  int use_log1p, float* Yout, void* Xout, int x_bf16, float* sf_out, const int64_t* ovf_indptr,
                  const void* ovf_entries, cudaStream_t s, const ExactXform* ex, const int32_t* rows) {
  const int64_t tot = (int64_t)M * (n / 8);
  const unsigned char* src = reinterpret_cast<const unsigned char*>(cnt);
  const int2* oe = ovf_indptr ? reinterpret_cast<const int2*>(ovf_entries) : nullptr;
  if (!oe) ovf_indptr = nullptr;
  const ExactXform e = ex ? *ex : ExactXform{};
#define DCA_EXPAND_X(BITS, XT, EX)                                                                                   \
  expand_counts_kernel<BITS, XT, EX><<<blocks_for(tot), 256, 0, s>>>(src, sf_in, M, n, mean, inv_std, use_sf, use_log1p, \
                                                                     Yout, (XT*)Xout, sf_out, ovf_indptr, oe, e, rows)
#define DCA_EXPAND(BITS)                                                                                             \
  do {                                                                                                               \
    if (x_bf16) { if (ex) DCA_EXPAND_X(BITS, __nv_bfloat16, true); else DCA_EXPAND_X(BITS, __nv_bfloat16, false); } \
    else { if (ex) DCA_EXPAND_X(BITS, float, true); else DCA_EXPAND_X(BITS, float, false); }                         \
  } while (0)
  if (bits == 16) DCA_EXPAND(16);
  else if (bits == 8) DCA_EXPAND(8);
  else if (bits == 4) DCA_EXPAND(4);
  else { set_error("expand_counts: bits must be 4, 8 or 16 (got %d)", bits); return DCA_ERR_BAD_ARG; }
#undef DCA_EXPAND
#undef DCA_EXPAND_X
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int cast_to_bf16(const float* in, __nv_bfloat16* out, int64_t n, cudaStream_t s) {
  if (n <= 0) return DCA_OK;
  cast_bf16_kernel<<<blocks_for(n), 256, 0, s>>>(in, out, n);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

}  // namespace dca

// ---- host mirror (include/dca_b200.h)
extern "C" int dca_init_fill_host(const dca_initializer* init, uint64_t seed, uint64_t sid, int32_t ndim, int32_t rows,
                                  int32_t cols, float* out) {
  DCA_TRY(dca::check_initializer(init));
  if (!out) { dca::set_error("dca_init_fill_host: out is NULL"); return DCA_ERR_BAD_ARG; }
  // Keras _compute_fans: 2-D (in, out) -> fan_in = in; 1-D of length n -> n
  const dca::InitTensor t{out, ndim, rows, cols, ndim == 1 ? cols : rows, sid, "the kernel"};
  dca::InitDraw d;
  DCA_TRY(dca::init_rule(*init, t, d));
  const int64_t n = (int64_t)rows * cols;
  if (init->kind == DCA_INIT_ORTHOGONAL) d = dca::InitDraw{dca::FILL_NORMAL, 0.f, 0.f, 1.0, 0.f, 0};   // the draws of A
  for (int64_t i = 0; i < n; ++i) out[i] = dca::init_draw(d, seed, sid, i);
  return DCA_OK;
}
