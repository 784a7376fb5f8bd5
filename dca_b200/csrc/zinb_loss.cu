// K3: ZINB / NB negative log-likelihood, forward + backward in ONE pass over the B x G head
// outputs (replaces dca/loss.py:72-156 and the TF autodiff of it; see zinb_math.cuh).
//
// Layout: every tensor is row-major cells x genes.  A thread owns 4 consecutive genes (one
// 128-bit load per tensor per row) and walks a strip of rows, so a warp touches 512 contiguous
// bytes per tensor per row and the per-gene reduction needed by the constant-dispersion
// variants stays in registers.  HBM traffic per element: y 4 B + nh*4 B in, nh*(4|2) B out.
// The loss scalar is reduced thread -> warp shuffle -> shared memory -> one double per block,
// and a second tiny kernel folds the block partials (deterministic, no float atomics).  The constant-dispersion
// models' per-gene dL/dtheta likewise: every block stores its column sums, theta_fold_kernel adds them in row order.
#include "dca_internal.cuh"
#include <string>
#include "zinb_math.cuh"
#include "tc_common.cuh"
#include "head_act.cuh"

namespace dca {
namespace tc { extern int g_gg_profile; extern int g_head_bwd_banded; extern int g_head_bwd_stagger; }

namespace {

constexpr int kThreads = 256;
constexpr int kVec = 4;
constexpr int kColsPerBlock = kThreads * kVec;   // 1024 genes per block
constexpr int kMaxBlocks = 65536;                // bound of the per-block loss-partial buffer
// workspace: kMaxBlocks loss partials (double), the last-block arrival counter, then the dL/dtheta partials of the
// constant-dispersion backward, one float per (row chunk, gene)
constexpr size_t kThetaOff = sizeof(double) * (size_t)kMaxBlocks + 256;

// Launch-plan override (dca_set_tunable "loss_target_blocks"): blocks per launch, 0 = auto (make_plan)
int g_target_blocks = 0;

int sm_count_cached() {
  static int n = 0;
  if (!n) { int dev = 0; if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132; }
  return n;
}

struct Plan { int col_blocks, rows_per_block, row_chunks; };

inline Plan make_plan(int B, int G, int cols_per_block, int max_rpb = 1 << 30) {
  Plan p;
  p.col_blocks = cdiv(G, cols_per_block);
  // auto: small batches (C2: 4096 x 2000) run as ONE wave of 3 resident blocks per SM (block start-up and the
  // partial last wave cost 15 % there), large ones as ~5 waves for dynamic balance
  const int target = g_target_blocks > 0 ? g_target_blocks
                     : ((long long)B * G <= (32ll << 20) ? 3 * sm_count_cached() : 16 * sm_count_cached());
  int chunks = target / p.col_blocks;
  if (chunks < 1) chunks = 1;
  if (chunks > B) chunks = B;
  int rpb = cdiv(B, chunks);
  if (rpb < 2 && B >= 2) rpb = 2;                // the software prefetch wants >= 2 rows per block
  if (rpb > max_rpb) rpb = max_rpb;
  while ((long long)cdiv(B, rpb) * p.col_blocks > kMaxBlocks && rpb < max_rpb) ++rpb;
  p.rows_per_block = rpb;
  p.row_chunks = cdiv(B, rpb);
  return p;
}

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 ld4_stream(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void st4(float* p, float a, float b, float c, float d) {
  *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d);
}
__device__ __forceinline__ void st4(__nv_bfloat16* p, float a, float b, float c, float d) {
  __nv_bfloat162 lo = __floats2bfloat162_rn(a, b), hi = __floats2bfloat162_rn(c, d);
  uint2 v;
  v.x = *reinterpret_cast<uint32_t*>(&lo);
  v.y = *reinterpret_cast<uint32_t*>(&hi);
  *reinterpret_cast<uint2*>(p) = v;
}
__device__ __forceinline__ void st1(float* p, float a) { *p = a; }
__device__ __forceinline__ void st1(__nv_bfloat16* p, float a) { *p = __float2bfloat16_rn(a); }

__device__ __forceinline__ double block_reduce_sum(float v, double* smem /* >= 8 */) {
  double d = (double)v;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) smem[w] = d;
  __syncthreads();
  double t = 0.0;
  if (w == 0) {
    t = (l < (kThreads >> 5)) ? smem[l] : 0.0;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  }
  return t;   // valid in thread 0
}

// per-row operands of one thread (VEC consecutive genes)
template <int VEC>
struct RowVals { float y[VEC], m[VEC], d[VEC], p[VEC]; float sf; };

template <bool HAS_PI, bool COND_DISP, int VEC>
__device__ __forceinline__ void load_row(RowVals<VEC>& v, const float* __restrict__ Y, int64_t ldy,
                                         const int32_t* __restrict__ rows, const float* __restrict__ sf,
                                         const float* m, const float* d, const float* pi, int64_t ld, int r, int col0) {
  const int64_t yr = rows ? (int64_t)rows[r] : (int64_t)r;
  v.sf = sf ? sf[yr] : 1.0f;
  const float* yp = Y + yr * ldy + col0;
  const int64_t off = (int64_t)r * ld + col0;
  if (VEC == 4) {
    float4 t = ld4_stream(yp); v.y[0] = t.x; v.y[1] = t.y; v.y[2] = t.z; v.y[3] = t.w;
    t = ld4(m + off); v.m[0] = t.x; v.m[1] = t.y; v.m[2] = t.z; v.m[3] = t.w;
    if (COND_DISP) { t = ld4(d + off); v.d[0] = t.x; v.d[1] = t.y; v.d[2] = t.z; v.d[3] = t.w; }
    if (HAS_PI) { t = ld4(pi + off); v.p[0] = t.x; v.p[1] = t.y; v.p[2] = t.z; v.p[3] = t.w; }
  } else {
    v.y[0] = yp[0]; v.m[0] = m[off];
    if (COND_DISP) v.d[0] = d[off];
    if (HAS_PI) v.p[0] = pi[off];
  }
}

// VEC == 4: aligned 128-bit path; VEC == 1: scalar fallback for ragged G / unaligned ld.
// The next row's operands are fetched before the current row is evaluated (software prefetch),
// so every warp keeps 4 x 512 B of loads in flight while the MUFU/FMA work proceeds.
template <bool HAS_PI, bool COND_DISP, typename GT, int VEC, bool BWD>
__global__ void __launch_bounds__(kThreads)
zinb_loss_kernel(const float* __restrict__ Y, int64_t ldy, const int32_t* __restrict__ rows,
                 const float* __restrict__ sf, const float* m, const float* d, const float* pi,
                 int64_t ld, int B, int G, float ridge, float inv_n, int rows_per_block,
                 GT* dzm, GT* dzd, GT* dzp, float* __restrict__ dth_part,
                 double* __restrict__ loss_partial, const float* __restrict__ lf_global) {
  __shared__ double red[8];
  __shared__ float lf[zmath::kLogFactN];
  if (threadIdx.x < zmath::kLogFactN) lf[threadIdx.x] = lf_global[threadIdx.x];
  __syncthreads();
  using Ops = zmath::FastOps;
  const int col0 = (blockIdx.x * kThreads + threadIdx.x) * VEC;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(B, r0 + rows_per_block);
  float lsum = 0.f;
  float tacc[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) tacc[j] = 0.f;

  if (col0 < G) {
    float thg[VEC];
    if (!COND_DISP) {
#pragma unroll
      for (int j = 0; j < VEC; ++j) thg[j] = (col0 + j < G) ? d[col0 + j] : 1.f;
    }
    RowVals<VEC> cur, nxt;
    load_row<HAS_PI, COND_DISP, VEC>(cur, Y, ldy, rows, sf, m, d, pi, ld, r0, col0);
    for (int r = r0; r < r1; ++r) {
      if (r + 1 < r1) load_row<HAS_PI, COND_DISP, VEC>(nxt, Y, ldy, rows, sf, m, d, pi, ld, r + 1, col0);
      const int64_t off = (int64_t)r * ld + col0;
      float gm[VEC], gd[VEC], gp[VEC];
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        const float th = COND_DISP ? cur.d[j] : thg[j];
        const float p = HAS_PI ? cur.p[j] : 0.f;
        if (BWD) {
          zmath::Elem e = zmath::zinb_elem<Ops, HAS_PI, COND_DISP>(cur.y[j], cur.m[j], cur.sf, th, p, ridge, lf);
          lsum += e.loss;
          gm[j] = e.gm * inv_n; gd[j] = e.gd * inv_n; gp[j] = e.gp * inv_n;
          if (!COND_DISP) tacc[j] += e.gd;
        } else {
          lsum += zmath::zinb_elem_loss<Ops, HAS_PI>(cur.y[j], cur.m[j], cur.sf, th, p, ridge, lf);
        }
      }
      if (BWD) {
        if (VEC == 4) {
          st4(dzm + off, gm[0], gm[1], gm[2], gm[3]);
          if (COND_DISP) st4(dzd + off, gd[0], gd[1], gd[2], gd[3]);
          if (HAS_PI) st4(dzp + off, gp[0], gp[1], gp[2], gp[3]);
        } else {
          st1(dzm + off, gm[0]);
          if (COND_DISP) st1(dzd + off, gd[0]);
          if (HAS_PI) st1(dzp + off, gp[0]);
        }
      }
      cur = nxt;
    }
    if (BWD && !COND_DISP) {                       // this row chunk's dL/dtheta, folded in row order by theta_fold_kernel
#pragma unroll
      for (int j = 0; j < VEC; ++j)
        if (col0 + j < G) dth_part[(size_t)blockIdx.y * G + col0 + j] = tacc[j];
    }
  }
  const double tot = block_reduce_sum(lsum, red);
  if (threadIdx.x == 0) loss_partial[blockIdx.y * gridDim.x + blockIdx.x] = tot;
}

// ---------------------------------------------------------------------------------------------------------------
// "Ring" kernel (ZINB backward on aligned shapes): operands are staged through shared memory by the threads
// themselves -- every thread streams the 16 bytes it owns of each tensor row (4 consecutive genes of y, m, [d], pi)
// with cp.async (LDGSTS, L2-only) into a kRing-deep ring of its own, kRing rows ahead of the arithmetic, and reads
// them back with one 128-bit LDS per tensor.  A thread only ever reads what it copied itself, so the pipeline needs
// no barrier of any kind (cp.async.wait_group orders a thread's own copies), no producer warp and no single-lane
// issue path.  A ring shared by the block would tie every warp to the slowest warp of its block (the one that met a
// large count and took the Stirling path): no warp could run more than the ring's depth ahead of it, and warps would
// spend their issue slots polling for a slot their neighbour had not released.  The gather of the count rows costs
// one address computation (rows[] cached in shared memory).  The arithmetic runs on f32x2 pairs (zinb_math.cuh:
// zinb_zero_pair / finish_factors_pair), the queued non-zero counts return raw derivatives only (zinb_nb_raw) and
// the activation chain / clip masks / 1/N are applied once per element by its owner.
constexpr int kRing = 3;                                  // rows in flight per thread
constexpr int kMaxRowsPerBlock = 256;                     // rows of one block (row indices / size factors in shared memory)

__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// One row of one warp's 128-gene group: lane owns genes 4 lane .. 4 lane + 3 (vy / vm / vd / vp; const-disp: vd = theta of
// those genes), lanes past G carry a duplicate of the last valid vector and are !active.  The unit of the plain / general
// decision below is this warp and row, so every kernel that calls this function rounds every element the same way.
// q: the warp's queue of 128 items (16 B); refill() runs once the queued operands are in shared memory.  Returns the
// finished gradients (dzm, dzd, dzp of genes 0,1 | 2,3); accumulates the loss terms and (const-disp) the raw dL/dtheta.
struct RowGrads { float2 gmA, gmB, gdA, gdB, gpA, gpB; };

template <bool COND_DISP, class Refill>
__device__ __forceinline__ RowGrads zinb_row_ring(const float4 vy, const float4 vm, const float4 vd, const float4 vp, const float row_sf,
                                                  const bool active, const float ridge, const float inv_n, float4* q,
                                                  const float* lf, float& lsum_lg, float& lsum_nb, float& lsum_r,
                                                  float (&tacc)[kVec], Refill refill) {
  using Ops = zmath::FastOps;
  using namespace zmath;
  constexpr unsigned kFull = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  const float y[kVec] = {vy.x, vy.y, vy.z, vy.w};
  const float2 mA = make_float2(vm.x, vm.y), mB = make_float2(vm.z, vm.w);
  const float2 dA = make_float2(vd.x, vd.y), dB = make_float2(vd.z, vd.w);
  const float2 pA = make_float2(vp.x, vp.y), pB = make_float2(vp.z, vp.w);
  const float2 muA = mul2(mA, splat(row_sf)), muB = mul2(mB, splat(row_sf));        // dca/layers.py:85
  const float mu[kVec] = {muA.x, muA.y, muB.x, muB.y};
  const float dd[kVec] = {dA.x, dA.y, dB.x, dB.y};
  const float pp[kVec] = {pA.x, pA.y, pB.x, pB.y};
  // ---- queue the non-zero counts of this warp's strip (ballot compaction: items ordered by j, then lane)
  bool isnz[kVec];
  int pos[kVec], base = 0;
#pragma unroll
  for (int j = 0; j < kVec; ++j) {
    isnz[j] = active && !(y[j] < 1e-8f);                           // loss.py:138
    const unsigned bal = __ballot_sync(kFull, isnz[j]);
    pos[j] = base + __popc(bal & lt); base += __popc(bal);
  }
  const int total = base;
#pragma unroll
  for (int j = 0; j < kVec; ++j)
    if (isnz[j]) q[pos[j]] = make_float4(y[j], mu[j], dd[j], pp[j]);
  __syncwarp();
  refill();
  // ---- zero branch of my four elements, two f32x2 chains.  One range test per thread and row (min / max over its four
  // genes, FMNMX3) decides warp-uniformly whether the clip masks / the small-theta series can be skipped.
  const float m_lo = fminf(fminf(vm.x, vm.y), fminf(vm.z, vm.w)), m_hi = fmaxf(fmaxf(vm.x, vm.y), fmaxf(vm.z, vm.w));
  const float d_lo = fminf(fminf(dd[0], dd[1]), fminf(dd[2], dd[3])), d_hi = fmaxf(fmaxf(dd[0], dd[1]), fmaxf(dd[2], dd[3]));
  const bool plain = (m_lo > 1e-5f) && (m_hi < 1e6f) &&
                     (COND_DISP ? (d_lo > 0.03125f) && (d_hi < 1e4f) : (d_hi <= 1e6f));   // const-disp: theta is not an activation
  Raw2 zA, zB; Fin2 fA, fB;
  if (__all_sync(kFull, plain)) {
    zA = zinb_zero_pair<Ops, true>(muA, dA, pA); zB = zinb_zero_pair<Ops, true>(muB, dB, pB);
    fA = finish_factors_pair_plain<Ops, COND_DISP>(dA, pA, inv_n); fB = finish_factors_pair_plain<Ops, COND_DISP>(dB, pB, inv_n);
  } else {
    zA = zinb_zero_pair<Ops>(muA, dA, pA); zB = zinb_zero_pair<Ops>(muB, dB, pB);
    fA = finish_factors_pair<Ops, COND_DISP>(mA, dA, pA, inv_n); fB = finish_factors_pair<Ops, COND_DISP>(mB, dB, pB, inv_n);
  }
  lsum_lg += ((active && !isnz[0]) ? zA.lgD.x : 0.f) + ((active && !isnz[1]) ? zA.lgD.y : 0.f)
           + ((active && !isnz[2]) ? zB.lgD.x : 0.f) + ((active && !isnz[3]) ? zB.lgD.y : 0.f);
  // ---- dense NB pass over the queue (item k by lane k mod 32): raw derivatives back into the queue
  for (int k = lane; k < total; k += 32) {
    const float4 it = q[k];
    const Raw1 e = zinb_nb_raw<Ops>(it.x, it.y, it.z, it.w, lf);
    lsum_nb += e.loss;
    q[k] = make_float4(e.gmu, e.dth, e.dpi, 0.f);
  }
  __syncwarp();
  if (isnz[0]) { const float4 e = q[pos[0]]; zA.gmu.x = e.x; zA.dth.x = e.y; zA.dpi.x = e.z; }
  if (isnz[1]) { const float4 e = q[pos[1]]; zA.gmu.y = e.x; zA.dth.y = e.y; zA.dpi.y = e.z; }
  if (isnz[2]) { const float4 e = q[pos[2]]; zB.gmu.x = e.x; zB.dth.x = e.y; zB.dpi.x = e.z; }
  if (isnz[3]) { const float4 e = q[pos[3]]; zB.gmu.y = e.x; zB.dth.y = e.y; zB.dpi.y = e.z; }
  __syncwarp();
  if (ridge != 0.f) {                                              // loss.py:139-140 (uniform; ridge defaults to 0)
    if (active) lsum_r += ridge * (pA.x * pA.x + pA.y * pA.y + pB.x * pB.x + pB.y * pB.y);
    zA.dpi = fma2(splat(2.0f * ridge), pA, zA.dpi); zB.dpi = fma2(splat(2.0f * ridge), pB, zB.dpi);
  }
  if (!COND_DISP && active) { tacc[0] += zA.dth.x; tacc[1] += zA.dth.y; tacc[2] += zB.dth.x; tacc[3] += zB.dth.y; }
  RowGrads g;
  g.gmA = mul2(zA.gmu, fA.fm); g.gmB = mul2(zB.gmu, fB.fm);
  g.gdA = mul2(zA.dth, fA.fd); g.gdB = mul2(zB.dth, fB.fd);
  g.gpA = mul2(zA.dpi, fA.fp); g.gpB = mul2(zB.dpi, fB.fp);
  return g;
}

// Where the last block of a launch folds the loss partials: its arrival counter, the loss sum and the optional loss slot
// (loss * inv_n + penalty, its finite flag) and epoch accumulator (loss * batch, batch).
struct FoldArgs {
  unsigned* counter; double* loss_sum; const double* penalty; float* loss_slot; double* epoch_acc; int batch;
};

// Block sum of the per-thread loss terms into loss_partial[block]; the last block to finish folds the per-block partials
// in a FIXED order (deterministic) and finalises the loss slot.  Called by all NT threads of the block.
template <int NT>
__device__ __forceinline__ void block_loss_fold(double dsum, double* red, int* s_last, double* __restrict__ loss_partial,
                                                const FoldArgs& fa, float inv_n) {
  constexpr unsigned kFull = 0xffffffffu;
  constexpr int kWarps = NT / 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dsum += __shfl_xor_sync(kFull, dsum, o);
  if (lane == 0) red[warp] = dsum;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) t += red[w];
    loss_partial[blockIdx.y * gridDim.x + blockIdx.x] = t;
    __threadfence();
    const unsigned nblk = gridDim.x * gridDim.y;
    const unsigned done = atomicAdd(fa.counter, 1u);
    *s_last = (done == nblk - 1);
    if (*s_last) *fa.counter = 0;                                      // self-resetting
  }
  __syncthreads();
  if (!*s_last) return;
  __threadfence();
  const int n = gridDim.x * gridDim.y;
  double a = 0.0;
  for (int i = threadIdx.x; i < n; i += NT) a += __ldcg(loss_partial + i);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(kFull, a, o);
  __syncthreads();
  if (lane == 0) red[warp] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) t += red[w];
    *fa.loss_sum = t;
    if (fa.loss_slot) {
      double l = t * (double)inv_n;
      if (l != l) l = INFINITY;                                        // _nan2inf, dca/loss.py:148
      if (fa.penalty) l += *fa.penalty;
      const float lf32 = (float)l;
      fa.loss_slot[0] = lf32;
      fa.loss_slot[1] = (isfinite(lf32)) ? 0.f : 1.f;
      if (fa.epoch_acc) { fa.epoch_acc[0] += l * (double)fa.batch; fa.epoch_acc[1] += (double)fa.batch; }
    }
  }
}

template <bool COND_DISP, typename GT>
__global__ void __launch_bounds__(kThreads, 3)
zinb_loss_bwd_ring_kernel(const float* __restrict__ Y, int64_t ldy, const int32_t* __restrict__ rows,
                          const float* __restrict__ sf, const float* m, const float* d, const float* pi,
                          int64_t ld, int B, int G, float ridge, float inv_n, int rows_per_block,
                          GT* dzm, GT* dzd, GT* dzp, float* __restrict__ dth_part,
                          double* __restrict__ loss_partial, const float* __restrict__ lf_global, const FoldArgs fa) {
  extern __shared__ __align__(128) unsigned char smem_ring[];
  constexpr int kWarps = kThreads / 32;
  constexpr int kArrays = COND_DISP ? 4 : 3;                           // y, m, [d], pi
  constexpr uint32_t kSegBytes = kThreads * 16;                        // one block-row segment of one tensor (4 KB)
  constexpr uint32_t kSlotBytes = kArrays * kSegBytes;
  float4* items = reinterpret_cast<float4*>(smem_ring + kRing * kSlotBytes);           // [8 warps][128] operand copies
  __shared__ double red[kWarps];
  __shared__ float lf[zmath::kLogFactN];
  __shared__ float s_sf[kMaxRowsPerBlock];
  __shared__ int s_row[kMaxRowsPerBlock];
  __shared__ int s_last;

  using namespace zmath;
  const int warp = threadIdx.x >> 5;
  const int c0 = blockIdx.x * kColsPerBlock;
  const bool active = c0 + (int)threadIdx.x * kVec < G;                // G % 4 == 0 on this path
  // threads past the last gene (only in the last column block) work on a DUPLICATE of the last valid vector: they copy,
  // load and compute like everyone else (no divergence, nothing uninitialised) and only their results are dropped
  const int col = active ? (int)threadIdx.x * kVec : (G - c0 - kVec);
  const int r0 = blockIdx.y * rows_per_block;
  const int nrows = min(rows_per_block, B - r0);
  if (threadIdx.x < kLogFactN) lf[threadIdx.x] = lf_global[threadIdx.x];
  for (int t = threadIdx.x; t < nrows; t += kThreads) {
    const int yr = rows ? rows[r0 + t] : (r0 + t);
    s_row[t] = yr;
    s_sf[t] = sf ? sf[yr] : 1.0f;
  }
  __syncthreads();

  const uint32_t my = tc::smem_u32(smem_ring) + threadIdx.x * 16;      // my 16 bytes inside every segment
  const uint32_t ring_end = my + kRing * kSlotBytes;
  const float* ysrc = Y + c0 + col;
  const float* msrc = m + (int64_t)r0 * ld + c0 + col;
  const float* dsrc = COND_DISP ? d + (int64_t)r0 * ld + c0 + col : nullptr;
  const float* psrc = pi + (int64_t)r0 * ld + c0 + col;
  const uint32_t ldy32 = (uint32_t)ldy;                                // leading dimensions are < 2^32 elements
  // copy cursor: the row that is streamed next, its slot and the advancing source pointers (no per-row 64-bit multiplies)
  int nxt = 0;
  uint32_t wslot = my;
  auto cp16 = [](uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
  };
  auto issue_next = [&]() {                                            // stream row `nxt` of my 4 genes into the next slot
    cp16(wslot, ysrc + (uint64_t)((uint32_t)s_row[nxt]) * ldy32);
    cp16(wslot + kSegBytes, msrc);
    if (COND_DISP) cp16(wslot + 2 * kSegBytes, dsrc);
    cp16(wslot + (kArrays - 1) * kSegBytes, psrc);
    msrc += ld; psrc += ld;
    if (COND_DISP) dsrc += ld;
    ++nxt; wslot += kSlotBytes;
    if (wslot == ring_end) wslot = my;
  };

  float lsum_lg = 0.f, lsum_nb = 0.f, lsum_r = 0.f;      // sum of lg2(D) over my zero counts | NLL of the items I evaluated | ridge
  float tacc[kVec] = {0.f, 0.f, 0.f, 0.f};
  {
#pragma unroll
    for (int i = 0; i < kRing; ++i) {                                  // one group per row, empty groups keep the count fixed
      if (i < nrows) issue_next();
      cp_async_commit();
    }
    float4* q = items + warp * (32 * kVec);
    float thg[kVec] = {1.f, 1.f, 1.f, 1.f};
    if (!COND_DISP) {
#pragma unroll
      for (int j = 0; j < kVec; ++j) thg[j] = d[c0 + col + j];
    }
    GT* om = dzm + (int64_t)r0 * ld + c0 + col;
    GT* od = COND_DISP ? dzd + (int64_t)r0 * ld + c0 + col : nullptr;
    GT* op = dzp + (int64_t)r0 * ld + c0 + col;
    uint32_t rslot = my;
    auto lds128 = [](uint32_t addr) {
      float4 v;
      asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
      return v;
    };
    for (int i = 0; i < nrows; ++i) {
      cp_async_wait<kRing - 1>();                                      // my copies of row i have landed
      const float4 vy = lds128(rslot), vm = lds128(rslot + kSegBytes);
      const float4 vd = COND_DISP ? lds128(rslot + 2 * kSegBytes) : make_float4(thg[0], thg[1], thg[2], thg[3]);
      const float4 vp = lds128(rslot + (kArrays - 1) * kSegBytes);
      rslot += kSlotBytes;
      if (rslot == ring_end) rslot = my;
      const float row_sf = s_sf[i];
      // refill: the operands of row i have been consumed (they fed the ballots / the queue): stream row i + kRing
      const RowGrads g = zinb_row_ring<COND_DISP>(vy, vm, vd, vp, row_sf, active, ridge, inv_n, q, lf, lsum_lg, lsum_nb,
                                                  lsum_r, tacc, [&] { if (nxt < nrows) issue_next(); cp_async_commit(); });
      if (active) {
        st4(om, g.gmA.x, g.gmA.y, g.gmB.x, g.gmB.y);
        if (COND_DISP) st4(od, g.gdA.x, g.gdA.y, g.gdB.x, g.gdB.y);
        st4(op, g.gpA.x, g.gpA.y, g.gpB.x, g.gpB.y);
      }
      om += ld; op += ld;
      if (COND_DISP) od += ld;
    }
    if (!COND_DISP && active)                      // this row chunk's dL/dtheta, folded in row order by theta_fold_kernel
      *reinterpret_cast<float4*>(dth_part + (size_t)blockIdx.y * G + c0 + col) = make_float4(tacc[0], tacc[1], tacc[2], tacc[3]);
  }
  // ---- block reduction, then the last block to finish folds the per-block partials in a FIXED order
  block_loss_fold<kThreads>((double)lsum_nb + (double)lsum_r - (double)kLn2 * (double)lsum_lg,   // -log D = -ln2 * lg2 D
                            red, &s_last, loss_partial, fa, inv_n);
}

// ---------------------------------------------------------------------------------------------------------------
// Heads + loss kernel (zinb-conddisp, tensor-core training step): the head pre-activations are computed where the loss is
// computed, so the fp32 mean / dispersion / pi never reach HBM.  Per element the kernel moves the count (4 B in) and the
// three bf16 gradients (6 B out); H3 and the head weights are re-read from L2.
//
// One CTA = four warpgroups sharing the bf16 weights of one 128-gene tile (3 x 16 KB, TMA).  A CTA owns a contiguous range
// of (gene tile, 64-cell block) units, tile-major; its warpgroups take the blocks of a tile in turn.  Per block a warpgroup
// loads H3 (TMA, 8 KB) and walks it in four pieces of 16 consecutive cells; warp w walks cells 4w .. 4w + 3 of a piece.
// Per piece the warpgroup computes each head's products once, gene-major (head_piece_mma: 128 genes x 16 cells, the three
// heads committed back to back), and every thread stores its raw fp32 accumulators into the staging rows of the warp that
// walks that cell (warp-private areas, 4 rows x 128 genes x 3 heads each); the counts of a warp's rows stream into its
// slot by cp.async under the products, so that no registers hold them next to the accumulators.  The warp then walks its
// 4 rows: each lane applies K2's epilogue (head_out, same inputs, so m, theta and pi carry K2's bits when the gene-major
// accumulators equal K2's cell-major ones) to its own 4 genes x 3 heads and runs zinb_row_ring -- the per-row body of the
// ring kernel, with the same warp / lane / 128-gene mapping -- and stores bf16 dZ.  Two warpgroup barriers per piece
// order the staging stores against the walks of the previous and the current piece.  The staging of one piece is what fits
// four warpgroups (16 warps to hide the latency of the row walk) on an SM with at most 128 registers per thread.
namespace hl {
constexpr int kWG = 4;                                       // warpgroups per CTA
constexpr int kCtaThreads = 128 * kWG;
constexpr int kRows = 4;                                     // rows per warp and piece
constexpr int kPieceCells = 4 * kRows;                       // cells per piece (the four warps of a warpgroup)
constexpr int kPieces = 64 / kPieceCells;                    // pieces per 64-cell block
constexpr uint32_t kWHeadBytes = 64 * 128 * 2;               // one head's W tile: two 64-gene boxes of [64 k][64 genes] bf16
constexpr uint32_t kHBytes = 64 * 64 * 2;                    // one 64-cell H3 block
constexpr uint32_t kRowBytes = 3 * 128 * 4;                  // m | d | pi accumulators of one row's 128 genes
constexpr uint32_t kQPad = 512;                              // the NB queue of row k (2 KB) starts 512 B ahead of row k's
                                                             // operands and overwrites them once they are in registers
constexpr uint32_t kOffY = kQPad + kRows * kRowBytes;        // the piece's count rows (cp.async, 16 B per lane and row)
constexpr uint32_t kWarpBytes = kOffY + kRows * 128 * 4 + 32;   // + 32: consecutive warps' areas 32 B apart modulo 128 B
static_assert(kWarpBytes % 128 == 32, "stage_head's stores are conflict-free only with warp areas 32 B apart modulo 128 B");
constexpr uint32_t kOffH = 3 * kWHeadBytes;
constexpr uint32_t kOffStage = kOffH + kWG * kHBytes;
constexpr uint32_t kOffBias = kOffStage + kWG * 4 * kWarpBytes;
constexpr uint32_t kSmemBytes = kOffBias + 3 * 128 * 4 + 1024;   // + alignment of the swizzled TMA destinations
static_assert(kSmemBytes + 1024 <= 227 * 1024, "heads_loss_kernel: dynamic + 1 KB static shared memory over the sm_90 limit");

struct Params {
  const float* bias[3];
  const float* Y; int64_t ldy; const int32_t* rows; const float* sf;
  int B, G, nblk, units;                                     // units < 2^31 (checked on the host)
  float ridge, inv_n;
  __nv_bfloat16* dz[3]; int64_t ldz;
  double* loss_partial; const float* lf;
};

// float4 slot of genes 4i..4i+3 in staged row k: XOR-swizzled so that the fragment stores of the 4 rows of a piece spread
// over all banks (rows are 1536 B apart, a multiple of 128 B)
__device__ __forceinline__ uint32_t slot16(int i, int k) { return (uint32_t)((i ^ ((2 * k) & 6)) * 16); }

// Stores head h's gene-major accumulators of a piece (head_piece_mma), raw, into the staging rows of the warps that walk
// them: cell c of the piece is row c % 4 of warp c / 4 of the warpgroup (`wg_stage`: its first warp's area).  In the
// fragment, acc[mb][i] of lane l is gene 64 mb + 16 warp + l / 4 + 8 (i / 2 % 2) and cell 8 (i / 4) + 2 (l % 4) + i % 2,
// i.e. row 2 (l & 1) + (i & 1) of warp 2 (i / 4) + (l >> 1 & 1).  Its 16-byte slot (slot16) is gene / 4 XOR 4 (l & 1) + 2
// (i & 1), and these bit fields do not overlap, so the address is a per-lane base plus a constant per (mb, i):
//   slot = (4 warp ^ 4 (l & 1)) | l >> 4   |   16 mb | 2 ((i / 2 ^ i) & 1).
// Each store instruction writes 32 distinct banks: lane bit 0 flips 16 banks (slot bit 2), bit 1 moves 8 (the next warp's
// area, 32 B further modulo 128 B), bits 2-3 pick the word and bit 4 moves 4 (slot bit 0).
__device__ __forceinline__ void stage_head(const float (&acc)[2][8], uint8_t* wg_stage, int h) {
  const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  uint8_t* base = wg_stage + ((lane >> 1) & 1) * kWarpBytes + kQPad + 2 * (lane & 1) * kRowBytes + h * 512 + ((lane >> 2) & 3) * 4 +
                  ((((4 * warp) ^ (4 * (lane & 1))) | (lane >> 4)) * 16);
#pragma unroll
  for (int mb = 0; mb < 2; ++mb)
#pragma unroll
    for (int i = 0; i < 8; ++i)
      *reinterpret_cast<float*>(base + 2 * (i >> 2) * kWarpBytes + (i & 1) * kRowBytes + (16 * mb | (2 * (((i >> 1) ^ i) & 1))) * 16) =
          acc[mb][i];
}

// K2's epilogue of one head on a lane's 4 genes
template <int KIND>
__device__ __forceinline__ float4 head_out4(const float4 a, const float4 b) {
  return make_float4(tc::head_out<KIND>(a.x, b.x, 1.0f), tc::head_out<KIND>(a.y, b.y, 1.0f),
                     tc::head_out<KIND>(a.z, b.z, 1.0f), tc::head_out<KIND>(a.w, b.w, 1.0f));
}
}  // namespace hl

__global__ void __launch_bounds__(hl::kCtaThreads, 1)
heads_loss_kernel(const __grid_constant__ CUtensorMap map_h, const __grid_constant__ CUtensorMap map_w0,
                  const __grid_constant__ CUtensorMap map_w1, const __grid_constant__ CUtensorMap map_w2, const hl::Params p,
                  const FoldArgs fa) {
  using namespace hl;
  using namespace tc;
  extern __shared__ __align__(1024) uint8_t smem_hl_raw[];
  uint8_t* smem = smem_hl_raw + ((1024u - (smem_u32(smem_hl_raw) & 1023u)) & 1023u);
  __shared__ uint64_t w_bar, h_bar[kWG];
  __shared__ float lf[zmath::kLogFactN];
  __shared__ double red[kCtaThreads / 32];
  __shared__ int s_last;
  const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
  float* s_bias = reinterpret_cast<float*>(smem + kOffBias);
  uint8_t* h_buf = smem + kOffH + wg * kHBytes;
  uint8_t* wg_stage = smem + kOffStage + wg * 4 * kWarpBytes;             // the warpgroup's four warp areas
  uint8_t* wbase = wg_stage + warp * kWarpBytes;                          // this warp's queue pad + 4 staged rows + counts
  uint8_t* rows_base = wbase + kQPad;
  const uint32_t my_y = smem_u32(wbase + kOffY) + lane * 16;             // my 16 bytes of the piece's count row 0
  if (tid < zmath::kLogFactN) lf[tid] = p.lf[tid];
  if (tid == 0) {
    mbar_init(&w_bar, 1);
    for (int g = 0; g < kWG; ++g) mbar_init(&h_bar[g], 1);
    fence_barrier_init();
  }
  __syncthreads();
  const CUtensorMap* mw[3] = {&map_w0, &map_w1, &map_w2};
  auto load_h = [&](int blk) {
    if ((tid & 127) == 0) { mbar_expect_tx(&h_bar[wg], kHBytes); tma_load_2d(h_buf, &map_h, 0, blk * 64, &h_bar[wg]); }
  };
  const int u0 = (int)((long long)blockIdx.x * p.units / gridDim.x), u1 = (int)((long long)(blockIdx.x + 1) * p.units / gridDim.x);
  uint32_t w_phase = 0, h_phase = 0;
  float lsum_lg = 0.f, lsum_nb = 0.f, lsum_r = 0.f;
  float tacc[kVec] = {0.f, 0.f, 0.f, 0.f};
  for (int u = u0; u < u1;) {
    const int t = u / p.nblk;
    const int seg_end = min(u1, (t + 1) * p.nblk);
    const int b_end = seg_end - t * p.nblk;
    int blk = u - t * p.nblk + wg;
    __syncthreads();                                                      // every warpgroup is done with the previous tile
    if (tid == 0) {
      mbar_expect_tx(&w_bar, 3 * kWHeadBytes);
      for (int h = 0; h < 3; ++h) {
        tma_load_2d(smem + h * kWHeadBytes, mw[h], t * 128, 0, &w_bar);
        tma_load_2d(smem + h * kWHeadBytes + kWHeadBytes / 2, mw[h], t * 128 + 64, 0, &w_bar);
      }
    }
    if (tid < 3 * 128) {
      const int gcol = t * 128 + (tid & 127);                             // 384 threads: one bias of each head each
      const float* bias = wg == 0 ? p.bias[0] : (wg == 1 ? p.bias[1] : p.bias[2]);   // (no local copy of p for p.bias[wg])
      s_bias[tid] = gcol < p.G ? bias[gcol] : 0.f;
    }
    if (blk < b_end) load_h(blk);
    __syncthreads();
    mbar_wait(&w_bar, w_phase); w_phase ^= 1;
    // my four genes; lanes past G duplicate the last valid vector (as in the ring kernel) and only their results are dropped
    const int gvalid = min(128, p.G - t * 128);
    const bool active = 4 * lane < gvalid;
    const int col = active ? 4 * lane : gvalid - kVec;
    const int64_t gcol0 = (int64_t)t * 128 + col;
    for (; blk < b_end; blk += kWG) {
      mbar_wait(&h_bar[wg], h_phase); h_phase ^= 1;
      // pieces wholly past the batch are skipped (the same for the whole warpgroup)
      const int last_piece = min(kPieces, (p.B - blk * 64 + kPieceCells - 1) / kPieceCells) - 1;
      for (int piece = 0; piece <= last_piece; ++piece) {
        float acc[3][2][8];                                               // [head][gene m-block][fragment]
        const uint32_t h_piece = smem_u32(h_buf) + piece * kPieceCells * 128;
        head_piece_mma(acc[0], h_piece, smem_u32(smem));
        head_piece_mma(acc[1], h_piece, smem_u32(smem) + kWHeadBytes);
        head_piece_mma(acc[2], h_piece, smem_u32(smem) + 2 * kWHeadBytes);
        const int r0 = blk * 64 + piece * kPieceCells + warp * kRows;     // first of this warp's 4 rows in the piece
        int my_yr = 0; float my_sf = 1.f;                                 // lane k < 4: count row / size factor of row r0 + k
        if (lane < kRows && r0 + lane < p.B) {
          my_yr = p.rows ? p.rows[r0 + lane] : r0 + lane;
          my_sf = p.sf ? p.sf[my_yr] : 1.0f;
        }
#pragma unroll
        for (int k = 0; k < kRows; ++k) {                                 // counts of the piece, in flight under the products
          const int yr = __shfl_sync(0xffffffffu, my_yr, k);              // (through shared memory: no registers held)
          if (r0 + k < p.B)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(my_y + k * 512), "l"(p.Y + (int64_t)yr * p.ldy + gcol0)
                         : "memory");
        }
        cp_async_commit();
        named_barrier_sync(1 + wg, 128);                                  // every warp has walked the previous piece's rows
        wgmma_wait<2>(); acc_fence(acc[0][0]); acc_fence(acc[0][1]);
        stage_head(acc[0], wg_stage, 0);
        wgmma_wait<1>(); acc_fence(acc[1][0]); acc_fence(acc[1][1]);
        stage_head(acc[1], wg_stage, 1);
        wgmma_wait<0>(); acc_fence(acc[2][0]); acc_fence(acc[2][1]);
        stage_head(acc[2], wg_stage, 2);
        named_barrier_sync(1 + wg, 128);                                  // the piece is staged and every product is done
        if (piece == last_piece && blk + kWG < b_end) load_h(blk + kWG);  // the warpgroup is done with this H3 block
        cp_async_wait<0>();                                               // my count copies have landed (I read only those)
        __syncwarp();
        for (int k = 0; k < kRows; ++k) {
          const int r = r0 + k;
          if (r >= p.B) break;                                            // warp-uniform: the last block's tail
          float4 vy;
          asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(vy.x), "=f"(vy.y), "=f"(vy.z), "=f"(vy.w) : "r"(my_y + k * 512)
                       : "memory");
          const float row_sf = __shfl_sync(0xffffffffu, my_sf, k);
          const uint8_t* src = rows_base + k * kRowBytes + slot16(col >> 2, k);
          const float4 am = *reinterpret_cast<const float4*>(src);
          const float4 ad = *reinterpret_cast<const float4*>(src + 512);
          const float4 ap = *reinterpret_cast<const float4*>(src + 1024);
          __syncwarp();                                                   // row k's queue overwrites these operands
          const float4 vm = head_out4<EPI_MEAN_ACT>(am, *reinterpret_cast<const float4*>(s_bias + col));
          const float4 vd = head_out4<EPI_DISP_ACT>(ad, *reinterpret_cast<const float4*>(s_bias + 128 + col));
          const float4 vp = head_out4<EPI_SIGMOID>(ap, *reinterpret_cast<const float4*>(s_bias + 256 + col));
          float4* q = reinterpret_cast<float4*>(wbase + k * kRowBytes);
          const RowGrads g = zinb_row_ring<true>(vy, vm, vd, vp, row_sf, active, p.ridge, p.inv_n, q, lf, lsum_lg, lsum_nb,
                                                 lsum_r, tacc, [] {});
          if (active) {
            const int64_t off = (int64_t)r * p.ldz + gcol0;
            st4(p.dz[0] + off, g.gmA.x, g.gmA.y, g.gmB.x, g.gmB.y);
            st4(p.dz[1] + off, g.gdA.x, g.gdA.y, g.gdB.x, g.gdB.y);
            st4(p.dz[2] + off, g.gpA.x, g.gpA.y, g.gpB.x, g.gpB.y);
          }
        }
      }
    }
    u = seg_end;
  }
  block_loss_fold<kCtaThreads>((double)lsum_nb + (double)lsum_r - (double)zmath::kLn2 * (double)lsum_lg, red, &s_last,
                            p.loss_partial, fa, p.inv_n);
}

// ---------------------------------------------------------------------------------------------------------------
// Debug checks (dca/loss.py:87-100, NB.loss with debug=True), per element in the reference's float32 form:
//   theta' = min(theta, 1e6) (a NaN theta stays NaN, as with tf.minimum), y_pred = m * sf,
//   t1 = lgamma(theta' + eps) + lgamma(y + 1) - lgamma(y + theta' + eps),
//   t2 = (theta' + y) log(1 + y_pred / (theta' + eps)) + y (log(theta' + eps) - log(y_pred + eps)).
// A launch of its own ahead of the loss kernel, reading the same operands: the loss kernels are not touched, so the
// loss, the gradients and every accumulator keep their bits with the checks on.  The report holds, per term, the count
// of non-finite elements and the complement of the smallest key (batch row << 32 | gene), so that an all-zero report
// means "nothing flagged": integer atomics only, one per warp and term that saw something, the same bits on every run.
struct DbgReport { unsigned long long count[3], inv_key[3]; };   // y_pred, t1, t2
static_assert(sizeof(DbgReport) == kDebugReportBytes, "dca_debug_report's device form");

__global__ void __launch_bounds__(256)
debug_check_kernel(const float* __restrict__ Y, int64_t ldy, const int32_t* __restrict__ rows, const float* __restrict__ sf,
                   const float* __restrict__ m, int64_t ldm, const float* __restrict__ theta, int64_t ld_theta, int B, int G,
                   DbgReport* __restrict__ rep) {
  constexpr float eps = 1e-10f;
  unsigned cnt[3] = {0u, 0u, 0u};
  unsigned long long inv_key[3] = {0ull, 0ull, 0ull};
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < G) {
    for (int r = blockIdx.y; r < B; r += gridDim.y) {
      const int64_t yr = rows ? (int64_t)rows[r] : (int64_t)r;
      const float y = Y[yr * ldy + g];
      const float s = sf ? sf[yr] : 1.0f;
      const float mv = m[(int64_t)r * ldm + g];
      const float tv = theta[(int64_t)r * ld_theta + g];
      const float th = tv > 1e6f ? 1e6f : tv;
      const float yp = mv * s;
      const float te = th + eps;
      const float t1 = lgammaf(te) + lgammaf(y + 1.0f) - lgammaf(y + th + eps);
      const float t2 = (th + y) * logf(1.0f + yp / te) + y * (logf(te) - logf(yp + eps));
      const bool bad[3] = {!isfinite(yp), !isfinite(t1), !isfinite(t2)};
      const unsigned long long inv = ~(((unsigned long long)(unsigned)r << 32) | (unsigned)g);
#pragma unroll
      for (int k = 0; k < 3; ++k)
        if (bad[k]) { ++cnt[k]; inv_key[k] = inv > inv_key[k] ? inv : inv_key[k]; }
    }
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {                       // warp sum / max, one set of atomics per warp that saw something
    unsigned c = cnt[k];
    unsigned long long v = inv_key[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      c += __shfl_xor_sync(0xffffffffu, c, o);
      const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
      v = w > v ? w : v;
    }
    if ((threadIdx.x & 31) == 0 && c) { atomicAdd(&rep->count[k], (unsigned long long)c); atomicMax(&rep->inv_key[k], v); }
  }
}

__global__ void fold_partials_kernel(const double* __restrict__ part, int n, double* out, int accumulate,
                                     const double* penalty, float inv_n, int batch, float* loss_slot, double* epoch_acc) {
  __shared__ double sm[32];
  double a = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) a += part[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = a;
  __syncthreads();
  if (threadIdx.x < 32) {
    a = (threadIdx.x < (blockDim.x >> 5)) ? sm[threadIdx.x] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (threadIdx.x == 0) {
      *out = accumulate ? (*out + a) : a;
      if (loss_slot) {                                            // fused finalize
        double l = a * (double)inv_n;
        if (l != l) l = INFINITY;                                 // _nan2inf, dca/loss.py:148
        if (penalty) l += *penalty;
        const float lf = (float)l;
        loss_slot[0] = lf;
        loss_slot[1] = (isfinite(lf)) ? 0.f : 1.f;
        if (epoch_acc) { epoch_acc[0] += l * (double)batch; epoch_acc[1] += (double)batch; }
      }
    }
  }
}

// dL/dtheta per gene: the row chunks' partials (dth_part[chunk][gene]) added in row-chunk order, so that the same
// inputs and plan give the same bits on every run.  One thread per gene reads 16 chunks before it adds them: at 103
// chunks x 20000 genes the fold takes 7-8 us, against about 10 us with 8 loads in flight (H100 80GB HBM3, 700 W).
__global__ void theta_fold_kernel(const float* __restrict__ part, int chunks, int G, float* __restrict__ dtheta) {
  constexpr int kBatch = 16;
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const float* p = part + g;
  float t = 0.f;
  int c = 0;
  for (; c + kBatch <= chunks; c += kBatch) {
    float v[kBatch];
#pragma unroll
    for (int k = 0; k < kBatch; ++k) v[k] = p[(size_t)(c + k) * G];
#pragma unroll
    for (int k = 0; k < kBatch; ++k) t += v[k];
  }
  for (; c < chunks; ++c) t += p[(size_t)c * G];
  dtheta[g] = t;
}

// Row chunks of the largest plan launch() can choose for a batch of at most B rows: make_plan's target-driven chunk
// count at the widest columns (the vector plans), or the ring plan's cdiv(B, kMaxRowsPerBlock) where its row cap binds.
// Non-decreasing in B, so a workspace sized for max_batch holds the plan of every smaller batch.
int max_row_chunks(int B, int G) {
  const int target = g_target_blocks > 0 ? g_target_blocks
                     : ((long long)B * G <= (32ll << 20) ? 3 * sm_count_cached() : 16 * sm_count_cached());
  const int chunks = std::max(1, target / cdiv(G, kColsPerBlock));
  return std::min(B, std::max(chunks, cdiv(B, kMaxRowsPerBlock)));
}

__device__ float g_log_fact[zmath::kLogFactN];

// log(k!) table in device global memory, filled once per device on first use
const float* log_fact_table_device() {
  static thread_local int ready_dev = -1;
  static thread_local float* cached = nullptr;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { set_error("cudaGetDevice failed"); return nullptr; }
  if (ready_dev == dev && cached) return cached;       // (also keeps stream capture free of non-stream API calls)
  float* p = nullptr;
  if (cudaGetSymbolAddress((void**)&p, g_log_fact) != cudaSuccess) { set_error("cudaGetSymbolAddress failed"); return nullptr; }
  cached = p;
  if (ready_dev != dev) {
    float t[zmath::kLogFactN];
    zmath::fill_log_fact(t);
    if (cudaMemcpy(p, t, sizeof(t), cudaMemcpyHostToDevice) != cudaSuccess) { set_error("log-factorial table upload failed"); return nullptr; }
    ready_dev = dev;
  }
  return p;
}

template <bool BWD>
int launch(const LossArgs& a, cudaStream_t s) {
  if (a.B <= 0 || a.G <= 0) { set_error("zinb_loss: empty batch (B=%d, G=%d)", a.B, a.G); return DCA_ERR_BAD_ARG; }
  const bool has_pi = (a.ae_type == DCA_AE_ZINB_CONDDISP || a.ae_type == DCA_AE_ZINB);
  const bool cond = (a.ae_type == DCA_AE_ZINB_CONDDISP || a.ae_type == DCA_AE_NB_CONDDISP);
  if (!a.Y || !a.m || !a.d || (has_pi && !a.pi) || !a.loss_sum) { set_error("zinb_loss: null input"); return DCA_ERR_BAD_ARG; }
  if (BWD && (!a.dzm || (cond && !a.dzd) || (has_pi && !a.dzp) || (!cond && !a.dtheta))) {
    set_error("zinb_loss: null gradient output"); return DCA_ERR_BAD_ARG;
  }
  const float* lf_dev = log_fact_table_device();
  if (!lf_dev) return DCA_ERR_CUDA;
  double* lpart = reinterpret_cast<double*>(a.ws);
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  bool vec = (a.G % 4 == 0) && (a.ld % 4 == 0) && (a.ldy % 4 == 0) && al16(a.Y) && al16(a.m) && (!cond || al16(a.d)) &&
             (!has_pi || al16(a.pi));
  if (BWD) vec = vec && al16(a.dzm) && (!cond || al16(a.dzd)) && (!has_pi || al16(a.dzp));
  const Plan p = make_plan(a.B, a.G, vec ? kColsPerBlock : kThreads);
  dim3 grid(p.col_blocks, p.row_chunks), block(kThreads);
  // ZINB backward on aligned shapes: the ring kernel, unless its plan (at most kMaxRowsPerBlock rows per block) needs
  // more blocks than the partial buffer holds or more row chunks than a grid's y dimension
  const Plan ps = make_plan(a.B, a.G, kColsPerBlock, kMaxRowsPerBlock);
  const bool ring = BWD && vec && has_pi && (long long)ps.row_chunks * ps.col_blocks <= kMaxBlocks && ps.row_chunks <= 65535;
  const int row_chunks = ring ? ps.row_chunks : p.row_chunks;
  const bool theta = BWD && !cond;                                    // const-disp: dL/dtheta partials per row chunk
  const size_t need = kThetaOff + (theta ? sizeof(float) * (size_t)row_chunks * (size_t)a.G : 0);
  if (!a.ws || a.ws_bytes < need) {
    set_error("zinb_loss: workspace too small for a plan of %d row chunks (%zu < %zu bytes)", row_chunks, a.ws_bytes, need);
    return DCA_ERR_BAD_ARG;
  }
  float* tpart = theta ? reinterpret_cast<float*>(static_cast<char*>(a.ws) + kThetaOff) : nullptr;
  auto fold_theta = [&]() -> int {
    if (!theta) return DCA_OK;
    theta_fold_kernel<<<cdiv(a.G, 128), 128, 0, s>>>(tpart, row_chunks, a.G, a.dtheta);
    DCA_LAUNCH_CHECK();
    return DCA_OK;
  };

  if (ring) {
    grid = dim3(ps.col_blocks, ps.row_chunks);
    FoldArgs fa{reinterpret_cast<unsigned*>(reinterpret_cast<char*>(a.ws) + sizeof(double) * (size_t)kMaxBlocks), a.loss_sum,
                a.fin_penalty, a.fin_loss_slot, a.fin_epoch_acc, a.fin_batch};
    if (!a.counter_ready) DCA_CUDA_OK(cudaMemsetAsync(fa.counter, 0, sizeof(unsigned), s));
#define DCA_RING(CD, GT)                                                                                          \
  do {                                                                                                             \
    constexpr size_t sm = (size_t)kRing * (CD ? 4 : 3) * kColsPerBlock * 4 + (size_t)(kThreads / 32) * 32 * kVec * 16; \
    static bool attr = false;                                                                                      \
    if (!attr) { DCA_CUDA_OK(cudaFuncSetAttribute(zinb_loss_bwd_ring_kernel<CD, GT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm)); attr = true; } \
    zinb_loss_bwd_ring_kernel<CD, GT><<<grid, kThreads, sm, s>>>(a.Y, a.ldy, a.rows, a.sf, a.m, a.d, a.pi, a.ld, a.B, a.G, a.ridge, \
        a.inv_n, ps.rows_per_block, (GT*)a.dzm, (GT*)a.dzd, (GT*)a.dzp, tpart, lpart, lf_dev, fa);                  \
  } while (0)
    if (a.grad_bf16) { if (cond) DCA_RING(true, __nv_bfloat16); else DCA_RING(false, __nv_bfloat16); }
    else             { if (cond) DCA_RING(true, float); else DCA_RING(false, float); }
#undef DCA_RING
    DCA_LAUNCH_CHECK();
    return fold_theta();                                                // the loss fold is done by the last block
  }
#define DCA_LOSS_LAUNCH(HP, CD, GT, V)                                                                 \
  zinb_loss_kernel<HP, CD, GT, V, BWD><<<grid, block, 0, s>>>(                                          \
      a.Y, a.ldy, a.rows, a.sf, a.m, a.d, a.pi, a.ld, a.B, a.G, a.ridge, a.inv_n, p.rows_per_block,      \
      (GT*)a.dzm, (GT*)a.dzd, (GT*)a.dzp, tpart, lpart, lf_dev)
#define DCA_LOSS_DISPATCH(GT, V)                                   \
  do {                                                             \
    if (has_pi && cond) DCA_LOSS_LAUNCH(true, true, GT, V);        \
    else if (has_pi && !cond) DCA_LOSS_LAUNCH(true, false, GT, V); \
    else if (!has_pi && cond) DCA_LOSS_LAUNCH(false, true, GT, V); \
    else DCA_LOSS_LAUNCH(false, false, GT, V);                     \
  } while (0)
  if (BWD && a.grad_bf16) {
    if (vec) DCA_LOSS_DISPATCH(__nv_bfloat16, 4); else DCA_LOSS_DISPATCH(__nv_bfloat16, 1);
  } else {
    if (vec) DCA_LOSS_DISPATCH(float, 4); else DCA_LOSS_DISPATCH(float, 1);
  }
#undef DCA_LOSS_DISPATCH
#undef DCA_LOSS_LAUNCH
  DCA_LAUNCH_CHECK();
  fold_partials_kernel<<<1, 256, 0, s>>>(lpart, (int)(grid.x * grid.y), a.loss_sum, BWD ? 0 : 1, a.fin_penalty, a.inv_n,
                                         a.fin_batch, BWD ? a.fin_loss_slot : nullptr, a.fin_epoch_acc);
  DCA_LAUNCH_CHECK();
  return fold_theta();
}

}  // namespace

const float* loss_log_fact_table() { return log_fact_table_device(); }
int g_fused_heads_default = 0;            // 1: engines created from now on use the fused head/loss/backward kernel

size_t loss_workspace_bytes(int B, int G) {
  return kThetaOff + sizeof(float) * (size_t)max_row_chunks(B, G) * (size_t)G;
}

int zinb_loss_fwd_bwd(const LossArgs& a, cudaStream_t s) { return launch<true>(a, s); }
int zinb_loss_fwd(const LossArgs& a, cudaStream_t s) { return launch<false>(a, s); }

int debug_check(const DebugCheckArgs& a, cudaStream_t s) {
  if (a.B <= 0 || a.G <= 0 || !a.Y || !a.m || !a.theta || !a.report || a.ld_theta < 0) {
    set_error("debug_check: bad argument"); return DCA_ERR_BAD_ARG;
  }
  // 256 genes per block; the rows strided over enough blocks to give every SM about eight
  const int gx = cdiv(a.G, 256);
  const int gy = std::max(1, std::min(a.B, std::min(65535, 8 * sm_count_cached() / gx + 1)));
  debug_check_kernel<<<dim3(gx, gy), 256, 0, s>>>(a.Y, a.ldy, a.rows, a.sf, a.m, a.ldm, a.theta, a.ld_theta, a.B, a.G,
                                                  reinterpret_cast<DbgReport*>(a.report));
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

void debug_report_decode(const unsigned long long raw[6], int64_t count[3], int32_t first_row[3], int32_t first_gene[3]) {
  for (int k = 0; k < 3; ++k) {
    count[k] = (int64_t)raw[k];
    const unsigned long long key = ~raw[3 + k];                      // raw 0: nothing flagged
    first_row[k] = raw[3 + k] ? (int32_t)(key >> 32) : -1;
    first_gene[k] = raw[3 + k] ? (int32_t)(key & 0xffffffffu) : -1;
  }
}

int heads_loss_tc(const HeadsLossArgs& a, cudaStream_t s) {
  using namespace hl;
  const int B = a.B, G = a.G;
  auto al = [](const void* q, uintptr_t n) { return (reinterpret_cast<uintptr_t>(q) & (n - 1)) == 0; };
  if (B <= 0 || G <= 0 || G % 8 != 0 || a.ldy % 4 != 0 || !al(a.Y, 16) || a.ldz % 4 != 0 || a.ldz < G ||
      !al(a.dz[0], 8) || !al(a.dz[1], 8) || !al(a.dz[2], 8)) {
    set_error("heads_loss_tc: need G %% 8 == 0, a 16-byte aligned Y with ldy %% 4 == 0 and 8-byte aligned dZ with ldz %% 4 == 0 (>= G)");
    return DCA_ERR_BAD_ARG;
  }
  const float* lf_dev = log_fact_table_device();
  if (!lf_dev) return DCA_ERR_CUDA;
  if (!a.ws || a.ws_bytes < kThetaOff) { set_error("heads_loss_tc: workspace too small"); return DCA_ERR_BAD_ARG; }   // loss partials + counter
  CUtensorMap mh, mw[3];
  DCA_TRY(tc::make_tensor_map_2d(&mh, a.H3, 2, 1, (uint64_t)B, 64, 64, 64, 64, 1));
  for (int i = 0; i < 3; ++i) DCA_TRY(tc::make_tensor_map_2d(&mw[i], a.W[i], 2, 1, 64, (uint64_t)G, (uint64_t)G, 64, 64, 1));
  Params p;
  for (int i = 0; i < 3; ++i) { p.bias[i] = a.bias[i]; p.dz[i] = a.dz[i]; }
  p.Y = a.Y; p.ldy = a.ldy; p.rows = a.rows; p.sf = a.sf; p.B = B; p.G = G; p.ldz = a.ldz;
  p.nblk = cdiv(B, 64);
  const long long units = (long long)cdiv(G, 128) * p.nblk;         // 2^31 units would be over 2^44 counts
  if (units > INT_MAX) { set_error("heads_loss_tc: %lld (gene tile, cell block) units, over 2^31 - 1", units); return DCA_ERR_BAD_ARG; }
  p.units = (int)units;
  p.ridge = a.ridge; p.inv_n = a.inv_n;
  p.loss_partial = reinterpret_cast<double*>(a.ws); p.lf = lf_dev;
  FoldArgs fa{reinterpret_cast<unsigned*>(reinterpret_cast<char*>(a.ws) + sizeof(double) * (size_t)kMaxBlocks), a.loss_sum,
              a.fin_penalty, a.fin_loss_slot, a.fin_epoch_acc, a.fin_batch};
  if (!a.counter_ready) DCA_CUDA_OK(cudaMemsetAsync(fa.counter, 0, sizeof(unsigned), s));
  static bool attr = false;
  if (!attr) { DCA_CUDA_OK(cudaFuncSetAttribute(heads_loss_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes)); attr = true; }
  // one CTA per SM, each a contiguous range of the (gene tile, cell block) units; the grid follows the device, not the
  // caller's SM budget, so that the loss is summed in the same order whatever the budget
  const int grid = (int)std::min<long long>(p.units, sm_count_cached());
  heads_loss_kernel<<<grid, kCtaThreads, kSmemBytes, s>>>(mh, mw[0], mw[1], mw[2], p, fa);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

}  // namespace dca

// ------------------------------------------------------------------------------------ C ABI
using namespace dca;

extern "C" int dca_set_tunable(const char* name, int64_t value) {
  if (!name) { set_error("dca_set_tunable: null name"); return DCA_ERR_BAD_ARG; }
  const std::string n(name);
  if (n == "loss_target_blocks" && value >= 0 && value <= kMaxBlocks) g_target_blocks = (int)value;
  else if (n == "fused_heads" && (value == 0 || value == 1)) g_fused_heads_default = (int)value;
  else if (n == "gg_profile" && (value == 0 || value == 1)) tc::g_gg_profile = (int)value;
  else if (n == "head_bwd_banded" && (value == 0 || value == 1)) tc::g_head_bwd_banded = (int)value;
  else if (n == "head_bwd_stagger" && value >= 0 && value <= 100000) tc::g_head_bwd_stagger = (int)value;
  else { set_error("dca_set_tunable: unknown name or value out of range (%s = %lld)", name, (long long)value); return DCA_ERR_BAD_ARG; }
  return DCA_OK;
}

extern "C" int dca_zinb_loss_workspace_bytes(int32_t batch, int32_t genes, size_t* bytes) {
  if (!bytes || batch <= 0 || genes <= 0) { set_error("dca_zinb_loss_workspace_bytes: bad argument"); return DCA_ERR_BAD_ARG; }
  *bytes = loss_workspace_bytes(batch, genes);
  return DCA_OK;
}

extern "C" int dca_zinb_loss_fwd_bwd(const float* Y, int64_t ldy, const int32_t* rows, const float* sf,
                                     const float* m, const float* d, const float* pi, int64_t ld,
                                     int32_t batch, int32_t genes, int32_t ae_type, float ridge, float inv_n,
                                     void* dzm, void* dzd, void* dzp, int32_t grad_dtype, float* dtheta,
                                     double* loss_sum, void* workspace, size_t workspace_bytes, void* stream) {
  if (ae_type < 0 || ae_type > 3) { set_error("dca_zinb_loss_fwd_bwd: unknown ae_type %d", ae_type); return DCA_ERR_BAD_ARG; }
  LossArgs a{Y, ldy, rows, sf, m, d, pi, ld, batch, genes, ae_type, ridge, inv_n, dzm, dzd, dzp,
             grad_dtype == DCA_BF16 ? 1 : 0, dtheta, loss_sum, workspace, workspace_bytes};
  return zinb_loss_fwd_bwd(a, (cudaStream_t)stream);
}

extern "C" int dca_tc_heads_loss(const void* Hb, int32_t batch, const void* Wk, const float* bias, int32_t genes,
                                 const float* Y, int64_t ldy, const int32_t* rows, const float* sf, float ridge, float inv_n,
                                 void* dzm, void* dzd, void* dzp, int64_t ldz, double* loss_sum, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  if (!Hb || !Wk || !bias || !Y || !dzm || !dzd || !dzp || !loss_sum || batch <= 0 || genes <= 0) {
    set_error("dca_tc_heads_loss: bad argument"); return DCA_ERR_BAD_ARG;
  }
  HeadsLossArgs a{};
  a.H3 = (const __nv_bfloat16*)Hb; a.B = batch; a.G = genes;
  for (int i = 0; i < 3; ++i) { a.W[i] = (const __nv_bfloat16*)Wk + (size_t)i * 64 * genes; a.bias[i] = bias + (size_t)i * genes; }
  a.Y = Y; a.ldy = ldy; a.rows = rows; a.sf = sf; a.ridge = ridge; a.inv_n = inv_n;
  a.dz[0] = (__nv_bfloat16*)dzm; a.dz[1] = (__nv_bfloat16*)dzd; a.dz[2] = (__nv_bfloat16*)dzp; a.ldz = ldz;
  a.loss_sum = loss_sum; a.ws = workspace; a.ws_bytes = workspace_bytes;
  return heads_loss_tc(a, (cudaStream_t)stream);
}

extern "C" int dca_zinb_loss_fwd(const float* Y, int64_t ldy, const int32_t* rows, const float* sf,
                                 const float* m, const float* d, const float* pi, int64_t ld, int32_t batch,
                                 int32_t genes, int32_t ae_type, float ridge, double* loss_sum, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  if (ae_type < 0 || ae_type > 3) { set_error("dca_zinb_loss_fwd: unknown ae_type %d", ae_type); return DCA_ERR_BAD_ARG; }
  LossArgs a{Y, ldy, rows, sf, m, d, pi, ld, batch, genes, ae_type, ridge, 1.0f, nullptr, nullptr, nullptr,
             0, nullptr, loss_sum, workspace, workspace_bytes};
  return zinb_loss_fwd(a, (cudaStream_t)stream);
}

extern "C" int dca_debug_check(const float* Y, int64_t ldy, const int32_t* rows, const float* sf, const float* m, int64_t ldm,
                               const float* theta, int64_t ld_theta, int32_t batch, int32_t genes, void* workspace,
                               dca_debug_report* out, void* stream) {
  if (!out || out->struct_bytes != (int32_t)sizeof(dca_debug_report)) {
    set_error("dca_debug_check: NULL or unversioned dca_debug_report (struct_bytes must be %d)", (int)sizeof(dca_debug_report));
    return DCA_ERR_BAD_ARG;
  }
  if (!workspace) { set_error("dca_debug_check: NULL workspace"); return DCA_ERR_BAD_ARG; }
  cudaStream_t s = (cudaStream_t)stream;
  DCA_CUDA_OK(cudaMemsetAsync(workspace, 0, kDebugReportBytes, s));
  DCA_TRY(debug_check(DebugCheckArgs{Y, ldy, rows, sf, m, ldm, theta, ld_theta, batch, genes, workspace}, s));
  unsigned long long raw[6];
  DCA_CUDA_OK(cudaMemcpyAsync(raw, workspace, sizeof(raw), cudaMemcpyDeviceToHost, s));
  DCA_CUDA_OK(cudaStreamSynchronize(s));
  debug_report_decode(raw, out->count, out->first_row, out->first_gene);
  return DCA_OK;
}

// Host mirror of the per-element device math (same source, compiled for the CPU) so the
// arithmetic can be unit-tested against the oracle on a machine without a GPU.
extern "C" int dca_zinb_elem_host(int32_t ae_type, float y, float m, float sf, float d, float pi, float ridge,
                                  float out[4]) {
  zmath::Elem e;
  static float lf[zmath::kLogFactN];
  static bool lf_ready = false;
  if (!lf_ready) { zmath::fill_log_fact(lf); lf_ready = true; }
  using P = zmath::PreciseOps;
  if (ae_type & 0x200) {
    // the formulation of zinb_loss_bwd_ring_kernel: f32x2 zero branch / raw NB derivatives + shared finishing factors
    const int base = ae_type & 0xff;
    if (base != DCA_AE_ZINB_CONDDISP && base != DCA_AE_ZINB) { set_error("dca_zinb_elem_host: kernel variant needs a ZINB type"); return DCA_ERR_BAD_ARG; }
    const bool cd = base == DCA_AE_ZINB_CONDDISP;
    const float2 m2 = zmath::splat(m), d2 = zmath::splat(d), p2 = zmath::splat(pi), mu2 = zmath::mul2(m2, zmath::splat(sf));
    const zmath::Fin2 f = cd ? zmath::finish_factors_pair<P, true>(m2, d2, p2, 1.0f) : zmath::finish_factors_pair<P, false>(m2, d2, p2, 1.0f);
    float loss, gmu, dth, dpi;
    if (y < 1e-8f) {
      const zmath::Raw2 z = zmath::zinb_zero_pair<P>(mu2, d2, p2);
      loss = -zmath::kLn2 * z.lgD.y; gmu = z.gmu.y; dth = z.dth.y; dpi = z.dpi.y;
    } else {
      const zmath::Raw1 r = zmath::zinb_nb_raw<P>(y, mu2.x, d, pi, lf);
      loss = r.loss; gmu = r.gmu; dth = r.dth; dpi = r.dpi;
    }
    if (ridge != 0.f) { loss += ridge * pi * pi; dpi = fmaf(2.0f * ridge, pi, dpi); }
    out[0] = loss; out[1] = gmu * f.fm.y; out[2] = dth * f.fd.y; out[3] = dpi * f.fp.y;
    return DCA_OK;
  }
  switch (ae_type) {
    case DCA_AE_ZINB_CONDDISP: e = zmath::zinb_elem<P, true, true>(y, m, sf, d, pi, ridge, lf); break;
    case DCA_AE_ZINB: e = zmath::zinb_elem<P, true, false>(y, m, sf, d, pi, ridge, lf); break;
    case DCA_AE_NB_CONDDISP: e = zmath::zinb_elem<P, false, true>(y, m, sf, d, pi, ridge, lf); break;
    case DCA_AE_NB: e = zmath::zinb_elem<P, false, false>(y, m, sf, d, pi, ridge, lf); break;
    default: set_error("dca_zinb_elem_host: unknown ae_type %d", ae_type); return DCA_ERR_BAD_ARG;
  }
  out[0] = e.loss; out[1] = e.gm; out[2] = e.gd; out[3] = e.gp;
  return DCA_OK;
}
