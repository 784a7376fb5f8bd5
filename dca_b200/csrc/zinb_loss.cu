// K3: ZINB / NB negative log-likelihood, forward + backward in ONE pass over the B x G head
// outputs (replaces dca/loss.py:72-156 and the TF autodiff of it; see zinb_math.cuh).
//
// Layout: every tensor is row-major cells x genes.  A thread owns 4 consecutive genes (one
// 128-bit load per tensor per row) and walks a strip of rows, so a warp touches 512 contiguous
// bytes per tensor per row and the per-gene reduction needed by the constant-dispersion
// variants stays in registers.  HBM traffic per element: y 4 B + nh*4 B in, nh*(4|2) B out.
// The loss scalar is reduced thread -> warp shuffle -> shared memory -> one double per block,
// and a second tiny kernel folds the block partials (deterministic, no float atomics).
#include "dca_internal.cuh"
#include <string>
#include "zinb_math.cuh"
#include "tc_common.cuh"
#include <cstdlib>

namespace dca {
namespace tc { extern int g_gg_profile; }

namespace {

constexpr int kThreads = 256;
constexpr int kVec = 4;
constexpr int kColsPerBlock = kThreads * kVec;   // 1024 genes per block
constexpr int kMaxBlocks = 65536;                // bound of the per-block loss-partial buffer

// Launch tunables (dca_set_tunable; defaults from a launch-parameter sweep, tests/diag_loss_sweep.py)
struct LossTune { int target_blocks; unsigned producer_sleep_ns, consumer_sleep_ns; int branch_free; int ring; };
LossTune g_tune = {0 /* auto */, 0u, 0u, 1 /* branch-free zero branch (the faster variant in the sweep) */,
                   1 /* per-warp rings + f32x2 arithmetic (zinb_loss_bwd_ring_kernel); 0 = block-wide ring (staged kernel) */};

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
  const int target = g_tune.target_blocks > 0 ? g_tune.target_blocks
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
                 GT* dzm, GT* dzd, GT* dzp, float* __restrict__ dth_partial,
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
    if (BWD && !COND_DISP) {
#pragma unroll
      for (int j = 0; j < VEC; ++j)
        if (col0 + j < G) atomicAdd(dth_partial + col0 + j, tacc[j]);
    }
  }
  const double tot = block_reduce_sum(lsum, red);
  if (threadIdx.x == 0) loss_partial[blockIdx.y * gridDim.x + blockIdx.x] = tot;
}

// ZINB models, 128-bit path, backward: the expensive NB branch (y > 0, ~10-20 % of a scRNA-seq
// matrix) is warp-compacted through shared memory.  Every lane evaluates the cheap zero branch
// for its own zero counts; the non-zero elements of the warp's 128-gene strip are queued in
// shared memory (16 B items), evaluated densely (item i by lane i mod 32) and handed back.
// Without this the NB branch runs once per vector slot with ~17 % of the lanes active.
template <bool COND_DISP, typename GT>
__global__ void __launch_bounds__(kThreads, 4)
zinb_loss_bwd_compact_kernel(const float* __restrict__ Y, int64_t ldy, const int32_t* __restrict__ rows,
                             const float* __restrict__ sf, const float* m, const float* d, const float* pi,
                             int64_t ld, int B, int G, float ridge, float inv_n, int rows_per_block,
                             GT* dzm, GT* dzd, GT* dzp, float* __restrict__ dth_acc,
                             double* __restrict__ loss_partial, const float* __restrict__ lf_global) {
  __shared__ double red[8];
  __shared__ float lf[zmath::kLogFactN];
  __shared__ float4 items[kThreads / 32][32 * kVec];                 // 16 KB
  if (threadIdx.x < zmath::kLogFactN) lf[threadIdx.x] = lf_global[threadIdx.x];
  __syncthreads();
  using Ops = zmath::FastOps;
  constexpr unsigned kFull = 0xffffffffu;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4* q = items[warp];
  const int col0 = (blockIdx.x * kThreads + threadIdx.x) * kVec;
  const bool active = col0 < G;                                       // G % 4 == 0 on this path
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(B, r0 + rows_per_block);
  float lsum = 0.f;
  float tacc[kVec] = {0.f, 0.f, 0.f, 0.f};
  float thg[kVec] = {1.f, 1.f, 1.f, 1.f};
  if (!COND_DISP && active) {
#pragma unroll
    for (int j = 0; j < kVec; ++j) thg[j] = d[col0 + j];
  }
  RowVals<kVec> cur, nxt;
  if (active) load_row<true, COND_DISP, kVec>(cur, Y, ldy, rows, sf, m, d, pi, ld, r0, col0);
  for (int r = r0; r < r1; ++r) {
    if (active && r + 1 < r1) load_row<true, COND_DISP, kVec>(nxt, Y, ldy, rows, sf, m, d, pi, ld, r + 1, col0);
    // ---- queue the non-zero counts of this warp's strip (ballot compaction: items ordered by j, then lane)
    unsigned bal[kVec];
    int nz = 0;
#pragma unroll
    for (int j = 0; j < kVec; ++j) {
      const bool is_nz = active && !(cur.y[j] < 1e-8f);                                  // loss.py:138
      bal[j] = __ballot_sync(kFull, is_nz);
      nz |= is_nz ? (1 << j) : 0;
    }
    const unsigned lt = (1u << lane) - 1u;
    int pos[kVec];
    int base = 0;
#pragma unroll
    for (int j = 0; j < kVec; ++j) { pos[j] = base + __popc(bal[j] & lt); base += __popc(bal[j]); }
    const int total = base;
    const float row_sf = __shfl_sync(kFull, active ? cur.sf : 1.0f, 0);                  // lane 0 of an active warp is active
#pragma unroll
    for (int j = 0; j < kVec; ++j)
      if (nz & (1 << j)) q[pos[j]] = make_float4(cur.y[j], cur.m[j], COND_DISP ? cur.d[j] : thg[j], cur.p[j]);
    __syncwarp();
    // ---- zero branch for my own zero counts (branch-free per element)
    float gm[kVec], gd[kVec], gp[kVec];
#pragma unroll
    for (int j = 0; j < kVec; ++j) {
      gm[j] = gd[j] = gp[j] = 0.f;
      if (active && !(nz & (1 << j))) {
        const zmath::Elem e = zmath::zinb_elem_zero<Ops, COND_DISP>(cur.m[j], cur.sf, COND_DISP ? cur.d[j] : thg[j], cur.p[j], ridge);
        lsum += e.loss; gm[j] = e.gm; gd[j] = e.gd; gp[j] = e.gp;
      }
    }
    // ---- dense NB pass over the queue
    for (int i = lane; i < total; i += 32) {
      const float4 it = q[i];
      const zmath::Elem e = zmath::zinb_elem_nb<Ops, true, COND_DISP>(it.x, it.y, row_sf, it.z, it.w, ridge, lf);
      q[i] = make_float4(e.loss, e.gm, e.gd, e.gp);
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < kVec; ++j)
      if (nz & (1 << j)) { const float4 e = q[pos[j]]; lsum += e.x; gm[j] = e.y; gd[j] = e.z; gp[j] = e.w; }
    __syncwarp();
    if (active) {
      const int64_t off = (int64_t)r * ld + col0;
      if (!COND_DISP) {
#pragma unroll
        for (int j = 0; j < kVec; ++j) tacc[j] += gd[j];
      }
      st4(dzm + off, gm[0] * inv_n, gm[1] * inv_n, gm[2] * inv_n, gm[3] * inv_n);
      if (COND_DISP) st4(dzd + off, gd[0] * inv_n, gd[1] * inv_n, gd[2] * inv_n, gd[3] * inv_n);
      st4(dzp + off, gp[0] * inv_n, gp[1] * inv_n, gp[2] * inv_n, gp[3] * inv_n);
    }
    cur = nxt;
  }
  if (!COND_DISP && active) {
#pragma unroll
    for (int j = 0; j < kVec; ++j) atomicAdd(dth_acc + col0 + j, tacc[j]);
  }
  const double tot = block_reduce_sum(lsum, red);
  if (threadIdx.x == 0) loss_partial[blockIdx.y * gridDim.x + blockIdx.x] = tot;
}

// Same arithmetic, operands STAGED THROUGH SHARED MEMORY: one producer warp streams the block's rows with bulk
// async copies (cp.async.bulk global->shared, one 16-byte-aligned row segment per tensor, completion on an
// mbarrier) into a 3-deep ring, eight consumer warps read their 128-bit vectors from the ring.  The gather of
// the count rows (rows[]) is free -- the producer simply points the copy at row rows[r] -- and the consumers
// carry no address arithmetic or load latency, only the math, the warp compaction and the coalesced stores.
struct FoldArgs {
  unsigned* counter; double* loss_sum; const double* penalty; float* loss_slot; double* epoch_acc; int batch;
};

constexpr int kStageRows = 3;
constexpr int kMaxRowsPerBlock = 256;
constexpr int kStagedThreads = kThreads + 32;      // 8 consumer warps + 1 producer warp

template <bool COND_DISP, typename GT, bool BF>
__global__ void __launch_bounds__(kStagedThreads, 3)
zinb_loss_bwd_staged_kernel(const float* __restrict__ Y, int64_t ldy, const int32_t* __restrict__ rows,
                            const float* __restrict__ sf, const float* m, const float* d, const float* pi,
                            int64_t ld, int B, int G, float ridge, float inv_n, int rows_per_block,
                            GT* dzm, GT* dzd, GT* dzp, float* __restrict__ dth_acc,
                            double* __restrict__ loss_partial, const float* __restrict__ lf_global, const FoldArgs fa,
                            const unsigned producer_sleep_ns, const unsigned consumer_sleep_ns) {
  extern __shared__ __align__(128) unsigned char smem_loss[];
  constexpr int kArrays = COND_DISP ? 4 : 3;                           // y, m, [d], pi
  constexpr uint32_t kArrBytes = kColsPerBlock * 4;                    // one row segment of one tensor
  constexpr uint32_t kStageBytes = kArrays * kArrBytes;
  float4* items = reinterpret_cast<float4*>(smem_loss + kStageRows * kStageBytes);   // [8 warps][128]
  __shared__ double red[8];
  __shared__ float lf[zmath::kLogFactN];
  __shared__ float s_sf[kMaxRowsPerBlock];
  __shared__ int s_row[kMaxRowsPerBlock];
  __shared__ uint64_t full_bar[kStageRows], empty_bar[kStageRows];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = blockIdx.x * kColsPerBlock;
  const int ncols = min(kColsPerBlock, G - c0);                        // multiple of 4 on this path
  const int r0 = blockIdx.y * rows_per_block;
  const int nrows = min(rows_per_block, B - r0);
  if (threadIdx.x < zmath::kLogFactN) lf[threadIdx.x] = lf_global[threadIdx.x];
  for (int t = threadIdx.x; t < nrows; t += kStagedThreads) {
    const int yr = rows ? rows[r0 + t] : (r0 + t);
    s_row[t] = yr;
    s_sf[t] = sf ? sf[yr] : 1.0f;
  }
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStageRows; ++i) { tc::mbar_init(&full_bar[i], 1); tc::mbar_init(&empty_bar[i], kThreads / 32); }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp == kThreads / 32) {
    // ===================================================== producer
    if (lane == 0) {
      const uint32_t bytes = (uint32_t)ncols * 4u;
      for (int i = 0; i < nrows; ++i) {
        const int st = i % kStageRows; const uint32_t ph = (i / kStageRows) & 1;
        tc::mbar_wait_backoff(&empty_bar[st], ph ^ 1, producer_sleep_ns);
        unsigned char* dst = smem_loss + (size_t)st * kStageBytes;
        tc::mbar_expect_tx(&full_bar[st], bytes * kArrays);
        const int64_t off = (int64_t)(r0 + i) * ld + c0;
        auto bulk = [&](unsigned char* to, const float* from) {
          asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                       ::"r"(tc::smem_u32(to)), "l"(reinterpret_cast<uint64_t>(from)), "r"(bytes), "r"(tc::smem_u32(&full_bar[st])) : "memory");
        };
        bulk(dst, Y + (int64_t)s_row[i] * ldy + c0);
        bulk(dst + kArrBytes, m + off);
        if (COND_DISP) bulk(dst + 2 * kArrBytes, d + off);
        bulk(dst + (kArrays - 1) * kArrBytes, pi + off);
      }
    }
    return;
  }

  // ======================================================= consumers
  using Ops = zmath::FastOps;
  constexpr unsigned kFull = 0xffffffffu;
  float4* q = items + warp * (32 * kVec);
  const int col = threadIdx.x * kVec;                                  // column inside the block tile
  const bool active = col < ncols;
  float lsum = 0.f;
  float tacc[kVec] = {0.f, 0.f, 0.f, 0.f};
  float thg[kVec] = {1.f, 1.f, 1.f, 1.f};
  if (!COND_DISP && active) {
#pragma unroll
    for (int j = 0; j < kVec; ++j) thg[j] = d[c0 + col + j];
  }
  const unsigned lt = (1u << lane) - 1u;
  GT* om = dzm + (int64_t)r0 * ld + c0 + col;
  GT* od = COND_DISP ? dzd + (int64_t)r0 * ld + c0 + col : nullptr;
  GT* op = dzp + (int64_t)r0 * ld + c0 + col;
  for (int i = 0; i < nrows; ++i) {
    const int st = i % kStageRows; const uint32_t ph = (i / kStageRows) & 1;
    const unsigned char* src = smem_loss + (size_t)st * kStageBytes + (size_t)threadIdx.x * 16;
    tc::mbar_wait_backoff(&full_bar[st], ph, consumer_sleep_ns);
    float4 vy = make_float4(0.f, 0.f, 0.f, 0.f), vm = vy, vd = vy, vp = vy;
    if (active) {
      vy = *reinterpret_cast<const float4*>(src);
      vm = *reinterpret_cast<const float4*>(src + kArrBytes);
      if (COND_DISP) vd = *reinterpret_cast<const float4*>(src + 2 * kArrBytes);
      vp = *reinterpret_cast<const float4*>(src + (kArrays - 1) * kArrBytes);
    }
    __syncwarp();
    if (lane == 0) tc::mbar_arrive(&empty_bar[st]);                    // operands are in registers: free the slot
    const float y[kVec] = {vy.x, vy.y, vy.z, vy.w}, mm[kVec] = {vm.x, vm.y, vm.z, vm.w};
    const float dd[kVec] = {COND_DISP ? vd.x : thg[0], COND_DISP ? vd.y : thg[1], COND_DISP ? vd.z : thg[2], COND_DISP ? vd.w : thg[3]};
    const float pp[kVec] = {vp.x, vp.y, vp.z, vp.w};
    const float row_sf = s_sf[i];
    // ---- queue the non-zero counts of this warp's strip (ballot compaction: items ordered by j, then lane)
    unsigned bal[kVec];
    int nz = 0, pos[kVec], base = 0;
#pragma unroll
    for (int j = 0; j < kVec; ++j) {
      const bool is_nz = active && !(y[j] < 1e-8f);                    // loss.py:138
      bal[j] = __ballot_sync(kFull, is_nz);
      nz |= is_nz ? (1 << j) : 0;
    }
#pragma unroll
    for (int j = 0; j < kVec; ++j) { pos[j] = base + __popc(bal[j] & lt); base += __popc(bal[j]); }
    const int total = base;
#pragma unroll
    for (int j = 0; j < kVec; ++j)
      if (nz & (1 << j)) q[pos[j]] = make_float4(y[j], mm[j], dd[j], pp[j]);
    __syncwarp();
    // ---- zero branch for my own zero counts
    float gm[kVec], gd[kVec], gp[kVec];
#pragma unroll
    for (int j = 0; j < kVec; ++j) {
      gm[j] = gd[j] = gp[j] = 0.f;
      if (BF) {   // branch-free: the four independent chains of a thread interleave (zinb_math.cuh)
        const zmath::Elem e = zmath::zinb_elem_zero_bf<Ops, COND_DISP>(mm[j], row_sf, dd[j], pp[j], ridge);
        const bool use = active && !(nz & (1 << j));
        lsum += use ? e.loss : 0.f; gm[j] = use ? e.gm : 0.f; gd[j] = use ? e.gd : 0.f; gp[j] = use ? e.gp : 0.f;
      } else if (active && !(nz & (1 << j))) {
        const zmath::Elem e = zmath::zinb_elem_zero<Ops, COND_DISP>(mm[j], row_sf, dd[j], pp[j], ridge);
        lsum += e.loss; gm[j] = e.gm; gd[j] = e.gd; gp[j] = e.gp;
      }
    }
    // ---- dense NB pass over the queue
    for (int k = lane; k < total; k += 32) {
      const float4 it = q[k];
      const zmath::Elem e = zmath::zinb_elem_nb<Ops, true, COND_DISP>(it.x, it.y, row_sf, it.z, it.w, ridge, lf);
      q[k] = make_float4(e.loss, e.gm, e.gd, e.gp);
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < kVec; ++j)
      if (nz & (1 << j)) { const float4 e = q[pos[j]]; lsum += e.x; gm[j] = e.y; gd[j] = e.z; gp[j] = e.w; }
    __syncwarp();
    if (active) {
      if (!COND_DISP) {
#pragma unroll
        for (int j = 0; j < kVec; ++j) tacc[j] += gd[j];
      }
      st4(om, gm[0] * inv_n, gm[1] * inv_n, gm[2] * inv_n, gm[3] * inv_n);
      if (COND_DISP) st4(od, gd[0] * inv_n, gd[1] * inv_n, gd[2] * inv_n, gd[3] * inv_n);
      st4(op, gp[0] * inv_n, gp[1] * inv_n, gp[2] * inv_n, gp[3] * inv_n);
    }
    om += ld; op += ld;
    if (COND_DISP) od += ld;
  }
  if (!COND_DISP && active) {
#pragma unroll
    for (int j = 0; j < kVec; ++j) atomicAdd(dth_acc + c0 + col + j, tacc[j]);
  }
  // block reduction over the 8 consumer warps (the producer warp has returned: named barrier on 256 threads)
  double dsum = (double)lsum;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dsum += __shfl_xor_sync(kFull, dsum, o);
  if (lane == 0) red[warp] = dsum;
  tc::named_barrier_sync(1, kThreads);
  __shared__ int s_last;
  if (threadIdx.x == 0) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) t += red[w];
    loss_partial[blockIdx.y * gridDim.x + blockIdx.x] = t;
    __threadfence();
    const unsigned nblk = gridDim.x * gridDim.y;
    const unsigned done = atomicAdd(fa.counter, 1u);
    s_last = (done == nblk - 1);
    if (s_last) *fa.counter = 0;                                       // self-resetting
  }
  tc::named_barrier_sync(1, kThreads);
  if (!s_last) return;
  // ---- the last block to finish folds the per-block partials in a FIXED order (deterministic) and finalises
  __threadfence();
  const int n = gridDim.x * gridDim.y;
  double a = 0.0;
  for (int i = threadIdx.x; i < n; i += kThreads) a += __ldcg(loss_partial + i);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(kFull, a, o);
  if (lane == 0) red[warp] = a;
  tc::named_barrier_sync(1, kThreads);
  if (threadIdx.x == 0) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) t += red[w];
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

// ---------------------------------------------------------------------------------------------------------------
// "Ring" kernel (default for ZINB backward on aligned shapes): operands are staged through shared memory by the
// threads themselves -- every thread streams the 16 bytes it owns of each tensor row (4 consecutive genes of y, m,
// [d], pi) with cp.async (LDGSTS, L2-only) into a kRing-deep ring of its own, kRing rows ahead of the arithmetic,
// and reads them back with one 128-bit LDS per tensor.  A thread only ever reads what it copied itself, so the
// pipeline needs no barrier of any kind (cp.async.wait_group orders a thread's own copies), no producer warp and
// no single-lane issue path: in the block-wide bulk-copy ring of zinb_loss_bwd_staged_kernel a warp could run at
// most three rows ahead of the slowest warp of its block (the one that met a large count and took the Stirling
// path), and a fifth of all issued instructions were mbarrier polls of warps waiting for a slot their neighbour
// had not released (3-instruction loops executed 9-13x per row).  The gather of the count
// rows costs one address computation (rows[] cached in shared memory).  The arithmetic runs on f32x2 pairs
// (zinb_math.cuh: zinb_zero_pair / finish_factors_pair), the queued non-zero counts return raw derivatives only
// (zinb_nb_raw) and the activation chain / clip masks / 1/N are applied once per element by its owner.
constexpr int kRing = 3;                                  // rows in flight per thread

__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// IDXQ (tunable loss_ring = 2): the queue of non-zero counts holds one-byte ELEMENT INDICES instead of 16-byte operand
// copies -- the evaluating lane reads y / m / d / pi of the element from the staging slot itself and writes the three raw
// derivatives back in place, the owner re-reads its vector -- which frees 15 KB of shared memory for a fourth ring slot.
template <bool COND_DISP, typename GT, bool IDXQ>
__global__ void __launch_bounds__(kThreads, 3)
zinb_loss_bwd_ring_kernel(const float* __restrict__ Y, int64_t ldy, const int32_t* __restrict__ rows,
                          const float* __restrict__ sf, const float* m, const float* d, const float* pi,
                          int64_t ld, int B, int G, float ridge, float inv_n, int rows_per_block,
                          GT* dzm, GT* dzd, GT* dzp, float* __restrict__ dth_acc,
                          double* __restrict__ loss_partial, const float* __restrict__ lf_global, const FoldArgs fa) {
  extern __shared__ __align__(128) unsigned char smem_ring[];
  constexpr int kWarps = kThreads / 32;
  constexpr int kArrays = COND_DISP ? 4 : 3;                           // y, m, [d], pi
  constexpr uint32_t kSegBytes = kThreads * 16;                        // one block-row segment of one tensor (4 KB)
  constexpr uint32_t kSlotBytes = kArrays * kSegBytes;
  constexpr int RING = IDXQ ? kRing + 1 : kRing;
  float4* items = reinterpret_cast<float4*>(smem_ring + RING * kSlotBytes);            // [8 warps][128] operand copies | indices
  __shared__ double red[kWarps];
  __shared__ float lf[zmath::kLogFactN];
  __shared__ float s_sf[kMaxRowsPerBlock];
  __shared__ int s_row[kMaxRowsPerBlock];
  __shared__ int s_last;

  using Ops = zmath::FastOps;
  using namespace zmath;
  constexpr unsigned kFull = 0xffffffffu;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
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
  const uint32_t ring_end = my + RING * kSlotBytes;
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
    for (int i = 0; i < RING; ++i) {                                   // one group per row, empty groups keep the count fixed
      if (i < nrows) issue_next();
      cp_async_commit();
    }
    float4* q = items + warp * (32 * kVec);
    unsigned char* qb = reinterpret_cast<unsigned char*>(items) + warp * (32 * kVec);
    auto lds32 = [](uint32_t addr) { float v; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory"); return v; };
    auto sts32 = [](uint32_t addr, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory"); };
    float thg[kVec] = {1.f, 1.f, 1.f, 1.f};
    if (!COND_DISP) {
#pragma unroll
      for (int j = 0; j < kVec; ++j) thg[j] = d[c0 + col + j];
    }
    const unsigned lt = (1u << lane) - 1u;
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
      cp_async_wait<RING - 1>();                                       // my copies of row i have landed
      const uint32_t cslot = rslot, wstrip = rslot - (uint32_t)lane * 16u;       // my vector / my warp's strip in this slot
      const float4 vy = lds128(rslot), vm = lds128(rslot + kSegBytes);
      const float4 vd = COND_DISP ? lds128(rslot + 2 * kSegBytes) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float4 vp = lds128(rslot + (kArrays - 1) * kSegBytes);
      rslot += kSlotBytes;
      if (rslot == ring_end) rslot = my;
      const float row_sf = s_sf[i];
      const float y[kVec] = {vy.x, vy.y, vy.z, vy.w};
      const float2 mA = make_float2(vm.x, vm.y), mB = make_float2(vm.z, vm.w);
      const float2 dA = COND_DISP ? make_float2(vd.x, vd.y) : make_float2(thg[0], thg[1]);
      const float2 dB = COND_DISP ? make_float2(vd.z, vd.w) : make_float2(thg[2], thg[3]);
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
        if (isnz[j]) { if (IDXQ) qb[pos[j]] = (unsigned char)(lane * kVec + j); else q[pos[j]] = make_float4(y[j], mu[j], dd[j], pp[j]); }
      __syncwarp();
      if (!IDXQ) {
        // the operands of row i have been consumed (they fed the ballots / the queue): refill my slot with row i + kRing
        if (nxt < nrows) issue_next();
        cp_async_commit();
      }
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
      if (IDXQ) {
        for (int k = lane; k < total; k += 32) {
          const int idx = qb[k];
          const uint32_t e4 = wstrip + (uint32_t)idx * 4u;
          const float th = COND_DISP ? lds32(e4 + 2 * kSegBytes) : __ldg(d + c0 + warp * (32 * kVec) + idx);
          const Raw1 e = zinb_nb_raw<Ops>(lds32(e4), lds32(e4 + kSegBytes) * row_sf, th, lds32(e4 + (kArrays - 1) * kSegBytes), lf);
          lsum_nb += e.loss;
          sts32(e4, e.gmu); sts32(e4 + kSegBytes, e.dth); sts32(e4 + (kArrays - 1) * kSegBytes, e.dpi);   // in place of y, m, pi
        }
        __syncwarp();
        const float4 r0v = lds128(cslot), r1v = lds128(cslot + kSegBytes), r2v = lds128(cslot + (kArrays - 1) * kSegBytes);
        zA.gmu.x = isnz[0] ? r0v.x : zA.gmu.x; zA.dth.x = isnz[0] ? r1v.x : zA.dth.x; zA.dpi.x = isnz[0] ? r2v.x : zA.dpi.x;
        zA.gmu.y = isnz[1] ? r0v.y : zA.gmu.y; zA.dth.y = isnz[1] ? r1v.y : zA.dth.y; zA.dpi.y = isnz[1] ? r2v.y : zA.dpi.y;
        zB.gmu.x = isnz[2] ? r0v.z : zB.gmu.x; zB.dth.x = isnz[2] ? r1v.z : zB.dth.x; zB.dpi.x = isnz[2] ? r2v.z : zB.dpi.x;
        zB.gmu.y = isnz[3] ? r0v.w : zB.gmu.y; zB.dth.y = isnz[3] ? r1v.w : zB.dth.y; zB.dpi.y = isnz[3] ? r2v.w : zB.dpi.y;
        __syncwarp();
        // the slot has been read back by its owners: refill it with row i + RING
        if (nxt < nrows) issue_next();
        cp_async_commit();
      } else {
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
      }
      if (ridge != 0.f) {                                              // loss.py:139-140 (uniform; ridge defaults to 0)
        if (active) lsum_r += ridge * (pA.x * pA.x + pA.y * pA.y + pB.x * pB.x + pB.y * pB.y);
        zA.dpi = fma2(splat(2.0f * ridge), pA, zA.dpi); zB.dpi = fma2(splat(2.0f * ridge), pB, zB.dpi);
      }
      if (active) {
        if (!COND_DISP) { tacc[0] += zA.dth.x; tacc[1] += zA.dth.y; tacc[2] += zB.dth.x; tacc[3] += zB.dth.y; }
        const float2 gmA = mul2(zA.gmu, fA.fm), gmB = mul2(zB.gmu, fB.fm);
        const float2 gpA = mul2(zA.dpi, fA.fp), gpB = mul2(zB.dpi, fB.fp);
        st4(om, gmA.x, gmA.y, gmB.x, gmB.y);
        if (COND_DISP) {
          const float2 gdA = mul2(zA.dth, fA.fd), gdB = mul2(zB.dth, fB.fd);
          st4(od, gdA.x, gdA.y, gdB.x, gdB.y);
        }
        st4(op, gpA.x, gpA.y, gpB.x, gpB.y);
      }
      om += ld; op += ld;
      if (COND_DISP) od += ld;
    }
    if (!COND_DISP && active) {
#pragma unroll
      for (int j = 0; j < kVec; ++j) atomicAdd(dth_acc + c0 + col + j, tacc[j]);
    }
  }
  // ---- block reduction, then the last block to finish folds the per-block partials in a FIXED order
  double dsum = (double)lsum_nb + (double)lsum_r - (double)kLn2 * (double)lsum_lg;       // -log D = -ln2 * lg2 D
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
    s_last = (done == nblk - 1);
    if (s_last) *fa.counter = 0;                                       // self-resetting
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const int n = gridDim.x * gridDim.y;
  double a = 0.0;
  for (int i = threadIdx.x; i < n; i += kThreads) a += __ldcg(loss_partial + i);
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
  const size_t need = loss_workspace_bytes(a.B, a.G);
  if (!a.ws || a.ws_bytes < need) { set_error("zinb_loss: workspace too small (%zu < %zu)", a.ws_bytes, need); return DCA_ERR_BAD_ARG; }
  double* lpart = reinterpret_cast<double*>(a.ws);
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  bool vec = (a.G % 4 == 0) && (a.ld % 4 == 0) && (a.ldy % 4 == 0) && al16(a.Y) && al16(a.m) && (!cond || al16(a.d)) &&
             (!has_pi || al16(a.pi));
  if (BWD) vec = vec && al16(a.dzm) && (!cond || al16(a.dzd)) && (!has_pi || al16(a.dzp));
  const Plan p = make_plan(a.B, a.G, vec ? kColsPerBlock : kThreads);
  dim3 grid(p.col_blocks, p.row_chunks), block(kThreads);
  float* tpart = a.dtheta;                                            // const-disp: accumulated with atomics
  if (BWD && !cond) DCA_CUDA_OK(cudaMemsetAsync(a.dtheta, 0, sizeof(float) * (size_t)a.G, s));

  static const bool use_compact = [] { const char* e = getenv("DCA_LOSS_KERNEL"); return e && e[0] == 'c'; }();
  const Plan ps = make_plan(a.B, a.G, kColsPerBlock, kMaxRowsPerBlock);
  const bool staged_ok = BWD && vec && has_pi && !use_compact && (long long)ps.row_chunks * ps.col_blocks <= kMaxBlocks &&
                         ps.row_chunks <= 65535;
  if (staged_ok) {
    grid = dim3(ps.col_blocks, ps.row_chunks);
    FoldArgs fa{reinterpret_cast<unsigned*>(reinterpret_cast<char*>(a.ws) + sizeof(double) * (size_t)kMaxBlocks), a.loss_sum,
                a.fin_penalty, a.fin_loss_slot, a.fin_epoch_acc, a.fin_batch};
    if (!a.counter_ready) DCA_CUDA_OK(cudaMemsetAsync(fa.counter, 0, sizeof(unsigned), s));
#define DCA_RING2(CD, GT, IQ)                                                                                     \
  do {                                                                                                             \
    constexpr size_t sm = IQ ? (size_t)(kRing + 1) * (CD ? 4 : 3) * kColsPerBlock * 4 + (size_t)(kThreads / 32) * 32 * kVec     \
                             : (size_t)kRing * (CD ? 4 : 3) * kColsPerBlock * 4 + (size_t)(kThreads / 32) * 32 * kVec * 16; \
    static bool attr = false;                                                                                      \
    if (!attr) { DCA_CUDA_OK(cudaFuncSetAttribute(zinb_loss_bwd_ring_kernel<CD, GT, IQ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm)); attr = true; } \
    zinb_loss_bwd_ring_kernel<CD, GT, IQ><<<grid, kThreads, sm, s>>>(a.Y, a.ldy, a.rows, a.sf, a.m, a.d, a.pi, a.ld, a.B, a.G, a.ridge, \
        a.inv_n, ps.rows_per_block, (GT*)a.dzm, (GT*)a.dzd, (GT*)a.dzp, tpart, lpart, lf_dev, fa);                  \
  } while (0)
#define DCA_RING(CD, GT) do { if (g_tune.ring == 2) DCA_RING2(CD, GT, true); else DCA_RING2(CD, GT, false); } while (0)
    if (g_tune.ring) {
      if (a.grad_bf16) { if (cond) DCA_RING(true, __nv_bfloat16); else DCA_RING(false, __nv_bfloat16); }
      else             { if (cond) DCA_RING(true, float); else DCA_RING(false, float); }
      DCA_LAUNCH_CHECK();
      return DCA_OK;                                                    // the fold is done by the last block
    }
#undef DCA_RING
#undef DCA_RING2
#define DCA_STAGED2(CD, GT, BFV)                                                                                   \
  do {                                                                                                             \
    constexpr size_t sm = (size_t)kStageRows * (CD ? 4 : 3) * kColsPerBlock * 4 + (size_t)(kThreads / 32) * 32 * kVec * 16; \
    static bool attr = false;                                                                                      \
    if (!attr) { DCA_CUDA_OK(cudaFuncSetAttribute(zinb_loss_bwd_staged_kernel<CD, GT, BFV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm)); attr = true; } \
    zinb_loss_bwd_staged_kernel<CD, GT, BFV><<<grid, kStagedThreads, sm, s>>>(a.Y, a.ldy, a.rows, a.sf, a.m, a.d, a.pi, a.ld, a.B, \
        a.G, a.ridge, a.inv_n, ps.rows_per_block, (GT*)a.dzm, (GT*)a.dzd, (GT*)a.dzp, tpart, lpart, lf_dev, fa,     \
        g_tune.producer_sleep_ns, g_tune.consumer_sleep_ns);                                                       \
  } while (0)
#define DCA_STAGED(CD, GT) do { if (g_tune.branch_free) DCA_STAGED2(CD, GT, true); else DCA_STAGED2(CD, GT, false); } while (0)
    if (a.grad_bf16) { if (cond) DCA_STAGED(true, __nv_bfloat16); else DCA_STAGED(false, __nv_bfloat16); }
    else             { if (cond) DCA_STAGED(true, float); else DCA_STAGED(false, float); }
#undef DCA_STAGED2
#undef DCA_STAGED
    DCA_LAUNCH_CHECK();
    return DCA_OK;                                                      // the fold is done by the last block
  } else if (BWD && vec && has_pi) {
#define DCA_COMPACT(CD, GT)                                                                                   \
  zinb_loss_bwd_compact_kernel<CD, GT><<<grid, block, 0, s>>>(a.Y, a.ldy, a.rows, a.sf, a.m, a.d, a.pi, a.ld, a.B, a.G, \
                                                              a.ridge, a.inv_n, p.rows_per_block, (GT*)a.dzm,  \
                                                              (GT*)a.dzd, (GT*)a.dzp, tpart, lpart, lf_dev)
    if (a.grad_bf16) { if (cond) DCA_COMPACT(true, __nv_bfloat16); else DCA_COMPACT(false, __nv_bfloat16); }
    else             { if (cond) DCA_COMPACT(true, float); else DCA_COMPACT(false, float); }
#undef DCA_COMPACT
  } else {
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
  }
  DCA_LAUNCH_CHECK();
  fold_partials_kernel<<<1, 256, 0, s>>>(lpart, (int)(grid.x * grid.y), a.loss_sum, BWD ? 0 : 1, a.fin_penalty, a.inv_n,
                                         a.fin_batch, BWD ? a.fin_loss_slot : nullptr, a.fin_epoch_acc);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

}  // namespace

const float* loss_log_fact_table() { return log_fact_table_device(); }
int g_fused_heads_default = 0;            // 1: engines created from now on use the fused head/loss/backward kernel

size_t loss_workspace_bytes(int B, int G) {
  (void)B; (void)G;
  return sizeof(double) * (size_t)kMaxBlocks + 256;
}

int zinb_loss_fwd_bwd(const LossArgs& a, cudaStream_t s) { return launch<true>(a, s); }
int zinb_loss_fwd(const LossArgs& a, cudaStream_t s) { return launch<false>(a, s); }

}  // namespace dca

// ------------------------------------------------------------------------------------ C ABI
using namespace dca;

extern "C" int dca_set_tunable(const char* name, int64_t value) {
  if (!name) { set_error("dca_set_tunable: null name"); return DCA_ERR_BAD_ARG; }
  const std::string n(name);
  if (n == "loss_target_blocks" && value >= 0 && value <= kMaxBlocks) g_tune.target_blocks = (int)value;
  else if (n == "loss_producer_sleep_ns" && value >= 0 && value <= 100000) g_tune.producer_sleep_ns = (unsigned)value;
  else if (n == "loss_consumer_sleep_ns" && value >= 0 && value <= 100000) g_tune.consumer_sleep_ns = (unsigned)value;
  else if (n == "fused_heads" && (value == 0 || value == 1)) g_fused_heads_default = (int)value;
  else if (n == "loss_branch_free" && (value == 0 || value == 1)) g_tune.branch_free = (int)value;
  else if (n == "loss_ring" && value >= 0 && value <= 2) g_tune.ring = (int)value;
  else if (n == "gg_profile" && (value == 0 || value == 1)) tc::g_gg_profile = (int)value;
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

extern "C" int dca_zinb_loss_fwd(const float* Y, int64_t ldy, const int32_t* rows, const float* sf,
                                 const float* m, const float* d, const float* pi, int64_t ld, int32_t batch,
                                 int32_t genes, int32_t ae_type, float ridge, double* loss_sum, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  if (ae_type < 0 || ae_type > 3) { set_error("dca_zinb_loss_fwd: unknown ae_type %d", ae_type); return DCA_ERR_BAD_ARG; }
  LossArgs a{Y, ldy, rows, sf, m, d, pi, ld, batch, genes, ae_type, ridge, 1.0f, nullptr, nullptr, nullptr,
             0, nullptr, loss_sum, workspace, workspace_bytes};
  return zinb_loss_fwd(a, (cudaStream_t)stream);
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
  if (ae_type & 0x100) {
    // the formulations the staged / fused kernels run: branch-free zero branch, NB branch evaluated from mu by a
    // different lane than the element's owner (which then applies the MeanAct clip mask)
    const int base = ae_type & 0xff;
    if (base != DCA_AE_ZINB_CONDDISP && base != DCA_AE_ZINB) { set_error("dca_zinb_elem_host: kernel variant needs a ZINB type"); return DCA_ERR_BAD_ARG; }
    if (y < 1e-8f) {
      e = base == DCA_AE_ZINB_CONDDISP ? zmath::zinb_elem_zero_bf<P, true>(m, sf, d, pi, ridge)
                                       : zmath::zinb_elem_zero_bf<P, false>(m, sf, d, pi, ridge);
    } else if (base == DCA_AE_ZINB_CONDDISP) {
      e = zmath::zinb_elem_nb_mu<P>(y, m * sf, d, pi, ridge, lf);
      if (!(m > 1e-5f && m < 1e6f)) e.gm = 0.f;
    } else {
      e = zmath::zinb_elem<P, true, false>(y, m, sf, d, pi, ridge, lf);
    }
    out[0] = e.loss; out[1] = e.gm; out[2] = e.gd; out[3] = e.gp;
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
