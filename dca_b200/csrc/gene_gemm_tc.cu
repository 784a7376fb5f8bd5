// One wgmma kernel for the gene-wide Dense products whose reduction or output dimension is the gene axis (all with a
// 64-wide partner dimension):
//
//   encoder forward  (K1)  A1[B x 64]  += X[B x G] . W1[G x 64]                      (b), W MN-major
//   head backward    (K4)  dH3[B x 64] += sum_h dZ_h . Wh^T                          (b), W K-major
//                          dWh[64 x G] += H3^T . dZ_h,  db_h += colsum(dZ_h)         (a) + column sums
//   encoder backward (K5)  dW1[G x 64] += X^T . dA1                                   (a), 64-gene blocks
//
// K5 has a kernel of its own (gene_gemm_enc_bwd_kernel, below) that spreads 64-gene blocks evenly over the SMs.
//
// "Z" is the cells x genes bf16 operand (X or dZ), brought into shared memory by TMA as 128-cell x 128-gene tiles
// (two SWIZZLE_128B boxes of 64 genes).  K1 and K5 may instead name the batch's cells by row index into a larger X
// (Params::rows): the tile rows are then copied by cp.async into the same shared-memory layout, so the batch is never
// copied out of X.  (b) reads a tile as a K-major A operand (M = 64 cells per warpgroup,
// K = genes), (a) as an MN-major A operand (M = 64 genes per warpgroup, K = cells) against H [cells x 64].  A CTA owns
// one item = (head, range of gene blocks, range of cell blocks) and keeps its fp32 accumulators in registers.
//
// Every output element is summed in a fixed order, so a step computes the same bits on every run:
//   (a) items span ALL cells of their gene blocks: one CTA owns each dW / db element and adds it once (TMA reduce-add
//       of a staging tile, one atomic per db element);
//   (b) items span one cell block and a gene range; each writes its partial [128 x 64] into its own slot of a
//       workspace, and gene_gemm_reduce_kernel adds the slots to the output in slot order.
//
// 256 threads = two warpgroups; thread 0 also issues the TMA loads, kStages - 1 tiles ahead (gathered rows: every
// thread also issues its share of the Z copies).
//
// The head backward runs both item kinds in one launch (BANDED; dca_set_tunable("head_bwd_banded", 0) gives the two
// launches of one kind each).  The items are the same as in the two launches, so every sum keeps its order and its bits;
// only their order changes.  A band is (head, (b) gene range): its (a) items (one gene block each, over all cell
// blocks) and its (b) items (one cell block each, over the band's gene blocks) alternate in the item order, so they
// run at about the same time and most tiles of dZ are read from HBM once, the second read hitting L2.
#include "engine.h"
#include "tc_common.cuh"

namespace dca {
namespace tc {
int g_gg_profile = 0;       // dca_set_tunable("gg_profile", 1): phase timeline of the hidden-stack kernels (mid_stack.cu)
int g_head_bwd_banded = 1;  // dca_set_tunable("head_bwd_banded", 0 | 1): head backward as one band-ordered launch
int g_head_bwd_stagger = 1300;  // dca_set_tunable("head_bwd_stagger", SM cycles): its start delay per band position
                                // (tests/diag_head_bwd.py sweep, DESIGN §8)
namespace gg {

constexpr int kThreads = 256;
constexpr uint32_t kZBytes = 128 * 128 * 2;          // 2 boxes x [128 cells x 64 genes] bf16
constexpr uint32_t kWBytes = 64 * 128 * 2;           // 2 boxes x [64 feats x 64 genes] | 1 box [128 genes x 64 feats] bf16
constexpr uint32_t kHBytes = 128 * 64 * 2;           // [128 cells x 64 feats] bf16
constexpr uint32_t kOutBytes = 128 * 64 * 4;         // fp32 staging tile of one flush
constexpr uint32_t kOnesBytes = 16 * 128;            // [16 x 64] bf16 ones, K-major B operand of the column sums
constexpr int kMaxGb = 4;                            // (a): gene blocks per item held in registers
constexpr int kMaxSlots = 16;                        // (b): partial slots (heads x gene ranges)

// BANDED: a stage holds Z and the W tile ((b) item) or the H tile ((a) item) at the same offset
static_assert(kWBytes == kHBytes, "the two item kinds of the banded launch share one stage shape");
template <bool DO_A, bool DO_B, bool BANDED>
constexpr int stages() { return DO_A && DO_B && !BANDED ? 2 : 3; }
template <bool DO_A, bool DO_B, bool BANDED>
constexpr uint32_t stage_bytes() { return BANDED ? kZBytes + kWBytes : kZBytes + (DO_B ? kWBytes : 0) + (DO_A ? kHBytes : 0); }
template <bool DO_A, bool DO_B, bool COLSUM, bool BANDED>
constexpr uint32_t smem_bytes() {
  return stages<DO_A, DO_B, BANDED>() * stage_bytes<DO_A, DO_B, BANDED>() + (DO_A ? kOutBytes : 0) + (COLSUM ? kOnesBytes : 0) + 1024;
}

// One item of the banded head backward.  kind 0: (a) item = gene block gb0 of head `head` over all cell blocks;
// kind 1: (b) item = cell block cb0 over gene blocks [gb0, gb0 + ng) = (b) gene range gr, partial slot
// head * ranges + gr.
struct BandItem { int kind, head, gr, gb0, ng, cb0, ncb; };

// Item k of the band order: bands (head, gene range of gpr gene blocks; only the last range of a head may be shorter)
// head-major; within a band (a) and (b) items alternate, (a) first, and the longer kind's remaining items follow.  Tile
// (gb0 + i, cell block j) of a band is read by its (a) item i at step j and by its (b) item j at step i.
__host__ __device__ inline BandItem band_item(int k, int n_gb, int n_cb, int gpr, int ranges) {
  const int per_head = n_gb + ranges * n_cb, full_band = gpr + n_cb;
  BandItem it;
  it.head = k / per_head; k -= it.head * per_head;
  it.gr = min(k / full_band, ranges - 1); k -= it.gr * full_band;
  const int gb0 = it.gr * gpr, ng = min(n_gb, gb0 + gpr) - gb0, m = min(ng, n_cb);
  int idx;
  if (k < 2 * m) { it.kind = k & 1; idx = k >> 1; }
  else { it.kind = ng > n_cb ? 0 : 1; idx = k - m; }
  if (it.kind == 0) { it.gb0 = gb0 + idx; it.ng = 1; it.cb0 = 0; it.ncb = n_cb; }
  else { it.gb0 = gb0; it.ng = ng; it.cb0 = idx; it.ncb = 1; }
  return it;
}

struct Params {
  int B, G, n_heads;
  int n_cb, n_gb;                 // cell blocks (128), gene blocks per head (128)
  int gb_per_item, cb_per_item;
  int gene_ranges, cell_splits;   // per head
  int total_items;
  int stagger;                    // BANDED: start delay per band position, SM cycles (0: none)
  float* db[3];                  // column sums of Z per head (COLSUM)
  float* part; int64_t part_stride;   // (b): partial slot (head * gene_ranges + gene range) of part_stride floats
  // cell i of the batch is row rows[i] of zsrc (ld ldz; one Z); rows == null: the tiles are rows of map_z*
  const int32_t* rows; const __nv_bfloat16* zsrc; int64_t ldz;
};

// 16-byte global -> shared copy through the load path, zero-filling the bytes past src_bytes (cp.async groups are per
// thread)
__device__ __forceinline__ void cp_async_16(uint32_t smem_dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// MAXG: gene blocks per item held in registers (the (a) accumulators); WK: W is K-major (Keras [64 x G] head kernel);
// BANDED (with DO_A, DO_B): each item is one kind, (a) or (b), in band order (band_item)
template <bool DO_A, bool DO_B, bool COLSUM, bool WK, int MAXG, bool BANDED>
__global__ void __launch_bounds__(kThreads, 1)
gene_gemm_kernel(const __grid_constant__ CUtensorMap map_z0, const __grid_constant__ CUtensorMap map_z1,
                 const __grid_constant__ CUtensorMap map_z2, const __grid_constant__ CUtensorMap map_h,
                 const __grid_constant__ CUtensorMap map_w0, const __grid_constant__ CUtensorMap map_w1,
                 const __grid_constant__ CUtensorMap map_w2, const __grid_constant__ CUtensorMap map_dw0, const __grid_constant__ CUtensorMap map_dw1,
                 const __grid_constant__ CUtensorMap map_dw2, const int dw_transposed, const Params p) {
  static_assert(!BANDED || (DO_A && DO_B && MAXG == 1), "banded items hold one gene block of (a) accumulators");
  constexpr int kStages = stages<DO_A, DO_B, BANDED>();
  constexpr uint32_t kStage = stage_bytes<DO_A, DO_B, BANDED>();
  constexpr uint32_t kHOff = kZBytes + (DO_B && !BANDED ? kWBytes : 0);   // H tile within a stage
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* s_st = smem;                                                  // [kStages][Z | W | H]
  float* s_o = reinterpret_cast<float*>(s_st + kStages * kStage);         // (a) flush staging
  uint8_t* s_ones = reinterpret_cast<uint8_t*>(s_o) + (DO_A ? kOutBytes : 0);
  __shared__ uint64_t full[kStages];

  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) mbar_init(&full[i], 1);
    fence_barrier_init();
  }
  if (COLSUM) {   // bf16 1.0 = 0x3F80
    for (int i = threadIdx.x; i < (int)kOnesBytes / 4; i += kThreads) reinterpret_cast<uint32_t*>(s_ones)[i] = 0x3F803F80u;
    fence_proxy_async_smem();
  }
  __syncthreads();

  const int wg = threadIdx.x >> 7, w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
  const int frow = 16 * w + (l >> 2), fcol = 2 * (l & 3);           // fragment origin (see tc_common.cuh)

  // staging tile -> global (+=) by TMA; the previous reduce must have read the tile before it is rewritten
  auto stage_begin = [&]() {
    if (threadIdx.x == 0) bulk_wait_read<0>();
    __syncthreads();
  };
  auto stage_end = [&](const CUtensorMap* m, int c0, int c1) {
    fence_proxy_async_smem();
    __syncthreads();
    if (threadIdx.x == 0) { tma_reduce_add_2d(m, c0, c1, s_o); bulk_commit(); }
  };

  // The grid may be smaller than the item count (SMs left to other work): CTAs stride over the items.  T0 = tiles this
  // CTA consumed in earlier items, so that stage and mbarrier phase continue across items (every issued tile is consumed
  // before the next item starts).
  uint32_t T0 = 0;
  // Gathered rows (Params::rows; K1): the Z half of a stage is filled by all 256 threads with 16-byte cp.async
  // copies instead of TMA boxes (a TMA box per 128-byte row half issues too slowly).  Thread (rh = tid / 8, c = tid % 8)
  // copies chunk c (genes 8c .. 8c+7) of half rh % 2 of tile rows rh / 2 + 16 i, i < 8: each warp instruction reads
  // four whole 128-byte row halves.  A chunk goes where SWIZZLE_128B puts it -- chunk c of row r at byte
  // 16 * (c ^ (r % 8)) of the row -- so the tile is laid out exactly as the TMA lays out a contiguous batch; genes past
  // G and rows past the batch are zero-filled.  Each thread waits for its own copies of a tile, makes them visible to
  // the async proxy (wgmma), and a CTA barrier publishes them; the next tile's row indices load while copies run.
  const bool gather = p.rows != nullptr;
  const int g_rh = threadIdx.x >> 3, g_c = threadIdx.x & 7, g_h = g_rh & 1, g_r0 = g_rh >> 1;
  const uint32_t g_dst = g_h * (kZBytes / 2) + g_r0 * 128 + ((g_c ^ (g_r0 & 7)) << 4);
  int src_row[8];
  if constexpr (BANDED) {
    // Start stagger: the CTA whose first item is a band's item i (of either kind) starts i x p.stagger SM cycles late,
    // about i tile steps.  (a) item i then reads tile (i, j) at about the time (b) item j does, so the second read of a
    // tile follows the first closely; later items keep the offset (equal item lengths, grid of whole bands).
    if (p.stagger > 0 && blockIdx.x < p.total_items) {
      const BandItem it = band_item(blockIdx.x, p.n_gb, p.n_cb, p.gb_per_item, p.gene_ranges);
      const long long wait = (long long)(it.kind ? it.cb0 : it.gb0 - it.gr * p.gb_per_item) * p.stagger;
      if (threadIdx.x == 0) {
        const long long c0 = clock64();
        while (clock64() - c0 < wait) __nanosleep(100);
      }
      __syncthreads();
    }
  }
  for (int item = blockIdx.x; item < p.total_items; item += gridDim.x) {
    // item -> (head, gene blocks [gb0, gb1), cell blocks [cb0, cb1)); ia / ib: the item computes (a) / (b)
    int head, gr, gb0, ng, cb0, ncb;
    bool ia = DO_A, ib = DO_B;
    if constexpr (BANDED) {
      const BandItem it = band_item(item, p.n_gb, p.n_cb, p.gb_per_item, p.gene_ranges);
      head = it.head; gr = it.gr; gb0 = it.gb0; ng = it.ng; cb0 = it.cb0; ncb = it.ncb;
      ia = it.kind == 0; ib = !ia;
    } else {
      const int cs = item % p.cell_splits, r = item / p.cell_splits;
      gr = r % p.gene_ranges; head = r / p.gene_ranges;
      gb0 = gr * p.gb_per_item; ng = min(p.n_gb, gb0 + p.gb_per_item) - gb0;
      cb0 = cs * p.cb_per_item; ncb = min(p.n_cb, cb0 + p.cb_per_item) - cb0;
    }
    const int n_tiles = ng * ncb;
    const CUtensorMap* mz = head == 0 ? &map_z0 : (head == 1 ? &map_z1 : &map_z2);
    const CUtensorMap* mw = head == 0 ? &map_w0 : (head == 1 ? &map_w1 : &map_w2);
    const CUtensorMap* mdw = head == 0 ? &map_dw0 : (head == 1 ? &map_dw1 : &map_dw2);

    auto issue = [&](int t) {                       // thread 0: TMA loads of the item's tile t into its stage
      const int st = (T0 + t) % kStages;
      const int cb = cb0 + t / ng, gb = gb0 + t % ng;
      uint8_t* dst = s_st + st * kStage;
      mbar_expect_tx(&full[st], gather ? kStage - kZBytes : kStage);
      if (!gather) {
        tma_load_2d(dst, mz, gb * 128, cb * 128, &full[st]);
        tma_load_2d(dst + kZBytes / 2, mz, gb * 128 + 64, cb * 128, &full[st]);
      }
      if (DO_B && ib) {
        if (WK) {        // head backward: W = Keras [64 x G] (K-major B): two [64 feats x 64 genes] boxes
          tma_load_2d(dst + kZBytes, mw, gb * 128, 0, &full[st]);
          tma_load_2d(dst + kZBytes + kWBytes / 2, mw, gb * 128 + 64, 0, &full[st]);
        } else {         // encoder forward: W = Keras [G x 64] (MN-major B): one [128 genes x 64 feats] box
          tma_load_2d(dst + kZBytes, mw, 0, gb * 128, &full[st]);
        }
      }
      if (DO_A && ia) tma_load_2d(dst + kHOff, &map_h, 0, cb * 128, &full[st]);
    };
    auto load_rows = [&](int t) {                   // gathered rows: source rows of this thread's rows of tile t
      const int cb = cb0 + t / ng;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = cb * 128 + g_r0 + 16 * i;
        src_row[i] = r < p.B ? __ldg(p.rows + r) : -1;
      }
    };
    auto copy_rows = [&](int t) {                   // gathered rows: this thread's 8 chunks of the Z half of tile t
      const int st = (T0 + t) % kStages, g0 = (gb0 + t % ng) * 128 + g_h * 64 + g_c * 8;
      const uint32_t gbytes = g0 < p.G ? (uint32_t)min(16, 2 * (p.G - g0)) : 0u;
      const uint32_t dst = smem_u32(s_st + st * kStage) + g_dst;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const bool ok = src_row[i] >= 0 && gbytes != 0;
        cp_async_16(dst + i * 2048, ok ? p.zsrc + (int64_t)src_row[i] * p.ldz + g0 : p.zsrc, ok ? gbytes : 0u);
      }
      if (t + 1 < n_tiles) load_rows(t + 1);
    };
    if (gather) load_rows(0);
    for (int t = 0; t < kStages - 1; ++t) {         // (gathered rows: one cp.async group per tile slot, empty or not)
      if (t < n_tiles) {
        if (threadIdx.x == 0) issue(t);
        if (gather) copy_rows(t);
      }
      if (gather) cp_async_commit();
    }

    float acc_b[DO_B ? 32 : 1];                                        // (b): cells 64*wg.. of the current cell block
    float acc_a[DO_A ? MAXG : 1][32];                                  // (a): genes 64*wg.. of each gene block of the item
    float acc_c[COLSUM ? MAXG : 1][8];                                 // column sums
#pragma unroll
    for (int j = 0; j < (DO_A ? MAXG : 1); ++j)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc_a[j][i] = 0.f;
#pragma unroll
    for (int j = 0; j < (COLSUM ? MAXG : 1); ++j)
#pragma unroll
      for (int i = 0; i < 8; ++i) acc_c[j][i] = 0.f;

    int t = 0;
    for (int cbi = 0; cbi < ncb; ++cbi) {
      const int cb = cb0 + cbi;
#pragma unroll
      for (int i = 0; i < (DO_B ? 32 : 1); ++i) acc_b[i] = 0.f;
      // (a) needs a compile-time accumulator index per gene block: unrolled over MAXG; the (b) products walk their
      // whole gene range with one accumulator
#pragma unroll
      for (int jj = 0; jj < (DO_A ? MAXG : 1); ++jj)
      for (int j = jj; j < (DO_A && ia ? min(jj + 1, ng) : ng); ++j) {
        if (t + kStages - 1 < n_tiles) {            // its stage was released at tile t-1
          if (threadIdx.x == 0) issue(t + kStages - 1);
          if (gather) copy_rows(t + kStages - 1);
        }
        if (gather) {   // this thread's copies of tile t have landed (younger groups may still run); publish them all
          cp_async_commit();
          cp_async_wait<kStages - 1>();
          fence_proxy_async_smem();
          __syncthreads();
        }
        const int st = (T0 + t) % kStages;
        mbar_wait(&full[st], ((T0 + t) / kStages) & 1);
        const uint32_t zb = smem_u32(s_st + st * kStage), wb = zb + kZBytes, hb = zb + kHOff;
        wgmma_fence();
        if constexpr (DO_B) {
          if (ib)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const uint64_t da = make_smem_desc(zb + h * (kZBytes / 2) + wg * 64 * 128 + k * 32, 0, 1024);
              if (WK) wgmma_m64n64k16<0, 0>(acc_b, da, make_smem_desc(wb + h * (kWBytes / 2) + k * 32, 0, 1024), 1u);
              else wgmma_m64n64k16<0, 1>(acc_b, da, make_smem_desc(wb + (h * 4 + k) * 2048, 0, 1024), 1u);
            }
        }
        if constexpr (DO_A) {
          if (ia)
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const uint64_t da = make_smem_desc(zb + wg * (kZBytes / 2) + k * 2048, 0, 1024);
            wgmma_m64n64k16<1, 1>(acc_a[jj], da, make_smem_desc(hb + k * 2048, 0, 1024), 1u);
            if constexpr (COLSUM) wgmma_m64n16k16<1, 0>(acc_c[jj], da, make_smem_desc(smem_u32(s_ones) + (k & 3) * 32, 0, 1024), 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        if constexpr (DO_B) acc_fence(acc_b);
        if constexpr (DO_A) {
#pragma unroll
          for (int jj2 = 0; jj2 < MAXG; ++jj2) acc_fence(acc_a[jj2]);
        }
        if constexpr (COLSUM) {
#pragma unroll
          for (int jj2 = 0; jj2 < MAXG; ++jj2) acc_fence(acc_c[jj2]);
        }
        __syncthreads();                            // every warpgroup is done with stage st
        ++t;
      }
      if constexpr (DO_B) if (ib) {  // (b) of this cell block -> this item's partial slot (rows padded to whole cell blocks)
        float* dst = p.part + (int64_t)(head * p.gene_ranges + gr) * p.part_stride + (int64_t)cb * 128 * 64;
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          const int row = wg * 64 + frow + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + fcol;
          *reinterpret_cast<float2*>(dst + row * 64 + col) = make_float2(acc_b[i], acc_b[i + 1]);
        }
      }
    }
    T0 += n_tiles;
    if (DO_A && ia) {      // (a) of the item: one [128 genes x 64] block per gene block
#pragma unroll
      for (int j = 0; j < MAXG; ++j) {
        if (j >= ng) break;
        const int gb = gb0 + j;
        stage_begin();
        if (dw_transposed) {      // Keras [64 x G]: staging [64 feats][128 genes]
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const int g = wg * 64 + frow + 8 * ((i >> 1) & 1), f = 8 * (i >> 2) + fcol + (i & 1);
            s_o[f * 128 + g] = acc_a[j][i];
          }
          stage_end(mdw, gb * 128, 0);
        } else {                  // [G x 64]: staging [128 genes][64 feats]
#pragma unroll
          for (int i = 0; i < 32; i += 2) {
            const int g = wg * 64 + frow + 8 * ((i >> 1) & 1), f = 8 * (i >> 2) + fcol;
            *reinterpret_cast<float2*>(s_o + g * 64 + f) = make_float2(acc_a[j][i], acc_a[j][i + 1]);
          }
          stage_end(mdw, 0, gb * 128);
        }
        if constexpr (COLSUM) {
          float* dbh = head == 0 ? p.db[0] : (head == 1 ? p.db[1] : p.db[2]);   // (no dynamic index into the parameters)
          if ((l & 3) == 0 && dbh) {               // every column of the column-sum accumulator holds the sum
            const int g = gb * 128 + wg * 64 + frow;
            if (g < p.G) atomicAdd(dbh + g, acc_c[j][0]);
            if (g + 8 < p.G) atomicAdd(dbh + g + 8, acc_c[j][2]);
          }
        }
      }
    }
  }
  if (threadIdx.x == 0) bulk_wait<0>();
}

// out[i] += sum over s of part[s * stride + i], s in slot order (float4 per thread; n and stride are multiples of 4)
__global__ void gene_gemm_reduce_kernel(const float* __restrict__ part, int slots, int64_t stride, float* __restrict__ out,
                                        int64_t n) {
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i >= n) return;
  float4 acc = *reinterpret_cast<const float4*>(out + i);
  for (int sl = 0; sl < slots; ++sl) {
    const float4 v = __ldcs(reinterpret_cast<const float4*>(part + sl * stride + i));
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
  }
  *reinterpret_cast<float4*>(out + i) = acc;
}

// Item plans; p holds n_cb and n_gb.  The (b) gene ranges fix the partial slots and so the bits of the Z.W products:
// the banded head backward takes them from plan_b.
// (a): items = (head, gene range) over all cells.  gpi (gene blocks per item, <= kMaxGb for the registers) by the
// shortest makespan in tile units: rounds x (tiles per item + a flush term per gene block)
void plan_a(Params& p, int n_heads, int sm_count) {
  int best_gpi = 1; long long best_cost = -1;
  for (int gpi = 1; gpi <= kMaxGb; ++gpi) {
    const long long items = (long long)cdiv(p.n_gb, gpi) * n_heads, rounds = (items + sm_count - 1) / sm_count;
    const long long cost = rounds * ((long long)gpi * p.n_cb + 2ll * gpi);
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best_gpi = gpi; }
  }
  p.gb_per_item = best_gpi; p.gene_ranges = cdiv(p.n_gb, best_gpi);
  p.cb_per_item = p.n_cb; p.cell_splits = 1;
  p.total_items = p.gene_ranges * n_heads;
}
// (b): items = (head, gene range, cell block), ~4 per SM, at most kMaxSlots partial slots
void plan_b(Params& p, int n_heads, int sm_count) {
  p.cb_per_item = 1; p.cell_splits = p.n_cb;
  int gsplits = cdiv(4 * sm_count, p.n_cb * n_heads); if (gsplits < 1) gsplits = 1;
  if (gsplits > kMaxSlots / n_heads) gsplits = kMaxSlots / n_heads;
  if (gsplits > p.n_gb) gsplits = p.n_gb;
  while (gsplits > 1 && cdiv(p.n_gb, gsplits) < 4) --gsplits;
  p.gb_per_item = cdiv(p.n_gb, gsplits); p.gene_ranges = cdiv(p.n_gb, p.gb_per_item);
  p.total_items = p.gene_ranges * p.cell_splits * n_heads;
}
// Banded head backward: plan_b's gene ranges, (a) items of one gene block (their bits do not depend on the item size).
// The grid is a whole number of full bands when the SM budget holds one, so that the bands of a wave start together.
void plan_banded(Params& p, int n_heads, int sm_count, int* grid) {
  plan_b(p, n_heads, sm_count);
  p.total_items = n_heads * (p.n_gb + p.gene_ranges * p.n_cb);
  const int band = p.gb_per_item + p.n_cb;
  *grid = min(p.total_items, sm_count >= band ? sm_count / band * band : sm_count);
}

// ------------------------------------------------------------------------------------ encoder backward (K5)
// dW1[G x 64] += X^T . dA1 in 64-gene blocks: one warpgroup owns a block over all cells, which is the (a) product of
// the gene_gemm_kernel warpgroup for those genes -- the same m64n64k16 chain over cell tiles 0, 1, ... and k16 steps in
// order, from zero, added to dW once by a staging-tile reduce-add -- so dW1 has the same bits whatever the schedule.
// CTA c of `ctas` owns the contiguous blocks [eb_first(c), eb_first(c + 1)), within one of each other in count, and
// walks them in passes of up to kEbMaxW blocks, one consumer warpgroup each, sharing each stage's dA1 tile.  At
// G = 20000 (313 blocks) on 132 SMs that is 3 blocks on 49 CTAs and 2 on 83, one pass each: 3 x 64 genes in the
// longest lane, where 128-gene items take 4 x 64 (two rounds of one item or one round of two).
constexpr int kEbMaxW = 3;                                 // 64-gene blocks per pass = consumer warpgroups
constexpr int kEbThreads = 128 * kEbMaxW;
constexpr uint32_t kEbSub = 128 * 128;                     // [128 cells x 64 genes] bf16: one SWIZZLE_128B box
constexpr uint32_t kEbStage = kEbMaxW * kEbSub + kHBytes;  // X sub-tiles of the pass's blocks | dA1 tile
constexpr int kEbStages = 3;
constexpr uint32_t kEbSmem = kEbStages * kEbStage + 1024;
static_assert(kEbMaxW * 64 * 64 * 4 <= kEbStage, "the flush staging tiles fit in the first stage");

struct EncBwdParams {
  int B, G, n_cb, n_blk;          // cell blocks (128), gene blocks (64)
  const int32_t* rows; const __nv_bfloat16* zsrc; int64_t ldz;   // gathered rows as in Params; rows == null: map_z
};

// first 64-gene block of CTA c (c = ctas: n_blk); the first n_blk % ctas CTAs own one block more than the others
__host__ __device__ inline int eb_first(int c, int n_blk, int ctas) { return c * (n_blk / ctas) + min(c, n_blk % ctas); }
inline int eb_ctas(int n_blk, int sm_count) { return max(1, min(sm_count, n_blk)); }

__global__ void __launch_bounds__(kEbThreads, 1)
gene_gemm_enc_bwd_kernel(const __grid_constant__ CUtensorMap map_z, const __grid_constant__ CUtensorMap map_h,
                         const __grid_constant__ CUtensorMap map_dw, const int dw_transposed, const EncBwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* s_st = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // [kEbStages][X x kEbMaxW | dA1]
  __shared__ uint64_t full[kEbStages];
  if (threadIdx.x == 0) {
    for (int i = 0; i < kEbStages; ++i) mbar_init(&full[i], 1);
    fence_barrier_init();
  }
  __syncthreads();

  const int wg = threadIdx.x >> 7, w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
  const int frow = 16 * w + (l >> 2), fcol = 2 * (l & 3);
  // Gathered rows: warpgroup wg copies its own block's sub-tile, thread (r0 = tid / 8, c = tid % 8) chunk c of tile rows
  // r0 + 16 i, i < 8, at its SWIZZLE_128B place (as in gene_gemm_kernel, one 64-gene half per warpgroup)
  const bool gather = p.rows != nullptr;
  const int g_r0 = (threadIdx.x & 127) >> 3, g_c = threadIdx.x & 7;
  const uint32_t g_dst = wg * kEbSub + g_r0 * 128 + ((g_c ^ (g_r0 & 7)) << 4);
  int src_row[8];

  const int last = eb_first(blockIdx.x + 1, p.n_blk, gridDim.x);
  uint32_t T0 = 0;                                 // tiles consumed in earlier passes: stage and phase continue
  for (int blk0 = eb_first(blockIdx.x, p.n_blk, gridDim.x); blk0 < last; blk0 += kEbMaxW) {
    const int nw = min(kEbMaxW, last - blk0);
    const bool mine = wg < nw;                     // this warpgroup owns block blk0 + wg in this pass
    // the previous pass's flush has read its staging tiles (stage memory) before this pass loads into it
    if (threadIdx.x == 0) bulk_wait_read<0>();
    __syncthreads();

    auto issue = [&](int t) {                      // thread 0: dA1 tile t (and the X sub-tiles when not gathered)
      const int st = (T0 + t) % kEbStages;
      uint8_t* dst = s_st + st * kEbStage;
      mbar_expect_tx(&full[st], kHBytes + (gather ? 0u : nw * kEbSub));
      if (!gather)
        for (int j = 0; j < nw; ++j) tma_load_2d(dst + j * kEbSub, &map_z, (blk0 + j) * 64, t * 128, &full[st]);
      tma_load_2d(dst + kEbMaxW * kEbSub, &map_h, 0, t * 128, &full[st]);
    };
    auto load_rows = [&](int t) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = t * 128 + g_r0 + 16 * i;
        src_row[i] = r < p.B ? __ldg(p.rows + r) : -1;
      }
    };
    auto copy_rows = [&](int t) {                  // this thread's 8 chunks of its warpgroup's sub-tile of tile t
      if (mine) {
        const int g0 = (blk0 + wg) * 64 + g_c * 8;
        const uint32_t gbytes = g0 < p.G ? (uint32_t)min(16, 2 * (p.G - g0)) : 0u;
        const uint32_t dst = smem_u32(s_st + ((T0 + t) % kEbStages) * kEbStage) + g_dst;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const bool ok = src_row[i] >= 0 && gbytes != 0;
          cp_async_16(dst + i * 2048, ok ? p.zsrc + (int64_t)src_row[i] * p.ldz + g0 : p.zsrc, ok ? gbytes : 0u);
        }
        if (t + 1 < p.n_cb) load_rows(t + 1);
      }
    };
    if (gather && mine) load_rows(0);
    for (int t = 0; t < kEbStages - 1; ++t) {      // (gathered rows: one cp.async group per tile slot, empty or not)
      if (t < p.n_cb) {
        if (threadIdx.x == 0) issue(t);
        if (gather) copy_rows(t);
      }
      if (gather) cp_async_commit();
    }

    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    for (int t = 0; t < p.n_cb; ++t) {
      if (t + kEbStages - 1 < p.n_cb) {            // its stage was released at tile t-1
        if (threadIdx.x == 0) issue(t + kEbStages - 1);
        if (gather) copy_rows(t + kEbStages - 1);
      }
      if (gather) {
        cp_async_commit();
        cp_async_wait<kEbStages - 1>();
        fence_proxy_async_smem();
        __syncthreads();
      }
      const int st = (T0 + t) % kEbStages;
      mbar_wait(&full[st], ((T0 + t) / kEbStages) & 1);
      if (mine) {
        const uint32_t zb = smem_u32(s_st + st * kEbStage) + wg * kEbSub, hb = smem_u32(s_st + st * kEbStage) + kEbMaxW * kEbSub;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 8; ++k)
          wgmma_m64n64k16<1, 1>(acc, make_smem_desc(zb + k * 2048, 0, 1024), make_smem_desc(hb + k * 2048, 0, 1024), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        acc_fence(acc);
      }
      __syncthreads();                             // every warpgroup is done with stage st
    }
    T0 += p.n_cb;

    // flush: every tile is consumed, so block j's [64 x 64] fp32 staging tile goes at byte j * kEbSub of the stages
    float* s_o = reinterpret_cast<float*>(s_st + wg * kEbSub);
    if (mine) {
      if (dw_transposed) {                         // Keras [64 x G]: staging [64 feats][64 genes]
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int g = frow + 8 * ((i >> 1) & 1), f = 8 * (i >> 2) + fcol + (i & 1);
          s_o[f * 64 + g] = acc[i];
        }
      } else {                                     // [G x 64]: staging [64 genes][64 feats]
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          const int g = frow + 8 * ((i >> 1) & 1), f = 8 * (i >> 2) + fcol;
          *reinterpret_cast<float2*>(s_o + g * 64 + f) = make_float2(acc[i], acc[i + 1]);
        }
      }
    }
    fence_proxy_async_smem();
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int j = 0; j < nw; ++j) {
        const int g = (blk0 + j) * 64;
        tma_reduce_add_2d(&map_dw, dw_transposed ? g : 0, dw_transposed ? 0 : g, s_st + j * kEbSub);
      }
      bulk_commit();
    }
  }
  if (threadIdx.x == 0) bulk_wait<0>();
}

}  // namespace gg

size_t gene_gemm_workspace_bytes(int B) { return sizeof(float) * (size_t)gg::kMaxSlots * cdiv(B, 128) * 128 * 64; }

// Z: bf16 [B x G] per head (ldz elements); H: bf16 [B x 64]; W[i]: bf16 Keras-layout kernels -- [G x 64] for mode 1 (the
// encoder kernel), [64 x G] per head for mode 3; out_b: fp32 [B x 64] (+=).
// mode: 1 = encoder forward (K1), 2 = encoder backward (K5), 3 = head backward (K4: one band-ordered launch of the dW /
// db and dH items, or with head_bwd_banded = 0 the dW / db pass, then the dH pass).
// ws: gene_gemm_workspace_bytes(B) of device memory for the partial slots of modes 1 and 3.
// rows (modes 1 and 2, may be null): cell i of the batch is row rows[i] of Z[0]; every index must be a row of Z[0].
int gene_gemm_tc(int mode, const __nv_bfloat16* const Z[3], int64_t ldz, const int32_t* rows, int B, int G, int n_heads,
                 const __nv_bfloat16* H, const __nv_bfloat16* const W[3], float* out_b, float* const dW[3], int64_t dW_ld,
                 int dW_transposed, float* const db[3], void* ws, size_t ws_bytes, int sm_count, cudaStream_t s) {
  using namespace gg;
  if (ldz % 8 != 0) { set_error("gene_gemm_tc: ldz must be a multiple of 8 (16-byte TMA stride)"); return DCA_ERR_BAD_ARG; }
  if (mode < 1 || mode > 3) { set_error("gene_gemm_tc: bad mode %d", mode); return DCA_ERR_BAD_ARG; }
  if (rows && (mode == 3 || n_heads != 1)) { set_error("gene_gemm_tc: row indices are for modes 1 and 2 (one Z)"); return DCA_ERR_BAD_ARG; }
  const bool do_a = mode & 2, do_b = mode & 1;
  if (do_b && (!ws || ws_bytes < gene_gemm_workspace_bytes(B))) { set_error("gene_gemm_tc: workspace too small"); return DCA_ERR_BAD_ARG; }
  CUtensorMap mz[3], mh, mw[3], mdw[3];
  for (int i = 0; i < 3; ++i) DCA_TRY(make_tensor_map_2d(&mz[i], Z[i < n_heads ? i : 0], 2, 1, (uint64_t)B, (uint64_t)G, (uint64_t)ldz, 128, 64, 1));
  mh = mz[0];
  for (int i = 0; i < 3; ++i) mw[i] = mdw[i] = mz[0];
  if (do_a) {
    DCA_TRY(make_tensor_map_2d(&mh, H, 2, 1, (uint64_t)B, 64, 64, 128, 64, 1));
    for (int i = 0; i < 3; ++i) {
      float* d = dW[i < n_heads ? i : 0];
      if (dW_transposed) DCA_TRY(make_tensor_map_2d(&mdw[i], d, 4, 0, 64, (uint64_t)G, (uint64_t)dW_ld, 64, 128, 0));
      else {
        if (dW_ld != 64) { set_error("gene_gemm_tc: non-transposed dW needs ld == 64"); return DCA_ERR_BAD_ARG; }
        DCA_TRY(make_tensor_map_2d(&mdw[i], d, 4, 0, (uint64_t)G, 64, 64, 128, 64, 0));
      }
    }
  }
  if (do_b) {
    for (int i = 0; i < 3; ++i) {
      const __nv_bfloat16* w = W[i < n_heads ? i : 0];
      if (mode == 3) DCA_TRY(make_tensor_map_2d(&mw[i], w, 2, 1, 64, (uint64_t)G, (uint64_t)G, 64, 64, 1));
      else DCA_TRY(make_tensor_map_2d(&mw[i], w, 2, 1, (uint64_t)G, 64, 64, 128, 64, 1));
    }
  }
  Params base{};
  base.B = B; base.G = G; base.n_heads = n_heads;
  base.n_cb = cdiv(B, 128); base.n_gb = cdiv(G, 128);
  for (int i = 0; i < 3; ++i) base.db[i] = db ? db[i] : nullptr;
  base.part = reinterpret_cast<float*>(ws); base.part_stride = (int64_t)base.n_cb * 128 * 64;
  base.rows = rows; base.zsrc = Z[0]; base.ldz = ldz;

  // at most one CTA per SM (shared memory) and at most sm_count CTAs: a caller that passes fewer SMs than the device has
  // leaves the others free; the CTAs stride over the items
#define DCA_GG_LAUNCH(P, GRID, A, Bb, Cc, WKk, MG, BND)                                                                \
  do {                                                                                                                 \
    static bool attr = false;                                                                                          \
    constexpr uint32_t sm = smem_bytes<A, Bb, Cc, BND>();                                                              \
    if (!attr) { DCA_CUDA_OK(cudaFuncSetAttribute(gene_gemm_kernel<A, Bb, Cc, WKk, MG, BND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm)); attr = true; } \
    gene_gemm_kernel<A, Bb, Cc, WKk, MG, BND><<<GRID, kThreads, sm, s>>>(mz[0], mz[1], mz[2], mh, mw[0], mw[1], mw[2],  \
                                                                          mdw[0], mdw[1], mdw[2], dW_transposed, P);  \
    DCA_LAUNCH_CHECK();                                                                                                \
  } while (0)

  if (mode == 3 && g_head_bwd_banded) {
    Params p = base;
    int grid = 0;
    plan_banded(p, n_heads, sm_count, &grid);
    p.stagger = g_head_bwd_stagger;
    DCA_GG_LAUNCH(p, grid, true, true, true, true, 1, true);
    const int64_t n = (int64_t)B * 64;
    gene_gemm_reduce_kernel<<<(unsigned)cdiv(n / 4, 256), 256, 0, s>>>(p.part, p.gene_ranges * n_heads, p.part_stride, out_b, n);
    DCA_LAUNCH_CHECK();
    return DCA_OK;
  }
  if (mode == 2) {        // 64-gene blocks, the staging tile one block: [64 x 64] boxes of dW
    EncBwdParams p{B, G, base.n_cb, cdiv(G, 64), rows, Z[0], ldz};
    CUtensorMap mdw64;
    if (dW_transposed) DCA_TRY(make_tensor_map_2d(&mdw64, dW[0], 4, 0, 64, (uint64_t)G, (uint64_t)dW_ld, 64, 64, 0));
    else DCA_TRY(make_tensor_map_2d(&mdw64, dW[0], 4, 0, (uint64_t)G, 64, 64, 64, 64, 0));
    static bool attr = false;
    if (!attr) { DCA_CUDA_OK(cudaFuncSetAttribute(gene_gemm_enc_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kEbSmem)); attr = true; }
    gene_gemm_enc_bwd_kernel<<<eb_ctas(p.n_blk, sm_count), kEbThreads, kEbSmem, s>>>(mz[0], mh, mdw64, dW_transposed, p);
    DCA_LAUNCH_CHECK();
    return DCA_OK;
  }
  if (do_a) {             // head backward, dW / db pass
    Params p = base;
    plan_a(p, n_heads, sm_count);
    DCA_GG_LAUNCH(p, min(p.total_items, sm_count), true, false, true, false, kMaxGb, false);
  }
  if (do_b) {
    Params p = base;
    plan_b(p, n_heads, sm_count);
    const int grid = min(p.total_items, sm_count);
    if (mode == 3) DCA_GG_LAUNCH(p, grid, false, true, false, true, 1, false);
    else DCA_GG_LAUNCH(p, grid, false, true, false, false, 1, false);
    const int64_t n = (int64_t)B * 64;
    gene_gemm_reduce_kernel<<<(unsigned)cdiv(n / 4, 256), 256, 0, s>>>(p.part, p.gene_ranges * n_heads, p.part_stride, out_b, n);
    DCA_LAUNCH_CHECK();
  }
#undef DCA_GG_LAUNCH
  return DCA_OK;
}

}  // namespace tc
}  // namespace dca

// ------------------------------------------------------------------------------------ C ABI (tests / profiling)
using namespace dca;
extern "C" int dca_tc_gene_gemm_rows(int32_t mode, const void* Z0, const void* Z1, const void* Z2, int64_t ldz,
                                     const int32_t* rows, int32_t batch, int32_t genes, int32_t n_heads, const void* H,
                                     const void* W, float* out_b, float* dW0, float* dW1, float* dW2, int64_t dW_ld,
                                     int32_t dW_transposed, float* db0, float* db1, float* db2, void* stream, int32_t sm_count) {
  if (!Z0 || batch <= 0 || genes <= 0 || n_heads < 1 || n_heads > 3) { set_error("dca_tc_gene_gemm: bad argument"); return DCA_ERR_BAD_ARG; }
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (sm_count > 0 && sm_count < sms) sms = sm_count;      // a smaller grid: the CTAs stride over the items
  const __nv_bfloat16* Z[3] = {(const __nv_bfloat16*)Z0, (const __nv_bfloat16*)Z1, (const __nv_bfloat16*)Z2};
  float* dW[3] = {dW0, dW1, dW2};
  float* db[3] = {db0, db1, db2};
  const __nv_bfloat16* Wp[3];
  for (int i = 0; i < 3; ++i) Wp[i] = (const __nv_bfloat16*)W + (mode == 3 ? (size_t)(i < n_heads ? i : 0) * 64 * genes : 0);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t ws_bytes = tc::gene_gemm_workspace_bytes(batch);
  void* ws = nullptr;
  DCA_CUDA_OK(cudaMallocAsync(&ws, ws_bytes, st));
  const int rc = tc::gene_gemm_tc(mode, Z, ldz, rows, batch, genes, n_heads, (const __nv_bfloat16*)H, Wp, out_b, dW,
                                  dW_ld, dW_transposed, db, ws, ws_bytes, sms, st);
  DCA_CUDA_OK(cudaFreeAsync(ws, st));
  return rc;
}
extern "C" int dca_tc_gene_gemm_sms(int32_t mode, const void* Z0, const void* Z1, const void* Z2, int64_t ldz,
                                    int32_t batch, int32_t genes, int32_t n_heads, const void* H, const void* W, float* out_b,
                                    float* dW0, float* dW1, float* dW2, int64_t dW_ld, int32_t dW_transposed, float* db0,
                                    float* db1, float* db2, void* stream, int32_t sm_count) {
  return dca_tc_gene_gemm_rows(mode, Z0, Z1, Z2, ldz, nullptr, batch, genes, n_heads, H, W, out_b, dW0, dW1, dW2, dW_ld,
                               dW_transposed, db0, db1, db2, stream, sm_count);
}
extern "C" int dca_tc_gene_gemm(int32_t mode, const void* Z0, const void* Z1, const void* Z2, int64_t ldz, int32_t batch,
                                int32_t genes, int32_t n_heads, const void* H, const void* W, float* out_b, float* dW0,
                                float* dW1, float* dW2, int64_t dW_ld, int32_t dW_transposed, float* db0, float* db1,
                                float* db2, void* stream) {
  return dca_tc_gene_gemm_sms(mode, Z0, Z1, Z2, ldz, batch, genes, n_heads, H, W, out_b, dW0, dW1, dW2, dW_ld,
                              dW_transposed, db0, db1, db2, stream, 0);
}
extern "C" int dca_head_bwd_schedule(int32_t batch, int32_t genes, int32_t n_heads, int32_t sm_count, int32_t banded,
                                     int32_t* items, int64_t cap, int64_t* n_items, int32_t* grid) {
  if (batch <= 0 || genes <= 0 || n_heads < 1 || n_heads > 3 || sm_count < 1 || !n_items || !grid) {
    set_error("dca_head_bwd_schedule: bad argument"); return DCA_ERR_BAD_ARG;
  }
  tc::gg::Params base{};
  base.n_cb = cdiv(batch, 128); base.n_gb = cdiv(genes, 128);
  int64_t k = 0;
  auto put = [&](int launch, int kind, int head, int gb0, int ng, int cb0, int ncb, int slot) {
    if (items && k < cap) {
      int32_t* r = items + 8 * k;
      r[0] = launch; r[1] = kind; r[2] = head; r[3] = gb0; r[4] = ng; r[5] = cb0; r[6] = ncb; r[7] = slot;
    }
    ++k;
  };
  if (banded) {
    tc::gg::Params p = base;
    plan_banded(p, n_heads, sm_count, &grid[0]);
    grid[1] = 0;
    for (int i = 0; i < p.total_items; ++i) {
      const tc::gg::BandItem it = tc::gg::band_item(i, p.n_gb, p.n_cb, p.gb_per_item, p.gene_ranges);
      put(0, it.kind, it.head, it.gb0, it.ng, it.cb0, it.ncb, it.kind ? it.head * p.gene_ranges + it.gr : -1);
    }
  } else {   // the kernel's item decoding of the two launches
    tc::gg::Params pa = base, pb = base;
    plan_a(pa, n_heads, sm_count);
    plan_b(pb, n_heads, sm_count);
    grid[0] = std::min(pa.total_items, (int)sm_count); grid[1] = std::min(pb.total_items, (int)sm_count);
    for (int pass = 0; pass < 2; ++pass) {
      const tc::gg::Params& p = pass ? pb : pa;
      for (int i = 0; i < p.total_items; ++i) {
        const int cs = i % p.cell_splits, r = i / p.cell_splits, gr = r % p.gene_ranges, head = r / p.gene_ranges;
        const int gb0 = gr * p.gb_per_item, cb0 = cs * p.cb_per_item;
        put(pass, pass, head, gb0, std::min(p.n_gb, gb0 + p.gb_per_item) - gb0, cb0, std::min(p.n_cb, cb0 + p.cb_per_item) - cb0,
            pass ? head * p.gene_ranges + gr : -1);
      }
    }
  }
  *n_items = k;
  return DCA_OK;
}
extern "C" int dca_enc_bwd_schedule(int32_t genes, int32_t sm_count, int32_t* first, int64_t cap, int32_t* ctas) {
  if (genes <= 0 || sm_count < 1 || !ctas) { set_error("dca_enc_bwd_schedule: bad argument"); return DCA_ERR_BAD_ARG; }
  const int n_blk = cdiv(genes, 64);
  *ctas = tc::gg::eb_ctas(n_blk, sm_count);
  for (int64_t c = 0; first && c < cap && c <= *ctas; ++c) first[c] = tc::gg::eb_first((int)c, n_blk, *ctas);
  return DCA_OK;
}
