// One wgmma kernel for the gene-wide Dense products whose reduction or output dimension is the gene axis (all with a
// 64-wide partner dimension):
//
//   encoder forward  (K1)  A1[B x 64]  += X[B x G] . W1[G x 64]                      (b), W MN-major
//   head backward    (K4)  dH3[B x 64] += sum_h dZ_h . Wh^T                          (b), W K-major
//                          dWh[64 x G] += H3^T . dZ_h,  db_h += colsum(dZ_h)         (a) + column sums
//   encoder backward (K5)  dW1[G x 64] += X^T . dA1                                   (a)
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
#include "engine.h"
#include "tc_common.cuh"

namespace dca {
namespace tc {
int g_gg_profile = 0;       // dca_set_tunable("gg_profile", 1): phase timeline of the hidden-stack kernels (mid_stack.cu)
namespace gg {

constexpr int kThreads = 256;
constexpr uint32_t kZBytes = 128 * 128 * 2;          // 2 boxes x [128 cells x 64 genes] bf16
constexpr uint32_t kWBytes = 64 * 128 * 2;           // 2 boxes x [64 feats x 64 genes] | 1 box [128 genes x 64 feats] bf16
constexpr uint32_t kHBytes = 128 * 64 * 2;           // [128 cells x 64 feats] bf16
constexpr uint32_t kOutBytes = 128 * 64 * 4;         // fp32 staging tile of one flush
constexpr uint32_t kOnesBytes = 16 * 128;            // [16 x 64] bf16 ones, K-major B operand of the column sums
constexpr int kMaxGb = 4;                            // (a): gene blocks per item held in registers
constexpr int kMaxSlots = 16;                        // (b): partial slots (heads x gene ranges)

template <bool DO_A, bool DO_B>
constexpr int stages() { return DO_A && DO_B ? 2 : 3; }
template <bool DO_A, bool DO_B>
constexpr uint32_t stage_bytes() { return kZBytes + (DO_B ? kWBytes : 0) + (DO_A ? kHBytes : 0); }
template <bool DO_A, bool DO_B, bool COLSUM>
constexpr uint32_t smem_bytes() {
  return stages<DO_A, DO_B>() * stage_bytes<DO_A, DO_B>() + (DO_A ? kOutBytes : 0) + (COLSUM ? kOnesBytes : 0) + 1024;
}

struct Params {
  int B, G, n_heads;
  int n_cb, n_gb;                 // cell blocks (128), gene blocks per head (128)
  int gb_per_item, cb_per_item;
  int gene_ranges, cell_splits;   // per head
  int total_items;
  float* db[3];                   // column sums of Z per head (COLSUM)
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

// MAXG: gene blocks per item held in registers (the (a) accumulators); WK: W is K-major (Keras [64 x G] head kernel)
template <bool DO_A, bool DO_B, bool COLSUM, bool WK, int MAXG>
__global__ void __launch_bounds__(kThreads, 1)
gene_gemm_kernel(const __grid_constant__ CUtensorMap map_z0, const __grid_constant__ CUtensorMap map_z1,
                 const __grid_constant__ CUtensorMap map_z2, const __grid_constant__ CUtensorMap map_h,
                 const __grid_constant__ CUtensorMap map_w0, const __grid_constant__ CUtensorMap map_w1,
                 const __grid_constant__ CUtensorMap map_w2, const __grid_constant__ CUtensorMap map_dw0, const __grid_constant__ CUtensorMap map_dw1,
                 const __grid_constant__ CUtensorMap map_dw2, const int dw_transposed, const Params p) {
  constexpr int kStages = stages<DO_A, DO_B>();
  constexpr uint32_t kStage = stage_bytes<DO_A, DO_B>();
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
  // Gathered rows (Params::rows; K1 / K5): the Z half of a stage is filled by all 256 threads with 16-byte cp.async
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
  for (int item = blockIdx.x; item < p.total_items; item += gridDim.x) {
    // item -> (head, gene blocks [gb0, gb1), cell blocks [cb0, cb1))
    const int cs = item % p.cell_splits, r = item / p.cell_splits;
    const int gr = r % p.gene_ranges, head = r / p.gene_ranges;
    const int gb0 = gr * p.gb_per_item, ng = min(p.n_gb, gb0 + p.gb_per_item) - gb0;
    const int cb0 = cs * p.cb_per_item, ncb = min(p.n_cb, cb0 + p.cb_per_item) - cb0;
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
      if (DO_B) {
        if (WK) {        // head backward: W = Keras [64 x G] (K-major B): two [64 feats x 64 genes] boxes
          tma_load_2d(dst + kZBytes, mw, gb * 128, 0, &full[st]);
          tma_load_2d(dst + kZBytes + kWBytes / 2, mw, gb * 128 + 64, 0, &full[st]);
        } else {         // encoder forward: W = Keras [G x 64] (MN-major B): one [128 genes x 64 feats] box
          tma_load_2d(dst + kZBytes, mw, 0, gb * 128, &full[st]);
        }
      }
      if (DO_A) tma_load_2d(dst + kZBytes + (DO_B ? kWBytes : 0), &map_h, 0, cb * 128, &full[st]);
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
      for (int j = jj; j < (DO_A ? min(jj + 1, ng) : ng); ++j) {
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
        const uint32_t zb = smem_u32(s_st + st * kStage), wb = zb + kZBytes, hb = wb + (DO_B ? kWBytes : 0);
        wgmma_fence();
        if constexpr (DO_B) {
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
      if constexpr (DO_B) {  // (b) of this cell block -> this item's partial slot (rows padded to whole cell blocks)
        float* dst = p.part + (int64_t)(head * p.gene_ranges + gr) * p.part_stride + (int64_t)cb * 128 * 64;
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
          const int row = wg * 64 + frow + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + fcol;
          *reinterpret_cast<float2*>(dst + row * 64 + col) = make_float2(acc_b[i], acc_b[i + 1]);
        }
      }
    }
    T0 += n_tiles;
    if constexpr (DO_A) {  // (a) of the item: one [128 genes x 64] block per gene block
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

}  // namespace gg

size_t gene_gemm_workspace_bytes(int B) { return sizeof(float) * (size_t)gg::kMaxSlots * cdiv(B, 128) * 128 * 64; }

// Z: bf16 [B x G] per head (ldz elements); H: bf16 [B x 64]; W[i]: bf16 Keras-layout kernels -- [G x 64] for mode 1 (the
// encoder kernel), [64 x G] per head for mode 3; out_b: fp32 [B x 64] (+=).
// mode: 1 = encoder forward (K1), 2 = encoder backward (K5), 3 = head backward (K4: dW / db pass, then the dH pass).
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
#define DCA_GG_LAUNCH(P, A, Bb, Cc, WKk, MG)                                                                           \
  do {                                                                                                                 \
    static bool attr = false;                                                                                          \
    constexpr uint32_t sm = smem_bytes<A, Bb, Cc>();                                                                       \
    if (!attr) { DCA_CUDA_OK(cudaFuncSetAttribute(gene_gemm_kernel<A, Bb, Cc, WKk, MG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm)); attr = true; } \
    gene_gemm_kernel<A, Bb, Cc, WKk, MG><<<min(P.total_items, sm_count), kThreads, sm, s>>>(mz[0], mz[1], mz[2], mh, mw[0], mw[1], mw[2],      \
                                                                          mdw[0], mdw[1], mdw[2], dW_transposed, P);  \
    DCA_LAUNCH_CHECK();                                                                                                \
  } while (0)

  if (do_a) {
    // (a): items = (head, gene range) over all cells.  gpi (gene blocks per item, <= kMaxGb for the registers) by the
    // shortest makespan in tile units: rounds x (tiles per item + a flush term per gene block)
    Params p = base;
    int best_gpi = 1; long long best_cost = -1;
    for (int gpi = 1; gpi <= kMaxGb; ++gpi) {
      const long long items = (long long)cdiv(p.n_gb, gpi) * n_heads, rounds = (items + sm_count - 1) / sm_count;
      const long long cost = rounds * ((long long)gpi * p.n_cb + 2ll * gpi);
      if (best_cost < 0 || cost < best_cost) { best_cost = cost; best_gpi = gpi; }
    }
    p.gb_per_item = best_gpi; p.gene_ranges = cdiv(p.n_gb, best_gpi);
    p.cb_per_item = p.n_cb; p.cell_splits = 1;
    p.total_items = p.gene_ranges * n_heads;
    if (mode == 3) DCA_GG_LAUNCH(p, true, false, true, false, kMaxGb);
    else DCA_GG_LAUNCH(p, true, false, false, false, kMaxGb);
  }
  if (do_b) {
    // (b): items = (head, gene range, cell block), ~4 per SM, at most kMaxSlots partial slots
    Params p = base;
    p.cb_per_item = 1; p.cell_splits = p.n_cb;
    int gsplits = cdiv(4 * sm_count, p.n_cb * n_heads); if (gsplits < 1) gsplits = 1;
    if (gsplits > kMaxSlots / n_heads) gsplits = kMaxSlots / n_heads;
    if (gsplits > p.n_gb) gsplits = p.n_gb;
    while (gsplits > 1 && cdiv(p.n_gb, gsplits) < 4) --gsplits;
    p.gb_per_item = cdiv(p.n_gb, gsplits); p.gene_ranges = cdiv(p.n_gb, p.gb_per_item);
    p.total_items = p.gene_ranges * p.cell_splits * n_heads;
    if (mode == 3) DCA_GG_LAUNCH(p, false, true, false, true, 1);
    else DCA_GG_LAUNCH(p, false, true, false, false, 1);
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
