// wgmma / TMA Dense kernels for the gene-wide layers of the flagship shape (hidden 64).
//
//   heads_fwd_tc (K2): Z = H3[B x 64] . Wh[64 x nh*G] + b, MeanAct / DispAct / sigmoid fused into the
//       epilogue (dca/network.py:369-381, :38-39; dca/layers.py:85 for predict).  bf16 operands staged
//       by TMA (SWIZZLE_128B), fp32 accumulators in registers (two warpgroups x m64n128), epilogue
//       registers -> global.  HBM-bound: 128 flop per 4-byte output element (SURVEY.md 7.3-1).
//   tc_probe: single-tile kernel used by the tests to pin the wgmma descriptor conventions
//       (K-major / MN-major operands) against a plain matmul.
#include <mutex>
#include "engine.h"
#include "tc_common.cuh"
#include "head_act.cuh"

namespace dca {
namespace tc {

// ------------------------------------------------------------------------------------ tensor maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

int make_tensor_map_2d(CUtensorMap* out, const void* base, int elem_bytes, int is_bf16, uint64_t rows, uint64_t cols,
                       uint64_t ld_elems, uint32_t box_rows, uint32_t box_cols, int swizzle) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled is not available from the driver"); return DCA_ERR_CUDA; }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld_elems * (uint64_t)elem_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType dt = is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUresult r = fn(out, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): rows=%llu cols=%llu ld=%llu box=%ux%u elem=%d", (int)r,
              (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld_elems, box_rows, box_cols, elem_bytes);
    return DCA_ERR_CUDA;
  }
  return DCA_OK;
}

// ------------------------------------------------------------------------------------ probe kernel
struct ProbeParams {
  int a_mn, b_mn, M, N, K;
  int a_boxes, a_box_bytes, a_box_c0, a_box_c1;      // per box: coordinate increments (cols, rows)
  int b_boxes, b_box_bytes, b_box_c0, b_box_c1;
  uint32_t a_lbo, a_sbo, a_kstep, a_kblock_steps, a_kblock_bytes, a_mn64_bytes;
  uint32_t b_lbo, b_sbo, b_kstep, b_kblock_steps, b_kblock_bytes, b_mn64_bytes;   // mn64: bytes per 64 M / N elements
};

template <int NC, int TA, int TB>
__device__ __forceinline__ void probe_mma(float (&acc)[NC / 2], uint64_t da, uint64_t db) {
  if constexpr (NC == 128) wgmma_m64n128k16<TA, TB>(acc, da, db, 1u);
  else wgmma_m64n64k16<TA, TB>(acc, da, db, 1u);
}

// one warpgroup: D[rows m0.., cols n0..n0+NC) of the 128 x N product, K / 16 wgmma steps
template <int NC>
__device__ __forceinline__ void probe_chunk(const ProbeParams& p, uint32_t sa, uint32_t sb, int m0, int n0, float* D) {
  float acc[NC / 2];
#pragma unroll
  for (int i = 0; i < NC / 2; ++i) acc[i] = 0.f;
  const uint32_t a0 = sa + (uint32_t)(m0 / 64) * p.a_mn64_bytes, b0 = sb + (uint32_t)(n0 / 64) * p.b_mn64_bytes;
  wgmma_fence();
  for (int j = 0; j < p.K / 16; ++j) {
    const uint32_t aoff = (j / p.a_kblock_steps) * p.a_kblock_bytes + (j % p.a_kblock_steps) * p.a_kstep;
    const uint32_t boff = (j / p.b_kblock_steps) * p.b_kblock_bytes + (j % p.b_kblock_steps) * p.b_kstep;
    const uint64_t da = make_smem_desc(a0 + aoff, p.a_lbo, p.a_sbo), db = make_smem_desc(b0 + boff, p.b_lbo, p.b_sbo);
    // transpose flags are immediates: one instantiation per operand-major combination
    if (p.a_mn) { if (p.b_mn) probe_mma<NC, 1, 1>(acc, da, db); else probe_mma<NC, 1, 0>(acc, da, db); }
    else        { if (p.b_mn) probe_mma<NC, 0, 1>(acc, da, db); else probe_mma<NC, 0, 0>(acc, da, db); }
  }
  wgmma_commit();
  wgmma_wait<0>();
  acc_fence(acc);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < NC / 2; ++i) {
    const int row = m0 + 16 * w + (l >> 2) + 8 * ((i >> 1) & 1), col = n0 + 8 * (i >> 2) + 2 * (l & 3) + (i & 1);
    D[(size_t)row * p.N + col] = acc[i];
  }
}

__global__ void __launch_bounds__(128, 1)
tc_probe_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                const ProbeParams p, float* __restrict__ D) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  __shared__ uint64_t bar_load;
  uint8_t* sa = smem;
  uint8_t* sb = smem + (size_t)p.a_boxes * p.a_box_bytes;
  if (threadIdx.x == 0) { mbar_init(&bar_load, 1); fence_barrier_init(); }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(&bar_load, (uint32_t)(p.a_boxes * p.a_box_bytes + p.b_boxes * p.b_box_bytes));
    for (int i = 0; i < p.a_boxes; ++i) tma_load_2d(sa + (size_t)i * p.a_box_bytes, &map_a, i * p.a_box_c0, i * p.a_box_c1, &bar_load);
    for (int i = 0; i < p.b_boxes; ++i) tma_load_2d(sb + (size_t)i * p.b_box_bytes, &map_b, i * p.b_box_c0, i * p.b_box_c1, &bar_load);
  }
  mbar_wait(&bar_load, 0);
  // N chunks of 128 where possible: an MN-major B operand then spans two 64-wide blocks (exercises its LBO)
  for (int m0 = 0; m0 < p.M; m0 += 64)
    for (int n0 = 0; n0 < p.N;) {
      if (p.N - n0 >= 128) { probe_chunk<128>(p, smem_u32(sa), smem_u32(sb), m0, n0, D); n0 += 128; }
      else { probe_chunk<64>(p, smem_u32(sa), smem_u32(sb), m0, n0, D); n0 += 64; }
    }
}

// ------------------------------------------------------------------------------------ K2: heads forward
namespace k2 {
constexpr int BM = 128, BN = 128, BK = 64;
constexpr int kThreads = 256;                                     // two warpgroups, 64 cells each
constexpr uint32_t kABytes = BM * BK * 2, kBBytes = BN * BK * 2;  // 16 KB, 16 KB
constexpr uint32_t kSmemBytes = kABytes + kBBytes + 1024;

struct Params {
  int B, G, n_heads;
  int kind[3];                 // EPI_MEAN_ACT / EPI_DISP_ACT / EPI_SIGMOID per packed head slot
  int m_tiles, n_tiles_per_head;
  const float* bias[3];        // per head slot: float[G]
  const float* row_scale;      // [B] or nullptr
  float* out[3]; int64_t ld_out;
};

// One 128 x 128 output tile per CTA (grid = m tiles fastest, so that consecutive CTAs share the weight tile in L2).
// K = 64: the whole operand pair arrives with one TMA transaction; two CTAs per SM overlap one tile's loads with the
// other's MMA and stores.  The kernel is bound by the fp32 output stores (128 flop per 4-byte element): every warp
// store instruction covers 8 rows x 32 contiguous bytes, i.e. whole sectors.
__global__ void __launch_bounds__(kThreads, 2)
heads_fwd_kernel(const __grid_constant__ CUtensorMap map_h, const __grid_constant__ CUtensorMap map_w0,
                 const __grid_constant__ CUtensorMap map_w1, const __grid_constant__ CUtensorMap map_w2, const Params p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  __shared__ uint64_t full_bar;
  const int mt = blockIdx.x % p.m_tiles, r = blockIdx.x / p.m_tiles;
  const int nt = r % p.n_tiles_per_head, hs = r / p.n_tiles_per_head;
  if (threadIdx.x == 0) {
    mbar_init(&full_bar, 1);
    fence_barrier_init();
    const CUtensorMap* mw = hs == 0 ? &map_w0 : (hs == 1 ? &map_w1 : &map_w2);
    mbar_expect_tx(&full_bar, kABytes + kBBytes);
    tma_load_2d(smem, &map_h, 0, mt * BM, &full_bar);
    // B = the head kernel in its Keras layout [64 k][G genes] (bf16 shadow): two 64-gene boxes, MN-major
    tma_load_2d(smem + kABytes, mw, nt * BN, 0, &full_bar);
    tma_load_2d(smem + kABytes + kBBytes / 2, mw, nt * BN + 64, 0, &full_bar);
  }
  __syncthreads();
  const int wg = threadIdx.x >> 7, w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
  // bias / row scale of this thread's fragment, fetched while the operands are in flight
  const int col0 = nt * BN + 2 * (l & 3);
  const int row0 = mt * BM + wg * 64 + 16 * w + (l >> 2);
  const float* bias = p.bias[hs];
  const int kind = p.kind[hs];
  float2 bz[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) bz[c] = (col0 + 8 * c < p.G) ? *reinterpret_cast<const float2*>(bias + col0 + 8 * c) : make_float2(0.f, 0.f);
  float rs[2] = {1.f, 1.f};
  if (kind == EPI_MEAN_ACT && p.row_scale) {
    if (row0 < p.B) rs[0] = p.row_scale[row0];
    if (row0 + 8 < p.B) rs[1] = p.row_scale[row0 + 8];
  }
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  mbar_wait(&full_bar, 0);
  const uint32_t a0 = smem_u32(smem) + wg * 64 * 128, b0 = smem_u32(smem) + kABytes;
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < BK / 16; ++k)
    wgmma_m64n128k16<0, 1>(acc, make_smem_desc(a0 + k * 32, 0, 1024), make_smem_desc(b0 + k * 2048, kBBytes / 2, 1024), k > 0);
  wgmma_commit();
  wgmma_wait<0>();
  acc_fence(acc);
  float* out = p.out[hs];
  auto emit = [&](auto act) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + 8 * h;
      if (row >= p.B) continue;
      float* orow = out + (int64_t)row * p.ld_out;
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        const int col = col0 + 8 * c;
        if (col < p.G)      // G % 8 == 0: the pair is all in or all out
          *reinterpret_cast<float2*>(orow + col) =
              make_float2(act(acc[4 * c + 2 * h] + bz[c].x, rs[h]), act(acc[4 * c + 2 * h + 1] + bz[c].y, rs[h]));
      }
    }
  };
  if (kind == EPI_MEAN_ACT) emit([](float z, float s) { return act_mean(z) * s; });
  else if (kind == EPI_DISP_ACT) emit([](float z, float) { return act_disp(z); });
  else emit([](float z, float) { return act_sigmoid(z); });
}
}  // namespace k2

// Host launcher.  Hb: bf16 [B x 64]; W[i]: bf16 [64 x G] (Keras layout) and bias[i]: float[G] per head slot.
int heads_fwd_tc(const __nv_bfloat16* Hb, int B, const __nv_bfloat16* const W[3], const float* const bias[3], int G,
                 int n_heads, const int kind[3], const float* row_scale, float* const out[3], int64_t ld_out, int sm_count,
                 cudaStream_t s) {
  using namespace k2;
  if (ld_out % 4 != 0 || G % 8 != 0) { set_error("heads_fwd_tc: G must be a multiple of 8 and ld_out of 4 (TMA strides)"); return DCA_ERR_BAD_ARG; }
  CUtensorMap mh, mw[3];
  DCA_TRY(make_tensor_map_2d(&mh, Hb, 2, 1, (uint64_t)B, 64, 64, BM, BK, 1));
  for (int i = 0; i < 3; ++i)
    DCA_TRY(make_tensor_map_2d(&mw[i], W[i < n_heads ? i : 0], 2, 1, 64, (uint64_t)G, (uint64_t)G, 64, 64, 1));
  Params p;
  p.B = B; p.G = G; p.n_heads = n_heads;
  for (int i = 0; i < 3; ++i) { const int k = i < n_heads ? i : 0; p.kind[i] = kind[i]; p.bias[i] = bias[k]; p.out[i] = out[k]; }
  p.m_tiles = cdiv(B, BM); p.n_tiles_per_head = cdiv(G, BN);
  p.row_scale = row_scale; p.ld_out = ld_out;
  (void)sm_count;
  static bool attr_set = false;
  if (!attr_set) {
    DCA_CUDA_OK(cudaFuncSetAttribute(heads_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes));
    attr_set = true;
  }
  const int grid = p.m_tiles * p.n_tiles_per_head * n_heads;
  heads_fwd_kernel<<<grid, kThreads, kSmemBytes, s>>>(mh, mw[0], mw[1], mw[2], p);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

}  // namespace tc

Engine::~Engine() {
  comm_destroy();
  for (auto e : prof.ev) cudaEventDestroy(e);
  for (auto& g : graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
  if (hs.copy) cudaStreamDestroy(hs.copy);
  if (hs.expand) cudaStreamDestroy(hs.expand);
  for (int k = 0; k < 3; ++k) {
    if (hs.ready[k]) cudaEventDestroy(hs.ready[k]);
    if (hs.step_done[k]) cudaEventDestroy(hs.step_done[k]);
  }
  for (int k = 0; k < 2; ++k) {
    if (hs.h2d_done[k]) cudaEventDestroy(hs.h2d_done[k]);
    if (hs.cnt_free[k]) cudaEventDestroy(hs.cnt_free[k]);
  }
}

}  // namespace dca

// ------------------------------------------------------------------------------------ C ABI (test / profiling entry points)
using namespace dca;

extern "C" int dca_tc_probe(const void* A, int32_t a_rows, int32_t a_cols, const void* Bm, int32_t b_rows, int32_t b_cols,
                            int32_t a_mn_major, int32_t b_mn_major, int32_t M, int32_t N, int32_t K,
                            int32_t a_lbo, int32_t a_sbo, int32_t b_lbo, int32_t b_sbo, float* D, void* stream) {
  using namespace tc;
  if (M != 128 || N % 64 != 0 || N < 64 || N > 256 || K % 64 != 0 || K <= 0 || K > 256) {
    set_error("dca_tc_probe: need M=128, N%%64==0 (64..256), K%%64==0 (<=256)"); return DCA_ERR_BAD_ARG;
  }
  ProbeParams p{};
  p.a_mn = a_mn_major; p.b_mn = b_mn_major; p.M = M; p.N = N; p.K = K;
  CUtensorMap ma, mb;
  auto setup = [&](int mn, int mn_extent, int rows, int cols, const void* base, CUtensorMap* map, int& boxes, int& box_bytes,
                   int& c0, int& c1, uint32_t& lbo, uint32_t& sbo, uint32_t& kstep, uint32_t& kb_steps, uint32_t& kb_bytes,
                   uint32_t& mn64_bytes, int lbo_o, int sbo_o) -> int {
    if (!mn) {   // K-major: storage [mn_extent rows][K cols]; one box per 64-wide K block
      if (rows != mn_extent || cols != K) { set_error("dca_tc_probe: K-major operand must be [MN x K]"); return DCA_ERR_BAD_ARG; }
      DCA_TRY(make_tensor_map_2d(map, base, 2, 1, rows, cols, cols, mn_extent, 64, 1));
      boxes = K / 64; box_bytes = mn_extent * 128; c0 = 64; c1 = 0;
      lbo = 0; sbo = 1024; kstep = 32; kb_steps = 4; kb_bytes = box_bytes; mn64_bytes = 64 * 128;
    } else {     // MN-major: storage [K rows][mn_extent cols]; one box per 64-wide MN block
      if (rows != K || cols != mn_extent || mn_extent % 64) { set_error("dca_tc_probe: MN-major operand must be [K x MN], MN%%64==0"); return DCA_ERR_BAD_ARG; }
      DCA_TRY(make_tensor_map_2d(map, base, 2, 1, rows, cols, cols, K, 64, 1));
      boxes = mn_extent / 64; box_bytes = K * 128; c0 = 64; c1 = 0;
      lbo = box_bytes; sbo = 1024; kstep = 2048; kb_steps = 1u << 30; kb_bytes = 0; mn64_bytes = box_bytes;
    }
    if (lbo_o >= 0) lbo = lbo_o;
    if (sbo_o >= 0) sbo = sbo_o;
    return DCA_OK;
  };
  DCA_TRY(setup(a_mn_major, M, a_rows, a_cols, A, &ma, p.a_boxes, p.a_box_bytes, p.a_box_c0, p.a_box_c1, p.a_lbo, p.a_sbo,
                p.a_kstep, p.a_kblock_steps, p.a_kblock_bytes, p.a_mn64_bytes, a_lbo, a_sbo));
  DCA_TRY(setup(b_mn_major, N, b_rows, b_cols, Bm, &mb, p.b_boxes, p.b_box_bytes, p.b_box_c0, p.b_box_c1, p.b_lbo, p.b_sbo,
                p.b_kstep, p.b_kblock_steps, p.b_kblock_bytes, p.b_mn64_bytes, b_lbo, b_sbo));
  const size_t smem = (size_t)p.a_boxes * p.a_box_bytes + (size_t)p.b_boxes * p.b_box_bytes + 1024;
  DCA_CUDA_OK(cudaFuncSetAttribute(tc_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  tc_probe_kernel<<<1, 128, smem, (cudaStream_t)stream>>>(ma, mb, p, D);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

extern "C" int dca_tc_heads_fwd(const void* Hb, int32_t batch, const void* Wk, const float* bias, int32_t genes,
                                int32_t n_heads, const int32_t kind[3], const float* row_scale, float* out0, float* out1,
                                float* out2, int64_t ld_out, void* stream) {
  if (!Hb || !Wk || !bias || batch <= 0 || genes <= 0 || n_heads < 1 || n_heads > 3 || !out0) {
    set_error("dca_tc_heads_fwd: bad argument"); return DCA_ERR_BAD_ARG;
  }
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int k[3] = {kind[0], n_heads > 1 ? kind[1] : 0, n_heads > 2 ? kind[2] : 0};
  float* outs[3] = {out0, out1, out2};
  const __nv_bfloat16* W[3]; const float* b[3];
  for (int i = 0; i < 3; ++i) {
    const int j = i < n_heads ? i : 0;
    W[i] = (const __nv_bfloat16*)Wk + (size_t)j * 64 * genes; b[i] = bias + (size_t)j * genes;
  }
  return tc::heads_fwd_tc((const __nv_bfloat16*)Hb, batch, W, b, genes, n_heads, k, row_scale, outs, ld_out, sms,
                          (cudaStream_t)stream);
}
