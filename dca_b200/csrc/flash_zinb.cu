// Fused head forward -> ZINB loss + gradient -> head backward for the conditional-dispersion ZINB model
// (SURVEY.md 8f-2; replaces K2 + K3 + K4 of one training step, dca/network.py:369-381 + dca/loss.py:122-148 +
// their autodiff).  The B x 3G head activations and their gradients never reach HBM:
//
//   per tile (128 cells x 64 genes, all three heads):
//     MMA1   Z_h[128 x 64] = H3[128 x 64] . W_h[64 x 64]                     -> registers (fp32, wgmma)
//     elements  z + bias -> MeanAct / DispAct / sigmoid -> ZINB NLL and d/dz (zinb_math.cuh, the arithmetic of the
//               stand-alone loss kernel) -> dZ bf16 written into shared memory in the SWIZZLE_128B operand layout
//     MMA2   dH3[128 x 64]  = sum_h dZ_h[128 x 64] . W_h^T                    (dZ as K-major A)
//     MMA3   dW_h[64g x 64] += dZ_h^T . H3, db_h += dZ_h^T . 1                (the same bytes as MN-major A)
//   HBM traffic: the count tile (4 B / element) in, 1/64 of it out.  dH3 leaves per tile by TMA reduce-add,
//   dW / db stay in shared memory over all cell blocks of a gene tile and are added to the gradient buffer once.
#include "engine.h"
#include "tc_common.cuh"
#include "head_act.cuh"
#include "zinb_math.cuh"

namespace dca {
namespace tc {
namespace fz {

constexpr int kThreads = 256;                                  // two warpgroups, 64 cells of the tile each
constexpr uint32_t kHBytes = 128 * 64 * 2;                     // [128 cells x 64 feats] bf16
constexpr uint32_t kWBox = 64 * 64 * 2, kWBytes = 3 * kWBox;   // per head [64 feats x 64 genes] bf16
constexpr uint32_t kZBox = 128 * 64 * 2, kZBytes = 3 * kZBox;  // per head dZ [128 cells x 64 genes] bf16
constexpr uint32_t kOutBytes = 128 * 64 * 4;                   // dH3 staging [128 x 64] fp32
constexpr uint32_t kDwFloats = 3 * 64 * 64;                    // dW accumulators [head][feat][gene] fp32
constexpr uint32_t kOffH = 0, kOffW = kOffH + 2 * kHBytes, kOffZ = kOffW + kWBytes, kOffO = kOffZ + kZBytes,
                   kOffDw = kOffO + kOutBytes, kOffDb = kOffDw + kDwFloats * 4, kOffOnes = kOffDb + 3 * 64 * 4,
                   kSmemUsed = kOffOnes + 2048;
constexpr uint32_t kSmemBytes = kSmemUsed + 1024;

struct Params {
  int B, G, n_cb, n_gt, total_tiles;
  const float* Y; int64_t ldy; const int32_t* rows; const float* sf;
  const float* bias[3];
  float* dW[3]; int64_t dW_ld; float* db[3];
  float ridge, inv_n;
  const float* lf_global;
  double* loss_partial; unsigned* counter; double* loss_sum; const double* penalty; float* loss_slot; double* epoch_acc;
  int batch;
};

// NB branch of one element; deliberately not inlined (one copy of the lgamma / digamma code keeps the element loop
// inside the instruction cache)
__device__ __noinline__ zmath::Raw1 nb_item(float y, float mu, float th, float pi, const float* lf) {
  return zmath::zinb_nb_raw<zmath::FastOps>(y, mu, th, pi, lf);       // raw derivatives, see zinb_math.cuh
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

// One CTA walks a contiguous range of tiles; tile t -> gene tile t / n_cb, cell block t % n_cb (cells fastest, so the
// weight tile and the dW accumulators stay put over a run of cell blocks = one "segment").  Per tile:
//   MMA1 (wgmma, registers)  z_h[64 cells x 64 genes] = H3 . W_h for the three heads, per warpgroup
//   element loop             activations, ZINB NLL and d/dz of the thread's 2 x 16 element pairs (the f32x2
//                            formulation of the stand-alone loss kernel) -> dZ_h bf16 into shared memory in the
//                            SWIZZLE_128B operand layout
//   MMA2                     dH3 = sum_h dZ_h . W_h^T (dZ as K-major A) -> staging tile -> TMA reduce-add
//   MMA3                     dW_h^T += dZ_h^T . H3, db_h += dZ_h^T . 1 (the same bytes as MN-major A; the two
//                            warpgroups split the cells) -> shared-memory fp32 accumulators, added to the gradient
//                            buffer once per segment
__global__ void __launch_bounds__(kThreads, 1)
flash_zinb_kernel(const __grid_constant__ CUtensorMap map_h, const __grid_constant__ CUtensorMap map_w0,
                  const __grid_constant__ CUtensorMap map_w1, const __grid_constant__ CUtensorMap map_w2,
                  const __grid_constant__ CUtensorMap map_o, const Params p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* s_h = smem + kOffH; uint8_t* s_w = smem + kOffW; uint8_t* s_z = smem + kOffZ;
  float* s_o = reinterpret_cast<float*>(smem + kOffO);
  float* s_dw = reinterpret_cast<float*>(smem + kOffDw);
  float* s_db = reinterpret_cast<float*>(smem + kOffDb);
  uint8_t* s_ones = smem + kOffOnes;
  __shared__ uint64_t h_full[2], w_full;
  __shared__ float lf[zmath::kLogFactN];
  __shared__ double red[kThreads / 32];
  __shared__ int s_last;

  const int t0 = (int)((long long)p.total_tiles * blockIdx.x / gridDim.x);
  const int t1 = (int)((long long)p.total_tiles * (blockIdx.x + 1) / gridDim.x);
  auto issue_h = [&](int t, int buf) {
    mbar_expect_tx(&h_full[buf], kHBytes);
    tma_load_2d(s_h + buf * kHBytes, &map_h, 0, (t % p.n_cb) * 128, &h_full[buf]);
  };
  auto issue_w = [&](int t) {
    const int gt = t / p.n_cb;
    mbar_expect_tx(&w_full, kWBytes);
    tma_load_2d(s_w, &map_w0, gt * 64, 0, &w_full);
    tma_load_2d(s_w + kWBox, &map_w1, gt * 64, 0, &w_full);
    tma_load_2d(s_w + 2 * kWBox, &map_w2, gt * 64, 0, &w_full);
  };
  if (threadIdx.x == 0) {
    mbar_init(&h_full[0], 1); mbar_init(&h_full[1], 1); mbar_init(&w_full, 1);
    fence_barrier_init();
    if (t0 < t1) { issue_w(t0); issue_h(t0, 0); }
  }
  if (threadIdx.x < zmath::kLogFactN) lf[threadIdx.x] = p.lf_global[threadIdx.x];
  for (int i = threadIdx.x; i < 2048 / 4; i += kThreads) reinterpret_cast<uint32_t*>(s_ones)[i] = 0x3F803F80u;   // bf16 ones
  for (int i = threadIdx.x; i < (int)kDwFloats; i += kThreads) s_dw[i] = 0.f;
  for (int i = threadIdx.x; i < 3 * 64; i += kThreads) s_db[i] = 0.f;
  fence_proxy_async_smem();
  __syncthreads();

  using Ops = zmath::FastOps;
  using namespace zmath;
  const int wg = threadIdx.x >> 7, w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
  const int frow = 16 * w + (l >> 2), fcol = 2 * (l & 3);            // fragment origin (see tc_common.cuh)
  const uint32_t wb = smem_u32(s_w), zb = smem_u32(s_z), ob = smem_u32(s_ones);
  float lsum = 0.f, lsum_lg = 0.f;        // NLL of the NB elements (+ ridge) | sum of lg2(D) over the zero counts
  uint32_t seg = 0;
  for (int t = t0, ti = 0; t < t1; ++t, ++ti) {
    const int gt = t / p.n_cb, cb = t % p.n_cb;
    const bool new_seg = (t == t0 || cb == 0);
    if (threadIdx.x == 0) {
      if (new_seg && t != t0) issue_w(t);                              // the previous segment's MMAs are complete
      if (t + 1 < t1) issue_h(t + 1, (ti + 1) & 1);                     // its buffer was released at the end of tile ti-1
    }
    if (new_seg) { mbar_wait(&w_full, seg & 1); ++seg; }
    const int hbuf = ti & 1;
    mbar_wait(&h_full[hbuf], (ti >> 1) & 1);
    const uint32_t hb = smem_u32(s_h + hbuf * kHBytes);

    // ---- MMA1: pre-activations of the three heads, rows 64*wg.. of the tile
    float zm[32], zd[32], zp[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { zm[i] = 0.f; zd[i] = 0.f; zp[i] = 0.f; }
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t da = make_smem_desc(hb + wg * 64 * 128 + k * 32, 0, 1024);
      wgmma_m64n64k16<0, 1>(zm, da, make_smem_desc(wb + k * 2048, 0, 1024), k > 0);
      wgmma_m64n64k16<0, 1>(zd, da, make_smem_desc(wb + kWBox + k * 2048, 0, 1024), k > 0);
      wgmma_m64n64k16<0, 1>(zp, da, make_smem_desc(wb + 2 * kWBox + k * 2048, 0, 1024), k > 0);
    }
    wgmma_commit();

    // ---- per-row operands while the MMAs run
    int yr[2]; float sfv[2]; bool vrow[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int grow = cb * 128 + wg * 64 + frow + 8 * h;
      vrow[h] = grow < p.B; yr[h] = 0; sfv[h] = 1.0f;
      if (vrow[h]) { yr[h] = p.rows ? p.rows[grow] : grow; sfv[h] = p.sf ? p.sf[yr[h]] : 1.0f; }
    }
    wgmma_wait<0>();
    acc_fence(zm); acc_fence(zd); acc_fence(zp);

    // ---- element loop: pair c of row half h = columns 8*c + fcol, +1 of row frow + 8*h
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const int col = 8 * c + fcol, g = gt * 64 + col;
      const bool cols_in = g < p.G;                                      // G % 8 == 0: the pair is all in or all out
      float2 bm = make_float2(0.f, 0.f), bd = bm, bp = bm;
      if (cols_in) {
        bm = *reinterpret_cast<const float2*>(p.bias[0] + g);
        bd = *reinterpret_cast<const float2*>(p.bias[1] + g);
        bp = *reinterpret_cast<const float2*>(p.bias[2] + g);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = 4 * c + 2 * h;
        const bool active = vrow[h] && cols_in;
        float2 y = make_float2(0.f, 0.f);
        if (active) y = *reinterpret_cast<const float2*>(p.Y + (int64_t)yr[h] * p.ldy + g);
        const float2 m = make_float2(act_mean(zm[i] + bm.x), act_mean(zm[i + 1] + bm.y));
        const float2 d = make_float2(act_disp(zd[i] + bd.x), act_disp(zd[i + 1] + bd.y));
        const float2 pi = make_float2(act_sigmoid(zp[i] + bp.x), act_sigmoid(zp[i + 1] + bp.y));
        const float2 mu = mul2(m, splat(sfv[h]));                                          // dca/layers.py:85
        Raw2 z = zinb_zero_pair<Ops>(mu, d, pi);
        const Fin2 f = finish_factors_pair<Ops, true>(m, d, pi, p.inv_n);
        const bool nz0 = active && !(y.x < 1e-8f), nz1 = active && !(y.y < 1e-8f);       // loss.py:138
        if (nz0) { const Raw1 e = nb_item(y.x, mu.x, d.x, pi.x, lf); lsum += e.loss; z.gmu.x = e.gmu; z.dth.x = e.dth; z.dpi.x = e.dpi; }
        if (nz1) { const Raw1 e = nb_item(y.y, mu.y, d.y, pi.y, lf); lsum += e.loss; z.gmu.y = e.gmu; z.dth.y = e.dth; z.dpi.y = e.dpi; }
        lsum_lg += ((active && !nz0) ? z.lgD.x : 0.f) + ((active && !nz1) ? z.lgD.y : 0.f);
        if (p.ridge != 0.f) {                                                              // loss.py:139-140
          if (active) lsum += p.ridge * (pi.x * pi.x + pi.y * pi.y);
          z.dpi = fma2(splat(2.0f * p.ridge), pi, z.dpi);
        }
        const float2 msk = splat(active ? 1.0f : 0.0f);        // rows / genes outside the matrix contribute exact zeros
        const float2 gm = mul2(mul2(z.gmu, f.fm), msk), gd = mul2(mul2(z.dth, f.fd), msk), gp = mul2(mul2(z.dpi, f.fp), msk);
        // SWIZZLE_128B operand layout: 16-byte chunk (8 genes) c ^ (row % 8) of the row's 128 bytes
        const int row = wg * 64 + frow + 8 * h;
        uint8_t* dst = s_z + row * 128 + ((c ^ (row & 7)) << 4) + fcol * 2;
        *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(gm.x, gm.y);
        *reinterpret_cast<uint32_t*>(dst + kZBox) = pack_bf16x2(gd.x, gd.y);
        *reinterpret_cast<uint32_t*>(dst + 2 * kZBox) = pack_bf16x2(gp.x, gp.y);
      }
    }
    fence_proxy_async_smem();
    if (threadIdx.x == 0) bulk_wait_read<0>();                           // the previous dH3 reduce has read the staging tile
    __syncthreads();

    // ---- MMA2: dH3 rows 64*wg.. = sum_h dZ_h . W_h^T
    {
      float dh[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) dh[i] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int h = 0; h < 3; ++h)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_m64n64k16<0, 0>(dh, make_smem_desc(zb + h * kZBox + wg * 64 * 128 + k * 32, 0, 1024),
                                make_smem_desc(wb + h * kWBox + k * 32, 0, 1024), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(dh);
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int row = wg * 64 + frow + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + fcol;
        *reinterpret_cast<float2*>(s_o + row * 64 + col) = make_float2(dh[i], dh[i + 1]);
      }
    }
    // ---- MMA3: dW_h^T [64 genes x 64 feats] and column sums, cells 64*wg.. of the tile
#pragma unroll 1
    for (int h = 0; h < 3; ++h) {
      float dw[32], cs[8];
#pragma unroll
      for (int i = 0; i < 32; ++i) dw[i] = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) cs[i] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int kk = wg * 4 + k;
        const uint64_t da = make_smem_desc(zb + h * kZBox + kk * 2048, 0, 1024);
        wgmma_m64n64k16<1, 1>(dw, da, make_smem_desc(hb + kk * 2048, 0, 1024), 1u);
        wgmma_m64n16k16<1, 0>(cs, da, make_smem_desc(ob + k * 32, 0, 1024), 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(dw); acc_fence(cs);
      float* acc = s_dw + h * 4096;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int gl = frow + 8 * ((i >> 1) & 1), f = 8 * (i >> 2) + fcol + (i & 1);
        atomicAdd(acc + f * 64 + gl, dw[i]);
      }
      if ((l & 3) == 0) { atomicAdd(s_db + h * 64 + frow, cs[0]); atomicAdd(s_db + h * 64 + frow + 8, cs[2]); }
    }
    fence_proxy_async_smem();
    __syncthreads();                                   // dZ, H and W buffers free; staging tile and accumulators complete
    if (threadIdx.x == 0) { tma_reduce_add_2d(&map_o, 0, cb * 128, s_o); bulk_commit(); }
    const bool last = (t + 1 == t1) || ((t + 1) % p.n_cb == 0);
    if (last) {                                        // end of the segment: dW / db of this gene tile -> gradient buffer
      for (int idx = threadIdx.x; idx < (int)kDwFloats; idx += kThreads) {
        const int h = idx >> 12, f = (idx >> 6) & 63, g = gt * 64 + (idx & 63);
        if (g < p.G) atomicAdd(p.dW[h] + (int64_t)f * p.dW_ld + g, s_dw[idx]);
        s_dw[idx] = 0.f;
      }
      for (int idx = threadIdx.x; idx < 3 * 64; idx += kThreads) {
        const int h = idx >> 6, g = gt * 64 + (idx & 63);
        if (g < p.G) atomicAdd(p.db[h] + g, s_db[idx]);
        s_db[idx] = 0.f;
      }
      __syncthreads();
    }
  }
  if (threadIdx.x == 0) bulk_wait<0>();

  // ---- loss: CTA partial, the last CTA folds all partials in a fixed order and finalises (as in zinb_loss.cu)
  constexpr unsigned kFull = 0xffffffffu;
  double dsum = (double)lsum - (double)zmath::kLn2 * (double)lsum_lg;        // -log D = -ln2 * lg2 D
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dsum += __shfl_xor_sync(kFull, dsum, o);
  if (l == 0) red[threadIdx.x >> 5] = dsum;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tsum = 0.0;
#pragma unroll
    for (int i = 0; i < kThreads / 32; ++i) tsum += red[i];
    p.loss_partial[blockIdx.x] = tsum;
    __threadfence();
    const unsigned done = atomicAdd(p.counter, 1u);
    s_last = (done == gridDim.x - 1);
    if (s_last) *p.counter = 0;                                       // self-resetting
  }
  __syncthreads();
  if (s_last && threadIdx.x < 32) {
    __threadfence();
    double a = 0.0;
    for (int i = l; i < (int)gridDim.x; i += 32) a += __ldcg(p.loss_partial + i);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(kFull, a, o);
    if (l == 0) {
      *p.loss_sum = a;
      if (p.loss_slot) {
        double lv = a * (double)p.inv_n;
        if (lv != lv) lv = INFINITY;                                  // _nan2inf, dca/loss.py:148
        if (p.penalty) lv += *p.penalty;
        const float lf32 = (float)lv;
        p.loss_slot[0] = lf32;
        p.loss_slot[1] = (isfinite(lf32)) ? 0.f : 1.f;
        if (p.epoch_acc) { p.epoch_acc[0] += lv * (double)p.batch; p.epoch_acc[1] += (double)p.batch; }
      }
    }
  }
}

}  // namespace fz

// H3: bf16 [B x 64]; W[h]: bf16 Keras-layout head kernels [64 x G] (mean, dispersion, pi); bias[h]: float[G];
// Y: float counts (row gather through rows[], ldy); outputs: dH3 (+=, fp32 [B x 64]), dW[h] (+=, [64 x G]),
// db[h] (+=, [G]), loss partial fold into loss_sum / loss_slot / epoch_acc like zinb_loss_fwd_bwd.
int flash_zinb_tc(const __nv_bfloat16* H3, int B, int G, const __nv_bfloat16* const W[3], const float* const bias[3],
                  const float* Y, int64_t ldy, const int32_t* rows, const float* sf, float ridge, float inv_n,
                  float* dH3, float* const dW[3], float* const db[3], void* ws, size_t ws_bytes, double* loss_sum,
                  const double* penalty, float* loss_slot, double* epoch_acc, int batch, const float* lf_dev, int sm_count,
                  cudaStream_t s) {
  using namespace fz;
  if (G % 8 != 0 || ldy % 4 != 0 || (reinterpret_cast<uintptr_t>(Y) & 15) != 0) {
    set_error("flash_zinb_tc: needs G %% 8 == 0 and 16-byte aligned count rows"); return DCA_ERR_BAD_ARG;
  }
  if (!ws || ws_bytes < sizeof(double) * 65536 + 256) { set_error("flash_zinb_tc: workspace too small"); return DCA_ERR_BAD_ARG; }
  CUtensorMap mh, mw[3], mo;
  DCA_TRY(make_tensor_map_2d(&mh, H3, 2, 1, (uint64_t)B, 64, 64, 128, 64, 1));
  for (int i = 0; i < 3; ++i) DCA_TRY(make_tensor_map_2d(&mw[i], W[i], 2, 1, 64, (uint64_t)G, (uint64_t)G, 64, 64, 1));
  DCA_TRY(make_tensor_map_2d(&mo, dH3, 4, 0, (uint64_t)B, 64, 64, 128, 64, 0));
  Params p{};
  p.B = B; p.G = G; p.n_cb = cdiv(B, 128); p.n_gt = cdiv(G, 64); p.total_tiles = p.n_cb * p.n_gt;
  p.Y = Y; p.ldy = ldy; p.rows = rows; p.sf = sf;
  for (int i = 0; i < 3; ++i) { p.bias[i] = bias[i]; p.dW[i] = dW[i]; p.db[i] = db[i]; }
  p.dW_ld = G; p.ridge = ridge; p.inv_n = inv_n; p.lf_global = lf_dev;
  p.loss_partial = reinterpret_cast<double*>(ws);
  p.counter = reinterpret_cast<unsigned*>(reinterpret_cast<char*>(ws) + sizeof(double) * 65536);
  p.loss_sum = loss_sum; p.penalty = penalty; p.loss_slot = loss_slot; p.epoch_acc = epoch_acc; p.batch = batch;
  static bool attr = false;
  if (!attr) { DCA_CUDA_OK(cudaFuncSetAttribute(flash_zinb_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes)); attr = true; }
  const int grid = p.total_tiles < sm_count ? p.total_tiles : sm_count;
  flash_zinb_kernel<<<grid, kThreads, kSmemBytes, s>>>(mh, mw[0], mw[1], mw[2], mo, p);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

}  // namespace tc
}  // namespace dca
