// On-device preprocessing of raw counts: dca/io.py:88-111 (scanpy's filter_genes / filter_cells, normalize_per_cell,
// log1p and scale, restated in dca_b200/io.py:normalize) computed in HBM from the fp32 count matrix Y the training step
// reads anyway.  Every kernel streams over Y; none uses atomics.  Reductions over cells write per-CTA partials into
// workspace slots and a fold kernel adds them in slot order, so two calls with the same shapes are bit-identical.
//
// Arithmetic (include/dca_b200.h, "preprocessing"): sf64 = n_counts / median (fp64), q = float((double)y / sf64),
// l = float(log1p((double)q)) (rounded from the double log1p; NumPy's float32 log1p is not), gene moments in fp64
// (two passes, as NumPy's var), X = float(((double)l - mean) / std), bf16 X = __float2bfloat16_rn of that float.
#include <cmath>
#include "dca_internal.cuh"

namespace dca {
namespace {

constexpr int kThreads = 256;          // 8 warps
constexpr int kGenesPerCta = 256;      // lane owns genes g0 + 32k, k < 8: every load of a warp is 128 contiguous bytes
constexpr int kPerLane = kGenesPerCta / 32;
constexpr int kTargetCtas = 1056;      // column-pass grid size aimed at (8 x 132 SMs); depends on N and G only

enum { PRE_SF = DCA_PRE_SIZE_FACTORS, PRE_LOG = DCA_PRE_LOG1P, PRE_SCALE = DCA_PRE_SCALE };

struct ColPlan {
  int gblocks, slices, rows_per_slice;
  size_t gene_part, cell_part, bad_part;   // byte offsets in the workspace
  size_t bytes;
};

inline size_t align256(size_t v) { return (v + 255) / 256 * 256; }

ColPlan col_plan(int64_t N, int G) {
  ColPlan p;
  p.gblocks = cdiv(G, kGenesPerCta);
  int s = cdiv(kTargetCtas, p.gblocks);
  s = (int)std::min<int64_t>(s, std::max<int64_t>(1, (N + 63) / 64));
  p.rows_per_slice = (int)((N + s - 1) / s);
  p.slices = (int)((N + p.rows_per_slice - 1) / p.rows_per_slice);
  p.gene_part = 0;
  p.cell_part = align256((size_t)p.slices * G * sizeof(double));
  p.bad_part = p.cell_part + align256((size_t)p.gblocks * N * sizeof(double));
  p.bytes = p.bad_part + align256((size_t)p.slices * p.gblocks * sizeof(long long));
  return p;
}

// The per-element input transform: l of the header's definition (y when no flag is set).
__device__ __forceinline__ float log_value(float y, double sf64, int flags) { return pre_log_value(y, sf64, flags); }

__device__ __forceinline__ double row_sf(const double* n_counts, double median, int r, int flags) {
  return (flags & PRE_SF) ? n_counts[r] / median : 1.0;
}

// One row of a warp's share of a column pass: lane owns genes g0 + 32k.  MODE 0 adds y to acc, counts bad entries and
// writes the row's sum over the 256 genes of the block to *cell_out (lane 0); MODE 1 adds l; MODE 2 adds (l - mu)^2.
template <int MODE>
__device__ __forceinline__ void col_row(const float* __restrict__ row, int g0, int G, int lane, double sf, int flags,
                                        const double (&mu)[kPerLane], double (&acc)[kPerLane], long long& bad,
                                        double* cell_out) {
  float v[kPerLane];
#pragma unroll
  for (int k = 0; k < kPerLane; ++k) v[k] = (g0 + 32 * k < G) ? __ldg(row + g0 + 32 * k) : 0.f;
  if (MODE == 0) {
    double rs = 0.0;
#pragma unroll
    for (int k = 0; k < kPerLane; ++k) {
      if (g0 + 32 * k < G) {
        const double d = (double)v[k];
        acc[k] += d;
        rs += d;
        bad += !(isfinite(v[k]) && v[k] >= 0.f && v[k] == floorf(v[k]));
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, off);
    if (lane == 0) *cell_out = rs;
  } else {
#pragma unroll
    for (int k = 0; k < kPerLane; ++k) {
      if (g0 + 32 * k < G) {
        const float l = log_value(v[k], sf, flags);
        if (MODE == 1) {
          acc[k] += (double)l;
        } else {
          const double d = (double)l - mu[k];
          acc[k] = __dadd_rn(acc[k], __dmul_rn(d, d));     // no FMA contraction: (l - mean)^2 rounded, then added
        }
      }
    }
  }
}

// One pass over a [rows_per_slice x 256-gene] tile per CTA.
//   MODE 0: per-gene sum of y, per-(gene block, cell) sum of y, count of entries that are not finite non-negative integers
//   MODE 1: per-gene sum of l
//   MODE 2: per-gene sum of (l - mean)^2
// Warp w takes rows r0 + w, r0 + w + 8, ...; the 8 warps' gene sums are added in warp order.
template <int MODE>
__global__ void __launch_bounds__(kThreads) col_pass_kernel(const float* __restrict__ Y, int64_t ldy, int N, int G,
                                                            int rows_per_slice, const double* __restrict__ n_counts,
                                                            double median, int flags, const double* __restrict__ mean,
                                                            double* __restrict__ gene_part, double* __restrict__ cell_part,
                                                            long long* __restrict__ bad_part) {
  __shared__ double sm[kThreads / 32][kGenesPerCta];
  __shared__ long long sbad[kThreads / 32];
  const int gb = blockIdx.x, slice = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g0 = gb * kGenesPerCta + lane;
  const int r0 = slice * rows_per_slice, r1 = (int)min((int64_t)N, (int64_t)r0 + rows_per_slice);
  double acc[kPerLane], mu[kPerLane];
#pragma unroll
  for (int k = 0; k < kPerLane; ++k) {
    acc[k] = 0.0;
    mu[k] = (MODE == 2 && g0 + 32 * k < G) ? mean[g0 + 32 * k] : 0.0;
  }
  long long bad = 0;
  for (int r = r0 + warp; r < r1; r += kThreads / 32)
    col_row<MODE>(Y + (int64_t)r * ldy, g0, G, lane, MODE ? row_sf(n_counts, median, r, flags) : 1.0, flags, mu, acc, bad,
                  cell_part + (int64_t)gb * N + r);
#pragma unroll
  for (int k = 0; k < kPerLane; ++k) sm[warp][32 * k + lane] = acc[k];
  if (MODE == 0) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, off);
    if (lane == 0) sbad[warp] = bad;
  }
  __syncthreads();
  const int g = gb * kGenesPerCta + threadIdx.x;
  if (g < G) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) s += sm[w][threadIdx.x];
    gene_part[(int64_t)slice * G + g] = s;
  }
  if (MODE == 0 && threadIdx.x == 0) {
    long long b = 0;
    for (int w = 0; w < kThreads / 32; ++w) b += sbad[w];
    bad_part[(int64_t)slice * gridDim.x + gb] = b;
  }
}

// The same pass fed rows [row0, row0 + n) of the N-row matrix at a time (Y holds those rows).  The CTA plan is
// col_plan(N, G) for the whole matrix; only the (gene block, slice) CTAs that overlap the chunk run (grid.y counts
// slices from slice0).  Warp w of slice s loads its accumulators from carry[s][w][genes], adds the chunk's rows
// s0 + w, s0 + w + 8, ... in order and stores them back, so after the last chunk carry holds exactly the warp sums of
// col_pass_kernel.  MODE 0: per-(gene block, chunk row) sums go to cell_part[gb][r - row0], bad-entry counts are
// added to bad_carry[s][gb].  A slot is touched by one CTA per launch and launches are stream-ordered: no atomics.
template <int MODE>
__global__ void __launch_bounds__(kThreads) col_chunk_kernel(const float* __restrict__ Y, int64_t ldy, int row0, int n,
                                                             int G, int rows_per_slice, int slice0,
                                                             const double* __restrict__ n_counts, double median, int flags,
                                                             const double* __restrict__ mean, double* __restrict__ carry,
                                                             double* __restrict__ cell_part,
                                                             long long* __restrict__ bad_carry) {
  __shared__ long long sbad[kThreads / 32];
  const int gb = blockIdx.x, slice = slice0 + blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g0 = gb * kGenesPerCta + lane;
  const int s0 = slice * rows_per_slice;
  const int lo = max(s0, row0), hi = min(s0 + rows_per_slice, row0 + n);
  double* cw = carry + ((int64_t)slice * (kThreads / 32) + warp) * G;
  double acc[kPerLane], mu[kPerLane];
#pragma unroll
  for (int k = 0; k < kPerLane; ++k) {
    const bool in = g0 + 32 * k < G;
    acc[k] = in ? cw[g0 + 32 * k] : 0.0;
    mu[k] = (MODE == 2 && in) ? mean[g0 + 32 * k] : 0.0;
  }
  long long bad = 0;
  const int first = lo + (((warp - (lo - s0)) % 8) + 8) % 8;      // first row of the chunk in this warp's residue class
  for (int r = first; r < hi; r += kThreads / 32)
    col_row<MODE>(Y + (int64_t)(r - row0) * ldy, g0, G, lane, MODE ? row_sf(n_counts, median, r, flags) : 1.0, flags, mu,
                  acc, bad, cell_part + (int64_t)gb * n + (r - row0));
#pragma unroll
  for (int k = 0; k < kPerLane; ++k)
    if (g0 + 32 * k < G) cw[g0 + 32 * k] = acc[k];
  if (MODE == 0) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, off);
    if (lane == 0) sbad[warp] = bad;
    __syncthreads();
    if (threadIdx.x == 0) {
      long long b = bad_carry[(int64_t)slice * gridDim.x + gb];
      for (int w = 0; w < kThreads / 32; ++w) b += sbad[w];
      bad_carry[(int64_t)slice * gridDim.x + gb] = b;
    }
  }
}

__device__ __forceinline__ double finish_fold(double s, int64_t N, int kind) {
  if (kind == 1) {
    s = s / (double)N;
  } else if (kind == 2) {
    s = N > 1 ? sqrt(s / (double)(N - 1)) : 1.0;
    if (s == 0.0) s = 1.0;
  }
  return s;
}

// out[g] = sum over slots s = 0, 1, ... of part[s][g]; then
//   kind 0: out = sum           kind 1: out = sum / N (mean)
//   kind 2: out = std = sqrt(sum / (N - 1)) (1 for N = 1), std == 0 -> 1
__global__ void fold_genes_kernel(const double* __restrict__ part, int slots, int G, int64_t N, int kind,
                                  double* __restrict__ out) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  double s = 0.0;
  for (int i = 0; i < slots; ++i) s += part[(int64_t)i * G + g];
  out[g] = finish_fold(s, N, kind);
}

// fold_genes_kernel over the carried warp sums of col_chunk_kernel: slot s is the warp-order sum of carry[s][0..7][g]
// (the gene_part col_pass_kernel writes), the slots are added in slot order
__global__ void fold_carry_kernel(const double* __restrict__ carry, int slices, int G, int64_t N, int kind,
                                  double* __restrict__ out) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  double s = 0.0;
  for (int i = 0; i < slices; ++i) {
    double p = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) p += carry[((int64_t)i * (kThreads / 32) + w) * G + g];
    s += p;
  }
  out[g] = finish_fold(s, N, kind);
}

// n_counts[r] = sum over gene blocks in order; thread 0 of block 0 also folds the bad-entry counts
__global__ void fold_cells_kernel(const double* __restrict__ cell_part, int gblocks, int N, double* __restrict__ out,
                                  const long long* __restrict__ bad_part, int n_bad_slots, long long* __restrict__ n_bad) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < N && out) {
    double s = 0.0;
    for (int b = 0; b < gblocks; ++b) s += cell_part[(int64_t)b * N + r];
    out[r] = s;
  }
  if (r == 0 && n_bad) {
    long long b = 0;
    for (int i = 0; i < n_bad_slots; ++i) b += bad_part[i];
    *n_bad = b;
  }
}

__global__ void fill_moments_kernel(double* mean, double* std, int G) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < G) { mean[g] = 0.0; std[g] = 1.0; }
}

__global__ void fill_value_kernel(double* out, int G, double v) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < G) out[g] = v;
}

// One warp per row: zero the whole row, then scatter the row's entries (canonical CSR: sorted, no duplicates).
__global__ void __launch_bounds__(kThreads) csr_to_dense_kernel(const int64_t* __restrict__ indptr,
                                                                const int32_t* __restrict__ indices,
                                                                const float* __restrict__ data, int N, int G,
                                                                float* __restrict__ Y, int64_t ldy) {
  const int row = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= N) return;
  float* y = Y + (int64_t)row * ldy;
  for (int g = lane; g < G; g += 32) y[g] = 0.f;
  __syncwarp();
  const int64_t e = indptr[row + 1];
  for (int64_t i = indptr[row] + lane; i < e; i += 32) y[indices[i]] = data[i];
}

// out[i][j] = Y[rows[i]][cols[j]] (NULL rows / cols: the identity)
__global__ void gather_kernel(const float* __restrict__ Y, int64_t ldy, const int32_t* __restrict__ rows, int nr,
                              const int32_t* __restrict__ cols, int nc, float* __restrict__ out, int64_t ldo) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nc) return;
  const int c = cols ? cols[j] : j;
  for (int i = blockIdx.y; i < nr; i += gridDim.y) {
    const int64_t r = rows ? rows[i] : i;
    out[(int64_t)i * ldo + j] = Y[r * ldy + c];
  }
}

// bf16 X is the fp32 X rounded once more: rounding the double straight to bf16 differs where the fp32 value is a bf16 tie
__device__ __forceinline__ __nv_bfloat16 to_bf16(double x) { return __float2bfloat16_rn((float)x); }

template <bool BF16>
__device__ __forceinline__ void store_x(void* X, int64_t idx, double x) {
  if (BF16) reinterpret_cast<__nv_bfloat16*>(X)[idx] = to_bf16(x);
  else reinterpret_cast<float*>(X)[idx] = (float)x;
}

// (l - mean) / std in double (l itself when there is no scaling); stored as float or bf16 by the caller
__device__ __forceinline__ double x_value(float y, double sf, int flags, const double* mean, const double* std, int g) {
  const float l = log_value(y, sf, flags);
  return mean ? ((double)l - mean[g]) / std[g] : (double)l;
}

// X[r][g] for V consecutive genes per thread.  V > 1 needs G % V == 0, ldy % 4 == 0, ldx % V == 0 and 16-byte
// aligned Y and X: then Y is read and X written with 128-bit accesses (fp32: 4 genes, bf16: 8 genes).
template <bool BF16, int V>
__global__ void __launch_bounds__(kThreads) normalize_write_kernel(const float* __restrict__ Y, int64_t ldy, int N, int G,
                                                                   const double* __restrict__ n_counts, double median,
                                                                   int flags, const double* __restrict__ mean,
                                                                   const double* __restrict__ std, void* __restrict__ X,
                                                                   int64_t ldx) {
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (g >= G) return;
  for (int r = blockIdx.y; r < N; r += gridDim.y) {
    const double sf = row_sf(n_counts, median, r, flags);
    const float* yr = Y + (int64_t)r * ldy + g;
    const int64_t o = (int64_t)r * ldx + g;
    if (V == 1) {
      store_x<BF16>(X, o, x_value(__ldg(yr), sf, flags, mean, std, g));
    } else {
      double x[V];
#pragma unroll
      for (int v = 0; v < V; v += 4) {
        const float4 y4 = __ldg(reinterpret_cast<const float4*>(yr + v));
        x[v + 0] = x_value(y4.x, sf, flags, mean, std, g + v + 0);
        x[v + 1] = x_value(y4.y, sf, flags, mean, std, g + v + 1);
        x[v + 2] = x_value(y4.z, sf, flags, mean, std, g + v + 2);
        x[v + 3] = x_value(y4.w, sf, flags, mean, std, g + v + 3);
      }
      if (BF16) {
        uint4 pk;
        uint32_t* w = reinterpret_cast<uint32_t*>(&pk);
#pragma unroll
        for (int v = 0; v < V; v += 2) {
          const __nv_bfloat162 h = __halves2bfloat162(to_bf16(x[v]), to_bf16(x[v + 1]));
          w[v / 2] = *reinterpret_cast<const uint32_t*>(&h);
        }
        *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(X) + o) = pk;
      } else {
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(X) + o) = make_float4((float)x[0], (float)x[1], (float)x[2], (float)x[3]);
      }
    }
  }
}

int need_device(const char* who) {
  static int ndev = -1;
  if (ndev < 0) {
    if (cudaGetDeviceCount(&ndev) != cudaSuccess) { (void)cudaGetLastError(); ndev = 0; }
  }
  if (ndev == 0) {
    set_error("%s: no CUDA device available (this library has no CPU fallback)", who);
    return DCA_ERR_NO_DEVICE;
  }
  return DCA_OK;
}

int check_matrix(const char* who, const void* p, int64_t ld, int64_t N, int32_t G) {
  if (!p || N <= 0 || G <= 0 || ld < G || N > INT32_MAX) {
    set_error("%s: bad matrix (ptr %p, %lld x %d, ld %lld; need 0 < rows < 2^31, 0 < genes <= ld)", who, p,
              (long long)N, G, (long long)ld);
    return DCA_ERR_BAD_ARG;
  }
  return DCA_OK;
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int col_pass(int mode, const float* Y, int64_t ldy, int N, int G, const double* n_counts, double median, int flags,
             const double* mean, const ColPlan& p, char* ws, cudaStream_t s) {
  double* gp = reinterpret_cast<double*>(ws + p.gene_part);
  double* cp = reinterpret_cast<double*>(ws + p.cell_part);
  long long* bp = reinterpret_cast<long long*>(ws + p.bad_part);
  const dim3 grid(p.gblocks, p.slices);
  if (mode == 0)
    col_pass_kernel<0><<<grid, kThreads, 0, s>>>(Y, ldy, N, G, p.rows_per_slice, n_counts, median, flags, mean, gp, cp, bp);
  else if (mode == 1)
    col_pass_kernel<1><<<grid, kThreads, 0, s>>>(Y, ldy, N, G, p.rows_per_slice, n_counts, median, flags, mean, gp, cp, bp);
  else
    col_pass_kernel<2><<<grid, kThreads, 0, s>>>(Y, ldy, N, G, p.rows_per_slice, n_counts, median, flags, mean, gp, cp, bp);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

// Workspace of the chunked passes: the carried warp sums [slices][8][G], the carried bad-entry counts [slices][gblocks]
// and the per-(gene block, row) sums of one chunk [gblocks][max_rows]
struct ChunkPlan {
  ColPlan p;
  size_t carry, bad, cell, bytes;
};

ChunkPlan chunk_plan(int64_t N, int G, int64_t max_rows) {
  ChunkPlan c;
  c.p = col_plan(N, G);
  c.carry = 0;
  c.bad = align256((size_t)c.p.slices * (kThreads / 32) * G * sizeof(double));
  c.cell = c.bad + align256((size_t)c.p.slices * c.p.gblocks * sizeof(long long));
  c.bytes = c.cell + align256((size_t)c.p.gblocks * max_rows * sizeof(double));
  return c;
}

int check_chunk(const char* who, const void* Y, int64_t ldy, int64_t row0, int64_t n_rows, int64_t n_cells, int32_t genes,
                const void* ws, size_t ws_bytes, ChunkPlan* out) {
  DCA_TRY(need_device(who));
  if (!Y || n_cells <= 0 || n_cells > INT32_MAX || genes <= 0 || ldy < genes || row0 < 0 || n_rows <= 0 ||
      row0 + n_rows > n_cells) {
    set_error("%s: bad chunk (Y %p, rows [%lld, %lld) of %lld, %d genes, ld %lld)", who, Y, (long long)row0,
              (long long)(row0 + n_rows), (long long)n_cells, genes, (long long)ldy);
    return DCA_ERR_BAD_ARG;
  }
  *out = chunk_plan(n_cells, genes, n_rows);
  if (!ws || ws_bytes < out->bytes) {
    set_error("%s: workspace too small for a chunk of %lld rows (%zu < %zu bytes)", who, (long long)n_rows, ws_bytes,
              out->bytes);
    return DCA_ERR_BAD_ARG;
  }
  return DCA_OK;
}

template <int MODE>
int col_chunk(const float* Y, int64_t ldy, int64_t row0, int64_t n_rows, const ChunkPlan& c, int G, const double* n_counts,
              double median, int flags, const double* mean, char* ws, cudaStream_t s) {
  const int rps = c.p.rows_per_slice;
  const int slice0 = (int)(row0 / rps), slice1 = (int)((row0 + n_rows - 1) / rps);
  const dim3 grid(c.p.gblocks, slice1 - slice0 + 1);
  col_chunk_kernel<MODE><<<grid, kThreads, 0, s>>>(Y, ldy, (int)row0, (int)n_rows, G, rps, slice0, n_counts, median, flags,
                                                   mean, reinterpret_cast<double*>(ws + c.carry),
                                                   reinterpret_cast<double*>(ws + c.cell),
                                                   reinterpret_cast<long long*>(ws + c.bad));
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

}  // namespace
}  // namespace dca

using namespace dca;

extern "C" {

int dca_preprocess_workspace_bytes(int64_t n_cells, int32_t genes, size_t* bytes) {
  if (!bytes || n_cells <= 0 || genes <= 0 || n_cells > INT32_MAX) {
    set_error("dca_preprocess_workspace_bytes: bad argument (%lld cells, %d genes)", (long long)n_cells, genes);
    return DCA_ERR_BAD_ARG;
  }
  *bytes = col_plan(n_cells, genes).bytes;
  return DCA_OK;
}

int dca_counts_csr_to_dense(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_cells,
                            int32_t genes, float* Y, int64_t ldy, void* stream) {
  DCA_TRY(need_device("dca_counts_csr_to_dense"));
  DCA_TRY(check_matrix("dca_counts_csr_to_dense", Y, ldy, n_cells, genes));
  if (!indptr) { set_error("dca_counts_csr_to_dense: indptr is NULL"); return DCA_ERR_BAD_ARG; }
  csr_to_dense_kernel<<<cdiv(n_cells, kThreads / 32), kThreads, 0, (cudaStream_t)stream>>>(
      indptr, indices, data, (int)n_cells, genes, Y, ldy);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int dca_count_totals(const float* Y, int64_t ldy, int64_t n_cells, int32_t genes, double* cell_totals,
                     double* gene_totals, int64_t* n_bad, void* workspace, size_t workspace_bytes, void* stream) {
  DCA_TRY(need_device("dca_count_totals"));
  DCA_TRY(check_matrix("dca_count_totals", Y, ldy, n_cells, genes));
  const ColPlan p = col_plan(n_cells, genes);
  if (!workspace || workspace_bytes < p.bytes) {
    set_error("dca_count_totals: workspace too small (%zu < %zu bytes)", workspace_bytes, p.bytes);
    return DCA_ERR_BAD_ARG;
  }
  cudaStream_t s = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  const int N = (int)n_cells;
  DCA_TRY(col_pass(0, Y, ldy, N, genes, nullptr, 1.0, 0, nullptr, p, ws, s));
  if (gene_totals) {
    fold_genes_kernel<<<cdiv(genes, 256), 256, 0, s>>>(reinterpret_cast<double*>(ws + p.gene_part), p.slices, genes, N, 0,
                                                       gene_totals);
    DCA_LAUNCH_CHECK();
  }
  if (cell_totals || n_bad) {
    fold_cells_kernel<<<cdiv(N, 256), 256, 0, s>>>(reinterpret_cast<double*>(ws + p.cell_part), p.gblocks, N, cell_totals,
                                                   reinterpret_cast<long long*>(ws + p.bad_part), p.slices * p.gblocks,
                                                   reinterpret_cast<long long*>(n_bad));
    DCA_LAUNCH_CHECK();
  }
  return DCA_OK;
}

int dca_gather_counts(const float* Y, int64_t ldy, const int32_t* rows, int64_t n_rows, const int32_t* cols,
                      int32_t n_cols, float* out, int64_t ldo, void* stream) {
  DCA_TRY(need_device("dca_gather_counts"));
  DCA_TRY(check_matrix("dca_gather_counts", out, ldo, n_rows, n_cols));
  if (!Y || ldy <= 0) { set_error("dca_gather_counts: bad source matrix"); return DCA_ERR_BAD_ARG; }
  const dim3 grid(cdiv(n_cols, 256), (unsigned)std::min<int64_t>(n_rows, 65535));
  gather_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(Y, ldy, rows, (int)n_rows, cols, n_cols, out, ldo);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int dca_log_moments(const float* Y, int64_t ldy, int64_t n_cells, int32_t genes, const double* n_counts, double median,
                    int32_t flags, double* mean, double* std, void* workspace, size_t workspace_bytes, void* stream) {
  DCA_TRY(need_device("dca_log_moments"));
  DCA_TRY(check_matrix("dca_log_moments", Y, ldy, n_cells, genes));
  if (flags < 0 || flags > 7 || !mean || !std || ((flags & PRE_SF) && (!n_counts || !(median > 0.0)))) {
    set_error("dca_log_moments: bad argument (flags %d; size factors need n_counts and a median > 0)", flags);
    return DCA_ERR_BAD_ARG;
  }
  cudaStream_t s = (cudaStream_t)stream;
  if (!(flags & PRE_SCALE)) {
    fill_moments_kernel<<<cdiv(genes, 256), 256, 0, s>>>(mean, std, genes);
    DCA_LAUNCH_CHECK();
    return DCA_OK;
  }
  const ColPlan p = col_plan(n_cells, genes);
  if (!workspace || workspace_bytes < p.bytes) {
    set_error("dca_log_moments: workspace too small (%zu < %zu bytes)", workspace_bytes, p.bytes);
    return DCA_ERR_BAD_ARG;
  }
  char* ws = (char*)workspace;
  const int N = (int)n_cells;
  double* gp = reinterpret_cast<double*>(ws + p.gene_part);
  DCA_TRY(col_pass(1, Y, ldy, N, genes, n_counts, median, flags, nullptr, p, ws, s));
  fold_genes_kernel<<<cdiv(genes, 256), 256, 0, s>>>(gp, p.slices, genes, N, 1, mean);
  DCA_LAUNCH_CHECK();
  DCA_TRY(col_pass(2, Y, ldy, N, genes, n_counts, median, flags, mean, p, ws, s));
  fold_genes_kernel<<<cdiv(genes, 256), 256, 0, s>>>(gp, p.slices, genes, N, 2, std);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

int dca_normalize_write(const float* Y, int64_t ldy, int64_t n_cells, int32_t genes, const double* n_counts,
                        double median, int32_t flags, const double* mean, const double* std, void* X, int32_t x_dtype,
                        int64_t ldx, void* stream) {
  DCA_TRY(need_device("dca_normalize_write"));
  DCA_TRY(check_matrix("dca_normalize_write", Y, ldy, n_cells, genes));
  DCA_TRY(check_matrix("dca_normalize_write", X, ldx, n_cells, genes));
  if (flags < 0 || flags > 7 || (x_dtype != DCA_F32 && x_dtype != DCA_BF16) || (!mean) != (!std) ||
      ((flags & PRE_SF) && (!n_counts || !(median > 0.0)))) {
    set_error("dca_normalize_write: bad argument (flags %d, x_dtype %d; mean and std go together; size factors need "
              "n_counts and a median > 0)", flags, x_dtype);
    return DCA_ERR_BAD_ARG;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const int N = (int)n_cells;
  const bool bf16 = x_dtype == DCA_BF16;
  const int V = bf16 ? 8 : 4;
  const bool vec = genes % V == 0 && ldy % 4 == 0 && ldx % V == 0 && aligned16(Y) && aligned16(X);
  const int per_thread = vec ? V : 1;
  const int gx = cdiv(cdiv(genes, per_thread), kThreads);
  const dim3 grid(gx, (unsigned)std::min<int64_t>(N, std::max(1, 8192 / gx)));
  if (bf16) {
    if (vec) normalize_write_kernel<true, 8><<<grid, kThreads, 0, s>>>(Y, ldy, N, genes, n_counts, median, flags, mean, std, X, ldx);
    else normalize_write_kernel<true, 1><<<grid, kThreads, 0, s>>>(Y, ldy, N, genes, n_counts, median, flags, mean, std, X, ldx);
  } else {
    if (vec) normalize_write_kernel<false, 4><<<grid, kThreads, 0, s>>>(Y, ldy, N, genes, n_counts, median, flags, mean, std, X, ldx);
    else normalize_write_kernel<false, 1><<<grid, kThreads, 0, s>>>(Y, ldy, N, genes, n_counts, median, flags, mean, std, X, ldx);
  }
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

// ---------------------------------------------------------------- the same statistics over row chunks
int dca_stats_workspace_bytes(int64_t n_cells, int32_t genes, int64_t max_chunk_rows, size_t* bytes) {
  if (!bytes || n_cells <= 0 || genes <= 0 || n_cells > INT32_MAX || max_chunk_rows <= 0) {
    set_error("dca_stats_workspace_bytes: bad argument (%lld cells, %d genes, chunks of %lld rows)", (long long)n_cells,
              genes, (long long)max_chunk_rows);
    return DCA_ERR_BAD_ARG;
  }
  *bytes = chunk_plan(n_cells, genes, std::min<int64_t>(max_chunk_rows, n_cells)).bytes;
  return DCA_OK;
}

int dca_stats_begin(int64_t n_cells, int32_t genes, void* workspace, size_t workspace_bytes, void* stream) {
  DCA_TRY(need_device("dca_stats_begin"));
  if (n_cells <= 0 || genes <= 0 || n_cells > INT32_MAX) {
    set_error("dca_stats_begin: bad argument (%lld cells, %d genes)", (long long)n_cells, genes);
    return DCA_ERR_BAD_ARG;
  }
  const ChunkPlan c = chunk_plan(n_cells, genes, 1);
  if (!workspace || workspace_bytes < c.bytes) {
    set_error("dca_stats_begin: workspace too small (%zu < %zu bytes)", workspace_bytes, c.bytes);
    return DCA_ERR_BAD_ARG;
  }
  DCA_CUDA_OK(cudaMemsetAsync(workspace, 0, c.cell, (cudaStream_t)stream));     // carried sums and bad-entry counts
  return DCA_OK;
}

int dca_count_totals_rows(const float* Y, int64_t ldy, int64_t row0, int64_t n_rows, int64_t n_cells, int32_t genes,
                          double* cell_totals, void* workspace, size_t workspace_bytes, void* stream) {
  ChunkPlan c;
  DCA_TRY(check_chunk("dca_count_totals_rows", Y, ldy, row0, n_rows, n_cells, genes, workspace, workspace_bytes, &c));
  cudaStream_t s = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  DCA_TRY(col_chunk<0>(Y, ldy, row0, n_rows, c, genes, nullptr, 1.0, 0, nullptr, ws, s));
  if (cell_totals) {
    fold_cells_kernel<<<cdiv(n_rows, 256), 256, 0, s>>>(reinterpret_cast<double*>(ws + c.cell), c.p.gblocks, (int)n_rows,
                                                        cell_totals + row0, nullptr, 0, nullptr);
    DCA_LAUNCH_CHECK();
  }
  return DCA_OK;
}

int dca_count_totals_finish(int64_t n_cells, int32_t genes, double* gene_totals, int64_t* n_bad, void* workspace,
                            size_t workspace_bytes, void* stream) {
  DCA_TRY(need_device("dca_count_totals_finish"));
  if (n_cells <= 0 || genes <= 0 || n_cells > INT32_MAX) {
    set_error("dca_count_totals_finish: bad argument (%lld cells, %d genes)", (long long)n_cells, genes);
    return DCA_ERR_BAD_ARG;
  }
  const ChunkPlan c = chunk_plan(n_cells, genes, 1);
  if (!workspace || workspace_bytes < c.bytes) {
    set_error("dca_count_totals_finish: workspace too small (%zu < %zu bytes)", workspace_bytes, c.bytes);
    return DCA_ERR_BAD_ARG;
  }
  cudaStream_t s = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  if (gene_totals) {
    fold_carry_kernel<<<cdiv(genes, 256), 256, 0, s>>>(reinterpret_cast<double*>(ws + c.carry), c.p.slices, genes, n_cells,
                                                       0, gene_totals);
    DCA_LAUNCH_CHECK();
  }
  if (n_bad) {
    fold_cells_kernel<<<1, 256, 0, s>>>(nullptr, 0, 1, nullptr, reinterpret_cast<long long*>(ws + c.bad),
                                        c.p.slices * c.p.gblocks, reinterpret_cast<long long*>(n_bad));
    DCA_LAUNCH_CHECK();
  }
  return DCA_OK;
}

int dca_log_moments_rows(int32_t pass, const float* Y, int64_t ldy, int64_t row0, int64_t n_rows, int64_t n_cells,
                         int32_t genes, const double* n_counts, double median, int32_t flags, const double* mean,
                         void* workspace, size_t workspace_bytes, void* stream) {
  ChunkPlan c;
  DCA_TRY(check_chunk("dca_log_moments_rows", Y, ldy, row0, n_rows, n_cells, genes, workspace, workspace_bytes, &c));
  if ((pass != 1 && pass != 2) || flags < 0 || flags > 7 || (pass == 2 && (flags & PRE_SCALE) && !mean) ||
      ((flags & PRE_SF) && (!n_counts || !(median > 0.0)))) {
    set_error("dca_log_moments_rows: bad argument (pass %d, flags %d; pass 2 needs the mean, size factors need "
              "n_counts and a median > 0)", pass, flags);
    return DCA_ERR_BAD_ARG;
  }
  if (!(flags & PRE_SCALE)) return DCA_OK;
  cudaStream_t s = (cudaStream_t)stream;
  if (pass == 1) return col_chunk<1>(Y, ldy, row0, n_rows, c, genes, n_counts, median, flags, nullptr, (char*)workspace, s);
  return col_chunk<2>(Y, ldy, row0, n_rows, c, genes, n_counts, median, flags, mean, (char*)workspace, s);
}

int dca_log_moments_finish(int32_t pass, int64_t n_cells, int32_t genes, int32_t flags, double* out, void* workspace,
                           size_t workspace_bytes, void* stream) {
  DCA_TRY(need_device("dca_log_moments_finish"));
  if ((pass != 1 && pass != 2) || !out || n_cells <= 0 || genes <= 0 || n_cells > INT32_MAX || flags < 0 || flags > 7) {
    set_error("dca_log_moments_finish: bad argument (pass %d, %lld cells, %d genes, flags %d)", pass, (long long)n_cells,
              genes, flags);
    return DCA_ERR_BAD_ARG;
  }
  cudaStream_t s = (cudaStream_t)stream;
  if (!(flags & PRE_SCALE)) {                     // mean = 0, std = 1, as dca_log_moments
    fill_value_kernel<<<cdiv(genes, 256), 256, 0, s>>>(out, genes, pass == 1 ? 0.0 : 1.0);
    DCA_LAUNCH_CHECK();
    return DCA_OK;
  }
  const ChunkPlan c = chunk_plan(n_cells, genes, 1);
  if (!workspace || workspace_bytes < c.bytes) {
    set_error("dca_log_moments_finish: workspace too small (%zu < %zu bytes)", workspace_bytes, c.bytes);
    return DCA_ERR_BAD_ARG;
  }
  fold_carry_kernel<<<cdiv(genes, 256), 256, 0, s>>>(reinterpret_cast<double*>((char*)workspace + c.carry), c.p.slices,
                                                     genes, n_cells, pass, out);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

}  // extern "C"
