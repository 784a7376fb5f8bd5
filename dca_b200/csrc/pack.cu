// GPU packer of raw counts (include/dca_b200.h, "packed counts resident in device memory"): the formats io.pack_counts /
// dca_pack_counts / dca_pack_sparse write on the host, written on the device from fp32 counts already there.
//   count pass  dca_pack_count_rows   per row: non-zeros, escapes at 4 / 8 / 16 bits, bad entries
//   pack pass   dca_pack_rows_device  packed rows (dense widths) or bitmap + 4-bit codes (sparse), overflow entries
// One warp per row, genes in 32-wide segments: a __ballot_sync per segment gives the bitmap word and, with the running
// count of the row, every code's and every overflow entry's position.  No atomics: each output byte is written by
// exactly one lane, so the arrays are a pure function of the counts.
#include "dca_internal.cuh"

namespace dca {
namespace {

constexpr int kThreads = 256;               // 8 warps = 8 rows per CTA
constexpr int kRowsPerCta = kThreads / 32;
constexpr unsigned kFull = 0xffffffffu;

// genes % 8 == 0, ldy % 4 == 0, 16-byte aligned Y: each lane reads 4 genes with one 128-bit load
__global__ void __launch_bounds__(kThreads) pack_count_kernel(const float* __restrict__ Y, int64_t ldy, int N, int G,
                                                              int64_t* __restrict__ stats, int64_t ld) {
  const int row = blockIdx.x * kRowsPerCta + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= N) return;
  const float* y = Y + (int64_t)row * ldy;
  int c[5] = {0, 0, 0, 0, 0};
  for (int g = lane * 4; g < G; g += 128) {
    const float4 q = __ldg(reinterpret_cast<const float4*>(y + g));
    const float v[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      c[0] += v[k] != 0.f;
      c[1] += v[k] >= 15.f;
      c[2] += v[k] >= 255.f;
      c[3] += v[k] >= 65535.f;
      c[4] += !(v[k] >= 0.f) || v[k] != floorf(v[k]) || isinf(v[k]);    // negative, NaN, non-integer, infinite
    }
  }
#pragma unroll
  for (int k = 0; k < 5; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c[k] += __shfl_xor_sync(kFull, c[k], o);
  }
  if (lane < 5) {
    int v = c[0];
#pragma unroll
    for (int k = 1; k < 5; ++k) if (lane == k) v = c[k];
    stats[(int64_t)lane * ld + row] = v;
  }
}

// Sparse format: bitmap byte g/8 bit g%8 = (count != 0); the row's non-zero counts as 4-bit codes min(count, 15) in gene
// order, low nibble first, from byte nib_indptr[R]; counts >= 15 listed as overflow entries from ovf_indptr[R].  A
// code pair may straddle two segments: the low nibble of an unfinished byte is carried to the next segment (and
// written alone, high nibble 0, at the row's end).
__global__ void __launch_bounds__(kThreads) pack_sparse_kernel(const float* __restrict__ Y, int64_t ldy, int N, int G,
                                                               int64_t row0, unsigned char* __restrict__ bitmap,
                                                               const int64_t* __restrict__ nib_indptr,
                                                               unsigned char* __restrict__ nibbles,
                                                               const int64_t* __restrict__ ovf_indptr,
                                                               int2* __restrict__ entries) {
  const int row = blockIdx.x * kRowsPerCta + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= N) return;
  const float* y = Y + (int64_t)row * ldy;
  const int64_t R = row0 + row;
  unsigned char* bm = bitmap + R * (G / 8);
  unsigned char* nib = nibbles + nib_indptr[R];
  int2* ent = ovf_indptr ? entries + ovf_indptr[R] : nullptr;
  const unsigned lt = (1u << lane) - 1u;
  const unsigned gt = lane == 31 ? 0u : (kFull << (lane + 1));
  int nz_before = 0, ov_before = 0;
  unsigned carry = 0;                                   // low nibble of the row's last byte when nz_before is odd
  for (int c0 = 0; c0 < G; c0 += 32) {
    const int g = c0 + lane;
    const float v = g < G ? y[g] : 0.f;
    const unsigned nzm = __ballot_sync(kFull, v != 0.f);
    const unsigned ovm = __ballot_sync(kFull, v >= 15.f);
    if ((lane & 7) == 0 && g < G) bm[g >> 3] = (unsigned char)((nzm >> lane) & 0xffu);
    const bool nz = (nzm >> lane) & 1u;
    const unsigned code = nz ? (v >= 15.f ? 15u : (unsigned)v) : 0u;
    const int k = nz_before + __popc(nzm & lt);          // index of this code in the row
    const unsigned above = nzm & gt;
    const unsigned ncode = __shfl_sync(kFull, code, above ? __ffs(above) - 1 : lane);
    if (nz) {
      if ((k & 1) == 0) {
        if (above) nib[k >> 1] = (unsigned char)(code | (ncode << 4));
      } else if ((nzm & lt) == 0) {
        nib[k >> 1] = (unsigned char)(carry | (code << 4));      // completes the byte begun in an earlier segment
      }
    }
    const int cnt = __popc(nzm);
    if (cnt) {
      const unsigned lcode = __shfl_sync(kFull, code, 31 - __clz(nzm));
      if (((nz_before + cnt - 1) & 1) == 0) carry = lcode;
    }
    nz_before += cnt;
    if (ent && ((ovm >> lane) & 1u)) ent[ov_before + __popc(ovm & lt)] = make_int2(g, __float_as_int(v));
    ov_before += __popc(ovm);
  }
  if ((nz_before & 1) && lane == 0) nib[(nz_before - 1) >> 1] = (unsigned char)carry;
}

// Dense widths: entry min(count, 2^BITS - 1) per gene (4 bits: gene c in byte c/2, low nibble = even c), counts >=
// 2^BITS - 1 listed as overflow entries from ovf_indptr[R].
template <int BITS>
__global__ void __launch_bounds__(kThreads) pack_dense_kernel(const float* __restrict__ Y, int64_t ldy, int N, int G,
                                                              int64_t row0, unsigned char* __restrict__ packed,
                                                              const int64_t* __restrict__ ovf_indptr,
                                                              int2* __restrict__ entries) {
  const int row = blockIdx.x * kRowsPerCta + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= N) return;
  constexpr unsigned kEsc = (1u << BITS) - 1u;
  const float* y = Y + (int64_t)row * ldy;
  const int64_t R = row0 + row;
  unsigned char* dst = packed + R * (int64_t)G * BITS / 8;
  int2* ent = ovf_indptr ? entries + ovf_indptr[R] : nullptr;
  const unsigned lt = (1u << lane) - 1u;
  int ov_before = 0;
  for (int c0 = 0; c0 < G; c0 += 32) {
    const int g = c0 + lane;
    const float v = g < G ? y[g] : 0.f;
    const bool over = v >= (float)kEsc;
    const unsigned q = over ? kEsc : (unsigned)v;
    const unsigned ovm = __ballot_sync(kFull, over);
    const unsigned qn = __shfl_down_sync(kFull, q, 1);
    if (g < G) {
      if (BITS == 4) { if ((lane & 1) == 0) dst[g >> 1] = (unsigned char)(q | (qn << 4)); }
      else if (BITS == 8) dst[g] = (unsigned char)q;
      else reinterpret_cast<uint16_t*>(dst)[g] = (uint16_t)q;
    }
    if (ent && over) ent[ov_before + __popc(ovm & lt)] = make_int2(g, __float_as_int(v));
    ov_before += __popc(ovm);
  }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int check_rows(const char* who, const float* Y, int64_t ldy, int64_t n_rows, int32_t genes) {
  if (!Y || n_rows <= 0 || n_rows > INT32_MAX || genes <= 0 || genes % 8 != 0 || ldy < genes || ldy % 4 != 0 ||
      !aligned16(Y)) {
    set_error("%s: bad counts (%lld rows, %d genes, ld %lld: need 0 < rows < 2^31, genes a positive multiple of 8, "
              "ld >= genes and a multiple of 4, 16-byte aligned Y)", who, (long long)n_rows, genes, (long long)ldy);
    return DCA_ERR_BAD_ARG;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    (void)cudaGetLastError();
    set_error("%s: no CUDA device available (this library has no CPU fallback)", who);
    return DCA_ERR_NO_DEVICE;
  }
  return DCA_OK;
}

}  // namespace

// shared with engine.cu (dca_expand_rows_exact, dca_packed_*): the checks every consumer of a dca_packed_counts makes
int check_packed_counts(const char* who, const dca_packed_counts* p) {
  if (!p || p->struct_bytes != (int32_t)sizeof(dca_packed_counts)) {
    set_error("%s: NULL or unversioned dca_packed_counts (struct_bytes must be %d)", who, (int)sizeof(dca_packed_counts));
    return DCA_ERR_BAD_ARG;
  }
  if ((p->bits != 1 && p->bits != 4 && p->bits != 8 && p->bits != 16) || !p->packed || p->n_rows <= 0 ||
      p->n_rows > INT32_MAX || p->genes <= 0 || p->genes % 8 != 0 || !aligned16(p->packed) ||
      (p->ovf_indptr == nullptr) != (p->ovf_entries == nullptr) ||
      (p->bits == 1 && (!p->nib_indptr || !p->nibbles || p->max_row_nibble_bytes < 0))) {
    set_error("%s: bad dca_packed_counts (bits %d, %lld rows, %d genes: need bits 1/4/8/16, a 16-byte aligned matrix, "
              "genes a positive multiple of 8, both overflow arrays or neither, the nibble arrays with bits 1)", who,
              p->bits, (long long)p->n_rows, p->genes);
    return DCA_ERR_BAD_ARG;
  }
  if (p->bits == 1 && p->genes > 65536) {
    set_error("%s: at most 65536 genes in the sparse format (got %d)", who, p->genes);
    return DCA_ERR_UNSUPPORTED;
  }
  return DCA_OK;
}

}  // namespace dca

using namespace dca;

extern "C" int dca_pack_count_rows(const float* Y, int64_t ldy, int64_t n_rows, int32_t genes, int64_t* stats,
                                   int64_t ld_stats, void* stream) {
  DCA_TRY(check_rows("dca_pack_count_rows", Y, ldy, n_rows, genes));
  if (!stats || ld_stats < n_rows) { set_error("dca_pack_count_rows: stats is NULL or ld_stats < rows"); return DCA_ERR_BAD_ARG; }
  const int N = (int)n_rows;
  pack_count_kernel<<<(N + kRowsPerCta - 1) / kRowsPerCta, kThreads, 0, (cudaStream_t)stream>>>(Y, ldy, N, genes, stats,
                                                                                                 ld_stats);
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}

extern "C" int dca_pack_rows_device(const float* Y, int64_t ldy, int64_t n_rows, int64_t row0, const dca_packed_counts* dst,
                                    void* stream) {
  DCA_TRY(check_packed_counts("dca_pack_rows_device", dst));
  DCA_TRY(check_rows("dca_pack_rows_device", Y, ldy, n_rows, dst->genes));
  if (row0 < 0 || row0 + n_rows > dst->n_rows) {
    set_error("dca_pack_rows_device: rows [%lld, %lld) outside the %lld rows of the matrix", (long long)row0,
              (long long)(row0 + n_rows), (long long)dst->n_rows);
    return DCA_ERR_BAD_ARG;
  }
  const int N = (int)n_rows, G = dst->genes;
  const int grid = (N + kRowsPerCta - 1) / kRowsPerCta;
  cudaStream_t s = (cudaStream_t)stream;
  unsigned char* packed = reinterpret_cast<unsigned char*>(const_cast<void*>(dst->packed));
  int2* ent = reinterpret_cast<int2*>(const_cast<void*>(dst->ovf_entries));
  switch (dst->bits) {
    case 1:
      pack_sparse_kernel<<<grid, kThreads, 0, s>>>(Y, ldy, N, G, row0, packed, dst->nib_indptr,
                                                   reinterpret_cast<unsigned char*>(const_cast<void*>(dst->nibbles)),
                                                   dst->ovf_indptr, ent);
      break;
    case 4: pack_dense_kernel<4><<<grid, kThreads, 0, s>>>(Y, ldy, N, G, row0, packed, dst->ovf_indptr, ent); break;
    case 8: pack_dense_kernel<8><<<grid, kThreads, 0, s>>>(Y, ldy, N, G, row0, packed, dst->ovf_indptr, ent); break;
    default: pack_dense_kernel<16><<<grid, kThreads, 0, s>>>(Y, ldy, N, G, row0, packed, dst->ovf_indptr, ent); break;
  }
  DCA_LAUNCH_CHECK();
  return DCA_OK;
}
