// GPU gzip compressor (dca_gzip_device, and the writer's dca_write_text_device_gz): the block encoder of deflate.cuh
// with one CTA per block of kBlock input bytes, and the same encoder on the CPU (dca_gzip_host).
//
// A member is fed in pieces (GzipMember::feed).  Per piece, in rounds of up to kRoundBlocks blocks, on the caller's
// stream:
//   encode  one CTA per block: the block's compressed bytes into its staging slot, their count, kind and linear CRC
//   place   one CTA: exclusive scan of the sizes into output offsets after the bytes so far (a device counter), and
//           the blocks' CRCs folded into the member's in block order (x^(8 n) mod P)
//   copy    one CTA per block: its staged bytes to their offset
// A block's matches reach up to 32 KB back, but not before the start of its piece.  Every non-final block ends on a
// byte, so the offsets are plain byte offsets, and the bytes depend on the input and the piece boundaries alone.
#include "dca_internal.cuh"
#include "deflate.cuh"

#include <algorithm>
#include <cstring>
#include <memory>

namespace dca {
namespace deflate {
namespace {

constexpr int kRoundBlocks = 2048;             // blocks per round: 64 MB of input, 64 MB of staging
constexpr int kPlaceThreads = 1024;

struct State {
  long long len;                               // bytes of the piece's output so far
  long long stored;                            // stored blocks of the member
  uint32_t crc;                                // linear CRC of the member's input so far
};

__device__ __forceinline__ Block block_of(const uint8_t* in, long long n, long long b, long long blocks, int last) {
  const long long off = b * kBlock;
  return Block{in + off, (int)min((long long)kBlock, n - off), (int)min(off, (long long)kWindow),
               last && b == blocks - 1};
}

__global__ void __launch_bounds__(kThreads, 1) encode_kernel(const uint8_t* __restrict__ in, long long n, long long b0,
                                                             long long blocks, int last, uint8_t* slots, int* sizes,
                                                             uint32_t* crcs, int* kinds) {
  extern __shared__ __align__(16) uint8_t smem[];
  Shared& s = *reinterpret_cast<Shared*>(smem);
  const int t = threadIdx.x;
  const Block b = block_of(in, n, b0 + blockIdx.x, blocks, last);
  init_phase(s, b, t);
  __syncthreads();
  hd_xor(&s.crc, crc_part(s, b, t));
  history_phase(s, b, t);
  __syncthreads();
  for (int r = 0; r * kThreads < b.len; ++r) {
    round_read(s, b, r, t);
    __syncthreads();
    round_write(s, b, r, t);
    __syncthreads();
  }
  for (;;) {
    parse_phase(s, b, t);
    __syncthreads();
    if (!__syncthreads_or(chain_phase(s, t))) break;
  }
  count_phase(s, b, t);
  __syncthreads();
  if (t == 0) codes_phase(s, b);
  __syncthreads();
  uint8_t* out = slots + (long long)blockIdx.x * kSlot;
  if (s.kind == KIND_STORED) {
    stored_phase(b, t, out);
  } else {
    uint32_t* w = reinterpret_cast<uint32_t*>(out);
    for (int i = t; i < kSlot / 4; i += kThreads) w[i] = 0;
    size_phase(s, b, t);
    __syncthreads();
    if (t == 0) header_phase(s, b, w);
    __syncthreads();
    emit_phase(s, b, t, w);
  }
  if (t == 0) { sizes[blockIdx.x] = s.bytes; crcs[blockIdx.x] = s.crc; kinds[blockIdx.x] = s.kind; }
}

// one CTA: offs[i] = st->len + sizes[0] + ... + sizes[i - 1]; then the counter, the stored count and the CRC move on
__global__ void __launch_bounds__(kPlaceThreads) place_kernel(const int* sizes, const uint32_t* crcs, const int* kinds,
                                                              int nb, int last_len, State* st, long long* offs) {
  __shared__ long long warp_sums[kPlaceThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int per = (nb + kPlaceThreads - 1) / kPlaceThreads;
  const int a = min(nb, (int)threadIdx.x * per), e = min(nb, a + per);
  long long sum = 0;
  for (int i = a; i < e; ++i) sum += sizes[i];
  long long x = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const long long y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    long long w = warp_sums[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const long long y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
    warp_sums[lane] = w;
  }
  __syncthreads();
  const long long base = st->len;
  long long run = base + (warp ? warp_sums[warp - 1] : 0) + x - sum;
  for (int i = a; i < e; ++i) { offs[i] = run; run += sizes[i]; }
  __syncthreads();
  if (threadIdx.x == 0) {
    st->len = base + warp_sums[31];
    const uint32_t full = inflate::crc_x8n(kBlock);
    uint32_t crc = st->crc;
    long long stored = 0;
    for (int i = 0; i < nb; ++i) {
      crc = inflate::crc_mul(i + 1 < nb ? full : inflate::crc_x8n((unsigned long long)last_len), crc) ^ crcs[i];
      stored += kinds[i] == KIND_STORED;
    }
    st->crc = crc;
    st->stored += stored;
  }
}

__global__ void __launch_bounds__(256) copy_kernel(const uint8_t* __restrict__ slots, const int* sizes,
                                                   const long long* offs, uint8_t* out) {
  const uint8_t* src = slots + (long long)blockIdx.x * kSlot;
  uint8_t* dst = out + offs[blockIdx.x];
  for (int i = threadIdx.x; i < sizes[blockIdx.x]; i += blockDim.x) dst[i] = src[i];
}

__global__ void begin_kernel(State* st, uint8_t* out, int first) {
  st->len = first ? 10 : 0;
  if (first) {
    st->crc = 0; st->stored = 0;
    const uint8_t h[10] = {0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 255};
    for (int i = 0; i < 10; ++i) out[i] = h[i];
  }
}

// the empty final block when the last piece has no block, then CRC-32 and ISIZE
__global__ void end_kernel(State* st, uint8_t* out, int empty, unsigned long long isize) {
  long long p = st->len;
  if (empty) { out[p] = 0x03; out[p + 1] = 0x00; p += 2; }
  const uint32_t crc = inflate::crc_finish(st->crc, isize);
  for (int i = 0; i < 4; ++i) { out[p + i] = (uint8_t)(crc >> (8 * i)); out[p + 4 + i] = (uint8_t)(isize >> (8 * i)); }
  st->len = p + 8;
}

// the encoder of encode_kernel on the CPU, its threads run one after the other between the barriers
void encode_block_host(Shared& s, const Block& b, uint8_t* out, int* bytes, uint32_t* crc, int* kind) {
  for (int t = 0; t < kThreads; ++t) init_phase(s, b, t);
  for (int t = 0; t < kThreads; ++t) { hd_xor(&s.crc, crc_part(s, b, t)); history_phase(s, b, t); }
  for (int r = 0; r * kThreads < b.len; ++r) {
    for (int t = 0; t < kThreads; ++t) round_read(s, b, r, t);
    for (int t = 0; t < kThreads; ++t) round_write(s, b, r, t);
  }
  for (;;) {
    for (int t = 0; t < kThreads; ++t) parse_phase(s, b, t);
    bool any = false;
    for (int t = 0; t < kThreads; ++t) any |= chain_phase(s, t);
    if (!any) break;
  }
  for (int t = 0; t < kThreads; ++t) count_phase(s, b, t);
  codes_phase(s, b);
  if (s.kind == KIND_STORED) {
    for (int t = 0; t < kThreads; ++t) stored_phase(b, t, out);
  } else {
    uint32_t* w = reinterpret_cast<uint32_t*>(out);
    std::memset(w, 0, kSlot);
    for (int t = 0; t < kThreads; ++t) size_phase(s, b, t);
    header_phase(s, b, w);
    for (int t = 0; t < kThreads; ++t) emit_phase(s, b, t, w);
  }
  *bytes = s.bytes; *crc = s.crc; *kind = s.kind;
}

}  // namespace

GzipMember::~GzipMember() {
  cudaFree(slots_); cudaFree(sizes_); cudaFree(crcs_); cudaFree(kinds_); cudaFree(offs_); cudaFree(st_);
  cudaFreeHost(h_st_);
}

int GzipMember::init(cudaStream_t s) {
  s_ = s;
  DCA_CUDA_OK(cudaFuncSetAttribute(encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Shared)));
  DCA_CUDA_OK(cudaMalloc(&slots_, (size_t)kRoundBlocks * kSlot));
  DCA_CUDA_OK(cudaMalloc(&sizes_, kRoundBlocks * sizeof(int)));
  DCA_CUDA_OK(cudaMalloc(&crcs_, kRoundBlocks * sizeof(uint32_t)));
  DCA_CUDA_OK(cudaMalloc(&kinds_, kRoundBlocks * sizeof(int)));
  DCA_CUDA_OK(cudaMalloc(&offs_, kRoundBlocks * sizeof(long long)));
  DCA_CUDA_OK(cudaMalloc(&st_, sizeof(State)));
  DCA_CUDA_OK(cudaHostAlloc(&h_st_, sizeof(State), cudaHostAllocDefault));
  return DCA_OK;
}

long long GzipMember::device_bytes() {
  return (long long)kRoundBlocks * (kSlot + 2 * sizeof(int) + sizeof(uint32_t) + sizeof(long long)) + sizeof(State);
}

int GzipMember::feed(const uint8_t* in, long long n, bool first, bool last, uint8_t* out, long long* out_len) {
  if (first) { isize_ = 0; blocks_ = 0; }
  begin_kernel<<<1, 1, 0, s_>>>(static_cast<State*>(st_), out, first);
  DCA_LAUNCH_CHECK();
  const long long blocks = (n + kBlock - 1) / kBlock;
  for (long long b0 = 0; b0 < blocks; b0 += kRoundBlocks) {
    const int nb = (int)std::min<long long>(kRoundBlocks, blocks - b0);
    encode_kernel<<<nb, kThreads, sizeof(Shared), s_>>>(in, n, b0, blocks, last, slots_, sizes_, crcs_, kinds_);
    DCA_LAUNCH_CHECK();
    const int last_len = (int)std::min<long long>(kBlock, n - (b0 + nb - 1) * kBlock);
    place_kernel<<<1, kPlaceThreads, 0, s_>>>(sizes_, crcs_, kinds_, nb, last_len, static_cast<State*>(st_), offs_);
    DCA_LAUNCH_CHECK();
    copy_kernel<<<nb, 256, 0, s_>>>(slots_, sizes_, offs_, out);
    DCA_LAUNCH_CHECK();
  }
  isize_ += (unsigned long long)n;
  blocks_ += blocks;
  if (last) {
    end_kernel<<<1, 1, 0, s_>>>(static_cast<State*>(st_), out, blocks == 0, isize_);
    DCA_LAUNCH_CHECK();
  }
  DCA_CUDA_OK(cudaMemcpyAsync(h_st_, st_, sizeof(State), cudaMemcpyDeviceToHost, s_));
  DCA_CUDA_OK(cudaStreamSynchronize(s_));
  const State* h = static_cast<const State*>(h_st_);
  *out_len = h->len;
  stored_ = h->stored;
  return DCA_OK;
}

}  // namespace deflate
}  // namespace dca

using namespace dca;
using namespace dca::deflate;

extern "C" int dca_gzip_device(const void* in, int64_t n, void* out, int64_t out_cap, int32_t device, void* stream,
                               int64_t* info) {
  if (n < 0 || (out && n > 0 && !in) || !info || (out && out_cap < 0)) { set_error("dca_gzip_device: bad argument"); return DCA_ERR_BAD_ARG; }
  if (!out) { info[0] = gzip_bound(n); return DCA_OK; }
  if (out_cap < gzip_bound(n)) {
    set_error("dca_gzip_device: out_cap %lld is below the bound %lld", (long long)out_cap, gzip_bound(n));
    return DCA_ERR_BAD_ARG;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    (void)cudaGetLastError();
    set_error("dca_gzip_device: no CUDA device available (this library has no CPU fallback)");
    return DCA_ERR_NO_DEVICE;
  }
  if (device < 0 || device >= ndev) { set_error("dca_gzip_device: no CUDA device %d", device); return DCA_ERR_BAD_ARG; }
  int prev = -1;
  DCA_CUDA_OK(cudaGetDevice(&prev));
  DCA_CUDA_OK(cudaSetDevice(device));
  struct Restore { int d; ~Restore() { if (d >= 0) cudaSetDevice(d); } } restore{prev};
  GzipMember g;
  DCA_TRY(g.init((cudaStream_t)stream));
  long long len = 0;
  DCA_TRY(g.feed((const uint8_t*)in, n, true, true, (uint8_t*)out, &len));
  info[0] = len;
  info[1] = g.blocks();
  info[2] = g.stored();
  return DCA_OK;
}

extern "C" int dca_gzip_host(const void* in, int64_t n, void* out, int64_t out_cap, int64_t* out_len) {
  if (n < 0 || (out && n > 0 && !in) || !out_len || (out && out_cap < 0)) { set_error("dca_gzip_host: bad argument"); return DCA_ERR_BAD_ARG; }
  if (!out) { *out_len = gzip_bound(n); return DCA_OK; }
  if (out_cap < gzip_bound(n)) {
    set_error("dca_gzip_host: out_cap %lld is below the bound %lld", (long long)out_cap, gzip_bound(n));
    return DCA_ERR_BAD_ARG;
  }
  const uint8_t* src = (const uint8_t*)in;
  uint8_t* dst = (uint8_t*)out;
  const uint8_t h[10] = {0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 255};
  std::memcpy(dst, h, 10);
  long long p = 10;
  std::unique_ptr<Shared> s(new Shared);
  std::unique_ptr<uint32_t[]> slot(new uint32_t[kSlot / 4]);
  const long long blocks = (n + kBlock - 1) / kBlock;
  uint32_t crc = 0;
  for (long long k = 0; k < blocks; ++k) {
    const long long off = k * kBlock;
    const Block b{src + off, (int)std::min<long long>(kBlock, n - off), (int)std::min<long long>(off, kWindow),
                  k == blocks - 1};
    int bytes = 0, kind = 0;
    uint32_t c = 0;
    encode_block_host(*s, b, reinterpret_cast<uint8_t*>(slot.get()), &bytes, &c, &kind);
    std::memcpy(dst + p, slot.get(), (size_t)bytes);
    p += bytes;
    crc = inflate::crc_mul(inflate::crc_x8n((unsigned long long)b.len), crc) ^ c;
  }
  if (!blocks) { dst[p] = 0x03; dst[p + 1] = 0x00; p += 2; }
  const uint32_t fin = inflate::crc_finish(crc, (unsigned long long)n);
  for (int i = 0; i < 4; ++i) { dst[p + i] = (uint8_t)(fin >> (8 * i)); dst[p + 4 + i] = (uint8_t)((unsigned long long)n >> (8 * i)); }
  *out_len = p + 8;
  return DCA_OK;
}
