// GPU writer of the '%.6f' TSV files (dca_write_text_device): the bytes dca_write_text_matrix (text_io.cu) writes,
// formatted on the device from a float32 matrix in device memory, so that an output matrix never has to exist on the
// host.  Per group of output lines, on the caller's stream:
//   field_len   per tile of 256 fields of one line: the sum of the fields' widths (number + its '\t' or '\n')
//   scan_segs   one CTA: exclusive prefix, in (line, label, tile 0, tile 1, ...) order, of the label and tile widths
//   label_write / field_write   fill the bytes at those offsets (a tile is formatted in shared memory, then copied)
// The offsets depend on the values only, so the text is a function of the input.  The group's text goes to the host in
// pieces through two pinned buffers; a writer thread appends one piece to the file while the next is formatted and
// copied.  dca_write_text_device_gz takes the same path with one more step per group: the header and each group's
// text are compressed on the device (deflate.cu, one gzip member per call), and the pieces carry the compressed bytes.
//
// Number format: '%.6f' of the float32 value (exact in double), correctly rounded, ties to even, on integers only.
// v = +-m * 2^e with m < 2^24: for e < 0, m * 10^6 < 2^44 is shifted right by -e with round-half-even on the bits
// shifted out; for e >= 0, v is an integer below 2^128, written in base-10^9 groups, then ".000000".
#include "dca_internal.cuh"
#include "deflate.cuh"
#include "text_chunks.cuh"

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <deque>
#include <mutex>
#include <thread>

namespace dca {
namespace {

constexpr int kFmtThreads = chunked::kThreads;     // fields per tile (256)
constexpr int kMaxField = 48;                      // '-' + 39 digits + '.' + 6 digits + separator
constexpr int kScanThreads = 1024;
constexpr long long kDefaultPiece = 16ll << 20;

// |v| of the float32 with bit pattern b in '%.6f' digits: integer part in base-10^9 groups g0 (lowest) .. g4, six
// fraction digits, sign; kind 0 finite, 1 NaN (empty field), 2 infinity.  len: bytes of the text
struct Fixed6 {
  unsigned g0, g1, g2, g3, g4, frac;
  int top, neg, kind, len;
};

__host__ __device__ __forceinline__ unsigned group_at(const Fixed6& f, int k) {
  return k == 0 ? f.g0 : k == 1 ? f.g1 : k == 2 ? f.g2 : k == 3 ? f.g3 : f.g4;
}

__host__ __device__ __forceinline__ int u32_digits(unsigned x) {
  int n = 1;
  while (x >= 10u) { x /= 10u; ++n; }
  return n;
}

// (hi:lo) / 10^9 in place over four 32-bit limbs (remainder < 2^30, so every partial fits in 64 bits); the remainder
__host__ __device__ __forceinline__ unsigned divmod_1e9(unsigned long long& hi, unsigned long long& lo) {
  unsigned long long r = 0, q;
  unsigned long long x = (r << 32) | (hi >> 32);          q = x / 1000000000ull; r = x - q * 1000000000ull;
  unsigned long long h = q << 32;
  x = (r << 32) | (hi & 0xffffffffull);                    q = x / 1000000000ull; r = x - q * 1000000000ull;
  hi = h | q;
  x = (r << 32) | (lo >> 32);                              q = x / 1000000000ull; r = x - q * 1000000000ull;
  unsigned long long l = q << 32;
  x = (r << 32) | (lo & 0xffffffffull);                    q = x / 1000000000ull; r = x - q * 1000000000ull;
  lo = l | q;
  return (unsigned)r;
}

// host and device: dca_format_fixed6_host runs the same code on the CPU
__host__ __device__ __forceinline__ Fixed6 fixed6(unsigned b) {
  Fixed6 f{0u, 0u, 0u, 0u, 0u, 0u, 0, 0, 0, 0};
  f.neg = (int)(b >> 31);
  const unsigned ef = (b >> 23) & 0xffu, mf = b & 0x7fffffu;
  if (ef == 0xffu) {
    f.kind = mf ? 1 : 2;
    f.len = mf ? 0 : 3 + f.neg;
    return f;
  }
  const unsigned long long m = ef ? (mf | 0x800000u) : mf;
  const int e = ef ? (int)ef - 150 : -149;
  if (e < 0) {
    const unsigned long long p = m * 1000000ull;           // < 2^44
    const int sh = -e;
    unsigned long long q = 0;                              // shifts of 64 or more leave less than half: 0
    if (sh < 64) {
      q = p >> sh;
      const unsigned long long rem = p - (q << sh), half = 1ull << (sh - 1);
      if (rem > half || (rem == half && (q & 1ull))) ++q;
    }
    const unsigned long long ip = q / 1000000ull;          // <= 2^24
    f.frac = (unsigned)(q - ip * 1000000ull);
    f.g0 = (unsigned)ip;
  } else {                                                 // an integer m * 2^e < 2^128
    unsigned long long hi, lo;
    if (e >= 64) { hi = m << (e - 64); lo = 0; }
    else { lo = m << e; hi = e ? (m >> (64 - e)) : 0; }
    f.g0 = divmod_1e9(hi, lo); f.g1 = divmod_1e9(hi, lo); f.g2 = divmod_1e9(hi, lo);
    f.g3 = divmod_1e9(hi, lo); f.g4 = (unsigned)lo;        // < 2^128 / 10^36 < 10^9
  }
  f.top = f.g4 ? 4 : f.g3 ? 3 : f.g2 ? 2 : f.g1 ? 1 : 0;
  f.len = f.neg + 9 * f.top + u32_digits(group_at(f, f.top)) + 7;
  return f;
}

// the f.len bytes of the number at dst
__host__ __device__ __forceinline__ void put_fixed6(char* dst, const Fixed6& f) {
  if (f.kind == 1) return;
  if (f.kind == 2) {
    int p = 0;
    if (f.neg) dst[p++] = '-';
    dst[p] = 'i'; dst[p + 1] = 'n'; dst[p + 2] = 'f';
    return;
  }
  int p = f.len;
  unsigned fr = f.frac;
  for (int i = 0; i < 6; ++i) { dst[--p] = (char)('0' + fr % 10u); fr /= 10u; }
  dst[--p] = '.';
  for (int k = 0; k <= f.top; ++k) {
    unsigned g = group_at(f, k);
    if (k < f.top) {
      for (int i = 0; i < 9; ++i) { dst[--p] = (char)('0' + g % 10u); g /= 10u; }
    } else {
      do { dst[--p] = (char)('0' + g % 10u); g /= 10u; } while (g);
    }
  }
  if (f.neg) dst[--p] = '-';
}

// field j of output line i
__device__ __forceinline__ float field_value(const float* m, long long ld, int transpose, long long i, long long j) {
  return transpose ? m[j * ld + i] : m[i * ld + j];
}

// block (line li, tile k) of a group: seg[li * (tiles + 1) + 1 + k] = bytes of the tile's fields; tile 0 also stores the
// line's label bytes (+ '\t') in seg[li * (tiles + 1)]
__global__ void __launch_bounds__(kFmtThreads) field_len_kernel(const float* m, long long ld, int transpose,
                                                                long long line0, long long cols, int tiles,
                                                                const long long* lab_off, long long* seg) {
  __shared__ int warp_sums[kFmtThreads / 32];
  const long long t = blockIdx.x;
  const long long li = t / tiles;
  const int k = (int)(t - li * tiles);
  const long long j = (long long)k * kFmtThreads + threadIdx.x;
  const int w = j < cols ? fixed6(__float_as_uint(field_value(m, ld, transpose, line0 + li, j))).len + 1 : 0;
  int total;
  chunked::block_exclusive_scan(w, warp_sums, &total);
  if (threadIdx.x == 0) {
    seg[li * (tiles + 1) + 1 + k] = total;
    if (k == 0) seg[li * (tiles + 1)] = lab_off ? lab_off[line0 + li + 1] - lab_off[line0 + li] + 1 : 0;
  }
}

// one CTA: pos[i] = seg[0] + ... + seg[i - 1] for i <= n (pos[n] is the group's byte count), in a fixed order
__global__ void __launch_bounds__(kScanThreads) scan_segs_kernel(const long long* seg, long long n, long long* pos) {
  __shared__ long long warp_sums[kScanThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long per = (n + kScanThreads - 1) / kScanThreads;
  const long long a = std::min(n, (long long)threadIdx.x * per), b = std::min(n, a + per);
  long long s = 0;
  for (long long i = a; i < b; ++i) s += seg[i];
  long long x = s;
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
  long long run = (warp ? warp_sums[warp - 1] : 0) + x - s;
  for (long long i = a; i < b; ++i) { pos[i] = run; run += seg[i]; }
  if (threadIdx.x == kScanThreads - 1) pos[n] = warp_sums[31];
}

// one CTA per line of the group: the label bytes and a '\t'
__global__ void label_write_kernel(const char* labels, const long long* lab_off, long long line0, int tiles,
                                   const long long* pos, char* text) {
  const long long li = blockIdx.x;
  const long long a = lab_off[line0 + li], n = lab_off[line0 + li + 1] - a;
  char* dst = text + pos[li * (tiles + 1)];
  for (long long i = threadIdx.x; i < n; i += blockDim.x) dst[i] = labels[a + i];
  if (threadIdx.x == 0) dst[n] = '\t';
}

// block (line li, tile k): the tile's fields formatted in shared memory at their offsets, then copied out whole
__global__ void __launch_bounds__(kFmtThreads) field_write_kernel(const float* m, long long ld, int transpose,
                                                                  long long line0, long long cols, int tiles,
                                                                  const long long* pos, char* text) {
  __shared__ int warp_sums[kFmtThreads / 32];
  __shared__ char buf[kFmtThreads * kMaxField];
  const long long t = blockIdx.x;
  const long long li = t / tiles;
  const int k = (int)(t - li * tiles);
  const long long j = (long long)k * kFmtThreads + threadIdx.x;
  Fixed6 f{0u, 0u, 0u, 0u, 0u, 0u, 0, 0, 1, 0};
  if (j < cols) f = fixed6(__float_as_uint(field_value(m, ld, transpose, line0 + li, j)));
  const int w = j < cols ? f.len + 1 : 0;
  int total;
  const int off = chunked::block_exclusive_scan(w, warp_sums, &total);
  if (w) {
    put_fixed6(buf + off, f);
    buf[off + w - 1] = j == cols - 1 ? '\n' : '\t';
  }
  __syncthreads();
  char* dst = text + pos[li * (tiles + 1) + 1 + k];
  for (int i = threadIdx.x; i < total; i += kFmtThreads) dst[i] = buf[i];
}

// Everything one call owns; the destructor stops and joins the writer thread and frees on every return path.
struct DeviceTextWriter {
  FILE* f = nullptr;
  int prev_device = -1;
  cudaStream_t s = nullptr;
  char* d_labels = nullptr;
  long long* d_lab_off = nullptr;
  long long *d_seg = nullptr, *d_pos = nullptr;
  char* d_text = nullptr;
  long long text_cap = 0;
  uint8_t* d_gz = nullptr;                             // gzip: the compressed header or group
  long long gz_cap = 0;
  char* h_buf[2] = {nullptr, nullptr};
  long long* h_total = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  // writer thread: appends the pinned pieces in the order they were queued
  std::thread th;
  std::mutex mu;
  std::condition_variable cv;
  std::deque<int> queue;
  long long len[2] = {0, 0};
  bool busy[2] = {false, false};
  bool stop = false, failed = false;
  double wait_ms = 0.0;

  void start() {
    th = std::thread([this] {
      std::unique_lock<std::mutex> lk(mu);
      for (;;) {
        cv.wait(lk, [this] { return stop || !queue.empty(); });
        if (queue.empty()) return;                         // stop with nothing left to write
        const int slot = queue.front();
        queue.pop_front();
        lk.unlock();
        const bool ok = fwrite(h_buf[slot], 1, (size_t)len[slot], f) == (size_t)len[slot];
        lk.lock();
        if (!ok) failed = true;
        busy[slot] = false;
        cv.notify_all();
        if (stop) return;
      }
    });
  }
  // waits until `slot` has been written (or, with slot < 0, both)
  void wait_free(int slot) {
    std::unique_lock<std::mutex> lk(mu);
    cv.wait(lk, [&] { return slot < 0 ? !busy[0] && !busy[1] : !busy[slot]; });
  }
  void submit(int slot, long long n) {
    std::lock_guard<std::mutex> lk(mu);
    len[slot] = n;
    busy[slot] = true;
    queue.push_back(slot);
    cv.notify_all();
  }
  ~DeviceTextWriter() {
    if (th.joinable()) {
      { std::lock_guard<std::mutex> lk(mu); stop = true; queue.clear(); }
      cv.notify_all();
      th.join();
    }
    if (s) (void)cudaStreamSynchronize(s);
    cudaFree(d_labels); cudaFree(d_lab_off); cudaFree(d_seg); cudaFree(d_pos); cudaFree(d_text); cudaFree(d_gz);
    cudaFreeHost(h_buf[0]); cudaFreeHost(h_buf[1]); cudaFreeHost(h_total);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (f) fclose(f);
    if (prev_device >= 0) (void)cudaSetDevice(prev_device);
  }
  // src[0, total) (device) to the file, piece by piece, alternating the pinned buffers
  int send(const char* src, long long total, long long piece, int* slot) {
    for (long long off = 0; off < total; off += piece, *slot ^= 1) {
      const long long n = std::min(piece, total - off);
      const auto t0 = std::chrono::steady_clock::now();
      wait_free(*slot);
      wait_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
      DCA_CUDA_OK(cudaMemcpyAsync(h_buf[*slot], src + off, (size_t)n, cudaMemcpyDeviceToHost, s));
      DCA_CUDA_OK(cudaStreamSynchronize(s));
      submit(*slot, n);
    }
    return DCA_OK;
  }
  // gzip: room for the compressed form of `n` bytes
  int gz_room(long long n) {
    const long long want = deflate::gzip_bound(n);
    if (want <= gz_cap) return DCA_OK;
    DCA_CUDA_OK(cudaFree(d_gz));
    d_gz = nullptr;
    gz_cap = want + want / 4;
    DCA_CUDA_OK(cudaMalloc(&d_gz, (size_t)gz_cap));
    return DCA_OK;
  }
};

}  // namespace
}  // namespace dca

using namespace dca;

namespace {

// dca_write_text_device (who = its name, gz = false) and dca_write_text_device_gz
int write_text_device(const char* who, bool gz, const char* path, int32_t append, const float* matrix, int64_t rows,
                      int64_t cols, int64_t ld, int32_t transpose, const char* header, int64_t header_len,
                      const char* labels, const int64_t* label_offsets, int64_t chunk_bytes, int32_t device,
                      void* stream, int64_t* info) {
  if (!path || !matrix || rows < 1 || cols < 1 || ld < cols || header_len < 0 ||
      (header_len > 0 && !header) || chunk_bytes < 0 || (label_offsets && !labels)) {
    set_error("%s: bad argument", who);
    return DCA_ERR_BAD_ARG;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    (void)cudaGetLastError();
    set_error("%s: no CUDA device available (this library has no CPU fallback)", who);
    return DCA_ERR_NO_DEVICE;
  }
  if (device < 0 || device >= ndev) { set_error("%s: no CUDA device %d", who, device); return DCA_ERR_BAD_ARG; }
  const long long out_rows = transpose ? cols : rows, out_cols = transpose ? rows : cols;
  const long long piece = chunk_bytes ? chunk_bytes : kDefaultPiece;
  const int tiles = cdiv(out_cols, kFmtThreads);
  // whole lines per group: about piece / 8 fields (a field takes 9 to 11 bytes at typical magnitudes)
  const long long group = std::max(1ll, std::min(out_rows, std::max(1ll, piece / 8) / out_cols));
  if (group * (tiles + 1) >= (1ll << 31)) { set_error("%s: too many tiles in a line group", who); return DCA_ERR_BAD_ARG; }

  DeviceTextWriter w;
  DCA_CUDA_OK(cudaGetDevice(&w.prev_device));
  DCA_CUDA_OK(cudaSetDevice(device));
  w.s = (cudaStream_t)stream;
  cudaStream_t s = w.s;
  if (label_offsets) {
    const long long nb = label_offsets[out_rows];
    DCA_CUDA_OK(cudaMalloc(&w.d_lab_off, (size_t)(out_rows + 1) * sizeof(long long)));
    DCA_CUDA_OK(cudaMemcpyAsync(w.d_lab_off, label_offsets, (size_t)(out_rows + 1) * sizeof(long long),
                                cudaMemcpyHostToDevice, s));
    DCA_CUDA_OK(cudaMalloc(&w.d_labels, (size_t)std::max(nb, 1ll)));
    if (nb) DCA_CUDA_OK(cudaMemcpyAsync(w.d_labels, labels, (size_t)nb, cudaMemcpyHostToDevice, s));
  }
  const long long nseg = group * (tiles + 1);
  DCA_CUDA_OK(cudaMalloc(&w.d_seg, (size_t)nseg * sizeof(long long)));
  DCA_CUDA_OK(cudaMalloc(&w.d_pos, (size_t)(nseg + 1) * sizeof(long long)));
  w.text_cap = std::max(1ll << 20, group * out_cols * 12);
  DCA_CUDA_OK(cudaMalloc(&w.d_text, (size_t)w.text_cap));
  DCA_CUDA_OK(cudaHostAlloc(&w.h_buf[0], (size_t)piece, cudaHostAllocDefault));
  DCA_CUDA_OK(cudaHostAlloc(&w.h_buf[1], (size_t)piece, cudaHostAllocDefault));
  DCA_CUDA_OK(cudaHostAlloc(&w.h_total, sizeof(long long), cudaHostAllocDefault));
  DCA_CUDA_OK(cudaEventCreate(&w.ev0));
  DCA_CUDA_OK(cudaEventCreate(&w.ev1));
  deflate::GzipMember member;
  if (gz) {
    DCA_TRY(member.init(s));
    DCA_TRY(w.gz_room(std::max(w.text_cap, (long long)header_len)));
  }

  w.f = fopen(path, append ? "ab" : "wb");
  if (!w.f) { set_error("%s: cannot open %s", who, path); return DCA_ERR_BAD_ARG; }
  long long bytes = 0, groups = 0;
  double kernel_ms = 0.0;
  int slot = 0;
  if (header_len && !gz) {
    if (fwrite(header, 1, (size_t)header_len, w.f) != (size_t)header_len) {
      set_error("%s: write to %s failed", who, path);
      return DCA_ERR_CUDA;
    }
    bytes = header_len;
  }
  w.start();
  if (header_len && gz) {                              // the header line opens the member
    if (header_len > w.text_cap) {
      DCA_CUDA_OK(cudaFree(w.d_text));
      w.d_text = nullptr;
      w.text_cap = header_len;
      DCA_CUDA_OK(cudaMalloc(&w.d_text, (size_t)w.text_cap));
    }
    DCA_CUDA_OK(cudaMemcpyAsync(w.d_text, header, (size_t)header_len, cudaMemcpyHostToDevice, s));
    long long zn = 0;
    DCA_TRY(member.feed((const uint8_t*)w.d_text, header_len, true, false, w.d_gz, &zn));
    DCA_TRY(w.send((const char*)w.d_gz, zn, piece, &slot));
    bytes += zn;
  }
  for (long long line0 = 0; line0 < out_rows; line0 += group, ++groups) {
    const long long lines = std::min(group, out_rows - line0);
    const long long n = lines * (tiles + 1);
    DCA_CUDA_OK(cudaEventRecord(w.ev0, s));
    field_len_kernel<<<(unsigned)(lines * tiles), kFmtThreads, 0, s>>>(matrix, ld, transpose, line0, out_cols, tiles,
                                                                       w.d_lab_off, w.d_seg);
    DCA_LAUNCH_CHECK();
    scan_segs_kernel<<<1, kScanThreads, 0, s>>>(w.d_seg, n, w.d_pos);
    DCA_LAUNCH_CHECK();
    DCA_CUDA_OK(cudaMemcpyAsync(w.h_total, w.d_pos + n, sizeof(long long), cudaMemcpyDeviceToHost, s));
    DCA_CUDA_OK(cudaStreamSynchronize(s));
    float ms = 0.f;
    DCA_CUDA_OK(cudaEventRecord(w.ev1, s));
    DCA_CUDA_OK(cudaEventSynchronize(w.ev1));
    DCA_CUDA_OK(cudaEventElapsedTime(&ms, w.ev0, w.ev1));
    kernel_ms += ms;
    const long long total = *w.h_total;
    if (total > w.text_cap) {
      DCA_CUDA_OK(cudaFree(w.d_text));
      w.d_text = nullptr;
      w.text_cap = total + total / 4;
      DCA_CUDA_OK(cudaMalloc(&w.d_text, (size_t)w.text_cap));
    }
    DCA_CUDA_OK(cudaEventRecord(w.ev0, s));
    if (w.d_lab_off) {
      label_write_kernel<<<(unsigned)lines, 128, 0, s>>>(w.d_labels, w.d_lab_off, line0, tiles, w.d_pos, w.d_text);
      DCA_LAUNCH_CHECK();
    }
    field_write_kernel<<<(unsigned)(lines * tiles), kFmtThreads, 0, s>>>(matrix, ld, transpose, line0, out_cols, tiles,
                                                                         w.d_pos, w.d_text);
    DCA_LAUNCH_CHECK();
    const char* src = w.d_text;
    long long len = total;
    if (gz) {
      DCA_TRY(w.gz_room(total));
      DCA_TRY(member.feed((const uint8_t*)w.d_text, total, groups == 0 && !header_len, line0 + lines == out_rows,
                          w.d_gz, &len));
      src = (const char*)w.d_gz;
    }
    DCA_CUDA_OK(cudaEventRecord(w.ev1, s));
    DCA_CUDA_OK(cudaEventSynchronize(w.ev1));
    DCA_CUDA_OK(cudaEventElapsedTime(&ms, w.ev0, w.ev1));
    kernel_ms += ms;
    DCA_TRY(w.send(src, len, piece, &slot));
    bytes += len;
  }
  const auto t0 = std::chrono::steady_clock::now();
  w.wait_free(-1);
  w.wait_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  const bool failed = w.failed;
  const int cl = fclose(w.f);
  w.f = nullptr;
  if (failed || cl != 0) { set_error("%s: write to %s failed", who, path); return DCA_ERR_CUDA; }
  if (info) {
    info[0] = bytes;
    info[1] = groups;
    info[2] = (int64_t)(kernel_ms * 1e3);
    info[3] = (int64_t)(w.wait_ms * 1e3);
  }
  return DCA_OK;
}

}  // namespace

extern "C" int dca_write_text_device(const char* path, int32_t append, const float* matrix, int64_t rows, int64_t cols,
                                     int64_t ld, int32_t transpose, const char* header, int64_t header_len,
                                     const char* labels, const int64_t* label_offsets, int64_t chunk_bytes,
                                     int32_t device, void* stream, int64_t* info) {
  return write_text_device("dca_write_text_device", false, path, append, matrix, rows, cols, ld, transpose, header,
                           header_len, labels, label_offsets, chunk_bytes, device, stream, info);
}

extern "C" int dca_write_text_device_gz(const char* path, int32_t append, const float* matrix, int64_t rows,
                                        int64_t cols, int64_t ld, int32_t transpose, const char* header,
                                        int64_t header_len, const char* labels, const int64_t* label_offsets,
                                        int64_t chunk_bytes, int32_t device, void* stream, int64_t* info) {
  return write_text_device("dca_write_text_device_gz", true, path, append, matrix, rows, cols, ld, transpose, header,
                           header_len, labels, label_offsets, chunk_bytes, device, stream, info);
}

// The formatter of the kernels above, run on the CPU: out gets the '%.6f' text of the float32 bit patterns bits[0..n)
// back to back, offsets[i] .. offsets[i + 1] that of bits[i] (int64[n + 1]; out holds at least 47 * n bytes).
extern "C" int dca_format_fixed6_host(const uint32_t* bits, int64_t n, char* out, int64_t* offsets) {
  if (!bits || !out || !offsets || n < 0) { set_error("dca_format_fixed6_host: bad argument"); return DCA_ERR_BAD_ARG; }
  int64_t p = 0;
  for (int64_t i = 0; i < n; ++i) {
    offsets[i] = p;
    const Fixed6 f = fixed6(bits[i]);
    put_fixed6(out + p, f);
    p += f.len;
  }
  offsets[n] = p;
  return DCA_OK;
}
