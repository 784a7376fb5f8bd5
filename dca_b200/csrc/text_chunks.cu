// Chunked reading of a text file on the device (text_chunks.cuh): the pinned double buffer, the carry of a partial
// line, and the tile count and scan of line ends every chunk goes through.
#include "text_chunks.cuh"

#include <fcntl.h>
#include <unistd.h>

#include <algorithm>
#include <climits>
#include <cstring>

namespace dca {
namespace chunked {
namespace {

__global__ void __launch_bounds__(kThreads) tile_count_kernel(const unsigned char* __restrict__ buf, long long n,
                                                              unsigned char sep, int* tile_nl, int* tile_sep,
                                                              ChunkState* st, long long file_off) {
  __shared__ int sw[kThreads / 32];
  const long long p = (long long)blockIdx.x * kTile + threadIdx.x * kBytesPerThread;
  const uint4 q = load16(buf, p);
  const int c = count16(q, p, n, sep);
#pragma unroll
  for (int i = 0; i < kBytesPerThread; ++i) {
    if (p + i >= n) break;
    const unsigned x = byte_at(q, i);
    if (x == '"') flag(st, file_off + p + i, R_QUOTE);
    else if (x == 0) flag(st, file_off + p + i, R_NUL);
    else if (x == '\r' && (p + i + 1 >= n || buf[p + i + 1] != '\n')) flag(st, file_off + p + i, R_CR);
  }
  int total;
  (void)block_exclusive_scan(c, sw, &total);
  if (threadIdx.x == 0) { tile_nl[blockIdx.x] = total >> 16; tile_sep[blockIdx.x] = total & 0xffff; }
}

// one CTA: exclusive prefixes of the tile counts, the chunk's line count (+1 for an unterminated last line, which
// gets a virtual '\n' at n) and its first line
__global__ void __launch_bounds__(1024) scan_tiles_kernel(int* tile_nl, int* tile_sep, int tiles, long long n, int tail_line,
                                                          int max_lines, int* nl_pos, int* nl_seprank, ChunkState* st,
                                                          int* h_count, long long file_off) {
  __shared__ int s_nl[1024], s_sep[1024];
  __shared__ int carry_nl, carry_sep;
  if (threadIdx.x == 0) { carry_nl = 0; carry_sep = 0; }
  __syncthreads();
  for (int base = 0; base < tiles; base += 1024) {
    const int i = base + threadIdx.x;
    const int a = i < tiles ? tile_nl[i] : 0, b = i < tiles ? tile_sep[i] : 0;
    s_nl[threadIdx.x] = a; s_sep[threadIdx.x] = b;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {          // Hillis-Steele inclusive scan
      const int x = threadIdx.x >= o ? s_nl[threadIdx.x - o] : 0, y = threadIdx.x >= o ? s_sep[threadIdx.x - o] : 0;
      __syncthreads();
      s_nl[threadIdx.x] += x; s_sep[threadIdx.x] += y;
      __syncthreads();
    }
    if (i < tiles) { tile_nl[i] = carry_nl + s_nl[threadIdx.x] - a; tile_sep[i] = carry_sep + s_sep[threadIdx.x] - b; }
    __syncthreads();
    if (threadIdx.x == 0) { carry_nl += s_nl[1023]; carry_sep += s_sep[1023]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    int lines = carry_nl + tail_line;
    if (lines > max_lines) { flag(st, file_off, R_LINES); lines = max_lines; }
    if (tail_line && carry_nl < max_lines) { nl_pos[carry_nl] = (int)n; nl_seprank[carry_nl] = carry_sep; }
    st->chunk_base = st->lines_done;
    st->lines_done += lines;
    st->chunk_lines = lines;
    st->chunk_seps = carry_sep;
    *h_count = lines;
  }
}

__global__ void __launch_bounds__(kThreads) line_ends_kernel(const unsigned char* __restrict__ buf, long long n,
                                                             unsigned char sep, const int* __restrict__ tile_nl,
                                                             const int* __restrict__ tile_sep, int max_lines, int* nl_pos,
                                                             int* nl_seprank) {
  __shared__ int sw[kThreads / 32];
  const long long p = (long long)blockIdx.x * kTile + threadIdx.x * kBytesPerThread;
  const uint4 q = load16(buf, p);
  int total;
  const int before = block_exclusive_scan(count16(q, p, n, sep), sw, &total);
  int nl = tile_nl[blockIdx.x] + (before >> 16), sp = tile_sep[blockIdx.x] + (before & 0xffff);
#pragma unroll
  for (int i = 0; i < kBytesPerThread; ++i) {
    if (p + i >= n) break;
    const unsigned x = byte_at(q, i);
    if (x == '\n') {
      if (nl < max_lines) { nl_pos[nl] = (int)(p + i); nl_seprank[nl] = sp; }
      ++nl;
    } else if (x == sep) {
      ++sp;
    }
  }
}

}  // namespace

long long read_full(int fd, unsigned char* dst, long long want) {
  long long got = 0;
  while (got < want) {
    const ssize_t r = ::read(fd, dst + got, (size_t)std::min<long long>(want - got, 1ll << 30));
    if (r < 0) return -1;
    if (r == 0) break;
    got += r;
  }
  return got;
}

namespace {
class FileSource : public ByteSource {
 public:
  FileSource(const char* who, int fd) : who_(who), fd_(fd) {}
  ~FileSource() override { close(fd_); }
  long long read(unsigned char* dst, long long want) override {
    const long long got = read_full(fd_, dst, want);
    if (got < 0) { set_error("%s: read failed", who_); return DCA_ERR_BAD_ARG; }
    return got;
  }
  int seek(long long off) override {
    if (lseek(fd_, off, SEEK_SET) != off) { set_error("%s: seek failed", who_); return DCA_ERR_BAD_ARG; }
    return DCA_OK;
  }
  long long tell() override { return lseek(fd_, 0, SEEK_CUR); }

 private:
  const char* who_;
  int fd_;
};
}  // namespace

int open_file_source(const char* who, const char* path, std::unique_ptr<ByteSource>* out) {
  const int fd = open(path, O_RDONLY);
  if (fd < 0) { set_error("%s: cannot open %s", who, path); return DCA_ERR_BAD_ARG; }
  out->reset(new FileSource(who, fd));
  return DCA_OK;
}

ChunkGeometry chunk_geometry(long long chunk_bytes, int fields) {
  ChunkGeometry g;
  g.cap = chunk_bytes ? chunk_bytes : kDefaultChunk;
  g.padded = (g.cap + 16 + kTile - 1) / kTile * kTile;       // whole tiles + the byte after the last one
  g.tiles_cap = (int)(g.padded / kTile);
  g.max_lines = (int)std::min<long long>(g.cap / (2ll * fields) + 2, INT32_MAX / 2);
  return g;
}

int ChunkBuffers::alloc(const ChunkGeometry& g) {
  DCA_CUDA_OK(cudaHostAlloc(&h_buf, (size_t)g.padded, cudaHostAllocDefault));
  DCA_CUDA_OK(cudaHostAlloc(&h_count, sizeof(int), cudaHostAllocMapped));
  DCA_CUDA_OK(cudaHostGetDevicePointer((void**)&d_count, h_count, 0));
  DCA_CUDA_OK(cudaMalloc(&d_buf, (size_t)g.padded));
  DCA_CUDA_OK(cudaMalloc(&tile_nl, (size_t)g.tiles_cap * sizeof(int)));
  DCA_CUDA_OK(cudaMalloc(&tile_sep, (size_t)g.tiles_cap * sizeof(int)));
  DCA_CUDA_OK(cudaMalloc(&nl_pos, (size_t)g.max_lines * sizeof(int)));
  DCA_CUDA_OK(cudaMalloc(&nl_seprank, (size_t)g.max_lines * sizeof(int)));
  DCA_CUDA_OK(cudaEventCreateWithFlags(&done, cudaEventDisableTiming));
  return DCA_OK;
}

void ChunkBuffers::release() {
  if (done) { cudaEventSynchronize(done); cudaEventDestroy(done); done = nullptr; }
  cudaFreeHost(h_buf); cudaFreeHost(h_count);
  cudaFree(d_buf); cudaFree(tile_nl); cudaFree(tile_sep); cudaFree(nl_pos); cudaFree(nl_seprank);
  h_buf = nullptr; h_count = nullptr; d_buf = nullptr; tile_nl = tile_sep = nl_pos = nl_seprank = nullptr;
}

int for_each_chunk(const char* who, ByteSource& src, long long file_off, const ChunkGeometry& g, ChunkBuffers& b0,
                   ChunkBuffers& b1, unsigned char sep, ChunkState* st, cudaStream_t s,
                   const std::function<int(ChunkBuffers&, long long, long long, long long, int)>& launch,
                   const std::function<int(ChunkBuffers&)>& collect) {
  ChunkBuffers* b[2] = {&b0, &b1};
  // a finished chunk: collect() before its buffer is reused; > 0 stops the read
  auto finish = [&](ChunkBuffers& x) -> int {
    if (!x.busy) return DCA_OK;
    DCA_CUDA_OK(cudaEventSynchronize(x.done));
    x.busy = false;
    return collect(x);
  };
  const long long cap = g.cap;
  long long carry = 0, chunk = 0;
  int cur = 0;
  for (;;) {
    ChunkBuffers& x = *b[cur];
    const long long got = src.read(x.h_buf + carry, cap - carry);
    if (got < 0) return (int)got;
    const long long len = carry + got;
    if (len == 0) break;
    const bool eof = got < cap - carry;
    long long end = len;
    if (!eof) {
      const void* q = nullptr;
      for (long long i = len - 1; i >= 0 && !q; --i) if (x.h_buf[i] == '\n') q = x.h_buf + i;
      if (!q) {
        set_error("%s: unsupported file: a line longer than chunk_bytes (%lld) at byte %lld", who, cap, file_off);
        return DCA_ERR_UNSUPPORTED;
      }
      end = (const unsigned char*)q - x.h_buf + 1;
    }
    ChunkBuffers& y = *b[cur ^ 1];
    const int stop = finish(y);               // the other buffer's chunk is done: collected, then its staging is free
    if (stop < 0) return stop;
    if (stop > 0) break;
    carry = len - end;
    if (carry) memcpy(y.h_buf, x.h_buf + end, (size_t)carry);
    const int tail_line = x.h_buf[end - 1] != '\n';
    const int tiles = (int)((end + kTile - 1) / kTile);
    DCA_CUDA_OK(cudaMemcpyAsync(x.d_buf, x.h_buf, (size_t)end, cudaMemcpyHostToDevice, s));
    DCA_CUDA_OK(cudaMemsetAsync(x.d_buf + end, 0, (size_t)(g.padded - end), s));
    tile_count_kernel<<<tiles, kThreads, 0, s>>>(x.d_buf, end, sep, x.tile_nl, x.tile_sep, st, file_off);
    DCA_LAUNCH_CHECK();
    scan_tiles_kernel<<<1, 1024, 0, s>>>(x.tile_nl, x.tile_sep, tiles, end, tail_line, g.max_lines, x.nl_pos,
                                         x.nl_seprank, st, x.d_count, file_off);
    DCA_LAUNCH_CHECK();
    line_ends_kernel<<<tiles, kThreads, 0, s>>>(x.d_buf, end, sep, x.tile_nl, x.tile_sep, g.max_lines, x.nl_pos,
                                                x.nl_seprank);
    DCA_LAUNCH_CHECK();
    DCA_TRY(launch(x, chunk, end, file_off, tiles));
    DCA_CUDA_OK(cudaEventRecord(x.done, s));
    x.busy = true;
    file_off += end;
    ++chunk;
    cur ^= 1;
    if (eof && carry == 0) break;
  }
  const int s0 = finish(*b[0]);
  if (s0 < 0) return s0;
  const int s1 = finish(*b[1]);
  return s1 < 0 ? s1 : DCA_OK;
}

}  // namespace chunked
}  // namespace dca
