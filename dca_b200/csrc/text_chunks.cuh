// Chunked reading of a text file on the device, shared by the GPU readers of count tables (read_text.cu) and of
// Matrix Market files (read_mtx.cu).
//
// The host reads the bytes (of the file, or of a gzip file's inflated stream: ByteSource) in chunks into two pinned
// staging buffers; a chunk ends at its last '\n' and the partial
// line carries over to the next one, so the disk read of one chunk overlaps the copy and the kernels of the other.
// Per chunk, on the caller's stream (text_chunks.cu):
//   tile_count    per 4 KB tile: '\n' and separator counts; flags quotes, NUL bytes and a '\r' without '\n'
//   scan_tiles    one CTA: exclusive prefix of both counts over the tiles; the chunk's line count and first line
//   line_ends     position of every '\n' and the number of separators before it
// and then the reader's own kernels.  Problems are recorded as min((file offset << 8) | reason), so the first one in
// file order is reported.
#pragma once
#include "dca_internal.cuh"

#include <functional>
#include <memory>

namespace dca {
namespace chunked {

constexpr int kThreads = 256;
constexpr int kBytesPerThread = 16;
constexpr int kTile = kThreads * kBytesPerThread;      // 4096 bytes per CTA
constexpr int64_t kDefaultChunk = 64ll << 20;

// reasons flagged by the shared kernels (the readers number their own reasons around these)
enum : int { R_NONE = 0, R_QUOTE = 1, R_NUL = 2, R_CR = 3, R_LINES = 9 };

// device state of one read (zeroed, err = ~0, by the host before the first chunk); readers extend it
struct ChunkState {
  unsigned long long err;        // min((file offset << 8) | reason), ~0 when clean
  long long lines_done;          // lines of the chunks before the current one, then including it
  long long chunk_base;          // first line of the current chunk
  int chunk_lines;               // lines of the current chunk (including an unterminated last line)
  int chunk_seps;
};

__device__ __forceinline__ void flag(ChunkState* st, long long pos, int reason) {
  atomicMin(&st->err, ((unsigned long long)pos << 8) | (unsigned)reason);
}

// exclusive block scan of one int per thread (kThreads threads); returns the block total in *total
__device__ __forceinline__ int block_exclusive_scan(int v, int* smem_warp, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) smem_warp[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = lane < kThreads / 32 ? smem_warp[lane] : 0;
#pragma unroll
    for (int o = 1; o < kThreads / 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
    if (lane < kThreads / 32) smem_warp[lane] = w;          // inclusive warp totals
  }
  __syncthreads();
  const int before = (warp ? smem_warp[warp - 1] : 0) + x - v;
  *total = smem_warp[kThreads / 32 - 1];
  return before;
}

// the 16 bytes of this thread (the buffer is padded to whole tiles), and byte i of them without a local array
__device__ __forceinline__ uint4 load16(const unsigned char* buf, long long p) {
  return *reinterpret_cast<const uint4*>(buf + p);
}
__device__ __forceinline__ unsigned byte_at(const uint4& q, int i) {
  const unsigned w = i < 8 ? (i < 4 ? q.x : q.y) : (i < 12 ? q.z : q.w);
  return (w >> ((i & 3) * 8)) & 0xffu;
}

// packed ('\n' count << 16) | separator count of 16 bytes from p (bytes at or beyond n do not count)
__device__ __forceinline__ int count16(const uint4& q, long long p, long long n, unsigned char sep) {
  int nl = 0, sp = 0;
#pragma unroll
  for (int i = 0; i < kBytesPerThread; ++i) {
    const bool in = p + i < n;
    const unsigned x = byte_at(q, i);
    nl += in && x == '\n';
    sp += in && x == sep;
  }
  return (nl << 16) | sp;
}

// read() until `want` bytes or the end of the file: the bytes read, -1 on an error
long long read_full(int fd, unsigned char* dst, long long want);

// Where a reader's bytes come from: the file (open_file_source), or the inflated stream of a gzip file
// (open_gzip_source, inflate.cu), whose bytes are inflated on the device segment by segment as they are read.
struct ByteSource {
  virtual ~ByteSource() = default;
  // up to `want` bytes into dst (fewer only at the end); a negative status (message set) on an error or a decline
  virtual long long read(unsigned char* dst, long long want) = 0;
  virtual int seek(long long off) = 0;       // to byte `off` of the stream
  virtual long long tell() = 0;
};
int open_file_source(const char* who, const char* path, std::unique_ptr<ByteSource>* out);
int open_gzip_source(const char* who, const char* path, std::unique_ptr<ByteSource>* out);
long long gzip_source_device_bytes();        // device memory of a gzip source at most

// chunk sizes of one read: chunk bytes, the padded device buffer, its tiles, and the most lines a chunk may hold when
// every line has `fields` non-empty fields (at least 2 * fields - 1 bytes besides its '\n'; more is flagged R_LINES)
struct ChunkGeometry {
  long long cap = 0, padded = 0;
  int tiles_cap = 0, max_lines = 0;
};
ChunkGeometry chunk_geometry(long long chunk_bytes, int fields);

// one of the two staging buffers and the per-chunk arrays of the shared kernels
struct ChunkBuffers {
  unsigned char* h_buf = nullptr;      // pinned staging
  int* h_count = nullptr;              // mapped: lines of the chunk
  int* d_count = nullptr;              // device view of h_count
  unsigned char* d_buf = nullptr;
  int *tile_nl = nullptr, *tile_sep = nullptr, *nl_pos = nullptr, *nl_seprank = nullptr;
  cudaEvent_t done = nullptr;
  bool busy = false;
  int alloc(const ChunkGeometry& g);
  void release();                      // waits for the chunk in flight, then frees
};

// Reads the source from its current offset (file_off bytes into it) to the end, chunk by chunk through b0 / b1, and per
// chunk enqueues the copy, the three shared kernels (separator `sep`, state st) and launch(buffer, chunk index, chunk
// bytes, file offset, tiles), then an event.  collect(buffer) runs on the host once a buffer's chunk is done, before
// the buffer is reused and for both buffers at the end; a positive return stops the read (no further chunk is
// started), a negative one is returned as the status.  `who` prefixes the error messages.
int for_each_chunk(const char* who, ByteSource& src, long long file_off, const ChunkGeometry& g, ChunkBuffers& b0,
                   ChunkBuffers& b1, unsigned char sep, ChunkState* st, cudaStream_t s,
                   const std::function<int(ChunkBuffers&, long long chunk, long long end, long long file_off, int tiles)>& launch,
                   const std::function<int(ChunkBuffers&)>& collect);

}  // namespace chunked
}  // namespace dca
