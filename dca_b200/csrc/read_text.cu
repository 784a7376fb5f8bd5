// GPU reader of gene x cell count tables in TSV / CSV (dca_read_text_counts, include/dca_b200.h): the matrix and
// labels pd.read_csv(path, sep=sep, index_col=0).values.astype(np.float32) gives, bit for bit, for the files whose
// every value field is [0-9]+ or [0-9]+\.0* (anything else is reported as DCA_ERR_UNSUPPORTED and read by pandas).
//
// The file goes through the chunked reader of text_chunks.cuh (two pinned staging buffers; per chunk the tile count,
// the tile scan and the line ends).  Then per chunk, on the caller's stream:
//   parse_values  every separator starts a value field: line = '\n' rank, column = separator rank - the line's first
//                 separator rank; digits go into a uint64 and __ull2float_rn (NumPy's int64 -> float32 cast)
//   line_check    field count of every line; label extents into mapped host memory for the host to copy
//   transpose     (transpose != 0) the chunk's rows, staged in file order, into columns of the output by 32 x 32 tiles
// Problems are recorded as min((file offset << 8) | reason), so the first one in file order is reported.
#include "text_chunks.cuh"

#include <fcntl.h>
#include <unistd.h>

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

namespace dca {
namespace {

using namespace chunked;

constexpr int kMaxDigits = 18;                         // < 2^63: pandas parses the column as int64
constexpr int kMaxToken = 64;                          // longer value fields ("1.000...") go to pandas

enum Reason : int { R_FIELDS = 4, R_EMPTY, R_CHAR, R_DIGITS, R_ROWS, R_BIG_DOT = 10 };   // R_QUOTE..R_CR, R_LINES: chunked
const char* reason_text(int r) {
  switch (r) {
    case R_QUOTE: return "a quote character in a data line";
    case R_NUL: return "a NUL byte";
    case R_CR: return "a carriage return not followed by a line feed";
    case R_FIELDS: return "a line whose field count differs from the header's (ragged or blank line, or implicit index)";
    case R_EMPTY: return "an empty value field";
    case R_CHAR: return "a value field that is not [0-9]+ or [0-9]+.0* (sign, fraction, exponent, NA token or space)";
    case R_DIGITS: return "a value with more than 18 digits";
    case R_ROWS: return "more data lines than the first pass counted (the file changed)";
    case R_LINES: return "more lines in a chunk than its fields allow (blank or short lines)";
    case R_BIG_DOT: return "a '.0' value field next to a value above 2^53 (pandas rounds those through float64)";
    default: return "unknown";
  }
}

// device state of one read (zeroed / set by the host before the first chunk)
struct ReadState : ChunkState {
  unsigned long long max_val;    // largest value field
  int any_dot;                   // some value field has a '.'
};

// Value fields.  Every separator starts one; its line is the number of '\n' before it and its column the number of
// separators between the line's start and it.  out: row-major [rows x cols] (row = file line) when stage == NULL,
// else the chunk's rows go to stage [chunk lines x cols]; neither when both are NULL (first pass).
__global__ void __launch_bounds__(kThreads) parse_values_kernel(const unsigned char* __restrict__ buf, long long n,
                                                                unsigned char sep, const int* __restrict__ tile_nl,
                                                                const int* __restrict__ tile_sep,
                                                                const int* __restrict__ nl_seprank, int* label_end,
                                                                int max_lines, int cols, long long rows, float* out,
                                                                float* stage, ReadState* st, long long file_off) {
  __shared__ int sw[kThreads / 32];
  const long long p = (long long)blockIdx.x * kTile + threadIdx.x * kBytesPerThread;
  const uint4 q = load16(buf, p);
  int total;
  const int before = block_exclusive_scan(count16(q, p, n, sep), sw, &total);
  int nl = tile_nl[blockIdx.x] + (before >> 16), sp = tile_sep[blockIdx.x] + (before & 0xffff);
  const long long row0 = st->chunk_base;
  int line_first = -1, line_of_first = -1;            // separator rank of the first separator of line `nl`
  unsigned long long vmax = 0;
  int dot = 0;
  for (int i = 0; i < kBytesPerThread; ++i) {
    const long long s = p + i;
    if (s >= n) break;
    const unsigned c = byte_at(q, i);
    if (c == '\n') { ++nl; continue; }
    if (c != sep) continue;
    const int rank = sp++;
    if (nl >= max_lines) continue;                      // flagged by scan_tiles_kernel
    if (line_of_first != nl) { line_first = nl ? nl_seprank[nl - 1] : 0; line_of_first = nl; }
    const int col = rank - line_first;
    if (col == 0) label_end[nl] = (int)s;
    // the value field after the separator
    unsigned long long v = 0;
    int digits = 0, len = 0, state = 0, bad = R_NONE;     // state 0: digits, 1: after '.', zeros only
    long long q = s + 1;
    for (; q < n; ++q, ++len) {
      const unsigned char x = buf[q];
      if (x == sep || x == '\n' || x == '\r') break;
      if (len >= kMaxToken) { bad = R_CHAR; break; }
      if (x >= '0' && x <= '9') {
        if (state == 0) { v = v * 10ull + (x - '0'); if (++digits > kMaxDigits) { bad = R_DIGITS; break; } }
        else if (x != '0') { bad = R_CHAR; break; }
      } else if (x == '.' && state == 0 && digits > 0) {
        state = 1; dot = 1;
      } else {
        bad = R_CHAR; break;
      }
    }
    if (!bad && len == 0) bad = R_EMPTY;
    if (!bad && col >= cols) bad = R_FIELDS;
    if (bad) { flag(st, file_off + s + 1, bad); continue; }
    vmax = v > vmax ? v : vmax;
    const float f = __ull2float_rn(v);
    if (stage) stage[(long long)nl * cols + col] = f;
    else if (out && row0 + nl < rows) out[(row0 + nl) * (long long)cols + col] = f;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const unsigned long long y = __shfl_xor_sync(0xffffffffu, vmax, o);
    vmax = y > vmax ? y : vmax;
    dot |= __shfl_xor_sync(0xffffffffu, dot, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (vmax) atomicMax(&st->max_val, vmax);
    if (dot) atomicOr(&st->any_dot, 1);
  }
}

// per line of the chunk: field count, row bound, label extent (chunk offsets) into mapped host memory
__global__ void __launch_bounds__(kThreads) line_check_kernel(const int* __restrict__ nl_pos, const int* __restrict__ nl_seprank,
                                                              const int* __restrict__ label_end, int fields, long long rows,
                                                              int* h_lab, ReadState* st, long long file_off) {
  const int lines = st->chunk_lines;
  const long long row0 = st->chunk_base;
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < lines; k += gridDim.x * blockDim.x) {
    const int start = k ? nl_pos[k - 1] + 1 : 0;
    const int f = nl_seprank[k] - (k ? nl_seprank[k - 1] : 0) + 1;
    if (f != fields) flag(st, file_off + start, R_FIELDS);
    else if (rows >= 0 && row0 + k >= rows) flag(st, file_off + start, R_ROWS);
    h_lab[2 * k] = start;
    h_lab[2 * k + 1] = f == fields ? label_end[k] : start;
  }
}

// stage [chunk lines x cols] (file order) -> out[c * rows + chunk_base + r]
__global__ void __launch_bounds__(1024) transpose_kernel(const float* __restrict__ stage, int cols, long long rows,
                                                         float* __restrict__ out, const ReadState* st) {
  __shared__ float t[32][33];
  const int lines = st->chunk_lines;
  const long long row0 = st->chunk_base;
  const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  if (r0 >= lines) return;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  if (r0 + ty < lines && c0 + tx < cols) t[ty][tx] = stage[(long long)(r0 + ty) * cols + c0 + tx];
  __syncthreads();
  if (c0 + ty < cols && r0 + tx < lines && row0 + r0 + tx < rows) out[(long long)(c0 + ty) * rows + row0 + r0 + tx] = t[tx][ty];
}

// ---------------------------------------------------------------------------------------------------------- host
// a staging buffer with the label and transpose arrays of this reader
struct Buffers : ChunkBuffers {
  int* h_lab = nullptr;                // mapped: 2 ints per line
  int* d_lab = nullptr;                // device view of h_lab
  int* label_end = nullptr;
  float* stage = nullptr;
};

struct Reader {
  std::unique_ptr<ByteSource> src;
  int prev_device = -1;                // the caller's current device, restored on return
  ReadState* d_state = nullptr;
  Buffers b[2];
  ~Reader() {
    release();
    if (prev_device >= 0) cudaSetDevice(prev_device);
  }
  void release() {
    src.reset();
    for (Buffers& x : b) {
      x.release();
      cudaFreeHost(x.h_lab); cudaFree(x.label_end); cudaFree(x.stage);
    }
    cudaFree(d_state);
  }
};

// The header line: its byte length (with the line end) and field count; DCA_ERR_UNSUPPORTED for a header pandas would
// read differently from a plain split (quotes, NUL, a lone '\r') or a file without data lines.
int read_header(const char* who, ByteSource& src, unsigned char sep, long long* header_bytes, int* fields) {
  std::string h;
  unsigned char tmp[65536];
  long long nl = -1;
  while (nl < 0) {
    const long long r = src.read(tmp, sizeof(tmp));
    if (r < 0) return (int)r;
    const size_t old = h.size();
    h.append((const char*)tmp, (size_t)r);
    const void* q = memchr(h.data() + old, '\n', (size_t)r);
    if (q) nl = (const char*)q - h.data();
    else if (r == 0) { set_error("%s: unsupported file: no data lines", who); return DCA_ERR_UNSUPPORTED; }
  }
  long long end = nl;
  if (end > 0 && h[(size_t)end - 1] == '\r') --end;
  int f = 1;
  for (long long i = 0; i < end; ++i) {
    const unsigned char c = (unsigned char)h[(size_t)i];
    if (c == '"' || c == 0 || c == '\r') {
      set_error("%s: unsupported file: a quote, NUL or carriage return in the header line", who);
      return DCA_ERR_UNSUPPORTED;
    }
    f += c == sep;
  }
  *header_bytes = nl + 1;
  *fields = f;
  return DCA_OK;
}

}  // namespace
}  // namespace dca

using namespace dca;

namespace {
// both entry points: the file's bytes, or (gz) the inflated bytes of a gzip file
int read_text_counts(const char* who, bool gz, const char* path, int32_t sep, int32_t transpose, int64_t chunk_bytes,
                     int32_t device, void* stream, float* out, int64_t out_elems, int64_t* label_offsets,
                     char* label_bytes, int64_t label_cap, int64_t* info) {
  if (!path || !info || sep <= 0 || sep > 127 || sep == '\n' || sep == '\r' || sep == '"' || chunk_bytes < 0 ||
      (out && (!label_offsets || (label_cap > 0 && !label_bytes)))) {
    set_error("%s: bad argument", who); return DCA_ERR_BAD_ARG;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    (void)cudaGetLastError();
    set_error("%s: no CUDA device available (this library has no CPU fallback)", who);
    return DCA_ERR_NO_DEVICE;
  }
  if (device < 0 || device >= ndev) { set_error("%s: no CUDA device %d", who, device); return DCA_ERR_BAD_ARG; }
  Reader rd;
  DCA_CUDA_OK(cudaGetDevice(&rd.prev_device));
  DCA_CUDA_OK(cudaSetDevice(device));
  const bool fill = out != nullptr;
  const long long rows_expect = fill ? info[0] : -1;
  if (fill && (info[0] <= 0 || info[1] <= 0 || out_elems < info[0] * info[1] || label_cap < info[2])) {
    set_error("%s: the outputs do not match the sizes of the first call", who); return DCA_ERR_BAD_ARG;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned char sp = (unsigned char)sep;

  DCA_TRY(gz ? open_gzip_source(who, path, &rd.src) : open_file_source(who, path, &rd.src));
  long long header_bytes = 0; int fields = 0;
  DCA_TRY(read_header(who, *rd.src, sp, &header_bytes, &fields));
  if (fields < 2) { set_error("%s: unsupported file: no value columns", who); return DCA_ERR_UNSUPPORTED; }
  const int cols = fields - 1;
  DCA_TRY(rd.src->seek(header_bytes));

  const ChunkGeometry geo = chunk_geometry(chunk_bytes, fields);
  const long long cap = geo.cap, padded = geo.padded;
  if (cap > (1ll << 30)) { set_error("%s: chunk_bytes above 1 GB", who); return DCA_ERR_BAD_ARG; }
  const int tiles_cap = geo.tiles_cap, max_lines = geo.max_lines;
  const bool staged = fill && transpose;

  DCA_CUDA_OK(cudaMalloc(&rd.d_state, sizeof(ReadState)));
  for (Buffers& x : rd.b) {
    DCA_TRY(x.alloc(geo));
    DCA_CUDA_OK(cudaHostAlloc(&x.h_lab, (size_t)max_lines * 2 * sizeof(int), cudaHostAllocMapped));
    DCA_CUDA_OK(cudaHostGetDevicePointer((void**)&x.d_lab, x.h_lab, 0));
    DCA_CUDA_OK(cudaMalloc(&x.label_end, (size_t)max_lines * sizeof(int)));
    if (staged) DCA_CUDA_OK(cudaMalloc(&x.stage, (size_t)max_lines * cols * sizeof(float)));
  }
  {
    ReadState init{};
    init.err = ~0ull;
    DCA_CUDA_OK(cudaMemcpyAsync(rd.d_state, &init, sizeof(init), cudaMemcpyHostToDevice, s));
  }

  long long rows = 0, labels = 0;
  // labels of a finished chunk, from its staging bytes (the buffer is reused only after this)
  auto collect = [&](ChunkBuffers& cb) -> int {
    const Buffers& x = static_cast<const Buffers&>(cb);
    const int n = *x.h_count;
    for (int k = 0; k < n; ++k) {
      const int a = x.h_lab[2 * k], e = x.h_lab[2 * k + 1];
      const long long len = e - a;
      if (fill && rows < rows_expect && labels + len <= label_cap) {
        label_offsets[rows] = labels;
        if (len) memcpy(label_bytes + labels, x.h_buf + a, (size_t)len);
      }
      labels += len;
      ++rows;
    }
    return DCA_OK;
  };
  auto launch = [&](ChunkBuffers& cb, long long, long long end, long long file_off, int tiles) -> int {
    Buffers& x = static_cast<Buffers&>(cb);
    parse_values_kernel<<<tiles, kThreads, 0, s>>>(x.d_buf, end, sp, x.tile_nl, x.tile_sep, x.nl_seprank, x.label_end,
                                                   max_lines, cols, rows_expect, staged ? nullptr : out, x.stage,
                                                   rd.d_state, file_off);
    DCA_LAUNCH_CHECK();
    line_check_kernel<<<std::max(1, std::min(1024, cdiv(max_lines, kThreads))), kThreads, 0, s>>>(
        x.nl_pos, x.nl_seprank, x.label_end, fields, rows_expect, x.d_lab, rd.d_state, file_off);
    DCA_LAUNCH_CHECK();
    if (staged) {
      const dim3 grid((unsigned)cdiv(max_lines, 32), (unsigned)cdiv(cols, 32));
      transpose_kernel<<<grid, 1024, 0, s>>>(x.stage, cols, rows_expect, out, rd.d_state);
      DCA_LAUNCH_CHECK();
    }
    return DCA_OK;
  };
  DCA_TRY(for_each_chunk(who, *rd.src, header_bytes, geo, rd.b[0], rd.b[1], sp, rd.d_state, s, launch,
                         collect));
  const long long file_off = rd.src->tell();

  ReadState fin;
  DCA_CUDA_OK(cudaMemcpyAsync(&fin, rd.d_state, sizeof(fin), cudaMemcpyDeviceToHost, s));
  DCA_CUDA_OK(cudaStreamSynchronize(s));
  int reason = fin.err == ~0ull ? R_NONE : (int)(fin.err & 0xff);
  long long where = fin.err == ~0ull ? 0 : (long long)(fin.err >> 8);
  if (!reason && fin.any_dot && fin.max_val > (1ull << 53)) reason = R_BIG_DOT;
  if (!reason && rows == 0) { set_error("%s: unsupported file: no data lines", who); return DCA_ERR_UNSUPPORTED; }
  if (!reason && fill && rows != rows_expect) { reason = R_ROWS; where = file_off; }
  if (reason) {
    set_error("%s: unsupported file: %s (byte %lld)%s", who, reason_text(reason), where, gz ? " of the inflated stream" : "");
    return DCA_ERR_UNSUPPORTED;
  }
  if (fill) label_offsets[rows] = labels;
  info[0] = rows;
  info[1] = cols;
  info[2] = labels;
  // device bytes of the two chunk buffers (with the transpose stage of the second call)
  info[3] = 2 * (padded + 2ll * tiles_cap * 4 + 3ll * max_lines * 4 + (transpose ? (long long)max_lines * cols * 4 : 0)) +
            (gz ? gzip_source_device_bytes() : 0);
  return DCA_OK;
}
}  // namespace

extern "C" int dca_read_text_counts(const char* path, int32_t sep, int32_t transpose, int64_t chunk_bytes, int32_t device,
                                    void* stream, float* out, int64_t out_elems, int64_t* label_offsets, char* label_bytes,
                                    int64_t label_cap, int64_t* info) {
  return read_text_counts("dca_read_text_counts", false, path, sep, transpose, chunk_bytes, device, stream, out, out_elems,
                          label_offsets, label_bytes, label_cap, info);
}

extern "C" int dca_read_text_counts_gz(const char* path, int32_t sep, int32_t transpose, int64_t chunk_bytes,
                                       int32_t device, void* stream, float* out, int64_t out_elems,
                                       int64_t* label_offsets, char* label_bytes, int64_t label_cap, int64_t* info) {
  return read_text_counts("dca_read_text_counts_gz", true, path, sep, transpose, chunk_bytes, device, stream, out,
                          out_elems, label_offsets, label_bytes, label_cap, info);
}
