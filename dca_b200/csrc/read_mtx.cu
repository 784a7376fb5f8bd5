// GPU reader of Matrix Market coordinate files of counts (dca_read_mtx_counts, include/dca_b200.h): the CSR arrays
// scipy.sparse.csr_matrix(scipy.io.mmread(path).astype(numpy.float32)) has (or its .T.tocsr() with transpose), bit
// for bit, for the files whose entries are already in CSR order of the output; anything else is reported as
// DCA_ERR_UNSUPPORTED and read by scipy.
//
// The header (banner, comments, size line) is read on the host; it gives the shape and the number of entries, so the
// outputs are allocated before any entry is read and entry k of the file goes to slot k.  The entries go through the
// chunked reader of text_chunks.cuh (separator ' ') in one pass; then per chunk, on the caller's stream:
//   parse_entries  one thread per line: "i j v" with single spaces, indices in range, v = [0-9]+ of at most 18 (integer)
//                  or 15 (real) digits -> __ull2float_rn (NumPy's int64 -> float32 cast, and float64 -> float32 of an
//                  exact integer); the column and value go to slot (entry ordinal), the key row * cols + col to a
//                  per-line buffer
//   order_check    the key of every entry must exceed the one before it (across chunks through a carried key, one slot
//                  per chunk parity); an entry whose row differs from the previous entry's writes indptr of the rows
//                  in between, so indptr needs no atomics
// and after the last chunk fill_tail writes indptr of the rows after the last entry.
#include "text_chunks.cuh"

#include <fcntl.h>
#include <unistd.h>

#include <algorithm>
#include <cstring>
#include <string>

namespace dca {
namespace {

using namespace chunked;

constexpr int kMaxIntDigits = 18;     // integer field: < 2^63, exact in int64
constexpr int kMaxRealDigits = 15;    // real field: exact in float64

enum Reason : int { R_ENTRY = 10, R_DIGITS, R_INDEX, R_MORE, R_ORDER, R_FEWER };   // R_QUOTE..R_CR, R_LINES: chunked
const char* reason_text(int r) {
  switch (r) {
    case R_QUOTE: return "a quote character";
    case R_NUL: return "a NUL byte";
    case R_CR: return "a carriage return not followed by a line feed";
    case R_LINES: return "more lines in a chunk than entries allow (blank or short lines)";
    case R_ENTRY: return "an entry line that is not 'i j v' with single spaces and unsigned decimal fields "
                         "(sign, fraction, exponent, tab, extra space, blank or comment line)";
    case R_DIGITS: return "a field with too many digits (indices 18, values 18 for integer and 15 for real)";
    case R_INDEX: return "an index outside 1..M or 1..N";
    case R_MORE: return "more entries than the size line states";
    case R_ORDER: return "an entry not after the one before it in CSR order of the output (unsorted or duplicate)";
    case R_FEWER: return "fewer entries than the size line states";
    default: return "unknown";
  }
}

struct MtxState : ChunkState {
  long long last_key[2];   // key of the last line of the chunk before, by chunk parity (-1: no entry yet, -2: bad line)
};

__global__ void __launch_bounds__(kThreads) parse_entries_kernel(const unsigned char* __restrict__ buf,
                                                                 const int* __restrict__ nl_pos, long long M, long long N,
                                                                 int transpose, int max_digits, long long nnz,
                                                                 long long out_cols, long long* __restrict__ keys,
                                                                 int32_t* __restrict__ indices, float* __restrict__ data,
                                                                 MtxState* st, long long file_off) {
  const int lines = st->chunk_lines;
  const long long base = st->chunk_base;
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < lines; k += gridDim.x * blockDim.x) {
    const int start = k ? nl_pos[k - 1] + 1 : 0;
    int end = nl_pos[k];
    if (end > start && buf[end - 1] == '\r') --end;
    unsigned long long f[3] = {0, 0, 0};
    int p = start, reason = R_NONE, at = start;
    for (int t = 0; t < 3; ++t) {
      const int first = p;
      for (; p < end && p - first <= kMaxIntDigits; ++p) {      // at most 19 digits: no uint64 overflow
        const unsigned c = buf[p];
        if (c < '0' || c > '9') break;
        f[t] = f[t] * 10ull + (c - '0');
      }
      if (p == first) { reason = R_ENTRY; at = p; break; }
      if (p - first > (t == 2 ? max_digits : kMaxIntDigits)) { reason = R_DIGITS; at = first; break; }
      if (t < 2) {
        if (p < end && buf[p] == ' ') ++p;
        else { reason = R_ENTRY; at = p; break; }
      }
    }
    if (!reason && p != end) { reason = R_ENTRY; at = p; }
    if (!reason && (f[0] < 1 || f[0] > (unsigned long long)M || f[1] < 1 || f[1] > (unsigned long long)N)) reason = R_INDEX;
    const long long ord = base + k;
    if (!reason && ord >= nnz) reason = R_MORE;
    if (reason) {
      flag(st, file_off + at, reason);
      keys[k] = -2;
      continue;
    }
    const long long row = (long long)(transpose ? f[1] : f[0]) - 1, col = (long long)(transpose ? f[0] : f[1]) - 1;
    keys[k] = row * out_cols + col;
    indices[ord] = (int32_t)col;
    data[ord] = __ull2float_rn(f[2]);
  }
}

__global__ void __launch_bounds__(kThreads) order_check_kernel(const long long* __restrict__ keys,
                                                               const int* __restrict__ nl_pos, long long out_cols,
                                                               int64_t* __restrict__ indptr, int parity, MtxState* st,
                                                               long long file_off) {
  const int lines = st->chunk_lines;
  const long long base = st->chunk_base;
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < lines; k += gridDim.x * blockDim.x) {
    const long long key = keys[k];
    const long long prev = k ? keys[k - 1] : st->last_key[parity];
    if (k == lines - 1) st->last_key[parity ^ 1] = key;
    if (key < 0 || prev < -1) continue;                  // a bad line, flagged by parse_entries_kernel
    if (key <= prev) { flag(st, file_off + (k ? nl_pos[k - 1] + 1 : 0), R_ORDER); continue; }
    const long long row = key / out_cols, prev_row = prev < 0 ? -1 : prev / out_cols;
    for (long long r = prev_row + 1; r <= row; ++r) indptr[r] = base + k;
  }
}

// indptr of the rows after the last entry (all of them without entries)
__global__ void __launch_bounds__(kThreads) fill_tail_kernel(int64_t* indptr, long long rows, long long nnz,
                                                             long long out_cols, int parity, const MtxState* st) {
  const long long last = st->last_key[parity];
  const long long first = last < 0 ? 0 : last / out_cols + 1;
  for (long long r = first + blockIdx.x * (long long)blockDim.x + threadIdx.x; r <= rows; r += (long long)gridDim.x * blockDim.x)
    indptr[r] = nnz;
}

// ---------------------------------------------------------------------------------------------------------- host
struct Buffers : ChunkBuffers {
  long long* keys = nullptr;             // key of every line of the chunk
  unsigned long long* h_err = nullptr;   // pinned: the error word once the chunk is done
};

struct Reader {
  std::unique_ptr<ByteSource> src;
  int prev_device = -1;                // the caller's current device, restored on return
  MtxState* d_state = nullptr;
  Buffers b[2];
  ~Reader() {
    src.reset();
    for (Buffers& x : b) { x.release(); cudaFree(x.keys); cudaFreeHost(x.h_err); }
    cudaFree(d_state);
    if (prev_device >= 0) cudaSetDevice(prev_device);
  }
};

struct Header {
  long long bytes = 0;                 // banner, comments and size line, with their line ends
  long long m = 0, n = 0, nnz = 0;
  int max_digits = 0;
};

// digits-only decimal of at most 18 digits at h[*p], advancing *p; false when there is none or it is longer
bool header_number(const std::string& h, size_t* p, long long* v) {
  const size_t first = *p;
  long long x = 0;
  while (*p < h.size() && h[*p] >= '0' && h[*p] <= '9' && *p - first < 19) x = x * 10 + (h[(*p)++] - '0');
  *v = x;
  return *p > first && *p - first <= 18;
}

// The banner, the '%' comment lines and the size line "M N NNZ", read on the host.
int read_header(const char* who, ByteSource& src, Header* hd) {
  static const char* kBanner[2] = {"%%MatrixMarket matrix coordinate integer general",
                                   "%%MatrixMarket matrix coordinate real general"};
  std::string h;
  unsigned char tmp[65536];
  bool eof = false;
  int status = DCA_OK;                 // of a failed read
  size_t pos = 0;                      // start of the current line
  // the line starting at pos without its line end; false at the end of the file without one
  auto line = [&](size_t* end, size_t* next) -> int {
    for (;;) {
      const size_t nl = h.find('\n', pos);
      if (nl != std::string::npos) { *next = nl + 1; *end = nl > pos && h[nl - 1] == '\r' ? nl - 1 : nl; return 1; }
      if (eof) { *end = *next = h.size(); return 0; }
      const long long r = src.read(tmp, sizeof(tmp));
      if (r < 0) { status = (int)r; return -1; }
      eof = r < (long long)sizeof(tmp);
      h.append((const char*)tmp, (size_t)r);
    }
  };
  auto unsupported = [who](const char* what) {
    set_error("%s: unsupported file: %s", who, what);
    return DCA_ERR_UNSUPPORTED;
  };
  size_t end = 0, next = 0;
  int st = line(&end, &next);
  if (st < 0) return status;
  const std::string banner = h.substr(0, end);
  if (banner == kBanner[0]) hd->max_digits = kMaxIntDigits;
  else if (banner == kBanner[1]) hd->max_digits = kMaxRealDigits;
  else return unsupported("the first line is not '%%MatrixMarket matrix coordinate integer|real general'");
  for (;;) {
    if (!st) return unsupported("no size line");
    pos = next;
    st = line(&end, &next);
    if (st < 0) return status;
    if (pos < h.size() && h[pos] == '%') continue;
    break;
  }
  size_t p = pos;
  long long v[3];
  for (int t = 0; t < 3; ++t) {
    if (!header_number(h, &p, &v[t]) || (t < 2 ? (p >= end || h[p++] != ' ') : p != end))
      return unsupported("the size line is not 'M N NNZ' with single spaces and at most 18 digits each");
  }
  if (v[0] < 1 || v[1] < 1 || v[0] > INT32_MAX || v[1] > INT32_MAX)
    return unsupported("a dimension outside 1 .. 2^31 - 1");
  hd->m = v[0]; hd->n = v[1]; hd->nnz = v[2];
  hd->bytes = (long long)next;
  return DCA_OK;
}

}  // namespace
}  // namespace dca

using namespace dca;

namespace {
// both entry points: the file's bytes, or (gz) the inflated bytes of a gzip file
int read_mtx_counts(const char* who, bool gz, const char* path, int32_t transpose, int64_t chunk_bytes, int32_t device,
                    void* stream, int64_t* indptr, int32_t* indices, float* data, int64_t* info) {
  const bool fill = indptr != nullptr;
  if (!path || !info || chunk_bytes < 0 || (fill && info[2] > 0 && (!indices || !data))) {
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
  cudaStream_t s = (cudaStream_t)stream;

  DCA_TRY(gz ? open_gzip_source(who, path, &rd.src) : open_file_source(who, path, &rd.src));
  Header hd;
  DCA_TRY(read_header(who, *rd.src, &hd));
  const long long rows = transpose ? hd.n : hd.m, cols = transpose ? hd.m : hd.n;
  const ChunkGeometry geo = chunk_geometry(chunk_bytes, 3);      // "i j v": 3 fields
  if (geo.cap > (1ll << 30)) { set_error("%s: chunk_bytes above 1 GB", who); return DCA_ERR_BAD_ARG; }
  if (!fill) {
    info[0] = rows;
    info[1] = cols;
    info[2] = hd.nnz;
    // device bytes of the two chunk buffers
    info[3] = 2 * (geo.padded + 2ll * geo.tiles_cap * 4 + 2ll * geo.max_lines * 4 + 8ll * geo.max_lines) +
              (gz ? gzip_source_device_bytes() : 0);
    return DCA_OK;
  }
  if (info[0] != rows || info[1] != cols || info[2] != hd.nnz) {
    set_error("%s: unsupported file: its size line changed since the first call", who);
    return DCA_ERR_UNSUPPORTED;
  }
  DCA_TRY(rd.src->seek(hd.bytes));

  DCA_CUDA_OK(cudaMalloc(&rd.d_state, sizeof(MtxState)));
  for (Buffers& x : rd.b) {
    DCA_TRY(x.alloc(geo));
    DCA_CUDA_OK(cudaMalloc(&x.keys, (size_t)geo.max_lines * sizeof(long long)));
    DCA_CUDA_OK(cudaHostAlloc(&x.h_err, sizeof(unsigned long long), cudaHostAllocDefault));
  }
  {
    MtxState init{};
    init.err = ~0ull;
    init.last_key[0] = init.last_key[1] = -1;
    DCA_CUDA_OK(cudaMemcpyAsync(rd.d_state, &init, sizeof(init), cudaMemcpyHostToDevice, s));
  }
  const int grid = std::max(1, std::min(1024, cdiv(geo.max_lines, kThreads)));
  long long chunks = 0;
  auto launch = [&](ChunkBuffers& cb, long long chunk, long long, long long file_off, int) -> int {
    Buffers& x = static_cast<Buffers&>(cb);
    parse_entries_kernel<<<grid, kThreads, 0, s>>>(x.d_buf, x.nl_pos, hd.m, hd.n, transpose ? 1 : 0, hd.max_digits,
                                                   hd.nnz, cols, x.keys, indices, data, rd.d_state, file_off);
    DCA_LAUNCH_CHECK();
    order_check_kernel<<<grid, kThreads, 0, s>>>(x.keys, x.nl_pos, cols, indptr, (int)(chunk & 1), rd.d_state, file_off);
    DCA_LAUNCH_CHECK();
    DCA_CUDA_OK(cudaMemcpyAsync(x.h_err, &rd.d_state->err, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    chunks = chunk + 1;
    return DCA_OK;
  };
  // a problem ends the read: the first one in file order is in the chunks read so far
  auto collect = [&](ChunkBuffers& cb) -> int { return *static_cast<Buffers&>(cb).h_err != ~0ull ? 1 : DCA_OK; };
  DCA_TRY(for_each_chunk(who, *rd.src, hd.bytes, geo, rd.b[0], rd.b[1], ' ', rd.d_state, s, launch,
                         collect));
  fill_tail_kernel<<<std::max(1, std::min(1024, cdiv(rows + 1, kThreads))), kThreads, 0, s>>>(
      indptr, rows, hd.nnz, cols, (int)(chunks & 1), rd.d_state);
  DCA_LAUNCH_CHECK();
  MtxState fin;
  DCA_CUDA_OK(cudaMemcpyAsync(&fin, rd.d_state, sizeof(fin), cudaMemcpyDeviceToHost, s));
  DCA_CUDA_OK(cudaStreamSynchronize(s));
  int reason = fin.err == ~0ull ? R_NONE : (int)(fin.err & 0xff);
  long long where = fin.err == ~0ull ? 0 : (long long)(fin.err >> 8);
  if (!reason && fin.lines_done != hd.nnz) { reason = R_FEWER; where = rd.src->tell(); }
  if (reason) {
    set_error("%s: unsupported file: %s (byte %lld)%s", who, reason_text(reason), where, gz ? " of the inflated stream" : "");
    return DCA_ERR_UNSUPPORTED;
  }
  return DCA_OK;
}
}  // namespace

extern "C" int dca_read_mtx_counts(const char* path, int32_t transpose, int64_t chunk_bytes, int32_t device, void* stream,
                                   int64_t* indptr, int32_t* indices, float* data, int64_t* info) {
  return read_mtx_counts("dca_read_mtx_counts", false, path, transpose, chunk_bytes, device, stream, indptr, indices, data,
                         info);
}

extern "C" int dca_read_mtx_counts_gz(const char* path, int32_t transpose, int64_t chunk_bytes, int32_t device,
                                      void* stream, int64_t* indptr, int32_t* indices, float* data, int64_t* info) {
  return read_mtx_counts("dca_read_mtx_counts_gz", true, path, transpose, chunk_bytes, device, stream, indptr, indices,
                         data, info);
}
