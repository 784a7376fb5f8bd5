// GPU reader of Matrix Market coordinate files of counts (dca_read_mtx_counts, include/dca_b200.h): the CSR arrays
// scipy.sparse.csr_matrix(scipy.io.mmread(path).astype(numpy.float32)) has (or its .T.tocsr() with transpose), bit
// for bit, for the files whose entries are already in CSR order of the output; anything else is reported as
// DCA_ERR_UNSUPPORTED and read by scipy.  dca_read_mtx_counts_map reads the same files keeping only the features (the
// file's rows: the output's columns with transpose, its rows without) a host map numbers, as those arrays with the
// dropped features' columns (rows) taken out; the map is monotone, so the kept entries stay in CSR order.
//
// The header (banner, comments, size line) is read on the host; it gives the shape and the number of entries, so the
// outputs are allocated before any entry is read (the file's NNZ bounds the kept entries).  The entries go through the
// chunked reader of text_chunks.cuh (separator ' ') in one pass; then per chunk, on the caller's stream, in groups of
// kThreads lines:
//   parse_entries  one thread per line: "i j v" with single spaces, indices in range, v = [0-9]+ of at most 18 (integer)
//                  or 15 (real) digits -> __ull2float_rn (NumPy's int64 -> float32 cast, and float64 -> float32 of an
//                  exact integer); the feature i goes through the map; a kept entry's key row * cols + col and value go
//                  to per-line buffers; per group the kept lines and the key of the last one
//   scan_groups    one CTA: per group the slot of its first kept entry and the key of the kept entry before it, with
//                  the kept entries and the last key carried across chunks
//   scatter_check  kept entry k of the read goes to slot k (a block scan of the group's keep flags, no atomics); its
//                  key must exceed the one of the kept entry before it, and an entry whose row differs from that
//                  entry's writes indptr of the rows in between, so indptr needs no atomics either
// and after the last chunk fill_tail writes indptr of the rows after the last kept entry.
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

__device__ __forceinline__ int cdiv_dev(int a, int b) { return (a + b - 1) / b; }

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
  long long kept_done;     // entries kept by the chunks before the current one, then including it
  long long last_key;      // key of the last entry kept so far (-1: none yet)
};

// Keys of a chunk's lines: row * out_cols + col of a kept entry, or one of these
constexpr long long kDropped = -3;     // a line whose feature the map drops (or no line: past the chunk's last)
constexpr long long kBad = -2;         // a line with a problem, flagged by parse_entries_kernel

// A chunk's lines are taken in groups of kThreads lines, one CTA pass per group.
__global__ void __launch_bounds__(kThreads) parse_entries_kernel(const unsigned char* __restrict__ buf,
                                                                 const int* __restrict__ nl_pos, long long M, long long N,
                                                                 int transpose, int max_digits, long long nnz,
                                                                 long long out_cols, const int32_t* __restrict__ fmap,
                                                                 long long* __restrict__ keys, float* __restrict__ vals,
                                                                 int* __restrict__ group_kept,
                                                                 long long* __restrict__ group_last, MtxState* st,
                                                                 long long file_off) {
  __shared__ int sw[kThreads / 32];
  const int lines = st->chunk_lines;
  const long long base = st->chunk_base;
  for (int g = blockIdx.x; (long long)g * kThreads < lines; g += gridDim.x) {      // uniform over the CTA
    const int k = g * kThreads + threadIdx.x;
    long long key = kDropped;
    if (k < lines) {
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
      if (!reason && base + k >= nnz) reason = R_MORE;
      if (reason) {
        flag(st, file_off + at, reason);
        key = kBad;
      } else {
        const long long feature = fmap ? (long long)fmap[f[0] - 1] : (long long)f[0] - 1;    // -1: dropped
        if (feature >= 0) {
          const long long other = (long long)f[1] - 1;
          key = transpose ? other * out_cols + feature : feature * out_cols + other;
          vals[k] = __ull2float_rn(f[2]);
        }
      }
      keys[k] = key;
    }
    // the group's kept lines and the key of its last one
    int total;
    const int before = block_exclusive_scan(key >= 0, sw, &total);
    if (key >= 0 && before == total - 1) group_last[g] = key;
    if (threadIdx.x == 0) {
      group_kept[g] = total;
      if (!total) group_last[g] = -1;
    }
    __syncthreads();                                   // sw is reused by the next group
  }
}

// One CTA: per group, the output slot of its first kept line (kept entries of the chunks before + of the groups
// before) and the key of the kept entry before it; then the carry to the next chunk.
__global__ void __launch_bounds__(kThreads) scan_groups_kernel(const int* __restrict__ group_kept,
                                                               const long long* __restrict__ group_last,
                                                               long long* __restrict__ group_slot,
                                                               long long* __restrict__ group_prev, MtxState* st) {
  __shared__ long long s_sum[kThreads];
  __shared__ int s_last[kThreads];
  const long long kept_before = st->kept_done, key_before = st->last_key;
  const int groups = cdiv_dev(st->chunk_lines, kThreads);
  const int per = cdiv_dev(groups, kThreads);
  const int g0 = min(groups, threadIdx.x * per), g1 = min(groups, g0 + per);
  long long sum = 0;
  int last = -1;                                       // the last group of this thread's run that keeps an entry
  for (int g = g0; g < g1; ++g) {
    const int c = group_kept[g];
    sum += c;
    if (c) last = g;
  }
  s_sum[threadIdx.x] = sum;
  s_last[threadIdx.x] = last;
  __syncthreads();
  for (int o = 1; o < kThreads; o <<= 1) {             // Hillis-Steele inclusive scans: + and max
    const long long x = threadIdx.x >= o ? s_sum[threadIdx.x - o] : 0;
    const int y = threadIdx.x >= o ? s_last[threadIdx.x - o] : -1;
    __syncthreads();
    s_sum[threadIdx.x] += x;
    s_last[threadIdx.x] = max(s_last[threadIdx.x], y);
    __syncthreads();
  }
  long long slot = kept_before + s_sum[threadIdx.x] - sum;
  const int lg = threadIdx.x ? s_last[threadIdx.x - 1] : -1;
  long long prev = lg >= 0 ? group_last[lg] : key_before;
  for (int g = g0; g < g1; ++g) {
    group_slot[g] = slot;
    group_prev[g] = prev;
    const int c = group_kept[g];
    slot += c;
    if (c) prev = group_last[g];
  }
  __syncthreads();                                     // every thread has read the carry
  if (threadIdx.x == kThreads - 1) {
    st->kept_done = slot;
    st->last_key = prev;
  }
}

// Kept entry k of the whole read goes to slot k.  The key of every kept entry must exceed the one of the kept entry
// before it; an entry whose row differs from that entry's writes indptr of the rows in between, so indptr needs no
// atomics.
__global__ void __launch_bounds__(kThreads) scatter_check_kernel(const long long* __restrict__ keys,
                                                                 const float* __restrict__ vals,
                                                                 const int* __restrict__ nl_pos,
                                                                 const long long* __restrict__ group_slot,
                                                                 const long long* __restrict__ group_prev,
                                                                 long long out_cols, int64_t* __restrict__ indptr,
                                                                 int32_t* __restrict__ indices, float* __restrict__ data,
                                                                 MtxState* st, long long file_off) {
  __shared__ int sw[kThreads / 32];
  __shared__ long long s_key[kThreads];
  const int lines = st->chunk_lines;
  for (int g = blockIdx.x; (long long)g * kThreads < lines; g += gridDim.x) {
    const int k = g * kThreads + threadIdx.x;
    const long long key = k < lines ? keys[k] : kDropped;
    int total;
    const int pos = block_exclusive_scan(key >= 0, sw, &total);
    if (key >= 0) s_key[pos] = key;
    __syncthreads();
    if (key >= 0) {
      const long long prev = pos ? s_key[pos - 1] : group_prev[g];
      const long long slot = group_slot[g] + pos;
      const long long row = key / out_cols;
      if (key <= prev) {
        flag(st, file_off + (k ? nl_pos[k - 1] + 1 : 0), R_ORDER);
      } else {
        for (long long r = (prev < 0 ? -1 : prev / out_cols) + 1; r <= row; ++r) indptr[r] = slot;
      }
      indices[slot] = (int32_t)(key - row * out_cols);
      data[slot] = vals[k];
    }
    __syncthreads();                                   // sw and s_key are reused by the next group
  }
}

// indptr of the rows after the last kept entry (all of them without entries)
__global__ void __launch_bounds__(kThreads) fill_tail_kernel(int64_t* indptr, long long rows, long long out_cols,
                                                             const MtxState* st) {
  const long long last = st->last_key, kept = st->kept_done;
  const long long first = last < 0 ? 0 : last / out_cols + 1;
  for (long long r = first + blockIdx.x * (long long)blockDim.x + threadIdx.x; r <= rows; r += (long long)gridDim.x * blockDim.x)
    indptr[r] = kept;
}

// ---------------------------------------------------------------------------------------------------------- host
struct Buffers : ChunkBuffers {
  long long* keys = nullptr;             // key of every line of the chunk
  float* vals = nullptr;                 // value of every kept line of the chunk
  int* group_kept = nullptr;             // per group of kThreads lines: kept lines,
  long long *group_last = nullptr, *group_slot = nullptr, *group_prev = nullptr;   // last key, first slot, key before
  unsigned long long* h_err = nullptr;   // pinned: the error word once the chunk is done
  int alloc_lines(const ChunkGeometry& g) {
    const size_t lines = (size_t)g.max_lines, groups = (size_t)cdiv(g.max_lines, kThreads);
    DCA_CUDA_OK(cudaMalloc(&keys, lines * sizeof(long long)));
    DCA_CUDA_OK(cudaMalloc(&vals, lines * sizeof(float)));
    DCA_CUDA_OK(cudaMalloc(&group_kept, groups * sizeof(int)));
    DCA_CUDA_OK(cudaMalloc(&group_last, groups * sizeof(long long)));
    DCA_CUDA_OK(cudaMalloc(&group_slot, groups * sizeof(long long)));
    DCA_CUDA_OK(cudaMalloc(&group_prev, groups * sizeof(long long)));
    DCA_CUDA_OK(cudaHostAlloc(&h_err, sizeof(unsigned long long), cudaHostAllocDefault));
    return DCA_OK;
  }
  void release_lines() {
    cudaFree(keys); cudaFree(vals); cudaFree(group_kept); cudaFree(group_last); cudaFree(group_slot);
    cudaFree(group_prev); cudaFreeHost(h_err);
  }
};

// device bytes of alloc_lines
long long line_bytes(const ChunkGeometry& g) {
  return 12ll * g.max_lines + 28ll * cdiv(g.max_lines, kThreads);
}

struct Reader {
  std::unique_ptr<ByteSource> src;
  int prev_device = -1;                // the caller's current device, restored on return
  MtxState* d_state = nullptr;
  int32_t* d_map = nullptr;
  Buffers b[2];
  ~Reader() {
    src.reset();
    for (Buffers& x : b) { x.release(); x.release_lines(); }
    cudaFree(d_state);
    cudaFree(d_map);
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
// every entry point: the file's bytes, or (gz) the inflated bytes of a gzip file; fmap NULL keeps every feature
int read_mtx_counts(const char* who, bool gz, const char* path, int32_t transpose, int64_t chunk_bytes, int32_t device,
                    void* stream, int64_t* indptr, int32_t* indices, float* data, int64_t* info, const int32_t* fmap,
                    int64_t map_len) {
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
  // the kept features (the file's rows), numbered 0, 1, ... in file order
  long long features = hd.m;
  if (fmap) {
    if (map_len != hd.m) {
      set_error("%s: feature_map has %lld entries for the file's %lld rows", who, (long long)map_len, hd.m);
      return DCA_ERR_BAD_ARG;
    }
    features = 0;
    for (long long r = 0; r < map_len; ++r) {
      if (fmap[r] < -1 || (fmap[r] >= 0 && fmap[r] != features)) {
        set_error("%s: feature_map[%lld] is %d: it must be -1 or the number of features kept before it (%lld)", who, r,
                  (int)fmap[r], features);
        return DCA_ERR_BAD_ARG;
      }
      features += fmap[r] >= 0;
    }
  }
  const long long rows = transpose ? hd.n : features, cols = transpose ? features : hd.n;
  const ChunkGeometry geo = chunk_geometry(chunk_bytes, 3);      // "i j v": 3 fields
  if (geo.cap > (1ll << 30)) { set_error("%s: chunk_bytes above 1 GB", who); return DCA_ERR_BAD_ARG; }
  if (!fill) {
    info[0] = rows;
    info[1] = cols;
    info[2] = hd.nnz;
    // device bytes of the two chunk buffers
    info[3] = 2 * (geo.padded + 2ll * geo.tiles_cap * 4 + 2ll * geo.max_lines * 4 + line_bytes(geo)) +
              (gz ? gzip_source_device_bytes() : 0) + (fmap ? 4 * map_len : 0);
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
    DCA_TRY(x.alloc_lines(geo));
  }
  if (fmap) {
    DCA_CUDA_OK(cudaMalloc(&rd.d_map, (size_t)map_len * sizeof(int32_t)));
    DCA_CUDA_OK(cudaMemcpyAsync(rd.d_map, fmap, (size_t)map_len * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  }
  {
    MtxState init{};
    init.err = ~0ull;
    init.last_key = -1;
    DCA_CUDA_OK(cudaMemcpyAsync(rd.d_state, &init, sizeof(init), cudaMemcpyHostToDevice, s));
  }
  const int grid = std::max(1, std::min(1024, cdiv(geo.max_lines, kThreads)));
  auto launch = [&](ChunkBuffers& cb, long long, long long, long long file_off, int) -> int {
    Buffers& x = static_cast<Buffers&>(cb);
    parse_entries_kernel<<<grid, kThreads, 0, s>>>(x.d_buf, x.nl_pos, hd.m, hd.n, transpose ? 1 : 0, hd.max_digits,
                                                   hd.nnz, cols, rd.d_map, x.keys, x.vals, x.group_kept, x.group_last,
                                                   rd.d_state, file_off);
    DCA_LAUNCH_CHECK();
    scan_groups_kernel<<<1, kThreads, 0, s>>>(x.group_kept, x.group_last, x.group_slot, x.group_prev, rd.d_state);
    DCA_LAUNCH_CHECK();
    scatter_check_kernel<<<grid, kThreads, 0, s>>>(x.keys, x.vals, x.nl_pos, x.group_slot, x.group_prev, cols, indptr,
                                                   indices, data, rd.d_state, file_off);
    DCA_LAUNCH_CHECK();
    DCA_CUDA_OK(cudaMemcpyAsync(x.h_err, &rd.d_state->err, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    return DCA_OK;
  };
  // a problem ends the read: the first one in file order is in the chunks read so far
  auto collect = [&](ChunkBuffers& cb) -> int { return *static_cast<Buffers&>(cb).h_err != ~0ull ? 1 : DCA_OK; };
  DCA_TRY(for_each_chunk(who, *rd.src, hd.bytes, geo, rd.b[0], rd.b[1], ' ', rd.d_state, s, launch,
                         collect));
  fill_tail_kernel<<<std::max(1, std::min(1024, cdiv(rows + 1, kThreads))), kThreads, 0, s>>>(
      indptr, rows, cols, rd.d_state);
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
  info[2] = fin.kept_done;
  return DCA_OK;
}
}  // namespace

extern "C" int dca_read_mtx_counts(const char* path, int32_t transpose, int64_t chunk_bytes, int32_t device, void* stream,
                                   int64_t* indptr, int32_t* indices, float* data, int64_t* info) {
  return read_mtx_counts("dca_read_mtx_counts", false, path, transpose, chunk_bytes, device, stream, indptr, indices, data,
                         info, nullptr, 0);
}

extern "C" int dca_read_mtx_counts_gz(const char* path, int32_t transpose, int64_t chunk_bytes, int32_t device,
                                      void* stream, int64_t* indptr, int32_t* indices, float* data, int64_t* info) {
  return read_mtx_counts("dca_read_mtx_counts_gz", true, path, transpose, chunk_bytes, device, stream, indptr, indices,
                         data, info, nullptr, 0);
}

extern "C" int dca_read_mtx_counts_map(const char* path, int32_t transpose, int64_t chunk_bytes, int32_t device,
                                       void* stream, int64_t* indptr, int32_t* indices, float* data, int64_t* info,
                                       const int32_t* feature_map, int64_t map_len) {
  return read_mtx_counts("dca_read_mtx_counts_map", false, path, transpose, chunk_bytes, device, stream, indptr, indices,
                         data, info, feature_map, map_len);
}

extern "C" int dca_read_mtx_counts_gz_map(const char* path, int32_t transpose, int64_t chunk_bytes, int32_t device,
                                          void* stream, int64_t* indptr, int32_t* indices, float* data, int64_t* info,
                                          const int32_t* feature_map, int64_t map_len) {
  return read_mtx_counts("dca_read_mtx_counts_gz_map", true, path, transpose, chunk_bytes, device, stream, indptr,
                         indices, data, info, feature_map, map_len);
}
