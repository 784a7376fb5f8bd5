// GPU inflate of gzip files (dca_gunzip, dca_read_*_counts_gz; include/dca_b200.h): speculative, span-parallel
// decoding of DEFLATE (the decoder itself is inflate.cuh, shared with the host mirrors at the end of this file).
//
// The compressed file is read in segments of kSegBytes from the verified position (a block boundary), and each
// segment is cut into regions of kSpanBytes.  Per segment, on the caller's stream:
//   find_starts   one CTA per region: every bit offset of the region is tested in parallel for a plausible block start
//                 (inflate.cuh block_start); the region's candidate is the first one (region 0: the verified position)
//   decode_spans  one warp per span (candidate to next candidate): pass 1 counts the output up to the first block
//                 boundary at or beyond the next candidate (no window needed for that); pass 2 writes 16-bit symbols
//                 to the span's offset, back-references before the span's start as markers
//   resolve_tails one CTA: the last 32 KB of each span in span order, markers replaced by the bytes they refer to
//   resolve_spans one CTA per span: the rest of each span, in parallel
//   member_crc    one thread per 16 KB of output: the linear CRC of its piece of each member, moved to the end of the
//                 member's part in this round (x^(8 n) mod P) and XOR-ed into the part's slot
// Between pass 1 and pass 2 the host chains the spans: a span counts only if it starts where the span before it
// stopped; one that does not is decoded again from there in another round (kMaxRounds per segment, then the file is
// declined).  The host checks the CRC-32 and ISIZE of each member from the part CRCs.
#include "inflate.cuh"
#include "text_chunks.cuh"

#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cstring>
#include <memory>
#include <vector>

namespace dca {
namespace inflate {
namespace {

constexpr long long kSpanBytes = 32ll << 10;       // compressed bytes per region
constexpr long long kSegBytes = 64ll << 20;        // compressed bytes per segment
constexpr long long kLookahead = 1ll << 20;        // bytes past the last region a span may read to reach a boundary
constexpr long long kRoundOut = 256ll << 20;       // output bytes of one segment at most (spans beyond go to the next)
constexpr long long kSpanOutStop = kRoundOut / 2;  // a span stops at the first block boundary past this output
constexpr int kMaxRounds = 16;
constexpr long long kWindow = 32768;
constexpr int kMaxSpans = (int)(kSegBytes / kSpanBytes) + 1;
constexpr int kSearchThreads = 128;
constexpr int kCrcPiece = 16384;
constexpr long long kNone = 1ll << 62;
constexpr long long kMaxMembers = kSegBytes / 20;     // a member takes at least 20 bytes (header, empty block, trailer)

__global__ void __launch_bounds__(kSearchThreads) find_starts_kernel(const uint8_t* __restrict__ in, long long n,
                                                                     long long p0, long long limit, long long* cand) {
  __shared__ long long found;
  const long long r0 = p0 + (long long)blockIdx.x * kSpanBytes * 8, r1 = min(r0 + kSpanBytes * 8, limit);
  if (blockIdx.x == 0) { if (threadIdx.x == 0) cand[0] = p0; return; }
  if (threadIdx.x == 0) found = kNone;
  __syncthreads();
  Tables t;
  for (long long base = r0; base < r1; base += kSearchThreads) {
    const long long bit = base + threadIdx.x;
    if (bit < r1 && block_start(in, n, bit, t)) atomicMin((unsigned long long*)&found, (unsigned long long)bit);
    if (__syncthreads_or(found != kNone)) break;
  }
  if (threadIdx.x == 0) cand[blockIdx.x] = found;
}

struct Job {
  long long start, stop, out_off;
  int mem_off, run;
};

// One span per CTA of one warp, decoded by lane 0: spans take different paths through the decoder on every symbol, so
// two spans in one warp would run one after the other.  write == 0: pass 1 of the spans with run != 0; write != 0:
// pass 2 of every span, into stage / mem at its offsets, checked against its pass-1 result.
__global__ void __launch_bounds__(32) decode_spans_kernel(const uint8_t* __restrict__ in, long long n, int eof,
                                                          const Job* __restrict__ jobs, int spans, SpanResult* res,
                                                          int write, uint16_t* stage, long long stage_cap,
                                                          MemberEnd* mem, int mem_cap, int* mismatch) {
  const int k = blockIdx.x;
  if (k >= spans || threadIdx.x) return;
  const Job j = jobs[k];
  Tables t;
  if (!write) {
    if (j.run) res[k] = decode_span(in, n, eof != 0, j.start, j.stop, kSpanOutStop, nullptr, 0, nullptr, 0, t);
    return;
  }
  const SpanResult p1 = res[k];
  const long long cap = min(p1.out_len, stage_cap - j.out_off);
  const int mcap = min(p1.members, mem_cap - j.mem_off);
  const SpanResult p2 = decode_span(in, n, eof != 0, j.start, j.stop, kSpanOutStop, stage + j.out_off, cap,
                                    mem + j.mem_off, mcap, t);
  if (p2.status != p1.status || p2.end_bit != p1.end_bit || p2.out_len != p1.out_len || p2.members != p1.members)
    atomicExch(mismatch, 1);
}

__device__ __forceinline__ uint8_t resolved(const uint16_t v, const uint8_t* dst, long long off) {
  return v & kMarker ? dst[off - (long long)(v & 0x7fff) - 1] : (uint8_t)v;
}

__global__ void __launch_bounds__(1024) resolve_tails_kernel(const uint16_t* __restrict__ stage, uint8_t* dst,
                                                             const Job* __restrict__ jobs, const SpanResult* res, int spans) {
  for (int k = 0; k < spans; ++k) {
    const long long off = jobs[k].out_off, len = res[k].out_len;
    for (long long p = max(0ll, len - kWindow) + threadIdx.x; p < len; p += blockDim.x)
      dst[off + p] = resolved(stage[off + p], dst, off);
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256) resolve_spans_kernel(const uint16_t* __restrict__ stage, uint8_t* dst,
                                                            const Job* __restrict__ jobs, const SpanResult* res) {
  const long long off = jobs[blockIdx.x].out_off, len = res[blockIdx.x].out_len;
  for (long long p = threadIdx.x; p < len - kWindow; p += blockDim.x) dst[off + p] = resolved(stage[off + p], dst, off);
}

// bounds[0, parts]: output positions of the round's member parts (part j = [bounds[j], bounds[j + 1]))
__global__ void __launch_bounds__(256) member_crc_kernel(const uint8_t* __restrict__ dst, long long total,
                                                         const long long* __restrict__ bounds, int parts, uint32_t* part_crc) {
  __shared__ uint32_t table[256];
  {
    uint32_t c = threadIdx.x;
    for (int k = 0; k < 8; ++k) c = c & 1 ? (c >> 1) ^ kCrcPoly : c >> 1;
    table[threadIdx.x] = c;
  }
  __syncthreads();
  const long long c0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * kCrcPiece;
  if (c0 >= total) return;
  const long long c1 = min(total, c0 + kCrcPiece);
  int lo = 0, hi = parts - 1;                            // first part ending after c0
  while (lo < hi) { const int m = (lo + hi) / 2; if (bounds[m + 1] > c0) hi = m; else lo = m + 1; }
  for (int j = lo; j < parts; ++j) {
    const long long a = max(c0, bounds[j]), b = min(c1, bounds[j + 1]);
    if (a < b) {
      uint32_t c = 0;
      for (long long p = a; p < b; ++p) c = table[(c ^ dst[p]) & 0xff] ^ (c >> 8);
      atomicXor(&part_crc[j], crc_mul(crc_x8n((unsigned long long)(bounds[j + 1] - b)), c));
    }
    if (bounds[j + 1] >= c1) break;
  }
}

template <class T>
int grow(T** p, long long* cap, long long want) {
  if (*cap >= want) return DCA_OK;
  cudaFree(*p);
  *p = nullptr;
  *cap = 0;
  DCA_CUDA_OK(cudaMalloc(p, (size_t)want * sizeof(T)));
  *cap = want;
  return DCA_OK;
}

// win = [32 KB before the output][kRoundOut of output][32 KB scratch]: after `have` bytes of output, the 32 KB before
// the next output are the last 32 KB of the first two parts
int shift_history(uint8_t* win, long long have, cudaStream_t s) {
  uint8_t* tmp = win + kWindow + kRoundOut;
  DCA_CUDA_OK(cudaMemcpyAsync(tmp, win + have, (size_t)kWindow, cudaMemcpyDeviceToDevice, s));
  DCA_CUDA_OK(cudaMemcpyAsync(win, tmp, (size_t)kWindow, cudaMemcpyDeviceToDevice, s));
  return DCA_OK;
}

}  // namespace

// One gzip file inflated in segments.  next() writes the output of one segment to device memory whose 32 KB before
// it hold the output before (when there is any).
class Inflater {
 public:
  ~Inflater() {
    if (fd_ >= 0) close(fd_);
    cudaFreeHost(h_in_); cudaFreeHost(h_jobs_); cudaFreeHost(h_res_); cudaFreeHost(h_cand_);
    cudaFree(d_in_); cudaFree(d_cand_); cudaFree(d_jobs_); cudaFree(d_res_); cudaFree(stage_); cudaFree(mem_);
    cudaFree(bounds_); cudaFree(parts_); cudaFree(d_mismatch_);
  }
  int open(const char* who, const char* path, cudaStream_t s) {
    who_ = who; s_ = s;
    fd_ = ::open(path, O_RDONLY);
    if (fd_ < 0) { set_error("%s: cannot open %s", who, path); return DCA_ERR_BAD_ARG; }
    struct stat st;
    if (fstat(fd_, &st) != 0) { set_error("%s: cannot stat %s", who, path); return DCA_ERR_BAD_ARG; }
    size_ = st.st_size;
    DCA_CUDA_OK(cudaHostAlloc(&h_in_, (size_t)kSegBytes, cudaHostAllocDefault));
    DCA_CUDA_OK(cudaHostAlloc(&h_jobs_, kMaxSpans * sizeof(Job), cudaHostAllocDefault));
    DCA_CUDA_OK(cudaHostAlloc(&h_res_, kMaxSpans * sizeof(SpanResult), cudaHostAllocDefault));
    DCA_CUDA_OK(cudaHostAlloc(&h_cand_, kMaxSpans * sizeof(long long), cudaHostAllocDefault));
    DCA_CUDA_OK(cudaMalloc(&d_in_, (size_t)kSegBytes + 16));
    DCA_CUDA_OK(cudaMalloc(&d_cand_, kMaxSpans * sizeof(long long)));
    DCA_CUDA_OK(cudaMalloc(&d_jobs_, kMaxSpans * sizeof(Job)));
    DCA_CUDA_OK(cudaMalloc(&d_res_, kMaxSpans * sizeof(SpanResult)));
    DCA_CUDA_OK(cudaMalloc(&d_mismatch_, sizeof(int)));
    // the first member's header
    long long n = 0;
    DCA_TRY(load(0, &n));
    long long hlen = 0;
    if (n == 0 || parse_header(h_in_, n, 0, n == size_, &hlen) != H_OK) return decline("not a gzip member header");
    pos_ = hlen * 8;
    return DCA_OK;
  }
  bool done() const { return done_; }
  long long produced() const { return produced_; }
  int rounds() const { return max_rounds_; }
  long long members() const { return members_; }
  long long device_bytes() const {
    return kSegBytes + 16 + kMaxSpans * (long long)(sizeof(long long) + sizeof(Job) + sizeof(SpanResult)) + sizeof(int) +
           stage_cap_ * 2 + mem_cap_ * (long long)sizeof(MemberEnd) + bounds_cap_ * 8 + parts_cap_ * 4;
  }
  // the most device_bytes() can reach: a window of 16-bit symbols, and member arrays for a segment of tiny members
  static long long max_device_bytes() {
    return kSegBytes + 16 + kMaxSpans * (long long)(sizeof(long long) + sizeof(Job) + sizeof(SpanResult)) + sizeof(int) +
           kRoundOut * 2 + (kMaxMembers + 2) * (long long)(sizeof(MemberEnd) + 8 + 4);
  }

  // The next verified spans' output to dst[0, *len), *len <= cap (cap >= kRoundOut unless the output ends before).
  // A segment's verified spans are kept until their output has been written, window by window, so no span is decoded
  // again because the output of its segment was longer than one window.
  int next(uint8_t* dst, long long cap, long long* len) {
    *len = 0;
    if (done_) return DCA_OK;
    if (next_span_ == verified_) DCA_TRY(segment());
    const int b0 = next_span_;
    int b1 = b0;
    long long total = 0;
    const long long room = std::min(cap, kRoundOut);
    while (b1 < verified_ && total + h_res_[b1].out_len <= room) total += h_res_[b1++].out_len;
    if (b1 == b0) return decline("a span's output is longer than the output window");
    const int spans = b1 - b0;

    // pass 2, resolve, member CRCs of spans [b0, b1)
    int members = 0;
    for (int k = b0; k < b1; ++k) {
      h_jobs_[k].out_off = span_out_[k] - span_out_[b0];
      h_jobs_[k].mem_off = members;
      members += h_res_[k].members;
    }
    DCA_TRY(grow(&stage_, &stage_cap_, std::max(total, 1ll)));
    DCA_TRY(grow(&mem_, &mem_cap_, std::max(members, 1)));
    DCA_TRY(grow(&bounds_, &bounds_cap_, members + 2ll));
    DCA_TRY(grow(&parts_, &parts_cap_, members + 1ll));
    Job* jobs = d_jobs_ + b0;
    SpanResult* res = d_res_ + b0;
    DCA_CUDA_OK(cudaMemcpyAsync(jobs, h_jobs_ + b0, spans * sizeof(Job), cudaMemcpyHostToDevice, s_));
    DCA_CUDA_OK(cudaMemcpyAsync(res, h_res_ + b0, spans * sizeof(SpanResult), cudaMemcpyHostToDevice, s_));
    DCA_CUDA_OK(cudaMemsetAsync(d_mismatch_, 0, sizeof(int), s_));
    decode_spans_kernel<<<spans, 32, 0, s_>>>(d_in_, seg_n_, seg_eof_, jobs, spans, res, 1, stage_, stage_cap_, mem_,
                                              (int)mem_cap_, d_mismatch_);
    DCA_LAUNCH_CHECK();
    resolve_tails_kernel<<<1, 1024, 0, s_>>>(stage_, dst, jobs, res, spans);
    DCA_LAUNCH_CHECK();
    resolve_spans_kernel<<<spans, 256, 0, s_>>>(stage_, dst, jobs, res);
    DCA_LAUNCH_CHECK();
    std::vector<MemberEnd> me(members);
    int mismatch = 0;
    if (members) DCA_CUDA_OK(cudaMemcpyAsync(me.data(), mem_, members * sizeof(MemberEnd), cudaMemcpyDeviceToHost, s_));
    DCA_CUDA_OK(cudaMemcpyAsync(&mismatch, d_mismatch_, sizeof(int), cudaMemcpyDeviceToHost, s_));
    DCA_CUDA_OK(cudaStreamSynchronize(s_));
    if (mismatch) { set_error("%s: internal error: the two passes of a span differ", who_); return DCA_ERR_CUDA; }
    std::vector<long long> bounds(members + 2);
    bounds[0] = 0;
    for (int k = b0, m = 0; k < b1; ++k)
      for (int i = 0; i < h_res_[k].members; ++i, ++m) bounds[m + 1] = h_jobs_[k].out_off + me[m].end;
    bounds[members + 1] = total;
    const int parts = members + 1;
    std::vector<uint32_t> part_crc(parts);
    DCA_CUDA_OK(cudaMemcpyAsync(bounds_, bounds.data(), (members + 2) * sizeof(long long), cudaMemcpyHostToDevice, s_));
    DCA_CUDA_OK(cudaMemsetAsync(parts_, 0, parts * sizeof(uint32_t), s_));
    if (total) {
      member_crc_kernel<<<cdiv(cdiv(total, kCrcPiece), 256), 256, 0, s_>>>(dst, total, bounds_, parts, parts_);
      DCA_LAUNCH_CHECK();
    }
    DCA_CUDA_OK(cudaMemcpyAsync(part_crc.data(), parts_, parts * sizeof(uint32_t), cudaMemcpyDeviceToHost, s_));
    DCA_CUDA_OK(cudaStreamSynchronize(s_));
    for (int j = 0; j < parts; ++j) {
      const unsigned long long l = (unsigned long long)(bounds[j + 1] - bounds[j]);
      crc_ = crc_concat(crc_, part_crc[j], l);
      member_len_ += l;
      if (j == members) break;
      if (crc_finish(crc_, member_len_) != me[j].crc || (uint32_t)member_len_ != me[j].isize)
        return decline("a member's CRC-32 or ISIZE does not match its data");
      crc_ = 0; member_len_ = 0;
      ++members_;
    }
    floor_ = span_floor_[b1 - 1];
    produced_ += total;
    pos_ = seg_base_ * 8 + h_res_[b1 - 1].end_bit;
    next_span_ = b1;
    done_ = b1 == verified_ && seg_end_;
    *len = total;
    return DCA_OK;
  }

 private:
  // Loads the segment at the verified position, finds the candidates, and decodes and chains the spans in rounds
  // until a prefix of them is verified: verified_ spans, with their output positions and member floors.
  int segment() {
    const long long base = pos_ >> 3;
    long long n = 0;
    DCA_TRY(load(base, &n));
    const bool eof = base + n == size_;
    seg_base_ = base; seg_n_ = n; seg_eof_ = eof;
    DCA_CUDA_OK(cudaMemcpyAsync(d_in_, h_in_, (size_t)n, cudaMemcpyHostToDevice, s_));
    const long long p0 = pos_ - base * 8;
    const long long limit = eof ? n * 8 : n * 8 - kLookahead * 8;
    if (limit <= p0) return decline("truncated");
    const int regions = cdiv(limit - p0, kSpanBytes * 8);
    find_starts_kernel<<<regions, kSearchThreads, 0, s_>>>(d_in_, n, p0, limit, d_cand_);
    DCA_LAUNCH_CHECK();
    DCA_CUDA_OK(cudaMemcpyAsync(h_cand_, d_cand_, regions * sizeof(long long), cudaMemcpyDeviceToHost, s_));
    DCA_CUDA_OK(cudaStreamSynchronize(s_));
    int spans = 0;
    for (int i = 0; i < regions; ++i)
      if (h_cand_[i] != kNone) h_jobs_[spans++] = Job{h_cand_[i], 0, 0, 0, 1};
    for (int k = 0; k < spans; ++k) h_jobs_[k].stop = k + 1 < spans ? h_jobs_[k + 1].start : eof ? kNone : limit;
    span_out_.assign(spans, 0);
    span_floor_.assign(spans, 0);

    // Span k restarted at bit e: when e is at or past its stop the decoder would stop at once with no output, so
    // that result is set here and the chain goes on in the same round.
    auto restart = [&](int k, long long e) {
      h_jobs_[k].start = e;
      if (e >= h_jobs_[k].stop) { h_res_[k] = SpanResult{e, 0, 0, -1, ST_STOP, 0}; return false; }
      h_jobs_[k].run = 1;
      return true;
    };
    int accepted = 0, rounds = 0;
    bool end = false;
    for (;;) {
      if (++rounds > kMaxRounds) return decline("more than 16 rounds of span decoding in one segment");
      DCA_CUDA_OK(cudaMemcpyAsync(d_jobs_, h_jobs_, spans * sizeof(Job), cudaMemcpyHostToDevice, s_));
      decode_spans_kernel<<<spans, 32, 0, s_>>>(d_in_, n, eof, d_jobs_, spans, d_res_, 0, nullptr, 0, nullptr, 0,
                                                nullptr);
      DCA_LAUNCH_CHECK();
      // only the spans that ran have new results; the others keep theirs (or the one set by restart)
      for (int k = 0; k < spans;) {
        int e = k;
        while (e < spans && h_jobs_[e].run) ++e;
        if (e > k) DCA_CUDA_OK(cudaMemcpyAsync(h_res_ + k, d_res_ + k, (e - k) * sizeof(SpanResult),
                                               cudaMemcpyDeviceToHost, s_));
        k = e + 1;
      }
      DCA_CUDA_OK(cudaStreamSynchronize(s_));
      for (int k = 0; k < spans; ++k) h_jobs_[k].run = 0;
      accepted = 0; end = false;
      long long total = 0, floor = floor_, expected = p0;
      bool verified = true, redo = false;
      for (int k = 0; k < spans; ++k) {
        if (!verified) {                                 // tentatively: the span before is right
          const SpanResult& q = h_res_[k - 1];
          if (h_jobs_[k - 1].run || q.status != ST_STOP) continue;
          if (h_jobs_[k].start != q.end_bit) redo |= restart(k, q.end_bit);
          continue;
        }
        if (h_jobs_[k].start != expected && restart(k, expected)) {
          redo = true; verified = false;
          continue;
        }
        const SpanResult& r = h_res_[k];
        if (r.status == ST_BAD) return decline("invalid deflate data, a bad header or trailing bytes");
        if (r.status == ST_NEED) break;
        if (r.min_ref < 0 && produced_ + total + r.min_ref < floor) return decline("a distance before the member's start");
        if (r.member_start >= 0) floor = produced_ + total + r.member_start;
        span_out_[k] = total;
        span_floor_[k] = floor;
        total += r.out_len;
        expected = r.end_bit;
        ++accepted;
        if (r.status == ST_END) { end = true; break; }
        if (r.status == ST_FULL) break;
      }
      if (verified || !redo) break;
    }
    if (accepted == 0) return decline(eof ? "truncated" : "a deflate block longer than a segment or its output");
    max_rounds_ = std::max(max_rounds_, rounds);
    verified_ = accepted;
    next_span_ = 0;
    seg_end_ = end;
    return DCA_OK;
  }

  int decline(const char* why) {
    set_error("%s: unsupported file: %s (compressed byte %lld)", who_, why, pos_ >> 3);
    return DCA_ERR_UNSUPPORTED;
  }
  int load(long long base, long long* n) {
    long long got = 0;
    const long long want = std::min(kSegBytes, size_ - base);
    while (got < want) {
      const ssize_t r = pread(fd_, h_in_ + got, (size_t)(want - got), (off_t)(base + got));
      if (r < 0) { set_error("%s: read failed", who_); return DCA_ERR_BAD_ARG; }
      if (r == 0) break;
      got += r;
    }
    *n = got;
    return DCA_OK;
  }

  const char* who_ = "";
  cudaStream_t s_ = nullptr;
  int fd_ = -1;
  long long size_ = 0;
  long long pos_ = 0;              // verified bit of the file: a block boundary or a member's first block
  long long produced_ = 0;         // output bytes before the next segment
  long long floor_ = 0;            // output position where the current member starts
  uint32_t crc_ = 0;               // linear CRC and length of the current member so far
  unsigned long long member_len_ = 0;
  long long members_ = 0;
  int max_rounds_ = 0;
  bool done_ = false;
  // the current segment: its first byte, bytes, whether it ends the file; its verified spans, the next one to write,
  // whether the last one ends the file; per span its output position and the member floor after it
  long long seg_base_ = 0, seg_n_ = 0;
  bool seg_eof_ = false, seg_end_ = false;
  int verified_ = 0, next_span_ = 0;
  std::vector<long long> span_out_, span_floor_;
  uint8_t* h_in_ = nullptr;
  Job* h_jobs_ = nullptr;
  SpanResult* h_res_ = nullptr;
  long long* h_cand_ = nullptr;
  uint8_t* d_in_ = nullptr;
  long long* d_cand_ = nullptr;
  Job* d_jobs_ = nullptr;
  SpanResult* d_res_ = nullptr;
  int* d_mismatch_ = nullptr;
  uint16_t* stage_ = nullptr;
  long long stage_cap_ = 0;
  MemberEnd* mem_ = nullptr;
  long long mem_cap_ = 0;
  long long* bounds_ = nullptr;
  long long bounds_cap_ = 0;
  uint32_t* parts_ = nullptr;
  long long parts_cap_ = 0;
};

namespace {

// the readers' byte source over the inflated stream: segments go to a device window (shift_history), and read() copies from there into the caller's pinned staging
class GzipSource : public chunked::ByteSource {
 public:
  ~GzipSource() override {
    inf_.reset();
    cudaFree(win_);
    if (s_) cudaStreamDestroy(s_);
  }
  // The inflate runs on a stream of its own, so the parser's kernels on the caller's stream overlap the inflate of the
  // next segment; read() waits for this stream only.
  int open(const char* who, const char* path) {
    who_ = who; path_ = path;
    if (!s_) DCA_CUDA_OK(cudaStreamCreateWithFlags(&s_, cudaStreamNonBlocking));
    inf_.reset(new Inflater);
    DCA_TRY(inf_->open(who, path, s_));
    if (!win_) DCA_CUDA_OK(cudaMalloc(&win_, (size_t)(2 * kWindow + kRoundOut)));
    win_off_ = 0; have_ = 0; rd_ = 0;
    return DCA_OK;
  }
  long long read(unsigned char* dst, long long want) override {
    long long got = 0;
    while (got < want) {
      if (rd_ == have_) {
        if (inf_->done()) break;
        const int st = refill();
        if (st != DCA_OK) return st;
        continue;
      }
      const long long c = std::min(want - got, have_ - rd_);
      if (cudaMemcpyAsync(dst + got, win_ + kWindow + rd_, (size_t)c, cudaMemcpyDeviceToHost, s_) != cudaSuccess ||
          cudaStreamSynchronize(s_) != cudaSuccess) {
        set_error("%s: device copy failed", who_);
        return DCA_ERR_CUDA;
      }
      rd_ += c; got += c;
    }
    return got;
  }
  int seek(long long off) override {
    if (off < win_off_) DCA_TRY(open(who_, path_));
    while (off > win_off_ + have_) {
      if (inf_->done()) { set_error("%s: seek past the end", who_); return DCA_ERR_BAD_ARG; }
      DCA_TRY(refill());
    }
    rd_ = off - win_off_;
    return DCA_OK;
  }
  long long tell() override { return win_off_ + rd_; }

 private:
  // the next segment into the window, after the last 32 KB of the output so far
  int refill() {
    if (have_) DCA_TRY(shift_history(win_, have_, s_));
    win_off_ += have_;
    have_ = 0; rd_ = 0;
    return inf_->next(win_ + kWindow, kRoundOut, &have_);
  }
  const char* who_ = "";
  const char* path_ = "";
  cudaStream_t s_ = nullptr;
  std::unique_ptr<Inflater> inf_;
  uint8_t* win_ = nullptr;
  long long win_off_ = 0, have_ = 0, rd_ = 0;
};

}  // namespace
}  // namespace inflate

namespace chunked {

int open_gzip_source(const char* who, const char* path, std::unique_ptr<ByteSource>* out) {
  std::unique_ptr<inflate::GzipSource> g(new inflate::GzipSource);
  DCA_TRY(g->open(who, path));
  *out = std::move(g);
  return DCA_OK;
}

long long gzip_source_device_bytes() {
  using namespace inflate;
  return 2 * kWindow + kRoundOut + Inflater::max_device_bytes();
}

}  // namespace chunked
}  // namespace dca

using namespace dca;
using namespace dca::inflate;

extern "C" int dca_gunzip(const char* path, int32_t device, void* stream, void* out, int64_t out_bytes, int64_t* info) {
  if (!path || !info || (out && out_bytes < 0)) { set_error("dca_gunzip: bad argument"); return DCA_ERR_BAD_ARG; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    (void)cudaGetLastError();
    set_error("dca_gunzip: no CUDA device available (this library has no CPU fallback)");
    return DCA_ERR_NO_DEVICE;
  }
  if (device < 0 || device >= ndev) { set_error("dca_gunzip: no CUDA device %d", device); return DCA_ERR_BAD_ARG; }
  int prev = -1;
  DCA_CUDA_OK(cudaGetDevice(&prev));
  DCA_CUDA_OK(cudaSetDevice(device));
  struct Restore { int d; ~Restore() { if (d >= 0) cudaSetDevice(d); } } restore{prev};
  cudaStream_t s = (cudaStream_t)stream;
  Inflater inf;
  DCA_TRY(inf.open("dca_gunzip", path, s));
  // without `out` the output goes to a scratch window (with the 32 KB before it) and only its size is kept
  uint8_t* scratch = nullptr;
  struct Free { uint8_t** p; ~Free() { cudaFree(*p); } } free_scratch{&scratch};
  if (!out) DCA_CUDA_OK(cudaMalloc(&scratch, (size_t)(2 * kWindow + kRoundOut)));
  while (!inf.done()) {
    long long len = 0;
    if (out) {
      const long long room = out_bytes - inf.produced();
      if (room < 0) { set_error("dca_gunzip: the output is longer than out_bytes"); return DCA_ERR_BAD_ARG; }
      DCA_TRY(inf.next((uint8_t*)out + inf.produced(), std::max(room, 0ll), &len));
    } else {
      DCA_TRY(inf.next(scratch + kWindow, kRoundOut, &len));
      DCA_TRY(shift_history(scratch, len, s));
    }
  }
  if (out && inf.produced() != out_bytes) { set_error("dca_gunzip: the output is not out_bytes long"); return DCA_ERR_BAD_ARG; }
  info[0] = inf.produced();
  info[1] = inf.device_bytes() + (out ? 0 : 2 * kWindow + kRoundOut);
  info[2] = inf.rounds();
  info[3] = inf.members();
  return DCA_OK;
}

// ------------------------------------------------------------------------------------------------- host mirrors
extern "C" int dca_inflate_span_host(const uint8_t* in, int64_t n, int32_t eof, int64_t start, int64_t stop,
                                     uint16_t* out, int64_t out_cap, int64_t* info) {
  if (!in || n < 0 || !info || start < 0 || (out && out_cap < 0)) {
    set_error("dca_inflate_span_host: bad argument"); return DCA_ERR_BAD_ARG;
  }
  std::unique_ptr<Tables> t(new Tables);
  const SpanResult r = decode_span(in, n, eof != 0, start, stop, kNone, out, out ? out_cap : 0, nullptr, 0, *t);
  info[0] = r.status; info[1] = r.end_bit; info[2] = r.out_len; info[3] = r.min_ref; info[4] = r.member_start;
  info[5] = r.members;
  return DCA_OK;
}

extern "C" int dca_inflate_find_host(const uint8_t* in, int64_t n, int64_t first_bit, int64_t end_bit, int64_t* found) {
  if (!in || n < 0 || !found || first_bit < 0) { set_error("dca_inflate_find_host: bad argument"); return DCA_ERR_BAD_ARG; }
  std::unique_ptr<Tables> t(new Tables);
  *found = -1;
  for (int64_t b = first_bit; b < end_bit; ++b)
    if (block_start(in, n, b, *t)) { *found = b; break; }
  return DCA_OK;
}
