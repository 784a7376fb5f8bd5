// DEFLATE (RFC 1951) and gzip member (RFC 1952) decoding, written once for the host and the device: the span decoder
// and the block-start test of the speculative inflate (inflate.cu), and the gzip header check.  The host build runs
// the same code on the CPU (dca_inflate_span_host, dca_inflate_find_host) so the algorithm is testable without a GPU.
//
// Every read of the compressed bytes goes through Bits, which reads zeros past the end and reports the overrun, and
// every write of output is checked against its capacity: a malformed stream ends in a status, never in an access
// outside a buffer.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define DCA_HD __host__ __device__
#else
#define DCA_HD
#endif

namespace dca {
namespace inflate {

// status of a span decode
enum : int {
  ST_STOP = 0,     // stopped at a block boundary at or beyond the stop bit
  ST_END = 1,      // decoded the last member of the file up to the file's last byte
  ST_NEED = 2,     // ran out of loaded input before a stop (the file goes on)
  ST_BAD = 3,      // not a valid stream from this start (or truncated at the end of the file)
  ST_FULL = 4,     // stopped at a block boundary because the output reached the span's output cap
};

// the 16-bit symbols of the write pass: a byte, or a marker for the byte `k + 1` positions before the span's first
// output byte (k < 32768), which the resolve step replaces once the bytes before the span are known
constexpr uint16_t kMarker = 0x8000;

// LSB-first bit reader over in[0, n) with a 64-bit buffer; bytes at or past n read as zero and pos() > 8 n tells
struct Bits {
  const uint8_t* p;
  long long n, next;
  uint64_t buf;
  int cnt;
  DCA_HD void init(const uint8_t* p_, long long n_, long long bit) {
    p = p_; n = n_; next = bit >> 3; buf = 0; cnt = 0;
    refill();
    buf >>= (bit & 7); cnt -= (int)(bit & 7);
  }
  DCA_HD void refill() {
    while (cnt <= 56) {
      const uint64_t b = next >= 0 && next < n ? p[next] : 0;
      buf |= b << cnt; cnt += 8; ++next;
    }
  }
  DCA_HD long long pos() const { return next * 8 - cnt; }
  DCA_HD bool over() const { return pos() > n * 8; }
  DCA_HD uint32_t bits(int k) {        // k <= 32
    refill();
    const uint32_t v = (uint32_t)(buf & ((1ull << k) - 1));
    buf >>= k; cnt -= k;
    return v;
  }
  DCA_HD void align() { const int r = (int)(pos() & 7); if (r) { buf >>= (8 - r); cnt -= 8 - r; } }
};

// canonical Huffman code: codes per length and symbols in code order
template <int N>
struct Huff {
  int16_t count[16];
  int16_t sym[N];
};

// lengths[0, n) -> h; returns 0 for a complete code (or no code at all), > 0 incomplete, < 0 over-subscribed
template <int N>
DCA_HD int build(Huff<N>& h, const uint8_t* lengths, int n) {
  for (int l = 0; l < 16; ++l) h.count[l] = 0;
  for (int s = 0; s < n; ++s) h.count[lengths[s]]++;
  if (h.count[0] == n) return 0;
  int left = 1;
  for (int l = 1; l < 16; ++l) { left <<= 1; left -= h.count[l]; if (left < 0) return left; }
  int16_t offs[16];
  offs[1] = 0;
  for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + h.count[l];
  for (int s = 0; s < n; ++s) if (lengths[s]) h.sym[offs[lengths[s]]++] = (int16_t)s;
  return left;
}

// one symbol, or -1 for a code the table does not have
template <int N>
DCA_HD int decode(Bits& b, const Huff<N>& h) {
  b.refill();
  uint32_t bits = (uint32_t)b.buf;
  int code = 0, first = 0, index = 0;
  for (int l = 1; l < 16; ++l) {
    code |= bits & 1; bits >>= 1;
    const int c = h.count[l];
    if (code - c < first) { b.buf >>= l; b.cnt -= l; return h.sym[index + (code - first)]; }
    index += c; first += c; first <<= 1; code <<= 1;
  }
  return -1;
}

struct Tables {
  Huff<288> lit;
  Huff<30> dist;
};

// the header of a dynamic block after BTYPE; strict (block-start search): every code complete
DCA_HD inline bool dynamic_tables(Bits& b, Tables& t, bool strict) {
  const int nlen = (int)b.bits(5) + 257, ndist = (int)b.bits(5) + 1, ncode = (int)b.bits(4) + 4;
  if (nlen > 286 || ndist > 30) return false;
  const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  uint8_t lengths[286 + 30];
  for (int i = 0; i < 19; ++i) lengths[order[i]] = i < ncode ? (uint8_t)b.bits(3) : 0;
  Huff<19> lc;
  if (build(lc, lengths, 19) != 0) return false;          // the code-length code must be complete
  int index = 0;
  while (index < nlen + ndist) {
    int sym = decode(b, lc);
    if (sym < 0 || b.over()) return false;
    if (sym < 16) { lengths[index++] = (uint8_t)sym; continue; }
    uint8_t len = 0;
    if (sym == 16) { if (index == 0) return false; len = lengths[index - 1]; sym = 3 + (int)b.bits(2); }
    else if (sym == 17) sym = 3 + (int)b.bits(3);
    else sym = 11 + (int)b.bits(7);
    if (index + sym > nlen + ndist) return false;
    while (sym--) lengths[index++] = len;
  }
  if (lengths[256] == 0) return false;                    // end-of-block needs a code
  const int e1 = build(t.lit, lengths, nlen);
  if (!(e1 == 0 || (!strict && e1 > 0 && t.lit.count[1] == 1 && nlen - t.lit.count[0] == 1))) return false;
  const int e2 = build(t.dist, lengths + nlen, ndist);
  if (!(e2 == 0 || (!strict && e2 > 0 && t.dist.count[1] == 1 && ndist - t.dist.count[0] == 1))) return false;
  return !b.over();
}

DCA_HD inline void fixed_tables(Tables& t) {
  uint8_t l[288];
  for (int s = 0; s < 288; ++s) l[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
  build(t.lit, l, 288);
  for (int s = 0; s < 30; ++s) l[s] = 5;
  build(t.dist, l, 30);
}

// ------------------------------------------------------------------------------------------------- CRC-32 (RFC 1952)
constexpr uint32_t kCrcPoly = 0xedb88320u;     // reflected x^32 + x^26 + ... + 1

DCA_HD inline uint32_t crc32_bytes(uint32_t crc, const uint8_t* p, long long n) {    // bitwise: headers only
  crc = ~crc;
  for (long long i = 0; i < n; ++i) {
    crc ^= p[i];
    for (int k = 0; k < 8; ++k) crc = crc & 1 ? (crc >> 1) ^ kCrcPoly : crc >> 1;
  }
  return ~crc;
}
// a * b modulo the CRC polynomial, both reflected (bit 31 is x^0)
DCA_HD inline uint32_t crc_mul(uint32_t a, uint32_t b) {
  uint32_t p = 0;
  for (uint32_t m = 1u << 31; m; m >>= 1) {
    if (a & m) p ^= b;
    b = b & 1 ? (b >> 1) ^ kCrcPoly : b >> 1;
  }
  return p;
}
// x^(8 n) modulo the polynomial: the factor that appends n zero bytes to a linear CRC
DCA_HD inline uint32_t crc_x8n(unsigned long long n) {
  uint32_t p = 1u << 31, sq = 1u << 23;                    // x^0, x^8
  for (; n; n >>= 1) {
    if (n & 1) p = crc_mul(sq, p);
    sq = crc_mul(sq, sq);
  }
  return p;
}
// linear CRC (initial 0, no final inversion) of data followed by n more bytes whose linear CRC is b
DCA_HD inline uint32_t crc_concat(uint32_t a, uint32_t b, unsigned long long n) { return crc_mul(crc_x8n(n), a) ^ b; }
// the CRC-32 of a gzip trailer from the linear CRC of n bytes
DCA_HD inline uint32_t crc_finish(uint32_t lin, unsigned long long n) { return ~(lin ^ crc_mul(crc_x8n(n), 0xffffffffu)); }

// ------------------------------------------------------------------------------------------------------ gzip header
enum : int { H_OK = 0, H_NEED = 1, H_BAD = 2 };
// The member header at byte `at` of p[0, n): ID1 ID2, CM = 8, no reserved FLG bits, MTIME XFL OS, then FEXTRA, FNAME,
// FCOMMENT and FHCRC (checked) when flagged.  *len = header bytes.  H_NEED when it runs past n and the file goes on.
DCA_HD inline int parse_header(const uint8_t* p, long long n, long long at, bool eof, long long* len) {
  const int need = eof ? H_BAD : H_NEED;
  if (at + 10 > n) return at < n && p[at] != 0x1f ? H_BAD : need;
  if (p[at] != 0x1f || p[at + 1] != 0x8b || p[at + 2] != 8 || (p[at + 3] & 0xe0)) return H_BAD;
  const int flg = p[at + 3];
  long long q = at + 10;
  if (flg & 4) {                                          // FEXTRA
    if (q + 2 > n) return need;
    q += 2 + (p[q] | (p[q + 1] << 8));
    if (q > n) return need;
  }
  for (int f = 8; f <= 16; f <<= 1) {                     // FNAME, FCOMMENT: zero-terminated
    if (!(flg & f)) continue;
    while (q < n && p[q]) ++q;
    if (q >= n) return need;
    ++q;
  }
  if (flg & 2) {                                          // FHCRC: the low 16 bits of the CRC-32 of the bytes before
    if (q + 2 > n) return need;
    if ((crc32_bytes(0, p + at, q - at) & 0xffffu) != (uint32_t)(p[q] | (p[q + 1] << 8))) return H_BAD;
    q += 2;
  }
  *len = q - at;
  return H_OK;
}

// -------------------------------------------------------------------------------------------------- span decoder
struct MemberEnd {
  long long end;             // output position (of the span) after the member's last byte
  uint32_t crc, isize;       // its trailer
};

struct SpanResult {
  long long end_bit;         // where decoding stopped
  long long out_len;         // bytes of output
  long long min_ref;         // lowest output position a back-reference reached while the member was the span's first
                             // (< 0: before the span; 0 when none reached back)
  long long member_start;    // output position where the last member starting in the span starts, -1 without one
  int status;
  int members;               // member ends (trailers) in the span
};

// Decodes blocks from bit `start` of in[0, n) (eof: n is the end of the file) until a block boundary at or beyond
// `stop` (ST_STOP), or at least `out_stop` bytes of output (ST_FULL).  A block with BFINAL ends a member: its trailer
// is read, and when bytes remain the next member's header, and decoding goes on with an empty window.
// out == nullptr counts only; else out[0, out_cap) gets 16-bit symbols (bytes and kMarker references to the window
// before the span) and mem[0, mem_cap) the member ends.
DCA_HD inline SpanResult decode_span(const uint8_t* in, long long n, bool eof, long long start, long long stop,
                                     long long out_stop, uint16_t* out, long long out_cap, MemberEnd* mem, int mem_cap,
                                     Tables& t) {
  SpanResult r{start, 0, 0, -1, ST_BAD, 0};
  Bits b;
  b.init(in, n, start);
  long long o = 0;
  long long floor = -(1ll << 62);                       // first output position of the current member, when known
  const int short_input = eof ? ST_BAD : ST_NEED;
  for (;;) {
    const long long at = b.pos();
    if (at >= stop) { r.status = ST_STOP; break; }
    if (o >= out_stop) { r.status = ST_FULL; break; }
    const int last = (int)b.bits(1), type = (int)b.bits(2);
    if (type == 0) {                                     // stored
      b.align();
      const uint32_t len = b.bits(16), nlen = b.bits(16);
      if (b.over()) { r.status = short_input; return r; }
      if (len != (~nlen & 0xffffu)) return r;
      if (b.pos() + 8ll * len > n * 8) { r.status = short_input; return r; }
      for (uint32_t i = 0; i < len; ++i) {
        const uint32_t c = b.bits(8);
        if (out) { if (o >= out_cap) return r; out[o] = (uint16_t)c; }
        ++o;
      }
    } else if (type == 3) {
      return r;
    } else {
      if (type == 1) fixed_tables(t);
      else if (!dynamic_tables(b, t, false)) { if (b.over()) r.status = short_input; return r; }
      for (;;) {
        // every symbol takes at least one bit, so checking the input after each one bounds the loop by the input:
        // past it the bit reader reads zeros, which decode to a symbol for ever
        int sym = decode(b, t.lit);
        if (b.over()) { r.status = short_input; return r; }
        if (sym < 0) return r;
        if (sym < 256) {
          if (out) { if (o >= out_cap) return r; out[o] = (uint16_t)sym; }
          ++o;
          continue;
        }
        if (sym == 256) break;
        sym -= 257;
        if (sym >= 29) return r;
        int len;
        if (sym < 8) len = 3 + sym;
        else if (sym == 28) len = 258;
        else { const int e = (sym >> 2) - 1; len = ((4 | (sym & 3)) << e) + 3 + (int)b.bits(e); }
        const int ds = decode(b, t.dist);
        if (ds < 0 || ds >= 30) { if (b.over()) r.status = short_input; return r; }
        int dist = ds < 4 ? ds + 1 : ((2 | (ds & 1)) << ((ds >> 1) - 1)) + 1 + (int)b.bits((ds >> 1) - 1);
        if (b.over()) { r.status = short_input; return r; }
        const long long src = o - dist;
        if (src < floor) return r;                       // before the member's first byte
        if (src < r.min_ref) r.min_ref = src;
        if (out) {
          if (o + len > out_cap) return r;
          for (int i = 0; i < len; ++i) {
            const long long s = src + i;
            out[o + i] = s >= 0 ? out[s] : (uint16_t)(kMarker | (uint16_t)(-s - 1));
          }
        }
        o += len;
      }
    }
    if (b.over()) { r.status = short_input; return r; }
    if (!last) continue;
    // end of a member: the trailer, then the next member's header or the end of the file
    b.align();
    const uint32_t crc = b.bits(32), isize = b.bits(32);
    if (b.over()) { r.status = short_input; return r; }
    if (mem) {
      if (r.members >= mem_cap) return r;
      mem[r.members] = MemberEnd{o, crc, isize};
    }
    ++r.members;
    const long long byte = b.pos() >> 3;
    if (byte == n && eof) { r.end_bit = b.pos(); r.out_len = o; r.status = ST_END; return r; }
    long long hlen = 0;
    const int h = parse_header(in, n, byte, eof, &hlen);
    if (h == H_NEED) { r.status = ST_NEED; return r; }
    if (h == H_BAD) return r;                            // trailing garbage or a bad header
    b.init(in, n, (byte + hlen) * 8);
    floor = o;
    r.member_start = o;
  }
  r.end_bit = b.pos();
  r.out_len = o;
  return r;
}

// whether a block plausibly starts at `bit`: a dynamic block whose header is fully valid (HLIT <= 286, HDIST <= 30,
// complete code-length, literal/length and distance codes, a code for end-of-block), or a stored block whose padding
// is zero and whose LEN = ~NLEN
DCA_HD inline bool block_start(const uint8_t* in, long long n, long long bit, Tables& t) {
  Bits b;
  b.init(in, n, bit);
  b.bits(1);
  const int type = (int)b.bits(2);
  if (type == 2) return dynamic_tables(b, t, true);
  if (type != 0) return false;
  const int r = (int)(b.pos() & 7);
  if (r && b.bits(8 - r)) return false;
  const uint32_t len = b.bits(16), nlen = b.bits(16);
  return !b.over() && len == (~nlen & 0xffffu);
}

}  // namespace inflate
}  // namespace dca
