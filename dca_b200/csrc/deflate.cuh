// DEFLATE (RFC 1951) block encoder, written once for the host and the device: deflate.cu runs it with one CTA per
// block of kBlock input bytes (dca_gzip_device, dca_write_text_device_gz) and dca_gzip_host runs the same phases on the
// CPU, thread by thread, so that both give the same bytes.
//
// A block is encoded in phases separated by barriers; within a phase every thread's work is independent of the others'
// order (plain stores to its own slots, atomic max / add / or / xor), so the output depends on the input alone:
//   hash      positions of the 32 KB before the block go into a table of 4-byte hashes (atomic max: the latest wins);
//             then the block's positions in rounds of kThreads: each reads the table (the latest position before its
//             round with its hash) into prev[], then all of the round write themselves (atomic max)
//   parse     greedy LZ77: thread t parses from start[t] to the first token boundary at or past its nominal end, walking
//             up to kChain candidates of prev[]; start[t + 1] = end[t] is iterated to a fixed point, so the parse is
//             the serial greedy parse of the block whatever the number of threads
//   codes     symbol counts (atomic add), then thread 0 builds length-limited Huffman codes (15 bits, 7 for the code-
//             length code) and picks the smallest of a dynamic, a fixed and a stored block
//   emit      per-thread bit counts, one exclusive scan, then every thread ORs its bits into the zeroed output
// A non-final dynamic or fixed block ends with an empty stored block (a sync flush), so every block ends on a byte and
// blocks concatenate at byte offsets.  crc is the linear CRC-32 (initial 0, no final inversion) of the block's bytes.
#pragma once
#include "inflate.cuh"

namespace dca {
namespace deflate {

constexpr int kBlock = 32768;                 // input bytes per block
constexpr int kThreads = 512;
constexpr int kSub = kBlock / kThreads;       // nominal parse range of a thread
constexpr int kWindow = 32768;
constexpr int kHashBits = 13;
constexpr int kChain = 8;                     // candidates tried per position
constexpr int kNice = 128;                    // a match this long ends the search
constexpr int kMinMatch = 3, kMaxMatch = 258;
constexpr int kSlot = kBlock + 16;            // staged bytes of one block (a stored block takes kBlock + 5)
constexpr int kEmpty = -(1 << 30);
constexpr int kLit = 286, kDist = 30, kCl = 19;

enum : int { KIND_STORED = 0, KIND_FIXED = 1, KIND_DYNAMIC = 2 };

// ------------------------------------------------------------------------------------------ host / device atomics
DCA_HD inline void hd_max(int* p, int v) {
#ifdef __CUDA_ARCH__
  atomicMax(p, v);
#else
  if (v > *p) *p = v;
#endif
}
DCA_HD inline void hd_add(uint32_t* p, uint32_t v) {
#ifdef __CUDA_ARCH__
  atomicAdd(p, v);
#else
  *p += v;
#endif
}
DCA_HD inline void hd_or(uint32_t* p, uint32_t v) {
#ifdef __CUDA_ARCH__
  atomicOr(p, v);
#else
  *p |= v;
#endif
}
DCA_HD inline void hd_xor(uint32_t* p, uint32_t v) {
#ifdef __CUDA_ARCH__
  atomicXor(p, v);
#else
  *p ^= v;
#endif
}

// -------------------------------------------------------------------------------------------------- symbol tables
DCA_HD inline int len_sym(int len) {          // 257..285 for a match length 3..258
  if (len < 11) return 254 + len;
  if (len == 258) return 285;
  int e = 1;
  while ((len - 3) >> (e + 2) > 1) ++e;       // lengths of symbol class e: (4..7) << e, offset 3
  return 261 + 4 * e + (((len - 3) >> e) & 3);
}
DCA_HD inline int len_extra(int sym) { return sym < 265 || sym == 285 ? 0 : (sym - 261) >> 2; }
DCA_HD inline int len_base(int sym) {
  if (sym < 265) return sym - 254;
  if (sym == 285) return 258;
  const int e = (sym - 261) >> 2;
  return ((4 | ((sym - 261) & 3)) << e) + 3;
}
DCA_HD inline int dist_sym(int d) {           // 0..29 for a distance 1..32768
  if (d <= 4) return d - 1;
  int e = 1;
  while ((d - 1) >> (e + 1) > 1) ++e;         // distances of class e: (2..3) << e, offset 1
  return 2 * e + 2 + (((d - 1) >> e) & 1);
}
DCA_HD inline int dist_extra(int sym) { return sym < 4 ? 0 : (sym >> 1) - 1; }
DCA_HD inline int dist_base(int sym) { return sym < 4 ? sym + 1 : ((2 | (sym & 1)) << ((sym >> 1) - 1)) + 1; }
DCA_HD inline int fixed_len(int sym) { return sym < 144 ? 8 : sym < 256 ? 9 : sym < 280 ? 7 : 8; }

// --------------------------------------------------------------------------------------------- per-block state
struct Shared {
  int head[1 << kHashBits];
  uint16_t prev[kBlock];                      // distance to the previous position with the same hash, 0: none
  uint16_t dist[kBlock];                      // at a token's first byte: its distance, 0 for a literal
  uint8_t mlen[kBlock];                       // and its length - 3
  int start[kThreads], end[kThreads], dirty[kThreads];
  uint32_t bits[kThreads + 1];                // per-thread token bits, then their exclusive prefix
  uint32_t lfreq[kLit], dfreq[kDist], cfreq[kCl];
  uint8_t llen[kLit], dlen[kDist], clen[kCl];
  uint16_t lcode[kLit], dcode[kDist], ccode[kCl];
  uint16_t rank[kLit];                        // Huffman scratch: symbols in code-building order
  uint16_t rle[kLit + kDist];                 // code-length symbols (low 5 bits) and their extra value (<< 5)
  int nrle, hlit, hdist, hclen;
  uint32_t crc, hdr_bits;
  int kind, bytes, any;
  uint32_t crc_table[256];
};

// one block: in[0, len), with in[-hist, 0) readable as history (hist <= kWindow)
struct Block {
  const uint8_t* in;
  int len, hist, final;
};

DCA_HD inline uint32_t load4(const uint8_t* p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
DCA_HD inline int hash_at(const Block& b, int p) { return (int)((load4(b.in + p) * 2654435761u) >> (32 - kHashBits)); }

// ------------------------------------------------------------------------------------------------------ phases
// phase 0 (thread t): empty table, zero counts, CRC table, the thread's part of the block CRC
DCA_HD inline void init_phase(Shared& s, const Block& b, int t) {
  for (int i = t; i < (1 << kHashBits); i += kThreads) s.head[i] = kEmpty;
  for (int i = t; i < kLit; i += kThreads) s.lfreq[i] = 0;
  if (t < kDist) s.dfreq[t] = 0;
  if (t < 256) {
    uint32_t c = (uint32_t)t;
    for (int k = 0; k < 8; ++k) c = c & 1 ? (c >> 1) ^ inflate::kCrcPoly : c >> 1;
    s.crc_table[t] = c;
  }
  s.start[t] = t * kSub < b.len ? t * kSub : b.len;
  s.dirty[t] = 1;
  if (t == 0) { s.crc = 0; s.any = 1; }
}
DCA_HD inline uint32_t crc_part(const Shared& s, const Block& b, int t) {     // needs crc_table
  const int a = t * kSub < b.len ? t * kSub : b.len, e = a + kSub < b.len ? a + kSub : b.len;
  uint32_t c = 0;
  for (int p = a; p < e; ++p) c = s.crc_table[(c ^ b.in[p]) & 0xff] ^ (c >> 8);
  return inflate::crc_mul(inflate::crc_x8n((unsigned long long)(b.len - e)), c);
}
// phase 1: the history's positions (those whose 4 bytes lie before the block's end)
DCA_HD inline void history_phase(Shared& s, const Block& b, int t) {
  for (int p = -b.hist + t; p < 0 && p + 3 < b.len; p += kThreads) hd_max(&s.head[hash_at(b, p)], p);
}
// phase 2 of round r, read half: prev[] of the round's positions
DCA_HD inline void round_read(Shared& s, const Block& b, int r, int t) {
  const int p = r * kThreads + t;
  if (p >= b.len) return;
  int d = 0;
  if (p + 3 < b.len) {
    const int c = s.head[hash_at(b, p)];
    if (c != kEmpty && p - c <= kWindow) d = p - c;
  }
  s.prev[p] = (uint16_t)d;
}
DCA_HD inline void round_write(Shared& s, const Block& b, int r, int t) {
  const int p = r * kThreads + t;
  if (p + 3 < b.len) hd_max(&s.head[hash_at(b, p)], p);
}

// longest match at p among the chain's candidates (the first of the longest); returns its length, 0 for none
DCA_HD inline int find_match(const Shared& s, const Block& b, int p, int* dist) {
  if (p + 3 >= b.len || !s.prev[p]) return 0;
  const int maxl = b.len - p < kMaxMatch ? b.len - p : kMaxMatch;
  const uint8_t* q = b.in + p;
  int best = 0, c = p - s.prev[p];
  for (int k = 0; k < kChain; ++k) {
    const int d = p - c;
    if (d > kWindow) break;
    const uint8_t* r = b.in + c;
    if (r[best] == q[best]) {                 // cannot beat `best` otherwise
      int l = 0;
      while (l < maxl && r[l] == q[l]) ++l;
      if (l > best) { best = l; *dist = d; if (l >= kNice || l == maxl) break; }
    }
    if (c < 0 || !s.prev[c]) break;           // history positions have no chain
    c -= s.prev[c];
  }
  return best >= kMinMatch ? best : 0;
}
// phase 3: thread t's greedy parse from start[t] (when it changed) to its token boundary at or past its nominal end
DCA_HD inline void parse_phase(Shared& s, const Block& b, int t) {
  if (!s.dirty[t]) return;
  const int stop = (t + 1) * kSub < b.len ? (t + 1) * kSub : b.len;
  int p = s.start[t];
  while (p < stop) {
    int d = 0;
    const int l = find_match(s, b, p, &d);
    if (l) { s.dist[p] = (uint16_t)d; s.mlen[p] = (uint8_t)(l - kMinMatch); p += l; }
    else { s.dist[p] = 0; ++p; }
  }
  s.end[t] = p > s.start[t] ? p : s.start[t];
}
// phase 3b: the next start of thread t (the end of the parse before it, never before its nominal start); returns
// whether it changed
DCA_HD inline bool chain_phase(Shared& s, int t) {
  if (t == 0) { s.dirty[0] = 0; return false; }
  const int want = s.end[t - 1];
  s.dirty[t] = want != s.start[t];
  s.start[t] = want;
  return s.dirty[t] != 0;
}
// after the fixed point: thread t's tokens are the tokens from start[t] before its end
template <class F>
DCA_HD inline void for_tokens(const Shared& s, int t, F f) {
  for (int p = s.start[t]; p < s.end[t];) {
    const int d = s.dist[p];
    if (d) { const int l = s.mlen[p] + kMinMatch; f(p, l, d); p += l; }
    else { f(p, 0, 0); ++p; }
  }
}
// phase 4: symbol counts
DCA_HD inline void count_phase(Shared& s, const Block& b, int t) {
  for_tokens(s, t, [&](int p, int l, int d) {
    if (l) { hd_add(&s.lfreq[len_sym(l)], 1u); hd_add(&s.dfreq[dist_sym(d)], 1u); }
    else hd_add(&s.lfreq[b.in[p]], 1u);
  });
}

// ------------------------------------------------------------------------------------- Huffman codes (thread 0)
// Code lengths for freq[0, n) limited to `limit` bits; at least two symbols get a code (RFC 1951 decoders differ on
// codes of one symbol).  order: scratch of n.  Minimum-redundancy lengths by the in-place method of Moffat and
// Katajainen on the symbols sorted by (count, symbol), then lengths over the limit folded in by Kraft's inequality.
DCA_HD inline void huffman_lengths(const uint32_t* freq0, int n, int limit, uint8_t* len, uint16_t* order) {
  uint32_t freq[kLit];
  int used = 0;
  for (int i = 0; i < n; ++i) { freq[i] = freq0[i]; if (freq[i]) ++used; }
  for (int i = 0; i < n && used < 2; ++i) if (!freq[i]) { freq[i] = 1; ++used; }
  int m = 0;
  for (int i = 0; i < n; ++i) {               // insertion sort of the used symbols by (count, symbol)
    len[i] = 0;
    if (!freq[i]) continue;
    int j = m++;
    while (j > 0 && freq[order[j - 1]] > freq[i]) { order[j] = order[j - 1]; --j; }
    order[j] = (uint16_t)i;
  }
  int A[kLit];
  A[0] = A[1] = 0;
  for (int i = 0; i < m; ++i) A[i] = (int)freq[order[i]];
  // pass 1: internal node weights, with parent links of the consumed nodes
  A[0] += A[1];
  int root = 0, leaf = 2;
  for (int next = 1; next < m - 1; ++next) {
    if (leaf >= m || A[root] < A[leaf]) { A[next] = A[root]; A[root++] = next; }
    else A[next] = A[leaf++];
    if (leaf >= m || (root < next && A[root] < A[leaf])) { A[next] += A[root]; A[root++] = next; }
    else A[next] += A[leaf++];
  }
  // pass 2: internal node depths; pass 3: leaf depths, the least frequent symbols deepest
  A[m - 2] = 0;
  for (int next = m - 3; next >= 0; --next) A[next] = A[A[next]] + 1;
  int avail = 1, usedn = 0, depth = 0, next = m - 1;
  root = m - 2;
  while (avail > 0) {
    while (root >= 0 && A[root] == depth) { ++usedn; --root; }
    while (avail > usedn) { A[next--] = depth; --avail; }
    avail = 2 * usedn; ++depth; usedn = 0;
  }
  // counts per length, lengths past the limit folded to the limit, then Kraft restored by lengthening shorter codes
  int count[32];
  for (int l = 0; l < 32; ++l) count[l] = 0;
  for (int i = 0; i < m; ++i) count[A[i] < limit ? A[i] : limit]++;
  uint32_t kraft = 0;
  for (int l = 1; l <= limit; ++l) kraft += (uint32_t)count[l] << (limit - l);
  while (kraft > (1u << limit)) {
    count[limit]--;
    for (int l = limit - 1; l > 0; --l)
      if (count[l]) { count[l]--; count[l + 1] += 2; break; }
    kraft--;
  }
  int i = 0;                                  // least frequent first: the longest codes
  for (int l = limit; l >= 1; --l)
    for (int k = 0; k < count[l]; ++k) len[order[i++]] = (uint8_t)l;
}

// canonical codes of RFC 1951 3.2.2, bit-reversed for the LSB-first writer
DCA_HD inline void canonical_codes(const uint8_t* len, int n, uint16_t* code) {
  int count[16], next[16];
  for (int l = 0; l < 16; ++l) count[l] = 0;
  for (int i = 0; i < n; ++i) count[len[i]]++;
  count[0] = 0;
  int c = 0;
  for (int l = 1; l < 16; ++l) { c = (c + count[l - 1]) << 1; next[l] = c; }
  for (int i = 0; i < n; ++i) {
    if (!len[i]) { code[i] = 0; continue; }
    uint32_t v = (uint32_t)next[len[i]]++, r = 0;
    for (int k = 0; k < len[i]; ++k) { r = (r << 1) | (v & 1); v >>= 1; }
    code[i] = (uint16_t)r;
  }
}

DCA_HD inline int cl_order(int i) {           // the order of the code-length code's lengths in the header
  const uint8_t order[kCl] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  return order[i];
}

// phase 5 (thread 0): both codes, the code-length sequence, the block kind and its size in bytes
DCA_HD inline void codes_phase(Shared& s, const Block& b) {
  s.lfreq[256] = 1;
  huffman_lengths(s.lfreq, kLit, 15, s.llen, s.rank);
  huffman_lengths(s.dfreq, kDist, 15, s.dlen, s.rank);
  int hlit = kLit, hdist = kDist;
  while (hlit > 257 && !s.llen[hlit - 1]) --hlit;
  while (hdist > 1 && !s.dlen[hdist - 1]) --hdist;
  s.hlit = hlit; s.hdist = hdist;
  // run-length coded lengths over the one sequence of hlit + hdist values
  uint8_t seq[kLit + kDist];
  const int total = hlit + hdist;
  for (int i = 0; i < hlit; ++i) seq[i] = s.llen[i];
  for (int i = 0; i < hdist; ++i) seq[hlit + i] = s.dlen[i];
  for (int i = 0; i < kCl; ++i) s.cfreq[i] = 0;
  int nr = 0;
  for (int i = 0; i < total;) {
    const int v = seq[i];
    int run = 1;
    while (i + run < total && seq[i + run] == v) ++run;
    if (v == 0 && run >= 3) {
      const int k = run < 138 ? run : 138;
      if (k <= 10) s.rle[nr++] = (uint16_t)(17 | ((k - 3) << 5));
      else s.rle[nr++] = (uint16_t)(18 | ((k - 11) << 5));
      i += k;
    } else if (v != 0 && run >= 4) {
      s.rle[nr++] = (uint16_t)v;
      const int k = run - 1 < 6 ? run - 1 : 6;
      s.rle[nr++] = (uint16_t)(16 | ((k - 3) << 5));
      i += 1 + k;
    } else {
      s.rle[nr++] = (uint16_t)v;
      ++i;
    }
  }
  s.nrle = nr;
  for (int i = 0; i < nr; ++i) s.cfreq[s.rle[i] & 31]++;
  huffman_lengths(s.cfreq, kCl, 7, s.clen, s.rank);
  int hclen = kCl;
  while (hclen > 4 && !s.clen[cl_order(hclen - 1)]) --hclen;
  s.hclen = hclen;
  canonical_codes(s.llen, kLit, s.lcode);
  canonical_codes(s.dlen, kDist, s.dcode);
  canonical_codes(s.clen, kCl, s.ccode);
  // sizes in bits after the 3 header bits
  unsigned long long hdr = 5 + 5 + 4 + 3ull * hclen, dyn = 0, fix = 0;
  for (int i = 0; i < nr; ++i) {
    const int sym = s.rle[i] & 31;
    hdr += s.clen[sym] + (sym == 16 ? 2 : sym == 17 ? 3 : sym == 18 ? 7 : 0);
  }
  for (int i = 0; i < kLit; ++i) {
    const unsigned long long f = s.lfreq[i], x = i > 256 ? (unsigned long long)len_extra(i) : 0ull;
    dyn += f * (s.llen[i] + x);
    fix += f * (fixed_len(i) + x);
  }
  for (int i = 0; i < kDist; ++i) {
    const unsigned long long f = s.dfreq[i], x = (unsigned long long)dist_extra(i);
    dyn += f * (s.dlen[i] + x);
    fix += f * (5 + x);
  }
  // a non-final block is followed by the 3 bits of an empty stored block, the padding and LEN / NLEN
  const unsigned long long tail = b.final ? 0 : 3;
  const long long dyn_bytes = (long long)((3 + hdr + dyn + tail + 7) / 8) + (b.final ? 0 : 4);
  const long long fix_bytes = (long long)((3 + fix + tail + 7) / 8) + (b.final ? 0 : 4);
  const long long stored_bytes = 5ll + b.len;
  if (dyn_bytes < fix_bytes && dyn_bytes < stored_bytes) { s.kind = KIND_DYNAMIC; s.bytes = (int)dyn_bytes; s.hdr_bits = (uint32_t)(3 + hdr); }
  else if (fix_bytes < stored_bytes) { s.kind = KIND_FIXED; s.bytes = (int)fix_bytes; s.hdr_bits = 3; }
  else { s.kind = KIND_STORED; s.bytes = (int)stored_bytes; s.hdr_bits = 0; }
}

// LSB-first bits ORed into out words from bit `pos` on (the words are zero where this writer writes)
struct BitSink {
  uint32_t* w;
  long long word;
  uint64_t acc;
  int fill;
  DCA_HD void init(uint32_t* words, long long pos) { w = words; word = pos >> 5; fill = (int)(pos & 31); acc = 0; }
  DCA_HD void put(uint32_t v, int k) {        // k <= 32
    acc |= (uint64_t)v << fill;
    fill += k;
    if (fill >= 32) { hd_or(&w[word++], (uint32_t)acc); acc >>= 32; fill -= 32; }
  }
  DCA_HD void flush() { if (fill) hd_or(&w[word], (uint32_t)acc); }
};

DCA_HD inline uint32_t token_bits(const Shared& s, int l, int d, int lit) {
  if (!l) return s.kind == KIND_DYNAMIC ? s.llen[lit] : fixed_len(lit);
  const int ls = len_sym(l), ds = dist_sym(d);
  return (s.kind == KIND_DYNAMIC ? s.llen[ls] + s.dlen[ds] : fixed_len(ls) + 5) + len_extra(ls) + dist_extra(ds);
}
DCA_HD inline uint32_t fixed_code(int sym) {  // bit-reversed fixed code
  int v, n;
  if (sym < 144) { v = 0x30 + sym; n = 8; }
  else if (sym < 256) { v = 0x190 + sym - 144; n = 9; }
  else if (sym < 280) { v = sym - 256; n = 7; }
  else { v = 0xc0 + sym - 280; n = 8; }
  uint32_t r = 0;
  for (int k = 0; k < n; ++k) { r = (r << 1) | (v & 1); v >>= 1; }
  return r;
}
DCA_HD inline void put_sym(BitSink& o, const Shared& s, int sym) {
  if (s.kind == KIND_DYNAMIC) o.put(s.lcode[sym], s.llen[sym]);
  else o.put(fixed_code(sym), fixed_len(sym));
}

// phase 6: bit count of thread t's tokens
DCA_HD inline void size_phase(Shared& s, const Block& b, int t) {
  uint32_t n = 0;
  for_tokens(s, t, [&](int p, int l, int d) { n += token_bits(s, l, d, l ? 0 : b.in[p]); });
  s.bits[t] = n;
}
// phase 7 (thread 0): exclusive prefix of the bit counts after the header; the header itself
DCA_HD inline void header_phase(Shared& s, const Block& b, uint32_t* out) {
  uint32_t run = s.hdr_bits;
  for (int t = 0; t < kThreads; ++t) { const uint32_t n = s.bits[t]; s.bits[t] = run; run += n; }
  s.bits[kThreads] = run;
  BitSink o;
  o.init(out, 0);
  o.put(b.final ? 1u : 0u, 1);
  o.put((uint32_t)s.kind, 2);                 // BTYPE 01 fixed, 10 dynamic
  if (s.kind == KIND_DYNAMIC) {
    o.put((uint32_t)(s.hlit - 257), 5);
    o.put((uint32_t)(s.hdist - 1), 5);
    o.put((uint32_t)(s.hclen - 4), 4);
    for (int i = 0; i < s.hclen; ++i) o.put(s.clen[cl_order(i)], 3);
    for (int i = 0; i < s.nrle; ++i) {
      const int sym = s.rle[i] & 31, x = s.rle[i] >> 5;
      o.put(s.ccode[sym], s.clen[sym]);
      if (sym == 16) o.put((uint32_t)x, 2);
      else if (sym == 17) o.put((uint32_t)x, 3);
      else if (sym == 18) o.put((uint32_t)x, 7);
    }
  }
  o.flush();
}
// phase 8: thread t's tokens; the last thread adds the end of block and, before another block, the sync flush
DCA_HD inline void emit_phase(const Shared& s, const Block& b, int t, uint32_t* out) {
  BitSink o;
  o.init(out, s.bits[t]);
  for_tokens(s, t, [&](int p, int l, int d) {
    if (!l) { put_sym(o, s, b.in[p]); return; }
    const int ls = len_sym(l), ds = dist_sym(d);
    put_sym(o, s, ls);
    if (len_extra(ls)) o.put((uint32_t)(l - len_base(ls)), len_extra(ls));
    if (s.kind == KIND_DYNAMIC) o.put(s.dcode[ds], s.dlen[ds]);
    else { uint32_t r = 0, v = (uint32_t)ds; for (int k = 0; k < 5; ++k) { r = (r << 1) | (v & 1); v >>= 1; } o.put(r, 5); }
    if (dist_extra(ds)) o.put((uint32_t)(d - dist_base(ds)), dist_extra(ds));
  });
  if (t == kThreads - 1) {
    put_sym(o, s, 256);
    if (!b.final) {                           // empty stored block: 3 zero bits, padding, LEN 0, NLEN 0xffff
      o.put(0u, 3);
      if (o.fill & 7) o.put(0u, 8 - (o.fill & 7));
      o.put(0xffff0000u, 32);
    }
  }
  o.flush();
}
// stored block (byte t and on, stride kThreads): header byte, LEN, NLEN, the bytes
DCA_HD inline void stored_phase(const Block& b, int t, uint8_t* out) {
  if (t == 0) {
    out[0] = b.final ? 1 : 0;
    out[1] = (uint8_t)b.len; out[2] = (uint8_t)(b.len >> 8);
    out[3] = (uint8_t)~b.len; out[4] = (uint8_t)(~b.len >> 8);
  }
  for (int i = t; i < b.len; i += kThreads) out[5 + i] = b.in[i];
}

// the empty final block ending a member (fixed Huffman, BFINAL, end of block) is the bytes 0x03 0x00

// the most bytes a gzip member of n input bytes takes: header, trailer, and per block a stored block's
DCA_HD inline long long gzip_bound(long long n) {
  const long long blocks = (n + kBlock - 1) / kBlock;
  return 18 + (n ? n + 5 * blocks : 2);
}

#ifdef __CUDACC__
// One gzip member compressed on the device, fed in pieces of device memory on one stream (deflate.cu).  feed() appends
// to out: the member's header when `first`, the blocks of in[0, n), and when `last` the final block and the trailer;
// *out_len = the bytes it wrote, at most gzip_bound(n).  It returns when they are written.
class GzipMember {
 public:
  ~GzipMember();
  int init(cudaStream_t s);
  int feed(const uint8_t* in, long long n, bool first, bool last, uint8_t* out, long long* out_len);
  long long blocks() const { return blocks_; }
  long long stored() const { return stored_; }
  static long long device_bytes();
 private:
  cudaStream_t s_ = nullptr;
  uint8_t* slots_ = nullptr;
  int *sizes_ = nullptr, *kinds_ = nullptr;
  uint32_t* crcs_ = nullptr;
  long long* offs_ = nullptr;
  void *st_ = nullptr, *h_st_ = nullptr;
  unsigned long long isize_ = 0;
  long long blocks_ = 0, stored_ = 0;
};
#endif

}  // namespace deflate
}  // namespace dca
