// toplingdb_b200/csrc/inflate_rules.h — raw DEFLATE (RFC 1951) decoder for one data block, host + device.
//
// The reference stores a kZlibCompression block as  varint32 uncompressed_size ‖ raw deflate stream  (Zlib_Compress,
// util/compression.h:746-826: compress_format_version 2, window_bits -14 = no zlib header / Adler-32) and reads it back with
// Zlib_Uncompress (:834-924) from UncompressBlockData (table/format.cc:511).  On the device every compressed block is inflated by
// ONE WARP (decode.cu inflate_blocks_kernel): lane 0 runs this sequential decoder with its tables and output window in shared memory;
// the host runs it on compressed index blocks (api.cu).  Canonical Huffman decoding: a first-level table, then by code length
// (count[] / symbol[] per code, one bit per step).  tests/test_inflate_rules_host.py compiles this header for the host and checks it
// against zlib on reference-written blocks and on random streams of all three block types.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B200C_INF_HD __host__ __device__
#else
#define B200C_INF_HD
#endif

namespace b200c {

constexpr int kInfMaxBits = 15, kInfMaxLCodes = 286, kInfMaxDCodes = 30, kInfFixLCodes = 288;

struct InfBits {  // LSB-first bit reader over [p, end)
  const uint8_t* p;
  const uint8_t* end;
  uint64_t buf;
  int cnt;
  int err;
};
B200C_INF_HD inline void inf_refill(InfBits& b) {
  while (b.cnt <= 56 && b.p < b.end) {
    b.buf |= (uint64_t)(*b.p++) << b.cnt;
    b.cnt += 8;
  }
}
B200C_INF_HD inline uint32_t inf_bits(InfBits& b, int n) {  // n <= 16
  if (b.cnt < n) {
    inf_refill(b);
    if (b.cnt < n) {
      b.err = 1;
      return 0;
    }
  }
  const uint32_t v = (uint32_t)(b.buf & ((1ull << n) - 1));
  b.buf >>= n;
  b.cnt -= n;
  return v;
}

struct InfHuff {  // canonical code: count[len] codes of each length, symbols ordered by (length, value)
  uint16_t* count;   // [kInfMaxBits + 1]
  uint16_t* symbol;
};
// The decoder's tables.  On the device they live in SHARED memory, one slice per warp (as thread-local arrays they go to local
// memory, and with tens of thousands of blocks in flight every count[] / symbol[] probe of the bit-by-bit decode was an L2 round
// trip).
constexpr int kInfLBits = 9, kInfDBits = 6;  // first-level lookup: codes of up to this many bits decode with one table probe
struct InfWork {
  uint16_t lcount[kInfMaxBits + 1], dcount[kInfMaxBits + 1];
  uint16_t lsym[kInfFixLCodes], dsym[kInfMaxDCodes];
  uint8_t lengths[kInfFixLCodes + kInfMaxDCodes + 2];
  uint16_t ltab[1 << kInfLBits], dtab[1 << kInfDBits];  // (symbol << 4) | code length, indexed by the next bits of the stream; 0: longer code
};
static_assert(sizeof(InfWork) == 2172 && (sizeof(InfWork) / 4) % 2 == 1, "an odd number of 32-bit words per thread / warp slice");
// lengths[n] -> code; returns 0 for a complete code, > 0 incomplete, < 0 over-subscribed (as zlib's inflate_table reports them)
B200C_INF_HD inline int inf_build(InfHuff& h, const uint8_t* lengths, int n) {
  for (int l = 0; l <= kInfMaxBits; l++) h.count[l] = 0;
  for (int s = 0; s < n; s++) h.count[lengths[s]]++;
  if (h.count[0] == n) return 0;  // no codes: legal for the distance code of a block without matches
  int left = 1;
  for (int l = 1; l <= kInfMaxBits; l++) {
    left <<= 1;
    left -= h.count[l];
    if (left < 0) return left;
  }
  uint16_t offs[kInfMaxBits + 1];
  offs[1] = 0;
  for (int l = 1; l < kInfMaxBits; l++) offs[l + 1] = (uint16_t)(offs[l] + h.count[l]);
  for (int s = 0; s < n; s++)
    if (lengths[s] != 0) h.symbol[offs[lengths[s]]++] = (uint16_t)s;
  return left;
}
B200C_INF_HD inline int inf_decode(InfBits& b, const InfHuff& h) {
  if (b.cnt < kInfMaxBits) inf_refill(b);
  int code = 0, first = 0, index = 0;
  uint64_t buf = b.buf;
  const int avail = b.cnt;
  for (int len = 1; len <= kInfMaxBits; len++) {
    if (len > avail) break;
    code |= (int)(buf & 1);
    buf >>= 1;
    const int count = h.count[len];
    if (code - count < first) {
      b.buf = buf;
      b.cnt = avail - len;
      return h.symbol[index + (code - first)];
    }
    index += count;
    first += count;
    first <<= 1;
    code <<= 1;
  }
  b.err = 1;
  return -1;
}

// First-level table of a canonical code: entry[next kbits of the stream] = (symbol << 4) | length for every code of at most kbits
// bits (the stream delivers a code's first bit in the lowest position, so the table is indexed by the bit-reversed code).
B200C_INF_HD inline void inf_build_table(const InfHuff& h, const uint8_t* lengths, int n, uint16_t* tab, int kbits) {
  for (int i = 0; i < (1 << kbits); i++) tab[i] = 0;
  uint32_t next[kInfMaxBits + 2];
  uint32_t code = 0;
  next[0] = 0;
  for (int l = 1; l <= kInfMaxBits; l++) {
    code = (code + (l > 1 ? h.count[l - 1] : 0)) << 1;
    next[l] = code;
  }
  for (int s = 0; s < n; s++) {
    const int l = lengths[s];
    if (l == 0) continue;
    const uint32_t c = next[l]++;
    if (l > kbits) continue;
    uint32_t r = 0;
    for (int i = 0; i < l; i++) r |= ((c >> i) & 1u) << (l - 1 - i);
    const uint16_t e = (uint16_t)((s << 4) | l);
    for (uint32_t f = r; f < (1u << kbits); f += 1u << l) tab[f] = e;
  }
}
B200C_INF_HD inline int inf_decode_fast(InfBits& b, const InfHuff& h, const uint16_t* tab, int kbits) {
  if (b.cnt < kInfMaxBits) inf_refill(b);
  const uint32_t e = tab[(uint32_t)b.buf & ((1u << kbits) - 1)];
  const int l = (int)(e & 15u);
  if (l != 0 && l <= b.cnt) {
    b.buf >>= l;
    b.cnt -= l;
    return (int)(e >> 4);
  }
  return inf_decode(b, h);  // a code longer than the table's reach (or the tail of the stream)
}

// Inflates the raw deflate stream src[0, n) into dst[0, cap); returns the number of bytes written or -1 (malformed stream, output
// larger than cap, input exhausted).  dst may be global or local memory: back references are read from dst itself.
B200C_INF_HD inline long inflate_raw(const uint8_t* src, uint32_t n, uint8_t* dst, uint32_t cap, InfWork* wk) {
  // (the length / distance base tables of RFC 1951 3.2.5 and the code-length order of 3.2.7 are computed, not stored: a thread's
  //  constant arrays would live in local memory on the device)
  const uint64_t order_lo = 16ull | 17ull << 5 | 18ull << 10 | 0ull << 15 | 8ull << 20 | 7ull << 25 | 9ull << 30 | 6ull << 35 | 10ull << 40 |
                            5ull << 45 | 11ull << 50 | 4ull << 55;
  const uint64_t order_hi = 12ull | 3ull << 5 | 13ull << 10 | 2ull << 15 | 14ull << 20 | 1ull << 25 | 15ull << 30;
  InfBits b{src, src + n, 0, 0, 0};
  uint8_t* lengths = wk->lengths;
  InfHuff lc, dc;
  lc.count = wk->lcount;
  lc.symbol = wk->lsym;
  dc.count = wk->dcount;
  dc.symbol = wk->dsym;
  uint32_t out = 0;
  for (;;) {
    const uint32_t last = inf_bits(b, 1), type = inf_bits(b, 2);
    if (b.err) return -1;
    if (type == 0) {  // stored: skip to the byte boundary, LEN, NLEN, bytes
      b.buf >>= b.cnt & 7;
      b.cnt -= b.cnt & 7;
      const uint32_t len = inf_bits(b, 16), nlen = inf_bits(b, 16);
      if (b.err || len != (~nlen & 0xffffu)) return -1;
      for (uint32_t i = 0; i < len; i++) {
        const uint32_t c = inf_bits(b, 8);
        if (b.err || out >= cap) return -1;
        dst[out++] = (uint8_t)c;
      }
    } else if (type == 1 || type == 2) {
      if (type == 1) {  // fixed code (RFC 1951 3.2.6)
        int s = 0;
        for (; s < 144; s++) lengths[s] = 8;
        for (; s < 256; s++) lengths[s] = 9;
        for (; s < 280; s++) lengths[s] = 7;
        for (; s < kInfFixLCodes; s++) lengths[s] = 8;
        inf_build(lc, lengths, kInfFixLCodes);
        inf_build_table(lc, lengths, kInfFixLCodes, wk->ltab, kInfLBits);
        for (s = 0; s < kInfMaxDCodes; s++) lengths[s] = 5;
        inf_build(dc, lengths, kInfMaxDCodes);
        inf_build_table(dc, lengths, kInfMaxDCodes, wk->dtab, kInfDBits);
      } else {  // dynamic code: code-length code, then the literal/length and distance code lengths (3.2.7)
        const int nlen = (int)inf_bits(b, 5) + 257, ndist = (int)inf_bits(b, 5) + 1, ncode = (int)inf_bits(b, 4) + 4;
        if (b.err || nlen > kInfMaxLCodes || ndist > kInfMaxDCodes) return -1;
        int i = 0;
        for (; i < 19; i++) {
          const uint32_t o = (uint32_t)((i < 12 ? order_lo >> (5 * i) : order_hi >> (5 * (i - 12))) & 31);
          lengths[o] = i < ncode ? (uint8_t)inf_bits(b, 3) : (uint8_t)0;
        }
        if (b.err) return -1;
        if (inf_build(lc, lengths, 19) != 0) return -1;  // the code-length code must be complete
        i = 0;
        while (i < nlen + ndist) {
          int sym = inf_decode(b, lc);
          if (sym < 0) return -1;
          if (sym < 16) {
            lengths[i++] = (uint8_t)sym;
          } else {
            int prev = 0, rep;
            if (sym == 16) {
              if (i == 0) return -1;
              prev = lengths[i - 1];
              rep = 3 + (int)inf_bits(b, 2);
            } else if (sym == 17) {
              rep = 3 + (int)inf_bits(b, 3);
            } else {
              rep = 11 + (int)inf_bits(b, 7);
            }
            if (b.err || i + rep > nlen + ndist) return -1;
            while (rep--) lengths[i++] = (uint8_t)prev;
          }
        }
        if (lengths[256] == 0) return -1;  // no end-of-block code
        // an incomplete code is only legal when it has a single code word (zlib's inflate_table, puff.c)
        int e = inf_build(lc, lengths, nlen);
        if (e < 0 || (e > 0 && nlen - lc.count[0] != 1)) return -1;
        inf_build_table(lc, lengths, nlen, wk->ltab, kInfLBits);
        uint8_t* dl = lengths + nlen;
        e = inf_build(dc, dl, ndist);
        if (e < 0 || (e > 0 && ndist - dc.count[0] != 1)) return -1;
        inf_build_table(dc, dl, ndist, wk->dtab, kInfDBits);
      }
      for (;;) {  // literals and matches until end-of-block
        int sym = inf_decode_fast(b, lc, wk->ltab, kInfLBits);
        if (sym < 0) return -1;
        if (sym < 256) {
          if (out >= cap) return -1;
          dst[out++] = (uint8_t)sym;
        } else if (sym == 256) {
          break;
        } else {
          sym -= 257;
          if (sym >= 29) return -1;
          const int le = sym < 8 || sym == 28 ? 0 : (sym >> 2) - 1;
          uint32_t len = (sym < 8 ? 3u + (uint32_t)sym : sym == 28 ? 258u : (((4u + ((uint32_t)sym & 3u)) << le) + 3u)) + inf_bits(b, le);
          const int ds = inf_decode_fast(b, dc, wk->dtab, kInfDBits);
          if (ds < 0 || ds >= 30) return -1;
          const int de = ds < 4 ? 0 : (ds >> 1) - 1;
          const uint32_t dist = (ds < 4 ? 1u + (uint32_t)ds : (((2u + ((uint32_t)ds & 1u)) << de) + 1u)) + inf_bits(b, de);
          if (b.err || dist > out || out + len > cap) return -1;
          while (len--) {
            dst[out] = dst[out - dist];
            out++;
          }
        }
      }
    } else {
      return -1;
    }
    if (last) break;
  }
  return (long)out;
}

constexpr uint8_t kZlibCompressionType = 2;  // block trailer type byte of kZlibCompression (include/rocksdb/compression_type.h)
// The varint32 prefix of a compressed block p[0, size): its length in bytes, 0 when it does not end within the block's first five
// bytes; the announced uncompressed size in *u.  Each caller bounds *u by what it accepts.
B200C_INF_HD inline int inf_size_prefix(const uint8_t* p, uint32_t size, uint64_t* u) {
  const uint8_t* end = p + (size < 5 ? size : 5);
  uint64_t r = 0;
  int n = 0;
#pragma unroll 1
  for (int s = 0; s <= 28; s += 7) {
    if (p + n >= end) return 0;
    const uint8_t c = p[n++];
    r |= (uint64_t)(c & 127) << s;
    if (c < 128) {
      *u = r;
      return n;
    }
  }
  return 0;
}

}  // namespace b200c
