/* oracle/compaction_oracle.c — CPU restatement of ToplingDB's compaction hot path (see header).
 * TEST INFRASTRUCTURE ONLY — the checker, never the product.  Parity status: PINNED (header). */
#define _GNU_SOURCE
#include "compaction_oracle.h"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <zlib.h>

static __thread char g_err[256];
const char* orc_last_error(void) { return g_err; }
#define FAIL(code, ...)                         \
  do {                                          \
    snprintf(g_err, sizeof g_err, __VA_ARGS__); \
    return (code);                              \
  } while (0)
void orc_free(void* p) { free(p); }

/* ------------------------------------------------------------------ byte buffer */
typedef struct buf {
  uint8_t* p;
  size_t n, cap;
} buf;
static void buf_reserve(buf* b, size_t extra) {
  if (b->n + extra > b->cap) {
    size_t c = b->cap ? b->cap * 2 : 256;
    while (c < b->n + extra) c *= 2;
    b->p = (uint8_t*)realloc(b->p, c);
    b->cap = c;
  }
}
static void buf_put(buf* b, const void* d, size_t n) {
  buf_reserve(b, n);
  if (n) memcpy(b->p + b->n, d, n);
  b->n += n;
}
static void buf_u32(buf* b, uint32_t v) { buf_put(b, &v, 4); } /* little-endian hosts only */
static void buf_free(buf* b) {
  free(b->p);
  b->p = NULL;
  b->n = b->cap = 0;
}

/* ------------------------------------------------------------------ varints (util/coding.h) */
int orc_put_varint64(uint8_t* dst, uint64_t v) {
  int i = 0;
  while (v >= 128) {
    dst[i++] = (uint8_t)(v | 128);
    v >>= 7;
  }
  dst[i++] = (uint8_t)v;
  return i;
}
static void buf_varint(buf* b, uint64_t v) {
  uint8_t t[10];
  buf_put(b, t, (size_t)orc_put_varint64(t, v));
}
static int varint_len(uint64_t v) { /* VarintLength, util/coding.cc */
  int n = 1;
  while (v >= 128) {
    v >>= 7;
    n++;
  }
  return n;
}
static const uint8_t* get_varint(const uint8_t* p, const uint8_t* end, uint64_t* v) {
  uint64_t r = 0;
  for (int s = 0; s <= 63 && p < end; s += 7) {
    uint8_t c = *p++;
    r |= (uint64_t)(c & 127) << s;
    if (c < 128) {
      *v = r;
      return p;
    }
  }
  return NULL;
}
static uint64_t zigzag_enc(int64_t v) { return ((uint64_t)v << 1) ^ (uint64_t)(v >> 63); } /* PutVarsignedint64 */

/* ------------------------------------------------------------------ CRC32C (util/crc32c.cc; Castagnoli, reflected) */
static uint32_t crc_tab[256];
static int crc_tab_ready;
static void crc_init(void) {
  for (uint32_t i = 0; i < 256; i++) {
    uint32_t c = i;
    for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0x82F63B78u & (0u - (c & 1)));
    crc_tab[i] = c;
  }
  crc_tab_ready = 1;
}
uint32_t orc_crc32c_extend(uint32_t crc, const void* data, size_t n) {
  if (!crc_tab_ready) crc_init();
  const uint8_t* p = (const uint8_t*)data;
  uint32_t c = crc ^ 0xffffffffu;
  for (size_t i = 0; i < n; i++) c = crc_tab[(c ^ p[i]) & 0xff] ^ (c >> 8);
  return c ^ 0xffffffffu;
}
uint32_t orc_crc32c_value(const void* data, size_t n) { return orc_crc32c_extend(0, data, n); }
uint32_t orc_crc32c_mask(uint32_t crc) { return ((crc >> 15) | (crc << 17)) + 0xa282ead8u; }

/* ------------------------------------------------------------------ XXH3-64 (util/xxhash.h:3644-5235, seed 0, default secret) */
static const uint8_t kSecret[192] = {
    0xb8, 0xfe, 0x6c, 0x39, 0x23, 0xa4, 0x4b, 0xbe, 0x7c, 0x01, 0x81, 0x2c, 0xf7, 0x21, 0xad, 0x1c, 0xde, 0xd4, 0x6d, 0xe9,
    0x83, 0x90, 0x97, 0xdb, 0x72, 0x40, 0xa4, 0xa4, 0xb7, 0xb3, 0x67, 0x1f, 0xcb, 0x79, 0xe6, 0x4e, 0xcc, 0xc0, 0xe5, 0x78,
    0x82, 0x5a, 0xd0, 0x7d, 0xcc, 0xff, 0x72, 0x21, 0xb8, 0x08, 0x46, 0x74, 0xf7, 0x43, 0x24, 0x8e, 0xe0, 0x35, 0x90, 0xe6,
    0x81, 0x3a, 0x26, 0x4c, 0x3c, 0x28, 0x52, 0xbb, 0x91, 0xc3, 0x00, 0xcb, 0x88, 0xd0, 0x65, 0x8b, 0x1b, 0x53, 0x2e, 0xa3,
    0x71, 0x64, 0x48, 0x97, 0xa2, 0x0d, 0xf9, 0x4e, 0x38, 0x19, 0xef, 0x46, 0xa9, 0xde, 0xac, 0xd8, 0xa8, 0xfa, 0x76, 0x3f,
    0xe3, 0x9c, 0x34, 0x3f, 0xf9, 0xdc, 0xbb, 0xc7, 0xc7, 0x0b, 0x4f, 0x1d, 0x8a, 0x51, 0xe0, 0x4b, 0xcd, 0xb4, 0x59, 0x31,
    0xc8, 0x9f, 0x7e, 0xc9, 0xd9, 0x78, 0x73, 0x64, 0xea, 0xc5, 0xac, 0x83, 0x34, 0xd3, 0xeb, 0xc3, 0xc5, 0x81, 0xa0, 0xff,
    0xfa, 0x13, 0x63, 0xeb, 0x17, 0x0d, 0xdd, 0x51, 0xb7, 0xf0, 0xda, 0x49, 0xd3, 0x16, 0x55, 0x26, 0x29, 0xd4, 0x68, 0x9e,
    0x2b, 0x16, 0xbe, 0x58, 0x7d, 0x47, 0xa1, 0xfc, 0x8f, 0xf8, 0xb8, 0xd1, 0x7a, 0xd0, 0x31, 0xce, 0x45, 0xcb, 0x3a, 0x8f,
    0x95, 0x16, 0x04, 0x28, 0xaf, 0xd7, 0xfb, 0xca, 0xbb, 0x4b, 0x40, 0x7e};
#define P32_1 0x9E3779B1ull
#define P32_2 0x85EBCA77ull
#define P32_3 0xC2B2AE3Dull
#define P64_1 0x9E3779B185EBCA87ull
#define P64_2 0xC2B2AE3D27D4EB4Full
#define P64_3 0x165667B19E3779F9ull
#define P64_4 0x85EBCA77C2B2AE63ull
#define P64_5 0x27D4EB2F165667C5ull
static uint64_t rd64(const uint8_t* p) {
  uint64_t v;
  memcpy(&v, p, 8);
  return v;
}
static uint32_t rd32(const uint8_t* p) {
  uint32_t v;
  memcpy(&v, p, 4);
  return v;
}
static uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
static uint64_t mul128_fold64(uint64_t a, uint64_t b) {
  unsigned __int128 m = (unsigned __int128)a * b;
  return (uint64_t)m ^ (uint64_t)(m >> 64);
}
static uint64_t xxh64_avalanche(uint64_t h) {
  h ^= h >> 33;
  h *= P64_2;
  h ^= h >> 29;
  h *= P64_3;
  h ^= h >> 32;
  return h;
}
static uint64_t xxh3_avalanche(uint64_t h) {
  h ^= h >> 37;
  h *= 0x165667919E3779F9ull;
  h ^= h >> 32;
  return h;
}
static uint64_t mix16(const uint8_t* in, const uint8_t* sec) {
  return mul128_fold64(rd64(in) ^ rd64(sec), rd64(in + 8) ^ rd64(sec + 8));
}
static void xxh3_accumulate_stripe(uint64_t acc[8], const uint8_t* in, const uint8_t* sec) {
  for (int i = 0; i < 8; i++) {
    uint64_t dv = rd64(in + 8 * i), dk = dv ^ rd64(sec + 8 * i);
    acc[i ^ 1] += dv;
    acc[i] += (dk & 0xffffffffull) * (dk >> 32);
  }
}
uint64_t orc_xxh3_64(const void* data, size_t len) {
  const uint8_t* in = (const uint8_t*)data;
  if (len <= 16) {
    if (len > 8) {
      uint64_t f1 = rd64(kSecret + 24) ^ rd64(kSecret + 32), f2 = rd64(kSecret + 40) ^ rd64(kSecret + 48);
      uint64_t lo = rd64(in) ^ f1, hi = rd64(in + len - 8) ^ f2;
      return xxh3_avalanche(len + __builtin_bswap64(lo) + hi + mul128_fold64(lo, hi));
    }
    if (len >= 4) {
      uint64_t i1 = rd32(in), i2 = rd32(in + len - 4);
      uint64_t flip = rd64(kSecret + 8) ^ rd64(kSecret + 16);
      uint64_t h = (i2 + (i1 << 32)) ^ flip;
      h ^= rotl64(h, 49) ^ rotl64(h, 24);
      h *= 0x9FB21C651E98DF25ull;
      h ^= (h >> 35) + len;
      h *= 0x9FB21C651E98DF25ull;
      return h ^ (h >> 28);
    }
    if (len) {
      uint32_t c = ((uint32_t)in[0] << 16) | ((uint32_t)in[len >> 1] << 24) | in[len - 1] | ((uint32_t)len << 8);
      return xxh64_avalanche((uint64_t)c ^ (uint64_t)(rd32(kSecret) ^ rd32(kSecret + 4)));
    }
    return xxh64_avalanche(rd64(kSecret + 56) ^ rd64(kSecret + 64));
  }
  if (len <= 128) {
    uint64_t acc = len * P64_1, acc_end;
    acc += mix16(in, kSecret);
    acc_end = mix16(in + len - 16, kSecret + 16);
    if (len > 32) {
      acc += mix16(in + 16, kSecret + 32);
      acc_end += mix16(in + len - 32, kSecret + 48);
      if (len > 64) {
        acc += mix16(in + 32, kSecret + 64);
        acc_end += mix16(in + len - 48, kSecret + 80);
        if (len > 96) {
          acc += mix16(in + 48, kSecret + 96);
          acc_end += mix16(in + len - 64, kSecret + 112);
        }
      }
    }
    return xxh3_avalanche(acc + acc_end);
  }
  if (len <= 240) {
    uint64_t acc = len * P64_1, acc_end;
    unsigned rounds = (unsigned)len / 16;
    for (unsigned i = 0; i < 8; i++) acc += mix16(in + 16 * i, kSecret + 16 * i);
    acc_end = mix16(in + len - 16, kSecret + 136 - 17);
    acc = xxh3_avalanche(acc);
    for (unsigned i = 8; i < rounds; i++) acc_end += mix16(in + 16 * i, kSecret + 16 * (i - 8) + 3);
    return xxh3_avalanche(acc + acc_end);
  }
  uint64_t acc[8] = {P32_3, P64_1, P64_2, P64_3, P64_4, P32_2, P64_5, P32_1};
  const size_t stripes_per_block = (192 - 64) / 8, block_len = 64 * stripes_per_block; /* 16, 1024 */
  size_t nb_blocks = (len - 1) / block_len;
  for (size_t n = 0; n < nb_blocks; n++) {
    for (size_t s = 0; s < stripes_per_block; s++) xxh3_accumulate_stripe(acc, in + n * block_len + 64 * s, kSecret + 8 * s);
    for (int i = 0; i < 8; i++) {
      uint64_t a = acc[i];
      a ^= a >> 47;
      a ^= rd64(kSecret + 192 - 64 + 8 * i);
      a *= P32_1;
      acc[i] = a;
    }
  }
  size_t nb_stripes = ((len - 1) - block_len * nb_blocks) / 64;
  for (size_t s = 0; s < nb_stripes; s++) xxh3_accumulate_stripe(acc, in + nb_blocks * block_len + 64 * s, kSecret + 8 * s);
  xxh3_accumulate_stripe(acc, in + len - 64, kSecret + 192 - 64 - 7);
  uint64_t r = (uint64_t)len * P64_1;
  for (int i = 0; i < 4; i++)
    r += mul128_fold64(acc[2 * i] ^ rd64(kSecret + 11 + 16 * i), acc[2 * i + 1] ^ rd64(kSecret + 11 + 16 * i + 8));
  return xxh3_avalanche(r);
}

/* table/format.cc:436-509 */
uint32_t orc_block_checksum(uint32_t type, const void* data, size_t n, uint8_t last_byte) {
  if (type == ORC_CKSUM_CRC32C) return orc_crc32c_mask(orc_crc32c_extend(orc_crc32c_value(data, n), &last_byte, 1));
  if (type == ORC_CKSUM_XXH3) return (uint32_t)orc_xxh3_64(data, n) ^ (uint32_t)last_byte * 0x6b9083d9u;
  return 0;
}
uint32_t orc_checksum(uint32_t type, const void* data, size_t n) {
  const uint8_t* p = (const uint8_t*)data;
  if (type == ORC_CKSUM_CRC32C) return orc_crc32c_mask(orc_crc32c_value(data, n));
  if (type == ORC_CKSUM_XXH3) return n == 0 ? 0 : ((uint32_t)orc_xxh3_64(p, n - 1) ^ (uint32_t)p[n - 1] * 0x6b9083d9u);
  return 0;
}

/* ------------------------------------------------------------------ internal keys (db/dbformat.h:99-178,1057-1097) */
static uint64_t trailer_of(const uint8_t* ikey, size_t n) { return rd64(ikey + n - 8); }
static int ukey_cmp(const uint8_t* a, size_t an, const uint8_t* b, size_t bn) {
  size_t m = an < bn ? an : bn;
  int r = m ? memcmp(a, b, m) : 0;
  if (r) return r;
  return an < bn ? -1 : an > bn;
}
int orc_internal_key_less(const uint8_t* a, size_t an, const uint8_t* b, size_t bn) {
  int r = ukey_cmp(a, an - 8, b, bn - 8);
  if (r) return r < 0;
  return trailer_of(a, an) > trailer_of(b, bn); /* newer (larger seq) first */
}

/* ------------------------------------------------------------------ SST reader
 * footer table/format.cc:262-345; block trailer block_fetcher.cc:32-40; entries block.cc:37-64,617-665 */
typedef struct sst {
  const uint8_t* d;
  size_t len;
  uint32_t cksum_type, fv;
  uint64_t index_off, index_size, meta_off, meta_size;
  /* decoded index: data block handles */
  uint64_t* boff;
  uint64_t* bsize;
  size_t nblocks;
} sst;
#define SST_MAGIC 0x88e241b785f4cff7ull
/* BlockFetcher::ReadBlockContents + UncompressBlockData (table/block_fetcher.cc:211, table/format.cc:511): the checksum covers the stored
 * bytes and the type byte; a kZlibCompression block (type 2) is  varint32 uncompressed size | raw deflate stream  (Zlib_Uncompress,
 * util/compression.h:834-924, window_bits -14, compress_format_version 2) and is inflated with zlib itself -- the oracle is test
 * infrastructure.  *payload / *psize: the uncompressed block; *owned: malloc'ed copy the caller frees (NULL for a stored block). */
static int sst_read_block(const sst* s, uint64_t off, uint64_t size, const uint8_t** payload, uint64_t* psize, uint8_t** owned) {
  *owned = NULL;
  if (off + size + 5 > s->len) FAIL(-2, "block handle out of range");
  uint8_t ctype = s->d[off + size];
  uint32_t want = rd32(s->d + off + size + 1);
  uint32_t got = orc_block_checksum(s->cksum_type, s->d + off, size, ctype);
  if (s->cksum_type != ORC_CKSUM_NONE && want != got) FAIL(-4, "block checksum mismatch at %llu", (unsigned long long)off);
  if (ctype == 0) {
    *payload = s->d + off;
    *psize = size;
    return 0;
  }
  if (ctype != 2) FAIL(-3, "compressed block (type %u) not supported", ctype);
  uint64_t u = 0;
  const uint8_t* p = get_varint(s->d + off, s->d + off + size, &u);
  if (!p || u > (1ull << 31)) FAIL(-5, "bad uncompressed size of a zlib block");
  uint8_t* out = (uint8_t*)malloc(u ? u : 1);
  z_stream z;
  memset(&z, 0, sizeof z);
  if (inflateInit2(&z, -14) != Z_OK) {
    free(out);
    FAIL(-5, "inflateInit2 failed");
  }
  z.next_in = (Bytef*)p;
  z.avail_in = (uInt)(s->d + off + size - p);
  z.next_out = out;
  z.avail_out = (uInt)u;
  int st = inflate(&z, Z_FINISH);
  uint64_t produced = (uint64_t)z.total_out;
  inflateEnd(&z);
  if (st != Z_STREAM_END || produced != u) {
    free(out);
    FAIL(-5, "zlib block does not inflate to its announced size");
  }
  *payload = out;
  *psize = u;
  *owned = out;
  return 0;
}
/* iterate entries of one block payload; cb gets the fully rebuilt key. value_delta: index blocks (fv>=4). */
typedef int (*entry_cb)(void* ctx, const uint8_t* key, size_t klen, const uint8_t* val, size_t vlen, uint32_t shared);
static int block_foreach(const uint8_t* blk, size_t size, int value_delta, entry_cb cb, void* ctx) {
  if (size < 4) FAIL(-5, "block too small");
  uint32_t nr = rd32(blk + size - 4) & 0x7fffffffu;
  if ((uint64_t)nr * 4 + 4 > size) FAIL(-5, "bad restart count");
  const uint8_t *p = blk, *end = blk + size - 4 - 4 * (size_t)nr;
  buf key = {0};
  int rc = 0;
  while (p < end) {
    uint64_t shared, non_shared, vlen = 0;
    if (!(p = get_varint(p, end, &shared)) || !(p = get_varint(p, end, &non_shared))) {
      rc = -5;
      break;
    }
    if (!value_delta && !(p = get_varint(p, end, &vlen))) {
      rc = -5;
      break;
    }
    if (shared > key.n || p + non_shared > end) {
      rc = -5;
      break;
    }
    key.n = shared;
    buf_put(&key, p, non_shared);
    p += non_shared;
    if (value_delta) { /* IndexValue: varint64 offset, varint64 size | varsigned64 delta (table/format.cc:102-118) */
      const uint8_t* q = p;
      uint64_t t;
      if (shared == 0) {
        if (!(q = get_varint(q, end, &t)) || !(q = get_varint(q, end, &t))) {
          rc = -5;
          break;
        }
      } else if (!(q = get_varint(q, end, &t))) {
        rc = -5;
        break;
      }
      vlen = (uint64_t)(q - p);
    }
    if (p + vlen > end) {
      rc = -5;
      break;
    }
    if ((rc = cb(ctx, key.p, key.n, p, vlen, (uint32_t)shared)) != 0) break;
    p += vlen;
  }
  buf_free(&key);
  if (rc == -5) FAIL(-5, "corrupt block entry");
  return rc;
}
typedef struct idx_ctx {
  sst* s;
  uint64_t prev_off, prev_size;
  size_t cap;
} idx_ctx;
static int index_cb(void* vctx, const uint8_t* key, size_t klen, const uint8_t* val, size_t vlen, uint32_t shared) {
  (void)key;
  (void)klen;
  idx_ctx* c = (idx_ctx*)vctx;
  uint64_t off = 0, size = 0, t = 0;
  const uint8_t* end = val + vlen;
  if (shared == 0 || c->s->fv < 4) { /* before format_version 4 every index value is a whole BlockHandle */
    val = get_varint(val, end, &off);
    get_varint(val, end, &size);
  } else {
    get_varint(val, end, &t);
    int64_t delta = (int64_t)(t >> 1) ^ -(int64_t)(t & 1);
    size = c->prev_size + (uint64_t)delta;
    off = c->prev_off + c->prev_size + 5;
  }
  sst* s = c->s;
  if (s->nblocks == c->cap) {
    c->cap = c->cap ? c->cap * 2 : 64;
    s->boff = (uint64_t*)realloc(s->boff, c->cap * 8);
    s->bsize = (uint64_t*)realloc(s->bsize, c->cap * 8);
  }
  s->boff[s->nblocks] = off;
  s->bsize[s->nblocks] = size;
  s->nblocks++;
  c->prev_off = off;
  c->prev_size = size;
  return 0;
}
static void sst_close(sst* s) {
  free(s->boff);
  free(s->bsize);
  s->boff = s->bsize = NULL;
}
static int sst_open(sst* s, const uint8_t* d, size_t len) {
  memset(s, 0, sizeof *s);
  s->d = d;
  s->len = len;
  if (len < 53) FAIL(-1, "file too short");
  const uint8_t* f = d + len - 53;
  if (rd64(f + 45) != SST_MAGIC) FAIL(-1, "bad magic");
  s->cksum_type = f[0];
  s->fv = rd32(f + 41);
  const uint8_t *p = f + 1, *e = f + 41;
  if (!(p = get_varint(p, e, &s->meta_off)) || !(p = get_varint(p, e, &s->meta_size)) ||
      !(p = get_varint(p, e, &s->index_off)) || !(p = get_varint(p, e, &s->index_size)))
    FAIL(-1, "bad footer handles");
  const uint8_t* ib;
  uint64_t isz;
  uint8_t* iown;
  int rc = sst_read_block(s, s->index_off, s->index_size, &ib, &isz, &iown);
  if (rc) return rc;
  idx_ctx c = {s, 0, 0, 0};
  rc = block_foreach(ib, isz, s->fv >= 4, index_cb, &c);
  free(iown);
  if (rc) sst_close(s);
  return rc;
}
/* sequential entry iterator over all data blocks */
typedef struct sst_iter {
  sst s;
  size_t blk; /* next block to load */
  const uint8_t *p, *end;
  buf key;
  const uint8_t* val;
  size_t vlen;
  int valid, err;
  uint64_t yielded; /* entries produced so far */
  uint8_t* ublock;  /* the current block's inflated bytes (kZlibCompression), NULL for a stored block */
} sst_iter;
static void sst_iter_next(sst_iter* it) {
  for (;;) {
    if (it->p < it->end) {
      uint64_t shared, non_shared, vlen;
      const uint8_t* p = it->p;
      if (!(p = get_varint(p, it->end, &shared)) || !(p = get_varint(p, it->end, &non_shared)) ||
          !(p = get_varint(p, it->end, &vlen)) || shared > it->key.n || p + non_shared + vlen > it->end) {
        it->err = -5;
        it->valid = 0;
        snprintf(g_err, sizeof g_err, "corrupt data block entry");
        return;
      }
      it->key.n = shared;
      buf_put(&it->key, p, non_shared);
      it->val = p + non_shared;
      it->vlen = vlen;
      it->p = it->val + vlen;
      it->valid = 1;
      it->yielded++;
      return;
    }
    if (it->blk >= it->s.nblocks) {
      it->valid = 0;
      return;
    }
    uint64_t off = it->s.boff[it->blk], size = it->s.bsize[it->blk];
    it->blk++;
    free(it->ublock);
    it->ublock = NULL;
    const uint8_t* b;
    if ((it->err = sst_read_block(&it->s, off, size, &b, &size, &it->ublock)) != 0) {
      it->valid = 0;
      return;
    }
    if (size < 4) {
      it->err = -5;
      it->valid = 0;
      return;
    }
    uint32_t nr = rd32(b + size - 4) & 0x7fffffffu;
    it->p = b;
    it->end = b + size - 4 - 4 * (size_t)nr;
    it->key.n = 0;
  }
}
static int sst_iter_open(sst_iter* it, const uint8_t* d, size_t len) {
  memset(it, 0, sizeof *it);
  int rc = sst_open(&it->s, d, len);
  if (rc) return rc;
  sst_iter_next(it);
  return it->err;
}
static void sst_iter_close(sst_iter* it) {
  free(it->ublock);
  it->ublock = NULL;
  sst_close(&it->s);
  buf_free(&it->key);
}

int orc_sst_to_kvstream(const uint8_t* file, size_t len, uint8_t** out, size_t* out_len, uint64_t* num_entries) {
  sst_iter it;
  int rc = sst_iter_open(&it, file, len);
  if (rc) {
    sst_iter_close(&it);
    return rc;
  }
  buf o = {0};
  uint64_t n = 0;
  while (it.valid) {
    buf_u32(&o, (uint32_t)it.key.n);
    buf_u32(&o, (uint32_t)it.vlen);
    buf_put(&o, it.key.p, it.key.n);
    buf_put(&o, it.val, it.vlen);
    n++;
    sst_iter_next(&it);
  }
  rc = it.err;
  sst_iter_close(&it);
  if (rc) {
    buf_free(&o);
    return rc;
  }
  *out = o.p;
  *out_len = o.n;
  if (num_entries) *num_entries = n;
  return 0;
}

/* ------------------------------------------------------------------ merged input abstraction */
typedef struct input {
  int valid;
  const uint8_t *key, *val;
  size_t klen, vlen;
  void (*next)(struct input*);
  void* impl;
} input;

/* kv stream input */
typedef struct kvs_in {
  const uint8_t *p, *end;
} kvs_in;
static void kvs_next(input* in) {
  kvs_in* k = (kvs_in*)in->impl;
  if (k->p + 8 > k->end) {
    in->valid = 0;
    return;
  }
  uint32_t kl = rd32(k->p), vl = rd32(k->p + 4);
  in->key = k->p + 8;
  in->klen = kl;
  in->val = in->key + kl;
  in->vlen = vl;
  k->p = in->val + vl;
  in->valid = 1;
}

/* k-way merge: binary min-heap of child iterators, replace_top on advance.
 * table/compaction_merging_iterator.cc:239-320, util/heap.h:42-211 */
typedef struct merge_in {
  sst_iter* its;
  int n;
  int* heap; /* child indices */
  int hn;
  int err;
} merge_in;
static int child_less(merge_in* m, int a, int b) {
  sst_iter *x = &m->its[a], *y = &m->its[b];
  if (orc_internal_key_less(x->key.p, x->key.n, y->key.p, y->key.n)) return 1;
  if (orc_internal_key_less(y->key.p, y->key.n, x->key.p, x->key.n)) return 0;
  return a < b; /* identical internal keys: lower child index (newer L0 file) first */
}
static void heap_down(merge_in* m, int i) {
  for (;;) {
    int l = 2 * i + 1, r = l + 1, s = i;
    if (l < m->hn && child_less(m, m->heap[l], m->heap[s])) s = l;
    if (r < m->hn && child_less(m, m->heap[r], m->heap[s])) s = r;
    if (s == i) return;
    int t = m->heap[i];
    m->heap[i] = m->heap[s];
    m->heap[s] = t;
    i = s;
  }
}
static void merge_publish(input* in) {
  merge_in* m = (merge_in*)in->impl;
  if (m->hn == 0) {
    in->valid = 0;
    return;
  }
  sst_iter* t = &m->its[m->heap[0]];
  in->key = t->key.p;
  in->klen = t->key.n;
  in->val = t->val;
  in->vlen = t->vlen;
  in->valid = 1;
}
static void merge_next(input* in) {
  merge_in* m = (merge_in*)in->impl;
  sst_iter* t = &m->its[m->heap[0]];
  sst_iter_next(t);
  if (t->err) m->err = t->err;
  if (!t->valid) m->heap[0] = m->heap[--m->hn];
  heap_down(m, 0);
  merge_publish(in);
}

/* ClippingIterator (db/compaction/clipping_iterator.h:55-358) as ProcessKeyValueCompaction sets it up for a sub-compaction
 * (compaction_job.cc:1495-1519): bounds are (user key, kMaxSequenceNumber, kValueTypeForSeek), i.e. start <= user key < end */
typedef struct clip_in {
  input* base;
  const orc_params* p;
  uint64_t delivered;
} clip_in;
static void clip_publish(input* in) {
  clip_in* c = (clip_in*)in->impl;
  input* b = c->base;
  in->valid = b->valid;
  if (b->valid && c->p->has_range_end && ukey_cmp(b->key, b->klen - 8, c->p->range_end, c->p->range_end_len) >= 0) in->valid = 0;
  if (!in->valid) return;
  in->key = b->key;
  in->klen = b->klen;
  in->val = b->val;
  in->vlen = b->vlen;
  c->delivered++;
}
static void clip_next(input* in) {
  clip_in* c = (clip_in*)in->impl;
  c->base->next(c->base);
  clip_publish(in);
}
static void clip_seek_to_first(input* in) {
  clip_in* c = (clip_in*)in->impl;
  input* b = c->base;
  while (b->valid && c->p->has_range_start && ukey_cmp(b->key, b->klen - 8, c->p->range_start, c->p->range_start_len) < 0) b->next(b);
  clip_publish(in);
}

/* ------------------------------------------------------------------ CompactionIterator
 * db/compaction/compaction_iterator.cc: NextFromInput :475-1087, PrepareOutput :1274-1341,
 * findEarliestVisibleSnapshot :1343-1396, Next :…; restricted to kTypeValue / kTypeDeletion, no snapshot
 * checker, no merge operator, no range tombstones, no timestamps; compaction filter: the built-in
 * RemoveEmptyValueCompactionFilter only (SURVEY.md App. B). */
typedef struct citer {
  input* in;
  const orc_params* p;
  orc_stats* st;
  int visible_at_tip;
  uint64_t earliest_snapshot;
  int has_current_user_key;
  buf current_key; /* internal key being emitted (user key + trailer) */
  uint64_t cur_seq, cur_snap;
  int valid, at_next, err;
  uint64_t out_seq;
  uint8_t out_type;
  buf out_val;
  /* SingleDelete bookkeeping (compaction_iterator.h): */
  int has_outputted_key;          /* a record of the current user key went out (set in Next() :223-226, not in SeekToFirst) */
  int last_key_seq_zeroed;        /* PrepareOutput zeroed the sequence number of the last output (:1323-1324) */
  int clear_and_output_next_key;  /* the SingleDelete was kept for write-conflict checking: its Put follows with an empty value */
  uint64_t earliest_write_conflict_snapshot;
} citer;
static uint64_t find_earliest_visible_snapshot(const orc_params* p, uint64_t in, uint64_t* prev) {
  uint32_t lo = 0, hi = p->num_snapshots; /* lower_bound */
  while (lo < hi) {
    uint32_t mid = (lo + hi) / 2;
    if (p->snapshots[mid] < in) lo = mid + 1;
    else hi = mid;
  }
  *prev = lo == 0 ? 0 : p->snapshots[lo - 1];
  return lo < p->num_snapshots ? p->snapshots[lo] : ORC_MAX_SEQ;
}
static int key_not_exists_beyond_output_level(const citer* c) {
  /* Compaction::KeyNotExistsBeyondOutputLevel (db/compaction/compaction.cc:548-586): true at the bottommost level; on a compaction
   * worker false otherwise (:555-556) -- the deployment this repo targets; for a job the DB runs itself the deeper levels' file ranges
   * decide (key_not_exists_mode 1, used to replay the reference's own CompactionJob tests). */
  if (c->p->bottommost_level) return 1;
  if (c->p->key_not_exists_mode != 1) return 0;
  const uint8_t* uk = c->current_key.p;
  size_t un = c->current_key.n - 8;
  for (uint32_t i = 0; i < c->p->num_deeper_files; i++) {
    const orc_grandparent* f = &c->p->deeper_files[i];
    if (ukey_cmp(uk, un, f->largest, f->largest_len) <= 0 && ukey_cmp(uk, un, f->smallest, f->smallest_len) >= 0) return 0;
  }
  return 1;
}
static void citer_set_trailer(citer* c, uint64_t seq, uint8_t type) {
  uint64_t t = (seq << 8) | type;
  memcpy(c->current_key.p + c->current_key.n - 8, &t, 8);
}
static void citer_next_from_input(citer* c) {
  input* in = c->in;
  c->at_next = 0;
  c->valid = 0;
  while (!c->valid && in->valid) {
    c->st->num_input_records++;
    if (in->klen < 8) {
      c->err = -6;
      snprintf(g_err, sizeof g_err, "internal key shorter than 8 bytes");
      return;
    }
    uint64_t tr = trailer_of(in->key, in->klen), seq = tr >> 8;
    uint8_t type = (uint8_t)(tr & 0xff);
    size_t ulen = in->klen - 8;
    if (type == ORC_TYPE_DELETION || type == ORC_TYPE_SINGLE_DELETION) c->st->num_input_deletion_records++;
    c->st->total_input_raw_key_bytes += in->klen;
    c->st->total_input_raw_value_bytes += in->vlen;
    if (type != ORC_TYPE_VALUE && type != ORC_TYPE_DELETION && type != ORC_TYPE_SINGLE_DELETION) {
      c->err = -7;
      snprintf(g_err, sizeof g_err, "value type %u outside the restated rule set", type);
      return;
    }
    int filtered = 0; /* the compaction filter removed this entry: tombstone without a value (:385-391) */
    int same = c->has_current_user_key && c->current_key.n - 8 == ulen &&
               memcmp(c->current_key.p, in->key, ulen) == 0;
    if (!same) { /* :538-588 first occurrence of this user key */
      c->current_key.n = 0;
      buf_put(&c->current_key, in->key, in->klen);
      c->cur_seq = ORC_MAX_SEQ;
      c->cur_snap = 0;
      c->has_current_user_key = 1;
      c->has_outputted_key = 0; /* :578-580 */
      c->last_key_seq_zeroed = 0;
      /* :579-584 the filter sees the first (newest) committed version of a user key, kTypeValue only (:236-239);
       * Decision::kRemove turns it into a tombstone with no value (:385-391) */
      int remove = 0;
      if (type == ORC_TYPE_VALUE) {
        if (c->p->compaction_filter == ORC_FILTER_REMOVE_EMPTY_VALUE) remove = in->vlen == 0;
        else if (c->p->compaction_filter == ORC_FILTER_TTL && c->p->ttl > 0 && in->vlen >= 4) {
          /* DBWithTTLImpl::IsStale: the last four value bytes are the write time (fixed32), stale iff ts + ttl < now */
          const uint8_t* t = in->val + in->vlen - 4;
          int64_t ts = (int64_t)((uint32_t)t[0] | (uint32_t)t[1] << 8 | (uint32_t)t[2] << 16 | (uint32_t)t[3] << 24);
          remove = ts + c->p->ttl < c->p->now;
        }
      }
      if (remove) {
        filtered = 1;
        type = ORC_TYPE_DELETION;
        citer_set_trailer(c, seq, type);
        c->st->num_record_drop_user++;
      }
    } else { /* :589-611 */
      citer_set_trailer(c, seq, type);
    }
    c->out_seq = seq;
    c->out_type = type;
    c->out_val.n = 0;
    if (!filtered) buf_put(&c->out_val, in->val, in->vlen);
    /* :619-629 */
    uint64_t last_snapshot = c->cur_snap, prev_snapshot = 0;
    c->cur_seq = seq;
    c->cur_snap = c->visible_at_tip ? c->earliest_snapshot : find_earliest_visible_snapshot(c->p, seq, &prev_snapshot);
    if (c->clear_and_output_next_key) { /* :635-661 the Put behind a SingleDelete that had to stay: keep it, without its value */
      if (type != ORC_TYPE_VALUE) {
        c->err = -9;
        snprintf(g_err, sizeof g_err, "unexpected type %u behind a kept SingleDelete", type);
        return;
      }
      c->out_val.n = 0;
      c->valid = 1;
      c->clear_and_output_next_key = 0;
    } else if (type == ORC_TYPE_SINGLE_DELETION) { /* :662-887 */
      in->next(in);
      int next_same = in->valid && in->klen >= 8 && in->klen - 8 == ulen && memcmp(in->key, c->current_key.p, ulen) == 0;
      if (next_same) {
        uint64_t ntr = trailer_of(in->key, in->klen), nseq = ntr >> 8;
        uint8_t ntype = (uint8_t)(ntr & 0xff);
        if (c->last_key_seq_zeroed) { /* :753-757 */
          c->st->num_records_replaced++;
          c->st->num_expired_deletion_records++;
          in->next(in);
        } else if (prev_snapshot == 0 || nseq > prev_snapshot) { /* the next key is in the SingleDelete's snapshot stripe */
          if (ntype == ORC_TYPE_SINGLE_DELETION) { /* :765-778 two in a row: drop the first */
            c->st->num_expired_deletion_records++;
          } else if (ntype == ORC_TYPE_DELETION) { /* :779-800 contract violation; enforce_single_del_contracts defaults to true */
            c->st->num_expired_deletion_records++;
            c->err = -10;
            snprintf(g_err, sizeof g_err, "SingleDelete and Delete on the same key");
            return;
          } else if (c->has_outputted_key || seq <= c->earliest_write_conflict_snapshot ||
                     (c->earliest_snapshot < c->earliest_write_conflict_snapshot && seq <= c->earliest_snapshot)) {
            c->st->num_records_replaced++; /* :803-829 the pair cancels out */
            c->st->num_expired_deletion_records++;
            in->next(in);
          } else { /* :830-846 keep the SingleDelete for write-conflict checking, its Put follows without a value */
            c->valid = 1;
            c->clear_and_output_next_key = 1;
          }
        } else { /* :847-853 the next version belongs to an older snapshot */
          c->valid = 1;
        }
      } else { /* :854-884 last version of this user key in the input */
        c->has_current_user_key = 0;
        if (seq <= c->earliest_snapshot && key_not_exists_beyond_output_level(c)) {
          c->st->num_expired_deletion_records++;
          if (!c->p->bottommost_level) c->st->num_optimized_del_drop_obsolete++;
        } else if (c->last_key_seq_zeroed) {
          c->st->num_records_replaced++;
          c->st->num_expired_deletion_records++;
        } else {
          c->valid = 1;
        }
      }
      if (c->valid) c->at_next = 1;
    } else if (last_snapshot == c->cur_snap || (last_snapshot > 0 && last_snapshot < c->cur_snap)) {
      c->st->num_records_replaced++; /* rule (A) :890-911 */
      in->next(in);
    } else if (type == ORC_TYPE_DELETION && seq <= c->earliest_snapshot && key_not_exists_beyond_output_level(c)) {
      c->st->num_expired_deletion_records++; /* :912-946 */
      if (!c->p->bottommost_level) c->st->num_optimized_del_drop_obsolete++;
      in->next(in);
    } else if (type == ORC_TYPE_DELETION && c->p->bottommost_level) { /* :947-990 */
      in->next(in);
      while (in->valid && in->klen - 8 == ulen && memcmp(in->key, c->current_key.p, ulen) == 0 &&
             (prev_snapshot == 0 || (trailer_of(in->key, in->klen) >> 8) > prev_snapshot))
        in->next(in);
      if (in->valid && in->klen - 8 == ulen && memcmp(in->key, c->current_key.p, ulen) == 0) {
        c->valid = 1;
        c->at_next = 1;
      }
    } else {
      c->valid = 1; /* kNewUserKey :1045-1068 (no range tombstones) */
    }
  }
}
static void citer_prepare_output(citer* c) { /* :1274-1341 */
  if (c->valid && c->p->bottommost_level && c->out_seq <= c->earliest_snapshot && c->out_type != ORC_TYPE_MERGE) {
    c->out_seq = 0;
    c->last_key_seq_zeroed = 1;
    citer_set_trailer(c, 0, c->out_type);
  }
}
static void citer_init(citer* c, input* in, const orc_params* p, orc_stats* st) {
  memset(c, 0, sizeof *c);
  c->in = in;
  c->p = p;
  c->st = st;
  c->visible_at_tip = p->num_snapshots == 0;
  c->earliest_snapshot = p->num_snapshots ? p->snapshots[0] : ORC_MAX_SEQ;
  c->earliest_write_conflict_snapshot = p->earliest_write_conflict_snapshot ? p->earliest_write_conflict_snapshot : ORC_MAX_SEQ;
  citer_next_from_input(c); /* SeekToFirst :199-203 */
  citer_prepare_output(c);
}
static void citer_next(citer* c) {
  if (!c->at_next) c->in->next(c->in);
  citer_next_from_input(c);
  if (c->valid) c->has_outputted_key = 1; /* Next() :223-226 */
  citer_prepare_output(c);
}
static void citer_free(citer* c) {
  buf_free(&c->current_key);
  buf_free(&c->out_val);
}

int orc_compaction_iterator(const orc_params* p, const uint8_t* kv, size_t kv_len, uint8_t** out, size_t* out_len,
                            orc_stats* stats) {
  kvs_in k = {kv, kv + kv_len};
  input in = {0};
  in.impl = &k;
  in.next = kvs_next;
  kvs_next(&in);
  orc_stats st = {0};
  citer c;
  citer_init(&c, &in, p, &st);
  buf o = {0};
  while (c.valid && !c.err) {
    buf_u32(&o, (uint32_t)c.current_key.n);
    buf_u32(&o, (uint32_t)c.out_val.n);
    buf_put(&o, c.current_key.p, c.current_key.n);
    buf_put(&o, c.out_val.p, c.out_val.n);
    st.num_output_records++;
    citer_next(&c);
  }
  int rc = c.err;
  citer_free(&c);
  if (rc) {
    buf_free(&o);
    return rc;
  }
  *out = o.p;
  *out_len = o.n;
  if (stats) *stats = st;
  return 0;
}

/* ------------------------------------------------------------------ BlockBuilder (table/block_based/block_builder.cc) */
typedef struct bbuilder {
  int restart_interval, value_delta;
  buf b;
  uint32_t* restarts;
  size_t nrestarts, rcap;
  int counter;
  buf last_key;
} bbuilder;
static void bb_reset(bbuilder* x) {
  x->b.n = 0;
  x->nrestarts = 1;
  x->restarts[0] = 0;
  x->counter = 0;
  x->last_key.n = 0;
}
static void bb_init(bbuilder* x, int restart_interval, int value_delta) {
  memset(x, 0, sizeof *x);
  x->restart_interval = restart_interval;
  x->value_delta = value_delta;
  x->rcap = 16;
  x->restarts = (uint32_t*)malloc(4 * x->rcap);
  bb_reset(x);
}
static void bb_free(bbuilder* x) {
  buf_free(&x->b);
  buf_free(&x->last_key);
  free(x->restarts);
}
static int bb_empty(const bbuilder* x) { return x->b.n == 0; }
static size_t bb_current_size(const bbuilder* x) { return x->b.n + 4 * x->nrestarts + 4; } /* estimate_ :97,251 */
static size_t bb_size_after(const bbuilder* x, size_t klen, size_t vlen) { /* EstimateSizeAfterKV :97-126 (data blocks) */
  size_t e = bb_current_size(x) + klen + vlen;
  if (x->counter >= x->restart_interval) e += 4;
  e += 4;
  e += (size_t)varint_len(klen);
  e += (size_t)varint_len(vlen);
  return e;
}
static void bb_add(bbuilder* x, const uint8_t* key, size_t klen, const uint8_t* val, size_t vlen, const uint8_t* dval,
                   size_t dvlen) { /* AddWithLastKeyImpl :189-253 */
  size_t shared = 0;
  if (x->counter >= x->restart_interval) {
    if (x->nrestarts == x->rcap) {
      x->rcap *= 2;
      x->restarts = (uint32_t*)realloc(x->restarts, 4 * x->rcap);
    }
    x->restarts[x->nrestarts++] = (uint32_t)x->b.n;
    x->counter = 0;
  } else {
    size_t m = klen < x->last_key.n ? klen : x->last_key.n;
    while (shared < m && key[shared] == x->last_key.p[shared]) shared++;
  }
  buf_varint(&x->b, shared);
  buf_varint(&x->b, klen - shared);
  if (!x->value_delta) buf_varint(&x->b, vlen);
  buf_put(&x->b, key + shared, klen - shared);
  if (shared != 0 && x->value_delta) buf_put(&x->b, dval, dvlen);
  else buf_put(&x->b, val, vlen);
  x->last_key.n = 0;
  buf_put(&x->last_key, key, klen);
  x->counter++;
}
static void bb_finish(bbuilder* x) { /* Finish :128-149 */
  for (size_t i = 0; i < x->nrestarts; i++) buf_u32(&x->b, x->restarts[i]);
  buf_u32(&x->b, (uint32_t)x->nrestarts);
}

/* BytewiseComparator::FindShortestSeparator (util/comparator.cc:42-91) on user keys, then
 * ShortenedIndexBuilder::FindShortestInternalKeySeparator (table/block_based/index_builder.cc:77-94).
 * `start` is an internal key in a buffer with room for start_len bytes; returns the new length. */
size_t orc_shortest_separator(uint8_t* start, size_t start_len, const uint8_t* limit, size_t limit_len) {
  size_t us = start_len - 8, ul = limit_len - 8;
  uint8_t* tmp = (uint8_t*)malloc(us + 8);
  memcpy(tmp, start, us);
  size_t tn = us;
  size_t minl = us < ul ? us : ul, d = 0;
  while (d < minl && tmp[d] == limit[d]) d++;
  if (d < minl) {
    uint8_t sb = tmp[d], lb = limit[d];
    if (sb < lb) {
      if (d < ul - 1 || sb + 1 < lb) {
        tmp[d]++;
        tn = d + 1;
      } else {
        d++;
        while (d < tn) {
          if (tmp[d] < 0xff) {
            tmp[d]++;
            tn = d + 1;
            break;
          }
          d++;
        }
      }
    }
  }
  size_t out_len = start_len;
  if (tn <= us && ukey_cmp(start, us, tmp, tn) < 0) {
    uint64_t tr = (ORC_MAX_SEQ << 8) | ORC_VALUE_TYPE_FOR_SEEK; /* PackSequenceAndType(kMaxSequenceNumber, kValueTypeForSeek) */
    memcpy(tmp + tn, &tr, 8);
    memcpy(start, tmp, tn + 8);
    out_len = tn + 8;
  }
  free(tmp);
  return out_len;
}

/* ------------------------------------------------------------------ table builder
 * table/block_based/block_based_table_builder.cc: Add :961-1071, Flush/WriteBlock :1073-1133,
 * WriteMaybeCompressedBlock :1277-1378, Finish :1921-1977; flush policy flush_block_policy.cc:37-69;
 * index builder index_builder.h:130-274; properties meta_blocks.cc:54-175; footer format.cc:211-259 */
/* ------------------------------------------------------------------ full Bloom filter block
 * Hash64 = XXPH3_64bits (util/hash.cc:81-88; util/xxph3.h is the frozen PREVIEW of XXH3: its short-input paths :1083-1138 and
 * 17..128-byte path :1640-1677 differ from the final XXH3 used for block checksums); seed 0, default secret (same 192 bytes). */
static uint64_t xxph_mul_fold(uint64_t a, uint64_t b) {
  __uint128_t m = (__uint128_t)a * b;
  return (uint64_t)m ^ (uint64_t)(m >> 64);
}
static uint64_t xxph_avalanche(uint64_t h) {
  h ^= h >> 37;
  h *= 0x165667B19E3779F9ull;
  h ^= h >> 32;
  return h;
}
static uint64_t xxph_mix16(const uint8_t* in, const uint8_t* sec) { return xxph_mul_fold(rd64(in) ^ rd64(sec), rd64(in + 8) ^ rd64(sec + 8)); }
int orc_xxph3_64(const uint8_t* in, size_t len, uint64_t* out) {
  if (len > 128) return -1; /* longer inputs take the striped long-hash loop: not restated (user keys here are short) */
  if (len > 16) {
    uint64_t acc = (uint64_t)len * 0x9E3779B185EBCA87ull;
    if (len > 32) {
      if (len > 64) {
        if (len > 96) {
          acc += xxph_mix16(in + 48, kSecret + 96);
          acc += xxph_mix16(in + len - 64, kSecret + 112);
        }
        acc += xxph_mix16(in + 32, kSecret + 64);
        acc += xxph_mix16(in + len - 48, kSecret + 80);
      }
      acc += xxph_mix16(in + 16, kSecret + 32);
      acc += xxph_mix16(in + len - 32, kSecret + 48);
    }
    acc += xxph_mix16(in, kSecret);
    acc += xxph_mix16(in + len - 16, kSecret + 16);
    *out = xxph_avalanche(acc);
  } else if (len > 8) {
    uint64_t lo = rd64(in) ^ rd64(kSecret), hi = rd64(in + len - 8) ^ rd64(kSecret + 8);
    *out = xxph_avalanche((uint64_t)len + (lo + hi) + xxph_mul_fold(lo, hi));
  } else if (len >= 4) {
    uint64_t in64 = (uint64_t)rd32(in) | ((uint64_t)rd32(in + len - 4) << 32);
    uint64_t keyed = in64 ^ rd64(kSecret);
    uint64_t mix = (uint64_t)len + ((keyed ^ (keyed >> 51)) * 0x9E3779B1ull);
    *out = xxph_avalanche((mix ^ (mix >> 47)) * 0xC2B2AE3D27D4EB4Full);
  } else if (len) {
    uint32_t comb = (uint32_t)in[0] | ((uint32_t)in[len >> 1] << 8) | ((uint32_t)in[len - 1] << 16) | ((uint32_t)len << 24);
    *out = xxph_avalanche(((uint64_t)comb ^ (uint64_t)rd32(kSecret)) * 0x9E3779B185EBCA87ull);
  } else {
    *out = xxph_mul_fold(rd64(kSecret), 0xC2B2AE3D27D4EB4Full); /* RocksDB's change to the preview: hash of the seed */
  }
  return 0;
}
/* FastLocalBloomImpl::ChooseNumProbes (util/bloom_impl.h:156-198) */
static int bloom_num_probes(int mb) {
  static const int lim[] = {2080, 3580, 5100, 6640, 8300, 10070, 11720, 14001, 16050, 18300, 22001, 25501};
  for (int i = 0; i < 12; i++)
    if (mb <= lim[i]) return i + 1;
  if (mb > 50000) return 24;
  return (mb - 1) / 2000 - 1;
}
/* FastLocalBloomBitsBuilder::Finish / CalculateSpace / AddAllEntries (filter_policy.cc:326-424,462-506) +
 * FastLocalBloomImpl::AddHash (bloom_impl.h:200-214): filter bytes incl. the 5 metadata bytes; caller frees */
uint8_t* orc_bloom_build(const uint64_t* hashes, size_t n, uint32_t millibits, size_t* out_len) {
  uint64_t raw = ((uint64_t)n * millibits + 7999) / 8000;
  if (raw >= 0xffffffc0ull) raw = 0xffffffc0ull;
  uint32_t len = (uint32_t)((raw + 63) & ~63ull);
  uint8_t* d = (uint8_t*)calloc((size_t)len + 5, 1);
  int probes = bloom_num_probes((int)millibits);
  for (size_t i = 0; i < n && len; i++) {
    uint32_t h1 = (uint32_t)hashes[i], h = (uint32_t)(hashes[i] >> 32);
    uint8_t* line = d + ((size_t)(((uint64_t)h1 * (len >> 6)) >> 32) << 6); /* FastRange32 */
    for (int k = 0; k < probes; k++, h *= 0x9e3779b9u) {
      uint32_t bit = h >> (32 - 9);
      line[bit >> 3] |= (uint8_t)(1u << (bit & 7));
    }
  }
  d[len] = 0xff; /* marker: newer Bloom implementations */
  d[len + 1] = 0; /* sub-implementation: FastLocalBloom */
  d[len + 2] = (uint8_t)probes;
  *out_len = (size_t)len + 5;
  return d;
}

typedef struct tbuilder {
  uint64_t* fhash; /* XXPH3FilterBitsBuilder::hash_entries_ (filter_policy.cc:73-92): consecutive duplicates are dropped */
  size_t fhash_n, fhash_cap;
  const orc_params* p;
  buf file;
  bbuilder data, idx_seq, idx_noseq;
  int sep_is_key_plus_seq;
  buf last_key; /* r->last_key */
  uint64_t pending_off, pending_size;
  int have_pending;
  uint64_t last_h_off, last_h_size;
  int have_last_handle;
  uint64_t num_entries, num_deletions, raw_key_size, raw_value_size, num_data_blocks, data_size;
  uint64_t file_number, file_creation_time;
  int filter_err;
} tbuilder;
static void tb_write_raw_block(tbuilder* t, const uint8_t* d, size_t n, uint64_t* off, uint64_t* size) {
  *off = t->file.n;
  *size = n;
  uint32_t ck = orc_block_checksum(t->p->checksum_type, d, n, 0);
  buf_put(&t->file, d, n);
  uint8_t tr[5] = {0};
  memcpy(tr + 1, &ck, 4);
  buf_put(&t->file, tr, 5);
}
static void tb_init(tbuilder* t, const orc_params* p, uint64_t file_number, uint64_t file_creation_time) {
  memset(t, 0, sizeof *t);
  t->p = p;
  bb_init(&t->data, (int)p->block_restart_interval, 0);
  bb_init(&t->idx_seq, (int)p->index_block_restart_interval, p->format_version >= 4);
  bb_init(&t->idx_noseq, (int)p->index_block_restart_interval, p->format_version >= 4);
  t->sep_is_key_plus_seq = p->format_version <= 2;
  t->file_number = file_number;
  t->file_creation_time = file_creation_time;
}
static void tb_free(tbuilder* t) {
  free(t->fhash);
  buf_free(&t->file);
  buf_free(&t->last_key);
  bb_free(&t->data);
  bb_free(&t->idx_seq);
  bb_free(&t->idx_noseq);
}
static void tb_add_index_entry(tbuilder* t, const uint8_t* next_key, size_t next_len) { /* index_builder.h:165-233 */
  buf sep = {0};
  buf_put(&sep, t->last_key.p, t->last_key.n);
  if (next_key) {
    sep.n = orc_shortest_separator(sep.p, sep.n, next_key, next_len);
    if (!t->sep_is_key_plus_seq && ukey_cmp(t->last_key.p, t->last_key.n - 8, next_key, next_len - 8) == 0)
      t->sep_is_key_plus_seq = 1;
  }
  uint8_t enc[20], denc[10];
  int en = orc_put_varint64(enc, t->pending_off);
  en += orc_put_varint64(enc + en, t->pending_size);
  int dn = 0;
  if (t->have_last_handle) dn = orc_put_varint64(denc, zigzag_enc((int64_t)(t->pending_size - t->last_h_size)));
  t->last_h_off = t->pending_off;
  t->last_h_size = t->pending_size;
  t->have_last_handle = 1;
  bb_add(&t->idx_seq, sep.p, sep.n, enc, (size_t)en, denc, (size_t)dn);
  if (!t->sep_is_key_plus_seq) bb_add(&t->idx_noseq, sep.p, sep.n - 8, enc, (size_t)en, denc, (size_t)dn);
  buf_free(&sep);
}
static void tb_flush(tbuilder* t) {
  if (bb_empty(&t->data)) return;
  bb_finish(&t->data);
  tb_write_raw_block(t, t->data.b.p, t->data.b.n, &t->pending_off, &t->pending_size);
  t->have_pending = 1;
  bb_reset(&t->data);
  t->data_size = t->file.n;
  t->num_data_blocks++;
}
static void tb_add(tbuilder* t, const uint8_t* key, size_t klen, const uint8_t* val, size_t vlen) {
  if (!bb_empty(&t->data)) { /* FlushBlockBySizePolicy::Update */
    size_t cur = bb_current_size(&t->data);
    size_t limit = ((size_t)t->p->block_size * (100 - t->p->block_size_deviation) + 99) / 100;
    int flush = cur >= t->p->block_size;
    if (!flush && limit != 0) flush = bb_size_after(&t->data, klen, vlen) > t->p->block_size && cur > limit;
    if (flush) {
      tb_flush(t);
      tb_add_index_entry(t, key, klen);
      t->have_pending = 0;
    }
  }
  bb_add(&t->data, key, klen, val, vlen, NULL, 0);
  t->last_key.n = 0;
  buf_put(&t->last_key, key, klen);
  if (t->p->bloom_millibits_per_key) { /* BlockBasedTableBuilder::Add :1010-1014 -> FullFilterBlockBuilder::Add(user key) */
    uint64_t h = 0;
    if (orc_xxph3_64(key, klen - 8, &h)) t->filter_err = 1;
    if (t->fhash_n == 0 || t->fhash[t->fhash_n - 1] != h) {
      if (t->fhash_n == t->fhash_cap) {
        t->fhash_cap = t->fhash_cap ? 2 * t->fhash_cap : 1024;
        t->fhash = (uint64_t*)realloc(t->fhash, 8 * t->fhash_cap);
      }
      t->fhash[t->fhash_n++] = h;
    }
  }
  t->num_entries++;
  t->raw_key_size += klen;
  t->raw_value_size += vlen;
  uint8_t type = key[klen - 8];
  if (type == ORC_TYPE_DELETION || type == ORC_TYPE_SINGLE_DELETION) t->num_deletions++;
}
typedef struct prop {
  const char* name;
  buf val;
} prop;
static int prop_cmp(const void* a, const void* b) { return strcmp(((const prop*)a)->name, ((const prop*)b)->name); }
static void prop_u64(prop* ps, int* n, const char* name, uint64_t v) {
  ps[*n].name = name;
  memset(&ps[*n].val, 0, sizeof(buf));
  buf_varint(&ps[*n].val, v);
  (*n)++;
}
static void prop_str(prop* ps, int* n, const char* name, const char* s, size_t len) {
  ps[*n].name = name;
  memset(&ps[*n].val, 0, sizeof(buf));
  buf_put(&ps[*n].val, s, len);
  (*n)++;
}
static void tb_finish(tbuilder* t) {
  int empty = bb_empty(&t->data);
  tb_flush(t);
  if (!empty) tb_add_index_entry(t, NULL, 0);
  uint64_t tail_start = t->file.n;
  /* filter block first (Finish :1958 WriteFilterBlock :1488-1538): uncompressed, ordinary trailer */
  uint64_t foff = 0, fsize = 0, filter_entries = t->fhash_n;
  if (t->fhash_n) {
    size_t flen = 0;
    uint8_t* fd = orc_bloom_build(t->fhash, t->fhash_n, t->p->bloom_millibits_per_key, &flen);
    tb_write_raw_block(t, fd, flen, &foff, &fsize);
    free(fd);
  }
  /* index block (WriteIndexBlock :1540-1603; goes through WriteBlock, uncompressed here) */
  bbuilder* ib = t->sep_is_key_plus_seq ? &t->idx_seq : &t->idx_noseq;
  bb_finish(ib);
  uint64_t ioff, isize, poff, psize, moff, msize;
  tb_write_raw_block(t, ib->b.p, ib->b.n, &ioff, &isize);
  /* properties (WritePropertiesBlock :1605-1716, PropertyBlockBuilder meta_blocks.cc:79-175,
   * BlockBasedTablePropertiesCollector block_based_table_builder.cc:237-246) */
  const orc_params* p = t->p;
  prop ps[48];
  int n = 0;
  static const char kCompressionOpts[] =
      "window_bits=-14; level=32767; strategy=0; max_dict_bytes=0; zstd_max_train_bytes=0; enabled=0; "
      "max_dict_buffer_bytes=0; use_zstd_dict_trainer=1; ";
  uint32_t index_type = 0;
  prop_str(ps, &n, "rocksdb.block.based.table.index.type", (const char*)&index_type, 4);
  prop_str(ps, &n, "rocksdb.block.based.table.prefix.filtering", "0", 1);
  prop_str(ps, &n, "rocksdb.block.based.table.whole.key.filtering", "1", 1);
  prop_u64(ps, &n, "rocksdb.column.family.id", p->column_family_id);
  if (p->column_family_name && *p->column_family_name)
    prop_str(ps, &n, "rocksdb.column.family.name", p->column_family_name, strlen(p->column_family_name));
  prop_str(ps, &n, "rocksdb.comparator", "leveldb.BytewiseComparator", 26);
  prop_str(ps, &n, "rocksdb.compression", "NoCompression", 13);
  prop_str(ps, &n, "rocksdb.compression_options", kCompressionOpts, sizeof kCompressionOpts - 1);
  if (p->db_id && *p->db_id) prop_str(ps, &n, "rocksdb.creating.db.identity", p->db_id, strlen(p->db_id));
  if (p->db_host_id && *p->db_host_id)
    prop_str(ps, &n, "rocksdb.creating.host.identity", p->db_host_id, strlen(p->db_host_id));
  if (p->db_session_id && *p->db_session_id)
    prop_str(ps, &n, "rocksdb.creating.session.identity", p->db_session_id, strlen(p->db_session_id));
  prop_u64(ps, &n, "rocksdb.creation.time", p->creation_time);
  prop_u64(ps, &n, "rocksdb.data.size", t->data_size);
  prop_u64(ps, &n, "rocksdb.deleted.keys", t->num_deletions);
  if (t->file_creation_time > 0) prop_u64(ps, &n, "rocksdb.file.creation.time", t->file_creation_time);
  if (p->bloom_millibits_per_key) prop_str(ps, &n, "rocksdb.filter.policy", "bloomfilter", 11); /* props.filter_policy_name :1610 */
  prop_u64(ps, &n, "rocksdb.filter.size", fsize);
  prop_u64(ps, &n, "rocksdb.fixed.key.length", 0);
  prop_u64(ps, &n, "rocksdb.format.version", 0);
  prop_u64(ps, &n, "rocksdb.index.key.is.user.key", !t->sep_is_key_plus_seq);
  prop_u64(ps, &n, "rocksdb.index.size", isize + 5);
  prop_u64(ps, &n, "rocksdb.index.value.is.delta.encoded", p->format_version >= 4);
  prop_u64(ps, &n, "rocksdb.merge.operands", 0);
  prop_str(ps, &n, "rocksdb.merge.operator", "nullptr", 7);
  prop_u64(ps, &n, "rocksdb.num.data.blocks", t->num_data_blocks);
  prop_u64(ps, &n, "rocksdb.num.entries", t->num_entries);
  prop_u64(ps, &n, "rocksdb.num.filter_entries", filter_entries);
  prop_u64(ps, &n, "rocksdb.num.range-deletions", 0);
  prop_u64(ps, &n, "rocksdb.oldest.key.time", p->oldest_key_time);
  prop_u64(ps, &n, "rocksdb.original.file.number", t->file_number);
  prop_str(ps, &n, "rocksdb.prefix.extractor.name", "nullptr", 7);
  prop_str(ps, &n, "rocksdb.property.collectors", "[]", 2);
  prop_u64(ps, &n, "rocksdb.raw.key.size", t->raw_key_size);
  prop_u64(ps, &n, "rocksdb.raw.value.size", t->raw_value_size);
  prop_u64(ps, &n, "rocksdb.tail.start.offset", tail_start);
  qsort(ps, (size_t)n, sizeof(prop), prop_cmp);
  bbuilder pb;
  bb_init(&pb, 0x7fffffff, 0);
  for (int i = 0; i < n; i++) {
    bb_add(&pb, (const uint8_t*)ps[i].name, strlen(ps[i].name), ps[i].val.p, ps[i].val.n, NULL, 0);
    buf_free(&ps[i].val);
  }
  bb_finish(&pb);
  tb_write_raw_block(t, pb.b.p, pb.b.n, &poff, &psize);
  bb_free(&pb);
  /* metaindex (MetaIndexBuilder meta_blocks.cc:35-49) */
  bbuilder mb;
  bb_init(&mb, 1, 0);
  uint8_t h[20];
  int hn;
  if (fsize) { /* "fullfilter." + filter_policy->CompatibilityName() :1532-1536; metaindex keys are sorted */
    hn = orc_put_varint64(h, foff);
    hn += orc_put_varint64(h + hn, fsize);
    bb_add(&mb, (const uint8_t*)"fullfilter.rocksdb.BuiltinBloomFilter", 37, h, (size_t)hn, NULL, 0);
  }
  hn = orc_put_varint64(h, poff);
  hn += orc_put_varint64(h + hn, psize);
  bb_add(&mb, (const uint8_t*)"rocksdb.properties", 18, h, (size_t)hn, NULL, 0);
  bb_finish(&mb);
  tb_write_raw_block(t, mb.b.p, mb.b.n, &moff, &msize);
  bb_free(&mb);
  /* footer (FooterBuilder::Build table/format.cc:211-259), format_version >= 1 */
  uint8_t f[53];
  memset(f, 0, sizeof f);
  f[0] = (uint8_t)p->checksum_type;
  int q = 1;
  q += orc_put_varint64(f + q, moff);
  q += orc_put_varint64(f + q, msize);
  q += orc_put_varint64(f + q, ioff);
  q += orc_put_varint64(f + q, isize);
  uint32_t fv = p->format_version;
  uint64_t magic = SST_MAGIC;
  memcpy(f + 41, &fv, 4);
  memcpy(f + 45, &magic, 8);
  buf_put(&t->file, f, 53);
}

int orc_build_sst(const orc_params* p, const uint8_t* kv, size_t kv_len, uint8_t** out, size_t* out_len) {
  tbuilder t;
  tb_init(&t, p, p->first_file_number, p->num_file_creation_times ? p->file_creation_times[0] : 0);
  const uint8_t *q = kv, *end = kv + kv_len;
  while (q + 8 <= end) {
    uint32_t kl = rd32(q), vl = rd32(q + 4);
    tb_add(&t, q + 8, kl, q + 8 + kl, vl);
    q += 8 + (size_t)kl + vl;
  }
  tb_finish(&t);
  *out = t.file.p;
  *out_len = t.file.n;
  t.file.p = NULL;
  tb_free(&t);
  return 0;
}

/* ------------------------------------------------------------------ whole job
 * CompactionJob::ProcessKeyValueCompaction compaction_job.cc:1390-1780 (loop :1643-1674),
 * CompactionOutputs::AddToOutput / ShouldStopBefore compaction_outputs.cc:231-427,
 * FileMetaData::UpdateBoundaries db/version_edit.cc:31-61 */
typedef struct out_file {
  uint8_t* data;
  uint64_t len;
  orc_file_meta meta;
} out_file;
struct orc_result {
  out_file* files;
  int nfiles, cap;
  orc_stats stats;
};
static void result_push(orc_result* r, tbuilder* t, orc_file_meta* m) {
  if (r->nfiles == r->cap) {
    r->cap = r->cap ? r->cap * 2 : 8;
    r->files = (out_file*)realloc(r->files, sizeof(out_file) * (size_t)r->cap);
  }
  m->file_size = t->file.n;
  m->num_entries = t->num_entries;
  m->num_deletions = t->num_deletions;
  m->raw_key_size = t->raw_key_size;
  m->raw_value_size = t->raw_value_size;
  m->num_data_blocks = t->num_data_blocks;
  out_file* f = &r->files[r->nfiles++];
  f->data = t->file.p;
  f->len = t->file.n;
  f->meta = *m;
  t->file.p = NULL;
  t->file.n = t->file.cap = 0;
}
static uint64_t fct_for(const orc_params* p, int file_idx) {
  if (!p->num_file_creation_times) return 0;
  uint32_t i = (uint32_t)file_idx < p->num_file_creation_times ? (uint32_t)file_idx : p->num_file_creation_times - 1;
  return p->file_creation_times[i];
}
/* ------------------------------------------------------------------ grandparent-aware cutting
 * CompactionOutputs::{UpdateGrandparentBoundaryInfo :133-187, GetCurrentKeyGrandparentOverlappedBytes :189-229,
 * ShouldStopBefore :231-354}; sstableKeyCompare (compaction.cc:28-43) reduces to a user-key compare here (no range
 * tombstone sentinels on the path). */
typedef struct gp_state {
  int being_gap, seen_key;
  size_t index, switched;
  uint64_t overlapped;
} gp_state;
static size_t gp_update(gp_state* g, const orc_params* p, const uint8_t* uk, size_t un) {
  size_t crossed = 0;
  const orc_grandparent* gp = p->grandparents;
  const size_t n = p->num_grandparents;
  while (g->index < n) {
    if (g->being_gap) {
      if (ukey_cmp(uk, un, gp[g->index].smallest, gp[g->index].smallest_len) < 0) break;
      if (g->seen_key) {
        crossed++;
        g->overlapped += gp[g->index].file_size;
        g->switched++;
      }
      g->being_gap = 0;
    } else {
      int c = ukey_cmp(uk, un, gp[g->index].largest, gp[g->index].largest_len);
      if (c < 0 || (c == 0 && (g->index == n - 1 ||
                               ukey_cmp(uk, un, gp[g->index + 1].smallest, gp[g->index + 1].smallest_len) < 0)))
        break;
      if (g->seen_key) {
        crossed++;
        g->switched++;
      }
      g->being_gap = 1;
      g->index++;
    }
  }
  if (!g->seen_key && !g->being_gap) { /* the first key sits inside a grandparent file */
    g->overlapped = gp[g->index].file_size;
    for (long i = (long)g->index - 1; i >= 0 && ukey_cmp(uk, un, gp[i].largest, gp[i].largest_len) == 0; i--)
      g->overlapped += gp[i].file_size;
  }
  g->seen_key = 1;
  return crossed;
}
static uint64_t gp_current_key_overlap(const gp_state* g, const orc_params* p, const uint8_t* uk, size_t un) {
  if (g->being_gap) return 0;
  const orc_grandparent* gp = p->grandparents;
  uint64_t b = gp[g->index].file_size;
  for (long i = (long)g->index - 1; i >= 0 && ukey_cmp(uk, un, gp[i].largest, gp[i].largest_len) == 0; i--) b += gp[i].file_size;
  return b;
}
static int should_stop_before(gp_state* g, const orc_params* p, const uint8_t* uk, size_t un, int have_builder,
                              uint64_t cur_file_size) {
  const uint64_t prev_overlapped = g->overlapped;
  size_t crossed = 0;
  if (p->output_level > 0 && p->num_grandparents) crossed = gp_update(g, p, uk, un);
  if (!have_builder) return 0;
  if (p->output_level == 0) return 0; /* :272 */
  if (cur_file_size >= p->max_output_file_size) return 1; /* :277 */
  if (crossed > 0) {
    if (g->overlapped + cur_file_size > p->max_compaction_bytes) return 1; /* :299 */
    const size_t skippable = g->being_gap ? 2 : 3;
    if (p->level_compaction_dynamic_file_size && crossed >= skippable &&
        g->overlapped - prev_overlapped > p->target_output_file_size / 8) /* :325-331 */
      return 1;
    size_t pct = g->switched * 5 < 40 ? g->switched * 5 : 40;
    if (p->level_compaction_dynamic_file_size &&
        cur_file_size >= ((p->target_output_file_size + 99) / 100) * (50 + pct)) /* :343-349 */
      return 1;
  }
  return 0;
}

/* Test hook: the output-file cut rules alone, over a key list and a caller-supplied size model.  The reference's own known-answer
 * tests for these rules (db/compaction/compaction_job_test.cc:1755-2150, CompactionJobDynamicFileSizeTest) run on mock tables whose
 * FileSize() is entries x constant (table/mock_table.cc:180), which a BlockBasedTable job cannot reproduce; this runs the same
 * should_stop_before / reset sequence as orc_compact with that size model.  cut_before[i] = 1: a new output file starts at key i. */
int orc_file_cut_sim(const orc_params* p, int n, const uint8_t* const* ukeys, const uint32_t* ulens, uint64_t bytes_per_entry,
                     uint8_t* cut_before) {
  gp_state gps = {1, 0, 0, 0, 0};
  int have_builder = 0;
  uint64_t in_file = 0;
  for (int i = 0; i < n; i++) {
    cut_before[i] = 0;
    if (should_stop_before(&gps, p, ukeys[i], ulens[i], have_builder, in_file * bytes_per_entry) && have_builder) {
      have_builder = 0;
      gps.switched = 0;
      gps.overlapped = p->num_grandparents ? gp_current_key_overlap(&gps, p, ukeys[i], ulens[i]) : 0;
    }
    if (!have_builder) {
      cut_before[i] = 1;
      have_builder = 1;
      in_file = 0;
    }
    in_file++;
  }
  return 0;
}

int orc_compact(const orc_params* p, int n_inputs, const uint8_t* const* inputs, const uint64_t* input_lens,
                orc_result** out) {
  merge_in m;
  memset(&m, 0, sizeof m);
  m.its = (sst_iter*)calloc((size_t)n_inputs, sizeof(sst_iter));
  m.heap = (int*)malloc(sizeof(int) * (size_t)(n_inputs ? n_inputs : 1));
  m.n = n_inputs;
  int rc = 0;
  for (int i = 0; i < n_inputs && !rc; i++) {
    rc = sst_iter_open(&m.its[i], inputs[i], input_lens[i]);
    if (!rc && m.its[i].valid) m.heap[m.hn++] = i;
  }
  orc_result* r = (orc_result*)calloc(1, sizeof *r);
  if (!rc) {
    for (int i = m.hn / 2 - 1; i >= 0; i--) heap_down(&m, i);
    input in = {0};
    in.impl = &m;
    in.next = merge_next;
    merge_publish(&in);
    const int clipped = p->has_range_start || p->has_range_end;
    clip_in clip = {&in, p, 0};
    input cin = {0};
    cin.impl = &clip;
    cin.next = clip_next;
    if (clipped) clip_seek_to_first(&cin);
    citer c;
    citer_init(&c, clipped ? &cin : &in, p, &r->stats);
    tbuilder t;
    int have_builder = 0, file_idx = 0;
    uint64_t cur_file_size = 0;
    orc_file_meta meta;
    gp_state gps = {1, 0, 0, 0, 0}; /* compaction_outputs.h:331-372 initial values */
    while (c.valid && !c.err && !m.err) {
      /* AddToOutput :356-384: ShouldStopBefore (no partitioner / TTL-file cut / round-robin), then the grandparent reset */
      if (should_stop_before(&gps, p, c.current_key.p, c.current_key.n - 8, have_builder, cur_file_size) && have_builder) {
        tb_finish(&t);
        result_push(r, &t, &meta);
        tb_free(&t);
        have_builder = 0;
        gps.switched = 0;
        gps.overlapped = p->num_grandparents ? gp_current_key_overlap(&gps, p, c.current_key.p, c.current_key.n - 8) : 0;
      }
      if (!have_builder) {
        tb_init(&t, p, p->first_file_number + (uint64_t)file_idx, fct_for(p, file_idx));
        memset(&meta, 0, sizeof meta);
        meta.file_number = t.file_number;
        meta.smallest_seqno = ORC_MAX_SEQ;
        file_idx++;
        have_builder = 1;
      }
      tb_add(&t, c.current_key.p, c.current_key.n, c.out_val.p, c.out_val.n);
      if (t.filter_err) {
        c.err = -8; /* filter key longer than the restated XXPH3 paths */
        break;
      }
      r->stats.num_output_records++;
      cur_file_size = t.file.n; /* EstimatedFileSize() == offset, builder :1997-2010 */
      size_t kl = c.current_key.n < 256 ? c.current_key.n : 256;
      if (meta.smallest_len == 0) {
        memcpy(meta.smallest, c.current_key.p, kl);
        meta.smallest_len = (uint32_t)c.current_key.n;
      }
      memcpy(meta.largest, c.current_key.p, kl);
      meta.largest_len = (uint32_t)c.current_key.n;
      if (c.out_seq < meta.smallest_seqno) meta.smallest_seqno = c.out_seq;
      if (c.out_seq > meta.largest_seqno) meta.largest_seqno = c.out_seq;
      citer_next(&c);
    }
    rc = c.err ? c.err : m.err;
    /* job-level num_input_records is the sum of the input files' entry counts
     * (UpdateCompactionInputStatsHelper, compaction_job.cc:2383-2396), not the iterator's own count */
    r->stats.num_input_records = 0;
    for (int i = 0; i < n_inputs; i++) r->stats.num_input_records += m.its[i].yielded;
    /* a sub-compaction's own count is what its CompactionIterator consumed (compaction_job.cc:1676-1683) */
    if (clipped) r->stats.num_input_records = clip.delivered;
    if (have_builder) {
      if (!rc) {
        tb_finish(&t);
        result_push(r, &t, &meta);
      }
      tb_free(&t);
    }
    citer_free(&c);
  }
  for (int i = 0; i < n_inputs; i++) sst_iter_close(&m.its[i]);
  free(m.its);
  free(m.heap);
  if (rc) {
    orc_result_free(r);
    return rc;
  }
  *out = r;
  return 0;
}
int orc_result_num_files(const orc_result* r) { return r->nfiles; }
const uint8_t* orc_result_file(const orc_result* r, int i, uint64_t* len) {
  *len = r->files[i].len;
  return r->files[i].data;
}
void orc_result_meta(const orc_result* r, int i, orc_file_meta* m) { *m = r->files[i].meta; }
void orc_result_stats(const orc_result* r, orc_stats* s) { *s = r->stats; }
void orc_result_free(orc_result* r) {
  if (!r) return;
  for (int i = 0; i < r->nfiles; i++) free(r->files[i].data);
  free(r->files);
  free(r);
}
