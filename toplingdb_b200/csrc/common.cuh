// toplingdb_b200/csrc/common.cuh — device-side building blocks shared by the decode / merge / encode kernels.
// sm_90a (H100).  Formats follow the reference (paths relative to the reference source tree):
//   internal key   db/dbformat.h:99-178        varints util/coding.h       block layout table/block_based/block_builder.cc:21-32
//   XXH3-64        util/xxhash.h:3644-5235     block checksum table/format.cc:436-509
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstddef>

namespace b200c {

// ---- error word (device) : first error wins per class, host maps to b200c_status ---------------------------
enum DevErr : uint32_t {
  kErrNone = 0,
  kErrCorruptBlock = 1u << 0,    // malformed entry / restart array / handle out of range
  kErrChecksum = 1u << 1,        // block checksum mismatch
  kErrKeyTooLong = 1u << 2,      // user key > 16 bytes
  kErrValueTooLong = 1u << 3,    // value >= 2^27 bytes
  kErrBadType = 1u << 4,         // value type outside {kTypeDeletion, kTypeValue}
  kErrCompressed = 1u << 5,      // block compression type != kNoCompression
  kErrKeyOrder = 1u << 6,        // input run not strictly sorted / partition invariant broken
  kErrBlockTooLong = 1u << 7,    // more entries in one output block than the encoder's window
  kErrInternal = 1u << 8,
  kErrCountMismatch = 1u << 9,   // entry count differs from rocksdb.num.entries
  kErrIrregularRestarts = 1u << 10,  // restart intervals of one block hold different numbers of entries
  kErrParanoid = 1u << 11,       // paranoid_file_checks: an output file does not read back as what was written
  kErrSingleDelContract = 1u << 12,  // a SingleDelete met a Delete of the same key in one snapshot stripe (enforce_single_del_contracts)
  kErrGroupTooLong = 1u << 13,   // a user key with a SingleDelete has more versions than the device walks serially
  kErrSdWriteConflict = 1u << 14,  // SingleDelete with an earliest_write_conflict_snapshot (transaction DB): not on the device
  kErrTooManyFiles = 1u << 15,   // the job cuts more output files than the encoder's file records hold (kMaxOutFiles)
  // not an error: some input entry is a kTypeSingleDeletion (the merge then keeps every user key's versions inside one tile)
  kFlagHasSingleDelete = 1u << 31,
};

constexpr int kMaxUserKey = 16;
constexpr uint32_t kMetaVlenBits = 27;
constexpr uint32_t kMetaVlenMask = (1u << kMetaVlenBits) - 1;
constexpr uint64_t kMaxSeq = (1ull << 56) - 1;
constexpr uint8_t kTypeDeletion = 0, kTypeValue = 1, kTypeSingleDeletion = 7;
// value types the device rule set covers (everything else: kErrBadType -> NOT_SUPPORTED)
__host__ __device__ __forceinline__ bool device_value_type(uint32_t t) { return t <= 1 || t == kTypeSingleDeletion; }
__host__ __device__ __forceinline__ bool is_deletion_type(uint32_t t) { return t == kTypeDeletion || t == kTypeSingleDeletion; }

__host__ __device__ __forceinline__ uint32_t make_meta(uint32_t ulen, uint32_t vlen) { return (ulen << kMetaVlenBits) | vlen; }
__host__ __device__ __forceinline__ uint32_t meta_ulen(uint32_t m) { return m >> kMetaVlenBits; }
__host__ __device__ __forceinline__ uint32_t meta_vlen(uint32_t m) { return m & kMetaVlenMask; }

// One sorted run / the merged stream, columnar in HBM.  hi/lo = first 16 user-key bytes as two big-endian
// integers (zero padded) so that bytewise user-key order == (hi, lo, ulen) order; tr = (seq << 8) | type.
struct KeyCols {
  const ulonglong2* pfx;  // .x = hi, .y = lo
  const uint64_t* tr;
  const uint64_t* vref;   // device address of the value bytes (inside the input file image)
  const uint32_t* meta;   // ulen << 27 | vlen
  uint64_t n;
};
struct KeyColsMut {
  ulonglong2* pfx;
  uint64_t* tr;
  uint64_t* vref;
  uint32_t* meta;
};

// ---- unaligned little-endian loads from generic (global or shared) memory ---------------------------------
__device__ __forceinline__ uint32_t ld_u32(const uint8_t* p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
__device__ __forceinline__ uint64_t ld_u64(const uint8_t* p) { return (uint64_t)ld_u32(p) | ((uint64_t)ld_u32(p + 4) << 32); }

__device__ __forceinline__ uint64_t ld_u64_aligned(const uint8_t* p) { return *reinterpret_cast<const uint64_t*>(p); }
// 8 bytes at ANY alignment from two naturally aligned 8-byte loads (global or shared).  May touch up to 7 bytes past p+8.
__device__ __forceinline__ uint64_t ld_u64_funnel(const uint8_t* p) {
  const uint32_t a = (uint32_t)((uintptr_t)p & 7);
  const uint64_t* q = reinterpret_cast<const uint64_t*>((uintptr_t)p - a);
  const uint64_t lo = q[0];
  if (a == 0) return lo;
  return (lo >> (8 * a)) | (q[1] << (64 - 8 * a));
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }

// varint32/64 decode; returns bytes consumed or 0 on malformed / overrun
__device__ __forceinline__ int get_varint(const uint8_t* p, const uint8_t* end, uint64_t* v) {
  uint64_t r = 0;
  int n = 0;
#pragma unroll 1
  for (int s = 0; s <= 63; s += 7) {
    if (p + n >= end) return 0;
    uint8_t c = p[n++];
    r |= (uint64_t)(c & 127) << s;
    if (c < 128) {
      *v = r;
      return n;
    }
  }
  return 0;
}
__host__ __device__ __forceinline__ int varint_len(uint64_t v) {
  int n = 1;
  while (v >= 128) {
    v >>= 7;
    n++;
  }
  return n;
}
// branch-free length of a varint32
__host__ __device__ __forceinline__ uint32_t varint_len32(uint32_t v) {
  return 1u + (v >= (1u << 7)) + (v >= (1u << 14)) + (v >= (1u << 21)) + (v >= (1u << 28));
}
__host__ __device__ __forceinline__ int put_varint(uint8_t* p, uint64_t v) {
  int n = 0;
  while (v >= 128) {
    p[n++] = (uint8_t)(v | 128);
    v >>= 7;
  }
  p[n++] = (uint8_t)v;
  return n;
}
// little-endian 32-bit store at any alignment (EncodeFixed32)
__device__ __forceinline__ void put_fixed32(uint8_t* p, uint32_t v) {
  p[0] = (uint8_t)v;
  p[1] = (uint8_t)(v >> 8);
  p[2] = (uint8_t)(v >> 16);
  p[3] = (uint8_t)(v >> 24);
}
// 5-byte block trailer behind a block's contents: compression type kNoCompression + checksum (WriteMaybeCompressedBlock,
// block_based_table_builder.cc:1305-1329)
__device__ __forceinline__ void put_block_trailer(uint8_t* p, uint32_t cksum) {
  p[0] = 0;
  put_fixed32(p + 1, cksum);
}

// ---- key order (BytewiseCompareInternalKey, db/dbformat.h:1057-1097) ---------------------------------------
struct Key {
  uint64_t hi, lo, tr;
  uint32_t ulen;
};
// user key compare: <0, 0, >0
__device__ __forceinline__ int ukey_cmp(uint64_t ahi, uint64_t alo, uint32_t alen, uint64_t bhi, uint64_t blo, uint32_t blen) {
  if (ahi != bhi) return ahi < bhi ? -1 : 1;
  if (alo != blo) return alo < blo ? -1 : 1;
  return (int)alen - (int)blen;  // equal zero-padded prefix: the shorter key is a proper prefix => smaller
}
__device__ __forceinline__ bool ikey_less(const Key& a, const Key& b) {
  int c = ukey_cmp(a.hi, a.lo, a.ulen, b.hi, b.lo, b.ulen);
  if (c) return c < 0;
  return a.tr > b.tr;  // larger (seq,type) first
}
__device__ __forceinline__ bool same_ukey(const Key& a, uint64_t hi, uint64_t lo, uint32_t ulen) {
  return (a.hi == hi) & (a.lo == lo) & (a.ulen == ulen);
}
__device__ __forceinline__ bool same_ukey(const Key& a, const Key& b) { return same_ukey(a, b.hi, b.lo, b.ulen); }
// first entry of [a, b) of sorted key columns whose user key is >= (hi, lo, ulen), or > it when `upper`
__device__ __forceinline__ uint64_t ukey_bound(const KeyCols& c, uint64_t a, uint64_t b, uint64_t hi, uint64_t lo, uint32_t ulen, bool upper) {
  while (a < b) {
    const uint64_t mid = a + ((b - a) >> 1);
    const ulonglong2 p = c.pfx[mid];
    const int d = ukey_cmp(p.x, p.y, meta_ulen(c.meta[mid]), hi, lo, ulen);
    if (d < 0 || (upper && d == 0)) a = mid + 1;
    else b = mid;
  }
  return a;
}

// ---- decoupled look-back: exclusive prefix sums over parts (decoded blocks, merge tiles) that finish in any order -----------
// One state word per part, zero until the part publishes: the top two bits are the flag (kLbCount: the part's own count,
// kLbPrefix: the inclusive prefix through the part), the low 62 bits are the value.
constexpr unsigned long long kLbCount = 1ull << 62, kLbPrefix = 2ull << 62, kLbValue = (1ull << 62) - 1;
// value of a state word (also of a plain prefix without flag bits, as encode_sizes_kernel writes them)
__device__ __forceinline__ uint64_t lb_value(unsigned long long sv) { return sv & kLbValue; }
// part p's own count; part 0's count is already its inclusive prefix.  One thread per part.
__device__ __forceinline__ void lb_publish(unsigned long long* state, uint64_t p, uint64_t cnt) {
  atomicExch(&state[p], (p == 0 ? kLbPrefix : kLbCount) | cnt);
}
// One warp, after part p published its count: the sum of the counts of the parts in front of p, which then becomes p's inclusive
// prefix.  Lanes read 32 predecessors per step and stop at the nearest inclusive prefix; a predecessor that has not published yet
// is polled every sleep_ns nanoseconds, which leaves the issue slots to warps that still work.  Every lane returns the sum.
__device__ __forceinline__ uint64_t lb_exclusive_prefix(unsigned long long* state, uint64_t p, uint64_t cnt, unsigned lane, uint32_t sleep_ns) {
  uint64_t base = 0;
  if (p != 0) {
    int64_t look = (int64_t)p - 1;
    while (true) {
      const int64_t idx = look - lane;
      unsigned long long sv = kLbPrefix;  // virtual parts before 0 contribute a zero prefix
      if (idx >= 0) {
        sv = *((volatile unsigned long long*)&state[idx]);
        while ((sv >> 62) == 0) {
          __nanosleep(sleep_ns);
          sv = *((volatile unsigned long long*)&state[idx]);
        }
      }
      const unsigned pre_mask = __ballot_sync(0xffffffffu, (sv >> 62) == 2);
      const int first_pre = pre_mask ? __ffs(pre_mask) - 1 : 32;
      uint64_t contrib = ((int)lane <= first_pre) ? lb_value(sv) : 0;
#pragma unroll
      for (int dd = 16; dd; dd >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, dd);
      base += contrib;
      if (pre_mask) break;
      look -= 32;
    }
    if (lane == 0) atomicExch(&state[p], kLbPrefix | (base + cnt));
  }
  return base;
}

// ---- partial sums of a TileStat (kernels.h): key bytes, value bytes, deletions, smallest / largest sequence number ---------------
// Each thread adds entries (or whole stat tiles), then flush() reduces over the warp and adds into five shared slots that
// stat_slots_init prepared.  C is the width of the key-byte and deletion sums: 32 bits where a thread holds few entries, so that
// each is reduced by one redux instruction.
__device__ __forceinline__ void stat_slots_init(unsigned long long* slots, uint32_t t) {
  if (t < 5) slots[t] = t == 3 ? ~0ull : 0ull;
}
template <typename C>
struct StatAcc {
  C kb = 0, nd = 0;
  unsigned long long vb = 0, smin = ~0ull, smax = 0;
  __device__ __forceinline__ void add(C key_bytes, unsigned long long value_bytes, C deletions, unsigned long long seq_lo,
                                      unsigned long long seq_hi) {
    kb += key_bytes;
    vb += value_bytes;
    nd += deletions;
    smin = seq_lo < smin ? seq_lo : smin;
    smax = seq_hi > smax ? seq_hi : smax;
  }
  __device__ __forceinline__ void add_entry(uint32_t key_bytes, uint32_t vlen, uint64_t tr) {
    add(key_bytes, vlen, is_deletion_type((uint32_t)(tr & 0xff)), tr >> 8, tr >> 8);
  }
  __device__ __forceinline__ void flush(unsigned long long* slots) {
    if constexpr (sizeof(C) == 4) {
      kb = __reduce_add_sync(0xffffffffu, kb);
      nd = __reduce_add_sync(0xffffffffu, nd);
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) {
      if constexpr (sizeof(C) == 8) {
        kb += __shfl_xor_sync(0xffffffffu, kb, d);
        nd += __shfl_xor_sync(0xffffffffu, nd, d);
      }
      vb += __shfl_xor_sync(0xffffffffu, vb, d);
      const unsigned long long a = __shfl_xor_sync(0xffffffffu, smin, d), b = __shfl_xor_sync(0xffffffffu, smax, d);
      smin = a < smin ? a : smin;
      smax = b > smax ? b : smax;
    }
    if ((threadIdx.x & 31) == 0) {
      atomicAdd(&slots[0], (unsigned long long)kb);
      atomicAdd(&slots[1], vb);
      atomicAdd(&slots[2], (unsigned long long)nd);
      atomicMin(&slots[3], smin);
      atomicMax(&slots[4], smax);
    }
  }
};

// ---- XXH3-64, seed 0, default secret ------------------------------------------------------------------------
static __device__ __constant__ uint8_t kXxhSecret[192] = {
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
// the same secret in global memory: lane-dependent offsets are served by the L1 instead of serialised constant-bank replays
static __device__ const uint64_t kXxhSecretW[25] = {
    0xbe4ba423396cfeb8ull, 0x1cad21f72c81017cull, 0xdb979083e96dd4deull, 0x1f67b3b7a4a44072ull, 0x78e5c0cc4ee679cbull,
    0x2172ffcc7dd05a82ull, 0x8e2443f7744608b8ull, 0x4c263a81e69035e0ull, 0xcb00c391bb52283cull, 0xa32e531b8b65d088ull,
    0x4ef90da297486471ull, 0xd8acdea946ef1938ull, 0x3f349ce33f76faa8ull, 0x1d4f0bc7c7bbdcf9ull, 0x3159b4cd4be0518aull,
    0x647378d9c97e9fc8ull, 0xc3ebd33483acc5eaull, 0xeb6313faffa081c5ull, 0x49daf0b751dd0d17ull, 0x9e68d429265516d3ull,
    0xfca1477d58be162bull, 0xce31d07ad1b8f88full, 0x280416958f3acb45ull, 0x7e404bbbcafbd7afull, 0ull};
__device__ __forceinline__ uint64_t sec64g(int off) {  // unaligned 8 bytes of the secret, lane-divergent offsets welcome
  const int wi = off >> 3, sh = (off & 7) * 8;
  const uint64_t lo = kXxhSecretW[wi];
  return sh ? (lo >> sh) | (kXxhSecretW[wi + 1] << (64 - sh)) : lo;
}
constexpr uint64_t kP32_1 = 0x9E3779B1ull, kP32_2 = 0x85EBCA77ull, kP32_3 = 0xC2B2AE3Dull;
constexpr uint64_t kP64_1 = 0x9E3779B185EBCA87ull, kP64_2 = 0xC2B2AE3D27D4EB4Full, kP64_3 = 0x165667B19E3779F9ull,
                   kP64_4 = 0x85EBCA77C2B2AE63ull, kP64_5 = 0x27D4EB2F165667C5ull;

__device__ __forceinline__ uint64_t sec64(int off) {  // unaligned read of the constant secret
  uint64_t v = 0;
#pragma unroll
  for (int i = 7; i >= 0; --i) v = (v << 8) | kXxhSecret[off + i];
  return v;
}
__device__ __forceinline__ uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ uint64_t bswap64(uint64_t x) {
  return ((uint64_t)__byte_perm((uint32_t)x, 0, 0x0123) << 32) | (uint64_t)__byte_perm((uint32_t)(x >> 32), 0, 0x0123);
}
__device__ __forceinline__ uint64_t mul128_fold64(uint64_t a, uint64_t b) { return (a * b) ^ __umul64hi(a, b); }
__device__ __forceinline__ uint64_t xxh64_avalanche(uint64_t h) {
  h ^= h >> 33;
  h *= kP64_2;
  h ^= h >> 29;
  h *= kP64_3;
  h ^= h >> 32;
  return h;
}
__device__ __forceinline__ uint64_t xxh3_avalanche(uint64_t h) {
  h ^= h >> 37;
  h *= 0x165667919E3779F9ull;
  h ^= h >> 32;
  return h;
}
__device__ __forceinline__ uint64_t xxh_mix16(const uint8_t* in, int soff) {
  return mul128_fold64(ld_u64(in) ^ sec64(soff), ld_u64(in + 8) ^ sec64(soff + 8));
}
// inputs of at most 240 bytes: evaluated by a single thread (every lane of a warp may call it redundantly)
__device__ inline uint64_t xxh3_64_short(const uint8_t* in, uint32_t len) {
  if (len <= 16) {
    if (len > 8) {
      uint64_t lo = ld_u64(in) ^ (sec64(24) ^ sec64(32)), hi = ld_u64(in + len - 8) ^ (sec64(40) ^ sec64(48));
      return xxh3_avalanche(len + bswap64(lo) + hi + mul128_fold64(lo, hi));
    }
    if (len >= 4) {
      uint64_t i1 = ld_u32(in), i2 = ld_u32(in + len - 4);
      uint64_t h = (i2 + (i1 << 32)) ^ (sec64(8) ^ sec64(16));
      h ^= rotl64(h, 49) ^ rotl64(h, 24);
      h *= 0x9FB21C651E98DF25ull;
      h ^= (h >> 35) + len;
      h *= 0x9FB21C651E98DF25ull;
      return h ^ (h >> 28);
    }
    if (len) {
      uint32_t c = ((uint32_t)in[0] << 16) | ((uint32_t)in[len >> 1] << 24) | in[len - 1] | (len << 8);
      uint32_t s0 = (uint32_t)sec64(0), s1 = (uint32_t)(sec64(0) >> 32);
      return xxh64_avalanche((uint64_t)c ^ (uint64_t)(s0 ^ s1));
    }
    return xxh64_avalanche(sec64(56) ^ sec64(64));
  }
  if (len <= 128) {
    uint64_t acc = len * kP64_1, acc_end;
    acc += xxh_mix16(in, 0);
    acc_end = xxh_mix16(in + len - 16, 16);
    if (len > 32) {
      acc += xxh_mix16(in + 16, 32);
      acc_end += xxh_mix16(in + len - 32, 48);
      if (len > 64) {
        acc += xxh_mix16(in + 32, 64);
        acc_end += xxh_mix16(in + len - 48, 80);
        if (len > 96) {
          acc += xxh_mix16(in + 48, 96);
          acc_end += xxh_mix16(in + len - 64, 112);
        }
      }
    }
    return xxh3_avalanche(acc + acc_end);
  }
  uint64_t acc = len * kP64_1, acc_end;
  uint32_t rounds = len / 16;
  for (uint32_t i = 0; i < 8; i++) acc += xxh_mix16(in + 16 * i, 16 * i);
  acc_end = xxh_mix16(in + len - 16, 136 - 17);
  acc = xxh3_avalanche(acc);
  for (uint32_t i = 8; i < rounds; i++) acc_end += xxh_mix16(in + 16 * i, 16 * (i - 8) + 3);
  return xxh3_avalanche(acc + acc_end);
}

// Warp-cooperative XXH3-64 of a buffer in generic memory (all 32 lanes call with identical arguments; every
// lane returns the hash).  Long inputs: lane l owns accumulator lane (l & 7) of stripe group (l >> 3); the four
// groups take stripes g, g+4, ... of each 1024-byte block, partial sums are folded with shuffles before the
// scramble (additions commute inside a block; the scramble is the only sequential step).
// per-lane secret words of the four stripes a lane owns inside a 1024-byte block (stripe g + 4i, accumulator lane a)
struct XxhLaneSecret {
  uint64_t k[4];
};
__device__ __forceinline__ XxhLaneSecret xxh_lane_secret() {
  const unsigned lane = threadIdx.x & 31;
  const int a = lane & 7, g = lane >> 3;
  XxhLaneSecret r;
#pragma unroll
  for (int i = 0; i < 4; i++) r.k[i] = sec64g(8 * (g + 4 * i) + 8 * a);
  return r;
}
// accumulator contribution of `nstripes` (<= 16) 64-byte stripes starting at blk: every lane returns the total for its
// accumulator lane a = lane & 7 (additions commute inside a 1024-byte block; raw data goes to lane a ^ 1)
template <bool kAligned8>
__device__ __forceinline__ uint64_t xxh3_block_contrib(const uint8_t* blk, uint64_t nstripes, const XxhLaneSecret& ks) {
  const unsigned lane = threadIdx.x & 31;
  const int a = lane & 7, g = lane >> 3;
  uint64_t mul = 0, add = 0;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const uint64_t s = g + 4 * i;
    if (s < nstripes) {
      const uint64_t dv = kAligned8 ? ld_u64_aligned(blk + 64 * s + 8 * a) : ld_u64_funnel(blk + 64 * s + 8 * a);
      const uint64_t dk = dv ^ ks.k[i];
      mul += (dk & 0xffffffffull) * (dk >> 32);
      add += dv;
    }
  }
  uint64_t part = mul + __shfl_xor_sync(0xffffffffu, add, 1);
  part += __shfl_xor_sync(0xffffffffu, part, 8);
  part += __shfl_xor_sync(0xffffffffu, part, 16);
  return part;
}
// pre != nullptr: contributions of the full 1024-byte blocks were computed elsewhere (pre[8 * n + a])
template <bool kAligned8>
__device__ inline uint64_t xxh3_64_warp_t(const uint8_t* in, uint64_t len, const uint64_t* pre = nullptr) {
  const unsigned lane = threadIdx.x & 31;
  if (len <= 240) return xxh3_64_short(in, (uint32_t)len);
  const int a = lane & 7;
  const uint64_t init[8] = {kP32_3, kP64_1, kP64_2, kP64_3, kP64_4, kP32_2, kP64_5, kP32_1};
  uint64_t acc = init[a];  // identical in the four lane groups
  const uint64_t nb_blocks = (len - 1) / 1024;
  const uint64_t kscr = sec64g(192 - 64 + 8 * a);
  const XxhLaneSecret ks = xxh_lane_secret();
  uint64_t n = 0;
  if (pre) {
    // precomputed block contributions: the scramble chain is sequential, the loads are not -- fetch eight blocks' values
    // before the first is consumed (a load-use loop body costs one memory round trip per iteration)
    for (; n + 8 <= nb_blocks; n += 8) {
      uint64_t pv[8];
#pragma unroll
      for (int q = 0; q < 8; q++) pv[q] = pre[8 * (n + q) + a];
#pragma unroll
      for (int q = 0; q < 8; q++) {
        acc += pv[q];
        acc ^= acc >> 47;
        acc ^= kscr;
        acc *= kP32_1;
      }
    }
  }
  for (; n <= nb_blocks; n++) {
    const uint64_t nstripes = n < nb_blocks ? 16 : ((len - 1) - 1024 * nb_blocks) / 64;
    acc += (pre && n < nb_blocks) ? pre[8 * n + a] : xxh3_block_contrib<kAligned8>(in + n * 1024, nstripes, ks);
    if (n < nb_blocks) {
      acc ^= acc >> 47;
      acc ^= kscr;
      acc *= kP32_1;
    }
  }
  // last stripe: input + len - 64 with secret offset 192 - 64 - 7
  {
    uint64_t dv = ld_u64_funnel(in + len - 64 + 8 * a), dk = dv ^ sec64g(192 - 64 - 7 + 8 * a);
    uint64_t mul = (dk & 0xffffffffull) * (dk >> 32);
    uint64_t add_sw = __shfl_xor_sync(0xffffffffu, dv, 1);
    acc += mul + add_sw;
  }
  // merge: result = len*P64_1 + sum_i fold(acc[2i] ^ sec(11+16i), acc[2i+1] ^ sec(11+16i+8))
  uint64_t keyed = acc ^ sec64g(11 + 8 * a);
  uint64_t other = __shfl_xor_sync(0xffffffffu, keyed, 1);
  uint64_t m = (a & 1) ? 0 : mul128_fold64(keyed, other);
  m += __shfl_xor_sync(0xffffffffu, m, 2);
  m += __shfl_xor_sync(0xffffffffu, m, 4);
  uint64_t r = xxh3_avalanche(len * kP64_1 + m);
  return __shfl_sync(0xffffffffu, r, 0);
}

__device__ inline uint64_t xxh3_64_warp(const uint8_t* in, uint64_t len) {
  return (((uintptr_t)in & 7) == 0) ? xxh3_64_warp_t<true>(in, len) : xxh3_64_warp_t<false>(in, len);
}

// CRC32C (Castagnoli, reflected polynomial 0x82F63B78) — byte-wise table step used by the warp routine below.
static __device__ __constant__ uint32_t kCrcTable[256] = {
    0x00000000u, 0xf26b8303u, 0xe13b70f7u, 0x1350f3f4u, 0xc79a971fu, 0x35f1141cu, 0x26a1e7e8u, 0xd4ca64ebu,
    0x8ad958cfu, 0x78b2dbccu, 0x6be22838u, 0x9989ab3bu, 0x4d43cfd0u, 0xbf284cd3u, 0xac78bf27u, 0x5e133c24u,
    0x105ec76fu, 0xe235446cu, 0xf165b798u, 0x030e349bu, 0xd7c45070u, 0x25afd373u, 0x36ff2087u, 0xc494a384u,
    0x9a879fa0u, 0x68ec1ca3u, 0x7bbcef57u, 0x89d76c54u, 0x5d1d08bfu, 0xaf768bbcu, 0xbc267848u, 0x4e4dfb4bu,
    0x20bd8edeu, 0xd2d60dddu, 0xc186fe29u, 0x33ed7d2au, 0xe72719c1u, 0x154c9ac2u, 0x061c6936u, 0xf477ea35u,
    0xaa64d611u, 0x580f5512u, 0x4b5fa6e6u, 0xb93425e5u, 0x6dfe410eu, 0x9f95c20du, 0x8cc531f9u, 0x7eaeb2fau,
    0x30e349b1u, 0xc288cab2u, 0xd1d83946u, 0x23b3ba45u, 0xf779deaeu, 0x05125dadu, 0x1642ae59u, 0xe4292d5au,
    0xba3a117eu, 0x4851927du, 0x5b016189u, 0xa96ae28au, 0x7da08661u, 0x8fcb0562u, 0x9c9bf696u, 0x6ef07595u,
    0x417b1dbcu, 0xb3109ebfu, 0xa0406d4bu, 0x522bee48u, 0x86e18aa3u, 0x748a09a0u, 0x67dafa54u, 0x95b17957u,
    0xcba24573u, 0x39c9c670u, 0x2a993584u, 0xd8f2b687u, 0x0c38d26cu, 0xfe53516fu, 0xed03a29bu, 0x1f682198u,
    0x5125dad3u, 0xa34e59d0u, 0xb01eaa24u, 0x42752927u, 0x96bf4dccu, 0x64d4cecfu, 0x77843d3bu, 0x85efbe38u,
    0xdbfc821cu, 0x2997011fu, 0x3ac7f2ebu, 0xc8ac71e8u, 0x1c661503u, 0xee0d9600u, 0xfd5d65f4u, 0x0f36e6f7u,
    0x61c69362u, 0x93ad1061u, 0x80fde395u, 0x72966096u, 0xa65c047du, 0x5437877eu, 0x4767748au, 0xb50cf789u,
    0xeb1fcbadu, 0x197448aeu, 0x0a24bb5au, 0xf84f3859u, 0x2c855cb2u, 0xdeeedfb1u, 0xcdbe2c45u, 0x3fd5af46u,
    0x7198540du, 0x83f3d70eu, 0x90a324fau, 0x62c8a7f9u, 0xb602c312u, 0x44694011u, 0x5739b3e5u, 0xa55230e6u,
    0xfb410cc2u, 0x092a8fc1u, 0x1a7a7c35u, 0xe811ff36u, 0x3cdb9bddu, 0xceb018deu, 0xdde0eb2au, 0x2f8b6829u,
    0x82f63b78u, 0x709db87bu, 0x63cd4b8fu, 0x91a6c88cu, 0x456cac67u, 0xb7072f64u, 0xa457dc90u, 0x563c5f93u,
    0x082f63b7u, 0xfa44e0b4u, 0xe9141340u, 0x1b7f9043u, 0xcfb5f4a8u, 0x3dde77abu, 0x2e8e845fu, 0xdce5075cu,
    0x92a8fc17u, 0x60c37f14u, 0x73938ce0u, 0x81f80fe3u, 0x55326b08u, 0xa759e80bu, 0xb4091bffu, 0x466298fcu,
    0x1871a4d8u, 0xea1a27dbu, 0xf94ad42fu, 0x0b21572cu, 0xdfeb33c7u, 0x2d80b0c4u, 0x3ed04330u, 0xccbbc033u,
    0xa24bb5a6u, 0x502036a5u, 0x4370c551u, 0xb11b4652u, 0x65d122b9u, 0x97baa1bau, 0x84ea524eu, 0x7681d14du,
    0x2892ed69u, 0xdaf96e6au, 0xc9a99d9eu, 0x3bc21e9du, 0xef087a76u, 0x1d63f975u, 0x0e330a81u, 0xfc588982u,
    0xb21572c9u, 0x407ef1cau, 0x532e023eu, 0xa145813du, 0x758fe5d6u, 0x87e466d5u, 0x94b49521u, 0x66df1622u,
    0x38cc2a06u, 0xcaa7a905u, 0xd9f75af1u, 0x2b9cd9f2u, 0xff56bd19u, 0x0d3d3e1au, 0x1e6dcdeeu, 0xec064eedu,
    0xc38d26c4u, 0x31e6a5c7u, 0x22b65633u, 0xd0ddd530u, 0x0417b1dbu, 0xf67c32d8u, 0xe52cc12cu, 0x1747422fu,
    0x49547e0bu, 0xbb3ffd08u, 0xa86f0efcu, 0x5a048dffu, 0x8ecee914u, 0x7ca56a17u, 0x6ff599e3u, 0x9d9e1ae0u,
    0xd3d3e1abu, 0x21b862a8u, 0x32e8915cu, 0xc083125fu, 0x144976b4u, 0xe622f5b7u, 0xf5720643u, 0x07198540u,
    0x590ab964u, 0xab613a67u, 0xb831c993u, 0x4a5a4a90u, 0x9e902e7bu, 0x6cfbad78u, 0x7fab5e8cu, 0x8dc0dd8fu,
    0xe330a81au, 0x115b2b19u, 0x020bd8edu, 0xf0605beeu, 0x24aa3f05u, 0xd6c1bc06u, 0xc5914ff2u, 0x37faccf1u,
    0x69e9f0d5u, 0x9b8273d6u, 0x88d28022u, 0x7ab90321u, 0xae7367cau, 0x5c18e4c9u, 0x4f48173du, 0xbd23943eu,
    0xf36e6f75u, 0x0105ec76u, 0x12551f82u, 0xe03e9c81u, 0x34f4f86au, 0xc69f7b69u, 0xd5cf889du, 0x27a40b9eu,
    0x79b737bau, 0x8bdcb4b9u, 0x988c474du, 0x6ae7c44eu, 0xbe2da0a5u, 0x4c4623a6u, 0x5f16d052u, 0xad7d5351u};
__device__ __forceinline__ uint32_t crc32c_bytes(uint32_t c, const uint8_t* p, uint64_t n) {
  for (uint64_t i = 0; i < n; i++) c = kCrcTable[(c ^ p[i]) & 0xff] ^ (c >> 8);
  return c;
}
// multiply two polynomials mod the CRC32C polynomial (reflected representation)
__device__ __forceinline__ uint32_t crc_gf_mul(uint32_t a, uint32_t b) {
  uint32_t p = 0;
#pragma unroll 1
  for (int i = 0; i < 32; i++) {
    p ^= (b & 0x80000000u) ? a : 0;
    a = (a >> 1) ^ ((a & 1) ? 0x82F63B78u : 0);
    b <<= 1;
  }
  return p;
}
// x^(8*nbytes) mod P, reflected
__device__ inline uint32_t crc_xpow8n(uint64_t nbytes) {
  uint32_t r = 0x80000000u;      // x^0
  uint32_t base = 0x00800000u;   // x^8
  while (nbytes) {
    if (nbytes & 1) r = crc_gf_mul(r, base);
    base = crc_gf_mul(base, base);
    nbytes >>= 1;
  }
  return r;
}
// Warp-cooperative raw CRC state update over a buffer: returns crc32c::Extend(init=0) style *unfinalised* value
// handling (internal state with pre/post inversion applied by caller).  Each lane CRCs a contiguous slice with a
// zero initial state; slices are combined left to right: state = state * x^(8*len_slice) + crc_slice.
__device__ inline uint32_t crc32c_value_warp(const uint8_t* in, uint64_t len) {
  const unsigned lane = threadIdx.x & 31;
  uint64_t per = (len + 31) / 32;
  uint64_t b = per * lane < len ? per * lane : len, e = per * (lane + 1) < len ? per * (lane + 1) : len;
  // raw polynomial remainder of the slice (no inversion): start state 0 except lane 0 which carries the 0xffffffff preset
  uint32_t c = crc32c_bytes(lane == 0 ? 0xffffffffu : 0u, in + b, e - b);
  uint64_t mylen = e - b;
  // inclusive combine (left fold) via log-step scan: state over [0, end_of_lane)
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t pc = __shfl_up_sync(0xffffffffu, c, d);
    uint64_t plen = __shfl_up_sync(0xffffffffu, mylen, d);
    if ((int)lane >= d) {
      c = crc_gf_mul(pc, crc_xpow8n(mylen)) ^ c;
      mylen += plen;
    }
  }
  uint32_t total = __shfl_sync(0xffffffffu, c, 31);
  return total ^ 0xffffffffu;
}
__device__ __forceinline__ uint32_t crc32c_mask(uint32_t crc) { return ((crc >> 15) | (crc << 17)) + 0xa282ead8u; }

// ComputeBuiltinChecksumWithLastByte (table/format.cc:468-509); warp-cooperative, all lanes get the value.
__device__ inline uint32_t block_checksum_warp(uint32_t type, const uint8_t* data, uint64_t n, uint8_t last_byte) {
  if (type == 4) return (uint32_t)xxh3_64_warp(data, n) ^ (uint32_t)last_byte * 0x6b9083d9u;
  if (type == 1) {
    uint32_t crc = crc32c_value_warp(data, n);
    uint32_t c = crc ^ 0xffffffffu;
    c = kCrcTable[(c ^ last_byte) & 0xff] ^ (c >> 8);
    return crc32c_mask(c ^ 0xffffffffu);
  }
  return 0;
}

// ---- explicit shared-memory accesses by 32-bit shared address (keeps the hot loops free of generic 64-bit addressing)
__device__ __forceinline__ uint64_t lds64(uint32_t a) {
  uint64_t v;
  asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ uint32_t lds8(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ uint32_t lds16(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts16(uint32_t a, uint32_t v) { asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
// 4 / 8 bytes at any alignment (reads up to 7 bytes past the value, inside the slice)
__device__ __forceinline__ uint32_t lds32_any(uint32_t a) {
  const uint32_t al = a & ~3u;
  return __funnelshift_r(lds32(al), lds32(al + 4), (a & 3) * 8);
}
__device__ __forceinline__ uint64_t shr128(uint64_t lo, uint64_t hi, uint32_t s) {  // (hi:lo) >> s, s in {0, 8, .., 56}
  return s ? (lo >> s) | (hi << (64 - s)) : lo;
}
__device__ __forceinline__ uint64_t lds64_any(uint32_t a) {
  const uint32_t al = a & ~7u;
  return shr128(lds64(al), lds64(al + 8), (a & 7) * 8);
}
// per-lane XXH3 constants (lane l: accumulator lane a = l & 7, stripe group g = l >> 3), computed once per CTA
struct XxhLaneTab {
  uint64_t k[4][32];   // secret words of the four stripes a lane owns inside a 1024-byte block
  uint64_t kscr[32];   // scramble secret
  uint64_t klast[32];  // secret of the last stripe
  uint64_t kmrg[32];   // merge secret
  uint64_t kinit[32];  // initial value of the lane's accumulator
};

// ---- mbarrier + TMA bulk copy (global -> shared), sm_90+ ----------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// size: multiple of 16; dst / src: 16-byte aligned
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes),
               "r"(bar)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
  }
}

// shared -> global bulk copy (TMA): size multiple of 16, both addresses 16-byte aligned; completion by bulk groups
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// the bulk stores this thread issued have finished READING shared memory (the source may be overwritten)
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// generic-proxy writes to shared memory become visible to the async proxy (TMA) / are ordered before its accesses
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- XXH3-64 (seed 0) of a block staged in shared memory, warp-cooperative, lean: the per-lane secrets come from a table the CTA
// fills once (XxhLaneTab), the data is read with the cheapest loads the block's byte phase allows.  Same arithmetic as
// xxh3_64_warp_t (common.cuh); inputs of at most 240 bytes take the generic routine.
__device__ __forceinline__ void fill_xxh_lane_tab(XxhLaneTab* t) {
  for (uint32_t i = threadIdx.x; i < 32; i += blockDim.x) {
    const int a = i & 7, g = i >> 3;
    for (int q = 0; q < 4; q++) t->k[q][i] = sec64g(8 * (g + 4 * q) + 8 * a);
    t->kscr[i] = sec64g(192 - 64 + 8 * a);
    t->klast[i] = sec64g(192 - 64 - 7 + 8 * a);
    t->kmrg[i] = sec64g(11 + 8 * a);
    const uint64_t init[8] = {kP32_3, kP64_1, kP64_2, kP64_3, kP64_4, kP32_2, kP64_5, kP32_1};
    t->kinit[i] = init[a];
  }
}
// 8 bytes at shared address p; o = p & 7 is the same for every lane (kPhase: 0 aligned, 1 o in 1..3, 2 o in 4..7)
template <int kPhase>
__device__ __forceinline__ uint64_t lds64_phase(uint32_t p, uint32_t o) {
  if (kPhase == 0) return lds64(p);
  const uint32_t al = p - o;
  if (kPhase == 1) {
    const uint64_t w01 = lds64(al);
    const uint32_t w2 = lds32(al + 8), bs = 8 * o;
    return (uint64_t)__funnelshift_r((uint32_t)w01, (uint32_t)(w01 >> 32), bs) | ((uint64_t)__funnelshift_r((uint32_t)(w01 >> 32), w2, bs) << 32);
  }
  const uint32_t w1 = lds32(al + 4), bs = 8 * (o - 4);
  const uint64_t w23 = lds64(al + 8);
  return (uint64_t)__funnelshift_r(w1, (uint32_t)w23, bs) | ((uint64_t)__funnelshift_r((uint32_t)w23, (uint32_t)(w23 >> 32), bs) << 32);
}
template <int kPhase>
__device__ __forceinline__ uint64_t xxh3_staged_t(uint32_t sp, uint32_t len, uint32_t tab, unsigned lane) {
  const uint32_t a = lane & 7, g = lane >> 3, o = sp & 7;
  const uint32_t tl = tab + 8 * lane;  // this lane's column of the table
  uint64_t acc = lds64(tl + 1792);     // (from the table: selecting it from a constant array put the array in local memory)
  const uint64_t k0 = lds64(tl), k1 = lds64(tl + 256), k2 = lds64(tl + 512), k3 = lds64(tl + 768), kscr = lds64(tl + 1024);
  const uint32_t nb_blocks = (len - 1) >> 10;
  uint32_t p = sp + 64 * g + 8 * a;  // stripe g of the current 1024-byte block, this lane's word
  for (uint32_t n = 0; n < nb_blocks; n++, p += 1024) {
    const uint64_t d0 = lds64_phase<kPhase>(p, o), d1 = lds64_phase<kPhase>(p + 256, o), d2 = lds64_phase<kPhase>(p + 512, o),
                   d3 = lds64_phase<kPhase>(p + 768, o);
    const uint64_t e0 = d0 ^ k0, e1 = d1 ^ k1, e2 = d2 ^ k2, e3 = d3 ^ k3;
    uint64_t mul = (e0 & 0xffffffffull) * (e0 >> 32);
    mul += (e1 & 0xffffffffull) * (e1 >> 32);
    mul += (e2 & 0xffffffffull) * (e2 >> 32);
    mul += (e3 & 0xffffffffull) * (e3 >> 32);
    const uint64_t add = d0 + d1 + d2 + d3;
    uint64_t part = mul + __shfl_xor_sync(0xffffffffu, add, 1);
    part += __shfl_xor_sync(0xffffffffu, part, 8);
    part += __shfl_xor_sync(0xffffffffu, part, 16);
    acc += part;
    acc ^= acc >> 47;
    acc ^= kscr;
    acc *= kP32_1;
  }
  {  // the partial last block: stripes g + 4i < nstripes
    const uint32_t nstripes = ((len - 1) - 1024 * nb_blocks) >> 6;
    uint64_t mul = 0, add = 0;
    const uint64_t kq[4] = {k0, k1, k2, k3};
#pragma unroll
    for (int i = 0; i < 4; i++) {
      if (g + 4 * i < nstripes) {
        const uint64_t dv = lds64_phase<kPhase>(p + 256 * i, o), dk = dv ^ kq[i];
        mul += (dk & 0xffffffffull) * (dk >> 32);
        add += dv;
      }
    }
    uint64_t part = mul + __shfl_xor_sync(0xffffffffu, add, 1);
    part += __shfl_xor_sync(0xffffffffu, part, 8);
    part += __shfl_xor_sync(0xffffffffu, part, 16);
    acc += part;
  }
  {  // last stripe: input + len - 64 with secret offset 192 - 64 - 7 (any phase)
    const uint64_t dv = lds64_any(sp + len - 64 + 8 * a), dk = dv ^ lds64(tl + 1280);
    acc += (dk & 0xffffffffull) * (dk >> 32) + __shfl_xor_sync(0xffffffffu, dv, 1);
  }
  const uint64_t keyed = acc ^ lds64(tl + 1536);
  const uint64_t other = __shfl_xor_sync(0xffffffffu, keyed, 1);
  uint64_t m = (a & 1) ? 0 : mul128_fold64(keyed, other);
  m += __shfl_xor_sync(0xffffffffu, m, 2);
  m += __shfl_xor_sync(0xffffffffu, m, 4);
  return xxh3_avalanche((uint64_t)len * kP64_1 + m);  // lanes 0..7 of a group hold the sum; every lane with a == 0..7 has it after the xors
}
static_assert(offsetof(XxhLaneTab, k) == 0 && offsetof(XxhLaneTab, kscr) == 1024 && offsetof(XxhLaneTab, klast) == 1280 &&
                  offsetof(XxhLaneTab, kmrg) == 1536 && offsetof(XxhLaneTab, kinit) == 1792,
              "xxh3_staged_t addresses the lane table by these offsets");
// block checksum (table/format.cc:468-509) of the staged block: type 4 = XXH3, 1 = CRC32C
__device__ __forceinline__ uint32_t staged_block_checksum(uint32_t type, uint32_t sp, const uint8_t* p, uint32_t n, uint8_t last_byte, uint32_t xtab,
                                                          unsigned lane) {
  if (type == 4 && n > 240) {
    const uint32_t o = sp & 7;
    const uint64_t h = o == 0 ? xxh3_staged_t<0>(sp, n, xtab, lane) : o < 4 ? xxh3_staged_t<1>(sp, n, xtab, lane) : xxh3_staged_t<2>(sp, n, xtab, lane);
    return (uint32_t)__shfl_sync(0xffffffffu, h, 0) ^ (uint32_t)last_byte * 0x6b9083d9u;
  }
  return block_checksum_warp(type, p, n, last_byte);
}

// ---- encoded entry sizes (BlockBuilder::AddWithLastKey, block_builder.cc:177-253) --------------------------------------
__device__ __forceinline__ uint32_t ikey_byte(uint64_t hi, uint64_t lo, uint32_t ulen, uint64_t tr, uint32_t j) {
  if (j < ulen) return (uint32_t)(((j < 8) ? (hi >> (56 - 8 * j)) : (lo >> (56 - 8 * (j - 8)))) & 0xff);
  return (uint32_t)((tr >> (8 * (j - ulen))) & 0xff);
}
// bytes shared by two internal keys (Slice::difference_offset on the raw key bytes, block_builder.cc:214)
__device__ __forceinline__ uint32_t shared_prefix(uint64_t ahi, uint64_t alo, uint32_t alen, uint64_t atr, uint64_t bhi, uint64_t blo,
                                                  uint32_t blen, uint64_t btr) {
  if (alen == blen) {
    uint32_t cb;
    uint64_t x = ahi ^ bhi;
    if (x) cb = (uint32_t)__clzll((long long)x) >> 3;
    else {
      uint64_t y = alo ^ blo;
      cb = y ? 8 + ((uint32_t)__clzll((long long)y) >> 3) : 16;
    }
    if (cb < alen) return cb;
    uint64_t z = atr ^ btr;
    uint32_t tb = z ? ((uint32_t)(__ffsll((long long)z) - 1) >> 3) : 8;
    return alen + tb;
  }
  uint32_t n = (alen < blen ? alen : blen) + 8, j = 0;
  while (j < n && ikey_byte(ahi, alo, alen, atr, j) == ikey_byte(bhi, blo, blen, btr, j)) j++;
  return j;
}
__device__ __forceinline__ uint32_t entry_size(uint32_t shared, uint32_t ks, uint32_t vs) {
  return varint_len32(shared) + varint_len32(ks - shared) + varint_len32(vs) + (ks - shared) + vs;
}
// restart surcharge: entry_size of the entry stored as a restart entry (shared == 0) minus entry_size with `shared` bytes shared
__host__ __device__ __forceinline__ uint32_t restart_surcharge(uint32_t shared, uint32_t ks) {
  return 1u + varint_len32(ks) + shared - varint_len32(shared) - varint_len32(ks - shared);
}
// ---- warp scans ---------------------------------------------------------------------------------------------
// Cooperative global -> shared copy with kDepth loads per thread in flight: a plain `dst[i] = src[i]` loop issues in
// order, so each iteration would wait for its own DRAM round trip before the next load leaves.
template <typename T, int kDepth = 8>
__device__ __forceinline__ void coop_copy(T* __restrict__ dst, const T* __restrict__ src, uint32_t n) {
  const uint32_t nt = blockDim.x;
  for (uint32_t base = 0; base < n; base += kDepth * nt) {
    T v[kDepth];
#pragma unroll
    for (int k = 0; k < kDepth; k++) {
      const uint32_t i = base + k * nt + threadIdx.x;
      if (i < n) v[k] = src[i];
    }
#pragma unroll
    for (int k = 0; k < kDepth; k++) {
      const uint32_t i = base + k * nt + threadIdx.x;
      if (i < n) dst[i] = v[k];
    }
  }
}

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v) {
  const unsigned lane = threadIdx.x & 31;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t t = __shfl_up_sync(0xffffffffu, v, d);
    if ((int)lane >= d) v += t;
  }
  return v;
}
__device__ __forceinline__ uint64_t warp_incl_scan64(uint64_t v) {
  const unsigned lane = threadIdx.x & 31;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint64_t t = __shfl_up_sync(0xffffffffu, v, d);
    if ((int)lane >= d) v += t;
  }
  return v;
}

}  // namespace b200c
