// toplingdb_b200/csrc/decode.cu — BlockBasedTable input decode on the device.
//
// Replaces, for the compaction read path, BlockBasedTableIterator::{InitDataBlock,Next}
// (table/block_based/block_based_table_iterator.cc:224-411), BlockFetcher::ReadBlockContents + checksum check
// (table/block_fetcher.cc:32-40,211), DataBlockIter::ParseNextKey / DecodeEntry (table/block_based/block.cc:37-64,
// 617-665) and the IndexBlockIter walk that feeds them.
//
// Layout produced: every run decoded into one set of columns (KeyCols) indexed by a global entry number; run r
// owns [run_start[r], run_start[r+1]).  Values are NOT copied: vref[i] is the device address of the value bytes
// inside the resident file image, so each value byte crosses HBM once more only (file image -> output block).
//
// Kernels (algorithmic bytes = file bytes read once + 36 B of columns written per entry):
//   index_decode_kernel        one thread per index restart point -> data block handles
//   block_decode_fused_kernel  one warp per data block: cp.async staging into shared memory, restart-interval walk (one lane
//                              per interval), block checksum (warp-cooperative XXH3 / CRC32C), decoupled look-back for
//                              the global entry position, one-entry-per-lane key reconstruction by a scan over the
//                              prefix-decompression maps, coalesced column stores (details above the kernel)
#include <cstddef>
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"
#include "inflate_rules.h"
#include "range_rules.h"

namespace b200c {

__device__ __forceinline__ int file_of_block(const FileDesc* files, int nfiles, uint32_t gblk) {
  int f = 0;
  while (f + 1 < nfiles && gblk >= files[f + 1].gblk_first) f++;
  return f;
}

// ---------------------------------------------------------------------------------------------- index block
// IndexValue decode (table/format.cc:120-140): shared == 0 -> varint64 offset, varint64 size; else (fv >= 4)
// varsigned64 size delta and offset = prev_offset + prev_size + kBlockTrailerSize.
// blk_off[b] = offset of the block inside its file | file index << kBlkFileShift (the block decoder gets both with one load)
constexpr int kBlkFileShift = 48;
constexpr uint64_t kBlkOffMask = (1ull << kBlkFileShift) - 1;
// a block that was stored compressed: the offset (bit 47 set) counts from the job's arena of inflated blocks, not from the file image
constexpr uint64_t kBlkArenaBit = 1ull << 47;
struct IndexEntry {
  uint64_t shared, non_shared;
  const uint8_t* sep;  // the separator's non_shared bytes
  uint64_t off, size;  // block handle; on entry the previous entry's (a delta-encoded handle counts from it)
};
// the index entry at p, which ends before `end`; returns where the next entry starts, nullptr when malformed
__device__ __forceinline__ const uint8_t* read_index_entry(const FileDesc& fd, const uint8_t* p, const uint8_t* end, IndexEntry& e) {
  uint64_t vl;
  int c;
  if (!(c = get_varint(p, end, &e.shared))) return nullptr;
  p += c;
  if (!(c = get_varint(p, end, &e.non_shared))) return nullptr;
  p += c;
  if (!fd.value_delta) {
    if (!(c = get_varint(p, end, &vl))) return nullptr;
    p += c;
  }
  if (e.non_shared > (uint64_t)(end - p)) return nullptr;
  e.sep = p;
  p += e.non_shared;
  if (e.shared == 0 || !fd.value_delta) {
    if (!(c = get_varint(p, end, &e.off))) return nullptr;
    p += c;
    if (!(c = get_varint(p, end, &e.size))) return nullptr;
    return p + c;
  }
  uint64_t t;
  if (!(c = get_varint(p, end, &t))) return nullptr;
  e.off += e.size + 5;
  e.size += (uint64_t)((int64_t)(t >> 1) ^ -(int64_t)(t & 1));
  return p + c;
}
__device__ __forceinline__ bool handle_in_file(const FileDesc& fd, const IndexEntry& e) {
  return e.off + e.size + 5 <= fd.len && e.size >= 4 && e.size <= 0xffffffffull && e.off < kBlkArenaBit;
}

__device__ void index_decode_sequential(const FileDesc& fd, uint32_t file_idx, const uint8_t* blk, uint32_t nr, uint64_t* blk_off,
                                        uint32_t* blk_size, uint32_t* err) {
  const uint8_t* end = blk + fd.index_size - 4 - 4ull * nr;
  const uint8_t* p = blk;
  IndexEntry e{0, 0, nullptr, 0, 0};
  uint32_t n = 0;
  while (p < end) {
    const uint8_t* next = read_index_entry(fd, p, end, e);
    if (!next) break;
    p = next;
    if (n >= fd.nblocks) {
      n++;
      break;
    }
    if (!handle_in_file(fd, e)) {
      atomicOr(err, kErrCorruptBlock);
      e.off = 0;
      e.size = 4;
    }
    blk_off[fd.gblk_first + n] = e.off | ((uint64_t)file_idx << kBlkFileShift);
    blk_size[fd.gblk_first + n] = (uint32_t)e.size;
    n++;
  }
  if (p != end || n != fd.nblocks) atomicOr(err, kErrCorruptBlock);
}

// separator key of the index entry at restart offset ro (restart interval 1: shared == 0) as a range key; false when it is longer than
// 16 bytes or the entry is malformed -- the block is then kept
__device__ __forceinline__ bool index_separator(const FileDesc& fd, const uint8_t* blk, uint32_t ro, const uint8_t* rs, RangeKey* out) {
  IndexEntry e{0, 0, nullptr, 0, 0};
  if (ro >= fd.index_size || !read_index_entry(fd, blk + ro, rs, e) || e.shared != 0) return false;
  uint64_t ulen = e.non_shared;
  if (!fd.index_user_key) {
    if (ulen < 8) return false;
    ulen -= 8;
  }
  if (ulen > (uint64_t)kMaxUserKey) return false;
  uint64_t hi = 0, lo = 0;
  for (uint32_t t = 0; t < 8; t++) hi = (hi << 8) | (t < ulen ? e.sep[t] : 0);
  for (uint32_t t = 8; t < 16; t++) lo = (lo << 8) | (t < ulen ? e.sep[t] : 0);
  *out = RangeKey{hi, lo, (uint32_t)ulen};
  return true;
}

__global__ void index_decode_kernel(const FileDesc* __restrict__ files, int nfiles, uint64_t* __restrict__ blk_off,
                                    uint32_t* __restrict__ blk_size, BoundKey start, uint32_t has_start, BoundKey end, uint32_t has_end,
                                    uint32_t* __restrict__ err) {
  const int f = blockIdx.y;
  if (f >= nfiles) return;
  const FileDesc fd = files[f];
  if (fd.index_size < 8 || (fd.index_ptr == nullptr && fd.index_off + fd.index_size + 5 > fd.len)) {
    if (threadIdx.x == 0 && blockIdx.x == 0) atomicOr(err, kErrCorruptBlock);
    return;
  }
  const uint8_t* blk = fd.index_ptr ? fd.index_ptr : fd.base + fd.index_off;
  const uint32_t nr = ld_u32(blk + fd.index_size - 4) & 0x7fffffffu;
  if (4ull * nr + 4 > fd.index_size) {
    if (threadIdx.x == 0 && blockIdx.x == 0) atomicOr(err, kErrCorruptBlock);
    return;
  }
  if (nr != fd.nblocks) {  // index_block_restart_interval != 1: rare, walk it with one thread
    if (threadIdx.x == 0 && blockIdx.x == 0) index_decode_sequential(fd, (uint32_t)f, blk, nr, blk_off, blk_size, err);
    return;
  }
  const uint8_t* rs = blk + fd.index_size - 4 - 4ull * nr;
  const RangeKey rstart{start.hi, start.lo, start.ulen}, rend{end.hi, end.lo, end.ulen};
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < nr; j += gridDim.x * blockDim.x) {
    const uint32_t ro = ld_u32(rs + 4ull * j);
    IndexEntry e{0, 0, nullptr, 0, 0};
    if (ro >= fd.index_size || !read_index_entry(fd, blk + ro, rs, e) || e.shared != 0 || !handle_in_file(fd, e)) {
      atomicOr(err, kErrCorruptBlock);
      e.off = 0;
      e.size = 4;
    } else if (has_start || has_end) {
      // sub-compaction key range: block j holds only user keys in (separator j - 1, separator j] (range_rules.h)
      RangeKey sep, prev;
      bool have_prev = false;
      if (index_separator(fd, blk, ro, rs, &sep)) {
        bool usable = true;
        if (j > 0) {
          have_prev = index_separator(fd, blk, ld_u32(rs + 4ull * (j - 1)), rs, &prev);
          usable = have_prev;  // an unreadable predecessor: keep the block
        }
        if (usable && !block_may_touch_range(sep, have_prev, prev, has_start != 0, rstart, has_end != 0, rend)) e.size = 0;  // skipped
      }
    }
    blk_off[fd.gblk_first + j] = e.off | ((uint64_t)f << kBlkFileShift);
    blk_size[fd.gblk_first + j] = (uint32_t)e.size;
  }
}

// ---------------------------------------------------------------------------------------------- data blocks
struct Win {  // 40 bytes starting at the 8-byte aligned address below p (generic loads: shared-memory staging or image)
  uint64_t w0, w1, w2, w3, w4;
};
__device__ __forceinline__ Win load_win_any(const uint8_t* p) {
  const uint64_t* a = reinterpret_cast<const uint64_t*>((uintptr_t)p & ~(uintptr_t)7);
  Win w;
  w.w0 = a[0];
  w.w1 = a[1];
  w.w2 = a[2];
  w.w3 = a[3];
  w.w4 = a[4];
  return w;
}
// 8 bytes of the window starting at byte k (0 <= k <= 32)
__device__ __forceinline__ uint64_t win64(const Win& w, uint32_t k) {
  const uint32_t i = k >> 3, sh = (k & 7) * 8;
  uint64_t lo = i == 0 ? w.w0 : i == 1 ? w.w1 : i == 2 ? w.w2 : i == 3 ? w.w3 : w.w4;
  uint64_t hi = i == 0 ? w.w1 : i == 1 ? w.w2 : i == 2 ? w.w3 : i == 3 ? w.w4 : 0;
  return sh ? (lo >> sh) | (hi << (64 - sh)) : lo;
}
__device__ __forceinline__ uint64_t low_bytes_mask(uint32_t nbytes) {  // nbytes in 0..8
  return nbytes >= 8 ? ~0ull : ((1ull << (8 * nbytes)) - 1);
}

// Entry header (block.cc:37-64): three varint32 -- shared key bytes, non_shared key bytes, value length -- then the key suffix and
// the value.  header8 is the fast path's rule: it reads the header from its first 8 bytes h, and fails when the three varints take
// more than 8 bytes, one of them more than 5 (a fifth byte counts modulo 2^32, as in GetVarint32Ptr) or the value length exceeds the
// device format.  header_bytewise reads any header byte by byte from memory.  Each caller decides what a header that fails or exceeds the device's limits means where it reads it: the slow
// path, or an error bit.
struct EntryHeader {
  uint32_t shared, non_shared, vlen, len;  // len: bytes of the header
};
__device__ __forceinline__ bool header8(uint64_t h, EntryHeader& e) {
  if (((h | (h >> 8) | (h >> 16)) & 0x80) == 0) {  // DecodeEntry fast path (block.cc:44-50): three one-byte lengths
    e = EntryHeader{(uint32_t)(h & 0xff), (uint32_t)((h >> 8) & 0xff), (uint32_t)((h >> 16) & 0xff), 3};
    return true;
  }
  uint32_t k = 0, v[3];
  bool ok = true;
#pragma unroll
  for (int q = 0; q < 3; q++) {
    uint32_t x = 0, sft = 0;
    for (;;) {
      if (k >= 8 || sft > 28) {
        ok = false;
        break;
      }
      const uint32_t c = (uint32_t)((h >> (8 * k)) & 0xff);
      k++;
      x |= (c & 127) << sft;
      if (c < 128) break;
      sft += 7;
    }
    v[q] = x;
  }
  e = EntryHeader{v[0], v[1], v[2], k};
  return ok && v[2] <= kMetaVlenMask;
}
// the header at p byte by byte (lengths past 32 bits read as 0xffffffff, which no block can hold); false when a varint is malformed
// or runs past end
__device__ __forceinline__ bool header_bytewise(const uint8_t* p, const uint8_t* end, EntryHeader& e) {
  uint32_t n = 0, v[3];
#pragma unroll
  for (int q = 0; q < 3; q++) {
    uint64_t x;
    const int c = get_varint(p + n, end, &x);
    if (!c) return false;
    v[q] = x > 0xffffffffull ? 0xffffffffu : (uint32_t)x;
    n += (uint32_t)c;
  }
  e = EntryHeader{v[0], v[1], v[2], n};
  return true;
}
// the header at p of an entry inside [p, end), from the 8 bytes h at p or else byte by byte
__device__ __forceinline__ bool read_header(uint64_t h, const uint8_t* p, const uint8_t* end, EntryHeader& e) {
  return header8(h, e) || header_bytewise(p, end, e);
}

// entries in one restart interval [p, end); 0xffffffff on malformed data
__device__ __forceinline__ uint32_t count_interval(const uint8_t* p, const uint8_t* end) {
  uint32_t n = 0;
  while (p < end) {
    EntryHeader e;
    if (!read_header(ld_u64_funnel(p), p, end, e) || e.len > end - p ||
        (uint64_t)e.non_shared + e.vlen > (uint64_t)(end - p) - e.len)
      return 0xffffffffu;
    p += e.len + e.non_shared + e.vlen;
    n++;
  }
  return n;
}

// ---- fused checksum + count + decode: one warp per data block ----------------------------------------------------
// The file image is read exactly once.  A warp
//   1. stages its block in shared memory with 16-byte cp.async copies (the staged copy keeps the file's 16-byte phase,
//      so there is no re-alignment work),
//   2. verifies the block checksum out of shared memory (warp-cooperative XXH3 / CRC32C),
//   3. walks the restart intervals, one lane per interval (the only inherently sequential part: an entry starts
//      where the previous one ends), recording every entry's offset,
//   4. gets its global output position with a decoupled look-back over per-block states (blocks are handed out in
//      ticket order, so every predecessor is already running),
//   5. decodes ONE ENTRY PER LANE: prefix decompression "key = first `shared` bytes of the previous key + suffix" is the
//      map K -> (K & mask(shared)) | (suffix << shared); such maps compose associatively
//      ((m1,D1) then (m2,D2) = (min(m1,m2), (D1 & mask(m2)) | D2)), so a warp inclusive scan rebuilds 32 keys at once,
//   6. stores the columns coalesced (lane i -> entry base + i).
// Blocks outside the fast path's limits (larger than the staging slice, more than 16 restart intervals, more than 16
// entries in an interval) take a slower lane-per-interval path that needs regular intervals (what BlockBuilder writes).
constexpr int kDecWarps = 8;
constexpr int kDecSlice = 4608;            // bytes staged per warp and buffer (block + trailer + phase); larger blocks are read in place
constexpr int kDecVecs = kDecSlice / 16;   // 288
constexpr int kDecRows = 16, kDecRowLen = 16;  // fast path: restart intervals per block, entries per interval
// A warp stages its block with ONE bulk copy (TMA, cp.async.bulk) that completes on the warp's mbarrier.  (Measured: a second slice
// per warp with the next block's copy in flight made the kernel slower -- a ticket taken ahead of time delays the moment its block's
// entry count is published, and the successors' look-backs wait for it.)
struct DecWarpSmem {
  uint4 slice[kDecVecs];
  uint16_t tab[kDecRows * kDecRowLen];  // entry offsets, one row per restart interval
  uint16_t ex[32];                      // entries before each interval
  uint64_t bar;                         // mbarrier: the slice has landed
  uint64_t pad;
};
// 24-byte key K as three little-endian words: masks of its first m bytes
__device__ __forceinline__ void key_mask(uint32_t m, uint64_t* M0, uint64_t* M1, uint64_t* M2) {
  *M0 = low_bytes_mask(m);
  *M1 = m > 8 ? low_bytes_mask(m - 8) : 0;
  *M2 = m > 16 ? low_bytes_mask(m - 16) : 0;
}
// D = S << (8 * shared) over three words
__device__ __forceinline__ void key_shift(uint64_t S0, uint64_t S1, uint64_t S2, uint32_t shared, uint64_t* D0, uint64_t* D1, uint64_t* D2) {
  const uint32_t wsh = shared >> 3, bs = (shared & 7) * 8;
  const uint64_t c0 = bs ? S0 >> (64 - bs) : 0, c1 = bs ? S1 >> (64 - bs) : 0;
  const uint64_t T0 = S0 << bs, T1 = (S1 << bs) | c0, T2 = (S2 << bs) | c1;
  *D0 = wsh == 0 ? T0 : 0;
  *D1 = wsh == 0 ? T1 : wsh == 1 ? T0 : 0;
  *D2 = wsh == 0 ? T2 : wsh == 1 ? T1 : wsh == 2 ? T0 : 0;
}
// columns of one decoded entry from its 24-byte key image
__device__ __forceinline__ void key_columns(uint64_t K0, uint64_t K1, uint64_t K2, uint32_t klen, uint64_t* hi, uint64_t* lo, uint64_t* tr) {
  const uint32_t ulen = klen - 8;
  *hi = bswap64(K0 & low_bytes_mask(ulen));
  *lo = bswap64(ulen > 8 ? K1 & low_bytes_mask(ulen - 8) : 0);
  const uint32_t wsh = ulen >> 3, bs = (ulen & 7) * 8;
  const uint64_t a = wsh == 0 ? K0 : wsh == 1 ? K1 : K2, c = wsh == 0 ? K1 : wsh == 1 ? K2 : 0;
  *tr = bs ? (a >> bs) | (c << (64 - bs)) : a;
}

// Slow path: decodes the restart interval [p, end) sequentially straight into the global columns at e0.
__device__ __noinline__ uint32_t decode_interval_seq(const uint8_t* p, const uint8_t* end, KeyColsMut out, uint64_t e0, uint64_t n_total,
                                                     uint32_t* __restrict__ err) {
  uint64_t K0 = 0, K1 = 0, K2 = 0;
  uint32_t klen = 0, n = 0;
  while (p < end) {
    const Win w = load_win_any(p);
    const uint32_t o = (uint32_t)((uintptr_t)p & 7);
    EntryHeader h;
    if (!read_header(win64(w, o), p, end, h)) {
      atomicOr(err, kErrCorruptBlock);
      break;
    }
    if (h.vlen > kMetaVlenMask) {
      atomicOr(err, kErrValueTooLong);
      break;
    }
    // a header with a multi-byte length: keys longer than the device format, or a header longer than 8 bytes, stop here (three
    // one-byte lengths go on to the key checks below)
    if (h.len > 3 && (h.shared > 64 || h.non_shared > 64 || h.len > 8)) {
      atomicOr(err, (uint64_t)h.shared + h.non_shared > (uint64_t)(kMaxUserKey + 8) ? kErrKeyTooLong : kErrCorruptBlock);
      break;
    }
    const uint32_t shared = h.shared, non_shared = h.non_shared, vlen = h.vlen, hdr = h.len;
    if (shared > klen || shared + non_shared < 8) {
      atomicOr(err, kErrCorruptBlock);
      break;
    }
    if (shared + non_shared > (uint32_t)(kMaxUserKey + 8)) {
      atomicOr(err, kErrKeyTooLong);
      break;
    }
    const uint32_t so = o + hdr;
    uint64_t S0 = win64(w, so), S1 = win64(w, so + 8), S2 = win64(w, so + 16), M0, M1, M2, D0, D1, D2;
    key_mask(non_shared, &M0, &M1, &M2);
    key_shift(S0 & M0, S1 & M1, S2 & M2, shared, &D0, &D1, &D2);
    key_mask(shared, &M0, &M1, &M2);
    K0 = (K0 & M0) | D0;
    K1 = (K1 & M1) | D1;
    K2 = (K2 & M2) | D2;
    klen = shared + non_shared;
    uint64_t hi, lo, tr;
    key_columns(K0, K1, K2, klen, &hi, &lo, &tr);
    if (!device_value_type((uint32_t)(tr & 0xff))) atomicOr(err, kErrBadType);
    else if ((tr & 0xff) == kTypeSingleDeletion) atomicOr(err, (uint32_t)kFlagHasSingleDelete);
    const uint8_t* val = p + hdr + non_shared;
    if ((uint64_t)(end - val) < vlen) {
      atomicOr(err, kErrCorruptBlock);
      break;
    }
    const uint64_t e = e0 + n;
    if (e < n_total) {
      out.pfx[e] = make_ulonglong2(hi, lo);
      out.tr[e] = tr;
      out.vref[e] = (uint64_t)(uintptr_t)val;
      out.meta[e] = make_meta(klen - 8, vlen);
    }
    n++;
    p = val + vlen;
  }
  return n;
}

// the block decoder's per-job arguments
struct DecodeJob {
  const FileDesc* files;
  int nfiles;
  uint32_t nblk;
  uint64_t n_total;  // entries of all runs (rocksdb.num.entries)
  KeyColsMut out;
  unsigned long long* blk_state;  // look-back states, one per block
  uint64_t* run_start;
  uint64_t* total_out;
  uint32_t* err;
};

// Block check, in two steps.  The restart-array footer: the number of restart points and where the entries end; false for a block
// with the data-block hash index (not produced by accepted configs), without restart points or with an array past its end (nr and
// data_end are then meaningless).
__device__ __forceinline__ bool restart_footer(uint32_t foot, uint32_t size, uint32_t* nr, uint32_t* data_end) {
  const uint32_t n = foot & 0x7fffffffu;
  *nr = n;
  *data_end = size - 4 - 4 * n;
  return !((foot >> 31) || n == 0 || 4ull * n + 4 > size);
}
// The trailer (block_fetcher.cc:32-40): compression type, then -- with a checksum type (cksum != 0) -- the block checksum, read from
// the staging slice at shared address sp (kStaged) or from the image p in place.  False with kErrCompressed / kErrChecksum raised.
template <bool kStaged>
__device__ __forceinline__ bool block_trailer_ok(const uint8_t* p, uint32_t sp, uint32_t size, uint32_t cksum, uint32_t xtab, unsigned lane,
                                                 uint32_t* __restrict__ err) {
  const uint32_t ctype = kStaged ? lds8(sp + size) : p[size];
  if (ctype != 0) {
    if (lane == 0) atomicOr(err, kErrCompressed);
    return false;
  }
  if (cksum == 0) return true;
  const uint32_t want = kStaged ? lds32_any(sp + size + 1) : ld_u32(p + size + 1);
  const uint32_t got = kStaged ? staged_block_checksum(cksum, sp, p, size, 0, xtab, lane) : block_checksum_warp(cksum, p, size, 0);
  if (want == got) return true;
  if (lane == 0) atomicOr(err, kErrChecksum);
  return false;
}

// Placement, once the block's entry count is published: the global position of its first entry by a look-back over its
// predecessors, the runs that start at this block (runs without blocks start where the next one does) and, at the last block, the
// job's end.  False when the block writes no entries: rejected (!ok), empty, or past the entries the runs announced.
constexpr uint32_t kLookbackSleepNs = 40;  // look-back poll period: a block that has not published its count is still being walked
__device__ __forceinline__ bool place_block(const DecodeJob& job, uint32_t b, int f, uint32_t cnt, bool ok, unsigned lane, uint64_t* base) {
  *base = lb_exclusive_prefix(job.blk_state, b, cnt, lane, kLookbackSleepNs);
  if (lane == 0) {
    for (int r = f; r >= 0 && job.files[r].gblk_first == b; r--) job.run_start[r] = *base;
    if (b + 1 == job.nblk) {
      for (int r = job.nfiles; r > f && (r == job.nfiles || job.files[r].gblk_first >= job.nblk); r--) job.run_start[r] = *base + cnt;
      *job.total_out = *base + cnt;
    }
  }
  if (!ok || cnt == 0) return false;
  if (*base + cnt > job.n_total) {
    if (lane == 0) atomicOr(job.err, kErrCountMismatch);
    return false;
  }
  return true;
}

// masks of the first m (0..24) key bytes, as a table in shared memory: [m][3]
__device__ __forceinline__ void fill_key_mask_table(uint64_t* tab) {
  for (uint32_t i = threadIdx.x; i < 25 * 3; i += blockDim.x) {
    const uint32_t m = i / 3, wd = i % 3;
    const uint32_t nb = m > 8 * wd ? (m - 8 * wd > 8 ? 8 : m - 8 * wd) : 0;
    tab[i] = low_bytes_mask(nb);
  }
}

// inclusive scan of the prefix-decompression maps (m, D) inside a half-warp, over the first kNW key words only: word w of every
// key of the row is its own suffix when no entry of the row shares more than 8 w bytes with its predecessor
template <int kNW>
__device__ __forceinline__ void scan_key_maps(uint32_t mask_tab, uint32_t i, uint32_t& m, uint64_t& D0, uint64_t& D1, uint64_t& D2) {
#pragma unroll
  for (int d = 1; d < 16; d <<= 1) {
    const uint32_t lm = __shfl_up_sync(0xffffffffu, m, d, 16);
    uint64_t l0 = 0, l1 = 0, l2 = 0;
    if (kNW > 0) l0 = __shfl_up_sync(0xffffffffu, D0, d, 16);
    if (kNW > 1) l1 = __shfl_up_sync(0xffffffffu, D1, d, 16);
    if (kNW > 2) l2 = __shfl_up_sync(0xffffffffu, D2, d, 16);
    if (i >= (uint32_t)d) {
      const uint32_t mt = mask_tab + 24 * m;
      if (kNW > 0) D0 |= l0 & lds64(mt);
      if (kNW > 1) D1 |= l1 & lds64(mt + 8);
      if (kNW > 2) D2 |= l2 & lds64(mt + 16);
      m = lm < m ? lm : m;
    }
  }
}

// Fast path for a block staged in shared memory at address sp (generic pointer p).  Returns false (nothing published) when the
// block is outside the fast path's limits (restart intervals / entries per interval / header length) and has to take
// decode_block_slow.
__device__ __forceinline__ bool decode_block_fast(const DecodeJob& job, DecWarpSmem& ws, uint32_t sp, const uint8_t* p, uint32_t mask_tab,
                                                  uint32_t xtab, const uint8_t* src, uint32_t size, uint32_t cksum, uint32_t b, int f,
                                                  unsigned lane) {
  // shared addresses of the offset table and the interval prefix.  The empty asm makes them opaque: under register pressure
  // the compiler otherwise re-derives them (S2R + address arithmetic) inside the hot loops
  uint32_t stab = (uint32_t)__cvta_generic_to_shared(ws.tab), sex = (uint32_t)__cvta_generic_to_shared(ws.ex);
  asm volatile("" : "+r"(sp), "+r"(stab), "+r"(sex), "+r"(mask_tab));
  uint32_t nr, data_end;
  if (!restart_footer(lds32_any(sp + size - 4), size, &nr, &data_end) || nr > (uint32_t)kDecRows) return false;
  const uint32_t srest = sp + data_end;
  // ---- walk the restart intervals, one lane each, recording entry offsets
  uint32_t c = 0;
  bool bad = false, exotic = false;
  if (lane < nr) {
    const uint32_t r0 = lds32_any(srest + 4 * lane);
    const uint32_t r1 = lane + 1 < nr ? lds32_any(srest + 4 * (lane + 1)) : data_end;
    if (!(r0 <= r1 && r1 <= data_end && (lane != 0 || r0 == 0))) bad = true;
    uint32_t q = r0;
    const uint32_t trow = stab + 2 * (lane * kDecRowLen);
    while (!bad && q < r1) {
      // the common header is three one-byte lengths (DecodeEntry fast path, block.cc:44-50): shared, non_shared, value length
      const uint32_t a = sp + q;
      const uint32_t h0 = lds8(a), h1 = lds8(a + 1), h2 = lds8(a + 2);
      uint32_t adv;
      if (((h0 | h1 | h2) & 0x80u) == 0) {
        adv = 3 + h1 + h2;
      } else {
        EntryHeader e;
        if (!header8(lds64_any(a), e)) {
          exotic = true;
          break;
        }
        adv = e.len + e.non_shared + e.vlen;
      }
      if (adv > r1 - q) {
        bad = true;
        break;
      }
      if (c < (uint32_t)kDecRowLen) sts16(trow + 2 * c, q);
      q += adv;
      c++;
    }
  }
  if (__ballot_sync(0xffffffffu, exotic || (!bad && c > (uint32_t)kDecRowLen))) return false;  // unusual block: slow path
  bool ok = true;
  if (__ballot_sync(0xffffffffu, bad)) {
    if (lane == 0) atomicOr(job.err, kErrCorruptBlock);
    ok = false;
    c = 0;
  }
  const uint32_t inc = warp_incl_scan(c);
  const uint32_t cnt = __shfl_sync(0xffffffffu, inc, 31);
  if (lane <= nr) sts16(sex + 2 * lane, inc - c);  // ex[nr] = cnt
  if (lane == 0) lb_publish(job.blk_state, b, cnt);  // successors can look back while this warp checksums
  ok = block_trailer_ok<true>(p, sp, size, cksum, xtab, lane, job.err) && ok;
  uint64_t base;
  if (!place_block(job, b, f, cnt, ok, lane, &base)) return true;
  __syncwarp();
  // ---- one entry per lane, one restart interval per half-warp; keys by a segmented scan over the decompression maps
  for (uint32_t row0 = 0; row0 < nr; row0 += 2) {
    const uint32_t row = row0 + (lane >> 4), i = lane & 15;
    uint32_t ex0 = 0, rc = 0;
    if (row < nr) {
      ex0 = lds16(sex + 2 * row);
      rc = lds16(sex + 2 * row + 2) - ex0;
    }
    const bool valid = i < rc;
    uint32_t m = 24, klen = 0, vlen = 0, voff = 0, shared = 0;
    uint64_t D0 = 0, D1 = 0, D2 = 0;
    bool ebad = false;
    if (valid) {
      const uint32_t q = lds16(stab + 2 * (row * kDecRowLen + i));
      uint32_t non_shared, hdr;
      {
        const uint32_t a = sp + q;
        const uint32_t h0 = lds8(a), h1 = lds8(a + 1), h2 = lds8(a + 2);
        if (((h0 | h1 | h2) & 0x80u) == 0) {
          shared = h0;
          non_shared = h1;
          vlen = h2;
          hdr = 3;
        } else {
          EntryHeader e;
          header8(lds64_any(a), e);  // validated by the walk
          shared = e.shared;
          non_shared = e.non_shared;
          vlen = e.vlen;
          hdr = e.len;
        }
      }
      if (shared + non_shared < 8) {
        atomicOr(job.err, kErrCorruptBlock);
        ebad = true;
      } else if (shared + non_shared > (uint32_t)(kMaxUserKey + 8)) {
        atomicOr(job.err, kErrKeyTooLong);
        ebad = true;
        klen = shared + non_shared;  // the successor's `shared` is still bounded by this length
      } else {
        // key suffix: non_shared (<= 24) bytes after the header, from four aligned words
        const uint32_t ks = sp + q + hdr, al = ks & ~7u, sft = (ks & 7) * 8;
        const uint64_t A0 = lds64(al), A1 = lds64(al + 8), A2 = lds64(al + 16), A3 = lds64(al + 24);
        const uint32_t mt = mask_tab + 24 * non_shared;
        key_shift(shr128(A0, A1, sft) & lds64(mt), shr128(A1, A2, sft) & lds64(mt + 8), shr128(A2, A3, sft) & lds64(mt + 16), shared, &D0,
                  &D1, &D2);
        m = shared;
        klen = shared + non_shared;
        voff = q + hdr + non_shared;
      }
    }
    // `shared` is bounded by the previous entry's key length (0 before a restart point)
    uint32_t pk = __shfl_up_sync(0xffffffffu, klen, 1, 16);
    uint32_t pbad = __shfl_up_sync(0xffffffffu, (uint32_t)ebad, 1, 16);
    if (i == 0) pk = 0, pbad = 0;
    if (valid && !ebad && !pbad && shared > pk) {  // (after a rejected entry the bound is unknown: already an error)
      atomicOr(job.err, kErrCorruptBlock);
      ebad = true;
    }
    // inclusive scan of (m, D) inside the half-warp: left = earlier entries, right = own accumulated map.  Only the key words that
    // some entry of these two rows shares with its predecessor take part (sorted keys usually share a few leading bytes only).
    {
      const uint32_t mx = __reduce_max_sync(0xffffffffu, shared);
      if (mx == 0) {
      } else if (mx <= 8) scan_key_maps<1>(mask_tab, i, m, D0, D1, D2);
      else if (mx <= 16) scan_key_maps<2>(mask_tab, i, m, D0, D1, D2);
      else scan_key_maps<3>(mask_tab, i, m, D0, D1, D2);
    }
    if (valid && !ebad) {  // the interval's first entry has shared == 0, so D is the whole key
      uint64_t hi, lo, tr;
      key_columns(D0, D1, D2, klen, &hi, &lo, &tr);
      if (!device_value_type((uint32_t)(tr & 0xff))) atomicOr(job.err, kErrBadType);
      else if ((tr & 0xff) == kTypeSingleDeletion) atomicOr(job.err, (uint32_t)kFlagHasSingleDelete);
      const uint64_t e = base + ex0 + i;
      job.out.pfx[e] = make_ulonglong2(hi, lo);
      job.out.tr[e] = tr;
      job.out.vref[e] = (uint64_t)(uintptr_t)(src + voff);
      job.out.meta[e] = make_meta(klen - 8, vlen);
    }
  }
  return true;
}

// Slow path straight from the image: lane per restart interval, sequential decode, regular intervals required.
__device__ __noinline__ void decode_block_slow(const DecodeJob job, const uint8_t* p, uint32_t size, uint32_t cksum, uint32_t b, int f,
                                               unsigned lane) {
  uint32_t cnt = 0, nr = 0, data_end = 0, first = 0;
  bool ok = block_trailer_ok<false>(p, 0, size, cksum, 0, lane, job.err);
  if (ok && !restart_footer(ld_u32(p + size - 4), size, &nr, &data_end)) {
    if (lane == 0) atomicOr(job.err, kErrCorruptBlock);
    ok = false;
  }
  const uint8_t* restarts = p + data_end;
  if (ok) {
    uint32_t irregular = 0;
    for (uint32_t j0 = 0; j0 < nr; j0 += 32) {
      const uint32_t j = j0 + lane;
      uint32_t c = 0;
      if (j < nr) {
        const uint32_t r0 = ld_u32(restarts + 4ull * j);
        const uint32_t r1 = j + 1 < nr ? ld_u32(restarts + 4ull * (j + 1)) : data_end;
        c = (r0 <= r1 && r1 <= data_end && (j != 0 || r0 == 0)) ? count_interval(p + r0, p + r1) : 0xffffffffu;
        if (c == 0xffffffffu) {
          atomicOr(job.err, kErrCorruptBlock);
          c = 0;
          irregular = 1;
        }
      }
      if (j0 == 0) first = __shfl_sync(0xffffffffu, c, 0);
      if (j + 1 < nr && c != first) irregular = 1;
      if (j + 1 == nr && c > first) irregular = 1;
      cnt += c;
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
    if (__ballot_sync(0xffffffffu, irregular != 0)) {
      if (lane == 0) atomicOr(job.err, kErrIrregularRestarts);
      ok = false;  // positions inside the block are not derivable
    }
  }
  if (!ok) cnt = 0;  // a rejected block contributes no entries (the job fails anyway)
  if (lane == 0) lb_publish(job.blk_state, b, cnt);
  uint64_t base;
  if (!place_block(job, b, f, cnt, ok, lane, &base)) return;
  for (uint32_t j0 = 0; j0 < nr; j0 += 32) {
    const uint32_t j = j0 + lane;
    if (j < nr) {
      const uint32_t r0 = ld_u32(restarts + 4ull * j);
      const uint32_t r1 = j + 1 < nr ? ld_u32(restarts + 4ull * (j + 1)) : data_end;
      decode_interval_seq(p + r0, p + r1, job.out, base + (uint64_t)j * first, job.n_total, job.err);
    }
  }
}

constexpr int kDecCtasPerSm = 4;  // 64 registers (a small spill), but 32 independent warps per SM
__global__ void __launch_bounds__(kDecWarps * 32, kDecCtasPerSm)
block_decode_fused_kernel(const DecodeJob job, const uint64_t* __restrict__ blk_off, const uint32_t* __restrict__ blk_size, uint32_t verify,
                          uint32_t* ticket, const uint8_t* __restrict__ arena) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ uint64_t s_mask[25 * 3];
  __shared__ XxhLaneTab s_xtab;
  const unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  DecWarpSmem& ws = reinterpret_cast<DecWarpSmem*>(smem)[w];
  fill_key_mask_table(s_mask);
  fill_xxh_lane_tab(&s_xtab);
  const uint32_t mask_tab = (uint32_t)__cvta_generic_to_shared(s_mask), xtab = (uint32_t)__cvta_generic_to_shared(&s_xtab);
  const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&ws.bar);
  const uint32_t slice = (uint32_t)__cvta_generic_to_shared(&ws.slice[0]);
  if (lane == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();  // tables and barriers ready
  uint32_t parity = 0;
  for (;;) {
    // one ticket per warp and block: blocks are started in ticket order (the look-back needs every predecessor running),
    // and warps stay independent of each other -- no CTA-wide barrier couples a warp to its neighbours' look-back waits
    uint32_t tk = 0;
    if (lane == 0) tk = atomicAdd(ticket, 1u);
    const uint32_t b = __shfl_sync(0xffffffffu, tk, 0);
    if (b >= job.nblk) break;
    const uint64_t bo = blk_off[b];
    const int f = (int)(bo >> kBlkFileShift);
    // (an inflated block sits in the arena; its checksum was verified over the stored bytes by verify_compressed_kernel)
    const bool inflated = (bo & kBlkArenaBit) != 0;
    const uint8_t* src = inflated ? arena + (bo & (kBlkArenaBit - 1)) : job.files[f].base + (bo & kBlkOffMask);
    const uint32_t size = blk_size[b], cksum = inflated || !verify ? 0u : job.files[f].cksum;
    if (size == 0) {  // outside the sub-compaction's key range (index_decode_kernel): an empty block, nothing is read
      if (lane == 0) lb_publish(job.blk_state, b, 0);
      // its position only matters where a run starts / the stream ends; every 32nd skipped block still resolves its prefix so that
      // the look-back of the next real block does not have to walk a whole skipped stretch
      uint64_t base;
      if (job.files[f].gblk_first == b || b + 1 == job.nblk || (b & 31u) == 31u) place_block(job, b, f, 0, true, lane, &base);
      continue;
    }
    const uintptr_t a0 = (uintptr_t)src & ~(uintptr_t)15;
    const uint32_t shift = (uint32_t)((uintptr_t)src - a0);
    const uint32_t nvec = (shift + size + 5 + 15) >> 4;
    bool done = false;
    if (nvec <= (uint32_t)kDecVecs - 3 && size >= 8) {  // parse windows may run 32 bytes past the trailer
      if (lane == 0) {
        // every lane finished reading the slice (__syncwarp below); order those generic-proxy reads before the async-proxy write
        fence_async_smem();
        mbar_expect_tx(bar, nvec * 16);
        bulk_g2s(slice, reinterpret_cast<const void*>(a0), nvec * 16, bar);
      }
      mbar_wait(bar, parity);
      parity ^= 1;
      done = decode_block_fast(job, ws, slice + shift, reinterpret_cast<const uint8_t*>(&ws.slice[0]) + shift, mask_tab, xtab, src, size, cksum,
                               b, f, lane);
      __syncwarp();  // all lanes are done with the slice before the next block overwrites it
    }
    if (!done) decode_block_slow(job, src, size, cksum, b, f, lane);
  }
}

__global__ void gather_values_kernel(KeyCols in, const uint64_t* __restrict__ dst_off, uint8_t* __restrict__ dst) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < in.n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint8_t* s = (const uint8_t*)(uintptr_t)in.vref[i];
    uint32_t n = meta_vlen(in.meta[i]);
    uint8_t* d = dst + dst_off[i];
    for (uint32_t t = 0; t < n; t++) d[t] = s[t];
  }
}
// TableBuilder side with host records: entry i = internal key (klen[i] bytes) followed by its value, at arena + offs[i]; the next
// entry starts where the value ends.  One thread per entry: the key columns + a value reference into the (device) arena.
__global__ void kv_to_columns_kernel(const uint8_t* __restrict__ arena, const uint64_t* __restrict__ offs, const uint32_t* __restrict__ klens,
                                     uint64_t n, KeyColsMut out, uint32_t* __restrict__ err) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t o = offs[i], e = offs[i + 1];
    const uint32_t kl = klens[i];
    uint64_t hi = 0, lo = 0, tr = 0;
    uint32_t ulen = 0, vlen = 0;
    if (kl < 8 || o + kl > e) {
      atomicOr(err, (uint32_t)kErrCorruptBlock);
    } else if (kl > (uint32_t)kMaxUserKey + 8) {
      atomicOr(err, (uint32_t)kErrKeyTooLong);
    } else if (e - o - kl > kMetaVlenMask) {
      atomicOr(err, (uint32_t)kErrValueTooLong);
    } else {
      ulen = kl - 8;
      vlen = (uint32_t)(e - o - kl);
      const uint8_t* k = arena + o;
      for (uint32_t t = 0; t < 8; t++) hi = (hi << 8) | (t < ulen ? k[t] : 0);
      for (uint32_t t = 8; t < 16; t++) lo = (lo << 8) | (t < ulen ? k[t] : 0);
      tr = ld_u64(k + ulen);
      if (!device_value_type((uint32_t)(tr & 0xff))) atomicOr(err, (uint32_t)kErrBadType);  // (the table encoder itself is type-blind)
    }
    out.pfx[i] = make_ulonglong2(hi, lo);
    out.tr[i] = tr;
    out.vref[i] = (uint64_t)(uintptr_t)(arena + o + kl);
    out.meta[i] = make_meta(ulen, vlen);
  }
}
void launch_kv_to_columns(const uint8_t* arena, const uint64_t* offs, const uint32_t* klens, uint64_t n, KeyColsMut out, uint32_t* err,
                          int sms, cudaStream_t st) {
  if (n == 0) return;
  const uint64_t g = (n + 255) / 256;
  kv_to_columns_kernel<<<(unsigned)(g > (unsigned)sms * 16 ? (unsigned)sms * 16 : g), 256, 0, st>>>(arena, offs, klens, n, out, err);
}
__global__ void meta_vlen_kernel(const uint32_t* __restrict__ meta, uint64_t n, uint32_t* __restrict__ vlen) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    vlen[i] = meta_vlen(meta[i]);
}

// ---------------------------------------------------------------------------------------------- compressed data blocks
// UncompressBlockData (table/format.cc:511) for kZlibCompression, the codec this image can pin against (zlib is the only compression
// library here; the reference is built with -DZLIB for the oracle).  Three small passes in front of the block decoder:
//   block_usize_kernel        thread per block: compression type byte; for a compressed block the announced uncompressed size
//                             (varint32 prefix, compress_format_version 2) -> its slot size in the arena
//   (exclusive scan)          arena offsets
//   verify_compressed_kernel  warp per compressed block: the block checksum covers the STORED bytes (block_fetcher.cc:32-40)
//   inflate_blocks_kernel     warp per compressed block: lane 0 inflates it (inflate_rules.h) into a shared-memory window, the warp
//                             copies it with an uncompressed trailer to its arena slot, then the block's handle is redirected there.
// A data block may announce 4 <= u < 2^31 bytes: 4 is the smallest block the block decoder reads (handle_in_file), the rule a stored
// block meets too; below 2^31 a slot size and blk_size fit 32 bits.  An index block has its own bounds (api.cu input_index_block).
__device__ __forceinline__ bool compressed_prefix(const uint8_t* p, uint32_t size, uint32_t* usize, uint32_t* hdr) {
  uint64_t u = 0;
  const int c = inf_size_prefix(p, size, &u);
  if (c == 0 || u > 0x7fffffffull) return false;
  *usize = (uint32_t)u;
  *hdr = (uint32_t)c;
  return true;
}
// the bytes a compressed block takes in the arena: the inflated block and its trailer, to 16 bytes; 0: its size prefix is refused
__device__ __forceinline__ uint32_t arena_slot(const uint8_t* p, uint32_t size, uint32_t& u, uint32_t& h) {
  uint32_t s = 0;
  if (compressed_prefix(p, size, &u, &h) && u >= 4) s = (u + 5 + 15) & ~15u;
  return s;
}
__global__ void block_usize_kernel(const FileDesc* __restrict__ files, const uint64_t* __restrict__ blk_off, const uint32_t* __restrict__ blk_size,
                                   uint32_t nblk, uint32_t* __restrict__ slot, uint32_t* __restrict__ err) {
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nblk) return;
  uint32_t s = 0;
  const uint32_t size = blk_size[b];
  if (size != 0) {
    const uint64_t bo = blk_off[b];
    const uint8_t* p = files[bo >> kBlkFileShift].base + (bo & kBlkOffMask);
    const uint8_t ctype = p[size];
    if (ctype == kZlibCompressionType) {
      uint32_t u, h;
      s = arena_slot(p, size, u, h);
      if (s == 0) atomicOr(err, kErrCorruptBlock);
    } else if (ctype != 0) {
      atomicOr(err, kErrCompressed);  // a codec the device does not decode
    }
  }
  slot[b] = s;
}
__global__ void verify_compressed_kernel(const FileDesc* __restrict__ files, const uint64_t* __restrict__ blk_off, const uint32_t* __restrict__ blk_size,
                                         const uint32_t* __restrict__ slot, uint32_t nblk, uint32_t* __restrict__ err) {
  const uint32_t lane = threadIdx.x & 31;
  for (uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < nblk; b += (gridDim.x * blockDim.x) >> 5) {
    if (slot[b] == 0) continue;
    const uint64_t bo = blk_off[b];
    const FileDesc& fd = files[bo >> kBlkFileShift];
    if (fd.cksum == 0) continue;
    const uint8_t* p = fd.base + (bo & kBlkOffMask);
    const uint32_t size = blk_size[b];
    const uint32_t got = block_checksum_warp(fd.cksum, p, size, p[size]);
    if (lane == 0 && got != ld_u32(p + size + 1)) atomicOr(err, kErrChecksum);
  }
}
// One WARP per compressed block.  Inflating is control flow all the way down (a different path per symbol), so 32 blocks in the 32
// lanes of a warp serialise on each other -- slow whatever the tables cost, because the lanes' byte-by-byte
// match copies through global memory (a dependent L2 round trip per byte) take turns.  Here lane 0 runs the decoder with its tables
// AND its output window in shared memory (a match copy is a shared-memory load + store), and the whole warp then moves the inflated
// block to the arena with coalesced stores; other warps of the SM hide the single lane's latency.  Blocks larger than the window
// are inflated straight into the arena.
constexpr int kInflateWarps = 8;
constexpr uint32_t kInflateWindow = 6144;  // bytes of inflated block a warp keeps in shared memory (block_size 4096 + one entry fits)
struct InflateWarpSmem {
  InfWork wk;
  uint8_t pad[4];  // keeps the window 16-byte aligned
  uint8_t out[kInflateWindow + 16];
};
static_assert(sizeof(InflateWarpSmem) % 16 == 0 && (sizeof(InfWork) + 4) % 16 == 0, "warp slices and windows stay 16-byte aligned");
static_assert(3 * (sizeof(InflateWarpSmem) * kInflateWarps + 1024) <= 227 * 1024, "three inflate CTAs per SM");
__global__ void __launch_bounds__(kInflateWarps * 32)
inflate_blocks_kernel(const FileDesc* __restrict__ files, uint64_t* __restrict__ blk_off, uint32_t* __restrict__ blk_size,
                      const uint32_t* __restrict__ slot, const uint64_t* __restrict__ slot_off, uint32_t nblk, uint8_t* __restrict__ arena,
                      uint32_t* __restrict__ err) {
  extern __shared__ __align__(16) uint8_t inflate_smem[];
  const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  InflateWarpSmem& ws = reinterpret_cast<InflateWarpSmem*>(inflate_smem)[w];
  for (uint32_t b = blockIdx.x * kInflateWarps + w; b < nblk; b += gridDim.x * kInflateWarps) {
    if (slot[b] == 0) continue;
    const uint64_t bo = blk_off[b];
    const uint8_t* p = files[bo >> kBlkFileShift].base + (bo & kBlkOffMask);
    const uint32_t size = blk_size[b];
    uint32_t u = 0, h = 0;
    const uint32_t slot_bytes = arena_slot(p, size, u, h);
    uint8_t* dst = arena + slot_off[b];
    const bool windowed = u <= kInflateWindow;
    long n = 0;
    if (lane == 0) n = inflate_raw(p + h, size - h, windowed ? ws.out : dst, u, &ws.wk);
    n = __shfl_sync(0xffffffffu, n, 0);
    if (n != (long)u) {
      if (lane == 0) {
        atomicOr(err, kErrCorruptBlock);
        blk_size[b] = 0;  // (an empty block: the job fails anyway)
      }
      __syncwarp();
      continue;
    }
    __syncwarp();
    if (windowed) {  // slots are 16-byte aligned
      if (lane == 0) {
        ws.out[u] = 0;  // trailer of an uncompressed block; the checksum bytes are never read (cksum = 0 for arena blocks)
        ws.out[u + 1] = ws.out[u + 2] = ws.out[u + 3] = ws.out[u + 4] = 0;
      }
      __syncwarp();
      const uint32_t nvec = slot_bytes >> 4;
      const uint4* src4 = reinterpret_cast<const uint4*>(ws.out);
      uint4* dst4 = reinterpret_cast<uint4*>(dst);
      for (uint32_t i = lane; i < nvec; i += 32) dst4[i] = src4[i];
    } else if (lane == 0) {
      dst[u] = 0;
      dst[u + 1] = dst[u + 2] = dst[u + 3] = dst[u + 4] = 0;
    }
    if (lane == 0) {
      blk_off[b] = (bo & ~kBlkOffMask) | kBlkArenaBit | slot_off[b];
      blk_size[b] = u;
    }
    __syncwarp();  // the window is free for the next block
  }
}
void launch_block_usize(const FileDesc* files_dev, const uint64_t* blk_off, const uint32_t* blk_size, uint32_t nblk, uint32_t* slot, uint32_t* err,
                        cudaStream_t st, uint64_t* launches) {
  if (nblk == 0) return;
  block_usize_kernel<<<(nblk + 255) / 256, 256, 0, st>>>(files_dev, blk_off, blk_size, nblk, slot, err);
  *launches += 1;
}
void launch_inflate_blocks(const FileDesc* files_dev, uint64_t* blk_off, uint32_t* blk_size, const uint32_t* slot, const uint64_t* slot_off,
                           uint32_t nblk, uint8_t* arena, uint32_t verify, uint32_t* err, int sms, cudaStream_t st, uint64_t* launches) {
  if (nblk == 0) return;
  if (verify) {
    unsigned g = (nblk + 7) / 8;
    if (g > (unsigned)sms * 8) g = (unsigned)sms * 8;
    verify_compressed_kernel<<<g, 256, 0, st>>>(files_dev, blk_off, blk_size, slot, nblk, err);
  }
  static PerDeviceFlag attr;
  const uint64_t dev_bit = attr.bit_of_current_device();
  const size_t smem = sizeof(InflateWarpSmem) * kInflateWarps;
  if (!attr.is_set(dev_bit)) {
    cudaFuncSetAttribute(inflate_blocks_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr.set(dev_bit);
  }
  unsigned grid = (nblk + kInflateWarps - 1) / kInflateWarps;
  if (grid > (unsigned)sms * 3u) grid = (unsigned)sms * 3u;  // three CTAs (24 warps) per SM, each warp walks its share of the blocks
  inflate_blocks_kernel<<<grid, kInflateWarps * 32, smem, st>>>(files_dev, blk_off, blk_size, slot, slot_off, nblk, arena, err);
  *launches += verify ? 2 : 1;
}

// ---------------------------------------------------------------------------------------------- host launchers
void launch_index_decode(const FileDesc* files_dev, int nfiles, uint32_t max_blocks_per_file, uint64_t* blk_off, uint32_t* blk_size,
                         BoundKey start, uint32_t has_start, BoundKey end, uint32_t has_end, uint32_t* err, cudaStream_t st, uint64_t* launches) {
  dim3 grid((max_blocks_per_file + 255) / 256 ? (max_blocks_per_file + 255) / 256 : 1, nfiles);
  if (grid.x > 1024) grid.x = 1024;
  index_decode_kernel<<<grid, 256, 0, st>>>(files_dev, nfiles, blk_off, blk_size, start, has_start, end, has_end, err);
  *launches += 1;
}
void launch_block_decode_fused(const FileDesc* files_dev, int nfiles, const uint64_t* blk_off, const uint32_t* blk_size, uint32_t nblk,
                               uint32_t verify, uint64_t n_total, KeyColsMut out, unsigned long long* blk_state, uint32_t* ticket,
                               uint64_t* run_start, uint64_t* total_out, uint32_t* err, int sms, cudaStream_t st, uint64_t* launches, const uint8_t* arena) {
  const int smem = kDecWarps * (int)sizeof(DecWarpSmem);
  static_assert(kDecCtasPerSm * (kDecWarps * sizeof(DecWarpSmem) + 4096) <= 227 * 1024, "four decode CTAs must fit one SM");
  static PerDeviceFlag attr;
  const uint64_t dev_bit = attr.bit_of_current_device();
  if (!attr.is_set(dev_bit)) {
    cudaFuncSetAttribute(block_decode_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr.set(dev_bit);
  }
  const unsigned per = kDecWarps;
  unsigned want = (nblk + per - 1) / per, cap = (unsigned)sms * (unsigned)kDecCtasPerSm;
  const unsigned grid = want < cap ? (want ? want : 1) : cap;
  const DecodeJob job{files_dev, nfiles, nblk, n_total, out, blk_state, run_start, total_out, err};
  block_decode_fused_kernel<<<grid, kDecWarps * 32, smem, st>>>(job, blk_off, blk_size, verify, ticket, arena);
  *launches += 1;
}
void launch_gather_values(KeyCols in, const uint64_t* dst_off, uint8_t* dst, cudaStream_t st) {
  if (in.n == 0) return;
  unsigned g = (unsigned)((in.n + 255) / 256);
  gather_values_kernel<<<g > 4096 ? 4096 : g, 256, 0, st>>>(in, dst_off, dst);
}
void launch_meta_vlen(const uint32_t* meta, uint64_t n, uint32_t* vlen, cudaStream_t st) {
  if (n == 0) return;
  unsigned g = (unsigned)((n + 255) / 256);
  meta_vlen_kernel<<<g > 4096 ? 4096 : g, 256, 0, st>>>(meta, n, vlen);
}

// ---- paranoid_file_checks (OutputValidator, db/output_validator.cc:31-69 + compaction_job.cc:829-853): the reference hashes every key
// and value while writing and again while re-reading the finished file; here the re-read columns are compared with the written ones
// directly (equal sequences have equal rolling hashes, and a difference is found even where two hashes would collide).
__global__ void compare_columns_kernel(KeyCols a, KeyCols b, uint64_t n, uint32_t* __restrict__ err) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const ulonglong2 pa = a.pfx[i], pb = b.pfx[i];
    const uint32_t ma = a.meta[i];
    bool bad = pa.x != pb.x || pa.y != pb.y || a.tr[i] != b.tr[i] || ma != b.meta[i];
    if (!bad) {
      // values: eight bytes per step, each side read as two aligned words (the values sit at any alignment inside the images)
      const uint32_t vlen = meta_vlen(ma);
      const uint8_t* x = reinterpret_cast<const uint8_t*>((uintptr_t)a.vref[i]);
      const uint8_t* y = reinterpret_cast<const uint8_t*>((uintptr_t)b.vref[i]);
      uint32_t t = 0;
      uint64_t diff = 0;
      for (; t + 8 <= vlen; t += 8) diff |= ld_u64_funnel(x + t) ^ ld_u64_funnel(y + t);
      for (; t < vlen; t++) diff |= (uint64_t)(x[t] ^ y[t]);
      bad = diff != 0;
    }
    if (bad) atomicOr(err, (uint32_t)kErrParanoid);
  }
}
__global__ void flip_byte_kernel(uint8_t* p) { *p ^= 0x40; }
void launch_flip_byte(uint8_t* p, cudaStream_t st) { flip_byte_kernel<<<1, 1, 0, st>>>(p); }
void launch_compare_columns(KeyCols written, KeyCols reread, uint64_t n, uint32_t* err, int sms, cudaStream_t st, uint64_t* launches) {
  if (n == 0) return;
  const uint64_t blocks = (n + 255) / 256;
  compare_columns_kernel<<<(unsigned)(blocks < (unsigned)sms * 16 ? blocks : (unsigned)sms * 16), 256, 0, st>>>(written, reread, n, err);
  *launches += 1;
}

}  // namespace b200c
