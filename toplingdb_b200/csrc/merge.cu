// toplingdb_b200/csrc/merge.cu — the k-way merge with the compaction-iterator rules, on the device.
//
// Replaces CompactionMergingIterTmpl (table/compaction_merging_iterator.cc:10-402; heap of children, util/heap.h)
// + BytewiseCompareInternalKey (db/dbformat.h:1057-1097) + CompactionIterator::NextFromInput / PrepareOutput
// (db/compaction/compaction_iterator.cc:475-1087,1274-1341) for kTypeValue, kTypeDeletion and kTypeSingleDeletion entries.
//
// Kernels:
//   merge_partition_grouped_kernel (<= 16 runs) / merge_partition_kernel (<= 64 runs)
//                           one warp per tile boundary: exact k-way merge-path split (multi-sequence selection against
//                           a common pivot); with few runs a group of lanes per run probes several points per step
//   merge_tiles_kernel      one CTA per tile of kMergeTile merged entries, in phases:
//                             tile_segments      segment table and the tile's predecessor
//                             tile_load          coalesced load of the k segments into shared memory
//                             tile_merge_rounds  log2(k) rounds of pairwise merge-path merges (in place through registers)
//                             sd_walk_tile       serial walk of the user keys that hold a SingleDelete (kSD variant)
//                             tile_rules         compaction-iterator rules per merged position
//                             tile_ranks         tile-local output ranks; the tile's count is published for the look-back
//                             tile_compact       survivors in output order, in place
//                             tile_gather        value references of the survivors; then the look-back resolves the offset
//                             tile_store         coalesced write of the (key, value-ref) records, entry sizes, TileStat
//                             tile_count         CompactionIterationStats partial sums
// HBM-bound: algorithmic bytes = 36 B read per input entry + 36 B written per surviving entry.
#include "common.cuh"
#include "group_rules.h"
#include "kernels.h"

namespace b200c {

constexpr int kMT = kMergeTile;
constexpr int kMThreads = 256;
constexpr int kMV = kMT / kMThreads;  // 8 merged entries per thread
constexpr uint32_t kPartGroupedMaxRuns = 16;  // runs that merge_partition_grouped_kernel takes (a group of at least 2 lanes each)

__device__ __forceinline__ Key load_key(const KeyCols& c, uint64_t i) {
  Key k;
  ulonglong2 p = c.pfx[i];
  k.hi = p.x;
  k.lo = p.y;
  k.tr = c.tr[i];
  k.ulen = meta_ulen(c.meta[i]);
  return k;
}

// number of elements of run [base+lo, base+hi) that precede pivot X in the total order (key, run index):
// before_equal == true counts elements <= X (runs with a smaller index than the pivot's run)
__device__ __forceinline__ uint64_t count_before(const KeyCols& c, uint64_t base, uint64_t lo, uint64_t hi, const Key& x,
                                                 bool before_equal) {
  while (lo < hi) {
    uint64_t mid = lo + ((hi - lo) >> 1);
    Key e = load_key(c, base + mid);
    bool precedes = before_equal ? !ikey_less(x, e) : ikey_less(e, x);
    if (precedes) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(128)
merge_partition_kernel(KeyCols in, RunBounds runs, uint32_t nruns, uint64_t n_total, uint64_t ntiles,
                       uint64_t* __restrict__ splits, uint32_t* __restrict__ err) {
  const unsigned lane = threadIdx.x & 31;
  const uint64_t b = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b > ntiles) return;
  uint64_t d = b * (uint64_t)kMergeNominal;
  if (d > n_total) d = n_total;
  uint64_t base[2], lo[2], hi[2];
#pragma unroll
  for (int s = 0; s < 2; s++) {
    uint32_t r = lane + 32 * s;
    base[s] = r < nruns ? runs.begin[r] : 0;
    uint64_t n = r < nruns ? runs.end[r] - runs.begin[r] : 0;
    lo[s] = (d == n_total) ? n : 0;
    hi[s] = (d == 0) ? 0 : n;
  }
  for (int guard = 0; guard < 64 * 70; guard++) {
    // widest bracket decides the pivot run
    unsigned long long best = 0;
#pragma unroll
    for (int s = 0; s < 2; s++) {
      unsigned long long wdt = hi[s] - lo[s];
      unsigned long long enc = (wdt << 7) | (unsigned long long)(lane + 32 * s);
      if (wdt && enc > best) best = enc;
    }
#pragma unroll
    for (int dd = 16; dd; dd >>= 1) {
      unsigned long long o = __shfl_xor_sync(0xffffffffu, best, dd);
      if (o > best) best = o;
    }
    if (best == 0) break;
    const uint32_t p = (uint32_t)(best & 127);
    const int ps = p >> 5, pl = p & 31;
    uint64_t m = ps ? (lo[1] + ((hi[1] - lo[1]) >> 1)) : (lo[0] + ((hi[0] - lo[0]) >> 1));
    m = __shfl_sync(0xffffffffu, m, pl);
    uint64_t pbase = __shfl_sync(0xffffffffu, ps ? base[1] : base[0], pl);
    const Key x = load_key(in, pbase + m);
    uint64_t c[2], sum = 0;
#pragma unroll
    for (int s = 0; s < 2; s++) {
      uint32_t r = lane + 32 * s;
      if (r == p) c[s] = m;
      else if (r < nruns) c[s] = count_before(in, base[s], lo[s], hi[s], x, r < p);
      else c[s] = 0;
      sum += c[s];
    }
#pragma unroll
    for (int dd = 16; dd; dd >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, dd);
    const bool x_before = sum < d;  // pivot is among the first d elements
#pragma unroll
    for (int s = 0; s < 2; s++) {
      uint32_t r = lane + 32 * s;
      if (r >= nruns) continue;
      if (x_before) lo[s] = (r == p) ? m + 1 : c[s];
      else hi[s] = (r == p) ? m : c[s];
    }
  }
  uint64_t tot = lo[0] + lo[1];
#pragma unroll
  for (int dd = 16; dd; dd >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, dd);
  if (tot != d && lane == 0) atomicOr(err, kErrKeyOrder);
  // (tile cuts are not aligned to user keys here: SingleDeletes with more than 16 runs stay on the CPU)
  if (lane == 0 && (*reinterpret_cast<volatile uint32_t*>(err) & (uint32_t)kFlagHasSingleDelete)) atomicOr(err, (uint32_t)kErrGroupTooLong);
#pragma unroll
  for (int s = 0; s < 2; s++) {
    uint32_t r = lane + 32 * s;
    if (r < nruns) splits[b * nruns + r] = lo[s];
  }
}

// The same split for up to 16 runs with ALL lanes busy: run r is owned by a group of g = 32 / pow2(nruns) lanes that
// probe g points of its bracket per step (a (g+1)-ary search), which divides the depth of the dependent-load chain --
// the whole cost of this kernel -- by log2(g + 1).
//
// Two levels.  A split over 4.8 M-entry runs costs ~200 dependent DRAM round trips when it starts from the whole runs.  So the
// selection first runs over every kPartStride-th entry of each run (the "samples": a few MB in total, served by the L2 after the
// first touches), twice, for two sample ranks that bracket the wanted rank, and the exact selection then starts from brackets of
// about kPartStride * (2k + 1) entries in total:
//   sample j of run r = its entry kPartStride * j;  y = a sample, t_r = samples of run r that precede y, c_r = entries of run r
//   that precede y.  Entry kPartStride * t_r does not precede y and entry kPartStride * (t_r - 1) does, so
//       kPartStride * t_r - (kPartStride - 1) <= c_r <= min(kPartStride * t_r, n_r)            (c_r = 0 when t_r = 0).
//   Selecting sample rank T makes y the T-th sample and t_r the split.  With T_lo = d / kPartStride the entries that precede y
//   number at most kPartStride * T_lo <= d, so they all belong to the first d entries: s_r >= c_r.  With
//   T_hi = ceil((d + (kPartStride - 1) k) / kPartStride) they number at least d: s_r <= c_r.
constexpr uint32_t kPartStride = 64;
struct GroupLanes {
  uint32_t gshift, g, r, sub, gbase, nruns;
};
// Does entry i precede the pivot x (before_equal: or equal it)?  The 16-byte key prefix decides almost every probe; the length and
// the trailer columns are only touched on a tie (one DRAM sector per probe instead of three).
__device__ __forceinline__ bool entry_precedes(const KeyCols& c, uint64_t i, const Key& x, bool before_equal) {
  const ulonglong2 p = c.pfx[i];
  if (p.x != x.hi) return p.x < x.hi;
  if (p.y != x.lo) return p.y < x.lo;
  const uint32_t ul = meta_ulen(c.meta[i]);
  if (ul != x.ulen) return ul < x.ulen;
  const uint64_t tr = c.tr[i];
  if (tr != x.tr) return tr > x.tr;  // larger (seq, type) first
  return before_equal;
}
// multi-sequence selection of rank d over the runs' brackets [lo, hi) (units of `stride` entries; entry = base + stride * pos)
__device__ __forceinline__ void msel_grouped(const KeyCols& in, const GroupLanes& L, uint64_t base, uint64_t stride, uint64_t d, uint64_t& lo,
                                             uint64_t& hi) {
  const uint32_t g = L.g, r = L.r, sub = L.sub, gbase = L.gbase, gshift = L.gshift;
  for (int guard = 0; guard < 64 * 70; guard++) {
    // widest bracket decides the pivot run
    const unsigned long long wdt = hi - lo;
    unsigned long long best = wdt ? ((wdt << 7) | (unsigned long long)r) : 0;
#pragma unroll
    for (int dd = 16; dd; dd >>= 1) {
      const unsigned long long o = __shfl_xor_sync(0xffffffffu, best, dd);
      if (o > best) best = o;
    }
    if (best == 0) break;
    const uint32_t p = (uint32_t)(best & 127);
    const uint64_t m = __shfl_sync(0xffffffffu, lo + ((hi - lo) >> 1), (int)(p << gshift));
    const uint64_t pbase = __shfl_sync(0xffffffffu, base, (int)(p << gshift));
    const Key x = load_key(in, pbase + m * stride);
    // c = number of elements of run r that precede x in the total order (key, run index): (g+1)-ary search of [lo, hi)
    const bool before_equal = r < p;
    uint64_t clo = lo, chi = hi;
    if (r == p) clo = chi = m;
    while (__any_sync(0xffffffffu, chi > clo)) {
      const uint64_t w = chi - clo;
      uint64_t pos = clo;
      bool valid = false;
      if (w > 0) {
        if (w <= g) {
          pos = clo + sub;
          valid = sub < w;
        } else {
          pos = clo + (w * (sub + 1)) / (g + 1);
          valid = true;
        }
      }
      bool prec = false;
      if (valid) prec = entry_precedes(in, base + pos * stride, x, before_equal);
      const unsigned bal = __ballot_sync(0xffffffffu, prec);
      const uint32_t cp = __popc((bal >> gbase) & ((1u << g) - 1u));  // probes are increasing: the preceding ones form a prefix
      const uint32_t nvalid = w == 0 ? 0 : (w <= g ? (uint32_t)w : g);
      const uint64_t below = __shfl_sync(0xffffffffu, pos, (int)(gbase + (cp ? cp - 1 : 0)));
      const uint64_t above = __shfl_sync(0xffffffffu, pos, (int)(gbase + (cp < g ? cp : g - 1)));
      if (w > 0) {
        if (cp) clo = below + 1;
        if (cp < nvalid) chi = above;
        else if (w <= g) chi = clo;  // every remaining element precedes
      }
    }
    const uint64_t c = clo;
    uint64_t sum = sub == 0 ? c : 0;
#pragma unroll
    for (int dd = 16; dd; dd >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, dd);
    const bool x_before = sum < d;  // pivot is among the first d elements
    if (r < L.nruns) {
      if (x_before) lo = (r == p) ? m + 1 : c;
      else hi = (r == p) ? m : c;
    }
  }
}
// One warp resolves `chunk` CONSECUTIVE boundaries: the first one with the two-level search, every further one starting from
// its predecessor's split -- between rank d and rank d' >= d every run advances by at most d' - d entries, so the brackets are
// kMergeTile wide and lie in cache lines the previous search just touched.  The kernel is one chain of dependent loads per warp
// (about 135 for the two-level search, 55 for every further boundary), so the chunk is small: 3 boundaries per warp was the
// fastest of 2, 3 and 4 on the cfg2 job.
// 12 CTAs (48 warps) per SM: 42 registers with a small spill, but all of a job's warps are resident at once -- the kernel is one
// chain of dependent loads per warp, so residency is what counts (faster on cfg2 than the 64 registers ptxas takes unasked, or than
// 10 CTAs).
__global__ void __launch_bounds__(128, 12)
merge_partition_grouped_kernel(KeyCols in, RunBounds runs, uint32_t nruns, uint32_t gshift, uint64_t n_total,
                               uint64_t ntiles, uint64_t* __restrict__ splits, uint32_t* __restrict__ err, uint32_t chunk) {
  const unsigned lane = threadIdx.x & 31;
  const uint64_t b0 = ((uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * chunk;
  if (b0 > ntiles) return;
  GroupLanes L;
  L.gshift = gshift;
  L.g = 1u << gshift;
  L.r = lane >> gshift;
  L.sub = lane & (L.g - 1);
  L.gbase = L.r << gshift;
  L.nruns = nruns;
  const uint32_t r = L.r, sub = L.sub;
  const uint64_t base = r < nruns ? runs.begin[r] : 0;
  const uint64_t nrun = r < nruns ? runs.end[r] - runs.begin[r] : 0;
  uint64_t prev_lo = 0, prev_d = 0;
  const bool sd_mode = (*reinterpret_cast<volatile uint32_t*>(err) & (uint32_t)kFlagHasSingleDelete) != 0;  // set by the decoder
  for (uint32_t c = 0; c < chunk; c++) {
    const uint64_t b = b0 + c;
    if (b > ntiles) break;
    uint64_t d = b * (uint64_t)kMergeNominal;
    if (d > n_total) d = n_total;
    uint64_t lo = (d == n_total) ? nrun : 0, hi = (d == 0) ? 0 : nrun;
    if (d != 0 && d != n_total) {
      if (c != 0) {  // (prev_d may lie a few entries behind its nominal rank: see the alignment below)
        lo = prev_lo;
        hi = d > prev_d ? (prev_lo + (d - prev_d) < nrun ? prev_lo + (d - prev_d) : nrun) : prev_lo;
      } else {
        // ---- level 1: the samples
        const uint64_t S = kPartStride, msamp = (nrun + S - 1) / S;
        uint64_t M = sub == 0 ? msamp : 0;
#pragma unroll
        for (int dd = 16; dd; dd >>= 1) M += __shfl_xor_sync(0xffffffffu, M, dd);
        const uint64_t T_lo = d / S, T_hi = (d + (S - 1) * (uint64_t)nruns + S - 1) / S;
        uint64_t tlo = 0, tlo_hi = msamp;
        if (T_lo > 0) msel_grouped(in, L, base, S, T_lo, tlo, tlo_hi);  // T_lo < M because d < n_total
        if (tlo) lo = S * tlo - (S - 1);
        if (T_hi < M) {
          // the split of sample rank T_hi lies at most T_hi - T_lo samples further in every run
          uint64_t thi = tlo, thi_hi = tlo + (T_hi - T_lo) < msamp ? tlo + (T_hi - T_lo) : msamp;
          msel_grouped(in, L, base, S, T_hi, thi, thi_hi);
          const uint64_t h = S * thi;
          hi = h < nrun ? h : nrun;
        }
        if (hi < lo) hi = lo;  // cannot happen for sorted runs; the rank check below reports it
      }
    }
    // ---- exact
    msel_grouped(in, L, base, 1, d, lo, hi);
    uint64_t tot = sub == 0 ? lo : 0;
#pragma unroll
    for (int dd = 16; dd; dd >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, dd);
    if (tot != d && lane == 0) atomicOr(err, kErrKeyOrder);
    // ---- inputs with SingleDeletes: no user key may straddle a tile boundary.  The entry in front of the cut and the one behind it
    // share a user key => the cut moves behind that key's last version, in every run (they are the smallest entries left).
    if (sd_mode && d != 0 && d != n_total) {
      Key head, tail;  // per run: first entry behind / last entry in front of the cut (one lane per run: sub == 0)
      head.hi = head.lo = ~0ull, head.ulen = 0xffffffffu, head.tr = 0;
      tail.hi = tail.lo = 0, tail.ulen = 0, tail.tr = ~0ull;
      const bool have_head = r < nruns && sub == 0 && lo < nrun, have_tail = r < nruns && sub == 0 && lo > 0;
      if (have_head) head = load_key(in, base + lo);
      if (have_tail) tail = load_key(in, base + lo - 1);
      // smallest head user key / largest tail user key over the runs (user-key order; trailers do not matter here)
      Key mh = head, mt = tail;
      bool anyh = have_head, anyt = have_tail;
#pragma unroll
      for (int dd = 16; dd; dd >>= 1) {
        Key oh, ot;
        oh.hi = __shfl_xor_sync(0xffffffffu, mh.hi, dd), oh.lo = __shfl_xor_sync(0xffffffffu, mh.lo, dd), oh.ulen = __shfl_xor_sync(0xffffffffu, mh.ulen, dd);
        ot.hi = __shfl_xor_sync(0xffffffffu, mt.hi, dd), ot.lo = __shfl_xor_sync(0xffffffffu, mt.lo, dd), ot.ulen = __shfl_xor_sync(0xffffffffu, mt.ulen, dd);
        const bool ohv = __shfl_xor_sync(0xffffffffu, (int)anyh, dd) != 0, otv = __shfl_xor_sync(0xffffffffu, (int)anyt, dd) != 0;
        if (ohv && (!anyh || ukey_cmp(oh.hi, oh.lo, oh.ulen, mh.hi, mh.lo, mh.ulen) < 0)) mh = oh, anyh = true;
        if (otv && (!anyt || ukey_cmp(ot.hi, ot.lo, ot.ulen, mt.hi, mt.lo, mt.ulen) > 0)) mt = ot, anyt = true;
      }
      if (anyh && anyt && ukey_cmp(mh.hi, mh.lo, mh.ulen, mt.hi, mt.lo, mt.ulen) == 0) {
        uint32_t adv = 0;
        if (r < nruns && sub == 0) {
          while (lo < nrun && adv <= (uint32_t)kSdSpill) {
            const ulonglong2 p = in.pfx[base + lo];
            if (!same_ukey(mh, p.x, p.y, meta_ulen(in.meta[base + lo]))) break;
            lo++;
            adv++;
          }
        }
        uint32_t tadv = adv;
#pragma unroll
        for (int dd = 16; dd; dd >>= 1) tadv += __shfl_xor_sync(0xffffffffu, tadv, dd);
        if (tadv > (uint32_t)kSdSpill && lane == 0) atomicOr(err, (uint32_t)kErrGroupTooLong);
        d += tadv;
        lo = __shfl_sync(0xffffffffu, lo, (int)L.gbase);  // every lane of the run's group carries the moved cut
      }
    }
    if (r < nruns && sub == 0) splits[b * nruns + r] = lo;
    prev_lo = lo;
    prev_d = d;
  }
}

// ------------------------------------------------------------------------------------------------ tile merge
// Keys stay where the coalesced load put them (structure of arrays in shared memory); the merge rounds permute a list
// of 16-bit indices.  A comparison loads the high key word of both candidates and touches the other words only on a tie.
constexpr uint32_t kSnapCache = 16;
struct TileSmem {
  uint64_t hi[kMT], lo[kMT], tr[kMT];
  uint16_t idx[kMT];               // merge order: idx[o] = load position of the o-th smallest key
  uint8_t ulen[kMT];
  uint8_t verd[kMT];               // per merged position: verdict of the serial SingleDelete walk (bit 7: walked)
  uint32_t seg[kMaxRuns + 1];      // segment starts in load order
  uint32_t lst[2][kMaxRuns + 2];   // list bounds per merge round (ping-pong)
  uint64_t sbeg[kMaxRuns];         // absolute index of each segment's first element
  uint64_t snaps[kSnapCache];      // cached snapshots (the first kSnapCache)
  unsigned long long red[8];       // per-CTA counter staging
  unsigned long long stat[5];      // statistics of the tile's output entries (TileStat)
  uint32_t smin, smax;             // smallest / largest encoded entry size of the tile
  uint32_t wsum[40];
  uint64_t base_out;
  uint32_t tile_id, kept_total;
  Key pred;
  uint32_t has_pred;
};

__device__ __forceinline__ Key skey(const TileSmem& s, uint32_t id) {
  Key k;
  k.hi = s.hi[id];
  k.lo = s.lo[id];
  k.tr = s.tr[id];
  k.ulen = s.ulen[id] & 0x3fu;
  return k;
}
// column position of the entry at load position pos: load positions [seg[r], seg[r + 1]) hold run r's entries from sbeg[r] on
__device__ __forceinline__ uint64_t column_of(const TileSmem& s, uint32_t k, uint32_t pos) {
  uint32_t lo = 0, hi = k;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (s.seg[mid] <= pos) lo = mid;
    else hi = mid;
  }
  return s.sbeg[lo] + (pos - s.seg[lo]);
}
// List positions are XOR-swizzled inside 16-element groups: a thread owns kMV = 8 consecutive list positions, and with
// the plain layout the 32 lanes of one store to idx[] would fall on only eight banks (4-way conflict).
__device__ __forceinline__ uint32_t PH(uint32_t e) { return e ^ ((e >> 4) & 15u); }
// keys with equal high words: is the key at load position ib strictly before the one at ia?
__device__ __forceinline__ bool tie_less(const TileSmem& s, uint32_t ib, uint32_t ia) {
  const uint64_t lb = s.lo[ib], la = s.lo[ia];
  if (lb != la) return lb < la;
  const uint32_t ub = s.ulen[ib] & 0x3fu, ua = s.ulen[ia] & 0x3fu;
  if (ub != ua) return ub < ua;
  return s.tr[ib] > s.tr[ia];
}
// is key b (load position ib, high word hb) strictly before key a?
__device__ __forceinline__ bool id_less(const TileSmem& s, uint32_t ib, uint64_t hb, uint32_t ia, uint64_t ha) {
  if (hb != ha) return hb < ha;
  return tie_less(s, ib, ia);
}

struct PairState {
  uint32_t ai, a1, bi, b1, pend;  // cursors into A=[.., a1) and B=[.., b1) of the index list; pend = end of the pair's output
};
// locate the pair containing output position o and run the merge-path search for its diagonal
__device__ __noinline__ void init_pair(const TileSmem& s, const uint32_t* lst, uint32_t nlists, uint32_t o, PairState* ps) {
  uint32_t pi = 0;
  for (;;) {  // pair pi merges lists 2pi and 2pi+1 into [lst[2pi], lst[2pi+2])
    uint32_t e = 2 * pi + 2 <= nlists ? lst[2 * pi + 2] : lst[nlists];
    if (o < e) break;
    pi++;
  }
  uint32_t a0 = lst[2 * pi];
  uint32_t a1 = lst[2 * pi + 1];
  bool single = 2 * pi + 1 >= nlists;
  uint32_t b1 = single ? a1 : lst[2 * pi + 2];
  ps->pend = b1;
  ps->a1 = a1;
  ps->b1 = b1;
  if (single) {  // unpaired list: passes through
    ps->ai = o;
    ps->bi = b1;
    return;
  }
  uint32_t diag = o - a0, an = a1 - a0, bn = b1 - a1;
  uint32_t lo = diag > bn ? diag - bn : 0, hi = diag < an ? diag : an;
  while (lo < hi) {
    uint32_t mid = (lo + hi) >> 1;
    const uint32_t ia = s.idx[PH(a0 + mid)], ib = s.idx[PH(a1 + diag - 1 - mid)];
    if (!id_less(s, ib, s.hi[ib], ia, s.hi[ia])) lo = mid + 1;  // a <= b: a goes first (stable, lower run index wins ties)
    else hi = mid;
  }
  ps->ai = a0 + lo;
  ps->bi = a1 + (diag - lo);
}

__device__ __forceinline__ uint64_t stripe_of(const uint64_t* snaps_s, const uint64_t* snaps_g, uint32_t ns, uint64_t seq,
                                              uint64_t* prev) {
  // findEarliestVisibleSnapshot (compaction_iterator.cc:1343-1396, no snapshot checker): lower_bound(seq)
  uint32_t lo = 0, hi = ns;
  while (lo < hi) {
    uint32_t mid = (lo + hi) >> 1;
    uint64_t v = mid < kSnapCache ? snaps_s[mid] : snaps_g[mid];
    if (v < seq) lo = mid + 1;
    else hi = mid;
  }
  *prev = lo == 0 ? 0 : (lo - 1 < kSnapCache ? snaps_s[lo - 1] : snaps_g[lo - 1]);
  return lo < ns ? (lo < kSnapCache ? snaps_s[lo] : snaps_g[lo]) : kMaxSeq;
}

// slow path helpers for groups that leave the tile (only with snapshots at the bottommost level)
// oldest version of user key (hi,lo,ulen) over all runs has seq <= limit ?
__device__ bool oldest_version_at_most(const KeyCols& in, RunBounds runs, uint32_t nruns, uint64_t hi, uint64_t lo,
                                       uint32_t ulen, uint64_t limit) {
  const Key x{hi, lo, 0, ulen};  // (ukey, seq 0, type 0) sorts after every real version of ukey
  for (uint32_t r = 0; r < nruns; r++) {
    uint64_t base = runs.begin[r], n = runs.end[r] - base;
    uint64_t c = count_before(in, base, 0, n, x, true);
    if (c == 0) continue;
    Key e = load_key(in, base + c - 1);
    if (same_ukey(e, hi, lo, ulen) && (e.tr >> 8) <= limit) return true;
  }
  return false;
}
// Compaction filter decision (compaction_iterator.cc:231-473) for the kTypeValue entry at column position `src`: the built-in
// filters only look at the entry itself.  REMOVE_EMPTY_VALUE: empty value; TTL: the value's trailing fixed32 write time + ttl < now
// (DBWithTTLImpl::IsStale, utilities/ttl/db_ttl_impl.cc:445-461; values shorter than the 4-byte stamp are left alone).
__device__ __forceinline__ bool filter_removes(const MergeParams& mp, const KeyCols& in, uint64_t src) {
  const uint32_t vlen = meta_vlen(in.meta[src]);
  if (mp.filter == 1) return vlen == 0;
  if (mp.filter == 2) {
    if (mp.ttl <= 0 || vlen < 4) return false;
    const uint8_t* t = reinterpret_cast<const uint8_t*>((uintptr_t)in.vref[src]) + vlen - 4;
    const int64_t ts = (int64_t)((uint32_t)t[0] | (uint32_t)t[1] << 8 | (uint32_t)t[2] << 16 | (uint32_t)t[3] << 24);
    return ts + mp.ttl < mp.now;
  }
  return false;
}

// newest version of user key with seq <= stripe_hi: the head of that (user key, stripe) group.
// *head_tr carries the type the compaction iterator sees: with the remove-empty-value filter the NEWEST version of a user
// key is turned into a tombstone when it is a kTypeValue with an empty value (compaction_iterator.cc:579-584, :385-391)
__device__ bool group_head(const KeyCols& in, RunBounds runs, uint32_t nruns, uint64_t hi, uint64_t lo, uint32_t ulen,
                           uint64_t stripe_hi, const MergeParams& mp, uint64_t* head_tr) {
  const Key x{hi, lo, (stripe_hi << 8) | 0xff, ulen};  // sorts before every version with seq <= stripe_hi
  bool found = false, newer_exists = false;
  uint64_t best = 0, best_pos = 0;
  for (uint32_t r = 0; r < nruns; r++) {
    uint64_t base = runs.begin[r], n = runs.end[r] - base;
    uint64_t c = count_before(in, base, 0, n, x, false);
    if (c > 0) {  // the element in front of the lower bound: a version of the same user key with seq > stripe_hi?
      Key e = load_key(in, base + c - 1);
      if (same_ukey(e, hi, lo, ulen)) newer_exists = true;
    }
    if (c >= n) continue;
    Key e = load_key(in, base + c);
    if (same_ukey(e, hi, lo, ulen) && (!found || e.tr > best)) {
      found = true;
      best = e.tr;
      best_pos = base + c;
    }
  }
  if (found && mp.filter != 0 && !newer_exists && (best & 0xff) == kTypeValue && filter_removes(mp, in, best_pos))
    best = (best & ~0xffull) | kTypeDeletion;
  *head_tr = best;
  return found;
}

// SingleDelete (compaction_iterator.cc:662-887): whether a SingleDelete and the version below it cancel depends on what happened to
// the versions above them -- a chain through all versions of the user key.  Tiles are cut at user-key boundaries when an input holds
// one (merge_partition_grouped_kernel), so a key's versions are all in the tile: the thread that owns a key's first merged position
// walks the key with group_walk (group_rules.h, the reference's rules for one key) and leaves a verdict per version in s.verd.  Only called for tiles that contain a SingleDelete; kept out of line so that its local arrays do not
// weigh on the kernel's common path.
constexpr uint32_t kMaxGroup = 64;
__device__ __noinline__ void sd_walk_tile(TileSmem& s, const KeyCols& in, const MergeParams& mp, uint32_t cnt, uint32_t k, uint32_t* err,
                                          unsigned long long* w_hidden, unsigned long long* w_obsolete, unsigned long long* w_userdrop) {
  const uint32_t t = threadIdx.x;
  if (t == 0 && mp.write_conflict_snapshot) atomicOr(err, (uint32_t)kErrSdWriteConflict);
  for (int x = 0; x < kMV; x++) {
    const uint32_t o = t * kMV + x;
    if (o < cnt) s.verd[o] = 0;
  }
  __syncthreads();
  for (int x = 0; x < kMV; x++) {
    const uint32_t o = t * kMV + x;
    if (o >= cnt) break;
    const uint32_t id0 = s.idx[PH(o)];
    const Key k0 = skey(s, id0);
    bool head = true;
    if (o > 0) {
      head = !same_ukey(skey(s, s.idx[PH(o - 1)]), k0);
    } else if (s.has_pred && same_ukey(s.pred, k0) && k <= kPartGroupedMaxRuns) {
      // the grouped partition keeps keys inside one tile in this mode; with more runs merge_partition_kernel leaves the cuts where they
      // fall and has already refused the job (kErrGroupTooLong): that refusal is the job's answer, not an internal error
      atomicOr(err, (uint32_t)kErrInternal);
    }
    if (!head) continue;
    GroupVersion gv[kMaxGroup];
    uint32_t n = 0;
    bool has_sd = false;
    for (uint32_t q = o; q < cnt; q++) {
      const uint32_t id = s.idx[PH(q)];
      if (q != o && !same_ukey(k0, s.hi[id], s.lo[id], s.ulen[id] & 0x3fu)) break;
      const uint64_t tr = s.tr[id];
      has_sd = has_sd || (tr & 0xff) == kTypeSingleDeletion;
      if (n < kMaxGroup) gv[n] = GroupVersion{tr >> 8, (uint8_t)(tr & 0xff)};
      n++;
    }
    if (!has_sd) continue;
    if (n > kMaxGroup) {
      atomicOr(err, (uint32_t)kErrGroupTooLong);
      continue;
    }
    GroupRules gr;
    gr.snapshots = mp.snapshots;
    gr.num_snapshots = mp.nsnapshots;
    gr.bottommost = mp.bottommost;
    gr.earliest_write_conflict_snapshot = kGrMaxSeq;
    gr.key_not_exists_beyond_output_level = mp.bottommost;  // worker semantics (compaction.cc:555-556)
    gr.filter_removes_newest = 0;
    if (mp.filter != 0 && gv[0].type == kGrValue)  // (the filter may have to look at the newest version's value)
      gr.filter_removes_newest = mp.filter == 1 ? (s.ulen[id0] & 0x80u) != 0 : filter_removes(mp, in, column_of(s, k, id0));
    gr.first_key_of_the_job = 0;  // only matters with a write-conflict snapshot (rejected above)
    GroupVerdict vd[kMaxGroup];
    GroupCounters gc{0, 0, 0, 0};
    if (group_walk(gv, n, gr, vd, &gc) != 0) atomicOr(err, (uint32_t)kErrSingleDelContract);
    for (uint32_t i = 0; i < n; i++)
      s.verd[o + i] = (uint8_t)(0x80u | (vd[i].keep ? 1u : 0u) | (vd[i].zero_seq ? 2u : 0u) | ((vd[i].clear_value & 1u) ? 4u : 0u) |
                                (vd[i].out_type != gv[i].type ? 8u : 0u) | ((vd[i].clear_value & kGrSkipped) ? 16u : 0u));
    *w_hidden += gc.drop_hidden;
    *w_obsolete += gc.drop_obsolete;
    *w_userdrop += gc.drop_user;
  }
  __syncthreads();
}

// Phase: the tile's ticket and the CTA's shared counters and statistics; the first kSnapCache snapshots are cached.
__device__ __forceinline__ void tile_init(TileSmem& s, const MergeParams& mp, uint32_t* ticket) {
  const uint32_t t = threadIdx.x;
  if (t == 0) s.tile_id = atomicAdd(ticket, 1u);
  if (t < 8) s.red[t] = 0;
  stat_slots_init(s.stat, t);
  if (t == 0) {
    s.smin = 0xffffffffu;
    s.smax = 0;
  }
  if (t < kSnapCache && t < mp.nsnapshots) s.snaps[t] = mp.snapshots[t];
}

// Phase: the segment table (seg, sbeg, and lst[0] for the first merge round) and the tile's predecessor in merged order (pred,
// has_pred: the largest element in front of the split), fetched here one lane per run so that its DRAM round trip overlaps the split
// loads.  The per-run candidates are staged in hi[] and idx[], which the load phase overwrites later (keeps 3 CTAs per SM).
__device__ __forceinline__ void tile_segments(TileSmem& s, const KeyCols& in, RunBounds runs, const uint64_t* __restrict__ splits,
                                              uint64_t tile, uint32_t k, uint32_t* err) {
  const uint32_t t = threadIdx.x;
  Key* cand = reinterpret_cast<Key*>(s.hi);
  uint32_t* cand_ok = reinterpret_cast<uint32_t*>(s.idx);
  if (t < k) {
    const uint64_t s0 = splits[tile * k + t], s1 = splits[(tile + 1) * k + t];
    const uint64_t b0 = runs.begin[t] + s0;
    s.sbeg[t] = b0;
    s.lst[1][t] = (uint32_t)(s1 - s0);  // lengths, scanned below
    cand_ok[t] = s0 != 0;
    if (s0 != 0) cand[t] = load_key(in, b0 - 1);
  }
  __syncthreads();
  if (t == 0) {
    uint32_t acc = 0;
    for (uint32_t r = 0; r < k; r++) {
      s.seg[r] = acc;
      s.lst[0][r] = acc;
      acc += s.lst[1][r];
    }
    s.seg[k] = acc;
    s.lst[0][k] = acc;
    if (acc > kMT) {
      atomicOr(err, kErrKeyOrder);
      s.seg[k] = 0;
    }
    s.has_pred = 0;
    for (uint32_t r = 0; r < k; r++) {
      if (!cand_ok[r]) continue;
      const Key e = cand[r];
      if (!s.has_pred || ikey_less(s.pred, e)) {
        s.pred = e;
        s.has_pred = 1;
      }
    }
  }
}

// Phase: coalesced load of the k segments into hi / lo / tr / ulen (load order), idx[] = the identity.  All of a thread's loads are
// issued before the first one is consumed: a warp issues in order, so a load-then-store loop body would pay one DRAM round trip per
// iteration.  Returns whether this thread loaded a kTypeSingleDeletion (kSD only).
template <bool kSD>
__device__ __forceinline__ bool tile_load(TileSmem& s, const KeyCols& in, uint32_t cnt) {
  const uint32_t t = threadIdx.x;
  ulonglong2 lp[kMV];
  uint64_t ltr[kMV];
  uint32_t lmt[kMV];
  uint32_t lr = 0;
  bool my_sd = false;
#pragma unroll
  for (int j = 0; j < kMV; j++) {
    const uint32_t i = t + j * kMThreads;
    lp[j] = make_ulonglong2(0, 0);
    ltr[j] = 0;
    lmt[j] = 0;
    if (i < cnt) {
      while (i >= s.seg[lr + 1]) lr++;  // run with seg[lr] <= i < seg[lr + 1]; i grows with j, so the walk only moves forward
      const uint64_t src = s.sbeg[lr] + (i - s.seg[lr]);
      lp[j] = in.pfx[src];
      ltr[j] = in.tr[src];
      lmt[j] = in.meta[src];
    }
  }
#pragma unroll
  for (int j = 0; j < kMV; j++) {
    const uint32_t i = t + j * kMThreads;
    if (i < cnt) {
      s.hi[i] = lp[j].x;
      s.lo[i] = lp[j].y;
      s.tr[i] = ltr[j];
      if (kSD) my_sd = my_sd || (ltr[j] & 0xff) == kTypeSingleDeletion;
      s.ulen[i] = (uint8_t)(meta_ulen(lmt[j]) | (meta_vlen(lmt[j]) == 0 ? 0x80u : 0u));  // bit 7: empty value (compaction filter); bit 6 is set later: value removed by the filter
      s.idx[PH(i)] = (uint16_t)i;
    }
  }
  return my_sd;
}

// Phase: log2(k) rounds of pairwise merge-path merges over idx[], in place through registers; lst[] holds each round's list bounds.
// Leaves idx[o] = load position of the o-th smallest key.
__device__ __forceinline__ void tile_merge_rounds(TileSmem& s, uint32_t k, uint32_t cnt) {
  const uint32_t t = threadIdx.x;
  uint32_t nlists = k;
  int cur = 0;
  while (nlists > 1) {
    const uint32_t* lst = s.lst[cur];
    uint16_t rid[kMV];
    const uint32_t o0 = t * kMV;
    PairState ps;
    ps.pend = 0;
    ps.ai = ps.a1 = ps.bi = ps.b1 = 0;
    uint32_t ia = 0, ib = 0;
    uint64_t ha = 0, hb = 0;
    bool va = false, vb = false;
#pragma unroll
    for (int x = 0; x < kMV; x++) {
      uint32_t o = o0 + x;
      rid[x] = 0;
      if (o < cnt) {
        if (o >= ps.pend) {
          init_pair(s, lst, nlists, o, &ps);
          va = ps.ai < ps.a1;
          vb = ps.bi < ps.b1;
          if (va) {
            ia = s.idx[PH(ps.ai)];
            ha = s.hi[ia];
          }
          if (vb) {
            ib = s.idx[PH(ps.bi)];
            hb = s.hi[ib];
          }
        }
        const bool take_a = !vb || (va && !id_less(s, ib, hb, ia, ha));
        rid[x] = (uint16_t)(take_a ? ia : ib);
        if (take_a) {
          ps.ai++;
          va = ps.ai < ps.a1;
          if (va) {
            ia = s.idx[PH(ps.ai)];
            ha = s.hi[ia];
          }
        } else {
          ps.bi++;
          vb = ps.bi < ps.b1;
          if (vb) {
            ib = s.idx[PH(ps.bi)];
            hb = s.hi[ib];
          }
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int x = 0; x < kMV; x++) {
      uint32_t o = o0 + x;
      if (o < cnt) s.idx[PH(o)] = rid[x];
    }
    // next round's list bounds
    uint32_t nn = (nlists + 1) >> 1;
    if (t <= nn) s.lst[cur ^ 1][t] = t == nn ? cnt : lst[2 * t];
    __syncthreads();
    nlists = nn;
    cur ^= 1;
  }
}

// What the compaction-iterator rules decide for one merged position.
struct Verdict {
  uint64_t tr;     // output trailer (when kept)
  uint32_t flags;  // kV*
};
// written out / skipped without touching any input statistic / written out as a tombstone, without its value / value removed by the
// compaction filter (num_record_drop_user) / dropped: a newer version lies in the same snapshot stripe / dropped: an obsolete tombstone
constexpr uint32_t kVKeep = 1, kVSilent = 2, kVNoValue = 4, kVUserDrop = 8, kVHidden = 16, kVObsolete = 32;

// The verdict byte the SingleDelete walk (sd_walk_tile) left for a version of the entry with trailer tr.  Its drop counters come
// from the walk.
__device__ __forceinline__ Verdict sd_verdict(uint32_t vd, uint64_t tr) {
  Verdict v{0, 0};
  if (vd & 16u) {  // stepped over inside another version's branch: in none of the input statistics
    v.flags = kVSilent;
    return v;
  }
  if (vd & 1u) {
    const uint32_t type0 = (uint32_t)(tr & 0xff);
    const uint64_t out_type = (vd & 8u) ? (uint64_t)kTypeDeletion : (uint64_t)type0;  // a filtered Put leaves as a tombstone
    v.tr = (vd & 2u) ? out_type : (((tr >> 8) << 8) | out_type);
    v.flags = kVKeep | ((vd & 4u) ? kVNoValue : 0u);  // (written without its value)
  }
  return v;
}

// Merged position o is hidden behind a newer version of its (user key, stripe) group, at the bottommost level and in a stripe that
// is not the first.  Did the group's head take the bottommost-delete branch (compaction_iterator.cc:947-990)?  Its same-stripe
// followers are then skipped there without touching any counter.  The head is searched backwards through the tile, and over all
// runs when the group may start in front of the tile.
__device__ __forceinline__ bool hidden_head_is_tombstone(const TileSmem& s, const KeyCols& in, RunBounds runs, const MergeParams& mp,
                                                         uint32_t k, uint32_t o, const Key& c, uint64_t st_c) {
  int q = (int)o - 1;
  uint64_t head_tr = 0;
  uint32_t head_id = 0;
  bool have = false;
  while (q >= 0) {
    const uint32_t hid = s.idx[PH(q)];
    Key h = skey(s, hid);
    uint64_t d2;
    bool same_grp = same_ukey(h, c) && stripe_of(s.snaps, mp.snapshots, mp.nsnapshots, h.tr >> 8, &d2) == st_c;
    if (!same_grp) break;
    head_tr = h.tr;
    head_id = hid;
    have = true;
    q--;
  }
  if (have && mp.filter != 0 && (head_tr & 0xff) == kTypeValue &&
      (mp.filter == 1 ? (s.ulen[head_id] & 0x80u) != 0 : filter_removes(mp, in, column_of(s, k, head_id)))) {
    // the head is filtered if it is the first version of its user key: look at the entry in front of it
    const bool first_occ = q >= 0 ? !same_ukey(skey(s, s.idx[PH(q)]), c) : !(s.has_pred && same_ukey(s.pred, c));
    if (first_occ) head_tr = (head_tr & ~0xffull) | kTypeDeletion;
  }
  if (q < 0 && s.has_pred) {  // group may start before the tile
    uint64_t d2;
    bool pred_same = same_ukey(s.pred, c) && stripe_of(s.snaps, mp.snapshots, mp.nsnapshots, s.pred.tr >> 8, &d2) == st_c;
    if (pred_same) have = group_head(in, runs, k, c.hi, c.lo, c.ulen, st_c, mp, &head_tr);
  }
  return have && (head_tr & 0xff) == kTypeDeletion;  // head seq > earliest snapshot since its stripe is not the first
}

// CompactionIterator::NextFromInput / PrepareOutput (compaction_iterator.cc:475-1087,1274-1341) for the entry c at merged position o
// (load position id), against its predecessor in merged order: the previous position, or the tile's predecessor.
__device__ __forceinline__ Verdict position_rules(const TileSmem& s, const KeyCols& in, RunBounds runs, const MergeParams& mp, uint32_t k,
                                                  uint32_t cnt, uint32_t o, uint32_t id, Key c) {
  Key p;
  bool has_prev = true;
  if (o > 0) p = skey(s, s.idx[PH(o - 1)]);
  else {
    p = s.pred;
    has_prev = s.has_pred != 0;
  }
  const bool same = has_prev && same_ukey(p, c);
  const uint64_t seq = c.tr >> 8;
  uint32_t type = (uint32_t)(c.tr & 0xff);
  bool removed = false;
  if (mp.filter != 0 && !same && type == kTypeValue)
    removed = mp.filter == 1 ? (s.ulen[id] & 0x80u) != 0 : filter_removes(mp, in, column_of(s, k, id));
  if (removed) {
    // compaction filter on the first (newest) version of a user key: Decision::kRemove turns it into a tombstone, written out
    // without its value
    type = kTypeDeletion;
    c.tr = (seq << 8) | kTypeDeletion;
  }
  uint64_t prev_snap = 0, dummy;
  uint64_t st_c = mp.nsnapshots ? stripe_of(s.snaps, mp.snapshots, mp.nsnapshots, seq, &prev_snap) : kMaxSeq;
  bool hidden = same;
  if (same && mp.nsnapshots) hidden = stripe_of(s.snaps, mp.snapshots, mp.nsnapshots, p.tr >> 8, &dummy) == st_c;
  bool keep = false, silent = false, obsolete = false;
  if (hidden) {
    silent = mp.bottommost && mp.nsnapshots > 0 && st_c != mp.earliest_snapshot && hidden_head_is_tombstone(s, in, runs, mp, k, o, c, st_c);
  } else if (type == kTypeDeletion && seq <= mp.earliest_snapshot && mp.bottommost) {
    obsolete = true;  // :912-946 (KeyNotExistsBeyondOutputLevel == bottommost on a worker, compaction.cc:555-556)
  } else if (type == kTypeDeletion && mp.bottommost) {
    // :947-990 keep the tombstone only if an older stripe still holds a version of this user key
    bool resolved = false;
    for (uint32_t q = o + 1; q < cnt; q++) {
      Key nx = skey(s, s.idx[PH(q)]);
      if (!same_ukey(nx, c)) {
        resolved = true;
        break;
      }
      if ((nx.tr >> 8) <= prev_snap) {
        keep = true;
        resolved = true;
        break;
      }
    }
    if (!resolved) keep = oldest_version_at_most(in, runs, k, c.hi, c.lo, c.ulen, prev_snap);
  } else {
    keep = true;
  }
  Verdict v{0, (keep ? kVKeep : 0u) | (silent ? kVSilent : 0u) | (removed ? kVUserDrop | kVNoValue : 0u) | (hidden && !silent ? kVHidden : 0u) |
                   (obsolete ? kVObsolete : 0u)};
  // PrepareOutput :1299-1339 seqno zeroing
  if (keep) v.tr = (mp.bottommost && seq <= mp.earliest_snapshot) ? (uint64_t)type : c.tr;
  return v;
}

// per-thread partial CompactionIterationStats of the tile (MergeCounters)
struct TileCounts {
  unsigned long long kept, indel, hidden, obsolete, kbytes, vbytes, silent, userdrop;
};

// Phase: the rules for the thread's kMV merged positions.  The SingleDelete walk decided the versions of keys that hold a
// SingleDelete (verd[] bit 7); position_rules decides the others.  Leaves the verdicts in registers: keep_mask bit x = position x is
// kept, bit 16 + x = silent, bit 24 + x = written without its value; otr / oid = output trailer and load position.
template <bool kSD>
__device__ __forceinline__ void tile_rules(const TileSmem& s, const KeyCols& in, RunBounds runs, const MergeParams& mp, uint32_t k,
                                           uint32_t cnt, bool tile_sd, uint32_t& keep_mask, uint64_t (&otr)[kMV], uint16_t (&oid)[kMV],
                                           TileCounts& cn) {
#pragma unroll
  for (int x = 0; x < kMV; x++) {
    uint32_t o = threadIdx.x * kMV + x;
    otr[x] = 0;
    oid[x] = 0;
    if (o >= cnt) continue;
    const uint32_t id = s.idx[PH(o)];
    oid[x] = (uint16_t)id;
    const Key c = skey(s, id);
    const Verdict v = (kSD && tile_sd && (s.verd[o] & 0x80u)) ? sd_verdict(s.verd[o], c.tr) : position_rules(s, in, runs, mp, k, cnt, o, id, c);
    if (v.flags & kVSilent) {
      cn.silent++;
      keep_mask |= 1u << (16 + x);
    } else {
      cn.kbytes += c.ulen + 8;
      if (is_deletion_type((uint32_t)(c.tr & 0xff))) cn.indel++;  // the type as read
    }
    if (v.flags & kVHidden) cn.hidden++;
    if (v.flags & kVObsolete) cn.obsolete++;
    if (v.flags & kVUserDrop) cn.userdrop++;
    if (v.flags & kVKeep) {
      keep_mask |= 1u << x;
      cn.kept++;
      otr[x] = v.tr;
      if (v.flags & kVNoValue) keep_mask |= 1u << (24 + x);
    }
  }
}

// Phase: tile-local output rank of the thread's first kept position; leaves kept_total.
__device__ __forceinline__ uint32_t tile_ranks(TileSmem& s, uint32_t nkeep) {
  const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t inc = warp_incl_scan(nkeep);
  if (lane == 31) s.wsum[w] = inc;
  __syncthreads();
  if (w == 0) {
    uint32_t v = lane < (kMThreads / 32) ? s.wsum[lane] : 0;
    uint32_t vi = warp_incl_scan(v);
    s.wsum[lane] = vi - v;
    if (lane == 31) s.kept_total = vi;
  }
  __syncthreads();
  return s.wsum[w] + inc - nkeep;
}

// Value bytes of the thread's silent positions.  The value-byte statistic starts from the inputs' raw.value.size property, which
// already sums every entry; only the (rare) silently skipped entries are subtracted, so only they pay a gather.
__device__ __forceinline__ unsigned long long silent_value_bytes(const TileSmem& s, const KeyCols& in, uint32_t k, uint32_t cnt,
                                                                 uint32_t keep_mask, const uint16_t (&oid)[kMV]) {
  unsigned long long vb = 0;
#pragma unroll
  for (int x = 0; x < kMV; x++) {
    uint32_t o = threadIdx.x * kMV + x;
    if (o < cnt && ((keep_mask >> (16 + x)) & 1)) vb += meta_vlen(in.meta[column_of(s, k, oid[x])]);
  }
  return vb;
}

// Phase, once every read of idx[] / tr[] in merged order is done: compaction in place.  Leaves idx[0, kept_total) = load positions
// of the survivors in output order, tr[] = their output trailers, ulen[] bit 6 = written without its value.
__device__ __forceinline__ void tile_compact(TileSmem& s, uint32_t keep_mask, const uint64_t (&otr)[kMV], const uint16_t (&oid)[kMV],
                                             uint32_t rank) {
#pragma unroll
  for (int x = 0; x < kMV; x++) {
    if ((keep_mask >> x) & 1) {
      s.idx[PH(rank)] = oid[x];
      s.tr[oid[x]] = otr[x];  // each load position is owned by exactly one merged position
      if ((keep_mask >> (24 + x)) & 1) s.ulen[oid[x]] |= 0x40u;
      rank++;
    }
  }
}

// Phase: gather the value references of the survivors (random within k contiguous segments) for all of the thread's output slots
// first, then write: again one round trip instead of kMV.
__device__ __forceinline__ void tile_gather(const TileSmem& s, const KeyCols& in, uint32_t k, uint32_t kept_total, uint64_t (&gv)[kMV],
                                            uint32_t (&gm)[kMV], uint16_t (&gp)[kMV]) {
#pragma unroll
  for (int j = 0; j < kMV; j++) {
    const uint32_t i = threadIdx.x + j * kMThreads;
    gv[j] = 0;
    gm[j] = 0;
    gp[j] = 0;
    if (i < kept_total) {
      const uint32_t pos = s.idx[PH(i)];
      const uint64_t src = column_of(s, k, pos);
      gp[j] = (uint16_t)pos;
      gv[j] = in.vref[src];
      gm[j] = in.meta[src];
      if (s.ulen[pos] & 0x40u) gm[j] = make_meta(meta_ulen(gm[j]), 0);  // removed by the compaction filter: tombstone, no value
    }
  }
}

// Phase: write the survivors to the output columns from base_out on, with their encoded sizes against the previous output entry
// (BlockBuilder::AddWithLastKey); adds the tile's statistics (TileStat) and entry-size extremes into stat / smin / smax.
__device__ __forceinline__ void tile_store(TileSmem& s, KeyColsMut out, MergeSizes ms, uint64_t base_out, uint32_t kept_total,
                                           const uint64_t (&gv)[kMV], const uint32_t (&gm)[kMV], const uint16_t (&gp)[kMV]) {
  StatAcc<uint32_t> st;
  uint32_t mn = 0xffffffffu, mx = 0;
#pragma unroll
  for (int j = 0; j < kMV; j++) {
    const uint32_t i = threadIdx.x + j * kMThreads;
    if (i < kept_total) {
      const uint32_t pos = gp[j];
      const uint64_t dst = base_out + i;
      const uint64_t chi = s.hi[pos], clo = s.lo[pos], ctr = s.tr[pos];
      const uint32_t cul = s.ulen[pos] & 0x3fu, vlen = meta_vlen(gm[j]);
      out.pfx[dst] = make_ulonglong2(chi, clo);
      out.tr[dst] = ctr;
      out.vref[dst] = gv[j];
      out.meta[dst] = gm[j];
      // the tile's first entry is left to merge_sizes_fix_kernel: its predecessor is the last survivor of an earlier tile
      if (i > 0) {
        const uint32_t pp = s.idx[PH(i - 1)];
        const uint32_t sh = shared_prefix(chi, clo, cul, ctr, s.hi[pp], s.lo[pp], s.ulen[pp] & 0x3fu, s.tr[pp]);
        const uint32_t s1 = entry_size(sh, cul + 8, vlen);
        ms.esz[dst] = s1;
        ms.eshared[dst] = (uint8_t)sh;
        mn = s1 < mn ? s1 : mn;
        mx = s1 > mx ? s1 : mx;
      }
      st.add_entry(cul + 8, vlen, ctr);
    }
  }
  mn = __reduce_min_sync(0xffffffffu, mn);
  mx = __reduce_max_sync(0xffffffffu, mx);
  st.flush(s.stat);
  if ((threadIdx.x & 31) == 0) {
    atomicMin(&s.smin, mn);
    atomicMax(&s.smax, mx);
  }
}

// Phase: the thread's counters into red[] (MergeCounters order).  Per-thread partial counts are small (<= kMV entries, or a
// SingleDelete walk's drops), so the warp reduction is a single redux instruction per counter; only the (rare) value-byte
// correction needs 64 bits.
__device__ __forceinline__ void tile_count(TileSmem& s, const TileCounts& cn) {
  const uint32_t lane = threadIdx.x & 31;
  const unsigned vals[7] = {(unsigned)cn.kept,   (unsigned)cn.indel,  (unsigned)cn.hidden,  (unsigned)cn.obsolete,
                            (unsigned)cn.kbytes, (unsigned)cn.silent, (unsigned)cn.userdrop};
  const int slot[7] = {0, 1, 2, 3, 4, 6, 7};
#pragma unroll
  for (int i = 0; i < 7; i++) {
    const unsigned v = __reduce_add_sync(0xffffffffu, vals[i]);
    if (lane == 0 && v) atomicAdd(&s.red[slot[i]], (unsigned long long)v);
  }
  if (__any_sync(0xffffffffu, cn.vbytes != 0)) {
    unsigned long long v = cn.vbytes;
#pragma unroll
    for (int dd = 16; dd; dd >>= 1) v += __shfl_xor_sync(0xffffffffu, v, dd);
    if (lane == 0) atomicAdd(&s.red[5], v);
  }
}

// three CTAs per SM at 80 registers (four at 64 registers, with spills, were slower)
constexpr int kMergeCtasPerSm = 3;
// a predecessor tile that has not published its count is still merging
constexpr uint32_t kLookbackSleepNs = 64;
// kSD: the variant for jobs whose inputs hold a kTypeSingleDeletion (the decoder notes that in the error word).  Both variants are
// launched; the one that does not apply leaves at once.  Keeping the serial walk and its bookkeeping out of the common variant
// shortens the common case.
template <bool kSD>
__global__ void __launch_bounds__(kMThreads, kMergeCtasPerSm)
merge_tiles_kernel(KeyCols in, RunBounds runs, MergeParams mp, uint64_t n_total, uint64_t ntiles,
                   const uint64_t* __restrict__ splits, unsigned long long* tile_state, uint32_t* ticket, KeyColsMut out,
                   MergeCounters* counters, MergeSizes ms, uint32_t* __restrict__ err) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  TileSmem& s = *reinterpret_cast<TileSmem*>(smem_raw);
  const uint32_t t = threadIdx.x, lane = t & 31, w = t >> 5;
  const uint32_t k = mp.nruns;
  if (((*reinterpret_cast<volatile uint32_t*>(err) & (uint32_t)kFlagHasSingleDelete) != 0) != kSD) return;
  tile_init(s, mp, ticket);
  __syncthreads();
  const uint64_t tile = s.tile_id;
  if (tile >= ntiles) return;
  tile_segments(s, in, runs, splits, tile, k, err);
  __syncthreads();
  const uint32_t cnt = s.seg[k];
  bool tile_sd = tile_load<kSD>(s, in, cnt);  // some entry of the tile is a kTypeSingleDeletion
  if (kSD) tile_sd = __syncthreads_or(tile_sd) != 0;  // (also the barrier behind the load phase)
  else __syncthreads();
  tile_merge_rounds(s, k, cnt);
  unsigned long long w_hidden = 0, w_obsolete = 0, w_userdrop = 0;
  if (kSD && tile_sd) sd_walk_tile(s, in, mp, cnt, k, err, &w_hidden, &w_obsolete, &w_userdrop);
  TileCounts cn{0, 0, w_hidden, w_obsolete, 0, 0, 0, w_userdrop};
  uint32_t keep_mask = 0;
  uint64_t otr[kMV];
  uint16_t oid[kMV];
  tile_rules<kSD>(s, in, runs, mp, k, cnt, tile_sd, keep_mask, otr, oid, cn);
  uint32_t rank = tile_ranks(s, (uint32_t)cn.kept);
  const uint32_t kept_total = s.kept_total;
  // Decoupled look-back for the global output offset (tile ids are handed out in launch order), in two halves: the tile's count is
  // published now, the wait for the predecessors' counts comes after the compaction and the value-reference gathers -- a tile can
  // only resolve its offset once EVERY earlier tile has published its count, so waiting here would idle the whole CTA for the
  // spread of the predecessors' progress.
  if (t == 0) lb_publish(tile_state, tile, kept_total);
  cn.vbytes = silent_value_bytes(s, in, k, cnt, keep_mask, oid);
  __syncthreads();
  tile_compact(s, keep_mask, otr, oid, rank);
  __syncthreads();
  uint64_t gv[kMV];
  uint32_t gm[kMV];
  uint16_t gp[kMV];
  tile_gather(s, in, k, kept_total, gv, gm, gp);
  if (w == 0) {
    const uint64_t base = lb_exclusive_prefix(tile_state, tile, kept_total, lane, kLookbackSleepNs);
    if (lane == 0) s.base_out = base;
  }
  __syncthreads();
  tile_store(s, out, ms, s.base_out, kept_total, gv, gm, gp);
  tile_count(s, cn);
  __syncthreads();
  if (t < 8 && s.red[t]) atomicAdd(((unsigned long long*)counters) + t, s.red[t]);
  if (t == 0) {
    ms.tstat[tile] = TileStat{s.stat[0], s.stat[1], s.stat[2], s.stat[3], s.stat[4]};
    if (s.smin != 0xffffffffu) {
      atomicMin(ms.min_s1, s.smin);
      atomicMax(ms.min_s1 + 1, s.smax);
    }
  }
}

// The first output entry of every merge tile: its predecessor was written by an earlier tile.  One thread per tile.
__global__ void merge_sizes_fix_kernel(KeyCols m, const unsigned long long* __restrict__ tile_state, uint64_t ntiles, MergeSizes ms) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t s1 = 0xffffffffu;
  if (t < ntiles) {
    const uint64_t e = t ? lb_value(tile_state[t - 1]) : 0, end = lb_value(tile_state[t]);
    if (end > e) {  // the tile has survivors; e is the first
      const ulonglong2 c = m.pfx[e];
      const uint64_t ctr = m.tr[e];
      const uint32_t mt = m.meta[e], cul = meta_ulen(mt);
      uint32_t sh = 0;
      if (e > 0) {
        const ulonglong2 p = m.pfx[e - 1];
        sh = shared_prefix(c.x, c.y, cul, ctr, p.x, p.y, meta_ulen(m.meta[e - 1]), m.tr[e - 1]);
      }
      s1 = entry_size(sh, cul + 8, meta_vlen(mt));
      ms.esz[e] = s1;
      ms.eshared[e] = (uint8_t)sh;
    }
  }
  const uint32_t mn = __reduce_min_sync(0xffffffffu, s1);
  const uint32_t mx = __reduce_max_sync(0xffffffffu, s1 == 0xffffffffu ? 0u : s1);
  if ((threadIdx.x & 31) == 0 && mn != 0xffffffffu) {
    atomicMin(ms.min_s1, mn);
    atomicMax(ms.min_s1 + 1, mx);
  }
}

// ------------------------------------------------------------------------------------------------ sub-compaction key range
// ProcessKeyValueCompaction clips the merged input of a sub-compaction to [start, end) with a ClippingIterator whose bounds are
// (user key, kMaxSequenceNumber, kValueTypeForSeek) (compaction_job.cc:1495-1519), i.e. start <= user key < end.  Every run is
// sorted, so the clip is a sub-range per run: two binary searches; the merge then runs over the clipped runs and never sees the
// rest.  grid = (slices, runs): every CTA repeats its run's two searches (lanes 0 / 1), then the slices add up the value bytes of
// the run's entries in range (CompactionJobStats::total_input_raw_value_bytes counts what the iterator consumed).
constexpr int kClipSlices = 64;
__global__ void __launch_bounds__(256)
clip_runs_kernel(KeyCols in, RunBounds runs, uint32_t nruns, BoundKey start, uint32_t has_start, BoundKey end,
                 uint32_t has_end, uint64_t* __restrict__ clip, unsigned long long* __restrict__ totals) {
  __shared__ uint64_t sb[2];
  const uint32_t r = blockIdx.y;
  if (threadIdx.x < 2) {
    const bool is_end = threadIdx.x == 1;
    const uint64_t a0 = runs.begin[r], b0 = runs.end[r];
    uint64_t pos = is_end ? b0 : a0;
    if (is_end ? has_end : has_start) {  // first entry of the run with user key >= bound
      const BoundKey k = is_end ? end : start;
      pos = ukey_bound(in, a0, b0, k.hi, k.lo, k.ulen, false);
    }
    sb[threadIdx.x] = pos;
  }
  __syncthreads();
  const uint64_t b = sb[0];
  const uint64_t e = sb[1] > b ? sb[1] : b;  // end <= start: empty range
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    clip[r] = b;
    clip[nruns + r] = e;
    atomicAdd(&totals[0], (unsigned long long)(e - b));
  }
  unsigned long long sum = 0;
  for (uint64_t i = b + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (uint64_t)gridDim.x * blockDim.x)
    sum += meta_vlen(in.meta[i]);
#pragma unroll
  for (int d = 16; d; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
  if ((threadIdx.x & 31) == 0 && sum) atomicAdd(&totals[1], sum);
}
void launch_clip_runs(KeyCols in, RunBounds runs, uint32_t nruns, BoundKey start, uint32_t has_start, BoundKey end,
                      uint32_t has_end, uint64_t* clip, unsigned long long* totals, cudaStream_t st) {
  if (nruns) clip_runs_kernel<<<dim3(kClipSlices, nruns), 256, 0, st>>>(in, runs, nruns, start, has_start, end, has_end, clip, totals);
}
// one thread per run: its column range, and the order of the files inside it
__global__ void run_bounds_kernel(KeyCols in, const uint64_t* __restrict__ file_start, const uint32_t* __restrict__ run_first, uint32_t nruns,
                                  uint64_t* __restrict__ bounds, uint32_t* __restrict__ err) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nruns) return;
  const uint32_t f0 = run_first[r], f1 = run_first[r + 1];
  bounds[r] = file_start[f0];
  bounds[nruns + r] = file_start[f1];
  for (uint32_t f = f0 + 1; f < f1; f++) {
    const uint64_t e = file_start[f];  // first entry of file f; the entry before it is the last one of an earlier file of the run
    if (e > file_start[f0] && e < file_start[f1] && !ikey_less(load_key(in, e - 1), load_key(in, e))) atomicOr(err, (uint32_t)kErrKeyOrder);
  }
}
void launch_run_bounds(KeyCols in, const uint64_t* file_start, const uint32_t* run_first, uint32_t nruns, uint64_t* bounds, uint32_t* err,
                       cudaStream_t st) {
  if (nruns) run_bounds_kernel<<<(nruns + 63) / 64, 64, 0, st>>>(in, file_start, run_first, nruns, bounds, err);
}

// ------------------------------------------------------------------------------------------------ launchers
void launch_merge_partition(KeyCols in, RunBounds runs, uint32_t nruns, uint64_t n_total, uint64_t ntiles,
                            uint64_t* splits, uint32_t* err, int sms, cudaStream_t st) {
  unsigned warps = (unsigned)(ntiles + 1);
  if (nruns <= kPartGroupedMaxRuns) {
    uint32_t kp2 = 2;  // at most 16 lanes per run
    while (kp2 < nruns) kp2 <<= 1;
    uint32_t gshift = 0;
    while ((kp2 << (gshift + 1)) <= 32) gshift++;  // lanes per run = 32 / pow2(nruns)
    // about one and a half waves of warps (32 resident per SM at 64 registers)
    const unsigned wave = (unsigned)sms * 48u;
    uint32_t chunk = (uint32_t)((warps + wave - 1) / wave);
    if (chunk > 4) chunk = 4;
    if (chunk < 1) chunk = 1;
    const unsigned chunks = (warps + chunk - 1) / chunk;
    merge_partition_grouped_kernel<<<(chunks + 3) / 4, 128, 0, st>>>(in, runs, nruns, gshift, n_total, ntiles, splits, err, chunk);
    return;
  }
  merge_partition_kernel<<<(warps + 3) / 4, 128, 0, st>>>(in, runs, nruns, n_total, ntiles, splits, err);
}
static_assert(sizeof(Key) * kMaxRuns <= sizeof(uint64_t) * kMT && 4 * kMaxRuns <= 2 * kMT, "candidate staging must fit");
static_assert(kMergeCtasPerSm * (sizeof(TileSmem) + 1024) <= 227 * 1024, "merge tile must fit three CTAs per SM");
void launch_merge_tiles(KeyCols in, RunBounds runs, MergeParams mp, uint64_t n_total, uint64_t ntiles,
                        const uint64_t* splits, unsigned long long* tile_state, uint32_t* ticket, KeyColsMut out,
                        MergeCounters* counters, MergeSizes ms, uint32_t* err, cudaStream_t st) {
  if (ntiles == 0) return;
  static PerDeviceFlag attr;
  const uint64_t dev_bit = attr.bit_of_current_device();
  if (!attr.is_set(dev_bit)) {
    cudaFuncSetAttribute(merge_tiles_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TileSmem));
    cudaFuncSetAttribute(merge_tiles_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TileSmem));
    attr.set(dev_bit);
  }
  merge_tiles_kernel<false><<<(unsigned)ntiles, kMThreads, sizeof(TileSmem), st>>>(in, runs, mp, n_total, ntiles, splits, tile_state, ticket,
                                                                                   out, counters, ms, err);
  merge_tiles_kernel<true><<<(unsigned)ntiles, kMThreads, sizeof(TileSmem), st>>>(in, runs, mp, n_total, ntiles, splits, tile_state, ticket,
                                                                                  out, counters, ms, err);
}
void launch_merge_sizes_fix(KeyCols merged, const unsigned long long* tile_state, uint64_t ntiles, MergeSizes ms, cudaStream_t st) {
  if (ntiles) merge_sizes_fix_kernel<<<(unsigned)((ntiles + 127) / 128), 128, 0, st>>>(merged, tile_state, ntiles, ms);
}

}  // namespace b200c
