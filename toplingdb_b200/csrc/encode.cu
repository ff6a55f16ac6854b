// toplingdb_b200/csrc/encode.cu — BlockBasedTable output encode on the device, bit-exact with the reference builder.
//
// Replaces BlockBasedTableBuilder::{Add,Flush,WriteBlock,WriteMaybeCompressedBlock} (table/block_based/
// block_based_table_builder.cc:961-1133,1277-1378), BlockBuilder (block_builder.cc:97-253), FlushBlockBySizePolicy
// (flush_block_policy.cc:37-69), ShortenedIndexBuilder (index_builder.h:165-233, index_builder.cc:77-94,
// util/comparator.cc:42-91), the block checksums (table/format.cc:436-509) and the output-file cut rule of
// CompactionOutputs::ShouldStopBefore (db/compaction/compaction_outputs.cc:231-354, max-file-size rule :277).
//
// The reference cuts blocks with a sequential greedy rule.  Here it is evaluated in parallel:
//   encode_sizes      per entry: shared-prefix length with the previous internal key and encoded size; per tile: partial
//                     sums for the per-file statistics (TableBuilder path only: a compaction's merge kernel writes these)
//   encode_tables     per tile of kEncTile entries: next(a) = "where does a block that starts at entry a end" for every
//                     a (prefix sums + bisection in shared memory), then the tile's transfer function
//                     entry-point -> (exit point, bytes, #blocks) for every entry point a chain can arrive at
//   encode_stitch     one CTA walks the tile functions in order (rows prefetched in batches), applying the
//                     max_output_file_size rule exactly, and records the state at which the chain enters every tile
//   encode_blocklist  per tile: follow the real chain, emit one BlockRec per data block
//   encode_emit       one warp per data block: encode entries (varints, key suffix, value bytes fetched through vref)
//                     into a shared-memory image, restart array, checksum, coalesced store into the file image
//   encode_index_*    per block separator keys, per-file index block, its checksum
// HBM-bound; algorithmic bytes of encode_emit = 36 B of columns + value bytes read + block bytes written per entry.
#include "bloom_rules.h"
#include "common.cuh"
#include "gp_rules.h"
#include "kernels.h"
#include "scan.cuh"

namespace b200c {

constexpr int kTT = kEncTile;
constexpr int kW = kEncTile + kEncHalo;
constexpr int kEncThreads = 256;

// ------------------------------------------------------------------------------------------------ entry sizes
// (ikey_byte / shared_prefix / entry_size live in common.cuh: the merge kernel writes the sizes of the entries it emits, so this
// pass serves the TableBuilder path, which has no merge in front of it)
// One CTA per tile of kEncTile sorted entries (grid-stride over tiles): shared-prefix length + encoded size of every entry, the
// global min / max entry size, and the tile's partial sums for the per-file statistics (so that the statistics pass reads
// 40 bytes per tile instead of 12 bytes per entry).
__global__ void __launch_bounds__(256)
encode_sizes_kernel(KeyCols m, const unsigned long long* __restrict__ n_dev, uint32_t* __restrict__ esz, uint8_t* __restrict__ eshared,
                    TileStat* __restrict__ tstat, unsigned long long* __restrict__ tprefix, uint32_t* __restrict__ min_s1) {
  const uint64_t n = *n_dev;
  const uint64_t ntiles = (n + kEncTile - 1) / kEncTile;
  uint32_t mn = 0xffffffffu, mxs = 0;
  __shared__ unsigned long long red[5];
  __shared__ uint32_t s_mn, s_mx;
  if (threadIdx.x == 0) {
    s_mn = 0xffffffffu;
    s_mx = 0;
  }
  for (uint64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    stat_slots_init(red, threadIdx.x);
    __syncthreads();
    const uint64_t t0 = tile * kEncTile, t1 = (t0 + kEncTile) < n ? (t0 + kEncTile) : n;
    StatAcc<unsigned long long> st;
    // four entries per thread in flight; the previous entry (for the shared-prefix length) comes from the neighbouring lane,
    // only lane 0 of a warp fetches it from memory
    constexpr int kB = 4;
    for (uint64_t ib = t0; ib < t1; ib += (uint64_t)kB * blockDim.x) {
      ulonglong2 c[kB], pc[kB];
      uint64_t ctr[kB], ptr_[kB];
      uint32_t cm[kB], pm[kB];
      const unsigned lane = threadIdx.x & 31;
#pragma unroll
      for (int q = 0; q < kB; q++) {
        const uint64_t i = ib + (uint64_t)q * blockDim.x + threadIdx.x;
        c[q] = make_ulonglong2(0, 0);
        pc[q] = make_ulonglong2(0, 0);
        ctr[q] = ptr_[q] = 0;
        cm[q] = pm[q] = 0;
        if (i < t1) {
          c[q] = m.pfx[i];
          ctr[q] = m.tr[i];
          cm[q] = m.meta[i];
          if (lane == 0 && i > 0) {
            pc[q] = m.pfx[i - 1];
            ptr_[q] = m.tr[i - 1];
            pm[q] = m.meta[i - 1];
          }
        }
      }
#pragma unroll
      for (int q = 0; q < kB; q++) {
        const uint64_t i = ib + (uint64_t)q * blockDim.x + threadIdx.x;
        const uint64_t nx = __shfl_up_sync(0xffffffffu, c[q].x, 1), ny = __shfl_up_sync(0xffffffffu, c[q].y, 1);
        const uint64_t nt = __shfl_up_sync(0xffffffffu, ctr[q], 1);
        const uint32_t nm = __shfl_up_sync(0xffffffffu, cm[q], 1);
        if (lane != 0) {
          pc[q] = make_ulonglong2(nx, ny);
          ptr_[q] = nt;
          pm[q] = nm;
        }
        if (i < t1) {
          const uint32_t ulen = meta_ulen(cm[q]), vs = meta_vlen(cm[q]), ks = ulen + 8;
          const uint32_t sh = i > 0 ? shared_prefix(c[q].x, c[q].y, ulen, ctr[q], pc[q].x, pc[q].y, meta_ulen(pm[q]), ptr_[q]) : 0;
          const uint32_t s1 = entry_size(sh, ks, vs);
          esz[i] = s1;
          eshared[i] = (uint8_t)sh;
          mn = s1 < mn ? s1 : mn;
          mxs = s1 > mxs ? s1 : mxs;
          st.add_entry(ks, vs, ctr[q]);
        }
      }
    }
    st.flush(red);
    __syncthreads();
    if (threadIdx.x == 0) {
      tstat[tile] = TileStat{red[0], red[1], red[2], red[3], red[4]};
      tprefix[tile] = t1;  // entries up to and including this stat tile
    }
    __syncthreads();
  }
  mn = __reduce_min_sync(0xffffffffu, mn);
  mxs = __reduce_max_sync(0xffffffffu, mxs);
  // one pair of global atomics per CTA (same-address atomics serialise)
  __syncthreads();
  if ((threadIdx.x & 31) == 0) {
    atomicMin(&s_mn, mn);
    atomicMax(&s_mx, mxs);
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_mn != 0xffffffffu) {
    atomicMin(min_s1, s_mn);
    atomicMax(min_s1 + 1, s_mx);  // upper half of the slot: largest entry (selects the narrow block-cut window)
  }
}

// ------------------------------------------------------------------------------------------------ block-cut window
// PT = uint32_t when the bytes of a whole window fit 32 bits (decided on the host from the largest entry): the narrow
// window leaves room for three CTAs per SM instead of two
template <typename PT>
struct Window {
  PT P[kW + 1];         // P[j] = sum of s1 of window entries < j
  uint32_t Q[kW];       // Q[j] = D[j] + Q[j - R]: restart surcharge prefix per residue class (D = s0 - s1)
  uint64_t ws[33];
  uint32_t wlen;        // entries loaded
  uint32_t at_end;      // window reaches the end of the stream
  uint32_t smax;        // largest restart-encoded entry (s0) in the window
};

// cooperative: load the window of tile `tile` and build P / Q
template <typename PT>
__device__ void build_window(Window<PT>& w, const KeyCols& m, const uint32_t* esz, const uint8_t* eshared, uint64_t n, uint64_t tile,
                             uint32_t R) {
  const uint64_t wstart = tile * (uint64_t)kTT;
  const uint32_t wlen = (uint32_t)((n - wstart) < (uint64_t)kW ? (n - wstart) : (uint64_t)kW);
  // 1) coalesced load of the three size columns, eight entries per thread in flight at a time (a load-use loop body
  //    would cost one DRAM round trip per iteration); s1 is parked in P[j + 1], the restart surcharge D goes to Q[j]
  uint32_t mx = 0;
  if (threadIdx.x == 0) w.smax = 0;
  constexpr int kBatch = 8;
  for (uint32_t jb = 0; jb < wlen; jb += kBatch * kEncThreads) {
    uint32_t s1v[kBatch], shv[kBatch], mtv[kBatch];
#pragma unroll
    for (int i = 0; i < kBatch; i++) {
      const uint32_t j = jb + i * kEncThreads + threadIdx.x;
      s1v[i] = shv[i] = mtv[i] = 0;
      if (j < wlen) {
        s1v[i] = esz[wstart + j];
        shv[i] = eshared[wstart + j];
        mtv[i] = m.meta[wstart + j];
      }
    }
#pragma unroll
    for (int i = 0; i < kBatch; i++) {
      const uint32_t j = jb + i * kEncThreads + threadIdx.x;
      if (j < wlen) {
        const uint32_t d = restart_surcharge(shv[i], meta_ulen(mtv[i]) + 8);
        w.Q[j] = d;
        w.P[j + 1] = (PT)s1v[i];
        mx = s1v[i] + d > mx ? s1v[i] + d : mx;
      }
    }
  }
  __syncthreads();
  // 2) blocked exclusive scan of s1: consecutive entries per thread; an ODD count keeps the blocked shared-memory
  //    accesses conflict-free (24 would put the lanes of a warp on only four banks)
  constexpr int kPer = ((kW + kEncThreads - 1) / kEncThreads) | 1;  // 25
  const uint32_t j0 = threadIdx.x * kPer;
  uint64_t loc[kPer], sum = 0;
#pragma unroll
  for (int i = 0; i < kPer; i++) {
    const uint32_t j = j0 + i;
    loc[i] = j < wlen ? w.P[j + 1] : 0;
    sum += loc[i];
  }
#pragma unroll
  for (int d = 16; d; d >>= 1) {
    uint32_t o = __shfl_xor_sync(0xffffffffu, mx, d);
    mx = o > mx ? o : mx;
  }
  uint64_t ex = block_excl_scan64(sum, nullptr, w.ws);  // (contains the barrier that orders the smax reset above)
  if ((threadIdx.x & 31) == 0) atomicMax(&w.smax, mx);
#pragma unroll
  for (int i = 0; i < kPer; i++) {
    uint32_t j = j0 + i;
    if (j <= wlen && j <= (uint32_t)kW) w.P[j] = (PT)ex;
    ex += loc[i];
  }
  if (threadIdx.x == 0) {
    w.wlen = wlen;
    w.at_end = (wstart + wlen == n);
  }
  __syncthreads();
  // inclusive scan of Q with stride R, i.e. R independent prefix sums over the residue classes j mod R
  if ((R & (R - 1)) == 0 && R <= 32 && kEncThreads % R == 0) {
    // class c = t % R is shared by kEncThreads / R threads; each walks a contiguous range of its class (consecutive lanes
    // touch consecutive words: no bank conflicts), the partial sums are scanned with shuffles inside the class's threads
    const uint32_t c = threadIdx.x & (R - 1), part = threadIdx.x / R, nparts = kEncThreads / R;
    const uint32_t per_class = (wlen + R - 1) / R;                   // elements of the longest class
    const uint32_t chunk = (per_class + nparts - 1) / nparts;        // elements per thread
    const uint32_t first = part * chunk;                             // first element (within the class) of this thread
    uint32_t sum = 0;
    for (uint32_t i = 0; i < chunk; i++) {
      const uint32_t j = c + R * (first + i);
      if (j < wlen) sum += w.Q[j];
    }
    // exclusive scan of `sum` over the parts of class c: the parts of a class sit R threads apart
    __shared__ uint32_t part_sum[kEncThreads];
    part_sum[threadIdx.x] = sum;
    __syncthreads();
    uint32_t run = 0;
    for (uint32_t q = 0; q < part; q++) run += part_sum[c + R * q];
    for (uint32_t i = 0; i < chunk; i++) {
      const uint32_t j = c + R * (first + i);
      if (j < wlen) {
        run += w.Q[j];
        w.Q[j] = run;
      }
    }
    __syncthreads();
  } else {
    // generic restart interval: Hillis-Steele doubling
    for (uint32_t off = R; off < wlen; off <<= 1) {
      uint32_t add[kPer];
#pragma unroll
      for (int i = 0; i < kPer; i++) {
        uint32_t j = j0 + i;
        add[i] = (j < wlen && j >= off) ? w.Q[j - off] : 0;
      }
      __syncthreads();
#pragma unroll
      for (int i = 0; i < kPer; i++) {
        uint32_t j = j0 + i;
        if (j < wlen) w.Q[j] += add[i];
      }
      __syncthreads();
    }
  }
}

struct CutParams {
  uint32_t BS, LIM, R, rshift;  // rshift = log2(R) when R is a power of two, else 32
};
__host__ __device__ __forceinline__ CutParams make_cut(uint32_t bs, uint32_t lim, uint32_t r) {
  CutParams c{bs, lim, r, 32};
  if ((r & (r - 1)) == 0) {
    uint32_t sft = 0;
    while ((1u << sft) < r) sft++;
    c.rshift = sft;
  }
  return c;
}
__device__ __forceinline__ uint32_t div_r(uint32_t x, const CutParams& cp) { return cp.rshift < 32 ? x >> cp.rshift : x / cp.R; }
// payload bytes of a block holding window entries [a, b).  The terms that depend on the block start alone (P[a], Q[a - R]) are
// loaded once per start (BlockStart) instead of once per probe: the bisection below evaluates this several times per start.
template <typename PT>
struct BlockStart {
  uint32_t a;
  PT pa;        // P[a]
  uint32_t qa;  // Q[a - R] (0 when a < R)
};
template <typename PT>
__device__ __forceinline__ BlockStart<PT> block_start(const Window<PT>& w, uint32_t a, const CutParams& cp) {
  BlockStart<PT> s;
  s.a = a;
  s.pa = w.P[a];
  s.qa = a >= cp.R ? w.Q[a - cp.R] : 0u;
  return s;
}
// Block sizes are computed in the window's own integer type: 32 bits in the narrow window (the launcher picks it only when
// (largest entry + 64) x window length < 2^32, which bounds every sum formed here), 64 bits otherwise.
template <typename PT>
__device__ __forceinline__ PT blk_payload(const Window<PT>& w, const BlockStart<PT>& s, uint32_t b, const CutParams& cp) {
  const uint32_t nrm1 = div_r(b - 1 - s.a, cp);  // restarts - 1
  const uint32_t last = s.a + cp.R * nrm1;
  // Q is a per-residue prefix sum of 32-bit surcharges inside one window: the difference fits 32 bits
  const uint32_t q = w.Q[last] - s.qa;
  return (PT)(w.P[b] - s.pa) + (PT)q + (PT)(4u * (nrm1 + 1) + 4u);  // == BlockBuilder::CurrentSizeEstimate() (block_builder.cc:97,251)
}
template <typename PT>
__device__ __forceinline__ PT blk_payload(const Window<PT>& w, uint32_t a, uint32_t b, const CutParams& cp) {
  return blk_payload(w, block_start(w, a, cp), b, cp);
}
// first b > a at which FlushBlockBySizePolicy::Update (flush_block_policy.cc:37-69) fires for a block started at a.
// returns wlen at the end of the stream, 0xffffffff if the block does not end inside the window; *pay_out = payload bytes of [a, b).
// hint: a position near the answer (where the block of the neighbouring start ended, or start + block bytes / mean entry size):
// the search gallops away from it and bisects the bracket -- two probes when the hint is one off.  0 = none.
template <typename PT>
__device__ __forceinline__ uint32_t next_block(const Window<PT>& w, uint32_t a, const CutParams& cp, uint32_t hint, PT* pay_out) {
  const uint32_t wlen = w.wlen;
  const BlockStart<PT> bs = block_start(w, a, cp);
  // below `thr` neither flush condition can fire: condition 2 needs CurrentSizeEstimate > LIM and
  // CurrentSizeEstimate + (size of the next entry, at most smax + 7) > BS
  PT thr = (PT)(cp.BS - 1);
  if (cp.LIM) {
    thr = (PT)cp.LIM;
    const uint64_t guard = (uint64_t)w.smax + 7;
    if (cp.BS > guard && cp.BS - guard - 1 > thr) thr = (PT)(cp.BS - guard - 1);
  }
  // the first b in [lo, hi) with CurrentSizeEstimate(a, b) > thr (the estimate grows with b); hi = wlen + 1: none seen yet
  uint32_t lo = a + 1, hi = wlen + 1;
  PT ec_hi = 0;  // the estimate at hi (when hi <= wlen)
  if (hint > a + 1 && hint <= wlen) {
    const PT ph = blk_payload(w, bs, hint, cp);
    uint32_t step = 1;
    if (ph > thr) {
      hi = hint;
      ec_hi = ph;
      while (hi - lo >= step) {
        const uint32_t mid = hi - step;
        const PT pm = blk_payload(w, bs, mid, cp);
        if (pm > thr) {
          hi = mid;
          ec_hi = pm;
          step <<= 1;
        } else {
          lo = mid + 1;
          break;
        }
      }
    } else {
      lo = hint + 1;
      while (lo + step - 1 <= wlen) {
        const uint32_t mid = lo + step - 1;
        const PT pm = blk_payload(w, bs, mid, cp);
        if (pm > thr) {
          hi = mid;
          ec_hi = pm;
          break;
        }
        lo = mid + 1;
        step <<= 1;
      }
    }
  }
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    const PT pm = blk_payload(w, bs, mid, cp);
    if (pm > thr) {
      hi = mid;
      ec_hi = pm;
    } else {
      lo = mid + 1;
    }
  }
  if (lo >= wlen) {
    if (!w.at_end) return 0xffffffffu;
    *pay_out = blk_payload(w, bs, wlen, cp);
    return wlen;
  }
  PT ec = ec_hi;            // CurrentSizeEstimate before adding entry lo (lo == hi <= wlen was probed); updated incrementally
  uint32_t m = lo - a;      // entries already in the block
  uint32_t mr = cp.rshift < 32 ? (m & (cp.R - 1)) : (m % cp.R);
  for (uint32_t b = lo; b < wlen; b++) {
    if (ec >= cp.BS) {
      *pay_out = ec;
      return b;
    }
    const PT s1 = (PT)(w.P[b + 1] - w.P[b]);
    const bool at_restart = mr == 0;  // entry b would open a new restart interval
    const PT d = at_restart ? (PT)(w.Q[b] - (b >= cp.R ? w.Q[b - cp.R] : 0u)) : (PT)0;
    if (cp.LIM) {  // BlockAlmostFull: EstimateSizeAfterKV (block_builder.cc:97-126) = ec + |k|+|v|+4+varints (+4 at a restart)
      const PT dfull = at_restart ? d : (PT)(w.Q[b] - (b >= cp.R ? w.Q[b - cp.R] : 0u));
      if (ec + s1 + dfull + 3 + (at_restart ? 4 : 0) > cp.BS) {
        *pay_out = ec;
        return b;
      }
    }
    ec += s1 + (at_restart ? d + 4 : 0);
    mr = mr + 1 == cp.R ? 0 : mr + 1;
  }
  if (!w.at_end) return 0xffffffffu;
  *pay_out = ec;
  return wlen;
}

constexpr int kEncGroup = kEncGroupTiles;  // tiles per group
// loads that must see what OTHER CTAs of a still running kernel wrote (guarded by a flag / counter): L2 only, never a stale L1 line
__device__ __forceinline__ TileRow ldcg_row(const TileRow* p) {
  const uint4 v = __ldcg(reinterpret_cast<const uint4*>(p));
  TileRow r;
  r.exit = v.x;
  r.nblk = v.y;
  r.bytes = (uint64_t)v.z | ((uint64_t)v.w << 32);
  return r;
}
static_assert(sizeof(TileRow) == 16, "TileRow is moved as one 16-byte vector");

// ---- the row walk: a chain position (entry, blocks, bytes) crosses a span (tile or group) by the span's row of its entry point
// r = row of entry point cc of a span whose rows start at `rows`; false when cc is not tabulated (cc >= hc, or the chain from cc
// leaves the window).  kL2: the rows are written by other CTAs of the running tables kernel
template <bool kL2 = false>
__device__ __forceinline__ bool tabulated_row(const TileRow* rows, uint64_t cc, uint32_t hc, TileRow& r) {
  if (cc >= hc) return false;
  r = kL2 ? ldcg_row(rows + cc) : rows[cc];
  return r.exit != 0xffffffffu;
}
// moves the chain position past the span starting at entry `start` by its row r
__device__ __forceinline__ void follow_row(const TileRow& r, uint64_t start, uint64_t& a, uint64_t& blk, uint64_t& bytes) {
  a = start + r.exit;
  blk += r.nblk;
  bytes += r.bytes;
}
// the row of entry point x of a tile whose nxt / disk sit in shared memory: follows nxt to the first block start behind the tile's
// tl entries (exit 0xffffffff: a block does not end inside the window).  mark != nullptr: flags every block start on the way
__device__ __forceinline__ TileRow follow_nxt(const uint16_t* nxt, const uint32_t* disk, uint32_t x, uint32_t tl, uint8_t* mark = nullptr) {
  TileRow r{0, 0, 0};
  while (x < tl) {
    const uint32_t y = nxt[x];
    if (y == 0xffff || y <= x) {
      r.exit = 0xffffffffu;
      return r;
    }
    if (mark) mark[x] = 1;
    r.bytes += disk[x];
    r.nblk++;
    x = y;
  }
  r.exit = x;
  return r;
}
// The one descend rule of the stitch walk and the block list: a span cannot be crossed by its row r (from the chain position
// whose file holds `foff` bytes) when the row is not tabulated, the size rule fires inside, the stream ends inside, or a grandparent
// boundary or partition event (next_ev: the next event of the rules, or in the block list the next recorded cut) lies inside.
__device__ __forceinline__ bool must_descend(bool tabulated, const TileRow& r, uint64_t start, uint64_t n, uint64_t foff,
                                             const EncodeParams& ep, uint64_t next_ev) {
  return !tabulated || (ep.output_level != 0 && foff + r.bytes >= ep.max_output_file_size) || start + r.exit >= n ||
         next_ev <= start + r.exit;
}

// composes the transfer functions of the tiles [t0, t1) of group g per entry-point candidate (all threads of the CTA)
__device__ void compose_group(const EncodeWork& wk, uint64_t n, uint64_t g, uint64_t t0, uint64_t t1, uint32_t hc) {
  const uint64_t gstart = t0 * (uint64_t)kTT;
  for (uint32_t c = threadIdx.x; c < hc; c += blockDim.x) {
    uint64_t x = gstart + c, blk = 0, bytes = 0;
    bool ok = true;
    for (uint64_t t = t0; t < t1 && x < n; t++) {
      const uint64_t tstart = t * (uint64_t)kTT, tend = (tstart + kTT) < n ? (tstart + kTT) : n;
      if (x >= tend) continue;  // no block starts in this tile
      TileRow r;
      if (!(ok = tabulated_row<true>(wk.rows + t * hc, x - tstart, hc, r))) break;
      follow_row(r, tstart, x, blk, bytes);
    }
    wk.grows[g * hc + c] = TileRow{ok ? (uint32_t)(x - gstart) : 0xffffffffu, (uint32_t)blk, bytes};  // exit relative to the group
  }
}

// per tile: nxt / disk for every block start inside the tile, then the transfer function for hc entry points
template <typename PT>
struct TablesSmem {
  Window<PT> w;
  uint16_t nxt[kTT];   // window-relative end of the block that starts at j (0xffff = does not fit the window)
  uint32_t disk[kTT];  // on-disk bytes of that block (payload + 5-byte trailer)
};
template <typename PT>
__global__ void __launch_bounds__(kEncThreads, sizeof(PT) == 4 ? 3 : 2)
encode_tables_kernel(KeyCols m, EncodeParams ep, EncodeWork wk, uint64_t n, uint32_t hc) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  TablesSmem<PT>& s = *reinterpret_cast<TablesSmem<PT>*>(smem_raw);
  const uint64_t tile = blockIdx.x, wstart = tile * (uint64_t)kTT;
  const CutParams cp = make_cut(ep.block_size, ep.block_size_limit, ep.restart_interval);
  build_window(s.w, m, wk.esz, wk.eshared, n, tile, cp.R);
  const uint32_t tl = s.w.wlen < (uint32_t)kTT ? s.w.wlen : (uint32_t)kTT;
  {
    // thread t owns the 16 consecutive starts [16t, 16t+16) so that the previous answer is a tight hint for the next
    // start; it visits them in the rotated order (i + t) mod 16, which spreads the lanes of a warp over the
    // shared-memory banks (plain blocked order would put all 32 lanes on the same bank pair)
    constexpr int kPer = kTT / kEncThreads;
    // hint of a thread's first start: start + (block bytes / mean entry size of the window); of every later one: where the
    // neighbour's block ended (shifted by their distance when the rotation wraps from start 15 to start 0)
    const PT total = s.w.P[s.w.wlen];
    const uint32_t per_block = total ? (uint32_t)(((uint64_t)ep.block_size * s.w.wlen) / total) : 0;
    uint32_t prev_pos = 0, prev_b = 0;
    for (int i = 0; i < kPer; i++) {
      const uint32_t j = threadIdx.x * kPer + ((i + threadIdx.x) & (kPer - 1));
      if (j >= tl) continue;
      uint32_t hint = j + 1 + per_block;
      if (prev_b) hint = prev_b + j - prev_pos;  // (unsigned wrap when j < prev_pos is intended)
      if (hint > s.w.wlen) hint = s.w.wlen;
      PT pay = 0;
      uint32_t b = next_block(s.w, j, cp, hint, &pay);
      prev_pos = j;
      prev_b = b == 0xffffffffu ? 0 : b;
      uint16_t nx = 0xffff;
      uint32_t dk = 0;
      if (b != 0xffffffffu) {
        nx = (uint16_t)b;
        const uint64_t pay5 = (uint64_t)pay + 5;
        dk = pay5 > 0xffffffffull ? 0xffffffffu : (uint32_t)pay5;
      }
      s.nxt[j] = nx;
      s.disk[j] = dk;
    }
  }
  __syncthreads();
  for (uint32_t j = threadIdx.x; j < tl; j += kEncThreads) {  // coalesced copy for the block-list pass
    wk.nxt[wstart + j] = s.nxt[j];
    wk.disk[wstart + j] = s.disk[j];
  }
  __syncthreads();
  // exit window-relative: >= tile length unless the stream ended
  for (uint32_t c = threadIdx.x; c < hc; c += kEncThreads) wk.rows[tile * hc + c] = follow_nxt(s.nxt, s.disk, c, tl);
  // ---- group completion: the last tile CTA of a group of kEncGroup tiles composes the group's transfer function and raises the
  // group's ready flag; the stitch kernel runs concurrently on its own stream and consumes the groups as they appear
  __threadfence();  // this thread's nxt / disk / rows stores are visible device-wide before the counter moves
  __syncthreads();
  __shared__ uint32_t s_last;
  const uint64_t g = tile / kEncGroupTiles, ntiles = (n + kTT - 1) / kTT;
  const uint64_t t0 = g * kEncGroupTiles, t1 = (t0 + kEncGroupTiles) < ntiles ? (t0 + kEncGroupTiles) : ntiles;
  if (threadIdx.x == 0) s_last = atomicAdd(&wk.gdone[g], 1u) + 1 == (uint32_t)(t1 - t0);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  compose_group(wk, n, g, t0, t1, hc);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) atomicExch(&wk.gready[g], 1u);
}

// ------------------------------------------------------------------------------------------------ stitch
// The chain of block starts is resolved hierarchically:
//   encode_compose    composes the transfer functions of kEncGroup consecutive tiles per entry-point candidate
//   encode_stitch     one CTA walks the group functions (a few hundred dependent steps); only groups in which an
//                     output file ends are walked tile by tile, and only the tiles in which a file ends are walked
//                     block by block (pointer chasing through nxt/disk staged in shared memory)
//   encode_tilestate  per group: entry state of every tile, from the group's entry state
struct WalkState {
  uint64_t a;         // absolute entry index where the open block starts
  uint64_t blk;       // blocks completed so far
  uint64_t foff;      // bytes flushed to the current file
  uint64_t f_first_entry, f_first_blk;
  uint32_t f;         // current file index
};
__device__ __forceinline__ void close_file(FileRec* files, WalkState& st, uint64_t end_entry, uint32_t* err) {
  if (files == nullptr) return;  // block-list pass: the stitch kernel already wrote the file records
  if (st.f >= kMaxOutFiles) {  // a documented limit of the device rule set, not a fault: nothing is written past the records
    atomicOr(err, kErrTooManyFiles);
    return;
  }
  FileRec& fr = files[st.f];
  fr.first_entry = st.f_first_entry;
  fr.n_entries = end_entry - st.f_first_entry;
  fr.first_block = st.f_first_blk;
  fr.n_blocks = st.blk - st.f_first_blk;
  fr.data_size = st.foff;
  fr.index_size = 0;
  fr.raw_key_size = fr.raw_value_size = fr.num_deletions = 0;
  fr.smallest_seq = ~0ull;
  fr.largest_seq = 0;
  fr.index_has_seq = 0;
  fr.filter_entries = fr.filter_bytes = 0;
}
// on-disk bytes of a data block that holds the single entry y
__device__ __forceinline__ uint64_t single_entry_block_bytes(const KeyCols& m, const EncodeWork& wk, uint64_t y) {
  return (uint64_t)wk.esz[y] + restart_surcharge(wk.eshared[y], meta_ulen(m.meta[y]) + 8) + 4 + 4 + 5;
}
// ---- grandparent boundaries on entry ranks: the state machine itself is gp_rules.h (host + device)
// index of the first of the ncuts recorded cuts (sorted by entry) behind `entry`
__device__ __forceinline__ uint32_t first_cut_after(const EncodeParams& ep, uint32_t ncuts, uint64_t entry) {
  uint32_t lo = 0, hi = ncuts;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (ep.gp_cuts[mid].entry <= entry) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}
// on-disk bytes (payload + trailer) of a block holding the entries [a, e): what BlockBuilder would have written had the block
// been flushed there (every restart entry is stored with shared == 0)
__device__ uint64_t truncated_block_bytes(const KeyCols& m, const EncodeWork& wk, uint32_t R, uint64_t a, uint64_t e) {
  uint64_t sum = 0;
  for (uint64_t j0 = a; j0 < e; j0 += 8) {
    uint32_t s1[8], sh[8], mt[8];
#pragma unroll
    for (int q = 0; q < 8; q++) {
      const uint64_t j = j0 + q;
      s1[q] = sh[q] = mt[q] = 0;
      if (j < e) {
        s1[q] = wk.esz[j];
        sh[q] = wk.eshared[j];
        mt[q] = m.meta[j];
      }
    }
#pragma unroll
    for (int q = 0; q < 8; q++) {
      const uint64_t j = j0 + q;
      if (j < e) {
        sum += s1[q];
        if ((j - a) % R == 0) sum += restart_surcharge(sh[q], meta_ulen(mt[q]) + 8);
      }
    }
  }
  const uint64_t nrest = (e - a + R - 1) / R;
  return sum + 4 * nrest + 4 + 5;
}

// Follow the real chain through one tile whose nxt/disk sit in shared memory, applying the output-file cut rules
// (compaction_outputs.cc:277: cut in front of the first entry added after the flushed size reached the maximum; :294-351 the
// grandparent rules).  emit != nullptr: write BlockRecs.  files != nullptr: write FileRecs.
// kGp: 0 = no grandparents or partitioner; 1 = evaluate their rules (stitch; records the cuts); 2 = replay recorded cuts (block list).
// The walk state is copied into registers for the loop (taking its address would put it in local memory and turn every
// step of this single-thread pointer chase into a chain of dependent local loads and stores).
template <int kGp>
__device__ __forceinline__ bool chase_tile(const uint16_t* nxt, const uint32_t* disk, uint64_t tstart, uint32_t tl, uint64_t n,
                                           const EncodeParams& ep, const KeyCols& m, const EncodeWork& wk, WalkState& st_io, FileRec* files,
                                           BlockRec* emit, uint64_t emit_cap, uint32_t* err, GpState* gp_io = nullptr) {
  WalkState st = st_io;
  GpState g{};
  if (kGp == 1) g = *gp_io;
  uint32_t ncuts = 0, cut_i = 0;
  if (kGp == 2) {
    ncuts = *ep.gp_ncuts;
    cut_i = first_cut_after(ep, ncuts, st.a);
  }
  const uint64_t tend = tstart + tl;
  const bool cut_files = ep.output_level != 0;
  const uint64_t fmax = ep.max_output_file_size;
  bool ok = true;
  while (st.a < tend) {
    const uint32_t x = (uint32_t)(st.a - tstart);
    const uint32_t yr = nxt[x];
    if (yr == 0xffff || yr <= x) {
      ok = false;
      break;
    }
    const uint64_t y = tstart + yr;
    if (kGp != 0 && cut_files) {
      // entries a < e <= y are added while the block [a, y) is open: the flushed size they see is st.foff
      uint64_t cut_at = ~0ull, cut_bytes = 0;
      if (kGp == 1) {
        cut_at = gp_block_cut(g, ep.gp, y, n, st.foff);
        if (cut_at != ~0ull) {
          cut_bytes = cut_at == y ? (uint64_t)disk[x] : truncated_block_bytes(m, wk, ep.restart_interval, st.a, cut_at);
          const uint32_t ci = *ep.gp_ncuts;
          ep.gp_cuts[ci] = GpCut{cut_at, cut_bytes};
          *ep.gp_ncuts = ci + 1;
        }
      } else if (cut_i < ncuts && ep.gp_cuts[cut_i].entry <= y) {
        cut_at = ep.gp_cuts[cut_i].entry;
        cut_bytes = ep.gp_cuts[cut_i].block_bytes;
        cut_i++;
      }
      if (cut_at != ~0ull) {  // the file ends in front of entry cut_at: the open block is flushed with the entries [a, cut_at)
        if (emit && st.blk < emit_cap) emit[st.blk] = BlockRec{st.a, st.foff, st.f, (uint32_t)(cut_at - st.a)};
        st.foff += cut_bytes;
        st.blk++;
        close_file(files, st, cut_at, err);
        st.f++;
        st.foff = 0;
        st.f_first_entry = cut_at;
        st.f_first_blk = st.blk;
        st.a = cut_at;
        continue;
      }
    }
    if (emit && st.blk < emit_cap) emit[st.blk] = BlockRec{st.a, st.foff, st.f, (uint32_t)(y - st.a)};
    st.foff += disk[x];
    st.blk++;
    if (y >= n) {  // Finish(): last block of the stream
      close_file(files, st, n, err);
      st.a = n;
      st.f++;
      break;
    }
    if (cut_files && st.foff >= fmax) {
      // entry y (whose Add flushed the block) still goes to this file and ends it as a single-entry block
      const uint64_t d1 = single_entry_block_bytes(m, wk, y);
      if (emit && st.blk < emit_cap) emit[st.blk] = BlockRec{y, st.foff, st.f, 1u};
      st.foff += d1;
      st.blk++;
      close_file(files, st, y + 1, err);
      st.f++;
      st.foff = 0;
      st.f_first_entry = y + 1;
      st.f_first_blk = st.blk;
      st.a = y + 1;
      if (kGp == 1) gp_size_cut(g, ep.gp, y + 1, n);
    } else {
      st.a = y;
    }
  }
  st_io = st;
  if (kGp == 1) *gp_io = g;
  return ok;
}

struct StitchSmem {
  uint16_t nxt[kTT];
  uint32_t disk[kTT];
  uint64_t nd[kTT];       // (nxt << 32) | disk of the tile being chased: one shared-memory load per block link
  WalkState st;
  GpState gp;             // grandparent boundary state of the reference's CompactionOutputs (rules off: untouched)
  uint64_t g, t, tend;    // cursor: next group; next tile / end tile of the group being walked tile by tile
  uint64_t ga, ta;        // first group / tile held by the row caches
  uint32_t gn, tn;        // number of groups / tiles cached
  uint64_t req_idx;       // argument of the request
  uint32_t req;           // 0 none, 1 chase tile req_idx, 2 load group rows from req_idx, 3 load tile rows from req_idx
  uint32_t done;
  uint32_t refill;        // groups taken by the current group-row refill
};
// cooperative global -> shared copy of flag-guarded data (written by CTAs of the concurrently running tables kernel): L2 loads
template <typename T, int kDepth>
__device__ __forceinline__ void coop_copy_cg(T* __restrict__ dst, const T* __restrict__ src, uint32_t n) {
  const uint32_t nt = blockDim.x;
  for (uint32_t base = 0; base < n; base += kDepth * nt) {
    T v[kDepth];
#pragma unroll
    for (int k = 0; k < kDepth; k++) {
      const uint32_t i = base + k * nt + threadIdx.x;
      if (i < n) v[k] = __ldcg(src + i);
    }
#pragma unroll
    for (int k = 0; k < kDepth; k++) {
      const uint32_t i = base + k * nt + threadIdx.x;
      if (i < n) dst[i] = v[k];
    }
  }
}
// The stitch CTA shares the device with the tables kernel (it is launched on its own high-priority stream and needs a free slot on
// one SM next to two tables CTAs), so its row caches are small: 2 x cache_bytes, sized by the launcher from hc.
// Two launches per job.  The walk is one thread chasing dependent loads; next to the warps of a bulk kernel on the same SM it gets
// an issue slot every few cycles only and runs several times slower than alone.  So
//   attempt 1 is launched BEFORE the tables kernel with enough shared memory to keep an SM to itself, and consumes the groups as the
//             tables kernel (on the other SMs) completes them.  A tool that serialises kernels (ncu, compute-sanitizer) would
//             never start the producer while this waits: if the first group does not appear within `timeout_ns` it leaves
//             without having written anything;
//   attempt 2 is launched behind both: it returns at once when attempt 1 finished the walk (`sflag`), else does it.
__global__ void __launch_bounds__(kEncThreads)
encode_stitch_kernel(KeyCols m, EncodeParams ep, EncodeWork wk, uint64_t n, uint64_t ntiles, uint32_t hc, uint32_t cache_bytes,
                     uint32_t* __restrict__ err, uint32_t attempt, uint32_t* __restrict__ sflag, uint32_t timeout_ns) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  StitchSmem& s = *reinterpret_cast<StitchSmem*>(smem_raw);
  if (attempt == 2 && *reinterpret_cast<volatile uint32_t*>(sflag) != 0) return;
  bool first_wait = attempt == 1;
  TileRow* gcache = reinterpret_cast<TileRow*>(smem_raw + ((sizeof(StitchSmem) + 15) & ~(size_t)15));
  TileRow* tcache = gcache + cache_bytes / sizeof(TileRow);
  const uint32_t cache_rows = cache_bytes / (uint32_t)sizeof(TileRow) / hc;  // groups / tiles per cache (>= 1 by the launcher)
  const uint64_t ngroups = (ntiles + kEncGroup - 1) / kEncGroup;
  if (threadIdx.x == 0) {
    s.st = WalkState{0, 0, 0, 0, 0, 0};
    s.gp = gp_initial_state();
    if (gp_rules_on(ep.gp)) {
      *ep.gp_ncuts = 0;
      if (n) gp_advance(s.gp, ep.gp, 0);  // ShouldStopBefore of the first key: no builder yet, but the boundary state moves
    }
    s.done = (n == 0);
    s.req = 0;
    s.g = s.t = s.tend = 0;
    s.ga = s.ta = 0;
    s.gn = s.tn = 0;
  }
  __syncthreads();
  for (;;) {
    if (threadIdx.x == 0) {
      // everything the serial walk touches per step lives in registers; shared memory is read / written once per section
      WalkState st = s.st;
      const GpState gps = s.gp;  // only read here: boundaries are crossed (and the state changes) inside chase_tile
      const uint64_t next_ev = gp_rules_on(ep.gp) ? gp_next_event(gps, ep.gp) : ~0ull;
      uint64_t cg = s.g, ct = s.t, ctend = s.tend;
      const uint64_t cga = s.ga, cta = s.ta;
      const uint32_t cgn = s.gn, ctn = s.tn;
      uint32_t req = 0, fin = 0;
      uint64_t req_idx = 0;
      for (;;) {
        if (st.a >= n) {
          fin = 1;
          break;
        }
        if (ct < ctend) {  // inside a group that is walked tile by tile
          const uint64_t t = ct, tstart = t * (uint64_t)kTT, tend = (tstart + kTT) < n ? (tstart + kTT) : n;
          if (st.a < tend && !(t >= cta && t < cta + ctn)) {
            req = 3;
            req_idx = t;
            break;
          }
          wk.tstate[t] = TileState{st.a, st.blk, st.foff, st.f, 0};
          ct++;
          if (st.a >= tend) continue;  // no block starts in this tile
          TileRow r;
          if (must_descend(tabulated_row(tcache + (t - cta) * hc, st.a - tstart, hc, r), r, tstart, n, st.foff, ep, next_ev)) {
            req = 1;  // chase the tile block by block
            req_idx = t;
            break;
          }
          follow_row(r, tstart, st.a, st.blk, st.foff);
          continue;
        }
        // group level
        if (cg >= ngroups) {
          fin = 1;
          break;
        }
        const uint64_t gg = cg, t0 = gg * kEncGroup, gstart = t0 * (uint64_t)kTT;
        const uint64_t t1 = (t0 + kEncGroup) < ntiles ? (t0 + kEncGroup) : ntiles;
        const uint64_t gend = (t1 * (uint64_t)kTT) < n ? (t1 * (uint64_t)kTT) : n;
        if (st.a < gend && !(gg >= cga && gg < cga + cgn)) {
          req = 2;
          req_idx = gg;
          break;
        }
        wk.gstate[gg] = TileState{st.a, st.blk, st.foff, st.f, 0};
        wk.gflag[gg] = 0;
        cg++;
        if (st.a >= gend) continue;  // no block starts in this group
        TileRow r;
        if (must_descend(tabulated_row(gcache + (gg - cga) * hc, st.a - gstart, hc, r), r, gstart, n, st.foff, ep, next_ev)) {
          wk.gflag[gg] = 1;  // walk the group tile by tile
          ct = t0;
          ctend = t1;
          continue;
        }
        follow_row(r, gstart, st.a, st.blk, st.foff);
      }
      s.st = st;
      s.g = cg;
      s.t = ct;
      s.tend = ctend;
      s.req = req;
      s.req_idx = req_idx;
      if (fin) s.done = 1;
    }
    __syncthreads();
    const uint32_t req = s.req;  // stable: thread 0 writes these again only after the barrier that ends the iteration
    const uint64_t ridx = s.req_idx;
    uint32_t done = s.done;
    if (req == 2 || req == 3) {  // refill a row cache
      // group rows: as many as fit (the walk consumes them quickly); tile rows: only the rest of the group being walked
      const uint64_t total = req == 2 ? ngroups : s.tend;
      uint32_t cnt = (uint32_t)((total - ridx) < cache_rows ? (total - ridx) : cache_rows);
      if (req == 2) {
        // the tables kernel is still running: wait for the first group needed, then take the consecutive groups that are ready too
        if (threadIdx.x == 0) {
          volatile uint32_t* rdy = wk.gready;
          if (first_wait) {
            unsigned long long t0, t1;
            asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t0));
            while (rdy[ridx] == 0) {
              __nanosleep(256);
              asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t1));
              if (t1 - t0 > timeout_ns) {
                s.done = 2;  // give up: the producer is not running
                break;
              }
            }
          } else {
            while (rdy[ridx] == 0) __nanosleep(256);
          }
          uint32_t have = 1;
          while (have < cnt && rdy[ridx + have] != 0) have++;
          s.refill = have;
          __threadfence();
        }
        __syncthreads();
        if (s.done == 2) return;  // (nothing has been written yet: attempt 2 starts from scratch)
        first_wait = false;
        cnt = s.refill;
      }
      // tile rows (req == 3) belong to a group that was ready when its row entered the group cache
      const uint4* src = reinterpret_cast<const uint4*>((req == 2 ? wk.grows : wk.rows) + ridx * hc);
      uint4* dst = reinterpret_cast<uint4*>(req == 2 ? gcache : tcache);
      coop_copy_cg<uint4, 8>(dst, src, cnt * hc);
      if (threadIdx.x == 0) {
        if (req == 2) {
          s.ga = ridx;
          s.gn = cnt;
        } else {
          s.ta = ridx;
          s.tn = cnt;
        }
      }
    } else if (req == 1) {
      const uint64_t tstart = ridx * (uint64_t)kTT;
      const uint32_t tl = (uint32_t)(((tstart + kTT) < n ? (tstart + kTT) : n) - tstart);
      // only the part of the tile the chain can still touch: from the walk's position on (16-byte vectors: the tile starts are
      // multiples of kTT, so element c0 = position rounded down to 8 is 16-byte aligned in both arrays)
      const uint32_t c0 = (uint32_t)(s.st.a > tstart ? (s.st.a - tstart) & ~7ull : 0);
      const uint32_t c1 = (tl + 7u) & ~7u;  // (the arrays are allocated past n: reading up to 7 elements behind the end is harmless)
      coop_copy_cg<uint4, 4>(reinterpret_cast<uint4*>(s.nxt + c0), reinterpret_cast<const uint4*>(wk.nxt + tstart + c0), (c1 - c0) / 8);
      coop_copy_cg<uint4, 8>(reinterpret_cast<uint4*>(s.disk + c0), reinterpret_cast<const uint4*>(wk.disk + tstart + c0), (c1 - c0) / 4);
      __syncthreads();
      if (!gp_rules_on(ep.gp)) {
        for (uint32_t i = c0 + threadIdx.x; i < tl; i += blockDim.x) s.nd[i] = ((uint64_t)s.nxt[i] << 32) | s.disk[i];
        __syncthreads();
      }
      if (threadIdx.x == 0) {
        WalkState st = s.st;
        GpState g = s.gp;
        bool chased = true;
        if (gp_rules_on(ep.gp)) {
          chased = chase_tile<1>(s.nxt, s.disk, tstart, tl, n, ep, m, wk, st, wk.files, nullptr, 0, err, &g);
        } else {
          // Without grandparents or a partitioner the only events on the chain are the size rule and the end of the stream.  The walk is one thread
          // chasing dependent loads, so the common link is kept to a single 8-byte shared-memory load and a dozen 32-bit instructions
          // (the general loop costs ~320 cycles per link, measured with clock64: 58 links per file cut); the block in which an event
          // happens goes through the exact rule (chase_tile over that one block).
          const uint32_t nd_base = (uint32_t)__cvta_generic_to_shared(s.nd);
          const uint64_t left = n - tstart;
          const uint32_t nlocal = left < 0xffffull ? (uint32_t)left : 0xffffu;  // y >= n  <=>  yr >= nlocal  (0xffff: no block end tabulated)
          const bool cut_files = ep.output_level != 0;
          const uint64_t fmax = ep.max_output_file_size;
          uint32_t x = (uint32_t)(st.a - tstart);
          uint64_t foff = st.foff, blk = st.blk;
          while (x < tl) {
            for (;;) {
              uint64_t v;
              asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(nd_base + 8u * x));
              const uint32_t yr = (uint32_t)(v >> 32), d = (uint32_t)v;
              const uint64_t nf = foff + d;
              if (yr <= x || yr >= nlocal || (cut_files && nf >= fmax)) break;  // an event (or a broken link): exact rule below
              foff = nf;
              blk++;
              x = yr;
              if (x >= tl) break;
            }
            if (x >= tl) break;
            st.a = tstart + x;
            st.foff = foff;
            st.blk = blk;
            chased = chase_tile<0>(s.nxt, s.disk, tstart, x + 1, n, ep, m, wk, st, wk.files, nullptr, 0, err);
            if (!chased || st.a >= n) break;
            x = (uint32_t)(st.a - tstart);  // (behind the tile when the block ended there: the loop ends)
            foff = st.foff;
            blk = st.blk;
          }
          if (chased && st.a < n && x >= tl && st.a < tstart + x) {
            st.a = tstart + x;
            st.foff = foff;
            st.blk = blk;
          }
        }
        s.gp = g;
        if (!chased) {
          atomicOr(err, kErrBlockTooLong);
          s.done = 1;
        }
        s.st = st;
      }
      __syncthreads();
      done = s.done;
    }
    __syncthreads();
    if (done) break;
  }
  if (threadIdx.x == 0) {
    wk.totals[0] = s.st.blk;
    wk.totals[1] = s.st.f;
    // groups / tiles never entered (the stream ended before them) start past the end
    TileState ts{n, s.st.blk, 0, s.st.f, 0};
    for (uint64_t t = s.t; t < s.tend; t++) wk.tstate[t] = ts;
    for (uint64_t gg = s.g; gg < ngroups; gg++) {
      wk.gstate[gg] = ts;
      wk.gflag[gg] = 0;
    }
    __threadfence();
    if (attempt == 1) atomicExch(sflag, 1u);
  }
}

// per group: entry state of each of its tiles (groups walked tile by tile by the stitch kernel already have them)
__global__ void encode_tilestate_kernel(EncodeWork wk, uint64_t n, uint64_t ntiles, uint32_t hc, uint32_t* __restrict__ err) {
  const uint64_t g = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const uint64_t ngroups = (ntiles + kEncGroup - 1) / kEncGroup;
  if (g >= ngroups || wk.gflag[g]) return;
  const TileState gs = wk.gstate[g];
  uint64_t a = gs.entry, blk = gs.blk, foff = gs.file_off;
  const uint64_t t0 = g * kEncGroup, t1 = (t0 + kEncGroup) < ntiles ? (t0 + kEncGroup) : ntiles;
  for (uint64_t t = t0; t < t1; t++) {
    const uint64_t tstart = t * (uint64_t)kTT, tend = (tstart + kTT) < n ? (tstart + kTT) : n;
    TileState ts{a < n ? a : n, blk, foff, gs.file_idx, 0};
    wk.tstate[t] = ts;
    if (a >= n || a >= tend) continue;
    TileRow r;
    if (!tabulated_row(wk.rows + t * hc, a - tstart, hc, r)) {
      atomicOr(err, kErrBlockTooLong);
      return;
    }
    follow_row(r, tstart, a, blk, foff);
  }
}

// ------------------------------------------------------------------------------------------------ block list
struct BlistSmem {
  uint16_t nxt[kTT];
  uint32_t disk[kTT];
  uint8_t is_start[kTT];
  uint64_t ws[33];
  uint32_t serial;
};
__global__ void __launch_bounds__(kEncThreads)
encode_blocklist_kernel(KeyCols m, EncodeParams ep, EncodeWork wk, uint64_t n, uint64_t nblk_cap, uint32_t* __restrict__ err) {
  __shared__ BlistSmem s;
  const uint64_t tile = blockIdx.x, tstart = tile * (uint64_t)kTT;
  const uint64_t tend = (tstart + kTT) < n ? (tstart + kTT) : n;
  const uint32_t tl = (uint32_t)(tend - tstart);
  const TileState ts = wk.tstate[tile];
  if (ts.entry >= tend) return;  // no block starts here
  for (uint32_t j = threadIdx.x; j < tl; j += kEncThreads) {
    s.nxt[j] = wk.nxt[tstart + j];
    s.disk[j] = wk.disk[tstart + j];
    s.is_start[j] = 0;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // follow the chain, marking the block starts; a file ends inside this tile when the stitch walk would have descended into it,
    // with the recorded grandparent cuts in place of the rules' events
    const TileRow r = follow_nxt(s.nxt, s.disk, (uint32_t)(ts.entry - tstart), tl, s.is_start);
    const bool bad = r.exit == 0xffffffffu;
    if (bad) atomicOr(err, kErrBlockTooLong);
    uint64_t next_cut = ~0ull;
    if (gp_rules_on(ep.gp) && !bad) {
      const uint32_t nc = *ep.gp_ncuts, ci = first_cut_after(ep, nc, ts.entry);
      if (ci < nc) next_cut = ep.gp_cuts[ci].entry;
    }
    s.serial = bad ? 2 : must_descend(true, r, tstart, n, ts.file_off, ep, next_cut) ? 1 : 0;
    if (s.serial == 1) {  // an output file ends inside this tile: replay the exact serial rule
      WalkState st;
      st.a = ts.entry;
      st.blk = ts.blk;
      st.foff = ts.file_off;
      st.f = ts.file_idx;
      st.f_first_entry = 0;
      st.f_first_blk = 0;
      const bool chased = gp_rules_on(ep.gp) ? chase_tile<2>(s.nxt, s.disk, tstart, tl, n, ep, m, wk, st, nullptr, wk.blocks, nblk_cap, err)
                                  : chase_tile<0>(s.nxt, s.disk, tstart, tl, n, ep, m, wk, st, nullptr, wk.blocks, nblk_cap, err);
      if (!chased) atomicOr(err, kErrBlockTooLong);
    }
  }
  __syncthreads();
  if (s.serial != 0) return;
  // parallel path: ranks and byte offsets of the block starts
  constexpr int kPer = kTT / kEncThreads;  // 16
  const uint32_t j0 = threadIdx.x * kPer;
  uint32_t cnt = 0;
  uint64_t bytes = 0;
#pragma unroll
  for (int i = 0; i < kPer; i++) {
    uint32_t j = j0 + i;
    if (j < tl && s.is_start[j]) {
      cnt++;
      bytes += s.disk[j];
    }
  }
  uint64_t packed = ((uint64_t)cnt << 48) | bytes;  // tile bytes < 2^48, count < 2^16
  uint64_t ex = block_excl_scan64(packed, nullptr, s.ws);
  uint64_t r = ts.blk + (ex >> 48), off = ts.file_off + (ex & ((1ull << 48) - 1));
#pragma unroll
  for (int i = 0; i < kPer; i++) {
    uint32_t j = j0 + i;
    if (j < tl && s.is_start[j]) {
      if (r < nblk_cap) wk.blocks[r] = BlockRec{tstart + j, off, ts.file_idx, (uint32_t)(s.nxt[j] - j)};
      r++;
      off += s.disk[j];
    }
  }
}

// bytes of the index entries of file fr's first k blocks (k <= n_blocks): idx_eoff scans the entry sizes of all blocks without the
// 8 trailer bytes an index with sequence numbers adds to every key
__device__ __forceinline__ uint64_t index_entries_bytes(const EncodeWork& wk, const FileRec& fr, uint64_t k) {
  return wk.idx_eoff[fr.first_block + k] - wk.idx_eoff[fr.first_block] + 8 * fr.index_has_seq * k;
}

// ------------------------------------------------------------------------------------------------ per-file statistics
// One CTA per output file: stat tiles (merge tiles, or kEncTile entries on the TableBuilder-only path) that lie inside the file come
// from their partial sums, the partly covered ones at its ends are read entry by entry; also the file's smallest / largest key and
// the size of its index block (the index entries' sizes and their scan are complete: launch_encode_index_size runs first).
// Stat tile t covers the entries [prefix(t - 1), prefix(t)).
__global__ void encode_filestats_kernel(KeyCols m, EncodeWork wk, uint32_t nfiles) {
  const uint32_t f = blockIdx.x;
  if (f >= nfiles) return;
  const uint64_t f0 = wk.files[f].first_entry, f1 = f0 + wk.files[f].n_entries;
  __shared__ unsigned long long red[5];
  stat_slots_init(red, threadIdx.x);
  __syncthreads();
  StatAcc<unsigned long long> st;
  if (f1 > f0) {
    auto tile_start = [&](uint64_t t) -> uint64_t { return t ? lb_value(wk.tprefix[t - 1]) : 0; };
    auto first_tile_starting_at_or_after = [&](uint64_t e) -> uint64_t {  // tile starts are non-decreasing
      uint64_t lo = 0, hi = wk.nstat;
      while (lo < hi) {
        const uint64_t mid = lo + ((hi - lo) >> 1);
        if (tile_start(mid) < e) lo = mid + 1;
        else hi = mid;
      }
      return lo;
    };
    const uint64_t tA = first_tile_starting_at_or_after(f0);
    uint64_t tB = 0;  // first tile that ends behind f1: the tiles [tA, tB) lie inside the file
    {
      uint64_t lo = 0, hi = wk.nstat;
      while (lo < hi) {
        const uint64_t mid = lo + ((hi - lo) >> 1);
        if (lb_value(wk.tprefix[mid]) <= f1) lo = mid + 1;
        else hi = mid;
      }
      tB = lo;
    }
    auto scan_entries = [&](uint64_t lo, uint64_t hi) {
      for (uint64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        const uint32_t mt = m.meta[i];
        st.add_entry(meta_ulen(mt) + 8, meta_vlen(mt), m.tr[i]);
      }
    };
    if (tA >= tB) {
      scan_entries(f0, f1);  // the file covers no whole stat tile
    } else {
      scan_entries(f0, tile_start(tA));
      scan_entries(lb_value(wk.tprefix[tB - 1]), f1);
      for (uint64_t t = tA + threadIdx.x; t < tB; t += blockDim.x) {
        const TileStat ts = wk.tstat[t];
        st.add(ts.raw_key, ts.raw_value, ts.deletions, ts.smallest_seq, ts.largest_seq);
      }
    }
    if (threadIdx.x < 2) {  // boundary keys
      const uint64_t i = threadIdx.x == 0 ? f0 : f1 - 1;
      const ulonglong2 p = m.pfx[i];
      const KeyRec kr{p.x, p.y, m.tr[i], meta_ulen(m.meta[i]), 0};
      if (threadIdx.x == 0) wk.files[f].smallest = kr;
      else wk.files[f].largest = kr;
    }
  }
  st.flush(red);
  __syncthreads();
  if (threadIdx.x == 0) {
    wk.files[f].raw_key_size = red[0];
    wk.files[f].raw_value_size = red[1];
    wk.files[f].num_deletions = red[2];
    wk.files[f].smallest_seq = red[3];
    wk.files[f].largest_seq = red[4];
    const uint64_t nb = wk.files[f].n_blocks;
    if (nb) wk.files[f].index_size = index_entries_bytes(wk, wk.files[f], nb) + 4 * nb + 4;  // entries | restart array | restart count
  }
}

// ------------------------------------------------------------------------------------------------ emit data blocks
constexpr int kEmitWarps = 4;
// internal key bytes [sh, sh + n) (n <= 24) as three little-endian words, from the columnar (hi, lo, ulen, trailer) form
__device__ __forceinline__ void key_suffix_words(uint64_t hi, uint64_t lo, uint32_t ulen, uint64_t tr, uint32_t sh, uint64_t* S0,
                                                 uint64_t* S1, uint64_t* S2) {
  const uint64_t U0 = bswap64(hi), U1 = bswap64(lo);  // user key bytes in memory order (zero padded beyond ulen)
  uint64_t I0, I1, I2;
  {
    const uint32_t ws = ulen >> 3, bs = (ulen & 7) * 8;
    const uint64_t T0 = tr << bs, T1 = bs ? tr >> (64 - bs) : 0;
    if (ws == 0) {
      I0 = U0 | T0;
      I1 = T1;
      I2 = 0;
    } else if (ws == 1) {
      I0 = U0;
      I1 = U1 | T0;
      I2 = T1;
    } else {
      I0 = U0;
      I1 = U1;
      I2 = tr;
    }
  }
  const uint32_t ws = sh >> 3, bs = (sh & 7) * 8;
  const uint64_t A = ws == 0 ? I0 : ws == 1 ? I1 : ws == 2 ? I2 : 0;
  const uint64_t B = ws == 0 ? I1 : ws == 1 ? I2 : 0;
  const uint64_t Cw = ws == 0 ? I2 : 0;
  *S0 = bs ? (A >> bs) | (B << (64 - bs)) : A;
  *S1 = bs ? (B >> bs) | (Cw << (64 - bs)) : B;
  *S2 = Cw >> bs;
}
// L (<= 27) bytes held in seven little-endian words w[0..7) (w[7] must be 0) to an arbitrarily aligned shared-memory
// address: at most 3 head bytes, aligned 32-bit stores, at most 3 tail bytes -- instead of one store per byte
__device__ __forceinline__ void store_stream28(uint8_t* p, const uint32_t* w, uint32_t L) {
  uint32_t head = (4 - (uint32_t)((uintptr_t)p & 3)) & 3;
  if (head > L) head = L;
  if (head > 0) p[0] = (uint8_t)w[0];
  if (head > 1) p[1] = (uint8_t)(w[0] >> 8);
  if (head > 2) p[2] = (uint8_t)(w[0] >> 16);
  const uint32_t bs = head * 8, nwords = (L - head) >> 2;
  uint32_t* d32 = reinterpret_cast<uint32_t*>(p + head);
  uint32_t tailv = 0;
#pragma unroll
  for (int k = 0; k < 7; k++) {
    const uint32_t v = __funnelshift_r(w[k], w[k + 1], bs);
    if ((uint32_t)k < nwords) d32[k] = v;
    if ((uint32_t)k == nwords) tailv = v;
  }
  const uint32_t done = head + 4 * nwords, rem = L - done;
  if (rem > 0) p[done] = (uint8_t)tailv;
  if (rem > 1) p[done + 1] = (uint8_t)(tailv >> 8);
  if (rem > 2) p[done + 2] = (uint8_t)(tailv >> 16);
}
// n (<= 24) bytes of (S0, S1, S2) to an arbitrarily aligned (shared-memory) address
__device__ __forceinline__ void store_bytes24(uint8_t* p, uint64_t S0, uint64_t S1, uint64_t S2, uint32_t n) {
#pragma unroll
  for (int k = 0; k < 8; k++)
    if ((uint32_t)k < n) p[k] = (uint8_t)(S0 >> (8 * k));
#pragma unroll
  for (int k = 0; k < 8; k++)
    if ((uint32_t)(8 + k) < n) p[8 + k] = (uint8_t)(S1 >> (8 * k));
#pragma unroll
  for (int k = 0; k < 8; k++)
    if ((uint32_t)(16 + k) < n) p[16 + k] = (uint8_t)(S2 >> (8 * k));
}
// n value bytes whose aligned source words w[0..NW) are already in registers (w[NW] must be 0) to an arbitrarily aligned
// shared-memory address: byte stores only for the unaligned head / tail of the destination, 4-byte stores in between;
// a = source misalignment, n <= 4 * (NW - 1) bytes
template <int NW>
__device__ __forceinline__ void store_value_words(uint8_t* dst, const uint32_t* w, uint32_t a, uint32_t n) {
  if (n == 0) return;
  uint32_t head = (4 - (uint32_t)((uintptr_t)dst & 3)) & 3;
  if (head > n) head = n;
  {
    const uint32_t v = __funnelshift_r(w[0], w[1], a * 8);
    if (head > 0) dst[0] = (uint8_t)v;
    if (head > 1) dst[1] = (uint8_t)(v >> 8);
    if (head > 2) dst[2] = (uint8_t)(v >> 16);
  }
  const uint32_t t0 = a + head, bs = (t0 & 3) * 8;
  const uint32_t nwords = (n - head) >> 2;
  uint32_t* d32 = reinterpret_cast<uint32_t*>(dst + head);
  const uint32_t done = head + 4 * nwords, rem = n - done;  // 0..3 tail bytes
  uint32_t tailv = 0;
  if ((t0 >> 2) == 0) {
#pragma unroll
    for (int mI = 0; mI < NW - 1; mI++) {
      const uint32_t v = __funnelshift_r(w[mI], w[mI + 1], bs);
      if ((uint32_t)mI < nwords) d32[mI] = v;
      if ((uint32_t)mI == nwords) tailv = v;
    }
  } else {
#pragma unroll
    for (int mI = 0; mI < NW - 1; mI++) {
      const uint32_t v = __funnelshift_r(w[mI + 1], mI + 2 <= NW ? w[mI + 2] : 0u, bs);
      if ((uint32_t)mI < nwords) d32[mI] = v;
      if ((uint32_t)mI == nwords) tailv = v;
    }
  }
  if (rem) {
    dst[done] = (uint8_t)tailv;
    if (rem > 1) dst[done + 1] = (uint8_t)(tailv >> 8);
    if (rem > 2) dst[done + 2] = (uint8_t)(tailv >> 16);
  }
}
// n (1..64) value bytes: the 17 aligned words that cover them at any phase are loaded together, then stored as above
__device__ __forceinline__ void copy_value_small(uint8_t* dst, const uint8_t* src, uint32_t n) {
  const uint32_t a = (uint32_t)((uintptr_t)src & 3);
  const uint32_t* ws = reinterpret_cast<const uint32_t*>((uintptr_t)src - a);
  const uint32_t nw = (a + n + 3) >> 2;  // <= 17
  uint32_t w[18];
#pragma unroll
  for (int i = 0; i < 17; i++) w[i] = (uint32_t)i < nw ? __ldg(ws + i) : 0u;
  w[17] = 0;
  store_value_words<17>(dst, w, a, n);
}
constexpr int kEmitPerLane = 3;
constexpr int kEmitMaxEntries = 32 * kEmitPerLane;  // 96 entries per block on the fast path
// ---- pieces the emit kernels and emit_block_warp share.  Lane-level: encoded size of entry x of a block from its meta and shared-prefix
// columns, *pk = shared | ulen << 8 | restart << 16, *vs = value length (rmask = R - 1 for a power-of-two restart interval, else ~0).
__device__ __forceinline__ uint32_t entry_pack(uint32_t mt, uint32_t esh, uint32_t x, uint32_t R, uint32_t rmask, uint32_t* pk, uint32_t* vs) {
  const bool restart = (rmask != 0xffffffffu ? (x & rmask) : (x % R)) == 0;
  const uint32_t ul = meta_ulen(mt), sh = restart ? 0 : esh;
  *vs = meta_vlen(mt);
  *pk = sh | (ul << 8) | (restart ? 1u << 16 : 0);
  return entry_size(sh, ul + 8, *vs);
}
// Lane-level: the header + key suffix of entry x (image offset off, pk from entry_pack) and its restart-array slot; returns the image
// offset of the entry's value bytes.
__device__ __forceinline__ uint32_t emit_entry_key(uint8_t* img, uint32_t off, uint32_t pk, uint32_t vs, uint64_t hi, uint64_t lo, uint64_t tr,
                                                   uint32_t x, uint32_t body, uint32_t R, uint32_t rmask) {
  const uint32_t sh = pk & 0xff, ul = (pk >> 8) & 0xff;
  uint8_t* p = img + off;
  const uint32_t ks = ul + 8;
  uint64_t S0, S1, S2;
  key_suffix_words(hi, lo, ul, tr, sh, &S0, &S1, &S2);
  if ((sh | (ks - sh) | vs) < 128) {
    // three one-byte lengths + key suffix as one 27-byte stream
    const uint64_t hdr = (uint64_t)sh | ((uint64_t)(ks - sh) << 8) | ((uint64_t)vs << 16);
    const uint64_t W0 = hdr | (S0 << 24), W1 = (S0 >> 40) | (S1 << 24), W2 = (S1 >> 40) | (S2 << 24), W3 = S2 >> 40;
    const uint32_t wv[8] = {(uint32_t)W0, (uint32_t)(W0 >> 32), (uint32_t)W1, (uint32_t)(W1 >> 32),
                            (uint32_t)W2, (uint32_t)(W2 >> 32), (uint32_t)W3, 0u};
    store_stream28(p, wv, 3 + ks - sh);
    p += 3 + ks - sh;
  } else {
    p += put_varint(p, sh);
    p += put_varint(p, ks - sh);
    p += put_varint(p, vs);
    store_bytes24(p, S0, S1, S2, ks - sh);
    p += ks - sh;
  }
  if (pk >> 16)  // restart array slot (block_builder.cc:207-210,128-133)
    put_fixed32(img + body + 4u * (rmask != 0xffffffffu ? x >> __popc(rmask) : x / R), off);
  return (uint32_t)(p - img);
}
// Warp-level: one value of vl (> 64) bytes from sp to dp, aligned 4-byte source words funnel-shifted into byte stores.  Up to 512
// bytes per pass: all of a pass's loads are issued before the first store, so a value of up to 512 bytes costs one memory round
// trip, not one per 128 bytes.
__device__ __forceinline__ void emit_copy_long_value(uint8_t* dp, const uint8_t* sp, uint32_t vl, unsigned lane) {
  const uint32_t a = (uint32_t)((uintptr_t)sp & 3);
  const uint32_t* wsrc = reinterpret_cast<const uint32_t*>((uintptr_t)sp - a);
  const uint32_t nwords = (vl + 3) >> 2;
  for (uint32_t k0 = 0; k0 < nwords; k0 += 128) {
    uint32_t lo[4], hi[4];
#pragma unroll
    for (int t = 0; t < 4; t++) {
      const uint32_t k = k0 + lane + 32 * t;
      lo[t] = k < nwords ? __ldg(wsrc + k) : 0u;
      hi[t] = k < nwords ? __ldg(wsrc + k + 1) : 0u;
    }
#pragma unroll
    for (int t = 0; t < 4; t++) {
      const uint32_t k = k0 + lane + 32 * t;
      if (k < nwords) {
        const uint32_t v = __funnelshift_r(lo[t], hi[t], a * 8);
        const uint32_t o = 4 * k;
        dp[o] = (uint8_t)v;
        if (o + 1 < vl) dp[o + 1] = (uint8_t)(v >> 8);
        if (o + 2 < vl) dp[o + 2] = (uint8_t)(v >> 16);
        if (o + 3 < vl) dp[o + 3] = (uint8_t)(v >> 24);
      }
    }
  }
}
// Warp-level: the values longer than 64 bytes among the lanes' (value length vs, image offset voff), one after another, each
// copied by the whole warp; vref_of(sl) gives lane sl's value reference to every lane.
template <class VrefOf>
__device__ __forceinline__ void emit_long_values(uint8_t* img, uint32_t vs, uint32_t voff, VrefOf vref_of, unsigned lane) {
  unsigned big = __ballot_sync(0xffffffffu, vs > 64);
  while (big) {
    const int sl = __ffs(big) - 1;
    big &= big - 1;
    const uint32_t vl = __shfl_sync(0xffffffffu, vs, sl), vo = __shfl_sync(0xffffffffu, voff, sl);
    emit_copy_long_value(img + vo, (const uint8_t*)(uintptr_t)vref_of(sl), vl, lane);
  }
}
// Warp-level: restart count footer, checksum trailer, then the image (built at gdst's 16-byte phase `shift`) leaves as head bytes,
// ONE bulk copy (TMA) of everything between the first and the last 16-byte boundary, and tail bytes
__device__ __forceinline__ void emit_block_finish(uint8_t* img, uint8_t* gdst, uint32_t shift, uint32_t body, uint32_t nrest, uint32_t cksum,
                                                  uint32_t xtab, unsigned lane) {
  const uint32_t payload = body + 4 * nrest + 4;
  if (lane == 0) put_fixed32(img + body + 4u * nrest, nrest);
  __syncwarp();
  const uint32_t ck = staged_block_checksum(cksum, (uint32_t)__cvta_generic_to_shared(img), img, payload, 0, xtab, lane);
  __syncwarp();  // the checksum's 8-byte loads may touch the trailer bytes written next
  if (lane == 0) put_block_trailer(img + payload, ck);
  fence_async_smem();  // this lane's image bytes are visible to the TMA engine
  __syncwarp();
  const uint32_t total = payload + 5;
  uint32_t head = shift ? 16 - shift : 0;
  if (head > total) head = total;
  const uint32_t mid = (total - head) & ~15u;
  if (lane == 0 && mid) bulk_s2g(gdst + head, (uint32_t)__cvta_generic_to_shared(img + head), mid);
  if (lane < head) gdst[lane] = img[lane];
  const uint32_t done = head + mid;
  if (done + lane < total) gdst[done + lane] = img[done + lane];
}
// Warp-level, for the blocks the emit kernels do not build themselves (more than kEmitMaxEntries entries, or larger than the image
// slot): entries 32 at a time, columns read from global memory, entry offsets from a 64-bit scan across the rounds.  A block that fits
// the slot is built there at gdst's 16-byte phase and leaves through emit_block_finish; otherwise it is written straight into the file
// image.  Offsets inside one block fit 32 bits: a block is less than the block size plus one value, and values are < 128 MiB.  The
// caller has waited for the slot's previous bulk store to finish reading it.  Not inlined: a copy of this rarely taken path in the
// emit kernels costs their block path registers (inlined, it cost the long-entry kernel ~10 % on 256-byte values: H100 SXM, 700 W).
__device__ __noinline__ void emit_block_warp(KeyCols m, const uint8_t* eshared, BlockRec br, uint8_t* gdst, uint8_t* slot, uint32_t slot_bytes,
                                             uint32_t R, uint32_t cksum, uint32_t xtab) {
  const unsigned lane = threadIdx.x & 31;
  const uint32_t rmask = (R & (R - 1)) == 0 ? R - 1 : 0xffffffffu;
  const uint32_t ne = br.n_entries, nrest = (ne + R - 1) / R;
  // pass 1: payload size (entries + restart array + footer)
  uint64_t body = 0;
  for (uint32_t x = lane; x < ne; x += 32) {
    uint32_t pk, vs;
    body += entry_pack(m.meta[br.first_entry + x], eshared[br.first_entry + x], x, R, rmask, &pk, &vs);
  }
#pragma unroll
  for (int d = 16; d; d >>= 1) body += __shfl_xor_sync(0xffffffffu, body, d);
  const uint64_t payload = body + 4ull * nrest + 4;
  const uint32_t shift = (uint32_t)((uintptr_t)gdst & 15);
  const bool staged = payload + 5 + 16 <= slot_bytes;
  uint8_t* const img = staged ? slot + shift : gdst;
  // pass 2: encode entries, 32 at a time
  uint64_t off_base = 0;
  for (uint32_t x0 = 0; x0 < ne; x0 += 32) {
    const uint32_t x = x0 + lane;
    uint32_t sz = 0, pk = 0, vs = 0, voff = 0;
    ulonglong2 pp = make_ulonglong2(0, 0);
    uint64_t tr = 0, vref = 0;
    if (x < ne) {
      const uint64_t e = br.first_entry + x;
      sz = entry_pack(m.meta[e], eshared[e], x, R, rmask, &pk, &vs);
      pp = m.pfx[e];
      tr = m.tr[e];
      vref = m.vref[e];
    }
    const uint64_t inc = warp_incl_scan64(sz);
    const uint32_t off = (uint32_t)(off_base + inc - sz);
    off_base += __shfl_sync(0xffffffffu, inc, 31);
    if (x < ne) {
      voff = emit_entry_key(img, off, pk, vs, pp.x, pp.y, tr, x, (uint32_t)body, R, rmask);
      if (vs && vs <= 64) copy_value_small(img + voff, (const uint8_t*)(uintptr_t)vref, vs);
    }
    // values longer than 64 bytes: the warp copies each of them with all lanes
    emit_long_values(img, vs, voff, [&](int sl) { return __shfl_sync(0xffffffffu, vref, sl); }, lane);
  }
  if (staged) {
    emit_block_finish(img, gdst, shift, (uint32_t)body, nrest, cksum, xtab, lane);
    return;
  }
  if (lane == 0) put_fixed32(img + body + 4ull * nrest, nrest);
  __threadfence();
  __syncwarp();
  const uint32_t ck = block_checksum_warp(cksum, img, payload, 0);
  __syncwarp();  // the checksum's 8-byte loads may touch the trailer bytes written next
  if (lane == 0) put_block_trailer(img + payload, ck);
}
// ---- the fast path's steps, shared by both emit kernels (one warp per block of at most kEmitMaxEntries entries, lane l owning
// entries [3l, 3l + 3)).  The kernels differ only in where the columns come from -- the staged kernel reads a shared-memory stage,
// the long-entry kernel loads from global memory -- so the steps take the lane's columns as accessors of the entry index i.
constexpr int kEmitShortWords = 9;  // aligned words covering a value of <= 32 bytes at any 4-byte phase
// The fit rule: the block's payload (body, restart array, restart count), its trailer, 32 bytes and the image's 16-byte phase fit
// the warp's image slot.  A block that does not fit goes to emit_block_warp.
__device__ __forceinline__ bool emit_block_fits(uint64_t body, uint32_t nrest, uint32_t slot_bytes) {
  return body + 4ull * nrest + 4 + 5 + 32 + 16 <= slot_bytes;
}
// Lane-level size pass: sz / pk / vs of the lane's entries (0 beyond the block's E entries); returns the lane's total
template <class MetaOf, class EshOf>
__device__ __forceinline__ uint32_t emit_lane_sizes(uint32_t E, uint32_t R, uint32_t rmask, unsigned lane, MetaOf meta_of, EshOf esh_of,
                                                    uint32_t (&sz)[kEmitPerLane], uint32_t (&pk)[kEmitPerLane], uint32_t (&vs)[kEmitPerLane]) {
  uint32_t tsum = 0;
#pragma unroll
  for (int i = 0; i < kEmitPerLane; i++) {
    const uint32_t x = lane * kEmitPerLane + i;
    sz[i] = pk[i] = vs[i] = 0;
    if (x < E) {
      sz[i] = entry_pack(meta_of(i), esh_of(i), x, R, rmask, &pk[i], &vs[i]);
      tsum += sz[i];
    }
  }
  return tsum;
}
// Lane-level: the image offsets of the lane's entries from the start of its run (the exclusive warp scan of the lane totals)
__device__ __forceinline__ void emit_lane_offsets(uint32_t run, const uint32_t (&sz)[kEmitPerLane], uint32_t (&off)[kEmitPerLane]) {
#pragma unroll
  for (int i = 0; i < kEmitPerLane; i++) {
    off[i] = run;
    run += sz[i];
  }
}
// Lane-level: header + key suffix of the lane's entries; voff = image offset of each entry's value bytes
template <class PfxOf, class TrOf>
__device__ __forceinline__ void emit_lane_keys(uint8_t* img, uint32_t E, uint32_t body, uint32_t R, uint32_t rmask, unsigned lane,
                                               const uint32_t (&off)[kEmitPerLane], const uint32_t (&pk)[kEmitPerLane],
                                               const uint32_t (&vs)[kEmitPerLane], PfxOf pfx_of, TrOf tr_of, uint32_t (&voff)[kEmitPerLane]) {
#pragma unroll
  for (int i = 0; i < kEmitPerLane; i++) {
    const uint32_t x = lane * kEmitPerLane + i;
    voff[i] = 0;
    if (x < E) {
      const ulonglong2 pp = pfx_of(i);
      voff[i] = emit_entry_key(img, off[i], pk[i], vs[i], pp.x, pp.y, tr_of(i), x, body, R, rmask);
    }
  }
}
__device__ __forceinline__ bool emit_all_short(const uint32_t (&vs)[kEmitPerLane]) {
  bool all_short = true;
#pragma unroll
  for (int i = 0; i < kEmitPerLane; i++) all_short = all_short && vs[i] <= 32;
  return all_short;
}
// Lane-level: the values of a group whose values are all <= 32 bytes, from words the kernel has loaded: words(i, w) puts entry i's
// aligned words in w[0..kEmitShortWords) (w[kEmitShortWords] = 0) and returns the value's 4-byte phase
template <class Words>
__device__ __forceinline__ void emit_lane_short_values(uint8_t* img, const uint32_t (&voff)[kEmitPerLane], const uint32_t (&vs)[kEmitPerLane],
                                                       Words words) {
#pragma unroll
  for (int i = 0; i < kEmitPerLane; i++) {
    if (!vs[i]) continue;
    uint32_t w[12];
    const uint32_t a = words(i, w);
    store_value_words<kEmitShortWords>(img + voff[i], w, a, vs[i]);
  }
}
// Lane-level: the values of 1..64 bytes of a group that is not all short, each copied by its lane
template <class VrefOf>
__device__ __forceinline__ void emit_lane_copy_values(uint8_t* img, const uint32_t (&voff)[kEmitPerLane], const uint32_t (&vs)[kEmitPerLane],
                                                      VrefOf vref_of) {
#pragma unroll
  for (int i = 0; i < kEmitPerLane; i++)
    if (vs[i] && vs[i] <= 64) copy_value_small(img + voff[i], (const uint8_t*)(uintptr_t)vref_of(i), vs[i]);
}
// Warp-level: the values longer than 64 bytes of the lanes' groups, one after another, each copied by the whole warp
template <class VrefOf>
__device__ __forceinline__ void emit_group_long_values(uint8_t* img, const uint32_t (&voff)[kEmitPerLane], const uint32_t (&vs)[kEmitPerLane],
                                                       VrefOf vref_of, unsigned lane) {
#pragma unroll
  for (int i = 0; i < kEmitPerLane; i++) emit_long_values(img, vs[i], voff[i], [&](int sl) { return vref_of(sl, i); }, lane);
}
constexpr int kEmitCtasPerSm = 3;                   // 12 warps per SM (with kEmitWarps = 4): room for 168 registers, no spills
// A column stage holds one block's entries of every column, copied by TMA as the 16-byte-aligned cover of the entry range (the cover
// starts up to 15 bytes before the range and ends up to 15 bytes behind it, so a region holds kEmitMaxEntries elements + 16 bytes).
// Every 16-byte unit the cover reads holds at least one byte of the column, so it lies in a page the column occupies; the bytes
// around the range are never used.  On the compaction path the columns are DevBuf allocations with >= 256 bytes of slack, so the
// cover stays inside them; columns a caller hands to b200c_job_encode_columns may end within 15 bytes of the cover's end, and
// those reads then pass the end of the caller's allocation (but not of its page).  The 16-byte value loads below rely on the same
// property: a chunk is read only when it holds a byte of the value.
constexpr uint32_t kStPfx = 0, kStTr = kStPfx + 16 * kEmitMaxEntries + 16, kStVref = kStTr + 8 * kEmitMaxEntries + 16,
                   kStMeta = kStVref + 8 * kEmitMaxEntries + 16, kStEsh = kStMeta + 4 * kEmitMaxEntries + 16,
                   kStageBytes = kStEsh + kEmitMaxEntries + 16;
static_assert(kStTr % 16 == 0 && kStVref % 16 == 0 && kStMeta % 16 == 0 && kStEsh % 16 == 0 && kStageBytes % 16 == 0,
              "bulk copies need 16-byte aligned shared-memory destinations");
__device__ __forceinline__ uint32_t cover16(const void* p, uint32_t bytes, uintptr_t* a0) {
  *a0 = (uintptr_t)p & ~(uintptr_t)15;
  return (uint32_t)((((uintptr_t)p + bytes + 15) & ~(uintptr_t)15) - *a0);
}
// lane 0: start the bulk copies of the columns of entries [e0, e0 + E) into the stage at shared address `stage`, completing on `bar`
__device__ __forceinline__ void emit_stage_fill(const KeyCols& m, const EncodeWork& wk, uint64_t e0, uint32_t E, uint32_t stage, uint32_t bar) {
  uintptr_t a[5];
  const uint32_t n0 = cover16(m.pfx + e0, 16 * E, &a[0]), n1 = cover16(m.tr + e0, 8 * E, &a[1]), n2 = cover16(m.vref + e0, 8 * E, &a[2]),
                 n3 = cover16(m.meta + e0, 4 * E, &a[3]), n4 = cover16(wk.eshared + e0, E, &a[4]);
  mbar_expect_tx(bar, n0 + n1 + n2 + n3 + n4);
  bulk_g2s(stage + kStPfx, reinterpret_cast<const void*>(a[0]), n0, bar);
  bulk_g2s(stage + kStTr, reinterpret_cast<const void*>(a[1]), n1, bar);
  bulk_g2s(stage + kStVref, reinterpret_cast<const void*>(a[2]), n2, bar);
  bulk_g2s(stage + kStMeta, reinterpret_cast<const void*>(a[3]), n3, bar);
  bulk_g2s(stage + kStEsh, reinterpret_cast<const void*>(a[4]), n4, bar);
}
// One WARP per data block, no CTA-wide synchronisation: lane l owns the block's entries [3l, 3l + 3), a warp scan of the
// entry sizes gives every entry its byte position, the lanes write header + key suffix + value into the warp's block
// image in shared memory, then the warp appends restart array + footer, checksums the image and stores it re-aligned
// to the file offset.  The block's columns arrive in shared memory ahead of time: while the warp builds one block, lane 0 has
// TMA copy the next block's columns into the other of the warp's two stages.  The only DRAM round trip a block still waits
// for is its value words, and the key bytes are written while those loads are in flight.  Blocks with more than 96 entries
// or larger than the image slot take emit_block_warp (no stage: it reads the columns from global memory).
__global__ void __launch_bounds__(kEmitWarps * 32, kEmitCtasPerSm)
encode_emit_kernel(KeyCols m, EncodeParams ep, EncodeWork wk, uint64_t nblocks, uint8_t* const* __restrict__ out_base,
                   uint32_t slot_bytes) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ XxhLaneTab s_xtab;
  __shared__ __align__(8) uint64_t s_bar[kEmitWarps][2];
  const unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint8_t* const slot = smem + (size_t)w * slot_bytes;  // 16-byte aligned (slot_bytes is a multiple of 256)
  uint8_t* const stages = smem + (size_t)kEmitWarps * slot_bytes + (size_t)w * 2 * kStageBytes;
  const uint32_t stages_sa = (uint32_t)__cvta_generic_to_shared(stages), bar0 = (uint32_t)__cvta_generic_to_shared(&s_bar[w][0]);
  fill_xxh_lane_tab(&s_xtab);
  if (lane == 0) {
    mbar_init(bar0, 1);
    mbar_init(bar0 + 8, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const uint32_t xtab = (uint32_t)__cvta_generic_to_shared(&s_xtab);
  const uint32_t R = ep.restart_interval;
  const uint32_t rmask = (R & (R - 1)) == 0 ? R - 1 : 0xffffffffu;  // power-of-two restart interval: mask instead of %
  const uint64_t stride = (uint64_t)gridDim.x * kEmitWarps;
  uint64_t b = (uint64_t)blockIdx.x * kEmitWarps + w;
  // br = this block, brn = the warp's next block: its stage fill is issued at the top of the iteration.  The records of the two
  // blocks after this one are (re)loaded into nbr / nbrn before the checksum, which hides their latency and keeps them out of
  // the registers the entry work needs.
  BlockRec br{}, brn{}, nbr{}, nbrn{};
  if (b < nblocks) br = wk.blocks[b];
  if (b + stride < nblocks) brn = wk.blocks[b + stride];
  if (lane == 0 && b < nblocks && br.n_entries <= (uint32_t)kEmitMaxEntries) emit_stage_fill(m, wk, br.first_entry, br.n_entries, stages_sa, bar0);
  uint32_t s = 0, parity = 0;  // stage of block b; bit t of parity = phase parity of stage t's next completion
  for (; b < nblocks; b += stride, s ^= 1, br = nbr, brn = nbrn) {
    __syncwarp();
    if (lane == 0 && b + stride < nblocks && brn.n_entries <= (uint32_t)kEmitMaxEntries) {
      // every lane finished reading stage s ^ 1 (the previous block; __syncwarp above): order those generic-proxy reads before
      // the async-proxy writes of the refill
      fence_async_smem();
      emit_stage_fill(m, wk, brn.first_entry, brn.n_entries, stages_sa + (s ^ 1) * kStageBytes, bar0 + 8 * (s ^ 1));
    }
    auto load_next = [&]() {
      if (b + stride < nblocks) nbr = wk.blocks[b + stride];
      if (b + 2 * stride < nblocks) nbrn = wk.blocks[b + 2 * stride];
    };
    const uint32_t E = br.n_entries;
    const uint64_t e0 = br.first_entry;
    // The image is built at the destination's 16-byte phase, so that everything between the first and the last 16-byte boundary
    // of the block leaves shared memory as ONE bulk copy (TMA) instead of a load / re-align / store loop.
    uint8_t* const gdst = out_base[br.file_idx] + br.file_off;
    const uint32_t shift = (uint32_t)((uintptr_t)gdst & 15);
    uint8_t* const img = slot + shift;
    // the block's columns in stage s, each at the 16-byte phase of its global address
    const uint8_t* const stg = stages + s * kStageBytes;
    const ulonglong2* const c_pfx = reinterpret_cast<const ulonglong2*>(stg + kStPfx + ((uintptr_t)(m.pfx + e0) & 15));
    const uint64_t* const c_tr = reinterpret_cast<const uint64_t*>(stg + kStTr + ((uintptr_t)(m.tr + e0) & 15));
    const uint64_t* const c_vref = reinterpret_cast<const uint64_t*>(stg + kStVref + ((uintptr_t)(m.vref + e0) & 15));
    const uint32_t* const c_meta = reinterpret_cast<const uint32_t*>(stg + kStMeta + ((uintptr_t)(m.meta + e0) & 15));
    const uint8_t* const c_esh = stg + kStEsh + ((uintptr_t)(wk.eshared + e0) & 15);
    const uint32_t nrest = (E + R - 1) / R;
    // ---- sizes (only a block of at most kEmitMaxEntries entries had its stage filled)
    uint32_t sz[kEmitPerLane], pk[kEmitPerLane], vs[kEmitPerLane];  // pk = shared | ulen << 8 | restart << 16
    uint32_t tsum = 0;
    uint64_t inc = 0;
    bool fallback = E > (uint32_t)kEmitMaxEntries;  // (uniform)
    if (!fallback) {
      mbar_wait(bar0 + 8 * s, (parity >> s) & 1);
      parity ^= 1u << s;
      const uint32_t x0 = lane * kEmitPerLane;
      tsum = emit_lane_sizes(E, R, rmask, lane, [&](int i) { return c_meta[x0 + i]; }, [&](int i) { return c_esh[x0 + i]; }, sz, pk, vs);
      inc = warp_incl_scan64(tsum);
      fallback = !emit_block_fits(__shfl_sync(0xffffffffu, inc, 31), nrest, slot_bytes);
    }
    if (fallback) {
      load_next();
      if (lane == 0) bulk_wait_read0();  // the previous block's bulk store has finished reading the slot
      __syncwarp();
      emit_block_warp(m, wk.eshared, br, gdst, slot, slot_bytes, R, ep.checksum, xtab);
      continue;
    }
    const uint32_t body = (uint32_t)__shfl_sync(0xffffffffu, inc, 31);
    uint32_t off[kEmitPerLane];
    emit_lane_offsets((uint32_t)(inc - tsum), sz, off);
    // ---- value bytes of all the lane's entries (when every value is short) leave first; the key bytes are written meanwhile.
    // A value of <= 32 bytes lies in at most three aligned 16-byte chunks: three vector loads instead of nine word loads (the
    // lanes' values are scattered, so every load instruction touches one cache line per lane).  Value references are read from
    // the stage where they are used, so that no register holds them across the key work.
    const bool all_short = emit_all_short(vs);
    uint4 vc[kEmitPerLane][3];
    if (all_short) {
#pragma unroll
      for (int i = 0; i < kEmitPerLane; i++) {
        const uint64_t vr = vs[i] ? c_vref[lane * kEmitPerLane + i] : 0;  // (vs[i] == 0 beyond the block's entries)
        const uint32_t a = (uint32_t)(vr & 15);
        const uint4* csrc = reinterpret_cast<const uint4*>((uintptr_t)vr - a);
        const uint32_t nc = vs[i] ? (a + vs[i] + 15) >> 4 : 0;
#pragma unroll
        for (int k = 0; k < 3; k++) vc[i][k] = (uint32_t)k < nc ? __ldg(csrc + k) : make_uint4(0, 0, 0, 0);
      }
    }
    if (lane == 0) bulk_wait_read0();  // the previous block's bulk store has finished reading the slot
    __syncwarp();
    const uint32_t x0 = lane * kEmitPerLane;
    uint32_t voff[kEmitPerLane];  // image offset of the value bytes
    emit_lane_keys(img, E, body, R, rmask, lane, off, pk, vs, [&](int i) { return c_pfx[x0 + i]; }, [&](int i) { return c_tr[x0 + i]; }, voff);
    if (all_short) {
      emit_lane_short_values(img, voff, vs, [&](int i, uint32_t(&w)[12]) {
        const uint32_t a = (uint32_t)(c_vref[x0 + i] & 15);
        const uint32_t t[12] = {vc[i][0].x, vc[i][0].y, vc[i][0].z, vc[i][0].w, vc[i][1].x, vc[i][1].y,
                                vc[i][1].z, vc[i][1].w, vc[i][2].x, vc[i][2].y, vc[i][2].z, vc[i][2].w};
#pragma unroll
        for (int k = 0; k < 12; k++) w[k] = t[k];
        // drop the a / 4 words in front of the value: w[0..9) then covers it at the 4-byte phase a & 3 (a & 3 + 32 bytes end
        // inside w[8]), and w[9] = 0 as store_value_words expects
        if (a & 8) {
#pragma unroll
          for (int k = 0; k < 10; k++) w[k] = w[k + 2];
        }
        if (a & 4) {
#pragma unroll
          for (int k = 0; k < 11; k++) w[k] = w[k + 1];
        }
        w[kEmitShortWords] = 0;
        return a & 3;
      });
    } else {
      emit_lane_copy_values(img, voff, vs, [&](int i) { return c_vref[x0 + i]; });
    }
    emit_group_long_values(img, voff, vs, [&](int sl, int i) { return c_vref[sl * kEmitPerLane + i]; }, lane);
    load_next();
    emit_block_finish(img, gdst, shift, body, nrest, ep.checksum, xtab, lane);
  }
  if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // no bulk store may outlive the CTA's shared memory
}

constexpr int kEmitLongWarps = 8, kEmitLongCtasPerSm = 4;  // 32 warps per SM, 64 registers each
// Jobs whose entries are all long (the value path below copies them warp-wide): more warps per SM with fewer registers each,
// and no column stages.  One WARP per data block, no CTA-wide synchronisation: lane l owns the block's entries [3l, 3l + 3), a warp scan of the
// entry sizes gives every entry its byte position, the lanes write header + key suffix + value into the warp's block
// image in shared memory, then the warp appends restart array + footer, checksums the image and stores it re-aligned
// to the file offset.  Global loads are issued in groups (size columns; key columns; value words) so that a block costs
// three DRAM round trips.  Blocks with more than 96 entries or larger than the image slot take emit_block_warp.
__global__ void __launch_bounds__(kEmitLongWarps * 32, kEmitLongCtasPerSm)
encode_emit_long_kernel(KeyCols m, EncodeParams ep, EncodeWork wk, uint64_t nblocks, uint8_t* const* __restrict__ out_base,
                        uint32_t slot_bytes) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ XxhLaneTab s_xtab;
  const unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint8_t* const slot = smem + (size_t)w * slot_bytes;  // 16-byte aligned (slot_bytes is a multiple of 256)
  fill_xxh_lane_tab(&s_xtab);
  __syncthreads();
  const uint32_t xtab = (uint32_t)__cvta_generic_to_shared(&s_xtab);
  const uint32_t R = ep.restart_interval;
  const uint32_t rmask = (R & (R - 1)) == 0 ? R - 1 : 0xffffffffu;  // power-of-two restart interval: mask instead of %
  const uint64_t stride = (uint64_t)gridDim.x * kEmitLongWarps;
  for (uint64_t b = (uint64_t)blockIdx.x * kEmitLongWarps + w; b < nblocks; b += stride) {
    const BlockRec br = wk.blocks[b];
    const uint32_t E = br.n_entries;
    const uint64_t e0 = br.first_entry;
    // The image is built at the destination's 16-byte phase, so that everything between the first and the last 16-byte boundary
    // of the block leaves shared memory as ONE bulk copy (TMA) instead of a load / re-align / store loop.
    uint8_t* const gdst = out_base[br.file_idx] + br.file_off;
    const uint32_t shift = (uint32_t)((uintptr_t)gdst & 15);
    uint8_t* const img = slot + shift;
    const uint32_t nrest = (E + R - 1) / R;
    // ---- pass 1: sizes.  All column loads of the lane's entries are issued before the first use.
    uint32_t sz[kEmitPerLane], pk[kEmitPerLane], vs[kEmitPerLane];  // pk = shared | ulen << 8 | restart << 16
    uint64_t vrf[kEmitPerLane];
    uint32_t tsum = 0;
    uint64_t inc = 0;
    bool fallback = E > (uint32_t)kEmitMaxEntries;  // (uniform)
    if (!fallback) {
      uint32_t mtv[kEmitPerLane], shv[kEmitPerLane];
#pragma unroll
      for (int i = 0; i < kEmitPerLane; i++) {
        const uint32_t x = lane * kEmitPerLane + i;
        mtv[i] = 0;
        shv[i] = 0;
        vrf[i] = 0;
        if (x < E) {
          mtv[i] = m.meta[e0 + x];
          shv[i] = wk.eshared[e0 + x];
          vrf[i] = m.vref[e0 + x];
        }
      }
      tsum = emit_lane_sizes(E, R, rmask, lane, [&](int i) { return mtv[i]; }, [&](int i) { return shv[i]; }, sz, pk, vs);
      inc = warp_incl_scan64(tsum);
      fallback = !emit_block_fits(__shfl_sync(0xffffffffu, inc, 31), nrest, slot_bytes);
    }
    if (lane == 0) bulk_wait_read0();  // the previous block's bulk store has finished reading the slot (the loads above overlapped it)
    __syncwarp();
    if (fallback) {
      emit_block_warp(m, wk.eshared, br, gdst, slot, slot_bytes, R, ep.checksum, xtab);
      continue;
    }
    const uint32_t body = (uint32_t)__shfl_sync(0xffffffffu, inc, 31);
    uint32_t off[kEmitPerLane];
    emit_lane_offsets((uint32_t)(inc - tsum), sz, off);
    // ---- pass 2: key columns of all the lane's entries, then all value words (when every value is short)
    uint32_t voff[kEmitPerLane];  // image offset of the value bytes
    {
      ulonglong2 ppv[kEmitPerLane];
      uint64_t trv[kEmitPerLane];
#pragma unroll
      for (int i = 0; i < kEmitPerLane; i++) {
        const uint32_t x = lane * kEmitPerLane + i;
        ppv[i] = make_ulonglong2(0, 0);
        trv[i] = 0;
        if (x < E) {
          ppv[i] = m.pfx[e0 + x];
          trv[i] = m.tr[e0 + x];
        }
      }
      emit_lane_keys(img, E, body, R, rmask, lane, off, pk, vs, [&](int i) { return ppv[i]; }, [&](int i) { return trv[i]; }, voff);
    }
    if (emit_all_short(vs)) {
      uint32_t vw[kEmitPerLane][kEmitShortWords + 1];
#pragma unroll
      for (int i = 0; i < kEmitPerLane; i++) {
        const uint32_t a = (uint32_t)(vrf[i] & 3);
        const uint32_t* wsrc = reinterpret_cast<const uint32_t*>((uintptr_t)vrf[i] - a);
        const uint32_t nw = vs[i] ? (a + vs[i] + 3) >> 2 : 0;
#pragma unroll
        for (int k = 0; k < kEmitShortWords; k++) vw[i][k] = (uint32_t)k < nw ? __ldg(wsrc + k) : 0u;
        vw[i][kEmitShortWords] = 0;
      }
      emit_lane_short_values(img, voff, vs, [&](int i, uint32_t(&w)[12]) {
#pragma unroll
        for (int k = 0; k <= kEmitShortWords; k++) w[k] = vw[i][k];
        return (uint32_t)(vrf[i] & 3);
      });
    } else {
      emit_lane_copy_values(img, voff, vs, [&](int i) { return vrf[i]; });
    }
    emit_group_long_values(img, voff, vs, [&](int sl, int i) { return __shfl_sync(0xffffffffu, vrf[i], sl); }, lane);
    emit_block_finish(img, gdst, shift, body, nrest, ep.checksum, xtab, lane);
  }
  if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // no bulk store may outlive the CTA's shared memory
}

// ------------------------------------------------------------------------------------------------ index block
// the first n bytes (n <= 16) of a key in (hi, lo) word form, as a mask of each word
__device__ __forceinline__ ulonglong2 key_prefix_mask(uint32_t n) {
  return make_ulonglong2(n >= 8 ? ~0ull : n ? ~0ull << (64 - 8 * n) : 0ull, n >= 16 ? ~0ull : n > 8 ? ~0ull << (128 - 8 * n) : 0ull);
}
// index of the first non-zero byte of (hi, lo); 16 when both are zero
__device__ __forceinline__ uint32_t first_nonzero_byte(uint64_t hi, uint64_t lo) {
  return hi ? (uint32_t)__clzll((long long)hi) >> 3 : lo ? 8 + ((uint32_t)__clzll((long long)lo) >> 3) : 16;
}
// byte i (< 16) of a key in (hi, lo) word form
struct KeyWords {
  uint64_t hi, lo;
  __device__ __forceinline__ uint32_t operator[](uint32_t i) const { return (uint32_t)((i < 8 ? hi >> (56 - 8 * i) : lo >> (120 - 8 * i)) & 0xff); }
};
// BytewiseComparator::FindShortestSeparator (util/comparator.cc:42-91) on user keys s < l in (hi, lo) word form (zero padded), of
// lengths tn and nul: false when s stays the separator; else s becomes s[0, p] with byte p incremented (length tn = p + 1), where
// p is the first byte in which s differs from l, or (when l ends right there with the next byte value) the first byte of s behind
// it below 0xff
__device__ __forceinline__ bool shortest_separator(uint64_t& hi, uint64_t& lo, uint32_t& tn, uint64_t nhi, uint64_t nlo, uint32_t nul) {
  const KeyWords s{hi, lo}, l{nhi, nlo};
  const uint32_t d = first_nonzero_byte(hi ^ nhi, lo ^ nlo);
  if (d >= (tn < nul ? tn : nul)) return false;  // one key is a prefix of the other
  uint32_t p;
  if (d < nul - 1 || (uint32_t)s[d] + 1 < (uint32_t)l[d]) {
    p = d;
  } else {
    const ulonglong2 a = key_prefix_mask(tn), b = key_prefix_mask(d + 1);  // the bytes (d, tn) of s: a & ~b
    p = first_nonzero_byte(~hi & a.x & ~b.x, ~lo & a.y & ~b.y);
    if (p == 16) return false;  // all 0xff
  }
  const ulonglong2 k = key_prefix_mask(p + 1);
  hi = (hi & k.x) + (p < 8 ? 1ull << (56 - 8 * p) : 0ull);  // byte p is below 0xff: no carry
  lo = (lo & k.y) + (p < 8 ? 0ull : 1ull << (120 - 8 * p));
  tn = p + 1;
  return true;
}
// The index entry of data block b (index_builder.h:160-200, one restart per entry): its key is the separator between the block's
// last key and the next block's first key in the same file (the last key itself behind a file's last block); its value is the
// block handle.  Equal user keys on both sides (same_ukey) make the file's index keep the 8-byte trailers.
struct IndexEntry {
  KeyRec key;           // ulen excludes the trailer; a shortened key (pad = 1) ends in (kMaxSequenceNumber, kValueTypeForSeek)
  uint64_t off, size;   // the block handle
  uint32_t file, hlen;  // hlen: bytes of the handle's two varints
  bool same_ukey;
};
// the handle part of block br = blocks[b]: its payload runs up to the next block of the file, or to the end of the file's data blocks
__device__ __forceinline__ IndexEntry index_handle(const EncodeWork& wk, const BlockRec& br, uint64_t b, uint64_t nblocks, bool* has_next) {
  IndexEntry ie{KeyRec{}, br.file_off, 0, br.file_idx, 0, false};
  *has_next = b + 1 < nblocks && wk.blocks[b + 1].file_idx == br.file_idx;
  ie.size = (*has_next ? wk.blocks[b + 1].file_off : wk.files[br.file_idx].data_size) - br.file_off - kBlockTrailerLen;
  ie.hlen = (uint32_t)varint_len(ie.off) + (uint32_t)varint_len(ie.size);
  return ie;
}
__device__ __forceinline__ IndexEntry index_entry(const KeyCols& m, const EncodeWork& wk, uint64_t b, uint64_t nblocks) {
  const BlockRec br = wk.blocks[b];
  bool has_next;
  IndexEntry ie = index_handle(wk, br, b, nblocks, &has_next);
  const uint64_t le = br.first_entry + br.n_entries - 1;
  const ulonglong2 lp = m.pfx[le];
  ie.key = KeyRec{lp.x, lp.y, m.tr[le], meta_ulen(m.meta[le]), 0};
  if (has_next) {
    const ulonglong2 np = m.pfx[le + 1];
    const uint32_t nul = meta_ulen(m.meta[le + 1]);
    KeyRec& sep = ie.key;
    ie.same_ukey = np.x == lp.x && np.y == lp.y && nul == sep.ulen;
    uint64_t hi = lp.x, lo = lp.y;
    uint32_t tn = sep.ulen;
    if (!ie.same_ukey && shortest_separator(hi, lo, tn, np.x, np.y, nul)) sep = KeyRec{hi, lo, (kMaxSeq << 8) | 0x16, tn, 1};
  }
  return ie;
}
// An entry is  varint shared (0) | varint key length | [varint handle length, format_version < 4] | key | handle.  Each header varint
// is one byte, so the 8 trailer bytes an index with sequence numbers adds to every key change no header: sizes are stored without them.
static_assert(kMaxUserKey + 8 < 128 && 2 * 10 < 128, "index entry header varints are one byte each");
// separators, entry sizes (without the key trailers) and the index_has_seq flag of every file
__global__ void encode_index_size_kernel(KeyCols m, EncodeWork wk, uint64_t nblocks, uint32_t format_version) {
  for (uint64_t b = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; b < nblocks; b += (uint64_t)gridDim.x * blockDim.x) {
    const IndexEntry ie = index_entry(m, wk, b, nblocks);
    if (ie.same_ukey) atomicOr(&wk.files[ie.file].index_has_seq, 1u);
    wk.idx_sep[b] = ie.key;
    wk.idx_esz[b] = (format_version >= 4 ? 2 : 3) + ie.key.ulen + ie.hlen;
  }
}
// The separator is read back rather than recomputed: this kernel runs behind the emit kernel, on the job's critical path, and the
// key-column loads of index_entry are scattered and dependent on the block record (H100: 0.1 ms per cfg2 job, profiles/README.md).
__global__ void encode_index_write_kernel(EncodeWork wk, uint64_t nblocks, uint32_t format_version, uint8_t* const* __restrict__ out_base) {
  for (uint64_t b = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; b < nblocks; b += (uint64_t)gridDim.x * blockDim.x) {
    bool has_next;
    IndexEntry ie = index_handle(wk, wk.blocks[b], b, nblocks, &has_next);
    ie.key = wk.idx_sep[b];
    const FileRec& fr = wk.files[ie.file];
    const uint32_t klen = ie.key.ulen + (fr.index_has_seq ? 8 : 0);
    const uint64_t bi = b - fr.first_block;
    const uint64_t eoff = index_entries_bytes(wk, fr, bi), entries_bytes = index_entries_bytes(wk, fr, fr.n_blocks);
    uint8_t* ib = out_base[ie.file] + fr.index_start();
    uint8_t* p = ib + eoff;
    *p++ = 0;
    *p++ = (uint8_t)klen;
    if (format_version < 4) *p++ = (uint8_t)ie.hlen;
    for (uint32_t t = 0; t < klen; t++) *p++ = (uint8_t)ikey_byte(ie.key.hi, ie.key.lo, ie.key.ulen, ie.key.tr, t);
    p += put_varint(p, ie.off);
    put_varint(p, ie.size);
    // restart array: one restart per entry (index_block_restart_interval == 1)
    put_fixed32(ib + entries_bytes + 4 * bi, (uint32_t)eoff);
    if (bi == 0) put_fixed32(ib + entries_bytes + 4 * fr.n_blocks, (uint32_t)fr.n_blocks);
  }
}
// ---- checksum and trailer of a file's index block or filter block: both are one large block per file, behind its data blocks
enum FileBlock : uint32_t { kIndexBlock, kFilterBlock };
// where block `which` of a file starts in the file image, and its length without the trailer (0: the file has no such block)
__device__ __forceinline__ uint64_t file_block(const FileRec& fr, uint32_t which, uint64_t* start) {
  *start = which == kFilterBlock ? fr.filter_start() : fr.index_start();
  return which == kFilterBlock ? fr.filter_len() : fr.n_blocks ? fr.index_size : 0;
}
// XXH3 accumulator contributions of the full 1024-byte blocks of every file's block `which`, one warp per 1024-byte block: they do not
// depend on the running state, and the checksum of a 1.5 MB filter by a single warp would be a chain of 1500 dependent memory round trips.
// The trailer kernel then only folds them (scramble chain).
__global__ void file_block_contrib_kernel(const FileRec* __restrict__ files, uint32_t nfiles, uint32_t which, uint8_t* const* __restrict__ out_base,
                                          uint64_t* __restrict__ contrib, const uint64_t* __restrict__ contrib_off) {
  const uint32_t f = blockIdx.y;
  if (f >= nfiles) return;
  uint64_t start;
  const uint64_t len = file_block(files[f], which, &start);
  if (len <= 240) return;
  const uint8_t* p = out_base[f] + start;
  const uint64_t nb_blocks = (len - 1) / 1024;
  const unsigned lane = threadIdx.x & 31;
  const XxhLaneSecret ks = xxh_lane_secret();
  for (uint64_t k = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); k < nb_blocks; k += (uint64_t)gridDim.x * (blockDim.x >> 5)) {
    const uint64_t part = xxh3_block_contrib<false>(p + 1024 * k, 16, ks);
    if (lane < 8) contrib[(contrib_off[f] + k) * 8 + lane] = part;
  }
}
// one warp per file: checksum of the file's block `which`, trailer written behind it
__global__ void file_block_trailer_kernel(const FileRec* __restrict__ files, uint32_t nfiles, uint32_t which, uint32_t cksum,
                                          uint8_t* const* __restrict__ out_base, const uint64_t* __restrict__ contrib,
                                          const uint64_t* __restrict__ contrib_off) {
  const uint32_t f = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (f >= nfiles) return;
  uint64_t start;
  const uint64_t len = file_block(files[f], which, &start);
  if (len == 0) return;
  uint8_t* p = out_base[f] + start;
  uint32_t ck;
  if (cksum == 4) ck = (uint32_t)xxh3_64_warp_t<false>(p, len, contrib + contrib_off[f] * 8);  // last byte (type 0) adds nothing
  else ck = block_checksum_warp(cksum, p, len, 0);
  if ((threadIdx.x & 31) == 0) put_block_trailer(p + len, ck);
}

// checksum test entry point: one warp per buffer
__global__ void block_checksums_kernel(uint32_t type, const uint8_t* __restrict__ data, const uint64_t* __restrict__ offsets, uint32_t n,
                                       uint8_t last_byte, uint32_t* __restrict__ out) {
  const uint32_t i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= n) return;
  uint32_t ck = block_checksum_warp(type, data + offsets[i], offsets[i + 1] - offsets[i], last_byte);
  if ((threadIdx.x & 31) == 0) out[i] = ck;
}

// ------------------------------------------------------------------------------------------------ Bloom filter block
// One FastLocalBloom filter per output file over the XXPH3 hashes of its user keys (bloom_rules.h).  The hash is recomputed from the
// key columns wherever it is needed (a few integer ops) instead of being stored: 8 B per entry of extra traffic would cost more.
__device__ __forceinline__ uint64_t entry_key_hash(const KeyCols& m, uint64_t e) {
  const ulonglong2 p = m.pfx[e];
  return xxph3_of_key(p.x, p.y, meta_ulen(m.meta[e]));
}
__device__ __forceinline__ uint32_t file_of_entry(const FileRec* __restrict__ files, uint32_t nfiles, uint64_t e) {
  uint32_t lo = 0, hi = nfiles;  // last file with first_entry <= e
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (files[mid].first_entry <= e) lo = mid;
    else hi = mid;
  }
  return lo;
}
// Whether entry e adds its hash h to its file's filter (XXPH3FilterBitsBuilder::AddKey, filter_policy.cc:73-92): not when h equals
// the hash of the key ADDED TO THIS FILTER before; every entry of a file is offered to it, so that is the file's previous entry.
__device__ __forceinline__ bool bloom_adds(uint64_t e, uint64_t file_first, uint64_t h, uint64_t prev_h) {
  return e == file_first || prev_h != h;
}
__global__ void __launch_bounds__(256)
bloom_count_kernel(KeyCols m, uint64_t n, FileRec* __restrict__ files, const uint64_t* __restrict__ nfiles_dev, uint64_t* __restrict__ hashes) {
  const uint32_t nfiles = (uint32_t)*nfiles_dev;
  if (nfiles == 0 || nfiles > kMaxOutFiles) return;
  const unsigned lane = threadIdx.x & 31;
  constexpr int kU = 4;  // a warp takes 4 x 32 consecutive entries per step, all key loads issued before the first hash
  // every warp owns one contiguous range of entries, so it stays inside one file almost always and adds its count to the file's
  // record once (thousands of warps adding after every 32 entries serialise on the 32 counters: that was most of this kernel)
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  const uint64_t per_warp = ((n + nwarps - 1) / nwarps + 32 * kU - 1) / (32 * kU) * (32 * kU);
  const uint64_t w_begin = warp0 * per_warp, w_end = w_begin + per_warp < n ? w_begin + per_warp : n;
  unsigned long long acc = 0;
  uint32_t acc_f = 0xffffffffu;
  for (uint64_t e0 = w_begin; e0 < w_end; e0 += 32 * kU) {
    ulonglong2 kp[kU];
    uint32_t km[kU];
#pragma unroll
    for (int u = 0; u < kU; u++) {
      const uint64_t e = e0 + 32 * u + lane;
      if (e < n) {
        kp[u] = m.pfx[e];
        km[u] = m.meta[e];
      }
    }
    // the 128 entries of a step almost always belong to one file: one lookup for all of them then
    const uint64_t e_last = e0 + 32 * kU - 1 < n ? e0 + 32 * kU - 1 : n - 1;
    const uint32_t f_lo = file_of_entry(files, nfiles, e0), f_hi = file_of_entry(files, nfiles, e_last);
    uint64_t carry = 0;  // hash of the entry in front of this group of 32 (lane 31 of the previous group)
#pragma unroll
    for (int u = 0; u < kU; u++) {
      const uint64_t e = e0 + 32 * u + lane;
      uint32_t f = 0xffffffffu;
      bool add = false;
      const uint64_t h = e < n ? xxph3_of_key(kp[u].x, kp[u].y, meta_ulen(km[u])) : 0;
      if (e < n) hashes[e] = h;  // the filter build reads these instead of hashing the keys again
      uint64_t ph = __shfl_up_sync(0xffffffffu, h, 1);
      if (lane == 0) ph = carry;
      if (e < n) {
        f = f_lo == f_hi ? f_lo : file_of_entry(files, nfiles, e);
        const uint64_t ff = files[f].first_entry;
        if (u == 0 && lane == 0 && e > ff) ph = entry_key_hash(m, e - 1);
        add = bloom_adds(e, ff, h, ph);
      }
      carry = __shfl_sync(0xffffffffu, h, 31);
      // a warp's 32 consecutive entries almost always belong to one file: one atomic per warp then
      const uint32_t f0 = __shfl_sync(0xffffffffu, f, 0);
      const bool uniform = __all_sync(0xffffffffu, f == f0 || f == 0xffffffffu);
      if (uniform) {
        const unsigned cnt = __popc(__ballot_sync(0xffffffffu, add));
        if (f0 != 0xffffffffu) {
          if (f0 != acc_f) {
            if (lane == 0 && acc) atomicAdd(reinterpret_cast<unsigned long long*>(&files[acc_f].filter_entries), acc);
            acc = 0;
            acc_f = f0;
          }
          acc += cnt;
        }
      } else if (add) {
        atomicAdd(reinterpret_cast<unsigned long long*>(&files[f].filter_entries), 1ull);
      }
    }
  }
  if (lane == 0 && acc) atomicAdd(reinterpret_cast<unsigned long long*>(&files[acc_f].filter_entries), acc);
}
__global__ void bloom_layout_kernel(FileRec* __restrict__ files, const uint64_t* __restrict__ nfiles_dev, uint32_t millibits) {
  const uint32_t nfiles = (uint32_t)*nfiles_dev;
  for (uint32_t f = blockIdx.x * blockDim.x + threadIdx.x; f < nfiles && f < kMaxOutFiles; f += gridDim.x * blockDim.x) {
    const uint64_t cnt = files[f].filter_entries;
    files[f].filter_bytes = cnt ? (uint64_t)bloom_bits_bytes(cnt, millibits) + kBloomMetadataLen + kBlockTrailerLen : 0;
  }
}
void launch_bloom_count(KeyCols m, uint64_t n, FileRec* files, const uint64_t* nfiles_dev, uint32_t millibits, uint64_t* hashes, int sms, cudaStream_t st,
                        uint64_t* launches) {
  if (n == 0) return;
  const uint64_t blocks = (n + 1023) / 1024;
  bloom_count_kernel<<<(unsigned)(blocks < (unsigned)sms * 8 ? blocks : (unsigned)sms * 8), 256, 0, st>>>(m, n, files, nfiles_dev, hashes);
  bloom_layout_kernel<<<(kMaxOutFiles + 255) / 256, 256, 0, st>>>(files, nfiles_dev, millibits);
  *launches += 2;
}
// ---- filter bits.  FastLocalBloom puts all probes of a key into ONE 64-byte line of the filter (util/bloom_impl.h:200-214), and a
// file's whole filter is small (1.25 bytes per key at 10 bits).  So the filter is built in SLICES of shared memory: a CTA owns
// kBloomSliceBytes of one file's filter, scans the hashes of all of the file's keys (8 bytes per key, written by bloom_count_kernel and
// served by the L2 to the slice CTAs of a file), applies the keys whose line falls into its slice with shared-memory atomics and
// writes the finished slice with one bulk store.  (Slower alternatives: OR-ing the bits into L2 with global atomics; slice CTAs
// that re-hash the key columns; a cluster of eight CTAs setting bits in each other's shared memory.)
constexpr uint32_t kBloomSliceBytes = 176 * 1024;
constexpr int kBloomThreads = 1024;
constexpr uint32_t kBloomStage = 64;  // hashes a warp can queue
__global__ void __launch_bounds__(kBloomThreads, 1)
bloom_slices_kernel(const uint64_t* __restrict__ hashes, const FileRec* __restrict__ files, uint32_t nfiles, int probes,
                    uint8_t* const* __restrict__ out_base) {
  extern __shared__ __align__(128) uint8_t bsm[];
  const uint32_t f = blockIdx.y;
  if (f >= nfiles) return;
  const FileRec& fr = files[f];
  if (fr.filter_len() <= kBloomMetadataLen) return;
  const uint32_t bits_bytes = (uint32_t)(fr.filter_len() - kBloomMetadataLen);
  const uint32_t s0 = blockIdx.x * kBloomSliceBytes;
  if (s0 >= bits_bytes) return;
  const uint32_t s1 = s0 + kBloomSliceBytes < bits_bytes ? s0 + kBloomSliceBytes : bits_bytes;
  uint8_t* const gdst = out_base[f] + fr.filter_start() + s0;  // at any byte alignment
  const uint32_t shift = (uint32_t)((uintptr_t)gdst & 15);
  uint8_t* const img = bsm + shift;  // the slice at the destination's 16-byte phase (so that it leaves as one bulk copy)
  uint32_t* const w32 = reinterpret_cast<uint32_t*>(bsm);
  for (uint32_t i = threadIdx.x; i < (kBloomSliceBytes + 16) / 4; i += kBloomThreads) w32[i] = 0;
  __syncthreads();
  const uint64_t e0 = fr.first_entry, e1 = e0 + fr.n_entries;
  constexpr int kU = 8;  // hash loads in flight per thread: the scan is a chain of L2 round trips otherwise
  // Only one key in `slices` belongs to this slice.  Setting its bits right away would issue every shared-memory atomic with a few
  // active lanes; instead a warp queues the hashes that fall into the slice and sets the bits of 32 keys at a time.
  uint64_t* const stage = reinterpret_cast<uint64_t*>(bsm + kBloomSliceBytes + 16) + (threadIdx.x >> 5) * kBloomStage;
  const unsigned lane = threadIdx.x & 31;
  uint32_t queued = 0;  // (warp-uniform)
  auto set_bits = [&](uint64_t h) {
    const uint32_t line = bloom_line_offset(h, bits_bytes);
    uint32_t p = bloom_first_probe(h);
    for (int k = 0; k < probes; k++, p = bloom_next_probe(p)) {
      const uint32_t bit = bloom_probe_bit(p);
      const uint32_t byte = shift + (line - s0) + (bit >> 3);  // offset inside bsm
      atomicOr(&w32[byte >> 2], 1u << (8 * (byte & 3) + (bit & 7)));
    }
  };
  for (uint64_t eb = e0; eb < e1; eb += (uint64_t)kU * kBloomThreads) {
    uint64_t hv[kU], pv[kU];
#pragma unroll
    for (int u = 0; u < kU; u++) {
      const uint64_t e = eb + (uint64_t)u * kBloomThreads + threadIdx.x;
      hv[u] = pv[u] = 0;
      if (e < e1) {
        hv[u] = hashes[e];
        if (e > e0) pv[u] = hashes[e - 1];  // (the neighbouring lane's line: an L1 hit)
      }
    }
#pragma unroll
    for (int u = 0; u < kU; u++) {
      const uint64_t e = eb + (uint64_t)u * kBloomThreads + threadIdx.x;
      const uint64_t h = hv[u];
      bool mine = e < e1 && bloom_adds(e, e0, h, pv[u]);
      if (mine) {
        const uint32_t line = bloom_line_offset(h, bits_bytes);
        mine = line >= s0 && line < s1;
      }
      const unsigned mask = __ballot_sync(0xffffffffu, mine);
      if (mine) stage[queued + __popc(mask & ((1u << lane) - 1u))] = h;
      queued += __popc(mask);
      __syncwarp();
      if (queued >= 32) {
        const uint64_t hq = stage[lane];
        const uint64_t rest = lane + 32 < queued ? stage[lane + 32] : 0;
        __syncwarp();
        queued -= 32;
        if (lane < queued) stage[lane] = rest;
        set_bits(hq);
        __syncwarp();
      }
    }
  }
  if (lane < queued) set_bits(stage[lane]);
  __syncthreads();
  // store: head bytes up to the first 16-byte boundary, the aligned middle as one bulk copy (TMA), tail bytes
  const uint32_t total = s1 - s0;
  uint32_t head = shift ? 16 - shift : 0;
  if (head > total) head = total;
  const uint32_t mid = (total - head) & ~15u;
  fence_async_smem();
  __syncthreads();
  if (threadIdx.x == 0 && mid) {
    bulk_s2g(gdst + head, (uint32_t)__cvta_generic_to_shared(img + head), mid);
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
  if (threadIdx.x < head) gdst[threadIdx.x] = img[threadIdx.x];
  const uint32_t done = head + mid;
  if (done + threadIdx.x < total) gdst[done + threadIdx.x] = img[done + threadIdx.x];
  if (s1 == bits_bytes && threadIdx.x == 32) {  // the CTA of the last slice also writes the metadata bytes behind the bits
    uint8_t* md = out_base[f] + fr.filter_start() + bits_bytes;
    md[0] = 0xff;  // marker: newer Bloom implementations (filter_policy.cc:378-385)
    md[1] = 0;     // sub-implementation: FastLocalBloom
    md[2] = (uint8_t)probes;
    md[3] = 0;
    md[4] = 0;
  }
}
// checksum and trailer of block `which` of every file: the XXH3 contributions over contrib_ctas CTAs per file, then a warp per file
static void launch_file_block_checksums(const EncodeWork& w, uint32_t nfiles, FileBlock which, unsigned contrib_ctas, uint32_t cksum,
                                        uint8_t* const* out_base, cudaStream_t st, uint64_t* launches) {
  const uint64_t* contrib_off = w.cksum_contrib_off + (which == kFilterBlock ? nfiles : 0);
  if (cksum == 4) {
    file_block_contrib_kernel<<<dim3(contrib_ctas, nfiles), 256, 0, st>>>(w.files, nfiles, which, out_base, w.cksum_contrib, contrib_off);
    *launches += 1;
  }
  file_block_trailer_kernel<<<(nfiles + 3) / 4, 128, 0, st>>>(w.files, nfiles, which, cksum, out_base, w.cksum_contrib, contrib_off);
  *launches += 1;
}
void launch_bloom_build(const uint64_t* hashes, uint64_t n, const EncodeWork& w, uint32_t nfiles, uint32_t max_filter_bytes, uint32_t millibits,
                        uint32_t cksum, uint8_t* const* out_base, cudaStream_t st, uint64_t* launches) {
  if (n == 0 || nfiles == 0) return;
  const int probes = bloom_num_probes((int)millibits);
  static PerDeviceFlag attr;
  const uint64_t dev_bit = attr.bit_of_current_device();
  const int smem = (int)kBloomSliceBytes + 16 + (kBloomThreads / 32) * kBloomStage * 8;
  if (!attr.is_set(dev_bit)) {
    cudaFuncSetAttribute(bloom_slices_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr.set(dev_bit);
  }
  const unsigned slices = (max_filter_bytes + kBloomSliceBytes - 1) / kBloomSliceBytes;
  bloom_slices_kernel<<<dim3(slices ? slices : 1, nfiles), kBloomThreads, smem, st>>>(hashes, w.files, nfiles, probes, out_base);
  *launches += 1;
  launch_file_block_checksums(w, nfiles, kFilterBlock, 32, cksum, out_base, st, launches);
}

// ranks of the grandparent boundary keys in the merged stream (one thread per grandparent file)
__global__ void gp_rank_kernel(KeyCols m, const GpKey* __restrict__ smallest, const GpKey* __restrict__ largest, uint32_t n,
                               uint64_t* __restrict__ lo, uint64_t* __restrict__ eq, uint64_t* __restrict__ hi) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  auto bound = [&](const GpKey& k, bool upper) -> uint64_t { return ukey_bound(m, 0, m.n, k.hi, k.lo, k.ulen, upper); };
  lo[i] = bound(smallest[i], false);
  eq[i] = bound(largest[i], false);
  hi[i] = bound(largest[i], true);
}
void launch_gp_ranks(KeyCols m, const GpKey* smallest, const GpKey* largest, uint32_t n, uint64_t* lo, uint64_t* eq, uint64_t* hi,
                     cudaStream_t st, uint64_t* launches) {
  if (n == 0) return;
  gp_rank_kernel<<<(n + 63) / 64, 64, 0, st>>>(m, smallest, largest, n, lo, eq, hi);
  *launches += 1;
}

// ---- fixed-prefix SST partitioner (SstPartitionerFixedPrefix::ShouldPartition, db/compaction/sst_partitioner.cc): entry e >= 1
// of the merged stream is an event when its user key and entry e - 1's, each truncated to len bytes (a shorter key stays whole),
// differ.  The merged stream is exactly what the reference adds to its outputs (last_key_for_partitioner_, compaction_outputs.cc:
// 394-398), so dropped versions never count.  Keys are at most 16 bytes: the compare is one on the (hi, lo) words under a byte mask.
__device__ __forceinline__ bool partition_prefix_differs(ulonglong2 a, uint32_t alen, ulonglong2 b, uint32_t blen, uint32_t len) {
  const uint32_t la = alen < len ? alen : len, lb = blen < len ? blen : len;
  if (la != lb) return true;
  const ulonglong2 k = key_prefix_mask(la);
  return (((a.x ^ b.x) & k.x) | ((a.y ^ b.y) & k.y)) != 0;
}
constexpr int kPevThreads = 256, kPevItems = 8, kPevTile = kPevThreads * kPevItems;
// One CTA per kPevTile entries, taken in ticket order: flag every entry, count per warp and round, find the CTA's first event rank by
// the decoupled look-back over the CTAs in front, then write the events in entry order.  Ranks >= cap (more files than the encoder's
// records hold) are not stored; they mark the job kErrTooManyFiles, which the host reads before any file is written.
__global__ void __launch_bounds__(kPevThreads)
partition_events_kernel(KeyCols m, uint32_t len, uint32_t cap, uint32_t* __restrict__ ticket, unsigned long long* __restrict__ state,
                        uint64_t* __restrict__ ev, uint32_t* __restrict__ err) {
  constexpr int kWarps = kPevThreads / 32;
  __shared__ uint32_t s_tile, s_off[kPevItems][kWarps];
  __shared__ uint64_t s_base;
  if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
  __syncthreads();
  const uint64_t t0 = (uint64_t)s_tile * kPevTile;
  const unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t flags = 0;
#pragma unroll
  for (int i = 0; i < kPevItems; i++) {  // round i: the CTA's threads on kPevThreads consecutive entries
    const uint64_t e = t0 + (uint64_t)i * kPevThreads + threadIdx.x;
    bool f = false;
    if (e >= 1 && e < m.n) f = partition_prefix_differs(m.pfx[e - 1], meta_ulen(m.meta[e - 1]), m.pfx[e], meta_ulen(m.meta[e]), len);
    const unsigned b = __ballot_sync(0xffffffffu, f);
    if (lane == 0) s_off[i][w] = __popc(b);
    flags |= (uint32_t)f << i;
  }
  __syncthreads();
  if (w == 0) {
    uint32_t total = 0;
    if (lane == 0) {  // (round, warp) order is entry order: exclusive offsets of the 64 counts
      for (int i = 0; i < kPevItems; i++)
        for (int k = 0; k < kWarps; k++) {
          const uint32_t c = s_off[i][k];
          s_off[i][k] = total;
          total += c;
        }
      lb_publish(state, s_tile, total);
    }
    total = __shfl_sync(0xffffffffu, total, 0);
    const uint64_t base = lb_exclusive_prefix(state, s_tile, total, lane, 64);
    if (lane == 0) s_base = base;
  }
  __syncthreads();
  const uint64_t base = s_base;
#pragma unroll
  for (int i = 0; i < kPevItems; i++) {
    const bool f = (flags >> i) & 1u;
    const unsigned b = __ballot_sync(0xffffffffu, f);
    if (!f) continue;
    const uint64_t r = base + s_off[i][w] + __popc(b & ((1u << lane) - 1u));
    if (r < cap) ev[r] = t0 + (uint64_t)i * kPevThreads + threadIdx.x;
    else atomicOr(err, kErrTooManyFiles);
  }
}
uint64_t partition_event_tiles(uint64_t n) { return (n + kPevTile - 1) / kPevTile; }
void launch_partition_events(KeyCols m, uint32_t len, uint32_t cap, uint32_t* ticket, unsigned long long* state, uint64_t* ev, uint32_t* err,
                             cudaStream_t st, uint64_t* launches) {
  const uint64_t tiles = partition_event_tiles(m.n);
  if (tiles == 0) return;
  partition_events_kernel<<<(unsigned)tiles, kPevThreads, 0, st>>>(m, len, cap, ticket, state, ev, err);
  *launches += 1;
}

// file tails (properties | metaindex | footer, built on the host) from their staging buffer into the output images
__global__ void scatter_tails_kernel(const TailCopy* __restrict__ recs, const uint8_t* __restrict__ staged, uint8_t* __restrict__ out) {
  const TailCopy r = recs[blockIdx.x];
  for (uint32_t i = threadIdx.x; i < r.len; i += blockDim.x) out[r.dst_off + i] = staged[r.src_off + i];
}

// `small` slots (+ the first *nfiles_dev file records behind them) into mapped pinned host memory
__global__ void gather_small_kernel(const uint64_t* __restrict__ small, uint32_t small_words, const FileRec* __restrict__ files,
                                    const uint64_t* __restrict__ nfiles_dev, uint64_t* __restrict__ dst) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
  for (uint32_t i = t; i < small_words; i += nt) dst[i] = small[i];
  if (files) {
    uint64_t n = *nfiles_dev;
    if (n > kMaxOutFiles) n = kMaxOutFiles;
    const uint64_t words = n * (sizeof(FileRec) / 8);
    const uint64_t* src = reinterpret_cast<const uint64_t*>(files);
    for (uint64_t i = t; i < words; i += nt) dst[small_words + i] = src[i];
  }
}
static_assert(sizeof(FileRec) % 8 == 0, "FileRec is copied word-wise");

// ------------------------------------------------------------------------------------------------ launchers
void launch_gather_small(const uint64_t* small, uint32_t small_bytes, const FileRec* files, const uint64_t* nfiles_dev, uint8_t* dst,
                         cudaStream_t st) {
  gather_small_kernel<<<files ? 8 : 1, 256, 0, st>>>(small, small_bytes / 8, files, nfiles_dev, reinterpret_cast<uint64_t*>(dst));
}
__global__ void copy_small_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint32_t n) {
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}
void launch_copy_small(const void* src, void* dst, uint32_t n, cudaStream_t st) {
  if (n) copy_small_kernel<<<1, 256, 0, st>>>(static_cast<const uint8_t*>(src), static_cast<uint8_t*>(dst), n);
}
void launch_scatter_tails(const TailCopy* recs, uint32_t n, const uint8_t* staged, uint8_t* out, cudaStream_t st) {
  if (n) scatter_tails_kernel<<<n, 256, 0, st>>>(recs, staged, out);
}
void launch_encode_sizes(KeyCols m, const unsigned long long* n_dev, EncodeWork w, unsigned long long* tprefix_out, uint64_t n_cap,
                         int sms, cudaStream_t st) {
  if (n_cap == 0) return;
  const uint64_t tiles = (n_cap + kEncTile - 1) / kEncTile;
  encode_sizes_kernel<<<(unsigned)(tiles < (unsigned)sms * 8 ? tiles : (unsigned)sms * 8), 256, 0, st>>>(m, n_dev, w.esz, w.eshared, w.tstat, tprefix_out, w.min_s1);
}
void launch_encode_tables(KeyCols m, EncodeParams ep, EncodeWork w, uint64_t ntiles, uint32_t hc, uint32_t max_s1, cudaStream_t st,
                          uint64_t* launches) {
  if (ntiles == 0) return;
  static PerDeviceFlag attr;
  const uint64_t dev_bit = attr.bit_of_current_device();
  if (!attr.is_set(dev_bit)) {
    cudaFuncSetAttribute(encode_tables_kernel<uint32_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TablesSmem<uint32_t>));
    cudaFuncSetAttribute(encode_tables_kernel<uint64_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TablesSmem<uint64_t>));
    attr.set(dev_bit);
  }
  // all prefix sums of a window stay below 2^32 when (largest entry) x (window length) does
  if (((uint64_t)max_s1 + 64) * (uint64_t)(kW + 1) < (1ull << 32))
    encode_tables_kernel<uint32_t><<<(unsigned)ntiles, kEncThreads, sizeof(TablesSmem<uint32_t>), st>>>(m, ep, w, m.n, hc);
  else
    encode_tables_kernel<uint64_t><<<(unsigned)ntiles, kEncThreads, sizeof(TablesSmem<uint64_t>), st>>>(m, ep, w, m.n, hc);
  *launches += 1;
}
void launch_encode_stitch(KeyCols m, EncodeParams ep, EncodeWork w, uint64_t ntiles, uint32_t hc, uint32_t* err, uint32_t attempt,
                          uint32_t* sflag, cudaStream_t st, uint64_t* launches) {
  if (ntiles == 0) return;
  static PerDeviceFlag attr;
  const uint64_t dev_bit = attr.bit_of_current_device();
  constexpr size_t kSolo = 200 * 1024;  // attempt 1: no tables CTA (>= 60 KB of shared memory) fits next to it
  if (!attr.is_set(dev_bit)) {
    cudaFuncSetAttribute(encode_stitch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSolo);
    attr.set(dev_bit);
  }
  const size_t fixed = (sizeof(StitchSmem) + 15) & ~(size_t)15;
  // row caches: at least one group / one tile.  Attempt 2 may have to run next to two tables CTAs: 16 KB each when that is enough;
  // attempt 1 owns its SM: half of what is left each (a whole group of tile rows per refill)
  uint32_t cache_bytes = 16 * 1024;
  while (cache_bytes < hc * (uint32_t)sizeof(TileRow)) cache_bytes *= 2;
  size_t smem = fixed + 2 * (size_t)cache_bytes;
  if (attempt == 1) {
    const uint32_t big = (uint32_t)(((kSolo - fixed) / 2) & ~(size_t)15);
    if (big > cache_bytes) cache_bytes = big;
    smem = kSolo;
  }
  encode_stitch_kernel<<<1, kEncThreads, smem, st>>>(m, ep, w, m.n, ntiles, hc, cache_bytes, err, attempt, sflag, 300000u);
  *launches += 1;
}
void launch_encode_tilestate(KeyCols m, EncodeWork w, uint64_t ntiles, uint32_t hc, uint32_t* err, cudaStream_t st, uint64_t* launches) {
  if (ntiles == 0) return;
  const uint64_t ngroups = (ntiles + kEncGroup - 1) / kEncGroup;
  encode_tilestate_kernel<<<(unsigned)((ngroups + 63) / 64), 64, 0, st>>>(w, m.n, ntiles, hc, err);
  *launches += 1;
}
void launch_encode_blocklist(KeyCols m, EncodeParams ep, EncodeWork w, uint64_t ntiles, uint64_t nblk_cap, uint32_t* err,
                             cudaStream_t st, uint64_t* launches) {
  if (ntiles == 0) return;
  encode_blocklist_kernel<<<(unsigned)ntiles, kEncThreads, 0, st>>>(m, ep, w, m.n, nblk_cap, err);
  *launches += 1;
}
void launch_encode_filestats(KeyCols m, EncodeWork w, uint32_t nfiles, cudaStream_t st, uint64_t* launches) {
  if (m.n == 0 || nfiles == 0) return;
  encode_filestats_kernel<<<nfiles, 256, 0, st>>>(m, w, nfiles);
  *launches += 1;
}
constexpr uint32_t kEmitMaxSmem = 224 * 1024;  // dynamic shared memory of one emit CTA at most (+ ~2 KB static: XXH3 lane table, mbarriers)
uint32_t encode_emit_slice(uint32_t block_size) {
  uint32_t s = block_size + block_size / 4 + 512;
  s = (s + 255) & ~255u;
  if (s < 5632) s = 5632;
  if (s > 24 * 1024) s = 24 * 1024;
  return s;
}
static_assert(kEmitWarps * (24 * 1024 + 2 * kStageBytes) <= kEmitMaxSmem, "the largest slots and their column stages fit one CTA");
void launch_encode_emit(KeyCols m, EncodeParams ep, EncodeWork w, uint64_t nblocks, uint8_t* const* out_base, uint64_t data_bytes,
                        int sms, cudaStream_t st, uint64_t* launches) {
  if (nblocks == 0) return;
  static PerDeviceFlag attr;
  const uint64_t dev_bit = attr.bit_of_current_device();
  if (!attr.is_set(dev_bit)) {
    cudaFuncSetAttribute(encode_emit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kEmitMaxSmem);
    cudaFuncSetAttribute(encode_emit_long_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kEmitMaxSmem);
    attr.set(dev_bit);
  }
  // Mean on-disk bytes per entry above 64 (data_bytes: the job's data blocks with their trailers): most values are longer than the
  // staged kernel's 32-byte vector path and go through per-lane word copies or the warp-wide copy, a chain of dependent loads per
  // value.  The 32 warps per SM of the long-entry kernel hide those chains better than the staged kernel's 12 (measured on H100
  // with 128 B and 256 B values: profiles/README.md).  A mean, unlike the smallest entry, does not flip on a few tombstones or
  // short values in a long-value job.
  const bool long_entries = data_bytes > 64 * m.n;
  const int warps = long_entries ? kEmitLongWarps : kEmitWarps, ctas = long_entries ? kEmitLongCtasPerSm : kEmitCtasPerSm;
  const uint32_t slot = encode_emit_slice(ep.block_size);
  const size_t smem = (size_t)warps * (slot + (long_entries ? 0 : 2 * kStageBytes));
  int per_sm = 0;  // resident CTAs per SM at this slot size (registers, static + dynamic shared memory)
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, long_entries ? (const void*)encode_emit_long_kernel : (const void*)encode_emit_kernel,
                                                warps * 32, smem);
  if (per_sm < 1) per_sm = 1;
  if (per_sm > ctas) per_sm = ctas;
  const uint64_t want = (nblocks + warps - 1) / warps;
  // The persistent CTAs own every register of the SMs they sit on, so the side stream's kernels (index-block writes and checksums)
  // queue behind the last emit CTA.
  const uint64_t cap = (uint64_t)sms * per_sm;
  const unsigned grid = (unsigned)(want < cap ? want : cap);
  if (long_entries) encode_emit_long_kernel<<<grid, warps * 32, smem, st>>>(m, ep, w, nblocks, out_base, slot);
  else encode_emit_kernel<<<grid, warps * 32, smem, st>>>(m, ep, w, nblocks, out_base, slot);
  *launches += 1;
}
static unsigned index_grid(uint64_t nblocks, int sms) {
  const uint64_t g = (nblocks + 255) / 256;
  return (unsigned)(g < (uint64_t)sms * 8 ? g : (uint64_t)sms * 8);
}
void launch_encode_index_size(KeyCols m, EncodeParams ep, EncodeWork w, uint64_t nblocks, int sms, cudaStream_t st, uint64_t* launches) {
  if (nblocks == 0) return;
  encode_index_size_kernel<<<index_grid(nblocks, sms), 256, 0, st>>>(m, w, nblocks, ep.format_version);
  *launches += 1;
  exclusive_scan<uint32_t>(w.idx_esz, w.idx_eoff, nblocks, w.scan_tmp, w.idx_eoff + nblocks, st, launches);
}
void launch_encode_index_write(EncodeParams ep, EncodeWork w, uint64_t nblocks, uint32_t nfiles, uint8_t* const* out_base, int sms,
                               cudaStream_t st, uint64_t* launches) {
  if (nblocks == 0) return;
  encode_index_write_kernel<<<index_grid(nblocks, sms), 256, 0, st>>>(w, nblocks, ep.format_version, out_base);
  *launches += 1;
  launch_file_block_checksums(w, nfiles, kIndexBlock, 64, ep.checksum, out_base, st, launches);
}
void launch_block_checksums(uint32_t type, const uint8_t* data, const uint64_t* offsets, uint32_t n, uint8_t last_byte, uint32_t* out,
                            cudaStream_t st) {
  if (n == 0) return;
  block_checksums_kernel<<<(n + 3) / 4, 128, 0, st>>>(type, data, offsets, n, last_byte, out);
}

}  // namespace b200c
