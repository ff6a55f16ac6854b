// toplingdb_b200/csrc/gp_rules.h — grandparent-aware output cutting on entry ranks.
//
// CompactionOutputs::UpdateGrandparentBoundaryInfo (db/compaction/compaction_outputs.cc:133-187) walks the grandparent files with
// every output key; its comparisons `key < smallest_i`, `key < / == largest_i`, `key < smallest_{i+1}` are the rank comparisons
// `e < lo_i`, `e < eq_i` / `eq_i <= e < hi_i`, `e < lo_{i+1}` for the merged entry e (GpCtx, kernels.h), so the state machine only
// has to run at the entries where a rank is reached.  Host + device: the encoder's stitch walk (encode.cu, chase_tile) runs it on
// the GPU, tests/native/gp_rules_sim.cc runs the same code on the CPU against the oracle's file boundaries.
//
// A second source of events, checked before the size and grandparent rules (ShouldStopBefore :264-269): the fixed-prefix SST
// partitioner (SstPartitionerFixedPrefix::ShouldPartition, db/compaction/sst_partitioner.cc) cuts in front of every output
// entry whose user key, truncated to the prefix length, differs from the previous output entry's.  That is a function of the merged
// stream alone, so the entries are listed once (partition_events_kernel, encode.cu) and the walk meets them like grandparent events.
// tests/native/partition_rules_sim.cc runs them on the CPU.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B200C_HD __host__ __device__ __forceinline__
#else
#define B200C_HD inline
#endif

namespace b200c {

struct GpCtx {
  uint32_t n;                  // grandparent files (0: rules off)
  uint32_t dynamic_file_size;  // level_compaction_dynamic_file_size
  const uint64_t* lo;          // [n] first merged entry with user key >= smallest_i
  const uint64_t* eq;          // [n] first merged entry with user key >= largest_i
  const uint64_t* hi;          // [n] first merged entry with user key >  largest_i
  const uint64_t* size;        // [n] file sizes
  const uint8_t* next_same;    // [n] smallest_{i+1} == largest_i (the key spans both files)
  uint64_t max_compaction_bytes, target_output_file_size;
  const uint64_t* pev;         // [np] ascending entries in front of which the partitioner cuts; ~0 past the last one
  uint32_t np;                 // slots of pev (0: no partitioner)
};

struct GpState {               // compaction_outputs.h:331-372 (being_grandparent_gap_, seen_key_, grandparent_index_, ...)
  uint32_t being_gap, seen, index, part;  // part: next partition event (pev index)
  uint64_t overlapped, switched;
};
B200C_HD GpState gp_initial_state() { return GpState{1, 0, 0, 0, 0, 0}; }

// the walk evaluates these rules (grandparents or a partitioner); without them only the size rule cuts files
B200C_HD bool gp_rules_on(const GpCtx& c) { return c.n != 0 || c.np != 0; }
// the next partition event, ~0 when there is none
B200C_HD uint64_t gp_next_partition(const GpState& g, const GpCtx& c) { return g.part < c.np ? c.pev[g.part] : ~0ull; }
// the entry at which the next boundary is crossed or the partitioner cuts, whichever comes first
B200C_HD uint64_t gp_next_event(const GpState& g, const GpCtx& c) {
  const uint64_t pe = gp_next_partition(g, c);
  if (g.index >= c.n) return pe;
  const uint64_t be = g.being_gap ? c.lo[g.index] : (c.next_same[g.index] ? c.eq[g.index] : c.hi[g.index]);
  return be < pe ? be : pe;
}
// GetCurrentKeyGrandparentOverlappedBytes (:189-229) for the key of entry e
B200C_HD uint64_t gp_overlap_at(const GpState& g, const GpCtx& c, uint64_t e) {
  if (g.being_gap || g.index >= c.n) return 0;
  uint64_t b = c.size[g.index];
  for (int64_t i = (int64_t)g.index - 1; i >= 0 && c.eq[i] <= e && e < c.hi[i]; i--) b += c.size[i];
  return b;
}
// UpdateGrandparentBoundaryInfo for the key of entry e: returns the number of boundaries crossed
B200C_HD uint32_t gp_advance(GpState& g, const GpCtx& c, uint64_t e) {
  uint32_t crossed = 0;
  while (g.index < c.n) {
    if (g.being_gap) {
      if (e < c.lo[g.index]) break;
      if (g.seen) {
        crossed++;
        g.overlapped += c.size[g.index];
        g.switched++;
      }
      g.being_gap = 0;
    } else {
      const uint64_t x = c.next_same[g.index] ? c.eq[g.index] : c.hi[g.index];
      if (e < x) break;
      if (g.seen) {
        crossed++;
        g.switched++;
      }
      g.being_gap = 1;
      g.index++;
    }
  }
  if (!g.seen && !g.being_gap) g.overlapped = gp_overlap_at(g, c, e);
  g.seen = 1;
  return crossed;
}
// the grandparent rules of ShouldStopBefore (:294-351) for an entry that crossed `crossed` boundaries; cur = bytes flushed so far
B200C_HD bool gp_should_stop(const GpState& g, const GpCtx& c, uint32_t crossed, uint64_t prev_overlapped, uint64_t cur) {
  if (crossed == 0) return false;
  if (g.overlapped + cur > c.max_compaction_bytes) return true;
  if (!c.dynamic_file_size) return false;
  const uint32_t skippable = g.being_gap ? 2 : 3;
  if (crossed >= skippable && g.overlapped - prev_overlapped > c.target_output_file_size / 8) return true;
  const uint64_t pct = g.switched * 5 < 40 ? g.switched * 5 : 40;
  return cur >= ((c.target_output_file_size + 99) / 100) * (50 + pct);
}
// AddToOutput :371-374: a new output file starts at entry e
B200C_HD void gp_file_started(GpState& g, const GpCtx& c, uint64_t e) {
  g.switched = 0;
  g.overlapped = gp_overlap_at(g, c, e);
}

// The two steps of the output-file walk over a stream of n entries (encode.cu chase_tile; tests/native/gp_rules_sim.cc).
// The entries a < e <= end are added while one block is open and `cur` bytes are flushed to the file: crosses the boundaries up to
// `end` and returns the first entry in front of which the rules end the file (the boundary state is then the next file's), or ~0.
// Every event seen here lies behind the open file's first entry: each file start was passed to gp_advance (the stream's first entry
// before the walk, the cut returned here, the entry behind gp_size_cut's), and gp_next_event is always beyond the last entry
// advanced to.  So the rules never stop in front of a file's first key, and no guard for that is needed.
// A partition event ends the file whatever the other rules say; the boundary state has moved to that entry first (:247-253).
B200C_HD uint64_t gp_block_cut(GpState& g, const GpCtx& c, uint64_t end, uint64_t n, uint64_t cur) {
  uint64_t ev;
  while ((ev = gp_next_event(g, c)) <= end && ev < n) {
    const uint64_t prev_overlapped = g.overlapped;
    const uint32_t crossed = gp_advance(g, c, ev);
    const bool partition = ev == gp_next_partition(g, c);
    if (partition) g.part++;
    if (partition || gp_should_stop(g, c, crossed, prev_overlapped, cur)) {
      gp_file_started(g, c, ev);
      return ev;
    }
  }
  return ~0ull;
}
// the size rule closed the file behind entry e - 1 (:277): ShouldStopBefore(e) moved the boundary state before the rule fired, and
// entry e starts the next file.  A partition event at e asks for the same cut (it is checked first, :264-269) and is used up by it.
B200C_HD void gp_size_cut(GpState& g, const GpCtx& c, uint64_t e, uint64_t n) {
  if (e >= n) return;
  gp_advance(g, c, e);
  if (gp_next_partition(g, c) == e) g.part++;
  gp_file_started(g, c, e);
}

}  // namespace b200c
