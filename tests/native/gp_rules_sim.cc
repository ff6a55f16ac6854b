// tests/native/gp_rules_sim.cc — test infrastructure: runs the product's grandparent cut rules (toplingdb_b200/csrc/gp_rules.h, the
// same code the encoder's stitch kernel runs on the device) on the CPU over the block layout of a finished job through the two
// steps encode.cu's chase_tile takes (gp_block_cut per open block, gp_size_cut behind a size cut), and reports where they cut.
// tests/test_gp_rules_host.py compares that with the file boundaries the oracle / the reference produced.
#include <stdint.h>

#include "gp_rules.h"

using namespace b200c;

extern "C" {

// blocks: per data block of the whole job, in order: first entry, entry count, bytes flushed to the block's file before it.
// last_of_file[b] != 0: the block is the last one of its output file.  max_output_file_size: the size rule (:277).
// Writes the entries in front of which the grandparent rules cut a file to cuts[] (capacity cap); returns their number, or
// -(b + 1) when block b is inconsistent with the rules (a cut inside a block that the layout continues, ...).
int64_t gp_rules_sim(uint32_t n_gp, const uint64_t* lo, const uint64_t* eq, const uint64_t* hi, const uint64_t* size,
                     const uint8_t* next_same, uint32_t dynamic_file_size, uint64_t max_compaction_bytes,
                     uint64_t target_output_file_size, uint64_t max_output_file_size, uint64_t n_entries, uint64_t n_blocks,
                     const uint64_t* blk_first, const uint32_t* blk_count, const uint64_t* blk_foff, const uint8_t* last_of_file,
                     uint64_t* cuts, uint64_t cap) {
  GpCtx c{n_gp, dynamic_file_size, lo, eq, hi, size, next_same, max_compaction_bytes, target_output_file_size};
  GpState g = gp_initial_state();
  if (n_entries) gp_advance(g, c, 0);
  uint64_t ncuts = 0;
  for (uint64_t b = 0; b < n_blocks; b++) {
    const uint64_t a = blk_first[b], end = a + blk_count[b], foff = blk_foff[b];
    if (last_of_file[b] && foff >= max_output_file_size) {  // the size rule closed the file behind this single-entry block
      if (blk_count[b] != 1) return -(int64_t)(b + 1);
      gp_size_cut(g, c, end, n_entries);
      continue;
    }
    const uint64_t cut = gp_block_cut(g, c, end, n_entries, foff);
    if (cut != ~0ull) {
      if (cut != end || !last_of_file[b]) return -(int64_t)(b + 1);  // the layout does not end a file here
      if (ncuts < cap) cuts[ncuts] = cut;
      ncuts++;
    } else if (last_of_file[b] && end < n_entries) {
      return -(int64_t)(b + 1);  // the layout ends a file the rules would not end
    }
  }
  return (int64_t)ncuts;
}

}  // extern "C"
