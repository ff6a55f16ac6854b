// toplingdb_b200/csrc/kernels.h — host-visible declarations of the kernel launchers (decode.cu, merge.cu, encode.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

#include "common.cuh"
#include "gp_rules.h"

namespace b200c {

// cudaFuncSetAttribute acts on the current device only, and one process may drive several devices (one executor factory per GPU):
// remember per device ordinal which kernels already carry their dynamic shared memory limit.  Racing threads just set it twice.
struct PerDeviceFlag {
  std::atomic<uint64_t> mask{0};
  uint64_t bit_of_current_device() const {
    int d = 0;
    cudaGetDevice(&d);
    return 1ull << (d & 63);
  }
  bool is_set(uint64_t bit) const { return (mask.load(std::memory_order_acquire) & bit) != 0; }
  void set(uint64_t bit) { mask.fetch_or(bit, std::memory_order_release); }
};

struct FileDesc {          // one input BlockBasedTable image resident in HBM
  const uint8_t* base;
  uint64_t len;
  uint64_t index_off;
  uint32_t index_size;
  uint32_t value_delta;    // index values delta-encoded (format_version >= 4)
  uint32_t cksum;          // footer checksum type
  uint32_t gblk_first;     // first global data-block number of this file
  uint32_t nblocks;        // rocksdb.num.data.blocks
  uint32_t index_user_key; // rocksdb.index.key.is.user.key: index separators are user keys (no trailer)
  const uint8_t* index_ptr; // nullptr: the index block lies at base + index_off; else its inflated copy (index_size = inflated size)
};

struct BoundKey {              // a user key in column form (grandparent boundary, sub-compaction range bound)
  uint64_t hi, lo;
  uint32_t ulen, pad;
};

// ---- decode.cu
// blk_size[b] == 0 marks a data block that a sub-compaction's key range [start, end) cannot touch (range_rules.h): the block decoder
// publishes an empty block for it without reading the image
void launch_index_decode(const FileDesc* files_dev, int nfiles, uint32_t max_blocks_per_file, uint64_t* blk_off, uint32_t* blk_size,
                         BoundKey start, uint32_t has_start, BoundKey end, uint32_t has_end, uint32_t* err, cudaStream_t st, uint64_t* launches);
void launch_block_decode_fused(const FileDesc* files_dev, int nfiles, const uint64_t* blk_off, const uint32_t* blk_size, uint32_t nblk,
                               uint32_t verify, uint64_t n_total, KeyColsMut out, unsigned long long* blk_state, uint32_t* ticket,
                               uint64_t* run_start, uint64_t* total_out, uint32_t* err, int sms, cudaStream_t st, uint64_t* launches,
                               const uint8_t* arena = nullptr);
// Inputs with kZlibCompression data blocks (UncompressBlockData, table/format.cc:511): slot[b] = bytes block b needs in the arena of
// inflated blocks (0: stored uncompressed / outside the key range); after an exclusive scan of the slots, launch_inflate_blocks verifies
// the stored bytes' checksums, inflates every compressed block into its slot and redirects its handle (blk_off / blk_size) there.
void launch_block_usize(const FileDesc* files_dev, const uint64_t* blk_off, const uint32_t* blk_size, uint32_t nblk, uint32_t* slot, uint32_t* err,
                        cudaStream_t st, uint64_t* launches);
void launch_inflate_blocks(const FileDesc* files_dev, uint64_t* blk_off, uint32_t* blk_size, const uint32_t* slot, const uint64_t* slot_off,
                           uint32_t nblk, uint8_t* arena, uint32_t verify, uint32_t* err, int sms, cudaStream_t st, uint64_t* launches);
// paranoid_file_checks: entry i of `written` (what the encoder consumed) and of `reread` (the output images decoded again) must be
// the same key, the same trailer and the same value bytes; a difference sets kErrParanoid
void launch_flip_byte(uint8_t* p, cudaStream_t st);  // test hook of paranoid_file_checks
void launch_compare_columns(KeyCols written, KeyCols reread, uint64_t n, uint32_t* err, int sms, cudaStream_t st, uint64_t* launches);
void launch_gather_values(KeyCols in, const uint64_t* dst_off, uint8_t* dst, cudaStream_t st);
void launch_meta_vlen(const uint32_t* meta, uint64_t n, uint32_t* vlen, cudaStream_t st);
// host records (internal key + value, back to back) -> key columns with value references into the device arena
void launch_kv_to_columns(const uint8_t* arena, const uint64_t* offs, const uint32_t* klens, uint64_t n, KeyColsMut out, uint32_t* err,
                          int sms, cudaStream_t st);

struct TailCopy {  // one finished file tail: staged bytes [src_off, src_off + len) -> output buffer at dst_off
  uint64_t dst_off;
  uint32_t src_off, len;
};
struct FileRec;
void launch_gather_small(const uint64_t* small, uint32_t small_bytes, const FileRec* files, const uint64_t* nfiles_dev, uint8_t* dst,
                         cudaStream_t st);
void launch_copy_small(const void* src, void* dst, uint32_t n, cudaStream_t st);  // byte copy, either side may be mapped host memory
void launch_scatter_tails(const TailCopy* recs, uint32_t n, const uint8_t* staged, uint8_t* out, cudaStream_t st);

// ---- merge.cu
constexpr int kMergeTile = 2048;     // capacity of a CTA tile (merged entries)
// Tiles are cut every kMergeNominal merged entries.  When an input holds a kTypeSingleDeletion the cut moves forward to the end of the
// user key it falls into (at most kSdSpill entries), so that all versions of a key meet in one tile: the SingleDelete rules are a
// chain through the versions of a key (compaction_iterator.cc:662-887) and are walked serially per key (group_rules.h).
constexpr int kSdSpill = 32;
constexpr int kMergeNominal = kMergeTile - kSdSpill;
constexpr int kMaxRuns = 64;
struct MergeParams {
  uint32_t nruns;
  uint32_t bottommost;               // Compaction::bottommost_level()
  uint32_t nsnapshots;
  const uint64_t* snapshots;         // device, ascending
  uint64_t earliest_snapshot;        // snapshots[0] or kMaxSeq
  uint32_t filter;                   // b200c_compaction_filter
  int32_t ttl;                       // B200C_FILTER_TTL
  int64_t now;
  uint32_t write_conflict_snapshot;  // CompactionParams::earliest_write_conflict_snapshot is set (transaction DB): SingleDelete -> CPU
};
struct TileStat {            // partial sums for the per-file statistics over one "stat tile" of consecutive output entries
  uint64_t raw_key, raw_value, deletions, smallest_seq, largest_seq;
};
// What the merge kernel writes for the encoder besides the merged columns (it holds every output entry and its predecessor in
// shared memory anyway): the encoded size / shared-prefix length of every entry except the first one of a tile (its predecessor
// is the previous tile's last survivor: merge_sizes_fix_kernel fills those in), the statistics of the tile's output entries, and
// the smallest / largest entry size of the job.
struct MergeSizes {
  uint32_t* esz;        // n_out
  uint8_t* eshared;     // n_out
  TileStat* tstat;      // one per merge tile; the tile's output range is [prefix(t-1), prefix(t)) from tile_state
  uint32_t* min_s1;     // [0] min, [1] max of esz
};
struct MergeCounters {               // device-side CompactionIterationStats
  unsigned long long n_out, n_input_deletions, n_hidden, n_obsolete, raw_key_bytes, raw_value_bytes, n_silent, n_user_drop;
};
// splits: (ntiles + 1) x nruns u64; tile_state: ntiles u64 (zeroed); ticket: u32 (zeroed)
// run r of the merge = entries [begin[r], end[r]) of the decoded columns.  Whole input files: end = begin + 1 over the run_start
// array the decoder fills; a sub-compaction's key range: the clipped bounds from launch_clip_runs.
struct RunBounds {
  const uint64_t* begin;
  const uint64_t* end;
};
// Sub-compaction key range (ClippingIterator, db/compaction/clipping_iterator.h:55-358): per run the entries with
// start <= user key < end.  clip[r] / clip[nruns + r] = first / one-past-last entry of run r in range; totals[0] += entries in
// range, totals[1] += their value bytes.
void launch_clip_runs(KeyCols in, RunBounds runs, uint32_t nruns, BoundKey start, uint32_t has_start, BoundKey end,
                      uint32_t has_end, uint64_t* clip, unsigned long long* totals, cudaStream_t st, uint64_t* launches);
// Sorted runs from decoded files: run r = the files [run_first[r], run_first[r + 1]), decoded back to back; bounds = begin[nruns] |
// end[nruns].  Checks that consecutive files of one run are in order (a level's files are disjoint and sorted): kErrKeyOrder.
void launch_run_bounds(KeyCols in, const uint64_t* file_start, const uint32_t* run_first, uint32_t nruns, uint64_t* bounds, uint32_t* err,
                       cudaStream_t st, uint64_t* launches);
void launch_merge_partition(KeyCols in, RunBounds runs, uint32_t nruns, uint64_t n_total, uint64_t ntiles,
                            uint64_t* splits, uint32_t* err, int sms, cudaStream_t st, uint64_t* launches);
void launch_merge_tiles(KeyCols in, RunBounds runs, MergeParams mp, uint64_t n_total, uint64_t ntiles,
                        const uint64_t* splits, unsigned long long* tile_state, uint32_t* ticket, KeyColsMut out,
                        MergeCounters* counters, MergeSizes ms, uint32_t* err, cudaStream_t st, uint64_t* launches);
// sizes of each tile's first output entry (needs the finished tile_state prefixes and merged columns)
void launch_merge_sizes_fix(KeyCols merged, const unsigned long long* tile_state, uint64_t ntiles, MergeSizes ms, cudaStream_t st, uint64_t* launches);

// ---- encode.cu
// Grandparent-aware output cutting (CompactionOutputs::ShouldStopBefore, compaction_outputs.cc:231-354).  The walk over the block
// chain only needs to know at which merged ENTRY each boundary of a grandparent file is crossed, so the boundaries are turned
// into entry ranks once (gp_rank_kernel) and the reference's key-driven state machine runs on ranks.
struct GpCut {                 // an output file that was cut in front of `entry` by a grandparent rule or the partitioner
  uint64_t entry;
  uint64_t block_bytes;        // on-disk bytes of the (truncated) block that ends in front of it
};
struct EncodeParams {
  uint32_t block_size, block_size_limit /* ceil(block_size*(100-deviation)/100), 0 = disabled */, restart_interval;
  uint32_t checksum, format_version, output_level;
  uint64_t max_output_file_size;
  GpCtx gp;
  GpCut* gp_cuts;              // written by the stitch kernel (capacity 2 * gp.n + 2 + gp.np), replayed by the block-list kernel
  uint32_t* gp_ncuts;
};
using GpKey = BoundKey;       // grandparent boundary key in column form
// ---- full Bloom filter block (bloom_rules.h).  count: per file the number of entries whose key hash differs from the predecessor's
// (XXPH3FilterBitsBuilder::AddKey drops consecutive duplicates) and from it the block size; build: set the bits, metadata, trailer.
void launch_bloom_count(KeyCols m, uint64_t n, FileRec* files, const uint64_t* nfiles_dev, uint32_t millibits, uint64_t* hashes, int sms, cudaStream_t st,
                        uint64_t* launches);
// max_filter_bytes: largest filter_bytes of a file (grid sizing); the checksums use w.files and w.cksum_contrib*
struct EncodeWork;
void launch_bloom_build(const uint64_t* hashes, uint64_t n, const EncodeWork& w, uint32_t nfiles, uint32_t max_filter_bytes, uint32_t millibits,
                        uint32_t cksum, uint8_t* const* out_base, cudaStream_t st, uint64_t* launches);
// fixed-prefix partitioner: the merged entries in front of which it cuts (gp_rules.h), ascending, into ev[0, cap); ev must hold ~0
// and ticket / state (partition_event_tiles(m.n) words) zero beforehand.  More than cap events set kErrTooManyFiles.
uint64_t partition_event_tiles(uint64_t n);
void launch_partition_events(KeyCols m, uint32_t len, uint32_t cap, uint32_t* ticket, unsigned long long* state, uint64_t* ev, uint32_t* err,
                             cudaStream_t st, uint64_t* launches);
void launch_gp_ranks(KeyCols m, const GpKey* smallest, const GpKey* largest, uint32_t n, uint64_t* lo, uint64_t* eq, uint64_t* hi,
                     cudaStream_t st, uint64_t* launches);
struct BlockRec {            // one output data block
  uint64_t first_entry;
  uint64_t file_off;         // offset of the block payload inside its file
  uint32_t file_idx;
  uint32_t n_entries;
};
struct KeyRec {
  uint64_t hi, lo, tr;
  uint32_t ulen, pad;
};
constexpr uint32_t kBlockTrailerLen = 5;  // compression type + checksum behind every block
// An output image is  data blocks | filter block | index block | tail (properties, metaindex, footer);  the filter and the index
// block each carry a trailer.  The accessors below are the one statement of that layout.
struct FileRec {             // one output file (device-computed part)
  uint64_t first_entry, n_entries;
  uint64_t first_block, n_blocks;
  uint64_t data_size;        // bytes of data blocks incl. trailers
  uint64_t index_size;       // index block payload bytes (without trailer)
  uint64_t raw_key_size, raw_value_size, num_deletions;
  uint64_t smallest_seq, largest_seq;
  KeyRec smallest, largest;
  uint32_t index_has_seq;    // some adjacent blocks share a user key => index keys keep the 8-byte trailer
  uint64_t filter_entries;   // hashes in the Bloom filter (rocksdb.num.filter_entries); 0 without a filter policy
  uint64_t filter_bytes;     // filter block on disk: bits + 5 metadata bytes + trailer; 0 without a filter

  __host__ __device__ uint64_t filter_start() const { return data_size; }
  // filter bits + metadata, without the trailer (0: no filter block)
  __host__ __device__ uint64_t filter_len() const { return filter_bytes ? filter_bytes - kBlockTrailerLen : 0; }
  __host__ __device__ uint64_t index_start() const { return data_size + filter_bytes; }
  __host__ __device__ uint64_t tail_start() const { return index_start() + index_size + kBlockTrailerLen; }
  // the index block with its trailer takes at most this (<= 45 B per data block + 9), before index_size is known
  __host__ __device__ uint64_t index_bound() const { return n_blocks * 48 + 64; }
  // bytes the image needs at most with a tail of tail_bytes
  __host__ __device__ uint64_t image_bound(uint64_t tail_bytes) const { return index_start() + index_bound() + tail_bytes; }
  // rocksdb.index.key.is.user.key (index_builder.h:175-180): no two adjacent blocks share a user key, from format_version 3 on
  __host__ __device__ bool index_key_is_user_key(uint32_t format_version) const { return !index_has_seq && format_version > 2; }
};
struct TileRow {             // block-cut transfer function of one tile for one entry-point candidate
  uint32_t exit;             // chain exit, entries past the tile end
  uint32_t nblk;             // blocks started inside the tile
  uint64_t bytes;            // on-disk bytes (payload + 5) of those blocks
};
struct TileState {           // resolved state when the chain enters a tile
  uint64_t entry;            // absolute index of the first block start at/after the tile start
  uint64_t blk;              // index of that block
  uint64_t file_off;         // bytes already flushed to the current file
  uint32_t file_idx;
  uint32_t pad;
};
constexpr int kEncTile = 4096;       // entries per block-cut tile
constexpr int kEncHalo = 2048;       // look-ahead window = the longest block (in entries) the encoder accepts
constexpr int kEncGroupTiles = 16;   // tiles per stitch group (encode.cu kEncGroup)
constexpr uint32_t kMaxOutFiles = 4096;

struct EncodeWork {                  // device scratch owned by the job
  uint32_t* esz;        // n: encoded size of entry i as a non-restart entry (s1)
  uint8_t* eshared;     // n: bytes shared with the previous internal key
  TileStat* tstat;      // statistics per stat tile: merge tiles (written by the merge kernel) or kEncTile entries (sizes kernel)
  const unsigned long long* tprefix;  // per stat tile: entries up to and including the tile (low 62 bits; the top bits are flags)
  uint64_t nstat;       // number of stat tiles
  uint32_t* min_s1;     // 2: [0] global min of esz (bounds the entry-point candidate window), [1] global max
  TileRow* rows;        // ntiles x hc
  TileRow* grows;       // ngroups x hc: composed transfer functions of kEncGroup tiles (exit relative to the group start)
  TileState* gstate;    // ngroups: state at which the chain enters the group
  uint32_t* gflag;      // ngroups: 1 = the stitch kernel walked this group tile by tile (a file ends inside)
  uint32_t* gdone;      // ngroups (zeroed): tile CTAs of the tables kernel that finished the group; the last one composes the group row
  uint32_t* gready;     // ngroups (zeroed): 1 = rows / nxt / disk of the group's tiles and its composed row are complete -- the stitch
                        // kernel runs CONCURRENTLY with the tables kernel (second stream) and waits on these flags
  TileState* tstate;    // ntiles
  uint64_t* totals;     // [0] = number of blocks, [1] = number of files
  BlockRec* blocks;     // capacity nblk_cap
  FileRec* files;       // kMaxOutFiles
  uint32_t* idx_esz;    // per block: encoded index entry size without the key's 8-byte trailer (index_has_seq adds it)
  uint64_t* idx_eoff;   // nblocks + 1: exclusive scan of idx_esz, the total behind it
  KeyRec* idx_sep;      // per block: separator key (ulen excludes the trailer; pad=1 when the trailer was replaced)
  uint64_t* scan_tmp;
  // XXH3 accumulator contributions of the 1024-byte blocks of every index and filter block (8 u64 each); first slot per file:
  // cksum_contrib_off[f] for its index block, cksum_contrib_off[nfiles + f] for its filter block (file_block_contrib_offsets)
  uint64_t* cksum_contrib;
  uint64_t* cksum_contrib_off;
  uint16_t* nxt;        // n: tile-relative end of the block that would start at entry i
  uint32_t* disk;       // n: on-disk bytes of that block
};
// TableBuilder-only path (no merge in front): sizes + statistics per kEncTile entries + their prefix array (tprefix_out)
void launch_encode_sizes(KeyCols m, const unsigned long long* n_dev, EncodeWork w, unsigned long long* tprefix_out, uint64_t n_cap, int sms, cudaStream_t st);
void launch_encode_tables(KeyCols m, EncodeParams ep, EncodeWork w, uint64_t ntiles, uint32_t hc, uint32_t max_s1, cudaStream_t st,
                          uint64_t* launches);
// stitch: launched on its own stream BEFORE / alongside launch_encode_tables (it consumes groups as their gready flag appears);
// tilestate: after both have finished
void launch_encode_stitch(KeyCols m, EncodeParams ep, EncodeWork w, uint64_t ntiles, uint32_t hc, uint32_t* err, uint32_t attempt,
                          uint32_t* sflag, cudaStream_t st, uint64_t* launches);
void launch_encode_tilestate(KeyCols m, EncodeWork w, uint64_t ntiles, uint32_t hc, uint32_t* err, cudaStream_t st, uint64_t* launches);
void launch_encode_blocklist(KeyCols m, EncodeParams ep, EncodeWork w, uint64_t ntiles, uint64_t nblk_cap, uint32_t* err,
                             cudaStream_t st, uint64_t* launches);
// per-file statistics, boundary keys and index-block size: after launch_encode_index_size
void launch_encode_filestats(KeyCols m, EncodeWork w, uint32_t nfiles, cudaStream_t st, uint64_t* launches);
uint32_t encode_emit_slice(uint32_t block_size);
// out_base[f] = device address where file f's image starts; data_bytes = all data blocks incl. trailers (with m.n: selects the kernel)
void launch_encode_emit(KeyCols m, EncodeParams ep, EncodeWork w, uint64_t nblocks, uint8_t* const* out_base, uint64_t data_bytes,
                        int sms, cudaStream_t st, uint64_t* launches);
// index blocks in two steps: separators, entry sizes and their scan (what the file sizes need), then the entries, restart arrays and
// trailers written into the images
void launch_encode_index_size(KeyCols m, EncodeParams ep, EncodeWork w, uint64_t nblocks, int sms, cudaStream_t st, uint64_t* launches);
void launch_encode_index_write(EncodeParams ep, EncodeWork w, uint64_t nblocks, uint32_t nfiles, uint8_t* const* out_base, int sms,
                               cudaStream_t st, uint64_t* launches);
void launch_block_checksums(uint32_t type, const uint8_t* data, const uint64_t* offsets, uint32_t n, uint8_t last_byte,
                            uint32_t* out, cudaStream_t st);

}  // namespace b200c
