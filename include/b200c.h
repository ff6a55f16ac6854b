/* include/b200c.h — C ABI of the B200 compaction engine (libb200c.so).
 *
 * This is the drop-in boundary for ToplingDB's compaction hot path.  The reference has no C ABI / FFI for
 * this path (db/c.cc only exposes rocksdb_compact_range); the path sits behind two C++ virtual interfaces:
 *   - CompactionExecutorFactory / CompactionExecutor   db/compaction/compaction_executor.h:160-178
 *       SetParams(CompactionParams*, const Compaction*), Execute(const CompactionParams&, CompactionResults*)
 *   - TableFactory / TableReader / TableBuilder         include/rocksdb/table.h:844-934
 * The plugin classes registered with ROCKSDB_FACTORY_REG("B200Compact", ...) (see INTEGRATION.md and
 * toplingdb_b200/plugin/) translate those objects into the calls below.  What each entry point replaces:
 *
 *   b200c_job_create        CompactionJob ctor + CompactionExecutor::SetParams   compaction_job.cc:921-963
 *   b200c_job_add_input     VersionSet::MakeInputIterator: one child per L0 file / level   db/version_set.cc:7269-7352
 *   b200c_job_run           CompactionExecutor::Execute -> CompactionJob::RunLocal ->
 *                           ProcessKeyValueCompaction                          compaction_job.cc:659,971,1390-1780
 *   b200c_job_output_*      CompactionResults::output_files[i] = FileMinMeta   compaction_executor.h:120-158
 *   b200c_job_get_stats     CompactionResults::job_stats (CompactionJobStats)  include/rocksdb/compaction_job_stats.h
 *
 * Conventions: plain pointers and sizes only; integer status codes (0 = OK), never exceptions; the last
 * error text of the calling thread is b200c_last_error().  One job handle may be used by one thread at a
 * time; different handles are independent and the library is re-entrant across handles (the reference calls
 * Execute() concurrently from several background compaction threads).  Input buffers are borrowed until
 * b200c_job_destroy / b200c_job_run returns; output buffers are owned by the job.
 * There is NO CPU fallback: every data-path call fails with B200C_ERR_NO_DEVICE when no CUDA device is usable.
 */
#ifndef B200C_H_
#define B200C_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200C_ABI_VERSION 8
#if defined(__GNUC__)
#define B200C_API __attribute__((visibility("default")))
#else
#define B200C_API
#endif

enum b200c_status {
  B200C_OK = 0,
  B200C_ERR_INVALID_ARGUMENT = 1,
  B200C_ERR_NO_DEVICE = 2,       /* no CUDA device / driver: the path has no CPU implementation */
  B200C_ERR_CUDA = 3,            /* a CUDA runtime call failed (message has the call and error string) */
  B200C_ERR_CORRUPTION = 4,      /* bad magic / handle / block checksum / key order in an input file */
  B200C_ERR_NOT_SUPPORTED = 5,   /* input needs a rule outside the device rule set (merge operands, range
                                    tombstones, compressed blocks, user keys > 16 bytes, ...):
                                    the executor must report ShouldRunLocal()==true / fall back (compaction_job.cc:649-652) */
  B200C_ERR_OUT_OF_MEMORY = 6,
  B200C_ERR_STATE = 7            /* call order violated (e.g. output queried before run) */
};

enum b200c_mem_kind {
  B200C_MEM_HOST = 0,
  B200C_MEM_DEVICE = 1,
  B200C_MEM_HOST_DEFERRED = 2 /* b200c_job_add_input only: a host image whose upload waits for b200c_job_upload_by_ranges / the run */
};
/* CompactionFilter applied inside the merge kernel (compaction_iterator.cc:231-473, :579-584): only built-in filters whose
 * decision is a function of the entry itself can run on the device */
enum b200c_compaction_filter {
  B200C_FILTER_NONE = 0,
  B200C_FILTER_REMOVE_EMPTY_VALUE = 1, /* RemoveEmptyValueCompactionFilter (utilities/compaction_filters/remove_emptyvalue_compactionfilter.cc:15-22) */
  B200C_FILTER_TTL = 2                 /* TtlCompactionFilter of DBWithTTL without a user filter (utilities/ttl/db_ttl_impl.cc:200-206,
                                          445-461): a value whose trailing fixed32 write time + ttl < ttl_now is removed */
};
enum b200c_checksum { B200C_CKSUM_NONE = 0, B200C_CKSUM_CRC32C = 1, B200C_CKSUM_XXH3 = 4 }; /* ChecksumType, table.h:54-60 */

/* One file of the level below the output level (Compaction::grandparents(), compaction_executor.h:66-110 `grandparents`): user-key
 * range and size.  With grandparents the output files are also cut at grandparent boundaries
 * (CompactionOutputs::ShouldStopBefore, db/compaction/compaction_outputs.cc:294-351). */
typedef struct b200c_grandparent {
  const void* smallest_user_key;
  uint32_t smallest_len;
  const void* largest_user_key;
  uint32_t largest_len;
  uint64_t file_size;
} b200c_grandparent;

/* Job parameters: the fields of CompactionParams (compaction_executor.h:33-118), of the output
 * BlockBasedTableOptions (include/rocksdb/table.h:237-564) and of TableBuilderOptions
 * (compaction_job.cc:2258-2331) that decide the output bytes.  Zero-initialise, then b200c_params_init(). */
typedef struct b200c_params {
  uint32_t abi_version;            /* B200C_ABI_VERSION */
  int32_t device;                  /* CUDA device ordinal for this job */
  int32_t output_level;            /* CompactionParams::output_level; 0 => never cut files (compaction_outputs.cc:272) */
  int32_t bottommost_level;        /* CompactionParams::bottommost_level */
  uint64_t max_output_file_size;   /* Compaction::max_output_file_size() (compaction.cc:291-295) */
  uint32_t block_size;             /* 4096 */
  uint32_t block_size_deviation;   /* 10 */
  uint32_t block_restart_interval; /* 16 */
  uint32_t index_block_restart_interval; /* 1 (only value the device index builder accepts) */
  uint32_t format_version;         /* 5 */
  uint32_t checksum;               /* enum b200c_checksum of the OUTPUT files; inputs carry their own */
  uint32_t verify_input_checksums; /* ReadOptions::verify_checksums of the compaction read (default 1) */
  const uint64_t* snapshots;       /* CompactionParams::existing_snapshots, ascending; may be NULL */
  uint32_t num_snapshots;
  uint32_t column_family_id;
  const char* column_family_name;  /* rocksdb.column.family.name */
  const char* db_id;               /* rocksdb.creating.db.identity */
  const char* db_session_id;       /* rocksdb.creating.session.identity */
  const char* db_host_id;          /* rocksdb.creating.host.identity */
  uint64_t creation_time;          /* rocksdb.creation.time = oldest ancestor time of the inputs */
  uint64_t oldest_key_time;        /* rocksdb.oldest.key.time */
  const uint64_t* file_creation_times; /* clock reading at each OpenCompactionOutputFile (compaction_job.cc:2258-2266);
                                          entry i for output i, the last one repeats; NULL => 0 (property omitted) */
  uint32_t num_file_creation_times;
  uint64_t first_file_number;      /* outputs are numbered first_file_number, +1, ... (orig_file_number property) */
  uint32_t output_mem;             /* enum b200c_mem_kind: where b200c_job_output_data() pointers live */
  uint32_t profile;                /* != 0: bracket every kernel group with CUDA events (b200c_job_kernel_time) */
  uint32_t compaction_filter;      /* enum b200c_compaction_filter */
  int32_t ttl;                     /* B200C_FILTER_TTL: seconds; <= 0 keeps everything */
  int64_t ttl_now;                 /* B200C_FILTER_TTL: clock reading (seconds) the write times are compared with */
  const b200c_grandparent* grandparents; /* sorted by key, as Compaction::grandparents(); NULL / 0: size rule only */
  uint32_t num_grandparents;
  uint32_t level_compaction_dynamic_file_size; /* ImmutableOptions::level_compaction_dynamic_file_size (default 1) */
  uint64_t max_compaction_bytes;       /* Compaction::max_compaction_bytes(); 0 => 25 x target_output_file_size */
  uint64_t target_output_file_size;    /* Compaction::target_output_file_size(); 0 => max_output_file_size */
  /* Sub-compaction key range (SubcompactionState::start / end, db/compaction/subcompaction_state.h; ProcessKeyValueCompaction clips
   * the merged input with a ClippingIterator, compaction_job.cc:1433-1519, db/compaction/clipping_iterator.h:55-358): only entries
   * with range_start <= user key < range_end are compacted; the job's statistics count those entries only.  has_* == 0: unbounded
   * on that side.  Jobs over disjoint ranges of the same inputs are independent (one per GPU / stream). */
  const void* range_start_user_key;
  uint32_t range_start_len;
  uint32_t has_range_start;
  const void* range_end_user_key;
  uint32_t range_end_len;
  uint32_t has_range_end;
  /* CompactionParams::paranoid_file_checks (compaction_executor.h:71; CompactionJob::Run, compaction_job.cc:829-853, re-reads every
   * output file and compares an OutputValidator hash of its keys and values with the one taken while writing).  != 0: after the
   * output images are complete they are decoded again on the device (block checksums verified) and every key and value is compared
   * with what the encoder was given; a difference fails the job with B200C_ERR_CORRUPTION "Paranoid checksums do not match". */
  uint32_t paranoid_file_checks;
  /* BlockBasedTableOptions::filter_policy = NewBloomFilterPolicy(bits_per_key): BloomLikeFilterPolicy::millibits_per_key_
   * (= int(bits_per_key * 1000 + 0.500001), table/block_based/filter_policy.cc:1327-1343).  != 0: every output file gets a full
   * (non-partitioned) FastLocalBloom filter block over its whole user keys, between the data blocks and the index block
   * (BlockBasedTableBuilder::WriteFilterBlock, block_based_table_builder.cc:1488-1538), the metaindex entry
   * "fullfilter.rocksdb.BuiltinBloomFilter" and the filter properties.  Needs format_version >= 5 (older versions build the legacy
   * Bloom filter), whole_key_filtering, no prefix extractor, optimize_filters_for_memory = false (the defaults). */
  uint32_t bloom_millibits_per_key;
  /* CompactionParams::earliest_write_conflict_snapshot (compaction_executor.h:70): 0 or kMaxSequenceNumber = none.  It only changes
   * what happens to a SingleDelete (compaction_iterator.cc:801-838); with one set (transaction DBs) an input that holds a
   * SingleDelete is answered with B200C_ERR_NOT_SUPPORTED. */
  uint64_t earliest_write_conflict_snapshot;
  /* ColumnFamilyOptions::sst_partitioner_factory = NewSstPartitionerFixedPrefixFactory(len): the prefix length, 0 = no partitioner.
   * Appended to the struct (the ABI version did not change): a caller that zero-initialises it, or leaves it as b200c_params_init
   * sets it, keeps the old behaviour.  An output file never holds two user keys whose first `len` bytes differ: CompactionOutputs::
   * ShouldStopBefore (db/compaction/compaction_outputs.cc:264-269) ends the file in front of every output entry whose user key,
   * truncated to len bytes (a shorter key stays whole), differs from the previous output entry's (SstPartitionerFixedPrefix::
   * ShouldPartition, db/compaction/sst_partitioner.cc) -- before the size and grandparent rules, never at a file's first entry.
   * Ignored when output_level == 0 (no partitioner for L0 outputs, compaction_outputs.cc:793-795).  A job whose partition cuts alone
   * would give more output files than the device's file records hold (4096) is answered with B200C_ERR_NOT_SUPPORTED before any
   * file is written. */
  uint32_t sst_partitioner_prefix_len;
} b200c_params;

/* FileMinMeta (compaction_executor.h:120-131) + the TableProperties RunRemote re-reads (compaction_job.cc:1043-1061) */
typedef struct b200c_file_meta {
  uint64_t file_number, file_size;
  uint64_t smallest_seqno, largest_seqno;
  uint64_t num_entries, num_deletions, raw_key_size, raw_value_size, num_data_blocks, data_size, index_size;
  uint32_t smallest_ikey_len, largest_ikey_len;
  uint8_t smallest_ikey[64], largest_ikey[64];
} b200c_file_meta;

/* CompactionJobStats subset (include/rocksdb/compaction_job_stats.h) + device timings */
typedef struct b200c_stats {
  uint64_t num_input_records, num_output_records;
  uint64_t num_input_deletion_records;
  uint64_t num_records_replaced;         /* CompactionIterationStats::num_record_drop_hidden */
  uint64_t num_expired_deletion_records; /* num_record_drop_obsolete */
  uint64_t total_input_raw_key_bytes, total_input_raw_value_bytes;
  uint64_t total_input_bytes, total_output_bytes;
  uint64_t num_input_files, num_output_files;
  /* device time of the last run, microseconds, CUDA events on the job stream */
  double decode_us, merge_us, encode_us, total_us;
  uint64_t kernel_launches; /* kernels of this library launched by the last run */
  uint64_t num_record_drop_user; /* entries the compaction filter turned into tombstones (CompactionIterationStats) */
} b200c_stats;

typedef struct b200c_job b200c_job;

B200C_API const char* b200c_last_error(void);
B200C_API uint32_t b200c_abi_version(void);
B200C_API int b200c_device_count(void); /* >= 0, or -B200C_ERR_NO_DEVICE */

B200C_API void b200c_params_init(b200c_params* p); /* reference defaults (table.h:237-564, advanced_options.h:599) */

B200C_API int b200c_job_create(const b200c_params* p, b200c_job** out);
/* Append one sorted run (a whole BlockBasedTable file image).  Order matters exactly as in MakeInputIterator:
 * L0 files newest first, then one run per deeper level.  `data` may be host or device memory (mem_kind).
 * Device memory is read by the job's own non-blocking CUDA streams from b200c_job_run() on: whatever produces it (a copy or a
 * kernel on the caller's stream) must have COMPLETED before the run call -- the library does not join the caller's streams. */
B200C_API int b200c_job_add_input(b200c_job* j, int level, uint64_t file_number, const void* data, uint64_t len, int mem_kind);
/* Files added with the same level > 0 one after the other form ONE sorted run, like the LevelIterator MakeInputIterator builds for a
 * level (db/version_set.cc:1076,7311-7352): they must be disjoint and in key order (checked on the device).  A job may hold any number
 * of files but at most 64 runs (L0 files + deeper levels).  For a host image of at least 1 MiB the host -> device copy starts inside
 * this call on a copy stream of the job (the caller's next file read overlaps it); the buffer must stay unchanged until the run ends. */

/* Page-locked host memory for input images (cudaHostAlloc, portable): copies from it run at full PCIe speed and truly asynchronously.
 * A thread that set a NUMA memory policy before the call gets the pages from that node.  ReadFile targets of the executor plugin
 * (plugin/b200_compaction_executor.cc) come from here; replaces nothing in the reference (its local path reads through the block cache). */
B200C_API int b200c_host_alloc(int device, uint64_t bytes, void** out);
B200C_API void b200c_host_free(void* p);
/* decode -> k-way merge with the compaction-iterator rules -> encode, all on the device.  Synchronous. */
B200C_API int b200c_job_run(b200c_job* j);
B200C_API int b200c_job_output_count(const b200c_job* j);
B200C_API int b200c_job_output_meta(const b200c_job* j, int i, b200c_file_meta* m);
/* Pointer to the finished file image of output i (host or device memory according to params.output_mem). */
B200C_API int b200c_job_output_data(b200c_job* j, int i, const void** data, uint64_t* len);
/* Copy output i into caller memory (host; with output_mem == DEVICE the destination may also be device memory). */
B200C_API int b200c_job_output_read(b200c_job* j, int i, void* dst, uint64_t cap);
B200C_API int b200c_job_get_stats(const b200c_job* j, b200c_stats* s);
B200C_API void b200c_job_destroy(b200c_job* j);

/* ---- one job over several key ranges: the reference's sub-compactions (CompactionJob::Prepare / GenSubcompactionBoundaries,
 * db/compaction/compaction_job.cc:264-281,465-640; CompactionResults::output_files[sub], compaction_executor.h:120-158) ----
 * b200c_job_plan_ranges: up to max_ranges - 1 boundary user keys (ascending; keys: 16 bytes per slot, key_lens: their lengths) that
 * cut the job's inputs into ranges [.., k0) [k0, k1) ... [k_last, ..) of about equal input bytes, none smaller than min_range_bytes
 * (the reference: at least one output file per range).  The boundaries come from ~128 anchors per input file read off its index
 * block, as GenSubcompactionBoundaries reads them from TableReader::ApproximateKeyAnchors.  Host work only (O(index blocks)).
 * b200c_job_create_sub: a job over the SAME inputs as `parent` -- their device copies are made once, by the parent -- restricted to
 * the key range in `p` (range_start / range_end) on the parent's device, with its own streams and buffers: sub-jobs of one parent may
 * run concurrently from different host threads.  The parent must outlive its sub-jobs; it does not have to run itself.  Create the
 * sub-jobs from one thread, after the last b200c_job_add_input on the parent. */
B200C_API int b200c_job_plan_ranges(b200c_job* j, uint32_t max_ranges, uint64_t min_range_bytes, uint8_t* keys, uint32_t* key_lens,
                                    uint32_t* n_boundaries);
B200C_API int b200c_job_create_sub(b200c_job* parent, const b200c_params* p, b200c_job** out);
/* Pipelines ONE job over its own PCIe link: the parent's host inputs (added with B200C_MEM_HOST_DEFERRED) are uploaded in KEY order --
 * first the index / metadata tail of every file, then, range after range, the data blocks that range can touch (cut at the first block
 * whose index separator reaches the boundary) -- and an event is recorded behind every range.  A sub-job created afterwards for
 * [boundary r-1, boundary r) only waits for ITS event: it decodes, merges, encodes and downloads its outputs while the later ranges
 * are still going up, so host -> device, compute and device -> host of one job overlap (a job that is uploaded whole, compacted and
 * downloaded is two PCIe copies long: 78 of 83 ms on the bench job).  keys / key_lens / n_boundaries as b200c_job_plan_ranges fills
 * them.  The reference has no counterpart (its sub-compactions share the block cache); results are per range, as for any sub-job. */
B200C_API int b200c_job_upload_by_ranges(b200c_job* parent, const uint8_t* keys, const uint32_t* key_lens, uint32_t n_boundaries);

/* ---- stage-level entry points (used by the parity tests and by bench.py's per-kernel roofline) ---- */
enum b200c_debug_array {
  B200C_DBG_DECODED_KEYS = 1, /* run r: per entry { u64 hi, u64 lo, u64 trailer, u32 ulen, u32 vlen } (32 B) */
  B200C_DBG_DECODED_VALUES = 2, /* run r: value bytes, concatenated in entry order */
  B200C_DBG_MERGED_KEYS = 3,  /* surviving merged stream, same 32 B records */
  B200C_DBG_MERGED_VALUES = 4,
  B200C_DBG_BLOCK_LIST = 5    /* per output data block { u64 first_entry, u64 file_offset, u32 file_index, u32 n_entries } */
};
/* Run only up to a stage (1 = decode, 2 = merge, 3 = everything) keeping intermediates for b200c_job_debug_read. */
B200C_API int b200c_job_run_until(b200c_job* j, int stage);
/* Copies the array into dst (host) and returns the byte count needed in *len. run is ignored for merged arrays. */
B200C_API int b200c_job_debug_read(b200c_job* j, int what, int run, void* dst, uint64_t cap, uint64_t* len);

/* Per-kernel-group device times of the last run (params.profile != 0): name and microseconds. */
B200C_API int b200c_job_kernel_time_count(const b200c_job* j);
B200C_API int b200c_job_kernel_time(const b200c_job* j, int i, const char** name, double* us);

/* TableBuilder side of the path alone (BlockBasedTableBuilder::Add/Finish, table/table_builder.h:168-235): encode one
 * sorted run that already sits in device memory as columns into BlockBasedTable image(s), cut like compaction outputs.
 * Columns, n entries each:  pfx  16 B  first 16 user-key bytes as two big-endian-decoded u64 (hi, lo), zero padded
 *                           tr    8 B  (sequence << 8) | value type
 *                           vref  8 B  device address of the value bytes
 *                           meta  4 B  user_key_len << 27 | value_len
 * Results are read with b200c_job_output_*.  Used by the table-factory plugin and to pre-stage synthetic inputs. */
B200C_API int b200c_job_encode_columns(b200c_job* j, uint64_t n, const void* pfx, const void* tr, const void* vref, const void* meta);
/* The same for a caller that holds its entries in HOST memory, as a TableBuilder does between Add() calls (table/table_builder.h:168-
 * 239; BlockBasedTableBuilder::Add / Finish, block_based_table_builder.cc:961-1133, 1921-1977): n entries in internal-key order; entry i
 * is its internal key (klens[i] bytes, user key + 8-byte trailer) immediately followed by its value and starts at arena + offs[i]; the
 * value ends where entry i + 1 starts, offs[n] = bytes used.  The plugin's B200TableBuilder (plugin/b200_table_factory.cc) calls this
 * from Finish().  B200C_ERR_NOT_SUPPORTED for what the device encoder does not take (user keys > 16 bytes, types other than
 * kTypeValue / kTypeDeletion): the builder then replays its records into the reference's own BlockBasedTableBuilder. */
B200C_API int b200c_job_encode_kv(b200c_job* j, uint64_t n, const void* arena, const uint64_t* offs, const uint32_t* klens);

/* Block checksum of table/format.cc:468-509 computed on the device for n independent buffers laid out
 * back to back (offsets[n+1]); results in out[n].  type = enum b200c_checksum. */
B200C_API int b200c_block_checksums(int device, uint32_t type, const void* host_data, const uint64_t* offsets, uint32_t n,
                          uint8_t last_byte, uint32_t* out);

#ifdef __cplusplus
}
#endif
#endif /* B200C_H_ */
