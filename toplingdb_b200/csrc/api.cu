// toplingdb_b200/csrc/api.cu — the C ABI of include/b200c.h: job object + host orchestration of the three device stages.
// Host work is O(files): parse the ~1 KB tail of every input, lay out the output images, build the ~1 KB tail of every
// output.  Everything per entry / per block is a kernel launch (decode.cu, merge.cu, encode.cu).  No CPU data path exists.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <memory>
#include <mutex>
#include <unordered_map>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

#include "../../include/b200c.h"
#include "inflate_rules.h"
#include "kernels.h"
#include "range_plan.h"
#include "scan.cuh"
#include "sst_host.h"

using namespace b200c;

namespace {

thread_local std::string g_err;
size_t g_last_want = 0;  // size of the last device allocation attempted (diagnostics of an out-of-memory status)
std::mutex g_host_allocs_mu;
std::unordered_map<void*, std::pair<size_t, int>> g_host_allocs;  // b200c_host_alloc: size class and device of every live buffer
int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}
std::string mem_note() {
  size_t fr = 0, tot = 0;
  cudaMemGetInfo(&fr, &tot);
  cudaGetLastError();
  return " (requested " + std::to_string(g_last_want) + " bytes; device free " + std::to_string(fr) + " of " + std::to_string(tot) + ")";
}
#define CU(call)                                                                                                  \
  do {                                                                                                            \
    cudaError_t e_ = (call);                                                                                      \
    if (e_ != cudaSuccess) {                                                                                      \
      cudaGetLastError();                                                                                         \
      return fail(e_ == cudaErrorMemoryAllocation ? B200C_ERR_OUT_OF_MEMORY : B200C_ERR_CUDA,                      \
                  std::string(#call) + ": " + cudaGetErrorString(e_) + (e_ == cudaErrorMemoryAllocation ? mem_note() : ""));  \
    }                                                                                                             \
  } while (0)

// Buffers of finished jobs are kept for the next one.  A DB hands the executor a fresh job handle per compaction, and allocating a
// job's working set anew costs more than the job itself: cudaHostAlloc pins page by page (~0.3 ms per MiB), cudaMalloc / cudaFree of
// gigabytes synchronise the device.  One cache per kind (device / pinned host) and device, bounded (B200C_CACHE_DEVICE_MB, default
// 49152; B200C_CACHE_HOST_MB, default 16384; 0 = off).  Requests are rounded to a few size classes; a cached buffer serves requests
// between half its size and its size.  Nothing is zeroed: every kernel writes what it later reads (the same rule a job handle that
// runs twice already relies on).  When an allocation fails the caches of the device are emptied and the call is retried once.
constexpr int kCacheDevices = 16;
inline size_t size_class(size_t n) {
  size_t c = 4096;
  while (c < n) c <<= 1;
  if (c >= (size_t(1) << 20)) {  // above 1 MiB: eighths of the power of two
    const size_t step = c >> 4;  // (c/2)/8
    c = (c >> 1) + ((n - (c >> 1) + step - 1) / step) * step;
  }
  return c;
}
class BufCache {
 public:
  BufCache(bool host, const char* env, size_t default_mb) : host_(host) {
    const char* e = getenv(env);
    cap_ = (e ? strtoull(e, nullptr, 10) : default_mb) << 20;
  }
  void* take(int dev, size_t n, size_t* got) {
    if (dev < 0 || dev >= kCacheDevices || cap_ == 0) return nullptr;
    std::lock_guard<std::mutex> l(mu_);
    auto it = free_[dev].lower_bound(n);
    if (it == free_[dev].end() || it->first > 2 * n) return nullptr;
    void* p = it->second;
    *got = it->first;
    held_[dev] -= it->first;
    free_[dev].erase(it);
    return p;
  }
  bool give(int dev, void* p, size_t n) {  // false: not kept, the caller frees
    if (dev < 0 || dev >= kCacheDevices || cap_ == 0) return false;
    std::lock_guard<std::mutex> l(mu_);
    if (held_[dev] + n > cap_) return false;
    free_[dev].emplace(n, p);
    held_[dev] += n;
    return true;
  }
  void flush(int dev) {
    if (dev < 0 || dev >= kCacheDevices) return;
    std::multimap<size_t, void*> drop;
    {
      std::lock_guard<std::mutex> l(mu_);
      drop.swap(free_[dev]);
      held_[dev] = 0;
    }
    for (auto& kv : drop) {
      if (host_) cudaFreeHost(kv.second);
      else cudaFree(kv.second);
    }
  }

 private:
  bool host_;
  size_t cap_ = 0;
  std::mutex mu_;
  std::multimap<size_t, void*> free_[kCacheDevices];
  size_t held_[kCacheDevices] = {};
};
BufCache& dev_cache() {
  static BufCache* c = new BufCache(false, "B200C_CACHE_DEVICE_MB", 49152);  // leaked on purpose: no CUDA calls at process exit
  return *c;
}
BufCache& host_cache() {
  static BufCache* c = new BufCache(true, "B200C_CACHE_HOST_MB", 16384);
  return *c;
}
inline int current_device() {
  int d = -1;
  cudaGetDevice(&d);
  return d;
}
cudaError_t cached_alloc(bool host, size_t n, void** out, size_t* cap, int* dev_out) {
  const int dev = current_device();
  const size_t want = size_class(n);
  *dev_out = dev;
  BufCache& c = host ? host_cache() : dev_cache();
  if (void* p = c.take(dev, want, cap)) {
    *out = p;
    return cudaSuccess;
  }
  g_last_want = want;
  // (pinned buffers are mapped: kernels read / write them directly -- same address under UVA, see read_small())
  auto raw = [&]() { return host ? cudaHostAlloc(out, want, cudaHostAllocMapped | cudaHostAllocPortable) : cudaMalloc(out, want); };
  cudaError_t e = raw();
  if (e == cudaErrorMemoryAllocation) {
    cudaGetLastError();
    dev_cache().flush(dev);
    host_cache().flush(dev);
    e = raw();
  }
  if (e == cudaSuccess) *cap = want;
  return e;
}
void cached_free(bool host, void* p, size_t cap, int dev) {
  if (!p) return;
  if ((host ? host_cache() : dev_cache()).give(dev, p, cap)) return;
  if (host) cudaFreeHost(p);
  else cudaFree(p);
}

// Grow-only allocation in device memory or in mapped pinned host memory, reused across runs of the same job (and, through the
// cache, by later jobs).  The destructor gives it back to the cache, so nothing that uses it may be in flight when it goes out of
// scope.  Move-only: a copy would give one allocation to the cache twice, and the cache would hand it to two jobs.
template <bool kPinned>
struct Buf {
  uint8_t* p = nullptr;
  size_t cap = 0;
  int dev = -1;
  Buf() = default;
  Buf(Buf&& o) noexcept : p(o.p), cap(o.cap), dev(o.dev) {
    o.p = nullptr;
    o.cap = 0;
  }
  Buf(const Buf&) = delete;
  Buf& operator=(const Buf&) = delete;
  ~Buf() { cached_free(kPinned, p, cap, dev); }
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    // growing in the middle of a job: earlier launches may still use the old block, cudaFree waits for them
    if (p) kPinned ? cudaFreeHost(p) : cudaFree(p);
    p = nullptr;
    cap = 0;
    void* q = nullptr;
    const cudaError_t e = cached_alloc(kPinned, n + (n >> 4) + 256, &q, &cap, &dev);
    if (e == cudaSuccess) p = static_cast<uint8_t*>(q);
    return e;
  }
  template <class T>
  T* as() const {
    return reinterpret_cast<T*>(p);
  }
};
using DevBuf = Buf<false>;  // device memory
using HostBuf = Buf<true>;  // pinned host memory: D2H target of the finished images, small staging areas
static_assert(!std::is_copy_constructible_v<DevBuf> && !std::is_copy_assignable_v<DevBuf>, "a buffer has one owner");

// The key columns of decoded or merged entries: pfx 16 B (.x = hi, .y = lo), tr 8 B, vref 8 B, meta 4 B per entry.
struct KeyBufs {
  DevBuf pfx, tr, vref, meta;
  cudaError_t reserve(uint64_t n) {  // n entries and one spare
    cudaError_t e = pfx.reserve(16 * (n + 1));
    if (e == cudaSuccess) e = tr.reserve(8 * (n + 1));
    if (e == cudaSuccess) e = vref.reserve(8 * (n + 1));
    if (e == cudaSuccess) e = meta.reserve(4 * (n + 1));
    return e;
  }
  KeyColsMut mut() const { return {pfx.as<ulonglong2>(), tr.as<uint64_t>(), vref.as<uint64_t>(), meta.as<uint32_t>()}; }
  KeyCols cols(uint64_t n) const { return {pfx.as<ulonglong2>(), tr.as<uint64_t>(), vref.as<uint64_t>(), meta.as<uint32_t>(), n}; }
};

struct HostCopy {  // the device copy of a host input (stage_input)
  DevBuf buf;
  cudaEvent_t done = nullptr;  // recorded behind the last copy into buf, on the stream that made it (nullptr: no copy yet)
  bool fresh = false;          // b200c_job_add_input's eager copy: the next run consumes it (later runs copy anew: the host buffer may change)
};
struct IndexBlock {            // the index block of an input as the host reads it (input_index_block)
  const uint8_t* p = nullptr;  // into a host image, or into buf: the block read from device memory, or inflated
  uint64_t len = 0;
  bool inflated = false;
  std::vector<uint8_t> buf;
};
struct Input {
  int level;
  uint64_t file_number;
  const uint8_t* data;
  uint64_t len;
  int mem_kind;
  HostCopy copy;
  IndexBlock index;       // a compressed input's index block, read by run_job (the source of the upload; kept until the run ends)
  DevBuf index_inflated;  // ... its device copy when it was inflated
  InputTail tail;
};
constexpr uint64_t kTailFetch = 4096;  // bytes read from the end of an input: footer + metaindex + properties live there
struct Output {
  b200c_file_meta meta;
  uint64_t dev_off = 0;   // offset of the image inside out_buf
  uint64_t host_off = 0;  // offset inside host_out when output_mem == HOST
};
struct KernelTime {
  const char* name;
  cudaEvent_t a, b;
  float us;
};

}  // namespace

struct b200c_job {
  b200c_params p;
  std::vector<uint64_t> snapshots, fct;
  std::string cf_name, db_id, db_session_id, db_host_id;
  std::vector<Input> inputs;
  std::vector<Output> outputs;
  b200c_stats stats;
  int stage_done = 0;  // last stage the current run completed: 1 decode, 2 merge, 3 encode (the outputs can be read)
  uint64_t launches = 0;  // kernel launches of the current run (stats.kernel_launches)
  int sms = 132;  // replaced by the device's own count when the job binds its device
  cudaStream_t st = nullptr;
  cudaStream_t st2 = nullptr;  // side stream (higher priority): serial / small kernels that overlap a bulk kernel on `st`
  cudaStream_t st_up = nullptr;  // copy stream of the eager input uploads
  cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t evx[4] = {nullptr, nullptr, nullptr, nullptr};  // fork / join points between st and st2
  // device state
  DevBuf files_d, blk_off, blk_size, blk_state, scan_tmp, run_start, small;  // small: err, totals, counters...
  KeyBufs dec, mrg;
  DevBuf splits, tile_state, snaps_d;
  DevBuf esz, eshared, tstat, nxt, disk, rows, tstate, grows, gstate, gflag, gsync, blocks, files_rec, idx_esz, idx_eoff, idx_sep, out_buf, out_base_d;
  uint64_t n_total = 0, n_out = 0, nblk_in = 0, nblocks_out = 0;
  uint32_t nfiles_out = 0, nruns = 0;
  DevBuf cksum_contrib, cksum_contrib_off;  // scratch of the index and filter blocks' checksums
  DevBuf bloom_hashes;                      // key hashes of the output entries (filter policy jobs)
  DevBuf kv_arena, kv_offs, kv_klens;  // b200c_job_encode_kv: the caller's records on the device
  DevBuf run_bounds, run_first_d;  // [begin[K] | end[K]] of the sorted runs in the decoded columns; first file of each run
  std::vector<uint64_t> run_start_h;
  HostBuf host_out;
  std::vector<GpKey> gp_small, gp_large;  // grandparent boundaries in column form (packed at job creation)
  std::vector<uint64_t> gp_size;
  std::vector<uint8_t> gp_same;
  DevBuf gp_keys_d, gp_ranks_d, gp_size_d, gp_same_d, gp_cuts_d;
  DevBuf pev_d;  // fixed-prefix partitioner: event entries, look-back ticket and state
  BoundKey range_lo{}, range_hi{};  // sub-compaction key range in column form (has_range_start / has_range_end in p)
  DevBuf clip_d;                    // clipped run bounds: begin[k] | end[k]
  DevBuf cslot, cslot_off, arena;   // compressed inputs: arena slot size / offset per data block, the inflated blocks
  std::vector<cudaEvent_t> range_events;   // b200c_job_upload_by_ranges: event r = the blocks of ranges 0..r (and every file's tail) are on the device
  std::vector<std::string> range_bounds;   // ... the boundary user keys it was called with
  cudaEvent_t wait_ev = nullptr;           // sub-job of such a parent: what its streams wait for before they touch the inputs (owned by the parent)
  DevBuf vfiles_d, vrun_start;      // paranoid_file_checks: descriptors / run table of the outputs being read back
  HostBuf pin_small, pin_tails, pin_rd, pin_up;
  size_t pin_up_used = 0;  // pinned staging: input tails / tail-copy records, output tails
  std::vector<KernelTime> ktimes;
  size_t kt_used = 0;
  // profiling: bracket a named group of launches with events (only when params.profile != 0)
  // names that start with '~' run on the side stream, overlapped with the neighbouring group on the main stream
  size_t kt_begin(const char* name, cudaStream_t s = nullptr) {
    if (!p.profile) return 0;
    if (kt_used == ktimes.size()) {
      KernelTime k{name, nullptr, nullptr, 0.f};
      cudaEventCreate(&k.a);
      cudaEventCreate(&k.b);
      ktimes.push_back(k);
    }
    ktimes[kt_used].name = name;
    cudaEventRecord(ktimes[kt_used].a, s ? s : st);
    return kt_used++;
  }
  void kt_end(size_t slot = ~(size_t)0, cudaStream_t s = nullptr) {
    if (!p.profile) return;
    cudaEventRecord(ktimes[slot == ~(size_t)0 ? kt_used - 1 : slot].b, s ? s : st);
  }
};

namespace {

// layout of the `small` buffer (u64 slots)
enum { kSlotErr = 0, kSlotTicket = 1, kSlotTotalIn = 2, kSlotMinS1 = 3, kSlotTotals = 4 /* 2 */, kSlotDecTicket = 6, kSlotGpCuts = 7, kSlotCounters = 8 /* 8 */, kSlotClip = 16 /* 2: entries, value bytes in range */, kSlotStitchDone = 18, kSlotArena = 19 /* bytes of the inflated-block arena */, kSmallSlots = 32 };

int map_dev_err(uint32_t e) {
  e &= ~(uint32_t)kFlagHasSingleDelete;  // a note of the decoder, not an error
  if (e == 0) return B200C_OK;
  std::string m = "device reported:";
  int code = B200C_ERR_CORRUPTION;
  if (e & kErrCorruptBlock) m += " corrupt-block";
  if (e & kErrChecksum) m += " block-checksum-mismatch";
  if (e & kErrKeyOrder) m += " key-order/partition";
  if (e & kErrCountMismatch) m += " entry-count-mismatch";
  if (e & kErrParanoid) m += " Paranoid checksums do not match (an output file does not read back as written)";
  if (e & kErrSingleDelContract) m += " SingleDelete and Delete of the same key in one snapshot stripe (enforce_single_del_contracts)";
  const uint32_t unsup = kErrKeyTooLong | kErrValueTooLong | kErrBadType | kErrCompressed | kErrBlockTooLong | kErrIrregularRestarts |
                         kErrGroupTooLong | kErrSdWriteConflict | kErrTooManyFiles;
  if (e & unsup) {
    if (!(e & ~(unsup))) code = B200C_ERR_NOT_SUPPORTED;
    if (e & kErrKeyTooLong) m += " user-key-longer-than-16-bytes";
    if (e & kErrValueTooLong) m += " value>=128MiB";
    if (e & kErrBadType) m += " value-type-outside-{Value,Deletion,SingleDeletion}";
    if (e & kErrGroupTooLong) m += " SingleDelete-on-a-key-with-too-many-versions-or-with-more-than-16-runs";
    if (e & kErrSdWriteConflict) m += " SingleDelete-with-an-earliest_write_conflict_snapshot";
    if (e & kErrCompressed) m += " compressed-block";
    if (e & kErrBlockTooLong) m += " output-block-with-too-many-entries";
    if (e & kErrIrregularRestarts) m += " restart-intervals-of-unequal-length";
    if (e & kErrTooManyFiles) m += " more-than-" + std::to_string(kMaxOutFiles) + "-output-files";
  }
  if (e & kErrInternal) {
    m += " internal";
    code = B200C_ERR_CUDA;
  }
  return fail(code, m);
}

// checksum of a block read on the host against its trailer: compression type, then the checksum as 4 little-endian bytes
bool trailer_ok(const Input& in, const uint8_t* blk, uint64_t size, const uint8_t* trailer) {
  const uint32_t stored = (uint32_t)trailer[1] | (uint32_t)trailer[2] << 8 | (uint32_t)trailer[3] << 16 | (uint32_t)trailer[4] << 24;
  return !in.tail.checksum_type || host_block_checksum(in.tail.checksum_type, blk, size, trailer[0]) == stored;
}

// Bytes [off, off + n) of an input image for the host: *p points into a host image, or into *buf, where they are copied from a
// device image on the job's stream (behind its wait_ev: job_bind).
int read_image(b200c_job* j, const Input& in, uint64_t off, uint64_t n, std::vector<uint8_t>* buf, const uint8_t** p) {
  *p = in.data + off;
  if (in.mem_kind == B200C_MEM_HOST) return B200C_OK;
  buf->resize(n);
  CU(cudaMemcpyAsync(buf->data(), *p, n, cudaMemcpyDeviceToHost, j->st));
  CU(cudaStreamSynchronize(j->st));
  *p = buf->data();
  return B200C_OK;
}

// The tail of an input -- footer, metaindex, properties -- into in.tail, and every refusal of a single input.  tp: the last
// kTailFetch bytes of a device image, already read (run_job reads those of all its device images in one batch).
int open_input(b200c_job* j, Input& in, const uint8_t* tp = nullptr) {
  if (in.len < 53) return fail(B200C_ERR_CORRUPTION, "input shorter than a footer");
  const uint64_t tail_off = in.len - std::min<uint64_t>(in.len, kTailFetch);
  std::vector<uint8_t> tail, tmp;
  if (!tp)
    if (int rc = read_image(j, in, tail_off, in.len - tail_off, &tail, &tp)) return rc;
  // bytes [off, off + n) of the image, n <= len - off: inside its tail, or read on their own
  auto view = [&](uint64_t off, uint64_t n, const uint8_t** p) -> int {
    if (off < tail_off) return read_image(j, in, off, n, &tmp, p);
    *p = tp + (off - tail_off);
    return B200C_OK;
  };
  const uint8_t* blk;
  if (int rc = view(in.len - 53, 53, &blk)) return rc;
  std::string e = parse_footer(blk, in.len, &in.tail);
  if (!e.empty()) return fail(B200C_ERR_CORRUPTION, e);
  if (int rc = view(in.tail.meta_off, in.tail.meta_size + 5, &blk)) return rc;
  if (!trailer_ok(in, blk, in.tail.meta_size, blk + in.tail.meta_size)) return fail(B200C_ERR_CORRUPTION, "metaindex block checksum mismatch");
  std::map<std::string, std::pair<uint64_t, uint64_t>> meta;
  e = parse_metaindex(blk, in.tail.meta_size, &meta);
  if (!e.empty()) return fail(B200C_ERR_CORRUPTION, e);
  for (auto& kv : meta) {
    if (kv.first == "rocksdb.range_del") in.tail.has_range_del = true;
    if (kv.first.compare(0, 11, "fullfilter.") == 0 || kv.first.compare(0, 18, "partitionedfilter.") == 0) in.tail.has_filter = true;
    if (kv.first == "rocksdb.compression_dict") in.tail.has_dict = true;
  }
  auto it = meta.find("rocksdb.properties");
  if (it == meta.end()) return fail(B200C_ERR_CORRUPTION, "input has no properties block");
  in.tail.props_off = it->second.first;
  in.tail.props_size = it->second.second;
  if (in.tail.props_off + in.tail.props_size + 5 > in.len) return fail(B200C_ERR_CORRUPTION, "properties handle out of range");
  if (int rc = view(in.tail.props_off, in.tail.props_size + 5, &blk)) return rc;
  // num_entries / num_data_blocks from this block size every device buffer: its checksum is verified like the metaindex block's
  if (!trailer_ok(in, blk, in.tail.props_size, blk + in.tail.props_size)) return fail(B200C_ERR_CORRUPTION, "properties block checksum mismatch");
  e = parse_properties(blk, in.tail.props_size, &in.tail);
  if (!e.empty()) return fail(B200C_ERR_CORRUPTION, e);
  // a file written earlier under other table options (two-level / hash index) must be refused as such, not fed to the flat index
  // decoder (it would fail late as a count mismatch = Corruption, which AllowFallbackToLocal() does not cover)
  if (in.tail.index_type != 0)
    return fail(B200C_ERR_NOT_SUPPORTED, "input index type " + std::to_string(in.tail.index_type) + " (only kBinarySearch runs on the device)");
  if (in.tail.has_range_del || in.tail.num_range_deletions)
    return fail(B200C_ERR_NOT_SUPPORTED, "input holds range tombstones (CompactionRangeDelAggregator is not on the device path)");
  if (in.tail.num_merge_operands) return fail(B200C_ERR_NOT_SUPPORTED, "input holds merge operands");
  if (in.tail.has_dict) return fail(B200C_ERR_NOT_SUPPORTED, "input uses a compression dictionary");
  if (!in.tail.comparator_name.empty() && in.tail.comparator_name != "leveldb.BytewiseComparator")
    return fail(B200C_ERR_NOT_SUPPORTED, "comparator " + in.tail.comparator_name + " (only leveldb.BytewiseComparator runs on the device)");
  if (in.tail.num_data_blocks > 0xffffffffull) return fail(B200C_ERR_NOT_SUPPORTED, "too many data blocks");
  if (in.mem_kind != B200C_MEM_HOST && ((uintptr_t)in.data & 15)) return fail(B200C_ERR_INVALID_ARGUMENT, "device input images must be 16-byte aligned");
  if (in.tail.index_size > 0xffffffffull) return fail(B200C_ERR_NOT_SUPPORTED, "index block >= 4 GiB");
  return B200C_OK;
}

bool input_is_compressed(const Input& in) { return !in.tail.compression_name.empty() && in.tail.compression_name != "NoCompression"; }
// The index block of an opened input.  A file written with block compression stores it through the same WriteBlock as its data
// blocks (enable_index_compression, block_based_table_builder.cc:1566-1573): O(blocks) metadata that the host reads anyway, so a
// compressed one is inflated here (inflate_rules.h compiled for the host) once its checksum is verified.  It may announce
// 8 <= u <= 2^31 bytes: 8 is the smallest index block (a restart offset and the restart count; the device's index decoder refuses
// less).  A data block has its own bounds (decode.cu compressed_prefix); the upper bounds' difference of one is kept as it was.
int input_index_block(b200c_job* j, const Input& in, IndexBlock* out) {
  const uint64_t size = in.tail.index_size;
  out->len = size;
  out->inflated = false;
  if (int rc = read_image(j, in, in.tail.index_off, size + 5, &out->buf, &out->p)) return rc;  // (inside the image: parse_footer)
  const uint8_t* trailer = out->p + size;
  if (!input_is_compressed(in) || trailer[0] == 0) return B200C_OK;
  if (trailer[0] != kZlibCompressionType)
    return fail(B200C_ERR_NOT_SUPPORTED, "index block compressed with a codec the device path does not decode");
  if (!trailer_ok(in, out->p, size, trailer)) return fail(B200C_ERR_CORRUPTION, "index block checksum mismatch");
  uint64_t u = 0;
  const int h = inf_size_prefix(out->p, (uint32_t)size, &u);
  if (h == 0 || u < 8 || u > (1ull << 31)) return fail(B200C_ERR_CORRUPTION, "compressed index block announces a bad size");
  std::vector<uint8_t> raw((size_t)u);
  std::unique_ptr<b200c::InfWork> iw(new b200c::InfWork);
  if (b200c::inflate_raw(out->p + h, (uint32_t)(size - h), raw.data(), (uint32_t)u, iw.get()) != (long)u)
    return fail(B200C_ERR_CORRUPTION, "compressed index block does not inflate to its announced size");
  out->buf.swap(raw);
  out->p = out->buf.data();
  out->len = u;
  out->inflated = true;
  return B200C_OK;
}

// Hands stream s the device copy of host input `in`.  With reuse and a copy made before (by any writer), s waits for it; otherwise
// bytes [lo, hi) are copied on s, and `done` is recorded behind them.
int stage_input(Input& in, cudaStream_t s, bool reuse, uint64_t lo = 0, uint64_t hi = ~0ull) {
  HostCopy& c = in.copy;
  if (reuse && c.done) {
    CU(cudaStreamWaitEvent(s, c.done, 0));
    return B200C_OK;
  }
  hi = std::min(hi, in.len);
  CU(c.buf.reserve(in.len + 64));
  if (hi > lo) CU(cudaMemcpyAsync(c.buf.p + lo, in.data + lo, hi - lo, cudaMemcpyHostToDevice, s));
  if (!c.done) CU(cudaEventCreateWithFlags(&c.done, cudaEventDisableTiming));
  CU(cudaEventRecord(c.done, s));
  return B200C_OK;
}

void ikey_bytes(const KeyRec& k, uint8_t* out, uint32_t* len) {
  uint32_t n = 0;
  for (uint32_t t = 0; t < k.ulen && t < 16; t++) out[n++] = (uint8_t)((t < 8 ? k.hi >> (56 - 8 * t) : k.lo >> (56 - 8 * (t - 8))) & 0xff);
  for (int t = 0; t < 8; t++) out[n++] = (uint8_t)(k.tr >> (8 * t));
  *len = n;
}

// encode stage: merged columns (device) -> output file images + metas.  `h` holds the small-slot snapshot read at sync #1.
// Small host -> device uploads (descriptors, offsets, snapshots): staged in mapped pinned memory and moved by a tiny kernel, for
// the same reason as read_small(): a cudaMemcpy would wait on the copy engine behind other jobs' multi-GB input uploads.
// The staging area is a bump allocator that is reset at the start of a run (the previous run has been synchronised).
int upload_small(b200c_job* j, void* dev_dst, const void* host_src, size_t n) {
  const size_t kCap = 256 * 1024;
  CU(j->pin_up.reserve(kCap));
  const size_t off = (j->pin_up_used + 15) & ~(size_t)15;
  if (off + n > kCap) {  // unusually many files / snapshots: plain copy
    CU(cudaMemcpyAsync(dev_dst, host_src, n, cudaMemcpyHostToDevice, j->st));
    return B200C_OK;
  }
  memcpy(j->pin_up.p + off, host_src, n);
  j->pin_up_used = off + n;
  launch_copy_small(j->pin_up.p + off, dev_dst, (uint32_t)n, j->st);
  return B200C_OK;
}

// Small device -> host reads (counters, per-file records) go through a tiny kernel that writes mapped pinned memory, not
// through cudaMemcpy: a D2H copy would queue on the copy engine behind the multi-GB output downloads of OTHER jobs running
// on the same device, and every host decision point of this job would wait for them.
// gather_small() enqueues the copy of the `small` slots and (files != nullptr) the first *nfiles_dev file records; take_small() reads
// them once the stream has passed that point.  read_small() does both around a synchronisation of the stream.
constexpr size_t kRdSmall = kSmallSlots * 8;
int gather_small(b200c_job* j, const FileRec* files) {
  const uint64_t* small = j->small.as<uint64_t>();
  CU(j->pin_rd.reserve(kRdSmall + sizeof(FileRec) * (size_t)kMaxOutFiles));
  launch_gather_small(small, (uint32_t)kRdSmall, files, files ? small + kSlotTotals + 1 : nullptr, j->pin_rd.p, j->st);
  return B200C_OK;
}
void take_small(b200c_job* j, uint64_t* h, const FileRec* files, std::vector<FileRec>* frs) {
  memcpy(h, j->pin_rd.p, kRdSmall);
  if (files && frs) {
    uint64_t n = h[kSlotTotals + 1];
    if (n > kMaxOutFiles) n = kMaxOutFiles;
    frs->resize(n);
    memcpy(frs->data(), j->pin_rd.p + kRdSmall, sizeof(FileRec) * n);
  }
}
int read_small(b200c_job* j, uint64_t* h, const FileRec* files = nullptr, std::vector<FileRec>* frs = nullptr) {
  if (int rc = gather_small(j, files)) return rc;
  CU(cudaStreamSynchronize(j->st));
  CU(cudaGetLastError());
  take_small(j, h, files, frs);
  return B200C_OK;
}
// read_small() and then the error word the kernels raised: the checked synchronisation point between two stages
int checked_sync(b200c_job* j, uint64_t* h, const FileRec* files = nullptr, std::vector<FileRec>* frs = nullptr) {
  if (int rc = read_small(j, h, files, frs)) return rc;
  return map_dev_err((uint32_t)h[kSlotErr]);
}

// the tails of the outputs (properties, metaindex, footer) and their metas: built on the host, written into the images by one launch.
// pin_tails (4096 bytes per file) and pin_small (the TailCopy records) are reserved by encode_stage before the emit kernel starts.
int write_tails(b200c_job* j, const std::vector<FileRec>& frs, const std::vector<uint64_t>& base_off) {
  const b200c_params& P = j->p;
  const uint32_t nfiles = (uint32_t)frs.size();
  j->outputs.resize(nfiles);
  std::vector<TailCopy> tcs(nfiles);
  for (uint32_t f = 0; f < nfiles; f++) {
    const FileRec& fr = frs[f];
    OutputTailInput ti;
    ti.checksum_type = P.checksum;
    ti.format_version = P.format_version;
    ti.data_size = fr.data_size;
    ti.index_size = fr.index_size;
    ti.filter_size = fr.filter_len();
    ti.filter_entries = fr.filter_entries;
    ti.num_entries = fr.n_entries;
    ti.num_deletions = fr.num_deletions;
    ti.raw_key_size = fr.raw_key_size;
    ti.raw_value_size = fr.raw_value_size;
    ti.num_data_blocks = fr.n_blocks;
    ti.index_key_is_user_key = fr.index_key_is_user_key(P.format_version);
    ti.column_family_id = P.column_family_id;
    ti.column_family_name = j->cf_name;
    ti.db_id = j->db_id;
    ti.db_session_id = j->db_session_id;
    ti.db_host_id = j->db_host_id;
    ti.creation_time = P.creation_time;
    ti.oldest_key_time = P.oldest_key_time;
    ti.file_creation_time = j->fct.empty() ? 0 : j->fct[std::min<size_t>(f, j->fct.size() - 1)];
    ti.orig_file_number = P.first_file_number + f;
    std::vector<uint8_t> tail = build_output_tail(ti);
    const uint64_t tail_off = fr.tail_start();
    if (tail_off + tail.size() > base_off[f + 1] - base_off[f]) return fail(B200C_ERR_CUDA, "internal: output image overflow");
    const size_t so = (size_t)f * 4096;
    if (tail.size() > 4096) return fail(B200C_ERR_CUDA, "internal: tail larger than its staging slot");
    memcpy(j->pin_tails.p + so, tail.data(), tail.size());
    tcs[f] = TailCopy{base_off[f] + tail_off, (uint32_t)so, (uint32_t)tail.size()};
    Output& o = j->outputs[f];
    memset(&o.meta, 0, sizeof o.meta);
    o.dev_off = base_off[f];
    o.meta.file_number = ti.orig_file_number;
    o.meta.file_size = tail_off + tail.size();
    o.meta.smallest_seqno = fr.smallest_seq;
    o.meta.largest_seqno = fr.largest_seq;
    o.meta.num_entries = fr.n_entries;
    o.meta.num_deletions = fr.num_deletions;
    o.meta.raw_key_size = fr.raw_key_size;
    o.meta.raw_value_size = fr.raw_value_size;
    o.meta.num_data_blocks = fr.n_blocks;
    o.meta.data_size = fr.data_size;
    o.meta.index_size = fr.index_size;
    ikey_bytes(fr.smallest, o.meta.smallest_ikey, &o.meta.smallest_ikey_len);
    ikey_bytes(fr.largest, o.meta.largest_ikey, &o.meta.largest_ikey_len);
    j->stats.total_output_bytes += o.meta.file_size;
  }
  // all tails with one scatter launch
  const size_t rec_bytes = sizeof(TailCopy) * nfiles;
  memcpy(j->pin_small.p, tcs.data(), rec_bytes);
  // the scatter kernel reads records and bytes straight from mapped pinned memory: no copy-engine queue involved
  launch_scatter_tails(reinterpret_cast<const TailCopy*>(j->pin_small.p), nfiles, j->pin_tails.p, j->out_buf.as<uint8_t>(), j->st);
  j->launches++;
  return B200C_OK;
}

// CompactionParams::paranoid_file_checks (compaction_job.cc:829-853): read every finished output back -- the decoder verifies each
// block checksum -- and compare the entries with what the encoder was given.  The input columns of the merge are free by now and
// hold the re-read entries.
int paranoid_reread(b200c_job* j, KeyCols mcols, const std::vector<FileRec>& frs, const std::vector<uint64_t>& base_off) {
  const b200c_params& P = j->p;
  cudaStream_t st = j->st;
  const uint32_t nfiles = (uint32_t)frs.size();
  const uint64_t nblocks = j->nblocks_out, n_out = mcols.n;
  uint64_t* small = j->small.as<uint64_t>();
  uint32_t* err = reinterpret_cast<uint32_t*>(small + kSlotErr);
  std::vector<FileDesc> ofd(nfiles);
  uint32_t g = 0, maxb = 0;
  for (uint32_t f = 0; f < nfiles; f++) {
    const FileRec& fr = frs[f];
    FileDesc d;
    memset(&d, 0, sizeof d);
    d.base = j->out_buf.as<uint8_t>() + base_off[f];
    d.len = j->outputs[f].meta.file_size;
    d.index_off = fr.index_start();
    d.index_size = (uint32_t)fr.index_size;
    d.value_delta = P.format_version >= 4;
    d.cksum = P.checksum;
    d.gblk_first = g;
    d.nblocks = (uint32_t)fr.n_blocks;
    d.index_user_key = fr.index_key_is_user_key(P.format_version) ? 1u : 0u;
    g += d.nblocks;
    maxb = std::max(maxb, d.nblocks);
    ofd[f] = d;
  }
  if (g != nblocks) return fail(B200C_ERR_CUDA, "internal: block count of the outputs changed");
  CU(j->vfiles_d.reserve(sizeof(FileDesc) * nfiles));
  if (int rc = upload_small(j, j->vfiles_d.p, ofd.data(), sizeof(FileDesc) * nfiles)) return rc;
  CU(cudaStreamSynchronize(st));  // ofd is a temporary
  CU(j->blk_off.reserve(8 * (nblocks + 1)));
  CU(j->blk_size.reserve(4 * (nblocks + 1)));
  CU(j->blk_state.reserve(8 * (nblocks + 1)));
  CU(j->vrun_start.reserve(8 * ((size_t)nfiles + 1)));
  CU(j->dec.reserve(n_out));
  if (const char* flip = getenv("B200C_TEST_FLIP_OUTPUT_BYTE")) {  // test hook: damage file 0 before it is read back
    const uint64_t at = strtoull(flip, nullptr, 10);
    if (at < j->outputs[0].meta.file_size) launch_flip_byte(j->out_buf.as<uint8_t>() + base_off[0] + at, st);
  }
  CU(cudaMemsetAsync(small + kSlotDecTicket, 0, 8, st));
  CU(cudaMemsetAsync(small + kSlotTotalIn, 0, 8, st));
  CU(cudaMemsetAsync(j->vrun_start.p, 0, 8 * ((size_t)nfiles + 1), st));
  CU(cudaMemsetAsync(j->blk_state.p, 0, 8 * (nblocks + 1), st));
  const FileDesc* vf = j->vfiles_d.as<FileDesc>();
  j->kt_begin("verify.reread");
  launch_index_decode(vf, (int)nfiles, maxb, j->blk_off.as<uint64_t>(), j->blk_size.as<uint32_t>(), BoundKey{}, 0, BoundKey{}, 0, err, st,
                      &j->launches);
  launch_block_decode_fused(vf, (int)nfiles, j->blk_off.as<uint64_t>(), j->blk_size.as<uint32_t>(), (uint32_t)nblocks, 1, n_out, j->dec.mut(),
                            j->blk_state.as<unsigned long long>(), reinterpret_cast<uint32_t*>(small + kSlotDecTicket),
                            j->vrun_start.as<uint64_t>(), small + kSlotTotalIn, err, j->sms, st, &j->launches);
  launch_compare_columns(mcols, j->dec.cols(n_out), n_out, err, j->sms, st, &j->launches);
  j->kt_end();
  uint64_t hv[kSmallSlots];
  if (int rc = read_small(j, hv)) return rc;
  if ((uint32_t)hv[kSlotErr] & ~(uint32_t)kFlagHasSingleDelete) {  // whatever the reader tripped over, the file is not what was written
    map_dev_err((uint32_t)hv[kSlotErr]);
    const std::string detail = g_err;
    return fail(B200C_ERR_CORRUPTION, "Paranoid checksums do not match: " + detail);
  }
  if (hv[kSlotTotalIn] != n_out) return fail(B200C_ERR_CORRUPTION, "Paranoid checksums do not match (entry count of the outputs)");
  return B200C_OK;
}

// First XXH3 contribution slot (8 u64 per full 1024-byte block) of every file's index block, at [f], and filter block, at
// [nfiles + f], in one scratch; the total behind them.  The two blocks of a file are checksummed concurrently on two streams: their
// regions do not overlap.  The index block is sized by its bound: its length is not known yet.
static std::vector<uint64_t> file_block_contrib_offsets(const std::vector<FileRec>& frs) {
  const size_t n = frs.size();
  std::vector<uint64_t> off(2 * n + 1, 0);
  for (size_t i = 0; i < 2 * n; i++) off[i + 1] = off[i] + (i < n ? frs[i].index_bound() : frs[i - n].filter_len()) / 1024 + 1;
  return off;
}

int encode_stage(b200c_job* j, KeyCols mcols, uint64_t n_out, uint32_t min_s1, uint32_t max_s1, EncodeWork& W, uint32_t* err, uint64_t* small) {
  const b200c_params& P = j->p;
  cudaStream_t st = j->st;
  uint64_t h[kSmallSlots];
  std::vector<FileRec> frs;
  std::vector<uint64_t> base_off;
  if (n_out) {
    if (P.index_block_restart_interval != 1)
      return fail(B200C_ERR_NOT_SUPPORTED, "index_block_restart_interval != 1 is not built on the device");
    EncodeParams ep{};
    ep.block_size = P.block_size;
    ep.block_size_limit = P.block_size_deviation ? (uint32_t)(((uint64_t)P.block_size * (100 - P.block_size_deviation) + 99) / 100) : 0;
    ep.restart_interval = P.block_restart_interval;
    ep.checksum = P.checksum;
    ep.format_version = P.format_version;
    ep.output_level = (uint32_t)P.output_level;
    ep.max_output_file_size = P.max_output_file_size;
    // L0 outputs are never cut by grandparents or a partitioner (compaction_outputs.cc:247-253, :793-795)
    const uint32_t G = P.output_level > 0 ? (uint32_t)j->gp_small.size() : 0;
    const uint32_t plen = P.output_level > 0 ? P.sst_partitioner_prefix_len : 0;
    if (G) {
      // grandparent boundaries -> ranks in the merged stream; the cut rules themselves run inside the stitch kernel
      CU(j->gp_keys_d.reserve(sizeof(GpKey) * 2 * G));
      CU(j->gp_ranks_d.reserve(8 * 3 * (size_t)G));
      CU(j->gp_size_d.reserve(8 * (size_t)G));
      CU(j->gp_same_d.reserve(G + 16));
      GpKey* keys = j->gp_keys_d.as<GpKey>();
      if (int rc = upload_small(j, keys, j->gp_small.data(), sizeof(GpKey) * G)) return rc;
      if (int rc = upload_small(j, keys + G, j->gp_large.data(), sizeof(GpKey) * G)) return rc;
      if (int rc = upload_small(j, j->gp_size_d.p, j->gp_size.data(), 8 * (size_t)G)) return rc;
      if (int rc = upload_small(j, j->gp_same_d.p, j->gp_same.data(), G)) return rc;
      uint64_t* ranks = j->gp_ranks_d.as<uint64_t>();
      launch_gp_ranks(mcols, keys, keys + G, G, ranks, ranks + G, ranks + 2 * G, st, &j->launches);
      ep.gp.n = G;
      ep.gp.dynamic_file_size = P.level_compaction_dynamic_file_size;
      ep.gp.lo = ranks;
      ep.gp.eq = ranks + G;
      ep.gp.hi = ranks + 2 * G;
      ep.gp.size = j->gp_size_d.as<uint64_t>();
      ep.gp.next_same = j->gp_same_d.as<uint8_t>();
      ep.gp.target_output_file_size = P.target_output_file_size ? P.target_output_file_size : P.max_output_file_size;
      ep.gp.max_compaction_bytes = P.max_compaction_bytes ? P.max_compaction_bytes : ep.gp.target_output_file_size * 25;
    }
    if (plen) {
      // the partition events as a sorted entry list: k events make k + 1 files, so kMaxOutFiles - 1 of them fill the file records
      const uint32_t cap = kMaxOutFiles - 1;
      const uint64_t ptiles = partition_event_tiles(n_out);
      CU(j->pev_d.reserve(8 * ((size_t)cap + 1 + ptiles)));
      uint64_t* pev = j->pev_d.as<uint64_t>();  // events [cap] | look-back ticket | look-back state [ptiles]
      CU(cudaMemsetAsync(pev, 0xff, 8 * (size_t)cap, st));
      CU(cudaMemsetAsync(pev + cap, 0, 8 * (1 + ptiles), st));
      j->kt_begin("encode.partition_events");
      launch_partition_events(mcols, plen, cap, reinterpret_cast<uint32_t*>(pev + cap), reinterpret_cast<unsigned long long*>(pev + cap + 1),
                              pev, err, st, &j->launches);
      j->kt_end();
      ep.gp.pev = pev;
      ep.gp.np = cap;
    }
    if (G || plen) {  // every cut the stitch walk makes by these rules, for the block-list kernel: at most two per grandparent + the events
      CU(j->gp_cuts_d.reserve(sizeof(GpCut) * (2 * (size_t)G + 2 + ep.gp.np)));
      ep.gp_cuts = j->gp_cuts_d.as<GpCut>();
      ep.gp_ncuts = reinterpret_cast<uint32_t*>(small + kSlotGpCuts);
    }
    uint64_t hop = (uint64_t)(P.block_size - 1) / std::max<uint32_t>(min_s1, 1) + 3;
    if (hop > (uint64_t)kEncHalo) return fail(B200C_ERR_NOT_SUPPORTED, "block_size / smallest entry exceeds the encoder's 2048-entry block window");
    const uint32_t hc = (uint32_t)hop;
    const uint64_t etiles = (n_out + kEncTile - 1) / kEncTile;
    CU(j->rows.reserve(sizeof(TileRow) * etiles * hc));
    CU(j->tstate.reserve(sizeof(TileState) * etiles));
    const uint64_t egroups = (etiles + kEncGroupTiles - 1) / kEncGroupTiles;
    CU(j->grows.reserve(sizeof(TileRow) * egroups * hc));
    CU(j->gstate.reserve(sizeof(TileState) * egroups));
    CU(j->gflag.reserve(4 * egroups));
    CU(j->nxt.reserve(2 * (n_out + 1)));
    CU(j->disk.reserve(4 * (n_out + 1)));
    CU(j->files_rec.reserve(sizeof(FileRec) * (kMaxOutFiles + 2)));
    W.rows = j->rows.as<TileRow>();
    W.tstate = j->tstate.as<TileState>();
    W.grows = j->grows.as<TileRow>();
    W.gstate = j->gstate.as<TileState>();
    W.gflag = j->gflag.as<uint32_t>();
    W.nxt = j->nxt.as<uint16_t>();
    W.disk = j->disk.as<uint32_t>();
    W.files = j->files_rec.as<FileRec>();
    W.scan_tmp = j->scan_tmp.as<uint64_t>();
    CU(j->gsync.reserve(8 * egroups + 16));
    CU(cudaMemsetAsync(j->gsync.p, 0, 8 * egroups + 16, st));
    W.gdone = j->gsync.as<uint32_t>();
    W.gready = W.gdone + egroups;
    // The serial stitch walk runs on the side stream WHILE the tables kernel fills the tile / group rows: each group raises a flag
    // when its rows are complete and the walk waits on the flags.  It is launched twice, in front of the tables kernel (so that it
    // gets an SM to itself) and behind it (for tools that serialise kernels: ncu, compute-sanitizer) -- see encode_stitch_kernel.
    uint32_t* sflag = reinterpret_cast<uint32_t*>(small + kSlotStitchDone);
    CU(cudaEventRecord(j->evx[0], st));
    CU(cudaStreamWaitEvent(j->st2, j->evx[0], 0));
    {
      const size_t slot = j->kt_begin("~encode.stitch", j->st2);
      launch_encode_stitch(mcols, ep, W, etiles, hc, err, 1, sflag, j->st2, &j->launches);
      j->kt_end(slot, j->st2);
    }
    j->kt_begin("encode.tables");
    launch_encode_tables(mcols, ep, W, etiles, hc, max_s1, st, &j->launches);
    j->kt_end();
    {
      const size_t slot = j->kt_begin("~encode.stitch_retry", j->st2);
      launch_encode_stitch(mcols, ep, W, etiles, hc, err, 2, sflag, j->st2, &j->launches);
      j->kt_end(slot, j->st2);
    }
    CU(cudaEventRecord(j->evx[1], j->st2));
    CU(cudaStreamWaitEvent(st, j->evx[1], 0));
    j->kt_begin("encode.tilestate");
    launch_encode_tilestate(mcols, W, etiles, hc, err, st, &j->launches);
    j->kt_end();
    if (P.bloom_millibits_per_key) {  // filter entries per file decide where each file's index block starts
      j->kt_begin("encode.bloom_count");
      CU(j->bloom_hashes.reserve(8 * (n_out + 1)));  // XXPH3 of every output key: computed once, read by the slices of the filter build
      launch_bloom_count(mcols, n_out, W.files, small + kSlotTotals + 1, P.bloom_millibits_per_key, j->bloom_hashes.as<uint64_t>(), j->sms, st,
                         &j->launches);
      j->kt_end();
    }
    if (int rc = checked_sync(j, h, W.files, &frs)) return rc;  // sync #2: number of blocks / files, per-file records
    const uint64_t nblocks = j->nblocks_out = h[kSlotTotals];
    const uint32_t nfiles = j->nfiles_out = (uint32_t)h[kSlotTotals + 1];
    if (nfiles == 0 || nfiles > kMaxOutFiles) return fail(B200C_ERR_CUDA, "internal: bad output file count");
    CU(j->blocks.reserve(sizeof(BlockRec) * (nblocks + 1)));
    CU(j->idx_esz.reserve(4 * (nblocks + 1)));
    CU(j->idx_eoff.reserve(8 * (nblocks + 1)));
    CU(j->idx_sep.reserve(sizeof(KeyRec) * (nblocks + 1)));
    W.blocks = j->blocks.as<BlockRec>();
    W.idx_esz = j->idx_esz.as<uint32_t>();
    W.idx_eoff = j->idx_eoff.as<uint64_t>();
    W.idx_sep = j->idx_sep.as<KeyRec>();
    // write_tails' pinned staging, reserved here: it runs while the emit kernel does, and a page-locked allocation would
    // synchronise the device
    CU(j->pin_tails.reserve((size_t)nfiles * 4096 + 64));
    CU(j->pin_small.reserve(sizeof(TailCopy) * nfiles));
    base_off.resize(nfiles + 1);
    uint64_t off = 0;
    for (uint32_t f = 0; f < nfiles; f++) {
      base_off[f] = off;
      off += (frs[f].image_bound(4096) + 255) & ~255ull;  // the tail is at most 4096 bytes (write_tails)
    }
    base_off[nfiles] = off;
    CU(j->out_buf.reserve(off + 256));
    {  // scratch for the parallel part of the index and filter blocks' checksums
      const std::vector<uint64_t> coff = file_block_contrib_offsets(frs);
      CU(j->cksum_contrib.reserve(64 * (coff.back() + 1)));
      CU(j->cksum_contrib_off.reserve(8 * coff.size()));
      if (int rc = upload_small(j, j->cksum_contrib_off.p, coff.data(), 8 * coff.size())) return rc;  // (copied into pinned staging)
      W.cksum_contrib = j->cksum_contrib.as<uint64_t>();
      W.cksum_contrib_off = j->cksum_contrib_off.as<uint64_t>();
    }
    std::vector<uint8_t*> bases(nfiles);
    for (uint32_t f = 0; f < nfiles; f++) bases[f] = j->out_buf.as<uint8_t>() + base_off[f];
    CU(j->out_base_d.reserve(8 * nfiles));
    if (int rc = upload_small(j, j->out_base_d.p, bases.data(), 8 * nfiles)) return rc;
    uint8_t* const* out_base_d = j->out_base_d.as<uint8_t*>();
    j->kt_begin("encode.blocklist");
    launch_encode_blocklist(mcols, ep, W, etiles, nblocks, err, st, &j->launches);
    j->kt_end();
    // The file tails (write_tails) need only the per-file records: statistics, boundary keys, index-block sizes.  Those kernels
    // run on the main stream in front of the emit kernel (behind it they would wait for its last CTA, see
    // launch_encode_emit); the records are gathered right behind them, and the host builds the tails while the data blocks are emitted.
    j->kt_begin("encode.filestats+index_size");
    launch_encode_index_size(mcols, ep, W, nblocks, j->sms, st, &j->launches);
    launch_encode_filestats(mcols, W, nfiles, st, &j->launches);
    j->kt_end();
    if (int rc = gather_small(j, W.files)) return rc;
    CU(cudaEventRecord(j->evx[2], st));
    uint64_t data_bytes = 0;
    for (uint32_t f = 0; f < nfiles; f++) data_bytes += frs[f].data_size;
    j->kt_begin("encode.emit");
    launch_encode_emit(mcols, ep, W, nblocks, out_base_d, data_bytes, j->sms, st, &j->launches);
    j->kt_end();
    // The index blocks are written on the side stream beside the emit kernel (a file's index block lies behind its data and filter
    // blocks: disjoint bytes).  They are enqueued after the emit so that the main stream does not idle while the host enqueues them.
    CU(cudaStreamWaitEvent(j->st2, j->evx[2], 0));
    {
      const size_t slot = j->kt_begin("~encode.index", j->st2);
      launch_encode_index_write(ep, W, nblocks, nfiles, out_base_d, j->sms, j->st2, &j->launches);
      j->kt_end(slot, j->st2);
    }
    CU(cudaEventRecord(j->evx[3], j->st2));
    if (P.bloom_millibits_per_key) {
      j->kt_begin("encode.bloom_build");
      uint64_t max_fb = 0;
      for (uint32_t f = 0; f < nfiles; f++) max_fb = std::max<uint64_t>(max_fb, frs[f].filter_bytes);
      launch_bloom_build(j->bloom_hashes.as<uint64_t>(), n_out, W, nfiles, (uint32_t)std::min<uint64_t>(max_fb, 0xffffffffull), P.bloom_millibits_per_key,
                         P.checksum, out_base_d, st, &j->launches);
      j->kt_end();
    }
    // sync #3 waits for the records gathered in front of the emit kernel only.  The error word the emit, index and filter kernels
    // may still raise is checked by finish_run().
    CU(cudaEventSynchronize(j->evx[2]));
    CU(cudaGetLastError());
    take_small(j, h, W.files, &frs);
    CU(cudaStreamWaitEvent(st, j->evx[3], 0));
    int rc = map_dev_err((uint32_t)h[kSlotErr]);
    if (rc == B200C_OK && frs.size() != nfiles) rc = fail(B200C_ERR_CUDA, "internal: output file count changed");
    if (rc == B200C_OK) rc = write_tails(j, frs, base_off);
    if (rc != B200C_OK) {  // the emit, filter and index kernels may still read the columns (caller-owned on the TableBuilder path)
      cudaStreamSynchronize(st);  // (st waits for the side stream's index kernels)
      return rc;
    }
    if (P.paranoid_file_checks) {
      if (int rc = checked_sync(j, h)) return rc;  // an encoder error keeps its own status instead of the re-read's Corruption
      return paranoid_reread(j, mcols, frs, base_off);
    }
  }
  return B200C_OK;
}

// D2H of the finished images (host outputs), event times, bookkeeping
int finish_run(b200c_job* j) {
  const b200c_params& P = j->p;
  cudaStream_t st = j->st;
  CU(cudaEventRecord(j->ev[3], st));
  if (P.output_mem == B200C_MEM_HOST) {
    uint64_t tot = 0;
    for (auto& o : j->outputs) {
      o.host_off = tot;
      tot += (o.meta.file_size + 63) & ~63ull;
    }
    CU(j->host_out.reserve(tot + 64));
    for (auto& o : j->outputs)
      CU(cudaMemcpyAsync(j->host_out.p + o.host_off, j->out_buf.as<uint8_t>() + o.dev_off, o.meta.file_size, cudaMemcpyDeviceToHost, st));
  }
  CU(cudaEventRecord(j->ev[4], st));
  {  // the run's last checked synchronisation: errors the emit, index and filter kernels raised after sync #3
    uint64_t h[kSmallSlots];
    if (int rc = checked_sync(j, h)) return rc;
  }
  float ms;
  cudaEventElapsedTime(&ms, j->ev[0], j->ev[1]);
  j->stats.decode_us = ms * 1000.0;
  cudaEventElapsedTime(&ms, j->ev[1], j->ev[2]);
  j->stats.merge_us = ms * 1000.0;
  cudaEventElapsedTime(&ms, j->ev[2], j->ev[3]);
  j->stats.encode_us = ms * 1000.0;
  cudaEventElapsedTime(&ms, j->ev[0], j->ev[4]);
  j->stats.total_us = ms * 1000.0;
  for (size_t i = 0; i < j->kt_used; i++) {
    float kms = 0;
    cudaEventElapsedTime(&kms, j->ktimes[i].a, j->ktimes[i].b);
    j->ktimes[i].us = kms * 1000.f;
  }
  j->stats.num_output_files = j->nfiles_out;
  j->stats.kernel_launches = j->launches;
  j->stage_done = 3;
  return B200C_OK;
}

int encode_columns(b200c_job* j, uint64_t n, const void* pfx, const void* tr, const void* vref, const void* meta, bool prepared = false);

int run_merge_encode(b200c_job* j, int until, KeyCols decc, RunBounds runs, uint64_t n_decoded, uint64_t N, bool clipped,
                     uint64_t range_value_bytes, uint64_t* small, uint32_t* err);

// The job's device, streams and events (made on first use).  A sub-job of a range-pipelined parent: st waits for the uploads of its
// part of the inputs before anything reads them.
int job_bind(b200c_job* j) {
  CU(cudaSetDevice(j->p.device));
  if (!j->st) {
    CU(cudaStreamCreateWithFlags(&j->st, cudaStreamNonBlocking));
    int prio_lo = 0, prio_hi = 0;
    CU(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
    CU(cudaStreamCreateWithPriority(&j->st2, cudaStreamNonBlocking, prio_hi));
    for (auto& e : j->ev) CU(cudaEventCreate(&e));
    for (auto& e : j->evx) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    CU(cudaDeviceGetAttribute(&j->sms, cudaDevAttrMultiProcessorCount, j->p.device));
  }
  if (j->wait_ev) CU(cudaStreamWaitEvent(j->st, j->wait_ev, 0));
  return B200C_OK;
}

int job_prepare(b200c_job* j) {
  if (int rc = job_bind(j)) return rc;
  j->outputs.clear();
  j->stage_done = 0;
  j->launches = 0;
  j->nblocks_out = 0;
  j->nfiles_out = 0;
  j->kt_used = 0;
  j->pin_up_used = 0;
  memset(&j->stats, 0, sizeof j->stats);
  return B200C_OK;
}

int run_job(b200c_job* j, int until) {
  const b200c_params& P = j->p;
  if (int rc = job_prepare(j)) return rc;
  cudaStream_t st = j->st;
  const int k = (int)j->inputs.size();
  if (k == 0) return fail(B200C_ERR_INVALID_ARGUMENT, "job has no inputs");

  // ---------------- inputs: resident image + tail
  CU(cudaEventRecord(j->ev[0], st));
  uint64_t nblk = 0, n_props = 0, in_bytes = 0;
  bool any_compressed = false;
  std::vector<FileDesc> fds(k);
  {  // tails of device-resident inputs: one batch of small D2H copies and a single synchronisation
    bool any_dev = false;
    for (int i = 0; i < k; i++) any_dev = any_dev || j->inputs[i].mem_kind != B200C_MEM_HOST;
    if (any_dev) {
      CU(j->pin_small.reserve((size_t)k * kTailFetch));
      for (int i = 0; i < k; i++) {
        const Input& in = j->inputs[i];
        if (in.mem_kind == B200C_MEM_HOST || in.len < 53) continue;
        const uint64_t tn = std::min<uint64_t>(in.len, kTailFetch);
        CU(cudaMemcpyAsync(j->pin_small.p + (size_t)i * kTailFetch, in.data + in.len - tn, tn, cudaMemcpyDeviceToHost, st));
      }
      CU(cudaStreamSynchronize(st));
    }
  }
  for (int i = 0; i < k; i++) {
    Input& in = j->inputs[i];
    const bool host = in.mem_kind == B200C_MEM_HOST;
    if (int rc = open_input(j, in, host ? nullptr : j->pin_small.p + (size_t)i * kTailFetch)) return rc;
    if (host) {  // b200c_job_add_input's eager copy once (it overlapped the caller's file reads), else a new one
      if (int rc = stage_input(in, st, in.copy.fresh)) return rc;
      in.copy.fresh = false;
    }
    FileDesc& fd = fds[i];
    fd.base = host ? in.copy.buf.as<uint8_t>() : in.data;
    fd.len = in.len;
    fd.index_off = in.tail.index_off;
    fd.index_size = (uint32_t)in.tail.index_size;
    fd.value_delta = in.tail.format_version >= 4;
    fd.cksum = in.tail.checksum_type;
    fd.gblk_first = (uint32_t)nblk;
    fd.nblocks = (uint32_t)in.tail.num_data_blocks;
    fd.index_user_key = in.tail.index_key_is_user_key ? 1u : 0u;  // (index_ptr: the vector zeroed it)
    if (input_is_compressed(in)) any_compressed = true;  // kZlibCompression: data blocks are inflated on the device, the index block below
    nblk += in.tail.num_data_blocks;
    n_props += in.tail.num_entries;
    in_bytes += in.len;
  }
  if (any_compressed) {
    // compressed index blocks: inflated on the host, one thread per file (a 256 MiB file has ~3.5 MB of index: ~17 ms on one core)
    std::vector<int> rcs(k, B200C_OK);
    std::vector<std::string> msgs(k);
    std::vector<std::thread> pool;
    for (int i = 0; i < k; i++) {
      if (!input_is_compressed(j->inputs[i])) continue;
      pool.emplace_back([&, i]() {
        cudaSetDevice(P.device);
        rcs[i] = input_index_block(j, j->inputs[i], &j->inputs[i].index);
        if (rcs[i]) msgs[i] = g_err;  // (the message is per thread)
      });
    }
    for (auto& th : pool) th.join();
    for (int i = 0; i < k; i++) {
      if (rcs[i]) return fail(rcs[i], msgs[i]);
      Input& in = j->inputs[i];
      if (!input_is_compressed(in) || !in.index.inflated) continue;
      CU(in.index_inflated.reserve(in.index.len + 64));
      CU(cudaMemcpyAsync(in.index_inflated.p, in.index.p, in.index.len, cudaMemcpyHostToDevice, st));
      fds[i].index_ptr = in.index_inflated.as<uint8_t>();
      fds[i].index_size = (uint32_t)in.index.len;
    }
  }
  if (nblk > 0xfffffff0ull) return fail(B200C_ERR_NOT_SUPPORTED, "too many data blocks");
  j->nblk_in = nblk;
  j->n_total = n_props;
  j->stats.num_input_files = k;
  j->stats.total_input_bytes = in_bytes;
  j->stats.num_input_records = n_props;

  CU(j->small.reserve(kSmallSlots * 8));
  CU(cudaMemsetAsync(j->small.p, 0, kSmallSlots * 8, st));
  uint64_t* small = j->small.as<uint64_t>();
  uint32_t* err = reinterpret_cast<uint32_t*>(small + kSlotErr);
  {
    uint32_t ff = 0xffffffffu;
    if (int rc = upload_small(j, small + kSlotMinS1, &ff, 4)) return rc;
  }
  CU(j->files_d.reserve(sizeof(FileDesc) * k));
  if (int rc = upload_small(j, j->files_d.p, fds.data(), sizeof(FileDesc) * k)) return rc;
  const uint64_t N = n_props;
  CU(j->blk_off.reserve(8 * (nblk + 1)));
  CU(j->blk_size.reserve(4 * (nblk + 1)));
  CU(j->blk_state.reserve(8 * (nblk + 1)));
  CU(j->scan_tmp.reserve(8 * ((std::max<uint64_t>(nblk, N) / kScanTile) + 2)));
  CU(j->run_start.reserve(8 * (k + 1)));
  CU(j->dec.reserve(N));
  const FileDesc* files_d = j->files_d.as<FileDesc>();

  // ---------------- decode
  uint32_t maxb = 0;
  for (auto& f : fds) maxb = std::max(maxb, f.nblocks);
  if (nblk) {
    j->kt_begin("decode.index");
    // a sub-compaction's key range: data blocks that cannot hold a key of [start, end) are dropped here, before anything of them is read
    launch_index_decode(files_d, k, maxb, j->blk_off.as<uint64_t>(), j->blk_size.as<uint32_t>(), j->range_lo, P.has_range_start, j->range_hi,
                        P.has_range_end, err, st, &j->launches);
    j->kt_end();
  }
  const uint8_t* arena = nullptr;
  if (nblk && any_compressed) {
    // compressed data blocks -> the arena of inflated blocks; their handles are redirected there (decode.cu)
    CU(j->cslot.reserve(4 * (nblk + 1)));
    CU(j->cslot_off.reserve(8 * (nblk + 1)));
    j->kt_begin("decode.inflate");
    launch_block_usize(files_d, j->blk_off.as<uint64_t>(), j->blk_size.as<uint32_t>(), (uint32_t)nblk, j->cslot.as<uint32_t>(), err, st, &j->launches);
    exclusive_scan<uint32_t>(j->cslot.as<uint32_t>(), j->cslot_off.as<uint64_t>(), nblk, j->scan_tmp.as<uint64_t>(), small + kSlotArena, st, &j->launches);
    uint64_t hc[kSmallSlots];
    if (int rc = checked_sync(j, hc)) return rc;  // sync: the arena is sized by what the blocks announce
    CU(j->arena.reserve(hc[kSlotArena] + 256));
    arena = j->arena.as<uint8_t>();
    launch_inflate_blocks(files_d, j->blk_off.as<uint64_t>(), j->blk_size.as<uint32_t>(), j->cslot.as<uint32_t>(), j->cslot_off.as<uint64_t>(),
                          (uint32_t)nblk, j->arena.as<uint8_t>(), P.verify_input_checksums, err, j->sms, st, &j->launches);
    j->kt_end();
  }
  CU(cudaMemsetAsync(j->run_start.p, 0, 8 * (k + 1), st));  // stays zero when there is no data block at all
  if (nblk) {
    CU(cudaMemsetAsync(j->blk_state.p, 0, 8 * (nblk + 1), st));
    j->kt_begin("decode.blocks");
    launch_block_decode_fused(files_d, k, j->blk_off.as<uint64_t>(), j->blk_size.as<uint32_t>(), (uint32_t)nblk, P.verify_input_checksums, N,
                              j->dec.mut(), j->blk_state.as<unsigned long long>(), reinterpret_cast<uint32_t*>(small + kSlotDecTicket),
                              j->run_start.as<uint64_t>(), small + kSlotTotalIn, err, j->sms, st, &j->launches, arena);
    j->kt_end();
  }
  CU(cudaEventRecord(j->ev[1], st));
  const KeyCols decc = j->dec.cols(N);
  if (until == 1) {
    uint64_t h[kSmallSlots];
    j->run_start_h.resize(k + 1);
    CU(cudaMemcpyAsync(j->run_start_h.data(), j->run_start.p, 8 * (k + 1), cudaMemcpyDeviceToHost, st));
    if (int rc = checked_sync(j, h)) return rc;
    if (h[kSlotTotalIn] != N && !(P.has_range_start || P.has_range_end))  // (a key range skips the blocks outside it)
      return fail(B200C_ERR_CORRUPTION, "decoded entry count differs from rocksdb.num.entries");
    j->stage_done = 1;
    j->stats.kernel_launches = j->launches;
    return B200C_OK;
  }

  // ---------------- runs: an L0 file is a run of its own, all files of a deeper level form ONE run (they are disjoint and ordered:
  // LevelIterator, db/version_set.cc:1076,7311-7352).  The files were decoded back to back, so a run is a range of the columns.
  std::vector<uint32_t> run_first;  // first file of every run, plus the file count
  for (int i = 0; i < k; i++)
    if (i == 0 || j->inputs[i].level <= 0 || j->inputs[i].level != j->inputs[i - 1].level) run_first.push_back((uint32_t)i);
  const uint32_t K = (uint32_t)run_first.size();
  run_first.push_back((uint32_t)k);
  if (K > (uint32_t)kMaxRuns) return fail(B200C_ERR_NOT_SUPPORTED, "more than 64 sorted runs (L0 files + levels)");
  j->nruns = K;
  CU(j->run_bounds.reserve(16 * (size_t)(K + 1)));
  CU(j->run_first_d.reserve(4 * (size_t)(K + 2)));
  if (int rc = upload_small(j, j->run_first_d.p, run_first.data(), 4 * (size_t)(K + 1))) return rc;
  launch_run_bounds(decc, j->run_start.as<uint64_t>(), j->run_first_d.as<uint32_t>(), K, j->run_bounds.as<uint64_t>(), err, st, &j->launches);
  RunBounds runs{j->run_bounds.as<uint64_t>(), j->run_bounds.as<uint64_t>() + K};
  // ---------------- sub-compaction key range: clip every run, the merge and everything behind it only see [start, end)
  const bool clipped = P.has_range_start || P.has_range_end;
  const uint64_t n_decoded = N;
  uint64_t N_in = N, range_value_bytes = 0;
  if (clipped) {
    CU(j->clip_d.reserve(16 * (size_t)(K + 1)));
    j->kt_begin("merge.clip");
    launch_clip_runs(decc, runs, K, j->range_lo, P.has_range_start, j->range_hi, P.has_range_end,
                     j->clip_d.as<uint64_t>(), reinterpret_cast<unsigned long long*>(small + kSlotClip), st, &j->launches);
    j->kt_end();
    uint64_t hc[kSmallSlots];
    if (int rc = checked_sync(j, hc)) return rc;  // sync: the merge grid depends on the number of entries in range
    N_in = hc[kSlotClip];
    range_value_bytes = hc[kSlotClip + 1];
    if (N_in > n_decoded) return fail(B200C_ERR_CUDA, "internal: clipped entry count exceeds the input");
    runs = RunBounds{j->clip_d.as<uint64_t>(), j->clip_d.as<uint64_t>() + K};
    j->stats.num_input_records = N_in;
  }
  return run_merge_encode(j, until, decc, runs, n_decoded, N_in, clipped, range_value_bytes, small, err);
}

// merge + encode over the (possibly clipped) runs; N = entries the merge consumes
int run_merge_encode(b200c_job* j, int until, KeyCols decc, RunBounds runs, uint64_t n_decoded, uint64_t N, bool clipped,
                     uint64_t range_value_bytes, uint64_t* small, uint32_t* err) {
  const b200c_params& P = j->p;
  cudaStream_t st = j->st;
  const size_t k = j->nruns;  // sorted runs (not files)
  // ---------------- merge
  const uint64_t mtiles = (N + kMergeNominal - 1) / kMergeNominal;  // tiles are cut every kMergeNominal entries (kernels.h)
  CU(j->splits.reserve(8 * (mtiles + 1) * k));
  CU(j->tile_state.reserve(8 * (mtiles + 1)));
  CU(cudaMemsetAsync(j->tile_state.p, 0, 8 * (mtiles + 1), st));
  CU(j->snaps_d.reserve(8 * (P.num_snapshots + 1)));
  if (P.num_snapshots)
    if (int rc = upload_small(j, j->snaps_d.p, j->snapshots.data(), 8 * P.num_snapshots)) return rc;
  CU(j->mrg.reserve(N));
  CU(j->esz.reserve(4 * (N + 1)));
  CU(j->eshared.reserve(N + 1));
  CU(j->tstat.reserve(sizeof(TileStat) * (mtiles + 2)));
  MergeParams mp;
  mp.nruns = (uint32_t)k;
  mp.bottommost = P.bottommost_level != 0;
  mp.nsnapshots = P.num_snapshots;
  mp.snapshots = j->snaps_d.as<uint64_t>();
  mp.earliest_snapshot = P.num_snapshots ? j->snapshots[0] : kMaxSeq;
  mp.filter = P.compaction_filter;
  mp.ttl = P.ttl;
  mp.now = P.ttl_now;
  mp.write_conflict_snapshot = P.earliest_write_conflict_snapshot != 0 && P.earliest_write_conflict_snapshot < kMaxSeq;
  MergeCounters* counters = reinterpret_cast<MergeCounters*>(small + kSlotCounters);
  EncodeWork W;
  memset(&W, 0, sizeof W);
  W.esz = j->esz.as<uint32_t>();
  W.eshared = j->eshared.as<uint8_t>();
  W.tstat = j->tstat.as<TileStat>();
  W.min_s1 = reinterpret_cast<uint32_t*>(small + kSlotMinS1);
  W.totals = small + kSlotTotals;
  if (N) {
    j->kt_begin("merge.partition");
    launch_merge_partition(decc, runs, (uint32_t)k, N, mtiles, j->splits.as<uint64_t>(), err, j->sms, st, &j->launches);
    j->kt_end();
    // the merge kernel also writes what the encoder needs per entry (encoded size, shared-prefix length) and per tile (statistics)
    const MergeSizes msz{W.esz, W.eshared, W.tstat, W.min_s1};
    W.tprefix = j->tile_state.as<unsigned long long>();
    W.nstat = mtiles;
    j->kt_begin("merge.tiles");
    launch_merge_tiles(decc, runs, mp, N, mtiles, j->splits.as<uint64_t>(),
                       j->tile_state.as<unsigned long long>(), reinterpret_cast<uint32_t*>(small + kSlotTicket), j->mrg.mut(), counters, msz, err, st,
                       &j->launches);
    j->kt_end();
    j->kt_begin("merge.sizes_fix");
    launch_merge_sizes_fix(j->mrg.cols(0), j->tile_state.as<unsigned long long>(), mtiles, msz, st, &j->launches);
    j->kt_end();
  }
  CU(cudaEventRecord(j->ev[2], st));
  uint64_t h[kSmallSlots];
  if (int rc = checked_sync(j, h)) return rc;  // sync #1: survivors, smallest entry, error word
  if (clipped ? h[kSlotTotalIn] > n_decoded : h[kSlotTotalIn] != n_decoded)  // (a key range skips the data blocks outside it)
    return fail(B200C_ERR_CORRUPTION, "decoded entry count differs from rocksdb.num.entries");
  MergeCounters mc;
  memcpy(&mc, h + kSlotCounters, sizeof mc);
  const uint64_t n_out = mc.n_out;
  j->n_out = n_out;
  j->stats.num_output_records = n_out;
  j->stats.num_input_deletion_records = mc.n_input_deletions;
  j->stats.num_records_replaced = mc.n_hidden;
  j->stats.num_expired_deletion_records = mc.n_obsolete;
  j->stats.num_record_drop_user = mc.n_user_drop;
  j->stats.total_input_raw_key_bytes = mc.raw_key_bytes;
  {  // every input value byte (rocksdb.raw.value.size of the inputs) minus the silently skipped entries
    uint64_t all = 0;
    for (auto& in : j->inputs) all += in.tail.raw_value_size;
    if (clipped) all = range_value_bytes;  // a sub-compaction counts what its clipped iterator consumed
    j->stats.total_input_raw_value_bytes = all - mc.raw_value_bytes;
  }
  if (until == 2) {
    j->stage_done = 2;
    j->stats.kernel_launches = j->launches;
    return B200C_OK;
  }

  // ---------------- encode
  if (int rc = encode_stage(j, j->mrg.cols(n_out), n_out, (uint32_t)h[kSlotMinS1], (uint32_t)(h[kSlotMinS1] >> 32), W, err, small)) return rc;
  return finish_run(j);
}

// TableBuilder side only: one sorted run given as device columns -> BlockBasedTable image(s)
int encode_columns(b200c_job* j, uint64_t n, const void* pfx, const void* tr, const void* vref, const void* meta, bool prepared) {
  int rc = prepared ? B200C_OK : job_prepare(j);
  if (rc) return rc;
  cudaStream_t st = j->st;
  CU(cudaEventRecord(j->ev[0], st));
  CU(cudaEventRecord(j->ev[1], st));
  CU(cudaEventRecord(j->ev[2], st));
  CU(j->small.reserve(kSmallSlots * 8));
  CU(cudaMemsetAsync(j->small.p, 0, kSmallSlots * 8, st));
  uint64_t* small = j->small.as<uint64_t>();
  uint32_t* err = reinterpret_cast<uint32_t*>(small + kSlotErr);
  uint32_t ff = 0xffffffffu;
  CU(cudaMemcpyAsync(small + kSlotMinS1, &ff, 4, cudaMemcpyHostToDevice, st));
  MergeCounters* counters = reinterpret_cast<MergeCounters*>(small + kSlotCounters);
  CU(cudaMemcpyAsync(&counters->n_out, &n, 8, cudaMemcpyHostToDevice, st));
  CU(j->esz.reserve(4 * (n + 1)));
  CU(j->eshared.reserve(n + 1));
  CU(j->tstat.reserve(sizeof(TileStat) * (n / kEncTile + 2)));
  CU(j->tile_state.reserve(8 * (n / kEncTile + 2)));
  CU(j->scan_tmp.reserve(8 * ((n / kScanTile) + 2)));
  EncodeWork W;
  memset(&W, 0, sizeof W);
  W.esz = j->esz.as<uint32_t>();
  W.eshared = j->eshared.as<uint8_t>();
  W.tstat = j->tstat.as<TileStat>();
  W.min_s1 = reinterpret_cast<uint32_t*>(small + kSlotMinS1);
  W.totals = small + kSlotTotals;
  KeyCols mcols{static_cast<const ulonglong2*>(pfx), static_cast<const uint64_t*>(tr), static_cast<const uint64_t*>(vref),
                static_cast<const uint32_t*>(meta), n};
  if (n) {
    j->kt_begin("encode.sizes");
    W.tprefix = j->tile_state.as<unsigned long long>();
    W.nstat = (n + kEncTile - 1) / kEncTile;
    launch_encode_sizes(mcols, reinterpret_cast<const unsigned long long*>(&counters->n_out), W, j->tile_state.as<unsigned long long>(), n, j->sms, st);
    j->kt_end();
    j->launches++;
  }
  uint64_t h[kSmallSlots];
  rc = checked_sync(j, h);
  if (rc) return rc;
  rc = encode_stage(j, mcols, n, (uint32_t)h[kSlotMinS1], (uint32_t)(h[kSlotMinS1] >> 32), W, err, small);
  if (rc) return rc;
  j->n_out = n;
  j->stats.num_output_records = n;
  return finish_run(j);
}

}  // namespace

extern "C" {

const char* b200c_last_error(void) { return g_err.c_str(); }
uint32_t b200c_abi_version(void) { return B200C_ABI_VERSION; }
int b200c_device_count(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) {
    cudaGetLastError();
    g_err = std::string("cudaGetDeviceCount: ") + cudaGetErrorString(e);
    return -B200C_ERR_NO_DEVICE;
  }
  return n;
}

void b200c_params_init(b200c_params* p) {
  memset(p, 0, sizeof *p);
  p->abi_version = B200C_ABI_VERSION;
  p->device = 0;
  p->output_level = 1;
  p->bottommost_level = 0;
  p->max_output_file_size = 64ull << 20;  // target_file_size_base, advanced_options.h:599
  p->block_size = 4096;
  p->block_size_deviation = 10;
  p->block_restart_interval = 16;
  p->index_block_restart_interval = 1;
  p->format_version = 5;
  p->checksum = B200C_CKSUM_XXH3;
  p->verify_input_checksums = 1;
  p->level_compaction_dynamic_file_size = 1;  // advanced_options.h (default true)
  p->column_family_name = "default";
  p->output_mem = B200C_MEM_HOST;
}

int b200c_job_create(const b200c_params* p, b200c_job** out) {
  if (!p || !out) return fail(B200C_ERR_INVALID_ARGUMENT, "null argument");
  if (p->abi_version != B200C_ABI_VERSION) return fail(B200C_ERR_INVALID_ARGUMENT, "ABI version mismatch");
  if (p->block_size < 64 || p->block_size > (1u << 20)) return fail(B200C_ERR_INVALID_ARGUMENT, "block_size out of range");
  if (p->block_restart_interval < 1) return fail(B200C_ERR_INVALID_ARGUMENT, "block_restart_interval < 1");
  if (p->block_size_deviation > 100) return fail(B200C_ERR_INVALID_ARGUMENT, "block_size_deviation > 100");
  if (p->format_version < 3 || p->format_version > 5) return fail(B200C_ERR_NOT_SUPPORTED, "output format_version must be 3..5");
  if (p->compaction_filter != B200C_FILTER_NONE && p->compaction_filter != B200C_FILTER_REMOVE_EMPTY_VALUE &&
      p->compaction_filter != B200C_FILTER_TTL)
    return fail(B200C_ERR_NOT_SUPPORTED, "compaction filter is not one of the built-in device filters");
  if (p->checksum != B200C_CKSUM_XXH3 && p->checksum != B200C_CKSUM_CRC32C && p->checksum != B200C_CKSUM_NONE)
    return fail(B200C_ERR_NOT_SUPPORTED, "output checksum must be kNoChecksum, kCRC32c or kXXH3");
  for (uint32_t i = 1; i < p->num_snapshots; i++)
    if (p->snapshots[i] <= p->snapshots[i - 1]) return fail(B200C_ERR_INVALID_ARGUMENT, "snapshots must be strictly ascending");
  int n = b200c_device_count();
  if (n <= 0) return fail(B200C_ERR_NO_DEVICE, "no CUDA device: the compaction path has no CPU implementation in this library");
  if (p->device < 0 || p->device >= n) return fail(B200C_ERR_INVALID_ARGUMENT, "device ordinal out of range");
  b200c_job* j = new b200c_job();
  j->p = *p;
  if (p->num_snapshots) j->snapshots.assign(p->snapshots, p->snapshots + p->num_snapshots);
  if (p->num_file_creation_times) j->fct.assign(p->file_creation_times, p->file_creation_times + p->num_file_creation_times);
  j->cf_name = p->column_family_name ? p->column_family_name : "";
  j->db_id = p->db_id ? p->db_id : "";
  j->db_session_id = p->db_session_id ? p->db_session_id : "";
  j->db_host_id = p->db_host_id ? p->db_host_id : "";
  j->p.snapshots = nullptr;
  j->p.file_creation_times = nullptr;
  // grandparents: user keys packed like the key columns (two big-endian words + length)
  auto pack = [](const void* key, uint32_t len, GpKey* k) {
    uint8_t b[16] = {0};
    if (len) memcpy(b, key, len);
    k->hi = k->lo = 0;
    for (int i = 0; i < 8; i++) k->hi = (k->hi << 8) | b[i], k->lo = (k->lo << 8) | b[8 + i];
    k->ulen = len;
    k->pad = 0;
  };
  for (uint32_t i = 0; i < p->num_grandparents; i++) {
    const b200c_grandparent& g = p->grandparents[i];
    if (g.smallest_len > kMaxUserKey || g.largest_len > kMaxUserKey || (!g.smallest_user_key && g.smallest_len) ||
        (!g.largest_user_key && g.largest_len)) {
      delete j;
      return fail(B200C_ERR_NOT_SUPPORTED, "grandparent boundary key longer than 16 bytes");
    }
    GpKey a, b;
    pack(g.smallest_user_key, g.smallest_len, &a);
    pack(g.largest_user_key, g.largest_len, &b);
    if (i && (j->gp_large[i - 1].hi > a.hi || (j->gp_large[i - 1].hi == a.hi && (j->gp_large[i - 1].lo > a.lo ||
              (j->gp_large[i - 1].lo == a.lo && j->gp_large[i - 1].ulen > a.ulen))))) {
      delete j;
      return fail(B200C_ERR_INVALID_ARGUMENT, "grandparents must be sorted and non-overlapping");
    }
    j->gp_small.push_back(a);
    j->gp_large.push_back(b);
    j->gp_size.push_back(g.file_size);
  }
  for (uint32_t i = 0; i < p->num_grandparents; i++) {
    const bool same = i + 1 < p->num_grandparents && j->gp_small[i + 1].hi == j->gp_large[i].hi &&
                      j->gp_small[i + 1].lo == j->gp_large[i].lo && j->gp_small[i + 1].ulen == j->gp_large[i].ulen;
    j->gp_same.push_back(same ? 1 : 0);
  }
  j->p.grandparents = nullptr;
  if (p->bloom_millibits_per_key && (p->format_version < 5 || p->bloom_millibits_per_key < 1000)) {
    delete j;
    return fail(B200C_ERR_NOT_SUPPORTED, "Bloom filter block needs format_version >= 5 (FastLocalBloom) and >= 1000 millibits per key");
  }
  // sub-compaction key range
  if ((p->has_range_start && (p->range_start_len > kMaxUserKey || (!p->range_start_user_key && p->range_start_len))) ||
      (p->has_range_end && (p->range_end_len > kMaxUserKey || (!p->range_end_user_key && p->range_end_len)))) {
    delete j;
    return fail(B200C_ERR_NOT_SUPPORTED, "sub-compaction range bound longer than 16 bytes");
  }
  if (p->has_range_start) pack(p->range_start_user_key, p->range_start_len, &j->range_lo);
  if (p->has_range_end) pack(p->range_end_user_key, p->range_end_len, &j->range_hi);
  j->p.range_start_user_key = j->p.range_end_user_key = nullptr;
  memset(&j->stats, 0, sizeof j->stats);
  *out = j;
  return B200C_OK;
}

int b200c_job_add_input(b200c_job* j, int level, uint64_t file_number, const void* data, uint64_t len, int mem_kind) {
  if (!j || !data) return fail(B200C_ERR_INVALID_ARGUMENT, "null argument");
  if (mem_kind != B200C_MEM_HOST && mem_kind != B200C_MEM_DEVICE && mem_kind != B200C_MEM_HOST_DEFERRED)
    return fail(B200C_ERR_INVALID_ARGUMENT, "bad mem_kind");
  const bool deferred = mem_kind == B200C_MEM_HOST_DEFERRED;
  if (deferred) mem_kind = B200C_MEM_HOST;
  j->inputs.emplace_back();
  Input& in = j->inputs.back();
  in.level = level;
  in.file_number = file_number;
  in.data = static_cast<const uint8_t*>(data);
  in.len = len;
  in.mem_kind = mem_kind;
  if (mem_kind == B200C_MEM_HOST && !deferred && len >= (1u << 20)) {
    // Start the host -> device copy now, on the job's copy stream: a caller that reads its input files one after the other (the
    // executor plugin) gets the PCIe transfer of file i overlapped with the read of file i + 1.  Failures here are not errors: the
    // run copies the file itself when no eager copy is pending.
    if (cudaSetDevice(j->p.device) == cudaSuccess && (j->st_up || cudaStreamCreateWithFlags(&j->st_up, cudaStreamNonBlocking) == cudaSuccess) &&
        stage_input(in, j->st_up, false) == B200C_OK)
      in.copy.fresh = true;
    else
      cudaGetLastError();
  }
  return B200C_OK;
}

// ---- one job over several key ranges (sub-compactions, db/compaction/compaction_job.cc:264-281,465-640)
namespace {
static_assert(kPlanMaxUserKey == kMaxUserKey, "range planning and the device columns agree on the key width");
}  // namespace

int b200c_job_plan_ranges(b200c_job* j, uint32_t max_ranges, uint64_t min_range_bytes, uint8_t* keys, uint32_t* key_lens, uint32_t* n_boundaries) {
  if (!j || !n_boundaries || (max_ranges > 1 && (!keys || !key_lens))) return fail(B200C_ERR_INVALID_ARGUMENT, "null argument");
  *n_boundaries = 0;
  if (max_ranges <= 1 || j->inputs.empty()) return B200C_OK;
  if (b200c_device_count() <= 0) return fail(B200C_ERR_NO_DEVICE, "no CUDA device");
  if (int rc = job_bind(j)) return rc;
  std::vector<Anchor> anchors;
  uint64_t total = 0;
  IndexBlock idx;
  for (Input& in : j->inputs) {
    if (int rc = open_input(j, in)) return rc;
    total += in.tail.data_size ? in.tail.data_size : in.len;
    if (in.tail.num_data_blocks < 2) continue;
    if (int rc = input_index_block(j, in, &idx)) return rc;
    const std::string e = index_anchors(idx.p, idx.len, in.tail, 128, &anchors);
    if (!e.empty()) return fail(B200C_ERR_CORRUPTION, e);
  }
  const std::vector<Anchor> bnd = plan_boundaries(std::move(anchors), total, max_ranges, min_range_bytes);
  uint32_t nb = 0;
  for (const Anchor& a : bnd) {
    memcpy(keys + (size_t)nb * kMaxUserKey, a.key, kMaxUserKey);
    key_lens[nb] = a.klen;
    nb++;
  }
  *n_boundaries = nb;
  return B200C_OK;
}

int b200c_job_create_sub(b200c_job* parent, const b200c_params* p, b200c_job** out) {
  if (!parent || !p || !out) return fail(B200C_ERR_INVALID_ARGUMENT, "null argument");
  if (p->device != parent->p.device) return fail(B200C_ERR_INVALID_ARGUMENT, "a sub-job runs on its parent's device");
  if (parent->inputs.empty()) return fail(B200C_ERR_STATE, "parent job has no inputs");
  CU(cudaSetDevice(parent->p.device));
  // the device copies of the parent's host inputs, complete before a sub-job reads them (range-pipelined: it waits for its event)
  for (Input& in : parent->inputs) {
    if (in.mem_kind != B200C_MEM_HOST || !parent->range_events.empty()) continue;
    if (int rc = stage_input(in, nullptr, true)) return rc;
    CU(cudaEventSynchronize(in.copy.done));
  }
  b200c_job* j = nullptr;
  if (int rc = b200c_job_create(p, &j)) return rc;
  for (const Input& in : parent->inputs) {
    j->inputs.emplace_back();
    Input& s = j->inputs.back();
    s.level = in.level;
    s.file_number = in.file_number;
    s.len = in.len;
    s.mem_kind = B200C_MEM_DEVICE;
    s.data = in.mem_kind == B200C_MEM_HOST ? in.copy.buf.as<uint8_t>() : in.data;
  }
  if (!parent->range_events.empty()) {
    // the range that ends at boundary r needs the uploads up to event r; an open end (or a bound that is not one of the boundaries)
    // needs everything
    size_t r = parent->range_events.size() - 1;
    if (p->has_range_end) {
      const std::string end(static_cast<const char*>(p->range_end_user_key ? p->range_end_user_key : ""), p->range_end_len);
      for (size_t i = 0; i < parent->range_bounds.size(); i++)
        if (parent->range_bounds[i] == end) {
          r = i;
          break;
        }
    }
    j->wait_ev = parent->range_events[r];
  }
  *out = j;
  return B200C_OK;
}

int b200c_job_upload_by_ranges(b200c_job* j, const uint8_t* keys, const uint32_t* key_lens, uint32_t nb) {
  if (!j || (nb && (!keys || !key_lens))) return fail(B200C_ERR_INVALID_ARGUMENT, "null argument");
  if (j->inputs.empty()) return fail(B200C_ERR_STATE, "job has no inputs");
  if (!j->range_events.empty()) return fail(B200C_ERR_STATE, "the inputs of this job are already uploaded by ranges");
  if (b200c_device_count() <= 0) return fail(B200C_ERR_NO_DEVICE, "no CUDA device");
  if (int rc = job_bind(j)) return rc;
  if (!j->st_up) CU(cudaStreamCreateWithFlags(&j->st_up, cudaStreamNonBlocking));
  std::vector<Anchor> bounds(nb);
  for (uint32_t r = 0; r < nb; r++) {
    if (key_lens[r] > (uint32_t)kMaxUserKey) return fail(B200C_ERR_NOT_SUPPORTED, "range boundary longer than 16 bytes");
    memset(&bounds[r], 0, sizeof(Anchor));
    memcpy(bounds[r].key, keys + (size_t)r * kMaxUserKey, key_lens[r]);
    bounds[r].klen = key_lens[r];
    if (r && anchor_cmp(bounds[r - 1], bounds[r]) >= 0) return fail(B200C_ERR_INVALID_ARGUMENT, "range boundaries must be strictly ascending");
  }
  const size_t k = j->inputs.size();
  std::vector<std::vector<uint64_t>> cuts(k, std::vector<uint64_t>(nb, 0));  // end of chunk r inside file f's data region
  std::vector<uint64_t> data_end(k, 0);
  IndexBlock idx;
  for (size_t f = 0; f < k; f++) {
    Input& in = j->inputs[f];
    if (in.mem_kind != B200C_MEM_HOST || in.copy.fresh)
      return fail(B200C_ERR_STATE, "upload by ranges needs host inputs added with B200C_MEM_HOST_DEFERRED");
    if (int rc = open_input(j, in)) return rc;
    if (int rc = input_index_block(j, in, &idx)) return rc;
    const std::string e = index_range_cuts(idx.p, idx.len, in.tail, in.len, bounds.data(), nb, cuts[f].data(), &data_end[f]);
    if (!e.empty()) return fail(B200C_ERR_CORRUPTION, e);
    CU(in.copy.buf.reserve(in.len + 64));  // every buffer before the first copy: a refusal leaves no copy in flight
  }
  // 1. what every range needs of every file: everything behind the data blocks (filter, index, properties, metaindex, footer)
  for (size_t f = 0; f < k; f++)
    if (int rc = stage_input(j->inputs[f], j->st_up, false, data_end[f])) return rc;
  // 2. the data blocks, range after range
  j->range_events.resize((size_t)nb + 1, nullptr);
  for (uint32_t r = 0; r <= nb; r++) {
    for (size_t f = 0; f < k; f++) {
      const uint64_t lo = r == 0 ? 0 : cuts[f][r - 1], hi = r == nb ? data_end[f] : cuts[f][r];
      if (int rc = stage_input(j->inputs[f], j->st_up, false, lo, hi)) return rc;
    }
    CU(cudaEventCreateWithFlags(&j->range_events[r], cudaEventDisableTiming));
    CU(cudaEventRecord(j->range_events[r], j->st_up));
  }
  j->range_bounds.clear();
  for (uint32_t r = 0; r < nb; r++) j->range_bounds.emplace_back(reinterpret_cast<const char*>(bounds[r].key), bounds[r].klen);
  return B200C_OK;
}

int b200c_host_alloc(int device, uint64_t bytes, void** out) {
  if (!out) return fail(B200C_ERR_INVALID_ARGUMENT, "null argument");
  *out = nullptr;
  if (b200c_device_count() <= 0) return fail(B200C_ERR_NO_DEVICE, "no CUDA device");
  CU(cudaSetDevice(device));
  size_t cap = 0;
  int dev = -1;
  CU(cached_alloc(true, bytes ? bytes : 1, out, &cap, &dev));
  std::lock_guard<std::mutex> l(g_host_allocs_mu);
  g_host_allocs[*out] = {cap, dev};
  return B200C_OK;
}
void b200c_host_free(void* p) {
  if (!p) return;
  std::pair<size_t, int> rec{0, -1};
  {
    std::lock_guard<std::mutex> l(g_host_allocs_mu);
    auto it = g_host_allocs.find(p);
    if (it == g_host_allocs.end()) return;  // not ours
    rec = it->second;
    g_host_allocs.erase(it);
  }
  cached_free(true, p, rec.first, rec.second);
}

int b200c_job_run(b200c_job* j) {
  if (!j) return fail(B200C_ERR_INVALID_ARGUMENT, "null job");
  return run_job(j, 3);
}
int b200c_job_run_until(b200c_job* j, int stage) {
  if (!j || stage < 1 || stage > 3) return fail(B200C_ERR_INVALID_ARGUMENT, "bad stage");
  return run_job(j, stage);
}
int b200c_job_output_count(const b200c_job* j) { return j && j->stage_done == 3 ? (int)j->outputs.size() : -B200C_ERR_STATE; }
int b200c_job_output_meta(const b200c_job* j, int i, b200c_file_meta* m) {
  if (!j || j->stage_done != 3 || i < 0 || i >= (int)j->outputs.size() || !m) return fail(B200C_ERR_STATE, "no such output");
  *m = j->outputs[i].meta;
  return B200C_OK;
}
int b200c_job_output_data(b200c_job* j, int i, const void** data, uint64_t* len) {
  if (!j || j->stage_done != 3 || i < 0 || i >= (int)j->outputs.size()) return fail(B200C_ERR_STATE, "no such output");
  Output& o = j->outputs[i];
  *len = o.meta.file_size;
  *data = j->p.output_mem == B200C_MEM_HOST ? (const void*)(j->host_out.p + o.host_off) : (const void*)(j->out_buf.as<uint8_t>() + o.dev_off);
  return B200C_OK;
}
int b200c_job_output_read(b200c_job* j, int i, void* dst, uint64_t cap) {
  if (!j || j->stage_done != 3 || i < 0 || i >= (int)j->outputs.size()) return fail(B200C_ERR_STATE, "no such output");
  Output& o = j->outputs[i];
  if (cap < o.meta.file_size) return fail(B200C_ERR_INVALID_ARGUMENT, "destination too small");
  if (j->p.output_mem == B200C_MEM_HOST) {
    memcpy(dst, j->host_out.p + o.host_off, o.meta.file_size);
    return B200C_OK;
  }
  CU(cudaSetDevice(j->p.device));
  CU(cudaMemcpy(dst, j->out_buf.as<uint8_t>() + o.dev_off, o.meta.file_size, cudaMemcpyDefault));  // dst: host or device
  return B200C_OK;
}
int b200c_job_get_stats(const b200c_job* j, b200c_stats* s) {
  if (!j || !s) return fail(B200C_ERR_INVALID_ARGUMENT, "null argument");
  *s = j->stats;
  return B200C_OK;
}
void b200c_job_destroy(b200c_job* j) {
  if (!j) return;
  cudaSetDevice(j->p.device);
  // The job's buffers go back to the cache when `delete j` destroys them: nothing of the job may be in flight by then, or a later
  // job could be handed a buffer that a kernel or copy of this one still uses.
  if (j->st) cudaStreamSynchronize(j->st);
  if (j->st2) cudaStreamSynchronize(j->st2);
  if (j->st_up) cudaStreamSynchronize(j->st_up);  // (an eager upload may also still be reading a caller's buffer)
  for (cudaEvent_t e : j->range_events)
    if (e) cudaEventDestroy(e);
  for (auto& in : j->inputs)
    if (in.copy.done) cudaEventDestroy(in.copy.done);
  if (j->st_up) cudaStreamDestroy(j->st_up);
  for (auto& kt : j->ktimes) {
    cudaEventDestroy(kt.a);
    cudaEventDestroy(kt.b);
  }
  for (auto& e : j->ev)
    if (e) cudaEventDestroy(e);
  for (auto& e : j->evx)
    if (e) cudaEventDestroy(e);
  if (j->st2) cudaStreamDestroy(j->st2);
  if (j->st) cudaStreamDestroy(j->st);
  delete j;
}

int b200c_job_kernel_time_count(const b200c_job* j) { return j ? (int)j->kt_used : 0; }
int b200c_job_kernel_time(const b200c_job* j, int i, const char** name, double* us) {
  if (!j || i < 0 || (size_t)i >= j->kt_used) return fail(B200C_ERR_INVALID_ARGUMENT, "no such kernel time");
  *name = j->ktimes[i].name;
  *us = j->ktimes[i].us;
  return B200C_OK;
}

int b200c_job_encode_columns(b200c_job* j, uint64_t n, const void* pfx, const void* tr, const void* vref, const void* meta) {
  if (!j || (n && (!pfx || !tr || !vref || !meta))) return fail(B200C_ERR_INVALID_ARGUMENT, "null argument");
  return encode_columns(j, n, pfx, tr, vref, meta);
}

int b200c_job_encode_kv(b200c_job* j, uint64_t n, const void* arena, const uint64_t* offs, const uint32_t* klens) {
  if (!j || (n && (!arena || !offs || !klens))) return fail(B200C_ERR_INVALID_ARGUMENT, "null argument");
  int rc = job_prepare(j);
  if (rc) return rc;
  cudaStream_t st = j->st;
  const uint64_t bytes = n ? offs[n] : 0;
  // records, offsets and key lengths move to the device; the columns are built there (one thread per entry) in the buffers the
  // merge stage writes on the compaction path (paranoid_file_checks re-reads into the decoder's)
  CU(j->kv_arena.reserve(bytes + 64));
  CU(j->kv_offs.reserve(8 * (n + 1)));
  CU(j->kv_klens.reserve(4 * (n + 1)));
  CU(j->mrg.reserve(n));
  CU(j->small.reserve(kSmallSlots * 8));
  CU(cudaMemsetAsync(j->small.p, 0, kSmallSlots * 8, st));
  if (n) {
    CU(cudaMemcpyAsync(j->kv_arena.p, arena, bytes, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(j->kv_offs.p, offs, 8 * (n + 1), cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(j->kv_klens.p, klens, 4 * n, cudaMemcpyHostToDevice, st));
  }
  const KeyColsMut cols = j->mrg.mut();
  uint32_t* err = reinterpret_cast<uint32_t*>(j->small.as<uint64_t>() + kSlotErr);
  launch_kv_to_columns(j->kv_arena.as<uint8_t>(), j->kv_offs.as<uint64_t>(), j->kv_klens.as<uint32_t>(), n, cols, err, j->sms, st);
  uint64_t h[kSmallSlots];
  rc = checked_sync(j, h);
  if (rc) return rc;
  return encode_columns(j, n, cols.pfx, cols.tr, cols.vref, cols.meta, /*prepared=*/true);
}

int b200c_job_debug_read(b200c_job* j, int what, int run, void* dst, uint64_t cap, uint64_t* len) {
  if (!j || !len) return fail(B200C_ERR_INVALID_ARGUMENT, "null argument");
  CU(cudaSetDevice(j->p.device));
  cudaStream_t st = j->st;
  struct Rec {
    uint64_t hi, lo, tr;
    uint32_t ulen, vlen;
  };
  auto read_keys = [&](const KeyBufs& c, uint64_t first, uint64_t n) -> int {
    *len = n * sizeof(Rec);
    if (!dst || cap < *len) return B200C_OK;
    std::vector<ulonglong2> pfx(n);
    std::vector<uint64_t> tr(n);
    std::vector<uint32_t> meta(n);
    if (n) {
      CU(cudaMemcpy(pfx.data(), c.pfx.as<ulonglong2>() + first, 16 * n, cudaMemcpyDeviceToHost));
      CU(cudaMemcpy(tr.data(), c.tr.as<uint64_t>() + first, 8 * n, cudaMemcpyDeviceToHost));
      CU(cudaMemcpy(meta.data(), c.meta.as<uint32_t>() + first, 4 * n, cudaMemcpyDeviceToHost));
    }
    Rec* r = static_cast<Rec*>(dst);
    for (uint64_t i = 0; i < n; i++) r[i] = Rec{pfx[i].x, pfx[i].y, tr[i], meta_ulen(meta[i]), meta_vlen(meta[i])};
    return B200C_OK;
  };
  auto read_values = [&](const KeyBufs& c, uint64_t first, uint64_t n) -> int {
    DevBuf vl, off, tmp, tot, bytes;
    CU(vl.reserve(4 * (n + 1)));
    CU(off.reserve(8 * (n + 1)));
    CU(tmp.reserve(8 * (n / kScanTile + 2)));
    CU(tot.reserve(8));
    int rc = B200C_OK;
    KeyCols kc{c.pfx.as<ulonglong2>() + first, c.tr.as<uint64_t>() + first, c.vref.as<uint64_t>() + first, c.meta.as<uint32_t>() + first, n};
    launch_meta_vlen(kc.meta, n, vl.as<uint32_t>(), st);
    exclusive_scan<uint32_t>(vl.as<uint32_t>(), off.as<uint64_t>(), n, tmp.as<uint64_t>(), tot.as<uint64_t>(), st, nullptr);
    uint64_t total = 0;
    cudaMemcpyAsync(&total, tot.p, 8, cudaMemcpyDeviceToHost, st);
    cudaStreamSynchronize(st);
    *len = total;
    if (dst && cap >= total && total) {
      if (bytes.reserve(total) != cudaSuccess) rc = fail(B200C_ERR_OUT_OF_MEMORY, "debug value buffer");
      else {
        launch_gather_values(kc, off.as<uint64_t>(), bytes.as<uint8_t>(), st);
        cudaMemcpyAsync(dst, bytes.p, total, cudaMemcpyDeviceToHost, st);
        cudaStreamSynchronize(st);
      }
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(B200C_ERR_CUDA, cudaGetErrorString(e));
    return rc;
  };
  switch (what) {
    case B200C_DBG_DECODED_KEYS:
    case B200C_DBG_DECODED_VALUES: {
      if (j->stage_done < 1) return fail(B200C_ERR_STATE, "decode stage has not run");
      if (j->run_start_h.empty()) {
        j->run_start_h.resize(j->inputs.size() + 1);
        CU(cudaMemcpy(j->run_start_h.data(), j->run_start.p, 8 * (j->inputs.size() + 1), cudaMemcpyDeviceToHost));
      }
      if (run < 0 || run >= (int)j->inputs.size()) return fail(B200C_ERR_INVALID_ARGUMENT, "bad run index");
      uint64_t first = j->run_start_h[run], n = j->run_start_h[run + 1] - first;
      return what == B200C_DBG_DECODED_KEYS ? read_keys(j->dec, first, n) : read_values(j->dec, first, n);
    }
    case B200C_DBG_MERGED_KEYS:
      if (j->stage_done < 2) return fail(B200C_ERR_STATE, "merge stage has not run");
      return read_keys(j->mrg, 0, j->n_out);
    case B200C_DBG_MERGED_VALUES:
      if (j->stage_done < 2) return fail(B200C_ERR_STATE, "merge stage has not run");
      return read_values(j->mrg, 0, j->n_out);
    case B200C_DBG_BLOCK_LIST: {
      if (j->stage_done < 3) return fail(B200C_ERR_STATE, "encode stage has not run");
      *len = j->nblocks_out * sizeof(BlockRec);
      if (dst && cap >= *len && *len) CU(cudaMemcpy(dst, j->blocks.p, *len, cudaMemcpyDeviceToHost));
      return B200C_OK;
    }
  }
  return fail(B200C_ERR_INVALID_ARGUMENT, "unknown debug array");
}

int b200c_block_checksums(int device, uint32_t type, const void* host_data, const uint64_t* offsets, uint32_t n, uint8_t last_byte,
                          uint32_t* out) {
  if (!host_data || !offsets || !out) return fail(B200C_ERR_INVALID_ARGUMENT, "null argument");
  int cnt = b200c_device_count();
  if (cnt <= 0) return fail(B200C_ERR_NO_DEVICE, "no CUDA device");
  CU(cudaSetDevice(device));
  DevBuf d, o, r;
  uint64_t total = offsets[n];
  CU(d.reserve(total + 16));
  CU(o.reserve(8 * (n + 1)));
  CU(r.reserve(4 * (n + 1)));
  CU(cudaMemcpy(d.p, host_data, total, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(o.p, offsets, 8 * (n + 1), cudaMemcpyHostToDevice));
  launch_block_checksums(type, d.as<uint8_t>(), o.as<uint64_t>(), n, last_byte, r.as<uint32_t>(), 0);
  CU(cudaDeviceSynchronize());
  CU(cudaMemcpy(out, r.p, 4 * n, cudaMemcpyDeviceToHost));
  return B200C_OK;
}

}  // extern "C"
