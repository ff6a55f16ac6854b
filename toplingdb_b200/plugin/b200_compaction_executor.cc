// toplingdb_b200/plugin/b200_compaction_executor.cc — see the header.  Host glue only: every byte of the data path goes
// through libb200c.so (include/b200c.h).  Error behaviour mirrors RunRemote's contract (compaction_job.cc:921-1152):
// Execute returns a Status, results->status carries the job status, no exception crosses the executor.
#include "b200_compaction_executor.h"

#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <set>
#include <thread>
#include <vector>

#include "b200c.h"
#include "rocksdb/compaction_filter.h"
#include "rocksdb/convenience.h"
#include "db/compaction/compaction.h"
#include "db/version_edit.h"
#include "file/filename.h"
#include "rocksdb/comparator.h"
#include "rocksdb/env.h"
#include "rocksdb/file_system.h"
#include "rocksdb/sst_partitioner.h"
#include "rocksdb/table.h"
#include "table/block_based/filter_policy_internal.h"

namespace ROCKSDB_NAMESPACE {

namespace {

// Which device filter (include/b200c.h b200c_compaction_filter) the column family's filter factory stands for; NONE when the
// family has no factory or the filter is not one the merge kernel implements.  Filters are recognised by CompactionFilter::Name().
uint32_t DeviceFilterOf(const Compaction* c, int32_t* ttl = nullptr) {
  const auto& factory = c->immutable_options()->compaction_filter_factory;
  if (!factory) return B200C_FILTER_NONE;
  if (std::string(factory->Name()) == "TtlCompactionFilterFactory") {
    // DBWithTTL (utilities/ttl/db_ttl_impl.h:183-206): only without a user filter stacked underneath; "ttl" is a registered option
    if (factory->Inner() != nullptr) return B200C_FILTER_NONE;
    std::string v;
    ConfigOptions co;
    if (!factory->GetOption(co, "ttl", &v).ok()) return B200C_FILTER_NONE;
    if (ttl) *ttl = (int32_t)strtol(v.c_str(), nullptr, 10);
    return B200C_FILTER_TTL;
  }
  CompactionFilter::Context ctx;
  ctx.is_full_compaction = c->is_full_compaction();
  ctx.is_manual_compaction = c->is_manual_compaction();
  ctx.column_family_id = c->column_family_data()->GetID();
  std::unique_ptr<CompactionFilter> f = factory->CreateCompactionFilter(ctx);
  if (f && std::string(f->Name()) == "RemoveEmptyValueCompactionFilter") return B200C_FILTER_REMOVE_EMPTY_VALUE;
  return B200C_FILTER_NONE;
}

// Filter block of the output files: 0 = none; > 0 = millibits per key of a BloomFilterPolicy (NewBloomFilterPolicy) in the one shape the
// device builds -- full filter over whole keys, format_version >= 5 (FastLocalBloom), no prefix extractor, no malloc-size dependent
// rounding; < 0 = any other filter (Ribbon, partitioned, prefixes, user policies): the job stays on the CPU.
int DeviceBloomMillibits(const Compaction* c, const BlockBasedTableOptions* t) {
  const FilterPolicy* fp = t->filter_policy.get();
  if (fp == nullptr) return 0;
  if (strcmp(fp->Name(), "bloomfilter") != 0) return -1;
  if (t->partition_filters || !t->whole_key_filtering || t->optimize_filters_for_memory || t->format_version < 5) return -1;
  if (c->mutable_cf_options()->prefix_extractor != nullptr) return -1;
  return static_cast<const BloomLikeFilterPolicy*>(fp)->GetMillibitsPerKey();
}

// Output partitioner of the column family (b200c_params::sst_partitioner_prefix_len): 0 = none; the prefix length of the stock
// SstPartitionerFixedPrefixFactory, read through its registered option "length" (db/compaction/sst_partitioner.cc); < 0 = any
// other partitioner, whose cuts the device cannot know: the job stays on the CPU.
int64_t DevicePartitionerPrefixLen(const Compaction* c) {
  const auto& f = c->immutable_options()->sst_partitioner_factory;
  if (f == nullptr) return 0;
  if (strcmp(f->Name(), SstPartitionerFixedPrefixFactory::kClassName()) != 0) return -1;
  std::string v;
  ConfigOptions co;
  if (!f->GetOption(co, "length", &v).ok()) return -1;
  const unsigned long long len = strtoull(v.c_str(), nullptr, 10);
  return (int64_t)std::min<unsigned long long>(len, 0xffffffffull);  // >= 16 already means "the user key changed" on the device
}

// Output-file cut rules of CompactionOutputs::ShouldStopBefore (compaction_outputs.cc:231-354) that the device does NOT evaluate: the
// TTL cut at old files of the output level (FillFilesToCutForTtl :737-777, same conditions restated here) and the round-robin cursor
// split (:282-291).  When one of them could fire, the reference must cut the files itself.
bool HasHostOnlyFileCutRule(const Compaction* c) {
  if (c->output_level() == 0) return false;
  if (c->GetOutputSplitKey() != nullptr) return true;
  const auto* io = c->immutable_options();
  const auto* mo = c->mutable_cf_options();
  if (io->compaction_style != kCompactionStyleLevel || io->compaction_pri != kMinOverlappingRatio || mo->ttl == 0 ||
      c->num_input_levels() < 2 || c->bottommost_level())
    return false;
  int64_t now = 0;
  if (!io->clock->GetCurrentTime(&now).ok() || (uint64_t)now < mo->ttl) return false;
  const uint64_t old_age_thres = (uint64_t)now - mo->ttl / 2;
  for (FileMetaData* f : *c->inputs(c->num_input_levels() - 1))
    if (f->TryGetOldestAncesterTime() < old_age_thres && f->fd.GetFileSize() > mo->target_file_size_base / 2) return true;
  return false;
}

const BlockBasedTableOptions* BlockBasedOptionsOf(const Compaction* c) {
  auto* tf = c->immutable_options()->table_factory.get();
  if (tf == nullptr) return nullptr;
  // the stock factory, or the B200 table factory (plugin/b200_table_factory.h), which answers with its stock factory's options
  if (strcmp(tf->Name(), TableFactory::kBlockBasedTableName()) != 0 && strcmp(tf->Name(), "B200BlockBasedTable") != 0) return nullptr;
  return tf->GetOptions<BlockBasedTableOptions>();
}

Status FromB200(int rc) {
  const char* msg = b200c_last_error();
  switch (rc) {
    case B200C_OK: return Status::OK();
    case B200C_ERR_NOT_SUPPORTED: return Status::NotSupported("b200c", msg);
    case B200C_ERR_CORRUPTION: return Status::Corruption("b200c", msg);
    case B200C_ERR_INVALID_ARGUMENT: return Status::InvalidArgument("b200c", msg);
    case B200C_ERR_OUT_OF_MEMORY: return Status::MemoryLimit("b200c", msg);
    default: return Status::Aborted("b200c", msg);
  }
}

// All file I/O goes through the DB's own FileSystem (ImmutableDBOptions::fs): an EncryptedEnv, a custom file system, a mock Env in
// tests see every byte, exactly as they do for the reference's local compaction (file/writable_file_writer.cc, table_cache.cc).
IOStatus ReadFileFS(FileSystem* fs, const std::string& fname, char* dst, uint64_t size) {
  std::unique_ptr<FSRandomAccessFile> f;
  FileOptions fo;
  IOStatus s = fs->NewRandomAccessFile(fname, fo, &f, nullptr);
  if (!s.ok()) return s;
  uint64_t off = 0;
  while (off < size) {
    const size_t n = (size_t)std::min<uint64_t>(size - off, 64ull << 20);
    Slice res;
    s = f->Read(off, n, IOOptions(), &res, dst + off, nullptr);
    if (!s.ok()) return s;
    if (res.size() == 0) return IOStatus::Corruption("short read", fname);
    if (res.data() != dst + off) memmove(dst + off, res.data(), res.size());
    off += res.size();
  }
  return IOStatus::OK();
}
// An output table is durable before Execute returns: appended, synced (fsync when DBOptions::use_fsync), closed with the close
// status checked -- what CompactionOutputs::Finish / WritableFileWriter::Sync do on the local path (compaction_outputs.cc:63,
// compaction_job.cc:1905-1921).  RunRemote installs the file in a synced MANIFEST right after the rename.
IOStatus WriteFileFS(FileSystem* fs, const std::string& fname, const char* data, uint64_t len, bool use_fsync) {
  std::unique_ptr<FSWritableFile> f;
  FileOptions fo;
  IOStatus s = fs->NewWritableFile(fname, fo, &f, nullptr);
  if (!s.ok()) return s;
  uint64_t off = 0;
  while (s.ok() && off < len) {
    const size_t n = (size_t)std::min<uint64_t>(len - off, 64ull << 20);
    s = f->Append(Slice(data + off, n), IOOptions(), nullptr);
    off += n;
  }
  if (s.ok()) s = use_fsync ? f->Fsync(IOOptions(), nullptr) : f->Sync(IOOptions(), nullptr);
  IOStatus c = f->Close(IOOptions(), nullptr);
  return s.ok() ? c : s;
}
IOStatus SyncDirFS(FileSystem* fs, const std::string& dir) {
  std::unique_ptr<FSDirectory> d;
  IOStatus s = fs->NewDirectory(dir, IOOptions(), &d, nullptr);
  if (!s.ok()) return s;
  s = d->FsyncWithDirOptions(IOOptions(), nullptr, DirFsyncOptions());
  IOStatus c = d->Close(IOOptions(), nullptr);
  return s.ok() ? c : s;
}
std::string DirOf(const std::string& path) {
  const size_t p = path.find_last_of('/');
  return p == std::string::npos ? std::string(".") : (p == 0 ? std::string("/") : path.substr(0, p));
}

// pinned host buffer from the library (cudaHostAlloc behind the C ABI: the plugin itself stays free of CUDA headers); a plain
// allocation when pinning fails (the copy is slower then, nothing else changes)
struct HostImage {
  char* p = nullptr;
  uint64_t len = 0;
  bool pinned = false;
  HostImage() = default;
  HostImage(const HostImage&) = delete;
  HostImage& operator=(const HostImage&) = delete;
  bool Alloc(int device, uint64_t n) {
    len = n;
    void* q = nullptr;
    if (b200c_host_alloc(device, n ? n : 1, &q) == B200C_OK) {
      p = static_cast<char*>(q);
      pinned = true;
    } else {
      p = static_cast<char*>(malloc(n ? n : 1));
    }
    return p != nullptr;
  }
  ~HostImage() {
    if (p && pinned) b200c_host_free(p);
    else free(p);
  }
};

class B200CompactionExecutor : public CompactionExecutor {
 public:
  B200CompactionExecutor(const B200CompactOptions& o, const Compaction* c) : opt_(o), c_(c) {}

  void SetParams(CompactionParams* p, const Compaction* c) override {
    // the fields RunRemote leaves to the executor (compaction_job.cc:944-963 fills the rest)
    auto* cfd = c->column_family_data();
    p->num_levels = c->number_levels();
    p->output_level = c->output_level();
    p->cf_id = cfd->GetID();
    p->cf_name = cfd->GetName();
    p->inputs = c->inputs();
    p->target_file_size = c->max_output_file_size();
    p->max_compaction_bytes = c->max_compaction_bytes();
    p->cf_paths = c->immutable_options()->cf_paths;
    p->compression = c->output_compression();
    p->compression_opts = c->output_compression_opts();
    p->grandparents = &c->grandparents();
    p->score = c->score();
    p->manual_compaction = c->is_manual_compaction();
    p->deletion_compaction = c->deletion_compaction();
    p->compaction_reason = c->compaction_reason();
    p->bottommost_level = c->bottommost_level();
    p->smallest_user_key = c->GetSmallestUserKey().ToString();
    p->largest_user_key = c->GetLargestUserKey().ToString();
    p->level_compaction_dynamic_file_size = c->immutable_options()->level_compaction_dynamic_file_size;
    p->compaction_style = c->immutable_options()->compaction_style;
    p->compaction_pri = c->immutable_options()->compaction_pri;
    p->is_deserialized = false;  // in-process: the struct borrows the DB's objects (compaction_executor.cc:12-38)
  }

  Status Execute(const CompactionParams& p, CompactionResults* r) override {
    const auto t0 = std::chrono::steady_clock::now();
    const BlockBasedTableOptions* bbt = BlockBasedOptionsOf(c_);
    if (bbt == nullptr) return Fail(r, Status::NotSupported("B200Compact needs a BlockBasedTable output"));
    b200c_params bp;
    b200c_params_init(&bp);
    bp.device = opt_.device;
    bp.output_level = p.output_level;
    bp.bottommost_level = p.bottommost_level;
    bp.max_output_file_size = c_->max_output_file_size();
    bp.block_size = (uint32_t)bbt->block_size;
    bp.block_size_deviation = (uint32_t)bbt->block_size_deviation;
    bp.block_restart_interval = (uint32_t)bbt->block_restart_interval;
    bp.index_block_restart_interval = (uint32_t)bbt->index_block_restart_interval;
    bp.format_version = bbt->format_version;
    bp.checksum = (uint32_t)bbt->checksum;
    bp.verify_input_checksums = opt_.verify_input_checksums;
    bp.paranoid_file_checks = p.paranoid_file_checks;  // RunRemote cannot hash what it did not write (compaction_job.cc:1065-1068)
    bp.bloom_millibits_per_key = (uint32_t)std::max(0, DeviceBloomMillibits(c_, bbt));
    bp.earliest_write_conflict_snapshot = p.earliest_write_conflict_snapshot;
    bp.sst_partitioner_prefix_len = (uint32_t)std::max<int64_t>(0, DevicePartitionerPrefixLen(c_));
    std::vector<uint64_t> snaps;
    if (p.existing_snapshots) snaps.assign(p.existing_snapshots->begin(), p.existing_snapshots->end());
    bp.snapshots = snaps.data();
    bp.num_snapshots = (uint32_t)snaps.size();
    bp.column_family_id = p.cf_id;
    bp.column_family_name = p.cf_name.c_str();
    bp.db_id = p.db_id.c_str();
    bp.db_session_id = p.db_session_id.c_str();
    std::string host = c_->immutable_options()->db_host_id;
    if (host == kHostnameForDbHostId) {
      host.clear();
      c_->immutable_options()->env->GetHostNameString(&host).PermitUncheckedError();
    }
    bp.db_host_id = host.c_str();
    int64_t now = 0;
    c_->immutable_options()->clock->GetCurrentTime(&now).PermitUncheckedError();
    uint64_t oldest = c_->MinInputFileOldestAncesterTime(nullptr, nullptr);
    bp.creation_time = oldest == std::numeric_limits<uint64_t>::max() ? (uint64_t)now : oldest;  // compaction_job.cc:2258-2276
    uint64_t fct = (uint64_t)now;
    bp.file_creation_times = &fct;
    bp.num_file_creation_times = 1;
    // Numbers are local to output_dir -- RunRemote gives every file a fresh number and renames it (compaction_job.cc:1019-1033) --
    // but the number also lands in the table property rocksdb.original.file.number, which together with the session id derives
    // the file's unique id and (in builds with stable cache keys) its block-cache key.  It is therefore unique per job within a DB
    // session: job ids are, and no job writes 2^20 files.
    bp.first_file_number = ((uint64_t)(uint32_t)p.job_id << 20) | 1;
    bp.output_mem = B200C_MEM_HOST;
    // grandparents: CompactionOutputs::ShouldStopBefore cuts output files at their boundaries (compaction_outputs.cc:294-351)
    std::vector<b200c_grandparent> gps;
    std::vector<std::string> gp_keys;  // owns the user-key bytes
    gp_keys.reserve(2 * c_->grandparents().size());
    for (const FileMetaData* fm : c_->grandparents()) {
      // a boundary that is a range-tombstone sentinel compares as an EXCLUSIVE bound (sstableKeyCompare, compaction.cc:28-43); the
      // device rules treat boundaries as plain user keys, so such a job keeps the reference's own file cuts by running locally
      const uint64_t sentinel = PackSequenceAndType(kMaxSequenceNumber, kTypeRangeDeletion);
      if (ExtractInternalKeyFooter(fm->smallest.Encode()) == sentinel || ExtractInternalKeyFooter(fm->largest.Encode()) == sentinel)
        return Fail(r, Status::NotSupported("B200Compact: grandparent file bounded by a range tombstone"));
      gp_keys.push_back(fm->smallest.user_key().ToString());
      gp_keys.push_back(fm->largest.user_key().ToString());
    }
    for (size_t i = 0; i < c_->grandparents().size(); i++) {
      b200c_grandparent g;
      g.smallest_user_key = gp_keys[2 * i].data();
      g.smallest_len = (uint32_t)gp_keys[2 * i].size();
      g.largest_user_key = gp_keys[2 * i + 1].data();
      g.largest_len = (uint32_t)gp_keys[2 * i + 1].size();
      g.file_size = c_->grandparents()[i]->fd.GetFileSize();
      gps.push_back(g);
    }
    bp.grandparents = gps.data();
    bp.num_grandparents = (uint32_t)gps.size();
    bp.level_compaction_dynamic_file_size = p.level_compaction_dynamic_file_size;
    bp.max_compaction_bytes = c_->max_compaction_bytes();
    bp.target_output_file_size = c_->target_output_file_size();
    bp.compaction_filter = DeviceFilterOf(c_, &bp.ttl);
    bp.ttl_now = now;  // TtlCompactionFilter reads the clock per entry; one reading per job here

    b200c_job* job = nullptr;
    Status s = FromB200(b200c_job_create(&bp, &job));
    if (!s.ok()) return Fail(r, s);
    // child order of VersionSet::MakeInputIterator (db/version_set.cc:7269-7352): L0 files as listed, then each level
    FileSystem* fs = c_->immutable_options()->fs.get();
    const bool use_fsync = c_->immutable_options()->use_fsync;
    size_t nfiles_in = 0;
    for (const auto& lvl : *p.inputs) nfiles_in += lvl.files.size();
    // one pinned buffer per input file; they never move (the library keeps the pointers until the job is destroyed).  The files are
    // read by up to io_threads threads; this thread hands each file to the library as soon as it and all files before it are in
    // memory (the order of the calls is the order of the merge's children), and the library starts its host -> device copy at once
    struct InFile {
      int level;
      const FileMetaData* fm;
    };
    std::vector<InFile> in_files;
    in_files.reserve(nfiles_in);
    for (const auto& lvl : *p.inputs)
      for (const FileMetaData* fm : lvl.files) {
        if (fm->num_range_deletions) s = Status::NotSupported("B200Compact: range tombstones in input");
        in_files.push_back(InFile{lvl.level, fm});
      }
    std::vector<std::unique_ptr<HostImage>> images(in_files.size());
    uint64_t in_bytes = 0;
    for (size_t i = 0; i < in_files.size() && s.ok(); i++) {
      images[i].reset(new HostImage());
      if (!images[i]->Alloc(opt_.device, in_files[i].fm->fd.GetFileSize())) s = Status::MemoryLimit("B200Compact: input buffer");
    }
    if (s.ok() && !in_files.empty()) {
      const size_t nf = in_files.size();
      std::vector<Status> rstat(nf);
      std::vector<char> ready(nf, 0);
      std::mutex mu;
      std::condition_variable cv;
      std::atomic<size_t> next{0};
      std::atomic<bool> stop{false};
      auto reader = [&]() {
        for (size_t i; !stop.load(std::memory_order_relaxed) && (i = next.fetch_add(1)) < nf;) {
          const FileMetaData* fm = in_files[i].fm;
          Status rs = ReadFileFS(fs, TableFileName(p.cf_paths, fm->fd.GetNumber(), fm->fd.GetPathId()), images[i]->p, fm->fd.GetFileSize());
          std::lock_guard<std::mutex> l(mu);
          rstat[i] = rs;
          ready[i] = 1;
          cv.notify_all();
        }
      };
      const size_t nthreads = std::min<size_t>((size_t)std::max(1, opt_.io_threads), nf);
      std::vector<std::thread> pool;
      for (size_t t = 1; t < nthreads; t++) pool.emplace_back(reader);
      if (nthreads == 1) reader();
      for (size_t i = 0; i < nf && s.ok(); i++) {
        if (nthreads > 1) {
          std::unique_lock<std::mutex> l(mu);
          // with helpers running, this thread reads too whenever the file it waits for has not been claimed yet
          while (!ready[i]) {
            size_t mine = next.load();
            if (mine < nf && next.compare_exchange_strong(mine, mine + 1)) {
              l.unlock();
              const FileMetaData* fm = in_files[mine].fm;
              Status rs = ReadFileFS(fs, TableFileName(p.cf_paths, fm->fd.GetNumber(), fm->fd.GetPathId()), images[mine]->p, fm->fd.GetFileSize());
              l.lock();
              rstat[mine] = rs;
              ready[mine] = 1;
              cv.notify_all();
            } else {
              cv.wait(l, [&] { return ready[i] != 0; });
            }
          }
        }
        s = rstat[i];
        if (!s.ok()) break;
        const uint64_t fsize = in_files[i].fm->fd.GetFileSize();
        in_bytes += fsize;
        s = FromB200(b200c_job_add_input(job, in_files[i].level, in_files[i].fm->fd.GetNumber(), images[i]->p, fsize, B200C_MEM_HOST));
      }
      stop.store(true);
      for (auto& th : pool) th.join();
    }
    auto shutting_down = [&]() { return p.shutting_down && p.shutting_down->load(std::memory_order_acquire); };
    if (s.ok() && shutting_down()) s = Status::ShutdownInProgress();
    // ---- sub-compactions (CompactionJob::Prepare / GenSubcompactionBoundaries, compaction_job.cc:264-281,465-640): when the DB
    // would split this job over threads, the executor splits it into key ranges that run concurrently -- on the streams of one
    // device, or spread over the devices listed in B200CompactOptions::devices.  RunRemote accepts any number of result groups
    // (compaction_job.cc:986-1000).  The ranges share the uploaded input images (b200c_job_create_sub).
    std::vector<b200c_job*> parents{job};  // one holder of the inputs per device in use
    std::vector<b200c_job*> units;         // what actually runs: the job itself, or its sub-jobs in key order
    std::vector<std::string> bounds;       // owns the boundary user keys
    uint32_t want_subs = opt_.max_subcompactions > 0 ? (uint32_t)opt_.max_subcompactions : p.max_subcompactions;
    if (want_subs > 64) want_subs = 64;
    if (s.ok() && want_subs > 1 && c_->ShouldFormSubcompactions()) {
      std::vector<uint8_t> keys((size_t)want_subs * 16);
      std::vector<uint32_t> lens(want_subs);
      uint32_t nb = 0;
      s = FromB200(b200c_job_plan_ranges(job, want_subs, c_->max_output_file_size(), keys.data(), lens.data(), &nb));
      for (uint32_t i = 0; i < nb && s.ok(); i++) bounds.emplace_back(reinterpret_cast<const char*>(keys.data()) + 16 * (size_t)i, lens[i]);
    }
    if (s.ok() && !bounds.empty()) {
      const size_t nsub = bounds.size() + 1;
      std::vector<int> devs = opt_.devices.empty() ? std::vector<int>{opt_.device} : opt_.devices;
      if (devs.size() > nsub) devs.resize(nsub);
      if (getenv("B200C_PLUGIN_TRACE") != nullptr)
        fprintf(stderr, "B200Compact: job %d split into %zu key ranges over %zu device(s)\n", p.job_id, nsub, devs.size());
      for (size_t d = 1; d < devs.size() && s.ok(); d++) {  // the other devices get their own copy of the inputs (their own PCIe link)
        b200c_params dp = bp;
        dp.device = devs[d];
        b200c_job* pj = nullptr;
        s = FromB200(b200c_job_create(&dp, &pj));
        if (!s.ok()) break;
        parents.push_back(pj);
        for (size_t i = 0; i < in_files.size() && s.ok(); i++)
          s = FromB200(b200c_job_add_input(pj, in_files[i].level, in_files[i].fm->fd.GetNumber(), images[i]->p, in_files[i].fm->fd.GetFileSize(),
                                           B200C_MEM_HOST));
      }
      for (size_t i = 0; i < nsub && s.ok(); i++) {
        b200c_params sp = bp;
        sp.device = devs[i % devs.size()];
        sp.first_file_number = bp.first_file_number + ((uint64_t)i << 14);  // (job << 20 | sub << 14 | file): unique per session
        if (i > 0) {
          sp.range_start_user_key = bounds[i - 1].data();
          sp.range_start_len = (uint32_t)bounds[i - 1].size();
          sp.has_range_start = 1;
        }
        if (i + 1 < nsub) {
          sp.range_end_user_key = bounds[i].data();
          sp.range_end_len = (uint32_t)bounds[i].size();
          sp.has_range_end = 1;
        }
        b200c_job* sj = nullptr;
        s = FromB200(b200c_job_create_sub(parents[i % devs.size()], &sp, &sj));
        if (s.ok()) units.push_back(sj);
      }
      if (s.ok()) {
        std::vector<Status> rstat(units.size());
        std::vector<std::thread> pool;
        for (size_t i = 1; i < units.size(); i++)
          pool.emplace_back([&, i]() { rstat[i] = shutting_down() ? Status::ShutdownInProgress() : FromB200(b200c_job_run(units[i])); });
        rstat[0] = FromB200(b200c_job_run(units[0]));
        for (auto& th : pool) th.join();
        for (size_t i = 0; i < units.size() && s.ok(); i++) s = rstat[i];
      }
    } else if (s.ok()) {
      units.push_back(job);
      s = FromB200(b200c_job_run(job));
    }
    if (s.ok() && shutting_down()) s = Status::ShutdownInProgress();  // do not materialise files for a DB that is closing
    std::vector<std::string> written;
    if (s.ok()) {
      // scratch directory: unique per DB session and job, so that DBs sharing a factory / scratch_dir cannot collide
      const std::string root = opt_.scratch_dir.empty() ? p.dbname + "/b200c-tmp" : opt_.scratch_dir;
      r->output_dir = root + "/job-" + (p.db_session_id.empty() ? std::string("s") : p.db_session_id) + "-" + std::to_string(p.job_id);
      fs->CreateDirIfMissing(root, IOOptions(), nullptr).PermitUncheckedError();
      s = fs->CreateDirIfMissing(r->output_dir, IOOptions(), nullptr);
      r->output_files.resize(units.size());  // one result group per sub-compaction, in key order
      struct OutFile {
        b200c_file_meta m;
        const void* data;
        uint64_t len;
        std::string fname;
        size_t unit;
      };
      std::vector<OutFile> outs;
      for (size_t u = 0; u < units.size() && s.ok(); u++) {
        const int nu = b200c_job_output_count(units[u]);
        for (int i = 0; i < nu && s.ok(); i++) {
          OutFile o;
          o.unit = u;
          s = FromB200(b200c_job_output_meta(units[u], i, &o.m));
          if (s.ok()) s = FromB200(b200c_job_output_data(units[u], i, &o.data, &o.len));
          if (s.ok()) o.fname = MakeTableFileName(r->output_dir, o.m.file_number);
          if (s.ok()) outs.push_back(std::move(o));
        }
      }
      const int n = (int)outs.size();
      if (s.ok() && n > 0) {  // write + sync the files, up to io_threads at a time
        for (auto& o : outs) written.push_back(o.fname);
        std::vector<Status> wstat((size_t)n);
        std::atomic<int> next{0};
        auto writer = [&]() {
          for (int i; (i = next.fetch_add(1)) < n;)
            wstat[i] = WriteFileFS(fs, outs[i].fname, static_cast<const char*>(outs[i].data), outs[i].len, use_fsync);
        };
        const int nthreads = std::min(std::max(1, opt_.io_threads), n);
        std::vector<std::thread> pool;
        for (int t = 1; t < nthreads; t++) pool.emplace_back(writer);
        writer();
        for (auto& th : pool) th.join();
        for (int i = 0; i < n && s.ok(); i++) s = wstat[i];
      }
      for (int i = 0; i < n && s.ok(); i++) {
        const b200c_file_meta& m = outs[i].m;
        CompactionResults::FileMinMeta fm;
        fm.file_number = m.file_number;
        fm.file_size = m.file_size;
        fm.smallest_seqno = m.smallest_seqno;
        fm.largest_seqno = m.largest_seqno;
        fm.smallest_ikey.DecodeFrom(Slice((const char*)m.smallest_ikey, m.smallest_ikey_len));
        fm.largest_ikey.DecodeFrom(Slice((const char*)m.largest_ikey, m.largest_ikey_len));
        fm.marked_for_compaction = false;
        r->output_files[outs[i].unit].push_back(std::move(fm));
      }
      if (s.ok()) s = SyncDirFS(fs, r->output_dir);  // the new names are durable too
      if (!s.ok()) {  // nothing of a failed job stays behind
        for (const auto& f : written) fs->DeleteFile(f, IOOptions(), nullptr).PermitUncheckedError();
        fs->DeleteDir(r->output_dir, IOOptions(), nullptr).PermitUncheckedError();
        r->output_files.clear();
      }
    }
    if (s.ok()) {
      b200c_stats st;
      memset(&st, 0, sizeof st);
      for (b200c_job* u : units) {  // the ranges partition the job: their counters add up (AggregateStatistics on the local path)
        b200c_stats us;
        b200c_job_get_stats(u, &us);
        st.num_input_records += us.num_input_records;
        st.num_output_records += us.num_output_records;
        st.num_input_deletion_records += us.num_input_deletion_records;
        st.num_records_replaced += us.num_records_replaced;
        st.num_expired_deletion_records += us.num_expired_deletion_records;
        st.total_input_raw_key_bytes += us.total_input_raw_key_bytes;
        st.total_input_raw_value_bytes += us.total_input_raw_value_bytes;
        st.total_output_bytes += us.total_output_bytes;
        st.num_output_files += us.num_output_files;
        st.num_input_files = us.num_input_files;      // every range reads the same files
        st.total_input_bytes = us.total_input_bytes;
      }
      auto& js = r->job_stats;
      js.Reset();
      js.num_input_records = st.num_input_records;
      js.num_output_records = st.num_output_records;
      js.num_input_files = st.num_input_files;
      js.num_output_files = st.num_output_files;
      js.total_input_bytes = st.total_input_bytes;
      js.total_output_bytes = st.total_output_bytes;
      js.num_records_replaced = st.num_records_replaced;
      js.num_expired_deletion_records = st.num_expired_deletion_records;
      js.num_input_deletion_records = st.num_input_deletion_records;
      js.total_input_raw_key_bytes = st.total_input_raw_key_bytes;
      js.total_input_raw_value_bytes = st.total_input_raw_value_bytes;
      js.is_manual_compaction = p.manual_compaction;
      auto& cs = r->compaction_stats;
      cs.num_input_records = st.num_input_records;
      cs.num_output_records = st.num_output_records;
      cs.bytes_written = st.total_output_bytes;
      cs.num_output_files = (int)st.num_output_files;
      cs.count = 1;
      for (const auto& lvl : *p.inputs) {
        uint64_t b = 0;
        for (const FileMetaData* fm : lvl.files) b += fm->fd.GetFileSize();
        if (lvl.level == p.output_level) {
          cs.bytes_read_output_level += b;
          cs.num_input_files_in_output_level += (int)lvl.files.size();
        } else {
          cs.bytes_read_non_output_levels += b;
          cs.num_input_files_in_non_output_levels += (int)lvl.files.size();
        }
      }
      cs.num_dropped_records = st.num_input_records - st.num_output_records;
      r->statistics.tickers[COMPACT_READ_BYTES] = in_bytes;
      r->statistics.tickers[COMPACT_WRITE_BYTES] = st.total_output_bytes;
      r->statistics.tickers[LCOMPACT_WRITE_BYTES_RAW] = 0;
      const auto us = std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t0).count();
      js.elapsed_micros = (uint64_t)us;
      cs.micros = (uint64_t)us;
      r->work_time_usec = (size_t)us;
      r->curl_time_usec = r->mount_time_usec = r->prepare_time_usec = r->waiting_time_usec = 0;
      r->status = Status::OK();
    }
    for (b200c_job* u : units)
      if (u != job) b200c_job_destroy(u);  // sub-jobs first: they borrow their parents' input images
    for (b200c_job* pj : parents) b200c_job_destroy(pj);
    return s.ok() ? s : Fail(r, s);
  }

  Status RenameFile(const std::string& src, const std::string& dst, off_t fsize) override {
    FileSystem* fs = c_->immutable_options()->fs.get();
    IOStatus s = fs->RenameFile(src, dst, IOOptions(), nullptr);
    if (!s.ok()) {  // scratch directory on another file system: copy (synced), then drop the source
      Status c = CopyOneFile(src, dst, fsize);
      if (!c.ok()) return c;
      fs->DeleteFile(src, IOOptions(), nullptr).PermitUncheckedError();
    }
    renamed_dirs_.insert(DirOf(dst));
    return Status::OK();
  }
  Status CopyOneFile(const std::string& src, const std::string& dst, off_t) override {
    FileSystem* fs = c_->immutable_options()->fs.get();
    uint64_t size = 0;
    IOStatus s = fs->GetFileSize(src, IOOptions(), &size, nullptr);
    if (!s.ok()) return s;
    std::unique_ptr<char[]> buf(new char[size ? size : 1]);
    s = ReadFileFS(fs, src, buf.get(), size);
    if (s.ok()) s = WriteFileFS(fs, dst, buf.get(), size, c_->immutable_options()->use_fsync);
    return s;
  }
  // RunRemote calls this after the last rename and before Install(): the destination directories are synced here (the local path
  // syncs the output directory at the end of CompactionJob::Run, compaction_job.cc:766), then the scratch directory goes away
  void CleanFiles(const CompactionParams&, const CompactionResults& r) override {
    FileSystem* fs = c_->immutable_options()->fs.get();
    for (const auto& d : renamed_dirs_) SyncDirFS(fs, d).PermitUncheckedError();
    renamed_dirs_.clear();
    if (!r.output_dir.empty()) fs->DeleteDir(r.output_dir, IOOptions(), nullptr).PermitUncheckedError();  // outputs were renamed away
  }

 private:
  static Status Fail(CompactionResults* r, const Status& s) {
    r->status = s;
    return s;
  }
  B200CompactOptions opt_;
  const Compaction* c_;
  std::set<std::string> renamed_dirs_;  // directories that received an output file of this job
};

}  // namespace

B200CompactionExecutorFactory::B200CompactionExecutorFactory(const B200CompactOptions& o) : opt_(o) {
  have_device_ = b200c_device_count() > opt_.device;
  if (have_device_) {
    // create the device context now (hundreds of milliseconds) instead of inside the first compaction job; the buffer goes to the
    // library's cache of pinned memory
    void* p = nullptr;
    if (b200c_host_alloc(opt_.device, 1 << 20, &p) == B200C_OK) b200c_host_free(p);
  }
}
B200CompactionExecutorFactory::~B200CompactionExecutorFactory() = default;

// Why a job has to stay on the reference's own CPU path (nullptr: the device takes it).  Everything here is decided from the job's
// OPTIONS and metadata; data-dependent reasons (a Merge / SingleDelete record, a long key) surface later as Status::NotSupported from
// Execute().  The list errs on the side of running locally: an option that changes what CompactionIterator, CompactionOutputs or the
// table builder do and that the device does not implement must keep the reference's own behaviour.
static const char* WhyLocal(const Compaction* c) {
  const auto* io = c->immutable_options();
  const auto* mo = c->mutable_cf_options();
  if (io->merge_operator != nullptr) return "merge operator";
  // RunRemote needs the filter to come from a factory (compaction_job.cc:942-943); only filters the merge kernel implements run remotely
  if (io->compaction_filter != nullptr) return "compaction filter object (not a factory)";
  if (io->compaction_filter_factory != nullptr && DeviceFilterOf(c) == B200C_FILTER_NONE) return "compaction filter the device does not implement";
  if (io->user_comparator != BytewiseComparator()) return "comparator other than the bytewise one (incl. user-defined timestamps)";
  if (c->output_compression() != kNoCompression) return "block compression";
  if (DevicePartitionerPrefixLen(c) < 0) return "sst partitioner";
  if (io->allow_ingest_behind) return "allow_ingest_behind (no sequence-number zeroing, compaction_iterator.cc:1299-1304)";
  if (io->preclude_last_level_data_seconds > 0 || io->preserve_internal_time_seconds > 0)
    return "seqno-to-time preservation (preserve_time_min_seqno_, per-key placement)";
  if (c->SupportsPerKeyPlacement()) return "per-key placement (penultimate level output)";
  if (mo->enable_blob_files) return "blob files (large values are extracted while compacting)";
  if (!io->table_properties_collector_factories.empty()) return "user table-properties collectors";
  if (mo->sample_for_compression > 0) return "sample_for_compression (adds table properties)";
  if (HasHostOnlyFileCutRule(c)) return "an output-file cut rule the device does not evaluate (TTL cut / round-robin split)";
  const BlockBasedTableOptions* t = BlockBasedOptionsOf(c);
  if (t == nullptr) return "table factory other than BlockBasedTable";
  if (DeviceBloomMillibits(c, t) < 0) return "filter policy other than a full Bloom filter over whole keys (format_version >= 5)";
  if (t->index_type != BlockBasedTableOptions::kBinarySearch || t->data_block_index_type != BlockBasedTableOptions::kDataBlockBinarySearch ||
      t->index_block_restart_interval != 1 || t->block_align || t->format_version < 3 || t->format_version > 5 ||
      (t->checksum != kXXH3 && t->checksum != kCRC32c && t->checksum != kNoChecksum))
    return "BlockBasedTableOptions outside the device's format subset";
  size_t runs = 0, files = 0;  // sorted runs as MakeInputIterator forms them: every L0 file, every deeper level (version_set.cc:7311-7352)
  for (const auto& lvl : *c->inputs()) {
    files += lvl.files.size();
    runs += lvl.level == 0 ? lvl.files.size() : (lvl.files.empty() ? 0 : 1);
    for (const FileMetaData* fm : lvl.files)
      if (fm->num_range_deletions) return "range tombstones in an input file";
  }
  if (files == 0) return "no input files";
  if (runs > 64) return "more than 64 sorted runs (L0 files + levels)";
  return nullptr;
}

bool B200CompactionExecutorFactory::ShouldRunLocal(const Compaction* c) const {
  const char* why = WhyLocal(c);
  if (getenv("B200C_PLUGIN_TRACE") != nullptr)  // one line per job: where it runs and why
    fprintf(stderr, "B200Compact: job L%d -> L%d: %s%s\n", c->start_level(), c->output_level(), why ? why : "device-eligible",
            have_device_ ? "" : " [no CUDA device: runs locally]");
  return !have_device_ || why != nullptr;
}
bool B200CompactionExecutorFactory::AllowFallbackToLocal() const { return opt_.allow_fallback_to_local; }
CompactionExecutor* B200CompactionExecutorFactory::NewExecutor(const Compaction* c) const {
  return new B200CompactionExecutor(opt_, c);
}
const char* B200CompactionExecutorFactory::Name() const { return "B200Compact"; }
std::string B200CompactionExecutorFactory::JobUrl(const std::string& dbname, int job_id, int attempt) const {
  return "b200c://cuda:" + std::to_string(opt_.device) + "/" + dbname + "/job-" + std::to_string(job_id) + "/att-" +
         std::to_string(attempt);
}

std::shared_ptr<CompactionExecutorFactory> NewB200CompactionExecutorFactory(const B200CompactOptions& o) {
  return std::make_shared<B200CompactionExecutorFactory>(o);
}

#ifdef B200C_WITH_SIDEPLUGIN
// rockside registration (sideplugin/rockside/src/topling/side_plugin_factory.h:290-293): selectable from JSON/YAML as
//   "CompactionExecutorFactory": { "b200": { "class": "B200Compact", "params": { "device": 0 } } }
}  // namespace ROCKSDB_NAMESPACE
#include "topling/side_plugin_factory.h"
namespace ROCKSDB_NAMESPACE {
static std::shared_ptr<CompactionExecutorFactory> JS_NewB200Compact(const json& js, const SidePluginRepo&) {
  B200CompactOptions o;
  ROCKSDB_JSON_OPT_PROP_3(js, o.device, "device");
  ROCKSDB_JSON_OPT_PROP_3(js, o.allow_fallback_to_local, "allow_fallback_to_local");
  ROCKSDB_JSON_OPT_PROP_3(js, o.verify_input_checksums, "verify_input_checksums");
  ROCKSDB_JSON_OPT_PROP_3(js, o.scratch_dir, "scratch_dir");
  ROCKSDB_JSON_OPT_PROP_3(js, o.io_threads, "io_threads");
  ROCKSDB_JSON_OPT_PROP_3(js, o.max_subcompactions, "max_subcompactions");
  ROCKSDB_JSON_OPT_PROP_3(js, o.devices, "devices");
  return std::make_shared<B200CompactionExecutorFactory>(o);
}
ROCKSDB_FACTORY_REG("B200Compact", JS_NewB200Compact);
#endif

}  // namespace ROCKSDB_NAMESPACE
