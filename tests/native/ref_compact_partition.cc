// tests/native/ref_compact_partition.cc — test infrastructure: the reference driver oracle/ref_compact.cc, compiled from its own source,
// with two more column-family options for the fixed-prefix SST partitioner tests:
//   partitioner_prefix_len=N   ColumnFamilyOptions::sst_partitioner_factory = NewSstPartitionerFixedPrefixFactory(N) (0: none)
//   dynamic_file_size=0|1      ColumnFamilyOptions::level_compaction_dynamic_file_size (default 1)
// Every other argument goes to the driver unchanged.  The driver builds its Options inside main(); the two options are set where it
// installs the table factory, before any DB is opened, so the manifest it writes reports them as the DB saw them.
// Built by tests/native/ref_partition.mk (with -DWITH_B200_PLUGIN: the same driver with the B200 executor plugin).
#include <dirent.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "env/composite_env_wrapper.h"
#include "rocksdb/compaction_filter.h"
#include "rocksdb/db.h"
#include "rocksdb/filter_policy.h"
#include "rocksdb/listener.h"
#include "rocksdb/options.h"
#include "rocksdb/sst_partitioner.h"
#include "rocksdb/system_clock.h"
#include "rocksdb/table.h"
#include "rocksdb/utilities/db_ttl.h"
#include "rocksdb/write_batch.h"
#include "util/compression.h"
#include "utilities/compaction_filters/remove_emptyvalue_compactionfilter.h"
#ifdef WITH_B200_PLUGIN
#include "rocksdb/statistics.h"
#include "toplingdb_b200/plugin/b200_compaction_executor.h"
#include "toplingdb_b200/plugin/b200_table_factory.h"
#endif

namespace {
uint32_t g_partitioner_prefix_len = 0;
int g_dynamic_file_size = 1;
void ApplyCfOptions(ROCKSDB_NAMESPACE::Options& opt) {
  opt.level_compaction_dynamic_file_size = g_dynamic_file_size != 0;
  if (g_partitioner_prefix_len) opt.sst_partitioner_factory = ROCKSDB_NAMESPACE::NewSstPartitionerFixedPrefixFactory(g_partitioner_prefix_len);
}
}  // namespace

// (the headers above are in already: the two names are replaced in the driver's own code only)
#define main ref_compact_main
#define NewBlockBasedTableFactory(t) (ApplyCfOptions(opt), ROCKSDB_NAMESPACE::NewBlockBasedTableFactory(t))
#include "oracle/ref_compact.cc"
#undef NewBlockBasedTableFactory
#undef main

int main(int argc, char** argv) {
  std::vector<char*> args;
  for (int i = 0; i < argc; i++) {
    const char* a = argv[i];
    if (i >= 3 && strncmp(a, "partitioner_prefix_len=", 23) == 0) g_partitioner_prefix_len = (uint32_t)strtoul(a + 23, nullptr, 0);
    else if (i >= 3 && strncmp(a, "dynamic_file_size=", 18) == 0) g_dynamic_file_size = atoi(a + 18);
    else args.push_back(argv[i]);
  }
  args.push_back(nullptr);
  return ref_compact_main((int)args.size() - 1, args.data());
}
