// tests/native/ref_compact_zlib.cc — test infrastructure: the reference driver oracle/ref_compact.cc, compiled from its own source,
// with the zlib CompressionOptions of the job's input files (flushes and set-up compactions, input_compression=zlib):
//   zlib_level=N                    CompressionOptions::level (default: Z_DEFAULT_COMPRESSION; 0 writes stored deflate blocks)
//   zlib_strategy=N                 CompressionOptions::strategy (0 default, 1 filtered, 2 Huffman only, 3 RLE, 4 fixed)
//   zlib_window_bits=N              CompressionOptions::window_bits (-9 ... -15; default -14)
//   max_compressed_bytes_per_kb=N   CompressionOptions::max_compressed_bytes_per_kb (default 896; above 1024 stored streams are kept)
//   max_dict_bytes=N                CompressionOptions::max_dict_bytes (> 0: the tables carry a compression dictionary)
// Every other argument goes to the driver unchanged.  The options are set where the driver installs the table factory, before any
// DB is opened, and are reset to their defaults before the measured job, which writes uncompressed outputs.
// Built by tests/native/ref_zlib.mk (with -DWITH_B200_PLUGIN: the same driver with the B200 executor plugin).
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
ROCKSDB_NAMESPACE::CompressionOptions g_zlib_opts;
void ApplyCfOptions(ROCKSDB_NAMESPACE::Options& opt) { opt.compression_opts = g_zlib_opts; }
// The measured job writes uncompressed outputs, but their rocksdb.compression_options property spells out the column family's
// CompressionOptions.  Once the inputs are written (the driver's first look at the DB's files after the script), the options go back
// to their defaults, so the job's outputs are the files a DB with default options writes from these inputs.
bool g_reset_done = false;
void ResetCompressionOptions(ROCKSDB_NAMESPACE::DB* db) {
  if (g_reset_done) return;
  g_reset_done = true;
  ROCKSDB_NAMESPACE::Status s = db->SetOptions({{"compression_opts", "{window_bits=-14;level=32767;strategy=0;max_dict_bytes=0;"
                                                                      "max_compressed_bytes_per_kb=896}"}});
  if (!s.ok()) {
    fprintf(stderr, "ref_compact_zlib: SetOptions(compression_opts): %s\n", s.ToString().c_str());
    exit(2);
  }
}
}  // namespace

// (the headers above are in already: the names are replaced in the driver's own code only)
#define main ref_compact_main
#define NewBlockBasedTableFactory(t) (ApplyCfOptions(opt), ROCKSDB_NAMESPACE::NewBlockBasedTableFactory(t))
#define GetColumnFamilyMetaData(m) GetColumnFamilyMetaData((ResetCompressionOptions(db), (m)))
#include "oracle/ref_compact.cc"
#undef GetColumnFamilyMetaData
#undef NewBlockBasedTableFactory
#undef main

int main(int argc, char** argv) {
  std::vector<char*> args;
  auto opt = [](const char* a, const char* name, int* v) {
    const size_t n = strlen(name);
    if (strncmp(a, name, n) != 0 || a[n] != '=') return false;
    *v = (int)strtol(a + n + 1, nullptr, 0);
    return true;
  };
  ROCKSDB_NAMESPACE::CompressionOptions& z = g_zlib_opts;
  int dict = 0;
  for (int i = 0; i < argc; i++) {
    const char* a = argv[i];
    if (i >= 3 && (opt(a, "zlib_level", &z.level) || opt(a, "zlib_strategy", &z.strategy) || opt(a, "zlib_window_bits", &z.window_bits) ||
                   opt(a, "max_compressed_bytes_per_kb", &z.max_compressed_bytes_per_kb) || opt(a, "max_dict_bytes", &dict)))
      continue;
    args.push_back(argv[i]);
  }
  z.max_dict_bytes = (uint32_t)dict;
  if (z.window_bits < -15 || z.window_bits > -9) {
    fprintf(stderr, "ref_compact_zlib: zlib_window_bits=%d outside -15 ... -9 (raw deflate)\n", z.window_bits);
    return 1;
  }
  args.push_back(nullptr);
  return ref_compact_main((int)args.size() - 1, args.data());
}
