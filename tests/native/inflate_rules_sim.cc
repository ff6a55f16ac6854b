// tests/native/inflate_rules_sim.cc — toplingdb_b200/csrc/inflate_rules.h compiled for the host (test infrastructure)
#include "inflate_rules.h"
extern "C" long inflate_sim(const uint8_t* src, uint32_t n, uint8_t* dst, uint32_t cap) {
  b200c::InfWork wk;
  return b200c::inflate_raw(src, n, dst, cap, &wk);
}
extern "C" int size_prefix_sim(const uint8_t* p, uint32_t size, uint64_t* u) { return b200c::inf_size_prefix(p, size, u); }
