// engine_inorder_index_shim.cpp — TEST INFRASTRUCTURE ONLY: what host_inorder_index_test.cpp reads from its engine, for a build
// against the real libeppscore.so (the GPU run of the host program): the calls are counted through -Wl,--wrap of
// eppscore_schedule_batch_inorder_index and eppscore_commit_picks, and the index is read through the C ABI.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../include/eppscore.h"

uint64_t g_inorder_index_calls = 0;
uint64_t g_host_commits = 0;

extern "C" {
int32_t __real_eppscore_schedule_batch_inorder_index(eppscore_engine* e, const eppscore_batch* b, const int64_t* tokens,
                                                     const eppscore_inorder_index* x);
int32_t __wrap_eppscore_schedule_batch_inorder_index(eppscore_engine* e, const eppscore_batch* b, const int64_t* tokens,
                                                     const eppscore_inorder_index* x) {
  g_inorder_index_calls++;
  return __real_eppscore_schedule_batch_inorder_index(e, b, tokens, x);
}
int32_t __real_eppscore_commit_picks(eppscore_engine* e, int32_t R, const int32_t* pick, const uint64_t* hashes, const uint16_t* n_hashes,
                                     int32_t hash_stride, const int32_t* lru_capacity);
int32_t __wrap_eppscore_commit_picks(eppscore_engine* e, int32_t R, const int32_t* pick, const uint64_t* hashes, const uint16_t* n_hashes,
                                     int32_t hash_stride, const int32_t* lru_capacity) {
  g_host_commits++;
  return __real_eppscore_commit_picks(e, R, pick, hashes, n_hashes, hash_stride, lru_capacity);
}
}

std::vector<uint64_t> StandInLruKeys(eppscore_engine* e, int32_t endpoint) {
  const int32_t n = eppscore_prefix_lru_len(e, endpoint);
  std::vector<uint64_t> k((size_t)std::max(n, 0));
  if (n > 0) eppscore_prefix_lru_keys(e, endpoint, k.data(), n);
  return k;
}
int64_t StandInNumHashes(eppscore_engine* e) {
  eppscore_stats s{};
  s.struct_size = sizeof(s);
  eppscore_get_stats(e, &s);
  return s.prefix_live_hashes;
}
