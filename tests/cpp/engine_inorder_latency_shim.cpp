// engine_inorder_latency_shim.cpp — TEST INFRASTRUCTURE ONLY: what host_inorder_latency_test.cpp reads from its engine, for a
// build against the real libeppscore.so (the GPU run of the host program): the calls are counted through -Wl,--wrap of
// eppscore_schedule_batch_inorder_latency and eppscore_running_add, and the index is read through the C ABI.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../include/eppscore.h"

uint64_t g_inorder_latency_calls = 0;
uint64_t g_host_running_adds = 0;

extern "C" {
int32_t __real_eppscore_schedule_batch_inorder_latency(eppscore_engine* e, const eppscore_batch* b, const int64_t* tokens,
                                                       const eppscore_inorder_index* x, const eppscore_inorder_running* q);
int32_t __wrap_eppscore_schedule_batch_inorder_latency(eppscore_engine* e, const eppscore_batch* b, const int64_t* tokens,
                                                       const eppscore_inorder_index* x, const eppscore_inorder_running* q) {
  g_inorder_latency_calls++;
  return __real_eppscore_schedule_batch_inorder_latency(e, b, tokens, x, q);
}
int32_t __real_eppscore_running_add(eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint,
                                    const uint64_t* request_key, const double* tpot_slo, uint8_t* added_out, void* stream);
int32_t __wrap_eppscore_running_add(eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint,
                                    const uint64_t* request_key, const double* tpot_slo, uint8_t* added_out, void* stream) {
  g_host_running_adds++;
  return __real_eppscore_running_add(e, R, location, endpoint, request_key, tpot_slo, added_out, stream);
}
}

std::vector<uint64_t> StandInLruKeys(eppscore_engine* e, int32_t endpoint) {
  const int32_t n = eppscore_prefix_lru_len(e, endpoint);
  std::vector<uint64_t> k((size_t)std::max(n, 0));
  if (n > 0) eppscore_prefix_lru_keys(e, endpoint, k.data(), n);
  return k;
}
