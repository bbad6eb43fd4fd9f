// oracle_backed_prefix_match.cpp — TEST INFRASTRUCTURE ONLY: eppscore_prefix_match for the oracle-backed stand-in of the C ABI,
// so that the host layer's PrefixCacheMatchInfo and prefix-indexer metrics run in the `-m "not gpu"` suite.  It includes
// oracle_backed_profiles_topk.cpp (link this file instead of that one).  Each entry is the oracle's matchLongestPrefix
// (orc_match_longest_prefix) read at the listed endpoint; host arrays only.  oracle_backed_prefix_match_calls counts the calls.
#include "oracle_backed_profiles_topk.cpp"

extern "C" {

int64_t oracle_backed_prefix_match_calls = 0;

int32_t eppscore_prefix_match(eppscore_engine* e, int32_t R, int32_t k, int32_t location, const uint64_t* hashes, const uint16_t* n_hashes,
                              int32_t hash_stride, const int32_t* endpoints, uint16_t* match_out, void*) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (location != 0) return fail(e, EPPSCORE_ERR_INVALID, "the stand-in takes host arrays only");
  if (k < 1 || k > e->cfg.max_endpoints) return fail(e, EPPSCORE_ERR_INVALID, "prefix_match: k must be in [1, max_endpoints]");
  if (R < 0 || (R > 0 && (!hashes || !n_hashes || !endpoints || !match_out))) return fail(e, EPPSCORE_ERR_INVALID, "NULL argument");
  if (R > 0 && hash_stride <= 0) return fail(e, EPPSCORE_ERR_INVALID, "hash_stride must be > 0");
  oracle_backed_prefix_match_calls++;
  const int32_t limit = e->cfg.max_endpoints;
  std::vector<uint16_t> m((size_t)limit);
  for (int32_t r = 0; r < R; r++) {
    if (n_hashes[r] > hash_stride) return fail(e, EPPSCORE_ERR_INVALID, "n_hashes exceeds hash_stride");
    orc_match_longest_prefix(e->idx, hashes + (size_t)r * hash_stride, n_hashes[r], limit, m.data());
    for (int32_t j = 0; j < k; j++) {
      const int32_t ep = endpoints[(size_t)r * k + j];
      match_out[(size_t)r * k + j] = (ep >= 0 && ep < limit) ? m[(size_t)ep] : 0;
    }
  }
  return EPPSCORE_OK;
}

}  // extern "C"
