// oracle_backed_latency_info.cpp — TEST INFRASTRUCTURE ONLY: eppscore_predict_latency for the oracle-backed stand-in of the C ABI,
// so that the host layer's LatencyPredictionInfo and dispatch record run in the `-m "not gpu"` suite.  It includes
// oracle_backed_prefix_match.cpp (link this file instead of that one).  Each entry is orc_latency_predict + orc_latency_validate
// at the listed endpoint, fed the stand-in's snapshot and the oracle's matchLongestPrefix; host arrays only.
// oracle_backed_predict_latency_calls counts the calls.
#include <cmath>

#include "oracle_backed_prefix_match.cpp"

extern "C" {

int64_t oracle_backed_predict_latency_calls = 0;

int32_t eppscore_predict_latency(eppscore_engine* e, int32_t R, int32_t k, int32_t location, const uint64_t* hashes, const uint16_t* n_hashes,
                                 int32_t hash_stride, const int32_t* input_tokens, const double* ttft_slo, const double* tpot_slo,
                                 const int32_t* endpoints, eppscore_latency_info* info_out, uint16_t* match_out, void*) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (location != 0) return fail(e, EPPSCORE_ERR_INVALID, "the stand-in takes host arrays only");
  if (k < 1 || k > e->cfg.max_endpoints) return fail(e, EPPSCORE_ERR_INVALID, "predict_latency: k must be in [1, max_endpoints]");
  if (R < 0 || (R > 0 && (!hashes || !n_hashes || !endpoints || !info_out))) return fail(e, EPPSCORE_ERR_INVALID, "NULL argument");
  if (!e->have_snapshot || !e->have_lat) return fail(e, EPPSCORE_ERR_INVALID, "no snapshot, or no latency params");
  if (R > 0 && hash_stride <= 0) return fail(e, EPPSCORE_ERR_INVALID, "hash_stride must be > 0");
  oracle_backed_predict_latency_calls++;
  const int32_t limit = e->cfg.max_endpoints;
  std::vector<uint16_t> m((size_t)limit);
  for (int32_t r = 0; r < R; r++) {
    if (n_hashes[r] > hash_stride) return fail(e, EPPSCORE_ERR_INVALID, "n_hashes exceeds hash_stride");
    orc_match_longest_prefix(e->idx, hashes + (size_t)r * hash_stride, n_hashes[r], limit, m.data());
    for (int32_t j = 0; j < k; j++) {
      const int32_t ep = endpoints[(size_t)r * k + j];
      const uint16_t c = (ep >= 0 && ep < limit) ? m[(size_t)ep] : 0;
      if (match_out) match_out[(size_t)r * k + j] = c;
      eppscore_latency_info& o = info_out[(size_t)r * k + j];
      o = eppscore_latency_info{};
      if (!e->lat.has_predictions || ep < 0 || ep >= e->M) continue;
      double prefix = (double)c / (double)n_hashes[r];  // preparedata_hooks.go:44-56: NaN => 0
      if (std::isnan(prefix)) prefix = 0.0;
      double ttft, tpot, hr[2];
      int32_t ok[3];
      orc_latency_predict(&e->lat, e->kv[(size_t)ep], input_tokens ? input_tokens[r] : 0, e->queue[(size_t)ep], e->running[(size_t)ep], 1,
                          prefix, &ttft, &tpot);
      const int neutral = !e->lat.streaming_mode || (e->have_prefill && e->prefill[(size_t)ep]);
      orc_latency_validate(&e->lat, ttft, tpot, ttft_slo ? ttft_slo[r] : 0.0, tpot_slo ? tpot_slo[r] : 0.0,
                           e->have_min_tpot ? e->min_tpot[(size_t)ep] : 0.0, neutral, ok, hr);
      o.ttft = ttft;
      o.tpot = tpot;
      o.ttft_headroom = hr[1];
      o.tpot_headroom = hr[0];
      o.prefix_cache_score = prefix;
      o.dispatched = e->have_dispatched ? e->dispatched[(size_t)ep] : 0;
      o.present = 1;
      o.ttft_valid = (uint8_t)ok[0];
      o.tpot_valid = (uint8_t)ok[1];
    }
  }
  return EPPSCORE_OK;
}

}  // extern "C"
