// oracle_backed_topk_wide.cpp — TEST INFRASTRUCTURE ONLY: eppscore_schedule_batch_topk_wide for the oracle-backed stand-in of
// the C ABI, next to eppscore_schedule_batch_topk, so that the host layer's wide route (Scheduler with maxNumOfEndpoints > 8)
// runs in the `-m "not gpu"` suite.  It reuses oracle_backed_topk.cpp's recording of the profile (the same link-time
// wrapping: -Wl,--wrap=eppscore_create -Wl,--wrap=eppscore_set_snapshot), so link this file instead of that one.  Calls are
// counted in oracle_backed_topk_wide_calls, so a test can tell which route the host layer took.
#include "oracle_backed_topk.cpp"

extern "C" {

int64_t oracle_backed_topk_wide_calls = 0;

int32_t eppscore_schedule_batch_topk_wide(eppscore_engine* e, const eppscore_batch* b, const eppscore_topk* t) {
  if (!e || !b || b->struct_size != sizeof(*b)) return EPPSCORE_ERR_INVALID;
  Seen seen;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    seen = g_seen[e];
  }
  if (!t || t->struct_size != sizeof(*t) || t->k < 1 || t->k > seen.cfg.max_endpoints || !t->endpoints || !t->scores)
    return EPPSCORE_ERR_INVALID;
  oracle_backed_topk_wide_calls++;
  if (b->R <= 0) return EPPSCORE_OK;
  std::vector<double> weighted;  // the weighted score map of every request, NaN for non-candidates
  eppscore_batch bb = *b;
  if (!bb.scores_out) {
    weighted.resize((size_t)b->R * (size_t)seen.M);
    bb.scores_out = weighted.data();
  }
  const int32_t rc = eppscore_schedule_batch(e, &bb);
  if (rc != EPPSCORE_OK) return rc;
  for (int32_t r = 0; r < b->R; r++)
    topk_oracle_pick(bb.scores_out + (size_t)r * seen.M, seen.M, seen.cfg.pick_mode, seen.cfg.tie_mode, seen.cfg.tie_seed,
                     b->request_base + r, t->k, t->endpoints + (size_t)r * t->k, t->scores + (size_t)r * t->k);
  return EPPSCORE_OK;
}

}  // extern "C"
