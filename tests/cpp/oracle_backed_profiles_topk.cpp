// oracle_backed_profiles_topk.cpp — TEST INFRASTRUCTURE ONLY: eppscore_schedule_batch_profiles_topk for the oracle-backed
// stand-in of the C ABI, so that the host layer's maxNumOfEndpoints lists per profile run in the `-m "not gpu"` suite.  It
// includes oracle_backed_profiles.cpp (link this file instead of that one).  Each run is the oracle's schedule_batch with the
// run's profile and mask = subset ∧ run mask (eppscore_schedule_batch_profiles of the stand-in, with the weighted score map
// asked for), and its list is tests/cpp/topk_oracle.c's order over that map with the profile's pick mode and tie seed.
#include "oracle_backed_profiles.cpp"

extern "C" {

int32_t topk_oracle_pick(const double* weighted, int32_t M, int32_t pick_mode, int32_t tie_mode, uint64_t tie_seed,
                         int64_t request_index, int32_t k, int32_t* m_out, double* score_out);

int64_t oracle_backed_profiles_topk_calls = 0;

int32_t eppscore_schedule_batch_profiles_topk(eppscore_engine* e, const eppscore_batch* b, int32_t n_runs, const eppscore_profile_run* runs,
                                              const eppscore_topk* topk) {
  if (!e || !b || !runs || !topk || n_runs < 1 || n_runs > EPPSCORE_MAX_PROFILES) return EPPSCORE_ERR_INVALID;
  for (int32_t i = 0; i < n_runs; i++) {
    const eppscore_topk& t = topk[i];
    if (t.struct_size != sizeof(t) || t.k < 0 || t.k > e->cfg.max_endpoints || (t.k > 0 && (!t.endpoints || !t.scores)))
      return fail(e, EPPSCORE_ERR_INVALID, "bad topk");
  }
  oracle_backed_profiles_topk_calls++;
  const int32_t M = e->M;
  std::vector<eppscore_profile_run> rr(runs, runs + n_runs);
  std::vector<std::vector<double>> weighted((size_t)n_runs);
  for (int32_t i = 0; i < n_runs; i++)
    if (topk[i].k > 0 && !rr[(size_t)i].scores_out) {
      weighted[(size_t)i].resize((size_t)b->R * (size_t)M);
      rr[(size_t)i].scores_out = weighted[(size_t)i].data();
    }
  const int32_t rc = eppscore_schedule_batch_profiles(e, b, n_runs, rr.data());
  if (rc != EPPSCORE_OK) return rc;
  Profiles ps;
  {
    std::lock_guard<std::mutex> lk(g_pmu);
    ps = profiles_of(e);
  }
  for (int32_t i = 0; i < n_runs; i++) {
    const eppscore_topk& t = topk[i];
    if (t.k <= 0) continue;
    const orc_profile& p = ps.prof[(size_t)rr[(size_t)i].profile];
    for (int32_t r = 0; r < b->R; r++)
      topk_oracle_pick(rr[(size_t)i].scores_out + (size_t)r * M, M, p.pick_mode, p.tie_mode, p.tie_seed, b->request_base + r, t.k,
                       t.endpoints + (size_t)r * t.k, t.scores + (size_t)r * t.k);
  }
  return EPPSCORE_OK;
}

}  // extern "C"
