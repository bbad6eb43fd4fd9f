// oracle_backed_profiles.cpp — TEST INFRASTRUCTURE ONLY: the multi-profile entry points (eppscore_add_profile,
// eppscore_set_profile_endpoints, eppscore_schedule_batch_profiles, eppscore_commit_picks_profiles) for the oracle-backed
// stand-in of the C ABI, so that the host layer's several-profile route runs in the `-m "not gpu"` suite.  It includes
// oracle_backed_abi.cpp (link this file instead of that one).  Each run is the oracle's schedule_batch with the run's profile
// (tie seed tie_seed ^ p * 0x9E3779B97F4A7C15) and mask = subset ∧ run mask; a commit applies indexer.Add per request in pick
// slot order.  One simplification: a subset applies at once, not at the next snapshot (the host layer sets it right before
// packing the snapshot).
#include <map>
#include <mutex>

#include "oracle_backed_abi.cpp"

namespace {
struct Profiles {
  std::vector<orc_profile> prof;               // [0] = the create profile, recorded at first use
  std::vector<std::vector<uint32_t>> subset;   // empty: every endpoint
};
std::mutex g_pmu;
std::map<const eppscore_engine*, Profiles> g_prof;
Profiles& profiles_of(eppscore_engine* e) {
  Profiles& p = g_prof[e];
  if (p.prof.empty()) {
    p.prof.push_back(e->prof);
    p.subset.emplace_back();
  }
  return p;
}
}  // namespace

extern "C" {

orc_index* oracle_backed_index(eppscore_engine* e) { return e ? e->idx : nullptr; }

int32_t eppscore_add_profile(eppscore_engine* e, const eppscore_profile* p, int32_t* id_out) {
  if (!e || !p || p->struct_size != sizeof(*p) || !id_out) return EPPSCORE_ERR_INVALID;
  std::lock_guard<std::mutex> lk(g_pmu);
  Profiles& ps = profiles_of(e);
  if ((int)ps.prof.size() >= EPPSCORE_MAX_PROFILES) return fail(e, EPPSCORE_ERR_CAPACITY, "at most EPPSCORE_MAX_PROFILES profiles");
  if (p->n_scorers < 0 || p->n_scorers > EPPSCORE_MAX_SCORERS) return fail(e, EPPSCORE_ERR_INVALID, "n_scorers out of range");
  orc_profile o = e->prof;
  o.n_scorers = p->n_scorers;
  for (int i = 0; i < p->n_scorers; i++) {
    o.scorer_kind[i] = p->scorer_kind[i];
    o.scorer_weight[i] = p->scorer_weight[i];
  }
  o.pick_mode = p->pick_mode;
  o.n_filters = p->n_filters;
  for (int f = 0; f < p->n_filters && f < ORC_MAX_FILTERS; f++) {
    o.filter_kind[f] = p->filter_kind[f];
    for (int q = 0; q < 3; q++) o.filter_param[f][q] = p->filter_param[f][q];
  }
  const int32_t id = (int32_t)ps.prof.size();
  o.tie_seed = e->cfg.tie_seed ^ ((uint64_t)id * 0x9E3779B97F4A7C15ull);
  ps.prof.push_back(o);
  ps.subset.emplace_back();
  *id_out = id;
  return EPPSCORE_OK;
}

int32_t eppscore_set_profile_endpoints(eppscore_engine* e, int32_t profile, const uint32_t* mask, int32_t words) {
  if (!e) return EPPSCORE_ERR_INVALID;
  std::lock_guard<std::mutex> lk(g_pmu);
  Profiles& ps = profiles_of(e);
  if (profile < 0 || profile >= (int)ps.prof.size()) return fail(e, EPPSCORE_ERR_INVALID, "unknown profile");
  ps.subset[(size_t)profile].clear();
  if (mask) {
    ps.subset[(size_t)profile].assign((size_t)(e->cfg.max_endpoints + 31) / 32, 0u);
    for (int32_t w = 0; w < words && w < (int32_t)ps.subset[(size_t)profile].size(); w++) ps.subset[(size_t)profile][(size_t)w] = mask[w];
  }
  return EPPSCORE_OK;
}

int32_t eppscore_schedule_batch_profiles(eppscore_engine* e, const eppscore_batch* b, int32_t n_runs, const eppscore_profile_run* runs) {
  if (!e || !b || b->struct_size != sizeof(*b)) return EPPSCORE_ERR_INVALID;
  if (b->pick || b->pick_score || b->tie_count || b->cand_mask || b->scores_out || b->pred_out || b->filter_mask_out)
    return fail(e, EPPSCORE_ERR_INVALID, "per-profile batch fields must be NULL");
  if (n_runs < 1 || n_runs > EPPSCORE_MAX_PROFILES || !runs) return fail(e, EPPSCORE_ERR_INVALID, "n_runs out of range");
  Profiles ps;
  {
    std::lock_guard<std::mutex> lk(g_pmu);
    ps = profiles_of(e);
  }
  const orc_profile saved = e->prof;
  const int mw = (e->M + 31) / 32;
  int32_t rc = EPPSCORE_OK;
  for (int32_t i = 0; i < n_runs && rc == EPPSCORE_OK; i++) {
    const eppscore_profile_run& x = runs[i];
    if (x.struct_size != sizeof(x) || x.profile < 0 || x.profile >= (int)ps.prof.size()) {
      rc = fail(e, EPPSCORE_ERR_INVALID, "bad profile run");
      break;
    }
    eppscore_batch bb = *b;
    std::vector<uint32_t> mask;
    const auto& sub = ps.subset[(size_t)x.profile];
    if (x.cand_mask || !sub.empty()) {
      mask.assign((size_t)b->R * mw, 0xFFFFFFFFu);
      for (int32_t r = 0; r < b->R; r++)
        for (int w = 0; w < mw; w++) {
          uint32_t v = x.cand_mask ? x.cand_mask[(size_t)r * mw + w] : 0xFFFFFFFFu;
          if (!sub.empty()) v &= sub[(size_t)w];
          mask[(size_t)r * mw + w] = v;
        }
      bb.cand_mask = mask.data();
    }
    bb.pick = x.pick;
    bb.pick_score = x.pick_score;
    bb.tie_count = x.tie_count;
    bb.scores_out = x.scores_out;
    bb.pred_out = x.pred_out;
    bb.filter_mask_out = x.filter_mask_out;
    if (i > 0) {  // the profile-independent outputs come from the first run
      bb.total_blocks = nullptr;
      bb.hashes_out = nullptr;
      bb.match_blocks = nullptr;
    }
    e->prof = ps.prof[(size_t)x.profile];
    rc = eppscore_schedule_batch(e, &bb);
  }
  e->prof = saved;
  return rc;
}

int32_t eppscore_commit_picks_profiles(eppscore_engine* e, int32_t R, int32_t n_picks, const int32_t* const* picks, const uint64_t* hashes,
                                       const uint16_t* n_hashes, int32_t hash_stride, const int32_t* lru_capacity, int32_t location,
                                       int64_t, void*) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (location != 0) return fail(e, EPPSCORE_ERR_INVALID, "the stand-in takes host arrays only");
  if (n_picks < 1 || n_picks > EPPSCORE_MAX_PROFILES || (R > 0 && (!picks || !hashes || !n_hashes))) return fail(e, EPPSCORE_ERR_INVALID, "bad arguments");
  for (int32_t r = 0; r < R; r++)
    for (int32_t p = 0; p < n_picks; p++)
      if (picks[p][r] >= 0) orc_commit_picks(e->idx, 1, &picks[p][r], hashes + (size_t)r * hash_stride, n_hashes + r, hash_stride, lru_capacity);
  return EPPSCORE_OK;
}

}  // extern "C"
