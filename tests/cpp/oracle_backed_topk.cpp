// oracle_backed_topk.cpp — TEST INFRASTRUCTURE ONLY: eppscore_schedule_batch_topk for the oracle-backed stand-in of the
// C ABI (oracle_backed_abi.cpp), so that the host layer's top-k route (Scheduler with maxNumOfEndpoints 2..8, every picker)
// runs in the `-m "not gpu"` suite.  The weighted score map comes from the stand-in's eppscore_schedule_batch, the order
// from tests/cpp/topk_oracle.c.  The stand-in keeps its engine state private, so the profile (pick mode, tie mode, seed)
// and the snapshot's M are recorded on the way in: link with -Wl,--wrap=eppscore_create -Wl,--wrap=eppscore_set_snapshot.
#include <map>
#include <mutex>
#include <vector>

#include "../../include/eppscore.h"

extern "C" {
int32_t topk_oracle_pick(const double* weighted, int32_t M, int32_t pick_mode, int32_t tie_mode, uint64_t tie_seed,
                         int64_t request_index, int32_t k, int32_t* m_out, double* score_out);
int32_t __real_eppscore_create(int32_t device, const eppscore_config* cfg, eppscore_engine** out);
int32_t __real_eppscore_set_snapshot(eppscore_engine* e, const eppscore_snapshot* s);
}

namespace {
struct Seen {
  eppscore_config cfg{};
  int32_t M = 0;
};
std::mutex g_mu;
std::map<const eppscore_engine*, Seen> g_seen;
}  // namespace

extern "C" {

int32_t __wrap_eppscore_create(int32_t device, const eppscore_config* cfg, eppscore_engine** out) {
  const int32_t rc = __real_eppscore_create(device, cfg, out);
  if (rc == EPPSCORE_OK) {
    std::lock_guard<std::mutex> lk(g_mu);
    g_seen[*out] = Seen{*cfg, 0};
  }
  return rc;
}

int32_t __wrap_eppscore_set_snapshot(eppscore_engine* e, const eppscore_snapshot* s) {
  const int32_t rc = __real_eppscore_set_snapshot(e, s);
  if (rc == EPPSCORE_OK) {
    std::lock_guard<std::mutex> lk(g_mu);
    g_seen[e].M = s->M;
  }
  return rc;
}

int32_t eppscore_schedule_batch_topk(eppscore_engine* e, const eppscore_batch* b, const eppscore_topk* t) {
  if (!e || !b || b->struct_size != sizeof(*b)) return EPPSCORE_ERR_INVALID;
  if (!t || t->struct_size != sizeof(*t) || t->k < 1 || t->k > EPPSCORE_MAX_TOPK || !t->endpoints || !t->scores)
    return EPPSCORE_ERR_INVALID;
  if (b->R <= 0) return EPPSCORE_OK;
  Seen seen;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    seen = g_seen[e];
  }
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
