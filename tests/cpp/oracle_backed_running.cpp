// oracle_backed_running.cpp — TEST INFRASTRUCTURE ONLY: the running-request queue entry points (eppscore_running_*) for the
// oracle-backed stand-in of the C ABI (oracle_backed_abi.cpp), so that the host layer's TrackRunningRequests runs in the
// `-m "not gpu"` suite.  The queues come from tests/cpp/running_oracle.c.  The stand-in keeps its engine state private, so
// the config is recorded on the way in, and a snapshot without min_tpot_slo / dispatched reaches the stand-in with the
// queues' view when the profile has the latency scorer — the engine's source rule, field by field: link with
// -Wl,--wrap=eppscore_create -Wl,--wrap=eppscore_set_snapshot.
#include <cmath>
#include <map>
#include <mutex>
#include <vector>

#include "../../include/eppscore.h"

extern "C" {
void* orc_running_new(int32_t n_ep);
void orc_running_add(void* h, int32_t R, const int32_t* ep, const uint64_t* key, const double* tpot, uint8_t* added);
void orc_running_remove(void* h, int32_t R, const int32_t* ep, const uint64_t* key, uint8_t* removed);
void orc_running_remove_endpoint(void* h, int32_t ep);
void orc_running_get(void* h, int32_t M, double* min_out, int32_t* count_out);
int32_t __real_eppscore_create(int32_t device, const eppscore_config* cfg, eppscore_engine** out);
int32_t __real_eppscore_set_snapshot(eppscore_engine* e, const eppscore_snapshot* s);
}

namespace {
struct Seen {
  eppscore_config cfg{};
  void* queues = nullptr;  // never freed: one per engine of a short-lived test program
};
std::mutex g_mu;
std::map<const eppscore_engine*, Seen> g_seen;

Seen* seen(const eppscore_engine* e) {
  auto it = g_seen.find(e);
  return it == g_seen.end() ? nullptr : &it->second;
}
}  // namespace

extern "C" {

int32_t __wrap_eppscore_create(int32_t device, const eppscore_config* cfg, eppscore_engine** out) {
  const int32_t rc = __real_eppscore_create(device, cfg, out);
  if (rc == EPPSCORE_OK) {
    std::lock_guard<std::mutex> lk(g_mu);
    g_seen[*out] = Seen{*cfg, orc_running_new(cfg->max_endpoints)};
  }
  return rc;
}

int32_t __wrap_eppscore_set_snapshot(eppscore_engine* e, const eppscore_snapshot* s) {
  std::vector<double> mn;
  std::vector<int32_t> cnt;
  eppscore_snapshot sub;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    Seen* x = seen(e);
    bool latency = false;
    if (x)
      for (int i = 0; i < x->cfg.n_scorers; i++) latency = latency || x->cfg.scorer_kind[i] == EPPSCORE_SCORER_LATENCY;
    if (!x || !s || s->struct_size != sizeof(*s) || !latency || s->M <= 0 || (s->min_tpot_slo && s->dispatched))
      return __real_eppscore_set_snapshot(e, s);
    mn.resize((size_t)s->M);
    cnt.resize((size_t)s->M);
    orc_running_get(x->queues, s->M, mn.data(), cnt.data());
    for (double& v : mn) v = v == 0.0 ? 0.0 : v;  // the engine stores a zero tpot as +0.0
    sub = *s;
  }
  if (!sub.min_tpot_slo) sub.min_tpot_slo = mn.data();
  if (!sub.dispatched) sub.dispatched = cnt.data();
  return __real_eppscore_set_snapshot(e, &sub);
}

static int32_t update(eppscore_engine* e, int op, int32_t R, int32_t location, const int32_t* endpoint, const uint64_t* key,
                      const double* tpot, uint8_t* out) {
  if (!e || R < 0 || (R > 0 && (!endpoint || !key)) || location != 0) return EPPSCORE_ERR_INVALID;
  std::lock_guard<std::mutex> lk(g_mu);
  Seen* x = seen(e);
  if (!x) return EPPSCORE_ERR_INVALID;
  for (int32_t r = 0; r < R; r++)
    if (endpoint[r] >= x->cfg.max_endpoints || (tpot && std::isnan(tpot[r]))) return EPPSCORE_ERR_INVALID;
  if (op == 0) orc_running_add(x->queues, R, endpoint, key, tpot, out);
  else orc_running_remove(x->queues, R, endpoint, key, out);
  return EPPSCORE_OK;
}

int32_t eppscore_running_add(eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint, const uint64_t* request_key,
                             const double* tpot_slo, uint8_t* added_out, void*) {
  return update(e, 0, R, location, endpoint, request_key, tpot_slo, added_out);
}

int32_t eppscore_running_remove(eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint,
                                const uint64_t* request_key, uint8_t* removed_out, void*) {
  return update(e, 1, R, location, endpoint, request_key, nullptr, removed_out);
}

int32_t eppscore_running_remove_endpoint(eppscore_engine* e, int32_t endpoint) {
  std::lock_guard<std::mutex> lk(g_mu);
  Seen* x = seen(e);
  if (!x || endpoint < 0 || endpoint >= x->cfg.max_endpoints) return EPPSCORE_ERR_INVALID;
  orc_running_remove_endpoint(x->queues, endpoint);
  return EPPSCORE_OK;
}

int32_t eppscore_running_get(eppscore_engine* e, double* min_tpot_out, int32_t* count_out, int32_t M) {
  std::lock_guard<std::mutex> lk(g_mu);
  Seen* x = seen(e);
  if (!x || M < 0 || M > x->cfg.max_endpoints) return EPPSCORE_ERR_INVALID;
  orc_running_get(x->queues, M, min_tpot_out, count_out);
  if (min_tpot_out)
    for (int32_t m = 0; m < M; m++) min_tpot_out[m] = min_tpot_out[m] == 0.0 ? 0.0 : min_tpot_out[m];
  return EPPSCORE_OK;
}

int32_t eppscore_running_reserve(eppscore_engine* e, int64_t live_entries) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (!seen(e) || live_entries < 0) return EPPSCORE_ERR_INVALID;
  return 1 << 29;  // the oracle's queues grow without bound
}

}  // extern "C"
