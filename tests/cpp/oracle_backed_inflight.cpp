// oracle_backed_inflight.cpp — TEST INFRASTRUCTURE ONLY: the in-flight load producer's entry points (eppscore_estimate_tokens,
// eppscore_inflight_*) for the oracle-backed stand-in of the C ABI (oracle_backed_abi.cpp), so that the host layer's
// InFlightLoadProducer runs in the `-m "not gpu"` suite.  The counters and the estimate come from tests/cpp/inflight_oracle.c.
// The stand-in keeps its engine state private, so the profile is recorded on the way in, and a snapshot without
// inflight_tokens reaches the stand-in with the tracker's tokens when the profile has the token-load scorer — the engine's
// source rule: link with -Wl,--wrap=eppscore_create -Wl,--wrap=eppscore_set_snapshot.
#include <map>
#include <mutex>
#include <vector>

#include "../../include/eppscore.h"

extern "C" {
typedef struct orc_inflight orc_inflight;
int64_t orc_estimate_tokens(int64_t request_size_bytes, int32_t token_hint, int32_t prompt_chars);
orc_inflight* orc_inflight_new(void);
void orc_inflight_add(orc_inflight* t, int32_t R, const int32_t* endpoint, const int64_t* tokens);
void orc_inflight_release(orc_inflight* t, int32_t R, const int32_t* endpoint, const int64_t* tokens);
void orc_inflight_remove(orc_inflight* t, int32_t endpoint);
void orc_inflight_get(const orc_inflight* t, int32_t M, int64_t* requests_out, int64_t* tokens_out);
int32_t __real_eppscore_create(int32_t device, const eppscore_config* cfg, eppscore_engine** out);
int32_t __real_eppscore_set_snapshot(eppscore_engine* e, const eppscore_snapshot* s);
}

namespace {
struct Seen {
  eppscore_config cfg{};
  orc_inflight* tracker = nullptr;  // never freed: one per engine of a short-lived test program
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
    g_seen[*out] = Seen{*cfg, orc_inflight_new()};
  }
  return rc;
}

int32_t __wrap_eppscore_set_snapshot(eppscore_engine* e, const eppscore_snapshot* s) {
  std::vector<int64_t> tokens;
  eppscore_snapshot sub;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    Seen* x = seen(e);
    bool token_load = false;
    if (x)
      for (int i = 0; i < x->cfg.n_scorers; i++) token_load = token_load || x->cfg.scorer_kind[i] == EPPSCORE_SCORER_TOKEN_LOAD;
    if (!x || !s || s->struct_size != sizeof(*s) || s->inflight_tokens || !token_load || s->M <= 0) return __real_eppscore_set_snapshot(e, s);
    tokens.resize((size_t)s->M);
    orc_inflight_get(x->tracker, s->M, nullptr, tokens.data());
    sub = *s;
  }
  sub.inflight_tokens = tokens.data();
  return __real_eppscore_set_snapshot(e, &sub);
}

int32_t eppscore_estimate_tokens(eppscore_engine* e, int32_t R, int32_t location, const int64_t* request_size_bytes,
                                 const int32_t* token_hint, const int32_t* prompt_chars, int64_t* out, void*) {
  if (!e || R < 0 || (R > 0 && !out) || location != 0) return EPPSCORE_ERR_INVALID;
  for (int32_t r = 0; r < R; r++)
    out[r] = orc_estimate_tokens(request_size_bytes ? request_size_bytes[r] : 0, token_hint ? token_hint[r] : -1,
                                 prompt_chars ? prompt_chars[r] : 0);
  return EPPSCORE_OK;
}

static int32_t update(eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint, const int64_t* tokens, int sign) {
  if (!e || R < 0 || (R > 0 && !endpoint) || location != 0) return EPPSCORE_ERR_INVALID;
  std::lock_guard<std::mutex> lk(g_mu);
  Seen* x = seen(e);
  if (!x) return EPPSCORE_ERR_INVALID;
  for (int32_t r = 0; r < R; r++)
    if (endpoint[r] >= x->cfg.max_endpoints) return EPPSCORE_ERR_INVALID;
  (sign > 0 ? orc_inflight_add : orc_inflight_release)(x->tracker, R, endpoint, tokens);
  return EPPSCORE_OK;
}

int32_t eppscore_inflight_add(eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint, const int64_t* tokens, void*) {
  return update(e, R, location, endpoint, tokens, 1);
}

int32_t eppscore_inflight_release(eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint, const int64_t* tokens,
                                  void*) {
  return update(e, R, location, endpoint, tokens, -1);
}

int32_t eppscore_inflight_remove_endpoint(eppscore_engine* e, int32_t endpoint) {
  std::lock_guard<std::mutex> lk(g_mu);
  Seen* x = seen(e);
  if (!x || endpoint < 0 || endpoint >= x->cfg.max_endpoints) return EPPSCORE_ERR_INVALID;
  orc_inflight_remove(x->tracker, endpoint);
  return EPPSCORE_OK;
}

int32_t eppscore_inflight_get(eppscore_engine* e, int64_t* requests_out, int64_t* tokens_out, int32_t M) {
  std::lock_guard<std::mutex> lk(g_mu);
  Seen* x = seen(e);
  if (!x || M < 0 || M > x->cfg.max_endpoints) return EPPSCORE_ERR_INVALID;
  orc_inflight_get(x->tracker, M, requests_out, tokens_out);
  return EPPSCORE_OK;
}

}  // extern "C"
