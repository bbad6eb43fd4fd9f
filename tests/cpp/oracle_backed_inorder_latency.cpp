// oracle_backed_inorder_latency.cpp — TEST INFRASTRUCTURE ONLY: eppscore_schedule_batch_inorder_latency for the oracle-backed
// stand-in of the C ABI, so that the host layer's InOrderRunningRequests runs in the `-m "not gpu"` suite.  It is the call's
// contract restated: for each request in order, the running-request view of oracle_backed_running.cpp's queue oracle (when the
// call has keys) and the in-flight counters of oracle_backed_inflight.cpp go into the stand-in's snapshot, the stand-in schedules
// the request alone, then the queue add of (pick, key, tpot), the in-flight add of its tokens and, in the index form, the match at
// its pick before its own Add and the Add of its blocks.  Link with oracle_backed_inflight.cpp, oracle_backed_running.cpp and
// their --wrap flags, plus -Wl,--wrap=eppscore_running_add: the host layer's own queue adds are counted (g_host_running_adds).
// Both of those files hook eppscore_create and eppscore_set_snapshot; tests/test_host_inorder_latency_cpu.py compiles them so
// that the running hook calls the in-flight one, which calls the stand-in.
#include <algorithm>

#include "oracle_backed_inorder.cpp"

uint64_t g_inorder_latency_calls = 0;
uint64_t g_host_running_adds = 0;
static bool g_in_call = false;  // the stand-in's own adds are not the host layer's

// The stand-in's index, for a test's comparisons: lru.Keys() of an endpoint (empty without an LRU).
std::vector<uint64_t> StandInLruKeys(eppscore_engine* e, int32_t endpoint) {
  const int32_t n = orc_index_lru_len(e->idx, endpoint);
  std::vector<uint64_t> k((size_t)std::max(n, 0));
  if (n > 0) orc_index_lru_keys(e->idx, endpoint, k.data(), n);
  return k;
}

extern "C" int32_t __real_eppscore_running_add(eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint,
                                               const uint64_t* request_key, const double* tpot_slo, uint8_t* added_out, void* stream);
extern "C" int32_t __wrap_eppscore_running_add(eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint,
                                               const uint64_t* request_key, const double* tpot_slo, uint8_t* added_out, void* stream) {
  if (!g_in_call) g_host_running_adds++;
  return __real_eppscore_running_add(e, R, location, endpoint, request_key, tpot_slo, added_out, stream);
}

extern "C" int32_t eppscore_schedule_batch_inorder_latency(eppscore_engine* e, const eppscore_batch* b, const int64_t* tokens,
                                                           const eppscore_inorder_index* x, const eppscore_inorder_running* q) {
  if (!e) return EPPSCORE_ERR_INVALID;
  g_inorder_latency_calls++;
  if (!q || q->struct_size != sizeof(*q)) return fail(e, EPPSCORE_ERR_INVALID, "inorder_running NULL or struct_size mismatch");
  if (x && x->struct_size != sizeof(*x)) return fail(e, EPPSCORE_ERR_INVALID, "inorder_index struct_size mismatch");
  if (!b || b->struct_size != sizeof(*b) || b->location != 0) return fail(e, EPPSCORE_ERR_INVALID, "batch NULL, struct_size or location");
  bool lat = false;
  for (int i = 0; i < e->prof.n_scorers; i++) lat = lat || e->prof.scorer_kind[i] == ORC_SCORER_LATENCY;
  if (!lat) return fail(e, EPPSCORE_ERR_INVALID, "schedule_batch_inorder_latency: profile 0 has no latency scorer");
  if (!e->have_snapshot) return fail(e, EPPSCORE_ERR_NO_SNAPSHOT, "schedule_batch_inorder_latency before set_snapshot");
  if (b->R < 0) return fail(e, EPPSCORE_ERR_INVALID, "R < 0");
  const size_t mw = (size_t)(e->M + 31) / 32, mb = (size_t)(b->max_blocks > 0 ? b->max_blocks : e->cfg.max_blocks);
  const size_t M1 = (size_t)std::max(e->M, 1);
  std::vector<int64_t> tok(M1);
  std::vector<double> mn(M1);
  std::vector<int32_t> cnt(M1);
  std::vector<uint64_t> h(mb);
  std::vector<uint16_t> match(M1);
  g_in_call = true;
  int32_t rc = EPPSCORE_OK;
  for (int32_t r = 0; r < b->R && rc == EPPSCORE_OK; r++) {
    if (eppscore_inflight_get(e, nullptr, tok.data(), e->M) != EPPSCORE_OK) rc = EPPSCORE_ERR_INVALID;
    e->tokens.assign(tok.begin(), tok.begin() + e->M);
    e->have_tokens = true;
    if (q->request_key) {  // the queues as the next single-request Schedule sees them
      if (eppscore_running_get(e, mn.data(), cnt.data(), e->M) != EPPSCORE_OK) rc = EPPSCORE_ERR_INVALID;
      e->min_tpot.assign(mn.begin(), mn.begin() + e->M);
      e->dispatched.assign(cnt.begin(), cnt.begin() + e->M);
      e->have_min_tpot = e->have_dispatched = true;
    }
    eppscore_batch one = *b;
    one.R = 1;
    one.request_base = b->request_base + r;
    if (b->prompt_off) one.prompt_off = b->prompt_off + r;
    if (b->prompt_len) one.prompt_len = b->prompt_len + r;
    if (b->model_seed) one.model_seed = b->model_seed + r;
    if (b->adapter_id) one.adapter_id = b->adapter_id + r;
    if (b->cand_mask) one.cand_mask = b->cand_mask + (size_t)r * mw;
    if (b->input_tokens) one.input_tokens = b->input_tokens + r;
    if (b->ttft_slo) one.ttft_slo = b->ttft_slo + r;
    if (b->tpot_slo) one.tpot_slo = b->tpot_slo + r;
    one.pick = b->pick + r;
    one.pick_score = b->pick_score + r;
    one.tie_count = b->tie_count + r;
    uint16_t n = 0;
    one.total_blocks = &n;
    std::fill(h.begin(), h.end(), 0);
    one.hashes_out = b->prompt_bytes ? h.data() : nullptr;
    if (rc == EPPSCORE_OK) rc = eppscore_schedule_batch(e, &one);
    if (rc != EPPSCORE_OK) break;
    if (b->total_blocks) b->total_blocks[r] = n;
    const int32_t p = b->pick[r];
    uint8_t added = 0;
    if (q->request_key && p >= 0)
      rc = eppscore_running_add(e, 1, 0, &b->pick[r], q->request_key + r, b->tpot_slo ? b->tpot_slo + r : nullptr, &added, nullptr);
    if (q->added_out) q->added_out[r] = added;
    if (rc == EPPSCORE_OK) rc = eppscore_inflight_add(e, 1, 0, b->pick + r, tokens ? tokens + r : nullptr, nullptr);
    if (x) {
      uint16_t pm = 0;
      if (p >= 0 && n > 0) {
        orc_match_longest_prefix(e->idx, h.data(), n, e->M, match.data());
        pm = match[(size_t)p];
      }
      if (x->pick_match) x->pick_match[r] = pm;
      if (p >= 0) orc_commit_picks(e->idx, 1, &b->pick[r], h.data(), &n, (int32_t)mb, x->lru_capacity);
    }
  }
  g_in_call = false;
  if (rc != EPPSCORE_OK) return rc;
  if (eppscore_inflight_get(e, nullptr, tok.data(), e->M) != EPPSCORE_OK) return EPPSCORE_ERR_INVALID;
  e->tokens.assign(tok.begin(), tok.begin() + e->M);
  if (q->request_key) {  // a later plain batch sees the queues the call left, as after the engine's call
    if (eppscore_running_get(e, mn.data(), cnt.data(), e->M) != EPPSCORE_OK) return EPPSCORE_ERR_INVALID;
    e->min_tpot.assign(mn.begin(), mn.begin() + e->M);
    e->dispatched.assign(cnt.begin(), cnt.begin() + e->M);
  }
  return EPPSCORE_OK;
}
