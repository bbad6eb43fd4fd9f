// oracle_backed_inorder_profiles.cpp — TEST INFRASTRUCTURE ONLY: eppscore_schedule_batch_inorder_profiles for the oracle-backed
// stand-in of the C ABI, so that the host layer's in-order Profiles route runs in the `-m "not gpu"` suite.  It is the call's
// contract restated: for each request in order, the stand-in's single-request eppscore_schedule_batch_profiles over the runs of
// its run mask against the in-flight counters, then, when the primary run picked, the match at every pick before the request's
// Adds, the in-flight add at every pick and (index form) the Adds at the primary and the prefill pick.  It includes
// oracle_backed_profiles.cpp (link this file instead); link with oracle_backed_inflight.cpp and its --wrap flags.
#include <algorithm>

#include "oracle_backed_profiles.cpp"

uint64_t g_inorder_profiles_calls = 0;

extern "C" int32_t eppscore_schedule_batch_inorder_profiles(eppscore_engine* e, const eppscore_batch* b, const int64_t* tokens,
                                                            int32_t n_runs, const eppscore_profile_run* runs,
                                                            const eppscore_inorder_profiles* x) {
  if (!e) return EPPSCORE_ERR_INVALID;
  g_inorder_profiles_calls++;
  if (!x || x->struct_size != sizeof(*x) || (x->index != 0 && x->index != 1)) return fail(e, EPPSCORE_ERR_INVALID, "inorder_profiles");
  if (!b || b->struct_size != sizeof(*b) || b->location != 0) return fail(e, EPPSCORE_ERR_INVALID, "batch NULL, struct_size or location");
  if (n_runs < 1 || n_runs > EPPSCORE_MAX_PROFILES || !runs || x->primary_run < 0 || x->primary_run >= n_runs ||
      x->prefill_run < -1 || x->prefill_run >= n_runs || x->prefill_run == x->primary_run)
    return fail(e, EPPSCORE_ERR_INVALID, "runs, primary_run or prefill_run");
  const size_t mw = (size_t)(e->M + 31) / 32, mb = (size_t)(b->max_blocks > 0 ? b->max_blocks : e->cfg.max_blocks);
  std::vector<int64_t> tok((size_t)std::max(e->M, 1));
  std::vector<uint64_t> h(mb);
  std::vector<uint16_t> match((size_t)std::max(e->M, 1));
  for (int32_t r = 0; r < b->R; r++) {
    if (eppscore_inflight_get(e, nullptr, tok.data(), e->M) != EPPSCORE_OK) return EPPSCORE_ERR_INVALID;
    e->tokens.assign(tok.begin(), tok.begin() + e->M);  // the counters as the next single-request Schedule sees them
    e->have_tokens = true;
    eppscore_batch one = *b;
    one.R = 1;
    one.request_base = b->request_base + r;
    if (b->prompt_off) one.prompt_off = b->prompt_off + r;
    if (b->prompt_len) one.prompt_len = b->prompt_len + r;
    if (b->model_seed) one.model_seed = b->model_seed + r;
    if (b->hashes_in) one.hashes_in = b->hashes_in + (size_t)r * b->hash_stride;
    if (b->n_hashes_in) one.n_hashes_in = b->n_hashes_in + r;
    if (b->adapter_id) one.adapter_id = b->adapter_id + r;
    uint16_t n = 0;
    std::fill(h.begin(), h.end(), 0);
    one.total_blocks = &n;
    one.hashes_out = b->prompt_bytes && !b->hashes_in ? h.data() : nullptr;
    const unsigned bits = x->run_mask ? x->run_mask[r] : 0xFu;
    std::vector<eppscore_profile_run> sel;
    for (int32_t i = 0; i < n_runs; i++) {
      runs[i].pick[r] = -1;
      runs[i].pick_score[r] = 0.0;
      runs[i].tie_count[r] = 0;
      if (!((bits >> i) & 1u)) continue;
      eppscore_profile_run u = runs[i];
      if (u.cand_mask) u.cand_mask += (size_t)r * mw;
      u.pick += r;
      u.pick_score += r;
      u.tie_count += r;
      sel.push_back(u);
    }
    if (!sel.empty()) {
      const int32_t rc = eppscore_schedule_batch_profiles(e, &one, (int32_t)sel.size(), sel.data());
      if (rc != EPPSCORE_OK) return rc;
    }
    if (b->hashes_in) std::copy(b->hashes_in + (size_t)r * b->hash_stride, b->hashes_in + (size_t)r * b->hash_stride + n, h.begin());
    if (b->total_blocks) b->total_blocks[r] = n;
    if (b->hashes_out) std::copy(h.begin(), h.end(), b->hashes_out + (size_t)r * mb);
    for (int32_t i = 0; i < n_runs; i++)
      if (x->pick_match[i]) x->pick_match[i][r] = 0;
    if (runs[x->primary_run].pick[r] < 0) continue;  // no PreRequest for a failed schedule
    if (n > 0) orc_match_longest_prefix(e->idx, h.data(), n, e->M, match.data());
    std::vector<int32_t> eps;
    for (int32_t i = 0; i < n_runs; i++) {
      const int32_t p = runs[i].pick[r];
      if (p < 0) continue;
      eps.push_back(p);
      if (x->pick_match[i]) x->pick_match[i][r] = n > 0 ? match[(size_t)p] : 0;
    }
    std::vector<int64_t> t(eps.size(), tokens ? tokens[r] : 0);
    if (int32_t rc = eppscore_inflight_add(e, (int32_t)eps.size(), 0, eps.data(), t.data(), nullptr); rc != EPPSCORE_OK) return rc;
    if (x->index)
      for (int32_t i : {x->primary_run, x->prefill_run})
        if (i >= 0 && runs[i].pick[r] >= 0) orc_commit_picks(e->idx, 1, &runs[i].pick[r], h.data(), &n, (int32_t)mb, x->lru_capacity);
  }
  if (eppscore_inflight_get(e, nullptr, tok.data(), e->M) != EPPSCORE_OK) return EPPSCORE_ERR_INVALID;
  e->tokens.assign(tok.begin(), tok.begin() + e->M);  // a later plain batch sees the new counters, as after the engine's call
  return EPPSCORE_OK;
}
