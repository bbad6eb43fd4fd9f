// oracle_backed_inorder.cpp — TEST INFRASTRUCTURE ONLY: eppscore_schedule_batch_inorder for the oracle-backed stand-in of the C ABI,
// so that the host layer's InOrderInFlightLoad runs in the `-m "not gpu"` suite.  It is the call's contract restated: for each
// request in order, the stand-in's single-request schedule against the in-flight counters of oracle_backed_inflight.cpp, then
// the in-flight add of its pick.  Link with oracle_backed_inflight.cpp and its --wrap flags; this file replaces
// oracle_backed_abi.cpp, which it includes for the stand-in's engine state.
#include "oracle_backed_abi.cpp"

uint64_t g_inorder_calls = 0;  // calls made, so a test can tell which route the host layer took

extern "C" int32_t eppscore_schedule_batch_inorder(eppscore_engine* e, const eppscore_batch* b, const int64_t* tokens) {
  if (!e) return EPPSCORE_ERR_INVALID;
  g_inorder_calls++;
  if (!b || b->struct_size != sizeof(*b) || b->location != 0) return fail(e, EPPSCORE_ERR_INVALID, "batch NULL, struct_size or location");
  if (b->dense_feat || b->scores_out || b->match_blocks || b->pred_out || b->filter_mask_out)
    return fail(e, EPPSCORE_ERR_INVALID, "schedule_batch_inorder: R x M outputs and dense rows are not available");
  for (int i = 0; i < e->prof.n_scorers; i++)
    if (e->prof.scorer_kind[i] == ORC_SCORER_LATENCY) return fail(e, EPPSCORE_ERR_INVALID, "schedule_batch_inorder: latency scorer");
  if (!e->have_snapshot) return fail(e, EPPSCORE_ERR_NO_SNAPSHOT, "schedule_batch_inorder before set_snapshot");
  if (b->R < 0) return fail(e, EPPSCORE_ERR_INVALID, "R < 0");
  const size_t mw = (size_t)(e->M + 31) / 32, mb = (size_t)(b->max_blocks > 0 ? b->max_blocks : e->cfg.max_blocks);
  std::vector<int64_t> tok((size_t)std::max(e->M, 1));
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
    if (b->cand_mask) one.cand_mask = b->cand_mask + (size_t)r * mw;
    one.pick = b->pick + r;
    one.pick_score = b->pick_score + r;
    one.tie_count = b->tie_count + r;
    if (b->total_blocks) one.total_blocks = b->total_blocks + r;
    if (b->hashes_out) one.hashes_out = b->hashes_out + (size_t)r * mb;
    int32_t rc = eppscore_schedule_batch(e, &one);
    if (rc != EPPSCORE_OK) return rc;
    if ((rc = eppscore_inflight_add(e, 1, 0, b->pick + r, tokens ? tokens + r : nullptr, nullptr)) != EPPSCORE_OK) return rc;
  }
  if (eppscore_inflight_get(e, nullptr, tok.data(), e->M) != EPPSCORE_OK) return EPPSCORE_ERR_INVALID;
  e->tokens.assign(tok.begin(), tok.begin() + e->M);  // a later plain batch sees the new counters, as after the engine's call
  return EPPSCORE_OK;
}
