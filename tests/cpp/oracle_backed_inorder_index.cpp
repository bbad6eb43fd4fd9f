// oracle_backed_inorder_index.cpp — TEST INFRASTRUCTURE ONLY: eppscore_schedule_batch_inorder_index for the oracle-backed stand-in
// of the C ABI, so that the host layer's InOrderPrefixIndex runs in the `-m "not gpu"` suite.  It is the call's contract
// restated: for each request in order, the stand-in's single-request schedule against the in-flight counters (with its hashes),
// the match at its pick before its own Add, the in-flight add of its tokens and the Add of its blocks.  Link with
// oracle_backed_inflight.cpp and its --wrap flags, plus -Wl,--wrap=eppscore_commit_picks: the host layer's own commits are
// counted (g_host_commits) and passed on.
#include <algorithm>

#include "oracle_backed_inorder.cpp"

uint64_t g_inorder_index_calls = 0;
uint64_t g_host_commits = 0;

extern "C" int32_t __real_eppscore_commit_picks(eppscore_engine* e, int32_t R, const int32_t* pick, const uint64_t* hashes,
                                                const uint16_t* n_hashes, int32_t hash_stride, const int32_t* lru_capacity);
extern "C" int32_t __wrap_eppscore_commit_picks(eppscore_engine* e, int32_t R, const int32_t* pick, const uint64_t* hashes,
                                                const uint16_t* n_hashes, int32_t hash_stride, const int32_t* lru_capacity) {
  g_host_commits++;
  return __real_eppscore_commit_picks(e, R, pick, hashes, n_hashes, hash_stride, lru_capacity);
}

// The stand-in's index, for a test's comparisons: lru.Keys() of an endpoint (empty without an LRU) and len(hashToPods).
std::vector<uint64_t> StandInLruKeys(eppscore_engine* e, int32_t endpoint) {
  const int32_t n = orc_index_lru_len(e->idx, endpoint);
  std::vector<uint64_t> k((size_t)std::max(n, 0));
  if (n > 0) orc_index_lru_keys(e->idx, endpoint, k.data(), n);
  return k;
}
int64_t StandInNumHashes(eppscore_engine* e) { return orc_index_num_hashes(e->idx); }

extern "C" int32_t eppscore_schedule_batch_inorder_index(eppscore_engine* e, const eppscore_batch* b, const int64_t* tokens,
                                                         const eppscore_inorder_index* x) {
  if (!e) return EPPSCORE_ERR_INVALID;
  g_inorder_index_calls++;
  if (!x || x->struct_size != sizeof(*x)) return fail(e, EPPSCORE_ERR_INVALID, "inorder_index NULL or struct_size mismatch");
  if (!b || b->struct_size != sizeof(*b) || b->location != 0) return fail(e, EPPSCORE_ERR_INVALID, "batch NULL, struct_size or location");
  if (b->R < 0) return fail(e, EPPSCORE_ERR_INVALID, "R < 0");
  const size_t mb = (size_t)(b->max_blocks > 0 ? b->max_blocks : e->cfg.max_blocks);
  std::vector<uint64_t> h(mb);
  std::vector<uint16_t> match((size_t)std::max(e->M, 1));
  for (int32_t r = 0; r < b->R; r++) {
    eppscore_batch one = *b;
    one.R = 1;
    one.request_base = b->request_base + r;
    if (b->prompt_off) one.prompt_off = b->prompt_off + r;
    if (b->prompt_len) one.prompt_len = b->prompt_len + r;
    if (b->model_seed) one.model_seed = b->model_seed + r;
    if (b->adapter_id) one.adapter_id = b->adapter_id + r;
    if (b->cand_mask) one.cand_mask = b->cand_mask + (size_t)r * ((e->M + 31) / 32);
    one.pick = b->pick + r;
    one.pick_score = b->pick_score + r;
    one.tie_count = b->tie_count + r;
    uint16_t n = 0;
    one.total_blocks = &n;
    std::fill(h.begin(), h.end(), 0);
    one.hashes_out = b->prompt_bytes ? h.data() : nullptr;
    int32_t rc = eppscore_schedule_batch_inorder(e, &one, tokens ? tokens + r : nullptr);  // schedule + in-flight add
    if (rc != EPPSCORE_OK) return rc;
    if (b->total_blocks) b->total_blocks[r] = n;
    if (b->hashes_out) std::copy(h.begin(), h.end(), b->hashes_out + (size_t)r * mb);
    const int32_t p = b->pick[r];
    uint16_t pm = 0;
    if (p >= 0 && n > 0) {
      orc_match_longest_prefix(e->idx, h.data(), n, e->M, match.data());
      pm = match[(size_t)p];
    }
    if (x->pick_match) x->pick_match[r] = pm;
    if (p >= 0) orc_commit_picks(e->idx, 1, &b->pick[r], h.data(), &n, (int32_t)mb, x->lru_capacity);
  }
  return EPPSCORE_OK;
}
