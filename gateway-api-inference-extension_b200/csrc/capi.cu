// capi.cu — the C ABI of libeppscore.so (include/eppscore.h): engine object, snapshot ingestion,
// the batched Schedule call, the prefix index plumbing.  Host code only orchestrates; all path
// arithmetic runs in the kernels of kernels.cu.  There is deliberately no CPU fallback here.
#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <cassert>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iterator>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/eppscore.h"
#include "cuda_owners.hpp"
#include "kernels.cuh"
#include "prefix_index.hpp"
#include "xxh64.cuh"

using namespace eppscore;

namespace {

thread_local std::string g_create_error;

struct PlanSet {
  Plan plan;
  const double* term_ptr[kMaxSteps];
};

// The last device-location batch a caller stream ran outside a capture (pending_record / pending_wait).
struct PendingBatch {
  cudaStream_t stream = nullptr;
  Event done;          // recorded behind that batch
  bool armed = false;  // the batch may not have completed
};

// One scheduler profile (eppscore_add_profile): its configuration and everything prepared for it from the shared snapshot.
struct Profile {
  eppscore_config cfg{};  // the engine's config with this profile's scorers, picker and filters, and its own tie seed
  DevBuf term[kMaxSteps], fold_unmasked, fold_masked, summ, tiemask, prefix_lut2d, qhdr[2], qbucket[2];
  bool have_lut2d = false;
  PlanSet plan_unmasked{}, plan_masked{};
  PrepareArgs pa{};  // what the current snapshot was prepared with
  // endpoint subset: natural-order [Mpad/32] and permuted [row_words] bit rows, live (what the current snapshot was prepared with)
  // and next (eppscore_set_profile_endpoints, copied to live by the next set_snapshot)
  DevBuf member_nat, member_perm, next_nat, next_perm;
  bool subset = false, next_subset = false;
};

}  // namespace

struct eppscore_engine {
  int device = 0;
  int sm_count = 132;
  eppscore_config cfg{};
  Geo geo{};
  int32_t A_cap = 64;
  Event ev_snapshot, ev_table, ev_caller;
  Event ev_index_join;  // behind a commit captured on the engine stream: the caller's stream joins on it inside the capture
  Event ev_subset;  // behind the last set_snapshot outside a capture: its copies of the profiles' next subset rows are done
  cudaStream_t snapshot_stream = nullptr;        // stream the last snapshot preparation ran on
  unsigned long long snapshot_capture_id = 0;    // != 0: ev_snapshot was recorded inside that CUDA-graph capture
  std::string err;
  uint64_t launches = 0;
  bool force_generic = false;  // EPPSCORE_FORCE_GENERIC=1 / eppscore_set_debug(1): skip the specialised kernels
  bool use_pdl = true;          // eppscore_set_debug(4): programmatic dependent launch between the kernels of a batch
  int32_t hash_stage_mask = 27;  // eppscore_set_debug(2): profiling only (see include/eppscore.h)

  // snapshot
  bool have_snapshot = false;
  int32_t M = 0, A = 0, lora_words = 0;
  uint64_t epoch = 0;
  DevBuf raw_kv, raw_queue, raw_running, raw_act, raw_wait, raw_nmodels, raw_max, raw_col[4];
  DevBuf raw_min_tpot, raw_dispatched, raw_prefill, raw_tokens, lat_ep;
  eppscore_latency_params lat_params{};  // pending: applied by the next set_snapshot
  LatArgs lat_args{};                    // what the current snapshot was prepared with
  bool have_col[4] = {false, false, false, false};
  bool have_running = false;
  const int64_t* cur_queue = nullptr;    // raw WaitingQueueSize / RunningRequestsSize of the current snapshot
  const int64_t* cur_running = nullptr;  // (engine copy for host snapshots, the caller's buffer for device ones)
  DevBuf cls_lo, cls_hi;                 // LoRA class planes (snapshot only: every profile's adapter kernel writes the same)
  Profile prof[EPPSCORE_MAX_PROFILES];
  int32_t n_prof = 0;
  PrepareArgs base_pa{};                 // the profile-independent part of the current snapshot's preparation

  // prefix index: hashToPods + the per-endpoint LRUs, both device-resident (prefix_index.hpp); mutated on `stream`
  std::unique_ptr<DeviceIndex> index;
  // device-location batches on caller streams that may still read the table, the terms or a scratch set (pending_record)
  std::vector<PendingBatch> pending;
  // Staging for the synchronous host-array calls (HostStage): slot i holds the call's i-th array.  Each of those calls runs on
  // `stream` and synchronises it before it returns, so one set serves them all.
  DevBuf stage[8];

  // Producer state the scorers read: mutations of either producer below prepare the terms of the profiles that read the state
  // again (with their Profile::pa).  Mutations outside a CUDA-graph capture are ordered through ev_producer, recorded after
  // each one on its stream, so the two families never rewrite the terms concurrently (producer_begin / producer_end).
  Event ev_producer;
  bool producer_pending = false;

  // in-flight load producer (inflightload/producer.go): per-endpoint request and token counters, [Mpad] int64 each, zeroed at
  // create.  They feed the token-load scorer when the snapshot carries no inflight_tokens.
  DevBuf inflight_req, inflight_tok, inflight_err;
  // requests the probing hash kernel has resolved since creation (u64; eppscore_stats.probe_resolved, modulo 2^32)
  DevBuf probe_resolved;
  bool snapshot_has_tokens = false;  // the current snapshot carries inflight_tokens

  // predicted-latency producer's running-request queues (running_kernel.cu): the (endpoint, key) -> tpot table and the
  // per-endpoint count / minimum.  They feed the latency fold-in when the snapshot lacks min_tpot_slo or dispatched.
  std::array<DevBuf, 8> run_tab;  // two tables of run_cap slots (slot, tpot, owner, rm each): the table and its spare, in either role
  DevBuf run_desc;    // the device descriptor (RunDev) every running kernel reads the tables and the scratch through
  RunDev run_host{};  // its host copy (re-read before a change: the device-side compaction swaps the two tables)
  DevBuf run_count, run_min_bits, run_min_cnt, run_min_view, run_dirty, run_rc_min, run_rc_cnt, run_ctr;
  DevBuf c_rslot, c_rwon;  // the per-call [R] scratch
  int64_t run_cap = 0;
  // host upper bounds of the live entries and tombstones: the counters copied back behind the last mutation (h_run,
  // ev_run_copy) once that copy has landed, plus R per call issued since
  int64_t run_bound_live = 0;
  PinnedBuf h_run;  // RunCounters
  Event ev_run_copy;
  bool run_copy_issued = false;
  bool run_captured = false;  // a mutation was captured since the last exact read: its replays are invisible to the bound
  bool snapshot_has_min_tpot = false, snapshot_has_dispatched = false;
  // Device-location eppscore_predict_latency calls read the running-request counts in place, so a running-request update must
  // not rewrite them before those reads are done (count_reads_wait).  count_readers: a call on a caller stream may still be
  // pending (it is in the pending set); cleared once that set has drained.  ev_count_read: recorded behind the last call on the
  // engine stream (count_read_engine until it has completed).
  bool count_readers = false, count_read_engine = false;
  Event ev_count_read;

  // scratch for host-location batches and internal hashes: two sets, so the chunks of a host batch can alternate
  // between two streams (H2D of chunk i+1 under the kernels and the D2H of chunk i).  sc[0] also serves device-location
  // batches on streams without a set of their own (eppscore_reserve_stream), sc[1..3] the slices of a sliced one.
  struct Scratch {
    DevBuf s_prompts, s_off, s_len, s_seed, s_hashes, s_nh, s_adapter, s_mask, s_dense, s_dtotal, s_pick, s_score,
        s_tie, s_match, s_total, s_scores, s_intok, s_tokens, s_tslo, s_pslo, s_pred, s_fields, s_fmask, s_topk_m, s_topk_s, s_probe,
        s_subset,  // candidate rows subset ∧ cand_mask of a run on a profile with an endpoint subset
        // an in-order batch's slice (schedule_inorder): match rows, totals and candidate min / max.  Allocated by the first call
        // outside a capture for a fixed number of rows and never reallocated, like `wide`.
        s_io_match, s_io_total, s_io_minmax;
    int32_t io_rows = 0;
    // score rows of a wide top-k batch's slice ([wide_rows][Mpad] float64, schedule_wide).  Allocated by the first call that
    // needs them and never reallocated, so a graph captured after that call keeps pointing at live memory.
    DevBuf wide;
    int32_t rows = 0;  // > 0: a reserved stream's set, allocated for this many requests and never grown
  } sc[4];
  // A caller stream's own scratch set (eppscore_reserve_stream): its device-location batches use it instead of sc[0], so
  // they can run while batches on other streams do, and a graph captured on the stream never sees it move.  The set is
  // freed only after the work queued on the stream has finished.
  struct StreamScratch {
    cudaStream_t stream = nullptr;
    int32_t max_R = 0, max_blocks = 0;
    Scratch sc;
    ~StreamScratch() {
      if (stream) cudaStreamSynchronize(stream);
    }
  };
  // pinned staging for the small per-request results of a host batch: a D2H copy into the caller's (usually pageable)
  // arrays would block the host after every chunk and serialise the pipeline
  PinnedBuf h_res;
  int32_t wide_rows = 0;
  int32_t io_cluster = 0;          // CTAs per cluster of inorder_pick_kernel (0: not decided yet)
  int32_t host_chunk = 8192;       // requests per chunk of a host-location batch (eppscore_set_debug key 3)
  // device-location batches cut into `dev_split` slices over `dev_streams` streams (the caller's + internal ones): the
  // HBM-bound body hashing of slice i+1 runs under the latency-bound chain and probe kernels of slice i
  // (eppscore_set_debug keys 5 and 6)
  int32_t dev_split = 1, dev_streams = 2;
  Event ev_fork, ev_join[3];

  // The streams come last: members are destroyed in reverse order, and a Stream synchronises before it is destroyed, so
  // every buffer above is freed only after the work queued on these streams has finished.
  Stream stream;           // the engine stream
  Stream stream2;          // second copy/compute stream of the chunked host path
  Stream split_stream[3];  // the internal streams of a sliced device-location batch
  // After the engine's streams, so destroyed before them: each set waits for its caller stream before it is freed, and so
  // before anything else the stream's batches read is freed.
  std::vector<std::unique_ptr<StreamScratch>> reserved;
};
using Scratch = eppscore_engine::Scratch;
using StreamScratch = eppscore_engine::StreamScratch;

namespace {

int32_t fail(eppscore_engine* e, int32_t code, const std::string& msg) {
  if (e) e->err = msg;
  else g_create_error = msg;
  return code;
}
int32_t cuda_fail(eppscore_engine* e, cudaError_t c, const char* what) {
  return fail(e, EPPSCORE_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(c));
}
#define CK(e, call)                                            \
  do {                                                         \
    cudaError_t _c = (call);                                   \
    if (_c != cudaSuccess) return cuda_fail((e), _c, #call);   \
  } while (0)

// Whether `st` is being captured into a CUDA graph; *id (when given) receives the capture's id, 0 outside a capture.
bool is_capturing(cudaStream_t st, unsigned long long* id = nullptr) {
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  unsigned long long cap_id = 0;
  cudaStreamGetCaptureInfo(st, &cap, &cap_id);
  const bool capturing = cap != cudaStreamCaptureStatusNone;
  if (id) *id = capturing ? cap_id : 0;
  return capturing;
}

// A device-location batch on caller stream `s` may still read the index table, the snapshot terms and its scratch set (sc[0],
// or the stream's own) when its call returns.  Outside a capture its stream's event is recorded again behind it, so the set
// of pending batches holds one event per caller stream.  Whatever rewrites those first waits for all of them (pending_wait).  Inside a capture
// the graph's edges order this instead, and the engine stream orders itself.
int32_t pending_record(eppscore_engine* e, cudaStream_t s) {
  if (s == e->stream || is_capturing(s)) return EPPSCORE_OK;
  PendingBatch* slot = nullptr;
  for (PendingBatch& p : e->pending) {
    if (p.armed && p.stream == s) {
      slot = &p;
      break;
    }
    if (!p.armed && !slot) slot = &p;
  }
  if (!slot) slot = &e->pending.emplace_back();
  if (!slot->done) CK(e, make(slot->done));
  CK(e, cudaEventRecord(slot->done, s));
  slot->stream = s;
  slot->armed = true;
  return EPPSCORE_OK;
}
// `st` waits for every pending batch.  A batch leaves the set once it has completed, not when a stream waits for it: the wait
// orders only `st`, and a later rewrite on another stream must still wait.
int32_t pending_wait(eppscore_engine* e, cudaStream_t st) {
  for (PendingBatch& p : e->pending) {
    if (!p.armed) continue;
    if (cudaEventQuery(p.done) == cudaSuccess) p.armed = false;
    else CK(e, cudaStreamWaitEvent(st, p.done, 0));
  }
  return EPPSCORE_OK;
}

// Orders a device-location reader on caller stream `s` after the index mutations issued before it (ev_table; the engine stream
// orders itself, and inside a capture the graph's edges do).  *wait_snapshot (when given) says whether `s` must also wait for
// ev_snapshot before it reads the snapshot terms: outside a capture when the last preparation ran outside one on another
// stream, inside one when it was recorded in this same capture (a captured stream may only wait on events of its own
// capture).  *capturing (when given) receives whether `s` is being captured.
int32_t reader_begin(eppscore_engine* e, cudaStream_t s, bool* capturing, bool* wait_snapshot) {
  unsigned long long cap_id = 0;
  const bool cap = is_capturing(s, &cap_id);
  if (!cap && s != e->stream) CK(e, cudaStreamWaitEvent(s, e->ev_table, 0));
  if (capturing) *capturing = cap;
  if (wait_snapshot)
    *wait_snapshot = cap ? (e->snapshot_capture_id != 0 && e->snapshot_capture_id == cap_id)
                         : (e->snapshot_capture_id == 0 && s != e->snapshot_stream);
  return EPPSCORE_OK;
}

// The scratch set reserved for caller stream `s`, or nullptr when it has none.
StreamScratch* reserved_scratch(eppscore_engine* e, cudaStream_t s) {
  for (const auto& r : e->reserved)
    if (r->stream == s) return r.get();
  return nullptr;
}
// Whether `s`, the engine stream or a reserved stream is being captured into a CUDA graph.
bool capture_open(eppscore_engine* e, cudaStream_t s) {
  if (is_capturing(s) || is_capturing(e->stream)) return true;
  for (const auto& r : e->reserved)
    if (is_capturing(r->stream)) return true;
  return false;
}

bool is_endpoint_term_kind(int k, bool masked) {
  if (k == EPPSCORE_SCORER_KV_CACHE || k == EPPSCORE_SCORER_TOKEN_LOAD) return true;
  if (k >= EPPSCORE_SCORER_ENDPOINT_COL0 && k < EPPSCORE_SCORER_ENDPOINT_COL0 + EPPSCORE_MAX_ENDPOINT_COLS) return true;
  if (!masked && (k == EPPSCORE_SCORER_QUEUE || k == EPPSCORE_SCORER_RUNNING)) return true;
  return false;
}
double clamp01_host(double s) { return s < 0 ? 0 : (s > 1 ? 1 : s); }

bool cfg_has(const eppscore_config& c, int kind) {
  for (int i = 0; i < c.n_scorers; i++)
    if (c.scorer_kind[i] == kind) return true;
  return false;
}

// Bit p: profile p has a scorer of this kind.
unsigned profiles_with(const eppscore_engine* e, int kind) {
  unsigned bits = 0;
  for (int p = 0; p < e->n_prof; p++)
    if (cfg_has(e->prof[p].cfg, kind)) bits |= 1u << p;
  return bits;
}
// The profiles whose current terms read the in-flight counters (token-load scorers).
unsigned counters_feed_scorer(const eppscore_engine* e) {
  return (e->have_snapshot && !e->snapshot_has_tokens) ? profiles_with(e, EPPSCORE_SCORER_TOKEN_LOAD) : 0u;
}
// The profiles whose latency fold-in reads the running-request queues (the per-endpoint minimum, or the count, or both).
unsigned running_feeds_scorer(const eppscore_engine* e) {
  return (e->have_snapshot && e->lat_ep.p && (!e->snapshot_has_min_tpot || !e->snapshot_has_dispatched))
             ? profiles_with(e, EPPSCORE_SCORER_LATENCY)
             : 0u;
}

// Translate the scorer list into kernel steps.  Leading request-independent scorers are folded into
// one precomputed array ((0.0+t0)+t1)+… — exact, because the kernel adds in the same order.
void build_plan(Profile& P, bool masked, PlanSet* ps) {
  Plan& p = ps->plan;
  memset(&p, 0, sizeof(p));
  const eppscore_config& c = P.cfg;
  int lead = 0;
  while (lead < c.n_scorers && is_endpoint_term_kind(c.scorer_kind[lead], masked)) lead++;
  int nt = 0, ns = 0;
  if (lead > 0) {
    ps->term_ptr[nt] = (masked ? P.fold_masked : P.fold_unmasked).as<double>();
    p.kind[ns] = STEP_EP_TERM;
    p.arg[ns] = nt++;
    ns++;
  }
  for (int s = lead; s < c.n_scorers; s++) {
    const int k = c.scorer_kind[s];
    const double w = c.scorer_weight[s];
    p.weight[ns] = w;
    if (is_endpoint_term_kind(k, masked)) {
      ps->term_ptr[nt] = P.term[s].as<double>();
      p.kind[ns] = STEP_EP_TERM;
      p.arg[ns] = nt++;
    } else if (k == EPPSCORE_SCORER_QUEUE || k == EPPSCORE_SCORER_RUNNING) {
      p.kind[ns] = STEP_MINMAX;
      p.arg[ns] = k == EPPSCORE_SCORER_QUEUE ? 0 : 1;
    } else if (k == EPPSCORE_SCORER_PREFIX) {
      p.kind[ns] = STEP_PREFIX;
    } else if (k == EPPSCORE_SCORER_LATENCY) {
      p.kind[ns] = STEP_LATENCY;
    } else if (k == EPPSCORE_SCORER_LORA) {
      p.kind[ns] = STEP_LORA;
      static const double cls_score[4] = {0.0, 0.6, 0.8, 1.0};  // lora_affinity.go:84-99
      for (int q = 0; q < 4; q++) p.lora_term[ns][q] = clamp01_host(cls_score[q]) * w;
    } else {
      p.kind[ns] = STEP_PAIR;
      p.arg[ns] = k - EPPSCORE_SCORER_PAIR_COL0;
    }
    ns++;
  }
  p.n_steps = ns;
  p.n_terms = nt;
  p.tie_mode = c.tie_mode;
  p.seed_lo = (uint32_t)c.tie_seed;
  p.seed_hi = (uint32_t)(c.tie_seed >> 32);
  // packed kind sequence: selects the template-specialised streaming kernels (score_dense.cu)
  p.seq = 0;
  if (ns <= 7)
    for (int i = 0; i < ns; i++) p.seq |= (uint32_t)(p.kind[i] + 1) << (4 * i);
  // sparse fast path (pick_sparse.cu): unmasked, only E/P/L steps, at most one prefix step and its
  // weight >= 0 (monotonicity: a positive match can only raise an endpoint's score)
  int n_prefix = 0;
  bool ok = !masked;
  for (int i = 0; i < ns; i++) {
    if (p.kind[i] == STEP_PREFIX) {
      n_prefix++;
      if (!(p.weight[i] >= 0.0)) ok = false;
    } else if (p.kind[i] != STEP_EP_TERM && p.kind[i] != STEP_LORA) {
      ok = false;
    }
  }
  p.pick_mode = c.pick_mode;
  p.sparse_ok = (ok && n_prefix <= 1 && c.pick_mode == EPPSCORE_PICK_MAX_SCORE) ? 1 : 0;
}

// Index mutations run on the engine stream.  They must not overtake scoring kernels that other streams launched
// earlier against the same table, and later scoring on other streams waits for ev_table.
int32_t index_begin(eppscore_engine* e) { return pending_wait(e, e->stream); }
int32_t index_end(eppscore_engine* e) {
  CK(e, cudaEventRecord(e->ev_table, e->stream));
  return EPPSCORE_OK;
}

// Prepares the terms of the profiles in `which` (bit p: profile p) from their Profile::pa on `st` and publishes them:
// ev_snapshot is recorded behind the kernels so that batches on other streams wait for the new terms (schedule_device).  The
// engine stream waits too, except while `st` is being captured into a CUDA graph: a captured stream may not take dependencies
// from outside its capture, so inside one ev_snapshot becomes a graph edge that other streams of the same capture join on, and
// in-stream order does the rest.
int32_t prepare_snapshot(eppscore_engine* e, cudaStream_t st, unsigned which) {
  for (int p = 0; p < e->n_prof; p++)
    if (which & (1u << p)) e->launches += launch_prepare_snapshot(e->prof[p].pa, st);
  CK(e, cudaGetLastError());
  unsigned long long cap_id = 0;
  const bool capturing = is_capturing(st, &cap_id);
  CK(e, cudaEventRecord(e->ev_snapshot, st));
  e->snapshot_stream = st;
  e->snapshot_capture_id = cap_id;
  if (!capturing && st != e->stream) CK(e, cudaStreamWaitEvent(e->stream, e->ev_snapshot, 0));
  return EPPSCORE_OK;
}

// Producer mutations (in-flight counters and running-request queues alike): each one waits for the previous one of either
// family (they do not all commute: remove_endpoint sets to zero, and both families prepare the same snapshot terms again),
// unless `st` is being captured, where the caller's graph edges order them.
int32_t producer_begin(eppscore_engine* e, cudaStream_t st, bool* capturing) {
  *capturing = is_capturing(st);
  if (!*capturing && e->producer_pending) CK(e, cudaStreamWaitEvent(st, e->ev_producer, 0));
  return EPPSCORE_OK;
}
// After a mutation: for the profiles whose terms read the producer's state (`feeds`, bit p: profile p), the terms that read it
// — the token-load term, the latency fold-in's endpoint arrays, the folded leading run and the per-adapter summaries of the
// sparse path — change, so those profiles are prepared again on the same stream, with eppscore_set_snapshot's ordering (a
// device-location batch another stream launched against the current terms finishes reading them first).
int32_t producer_end(eppscore_engine* e, cudaStream_t st, bool capturing, unsigned feeds) {
  if (feeds) {
    int32_t rc = capturing ? EPPSCORE_OK : pending_wait(e, st);
    if (rc == EPPSCORE_OK) rc = prepare_snapshot(e, st, feeds);
    if (rc != EPPSCORE_OK) return rc;
  }
  if (!capturing) {
    CK(e, cudaEventRecord(e->ev_producer, st));
    e->producer_pending = true;
  }
  return EPPSCORE_OK;
}

// One profile's share of a batch (eppscore_profile_run): its host-side filter result and outputs, device pointers.
struct DevRun {
  int32_t profile;
  const uint32_t* cand_mask;
  int32_t* pick;
  double* pick_score;
  int32_t* tie_count;
  double* scores_out;
  double* pred_out;
  uint32_t* filter_mask_out;
  int32_t topk;          // > 0: topk_m / topk_score [R*topk] are written
  int32_t* topk_m;
  double* topk_score;
  bool wide;             // the lists come from topk_select_kernel over the run's score rows (schedule_wide)
};

struct DevBatch {  // all device pointers
  int32_t R;
  int64_t request_base;
  const uint8_t* prompt_bytes;
  const int64_t* prompt_off;
  const int32_t* prompt_len;
  const uint64_t* model_seed;
  const uint64_t* hashes_in;
  const uint16_t* n_hashes_in;
  int32_t hash_stride;
  int32_t block_chars, max_blocks;
  const int32_t* adapter_id;
  const float* dense_feat;
  const uint16_t* dense_total;
  const int32_t* input_tokens;
  const double* ttft_slo;
  const double* tpot_slo;
  const int64_t* tokens;    // an in-order batch's per-request token estimates (schedule_inorder)
  uint16_t* match_blocks;   // profile-independent outputs, written by the kernels of run 0
  uint16_t* total_blocks;
  uint64_t* hashes_out;
  int32_t n_runs;
  DevRun run[EPPSCORE_MAX_PROFILES];
};

// How a per-request array of a batch flows.
enum class Rows {
  in,       // read by the kernels
  offsets,  // read by the kernels, R + 1 entries
  out,      // written by the kernels; a host batch copies it straight to the caller
  small,    // written by the kernels; a host batch brings it back through pinned staging (h_res)
  result,   // a small output the kernels always write: a host batch gives it scratch even when the caller did not ask for it
};

// The row layout of a batch: f(p, per, kind, slot) for each per-request array of `d` and its runs, with p a reference to the
// array's pointer (nullptr when the batch has none), per its elements per request, and slot the Scratch buffer a host batch
// stages it in (the runs share one per field).  prompt_bytes is not one of them: prompt_off indexes into it, so it is never cut.
template <typename F>
void for_each_row_array(DevBatch& d, size_t M, F&& f) {
  const size_t mw = (M + 31) / 32;
  f(d.prompt_off, 1, Rows::offsets, &Scratch::s_off);
  f(d.prompt_len, 1, Rows::in, &Scratch::s_len);
  f(d.model_seed, 1, Rows::in, &Scratch::s_seed);
  f(d.hashes_in, (size_t)d.hash_stride, Rows::in, &Scratch::s_hashes);
  f(d.n_hashes_in, 1, Rows::in, &Scratch::s_nh);
  f(d.adapter_id, 1, Rows::in, &Scratch::s_adapter);
  f(d.dense_feat, M * 4, Rows::in, &Scratch::s_dense);
  f(d.dense_total, 1, Rows::in, &Scratch::s_dtotal);
  f(d.input_tokens, 1, Rows::in, &Scratch::s_intok);
  f(d.ttft_slo, 1, Rows::in, &Scratch::s_tslo);
  f(d.tpot_slo, 1, Rows::in, &Scratch::s_pslo);
  f(d.tokens, 1, Rows::in, &Scratch::s_tokens);
  for (int i = 0; i < d.n_runs; i++) {
    DevRun& r = d.run[i];
    f(r.cand_mask, mw, Rows::in, &Scratch::s_mask);
    f(r.pick, 1, Rows::result, &Scratch::s_pick);
    f(r.pick_score, 1, Rows::result, &Scratch::s_score);
    f(r.tie_count, 1, Rows::result, &Scratch::s_tie);
    f(r.scores_out, M, Rows::out, &Scratch::s_scores);
    f(r.pred_out, M * 2, Rows::out, &Scratch::s_pred);
    f(r.filter_mask_out, mw, Rows::out, &Scratch::s_fmask);
    f(r.topk_m, (size_t)r.topk, Rows::small, &Scratch::s_topk_m);
    f(r.topk_score, (size_t)r.topk, Rows::small, &Scratch::s_topk_s);
  }
  f(d.match_blocks, M, Rows::out, &Scratch::s_match);
  f(d.total_blocks, 1, Rows::small, &Scratch::s_total);
  f(d.hashes_out, (size_t)d.max_blocks, Rows::out, &Scratch::s_hashes);  // (a host batch never has hashes_in with it)
}

// Rows [base, base + n) of a batch.
DevBatch slice_rows(DevBatch d, int32_t base, int32_t n, size_t M) {
  for_each_row_array(d, M, [base](auto*& p, size_t per, Rows, auto) {
    if (p) p += (size_t)base * per;
  });
  d.R = n;
  d.request_base += base;
  return d;
}

// The batch's arrays as one DevBatch, host or device pointers as b.location says, with block_chars / max_blocks and each run's
// list resolved.  runs: [n_runs], or nullptr for the batch's own single run on profile 0.  topk: [n_runs] validated lists, or
// nullptr for none; run i's list (k > 0) comes from the register lists of the full-matrix kernels, or from schedule_wide when
// `wide` is set or k > EPPSCORE_MAX_TOPK.
DevBatch make_batch(const eppscore_engine* e, const eppscore_batch& b, int32_t n_runs, const eppscore_profile_run* runs,
                    const eppscore_topk* topk, bool wide) {
  DevBatch d{};
  d.R = b.R;
  d.request_base = b.request_base;
  d.prompt_bytes = b.prompt_bytes;
  d.prompt_off = b.prompt_bytes ? b.prompt_off : nullptr;  // the offsets and counts are read only with what they describe
  d.prompt_len = b.prompt_len;
  d.model_seed = b.model_seed;
  d.hashes_in = b.hashes_in;
  d.n_hashes_in = b.hashes_in ? b.n_hashes_in : nullptr;
  d.hash_stride = b.hash_stride;
  d.block_chars = b.block_chars > 0 ? b.block_chars : e->cfg.block_chars;
  d.max_blocks = b.max_blocks > 0 ? b.max_blocks : e->cfg.max_blocks;
  d.adapter_id = b.adapter_id;
  d.dense_feat = b.dense_feat;
  d.dense_total = b.dense_total;
  d.input_tokens = b.input_tokens;
  d.ttft_slo = b.ttft_slo;
  d.tpot_slo = b.tpot_slo;
  d.match_blocks = b.match_blocks;
  d.total_blocks = b.total_blocks;
  d.hashes_out = b.hashes_out;
  d.n_runs = n_runs;
  for (int i = 0; i < n_runs; i++) {
    DevRun& y = d.run[i];
    auto set = [&y](const auto& x) {  // an eppscore_profile_run, or the batch itself
      y.cand_mask = x.cand_mask;
      y.pick = x.pick;
      y.pick_score = x.pick_score;
      y.tie_count = x.tie_count;
      y.scores_out = x.scores_out;
      y.pred_out = x.pred_out;
      y.filter_mask_out = x.filter_mask_out;
    };
    if (runs) {
      set(runs[i]);
      y.profile = runs[i].profile;
    } else {
      set(b);
    }
    y.topk = topk ? topk[i].k : 0;
    if (y.topk > 0) {
      y.topk_m = topk[i].endpoints;
      y.topk_score = topk[i].scores;
      y.wide = wide || y.topk > EPPSCORE_MAX_TOPK;
    }
  }
  return d;
}

// The hot path on device-resident buffers: [hash kernel] + each run's score/pick kernels, asynchronous on `s`.  The hash stage
// runs once for all runs.
int32_t schedule_device(eppscore_engine* e, const DevBatch& b, cudaStream_t s, Scratch& sc) {
  if (!e->have_snapshot) return fail(e, EPPSCORE_ERR_NO_SNAPSHOT, "schedule_batch before set_snapshot");
  if (b.R <= 0) return EPPSCORE_OK;
  const bool dense = b.dense_feat != nullptr;

  // The hash kernels do not read the snapshot terms, so the snapshot wait is issued only before the pick kernel: a caller
  // may prepare the snapshot on a second stream concurrently with the hashing of the batch.
  bool wait_snapshot = false;
  if (int32_t rc = reader_begin(e, s, nullptr, &wait_snapshot); rc != EPPSCORE_OK) return rc;

  // Per run: its profile's arguments.  A run on a profile with an endpoint subset and no cand_mask stays on the sparse path with
  // the member bitmap when that path takes it; every other run on such a profile is scored by the masked kernels on rows
  // subset ∧ cand_mask (`via_rows`).
  ScoreArgs a[EPPSCORE_MAX_PROFILES];
  bool via_rows[EPPSCORE_MAX_PROFILES] = {};
  bool any_lat = false, want_prefix = b.match_blocks || b.total_blocks || b.hashes_out;
  for (int i = 0; i < b.n_runs; i++) {
    const DevRun& run = b.run[i];
    Profile& P = e->prof[run.profile];
    if (!run.pick || !run.pick_score || !run.tie_count) return fail(e, EPPSCORE_ERR_INVALID, "pick/pick_score/tie_count required");
    if (dense && P.cfg.pick_mode != EPPSCORE_PICK_MAX_SCORE)
      return fail(e, EPPSCORE_ERR_INVALID, "the stochastic pickers are not available on dense feature rows");
    ScoreArgs& x = a[i];
    x = ScoreArgs{};
    x.geo = e->geo;
    x.geo.M = e->M;
    x.R = b.R;
    x.request_base = b.request_base;
    for (int which = 0; which < 2; which++) {
      x.minmax_q[which] = which == 0 ? e->cur_queue : e->cur_running;
      x.qhdr[which] = P.qhdr[which].as<QBucketHdr>();
      x.qbucket[which] = P.qbucket[which].as<uint32_t>();
    }
    x.cls_lo = e->cls_lo.as<uint32_t>();
    x.cls_hi = e->cls_hi.as<uint32_t>();
    x.prefix_lut2d = P.have_lut2d ? P.prefix_lut2d.as<double>() : nullptr;
    x.A = e->A;
    x.adapter_id = b.adapter_id;
    x.mask_words = (e->M + 31) / 32;
    x.dense = reinterpret_cast<const float4*>(b.dense_feat);
    x.dense_total = b.dense_total;
    x.pick = run.pick;
    x.pick_score = run.pick_score;
    x.tie_count = run.tie_count;
    x.scores_out = run.scores_out;
    x.topk = run.topk;
    x.topk_m = run.topk_m;
    x.topk_score = run.topk_score;
    if (i == 0) {
      x.match_out = b.match_blocks;
      x.total_out = b.total_blocks;
    }
    if (cfg_has(P.cfg, EPPSCORE_SCORER_LATENCY)) {
      if (dense) return fail(e, EPPSCORE_ERR_INVALID, "the latency scorer is not available on dense feature rows");
      if (!e->lat_args.enabled) return fail(e, EPPSCORE_ERR_INVALID, "latency scorer configured but the snapshot was prepared without latency params");
      any_lat = true;
      x.lat = e->lat_args;
      x.lat.input_tokens = b.input_tokens;
      x.lat.ttft_slo = b.ttft_slo;
      x.lat.tpot_slo = b.tpot_slo;
      x.lat.pred_out = run.pred_out;
      x.n_filters = P.cfg.n_filters;
      for (int f = 0; f < P.cfg.n_filters; f++) {
        x.filter_kind[f] = P.cfg.filter_kind[f];
        for (int q = 0; q < 3; q++) x.filter_param[f][q] = P.cfg.filter_param[f][q];
      }
      x.filter_mask_out = run.filter_mask_out;
    }
    if (cfg_has(P.cfg, EPPSCORE_SCORER_PREFIX) || cfg_has(P.cfg, EPPSCORE_SCORER_LATENCY)) want_prefix = true;
    // the unmasked form first: it decides whether the sparse path takes the run
    const PlanSet& pu = P.plan_unmasked;
    x.plan = pu.plan;
    for (int t = 0; t < pu.plan.n_terms; t++) x.term[t] = pu.term_ptr[t];
    x.summ = pu.plan.sparse_ok ? P.summ.as<AdapterSummary>() : nullptr;
    x.tiemask = pu.plan.sparse_ok ? P.tiemask.as<uint32_t>() : nullptr;
    x.member = P.subset ? P.member_perm.as<uint32_t>() : nullptr;
    x.cand_mask = run.cand_mask;
    if (P.subset && (run.cand_mask || dense || e->force_generic || !pick_sparse_applies(x))) {
      via_rows[i] = true;
      x.member = nullptr;
      x.cand_mask = nullptr;  // the rows in sc.s_subset (reserved below, before the first launch)
    }
    if (run.cand_mask || via_rows[i]) {
      const PlanSet& pm = P.plan_masked;
      x.plan = pm.plan;
      for (int t = 0; t < kMaxSteps; t++) x.term[t] = t < pm.plan.n_terms ? pm.term_ptr[t] : nullptr;
      x.summ = nullptr;
      x.tiemask = nullptr;
    }
  }
  const size_t rows_bytes = (size_t)b.R * ((e->M + 31) / 32) * 4;
  for (int i = 0; i < b.n_runs; i++)
    if (via_rows[i] || e->prof[b.run[i].profile].subset) {  // (a sparse run on a subset may defer requests to member rows)
      CK(e, sc.s_subset.reserve(rows_bytes));
      break;
    }
  for (int i = 0; i < b.n_runs; i++)
    if (via_rows[i]) a[i].cand_mask = sc.s_subset.as<uint32_t>();
  if (any_lat && !b.input_tokens && b.prompt_bytes && b.prompt_off) {  // count the fields of the prompt bytes on the device
    CK(e, sc.s_fields.reserve((size_t)b.R * 4));
    e->launches += launch_count_fields(b.prompt_bytes, b.prompt_off, b.prompt_len, b.R, sc.s_fields.as<int32_t>(), s, e->sm_count);
    for (int i = 0; i < b.n_runs; i++)
      if (a[i].lat.enabled) a[i].lat.input_tokens = sc.s_fields.as<int32_t>();
  }

  bool hashed_here = false;
  const uint64_t* hashes = nullptr;
  const uint16_t* n_hashes = nullptr;
  int32_t hash_stride = 0;
  const ProbeRec* probe = nullptr;
  const TableView* table = nullptr;
  if (!dense && want_prefix && (b.hashes_in || b.prompt_bytes)) {
    if (b.hashes_in) {
      if (!b.n_hashes_in || b.hash_stride <= 0) return fail(e, EPPSCORE_ERR_INVALID, "hashes_in needs n_hashes_in and hash_stride");
      hashes = b.hashes_in;
      n_hashes = b.n_hashes_in;
      hash_stride = b.hash_stride;
    } else {
      const int32_t bc = b.block_chars, mb = b.max_blocks;
      if (mb > EPPSCORE_MAX_BLOCKS) return fail(e, EPPSCORE_ERR_CAPACITY, "max_blocks > 65535");
      if (!b.prompt_off) return fail(e, EPPSCORE_ERR_INVALID, "prompt_off required with prompt_bytes");
      uint64_t* hout = b.hashes_out;
      if (!hout) {
        CK(e, sc.s_hashes.reserve((size_t)b.R * mb * 8));
        hout = sc.s_hashes.as<uint64_t>();
      }
      CK(e, sc.s_nh.reserve((size_t)b.R * 2));
      HashArgs h{};
      h.R = b.R;
      h.bytes = b.prompt_bytes;
      h.off = b.prompt_off;
      h.len = b.prompt_len;
      h.seed = b.model_seed;
      h.block_chars = bc;
      h.max_blocks = mb;
      h.hashes = hout;
      h.stride = mb;
      h.n_hashes = sc.s_nh.as<uint16_t>();
      h.stage_mask = e->hash_stage_mask;
      h.pdl = e->use_pdl ? 1 : 0;
      // the sparse pick kernel follows and would probe the index: the hash kernel probes it instead while it holds the
      // hashes, and leaves the rows it resolved out of the hash buffer.  Not when the caller wants every row (hashes_out,
      // the closed loop's commit input): then no write is saved, and on H100 the schedule call measured slower that way.
      // With several runs, every run that reads the hashes must be one that takes the records.
      bool probe_ok = !e->force_generic && !b.hashes_out && hash_probe_applies(h), probes = false;
      for (int i = 0; i < b.n_runs && probe_ok; i++) {
        const Plan& pl = a[i].plan;
        bool reads = a[i].match_out || a[i].total_out;
        for (int t = 0; t < pl.n_steps; t++) reads = reads || pl.kind[t] == STEP_PREFIX || pl.kind[t] == STEP_LATENCY;
        const bool takes = pick_sparse_probes(a[i]);
        if (reads && !takes) probe_ok = false;
        probes = probes || takes;
      }
      if (probe_ok && probes) {
        CK(e, sc.s_probe.reserve((size_t)b.R * sizeof(ProbeRec)));
        h.table = e->index->view();
        h.probe = sc.s_probe.as<ProbeRec>();
        h.resolved = e->probe_resolved.as<unsigned long long>();
        probe = h.probe;
      }
      e->launches += launch_hash_prompts(h, s, e->sm_count);
      hashed_here = true;
      hashes = hout;
      n_hashes = h.n_hashes;
      hash_stride = mb;
    }
    table = e->index->view();
  }
  if (wait_snapshot) CK(e, cudaStreamWaitEvent(s, e->ev_snapshot, 0));
  for (int i = 0; i < b.n_runs; i++) {
    ScoreArgs& x = a[i];
    const Profile& P = e->prof[b.run[i].profile];
    x.hashes = hashes;
    x.n_hashes = n_hashes;
    x.hash_stride = hash_stride;
    x.table = table;
    x.probe = pick_sparse_probes(x) ? probe : nullptr;
    if (via_rows[i]) {
      e->launches += launch_subset_mask(P.member_nat.as<uint32_t>(), b.run[i].cand_mask, b.R, x.mask_words, nullptr,
                                        sc.s_subset.as<uint32_t>(), s, e->sm_count);
      CK(e, cudaGetLastError());
    }
    // programmatic dependent launch when the previous kernel of the stream is this batch's hash kernel (the snapshot event,
    // when there is one, stays a full dependency of the pick kernel)
    x.pdl = (e->use_pdl && hashed_here && i == 0 && !via_rows[i]) ? 1 : 0;
    // dispatch: specialised fast paths first, the fully general kernels otherwise
    int launched = 0;
    if (!e->force_generic) launched = dense ? launch_score_dense_fast(x, s, e->sm_count) : launch_pick_sparse(x, s, e->sm_count);
    const bool sparse = launched > 0 && !dense;
    if (launched == 0) launched = launch_score_pick(x, dense, s, e->sm_count);
    if (launched > 0 && sparse && x.member && x.table && x.hashes) {
      // the requests the sparse kernel deferred: the masked full-matrix kernel on their member rows
      e->launches += launch_subset_mask(P.member_nat.as<uint32_t>(), nullptr, b.R, x.mask_words, x.pick, sc.s_subset.as<uint32_t>(),
                                        s, e->sm_count);
      ScoreArgs d = x;
      const PlanSet& pm = P.plan_masked;
      d.plan = pm.plan;
      for (int t = 0; t < kMaxSteps; t++) d.term[t] = t < pm.plan.n_terms ? pm.term_ptr[t] : nullptr;
      d.summ = nullptr;
      d.tiemask = nullptr;
      d.member = nullptr;
      d.probe = nullptr;
      d.cand_mask = sc.s_subset.as<uint32_t>();
      d.only_deferred = 1;
      d.pdl = 0;
      const int deferred = launch_score_matrix(d, s, e->sm_count);
      launched = deferred < 0 ? deferred : launched + deferred;
    }
    if (launched < 0) {
      cudaGetLastError();  // (a failed launch is not sticky: clear it so the next call does not report it again)
      return cuda_fail(e, (cudaError_t)-launched, "scoring kernel launch");
    }
    e->launches += launched;
    CK(e, cudaGetLastError());
  }
  return EPPSCORE_OK;
}

// Rows per slice of a wide top-k batch: a fixed byte budget of score rows.  Step 2 reads the slice right after step 1 wrote
// it, so a slice that fits the H100's 50 MB L2 is read from L2 instead of HBM.  Measured with tools/prof_topk_wide.py at the
// headline shape (64K x 1024, k = 16, H100 80GB HBM3 at 700 W): 32 MiB (16 slices) 1.96 / 2.57 / 2.06 ms for max-score /
// weighted-random / random, 512 MiB (one slice, -DEPP_WIDE_SLICE_BYTES) 1.70 / 2.32 / 1.85 ms.  The L2 reuse does not pay
// for the per-slice launches; 32 MiB stays because the large budget costs 16x the memory (two 512 MiB slots plus a hash
// scratch for 64K rows) for about 12 %.
#ifndef EPP_WIDE_SLICE_BYTES
#define EPP_WIDE_SLICE_BYTES (32ull << 20)
#endif
constexpr unsigned long long kWideSliceBytes = EPP_WIDE_SLICE_BYTES;

// eppscore_schedule_batch_topk_wide, and a batch of eppscore_schedule_batch_profiles_topk with a run of k > EPPSCORE_MAX_TOPK,
// on device buffers, asynchronous on `s`, in two steps per slice of rows:
//   1. one schedule_device over every run: a wide run takes the scores_out route (the diagnostics variants of the full-matrix
//      and generic dense kernels), which writes the slice's weighted scores, NaN for non-candidates, into the run's part of
//      sc.wide (or into the run's own scores_out, which then needs no slicing), together with pick / pick_score /
//      tie_count; the other runs compute what they compute outside this function, register lists included;
//   2. per wide run, topk_select_kernel turns its rows into its lists [R][k], with its profile's pick mode and seed.
// The scratch holds wide_rows rows whatever the runs: with n wide runs on it, a slice is wide_rows / n rows per run, so a graph
// captured after the first wide call keeps pointing at live memory.  The slices run in order on `s` (the scratch holds one
// slice), whatever the slicing keys 5 / 6 say.
int32_t schedule_wide(eppscore_engine* e, const DevBatch& d, cudaStream_t s, Scratch& sc) {
  if (!e->have_snapshot) return fail(e, EPPSCORE_ERR_NO_SNAPSHOT, "schedule_batch before set_snapshot");
  if (d.R <= 0) return EPPSCORE_OK;
  const size_t M = (size_t)e->M, mw = (M + 31) / 32, mb = (size_t)d.max_blocks;
  auto select = [&](const DevBatch& q, const DevRun& run) -> int32_t {
    const Profile& P = e->prof[run.profile];
    TopKSelectArgs t{};
    t.scores = run.scores_out;
    t.R = q.R;
    t.M = e->M;
    t.k = run.topk;
    t.pick_mode = P.cfg.pick_mode;
    t.tie_mode = P.cfg.tie_mode;
    t.seed_lo = (uint32_t)P.cfg.tie_seed;
    t.seed_hi = (uint32_t)(P.cfg.tie_seed >> 32);
    t.request_base = q.request_base;
    t.out_m = run.topk_m;
    t.out_s = run.topk_score;
    const int launched = launch_topk_select(t, s);
    if (launched < 0) {
      cudaGetLastError();
      return cuda_fail(e, (cudaError_t)-launched, "topk_select_kernel launch");
    }
    e->launches += launched;
    CK(e, cudaGetLastError());
    return EPPSCORE_OK;
  };
  // step 1 with the wide runs' lists left to step 2, then step 2
  auto run_slice = [&](const DevBatch& q) -> int32_t {
    DevBatch x = q;
    for (int i = 0; i < x.n_runs; i++)
      if (x.run[i].wide) x.run[i].topk = 0;
    int32_t rc = schedule_device(e, x, s, sc);
    for (int i = 0; i < q.n_runs && rc == EPPSCORE_OK; i++)
      if (q.run[i].wide) rc = select(q, q.run[i]);
    return rc;
  };
  int32_t n_scratch = 0;  // wide runs whose rows go to the scratch
  bool any_subset = false, any_lat = false;
  for (int i = 0; i < d.n_runs; i++) {
    const Profile& P = e->prof[d.run[i].profile];
    if (d.run[i].wide && !d.run[i].scores_out) n_scratch++;
    any_subset = any_subset || P.subset;
    any_lat = any_lat || cfg_has(P.cfg, EPPSCORE_SCORER_LATENCY);
  }
  if (n_scratch == 0) return run_slice(d);
  DevBuf& buf = sc.wide;
  if (!buf.p) {
    if (is_capturing(s))
      return fail(e, EPPSCORE_ERR_CAPACITY,
                  "the first eppscore_schedule_batch_topk_wide allocates the engine's score scratch: make one wide call outside "
                  "the CUDA-graph capture first");
    CK(e, buf.reserve((size_t)e->wide_rows * e->geo.Mpad * 8));
  }
  // the per-slice hash scratch is sized for a whole slice up front, so a larger wide call later does not move it under a
  // captured graph (a reserved stream's set holds every slice of the batches it takes already: no slice is longer than its batch)
  const size_t srows = (size_t)(sc.rows > 0 ? std::min(e->wide_rows, sc.rows) : e->wide_rows);
  if (d.prompt_bytes && !d.hashes_in && !d.hashes_out) {
    CK(e, sc.s_hashes.reserve(srows * mb * 8));
    CK(e, sc.s_nh.reserve(srows * 2));
  }
  if (d.prompt_bytes && !d.input_tokens && any_lat) CK(e, sc.s_fields.reserve(srows * 4));
  if (any_subset) CK(e, sc.s_subset.reserve(srows * mw * 4));
  // a run next to the wide ones may take the hash kernel's probe records
  if (d.n_runs > 1 && d.prompt_bytes && !d.hashes_in && !d.hashes_out) CK(e, sc.s_probe.reserve(srows * sizeof(ProbeRec)));
  // n_scratch parts of rows * M doubles must fit the wide_rows * Mpad of the scratch: a slice budget (EPP_WIDE_SLICE_BYTES) of
  // fewer rows than wide runs cannot hold one row per run
  if (e->wide_rows < n_scratch)
    return fail(e, EPPSCORE_ERR_CAPACITY, "the wide score scratch holds fewer rows than the call has wide runs (EPP_WIDE_SLICE_BYTES)");
  const int32_t rows = e->wide_rows / n_scratch;
  for (int32_t base = 0; base < d.R; base += rows) {
    DevBatch q = slice_rows(d, base, std::min(rows, d.R - base), M);
    for (int i = 0, j = 0; i < q.n_runs; i++)
      if (q.run[i].wide && !d.run[i].scores_out) q.run[i].scores_out = buf.as<double>() + (size_t)(j++) * rows * M;
    int32_t rc = run_slice(q);
    if (rc != EPPSCORE_OK) return rc;
  }
  return EPPSCORE_OK;
}

// Copies the bytes of prompts [r0, r1) from the host to `buf` on `st`; *out is the device base that the caller's offsets
// index into.  The extent comes from prompt_off (and prompt_len when given).  The copy starts at a 16-byte aligned source
// offset so every prompt keeps its alignment (the fast hash path needs 16-byte aligned starts), and is padded by 64 B so
// 16-byte vector loads of the last block never leave the allocation.
int32_t stage_prompts(eppscore_engine* e, DevBuf& buf, const uint8_t* bytes, const int64_t* off, const int32_t* len, int32_t r0,
                      int32_t r1, cudaStream_t st, const uint8_t** out) {
  size_t lo = (size_t)off[r0], hi = (size_t)off[r1];
  if (len) {
    lo = SIZE_MAX;
    hi = 0;
    for (int32_t r = r0; r < r1; r++) {
      lo = std::min(lo, (size_t)off[r]);
      hi = std::max(hi, (size_t)off[r] + (size_t)len[r]);
    }
    if (lo > hi) lo = hi = 0;
  }
  const size_t start = lo & ~(size_t)15;
  CK(e, buf.reserve(hi - start + 64));
  if (hi > start) CK(e, cudaMemcpyAsync(buf.p, bytes + start, hi - start, cudaMemcpyHostToDevice, st));
  *out = buf.as<uint8_t>() - start;
  return EPPSCORE_OK;
}

// One copy of a host-array call's results (HostStage, schedule_batch).
struct Copy {
  void* dst;
  const void* src;
  size_t bytes;
};

// The staging of one host-array call: its inputs, prompt bytes and outputs each take the next of e->stage's slots, in call
// order, and are copied on the engine stream.  finish() runs the call's device form, copies the outputs back and synchronises
// the engine stream, after which the caller's arrays may be reused and the slots serve the next call.  The first failure is
// kept: finish() returns it without running anything.
class HostStage {
 public:
  explicit HostStage(eppscore_engine* e) : e_(e) {}
  // The next slot, holding n elements of T.
  template <typename T>
  T* slot(size_t n) {
    DevBuf& b = next();
    return check(b.reserve(n * sizeof(T)), "staging allocation") ? b.as<T>() : nullptr;
  }
  // rows[0..n_rows) of n elements each, one after the other in one slot; nullptr when there are none.
  template <typename T>
  const T* in(const T* const* rows, int n_rows, size_t n) {
    if (!rows[0] || n == 0) return nullptr;
    T* d = slot<T>(n_rows * n);
    for (int i = 0; i < n_rows && d; i++)
      check(cudaMemcpyAsync(d + i * n, rows[i], n * sizeof(T), cudaMemcpyHostToDevice, e_->stream), "staging copy");
    return d;
  }
  template <typename T>
  const T* in(const T* src, size_t n) { return in(&src, 1, n); }
  // The bytes prompts [0, R) reach (stage_prompts).
  const uint8_t* prompts(const uint8_t* bytes, const int64_t* off, const int32_t* len, int32_t R) {
    const uint8_t* d = nullptr;
    DevBuf& b = next();
    if (rc_ == EPPSCORE_OK) rc_ = stage_prompts(e_, b, bytes, off, len, 0, R, e_->stream, &d);
    return d;
  }
  // A slot for n elements the device form writes, copied back to dst by finish(); zeroed first when `zero` is set.  nullptr
  // when dst is.
  template <typename T>
  T* out(T* dst, size_t n, bool zero = false) {
    if (!dst) return nullptr;
    T* d = slot<T>(n);
    if (d && zero) check(cudaMemsetAsync(d, 0, n * sizeof(T), e_->stream), "staging memset");
    if (d) back_.push_back({dst, d, n * sizeof(T)});
    return d;
  }
  template <typename F>
  int32_t finish(F&& call) {
    int32_t rc = rc_ == EPPSCORE_OK ? call() : rc_;
    if (rc != EPPSCORE_OK) return rc;
    for (const Copy& b : back_) CK(e_, cudaMemcpyAsync(b.dst, b.src, b.bytes, cudaMemcpyDeviceToHost, e_->stream));
    CK(e_, cudaStreamSynchronize(e_->stream));
    return EPPSCORE_OK;
  }

 private:
  DevBuf& next() {
    assert(next_ < (int)std::size(e_->stage) && "HostStage: more arrays than e->stage has slots");
    return e_->stage[next_++];
  }
  bool check(cudaError_t c, const char* what) {
    if (c != cudaSuccess && rc_ == EPPSCORE_OK) rc_ = cuda_fail(e_, c, what);
    return rc_ == EPPSCORE_OK;
  }
  eppscore_engine* e_;
  int next_ = 0;
  int32_t rc_ = EPPSCORE_OK;
  std::vector<Copy> back_;
};

constexpr int64_t kRunInitialSlots = 4096;

// A running-request table of `slots` slots (a power of two) in t[0..3] (slot, tpot, owner, rm), empty: slots {0, 0}, no
// bids.  tpot needs no initial value.
cudaError_t run_alloc_table(int64_t slots, DevBuf* t, cudaStream_t st) {
  const size_t n = (size_t)slots;
  cudaError_t c;
  if ((c = t[0].reserve(n * sizeof(RunSlot))) != cudaSuccess) return c;
  for (int i = 1; i < 4; i++)
    if ((c = t[i].reserve(n * 8)) != cudaSuccess) return c;
  if ((c = cudaMemsetAsync(t[0].p, 0, n * sizeof(RunSlot), st)) != cudaSuccess) return c;
  if ((c = cudaMemsetAsync(t[2].p, 0xff, n * 8, st)) != cudaSuccess) return c;
  return cudaMemsetAsync(t[3].p, 0xff, n * 8, st);
}

// The descriptor as created: tab[0..3] the table, tab[4..7] its spare, the per-endpoint arrays, the scratch.
void run_init_desc(eppscore_engine* e) {
  RunDev& d = e->run_host;
  d.slot = e->run_tab[0].as<RunSlot>();
  d.tpot = e->run_tab[1].as<unsigned long long>();
  d.owner = e->run_tab[2].as<unsigned long long>();
  d.rm = e->run_tab[3].as<unsigned long long>();
  d.spare_slot = e->run_tab[4].as<RunSlot>();
  d.spare_tpot = e->run_tab[5].as<unsigned long long>();
  d.spare_owner = e->run_tab[6].as<unsigned long long>();
  d.spare_rm = e->run_tab[7].as<unsigned long long>();
  d.mask = (unsigned long long)e->run_cap - 1;
  d.count = e->run_count.as<int>();
  d.min_bits = e->run_min_bits.as<unsigned long long>();
  d.min_cnt = e->run_min_cnt.as<int>();
  d.min_view = e->run_min_view.as<double>();
  d.dirty = e->run_dirty.as<unsigned>();
  d.rc_min = e->run_rc_min.as<unsigned long long>();
  d.rc_cnt = e->run_rc_cnt.as<int>();
  d.ctr = e->run_ctr.as<RunCounters>();
  d.slot_of = e->c_rslot.as<int32_t>();
  d.won = e->c_rwon.as<uint8_t>();
}

// The per-profile fields of a config (eppscore_create, eppscore_add_profile): nullptr when they are valid, else the reason.
const char* profile_error(const eppscore_config& c) {
  if (c.n_scorers < 0 || c.n_scorers > EPPSCORE_MAX_SCORERS) return "n_scorers out of range";
  int nlat = 0;
  for (int i = 0; i < c.n_scorers; i++) {
    const int k = c.scorer_kind[i];
    const bool ok = (k >= 0 && k <= 6) || (k >= 8 && k < 12) || (k >= 16 && k < 18);
    if (!ok) return "unknown scorer kind";
    nlat += k == EPPSCORE_SCORER_LATENCY;
  }
  if (nlat > 1) return "at most one latency scorer per profile";
  if (c.pick_mode < 0 || c.pick_mode > EPPSCORE_PICK_RANDOM) return "unknown pick_mode";
  if (c.n_filters < 0 || c.n_filters > EPPSCORE_MAX_FILTERS) return "n_filters out of range";
  if (c.n_filters > 0) {
    if (!cfg_has(c, EPPSCORE_SCORER_LATENCY)) return "device-side filters need the latency scorer in the profile";
    if (cfg_has(c, EPPSCORE_SCORER_QUEUE) || cfg_has(c, EPPSCORE_SCORER_RUNNING))
      return "device-side filters cannot be combined with the queue / running scorers";
    for (int f = 0; f < c.n_filters; f++) {
      const int k = c.filter_kind[f];
      const double* par = c.filter_param[f];
      if (k == EPPSCORE_FILTER_PREFIX_AFFINITY) {  // prefixcacheaffinity/plugin.go:80-91
        if (par[0] > 1.0 || par[1] < 0 || par[1] > 1.0 || par[2] < 0) return "prefix-cache-affinity-filter: invalid parameters";
      } else if (k == EPPSCORE_FILTER_SLO_HEADROOM_TIER) {  // sloheadroomtier/plugin.go:66-68
        if (par[0] < 0 || par[0] > 1.0) return "slo-headroom-tier-filter: epsilonExploreNeg must be in [0, 1]";
      } else {
        return "unknown filter kind";
      }
    }
  }
  return nullptr;
}

// Sizes profile p's buffers (and the engine's latency buffers when it is the first latency profile), builds its plans and its
// prefix term table, synchronously on the engine stream.  `ef` receives the error (nullptr inside eppscore_create).
int32_t profile_init(eppscore_engine* e, eppscore_engine* ef, int32_t p) {
  Profile& P = e->prof[p];
  const size_t mp = (size_t)e->geo.Mpad;
  for (int which = 0; which < 2; which++)  // value buckets for the masked min/max of the queue / running scorers
    if (cfg_has(P.cfg, which == 0 ? EPPSCORE_SCORER_QUEUE : EPPSCORE_SCORER_RUNNING)) {
      CK(ef, P.qhdr[which].reserve(sizeof(QBucketHdr)));
      CK(ef, P.qbucket[which].reserve((size_t)kQBuckets * (mp / 32) * 4));
      CK(ef, cudaMemsetAsync(P.qhdr[which].p, 0, sizeof(QBucketHdr), e->stream));
    }
  if (cfg_has(P.cfg, EPPSCORE_SCORER_LATENCY) && !e->lat_ep.p) {
    CK(ef, e->raw_min_tpot.reserve(mp * 8));
    CK(ef, e->raw_dispatched.reserve(mp * 4));
    CK(ef, e->raw_prefill.reserve(mp));
    CK(ef, e->lat_ep.reserve(mp * 8 * kLatArrays));
  }
  for (int i = 0; i < kMaxSteps; i++) CK(ef, P.term[i].reserve(mp * 8));
  CK(ef, P.fold_unmasked.reserve(mp * 8));
  CK(ef, P.fold_masked.reserve(mp * 8));
  CK(ef, P.summ.reserve((size_t)(e->A_cap + 1) * sizeof(AdapterSummary)));
  CK(ef, P.tiemask.reserve((size_t)(e->A_cap + 1) * e->geo.row_words * 4));
  for (DevBuf* b : {&P.member_nat, &P.next_nat}) CK(ef, b->reserve(mp / 32 * 4));
  for (DevBuf* b : {&P.member_perm, &P.next_perm}) CK(ef, b->reserve((size_t)e->geo.row_words * 4));
  build_plan(P, false, &P.plan_unmasked);
  build_plan(P, true, &P.plan_masked);
  // prefix term table for the sparse path: lut2d[total][c] = clamp(c/total) * w  (prefix/plugin.go:108-110,
  // scheduler_profile.go:168) — one IEEE divide and one multiply per entry, computed here on the host (no contraction:
  // this file is compiled with -ffp-contract=off)
  for (int sidx = 0; sidx < P.plan_unmasked.plan.n_steps; sidx++) {
    if (P.plan_unmasked.plan.kind[sidx] != STEP_PREFIX) continue;
    const double w = P.plan_unmasked.plan.weight[sidx];
    std::vector<double> lut((size_t)(kLutMax + 1) * (kLutMax + 1), 0.0);
    for (int total = 0; total <= kLutMax; total++)
      for (int c = 0; c <= kLutMax; c++) {
        volatile double sc = 0.0;
        if (total != 0) sc = (double)c / (double)total;
        volatile double cl = clamp01_host(sc);
        lut[(size_t)total * (kLutMax + 1) + c] = cl * w;
      }
    CK(ef, P.prefix_lut2d.reserve(lut.size() * 8));
    CK(ef, cudaMemcpy(P.prefix_lut2d.p, lut.data(), lut.size() * 8, cudaMemcpyHostToDevice));
    P.have_lut2d = true;
    break;
  }
  return EPPSCORE_OK;
}

// Profile p's preparation arguments: the snapshot's shared part (e->base_pa) and the profile's own scorers, buffers and subset.
void profile_pa(eppscore_engine* e, int32_t p) {
  Profile& P = e->prof[p];
  PrepareArgs pa = e->base_pa;
  const eppscore_config& c = P.cfg;
  pa.n_scorers = c.n_scorers;
  for (int i = 0; i < c.n_scorers; i++) {
    pa.kind[i] = c.scorer_kind[i];
    pa.weight[i] = c.scorer_weight[i];
    pa.term[i] = is_endpoint_term_kind(pa.kind[i], false) ? P.term[i].as<double>() : nullptr;
  }
  for (int which = 0; which < 2; which++) {
    pa.qhdr[which] = P.qhdr[which].as<QBucketHdr>();
    pa.qbucket[which] = P.qbucket[which].as<uint32_t>();
  }
  if (!cfg_has(c, EPPSCORE_SCORER_LATENCY)) pa.lat_ep = nullptr;  // (the latency profiles write the engine's arrays)
  int lead_u = 0, lead_m = 0;
  while (lead_u < c.n_scorers && is_endpoint_term_kind(c.scorer_kind[lead_u], false)) lead_u++;
  while (lead_m < c.n_scorers && is_endpoint_term_kind(c.scorer_kind[lead_m], true)) lead_m++;
  pa.fold_unmasked = lead_u ? P.fold_unmasked.as<double>() : nullptr;
  pa.fold_unmasked_n = lead_u;
  pa.fold_masked = lead_m ? P.fold_masked.as<double>() : nullptr;
  pa.fold_masked_n = lead_m;
  pa.plan_u = P.plan_unmasked.plan;
  for (int t = 0; t < kMaxSteps; t++) pa.plan_term[t] = P.plan_unmasked.term_ptr[t];
  pa.summ = P.plan_unmasked.plan.sparse_ok ? P.summ.as<AdapterSummary>() : nullptr;
  pa.tiemask = P.tiemask.as<uint32_t>();
  pa.member = P.subset ? P.member_nat.as<uint32_t>() : nullptr;
  P.pa = pa;
}

}  // namespace

// ================================================================================================
// C ABI
// ================================================================================================
extern "C" {

int32_t eppscore_abi_version(void) { return EPPSCORE_ABI_VERSION; }

void eppscore_config_default(eppscore_config* c) {
  memset(c, 0, sizeof(*c));
  c->struct_size = sizeof(*c);
  // loader/defaults.go:46-103: queue 2, kv 2, prefix 3, max-score picker
  c->n_scorers = 3;
  c->scorer_kind[0] = EPPSCORE_SCORER_QUEUE;
  c->scorer_weight[0] = 2.0;
  c->scorer_kind[1] = EPPSCORE_SCORER_KV_CACHE;
  c->scorer_weight[1] = 2.0;
  c->scorer_kind[2] = EPPSCORE_SCORER_PREFIX;
  c->scorer_weight[2] = 3.0;
  c->block_chars = 16 * 4;  // approximateprefix/types.go:91,112
  c->max_blocks = 256;      // types.go:98
  c->tie_mode = EPPSCORE_TIE_LOWEST_INDEX;
  c->tie_seed = 0;
  c->max_endpoints = 1024;
  c->max_adapters = 64;
  c->prefix_capacity = 1 << 18;
  c->lru_capacity_default = 31250;  // types.go:109
  c->token_load_threshold = 4194304.0;  // tokenQueueThresholdDefault, token_load.go:33
}

void eppscore_latency_params_default(eppscore_latency_params* p) {
  memset(p, 0, sizeof(*p));
  p->struct_size = sizeof(*p);
  p->has_predictions = 1;
  p->slo_buffer_factor = 1.0;  // predictedlatency/plugin.go:132
  p->streaming_mode = 0;       // :134
  p->strategy_most = 0;        // scorer/latency/plugin.go:86 "least"
  p->ttft_weight = 0.8;        // :84-85
  p->tpot_weight = 0.2;
  p->composite_kv = p->composite_queue = p->composite_prefix = 1.0;  // :87-89
}

int32_t eppscore_set_latency_params(eppscore_engine* e, const eppscore_latency_params* p) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (!p || p->struct_size != sizeof(eppscore_latency_params)) return fail(e, EPPSCORE_ERR_INVALID, "latency params NULL or struct_size mismatch");
  if (!(p->slo_buffer_factor > 0)) return fail(e, EPPSCORE_ERR_INVALID, "sloBufferFactor must be > 0");  // predictedlatency/plugin.go:169
  e->lat_params = *p;
  return EPPSCORE_OK;
}

int32_t eppscore_create(int32_t device, const eppscore_config* cfg, eppscore_engine** out) {
  if (!out) return fail(nullptr, EPPSCORE_ERR_INVALID, "out is NULL");
  *out = nullptr;
  if (!cfg || cfg->struct_size != sizeof(eppscore_config))
    return fail(nullptr, EPPSCORE_ERR_INVALID, "config NULL or struct_size mismatch");
  if (const char* why = profile_error(*cfg)) return fail(nullptr, EPPSCORE_ERR_INVALID, why);
  if (cfg->max_endpoints < 1 || cfg->max_endpoints > 8192)
    return fail(nullptr, EPPSCORE_ERR_CAPACITY, "max_endpoints must be in [1, 8192]");
  if (cfg->max_blocks < 0 || cfg->max_blocks > EPPSCORE_MAX_BLOCKS) return fail(nullptr, EPPSCORE_ERR_CAPACITY, "max_blocks out of range");
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev <= 0)
    return fail(nullptr, EPPSCORE_ERR_NO_DEVICE,
                std::string("no CUDA device (the engine has no CPU path): ") + cudaGetErrorString(ce));
  if (device < 0 || device >= ndev) return fail(nullptr, EPPSCORE_ERR_NO_DEVICE, "device index out of range");
  auto e = std::make_unique<eppscore_engine>();
  e->device = device;
  e->cfg = *cfg;
  if (e->cfg.block_chars == 0) e->cfg.block_chars = 64;
  if (e->cfg.max_blocks == 0) e->cfg.max_blocks = 256;
  if (e->cfg.max_adapters < 1) e->cfg.max_adapters = 64;
  if (e->cfg.prefix_capacity <= 0) e->cfg.prefix_capacity = 1 << 18;
  if (e->cfg.lru_capacity_default <= 0) e->cfg.lru_capacity_default = 31250;
  if (!(e->cfg.token_load_threshold > 0)) e->cfg.token_load_threshold = 4194304.0;  // token_load.go:57-61
  eppscore_latency_params_default(&e->lat_params);
  e->geo = make_geo(e->cfg.max_endpoints);
  e->A_cap = (e->cfg.max_adapters + 63) / 64 * 64;
  e->wide_rows = (int32_t)std::max<unsigned long long>(1, kWideSliceBytes / ((unsigned long long)e->geo.Mpad * 8));
  if (e->cfg.lru_capacity_max < 0) return fail(nullptr, EPPSCORE_ERR_INVALID, "lru_capacity_max < 0");
  eppscore_engine* ep = e.get();
  CK(nullptr, cudaSetDevice(device));
  cudaDeviceProp prop;
  CK(nullptr, cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(nullptr, EPPSCORE_ERR_NO_DEVICE, "device is not sm_90 (this library ships sm_90a code only)");
  ep->sm_count = prop.multiProcessorCount;
  {
    const char* fg = getenv("EPPSCORE_FORCE_GENERIC");
    ep->force_generic = fg && fg[0] == '1';
  }
  // every failure below frees what was allocated before it (the engine's members own it)
  CK(nullptr, make(ep->stream));
  CK(nullptr, make(ep->ev_snapshot));
  CK(nullptr, make(ep->ev_subset));
  CK(nullptr, make(ep->ev_table));
  // endpoint tile buffers
  const size_t mp = (size_t)ep->geo.Mpad;
  CK(nullptr, ep->raw_kv.reserve(mp * 8));
  CK(nullptr, ep->raw_queue.reserve(mp * 8));
  CK(nullptr, ep->raw_running.reserve(mp * 8));
  CK(nullptr, ep->raw_act.reserve(mp * (ep->A_cap / 64) * 8));
  CK(nullptr, ep->raw_wait.reserve(mp * (ep->A_cap / 64) * 8));
  CK(nullptr, ep->raw_nmodels.reserve(mp * 4));
  CK(nullptr, ep->raw_max.reserve(mp * 4));
  for (int i = 0; i < 4; i++) CK(nullptr, ep->raw_col[i].reserve(mp * 8));
  CK(nullptr, ep->raw_tokens.reserve(mp * 8));
  CK(nullptr, ep->inflight_req.reserve(mp * 8));
  CK(nullptr, ep->inflight_tok.reserve(mp * 8));
  CK(nullptr, ep->inflight_err.reserve(4));
  CK(nullptr, cudaMemsetAsync(ep->inflight_req.p, 0, mp * 8, ep->stream));
  CK(nullptr, cudaMemsetAsync(ep->inflight_tok.p, 0, mp * 8, ep->stream));
  CK(nullptr, cudaMemsetAsync(ep->inflight_err.p, 0, 4, ep->stream));
  CK(nullptr, ep->probe_resolved.reserve(8));
  CK(nullptr, cudaMemsetAsync(ep->probe_resolved.p, 0, 8, ep->stream));
  CK(nullptr, make(ep->ev_producer));
  CK(nullptr, make(ep->ev_count_read));
  CK(nullptr, init_inflight_update());
  {  // running-request queues: every endpoint empty, a small table (grown by the first calls that need room)
    CK(nullptr, ep->run_count.reserve(mp * 4));
    CK(nullptr, ep->run_min_bits.reserve(mp * 8));
    CK(nullptr, ep->run_min_cnt.reserve(mp * 4));
    CK(nullptr, ep->run_min_view.reserve(mp * 8));
    CK(nullptr, ep->run_dirty.reserve(mp * 4));
    CK(nullptr, ep->run_rc_min.reserve(mp * 8));
    CK(nullptr, ep->run_rc_cnt.reserve(mp * 4));
    CK(nullptr, ep->run_ctr.reserve(sizeof(RunCounters)));
    CK(nullptr, cudaMemsetAsync(ep->run_count.p, 0, mp * 4, ep->stream));
    CK(nullptr, cudaMemsetAsync(ep->run_min_bits.p, 0xff, mp * 8, ep->stream));
    CK(nullptr, cudaMemsetAsync(ep->run_min_cnt.p, 0, mp * 4, ep->stream));
    CK(nullptr, cudaMemsetAsync(ep->run_min_view.p, 0, mp * 8, ep->stream));
    CK(nullptr, cudaMemsetAsync(ep->run_dirty.p, 0, mp * 4, ep->stream));
    CK(nullptr, cudaMemsetAsync(ep->run_rc_min.p, 0xff, mp * 8, ep->stream));
    CK(nullptr, cudaMemsetAsync(ep->run_rc_cnt.p, 0, mp * 4, ep->stream));
    RunCounters c0{};
    c0.gen = 1;  // owner words of slots that predate every call are 0 (gen 0)
    CK(nullptr, cudaMemcpyAsync(ep->run_ctr.p, &c0, sizeof(c0), cudaMemcpyHostToDevice, ep->stream));
    CK(nullptr, ep->h_run.reserve(sizeof(RunCounters)));
    memset(ep->h_run.p, 0, sizeof(RunCounters));
    CK(nullptr, make(ep->ev_run_copy));
    CK(nullptr, run_alloc_table(kRunInitialSlots, &ep->run_tab[0], ep->stream));
    CK(nullptr, run_alloc_table(kRunInitialSlots, &ep->run_tab[4], ep->stream));
    ep->run_cap = kRunInitialSlots;
    CK(nullptr, ep->c_rslot.reserve(kRunInitialSlots * 4));
    CK(nullptr, ep->c_rwon.reserve(kRunInitialSlots));
    CK(nullptr, ep->run_desc.reserve(sizeof(RunDev)));
    run_init_desc(ep);
    CK(nullptr, cudaMemcpyAsync(ep->run_desc.p, &ep->run_host, sizeof(RunDev), cudaMemcpyHostToDevice, ep->stream));
    CK(nullptr, init_running_kernels());
  }
  CK(nullptr, ep->cls_lo.reserve((size_t)(ep->A_cap + 1) * ep->geo.row_words * 4));
  CK(nullptr, ep->cls_hi.reserve((size_t)(ep->A_cap + 1) * ep->geo.row_words * 4));
  ep->prof[0].cfg = ep->cfg;
  ep->n_prof = 1;
  if (int32_t rc = profile_init(ep, nullptr, 0)) return rc;
  // prefix index (device-resident: slot table + per-endpoint LRUs; the LRU regions are allocated by the first Add)
  CK(nullptr, make(ep->ev_caller));
  CK(nullptr, make(ep->ev_index_join));
  ep->index = std::make_unique<DeviceIndex>(ep->geo.Mpad, ep->geo.Mpad / 32, ep->cfg.prefix_capacity, ep->cfg.lru_capacity_default,
                                            ep->cfg.lru_capacity_max);
  CK(nullptr, ep->index->init(ep->stream));
  CK(nullptr, cudaEventRecord(ep->ev_table, ep->stream));
  CK(nullptr, cudaEventRecord(ep->ev_snapshot, ep->stream));
  CK(nullptr, cudaStreamSynchronize(ep->stream));
  *out = e.release();
  return EPPSCORE_OK;
}

void eppscore_destroy(eppscore_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  delete e;  // the engine's streams synchronise first, then everything else is freed (eppscore_engine's member order)
}

const char* eppscore_last_error(const eppscore_engine* e) { return e ? e->err.c_str() : g_create_error.c_str(); }

int32_t eppscore_get_stats(const eppscore_engine* ce, eppscore_stats* out) {
  eppscore_engine* e = const_cast<eppscore_engine*>(ce);
  if (!e || !out) return EPPSCORE_ERR_INVALID;
  memset(out, 0, sizeof(*out));
  out->struct_size = sizeof(*out);
  out->M = e->M;
  out->epoch = e->epoch;
  CK(e, cudaSetDevice(e->device));
  IndexStats st{};
  CK(e, e->index->stats(&st, e->stream));
  out->kernel_launches = e->launches + e->index->launches();
  out->prefix_hashes = st.used;
  out->prefix_live_hashes = st.live;
  out->prefix_capacity = st.capacity;
  out->prefix_table_bytes = st.table_bytes;
  out->lru_entries = st.lru_entries;
  out->lru_bytes = st.lru_bytes;
  out->prefix_overflow_rows = st.ovf_rows;
  out->prefix_rebuilds = st.rebuilds;
  out->index_error = st.error;
  unsigned long long resolved = 0;  // (the caller has waited for its batches)
  CK(e, cudaMemcpy(&resolved, e->probe_resolved.p, 8, cudaMemcpyDeviceToHost));
  out->probe_resolved = (uint32_t)resolved;
  return EPPSCORE_OK;
}

int32_t eppscore_set_debug(eppscore_engine* e, int32_t key, int64_t value) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (key == 1) {
    e->force_generic = value != 0;
    return EPPSCORE_OK;
  }
  if (key == 2) {
    e->hash_stage_mask = (int32_t)(value & 63);
    return EPPSCORE_OK;
  }
  if (key == 3) {
    e->host_chunk = (int32_t)value;
    return EPPSCORE_OK;
  }
  if (key == 4) {
    e->use_pdl = value != 0;
    return EPPSCORE_OK;
  }
  if (key == 5) {
    e->dev_split = value < 1 ? 1 : (value > 64 ? 64 : (int32_t)value);
    return EPPSCORE_OK;
  }
  if (key == 6) {
    e->dev_streams = value < 1 ? 1 : (value > 4 ? 4 : (int32_t)value);
    return EPPSCORE_OK;
  }
  return fail(e, EPPSCORE_ERR_INVALID, "unknown debug key");
}

int32_t eppscore_set_snapshot(eppscore_engine* e, const eppscore_snapshot* s) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (!s || s->struct_size != sizeof(eppscore_snapshot)) return fail(e, EPPSCORE_ERR_INVALID, "snapshot NULL or struct_size mismatch");
  if (s->M < 0 || s->M > e->geo.Mpad) return fail(e, EPPSCORE_ERR_CAPACITY, "M exceeds config.max_endpoints");
  if (s->lora_words < 0 || s->lora_words * 64 > e->A_cap) return fail(e, EPPSCORE_ERR_CAPACITY, "lora_words*64 exceeds config.max_adapters");
  if (s->M > 0 && (!s->kv_usage || !s->queue)) return fail(e, EPPSCORE_ERR_INVALID, "kv_usage and queue are required");
  CK(e, cudaSetDevice(e->device));
  const bool on_device = s->location == 1;
  cudaStream_t st = (on_device && s->stream) ? (cudaStream_t)s->stream : e->stream;
  const size_t M = (size_t)s->M;
  const bool have_lora = s->lora_active && s->lora_waiting && s->lora_words > 0;
  const bool capturing = is_capturing(st);
  int32_t rc;
  // the term / class-plane / summary buffers are rewritten below: a device-location batch that another stream launched
  // against the previous snapshot must have finished with them (inside a capture the graph's own edges order this)
  if (!capturing && (rc = pending_wait(e, st)) != EPPSCORE_OK) return rc;
  // Host snapshots are copied into the engine's tile buffers; device snapshots (e.g. the buffer an NCCL
  // broadcast just filled) are used IN PLACE — they must stay valid until the next set_snapshot.
  if (!on_device) {
    auto cp = [&](DevBuf& dst, const void* src, size_t bytes) -> cudaError_t {
      if (!src || bytes == 0) return cudaSuccess;
      return cudaMemcpyAsync(dst.p, src, bytes, cudaMemcpyHostToDevice, st);
    };
    CK(e, cp(e->raw_kv, s->kv_usage, M * 8));
    CK(e, cp(e->raw_queue, s->queue, M * 8));
    CK(e, cp(e->raw_running, s->running, M * 8));
    if (have_lora) {
      CK(e, cp(e->raw_act, s->lora_active, M * s->lora_words * 8));
      CK(e, cp(e->raw_wait, s->lora_waiting, M * s->lora_words * 8));
    }
    CK(e, cp(e->raw_nmodels, s->lora_nmodels, M * 4));
    CK(e, cp(e->raw_max, s->lora_max, M * 4));
    for (int i = 0; i < 4; i++) CK(e, cp(e->raw_col[i], s->endpoint_col[i], M * 8));
    CK(e, cp(e->raw_tokens, s->inflight_tokens, M * 8));
    if (e->lat_ep.p) {
      CK(e, cp(e->raw_min_tpot, s->min_tpot_slo, M * 8));
      CK(e, cp(e->raw_dispatched, s->dispatched, M * 4));
      CK(e, cp(e->raw_prefill, s->prefill_role, M));
    }
  }
  e->cur_queue = on_device ? s->queue : e->raw_queue.as<int64_t>();
  e->cur_running = s->running ? (on_device ? s->running : e->raw_running.as<int64_t>()) : nullptr;
  e->M = s->M;
  e->lora_words = have_lora ? s->lora_words : 0;
  e->A = e->lora_words * 64;
  e->epoch = s->epoch;

  PrepareArgs pa{};
  pa.geo = e->geo;
  pa.geo.M = s->M;
  pa.kv = on_device ? s->kv_usage : e->raw_kv.as<double>();
  pa.queue = e->cur_queue;
  pa.running = e->cur_running;
  pa.act = have_lora ? (on_device ? s->lora_active : e->raw_act.as<uint64_t>()) : nullptr;
  pa.wait = have_lora ? (on_device ? s->lora_waiting : e->raw_wait.as<uint64_t>()) : nullptr;
  pa.nmodels = s->lora_nmodels ? (on_device ? s->lora_nmodels : e->raw_nmodels.as<int32_t>()) : nullptr;
  pa.maxm = s->lora_max ? (on_device ? s->lora_max : e->raw_max.as<int32_t>()) : nullptr;
  for (int i = 0; i < 4; i++)
    pa.col[i] = s->endpoint_col[i] ? (on_device ? s->endpoint_col[i] : e->raw_col[i].as<double>()) : nullptr;
  // InFlightLoad.Tokens: the snapshot's array when it carries one, else the in-flight counters (all 0 until the first
  // eppscore_inflight_add, which scores exactly like an absent attribute, token_load.go:91-98)
  pa.tokens = s->inflight_tokens ? (on_device ? s->inflight_tokens : e->raw_tokens.as<int64_t>()) : e->inflight_tok.as<int64_t>();
  const bool reads_running = e->lat_ep.p && (!s->min_tpot_slo || !s->dispatched);
  if ((!s->inflight_tokens || reads_running) && e->producer_pending && !capturing)  // producer state last changed on another stream
    CK(e, cudaStreamWaitEvent(st, e->ev_producer, 0));
  pa.token_threshold = e->cfg.token_load_threshold;
  e->lat_args = LatArgs{};
  if (e->lat_ep.p) {
    // latency fold-in: split the linear forms into endpoint-only arrays (prepared on the device) and
    // per-request / per-pair terms (LatArgs); the weight normalisations are single IEEE divides
    // (scorer/latency/plugin.go:325-333,373-379) done here on the host (-ffp-contract=off).
    const eppscore_latency_params& lp = e->lat_params;
    // getEndpointMinTPOTSLO / getEndpointRunningRequestCount: the snapshot's arrays when it carries them, field by field,
    // else the running-request queues (min 0 and count 0 until the first eppscore_running_add, which score exactly like
    // absent arrays)
    pa.min_tpot = s->min_tpot_slo ? (on_device ? s->min_tpot_slo : e->raw_min_tpot.as<double>()) : e->run_min_view.as<double>();
    pa.dispatched = s->dispatched ? (on_device ? s->dispatched : e->raw_dispatched.as<int32_t>()) : e->run_count.as<int32_t>();
    pa.prefill = s->prefill_role ? (on_device ? s->prefill_role : e->raw_prefill.as<uint8_t>()) : nullptr;
    const double coef[8] = {lp.ttft_intercept, lp.ttft_kv, lp.ttft_waiting, lp.ttft_running,
                            lp.tpot_intercept, lp.tpot_kv, lp.tpot_waiting, lp.tpot_running};
    for (int i = 0; i < 8; i++) pa.lat_coef[i] = coef[i];
    pa.lat_buffer = lp.slo_buffer_factor;
    pa.lat_streaming = lp.streaming_mode;
    volatile double wkv = lp.composite_kv, wq = lp.composite_queue, wpref = lp.composite_prefix;
    volatile double sumw = wkv + wq;
    sumw = sumw + wpref;
    if (sumw <= 0) {
      wkv = 1;
      wq = 0;
      wpref = 0;
      sumw = 1;
    }
    wkv = wkv / sumw;
    wq = wq / sumw;
    wpref = wpref / sumw;
    pa.lat_ckv = wkv;
    pa.lat_ep = e->lat_ep.as<double>();
    pa.lat_has_predictions = lp.has_predictions;
    LatArgs& L = e->lat_args;
    L.enabled = 1;
    L.has_predictions = lp.has_predictions;
    L.strategy_most = lp.strategy_most;
    L.ttft_input = lp.ttft_input;
    L.ttft_prefix = lp.ttft_prefix;
    L.tpot_input = lp.tpot_input;
    L.tpot_generated = lp.tpot_generated;  // * float64(NumTokensGenerated = 1) is exact
    L.buffer = lp.slo_buffer_factor;
    volatile double wsum = lp.ttft_weight + lp.tpot_weight;
    if (wsum <= 0) {
      L.alpha = 1.0;
      L.beta = 0.0;
    } else {
      volatile double al = lp.ttft_weight / wsum, be = lp.tpot_weight / wsum;
      L.alpha = al;
      L.beta = be;
    }
    L.wq = wq;
    L.wpref = wpref;
    L.ep = pa.lat_ep;
  }
  pa.lora_words = e->lora_words;
  pa.A = e->A;
  pa.cls_lo = e->cls_lo.as<uint32_t>();
  pa.cls_hi = e->cls_hi.as<uint32_t>();
  e->snapshot_has_tokens = s->inflight_tokens != nullptr;
  e->snapshot_has_min_tpot = s->min_tpot_slo != nullptr;
  e->snapshot_has_dispatched = s->dispatched != nullptr;
  e->base_pa = pa;
  // every profile: its endpoint subset as set since (eppscore_set_profile_endpoints), then its terms
  for (int p = 0; p < e->n_prof; p++) {
    Profile& P = e->prof[p];
    P.subset = P.next_subset;
    if (P.subset) {
      CK(e, cudaMemcpyAsync(P.member_nat.p, P.next_nat.p, P.next_nat.bytes, cudaMemcpyDeviceToDevice, st));
      CK(e, cudaMemcpyAsync(P.member_perm.p, P.next_perm.p, P.next_perm.bytes, cudaMemcpyDeviceToDevice, st));
    }
    profile_pa(e, p);
  }
  // (inside a capture the copies run at each replay, and eppscore_set_profile_endpoints leaves ordering against those to the caller)
  if (!capturing) CK(e, cudaEventRecord(e->ev_subset, st));
  if ((rc = prepare_snapshot(e, st, (1u << e->n_prof) - 1)) != EPPSCORE_OK) return rc;
  if (!capturing && !on_device) CK(e, cudaStreamSynchronize(st));  // host arrays may be reused by the caller
  e->have_snapshot = true;
  return EPPSCORE_OK;
}

}  // extern "C"

namespace {

// Rows per slice of an in-order batch: a fixed byte budget of match rows (uint16 per endpoint), so the scratch depends on
// max_endpoints only and a captured graph never sees it move.
constexpr size_t kInOrderSliceBytes = 32ull << 20;

// eppscore_schedule_batch_inorder on device buffers, asynchronous on `s`.  Per slice of rows: the batch kernels of
// schedule_device with their match_out route (the prefix match counts and totals, which depend on no load; their provisional
// picks are overwritten), the candidates' queue / running min / max when the profile has those scorers, then
// inorder_pick_kernel, which reads the in-flight counters, walks the slice's requests in order and writes the counters back,
// so the next slice continues from them.
int32_t schedule_inorder(eppscore_engine* e, const DevBatch& d, cudaStream_t s, Scratch& sc) {
  const Profile& P = e->prof[0];
  const eppscore_config& c = P.cfg;
  if (!sc.s_io_match.p) {
    if (is_capturing(s))
      return fail(e, EPPSCORE_ERR_CAPACITY,
                  "the first eppscore_schedule_batch_inorder on a stream allocates its slice scratch: make one call outside the "
                  "CUDA-graph capture first");
    int32_t rows = (int32_t)std::max<size_t>(1, kInOrderSliceBytes / ((size_t)e->geo.Mpad * 2));
    if (sc.rows > 0) rows = std::min(rows, sc.rows);
    CK(e, sc.s_io_match.reserve((size_t)rows * e->geo.Mpad * 2));
    CK(e, sc.s_io_total.reserve((size_t)rows * 2));
    CK(e, sc.s_io_minmax.reserve((size_t)rows * 32));
    sc.io_rows = rows;
  }
  InOrderArgs a{};
  a.M = e->M;
  a.Mpad = e->geo.Mpad;
  a.log_epl = e->geo.log_epl;
  a.RW = e->geo.row_words;
  a.A = e->A;
  a.mask_words = (e->M + 31) / 32;
  a.n_scorers = c.n_scorers;
  bool minmax = false;
  static const double cls_score[4] = {0.0, 0.6, 0.8, 1.0};  // lora_affinity.go:84-99
  for (int i = 0; i < c.n_scorers; i++) {
    const int k = c.scorer_kind[i];
    a.kind[i] = k;
    a.weight[i] = c.scorer_weight[i];
    const bool static_term = k == EPPSCORE_SCORER_KV_CACHE || (k >= EPPSCORE_SCORER_ENDPOINT_COL0 && k < EPPSCORE_SCORER_ENDPOINT_COL0 + 4);
    a.term[i] = static_term ? P.term[i].as<double>() : nullptr;
    for (int q = 0; q < 4; q++) a.lora_term[i][q] = clamp01_host(cls_score[q]) * c.scorer_weight[i];
    minmax = minmax || k == EPPSCORE_SCORER_QUEUE || k == EPPSCORE_SCORER_RUNNING;
  }
  a.pick_mode = c.pick_mode;
  a.tie_mode = c.tie_mode;
  a.seed_lo = (uint32_t)c.tie_seed;
  a.seed_hi = (uint32_t)(c.tie_seed >> 32);
  a.token_threshold = e->base_pa.token_threshold;
  a.member = P.subset ? P.member_nat.as<uint32_t>() : nullptr;
  a.queue = e->cur_queue;
  a.running = e->cur_running;
  a.cls_lo = e->cls_lo.as<uint32_t>();
  a.cls_hi = e->cls_hi.as<uint32_t>();
  a.inflight_req = e->inflight_req.as<int64_t>();
  a.inflight_tok = e->inflight_tok.as<int64_t>();
  for (int32_t base = 0; base < d.R; base += sc.io_rows) {
    DevBatch q = slice_rows(d, base, std::min(sc.io_rows, d.R - base), (size_t)e->M);
    q.match_blocks = sc.s_io_match.as<uint16_t>();
    if (!q.total_blocks) q.total_blocks = sc.s_io_total.as<uint16_t>();
    int32_t rc = schedule_device(e, q, s, sc);
    if (rc != EPPSCORE_OK) return rc;
    a.R = q.R;
    a.request_base = q.request_base;
    a.match = q.match_blocks;
    a.total = q.total_blocks;
    a.adapter_id = q.adapter_id;
    a.cand_mask = q.run[0].cand_mask;
    a.tokens = q.tokens;
    a.pick = q.run[0].pick;
    a.pick_score = q.run[0].pick_score;
    a.tie_count = q.run[0].tie_count;
    a.minmax = minmax ? sc.s_io_minmax.as<long long>() : nullptr;
    if (minmax) e->launches += launch_inorder_minmax(a, s, e->sm_count);
    const int launched = launch_inorder_pick(a, e->io_cluster, s);
    if (launched < 0) {
      cudaGetLastError();
      return cuda_fail(e, (cudaError_t)-launched, "inorder_pick_kernel launch");
    }
    e->launches += launched;
    CK(e, cudaGetLastError());
  }
  return EPPSCORE_OK;
}

// eppscore_schedule_batch(_topk, _topk_wide, _profiles, _profiles_topk, _inorder): the runs (profile + per-profile filter
// result and outputs) of one batch, as make_batch takes them.  `inorder`: the batch's single run is scheduled in arrival order
// against the in-flight counters (schedule_inorder), with `tokens` its requests' estimates.
int32_t schedule_batch(eppscore_engine* e, const eppscore_batch* b, int32_t n_runs, const eppscore_profile_run* runs,
                       const eppscore_topk* topk, bool wide = false, bool inorder = false, const int64_t* tokens = nullptr) {
  if (b->R < 0) return fail(e, EPPSCORE_ERR_INVALID, "R < 0");
  if (b->R == 0) return EPPSCORE_OK;
  CK(e, cudaSetDevice(e->device));
  int32_t rc = EPPSCORE_OK;
  DevBatch d = make_batch(e, *b, n_runs, runs, topk, wide);
  d.tokens = tokens;
  const size_t M = (size_t)e->M;
  bool any_wide = false;
  for (int i = 0; i < n_runs; i++) any_wide = any_wide || d.run[i].wide;
  // What one piece of the batch runs on `st` with scratch set `sc`.  The in-order step reads and writes the in-flight counters,
  // so it is ordered as a producer mutation.
  auto step = [&](const DevBatch& x, cudaStream_t st, Scratch& sc) -> int32_t {
    if (!inorder) return any_wide ? schedule_wide(e, x, st, sc) : schedule_device(e, x, st, sc);
    bool capturing = false;
    int32_t rc = producer_begin(e, st, &capturing);
    if (rc == EPPSCORE_OK) rc = schedule_inorder(e, x, st, sc);
    if (rc == EPPSCORE_OK) rc = producer_end(e, st, capturing, counters_feed_scorer(e));
    return rc;
  };
  if (b->location == 1) {
    bool per_pair = false;  // R x M outputs or masks on some run
    for (int i = 0; i < n_runs; i++) {
      const DevRun& x = d.run[i];
      per_pair = per_pair || x.cand_mask || x.scores_out || x.pred_out || x.filter_mask_out;
    }
    cudaStream_t cs = b->stream ? (cudaStream_t)b->stream : e->stream;
    StreamScratch* own = reserved_scratch(e, cs);
    if (own) {  // refused before anything is launched: the stream's set is never grown
      if (b->R > own->max_R) return fail(e, EPPSCORE_ERR_CAPACITY, "R exceeds the max_R the batch's stream was reserved for");
      if (d.prompt_bytes && !d.hashes_in && d.max_blocks > own->max_blocks)
        return fail(e, EPPSCORE_ERR_CAPACITY, "max_blocks exceeds the max_blocks the batch's stream was reserved for");
    }
    Scratch& sc = own ? own->sc : e->sc[0];
    // R x M outputs, masks, supplied hashes and dense rows go as one slice (their layouts are not sliced here), and so does a
    // batch on a reserved stream (the slices share the engine's fork / join events and internal streams), a wide batch
    // (schedule_wide slices it in order on `cs`) and an in-order one (its requests run in order against one set of counters)
    const bool sliceable = d.prompt_bytes && !d.hashes_in && !per_pair && !d.dense_feat && !d.match_blocks && !d.input_tokens &&
                           !d.ttft_slo && !d.tpot_slo && !own && !any_wide && !inorder;
    int K = e->dev_split;
    if (!sliceable || e->dev_streams < 2) K = 1;
    while (K > 1 && b->R / K < 2048) K--;
    if (K <= 1) {
      if ((rc = step(d, cs, sc)) != EPPSCORE_OK) return rc;
      return pending_record(e, cs);
    }
    // fork: the internal streams join the caller's stream (also inside a CUDA-graph capture), slice c goes to stream c mod S
    const int S = e->dev_streams < K ? e->dev_streams : K;
    if (!e->ev_fork) CK(e, make(e->ev_fork));
    for (int i = 0; i < S - 1; i++) {
      if (!e->split_stream[i]) CK(e, make(e->split_stream[i]));
      if (!e->ev_join[i]) CK(e, make(e->ev_join[i]));
    }
    CK(e, cudaEventRecord(e->ev_fork, cs));
    for (int i = 0; i < S - 1; i++) CK(e, cudaStreamWaitEvent(e->split_stream[i], e->ev_fork, 0));
    const int32_t per = ((b->R + K - 1) / K + 63) / 64 * 64;
    for (int c = 0, base = 0; base < b->R; c++, base += per) {
      const int si = c % S;
      rc = schedule_device(e, slice_rows(d, base, std::min(per, b->R - base), M), si == 0 ? cs : e->split_stream[si - 1], e->sc[si]);
      if (rc != EPPSCORE_OK) break;
    }
    for (int i = 0; i < S - 1; i++) {  // join, also on the error path (a capture must not be left forked)
      cudaEventRecord(e->ev_join[i], e->split_stream[i]);
      cudaStreamWaitEvent(cs, e->ev_join[i], 0);
    }
    if (rc != EPPSCORE_OK) return rc;
    return pending_record(e, cs);
  }
  // ---- host buffers: H2D, kernels, D2H, all inside this call ----
  // The batch is cut into chunks that alternate between two streams (each with its own scratch set): the H2D copy of
  // chunk i+1 runs under the kernels and the D2H copy of chunk i, so the call costs about max(copy, compute) instead of
  // their sum.  Requests are independent given (snapshot, table), so any cut gives identical results (request_base keeps
  // the tie priorities of the whole batch).
  if (!e->have_snapshot) return fail(e, EPPSCORE_ERR_NO_SNAPSHOT, "schedule_batch before set_snapshot");
  if (b->prompt_bytes && !b->prompt_off) return fail(e, EPPSCORE_ERR_INVALID, "prompt_off required with prompt_bytes");
  if (b->hashes_out && (b->hashes_in || !b->prompt_bytes))
    return fail(e, EPPSCORE_ERR_INVALID, "hashes_out needs prompt_bytes (hashes supplied as hashes_in are already the caller's)");
  bool diag = d.match_blocks || d.dense_feat;  // R x M arrays: one chunk at a time is plenty
  for (int i = 0; i < n_runs; i++) diag = diag || d.run[i].scores_out || d.run[i].pred_out;
  int32_t chunk = e->host_chunk > 0 ? e->host_chunk : b->R;
  if (diag || inorder || b->R < 2 * chunk) chunk = b->R;  // (an in-order batch: its requests run in order on one stream)
  const int nstreams = chunk < b->R ? 2 : 1;
  if (nstreams == 2 && !e->stream2) CK(e, make(e->stream2));
  // the chunks reuse sc[0] / sc[1], which a device-location batch may still hold
  if ((rc = pending_wait(e, e->stream)) != EPPSCORE_OK) return rc;
  if (nstreams == 2 && (rc = pending_wait(e, e->stream2)) != EPPSCORE_OK) return rc;
  auto at = [](auto* p, void* base, size_t off) { return reinterpret_cast<decltype(p)>(static_cast<unsigned char*>(base) + off); };
  // The small results come back through pinned staging, since a D2H copy into the caller's (usually pageable) arrays would
  // block the host after every chunk: `pinned` is the batch with those outputs in h_res, the 8-byte arrays first so that each
  // one is aligned, and `results` lists the copies from there to the caller.
  DevBatch pinned = d;
  std::vector<Copy> results, d2h;
  size_t h_end[9] = {};  // by element size: the end of the 8-byte arrays, then of the 4- and 2-byte ones
  auto via_pinned = [](auto* p, Rows kind) { return p && (kind == Rows::small || kind == Rows::result); };
  for_each_row_array(pinned, M, [&](auto*& p, size_t per, Rows kind, auto) {
    if (via_pinned(p, kind)) h_end[sizeof *p] += (size_t)b->R * per * sizeof *p;
  });
  h_end[4] += h_end[8];
  h_end[2] += h_end[4];
  CK(e, e->h_res.reserve(h_end[2]));
  for_each_row_array(pinned, M, [&](auto*& p, size_t per, Rows kind, auto) {
    if (!via_pinned(p, kind)) return;
    const size_t bytes = (size_t)b->R * per * sizeof *p;
    h_end[sizeof *p] -= bytes;  // (each array takes the bytes just below the end of its size's part)
    auto* h = at(p, e->h_res.p, h_end[sizeof *p]);
    results.push_back({(void*)p, h, bytes});
    p = h;
  });
  std::vector<std::pair<DevBuf*, size_t>> parts;  // a chunk's scratch buffers and their bytes
  auto part = [&parts](DevBuf& buf) -> size_t& {
    for (auto& x : parts)
      if (x.first == &buf) return x.second;
    return parts.emplace_back(&buf, 0).second;
  };
  int ci = 0;
  for (int32_t r0 = 0; r0 < b->R; r0 += chunk, ci++) {
    const int32_t n = std::min(b->R, r0 + chunk) - r0;
    Scratch& sc = e->sc[ci & 1];
    cudaStream_t st = (ci & 1) ? e->stream2 : e->stream;
    // the chunk on the host (`q`: the caller's inputs, its outputs where they come back to), then on the device (`x`): the
    // prompt bytes its offsets reach, and every other array in a part of its scratch buffer
    const DevBatch q = slice_rows(pinned, r0, n, M);
    DevBatch x = q;
    if (q.prompt_bytes &&
        (rc = stage_prompts(e, sc.s_prompts, q.prompt_bytes, q.prompt_off, q.prompt_len, 0, n, st, &x.prompt_bytes)) != EPPSCORE_OK)
      return rc;
    auto bytes = [n](auto* p, size_t per, Rows kind) -> size_t {
      return (p || kind == Rows::result) ? (n + (kind == Rows::offsets ? 1 : 0)) * per * sizeof *p : 0;
    };
    parts.clear();
    for_each_row_array(x, M, [&](auto*& p, size_t per, Rows kind, DevBuf Scratch::*slot) {
      if (const size_t nb = bytes(p, per, kind)) part(sc.*slot) += nb;
    });
    for (auto& [buf, size] : parts) {
      CK(e, buf->reserve(size));
      size = 0;
    }
    d2h.clear();
    cudaError_t c = cudaSuccess;
    for_each_row_array(x, M, [&](auto*& p, size_t per, Rows kind, DevBuf Scratch::*slot) {
      const size_t nb = bytes(p, per, kind);
      if (nb == 0) {
        p = nullptr;
        return;
      }
      size_t& off = part(sc.*slot);
      auto* dev = at(p, (sc.*slot).p, off);
      off += nb;
      if (kind == Rows::in || kind == Rows::offsets) {
        if (c == cudaSuccess) c = cudaMemcpyAsync((void*)dev, p, nb, cudaMemcpyHostToDevice, st);
      } else if (p) {
        d2h.push_back({(void*)p, dev, nb});
      }
      p = dev;
    });
    CK(e, c);
    // hashes_out from the device: entries past n_hashes[r] are zero
    if (x.hashes_out) CK(e, cudaMemsetAsync(x.hashes_out, 0, (size_t)n * x.max_blocks * 8, st));
    if ((rc = step(x, st, sc)) != EPPSCORE_OK) return rc;
    for (const Copy& y : d2h) CK(e, cudaMemcpyAsync(y.dst, y.src, y.bytes, cudaMemcpyDeviceToHost, st));
  }
  CK(e, cudaStreamSynchronize(e->stream));
  if (nstreams == 2) CK(e, cudaStreamSynchronize(e->stream2));
  for (const Copy& y : results) memcpy(y.dst, y.src, y.bytes);
  return EPPSCORE_OK;
}

// One eppscore_topk with k in [k_min, k_max] (`range` says which in the message).
int32_t check_topk(eppscore_engine* e, const eppscore_topk& t, int32_t k_min, int32_t k_max, const char* range) {
  if (t.struct_size != sizeof(eppscore_topk)) return fail(e, EPPSCORE_ERR_INVALID, "topk struct_size mismatch");
  if (t.k < k_min || t.k > k_max) return fail(e, EPPSCORE_ERR_INVALID, std::string("topk k must be in ") + range);
  if (t.k > 0 && (!t.endpoints || !t.scores)) return fail(e, EPPSCORE_ERR_INVALID, "topk endpoints/scores required");
  return EPPSCORE_OK;
}

// eppscore_schedule_batch and its top-k forms: one run of profile 0 from the batch's own filter result and outputs
int32_t schedule_batch(eppscore_engine* e, const eppscore_batch* b, const eppscore_topk* t, bool wide = false) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (!b || b->struct_size != sizeof(eppscore_batch)) return fail(e, EPPSCORE_ERR_INVALID, "batch NULL or struct_size mismatch");
  if (t) {
    const int32_t rc = wide ? check_topk(e, *t, 1, e->cfg.max_endpoints, "[1, max_endpoints]")
                            : check_topk(e, *t, 1, EPPSCORE_MAX_TOPK, "[1, EPPSCORE_MAX_TOPK]");
    if (rc != EPPSCORE_OK) return rc;
  }
  return schedule_batch(e, b, 1, nullptr, t, wide);
}

}  // namespace

extern "C" {

int32_t eppscore_schedule_batch(eppscore_engine* e, const eppscore_batch* b) { return schedule_batch(e, b, nullptr); }

int32_t eppscore_schedule_batch_topk(eppscore_engine* e, const eppscore_batch* b, const eppscore_topk* t) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (!t) return fail(e, EPPSCORE_ERR_INVALID, "topk NULL");
  return schedule_batch(e, b, t);
}

int32_t eppscore_schedule_batch_topk_wide(eppscore_engine* e, const eppscore_batch* b, const eppscore_topk* t) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (!t) return fail(e, EPPSCORE_ERR_INVALID, "topk NULL");
  return schedule_batch(e, b, t, true);
}

int32_t eppscore_schedule_batch_inorder(eppscore_engine* e, const eppscore_batch* b, const int64_t* tokens) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (!b || b->struct_size != sizeof(eppscore_batch)) return fail(e, EPPSCORE_ERR_INVALID, "batch NULL or struct_size mismatch");
  if (b->R < 0) return fail(e, EPPSCORE_ERR_INVALID, "R < 0");
  if (cfg_has(e->prof[0].cfg, EPPSCORE_SCORER_LATENCY))
    return fail(e, EPPSCORE_ERR_INVALID, "schedule_batch_inorder: the latency scorer's inputs are PreRequest state the call does not order");
  if (e->have_snapshot && e->snapshot_has_tokens)
    return fail(e, EPPSCORE_ERR_INVALID, "schedule_batch_inorder: the snapshot supplies inflight_tokens; the in-order view needs the engine's counters");
  if (b->dense_feat || b->scores_out || b->match_blocks || b->pred_out || b->filter_mask_out)
    return fail(e, EPPSCORE_ERR_INVALID, "schedule_batch_inorder: dense_feat, scores_out, match_blocks, pred_out and filter_mask_out are not available");
  if (!b->pick || !b->pick_score || !b->tie_count) return fail(e, EPPSCORE_ERR_INVALID, "pick/pick_score/tie_count required");
  if (b->location != 0 && b->location != 1) return fail(e, EPPSCORE_ERR_INVALID, "location must be 0 or 1");
  if (b->R == 0) return EPPSCORE_OK;
  if (!e->have_snapshot) return fail(e, EPPSCORE_ERR_NO_SNAPSHOT, "schedule_batch_inorder before set_snapshot");
  if (b->prompt_bytes && !b->prompt_off) return fail(e, EPPSCORE_ERR_INVALID, "prompt_off required with prompt_bytes");
  CK(e, cudaSetDevice(e->device));
  if (e->io_cluster == 0) {  // the cluster shape, decided once per engine and before the first call launches anything
    const int C = inorder_cluster_size(e->geo.Mpad);
    if (C < 0) return cuda_fail(e, (cudaError_t)-C, "inorder_pick_kernel cluster attributes");
    if (C == 0)
      return fail(e, EPPSCORE_ERR_CAPACITY, "schedule_batch_inorder: no thread-block cluster of this device holds max_endpoints "
                                            "endpoints (8192 needs the non-portable cluster size 16)");
    e->io_cluster = C;
  }
  return schedule_batch(e, b, 1, nullptr, nullptr, false, true, tokens);
}

int32_t eppscore_add_profile(eppscore_engine* e, const eppscore_profile* p, int32_t* id_out) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (!p || p->struct_size != sizeof(eppscore_profile) || !id_out) return fail(e, EPPSCORE_ERR_INVALID, "profile NULL, struct_size mismatch or id_out NULL");
  if (e->n_prof >= EPPSCORE_MAX_PROFILES) return fail(e, EPPSCORE_ERR_CAPACITY, "at most EPPSCORE_MAX_PROFILES profiles");
  CK(e, cudaSetDevice(e->device));
  if (is_capturing(e->stream)) return fail(e, EPPSCORE_ERR_INVALID, "add_profile under CUDA-graph capture");
  eppscore_config c = e->cfg;  // engine-wide fields stay the engine's
  c.n_scorers = p->n_scorers;
  memcpy(c.scorer_kind, p->scorer_kind, sizeof(c.scorer_kind));
  memcpy(c.scorer_weight, p->scorer_weight, sizeof(c.scorer_weight));
  c.pick_mode = p->pick_mode;
  c.n_filters = p->n_filters;
  memcpy(c.filter_kind, p->filter_kind, sizeof(c.filter_kind));
  memcpy(c.filter_param, p->filter_param, sizeof(c.filter_param));
  if (const char* why = profile_error(c)) return fail(e, EPPSCORE_ERR_INVALID, why);
  const int32_t id = e->n_prof;
  c.tie_seed = e->cfg.tie_seed ^ ((uint64_t)id * 0x9E3779B97F4A7C15ull);  // (include/eppscore.h: eppscore_profile)
  Profile& P = e->prof[id];
  P.cfg = c;
  int32_t rc = profile_init(e, e, id);
  if (rc != EPPSCORE_OK) {
    P = Profile{};
    return rc;
  }
  e->n_prof = id + 1;
  if (e->have_snapshot) {  // prepared for the current snapshot at once, behind everything that reads or rewrites the terms
    if ((rc = pending_wait(e, e->stream)) != EPPSCORE_OK) return rc;
    if (e->producer_pending) CK(e, cudaStreamWaitEvent(e->stream, e->ev_producer, 0));
    profile_pa(e, id);
    if ((rc = prepare_snapshot(e, e->stream, 1u << id)) != EPPSCORE_OK) return rc;
  }
  CK(e, cudaStreamSynchronize(e->stream));
  *id_out = id;
  return EPPSCORE_OK;
}

int32_t eppscore_set_profile_endpoints(eppscore_engine* e, int32_t profile, const uint32_t* mask, int32_t words) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (profile < 0 || profile >= e->n_prof) return fail(e, EPPSCORE_ERR_INVALID, "set_profile_endpoints: unknown profile");
  if (mask && words < 0) return fail(e, EPPSCORE_ERR_INVALID, "set_profile_endpoints: words < 0");
  CK(e, cudaSetDevice(e->device));
  if (is_capturing(e->stream)) return fail(e, EPPSCORE_ERR_INVALID, "set_profile_endpoints under CUDA-graph capture");
  Profile& P = e->prof[profile];
  // the next rows are copied by set_snapshot on its stream: the last one outside a capture (on whatever stream) has finished
  // copying them.  Not ev_snapshot: that may have been recorded inside a capture, and such an event cannot be waited for.
  CK(e, cudaEventSynchronize(e->ev_subset));
  // NULL writes rows with every endpoint: a set_snapshot captured while the profile had a subset copies the next rows at each
  // replay, and then sees every endpoint
  const int32_t nw = e->geo.Mpad / 32;
  std::vector<uint32_t> nat((size_t)nw, mask ? 0u : ~0u), perm((size_t)e->geo.row_words, 0u);
  for (int32_t w = 0; mask && w < nw && w < words; w++) nat[(size_t)w] = mask[w];
  const uint32_t max_ep = (uint32_t)e->cfg.max_endpoints;
  for (uint32_t m = 0; m < (uint32_t)e->geo.Mpad; m++) {
    const bool in = m < max_ep && ((nat[m >> 5] >> (m & 31)) & 1u);
    if (!in) {
      nat[m >> 5] &= ~(1u << (m & 31));
      continue;
    }
    const uint32_t pos = perm_bitpos(m, e->geo.log_epl);
    perm[pos >> 5] |= 1u << (pos & 31);
  }
  // the next rows are only read by the next set_snapshot (stream-ordered after this copy)
  CK(e, cudaMemcpyAsync(P.next_nat.p, nat.data(), nat.size() * 4, cudaMemcpyHostToDevice, e->stream));
  CK(e, cudaMemcpyAsync(P.next_perm.p, perm.data(), perm.size() * 4, cudaMemcpyHostToDevice, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  P.next_subset = mask != nullptr;
  return EPPSCORE_OK;
}

}  // extern "C"

namespace {

// the arguments eppscore_schedule_batch_profiles refuses
int32_t check_profile_runs(eppscore_engine* e, const eppscore_batch* b, int32_t n_runs, const eppscore_profile_run* runs) {
  if (!b || b->struct_size != sizeof(eppscore_batch)) return fail(e, EPPSCORE_ERR_INVALID, "batch NULL or struct_size mismatch");
  if (b->pick || b->pick_score || b->tie_count || b->cand_mask || b->scores_out || b->pred_out || b->filter_mask_out)
    return fail(e, EPPSCORE_ERR_INVALID, "schedule_batch_profiles: per-profile batch fields belong to the runs (must be NULL)");
  if (n_runs < 1 || n_runs > EPPSCORE_MAX_PROFILES || !runs) return fail(e, EPPSCORE_ERR_INVALID, "n_runs outside [1, EPPSCORE_MAX_PROFILES]");
  unsigned seen = 0;
  for (int32_t i = 0; i < n_runs; i++) {
    const eppscore_profile_run& x = runs[i];
    if (x.struct_size != sizeof(eppscore_profile_run)) return fail(e, EPPSCORE_ERR_INVALID, "profile_run struct_size mismatch");
    if (x.profile < 0 || x.profile >= e->n_prof) return fail(e, EPPSCORE_ERR_INVALID, "profile_run: unknown profile");
    if (seen & (1u << x.profile)) return fail(e, EPPSCORE_ERR_INVALID, "profile_run: a profile appears in two runs");
    seen |= 1u << x.profile;
    if (!x.pick || !x.pick_score || !x.tie_count) return fail(e, EPPSCORE_ERR_INVALID, "profile_run: pick/pick_score/tie_count required");
  }
  return EPPSCORE_OK;
}

}  // namespace

extern "C" {

int32_t eppscore_schedule_batch_profiles(eppscore_engine* e, const eppscore_batch* b, int32_t n_runs, const eppscore_profile_run* runs) {
  if (!e) return EPPSCORE_ERR_INVALID;
  const int32_t rc = check_profile_runs(e, b, n_runs, runs);
  if (rc != EPPSCORE_OK) return rc;
  return schedule_batch(e, b, n_runs, runs, nullptr);
}

int32_t eppscore_schedule_batch_profiles_topk(eppscore_engine* e, const eppscore_batch* b, int32_t n_runs,
                                              const eppscore_profile_run* runs, const eppscore_topk* topk) {
  if (!e) return EPPSCORE_ERR_INVALID;
  int32_t rc = check_profile_runs(e, b, n_runs, runs);
  if (rc != EPPSCORE_OK) return rc;
  if (!topk) return fail(e, EPPSCORE_ERR_INVALID, "topk NULL");
  for (int32_t i = 0; i < n_runs; i++)
    if ((rc = check_topk(e, topk[i], 0, e->cfg.max_endpoints, "[0, max_endpoints]")) != EPPSCORE_OK) return rc;
  return schedule_batch(e, b, n_runs, runs, topk);
}

int32_t eppscore_hash_prompts(eppscore_engine* e, int32_t R, int32_t location, const uint8_t* prompt_bytes,
                              const int64_t* prompt_off, const int32_t* prompt_len, const uint64_t* model_seed,
                              int32_t block_chars, int32_t max_blocks, uint64_t* hashes_out, uint16_t* n_hashes_out,
                              void* stream) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (R <= 0) return EPPSCORE_OK;
  if (!prompt_bytes || !prompt_off || !hashes_out || !n_hashes_out) return fail(e, EPPSCORE_ERR_INVALID, "NULL argument");
  const int32_t bc = block_chars > 0 ? block_chars : e->cfg.block_chars;
  const int32_t mb = max_blocks > 0 ? max_blocks : e->cfg.max_blocks;
  if (mb > EPPSCORE_MAX_BLOCKS) return fail(e, EPPSCORE_ERR_CAPACITY, "max_blocks > 65535");
  CK(e, cudaSetDevice(e->device));
  if (location == 1) {
    HashArgs h{};
    h.R = R;
    h.block_chars = bc;
    h.max_blocks = mb;
    h.stride = mb;
    h.stage_mask = e->hash_stage_mask;
    h.bytes = prompt_bytes;
    h.off = prompt_off;
    h.len = prompt_len;
    h.seed = model_seed;
    h.hashes = hashes_out;
    h.n_hashes = n_hashes_out;
    e->launches += launch_hash_prompts(h, stream ? (cudaStream_t)stream : e->stream, e->sm_count);
    CK(e, cudaGetLastError());
    return EPPSCORE_OK;
  }
  // host arrays: staged, hashed by the device form on the engine stream, copied back
  HostStage st(e);
  const uint8_t* d_bytes = st.prompts(prompt_bytes, prompt_off, prompt_len, R);
  const int64_t* d_off = st.in(prompt_off, (size_t)R + 1);
  const int32_t* d_len = st.in(prompt_len, R);
  const uint64_t* d_seed = st.in(model_seed, R);
  uint64_t* d_hashes = st.out(hashes_out, (size_t)R * mb, true);  // entries past n_hashes[r] are zero
  uint16_t* d_nh = st.out(n_hashes_out, R);
  return st.finish([&] { return eppscore_hash_prompts(e, R, 1, d_bytes, d_off, d_len, d_seed, bc, mb, d_hashes, d_nh, e->stream); });
}

uint64_t eppscore_xxh64(const void* data, size_t len, uint64_t seed) { return xxh64_host(data, len, seed); }

uint64_t eppscore_model_seed(const void* model, size_t model_len, const void* salt, size_t salt_len) {
  std::string buf;
  buf.reserve(model_len + salt_len);
  if (model_len) buf.append(static_cast<const char*>(model), model_len);
  if (salt_len) buf.append(static_cast<const char*>(salt), salt_len);
  return xxh64_host(buf.data(), buf.size(), 0);
}

// ---------------- prefix index ----------------
int32_t eppscore_count_fields(eppscore_engine* e, int32_t R, int32_t location, const uint8_t* prompt_bytes,
                              const int64_t* prompt_off, const int32_t* prompt_len, int32_t* out, void* stream) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (R < 0 || (R > 0 && (!prompt_bytes || !prompt_off || !out))) return fail(e, EPPSCORE_ERR_INVALID, "count_fields: NULL argument");
  if (R == 0) return EPPSCORE_OK;
  CK(e, cudaSetDevice(e->device));
  if (location == 1) {
    cudaStream_t s = stream ? (cudaStream_t)stream : e->stream;
    e->launches += launch_count_fields(prompt_bytes, prompt_off, prompt_len, R, out, s, e->sm_count);
    CK(e, cudaGetLastError());
    return EPPSCORE_OK;
  }
  // host arrays: staged, counted by the device form on the engine stream, copied back
  HostStage st(e);
  const uint8_t* d_bytes = st.prompts(prompt_bytes, prompt_off, prompt_len, R);
  const int64_t* d_off = st.in(prompt_off, (size_t)R + 1);
  const int32_t* d_len = st.in(prompt_len, R);
  int32_t* d_out = st.out(out, R);
  return st.finish([&] { return eppscore_count_fields(e, R, 1, d_bytes, d_off, d_len, d_out, e->stream); });
}

// lru_capacity (host, [M] or NULL) -> a padded host vector the index can copy; validates the values
static int32_t pad_caps(eppscore_engine* e, const int32_t* lru_capacity, std::vector<int32_t>* out) {
  out->clear();
  if (!lru_capacity) return EPPSCORE_OK;
  out->assign((size_t)e->geo.Mpad, 0);
  const int32_t n = e->M > 0 ? e->M : e->geo.Mpad;
  for (int32_t i = 0; i < n; i++) (*out)[i] = lru_capacity[i] > 0 ? lru_capacity[i] : 0;
  return EPPSCORE_OK;
}
// A reserved index reports a mutation it skipped for lack of room to the next index call outside a capture, which is refused.
static int32_t index_skips(eppscore_engine* e, bool exact, const char* what) {
  if (!e->index->reserved()) return EPPSCORE_OK;
  bool skipped = false;
  CK(e, e->index->new_skips(exact, e->stream, &skipped));
  if (!skipped) return EPPSCORE_OK;
  return fail(e, EPPSCORE_ERR_CAPACITY, std::string(what) + ": an earlier index mutation found no room within eppscore_prefix_reserve's "
                                        "sizes and was skipped whole (stats.index_error bit 4); this call was not run");
}
static int32_t index_status(eppscore_engine* e, cudaError_t c, const char* what) {
  if (c == cudaSuccess) return EPPSCORE_OK;
  if (c == cudaErrorInvalidValue)
    return fail(e, EPPSCORE_ERR_CAPACITY, std::string(what) + ": an LRU capacity above the engine's lru_capacity_max (the per-endpoint regions were sized at the first Add)");
  return cuda_fail(e, c, what);
}

// PreRequest for R requests with n_picks picks each (eppscore_commit_picks[_device|_profiles]): host arrays are staged and the
// call returns when the commit is done; device arrays are committed asynchronously, ordered on `stream`.
static int32_t commit_calls(eppscore_engine* e, int32_t R, int32_t n_picks, const int32_t* const* picks, const uint64_t* hashes,
                            const uint16_t* n_hashes, int32_t hash_stride, const int32_t* lru_capacity, bool on_device,
                            int64_t touch_bound, void* stream, const char* what) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (n_picks < 1 || n_picks > EPPSCORE_MAX_PROFILES || (R > 0 && !picks)) return fail(e, EPPSCORE_ERR_INVALID, "n_picks outside [1, EPPSCORE_MAX_PROFILES]");
  bool null_pick = false;
  for (int32_t p = 0; R > 0 && p < n_picks; p++) null_pick = null_pick || !picks[p];
  if (R < 0 || (R > 0 && (null_pick || !hashes || !n_hashes))) return fail(e, EPPSCORE_ERR_INVALID, "NULL argument");
  if (R == 0) return EPPSCORE_OK;
  if (hash_stride <= 0) return fail(e, EPPSCORE_ERR_INVALID, "hash_stride must be > 0");
  CK(e, cudaSetDevice(e->device));
  std::vector<int32_t> caps;
  int32_t rc = pad_caps(e, lru_capacity, &caps);
  if (rc != EPPSCORE_OK) return rc;
  const int32_t* d_picks[EPPSCORE_MAX_PROFILES] = {};
  if (on_device) {
    cudaStream_t cs = stream ? (cudaStream_t)stream : e->stream;
    // Under CUDA-graph capture only a reserved index can commit: room is then decided on the device at each replay.  Refused
    // before anything is enqueued, so the capture stays valid.
    const bool capturing = is_capturing(cs);
    if (capturing && !e->index->reserved())
      return fail(e, EPPSCORE_ERR_CAPACITY, std::string(what) + " under CUDA-graph capture: reserve the prefix index before capturing "
                                            "commits (eppscore_prefix_reserve)");
    if (capturing && lru_capacity)
      return fail(e, EPPSCORE_ERR_INVALID, std::string(what) + " under CUDA-graph capture: lru_capacity must be NULL (create the "
                                           "endpoints' LRUs outside the capture, e.g. eppscore_prefix_add with n = 0)");
    if (!capturing && (rc = index_skips(e, false, what)) != EPPSCORE_OK) return rc;
    if (cs != e->stream) {  // the arrays are produced on the caller's stream
      CK(e, cudaEventRecord(e->ev_caller, cs));
      CK(e, cudaStreamWaitEvent(e->stream, e->ev_caller, 0));
    }
    if (!capturing && (rc = index_begin(e)) != EPPSCORE_OK) return rc;  // (inside a capture the graph's edges order this)
    for (int32_t p = 0; p < n_picks; p++) d_picks[p] = picks[p];
    // a graph covers every endpoint row: a replay after set_snapshot raised M still commits the new endpoints' picks
    const int32_t n_eps = (e->M > 0 && !capturing) ? e->M : e->geo.Mpad;
    rc = index_status(e, e->index->commit(R, n_picks, d_picks, hashes, n_hashes, hash_stride, caps.empty() ? nullptr : caps.data(), 0, 0,
                                          n_eps, touch_bound, e->stream, capturing),
                      what);
    if (rc != EPPSCORE_OK) return rc;
    if (capturing) {  // the engine stream joins the caller's capture again through an event recorded inside it
      if (cs != e->stream) {
        CK(e, cudaEventRecord(e->ev_index_join, e->stream));
        CK(e, cudaStreamWaitEvent(cs, e->ev_index_join, 0));
      }
      return EPPSCORE_OK;
    }
    if ((rc = index_end(e)) != EPPSCORE_OK) return rc;
    if (cs != e->stream) CK(e, cudaStreamWaitEvent(cs, e->ev_table, 0));  // stream-ordered for the caller
    return EPPSCORE_OK;
  }
  int32_t lo = e->geo.Mpad, hi = -1;
  int64_t touches = 0;
  for (int32_t r = 0; r < R; r++)
    for (int32_t p = 0; p < n_picks; p++) {
      const int32_t ep = picks[p][r];
      if (ep < 0) continue;  // no target endpoint: nothing to record (plugin.go:173-175)
      if (ep >= e->geo.Mpad) return fail(e, EPPSCORE_ERR_INVALID, "pick out of range");
      if (n_hashes[r] > hash_stride) return fail(e, EPPSCORE_ERR_INVALID, "n_hashes exceeds hash_stride");
      lo = std::min(lo, ep);
      hi = std::max(hi, ep);
      touches += n_hashes[r];
    }
  if (hi < 0) return EPPSCORE_OK;  // (a pick with zero hashes still creates the endpoint's LRU, indexer.go:57-68)
  if ((rc = index_begin(e)) != EPPSCORE_OK) return rc;
  HostStage st(e);
  const int32_t* d_pk = st.in(picks, n_picks, R);  // pick array p at row p
  const uint64_t* d_hash = st.in(hashes, (size_t)R * hash_stride);
  const uint16_t* d_nh = st.in(n_hashes, R);
  rc = st.finish([&] {
    for (int32_t p = 0; p < n_picks; p++) d_picks[p] = d_pk + (size_t)p * R;
    return index_status(e, e->index->commit(R, n_picks, d_picks, d_hash, d_nh, hash_stride, caps.empty() ? nullptr : caps.data(), 0,
                                            lo, hi - lo + 1, std::max<int64_t>(touches, 1), e->stream),
                        what);
  });
  if (rc != EPPSCORE_OK) return rc;
  return index_end(e);
}

int32_t eppscore_commit_picks(eppscore_engine* e, int32_t R, const int32_t* pick, const uint64_t* hashes,
                              const uint16_t* n_hashes, int32_t hash_stride, const int32_t* lru_capacity) {
  return commit_calls(e, R, 1, &pick, hashes, n_hashes, hash_stride, lru_capacity, false, 0, nullptr, "commit_picks");
}

int32_t eppscore_commit_picks_device(eppscore_engine* e, int32_t R, const int32_t* pick, const uint64_t* hashes,
                                     const uint16_t* n_hashes, int32_t hash_stride, const int32_t* lru_capacity,
                                     int64_t touch_bound, void* stream) {
  return commit_calls(e, R, 1, &pick, hashes, n_hashes, hash_stride, lru_capacity, true, touch_bound, stream, "commit_picks_device");
}

int32_t eppscore_commit_picks_profiles(eppscore_engine* e, int32_t R, int32_t n_picks, const int32_t* const* picks,
                                       const uint64_t* hashes, const uint16_t* n_hashes, int32_t hash_stride,
                                       const int32_t* lru_capacity, int32_t location, int64_t touch_bound, void* stream) {
  if (e && location != 0 && location != 1) return fail(e, EPPSCORE_ERR_INVALID, "commit_picks_profiles: location must be 0 or 1");
  return commit_calls(e, R, n_picks, picks, hashes, n_hashes, hash_stride, lru_capacity, location == 1, touch_bound, stream,
                      "commit_picks_profiles");
}

int32_t eppscore_prefix_add(eppscore_engine* e, const uint64_t* hashes, int32_t n, int32_t endpoint, int32_t lru_capacity) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (n < 0 || (n > 0 && !hashes)) return fail(e, EPPSCORE_ERR_INVALID, "NULL argument");
  if (n > EPPSCORE_MAX_BLOCKS) return fail(e, EPPSCORE_ERR_CAPACITY, "more than 65535 hashes in one Add");
  if (endpoint < 0 || endpoint >= e->geo.Mpad) return fail(e, EPPSCORE_ERR_INVALID, "endpoint out of range");
  CK(e, cudaSetDevice(e->device));
  int32_t rc = index_skips(e, true, "prefix_add");
  if (rc == EPPSCORE_OK) rc = index_begin(e);
  if (rc != EPPSCORE_OK) return rc;
  const uint16_t nh = (uint16_t)n;
  HostStage st(e);
  const int32_t* d_ep = st.in(&endpoint, 1);
  const uint64_t* d_hash = st.in(hashes, n);  // (nullptr for n = 0: the commit reads n hashes)
  const uint16_t* d_nh = st.in(&nh, 1);
  rc = st.finish([&] {
    return index_status(e, e->index->commit(1, 1, &d_ep, d_hash, d_nh, std::max(n, 1), nullptr, lru_capacity, endpoint, 1,
                                            std::max(n, 1), e->stream),
                        "prefix_add");
  });
  if (rc != EPPSCORE_OK) return rc;
  return index_end(e);
}

int32_t eppscore_prefix_apply(eppscore_engine* e, int64_t n, const uint64_t* hash, const int32_t* endpoint, const uint8_t* op) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (n < 0 || (n > 0 && (!hash || !endpoint || !op))) return fail(e, EPPSCORE_ERR_INVALID, "NULL argument");
  if (n == 0) return EPPSCORE_OK;
  for (int64_t i = 0; i < n; i++)
    if (endpoint[i] < 0 || endpoint[i] >= e->geo.Mpad) return fail(e, EPPSCORE_ERR_CAPACITY, "prefix_apply: endpoint out of range");
  CK(e, cudaSetDevice(e->device));
  int32_t rc = index_skips(e, true, "prefix_apply");
  if (rc == EPPSCORE_OK) rc = index_begin(e);
  if (rc != EPPSCORE_OK) return rc;
  HostStage st(e);
  const uint64_t* d_hash = st.in(hash, n);
  const int32_t* d_ep = st.in(endpoint, n);
  const uint8_t* d_op = st.in(op, n);
  rc = st.finish([&] { return index_status(e, e->index->apply(n, d_hash, d_ep, d_op, e->stream), "prefix_apply"); });
  if (rc != EPPSCORE_OK) return rc;
  return index_end(e);
}

int32_t eppscore_prefix_remove_endpoint(eppscore_engine* e, int32_t endpoint) {
  if (!e) return EPPSCORE_ERR_INVALID;
  CK(e, cudaSetDevice(e->device));
  int32_t rc = index_skips(e, true, "prefix_remove_endpoint");
  if (rc == EPPSCORE_OK) rc = index_begin(e);
  if (rc != EPPSCORE_OK) return rc;
  rc = index_status(e, e->index->remove_endpoint(endpoint, e->stream), "prefix_remove_endpoint");
  if (rc != EPPSCORE_OK) return rc;
  return index_end(e);
}

int32_t eppscore_prefix_lru_len(const eppscore_engine* ce, int32_t endpoint) {
  eppscore_engine* e = const_cast<eppscore_engine*>(ce);
  if (!e) return -1;
  if (cudaSetDevice(e->device) != cudaSuccess) return -1;
  int32_t len = -1;
  if (e->index->lru_keys(endpoint, nullptr, 0, &len, e->stream) != cudaSuccess) return -1;
  return len;
}
int32_t eppscore_prefix_lru_keys(const eppscore_engine* ce, int32_t endpoint, uint64_t* out, int32_t cap) {
  eppscore_engine* e = const_cast<eppscore_engine*>(ce);
  if (!e) return -1;
  if (cudaSetDevice(e->device) != cudaSuccess) return -1;
  int32_t len = -1;
  if (e->index->lru_keys(endpoint, out, cap, &len, e->stream) != cudaSuccess) return -1;
  return len;
}

int32_t eppscore_prefix_get(eppscore_engine* e, uint64_t hash, uint32_t* bitset_out, int32_t words) {
  if (!e) return EPPSCORE_ERR_INVALID;
  CK(e, cudaSetDevice(e->device));
  int32_t count = 0;
  CK(e, e->index->get(hash, bitset_out, bitset_out ? words : 0, &count, e->stream));
  return count;
}

int32_t eppscore_prefix_match(eppscore_engine* e, int32_t R, int32_t k, int32_t location, const uint64_t* hashes,
                              const uint16_t* n_hashes, int32_t hash_stride, const int32_t* endpoints, uint16_t* match_out,
                              void* stream) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (location != 0 && location != 1) return fail(e, EPPSCORE_ERR_INVALID, "prefix_match: location must be 0 or 1");
  if (k < 1 || k > e->cfg.max_endpoints) return fail(e, EPPSCORE_ERR_INVALID, "prefix_match: k must be in [1, max_endpoints]");
  if (R < 0 || (R > 0 && (!hashes || !n_hashes || !endpoints || !match_out))) return fail(e, EPPSCORE_ERR_INVALID, "prefix_match: NULL argument");
  if (R == 0) return EPPSCORE_OK;
  if (hash_stride <= 0) return fail(e, EPPSCORE_ERR_INVALID, "prefix_match: hash_stride must be > 0");
  CK(e, cudaSetDevice(e->device));
  if (location == 1) {
    // Ordered like a device-location batch: after the index mutations issued before it (ev_table), and registered as pending so
    // that later mutations wait for it.  Inside a capture the graph's edges order it.
    // It reads no snapshot term, so it does not wait for the snapshot preparation.
    cudaStream_t cs = stream ? (cudaStream_t)stream : e->stream;
    if (int32_t rc = reader_begin(e, cs, nullptr, nullptr); rc != EPPSCORE_OK) return rc;
    e->index->match(R, k, e->cfg.max_endpoints, hashes, n_hashes, hash_stride, endpoints, match_out, cs);
    CK(e, cudaGetLastError());
    return pending_record(e, cs);
  }
  for (int32_t r = 0; r < R; r++)
    if (n_hashes[r] > hash_stride) return fail(e, EPPSCORE_ERR_INVALID, "prefix_match: n_hashes exceeds hash_stride");
  // host arrays: staged, matched by the device form on the engine stream, copied back
  HostStage st(e);
  const uint64_t* d_hash = st.in(hashes, (size_t)R * hash_stride);
  const uint16_t* d_nh = st.in(n_hashes, R);
  const int32_t* d_ep = st.in(endpoints, (size_t)R * k);
  uint16_t* d_out = st.out(match_out, (size_t)R * k);
  return st.finish([&] { return eppscore_prefix_match(e, R, k, 1, d_hash, d_nh, hash_stride, d_ep, d_out, e->stream); });
}

int32_t eppscore_predict_latency(eppscore_engine* e, int32_t R, int32_t k, int32_t location, const uint64_t* hashes,
                                 const uint16_t* n_hashes, int32_t hash_stride, const int32_t* input_tokens, const double* ttft_slo,
                                 const double* tpot_slo, const int32_t* endpoints, eppscore_latency_info* info_out,
                                 uint16_t* match_out, void* stream) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (location != 0 && location != 1) return fail(e, EPPSCORE_ERR_INVALID, "predict_latency: location must be 0 or 1");
  if (k < 1 || k > e->cfg.max_endpoints) return fail(e, EPPSCORE_ERR_INVALID, "predict_latency: k must be in [1, max_endpoints]");
  if (R < 0 || (R > 0 && (!hashes || !n_hashes || !endpoints || !info_out)))
    return fail(e, EPPSCORE_ERR_INVALID, "predict_latency: NULL argument");
  if (!e->have_snapshot) return fail(e, EPPSCORE_ERR_INVALID, "predict_latency before set_snapshot");
  if (!e->lat_ep.p || !e->lat_args.enabled)
    return fail(e, EPPSCORE_ERR_INVALID, "predict_latency: the snapshot was prepared without a profile with a latency scorer");
  if (R == 0) return EPPSCORE_OK;
  if (hash_stride <= 0) return fail(e, EPPSCORE_ERR_INVALID, "predict_latency: hash_stride must be > 0");
  CK(e, cudaSetDevice(e->device));
  if (location == 0) {
    for (int32_t r = 0; r < R; r++)
      if (n_hashes[r] > hash_stride) return fail(e, EPPSCORE_ERR_INVALID, "predict_latency: n_hashes exceeds hash_stride");
    // host arrays: staged, predicted by the device form on the engine stream, copied back
    HostStage st(e);
    const uint64_t* d_hash = st.in(hashes, (size_t)R * hash_stride);
    const uint16_t* d_nh = st.in(n_hashes, R);
    const int32_t* d_ep = st.in(endpoints, (size_t)R * k);
    const int32_t* d_tok = st.in(input_tokens, R);
    const double* d_ttft = st.in(ttft_slo, R);
    const double* d_tpot = st.in(tpot_slo, R);
    eppscore_latency_info* d_info = st.out(info_out, (size_t)R * k);
    uint16_t* d_match = st.out(match_out, (size_t)R * k);
    return st.finish([&] {
      return eppscore_predict_latency(e, R, k, 1, d_hash, d_nh, hash_stride, d_tok, d_ttft, d_tpot, d_ep, d_info, d_match, e->stream);
    });
  }
  // Ordered like a device-location batch: after the index mutations, snapshot preparations and producer updates issued before
  // it, and registered as pending so that later ones wait for it.  Inside a capture the graph's edges order it.
  cudaStream_t cs = stream ? (cudaStream_t)stream : e->stream;
  bool capturing = false, wait_snapshot = false;
  if (int32_t rc = reader_begin(e, cs, &capturing, &wait_snapshot); rc != EPPSCORE_OK) return rc;
  if (!capturing && e->producer_pending) CK(e, cudaStreamWaitEvent(cs, e->ev_producer, 0));
  if (wait_snapshot) CK(e, cudaStreamWaitEvent(cs, e->ev_snapshot, 0));
  const LatArgs& L = e->lat_args;
  LatInfoArgs a{};
  a.R = R;
  a.k = k;
  a.M = e->M;
  a.has_predictions = L.has_predictions;
  a.stride = hash_stride;
  a.ep = L.ep;
  a.dispatched = e->base_pa.dispatched;  // the snapshot's array, else the running-request counts (eppscore_set_snapshot)
  a.ttft_input = L.ttft_input;
  a.ttft_prefix = L.ttft_prefix;
  a.tpot_input = L.tpot_input;
  a.tpot_generated = L.tpot_generated;
  a.buffer = L.buffer;
  a.hashes = hashes;
  a.n_hashes = n_hashes;
  a.endpoints = endpoints;
  a.input_tokens = input_tokens;
  a.ttft_slo = ttft_slo;
  a.tpot_slo = tpot_slo;
  a.match_out = match_out;
  a.out = info_out;
  e->index->latency_info(a, e->cfg.max_endpoints, cs);
  CK(e, cudaGetLastError());
  if (!capturing && !e->snapshot_has_dispatched) {  // it reads the running-request counts in place (count_reads_wait)
    if (cs == e->stream) {
      CK(e, cudaEventRecord(e->ev_count_read, cs));
      e->count_read_engine = true;
    } else {
      e->count_readers = true;
    }
  }
  return pending_record(e, cs);
}

// ---------------- in-flight load producer ----------------
int32_t eppscore_estimate_tokens(eppscore_engine* e, int32_t R, int32_t location, const int64_t* request_size_bytes,
                                 const int32_t* token_hint, const int32_t* prompt_chars, int64_t* out, void* stream) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (R < 0 || (R > 0 && !out)) return fail(e, EPPSCORE_ERR_INVALID, "estimate_tokens: R < 0 or out NULL");
  if (R == 0) return EPPSCORE_OK;
  CK(e, cudaSetDevice(e->device));
  if (location == 1) {
    e->launches += launch_estimate_tokens(request_size_bytes, token_hint, prompt_chars, R, out, stream ? (cudaStream_t)stream : e->stream);
    CK(e, cudaGetLastError());
    return EPPSCORE_OK;
  }
  // host arrays: staged, estimated by the device form on the engine stream, copied back
  HostStage st(e);
  const int64_t* d_size = st.in(request_size_bytes, R);
  const int32_t* d_hint = st.in(token_hint, R);
  const int32_t* d_chars = st.in(prompt_chars, R);
  int64_t* d_out = st.out(out, R);
  return st.finish([&] { return eppscore_estimate_tokens(e, R, 1, d_size, d_hint, d_chars, d_out, e->stream); });
}

static int32_t inflight_update(eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint, const int64_t* tokens,
                               void* stream, int sign) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (R < 0 || (R > 0 && !endpoint)) return fail(e, EPPSCORE_ERR_INVALID, "inflight update: R < 0 or endpoint NULL");
  if (R == 0) return EPPSCORE_OK;
  CK(e, cudaSetDevice(e->device));
  const bool on_device = location == 1;
  cudaStream_t st = (on_device && stream) ? (cudaStream_t)stream : e->stream;
  const int32_t* d_ep = endpoint;
  const int64_t* d_tok = tokens;
  HostStage staged(e);
  if (!on_device) {
    for (int32_t r = 0; r < R; r++)
      if (endpoint[r] >= e->cfg.max_endpoints) return fail(e, EPPSCORE_ERR_INVALID, "inflight update: endpoint >= max_endpoints");
    d_ep = staged.in(endpoint, R);
    d_tok = staged.in(tokens, R);
  }
  auto update = [&]() -> int32_t {
    bool capturing = false;
    int32_t rc = producer_begin(e, st, &capturing);
    if (rc != EPPSCORE_OK) return rc;
    e->launches += launch_inflight_update(d_ep, d_tok, R, e->cfg.max_endpoints, sign, e->inflight_req.as<int64_t>(),
                                          e->inflight_tok.as<int64_t>(), e->inflight_err.as<uint32_t>(), st);
    CK(e, cudaGetLastError());
    return producer_end(e, st, capturing, counters_feed_scorer(e));
  };
  return on_device ? update() : staged.finish(update);
}

int32_t eppscore_inflight_add(eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint, const int64_t* tokens,
                              void* stream) {
  return inflight_update(e, R, location, endpoint, tokens, stream, 1);
}

int32_t eppscore_inflight_release(eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint, const int64_t* tokens,
                                  void* stream) {
  return inflight_update(e, R, location, endpoint, tokens, stream, -1);
}

int32_t eppscore_inflight_remove_endpoint(eppscore_engine* e, int32_t endpoint) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (endpoint < 0 || endpoint >= e->cfg.max_endpoints) return fail(e, EPPSCORE_ERR_INVALID, "inflight_remove_endpoint: endpoint out of range");
  CK(e, cudaSetDevice(e->device));
  bool capturing = false;
  int32_t rc = producer_begin(e, e->stream, &capturing);
  if (rc != EPPSCORE_OK) return rc;
  CK(e, cudaMemsetAsync(e->inflight_req.as<int64_t>() + endpoint, 0, 8, e->stream));
  CK(e, cudaMemsetAsync(e->inflight_tok.as<int64_t>() + endpoint, 0, 8, e->stream));
  return producer_end(e, e->stream, capturing, counters_feed_scorer(e));
}

int32_t eppscore_inflight_get(eppscore_engine* e, int64_t* requests_out, int64_t* tokens_out, int32_t M) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (M < 0 || M > e->cfg.max_endpoints) return fail(e, EPPSCORE_ERR_INVALID, "inflight_get: M outside [0, max_endpoints]");
  CK(e, cudaSetDevice(e->device));
  if (e->producer_pending) CK(e, cudaStreamWaitEvent(e->stream, e->ev_producer, 0));
  uint32_t err = 0;
  if (M > 0 && requests_out) CK(e, cudaMemcpyAsync(requests_out, e->inflight_req.p, (size_t)M * 8, cudaMemcpyDeviceToHost, e->stream));
  if (M > 0 && tokens_out) CK(e, cudaMemcpyAsync(tokens_out, e->inflight_tok.p, (size_t)M * 8, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaMemcpyAsync(&err, e->inflight_err.p, 4, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  if (err) {
    CK(e, cudaMemsetAsync(e->inflight_err.p, 0, 4, e->stream));
    return fail(e, EPPSCORE_ERR_INVALID, "an inflight update on device arrays named an endpoint >= max_endpoints (those entries were skipped)");
  }
  return EPPSCORE_OK;
}

}  // extern "C"

// ---------------- running-request queues (predicted-latency producer) ----------------
namespace {

// The live / tombstone counters as of every mutation ordered before `st`'s current end: read synchronously.  This also
// re-bases the bounds after graph replays, which the host does not see.
int32_t run_read_exact(eppscore_engine* e, cudaStream_t st) {
  CK(e, cudaMemcpyAsync(e->h_run.p, e->run_ctr.p, sizeof(RunCounters), cudaMemcpyDeviceToHost, st));
  CK(e, cudaStreamSynchronize(st));
  e->run_bound_live = (int64_t)e->h_run.as<RunCounters>()->live;
  e->run_copy_issued = false;
  e->run_captured = false;
  return EPPSCORE_OK;
}

// The device descriptor the kernels read the table and the scratch through.  The compaction kernels swap the table with its
// spare on the device, so the host reads the descriptor back before it changes it.  Both run synchronously on `st`.
int32_t run_desc_download(eppscore_engine* e, cudaStream_t st) {
  CK(e, cudaStreamSynchronize(st));
  CK(e, cudaMemcpyAsync(&e->run_host, e->run_desc.p, sizeof(RunDev), cudaMemcpyDeviceToHost, st));
  CK(e, cudaStreamSynchronize(st));
  return EPPSCORE_OK;
}
int32_t run_desc_upload(eppscore_engine* e, cudaStream_t st) {
  CK(e, cudaMemcpyAsync(e->run_desc.p, &e->run_host, sizeof(RunDev), cudaMemcpyHostToDevice, st));
  CK(e, cudaStreamSynchronize(st));
  return EPPSCORE_OK;
}

// Grows the table to `slots` slots on `st` (outside a capture): a new table and spare, the live entries moved into it, the
// descriptor pointed at it.  Graphs captured earlier read the table through the descriptor and the grid-stride passes loop
// over its capacity, so they stay valid.
int32_t run_grow(eppscore_engine* e, cudaStream_t st, int64_t slots) {
  std::array<DevBuf, 8> nb;
  cudaError_t c = run_alloc_table(slots, &nb[0], st);
  if (c == cudaSuccess) c = run_alloc_table(slots, &nb[4], st);
  if (c != cudaSuccess) return cuda_fail(e, c, "running-request table allocation");
  int32_t rc = run_desc_download(e, st);
  if (rc != EPPSCORE_OK) return rc;
  const RunDev src = e->run_host;
  RunDev& d = e->run_host;
  d.slot = nb[0].as<RunSlot>();
  d.tpot = nb[1].as<unsigned long long>();
  d.owner = nb[2].as<unsigned long long>();
  d.rm = nb[3].as<unsigned long long>();
  d.spare_slot = nb[4].as<RunSlot>();
  d.spare_tpot = nb[5].as<unsigned long long>();
  d.spare_owner = nb[6].as<unsigned long long>();
  d.spare_rm = nb[7].as<unsigned long long>();
  d.mask = (unsigned long long)slots - 1;
  e->launches += launch_running_rebuild(src, d, e->sm_count, st);  // also zeroes the tombstone count
  CK(e, cudaGetLastError());
  if ((rc = run_desc_upload(e, st)) != EPPSCORE_OK) return rc;
  e->run_tab = std::move(nb);  // nb takes the old tables and frees them
  e->run_cap = slots;
  return EPPSCORE_OK;
}

// Room for R more entries before an add.  Tombstones are the device's business (the compaction launched before every add),
// so the host only guarantees live + R <= capacity / 2, from its upper bound on the live entries: the counters copied back
// behind an earlier call once that copy has landed, plus R per add issued since.  Outside a capture the bound is held to a
// quarter, so that compactions stay rare; when it does not hold, the exact count decides whether the table doubles (only
// while live + R exceed a quarter of the slots: churn never grows it).  Inside a capture nothing can grow.
int32_t run_make_room(eppscore_engine* e, cudaStream_t st, int64_t R, bool capturing) {
  if (capturing) {
    if (e->run_bound_live + R <= e->run_cap / 2) return EPPSCORE_OK;
    return fail(e, EPPSCORE_ERR_CAPACITY, "running_add under CUDA-graph capture: the table may not have room for R more entries "
                                          "(size it with eppscore_running_reserve before the capture)");
  }
  bool exact = false;
  if (e->run_captured) {  // graph replays may have changed the counters since: read them once
    int32_t rc = run_read_exact(e, st);
    if (rc != EPPSCORE_OK) return rc;
    exact = true;
  } else if (e->run_copy_issued && cudaEventQuery(e->ev_run_copy) == cudaSuccess) {
    e->run_bound_live = (int64_t)e->h_run.as<RunCounters>()->live;
    e->run_copy_issued = false;
  }
  if (e->run_bound_live + R <= e->run_cap / 4) return EPPSCORE_OK;
  if (!exact) {
    int32_t rc = run_read_exact(e, st);
    if (rc != EPPSCORE_OK) return rc;
  }
  int64_t slots = e->run_cap;
  while (e->run_bound_live + R > slots / 4) slots *= 2;
  return slots == e->run_cap ? EPPSCORE_OK : run_grow(e, st, slots);
}

// Per-call scratch of at least R entries.  Under a capture it cannot be allocated; outside one a larger scratch replaces the
// old one in the descriptor.
int32_t run_scratch(eppscore_engine* e, cudaStream_t st, int64_t R, bool capturing) {
  if ((size_t)R * 4 <= e->c_rslot.bytes && (size_t)R <= e->c_rwon.bytes) return EPPSCORE_OK;
  if (capturing)
    return fail(e, EPPSCORE_ERR_CAPACITY, "running update under CUDA-graph capture: R exceeds the scratch sized by "
                                          "eppscore_running_reserve");
  int32_t rc = run_desc_download(e, st);
  if (rc != EPPSCORE_OK) return rc;
  CK(e, e->c_rslot.reserve((size_t)R * 4));
  CK(e, e->c_rwon.reserve((size_t)R));
  e->run_host.slot_of = e->c_rslot.as<int32_t>();
  e->run_host.won = e->c_rwon.as<uint8_t>();
  return run_desc_upload(e, st);
}

// Behind every mutation outside a capture: the counters are copied back asynchronously, for the next room check.
int32_t run_copy_back(eppscore_engine* e, cudaStream_t st, bool capturing) {
  if (capturing) {
    e->run_captured = true;
    return EPPSCORE_OK;
  }
  CK(e, cudaMemcpyAsync(e->h_run.p, e->run_ctr.p, sizeof(RunCounters), cudaMemcpyDeviceToHost, st));
  CK(e, cudaEventRecord(e->ev_run_copy, st));
  e->run_copy_issued = true;
  return EPPSCORE_OK;
}

// Before a running-request update's kernel on `st` (outside a capture): every device-location eppscore_predict_latency issued
// earlier that reads the counts in place has finished reading them.  The flags clear once those reads are known to be done, so
// the extra waits last only while such a call may be in flight.
int32_t count_reads_wait(eppscore_engine* e, cudaStream_t st) {
  if (e->count_readers) {
    int32_t rc = pending_wait(e, st);
    if (rc != EPPSCORE_OK) return rc;
    bool armed = false;
    for (const PendingBatch& p : e->pending) armed = armed || p.armed;
    if (!armed) e->count_readers = false;
  }
  if (e->count_read_engine) {
    if (cudaEventQuery(e->ev_count_read) == cudaSuccess) e->count_read_engine = false;
    else if (st != e->stream) CK(e, cudaStreamWaitEvent(st, e->ev_count_read, 0));
  }
  return EPPSCORE_OK;
}

int32_t running_update(eppscore_engine* e, int op, int32_t R, int32_t location, const int32_t* endpoint, const uint64_t* key,
                       const double* tpot, uint8_t* out, void* stream) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (R < 0 || (R > 0 && (!endpoint || !key))) return fail(e, EPPSCORE_ERR_INVALID, "running update: R < 0, or endpoint / request_key NULL");
  if (R == 0) return EPPSCORE_OK;
  CK(e, cudaSetDevice(e->device));
  const bool on_device = location == 1;
  cudaStream_t st = (on_device && stream) ? (cudaStream_t)stream : e->stream;
  const int32_t* d_ep = endpoint;
  const uint64_t* d_key = key;
  const double* d_tpot = tpot;
  HostStage staged(e);
  if (!on_device) {
    for (int32_t r = 0; r < R; r++) {
      if (endpoint[r] >= e->cfg.max_endpoints) return fail(e, EPPSCORE_ERR_INVALID, "running update: endpoint >= max_endpoints");
      if (tpot && std::isnan(tpot[r])) return fail(e, EPPSCORE_ERR_INVALID, "running_add: tpot_slo is NaN");
    }
    d_ep = staged.in(endpoint, R);
    d_key = staged.in(key, R);
    d_tpot = staged.in(tpot, R);
  }
  auto update = [&]() -> int32_t {
    bool capturing = false;
    int32_t rc = producer_begin(e, st, &capturing);
    if (rc != EPPSCORE_OK) return rc;
    if (!capturing && (rc = count_reads_wait(e, st)) != EPPSCORE_OK) return rc;
    if (op == 0 && (rc = run_make_room(e, st, R, capturing)) != EPPSCORE_OK) return rc;
    if ((rc = run_scratch(e, st, R, capturing)) != EPPSCORE_OK) return rc;
    e->launches += launch_running_update(e->run_desc.as<RunDev>(), (unsigned long long)e->run_cap, op, d_ep, d_key,
                                          op == 0 ? d_tpot : nullptr, R, e->cfg.max_endpoints, on_device ? out : nullptr,
                                          e->sm_count, st);
    CK(e, cudaGetLastError());
    if (!on_device && out) CK(e, cudaMemcpyAsync(out, e->c_rwon.p, (size_t)R, cudaMemcpyDeviceToHost, st));
    if (op == 0) e->run_bound_live += R;
    if ((rc = run_copy_back(e, st, capturing)) != EPPSCORE_OK) return rc;
    return producer_end(e, st, capturing, running_feeds_scorer(e));
  };
  return on_device ? update() : staged.finish(update);
}

}  // namespace

extern "C" {

int32_t eppscore_running_add(eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint, const uint64_t* request_key,
                             const double* tpot_slo, uint8_t* added_out, void* stream) {
  return running_update(e, 0, R, location, endpoint, request_key, tpot_slo, added_out, stream);
}

int32_t eppscore_running_remove(eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint,
                                const uint64_t* request_key, uint8_t* removed_out, void* stream) {
  return running_update(e, 1, R, location, endpoint, request_key, nullptr, removed_out, stream);
}

int32_t eppscore_running_remove_endpoint(eppscore_engine* e, int32_t endpoint) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (endpoint < 0 || endpoint >= e->cfg.max_endpoints) return fail(e, EPPSCORE_ERR_INVALID, "running_remove_endpoint: endpoint out of range");
  CK(e, cudaSetDevice(e->device));
  bool capturing = false;
  int32_t rc = producer_begin(e, e->stream, &capturing);
  if (rc == EPPSCORE_OK && !capturing) rc = count_reads_wait(e, e->stream);
  if (rc != EPPSCORE_OK) return rc;
  e->launches += launch_running_drop_endpoint(e->run_desc.as<RunDev>(), (unsigned long long)e->run_cap, endpoint,
                                              e->cfg.max_endpoints, e->sm_count, e->stream);
  CK(e, cudaGetLastError());
  if ((rc = run_copy_back(e, e->stream, capturing)) != EPPSCORE_OK) return rc;
  if ((rc = producer_end(e, e->stream, capturing, running_feeds_scorer(e))) != EPPSCORE_OK) return rc;
  // the live count only goes down: the host bound stays an upper bound
  return EPPSCORE_OK;
}

int32_t eppscore_running_get(eppscore_engine* e, double* min_tpot_out, int32_t* count_out, int32_t M) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (M < 0 || M > e->cfg.max_endpoints) return fail(e, EPPSCORE_ERR_INVALID, "running_get: M outside [0, max_endpoints]");
  CK(e, cudaSetDevice(e->device));
  if (e->producer_pending) CK(e, cudaStreamWaitEvent(e->stream, e->ev_producer, 0));
  if (M > 0 && min_tpot_out) CK(e, cudaMemcpyAsync(min_tpot_out, e->run_min_view.p, (size_t)M * 8, cudaMemcpyDeviceToHost, e->stream));
  if (M > 0 && count_out) CK(e, cudaMemcpyAsync(count_out, e->run_count.p, (size_t)M * 4, cudaMemcpyDeviceToHost, e->stream));
  int32_t rc = run_read_exact(e, e->stream);
  if (rc != EPPSCORE_OK) return rc;
  const unsigned err = e->h_run.as<RunCounters>()->err;
  if (err) {
    CK(e, cudaMemsetAsync(&e->run_ctr.as<RunCounters>()->err, 0, 4, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    if (err & kRunErrCapacity)
      return fail(e, EPPSCORE_ERR_CAPACITY, "a running_add found no empty slot (a graph was replayed past the room "
                                            "eppscore_running_reserve made); those entries were not added");
    return fail(e, EPPSCORE_ERR_INVALID, "a running update on device arrays named an endpoint >= max_endpoints or a NaN "
                                         "tpot (those entries were skipped)");
  }
  return EPPSCORE_OK;
}

int32_t eppscore_running_reserve(eppscore_engine* e, int64_t live_entries) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (live_entries < 0 || live_entries > (int64_t)1 << 29) return fail(e, EPPSCORE_ERR_INVALID, "running_reserve: live_entries outside [0, 2^29]");
  if (live_entries > 0) {
    CK(e, cudaSetDevice(e->device));
    if (e->producer_pending) CK(e, cudaStreamWaitEvent(e->stream, e->ev_producer, 0));
    int32_t rc = run_read_exact(e, e->stream);
    if (rc != EPPSCORE_OK) return rc;
    int64_t slots = e->run_cap;
    while (live_entries > slots / 2) slots *= 2;
    if (slots != e->run_cap && (rc = run_grow(e, e->stream, slots)) != EPPSCORE_OK) return rc;
    if ((rc = run_scratch(e, e->stream, live_entries, false)) != EPPSCORE_OK) return rc;
  }
  return (int32_t)(e->run_cap / 2);
}

int32_t eppscore_prefix_reserve(eppscore_engine* e, int64_t live_hashes, int64_t touches_per_call, int64_t overflow_rows) {
  if (!e) return EPPSCORE_ERR_INVALID;
  const int64_t lim = (int64_t)1 << 34;
  if (live_hashes < 0 || touches_per_call < 0 || overflow_rows < 0 || live_hashes > lim || touches_per_call > lim || overflow_rows >= 0xFFFFFFF0LL)
    return fail(e, EPPSCORE_ERR_INVALID, "prefix_reserve: an argument is negative or too large");
  CK(e, cudaSetDevice(e->device));
  if (capture_open(e, e->stream)) return fail(e, EPPSCORE_ERR_INVALID, "prefix_reserve under CUDA-graph capture");
  if (live_hashes == 0) live_hashes = e->cfg.prefix_capacity;
  if (touches_per_call == 0) touches_per_call = 65536;
  if (overflow_rows == 0) overflow_rows = 2 * touches_per_call;
  int32_t rc = index_begin(e);
  if (rc != EPPSCORE_OK) return rc;
  CK(e, e->index->reserve(live_hashes, touches_per_call, overflow_rows, e->stream));
  return index_end(e);
}

int32_t eppscore_reserve_stream(eppscore_engine* e, void* stream, int32_t max_R, int32_t max_blocks) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (!stream) return fail(e, EPPSCORE_ERR_INVALID, "reserve_stream: stream is NULL");
  if (max_R < 1) return fail(e, EPPSCORE_ERR_INVALID, "reserve_stream: max_R < 1");
  if (max_blocks < 0 || max_blocks > EPPSCORE_MAX_BLOCKS) return fail(e, EPPSCORE_ERR_INVALID, "reserve_stream: max_blocks outside [0, 65535]");
  CK(e, cudaSetDevice(e->device));
  cudaStream_t s = (cudaStream_t)stream;
  if (capture_open(e, s)) return fail(e, EPPSCORE_ERR_INVALID, "reserve_stream under CUDA-graph capture");
  if (reserved_scratch(e, s)) return fail(e, EPPSCORE_ERR_INVALID, "reserve_stream: the stream is already reserved (release it first)");
  if (e->reserved.size() >= EPPSCORE_MAX_STREAMS) return fail(e, EPPSCORE_ERR_CAPACITY, "reserve_stream: at most EPPSCORE_MAX_STREAMS streams");
  // everything schedule_device and schedule_wide reserve in a set, for max_R requests; the wide score rows come with the
  // first wide call, as for sc[0]
  auto r = std::make_unique<StreamScratch>();
  const int32_t mb = max_blocks > 0 ? max_blocks : e->cfg.max_blocks;
  const size_t R = (size_t)max_R, mw = (size_t)e->geo.Mpad / 32;
  Scratch& sc = r->sc;
  CK(e, sc.s_hashes.reserve(R * mb * 8));
  CK(e, sc.s_nh.reserve(R * 2));
  CK(e, sc.s_fields.reserve(R * 4));
  CK(e, sc.s_probe.reserve(R * sizeof(ProbeRec)));
  CK(e, sc.s_subset.reserve(R * mw * 4));  // whatever the profiles: profiles and subsets may come after the reserve
  sc.rows = max_R;
  r->max_R = max_R;
  r->max_blocks = mb;
  r->stream = s;  // (last: a set that failed above is freed without waiting for the stream)
  e->reserved.push_back(std::move(r));
  return EPPSCORE_OK;
}

int32_t eppscore_release_stream(eppscore_engine* e, void* stream) {
  if (!e) return EPPSCORE_ERR_INVALID;
  if (!stream) return fail(e, EPPSCORE_ERR_INVALID, "release_stream: stream is NULL");
  CK(e, cudaSetDevice(e->device));
  cudaStream_t s = (cudaStream_t)stream;
  if (capture_open(e, s)) return fail(e, EPPSCORE_ERR_INVALID, "release_stream under CUDA-graph capture");
  auto it = std::find_if(e->reserved.begin(), e->reserved.end(), [s](const auto& r) { return r->stream == s; });
  if (it == e->reserved.end()) return fail(e, EPPSCORE_ERR_INVALID, "release_stream: the stream is not reserved");
  CK(e, cudaStreamSynchronize(s));
  e->reserved.erase(it);
  return EPPSCORE_OK;
}

void* eppscore_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) return nullptr;
  return p;
}
void eppscore_host_free(void* p) {
  if (p) cudaFreeHost(p);
}

}  // extern "C"
