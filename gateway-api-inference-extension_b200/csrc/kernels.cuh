// kernels.cuh — device-side data layout and launchers of the Endpoint-Picker kernel family.
//
// Data layout in HBM (DESIGN.md §3):
//   * endpoint tile: per-endpoint float64 "term" arrays (clamp(score)*weight, already rounded exactly
//     as scheduler_profile.go:168 would) in natural endpoint order; the streaming kernels stage them
//     into shared memory once per CTA;
//   * every per-endpoint BIT structure (prefix-table rows, LoRA class planes, tie masks) uses one
//     lane-major permutation so that a lane owns the same endpoints in all of them:
//         endpoint m = (j*EPL + k)*32 + lane   <->   bit k of 32-bit word (j*32 + lane)
//     (EPL = endpoints per lane per pass = 8/16/32 chosen from max_endpoints, j = pass).  Natural-order
//     arrays (terms, candidate masks, dense rows, match output) are then read/written with consecutive
//     lanes touching consecutive endpoints — coalesced and bank-conflict free;
//   * prefix table: device-resident index (prefix_table.cuh): 32-byte open-addressing slots that carry sets of up to
//     8 endpoints inline, natural-order bitset rows for larger sets, per-endpoint log-structured LRUs.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "prefix_table.cuh"

namespace eppscore {

constexpr int kMaxSteps = 8;
constexpr int kLutMax = 256;  // per-warp prefix LUT covers total <= 256 (defaultMaxPrefixBlocks)

enum StepKind : int32_t {
  STEP_EP_TERM = 0,  // + term[arg][m]                  (request-independent scorer, precomputed)
  STEP_PREFIX = 1,   // + clamp(match/total)*w          (scorer/prefix/plugin.go:95-117)
  STEP_LORA = 2,     // + clamp(class score)*w          (scorer/loraaffinity/lora_affinity.go:76-102)
  STEP_PAIR = 3,     // + clamp(double(feat[arg]))*w    (dense per-pair column)
  STEP_MINMAX = 4,   // + clamp((max-q)/(max-min))*w over the candidate set (queue.go:78-108), arg: 0 queue 1 running
  STEP_LATENCY = 5   // + clamp(latency-scorer)*w: prediction + headroom + tier/bucket logic (scorer/latency/plugin.go:144-318)
};

// Latency fold-in (score_matrix.cu).  Per-endpoint values are prepared once per snapshot (prepare_kernel.cu) in
// TILES of 32 endpoints x 8 slots: slot i of endpoint (t*32 + lane) is ep[(t*8 + i)*32 + lane], so a warp reads a
// slot of 32 consecutive endpoints with one coalesced load and all slots of a pair sit at immediate offsets.
//   with predictions:  0 tA = ttft_intercept + ttft_kv*kv   1 tW = ttft_waiting*waiting   2 tR = ttft_running*running
//                      3 pA = tpot_intercept + tpot_kv*kv   4 pW = tpot_waiting*waiting   5 pR = tpot_running*running
//                      6 lim = podMinTPOTSLO > 0 ? podMinTPOTSLO*buffer : +inf
//                      7 flags (int64 bits): bit 0 dispatched == 0 (idle), bit 1 TPOT neutralised (!streaming || prefill)
//   composite fallback: 0 cK = composite_kv*(1-kv)           1 WaitingQueueSize (int64 bits)
constexpr int kLatArrays = 8;
struct LatArgs {
  int32_t enabled;
  int32_t has_predictions;
  int32_t strategy_most;
  int32_t pad;
  double ttft_input, ttft_prefix, tpot_input, tpot_generated;
  double buffer;            // SLOBufferFactor
  double alpha, beta;       // normalizedWeights(ttftWeight, tpotWeight), plugin.go:373-379
  double wq, wpref;         // normalised composite weights (queue, prefix); the kv one is folded into ep[7]
  const double* ep;         // [Mpad/32][kLatArrays][32] tiles
  const int32_t* input_tokens;  // [R] or null
  const double* ttft_slo;   // [R] or null
  const double* tpot_slo;   // [R] or null
  double* pred_out;         // [R][M][2] or null
};

struct Plan {
  int32_t n_steps;
  int32_t kind[kMaxSteps];
  int32_t arg[kMaxSteps];
  double weight[kMaxSteps];
  double lora_term[kMaxSteps][4];  // per LoRA step: clamp({0,0.6,0.8,1.0})*w, rounded on the host (one IEEE multiply)
  int32_t tie_mode;
  uint32_t seed_lo, seed_hi;
  int32_t n_terms;       // number of term arrays the steps reference
  uint32_t seq;          // the step kinds packed 4 bits each (kind+1), 0 = end: selects a specialised kernel
  int32_t sparse_ok;     // unmasked plan only: steps are E/P/L with at most one prefix step of weight >= 0
  int32_t pick_mode;     // 0 max-score, 1 weighted-random (A-Res), 2 random  (include/eppscore.h: eppscore_pick_mode)
};

// Geometry derived from config.max_endpoints (fixed per engine); M varies per snapshot.
struct Geo {
  int32_t M;
  int32_t log_epl;  // 3,4,5
  int32_t J;        // passes; Mpad = J*32*EPL
  int32_t Mpad;
  int32_t row_words;  // J*32
};

inline Geo make_geo(int32_t M) {
  Geo g;
  g.M = M;
  g.log_epl = M <= 256 ? 3 : (M <= 512 ? 4 : 5);
  const int per_pass = 32 << g.log_epl;
  int need = (M + per_pass - 1) / per_pass;
  if (need < 1) need = 1;
  int J = 1;  // J is a template parameter; round up to the instantiated set {1,2,4,8}
  while (J < need) J <<= 1;
  g.J = J;
  g.Mpad = g.J * per_pass;
  g.row_words = g.J * 32;
  return g;
}

// bit position of endpoint m inside a permuted bitset row (word = pos>>5, bit = pos&31)
__host__ __device__ inline uint32_t perm_bitpos(uint32_t m, int log_epl) {
  const uint32_t lane = m & 31u, t = m >> 5;  // t = j*EPL + k
  const uint32_t k = t & ((1u << log_epl) - 1u), j = t >> log_epl;
  return ((j * 32u + lane) << 5) + k;
}

// Per-adapter summary of the request-independent part of the score map (sparse fast path):
// over all endpoints m, G[a][m] = score with zero prefix match for a request whose adapter is a.
struct __align__(16) AdapterSummary {
  double gmax;   // max_m G[a][m]
  int32_t garg;  // lowest m attaining it (-1 when M == 0)
  int32_t gcnt;  // how many endpoints attain it
};

// Value buckets of WaitingQueueSize / RunningRequestsSize for the masked min/max (queue.go:79-91 over the FILTERED
// endpoints): bucket v holds a natural-order bitset (same layout as a candidate-mask row) of the endpoints whose value
// is base + v.  min/max over a request's candidates = first / last occupied bucket that intersects its mask row.
// Built per snapshot when max - min <= 255 over all endpoints, otherwise valid = 0 and the kernel scans.
struct QBucketHdr {
  long long base;
  int32_t valid;
  int32_t pad;
  uint32_t occ[8];  // bit v: bucket v is non-empty
};
constexpr int kQBuckets = 256;

// What the hashing kernel found in the prefix index for one request, when it probed the index itself (hash_warp_kernel<BC,
// true>): the request's n matched blocks are all hits carrying one inline set, {raw cnt word, ep0 | ep1 << 16, hi = ep2..ep9}
// exactly as pick_sparse_kernel loads a slot; n == kProbeUnresolved sends the request through pick_sparse's own probe.
struct __align__(16) ProbeRec {
  uint32_t raw, w, n, pad;
  uint4 hi;
};
constexpr uint32_t kProbeUnresolved = 0xFFFFFFFFu;

struct ScoreArgs {
  Geo geo;
  Plan plan;
  int32_t R;
  int64_t request_base;
  // endpoint tile (natural order, Mpad entries each; padding scores are never candidates)
  const double* term[kMaxSteps];
  const int64_t* minmax_q[2];   // queue / running raw values for STEP_MINMAX (masked mode)
  const QBucketHdr* qhdr[2];    // value buckets (null: not built)
  const uint32_t* qbucket[2];   // [kQBuckets][Mpad/32]
  // LoRA class planes, permuted layout: [A+1][row_words] each; row A = "adapter not in dictionary"
  const uint32_t* cls_lo;
  const uint32_t* cls_hi;
  int32_t A;
  const AdapterSummary* summ;   // [A+1]  (sparse path)
  const uint32_t* tiemask;      // [A+1][row_words] permuted bits: G[a][m] == gmax  (sparse path)
  const uint32_t* member;       // [row_words] permuted bits: the profile's endpoint subset (sparse path), or null: all endpoints
  const double* prefix_lut2d;  // [(kLutMax+1)^2]: lut2d[total*(kLutMax+1)+c] = clamp(c/total)*w_prefix, or null
  const int32_t* adapter_id;    // [R] or null
  const uint32_t* cand_mask;    // [R][mask_words] natural order or null
  int32_t mask_words;
  // prefix
  const uint64_t* hashes;       // [R][hash_stride] or null
  const uint16_t* n_hashes;     // [R]
  int32_t hash_stride;
  const TableView* table;       // device pointer to the prefix index's view (null: no table) — stable across rebuilds
  const ProbeRec* probe;        // [R] or null: the hashing kernel's probe of this batch (pick_sparse skips the resolved rows)
  // dense rows
  const float4* dense;          // [R][M]
  const uint16_t* dense_total;  // [R]
  // outputs
  int32_t* pick;
  double* pick_score;
  int32_t* tie_count;
  uint16_t* match_out;          // [R][M] or null
  uint16_t* total_out;          // [R] or null
  double* scores_out;           // [R][M] or null (diagnostics)
  int32_t topk;                 // > 0: the first topk entries of each request's pick order (full-matrix / generic dense kernels)
  int32_t* topk_m;              // [R][topk]
  double* topk_score;           // [R][topk]
  LatArgs lat;
  // device-side filters of the latency profile (run before the scorers, on top of cand_mask): kind 1 prefix-cache-affinity
  // {threshold, explorationProbability, maxTTFTPenaltyMs}, kind 2 slo-headroom-tier {epsilonExploreNeg}
  int32_t n_filters;
  int32_t filter_kind[4];
  double filter_param[4][3];
  uint32_t* filter_mask_out;    // [R][mask_words] or null: the candidate set after the filter chain
  int32_t only_deferred;        // full-matrix kernel: score only the requests the sparse kernel marked pick == kPickDeferred
  int32_t pdl;                  // launch the pick kernels with programmatic dependent launch (they follow the hash kernels)
  int32_t stage_terms;          // full-matrix / generic dense kernels: the term and min/max arrays sit in shared memory (set by
                                // their launchers; 0: they did not fit, the kernel reads them from global memory)
};
constexpr int32_t kPickDeferred = -2;

struct HashArgs {
  int32_t R;
  const uint8_t* bytes;
  const int64_t* off;       // [R+1]
  const int32_t* len;       // [R] or null
  const uint64_t* seed;     // [R] or null (=> 0)
  int32_t block_chars;
  int32_t max_blocks;
  uint64_t* hashes;         // [R][stride]
  int32_t stride;
  uint16_t* n_hashes;       // [R]
  int32_t pdl;              // launch the chain kernel with programmatic dependent launch
  int32_t stage_mask;       // diagnostics: eppscore_set_debug key 2 (include/eppscore.h); 0 = the default form
  // probe the prefix index too (hash_probe_applies): one record per request; the rows it resolves never reach `hashes`
  const TableView* table;
  ProbeRec* probe;          // [R] or null
  unsigned long long* resolved;  // with probe: += the requests resolved (one atomic per warp tile)
};

struct PrepareArgs {
  Geo geo;
  int32_t n_scorers;
  int32_t kind[kMaxSteps];
  double weight[kMaxSteps];
  // raw snapshot (device)
  const double* kv;
  const int64_t* queue;
  const int64_t* running;
  const uint64_t* act;
  const uint64_t* wait;
  const int32_t* nmodels;
  const int32_t* maxm;
  const double* col[4];
  const int64_t* tokens;        // InFlightLoad.Tokens or null
  const uint32_t* member;       // [Mpad/32] natural-order bits of the profile's endpoint subset, or null: every endpoint
  double token_threshold;
  int32_t lora_words;
  int32_t A;
  // latency fold-in inputs (null lat_ep: not configured)
  const double* min_tpot;
  const int32_t* dispatched;
  const uint8_t* prefill;
  double lat_coef[8];           // ttft {intercept, kv, waiting, running}, tpot {intercept, kv, waiting, running}
  double lat_buffer, lat_ckv;
  int32_t lat_streaming;
  QBucketHdr* qhdr[2];          // value buckets for the masked min/max (null: scorer not in the profile)
  uint32_t* qbucket[2];
  int32_t lat_has_predictions;
  double* lat_ep;               // [Mpad/32][kLatArrays][32] tiles
  // outputs of the endpoint kernel
  double* term[kMaxSteps];      // per scorer (null where not an endpoint term)
  double* fold_unmasked;        // leading run folded (or null)
  int32_t fold_unmasked_n;
  double* fold_masked;
  int32_t fold_masked_n;
  // outputs of the adapter kernel
  uint32_t* cls_lo;
  uint32_t* cls_hi;
  Plan plan_u;                  // the unmasked plan (evaluated with zero prefix match for the summaries)
  const double* plan_term[kMaxSteps];
  AdapterSummary* summ;         // null unless plan_u.sparse_ok
  uint32_t* tiemask;
};

// launchers. Each returns the number of kernels it launched (for gpu_launches); the scoring launchers return -(cudaError_t)
// when a launch failed.
int launch_hash_prompts(const HashArgs& a, cudaStream_t s, int sm_count);
bool hash_probe_applies(const HashArgs& a);   // launch_hash_prompts can probe the index for this batch (a.probe)
int launch_prepare_snapshot(const PrepareArgs& a, cudaStream_t s);
int launch_count_fields(const uint8_t* bytes, const int64_t* off, const int32_t* len, int R, int32_t* out, cudaStream_t s,
                        int sm_count);  // len(strings.Fields(prompt)) per request
int launch_score_pick(const ScoreArgs& a, bool dense, cudaStream_t s, int sm_count);   // generic (any plan, masks, diagnostics)
int launch_score_matrix(const ScoreArgs& a, cudaStream_t s, int sm_count);             // every pair scored (masks, diagnostics)
int launch_score_dense_fast(const ScoreArgs& a, cudaStream_t s, int sm_count);         // 0 if no specialisation applies
int launch_pick_sparse(const ScoreArgs& a, cudaStream_t s, int sm_count);              // 0 if not applicable
bool pick_sparse_probes(const ScoreArgs& a);  // launch_pick_sparse takes the batch and probes the index for it (plan, outputs and geometry set; table and hashes are not looked at)
bool pick_sparse_applies(const ScoreArgs& a);  // launch_pick_sparse takes the batch (same inputs)
// With a.member set, launch_pick_sparse leaves the requests it deferred (pick == kPickDeferred) to the caller, which scores them
// with the masked full-matrix kernel on the rows launch_subset_mask writes for them.
// Candidate rows for the masked kernels on a profile with an endpoint subset: out[r] = member & cand_mask[r] (member alone
// without cand_mask), [R][mask_words] natural order.  only_pick: only the rows whose pick is kPickDeferred are written.
int launch_subset_mask(const uint32_t* member, const uint32_t* cand_mask, int R, int mask_words, const int32_t* only_pick,
                       uint32_t* out, cudaStream_t s, int sm_count);

// top-k lists of any length from weighted score rows (topk_select.cu): row r of `scores` ([R][M], NaN = not a candidate) is
// request request_base + r; the first k entries of its pick order (device_common.cuh topk_key) go to out_m / out_s [R][k]
struct TopKSelectArgs {
  const double* scores;
  int32_t R, M, k;
  int32_t pick_mode, tie_mode;
  uint32_t seed_lo, seed_hi;
  int64_t request_base;
  int32_t* out_m;
  double* out_s;
};
int launch_topk_select(const TopKSelectArgs& a, cudaStream_t s);  // M <= 8192
// in-flight load producer (inflight_kernel.cu): requests[m] += sign * #{r : endpoint[r] == m}, token_sum[m] += sign * Σ tokens[r];
// endpoint < 0 is skipped, endpoint >= n_ep (<= 8192) is skipped and sets *err.  init_* opts the kernel into the 16 bytes of
// shared memory per endpoint it needs (once per device).
cudaError_t init_inflight_update();
int launch_inflight_update(const int32_t* endpoint, const int64_t* tokens, int R, int n_ep, int sign, int64_t* requests,
                           int64_t* token_sum, uint32_t* err, cudaStream_t s);
int launch_estimate_tokens(const int64_t* size, const int32_t* hint, const int32_t* chars, int R, int64_t* out, cudaStream_t s);

// a batch in arrival order against the in-flight counters (inorder_kernel.cu, eppscore_schedule_batch_inorder): profile 0's
// scorers in profile order, one request at a time; the owner of each pick adds the request's tokens to the counters
struct InOrderArgs {
  int32_t M, Mpad, log_epl, RW, A, mask_words;
  int32_t n_scorers;
  int32_t kind[kMaxSteps];             // eppscore_scorer_kind (the latency scorer only in the walk's latency form)
  double weight[kMaxSteps];
  double lora_term[kMaxSteps][4];      // per LoRA scorer: clamp({0,0.6,0.8,1.0})*w, as Plan::lora_term
  const double* term[kMaxSteps];       // the prepared [Mpad] terms of the kv-cache and endpoint-column scorers, else null
  int32_t pick_mode, tie_mode;
  uint32_t seed_lo, seed_hi;
  int64_t request_base;
  double token_threshold;
  int32_t R;
  const uint16_t* match;               // [R][M] match counts (the batch kernels' match_out) or null
  const uint16_t* total;               // [R] or null
  long long* minmax;                   // [R][4]: queue min, max, running min, max over the candidates (or null: no such scorer
                                       // and no latency scorer without predictions)
  const int32_t* adapter_id;           // [R] or null
  const uint32_t* cand_mask;           // [R][mask_words] natural order or null
  const uint32_t* member;              // [Mpad/32] natural-order bits of profile 0's endpoint subset, or null
  const int64_t* queue;
  const int64_t* running;
  const uint32_t* cls_lo;              // LoRA class planes, permuted, [A+1][RW]
  const uint32_t* cls_hi;
  const int64_t* tokens;               // [R] or null (0 tokens)
  int64_t* inflight_req;               // [Mpad] counters, read at the start and written back at the end
  int64_t* inflight_tok;
  int32_t* pick;
  double* pick_score;
  int32_t* tie_count;
};
int launch_inorder_minmax(const InOrderArgs& a, cudaStream_t s, int sm_count);  // fills a.minmax
struct RunDev;
// The latency scorer in the walk (eppscore_schedule_batch_inorder_latency): the snapshot's fold-in (its tiles and scalars, the
// slice's input_tokens / ttft_slo / tpot_slo) and the running-request queues, which the owner of each pick adds request r to.
struct InOrderLatArgs {
  LatArgs lat;
  RunDev* run;                    // the device descriptor of the queues (kernels.cuh: RunDev)
  const uint64_t* request_key;    // [R] or null: the queues are read (from the tiles), never changed
  uint8_t* added_out;             // [R] or null
  int32_t n_ep;                   // max_endpoints: the length of the queues' per-endpoint arrays
};
// CTAs per cluster of inorder_pick_kernel (lat: inorder_pick_lat_kernel) at this Mpad on the current device (sets the kernels'
// cluster attribute): > 0, 0 when no cluster shape fits, or -(cudaError_t)
int inorder_cluster_size(int Mpad, bool lat = false);
// one cluster of C CTAs; lt non-null: the latency form (inorder_pick_lat_kernel)
int launch_inorder_pick(const InOrderArgs& a, int C, cudaStream_t s, const InOrderLatArgs* lt = nullptr);
// The walk in index order (eppscore_schedule_batch_inorder_index): request r's match counts are read from the index as it
// stands after requests 0..r-1's commits, and the CTA that owns r's pick commits r's blocks (IndexProgram::commit) before
// request r + 1 probes.  a.match is unused; a.total holds n_hashes.
struct InOrderIndexArgs {
  TableView* tv;
  LruView* lv;
  const uint64_t* hashes;   // [R][stride]
  int32_t stride;
  const int32_t* cap_req;   // [n_endpoints] CacheNumBlocks or null
  uint16_t* pick_match;     // [R] the pick's match count as the request was scored, or null
};
int inorder_index_cluster_size(int Mpad, bool lat = false);  // as inorder_cluster_size, for launch_inorder_index's CTAs of kCommitThreads
int launch_inorder_index(const InOrderArgs& a, const InOrderIndexArgs& ix, int C, cudaStream_t s, const InOrderLatArgs* lt = nullptr);
// Several profiles in the walk (eppscore_schedule_batch_inorder_profiles): per run, what InOrderArgs holds for profile 0, read
// by every thread for its endpoint each request.  The InOrderArgs of the launch carry the request- and engine-wide fields (its
// per-profile fields are unused).
struct InOrderRun {
  int32_t n_scorers;
  int32_t term_base;                   // the run's first term slot in the walk's shared-memory staging (Σ earlier n_scorers)
  int32_t kind[kMaxSteps];
  double weight[kMaxSteps];
  double lora_term[kMaxSteps][4];
  const double* term[kMaxSteps];
  int32_t pick_mode;
  uint32_t seed_lo, seed_hi;           // the profile's derived tie seed
  const uint32_t* cand_mask;           // [R][mask_words] or null
  const uint32_t* member;              // the profile's endpoint subset, or null
  const long long* minmax;             // [R][4] over the run's candidates, or null
  int32_t* pick;
  double* pick_score;
  int32_t* tie_count;
  uint16_t* pick_match;                // [R] or null
};
constexpr int kMaxRuns = 4;  // EPPSCORE_MAX_PROFILES
struct InOrderProfArgs {
  int32_t n_runs, primary, prefill;    // prefill -1: no second Add
  const uint8_t* run_mask;             // [R] bit i: run i runs for request r, or null (every run)
  InOrderRun run[kMaxRuns];
};
// Dynamic shared memory of the profiles walk with `slots` term slots (Σ n_scorers); the device's opt-in limit bounds it.
size_t inorder_profiles_smem(int Mpad, int C, bool index, int slots);
// CTAs per cluster of the profiles walk of either form, as inorder_cluster_size / inorder_index_cluster_size
int inorder_profiles_cluster_size(int Mpad, bool index, size_t* smem_max);
int launch_inorder_profiles(const InOrderArgs& a, const InOrderIndexArgs* ix, const InOrderProfArgs& p, int C, int slots, cudaStream_t s);

// predicted-latency producer's running-request queues (running_kernel.cu).  Table slot: {key, meta}, meta = endpoint + 1
// (| kRunTomb once removed), {0, 0} empty; tpot[] holds the entry's tpot bits, owner[] / rm[] the (gen << 32 | r) bids of
// an add / remove call (~0 when none).  Per endpoint: count, min_bits (kRunMinNone when empty), min_cnt = live entries
// equal to min_bits, min_view = what the scorer reads (the minimum as a double, 0 when empty).
struct __align__(16) RunSlot {
  unsigned long long key, meta;
};
constexpr unsigned long long kRunTomb = 1ull << 32;
constexpr unsigned long long kRunMinNone = ~0ull;
constexpr unsigned kRunErrInvalid = 1u, kRunErrCapacity = 2u;
struct RunCounters {
  unsigned long long live, tomb;  // live entries, tombstones
  unsigned gen, any_dirty, err, pad;
};
struct RunDev {
  RunSlot* slot;
  unsigned long long *tpot, *owner, *rm;
  unsigned long long mask;  // capacity - 1 (a power of two)
  int* count;
  unsigned long long* min_bits;
  int* min_cnt;
  double* min_view;
  unsigned* dirty;
  unsigned long long* rc_min;  // recompute scratch: kRunMinNone / 0 between calls
  int* rc_cnt;
  RunCounters* ctr;
  RunSlot* spare_slot;  // a second table of the same capacity: the target of the device-side compaction
  unsigned long long *spare_tpot, *spare_owner, *spare_rm;
  int32_t* slot_of;  // per-call scratch, [scratch capacity]
  uint8_t* won;
};
cudaError_t init_running_kernels();
// The kernels of a call read the table through the DEVICE-resident descriptor `dp` (so captured graphs follow a table that
// grows or compacts later); `cap` only sizes the grid-stride passes.  op 0 = add (tpot may be NULL: 0), op 1 = remove;
// out: optional [R] added / removed flags.
int launch_running_update(RunDev* dp, unsigned long long cap, int op, const int32_t* endpoint, const uint64_t* key,
                          const double* tpot, int R, int n_ep, uint8_t* out, int sm_count, cudaStream_t s);
// The pre-add compaction alone (the first three launches of an add), and the end of every call (the view and the generation):
// for a caller that adds through its own kernel (the in-order walk's Add at each pick).
int launch_running_compact(RunDev* dp, unsigned long long cap, int R, int sm_count, cudaStream_t s);
int launch_running_finalize(RunDev* dp, int n_ep, cudaStream_t s);
int launch_running_drop_endpoint(RunDev* dp, unsigned long long cap, int m, int n_ep, int sm_count, cudaStream_t s);
int launch_running_rebuild(const RunDev& src, const RunDev& dst, int sm_count, cudaStream_t s);

}  // namespace eppscore
