/*
 * eppscore.h — C ABI of the H100-native batched Endpoint-Picker scoring engine (libeppscore.so).
 *
 * This is the drop-in boundary for ONE hot path of kubernetes-sigs/gateway-api-inference-extension
 * (reference @ c4c8fef; paths below are relative to it): the per-request Filter → Score → Pick
 * loop behind Scheduler.Schedule() plus the approximate-prefix producer that feeds it, executed
 * for a BATCH of R requests against M endpoints by hand-written sm_90a CUDA kernels.
 *
 * The reference has no FFI today (pure Go, CGO_ENABLED=0, Dockerfile:8); these entry points are
 * exactly what a cgo shim behind requestcontrol.Scheduler (pkg/epp/requestcontrol/director.go:68-70)
 * would bind.  INTEGRATION.md shows that shim.  Conventions:
 *   - plain C types, caller-owned contiguous little-endian arrays, no callbacks, no torch types;
 *   - every function returns int32 status (EPPSCORE_OK == 0, negative = error) and
 *     eppscore_last_error() gives the message; handles are opaque;
 *   - one engine per CUDA device; calls on one engine are serialised by the caller
 *     (the Go shim holds a mutex), different engines are independent;
 *   - there is NO CPU fallback: eppscore_create fails (EPPSCORE_ERR_NO_DEVICE) without a GPU.
 *
 * Numerics contract (SURVEY.md §8): all scheduler arithmetic is IEEE float64, multiply then add
 * without FMA contraction, accumulated in scorer order from 0.0 — bit-identical to
 * pkg/epp/scheduling/scheduler_profile.go:155-168 on GOARCH=amd64.  Block hashes are XXH64
 * (seed 0) chained as approximateprefix/hashing.go:70-94.  Picks are the arg-max; ties are
 * reported (tie_count) and broken deterministically (see eppscore_tie_mode) where the reference
 * breaks them with a time-seeded shuffle (picker/common.go:49-55, maxscore/picker.go:91-102).
 */
#ifndef EPPSCORE_H
#define EPPSCORE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EPPSCORE_ABI_VERSION 3
#define EPPSCORE_MAX_SCORERS 8
#define EPPSCORE_MAX_ENDPOINT_COLS 4
#define EPPSCORE_MAX_BLOCKS 65535 /* match/total are uint16 (attribute/prefix/data_types.go:27-34 are Go ints) */

typedef struct eppscore_engine eppscore_engine; /* opaque */

typedef enum eppscore_status {
  EPPSCORE_OK = 0,
  EPPSCORE_ERR_INVALID = -1,     /* bad argument / config */
  EPPSCORE_ERR_CUDA = -2,        /* CUDA runtime error (message in last_error) */
  EPPSCORE_ERR_CAPACITY = -3,    /* M / A / table capacity exceeded */
  EPPSCORE_ERR_NO_SNAPSHOT = -4, /* schedule called before set_snapshot */
  EPPSCORE_ERR_NO_DEVICE = -5    /* no CUDA device: the engine has no CPU path */
} eppscore_status;

/* Scorer kinds, in the sense of framework.Scorer (interface/scheduling/plugins.go:68-72). */
typedef enum eppscore_scorer_kind {
  EPPSCORE_SCORER_QUEUE = 0,    /* queue-scorer: scorer/queuedepth/queue.go:78-108 */
  EPPSCORE_SCORER_KV_CACHE = 1, /* kv-cache-utilization-scorer: scorer/kvcacheutilization/kvcache_utilization.go:76-82 */
  EPPSCORE_SCORER_PREFIX = 2,   /* prefix-cache-scorer: scorer/prefix/plugin.go:95-117 (+ producer approximateprefix/) */
  EPPSCORE_SCORER_LORA = 3,     /* lora-affinity-scorer: scorer/loraaffinity/lora_affinity.go:76-102 */
  EPPSCORE_SCORER_RUNNING = 4,  /* running-requests-size-scorer: scorer/runningrequests/runningrequest.go:78-108 */
  /* latency-scorer (scorer/latency/plugin.go:144-318) with the predicted-latency producer folded in: per
   * (request, endpoint) the Bayesian-ridge TTFT/TPOT prediction (sidecars/latencypredictorasync/prediction.go:164-194),
   * headroom/validity (predictedlatency/prediction.go:137-166), then the scorer's tier/bucket logic over the
   * candidate set.  Parameters: eppscore_set_latency_params. */
  EPPSCORE_SCORER_LATENCY = 5,
  EPPSCORE_SCORER_TOKEN_LOAD = 6, /* token-load-scorer: scorer/tokenload/token_load.go:83-111 (snapshot.inflight_tokens) */
  /* 8+k: a host-computed, request-independent scorer supplied as float64 column k of the snapshot
   * (any custom framework.Scorer whose output does not depend on the request); clamped+weighted in-kernel. */
  EPPSCORE_SCORER_ENDPOINT_COL0 = 8,
  /* 16+k: a per-(request,endpoint) float32 column k∈{0,1} of the dense feature rows (any per-pair scorer
   * computed elsewhere, e.g. a tree-ensemble latency model's output). */
  EPPSCORE_SCORER_PAIR_COL0 = 16
} eppscore_scorer_kind;

typedef enum eppscore_tie_mode {
  EPPSCORE_TIE_LOWEST_INDEX = 0, /* deterministic: lowest endpoint index in the arg-max set */
  /* counter-based stand-in for the reference's shuffle: the arg-max member with the largest
   * lowbias32-mixed priority of (tie_seed, request_base + r, endpoint) wins — uniform over the
   * tie set, reproducible, order-independent (so every GPU shard agrees). */
  EPPSCORE_TIE_SEEDED_RANDOM = 1
} eppscore_tie_mode;

/* Pickers (framework.Picker, interface/scheduling/plugins.go:74-78).  The reference's stochastic pickers draw from a
 * process-wide PCG seeded with the wall clock (picker/common.go:40-55), so they have no bit-parity definition; the
 * engine uses a counter-based generator keyed by (tie_seed, request_base + r, endpoint) — reproducible, identical on
 * every shard — and is checked at the distribution level (the reference's own picker tests do the same, ±5 %). */
typedef enum eppscore_pick_mode {
  EPPSCORE_PICK_MAX_SCORE = 0,       /* max-score-picker: picker/maxscore/picker.go:87-115 */
  /* weighted-random-picker (A-Res, picker/weightedrandom/picker.go:111-155): P(m) = score[m] / Σ score over the
   * candidates with score > 0; key U^(1/score) maximal ⇔ -ln(U)/score minimal; no positive score ⇒ random picker.
   * tie_count reports the size of the set the draw was over. */
  EPPSCORE_PICK_WEIGHTED_RANDOM = 1,
  EPPSCORE_PICK_RANDOM = 2           /* random-picker: picker/random/picker.go:85-101 — uniform over the candidates */
} eppscore_pick_mode;

/* Filter plugins evaluated on the device, in order, before the scorers and on top of batch.cand_mask (host-side Filters
 * of any other kind keep reaching the engine as that mask).  Both need the latency scorer in the profile (they read the same
 * per-pair predictions) and cannot be combined with the queue / running scorers.  Their rand.Float64() draws come from the
 * counter-based generator of eppscore_pick_mode: draw of filter f for request r is keyed by (tie_seed, request_base + r, -(f+1)). */
typedef enum eppscore_filter_kind {
  /* prefix-cache-affinity-filter (filter/prefixcacheaffinity/plugin.go:105-151): params {affinityThreshold,
   * explorationProbability, maxTTFTPenaltyMs}; reference defaults 0.80, 0.01, 5000 */
  EPPSCORE_FILTER_PREFIX_AFFINITY = 1,
  /* slo-headroom-tier-filter (filter/sloheadroomtier/plugin.go:82-137): params {epsilonExploreNeg}; default 0.01 */
  EPPSCORE_FILTER_SLO_HEADROOM_TIER = 2
} eppscore_filter_kind;
#define EPPSCORE_MAX_FILTERS 4

/* Scheduler profile + engine sizing.  Replaces SchedulerProfile{scorers, picker}
 * (pkg/epp/scheduling/scheduler_profile.go:41-98) and the approximateprefix config
 * (approximateprefix/types.go:77-141). Zero-initialise, set struct_size = sizeof, fill. */
typedef struct eppscore_config {
  uint32_t struct_size;
  int32_t n_scorers;                              /* profile order matters: float64 adds are not associative */
  int32_t scorer_kind[EPPSCORE_MAX_SCORERS];
  double scorer_weight[EPPSCORE_MAX_SCORERS];     /* WeightedScorer.Weight(), weighted_scorer.go:32 */
  int32_t block_chars;     /* blockSizeTokens*averageCharactersPerToken; default 16*4 (types.go:91,112) */
  int32_t max_blocks;      /* defaultMaxPrefixBlocks = 256 (types.go:98) */
  int32_t tie_mode;        /* eppscore_tie_mode */
  uint64_t tie_seed;
  int32_t max_endpoints;   /* capacity for M (rounded up internally); default 1024 */
  int32_t max_adapters;    /* capacity for the LoRA adapter dictionary A; default 64 */
  int64_t prefix_capacity; /* INITIAL capacity (distinct block hashes) of the device table; it is rebuilt (emptied keys
                              dropped) or doubled on demand. default 1<<18 */
  int32_t lru_capacity_default; /* defaultLRUCapacityPerServer = 31250 (types.go:109) */
  int32_t lru_capacity_max;     /* largest per-endpoint LRU size (CacheNumBlocks, plugin.go:207-216) the engine must support;
                                   0 ⇒ max(lru_capacity_default, the capacities named by the first Add).  It fixes the size of the
                                   per-endpoint device regions; a later Add that names a larger size fails with ERR_CAPACITY. */
  double token_load_threshold;  /* token-load-scorer queueThresholdTokens; <= 0 ⇒ 4194304 (token_load.go:33,57-61) */
  int32_t pick_mode;            /* eppscore_pick_mode; default max-score */
  int32_t n_filters;            /* device-side filters, see eppscore_filter_kind */
  int32_t filter_kind[EPPSCORE_MAX_FILTERS];
  double filter_param[EPPSCORE_MAX_FILTERS][3];
} eppscore_config;

/* ---- scheduler profiles (scheduler.go:54-102: profileHandler.Pick -> profile.Run per picked profile -> ProcessResults) ----
 * An engine serves up to EPPSCORE_MAX_PROFILES profiles over ONE snapshot, one prefix index and one set of producer state.
 * Profile 0 is the one given to eppscore_create; every call that names no profile serves profile 0.  A profile carries the
 * per-profile fields of eppscore_config, validated by the same rules; everything else stays engine-wide: tie mode, block size,
 * capacities, token-load threshold, and the latency parameters (the predicted-latency producer is one per engine, so every
 * profile with a latency scorer reads the same eppscore_set_latency_params).
 * The stochastic pickers and the seeded-random tie break of profile p draw with tie_seed ^ (p * 0x9E3779B97F4A7C15) (unsigned
 * 64-bit product), so two profiles do not draw the same numbers; profile 0 draws with tie_seed itself. */
#define EPPSCORE_MAX_PROFILES 4
typedef struct eppscore_profile {
  uint32_t struct_size;
  int32_t n_scorers;
  int32_t scorer_kind[EPPSCORE_MAX_SCORERS];
  double scorer_weight[EPPSCORE_MAX_SCORERS];
  int32_t pick_mode;
  int32_t n_filters;
  int32_t filter_kind[EPPSCORE_MAX_FILTERS];
  double filter_param[EPPSCORE_MAX_FILTERS][3];
} eppscore_profile;

/* One profile's share of eppscore_schedule_batch_profiles: its host-side filter result and its outputs, all [R] (or R x M /
 * R x ceil(M/32) like the eppscore_batch fields of the same name), where the batch's location says. */
typedef struct eppscore_profile_run {
  uint32_t struct_size;
  int32_t profile;             /* id from eppscore_add_profile, 0 = the create profile */
  const uint32_t *cand_mask;   /* optional [R*ceil(M/32)]: this profile's host Filters; ANDed with its endpoint subset */
  int32_t *pick;               /* [R], -1 = no candidate */
  double *pick_score;          /* [R] */
  int32_t *tie_count;          /* [R] */
  double *scores_out;          /* optional [R*M] */
  double *pred_out;            /* optional [R*M*2] */
  uint32_t *filter_mask_out;   /* optional [R*ceil(M/32)] */
} eppscore_profile_run;

/* Latency fold-in parameters: the cached Bayesian-ridge coefficients (MetricsResponse.Coefficients,
 * sidecars/latencypredictorasync/prediction.go:164-194), the producer's Config (predictedlatency/plugin.go:118-136)
 * and the latency-scorer's Config (scorer/latency/plugin.go:59-90).  Takes effect at the next eppscore_set_snapshot
 * (coefficients are refreshed on the metrics cadence, like the snapshot). */
typedef struct eppscore_latency_params {
  uint32_t struct_size;
  int32_t has_predictions;   /* 0 = no LatencyPredictionInfo (sidecar down / timed out) ⇒ composite fallback (plugin.go:169-172) */
  double ttft_intercept, ttft_kv, ttft_input, ttft_waiting, ttft_running, ttft_prefix;
  double tpot_intercept, tpot_kv, tpot_input, tpot_waiting, tpot_running, tpot_generated;
  double slo_buffer_factor;  /* SLOBufferFactor, default 1 */
  int32_t streaming_mode;    /* StreamingMode, default 0: TPOT neutralised (prediction.go:100-104) */
  int32_t strategy_most;     /* HeadroomSelectionStrategy: 0 "least" (default), 1 "most" */
  double ttft_weight, tpot_weight;                         /* defaults 0.8, 0.2 */
  double composite_kv, composite_queue, composite_prefix;  /* defaults 1, 1, 1 */
} eppscore_latency_params;

/* Immutable metrics snapshot: the fields of fwkdl.Metrics the path reads
 * (interface/datalayer/metrics.go:26-42), packed SoA.  LoRA maps become dictionary bitmasks:
 * bit a of lora_active[m*lora_words + a/64] ⇔ adapter a ∈ ActiveModels of endpoint m. */
typedef struct eppscore_snapshot {
  uint32_t struct_size;
  int32_t M;
  int32_t lora_words;            /* ceil(A/64) */
  int32_t location;              /* 0 = host pointers, 1 = device pointers (e.g. an NCCL-broadcast buffer) */
  const double *kv_usage;        /* KVCacheUsagePercent            [M] */
  const int64_t *queue;          /* WaitingQueueSize               [M] */
  const int64_t *running;        /* RunningRequestsSize            [M] (may be NULL) */
  const uint64_t *lora_active;   /* [M*lora_words] (may be NULL ⇒ empty) */
  const uint64_t *lora_waiting;  /* [M*lora_words] */
  const int32_t *lora_nmodels;   /* len(ActiveModels)+len(WaitingModels) as MAP sizes (lora_affinity.go:90) [M] */
  const int32_t *lora_max;       /* MaxActiveModels                [M] */
  const double *endpoint_col[EPPSCORE_MAX_ENDPOINT_COLS]; /* optional generic score columns [M] */
  uint64_t epoch;                /* caller's snapshot generation, echoed by eppscore_stats */
  void *stream;                  /* cudaStream_t for location==1 (NULL = engine stream) */
  /* predicted-latency producer state per endpoint (all optional, NULL ⇒ 0) */
  const double *min_tpot_slo;    /* getEndpointMinTPOTSLO (predictedlatency/plugin.go:347-355)        [M] */
  const int32_t *dispatched;     /* getEndpointRunningRequestCount (plugin.go:357-363)                [M] */
  const uint8_t *prefill_role;   /* hasPrefillRole(EndpointRoleLabel, endpoint) (prediction.go:168-175) [M] */
  const int64_t *inflight_tokens;/* InFlightLoad.Tokens attribute (token_load.go:91-95); NULL ⇒ the engine's in-flight
                                    counters (eppscore_inflight_add; all 0, i.e. absent, until the first add) [M] */
} eppscore_snapshot;

/* One batch = R concurrent Scheduler.Schedule() calls (pkg/epp/scheduling/scheduler.go:54). */
typedef struct eppscore_batch {
  uint32_t struct_size;
  int32_t R;
  int32_t location;            /* 0 = host pointers (copies happen inside the call), 1 = device pointers */
  int32_t reserved0;
  int64_t request_base;        /* global index of request 0 (multi-GPU shards; feeds the tie priority) */
  /* --- prefix producer inputs: EITHER prompts (hashed on the GPU) OR precomputed hashes --- */
  const uint8_t *prompt_bytes; /* flattened getUserInputBytes() output (hashing.go:106-135), concatenated */
  const int64_t *prompt_off;   /* [R+1] byte offsets into prompt_bytes */
  const int32_t *prompt_len;   /* optional [R]: explicit lengths, so a host may pad every prompt START to 16 bytes
                                  (fast aligned hash path); NULL ⇒ len[r] = prompt_off[r+1]-prompt_off[r] */
  const uint64_t *model_seed;  /* [R] XXH64(TargetModel || cacheSalt) (hashing.go:70-77); see eppscore_model_seed */
  const uint64_t *hashes_in;   /* [R*hash_stride] optional: block hashes computed elsewhere */
  const uint16_t *n_hashes_in; /* [R] */
  int32_t hash_stride;
  int32_t block_chars;         /* 0 ⇒ config default; per call because autotune reads endpoints[0] (plugin.go:238-250) */
  int32_t max_blocks;          /* 0 ⇒ config default */
  int32_t reserved1;
  /* --- per-request scorer inputs --- */
  const int32_t *adapter_id;   /* [R] dictionary id of TargetModel, -1 = not a known adapter; NULL ⇒ all -1 */
  const uint32_t *cand_mask;   /* [R*ceil(M/32)] filter-chain result (scheduler_profile.go:130-149); NULL ⇒ all M */
  /* --- dense feature rows (optional; replaces the in-kernel prefix match and LoRA lookup) ---
   * float4 per (r,m): {x = matchBlocks (integer valued), y = lora class 0..3 ↦ {0,0.6,0.8,1.0},
   *                    z = pair column 0, w = pair column 1}                                        */
  const float *dense_feat;     /* [R*M*4] */
  const uint16_t *dense_total; /* [R] totalBlocks for the dense rows */
  /* --- outputs --- */
  int32_t *pick;               /* [R] chosen endpoint, -1 = "no endpoints available" (scheduler_profile.go:119-121) */
  double *pick_score;          /* [R] weighted score of the pick (ScoredEndpoint.Score, types.go:152-155) */
  int32_t *tie_count;          /* [R] size of the arg-max set */
  uint16_t *match_blocks;      /* optional [R*M]: PrefixCacheMatchInfo.matchBlocks per endpoint */
  uint16_t *total_blocks;      /* optional [R]:   PrefixCacheMatchInfo.totalBlocks */
  uint64_t *hashes_out;        /* optional [R*max_blocks]: block hashes (state for eppscore_commit_picks / PreRequest) */
  double *scores_out;          /* optional [R*M]: the whole weightedScorePerEndpoint map (scheduler_profile.go:155-174),
                                  NaN for non-candidates — diagnostics / parity tests; 8*R*M bytes of HBM writes */
  void *stream;                /* cudaStream_t for location==1 (NULL = engine stream); the call is async on it.  Index
                                * mutations and eppscore_set_snapshot wait for the last device-location batch of every stream.
                                * A stream given its own scratch by eppscore_reserve_stream runs its batches concurrently with
                                * those of other streams, and graphs captured on it stay valid.  Streams without one share
                                * the engine's scratch: keep their device-location batches on ONE stream at a time */
  /* latency fold-in, per request (optional, NULL ⇒ 0) */
  const int32_t *input_tokens; /* [R] len(strings.Fields(prompt)) (predictedlatency/training.go:51); NULL with prompt_bytes given ⇒
                                * counted on the device from those bytes (hosts whose PromptText() differs from the hashed
                                * bytes, e.g. chat completions, pass it explicitly) */
  const double *ttft_slo;      /* [R] x-slo-ttft-ms header value or 0 (predictedlatency/plugin.go:330-343) */
  const double *tpot_slo;      /* [R] x-slo-tpot-ms header value or 0 */
  double *pred_out;            /* optional [R*M*2]: predicted {TTFT, TPOT} per (request, endpoint) — diagnostics */
  uint32_t *filter_mask_out;   /* optional [R*ceil(M/32)]: the candidate set left by the device-side filters — diagnostics */
} eppscore_batch;

/* maxNumOfEndpoints (picker/common.go:39-42): the first k endpoints of each request's pick order, for
 * eppscore_schedule_batch_topk.  Both arrays are [R*k], row r = request r, and live where batch.location says.
 * Entry 0 is pick / pick_score; a request with fewer than k candidates is padded with endpoint -1, score 0.0.
 * The order of each pick mode, on the weighted scores of the candidates:
 *   max-score      score descending; then (TIE_SEEDED_RANDOM) tie priority descending; then endpoint ascending
 *   weighted-random  candidates with score > 0 first, by A-Res key descending, then endpoint ascending; then the
 *                  candidates with score <= 0 (key 0 in weightedrandom/picker.go:126-129), by priority descending, then
 *                  endpoint ascending
 *   random         priority descending, then endpoint ascending
 * i.e. a shuffle inside each tie class (maxscore/picker.go:91-107), sampling without replacement
 * (weightedrandom/picker.go:121-152) and the first k of a shuffle (random/picker.go:90-96), drawn from the counter-based
 * generator of eppscore_pick_mode, so the lists do not depend on how a batch is cut into shards. */
#define EPPSCORE_MAX_TOPK 8
typedef struct eppscore_topk {
  uint32_t struct_size;
  int32_t k;                   /* 1..EPPSCORE_MAX_TOPK (eppscore_schedule_batch_topk_wide: 1..max_endpoints;
                                  eppscore_schedule_batch_profiles_topk: 0..max_endpoints, 0 = no list) */
  int32_t *endpoints;          /* [R*k] */
  double *scores;              /* [R*k] ScoredEndpoint.Score of each entry */
} eppscore_topk;

typedef struct eppscore_stats {
  uint32_t struct_size;
  int32_t M;
  uint64_t epoch;
  uint64_t kernel_launches;     /* CUDA kernels launched by this engine since creation */
  int64_t prefix_hashes;        /* table slots in use, emptied keys included (they are dropped at the next rebuild) */
  int64_t prefix_live_hashes;   /* hashes with a non-empty endpoint set == len(hashToPods) of the reference */
  int64_t prefix_capacity;      /* hashes the table holds at load 0.5 before it is rebuilt / doubled */
  int64_t prefix_table_bytes;   /* device bytes: 32-byte slots + overflow bitset rows */
  int64_t lru_entries;          /* Σ per-endpoint LRU lengths (prefix_indexer_size metric, metrics.go:349) */
  int64_t lru_bytes;            /* device bytes of the per-endpoint LRU regions (maps + logs) */
  int64_t prefix_overflow_rows; /* sets of more than 10 endpoints (bitset rows in use) */
  int64_t prefix_rebuilds;      /* table rebuilds so far */
  uint32_t index_error;         /* sticky device-side error flags of the index (0 = healthy; bit 4: a mutation was skipped
                                   for lack of room, see eppscore_prefix_reserve) */
  uint32_t probe_resolved;      /* requests whose prefix match the hashing kernel settled itself, so the pick kernel skipped
                                   their index probe; since creation, modulo 2^32 (diagnostics: read after the batches finished) */
} eppscore_stats;

/* ---- lifecycle ---- */
int32_t eppscore_abi_version(void);
void eppscore_config_default(eppscore_config *cfg); /* default-config weights queue 2, kv 2, prefix 3 (loader/defaults.go:46-103) */
int32_t eppscore_create(int32_t device, const eppscore_config *cfg, struct eppscore_engine **out);
void eppscore_destroy(struct eppscore_engine *e);
const char *eppscore_last_error(const struct eppscore_engine *e); /* e may be NULL: last create() error */
int32_t eppscore_get_stats(const struct eppscore_engine *e, eppscore_stats *out);
/* Diagnostics knobs (profiling / A-B runs only; never needed for correct operation):
 *   key 1: 1 = always use the fully general kernels (same as env EPPSCORE_FORCE_GENERIC=1), 0 = normal dispatch;
 *   key 2: hash stage mask (0 or 27 = the default: bit 3 the warp-tile fused kernel when the block size is a multiple of
 *          32, else the two-kernel form of bits 0, 1 and 4; 19 = always the two-kernel form: bit 0 run the body kernel,
 *          bit 1 run the chain kernel, bit 4 the CTA-tile chain kernel, without bit 4 the warp-tile chain kernel).  Bit 2
 *          the CTA-tile warp-specialised fused kernel; bit 5 the persistent software-pipelined body kernel;
 *   key 3: requests per chunk of a host-location batch (0: never chunk);
 *   key 4: 0 = ordinary launches, 1 (default) = programmatic dependent launch between the kernels of a batch;
 *   key 5: slices a device-location batch is cut into (default 1), key 6: streams the slices alternate over (default 2;
 *          the caller's stream plus internal ones, joined before the call returns — also inside a CUDA-graph capture).
 *          Each slice's chain and probe kernels are latency bound and pay their full latency per slice.  Batches on a
 *          reserved stream (eppscore_reserve_stream) are never cut. */
int32_t eppscore_set_debug(struct eppscore_engine *e, int32_t key, int64_t value);

/* ---- snapshot (replaces the per-request deep clone, director.go:342-349) ---- */
int32_t eppscore_set_snapshot(struct eppscore_engine *e, const eppscore_snapshot *s);

/* Latency fold-in parameters (see eppscore_latency_params); applied by the next eppscore_set_snapshot. */
void eppscore_latency_params_default(eppscore_latency_params *p);
int32_t eppscore_set_latency_params(struct eppscore_engine *e, const eppscore_latency_params *p);

/* ---- the hot path: Filter(mask) → Score → Pick for R requests ---- */
int32_t eppscore_schedule_batch(struct eppscore_engine *e, const eppscore_batch *b);
/* The same, plus the first t->k endpoints of every request's pick order (see eppscore_topk).  These batches run on the
 * full-matrix kernels.  ERR_INVALID: k outside [1, EPPSCORE_MAX_TOPK], a wrong struct_size or NULL arrays. */
int32_t eppscore_schedule_batch_topk(struct eppscore_engine *e, const eppscore_batch *b, const eppscore_topk *t);
/* The same lists for any k in [1, config.max_endpoints] (maxNumOfEndpoints has no upper bound in the reference), in the
 * order documented above eppscore_topk, on the device for every pick mode.  pick, pick_score and tie_count are those of
 * eppscore_schedule_batch, entry 0 is the pick, short lists are padded with -1 / 0.0, and for k <= EPPSCORE_MAX_TOPK the lists
 * equal eppscore_schedule_batch_topk's bit for bit.  It accepts the batches eppscore_schedule_batch_topk accepts and refuses
 * the others with the same status.  Per slice of requests, the batch's scores_out route writes the weighted scores into an
 * engine-owned scratch (a fixed byte budget of rows: its size depends on max_endpoints only), and a selection kernel orders
 * each row.  The scratch is allocated by the first wide call and never reallocated: a wide call inside a CUDA-graph capture
 * before any wide call outside one fails with ERR_CAPACITY.  A caller that passes scores_out gets the rows there and no
 * scratch is used.  The slices of a device-location batch run in order on its stream (debug keys 5 / 6 do not cut it).
 * ERR_INVALID: k outside [1, max_endpoints], a wrong struct_size or NULL arrays. */
int32_t eppscore_schedule_batch_topk_wide(struct eppscore_engine *e, const eppscore_batch *b, const eppscore_topk *t);

/* A batch in arrival order against the in-flight load: the outputs (pick, pick_score, tie_count, total_blocks, hashes_out) and
 * the in-flight counters afterwards equal, bit for bit, what this loop gives:
 *     for r in 0 .. R-1:
 *         eppscore_schedule_batch(request r alone, request_base = b->request_base + r)
 *         eppscore_inflight_add(1, &pick[r], &tokens[r])
 * so request r's token-load scorer sees the load requests 0..r-1 were sent with, as R consecutive Schedule + PreRequest calls
 * of the reference do (inflightload/producer.go:101-120, token_load.go:83-111), instead of one load view for the whole batch.
 * tokens: [R] where b->location says (usually eppscore_estimate_tokens' output); NULL = 0 tokens.  A request with pick -1 adds
 * nothing; both the requests and the tokens counters are updated.  Only the token-load terms move from one request to the next:
 * the queue / running min / max are over each request's own candidates, as in eppscore_schedule_batch.
 * Scope: profile 0, any scorer set without the latency scorer, cand_mask, hashes_in or prompt bytes, every pick and tie mode.
 * Locations and ordering: host arrays are staged and the call returns when done; device arrays run asynchronously on b->stream
 * (reserved streams use their own scratch).  The call is a batch and a producer update: it waits for pending device batches
 * and earlier producer updates as eppscore_inflight_add does, is registered as a pending batch, and ends by preparing the
 * snapshot terms again from the new counters, so a following eppscore_schedule_batch sees what it would see after the loop.
 * It can be captured into a CUDA graph once one call on the same stream (the engine stream for host arrays) has run outside a
 * capture: that call allocates a fixed slice scratch, and a first call under capture fails with ERR_CAPACITY.
 * Per slice of rows the batch kernels compute the prefix match (what does not depend on the load), then one thread-block
 * cluster walks the requests in order with the counters in its registers and reduces each request's pick across its CTAs.
 * Known cost: that pre-pass is the ordinary batch with its R x M match_blocks route (2 bytes per pair written and read back;
 * its provisional picks are overwritten), which a match-only pre-pass could avoid; today the in-order walk dominates.  The
 * cluster shape is decided by the engine's first call, before anything is launched: ERR_CAPACITY when no cluster of the device
 * holds max_endpoints endpoints (8192 needs the non-portable cluster size 16).
 * Not ordered: the prefix index (request r+1 does not see the blocks request r adds; commit after the call, or use
 * eppscore_schedule_batch_inorder_index), the latency scorer's running queues (use eppscore_schedule_batch_inorder_latency),
 * top-k lists, several profiles (eppscore_schedule_batch_inorder_profiles), and requests on other GPU shards (each engine orders
 * its own batch).
 * ERR_INVALID before anything is launched: a profile 0 with the latency scorer, a current snapshot that supplies
 * inflight_tokens, dense_feat / scores_out / match_blocks / pred_out / filter_mask_out set, and what eppscore_schedule_batch
 * refuses.  ERR_NO_SNAPSHOT before eppscore_set_snapshot. */
int32_t eppscore_schedule_batch_inorder(struct eppscore_engine *e, const eppscore_batch *b, const int64_t *tokens);

/* The index side of eppscore_schedule_batch_inorder_index. */
typedef struct eppscore_inorder_index {
  int32_t struct_size;          /* sizeof(eppscore_inorder_index) */
  const int32_t *lru_capacity;  /* HOST [M] CacheNumBlocks per endpoint (autotune), NULL/<=0 = default; NULL under capture */
  uint16_t *pick_match;         /* optional [R], where b->location says: matchBlocks of pick[r] as request r was scored */
} eppscore_inorder_index;

/* A batch in arrival order against the in-flight load AND the prefix index: the outputs (pick, pick_score, tie_count,
 * total_blocks, hashes_out, x->pick_match), the in-flight counters and the whole prefix index afterwards (every LRU's keys oldest
 * -> newest, every set, len(hashToPods)) equal, bit for bit, what this loop gives:
 *     for r in 0 .. R-1:
 *         eppscore_schedule_batch(request r alone, request_base = b->request_base + r, hashes_out)
 *         pick_match[r] = eppscore_prefix_match(request r's hashes, at pick[r])     (before its own Add)
 *         eppscore_inflight_add(1, &pick[r], &tokens[r])
 *         eppscore_commit_picks(1, &pick[r], hashes[r], n_hashes[r], x->lru_capacity)
 * so request r's prefix scorer sees the blocks requests 0..r-1 were sent with, as R consecutive Schedule + PreRequest calls of
 * the reference do (approximateprefix/plugin.go:169-204): a window of requests sharing a new prefix follows the first of them.
 * pick_match is PrefixCacheMatchInfo.matchBlocks at the target as the reference records it; an eppscore_prefix_match after the
 * call would see the batch's own Adds.  A request with pick -1 adds nothing anywhere.
 * Scope, validation, the cluster-shape decision and the first-call-outside-capture rule are those of
 * eppscore_schedule_batch_inorder (the walk runs in CTAs of 512 threads, one endpoint per thread).  The call is also an index
 * mutation, waited for and ordered like eppscore_commit_picks_device: it reports an earlier skipped mutation (ERR_CAPACITY), it
 * refuses an unreserved index and a non-NULL lru_capacity under capture, and it ensures the LRU regions before anything is
 * launched.  Device arrays run on b->stream; later readers and index mutations on other streams are ordered after it.
 * Room is decided once per slice of rows (the slices of eppscore_schedule_batch_inorder), before that slice's walk, for the
 * slice's sum of n_hashes.  An unreserved index grows on the host as a commit does (a synchronous read of the sum).  On a reserved
 * index the decision runs on the device and may rebuild in place; a slice that finds no room is walked WITHOUT commits, all or
 * nothing as a commit is: its outputs equal eppscore_schedule_batch_inorder's on the frozen index, the index stays
 * bit-identical, stats.index_error bit 4 and the skip counter are set, and the next index call reports it.
 * Per slice: the hash stage (no R x M match route), the candidates' min / max, the room, then one thread-block cluster walks the
 * requests in order: each request's blocks are probed up to the first miss, every endpoint's thread counts the hit blocks whose
 * set holds it, the request is scored and picked as in eppscore_schedule_batch_inorder, and the CTA that owns the pick runs the
 * index's commit program for that one Add before the cluster barrier that the next request's probes wait for.
 * Not covered: several picks per request and several profiles (eppscore_schedule_batch_inorder_profiles), top-k lists, the
 * latency scorer's running queues (eppscore_schedule_batch_inorder_latency with x), and replication across GPU shards (each engine commits its own batch inside the call; replaying an
 * all-gathered commit stream on top would apply its commits twice, so sharding.gather_commit_stream belongs to the
 * batch-wide path).  ERR_INVALID: x NULL or a wrong struct_size, and what eppscore_schedule_batch_inorder refuses. */
int32_t eppscore_schedule_batch_inorder_index(struct eppscore_engine *e, const eppscore_batch *b, const int64_t *tokens,
                                              const eppscore_inorder_index *x);

/* The running-request side of eppscore_schedule_batch_inorder_latency. */
typedef struct eppscore_inorder_running {
  int32_t struct_size;          /* sizeof(eppscore_inorder_running) */
  const uint64_t *request_key;  /* [R] where b->location says; NULL: the queues are read, never changed */
  uint8_t *added_out;           /* optional [R]: 1 where request r was added to pick[r]'s queue */
} eppscore_inorder_running;

/* A batch in arrival order with profile 0's latency scorer ordered too: request r's latency scorer sees the running-request
 * queues after requests 0..r-1 were added to them, and each request is added to its pick's queue inside the call.  The outputs
 * (pick, pick_score, tie_count, total_blocks, hashes_out, q->added_out, and x->pick_match in the index form), the in-flight
 * counters, the running-request view (eppscore_running_get) and, in the index form, the whole prefix index afterwards equal,
 * bit for bit, what this loop gives:
 *     for r in 0 .. R-1:
 *         eppscore_schedule_batch(request r alone, request_base = b->request_base + r)
 *         [x: pick_match[r] = eppscore_prefix_match(request r's hashes, at pick[r])]
 *         added_out[r] = eppscore_running_add(1, &pick[r], &request_key[r], &b->tpot_slo[r])
 *         eppscore_inflight_add(1, &pick[r], &tokens[r])
 *         [x: eppscore_commit_picks(1, &pick[r], hashes[r], n_hashes[r], x->lru_capacity)]
 * PreRequest adds the request to its target's queue (predictedlatency/requestcontrol_hooks.go:73-86) and the next Schedule reads
 * the queue's count (the idle preference, scorer/latency/plugin.go:189-202) and minimum TPOT SLO (the TPOT bound,
 * prediction.go:149-161): a batch-wide call gives every request of the batch the same view, so in an overloaded fleet every
 * request picks the same idle endpoint, and a tight TPOT SLO does not tighten its target for the requests after it.
 * Each request reads b->tpot_slo (the value queued), b->ttft_slo and b->input_tokens (counted from the prompt bytes when absent).
 * An add is refused (added_out[r] = 0) as eppscore_running_add refuses it: no pick, key 0, tpot < 0, or an (endpoint, key) pair
 * already live, before the call or from an earlier request of the batch.  x NULL: the in-flight form
 * (eppscore_schedule_batch_inorder's walk); x set: the index form (eppscore_schedule_batch_inorder_index's walk, with its index
 * ordering, room and capture rules).  The call is a running-queue mutation too, ordered like eppscore_running_add: room for R adds
 * is made once per call before the walk (under CUDA-graph capture it needs eppscore_running_reserve, and in the index form
 * eppscore_prefix_reserve), and the snapshot terms are prepared again behind it.  Per request the walk reduces the lowest tier
 * and its headroom ranges across the cluster (with predictions, one more cluster barrier than the walk without it); each thread
 * keeps its endpoint's running count and minimum in registers, and the owner of the pick runs the Add.
 * ERR_INVALID before anything is launched: q NULL or a wrong struct_size, a profile 0 without the latency scorer or with device
 * filters, request_key set while the current snapshot supplies min_tpot_slo or dispatched, a NaN tpot_slo in host arrays with
 * request_key set, a snapshot prepared without latency params, and what the call's form refuses apart from the latency scorer. */
int32_t eppscore_schedule_batch_inorder_latency(struct eppscore_engine *e, const eppscore_batch *b, const int64_t *tokens,
                                                const eppscore_inorder_index *x, const eppscore_inorder_running *q);

/* ---- several scheduler profiles (see eppscore_profile) ---- */
/* Adds a profile; *id_out receives its id (1, 2, ...).  With a snapshot present the profile is prepared for it at once, on the
 * engine stream (a profile with a latency scorer on an engine that had none is usable from the next eppscore_set_snapshot).
 * ERR_CAPACITY past EPPSCORE_MAX_PROFILES, ERR_INVALID for a bad profile or under CUDA-graph capture. */
int32_t eppscore_add_profile(struct eppscore_engine *e, const eppscore_profile *p, int32_t *id_out);
/* A request-independent Filter at the head of the profile's filter chain (e.g. the prefill / decode role label): mask is a host
 * bitmask over endpoint rows in natural order, `words` 32-bit words (bits past max_endpoints ignored, missing words are 0);
 * NULL = every endpoint (the default).  Takes effect at the next eppscore_set_snapshot, like eppscore_set_latency_params.  A
 * request's candidates are then subset ∧ cand_mask ∧ the device filters; the queue / running min/max run over those
 * candidates (queue.go:79-91); an empty candidate set gives pick -1.  On profile 0 it applies to eppscore_schedule_batch and
 * its top-k forms as well.  Batches without a cand_mask stay on the sparse path; every other route scores the profile through
 * the masked kernels on rows subset ∧ cand_mask built on the device.  ERR_INVALID under CUDA-graph capture.  The call first
 * waits for the last eppscore_set_snapshot made outside a capture to finish copying the previous subset.
 * A set_snapshot captured into a CUDA graph while the profile had a subset copies the subset as it stands when the graph is
 * REPLAYED, not when it was captured: the call may follow such a capture (it does not wait for the graph), and NULL then makes
 * the next replay see every endpoint.  A profile captured without a subset stays without one in that graph; a subset set
 * later applies from the next set_snapshot outside it.  Do not replay such a graph while this call runs. */
int32_t eppscore_set_profile_endpoints(struct eppscore_engine *e, int32_t profile, const uint32_t *mask, int32_t words);
/* Schedule.Run of several profiles for one batch: the prompts are hashed (and the prefix index probed) ONCE, then each run's
 * Filter -> Score -> Pick follows on the same stream.  b carries the request inputs and the profile-independent outputs
 * (total_blocks, match_blocks, hashes_out); its pick / pick_score / tie_count / cand_mask / scores_out / pred_out /
 * filter_mask_out must be NULL.  1 <= n_runs <= EPPSCORE_MAX_PROFILES, each profile at most once.  Locations, chunking,
 * request_base shards, device-batch ordering and CUDA-graph capture behave as in eppscore_schedule_batch.  Top-k lists
 * (maxNumOfEndpoints > 1) come from eppscore_schedule_batch_profiles_topk.  ERR_INVALID otherwise. */
int32_t eppscore_schedule_batch_profiles(struct eppscore_engine *e, const eppscore_batch *b, int32_t n_runs,
                                         const eppscore_profile_run *runs);
/* eppscore_schedule_batch_profiles plus, per run, the first topk[i].k endpoints of that run's pick order (maxNumOfEndpoints is
 * per profile in the reference: picker/common.go:36-42).  topk: [n_runs], one entry per run, in run order; k == 0 (endpoints /
 * scores may be NULL) = no list for that run.  k in [0, config.max_endpoints].
 *   - Run i's list equals, bit for bit, the list eppscore_schedule_batch_topk (k <= EPPSCORE_MAX_TOPK) or
 *     eppscore_schedule_batch_topk_wide (any k) returns on an engine whose profile 0 has that profile's scorers, picker,
 *     filters and endpoint subset, and tie_seed ^ (p * 0x9E3779B97F4A7C15) as its tie_seed: the order of each pick mode
 *     documented above eppscore_topk, entry 0 the run's pick, short lists padded with -1 / 0.0.
 *   - pick, pick_score and tie_count of every run are those of eppscore_schedule_batch_profiles, with or without lists.  A run
 *     with k <= EPPSCORE_MAX_TOPK takes the full-matrix kernels' register lists; a run with k == 0 keeps its route (a run
 *     without a list can stay on the sparse path next to a listed run).  A call with k == 0 on every run is
 *     eppscore_schedule_batch_profiles.
 *   - Runs with k > EPPSCORE_MAX_TOPK share the score scratch of eppscore_schedule_batch_topk_wide, which keeps its size: with n
 *     such runs a slice holds 1/n of its rows per run, the prompts are still hashed once per slice, and a run that passes its
 *     own scores_out uses that instead.  Such a run inside a CUDA-graph capture before any wide call outside one fails with
 *     ERR_CAPACITY.  Wide batches on device buffers run their slices in order on the batch's stream (keys 5 / 6 do not cut
 *     them); the other device batches are sliced as eppscore_schedule_batch_profiles slices them.
 * Locations, chunking, request_base, device-batch ordering and capture behave as in eppscore_schedule_batch_profiles.
 * ERR_INVALID: what eppscore_schedule_batch_profiles refuses, topk NULL, a wrong struct_size, k < 0 or k > max_endpoints, and
 * NULL arrays with k > 0. */
int32_t eppscore_schedule_batch_profiles_topk(struct eppscore_engine *e, const eppscore_batch *b, int32_t n_runs,
                                              const eppscore_profile_run *runs, const eppscore_topk *topk);

/* The arrival-order side of eppscore_schedule_batch_inorder_profiles. */
typedef struct eppscore_inorder_profiles {
  int32_t struct_size;               /* sizeof(eppscore_inorder_profiles) */
  int32_t index;                     /* 0: the in-flight form; 1: also ordered against the prefix index, committing as it goes */
  int32_t primary_run;               /* the run whose pick gates PreRequest and receives the first Add */
  int32_t prefill_run;               /* -1, or the run whose pick receives the second Add (approximateprefix/plugin.go:180-183) */
  const uint8_t *run_mask;           /* optional [R] where b->location says: bit i = run i runs for request r (ProfileHandler.Pick);
                                        NULL = every run for every request */
  const int32_t *lru_capacity;       /* HOST [M] CacheNumBlocks (index form), NULL/<=0 = default; NULL under capture */
  uint16_t *pick_match[EPPSCORE_MAX_PROFILES]; /* optional per run [R]: matchBlocks at that run's pick before request r's Adds */
} eppscore_inorder_profiles;

/* Several profiles in arrival order (prefill/decode disaggregation): every output (each run's pick / pick_score / tie_count and
 * pick_match, total_blocks, hashes_out), the in-flight counters and, in the index form, the whole prefix index afterwards (every
 * LRU oldest -> newest, every set, len(hashToPods)) equal, bit for bit, what this loop gives:
 *     for r in 0 .. R-1:
 *         eppscore_schedule_batch_profiles(request r alone, request_base = b->request_base + r,
 *                                          the runs whose bit is set in run_mask[r]; the others get pick -1)
 *         if pick[primary_run][r] >= 0:                  (the reference runs no PreRequest when scheduling fails)
 *             pick_match[i][r] = eppscore_prefix_match(request r's hashes, at pick[i][r])   for every run i that picked
 *             eppscore_inflight_add(one entry per run that picked, tokens[r] each)         (inflightload/producer.go:106-119)
 *             [index] eppscore_commit_picks_profiles(1, {pick[primary_run][r], pick[prefill_run][r]}, ..., x->lru_capacity)
 * pick_match is 0 where the loop records none.  Every run of request r is scored against what requests 0..r-1 left; none sees
 * request r's own Adds.  Two runs on one endpoint count it twice and Add twice, as the reference does.  Run i draws its
 * stochastic picks and seeded ties with its profile's derived seed, as eppscore_schedule_batch_profiles does.  With one run,
 * primary_run 0 and prefill_run -1 the outputs equal eppscore_schedule_batch_inorder (index 0) or
 * eppscore_schedule_batch_inorder_index (index 1) on that profile.
 * Locations, slicing, the capture rule (one call outside a capture first; in the index form a reserved index), the room per slice
 * (in the index form: the slice's Σ n_hashes once per Add a request can make) and the ordering as a producer update and an
 * index mutation are those of the single-profile in-order calls.  Per slice: the match rows (in-flight form) or the hash stage
 * (index form), each run's candidate min / max where its profile reads them, then one thread-block cluster walks the requests:
 * each thread scores its endpoint once per run, in that run's profile order, and the CTAs publish one winner per run behind the
 * request's one cluster barrier.  The walk stages Σ n_scorers request-independent terms per thread in shared memory (with the
 * index's commit state in the index form): runs that do not fit the device get ERR_CAPACITY before any launch.
 * ERR_INVALID before any launch: x NULL or a wrong struct_size, index outside {0, 1}, what eppscore_schedule_batch_profiles
 * refuses, primary_run or prefill_run out of range or equal, a run with scores_out, pred_out or filter_mask_out, a run whose
 * profile has the latency scorer or device filters, dense_feat or match_blocks set, and a snapshot that supplies
 * inflight_tokens.  ERR_NO_SNAPSHOT before eppscore_set_snapshot.
 * Not covered: top-k lists, the latency scorer's running queues, device filters, and order across GPU shards. */
int32_t eppscore_schedule_batch_inorder_profiles(struct eppscore_engine *e, const eppscore_batch *b, const int64_t *tokens,
                                                 int32_t n_runs, const eppscore_profile_run *runs,
                                                 const eppscore_inorder_profiles *x);

/* ---- stand-alone stages (same kernels; for parity tests and hosts that only want one stage) ---- */
/* hashPrompt for R prompts (hashing.go:34-98). hashes_out [R*max_blocks], n_hashes_out [R]. */
int32_t eppscore_hash_prompts(struct eppscore_engine *e, int32_t R, int32_t location, const uint8_t *prompt_bytes,
                              const int64_t *prompt_off, const int32_t *prompt_len /*optional*/,
                              const uint64_t *model_seed, int32_t block_chars, int32_t max_blocks,
                              uint64_t *hashes_out, uint16_t *n_hashes_out, void *stream);
/* len(strings.Fields(prompt)) for R prompts — the latency path's input_token_length
 * (predictedlatency/plugin.go:286, training.go:51); Go's rune decoding and unicode.IsSpace. out [R]. */
int32_t eppscore_count_fields(struct eppscore_engine *e, int32_t R, int32_t location, const uint8_t *prompt_bytes,
                              const int64_t *prompt_off, const int32_t *prompt_len /*optional*/, int32_t *out,
                              void *stream);
/* hashPrompt on the HOST cores (a persistent worker pool inside the library; n_threads <= 0: all of them) for callers that
 * ship hashes_in instead of prompt bytes: 8 bytes per 64-byte block cross PCIe instead of 64.  hashes_out [R*hash_stride]
 * (hash_stride >= max_blocks; entries past n_hashes_out[r] are zero).  Needs no engine and no GPU. */
int32_t eppscore_hash_prompts_host(int32_t R, const uint8_t *prompt_bytes, const int64_t *prompt_off,
                                   const int32_t *prompt_len /*optional*/, const uint64_t *model_seed, int32_t block_chars,
                                   int32_t max_blocks, uint64_t *hashes_out, int32_t hash_stride, uint16_t *n_hashes_out,
                                   int32_t n_threads);
/* host helper: XXH64(model || salt), hashing.go:70-77 */
uint64_t eppscore_model_seed(const void *model, size_t model_len, const void *salt, size_t salt_len);
uint64_t eppscore_xxh64(const void *data, size_t len, uint64_t seed);

/* ---- prefix index (approximateprefix/indexer.go) ----
 * Both halves of the reference's indexer are DEVICE-RESIDENT and maintained by kernels: hashToPods as an open-addressing
 * table of 32-byte slots (sets of up to 10 endpoints inline, bitset rows beyond), podToLRU as one log-structured exact LRU
 * per endpoint (hashicorp/golang-lru semantics).  The host keeps no copy. */
/* PreRequest for the batch (plugin.go:169-197): for r in order: indexer.Add(hashes[r], pick[r]) — one kernel, one CTA per
 * endpoint (Adds for different endpoints commute), calls replayed in request order within an endpoint.
 * lru_capacity: optional HOST [M] CacheNumBlocks per endpoint (autotune, plugin.go:207-216); NULL/<=0 ⇒ default. */
int32_t eppscore_commit_picks(struct eppscore_engine *e, int32_t R, const int32_t *pick, const uint64_t *hashes,
                              const uint16_t *n_hashes, int32_t hash_stride, const int32_t *lru_capacity);
/* The same with DEVICE arrays (e.g. the pick / hashes_out buffers of a device-location eppscore_schedule_batch): nothing
 * crosses PCIe, the call is asynchronous and ordered on `stream` (NULL = engine stream).  touch_bound: an upper bound on
 * Σ n_hashes (room is guaranteed up front); <= 0 ⇒ the engine sums n_hashes itself (one small synchronous read-back).
 * After eppscore_prefix_reserve the call never waits on the host (touch_bound is ignored: the device counts the touches and
 * decides the room) and may be captured into a CUDA graph; without the reserve a call on a stream under capture fails with
 * ERR_CAPACITY before anything is enqueued (the capture stays valid).  See eppscore_prefix_reserve. */
int32_t eppscore_commit_picks_device(struct eppscore_engine *e, int32_t R, const int32_t *pick, const uint64_t *hashes,
                                     const uint16_t *n_hashes, int32_t hash_stride, const int32_t *lru_capacity,
                                     int64_t touch_bound, void *stream);
/* PreRequest with several picks per request (plugin.go:177-197: the primary profile's pick, then the "prefill" profile's):
 * indexer.Add(hashes[r], picks[p][r]) for r ascending and, within r, p ascending, in one commit.  picks: n_picks pointers
 * (host array of pointers) to [R] arrays where `location` says (0 host, 1 device); pick -1 is skipped, the same endpoint twice
 * in one request is two Adds.  location 1 is asynchronous on `stream` with eppscore_commit_picks_device's touch_bound
 * contract (a bound on Σ n_hashes over all picks); location 0 ignores stream and touch_bound.  n_picks = 1 equals
 * eppscore_commit_picks[_device].  1 <= n_picks <= EPPSCORE_MAX_PROFILES. */
int32_t eppscore_commit_picks_profiles(struct eppscore_engine *e, int32_t R, int32_t n_picks, const int32_t *const *picks,
                                       const uint64_t *hashes, const uint16_t *n_hashes, int32_t hash_stride,
                                       const int32_t *lru_capacity, int32_t location, int64_t touch_bound, void *stream);
/* Reserves the prefix index up front, so that commits decide their room on the device and can run inside CUDA graphs.
 * Allocates, synchronously and outside any capture (ERR_INVALID under one): a slot table and a spare table of at least
 * 4 * (live_hashes + touches_per_call) slots each (a power of two; 32 bytes per slot), an overflow pool of at least
 * overflow_rows rows (max_endpoints / 8 bytes each), and the per-endpoint LRU regions for config.lru_capacity_max.  0 picks a
 * default: live_hashes = config.prefix_capacity, touches_per_call = 65536, overflow_rows = 2 * touches_per_call.  A later
 * reserve with larger sizes grows the table, the spare and the pool (never shrinks them, never the LRU regions); graphs
 * captured earlier stay valid, as every kernel reads the index through its device descriptor.
 * From then on every index mutation (commits, eppscore_prefix_add, eppscore_prefix_apply) runs a fixed kernel sequence that
 * counts the call's touches on the device and, with `used` slots ever claimed and `live` non-empty sets of `cap` slots:
 *   - proceeds when used + touches <= cap / 2;
 *   - else rebuilds the table into the spare (dead slots dropped, same size) and proceeds when live + touches <= cap / 4;
 *   - else, or when overflow rows in use + touches exceed the pool, skips the call whole: the index stays as it was,
 *     stats.index_error gets bit 4, and the next index mutation outside a capture fails with ERR_CAPACITY (a device commit
 *     sees it once the counters copied back behind the skipped call have landed, a host-array call at once).
 * The table never changes size behind a captured graph.  Inside a capture a commit's lru_capacity must be NULL (ERR_INVALID):
 * an LRU's size is fixed by the endpoint's first Add, so create the LRUs that need another size outside the capture (e.g.
 * eppscore_prefix_add with n = 0).  A captured commit covers every endpoint row up to max_endpoints, so a replay after
 * eppscore_set_snapshot raised M still records picks on the new endpoints.  After a captured commit, the next host-side index
 * call reads the device counters once, synchronously.  Returns EPPSCORE_OK or a negative status. */
int32_t eppscore_prefix_reserve(struct eppscore_engine *e, int64_t live_hashes, int64_t touches_per_call,
                                int64_t overflow_rows);
/* indexer.Add for one server (tests). */
int32_t eppscore_prefix_add(struct eppscore_engine *e, const uint64_t *hashes, int32_t n, int32_t endpoint,
                            int32_t lru_capacity);
/* Raw deltas for hosts that keep their own LRU: op 0 = insert (hash,endpoint), 1 = evict; applied in order. */
int32_t eppscore_prefix_apply(struct eppscore_engine *e, int64_t n, const uint64_t *hash, const int32_t *endpoint,
                              const uint8_t *op);
int32_t eppscore_prefix_remove_endpoint(struct eppscore_engine *e, int32_t endpoint); /* indexer.RemovePod :167-182 */
/* indexer.Get (reads the DEVICE table): bitset_out[ceil(M/32)] words, natural order; returns set size or <0. */
int32_t eppscore_prefix_get(struct eppscore_engine *e, uint64_t hash, uint32_t *bitset_out, int32_t words);
/* PrefixCacheMatchInfo.matchBlocks (approximateprefix/plugin.go:140-153,219-235) for chosen endpoints:
 * match_out[r*k + j] = number of blocks among request r's leading blocks that are all in the index (the walk stops at the
 * first block whose endpoint set is empty or absent, as matchLongestPrefix does) whose set holds endpoints[r*k + j].  Hits need
 * not be contiguous for an endpoint: every hit block before the first miss that holds it counts.  Entries outside
 * [0, max_endpoints) give 0, so -1 list padding needs no special case.  1 <= k <= config.max_endpoints: a pick (k = 1), a
 * top-k list, or one list per profile run.  hashes [R*hash_stride] / n_hashes [R] have the layout of eppscore_batch.hashes_out
 * and of the commit calls: pass the arrays given to eppscore_commit_picks*.
 *   location 0 (host arrays): staged through the engine's staging buffers; the call returns when match_out is filled.
 *     n_hashes[r] > hash_stride is ERR_INVALID.
 *   location 1 (device arrays): asynchronous on `stream` (NULL = engine stream); it needs no scratch, so it behaves the same on
 *     reserved and unreserved streams.  It reads the index under the ordering of a device-location batch: after the index
 *     mutations issued before it, and later mutations wait for it (it is registered like a pending device batch).  It may be
 *     captured into a CUDA graph wherever a batch may; the kernel reads the index through its device descriptor, so replays
 *     stay valid across device rebuilds and later reserves.
 * Documented use: schedule (with hashes_out) -> eppscore_prefix_match -> commit, in that order (the reference computes the match
 * before indexer.Add).  One kernel launch (counted in eppscore_stats.kernel_launches).  ERR_INVALID: k outside its range, R < 0,
 * NULL arrays with R > 0, hash_stride <= 0, a location other than 0 / 1. */
int32_t eppscore_prefix_match(struct eppscore_engine *e, int32_t R, int32_t k, int32_t location, const uint64_t *hashes,
                              const uint16_t *n_hashes, int32_t hash_stride, const int32_t *endpoints /* [R*k] */,
                              uint16_t *match_out /* [R*k] */, void *stream);
/* What the predicted-latency producer's PrepareRequestData stores on one endpoint for one request
 * (predictedlatency/preparedata_hooks.go:36-106, prediction.go:44-166): attrlatency.LatencyPredictionInfo
 * (datalayer/attribute/latency/data_types.go) plus the prefix cache score it also keeps. */
typedef struct eppscore_latency_info {
  double ttft, tpot;                  /* prediction.go:171-185, NumTokensGenerated = 1 */
  double ttft_headroom, tpot_headroom;/* ttft_slo - ttft; buffered - tpot, 0 when neutralised (prediction.go:99-103,143-161) */
  double prefix_cache_score;          /* match / total blocks, NaN (0/0) -> 0 (preparedata_hooks.go:44-56) */
  int32_t dispatched;                 /* getEndpointRunningRequestCount (plugin.go:357-363) */
  uint8_t present;                    /* 0: no prediction stored, every other field 0 */
  uint8_t ttft_valid;                 /* ttft < ttft_slo (strict: equality is not valid) */
  uint8_t tpot_valid;                 /* tpot < buffered; 1 when neutralised (!streaming_mode or a prefill-role endpoint) */
  uint8_t reserved;
} eppscore_latency_info;              /* 48 bytes */
/* The predicted-latency producer's values at chosen endpoints: info_out[r*k + j] is what PrepareRequestData would store on
 * endpoint endpoints[r*k + j] for request r, from the engine's current prepared snapshot, its latency parameters and its
 * running-request view (the inputs the last batch's latency fold-in read).  The prefix term is
 * ttft_prefix * prefix_cache_score with the match of eppscore_prefix_match; input_tokens / ttft_slo / tpot_slo [R] as
 * the eppscore_batch fields of the same names, NULL => 0.  buffered = tpot_slo * slo_buffer_factor, lowered to
 * podMinTPOTSLO * slo_buffer_factor when the endpoint's podMinTPOTSLO > 0.  dispatched comes from the snapshot's array
 * when it carries one, else from the running-request queues.  present = 0 (all fields 0) for entries outside [0, snapshot M), -1 padding included, and for every
 * entry while the snapshot was prepared with has_predictions = 0 (no attribute is stored).
 * match_out: optional [R*k], filled with what eppscore_prefix_match returns for the same arguments.
 * location, hashes / n_hashes / hash_stride, k and the stream semantics are those of eppscore_prefix_match; a device-location
 * call also waits for the snapshot preparations and producer updates issued before it, and later ones (set_snapshot,
 * running_add / running_remove / running_remove_endpoint, index commits) wait for it.  Running-request updates wait for it only
 * while a device call that reads the queue counts (a snapshot without `dispatched`) may still be in flight.
 * One known difference from the reference: each entry's TTFT uses that endpoint's own match count.  The reference keys the
 * prefix cache score it feeds the prediction by NamespacedName.Name (prediction.go:59-60), so where two candidates in different
 * namespaces share a Name, it predicts the earlier one's TTFT with the later one's score.  running_add and set_snapshot change the view, so the documented order is
 * schedule -> eppscore_predict_latency (and/or eppscore_prefix_match) -> commit / running_add / inflight_add.
 * One kernel launch.  ERR_INVALID: k outside [1, max_endpoints], a bad location, R < 0, NULL required arrays, hash_stride <= 0,
 * n_hashes > hash_stride (host location), no snapshot yet, or no profile with a latency scorer. */
int32_t eppscore_predict_latency(struct eppscore_engine *e, int32_t R, int32_t k, int32_t location, const uint64_t *hashes,
                                 const uint16_t *n_hashes, int32_t hash_stride, const int32_t *input_tokens,
                                 const double *ttft_slo, const double *tpot_slo, const int32_t *endpoints /* [R*k] */,
                                 eppscore_latency_info *info_out /* [R*k] */, uint16_t *match_out /* optional [R*k] */,
                                 void *stream);
int32_t eppscore_prefix_lru_len(const struct eppscore_engine *e, int32_t endpoint); /* -1: endpoint has no LRU */
int32_t eppscore_prefix_lru_keys(const struct eppscore_engine *e, int32_t endpoint, uint64_t *out, int32_t cap); /* oldest first */
/* Replication across GPUs: the index is a deterministic function of the ordered commit stream, so every rank applies the
 * same eppscore_commit_picks[_device] calls (the shards' picks all-gathered in global request order) — SURVEY §8e. */

/* ---- in-flight load producer (requestcontrol/dataproducer/inflightload/producer.go) ----
 * Two DEVICE-RESIDENT int64 counters per endpoint, requests and estimated tokens, zeroed by eppscore_create: the reference's
 * InFlightLoad attribute.  They feed EPPSCORE_SCORER_TOKEN_LOAD whenever the snapshot carries no inflight_tokens (a snapshot
 * that carries it keeps precedence); untouched counters are 0, which scores exactly like an absent attribute.  Every
 * mutation below prepares the current snapshot's terms again on its stream, with eppscore_set_snapshot's cross-stream
 * ordering (legal inside a CUDA-graph capture), so the next batch sees the new load; a batch sees one load view, as it sees
 * one index state.  Updates are integer adds: a batch's order does not matter, and replicas across GPUs only have to apply
 * the same SET of updates (sharding.gather_inflight_stream).  Device-location calls are asynchronous on `stream`
 * (NULL = engine stream); host-location calls return when the update is done. */
/* SimpleTokenEstimator.Estimate with its defaults, 4.0 characters per token and output ratio 1.5 (token_estimator.go:36-72),
 * for R requests, in integer arithmetic (equal to the reference for every input below 2^52 tokens):
 *   request_size_bytes[r] > 0   input = max(size / 4, 1)
 *   prompt_chars[r] < 0         Body == nil: the estimate is 0
 *   token_hint[r] >= 0          input = hint (Body.InputTokenCountHint())
 *   otherwise                   input = max(1, round(chars / 4.0)), chars = len(Body.PromptText())
 *   out[r] = input + round(1.5 * input), rounding half away from zero (math.Round).
 * Any input array may be NULL: size 0, hint -1, chars 0 (body present) respectively.  out [R]. */
int32_t eppscore_estimate_tokens(struct eppscore_engine *e, int32_t R, int32_t location, const int64_t *request_size_bytes,
                                 const int32_t *token_hint, const int32_t *prompt_chars, int64_t *out, void *stream);
/* PreRequest for a batch (producer.go:101-120): for every r with endpoint[r] >= 0, requests += 1 and tokens += tokens[r]
 * (tokens NULL: 0).  ERR_INVALID for an endpoint >= max_endpoints; device arrays cannot be checked before the launch: such
 * entries are skipped and the next eppscore_inflight_get returns ERR_INVALID. */
int32_t eppscore_inflight_add(struct eppscore_engine *e, int32_t R, int32_t location, const int32_t *endpoint,
                              const int64_t *tokens, void *stream);
/* ResponseBody at end of stream (producer.go:122-169): the same with the signs reversed.  Pass the estimate that was added:
 * the reference estimates the same request again and gets the same number. */
int32_t eppscore_inflight_release(struct eppscore_engine *e, int32_t R, int32_t location, const int32_t *endpoint,
                                  const int64_t *tokens, void *stream);
/* DeleteEndpoint (producer.go:181-187): both counters of `endpoint` to 0, so a recycled endpoint id starts from 0.  A later
 * release makes them negative, as in the reference (concurrencyTracker.add recreates the counter holding the delta); the
 * token-load scorer maps a load <= 0 to 1.0. */
int32_t eppscore_inflight_remove_endpoint(struct eppscore_engine *e, int32_t endpoint);
/* PrepareRequestData's view (producer.go:90-99): the first M counters, read synchronously on the engine stream after every
 * earlier mutation.  Either output may be NULL. */
int32_t eppscore_inflight_get(struct eppscore_engine *e, int64_t *requests_out, int64_t *tokens_out, int32_t M);

/* ---- running-request queues of the predicted-latency producer (predictedlatency/running_request_tpot_slo_queue.go) ----
 * Per endpoint, the multiset of live requests (request key, tpot SLO), DEVICE-RESIDENT, empty at create.  Its view feeds the
 * latency fold-in wherever the snapshot lacks the array (field by field; a snapshot array keeps precedence):
 *   min_tpot_slo[m] = the smallest live tpot, 0 without a live entry   (getEndpointMinTPOTSLO, plugin.go:347-355)
 *   dispatched[m]   = the number of live entries                        (getEndpointRunningRequestCount, plugin.go:357-363)
 * Empty queues give 0 and 0, which score exactly like absent arrays.  Every mutation prepares the current snapshot's terms
 * again on its stream when the queues feed them, with eppscore_set_snapshot's cross-stream ordering (legal inside a CUDA-graph
 * capture); mutations of these queues and of the in-flight counters are ordered with each other in call order.
 * Request keys are the caller's exact stand-ins for x-request-id (not hashes); 0 stands for an empty id.  The same key may be
 * live on two endpoints, as queues are per endpoint in the reference.
 * Order inside one call: equal to applying the R entries one by one in request order — of two adds of the same
 * (endpoint, key) the lower r is added and keeps its tpot, of two removes the second finds nothing.  Between calls: stream
 * order.  Entries with endpoint < 0 (unscheduled requests, pick -1) are skipped.  On host arrays an endpoint >= max_endpoints
 * or a NaN tpot is ERR_INVALID before anything changes; on device arrays such an entry is skipped and the next
 * eppscore_running_get returns ERR_INVALID.
 * tpot: finite or +Inf.  0 is a live entry like any other (no x-slo-tpot-ms header): it becomes its endpoint's minimum, and a
 * minimum of 0 turns the tightening of bufferedTPOT off (prediction.go:152, podMinTPOTSLO > 0).  -0.0 is accepted and stored
 * as +0.0; every consumer compares with > 0, so this is not observable.
 * Capacity: one open-addressing table of all live entries, at most half full counting tombstones.  Every add first compacts
 * the table on the device when live + tombstones + R would pass half the slots (the live entries move into a spare table of
 * the same size), so tombstones never run out, inside a replayed graph as well.  The kernels read the table through a
 * device-resident descriptor: a call outside a capture may double the table (only while live + R exceed a quarter of the
 * slots, so churn does not grow it), and graphs captured earlier keep working against the grown table.  A running_add under
 * CUDA-graph capture cannot grow it and fails with ERR_CAPACITY unless live + R fits half the slots
 * (eppscore_running_reserve makes room beforehand); replays must keep the live set within that room, or their adds are
 * skipped and the next eppscore_running_get returns ERR_CAPACITY.  The first call outside a capture after a captured one
 * reads the live count synchronously, as graph replays are invisible to the host.  Device-location calls are asynchronous
 * on `stream` (NULL = engine stream); host-location calls return when the update is done. */
/* PreRequest for a batch (requestcontrol_hooks.go:73-86): add (endpoint[r], request_key[r], tpot_slo[r]) for every r.  Refused
 * (added_out[r] = 0, nothing changes) for key 0, tpot < 0, and an (endpoint, key) already live (its first tpot stays:
 * running_request_tpot_slo_queue.go:127-137).  tpot_slo NULL: 0 for every entry.  added_out: optional [R], where the other
 * arrays live.  A device-resident loop passes the batch's pick and tpot_slo buffers straight in. */
int32_t eppscore_running_add(struct eppscore_engine *e, int32_t R, int32_t location, const int32_t *endpoint,
                             const uint64_t *request_key, const double *tpot_slo, uint8_t *added_out, void *stream);
/* End of stream (requestcontrol_hooks.go:219) or TTL expiry (plugin.go:190-196): remove each live (endpoint, key);
 * removed_out[r] = 1 for the entries that removed one.  Absent pairs change nothing. */
int32_t eppscore_running_remove(struct eppscore_engine *e, int32_t R, int32_t location, const int32_t *endpoint,
                                const uint64_t *request_key, uint8_t *removed_out, void *stream);
/* Empties `endpoint`'s queue, for a caller that recycles endpoint ids.  The reference has no counterpart: its queues are keyed
 * by pod name and outlive the pod, so this is the one place the engine differs — a pod that leaves while requests still run on
 * it and comes back under the same name starts empty here. */
int32_t eppscore_running_remove_endpoint(struct eppscore_engine *e, int32_t endpoint);
/* The view of the first M endpoints (min tpot as above, live count), read synchronously on the engine stream after every
 * earlier mutation.  Either output may be NULL.  ERR_INVALID reports skipped device-array entries (see above); ERR_CAPACITY
 * reports adds that found no room (a graph replayed past what eppscore_running_reserve provided). */
int32_t eppscore_running_get(struct eppscore_engine *e, double *min_tpot_out, int32_t *count_out, int32_t M);
/* Sizes the table so that it holds live_entries live entries (half its slots), and the per-call scratch for calls of up to
 * live_entries entries: do this before capturing running calls into a CUDA graph.  Returns that capacity in entries (> 0),
 * or a negative status; live_entries 0 only queries it. */
int32_t eppscore_running_reserve(struct eppscore_engine *e, int64_t live_entries);

/* ---- per-stream batch scratch ----
 * Device-location batches keep internal state in device scratch: hashes (when the batch passes no hashes_out), hash counts,
 * device-counted prompt fields, probe records, subset rows and the wide top-k score rows.  By default every stream shares one
 * set, which grows with the largest batch.  A reserved stream owns a set of its own, allocated here for batches of up to max_R
 * requests and max_blocks blocks per prompt and never reallocated (its wide score rows, one fixed byte budget, come with the
 * first wide call on the stream outside a capture).  So batches on distinct reserved streams run concurrently on the device,
 * and a graph captured on a reserved stream stays valid whatever larger calls run elsewhere.  Calls on one engine are still
 * serialised by the caller.
 * Every device-location call on a reserved stream uses its set (eppscore_schedule_batch, _topk, _topk_wide, _profiles,
 * _profiles_topk).  A batch with R > max_R, or one that hashes its prompt bytes with more blocks per prompt than max_blocks,
 * fails with ERR_CAPACITY before anything is launched.  Debug keys 5 / 6 do not cut batches on a reserved stream.  Pending
 * batches on reserved streams are waited for by index mutations, eppscore_set_snapshot and producer updates as on any stream. */
#define EPPSCORE_MAX_STREAMS 8
/* Gives caller stream `stream` its own batch scratch, sized for device-location batches of up to max_R requests and
 * max_blocks blocks per prompt (0 = config.max_blocks).  ERR_INVALID: stream NULL, max_R < 1, max_blocks outside
 * [0, EPPSCORE_MAX_BLOCKS], a stream already reserved (release it first), or while `stream`, the engine stream or a reserved
 * stream is being captured into a CUDA graph.  ERR_CAPACITY past EPPSCORE_MAX_STREAMS reserved streams. */
int32_t eppscore_reserve_stream(struct eppscore_engine *e, void *stream, int32_t max_R, int32_t max_blocks);
/* Waits for the work queued on `stream`, then frees its scratch.  Later batches on it use the shared scratch again.  Graphs
 * captured on the stream must not be replayed after this.  ERR_INVALID: stream NULL or not reserved, or under capture as
 * above.  eppscore_destroy releases every reserved stream the same way, so those streams must still exist then. */
int32_t eppscore_release_stream(struct eppscore_engine *e, void *stream);

/* pinned host memory for callers that want the fast copy path (cudaHostAlloc / cudaFreeHost) */
void *eppscore_host_alloc(size_t bytes);
void eppscore_host_free(void *p);

#ifdef __cplusplus
}
#endif
#endif /* EPPSCORE_H */
