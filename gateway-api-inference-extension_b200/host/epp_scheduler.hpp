// epp_scheduler.hpp — host side of the drop-in: the reference's Scheduler / SchedulerProfile / Filter /
// Scorer / Picker plugin interface for THIS path, restated in C++ above the C ABI (include/eppscore.h).
//
// The reference's toolchain (Go) is not in this image, so the layer a Go maintainer would write with cgo
// (INTEGRATION.md) is written here in C++ with the same names, argument meaning and error behaviour:
//   Scheduler.Schedule            pkg/epp/scheduling/scheduler.go:54-102
//   SchedulerProfile              pkg/epp/scheduling/scheduler_profile.go:41-128   (filters → scorers → picker)
//   WeightedScorer                pkg/epp/scheduling/weighted_scorer.go:32
//   Filter / Scorer / Picker      pkg/epp/framework/interface/scheduling/plugins.go:43-78
//   InferenceRequest / Endpoint / ScoredEndpoint / ProfileRunResult / SchedulingResult
//                                 pkg/epp/framework/interface/scheduling/types.go:44-170
//   Metrics                       pkg/epp/framework/interface/datalayer/metrics.go:26-42
//   SingleProfileHandler          pkg/epp/framework/plugins/scheduling/profile/single_profile_handler.go:66-99
//   PrepareRequestData/PreRequest pkg/epp/framework/plugins/requestcontrol/dataproducer/approximateprefix/plugin.go:140-205
// Scorers here are DESCRIPTORS: they name which kernel-side scorer runs and with what weight; the arithmetic
// itself happens in the CUDA kernels.  Filters run on the host exactly like the reference's filter chain and
// become the per-request candidate mask.  One Scheduler owns one engine (one GPU).
#pragma once
#include <algorithm>
#include <array>
#include <cstdint>
#include <functional>
#include <map>
#include <memory>
#include <numeric>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/eppscore.h"
#include "epp_types.hpp"
#include "host_eval.hpp"

// eppscore_schedule_batch_topk came after EPPSCORE_ABI_VERSION 3 without changing it, so an engine library of the same
// version may lack it: the symbol is bound weakly and EngineHasTopK() tells.  Without it, maxNumOfEndpoints > 1 takes the
// whole score map (max-score only, the route of k > 8); the stochastic pickers refuse k > 1.
extern "C" int32_t eppscore_schedule_batch_topk(struct eppscore_engine* e, const eppscore_batch* b, const eppscore_topk* t)
    __attribute__((weak));
// eppscore_schedule_batch_topk_wide (lists longer than 8) came the same way: EngineHasTopKWide() tells.  Without it, the
// stochastic pickers refuse k > 8 and max-score k > 8 takes the score map.
extern "C" int32_t eppscore_schedule_batch_topk_wide(struct eppscore_engine* e, const eppscore_batch* b, const eppscore_topk* t)
    __attribute__((weak));

// The in-flight load producer's entry points came the same way: bound weakly, EngineHasInFlightLoad() tells.
extern "C" int32_t eppscore_estimate_tokens(struct eppscore_engine* e, int32_t R, int32_t location, const int64_t* request_size_bytes,
                                            const int32_t* token_hint, const int32_t* prompt_chars, int64_t* out, void* stream)
    __attribute__((weak));
extern "C" int32_t eppscore_inflight_add(struct eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint,
                                         const int64_t* tokens, void* stream) __attribute__((weak));
extern "C" int32_t eppscore_inflight_release(struct eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint,
                                             const int64_t* tokens, void* stream) __attribute__((weak));
extern "C" int32_t eppscore_inflight_remove_endpoint(struct eppscore_engine* e, int32_t endpoint) __attribute__((weak));
extern "C" int32_t eppscore_inflight_get(struct eppscore_engine* e, int64_t* requests_out, int64_t* tokens_out, int32_t M)
    __attribute__((weak));

// The running-request queues of the predicted-latency producer came the same way: EngineHasRunningQueues() tells.
extern "C" int32_t eppscore_running_add(struct eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint,
                                        const uint64_t* request_key, const double* tpot_slo, uint8_t* added_out, void* stream)
    __attribute__((weak));
extern "C" int32_t eppscore_running_remove(struct eppscore_engine* e, int32_t R, int32_t location, const int32_t* endpoint,
                                           const uint64_t* request_key, uint8_t* removed_out, void* stream) __attribute__((weak));
extern "C" int32_t eppscore_running_remove_endpoint(struct eppscore_engine* e, int32_t endpoint) __attribute__((weak));
extern "C" int32_t eppscore_running_get(struct eppscore_engine* e, double* min_tpot_out, int32_t* count_out, int32_t M)
    __attribute__((weak));
extern "C" int32_t eppscore_running_reserve(struct eppscore_engine* e, int64_t live_entries) __attribute__((weak));

namespace epp {

inline bool EngineHasRunningQueues() {
  return &eppscore_running_add != nullptr && &eppscore_running_remove != nullptr && &eppscore_running_remove_endpoint != nullptr &&
         &eppscore_running_get != nullptr && &eppscore_running_reserve != nullptr;
}
inline bool EngineHasTopK() { return &eppscore_schedule_batch_topk != nullptr; }
inline bool EngineHasTopKWide() { return &eppscore_schedule_batch_topk_wide != nullptr; }
// Several scheduler profiles (eppscore_add_profile ...) came the same way: bound weakly, EngineHasProfiles() tells.  Without them
// a config with more than one profile is refused when the Scheduler is built.
extern "C" int32_t eppscore_add_profile(struct eppscore_engine* e, const eppscore_profile* p, int32_t* id_out) __attribute__((weak));
extern "C" int32_t eppscore_set_profile_endpoints(struct eppscore_engine* e, int32_t profile, const uint32_t* mask, int32_t words)
    __attribute__((weak));
extern "C" int32_t eppscore_schedule_batch_profiles(struct eppscore_engine* e, const eppscore_batch* b, int32_t n_runs,
                                                    const eppscore_profile_run* runs) __attribute__((weak));
extern "C" int32_t eppscore_commit_picks_profiles(struct eppscore_engine* e, int32_t R, int32_t n_picks, const int32_t* const* picks,
                                                  const uint64_t* hashes, const uint16_t* n_hashes, int32_t hash_stride,
                                                  const int32_t* lru_capacity, int32_t location, int64_t touch_bound, void* stream)
    __attribute__((weak));
inline bool EngineHasProfiles() {
  return &eppscore_add_profile != nullptr && &eppscore_set_profile_endpoints != nullptr && &eppscore_schedule_batch_profiles != nullptr &&
         &eppscore_commit_picks_profiles != nullptr;
}
// maxNumOfEndpoints lists per profile (eppscore_schedule_batch_profiles_topk) came the same way: EngineHasProfilesTopK() tells.
// Without it a multi-profile config with MaxNumOfEndpoints other than 1 is refused when the Scheduler is built.
extern "C" int32_t eppscore_schedule_batch_profiles_topk(struct eppscore_engine* e, const eppscore_batch* b, int32_t n_runs,
                                                         const eppscore_profile_run* runs, const eppscore_topk* topk)
    __attribute__((weak));
inline bool EngineHasProfilesTopK() { return EngineHasProfiles() && &eppscore_schedule_batch_profiles_topk != nullptr; }
// eppscore_prefix_match (PrefixCacheMatchInfo at chosen endpoints) came the same way: EngineHasPrefixMatch() tells.  Without it a
// config with SchedulerConfig::PrefixMatchInfo is refused when the Scheduler is built.
extern "C" int32_t eppscore_prefix_match(struct eppscore_engine* e, int32_t R, int32_t k, int32_t location, const uint64_t* hashes,
                                         const uint16_t* n_hashes, int32_t hash_stride, const int32_t* endpoints, uint16_t* match_out,
                                         void* stream) __attribute__((weak));
inline bool EngineHasPrefixMatch() { return &eppscore_prefix_match != nullptr; }
// eppscore_predict_latency (LatencyPredictionInfo at chosen endpoints) likewise: EngineHasPredictLatency() tells.  Without it a
// config with SchedulerConfig::LatencyPredictionInfo is refused when the Scheduler is built.
extern "C" int32_t eppscore_predict_latency(struct eppscore_engine* e, int32_t R, int32_t k, int32_t location, const uint64_t* hashes,
                                            const uint16_t* n_hashes, int32_t hash_stride, const int32_t* input_tokens,
                                            const double* ttft_slo, const double* tpot_slo, const int32_t* endpoints,
                                            eppscore_latency_info* info_out, uint16_t* match_out, void* stream) __attribute__((weak));
inline bool EngineHasPredictLatency() { return &eppscore_predict_latency != nullptr; }

// What PreRequest keeps per request id with SchedulerConfig::LatencyPredictionInfo, as predictedLatencyCtx holds it after
// processPreRequestForLatencyPrediction (requestcontrol_hooks.go:236-251) and predictFirstTPOT (:309-321): the predicted TTFT and
// the prefix cache score at the "prefill" profile's target when there is one, else at the primary target; the stored TPOT at
// the primary target; the request's SLOs.  0 where no prediction was stored.
struct PredictedLatencyAtDispatch {
  double PredictedTTFT = 0.0;
  double PrefixCacheScore = 0.0;
  double FirstPredictedTPOT = 0.0;
  double TTFTSLO = 0.0;
  double AvgTPOTSLO = 0.0;
};

// A prometheus histogram as client_golang keeps it: an observation lands in the first bucket whose upper bound is >= it
// (sort.SearchFloat64s over the bounds), past the last bound in +Inf; Count and Sum accumulate in observation order.
template <size_t N>
struct Histogram {
  std::array<double, N> UpperBounds;
  std::array<uint64_t, N + 1> Counts{};  // per bucket, not cumulative: Counts[i] for UpperBounds[i], Counts[N] for +Inf
  uint64_t Count = 0;
  double Sum = 0.0;
  void Observe(double v) {
    Counts[(size_t)(std::lower_bound(UpperBounds.begin(), UpperBounds.end(), v) - UpperBounds.begin())]++;
    Count++;
    Sum += v;
  }
};
// The approximate-prefix producer's two PreRequest histograms (metrics.go:358-377), fed by RecordPrefixCacheMatch (:830-841).
struct PrefixIndexerHistograms {
  Histogram<11> HitRatio{{0.0, 0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 1.0}};  // prefix_indexer_hit_ratio
  Histogram<14> HitBytes{{0, 16, 32, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536}};  // prefix_indexer_hit_bytes
};

// eppscore_schedule_batch_inorder (a batch in arrival order against the in-flight load) came the same way: EngineHasInOrderLoad()
// tells.  Without it a config with SchedulerConfig::InOrderInFlightLoad is refused when the Scheduler is built.
extern "C" int32_t eppscore_schedule_batch_inorder(struct eppscore_engine* e, const eppscore_batch* b, const int64_t* tokens)
    __attribute__((weak));
inline bool EngineHasInOrderLoad() { return &eppscore_schedule_batch_inorder != nullptr; }
// eppscore_schedule_batch_inorder_index (the same, ordered against the prefix index too) likewise: EngineHasInOrderPrefixIndex()
// tells.  Without it a config with SchedulerConfig::InOrderPrefixIndex is refused when the Scheduler is built.
extern "C" int32_t eppscore_schedule_batch_inorder_index(struct eppscore_engine* e, const eppscore_batch* b, const int64_t* tokens,
                                                         const eppscore_inorder_index* x) __attribute__((weak));
inline bool EngineHasInOrderPrefixIndex() { return &eppscore_schedule_batch_inorder_index != nullptr; }
// eppscore_schedule_batch_inorder_latency (either in-order call with the latency scorer ordered against the running-request
// queues) likewise: EngineHasInOrderLatency() tells.  Without it a config with SchedulerConfig::InOrderRunningRequests is refused.
extern "C" int32_t eppscore_schedule_batch_inorder_latency(struct eppscore_engine* e, const eppscore_batch* b, const int64_t* tokens,
                                                           const eppscore_inorder_index* x, const eppscore_inorder_running* q)
    __attribute__((weak));
inline bool EngineHasInOrderLatency() { return &eppscore_schedule_batch_inorder_latency != nullptr; }
// eppscore_schedule_batch_inorder_profiles (either in-order call over several profiles) likewise: EngineHasInOrderProfiles() tells.
// Without it a Profiles config with SchedulerConfig::InOrderInFlightLoad is refused.
extern "C" int32_t eppscore_schedule_batch_inorder_profiles(struct eppscore_engine* e, const eppscore_batch* b, const int64_t* tokens,
                                                            int32_t n_runs, const eppscore_profile_run* runs,
                                                            const eppscore_inorder_profiles* x) __attribute__((weak));
inline bool EngineHasInOrderProfiles() { return &eppscore_schedule_batch_inorder_profiles != nullptr; }

inline bool EngineHasInFlightLoad() {
  return &eppscore_estimate_tokens != nullptr && &eppscore_inflight_add != nullptr && &eppscore_inflight_release != nullptr &&
         &eppscore_inflight_remove_endpoint != nullptr && &eppscore_inflight_get != nullptr;
}

// ---- plugins (descriptors) ----
struct Scorer {
  std::string Type;
  int32_t Kind;
  virtual ~Scorer() = default;
  Scorer(std::string t, int32_t k) : Type(std::move(t)), Kind(k) {}
};
struct KVCacheUtilizationScorer : Scorer { KVCacheUtilizationScorer() : Scorer("kv-cache-utilization-scorer", EPPSCORE_SCORER_KV_CACHE) {} };
struct QueueScorer : Scorer { QueueScorer() : Scorer("queue-scorer", EPPSCORE_SCORER_QUEUE) {} };
struct LoraAffinityScorer : Scorer { LoraAffinityScorer() : Scorer("lora-affinity-scorer", EPPSCORE_SCORER_LORA) {} };
struct PrefixCacheScorer : Scorer { PrefixCacheScorer() : Scorer("prefix-cache-scorer", EPPSCORE_SCORER_PREFIX) {} };
struct RunningRequestsScorer : Scorer { RunningRequestsScorer() : Scorer("running-requests-size-scorer", EPPSCORE_SCORER_RUNNING) {} };
// token-load-scorer (scorer/tokenload/token_load.go:36-67)
struct TokenLoadScorer : Scorer {
  int64_t QueueThresholdTokens;
  explicit TokenLoadScorer(int64_t thr = 4194304) : Scorer("token-load-scorer", EPPSCORE_SCORER_TOKEN_LOAD), QueueThresholdTokens(thr > 0 ? thr : 4194304) {}
};
// latency-scorer (scorer/latency/plugin.go:59-90); fed by the PredictedLatencyProducer below
struct LatencyScorer : Scorer {
  double TTFTWeight = 0.8, TPOTWeight = 0.2;
  bool StrategyMost = false;  // HeadroomSelectionStrategy "most"; default "least"
  double CompositeKVWeight = 1, CompositeQueueWeight = 1, CompositePrefixWeight = 1;
  LatencyScorer() : Scorer("latency-scorer", EPPSCORE_SCORER_LATENCY) {}
};

// predicted-latency-producer (requestcontrol/dataproducer/predictedlatency): its Config (plugin.go:118-136), the
// Bayesian-ridge coefficients the Go client caches (latencypredictorasync/prediction.go:164-194) and the
// per-endpoint running-request bookkeeping it reads while predicting (plugin.go:347-363).
struct PredictedLatencyProducer {
  double SLOBufferFactor = 1.0;
  bool StreamingMode = false;
  std::string EndpointRoleLabel;
  bool HavePredictions = true;  // false = sidecar down / timed out: the scorer's composite fallback
  double TTFTIntercept = 0, TPOTIntercept = 0;
  std::map<std::string, double> TTFTCoeffs, TPOTCoeffs;  // keys as in the reference's MetricsResponse
  struct EndpointState {
    double MinTPOTSLO = 0;   // getEndpointMinTPOTSLO
    int RunningRequests = 0; // getEndpointRunningRequestCount
  };
  std::map<std::string, EndpointState> State;  // keyed by NamespacedName.String()
  // Opt-in: the Scheduler keeps the running-request queues itself, on the device (eppscore_running_*), as the reference's
  // producer does (requestcontrol_hooks.go:73-86,219, plugin.go:190-196): PreRequest adds each scheduled request with its
  // x-slo-tpot-ms to its TargetEndpoints[0], ResponseComplete and RequestExpired remove it, RemovePod empties the endpoint.
  // State is then not read.  A request with an empty RequestId is not tracked (requestcontrol_hooks.go:66-69).
  bool TrackRunningRequests = false;
};

// inflight-load-producer (requestcontrol/dataproducer/inflightload/producer.go): requests and estimated tokens in flight per
// endpoint, the InFlightLoad attribute the token-load scorer reads.  The counters live on the device (eppscore_inflight_*);
// the plugin has no parameters (its factory, producer.go:40-47, uses SimpleTokenEstimator's defaults).
struct InFlightLoadProducer {};

struct WeightedScorer {
  std::shared_ptr<Scorer> Scorer_;
  double Weight_;
  double Weight() const { return Weight_; }
};
inline WeightedScorer NewWeightedScorer(std::shared_ptr<Scorer> s, double w) { return WeightedScorer{std::move(s), w}; }

// framework.Filter: given the request and the current candidates (indices into the slice passed to Schedule),
// return the ones to keep.  Runs on the host, chained in order, early exit on empty (scheduler_profile.go:130-149).
struct Filter {
  virtual ~Filter() = default;
  virtual std::vector<int> Filter_(const InferenceRequest& req, const std::vector<Endpoint>& endpoints,
                                   const std::vector<int>& candidates) = 0;
};

// Filters the engine evaluates on the device (include/eppscore.h: eppscore_filter_kind).  They are descriptors like the
// scorers; any other Filter subclass runs on the host and reaches the engine as the candidate mask.  Device filters
// run AFTER the host filters, in the order given to WithDeviceFilters.
struct DeviceFilter {
  int32_t Kind;
  double Param[3];
};
// prefix-cache-affinity-filter (filter/prefixcacheaffinity/plugin.go:52-62): defaults 0.80 / 0.01 / 5000
inline DeviceFilter PrefixCacheAffinityFilter(double affinityThreshold = 0.80, double explorationProbability = 0.01,
                                              double maxTTFTPenaltyMs = 5000) {
  return DeviceFilter{EPPSCORE_FILTER_PREFIX_AFFINITY, {affinityThreshold, explorationProbability, maxTTFTPenaltyMs}};
}
// slo-headroom-tier-filter (filter/sloheadroomtier/plugin.go:50-52): default epsilonExploreNeg 0.01
inline DeviceFilter SLOHeadroomTierFilter(double epsilonExploreNeg = 0.01) {
  return DeviceFilter{EPPSCORE_FILTER_SLO_HEADROOM_TIER, {epsilonExploreNeg, 0, 0}};
}

struct MaxScorePicker {
  int MaxNumOfEndpoints = 1;  // picker.DefaultMaxNumOfEndpoints (picker/common.go:36); 2..8: the engine's top-k lists (every
                              // mode); > 8: the engine's wide lists (every mode; max-score with TIE_SEEDED_RANDOM, or an
                              // engine without the wide call: max-score only, from the engine's score rows)
  int Mode = EPPSCORE_PICK_MAX_SCORE;
};
// weighted-random-picker (A-Res, picker/weightedrandom/picker.go:111-155) and random-picker (picker/random/picker.go:85-101):
// same descriptor with another pick mode; the engine's generator is counter-based (SchedulerConfig.TieSeed).
struct WeightedRandomPicker : MaxScorePicker { WeightedRandomPicker() { Mode = EPPSCORE_PICK_WEIGHTED_RANDOM; } };
struct RandomPicker : MaxScorePicker { RandomPicker() { Mode = EPPSCORE_PICK_RANDOM; } };

class SchedulerProfile {
 public:
  SchedulerProfile& WithFilters(std::vector<std::shared_ptr<Filter>> f) { filters_ = std::move(f); return *this; }
  SchedulerProfile& WithScorers(std::vector<WeightedScorer> s) { scorers_ = std::move(s); return *this; }
  SchedulerProfile& WithPicker(MaxScorePicker p) { picker_ = p; return *this; }
  SchedulerProfile& WithDeviceFilters(std::vector<DeviceFilter> f) { device_filters_ = std::move(f); return *this; }
  // A request-independent Filter at the head of the profile's filter chain (e.g. a prefill / decode role label): the endpoints
  // it keeps are the profile's endpoint subset on the engine (eppscore_set_profile_endpoints), packed with every snapshot, so
  // batches need no per-request mask for it.  Multi-profile configs only.
  SchedulerProfile& WithEndpointSubset(std::function<bool(const Endpoint&)> keep) { subset_ = std::move(keep); return *this; }
  const std::function<bool(const Endpoint&)>& endpoint_subset() const { return subset_; }
  const std::vector<DeviceFilter>& device_filters() const { return device_filters_; }
  SchedulerProfile& WithPredictedLatencyProducer(std::shared_ptr<PredictedLatencyProducer> p) { producer_ = std::move(p); return *this; }
  const std::shared_ptr<PredictedLatencyProducer>& producer() const { return producer_; }
  const std::vector<std::shared_ptr<Filter>>& filters() const { return filters_; }
  const std::vector<WeightedScorer>& scorers() const { return scorers_; }
  const MaxScorePicker& picker() const { return picker_; }

 private:
  std::vector<std::shared_ptr<Filter>> filters_;
  std::vector<WeightedScorer> scorers_;
  MaxScorePicker picker_;
  std::shared_ptr<PredictedLatencyProducer> producer_;
  std::vector<DeviceFilter> device_filters_;
  std::function<bool(const Endpoint&)> subset_;
};

// framework.ProfileHandler (scheduler.go:54-102): Pick names the profiles to run for a request given the results so far (empty
// on the first round; an empty answer ends the loop), ProcessResults turns every profile's result (nullptr: the profile found
// no endpoint) into the request's SchedulingResult, or throws SchedulingError with the reference's error.
struct ProfileHandler {
  virtual ~ProfileHandler() = default;
  virtual std::vector<std::string> Pick(const InferenceRequest& request, const std::vector<std::string>& profiles,
                                        const std::map<std::string, const ProfileRunResult*>& results) = 0;
  virtual SchedulingResult ProcessResults(const InferenceRequest& request,
                                          const std::map<std::string, const ProfileRunResult*>& results) = 0;
};
// single-profile-handler (single_profile_handler.go): the one profile, once; its result is the primary one.
struct SingleProfileHandler : ProfileHandler {
  std::vector<std::string> Pick(const InferenceRequest&, const std::vector<std::string>& profiles,
                                const std::map<std::string, const ProfileRunResult*>& results) override {
    if (!results.empty() || profiles.empty()) return {};
    return {profiles[0]};
  }
  SchedulingResult ProcessResults(const InferenceRequest&, const std::map<std::string, const ProfileRunResult*>& results) override {
    const auto& kv = *results.begin();
    if (!kv.second) throw SchedulingError("failed to run scheduler profile '" + kv.first + "'");
    SchedulingResult r;
    r.ProfileResults[kv.first] = *kv.second;
    r.PrimaryProfileName = kv.first;
    return r;
  }
};

// approximateprefix config (types.go:77-141)
struct PrefixConfig {
  bool AutoTune = true;
  int BlockSizeTokens = 16;
  int MaxPrefixBlocksToMatch = 256;
  int MaxPrefixTokensToMatch = 0;
  int LRUCapacityPerServer = 31250;
};

struct SchedulerConfig {
  std::string ProfileName = "default";  // SingleProfileHandler: exactly one profile
  SchedulerProfile Profile;
  PrefixConfig Prefix;
  int Device = 0;
  int MaxEndpoints = 1024;
  int MaxAdapters = 64;
  int64_t PrefixCapacity = 1 << 18;
  int TieMode = EPPSCORE_TIE_LOWEST_INDEX;
  uint64_t TieSeed = 0;
  // Batches of at most this many requests whose profile is request-independent (queue / kv / running / lora / token-load
  // scorers, no device filters, max-score picker, lowest-index ties) are evaluated on the host (SmallBatchCpu): a launch
  // costs tens of microseconds, a 1 x 4 queue-scorer Schedule a fraction of one.  0 disables the route.
  int CpuBatchThreshold = 8;
  // Opt-in, as the plugin is in the reference's config.  With it, PreRequest also counts each request on its target endpoint,
  // ResponseComplete releases it, RemovePod drops the endpoint's counters, and a token-load scorer reads the counters
  // (Endpoint::InFlightTokens is then not used).  Batches always take the engine route: the counters live on the device.
  std::shared_ptr<InFlightLoadProducer> InFlightLoad;
  // Several named profiles, in order (the first is the engine's profile 0), and the handler that picks among them.  Empty: the
  // single `Profile` above with SingleProfileHandler semantics, on the path that has always served it.  A multi-profile config
  // needs an engine library with the profile calls; MaxNumOfEndpoints other than 1 on a profile needs
  // eppscore_schedule_batch_profiles_topk, and TargetEndpoints then carries that profile's whole list.  The latency parameters
  // are engine-wide, as the reference has one predicted-latency producer: every profile that has a producer must have the same
  // one (the same object or equal parameters; the first profile's is read), and every latency scorer equal parameters.  With
  // TrackRunningRequests, PreRequest queues each request on the primary profile's TargetEndpoints[0] only
  // (requestcontrol_hooks.go:55-95), and ResponseComplete / RequestExpired remove it there.  The profile named "prefill" gets the
  // second prefix-index Add of PreRequest (approximateprefix/plugin.go:177-197) and its in-flight load is released at
  // ResponseStarted (inflightload/producer.go:137-160).
  std::vector<std::pair<std::string, SchedulerProfile>> Profiles;
  std::shared_ptr<ProfileHandler> Handler;
  // Opt-in (off by default): after each engine batch that hashed its prompts, one eppscore_prefix_match call gives every
  // TargetEndpoints entry of every profile (lists and the "prefill" profile included) its PrefixCacheMatchInfo, as
  // PrepareRequestData puts it on every endpoint (approximateprefix/plugin.go:140-153), and PreRequest records the
  // prefix-indexer histograms for the primary target (plugin.go:199-204; Scheduler::PrefixIndexerMetrics).  Batches the engine
  // did not hash (the small-batch host route, a config without prefix hashing) leave it empty.  Needs an engine library with
  // eppscore_prefix_match.
  bool PrefixMatchInfo = false;
  // Opt-in (off by default): after each engine batch piece, one eppscore_predict_latency call gives every TargetEndpoints entry
  // of every profile (lists and the "prefill" profile included) its LatencyPredictionInfo (SchedulingResult::TargetLatency), as the
  // predicted-latency producer's PrepareRequestData stores it on every endpoint; with PrefixMatchInfo as well, the same call
  // fills the PrefixCacheMatchInfo.  PreRequest then keeps the dispatch record of each request with an id
  // (Scheduler::PredictedLatencyAtDispatch) until ResponseComplete / RequestExpired.  Batches of the small-batch host route leave
  // it empty.  Needs a profile with a latency scorer and an engine library with eppscore_predict_latency.
  bool LatencyPredictionInfo = false;
  // Opt-in (off by default), with InFlightLoad: every engine batch goes through eppscore_schedule_batch_inorder, so request r of
  // a batch is scored against the load requests 0..r-1 were sent with, as the reference's per-request Schedule + PreRequest
  // sequence does (inflightload/producer.go:101-120 before token_load.go:83-111), instead of one load view per batch.  The
  // call adds each request's estimate to its TargetEndpoints[0] while it schedules, so PreRequest does not add it again;
  // ResponseComplete releases it as before.  The counters after ScheduleBatch + PreRequest are those of the per-request
  // sequence.  Refused with a latency scorer, with MaxNumOfEndpoints > 1, without InFlightLoad and with an engine library without
  // the call.  With the Profiles list (every profile with MaxNumOfEndpoints 1, no latency scorer and no device filters) each
  // engine batch, LoRA pieces in order, is one eppscore_schedule_batch_inorder_profiles call: the runs are the profiles in order,
  // each request's run mask is the handler's first Pick, the primary run is the first profile and the prefill run the profile
  // named "prefill".  The call counts each request on every profile's target when the first profile picked, so PreRequest adds
  // no load.  A request whose ProcessResults names another primary profile gets an error, but its load (and with
  // InOrderPrefixIndex its blocks) was already recorded at the first profile's target.  Needs an engine library with
  // eppscore_schedule_batch_inorder_profiles.
  bool InOrderInFlightLoad = false;
  // Opt-in (off by default), with InOrderInFlightLoad and the approximate-prefix producer (prefix hashing on): every engine batch
  // goes through eppscore_schedule_batch_inorder_index, so request r is also scored against the prefix index as requests
  // 0..r-1's Adds left it (approximateprefix/plugin.go:169-197 before :219-235), and each request's blocks are added at its
  // pick inside the call, with LruCapacities().  PreRequest then does not commit that batch again, and with PrefixMatchInfo the
  // target's PrefixCacheMatchInfo is the pick's match as the request was scored, before its own Add (plugin.go:199-204).  A
  // batch cut into LoRA pieces runs its pieces in order, each committing before the next is scheduled.  Refused with
  // LatencyPredictionInfo (eppscore_predict_latency after the batch would read the index the batch left), without
  // InOrderInFlightLoad or prefix hashing, and with an engine library without the call.  With the Profiles list it is the index
  // form of that call: the primary and the "prefill" targets get their Adds inside it, PreRequest commits nothing, and with
  // PrefixMatchInfo every profile's target gets its run's pick_match.
  bool InOrderPrefixIndex = false;
  // Opt-in (off by default), with InOrderInFlightLoad and a profile with a latency scorer: every engine batch goes through
  // eppscore_schedule_batch_inorder_latency (its index form with InOrderPrefixIndex), so request r's latency scorer sees the
  // running-request queues after requests 0..r-1 joined them, as the reference's per-request Schedule + PreRequest sequence
  // does (requestcontrol_hooks.go:73-86 before scorer/latency/plugin.go:189-202 and prediction.go:149-161).  With
  // TrackRunningRequests each request is added to its TargetEndpoints[0]'s queue inside the call, under its x-request-id, so
  // PreRequest does not add it again; ResponseComplete, RequestExpired and RemovePod remove it as before.  Without
  // TrackRunningRequests the queues are read, never changed.  A batch cut into LoRA pieces runs its pieces in order.  Refused
  // without InOrderInFlightLoad, with LatencyPredictionInfo (eppscore_predict_latency after the batch would read the queues the
  // batch left), with device filters, with the Profiles list, with MaxNumOfEndpoints > 1 and with an engine library without
  // the call.
  bool InOrderRunningRequests = false;
};

class Scheduler {
 public:
  explicit Scheduler(const SchedulerConfig& cfg) : Scheduler(cfg, 0) {
    if (cfg.Profiles.empty()) return;
    for (size_t p = 1; p < cfg.Profiles.size(); p++) {  // profile 0 was created with the engine
      const SchedulerProfile& sp = cfg.Profiles[p].second;
      eppscore_profile ep{};
      ep.struct_size = sizeof(ep);
      if (sp.scorers().size() > EPPSCORE_MAX_SCORERS || sp.device_filters().size() > EPPSCORE_MAX_FILTERS)
        throw SchedulingError("too many scorers or device filters in profile '" + cfg.Profiles[p].first + "'");
      CopyProfile(sp, &ep);
      int32_t id = -1;
      Check(eppscore_add_profile(eng_, &ep, &id), "eppscore_add_profile");  // (the destructor frees the engine)
    }
  }

 private:
  // A profile's scorers, picker and device filters into eppscore_config or eppscore_profile, which name these fields alike.
  template <class EngineProfile>
  static void CopyProfile(const SchedulerProfile& sp, EngineProfile* c) {
    c->n_scorers = (int32_t)sp.scorers().size();
    for (size_t i = 0; i < sp.scorers().size(); i++) {
      c->scorer_kind[i] = sp.scorers()[i].Scorer_->Kind;
      c->scorer_weight[i] = sp.scorers()[i].Weight();
    }
    c->pick_mode = sp.picker().Mode;
    c->n_filters = (int32_t)sp.device_filters().size();
    for (size_t i = 0; i < sp.device_filters().size(); i++) {
      c->filter_kind[i] = sp.device_filters()[i].Kind;
      for (int q = 0; q < 3; q++) c->filter_param[i][q] = sp.device_filters()[i].Param[q];
    }
  }
  void Check(int32_t rc, const char* call) const {
    if (rc != EPPSCORE_OK) throw SchedulingError(std::string(call) + ": " + eppscore_last_error(eng_));
  }

  static SchedulerConfig SingleOrFirst(const SchedulerConfig& cfg) {  // the engine's profile 0 and the checks of its path
    if (cfg.Profiles.empty()) return cfg;
    if (!EngineHasProfiles()) throw SchedulingError("a config with several profiles needs an engine library with eppscore_add_profile");
    if (!cfg.Handler) throw SchedulingError("a config with several profiles needs a ProfileHandler");
    if (cfg.Profiles.size() > EPPSCORE_MAX_PROFILES) throw SchedulingError("more profiles than EPPSCORE_MAX_PROFILES");
    std::shared_ptr<PredictedLatencyProducer> prod;
    const LatencyScorer* lat = nullptr;
    for (const auto& np : cfg.Profiles) {
      const int k = np.second.picker().MaxNumOfEndpoints;
      if (k < 1) throw SchedulingError("maxNumOfEndpoints must be >= 1 (profile '" + np.first + "')");
      if (k != 1 && !EngineHasProfilesTopK())
        throw SchedulingError("maxNumOfEndpoints > 1 with several profiles needs an engine library with "
                              "eppscore_schedule_batch_profiles_topk (profile '" + np.first + "')");
      for (const auto& w : np.second.scorers())
        if (const auto* ls = dynamic_cast<const LatencyScorer*>(w.Scorer_.get())) {
          if (lat && !SameLatencyScorer(*lat, *ls))
            throw SchedulingError("the latency scorers of several profiles must have equal parameters, the engine has one set (profile '" +
                                  np.first + "')");
          lat = ls;
        }
      if (const auto& p = np.second.producer()) {
        if (prod && prod != p && !SameProducer(*prod, *p))
          throw SchedulingError("the profiles have different predicted-latency producers; the engine has one, so they must share it (profile '" +
                                np.first + "')");
        if (!prod) prod = p;
      }
    }
    SchedulerConfig c = cfg;
    c.ProfileName = cfg.Profiles[0].first;
    c.Profile = cfg.Profiles[0].second;
    if (prod) c.Profile.WithPredictedLatencyProducer(prod);  // the engine-wide producer, whichever profile names it
    c.CpuBatchThreshold = 0;  // the host route serves one profile
    return c;
  }
  static bool SameLatencyScorer(const LatencyScorer& a, const LatencyScorer& b) {
    return a.TTFTWeight == b.TTFTWeight && a.TPOTWeight == b.TPOTWeight && a.StrategyMost == b.StrategyMost &&
           a.CompositeKVWeight == b.CompositeKVWeight && a.CompositeQueueWeight == b.CompositeQueueWeight &&
           a.CompositePrefixWeight == b.CompositePrefixWeight;
  }
  static bool SameProducer(const PredictedLatencyProducer& a, const PredictedLatencyProducer& b) {
    if (a.State.size() != b.State.size()) return false;
    for (const auto& kv : a.State) {
      auto it = b.State.find(kv.first);
      if (it == b.State.end() || it->second.MinTPOTSLO != kv.second.MinTPOTSLO || it->second.RunningRequests != kv.second.RunningRequests)
        return false;
    }
    return a.SLOBufferFactor == b.SLOBufferFactor && a.StreamingMode == b.StreamingMode && a.EndpointRoleLabel == b.EndpointRoleLabel &&
           a.HavePredictions == b.HavePredictions && a.TTFTIntercept == b.TTFTIntercept && a.TPOTIntercept == b.TPOTIntercept &&
           a.TTFTCoeffs == b.TTFTCoeffs && a.TPOTCoeffs == b.TPOTCoeffs && a.TrackRunningRequests == b.TrackRunningRequests;
  }
  Scheduler(const SchedulerConfig& cfg0, int) : cfg_(SingleOrFirst(cfg0)) {
    const SchedulerConfig& cfg = cfg_;
    eppscore_config c;
    eppscore_config_default(&c);
    const auto& sc = cfg.Profile.scorers();
    if (sc.size() > EPPSCORE_MAX_SCORERS) throw SchedulingError("too many scorers in profile");
    if (cfg.Profile.picker().MaxNumOfEndpoints < 1) throw SchedulingError("maxNumOfEndpoints must be >= 1");
    if (cfg.Profile.picker().MaxNumOfEndpoints > EPPSCORE_MAX_TOPK && cfg.Profile.picker().Mode != EPPSCORE_PICK_MAX_SCORE &&
        !EngineHasTopKWide())
      throw SchedulingError("maxNumOfEndpoints > 8 with a stochastic picker needs an engine library with eppscore_schedule_batch_topk_wide");
    if (cfg.Profile.picker().MaxNumOfEndpoints > 1 && cfg.Profile.picker().Mode != EPPSCORE_PICK_MAX_SCORE && !EngineHasTopK())
      throw SchedulingError("maxNumOfEndpoints > 1 with a stochastic picker needs an engine library with eppscore_schedule_batch_topk");
    if (cfg.InFlightLoad && !EngineHasInFlightLoad())
      throw SchedulingError("the inflight-load-producer needs an engine library with eppscore_inflight_add");
    if (cfg.PrefixMatchInfo && !cfg0.InOrderPrefixIndex && !EngineHasPrefixMatch())  // (in order: the call returns the match)
      throw SchedulingError("SchedulerConfig::PrefixMatchInfo needs an engine library with eppscore_prefix_match");
    if (cfg.LatencyPredictionInfo && !EngineHasPredictLatency())
      throw SchedulingError("SchedulerConfig::LatencyPredictionInfo needs an engine library with eppscore_predict_latency");
    inflight_ = cfg.InFlightLoad != nullptr;
    if (cfg0.InOrderInFlightLoad) {
      if (!inflight_) throw SchedulingError("SchedulerConfig::InOrderInFlightLoad needs the inflight-load-producer (InFlightLoad)");
      if (cfg.Profile.picker().MaxNumOfEndpoints > 1) throw SchedulingError("SchedulerConfig::InOrderInFlightLoad needs maxNumOfEndpoints == 1");
      for (const auto& np : cfg0.Profiles) {
        if (np.second.picker().MaxNumOfEndpoints != 1)
          throw SchedulingError("SchedulerConfig::InOrderInFlightLoad needs maxNumOfEndpoints == 1 (profile '" + np.first + "')");
        for (const auto& w : np.second.scorers())
          if (dynamic_cast<const LatencyScorer*>(w.Scorer_.get()))
            throw SchedulingError("SchedulerConfig::InOrderInFlightLoad cannot order the latency scorer's inputs (profile '" + np.first + "')");
        if (!np.second.device_filters().empty())
          throw SchedulingError("SchedulerConfig::InOrderInFlightLoad does not order the device filters (profile '" + np.first + "')");
      }
      if (!cfg0.Profiles.empty() && cfg0.Profiles[0].first == "prefill")
        throw SchedulingError("SchedulerConfig::InOrderInFlightLoad needs the first profile (the primary) to be other than \"prefill\"");
      if (!cfg0.Profiles.empty() && !EngineHasInOrderProfiles())
        throw SchedulingError("SchedulerConfig::InOrderInFlightLoad with several profiles needs an engine library with "
                              "eppscore_schedule_batch_inorder_profiles");
      if (!cfg0.InOrderRunningRequests)
        for (const auto& w : sc)
          if (dynamic_cast<const LatencyScorer*>(w.Scorer_.get()))
            throw SchedulingError("SchedulerConfig::InOrderInFlightLoad cannot order the latency scorer's inputs");
      if (cfg0.Profiles.empty() && !EngineHasInOrderLoad())
        throw SchedulingError("SchedulerConfig::InOrderInFlightLoad needs an engine library with eppscore_schedule_batch_inorder");
      inorder_ = true;
    }
    if (cfg0.InOrderPrefixIndex) {
      if (!cfg0.InOrderInFlightLoad) throw SchedulingError("SchedulerConfig::InOrderPrefixIndex needs InOrderInFlightLoad");
      if (!Geometry({}).want_prefix) throw SchedulingError("SchedulerConfig::InOrderPrefixIndex needs the approximate-prefix producer (prefix hashing)");
      if (cfg.LatencyPredictionInfo)
        throw SchedulingError("SchedulerConfig::InOrderPrefixIndex cannot give LatencyPredictionInfo: the prediction would read the "
                              "prefix index the batch left");
      if (cfg0.Profiles.empty() && !(cfg0.InOrderRunningRequests ? EngineHasInOrderLatency() : EngineHasInOrderPrefixIndex()))  // (the route's one call)
        throw SchedulingError("SchedulerConfig::InOrderPrefixIndex needs an engine library with eppscore_schedule_batch_inorder_index");
      inorder_index_ = true;
    }
    if (cfg0.InOrderRunningRequests) {
      if (!cfg0.InOrderInFlightLoad) throw SchedulingError("SchedulerConfig::InOrderRunningRequests needs InOrderInFlightLoad");
      if (!cfg0.Profiles.empty()) throw SchedulingError("SchedulerConfig::InOrderRunningRequests serves the single-profile config, not the Profiles list");
      if (cfg.Profile.picker().MaxNumOfEndpoints > 1) throw SchedulingError("SchedulerConfig::InOrderRunningRequests needs maxNumOfEndpoints == 1");
      bool lat = false;
      for (const auto& w : sc) lat = lat || dynamic_cast<const LatencyScorer*>(w.Scorer_.get()) != nullptr;
      if (!lat) throw SchedulingError("SchedulerConfig::InOrderRunningRequests needs a profile with a latency-scorer");
      if (!cfg.Profile.device_filters().empty())
        throw SchedulingError("SchedulerConfig::InOrderRunningRequests does not order the device filters");
      if (cfg.LatencyPredictionInfo)
        throw SchedulingError("SchedulerConfig::InOrderRunningRequests cannot give LatencyPredictionInfo: the prediction would read "
                              "the running-request queues the batch left");
      if (!EngineHasInOrderLatency())
        throw SchedulingError("SchedulerConfig::InOrderRunningRequests needs an engine library with eppscore_schedule_batch_inorder_latency");
      inorder_latency_ = true;
    }
    running_ = cfg.Profile.producer() && cfg.Profile.producer()->TrackRunningRequests;
    if (running_ && !EngineHasRunningQueues())
      throw SchedulingError("TrackRunningRequests needs an engine library with eppscore_running_add");
    {  // the small-batch CPU route applies to request-independent profiles only
      std::vector<int32_t> kinds;
      std::vector<double> weights;
      for (auto& w : sc) {
        kinds.push_back(w.Scorer_->Kind);
        weights.push_back(w.Weight());
      }
      double thr = 4194304.0;
      for (auto& w : sc)
        if (auto* tl = dynamic_cast<TokenLoadScorer*>(w.Scorer_.get())) thr = (double)tl->QueueThresholdTokens;
      cpu_route_ok_ = cfg.CpuBatchThreshold > 0 && !inflight_ && !running_ && cfg.Profile.device_filters().empty() && cfg.Profile.picker().Mode == EPPSCORE_PICK_MAX_SCORE &&
                      cfg.Profile.picker().MaxNumOfEndpoints == 1 && cfg.TieMode == EPPSCORE_TIE_LOWEST_INDEX && cpu_.Configure(kinds, weights, thr);
    }
    for (const auto& w : sc) {
      if (auto* tl = dynamic_cast<TokenLoadScorer*>(w.Scorer_.get())) {
        c.token_load_threshold = (double)tl->QueueThresholdTokens;
        token_load_ = true;
      }
      if (auto* ls = dynamic_cast<LatencyScorer*>(w.Scorer_.get())) latency_scorer_ = ls;
    }
    for (const auto& np : cfg.Profiles)  // the latency parameters are engine-wide: any profile's scorer (they are equal)
      for (const auto& w : np.second.scorers())
        if (auto* ls = dynamic_cast<LatencyScorer*>(w.Scorer_.get())) latency_scorer_ = ls;
    if (latency_scorer_ && !cfg.Profile.producer()) throw SchedulingError("latency-scorer needs a predicted-latency-producer");
    if (cfg.LatencyPredictionInfo && !latency_scorer_)
      throw SchedulingError("SchedulerConfig::LatencyPredictionInfo needs a profile with a latency-scorer");
    c.block_chars = cfg.Prefix.BlockSizeTokens * 4;  // averageCharactersPerToken (types.go:112)
    c.max_blocks = cfg.Prefix.MaxPrefixBlocksToMatch;
    c.lru_capacity_default = cfg.Prefix.LRUCapacityPerServer;
    c.max_endpoints = cfg.MaxEndpoints;
    c.max_adapters = cfg.MaxAdapters;
    c.prefix_capacity = cfg.PrefixCapacity;
    if (cfg.Profile.device_filters().size() > EPPSCORE_MAX_FILTERS) throw SchedulingError("too many device filters");
    CopyProfile(cfg.Profile, &c);
    c.tie_mode = cfg.TieMode;
    c.tie_seed = cfg.TieSeed;
    if (eppscore_create(cfg.Device, &c, &eng_) != EPPSCORE_OK) throw SchedulingError(std::string("eppscore_create: ") + eppscore_last_error(nullptr));
  }

 public:
  ~Scheduler() { eppscore_destroy(eng_); }
  Scheduler(const Scheduler&) = delete;
  Scheduler& operator=(const Scheduler&) = delete;

  // Schedule one request (scheduler.go:54): a batch of one.
  SchedulingResult Schedule(const InferenceRequest& request, const std::vector<Endpoint>& candidateEndpoints) {
    auto res = ScheduleBatch({request}, candidateEndpoints);
    if (!res[0].error.empty()) throw SchedulingError(res[0].error);
    return res[0].result;
  }

  struct BatchItem {
    SchedulingResult result;
    std::string error;  // non-empty ⇒ the reference would have returned this error for that request
  };

  // R concurrent Schedule() calls against the same candidate slice, as ONE engine batch.  The engine's LoRA rows are the
  // batch's own target adapters (PackSnapshot); a batch that targets more adapters than the engine holds (MaxAdapters rounded
  // up to 64) runs as contiguous pieces of requests, each with its own snapshot, and comes back exactly as one batch would:
  // results, top-k lists and PreRequest's inputs in batch order, every request drawing with its index in the whole batch.
  std::vector<BatchItem> ScheduleBatch(const std::vector<InferenceRequest>& requests, const std::vector<Endpoint>& endpoints) {
    const int R = (int)requests.size(), M = (int)endpoints.size();
    if (cfg_.Profiles.empty() && cpu_route_ok_ && R > 0 && M > 0 && R <= cfg_.CpuBatchThreshold)  // scores by name: no pieces
      return ScheduleOnHost(requests, endpoints);
    std::map<unsigned, int64_t> set_base;  // profiles route: requests of each profile set in earlier pieces
    const std::vector<size_t> starts = PieceStarts(requests, endpoints);
    if (starts.size() <= 1)
      return cfg_.Profiles.empty() ? ScheduleBatchSingle(requests, endpoints, 0) : ScheduleBatchProfiles(requests, endpoints, set_base);
    std::vector<BatchItem> out;
    BatchRecord whole;
    for (size_t k = 0; k < starts.size(); k++) {
      const size_t a = starts[k], b = k + 1 < starts.size() ? starts[k + 1] : requests.size();
      const std::vector<InferenceRequest> piece(requests.begin() + (ptrdiff_t)a, requests.begin() + (ptrdiff_t)b);
      auto res = cfg_.Profiles.empty() ? ScheduleBatchSingle(piece, endpoints, (int64_t)a) : ScheduleBatchProfiles(piece, endpoints, set_base);
      for (auto& x : res) out.push_back(std::move(x));
      whole.Append(last_);
    }
    last_ = std::move(whole);
    return out;
  }
  uint64_t CpuRoutedRequests() const { return cpu_routed_; }

 private:
  // The small-batch route: tiny batch, request-independent profile, evaluated on the host (SmallBatchCpu).
  std::vector<BatchItem> ScheduleOnHost(const std::vector<InferenceRequest>& requests, const std::vector<Endpoint>& endpoints) {
    const int R = (int)requests.size();
    std::vector<BatchItem> out((size_t)R);
    last_.Clear(0);
    for (int r = 0; r < R; r++) {
      const std::vector<int> cand = Candidates(cfg_.Profile.filters(), requests[r], endpoints);
      const CpuPick p = cpu_.Schedule(endpoints, requests[r].TargetModel, cfg_.Profile.filters().empty() ? nullptr : &cand);
      if (p.pick < 0) {
        out[r].error = "failed to run scheduler profile '" + cfg_.ProfileName + "'";
        continue;
      }
      ScoredEndpoint se;
      se.Endpoint_ = &endpoints[(size_t)p.pick];
      se.Index = p.pick;
      se.Score = p.score;
      se.TieCount = p.tie_count;
      out[r].result.ProfileResults[cfg_.ProfileName].TargetEndpoints.push_back(se);
      out[r].result.PrimaryProfileName = cfg_.ProfileName;
    }
    cpu_routed_ += (uint64_t)R;
    return out;
  }

  // Where the pieces of a batch start: a new piece begins at the request whose target would be the engine's A_cap + 1st
  // distinct adapter of its piece.  Only targets some endpoint carries (active or waiting) need a row: any other name is in
  // neither map of any endpoint, so its class depends on the capacity rule alone, which the "not a known adapter" row
  // (adapter id -1) scores the same way (lora_affinity.go:84-99).
  std::vector<size_t> PieceStarts(const std::vector<InferenceRequest>& requests, const std::vector<Endpoint>& endpoints) const {
    const size_t cap = (size_t)std::max((cfg_.MaxAdapters + 63) / 64 * 64, 64);  // (the engine takes max_adapters < 1 as 64)
    std::vector<size_t> starts{0};
    std::unordered_set<std::string> targets, carried, piece;
    for (const auto& q : requests) targets.insert(q.TargetModel);
    if (targets.size() <= cap) return starts;
    for (const auto& e : endpoints) {
      for (const auto& kv : e.GetMetrics()->ActiveModels)
        if (targets.count(kv.first)) carried.insert(kv.first);
      for (const auto& kv : e.GetMetrics()->WaitingModels)
        if (targets.count(kv.first)) carried.insert(kv.first);
    }
    for (size_t r = 0; r < requests.size(); r++) {
      const std::string& t = requests[r].TargetModel;
      if (!carried.count(t) || piece.count(t)) continue;
      if (piece.size() == cap) {
        starts.push_back(r);
        piece.clear();
      }
      piece.insert(t);
    }
    return starts;
  }

  // GetBlockSize (endpoints[0]'s CacheBlockSize when autotuning, else the config's) and the prefix blocks a prompt is hashed to
  // (approximateprefix/plugin.go:140-165); stride is the length of a request's row of hashes_out.
  struct PrefixGeometry {
    int block_tokens, max_blocks;
    bool want_prefix;
    int32_t stride;
  };
  PrefixGeometry Geometry(const std::vector<Endpoint>& endpoints) const {
    PrefixGeometry g;
    g.block_tokens = cfg_.Prefix.BlockSizeTokens;
    if (!endpoints.empty() && cfg_.Prefix.AutoTune && endpoints[0].GetMetrics()->CacheBlockSize > 0)
      g.block_tokens = endpoints[0].GetMetrics()->CacheBlockSize;
    g.max_blocks = cfg_.Prefix.MaxPrefixBlocksToMatch;
    if (cfg_.Prefix.MaxPrefixTokensToMatch > 0 && g.block_tokens > 0) g.max_blocks = cfg_.Prefix.MaxPrefixTokensToMatch / g.block_tokens;
    g.want_prefix = g.max_blocks > 0 && g.block_tokens > 0;
    g.stride = g.want_prefix ? g.max_blocks : 1;
    return g;
  }

  // The engine inputs of some rows of a batch, in row order: the prompts, each starting 16-byte aligned (the fast hash path),
  // with 64 bytes of tail; model seeds; adapter ids in the snapshot's dictionary.  With a latency scorer also the latency
  // fold-in's inputs (predictedlatency/plugin.go:276-290, :315-343), which every profile of a call shares.
  struct PackedRequests {
    std::vector<uint8_t> bytes;
    std::vector<int64_t> off;
    std::vector<int32_t> len, adapter, in_tokens;
    std::vector<uint64_t> seed;
    std::vector<double> ttft_slo, tpot_slo;
  };
  PackedRequests Pack(const std::vector<InferenceRequest>& requests, const std::vector<int>& rows) const {
    const size_t n = rows.size();
    PackedRequests p;
    p.off.assign(n + 1, 0);
    p.len.resize(n);
    p.adapter.resize(n);
    p.seed.resize(n);
    if (latency_scorer_) {
      p.in_tokens.resize(n);
      p.ttft_slo.resize(n);
      p.tpot_slo.resize(n);
    }
    size_t total = 64;
    for (int r : rows) total += (requests[(size_t)r].Prompt.size() + 15) / 16 * 16;
    p.bytes.reserve(total);
    for (size_t i = 0; i < n; i++) {
      const InferenceRequest& q = requests[(size_t)rows[i]];
      if (latency_scorer_) {
        p.in_tokens[i] = CountFields(q.Prompt);
        p.ttft_slo[i] = SloHeader(q, "x-slo-ttft-ms");
        p.tpot_slo[i] = SloHeader(q, "x-slo-tpot-ms");
      }
      while (p.bytes.size() % 16) p.bytes.push_back(0);
      p.off[i] = (int64_t)p.bytes.size();
      p.len[i] = (int32_t)q.Prompt.size();
      p.bytes.insert(p.bytes.end(), q.Prompt.begin(), q.Prompt.end());
      p.seed[i] = eppscore_model_seed(q.TargetModel.data(), q.TargetModel.size(), q.CacheSalt.data(), q.CacheSalt.size());
      auto it = adapter_ids_.find(q.TargetModel);
      p.adapter[i] = it == adapter_ids_.end() ? -1 : it->second;
    }
    p.off[n] = (int64_t)p.bytes.size();
    p.bytes.resize(p.bytes.size() + 64, 0);
    return p;
  }
  // An engine batch over a packing: its request fields, and where the engine writes totalBlocks and (when it hashes) the block
  // hashes.  The route sets request_base, cand_mask and the pick outputs.
  static eppscore_batch BatchOf(const PackedRequests& p, const PrefixGeometry& g, uint16_t* total_blocks, uint64_t* hashes_out) {
    eppscore_batch b{};
    b.struct_size = sizeof(b);
    b.R = (int32_t)p.len.size();
    b.prompt_bytes = g.want_prefix ? p.bytes.data() : nullptr;
    b.prompt_off = p.off.data();
    b.prompt_len = p.len.data();
    b.model_seed = p.seed.data();
    b.block_chars = g.block_tokens * 4;
    b.max_blocks = g.max_blocks;
    b.adapter_id = p.adapter.data();
    if (!p.in_tokens.empty()) {
      b.input_tokens = p.in_tokens.data();
      b.ttft_slo = p.ttft_slo.data();
      b.tpot_slo = p.tpot_slo.data();
    }
    b.total_blocks = total_blocks;
    b.hashes_out = g.want_prefix ? hashes_out : nullptr;
    return b;
  }

  // The host filter chain (scheduler_profile.go:130-149) for one request: the positions of `endpoints` it keeps.
  static std::vector<int> Candidates(const std::vector<std::shared_ptr<Filter>>& filters, const InferenceRequest& q,
                                     const std::vector<Endpoint>& endpoints) {
    std::vector<int> cand(endpoints.size());
    std::iota(cand.begin(), cand.end(), 0);
    for (auto& f : filters) {
      cand = f->Filter_(q, endpoints, cand);
      if (cand.empty()) break;
    }
    return cand;
  }
  // The candidate mask of `rows` of `requests` under a profile's host filters, mw words per row.  Its bits are endpoint ids, so
  // an id without an endpoint in this list is never a candidate.
  static std::vector<uint32_t> CandidateMask(const std::vector<std::shared_ptr<Filter>>& filters, const std::vector<InferenceRequest>& requests,
                                             const std::vector<int>& rows, const std::vector<Endpoint>& endpoints, const std::vector<int>& ids,
                                             int mw) {
    std::vector<uint32_t> mask(rows.size() * (size_t)mw, 0u);
    for (size_t i = 0; i < rows.size(); i++)
      for (int m : Candidates(filters, requests[(size_t)rows[i]], endpoints)) mask[i * (size_t)mw + (ids[m] >> 5)] |= 1u << (ids[m] & 31);
    return mask;
  }

  // The endpoint the engine returned as id (pos_of_id: id -> position in the list, -1 for none) as a ScoredEndpoint; `what`
  // ("picked" or "listed") names the engine's error when the id has no endpoint in the list.
  static ScoredEndpoint Scored(int32_t id, double score, const std::vector<Endpoint>& endpoints, const std::vector<int>& pos_of_id,
                               const char* what) {
    if (id >= (int32_t)pos_of_id.size() || pos_of_id[(size_t)id] < 0)
      throw SchedulingError(std::string("engine ") + what + " an endpoint that is not in the candidate list");
    ScoredEndpoint se;
    se.Index = pos_of_id[(size_t)id];
    se.Endpoint_ = &endpoints[(size_t)se.Index];
    se.Score = score;
    return se;
  }
  // Entries 1..k-1 of a request's list from the engine (entry 0 is the pick), onto its TargetEndpoints; -1 past the last candidate.
  static void AppendList(std::vector<ScoredEndpoint>& te, const int32_t* list_ids, const double* list_scores, int k,
                         const std::vector<Endpoint>& endpoints, const std::vector<int>& pos_of_id) {
    for (int i = 1; i < k; i++) {
      if (list_ids[i] < 0) break;
      te.push_back(Scored(list_ids[i], list_scores[i], endpoints, pos_of_id, "listed"));
    }
  }

  std::vector<BatchItem> ScheduleBatchSingle(const std::vector<InferenceRequest>& requests, const std::vector<Endpoint>& endpoints,
                                             int64_t request_base) {
    const int R = (int)requests.size(), M = (int)endpoints.size();
    std::vector<BatchItem> out((size_t)R);
    last_.Clear(cfg_.LatencyPredictionInfo ? (size_t)R : 0);
    if (R == 0) return out;
    if (M == 0) {  // scheduler_profile.go:119-121 → single_profile_handler.go:89-91
      for (auto& o : out) o.error = "failed to run scheduler profile '" + cfg_.ProfileName + "'";
      return out;
    }
    // --- stable endpoint ids: the prefix index refers to endpoints by id (ServerID = NamespacedName, indexer.go:34-35), and
    // neither the order nor the membership of the candidate list is stable between calls (datastore PodList, subsetting:
    // director candidates.go:98).  An endpoint keeps the id it got when it was first seen; the engine's rows are ids, the
    // list's positions are mapped to and from them.  When the list is exactly ids 0..M-1 in order (the common case, and every
    // single-list use) nothing is remapped; a mask is only needed when some row has no endpoint in this list. ---
    std::vector<int> ids;
    int Mx = 0;
    bool identity = MapIds(endpoints, &ids, &Mx);
    identity = identity && Mx == M;
    if (Mx > cfg_.MaxEndpoints) throw SchedulingError("more endpoints than SchedulerConfig.MaxEndpoints");
    if (!identity) remapped_batches_++;
    std::vector<int> pos_of_id((size_t)Mx, -1);
    for (int m = 0; m < M; m++) pos_of_id[(size_t)ids[m]] = m;
    PackSnapshot(endpoints, ids, Mx, requests);
    std::vector<int> rows((size_t)R);
    std::iota(rows.begin(), rows.end(), 0);
    std::vector<uint32_t> mask;
    const bool need_mask = !cfg_.Profile.filters().empty() || Mx != M;  // a pure permutation of the rows has no holes: no mask, the fast path stays
    if (need_mask) mask = CandidateMask(cfg_.Profile.filters(), requests, rows, endpoints, ids, (Mx + 31) / 32);
    const PrefixGeometry g = Geometry(endpoints);
    const PackedRequests p = Pack(requests, rows);
    last_.Fill(requests, g.stride, inflight_, running_);
    std::vector<int32_t> pick((size_t)R), ties((size_t)R);
    std::vector<double> score((size_t)R);
    eppscore_batch b = BatchOf(p, g, last_.nh.data(), last_.hashes.data());
    b.request_base = request_base;
    b.cand_mask = need_mask ? mask.data() : nullptr;
    b.pick = pick.data();
    b.pick_score = score.data();
    b.tie_count = ties.data();
    const int topk = cfg_.Profile.picker().MaxNumOfEndpoints;
    // k > 8: the wide lists, except max-score with seeded-random ties, whose device order puts positions >= 1 of a tie class
    // in priority order where the score map's route has ascending index
    const bool engine_wide = topk > EPPSCORE_MAX_TOPK && EngineHasTopKWide() &&
                             (cfg_.Profile.picker().Mode != EPPSCORE_PICK_MAX_SCORE || cfg_.TieMode == EPPSCORE_TIE_LOWEST_INDEX);
    const bool engine_topk = (topk > 1 && topk <= EPPSCORE_MAX_TOPK && EngineHasTopK()) || engine_wide;
    const int klist = engine_wide ? std::min(topk, cfg_.MaxEndpoints) : topk;  // entries past max_endpoints would all be -1
    std::vector<double> all_scores;
    std::vector<uint16_t> pick_match;  // InOrderPrefixIndex: matchBlocks at each pick before its own Add
    std::vector<int32_t> topk_ids;
    std::vector<double> topk_scores;
    if (engine_topk) {  // the picker's first k endpoints, ordered on the device (eppscore_topk)
      topk_ids.resize((size_t)R * klist);
      topk_scores.resize((size_t)R * klist);
      eppscore_topk t{};
      t.struct_size = sizeof(t);
      t.k = klist;
      t.endpoints = topk_ids.data();
      t.scores = topk_scores.data();
      Check(engine_wide ? eppscore_schedule_batch_topk_wide(eng_, &b, &t) : eppscore_schedule_batch_topk(eng_, &b, &t),
            engine_wide ? "eppscore_schedule_batch_topk_wide" : "eppscore_schedule_batch_topk");
    } else {
      if (topk > 1) {  // k > 8, max-score (seeded-random ties or no wide call): the whole weightedScorePerEndpoint map, NaN for non-candidates (scheduler_profile.go:155-174)
        all_scores.resize((size_t)R * Mx);
        b.scores_out = all_scores.data();
      }
      if (inorder_latency_) {  // ... and each request joins its pick's running-request queue: PreRequest adds nothing more
        const std::vector<int64_t> est = EstimateTokens(R, last_.size.data(), last_.hint.data(), last_.chars.data());
        std::vector<int32_t> caps;
        eppscore_inorder_index x{};
        if (inorder_index_) {
          last_endpoints_ = &endpoints;  // (LruCapacities reads the batch's list)
          last_ids_ = ids;
          last_rows_ = Mx;
          caps = LruCapacities();
          pick_match.assign((size_t)R, 0);
          x.struct_size = sizeof(x);
          x.lru_capacity = caps.data();
          x.pick_match = pick_match.data();
        }
        std::vector<uint64_t> key;
        std::vector<uint8_t> added((size_t)R, 0);
        if (running_) {  // the batch's x-request-ids (KeyFor); no id: key 0, not tracked
          key.assign((size_t)R, 0);
          for (int r = 0; r < R; r++)
            if (!requests[r].RequestId.empty()) key[(size_t)r] = KeyFor(requests[r].RequestId);
        }
        eppscore_inorder_running q{};
        q.struct_size = sizeof(q);
        q.request_key = running_ ? key.data() : nullptr;
        q.added_out = added.data();
        Check(eppscore_schedule_batch_inorder_latency(eng_, &b, est.data(), inorder_index_ ? &x : nullptr, &q),
              "eppscore_schedule_batch_inorder_latency");
        if (running_)
          for (int r = 0; r < R; r++) {
            if (key[(size_t)r] == 0) continue;
            if (added[(size_t)r]) running_keys_[requests[r].RequestId].endpoints.push_back(pick[r]);
            else ReleaseKeyIfUnused(requests[r].RequestId);  // refused (already live there, a negative tpot, or no pick)
          }
      } else if (inorder_index_) {  // ... and each pick's blocks, in request order: PreRequest commits nothing more
        const std::vector<int64_t> est = EstimateTokens(R, last_.size.data(), last_.hint.data(), last_.chars.data());
        last_endpoints_ = &endpoints;  // (LruCapacities reads the batch's list)
        last_ids_ = ids;
        last_rows_ = Mx;
        const std::vector<int32_t> caps = LruCapacities();
        pick_match.assign((size_t)R, 0);
        eppscore_inorder_index x{};
        x.struct_size = sizeof(x);
        x.lru_capacity = caps.data();
        x.pick_match = pick_match.data();
        Check(eppscore_schedule_batch_inorder_index(eng_, &b, est.data(), &x), "eppscore_schedule_batch_inorder_index");
      } else if (inorder_) {  // the estimates go in with the batch: the call adds each pick's load in request order
        const std::vector<int64_t> est = EstimateTokens(R, last_.size.data(), last_.hint.data(), last_.chars.data());
        Check(eppscore_schedule_batch_inorder(eng_, &b, est.data()), "eppscore_schedule_batch_inorder");
      } else {
        Check(eppscore_schedule_batch(eng_, &b), "eppscore_schedule_batch");
      }
    }
    last_endpoints_ = &endpoints;
    last_ids_ = ids;
    last_rows_ = Mx;
    for (int r = 0; r < R; r++) {
      if (pick[r] < 0) {  // "no endpoints available for the given request" → profile result nil → ProcessResults error
        out[r].error = "failed to run scheduler profile '" + cfg_.ProfileName + "'";
        continue;
      }
      ScoredEndpoint se = Scored(pick[r], score[r], endpoints, pos_of_id, "picked");
      se.TieCount = ties[r];
      auto& te = out[r].result.ProfileResults[cfg_.ProfileName].TargetEndpoints;
      te.push_back(se);
      out[r].result.PrimaryProfileName = cfg_.ProfileName;
      if (engine_topk) {
        AppendList(te, topk_ids.data() + (size_t)r * klist, topk_scores.data() + (size_t)r * klist, klist, endpoints, pos_of_id);
      } else if (topk > 1) {  // picker/maxscore/picker.go:104-106: the next best candidates, descending score
        for (const auto& pr : TopK(all_scores.data() + (size_t)r * Mx, Mx, topk)) {  // (id, score), NaN rows skipped
          const int pos = pos_of_id[(size_t)pr.first];
          if (pos < 0 || pos == se.Index) continue;
          if ((int)te.size() >= topk) break;
          ScoredEndpoint o2;
          o2.Endpoint_ = &endpoints[(size_t)pos];
          o2.Index = pos;
          o2.Score = pr.second;
          te.push_back(o2);
        }
      }
    }
    if (inorder_index_ && cfg_.PrefixMatchInfo && g.want_prefix) {  // the target is the only entry (MaxNumOfEndpoints 1)
      if (g.block_tokens > 0xFFFF) throw SchedulingError("PrefixCacheMatchInfo: block size above 65535 tokens");
      for (int r = 0; r < R; r++)
        if (out[r].error.empty())
          out[r].result.ProfileResults[cfg_.ProfileName].TargetEndpoints[0].PrefixMatch =
              PrefixCacheMatchInfo{pick_match[(size_t)r], last_.nh[(size_t)r], (uint16_t)g.block_tokens};
    } else if (cfg_.LatencyPredictionInfo || cfg_.PrefixMatchInfo) {
      TargetRuns runs((size_t)R);
      for (int r = 0; r < R; r++)
        if (out[r].error.empty()) runs[(size_t)r].emplace_back(cfg_.ProfileName, &out[r].result.ProfileResults[cfg_.ProfileName]);
      FillTargetInfo(runs, rows, requests, endpoints, ids, last_.hashes.data(), last_.nh.data(), p, g);
    }
    if (cfg_.LatencyPredictionInfo)
      for (int r = 0; r < R; r++) AttachLatency(out[r], last_.lat[(size_t)r], endpoints, ids);
    return out;
  }

 public:
  // PreRequest for the last ScheduleBatch (approximateprefix/plugin.go:169-197): records the picks in the index, unless
  // InOrderPrefixIndex recorded them while scheduling; with the inflight-load-producer also counts every scheduled request, with
  // its estimated tokens, on its TargetEndpoints[0] (inflightload/producer.go:101-120), unless InOrderInFlightLoad counted it
  // while scheduling.
  void PreRequest(const std::vector<BatchItem>& results) {
    RecordPrefixCacheMatch(results);
    RecordDispatch(results);
    if (!last_endpoints_ || (last_.hashes.empty() && !inflight_ && !running_)) return;
    if (!cfg_.Profiles.empty()) return PreRequestProfiles(results);
    const int R = (int)results.size();
    std::vector<int32_t> pick((size_t)R, -1);
    for (int r = 0; r < R; r++)
      if (results[r].error.empty()) pick[r] = last_ids_[(size_t)results[r].result.ProfileResults.at(cfg_.ProfileName).TargetEndpoints[0].Index];
    if (!last_.hashes.empty() && !inorder_index_)  // (in order against the index: ScheduleBatch committed the batch already)
      Check(eppscore_commit_picks(eng_, R, pick.data(), last_.hashes.data(), last_.nh.data(), last_.stride, LruCapacities().data()),
            "eppscore_commit_picks");
    if (inflight_ && !inorder_ && (int)last_.size.size() == R) {  // (in order: ScheduleBatch added the load already)
      const std::vector<int64_t> est = EstimateTokens(R, last_.size.data(), last_.hint.data(), last_.chars.data());
      Check(eppscore_inflight_add(eng_, R, 0, pick.data(), est.data(), nullptr), "eppscore_inflight_add");
    }
    if (!inorder_latency_) RunningAdd(pick);  // (in order with the running queues: ScheduleBatch added them already)
  }

  // requestcontrol_hooks.go:73-86: (pick[r], request id, tpot) into the running-request queues, for PreRequest
  void RunningAdd(const std::vector<int32_t>& pick) {
    const int R = (int)pick.size();
    if (running_ && (int)last_.rid.size() == R) {
      std::vector<int32_t> ep((size_t)R, -1);
      std::vector<uint64_t> key((size_t)R, 0);
      for (int r = 0; r < R; r++) {
        if (pick[r] < 0 || last_.rid[r].empty()) continue;  // no target / missing x-request-id: not tracked
        ep[r] = pick[r];
        key[r] = KeyFor(last_.rid[r]);
      }
      std::vector<uint8_t> added((size_t)R, 0);
      Check(eppscore_running_add(eng_, R, 0, ep.data(), key.data(), last_.tpot.data(), added.data(), nullptr), "eppscore_running_add");
      for (int r = 0; r < R; r++)
        if (ep[r] >= 0) {
          if (added[r]) running_keys_[last_.rid[r]].endpoints.push_back(ep[r]);
          else ReleaseKeyIfUnused(last_.rid[r]);  // refused (already live there, or a negative tpot)
        }
    }
  }

  // Context TTL expiry (predictedlatency/plugin.go:190-196) for a request PreRequest added: removed from its endpoint's
  // running-request queue, as at the end of the stream.  The caller owns the TTL clock.
  void RequestExpired(const InferenceRequest& request, const SchedulingResult& result) {
    dispatch_.erase(request.RequestId);
    RunningRemove(request, result);
  }

  // ResponseBody at end of stream (inflightload/producer.go:122-169) for a request PreRequest counted, given the result it was
  // scheduled with (the reference reads it from request.SchedulingResult): its TargetEndpoints[0] gives back one request and the
  // request's estimate.  Without the producer, or for a server that has left the pool since (its id may already be another
  // server's), nothing happens.
  void ResponseComplete(const InferenceRequest& request, const SchedulingResult& result) {
    dispatch_.erase(request.RequestId);
    RunningRemove(request, result);  // requestcontrol_hooks.go:219
    if (!cfg_.Profiles.empty()) return ReleaseProfiles(request, result, false);
    if (!inflight_) return;
    auto pr = result.ProfileResults.find(cfg_.ProfileName);
    if (pr == result.ProfileResults.end() || pr->second.TargetEndpoints.empty() || !pr->second.TargetEndpoints[0].Endpoint_) return;
    const int32_t id = ServerId(pr->second.TargetEndpoints[0].Endpoint_->GetMetadata()->NamespacedName_.String());
    if (id < 0) return;
    int64_t size = 0;
    int32_t hint = -1, chars = 0;
    EstimateInputs(request, &size, &hint, &chars);
    const std::vector<int64_t> est = EstimateTokens(1, &size, &hint, &chars);
    Check(eppscore_inflight_release(eng_, 1, 0, &id, est.data(), nullptr), "eppscore_inflight_release");
  }

  // ResponseBody at start of stream (inflightload/producer.go:137-160): with several profiles, the "prefill" profile's target
  // gives back the request; its other targets stay counted until ResponseComplete.  Nothing for a single-profile config.
  void ResponseStarted(const InferenceRequest& request, const SchedulingResult& result) {
    if (!cfg_.Profiles.empty()) ReleaseProfiles(request, result, true);
  }

  // indexer.RemovePod (indexer.go:167-182), called when a model server leaves the pool: its LRU and its memberships go, its
  // id is free for the next new server.  With the inflight-load-producer also DeleteEndpoint (producer.go:181-187), so the next
  // server to get the id starts from 0.
  void RemovePod(const std::string& namespaced_name) {
    auto it = server_ids_.find(namespaced_name);
    if (it == server_ids_.end()) return;
    Check(eppscore_prefix_remove_endpoint(eng_, it->second), "eppscore_prefix_remove_endpoint");
    if (inflight_) Check(eppscore_inflight_remove_endpoint(eng_, it->second), "eppscore_inflight_remove_endpoint");
    if (running_) {  // the engine's one divergence: the recycled id's queue starts empty (include/eppscore.h)
      Check(eppscore_running_remove_endpoint(eng_, it->second), "eppscore_running_remove_endpoint");
      for (auto k = running_keys_.begin(); k != running_keys_.end();) {
        auto& v = k->second.endpoints;
        v.erase(std::remove(v.begin(), v.end(), it->second), v.end());
        k = v.empty() ? running_keys_.erase(k) : std::next(k);
      }
    }
    free_ids_.push_back(it->second);
    server_ids_.erase(it);
  }

  // PrepareRequestData's view (producer.go:90-99) of one server: {requests, tokens} in flight; {0, 0} without the producer or
  // for a server never seen.
  std::pair<int64_t, int64_t> InFlightLoad(const std::string& namespaced_name) {
    const int id = ServerId(namespaced_name);
    if (!inflight_ || id < 0) return {0, 0};
    std::vector<int64_t> req((size_t)id + 1), tok((size_t)id + 1);
    Check(eppscore_inflight_get(eng_, req.data(), tok.data(), id + 1), "eppscore_inflight_get");
    return {req[(size_t)id], tok[(size_t)id]};
  }
  // getEndpointMinTPOTSLO / getEndpointRunningRequestCount (plugin.go:347-363) of one server from the engine's queues:
  // {0, 0} without TrackRunningRequests or for a server never seen.
  std::pair<double, int32_t> RunningRequests(const std::string& namespaced_name) {
    const int id = ServerId(namespaced_name);
    if (!running_ || id < 0) return {0.0, 0};
    std::vector<double> mn((size_t)id + 1);
    std::vector<int32_t> cnt((size_t)id + 1);
    Check(eppscore_running_get(eng_, mn.data(), cnt.data(), id + 1), "eppscore_running_get");
    return {mn[(size_t)id], cnt[(size_t)id]};
  }
  size_t TrackedRequestIds() const { return running_keys_.size(); }  // ids with a live queue entry (their keys are kept)
  int ServerId(const std::string& namespaced_name) const {  // -1: never seen (or removed)
    auto it = server_ids_.find(namespaced_name);
    return it == server_ids_.end() ? -1 : it->second;
  }
  uint64_t RemappedBatches() const { return remapped_batches_; }  // batches whose list was not ids 0..M-1 in order

  const std::vector<uint16_t>& LastTotalBlocks() const { return last_.nh; }
  // The prefix-indexer histograms PreRequest records with SchedulerConfig::PrefixMatchInfo (empty without it).
  const PrefixIndexerHistograms& PrefixIndexerMetrics() const { return prefix_metrics_; }
  // The dispatch record PreRequest kept for a request id with SchedulerConfig::LatencyPredictionInfo, or nullptr (none kept, or
  // dropped at ResponseComplete / RequestExpired).
  const epp::PredictedLatencyAtDispatch* PredictedLatencyAtDispatch(const std::string& request_id) const {
    auto it = dispatch_.find(request_id);
    return it == dispatch_.end() ? nullptr : &it->second;
  }
  size_t TrackedDispatches() const { return dispatch_.size(); }

  eppscore_engine* engine() { return eng_; }

 private:
  // Per row of an engine call, the (profile name, result) pairs of every profile that ran for the row's request.
  using TargetRuns = std::vector<std::vector<std::pair<std::string, ProfileRunResult*>>>;

  // After an engine call: every TargetEndpoints entry of `runs` (row i is requests[rows[i]], packed as p) gets its
  // LatencyPredictionInfo with SchedulerConfig::LatencyPredictionInfo, and its PrefixCacheMatchInfo with
  // SchedulerConfig::PrefixMatchInfo when the call hashed the prompts into hashes / nh.
  void FillTargetInfo(const TargetRuns& runs, const std::vector<int>& rows, const std::vector<InferenceRequest>& requests,
                      const std::vector<Endpoint>& endpoints, const std::vector<int>& ids, const uint64_t* hashes, const uint16_t* nh,
                      const PackedRequests& p, const PrefixGeometry& g) {
    if (cfg_.LatencyPredictionInfo)
      FillLatency(runs, rows, requests, endpoints, ids, hashes, nh, p, g, cfg_.PrefixMatchInfo && g.want_prefix);
    else if (cfg_.PrefixMatchInfo && g.want_prefix)
      FillPrefixMatch(runs, hashes, nh, ids, g);
  }

  // One eppscore_prefix_match call for an engine call that hashed its prompts: hashes / nh its hashes_out and total_blocks, ids
  // the list position -> endpoint id map.  Each TargetEndpoints entry of `runs` gets {matchBlocks at its endpoint, totalBlocks,
  // the batch's block size} (plugin.go:140-153).  A request's endpoints are listed once each, so k never passes the number of
  // endpoint rows.
  void FillPrefixMatch(const TargetRuns& runs, const uint64_t* hashes, const uint16_t* nh, const std::vector<int>& ids,
                       const PrefixGeometry& g) {
    const int n = (int)runs.size();
    std::vector<std::vector<int32_t>> cols((size_t)n);
    size_t k = 0;
    for (int i = 0; i < n; i++) {
      for (const auto& run : runs[(size_t)i])
        for (const ScoredEndpoint& t : run.second->TargetEndpoints) {
          const int32_t id = ids[(size_t)t.Index];
          if (std::find(cols[(size_t)i].begin(), cols[(size_t)i].end(), id) == cols[(size_t)i].end()) cols[(size_t)i].push_back(id);
        }
      k = std::max(k, cols[(size_t)i].size());
    }
    if (n == 0 || k == 0) return;
    if (g.block_tokens > 0xFFFF) throw SchedulingError("PrefixCacheMatchInfo: block size above 65535 tokens");
    std::vector<int32_t> eps((size_t)n * k, -1);
    for (int i = 0; i < n; i++) std::copy(cols[(size_t)i].begin(), cols[(size_t)i].end(), eps.begin() + (ptrdiff_t)((size_t)i * k));
    std::vector<uint16_t> match((size_t)n * k, 0);
    Check(eppscore_prefix_match(eng_, n, (int32_t)k, 0, hashes, nh, g.stride, eps.data(), match.data(), nullptr), "eppscore_prefix_match");
    for (int i = 0; i < n; i++)
      for (const auto& run : runs[(size_t)i])
        for (ScoredEndpoint& t : run.second->TargetEndpoints) {
          const auto& c = cols[(size_t)i];
          const size_t j = (size_t)(std::find(c.begin(), c.end(), ids[(size_t)t.Index]) - c.begin());
          t.PrefixMatch = PrefixCacheMatchInfo{match[(size_t)i * k + j], nh[i], (uint16_t)g.block_tokens};
        }
  }

  // A batch row's share of the predicted-latency producer's request context: the request id and SLOs, the info of every endpoint
  // a profile chose for it (by endpoint id), and the values predictionsForScheduling / prefixCacheScoresForEndpoints hold.
  // Those are keyed by NamespacedName.Name (predictedlatency/preparedata_hooks.go:36-106), so of two candidates with one name
  // the later one's values stand for both.  The prefix cache score is match / total whether or not a prediction was stored:
  // PrepareRequestData fills it before, and independently of, the prediction branch (preparedata_hooks.go:42-58).
  struct LatencyCtx {
    bool set = false;
    std::string rid;
    double ttft_slo = 0.0, tpot_slo = 0.0;
    std::map<int32_t, std::optional<LatencyPredictionInfo>> by_id;  // endpoint id -> its info
    std::map<std::string, std::pair<std::optional<LatencyPredictionInfo>, double>> by_name;  // Name -> (info, prefix score)
  };

  // What the last engine batch leaves for PreRequest, per request in batch order.  PreRequest checks the sizes: the estimator
  // inputs are filled only with the inflight-load producer, the request ids and TPOT SLOs only with TrackRunningRequests, and a
  // batch that returns before Fill (no requests, no endpoints on the single route, the small-batch host route) leaves them as
  // they were.
  struct BatchRecord {
    std::vector<uint64_t> hashes;  // the engine's hashes_out, stride per request
    std::vector<uint16_t> nh;      // its total_blocks
    int32_t stride = 1;
    std::vector<int64_t> size;     // SimpleTokenEstimator's inputs (EstimateInputs)
    std::vector<int32_t> hint, chars;
    std::vector<std::string> rid;  // the request id and avgTPOTSLO (x-slo-tpot-ms)
    std::vector<double> tpot;
    std::vector<LatencyCtx> lat;   // SchedulerConfig::LatencyPredictionInfo

    void Clear(size_t lat_rows) {
      hashes.clear();
      nh.clear();
      lat.assign(lat_rows, LatencyCtx{});
    }
    void Fill(const std::vector<InferenceRequest>& requests, int32_t hash_stride, bool inflight, bool running) {
      const size_t R = requests.size();
      stride = hash_stride;
      nh.assign(R, 0);
      hashes.assign(R * (size_t)stride, 0);
      if (inflight) {
        size.resize(R);
        hint.resize(R);
        chars.resize(R);
        for (size_t r = 0; r < R; r++) EstimateInputs(requests[r], &size[r], &hint[r], &chars[r]);
      }
      if (running) {
        rid.resize(R);
        tpot.resize(R);
        for (size_t r = 0; r < R; r++) {
          rid[r] = requests[r].RequestId;
          tpot[r] = SloHeader(requests[r], "x-slo-tpot-ms");
        }
      }
    }
    // A later piece of the same batch.
    void Append(BatchRecord& piece) {
      auto append = [](auto& to, auto& from) { to.insert(to.end(), std::make_move_iterator(from.begin()), std::make_move_iterator(from.end())); };
      append(hashes, piece.hashes);
      append(nh, piece.nh);
      stride = piece.stride;
      append(size, piece.size);
      append(hint, piece.hint);
      append(chars, piece.chars);
      append(rid, piece.rid);
      append(tpot, piece.tpot);
      append(lat, piece.lat);
    }
  };

  // The final result's SchedulingResult::TargetLatency from the row's LatencyCtx: every profile's TargetEndpoints, in the order
  // the result holds them (after ProcessResults), looked up by endpoint id.
  void AttachLatency(BatchItem& it, const LatencyCtx& ctx, const std::vector<Endpoint>& endpoints, const std::vector<int>& ids) const {
    if (!ctx.set || !it.error.empty()) return;
    for (const auto& kv : it.result.ProfileResults) {
      auto& tl = it.result.TargetLatency[kv.first];
      tl.clear();
      for (const ScoredEndpoint& t : kv.second.TargetEndpoints) {
        const bool in_list = t.Index >= 0 && (size_t)t.Index < endpoints.size() && t.Endpoint_ == &endpoints[(size_t)t.Index];
        const auto f = in_list ? ctx.by_id.find(ids[(size_t)t.Index]) : ctx.by_id.end();
        tl.push_back(f == ctx.by_id.end() ? std::nullopt : f->second);
      }
    }
  }

  // One eppscore_predict_latency call for an engine call: runs[i] are row i's (profile name, result) pairs (rows[i] its index in
  // `requests`, p its packing), hashes / nh the call's hashes_out and total_blocks (all zero when the engine did not hash), ids
  // the list position -> endpoint id map.  Every TargetEndpoints entry's LatencyPredictionInfo goes into the row's LatencyCtx (AttachLatency
  // puts it on the final result); with fill_match the entry also gets its PrefixMatch (as FillPrefixMatch gives it).  The row's
  // LatencyCtx also gets each target name's values at the last candidate of that name.
  void FillLatency(const TargetRuns& runs, const std::vector<int>& rows, const std::vector<InferenceRequest>& requests,
                   const std::vector<Endpoint>& endpoints, const std::vector<int>& ids, const uint64_t* hashes, const uint16_t* nh,
                   const PackedRequests& p, const PrefixGeometry& g, bool fill_match) {
    const int n = (int)runs.size();
    std::map<std::string, int> last_of_name;  // Name -> the last candidate position with it
    for (size_t m = 0; m < endpoints.size(); m++) last_of_name[endpoints[m].GetMetadata()->NamespacedName_.Name] = (int)m;
    std::vector<std::vector<int32_t>> cols((size_t)n);
    auto col_of = [&](int i, int32_t id) {
      auto& c = cols[(size_t)i];
      const auto it = std::find(c.begin(), c.end(), id);
      if (it != c.end()) return (size_t)(it - c.begin());
      c.push_back(id);
      return c.size() - 1;
    };
    size_t k = 0;
    for (int i = 0; i < n; i++) {
      for (const auto& run : runs[(size_t)i])
        for (const ScoredEndpoint& t : run.second->TargetEndpoints) {
          col_of(i, ids[(size_t)t.Index]);
          col_of(i, ids[(size_t)last_of_name[endpoints[(size_t)t.Index].GetMetadata()->NamespacedName_.Name]]);
        }
      k = std::max(k, cols[(size_t)i].size());
    }
    if (n == 0 || k == 0) return;
    if (fill_match && g.block_tokens > 0xFFFF) throw SchedulingError("PrefixCacheMatchInfo: block size above 65535 tokens");
    std::vector<int32_t> eps((size_t)n * k, -1);
    for (int i = 0; i < n; i++) std::copy(cols[(size_t)i].begin(), cols[(size_t)i].end(), eps.begin() + (ptrdiff_t)((size_t)i * k));
    std::vector<eppscore_latency_info> info((size_t)n * k);
    std::vector<uint16_t> match((size_t)n * k);  // (also the prefix cache score when no prediction was stored)
    Check(eppscore_predict_latency(eng_, n, (int32_t)k, 0, hashes, nh, g.stride, p.in_tokens.data(), p.ttft_slo.data(), p.tpot_slo.data(),
                                   eps.data(), info.data(), match.data(), nullptr),
          "eppscore_predict_latency");
    auto as_info = [](const eppscore_latency_info& x) -> std::optional<LatencyPredictionInfo> {
      if (!x.present) return std::nullopt;
      LatencyPredictionInfo v;
      v.TTFTValid = x.ttft_valid != 0;
      v.TPOTValid = x.tpot_valid != 0;
      v.TTFTHeadroom = x.ttft_headroom;
      v.TPOTHeadroom = x.tpot_headroom;
      v.TTFT = x.ttft;
      v.TPOT = x.tpot;
      v.DispatchedRequestCount = x.dispatched;
      return v;
    };
    for (int i = 0; i < n; i++) {
      const InferenceRequest& q = requests[(size_t)rows[(size_t)i]];
      LatencyCtx& ctx = last_.lat[(size_t)rows[(size_t)i]];
      ctx.set = true;
      ctx.rid = q.RequestId;
      ctx.ttft_slo = p.ttft_slo[(size_t)i];
      ctx.tpot_slo = p.tpot_slo[(size_t)i];
      for (const auto& run : runs[(size_t)i]) {
        for (ScoredEndpoint& t : run.second->TargetEndpoints) {
          const int32_t id = ids[(size_t)t.Index];
          const size_t j = (size_t)i * k + col_of(i, id);
          ctx.by_id[id] = as_info(info[j]);
          if (fill_match) t.PrefixMatch = PrefixCacheMatchInfo{match[j], nh[i], (uint16_t)g.block_tokens};
          const std::string& name = endpoints[(size_t)t.Index].GetMetadata()->NamespacedName_.Name;
          const size_t a = (size_t)i * k + col_of(i, ids[(size_t)last_of_name[name]]);
          const double score = nh[i] ? (double)match[a] / (double)nh[i] : 0.0;  // match/total, NaN (0/0) => 0
          ctx.by_name[name] = {as_info(info[a]), score};
        }
      }
    }
  }

  // PreRequest's dispatch record (requestcontrol_hooks.go:236-251, :309-321), per request with an id, from the batch's LatencyCtx:
  // TTFT and prefix score at the "prefill" profile's target when it has one, else at the primary target; TPOT at the primary.
  void RecordDispatch(const std::vector<BatchItem>& results) {
    if (!cfg_.LatencyPredictionInfo) return;
    for (size_t r = 0; r < results.size() && r < last_.lat.size(); r++) {
      const LatencyCtx& ctx = last_.lat[r];
      const BatchItem& it = results[r];
      if (!ctx.set || ctx.rid.empty() || !it.error.empty()) continue;
      auto target = [&](const std::string& profile) -> const Endpoint* {
        auto pr = it.result.ProfileResults.find(profile);
        if (pr == it.result.ProfileResults.end() || pr->second.TargetEndpoints.empty()) return nullptr;
        return pr->second.TargetEndpoints[0].Endpoint_;
      };
      auto values = [&](const Endpoint* ep) -> const std::pair<std::optional<LatencyPredictionInfo>, double>* {
        if (!ep) return nullptr;
        auto v = ctx.by_name.find(ep->GetMetadata()->NamespacedName_.Name);
        return v == ctx.by_name.end() ? nullptr : &v->second;
      };
      const Endpoint* primary = target(it.result.PrimaryProfileName);
      const Endpoint* prefill = target("prefill");
      epp::PredictedLatencyAtDispatch d;
      d.TTFTSLO = ctx.ttft_slo;
      d.AvgTPOTSLO = ctx.tpot_slo;
      if (const auto* v = values(prefill ? prefill : primary)) {
        if (v->first) d.PredictedTTFT = v->first->TTFT;
        d.PrefixCacheScore = v->second;
      }
      if (const auto* v = values(primary))
        if (v->first) d.FirstPredictedTPOT = v->first->TPOT;
      dispatch_[ctx.rid] = d;
    }
  }

  // PreRequest's metrics (approximateprefix/plugin.go:199-204): per request with a primary target that carries its match, in
  // request order, RecordPrefixCacheMatch(matchLen * blockSize * 4, total * blockSize * 4) with GetBlockSize of the primary
  // profile's TargetEndpoints (the target's CacheBlockSize when autotuning); the ratio only when the total is > 0.
  void RecordPrefixCacheMatch(const std::vector<BatchItem>& results) {
    for (const BatchItem& it : results) {
      if (!it.error.empty()) continue;
      auto pr = it.result.ProfileResults.find(it.result.PrimaryProfileName);
      if (pr == it.result.ProfileResults.end() || pr->second.TargetEndpoints.empty()) continue;
      const ScoredEndpoint& t = pr->second.TargetEndpoints[0];
      if (!t.PrefixMatch || !t.Endpoint_) continue;
      int64_t bs = cfg_.Prefix.BlockSizeTokens;
      if (cfg_.Prefix.AutoTune && t.Endpoint_->GetMetrics()->CacheBlockSize > 0) bs = t.Endpoint_->GetMetrics()->CacheBlockSize;
      const int64_t matched = (int64_t)t.PrefixMatch->MatchBlocks * bs * 4, total = (int64_t)t.PrefixMatch->TotalBlocks * bs * 4;
      prefix_metrics_.HitBytes.Observe((double)matched);
      if (total > 0) prefix_metrics_.HitRatio.Observe((double)matched / (double)total);
    }
  }

  // x-slo-ttft-ms / x-slo-tpot-ms (predictedlatency/plugin.go:276-290): a parse error gives 0 (logged only)
  static double SloHeader(const InferenceRequest& q, const char* key) {
    auto it = q.Headers.find(key);
    if (it == q.Headers.end()) return 0.0;
    char* end = nullptr;
    const double v = strtod(it->second.c_str(), &end);
    return (end && *end == 0 && end != it->second.c_str()) ? v : 0.0;
  }

  // Exact request keys: x-request-id -> uint64 from 1, kept while the id has a live queue entry on some endpoint (the same id
  // may be live on two endpoints, as queues are per endpoint in the reference).
  struct KeyUse {
    uint64_t key;
    std::vector<int32_t> endpoints;  // where the id is live
  };
  uint64_t KeyFor(const std::string& rid) {
    auto it = running_keys_.find(rid);
    if (it != running_keys_.end()) return it->second.key;
    const uint64_t k = next_key_++;
    running_keys_.emplace(rid, KeyUse{k, {}});
    return k;
  }
  void ReleaseKeyIfUnused(const std::string& rid) {
    auto it = running_keys_.find(rid);
    if (it != running_keys_.end() && it->second.endpoints.empty()) running_keys_.erase(it);
  }
  // removes (the primary profile's TargetEndpoints[0], request id) from the queues; nothing for an untracked id or a server that
  // has left
  void RunningRemove(const InferenceRequest& request, const SchedulingResult& result) {
    if (!running_ || request.RequestId.empty()) return;
    auto k = running_keys_.find(request.RequestId);
    if (k == running_keys_.end()) return;
    auto pr = result.ProfileResults.find(cfg_.Profiles.empty() ? cfg_.ProfileName : result.PrimaryProfileName);
    if (pr == result.ProfileResults.end() || pr->second.TargetEndpoints.empty() || !pr->second.TargetEndpoints[0].Endpoint_) return;
    const int32_t id = ServerId(pr->second.TargetEndpoints[0].Endpoint_->GetMetadata()->NamespacedName_.String());
    auto& v = k->second.endpoints;
    if (id < 0 || std::find(v.begin(), v.end(), id) == v.end()) return;
    const uint64_t key = k->second.key;
    uint8_t removed = 0;
    Check(eppscore_running_remove(eng_, 1, 0, &id, &key, &removed, nullptr), "eppscore_running_remove");
    v.erase(std::find(v.begin(), v.end(), id));
    if (v.empty()) running_keys_.erase(k);
  }

  // The batch route with several profiles: the handler's first Pick per request on the host, then ONE
  // eppscore_schedule_batch_profiles call per distinct set of picked profiles (one hash pass for all of the set's profiles), then
  // ProcessResults.  A handler that asks for a second round gets that request's error.  Request i of a set's call draws with
  // index set_base[set] + i; set_base counts each set's requests in the earlier pieces of a batch, and is advanced here.
  std::vector<BatchItem> ScheduleBatchProfiles(const std::vector<InferenceRequest>& requests, const std::vector<Endpoint>& endpoints,
                                               std::map<unsigned, int64_t>& set_base) {
    const int R = (int)requests.size(), M = (int)endpoints.size(), P = (int)cfg_.Profiles.size();
    std::vector<BatchItem> out((size_t)R);
    last_.Clear(cfg_.LatencyPredictionInfo ? (size_t)R : 0);
    if (R == 0) return out;
    std::vector<std::string> names;
    for (const auto& np : cfg_.Profiles) names.push_back(np.first);
    std::vector<unsigned> sets((size_t)R, 0u);
    for (int r = 0; r < R; r++)
      for (const std::string& n : cfg_.Handler->Pick(requests[r], names, {})) {
        const auto it = std::find(names.begin(), names.end(), n);
        if (it == names.end()) out[r].error = "profile '" + n + "' is not defined";
        else sets[r] |= 1u << (it - names.begin());
      }
    std::vector<int> ids;
    int Mx = 0;
    if (M > 0) {
      MapIds(endpoints, &ids, &Mx);
      if (Mx > cfg_.MaxEndpoints) throw SchedulingError("more endpoints than SchedulerConfig.MaxEndpoints");
    }
    const int mw = (Mx + 31) / 32;
    if (M > 0) {
      for (int p = 0; p < P; p++) {  // the request-independent filters: each profile's endpoint subset, applied with the snapshot
        const auto& keep = cfg_.Profiles[(size_t)p].second.endpoint_subset();
        std::vector<uint32_t> row((size_t)std::max(mw, 1), 0u);
        if (keep)
          for (int m = 0; m < M; m++)
            if (keep(endpoints[(size_t)m])) row[(size_t)ids[m] >> 5] |= 1u << (ids[m] & 31);
        Check(eppscore_set_profile_endpoints(eng_, p, keep ? row.data() : nullptr, mw), "eppscore_set_profile_endpoints");
      }
      PackSnapshot(endpoints, ids, Mx, requests);
    }
    std::vector<int> pos_of_id((size_t)Mx, -1);
    for (int m = 0; m < M; m++) pos_of_id[(size_t)ids[m]] = m;
    const PrefixGeometry g = Geometry(endpoints);
    last_.Fill(requests, g.stride, inflight_, running_);
    // every profile's result per request (empty TargetEndpoints: the profile ran and found no endpoint)
    std::vector<std::map<std::string, ProfileRunResult>> got((size_t)R);
    std::vector<unsigned> distinct;
    for (int r = 0; r < R; r++)
      if (out[r].error.empty() && sets[r] && std::find(distinct.begin(), distinct.end(), sets[r]) == distinct.end()) distinct.push_back(sets[r]);
    if (inorder_) {
      if (M > 0) ScheduleInOrderProfiles(requests, endpoints, sets, out, got, ids, Mx, mw, g, set_base);
      distinct.clear();
    }
    for (unsigned S : distinct) {
      if (M == 0) break;  // no endpoints: every profile fails (scheduler_profile.go:119-121)
      std::vector<int> rows;
      for (int r = 0; r < R; r++)
        if (out[r].error.empty() && sets[r] == S) rows.push_back(r);
      const int n = (int)rows.size();
      const PackedRequests packed = Pack(requests, rows);
      std::vector<uint64_t> hashes((size_t)n * g.stride, 0);
      std::vector<uint16_t> nh((size_t)n, 0);
      std::vector<int> prof;
      for (int p = 0; p < P; p++)
        if (S & (1u << p)) prof.push_back(p);
      const int nr = (int)prof.size();
      std::vector<std::vector<uint32_t>> masks((size_t)nr);
      std::vector<std::vector<int32_t>> pick((size_t)nr, std::vector<int32_t>((size_t)n)), ties = pick;
      std::vector<std::vector<double>> score((size_t)nr, std::vector<double>((size_t)n));
      std::vector<eppscore_profile_run> runs((size_t)nr);
      // maxNumOfEndpoints per profile: entries past max_endpoints would all be -1
      std::vector<eppscore_topk> topk((size_t)nr);
      std::vector<std::vector<int32_t>> list_ids((size_t)nr);
      std::vector<std::vector<double>> list_scores((size_t)nr);
      bool lists = false;
      for (int k = 0; k < nr; k++) {
        const int kl = std::min(cfg_.Profiles[(size_t)prof[k]].second.picker().MaxNumOfEndpoints, cfg_.MaxEndpoints);
        eppscore_topk& t = topk[(size_t)k];
        t = eppscore_topk{};
        t.struct_size = sizeof(t);
        if (kl <= 1) continue;
        lists = true;
        list_ids[k].assign((size_t)n * kl, -1);
        list_scores[k].assign((size_t)n * kl, 0.0);
        t.k = kl;
        t.endpoints = list_ids[k].data();
        t.scores = list_scores[k].data();
      }
      for (int k = 0; k < nr; k++) {
        const auto& filters = cfg_.Profiles[(size_t)prof[k]].second.filters();
        eppscore_profile_run& x = runs[(size_t)k];
        x = eppscore_profile_run{};
        x.struct_size = sizeof(x);
        x.profile = prof[k];
        if (!filters.empty() || Mx != M) {  // host filters and rows without an endpoint in this list
          masks[k] = CandidateMask(filters, requests, rows, endpoints, ids, mw);
          x.cand_mask = masks[k].data();
        }
        x.pick = pick[k].data();
        x.pick_score = score[k].data();
        x.tie_count = ties[k].data();
      }
      eppscore_batch b = BatchOf(packed, g, nh.data(), hashes.data());
      b.request_base = set_base[S];
      set_base[S] += n;
      if (lists)
        Check(eppscore_schedule_batch_profiles_topk(eng_, &b, nr, runs.data(), topk.data()), "eppscore_schedule_batch_profiles_topk");
      else
        Check(eppscore_schedule_batch_profiles(eng_, &b, nr, runs.data()), "eppscore_schedule_batch_profiles");
      for (int i = 0; i < n; i++) {
        const int r = rows[i];
        last_.nh[(size_t)r] = nh[i];
        std::copy(hashes.begin() + (size_t)i * g.stride, hashes.begin() + (size_t)(i + 1) * g.stride, last_.hashes.begin() + (size_t)r * g.stride);
        for (int k = 0; k < nr; k++) {
          ProfileRunResult& pr = got[(size_t)r][names[(size_t)prof[k]]];
          const int32_t id = pick[k][i];
          if (id < 0) continue;
          ScoredEndpoint se = Scored(id, score[k][i], endpoints, pos_of_id, "picked");
          se.TieCount = ties[k][i];
          pr.TargetEndpoints.push_back(se);
          const int kl = topk[(size_t)k].k;
          AppendList(pr.TargetEndpoints, list_ids[k].data() + (size_t)i * kl, list_scores[k].data() + (size_t)i * kl, kl, endpoints, pos_of_id);
        }
      }
      if (cfg_.LatencyPredictionInfo || cfg_.PrefixMatchInfo) {  // every run's entries of this call's requests, before the next piece's snapshot
        TargetRuns truns((size_t)n);
        for (int i = 0; i < n; i++)
          for (int k = 0; k < nr; k++) {
            auto it = got[(size_t)rows[i]].find(names[(size_t)prof[k]]);
            if (it != got[(size_t)rows[i]].end()) truns[(size_t)i].emplace_back(it->first, &it->second);
          }
        FillTargetInfo(truns, rows, requests, endpoints, ids, hashes.data(), nh.data(), packed, g);
      }
    }
    for (int r = 0; r < R; r++) {
      if (!out[r].error.empty()) continue;
      std::map<std::string, const ProfileRunResult*> res;
      for (int p = 0; p < P; p++) {
        if (!(sets[r] & (1u << p))) continue;
        auto it = got[(size_t)r].find(names[(size_t)p]);
        res[names[(size_t)p]] = (it != got[(size_t)r].end() && !it->second.TargetEndpoints.empty()) ? &it->second : nullptr;
      }
      if (!cfg_.Handler->Pick(requests[r], names, res).empty()) {
        out[r].error = "multi-round profile handlers are not supported by the batch route";
        continue;
      }
      try {
        out[r].result = cfg_.Handler->ProcessResults(requests[r], res);
      } catch (const SchedulingError& ex) {
        out[r].error = ex.what();
      }
      if (inorder_ && out[r].error.empty() && out[r].result.PrimaryProfileName != names[0])  // (its load and Adds are at names[0]'s target)
        out[r].error = "the in-order batch route records PreRequest at the first profile's target ('" + names[0] +
                       "'), but ProcessResults named '" + out[r].result.PrimaryProfileName + "' the primary profile";
      if (cfg_.LatencyPredictionInfo) AttachLatency(out[r], last_.lat[(size_t)r], endpoints, ids);
    }
    last_endpoints_ = &endpoints;
    last_ids_ = ids;
    last_rows_ = Mx;
    return out;
  }

  // The in-order form of ScheduleBatchProfiles (SchedulerConfig::InOrderInFlightLoad): the requests the handler gave a profile
  // set go through ONE eppscore_schedule_batch_inorder_profiles call, every profile a run (run i = profile i), with the set as
  // each request's run mask; the index form with InOrderPrefixIndex.  Fills got[r] for the profiles of request r's set.
  void ScheduleInOrderProfiles(const std::vector<InferenceRequest>& requests, const std::vector<Endpoint>& endpoints,
                               const std::vector<unsigned>& sets, const std::vector<BatchItem>& out,
                               std::vector<std::map<std::string, ProfileRunResult>>& got, const std::vector<int>& ids, int Mx, int mw,
                               const PrefixGeometry& g, std::map<unsigned, int64_t>& set_base) {
    const int R = (int)requests.size(), P = (int)cfg_.Profiles.size(), M = (int)endpoints.size();
    std::vector<int> rows;
    for (int r = 0; r < R; r++)
      if (out[r].error.empty() && sets[r]) rows.push_back(r);
    const int n = (int)rows.size();
    if (n == 0) return;
    std::vector<int> pos_of_id((size_t)Mx, -1);
    for (int m = 0; m < M; m++) pos_of_id[(size_t)ids[m]] = m;
    const PackedRequests packed = Pack(requests, rows);
    std::vector<uint64_t> hashes((size_t)n * g.stride, 0);
    std::vector<uint16_t> nh((size_t)n, 0);
    std::vector<std::vector<uint32_t>> masks((size_t)P);
    std::vector<std::vector<int32_t>> pick((size_t)P, std::vector<int32_t>((size_t)n)), ties = pick;
    std::vector<std::vector<double>> score((size_t)P, std::vector<double>((size_t)n));
    std::vector<std::vector<uint16_t>> match((size_t)P, std::vector<uint16_t>((size_t)n, 0));
    std::vector<eppscore_profile_run> runs((size_t)P);
    eppscore_inorder_profiles x{};
    x.struct_size = sizeof(x);
    x.index = inorder_index_ ? 1 : 0;
    x.primary_run = 0;
    x.prefill_run = -1;
    for (int p = 0; p < P; p++) {
      if (cfg_.Profiles[(size_t)p].first == "prefill") x.prefill_run = p;
      eppscore_profile_run& u = runs[(size_t)p];
      u = eppscore_profile_run{};
      u.struct_size = sizeof(u);
      u.profile = p;
      const auto& filters = cfg_.Profiles[(size_t)p].second.filters();
      if (!filters.empty() || Mx != M) {  // host filters and rows without an endpoint in this list
        masks[(size_t)p] = CandidateMask(filters, requests, rows, endpoints, ids, mw);
        u.cand_mask = masks[(size_t)p].data();
      }
      u.pick = pick[(size_t)p].data();
      u.pick_score = score[(size_t)p].data();
      u.tie_count = ties[(size_t)p].data();
      x.pick_match[p] = match[(size_t)p].data();
    }
    std::vector<uint8_t> run_mask((size_t)n);
    std::vector<int64_t> size((size_t)n);
    std::vector<int32_t> hint((size_t)n), chars((size_t)n);
    for (int i = 0; i < n; i++) {
      run_mask[(size_t)i] = (uint8_t)sets[(size_t)rows[i]];
      size[(size_t)i] = last_.size[(size_t)rows[i]];
      hint[(size_t)i] = last_.hint[(size_t)rows[i]];
      chars[(size_t)i] = last_.chars[(size_t)rows[i]];
    }
    x.run_mask = run_mask.data();
    last_endpoints_ = &endpoints;  // (LruCapacities reads the batch's list)
    last_ids_ = ids;
    last_rows_ = Mx;
    const std::vector<int32_t> caps = LruCapacities();
    if (inorder_index_) x.lru_capacity = caps.data();
    const std::vector<int64_t> est = EstimateTokens(n, size.data(), hint.data(), chars.data());
    eppscore_batch b = BatchOf(packed, g, nh.data(), hashes.data());
    b.request_base = set_base[0u];  // (no profile set is 0: one count for the in-order calls of a batch)
    set_base[0u] += n;
    Check(eppscore_schedule_batch_inorder_profiles(eng_, &b, est.data(), P, runs.data(), &x), "eppscore_schedule_batch_inorder_profiles");
    const bool with_match = inorder_index_ && cfg_.PrefixMatchInfo && g.want_prefix;
    if (with_match && g.block_tokens > 0xFFFF) throw SchedulingError("PrefixCacheMatchInfo: block size above 65535 tokens");
    for (int i = 0; i < n; i++) {
      const int r = rows[i];
      last_.nh[(size_t)r] = nh[(size_t)i];
      std::copy(hashes.begin() + (size_t)i * g.stride, hashes.begin() + (size_t)(i + 1) * g.stride, last_.hashes.begin() + (size_t)r * g.stride);
      for (int p = 0; p < P; p++) {
        if (!(sets[(size_t)r] & (1u << p))) continue;
        ProfileRunResult& pr = got[(size_t)r][cfg_.Profiles[(size_t)p].first];
        const int32_t id = pick[(size_t)p][(size_t)i];
        if (id < 0) continue;
        ScoredEndpoint se = Scored(id, score[(size_t)p][(size_t)i], endpoints, pos_of_id, "picked");
        se.TieCount = ties[(size_t)p][(size_t)i];
        if (with_match) se.PrefixMatch = PrefixCacheMatchInfo{match[(size_t)p][(size_t)i], nh[(size_t)i], (uint16_t)g.block_tokens};
        pr.TargetEndpoints.push_back(se);
      }
    }
    if (cfg_.PrefixMatchInfo && !with_match) {  // the in-flight form: the index is the one the batch was scored against
      TargetRuns truns((size_t)n);
      for (int i = 0; i < n; i++)
        for (auto& kv : got[(size_t)rows[i]]) truns[(size_t)i].emplace_back(kv.first, &kv.second);
      FillTargetInfo(truns, rows, requests, endpoints, ids, hashes.data(), nh.data(), packed, g);
    }
  }

  // PreRequest with several profiles: the primary profile's target, then the "prefill" profile's, recorded in the prefix index
  // in one commit per request in that order (approximateprefix/plugin.go:177-197); the inflight-load-producer counts the
  // request on every profile's target (inflightload/producer.go:101-120).
  void PreRequestProfiles(const std::vector<BatchItem>& results) {
    const int R = (int)results.size();
    const bool has_prefill = std::any_of(cfg_.Profiles.begin(), cfg_.Profiles.end(), [](const auto& np) { return np.first == "prefill"; });
    std::vector<int32_t> primary((size_t)R, -1), prefill((size_t)R, -1);
    std::vector<int32_t> load_ep;
    std::vector<int> load_req;
    auto id_of = [&](const ProfileRunResult& pr) {
      return pr.TargetEndpoints.empty() ? -1 : last_ids_[(size_t)pr.TargetEndpoints[0].Index];
    };
    for (int r = 0; r < R; r++) {
      if (!results[r].error.empty()) continue;
      const SchedulingResult& sr = results[r].result;
      for (const auto& kv : sr.ProfileResults) {
        const int32_t id = id_of(kv.second);
        if (id < 0) continue;
        if (kv.first == sr.PrimaryProfileName) primary[r] = id;
        else if (kv.first == "prefill") prefill[r] = id;
        load_ep.push_back(id);
        load_req.push_back(r);
      }
    }
    if (!last_.hashes.empty() && !inorder_index_) {  // (in order against the index: ScheduleBatch committed the batch already)
      const int32_t* picks[2] = {primary.data(), prefill.data()};
      Check(eppscore_commit_picks_profiles(eng_, R, has_prefill ? 2 : 1, picks, last_.hashes.data(), last_.nh.data(), last_.stride,
                                           LruCapacities().data(), 0, 0, nullptr),
            "eppscore_commit_picks_profiles");
    }
    if (inflight_ && !inorder_ && (int)last_.size.size() == R && !load_ep.empty()) {  // (in order: ScheduleBatch counted them)
      const std::vector<int64_t> est = EstimateTokens(R, last_.size.data(), last_.hint.data(), last_.chars.data());
      std::vector<int64_t> tok(load_ep.size());
      for (size_t i = 0; i < load_ep.size(); i++) tok[i] = est[(size_t)load_req[i]];
      Check(eppscore_inflight_add(eng_, (int32_t)load_ep.size(), 0, load_ep.data(), tok.data(), nullptr), "eppscore_inflight_add");
    }
    RunningAdd(primary);  // the primary target only; the prefill target is not queued (requestcontrol_hooks.go:55-95)
  }

  // ResponseBody releases for a multi-profile result: the "prefill" profile's target at start of stream, the others at its end
  // (inflightload/producer.go:137-160).
  void ReleaseProfiles(const InferenceRequest& request, const SchedulingResult& result, bool prefill) {
    if (!inflight_) return;
    std::vector<int32_t> eps;
    for (const auto& kv : result.ProfileResults) {
      if ((kv.first == "prefill") != prefill || kv.second.TargetEndpoints.empty() || !kv.second.TargetEndpoints[0].Endpoint_) continue;
      const int32_t id = ServerId(kv.second.TargetEndpoints[0].Endpoint_->GetMetadata()->NamespacedName_.String());
      if (id >= 0) eps.push_back(id);
    }
    if (eps.empty()) return;
    int64_t size = 0;
    int32_t hint = -1, chars = 0;
    EstimateInputs(request, &size, &hint, &chars);
    std::vector<int64_t> tok(eps.size(), EstimateTokens(1, &size, &hint, &chars)[0]);
    Check(eppscore_inflight_release(eng_, (int32_t)eps.size(), 0, eps.data(), tok.data(), nullptr), "eppscore_inflight_release");
  }

  // SimpleTokenEstimator (eppscore_estimate_tokens) over n requests' EstimateInputs.
  std::vector<int64_t> EstimateTokens(int32_t n, const int64_t* size, const int32_t* hint, const int32_t* chars) const {
    std::vector<int64_t> est((size_t)n);
    Check(eppscore_estimate_tokens(eng_, n, 0, size, hint, chars, est.data(), nullptr), "eppscore_estimate_tokens");
    return est;
  }

  // makeserver (plugin.go:207-216): the LRU capacity of each endpoint row of the last engine batch, for its commit.
  std::vector<int32_t> LruCapacities() const {
    std::vector<int32_t> cap((size_t)last_rows_, 0);
    for (size_t m = 0; m < last_endpoints_->size(); m++) {
      const int blocks = (*last_endpoints_)[m].GetMetrics()->CacheNumBlocks;
      cap[(size_t)last_ids_[m]] = (cfg_.Prefix.AutoTune && blocks > 0) ? blocks : 0;
    }
    return cap;
  }

  // Stable endpoint ids of a candidate list (see ScheduleBatch): ids[i] is endpoint i's row, *rows the number of rows; true when
  // the list is exactly ids 0..M-1 in order.
  bool MapIds(const std::vector<Endpoint>& endpoints, std::vector<int>* ids_out, int* rows) {
    const int M = (int)endpoints.size();
    std::vector<int>& ids = *ids_out;
    ids.assign((size_t)M, 0);
    int Mx = 0;
    bool identity = true;
    {
      std::vector<int> seen;
      for (int m = 0; m < M; m++) {
        ids[m] = IdOf(endpoints[(size_t)m].GetMetadata()->NamespacedName_.String());
        Mx = std::max(Mx, ids[m] + 1);
        identity = identity && ids[m] == m;
      }
      seen.assign((size_t)Mx, 0);
      bool dup = false;
      for (int m = 0; m < M; m++) dup = dup || seen[(size_t)ids[m]]++ > 0;
      if (dup) {  // the same server twice in one list: positions are the only usable ids for this batch
        for (int m = 0; m < M; m++) ids[m] = m;
        Mx = M;
        identity = true;
      }
    }
    *rows = Mx;
    return identity;
  }

  // SimpleTokenEstimator's inputs for one request (eppscore_estimate_tokens): the body is always present here
  static void EstimateInputs(const InferenceRequest& q, int64_t* size, int32_t* hint, int32_t* chars) {
    *size = q.RequestSizeBytes;
    *hint = q.InputTokenCountHint;
    *chars = (int32_t)std::min<size_t>(q.Prompt.size(), 0x7fffffff);
  }

  // A server's stable endpoint id: the one it got when first seen, or a freed one for a newcomer.
  int IdOf(const std::string& namespaced_name) {
    auto it = server_ids_.find(namespaced_name);
    if (it != server_ids_.end()) return it->second;
    int id;
    if (!free_ids_.empty()) {
      id = free_ids_.back();
      free_ids_.pop_back();
    } else {
      id = (int)server_ids_.size();  // no free id ⇒ the ids in use are exactly 0..size-1
    }
    server_ids_.emplace(namespaced_name, id);
    return id;
  }

  // rows of the snapshot are endpoint ids: endpoint eps[i] fills row ids[i]; rows without an endpoint stay zero (they are
  // never candidates: the batch's mask excludes them).  The adapter dictionary is the batch's own: the TargetModels of
  // `requests` that some endpoint carries, in first-seen order over the endpoints.  A request's class on an endpoint reads only
  // whether its own target is in the endpoint's maps, plus the map sizes against MaxActiveModels (lora_affinity.go:84-99), so
  // the other names need no bit; nmodels still counts every name.
  void PackSnapshot(const std::vector<Endpoint>& eps, const std::vector<int>& ids, int rows, const std::vector<InferenceRequest>& requests) {
    const int N = (int)eps.size();
    const int M = rows;
    adapter_ids_.clear();
    std::unordered_set<std::string> targets;
    for (const auto& q : requests) targets.insert(q.TargetModel);
    for (auto& e : eps) {
      for (auto& kv : e.GetMetrics()->ActiveModels)
        if (targets.count(kv.first)) adapter_ids_.emplace(kv.first, (int)adapter_ids_.size());
      for (auto& kv : e.GetMetrics()->WaitingModels)
        if (targets.count(kv.first)) adapter_ids_.emplace(kv.first, (int)adapter_ids_.size());
    }
    const int words = (int)((adapter_ids_.size() + 63) / 64) > 0 ? (int)((adapter_ids_.size() + 63) / 64) : 1;
    std::vector<double> kv((size_t)M);
    std::vector<int64_t> queue((size_t)M), running((size_t)M);
    std::vector<uint64_t> act((size_t)M * words, 0), wait((size_t)M * words, 0);
    std::vector<int32_t> nm((size_t)M), mx((size_t)M), dispatched((size_t)M, 0);
    std::vector<int64_t> tokens((size_t)M, 0);
    std::vector<double> min_tpot((size_t)M, 0.0);
    std::vector<uint8_t> prefill((size_t)M, 0);
    bool have_tokens = false;
    const PredictedLatencyProducer* prod = cfg_.Profile.producer().get();
    for (int i = 0; i < N; i++) {
      const int m = ids[(size_t)i];  // the endpoint's row
      const Endpoint& ep = eps[(size_t)i];
      if (ep.InFlightTokens >= 0) {
        tokens[m] = ep.InFlightTokens;
        have_tokens = true;
      }
      if (prod) {
        auto st = prod->State.find(ep.GetMetadata()->NamespacedName_.String());
        if (st != prod->State.end()) {
          min_tpot[m] = st->second.RunningRequests > 0 ? st->second.MinTPOTSLO : 0.0;  // plugin.go:349-354
          dispatched[m] = st->second.RunningRequests;
        }
        if (!prod->EndpointRoleLabel.empty()) {  // hasPrefillRole, prediction.go:168-175
          auto lb = ep.GetMetadata()->Labels.find(prod->EndpointRoleLabel);
          prefill[m] = lb != ep.GetMetadata()->Labels.end() && lb->second == "prefill";
        }
      }
    }
    if (latency_scorer_ && prod) {
      eppscore_latency_params lp;
      eppscore_latency_params_default(&lp);
      auto coef = [](const std::map<std::string, double>& c, const char* k) {
        auto it = c.find(k);
        return it == c.end() ? 0.0 : it->second;  // Go map lookup of a missing key yields 0
      };
      lp.has_predictions = prod->HavePredictions ? 1 : 0;
      lp.ttft_intercept = prod->TTFTIntercept;
      lp.ttft_kv = coef(prod->TTFTCoeffs, "kv_cache_percentage");
      lp.ttft_input = coef(prod->TTFTCoeffs, "input_token_length");
      lp.ttft_waiting = coef(prod->TTFTCoeffs, "num_request_waiting");
      lp.ttft_running = coef(prod->TTFTCoeffs, "num_request_running");
      lp.ttft_prefix = coef(prod->TTFTCoeffs, "prefix_cache_score");
      lp.tpot_intercept = prod->TPOTIntercept;
      lp.tpot_kv = coef(prod->TPOTCoeffs, "kv_cache_percentage");
      lp.tpot_input = coef(prod->TPOTCoeffs, "input_token_length");
      lp.tpot_waiting = coef(prod->TPOTCoeffs, "num_request_waiting");
      lp.tpot_running = coef(prod->TPOTCoeffs, "num_request_running");
      lp.tpot_generated = coef(prod->TPOTCoeffs, "num_tokens_generated");
      lp.slo_buffer_factor = prod->SLOBufferFactor;
      lp.streaming_mode = prod->StreamingMode ? 1 : 0;
      lp.strategy_most = latency_scorer_->StrategyMost ? 1 : 0;
      lp.ttft_weight = latency_scorer_->TTFTWeight;
      lp.tpot_weight = latency_scorer_->TPOTWeight;
      lp.composite_kv = latency_scorer_->CompositeKVWeight;
      lp.composite_queue = latency_scorer_->CompositeQueueWeight;
      lp.composite_prefix = latency_scorer_->CompositePrefixWeight;
      Check(eppscore_set_latency_params(eng_, &lp), "eppscore_set_latency_params");
    }
    for (int i = 0; i < N; i++) {
      const int m = ids[(size_t)i];
      const Metrics* x = eps[(size_t)i].GetMetrics();
      kv[m] = x->KVCacheUsagePercent;
      queue[m] = x->WaitingQueueSize;
      running[m] = x->RunningRequestsSize;
      for (auto& a : x->ActiveModels) {
        const auto it = adapter_ids_.find(a.first);
        if (it != adapter_ids_.end()) act[(size_t)m * words + (it->second >> 6)] |= 1ULL << (it->second & 63);
      }
      for (auto& a : x->WaitingModels) {
        const auto it = adapter_ids_.find(a.first);
        if (it != adapter_ids_.end()) wait[(size_t)m * words + (it->second >> 6)] |= 1ULL << (it->second & 63);
      }
      nm[m] = (int32_t)(x->ActiveModels.size() + x->WaitingModels.size());  // len()+len() as MAP sizes (lora_affinity.go:90)
      mx[m] = x->MaxActiveModels;
    }
    eppscore_snapshot s{};
    s.struct_size = sizeof(s);
    s.M = M;
    s.lora_words = words;
    s.kv_usage = kv.data();
    s.queue = queue.data();
    s.running = running.data();
    s.lora_active = act.data();
    s.lora_waiting = wait.data();
    s.lora_nmodels = nm.data();
    s.lora_max = mx.data();
    // with the producer, a token-load scorer reads the engine's in-flight counters (a snapshot array would take precedence)
    s.inflight_tokens = (have_tokens && !(inflight_ && (token_load_ || inorder_))) ? tokens.data() : nullptr;
    if (prod) {
      // with TrackRunningRequests the engine's queues feed the latency fold-in: the arrays stay NULL
      s.min_tpot_slo = running_ ? nullptr : min_tpot.data();
      s.dispatched = running_ ? nullptr : dispatched.data();
      s.prefill_role = prefill.data();
    }
    s.epoch = ++epoch_;
    Check(eppscore_set_snapshot(eng_, &s), "eppscore_set_snapshot");
  }

  SchedulerConfig cfg_;
  SmallBatchCpu cpu_;
  bool cpu_route_ok_ = false;
  uint64_t cpu_routed_ = 0;
  eppscore_engine* eng_ = nullptr;
  const LatencyScorer* latency_scorer_ = nullptr;
  std::unordered_map<std::string, int> adapter_ids_;
  uint64_t epoch_ = 0;
  BatchRecord last_;  // the last engine batch's per-request record, for PreRequest
  const std::vector<Endpoint>* last_endpoints_ = nullptr;
  std::vector<int> last_ids_;                       // list position -> endpoint id of the last engine batch
  int last_rows_ = 0;
  std::unordered_map<std::string, int> server_ids_;  // ServerID (NamespacedName) -> stable endpoint id
  std::vector<int> free_ids_;
  uint64_t remapped_batches_ = 0;
  bool inflight_ = false;    // SchedulerConfig::InFlightLoad
  bool token_load_ = false;  // the profile has a token-load scorer
  bool inorder_ = false;     // SchedulerConfig::InOrderInFlightLoad
  bool inorder_index_ = false;  // SchedulerConfig::InOrderPrefixIndex
  bool inorder_latency_ = false;  // SchedulerConfig::InOrderRunningRequests
  bool running_ = false;  // PredictedLatencyProducer::TrackRunningRequests
  std::unordered_map<std::string, KeyUse> running_keys_;
  uint64_t next_key_ = 1;
  PrefixIndexerHistograms prefix_metrics_;
  std::unordered_map<std::string, epp::PredictedLatencyAtDispatch> dispatch_;
};

inline Scheduler* NewSchedulerWithConfig(const SchedulerConfig& c) { return new Scheduler(c); }

}  // namespace epp
