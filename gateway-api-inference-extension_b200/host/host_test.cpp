// host_test.cpp — the reference's own scheduler tests, restated against the C++ host mirror
// (epp_scheduler.hpp) so they run on the GPU engine through the C ABI.  Needs an H100; built by
// __graft_entry__.build() and executed by tests/test_host_cpp.py (-m gpu).
//   TestSchedule                      pkg/epp/scheduling/scheduler_test.go:42-159
//   TestSchedulePlugins (filters)     pkg/epp/scheduling/scheduler_profile_test.go:33-183
//   integration routing scenarios     test/integration/epp/common_tests.go:283-312, hermetic_test.go:120-272
//   TestPrefixPluginCompletion        .../approximateprefix/plugin_test.go:161-227 (via PreRequest)
//   TestTokenLoadScorer               pkg/epp/framework/plugins/scheduling/scorer/tokenload/token_load_test.go:32-61
//   TestPickWeightedRandomPicker      pkg/epp/framework/plugins/scheduling/picker/weightedrandom/picker_test.go:30-140
//   TestPickRandomPicker (top-k)      pkg/epp/framework/plugins/scheduling/picker/random/picker_test.go:40-119
//   TestScore* (latency-scorer)       pkg/epp/framework/plugins/scheduling/scorer/latency/plugin_test.go:52-208
#include <cmath>
#include <cstdio>
#include <cstring>

#include "epp_scheduler.hpp"
#include "coalescer.hpp"

#include <atomic>
#include <thread>

// 0: every batch goes to the GPU; 8: tiny request-independent batches take the host route (SmallBatchCpu).  The suite runs
// under both settings with the SAME expectations.
static int g_cpu_threshold = 0;

using namespace epp;

static int g_fail = 0;
#define CHECK(cond)                                                        \
  do {                                                                     \
    if (!(cond)) {                                                         \
      std::printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond);          \
      g_fail++;                                                            \
    }                                                                      \
  } while (0)

static Metrics M_(int queue, double kv, int maxActive, std::vector<std::string> active, std::vector<std::string> waiting = {}) {
  Metrics m;
  m.WaitingQueueSize = queue;
  m.KVCacheUsagePercent = kv;
  m.MaxActiveModels = maxActive;
  for (auto& a : active) m.ActiveModels[a] = 1;
  for (auto& w : waiting) m.WaitingModels[w] = 1;
  return m;
}

static SchedulerConfig DefaultFourScorerConfig() {
  // scheduler_test.go:49-57: kv, queue, prefix, lora — all weight 1, max-score picker
  SchedulerConfig c;
  c.CpuBatchThreshold = g_cpu_threshold;
  c.Profile.WithScorers({NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1),
                         NewWeightedScorer(std::make_shared<QueueScorer>(), 1),
                         NewWeightedScorer(std::make_shared<PrefixCacheScorer>(), 1),
                         NewWeightedScorer(std::make_shared<LoraAffinityScorer>(), 1)})
      .WithPicker(MaxScorePicker{});
  c.MaxEndpoints = 64;
  c.PrefixCapacity = 1 << 12;
  return c;
}

static void TestSchedule() {
  Scheduler scheduler(DefaultFourScorerConfig());
  {  // "no candidate endpoints" → error
    bool threw = false;
    try {
      scheduler.Schedule(InferenceRequest{"id0", "any-model", "", ""}, {});
    } catch (const SchedulingError& e) {
      threw = std::strstr(e.what(), "failed to run scheduler profile 'default'") != nullptr;
    }
    CHECK(threw);
  }
  {  // "finds optimal endpoint": pod2, Score == 2.8 (compared with == in the reference)
    std::vector<Endpoint> input = {NewEndpoint("pod1", M_(0, 0.2, 2, {"foo", "bar"})),
                                   NewEndpoint("pod2", M_(0, 0.2, 2, {"foo", "critical"})),
                                   NewEndpoint("pod3", M_(10, 0.8, 2, {"foo"}))};
    auto got = scheduler.Schedule(InferenceRequest{"id1", "critical", "", ""}, input);
    CHECK(got.PrimaryProfileName == "default");
    const auto& te = got.ProfileResults.at("default").TargetEndpoints;
    CHECK(te.size() == 1);
    CHECK(te[0].Endpoint_->GetMetadata()->NamespacedName_.Name == "pod2");
    CHECK(te[0].Score == 2.8);
    CHECK(te[0].TieCount == 1);
  }
}

// scheduler_profile_test.go's testPlugin as a Filter: keeps the endpoints whose names are listed
struct NameFilter : Filter {
  std::vector<std::string> keep;
  int calls = 0, seen = 0;
  explicit NameFilter(std::vector<std::string> k) : keep(std::move(k)) {}
  std::vector<int> Filter_(const InferenceRequest&, const std::vector<Endpoint>& eps, const std::vector<int>& cand) override {
    calls++;
    seen = (int)cand.size();
    std::vector<int> out;
    for (int m : cand)
      for (auto& k : keep)
        if (eps[(size_t)m].GetMetadata()->NamespacedName_.Name == k) out.push_back(m);
    return out;
  }
};

static void TestFilterChain() {
  std::vector<Endpoint> input = {NewEndpoint("pod1", M_(5, 0.5, 0, {})), NewEndpoint("pod2", M_(0, 0.1, 0, {})),
                                 NewEndpoint("pod3", M_(0, 0.0, 0, {}))};
  {  // filters narrow 3 → 3 → 2 (tp1 then tp2); pod3 would win unfiltered, pod2 wins among {pod1, pod2}
    auto f1 = std::make_shared<NameFilter>(std::vector<std::string>{"pod1", "pod2", "pod3"});
    auto f2 = std::make_shared<NameFilter>(std::vector<std::string>{"pod1", "pod2"});
    SchedulerConfig c;
    c.CpuBatchThreshold = g_cpu_threshold;
  c.CpuBatchThreshold = g_cpu_threshold;
    c.Profile.WithFilters({f1, f2})
        .WithScorers({NewWeightedScorer(std::make_shared<QueueScorer>(), 1), NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1)})
        .WithPicker(MaxScorePicker{});
    c.MaxEndpoints = 8;
    c.PrefixCapacity = 64;
    Scheduler s(c);
    auto got = s.Schedule(InferenceRequest{"id", "test-model", "", ""}, input);
    CHECK(got.ProfileResults.at("default").TargetEndpoints[0].Endpoint_->GetMetadata()->NamespacedName_.Name == "pod2");
    CHECK(f1->calls == 1 && f2->calls == 1);   // each filter called once
    CHECK(f1->seen == 3 && f2->seen == 3);     // chained: f2 received f1's output
    // the queue scorer normalises over the FILTERED set {5, 0}: pod2 = 1.0 + 0.9
    CHECK(got.ProfileResults.at("default").TargetEndpoints[0].Score == 1.0 + (1 - 0.1));
  }
  {  // "filter all" ⇒ error (no available endpoints after the filters)
    auto f1 = std::make_shared<NameFilter>(std::vector<std::string>{"pod1", "pod2", "pod3"});
    auto fall = std::make_shared<NameFilter>(std::vector<std::string>{});
    auto never = std::make_shared<NameFilter>(std::vector<std::string>{"pod1"});
    SchedulerConfig c;
    c.CpuBatchThreshold = g_cpu_threshold;
  c.CpuBatchThreshold = g_cpu_threshold;
    c.Profile.WithFilters({f1, fall, never}).WithScorers({NewWeightedScorer(std::make_shared<QueueScorer>(), 1)}).WithPicker(MaxScorePicker{});
    c.MaxEndpoints = 8;
    c.PrefixCapacity = 64;
    Scheduler s(c);
    bool threw = false;
    try {
      s.Schedule(InferenceRequest{"id", "test-model", "", ""}, input);
    } catch (const SchedulingError&) {
      threw = true;
    }
    CHECK(threw);
    CHECK(never->calls == 0);  // early break once the candidate list is empty (scheduler_profile.go:141-144)
  }
}

static std::vector<Endpoint> Pods(std::vector<std::tuple<int, int, double, std::vector<std::string>>> ps) {
  std::vector<Endpoint> out;
  for (auto& p : ps)  // P(idx, queue, kv, models...): models ACTIVE, MaxActiveModels = 0 (harness.go:386-391)
    out.push_back(NewEndpoint("pod" + std::to_string(std::get<0>(p)), M_(std::get<1>(p), std::get<2>(p), 0, std::get<3>(p))));
  return out;
}

static void TestIntegrationRouting() {
  // testdata/default-config.yaml: queue, kv, prefix, lora (weight 1)
  SchedulerConfig c;
  c.CpuBatchThreshold = g_cpu_threshold;
  c.Profile.WithScorers({NewWeightedScorer(std::make_shared<QueueScorer>(), 1), NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1),
                         NewWeightedScorer(std::make_shared<PrefixCacheScorer>(), 1), NewWeightedScorer(std::make_shared<LoraAffinityScorer>(), 1)})
      .WithPicker(MaxScorePicker{});
  c.MaxEndpoints = 8;
  c.PrefixCapacity = 256;
  Scheduler s(c);
  auto pick = [&](const std::string& model, const std::string& prompt, std::vector<Endpoint> pods) {
    return s.Schedule(InferenceRequest{"r", model, prompt, ""}, pods).ProfileResults.at("default").TargetEndpoints[0].Index;
  };
  CHECK(pick("my-model-12345", "test1", Pods({{0, 3, 0.2, {}}, {1, 0, 0.1, {}}, {2, 10, 0.2, {}}})) == 1);
  CHECK(pick("sql-lora-1fdg2", "test2", Pods({{0, 0, 0.2, {"foo", "bar"}}, {1, 0, 0.1, {"foo", "sql-lora-1fdg2"}}, {2, 10, 0.2, {"foo", "bar"}}})) == 1);
  CHECK(pick("sql-lora-1fdg2", "test3", Pods({{0, 10, 0.2, {"foo", "bar"}}, {1, 10, 0.4, {"foo", "sql-lora-1fdg2"}}, {2, 10, 0.3, {"foo"}}})) == 1);
  CHECK(pick("sql-lora-1fdg2", "test4", Pods({{0, 6, 0.2, {"foo", "bar", "sql-lora-1fdg2"}}, {1, 0, 0.85, {"foo"}}, {2, 10, 0.9, {"foo"}}})) == 0);
}

static void TestPrefixCompletionViaPreRequest() {
  // BlockSizeTokens 1 (4 chars), no autotune: "aaaaaa" → 2 hashes; after PreRequest(pick) "aaaabbbb" matches 1 of 2 there
  SchedulerConfig c;
  c.CpuBatchThreshold = g_cpu_threshold;
  c.Profile.WithScorers({NewWeightedScorer(std::make_shared<PrefixCacheScorer>(), 1)}).WithPicker(MaxScorePicker{});
  c.Prefix.AutoTune = false;
  c.Prefix.BlockSizeTokens = 1;
  c.MaxEndpoints = 8;
  c.PrefixCapacity = 256;
  Scheduler s(c);
  std::vector<Endpoint> eps = {NewEndpoint("pod1", Metrics{}), NewEndpoint("pod2", Metrics{}), NewEndpoint("pod3", Metrics{})};
  auto r1 = s.ScheduleBatch({InferenceRequest{"a", "test-model1", "aaaaaa", ""}}, eps);
  CHECK(s.LastTotalBlocks()[0] == 2);
  CHECK(r1[0].error.empty() && r1[0].result.ProfileResults.at("default").TargetEndpoints[0].TieCount == 3);  // empty index: all tie at 0
  const int first = r1[0].result.ProfileResults.at("default").TargetEndpoints[0].Index;
  s.PreRequest(r1);
  auto r2 = s.ScheduleBatch({InferenceRequest{"b", "test-model1", "aaaabbbb", ""}}, eps);
  const auto& te = r2[0].result.ProfileResults.at("default").TargetEndpoints[0];
  CHECK(te.Index == first);       // the endpoint that cached "aaaa" now wins
  CHECK(te.Score == 0.5);         // 1 matching block of 2 (prefix/plugin.go:108-110)
  CHECK(te.TieCount == 1);
  // a different model name changes the chain seed (hashing.go:69-71): no match any more
  auto r3 = s.ScheduleBatch({InferenceRequest{"c", "other-model", "aaaabbbb", ""}}, eps);
  CHECK(r3[0].result.ProfileResults.at("default").TargetEndpoints[0].Score == 0.0);
}


static void TestTokenLoadScorer() {
  SchedulerConfig c;
  c.CpuBatchThreshold = g_cpu_threshold;
  c.Profile.WithScorers({NewWeightedScorer(std::make_shared<TokenLoadScorer>(1000), 1)}).WithPicker(MaxScorePicker{});
  c.MaxEndpoints = 8;
  Scheduler s(c);
  std::vector<Endpoint> eps = {NewEndpoint("pod1", Metrics{}, "default"), NewEndpoint("pod2", Metrics{}, "default"),
                               NewEndpoint("pod3", Metrics{}, "default")};
  eps[1].InFlightTokens = 500;   // pod1: attribute absent => 0 tokens => 1.0
  eps[2].InFlightTokens = 1000;
  auto r = s.Schedule(InferenceRequest{"t", "m", "", ""}, eps);
  const auto& te = r.ProfileResults.at("default").TargetEndpoints[0];
  CHECK(te.Index == 0 && te.Score == 1.0 && te.TieCount == 1);
  eps[0].InFlightTokens = 750;   // 0.25 < pod2's 0.5
  r = s.Schedule(InferenceRequest{"t", "m", "", ""}, eps);
  CHECK(r.ProfileResults.at("default").TargetEndpoints[0].Index == 1);
  CHECK(std::fabs(r.ProfileResults.at("default").TargetEndpoints[0].Score - 0.5) < 1e-4);
}

// latency-scorer tests: the scorer consumes LatencyPredictionInfo{ttftHeadroom, tpotHeadroom, dispatched}. Here the
// producer is configured so that TTFT = WaitingQueueSize, TPOT = RunningRequestsSize and both SLO headers are
// 1000, i.e. headroom = 1000 - metric: each test's headroom values are encoded in the metrics.
struct LatEp { double th, ph; int dispatched; };
static int LatencyPick(const std::vector<LatEp>& info, double* score, int* ties) {
  SchedulerConfig c;
  c.CpuBatchThreshold = g_cpu_threshold;
  auto prod = std::make_shared<PredictedLatencyProducer>();
  prod->StreamingMode = true;
  prod->TTFTCoeffs["num_request_waiting"] = 1.0;
  prod->TPOTCoeffs["num_request_running"] = 1.0;
  c.Profile.WithScorers({NewWeightedScorer(std::make_shared<LatencyScorer>(), 1)}).WithPicker(MaxScorePicker{}).WithPredictedLatencyProducer(prod);
  c.MaxEndpoints = 8;
  std::vector<Endpoint> eps;
  for (size_t i = 0; i < info.size(); i++) {
    Metrics m;
    m.WaitingQueueSize = 1000 - (int)info[i].th;
    m.RunningRequestsSize = 1000 - (int)info[i].ph;
    eps.push_back(NewEndpoint("pod" + std::to_string(i), m, "default"));
    prod->State["default/pod" + std::to_string(i)].RunningRequests = info[i].dispatched;
  }
  Scheduler s(c);
  InferenceRequest q{"l", "m", "a prompt of five words", ""};
  q.Headers["x-slo-ttft-ms"] = "1000";
  q.Headers["x-slo-tpot-ms"] = "1000";
  auto r = s.Schedule(q, eps);
  const auto& te = r.ProfileResults.at("default").TargetEndpoints[0];
  *score = te.Score;
  *ties = te.TieCount;
  return te.Index;
}

// slo-headroom-tier-filter through the host mirror (sloheadroomtier/plugin_test.go:80-101): with both tiers present the
// positive tier is selected (epsilon 0) resp. the negative one (epsilon 1)
static int TierFilterPick(double epsilon) {
  SchedulerConfig c;
  c.CpuBatchThreshold = g_cpu_threshold;
  auto prod = std::make_shared<PredictedLatencyProducer>();
  prod->StreamingMode = true;
  prod->TTFTCoeffs["num_request_waiting"] = 1.0;
  prod->TPOTCoeffs["num_request_running"] = 1.0;
  c.Profile.WithScorers({NewWeightedScorer(std::make_shared<LatencyScorer>(), 1)}).WithPicker(MaxScorePicker{})
      .WithPredictedLatencyProducer(prod).WithDeviceFilters({SLOHeadroomTierFilter(epsilon)});
  c.MaxEndpoints = 8;
  const double th[3] = {100, 200, -100}, ph[3] = {50, 80, -50};
  std::vector<Endpoint> eps;
  for (int i = 0; i < 3; i++) {
    Metrics m;
    m.WaitingQueueSize = 1000 - (int)th[i];
    m.RunningRequestsSize = 1000 - (int)ph[i];
    eps.push_back(NewEndpoint("pod" + std::to_string(i), m, "default"));
  }
  Scheduler s(c);
  InferenceRequest q{"f", "m", "", ""};
  q.Headers["x-slo-ttft-ms"] = "1000";
  q.Headers["x-slo-tpot-ms"] = "1000";
  return s.Schedule(q, eps).ProfileResults.at("default").TargetEndpoints[0].Index;
}

static void TestLatencyScorer() {
  double sc;
  int ties;
  // TestScoreTierSplit (plugin_test.go:103-133): less headroom scores higher under "least"
  CHECK(LatencyPick({{10, 2, 0}, {50, 10, 0}}, &sc, &ties) == 0 && sc == 1.0 && ties == 1);
  // TestScoreNegativeOnly (:75-101): the smaller violation wins
  CHECK(LatencyPick({{-10, -5, 0}, {-100, -30, 0}}, &sc, &ties) == 0 && sc > 0);
  // TestScoreIdlePodPreference (:135-162): same deficit, only the idle pod is scored
  CHECK(LatencyPick({{-50, -10, 5}, {-50, -10, 0}}, &sc, &ties) == 1 && std::fabs(sc - 0.51) < 1e-12 && ties == 1);
  // TestScoreHierarchicalBuckets (:164-188): all negative and idle => one bucket; tpot-only deficit closest to SLO
  CHECK(LatencyPick({{-50, -10, 0}, {-30, 5, 0}, {10, -8, 0}}, &sc, &ties) == 2 && std::fabs(sc - 0.89) < 1e-12);
  // busy variants: the least severe non-empty bucket (negTPOTonly > negTTFTonly > bothNeg, :209-238) is the only one scored
  CHECK(LatencyPick({{-50, -10, 3}, {-30, 5, 2}, {10, -8, 1}}, &sc, &ties) == 2);
  CHECK(LatencyPick({{-50, -10, 3}, {-30, 5, 2}}, &sc, &ties) == 1);
  CHECK(TierFilterPick(0.0) != 2);  // positive tier kept: the overloaded pod is filtered out
  CHECK(TierFilterPick(1.0) == 2);  // epsilon-explore: only the negative tier is left
  // TestScoreCompositeFallback (:190-208): no predictions => kv/queue/prefix composite
  {
    SchedulerConfig c;
    c.CpuBatchThreshold = g_cpu_threshold;
  c.CpuBatchThreshold = g_cpu_threshold;
    auto prod = std::make_shared<PredictedLatencyProducer>();
    prod->HavePredictions = false;
    c.Profile.WithScorers({NewWeightedScorer(std::make_shared<LatencyScorer>(), 1)}).WithPicker(MaxScorePicker{}).WithPredictedLatencyProducer(prod);
    c.MaxEndpoints = 8;
    Scheduler s(c);
    Metrics a, b;
    a.KVCacheUsagePercent = 0.2; a.WaitingQueueSize = 0; a.RunningRequestsSize = 3;
    b.KVCacheUsagePercent = 0.8; b.WaitingQueueSize = 5; b.RunningRequestsSize = 10;
    auto r = s.Schedule(InferenceRequest{"c", "m", "", ""}, {NewEndpoint("pod1", a), NewEndpoint("pod2", b)});
    const auto& te = r.ProfileResults.at("default").TargetEndpoints[0];
    CHECK(te.Index == 0 && std::fabs(te.Score - 0.6) < 1e-12);
  }
  // strings.Fields semantics of the input-token count (predictedlatency/plugin.go:286)
  CHECK(CountFields("") == 0);
  CHECK(CountFields("  a  b\tc\n") == 3);
  CHECK(CountFields("one\xC2\xA0two\xE2\x80\x83three\xE3\x80\x80" "four") == 4);  // NBSP, EM SPACE, IDEOGRAPHIC SPACE
  CHECK(CountFields("\xE2\x80\x8B") == 1);                                          // ZERO WIDTH SPACE is not White_Space
}

// custom per-endpoint score column: lets a test hand the picker exact scores (score = clamp(col) * weight)
static void TestWeightedRandomPicker() {
  // "Multi-tier weighted test": scores 100, 90, 50, 30, 20 -> P = score / 290, +-5 % over 10000 picks
  const double scores[5] = {100, 90, 50, 30, 20};
  SchedulerConfig c;
  c.CpuBatchThreshold = g_cpu_threshold;
  c.Profile.WithScorers({NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 100)}).WithPicker(WeightedRandomPicker{});
  c.MaxEndpoints = 8;
  c.TieSeed = 2024;
  Scheduler s(c);
  std::vector<Endpoint> eps;
  for (int i = 0; i < 5; i++) {
    Metrics m;
    m.KVCacheUsagePercent = 1.0 - scores[i] / 100.0;  // kv scorer: 1 - usage
    eps.push_back(NewEndpoint("pod" + std::to_string(i + 1), m));
  }
  std::vector<InferenceRequest> reqs(10000, InferenceRequest{"w", "m", "", ""});
  auto res = s.ScheduleBatch(reqs, eps);
  int count[5] = {0, 0, 0, 0, 0};
  for (auto& r : res) count[r.result.ProfileResults.at("default").TargetEndpoints[0].Index]++;
  for (int i = 0; i < 5; i++) CHECK(std::fabs(count[i] / 10000.0 - scores[i] / 290.0) <= 0.05);
}

// max-score-picker with maxNumOfEndpoints = 3 (picker/maxscore/picker_test.go:43-110): descending score, the engine's pick first
static void TestTopK() {
  SchedulerConfig c;
  c.CpuBatchThreshold = g_cpu_threshold;
  MaxScorePicker pk;
  pk.MaxNumOfEndpoints = 3;
  c.Profile.WithScorers({NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1)}).WithPicker(pk);
  c.MaxEndpoints = 8;
  Scheduler s(c);
  std::vector<Endpoint> eps;
  const double usage[5] = {0.80, 0.75, 0.70, 0.85, 0.75};  // scores 0.20, 0.25, 0.30, 0.15, 0.25
  for (int i = 0; i < 5; i++) {
    Metrics m;
    m.KVCacheUsagePercent = usage[i];
    eps.push_back(NewEndpoint("pod" + std::to_string(i + 1), m));
  }
  auto got = s.Schedule(InferenceRequest{"id", "m", "", ""}, eps);
  const auto& te = got.ProfileResults.at("default").TargetEndpoints;
  CHECK(te.size() == 3);
  CHECK(te[0].Index == 2 && te[1].Index == 1 && te[2].Index == 4);  // 0.30, then the tie class {pod2, pod5}
  CHECK(te[0].Score == 1 - 0.70 && te[1].Score == 1 - 0.75 && te[2].Score == 1 - 0.75);
}

// weighted-random and random pickers with maxNumOfEndpoints = 3: k distinct candidates per request, entry 0 the pick; the random
// picker includes each of 5 endpoints with probability 3/5 (random/picker_test.go:40-119, +-5 %)
static void TestTopKStochastic() {
  if (!EngineHasTopK()) {
    std::printf("top-k stochastic pickers: skipped (the engine library has no eppscore_schedule_batch_topk)\n");
    return;
  }
  for (int mode = 0; mode < 2; mode++) {
    SchedulerConfig c;
    c.CpuBatchThreshold = g_cpu_threshold;
    MaxScorePicker pk = mode == 0 ? MaxScorePicker(WeightedRandomPicker{}) : MaxScorePicker(RandomPicker{});
    pk.MaxNumOfEndpoints = 3;
    c.Profile.WithScorers({NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1)}).WithPicker(pk);
    c.MaxEndpoints = 8;
    c.TieSeed = 77;
    Scheduler s(c);
    std::vector<Endpoint> eps;
    for (int i = 0; i < 5; i++) {
      Metrics m;
      m.KVCacheUsagePercent = 0.1 * (i + 1);  // scores 0.9 .. 0.5
      eps.push_back(NewEndpoint("pod" + std::to_string(i + 1), m));
    }
    const int n = 4000;
    std::vector<InferenceRequest> reqs(n, InferenceRequest{"t", "m", "", ""});
    auto res = s.ScheduleBatch(reqs, eps);
    int count[5] = {0, 0, 0, 0, 0};
    for (auto& r : res) {
      const auto& te = r.result.ProfileResults.at("default").TargetEndpoints;
      CHECK(r.error.empty() && te.size() == 3);
      if (te.size() != 3) continue;
      CHECK(te[0].Index != te[1].Index && te[0].Index != te[2].Index && te[1].Index != te[2].Index);
      for (const auto& se : te) {
        CHECK(se.Index >= 0 && se.Index < 5 && se.Score == 1.0 - 0.1 * (se.Index + 1));
        if (se.Index >= 0 && se.Index < 5) count[se.Index]++;
      }
    }
    if (mode == 1)
      for (int i = 0; i < 5; i++) CHECK(std::fabs(count[i] / (double)n - 0.6) <= 0.05);
  }
  std::printf("top-k stochastic pickers: checked\n");
}

// the coalescing front over the REAL scheduler: 32 caller threads, batches of up to 64, results handed back to their callers
static void TestCoalescedSchedule() {
  SchedulerConfig c = DefaultFourScorerConfig();
  c.CpuBatchThreshold = 0;
  Scheduler s(c);
  auto eps = std::make_shared<const std::vector<Endpoint>>(std::vector<Endpoint>{
      NewEndpoint("pod1", M_(0, 0.2, 2, {"foo", "bar"})), NewEndpoint("pod2", M_(0, 0.2, 2, {"foo", "critical"})),
      NewEndpoint("pod3", M_(10, 0.8, 2, {"foo"}))});
  BatchingScheduler<Scheduler> front(&s, std::chrono::microseconds(500), 64);
  std::vector<std::thread> th;
  std::atomic<int> bad{0};
  for (int t = 0; t < 32; t++)
    th.emplace_back([&, t] {
      for (int i = 0; i < 20; i++) {
        const bool crit = (t + i) % 2 == 0;
        auto item = front.Schedule(InferenceRequest{std::to_string(t * 100 + i), crit ? "critical" : "bar", "", ""}, eps);
        if (!item.error.empty()) { bad++; continue; }
        const auto& se = item.result.ProfileResults.at("default").TargetEndpoints[0];
        // scheduler_test.go:86-143: target "critical" -> pod2 with score 2.8; target "bar" -> pod1 by symmetry
        if (se.Endpoint_->GetMetadata()->NamespacedName_.Name != (crit ? "pod2" : "pod1") || se.Score != 2.8) bad++;
      }
    });
  for (auto& x : th) x.join();
  CHECK(bad == 0);
  const CoalescerStats st = front.stats();
  CHECK(st.requests == 640 && st.batches < 640 && st.max_batch > 1);
  std::printf("coalesced schedule: %llu requests in %llu engine batches (largest %llu)\n", (unsigned long long)st.requests,
              (unsigned long long)st.batches, (unsigned long long)st.max_batch);
}

int main() {
  try {
    for (int pass = 0; pass < 2; pass++) {
      g_cpu_threshold = pass == 0 ? 0 : 8;
      TestSchedule();
      TestFilterChain();
      TestIntegrationRouting();
      TestPrefixCompletionViaPreRequest();
      TestTokenLoadScorer();
      TestLatencyScorer();
      TestWeightedRandomPicker();
      TestTopK();
      TestTopKStochastic();
      std::printf("pass %d (CpuBatchThreshold = %d) done\n", pass, g_cpu_threshold);
    }
    TestCoalescedSchedule();
  } catch (const std::exception& e) {
    std::printf("FAIL exception: %s\n", e.what());
    return 2;
  }
  if (g_fail) {
    std::printf("%d check(s) failed\n", g_fail);
    return 1;
  }
  std::printf("host_test: all checks passed\n");
  return 0;
}
