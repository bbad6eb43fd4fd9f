// host_latency_info_test.cpp — the host layer's LatencyPredictionInfo (SchedulerConfig::LatencyPredictionInfo) and PreRequest's
// dispatch record, against the oracle's latency predict + validate fed the endpoints' metrics, the producer's state and a mirror
// of the prefix index (the same hashPrompt, the same Adds in PreRequest's order).  Runs on the oracle-backed stand-in of the C
// ABI (tests/test_host_latency_info_cpu.py) and on the engine (tests/test_gpu_latency_info.py).  Checks, printing one line per
// check:
//   - every SchedulingResult::TargetLatency entry (and, with PrefixMatchInfo too, every PrefixMatch) of single-profile results, top-k lists of 3
//     and 12, and decode / prefill results;
//   - the dispatch record: TTFT and prefix score at the "prefill" target when there is one, TPOT at the primary target, the SLOs;
//     dropped at ResponseComplete / RequestExpired;
//   - HavePredictions = false: every entry empty, the record 0;
//   - two endpoints sharing a Name in two namespaces: the record reads the later candidate's values (NamespacedName.Name keys);
//   - the option off: nothing filled or kept, no eppscore_predict_latency call (stand-in);
//   - through a BatchingScheduler: each caller's own result carries its TargetLatency, equal to a direct batch's.
// Built against a library without eppscore_predict_latency, the option is refused when the Scheduler is built.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include <thread>

#include "../../gateway-api-inference-extension_b200/host/coalescer.hpp"
#include "../../gateway-api-inference-extension_b200/host/epp_scheduler.hpp"
#include "../../oracle/oracle.h"

extern "C" int64_t oracle_backed_predict_latency_calls __attribute__((weak));

using namespace epp;

static int g_fail = 0;
#define CHECK(cond, what)               \
  do {                                  \
    if (!(cond)) {                      \
      std::printf("FAIL %s\n", what);   \
      g_fail++;                         \
    }                                   \
  } while (0)

static const int kMaxBlocks = 256;
static const int kBlock = 16;

struct Mirror {
  orc_index* idx = orc_index_new(31250);
  ~Mirror() { orc_index_free(idx); }
  static std::vector<uint64_t> hashes(const InferenceRequest& q) {
    std::vector<uint64_t> h(kMaxBlocks);
    const uint64_t seed = orc_model_seed(q.TargetModel.data(), q.TargetModel.size(), q.CacheSalt.data(), q.CacheSalt.size());
    const int n = orc_hash_prompt(reinterpret_cast<const uint8_t*>(q.Prompt.data()), (int64_t)q.Prompt.size(), seed, kBlock * 4,
                                  kMaxBlocks, h.data(), kMaxBlocks);
    h.resize((size_t)(n < 0 ? 0 : n));
    return h;
  }
  int match(const std::vector<uint64_t>& h, int id) const {
    std::vector<uint16_t> m(1024);
    orc_match_longest_prefix(idx, h.data(), (int32_t)h.size(), 1024, m.data());
    return m[(size_t)id];
  }
  void add(const std::vector<uint64_t>& h, int id) { orc_index_add(idx, h.data(), (int32_t)h.size(), id, 0); }
};

static std::shared_ptr<PredictedLatencyProducer> Producer(bool have) {
  auto p = std::make_shared<PredictedLatencyProducer>();
  p->StreamingMode = true;
  p->EndpointRoleLabel = "role";
  p->HavePredictions = have;
  p->SLOBufferFactor = 0.9;
  p->TTFTIntercept = 40.0;
  p->TPOTIntercept = 8.0;
  p->TTFTCoeffs = {{"kv_cache_percentage", 30.0}, {"input_token_length", 0.5}, {"num_request_waiting", 6.0},
                   {"num_request_running", 3.0}, {"prefix_cache_score", -25.0}};
  p->TPOTCoeffs = {{"kv_cache_percentage", 4.0}, {"input_token_length", 0.01}, {"num_request_waiting", 1.0},
                   {"num_request_running", 0.5}, {"num_tokens_generated", 0.25}};
  return p;
}
static orc_latency_params Params(const PredictedLatencyProducer& p) {
  orc_latency_params l;
  std::memset(&l, 0, sizeof(l));
  auto c = [](const std::map<std::string, double>& m, const char* k) {
    auto it = m.find(k);
    return it == m.end() ? 0.0 : it->second;
  };
  l.ttft_intercept = p.TTFTIntercept;
  l.ttft_kv = c(p.TTFTCoeffs, "kv_cache_percentage");
  l.ttft_input = c(p.TTFTCoeffs, "input_token_length");
  l.ttft_waiting = c(p.TTFTCoeffs, "num_request_waiting");
  l.ttft_running = c(p.TTFTCoeffs, "num_request_running");
  l.ttft_prefix = c(p.TTFTCoeffs, "prefix_cache_score");
  l.tpot_intercept = p.TPOTIntercept;
  l.tpot_kv = c(p.TPOTCoeffs, "kv_cache_percentage");
  l.tpot_input = c(p.TPOTCoeffs, "input_token_length");
  l.tpot_waiting = c(p.TPOTCoeffs, "num_request_waiting");
  l.tpot_running = c(p.TPOTCoeffs, "num_request_running");
  l.tpot_generated = c(p.TPOTCoeffs, "num_tokens_generated");
  l.slo_buffer_factor = p.SLOBufferFactor;
  l.streaming_mode = p.StreamingMode ? 1 : 0;
  l.has_predictions = p.HavePredictions ? 1 : 0;
  return l;
}

static double Slo(const InferenceRequest& q, const char* k) {
  auto it = q.Headers.find(k);
  return it == q.Headers.end() ? 0.0 : std::atof(it->second.c_str());
}

// PrepareRequestData's values for request q on endpoint e: (info or empty, prefix score)
static std::pair<std::optional<LatencyPredictionInfo>, double> Expect(const PredictedLatencyProducer& p, const Mirror& mir, Scheduler& s,
                                                                      const InferenceRequest& q, const Endpoint& e) {
  const orc_latency_params l = Params(p);
  const auto h = Mirror::hashes(q);
  const int id = s.ServerId(e.GetMetadata()->NamespacedName_.String());
  double prefix = (double)mir.match(h, id) / (double)h.size();  // stored whether or not a prediction is (preparedata_hooks.go:42-58)
  if (std::isnan(prefix)) prefix = 0.0;
  if (!p.HavePredictions) return {std::nullopt, prefix};
  const Metrics& m = *e.GetMetrics();
  double ttft, tpot, hr[2];
  int32_t ok[3];
  orc_latency_predict(&l, m.KVCacheUsagePercent, CountFields(q.Prompt), m.WaitingQueueSize, m.RunningRequestsSize, 1, prefix, &ttft, &tpot);
  double min_tpot = 0.0;
  int disp = 0;
  auto st = p.State.find(e.GetMetadata()->NamespacedName_.String());
  if (st != p.State.end()) {
    min_tpot = st->second.RunningRequests > 0 ? st->second.MinTPOTSLO : 0.0;
    disp = st->second.RunningRequests;
  }
  auto lb = e.GetMetadata()->Labels.find("role");
  const bool prefill = lb != e.GetMetadata()->Labels.end() && lb->second == "prefill";
  orc_latency_validate(&l, ttft, tpot, Slo(q, "x-slo-ttft-ms"), Slo(q, "x-slo-tpot-ms"), min_tpot, prefill ? 1 : 0, ok, hr);
  LatencyPredictionInfo v;
  v.TTFTValid = ok[0] != 0;
  v.TPOTValid = ok[1] != 0;
  v.TTFTHeadroom = hr[1];
  v.TPOTHeadroom = hr[0];
  v.TTFT = ttft;
  v.TPOT = tpot;
  v.DispatchedRequestCount = disp;
  return {v, prefix};
}
static bool Same(const std::optional<LatencyPredictionInfo>& a, const std::optional<LatencyPredictionInfo>& b) {
  if (!a || !b) return !a && !b;
  auto bits = [](double x) {
    uint64_t u;
    std::memcpy(&u, &x, 8);
    return u;
  };
  return a->TTFTValid == b->TTFTValid && a->TPOTValid == b->TPOTValid && bits(a->TTFTHeadroom) == bits(b->TTFTHeadroom) &&
         bits(a->TPOTHeadroom) == bits(b->TPOTHeadroom) && bits(a->TTFT) == bits(b->TTFT) && bits(a->TPOT) == bits(b->TPOT) &&
         a->DispatchedRequestCount == b->DispatchedRequestCount;
}

static Metrics Met(int i) {
  Metrics m;
  m.WaitingQueueSize = (i * 5) % 9;
  m.RunningRequestsSize = (i * 3) % 7;
  m.KVCacheUsagePercent = 0.1 * (i % 7);
  return m;
}
static std::vector<Endpoint> Pool(int n, std::vector<std::string> ns = {}) {
  std::vector<Endpoint> eps;
  for (int i = 0; i < n; i++) {
    eps.push_back(NewEndpoint("ep" + std::to_string(i), Met(i), ns.empty() ? "default" : ns[(size_t)i]));
    eps.back().Metadata.Labels["role"] = i % 2 ? "prefill" : "decode";
  }
  return eps;
}
static std::vector<InferenceRequest> Requests(int R, int round) {
  static const char* sys[] = {"You are a helpful assistant that answers questions about the weather in great detail. ",
                              "System: translate the following text into French, keeping the formatting as it is. ",
                              "Summarise the document below in three bullet points, citing the section numbers. "};
  std::vector<InferenceRequest> out;
  for (int r = 0; r < R; r++) {
    InferenceRequest q;
    q.RequestId = "req-" + std::to_string(round) + "-" + std::to_string(r);
    q.TargetModel = "m";
    std::string p;
    for (int i = 0; i < 6; i++) p += sys[(r + round) % 3];
    for (int i = 0; i < (r % 5); i++) p += "user turn " + std::to_string(r * 31 + round) + " with some more words to hash. ";
    q.Prompt = p;
    if (r % 4 != 3) q.Headers["x-slo-ttft-ms"] = std::to_string(100 + 40 * (r % 9));
    if (r % 5 != 4) q.Headers["x-slo-tpot-ms"] = std::to_string(10 + 3 * (r % 11));
    out.push_back(q);
  }
  return out;
}

// every entry of every profile; the dispatch record after PreRequest; returns the number of entries checked
static int CheckBatch(Scheduler& s, const PredictedLatencyProducer& p, Mirror& mir, const std::vector<InferenceRequest>& reqs,
                      const std::vector<Endpoint>& eps, const std::vector<Scheduler::BatchItem>& res, bool with_match, const char* what) {
  int n = 0;
  std::vector<double> want_ttft(res.size()), want_tpot(res.size()), want_pref(res.size());
  for (size_t r = 0; r < res.size(); r++) {
    if (!res[r].error.empty()) continue;
    for (const auto& kv : res[r].result.ProfileResults) {
      const auto& te = kv.second.TargetEndpoints;
      const auto tlit = res[r].result.TargetLatency.find(kv.first);
      const auto* tl = tlit == res[r].result.TargetLatency.end() ? nullptr : &tlit->second;
      CHECK(tl && tl->size() == te.size(), what);
      for (size_t j = 0; tl && j < te.size() && j < tl->size(); j++) {
        const auto w = Expect(p, mir, s, reqs[r], *te[j].Endpoint_);
        const bool ok = Same((*tl)[j], w.first);
        if (!ok) std::printf("  %s r=%zu %s j=%zu\n", what, r, kv.first.c_str(), j);
        CHECK(ok, what);
        if (with_match) {
          const auto h = Mirror::hashes(reqs[r]);
          const int id = s.ServerId(te[j].Endpoint_->GetMetadata()->NamespacedName_.String());
          CHECK(te[j].PrefixMatch && te[j].PrefixMatch->MatchBlocks == mir.match(h, id) && te[j].PrefixMatch->TotalBlocks == (int)h.size(),
                "match through the same call");
        }
        n++;
      }
    }
    // the record: the last candidate with the target's Name stands for it
    auto named = [&](const Endpoint* t) {
      const Endpoint* last = nullptr;
      for (const Endpoint& e : eps)
        if (e.GetMetadata()->NamespacedName_.Name == t->GetMetadata()->NamespacedName_.Name) last = &e;
      return Expect(p, mir, s, reqs[r], *last);
    };
    const auto& sr = res[r].result;
    const Endpoint* primary = sr.ProfileResults.at(sr.PrimaryProfileName).TargetEndpoints[0].Endpoint_;
    auto pf = sr.ProfileResults.find("prefill");
    const Endpoint* tt = (pf != sr.ProfileResults.end() && !pf->second.TargetEndpoints.empty()) ? pf->second.TargetEndpoints[0].Endpoint_ : primary;
    const auto a = named(tt), b = named(primary);
    want_ttft[r] = a.first ? a.first->TTFT : 0.0;
    want_pref[r] = a.second;
    want_tpot[r] = b.first ? b.first->TPOT : 0.0;
  }
  for (size_t r = 0; r < res.size(); r++) {  // PreRequest's Adds on the mirror: primary target, then the "prefill" target
    if (!res[r].error.empty()) continue;
    const auto& sr = res[r].result;
    const auto h = Mirror::hashes(reqs[r]);
    mir.add(h, s.ServerId(sr.ProfileResults.at(sr.PrimaryProfileName).TargetEndpoints[0].Endpoint_->GetMetadata()->NamespacedName_.String()));
    auto pf = sr.ProfileResults.find("prefill");
    if (pf != sr.ProfileResults.end() && !pf->second.TargetEndpoints.empty())
      mir.add(h, s.ServerId(pf->second.TargetEndpoints[0].Endpoint_->GetMetadata()->NamespacedName_.String()));
  }
  s.PreRequest(res);
  for (size_t r = 0; r < res.size(); r++) {
    if (!res[r].error.empty()) continue;
    const auto* d = s.PredictedLatencyAtDispatch(reqs[r].RequestId);
    const bool ok = d && d->PredictedTTFT == want_ttft[r] && d->FirstPredictedTPOT == want_tpot[r] && d->PrefixCacheScore == want_pref[r] &&
                    d->TTFTSLO == Slo(reqs[r], "x-slo-ttft-ms") && d->AvgTPOTSLO == Slo(reqs[r], "x-slo-tpot-ms");
    if (!ok) std::printf("  %s record r=%zu\n", what, r);
    CHECK(ok, "dispatch record");
  }
  return n;
}

static SchedulerConfig Single(int k, bool have = true) {
  SchedulerConfig c;
  c.Profile.WithScorers({NewWeightedScorer(std::make_shared<LatencyScorer>(), 2), NewWeightedScorer(std::make_shared<PrefixCacheScorer>(), 3),
                         NewWeightedScorer(std::make_shared<QueueScorer>(), 1)})
      .WithPredictedLatencyProducer(Producer(have));
  MaxScorePicker p;
  p.MaxNumOfEndpoints = k;
  c.Profile.WithPicker(p);
  c.MaxEndpoints = 64;
  c.CpuBatchThreshold = 0;
  c.LatencyPredictionInfo = true;
  return c;
}

static void SingleProfile(int k, bool have, bool with_match) {
  SchedulerConfig c = Single(k, have);
  c.PrefixMatchInfo = with_match;
  auto& prod = *c.Profile.producer();
  prod.State["default/ep2"] = {12.0, 2};
  prod.State["default/ep5"] = {70.0, 1};
  Scheduler s(c);
  const auto eps = Pool(16);
  Mirror mir;
  int n = 0;
  for (int round = 0; round < 3; round++) {
    const auto reqs = Requests(24, round);
    n += CheckBatch(s, prod, mir, reqs, eps, s.ScheduleBatch(reqs, eps), with_match, have ? "single entries" : "no predictions");
  }
  if (!have) {
    const auto* d = s.PredictedLatencyAtDispatch("req-0-0");
    CHECK(d && d->PredictedTTFT == 0.0 && d->FirstPredictedTPOT == 0.0, "no predictions: record 0");
  }
  std::printf("%s k=%d entries %d\n", have ? "single" : "nopred", k, n);
}

struct PdHandler : ProfileHandler {
  std::vector<std::string> Pick(const InferenceRequest&, const std::vector<std::string>&,
                                const std::map<std::string, const ProfileRunResult*>& results) override {
    if (!results.empty()) return {};
    return {"decode", "prefill"};
  }
  SchedulingResult ProcessResults(const InferenceRequest&, const std::map<std::string, const ProfileRunResult*>& res) override {
    if (!res.at("decode")) throw SchedulingError("failed to run scheduler profile 'decode'");
    SchedulingResult r;
    for (const auto& kv : res)
      if (kv.second) r.ProfileResults[kv.first] = *kv.second;
    r.PrimaryProfileName = "decode";
    return r;
  }
};

static void DecodePrefill() {
  SchedulerConfig c;
  c.MaxEndpoints = 64;
  c.LatencyPredictionInfo = true;
  c.Handler = std::make_shared<PdHandler>();
  auto prod = Producer(true);
  prod->State["default/ep3"] = {9.0, 3};
  for (const char* role : {"decode", "prefill"}) {
    SchedulerProfile p;
    p.WithScorers({NewWeightedScorer(std::make_shared<LatencyScorer>(), 2), NewWeightedScorer(std::make_shared<PrefixCacheScorer>(), 3)});
    const std::string rl = role;
    p.WithEndpointSubset([rl](const Endpoint& e) { return e.GetMetadata()->Labels.at("role") == rl; });
    MaxScorePicker pk;
    pk.MaxNumOfEndpoints = rl == "decode" ? 3 : 1;
    p.WithPicker(pk);
    p.WithPredictedLatencyProducer(prod);
    c.Profiles.emplace_back(rl, p);
  }
  Scheduler s(c);
  const auto eps = Pool(12);
  Mirror mir;
  int n = 0;
  for (int round = 0; round < 3; round++) {
    const auto reqs = Requests(20, round);
    n += CheckBatch(s, *prod, mir, reqs, eps, s.ScheduleBatch(reqs, eps), false, "pd entries");
  }
  std::printf("pd entries %d\n", n);
}

// ns-a/ep0 .. and ns-b/ep0: one Name in two namespaces; the later candidate's values stand for the earlier one in the record
static void SharedNames() {
  Scheduler s(Single(1));
  auto eps = Pool(6, {"ns-a", "ns-a", "ns-a", "ns-a", "ns-b", "ns-b"});
  eps[4] = NewEndpoint("ep0", Met(8), "ns-b");  // shares ep0's Name, different metrics
  eps[4].Metadata.Labels["role"] = "decode";
  const auto prodp = Single(1).Profile.producer();  // (the same coefficients as the Scheduler's producer)
  auto& prod = *prodp;
  Mirror mir;
  int n = 0, aliased = 0;
  for (int round = 0; round < 3; round++) {
    const auto reqs = Requests(16, round);
    const auto res = s.ScheduleBatch(reqs, eps);
    for (const auto& it : res)
      if (it.error.empty() && it.result.ProfileResults.at("default").TargetEndpoints[0].Endpoint_ == &eps[0]) aliased++;
    n += CheckBatch(s, prod, mir, reqs, eps, res, false, "shared names");
  }
  std::printf("names entries %d aliased %d\n", n, aliased);
}

static void DroppedAndOff() {
  Scheduler s(Single(1));
  const auto eps = Pool(8);
  const auto reqs = Requests(6, 0);
  const auto res = s.ScheduleBatch(reqs, eps);
  s.PreRequest(res);
  CHECK(s.TrackedDispatches() == 6, "six records kept");
  s.ResponseComplete(reqs[0], res[0].result);
  s.RequestExpired(reqs[1], res[1].result);
  CHECK(!s.PredictedLatencyAtDispatch(reqs[0].RequestId) && !s.PredictedLatencyAtDispatch(reqs[1].RequestId) && s.TrackedDispatches() == 4,
        "records dropped");
  const int64_t calls0 = &oracle_backed_predict_latency_calls ? oracle_backed_predict_latency_calls : 0;
  SchedulerConfig c = Single(3);
  c.LatencyPredictionInfo = false;
  Scheduler off(c);
  for (int round = 0; round < 2; round++) {
    const auto r2 = off.ScheduleBatch(Requests(10, round), eps);
    bool none = true;
    for (const auto& it : r2) none = none && it.result.TargetLatency.empty();
    CHECK(none, "option off: nothing filled");
    off.PreRequest(r2);
  }
  CHECK(off.TrackedDispatches() == 0, "option off: nothing kept");
  if (&oracle_backed_predict_latency_calls) CHECK(oracle_backed_predict_latency_calls == calls0, "option off: no engine call");
  SchedulerConfig nolat;
  nolat.Profile.WithScorers({NewWeightedScorer(std::make_shared<QueueScorer>(), 1)});
  nolat.LatencyPredictionInfo = true;
  try {
    Scheduler x(nolat);
    std::printf("FAIL the option was accepted without a latency scorer\n");
    g_fail++;
  } catch (const SchedulingError&) {
  }
  std::printf("option off checked\n");
}

// concurrent callers through the coalescing front: each gets back its own result, whose TargetLatency equals the one a direct
// ScheduleBatch of the same request gives (a second Scheduler, the same index state: nothing is committed)
static void ThroughCoalescer() {
  Scheduler s(Single(3)), direct(Single(3));
  auto eps = std::make_shared<const std::vector<Endpoint>>(Pool(12));
  BatchingScheduler<Scheduler> bs(&s, std::chrono::microseconds(200), 16);
  const auto reqs = Requests(24, 7);
  std::vector<Scheduler::BatchItem> got(reqs.size());
  std::vector<std::thread> th;
  for (size_t i = 0; i < reqs.size(); i++) th.emplace_back([&, i] { got[i] = bs.Schedule(reqs[i], eps); });
  for (auto& t : th) t.join();
  int n = 0;
  for (size_t i = 0; i < reqs.size(); i++) {
    const auto want = direct.ScheduleBatch({reqs[i]}, *eps)[0];
    CHECK(got[i].error.empty() && want.error.empty(), "coalescer: scheduled");
    const auto& tl = got[i].result.TargetLatency.at("default");
    const auto& wl = want.result.TargetLatency.at("default");
    CHECK(tl.size() == got[i].result.ProfileResults.at("default").TargetEndpoints.size(), "coalescer: parallel");
    bool same = tl.size() == wl.size();
    for (size_t j = 0; same && j < tl.size(); j++) {
      same = Same(tl[j], wl[j]) && got[i].result.ProfileResults.at("default").TargetEndpoints[j].Endpoint_ ==
                                      want.result.ProfileResults.at("default").TargetEndpoints[j].Endpoint_;
      n++;
    }
    CHECK(same, "coalescer: the caller's own result");
  }
  std::printf("coalescer entries %d\n", n);
}

int main() {
  if (!EngineHasPredictLatency()) {
    try {
      Scheduler s(Single(1));
      std::printf("FAIL the option was accepted without eppscore_predict_latency\n");
    } catch (const SchedulingError& e) {
      std::printf("refused %s\n", e.what());
    }
    SchedulerConfig c = Single(1);
    c.LatencyPredictionInfo = false;
    Scheduler s(c);  // without the option the library serves as before
    std::printf("done\n");
    return 0;
  }
  SingleProfile(1, true, false);
  SingleProfile(3, true, true);
  SingleProfile(12, true, false);
  SingleProfile(3, false, false);
  DecodePrefill();
  SharedNames();
  DroppedAndOff();
  ThroughCoalescer();
  std::printf(g_fail ? "FAILED %d\n" : "done\n", g_fail);
  return g_fail ? 1 : 0;
}
