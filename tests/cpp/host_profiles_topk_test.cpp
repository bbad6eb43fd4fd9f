// host_profiles_topk_test.cpp — the host layer's Scheduler with several profiles, maxNumOfEndpoints lists and the latency
// scorer, on the oracle-backed stand-in of the C ABI (a decode and a "prefill" profile over the two halves of the pool, split by
// a role label).  Checks, and prints one line per check for tests/test_host_profiles_topk_cpu.py:
//   - lists: decode MaxNumOfEndpoints 3, prefill 1; each profile's TargetEndpoints equal a single-profile Scheduler whose host
//     Filter keeps the same role (max-score, lowest-index ties: the score map's order is the engine's list order);
//   - latency: a latency scorer on the decode profile with TrackRunningRequests; its picks equal the filtered single-profile
//     Scheduler's, PreRequest queues each request on the decode target only, ResponseComplete removes it there;
//   - producers: two different predicted-latency producers are refused, two equal ones are accepted.
// Built without eppscore_schedule_batch_profiles_topk (oracle_backed_profiles.cpp instead of oracle_backed_profiles_topk.cpp),
// the list config is refused when the Scheduler is built, as before.
#include <cstdio>
#include <string>
#include <vector>

#include "../../gateway-api-inference-extension_b200/host/epp_scheduler.hpp"

using namespace epp;

static int g_fail = 0;
#define CHECK(cond, what)                         \
  do {                                            \
    if (!(cond)) {                                \
      std::printf("FAIL %s\n", what);             \
      g_fail++;                                   \
    }                                             \
  } while (0)

static const char* kRole = "role";

struct RoleFilter : Filter {
  std::string role;
  explicit RoleFilter(std::string r) : role(std::move(r)) {}
  std::vector<int> Filter_(const InferenceRequest&, const std::vector<Endpoint>& eps, const std::vector<int>& cand) override {
    std::vector<int> out;
    for (int i : cand)
      if (eps[(size_t)i].GetMetadata()->Labels.at(kRole) == role) out.push_back(i);
    return out;
  }
};

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

static const uint64_t kSeed = 91;
static const int kEndpoints = 24;

static std::vector<Endpoint> endpoints() {
  std::vector<Endpoint> eps;
  for (int i = 0; i < kEndpoints; i++) {
    Metrics m;
    m.KVCacheUsagePercent = 0.03 * ((i * 7) % 23);
    m.WaitingQueueSize = (i * 5) % 4;  // ties: the lists' order inside a tie class is exercised
    m.RunningRequestsSize = (i * 3) % 5;
    Endpoint e = NewEndpoint("pod" + std::to_string(i), m);
    e.Metadata.Labels[kRole] = i % 2 == 0 ? "prefill" : "decode";
    eps.push_back(e);
  }
  return eps;
}

static std::vector<InferenceRequest> requests(int round) {
  std::vector<InferenceRequest> reqs;
  for (int r = 0; r < 48; r++) {
    std::string prompt(256, 'a' + (r % 5));
    prompt += " tail words " + std::string(80, 'k' + ((r * 3 + round) % 11));
    InferenceRequest q{"req" + std::to_string(round) + "-" + std::to_string(r), "m", prompt, ""};
    q.Headers["x-slo-ttft-ms"] = std::to_string(200 + 10 * (r % 7));
    q.Headers["x-slo-tpot-ms"] = std::to_string(20 + (r % 5));
    reqs.push_back(q);
  }
  return reqs;
}

static SchedulerProfile decode_profile(int k) {
  SchedulerProfile p;
  p.WithScorers({NewWeightedScorer(std::make_shared<QueueScorer>(), 2), NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 2),
                 NewWeightedScorer(std::make_shared<PrefixCacheScorer>(), 3)});
  MaxScorePicker pk;
  pk.MaxNumOfEndpoints = k;
  p.WithPicker(pk);
  return p;
}
static SchedulerProfile prefill_profile() {
  SchedulerProfile p;
  p.WithScorers({NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1), NewWeightedScorer(std::make_shared<PrefixCacheScorer>(), 2)});
  return p;
}
static std::shared_ptr<PredictedLatencyProducer> producer(double buffer) {
  auto p = std::make_shared<PredictedLatencyProducer>();
  p->SLOBufferFactor = buffer;
  p->EndpointRoleLabel = kRole;
  p->TTFTIntercept = 12.5;
  p->TPOTIntercept = 9.0;
  p->TTFTCoeffs = {{"kv_cache_percentage", 80.0}, {"input_token_length", 0.031}, {"num_request_waiting", 7.25},
                   {"num_request_running", 1.5}, {"prefix_cache_score", -40.0}};
  p->TPOTCoeffs = {{"kv_cache_percentage", 11.0}, {"input_token_length", 0.0007}, {"num_request_waiting", 0.9},
                   {"num_request_running", 0.35}, {"num_tokens_generated", 0.01}};
  p->TrackRunningRequests = true;
  return p;
}
static SchedulerProfile latency_profile(std::shared_ptr<PredictedLatencyProducer> prod) {
  SchedulerProfile p;
  p.WithScorers({NewWeightedScorer(std::make_shared<LatencyScorer>(), 1), NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 0.5)});
  p.WithPredictedLatencyProducer(std::move(prod));
  return p;
}

static SchedulerConfig multi_config(SchedulerProfile dec, SchedulerProfile pre) {
  SchedulerConfig c;
  c.MaxEndpoints = 64;
  c.TieMode = EPPSCORE_TIE_LOWEST_INDEX;
  c.TieSeed = kSeed;
  c.Prefix.BlockSizeTokens = 16;
  c.Prefix.AutoTune = false;
  c.Profiles = {{"decode", dec.WithEndpointSubset([](const Endpoint& e) { return e.GetMetadata()->Labels.at(kRole) == "decode"; })},
                {"prefill", pre.WithEndpointSubset([](const Endpoint& e) { return e.GetMetadata()->Labels.at(kRole) == "prefill"; })}};
  c.Handler = std::make_shared<PdHandler>();
  return c;
}

static SchedulerConfig single_config(SchedulerProfile p, const char* role, uint64_t seed) {
  SchedulerConfig c;
  c.MaxEndpoints = 64;
  c.CpuBatchThreshold = 0;
  c.TieMode = EPPSCORE_TIE_LOWEST_INDEX;
  c.TieSeed = seed;
  c.Prefix.BlockSizeTokens = 16;
  c.Prefix.AutoTune = false;
  c.Profile = p.WithFilters({std::make_shared<RoleFilter>(role)});
  return c;
}

static bool same_list(const std::vector<ScoredEndpoint>& a, const std::vector<ScoredEndpoint>& b) {
  if (a.size() != b.size()) return false;
  for (size_t i = 0; i < a.size(); i++)
    if (a[i].Index != b[i].Index || a[i].Score != b[i].Score) return false;
  return true;
}

int main() {
  const std::vector<Endpoint> eps = endpoints();
  // lists: decode k = 3, prefill k = 1
  std::unique_ptr<Scheduler> multi;
  try {
    multi = std::make_unique<Scheduler>(multi_config(decode_profile(3), prefill_profile()));
  } catch (const SchedulingError& ex) {
    std::printf("refused %s\n", ex.what());
    std::printf("done\n");
    return 0;
  }
  {
    Scheduler dec(single_config(decode_profile(3), "decode", kSeed));
    Scheduler pre(single_config(prefill_profile(), "prefill", kSeed ^ 0x9E3779B97F4A7C15ull));
    const auto reqs = requests(0);
    auto got = multi->ScheduleBatch(reqs, eps);
    auto wd = dec.ScheduleBatch(reqs, eps), wp = pre.ScheduleBatch(reqs, eps);
    for (size_t r = 0; r < reqs.size(); r++) {
      CHECK(got[r].error.empty() && wd[r].error.empty() && wp[r].error.empty(), "lists: a request failed");
      if (!got[r].error.empty()) continue;
      const auto& d = got[r].result.ProfileResults.at("decode").TargetEndpoints;
      const auto& p = got[r].result.ProfileResults.at("prefill").TargetEndpoints;
      CHECK(d.size() == 3 && p.size() == 1, "lists: decode 3 entries, prefill 1");
      CHECK(same_list(d, wd[r].result.ProfileResults.at("default").TargetEndpoints), "lists: decode equals the filtered single profile");
      CHECK(same_list(p, wp[r].result.ProfileResults.at("default").TargetEndpoints), "lists: prefill equals the filtered single profile");
      CHECK(d[0].TieCount == wd[r].result.ProfileResults.at("default").TargetEndpoints[0].TieCount, "lists: tie count");
      for (const auto& se : d) CHECK(se.Index % 2 == 1, "lists: decode entries stay in their role");
      std::printf("list %d %d %d %d\n", d[0].Index, d[1].Index, d[2].Index, p[0].Index);
    }
    std::printf("lists checked\n");
  }
  // latency scorer on the decode profile with TrackRunningRequests; the prefill profile names the same producer object
  {
    auto prod = producer(1.0);
    Scheduler lat(multi_config(latency_profile(prod), prefill_profile().WithPredictedLatencyProducer(prod)));
    auto prod1 = producer(1.0);
    prod1->TrackRunningRequests = false;  // queues of its own would diverge from the multi scheduler's after round 0
    Scheduler dec(single_config(latency_profile(prod1), "decode", kSeed));
    const auto reqs = requests(1);
    auto got = lat.ScheduleBatch(reqs, eps);
    auto wd = dec.ScheduleBatch(reqs, eps);
    std::vector<int> expect(kEndpoints, 0);
    for (size_t r = 0; r < reqs.size(); r++) {
      CHECK(got[r].error.empty(), "latency: a request failed");
      if (!got[r].error.empty()) continue;
      const auto& a = got[r].result.ProfileResults.at("decode").TargetEndpoints[0];
      const auto& b = wd[r].result.ProfileResults.at("default").TargetEndpoints[0];
      CHECK(a.Index == b.Index && a.Score == b.Score && a.TieCount == b.TieCount, "latency: decode pick equals the filtered single profile");
      expect[(size_t)a.Index]++;
    }
    lat.PreRequest(got);
    auto count = [&](int m) { return lat.RunningRequests(eps[(size_t)m].GetMetadata()->NamespacedName_.String()).second; };
    for (int m = 0; m < kEndpoints; m++) CHECK(count(m) == expect[m], "latency: PreRequest queues the primary target only");
    CHECK(lat.TrackedRequestIds() == reqs.size(), "latency: every request tracked once");
    // the next batch sees the queues (dispatched / min tpot of the decode endpoints)
    auto next = lat.ScheduleBatch(requests(2), eps);
    for (const auto& it : next) CHECK(it.error.empty(), "latency: second batch");
    for (size_t r = 0; r < reqs.size(); r++) lat.ResponseComplete(reqs[r], got[r].result);
    for (int m = 0; m < kEndpoints; m++) CHECK(count(m) == 0, "latency: ResponseComplete removes it there");
    CHECK(lat.TrackedRequestIds() == 0, "latency: no id left");
    std::printf("latency checked\n");
  }
  // producers: two different ones are refused, two equal ones accepted
  {
    std::string why;
    try {
      Scheduler bad(multi_config(latency_profile(producer(1.0)), prefill_profile().WithPredictedLatencyProducer(producer(2.0))));
    } catch (const SchedulingError& ex) {
      why = ex.what();
    }
    CHECK(why.find("different predicted-latency producers") != std::string::npos, "producers: different ones refused");
    bool ok = true;
    try {
      Scheduler good(multi_config(latency_profile(producer(1.0)), prefill_profile().WithPredictedLatencyProducer(producer(1.0))));
    } catch (const SchedulingError&) {
      ok = false;
    }
    CHECK(ok, "producers: equal ones accepted");
    std::printf("producers checked\n");
  }
  std::printf(g_fail ? "FAILED\n" : "done\n");
  return g_fail ? 1 : 0;
}
