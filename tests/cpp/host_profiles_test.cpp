// host_profiles_test.cpp — the host layer's Scheduler with several profiles (a decode and a "prefill" profile over the two
// halves of the pool, split by a role label), on the oracle-backed stand-in of the C ABI.  Checks, and prints one line per
// check for tests/test_host_profiles_cpu.py:
//   - each profile's pick equals a single-profile Scheduler whose host Filter keeps the same role, with the profile's tie seed;
//   - PreRequest records the decode pick, then the prefill pick, per request: every LRU equals indexer.Add in that order;
//   - in-flight counts after PreRequest (every profile's target), ResponseStarted (prefill released) and ResponseComplete (all);
//   - a handler that asks for a second round gets the batch route's error;
//   - the single-profile output ("single" lines), which a build without the profile calls must print identically.
// Built without the profile calls (oracle_backed_abi.cpp instead of oracle_backed_profiles.cpp), a multi-profile config is
// refused when the Scheduler is built.
#include <cstdio>
#include <string>
#include <vector>

#include "../../gateway-api-inference-extension_b200/host/epp_scheduler.hpp"
#include "../../oracle/oracle.h"

extern "C" orc_index* oracle_backed_index(eppscore_engine* e) __attribute__((weak));

using namespace epp;

static int g_fail = 0;
#define CHECK(cond, what)                         \
  do {                                            \
    if (!(cond)) {                                \
      std::printf("FAIL %s\n", what);             \
      g_fail++;                                   \
    }                                             \
  } while (0)

struct RoleFilter : Filter {
  std::string role;
  explicit RoleFilter(std::string r) : role(std::move(r)) {}
  std::vector<int> Filter_(const InferenceRequest&, const std::vector<Endpoint>& eps, const std::vector<int>& cand) override {
    std::vector<int> out;
    for (int i : cand)
      if (eps[(size_t)i].GetMetadata()->Labels.at("role") == role) out.push_back(i);
    return out;
  }
};

// decode is the primary profile; the prefill result rides along (a P/D handler)
struct PdHandler : ProfileHandler {
  int rounds = 1;
  std::vector<std::string> Pick(const InferenceRequest&, const std::vector<std::string>&,
                                const std::map<std::string, const ProfileRunResult*>& results) override {
    if ((int)(results.empty() ? 0 : 1) >= rounds) return {};
    return results.empty() ? std::vector<std::string>{"decode", "prefill"} : std::vector<std::string>{"decode"};
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

static const uint64_t kSeed = 77;

static std::vector<Endpoint> endpoints() {
  std::vector<Endpoint> eps;
  for (int i = 0; i < 24; i++) {
    Metrics m;
    m.KVCacheUsagePercent = 0.03 * ((i * 7) % 23);
    m.WaitingQueueSize = (i * 5) % 9;
    Endpoint e = NewEndpoint("pod" + std::to_string(i), m);
    e.Metadata.Labels["role"] = i % 2 == 0 ? "prefill" : "decode";
    eps.push_back(e);
  }
  return eps;
}

static std::vector<InferenceRequest> requests(int round) {
  std::vector<InferenceRequest> reqs;
  for (int r = 0; r < 60; r++) {
    std::string prompt(256, 'a' + (r % 5));  // five shared prefixes of four blocks
    prompt += std::string(96, 'k' + ((r * 3 + round) % 11));
    InferenceRequest q{"req" + std::to_string(round) + "-" + std::to_string(r), "m", prompt, ""};
    q.RequestSizeBytes = 400 + 8 * r;
    reqs.push_back(q);
  }
  return reqs;
}

static SchedulerProfile decode_profile() {
  SchedulerProfile p;
  p.WithScorers({NewWeightedScorer(std::make_shared<QueueScorer>(), 2), NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 2),
                 NewWeightedScorer(std::make_shared<PrefixCacheScorer>(), 3)});
  return p;
}
static SchedulerProfile prefill_profile() {
  SchedulerProfile p;
  p.WithScorers({NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1), NewWeightedScorer(std::make_shared<PrefixCacheScorer>(), 2)});
  return p;
}

static SchedulerConfig multi_config(std::shared_ptr<ProfileHandler> h) {
  SchedulerConfig c;
  c.MaxEndpoints = 64;
  c.TieMode = EPPSCORE_TIE_SEEDED_RANDOM;
  c.TieSeed = kSeed;
  c.Prefix.BlockSizeTokens = 16;
  c.Prefix.AutoTune = false;
  c.InFlightLoad = std::make_shared<InFlightLoadProducer>();
  c.Profiles = {{"decode", decode_profile().WithEndpointSubset([](const Endpoint& e) { return e.GetMetadata()->Labels.at("role") == "decode"; })},
                {"prefill", prefill_profile().WithEndpointSubset([](const Endpoint& e) { return e.GetMetadata()->Labels.at("role") == "prefill"; })}};
  c.Handler = std::move(h);
  return c;
}

static SchedulerConfig single_config(SchedulerProfile p, const char* role, uint64_t seed) {
  SchedulerConfig c;
  c.MaxEndpoints = 64;
  c.CpuBatchThreshold = 0;
  c.TieMode = EPPSCORE_TIE_SEEDED_RANDOM;
  c.TieSeed = seed;
  c.Prefix.BlockSizeTokens = 16;
  c.Prefix.AutoTune = false;
  c.Profile = p.WithFilters({std::make_shared<RoleFilter>(role)});
  return c;
}

int main() {
  const std::vector<Endpoint> eps = endpoints();
  // the single-profile path: printed for the comparison with a build without the profile calls
  {
    Scheduler s(single_config(decode_profile(), "decode", kSeed));
    for (auto& it : s.ScheduleBatch(requests(0), eps)) std::printf("single %d %.17g\n", it.result.ProfileResults.at("default").TargetEndpoints[0].Index,
                                                                     it.result.ProfileResults.at("default").TargetEndpoints[0].Score);
  }
  std::unique_ptr<Scheduler> multi;
  auto handler = std::make_shared<PdHandler>();
  try {
    multi = std::make_unique<Scheduler>(multi_config(handler));
  } catch (const SchedulingError& ex) {
    std::printf("refused %s\n", ex.what());
    std::printf("done\n");
    return 0;
  }
  // each profile against a single-profile Scheduler with the same role as a host Filter and the profile's tie seed (the index is
  // empty in round 0 on both sides)
  Scheduler dec(single_config(decode_profile(), "decode", kSeed));
  Scheduler pre(single_config(prefill_profile(), "prefill", kSeed ^ 0x9E3779B97F4A7C15ull));
  const auto reqs0 = requests(0);
  auto got = multi->ScheduleBatch(reqs0, eps);
  auto wd = dec.ScheduleBatch(reqs0, eps), wp = pre.ScheduleBatch(reqs0, eps);
  for (size_t r = 0; r < reqs0.size(); r++) {
    CHECK(got[r].error.empty(), "multi-profile request failed");
    const auto& pr = got[r].result.ProfileResults;
    CHECK(got[r].result.PrimaryProfileName == "decode", "primary profile");
    const auto& a = pr.at("decode").TargetEndpoints[0];
    const auto& b = wd[r].result.ProfileResults.at("default").TargetEndpoints[0];
    CHECK(a.Index == b.Index && a.Score == b.Score && a.TieCount == b.TieCount, "decode pick equals the filtered single profile");
    const auto& c = pr.at("prefill").TargetEndpoints[0];
    const auto& d = wp[r].result.ProfileResults.at("default").TargetEndpoints[0];
    CHECK(c.Index == d.Index && c.Score == d.Score && c.TieCount == d.TieCount, "prefill pick equals the filtered single profile");
    CHECK(a.Index % 2 == 1 && c.Index % 2 == 0, "picks stay in their role");
  }
  std::printf("picks checked\n");
  // PreRequest: indexer.Add(decode pick) then indexer.Add(prefill pick) per request, against the oracle's indexer
  orc_index* want = orc_index_new(31250);
  for (int round = 0; round < 3; round++) {
    const auto reqs = round == 0 ? reqs0 : requests(round);
    if (round > 0) got = multi->ScheduleBatch(reqs, eps);
    multi->PreRequest(got);
    for (size_t r = 0; r < reqs.size(); r++) {
      if (!got[r].error.empty()) continue;
      uint64_t h[64];
      const uint64_t seed = orc_model_seed("m", 1, "", 0);
      const int n = orc_hash_prompt(reinterpret_cast<const uint8_t*>(reqs[r].Prompt.data()), (int64_t)reqs[r].Prompt.size(), seed, 64, 256, h, 64);
      for (const char* name : {"decode", "prefill"}) {
        const auto& te = got[r].result.ProfileResults.at(name).TargetEndpoints;
        orc_index_add(want, h, n, multi->ServerId(te[0].Endpoint_->GetMetadata()->NamespacedName_.String()), 0);
      }
    }
  }
  if (&oracle_backed_index) {
    orc_index* have = oracle_backed_index(multi->engine());
    CHECK(orc_index_num_hashes(want) > 0 && orc_index_num_hashes(have) == orc_index_num_hashes(want), "len(hashToPods)");
    for (int m = 0; m < 24; m++) {
      std::vector<uint64_t> x(4096), y(4096);
      const int nx = orc_index_lru_keys(have, m, x.data(), 4096), ny = orc_index_lru_keys(want, m, y.data(), 4096);
      CHECK(nx == ny && std::equal(x.begin(), x.begin() + std::max(nx, 0), y.begin()), "LRU keys in reference order");
    }
  }
  std::printf("commits checked\n");
  // in-flight load of one more batch: PreRequest counts every profile's target, ResponseStarted gives back the prefill targets,
  // ResponseComplete the decode ones (inflightload/producer.go:101-169)
  std::vector<int64_t> expect(24, 0);
  {
    auto reqs = requests(9);
    auto res = multi->ScheduleBatch(reqs, eps);
    auto load = [&](int m) { return multi->InFlightLoad(eps[(size_t)m].GetMetadata()->NamespacedName_.String()).first; };
    std::vector<int64_t> before(24);
    for (int m = 0; m < 24; m++) before[m] = load(m);
    multi->PreRequest(res);
    for (size_t r = 0; r < reqs.size(); r++)
      for (const auto& kv : res[r].result.ProfileResults) expect[(size_t)kv.second.TargetEndpoints[0].Index]++;
    for (int m = 0; m < 24; m++) CHECK(load(m) - before[m] == expect[m], "PreRequest counts every target");
    for (size_t r = 0; r < reqs.size(); r++) multi->ResponseStarted(reqs[r], res[r].result);
    for (size_t r = 0; r < reqs.size(); r++) expect[(size_t)res[r].result.ProfileResults.at("prefill").TargetEndpoints[0].Index]--;
    for (int m = 0; m < 24; m++) CHECK(load(m) - before[m] == expect[m], "ResponseStarted releases prefill");
    for (size_t r = 0; r < reqs.size(); r++) multi->ResponseComplete(reqs[r], res[r].result);
    for (int m = 0; m < 24; m++) CHECK(load(m) == before[m], "ResponseComplete releases the rest");
  }
  std::printf("inflight checked\n");
  handler->rounds = 2;  // a second round: refused per request
  for (auto& it : multi->ScheduleBatch(requests(5), eps))
    CHECK(it.error == "multi-round profile handlers are not supported by the batch route", "multi-round refused");
  std::printf("multi-round checked\n");
  orc_index_free(want);
  std::printf(g_fail ? "FAILED\n" : "done\n");
  return g_fail ? 1 : 0;
}
