// host_inorder_profiles_test.cpp — SchedulerConfig::InOrderInFlightLoad and InOrderPrefixIndex with the Profiles list, on the
// oracle-backed stand-in of the C ABI (oracle_backed_inorder_profiles.cpp).  A decode / "prefill" handler over the two halves of
// the pool, the prefill profile skipped for every fifth request.  Checks, and prints one line per check for
// tests/test_host_inorder_profiles_cpu.py:
//   - with each option, ScheduleBatch + PreRequest of whole batches give the picks, scores, tie counts, in-flight counters and
//     index (every LRU, len(hashToPods)) of the batch route fed one request at a time, each followed by PreRequest;
//   - the batch goes through one in-order call, and PreRequest adds no load and commits nothing more;
//   - with InOrderPrefixIndex and PrefixMatchInfo, every target's PrefixCacheMatchInfo is the match at that target before the
//     request's Adds;
//   - a handler that names another primary profile gets the per-request error;
//   - the refusals (InOrderRunningRequests with Profiles, maxNumOfEndpoints 2, a library without the call).
#include <cstdio>
#include <string>
#include <vector>

#include "../../gateway-api-inference-extension_b200/host/epp_scheduler.hpp"
#include "../../oracle/oracle.h"

extern "C" orc_index* oracle_backed_index(eppscore_engine* e);
extern uint64_t g_inorder_profiles_calls __attribute__((weak));

using namespace epp;

static int g_fail = 0;
#define CHECK(cond, what)             \
  do {                                \
    if (!(cond)) {                    \
      std::printf("FAIL %s\n", what); \
      g_fail++;                       \
    }                                 \
  } while (0)

struct PdHandler : ProfileHandler {
  std::string primary = "decode";
  std::vector<std::string> Pick(const InferenceRequest& q, const std::vector<std::string>&,
                                const std::map<std::string, const ProfileRunResult*>& results) override {
    if (!results.empty()) return {};
    const int r = std::stoi(q.RequestId.substr(q.RequestId.find('-') + 1));
    return r % 5 == 3 ? std::vector<std::string>{"decode"} : std::vector<std::string>{"decode", "prefill"};
  }
  SchedulingResult ProcessResults(const InferenceRequest&, const std::map<std::string, const ProfileRunResult*>& res) override {
    if (!res.at("decode")) throw SchedulingError("failed to run scheduler profile 'decode'");
    SchedulingResult r;
    for (const auto& kv : res)
      if (kv.second) r.ProfileResults[kv.first] = *kv.second;
    r.PrimaryProfileName = primary;
    return r;
  }
};

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
  for (int r = 0; r < 40; r++) {
    std::string prompt(256, 'a' + ((r + round) % 4));  // four shared prefixes of four blocks, new to the index each round
    prompt += std::string(64 * (round + 1), 'A' + round);
    prompt += std::string(96, 'k' + ((r * 3 + round) % 11));
    InferenceRequest q{"r" + std::to_string(round) + "-" + std::to_string(r), "m", prompt, ""};
    q.RequestSizeBytes = 400 + 8 * r;
    reqs.push_back(q);
  }
  return reqs;
}

static SchedulerConfig config(std::shared_ptr<ProfileHandler> h, bool in_order, bool index, int k = 1, bool prefix = true) {
  auto tl = std::make_shared<TokenLoadScorer>();
  tl->QueueThresholdTokens = 2000;
  SchedulerProfile dec, pre;
  if (prefix) {
    dec.WithScorers({NewWeightedScorer(std::make_shared<QueueScorer>(), 1), NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1),
                     NewWeightedScorer(std::make_shared<PrefixCacheScorer>(), 3), NewWeightedScorer(tl, 3)});
    pre.WithScorers({NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1), NewWeightedScorer(std::make_shared<PrefixCacheScorer>(), 3),
                     NewWeightedScorer(tl, 3)});
  } else {  // (the in-flight form leaves the index to PreRequest: the request-at-a-time route would see earlier requests' blocks)
    dec.WithScorers({NewWeightedScorer(std::make_shared<QueueScorer>(), 1), NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1),
                     NewWeightedScorer(tl, 3)});
    pre.WithScorers({NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1), NewWeightedScorer(tl, 3)});
  }
  MaxScorePicker pk;
  pk.MaxNumOfEndpoints = k;
  pre.WithPicker(pk);
  SchedulerConfig c;
  c.MaxEndpoints = 64;
  c.TieMode = EPPSCORE_TIE_LOWEST_INDEX;
  c.TieSeed = 77;
  c.Prefix.BlockSizeTokens = 16;
  c.Prefix.AutoTune = false;
  c.InFlightLoad = std::make_shared<InFlightLoadProducer>();
  c.Profiles = {{"decode", dec.WithEndpointSubset([](const Endpoint& e) { return e.GetMetadata()->Labels.at("role") == "decode"; })},
                {"prefill", pre.WithEndpointSubset([](const Endpoint& e) { return e.GetMetadata()->Labels.at("role") == "prefill"; })}};
  c.Handler = std::move(h);
  c.InOrderInFlightLoad = in_order;
  c.InOrderPrefixIndex = index;
  c.PrefixMatchInfo = index;
  return c;
}

static std::string refusal(const SchedulerConfig& c) {
  try {
    Scheduler s(c);
  } catch (const SchedulingError& ex) {
    return ex.what();
  }
  return "";
}

int main() {
  const std::vector<Endpoint> eps = endpoints();
  auto h = std::make_shared<PdHandler>();
  if (!&g_inorder_profiles_calls) {  // a library without the call
    std::printf("refused %s\n", refusal(config(h, true, false)).c_str());
    std::printf("done\n");
    return 0;
  }
  for (bool index : {false, true}) {
    Scheduler io(config(h, true, index, 1, index)), seq(config(h, false, false, 1, index));
    orc_index* ix_io = oracle_backed_index(io.engine());
    orc_index* ix_seq = oracle_backed_index(seq.engine());
    for (int round = 0; round < 3; round++) {
      const auto reqs = requests(round);
      const uint64_t calls = g_inorder_profiles_calls;
      auto got = io.ScheduleBatch(reqs, eps);
      CHECK(g_inorder_profiles_calls == calls + 1, "one in-order call per batch");
      const int64_t hashes_before = orc_index_num_hashes(ix_io);
      std::vector<std::pair<int64_t, int64_t>> load_before;
      for (const auto& e : eps) load_before.push_back(io.InFlightLoad(e.GetMetadata()->NamespacedName_.String()));
      io.PreRequest(got);
      for (size_t m = 0; m < eps.size(); m++)
        CHECK(io.InFlightLoad(eps[m].GetMetadata()->NamespacedName_.String()) == load_before[m], "PreRequest adds no load");
      if (index) CHECK(orc_index_num_hashes(ix_io) == hashes_before, "PreRequest commits nothing more");
      for (size_t r = 0; r < reqs.size(); r++) {
        uint64_t hh[64];
        const uint64_t seed = orc_model_seed("m", 1, "", 0);
        const int n = orc_hash_prompt(reinterpret_cast<const uint8_t*>(reqs[r].Prompt.data()), (int64_t)reqs[r].Prompt.size(), seed, 64, 256, hh, 64);
        std::vector<uint16_t> before(24, 0);
        if (n > 0) orc_match_longest_prefix(ix_seq, hh, n, 24, before.data());
        auto want = seq.ScheduleBatch({reqs[r]}, eps);
        seq.PreRequest(want);
        CHECK(got[r].error.empty() && want[0].error.empty(), "request failed");
        if (!got[r].error.empty() || !want[0].error.empty()) continue;
        const auto& a = got[r].result.ProfileResults;
        const auto& b = want[0].result.ProfileResults;
        CHECK(a.size() == b.size() && a.count("prefill") == (r % 5 == 3 ? 0u : 1u), "the handler's profiles ran");
        for (const auto& kv : b) {
          if (!a.count(kv.first)) continue;
          const auto& x = a.at(kv.first).TargetEndpoints[0];
          const auto& y = kv.second.TargetEndpoints[0];
          CHECK(x.Index == y.Index && x.Score == y.Score && x.TieCount == y.TieCount, "pick equals the request-at-a-time route");
          if (index) {
            const int id = io.ServerId(x.Endpoint_->GetMetadata()->NamespacedName_.String());
            CHECK(x.PrefixMatch && x.PrefixMatch->MatchBlocks == before[(size_t)id] && x.PrefixMatch->TotalBlocks == n,
                  "PrefixCacheMatchInfo before the request's Adds");
          }
        }
      }
      for (const auto& e : eps) {
        const std::string id = e.GetMetadata()->NamespacedName_.String();
        if (io.InFlightLoad(id) != seq.InFlightLoad(id))
          std::printf("FAIL in-flight counters %s %ld/%ld vs %ld/%ld\n", id.c_str(), (long)io.InFlightLoad(id).first, (long)io.InFlightLoad(id).second,
                      (long)seq.InFlightLoad(id).first, (long)seq.InFlightLoad(id).second), g_fail++;
      }
      CHECK(orc_index_num_hashes(ix_io) == orc_index_num_hashes(ix_seq), "len(hashToPods)");
      for (int m = 0; m < 24; m++) {
        std::vector<uint64_t> x(4096), y(4096);
        const int nx = orc_index_lru_keys(ix_io, m, x.data(), 4096), ny = orc_index_lru_keys(ix_seq, m, y.data(), 4096);
        CHECK(nx == ny && std::equal(x.begin(), x.begin() + std::max(nx, 0), y.begin()), "every LRU in reference order");
      }
    }
    std::printf(index ? "index form checked\n" : "in-flight form checked\n");
  }
  {  // another primary: the per-request error
    auto other = std::make_shared<PdHandler>();
    other->primary = "prefill";
    Scheduler io(config(other, true, true));
    for (auto& it : io.ScheduleBatch(requests(0), eps))
      CHECK(it.error.find("first profile's target ('decode')") != std::string::npos, "another primary refused per request");
    std::printf("primary checked\n");
  }
  SchedulerConfig c = config(h, true, true);
  c.InOrderRunningRequests = true;
  CHECK(refusal(c).find("InOrderRunningRequests serves the single-profile config") != std::string::npos, "running requests refused");
  CHECK(refusal(config(h, true, true, 2)).find("maxNumOfEndpoints") != std::string::npos, "lists refused");
  std::printf("refusals checked\n");
  std::printf(g_fail ? "FAILED\n" : "done\n");
  return g_fail ? 1 : 0;
}
