// host_inflight_test.cpp — the inflight-load-producer in the C++ host mirror (epp_scheduler.hpp): PreRequest counts each
// scheduled request and its estimated tokens on its target endpoint (inflightload/producer.go:101-120), ResponseComplete gives
// them back (:122-169), RemovePod drops the endpoint's counters so a recycled id starts from 0 (:181-187), and a token-load
// scorer (scorer/tokenload/token_load.go:83-111) reads the counters, so the next batch moves away from a loaded endpoint.
// Linked against the oracle-backed stand-in of the C ABI (tests/cpp/oracle_backed_abi.cpp + oracle_backed_inflight.cpp) on the
// CPU, and against libeppscore.so on the GPU.
#include <cstdio>
#include <string>
#include <vector>

#include "../../gateway-api-inference-extension_b200/host/epp_scheduler.hpp"

using namespace epp;

static int g_fail = 0;
#define CHECK(cond)                                               \
  do {                                                            \
    if (!(cond)) {                                                \
      std::printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); \
      g_fail++;                                                   \
    }                                                             \
  } while (0)

static Endpoint Pod(const std::string& name) {
  Metrics m;
  m.KVCacheUsagePercent = 0.5;
  return NewEndpoint(name, m);
}
static std::string Name(const Scheduler::BatchItem& it) {
  return it.result.ProfileResults.at("default").TargetEndpoints[0].Endpoint_->GetMetadata()->NamespacedName_.Name;
}
static InferenceRequest Req(const std::string& id, size_t chars) { return InferenceRequest{id, "m", std::string(chars, 'x'), ""}; }
static bool Load(Scheduler& s, const std::string& name, int64_t requests, int64_t tokens) {
  const auto l = s.InFlightLoad("/" + name);
  if (l.first != requests || l.second != tokens)
    std::printf("  %s: %lld requests, %lld tokens\n", name.c_str(), (long long)l.first, (long long)l.second);
  return l.first == requests && l.second == tokens;
}

static SchedulerConfig Config(bool producer) {
  SchedulerConfig c;
  // equal kv everywhere: the token-load term decides; 100 tokens saturate an endpoint
  c.Profile.WithScorers({NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1),
                         NewWeightedScorer(std::make_shared<TokenLoadScorer>(100), 1)})
      .WithPicker(MaxScorePicker{});
  c.Prefix.MaxPrefixBlocksToMatch = 0;
  c.MaxEndpoints = 8;
  c.PrefixCapacity = 256;
  if (producer) c.InFlightLoad = std::make_shared<InFlightLoadProducer>();
  return c;
}

int main() {
  try {
    std::vector<Endpoint> pods = {Pod("podA"), Pod("podB"), Pod("podC"), Pod("podD")};

    // 1. without the producer every call does what it did before: the small-batch host route, no counters, no feedback
    {
      Scheduler s(Config(false));
      auto r1 = s.ScheduleBatch({Req("1", 40)}, pods);
      s.PreRequest(r1);
      auto r2 = s.ScheduleBatch({Req("2", 40)}, pods);
      CHECK(Name(r1[0]) == "podA" && Name(r2[0]) == "podA");
      CHECK(s.CpuRoutedRequests() == 2);
      CHECK(Load(s, "podA", 0, 0));
      s.ResponseComplete(Req("1", 40), r1[0].result);  // no producer: nothing to release
      CHECK(Load(s, "podA", 0, 0));
    }

    Scheduler s(Config(true));
    // 2. PreRequest counts the request and its estimate (40 chars: 10 input + 15 output tokens); the next batch sees the load
    //    (0.75 on podA) and moves on, one endpoint per batch
    std::vector<Scheduler::BatchItem> sent;
    std::vector<InferenceRequest> reqs;
    const char* order[] = {"podA", "podB", "podC", "podD", "podA"};
    for (int i = 0; i < 5; i++) {
      reqs.push_back(Req(std::to_string(i), 40));
      auto r = s.ScheduleBatch({reqs.back()}, pods);
      CHECK(r[0].error.empty() && Name(r[0]) == order[i]);
      s.PreRequest(r);
      sent.push_back(r[0]);
    }
    CHECK(s.CpuRoutedRequests() == 0);  // the counters live on the engine: no host route
    CHECK(Load(s, "podA", 2, 50) && Load(s, "podB", 1, 25) && Load(s, "podC", 1, 25) && Load(s, "podD", 1, 25));

    // 3. ResponseComplete gives back what PreRequest added
    for (int i = 0; i < 5; i++) s.ResponseComplete(reqs[(size_t)i], sent[(size_t)i].result);
    CHECK(Load(s, "podA", 0, 0) && Load(s, "podB", 0, 0) && Load(s, "podC", 0, 0) && Load(s, "podD", 0, 0));

    // 4. one batch sees one load view: four requests all go to podA; the estimator's other inputs
    //    (RequestSizeBytes 1000: 250 + 375; InputTokenCountHint 7: 7 + 11; an empty prompt: 1 + 2)
    std::vector<InferenceRequest> four = {Req("a", 40), Req("b", 0), Req("c", 3), Req("d", 0)};
    four[1].RequestSizeBytes = 1000;
    four[3].InputTokenCountHint = 7;
    auto rb = s.ScheduleBatch(four, pods);
    for (auto& it : rb) CHECK(Name(it) == "podA");
    s.PreRequest(rb);
    CHECK(Load(s, "podA", 4, 25 + 625 + 3 + 18));
    auto next = s.ScheduleBatch({Req("e", 40)}, pods);
    CHECK(Name(next[0]) == "podB");  // podA saturated: token score 0

    // 5. with the producer, an Endpoint's own InFlightTokens does not reach the token-load scorer
    std::vector<Endpoint> marked = pods;
    marked[1].InFlightTokens = 1 << 20;
    auto rm = s.ScheduleBatch({Req("f", 40)}, marked);
    CHECK(Name(rm[0]) == "podB");

    // 6. RemovePod drops the counters; a new server that gets the recycled id starts from 0; a late release for the removed
    //    server is dropped
    s.PreRequest(rm);
    CHECK(Load(s, "podB", 1, 25));
    const int idB = s.ServerId("/podB");
    s.RemovePod("/podB");
    s.ResponseComplete(Req("f", 40), rm[0].result);
    std::vector<Endpoint> l2 = {Pod("podA"), Pod("podE"), Pod("podC"), Pod("podD")};
    auto re = s.ScheduleBatch({Req("g", 40)}, l2);
    CHECK(s.ServerId("/podE") == idB);
    CHECK(Load(s, "podE", 0, 0));
    CHECK(Name(re[0]) == "podE");  // podA is loaded; podE (the recycled id) is not
    CHECK(Load(s, "podA", 4, 671));
  } catch (const std::exception& ex) {
    std::printf("FAIL exception: %s\n", ex.what());
    return 1;
  }
  if (g_fail) {
    std::printf("host inflight: %d checks failed\n", g_fail);
    return 1;
  }
  std::printf("host inflight: all checks passed\n");
  return 0;
}
