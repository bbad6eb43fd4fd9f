// host_inorder_test.cpp — SchedulerConfig::InOrderInFlightLoad in the C++ host mirror (epp_scheduler.hpp): each engine batch goes
// through eppscore_schedule_batch_inorder, so its picks and the in-flight counters after ScheduleBatch + PreRequest equal the
// reference's per-request sequence (Schedule then PreRequest for each request, inflightload/producer.go:101-120 feeding
// token_load.go:83-111); PreRequest does not add the load a second time; ResponseComplete releases it; every refusal; and with
// the option off the host layer makes the calls it always made.  Linked against the oracle-backed stand-in of the C ABI
// (oracle_backed_inorder.cpp + oracle_backed_inflight.cpp).  Built with -DEPP_NO_INORDER_SYMBOL against a stand-in without
// the call, it checks only the refusal of a library that lacks it.
#include <algorithm>
#include <cstdio>
#include <string>
#include <vector>

#include "../../gateway-api-inference-extension_b200/host/epp_scheduler.hpp"

using namespace epp;

#ifndef EPP_NO_INORDER_SYMBOL
extern uint64_t g_inorder_calls;  // oracle_backed_inorder.cpp
#endif

static int g_fail = 0;
#define CHECK(cond)                                               \
  do {                                                            \
    if (!(cond)) {                                                \
      std::printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); \
      g_fail++;                                                   \
    }                                                             \
  } while (0)

static Endpoint Pod(const std::string& name, double kv) {
  Metrics m;
  m.KVCacheUsagePercent = kv;
  return NewEndpoint(name, m);
}
static std::string Name(const Scheduler::BatchItem& it) {
  return it.result.ProfileResults.at("default").TargetEndpoints[0].Endpoint_->GetMetadata()->NamespacedName_.Name;
}
static InferenceRequest Req(const std::string& id, size_t chars) { return InferenceRequest{id, "m", std::string(chars, 'x'), ""}; }

static SchedulerConfig Config(bool producer, bool inorder) {
  SchedulerConfig c;
  // kv differs a little between pods; a 200-token threshold lets a few requests' load outweigh it
  c.Profile.WithScorers({NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1),
                         NewWeightedScorer(std::make_shared<TokenLoadScorer>(200), 1)})
      .WithPicker(MaxScorePicker{});
  c.Prefix.MaxPrefixBlocksToMatch = 0;
  c.MaxEndpoints = 8;
  c.PrefixCapacity = 256;
  if (producer) c.InFlightLoad = std::make_shared<InFlightLoadProducer>();
  c.InOrderInFlightLoad = inorder;
  return c;
}

static bool Refused(const SchedulerConfig& c, const char* what) {
  try {
    Scheduler s(c);
  } catch (const SchedulingError& ex) {
    if (what && std::string(ex.what()).find(what) == std::string::npos) {
      std::printf("  unexpected refusal: %s\n", ex.what());
      return false;
    }
    return true;
  }
  return false;
}

int main() {
  try {
#ifdef EPP_NO_INORDER_SYMBOL
    CHECK(!EngineHasInOrderLoad());
    CHECK(Refused(Config(true, true), "eppscore_schedule_batch_inorder"));
    {  // the option off still builds and runs
      Scheduler s(Config(true, false));
      auto r = s.ScheduleBatch({Req("1", 40)}, {Pod("podA", 0.5)});
      CHECK(r[0].error.empty());
    }
#else
    const std::vector<Endpoint> pods = {Pod("podA", 0.30), Pod("podB", 0.32), Pod("podC", 0.35), Pod("podD", 0.50)};
    std::vector<InferenceRequest> reqs;
    for (int i = 0; i < 12; i++) reqs.push_back(Req(std::to_string(i), 40 + 8 * (size_t)(i % 5)));
    reqs[3].RequestSizeBytes = 600;
    reqs[7].InputTokenCountHint = 30;

    // 1. the reference's sequence: one request at a time, PreRequest after each
    Scheduler seq(Config(true, false));
    std::vector<std::string> want;
    for (const auto& q : reqs) {
      auto r = seq.ScheduleBatch({q}, pods);
      CHECK(r[0].error.empty());
      want.push_back(Name(r[0]));
      seq.PreRequest(r);
    }

    // 2. one batch in order: the same picks; the load is counted while scheduling, and PreRequest adds nothing more
    Scheduler s(Config(true, true));
    const uint64_t calls0 = g_inorder_calls;
    auto rb = s.ScheduleBatch(reqs, pods);
    CHECK(g_inorder_calls == calls0 + 1);
    std::vector<std::string> got;
    for (auto& it : rb) got.push_back(it.error.empty() ? Name(it) : "");
    CHECK(got == want);
    int distinct = 0;
    for (const char* n : {"podA", "podB", "podC", "podD"}) distinct += std::find(got.begin(), got.end(), n) != got.end();
    CHECK(distinct >= 3);  // the batch spreads
    std::vector<std::pair<int64_t, int64_t>> before;
    for (const auto& p : pods) before.push_back(s.InFlightLoad("/" + p.GetMetadata()->NamespacedName_.Name));
    s.PreRequest(rb);
    for (size_t m = 0; m < pods.size(); m++) {
      const std::string n = "/" + pods[m].GetMetadata()->NamespacedName_.Name;
      CHECK(s.InFlightLoad(n) == before[m]);   // no second add
      CHECK(s.InFlightLoad(n) == seq.InFlightLoad(n));  // the sequence's counters
    }
    CHECK(s.CpuRoutedRequests() == 0);

    // 3. the release path: ResponseComplete gives back what the batch added
    for (size_t i = 0; i < reqs.size(); i++) s.ResponseComplete(reqs[i], rb[i].result);
    for (const auto& p : pods) CHECK(s.InFlightLoad("/" + p.GetMetadata()->NamespacedName_.Name) == std::make_pair((int64_t)0, (int64_t)0));

    // 4. a second batch after the release starts from 0 again: the same picks as the first
    auto rb2 = s.ScheduleBatch(reqs, pods);
    for (size_t i = 0; i < reqs.size(); i++) CHECK(rb2[i].error.empty() && Name(rb2[i]) == want[i]);

    // 5. option off: today's calls and results — one load view (every request on podA), no in-order call, PreRequest adds
    {
      Scheduler off(Config(true, false));
      const uint64_t c0 = g_inorder_calls;
      auto r = off.ScheduleBatch(reqs, pods);
      for (auto& it : r) CHECK(Name(it) == "podA");
      CHECK(off.InFlightLoad("/podA") == std::make_pair((int64_t)0, (int64_t)0));
      off.PreRequest(r);
      CHECK(off.InFlightLoad("/podA").first == (int64_t)reqs.size());
      CHECK(g_inorder_calls == c0);
    }

    // 6. refusals
    CHECK(Refused(Config(false, true), "InFlightLoad"));
    {
      SchedulerConfig c = Config(true, true);
      c.Profile.WithPicker(MaxScorePicker{2});
      CHECK(Refused(c, "maxNumOfEndpoints"));
    }
    {
      SchedulerConfig c = Config(true, true);
      c.Profile.WithScorers({NewWeightedScorer(std::make_shared<LatencyScorer>(), 1),
                             NewWeightedScorer(std::make_shared<TokenLoadScorer>(200), 1)});
      CHECK(Refused(c, "latency"));
    }
    {
      SchedulerConfig c = Config(true, true);
      c.Profiles = {{"decode", c.Profile}, {"prefill", c.Profile}};
      CHECK(Refused(c, nullptr));
    }
#endif
  } catch (const std::exception& ex) {
    std::printf("FAIL exception: %s\n", ex.what());
    return 1;
  }
  if (g_fail) {
    std::printf("host inorder: %d checks failed\n", g_fail);
    return 1;
  }
  std::printf("host inorder: all checks passed\n");
  return 0;
}
