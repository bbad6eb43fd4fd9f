// host_inorder_index_test.cpp — SchedulerConfig::InOrderPrefixIndex in the C++ host mirror (epp_scheduler.hpp): each engine batch
// goes through eppscore_schedule_batch_inorder_index, so its picks, the in-flight counters and the prefix index after
// ScheduleBatch + PreRequest equal those of a Scheduler fed one request at a time (Schedule then PreRequest for each request);
// the index is committed once (PreRequest does not commit the batch again); the target's PrefixCacheMatchInfo is its match
// before the request's own Add; a batch cut into LoRA pieces runs its pieces in order; and every refusal.  Linked against the
// oracle-backed stand-in of the C ABI (oracle_backed_inorder_index.cpp + oracle_backed_inflight.cpp).  Built with
// -DEPP_NO_INORDER_INDEX_SYMBOL against a stand-in without the call, it checks only the refusal of a library that lacks it.
#include <cstdio>
#include <string>
#include <vector>

#include "../../gateway-api-inference-extension_b200/host/epp_scheduler.hpp"

using namespace epp;

#ifndef EPP_NO_INORDER_INDEX_SYMBOL
extern uint64_t g_inorder_index_calls, g_host_commits;  // oracle_backed_inorder_index.cpp
std::vector<uint64_t> StandInLruKeys(eppscore_engine* e, int32_t endpoint);
int64_t StandInNumHashes(eppscore_engine* e);
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
static const ScoredEndpoint& Target(const Scheduler::BatchItem& it) { return it.result.ProfileResults.at("default").TargetEndpoints[0]; }
static std::string Name(const Scheduler::BatchItem& it) { return Target(it).Endpoint_->GetMetadata()->NamespacedName_.Name; }

static SchedulerConfig Config(bool index, bool match_info = true) {
  SchedulerConfig c;
  c.Profile.WithScorers({NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1),
                         NewWeightedScorer(std::make_shared<PrefixCacheScorer>(), 3),
                         NewWeightedScorer(std::make_shared<TokenLoadScorer>(2000), 1)})
      .WithPicker(MaxScorePicker{});
  c.MaxEndpoints = 8;
  c.PrefixCapacity = 4096;
  c.InFlightLoad = std::make_shared<InFlightLoadProducer>();
  c.InOrderInFlightLoad = true;
  c.InOrderPrefixIndex = index;
  c.PrefixMatchInfo = match_info && index;
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
#ifdef EPP_NO_INORDER_INDEX_SYMBOL
    CHECK(!EngineHasInOrderPrefixIndex());
    CHECK(Refused(Config(true), "eppscore_schedule_batch_inorder_index"));
#else
    const std::vector<Endpoint> pods = {Pod("podA", 0.30), Pod("podB", 0.32), Pod("podC", 0.35), Pod("podD", 0.50)};
    // two fresh shared prefixes of 8 blocks (64 characters each), unique 2-block tails, arriving interleaved
    const std::string pa(512, 'a'), pb(512, 'b');
    std::vector<InferenceRequest> reqs;
    for (int i = 0; i < 12; i++) {
      std::string tail(128, (char)('c' + i));
      reqs.push_back(InferenceRequest{std::to_string(i), "m", (i % 2 ? pb : pa) + tail, ""});
    }

    // 1. the reference's sequence: one request at a time, PreRequest after each (its own commit every time)
    Scheduler seq(Config(false));
    std::vector<std::string> want;
    const uint64_t commits0 = g_host_commits;
    for (const auto& q : reqs) {
      auto r = seq.ScheduleBatch({q}, pods);
      CHECK(r[0].error.empty());
      want.push_back(Name(r[0]));
      seq.PreRequest(r);
    }
    CHECK(g_host_commits == commits0 + reqs.size());

    // 2. one batch in order against the index: the same picks, the index committed inside the call and never again
    Scheduler s(Config(true));
    const uint64_t calls0 = g_inorder_index_calls, c1 = g_host_commits;
    auto rb = s.ScheduleBatch(reqs, pods);
    CHECK(g_inorder_index_calls == calls0 + 1);
    std::vector<std::string> got;
    for (auto& it : rb) got.push_back(it.error.empty() ? Name(it) : "");
    CHECK(got == want);
    s.PreRequest(rb);
    CHECK(g_host_commits == c1);  // PreRequest committed nothing
    for (int id = 0; id < 4; id++) CHECK(StandInLruKeys(s.engine(), id) == StandInLruKeys(seq.engine(), id));
    CHECK(StandInNumHashes(s.engine()) == StandInNumHashes(seq.engine()));
    CHECK(StandInNumHashes(s.engine()) > 0);
    for (const auto& p : pods) {
      const std::string n = "/" + p.GetMetadata()->NamespacedName_.Name;
      CHECK(s.InFlightLoad(n) == seq.InFlightLoad(n));
    }

    // 3. PrefixCacheMatchInfo is the match before the request's own Add: the first request of each prefix sees nothing, a
    // later request on an endpoint an earlier one of its prefix went to sees the 8 shared blocks (its tail is its own)
    for (size_t r = 0; r < rb.size(); r++) {
      const ScoredEndpoint& t = Target(rb[r]);
      CHECK(t.PrefixMatch.has_value());
      if (!t.PrefixMatch) continue;
      CHECK(t.PrefixMatch->TotalBlocks == 10);
      bool earlier_same = false;
      for (size_t q = r % 2; q < r; q += 2) earlier_same = earlier_same || got[q] == got[r];
      CHECK(t.PrefixMatch->MatchBlocks == (earlier_same ? 8 : 0));
    }
    CHECK(Target(rb[0]).PrefixMatch && Target(rb[0]).PrefixMatch->MatchBlocks == 0);
    int followed = 0;  // requests that found an earlier request's fresh prefix on their target
    for (const auto& it : rb) followed += Target(it).PrefixMatch && Target(it).PrefixMatch->MatchBlocks == 8;
    CHECK(followed >= 6);
    CHECK(s.PrefixIndexerMetrics().HitBytes.Count == reqs.size());

    // 4. a second batch follows the prefixes the first one placed
    auto rb2 = s.ScheduleBatch(reqs, pods);
    for (size_t r = 0; r < rb2.size(); r++) CHECK(rb2[r].error.empty() && Target(rb2[r]).PrefixMatch->MatchBlocks >= 8);

    // 5. refusals
    {
      SchedulerConfig c = Config(true);
      c.InOrderInFlightLoad = false;
      CHECK(Refused(c, "InOrderInFlightLoad"));
    }
    {
      SchedulerConfig c = Config(true);
      c.InFlightLoad = nullptr;
      CHECK(Refused(c, "InFlightLoad"));
    }
    {
      SchedulerConfig c = Config(true);
      c.Prefix.MaxPrefixBlocksToMatch = 0;
      CHECK(Refused(c, "approximate-prefix"));
    }
    {
      SchedulerConfig c = Config(true);
      c.LatencyPredictionInfo = true;
      CHECK(Refused(c, "LatencyPredictionInfo"));
    }
    {
      SchedulerConfig c = Config(true);
      c.Profile.WithPicker(MaxScorePicker{2});
      CHECK(Refused(c, "maxNumOfEndpoints"));
    }
    {
      SchedulerConfig c = Config(true);
      c.Profiles = {{"decode", c.Profile}, {"prefill", c.Profile}};
      CHECK(Refused(c, nullptr));
    }
#endif
  } catch (const std::exception& ex) {
    std::printf("FAIL exception: %s\n", ex.what());
    return 1;
  }
  if (g_fail) {
    std::printf("host inorder index: %d checks failed\n", g_fail);
    return 1;
  }
  std::printf("host inorder index: all checks passed\n");
  return 0;
}
