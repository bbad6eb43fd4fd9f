// host_inorder_latency_test.cpp — SchedulerConfig::InOrderRunningRequests in the C++ host mirror (epp_scheduler.hpp): each engine
// batch goes through eppscore_schedule_batch_inorder_latency, so its picks, the in-flight counters, the running-request queues
// (and, with InOrderPrefixIndex, the prefix index) after ScheduleBatch + PreRequest equal those of a Scheduler fed one request at
// a time (Schedule then PreRequest for each request); each request is added to its queue exactly once (PreRequest adds nothing);
// ResponseComplete removes what the call added; and every refusal.  Linked against the oracle-backed stand-in of the C ABI
// (oracle_backed_inorder_latency.cpp + oracle_backed_inflight.cpp + oracle_backed_running.cpp), or against the engine itself
// (engine_inorder_latency_shim.cpp).  Built with -DEPP_NO_INORDER_LATENCY_SYMBOL against a stand-in without the call, it checks
// only the refusal of a library that lacks it.
#include <cstdio>
#include <string>
#include <vector>

#include "../../gateway-api-inference-extension_b200/host/epp_scheduler.hpp"

using namespace epp;

#ifndef EPP_NO_INORDER_LATENCY_SYMBOL
extern uint64_t g_inorder_latency_calls, g_host_running_adds;
std::vector<uint64_t> StandInLruKeys(eppscore_engine* e, int32_t endpoint);
#endif

static int g_fail = 0;
#define CHECK(cond)                                               \
  do {                                                            \
    if (!(cond)) {                                                \
      std::printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); \
      g_fail++;                                                   \
    }                                                             \
  } while (0)

static Endpoint Pod(const std::string& name, double kv, int64_t waiting, int64_t running) {
  Metrics m;
  m.KVCacheUsagePercent = kv;
  m.WaitingQueueSize = waiting;    // TTFT = waiting
  m.RunningRequestsSize = running;  // TPOT = running: a running request's tighter TPOT SLO can take the endpoint negative
  return NewEndpoint(name, m, "default");
}
static const ScoredEndpoint& Target(const Scheduler::BatchItem& it) { return it.result.ProfileResults.at("default").TargetEndpoints[0]; }
static std::string Name(const Scheduler::BatchItem& it) { return it.error.empty() ? Target(it).Endpoint_->GetMetadata()->NamespacedName_.Name : ""; }

static SchedulerConfig Config(bool inorder, bool index, bool track = true) {
  SchedulerConfig c;
  auto prod = std::make_shared<PredictedLatencyProducer>();
  prod->StreamingMode = true;
  prod->TTFTCoeffs["num_request_waiting"] = 1.0;
  prod->TPOTCoeffs["num_request_running"] = 1.0;
  prod->TrackRunningRequests = track;
  std::vector<WeightedScorer> sc = {NewWeightedScorer(std::make_shared<LatencyScorer>(), 2),
                                    NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1),
                                    NewWeightedScorer(std::make_shared<TokenLoadScorer>(2000), 1)};
  if (index) sc.push_back(NewWeightedScorer(std::make_shared<PrefixCacheScorer>(), 1));
  c.Profile.WithScorers(sc).WithPicker(MaxScorePicker{}).WithPredictedLatencyProducer(prod);
  if (!index) c.Prefix.MaxPrefixBlocksToMatch = 0;
  c.MaxEndpoints = 8;
  c.PrefixCapacity = 4096;
  c.InFlightLoad = std::make_shared<InFlightLoadProducer>();
  c.InOrderInFlightLoad = inorder;
  c.InOrderPrefixIndex = inorder && index;
  c.InOrderRunningRequests = inorder;
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

#ifndef EPP_NO_INORDER_LATENCY_SYMBOL
static void Compare(bool index, bool track) {
  const std::vector<Endpoint> pods = {Pod("podA", 0.30, 100, 10), Pod("podB", 0.32, 120, 15), Pod("podC", 0.35, 90, 20),
                                      Pod("podD", 0.50, 110, 25)};
  const char* tpots[] = {"30", "12", "", "40", "18", "26", "-1", "30"};
  std::vector<InferenceRequest> reqs;
  for (int i = 0; i < 24; i++) {
    std::string id = i == 5 ? "" : (i == 9 ? "r3" : "r" + std::to_string(i));  // no id; an id already in the batch
    InferenceRequest q{id, "m", std::string(256, (char)('a' + i % 3)) + " some words " + std::to_string(i), ""};
    q.Headers["x-slo-ttft-ms"] = i % 4 == 0 ? "50" : "1000";
    if (tpots[i % 8][0]) q.Headers["x-slo-tpot-ms"] = tpots[i % 8];
    reqs.push_back(q);
  }
  // 1. the reference's sequence: one request at a time, PreRequest after each
  Scheduler seq(Config(false, index, track));
  std::vector<std::string> want;
  std::vector<Scheduler::BatchItem> seq_items;
  for (const auto& q : reqs) {
    auto r = seq.ScheduleBatch({q}, pods);
    want.push_back(Name(r[0]));
    seq.PreRequest(r);
    seq_items.push_back(r[0]);
  }
  // 2. one batch in order: the same picks, the queues added inside the call and never again
  Scheduler s(Config(true, index, track));
  const uint64_t calls0 = g_inorder_latency_calls, adds0 = g_host_running_adds;
  auto rb = s.ScheduleBatch(reqs, pods);
  CHECK(g_inorder_latency_calls == calls0 + 1);
  std::vector<std::string> got;
  for (auto& it : rb) got.push_back(Name(it));
  CHECK(got == want);
  s.PreRequest(rb);
  CHECK(g_host_running_adds == adds0);  // PreRequest added nothing: one Add per request, inside the call
  int live = 0;
  for (const auto& p : pods) {
    const std::string n = p.GetMetadata()->NamespacedName_.String();
    CHECK(s.InFlightLoad(n) == seq.InFlightLoad(n));
    CHECK(s.RunningRequests(n) == seq.RunningRequests(n));
    live += s.RunningRequests(n).second;
  }
  CHECK(s.TrackedRequestIds() == seq.TrackedRequestIds());
  if (track) CHECK(live > 0 && live < (int)reqs.size());  // some adds refused: no id, a negative tpot, a live pair
  else CHECK(live == 0);
  if (index)
    for (int id = 0; id < 4; id++) CHECK(StandInLruKeys(s.engine(), id) == StandInLruKeys(seq.engine(), id));
  // 3. ResponseComplete removes what the call added
  for (size_t r = 0; r < reqs.size(); r++)
    if (rb[r].error.empty()) s.ResponseComplete(reqs[r], rb[r].result);
  for (const auto& p : pods) CHECK(s.RunningRequests(p.GetMetadata()->NamespacedName_.String()).second == 0);
  CHECK(s.TrackedRequestIds() == 0);
}
#endif

int main() {
  try {
#ifdef EPP_NO_INORDER_LATENCY_SYMBOL
    CHECK(!EngineHasInOrderLatency());
    CHECK(Refused(Config(true, false), "eppscore_schedule_batch_inorder_latency"));
#else
    CHECK(EngineHasInOrderLatency());
    Compare(false, true);
    Compare(true, true);
    Compare(false, false);
    // refusals
    {
      SchedulerConfig c = Config(true, false);
      c.InOrderInFlightLoad = false;
      CHECK(Refused(c, "InOrderInFlightLoad"));
    }
    {
      SchedulerConfig c = Config(true, false);
      c.LatencyPredictionInfo = true;
      CHECK(Refused(c, "LatencyPredictionInfo"));
    }
    {
      SchedulerConfig c = Config(true, false);
      c.Profile.WithPicker(MaxScorePicker{2});
      CHECK(Refused(c, "maxNumOfEndpoints"));
    }
    {
      SchedulerConfig c = Config(true, false);
      c.Profiles = {{"decode", c.Profile}, {"prefill", c.Profile}};
      CHECK(Refused(c, nullptr));
    }
    {
      SchedulerConfig c = Config(true, false);
      c.Profile.WithScorers({NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1)});
      CHECK(Refused(c, "latency-scorer"));
    }
    {
      SchedulerConfig c = Config(true, false);
      c.Profile.WithDeviceFilters({SLOHeadroomTierFilter()});
      CHECK(Refused(c, "device filters"));
    }
    {  // with the option off, a latency profile is still refused by InOrderInFlightLoad
      SchedulerConfig c = Config(true, false);
      c.InOrderRunningRequests = false;
      CHECK(Refused(c, "cannot order the latency scorer's inputs"));
    }
#endif
  } catch (const std::exception& ex) {
    std::printf("FAIL exception: %s\n", ex.what());
    return 1;
  }
  if (g_fail) {
    std::printf("host inorder latency: %d checks failed\n", g_fail);
    return 1;
  }
  std::printf("host inorder latency: all checks passed\n");
  return 0;
}
