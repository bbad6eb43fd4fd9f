// host_running_test.cpp — PredictedLatencyProducer::TrackRunningRequests in the C++ host mirror (epp_scheduler.hpp): PreRequest
// adds each scheduled request with its x-slo-tpot-ms to its target endpoint's running-request queue
// (predictedlatency/requestcontrol_hooks.go:73-86), ResponseComplete (:219) and RequestExpired (plugin.go:190-196) remove it,
// RemovePod empties the recycled id's queue, and the latency scorer reads getEndpointMinTPOTSLO / getEndpointRunningRequestCount
// from the engine.  Checked against the same host layer fed through PredictedLatencyProducer::State by the queue oracle
// (tests/cpp/running_oracle.c): picks, scores and tie counts equal, and every queue's view equal to the oracle's.
// Linked against the oracle-backed stand-in of the C ABI on the CPU, and against libeppscore.so on the GPU.
#include <cstdio>
#include <map>
#include <string>
#include <vector>

#include "../../gateway-api-inference-extension_b200/host/epp_scheduler.hpp"

extern "C" {
void* orc_running_new(int32_t n_ep);
void orc_running_add(void* h, int32_t R, const int32_t* ep, const uint64_t* key, const double* tpot, uint8_t* added);
void orc_running_remove(void* h, int32_t R, const int32_t* ep, const uint64_t* key, uint8_t* removed);
void orc_running_remove_endpoint(void* h, int32_t ep);
void orc_running_get(void* h, int32_t M, double* min_out, int32_t* count_out);
}

using namespace epp;

static int g_fail = 0;
#define CHECK(cond)                                               \
  do {                                                            \
    if (!(cond)) {                                                \
      std::printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); \
      g_fail++;                                                   \
    }                                                             \
  } while (0)

constexpr int kMax = 8;

static Endpoint Pod(const std::string& name) {
  Metrics m;
  m.WaitingQueueSize = 100;   // TTFT = 100 against an SLO of 1000: always valid
  m.RunningRequestsSize = 20; // TPOT = 20: valid against 30 unless a running request's tighter SLO limits the endpoint
  m.KVCacheUsagePercent = 0.5;
  return NewEndpoint(name, m, "default");
}
static std::string Name(const Scheduler::BatchItem& it) {
  return it.result.ProfileResults.at("default").TargetEndpoints[0].Endpoint_->GetMetadata()->NamespacedName_.Name;
}
static InferenceRequest Req(const std::string& id, const char* tpot) {
  InferenceRequest q{id, "m", "a prompt of several words " + id, ""};
  q.Headers["x-slo-ttft-ms"] = "1000";
  if (tpot) q.Headers["x-slo-tpot-ms"] = tpot;
  return q;
}

static SchedulerConfig Config(bool track, std::shared_ptr<PredictedLatencyProducer>* prod_out) {
  SchedulerConfig c;
  auto prod = std::make_shared<PredictedLatencyProducer>();
  prod->StreamingMode = true;
  prod->TTFTCoeffs["num_request_waiting"] = 1.0;
  prod->TPOTCoeffs["num_request_running"] = 1.0;
  prod->TrackRunningRequests = track;
  c.Profile.WithScorers({NewWeightedScorer(std::make_shared<LatencyScorer>(), 1),
                         NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1)})
      .WithPicker(MaxScorePicker{})
      .WithPredictedLatencyProducer(prod);
  c.Prefix.MaxPrefixBlocksToMatch = 0;
  c.MaxEndpoints = kMax;
  c.PrefixCapacity = 256;
  *prod_out = prod;
  return c;
}

int main() {
  try {
    std::shared_ptr<PredictedLatencyProducer> pa, pb;
    Scheduler a(Config(true, &pa));   // the engine's queues
    Scheduler b(Config(false, &pb));  // State, fed by the oracle
    void* q = orc_running_new(kMax);
    std::map<std::string, uint64_t> okey;  // the oracle's own exact keys
    auto key = [&](const std::string& id) { return okey.emplace(id, okey.size() + 1).first->second; };
    std::vector<Endpoint> pods = {Pod("podA"), Pod("podB"), Pod("podC"), Pod("podD")};
    auto feed_b = [&](const std::vector<Endpoint>& list) {  // State from the oracle's view, by name
      std::vector<double> mn(kMax);
      std::vector<int32_t> cnt(kMax);
      orc_running_get(q, kMax, mn.data(), cnt.data());
      pb->State.clear();
      for (auto& e : list) {
        const std::string n = e.GetMetadata()->NamespacedName_.String();
        const int id = a.ServerId(n);
        if (id >= 0) pb->State[n] = {mn[(size_t)id], cnt[(size_t)id]};
      }
    };
    auto same_views = [&](const std::vector<Endpoint>& list) {
      std::vector<double> mn(kMax);
      std::vector<int32_t> cnt(kMax);
      orc_running_get(q, kMax, mn.data(), cnt.data());
      bool ok = true;
      for (auto& e : list) {
        const std::string n = e.GetMetadata()->NamespacedName_.String();
        const auto v = a.RunningRequests(n);
        const int id = a.ServerId(n);
        ok = ok && v.first == mn[(size_t)id] && v.second == cnt[(size_t)id];
      }
      return ok;
    };

    // 1. a tight running request (tpot 15) makes podA's TPOT limit 15 < the predicted 20: the next request moves away
    auto r0 = a.ScheduleBatch({Req("tight", "15")}, pods);
    CHECK(Name(r0[0]) == "podA");
    a.PreRequest(r0);
    CHECK(a.RunningRequests("default/podA") == std::make_pair(15.0, 1));
    auto r1 = a.ScheduleBatch({Req("next", "30")}, pods);
    CHECK(Name(r1[0]) != "podA");
    // a request without x-slo-tpot-ms is added with tpot 0: its endpoint's minimum becomes 0, which turns tightening off
    const std::vector<Endpoint> only_a = {pods[0]};  // (the layer keeps the list until PreRequest)
    auto r2 = a.ScheduleBatch({Req("loose", nullptr)}, only_a);
    a.PreRequest(r2);
    CHECK(a.RunningRequests("default/podA") == std::make_pair(0.0, 2));
    // the same id again on the same endpoint is refused (the first tpot stays); an empty id is not tracked
    auto r3 = a.ScheduleBatch({Req("tight", "5"), Req("", "5")}, only_a);
    a.PreRequest(r3);
    CHECK(a.RunningRequests("default/podA") == std::make_pair(0.0, 2));
    CHECK(a.TrackedRequestIds() == 2);
    a.ResponseComplete(Req("tight", "15"), r0[0].result);
    a.RequestExpired(Req("loose", nullptr), r2[0].result);
    CHECK(a.RunningRequests("default/podA") == std::make_pair(0.0, 0) && a.TrackedRequestIds() == 0);

    // 2. batches against the State-fed layer: the same picks, scores and tie counts; every view equal to the oracle's
    const char* tp[] = {"15", "30", nullptr, "22", "50", "18"};
    std::vector<std::pair<InferenceRequest, SchedulingResult>> live;
    int n = 0, moved = 0;
    for (int k = 0; k < 12; k++) {
      std::vector<InferenceRequest> batch;
      for (int i = 0; i < 5; i++, n++) batch.push_back(Req(n % 7 == 6 ? std::string() : "r" + std::to_string(n), tp[n % 6]));
      if (k == 6) {  // podB leaves with requests still running; podE takes its id and starts empty
        const int idB = a.ServerId("default/podB");
        a.RemovePod("default/podB");
        b.RemovePod("default/podB");
        orc_running_remove_endpoint(q, idB);
        pods[1] = Pod("podE");
      }
      feed_b(pods);
      auto ra = a.ScheduleBatch(batch, pods);
      auto rb = b.ScheduleBatch(batch, pods);
      for (size_t i = 0; i < batch.size(); i++) {
        const auto& ta = ra[i].result.ProfileResults.at("default").TargetEndpoints[0];
        const auto& tb = rb[i].result.ProfileResults.at("default").TargetEndpoints[0];
        CHECK(Name(ra[i]) == Name(rb[i]) && ta.Score == tb.Score && ta.TieCount == tb.TieCount);
        moved += Name(ra[i]) != "podA";
      }
      a.PreRequest(ra);
      for (size_t i = 0; i < batch.size(); i++) {
        if (batch[i].RequestId.empty()) continue;
        const int32_t id = a.ServerId("default/" + Name(ra[i]));
        const uint64_t kk = key(batch[i].RequestId);
        const double t = tp[(n - 5 + (int)i) % 6] ? std::stod(tp[(n - 5 + (int)i) % 6]) : 0.0;
        orc_running_add(q, 1, &id, &kk, &t, nullptr);
        live.emplace_back(batch[i], ra[i].result);
      }
      if (k == 6) CHECK(a.RunningRequests("default/podE").second <= 5);  // the recycled id: only this batch's requests
      while (live.size() > 12) {  // the oldest finish: end of stream, every third one by TTL expiry
        auto& [req, res] = live.front();
        const std::string nm = res.ProfileResults.at("default").TargetEndpoints[0].Endpoint_->GetMetadata()->NamespacedName_.String();
        const int32_t id = a.ServerId(nm);
        if (id >= 0) {  // a server that has left: nothing to remove, on either side
          const uint64_t kk = key(req.RequestId);
          orc_running_remove(q, 1, &id, &kk, nullptr);
        }
        if (live.size() % 3 == 0) a.RequestExpired(req, res);
        else a.ResponseComplete(req, res);
        live.erase(live.begin());
      }
      CHECK(same_views(pods));
    }
    CHECK(moved > 0);
  } catch (const std::exception& ex) {
    std::printf("FAIL exception: %s\n", ex.what());
    return 1;
  }
  if (g_fail) {
    std::printf("host running: %d checks failed\n", g_fail);
    return 1;
  }
  std::printf("host running: all checks passed\n");
  return 0;
}
