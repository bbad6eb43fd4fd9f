// host_lora_width_test.cpp — the host layer's LoRA dictionary on fleets with more adapter names than the engine holds.
// The Scheduler gives engine rows only to the batch's own targets that some endpoint carries, and runs a batch with more such
// targets than MaxAdapters (rounded up to 64) as contiguous pieces.  Fleets of 64, 65, 200 and 1000 adapter names, MaxAdapters
// 64 and 100, batches with fewer, as many and more distinct targets than that capacity, targets nobody carries and adapters
// that are only waiting.  Every result is checked two ways:
//   - against a by-name restatement of lora_affinity.go:84-99 (no ids anywhere): pick, score, tie count and lists, as far as
//     the picker's order is determined by the scores;
//   - against a Scheduler whose MaxAdapters covers the whole fleet, so it never splits: every field, bit for bit (this is what
//     pins the seeded tie-breaks and the stochastic pickers to the request's index in the whole batch).
// Built against tests/cpp/oracle_backed_*.cpp on the CPU and against libeppscore.so on an H100.  Prints one line per scenario
// and "host lora width: all checks passed".
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../../gateway-api-inference-extension_b200/host/epp_scheduler.hpp"

using namespace epp;

static int g_fail = 0;
static std::string g_where;
#define CHECK(cond)                                                              \
  do {                                                                           \
    if (!(cond)) {                                                               \
      std::printf("FAIL %s:%d %s  [%s]\n", __FILE__, __LINE__, #cond, g_where.c_str()); \
      g_fail++;                                                                  \
    }                                                                            \
  } while (0)

static const int kEndpoints = 48;

static std::string Adapter(int a) { return "lora-" + std::to_string(a); }

// nA adapter names over kEndpoints pods.  Adapter a with a % 7 == 3 is only ever waiting (on two pods); every other one is
// active on pod a % M and waiting on pod (11a + 3) % M.  Pods with i % 6 == 0 have room for more adapters (class 0.8 for any
// target they do not run); the others are full, so active / waiting / neither decide.
static std::vector<Endpoint> Fleet(int nA) {
  std::vector<Metrics> ms((size_t)kEndpoints);
  for (int a = 0; a < nA; a++) {
    if (a % 7 == 3) {
      ms[(size_t)(a % kEndpoints)].WaitingModels[Adapter(a)] = 0;
      ms[(size_t)((5 * a + 1) % kEndpoints)].WaitingModels[Adapter(a)] = 0;
    } else {
      ms[(size_t)(a % kEndpoints)].ActiveModels[Adapter(a)] = 0;
      ms[(size_t)((11 * a + 3) % kEndpoints)].WaitingModels[Adapter(a)] = 0;
    }
  }
  std::vector<Endpoint> eps;
  for (int i = 0; i < kEndpoints; i++) {
    Metrics& m = ms[(size_t)i];
    m.MaxActiveModels = i % 6 == 0 ? 1 << 20 : 0;
    m.KVCacheUsagePercent = 0.01 * (i % 13);
    Endpoint e = NewEndpoint("pod" + std::to_string(i), m);
    e.Metadata.Labels["role"] = i % 2 ? "decode" : "prefill";
    eps.push_back(e);
  }
  return eps;
}

// R requests over D distinct carried targets (a seeded choice of the fleet's names) and 5 names nobody carries, in a seeded
// order; every prompt is different.
static std::vector<InferenceRequest> Batch(int nA, int D, int R, unsigned seed) {
  std::mt19937 rng(seed);
  std::vector<int> names((size_t)nA);
  for (int a = 0; a < nA; a++) names[(size_t)a] = a;
  std::shuffle(names.begin(), names.end(), rng);
  std::vector<std::string> pool;
  for (int j = 0; j < D; j++) pool.push_back(Adapter(names[(size_t)j]));
  for (int j = 0; j < 5; j++) pool.push_back("absent-" + std::to_string(j));
  std::vector<std::string> t;
  for (int r = 0; r < R; r++) t.push_back(pool[(size_t)r % pool.size()]);
  std::shuffle(t.begin(), t.end(), rng);
  std::vector<InferenceRequest> reqs;
  for (int r = 0; r < R; r++) {
    std::string prompt = "request " + std::to_string(seed) + "/" + std::to_string(r) + " ";
    prompt.resize(256, (char)('a' + r % 26));
    reqs.push_back(InferenceRequest{"q" + std::to_string(r), t[(size_t)r], prompt, ""});
  }
  return reqs;
}

// lora_affinity.go:84-99 by name
static double LoraByName(const Endpoint& e, const std::string& target) {
  const Metrics& m = *e.GetMetrics();
  if (m.ActiveModels.count(target)) return 1.0;
  if ((int)(m.ActiveModels.size() + m.WaitingModels.size()) < m.MaxActiveModels) return 0.8;
  if (m.WaitingModels.count(target)) return 0.6;
  return 0.0;
}

// candidates of `keep` by descending by-name score, ties in ascending index
static std::vector<std::pair<int, double>> Order(const std::vector<Endpoint>& eps, const std::string& target, bool (*keep)(const Endpoint&)) {
  std::vector<std::pair<int, double>> v;
  for (int i = 0; i < (int)eps.size(); i++)
    if (!keep || keep(eps[(size_t)i])) v.emplace_back(i, LoraByName(eps[(size_t)i], target));
  std::stable_sort(v.begin(), v.end(), [](const auto& a, const auto& b) { return a.second > b.second; });
  return v;
}

static bool SameBits(double a, double b) { return std::memcmp(&a, &b, sizeof a) == 0; }

static void CheckSame(const std::vector<Scheduler::BatchItem>& got, const std::vector<Scheduler::BatchItem>& want) {
  CHECK(got.size() == want.size());
  for (size_t r = 0; r < got.size() && r < want.size(); r++) {
    CHECK(got[r].error == want[r].error);
    CHECK(got[r].result.PrimaryProfileName == want[r].result.PrimaryProfileName);
    CHECK(got[r].result.ProfileResults.size() == want[r].result.ProfileResults.size());
    for (const auto& kv : want[r].result.ProfileResults) {
      auto it = got[r].result.ProfileResults.find(kv.first);
      if (it == got[r].result.ProfileResults.end()) {
        CHECK(false);
        continue;
      }
      const auto &g = it->second.TargetEndpoints, &w = kv.second.TargetEndpoints;
      CHECK(g.size() == w.size());
      for (size_t i = 0; i < g.size() && i < w.size(); i++) {
        CHECK(g[i].Index == w[i].Index);
        CHECK(SameBits(g[i].Score, w[i].Score));
        CHECK(g[i].TieCount == w[i].TieCount);
      }
    }
  }
}

enum Variant { kLowest, kSeeded, kWeighted, kTop3, kTop12, kTwoProfiles };
static const char* kVariantName[] = {"max_score_lowest", "max_score_seeded", "weighted_random", "top3", "top12", "two_profiles"};

static bool IsDecode(const Endpoint& e) { return e.GetMetadata()->Labels.at("role") == "decode"; }
static bool IsPrefill(const Endpoint& e) { return e.GetMetadata()->Labels.at("role") == "prefill"; }

// the decode profile is primary; the prefill result rides along
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

static SchedulerProfile LoraOnly(int mode, int k) {
  MaxScorePicker p;
  p.Mode = mode;
  p.MaxNumOfEndpoints = k;
  SchedulerProfile s;
  s.WithScorers({NewWeightedScorer(std::make_shared<LoraAffinityScorer>(), 1)}).WithPicker(p);
  return s;
}

static SchedulerConfig Config(Variant v, int max_adapters, int threshold) {
  SchedulerConfig c;
  c.MaxEndpoints = 64;
  c.MaxAdapters = max_adapters;
  c.CpuBatchThreshold = threshold;
  c.TieSeed = 1234;
  c.PrefixCapacity = 1 << 14;
  c.Prefix.AutoTune = false;
  switch (v) {
    case kLowest: c.Profile = LoraOnly(EPPSCORE_PICK_MAX_SCORE, 1); break;
    case kSeeded: c.Profile = LoraOnly(EPPSCORE_PICK_MAX_SCORE, 1); c.TieMode = EPPSCORE_TIE_SEEDED_RANDOM; break;
    case kWeighted: c.Profile = LoraOnly(EPPSCORE_PICK_WEIGHTED_RANDOM, 1); break;
    case kTop3: c.Profile = LoraOnly(EPPSCORE_PICK_MAX_SCORE, 3); break;
    case kTop12: c.Profile = LoraOnly(EPPSCORE_PICK_MAX_SCORE, 12); break;
    case kTwoProfiles:
      c.Profiles = {{"decode", LoraOnly(EPPSCORE_PICK_MAX_SCORE, 3).WithEndpointSubset(IsDecode)},
                    {"prefill", LoraOnly(EPPSCORE_PICK_WEIGHTED_RANDOM, 1).WithEndpointSubset(IsPrefill)}};
      c.Handler = std::make_shared<PdHandler>();
      break;
  }
  return c;
}

// the by-name expectations of one batch under variant v
static void CheckByName(Variant v, const std::vector<Endpoint>& eps, const std::vector<InferenceRequest>& reqs,
                        const std::vector<Scheduler::BatchItem>& got) {
  for (size_t r = 0; r < reqs.size(); r++) {
    CHECK(got[r].error.empty());
    if (!got[r].error.empty()) continue;
    const std::string& t = reqs[r].TargetModel;
    auto check_list = [&](const std::vector<ScoredEndpoint>& te, bool (*keep)(const Endpoint&), size_t k) {
      const auto want = Order(eps, t, keep);
      CHECK(te.size() == std::min(k, want.size()));
      for (size_t i = 0; i < te.size() && i < want.size(); i++) {
        CHECK(te[i].Index == want[i].first);
        CHECK(te[i].Score == want[i].second);
      }
    };
    auto check_stochastic = [&](const ScoredEndpoint& se, bool (*keep)(const Endpoint&)) {
      CHECK(se.Index >= 0 && se.Index < (int)eps.size() && (!keep || keep(eps[(size_t)se.Index])));
      CHECK(se.Score == LoraByName(eps[(size_t)se.Index], t));
    };
    if (v == kTwoProfiles) {
      check_list(got[r].result.ProfileResults.at("decode").TargetEndpoints, IsDecode, 3);
      check_stochastic(got[r].result.ProfileResults.at("prefill").TargetEndpoints.at(0), IsPrefill);
      continue;
    }
    const auto& te = got[r].result.ProfileResults.at("default").TargetEndpoints;
    const auto order = Order(eps, t, nullptr);
    const double best = order[0].second;
    const int ties = (int)std::count_if(order.begin(), order.end(), [&](const auto& p) { return p.second == best; });
    if (v == kWeighted) {
      check_stochastic(te.at(0), nullptr);
    } else if (v == kSeeded) {
      check_stochastic(te.at(0), nullptr);
      CHECK(te.at(0).Score == best && te.at(0).TieCount == ties);
    } else {
      check_list(te, nullptr, v == kTop3 ? 3 : (v == kTop12 ? 12 : 1));
      CHECK(te.at(0).TieCount == ties);
    }
  }
}

int main() {
  try {
    // 1. every fleet, capacity, target count and picker: the capped Scheduler against the by-name restatement and against an
    //    uncapped one
    for (int nA : {64, 65, 200, 1000}) {
      const std::vector<Endpoint> eps = Fleet(nA);
      for (int max_adapters : {64, 100}) {
        const int cap = (max_adapters + 63) / 64 * 64;
        std::vector<int> Ds;
        for (int D : {cap / 2, cap, 2 * cap + 5})
          if (std::min(D, nA) != (Ds.empty() ? -1 : Ds.back())) Ds.push_back(std::min(D, nA));
        for (int vi = kLowest; vi <= kTwoProfiles; vi++)
          for (int threshold : {0, 8}) {
            const Variant v = (Variant)vi;
            if (threshold == 8 && v != kLowest) continue;  // the small-batch host route serves this profile only
            Scheduler capped(Config(v, max_adapters, threshold)), whole(Config(v, std::max(nA, 64), 0));
            for (int D : Ds)
              for (int R : {6, 157}) {
                g_where = std::string(kVariantName[vi]) + " fleet=" + std::to_string(nA) + " max_adapters=" + std::to_string(max_adapters) +
                          " threshold=" + std::to_string(threshold) + " targets=" + std::to_string(D) + " R=" + std::to_string(R);
                const int before = g_fail;
                const auto reqs = Batch(nA, D, R, (unsigned)(nA * 31 + D * 7 + R + vi));
                const auto got = capped.ScheduleBatch(reqs, eps);
                CheckByName(v, eps, reqs, got);
                CheckSame(got, whole.ScheduleBatch(reqs, eps));
                std::printf("scenario %s %s\n", g_where.c_str(), g_fail == before ? "ok" : "FAILED");
              }
          }
      }
    }

    // 2. PreRequest after a split batch: prefix weight 10 over lora 1, every prompt distinct, so a second batch with the same
    //    prompts must land where the first one committed each request (the whole prompt is cached there and nowhere else)
    for (int nA : {65, 1000}) {
      const std::vector<Endpoint> eps = Fleet(nA);
      SchedulerConfig c = Config(kSeeded, 64, 0);
      c.Profile.WithScorers({NewWeightedScorer(std::make_shared<PrefixCacheScorer>(), 10), NewWeightedScorer(std::make_shared<LoraAffinityScorer>(), 1)});
      SchedulerConfig cw = c;
      cw.MaxAdapters = std::max(nA, 64);
      Scheduler capped(c), whole(cw);
      g_where = "prerequest fleet=" + std::to_string(nA) + " max_adapters=64 targets=" + std::to_string(std::min(nA, 133)) + " R=301";
      const int before = g_fail;
      const auto reqs = Batch(nA, std::min(nA, 133), 301, 99u + (unsigned)nA);
      const auto first = capped.ScheduleBatch(reqs, eps);
      CheckSame(first, whole.ScheduleBatch(reqs, eps));
      CHECK(capped.LastTotalBlocks().size() == reqs.size());
      capped.PreRequest(first);
      whole.PreRequest(first);
      const auto second = capped.ScheduleBatch(reqs, eps);
      CheckSame(second, whole.ScheduleBatch(reqs, eps));
      for (size_t r = 0; r < reqs.size(); r++) {
        const auto& a = first[r].result.ProfileResults.at("default").TargetEndpoints.at(0);
        const auto& b = second[r].result.ProfileResults.at("default").TargetEndpoints.at(0);
        CHECK(b.Index == a.Index);
        CHECK(b.Score == 10.0 + LoraByName(eps[(size_t)a.Index], reqs[r].TargetModel));
        CHECK(b.TieCount == 1);
      }
      std::printf("scenario %s %s\n", g_where.c_str(), g_fail == before ? "ok" : "FAILED");
    }
  } catch (const std::exception& e) {
    std::printf("FAIL exception: %s  [%s]\n", e.what(), g_where.c_str());
    return 2;
  }
  if (g_fail) {
    std::printf("%d check(s) failed\n", g_fail);
    return 1;
  }
  std::printf("host lora width: all checks passed\n");
  return 0;
}
