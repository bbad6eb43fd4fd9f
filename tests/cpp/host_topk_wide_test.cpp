// host_topk_wide_test.cpp — the host layer's Scheduler with maxNumOfEndpoints > 8.  Prints, per case, the route the
// Scheduler took (wide: eppscore_schedule_batch_topk_wide; map: the score map sorted on the host; refused: the Scheduler
// was not built) and every request's list as "index:score" pairs, so tests/test_host_topk_wide_cpu.py can compare the
// output of a build with the wide entry point against one without it.
#include <cstdio>
#include <string>
#include <vector>

#include "../../gateway-api-inference-extension_b200/host/epp_scheduler.hpp"

extern "C" int64_t oracle_backed_topk_wide_calls __attribute__((weak));

using namespace epp;

static void run(const char* name, int mode, int tie_mode, int k, int n_req) {
  SchedulerConfig c;
  c.CpuBatchThreshold = 0;
  MaxScorePicker pk = mode == 1 ? MaxScorePicker(WeightedRandomPicker{}) : (mode == 2 ? MaxScorePicker(RandomPicker{}) : MaxScorePicker{});
  pk.MaxNumOfEndpoints = k;
  c.Profile.WithScorers({NewWeightedScorer(std::make_shared<KVCacheUtilizationScorer>(), 1)}).WithPicker(pk);
  c.MaxEndpoints = 64;
  c.TieMode = tie_mode;
  c.TieSeed = 4242;
  std::vector<Endpoint> eps;
  for (int i = 0; i < 50; i++) {  // utilisation on a coarse grid: tie classes of several endpoints; a few score 0
    Metrics m;
    m.KVCacheUsagePercent = i % 7 == 0 ? 1.0 : 0.05 * (i % 11);
    eps.push_back(NewEndpoint("pod" + std::to_string(i), m));
  }
  const int64_t before = &oracle_backed_topk_wide_calls ? oracle_backed_topk_wide_calls : 0;
  std::vector<Scheduler::BatchItem> res;
  try {
    Scheduler s(c);
    std::vector<InferenceRequest> reqs(n_req, InferenceRequest{"r", "m", "", ""});
    res = s.ScheduleBatch(reqs, eps);
  } catch (const SchedulingError& ex) {
    std::printf("case %s route=refused\n", name);
    return;
  }
  const bool wide = &oracle_backed_topk_wide_calls && oracle_backed_topk_wide_calls > before;
  std::printf("case %s route=%s\n", name, wide ? "wide" : "map");
  for (auto& r : res) {
    if (!r.error.empty()) {
      std::printf("error\n");
      continue;
    }
    for (const auto& se : r.result.ProfileResults.at("default").TargetEndpoints) std::printf("%d:%.17g ", se.Index, se.Score);
    std::printf("\n");
  }
}

int main() {
  for (int k : {12, 40}) {
    run(("weighted_random_k" + std::to_string(k)).c_str(), 1, EPPSCORE_TIE_LOWEST_INDEX, k, 2000);
    run(("random_k" + std::to_string(k)).c_str(), 2, EPPSCORE_TIE_LOWEST_INDEX, k, 2000);
  }
  run("max_score_lowest_index_k12", 0, EPPSCORE_TIE_LOWEST_INDEX, 12, 4);
  run("max_score_lowest_index_k100", 0, EPPSCORE_TIE_LOWEST_INDEX, 100, 4);
  run("max_score_seeded_random_k12", 0, EPPSCORE_TIE_SEEDED_RANDOM, 12, 4);
  std::printf("done\n");
  return 0;
}
