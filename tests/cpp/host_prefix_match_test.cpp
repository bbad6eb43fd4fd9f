// host_prefix_match_test.cpp — the host layer's PrefixCacheMatchInfo (SchedulerConfig::PrefixMatchInfo) and PreRequest's
// prefix-indexer histograms, against a mirror of the prefix index kept with the oracle (the same hashPrompt, the same Adds in
// PreRequest's order).  Runs on the oracle-backed stand-in of the C ABI (tests/test_host_prefix_match_cpu.py) and on the engine
// (tests/test_gpu_prefix_match.py).  Checks, printing one line per check:
//   - every TargetEndpoints entry's {matchBlocks, totalBlocks, blockSize} on single-profile results, top-k lists of 3 and 12,
//     and decode / prefill results (every entry of both profiles);
//   - the histograms' buckets, count and sums against a hand restatement of RecordPrefixCacheMatch, with ratios of exactly 0.1
//     and 1.0 and a total of 0, and with autotuned block sizes that differ between endpoints[0] and the target;
//   - the option off: nothing filled, nothing recorded, no eppscore_prefix_match call (stand-in); the small-batch host route: empty.
// Built against a library without eppscore_prefix_match, the option is refused when the Scheduler is built.
#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

#include "../../gateway-api-inference-extension_b200/host/epp_scheduler.hpp"
#include "../../oracle/oracle.h"

extern "C" int64_t oracle_backed_prefix_match_calls __attribute__((weak));

using namespace epp;

static int g_fail = 0;
#define CHECK(cond, what)               \
  do {                                  \
    if (!(cond)) {                      \
      std::printf("FAIL %s\n", what);   \
      g_fail++;                         \
    }                                   \
  } while (0)

static const int kMaxBlocks = 256;

// RecordPrefixCacheMatch (metrics.go:830-841) restated by hand: per-bucket counts (+Inf last), count, sum
struct Hand {
  std::vector<double> bounds;
  std::vector<uint64_t> counts;
  uint64_t count = 0;
  double sum = 0;
  explicit Hand(std::vector<double> b) : bounds(b), counts(b.size() + 1, 0) {}
  void observe(double v) {
    size_t i = 0;
    while (i < bounds.size() && !(v <= bounds[i])) i++;
    counts[i]++;
    count++;
    sum += v;
  }
  template <size_t N>
  bool same(const Histogram<N>& h) const {
    return std::vector<double>(h.UpperBounds.begin(), h.UpperBounds.end()) == bounds &&
           std::vector<uint64_t>(h.Counts.begin(), h.Counts.end()) == counts && h.Count == count && h.Sum == sum;
  }
};
struct HandMetrics {
  Hand ratio{{0.0, 0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 1.0}};
  Hand bytes{{0, 16, 32, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536}};
  void record(int matched, int total) {
    bytes.observe((double)matched);
    if (total > 0) ratio.observe((double)matched / (double)total);
  }
  bool same(const PrefixIndexerHistograms& m) const { return ratio.same(m.HitRatio) && bytes.same(m.HitBytes); }
};

// The prefix index as the oracle keeps it, fed the Adds PreRequest makes.
struct Mirror {
  orc_index* idx = orc_index_new(31250);
  ~Mirror() { orc_index_free(idx); }
  static std::vector<uint64_t> hashes(const InferenceRequest& q, int block_tokens) {
    std::vector<uint64_t> h(kMaxBlocks);
    const uint64_t seed = orc_model_seed(q.TargetModel.data(), q.TargetModel.size(), q.CacheSalt.data(), q.CacheSalt.size());
    const int n = orc_hash_prompt(reinterpret_cast<const uint8_t*>(q.Prompt.data()), (int64_t)q.Prompt.size(), seed, block_tokens * 4,
                                  kMaxBlocks, h.data(), kMaxBlocks);
    h.resize((size_t)(n < 0 ? 0 : n));
    return h;
  }
  int match(const std::vector<uint64_t>& h, int id) const {
    std::vector<uint16_t> m(1024);
    orc_match_longest_prefix(idx, h.data(), (int32_t)h.size(), 1024, m.data());
    return m[(size_t)id];
  }
  void add(const std::vector<uint64_t>& h, int id) { orc_index_add(idx, h.data(), (int32_t)h.size(), id, 0); }
};

static Metrics Met(int queue, int block_size = 0) {
  Metrics m;
  m.WaitingQueueSize = queue;
  m.KVCacheUsagePercent = 0.1 * (queue % 7);
  m.CacheBlockSize = block_size;
  return m;
}

static std::vector<InferenceRequest> Requests(int R, int round, int n_sys = 3) {
  static const char* sys[] = {"You are a helpful assistant that answers questions about the weather in great detail. ",
                              "System: translate the following text into French, keeping the formatting as it is. ",
                              "Summarise the document below in three bullet points, citing the section numbers. "};
  std::vector<InferenceRequest> out;
  for (int r = 0; r < R; r++) {
    InferenceRequest q;
    q.RequestId = "req-" + std::to_string(round) + "-" + std::to_string(r);
    q.TargetModel = "m";
    std::string p;
    for (int i = 0; i < 6; i++) p += sys[(r + round) % n_sys];
    for (int i = 0; i < (r % 5); i++) p += "user turn " + std::to_string(r * 31 + round) + " with some more words to hash. ";
    q.Prompt = p;
    out.push_back(q);
  }
  return out;
}

// every entry of every profile against the mirror; returns the number of entries checked
static int CheckEntries(Scheduler& s, const std::vector<InferenceRequest>& reqs, const std::vector<Scheduler::BatchItem>& res,
                        const Mirror& mir, int block_tokens, const char* what) {
  int n = 0;
  for (size_t r = 0; r < res.size(); r++) {
    if (!res[r].error.empty()) continue;
    const auto h = Mirror::hashes(reqs[r], block_tokens);
    for (const auto& kv : res[r].result.ProfileResults)
      for (const ScoredEndpoint& t : kv.second.TargetEndpoints) {
        const int id = s.ServerId(t.Endpoint_->GetMetadata()->NamespacedName_.String());
        const bool ok = t.PrefixMatch && t.PrefixMatch->MatchBlocks == mir.match(h, id) && t.PrefixMatch->TotalBlocks == (int)h.size() &&
                        t.PrefixMatch->BlockSizeTokens == block_tokens;
        if (!ok)
          std::printf("  %s r=%zu %s ep=%d got=%d/%d want=%d/%zu\n", what, r, kv.first.c_str(), id, t.PrefixMatch ? t.PrefixMatch->MatchBlocks : -1,
                      t.PrefixMatch ? t.PrefixMatch->TotalBlocks : -1, mir.match(h, id), h.size());
        CHECK(ok, what);
        n++;
      }
  }
  return n;
}

// PreRequest's Adds on the mirror (primary target, then the "prefill" target) and its metrics on the hand restatement
static void Commit(Scheduler& s, const std::vector<InferenceRequest>& reqs, const std::vector<Scheduler::BatchItem>& res, Mirror& mir,
                   HandMetrics& hand, const PrefixConfig& pc, int block_tokens) {
  for (size_t r = 0; r < res.size(); r++) {  // every match of the batch was read before its Adds
    if (!res[r].error.empty()) continue;
    const auto& sr = res[r].result;
    const auto h = Mirror::hashes(reqs[r], block_tokens);
    const ScoredEndpoint& t = sr.ProfileResults.at(sr.PrimaryProfileName).TargetEndpoints[0];
    const int id = s.ServerId(t.Endpoint_->GetMetadata()->NamespacedName_.String());
    int bs = pc.BlockSizeTokens;
    if (pc.AutoTune && t.Endpoint_->GetMetrics()->CacheBlockSize > 0) bs = t.Endpoint_->GetMetrics()->CacheBlockSize;
    hand.record(mir.match(h, id) * bs * 4, (int)h.size() * bs * 4);
  }
  for (size_t r = 0; r < res.size(); r++) {
    if (!res[r].error.empty()) continue;
    const auto& sr = res[r].result;
    const auto h = Mirror::hashes(reqs[r], block_tokens);
    const ScoredEndpoint& t = sr.ProfileResults.at(sr.PrimaryProfileName).TargetEndpoints[0];
    mir.add(h, s.ServerId(t.Endpoint_->GetMetadata()->NamespacedName_.String()));
    auto pf = sr.ProfileResults.find("prefill");
    if (pf != sr.ProfileResults.end() && !pf->second.TargetEndpoints.empty())
      mir.add(h, s.ServerId(pf->second.TargetEndpoints[0].Endpoint_->GetMetadata()->NamespacedName_.String()));
  }
  s.PreRequest(res);
}

static SchedulerConfig Single(int k) {
  SchedulerConfig c;
  c.Profile.WithScorers({NewWeightedScorer(std::make_shared<PrefixCacheScorer>(), 3), NewWeightedScorer(std::make_shared<QueueScorer>(), 1)});
  MaxScorePicker p;
  p.MaxNumOfEndpoints = k;
  c.Profile.WithPicker(p);
  c.MaxEndpoints = 64;
  c.CpuBatchThreshold = 0;
  c.PrefixMatchInfo = true;
  return c;
}

static std::vector<Endpoint> Pool(int n, int first_block_size = 0) {
  std::vector<Endpoint> eps;
  for (int i = 0; i < n; i++) eps.push_back(NewEndpoint("ep" + std::to_string(i), Met((i * 5) % 9, i == 0 ? first_block_size : 0)));
  return eps;
}

static void SingleProfile(int k) {
  Scheduler s(Single(k));
  const auto eps = Pool(16);
  Mirror mir;
  HandMetrics hand;
  int n = 0;
  for (int round = 0; round < 4; round++) {
    const auto reqs = Requests(24, round);
    const auto res = s.ScheduleBatch(reqs, eps);
    n += CheckEntries(s, reqs, res, mir, 16, "single entries");
    Commit(s, reqs, res, mir, hand, Single(k).Prefix, 16);
  }
  CHECK(hand.same(s.PrefixIndexerMetrics()), "single metrics");
  std::printf("single k=%d entries %d observations %llu\n", k, n, (unsigned long long)s.PrefixIndexerMetrics().HitBytes.Count);
}

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

static void DecodePrefill() {
  SchedulerConfig c;
  c.MaxEndpoints = 64;
  c.PrefixMatchInfo = true;
  c.Handler = std::make_shared<PdHandler>();
  for (const char* role : {"decode", "prefill"}) {
    SchedulerProfile p;
    p.WithScorers({NewWeightedScorer(std::make_shared<PrefixCacheScorer>(), 3), NewWeightedScorer(std::make_shared<QueueScorer>(), 1)});
    const std::string rl = role;
    p.WithEndpointSubset([rl](const Endpoint& e) { return e.GetMetadata()->Labels.at("role") == rl; });
    MaxScorePicker pk;
    pk.MaxNumOfEndpoints = rl == "decode" ? 3 : 1;
    p.WithPicker(pk);
    c.Profiles.emplace_back(rl, p);
  }
  Scheduler s(c);
  auto eps = Pool(12);
  for (size_t i = 0; i < eps.size(); i++) eps[i].Metadata.Labels["role"] = i % 2 ? "prefill" : "decode";
  Mirror mir;
  HandMetrics hand;
  int n = 0;
  for (int round = 0; round < 4; round++) {
    const auto reqs = Requests(20, round);
    const auto res = s.ScheduleBatch(reqs, eps);
    n += CheckEntries(s, reqs, res, mir, 16, "pd entries");
    Commit(s, reqs, res, mir, hand, c.Prefix, 16);
  }
  CHECK(hand.same(s.PrefixIndexerMetrics()), "pd metrics");
  std::printf("pd entries %d observations %llu\n", n, (unsigned long long)s.PrefixIndexerMetrics().HitBytes.Count);
}

// one endpoint: a 10-block prompt, then the same first block with 9 new ones (ratio 0.1), the whole prompt again (1.0), a prompt
// shorter than a block (total 0: bytes observed, no ratio)
static void EdgeRatios() {
  Scheduler s(Single(1));
  const auto eps = Pool(1);
  Mirror mir;
  HandMetrics hand;
  std::string p;
  for (int i = 0; i < 640; i++) p += (char)('a' + (i * 7) % 26);
  std::string q = p.substr(0, 64);
  for (int i = 0; i < 576; i++) q += (char)('a' + (i * 11) % 23);
  for (const std::string& prompt : {p, q, p, std::string("hi")}) {
    InferenceRequest r;
    r.RequestId = "x";
    r.TargetModel = "m";
    r.Prompt = prompt;
    const auto res = s.ScheduleBatch({r}, eps);
    CheckEntries(s, {r}, res, mir, 16, "edge entries");
    Commit(s, {r}, res, mir, hand, Single(1).Prefix, 16);
  }
  const auto& m = s.PrefixIndexerMetrics();
  CHECK(hand.same(m), "edge metrics");
  const std::vector<uint64_t> ratio{1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 1, 0};  // 0/10, 1/10 (exactly 0.1), 10/10; the 0-total prompt none
  CHECK(std::vector<uint64_t>(m.HitRatio.Counts.begin(), m.HitRatio.Counts.end()) == ratio && m.HitRatio.Count == 3 && m.HitRatio.Sum == 0.0 + 0.1 + 1.0, "edge ratio buckets");
  const std::vector<uint64_t> bytes{2, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0};  // 0 twice, 64 (bound 64), 640 (bound 1024)
  CHECK(std::vector<uint64_t>(m.HitBytes.Counts.begin(), m.HitBytes.Counts.end()) == bytes && m.HitBytes.Count == 4 && m.HitBytes.Sum == 0.0 + 64.0 + 640.0 + 0.0, "edge byte buckets");
  std::printf("edges checked\n");
}

// endpoints[0] autotunes the hash block size to 8 tokens; the target (the only candidate left by a filter) reports 32: the info
// carries 8, the metric multiplies by 32 * 4
struct Only : Filter {
  int keep;
  explicit Only(int k) : keep(k) {}
  std::vector<int> Filter_(const InferenceRequest&, const std::vector<Endpoint>&, const std::vector<int>&) override { return {keep}; }
};
static void AutotunedBlockSizes() {
  SchedulerConfig c = Single(1);
  c.Profile.WithFilters({std::make_shared<Only>(1)});
  Scheduler s(c);
  std::vector<Endpoint> eps = {NewEndpoint("a", Met(0, 8)), NewEndpoint("b", Met(1, 32))};
  Mirror mir;
  HandMetrics hand;
  for (int round = 0; round < 3; round++) {
    const auto reqs = Requests(6, round, 1);
    const auto res = s.ScheduleBatch(reqs, eps);
    CheckEntries(s, reqs, res, mir, 8, "autotune entries");
    Commit(s, reqs, res, mir, hand, c.Prefix, 8);
  }
  CHECK(hand.same(s.PrefixIndexerMetrics()), "autotune metrics");
  CHECK(s.PrefixIndexerMetrics().HitBytes.Sum > 0 && std::fmod(s.PrefixIndexerMetrics().HitBytes.Sum, 128.0) == 0.0, "autotune target block size");
  std::printf("autotune checked\n");
}

static void OptionOffAndHostRoute() {
  const int64_t calls0 = &oracle_backed_prefix_match_calls ? oracle_backed_prefix_match_calls : 0;
  SchedulerConfig c = Single(3);
  c.PrefixMatchInfo = false;
  Scheduler s(c);
  const auto eps = Pool(8);
  for (int round = 0; round < 2; round++) {
    const auto reqs = Requests(10, round);
    const auto res = s.ScheduleBatch(reqs, eps);
    bool none = true;
    for (const auto& it : res)
      for (const auto& kv : it.result.ProfileResults)
        for (const auto& t : kv.second.TargetEndpoints) none = none && !t.PrefixMatch;
    CHECK(none, "option off: nothing filled");
    s.PreRequest(res);
  }
  CHECK(s.PrefixIndexerMetrics().HitBytes.Count == 0 && s.PrefixIndexerMetrics().HitRatio.Count == 0, "option off: nothing recorded");
  if (&oracle_backed_prefix_match_calls) CHECK(oracle_backed_prefix_match_calls == calls0, "option off: no engine call");
  // the small-batch host route (request-independent profile, no prefix producer) hashes nothing: the info stays empty
  SchedulerConfig h;
  h.Profile.WithScorers({NewWeightedScorer(std::make_shared<QueueScorer>(), 1)});
  h.PrefixMatchInfo = true;
  Scheduler hs(h);
  const auto res = hs.ScheduleBatch(Requests(2, 0), eps);
  CHECK(hs.CpuRoutedRequests() == 2, "host route taken");
  for (const auto& it : res) CHECK(!it.result.ProfileResults.begin()->second.TargetEndpoints[0].PrefixMatch, "host route: nothing filled");
  hs.PreRequest(res);
  CHECK(hs.PrefixIndexerMetrics().HitBytes.Count == 0, "host route: nothing recorded");
  std::printf("option off checked\n");
}

int main() {
  if (!EngineHasPrefixMatch()) {
    try {
      Scheduler s(Single(1));
      std::printf("FAIL the option was accepted without eppscore_prefix_match\n");
    } catch (const SchedulingError& e) {
      std::printf("refused %s\n", e.what());
    }
    SchedulerConfig c = Single(1);
    c.PrefixMatchInfo = false;
    Scheduler s(c);  // without the option the library serves as before
    std::printf("done\n");
    return 0;
  }
  SingleProfile(1);
  SingleProfile(3);
  SingleProfile(12);
  DecodePrefill();
  EdgeRatios();
  AutotunedBlockSizes();
  OptionOffAndHostRoute();
  std::printf(g_fail ? "FAILED %d\n" : "done\n", g_fail);
  return g_fail ? 1 : 0;
}
