// epp_types.hpp — the reference's carrier types for this path, restated in C++ (see epp_scheduler.hpp for the map):
// InferenceRequest / Endpoint / ScoredEndpoint / ProfileRunResult / SchedulingResult (interface/scheduling/types.go:44-170),
// Metrics (interface/datalayer/metrics.go:26-42), errcommon.Error as an exception.
#pragma once
#include <cstdint>
#include <map>
#include <optional>
#include <stdexcept>
#include <string>
#include <vector>

namespace epp {

struct NamespacedName {
  std::string Namespace, Name;
  std::string String() const { return Namespace + "/" + Name; }
  bool operator==(const NamespacedName& o) const { return Namespace == o.Namespace && Name == o.Name; }
};

// fwkdl.Metrics — the fields this path reads
struct Metrics {
  std::map<std::string, int> ActiveModels, WaitingModels;
  int MaxActiveModels = 0;
  int RunningRequestsSize = 0;
  int WaitingQueueSize = 0;
  double KVCacheUsagePercent = 0.0;
  int CacheBlockSize = 0;   // tokens; autotune source for the prefix block size (approximateprefix/plugin.go:238-250)
  int CacheNumBlocks = 0;   // autotune source for the per-endpoint LRU capacity (plugin.go:207-216)
};

struct EndpointMetadata {
  NamespacedName NamespacedName_;
  std::map<std::string, std::string> Labels;
};

struct Endpoint {
  EndpointMetadata Metadata;
  Metrics Metrics_;
  // attrconcurrency.InFlightLoad.Tokens (token_load.go:91-95); < 0 here = attribute absent
  int64_t InFlightTokens = -1;
  const EndpointMetadata* GetMetadata() const { return &Metadata; }
  const Metrics* GetMetrics() const { return &Metrics_; }
};
inline Endpoint NewEndpoint(const std::string& name, const Metrics& m, const std::string& ns = "") {
  Endpoint e;
  e.Metadata.NamespacedName_ = NamespacedName{ns, name};
  e.Metrics_ = m;
  return e;
}

struct InferenceRequest {
  std::string RequestId;
  std::string TargetModel;
  std::string Prompt;     // getUserInputBytes() output (hashing.go:106-135): Completions prompt or marshalled messages
  std::string CacheSalt;
  std::map<std::string, std::string> Headers;  // "x-slo-ttft-ms" / "x-slo-tpot-ms" feed the latency path
  // SimpleTokenEstimator inputs (inflightload/token_estimator.go:48-72): the request body's size when known (> 0 wins), and
  // Body.InputTokenCountHint() (>= 0: the exact input token count of token-ID prompts); otherwise len(Prompt) stands in for
  // len(Body.PromptText())
  int64_t RequestSizeBytes = 0;
  int InputTokenCountHint = -1;
};

// len(strings.Fields(s)) (predictedlatency/plugin.go:286): runs of unicode.IsSpace separate fields.  Go decodes
// runes with utf8.DecodeRuneInString (any invalid or short sequence = U+FFFD, width 1); because a lead byte is never
// a continuation byte, a byte belongs to a space rune exactly when it is an ASCII space or lies inside one of the
// UTF-8 encodings of U+0085, U+00A0, U+1680, U+2000..U+200A, U+2028, U+2029, U+202F, U+205F, U+3000 — the same
// byte-pattern rule the device kernel uses (csrc/fields_kernel.cu; fuzzed against the oracle's rune decoder).
inline int CountFields(const std::string& str) {
  const size_t n = str.size();
  const unsigned char* s = reinterpret_cast<const unsigned char*>(str.data());
  int count = 0;
  bool prev_space = true;
  size_t cover = 0;  // bytes [i, cover) still belong to a multi-byte space rune
  for (size_t i = 0; i < n; i++) {
    const unsigned b = s[i];
    bool sp = (b >= 9 && b <= 13) || b == 32 || i < cover;
    if (b == 0xC2 && i + 1 < n && (s[i + 1] == 0x85 || s[i + 1] == 0xA0)) {
      sp = true;
      cover = i + 2;
    } else if (i + 2 < n) {
      const unsigned b1 = s[i + 1], b2 = s[i + 2];
      if ((b == 0xE1 && b1 == 0x9A && b2 == 0x80) ||
          (b == 0xE2 && b1 == 0x80 && ((b2 >= 0x80 && b2 <= 0x8A) || b2 == 0xA8 || b2 == 0xA9 || b2 == 0xAF)) ||
          (b == 0xE2 && b1 == 0x81 && b2 == 0x9F) || (b == 0xE3 && b1 == 0x80 && b2 == 0x80)) {
        sp = true;
        cover = i + 3;
      }
    }
    if (!sp && prev_space) count++;
    prev_space = sp;
  }
  return count;
}

// attrprefix.PrefixCacheMatchInfo (datalayer/attribute/prefix/data_types.go): what PrepareRequestData puts on every endpoint
// (approximateprefix/plugin.go:150-153).  Block counts, and the block length in tokens the prompt was hashed with.  All three
// fit 16 bits: the engine hashes at most EPPSCORE_MAX_BLOCKS = 65535 blocks, and the Scheduler refuses block sizes past 65535
// tokens for the info, so a ScoredEndpoint keeps its size.
struct PrefixCacheMatchInfo {
  uint16_t MatchBlocks = 0;
  uint16_t TotalBlocks = 0;
  uint16_t BlockSizeTokens = 0;
};

struct ScoredEndpoint {
  const Endpoint* Endpoint_ = nullptr;
  double Score = 0.0;
  int Index = -1;  // position in the candidate slice given to Schedule
  int TieCount = 0;  // size of the arg-max set the reference would shuffle over (picker/maxscore/picker.go:91-102)
  // The endpoint's PrefixCacheMatchInfo attribute; set only with SchedulerConfig::PrefixMatchInfo on a batch whose prompts the
  // engine hashed.
  std::optional<PrefixCacheMatchInfo> PrefixMatch;
};
static_assert(sizeof(ScoredEndpoint) == 32, "the match info lives in the struct's tail");

// attrlatency.LatencyPredictionInfo (datalayer/attribute/latency/data_types.go): what the predicted-latency producer's
// PrepareRequestData stores on an endpoint for a request (predictedlatency/preparedata_hooks.go:36-106).
struct LatencyPredictionInfo {
  bool TTFTValid = false, TPOTValid = false;
  double TTFTHeadroom = 0.0, TPOTHeadroom = 0.0;
  double TTFT = 0.0, TPOT = 0.0;
  int DispatchedRequestCount = 0;
};

struct ProfileRunResult {
  std::vector<ScoredEndpoint> TargetEndpoints;
};
struct SchedulingResult {
  std::map<std::string, ProfileRunResult> ProfileResults;
  std::string PrimaryProfileName;
  // With SchedulerConfig::LatencyPredictionInfo, per profile name: each TargetEndpoints entry's LatencyPredictionInfo attribute,
  // parallel to ProfileResults[name].TargetEndpoints of this result (an entry is empty when no prediction was stored).  Filled
  // from the final result, after the profile handler's ProcessResults, so it follows whatever order and entries the handler
  // returned.  Empty without the option and for batches of the small-batch host route.
  std::map<std::string, std::vector<std::optional<LatencyPredictionInfo>>> TargetLatency;
};

// errcommon.Error{Code: Internal, ...} / fmt.Errorf of the reference, as an exception with the same text
struct SchedulingError : std::runtime_error {
  using std::runtime_error::runtime_error;
};

}  // namespace epp
