// lat_pair.cuh — the predicted-latency producer's arithmetic for one (request, endpoint) pair, shared by the latency fold-in of
// the scoring kernels (score_matrix.cu), the chosen-endpoint lookup (prefix_index.cu: latency_info_kernel), the in-order walk
// (inorder_kernel.cu) and the snapshot preparation of the tiles (prepare_kernel.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace eppscore {

// One (request, endpoint) pair of the predicted-latency producer: TTFT/TPOT (prediction.go:171-185, left to right),
// headrooms (predictedlatency/prediction.go:143-161, :100-104), the TPOT bound the headroom is taken against, and the
// endpoint's tier:
//   0 positive, 1 negative & idle, 2 only TPOT negative, 3 only TTFT negative, 4 both negative
// (plugin.go:177-238: the scorer scores the lowest non-empty tier only).
struct LatPair {
  double ttft, tpot, hT, hP;
  double buffered;  // min(bufferedTPOT, podMinTPOTSLO*factor)
  int rank;
};
// The pair from the endpoint's slot values (tile slots 0-5, lim = slot 6, fl = the flag bits of slot 7): the form of the
// in-order walk, which keeps the static slots in shared memory and lim / the idle bit in registers.
__device__ __forceinline__ LatPair lat_pair_slots(double tA, double tW, double tR, double pA, double pW, double pR, double lim,
                                                  int fl, double tpot_generated, double pref_term, double x_in, double y_in,
                                                  double ttft_slo, double buf_tpot) {
  LatPair o;
  o.ttft = __dadd_rn(__dadd_rn(__dadd_rn(__dadd_rn(tA, x_in), tW), tR), pref_term);
  o.tpot = __dadd_rn(__dadd_rn(__dadd_rn(__dadd_rn(pA, y_in), pW), pR), tpot_generated);  // NumTokensGenerated = 1 (prediction.go:69)
  o.hT = __dsub_rn(ttft_slo, o.ttft);
  o.buffered = lim < buf_tpot ? lim : buf_tpot;
  o.hP = (fl & 2) ? 0.0 : __dsub_rn(o.buffered, o.tpot);
  const bool tn = o.hT < 0.0, pn = o.hP < 0.0;
  o.rank = !(tn || pn) ? 0 : ((fl & 1) ? 1 : (tn && pn ? 4 : (tn ? 3 : 2)));
  return o;
}
// tile layout of the per-endpoint arrays: slot i of endpoint (t*32 + lane) lives at ((t*8 + i)*32 + lane), so one
// address per pair and seven coalesced 8-byte loads at immediate offsets (kernels.cuh: LatArgs)
__device__ __forceinline__ LatPair lat_pair(const double* tp, double tpot_generated, double pref_term, double x_in,
                                            double y_in, double ttft_slo, double buf_tpot) {
  return lat_pair_slots(__ldg(tp), __ldg(tp + 32), __ldg(tp + 64), __ldg(tp + 96), __ldg(tp + 128), __ldg(tp + 160),
                        __ldg(tp + 192), __ldg(reinterpret_cast<const int*>(tp + 224)), tpot_generated, pref_term, x_in, y_in,
                        ttft_slo, buf_tpot);
}

// The two tile values the running-request queues move (slot 6 and bit 0 of slot 7), from getEndpointMinTPOTSLO (0 when the
// endpoint has no running request) and getEndpointRunningRequestCount: lim = podMinTPOTSLO > 0 ? podMinTPOTSLO*buffer : +inf
// (prediction.go:149-161), idle = no running request (plugin.go:189-202).
__device__ __forceinline__ double lat_lim(double pod_min, double buffer) {
  return pod_min > 0.0 ? __dmul_rn(pod_min, buffer) : __longlong_as_double(0x7ff0000000000000LL);
}
__device__ __forceinline__ bool lat_idle(int dispatched) { return dispatched == 0; }

// An endpoint's |headroom| as it enters its tier's minimum: scoreBucket (plugin.go:262-318) starts the minimum at
// math.MaxFloat64 and lowers it with h < min, so an infinite headroom (an infinite SLO) leaves it at MaxFloat64, not +Inf.
__device__ __forceinline__ double lat_min_in(double h) { return h < 1.7976931348623157e308 ? h : 1.7976931348623157e308; }

// Go's int(x) on amd64 (CVTTSD2SQ) for scoreBucket's weight: truncation toward zero, and NaN as math.MinInt64, which the score
// range then clamps to 0.  The weight is NaN for an infinite headroom in a tier whose range is infinite ((+Inf - MaxFloat64) /
// +Inf), so NaN is mapped here explicitly rather than left to __double2ll_rz.
__device__ __forceinline__ long long go_int(double x) { return x == x ? __double2ll_rz(x) : (long long)0x8000000000000000ULL; }

// The inputs of latency_info_kernel beyond the match lookup's (DeviceIndex::latency_info): the engine's prepared snapshot
// (LatArgs' tiles and scalars) and the running-request view, plus the requests' own inputs and the output records.
struct LatInfoArgs {
  int32_t R, k, M;                 // M: the snapshot's endpoint count (entries outside [0, M) are not present)
  int32_t has_predictions;
  const uint64_t* hashes;          // [R][stride]
  const uint16_t* n_hashes;        // [R]
  int32_t stride;
  const int32_t* endpoints;        // [R][k]
  const double* ep;                // [Mpad/32][kLatArrays][32] tiles (kernels.cuh: LatArgs)
  const int32_t* dispatched;       // [M] getEndpointRunningRequestCount as the tiles were prepared from
  double ttft_input, ttft_prefix, tpot_input, tpot_generated, buffer;
  const int32_t* input_tokens;     // [R] or null (0)
  const double* ttft_slo;          // [R] or null (0)
  const double* tpot_slo;          // [R] or null (0)
  uint16_t* match_out;             // [R][k] or null
  void* out;                       // [R][k] eppscore_latency_info
};

}  // namespace eppscore
