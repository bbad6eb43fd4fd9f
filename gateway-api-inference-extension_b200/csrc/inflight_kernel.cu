// inflight_kernel.cu — the inflight-load-producer (requestcontrol/dataproducer/inflightload/producer.go) on the device:
//   (1) inflight_update_kernel: PreRequest (:101-120) / ResponseBody at end of stream (:122-169) for a whole batch — a signed
//       scatter-add of (1 request, tokens[r]) into the per-endpoint counters;
//   (2) estimate_tokens_kernel: SimpleTokenEstimator.Estimate with its defaults (token_estimator.go:36-72), one thread per
//       request, in integer arithmetic.
#include "kernels.cuh"

namespace eppscore {

constexpr int kInflightThreads = 512;
constexpr int kInflightPerCta = 4096;  // requests per CTA: the per-CTA histogram is zeroed and flushed once per 4096 requests

// Every update is an integer add, so the counters do not depend on the order the adds land in.  Under dog-piling (every
// pick on one endpoint) one global atomic per request would serialise in L2; instead the lanes of a warp that name the same
// endpoint are combined first (__match_any_sync), each group adds once into a per-CTA shared-memory histogram, and each CTA
// issues one global atomicAdd per endpoint it saw.  The histogram holds 16 bytes per endpoint (n_ep <= 8192: at most
// 128 KiB).  Counters are int64 kept as two's complement in uint64 atomics: adds of either sign are exact modulo 2^64.
__global__ void __launch_bounds__(kInflightThreads) inflight_update_kernel(const int32_t* __restrict__ endpoint,
                                                                         const int64_t* __restrict__ tokens, int R, int n_ep,
                                                                         int sign, unsigned long long* requests,
                                                                         unsigned long long* token_sum, uint32_t* err) {
  extern __shared__ unsigned long long s_hist[];  // [n_ep] requests, then [n_ep] tokens
  __shared__ unsigned long long s_val[kInflightThreads];
  unsigned long long* s_req = s_hist;
  unsigned long long* s_tok = s_hist + n_ep;
  for (int i = threadIdx.x; i < 2 * n_ep; i += blockDim.x) s_hist[i] = 0ull;
  __syncthreads();
  const int lane = threadIdx.x & 31, wbase = threadIdx.x & ~31;
  const int lo = blockIdx.x * kInflightPerCta, hi = min(R, lo + kInflightPerCta);
  for (int base = lo; base < hi; base += blockDim.x) {  // base is uniform per CTA: whole warps take every iteration
    const int r = base + threadIdx.x;
    int m = -1;
    unsigned long long t = 0ull;
    if (r < hi) {
      m = endpoint[r];
      t = tokens ? (unsigned long long)tokens[r] : 0ull;
      if (m >= n_ep) {  // host-array calls are validated before the launch; a device array may still name one
        atomicOr(err, 1u);
        m = -1;
      }
    }
    const unsigned peers = __match_any_sync(0xffffffffu, m);
    s_val[threadIdx.x] = t;
    __syncwarp();
    if (m >= 0 && lane == __ffs(peers) - 1) {
      unsigned long long sum = 0ull;
      for (unsigned p = peers; p; p &= p - 1) sum += s_val[wbase + __ffs(p) - 1];
      atomicAdd(&s_req[m], (unsigned long long)__popc(peers));
      atomicAdd(&s_tok[m], sum);
    }
    __syncwarp();
  }
  __syncthreads();
  for (int m = threadIdx.x; m < n_ep; m += blockDim.x) {
    const unsigned long long q = s_req[m];
    if (q == 0ull) continue;  // no request of this CTA named m
    const unsigned long long k = s_tok[m];
    atomicAdd(&requests[m], sign > 0 ? q : 0ull - q);
    atomicAdd(&token_sum[m], sign > 0 ? k : 0ull - k);
  }
}

// Estimate(request) for R requests (token_estimator.go:48-72, CharactersPerToken 4.0, OutputRatio 1.5):
//   RequestSizeBytes > 0       input = max(size / 4, 1)                       (integer division, :55-56)
//   else Body == nil           0                                              (chars < 0 here, :67-68)
//   else hint >= 0             input = hint                                   (:58-60)
//   else                       input = max(1, round(chars / 4.0))             (:64-65)
//   result = input + round(input * 1.5)                                       (:70-71)
// For c, i >= 0 Go's math.Round (half away from zero) gives round(c / 4.0) = (c + 2) >> 2 and round(1.5 i) = (3i + 1) >> 1,
// exact while 1.5 i is exact in float64 (i < 2^52).
__global__ void estimate_tokens_kernel(const int64_t* __restrict__ size, const int32_t* __restrict__ hint,
                                       const int32_t* __restrict__ chars, int R, int64_t* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const long long sz = size ? size[r] : 0;
  long long in;
  if (sz > 0) {
    in = max(sz / 4, 1LL);
  } else {
    const long long c = chars ? chars[r] : 0;
    if (c < 0) {
      out[r] = 0;
      return;
    }
    const long long h = hint ? hint[r] : -1;
    in = h >= 0 ? h : max((c + 2) >> 2, 1LL);
  }
  out[r] = in + ((3 * in + 1) >> 1);
}

// The attribute belongs to the kernel, not to an engine: always the largest histogram (8192 endpoints), so that engines of
// different sizes on one device never lower it under each other.
cudaError_t init_inflight_update() {
  return cudaFuncSetAttribute(inflight_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              8192 * 2 * (int)sizeof(unsigned long long));
}

int launch_inflight_update(const int32_t* endpoint, const int64_t* tokens, int R, int n_ep, int sign, int64_t* requests,
                           int64_t* token_sum, uint32_t* err, cudaStream_t s) {
  if (R <= 0) return 0;
  const size_t smem = (size_t)n_ep * 2 * sizeof(unsigned long long);
  const int grid = (R + kInflightPerCta - 1) / kInflightPerCta;
  inflight_update_kernel<<<grid, kInflightThreads, smem, s>>>(endpoint, tokens, R, n_ep, sign,
                                                              reinterpret_cast<unsigned long long*>(requests),
                                                              reinterpret_cast<unsigned long long*>(token_sum), err);
  return 1;
}

int launch_estimate_tokens(const int64_t* size, const int32_t* hint, const int32_t* chars, int R, int64_t* out, cudaStream_t s) {
  if (R <= 0) return 0;
  estimate_tokens_kernel<<<(R + 255) / 256, 256, 0, s>>>(size, hint, chars, R, out);
  return 1;
}

}  // namespace eppscore
