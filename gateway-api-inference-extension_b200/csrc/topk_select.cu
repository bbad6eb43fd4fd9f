// topk_select.cu — maxNumOfEndpoints past the register lists (eppscore_schedule_batch_topk_wide): the first k entries of each
// request's pick order, k up to max_endpoints, selected from the weighted score rows the scoring kernels wrote (scores_out,
// NaN = not a candidate).  The order is the one of device_common.cuh's topk_key / topk_before, recomputed here from
// (tie_seed, request_base + r, m) and the score, so a list equals the register lists of score_matrix_kernel<..., TOPK> for
// k <= kTopKMax.
//
// One CTA per request row:
//   1. every candidate's (key, ord) is staged in shared memory as two u64 that order like topk_before (key_bits);
//   2. a radix select over the 128-bit pairs, 8-bit digits from the top, finds the prefix of the min(k, |C|)-th pair; ord
//      carries the endpoint, so the pairs are distinct and exactly min(k, |C|) candidates are at or above it.  Digits that
//      every candidate shares are taken without a pass;
//   3. those winners are compacted in place (a winner's slot never passes its own index) and sorted descending (bitonic);
//   4. entry i gets the winner's endpoint and its score, read back from the row; short lists are padded with -1 / 0.0.
#include "device_common.cuh"

namespace eppscore {

constexpr int kSelBins = 256;

// key as an unsigned word with the order of the doubles (-0.0 first made +0.0, so keys equal as doubles stay equal)
__device__ __forceinline__ unsigned long long key_bits(double key) {
  const double k0 = key == 0.0 ? 0.0 : key;
  const unsigned long long b = (unsigned long long)__double_as_longlong(k0);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ULL);
}

__global__ void __launch_bounds__(1024) topk_select_kernel(const __grid_constant__ TopKSelectArgs a, int cap) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* s_key = reinterpret_cast<unsigned long long*>(smem_raw);  // [cap]
  unsigned long long* s_ord = s_key + cap;                                       // [cap]; 0 = not a candidate
  __shared__ int s_hist[kSelBins];
  __shared__ int s_warp[32];
  __shared__ int s_sel[4];  // chosen bin, rank still needed inside it, whole bin wins, candidate count
  __shared__ unsigned long long s_and[2], s_or[2];  // AND / OR of the candidates' key and ord words
  const int tid = threadIdx.x, B = blockDim.x, lane = tid & 31, warp = tid >> 5, NW = B >> 5;
  const int r = blockIdx.x, M = a.M;
  const double* row = a.scores + (size_t)r * M;
  const uint32_t areq = tie_areq(a.request_base + r, a.seed_lo);
  if (tid == 0) {
    s_sel[3] = 0;
    s_and[0] = s_and[1] = ~0ull;
    s_or[0] = s_or[1] = 0;
  }
  __syncthreads();

  // 1. keys (cap is a multiple of B: every loop below is warp-uniform)
  int n_local = 0;
  unsigned long long and_k = ~0ull, and_o = ~0ull, or_k = 0, or_o = 0;
  for (int m = tid; m < cap; m += B) {
    unsigned long long kb = 0, ord = 0;
    if (m < M) {
      const double s = row[m];
      if (!isnan(s)) {
        double key;
        topk_key(a.pick_mode, a.tie_mode, s, tie_prio(areq, m, a.seed_hi), m, key, ord);
        kb = key_bits(key);
        n_local++;
        and_k &= kb;
        and_o &= ord;
        or_k |= kb;
        or_o |= ord;
      }
    }
    s_key[m] = kb;
    s_ord[m] = ord;
  }
  n_local = __reduce_add_sync(0xffffffffu, n_local);
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    and_k &= __shfl_xor_sync(0xffffffffu, and_k, o);
    and_o &= __shfl_xor_sync(0xffffffffu, and_o, o);
    or_k |= __shfl_xor_sync(0xffffffffu, or_k, o);
    or_o |= __shfl_xor_sync(0xffffffffu, or_o, o);
  }
  if (lane == 0 && n_local) {
    atomicAdd(&s_sel[3], n_local);
    atomicAnd(&s_and[0], and_k);
    atomicAnd(&s_and[1], and_o);
    atomicOr(&s_or[0], or_k);
    atomicOr(&s_or[1], or_o);
  }
  __syncthreads();
  const int n = s_sel[3];
  const int kk = a.k < n ? a.k : n;

  // 2. radix select: the winners are the candidates whose pair, cut to the decided digits (msk), is >= th
  unsigned long long th_k = 0, th_o = 0, msk_k = 0, msk_o = 0;
  if (kk < n) {
    int need = kk;
    // a digit every candidate shares (ties: every key of the random picker is -inf, ord's top bytes are 0) needs no pass
    const unsigned long long same_k = ~(s_and[0] ^ s_or[0]), same_o = ~(s_and[1] ^ s_or[1]);
    for (int d = 0; d < 16; d++) {
      const int shift = 56 - 8 * (d & 7);
      if ((((d < 8 ? same_k : same_o) >> shift) & 255u) == 255u) {  // (block-uniform)
        if (d < 8) {
          th_k |= s_and[0] & (255ull << shift);
          msk_k |= 255ull << shift;
        } else {
          th_o |= s_and[1] & (255ull << shift);
          msk_o |= 255ull << shift;
        }
        continue;
      }
      for (int i = tid; i < kSelBins; i += B) s_hist[i] = 0;
      __syncthreads();
      for (int m0 = 0; m0 < cap; m0 += B) {
        const int m = m0 + tid;
        const unsigned long long kb = s_key[m], o = s_ord[m];
        int dig = -1;
        if (o && (kb & msk_k) == th_k && (o & msk_o) == th_o) dig = (int)(((d < 8 ? kb : o) >> shift) & 255u);
        // one shared-memory atomic per distinct digit of the warp: equal keys (ties) do not serialise on one bin
        const unsigned peers = __match_any_sync(0xffffffffu, dig);
        if (dig >= 0 && lane == __ffs(peers) - 1) atomicAdd(&s_hist[dig], __popc(peers));
      }
      __syncthreads();
      // suffix sums over the bins (thread t < 256 owns bin t; blockDim >= 256): the bin where the count from the top reaches need
      int h = 0, incl = 0;
      if (tid < kSelBins) {
        h = s_hist[tid];
        incl = h;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int v = __shfl_down_sync(0xffffffffu, incl, o);
          if (lane + o < 32) incl += v;
        }
        if (lane == 0) s_warp[warp] = incl;
      }
      __syncthreads();
      if (tid < kSelBins) {
        for (int w = warp + 1; w < kSelBins / 32; w++) incl += s_warp[w];
        const int above = incl - h;
        if (above < need && incl >= need) {
          s_sel[0] = tid;
          s_sel[1] = need - above;
          s_sel[2] = h == need - above;
        }
      }
      __syncthreads();
      const unsigned long long bin = (unsigned long long)s_sel[0];
      need = s_sel[1];
      const bool whole = s_sel[2] != 0;
      if (d < 8) {
        th_k |= bin << shift;
        msk_k |= 255ull << shift;
      } else {
        th_o |= bin << shift;
        msk_o |= 255ull << shift;
      }
      if (whole) break;  // (block-uniform) every candidate with this prefix wins; at the last digit a bin holds one pair
    }
  }

  // 3. compact the kk winners to the front, in rounds of B slots: a winner's new slot is at most its own index, and every
  // slot of the round is read before the first write of the round
  int base = 0;
  for (int m0 = 0; m0 < cap; m0 += B) {
    const int m = m0 + tid;
    const unsigned long long kb = s_key[m], o = s_ord[m];
    const unsigned long long kt = kb & msk_k, ot = o & msk_o;
    const bool win = o != 0 && (kt > th_k || (kt == th_k && ot >= th_o));
    const unsigned bal = __ballot_sync(0xffffffffu, win);
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int pos = base + __popc(bal & ((1u << lane) - 1u)), tot = 0;
    for (int w = 0; w < NW; w++) {
      const int c = s_warp[w];
      pos += w < warp ? c : 0;
      tot += c;
    }
    if (win) {
      s_key[pos] = kb;
      s_ord[pos] = o;
    }
    base += tot;
    __syncthreads();
  }

  // ... and sorted descending: bitonic over the next power of two, padded with (0, 0) (after every candidate)
  int P = 1;
  while (P < kk) P <<= 1;
  for (int i = kk + tid; i < P; i += B) {
    s_key[i] = 0;
    s_ord[i] = 0;
  }
  __syncthreads();
  for (int size = 2; size <= P; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < (P >> 1); i += B) {
        const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
        const unsigned long long k0 = s_key[lo], o0 = s_ord[lo], k1 = s_key[hi], o1 = s_ord[hi];
        const bool lo_first = k0 > k1 || (k0 == k1 && o0 > o1);
        if (((lo & size) == 0) != lo_first) {  // descending blocks where (lo & size) == 0: the whole range at size == P
          s_key[lo] = k1;
          s_ord[lo] = o1;
          s_key[hi] = k0;
          s_ord[hi] = o0;
        }
      }
      __syncthreads();
    }

  // 4. the list
  int32_t* om = a.out_m + (size_t)r * a.k;
  double* os = a.out_s + (size_t)r * a.k;
  for (int i = tid; i < a.k; i += B) {
    int m = -1;
    double s = 0.0;
    if (i < kk) {
      m = topk_endpoint(s_ord[i]);
      s = row[m];
    }
    om[i] = m;
    os[i] = s;
  }
}

int launch_topk_select(const TopKSelectArgs& a, cudaStream_t s) {
  if (a.R <= 0) return 0;
  int cap = 1;
  while (cap < a.M) cap <<= 1;
  // 256 threads (one per histogram bin) up to 2048 endpoints, then up to 1024 so a thread keeps at most 8 slots
  const int threads = cap <= 2048 ? 256 : (cap <= 4096 ? 512 : 1024);
  if (cap < threads) cap = threads;
  int warps = 0;
  int32_t staged = 0;
  size_t smem = 0;
  cudaError_t c = fit_cta_smem((size_t)cap * 16, 0, 0, threads / 32, false, &warps, &staged, &smem);
  if (c == cudaSuccess) c = cudaFuncSetAttribute(topk_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (c != cudaSuccess) return -(int)c;
  return launched_one(launch_maybe_pdl(false, topk_select_kernel, dim3(a.R), dim3(threads), smem, s, a, cap));
}

}  // namespace eppscore
