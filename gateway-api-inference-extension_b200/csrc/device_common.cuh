// device_common.cuh — small device helpers shared by the scoring kernels.
// All float64 arithmetic goes through the _rn intrinsics: never contracted into FMA, so every
// product and sum rounds exactly like the reference's Go code on GOARCH=amd64 (SURVEY.md "Key facts").
#pragma once
#include <utility>

#include "kernels.cuh"

namespace eppscore {

// Programmatic dependent launch (sm_90+): a kernel launched with the programmatic-serialization attribute may start while
// the previous kernel of its stream is still running; it blocks in pdl_wait() until that kernel has completed and its
// writes are visible.  Both are no-ops for an ordinary launch.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// launch with the programmatic-serialization attribute (pdl = false: an ordinary launch)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_maybe_pdl(bool pdl, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// Shared-memory plan of a CTA with up to max_warps warps: `staged` bytes of arrays the kernel can also read from global
// memory, `fixed` bytes per CTA and `per_warp` bytes per warp, within the device's opt-in limit.  Fewer warps come first;
// the staged arrays stay in global memory (only when the kernel can read them there: may_unstage) when not even one warp
// fits beside them.
inline cudaError_t fit_cta_smem(size_t staged, size_t fixed, size_t per_warp, int max_warps, bool may_unstage, int* warps,
                                int32_t* stage, size_t* smem) {
  int dev = 0, optin = 0;
  cudaError_t c = cudaGetDevice(&dev);
  if (c == cudaSuccess) c = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (c != cudaSuccess) return c;
  for (int st = 1; st >= (may_unstage ? 0 : 1); st--)
    for (int w = max_warps; w >= 1; w--) {
      const size_t need = fixed + (st ? staged : 0) + (size_t)w * per_warp;
      if (need <= (size_t)optin) {
        *warps = w;
        *stage = st;
        *smem = need;
        return cudaSuccess;
      }
    }
  return cudaErrorInvalidConfiguration;
}

// a launcher's result for one kernel launch: 1, or -(cudaError_t) when it failed
inline int launched_one(cudaError_t c) { return c == cudaSuccess ? 1 : -(int)c; }

__device__ __forceinline__ double clamp01(double s) {  // enforceScoreRange, scheduler_profile.go:194-202
  if (s < 0.0) return 0.0;
  if (s > 1.0) return 1.0;
  return s;
}
__device__ __forceinline__ uint32_t lowbias32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7feb352dU;
  x ^= x >> 15;
  x *= 0x846ca68bU;
  x ^= x >> 16;
  return x;
}
__device__ __forceinline__ double shfl_xor_f64(double v, int o) {
  int lo = __double2loint(v), hi = __double2hiint(v);
  lo = __shfl_xor_sync(0xffffffffu, lo, o);
  hi = __shfl_xor_sync(0xffffffffu, hi, o);
  return __hiloint2double(hi, lo);
}
__device__ __forceinline__ double shfl_f64(double v, int src) {
  int lo = __double2loint(v), hi = __double2hiint(v);
  lo = __shfl_sync(0xffffffffu, lo, src);
  hi = __shfl_sync(0xffffffffu, hi, src);
  return __hiloint2double(hi, lo);
}
__device__ __forceinline__ long long shfl_xor_i64(long long v, int o) { return __shfl_xor_sync(0xffffffffu, v, o); }
__device__ __forceinline__ uint4 ldg16(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }

// indexer.Get (indexer.go:86-102) on the prefix index, continued from the first load: lo holds the first 16 bytes of slot idx
// ({key.lo, key.hi, cnt, ep0 | ep1 << 16}).  Walks the linear probe to h's slot or to a never-used one and returns whether h
// is present with a non-empty set (an emptied set == a deleted key); idx / lo are left at the last slot loaded.
__device__ __forceinline__ bool table_find(const TSlot* slots, uint64_t mask, uint64_t h, uint64_t& idx, uint4& lo) {
  for (;;) {
    if (lo.z == kCntFree) return false;
    if ((((uint64_t)lo.y << 32) | lo.x) == h) return (lo.z & kCntMask) != 0;
    idx = (idx + 1) & mask;
    lo = ldg16(&slots[idx]);
  }
}
// do two inline sets with the same raw cnt word (not rows) have the same members?  Slots are kept CANONICAL by the index
// program (members sorted, unused entries 0xFFFF: prefix_table.cuh set_member / clear_member) and the second half of a slot
// is loaded for neither or both (same count), so equal sets are equal words.  A stale entry could only make two equal sets
// look different, which sends the request through its exception table — slower, never wrong.
__device__ __forceinline__ bool same_inline_set(uint32_t w0, const uint4& h0, uint32_t w1, const uint4& h1) {
  return ((w0 ^ w1) | (h0.x ^ h1.x) | (h0.y ^ h1.y) | (h0.z ^ h1.z) | (h0.w ^ h1.w)) == 0;
}
__device__ __forceinline__ double nan64() { return __longlong_as_double(0x7ff8000000000000LL); }

// clamp(match/total)*w, prefix/plugin.go:108-110 + scheduler_profile.go:168 (the slow, LUT-less form)
static __device__ __noinline__ double prefix_term_direct(int c, int total, double w) {
  double sc = 0.0;
  if (total != 0) sc = __ddiv_rn((double)c, (double)total);
  return __dmul_rn(clamp01(sc), w);
}

// Arg-max state: MaxScorePicker (maxscore/picker.go:87-115) as "max, size of the arg-max set, chosen member".
struct Best {
  double score;
  int32_t m;  // -1 = none yet
  int32_t cnt;
  uint32_t prio;
};
__device__ __forceinline__ Best best_none() {
  Best b;
  b.score = 0.0;
  b.m = -1;
  b.cnt = 0;
  b.prio = 0;
  return b;
}
__device__ __forceinline__ uint32_t tie_prio(uint32_t areq, int m, uint32_t seed_hi) {
  return lowbias32(areq + (uint32_t)m * 0x9E3779B1U + seed_hi);
}
__device__ __forceinline__ uint32_t tie_areq(int64_t request_index, uint32_t seed_lo) {
  return lowbias32((uint32_t)(uint64_t)request_index ^ seed_lo);
}
// candidates must arrive in ascending m per thread (ties then keep the lowest index in tie_mode 0)
__device__ __forceinline__ void best_update(Best& b, double s, int m, int tie_mode, uint32_t areq, uint32_t seed_hi) {
  // branch-free in the common (lowest-index) mode: two compares and a handful of selects
  const bool first = b.m < 0;
  const bool gt = first || s > b.score;
  const bool eq = !first && s == b.score;
  if (tie_mode) {  // warp-uniform
    if (gt || eq) {
      const uint32_t pr = tie_prio(areq, m, seed_hi);
      if (gt || pr > b.prio) {
        b.prio = pr;
        b.m = m;
      }
    }
  } else {
    b.m = gt ? m : b.m;
  }
  b.score = gt ? s : b.score;
  b.cnt = gt ? 1 : b.cnt + (eq ? 1 : 0);
}
// commutative + associative merge of two partial results
__device__ __forceinline__ void best_merge(Best& b, double os, int om, int oc, uint32_t op, int tie_mode) {
  if (om < 0) return;
  if (b.m < 0 || os > b.score) {
    b.score = os;
    b.m = om;
    b.cnt = oc;
    b.prio = op;
  } else if (os == b.score) {
    b.cnt += oc;
    const bool take = tie_mode ? (op > b.prio || (op == b.prio && om < b.m)) : (om < b.m);
    if (take) {
      b.m = om;
      b.prio = op;
    }
  }
}
template <int WIDTH = 32>
__device__ __forceinline__ void best_group_reduce(Best& b, int tie_mode) {
#pragma unroll
  for (int o = WIDTH / 2; o; o >>= 1) {
    const double os = shfl_xor_f64(b.score, o);
    const int om = __shfl_xor_sync(0xffffffffu, b.m, o);
    const int oc = __shfl_xor_sync(0xffffffffu, b.cnt, o);
    const uint32_t op = __shfl_xor_sync(0xffffffffu, b.prio, o);
    best_merge(b, os, om, oc, op, tie_mode);
  }
}

// ---- stochastic pickers (weightedrandom/picker.go:111-155, random/picker.go:85-101) ----
// 53-bit uniform in (0,1] derived from the tie priority; -ln(u) from +,-,*,/ only, in a fixed order, so the
// oracle (plain C) reproduces every bit: u = f*2^e, f in (sqrt(1/2), sqrt(2)], ln f = 2 atanh((f-1)/(f+1)).
__device__ __forceinline__ double uniform01(uint32_t prio, int m) {
  const uint32_t hi = lowbias32(prio ^ 0x85EBCA6BU);
  const uint32_t lo = lowbias32(hi + 0xC2B2AE35U + (uint32_t)m);
  const unsigned long long k = ((((unsigned long long)hi) << 32) | lo) >> 11;
  return __dmul_rn(__ull2double_rn(k + 1ULL), 1.1102230246251565e-16);  // * 2^-53, exact
}
__device__ __forceinline__ double neg_log(double u) {
  unsigned long long bits = (unsigned long long)__double_as_longlong(u);
  int e = (int)((bits >> 52) & 0x7ff) - 1023;
  double f = __longlong_as_double((long long)((bits & 0x000fffffffffffffULL) | 0x3ff0000000000000ULL));
  if (f > 1.4142135623730951) {
    f = __dmul_rn(f, 0.5);
    e += 1;
  }
  const double z = __ddiv_rn(__dsub_rn(f, 1.0), __dadd_rn(f, 1.0));
  const double z2 = __dmul_rn(z, z);
  double p = 1.0 / 21.0;
#pragma unroll
  for (int k = 19; k >= 1; k -= 2) p = __dadd_rn(__dmul_rn(p, z2), 1.0 / (double)k);
  const double lnf = __dmul_rn(__dmul_rn(2.0, z), p);
  return -__dadd_rn(__dmul_rn((double)e, 0.6931471805599453), lnf);
}
// A-Res key of a candidate with score > 0 (weightedrandom/picker.go:121-152): U^(1/score) maximal <=> -ln(U)/score minimal
__device__ __forceinline__ double ares_key(uint32_t prio, int m, double score) {
  return -__ddiv_rn(neg_log(uniform01(prio, m)), score);
}
// arg-max of a key with the pair's weighted score carried along; lowest index on (improbable) key ties
struct RBest {
  double key, score;
  int32_t m, n;
};
__device__ __forceinline__ RBest rbest_none() {
  RBest b;
  b.key = 0.0;
  b.score = 0.0;
  b.m = -1;
  b.n = 0;
  return b;
}
__device__ __forceinline__ void rbest_update(RBest& b, double key, double score, int m) {
  const bool t = b.m < 0 || key > b.key;
  b.key = t ? key : b.key;
  b.score = t ? score : b.score;
  b.m = t ? m : b.m;
  b.n++;
}
__device__ __forceinline__ void rbest_warp_reduce(RBest& b) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const double ok = shfl_xor_f64(b.key, o), os = shfl_xor_f64(b.score, o);
    const int om = __shfl_xor_sync(0xffffffffu, b.m, o), on = __shfl_xor_sync(0xffffffffu, b.n, o);
    const bool t = om >= 0 && (b.m < 0 || ok > b.key || (ok == b.key && om < b.m));
    b.key = t ? ok : b.key;
    b.score = t ? os : b.score;
    b.m = t ? om : b.m;
    b.n += on;
  }
}

// ---- top-k: maxNumOfEndpoints (picker/common.go:39-42) ----
// Every pick mode is one total order: key descending, then tie descending, then endpoint index ascending.  Its first
// element is what the arg-max states above pick:
//   max-score        key = score, tie = tie_mode ? tie_prio : 0                     (best_update / best_merge)
//   weighted-random  score > 0:  key = ares_key, tie = 2^32 (ahead of any priority)  (rb_pos of rbest_update)
//                    score <= 0: key = -inf, tie = tie_prio                          (rb_all: the random picker)
//   random           key = -inf, tie = tie_prio                                      (rb_all)
// tie and index travel packed in one word, ord = tie << 14 | (16383 - m), so the order is (key, ord) descending
// (m < 8192 = the largest max_endpoints); ord = 0 is an empty entry, after every endpoint.
constexpr int kTopKMax = 8;  // EPPSCORE_MAX_TOPK
constexpr unsigned long long kTopKIdx = 0x3FFF;
__device__ __forceinline__ double neg_inf() { return __longlong_as_double((long long)0xfff0000000000000ULL); }
__device__ __forceinline__ void topk_key(int pick_mode, int tie_mode, double score, uint32_t prio, int m, double& key,
                                         unsigned long long& ord) {
  unsigned long long tie;
  if (pick_mode == 0) {
    key = score;
    tie = tie_mode ? prio : 0u;
  } else if (pick_mode == 1 && score > 0.0) {
    key = ares_key(prio, m, score);
    tie = 1ULL << 32;
  } else {
    key = neg_inf();
    tie = prio;
  }
  ord = (tie << 14) | (kTopKIdx - (unsigned long long)m);
}
__device__ __forceinline__ int topk_endpoint(unsigned long long ord) { return ord ? (int)(kTopKIdx - (ord & kTopKIdx)) : -1; }
__device__ __forceinline__ bool topk_before(double ak, unsigned long long ao, double bk, unsigned long long bo) {
  return ak > bk || (ak == bk && ao > bo);
}
// one lane's best entries, sorted, in registers (every index is a compile-time constant after unrolling)
struct TopK {
  double key[kTopKMax], score[kTopKMax];
  unsigned long long ord[kTopKMax];
};
__device__ __forceinline__ void topk_clear(TopK& t) {
#pragma unroll
  for (int i = 0; i < kTopKMax; i++) {
    t.key[i] = neg_inf();
    t.score[i] = 0.0;
    t.ord[i] = 0;
  }
}
// keep the k best (k <= kTopKMax, warp-uniform)
__device__ __forceinline__ void topk_insert(TopK& t, int k, double key, unsigned long long ord, double score) {
  bool b[kTopKMax];
#pragma unroll
  for (int i = 0; i < kTopKMax; i++) b[i] = i < k && topk_before(key, ord, t.key[i], t.ord[i]);
#pragma unroll
  for (int i = kTopKMax - 1; i >= 0; i--) {
    if (!b[i]) continue;
    if (i > 0 && b[i - 1]) {  // the new entry goes further up: shift
      t.key[i] = t.key[i - 1];
      t.ord[i] = t.ord[i - 1];
      t.score[i] = t.score[i - 1];
    } else {
      t.key[i] = key;
      t.ord[i] = ord;
      t.score[i] = score;
    }
  }
}
// k rounds of a warp arg-max over the list heads; the lane that owns the winner (lane = m & 31 in every kernel's endpoint
// layout) pops its head.  Lane i returns the i-th entry of the warp's order (-1, 0.0 past the last candidate).
__device__ __forceinline__ void topk_warp_merge(TopK& t, int k, int lane, int& out_m, double& out_score) {
  out_m = -1;
  out_score = 0.0;
  for (int i = 0; i < k; i++) {
    double bk = t.key[0];
    unsigned long long bo = t.ord[0];
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      const double ok = shfl_xor_f64(bk, o);
      const unsigned long long oo = __shfl_xor_sync(0xffffffffu, bo, o);
      if (topk_before(ok, oo, bk, bo)) {
        bk = ok;
        bo = oo;
      }
    }
    if (bo == 0) break;  // (warp-uniform) no candidate left
    const int m = topk_endpoint(bo), owner = m & 31;
    const double s = shfl_f64(t.score[0], owner);
    if (lane == i) {
      out_m = m;
      out_score = s;
    }
    if (lane == owner) {
#pragma unroll
      for (int j = 0; j < kTopKMax - 1; j++) {
        t.key[j] = t.key[j + 1];
        t.ord[j] = t.ord[j + 1];
        t.score[j] = t.score[j + 1];
      }
      t.key[kTopKMax - 1] = neg_inf();
      t.ord[kTopKMax - 1] = 0;
    }
  }
}

// Weighted score of one (request, endpoint) pair, steps in profile order from 0.0
// (scheduler_profile.go:155-168). Runtime-generic: used on rare paths (exceptions, summaries).
__device__ __forceinline__ double eval_steps(const Plan& plan, const double* const* term, int m, int c, int total, int cls) {
  double acc = 0.0;
  for (int s = 0; s < plan.n_steps; s++) {
    const int kind = plan.kind[s];
    double t;
    if (kind == STEP_EP_TERM) {
      t = __ldg(term[plan.arg[s]] + m);
    } else if (kind == STEP_PREFIX) {
      t = (c == 0) ? __dmul_rn(0.0, plan.weight[s]) : prefix_term_direct(c, total, plan.weight[s]);
    } else if (kind == STEP_LORA) {
      const double* lt = plan.lora_term[s];
      t = cls == 3 ? lt[3] : (cls == 2 ? lt[2] : (cls == 1 ? lt[1] : lt[0]));
    } else {
      t = __dmul_rn(0.0, plan.weight[s]);
    }
    acc = __dadd_rn(acc, t);
  }
  return acc;
}

}  // namespace eppscore
