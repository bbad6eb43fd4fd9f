// inorder_kernel.cu — a batch scheduled in arrival order against the in-flight load (eppscore_schedule_batch_inorder): request r
// is scored with the token-load terms left by requests 0..r-1's picks, as R consecutive Scheduler.Schedule + PreRequest calls
// see them (inflightload/producer.go:101-120 feeding scorer/tokenload/token_load.go:83-111).
//   inorder_minmax_kernel  per request, in parallel: min / max of WaitingQueueSize and RunningRequestsSize over its candidates
//                          (queue.go:79-91 over the FILTERED endpoints)
//   inorder_pick_kernel    one thread-block cluster walks the requests in order.  Thread t of CTA c owns endpoint c*T + t: its
//                          in-flight counters live in its registers, its request-independent terms in shared memory.  Per
//                          request every thread scores its endpoint in profile order (the float64 operations of
//                          score_matrix_kernel, and of prepare_endpoints_kernel's token-load branch for the moving term), the
//                          CTA reduces to a winner, the cluster merges the CTA winners through distributed shared memory behind
//                          barrier.cluster, and the owner of the pick adds the request's tokens.
// The prefix match counts and totals come from the ordinary batch kernels (their match_out route), which depend on no load.
//   inorder_index_kernel   the same walk ordered against the prefix index too (eppscore_schedule_batch_inorder_index): each
//                          request's match counts are probed from the index as the earlier requests' Adds left it, and the CTA
//                          that owns the pick runs the index's commit program (IndexProgram::commit) for the request's Add.
//   inorder_pick_lat_kernel, inorder_index_lat_kernel   either walk with the latency scorer ordered against the running-request
//                          queues (eppscore_schedule_batch_inorder_latency): each thread keeps its endpoint's running count and
//                          minimum tpot in registers, the cluster reduces request r's tier and headroom ranges (one more
//                          barrier.cluster), and the owner of the pick adds request r to its queue (requestcontrol_hooks.go:73-86).
//   inorder_profiles_kernel, inorder_index_profiles_kernel   either walk over several profile runs
//                          (eppscore_schedule_batch_inorder_profiles): each thread scores its endpoint once per run in that
//                          run's profile order, every CTA publishes one winner per run behind the request's one
//                          barrier.cluster, and when the primary run picked, each run's pick owner adds the request's tokens and
//                          the owners of the primary and prefill picks run the index's commit program for those two Adds.
#include <cooperative_groups.h>

#include "device_common.cuh"
#include "index_device.cuh"
#include "lat_pair.cuh"
#include "running_slot.cuh"

namespace cg = cooperative_groups;

namespace eppscore {

constexpr int kInOrderMaxThreads = 512;  // 128 registers per thread: the next request's inputs are prefetched
constexpr int kInOrderWarps = kInOrderMaxThreads / 32;

__global__ void __launch_bounds__(256) inorder_minmax_kernel(const __grid_constant__ InOrderArgs a) {
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (int r = gw; r < a.R; r += nw) {
    long long mn[2] = {0x7fffffffffffffffLL, 0x7fffffffffffffffLL};
    long long mx[2] = {(long long)0x8000000000000000ULL, (long long)0x8000000000000000ULL};
    const uint32_t* mrow = a.cand_mask ? a.cand_mask + (size_t)r * a.mask_words : nullptr;
    for (int m = lane; m < a.M; m += 32) {
      if (mrow && !((__ldg(mrow + (m >> 5)) >> (m & 31)) & 1u)) continue;
      if (a.member && !((__ldg(a.member + (m >> 5)) >> (m & 31)) & 1u)) continue;
#pragma unroll
      for (int which = 0; which < 2; which++) {
        const int64_t* q = which == 0 ? a.queue : a.running;
        const long long v = q ? __ldg(reinterpret_cast<const long long*>(q) + m) : 0LL;
        mn[which] = v < mn[which] ? v : mn[which];
        mx[which] = v > mx[which] ? v : mx[which];
      }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1)
#pragma unroll
      for (int which = 0; which < 2; which++) {
        const long long omn = shfl_xor_i64(mn[which], o), omx = shfl_xor_i64(mx[which], o);
        mn[which] = omn < mn[which] ? omn : mn[which];
        mx[which] = omx > mx[which] ? omx : mx[which];
      }
    if (lane < 4) a.minmax[(size_t)r * 4 + lane] = lane == 0 ? mn[0] : (lane == 1 ? mx[0] : (lane == 2 ? mn[1] : mx[1]));
  }
}

// clamp(score) of the token-load scorer for an endpoint with `tokens` in flight (prepare_kernel.cu, token_load.go:96-106)
__device__ __forceinline__ double token_load_score(long long tokens, double threshold) {
  double load = __ll2double_rn(tokens);
  if (load <= 0.0) return 1.0;
  if (load > threshold) load = threshold;
  return clamp01(__dsub_rn(1.0, __ddiv_rn(load, threshold)));
}

// One CTA's (or warp's) partial result: the max-score state, or the two stochastic-picker states.
struct InOrderBest {
  Best b;
  RBest pos, all;
};

template <bool RND>
__device__ __forceinline__ void inorder_warp_reduce(InOrderBest& x, int tie_mode) {
  if (RND) {
    rbest_warp_reduce(x.pos);
    rbest_warp_reduce(x.all);
  } else {
    best_group_reduce<32>(x.b, tie_mode);
  }
}
__device__ __forceinline__ InOrderBest inorder_none() {
  InOrderBest x;
  x.b = best_none();
  x.pos = rbest_none();
  x.all = rbest_none();
  return x;
}

// Per-request inputs of one thread's endpoint: loaded one request ahead, while the previous request is reduced.
struct InOrderReq {
  long long mn0, mx0, mn1, mx1;  // queue, running
  int32_t c, total, cls;
  bool cand;
  long long tokens;
};

// The latency walk's per-request inputs (tile terms of the request, prediction.go:171-185 and :150), loaded one request ahead.
struct InOrderLatReq {
  double x, y;     // ttft_input * input_tokens, tpot_input * input_tokens
  double tslo;     // TTFT SLO
  double tpot;     // TPOT SLO (avgTPOTSLO): the bound's input and the value the Add queues
  unsigned long long key;
};

// One CTA's (or warp's) share of request r's tier selection (plugin.go:177-238): the lowest tier among its candidates and the
// |headroom| min / max inside it.  The merge keeps the lower tier, or combines the ranges of an equal one: associative and
// commutative, so any reduction order gives score_matrix_kernel's one-pass result.
struct LatTier {
  int rank;
  double mnT, mxT, mnP, mxP;
};
__device__ __forceinline__ LatTier lat_tier_none() {
  return LatTier{5, 1.7976931348623157e308, -1.7976931348623157e308, 1.7976931348623157e308, -1.7976931348623157e308};
}
__device__ __forceinline__ void lat_tier_merge(LatTier& x, const LatTier& o) {
  const bool better = o.rank < x.rank, same = o.rank == x.rank;
  x.mnT = (better || (same && o.mnT < x.mnT)) ? o.mnT : x.mnT;
  x.mxT = (better || (same && o.mxT > x.mxT)) ? o.mxT : x.mxT;
  x.mnP = (better || (same && o.mnP < x.mnP)) ? o.mnP : x.mnP;
  x.mxP = (better || (same && o.mxP > x.mxP)) ? o.mxP : x.mxP;
  x.rank = better ? o.rank : x.rank;
}
__device__ __forceinline__ void lat_tier_warp_reduce(LatTier& x) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    LatTier y;
    y.rank = __shfl_xor_sync(0xffffffffu, x.rank, o);
    y.mnT = shfl_xor_f64(x.mnT, o);
    y.mxT = shfl_xor_f64(x.mxT, o);
    y.mnP = shfl_xor_f64(x.mnP, o);
    y.mxP = shfl_xor_f64(x.mxP, o);
    lat_tier_merge(x, y);
  }
}
constexpr int kLatStatic = 6;  // tile slots 0-5: request-independent for the whole walk (kernels.cuh: LatArgs)

// The hit slots of one round of a request's probes, staged in shared memory (IDX): the cnt word and ep[0..10) of each.
struct InOrderHits {
  uint32_t raw[kCommitThreads];
  uint32_t ep[kCommitThreads][kInlineEps / 2];  // ep pairs as the slot holds them; in row mode ep[0] is the row id
  uint32_t first[2];                            // first miss of the current round (double-buffered, reset one round ahead)
};

// A run's pick of one request in the profiles walk.
struct InOrderPick {
  double score;
  int32_t m, cnt;
};

// The walk, in the in-flight form (IDX false: inorder_pick_kernel) or the index form (IDX true: inorder_index_kernel, CTAs of
// kCommitThreads threads; dynamic shared memory = the terms, then the CommitSmem of IndexProgram).  LAT: with the latency scorer
// (the _lat kernels): the terms are followed by the kLatStatic static tile slots of each thread's endpoint, before the CommitSmem.
// PROF: over the runs of pa (the _profiles kernels; RND unused, each run's picker is read at run time): the terms of run i sit
// in slots [term_base, term_base + n_scorers), Σ n_scorers slots before the CommitSmem.
template <bool RND, bool IDX, bool LAT, bool PROF = false>
__device__ __forceinline__ void inorder_walk(const InOrderArgs& a, const InOrderIndexArgs& ix, const InOrderLatArgs& lt,
                                             const InOrderProfArgs* pa = nullptr) {
  constexpr int kTermSlots = kMaxSteps + (LAT ? kLatStatic : 0);
  extern __shared__ __align__(16) double s_term[];  // [n_scorers][blockDim.x]: the request-independent terms of each thread's endpoint
  __shared__ InOrderBest s_warp[kInOrderWarps];
  __shared__ InOrderBest s_cta[2];  // the CTA's winner of the last two requests (read by the other CTAs of the cluster)
  cg::cluster_group cluster = cg::this_cluster();
  const int T = blockDim.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = T >> 5;
  const int C = (int)cluster.num_blocks();
  const int m = (int)cluster.block_rank() * T + tid;
  const bool real = m < a.M;
  const int tie_mode = a.tie_mode;

  if constexpr (!PROF)
    for (int s = 0; s < a.n_scorers; s++) s_term[(size_t)s * T + tid] = (real && a.term[s]) ? a.term[s][m] : 0.0;
  uint32_t members = 0;  // PROF: bit i = this endpoint is in run i's profile subset
  int slots = kTermSlots;
  if constexpr (PROF) {
#pragma unroll 1
    for (int i = 0; i < pa->n_runs; i++) {
      const InOrderRun& u = pa->run[i];
      for (int s = 0; s < u.n_scorers; s++) s_term[(size_t)(u.term_base + s) * T + tid] = (real && u.term[s]) ? u.term[s][m] : 0.0;
      if (real && (!u.member || ((__ldg(u.member + (m >> 5)) >> (m & 31)) & 1u))) members |= 1u << i;
    }
    slots = pa->run[pa->n_runs - 1].term_base + pa->run[pa->n_runs - 1].n_scorers;
  }
  const long long q0 = (real && a.queue) ? a.queue[m] : 0LL, q1 = (real && a.running) ? a.running[m] : 0LL;
  const bool member = real && (!a.member || ((__ldg(a.member + (m >> 5)) >> (m & 31)) & 1u));
  long long tok = m < a.Mpad ? a.inflight_tok[m] : 0, req = m < a.Mpad ? a.inflight_req[m] : 0;
  double tl = real ? token_load_score(tok, a.token_threshold) : 0.0;
  const uint32_t pos = perm_bitpos((uint32_t)(m < a.Mpad ? m : 0), a.log_epl);

  auto load = [&](int r) {
    InOrderReq x;
    x.cand = member && r < a.R;
    x.c = x.total = x.cls = 0;
    x.tokens = 0;
    x.mn0 = x.mx0 = x.mn1 = x.mx1 = 0;
    if (r >= a.R) return x;
    if (a.cand_mask) x.cand = x.cand && ((__ldg(a.cand_mask + (size_t)r * a.mask_words + (m >> 5)) >> (m & 31)) & 1u);
    if (a.match && real) x.c = __ldg(a.match + (size_t)r * a.M + m);
    if (a.total) x.total = __ldg(a.total + r);
    if (a.minmax) {
      const long long* mm = reinterpret_cast<const long long*>(a.minmax) + (size_t)r * 4;
      x.mn0 = __ldg(mm);
      x.mx0 = __ldg(mm + 1);
      x.mn1 = __ldg(mm + 2);
      x.mx1 = __ldg(mm + 3);
    }
    if (a.cls_lo && real) {
      int ad = a.adapter_id ? __ldg(a.adapter_id + r) : -1;
      if (ad < 0 || ad >= a.A) ad = a.A;
      const size_t word = (size_t)ad * a.RW + (pos >> 5);
      x.cls = (int)((__ldg(a.cls_lo + word) >> (pos & 31)) & 1u) | ((int)((__ldg(a.cls_hi + word) >> (pos & 31)) & 1u) << 1);
    }
    if (a.tokens) x.tokens = __ldg(reinterpret_cast<const long long*>(a.tokens) + r);
    return x;
  };
  // PROF: request r's candidate bit of each run at this endpoint: subset ∧ run_mask ∧ the run's cand_mask
  auto load_cands = [&](auto r) {  // (generic: instantiated by the PROF walk alone)
    uint32_t b = 0;
    if (r >= a.R) return b;
    const uint32_t rm = pa->run_mask ? (uint32_t)__ldg(pa->run_mask + r) : 0xFu;
#pragma unroll 1
    for (int i = 0; i < pa->n_runs; i++) {
      const uint32_t* cm = pa->run[i].cand_mask;
      bool c = ((members & rm) >> i) & 1u;
      if (c && cm) c = (__ldg(cm + (size_t)r * a.mask_words + (m >> 5)) >> (m & 31)) & 1u;
      b |= (uint32_t)c << i;
    }
    return b;
  };

  // LAT: this thread's endpoint in the latency fold-in.  The static tile slots go to shared memory; lim (slot 6) and the idle
  // bit (slot 7 bit 0) come from the tiles, or with request keys from this endpoint's running count, minimum tpot (bits) and
  // count at the minimum, which live in registers and move with its own Adds.
  double* s_lat = s_term + (size_t)kMaxSteps * T;  // [kLatStatic][T]
  double lim = 0.0;
  bool idle = false, neutral = false;
  int run_cnt = 0, run_mincnt = 0;
  unsigned long long run_min = kRunMinNone;
  if constexpr (LAT) {
    const bool tiled = m < a.Mpad;
    const double* tp = lt.lat.ep + (size_t)(m >> 5) * 256 + (m & 31);
#pragma unroll
    for (int i = 0; i < kLatStatic; i++) s_lat[(size_t)i * T + tid] = tiled ? __ldg(tp + 32 * i) : 0.0;
    if (tiled) {
      lim = __ldg(tp + 192);
      const int fl = __ldg(reinterpret_cast<const int*>(tp + 224));
      idle = fl & 1;
      neutral = fl & 2;
    }
    if (lt.request_key && m < lt.n_ep) {  // (then the snapshot took both values from the queues, as here; a later slice of the
                                          // call sees the earlier slices' Adds only here)
      const RunDev* d = lt.run;
      run_cnt = d->count[m];
      run_min = d->min_bits[m];
      run_mincnt = d->min_cnt[m];
      lim = lat_lim(run_cnt > 0 ? __longlong_as_double((long long)run_min) : 0.0, lt.lat.buffer);
      idle = lat_idle(run_cnt);
    }
  }
  auto load_lat = [&](int r) {
    InOrderLatReq x{};
    if (r >= a.R) return x;
    const LatArgs& L = lt.lat;
    const double in_tok = (double)(L.input_tokens ? __ldg(L.input_tokens + r) : 0);  // len(strings.Fields(prompt))
    x.x = __dmul_rn(L.ttft_input, in_tok);
    x.y = __dmul_rn(L.tpot_input, in_tok);
    x.tslo = L.ttft_slo ? __ldg(L.ttft_slo + r) : 0.0;
    x.tpot = L.tpot_slo ? __ldg(L.tpot_slo + r) : 0.0;
    x.key = lt.request_key ? __ldg(reinterpret_cast<const unsigned long long*>(lt.request_key) + r) : 0ull;
    return x;
  };

  // IDX: the index as the walk mutates it.  Every read goes through DevX's relaxed GPU-scope loads (never the read-only path:
  // the table changes under this kernel); barrier.cluster orders a commit before the next request's probes.
  DevX dx;
  InOrderHits* hits = nullptr;
  uint32_t parity = 0;
  if constexpr (IDX) {
    __shared__ InOrderHits s_hits;
    hits = &s_hits;
    if (tid < 2) hits->first[tid] = 0xFFFFFFFFu;
  }

  cluster.sync();  // every CTA of the cluster is running before any reads another's shared memory
  InOrderReq cur = load(0);
  uint32_t cands = 0;
  if constexpr (PROF) cands = load_cands(0);
  InOrderLatReq lcur{};  // (loaded one request ahead in the in-flight form; the index form has no registers to spare for that,
                         // and its probes cover the loads)
  if constexpr (LAT && !IDX) lcur = load_lat(0);
  for (int r = 0; r < a.R; r++) {
    const InOrderReq nxt = load(r + 1);
    uint32_t cands_nxt = 0;
    if constexpr (PROF) cands_nxt = load_cands(r + 1);
    InOrderLatReq lnxt{};
    if constexpr (LAT && IDX) lcur = load_lat(r);
    if constexpr (LAT && !IDX) lnxt = load_lat(r + 1);
    if constexpr (IDX) {
      // ---- matchLongestPrefix (plugin.go:219-235) at this thread's endpoint, against the index after requests 0..r-1's Adds:
      // T probes per round up to the first global miss, the hit slots staged in shared memory, then every thread counts the
      // hits whose set holds its endpoint (slot_holds: an inline member or bit m of the row) ----
      const uint32_t n = (uint32_t)cur.total;
      const uint64_t* h = ix.hashes + (size_t)r * ix.stride;
      const TableView* tv = ix.tv;
      uint32_t c = 0;
      for (uint32_t base = 0; base < n; base += (uint32_t)T) {
        const bool in = base + tid < n;
        uint32_t raw = 0;
        TSlot* sl = in ? table_find(dx, tv, __ldg(reinterpret_cast<const unsigned long long*>(h) + base + tid), &raw) : nullptr;
        if (sl) {
          hits->raw[tid] = raw;
          const uint32_t* w = reinterpret_cast<const uint32_t*>(sl) + 3;
#pragma unroll
          for (int k = 0; k < kInlineEps / 2; k++) hits->ep[tid][k] = dx.ld32(w + k);
        }
        const uint32_t miss = __ballot_sync(0xffffffffu, in && !sl);
        if (lane == 0 && miss) atomicMin(&hits->first[parity], (uint32_t)(warp * 32 + __ffs(miss) - 1));
        __syncthreads();
        const uint32_t first = hits->first[parity];
        if (tid == 0) hits->first[parity ^ 1] = 0xFFFFFFFFu;
        uint32_t nh = n - base < (uint32_t)T ? n - base : (uint32_t)T;
        nh = first < nh ? first : nh;
        if (real)
          for (uint32_t k = 0; k < nh; k++) c += staged_holds(dx, tv, hits->raw[k], hits->ep[k], (uint32_t)m) ? 1u : 0u;
        __syncthreads();  // the staged hits are read before the next round overwrites them
        parity ^= 1;
        if (first != 0xFFFFFFFFu) break;
      }
      cur.c = (int32_t)c;
    }
    // ---- The latency scorer (scorer/latency/plugin.go:144-360) at this thread's endpoint: w, the scoreBucket weight ----
    long long lat_w = 0;
    if constexpr (LAT) {
      const LatArgs& L = lt.lat;
      const double pt = __dmul_rn(L.has_predictions ? L.ttft_prefix : L.wpref,
                                  cur.total ? __ddiv_rn((double)cur.c, (double)cur.total) : 0.0);  // preparedata_hooks.go:44-58
      if (L.has_predictions) {
        const LatPair lp = lat_pair_slots(s_lat[tid], s_lat[(size_t)T + tid], s_lat[(size_t)2 * T + tid], s_lat[(size_t)3 * T + tid],
                                          s_lat[(size_t)4 * T + tid], s_lat[(size_t)5 * T + tid], lim,
                                          (idle ? 1 : 0) | (neutral ? 2 : 0), L.tpot_generated, pt, lcur.x, lcur.y, lcur.tslo,
                                          __dmul_rn(lcur.tpot, L.buffer));
        const double aT = fabs(lp.hT), aP = fabs(lp.hP);
        // the lowest tier over the candidates and the |headroom| ranges inside it: warp, CTA, then cluster (barrier.cluster)
        __shared__ LatTier s_wtier[kInOrderWarps];
        __shared__ LatTier s_ctier[2];
        LatTier t = cur.cand ? LatTier{lp.rank, lat_min_in(aT), aT, lat_min_in(aP), aP} : lat_tier_none();
        lat_tier_warp_reduce(t);
        if (lane == 0) s_wtier[warp] = t;
        __syncthreads();
        if (warp == 0) {
          t = lane < nwarps ? s_wtier[lane] : lat_tier_none();
          lat_tier_warp_reduce(t);
          if (lane == 0) s_ctier[r & 1] = t;
        }
        cluster.sync();
        t = lane < C ? *cluster.map_shared_rank(&s_ctier[r & 1], lane) : lat_tier_none();
        lat_tier_warp_reduce(t);
        // scoreBucket (plugin.go:262-318) with exact divisions, as the oracle
        const double rgT = __dsub_rn(t.mxT, t.mnT), rgP = __dsub_rn(t.mxP, t.mnP);
        const bool tok = rgT > 1e-9, pok = rgP > 1e-9;  // plugin.go:41
        double alpha = L.alpha, beta = L.beta;
        if (!tok && pok) {                               // plugin.go:275-279
          alpha = 0.0;
          beta = 1.0;
        } else if (!pok && tok) {
          alpha = 1.0;
          beta = 0.0;
        }
        const bool most = L.strategy_most && t.rank == 0;
        const double eT = tok ? __ddiv_rn(__dsub_rn(aT, t.mnT), rgT) : 0.5, eP = pok ? __ddiv_rn(__dsub_rn(aP, t.mnP), rgP) : 0.5;
        const double ec = __dadd_rn(__dmul_rn(alpha, eT), __dmul_rn(beta, eP));
        lat_w = lp.rank == t.rank ? go_int(most ? __dmul_rn(ec, 100.0) : __dmul_rn(__dsub_rn(1.0, ec), 100.0)) + 1 : 0;
      } else {
        // compositeScores (plugin.go:338-360): maxQ over the candidates from 0, the candidates' queue maximum
        const long long maxq = cur.mx0 > 0 ? cur.mx0 : 0;
        const long long q = __double_as_longlong(s_lat[(size_t)T + tid]);  // raw WaitingQueueSize
        const double rel = maxq > 0 ? __ddiv_rn(__ll2double_rn(maxq - q), __ll2double_rn(maxq)) : 1.0;
        lat_w = __double2ll_rz(round(__dmul_rn(100.0, __dadd_rn(__dadd_rn(s_lat[tid], __dmul_rn(L.wq, rel)), pt))));
      }
    }
    if constexpr (PROF) {
      // ---- Each run: its score in its profile order, its candidate, and this warp's winner (the run's picker, uniform) ----
      __shared__ InOrderBest s_pwarp[kMaxRuns][kInOrderWarps];
      __shared__ InOrderBest s_pcta[2][kMaxRuns];  // the CTA's winner per run of the last two requests (read cluster-wide)
      __shared__ InOrderPick s_pick[kMaxRuns];
      const int n_runs = pa->n_runs;
#pragma unroll 1
      for (int i = 0; i < n_runs; i++) {
        const InOrderRun& u = pa->run[i];
        long long mn0 = 0, mx0 = 0, mn1 = 0, mx1 = 0;  // (read at the request: a second run's min / max would not fit one ahead)
        if (u.minmax) {
          const long long* mm = u.minmax + (size_t)r * 4;
          mn0 = __ldg(mm);
          mx0 = __ldg(mm + 1);
          mn1 = __ldg(mm + 2);
          mx1 = __ldg(mm + 3);
        }
        double acc = 0.0;
        for (int s = 0; s < u.n_scorers; s++) {
          const int kind = u.kind[s];
          const double w = u.weight[s];
          double term;
          if (kind == 6) {
            term = __dmul_rn(tl, w);
          } else if (kind == 0 || kind == 4) {
            const bool queue = kind == 0;
            const long long mn = queue ? mn0 : mn1, mx = queue ? mx0 : mx1, qv = queue ? q0 : q1;
            term = mx == mn ? __dmul_rn(1.0, w) : __dmul_rn(clamp01(__ddiv_rn(__ll2double_rn(mx - qv), __ll2double_rn(mx - mn))), w);
          } else if (kind == 2) {
            term = prefix_term_direct(cur.c, cur.total, w);
          } else if (kind == 3) {
            term = u.lora_term[s][cur.cls];
          } else if (kind >= 16) {
            term = __dmul_rn(0.0, w);
          } else {
            term = s_term[(size_t)(u.term_base + s) * T + tid];
          }
          acc = __dadd_rn(acc, term);
        }
        const bool rnd = u.pick_mode != 0;
        const uint32_t areq = tie_areq(a.request_base + r, u.seed_lo);
        InOrderBest x = inorder_none();
        if ((cands >> i) & 1u) {
          const uint32_t pr = tie_prio(areq, m, u.seed_hi);
          if (rnd) {
            rbest_update(x.all, (double)pr, acc, m);
            if (u.pick_mode == 1 && acc > 0.0) rbest_update(x.pos, ares_key(pr, m, acc), acc, m);
          } else {
            best_update(x.b, acc, m, tie_mode, areq, u.seed_hi);
          }
        }
        if (rnd) inorder_warp_reduce<true>(x, tie_mode);
        else inorder_warp_reduce<false>(x, tie_mode);
        if (lane == 0) s_pwarp[i][warp] = x;
      }
      __syncthreads();
      // ---- The CTA's winner of each run (warp w reduces runs w, w + nwarps, ...), then one barrier.cluster for all runs ----
      for (int i = warp; i < n_runs; i += nwarps) {
        const bool rnd = pa->run[i].pick_mode != 0;
        InOrderBest x = lane < nwarps ? s_pwarp[i][lane] : inorder_none();
        if (rnd) inorder_warp_reduce<true>(x, tie_mode);
        else inorder_warp_reduce<false>(x, tie_mode);
        if (lane == 0) s_pcta[r & 1][i] = x;
      }
      cluster.sync();  // barrier.cluster: the CTA winners of request r, every run, are visible cluster-wide
      for (int i = warp; i < n_runs; i += nwarps) {
        const InOrderRun& u = pa->run[i];
        const bool rnd = u.pick_mode != 0;
        InOrderBest x = lane < C ? *cluster.map_shared_rank(&s_pcta[r & 1][i], lane) : inorder_none();
        InOrderPick p;
        if (rnd) {
          inorder_warp_reduce<true>(x, tie_mode);
          const RBest& wb = x.pos.m >= 0 ? x.pos : x.all;  // no positive score: the random picker (weightedrandom/picker.go:113-116)
          p = InOrderPick{wb.score, wb.m, wb.n};
        } else {
          inorder_warp_reduce<false>(x, tie_mode);
          p = InOrderPick{x.b.score, x.b.m, x.b.cnt};
        }
        if (lane == 0) {
          s_pick[i] = p;
          if (cluster.block_rank() == 0) {
            u.pick[r] = p.m;
            u.pick_score[r] = p.m >= 0 ? p.score : 0.0;
            u.tie_count[r] = p.cnt;
          }
        }
      }
      __syncthreads();  // every run's pick of request r is in s_pick
      // ---- PreRequest, when the primary run picked (no PreRequest for a failed schedule): requests += 1 and tokens += tokens[r]
      // on every run's pick (producer.go:106-119), PrefixCacheMatchInfo at each pick before the request's Adds
      // (plugin.go:199-204), then indexer.Add at the primary pick and at the prefill pick (plugin.go:177-197) ----
      const int p0 = s_pick[pa->primary].m;
      const int p1 = pa->prefill >= 0 ? s_pick[pa->prefill].m : -1;
      bool moved = false;
#pragma unroll 1
      for (int i = 0; i < n_runs; i++) {
        const int pk = p0 >= 0 ? s_pick[i].m : -1;
        if (pk == m) {
          tok += cur.tokens;
          req += 1;
          moved = true;
        }
        uint16_t* pm = pa->run[i].pick_match;
        if (pm && (pk >= 0 ? pk == m : m == 0)) pm[r] = pk >= 0 ? (uint16_t)cur.c : (uint16_t)0;
      }
      if (moved) tl = token_load_score(tok, a.token_threshold);
      if constexpr (IDX) {
        const int rank = (int)cluster.block_rank();
        const bool own0 = p0 >= 0 && p0 / T == rank, own1 = p1 >= 0 && p1 / T == rank && p1 != p0;  // CTA-uniform
        if (own0 || own1) {
          __shared__ int32_t s_adds[2];
          if (tid == 0) {  // (read inside the program's first parallel section, behind its barrier)
            s_adds[0] = p0;
            s_adds[1] = p1;
          }
          CommitArgs ca{};
          ca.R = 1;
          ca.pick = &s_adds[0];
          ca.hashes = ix.hashes + (size_t)r * ix.stride;
          ca.n_hashes = a.total + r;
          ca.stride = ix.stride;
          ca.cap_req = ix.cap_req;
          ca.n_picks = p1 >= 0 ? 2 : 1;
          ca.more_picks[0] = &s_adds[1];
          CommitSmem* sm = reinterpret_cast<CommitSmem*>(s_term + (size_t)slots * T);
          if (own0) {  // both Adds when both picks are this endpoint, primary first
            IndexProgram<DevX> prog(dx, ix.tv, ix.lv, sm, (uint32_t)p0);
            prog.commit(ca);
          }
          if (own1) {
            IndexProgram<DevX> prog(dx, ix.tv, ix.lv, sm, (uint32_t)p1);
            prog.commit(ca);
          }
        }
        cluster.sync();  // request r's Adds are visible to every CTA's probes of request r + 1
      }
      cands = cands_nxt;
      cur = nxt;
      continue;
    }
    // ---- Score (scheduler_profile.go:151-174): profile order from 0.0, the operations of score_matrix_kernel ----
    double acc = 0.0;
    for (int s = 0; s < a.n_scorers; s++) {
      const int kind = a.kind[s];
      const double w = a.weight[s];
      double term;
      if (kind == 6) {
        term = __dmul_rn(tl, w);                                                       // the moving term
      } else if (kind == 0 || kind == 4) {
        const bool queue = kind == 0;
        const long long mn = queue ? cur.mn0 : cur.mn1, mx = queue ? cur.mx0 : cur.mx1, qv = queue ? q0 : q1;
        term = mx == mn ? __dmul_rn(1.0, w)                                            // queue.go:95-98
                        : __dmul_rn(clamp01(__ddiv_rn(__ll2double_rn(mx - qv), __ll2double_rn(mx - mn))), w);
      } else if (kind == 2) {
        term = prefix_term_direct(cur.c, cur.total, w);                                // prefix/plugin.go:108-110
      } else if (kind == 3) {
        term = a.lora_term[s][cur.cls];
      } else if (LAT && kind == 5) {
        term = __dmul_rn(clamp01(__ddiv_rn(__ll2double_rn(lat_w), 100.0)), w);       // float64(w)/100, plugin.go:301-306
      } else if (kind >= 16) {
        term = __dmul_rn(0.0, w);                                                      // pair columns absent
      } else {
        term = s_term[(size_t)s * T + tid];                                            // kv-cache, endpoint columns
      }
      acc = __dadd_rn(acc, term);
    }
    // ---- Pick: this thread's candidate, then warp, CTA and cluster merges (all commutative and associative) ----
    const uint32_t areq = tie_areq(a.request_base + r, a.seed_lo);
    InOrderBest x = inorder_none();
    if (cur.cand) {
      const uint32_t pr = tie_prio(areq, m, a.seed_hi);
      if (RND) {
        rbest_update(x.all, (double)pr, acc, m);
        if (a.pick_mode == 1 && acc > 0.0) rbest_update(x.pos, ares_key(pr, m, acc), acc, m);
      } else {
        best_update(x.b, acc, m, tie_mode, areq, a.seed_hi);
      }
    }
    inorder_warp_reduce<RND>(x, tie_mode);
    if (lane == 0) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
      x = lane < nwarps ? s_warp[lane] : inorder_none();
      inorder_warp_reduce<RND>(x, tie_mode);
      if (lane == 0) s_cta[r & 1] = x;
    }
    cluster.sync();  // barrier.cluster: the CTA winners of request r are visible cluster-wide
    x = lane < C ? *cluster.map_shared_rank(&s_cta[r & 1], lane) : inorder_none();
    inorder_warp_reduce<RND>(x, tie_mode);
    int pick;
    double score;
    int cnt;
    if (RND) {
      const RBest& wb = x.pos.m >= 0 ? x.pos : x.all;  // no positive score: the random picker (weightedrandom/picker.go:113-116)
      pick = wb.m;
      score = wb.score;
      cnt = wb.n;
    } else {
      pick = x.b.m;
      score = x.b.score;
      cnt = x.b.cnt;
    }
    // ---- PreRequest: requests += 1, tokens += tokens[r] on the pick (producer.go:101-120) ----
    if (pick == m) {
      tok += cur.tokens;
      req += 1;
      tl = token_load_score(tok, a.token_threshold);
    }
    if (m == 0) {
      a.pick[r] = pick;
      a.pick_score[r] = pick >= 0 ? score : 0.0;
      a.tie_count[r] = cnt;
    }
    if constexpr (LAT) {
      // ---- PreRequest: the request joins its target's running-request queue (requestcontrol_hooks.go:73-86), refused for an
      // empty key, a negative tpot or a pair already live (running_request_tpot_slo_queue.go:127-132) ----
      uint8_t added = 0;
      if (pick == m && lcur.key != 0ull) {
        const RunDev* d = lt.run;
        const double tp = lcur.tpot;
        if (tp != tp) {
          atomicOr(&d->ctr->err, kRunErrInvalid);  // (host arrays are validated before the launch)
        } else if (!(tp < 0.0)) {
          const RunDev dv = *d;
          bool created = false;
          const long long h = run_find_or_create(dv, lcur.key, m, &created);
          if (h < 0) atomicOr(&d->ctr->err, kRunErrCapacity);
          if (created) {
            const unsigned long long v = tp == 0.0 ? 0ull : (unsigned long long)__double_as_longlong(tp);  // -0.0 as +0.0
            dv.tpot[h] = v;
            dv.owner[h] = ((unsigned long long)d->ctr->gen << 32) | (unsigned)r;  // older than any later call's bid: its add is refused
            atomicAdd(&d->ctr->live, 1ull);
            run_cnt += 1;
            if (v < run_min) {
              run_min = v;
              run_mincnt = 1;
            } else if (v == run_min) {
              run_mincnt += 1;
            }
            lim = lat_lim(__longlong_as_double((long long)run_min), lt.lat.buffer);
            idle = lat_idle(run_cnt);
            added = 1;
          }
        }
      }
      if (lt.added_out && (pick >= 0 ? pick == m : m == 0)) lt.added_out[r] = added;
      lcur = lnxt;
    }
    if constexpr (IDX) {
      // PrefixCacheMatchInfo at the target (plugin.go:199-204), before the request's own Add
      if (ix.pick_match && (pick >= 0 ? pick == m : m == 0)) ix.pick_match[r] = pick >= 0 ? (uint16_t)cur.c : (uint16_t)0;
      // indexer.Add(hashes[r], pick) (plugin.go:169-197) by the CTA that owns the pick: CTA-uniform, as IndexProgram needs
      if (pick >= 0 && pick / T == (int)cluster.block_rank()) {
        __shared__ int32_t s_pick;
        if (tid == 0) s_pick = pick;  // (read inside the program's first parallel section, behind its barrier)
        CommitArgs ca{};
        ca.R = 1;
        ca.pick = &s_pick;
        ca.hashes = ix.hashes + (size_t)r * ix.stride;
        ca.n_hashes = a.total + r;
        ca.stride = ix.stride;
        ca.cap_req = ix.cap_req;
        ca.n_picks = 1;
        CommitSmem* sm = reinterpret_cast<CommitSmem*>(s_term + (size_t)kTermSlots * T);
        IndexProgram<DevX> prog(dx, ix.tv, ix.lv, sm, (uint32_t)pick);
        prog.commit(ca);
      }
      cluster.sync();  // request r's Add is visible to every CTA's probes of request r + 1
    }
    cur = nxt;
  }
  if (m < a.Mpad) {
    a.inflight_tok[m] = tok;
    a.inflight_req[m] = req;
  }
  if constexpr (LAT) {
    if (lt.request_key && m < lt.n_ep) {  // (running_finalize_kernel publishes the view and advances the generation)
      const RunDev* d = lt.run;
      d->count[m] = run_cnt;
      d->min_bits[m] = run_min;
      d->min_cnt[m] = run_mincnt;
    }
  }
  cluster.sync();  // no CTA leaves while another may still read its winners
}

template <bool RND>
__global__ void __launch_bounds__(kInOrderMaxThreads, 1) inorder_pick_kernel(const __grid_constant__ InOrderArgs a) {
  inorder_walk<RND, false, false>(a, InOrderIndexArgs{}, InOrderLatArgs{});
}

template <bool RND>
__global__ void __launch_bounds__(kCommitThreads, 1) inorder_index_kernel(const __grid_constant__ InOrderArgs a,
                                                                          const __grid_constant__ InOrderIndexArgs ix) {
  inorder_walk<RND, true, false>(a, ix, InOrderLatArgs{});
}

template <bool RND>
__global__ void __launch_bounds__(kInOrderMaxThreads, 1) inorder_pick_lat_kernel(const __grid_constant__ InOrderArgs a,
                                                                                 const __grid_constant__ InOrderLatArgs lt) {
  inorder_walk<RND, false, true>(a, InOrderIndexArgs{}, lt);
}

template <bool RND>
__global__ void __launch_bounds__(kCommitThreads, 1) inorder_index_lat_kernel(const __grid_constant__ InOrderArgs a,
                                                                              const __grid_constant__ InOrderIndexArgs ix,
                                                                              const __grid_constant__ InOrderLatArgs lt) {
  inorder_walk<RND, true, true>(a, ix, lt);
}

int launch_inorder_minmax(const InOrderArgs& a, cudaStream_t s, int sm_count) {
  if (a.R <= 0) return 0;
  int blocks = (a.R + 7) / 8;
  if (blocks > sm_count * 8) blocks = sm_count * 8;
  inorder_minmax_kernel<<<blocks, 256, 0, s>>>(a);
  return 1;
}

// The cluster: C CTAs of T = Mpad / C threads, one endpoint per thread.  Up to 16 CTAs when the device grants the non-portable
// size, else 8 (then max_endpoints 8192 does not fit); fewer at small Mpad, so that a CTA keeps at least 256 endpoints (each
// CTA is one more arrival at every barrier).  The dynamic shared memory (8 bytes per scorer per thread, at most 32 KiB) needs no
// opt-in; the latency form's (8 more bytes per static tile slot, at most 56 KiB) is opted in by cluster_size.
template <bool RND>
static cudaLaunchConfig_t pick_config(int Mpad, int C, cudaStream_t s, cudaLaunchAttribute* at, bool lat = false) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(C);
  cfg.blockDim = dim3(Mpad / C);
  cfg.dynamicSmemBytes = (size_t)(kMaxSteps + (lat ? kLatStatic : 0)) * 8 * (Mpad / C);
  cfg.stream = s;
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = C;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  return cfg;
}

template <bool RND, bool LAT>
static int cluster_size(int Mpad) {
  auto kernel = LAT ? (const void*)inorder_pick_lat_kernel<RND> : (const void*)inorder_pick_kernel<RND>;
  cudaError_t c = cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  if (c == cudaSuccess && LAT)
    c = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (kMaxSteps + kLatStatic) * 8 * kInOrderMaxThreads);
  if (c != cudaSuccess) return -(int)c;
  for (int cmax = 16; cmax >= 8; cmax /= 2) {
    int C = Mpad / 256;
    if (C < 1) C = 1;
    if (C > cmax) C = cmax;
    if (Mpad / C > kInOrderMaxThreads) continue;
    cudaLaunchAttribute at[1];
    const cudaLaunchConfig_t cfg = pick_config<RND>(Mpad, C, nullptr, at, LAT);
    int clusters = 0;
    c = cudaOccupancyMaxActiveClusters(&clusters, kernel, &cfg);
    if (c == cudaSuccess && clusters >= 1) return C;
    cudaGetLastError();
  }
  return 0;
}

int inorder_cluster_size(int Mpad, bool lat) {
  const int a = lat ? cluster_size<false, true>(Mpad) : cluster_size<false, false>(Mpad);
  if (a <= 0) return a;
  const int b = lat ? cluster_size<true, true>(Mpad) : cluster_size<true, false>(Mpad);
  return b <= 0 ? b : (a < b ? a : b);
}

int launch_inorder_pick(const InOrderArgs& a, int C, cudaStream_t s, const InOrderLatArgs* lt) {
  if (a.R <= 0) return 0;
  cudaLaunchAttribute at[1];
  if (lt) {
    const cudaLaunchConfig_t cfg = pick_config<true>(a.Mpad, C, s, at, true);
    return launched_one(a.pick_mode != 0 ? cudaLaunchKernelEx(&cfg, inorder_pick_lat_kernel<true>, a, *lt)
                                         : cudaLaunchKernelEx(&cfg, inorder_pick_lat_kernel<false>, a, *lt));
  }
  if (a.pick_mode != 0) {
    const cudaLaunchConfig_t cfg = pick_config<true>(a.Mpad, C, s, at);
    return launched_one(cudaLaunchKernelEx(&cfg, inorder_pick_kernel<true>, a));
  }
  const cudaLaunchConfig_t cfg = pick_config<false>(a.Mpad, C, s, at);
  return launched_one(cudaLaunchKernelEx(&cfg, inorder_pick_kernel<false>, a));
}

// The index form: C CTAs of kCommitThreads threads (IndexProgram's CTA), thread t of CTA c owning endpoint c * 512 + t (threads
// past Mpad idle), so C = Mpad / 512 up to 16 (one CTA below 512 endpoints).  Dynamic shared memory: the terms of 512 threads,
// then the CommitSmem of the program (136 KiB, plus 13 KiB of static shared memory: one CTA per SM).  The latency form puts the
// static tile slots (24 KiB) between the two.
static size_t index_smem(bool lat) { return (size_t)(kMaxSteps + (lat ? kLatStatic : 0)) * 8 * kCommitThreads + sizeof(CommitSmem); }

static cudaLaunchConfig_t index_config(int C, cudaStream_t s, cudaLaunchAttribute* at, bool lat = false) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(C);
  cfg.blockDim = dim3(kCommitThreads);
  cfg.dynamicSmemBytes = index_smem(lat);
  cfg.stream = s;
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = C;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  return cfg;
}

template <bool RND, bool LAT>
static int index_cluster_size(int Mpad) {
  auto kernel = LAT ? (const void*)inorder_index_lat_kernel<RND> : (const void*)inorder_index_kernel<RND>;
  cudaError_t c = cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  if (c == cudaSuccess) c = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)index_smem(LAT));
  if (c != cudaSuccess) return -(int)c;
  const int C = Mpad <= kCommitThreads ? 1 : (Mpad + kCommitThreads - 1) / kCommitThreads;
  if (C > 16) return 0;
  cudaLaunchAttribute at[1];
  const cudaLaunchConfig_t cfg = index_config(C, nullptr, at, LAT);
  int clusters = 0;
  c = cudaOccupancyMaxActiveClusters(&clusters, kernel, &cfg);
  if (c == cudaSuccess && clusters >= 1) return C;
  cudaGetLastError();
  return 0;
}

int inorder_index_cluster_size(int Mpad, bool lat) {
  const int a = lat ? index_cluster_size<false, true>(Mpad) : index_cluster_size<false, false>(Mpad);
  if (a <= 0) return a;
  const int b = lat ? index_cluster_size<true, true>(Mpad) : index_cluster_size<true, false>(Mpad);
  return b <= 0 ? b : a;  // (both forms have the same shape)
}

int launch_inorder_index(const InOrderArgs& a, const InOrderIndexArgs& ix, int C, cudaStream_t s, const InOrderLatArgs* lt) {
  if (a.R <= 0) return 0;
  cudaLaunchAttribute at[1];
  if (lt) {
    const cudaLaunchConfig_t cfg = index_config(C, s, at, true);
    return launched_one(a.pick_mode != 0 ? cudaLaunchKernelEx(&cfg, inorder_index_lat_kernel<true>, a, ix, *lt)
                                         : cudaLaunchKernelEx(&cfg, inorder_index_lat_kernel<false>, a, ix, *lt));
  }
  if (a.pick_mode != 0) {
    const cudaLaunchConfig_t cfg = index_config(C, s, at);
    return launched_one(cudaLaunchKernelEx(&cfg, inorder_index_kernel<true>, a, ix));
  }
  const cudaLaunchConfig_t cfg = index_config(C, s, at);
  return launched_one(cudaLaunchKernelEx(&cfg, inorder_index_kernel<false>, a, ix));
}

template <bool IDX>
__global__ void __launch_bounds__(kInOrderMaxThreads, 1) inorder_profiles_walk_kernel(const __grid_constant__ InOrderArgs a,
                                                                                      const __grid_constant__ InOrderIndexArgs ix,
                                                                                      const __grid_constant__ InOrderProfArgs p) {
  inorder_walk<false, IDX, false, true>(a, ix, InOrderLatArgs{}, &p);
}

// The profiles walk: the cluster shapes of the single-profile walks (the in-flight form's CTAs of Mpad / C threads, the index
// form's of kCommitThreads), with Σ n_scorers term slots per thread, then (index form) the CommitSmem.  The kernels are opted in to
// the device's whole shared memory less their static part; a call whose runs need more is refused before any launch.
size_t inorder_profiles_smem(int Mpad, int C, bool index, int slots) {
  return index ? (size_t)slots * 8 * kCommitThreads + sizeof(CommitSmem) : (size_t)slots * 8 * (Mpad / C);
}

static cudaLaunchConfig_t profiles_config(int Mpad, int C, bool index, size_t smem, cudaStream_t s, cudaLaunchAttribute* at) {
  cudaLaunchConfig_t cfg = index ? index_config(C, s, at) : pick_config<false>(Mpad, C, s, at);
  cfg.dynamicSmemBytes = smem;
  return cfg;
}

// > 0: CTAs per cluster (and *smem_max the dynamic shared memory the kernel may use); 0: no cluster shape fits; -(cudaError_t)
int inorder_profiles_cluster_size(int Mpad, bool index, size_t* smem_max) {
  const void* kernel = index ? (const void*)inorder_profiles_walk_kernel<true> : (const void*)inorder_profiles_walk_kernel<false>;
  int dev = 0, optin = 0;
  cudaFuncAttributes fa{};
  cudaError_t c = cudaGetDevice(&dev);
  if (c == cudaSuccess) c = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (c == cudaSuccess) c = cudaFuncGetAttributes(&fa, kernel);
  if (c == cudaSuccess) c = cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  const int dyn = optin - (int)fa.sharedSizeBytes;
  if (c == cudaSuccess) c = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn);
  if (c != cudaSuccess) return -(int)c;
  *smem_max = (size_t)dyn;
  // the largest shape first, with the shared memory of the smallest call (one run of one scorer): a call past it is refused
  for (int cmax = 16; cmax >= (index ? 16 : 8); cmax /= 2) {
    int C;
    if (index) {
      C = Mpad <= kCommitThreads ? 1 : (Mpad + kCommitThreads - 1) / kCommitThreads;
    } else {
      C = Mpad / 256;
      if (C < 1) C = 1;
      if (C > cmax) C = cmax;
      if (Mpad / C > kInOrderMaxThreads) continue;
    }
    if (C > 16) return 0;
    cudaLaunchAttribute at[1];
    const cudaLaunchConfig_t cfg = profiles_config(Mpad, C, index, inorder_profiles_smem(Mpad, C, index, 1), nullptr, at);
    int clusters = 0;
    c = cudaOccupancyMaxActiveClusters(&clusters, kernel, &cfg);
    if (c == cudaSuccess && clusters >= 1) return C;
    cudaGetLastError();
  }
  return 0;
}

int launch_inorder_profiles(const InOrderArgs& a, const InOrderIndexArgs* ix, const InOrderProfArgs& p, int C, int slots, cudaStream_t s) {
  if (a.R <= 0) return 0;
  cudaLaunchAttribute at[1];
  const cudaLaunchConfig_t cfg = profiles_config(a.Mpad, C, ix != nullptr, inorder_profiles_smem(a.Mpad, C, ix != nullptr, slots), s, at);
  return launched_one(ix ? cudaLaunchKernelEx(&cfg, inorder_profiles_walk_kernel<true>, a, *ix, p)
                         : cudaLaunchKernelEx(&cfg, inorder_profiles_walk_kernel<false>, a, InOrderIndexArgs{}, p));
}

}  // namespace eppscore
