// pick_sparse.cu — the exact sparse fast path of Score+Pick (unmasked batches, E/P/L steps).
//
// For a request r with adapter a, the weighted score of endpoint m is
//     S(r,m) = steps(base terms[m], prefix term(c(r,m)), lora term(class(a,m)))   (scheduler_profile.go:155-168)
// and c(r,m) — the matched prefix blocks (approximateprefix/plugin.go:219-235) — is ZERO for all but the
// few endpoints that appear in the rows of the request's matched block hashes.  With c = 0 the score is
// G[a][m], which depends only on the snapshot and the adapter; prepare_adapters_kernel has already
// reduced it to (gmax, garg, gcnt, tie mask) per adapter.  Because the prefix weight is >= 0 and float64
// addition is monotone, S(r,e) >= G[a][e] for every "exception" e (c > 0), hence
//     max_m S(r,m) = max( gmax[a], max_e S(r,e) )
// and the arg-max set follows from three cases (T = max_e S(r,e), xg = #{e : G[a][e] == gmax}):
//     T > gmax : only exceptions attain it;
//     T < gmax : the precomputed arg-max set, untouched by any exception (xg == 0 by monotonicity);
//     T == gmax: (precomputed set minus its xg exception members) ∪ {e : S(r,e) == gmax}.
// So a request costs O(matched blocks + exceptions) instead of O(M) — bit-identical picks, scores and
// tie counts (tests compare against the oracle and against the generic kernel).
//
// Work split: a group of G = row_words/4 lanes serves one request, so a warp serves 32/G requests at once.  The table is
// the device-resident index of prefix_table.cuh: a hit brings its endpoint set along in the 32-byte slot (up to 10 members
// inline), so matchLongestPrefix is: probe -> each hit's lane adds 1 to its members' entries of a small per-request hash
// table in shared memory (endpoint -> matched blocks, 64 entries) -> the entries are the exceptions.  A request whose
// prefix is cached on more endpoints than the table holds (a system prompt cached everywhere) is DEFERRED: the kernel
// writes pick = kPickDeferred and the full-matrix kernel (score_matrix.cu), launched right after with a filter, scores
// it exactly — dense cases are what that kernel is for.
#include "device_common.cuh"
#include "prefix_table.cuh"

namespace eppscore {

constexpr int kSparseWarps = 8;
#ifndef EPP_SPARSE_MINBLOCKS
#define EPP_SPARSE_MINBLOCKS 4  // CTAs per SM the register allocation aims at (64 registers per thread)
#endif

// Score of an exception endpoint with the scorer sequence known at compile time (SEQ packs kind+1 per step,
// 4 bits each; SEQ == 0 selects the runtime-generic eval_steps).  The prefix term comes from the engine-wide
// table lut2d[total][c] = clamp(c/total)*w (built once on the host: one IEEE divide, one multiply per entry).
template <uint32_t SEQ>
__device__ __forceinline__ double eval_exception(const ScoreArgs& a, int m, int c, int total, int cls) {
  if (SEQ == 0) return eval_steps(a.plan, a.term, m, c, total, cls);
  double acc = 0.0;
#pragma unroll
  for (int s = 0; s < 8; s++) {
    const int kind = (int)((SEQ >> (4 * s)) & 15u) - 1;
    if (kind < 0) break;
    double t;
    if (kind == STEP_EP_TERM) {
      t = __ldg(a.term[a.plan.arg[s]] + m);
    } else if (kind == STEP_PREFIX) {
      t = (a.prefix_lut2d && total <= kLutMax) ? __ldg(a.prefix_lut2d + total * (kLutMax + 1) + c)
                                               : prefix_term_direct(c, total, a.plan.weight[s]);
    } else {  // STEP_LORA
      const double* lt = a.plan.lora_term[s];
      t = cls == 3 ? lt[3] : (cls == 2 ? lt[2] : (cls == 1 ? lt[1] : lt[0]));
    }
    acc = __dadd_rn(acc, t);
  }
  return acc;
}

constexpr int kExcSlots = 64;   // per-request exception table (power of two)
constexpr int kExcMax = 44;     // more distinct endpoints than this: defer the request to the full-matrix kernel

struct ExcTable {
  uint32_t tab[kExcSlots];      // (endpoint + 1) << 16 | matched blocks; 0 = empty
  uint8_t list[kExcSlots];      // slots in insertion order
  uint32_t n;                   // entries of list
  uint32_t overflow;
  uint32_t pad[2];
};

__device__ __forceinline__ uint32_t exc_home(uint32_t m) { return (m * 0x9E3779B1u) >> 26; }  // 6 bits

// res[server]++ (approximateprefix/plugin.go:229-231)
__device__ __forceinline__ void exc_add(ExcTable* t, uint32_t m, uint32_t len = 1u) {
  const uint32_t key = (m + 1u) << 16;
  uint32_t j = exc_home(m);
  for (int probes = 0; probes < kExcSlots; probes++, j = (j + 1) & (kExcSlots - 1)) {
    uint32_t cur = *reinterpret_cast<volatile uint32_t*>(&t->tab[j]);
    if (cur == 0) {
      cur = atomicCAS(&t->tab[j], 0u, key | len);
      if (cur == 0) {
        const uint32_t pos = atomicAdd(&t->n, 1u);
        if (pos < (uint32_t)kExcSlots) t->list[pos] = (uint8_t)j;
        if (pos >= (uint32_t)kExcMax) t->overflow = 1u;
        return;
      }
    }
    if ((cur >> 16) == m + 1u) {
      atomicAdd(&t->tab[j], len);
      return;
    }
  }
  t->overflow = 1u;
}
__device__ __forceinline__ bool exc_has(const ExcTable* t, uint32_t m) {
  uint32_t j = exc_home(m);
  for (int probes = 0; probes < kExcSlots; probes++, j = (j + 1) & (kExcSlots - 1)) {
    const uint32_t cur = t->tab[j];
    if (cur == 0) return false;
    if ((cur >> 16) == m + 1u) return true;
  }
  return false;
}
static __device__ __noinline__ void exc_add_row(ExcTable* t, const uint32_t* row, int nw) {
  for (int w0 = 0; w0 < nw && !*reinterpret_cast<volatile uint32_t*>(&t->overflow); w0++) {
    uint32_t x = __ldg(row + w0);
    while (x) {
      const int k = __ffs(x) - 1;
      x &= x - 1;
      exc_add(t, (uint32_t)(w0 * 32 + k));
    }
  }
}
// member k of an inline set held as {w = ep0 | ep1 << 16, hi = ep2..ep9}
__device__ __forceinline__ uint32_t slot_member(uint32_t w, const uint4& hi, uint32_t k) {
  const uint32_t x = k < 2 ? w : (k < 4 ? hi.x : (k < 6 ? hi.y : (k < 8 ? hi.z : hi.w)));
  return (k & 1) ? (x >> 16) : (x & 0xFFFFu);
}
// order-independent form of best_update (the exceptions of a lane arrive in table order, not ascending)
__device__ __forceinline__ void best_update_any(Best& b, double s, int m, int tie_mode, uint32_t areq, uint32_t seed_hi) {
  const bool first = b.m < 0;
  const bool gt = first || s > b.score;
  const bool eq = !first && s == b.score;
  if (tie_mode) {
    if (gt || eq) {
      const uint32_t pr = tie_prio(areq, m, seed_hi);
      if (gt || pr > b.prio || (pr == b.prio && m < b.m)) {
        b.prio = pr;
        b.m = m;
      }
    }
  } else {
    b.m = gt ? m : ((eq && m < b.m) ? m : b.m);
  }
  b.score = gt ? s : b.score;
  b.cnt = gt ? 1 : b.cnt + (eq ? 1 : 0);
}

template <int J, uint32_t SEQ>
__global__ void __launch_bounds__(kSparseWarps * 32, EPP_SPARSE_MINBLOCKS) pick_sparse_kernel(const __grid_constant__ ScoreArgs a) {
  const int LOG_EPL = a.geo.log_epl;
  constexpr int RW = J * 32;                       // words per PERMUTED bit row (LoRA class planes, tie masks)
  constexpr int G = (RW / 4 < 32) ? RW / 4 : 32;   // lanes per request
  constexpr int PW = RW / G;                       // permuted words per lane
  constexpr int RPW = 32 / G;                      // requests per warp
  __shared__ ExcTable s_exc[kSparseWarps * RPW];
  const Plan& plan = a.plan;
  const int M = a.geo.M;
  const int NW = a.geo.Mpad >> 5;                  // words of a natural-order overflow row
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int gi = lane / G, gl = lane % G;
  ExcTable* exc = &s_exc[warp * RPW + gi];

  {  // zero the tables once; afterwards each request re-zeroes exactly the entries it used
    uint32_t* z = reinterpret_cast<uint32_t*>(s_exc);
    for (int i = threadIdx.x; i < (int)(sizeof(s_exc) / 4); i += blockDim.x) z[i] = 0;
  }
  __syncthreads();

  int prefix_step = -1;
  for (int s = 0; s < plan.n_steps; s++)
    if (plan.kind[s] == STEP_PREFIX) prefix_step = s;
  const int tie_mode = plan.tie_mode;
  const bool have_table = a.table != nullptr && a.hashes != nullptr && prefix_step >= 0;
  const TSlot* slots = nullptr;
  uint64_t slot_mask = 0;
  const uint32_t* ovf_rows = nullptr;
  if (have_table) {
    slots = a.table->slots;
    slot_mask = a.table->mask;
    ovf_rows = a.table->ovf_rows;
  }

  pdl_wait();               // the hashes come from the previous kernel of the stream (everything above overlaps its tail)
  pdl_launch_dependents();
  const int wstride = gridDim.x * kSparseWarps * RPW;
  for (int rbase = (blockIdx.x * kSparseWarps + warp) * RPW; rbase < a.R; rbase += wstride) {
    const int r = rbase + gi;
    const bool valid = r < a.R;
    const int n = (valid && a.hashes) ? (int)a.n_hashes[r] : 0;
    int ad = (valid && a.adapter_id) ? a.adapter_id[r] : -1;
    if (ad < 0 || ad >= a.A) ad = a.A;
    const AdapterSummary sm = a.summ[ad];  // issued early: only consumed after the probe phase

    // ---------------- matchLongestPrefix: probe U*G hashes per round, stop at the first global miss ----------------
    uint32_t ref_raw = 0, ref_w = 0;           // the request's first hit: raw cnt word and members (see below)
    uint4 ref_hi = make_uint4(0, 0, 0, 0);
    bool use_table = false;                    // uniform within the request's lane group
    int n_same = 0;                            // matched blocks so far, all carrying the reference set
    if (have_table) {
      // a request the hashing kernel resolved (ProbeRec) skips the probe: it takes part in the rounds of the other requests of
      // its warp without a hit (no table, no count), and takes its count and set from the record afterwards
      // (only the count is held across the probe rounds: the set is loaded after them, which keeps the registers as they were)
      const uint32_t rec_n = (a.probe && valid) ? __ldg(&a.probe[r].n) : kProbeUnresolved;
      const bool resolved = rec_n != kProbeUnresolved;  // (uniform in the request's lane group)
      constexpr int U = 4;            // hashes probed per lane per round (independent loads in flight)
      bool stop = n == 0 || resolved;
      int c0 = 0;
      while (__any_sync(0xffffffffu, !stop)) {
        uint64_t h[U], idx[U];
        uint4 lo[U];   // {key.lo, key.hi, cnt, ep0 | ep1 << 16}
        bool act[U], hit[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
          const int i = c0 + u * G + gl;
          act[u] = !stop && i < n;
          h[u] = act[u] ? a.hashes[(size_t)r * a.hash_stride + i] : 0ULL;
          idx[u] = h[u] & slot_mask;
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
          lo[u] = make_uint4(0u, 0u, kCntFree, 0u);
          if (act[u]) lo[u] = ldg16(&slots[idx[u]]);
        }
#pragma unroll
        for (int u = 0; u < U; u++) hit[u] = act[u] && table_find(slots, slot_mask, h[u], idx[u], lo[u]);
        int nh_total = 0;   // blocks matched in this round before the first global miss
        bool open = !stop;
#pragma unroll
        for (int u = 0; u < U; u++) {
          const uint32_t miss = __ballot_sync(0xffffffffu, !hit[u]);
          const uint32_t gmiss = (G == 32) ? miss : ((miss >> (gi * G)) & ((1u << G) - 1u));
          if (open) {
            const int nh_u = gmiss ? (__ffs(gmiss) - 1) : G;
            nh_total += nh_u;
            if (nh_u < G) open = false;
          }
        }
        // every counted hit adds 1 to its members' entries: the members beyond the first two sit in the second half of
        // the slot (same 32-byte sector, already in L1); all those loads are issued before the first use
        uint4 hi[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
          hit[u] = hit[u] && (u * G + gl) < nh_total;
          hi[u] = make_uint4(0, 0, 0, 0);
          if (hit[u] && !(lo[u].z & kCntRow) && (lo[u].z & kCntMask) > 2u)
            hi[u] = ldg16(reinterpret_cast<const uint4*>(&slots[idx[u]]) + 1);
        }
        // The common case: every matched block of the request is cached on the SAME endpoints (a prefix is cached as a whole),
        // i.e. all hits carry the same inline set as the request's first hit.  Then the exceptions are that set's members,
        // each with the number of matched blocks — no table needed.  The first hit that differs switches the request to the
        // table: the reference set is entered with the count so far, every later hit adds 1 to its own members.
        if (c0 == 0) {  // the first hit of the request: lane 0 of the group, sub-round 0 (a resolved request takes its own below)
          ref_raw = __shfl_sync(0xffffffffu, hit[0] ? lo[0].z : 0u, gi * G);
          ref_w = __shfl_sync(0xffffffffu, lo[0].w, gi * G);
          ref_hi.x = __shfl_sync(0xffffffffu, hi[0].x, gi * G);
          ref_hi.y = __shfl_sync(0xffffffffu, hi[0].y, gi * G);
          ref_hi.z = __shfl_sync(0xffffffffu, hi[0].z, gi * G);
          ref_hi.w = __shfl_sync(0xffffffffu, hi[0].w, gi * G);
          if (ref_raw & kCntRow) use_table = true;               // a bitset row: always through the table
        }
        bool differs = false;
#pragma unroll
        for (int u = 0; u < U; u++) {
          if (!__any_sync(0xffffffffu, hit[u])) continue;        // (warp-uniform) no hit in this sub-round
          if (hit[u]) differs |= lo[u].z != ref_raw || !same_inline_set(ref_w, ref_hi, lo[u].w, hi[u]);
        }
        {
          const uint32_t db = __ballot_sync(0xffffffffu, differs);
          const uint32_t gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (gi * G));
          if (!use_table && (db & gmask)) {                      // (uniform within the request's lane group)
            use_table = true;
            if (n_same > 0 && !(ref_raw & kCntRow))
              for (uint32_t k = gl; k < (ref_raw & kCntMask); k += G) exc_add(exc, slot_member(ref_w, ref_hi, k), (uint32_t)n_same);
          }
        }
        if (!use_table) n_same += nh_total;
        if (__any_sync(0xffffffffu, use_table)) {                // (warp-uniform) some request of this warp needs its table
#pragma unroll
          for (int u = 0; u < U; u++) {
            if (!__any_sync(0xffffffffu, hit[u] && use_table)) continue;
            if (hit[u] && use_table) {
              const uint32_t c = lo[u].z & kCntMask;
              if (!(lo[u].z & kCntRow)) {
                const uint32_t cc = c < (uint32_t)kInlineEps ? c : (uint32_t)kInlineEps;
#pragma unroll 1
                for (uint32_t k = 0; k < cc; k++) exc_add(exc, slot_member(lo[u].w, hi[u], k));
              } else {                                           // a set of more than 10: one bitset row, natural order
                exc_add_row(exc, ovf_rows + (size_t)lo[u].w * NW, NW);
              }
            }
          }
        }
        c0 += U * G;
        if (nh_total < U * G || c0 >= n) stop = true;
      }
      if (resolved) {
        const uint2 set = __ldg(reinterpret_cast<const uint2*>(&a.probe[r].raw));
        n_same = (int)rec_n;
        ref_raw = set.x;
        ref_w = set.y;
        ref_hi = make_uint4(0u, 0u, 0u, 0u);  // members 2..9 exist only in sets of more than two
        if ((ref_raw & kCntMask) > 2u) ref_hi = ldg16(&a.probe[r].hi);
      }
      __syncwarp();
    }

    // ---------------- exceptions: endpoints with a non-zero match count ----------------
    const uint32_t areq = tie_areq(a.request_base + r, plan.seed_lo);
    const uint32_t nl = exc->n;
    const bool deferred = exc->overflow != 0;
    Best best = best_none();
    int xg = 0;
    auto consider = [&](int m, int c) {  // one exception: endpoint m matched c blocks
      if (m < M) {
        const uint32_t pos = perm_bitpos((uint32_t)m, LOG_EPL);
        const int wi = (int)(pos >> 5), kb = (int)(pos & 31);
        const uint32_t clo = __ldg(a.cls_lo + (size_t)ad * RW + wi), chi = __ldg(a.cls_hi + (size_t)ad * RW + wi);
        const uint32_t tmw = __ldg(a.tiemask + (size_t)ad * RW + wi);  // bit kb: G[ad][m] == gmax
        const int cls = (int)((clo >> kb) & 1u) | ((int)((chi >> kb) & 1u) << 1);
        const double s_true = eval_exception<SEQ>(a, m, c, n, cls);
        best_update_any(best, s_true, m, tie_mode, areq, plan.seed_hi);
        xg += (int)((tmw >> kb) & 1u);
      }
    };
    if (!deferred) {
      if (!use_table) {  // every matched block carries the reference set: its members are the exceptions
        if (n_same > 0)
          for (uint32_t k = gl; k < (ref_raw & kCntMask); k += G) consider((int)slot_member(ref_w, ref_hi, k), n_same);
      } else {
        for (uint32_t j0 = gl; j0 < nl; j0 += G) {
          const uint32_t e = exc->tab[exc->list[j0]];
          consider((int)(e >> 16) - 1, (int)(e & 0xFFFFu));
        }
      }
    }
    // reduce over the request's lane group (the merge rules — lowest index / highest priority — are order independent)
    const uint32_t gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (gi * G));
    if (tie_mode == 0) {
      // max-score with lowest-index ties through integer reductions (redux.sync): float64 scores order like their bit
      // patterns after the usual sign fold (scores are finite and never -0.0: the sum starts from +0.0)
      unsigned long long key = 0ULL;
      if (best.m >= 0) {
        const unsigned long long b = (unsigned long long)__double_as_longlong(best.score);
        key = (b >> 63) ? ~b : (b | 0x8000000000000000ULL);
      }
      const uint32_t khi = (uint32_t)(key >> 32), klo = (uint32_t)key;
      const uint32_t mh = __reduce_max_sync(gmask, khi);
      const uint32_t ml = __reduce_max_sync(gmask, khi == mh ? klo : 0u);
      const bool win = best.m >= 0 && khi == mh && klo == ml;
      const int cnt_all = (int)__reduce_add_sync(gmask, win ? (uint32_t)best.cnt : 0u);
      const int m_min = (int)__reduce_min_sync(gmask, win ? (uint32_t)best.m : 0x7fffffffu);
      const int src = __ffs(__ballot_sync(0xffffffffu, win) & gmask) - 1;  // a lane that holds the winning score
      const double s_win = shfl_f64(best.score, src < 0 ? lane : src);     // (every lane takes part in the shuffle)
      if (cnt_all > 0) {
        best.score = s_win;
        best.m = m_min;
        best.cnt = cnt_all;
      } else {
        best = best_none();
      }
    } else {
      best_group_reduce<G>(best, tie_mode);
    }
    xg = (int)__reduce_add_sync(gmask, (uint32_t)xg);

    // ---------------- combine with the per-adapter summary ----------------
    int pick, ties;
    double score;
    const bool exc_wins = best.m >= 0 && best.score > sm.gmax;
    const bool exc_ties = best.m >= 0 && best.score == sm.gmax;
    if (exc_wins) {
      pick = best.m;
      score = best.score;
      ties = best.cnt;
    } else {
      score = sm.gmax;
      ties = (sm.gcnt - xg) + (exc_ties ? best.cnt : 0);
      pick = exc_ties ? (best.m < sm.garg ? best.m : sm.garg) : sm.garg;
      if (sm.garg < 0) pick = exc_ties ? best.m : -1;
    }
    if (tie_mode) {  // warp-uniform: the shuffles below need every lane, whichever groups actually have a tie
      // seeded-random tie-break: the arg-max member with the highest priority, over
      // (precomputed tie set minus exceptions) ∪ (exceptions that tie)
      const bool need = !deferred && !exc_wins && ties > 1;  // uniform within a request's lane group only
      Best b2 = best_none();
      if (need && exc_ties && gl == 0) b2 = best;  // already reduced over the group
      if (need) {
#pragma unroll
        for (int q = 0; q < PW; q++) {
          const int wi = gl * PW + q;              // a word of the PERMUTED tie mask
          uint32_t x = __ldg(a.tiemask + (size_t)ad * RW + wi);
          const int j = wi >> 5, ln = wi & 31;
          while (x) {
            const int k = __ffs(x) - 1;
            x &= x - 1;
            const int m = (((j << LOG_EPL) + k) << 5) + ln;
            bool is_exc;
            if (use_table) {
              is_exc = exc_has(exc, (uint32_t)m);
            } else {
              is_exc = false;
              if (n_same > 0)
                for (uint32_t kk = 0; kk < (ref_raw & kCntMask); kk++) is_exc |= slot_member(ref_w, ref_hi, kk) == (uint32_t)m;
            }
            if (m < M && !is_exc) best_update_any(b2, sm.gmax, m, tie_mode, areq, plan.seed_hi);
          }
        }
      }
      __syncwarp();
      best_group_reduce<G>(b2, tie_mode);
      if (need) pick = b2.m;
    }
    __syncwarp();
    // reset the table: the listed entries, or all of it after an overflow (the list may be incomplete then)
    if (deferred) {
      for (int j0 = gl; j0 < kExcSlots; j0 += G) exc->tab[j0] = 0;
    } else {
      for (uint32_t j0 = gl; j0 < nl; j0 += G) exc->tab[exc->list[j0]] = 0;
    }
    if (gl == 0) {
      exc->n = 0;
      exc->overflow = 0;
    }
    // the warp-level shuffles above need every lane; only now drop the padding groups
    if (valid && gl == 0) {
      if (deferred) {
        a.pick[r] = kPickDeferred;   // scored by the full-matrix kernel launched right after this one
      } else {
        a.pick[r] = pick;
        a.pick_score[r] = pick >= 0 ? score : 0.0;
        a.tie_count[r] = pick >= 0 ? ties : 0;
      }
      if (a.total_out) a.total_out[r] = (uint16_t)n;
    }
    __syncwarp();
  }
}

template <int J, uint32_t SEQ>
static int launch_sparse_inst(const ScoreArgs& a, cudaStream_t s, int sm_count) {
  constexpr int RW = J * 32;
  constexpr int G = (RW / 4 < 32) ? RW / 4 : 32;
  constexpr int RPW = 32 / G;
  auto kernel = pick_sparse_kernel<J, SEQ>;
  int occ = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, kSparseWarps * 32, 0);
  if (occ < 1) occ = 1;
  const int per_block = kSparseWarps * RPW;
  int blocks = sm_count * occ;
  const int need = (a.R + per_block - 1) / per_block;
  if (blocks > need) blocks = need;
  if (blocks < 1) blocks = 1;
  return launched_one(launch_maybe_pdl(a.pdl != 0, kernel, dim3(blocks), dim3(kSparseWarps * 32), 0, s, a));
}

constexpr uint32_t sparse_seq() { return 0; }
template <typename... Rest>
constexpr uint32_t sparse_seq(int k, Rest... rest) {
  return (uint32_t)(k + 1) | (sparse_seq(rest...) << 4);
}

template <int J>
static int launch_sparse_seq(const ScoreArgs& a, cudaStream_t s, int sm_count) {
  constexpr uint32_t EPL_ = sparse_seq(STEP_EP_TERM, STEP_PREFIX, STEP_LORA);  // queue,kv folded | prefix | lora
  constexpr uint32_t EP_ = sparse_seq(STEP_EP_TERM, STEP_PREFIX);              // the reference's default config
  if (a.plan.seq == EPL_) return launch_sparse_inst<J, EPL_>(a, s, sm_count);
  if (a.plan.seq == EP_) return launch_sparse_inst<J, EP_>(a, s, sm_count);
  return launch_sparse_inst<J, 0>(a, s, sm_count);
}

// Applicable when: unmasked, not dense, no per-pair diagnostics, plan flagged sparse_ok, summaries present.
// Returns the number of launches: the sparse kernel plus the full-matrix kernel restricted to the requests it deferred.
static bool sparse_applies(const ScoreArgs& a) {
  if (a.R <= 0) return false;
  if (!a.plan.sparse_ok || !a.summ || !a.tiemask || a.cand_mask || a.dense || a.match_out || a.scores_out || a.topk > 0) return false;
  return a.geo.Mpad <= 65536;  // inline members are uint16
}

bool pick_sparse_probes(const ScoreArgs& a) {
  if (!sparse_applies(a)) return false;
  for (int s = 0; s < a.plan.n_steps; s++)
    if (a.plan.kind[s] == STEP_PREFIX) return true;
  return false;
}

int launch_pick_sparse(const ScoreArgs& a, cudaStream_t s, int sm_count) {
  if (!sparse_applies(a)) return 0;
  int launched;
  switch (a.geo.J) {
    case 1: launched = launch_sparse_seq<1>(a, s, sm_count); break;
    case 2: launched = launch_sparse_seq<2>(a, s, sm_count); break;
    case 4: launched = launch_sparse_seq<4>(a, s, sm_count); break;
    default: launched = launch_sparse_seq<8>(a, s, sm_count); break;
  }
  if (launched > 0 && a.table && a.hashes) {  // only a request with prefix matches can overflow its exception table
    ScoreArgs d = a;
    d.only_deferred = 1;
    const int deferred = launch_score_matrix(d, s, sm_count);
    if (deferred < 0) return deferred;
    launched += deferred;
  }
  return launched;
}

}  // namespace eppscore
