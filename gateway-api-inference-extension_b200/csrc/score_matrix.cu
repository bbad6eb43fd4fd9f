// score_matrix.cu — the full-matrix Score+Pick kernel: every (request, endpoint) pair is scored, nothing is
// assumed about the batch.  It is what candidate masks (the Filter chain's result), negative prefix weights
// and the diagnostics outputs (match_out / scores_out) run on, and the reference point the sparse path is
// tested against.  One warp per request; the R x M score matrix is never materialised.
//
//   matchLongestPrefix  approximateprefix/plugin.go:219-235   probe → run-length merge by interned row id →
//                                                             per-endpoint match counters in shared memory
//   queue scorer        scorer/queuedepth/queue.go:78-108     min/max over the FILTERED endpoints of the row,
//                                                             then a per-row LUT lut[d] = clamp(d/(max-min))*w
//   scorers + sum       scheduler_profile.go:151-174          float64, profile order, from 0.0
//   picker              maxscore/picker.go:87-115             branch-free arg-max + warp-shuffle reduce
//   latency fold-in     latencypredictorasync/prediction.go:164-194, predictedlatency/prediction.go:137-166,
//   (LAT variants)      scorer/latency/plugin.go:144-367      per pair: both linear predictions and the headrooms;
//                                                             per row: tier/bucket selection + min/max over the
//                                                             candidates in one pass, then the normalised score
// The scorer sequence is a template parameter (SEQ packs kind+1 per step, 4 bits each; 0 = runtime loop).
#include "device_common.cuh"
#include "lat_pair.cuh"
#include "prefix_table.cuh"

namespace eppscore {

constexpr int kMatrixWarps = 8;
constexpr int kMaxJ = 8;

constexpr int kLatW = 128;  // latency-scorer weights w/100 are tabulated for w in [0, 128) (plugin.go:301-306: w in [1,101])

__host__ __device__ constexpr bool seq_has_minmax(uint32_t seq) {
  return seq != 0 && ((int)(seq & 15u) - 1 == STEP_MINMAX || seq_has_minmax(seq >> 4));
}

// RND: the stochastic pickers (random / weighted-random) are compiled in; always for the runtime-generic SEQ == 0.
// TOPK: the first a.topk entries of each request's pick order are written too (runtime-generic SEQ == 0 only).  Those
// variants ask for one resident CTA per SM, so ptxas keeps the per-lane lists in registers instead of spilling them.
template <uint32_t SEQ, bool MASKED, bool DIAG, bool LAT, bool RND = (SEQ == 0), bool TOPK = false>
__global__ void __launch_bounds__(kMatrixWarps * 32, TOPK ? 1 : 0) score_matrix_kernel(const __grid_constant__ ScoreArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  pdl_wait();  // (no-op unless launched behind pick_sparse / the hash kernels with programmatic dependent launch)
  const int NWARPS = blockDim.x >> 5;  // kMatrixWarps, or fewer when that many do not fit in shared memory (launch_matrix)
  if (a.only_deferred) {  // the pass behind pick_sparse: normally nothing was deferred — leave before staging anything
    bool any = false;
    const int gw0 = blockIdx.x * NWARPS + (threadIdx.x >> 5), nw0 = gridDim.x * NWARPS;
    for (long long r = gw0 + (long long)(threadIdx.x & 31) * nw0; r < a.R; r += 32LL * nw0) any |= a.pick[r] == kPickDeferred;
    if (!__syncthreads_or(any ? 1 : 0)) return;
  }
  const Plan& plan = a.plan;
  const int M = a.geo.M, MPAD = a.geo.Mpad, J = a.geo.J, LOG_EPL = a.geo.log_epl, EPL = 1 << LOG_EPL;
  const int RW = a.geo.row_words;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool wide_cnt = a.hash_stride > 256;  // counters: 8-bit (0 decodes as 256 for touched slots) or 16-bit

  // ---- plan facts (warp-uniform) ----
  int prefix_step = -1, q_step = -1;
  bool has_minmax[2] = {false, false};
  for (int s = 0; s < plan.n_steps; s++) {
    if (plan.kind[s] == STEP_PREFIX && prefix_step < 0) prefix_step = s;
    if (plan.kind[s] == STEP_MINMAX) {
      has_minmax[plan.arg[s]] = true;
      if (q_step < 0) q_step = s;  // the first min/max scorer gets the per-row LUT
    }
  }

  // ---- shared memory carve-up ----
  // The term and min/max arrays are staged unless they do not fit beside one warp's counters (a.stage_terms == 0, only at
  // large Mpad with many terms); they are then read from global memory, where they stay L2-resident.  The specialised
  // sequences have at most one term array, which always fits: only the runtime-generic variants carry the global path.
  const bool stage = SEQ != 0 || a.stage_terms != 0;
  const bool q_smem = MASKED && (SEQ != 0 ? seq_has_minmax(SEQ) : (stage && (has_minmax[0] || has_minmax[1])));
  double* s_term = reinterpret_cast<double*>(smem_raw);
  long long* s_q = reinterpret_cast<long long*>(s_term + (stage ? (size_t)plan.n_terms * MPAD : 0));
  double* s_lora = reinterpret_cast<double*>(s_q + (q_smem ? 2 * MPAD : 0));
  double* s_latw = s_lora + kMaxSteps * 4;
  double* s_lut = s_latw + (LAT ? kLatW : 0);
  constexpr int NLUT = LAT ? 3 : 2;
  double* lut_p = s_lut + (size_t)warp * NLUT * (kLutMax + 1);
  double* lut_q = lut_p + (kLutMax + 1);
  double* lut_l = lut_q + (LAT ? (kLutMax + 1) : 0);  // coef * (c/total) of the prediction / composite
  unsigned char* s_cnt_all = reinterpret_cast<unsigned char*>(s_lut + (size_t)NWARPS * NLUT * (kLutMax + 1));
  const int cnt_bytes = MPAD * (wide_cnt ? 2 : 1) + RW * 4;  // match counters + the permuted bitmap of touched endpoints
  unsigned char* cnt_raw = s_cnt_all + (size_t)warp * cnt_bytes;
  uint32_t* tperm = reinterpret_cast<uint32_t*>(cnt_raw + MPAD * (wide_cnt ? 2 : 1));
  uint8_t* cnt8 = cnt_raw;
  uint16_t* cnt16 = reinterpret_cast<uint16_t*>(cnt_raw);

  if (stage)
    for (int t = 0; t < plan.n_terms; t++)
      for (int m = threadIdx.x; m < MPAD; m += blockDim.x) s_term[(size_t)t * MPAD + m] = a.term[t][m];
  if (q_smem)
    for (int which = 0; which < 2; which++)
      for (int m = threadIdx.x; m < MPAD; m += blockDim.x)
        s_q[which * MPAD + m] = (a.minmax_q[which] && m < M) ? a.minmax_q[which][m] : 0;
  auto qval = [&](int which, int m) -> long long {  // raw queue / running value of endpoint m (0 past M)
    if (q_smem) return s_q[which * MPAD + m];
    const long long* q = reinterpret_cast<const long long*>(a.minmax_q[which]);
    return (q && m < M) ? __ldg(q + m) : 0LL;
  };
  if (threadIdx.x < kMaxSteps * 4) s_lora[threadIdx.x] = plan.lora_term[threadIdx.x >> 2][threadIdx.x & 3];
  int lat_step = -1;
  if (LAT) {
    for (int s = 0; s < plan.n_steps; s++)
      if (plan.kind[s] == STEP_LATENCY && lat_step < 0) lat_step = s;
    // scores[ep] = w / wMax (plugin.go:306, :360), clamped and weighted like any scorer (scheduler_profile.go:168)
    if (threadIdx.x < kLatW)
      s_latw[threadIdx.x] = __dmul_rn(clamp01(__ddiv_rn((double)threadIdx.x, 100.0)), plan.weight[lat_step < 0 ? 0 : lat_step]);
  }
  for (int i = threadIdx.x; i < (NWARPS * cnt_bytes) / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(s_cnt_all)[i] = 0;
  __syncthreads();

  const bool want_prefix = prefix_step >= 0 || a.match_out != nullptr || a.total_out != nullptr || (LAT && lat_step >= 0);
  const int tie_mode = plan.tie_mode;
  int lut_total = -1, lutl_total = -1;

  const int gw = blockIdx.x * NWARPS + warp, nw = gridDim.x * NWARPS;
  for (int r = gw; r < a.R; r += nw) {
    if (a.only_deferred && a.pick[r] != kPickDeferred) continue;  // (warp-uniform) the sparse kernel already scored it
    // ---------------- matchLongestPrefix into the shared-memory counters ----------------
    uint32_t any[kMaxJ];
#pragma unroll
    for (int j = 0; j < kMaxJ; j++) any[j] = 0;
    int total = 0;
    if (want_prefix && a.hashes) {
      const int n = a.n_hashes[r];
      total = n;
      bool stop = n == 0 || a.table == nullptr;
      const TSlot* slots = stop ? nullptr : a.table->slots;
      const uint64_t slot_mask = stop ? 0 : a.table->mask;
      const uint32_t* ovf_rows = stop ? nullptr : a.table->ovf_rows;
      const int NW = MPAD >> 5;                               // words of a natural-order overflow row
      bool touched_any = false;
      for (int c0 = 0; !stop; c0 += 32) {
        const int i = c0 + lane;
        uint4 lo = make_uint4(0, 0, 0, 0), hi = make_uint4(0, 0, 0, 0);  // lo = {key.lo, key.hi, cnt, ep0|ep1<<16}, hi = ep2..ep9
        bool hit = false;
        if (i < n) {
          const uint64_t h = a.hashes[(size_t)r * a.hash_stride + i];
          uint64_t idx = h & slot_mask;
          for (;;) {                                        // indexer.Get, indexer.go:86-102
            lo = ldg16(&slots[idx]);
            if (lo.z == kCntFree) break;                    // never-used slot: hash unknown
            if ((((uint64_t)lo.y << 32) | lo.x) == h) {
              hit = (lo.z & kCntMask) != 0;                 // emptied set == deleted key
              if (hit && !(lo.z & kCntRow) && (lo.z & kCntMask) > 2u) hi = ldg16(reinterpret_cast<const uint4*>(&slots[idx]) + 1);
              break;
            }
            idx = (idx + 1) & slot_mask;
          }
        }
        const uint32_t miss = __ballot_sync(0xffffffffu, !hit);
        const int nh = miss ? (__ffs(miss) - 1) : 32;       // blocks matched before the first global miss
        // consecutive blocks are normally cached on the same endpoints: hits with identical (sorted) inline sets form one run
        const uint32_t pc = __shfl_up_sync(0xffffffffu, lo.z, 1), pw = __shfl_up_sync(0xffffffffu, lo.w, 1);
        const uint32_t p0 = __shfl_up_sync(0xffffffffu, hi.x, 1), p1 = __shfl_up_sync(0xffffffffu, hi.y, 1);
        const uint32_t p2 = __shfl_up_sync(0xffffffffu, hi.z, 1), p3 = __shfl_up_sync(0xffffffffu, hi.w, 1);
        const uint32_t c = lo.z & kCntMask;
        bool same = lane > 0 && !(lo.z & kCntRow) && pc == lo.z;
        if (same) {
          same = ((pw ^ lo.w) & (c >= 2 ? 0xFFFFFFFFu : 0x0000FFFFu)) == 0;
          if (c > 2) same = same && ((p0 ^ hi.x) & (c >= 4 ? 0xFFFFFFFFu : 0x0000FFFFu)) == 0;
          if (c > 4) same = same && ((p1 ^ hi.y) & (c >= 6 ? 0xFFFFFFFFu : 0x0000FFFFu)) == 0;
          if (c > 6) same = same && ((p2 ^ hi.z) & (c >= 8 ? 0xFFFFFFFFu : 0x0000FFFFu)) == 0;
          if (c > 8) same = same && ((p3 ^ hi.w) & (c >= 10 ? 0xFFFFFFFFu : 0x0000FFFFu)) == 0;
        }
        uint32_t bm = __ballot_sync(0xffffffffu, lane < nh && !same);
        while (bm) {
          const int s0 = __ffs(bm) - 1;
          bm &= bm - 1;
          const int len = (bm ? (__ffs(bm) - 1) : nh) - s0;
          const uint32_t rraw = __shfl_sync(0xffffffffu, lo.z, s0), ew = __shfl_sync(0xffffffffu, lo.w, s0);
          const uint32_t e0 = __shfl_sync(0xffffffffu, hi.x, s0), e1 = __shfl_sync(0xffffffffu, hi.y, s0);
          const uint32_t e2 = __shfl_sync(0xffffffffu, hi.z, s0), e3 = __shfl_sync(0xffffffffu, hi.w, s0);
          touched_any = true;
          if (!(rraw & kCntRow)) {                          // inline set: lane k bumps member k (res[server] += len)
            if (lane < (int)(rraw & kCntMask) && lane < kInlineEps) {
              const int wq = (lane - 2) >> 1;
              const uint32_t wsel = lane < 2 ? ew : (wq == 0 ? e0 : (wq == 1 ? e1 : (wq == 2 ? e2 : e3)));
              const uint32_t m = (lane & 1) ? (wsel >> 16) : (wsel & 0xFFFFu);
              const uint32_t pos = perm_bitpos(m, LOG_EPL);
              const int ci = (int)((pos >> 5) << LOG_EPL) + (int)(pos & 31);  // compact counter index of endpoint m
              if (wide_cnt) cnt16[ci] += (uint16_t)len;
              else cnt8[ci] += (uint8_t)len;
              atomicOr(&tperm[pos >> 5], 1u << (pos & 31));
            }
          } else {                                          // more than 10 members: a natural-order bitset row (id in ew)
            for (int w = lane; w < NW; w += 32) {
              uint32_t x = __ldg(ovf_rows + (size_t)ew * NW + w);
              while (x) {
                const int k = __ffs(x) - 1;
                x &= x - 1;
                const uint32_t pos = perm_bitpos((uint32_t)(w * 32 + k), LOG_EPL);
                const int ci = (int)((pos >> 5) << LOG_EPL) + (int)(pos & 31);
                if (wide_cnt) cnt16[ci] += (uint16_t)len;
                else cnt8[ci] += (uint8_t)len;
                atomicOr(&tperm[pos >> 5], 1u << (pos & 31));
              }
            }
          }
          __syncwarp();                                     // the next run may bump the same counters
        }
        if (nh < 32 || c0 + 32 >= n) stop = true;
      }
      if (touched_any) {                                    // each lane collects (and clears) the bits of its own endpoints
        __syncwarp();
#pragma unroll
        for (int j = 0; j < kMaxJ; j++)
          if (j < J) {
            any[j] = tperm[j * 32 + lane];
            tperm[j * 32 + lane] = 0;
          }
        __syncwarp();
      }
    }
    if (prefix_step >= 0 && total != lut_total && total <= kLutMax) {
      const double w = plan.weight[prefix_step];
      __syncwarp();
      for (int c = lane; c <= total; c += 32) lut_p[c] = prefix_term_direct(c, total, w);
      lut_total = total;
      __syncwarp();
    }
    const bool plut_ok = total <= kLutMax;

    // ---------------- per-request scorer inputs ----------------
    int ad = a.adapter_id ? a.adapter_id[r] : -1;
    if (ad < 0 || ad >= a.A) ad = a.A;
    const uint32_t* mrow = MASKED ? a.cand_mask + (size_t)r * a.mask_words : nullptr;
    // candidate-set min/max (queue.go:79-91 over the FILTERED endpoints), then the first such scorer's LUT
    long long mn[2] = {0, 0}, mx[2] = {0, 0};
    bool qlut_ok = false;
    if (MASKED && (has_minmax[0] || has_minmax[1])) {
      mn[0] = mn[1] = 0x7fffffffffffffffLL;
      mx[0] = mx[1] = (long long)0x8000000000000000ULL;
      bool scanned[2] = {!has_minmax[0], !has_minmax[1]};
      // fast path: first / last occupied value bucket that intersects the request's mask row
#pragma unroll
      for (int which = 0; which < 2; which++) {
        const QBucketHdr* hdr = a.qhdr[which];
        if (!has_minmax[which] || !hdr || !__ldg(&hdr->valid)) continue;
        const int MW = MPAD >> 5;
        uint32_t mw[kMaxJ];  // this lane's words of the mask row (MW <= 256 words)
#pragma unroll
        for (int t = 0; t < kMaxJ; t++) {
          const int w = t * 32 + lane;
          mw[t] = (t * 32 < MW && w < a.mask_words) ? __ldg(mrow + w) : 0u;
        }
        const uint32_t* tbl = a.qbucket[which];
        const long long base = __ldg(&hdr->base);
        int vmin = -1, vmax = -1;
        for (int wd = 0; wd < 8 && vmin < 0; wd++) {
          uint32_t occ = __ldg(&hdr->occ[wd]);
          while (occ && vmin < 0) {
            const int v = wd * 32 + __ffs(occ) - 1;
            occ &= occ - 1;
            bool hit = false;
#pragma unroll
            for (int t = 0; t < kMaxJ; t++)
              if (t * 32 < MW) hit = hit || (mw[t] & __ldg(tbl + (size_t)v * MW + t * 32 + lane)) != 0u;
            if (__any_sync(0xffffffffu, hit)) vmin = v;
          }
        }
        for (int wd = 7; wd >= 0 && vmin >= 0 && vmax < 0; wd--) {
          uint32_t occ = __ldg(&hdr->occ[wd]);
          while (occ && vmax < 0) {
            const int b = 31 - __clz(occ);
            const int v = wd * 32 + b;
            occ &= ~(1u << b);
            bool hit = false;
#pragma unroll
            for (int t = 0; t < kMaxJ; t++)
              if (t * 32 < MW) hit = hit || (mw[t] & __ldg(tbl + (size_t)v * MW + t * 32 + lane)) != 0u;
            if (__any_sync(0xffffffffu, hit)) vmax = v;
          }
        }
        if (vmin >= 0) {
          mn[which] = base + vmin;
          mx[which] = base + vmax;
        }
        scanned[which] = true;  // (no candidate at all: the sentinels stay, exactly like the scan)
      }
      if (!scanned[0] || !scanned[1]) {
        for (int t = 0; t < J * EPL; t++) {
          const int m = t * 32 + lane;
          if (m < M && ((__ldg(mrow + t) >> lane) & 1u)) {
#pragma unroll
            for (int which = 0; which < 2; which++) {
              if (scanned[which]) continue;
              const long long v = qval(which, m);
              mn[which] = v < mn[which] ? v : mn[which];
              mx[which] = v > mx[which] ? v : mx[which];
            }
          }
        }
#pragma unroll
        for (int o = 16; o; o >>= 1)
#pragma unroll
          for (int which = 0; which < 2; which++) {
            if (scanned[which]) continue;
            const long long omn = shfl_xor_i64(mn[which], o), omx = shfl_xor_i64(mx[which], o);
            mn[which] = omn < mn[which] ? omn : mn[which];
            mx[which] = omx > mx[which] ? omx : mx[which];
          }
      }
      if (q_step >= 0) {
        const int which = plan.arg[q_step];
        const long long range = mx[which] >= mn[which] ? mx[which] - mn[which] : 0;  // (no candidates: nothing to score)
        if (range > 0 && range <= kLutMax) {  // lut_q[d] = clamp(d / range) * w, d = max - q  (queue.go:99)
          const double w = plan.weight[q_step];
          __syncwarp();
          for (int d = lane; d <= (int)range; d += 32)
            lut_q[d] = __dmul_rn(clamp01(__ddiv_rn(__ll2double_rn((long long)d), __ll2double_rn(range))), w);
          __syncwarp();
          qlut_ok = true;
        }
      }
    }

    // ---------------- latency fold-in: per-request inputs and tier selection (plugin.go:174-243) ----------------
    double l_x = 0.0, l_y = 0.0, l_tslo = 0.0, l_buf = 0.0;
    double l_mnT = 0.0, l_rgT = 0.0, l_mnP = 0.0, l_rgP = 0.0, l_alpha = 0.0, l_beta = 0.0, l_qrange = 0.0;
    double l_rT = 0.0, l_rP = 0.0;
    long long l_maxq = 0;
    int l_sel = 5;
    bool l_tok = false, l_pok = false, l_fast = false;
    const bool llut_ok = total <= kLutMax;
    uint32_t cb[kMaxJ];
    const uint32_t areq_f = tie_areq(a.request_base + r, plan.seed_lo);
    if (LAT && lat_step >= 0) {
      const LatArgs& L = a.lat;
      const double in_tok = (double)(L.input_tokens ? L.input_tokens[r] : 0);  // len(strings.Fields(prompt)), training.go:51
      l_x = __dmul_rn(L.ttft_input, in_tok);
      l_y = __dmul_rn(L.tpot_input, in_tok);
      l_tslo = L.ttft_slo ? L.ttft_slo[r] : 0.0;
      l_buf = __dmul_rn(L.tpot_slo ? L.tpot_slo[r] : 0.0, L.buffer);            // prediction.go:150
      const double pcoef = L.has_predictions ? L.ttft_prefix : L.wpref;
      if (llut_ok && total != lutl_total) {  // match/total with NaN (0/0) => 0: preparedata_hooks.go:44-58, plugin.go:381-392
        __syncwarp();
        for (int c = lane; c <= total; c += 32)
          lut_l[c] = __dmul_rn(pcoef, total ? __ddiv_rn((double)c, (double)total) : 0.0);
        lutl_total = total;
        __syncwarp();
      }
      // this lane's candidates as bits (bit k of cb[j] = endpoint (j*EPL+k)*32+lane): the caller's mask, then narrowed by
      // the device-side filters
#pragma unroll
      for (int j = 0; j < kMaxJ; j++) {
        cb[j] = 0;
        if (j >= J) continue;
        for (int k = 0; k < EPL; k++) {
          const int t = j * EPL + k, m = t * 32 + lane;
          bool cand = m < M;
          if (MASKED) cand = cand && ((__ldg(mrow + t) >> lane) & 1u);
          cb[j] |= (cand ? 1u : 0u) << k;
        }
      }
      if (a.n_filters > 0) {
        int ncand = 0;
#pragma unroll
        for (int j = 0; j < kMaxJ; j++) ncand += __popc(cb[j]);
        ncand = __reduce_add_sync(0xffffffffu, ncand);
        for (int f = 0; f < a.n_filters && ncand > 1; f++) {  // (every filter returns its input when len(endpoints) <= 1)
          const double u = uniform01(tie_prio(areq_f, -(f + 1), plan.seed_hi), -(f + 1));  // the filter's rand.Float64()
          const int fkind = a.filter_kind[f];
          const double p0 = a.filter_param[f][0], p1 = a.filter_param[f][1], p2 = a.filter_param[f][2];
          uint32_t sb[kMaxJ];
          int nA = 0;                                         // |sticky| resp. |positive|
          double minA = 1.7976931348623157e308, minB = minA;  // bestTTFT of the two sides
          if (fkind == 1) {                                   // prefix-cache-affinity-filter, prefixcacheaffinity/plugin.go:105-151
            if (p0 <= 0.0 || u < p1 || total == 0) continue;  // disabled / exploration / no prefix info: keep all
            // smallest match count whose score match/total reaches the threshold (monotone in the count)
            int cmin = 0x7fffffff;
            for (int c0 = 0; c0 <= total && cmin == 0x7fffffff; c0 += 32) {
              const int c = c0 + lane;
              const bool ok = c <= total && __ddiv_rn((double)c, (double)total) >= p0;
              const uint32_t bal = __ballot_sync(0xffffffffu, ok);
              if (bal) cmin = c0 + __ffs(bal) - 1;
            }
#pragma unroll
            for (int j = 0; j < kMaxJ; j++) {
              sb[j] = 0;
              if (j >= J) continue;
              const uint32_t anyj = any[j];
              const int cbase = (j * 32 + lane) << LOG_EPL;
              for (int k = 0; k < EPL; k++) {
                int c = wide_cnt ? (int)cnt16[cbase + k] : (int)cnt8[cbase + k];
                c = (c == 0 && ((anyj >> k) & 1u)) ? (wide_cnt ? 65536 : 256) : c;
                const bool cand = (cb[j] >> k) & 1u, sticky = cand && c >= cmin;
                sb[j] |= (sticky ? 1u : 0u) << k;
                if (L.has_predictions && p2 > 0.0) {
                  const double pt = llut_ok ? lut_l[c] : __dmul_rn(pcoef, __ddiv_rn((double)c, (double)total));
                  const LatPair lp = lat_pair(L.ep + (size_t)(j * EPL + k) * 256 + lane, L.tpot_generated, pt, l_x, l_y, l_tslo, l_buf);
                  if (sticky) minA = lp.ttft < minA ? lp.ttft : minA;
                  if (cand && !sticky) minB = lp.ttft < minB ? lp.ttft : minB;
                }
              }
              nA += __popc(sb[j]);
            }
            nA = __reduce_add_sync(0xffffffffu, nA);
            if (nA == 0) continue;                            // no sticky endpoints: keep all
            if (p2 > 0.0 && nA < ncand) {                     // TTFT load gate (:133-142)
#pragma unroll
              for (int o = 16; o; o >>= 1) {
                const double oa = shfl_xor_f64(minA, o), ob = shfl_xor_f64(minB, o);
                minA = oa < minA ? oa : minA;
                minB = ob < minB ? ob : minB;
              }
              if (__dsub_rn(minA, minB) > p2) continue;       // stickiness would cost too much TTFT: keep all
            }
#pragma unroll
            for (int j = 0; j < kMaxJ; j++) cb[j] = sb[j];
            ncand = nA;
          } else if (fkind == 2) {                            // slo-headroom-tier-filter, sloheadroomtier/plugin.go:82-137
            if (!L.has_predictions) continue;                 // no predictions: keep all
#pragma unroll
            for (int j = 0; j < kMaxJ; j++) {
              sb[j] = 0;
              if (j >= J) continue;
              const uint32_t anyj = any[j];
              const int cbase = (j * 32 + lane) << LOG_EPL;
              for (int k = 0; k < EPL; k++) {
                int c = wide_cnt ? (int)cnt16[cbase + k] : (int)cnt8[cbase + k];
                c = (c == 0 && ((anyj >> k) & 1u)) ? (wide_cnt ? 65536 : 256) : c;
                const double pt = llut_ok ? lut_l[c] : __dmul_rn(pcoef, total ? __ddiv_rn((double)c, (double)total) : 0.0);
                const LatPair lp = lat_pair(L.ep + (size_t)(j * EPL + k) * 256 + lane, L.tpot_generated, pt, l_x, l_y, l_tslo, l_buf);
                sb[j] |= ((((cb[j] >> k) & 1u) && lp.rank == 0) ? 1u : 0u) << k;  // positive: both headrooms >= 0
              }
              nA += __popc(sb[j]);
            }
            nA = __reduce_add_sync(0xffffffffu, nA);
            if (nA > 0 && nA < ncand) {                       // both tiers present: explore the negative one with probability eps
              const bool neg = u < p0;
#pragma unroll
              for (int j = 0; j < kMaxJ; j++) cb[j] = neg ? (cb[j] & ~sb[j]) : sb[j];
              ncand = neg ? ncand - nA : nA;
            }
          }
        }
      }
      if (a.filter_mask_out) {  // natural-order mask words (bit = lane) of the surviving candidates
#pragma unroll
        for (int j = 0; j < kMaxJ; j++) {
          if (j >= J) continue;
          for (int k = 0; k < EPL; k++) {
            const uint32_t word = __ballot_sync(0xffffffffu, (cb[j] >> k) & 1u);
            const int t = j * EPL + k;
            if (lane == 0 && t < a.mask_words) a.filter_mask_out[(size_t)r * a.mask_words + t] = word;
          }
        }
      }
      if (L.has_predictions) {
        // one pass: every lane tracks the best (lowest) tier it has seen and the |headroom| min/max inside it
        // (branch-free: a non-candidate is tier 5, which never wins against a candidate)
        int rank_l = 5;
        double mnT = 1.7976931348623157e308, mxT = -1.7976931348623157e308, mnP = mnT, mxP = mxT;
#pragma unroll
        for (int j = 0; j < kMaxJ; j++) {
          if (j >= J) break;
          const uint32_t anyj = any[j];
          const int cbase = (j * 32 + lane) << LOG_EPL;
#pragma unroll 2
          for (int k = 0; k < EPL; k++) {
            const int t = j * EPL + k;
            const bool cand = (cb[j] >> k) & 1u;
            int c = wide_cnt ? (int)cnt16[cbase + k] : (int)cnt8[cbase + k];
            c = (c == 0 && ((anyj >> k) & 1u)) ? (wide_cnt ? 65536 : 256) : c;
            const double pt = llut_ok ? lut_l[c] : __dmul_rn(pcoef, total ? __ddiv_rn((double)c, (double)total) : 0.0);
            const LatPair lp = lat_pair(L.ep + (size_t)t * 256 + lane, L.tpot_generated, pt, l_x, l_y, l_tslo, l_buf);
            const int rk = cand ? lp.rank : 5;
            const double aT = fabs(lp.hT), aP = fabs(lp.hP);
            const bool better = rk < rank_l, same = rk == rank_l;
            mnT = (better || (same && aT < mnT)) ? aT : mnT;
            mxT = (better || (same && aT > mxT)) ? aT : mxT;
            mnP = (better || (same && aP < mnP)) ? aP : mnP;
            mxP = (better || (same && aP > mxP)) ? aP : mxP;
            rank_l = better ? rk : rank_l;
          }
        }
        l_sel = __reduce_min_sync(0xffffffffu, rank_l);
        if (rank_l != l_sel) {
          mnT = mnP = 1.7976931348623157e308;
          mxT = mxP = -1.7976931348623157e308;
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
          const double a0 = shfl_xor_f64(mnT, o), a1 = shfl_xor_f64(mxT, o), a2 = shfl_xor_f64(mnP, o), a3 = shfl_xor_f64(mxP, o);
          mnT = a0 < mnT ? a0 : mnT;
          mxT = a1 > mxT ? a1 : mxT;
          mnP = a2 < mnP ? a2 : mnP;
          mxP = a3 > mxP ? a3 : mxP;
        }
        l_mnT = mnT;
        l_mnP = mnP;
        l_rgT = __dsub_rn(mxT, mnT);
        l_rgP = __dsub_rn(mxP, mnP);
        const double eps = 1e-9;                                                // plugin.go:41
        l_tok = l_rgT > eps;
        l_pok = l_rgP > eps;
        l_rT = l_tok ? __drcp_rn(l_rgT) : 0.0;                                  // fast path of the normalisation, see below
        l_rP = l_pok ? __drcp_rn(l_rgP) : 0.0;
        l_alpha = L.alpha;
        l_beta = L.beta;
        if (!l_tok && l_pok) {                                                  // plugin.go:275-279
          l_alpha = 0.0;
          l_beta = 1.0;
        } else if (!l_pok && l_tok) {
          l_alpha = 1.0;
          l_beta = 0.0;
        }
        l_fast = l_alpha >= 0.0 && l_alpha <= 1.0 && l_beta >= 0.0 && l_beta <= 1.0;
      } else {
        // composite fallback: maxQ over the candidates, starting from 0 (plugin.go:338-344)
        long long mq = 0;
#pragma unroll
        for (int j = 0; j < kMaxJ; j++) {
          if (j >= J) continue;
          for (int k = 0; k < EPL; k++) {
            const int t = j * EPL + k;
            if ((cb[j] >> k) & 1u) {
              const long long q = __ldg(reinterpret_cast<const long long*>(L.ep + (size_t)t * 256 + 32 + lane));
              mq = q > mq ? q : mq;
            }
          }
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
          const long long oq = shfl_xor_i64(mq, o);
          mq = oq > mq ? oq : mq;
        }
        l_maxq = mq;
        l_qrange = __ll2double_rn(mq);
        l_rT = mq > 0 ? __drcp_rn(l_qrange) : 0.0;
        l_fast = L.wq >= 0.0 && L.wq <= 1.0;
      }
    }

    const uint32_t areq = tie_areq(a.request_base + r, plan.seed_lo);
    Best best = best_none();
    RBest rb_pos = rbest_none(), rb_all = rbest_none();  // stochastic pickers (runtime-generic variants only)
    const int pick_mode = RND ? plan.pick_mode : 0;
    TopK tk;
    if (TOPK) topk_clear(tk);

    // ---------------- Score (scheduler_profile.go:151-174) + Pick (maxscore/picker.go:87-115) ----------------
    // per-step constants hoisted out of the pair loop (compile-time step index when SEQ != 0)
    const double* tptr[8];
    double wq[8];
#pragma unroll
    for (int s = 0; s < 8; s++) {
      const int ta = s < plan.n_steps && plan.kind[s] == STEP_EP_TERM ? plan.arg[s] : 0;
      tptr[s] = stage ? s_term + (size_t)ta * MPAD : a.term[ta];
      wq[s] = s < plan.n_steps ? plan.weight[s] : 0.0;
    }
    const bool q_flat = !MASKED || q_step < 0 || mx[plan.arg[q_step < 0 ? 0 : q_step]] == mn[plan.arg[q_step < 0 ? 0 : q_step]];
#pragma unroll
    for (int j = 0; j < kMaxJ; j++) {
      if (j >= J) break;
      uint32_t clo = 0, chi = 0;
      if (a.cls_lo) {
        clo = __ldg(a.cls_lo + (size_t)ad * RW + j * 32 + lane);
        chi = __ldg(a.cls_hi + (size_t)ad * RW + j * 32 + lane);
      }
      const uint32_t anyj = any[j];
      const int cbase = (j * 32 + lane) << LOG_EPL;
#pragma unroll(LAT ? 2 : 4)
      for (int k = 0; k < EPL; k++) {
        const int t = j * EPL + k, m = t * 32 + lane;
        bool cand = m < M;
        if (LAT && lat_step >= 0) cand = (cb[j] >> k) & 1u;
        else if (MASKED) cand = cand && ((__ldg(mrow + t) >> lane) & 1u);
        // match count: untouched slots hold 0; a touched slot holds the count modulo 2^bits (never 0 modulo)
        int c = wide_cnt ? (int)cnt16[cbase + k] : (int)cnt8[cbase + k];
        c = (c == 0 && ((anyj >> k) & 1u)) ? (wide_cnt ? 65536 : 256) : c;
        if (DIAG && a.match_out && m < M) a.match_out[(size_t)r * M + m] = (uint16_t)c;
        const int cls = (int)((clo >> k) & 1u) | ((int)((chi >> k) & 1u) << 1);
        double acc = 0.0;  // weightedScorePerEndpoint[endpoint] = float64(0), scheduler_profile.go:156-158
        auto step = [&](int s, int kind) {
          double term;
          if (kind == STEP_EP_TERM) {
            term = tptr[s][m];
          } else if (kind == STEP_PREFIX) {
            term = (s == prefix_step && plut_ok) ? lut_p[c] : prefix_term_direct(c, total, wq[s]);
          } else if (kind == STEP_LORA) {
            term = s_lora[s * 4 + cls];
          } else if (kind == STEP_MINMAX) {
            const int which = plan.arg[s];
            if (s == q_step ? q_flat : (!MASKED || mx[which] == mn[which])) {
              term = __dmul_rn(1.0, wq[s]);                                  // queue.go:95-98
            } else if (s == q_step && qlut_ok) {
              long long d = mx[which] - qval(which, m);
              d = d < 0 ? 0 : (d > kLutMax ? kLutMax : d);                   // (non-candidates only)
              term = lut_q[(int)d];
            } else {
              const double sc = __ddiv_rn(__ll2double_rn(mx[which] - qval(which, m)),
                                          __ll2double_rn(mx[which] - mn[which]));  // queue.go:99
              term = __dmul_rn(clamp01(sc), wq[s]);
            }
          } else if (LAT && kind == STEP_LATENCY) {
            // The score is quantised (w/100 with w an integer), so the two normalising divides are only needed to
            // decide on which side of an integer boundary v falls.  Fast path: multiply by the correctly rounded
            // reciprocal of the range (|v' - v| < 2e-13 when alpha, beta are in [0,1]); if v' is farther than 1e-9
            // from an integer the truncation is already decided, otherwise redo it exactly as plugin.go:283-306.
            const LatArgs& L = a.lat;
            const double pt = llut_ok ? lut_l[c] : __dmul_rn(L.has_predictions ? L.ttft_prefix : L.wpref,
                                                             total ? __ddiv_rn((double)c, (double)total) : 0.0);
            const double* tp = L.ep + (size_t)t * 256 + lane;
            long long w = 0;  // Go's int: 64-bit, so no v below 2^63 saturates or wraps
            if (L.has_predictions) {
              const LatPair lp = lat_pair(tp, L.tpot_generated, pt, l_x, l_y, l_tslo, l_buf);
              if (DIAG && L.pred_out && m < M) {
                L.pred_out[((size_t)r * M + m) * 2] = lp.ttft;
                L.pred_out[((size_t)r * M + m) * 2 + 1] = lp.tpot;
              }
              const bool most = L.strategy_most && l_sel == 0;
              const double dT = __dsub_rn(fabs(lp.hT), l_mnT), dP = __dsub_rn(fabs(lp.hP), l_mnP);
              const double nT = l_tok ? __dmul_rn(dT, l_rT) : 0.5, nP = l_pok ? __dmul_rn(dP, l_rP) : 0.5;
              const double comb = __dadd_rn(__dmul_rn(l_alpha, nT), __dmul_rn(l_beta, nP));
              const double v = most ? __dmul_rn(comb, 100.0) : __dmul_rn(__dsub_rn(1.0, comb), 100.0);
              const int vn = __double2int_rn(v);
              const bool in_tier = lp.rank == l_sel;
              w = in_tier ? __double2ll_rz(v) + 1 : 0;                         // float64(int(x) + minWeight + 1); 0 outside the tier
              const bool redo = in_tier && (!l_fast || fabs(__dsub_rn(v, (double)vn)) < 1e-9);
              if (__any_sync(0xffffffffu, redo)) {                             // warp-uniform: scoreBucket, plugin.go:281-306, exactly
                const double eT = l_tok ? __ddiv_rn(dT, l_rgT) : 0.5, eP = l_pok ? __ddiv_rn(dP, l_rgP) : 0.5;
                const double ec = __dadd_rn(__dmul_rn(l_alpha, eT), __dmul_rn(l_beta, eP));
                const long long we = __double2ll_rz(most ? __dmul_rn(ec, 100.0) : __dmul_rn(__dsub_rn(1.0, ec), 100.0)) + 1;
                w = redo ? we : w;
              }
            } else {                                                           // compositeScores, plugin.go:346-360
              const long long q = __ldg(reinterpret_cast<const long long*>(tp + 32));
              const double dq = __ll2double_rn(l_maxq - q);
              const double rel = l_maxq > 0 ? __dmul_rn(dq, l_rT) : 1.0;
              const double ck = __ldg(tp);
              const double v = __dmul_rn(100.0, __dadd_rn(__dadd_rn(ck, __dmul_rn(L.wq, rel)), pt));
              const double fl = floor(v);
              w = __double2ll_rz(round(v));                                    // int(math.Round(0 + 100*composite))
              const bool redo = !l_fast || !(fabs(v) < 1e4) || fabs(__dsub_rn(__dsub_rn(v, fl), 0.5)) < 1e-9;
              if (__any_sync(0xffffffffu, redo)) {
                const double er = l_maxq > 0 ? __ddiv_rn(dq, l_qrange) : 1.0;
                const long long we = __double2ll_rz(round(__dmul_rn(100.0, __dadd_rn(__dadd_rn(ck, __dmul_rn(L.wq, er)), pt))));
                w = redo ? we : w;
              }
              if (DIAG && L.pred_out && m < M) {
                L.pred_out[((size_t)r * M + m) * 2] = nan64();
                L.pred_out[((size_t)r * M + m) * 2 + 1] = nan64();
              }
            }
            term = (unsigned long long)w < (unsigned long long)kLatW ? s_latw[w]
                                                                     : __dmul_rn(clamp01(__ddiv_rn(__ll2double_rn(w), 100.0)), wq[s]);
          } else {
            term = __dmul_rn(0.0, wq[s]);                                    // pair columns absent: score 0
          }
          acc = __dadd_rn(acc, term);  // += enforceScoreRange(score) * weight, scheduler_profile.go:168
        };
        if (SEQ == 0) {
          for (int s = 0; s < plan.n_steps; s++) step(s, plan.kind[s]);
        } else {
#pragma unroll
          for (int s = 0; s < 8; s++) {
            const int kind = (int)((SEQ >> (4 * s)) & 15u) - 1;
            if (kind >= 0) step(s, kind);
          }
        }
        if (DIAG && a.scores_out && m < M) a.scores_out[(size_t)r * M + m] = cand ? acc : nan64();
        if (RND && pick_mode != 0) {
          if (cand) {  // random: highest priority wins; weighted-random (A-Res): smallest -ln(U)/score among score > 0
            const uint32_t pr = tie_prio(areq, m, plan.seed_hi);
            rbest_update(rb_all, (double)pr, acc, m);
            if (pick_mode == 1 && acc > 0.0) rbest_update(rb_pos, ares_key(pr, m, acc), acc, m);
          }
        } else if (cand) {
          best_update(best, acc, m, tie_mode, areq, plan.seed_hi);
        }
        if (TOPK && cand) {
          double key;
          unsigned long long ord;
          topk_key(pick_mode, tie_mode, acc, tie_prio(areq, m, plan.seed_hi), m, key, ord);
          topk_insert(tk, a.topk, key, ord, acc);
        }
      }
      // re-zero exactly the counters this request touched
      uint32_t x = anyj;
      while (x) {
        const int k = __ffs(x) - 1;
        x &= x - 1;
        if (wide_cnt) cnt16[cbase + k] = 0;
        else cnt8[cbase + k] = 0;
      }
    }
    best_group_reduce<32>(best, tie_mode);
    if (RND && pick_mode != 0) {  // warp-uniform
      rbest_warp_reduce(rb_pos);
      rbest_warp_reduce(rb_all);
      const RBest& w = rb_pos.m >= 0 ? rb_pos : rb_all;  // no positive score: the random picker (weightedrandom/picker.go:113-116)
      best.m = w.m;
      best.score = w.score;
      best.cnt = w.n;
    }
    if (TOPK) {  // (warp-uniform) the per-lane lists merged into the request's first a.topk entries, lane i writes entry i
      int tm;
      double ts;
      topk_warp_merge(tk, a.topk, lane, tm, ts);
      if (lane < a.topk) {
        a.topk_m[(size_t)r * a.topk + lane] = tm;
        a.topk_score[(size_t)r * a.topk + lane] = ts;
      }
    }
    if (lane == 0) {
      a.pick[r] = best.m;
      a.pick_score[r] = best.m >= 0 ? best.score : 0.0;
      a.tie_count[r] = best.cnt;
      if (a.total_out) a.total_out[r] = (uint16_t)total;
    }
    __syncwarp();
  }
}

template <typename K>
static int launch_matrix(K kernel, const ScoreArgs& args, bool masked, bool lat, bool generic, cudaStream_t s, int sm_count) {
  ScoreArgs a = args;
  const int MPAD = a.geo.Mpad;
  const bool wide = a.hash_stride > 256;
  bool minmax = false;
  for (int i = 0; i < a.plan.n_steps; i++) minmax = minmax || a.plan.kind[i] == STEP_MINMAX;
  // the kernel's carve-up: term arrays [+ min/max values], LoRA terms [+ latency weights], then per warp the LUTs, the
  // match counters and the touched-endpoint bitmap
  const size_t staged = (size_t)a.plan.n_terms * MPAD * 8 + (masked && minmax ? 2 * (size_t)MPAD * 8 : 0);
  const size_t fixed = kMaxSteps * 4 * 8 + (lat ? kLatW * 8 : 0);
  const size_t per_warp = (size_t)(lat ? 3 : 2) * (kLutMax + 1) * 8 + (size_t)MPAD * (wide ? 2 : 1) + (size_t)a.geo.row_words * 4;
  int warps = 0;
  size_t smem = 0;
  cudaError_t c = fit_cta_smem(staged, fixed, per_warp, kMatrixWarps, generic, &warps, &a.stage_terms, &smem);
  if (c == cudaSuccess) c = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (c != cudaSuccess) return -(int)c;
  int occ = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, warps * 32, smem);
  if (occ < 1) occ = 1;
  const int need = (a.R + warps - 1) / warps;
  int blocks = sm_count * occ;  // persistent: one wave, warps stride over requests
  if (blocks > need) blocks = need;
  if (blocks < 1) blocks = 1;
  return launched_one(launch_maybe_pdl(a.pdl != 0, kernel, dim3(blocks), dim3(warps * 32), smem, s, a));
}

constexpr uint32_t mseq() { return 0; }
template <typename... Rest>
constexpr uint32_t mseq(int k, Rest... rest) {
  return (uint32_t)(k + 1) | (mseq(rest...) << 4);
}

#define E STEP_EP_TERM
#define P STEP_PREFIX
#define L STEP_LORA
#define Q STEP_MINMAX
#define T STEP_LATENCY
#define MK(...) launch_matrix(score_matrix_kernel<mseq(__VA_ARGS__), MASKED, DIAG, false>, a, MASKED, false, false, s, sm_count)
#define MKL(...) launch_matrix(score_matrix_kernel<mseq(__VA_ARGS__), MASKED, DIAG, true>, a, MASKED, true, false, s, sm_count)
#define MKR(...) launch_matrix(score_matrix_kernel<mseq(__VA_ARGS__), MASKED, DIAG, false, true>, a, MASKED, false, false, s, sm_count)
template <bool MASKED, bool DIAG>
static int launch_matrix_seq(const ScoreArgs& a, cudaStream_t s, int sm_count) {
  bool lat = false;
  for (int i = 0; i < a.plan.n_steps; i++) lat = lat || a.plan.kind[i] == STEP_LATENCY;
  if (a.plan.pick_mode != 0) {  // stochastic pickers: the default scorer sets have their own variants, the rest is runtime-generic
    if (a.plan.seq == mseq(E, P, L)) return MKR(E, P, L);
    if (a.plan.seq == mseq(E, P)) return MKR(E, P);
  }
  switch (a.plan.pick_mode == 0 ? a.plan.seq : 0xffffffffu) {
    case mseq(E): return MK(E);
    case mseq(E, P): return MK(E, P);
    case mseq(E, P, L): return MK(E, P, L);
    case mseq(E, L): return MK(E, L);
    case mseq(Q, E): return MK(Q, E);
    case mseq(Q, E, P): return MK(Q, E, P);
    case mseq(Q, E, P, L): return MK(Q, E, P, L);
    case mseq(E, Q, P, L): return MK(E, Q, P, L);
    case mseq(T): return MKL(T);          // the latency profile of the reference chart (config/charts/epplib/templates/_config.yaml:66-75)
    case mseq(T, L): return MKL(T, L);
    default:
      return lat ? launch_matrix(score_matrix_kernel<0, MASKED, DIAG, true>, a, MASKED, true, true, s, sm_count)
                 : launch_matrix(score_matrix_kernel<0, MASKED, DIAG, false>, a, MASKED, false, true, s, sm_count);
  }
}
// top-k lists: the runtime-generic variants only, every pick mode
template <bool MASKED, bool DIAG>
static int launch_matrix_topk(const ScoreArgs& a, cudaStream_t s, int sm_count) {
  bool lat = false;
  for (int i = 0; i < a.plan.n_steps; i++) lat = lat || a.plan.kind[i] == STEP_LATENCY;
  return lat ? launch_matrix(score_matrix_kernel<0, MASKED, DIAG, true, true, true>, a, MASKED, true, true, s, sm_count)
             : launch_matrix(score_matrix_kernel<0, MASKED, DIAG, false, true, true>, a, MASKED, false, true, s, sm_count);
}
#undef MK
#undef MKL
#undef MKR
#undef T
#undef E
#undef P
#undef L
#undef Q

// The file is compiled eight times (build.py: -DEPP_MATRIX_PART=0..7), one (MASKED, DIAG) combination of the kernel per object
// and the top-k variants apart (parts 4..7), so the 64 instantiations build in parallel (one translation unit took over three
// minutes); without the macro everything lands in one object.  The kernels are the same instantiations either way.
#ifndef EPP_MATRIX_PART
#define EPP_MATRIX_PART -1
#endif
int launch_matrix_part0(const ScoreArgs& a, cudaStream_t s, int sm_count);  // unmasked
int launch_matrix_part1(const ScoreArgs& a, cudaStream_t s, int sm_count);  // unmasked, diagnostics outputs
int launch_matrix_part2(const ScoreArgs& a, cudaStream_t s, int sm_count);  // masked
int launch_matrix_part3(const ScoreArgs& a, cudaStream_t s, int sm_count);  // masked, diagnostics outputs
int launch_matrix_part4(const ScoreArgs& a, cudaStream_t s, int sm_count);  // parts 0..3 with top-k lists
int launch_matrix_part5(const ScoreArgs& a, cudaStream_t s, int sm_count);
int launch_matrix_part6(const ScoreArgs& a, cudaStream_t s, int sm_count);
int launch_matrix_part7(const ScoreArgs& a, cudaStream_t s, int sm_count);
#if EPP_MATRIX_PART == -1 || EPP_MATRIX_PART == 0
int launch_matrix_part0(const ScoreArgs& a, cudaStream_t s, int sm_count) { return launch_matrix_seq<false, false>(a, s, sm_count); }
#endif
#if EPP_MATRIX_PART == -1 || EPP_MATRIX_PART == 1
int launch_matrix_part1(const ScoreArgs& a, cudaStream_t s, int sm_count) { return launch_matrix_seq<false, true>(a, s, sm_count); }
#endif
#if EPP_MATRIX_PART == -1 || EPP_MATRIX_PART == 2
int launch_matrix_part2(const ScoreArgs& a, cudaStream_t s, int sm_count) { return launch_matrix_seq<true, false>(a, s, sm_count); }
#endif
#if EPP_MATRIX_PART == -1 || EPP_MATRIX_PART == 3
int launch_matrix_part3(const ScoreArgs& a, cudaStream_t s, int sm_count) { return launch_matrix_seq<true, true>(a, s, sm_count); }
#endif
#if EPP_MATRIX_PART == -1 || EPP_MATRIX_PART == 4
int launch_matrix_part4(const ScoreArgs& a, cudaStream_t s, int sm_count) { return launch_matrix_topk<false, false>(a, s, sm_count); }
#endif
#if EPP_MATRIX_PART == -1 || EPP_MATRIX_PART == 5
int launch_matrix_part5(const ScoreArgs& a, cudaStream_t s, int sm_count) { return launch_matrix_topk<false, true>(a, s, sm_count); }
#endif
#if EPP_MATRIX_PART == -1 || EPP_MATRIX_PART == 6
int launch_matrix_part6(const ScoreArgs& a, cudaStream_t s, int sm_count) { return launch_matrix_topk<true, false>(a, s, sm_count); }
#endif
#if EPP_MATRIX_PART == -1 || EPP_MATRIX_PART == 7
int launch_matrix_part7(const ScoreArgs& a, cudaStream_t s, int sm_count) { return launch_matrix_topk<true, true>(a, s, sm_count); }
#endif

#if EPP_MATRIX_PART == -1 || EPP_MATRIX_PART == 0
// every (request, endpoint) pair scored; any plan without pair columns
int launch_score_matrix(const ScoreArgs& a, cudaStream_t s, int sm_count) {
  if (a.R <= 0) return 0;
  const bool diag = a.match_out != nullptr || a.scores_out != nullptr || a.lat.pred_out != nullptr;  // diagnostics variants keep the R x M stores out of the hot loop
  if (a.topk > 0)
    return a.cand_mask ? (diag ? launch_matrix_part7(a, s, sm_count) : launch_matrix_part6(a, s, sm_count))
                       : (diag ? launch_matrix_part5(a, s, sm_count) : launch_matrix_part4(a, s, sm_count));
  if (a.cand_mask) return diag ? launch_matrix_part3(a, s, sm_count) : launch_matrix_part2(a, s, sm_count);
  return diag ? launch_matrix_part1(a, s, sm_count) : launch_matrix_part0(a, s, sm_count);
}
#endif

}  // namespace eppscore
