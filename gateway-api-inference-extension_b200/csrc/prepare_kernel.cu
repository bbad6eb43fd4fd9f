// prepare_kernel.cu — per-SNAPSHOT work (never per request): turns one metrics snapshot into
//   (1) prepare_endpoints_kernel: the request-independent scorer terms clamp(score)*weight per endpoint
//       (kvcache_utilization.go:76-82, queue.go:78-108, runningrequest.go:78-108, custom columns) and
//       their folded leading runs;
//   (2) prepare_adapters_kernel (one CTA per LoRA adapter row): the 2-bit LoRA class planes
//       (lora_affinity.go:84-99 precedence) and — for the sparse fast path — the arg-max summary of the
//       zero-prefix-match score map G[a][m] (max, arg, count, tie mask).
#include "device_common.cuh"
#include "lat_pair.cuh"

namespace eppscore {

// Whether endpoint m is in the profile's endpoint subset (every endpoint without one).  A subset is the head of the profile's
// filter chain, so everything computed "over all endpoints" below is computed over the members.
__device__ __forceinline__ bool is_member(const uint32_t* member, int m) {
  return !member || ((__ldg(member + (m >> 5)) >> (m & 31)) & 1u);
}

__global__ void __launch_bounds__(1024) prepare_endpoints_kernel(const __grid_constant__ PrepareArgs a) {
  __shared__ long long s_red[2][2][32];  // [queue|running][min|max][warp]
  __shared__ long long s_mm[2][2];
  const int M = a.geo.M, Mpad = a.geo.Mpad;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // min / max of WaitingQueueSize and RunningRequestsSize over the profile's endpoints (queue.go:79-91)
  for (int which = 0; which < 2; which++) {
    const int64_t* q = which == 0 ? a.queue : a.running;
    long long mn = 0x7fffffffffffffffLL, mx = (long long)0x8000000000000000ULL;
    if (q)
      for (int m = tid; m < M; m += blockDim.x) {
        if (!is_member(a.member, m)) continue;
        const long long v = q[m];
        mn = v < mn ? v : mn;
        mx = v > mx ? v : mx;
      }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      const long long omn = shfl_xor_i64(mn, o), omx = shfl_xor_i64(mx, o);
      mn = omn < mn ? omn : mn;
      mx = omx > mx ? omx : mx;
    }
    if (lane == 0) {
      s_red[which][0][warp] = mn;
      s_red[which][1][warp] = mx;
    }
  }
  __syncthreads();
  if (tid < 4) {
    const int which = tid >> 1, isx = tid & 1;
    long long v = s_red[which][isx][0];
    for (int w = 1; w < (int)(blockDim.x >> 5); w++) {
      const long long o = s_red[which][isx][w];
      v = isx ? (o > v ? o : v) : (o < v ? o : v);
    }
    s_mm[which][isx] = v;
  }
  __syncthreads();

  // value buckets for the masked min/max (kernels.cuh: QBucketHdr)
  for (int which = 0; which < 2; which++) {
    QBucketHdr* hdr = a.qhdr[which];
    if (!hdr) continue;
    const int64_t* q = which == 0 ? a.queue : a.running;
    const long long mn = s_mm[which][0], mx = s_mm[which][1];
    const bool ok = q && M > 0 && mx >= mn && (unsigned long long)(mx - mn) < (unsigned long long)kQBuckets;
    const int MW = Mpad >> 5;
    uint32_t* tbl = a.qbucket[which];
    if (ok)
      for (int i = tid; i < kQBuckets * MW; i += blockDim.x) tbl[i] = 0;
    if (tid < 8) hdr->occ[tid] = 0;
    if (tid == 0) {
      hdr->base = mn;
      hdr->valid = ok ? 1 : 0;
    }
    __syncthreads();
    if (ok)
      for (int m = tid; m < M; m += blockDim.x) {
        if (!is_member(a.member, m)) continue;  // (the masked kernels only see members: their rows carry the subset)
        const int v = (int)(q[m] - mn);
        atomicOr(&tbl[v * MW + (m >> 5)], 1u << (m & 31));
        atomicOr(&hdr->occ[v >> 5], 1u << (v & 31));
      }
  }

  // per-scorer terms: clamp(score) * weight — the rounded product of scheduler_profile.go:168.
  // Each thread keeps its endpoints' terms in registers to fold the leading runs without a re-read.
  for (int m = tid; m < Mpad; m += blockDim.x) {
    double fold_u = 0.0, fold_m = 0.0;
    for (int s = 0; s < a.n_scorers; s++) {
      double* out = a.term[s];
      if (!out) continue;
      const int kind = a.kind[s];
      double sc = 0.0;
      if (m < M) {
        if (kind == 1) {
          sc = __dsub_rn(1.0, a.kv[m]);                                            // kvcache_utilization.go:79
        } else if (kind == 0 || kind == 4) {
          const int which = kind == 0 ? 0 : 1;
          const int64_t* q = which == 0 ? a.queue : a.running;
          const long long mn = s_mm[which][0], mx = s_mm[which][1];
          if (!q || mx == mn)
            sc = 1.0;                                                               // queue.go:95-98
          else
            sc = __ddiv_rn(__ll2double_rn(mx - q[m]), __ll2double_rn(mx - mn));    // queue.go:99
        } else if (kind == 6) {                                                      // token_load.go:96-106
          double load = a.tokens ? __ll2double_rn(a.tokens[m]) : 0.0;
          if (load <= 0.0) {
            sc = 1.0;
          } else {
            if (load > a.token_threshold) load = a.token_threshold;
            sc = __dsub_rn(1.0, __ddiv_rn(load, a.token_threshold));
          }
        } else {
          const double* col = a.col[kind - 8];
          sc = col ? col[m] : 0.0;
        }
      }
      const double t = (m < M) ? __dmul_rn(clamp01(sc), a.weight[s]) : 0.0;
      out[m] = t;
      // folded leading runs: ((0.0 + t0) + t1) + ... in scorer order
      if (s < a.fold_unmasked_n) fold_u = __dadd_rn(fold_u, t);
      if (s < a.fold_masked_n) fold_m = __dadd_rn(fold_m, t);
    }
    if (a.fold_unmasked) a.fold_unmasked[m] = fold_u;
    if (a.fold_masked) a.fold_masked[m] = fold_m;
    // latency fold-in: the endpoint-only prefixes of the two linear forms (prediction.go:171-185 evaluates
    // left to right, so "intercept + c_kv*kv" is a rounded partial sum and the products are rounded terms)
    if (a.lat_ep) {
      const double kv = m < M ? a.kv[m] : 0.0;
      const long long qi = (m < M && a.queue) ? a.queue[m] : 0;
      const double wt = __ll2double_rn(qi);
      const double rn = (m < M && a.running) ? __ll2double_rn(a.running[m]) : 0.0;
      const double pod_min = (m < M && a.min_tpot) ? a.min_tpot[m] : 0.0;
      double* tile = a.lat_ep + (size_t)(m >> 5) * 256 + (m & 31);  // slot i at tile[i*32] (kernels.cuh: LatArgs)
      if (a.lat_has_predictions) {
        tile[0 * 32] = __dadd_rn(a.lat_coef[0], __dmul_rn(a.lat_coef[1], kv));
        tile[1 * 32] = __dmul_rn(a.lat_coef[2], wt);
        tile[2 * 32] = __dmul_rn(a.lat_coef[3], rn);
        tile[3 * 32] = __dadd_rn(a.lat_coef[4], __dmul_rn(a.lat_coef[5], kv));
        tile[4 * 32] = __dmul_rn(a.lat_coef[6], wt);
        tile[5 * 32] = __dmul_rn(a.lat_coef[7], rn);
        tile[6 * 32] = lat_lim(pod_min, a.lat_buffer);
        const bool idle = lat_idle((m < M && a.dispatched) ? a.dispatched[m] : 0);
        const bool neutral = !a.lat_streaming || (m < M && a.prefill && a.prefill[m]);
        tile[7 * 32] = __longlong_as_double((long long)((idle ? 1 : 0) | (neutral ? 2 : 0)));
      } else {
        tile[0 * 32] = __dmul_rn(a.lat_ckv, __dsub_rn(1.0, kv));                    // plugin.go:351,355
        tile[1 * 32] = __longlong_as_double(qi);                                     // raw WaitingQueueSize
      }
    }
  }
}

constexpr int kAdapterThreads = 1024;  // one endpoint per thread at M = 1024: the kernel is latency bound, not work bound

__global__ void __launch_bounds__(kAdapterThreads) prepare_adapters_kernel(const __grid_constant__ PrepareArgs a) {
  extern __shared__ uint32_t s_u32[];  // [3][row_words]: class lo plane, hi plane, tie mask
  __shared__ double s_bs[kAdapterThreads / 32];
  __shared__ int s_bm[kAdapterThreads / 32], s_bc[kAdapterThreads / 32];
  __shared__ double s_gmax;
  const int rw = a.geo.row_words, log_epl = a.geo.log_epl;
  const int M = a.geo.M;
  const int ai = blockIdx.x;  // adapter row; row A = "adapter not in the dictionary"
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t* s_lo = s_u32;
  uint32_t* s_hi = s_u32 + rw;
  uint32_t* s_tie = s_u32 + 2 * rw;

  // LoRA class planes: class 3 active, 2 has capacity, 1 waiting, 0 none (lora_affinity.go:84-99).
  // One thread per endpoint (coalesced reads of the snapshot), bits merged into the permuted planes in smem.
  for (int word = tid; word < 3 * rw; word += blockDim.x) s_u32[word] = 0;
  __syncthreads();
  for (int m = tid; m < M; m += blockDim.x) {
    bool active = false, waiting = false;
    if (ai < a.A && a.act && a.wait) {
      const uint64_t bit = 1ULL << (ai & 63);
      active = (a.act[(size_t)m * a.lora_words + (ai >> 6)] & bit) != 0;
      waiting = (a.wait[(size_t)m * a.lora_words + (ai >> 6)] & bit) != 0;
    }
    const int nm = a.nmodels ? a.nmodels[m] : 0, mxm = a.maxm ? a.maxm[m] : 0;
    const int cls = active ? 3 : (nm < mxm ? 2 : (waiting ? 1 : 0));
    const uint32_t pos = perm_bitpos((uint32_t)m, log_epl);
    if (cls & 1) atomicOr(&s_lo[pos >> 5], 1u << (pos & 31));
    if (cls & 2) atomicOr(&s_hi[pos >> 5], 1u << (pos & 31));
  }
  __syncthreads();
  for (int word = tid; word < rw; word += blockDim.x) {
    a.cls_lo[(size_t)ai * rw + word] = s_lo[word];
    a.cls_hi[(size_t)ai * rw + word] = s_hi[word];
  }
  if (!a.summ) return;
  __syncthreads();

  // G[ai][m]: the weighted score with zero prefix match, steps in profile order; arg-max over the profile's endpoints (the
  // exactness argument of pick_sparse.cu holds over the member set: non-members are never candidates, exceptions included)
  auto score_of = [&](int m) {
    const uint32_t pos = perm_bitpos((uint32_t)m, log_epl);
    const int cls = (int)((s_lo[pos >> 5] >> (pos & 31)) & 1u) | ((int)((s_hi[pos >> 5] >> (pos & 31)) & 1u) << 1);
    return eval_steps(a.plan_u, a.plan_term, m, 0, 0, cls);
  };
  Best b = best_none();
  for (int m = tid; m < M; m += blockDim.x)
    if (is_member(a.member, m)) best_update(b, score_of(m), m, 0, 0, 0);
  best_group_reduce<32>(b, 0);
  if (lane == 0) {
    s_bs[warp] = b.score;
    s_bm[warp] = b.m;
    s_bc[warp] = b.cnt;
  }
  __syncthreads();
  if (tid == 0) {
    Best t = best_none();
    for (int w = 0; w < kAdapterThreads / 32; w++) best_merge(t, s_bs[w], s_bm[w], s_bc[w], 0, 0);
    AdapterSummary sm;
    sm.gmax = t.m >= 0 ? t.score : 0.0;
    sm.garg = t.m;
    sm.gcnt = t.cnt;
    a.summ[ai] = sm;
    s_gmax = sm.gmax;
  }
  __syncthreads();
  const double gmax = s_gmax;
  for (int m = tid; m < M; m += blockDim.x)
    if (is_member(a.member, m) && score_of(m) == gmax) {
      const uint32_t pos = perm_bitpos((uint32_t)m, log_epl);
      atomicOr(&s_tie[pos >> 5], 1u << (pos & 31));
    }
  __syncthreads();
  for (int word = tid; word < rw; word += blockDim.x) a.tiemask[(size_t)ai * rw + word] = s_tie[word];
}

int launch_prepare_snapshot(const PrepareArgs& a, cudaStream_t s) {
  prepare_endpoints_kernel<<<1, 1024, 0, s>>>(a);
  prepare_adapters_kernel<<<a.A + 1, kAdapterThreads, 3 * a.geo.row_words * sizeof(uint32_t), s>>>(a);
  return 2;
}

}  // namespace eppscore
