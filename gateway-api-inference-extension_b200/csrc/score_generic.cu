// score_generic.cu — the fully general DENSE-ROW Score+Pick kernel: any scorer order, candidate masks,
// pair columns, diagnostics outputs, runtime step dispatch.  It is the fallback of score_dense.cu's
// specialised streaming kernels; the full-matrix kernel for prompt-driven batches is score_matrix.cu.
//   matchLongestPrefix  approximateprefix/plugin.go:219-235
//   scorers + sum       scheduler_profile.go:151-174 (+ the four Score bodies)
//   picker              maxscore/picker.go:87-115
#include "device_common.cuh"

namespace eppscore {

// ---------------------------------------------------------------------------------------------
// Score + Pick
// ---------------------------------------------------------------------------------------------
constexpr int kScoreWarps = 8;

// Dense rows: float4 {matchBlocks, lora class, pair0, pair1} per (request, endpoint), streamed with
// coalesced 128-bit loads (lane l reads endpoint i*32+l); endpoint tile in shared memory.
// TOPK: the first a.topk entries of each request's max-score order are written too.
template <bool MASKED, bool TOPK = false>
__global__ void __launch_bounds__(kScoreWarps * 32) score_pick_dense_kernel(const __grid_constant__ ScoreArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Plan& plan = a.plan;
  const int M = a.geo.M;
  const int MP = (M + 31) & ~31;
  double* s_term = reinterpret_cast<double*>(smem_raw);
  long long* s_q = reinterpret_cast<long long*>(s_term + (size_t)plan.n_terms * MP);
  double* s_lut = reinterpret_cast<double*>(s_q + (MASKED ? 2 * MP : 0));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int t = 0; t < plan.n_terms; t++)
    for (int m = threadIdx.x; m < MP; m += blockDim.x) s_term[(size_t)t * MP + m] = m < M ? a.term[t][m] : 0.0;
  if (MASKED)
    for (int which = 0; which < 2; which++)
      for (int m = threadIdx.x; m < MP; m += blockDim.x)
        s_q[which * MP + m] = (a.minmax_q[which] && m < M) ? a.minmax_q[which][m] : 0;
  __syncthreads();

  double* lut = s_lut + warp * (kLutMax + 1);
  int lut_total = -1, prefix_step = -1;
  bool has_minmax[2] = {false, false};
  for (int s = 0; s < plan.n_steps; s++) {
    if (plan.kind[s] == STEP_PREFIX && prefix_step < 0) prefix_step = s;
    if (plan.kind[s] == STEP_MINMAX) has_minmax[plan.arg[s]] = true;
  }
  const int tie_mode = plan.tie_mode;
  const int nchunks = MP >> 5;

  const int gw = blockIdx.x * kScoreWarps + warp, nw = gridDim.x * kScoreWarps;
  for (int r = gw; r < a.R; r += nw) {
    const int total = a.dense_total ? a.dense_total[r] : 0;
    if (prefix_step >= 0 && total != lut_total) {
      const double w = plan.weight[prefix_step];
      const int top = total < kLutMax ? total : kLutMax;
      __syncwarp();
      for (int c = lane; c <= top; c += 32) lut[c] = prefix_term_direct(c, total, w);
      lut_total = total;
      __syncwarp();
    }
    const uint32_t* mrow = MASKED ? a.cand_mask + (size_t)r * a.mask_words : nullptr;
    long long mn[2] = {0, 0}, mx[2] = {0, 0};
    if (MASKED && (has_minmax[0] || has_minmax[1])) {
      mn[0] = mn[1] = 0x7fffffffffffffffLL;
      mx[0] = mx[1] = (long long)0x8000000000000000ULL;
      for (int i = 0; i < nchunks; i++) {
        const int m = i * 32 + lane;
        if (((__ldg(mrow + i) >> lane) & 1u) && m < M) {
#pragma unroll
          for (int which = 0; which < 2; which++) {
            const long long v = s_q[which * MP + m];
            mn[which] = v < mn[which] ? v : mn[which];
            mx[which] = v > mx[which] ? v : mx[which];
          }
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
    }
    const uint32_t areq = tie_areq(a.request_base + r, plan.seed_lo);
    Best best = best_none();
    TopK tk;
    if (TOPK) topk_clear(tk);
    const float4* row = a.dense + (size_t)r * M;
#pragma unroll 4
    for (int i = 0; i < nchunks; i++) {
      const int m = i * 32 + lane;
      bool cand = m < M;
      float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
      if (cand) f = __ldg(row + m);
      if (MASKED) cand = cand && ((__ldg(mrow + i) >> lane) & 1u);
      const int c = (int)(__float2uint_rz(f.x) & 0xFFFFu);
      const int cls = __float2int_rz(f.y) & 3;
      if (a.match_out && m < M) a.match_out[(size_t)r * M + m] = (uint16_t)c;
      double acc = 0.0;
      for (int s = 0; s < plan.n_steps; s++) {
        double term;
        switch (plan.kind[s]) {
          case STEP_EP_TERM: term = s_term[(size_t)plan.arg[s] * MP + m]; break;
          case STEP_PREFIX: {
            const int cc = c < 65535 ? c : 65535;
            term = (s == prefix_step && total <= kLutMax && cc <= total) ? lut[cc]
                                                                          : prefix_term_direct(cc, total, plan.weight[s]);
            break;
          }
          case STEP_LORA: {
              const double* lt = plan.lora_term[s];
              term = cls == 3 ? lt[3] : (cls == 2 ? lt[2] : (cls == 1 ? lt[1] : lt[0]));
              break;
            }
          case STEP_PAIR:
            term = __dmul_rn(clamp01((double)(plan.arg[s] == 0 ? f.z : f.w)), plan.weight[s]);
            break;
          case STEP_MINMAX: {
            const int which = plan.arg[s];
            double sc = 1.0;
            if (MASKED && mx[which] != mn[which])
              sc = __ddiv_rn(__ll2double_rn(mx[which] - s_q[which * MP + m]), __ll2double_rn(mx[which] - mn[which]));
            term = __dmul_rn(clamp01(sc), plan.weight[s]);
            break;
          }
          default: term = 0.0; break;
        }
        acc = __dadd_rn(acc, term);
      }
      if (a.scores_out && m < M) a.scores_out[(size_t)r * M + m] = cand ? acc : nan64();
      if (cand) best_update(best, acc, m, tie_mode, areq, plan.seed_hi);
      if (TOPK && cand) {
        double key;
        unsigned long long ord;
        topk_key(0, tie_mode, acc, tie_prio(areq, m, plan.seed_hi), m, key, ord);
        topk_insert(tk, a.topk, key, ord, acc);
      }
    }
    best_group_reduce<32>(best, tie_mode);
    if (TOPK) {
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
  }
}

template <typename K>
static int launch_with_smem(K kernel, const ScoreArgs& a, size_t smem, cudaStream_t s, int sm_count) {
  cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  int occ = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, kScoreWarps * 32, smem);
  if (occ < 1) occ = 1;
  const int need = (a.R + kScoreWarps - 1) / kScoreWarps;
  int blocks = sm_count * occ;  // persistent: one wave, warps stride over requests
  if (blocks > need) blocks = need;
  if (blocks < 1) blocks = 1;
  kernel<<<blocks, kScoreWarps * 32, smem, s>>>(a);
  return 1;
}

int launch_score_pick(const ScoreArgs& a, bool dense, cudaStream_t s, int sm_count) {
  if (a.R <= 0) return 0;
  const bool masked = a.cand_mask != nullptr;
  if (dense) {
    const int MP = (a.geo.M + 31) & ~31;
    size_t smem = (size_t)a.plan.n_terms * MP * 8 + (masked ? 2 * (size_t)MP * 8 : 0) +
                  (size_t)kScoreWarps * (kLutMax + 1) * 8;
    if (a.topk > 0)
      return masked ? launch_with_smem(score_pick_dense_kernel<true, true>, a, smem, s, sm_count)
                    : launch_with_smem(score_pick_dense_kernel<false, true>, a, smem, s, sm_count);
    if (masked) return launch_with_smem(score_pick_dense_kernel<true>, a, smem, s, sm_count);
    return launch_with_smem(score_pick_dense_kernel<false>, a, smem, s, sm_count);
  }
  return launch_score_matrix(a, s, sm_count);  // score_matrix.cu
}

}  // namespace eppscore
