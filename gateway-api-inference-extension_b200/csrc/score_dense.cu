// score_dense.cu — Score+Pick over caller-supplied feature rows, specialised per scorer sequence.
//
// Input: float4 per (request, endpoint) = {matchBlocks, lora class, pair col 0, pair col 1}, R x M rows in
// HBM (16*R*M bytes — the kernel is a pure stream over them: DESIGN.md §6 "dense-row accounting").
// One warp per request row; lane l reads endpoint i*32+l with a 128-bit coalesced load, four loads in
// flight per lane; the endpoint tile (folded request-independent terms), the per-step LoRA terms and a
// per-warp prefix LUT live in shared memory; float64 accumulate in profile order
// (scheduler_profile.go:155-168); warp-shuffle arg-max (maxscore/picker.go:87-115).  The scorer sequence
// is a template parameter pack, so the inner loop has no dispatch; sequences without a specialisation
// fall back to score_generic.cu.
#include "device_common.cuh"

namespace eppscore {

constexpr int kDenseWarps = 8;

struct DenseCtx {
  const double* s_term;  // [n_terms][MP]
  const double* s_lora;  // [kMaxSteps][4]
  const double* lut;     // per warp [kLutMax+1]
  int MP;
  int total;
  const Plan* plan;
};

template <int KIND, bool LUT_OK>
__device__ __forceinline__ double dense_term(const DenseCtx& cx, int s, int m, const float4& f, int c, int cls) {
  if (KIND == STEP_EP_TERM) return cx.s_term[cx.plan->arg[s] * cx.MP + m];
  if (KIND == STEP_PREFIX) return LUT_OK ? cx.lut[c] : prefix_term_direct(c, cx.total, cx.plan->weight[s]);
  if (KIND == STEP_LORA) return cx.s_lora[s * 4 + cls];
  // STEP_PAIR: float32 feature widened exactly, clamped, weighted
  return __dmul_rn(clamp01((double)(cx.plan->arg[s] == 0 ? f.z : f.w)), cx.plan->weight[s]);
}

template <bool LUT_OK, int... KINDS>
__device__ __forceinline__ void dense_pair(const DenseCtx& cx, const float4& f, int m, Best& best, int tie_mode,
                                           uint32_t areq, uint32_t seed_hi) {
  int c = (int)(__float2uint_rz(f.x) & 0xFFFFu);
  if (LUT_OK) c = c < cx.total ? c : cx.total;  // match > total clamps to score 1 == lut[total]
  const int cls = __float2int_rz(f.y) & 3;
  double acc = 0.0;  // weightedScorePerEndpoint[endpoint] = float64(0)
  int s = 0;
  ((acc = __dadd_rn(acc, dense_term<KINDS, LUT_OK>(cx, s, m, f, c, cls)), s++), ...);
  best_update(best, acc, m, tie_mode, areq, seed_hi);
}

// one request row: full 32-endpoint chunks with four 128-bit loads in flight, then the ragged tail
template <bool LUT_OK, int... KINDS>
__device__ __forceinline__ void dense_row(const DenseCtx& cx, const float4* __restrict__ row, int M, int lane, Best& best,
                                          int tie_mode, uint32_t areq, uint32_t seed_hi) {
  const int nfull = M >> 5;
  int i = 0;
  for (; i + 4 <= nfull; i += 4) {
    float4 f[4];
#pragma unroll
    for (int u = 0; u < 4; u++) f[u] = __ldg(row + (i + u) * 32 + lane);
#pragma unroll
    for (int u = 0; u < 4; u++) dense_pair<LUT_OK, KINDS...>(cx, f[u], (i + u) * 32 + lane, best, tie_mode, areq, seed_hi);
  }
  for (; i < nfull; i++) dense_pair<LUT_OK, KINDS...>(cx, __ldg(row + i * 32 + lane), i * 32 + lane, best, tie_mode, areq, seed_hi);
  const int m = nfull * 32 + lane;
  if (m < M) dense_pair<LUT_OK, KINDS...>(cx, __ldg(row + m), m, best, tie_mode, areq, seed_hi);
}

template <int... KINDS>
__global__ void __launch_bounds__(kDenseWarps * 32) score_dense_fast_kernel(const __grid_constant__ ScoreArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Plan& plan = a.plan;
  const int M = a.geo.M;
  const int MP = (M + 31) & ~31;
  double* s_term = reinterpret_cast<double*>(smem_raw);
  double* s_lora = s_term + (size_t)plan.n_terms * MP;
  double* s_lut = s_lora + kMaxSteps * 4;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // stage the endpoint tile once per CTA
  for (int t = 0; t < plan.n_terms; t++)
    for (int m = threadIdx.x; m < MP; m += blockDim.x) s_term[(size_t)t * MP + m] = m < M ? a.term[t][m] : 0.0;
  if (threadIdx.x < kMaxSteps * 4) s_lora[threadIdx.x] = plan.lora_term[threadIdx.x >> 2][threadIdx.x & 3];
  __syncthreads();

  double* lut = s_lut + warp * (kLutMax + 1);
  int prefix_step = -1;
  {
    int s = 0;
    ((prefix_step = (KINDS == STEP_PREFIX && prefix_step < 0) ? s : prefix_step, s++), ...);
  }
  int lut_total = -1;
  const int tie_mode = plan.tie_mode;
  DenseCtx cx;
  cx.s_term = s_term;
  cx.s_lora = s_lora;
  cx.lut = lut;
  cx.MP = MP;
  cx.plan = &plan;

  const int gw = blockIdx.x * kDenseWarps + warp, nw = gridDim.x * kDenseWarps;
  for (int r = gw; r < a.R; r += nw) {
    const int total = a.dense_total ? a.dense_total[r] : 0;
    const bool lut_ok = prefix_step < 0 || total <= kLutMax;  // larger totals divide per pair (rare: > 256 blocks)
    if (prefix_step >= 0 && lut_ok && total != lut_total) {
      const double w = plan.weight[prefix_step];
      __syncwarp();
      for (int c = lane; c <= total; c += 32) lut[c] = prefix_term_direct(c, total, w);
      lut_total = total;
      __syncwarp();
    }
    cx.total = total;
    const uint32_t areq = tie_areq(a.request_base + r, plan.seed_lo);
    Best best = best_none();
    const float4* row = a.dense + (size_t)r * M;
    if (lut_ok)
      dense_row<true, KINDS...>(cx, row, M, lane, best, tie_mode, areq, plan.seed_hi);
    else
      dense_row<false, KINDS...>(cx, row, M, lane, best, tie_mode, areq, plan.seed_hi);
    best_group_reduce<32>(best, tie_mode);
    if (lane == 0) {
      a.pick[r] = best.m;
      a.pick_score[r] = best.m >= 0 ? best.score : 0.0;
      a.tie_count[r] = best.cnt;
      if (a.total_out) a.total_out[r] = (uint16_t)total;
    }
  }
}

template <typename K>
static int launch_dense(K kernel, const ScoreArgs& a, cudaStream_t s, int sm_count) {
  const int MP = (a.geo.M + 31) & ~31;
  const size_t smem = (size_t)a.plan.n_terms * MP * 8 + kMaxSteps * 4 * 8 + (size_t)kDenseWarps * (kLutMax + 1) * 8;
  const cudaError_t c = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (c != cudaSuccess) return -(int)c;
  int occ = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, kDenseWarps * 32, smem);
  if (occ < 1) occ = 1;
  int blocks = sm_count * occ;
  const int need = (a.R + kDenseWarps - 1) / kDenseWarps;
  if (blocks > need) blocks = need;
  if (blocks < 1) blocks = 1;
  return launched_one(launch_maybe_pdl(false, kernel, dim3(blocks), dim3(kDenseWarps * 32), smem, s, a));
}

constexpr uint32_t seq_of() { return 0; }
template <typename... Rest>
constexpr uint32_t seq_of(int k, Rest... rest) {
  return (uint32_t)(k + 1) | (seq_of(rest...) << 4);
}

#define E STEP_EP_TERM
#define P STEP_PREFIX
#define L STEP_LORA
#define X STEP_PAIR
// Unmasked batches without per-pair diagnostics only; returns 0 when no specialisation matches.
int launch_score_dense_fast(const ScoreArgs& a, cudaStream_t s, int sm_count) {
  if (a.R <= 0 || !a.dense || a.cand_mask || a.match_out || a.scores_out || a.topk > 0) return 0;
  switch (a.plan.seq) {
    case seq_of(E): return launch_dense(score_dense_fast_kernel<E>, a, s, sm_count);
    case seq_of(E, P): return launch_dense(score_dense_fast_kernel<E, P>, a, s, sm_count);
    case seq_of(E, L): return launch_dense(score_dense_fast_kernel<E, L>, a, s, sm_count);
    case seq_of(L, E): return launch_dense(score_dense_fast_kernel<L, E>, a, s, sm_count);
    case seq_of(E, P, L): return launch_dense(score_dense_fast_kernel<E, P, L>, a, s, sm_count);
    case seq_of(E, P, L, X): return launch_dense(score_dense_fast_kernel<E, P, L, X>, a, s, sm_count);
    case seq_of(E, P, L, X, X): return launch_dense(score_dense_fast_kernel<E, P, L, X, X>, a, s, sm_count);
    case seq_of(P): return launch_dense(score_dense_fast_kernel<P>, a, s, sm_count);
    case seq_of(P, L): return launch_dense(score_dense_fast_kernel<P, L>, a, s, sm_count);
    default: return 0;
  }
}
#undef E
#undef P
#undef L
#undef X

}  // namespace eppscore
