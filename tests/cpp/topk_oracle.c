/*
 * topk_oracle.c — TEST INFRASTRUCTURE ONLY: maxNumOfEndpoints (picker/common.go:39-42) restated on the CPU oracle's
 * counter-based generator (oracle/oracle.h: orc_tie_priority, orc_uniform01, orc_neg_log).  Built by tests/topk_oracle.py
 * into tests/cpp/_build/libtopk_oracle.so; the checker of the engine's eppscore_schedule_batch_topk lists and the
 * stand-in behind the host layer's CPU tests (tests/cpp/oracle_backed_topk.cpp).  Written from the reference pickers,
 * not from the kernels.
 *
 * topk_oracle_pick: the first min(k, |C|) endpoints of the profile's picker over the candidates
 * C = {m : weighted[m] is not NaN} (weighted = orc_schedule_one's weighted_out), written to m_out[0..k) / score_out[0..k)
 * and padded with -1 / 0.0.  Returns |C| clipped to k.  Each order is one outcome of the reference's own distribution,
 * the shuffles drawn from orc_tie_priority:
 *   max-score (maxscore/picker.go:91-107: shuffle, stable sort by descending score, first k): descending score; inside
 *     a tie class ascending index (TIE_LOWEST_INDEX) or descending tie priority, then ascending index (TIE_SEEDED_RANDOM)
 *   weighted-random (weightedrandom/picker.go:121-152: the k largest A-Res keys U^(1/score)): the candidates with
 *     score > 0 by ascending -ln(U)/score, then ascending index; then those with score <= 0 (key 0, :126-129) in
 *     random-picker order.  No positive score: the random picker (:113-116)
 *   random (random/picker.go:90-96: the first k of a shuffle): descending priority, then ascending index
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include "../../oracle/oracle.h"

typedef struct topk_ent {
  int32_t m;
  int32_t cls;   /* weighted-random: 0 score > 0, 1 score <= 0 (key 0); 0 otherwise */
  int32_t by;    /* 0 descending score, 1 ascending key, 2 descending priority */
  uint32_t prio; /* orc_tie_priority (0 under TIE_LOWEST_INDEX for max-score) */
  double key;    /* by 1: -ln(U)/score */
  double score;
} topk_ent;

static int topk_cmp(const void *pa, const void *pb) {
  const topk_ent *a = (const topk_ent *)pa, *b = (const topk_ent *)pb;
  if (a->cls != b->cls) return a->cls < b->cls ? -1 : 1;
  if (a->by == 0 && a->score != b->score) return a->score > b->score ? -1 : 1;
  if (a->by == 1 && a->key != b->key) return a->key < b->key ? -1 : 1;
  if (a->by != 1 && a->prio != b->prio) return a->prio > b->prio ? -1 : 1;
  return a->m < b->m ? -1 : (a->m > b->m ? 1 : 0);
}

int32_t topk_oracle_pick(const double *weighted, int32_t M, int32_t pick_mode, int32_t tie_mode, uint64_t tie_seed,
                         int64_t request_index, int32_t k, int32_t *m_out, double *score_out) {
  for (int32_t i = 0; i < k; i++) {
    m_out[i] = -1;
    score_out[i] = 0.0;
  }
  topk_ent *v = (topk_ent *)malloc(sizeof(topk_ent) * (size_t)(M > 0 ? M : 1));
  int32_t n = 0;
  for (int32_t m = 0; m < M; m++) {
    const double w = weighted[m];
    if (isnan(w)) continue;
    topk_ent *e = &v[n++];
    e->m = m;
    e->score = w;
    e->cls = 0;
    e->key = 0;
    e->prio = orc_tie_priority(tie_seed, request_index, m);
    if (pick_mode == ORC_PICK_MAX_SCORE) {
      e->by = 0;
      if (tie_mode != ORC_TIE_SEEDED_RANDOM) e->prio = 0;
    } else if (pick_mode == ORC_PICK_WEIGHTED_RANDOM && w > 0) {
      e->by = 1;
      e->key = orc_neg_log(orc_uniform01(tie_seed, request_index, m)) / w;
    } else {
      e->by = 2;
      e->cls = pick_mode == ORC_PICK_WEIGHTED_RANDOM;
    }
  }
  qsort(v, (size_t)n, sizeof(topk_ent), topk_cmp);
  const int32_t out = n < k ? n : k;
  for (int32_t i = 0; i < out; i++) {
    m_out[i] = v[i].m;
    score_out[i] = v[i].score;
  }
  free(v);
  return out;
}
