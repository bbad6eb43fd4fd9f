/* inflight_oracle.c — TEST INFRASTRUCTURE ONLY: the inflight-load-producer restated on the CPU, the reference the engine's
 * in-flight counters and token estimator are checked against (tests/inflight_oracle.py binds it).
 *
 *   orc_estimate_tokens   SimpleTokenEstimator.Estimate       requestcontrol/dataproducer/inflightload/token_estimator.go:48-72
 *   orc_inflight_add      PreRequest                          producer.go:101-120 (TargetEndpoints[0], requestTracker.inc,
 *                                                             tokenTracker.add(estimate))
 *   orc_inflight_release  ResponseBody, EndOfStream           producer.go:122-169 (release: dec, add(-estimate))
 *   orc_inflight_remove   DeleteEndpoint                      producer.go:181-187
 *   orc_inflight_get      PrepareRequestData                  producer.go:90-99 (get: 0 for an endpoint without a counter)
 *
 * The trackers are concurrencyTracker (producer.go:189-247): a map from endpoint to counter; add() on a missing key creates
 * the counter holding the delta (:226-236), delete() drops it (:243-247).  Endpoints are the engine's integer ids here.
 * The estimator is written the way the Go code computes it, in float64 with a half-away-from-zero round (math.Round), with
 * the factory's defaults 4.0 and 1.5 (producer.go:40-47, token_estimator.go:37-42) — not in the engine's integer form. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

int64_t orc_estimate_tokens(int64_t request_size_bytes, int32_t token_hint, int32_t prompt_chars) {
  const double chars_per_token = 4.0, output_ratio = 1.5;
  int64_t input;
  if (request_size_bytes > 0) {                                 /* :55-56 */
    input = request_size_bytes / 4;
    if (input < 1) input = 1;
  } else if (prompt_chars >= 0) {                               /* Body != nil, :57-66 */
    if (token_hint >= 0) {
      input = token_hint;
    } else {
      input = (int64_t)fmax(1.0, round((double)prompt_chars / chars_per_token));  /* C round(): half away from zero */
    }
  } else {
    return 0;                                                   /* :67-68 */
  }
  const int64_t output = (int64_t)round((double)input * output_ratio);  /* :70 */
  return input + output;
}

typedef struct {
  int64_t n;         /* ids 0..n-1 have slots */
  uint8_t* present;  /* the map holds a counter for this id */
  int64_t* requests;
  int64_t* tokens;
} orc_inflight;

orc_inflight* orc_inflight_new(void) { return (orc_inflight*)calloc(1, sizeof(orc_inflight)); }

void orc_inflight_free(orc_inflight* t) {
  if (!t) return;
  free(t->present);
  free(t->requests);
  free(t->tokens);
  free(t);
}

static void grow(orc_inflight* t, int64_t id) {
  if (id < t->n) return;
  int64_t n = t->n ? t->n : 64;
  while (n <= id) n *= 2;
  t->present = (uint8_t*)realloc(t->present, (size_t)n);
  t->requests = (int64_t*)realloc(t->requests, (size_t)n * 8);
  t->tokens = (int64_t*)realloc(t->tokens, (size_t)n * 8);
  memset(t->present + t->n, 0, (size_t)(n - t->n));
  memset(t->requests + t->n, 0, (size_t)(n - t->n) * 8);
  memset(t->tokens + t->n, 0, (size_t)(n - t->n) * 8);
  t->n = n;
}

/* concurrencyTracker.add on both trackers (:216-237): an existing counter adds the delta, a missing one is created holding it */
static void tracker_add(orc_inflight* t, int32_t id, int64_t dreq, int64_t dtok) {
  grow(t, id);
  if (!t->present[id]) {
    t->present[id] = 1;
    t->requests[id] = 0;
    t->tokens[id] = 0;
  }
  t->requests[id] += dreq;
  t->tokens[id] += dtok;
}

/* one request per entry, in order; endpoint < 0 = no target endpoint (nothing to record, :106-114) */
void orc_inflight_add(orc_inflight* t, int32_t R, const int32_t* endpoint, const int64_t* tokens) {
  for (int32_t r = 0; r < R; r++)
    if (endpoint[r] >= 0) tracker_add(t, endpoint[r], 1, tokens ? tokens[r] : 0);
}

void orc_inflight_release(orc_inflight* t, int32_t R, const int32_t* endpoint, const int64_t* tokens) {
  for (int32_t r = 0; r < R; r++)
    if (endpoint[r] >= 0) tracker_add(t, endpoint[r], -1, tokens ? -tokens[r] : 0);
}

void orc_inflight_remove(orc_inflight* t, int32_t endpoint) {
  if (endpoint >= 0 && endpoint < t->n) {
    t->present[endpoint] = 0;
    t->requests[endpoint] = 0;
    t->tokens[endpoint] = 0;
  }
}

/* the first M endpoints' counters, 0 where the map has none (:201-210) */
void orc_inflight_get(const orc_inflight* t, int32_t M, int64_t* requests_out, int64_t* tokens_out) {
  for (int32_t m = 0; m < M; m++) {
    const int has = m < t->n && t->present[m];
    if (requests_out) requests_out[m] = has ? t->requests[m] : 0;
    if (tokens_out) tokens_out[m] = has ? t->tokens[m] : 0;
  }
}
