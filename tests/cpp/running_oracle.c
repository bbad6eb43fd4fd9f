/* running_oracle.c — TEST INFRASTRUCTURE ONLY: the predicted-latency producer's running-request queues restated on the CPU, the
 * reference the engine's device queues are checked against (tests/running_oracle.py binds it).
 *
 *   one queue per endpoint    requestPriorityQueue (predictedlatency/running_request_tpot_slo_queue.go:34-38): a binary
 *                             min-heap on tpot (Less, :74-76) with container/heap's up / down / Remove, plus the id lookup
 *   orc_running_add           PreRequest (requestcontrol_hooks.go:73-86) -> Add (:122-148): refused for an empty id (key 0
 *                             here), tpot < 0, or an id already in that endpoint's queue
 *   orc_running_remove        end of stream (requestcontrol_hooks.go:219) / TTL expiry (plugin.go:190-196) -> Remove (:169-181)
 *   orc_running_get           getEndpointMinTPOTSLO (plugin.go:347-355): Peek().tpot, 0 for an empty or missing queue;
 *                             getEndpointRunningRequestCount (plugin.go:357-363): GetSize()
 *   orc_running_remove_endpoint  the engine's id recycling (eppscore_running_remove_endpoint): the queue is dropped
 *
 * A batch is applied entry by entry in request order; endpoint < 0 is skipped.  The reference deletes an empty queue and
 * creates it again on the next Add: indistinguishable from an empty queue here.  Lookup: one open-addressing map from
 * (endpoint, key) to the heap position, kept up to date by every swap. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
  uint64_t key;
  double tpot;
} Item;

typedef struct {
  Item* items;
  int64_t n, cap;
} Heap;

typedef struct {
  uint64_t key;  /* 0: empty */
  int32_t ep;
  int32_t tomb;
  int64_t pos;
} MapSlot;

typedef struct {
  Heap* heaps;
  int32_t n_ep;
  MapSlot* map;
  int64_t map_cap, map_used;
} Running;

static uint64_t mix(uint64_t key, int32_t ep) {
  uint64_t x = key ^ ((uint64_t)(ep + 1) * 0x9E3779B97F4A7C15ull);
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

static MapSlot* map_find(Running* s, int32_t ep, uint64_t key) {
  for (uint64_t h = mix(key, ep) & (uint64_t)(s->map_cap - 1);; h = (h + 1) & (uint64_t)(s->map_cap - 1)) {
    MapSlot* m = &s->map[h];
    if (m->key == 0) return NULL;
    if (!m->tomb && m->key == key && m->ep == ep) return m;
  }
}

static void map_put(Running* s, int32_t ep, uint64_t key, int64_t pos);

static void map_grow(Running* s) {
  MapSlot* old = s->map;
  const int64_t oc = s->map_cap;
  s->map_cap = oc * 2;
  s->map = (MapSlot*)calloc((size_t)s->map_cap, sizeof(MapSlot));
  s->map_used = 0;
  for (int64_t i = 0; i < oc; i++)
    if (old[i].key && !old[i].tomb) map_put(s, old[i].ep, old[i].key, old[i].pos);
  free(old);
}

static void map_put(Running* s, int32_t ep, uint64_t key, int64_t pos) {
  if (2 * (s->map_used + 1) > s->map_cap) map_grow(s);
  for (uint64_t h = mix(key, ep) & (uint64_t)(s->map_cap - 1);; h = (h + 1) & (uint64_t)(s->map_cap - 1)) {
    MapSlot* m = &s->map[h];
    if (m->key == 0) {
      m->key = key;
      m->ep = ep;
      m->tomb = 0;
      m->pos = pos;
      s->map_used++;
      return;
    }
  }
}

static void set_pos(Running* s, int32_t ep, int64_t i) { map_find(s, ep, s->heaps[ep].items[i].key)->pos = i; }

static void heap_swap(Running* s, int32_t ep, int64_t i, int64_t j) { /* Swap (:78-82) */
  Heap* q = &s->heaps[ep];
  Item t = q->items[i];
  q->items[i] = q->items[j];
  q->items[j] = t;
  set_pos(s, ep, i);
  set_pos(s, ep, j);
}

static void up(Running* s, int32_t ep, int64_t j) { /* container/heap up */
  Heap* q = &s->heaps[ep];
  for (;;) {
    const int64_t i = (j - 1) / 2;
    if (i == j || !(q->items[j].tpot < q->items[i].tpot)) break;
    heap_swap(s, ep, i, j);
    j = i;
  }
}

static int down(Running* s, int32_t ep, int64_t i0, int64_t n) { /* container/heap down */
  Heap* q = &s->heaps[ep];
  int64_t i = i0;
  for (;;) {
    const int64_t j1 = 2 * i + 1;
    if (j1 >= n || j1 < 0) break;
    int64_t j = j1;
    const int64_t j2 = j1 + 1;
    if (j2 < n && q->items[j2].tpot < q->items[j1].tpot) j = j2;
    if (!(q->items[j].tpot < q->items[i].tpot)) break;
    heap_swap(s, ep, i, j);
    i = j;
  }
  return i > i0;
}

void* orc_running_new(int32_t n_ep) {
  Running* s = (Running*)calloc(1, sizeof(Running));
  s->n_ep = n_ep;
  s->heaps = (Heap*)calloc((size_t)n_ep, sizeof(Heap));
  s->map_cap = 1024;
  s->map = (MapSlot*)calloc((size_t)s->map_cap, sizeof(MapSlot));
  return s;
}

void orc_running_free(void* h) {
  Running* s = (Running*)h;
  for (int32_t m = 0; m < s->n_ep; m++) free(s->heaps[m].items);
  free(s->heaps);
  free(s->map);
  free(s);
}

static int add_one(Running* s, int32_t ep, uint64_t key, double tpot) {
  if (key == 0) return 0;                   /* id == "" (:127-129) */
  if (tpot < 0) return 0;                   /* (:130-132) */
  if (map_find(s, ep, key)) return 0;       /* already in the lookup (:135-137) */
  Heap* q = &s->heaps[ep];                  /* heap.Push (:143-145): Push appends, then up */
  if (q->n == q->cap) {
    q->cap = q->cap ? 2 * q->cap : 16;
    q->items = (Item*)realloc(q->items, (size_t)q->cap * sizeof(Item));
  }
  q->items[q->n].key = key;
  q->items[q->n].tpot = tpot;
  map_put(s, ep, key, q->n);
  q->n++;
  up(s, ep, q->n - 1);
  return 1;
}

static int remove_one(Running* s, int32_t ep, uint64_t key) {
  MapSlot* m = map_find(s, ep, key);
  if (!m) return 0;                         /* (:173-176) */
  const int64_t i = m->pos;                 /* heap.Remove(pq, item.index) */
  Heap* q = &s->heaps[ep];
  const int64_t n = q->n - 1;
  if (n != i) {
    heap_swap(s, ep, i, n);
    if (!down(s, ep, i, n)) up(s, ep, i);
  }
  map_find(s, ep, key)->tomb = 1;           /* delete(pq.lookup, id) */
  q->n--;
  return 1;
}

void orc_running_add(void* h, int32_t R, const int32_t* ep, const uint64_t* key, const double* tpot, uint8_t* added) {
  Running* s = (Running*)h;
  for (int32_t r = 0; r < R; r++) {
    const int ok = ep[r] >= 0 ? add_one(s, ep[r], key[r], tpot ? tpot[r] : 0.0) : 0;
    if (added) added[r] = (uint8_t)ok;
  }
}

void orc_running_remove(void* h, int32_t R, const int32_t* ep, const uint64_t* key, uint8_t* removed) {
  Running* s = (Running*)h;
  for (int32_t r = 0; r < R; r++) {
    const int ok = ep[r] >= 0 ? remove_one(s, ep[r], key[r]) : 0;
    if (removed) removed[r] = (uint8_t)ok;
  }
}

void orc_running_remove_endpoint(void* h, int32_t ep) {
  Running* s = (Running*)h;
  Heap* q = &s->heaps[ep];
  while (q->n > 0) remove_one(s, ep, q->items[q->n - 1].key);
}

void orc_running_get(void* h, int32_t M, double* min_out, int32_t* count_out) {
  Running* s = (Running*)h;
  for (int32_t m = 0; m < M; m++) {
    const Heap* q = &s->heaps[m];
    if (min_out) min_out[m] = q->n > 0 ? q->items[0].tpot : 0.0;
    if (count_out) count_out[m] = (int32_t)q->n;
  }
}
