// prefix_table.cuh — the prefix index of the approximate-prefix producer (approximateprefix/indexer.go) as a
// DEVICE-RESIDENT data structure: both halves of the reference's `indexer` live in HBM and are maintained by kernels.
//
//   hashToPods  map[blockHash]podSet  (indexer.go:34)  ->  open-addressing table of 32-byte slots (one DRAM/L2 sector):
//        { key u64 | cnt u32 | ep u16[10] }   linear probing from (hash & mask), load <= 0.5.
//        Sets of up to 10 endpoints are stored INLINE in the slot, sorted — a probe that hits needs no second access (the first
//        16 bytes already carry two members: enough for the unique tail blocks of a prompt); a block cached on more
//        endpoints points at a bitset row (natural bit order, Mpad bits) in an overflow pool (row id in ep[0..1]).  `cnt == 0` is an emptied
//        set (the reference deletes the key, indexer.go:109-112: a probe treats it as a miss); dead slots are reclaimed when
//        the table is rebuilt (prefix_index.cu).
//   podToLRU    map[ServerID]*lru.Cache (indexer.go:35) ->  per endpoint a LOG-STRUCTURED exact LRU:
//        map[key] -> seq  (open addressing, 16-byte entries)   +   log[seq & mask] = key   (ring, append only)
//        An entry of the log is live iff the map still points at its position; re-touching a key appends a new entry and
//        leaves the old one dead; the oldest live entry is found by advancing `tail`.  This reproduces
//        hashicorp/golang-lru/v2 v2.0.7 exactly (Add of an existing key refreshes recency without eviction; a new key
//        evicts the oldest when the length exceeds the size; Keys() oldest -> newest) — its state is a pure function of the
//        last-touch order, which is what makes a whole batch of Adds for one endpoint parallel.
//
// PreRequest for a batch (plugin.go:169-197: for r in order: indexer.Add(hashes[r], pick[r])) runs as ONE kernel with one
// CTA per endpoint: Adds for different endpoints only ever touch different members of the sets, so they commute; within an
// endpoint the calls are replayed in request order, CHUNKS of up to min(2048, capacity) touches at a time:
//     dedupe the chunk (last touch wins) -> look every distinct key up -> append / insert in last-touch order (new keys also
//     join hashToPods) -> evict the oldest live entries while len > capacity (they leave hashToPods).
// A chunk never evicts a key it touched itself (it holds at most `capacity` distinct keys), which is the only case where the
// order of the reference's two phases (all LRU adds of a call, indexer.go:70-72, THEN all map updates, :75-82) is observable;
// calls longer than the capacity — where that order leaves stale map entries — take a strictly sequential path that
// replays the reference statement by statement.
//
// The CTA program is written once against an execution policy X (par / scan / atomics): prefix_index.cu instantiates it
// with CUDA threads, tests/cpp/index_emu.cpp with a sequential emulation, so the logic is unit-tested on the CPU against the
// oracle's indexer (tests/test_device_index_emu.py) before it ever runs on a GPU.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define PT_HD __host__ __device__ __forceinline__
#else
#define PT_HD inline
#endif

namespace eppscore {

constexpr int kInlineEps = 10;
constexpr uint32_t kCntFree = 0xFFFFFFFFu;  // slot never used
constexpr uint32_t kCntLock = 0x80000000u;  // slot held by an updater (never visible to the scoring kernels)
constexpr uint32_t kCntRow = 0x40000000u;   // the set is a bitset row of the overflow pool; its id is the u32 at ep[0..1]
constexpr uint32_t kCntMask = 0x3FFFFFFFu;  // |set|
constexpr uint32_t kNoRow = 0xFFFFFFFFu;

struct alignas(32) TSlot {
  uint64_t key;
  uint32_t cnt;               // kCntFree | (kCntLock |) (kCntRow |) |set|
  uint16_t ep[kInlineEps];    // inline: the members, ascending, in ep[0..|set|); row mode: ep[0..1] = row id
};
static_assert(sizeof(TSlot) == 32, "one 32-byte sector per slot");
// As the scoring kernels load it: lo = {key.lo, key.hi, cnt, ep0 | ep1 << 16}, hi = {ep2|ep3<<16, ..., ep8|ep9<<16}.
PT_HD uint32_t* slot_row_id(TSlot* s) { return reinterpret_cast<uint32_t*>(&s->ep[0]); }

// What the scoring kernels need (first four fields) + the updaters' bookkeeping.  Lives in DEVICE memory: kernels take a
// pointer to it, so a table rebuild (new arrays) does not invalidate captured CUDA graphs.
struct TableView {
  TSlot* slots;
  uint64_t mask;        // capacity - 1 (capacity a power of two)
  uint32_t* ovf_rows;   // [ovf_cap][row_words] bitsets, natural bit order: endpoint m = bit (m & 31) of word (m >> 5)
  uint32_t row_words;
  uint32_t ovf_cap;
  unsigned long long used;  // slots ever claimed (dead ones included): bounds the load factor
  unsigned long long live;  // slots with a non-empty set == len(hashToPods) of the reference
  uint32_t ovf_next;        // bump allocator of the overflow pool
  uint32_t ovf_free_top;    // free-list stack of released rows
  uint32_t* ovf_free;       // [ovf_cap]
  uint32_t ovf_lock;
  uint32_t error;           // sticky: 1 = overflow pool exhausted (host sizing bug), 2 = table full, kErrSkipped
  // A reserved index (DeviceIndex::reserve) decides room on the device (RoomOps below): these fields stay zero otherwise.
  TSlot* spare;             // a second table of the same capacity: the target of a same-size rebuild, then swapped in
  uint64_t rebuilds;        // device-side rebuilds
  uint64_t skips;           // mutations skipped for lack of room
  uint32_t room;            // kRoomProceed / kRoomRebuild / kRoomSkip: the decision for the mutation being run
  uint32_t rebuild_done;    // CTAs of the rebuild kernel that have finished (the last one swaps the tables)
};
constexpr uint32_t kErrSkipped = 4u;  // sticky: a reserved mutation was skipped whole, the index is as it was before it

constexpr uint64_t kSeqFree = ~0ULL;
constexpr uint64_t kSeqTomb = ~0ULL - 1;
struct LruEntry {
  uint64_t key;
  uint64_t seq;  // kSeqFree, kSeqTomb, or the log position of the key's newest entry
};
struct LruDesc {
  uint64_t head, tail;  // log positions [tail, head)
  uint32_t live;        // == lru.Len()
  uint32_t tomb;        // deleted map entries not yet reclaimed
  uint32_t cap;         // lru size, fixed at creation (indexer.go:57-68)
  uint32_t created;
};
struct LruView {
  LruDesc* desc;        // [n_endpoints]
  LruEntry* maps;       // [n_endpoints][map_size]
  uint64_t* logs;       // [n_endpoints][log_size]
  uint32_t map_size, log_size;  // powers of two
  uint32_t default_cap; // defaultLRUCapacityPerServer (types.go:109) unless the call names CacheNumBlocks
  uint32_t max_cap;     // largest capacity the region sizes support
  uint32_t n_endpoints;
  uint32_t error;       // sticky: 1 = capacity request above max_cap
};

constexpr int kCommitThreads = 512;
constexpr int kChunkMax = 2048;              // touches per parallel chunk
constexpr int kDedupSlots = 2 * kChunkMax;   // CTA-local dedupe set
constexpr int kPicksPerThread = 8;           // the pick array is scanned in windows of 8 * 512 requests
constexpr int kPickWindow = kPicksPerThread * kCommitThreads;
static_assert(kChunkMax == 4 * kCommitThreads, "process_chunk: thread t owns touches [4t, 4t+4)");

PT_HD uint64_t lru_home(uint64_t k) {
  k *= 0x9E3779B97F4A7C15ULL;
  return k ^ (k >> 29);
}

// Region sizes for a given largest capacity: the map keeps live + tombstones <= 3/4 full with a whole chunk of room, the
// log holds every live entry plus the dead ones a steady state accumulates (about as many again) plus a chunk.
inline uint32_t pow2_ceil_u32(uint64_t v) {
  uint64_t c = 16;
  while (c < v) c <<= 1;
  return (uint32_t)c;
}
inline uint32_t lru_map_size_for(uint32_t max_cap) {
  const uint64_t a = 2ULL * max_cap, b = 2ULL * ((uint64_t)max_cap + kChunkMax);
  return pow2_ceil_u32(a > b ? a : b);
}
inline uint32_t lru_log_size_for(uint32_t max_cap) {
  const uint64_t a = 4ULL * max_cap, b = 2ULL * ((uint64_t)max_cap + kChunkMax);
  return pow2_ceil_u32(a > b ? a : b);
}

// ------------------------------------------------------------------------------------------------------------------
// hashToPods: concurrent updates (several endpoint CTAs may add themselves to the same block's set in one batch).
// A slot is updated under its own lock (the top bit of cnt); all accesses inside go to L2 (X::ldcg / plain stores).
// ------------------------------------------------------------------------------------------------------------------
template <class X>
struct TableOps {
  // Lock the slot of `h`, creating it when absent (create) — returns its index, or -1 when absent and !create.
  // *cnt receives the set size at lock time.
  static PT_HD long long lock_slot(X& x, TableView* tv, uint64_t h, bool create, uint32_t* cnt) {
    TSlot* slots = tv->slots;
    const uint64_t mask = tv->mask;
    uint64_t i = h & mask;
    uint64_t probes = 0;
    for (;;) {
      const uint32_t c = x.ld_acquire32(&slots[i].cnt);
      if (c == kCntFree) {
        if (!create) return -1;
        if (x.cas_acquire32(&slots[i].cnt, kCntFree, kCntLock) == kCntFree) {  // claimed and locked, empty set
          x.st64(&slots[i].key, h);
          x.add64(&tv->used, 1ULL);
          *cnt = 0;
          return (long long)i;
        }
        continue;  // somebody else claimed it: look again
      }
      if (c & kCntLock) continue;  // held (maybe being created): its key is not stable yet
      if (x.ld64(&slots[i].key) == h) {
        if (x.cas_acquire32(&slots[i].cnt, c, c | kCntLock) == c) {
          *cnt = c;
          return (long long)i;
        }
        continue;
      }
      i = (i + 1) & mask;
      if (++probes > mask) {  // table full: the host's capacity bound was violated
        x.st32(&tv->error, 2u);
        return -1;
      }
    }
  }
  static PT_HD void unlock_slot(X& x, TableView* tv, long long i, uint32_t cnt) {
    x.st_release32(&tv->slots[i].cnt, cnt);  // release: every store of the critical section is visible before the unlock
  }
  static PT_HD uint32_t alloc_row(X& x, TableView* tv) {
    uint32_t r = kNoRow;
    x.lock(&tv->ovf_lock);
    const uint32_t top = x.ld32(&tv->ovf_free_top);
    if (top > 0) {
      r = x.ld32(&tv->ovf_free[top - 1]);
      x.st32(&tv->ovf_free_top, top - 1);
    } else {
      const uint32_t n = x.ld32(&tv->ovf_next);
      if (n < tv->ovf_cap) {
        r = n;
        x.st32(&tv->ovf_next, n + 1);
      }
    }
    x.unlock(&tv->ovf_lock);
    if (r == kNoRow) {
      x.st32(&tv->error, 1u);
      return r;
    }
    uint32_t* row = tv->ovf_rows + (size_t)r * tv->row_words;
    for (uint32_t w = 0; w < tv->row_words; w++) x.st32(&row[w], 0u);
    return r;
  }
  static PT_HD void free_row(X& x, TableView* tv, uint32_t r) {
    x.lock(&tv->ovf_lock);
    const uint32_t top = x.ld32(&tv->ovf_free_top);
    x.st32(&tv->ovf_free[top], r);
    x.st32(&tv->ovf_free_top, top + 1);
    x.unlock(&tv->ovf_lock);
  }
  // hashToPods[h].insert(p)   (indexer.go:75-82)
  static PT_HD void set_member(X& x, TableView* tv, uint64_t h, uint32_t p) {
    uint32_t raw;
    const long long i = lock_slot(x, tv, h, true, &raw);
    if (i < 0) return;
    TSlot* s = &tv->slots[i];
    const uint32_t c = raw & kCntMask;
    uint32_t nraw = raw;
    if (raw & kCntRow) {
      const uint32_t r = x.ld32(slot_row_id(s));
      uint32_t* w = tv->ovf_rows + (size_t)r * tv->row_words + (p >> 5);
      const uint32_t old = x.ld32(w), bit = 1u << (p & 31);
      if (!(old & bit)) {
        x.st32(w, old | bit);
        nraw = raw + 1;
      }
    } else {
      // the inline members are kept SORTED: equal sets have equal representations whatever the order in which the
      // endpoints' CTAs got to the slot — the scoring kernels merge consecutive hits by comparing the slots' member words,
      // and replicas that replay the same commits hold bit-identical sets
      bool present = false;
      uint32_t pos = c;
      for (uint32_t k = 0; k < c; k++) {
        const uint32_t m = x.ld16(&s->ep[k]);
        present |= (m == p);
        if (m > p && pos == c) pos = k;
      }
      if (!present) {
        if (c < (uint32_t)kInlineEps) {
          for (uint32_t k = c; k > pos; k--) x.st16(&s->ep[k], (uint16_t)x.ld16(&s->ep[k - 1]));
          x.st16(&s->ep[pos], (uint16_t)p);
          nraw = raw + 1;
        } else {  // one member too many for the slot: move the set to a bitset row
          const uint32_t r = alloc_row(x, tv);
          if (r != kNoRow) {
            uint32_t* row = tv->ovf_rows + (size_t)r * tv->row_words;
            for (uint32_t k = 0; k < c; k++) {
              const uint32_t m = x.ld16(&s->ep[k]);
              x.st32(&row[m >> 5], x.ld32(&row[m >> 5]) | (1u << (m & 31)));
            }
            x.st32(&row[p >> 5], x.ld32(&row[p >> 5]) | (1u << (p & 31)));
            x.st32(slot_row_id(s), r);
            nraw = (raw + 1) | kCntRow;
          }
        }
      }
    }
    if (c == 0 && (nraw & kCntMask) == 1) x.add64(&tv->live, 1ULL);
    unlock_slot(x, tv, i, nraw);
  }
  // the eviction callback / RemovePod: delete(hashToPods[h], p); an emptied set behaves as a deleted key (indexer.go:105-115)
  static PT_HD void clear_member(X& x, TableView* tv, uint64_t h, uint32_t p) {
    uint32_t raw;
    const long long i = lock_slot(x, tv, h, false, &raw);
    if (i < 0) return;
    TSlot* s = &tv->slots[i];
    const uint32_t c = raw & kCntMask;
    uint32_t nraw = raw;
    if (raw & kCntRow) {
      const uint32_t r = x.ld32(slot_row_id(s));
      uint32_t* w = tv->ovf_rows + (size_t)r * tv->row_words + (p >> 5);
      const uint32_t old = x.ld32(w), bit = 1u << (p & 31);
      if (old & bit) {
        x.st32(w, old & ~bit);
        nraw = raw - 1;
        if ((nraw & kCntMask) == 0) {  // the set stays a row until it is empty
          free_row(x, tv, r);
          for (uint32_t k = 0; k < (uint32_t)kInlineEps; k++) x.st16(&s->ep[k], (uint16_t)0xFFFFu);  // canonical empty slot
          nraw = 0;
        }
      }
    } else {
      for (uint32_t k = 0; k < c; k++) {
        if (x.ld16(&s->ep[k]) == (uint16_t)p) {
          for (uint32_t j = k; j + 1 < c; j++) x.st16(&s->ep[j], (uint16_t)x.ld16(&s->ep[j + 1]));  // stays sorted and dense
          x.st16(&s->ep[c - 1], (uint16_t)0xFFFFu);  // canonical: unused entries read 0xFFFF, as in a never-used slot
          nraw = raw - 1;
          break;
        }
      }
    }
    if (c > 0 && (nraw & kCntMask) == 0) x.add64(&tv->live, ~0ULL);
    unlock_slot(x, tv, i, nraw);
  }
};

// ------------------------------------------------------------------------------------------------------------------
// Per-endpoint LRU: the map is owned by ONE CTA for the duration of a kernel, so no locks — phases separated by CTA
// barriers (read-only lookups / exclusive updates / inserts of keys known to be absent and pairwise distinct).
// ------------------------------------------------------------------------------------------------------------------
template <class X>
struct LruOps {
  // read-only lookup: index of the key's map entry or -1
  static PT_HD long long find(X& x, const LruEntry* map, uint32_t msize, uint64_t key) {
    const uint64_t mask = msize - 1;
    for (uint64_t i = lru_home(key) & mask, n = 0; n <= mask; i = (i + 1) & mask, n++) {
      const uint64_t s = x.ld64(&map[i].seq);
      if (s == kSeqFree) return -1;
      if (s != kSeqTomb && x.ld64(&map[i].key) == key) return (long long)i;
    }
    return -1;
  }
  // insert a key that is known to be absent; concurrent callers insert pairwise distinct keys (no key compares needed)
  static PT_HD long long insert_new(X& x, LruEntry* map, uint32_t msize, uint64_t key, uint64_t seq) {
    const uint64_t mask = msize - 1;
    for (uint64_t i = lru_home(key) & mask, n = 0; n <= mask; i = (i + 1) & mask, n++) {
      if (x.ld64(&map[i].seq) == kSeqFree && x.cas64(&map[i].seq, kSeqFree, seq) == kSeqFree) {
        x.st64(&map[i].key, key);
        return (long long)i;
      }
    }
    return -1;
  }
};

// Shared-memory state of one commit CTA (the emulation allocates it on the heap).
struct CommitSmem {
  uint64_t tkey[kChunkMax];        // the chunk's touches, in order
  uint64_t dkey[kDedupSlots];      // dedupe set: keys ...
  uint32_t didx[kDedupSlots];      // ... and 1 + index of each key's LAST touch in the chunk
  uint32_t mslot[kChunkMax];       // map entry of each final touch (0xFFFFFFFF: new key)
  uint16_t tslot[kChunkMax];       // dedupe slot of each touch
  uint16_t trank[kChunkMax];       // rank of each final touch among the finals (last-touch order)
  uint32_t req[kPickWindow];       // requests of this endpoint found in the current window of picks
  uint32_t scan[kCommitThreads];   // block-scan workspace
  uint64_t wkey[kCommitThreads];   // window of log keys (eviction / compaction)
  uint32_t wslot[kCommitThreads];
  uint64_t sentinel;
  uint32_t flag, total, n_new;
  uint64_t new_tail;
};

struct CommitArgs {
  int32_t R;
  const int32_t* pick;       // [R] chosen endpoint, < 0: nothing to record (plugin.go:173-175)
  const uint64_t* hashes;    // [R][stride]
  const uint16_t* n_hashes;  // [R]
  int32_t stride;
  const int32_t* cap_req;    // [n_endpoints] CacheNumBlocks per endpoint (autotune, plugin.go:207-216) or null
  int32_t single_cap;        // capacity request when cap_req is null (<= 0: default)
  int32_t ep_first;          // CTA b serves endpoint ep_first + b
  // Several picks per request (the primary profile's, then the "prefill" profile's, plugin.go:177-197): n_picks slots, slot 0
  // is `pick`, slot s > 0 is more_picks[s - 1].  The calls are (request, slot) in request order, slots ascending within a
  // request.  0 or 1: `pick` alone.
  int32_t n_picks;
  const int32_t* more_picks[3];
};

// Σ n_hashes over request r's calls that have a pick: the set_member calls request r can make
PT_HD uint64_t request_touches(const CommitArgs& a, int32_t r) {
  const int32_t np = a.n_picks > 1 ? a.n_picks : 1;
  uint64_t t = 0;
  for (int32_t s = 0; s < np; s++)
    if ((s == 0 ? a.pick : a.more_picks[s - 1])[r] >= 0) t += a.n_hashes[r];
  return t;
}

// ------------------------------------------------------------------------------------------------------------------
// Room on the device (a reserved index: table + spare of a fixed capacity, a fixed overflow pool).  Before every mutation
// that may claim `touches` slots and overflow rows (one each per set_member at most):
//     rows in use + touches > pool                    -> skip: the mutation does not run at all
//     used + touches <= cap / 2                       -> proceed
//     live + touches <= cap / 4                       -> rebuild into the spare (dead slots dropped, same size), proceed
//     otherwise                                       -> skip
// A skipped mutation leaves the index bit-identical and sets kErrSkipped; the table never changes size.
// ------------------------------------------------------------------------------------------------------------------
enum : uint32_t { kRoomProceed = 0, kRoomRebuild = 1, kRoomSkip = 2 };

PT_HD uint32_t room_decision(uint64_t used, uint64_t live, uint64_t cap, uint64_t ovf_in_use, uint64_t ovf_cap,
                             uint64_t touches) {
  if (ovf_in_use + touches > ovf_cap) return kRoomSkip;
  if ((used + touches) * 2 <= cap) return kRoomProceed;
  if ((live + touches) * 4 <= cap) return kRoomRebuild;
  return kRoomSkip;
}

template <class X>
struct RoomOps {
  // One thread, after every earlier mutation: publishes the decision in tv->room.  A rebuild keeps exactly the live slots.
  static PT_HD uint32_t decide(X& x, TableView* tv, uint64_t touches) {
    uint64_t* live_p = reinterpret_cast<uint64_t*>(&tv->live);
    uint64_t* used_p = reinterpret_cast<uint64_t*>(&tv->used);
    const uint64_t used = x.ld64(used_p), live = x.ld64(live_p);
    const uint64_t in_use = (uint64_t)x.ld32(&tv->ovf_next) - x.ld32(&tv->ovf_free_top);
    const uint32_t d = room_decision(used, live, tv->mask + 1, in_use, tv->ovf_cap, touches);
    if (d == kRoomRebuild) {
      x.st64(used_p, live);
      x.st64(&tv->rebuilds, x.ld64(&tv->rebuilds) + 1);
    } else if (d == kRoomSkip) {
      x.st64(&tv->skips, x.ld64(&tv->skips) + 1);
      x.st32(&tv->error, x.ld32(&tv->error) | kErrSkipped);
    }
    x.st32(&tv->room, d);
    return d;
  }
  // Rebuild, pass 1 (every 32-bit word i of the spare): empty
  static PT_HD void clear_spare_word(X& x, uint32_t* spare_words, uint64_t i) { x.st32(&spare_words[i], 0xFFFFFFFFu); }
  // Rebuild, pass 2 (every slot of the table): a slot with a non-empty set moves to table `ns` unchanged (members, filler and
  // row id: a canonical slot stays canonical); dead slots are dropped.  Keys are unique, so a claimed slot is never compared:
  // claim, fill, publish.  Returns whether the slot moved.
  static PT_HD bool rehash_slot(X& x, const TSlot* old, TSlot* ns, uint64_t mask) {
    const uint32_t cnt = x.ld32(&old->cnt);
    if (cnt == kCntFree || (cnt & kCntMask) == 0) return false;
    const uint64_t key = x.ld64(&old->key);
    const uint32_t* src = reinterpret_cast<const uint32_t*>(old);
    for (uint64_t j = key & mask;; j = (j + 1) & mask) {
      if (x.cas32(&ns[j].cnt, kCntFree, kCntLock) != kCntFree) continue;
      x.st64(&ns[j].key, key);
      uint32_t* dst = reinterpret_cast<uint32_t*>(ns + j);
      for (int k = 3; k < (int)(sizeof(TSlot) / 4); k++) x.st32(&dst[k], x.ld32(&src[k]));  // ep[0..10)
      x.st_release32(&ns[j].cnt, cnt);
      return true;
    }
  }
  // Rebuild, last: the spare becomes the table (the old table is the next rebuild's spare)
  static PT_HD void swap(TableView* tv) {
    TSlot* t = tv->slots;
    tv->slots = tv->spare;
    tv->spare = t;
  }
};

template <class X>
struct IndexProgram {
  X& x;
  TableView* tv;
  LruView* lv;
  CommitSmem* sm;
  uint32_t p;         // endpoint
  LruDesc* d;
  LruEntry* map;
  uint64_t* log;
  uint32_t msize, lsize;

  PT_HD IndexProgram(X& x_, TableView* tv_, LruView* lv_, CommitSmem* sm_, uint32_t p_)
      : x(x_), tv(tv_), lv(lv_), sm(sm_), p(p_) {
    d = lv->desc + p;
    msize = lv->map_size;
    lsize = lv->log_size;
    map = lv->maps + (size_t)p * msize;
    log = lv->logs + (size_t)p * lsize;
  }
  PT_HD uint64_t log_get(uint64_t pos) { return x.ld64(&log[pos & (lsize - 1)]); }
  PT_HD void log_put(uint64_t pos, uint64_t k) { x.st64(&log[pos & (lsize - 1)], k); }

  // indexer.go:57-68: the LRU is created by the first Add, sized CacheNumBlocks when > 0, else the default
  PT_HD void ensure_created(int32_t cap_req) {
    x.par([&](int tid) {
      if (tid == 0 && !x.ld32(&d->created)) {
        uint32_t c = cap_req > 0 ? (uint32_t)cap_req : lv->default_cap;
        if (c < 1) c = 1;
        if (c > lv->max_cap) {
          x.st32(&lv->error, 1u);
          c = lv->max_cap;
        }
        x.st32(&d->cap, c);
        x.st32(&d->created, 1u);
      }
    });
  }

  // ---- compaction of the log + rebuild of the map: drops dead log entries and tombstones ----
  PT_HD void rebuild() {
    const uint64_t tail = x.ld64(&d->tail), head = x.ld64(&d->head);
    x.par([&](int tid) {
      if (tid == 0) sm->new_tail = tail;
    });
    for (uint64_t w = tail; w < head; w += kCommitThreads) {
      x.par([&](int tid) {
        const uint64_t pos = w + tid;
        uint32_t f = 0;
        if (pos < head) {
          const uint64_t k = log_get(pos);
          const long long e = LruOps<X>::find(x, map, msize, k);
          if (e >= 0 && x.ld64(&map[e].seq) == pos) {
            f = 1;
            sm->wkey[tid] = k;
            sm->wslot[tid] = (uint32_t)e;
          }
        }
        sm->scan[tid] = f;
      });
      const uint32_t tot = x.scan(sm->scan, &sm->total);
      const uint64_t base = sm->new_tail;
      x.par([&](int tid) {
        const uint64_t pos = w + tid;
        const bool mine = pos < head && (tid + 1 < kCommitThreads ? sm->scan[tid + 1] : tot) != sm->scan[tid];
        if (mine) {
          const uint64_t np = base + sm->scan[tid];
          log_put(np, sm->wkey[tid]);
          x.st64(&map[sm->wslot[tid]].seq, np);
        }
        if (tid == 0) sm->new_tail = base + tot;
      });
    }
    const uint64_t nhead = sm->new_tail;
    // tombstones: clear the map and re-insert the (now contiguous, all live) entries
    for (uint32_t w = 0; w < msize; w += kCommitThreads)
      x.par([&](int tid) {
        if (w + tid < msize) x.st64(&map[w + tid].seq, kSeqFree);
      });
    for (uint64_t w = tail; w < nhead; w += kCommitThreads)
      x.par([&](int tid) {
        const uint64_t pos = w + tid;
        if (pos < nhead) LruOps<X>::insert_new(x, map, msize, log_get(pos), pos);
      });
    x.par([&](int tid) {
      if (tid == 0) {
        x.st64(&d->head, nhead);
        x.st32(&d->tomb, 0u);
      }
    });
  }
  PT_HD void make_room(uint32_t n) {
    const uint64_t span = x.ld64(&d->head) - x.ld64(&d->tail);
    const uint64_t occ = (uint64_t)x.ld32(&d->live) + x.ld32(&d->tomb) + n;
    if (span + n > lsize || occ * 4 > (uint64_t)msize * 3) rebuild();
  }

  // ---- evict the oldest live entries until len <= cap; each leaves hashToPods (makeEvictionFn, indexer.go:105-115) ----
  PT_HD void evict_down() {
    for (;;) {
      const uint32_t live = x.ld32(&d->live), cap = x.ld32(&d->cap);
      if (live <= cap) break;
      const uint32_t need = live - cap;
      const uint64_t tail = x.ld64(&d->tail), head = x.ld64(&d->head);
      x.par([&](int tid) {
        const uint64_t pos = tail + tid;
        uint32_t f = 0;
        if (pos < head) {
          const uint64_t k = log_get(pos);
          const long long e = LruOps<X>::find(x, map, msize, k);
          if (e >= 0 && x.ld64(&map[e].seq) == pos) {
            f = 1;
            sm->wkey[tid] = k;
            sm->wslot[tid] = (uint32_t)e;
          }
        }
        sm->scan[tid] = f;
        if (tid == 0) sm->new_tail = (tail + kCommitThreads < head) ? tail + kCommitThreads : head;
      });
      const uint32_t tot = x.scan(sm->scan, &sm->total);
      x.par([&](int tid) {
        const bool isl = (tid + 1 < kCommitThreads ? sm->scan[tid + 1] : tot) != sm->scan[tid];
        if (isl && sm->scan[tid] < need) {
          x.st64(&map[sm->wslot[tid]].seq, kSeqTomb);
          TableOps<X>::clear_member(x, tv, sm->wkey[tid], p);
          if (sm->scan[tid] == need - 1) sm->new_tail = tail + tid + 1;  // the last eviction of this round
        }
      });
      x.par([&](int tid) {
        if (tid == 0) {
          const uint32_t ev = tot < need ? tot : need;
          x.st64(&d->tail, sm->new_tail);
          x.st32(&d->live, live - ev);
          x.st32(&d->tomb, x.ld32(&d->tomb) + ev);
        }
      });
    }
  }

  // ---- one parallel chunk: n <= min(kChunkMax, cap) touches in sm->tkey, every call they come from has n_c <= cap ----
  PT_HD void process_chunk(uint32_t n) {
    if (n == 0) return;
    make_room(n);
    // a sentinel that is not one of the chunk's keys marks empty dedupe slots
    x.par([&](int tid) {
      if (tid == 0) sm->sentinel = ~0ULL;
    });
    for (;;) {
      x.par([&](int tid) {
        if (tid == 0) sm->flag = 0;
      });
      const uint64_t s = sm->sentinel;
      x.par([&](int tid) {
        for (uint32_t i = tid; i < n; i += kCommitThreads)
          if (sm->tkey[i] == s) sm->flag = 1;
      });
      if (!sm->flag) break;
      x.par([&](int tid) {
        if (tid == 0) sm->sentinel = s - 1;
      });
    }
    const uint64_t S = sm->sentinel;
    x.par([&](int tid) {
      for (uint32_t j = tid; j < (uint32_t)kDedupSlots; j += kCommitThreads) {
        sm->dkey[j] = S;
        sm->didx[j] = 0;
      }
    });
    x.par([&](int tid) {  // dedupe: the LAST touch of a key carries its recency
      for (uint32_t i = tid; i < n; i += kCommitThreads) {
        const uint64_t k = sm->tkey[i];
        uint32_t j = (uint32_t)lru_home(k) & (kDedupSlots - 1);
        for (;;) {
          const uint64_t old = x.smem_cas64(&sm->dkey[j], S, k);
          if (old == S || old == k) break;
          j = (j + 1) & (kDedupSlots - 1);
        }
        x.smem_max32(&sm->didx[j], i + 1);
        sm->tslot[i] = (uint16_t)j;
      }
    });
    // finals in touch order -> dense ranks.  Thread t owns touches [t*4, t*4+4) (kChunkMax == 4 * kCommitThreads).
    x.par([&](int tid) {
      uint32_t c = 0;
      for (uint32_t i = (uint32_t)tid * 4; i < (uint32_t)tid * 4 + 4 && i < n; i++) c += (sm->didx[sm->tslot[i]] == i + 1);
      sm->scan[tid] = c;
    });
    const uint32_t n_final = x.scan(sm->scan, &sm->total);
    x.par([&](int tid) {  // read-only lookups
      uint32_t rk = sm->scan[tid];
      for (uint32_t i = (uint32_t)tid * 4; i < (uint32_t)tid * 4 + 4 && i < n; i++) {
        if (sm->didx[sm->tslot[i]] == i + 1) {
          sm->trank[i] = (uint16_t)rk++;
          const long long e = LruOps<X>::find(x, map, msize, sm->tkey[i]);
          sm->mslot[i] = e >= 0 ? (uint32_t)e : 0xFFFFFFFFu;
        }
      }
      if (tid == 0) sm->n_new = 0;
    });
    const uint64_t head = x.ld64(&d->head);
    x.par([&](int tid) {  // refresh / insert in last-touch order; new keys join hashToPods
      for (uint32_t i = tid; i < n; i += kCommitThreads) {
        if (sm->didx[sm->tslot[i]] != i + 1) continue;
        const uint64_t k = sm->tkey[i], seq = head + sm->trank[i];
        log_put(seq, k);
        if (sm->mslot[i] != 0xFFFFFFFFu) {
          x.st64(&map[sm->mslot[i]].seq, seq);
        } else {
          LruOps<X>::insert_new(x, map, msize, k, seq);
          TableOps<X>::set_member(x, tv, k, p);
          x.smem_add32(&sm->n_new, 1u);
        }
      }
    });
    x.par([&](int tid) {
      if (tid == 0) {
        x.st64(&d->head, head + n_final);
        x.st32(&d->live, x.ld32(&d->live) + sm->n_new);
      }
    });
    evict_down();
  }

  // ---- a call longer than the LRU: replay indexer.Add statement by statement (one thread) ----
  PT_HD void sequential_call(const uint64_t* h, uint32_t n) {
    for (uint32_t c0 = 0; c0 < n; c0 += kChunkMax) {  // phase 1 (indexer.go:70-72), in pieces so the log/map never overflow
      const uint32_t m = n - c0 < (uint32_t)kChunkMax ? n - c0 : (uint32_t)kChunkMax;
      make_room(m);
      x.par([&](int tid) {
        if (tid != 0) return;
        uint64_t head = x.ld64(&d->head), tail = x.ld64(&d->tail);
        uint32_t live = x.ld32(&d->live), tomb = x.ld32(&d->tomb);
        const uint32_t cap = x.ld32(&d->cap);
        for (uint32_t i = 0; i < m; i++) {
          const uint64_t k = x.ld64(&h[c0 + i]);
          const long long e = LruOps<X>::find(x, map, msize, k);
          log_put(head, k);
          if (e >= 0) {
            x.st64(&map[e].seq, head);  // refresh recency, no eviction
          } else {
            LruOps<X>::insert_new(x, map, msize, k, head);
            live++;
          }
          head++;
          if (live > cap) {  // RemoveOldest + eviction callback
            for (;; tail++) {
              const uint64_t ok = log_get(tail);
              const long long oe = LruOps<X>::find(x, map, msize, ok);
              if (oe >= 0 && x.ld64(&map[oe].seq) == tail) {
                x.st64(&map[oe].seq, kSeqTomb);
                TableOps<X>::clear_member(x, tv, ok, p);
                tail++;
                break;
              }
            }
            live--;
            tomb++;
          }
        }
        x.st64(&d->head, head);
        x.st64(&d->tail, tail);
        x.st32(&d->live, live);
        x.st32(&d->tomb, tomb);
      });
    }
    // phase 2 (indexer.go:75-82): EVERY hash of the call joins hashToPods, evicted or not — the stale-entry quirk
    for (uint32_t c0 = 0; c0 < n; c0 += kCommitThreads)
      x.par([&](int tid) {
        if (c0 + tid < n) TableOps<X>::set_member(x, tv, x.ld64(&h[c0 + tid]), p);
      });
  }

  // ---- PreRequest for this endpoint's share of a batch ----
  // `fill` (touches waiting in sm->tkey) and every branch below are CTA-uniform: all threads compute them identically
  // from values that were published by a completed parallel section.
  PT_HD void commit(const CommitArgs& a) {
    if (x.ld32(&tv->room) == kRoomSkip) return;  // all or nothing: no room was guaranteed for this call (RoomOps)
    bool created = x.ld32(&d->created) != 0;
    const int32_t cap_req = a.cap_req ? a.cap_req[p] : a.single_cap;
    uint32_t fill = 0, cap = 0, chunk_cap = 0;
    // call i is (request i / np, slot i % np): this endpoint's calls in call order, then each call's request
    const int32_t np = a.n_picks > 1 ? a.n_picks : 1;
    const int32_t n_calls = a.R * np;
    auto call_pick = [&](int32_t i) {
      if (np == 1) return a.pick[i];
      const int32_t r = i / np, s = i - r * np;
      return (s == 0 ? a.pick : a.more_picks[s - 1])[r];
    };
    for (int32_t r0 = 0; r0 < n_calls; r0 += kPickWindow) {
      // this endpoint's calls in the window, in call order: thread t looks at calls [r0 + 8t, r0 + 8t + 8)
      x.par([&](int tid) {
        uint32_t c = 0;
        const int32_t rb = r0 + tid * kPicksPerThread;
        for (int32_t k = 0; k < kPicksPerThread; k++) c += (rb + k < n_calls && call_pick(rb + k) == (int32_t)p) ? 1u : 0u;
        sm->scan[tid] = c;
      });
      const uint32_t nreq = x.scan(sm->scan, &sm->total);
      if (nreq == 0) continue;
      x.par([&](int tid) {
        uint32_t at = sm->scan[tid];
        const int32_t rb = r0 + tid * kPicksPerThread;
        for (int32_t k = 0; k < kPicksPerThread; k++)
          if (rb + k < n_calls && call_pick(rb + k) == (int32_t)p) sm->req[at++] = (uint32_t)((rb + k) / np);
      });
      if (!created) {
        ensure_created(cap_req);
        created = true;
      }
      if (chunk_cap == 0) {
        cap = x.ld32(&d->cap);
        chunk_cap = cap < (uint32_t)kChunkMax ? cap : (uint32_t)kChunkMax;
      }
      for (uint32_t q = 0; q < nreq; q++) {
        const uint32_t r = sm->req[q];
        const uint32_t n = a.n_hashes[r];
        const uint64_t* h = a.hashes + (size_t)r * a.stride;
        if (n > cap) {  // longer than the LRU: strictly sequential
          process_chunk(fill);
          fill = 0;
          sequential_call(h, n);
          continue;
        }
        uint32_t done = 0;
        while (done < n) {
          const uint32_t take = (n - done < chunk_cap - fill) ? n - done : chunk_cap - fill;
          x.par([&](int tid) {
            for (uint32_t i = (uint32_t)tid; i < take; i += kCommitThreads) sm->tkey[fill + i] = x.ld64(&h[done + i]);
          });
          done += take;
          fill += take;
          if (fill == chunk_cap) {
            process_chunk(fill);
            fill = 0;
          }
        }
      }
    }
    process_chunk(fill);
  }

  // ---- indexer.RemovePod (indexer.go:167-182): every key of the LRU leaves hashToPods, then the LRU is dropped ----
  PT_HD void remove_endpoint() {
    if (!x.ld32(&d->created)) return;
    const uint64_t tail = x.ld64(&d->tail), head = x.ld64(&d->head);
    for (uint64_t w = tail; w < head; w += kCommitThreads)
      x.par([&](int tid) {
        const uint64_t pos = w + tid;
        if (pos < head) {
          const uint64_t k = log_get(pos);
          const long long e = LruOps<X>::find(x, map, msize, k);
          if (e >= 0 && x.ld64(&map[e].seq) == pos) TableOps<X>::clear_member(x, tv, k, p);
        }
      });
    for (uint32_t w = 0; w < msize; w += kCommitThreads)
      x.par([&](int tid) {
        if (w + tid < msize) x.st64(&map[w + tid].seq, kSeqFree);
      });
    x.par([&](int tid) {
      if (tid == 0) {
        x.st64(&d->head, 0);
        x.st64(&d->tail, 0);
        x.st32(&d->live, 0);
        x.st32(&d->tomb, 0);
        x.st32(&d->cap, 0);
        x.st32(&d->created, 0);
      }
    });
  }

  // ---- lru.Keys(): oldest -> newest; returns the length, writes at most cap_out keys ----
  PT_HD uint32_t export_keys(uint64_t* out, uint32_t cap_out) {
    const uint64_t tail = x.ld64(&d->tail), head = x.ld64(&d->head);
    x.par([&](int tid) {
      if (tid == 0) sm->new_tail = 0;  // running count
    });
    for (uint64_t w = tail; w < head; w += kCommitThreads) {
      x.par([&](int tid) {
        const uint64_t pos = w + tid;
        uint32_t f = 0;
        if (pos < head) {
          const uint64_t k = log_get(pos);
          const long long e = LruOps<X>::find(x, map, msize, k);
          if (e >= 0 && x.ld64(&map[e].seq) == pos) {
            f = 1;
            sm->wkey[tid] = k;
          }
        }
        sm->scan[tid] = f;
      });
      const uint32_t tot = x.scan(sm->scan, &sm->total);
      const uint64_t base = sm->new_tail;
      x.par([&](int tid) {
        const bool mine = (tid + 1 < kCommitThreads ? sm->scan[tid + 1] : tot) != sm->scan[tid];
        if (mine && base + sm->scan[tid] < cap_out) out[base + sm->scan[tid]] = sm->wkey[tid];
        if (tid == 0) sm->new_tail = base + tot;
      });
    }
    return (uint32_t)sm->new_tail;
  }
};

// indexer.Get's lookup (indexer.go:86-102), read-only: found(slot, cnt word) when `h` has a non-empty set, else 0 (absent, or an
// emptied set, which the reference has deleted).
template <class X, class F>
PT_HD uint32_t table_probe(X& x, const TableView* tv, uint64_t h, F found) {
  for (uint64_t i = h & tv->mask, n = 0; n <= tv->mask; i = (i + 1) & tv->mask, n++) {
    TSlot* s = &tv->slots[i];
    const uint32_t raw = x.ld32(&s->cnt);
    if (raw == kCntFree) return 0;
    if (x.ld64(&s->key) != h) continue;
    if ((raw & kCntMask) == 0) return 0;
    return found(s, raw);
  }
  return 0;
}
// The slot of `h` when its set is non-empty, else nullptr; *raw receives the slot's cnt word.
template <class X>
PT_HD TSlot* table_find(X& x, const TableView* tv, uint64_t h, uint32_t* raw) {
  TSlot* hit = nullptr;
  table_probe(x, tv, h, [&](TSlot* s, uint32_t c) {
    hit = s;
    *raw = c;
    return 1u;
  });
  return hit;
}

// The membership rule of a set given its cnt word `raw`: a compare against the inline members (member(k) = ep[k]), or bit p of
// the row (row() = its id).  slot_holds reads them from the slot, staged_holds from a copy of the slot's ep words.
template <class X, class Row, class Member>
PT_HD bool set_holds(X& x, const TableView* tv, uint32_t raw, uint32_t p, Row row, Member member) {
  if (raw & kCntRow) {
    if ((p >> 5) >= tv->row_words) return false;
    const uint32_t r = row();
    return (x.ld32(&tv->ovf_rows[(size_t)r * tv->row_words + (p >> 5)]) >> (p & 31)) & 1u;
  }
  const uint32_t c = raw & kCntMask;
  for (uint32_t k = 0; k < c; k++)
    if (member(k) == p) return true;
  return false;
}
// Whether endpoint p is in the set of a slot table_find returned.
template <class X>
PT_HD bool slot_holds(X& x, const TableView* tv, TSlot* s, uint32_t raw, uint32_t p) {
  return set_holds(x, tv, raw, p, [&] { return x.ld32(slot_row_id(s)); }, [&](uint32_t k) { return x.ld16(&s->ep[k]); });
}
// The same for a slot whose ep[0..kInlineEps) were copied as kInlineEps / 2 words (ep[2i] | ep[2i+1] << 16, as the slot holds
// them; in row mode word 0 is the row id).
template <class X>
PT_HD bool staged_holds(X& x, const TableView* tv, uint32_t raw, const uint32_t* ep_words, uint32_t p) {
  return set_holds(x, tv, raw, p, [&] { return ep_words[0]; },
                   [&](uint32_t k) { return (ep_words[k >> 1] >> ((k & 1) * 16)) & 0xFFFFu; });
}

// indexer.Get (indexer.go:86-102) for one hash, read-only: writes the set as a natural-order bitset, returns its size.
template <class X>
PT_HD uint32_t table_get(X& x, const TableView* tv, uint64_t h, uint32_t* bits, uint32_t words) {
  for (uint32_t w = 0; w < words; w++) bits[w] = 0;
  return table_probe(x, tv, h, [&](TSlot* s, uint32_t raw) {
    const uint32_t c = raw & kCntMask;
    if (raw & kCntRow) {
      const uint32_t r = x.ld32(slot_row_id(s));
      for (uint32_t w = 0; w < words && w < tv->row_words; w++) bits[w] = x.ld32(&tv->ovf_rows[(size_t)r * tv->row_words + w]);
    } else {
      for (uint32_t k = 0; k < c; k++) {
        const uint32_t m = x.ld16(&s->ep[k]);
        if ((m >> 5) < words) bits[m >> 5] |= 1u << (m & 31);
      }
    }
    return c;
  });
}

}  // namespace eppscore
