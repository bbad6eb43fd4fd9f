// Test-only: a RESERVED prefix index (DeviceIndex::reserve) under the sequential execution policy of index_emu.cpp.  Every
// mutation runs the shared room code of csrc/prefix_table.cuh (RoomOps: the decision, the same-size rebuild into the spare,
// the swap) in the order the device runs its kernels, so tests/test_index_room_cpu.py checks that code against the oracle's
// indexer on the CPU.  The emu_* entry points of index_emu.cpp (lookups, LRU exports, stats) work on these handles too.
#include "index_emu.cpp"

struct RoomEmu : Emu {
  std::vector<TSlot> other;  // the second table: the spare, or the table after an odd number of swaps
};

// one mutation's room, as index_room_kernel -> table_clear_spare_kernel -> table_rebuild_kernel run it
static uint32_t room_step(RoomEmu* e, uint64_t touches) {
  const uint32_t d = RoomOps<EmuX>::decide(e->x, &e->tv, touches);
  if (d != kRoomRebuild) return d;
  const uint64_t cap = e->tv.mask + 1;
  uint32_t* w = reinterpret_cast<uint32_t*>(e->tv.spare);
  for (uint64_t i = 0; i < cap * (sizeof(TSlot) / 4); i++) RoomOps<EmuX>::clear_spare_word(e->x, w, i);
  for (uint64_t i = 0; i < cap; i++) RoomOps<EmuX>::rehash_slot(e->x, e->tv.slots + i, e->tv.spare, e->tv.mask);
  RoomOps<EmuX>::swap(&e->tv);
  return d;
}

extern "C" {
// an emulated index of `capacity` hashes, reserved as eppscore_prefix_reserve(live, touches, overflow_rows) reserves it
void* room_emu_new(int n_endpoints, long long capacity, int default_lru, int lru_max, long long live, long long touches,
                   long long overflow_rows) {
  Emu* base = static_cast<Emu*>(emu_new(n_endpoints, capacity, default_lru, lru_max));
  RoomEmu* e = new RoomEmu();
  static_cast<Emu&>(*e) = std::move(*base);  // (the vectors keep their buffers: tv / lv stay valid)
  delete base;
  uint64_t want = 32;
  while (want < 4 * (uint64_t)(live + touches)) want <<= 1;
  if (want > e->tv.mask + 1) e->set_slots(want);  // (the table is still empty)
  TSlot f;
  memset(&f, 0x5A, sizeof(f));  // garbage: a rebuild must clear the spare itself
  e->other.assign(e->tv.mask + 1, f);
  e->tv.spare = e->other.data();
  e->ovf_rows.resize((size_t)overflow_rows * e->tv.row_words);
  e->ovf_free.resize((size_t)overflow_rows);
  e->tv.ovf_rows = e->ovf_rows.data();
  e->tv.ovf_free = e->ovf_free.data();
  e->tv.ovf_cap = (uint32_t)overflow_rows;
  return e;
}
void room_emu_free(void* h) {
  RoomEmu* e = static_cast<RoomEmu*>(h);
  delete e->sm;
  delete e;
}
int room_emu_decision(unsigned long long used, unsigned long long live, unsigned long long cap, unsigned long long ovf_in_use,
                      unsigned long long ovf_cap, unsigned long long touches) {
  return (int)room_decision(used, live, cap, ovf_in_use, ovf_cap, touches);
}
// PreRequest on the reserved index; returns the room decision (kRoomProceed / kRoomRebuild / kRoomSkip)
int room_emu_commit(void* h, int R, const int32_t* pick, const uint64_t* hashes, const uint16_t* nh, int stride,
                    const int32_t* cap_req, int single_cap) {
  RoomEmu* e = static_cast<RoomEmu*>(h);
  CommitArgs a{};
  a.R = R;
  a.pick = pick;
  a.hashes = hashes;
  a.n_hashes = nh;
  a.stride = stride;
  a.cap_req = cap_req;
  a.single_cap = single_cap;
  uint64_t touches = 0;
  for (int r = 0; r < R; r++) touches += request_touches(a, r);
  const uint32_t d = room_step(e, touches);
  for (uint32_t p = 0; p < e->lv.n_endpoints; p++) {  // every endpoint's "CTA" (each exits at once on a skip)
    IndexProgram<EmuX> prog(e->x, &e->tv, &e->lv, e->sm, p);
    prog.commit(a);
  }
  return (int)d;
}
// raw deltas on the reserved index: room for n touches, then all of them or none
int room_emu_apply(void* h, long long n, const uint64_t* hash, const int32_t* ep, const uint8_t* op) {
  RoomEmu* e = static_cast<RoomEmu*>(h);
  const uint32_t d = room_step(e, (uint64_t)n);
  if (d == kRoomSkip) return (int)d;
  for (long long i = 0; i < n; i++) {
    if (op[i] == 0) TableOps<EmuX>::set_member(e->x, &e->tv, hash[i], (uint32_t)ep[i]);
    else TableOps<EmuX>::clear_member(e->x, &e->tv, hash[i], (uint32_t)ep[i]);
  }
  return (int)d;
}
// 0: skips, 1: device rebuilds, 2: error bits, 3: whether the table and the spare swapped roles an odd number of times
long long room_emu_stat(void* h, int which) {
  RoomEmu* e = static_cast<RoomEmu*>(h);
  switch (which) {
    case 0: return (long long)e->tv.skips;
    case 1: return (long long)e->tv.rebuilds;
    case 2: return (long long)e->tv.error;
    case 3: return e->tv.slots == e->other.data() ? 1 : 0;
    default: return -1;
  }
}
// FNV-1a over everything a mutation may change except the room bookkeeping (decision, skip count, error bits): the table,
// the overflow rows and free list, the LRU descriptors, maps and logs, and the table's counters
unsigned long long room_emu_digest(void* h) {
  RoomEmu* e = static_cast<RoomEmu*>(h);
  uint64_t f = 1469598103934665603ULL;
  auto mix = [&](const void* p, size_t n) {
    const unsigned char* b = static_cast<const unsigned char*>(p);
    for (size_t i = 0; i < n; i++) f = (f ^ b[i]) * 1099511628211ULL;
  };
  mix(e->tv.slots, (e->tv.mask + 1) * sizeof(TSlot));
  mix(e->ovf_rows.data(), e->ovf_rows.size() * 4);
  mix(e->ovf_free.data(), e->ovf_free.size() * 4);
  mix(e->desc.data(), e->desc.size() * sizeof(LruDesc));
  mix(e->maps.data(), e->maps.size() * sizeof(LruEntry));
  mix(e->logs.data(), e->logs.size() * 8);
  const uint64_t c[5] = {(uint64_t)e->tv.used, (uint64_t)e->tv.live, e->tv.ovf_next, e->tv.ovf_free_top, e->tv.rebuilds};
  mix(c, sizeof(c));
  return f;
}
}
