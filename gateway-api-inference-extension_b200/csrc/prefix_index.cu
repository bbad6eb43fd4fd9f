// prefix_index.cu — kernels and host-side owner of the device-resident prefix index (prefix_table.cuh).
//
// The host keeps NO mirror of the index: it only sizes the arrays.  After every mutating launch it enqueues a copy of the
// table's counters (TableView, 96 bytes) into pinned memory; the next mutating call waits for that copy (i.e. for the
// previous index operation, nothing else) and derives exact bounds from it:
//     used slots + touches of this call  <= capacity / 2      else the table is rebuilt (dead slots dropped) or doubled,
//     overflow rows in use + touches     <= overflow capacity else the pool is grown,
// so no kernel can ever run out of room and nothing is retried.
// A RESERVED index (reserve()) has a fixed table, a spare table of the same size and a fixed overflow pool; every mutation
// first runs the room kernels (RoomOps in prefix_table.cuh), which take the same decision on the device — proceed, rebuild
// into the spare, or skip the mutation whole — so no host wait is needed and the sequence can be captured into a CUDA graph.
#include "prefix_index.hpp"

#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/eppscore.h"
#include "index_device.cuh"

namespace eppscore {

// ---------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kCommitThreads) index_commit_kernel(TableView* tv, LruView* lv, const CommitArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  DevX x;
  const uint32_t p = (uint32_t)a.ep_first + blockIdx.x;
  if (p >= lv->n_endpoints) return;
  IndexProgram<DevX> prog(x, tv, lv, reinterpret_cast<CommitSmem*>(smem_raw), p);
  prog.commit(a);
}

__global__ void __launch_bounds__(kCommitThreads) index_remove_kernel(TableView* tv, LruView* lv, uint32_t p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  DevX x;
  IndexProgram<DevX> prog(x, tv, lv, reinterpret_cast<CommitSmem*>(smem_raw), p);
  prog.remove_endpoint();
}

// out[0] = lru.Len() (0xFFFFFFFF: the endpoint has no LRU), keys oldest -> newest from out_keys
__global__ void __launch_bounds__(kCommitThreads) index_export_kernel(TableView* tv, LruView* lv, uint32_t p, uint64_t* out_keys,
                                                                      uint32_t cap, uint32_t* out_len) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  DevX x;
  IndexProgram<DevX> prog(x, tv, lv, reinterpret_cast<CommitSmem*>(smem_raw), p);
  if (!x.ld32(&lv->desc[p].created)) {
    if (threadIdx.x == 0) *out_len = 0xFFFFFFFFu;
    return;
  }
  const uint32_t n = prog.export_keys(out_keys, cap);
  if (threadIdx.x == 0) *out_len = n;
}

// Raw deltas from a host that runs its own LRU: applied in order per endpoint (ops on different endpoints commute).
__global__ void index_apply_kernel(TableView* tv, int64_t n, const uint64_t* hash, const int32_t* endpoint, const uint8_t* op,
                                   uint32_t n_endpoints) {
  DevX x;
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_endpoints || x.ld32(&tv->room) == kRoomSkip) return;
  for (int64_t i = 0; i < n; i++) {
    if ((uint32_t)endpoint[i] != p) continue;
    if (op[i] == 0) TableOps<DevX>::set_member(x, tv, hash[i], p);
    else TableOps<DevX>::clear_member(x, tv, hash[i], p);
  }
}

// indexer.Get for one hash, read from the device table: out[0] = |set|, out[1..] natural-order bitset
__global__ void table_get_kernel(const TableView* tv, uint64_t h, uint32_t* out, uint32_t words) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  DevX x;
  out[0] = table_get(x, tv, h, out + 1, words);
}

// Loads for a kernel that only reads the index while no mutation runs (stream order and the pending-batch rules order it
// against them): through the read-only cache, so the member loads of a probe hit the line its first load brought in.
struct ReadX {
  __device__ __forceinline__ uint32_t ld32(const uint32_t* p) { return __ldg(p); }
  __device__ __forceinline__ uint64_t ld64(const uint64_t* p) { return __ldg(reinterpret_cast<const unsigned long long*>(p)); }
  __device__ __forceinline__ uint32_t ld16(const uint16_t* p) { return __ldg(p); }
};

// matchLongestPrefix (approximateprefix/plugin.go:219-235) read at k endpoints per request: one warp per request.  Lane b probes
// block base + b (32 probes in flight), the ballot of misses gives the first one, and each listed endpoint's count of the hits
// before it is a ballot of the lanes whose set holds the endpoint.  Lane j keeps endpoint j's count (j < 32); the counts of
// endpoints past 32 accumulate in the request's out row.
// One request's walk, by its whole warp: returns lane j's count for endpoint j < min(k, 32); the counts of entries j >= 32
// accumulate in o[j * os] (written by lane j & 31, which alone reads them back).
constexpr int kMatchThreads = 256;
template <class X>
__device__ __forceinline__ uint32_t match_walk(X& x, const TableView* tv, uint32_t lane, int32_t k, uint32_t limit, uint32_t n,
                                               const uint64_t* h, const int32_t* eps, uint16_t* o, int32_t os) {
  const int32_t k0 = k < 32 ? k : 32;
  const uint32_t e0 = (int32_t)lane < k0 ? (uint32_t)eps[lane] : 0xFFFFFFFFu;  // (-1 and >= limit never match)
  uint32_t c0 = 0;
  for (uint32_t base = 0;; base += 32) {  // at least one round: it writes the row's entries past 32
    uint32_t raw = 0;
    TSlot* s = base + lane < n ? table_find(x, tv, h[base + lane], &raw) : nullptr;
    const uint32_t miss = __ballot_sync(0xffffffffu, base + lane < n && !s);
    const uint32_t left = n > base ? n - base : 0;
    const uint32_t hits = miss ? (uint32_t)__ffs(miss) - 1 : (left < 32 ? left : 32);
    const bool hit = lane < hits;
    for (int32_t j = 0; j < k0; j++) {
      const uint32_t e = __shfl_sync(0xffffffffu, e0, j);
      const uint32_t c = __popc(__ballot_sync(0xffffffffu, hit && e < limit && slot_holds(x, tv, s, raw, e)));
      if ((int32_t)lane == j) c0 += c;
    }
    for (int32_t j = 32; j < k; j++) {
      const uint32_t e = (uint32_t)__ldg(&eps[j]);
      const uint32_t c = __popc(__ballot_sync(0xffffffffu, hit && e < limit && slot_holds(x, tv, s, raw, e)));
      if (lane == (uint32_t)(j & 31)) o[(size_t)j * os] = (uint16_t)((base == 0 ? 0u : o[(size_t)j * os]) + c);
    }
    if (miss || base + 32 >= n) break;
  }
  return c0;
}

__global__ void __launch_bounds__(kMatchThreads) prefix_match_kernel(const TableView* tv, int32_t R, int32_t k, uint32_t limit,
                                                                     const uint64_t* hashes, const uint16_t* n_hashes, int32_t stride,
                                                                     const int32_t* endpoints, uint16_t* out) {
  ReadX x;
  const uint32_t lane = threadIdx.x & 31;
  const int32_t warps = gridDim.x * (kMatchThreads / 32);
  for (int32_t r = blockIdx.x * (kMatchThreads / 32) + (threadIdx.x >> 5); r < R; r += warps) {
    uint16_t* o = out + (size_t)r * k;
    const uint32_t c0 = match_walk(x, tv, lane, k, limit, n_hashes[r], hashes + (size_t)r * stride, endpoints + (size_t)r * k, o, 1);
    if ((int32_t)lane < (k < 32 ? k : 32)) o[lane] = (uint16_t)c0;
  }
}

// PrepareRequestData of the predicted-latency producer (predictedlatency/preparedata_hooks.go:36-106, prediction.go:44-166) at
// k listed endpoints per request: the walk of prefix_match_kernel gives each entry's match count c, then lane j owns entries
// j, j + 32, ...: it gathers the endpoint's tile column and evaluates lat_pair with the prefix term pcoef * (c/total) exactly
// as score_matrix_kernel forms it, and writes the entry's 48-byte record.  Without match_out the counts of entries past 32
// accumulate in their own record's `dispatched` field until the record is written.
__global__ void __launch_bounds__(kMatchThreads) latency_info_kernel(const TableView* tv, uint32_t limit, const LatInfoArgs a) {
  ReadX x;
  const uint32_t lane = threadIdx.x & 31;
  const int32_t warps = gridDim.x * (kMatchThreads / 32), k = a.k;
  eppscore_latency_info* const out = static_cast<eppscore_latency_info*>(a.out);
  for (int32_t r = blockIdx.x * (kMatchThreads / 32) + (threadIdx.x >> 5); r < a.R; r += warps) {
    const uint32_t n = a.n_hashes[r];
    const int32_t* eps = a.endpoints + (size_t)r * k;
    eppscore_latency_info* rec = out + (size_t)r * k;
    uint16_t* o = a.match_out ? a.match_out + (size_t)r * k : reinterpret_cast<uint16_t*>(&rec->dispatched);
    const int32_t os = a.match_out ? 1 : (int32_t)(sizeof(eppscore_latency_info) / 2);
    const uint32_t c0 = match_walk(x, tv, lane, k, limit, n, a.hashes + (size_t)r * a.stride, eps, o, os);
    const double in_tok = (double)(a.input_tokens ? a.input_tokens[r] : 0);  // len(strings.Fields(prompt)), training.go:51
    const double x_in = __dmul_rn(a.ttft_input, in_tok), y_in = __dmul_rn(a.tpot_input, in_tok);
    const double tslo = a.ttft_slo ? a.ttft_slo[r] : 0.0;
    const double buf = __dmul_rn(a.tpot_slo ? a.tpot_slo[r] : 0.0, a.buffer);  // prediction.go:150
    for (int32_t j = (int32_t)lane; j < k; j += 32) {
      const uint32_t c = j < 32 ? c0 : o[(size_t)j * os];
      if (a.match_out) o[j] = (uint16_t)c;
      const int32_t m = __ldg(&eps[j]);
      double v[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
      int32_t disp = 0;
      uint32_t flags = 0;  // present | ttft_valid << 8 | tpot_valid << 16 (little-endian bytes of the record)
      if (a.has_predictions && m >= 0 && m < a.M) {
        const double frac = n ? __ddiv_rn((double)c, (double)n) : 0.0;  // match/total, NaN (0/0) => 0
        const LatPair lp = lat_pair(a.ep + (size_t)(m >> 5) * 256 + (m & 31), a.tpot_generated, __dmul_rn(a.ttft_prefix, frac),
                                    x_in, y_in, tslo, buf);
        const bool neutral = (__ldg(reinterpret_cast<const int*>(a.ep + (size_t)(m >> 5) * 256 + (m & 31) + 224)) & 2) != 0;
        v[0] = lp.ttft;
        v[1] = lp.tpot;
        v[2] = lp.hT;
        v[3] = lp.hP;
        v[4] = frac;
        disp = __ldg(&a.dispatched[m]);
        flags = 1u | (lp.ttft < tslo ? 1u << 8 : 0u) | ((neutral || lp.tpot < lp.buffered) ? 1u << 16 : 0u);
      }
      double* d = reinterpret_cast<double*>(rec + j);
      for (int i = 0; i < 5; i++) d[i] = v[i];
      reinterpret_cast<int2*>(d + 5)[0] = make_int2(disp, (int32_t)flags);
    }
  }
}

// Rebuild: re-insert every slot with a non-empty set into a fresh table (dead slots are dropped).
__global__ void table_rehash_kernel(const TSlot* old_slots, uint64_t old_cap, TableView* nv) {
  DevX x;
  unsigned long long moved = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < old_cap; i += (uint64_t)gridDim.x * blockDim.x)
    moved += RoomOps<DevX>::rehash_slot(x, old_slots + i, nv->slots, nv->mask) ? 1 : 0;
  if (moved) {
    atomicAdd(&nv->used, moved);
    atomicAdd(&nv->live, moved);
  }
}

// Σ n_hashes over the calls that have a pick: the exact number of touches of a commit whose arrays are on the device
__global__ void sum_touches_kernel(const CommitArgs a, unsigned long long* out) {
  unsigned long long t = 0;
  for (int32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < a.R; r += gridDim.x * blockDim.x) t += request_touches(a, r);
#pragma unroll
  for (int o = 16; o; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if ((threadIdx.x & 31) == 0 && t) atomicAdd(out, t);
}

// ---- a reserved index: room decided on the device (RoomOps), so a mutation never waits on the host ----
// Every reserved mutation runs room -> clear spare -> rebuild -> the mutation, with launch shapes that depend only on the
// reservation; the kernels with nothing to do exit at once.
constexpr int kRoomThreads = 1024;
constexpr int kRebuildCtas = 264, kRebuildThreads = 512;

// The decision for one mutation: its touches are host_touches (>= 0), or summed here over a commit's calls.
__global__ void __launch_bounds__(kRoomThreads) index_room_kernel(TableView* tv, const CommitArgs a, long long host_touches) {
  __shared__ unsigned long long part[kRoomThreads / 32];
  unsigned long long t = 0;
  if (host_touches < 0)
    for (int32_t r = threadIdx.x; r < a.R; r += kRoomThreads) t += request_touches(a, r);
#pragma unroll
  for (int o = 16; o; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long total = host_touches < 0 ? 0ULL : (unsigned long long)host_touches;
    for (int w = 0; w < kRoomThreads / 32; w++) total += part[w];
    DevX x;
    RoomOps<DevX>::decide(x, tv, total);
  }
}

// Σ n_hashes[0..R): the touches a batch that commits as it schedules may make (every request's pick is still unknown).  decide:
// take the room decision for them (a reserved index), else write the sum to *out.
__global__ void __launch_bounds__(kRoomThreads) index_room_rows_kernel(TableView* tv, const uint16_t* n_hashes, int32_t R, int decide,
                                                                       unsigned long long* out) {
  __shared__ unsigned long long part[kRoomThreads / 32];
  unsigned long long t = 0;
  for (int32_t r = threadIdx.x; r < R; r += kRoomThreads) t += n_hashes[r];
#pragma unroll
  for (int o = 16; o; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long total = 0;
    for (int w = 0; w < kRoomThreads / 32; w++) total += part[w];
    DevX x;
    if (decide) RoomOps<DevX>::decide(x, tv, total);
    else *out = total;
  }
}

__global__ void __launch_bounds__(kRebuildThreads) table_clear_spare_kernel(TableView* tv) {
  DevX x;
  if (x.ld32(&tv->room) != kRoomRebuild) return;
  const uint64_t words = (tv->mask + 1) * (sizeof(TSlot) / 4);
  uint32_t* w = reinterpret_cast<uint32_t*>(tv->spare);
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (uint64_t)gridDim.x * blockDim.x)
    RoomOps<DevX>::clear_spare_word(x, w, i);
}

// Rehashes the live slots into the (cleared) spare; the last CTA to finish swaps the two tables in the descriptor.
__global__ void __launch_bounds__(kRebuildThreads) table_rebuild_kernel(TableView* tv) {
  DevX x;
  if (x.ld32(&tv->room) != kRoomRebuild) return;
  const TSlot* old = tv->slots;
  TSlot* ns = tv->spare;
  const uint64_t mask = tv->mask;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= mask; i += (uint64_t)gridDim.x * blockDim.x)
    RoomOps<DevX>::rehash_slot(x, old + i, ns, mask);
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&tv->rebuild_done, 1u) == gridDim.x - 1) {
      __threadfence();
      RoomOps<DevX>::swap(tv);
      tv->rebuild_done = 0;
    }
  }
}

// Σ lru.Len() over the endpoints (prefix_indexer_size metric, metrics.go:349)
__global__ void lru_total_kernel(const LruView* lv, unsigned long long* out) {
  unsigned long long t = 0;
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < lv->n_endpoints; p += gridDim.x * blockDim.x)
    if (lv->desc[p].created) t += lv->desc[p].live;
  if (t) atomicAdd(out, t);
}

// ---------------------------------------------------------------------------------------------
// DeviceIndex
// ---------------------------------------------------------------------------------------------
#define IX_CK(call)                     \
  do {                                  \
    cudaError_t _c = (call);            \
    if (_c != cudaSuccess) return _c;   \
  } while (0)

DeviceIndex::DeviceIndex(int32_t n_endpoints, int32_t row_words, int64_t capacity_hashes, int32_t default_lru, int32_t lru_max)
    : n_endpoints_(n_endpoints), row_words_(row_words), default_lru_(default_lru < 1 ? 1 : default_lru) {
  max_cap_ = (uint32_t)std::max(default_lru_, lru_max);
  if (capacity_hashes < 16) capacity_hashes = 16;
  init_capacity_ = capacity_hashes;
}

DeviceIndex::~DeviceIndex() {
  if (d_slots_) cudaFree(d_slots_);
  if (d_spare_) cudaFree(d_spare_);
  if (d_ovf_rows_) cudaFree(d_ovf_rows_);
  if (d_ovf_free_) cudaFree(d_ovf_free_);
  if (d_tv_) cudaFree(d_tv_);
  if (d_lv_) cudaFree(d_lv_);
  if (d_desc_) cudaFree(d_desc_);
  if (d_maps_) cudaFree(d_maps_);
  if (d_logs_) cudaFree(d_logs_);
  if (d_capreq_) cudaFree(d_capreq_);
  if (d_scratch_) cudaFree(d_scratch_);
  if (h_snap_) cudaFreeHost(h_snap_);
  if (ev_snap_) cudaEventDestroy(ev_snap_);
}

cudaError_t DeviceIndex::init(cudaStream_t s) {
  uint64_t c = 32;
  while (c < (uint64_t)init_capacity_ * 2) c <<= 1;
  IX_CK(cudaMalloc(&d_slots_, c * sizeof(TSlot)));
  IX_CK(cudaMemsetAsync(d_slots_, 0xFF, c * sizeof(TSlot), s));
  IX_CK(cudaMalloc(&d_tv_, sizeof(TableView)));
  IX_CK(cudaHostAlloc(&h_snap_, sizeof(TableView), cudaHostAllocDefault));
  IX_CK(cudaEventCreateWithFlags(&ev_snap_, cudaEventDisableTiming));
  IX_CK(cudaMalloc(&d_scratch_, 64));
  memset(&tv_, 0, sizeof(tv_));
  tv_.slots = d_slots_;
  tv_.mask = c - 1;
  tv_.row_words = (uint32_t)row_words_;
  memcpy(h_snap_, &tv_, sizeof(tv_));
  IX_CK(cudaMemcpyAsync(d_tv_, h_snap_, sizeof(TableView), cudaMemcpyHostToDevice, s));
  IX_CK(cudaStreamSynchronize(s));
  snap_pending_ = false;
  return cudaSuccess;
}

// exact counters of the table as of the last mutating launch
cudaError_t DeviceIndex::refresh() {
  if (snap_pending_) {
    IX_CK(cudaEventSynchronize(ev_snap_));
    snap_pending_ = false;
    const TableView* h = h_snap_;
    tv_.used = h->used;
    tv_.live = h->live;
    tv_.ovf_next = h->ovf_next;
    tv_.ovf_free_top = h->ovf_free_top;
    tv_.error = h->error;
    tv_.rebuilds = h->rebuilds;
    tv_.skips = h->skips;
  }
  return cudaSuccess;
}
// the whole descriptor as of every mutation enqueued on `s` (synchronous): after graph replays, and before a reservation
cudaError_t DeviceIndex::read_exact(cudaStream_t s) {
  IX_CK(cudaStreamSynchronize(s));
  IX_CK(cudaMemcpy(&tv_, d_tv_, sizeof(tv_), cudaMemcpyDeviceToHost));
  d_slots_ = tv_.slots;  // the device may have swapped the table with its spare
  d_spare_ = tv_.spare;
  snap_pending_ = false;
  captured_ = false;
  return cudaSuccess;
}
cudaError_t DeviceIndex::snapshot_after(cudaStream_t s) {
  IX_CK(cudaMemcpyAsync(h_snap_, d_tv_, sizeof(TableView), cudaMemcpyDeviceToHost, s));
  IX_CK(cudaEventRecord(ev_snap_, s));
  snap_pending_ = true;
  return cudaSuccess;
}

// Moves the live slots into a new table of ncap slots (dead slots dropped) and points the descriptor at it; synchronous.
cudaError_t DeviceIndex::rehash_into(uint64_t ncap, cudaStream_t s) {
  const uint64_t cap = tv_.mask + 1;
  TSlot* ns = nullptr;
  IX_CK(cudaMalloc(&ns, ncap * sizeof(TSlot)));
  IX_CK(cudaMemsetAsync(ns, 0xFF, ncap * sizeof(TSlot), s));
  TableView nv = tv_;
  nv.slots = ns;
  nv.mask = ncap - 1;
  nv.used = 0;
  nv.live = 0;
  IX_CK(cudaMemcpyAsync(d_tv_, &nv, sizeof(nv), cudaMemcpyHostToDevice, s));  // pageable source: staged before return
  table_rehash_kernel<<<1184, 256, 0, s>>>(d_slots_, cap, d_tv_);
  launches_++;
  IX_CK(cudaGetLastError());
  IX_CK(cudaStreamSynchronize(s));  // rare (amortised over >= cap/4 touches); lets the old array go right away
  cudaFree(d_slots_);
  d_slots_ = ns;
  tv_.slots = ns;
  tv_.mask = ncap - 1;
  tv_.used = tv_.live;  // d_tv_ already holds the new view (counters were rebuilt by the kernel)
  rebuilds_++;
  return cudaSuccess;
}

// Replaces the overflow pool with one of ncap rows holding the same rows and free list; synchronous.
cudaError_t DeviceIndex::grow_pool(uint64_t ncap, cudaStream_t s) {
  if (ncap >= 0xFFFFFFF0ULL) return cudaErrorMemoryAllocation;
  uint32_t* nr = nullptr;
  uint32_t* nf = nullptr;
  IX_CK(cudaMalloc(&nr, ncap * (size_t)row_words_ * 4));
  IX_CK(cudaMalloc(&nf, ncap * 4));
  if (tv_.ovf_next) IX_CK(cudaMemcpyAsync(nr, d_ovf_rows_, (size_t)tv_.ovf_next * row_words_ * 4, cudaMemcpyDeviceToDevice, s));
  if (tv_.ovf_free_top) IX_CK(cudaMemcpyAsync(nf, d_ovf_free_, (size_t)tv_.ovf_free_top * 4, cudaMemcpyDeviceToDevice, s));
  IX_CK(cudaStreamSynchronize(s));
  if (d_ovf_rows_) cudaFree(d_ovf_rows_);
  if (d_ovf_free_) cudaFree(d_ovf_free_);
  d_ovf_rows_ = nr;
  d_ovf_free_ = nf;
  tv_.ovf_rows = nr;
  tv_.ovf_free = nf;
  tv_.ovf_cap = (uint32_t)ncap;
  // only the pointer/capacity fields change; the counters on the device are current (no launch in flight: the caller waited)
  IX_CK(cudaMemcpyAsync(&d_tv_->ovf_rows, &tv_.ovf_rows, sizeof(tv_.ovf_rows), cudaMemcpyHostToDevice, s));
  IX_CK(cudaMemcpyAsync(&d_tv_->ovf_cap, &tv_.ovf_cap, sizeof(tv_.ovf_cap), cudaMemcpyHostToDevice, s));
  IX_CK(cudaMemcpyAsync(&d_tv_->ovf_free, &tv_.ovf_free, sizeof(tv_.ovf_free), cudaMemcpyHostToDevice, s));
  IX_CK(cudaStreamSynchronize(s));
  return cudaSuccess;
}

// Make room for `touches` more set_member calls: each may claim one slot and one overflow row.
cudaError_t DeviceIndex::ensure_room(int64_t touches, cudaStream_t s) {
  IX_CK(refresh());
  const uint64_t cap = tv_.mask + 1;
  if ((tv_.used + (uint64_t)touches) * 2 > cap) {
    // rebuild: same size when dropping the dead slots is enough (live + touches <= cap/4), else the next power of two
    uint64_t ncap = cap;
    while ((tv_.live + (uint64_t)touches) * 4 > ncap) ncap <<= 1;
    IX_CK(rehash_into(ncap, s));
  }
  const uint64_t in_use = (uint64_t)tv_.ovf_next - tv_.ovf_free_top;
  if (in_use + (uint64_t)touches > tv_.ovf_cap) IX_CK(grow_pool(std::max<uint64_t>((in_use + (uint64_t)touches) * 5 / 4, 1024), s));
  return cudaSuccess;
}

cudaError_t DeviceIndex::reserve(int64_t live_hashes, int64_t touches_per_call, int64_t overflow_rows, cudaStream_t s) {
  IX_CK(read_exact(s));
  uint64_t want = 32;
  while (want < 4 * (uint64_t)(live_hashes + touches_per_call)) want <<= 1;
  const bool grow = want > tv_.mask + 1;
  if (grow) IX_CK(rehash_into(want, s));
  if (grow || !d_spare_) {  // the spare needs no contents: every rebuild clears it first
    if (d_spare_) cudaFree(d_spare_);
    d_spare_ = nullptr;
    IX_CK(cudaMalloc(&d_spare_, (tv_.mask + 1) * sizeof(TSlot)));
    tv_.spare = d_spare_;
  }
  if ((uint64_t)overflow_rows > tv_.ovf_cap) IX_CK(grow_pool((uint64_t)overflow_rows, s));
  IX_CK(ensure_lru(0, s));
  tv_.room = kRoomProceed;
  tv_.rebuild_done = 0;
  IX_CK(cudaMemcpyAsync(d_tv_, &tv_, sizeof(tv_), cudaMemcpyHostToDevice, s));
  IX_CK(cudaStreamSynchronize(s));
  reserved_ = true;
  return cudaSuccess;
}

cudaError_t DeviceIndex::new_skips(bool exact, cudaStream_t s, bool* out) {
  if (exact || captured_) IX_CK(read_exact(s));
  else if (snap_pending_ && cudaEventQuery(ev_snap_) == cudaSuccess) IX_CK(refresh());
  *out = tv_.skips > skips_seen_;
  skips_seen_ = tv_.skips;
  return cudaSuccess;
}

void DeviceIndex::launch_room(const CommitArgs& a, long long host_touches, cudaStream_t s) {
  index_room_kernel<<<1, kRoomThreads, 0, s>>>(d_tv_, a, host_touches);
  table_clear_spare_kernel<<<kRebuildCtas, kRebuildThreads, 0, s>>>(d_tv_);
  table_rebuild_kernel<<<kRebuildCtas, kRebuildThreads, 0, s>>>(d_tv_);
  launches_ += 3;
}

cudaError_t DeviceIndex::ensure_lru(uint32_t want_cap, cudaStream_t s) {
  if (d_lv_) return cudaSuccess;
  if (want_cap > max_cap_) max_cap_ = want_cap;
  lv_.map_size = lru_map_size_for(max_cap_);
  lv_.log_size = lru_log_size_for(max_cap_);
  lv_.default_cap = (uint32_t)default_lru_;
  lv_.max_cap = max_cap_;
  lv_.n_endpoints = (uint32_t)n_endpoints_;
  lv_.error = 0;
  const size_t n = (size_t)n_endpoints_;
  IX_CK(cudaMalloc(&d_desc_, n * sizeof(LruDesc)));
  IX_CK(cudaMalloc(&d_maps_, n * lv_.map_size * sizeof(LruEntry)));
  IX_CK(cudaMalloc(&d_logs_, n * lv_.log_size * sizeof(uint64_t)));
  IX_CK(cudaMalloc(&d_lv_, sizeof(LruView)));
  IX_CK(cudaMalloc(&d_capreq_, n * sizeof(int32_t)));
  IX_CK(cudaMemsetAsync(d_desc_, 0, n * sizeof(LruDesc), s));
  IX_CK(cudaMemsetAsync(d_maps_, 0xFF, n * lv_.map_size * sizeof(LruEntry), s));
  lv_.desc = d_desc_;
  lv_.maps = d_maps_;
  lv_.logs = d_logs_;
  IX_CK(cudaMemcpyAsync(d_lv_, &lv_, sizeof(lv_), cudaMemcpyHostToDevice, s));
  IX_CK(cudaStreamSynchronize(s));
  cudaFuncSetAttribute(index_commit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CommitSmem));
  cudaFuncSetAttribute(index_remove_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CommitSmem));
  cudaFuncSetAttribute(index_export_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CommitSmem));
  return cudaSuccess;
}

int64_t DeviceIndex::lru_bytes() const {
  if (!d_lv_) return 0;
  return (int64_t)n_endpoints_ * ((int64_t)lv_.map_size * sizeof(LruEntry) + (int64_t)lv_.log_size * 8 + sizeof(LruDesc));
}

// PreRequest for a batch whose arrays are on the device; async on `s` (which must be the index's stream).
cudaError_t DeviceIndex::commit(int32_t R, int32_t n_picks, const int32_t* const* picks, const uint64_t* hashes,
                                const uint16_t* n_hashes, int32_t stride, const int32_t* cap_req_host, int32_t single_cap,
                                int32_t ep_first, int32_t n_eps, int64_t max_touches, cudaStream_t s, bool capturing) {
  if (R <= 0 || n_eps <= 0 || n_picks < 1 || n_picks > 4) return cudaSuccess;
  uint32_t want = (uint32_t)std::max(single_cap, 0);
  if (cap_req_host)
    for (int32_t i = 0; i < n_endpoints_; i++) want = std::max(want, (uint32_t)std::max(cap_req_host[i], 0));
  IX_CK(ensure_lru(want, s));
  if (want > lv_.max_cap) return cudaErrorInvalidValue;  // the LRU regions were sized for a smaller largest capacity
  CommitArgs a{};
  a.hashes = hashes;
  a.n_hashes = n_hashes;
  a.stride = stride;
  a.single_cap = single_cap;
  a.ep_first = ep_first;
  a.n_picks = n_picks;
  if (cap_req_host) {
    IX_CK(cudaMemcpyAsync(d_capreq_, cap_req_host, (size_t)n_endpoints_ * 4, cudaMemcpyHostToDevice, s));
    a.cap_req = d_capreq_;
  }
  // sub-batches bound the room (slots + overflow rows) that has to be guaranteed up front
  const int32_t kSub = 65536;
  for (int32_t r0 = 0; r0 < R; r0 += kSub) {
    const int32_t n = std::min(kSub, R - r0);
    a.R = n;
    a.pick = picks[0] + r0;
    for (int32_t p = 1; p < n_picks; p++) a.more_picks[p - 1] = picks[p] + r0;
    a.hashes = hashes + (size_t)r0 * stride;
    a.n_hashes = n_hashes + r0;
    if (reserved_) {  // room decided on the device: nothing here waits on the host
      launch_room(a, -1, s);
      index_commit_kernel<<<n_eps, kCommitThreads, sizeof(CommitSmem), s>>>(d_tv_, d_lv_, a);
      launches_++;
      IX_CK(cudaGetLastError());
      if (capturing) captured_ = true;
      else IX_CK(snapshot_after(s));
      continue;
    }
    int64_t touches = std::min<int64_t>(max_touches, (int64_t)n * n_picks * stride);
    if (max_touches <= 0) {  // no bound from the caller: count them (one small synchronous read-back)
      unsigned long long* d_t = reinterpret_cast<unsigned long long*>(d_scratch_);
      unsigned long long t = 0;
      IX_CK(cudaMemsetAsync(d_t, 0, 8, s));
      sum_touches_kernel<<<64, 256, 0, s>>>(a, d_t);
      launches_++;
      IX_CK(cudaMemcpyAsync(&t, d_t, 8, cudaMemcpyDeviceToHost, s));
      IX_CK(cudaStreamSynchronize(s));
      touches = (int64_t)t;
    }
    if (touches < 1) touches = 1;
    IX_CK(ensure_room(touches, s));
    index_commit_kernel<<<n_eps, kCommitThreads, sizeof(CommitSmem), s>>>(d_tv_, d_lv_, a);
    launches_++;
    IX_CK(cudaGetLastError());
    IX_CK(snapshot_after(s));
  }
  return cudaSuccess;
}

cudaError_t DeviceIndex::ordered_begin(const int32_t* cap_req_host, cudaStream_t s, OrderedRefs* out) {
  uint32_t want = 0;
  if (cap_req_host)
    for (int32_t i = 0; i < n_endpoints_; i++) want = std::max(want, (uint32_t)std::max(cap_req_host[i], 0));
  IX_CK(ensure_lru(want, s));
  if (want > lv_.max_cap) return cudaErrorInvalidValue;  // the LRU regions were sized for a smaller largest capacity
  if (cap_req_host) IX_CK(cudaMemcpyAsync(d_capreq_, cap_req_host, (size_t)n_endpoints_ * 4, cudaMemcpyHostToDevice, s));
  out->tv = d_tv_;
  out->lv = d_lv_;
  out->cap_req = cap_req_host ? d_capreq_ : nullptr;
  return cudaSuccess;
}

cudaError_t DeviceIndex::ordered_room(int32_t R, const uint16_t* n_hashes, cudaStream_t s) {
  if (R <= 0) return cudaSuccess;
  if (reserved_) {  // room decided on the device: nothing here waits on the host
    index_room_rows_kernel<<<1, kRoomThreads, 0, s>>>(d_tv_, n_hashes, R, 1, nullptr);
    table_clear_spare_kernel<<<kRebuildCtas, kRebuildThreads, 0, s>>>(d_tv_);
    table_rebuild_kernel<<<kRebuildCtas, kRebuildThreads, 0, s>>>(d_tv_);
    launches_ += 3;
    return cudaGetLastError();
  }
  unsigned long long* d_t = reinterpret_cast<unsigned long long*>(d_scratch_);
  unsigned long long t = 0;
  index_room_rows_kernel<<<1, kRoomThreads, 0, s>>>(d_tv_, n_hashes, R, 0, d_t);
  launches_++;
  IX_CK(cudaMemcpyAsync(&t, d_t, 8, cudaMemcpyDeviceToHost, s));
  IX_CK(cudaStreamSynchronize(s));
  return ensure_room(std::max<int64_t>((int64_t)t, 1), s);
}

cudaError_t DeviceIndex::ordered_end(cudaStream_t s, bool capturing) {
  if (capturing) {
    captured_ = true;
    return cudaSuccess;
  }
  return snapshot_after(s);
}

void DeviceIndex::match(int32_t R, int32_t k, int32_t limit, const uint64_t* hashes, const uint16_t* n_hashes, int32_t stride,
                        const int32_t* endpoints, uint16_t* out, cudaStream_t s) {
  const int32_t ctas = std::min((R + kMatchThreads / 32 - 1) / (kMatchThreads / 32), 8192);
  prefix_match_kernel<<<ctas, kMatchThreads, 0, s>>>(d_tv_, R, k, (uint32_t)limit, hashes, n_hashes, stride, endpoints, out);
  launches_++;
}

void DeviceIndex::latency_info(const LatInfoArgs& a, int32_t limit, cudaStream_t s) {
  const int32_t ctas = std::min((a.R + kMatchThreads / 32 - 1) / (kMatchThreads / 32), 8192);
  latency_info_kernel<<<ctas, kMatchThreads, 0, s>>>(d_tv_, (uint32_t)limit, a);
  launches_++;
}

cudaError_t DeviceIndex::apply(int64_t n, const uint64_t* hash, const int32_t* endpoint, const uint8_t* op, cudaStream_t s) {
  if (n <= 0) return cudaSuccess;
  if (reserved_) launch_room(CommitArgs{}, n, s);
  else IX_CK(ensure_room(n, s));
  index_apply_kernel<<<(n_endpoints_ + 127) / 128, 128, 0, s>>>(d_tv_, n, hash, endpoint, op, (uint32_t)n_endpoints_);
  launches_++;
  IX_CK(cudaGetLastError());
  return snapshot_after(s);
}

cudaError_t DeviceIndex::remove_endpoint(int32_t p, cudaStream_t s) {
  if (!d_lv_ || p < 0 || p >= n_endpoints_) return cudaSuccess;
  if (!reserved_) IX_CK(refresh());  // (frees slots and rows only: no room to check)
  index_remove_kernel<<<1, kCommitThreads, sizeof(CommitSmem), s>>>(d_tv_, d_lv_, (uint32_t)p);
  launches_++;
  IX_CK(cudaGetLastError());
  return snapshot_after(s);
}

// lru.Len() / lru.Keys() of one endpoint (synchronous; tests and diagnostics). Returns -1 when the endpoint has no LRU.
cudaError_t DeviceIndex::lru_keys(int32_t p, uint64_t* out_host, int32_t cap, int32_t* len, cudaStream_t s) {
  *len = -1;
  if (!d_lv_ || p < 0 || p >= n_endpoints_) return cudaSuccess;
  const uint32_t want = cap > 0 ? (uint32_t)cap : 0u;
  uint64_t* d_keys = nullptr;
  uint32_t* d_len = nullptr;
  IX_CK(cudaMalloc(&d_keys, std::max<size_t>((size_t)want, 1) * 8));
  IX_CK(cudaMalloc(&d_len, 4));
  index_export_kernel<<<1, kCommitThreads, sizeof(CommitSmem), s>>>(d_tv_, d_lv_, (uint32_t)p, d_keys, want, d_len);
  launches_++;
  uint32_t n = 0;
  cudaError_t e = cudaMemcpyAsync(&n, d_len, 4, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e == cudaSuccess && n != 0xFFFFFFFFu) {
    *len = (int32_t)n;
    const uint32_t m = std::min(n, want);
    if (m && out_host) e = cudaMemcpy(out_host, d_keys, (size_t)m * 8, cudaMemcpyDeviceToHost);
  }
  cudaFree(d_keys);
  cudaFree(d_len);
  return e;
}

cudaError_t DeviceIndex::get(uint64_t h, uint32_t* bits_host, int32_t words, int32_t* count, cudaStream_t s) {
  uint32_t* d_out = nullptr;
  const uint32_t w = (uint32_t)row_words_;
  IX_CK(cudaMalloc(&d_out, (size_t)(w + 1) * 4));
  table_get_kernel<<<1, 32, 0, s>>>(d_tv_, h, d_out, w);
  launches_++;
  std::vector<uint32_t> host((size_t)w + 1);
  cudaError_t e = cudaMemcpyAsync(host.data(), d_out, host.size() * 4, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  cudaFree(d_out);
  if (e != cudaSuccess) return e;
  *count = (int32_t)host[0];
  if (bits_host)
    for (int32_t i = 0; i < words; i++) bits_host[i] = (uint32_t)i < w ? host[1 + i] : 0u;
  return cudaSuccess;
}

cudaError_t DeviceIndex::stats(IndexStats* out, cudaStream_t s) {
  IX_CK(cudaStreamSynchronize(s));
  IX_CK(refresh());
  TableView h;
  IX_CK(cudaMemcpy(&h, d_tv_, sizeof(h), cudaMemcpyDeviceToHost));
  out->used = (int64_t)h.used;
  out->live = (int64_t)h.live;
  out->capacity = (int64_t)((h.mask + 1) / 2);
  out->ovf_rows = (int64_t)h.ovf_next - (int64_t)h.ovf_free_top;
  out->table_bytes = (int64_t)((h.mask + 1) * sizeof(TSlot)) * (h.spare ? 2 : 1) + (int64_t)h.ovf_cap * row_words_ * 4;
  out->lru_bytes = lru_bytes();
  out->error = h.error;
  out->rebuilds = rebuilds_ + (int64_t)h.rebuilds;
  out->lru_entries = 0;
  if (d_lv_) {
    unsigned long long* d_t = reinterpret_cast<unsigned long long*>(d_scratch_);
    IX_CK(cudaMemsetAsync(d_t, 0, 8, s));
    lru_total_kernel<<<8, 256, 0, s>>>(d_lv_, d_t);
    launches_++;
    unsigned long long t = 0;
    IX_CK(cudaMemcpyAsync(&t, d_t, 8, cudaMemcpyDeviceToHost, s));
    IX_CK(cudaStreamSynchronize(s));
    out->lru_entries = (int64_t)t;
    LruView lvh;
    IX_CK(cudaMemcpy(&lvh, d_lv_, sizeof(lvh), cudaMemcpyDeviceToHost));
    out->error |= lvh.error << 8;
  }
  return cudaSuccess;
}

}  // namespace eppscore
