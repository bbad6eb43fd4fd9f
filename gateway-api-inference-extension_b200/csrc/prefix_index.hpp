// prefix_index.hpp — host-side owner of the device-resident prefix index (prefix_table.cuh, prefix_index.cu).
// Replaces approximateprefix/indexer.go's `indexer` object: the host holds no copy of hashToPods or of the LRUs, it
// sizes the device arrays and launches the kernels that maintain them.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "prefix_table.cuh"

namespace eppscore {

struct IndexStats {
  int64_t used, live, capacity, ovf_rows, table_bytes, lru_bytes, lru_entries, rebuilds;
  uint32_t error;
};

class DeviceIndex {
 public:
  // n_endpoints: endpoint ids are < n_endpoints (the engine's padded capacity); row_words = n_endpoints / 32;
  // capacity_hashes: initial table capacity (it is rebuilt / doubled on demand); lru_max: largest LRU size the engine
  // must support (0: the default size) — it fixes the per-endpoint region sizes at the first Add.
  DeviceIndex(int32_t n_endpoints, int32_t row_words, int64_t capacity_hashes, int32_t default_lru, int32_t lru_max);
  ~DeviceIndex();
  DeviceIndex(const DeviceIndex&) = delete;
  DeviceIndex& operator=(const DeviceIndex&) = delete;

  cudaError_t init(cudaStream_t s);
  const TableView* view() const { return d_tv_; }  // device pointer, stable for the engine's lifetime

  // Fixes the index's room up front (outside any capture, synchronous on `s`): a table and a spare of at least
  // 4 * (live_hashes + touches_per_call) slots, an overflow pool of at least overflow_rows rows, the LRU regions.  From then on
  // every mutation decides its room on the device (RoomOps) and never waits on the host; a later, larger reserve grows the
  // arrays behind the same descriptor.
  cudaError_t reserve(int64_t live_hashes, int64_t touches_per_call, int64_t overflow_rows, cudaStream_t s);
  bool reserved() const { return reserved_; }
  // Reserved index: whether a mutation was skipped for lack of room since the last call that said so.  exact: the device
  // counters are read synchronously; otherwise they are read from a copy-back that has already landed, and exactly once after
  // mutations were captured into a graph (their replays are invisible to the host).
  cudaError_t new_skips(bool exact, cudaStream_t s, bool* out);

  // PreRequest for R requests (device arrays), endpoints [ep_first, ep_first + n_eps): picks[0..n_picks) are [R] each, applied
  // per request in slot order (CommitArgs).  max_touches: an upper bound on Σ n_hashes over the calls (<= 0: counted on the
  // device; a reserved index ignores it).  cap_req_host: optional [n_endpoints] CacheNumBlocks.  capturing: `s` is being
  // captured into a CUDA graph (a reserved index only).
  cudaError_t commit(int32_t R, int32_t n_picks, const int32_t* const* picks, const uint64_t* hashes, const uint16_t* n_hashes, int32_t stride,
                     const int32_t* cap_req_host, int32_t single_cap, int32_t ep_first, int32_t n_eps, int64_t max_touches,
                     cudaStream_t s, bool capturing = false);
  cudaError_t apply(int64_t n, const uint64_t* hash, const int32_t* endpoint, const uint8_t* op, cudaStream_t s);  // device arrays
  cudaError_t remove_endpoint(int32_t p, cudaStream_t s);
  cudaError_t lru_keys(int32_t p, uint64_t* out_host, int32_t cap, int32_t* len, cudaStream_t s);
  cudaError_t get(uint64_t h, uint32_t* bits_host, int32_t words, int32_t* count, cudaStream_t s);
  cudaError_t stats(IndexStats* out, cudaStream_t s);
  uint64_t launches() const { return launches_; }
  uint32_t max_cap() const { return max_cap_; }

 private:
  cudaError_t refresh();
  cudaError_t snapshot_after(cudaStream_t s);
  cudaError_t ensure_room(int64_t touches, cudaStream_t s);
  cudaError_t ensure_lru(uint32_t want_cap, cudaStream_t s);
  cudaError_t rehash_into(uint64_t ncap, cudaStream_t s);
  cudaError_t grow_pool(uint64_t ncap, cudaStream_t s);
  cudaError_t read_exact(cudaStream_t s);
  void launch_room(const CommitArgs& a, long long host_touches, cudaStream_t s);
  int64_t lru_bytes() const;

  int32_t n_endpoints_, row_words_, default_lru_;
  uint32_t max_cap_ = 0;
  int64_t init_capacity_ = 0;
  TableView tv_{};          // host copy: pointers + the counters as of the last snapshot
  LruView lv_{};
  TSlot* d_slots_ = nullptr;
  TSlot* d_spare_ = nullptr;  // reserved index: the spare (the device swaps the two roles; tv_ says which is which once read)
  uint32_t* d_ovf_rows_ = nullptr;
  uint32_t* d_ovf_free_ = nullptr;
  TableView* d_tv_ = nullptr;
  LruView* d_lv_ = nullptr;
  LruDesc* d_desc_ = nullptr;
  LruEntry* d_maps_ = nullptr;
  uint64_t* d_logs_ = nullptr;
  int32_t* d_capreq_ = nullptr;
  void* d_scratch_ = nullptr;
  TableView* h_snap_ = nullptr;  // pinned
  cudaEvent_t ev_snap_ = nullptr;
  bool snap_pending_ = false;
  uint64_t launches_ = 0;
  int64_t rebuilds_ = 0;       // host-side rebuilds (the device counts its own in TableView::rebuilds)
  bool reserved_ = false;
  bool captured_ = false;      // a mutation was captured since the last exact read
  uint64_t skips_seen_ = 0;    // TableView::skips as of the last call that reported new skips
};

}  // namespace eppscore
