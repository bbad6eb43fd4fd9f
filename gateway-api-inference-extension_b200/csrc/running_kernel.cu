// running_kernel.cu — the predicted-latency producer's running-request queues (predictedlatency/
// running_request_tpot_slo_queue.go, requestcontrol_hooks.go:73-86,219, plugin.go:190-196,347-363) on the device.
//
// One open-addressing table holds every live (endpoint, request key) -> tpot entry of every endpoint; per endpoint the engine
// keeps the live count, the smallest live tpot (as the bit pattern of a non-negative double: those order like their bits, so
// an unsigned atomicMin is exact) and the number of live entries equal to that minimum.  A call is a fixed sequence of
// launches (legal under CUDA-graph capture):
//   add:    running_claim_kernel (lowest r wins each new key) -> running_apply_kernel (count, min) -> running_mincount_kernel
//           -> running_finalize_kernel
//   remove: running_claim_kernel (lowest r wins each live key) -> running_apply_kernel (tombstones, count, count at min)
//           -> running_recompute_kernel x2 (endpoints whose last minimum left; exit at once when there are none)
//           -> running_finalize_kernel
// The apply kernels have the structure of inflight_update_kernel: lanes of a warp that name the same endpoint are combined
// (__match_any_sync), each group updates a per-CTA shared-memory histogram once, and each CTA issues one global atomic per
// endpoint it saw, so 64K entries on one endpoint do not serialise on one address.
#include "running_slot.cuh"

namespace eppscore {

constexpr int kRunThreads = 512;
constexpr int kRunPerCta = 4096;  // entries per CTA of the apply kernels: the histogram is zeroed and flushed once per 4096

__device__ __forceinline__ bool run_live(unsigned long long meta) { return meta != 0ull && !(meta & kRunTomb); }

// claim: one thread per entry.  add (op 0): validates the entry, finds or creates the (endpoint, key) slot (run_find_or_create:
// two entries of the call with the same pair meet in one slot) and bids (gen << 32 | r) for
// it with atomicMin.  A slot that existed before the call holds an older generation and always wins: the add is refused.
// remove (op 1): finds the live slot and bids the same way; the lowest r removes it.  slot_of[r] = slot, or -1.
__global__ void running_claim_kernel(const RunDev* __restrict__ dp, int op, const int32_t* __restrict__ endpoint,
                                     const uint64_t* __restrict__ key, const double* __restrict__ tpot, int R, int n_ep) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const RunDev d = *dp;
  int32_t* slot_of = d.slot_of;
  slot_of[r] = -1;
  const int m = endpoint[r];
  if (m < 0) return;  // unscheduled request (pick -1)
  double t = 0.0;
  if (op == 0 && tpot) t = tpot[r];
  if (m >= n_ep || t != t) {  // host-array calls are validated before the launch; a device array may still hold these
    atomicOr(&d.ctr->err, kRunErrInvalid);
    return;
  }
  const unsigned long long k = key[r];
  if (k == 0ull || t < 0.0) return;  // empty x-request-id, negative tpot: refused (running_request_tpot_slo_queue.go:127-132)
  const unsigned long long bid = ((unsigned long long)d.ctr->gen << 32) | (unsigned)r;
  if (op == 0) {
    bool created;
    const long long h = run_find_or_create(d, k, m, &created);
    if (h < 0) {
      atomicOr(&d.ctr->err, kRunErrCapacity);
      return;
    }
    atomicMin(&d.owner[h], bid);
    slot_of[r] = (int32_t)h;
    return;
  }
  const unsigned long long want_meta = (unsigned long long)(m + 1);
  unsigned long long h = run_hash(k, m) & d.mask;
  for (unsigned long long i = 0; i <= d.mask; i++, h = (h + 1) & d.mask) {
    const RunSlot cur = d.slot[h];  // nothing creates or tombstones slots during a remove's claim
    if (cur.key == 0ull && cur.meta == 0ull) return;  // an empty slot ends the chain: the pair is not live
    if (cur.key == k && cur.meta == want_meta) {
      atomicMin(&d.rm[h], bid);
      slot_of[r] = (int32_t)h;
      return;
    }
  }
}

// apply: the winners of the claim.  add: store tpot, count += n, min = min(min, tpot); an endpoint whose minimum went down
// restarts its count at the minimum from 0 (every older entry is above the new minimum).  remove: tombstone, count -= n,
// count at the minimum -= (winners equal to the minimum); the endpoint whose count at the minimum reaches 0 is marked dirty.
// won[r] (and out[r] when given) = 1 for a winner.
__global__ void __launch_bounds__(kRunThreads) running_apply_kernel(const RunDev* __restrict__ dp, int op,
                                                                   const int32_t* __restrict__ endpoint,
                                                                   const double* __restrict__ tpot, int R, int n_ep,
                                                                   uint8_t* __restrict__ out) {
  const RunDev d = *dp;
  const int32_t* slot_of = d.slot_of;
  uint8_t* won = d.won;
  extern __shared__ unsigned long long s_aux[];  // [n_ep] min bits (add) or count at the minimum (remove), then [n_ep] int32
  int* s_cnt = reinterpret_cast<int*>(s_aux + n_ep);
  __shared__ unsigned long long s_val[kRunThreads];
  __shared__ int s_total;
  for (int i = threadIdx.x; i < n_ep; i += blockDim.x) {
    s_aux[i] = op == 0 ? kRunMinNone : 0ull;
    s_cnt[i] = 0;
  }
  if (threadIdx.x == 0) s_total = 0;
  __syncthreads();
  const unsigned long long gen = d.ctr->gen;
  const int lane = threadIdx.x & 31, wbase = threadIdx.x & ~31;
  const int lo = blockIdx.x * kRunPerCta, hi = min(R, lo + kRunPerCta);
  for (int base = lo; base < hi; base += blockDim.x) {  // base is uniform per CTA: whole warps take every iteration
    const int r = base + threadIdx.x;
    int m = -1;
    unsigned long long v = 0ull;
    if (r < hi) {
      const int h = slot_of[r];
      bool win = false;
      if (h >= 0) {
        win = (op == 0 ? d.owner[h] : d.rm[h]) == ((gen << 32) | (unsigned)r);
        if (win) {
          m = endpoint[r];
          if (op == 0) {
            const double t = tpot ? tpot[r] : 0.0;
            v = t == 0.0 ? 0ull : (unsigned long long)__double_as_longlong(t);  // -0.0 is stored as +0.0
            d.tpot[h] = v;
          } else {
            d.slot[h].meta = (unsigned long long)(m + 1) | kRunTomb;
            v = d.tpot[h] == d.min_bits[m] ? 1ull : 0ull;
          }
        }
      }
      won[r] = win ? 1 : 0;
      if (out) out[r] = win ? 1 : 0;
    }
    const unsigned peers = __match_any_sync(0xffffffffu, m);
    s_val[threadIdx.x] = v;
    __syncwarp();
    if (m >= 0 && lane == __ffs(peers) - 1) {
      unsigned long long a = op == 0 ? kRunMinNone : 0ull;
      for (unsigned p = peers; p; p &= p - 1) {
        const unsigned long long x = s_val[wbase + __ffs(p) - 1];
        a = op == 0 ? min(a, x) : a + x;
      }
      if (op == 0) atomicMin(&s_aux[m], a);
      else atomicAdd(&s_aux[m], a);
      atomicAdd(&s_cnt[m], __popc(peers));
      atomicAdd(&s_total, __popc(peers));
    }
    __syncwarp();
  }
  __syncthreads();
  for (int m = threadIdx.x; m < n_ep; m += blockDim.x) {
    const int c = s_cnt[m];
    if (c == 0) continue;  // no winner of this CTA named m
    if (op == 0) {
      atomicAdd(&d.count[m], c);
      const unsigned long long old = atomicMin(&d.min_bits[m], s_aux[m]);
      if (s_aux[m] < old) d.min_cnt[m] = 0;  // every CTA that lowers the minimum writes the same 0; counted again next kernel
    } else {
      atomicSub(&d.count[m], c);
      const int at_min = (int)s_aux[m];
      if (at_min > 0 && atomicSub(&d.min_cnt[m], at_min) == at_min) {
        d.dirty[m] = 1u;
        d.ctr->any_dirty = 1u;
      }
    }
  }
  if (threadIdx.x == 0 && s_total > 0) {
    atomicAdd(&d.ctr->live, op == 0 ? (unsigned long long)s_total : 0ull - (unsigned long long)s_total);
    if (op == 1) atomicAdd(&d.ctr->tomb, (unsigned long long)s_total);
  }
}

// add, after apply: every winner equal to its endpoint's (final) minimum adds 1 to the count at the minimum
__global__ void __launch_bounds__(kRunThreads) running_mincount_kernel(const RunDev* __restrict__ dp,
                                                                      const int32_t* __restrict__ endpoint, int R, int n_ep) {
  const RunDev d = *dp;
  const int32_t* slot_of = d.slot_of;
  const uint8_t* won = d.won;
  extern __shared__ unsigned long long s_aux[];
  int* s_cnt = reinterpret_cast<int*>(s_aux + n_ep);
  for (int i = threadIdx.x; i < n_ep; i += blockDim.x) s_cnt[i] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int lo = blockIdx.x * kRunPerCta, hi = min(R, lo + kRunPerCta);
  for (int base = lo; base < hi; base += blockDim.x) {
    const int r = base + threadIdx.x;
    int m = -1;
    if (r < hi && won[r]) {
      const int e = endpoint[r];
      if (d.tpot[slot_of[r]] == d.min_bits[e]) m = e;
    }
    const unsigned peers = __match_any_sync(0xffffffffu, m);
    if (m >= 0 && lane == __ffs(peers) - 1) atomicAdd(&s_cnt[m], __popc(peers));
  }
  __syncthreads();
  for (int m = threadIdx.x; m < n_ep; m += blockDim.x)
    if (s_cnt[m]) atomicAdd(&d.min_cnt[m], s_cnt[m]);
}

// remove, after apply: for the dirty endpoints only, pass 0 takes the minimum over their live entries into rc_min, pass 1
// counts the entries equal to it into rc_cnt.  Launched after every remove with a fixed grid; returns at once when no
// endpoint is dirty.  The cost is one read of the table, whatever the history.
__global__ void running_recompute_kernel(const RunDev* __restrict__ dp, int pass) {
  const RunDev d = *dp;
  if (d.ctr->any_dirty == 0u) return;
  const int lane = threadIdx.x & 31, wbase = threadIdx.x & ~31;
  __shared__ unsigned long long s_val[256];
  const unsigned long long cap = d.mask + 1;
  for (unsigned long long base = (unsigned long long)blockIdx.x * blockDim.x; base < cap; base += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long h = base + threadIdx.x;
    int m = -1;
    unsigned long long v = 0ull;
    if (h < cap) {
      const unsigned long long meta = d.slot[h].meta;
      if (run_live(meta) && d.dirty[(int)meta - 1]) {
        m = (int)meta - 1;
        v = d.tpot[h];
        if (pass == 1 && v != d.rc_min[m]) m = -1;
      }
    }
    const unsigned peers = __match_any_sync(0xffffffffu, m);
    s_val[threadIdx.x] = v;
    __syncwarp();
    if (m >= 0 && lane == __ffs(peers) - 1) {
      if (pass == 0) {
        unsigned long long a = kRunMinNone;
        for (unsigned p = peers; p; p &= p - 1) a = min(a, s_val[wbase + __ffs(p) - 1]);
        atomicMin(&d.rc_min[m], a);
      } else {
        atomicAdd(&d.rc_cnt[m], __popc(peers));
      }
    }
    __syncwarp();
  }
}

// The end of every call: dirty endpoints take the recomputed minimum (kRunMinNone when empty), the scratch is reset, the
// view the scorer reads is written (min_view = the minimum, 0 without a live entry: plugin.go:349-354), and the generation
// advances.  One thread per endpoint.
__global__ void running_finalize_kernel(const RunDev* __restrict__ dp, int n_ep) {
  const RunDev d = *dp;
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m == 0) {
    d.ctr->gen += 1u;
    d.ctr->any_dirty = 0u;
  }
  if (m >= n_ep) return;
  if (d.dirty[m]) {
    d.min_bits[m] = d.rc_min[m];
    d.min_cnt[m] = d.rc_cnt[m];
    d.rc_min[m] = kRunMinNone;
    d.rc_cnt[m] = 0;
    d.dirty[m] = 0u;
  }
  d.min_view[m] = d.count[m] > 0 ? __longlong_as_double((long long)d.min_bits[m]) : 0.0;
}

// remove_endpoint: every live entry of m becomes a tombstone; its count, minimum and count at the minimum start over
__global__ void running_drop_endpoint_kernel(const RunDev* __restrict__ dp, int m) {
  const RunDev d = *dp;
  const unsigned long long cap = d.mask + 1;
  const unsigned long long want = (unsigned long long)(m + 1);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    d.count[m] = 0;
    d.min_bits[m] = kRunMinNone;
    d.min_cnt[m] = 0;
  }
  for (unsigned long long h = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; h < cap; h += (unsigned long long)gridDim.x * blockDim.x) {
    if (d.slot[h].meta == want) {
      d.slot[h].meta = want | kRunTomb;
      atomicAdd(&d.ctr->live, 0ull - 1ull);
      atomicAdd(&d.ctr->tomb, 1ull);
    }
  }
}

// rebuild: every live entry of `src` is inserted into the empty table `dst` (keys are distinct: no duplicate check), with an
// owner word older than any generation and no remove bid; the tombstones stay behind.
__global__ void running_rebuild_kernel(RunDev src, RunDev dst) {
  const unsigned long long cap = src.mask + 1;
  if (blockIdx.x == 0 && threadIdx.x == 0) dst.ctr->tomb = 0ull;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (unsigned long long)gridDim.x * blockDim.x) {
    const RunSlot s = src.slot[i];
    if (!run_live(s.meta)) continue;
    unsigned long long h = run_hash(s.key, (int)s.meta - 1) & dst.mask;
    while (true) {
      const RunSlot cur = atomicCAS(&dst.slot[h], RunSlot{0ull, 0ull}, s);
      if (cur.key == 0ull && cur.meta == 0ull) break;
      h = (h + 1) & dst.mask;
    }
    dst.tpot[h] = src.tpot[i];
    dst.owner[h] = 0ull;
  }
}

// Compaction before every add, on the device so that it also runs inside a captured graph: when live + tombstones + R would
// pass half the slots, the live entries move into the spare table of the same size (cleared first) and the two swap places
// in the device descriptor; tombstones go.  The three launches read the same counters (nothing changes them in between), so
// they agree on whether to act; each returns at once when not.
__device__ __forceinline__ bool run_compact_due(const RunDev& d, int R) {
  return 2 * (d.ctr->live + d.ctr->tomb + (unsigned long long)R) > d.mask + 1;
}
__global__ void running_compact_clear_kernel(const RunDev* __restrict__ dp, int R) {
  const RunDev d = *dp;
  if (!run_compact_due(d, R)) return;
  for (unsigned long long h = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; h <= d.mask; h += (unsigned long long)gridDim.x * blockDim.x) {
    d.spare_slot[h] = RunSlot{0ull, 0ull};
    d.spare_owner[h] = ~0ull;
    d.spare_rm[h] = ~0ull;
  }
}
__global__ void running_compact_move_kernel(const RunDev* __restrict__ dp, int R) {
  const RunDev d = *dp;
  if (!run_compact_due(d, R)) return;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i <= d.mask; i += (unsigned long long)gridDim.x * blockDim.x) {
    const RunSlot s = d.slot[i];
    if (!run_live(s.meta)) continue;
    unsigned long long h = run_hash(s.key, (int)s.meta - 1) & d.mask;
    while (true) {  // at most half the slots are live: an empty one is always found
      const RunSlot cur = atomicCAS(&d.spare_slot[h], RunSlot{0ull, 0ull}, s);
      if (cur.key == 0ull && cur.meta == 0ull) break;
      h = (h + 1) & d.mask;
    }
    d.spare_tpot[h] = d.tpot[i];
    d.spare_owner[h] = 0ull;
  }
}
__global__ void running_compact_swap_kernel(RunDev* dp, int R) {
  RunDev d = *dp;
  if (!run_compact_due(d, R)) return;
  dp->slot = d.spare_slot, dp->spare_slot = d.slot;
  dp->tpot = d.spare_tpot, dp->spare_tpot = d.tpot;
  dp->owner = d.spare_owner, dp->spare_owner = d.owner;
  dp->rm = d.spare_rm, dp->spare_rm = d.rm;
  d.ctr->tomb = 0ull;
}

cudaError_t init_running_kernels() {  // the largest histogram (8192 endpoints), as init_inflight_update
  const int smem = 8192 * (int)(sizeof(unsigned long long) + sizeof(int));
  cudaError_t c = cudaFuncSetAttribute(running_apply_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (c != cudaSuccess) return c;
  return cudaFuncSetAttribute(running_mincount_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
}

static int run_grid(unsigned long long cap, int max_ctas) {  // grid-stride passes over the table, 256 slots per thread block
  const unsigned long long want = (cap + 255) / 256;
  return want < (unsigned long long)max_ctas ? (int)want : max_ctas;
}

int launch_running_compact(RunDev* dp, unsigned long long cap, int R, int sm_count, cudaStream_t s) {
  const int g = run_grid(cap, sm_count * 4);
  running_compact_clear_kernel<<<g, 256, 0, s>>>(dp, R);
  running_compact_move_kernel<<<g, 256, 0, s>>>(dp, R);
  running_compact_swap_kernel<<<1, 1, 0, s>>>(dp, R);
  return 3;
}

int launch_running_finalize(RunDev* dp, int n_ep, cudaStream_t s) {
  running_finalize_kernel<<<(n_ep + 255) / 256, 256, 0, s>>>(dp, n_ep);
  return 1;
}

// The table passes are grid-stride loops over the descriptor's capacity, so a captured graph stays valid after the table
// grows: its grid was sized for the capacity at capture time, and its kernels read the table through `dp`.
int launch_running_update(RunDev* dp, unsigned long long cap, int op, const int32_t* endpoint, const uint64_t* key,
                          const double* tpot, int R, int n_ep, uint8_t* out, int sm_count, cudaStream_t s) {
  int n = 0;
  const size_t smem = (size_t)n_ep * (sizeof(unsigned long long) + sizeof(int));
  const int grid = (R + kRunPerCta - 1) / kRunPerCta;
  const int g = run_grid(cap, sm_count * 4);
  if (R > 0) {
    if (op == 0) n += launch_running_compact(dp, cap, R, sm_count, s);
    running_claim_kernel<<<(R + 255) / 256, 256, 0, s>>>(dp, op, endpoint, key, tpot, R, n_ep);
    running_apply_kernel<<<grid, kRunThreads, smem, s>>>(dp, op, endpoint, tpot, R, n_ep, out);
    n += 2;
    if (op == 0) {
      running_mincount_kernel<<<grid, kRunThreads, smem, s>>>(dp, endpoint, R, n_ep);
      n++;
    }
  }
  if (op == 1) {
    running_recompute_kernel<<<g, 256, 0, s>>>(dp, 0);
    running_recompute_kernel<<<g, 256, 0, s>>>(dp, 1);
    n += 2;
  }
  return n + launch_running_finalize(dp, n_ep, s);
}

int launch_running_drop_endpoint(RunDev* dp, unsigned long long cap, int m, int n_ep, int sm_count, cudaStream_t s) {
  const int g = run_grid(cap, sm_count * 4);
  running_drop_endpoint_kernel<<<g, 256, 0, s>>>(dp, m);
  return 1 + launch_running_finalize(dp, n_ep, s);
}

int launch_running_rebuild(const RunDev& src, const RunDev& dst, int sm_count, cudaStream_t s) {
  const unsigned long long cap = src.mask + 1;
  const int g = run_grid(cap, sm_count * 8);
  running_rebuild_kernel<<<g, 256, 0, s>>>(src, dst);
  return 1;
}

}  // namespace eppscore
