// running_slot.cuh — the slot probe of the running-request table (kernels.cuh: RunSlot, RunDev), shared by the add of
// running_claim_kernel and the in-order walk's Add at each pick (inorder_kernel.cu).
#pragma once
#include "kernels.cuh"

namespace eppscore {

__device__ __forceinline__ unsigned long long run_hash(unsigned long long key, int m) {
  unsigned long long x = key ^ ((unsigned long long)(m + 1) * 0x9E3779B97F4A7C15ull);  // splitmix64 finaliser
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// The (endpoint m, key) slot of an add: found, or created by one 16-byte CAS of an empty slot, so two adds of the same pair
// meet in one slot.  *created: this call created it.  -1 when no empty slot is left (only a graph replayed past its reserve).
__device__ __forceinline__ long long run_find_or_create(const RunDev& d, unsigned long long k, int m, bool* created) {
  const unsigned long long want_meta = (unsigned long long)(m + 1);
  unsigned long long h = run_hash(k, m) & d.mask;
  for (unsigned long long i = 0; i <= d.mask; i++, h = (h + 1) & d.mask) {
    const RunSlot cur = atomicCAS(&d.slot[h], RunSlot{0ull, 0ull}, RunSlot{k, want_meta});
    *created = cur.key == 0ull && cur.meta == 0ull;
    if (*created || (cur.key == k && cur.meta == want_meta)) return (long long)h;
  }
  return -1;
}

}  // namespace eppscore
