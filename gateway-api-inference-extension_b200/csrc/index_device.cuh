// index_device.cuh — DevX: the execution policy the index's CTA programs (prefix_table.cuh) run on as the CUDA threads of one
// CTA of kCommitThreads threads.  Shared by the index kernels (prefix_index.cu) and the in-order walk that commits as it
// schedules (inorder_kernel.cu), so both run the same IndexProgram with the same memory policy.
#pragma once
#include "prefix_table.cuh"

namespace eppscore {

struct DevX {
  template <class F>
  __device__ __forceinline__ void par(F f) {
    __syncthreads();  // everything the previous section wrote is visible, every uniform read before this point is done
    f((int)threadIdx.x);
    __syncthreads();
  }
  // in-place exclusive scan of arr[0..kCommitThreads); returns the total (uniform)
  __device__ __forceinline__ uint32_t scan(uint32_t* arr, uint32_t* /*unused*/) {
    __shared__ uint32_t wt[kCommitThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    __syncthreads();
    const uint32_t v = arr[tid];
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) wt[w] = inc;
    __syncthreads();
    uint32_t base = 0, total = 0;
#pragma unroll
    for (int i = 0; i < kCommitThreads / 32; i++) {
      const uint32_t t = wt[i];
      if (i < w) base += t;
      total += t;
    }
    arr[tid] = base + inc - v;
    __syncthreads();
    return total;
  }
  // Index structures are read and written at GPU scope (L2), never through a stale L1 line, and every access is a
  // compiler barrier: the intrinsics (__ldcg) are plain asm statements the compiler may hoist out of a spin loop or CSE
  // across a lock acquisition — a stale `key` of a slot that another CTA was still creating made a second slot for the
  // same hash (r2 first GPU run: one member of a 200-endpoint set missing).
  __device__ __forceinline__ uint32_t ld32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
  }
  __device__ __forceinline__ uint64_t ld64(const uint64_t* p) {
    uint64_t v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
  }
  __device__ __forceinline__ uint32_t ld16(const uint16_t* p) {
    uint16_t v;
    asm volatile("ld.relaxed.gpu.global.u16 %0, [%1];" : "=h"(v) : "l"(p) : "memory");
    return v;
  }
  __device__ __forceinline__ void st32(uint32_t* p, uint32_t v) { asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
  __device__ __forceinline__ void st64(uint64_t* p, uint64_t v) { asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
  __device__ __forceinline__ void st16(uint16_t* p, uint16_t v) { asm volatile("st.relaxed.gpu.global.u16 [%0], %1;" ::"l"(p), "h"(v) : "memory"); }
  __device__ __forceinline__ uint32_t ld_acquire32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
  }
  __device__ __forceinline__ void st_release32(uint32_t* p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
  }
  __device__ __forceinline__ uint32_t cas32(uint32_t* p, uint32_t cmp, uint32_t val) { return atomicCAS(p, cmp, val); }
  __device__ __forceinline__ uint32_t cas_acquire32(uint32_t* p, uint32_t cmp, uint32_t val) {
    uint32_t old;
    asm volatile("atom.acquire.gpu.global.cas.b32 %0, [%1], %2, %3;" : "=r"(old) : "l"(p), "r"(cmp), "r"(val) : "memory");
    return old;
  }
  __device__ __forceinline__ uint64_t cas64(uint64_t* p, uint64_t cmp, uint64_t val) {
    return atomicCAS(reinterpret_cast<unsigned long long*>(p), (unsigned long long)cmp, (unsigned long long)val);
  }
  __device__ __forceinline__ void add64(unsigned long long* p, unsigned long long v) { atomicAdd(p, v); }
  __device__ __forceinline__ void fence() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
  __device__ __forceinline__ void lock(uint32_t* p) {
    while (cas_acquire32(p, 0u, 1u) != 0u) {
    }
  }
  __device__ __forceinline__ void unlock(uint32_t* p) { st_release32(p, 0u); }
  __device__ __forceinline__ uint64_t smem_cas64(uint64_t* p, uint64_t cmp, uint64_t val) {
    return atomicCAS(reinterpret_cast<unsigned long long*>(p), (unsigned long long)cmp, (unsigned long long)val);
  }
  __device__ __forceinline__ void smem_max32(uint32_t* p, uint32_t v) { atomicMax(p, v); }
  __device__ __forceinline__ void smem_add32(uint32_t* p, uint32_t v) { atomicAdd(p, v); }
};

}  // namespace eppscore
