// cuda_owners.hpp — owners of the engine's CUDA resources (capi.cu).  Each frees what it holds when it is destroyed, and
// moves but does not copy, so every buffer, stream and event has exactly one owner and nothing is freed by hand.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <utility>

namespace eppscore {

// A growable allocation: device memory (DevBuf) or pinned host memory (PinnedBuf).  reserve() keeps the contents only when
// the buffer is already large enough.
template <cudaError_t (*Alloc)(void**, size_t), cudaError_t (*Free)(void*)>
struct Buf {
  void* p = nullptr;
  size_t bytes = 0;
  Buf() = default;
  Buf(Buf&& o) noexcept : p(std::exchange(o.p, nullptr)), bytes(std::exchange(o.bytes, 0)) {}
  Buf& operator=(Buf&& o) noexcept {  // o takes the old allocation and frees it when it goes
    std::swap(p, o.p);
    std::swap(bytes, o.bytes);
    return *this;
  }
  ~Buf() {
    if (p) Free(p);
  }
  cudaError_t reserve(size_t n) {
    if (n <= bytes) return cudaSuccess;
    if (p) Free(p);
    p = nullptr;
    bytes = 0;
    size_t want = n + n / 8;  // a little slack so slowly growing batches do not reallocate every call
    cudaError_t e = Alloc(&p, want);
    if (e == cudaSuccess) bytes = want;
    return e;
  }
  template <typename T>
  T* as() const { return static_cast<T*>(p); }
};
using DevBuf = Buf<cudaMalloc, cudaFree>;
using PinnedBuf = Buf<cudaMallocHost, cudaFreeHost>;

// A stream or event handle; converts to the raw handle.
template <typename T, cudaError_t (*Destroy)(T)>
class Handle {
 public:
  Handle() = default;
  Handle(Handle&& o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
  Handle& operator=(Handle&& o) noexcept {
    std::swap(h_, o.h_);
    return *this;
  }
  ~Handle() {
    if (h_) Destroy(h_);
  }
  operator T() const { return h_; }
  T* put() {  // for the create call: destroys the current handle first
    *this = Handle();
    return &h_;
  }

 private:
  T h_ = nullptr;
};

// A stream finishes its work before it is destroyed, so nothing queued on it outlives the buffers freed after it.
inline cudaError_t sync_and_destroy(cudaStream_t s) {
  cudaStreamSynchronize(s);
  return cudaStreamDestroy(s);
}
using Stream = Handle<cudaStream_t, sync_and_destroy>;
using Event = Handle<cudaEvent_t, cudaEventDestroy>;
inline cudaError_t make(Stream& s) { return cudaStreamCreateWithFlags(s.put(), cudaStreamNonBlocking); }
inline cudaError_t make(Event& ev) { return cudaEventCreateWithFlags(ev.put(), cudaEventDisableTiming); }

}  // namespace eppscore
