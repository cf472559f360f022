// Move-only owners of the CUDA resources the bank runtime holds. Each releases its handle when it is destroyed or replaced, so a
// buffer can neither leak nor be freed twice, and a failed allocation leaves an empty owner rather than a pointer to freed memory.
#pragma once
#include <cuda_runtime.h>

#include <string>
#include <utility>

namespace fdsp {
namespace host {

// Error convention of the runtime (bank.h): "" = ok, otherwise the message.
inline std::string cuerr(const char* what, cudaError_t e) { return std::string(what) + ": " + cudaGetErrorString(e); }
#define CU(call)                                                  \
  do {                                                            \
    cudaError_t e_ = (call);                                      \
    if (e_ != cudaSuccess) return ::fdsp::host::cuerr(#call, e_); \
  } while (0)

// An array of T with its element count, in device memory or in page-locked host memory (Mapped: dev() is the device's pointer to it).
enum class Mem { Device, Pinned, Mapped };
template <class T, Mem M = Mem::Device> class Array {
  T *p_ = nullptr, *d_ = nullptr;
  size_t n_ = 0;
 public:
  Array() = default;
  Array(Array&& o) noexcept : p_(std::exchange(o.p_, nullptr)), d_(std::exchange(o.d_, nullptr)), n_(std::exchange(o.n_, 0)) {}
  Array& operator=(Array&& o) noexcept { if (this != &o) { reset(); std::swap(p_, o.p_); std::swap(d_, o.d_); std::swap(n_, o.n_); } return *this; }
  ~Array() { reset(); }
  operator T*() const { return p_; }
  T* get() const { return p_; }
  T* operator->() const { return p_; }
  T* dev() const { return d_; }
  size_t size() const { return n_; }
  void reset() {
    if (p_) M == Mem::Device ? cudaFree(p_) : cudaFreeHost(p_);
    p_ = d_ = nullptr; n_ = 0;
  }
  // Reallocates only when n exceeds the count, freeing the old array first; the contents are not kept.
  std::string grow(size_t n) {
    if (n <= n_) return "";
    reset();
    T* p = nullptr;
    if (M == Mem::Device) CU(cudaMalloc((void**)&p, n * sizeof(T)));
    else CU(cudaHostAlloc((void**)&p, n * sizeof(T), M == Mem::Mapped ? (unsigned)cudaHostAllocMapped : 0u));
    p_ = p;
    if (M == Mem::Mapped) CU(cudaHostGetDevicePointer((void**)&d_, p_, 0));   // (on failure the count stays 0: the next grow retries)
    n_ = n;
    return "";
  }
};
template <class T> using PinnedArray = Array<T, Mem::Pinned>;
template <class T> using MappedArray = Array<T, Mem::Mapped>;

// A stream or an event. put() releases the one held and gives the address the CUDA call that creates the next one fills in.
template <class H, cudaError_t (*Destroy)(H)> class Handle {
  H h_ = nullptr;
 public:
  Handle() = default;
  Handle(Handle&& o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
  Handle& operator=(Handle&& o) noexcept { if (this != &o) { reset(); std::swap(h_, o.h_); } return *this; }
  ~Handle() { reset(); }
  operator H() const { return h_; }
  void reset() { if (h_) Destroy(h_); h_ = nullptr; }
  H* put() { reset(); return &h_; }
};
using Stream = Handle<cudaStream_t, cudaStreamDestroy>;
using Event = Handle<cudaEvent_t, cudaEventDestroy>;

}  // namespace host
}  // namespace fdsp
