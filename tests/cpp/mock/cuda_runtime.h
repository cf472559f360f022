// TEST INFRASTRUCTURE — a stand-in for <cuda_runtime.h> that lets the HOST runtime of fundsp_b200 (csrc/host/bank.cpp, graph.cpp,
// capi.cpp: class building, word layout, streams of launches, sequencer clock, live edits, growth in place ...) run in the CPU-only
// test suite: "device" memory is host memory, every call is synchronous, streams and events are tokens. The kernels themselves are
// replaced by tests/cpp/mock/registry_mock.cpp, which runs the device node templates through the host emulation (FDSP_HOST_EMUL).
// Nothing here is ever part of the product library.
#pragma once
#include <atomic>
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <cstring>

typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2, cudaErrorInvalidDeviceFunction = 98, cudaErrorLaunchFailure = 719 };
typedef struct MockStream_* cudaStream_t;
typedef struct MockEvent_* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaHostAllocMapped = 2 };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16 };

// device and pinned allocations, streams and events that are live (registry_mock.cpp exports the count: every resource a bank takes
// must be given back)
inline std::atomic<long>& mock_live() { static std::atomic<long> n{0}; return n; }

inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "mock CUDA error"; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr, int) { *v = 132; return cudaSuccess; }
inline cudaError_t cudaDeviceGetStreamPriorityRange(int* lo, int* hi) { *lo = 0; *hi = -1; return cudaSuccess; }
// fresh "device" memory is POISONED (0xFF bytes: NaN as f32, huge as an index), like real cudaMalloc memory it is not zero: a kernel
// or host path that reads a word nobody wrote shows up as a wrong result instead of passing by luck
template <class T> inline cudaError_t cudaMalloc(T** p, size_t bytes) { *p = (T*)malloc(bytes ? bytes : 1); if (*p) { memset(*p, 0xFF, bytes ? bytes : 1); mock_live()++; } return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
inline cudaError_t cudaFree(void* p) { if (p) mock_live()--; free(p); return cudaSuccess; }
template <class T> inline cudaError_t cudaMallocHost(T** p, size_t bytes) { return cudaMalloc(p, bytes); }
template <class T> inline cudaError_t cudaHostAlloc(T** p, size_t bytes, unsigned) { return cudaMalloc(p, bytes); }
inline cudaError_t cudaFreeHost(void* p) { return cudaFree(p); }
template <class T> inline cudaError_t cudaHostGetDevicePointer(T** d, void* h, unsigned) { *d = (T*)h; return cudaSuccess; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { if (n) memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind k, cudaStream_t = nullptr) { return cudaMemcpy(d, s, n, k); }
inline cudaError_t cudaMemcpy2DAsync(void* d, size_t dpitch, const void* s, size_t spitch, size_t width, size_t height, cudaMemcpyKind, cudaStream_t = nullptr) {
  for (size_t r = 0; r < height; r++) memmove((char*)d + r * dpitch, (const char*)s + r * spitch, width);
  return cudaSuccess;
}
inline cudaError_t cudaMemcpy2D(void* d, size_t dpitch, const void* s, size_t spitch, size_t width, size_t height, cudaMemcpyKind k) { return cudaMemcpy2DAsync(d, dpitch, s, spitch, width, height, k); }
inline cudaError_t cudaMemset(void* d, int v, size_t n) { if (n) memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { return cudaMemset(d, v, n); }
inline cudaError_t cudaMemset2DAsync(void* d, size_t pitch, int v, size_t width, size_t height, cudaStream_t = nullptr) {
  for (size_t r = 0; r < height; r++) memset((char*)d + r * pitch, v, width);
  return cudaSuccess;
}
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = (cudaStream_t)malloc(1); mock_live()++; return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithPriority(cudaStream_t* s, unsigned f, int) { return cudaStreamCreateWithFlags(s, f); }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { if (s) mock_live()--; free(s); return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = (cudaEvent_t)malloc(1); mock_live()++; return cudaSuccess; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { return cudaEventCreate(e); }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { if (e) mock_live()--; free(e); return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.0f; return cudaSuccess; }
