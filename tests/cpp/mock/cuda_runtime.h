// TEST INFRASTRUCTURE — a stand-in for <cuda_runtime.h> that lets the HOST runtime of fundsp_b200 (csrc/host/bank.cpp, graph.cpp,
// capi.cpp: class building, word layout, streams of launches, sequencer clock, live edits, growth in place ...) run in the CPU-only
// test suite: "device" memory is host memory, and the kernels are replaced by tests/cpp/mock/registry_mock.cpp, which runs the device
// node templates through the host emulation (FDSP_HOST_EMUL). Nothing here is ever part of the product library.
//
// Asynchronous work runs AS LATE AS CUDA ALLOWS, so that a missing dependency between device operations changes a result here as it
// can on a GPU. Every stream, the legacy stream 0 included, is a FIFO of pending operations (kernel launches, copies, memsets, waits),
// and an operation runs only when something forces it: a stream or event synchronise, a cudaStreamWaitEvent when the waiting stream is
// drained, a copy that must complete before it returns, or cudaFree / cudaFreeHost / cudaDeviceSynchronize (the whole device). Nothing
// is granted beyond the Runtime API's "API synchronization behavior" page:
//   - legacy-stream operations are ordered with blocking streams, not with cudaStreamNonBlocking ones;
//   - cudaStreamWaitEvent waits for the event's latest record at the time of the call (an event never recorded: no wait);
//   - cudaMemcpy host-to-device from pageable memory snapshots the source and queues the write on the legacy stream; from pinned memory,
//     and device-to-host, it drains the legacy stream and copies; device-to-device and cudaMemset queue on the legacy stream;
//   - the *Async forms queue on their stream. A host source is read when the copy runs, and a source that changed between the call and
//     the copy (pinned staging rewritten early, a pageable vector freed early) is reported as a hazard. A device-to-host destination is
//     poisoned (0xFF) at the call, so a host read before the synchronise sees NaN.
// A kernel failure or a hazard becomes a sticky error that every later API call returns, as CUDA reports asynchronous errors.
// FDSP_MOCK_SCHEDULE picks the order in which one synchronisation that forces several streams drains them: `late` (the default, creation
// order, legacy stream first) or `late-reverse` (reverse creation order). A run that is correct under these rules is correct when every
// call runs at once as well.
#pragma once
#include <atomic>
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <functional>
#include <map>
#include <mutex>
#include <vector>

typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2, cudaErrorInvalidDeviceFunction = 98, cudaErrorLaunchFailure = 719,
       cudaErrorMockHazard = 9001 };
typedef struct MockStream_* cudaStream_t;
typedef struct MockEvent_* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum { cudaStreamDefault = 0, cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaHostAllocMapped = 2 };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16 };

// A stream: its pending operations, how many were ever queued and how many have run (positions count operations from the stream's start).
// Destroyed streams stay in the list, flagged, so that their pending work still runs and events recorded on them stay valid.
struct MockStream_ {
  bool blocking = true, destroyed = false;
  std::deque<std::function<cudaError_t()>> q;
  uint64_t queued = 0, done = 0;
};
// An event: the stream and position of its latest record (none: never recorded).
struct MockEvent_ { MockStream_* s = nullptr; uint64_t at = 0; };

// device and pinned allocations, streams and events that are live (registry_mock.cpp exports the count: every resource a bank takes
// must be given back)
inline std::atomic<long>& mock_live() { static std::atomic<long> n{0}; return n; }

namespace mockdev {
struct Device {
  std::recursive_mutex mu;
  std::vector<MockStream_*> streams;      // creation order; [0] is the legacy stream
  std::map<uintptr_t, size_t> pinned;     // host ranges from cudaHostAlloc / cudaMallocHost
  cudaError_t sticky = cudaSuccess;
  bool reverse = false;
};
inline Device& dev() {
  static Device* d = [] {
    Device* x = new Device;   // (never destroyed: banks may be released by static destructors after this header's statics)
    x->streams.push_back(new MockStream_);
    const char* s = getenv("FDSP_MOCK_SCHEDULE");
    if (s && *s && strcmp(s, "late") != 0 && strcmp(s, "late-reverse") != 0) { fprintf(stderr, "mock CUDA: unknown FDSP_MOCK_SCHEDULE `%s` (late, late-reverse)\n", s); abort(); }
    x->reverse = s && strcmp(s, "late-reverse") == 0;
    return x;
  }();
  return *d;
}
typedef std::lock_guard<std::recursive_mutex> Lock;
inline MockStream_* legacy() { return dev().streams[0]; }
inline MockStream_* of(cudaStream_t s) { return s ? s : legacy(); }
inline cudaError_t status() { return dev().sticky; }
inline void fail(cudaError_t e) { if (dev().sticky == cudaSuccess) dev().sticky = e; }

// run the operations of s until `upto` of them have run. A wait runs the stream it waits for up to the recorded position, which was
// queued before the wait: the recursion only ever goes back in time.
inline void drain(MockStream_* s, uint64_t upto) {
  while (s->done < upto) {
    std::function<cudaError_t()> op = std::move(s->q.front());
    s->q.pop_front();
    const cudaError_t e = op();
    s->done++;
    if (e != cudaSuccess) fail(e);
  }
}
inline void drain(MockStream_* s) { drain(s, s->queued); }
inline void drain_all() {
  Device& d = dev();
  const size_t n = d.streams.size();
  for (size_t k = 0; k < n; k++) drain(d.streams[d.reverse ? n - 1 - k : k]);
}
inline void push_raw(MockStream_* s, std::function<cudaError_t()> op) { s->q.push_back(std::move(op)); s->queued++; }
inline std::function<cudaError_t()> wait_for(MockStream_* t, uint64_t at) { return [t, at] { drain(t, at); return cudaSuccess; }; }
// queue op on s behind what the legacy-stream rules order it after
inline void push(MockStream_* s, std::function<cudaError_t()> op) {
  Device& d = dev();
  if (s == legacy()) {
    for (MockStream_* b : d.streams) if (b != s && b->blocking && b->queued > b->done) push_raw(s, wait_for(b, b->queued));
  } else if (s->blocking && legacy()->queued > legacy()->done) push_raw(s, wait_for(legacy(), legacy()->queued));
  push_raw(s, std::move(op));
}
inline bool is_pinned(const void* p, size_t n) {
  const auto& m = dev().pinned;
  auto it = m.upper_bound((uintptr_t)p);
  if (it == m.begin()) return false;
  --it;
  return (uintptr_t)p + n <= it->first + it->second;
}
// rows of a 2D copy, `width` bytes each
inline void copy_rows(void* d, size_t dpitch, const void* s, size_t spitch, size_t width, size_t height) {
  for (size_t r = 0; r < height; r++) memmove((char*)d + r * dpitch, (const char*)s + r * spitch, width);
}
inline std::vector<char> gather(const void* s, size_t spitch, size_t width, size_t height) {
  std::vector<char> v(width * height);
  copy_rows(v.data(), width, s, spitch, width, height);
  return v;
}
// an asynchronous 2D copy on st (a 1D copy is one row)
inline cudaError_t copy_async(void* d, size_t dpitch, const void* s, size_t spitch, size_t width, size_t height, cudaMemcpyKind k, cudaStream_t st) {
  Lock lk(dev().mu);
  if (!width || !height) return status();
  if (k == cudaMemcpyHostToHost) { copy_rows(d, dpitch, s, spitch, width, height); return status(); }
  if (k == cudaMemcpyHostToDevice) {
    std::vector<char> snap = gather(s, spitch, width, height);
    push(of(st), [=] {
      if (gather(s, spitch, width, height) != snap) {
        fprintf(stderr, "mock CUDA: hazard: the host source of an asynchronous copy (%p, %zu x %zu bytes) changed before the copy ran\n", s, height, width);
        return (cudaError_t)cudaErrorMockHazard;
      }
      copy_rows(d, dpitch, s, spitch, width, height);
      return (cudaError_t)cudaSuccess;
    });
    return status();
  }
  if (k == cudaMemcpyDeviceToHost) for (size_t r = 0; r < height; r++) memset((char*)d + r * dpitch, 0xFF, width);
  push(of(st), [=] { copy_rows(d, dpitch, s, spitch, width, height); return (cudaError_t)cudaSuccess; });
  return status();
}
// a synchronous 2D copy (cudaMemcpy, cudaMemcpy2D)
inline cudaError_t copy_sync(void* d, size_t dpitch, const void* s, size_t spitch, size_t width, size_t height, cudaMemcpyKind k) {
  Lock lk(dev().mu);
  if (!width || !height) return status();
  const bool pinned_src = k == cudaMemcpyHostToDevice && height == 1 && is_pinned(s, width);
  if (k == cudaMemcpyHostToDevice && !pinned_src) {   // staged: returns before the write lands
    std::vector<char> snap = gather(s, spitch, width, height);
    push(legacy(), [=] { copy_rows(d, dpitch, snap.data(), width, width, height); return (cudaError_t)cudaSuccess; });
    return status();
  }
  if (k == cudaMemcpyDeviceToDevice) return copy_async(d, dpitch, s, spitch, width, height, k, nullptr);
  drain(legacy());   // pinned host-to-device, device-to-host, host-to-host: complete on return, behind the legacy stream
  copy_rows(d, dpitch, s, spitch, width, height);
  return status();
}
inline cudaError_t memset_async(void* d, size_t pitch, int v, size_t width, size_t height, cudaStream_t st) {
  Lock lk(dev().mu);
  if (width && height) push(of(st), [=] { for (size_t r = 0; r < height; r++) memset((char*)d + r * pitch, v, width); return (cudaError_t)cudaSuccess; });
  return status();
}
}  // namespace mockdev

// A kernel launch on the mock device: `run` is queued on st with its arguments captured by value; its failure becomes the sticky error.
inline cudaError_t mock_launch(cudaStream_t st, std::function<cudaError_t()> run) {
  mockdev::Lock lk(mockdev::dev().mu);
  mockdev::push(mockdev::of(st), std::move(run));
  return mockdev::status();
}

inline const char* cudaGetErrorString(cudaError_t e) {
  return e == cudaSuccess ? "no error" : e == cudaErrorMockHazard ? "mock CUDA hazard: a host source changed before its asynchronous copy ran"
       : e == cudaErrorLaunchFailure ? "mock CUDA: a kernel failed" : "mock CUDA error";
}
inline cudaError_t cudaGetLastError() { mockdev::Lock lk(mockdev::dev().mu); return mockdev::status(); }
inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { mockdev::Lock lk(mockdev::dev().mu); return mockdev::status(); }
inline cudaError_t cudaDeviceSynchronize() { mockdev::Lock lk(mockdev::dev().mu); mockdev::drain_all(); return mockdev::status(); }
inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr, int) { *v = 132; return cudaSuccess; }
inline cudaError_t cudaDeviceGetStreamPriorityRange(int* lo, int* hi) { *lo = 0; *hi = -1; return cudaSuccess; }
// fresh "device" memory is POISONED (0xFF bytes: NaN as f32, huge as an index), like real cudaMalloc memory it is not zero: a kernel
// or host path that reads a word nobody wrote shows up as a wrong result instead of passing by luck
template <class T> inline cudaError_t cudaMalloc(T** p, size_t bytes) { *p = (T*)malloc(bytes ? bytes : 1); if (*p) { memset(*p, 0xFF, bytes ? bytes : 1); mock_live()++; } return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
inline cudaError_t cudaFree(void* p) {
  mockdev::Lock lk(mockdev::dev().mu);
  mockdev::drain_all();   // (cudaFree synchronises the device)
  if (p) mock_live()--;
  free(p);
  return mockdev::status();
}
template <class T> inline cudaError_t cudaHostAlloc(T** p, size_t bytes, unsigned) {
  mockdev::Lock lk(mockdev::dev().mu);
  const cudaError_t e = cudaMalloc(p, bytes);
  if (e == cudaSuccess) mockdev::dev().pinned[(uintptr_t)*p] = bytes;
  return e;
}
template <class T> inline cudaError_t cudaMallocHost(T** p, size_t bytes) { return cudaHostAlloc(p, bytes, 0u); }
inline cudaError_t cudaFreeHost(void* p) {
  mockdev::Lock lk(mockdev::dev().mu);
  mockdev::drain_all();
  mockdev::dev().pinned.erase((uintptr_t)p);
  if (p) mock_live()--;
  free(p);
  return mockdev::status();
}
template <class T> inline cudaError_t cudaHostGetDevicePointer(T** d, void* h, unsigned) { *d = (T*)h; return cudaSuccess; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind k) { return mockdev::copy_sync(d, n, s, n, n, 1, k); }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind k, cudaStream_t st = nullptr) { return mockdev::copy_async(d, n, s, n, n, 1, k, st); }
inline cudaError_t cudaMemcpy2DAsync(void* d, size_t dpitch, const void* s, size_t spitch, size_t width, size_t height, cudaMemcpyKind k, cudaStream_t st = nullptr) {
  return mockdev::copy_async(d, dpitch, s, spitch, width, height, k, st);
}
inline cudaError_t cudaMemcpy2D(void* d, size_t dpitch, const void* s, size_t spitch, size_t width, size_t height, cudaMemcpyKind k) { return mockdev::copy_sync(d, dpitch, s, spitch, width, height, k); }
inline cudaError_t cudaMemset(void* d, int v, size_t n) { return mockdev::memset_async(d, n, v, n, 1, nullptr); }
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t st = nullptr) { return mockdev::memset_async(d, n, v, n, 1, st); }
inline cudaError_t cudaMemset2DAsync(void* d, size_t pitch, int v, size_t width, size_t height, cudaStream_t st = nullptr) { return mockdev::memset_async(d, pitch, v, width, height, st); }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned flags) {
  mockdev::Lock lk(mockdev::dev().mu);
  *s = new MockStream_;
  (*s)->blocking = !(flags & cudaStreamNonBlocking);
  mockdev::dev().streams.push_back(*s);
  mock_live()++;
  return mockdev::status();
}
inline cudaError_t cudaStreamCreate(cudaStream_t* s) { return cudaStreamCreateWithFlags(s, cudaStreamDefault); }
inline cudaError_t cudaStreamCreateWithPriority(cudaStream_t* s, unsigned f, int) { return cudaStreamCreateWithFlags(s, f); }
// (the stream's pending work still runs when something forces it, as CUDA finishes it after cudaStreamDestroy returns)
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { mockdev::Lock lk(mockdev::dev().mu); if (s && !s->destroyed) { s->destroyed = true; mock_live()--; } return mockdev::status(); }
inline cudaError_t cudaStreamSynchronize(cudaStream_t s) { mockdev::Lock lk(mockdev::dev().mu); mockdev::drain(mockdev::of(s)); return mockdev::status(); }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t s, cudaEvent_t e, unsigned) {
  mockdev::Lock lk(mockdev::dev().mu);
  if (e && e->s) mockdev::push(mockdev::of(s), mockdev::wait_for(e->s, e->at));
  return mockdev::status();
}
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new MockEvent_; mock_live()++; return cudaSuccess; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { return cudaEventCreate(e); }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { if (e) mock_live()--; delete e; return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t st = nullptr) {
  mockdev::Lock lk(mockdev::dev().mu);
  MockStream_* s = mockdev::of(st);
  mockdev::push(s, [] { return (cudaError_t)cudaSuccess; });   // (a marker: on the legacy stream it also takes the blocking streams' waits)
  e->s = s; e->at = s->queued;
  return mockdev::status();
}
inline cudaError_t cudaEventSynchronize(cudaEvent_t e) { mockdev::Lock lk(mockdev::dev().mu); if (e->s) mockdev::drain(e->s, e->at); return mockdev::status(); }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.0f; return cudaSuccess; }
