// The rules of the mock device's streams (tests/cpp/mock/cuda_runtime.h), one positive and one negative case each: an operation runs as
// late as CUDA allows, and no later than CUDA promises. tests/test_mock_streams_cpu.py builds and runs this under both schedules.
// Build: g++ -std=c++17 -I tests/cpp/mock mock_streams_test.cpp
// Prints one line per case, "<case>: ok" or "<case>: FAIL <what>", and the final word of `schedule` (which depends on FDSP_MOCK_SCHEDULE).
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

static int failures = 0;
static void report(const char* name, bool ok, const std::string& what = "") {
  printf("%s: %s%s\n", name, ok ? "ok" : "FAIL ", ok ? "" : what.c_str());
  if (!ok) failures++;
}
// a "kernel" on st that copies *src into *dst when it runs
static void k_copy(cudaStream_t st, const int* src, int* dst) { mock_launch(st, [=] { *dst = *src; return (cudaError_t)cudaSuccess; }); }
static void k_set(cudaStream_t st, int* dst, int v) { mock_launch(st, [=] { *dst = v; return (cudaError_t)cudaSuccess; }); }
static int* dev_int(int v) { int* p = nullptr; cudaMalloc(&p, sizeof(int)); *p = v; return p; }   // (device memory is host memory here)

int main() {
  cudaStream_t nb, nb2, bl;
  cudaStreamCreateWithFlags(&nb, cudaStreamNonBlocking);
  cudaStreamCreateWithFlags(&nb2, cudaStreamNonBlocking);
  cudaStreamCreate(&bl);
  cudaEvent_t e;
  cudaEventCreateWithFlags(&e, cudaEventDisableTiming);

  {  // a launch runs when its stream is synchronised, not before
    int* x = dev_int(1);
    k_set(nb, x, 2);
    const int before = *x;
    cudaStreamSynchronize(nb);
    report("launch_deferred", before == 1 && *x == 2, "before " + std::to_string(before) + " after " + std::to_string(*x));
    cudaFree(x);
  }
  {  // legacy cudaMemset, then a kernel on a non-blocking stream: no order (old bytes); with an event between them: the new bytes
    int* x = dev_int(7); int* y = dev_int(0);
    cudaMemset(x, 0, sizeof(int));
    k_copy(nb, x, y);
    cudaStreamSynchronize(nb);
    report("legacy_then_nonblocking_unordered", *y == 7, "read " + std::to_string(*y));
    *x = 7;
    cudaMemset(x, 0, sizeof(int));
    cudaEventRecord(e, 0);
    cudaStreamWaitEvent(nb, e, 0);
    k_copy(nb, x, y);
    cudaStreamSynchronize(nb);
    report("legacy_then_nonblocking_with_event", *y == 0, "read " + std::to_string(*y));
    cudaFree(x); cudaFree(y);
  }
  {  // legacy and a blocking stream are ordered both ways
    int* x = dev_int(7); int* y = dev_int(0);
    cudaMemset(x, 0, sizeof(int));
    k_copy(bl, x, y);
    cudaStreamSynchronize(bl);
    report("legacy_then_blocking_ordered", *y == 0, "read " + std::to_string(*y));
    k_set(bl, x, 5);
    int* z = dev_int(0);
    cudaMemcpy(z, x, sizeof(int), cudaMemcpyDeviceToDevice);   // legacy: behind the blocking stream's kernel
    cudaStreamSynchronize(0);
    report("blocking_then_legacy_ordered", *z == 5, "read " + std::to_string(*z));
    k_set(nb, x, 9);   // ... but not behind a non-blocking stream's
    cudaMemcpy(z, x, sizeof(int), cudaMemcpyDeviceToDevice);
    cudaStreamSynchronize(0);
    report("nonblocking_then_legacy_unordered", *z == 5, "read " + std::to_string(*z));
    cudaStreamSynchronize(nb);
    cudaFree(x); cudaFree(y); cudaFree(z);
  }
  {  // cudaStreamWaitEvent waits for the event's latest record at the time of the call
    int* x = dev_int(0); int* y = dev_int(-1);
    k_set(nb, x, 1);
    cudaEventRecord(e, nb);
    cudaStreamWaitEvent(nb2, e, 0);
    k_set(nb, x, 2);
    cudaEventRecord(e, nb);   // (a record after the wait does not move it)
    k_copy(nb2, x, y);
    cudaStreamSynchronize(nb2);
    report("wait_takes_record_at_call", *y == 1, "read " + std::to_string(*y));
    cudaStreamWaitEvent(nb2, e, 0);
    k_copy(nb2, x, y);
    cudaStreamSynchronize(nb2);
    report("wait_after_second_record", *y == 2, "read " + std::to_string(*y));
    cudaEvent_t fresh; cudaEventCreate(&fresh);   // never recorded: no wait
    k_set(nb, x, 3);
    cudaStreamWaitEvent(nb2, fresh, 0);
    k_copy(nb2, x, y);
    cudaStreamSynchronize(nb2);
    report("wait_on_unrecorded_event", *y == 2, "read " + std::to_string(*y));
    cudaEventDestroy(fresh);
    cudaStreamSynchronize(nb);
    cudaFree(x); cudaFree(y);
  }
  {  // cudaEventSynchronize runs the stream up to the record, not past it
    int* x = dev_int(0);
    k_set(nb, x, 1);
    cudaEventRecord(e, nb);
    k_set(nb, x, 2);
    cudaEventSynchronize(e);
    const int at = *x;
    cudaStreamSynchronize(nb);
    report("event_synchronize", at == 1 && *x == 2, "at the record " + std::to_string(at) + ", after " + std::to_string(*x));
    cudaFree(x);
  }
  {  // pageable cudaMemcpy host-to-device: the source is taken at the call, the write lands on the legacy stream
    std::vector<int> h(1, 4);
    int* x = dev_int(0); int* y = dev_int(-1);
    cudaMemcpy(x, h.data(), sizeof(int), cudaMemcpyHostToDevice);
    h[0] = 8;   // (allowed: the call returned once the source was staged)
    const int before = *x;
    k_copy(nb, x, y);
    cudaStreamSynchronize(nb);
    report("pageable_h2d_queued_on_legacy", before == 0 && *y == 0, "before " + std::to_string(before) + ", kernel read " + std::to_string(*y));
    cudaStreamSynchronize(0);
    report("pageable_h2d_snapshot", *x == 4, "landed " + std::to_string(*x));
    cudaFree(x); cudaFree(y);
  }
  {  // pinned cudaMemcpy host-to-device completes on return; device-to-host drains the legacy stream but not a non-blocking one
    int* hp = nullptr; cudaHostAlloc(&hp, sizeof(int), 0); *hp = 6;
    int* x = dev_int(0);
    cudaMemcpy(x, hp, sizeof(int), cudaMemcpyHostToDevice);
    report("pinned_h2d_complete_on_return", *x == 6, "landed " + std::to_string(*x));
    cudaMemset(x, 0, sizeof(int));
    int r = -1;
    cudaMemcpy(&r, x, sizeof(int), cudaMemcpyDeviceToHost);
    report("d2h_drains_legacy", r == 0, "read " + std::to_string(r));
    k_set(nb, x, 3);
    cudaMemcpy(&r, x, sizeof(int), cudaMemcpyDeviceToHost);
    report("d2h_leaves_nonblocking", r == 0, "read " + std::to_string(r));
    cudaStreamSynchronize(nb);
    cudaMemcpy(&r, x, sizeof(int), cudaMemcpyDeviceToHost);
    report("d2h_after_stream_sync", r == 3, "read " + std::to_string(r));
    cudaFreeHost(hp); cudaFree(x);
  }
  {  // device-to-device cudaMemcpy is queued on the legacy stream
    int* x = dev_int(5); int* y = dev_int(0); int* z = dev_int(-1);
    cudaMemcpy(y, x, sizeof(int), cudaMemcpyDeviceToDevice);
    const int before = *y;
    k_copy(nb, y, z);
    cudaStreamSynchronize(nb);
    report("d2d_queued_on_legacy", before == 0 && *z == 0, "before " + std::to_string(before) + ", kernel read " + std::to_string(*z));
    cudaStreamSynchronize(0);
    report("d2d_lands_at_legacy_sync", *y == 5, "landed " + std::to_string(*y));
    cudaFree(x); cudaFree(y); cudaFree(z);
  }
  {  // *Async host-to-device: the source is read when the copy runs; one that changed in between is a hazard
    int* hp = nullptr; cudaHostAlloc(&hp, sizeof(int), 0); *hp = 11;
    int* x = dev_int(0);
    cudaMemcpyAsync(x, hp, sizeof(int), cudaMemcpyHostToDevice, nb);
    const int before = *x;
    const cudaError_t ok = cudaStreamSynchronize(nb);
    report("async_h2d_unchanged_source", before == 0 && *x == 11 && ok == cudaSuccess, "before " + std::to_string(before) + ", landed " + std::to_string(*x));
    cudaMemcpyAsync(x, hp, sizeof(int), cudaMemcpyHostToDevice, nb);
    *hp = 12;   // staging rewritten before the copy ran
    const cudaError_t bad = cudaStreamSynchronize(nb);
    const cudaError_t next = cudaGetLastError();
    report("async_h2d_source_rewritten_is_hazard", bad == cudaErrorMockHazard && next == cudaErrorMockHazard, "status " + std::to_string(bad));
    mockdev::dev().sticky = cudaSuccess;   // (this driver goes on; a product run stops at the first error)
    cudaFreeHost(hp); cudaFree(x);
  }
  {  // *Async device-to-host: the destination reads NaN until the stream is synchronised
    float* x = nullptr; cudaMalloc(&x, sizeof(float)); *x = 2.5f;
    float h = 0.0f;
    cudaMemcpyAsync(&h, x, sizeof(float), cudaMemcpyDeviceToHost, nb);
    const bool poisoned = std::isnan(h);
    cudaStreamSynchronize(nb);
    report("async_d2h_poisoned_until_sync", poisoned && h == 2.5f, "after the sync " + std::to_string(h));
    cudaFree(x);
  }
  {  // *Async memsets and 2D copies queue on their stream
    int* x = dev_int(3);
    cudaMemsetAsync(x, 0, sizeof(int), nb);
    const int before = *x;
    cudaStreamSynchronize(nb);
    report("memset_async_on_stream", before == 3 && *x == 0, "before " + std::to_string(before) + ", after " + std::to_string(*x));
    int* m = nullptr; cudaMalloc(&m, 4 * sizeof(int));
    const int src[2] = {21, 22};
    cudaMemcpy2DAsync(m, 2 * sizeof(int), src, sizeof(int), sizeof(int), 2, cudaMemcpyHostToDevice, nb);
    const bool untouched = m[0] == -1 && m[2] == -1;   // (fresh memory is 0xFF)
    cudaStreamSynchronize(nb);
    report("copy2d_async_on_stream", untouched && m[0] == 21 && m[2] == 22 && m[1] == -1, "rows " + std::to_string(m[0]) + " " + std::to_string(m[2]));
    cudaFree(m); cudaFree(x);
  }
  {  // cudaFree synchronises the whole device; cudaMalloc does not
    int* x = dev_int(0);
    k_set(nb, x, 1);
    int* y = nullptr; cudaMalloc(&y, 4);
    const int after_malloc = *x;
    cudaFree(y);
    report("free_drains_every_stream", after_malloc == 0 && *x == 1, "after cudaMalloc " + std::to_string(after_malloc) + ", after cudaFree " + std::to_string(*x));
    cudaFree(x);
  }
  {  // a failed launch is reported by the next call, not by the launch
    int* x = dev_int(0);
    const cudaError_t at_launch = mock_launch(nb, [] { return (cudaError_t)cudaErrorLaunchFailure; });
    const cudaError_t at_sync = cudaStreamSynchronize(nb);
    const cudaError_t later = cudaMemsetAsync(x, 0, 4, nb);
    report("launch_failure_is_sticky", at_launch == cudaSuccess && at_sync == cudaErrorLaunchFailure && later == cudaErrorLaunchFailure, "launch " + std::to_string(at_launch) + ", sync " + std::to_string(at_sync));
    mockdev::dev().sticky = cudaSuccess;
    cudaStreamSynchronize(nb);
    cudaFree(x);
  }
  {  // a destroyed stream's pending work still runs when it is forced
    cudaStream_t t; cudaStreamCreateWithFlags(&t, cudaStreamNonBlocking);
    int* x = dev_int(0);
    k_set(t, x, 4);
    cudaEventRecord(e, t);
    cudaStreamDestroy(t);
    const int before = *x;
    cudaEventSynchronize(e);
    report("destroyed_stream_work_runs", before == 0 && *x == 4, "before " + std::to_string(before) + ", after " + std::to_string(*x));
    cudaFree(x);
  }
  {  // the schedule: two independent streams forced by one device synchronisation drain in creation order (late) or reversed (late-reverse)
    int* x = dev_int(0);
    k_set(nb2, x, 2);
    k_set(nb, x, 1);
    cudaDeviceSynchronize();
    printf("schedule: %s\n", *x == 2 ? "creation" : "reverse");   // the last writer wins
    cudaFree(x);
  }
  cudaEventDestroy(e);
  cudaStreamDestroy(nb); cudaStreamDestroy(nb2); cudaStreamDestroy(bl);
  printf("live: %ld\n", (long)mock_live());
  return failures ? 1 : 0;
}
