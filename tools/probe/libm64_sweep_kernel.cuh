// Probe kernel (test infrastructure, not product): the PRODUCT's f64 math (csrc/dsp/libm64.cuh) over the arguments of the f64 math sweep
// (tests/golden/libm64_sweep_args.h). libm64_sweep_probe.cu compiles this file twice: with nvcc, and at run time through NVRTC with the
// JIT's options, which is how the prelude64 nodes are built. Headers are included by bare name: the nvcc build passes their directories
// with -I, the NVRTC build passes their text.
#include "libm64.cuh"
#include "libm64_sweep_args.h"

__device__ __forceinline__ double sweep64_eval(int fn, double x) {
  using namespace fdsp;
  switch (fn) {
    case sweep64::SIN: return m64::sin(x);
    case sweep64::COS: return m64::cos(x);
    case sweep64::TAN: return m64::tan(x);
    default: return m64::exp(x);
  }
}

// blockIdx.y = chunk - chunk0. hash[blockIdx.y] += the chunk's sum; dump, when given, receives one chunk's argument and result bits
// (gridDim.y == 1): x at [j], f at [2^24 + j].
extern "C" __global__ void libm64_sweep(int fn, unsigned chunk0, unsigned long long* hash, unsigned long long* dump) {
  const unsigned c = chunk0 + blockIdx.y;
  const unsigned long long i0 = (unsigned long long)c << sweep64::CHUNK_LOG2;
  const unsigned len = sweep64::chunk_len((int)c);
  unsigned long long h = 0;
  for (unsigned j = blockIdx.x * blockDim.x + threadIdx.x; j < len; j += gridDim.x * blockDim.x) {
    const unsigned long long i = i0 + j;
    const unsigned long long xb = sweep64::arg_bits(fn, i);
    const unsigned long long fb = (unsigned long long)__double_as_longlong(sweep64_eval(fn, __longlong_as_double((long long)xb)));
    h += sweep64::term(i, fb);
    if (dump) { dump[j] = xb; dump[(1u << sweep64::CHUNK_LOG2) + j] = fb; }
  }
  for (int o = 16; o; o >>= 1) h += __shfl_xor_sync(0xffffffffu, h, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(&hash[blockIdx.y], h);
}
