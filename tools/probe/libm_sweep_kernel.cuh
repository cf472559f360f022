// Probe kernel (test infrastructure, not product): the PRODUCT's scalar f32 math (csrc/dsp/libm.cuh, math.cuh) over the arguments of the
// scalar-math sweep (tests/golden/libm_sweep_args.h). libm_sweep_probe.cu compiles this file twice: with nvcc, and at run time through
// NVRTC with the closure JIT's options, which is how closure nodes are built. Headers are included by bare name: the nvcc build passes
// their directories with -I, the NVRTC build passes their text.
#include "libm.cuh"
#include "libm_sweep_args.h"

__device__ __forceinline__ float sweep_eval(int fn, float x, float y) {
  using namespace fdsp;
  switch (fn) {
    case sweep::SINF: return m::sinf_(x);
    case sweep::COSF: return m::cosf_(x);
    case sweep::TANF: return m::tanf_(x);
    case sweep::TANHF: return m::tanhf_(x);
    case sweep::EXPM1F: return m::expm1f_(x);
    case sweep::EXPF: return m::expf_(x);
    case sweep::ATANF: return m::atanf_(x);
    case sweep::WIDE_SINF: return wide_sinf(x);
    case sweep::WIDE_ATANF: return wide_atanf(x);
    default: return m::powf_(x, y);
  }
}
// CUDA's double-precision function at the (exact) f64 image of the arguments; NaN where the ulp error is not measured
// (wide_sinf outside |v| <= 2pi, the only domain Sine uses)
__device__ __forceinline__ double sweep_ref(int fn, float x, float y) {
  const double d = (double)x;
  switch (fn) {
    case sweep::SINF: return sin(d);
    case sweep::COSF: return cos(d);
    case sweep::TANF: return tan(d);
    case sweep::TANHF: return tanh(d);
    case sweep::EXPM1F: return expm1(d);
    case sweep::EXPF: return exp(d);
    case sweep::ATANF: return atan(d);
    case sweep::WIDE_SINF: return fabs(d) <= 6.2831854820251465 ? sin(d) : __longlong_as_double(0x7ff8000000000000ll);
    case sweep::WIDE_ATANF: return atan(d);
    default: return pow(d, (double)y);
  }
}
// |f - ref| in units of the f32 ulp at ref, for finite f and finite ref within the f32 range; powf only on normal results
__device__ __forceinline__ float sweep_ulp(int fn, float f, double r) {
  const double ar = fabs(r);
  if (!isfinite(f) || !(ar < 0x1p128)) return 0.0f;
  if (fn >= sweep::POW_X && ar < 0x1p-126) return 0.0f;
  int e;
  frexp(r, &e);                                     // |r| in [2^(e-1), 2^e)
  const int ue = e - 24 < -149 ? -149 : e - 24;    // ulp = 2^(ilogb(r) - 23), 2^-149 below the normal range
  return (float)(fabs((double)f - r) * __longlong_as_double((long long)(1023 - ue) << 52));
}

// blockIdx.y = chunk - chunk0. hash[blockIdx.y] += the chunk's sum; *ulp_bits = max(bits of the ulp error) (non-negative floats order as
// their bits); dump, when given, receives one chunk's argument and result bits (gridDim.y == 1): x at [j], y at [2^24 + j], f at [2^25 + j].
extern "C" __global__ void libm_sweep(int fn, unsigned chunk0, unsigned long long* hash, unsigned* ulp_bits, unsigned* dump) {
  const unsigned long long i0 = (unsigned long long)(chunk0 + blockIdx.y) << sweep::CHUNK_LOG2;
  unsigned long long h = 0;
  float worst = 0.0f;
  for (unsigned j = blockIdx.x * blockDim.x + threadIdx.x; j < (1u << sweep::CHUNK_LOG2); j += gridDim.x * blockDim.x) {
    const unsigned long long i = i0 + j;
    uint32_t xb, yb;
    sweep::arg_bits(fn, i, xb, yb);
    const float x = __uint_as_float(xb), y = __uint_as_float(yb);
    const float f = sweep_eval(fn, x, y);
    h += sweep::term(i, __float_as_uint(f));
    if (dump) { dump[j] = xb; dump[(1u << sweep::CHUNK_LOG2) + j] = yb; dump[(2u << sweep::CHUNK_LOG2) + j] = __float_as_uint(f); }
    else worst = fmaxf(worst, sweep_ulp(fn, f, sweep_ref(fn, x, y)));
  }
  for (int o = 16; o; o >>= 1) { h += __shfl_xor_sync(0xffffffffu, h, o); worst = fmaxf(worst, __shfl_xor_sync(0xffffffffu, worst, o)); }
  if ((threadIdx.x & 31) == 0) { atomicAdd(&hash[blockIdx.y], h); atomicMax(ulp_bits, __float_as_uint(worst)); }
}
