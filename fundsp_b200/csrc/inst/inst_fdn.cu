// Warp-per-voice reverb_stereo kernel (csrc/dsp/fdn_kernel.cuh) and its launcher.
#include "../dsp/fdn_kernel.cuh"
#include "../host/registry.h"

#include <cstdlib>
namespace fdsp { namespace host {
template <int NST> static cudaError_t launch_fdn_t(FdnArgs a, int warps, cudaStream_t st) {
  const size_t smem = (size_t)warps * fdn_warp_floats(NST) * sizeof(float);
  // function attributes belong to each device's context: set once per device
  static bool attr[64] = {};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64 || !attr[dev]) {
    e = cudaFuncSetAttribute(fdn_kernel<NST>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) attr[dev] = true;
  }
  if (smem > 227 * 1024) return cudaErrorInvalidValue;
  const unsigned grid = (a.V + (unsigned)warps - 1) / (unsigned)warps;
  fdn_kernel<NST><<<grid, 32 * warps, smem, st>>>(a);
  return cudaGetLastError();
}
cudaError_t launch_fdn(const FdnArgs& a0, int warps, cudaStream_t st) {
  static const uint32_t flags = [] { const char* e = getenv("FDSP_FDN_FLAGS"); return e ? (uint32_t)atoi(e) : 0u; }();
  FdnArgs a = a0; a.flags = flags;
  if (flags & 2u) { const int cap = (int)((227 * 1024) / (fdn_warp_floats(3) * sizeof(float))); return launch_fdn_t<3>(a, warps < cap ? warps : cap, st); }
  return launch_fdn_t<2>(a, warps, st);
}
int fdn_max_warps() { const int m = (int)((227 * 1024) / (FDN_WARP_FLOATS * sizeof(float))); return m < 10 ? m : 10; }   // __launch_bounds__(320)
}}
