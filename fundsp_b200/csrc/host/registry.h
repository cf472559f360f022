// Kernel programs: a fused voice program (device type expression, see graph.h `sig`) and how to launch it.
// Two sources: the ahead-of-time instance tables (csrc/inst/*.cu) and the NVRTC path (jit.cpp).
#pragma once
#include <cuda_runtime.h>

#include <memory>
#include <string>

#include "../dsp/bank_args.h"

namespace fdsp { struct FdnArgs; struct RtArgs; }

namespace fdsp {
namespace host {

// Preferred shared-memory carve-out (percent of the SM's unified L1 / shared memory) that the voice-kernel launchers apply to the kernel they
// launch; -1 = leave the driver's choice. The concurrent classes of a multi-class bank set it to the maximum, so that a class whose CTAs
// stage the wavetables (~195 KB) and the light classes beside it agree on ONE configuration and can share an SM (kernels that ask for
// different carve-outs are not co-resident). Set and read by the thread that drives the bank.
inline int& launch_carveout() { static thread_local int v = -1; return v; }

struct KernelEntry {  // AOT table row
  const char* sig;
  int IN, OUT, NP, NS, NU;
  // table_bytes > 0: stage that many bytes of wavetable data in shared memory (long renders of wavetable graphs)
  cudaError_t (*launch)(const BankArgs& a, int mode, size_t table_bytes, cudaStream_t stream);
  int (*threads)();
  int (*wave_kind)();  // first wavetable kind the program reads, -1 if none
  int stages;          // stages of the stage-pipelined form (dsp/bank_kernel_st.cuh); 1 = none built
  cudaError_t (*launch_st)(const BankArgs& a, int mode, size_t table_bytes, cudaStream_t stream);
  cudaError_t (*launch_rt)(const BankArgs& a, const RtArgs& rt, size_t table_bytes, cudaStream_t stream);   // resident process() kernel
};

struct Program {
  std::string sig;
  int IN = 0, OUT = 0, NP = 0, NS = 0, NU = 0, threads = 128, wave_kind = -1;
  bool jit = false;
  int stages = 1;      // >= 2: launch_staged runs the program as a pipeline of that many warp stages per voice (dsp/bank_kernel_st.cuh)
  virtual ~Program() {}
  // mode: FDSP_OUT_VOICES | FDSP_OUT_MIX bits
  virtual cudaError_t launch(const BankArgs& a, int mode, size_t table_bytes, cudaStream_t stream) const = 0;
  // a.vpc <= 32 selects the 32-voice CTA shape, else 128 voices per CTA; same word layout as `launch` (the two can alternate)
  virtual cudaError_t launch_staged(const BankArgs&, int, size_t, cudaStream_t) const { return cudaErrorInvalidValue; }
  // the resident process() kernel (dsp/bank_kernel_rt.cuh): serves 64-sample blocks on a doorbell until told to leave; mix mode only
  virtual cudaError_t launch_rt(const BankArgs&, const RtArgs&, size_t, cudaStream_t) const { return cudaErrorInvalidValue; }
  bool has_rt = false;
};

// Returns the program for `sig` (AOT if listed, else NVRTC-compiled and cached); nullptr + `err` on failure.
std::shared_ptr<const Program> get_program(const std::string& sig, int device, std::string& err);
const KernelEntry* find_kernel(const std::string& sig);
int registry_size();
const KernelEntry* registry_at(int i);
const char* registry_key(int i);
cudaError_t launch_mix_reduce(const float* partial, uint32_t nparts, uint32_t outs, uint32_t n, float* mix, uint32_t mix_stride,
                              uint32_t mix_offset, int accumulate, cudaStream_t stream);
// `scratch` (tree_mix_scratch_floats(V, outs, n) floats, or null): lets a big balanced tree reduce its 256-voice subtrees in parallel first
cudaError_t launch_tree_mix(const float* rows, uint32_t V, uint32_t outs, uint32_t row_stride, uint32_t row_offset, uint32_t n, float* mix,
                            uint32_t mix_stride, uint32_t mix_offset, int pairwise, cudaStream_t stream, float* scratch = nullptr);
size_t tree_mix_scratch_floats(uint32_t V, uint32_t outs, uint32_t n);
// warp-per-voice reverb_stereo kernel (inst/inst_fdn.cu)
cudaError_t launch_fdn(const FdnArgs& a, int warps, cudaStream_t stream);
int fdn_max_warps();
// tensor-core convolve path (inst/inst_conv.cu, dsp/conv_tc_kernel.cuh): Y = X * Toeplitz(h) as 3xTF32 wgmma GEMM tiles
struct ConvTcMaps { alignas(64) unsigned char m[4][128]; };   // four CUtensorMap objects: X, Xlo, T, Tlo
cudaError_t conv_tc_make_maps(float* x, float* xl, uint32_t V, uint32_t row_stride, float* th, float* tl, uint32_t J, ConvTcMaps* out);
cudaError_t launch_conv_tc(const ConvTcMaps& maps, float* y, uint32_t y_stride, uint32_t y_offset, const uint32_t* row_map, uint32_t V, uint32_t n, uint32_t K, uint32_t H,
                           cudaStream_t stream);
cudaError_t launch_conv_split(float* x, float* xl, uint32_t V, uint32_t row_stride, uint32_t col0, uint32_t n, cudaStream_t stream);
cudaError_t launch_conv_history(float* x, float* xl, uint32_t V, uint32_t row_stride, uint32_t H, uint32_t n, cudaStream_t stream);
cudaError_t launch_conv_toeplitz(const float* h, uint32_t K, float* th, float* tl, uint32_t J, cudaStream_t stream);
uint32_t conv_tc_toeplitz_cols(uint32_t K);
// NVRTC path (jit.cpp)
std::shared_ptr<const Program> jit_program(const std::string& sig, int device, std::string& err);
int jit_compiled_count();
void jit_cache_stats(int* hits, int* nvrtc_runs);                       // units served from the on-disk cache / compiled by NVRTC in this process
std::string jit_precompile(const std::string& sig, int mode, int tb, int staged_width = 0);   // fill the on-disk cache without a GPU (mode 0 = layout unit; staged_width 32 / 128 = that stage-pipelined kernel)

}  // namespace host
}  // namespace fdsp
