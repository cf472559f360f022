// Plain-data kernel arguments shared by host (csrc/host) and device (csrc/dsp) code.
#pragma once
#ifndef __CUDACC_RTC__
#include <cstddef>
#include <cstdint>
#endif

namespace fdsp {

// Wavetable set for one waveform (reference src/wavetable.rs:82-123): up to 48 tables, ascending pitch.
struct WaveTableDev {
  int n;
  float pitch[48];
  int off[48];
  int len[48];
  int total;          // floats in `data`
  const float* data;
};

// Depth (samples) of the CTA mix tile [OUT][TS][NT+1]: the tile is reduced and recycled every TS samples, so wide
// voices keep a ~33 KB tile and the 164 KB wavetable set still fits beside it in shared memory.
#ifdef __CUDACC__
#define FDSP_HDC __host__ __device__
#else
#define FDSP_HDC
#endif
FDSP_HDC constexpr int mix_tile_samples(int outs) { return outs <= 1 ? 64 : (outs == 2 ? 32 : (outs <= 4 ? 16 : 8)); }
FDSP_HDC constexpr size_t mix_tile_floats(int outs, int nt) { return (size_t)outs * (size_t)mix_tile_samples(outs) * (size_t)(nt + 1); }

// CTA shape of a class of V voices with NT threads per CTA on a device of `sms` SMs: enough CTAs to cover the voices, rounded up to
// whole waves of the SMs once every CTA can still have a full warp, and the voices spread evenly over them (a bank is bound by per-SM
// pipes and per-warp latency, so idle SMs are the first thing to use up).
inline uint32_t bank_grid(uint32_t V, uint32_t nt, uint32_t sms, uint32_t* vpc) {
  uint32_t grid = (V + nt - 1) / nt;
  if (V >= sms * 32u) grid = (grid + sms - 1u) / sms * sms;
  if (grid == 0) grid = 1;
  *vpc = (V + grid - 1) / grid;
  return (V + *vpc - 1) / *vpc;
}

struct BankArgs {
  const uint32_t* params;   // [NP][V]
  uint32_t* state;          // [NS][V]
  const uint32_t* uniform;  // [NU]
  float* dline;             // [sum(len)][V]
  const WaveTableDev* wt;   // [6]
  const float* in;          // shared bank input [IN][in_stride] or null
  float* out;               // per-voice output rows or null
  float* partial;           // [grid][OUT][n] per-CTA mix partials or null
  uint32_t V, n;
  uint32_t vpc;             // voices per CTA (<= threads per CTA): CTA b runs voices [b*vpc, min(V, (b+1)*vpc)); 0 means NT
  uint32_t in_stride, in_offset;
  uint32_t out_stride, out_offset;  // row stride / first sample (multiples of 4 for the vector path)
  const uint32_t* row_map;          // class-local voice -> first output row (voice-major rows) inside `out`
  float sr, sd64, sd32;
  // fused mix-down for short launches (process()-sized): when `ticket` is set, the last CTA to finish folds the per-CTA
  // partials in CTA order into mix[c*mix_stride + mix_offset + t] itself (no mix_reduce_kernel launch)
  uint32_t* ticket;
  float* mix;
  uint32_t mix_stride, mix_offset;
  int mix_accumulate;
  // reset image of the class's state words [NS][V] and delay-line floats per voice: what Event<X> of a looping sequencer needs to reset its unit
  // on the device (null / 0 when the class has no such voices)
  const uint32_t* state0;
  uint32_t dl_floats;
};

}  // namespace fdsp
