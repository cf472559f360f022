// Probe (measurement infrastructure, not product): what would a second warp per scheduler buy the headline saw + SVF voice?
// Instantiates bank_kernel<Pipe<SawHz, FixedSvf>, ...> from dsp/bank_kernel.cuh on synthetic inputs of the headline's shape (the saw table
// set's pitches, lengths and device layout, the bank's frequency / phase / filter distributions) and times 48 000 samples, mix only:
//   (a) 128 threads, 16 384 voices at 125 per CTA: one warp per scheduler, the headline bank's launch
//   (b) 256 threads, 33 000 voices at 250 per CTA: two warps per scheduler, the same program
// (b)/(a) bounds what any form that gives the headline a second warp per scheduler can gain while each thread keeps today's work, e.g.
// two lanes per voice that split each 8-sample group's table reads (DESIGN §5). Prints samples/s of both and (b)/(a), with the card's name,
// power limit and the SM clock sampled while timing.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -fmad=false -o tools/probe/_build/lane_split_probe tools/probe/lane_split_probe.cu -ldl
#include "../../fundsp_b200/csrc/dsp/bank_kernel.cuh"
#include <dlfcn.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
using namespace fdsp;

typedef Pipe<Pipe<Constant<1>, WaveSynth<0, 1>>, FixedSvf> Headline;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); exit(1); } } while (0)

static double u(uint64_t i, uint64_t k) {   // the workloads' seeded uniform (fundsp_b200/workloads.py rnd)
  const uint64_t M = ~0ull;
  uint64_t x = ((4 * i + k) ^ 0x5555555555555555ull) & M;
  x *= 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  x ^= x >> 31;
  return (double)(x >> 11) * (1.0 / 9007199254740992.0);
}
static double xerp(double a, double b, double t) { return exp(log(a) * (1 - t) + log(b) * t); }

// NVML, opened at run time (read-only queries: power limit and the current SM clock)
struct Nvml {
  void* lib = nullptr; void* dev = nullptr;
  int (*clock)(void*, int, unsigned*) = nullptr;
  unsigned power_mw = 0;
  Nvml() {
    lib = dlopen("libnvidia-ml.so.1", RTLD_NOW);
    if (!lib) return;
    auto init = (int (*)())dlsym(lib, "nvmlInit_v2");
    auto handle = (int (*)(unsigned, void**))dlsym(lib, "nvmlDeviceGetHandleByIndex_v2");
    auto power = (int (*)(void*, unsigned*))dlsym(lib, "nvmlDeviceGetEnforcedPowerLimit");
    clock = (int (*)(void*, int, unsigned*))dlsym(lib, "nvmlDeviceGetClockInfo");
    int d = 0; cudaGetDevice(&d);
    if (!init || !handle || init() != 0 || handle((unsigned)d, &dev) != 0) { dev = nullptr; return; }
    if (power) power(dev, &power_mw);
  }
  unsigned sm_mhz() const { unsigned v = 0; if (dev && clock) clock(dev, 1 /* NVML_CLOCK_SM */, &v); return v; }
};

struct Case {
  const char* name; uint32_t V, vpc, threads;
  std::vector<uint32_t> P, S;
  uint32_t *dP = nullptr, *dS = nullptr; float* dPart = nullptr; uint32_t grid = 0;
};

int main() {
  const uint32_t N = 48000, SMS = [] { int v = 0; cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, 0); return (uint32_t)v; }();
  const float SR = 48000.0f;
  // the saw table set's shape in the device layout of csrc/host/wavetable.cpp device_wavetable: [t[len-1]] t[0..len) [t[0] t[1]] per table
  WaveTableDev wt[6];
  memset(wt, 0, sizeof(wt));
  std::vector<float> data;
  int nt = 0;
  for (double p = 20.0; p <= 20000.0; p *= pow(2.0, 0.25)) {
    size_t h = (size_t)floor(22000.0 / p), p2 = 1;
    while (p2 < 4 * h) p2 <<= 1;
    const int len = (int)std::min<size_t>(std::max<size_t>(p2, 32), 8192);
    std::vector<float> w(len);
    for (int i = 0; i < len; i++) w[i] = (float)(1.0 - 2.0 * i / len);
    data.push_back(w[len - 1]);
    wt[0].pitch[nt] = (float)p; wt[0].len[nt] = len; wt[0].off[nt] = (int)data.size();
    data.insert(data.end(), w.begin(), w.end());
    data.push_back(w[0]); data.push_back(w[1]);
    nt++;
  }
  while (data.size() & 3) data.push_back(0.0f);
  wt[0].n = nt; wt[0].total = (int)data.size();
  float* dData; CK(cudaMalloc(&dData, data.size() * 4)); CK(cudaMemcpy(dData, data.data(), data.size() * 4, cudaMemcpyHostToDevice));
  wt[0].data = dData;
  WaveTableDev* dWt; CK(cudaMalloc(&dWt, sizeof(wt))); CK(cudaMemcpy(dWt, wt, sizeof(wt), cudaMemcpyHostToDevice));
  const size_t table_bytes = data.size() * 4;

  Case cs[2] = {{"(a) 128 threads, 16384 voices", 16384, 0, 128},
                {"(b) 256 threads, 33000 voices", 33000, 250, 256}};
  for (Case& c : cs) {
    if (!c.vpc) bank_grid(c.V, 128u, SMS, &c.vpc);
    c.grid = (c.V + c.vpc - 1) / c.vpc;
    c.P.assign(7 * (size_t)c.V, 0); c.S.assign(4 * (size_t)c.V, 0);
    for (uint32_t i = 0; i < c.V; i++) {   // saw_hz(f).phase(p) >> lowpass_hz(fc, q): words f | a1 a2 a3 m0 m1 m2, state phase hint ic1 ic2
      const double fc = xerp(100.0, 12000.0, u(i, 0)), q = 0.5 + 9.5 * u(i, 1), f = xerp(55.0, 1760.0, u(i, 2));
      const double g = tan(M_PI * fc / SR), k = 1.0 / q, a1 = 1.0 / (1.0 + g * (g + k)), a2 = g * a1, a3 = g * a2;
      const float w[7] = {(float)f, (float)a1, (float)a2, (float)a3, 0.0f, 0.0f, 1.0f};
      for (int j = 0; j < 7; j++) memcpy(&c.P[(size_t)j * c.V + i], &w[j], 4);
      const float ph = (float)u(i, 3);
      memcpy(&c.S[i], &ph, 4);
    }
    CK(cudaMalloc(&c.dP, c.P.size() * 4)); CK(cudaMemcpy(c.dP, c.P.data(), c.P.size() * 4, cudaMemcpyHostToDevice));
    CK(cudaMalloc(&c.dS, c.S.size() * 4));
    CK(cudaMalloc(&c.dPart, (size_t)c.grid * N * 4));
  }
  auto launch = [&](Case& c, bool reset) {
    if (reset) CK(cudaMemcpy(c.dS, c.S.data(), c.S.size() * 4, cudaMemcpyHostToDevice));
    BankArgs a{};
    a.params = c.dP; a.state = c.dS; a.wt = dWt; a.partial = c.dPart; a.V = c.V; a.n = N; a.vpc = c.vpc;
    a.sr = SR; a.sd64 = (float)(1.0 / SR); a.sd32 = 1.0f / SR;
    const size_t smem = sizeof(float) * mix_tile_floats(1, c.threads) + table_bytes;   // (b): 64 x 257 floats + tables, under 227 KB
    if (c.threads == 128) {
      CK(cudaFuncSetAttribute(bank_kernel<Headline, 128, 2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      bank_kernel<Headline, 128, 2, true><<<c.grid, 128, smem>>>(a);
    } else {
      CK(cudaFuncSetAttribute(bank_kernel<Headline, 256, 2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      bank_kernel<Headline, 256, 2, true><<<c.grid, 256, smem>>>(a);
    }
    CK(cudaGetLastError());
  };

  Nvml nv;
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  double rate[2];
  const int REPS = 10;
  for (int r = 0; r < 2; r++) {   // two alternating rounds; the second is reported
    for (int i = 0; i < 2; i++) {
      Case& c = cs[i];
      launch(c, true); CK(cudaDeviceSynchronize());   // warm-up
      unsigned mhz_sum = 0, mhz_n = 0;
      CK(cudaEventRecord(e0));
      for (int k = 0; k < REPS; k++) launch(c, false);
      CK(cudaEventRecord(e1));
      while (cudaEventQuery(e1) == cudaErrorNotReady) { const unsigned m = nv.sm_mhz(); if (m) { mhz_sum += m; mhz_n++; } }
      CK(cudaEventSynchronize(e1));
      float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
      rate[i] = (double)c.V * N * REPS / (ms * 1e-3);
      if (r == 1) printf("%s: vpc %u, grid %u: %.2f ms per launch, %.1f Gsample/s, SM clock %u MHz\n", c.name, c.vpc, c.grid, ms / REPS, rate[i] * 1e-9,
                         mhz_n ? mhz_sum / mhz_n : 0u);
    }
  }
  printf("card %s, power limit %.0f W\n", prop.name, nv.power_mw * 1e-3);
  printf("headroom (b)/(a) = %.3f\n", rate[1] / rate[0]);
  return 0;
}
