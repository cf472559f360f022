// Probe (test infrastructure, not product): the PRODUCT's f64 math (sin, cos, tan, exp of csrc/dsp/libm64.cuh) on the device over every
// argument of the f64 math sweep (tests/golden/libm64_sweep_args.h), in two builds of the same kernel source (libm64_sweep_kernel.cuh):
//   nvcc   compiled into this binary with the product's flags (-fmad=false, no fast math);
//   nvrtc  compiled at run time through NVRTC with the JIT's option list (kJitOpts below = kJitOpts in csrc/host/jit.cpp, which
//          tests/test_libm64_sweep_cpu.py checks). The prelude64 nodes are built this way only, so this is the build that ships.
// For each function it prints per-chunk hashes (compared with tests/golden/libm64_sweep.json by tests/test_gpu_libm64_sweep.py) and the
// wall time of the pass. One launch covers at most 16 chunks.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -fmad=false -Ifundsp_b200/csrc/dsp -Itests/golden \
//        -o tools/probe/_build/libm64_sweep_probe tools/probe/libm64_sweep_probe.cu \
//        -lnvrtc_static -lnvrtc-builtins_static -lnvptxcompiler_static      (as __graft_entry__.build() does)
//   libm64_sweep_probe --root REPO --build nvcc|nvrtc [fn ...]          one JSON line per function on stdout
//   libm64_sweep_probe --root REPO --build nvcc|nvrtc --chunk FN K OUT  chunk K of FN into OUT: argument and result bits (2 x 2^24 u64;
//                                                                        NaN past the end of the shorter special chunk)
//   libm64_sweep_probe --root REPO --build nvrtc --compile-only          the NVRTC compilation alone (no GPU needed)
#include <cuda_runtime.h>
#include <nvrtc.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "libm64_sweep_kernel.cuh"

static const char* kJitOpts[] = {"--gpu-architecture=sm_90a", "-std=c++17", "--fmad=false", "-lineinfo", "-default-device"};

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

static std::string slurp(const std::string& p) {
  std::ifstream f(p, std::ios::binary);
  if (!f) { fprintf(stderr, "cannot read %s\n", p.c_str()); exit(1); }
  std::stringstream s; s << f.rdbuf(); return s.str();
}

// the same kernel source through NVRTC with the JIT's options; headers handed over by name, as csrc/host/jit.cpp does
static std::vector<char> nvrtc_cubin(const std::string& root) {
  const std::string src = slurp(root + "/tools/probe/libm64_sweep_kernel.cuh");
  const std::string h[4] = {slurp(root + "/fundsp_b200/csrc/dsp/math.cuh"), slurp(root + "/fundsp_b200/csrc/dsp/libm.cuh"),
                            slurp(root + "/fundsp_b200/csrc/dsp/libm64.cuh"), slurp(root + "/tests/golden/libm64_sweep_args.h")};
  const char* hs[4] = {h[0].c_str(), h[1].c_str(), h[2].c_str(), h[3].c_str()};
  const char* hn[4] = {"math.cuh", "libm.cuh", "libm64.cuh", "libm64_sweep_args.h"};
  nvrtcProgram prog;
  if (nvrtcCreateProgram(&prog, src.c_str(), "libm64_sweep_kernel.cu", 4, hs, hn) != NVRTC_SUCCESS) { fprintf(stderr, "nvrtcCreateProgram failed\n"); exit(1); }
  const nvrtcResult rc = nvrtcCompileProgram(prog, (int)(sizeof(kJitOpts) / sizeof(kJitOpts[0])), kJitOpts);
  if (rc != NVRTC_SUCCESS) {
    size_t n = 0; nvrtcGetProgramLogSize(prog, &n);
    std::string log(n, '\0'); if (n) nvrtcGetProgramLog(prog, &log[0]);
    fprintf(stderr, "NVRTC compile failed: %s\n%s\n", nvrtcGetErrorString(rc), log.c_str());
    exit(1);
  }
  size_t n = 0; nvrtcGetCUBINSize(prog, &n);
  std::vector<char> cubin(n); nvrtcGetCUBIN(prog, cubin.data());
  nvrtcDestroyProgram(&prog);
  return cubin;
}

struct Launcher {
  cudaKernel_t jit = nullptr;   // null: the nvcc build
  void operator()(int fn, unsigned chunk0, unsigned nchunks, unsigned long long* hash, unsigned long long* dump) const {
    const dim3 grid(512, nchunks), block(256);
    if (!jit) { libm64_sweep<<<grid, block>>>(fn, chunk0, hash, dump); CK(cudaGetLastError()); return; }
    void* args[] = {&fn, &chunk0, &hash, &dump};
    CK(cudaLaunchKernel((const void*)jit, grid, block, args, 0, nullptr));
  }
};

int main(int argc, char** argv) {
  std::string root = ".", build = "nvcc";
  std::vector<std::string> rest;
  for (int a = 1; a < argc; a++) {
    const std::string s = argv[a];
    if (s == "--root" && a + 1 < argc) root = argv[++a];
    else if (s == "--build" && a + 1 < argc) build = argv[++a];
    else rest.push_back(s);
  }
  if (build != "nvcc" && build != "nvrtc") { fprintf(stderr, "--build nvcc|nvrtc\n"); return 2; }
  const char* names[] = SWEEP64_NAMES;
  auto fn_id = [&](const std::string& s) { for (int k = 0; k < sweep64::NFN; k++) if (s == names[k]) return k; fprintf(stderr, "unknown function %s\n", s.c_str()); exit(2); };
  std::vector<char> cubin;
  if (build == "nvrtc") cubin = nvrtc_cubin(root);
  if (!rest.empty() && rest[0] == "--compile-only") { printf("compiled (%zu bytes of cubin)\n", cubin.size()); return 0; }   // no GPU needed
  Launcher launch;
  cudaLibrary_t lib = nullptr;
  if (build == "nvrtc") { CK(cudaLibraryLoadData(&lib, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0)); CK(cudaLibraryGetKernel(&launch.jit, lib, "libm64_sweep")); }
  unsigned long long* d_hash;
  CK(cudaMalloc(&d_hash, sweep64::CHUNKS * 8));
  if (!rest.empty() && rest[0] == "--chunk") {
    if (rest.size() != 4) { fprintf(stderr, "--chunk FN K OUT\n"); return 2; }
    const int fn = fn_id(rest[1]); const unsigned k = (unsigned)atoi(rest[2].c_str());
    if ((int)k >= sweep64::CHUNKS) { fprintf(stderr, "chunk out of range\n"); return 2; }
    unsigned long long* d_dump; CK(cudaMalloc(&d_dump, (size_t)16 << sweep64::CHUNK_LOG2));
    CK(cudaMemset(d_dump, 0xff, (size_t)16 << sweep64::CHUNK_LOG2));   // past a short chunk's end: NaN arguments and results
    CK(cudaMemset(d_hash, 0, 8));
    launch(fn, k, 1, d_hash, d_dump);
    std::vector<unsigned long long> out((size_t)2 << sweep64::CHUNK_LOG2);
    CK(cudaMemcpy(out.data(), d_dump, out.size() * 8, cudaMemcpyDeviceToHost));
    FILE* f = fopen(rest[3].c_str(), "wb");
    if (!f || fwrite(out.data(), 8, out.size(), f) != out.size()) { fprintf(stderr, "cannot write %s\n", rest[3].c_str()); return 1; }
    fclose(f);
    CK(cudaFree(d_dump)); CK(cudaFree(d_hash));
    if (lib) CK(cudaLibraryUnload(lib));
    return 0;
  }
  std::vector<int> fns;
  for (auto& s : rest) fns.push_back(fn_id(s));
  if (fns.empty()) for (int k = 0; k < sweep64::NFN; k++) fns.push_back(k);
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  for (int fn : fns) {
    const int nc = sweep64::CHUNKS;
    CK(cudaMemset(d_hash, 0, nc * 8));
    CK(cudaEventRecord(e0));
    for (int c = 0; c < nc; c += 16) launch(fn, (unsigned)c, (unsigned)(nc - c < 16 ? nc - c : 16), d_hash + c, nullptr);
    CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
    std::vector<unsigned long long> h(nc);
    CK(cudaMemcpy(h.data(), d_hash, nc * 8, cudaMemcpyDeviceToHost));
    printf("{\"build\": \"%s\", \"fn\": \"%s\", \"ms\": %.2f, \"hashes\": [", build.c_str(), names[fn], ms);
    for (int c = 0; c < nc; c++) printf("%s\"%016llx\"", c ? ", " : "", h[c]);
    printf("]}\n");
    fflush(stdout);
  }
  CK(cudaEventDestroy(e0)); CK(cudaEventDestroy(e1)); CK(cudaFree(d_hash));
  if (lib) CK(cudaLibraryUnload(lib));
  return 0;
}
