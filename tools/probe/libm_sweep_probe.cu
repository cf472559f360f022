// Probe (test infrastructure, not product): the PRODUCT's scalar f32 math on the device over every argument of the scalar-math sweep
// (tests/golden/libm_sweep_args.h), in two builds of the same kernel source (libm_sweep_kernel.cuh):
//   nvcc   compiled into this binary with the product's flags (-fmad=false, no fast math);
//   nvrtc  compiled at run time through NVRTC with the closure JIT's option list (kJitOpts below = kJitOpts in csrc/host/jit.cpp,
//          which tests/test_libm_sweep_cpu.py checks), as closure nodes are.
// For each function it prints per-chunk hashes (compared with tests/golden/libm_sweep.json by tests/test_gpu_libm_sweep.py), the
// largest ulp error against CUDA's double-precision function and the wall time of the pass. One launch covers at most 16 chunks.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -fmad=false -Ifundsp_b200/csrc/dsp -Itests/golden \
//        -o tools/probe/_build/libm_sweep_probe tools/probe/libm_sweep_probe.cu \
//        -lnvrtc_static -lnvrtc-builtins_static -lnvptxcompiler_static      (as __graft_entry__.build() does)
//   libm_sweep_probe --root REPO --build nvcc|nvrtc [fn ...]          one JSON line per function on stdout
//   libm_sweep_probe --root REPO --build nvcc|nvrtc --chunk FN K OUT  chunk K of FN into OUT: x, y, result bits (3 x 2^24 u32)
//   libm_sweep_probe --root REPO --build nvrtc --compile-only          the NVRTC compilation alone (no GPU needed)
#include <cuda_runtime.h>
#include <nvrtc.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "libm_sweep_kernel.cuh"

static const char* kJitOpts[] = {"--gpu-architecture=sm_90a", "-std=c++17", "--fmad=false", "-lineinfo", "-default-device"};

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

static std::string slurp(const std::string& p) {
  std::ifstream f(p, std::ios::binary);
  if (!f) { fprintf(stderr, "cannot read %s\n", p.c_str()); exit(1); }
  std::stringstream s; s << f.rdbuf(); return s.str();
}

// the same kernel source through NVRTC with the JIT's options; headers handed over by name, as csrc/host/jit.cpp does
static std::vector<char> nvrtc_cubin(const std::string& root) {
  const std::string src = slurp(root + "/tools/probe/libm_sweep_kernel.cuh");
  const std::string h[3] = {slurp(root + "/fundsp_b200/csrc/dsp/math.cuh"), slurp(root + "/fundsp_b200/csrc/dsp/libm.cuh"),
                            slurp(root + "/tests/golden/libm_sweep_args.h")};
  const char* hs[3] = {h[0].c_str(), h[1].c_str(), h[2].c_str()};
  const char* hn[3] = {"math.cuh", "libm.cuh", "libm_sweep_args.h"};
  nvrtcProgram prog;
  if (nvrtcCreateProgram(&prog, src.c_str(), "libm_sweep_kernel.cu", 3, hs, hn) != NVRTC_SUCCESS) { fprintf(stderr, "nvrtcCreateProgram failed\n"); exit(1); }
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
  void operator()(int fn, unsigned chunk0, unsigned nchunks, unsigned long long* hash, unsigned* ulp, unsigned* dump) const {
    const dim3 grid(512, nchunks), block(256);
    if (!jit) { libm_sweep<<<grid, block>>>(fn, chunk0, hash, ulp, dump); CK(cudaGetLastError()); return; }
    void* args[] = {&fn, &chunk0, &hash, &ulp, &dump};
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
  const char* names[] = SWEEP_NAMES;
  auto fn_id = [&](const std::string& s) { for (int k = 0; k < sweep::NFN; k++) if (s == names[k]) return k; fprintf(stderr, "unknown function %s\n", s.c_str()); exit(2); };
  std::vector<char> cubin;
  if (build == "nvrtc") cubin = nvrtc_cubin(root);
  if (!rest.empty() && rest[0] == "--compile-only") { printf("compiled (%zu bytes of cubin)\n", cubin.size()); return 0; }   // no GPU needed
  Launcher launch;
  cudaLibrary_t lib = nullptr;
  if (build == "nvrtc") { CK(cudaLibraryLoadData(&lib, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0)); CK(cudaLibraryGetKernel(&launch.jit, lib, "libm_sweep")); }
  unsigned long long* d_hash; unsigned* d_ulp;
  CK(cudaMalloc(&d_hash, 256 * 8)); CK(cudaMalloc(&d_ulp, 4));
  if (!rest.empty() && rest[0] == "--chunk") {
    if (rest.size() != 4) { fprintf(stderr, "--chunk FN K OUT\n"); return 2; }
    const int fn = fn_id(rest[1]); const unsigned k = (unsigned)atoi(rest[2].c_str());
    if ((int)k >= sweep::chunks(fn)) { fprintf(stderr, "chunk out of range\n"); return 2; }
    unsigned* d_dump; CK(cudaMalloc(&d_dump, (size_t)12 << sweep::CHUNK_LOG2));
    CK(cudaMemset(d_hash, 0, 8));
    launch(fn, k, 1, d_hash, d_ulp, d_dump);
    std::vector<unsigned> out((size_t)3 << sweep::CHUNK_LOG2);
    CK(cudaMemcpy(out.data(), d_dump, out.size() * 4, cudaMemcpyDeviceToHost));
    FILE* f = fopen(rest[3].c_str(), "wb");
    if (!f || fwrite(out.data(), 4, out.size(), f) != out.size()) { fprintf(stderr, "cannot write %s\n", rest[3].c_str()); return 1; }
    fclose(f);
    CK(cudaFree(d_dump)); CK(cudaFree(d_hash)); CK(cudaFree(d_ulp));
    if (lib) CK(cudaLibraryUnload(lib));
    return 0;
  }
  std::vector<int> fns;
  for (auto& s : rest) fns.push_back(fn_id(s));
  if (fns.empty()) for (int k = 0; k < sweep::NFN; k++) fns.push_back(k);
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  for (int fn : fns) {
    const int nc = sweep::chunks(fn);
    CK(cudaMemset(d_hash, 0, 256 * 8)); CK(cudaMemset(d_ulp, 0, 4));
    CK(cudaEventRecord(e0));
    for (int c = 0; c < nc; c += 16) launch(fn, (unsigned)c, (unsigned)(nc - c < 16 ? nc - c : 16), d_hash + c, d_ulp, nullptr);
    CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
    std::vector<unsigned long long> h(nc); unsigned ub = 0;
    CK(cudaMemcpy(h.data(), d_hash, nc * 8, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(&ub, d_ulp, 4, cudaMemcpyDeviceToHost));
    float ulp; memcpy(&ulp, &ub, 4);
    printf("{\"build\": \"%s\", \"fn\": \"%s\", \"ms\": %.2f, \"max_ulp\": %.6f, \"hashes\": [", build.c_str(), names[fn], ms, ulp);
    for (int c = 0; c < nc; c++) printf("%s\"%016llx\"", c ? ", " : "", h[c]);
    printf("]}\n");
    fflush(stdout);
  }
  CK(cudaEventDestroy(e0)); CK(cudaEventDestroy(e1)); CK(cudaFree(d_hash)); CK(cudaFree(d_ulp));
  if (lib) CK(cudaLibraryUnload(lib));
  return 0;
}
