// Bring-up probe of the tensor-core convolver kernel (fundsp_b200/csrc/dsp/conv_tc_kernel.cuh), TEST INFRASTRUCTURE.
// usage: conv_tc_probe [K] [V] [n]   — runs the kernel on random rows and compares with an f64 convolution.
//   nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O2 -std=c++17 -I fundsp_b200/csrc tests/cpp/conv_tc_probe.cu fundsp_b200/csrc/inst/inst_conv.cu -o tests/cpp/_probe/conv_tc_probe -lcuda
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "host/registry.h"

using namespace fdsp;
using namespace fdsp::host;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("FAIL %s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

int main(int argc, char** argv) {
  const uint32_t K = argc > 1 ? atoi(argv[1]) : 100, V = argc > 2 ? atoi(argv[2]) : 200, n = argc > 3 ? atoi(argv[3]) : 300;
  const uint32_t H = (K - 1 + 31) / 32 * 32 ? (K - 1 + 31) / 32 * 32 : 32, stride = H + 1024, J = conv_tc_toeplitz_cols(K);
  std::vector<float> x((size_t)V * stride, 0.0f), h(K);
  srand(1);
  for (uint32_t v = 0; v < V; v++) for (uint32_t t = 0; t < n; t++) x[(size_t)v * stride + H + t] = (float)rand() / RAND_MAX * 2.0f - 1.0f;
  for (uint32_t k = 0; k < K; k++) h[k] = ((float)rand() / RAND_MAX * 2.0f - 1.0f) * expf(-(float)k / (K / 3.0f + 1.0f));
  float *dx, *dxl, *dh, *dth, *dtl, *dy; uint32_t* drow;
  CK(cudaMalloc(&dx, x.size() * 4)); CK(cudaMalloc(&dxl, x.size() * 4)); CK(cudaMalloc(&dh, K * 4)); CK(cudaMalloc(&dth, (size_t)128 * J * 4)); CK(cudaMalloc(&dtl, (size_t)128 * J * 4));
  CK(cudaMalloc(&dy, (size_t)V * 1024 * 4)); CK(cudaMalloc(&drow, V * 4));
  std::vector<uint32_t> rows(V); for (uint32_t v = 0; v < V; v++) rows[v] = v;
  CK(cudaMemcpy(dx, x.data(), x.size() * 4, cudaMemcpyHostToDevice)); CK(cudaMemset(dxl, 0, x.size() * 4)); CK(cudaMemcpy(dh, h.data(), K * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(drow, rows.data(), V * 4, cudaMemcpyHostToDevice)); CK(cudaMemset(dy, 0, (size_t)V * 1024 * 4));
  CK(launch_conv_toeplitz(dh, K, dth, dtl, J, 0)); CK(launch_conv_split(dx, dxl, V, stride, H, n, 0)); CK(cudaDeviceSynchronize());
  ConvTcMaps maps;
  CK(conv_tc_make_maps(dx, dxl, V, stride, dth, dtl, J, &maps));
  cudaError_t e = launch_conv_tc(maps, dy, 1024, 0, drow, V, n, K, H, 0);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  printf("K=%u V=%u n=%u: %s\n", K, V, n, cudaGetErrorString(e));
  if (e != cudaSuccess) return 1;
  std::vector<float> y((size_t)V * 1024);
  CK(cudaMemcpy(y.data(), dy, y.size() * 4, cudaMemcpyDeviceToHost));
  double worst = 0, peak = 0;
  for (uint32_t v : {0u, 1u, 77u % V, V - 1}) for (uint32_t t = 0; t < n; t++) {
    double s = 0;
    for (uint32_t k = 0; k < K && k <= t; k++) s += (double)h[k] * (double)x[(size_t)v * stride + H + t - k];
    worst = fmax(worst, fabs(s - y[(size_t)v * 1024 + t])); peak = fmax(peak, fabs(s));
  }
  printf("max |err| %.3g, peak %.3g, rel %.3g  %s\n", worst, peak, worst / peak, worst <= 1e-5 * peak ? "OK" : "MISMATCH");
  printf("y[0][0..4] = %g %g %g %g\n", y[0], y[1], y[2], y[3]);
  return worst <= 1e-5 * peak ? 0 : 2;
}
