// Tensor-core convolve path (csrc/dsp/conv_tc_kernel.cuh): tensor maps + launchers.
#include "../dsp/conv_tc_kernel.cuh"
#include "../host/registry.h"

#include <cstring>

namespace fdsp { namespace host {

namespace {
typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                             CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeFn encode_fn() {
  static EncodeFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) p = nullptr;
    return (EncodeFn)p;
  }();
  return fn;
}
// 2-D f32 tensor [rows][cols] (cols contiguous, row pitch `pitch` floats), box = 32 columns x `box_rows` rows, 128-byte swizzle, zero fill outside
bool make_map(CUtensorMap* m, float* base, uint64_t cols, uint64_t rows, uint64_t pitch, uint32_t box_rows) {
  EncodeFn enc = encode_fn();
  if (!enc) return false;
  const cuuint64_t dims[2] = {cols, rows}, strides[1] = {pitch * sizeof(float)};
  const cuuint32_t box[2] = {(cuuint32_t)CTC_KC, (cuuint32_t)box_rows}, estr[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
             CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
}  // namespace

static_assert(sizeof(CUtensorMap) == 128, "ConvTcMaps layout");

cudaError_t conv_tc_make_maps(float* x, float* xl, uint32_t V, uint32_t row_stride, float* th, float* tl, uint32_t J, ConvTcMaps* out) {
  CUtensorMap* m = reinterpret_cast<CUtensorMap*>(out->m);
  if (!make_map(&m[0], x, row_stride, V, row_stride, CTC_M) || !make_map(&m[1], xl, row_stride, V, row_stride, CTC_M) || !make_map(&m[2], th, J, CTC_N, J, CTC_N) ||
      !make_map(&m[3], tl, J, CTC_N, J, CTC_N))
    return cudaErrorInvalidValue;
  return cudaSuccess;
}
cudaError_t launch_conv_tc(const ConvTcMaps& maps, float* y, uint32_t y_stride, uint32_t y_offset, const uint32_t* row_map, uint32_t V, uint32_t n, uint32_t K, uint32_t H,
                           cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CTC_SMEM);
    if (e != cudaSuccess) return e;
    attr = true;
  }
  const CUtensorMap* m = reinterpret_cast<const CUtensorMap*>(maps.m);
  ConvTcArgs a{y, y_stride, y_offset, row_map, V, n, K, H};
  dim3 grid((n + CTC_N - 1) / CTC_N, (V + CTC_M - 1) / CTC_M);
  conv_tc_kernel<<<grid, CTC_THREADS, CTC_SMEM, st>>>(m[0], m[1], m[2], m[3], a);
  return cudaGetLastError();
}
cudaError_t launch_conv_split(float* x, float* xl, uint32_t V, uint32_t row_stride, uint32_t col0, uint32_t n, cudaStream_t st) {
  if (n == 0 || V == 0) return cudaSuccess;
  conv_split_lo_kernel<<<dim3((n + 255) / 256, V), 256, 0, st>>>(x, xl, V, row_stride, col0, n);
  return cudaGetLastError();
}
cudaError_t launch_conv_history(float* x, float* xl, uint32_t V, uint32_t row_stride, uint32_t H, uint32_t n, cudaStream_t st) {
  if (V == 0 || H == 0) return cudaSuccess;
  conv_history_kernel<<<dim3(V, 2), 256, (size_t)H * sizeof(float), st>>>(x, xl, row_stride, H, n);
  return cudaGetLastError();
}
cudaError_t launch_conv_toeplitz(const float* h, uint32_t K, float* th, float* tl, uint32_t J, cudaStream_t st) {
  conv_toeplitz_kernel<<<dim3((J + 255) / 256, CTC_N), 256, 0, st>>>(h, K, th, tl, J);
  return cudaGetLastError();
}
uint32_t conv_tc_toeplitz_cols(uint32_t K) { return (CTC_N + ((K - 1u + 3u) & ~3u) + CTC_KC - 1u) / CTC_KC * CTC_KC; }
}}
