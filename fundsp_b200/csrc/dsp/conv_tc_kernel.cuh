// fundsp_b200 tensor-core path of `convolve(h)` (reference src/convolve.rs:9-59, ID 100; the same contraction as a long `Fir`,
// src/fir.rs:43-89): V voices share ONE impulse response h of K taps, so a block of their outputs is a dense GEMM against the
// Toeplitz matrix of h — the one place on this path where tensor cores apply (north-star: "tensor cores are used only on the dense
// FIR/convolve tap contraction as a batched GEMM").
//
//     Y[v, t0 + n] = sum_j X[v, t0 - P + j] * T[j, n],     T[j, n] = h[P + n - j]  (0 outside the band),  j < N + P,  P = K - 1 rounded up to 4
//
//   M = 128 voices per CTA tile, N = 64 output samples, contraction over the N + K - 1 input samples the tile can see, in chunks
//   of 32 floats (one 128-byte swizzle row). Flops per tile = 2 * 128 * 64 * (63 + K)  (SURVEY.md §8d: 2 * V * 64 * (63 + K) per
//   64-block), of which 2 * 128 * 64 * K are the convolution's own.
//
// Precision: TF32 keeps 10 mantissa bits, the bar is 1e-5 of the output peak, so the product is taken in the 3xTF32 split
//     x ~ xh + xl,  h ~ hh + hl   (tf32(f) = f with the low 13 mantissa bits cleared; xh = tf32(x), xl = tf32(x - xh), same for h)
//     x * h  ~  xh*hl + xl*hh + xh*hh        (xh + xl and hh + hl are within 2^-20 of x and h; the dropped xl*hl is <= 2^-20 |x h|)
// as three `wgmma.mma_async ... .tf32` per 8-wide k-step. The split is stored: conv_split_lo_kernel rewrites the X rows as xh in place
// and writes xl beside them, conv_toeplitz_kernel writes hh and hl, all four already TF32, so the result does not depend on how the
// tensor core would have converted an FP32 operand. (xh + xl is exact in FP32: with a one-hot response the output is exactly xh + xl.)
// Accumulation: the tensor core rounds the FP32 accumulator at every MMA, and a 4096-tap response is 520 k-steps in a row (the error grows
// with K; DESIGN.md §2 has the errors measured on an H100 from 32 to 48 000 taps). So the sum is spread over FIVE register accumulators: the
// xh*hh products of k-step k = 0..3 of every chunk in four of them — a quarter of the sequential roundings each; the k-step picks the
// accumulator statically, so no branch sits between the asynchronous MMAs — and both cross terms, 2^-11 smaller, in the fifth, where
// their roundings do not count; the epilogue adds the five in FP32.
//
// Kernel (one output tile per CTA, 384 threads): warpgroups 0 and 1 = consumers, each owning 64 voices of the tile (m64n64k8
// `wgmma` from shared memory, 5 x 32 accumulator registers per thread, then the epilogue straight from registers to HBM); warpgroup 2
// hands its registers to them (`setmaxnreg`) and one of its threads is the TMA producer (4 `cp.async.bulk.tensor.2d` per stage: X, Xlo, T, Tlo tiles, 128-byte swizzle, 4-stage ring of 48 KB, full/empty
// mbarriers; a stage is released once both warpgroups' `wgmma` groups reading it have completed).
// X rows live in HBM as [voice][H + chunk] with the last H >= K - 1 samples of the previous chunk in front (conv_history_kernel
// moves them there), so a window never leaves its row; rows past V and columns past the data are zero-filled by TMA / ignored
// by the epilogue (the Toeplitz band is causal: they only reach outputs that are not stored).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>

namespace fdsp {

constexpr int CTC_M = 128, CTC_N = 64, CTC_KC = 32, CTC_STAGES = 4;
// Every CTC_FLUSH contraction chunks (and only if more follow) the consumers wait for their wgmma groups, add the five accumulators into a
// register sum on the CUDA cores and restart them from zero, so no accumulator takes more than CTC_FLUSH * 4 roundings in a row. 64 chunks:
// responses up to 1985 taps (K = 1000 is 34 chunks) never flush.
constexpr int CTC_FLUSH = 64;
constexpr int CTC_THREADS = 384;                                                          // 2 consumer warpgroups + 1 producer warpgroup
constexpr int CTC_TILE_A = CTC_M * CTC_KC * 4, CTC_TILE_B = CTC_N * CTC_KC * 4;          // bytes: 16 KB, 8 KB
constexpr int CTC_STAGE_BYTES = 2 * CTC_TILE_A + 2 * CTC_TILE_B;                          // X, Xlo, T, Tlo
constexpr int CTC_SMEM = CTC_STAGES * CTC_STAGE_BYTES + 1024 /*alignment slack*/ + 256 /*barriers*/;

struct ConvTcArgs {
  float* y; uint32_t y_stride, y_offset;       // output rows y[row_map[v] * y_stride + y_offset + t]
  const uint32_t* row_map;
  uint32_t V, n;                               // voices, samples of this launch
  uint32_t K, H;                               // taps; history columns in front of every X row (multiple of 32, >= K - 1)
};

__device__ __forceinline__ uint32_t ctc_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void ctc_mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count)); }
__device__ __forceinline__ void ctc_mbar_expect(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void ctc_mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void ctc_mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile("{\n\t.reg .pred p;\n\tCW_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra CD_%=;\n\tbra CW_%=;\n\tCD_%=:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void ctc_tma_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar) : "memory");
}
// wgmma shared-memory matrix descriptor (sm_90), K-major, 128-byte swizzle: start address >> 4 (bits 0-13), leading byte offset (unused
// with swizzle) = 1 (bits 16-29), stride byte offset = 1024 B between 8-row groups (bits 32-45), layout type 1 = SWIZZLE_128B (bits 62-63)
__device__ __forceinline__ uint64_t ctc_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3ffffu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// d[64 x 64] += A[64 x 8] * B[8 x 64], both operands TF32 from shared memory (K-major); d in the warpgroup's accumulator fragment
__device__ __forceinline__ void ctc_wgmma(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
        "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
        "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(1));
}
__device__ __forceinline__ void ctc_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void ctc_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void ctc_wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void ctc_fence_acc(float (&d)[32]) {   // the accumulators are read only after the wait
#pragma unroll
  for (int j = 0; j < 32; j++) asm volatile("" : "+f"(d[j])::"memory");
}

// one 8-wide k-step of a 32-wide contraction chunk:  hi += xh*hh,  cross += xh*hl + xl*hh
__device__ __forceinline__ void ctc_kstep(int k, float (&hi)[32], float (&cross)[32], uint64_t dxh, uint64_t dxl, uint64_t dth, uint64_t dtl) {
  const uint64_t adv = (uint64_t)((k * 32) >> 4);                                // 8 floats = 32 bytes further inside the swizzle row
  ctc_wgmma(hi, dxh + adv, dth + adv);
  ctc_wgmma(cross, dxh + adv, dtl + adv);
  ctc_wgmma(cross, dxl + adv, dth + adv);
}

// grid = (time tiles, voice tiles); block = CTC_THREADS
static __global__ void __launch_bounds__(CTC_THREADS, 1) conv_tc_kernel(const __grid_constant__ CUtensorMap mx, const __grid_constant__ CUtensorMap mxl,
                                                                 const __grid_constant__ CUtensorMap mt, const __grid_constant__ CUtensorMap mtl, const ConvTcArgs a) {
  extern __shared__ uint8_t ctc_raw[];
  const uint32_t base = (ctc_smem(ctc_raw) + 1023u) & ~1023u;                  // 128-byte swizzle atoms are 1024-byte aligned
  const uint32_t bars = base + CTC_STAGES * CTC_STAGE_BYTES;                   // full[S], empty[S]
  auto full_bar = [&](int s) { return bars + 8u * (uint32_t)s; };
  auto empty_bar = [&](int s) { return bars + 8u * (uint32_t)(CTC_STAGES + s); };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t t0 = blockIdx.x * CTC_N, v0 = blockIdx.y * CTC_M;
  const uint32_t P = (a.K - 1u + 3u) & ~3u;                                    // look-back padded to 4 samples: every window starts 16-byte aligned
  const int nchunk = (int)((CTC_N + P + CTC_KC - 1u) / CTC_KC);                // contraction chunks of 32 input samples

  if (threadIdx.x == 0) {
    for (int s = 0; s < CTC_STAGES; s++) { ctc_mbar_init(full_bar(s), 1); ctc_mbar_init(empty_bar(s), 8); }   // empty: one arrival per consumer warp
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 8 && lane == 0) {   // ---- TMA producer
      const int col0 = (int)(a.H - P + t0);                                    // window start inside the X rows
      for (int c = 0; c < nchunk; c++) {
        const int s = c % CTC_STAGES, use = c / CTC_STAGES;
        if (use > 0) ctc_mbar_wait(empty_bar(s), (uint32_t)(use - 1) & 1u);
        const uint32_t st = base + (uint32_t)s * CTC_STAGE_BYTES;
        ctc_mbar_expect(full_bar(s), CTC_STAGE_BYTES);
        ctc_tma_2d(st, &mx, col0 + c * CTC_KC, (int)v0, full_bar(s));
        ctc_tma_2d(st + CTC_TILE_A, &mxl, col0 + c * CTC_KC, (int)v0, full_bar(s));
        ctc_tma_2d(st + 2 * CTC_TILE_A, &mt, c * CTC_KC, 0, full_bar(s));
        ctc_tma_2d(st + 2 * CTC_TILE_A + CTC_TILE_B, &mtl, c * CTC_KC, 0, full_bar(s));
      }
    }
    return;
  }

  // ---- consumers: warpgroup g computes voices v0 + 64 g .. +63 of the tile
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int g = warp >> 2;
  float a0[32], a1[32], a2[32], a3[32], ax[32];
#pragma unroll
  for (int j = 0; j < 32; j++) { a0[j] = 0.0f; a1[j] = 0.0f; a2[j] = 0.0f; a3[j] = 0.0f; ax[j] = 0.0f; }
  float sum[32];                                                               // flushed partial sums, added on the CUDA cores (round to nearest)
#pragma unroll
  for (int j = 0; j < 32; j++) sum[j] = 0.0f;
  const uint32_t arow = (uint32_t)g * (64u * CTC_KC * 4u);                     // this warpgroup's 64 rows of the X tiles (8 swizzle atoms)
#pragma unroll 1
  for (int c = 0; c < nchunk; c++) {
    const int s = c % CTC_STAGES, use = c / CTC_STAGES;
    ctc_mbar_wait(full_bar(s), (uint32_t)use & 1u);
    const uint32_t st = base + (uint32_t)s * CTC_STAGE_BYTES;
    const uint64_t dxh = ctc_desc(st + arow), dxl = ctc_desc(st + CTC_TILE_A + arow), dth = ctc_desc(st + 2 * CTC_TILE_A), dtl = ctc_desc(st + 2 * CTC_TILE_A + CTC_TILE_B);
    ctc_wgmma_fence();
    ctc_kstep(0, a0, ax, dxh, dxl, dth, dtl);                                  // xh*hh: accumulator k
    ctc_kstep(1, a1, ax, dxh, dxl, dth, dtl);
    ctc_kstep(2, a2, ax, dxh, dxl, dth, dtl);
    ctc_kstep(3, a3, ax, dxh, dxl, dth, dtl);
    ctc_wgmma_commit();
    ctc_wgmma_wait<1>();                                                       // chunk c - 1 has been read: its stage is free
    __syncwarp();
    if (c > 0 && lane == 0) ctc_mbar_arrive(empty_bar((c - 1) % CTC_STAGES));
    if ((c + 1) % CTC_FLUSH == 0 && c + 1 < nchunk) {                     // long responses: bound the run of tensor-core accumulator roundings
      ctc_wgmma_wait<0>();
      ctc_fence_acc(a0); ctc_fence_acc(a1); ctc_fence_acc(a2); ctc_fence_acc(a3); ctc_fence_acc(ax);
#pragma unroll
      for (int j = 0; j < 32; j++) {
        sum[j] += ((a0[j] + a1[j]) + (a2[j] + a3[j])) + ax[j];
        a0[j] = 0.0f; a1[j] = 0.0f; a2[j] = 0.0f; a3[j] = 0.0f; ax[j] = 0.0f;
      }
    }
  }
  ctc_wgmma_wait<0>();
  ctc_fence_acc(a0); ctc_fence_acc(a1); ctc_fence_acc(a2); ctc_fence_acc(a3); ctc_fence_acc(ax);

  // ---- epilogue: fragment of m64nN: warp w of the warpgroup holds rows 16 w + lane / 4 (regs 4 i + 0, 1) and + 8 (4 i + 2, 3),
  // columns 8 i + 2 (lane % 4) + {0, 1}
  const int w = warp & 3;
  const bool vec_ok = ((a.y_stride | a.y_offset) & 1u) == 0u;
#pragma unroll
  for (int half = 0; half < 2; half++) {
    const uint32_t v = v0 + (uint32_t)(g * 64 + w * 16 + (lane >> 2) + half * 8);
    if (v >= a.V) continue;
    float* yrow = a.y + (size_t)__ldg(a.row_map + v) * a.y_stride + a.y_offset + t0;
#pragma unroll
    for (int i = 0; i < CTC_N / 8; i++) {
      const int j = 4 * i + 2 * half;
      const float y0 = sum[j] + (((a0[j] + a1[j]) + (a2[j] + a3[j])) + ax[j]);  // flushed + (((a0 + a1) + (a2 + a3)) + cross); 0 + y = y
      const float y1 = sum[j + 1] + (((a0[j + 1] + a1[j + 1]) + (a2[j + 1] + a3[j + 1])) + ax[j + 1]);
      const uint32_t col = (uint32_t)(8 * i + 2 * (lane & 3));
      const uint32_t left = a.n > t0 + col ? a.n - t0 - col : 0u;             // valid samples from this column on
      if (vec_ok && left >= 2u) *reinterpret_cast<float2*>(yrow + col) = make_float2(y0, y1);
      else { if (left >= 1u) yrow[col] = y0; if (left >= 2u) yrow[col + 1] = y1; }
    }
  }
}

__device__ __forceinline__ float ctc_tf32(float f) { return __uint_as_float(__float_as_uint(f) & 0xffffe000u); }   // low 13 mantissa bits cleared

// xh = tf32(x) (in place), xl = tf32(x - xh), over the new columns of every X row. Grid = (voices, time blocks): voices on x, which has
// no 65 535 limit.
static __global__ void conv_split_lo_kernel(float* __restrict__ x, float* __restrict__ xl, uint32_t V, uint32_t row_stride, uint32_t col0, uint32_t n) {
  const uint32_t t = blockIdx.y * blockDim.x + threadIdx.x, v = blockIdx.x;
  if (t >= n || v >= V) return;
  const size_t e = (size_t)v * row_stride + col0 + t;
  const float f = x[e], hi = ctc_tf32(f);
  x[e] = hi;
  xl[e] = ctc_tf32(f - hi);
}
// the last H samples of every row (columns [n, n + H)) move to the front (columns [0, H)): history for the next chunk. One CTA per
// (row, array). Source and destination overlap when n < H, so this is a memmove to lower addresses: tiles of CTC_HIST_TILE columns in
// ascending order, each read whole into registers before any of it is written. A later tile reads only columns >= n + its start, which
// no earlier tile wrote, so any H works without shared memory.
constexpr int CTC_HIST_THREADS = 256, CTC_HIST_PER = 4, CTC_HIST_TILE = CTC_HIST_THREADS * CTC_HIST_PER;
static __global__ void __launch_bounds__(CTC_HIST_THREADS) conv_history_kernel(float* x, float* xl, uint32_t row_stride, uint32_t H, uint32_t n) {
  float* row = (blockIdx.y ? xl : x) + (size_t)blockIdx.x * row_stride;
  for (uint32_t base = 0; base < H; base += CTC_HIST_TILE) {
    float r[CTC_HIST_PER];
#pragma unroll
    for (int q = 0; q < CTC_HIST_PER; q++) { const uint32_t i = base + q * CTC_HIST_THREADS + threadIdx.x; if (i < H) r[q] = row[n + i]; }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < CTC_HIST_PER; q++) { const uint32_t i = base + q * CTC_HIST_THREADS + threadIdx.x; if (i < H) row[i] = r[q]; }
    __syncthreads();
  }
}
// T[n][j] = h[P + n - j] inside the band, 0 outside (P = K - 1 rounded up to 4: window column j is input sample t0 - P + j); hi = tf32(h),
// lo = tf32(h - hi). Rows n < CTC_N, J columns (multiple of 32).
static __global__ void conv_toeplitz_kernel(const float* __restrict__ h, uint32_t K, float* th, float* tl, uint32_t J) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x, n = blockIdx.y;
  if (j >= J) return;
  const int k = (int)((K - 1u + 3u) & ~3u) + (int)n - (int)j;
  const float f = (k >= 0 && k < (int)K) ? h[k] : 0.0f, hi = ctc_tf32(f);
  th[(size_t)n * J + j] = hi;
  tl[(size_t)n * J + j] = ctc_tf32(f - hi);
}

}  // namespace fdsp
