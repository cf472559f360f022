// fundsp_b200 warp-per-voice kernel for `reverb_stereo` (reference src/prelude.rs:1732-1762): the 32-line Hadamard
// feedback delay network  multisplit<2,16> >> fdn<32>(stacki<32>(delay >> fir3)) >> sumf<32>(pan) * dc((1/16,1/16)).
//
// The reference ticks the whole inner graph per sample (src/feedback.rs:136-146): 32 x (Delay::tick src/delay.rs:116-124
// + Fir<U3>::tick src/fir.rs:57-70) + one 32-point Hadamard (src/feedback.rs:35-57). This is the one HBM-bound program of
// the path: 32 lines x (4 B read + 4 B write) per voice-sample, and the kernel is organised around moving those bytes.
//
// ONE WARP = one voice, and inside a 64-sample block the warp works TIME-parallel (round 2; round 1 had lane = delay line):
// every delay is >= 192 samples, so what the network writes in a block cannot reach what it reads in the same block — the
// 64 samples of a block are independent given the ring contents. Hence
//   * lane t evaluates samples t and t + 32 of the block with ALL 32 lines in its registers: the three FIR taps per line are
//     three neighbouring shared-memory words, the 32-point Hadamard is the reference's in-place butterfly (h = 1, 2, 4, 8, 16;
//     a[j], a[j+h] = x + y, x - y) on a register array — no shuffles —, the output `Reduce` (sum of 32 pans, src/audionode.rs:
//     2442-2463) is the same left fold in line order in two registers;
//   * the ring slice a block reads (32 lines x 64 samples, contiguous per line) is staged with 16-byte `cp.async.cg` (LDGSTS.128:
//     17 warp-instructions per block, lanes cover (line, 16-byte chunk) pairs), three blocks in flight per warp;
//   * the 64 new samples per line are produced in place in the same shared-memory rows and go back with 16-byte stores.
//   (A first round-2 version moved every line's slice with its own `cp.async.bulk` — 64..96 TMA operations of 256 bytes per block
//   and warp. It was bit-exact and no faster than round 1, because the TMA unit serves bulk operations at a fixed cost each regardless
//   of size. Bulk copies pay from about 1 KB up; a delay line hands out 256 contiguous bytes per block.)
// Ring storage (private to this kernel; the host only sizes, clears and copies it): voice-major [voice][line][ring], each
// line's ring padded to a multiple of 64 floats (`fdn_ring_phys`) so that block-aligned slices are 16-byte aligned and a
// block of new samples never straddles the end. The state word of a line holds its WRITE position w; the sample written at w is read
// L - 1 steps later (Delay::tick writes buffer[i], then returns buffer[i + 1], length L).
// Reads always fetch a 16-byte aligned superset of the slice (per-line shift 0..3 floats). After a ragged block (process(size)
// with size % 4 != 0) write positions lose their 16-byte alignment and the write-back falls back to 4-byte stores.
// The wet/dry composition around the reverb,  dry >> (multipass::<U2>() & s * reverb_stereo(..)), is applied in the epilogue.
// Word layout of the reverb inside the class arrays (DFS order, see csrc/host/graph.cpp):
//   P: 32 x Fir weights(3) | 32 x Panner(lw, rw) | Constant<2>          (162 words, first row p0)
//   S: Feedback value[32] | 32 x (Delay idx, Fir v[3])                   (160 words, first row s0)
//   U: 32 x ring length                                                  (first row u0)
#pragma once
#include "math.cuh"
#include "fdn_args.h"

namespace fdsp {

constexpr int FDN_NST_DEFAULT = 2;                      // ring-slice stages per warp: block b + 1 is fetched while block b is computed (a block takes ~6 us, HBM ~1 us)
constexpr int FDN_RS = 72;                      // row stride (floats): 4 lead + 3 shift + 64 samples, 16-byte multiple
constexpr int FDN_ROWS = 32 * FDN_RS;           // one stage
__host__ __device__ constexpr int fdn_warp_floats(int nst) { return nst * FDN_ROWS + nst * 128 + 128 + nst * 64 + 32 + 128; }
// per warp: stages | dbuf [NST][2][64] | wtab [32][4] (w0 w1 w2 lw) | tb2 [NST][32][2] (rw, row offset) | vcarry [32] | geo [32][4] (idx, len, lp, off)
constexpr int FDN_WARP_FLOATS = fdn_warp_floats(FDN_NST_DEFAULT);

FDSP_DEV uint32_t fdn_smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
FDSP_DEV void fdn_cp16(uint32_t dst, const void* src) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory"); }
FDSP_DEV void fdn_cp4(uint32_t dst, const void* src) { asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory"); }
FDSP_DEV void fdn_cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> FDSP_DEV void fdn_cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// blockDim.x = 32 * W (W voices per CTA), dynamic smem = W * FDN_WARP_FLOATS * 4 bytes
template <int FDN_NST>
__global__ void __launch_bounds__(320) fdn_kernel(const FdnArgs a) {
  constexpr int FDN_WARP_FLOATS = fdn_warp_floats(FDN_NST);
  extern __shared__ __align__(16) float fdn_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
  const uint32_t v = blockIdx.x * W + warp;
  const bool active = v < a.V;
  float* sm = fdn_smem + (size_t)warp * FDN_WARP_FLOATS;
  float* rbuf = sm;                                   // [NST][32][RS] ring slices; new samples are produced in place (slots 0..63 of a row)
  float* dbuf = rbuf + FDN_NST * FDN_ROWS;            // [NST][2][64] stereo input of the blocks in flight
  float4* wtab = reinterpret_cast<float4*>(dbuf + FDN_NST * 128);   // [32] (w0, w1, w2, lw)
  float2* tb2 = reinterpret_cast<float2*>(reinterpret_cast<float*>(wtab) + 128);   // [NST][32] (rw, float offset of d[0] of the line inside the stage)
  float* vcarry = reinterpret_cast<float*>(tb2) + FDN_NST * 64;      // [32] Feedback value entering the next block
  uint4* geo = reinterpret_cast<uint4*>(vcarry + 32);  // [32] (write position, length, physical length, ring offset) of every line, for the lanes that sweep (line, chunk)

  // ---- lane = line bookkeeping: ring geometry, write position, FIR shift register
  float f0 = 0, f1 = 0, f2 = 0, c0 = 0, c1 = 0, scalar = 1.0f;
  uint32_t idx = 0, len = 193, lp = 256, off = 0;
  if (active) {
    const uint32_t V = a.V;
    auto P = [&](uint32_t row) { return __uint_as_float(__ldg(a.params + (size_t)row * V + v)); };
    auto S = [&](uint32_t row) { return a.state[(size_t)row * V + v]; };
    wtab[lane] = make_float4(P(a.p0 + 3 * lane), P(a.p0 + 3 * lane + 1), P(a.p0 + 3 * lane + 2), P(a.p0 + 96 + 2 * lane));
    const float rw = P(a.p0 + 96 + 2 * lane + 1);
    for (int s = 0; s < FDN_NST; s++) tb2[s * 32 + lane] = make_float2(rw, 0.0f);
    c0 = P(a.p0 + 160); c1 = P(a.p0 + 161);
    if (a.scalar_row >= 0) scalar = P((uint32_t)a.scalar_row);
    vcarry[lane] = __uint_as_float(S(a.s0 + lane));
    idx = S(a.s0 + 32 + 4 * lane);
    f0 = __uint_as_float(S(a.s0 + 32 + 4 * lane + 1)); f1 = __uint_as_float(S(a.s0 + 32 + 4 * lane + 2)); f2 = __uint_as_float(S(a.s0 + 32 + 4 * lane + 3));
    len = __ldg(a.uniform + a.u0 + lane);
    lp = fdn_ring_phys(len);
    uint32_t incl = lp;  // inclusive scan over lanes -> ring offset of each line
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += y; }
    off = incl - lp;
    geo[lane] = make_uint4(idx, len, lp, off);
  }
  __syncwarp();
  float* const vring = active ? a.ring + (size_t)v * a.ring_voice_stride : nullptr;
  const float* dry = active ? a.dry + (size_t)v * a.dry_voice_stride + a.dry_offset : nullptr;
  const uint32_t rb0 = fdn_smem_addr(rbuf);

  // stage the slices of the block that starts `adv` samples after the current write positions: per line an aligned superset of
  // 17 x 16 bytes lands at float 4 of the row (d[t] of the block is row[4 + sh + t]); lanes sweep (line, chunk), 17 passes
  const uint32_t db0 = fdn_smem_addr(dbuf);
  auto prefetch = [&](int st, uint32_t t0, int nb, uint32_t adv) {
    if (active && nb > 0) {
      // half a warp per line: lanes 0-15 fetch chunks 0..15 of line 2i, lanes 16-31 those of line 2i + 1 (256 contiguous bytes each);
      // the 17th chunk of every line (needed whenever the slice starts off a 16-byte boundary) goes in one extra pass, lane = line
      const uint32_t nch = ((uint32_t)nb + 3u + 3u) >> 2;    // 16-byte chunks that cover shift + nb floats for any shift (17 for a full block)
      const uint32_t hl = (uint32_t)lane >> 4, k = (uint32_t)lane & 15u;
#pragma unroll 4
      for (uint32_t i = 0; i < 16u; i++) {
        const uint32_t l = 2u * i + hl;
        const uint4 g = geo[l];                               // (idx, len, lp, off)
        uint32_t rs = g.x + adv + g.z - (g.y - 1u);           // read start = write position - (L - 1)
        rs -= (rs >= g.z) ? g.z : 0u; rs -= (rs >= g.z) ? g.z : 0u;
        uint32_t pos = (rs & ~3u) + 4u * k;
        pos -= (pos >= g.z) ? g.z : 0u;                       // lp is a multiple of 4: a chunk never straddles the end
        if (k < nch) fdn_cp16(rb0 + 4u * (uint32_t)(st * FDN_ROWS + (int)l * FDN_RS + 4 + 4 * (int)k), vring + g.w + pos);
      }
      {
        uint32_t rs = idx + adv + lp - (len - 1u);            // lane = line: this lane's own registers
        rs -= (rs >= lp) ? lp : 0u; rs -= (rs >= lp) ? lp : 0u;
        uint32_t pos = (rs & ~3u) + 64u;
        pos -= (pos >= lp) ? lp : 0u;
        if (nch > 16u) fdn_cp16(rb0 + 4u * (uint32_t)(st * FDN_ROWS + lane * FDN_RS + 4 + 64), vring + off + pos);
        tb2[st * 32 + lane].y = __int_as_float(lane * FDN_RS + 4 + (int)(rs & 3u));
      }
      // stereo input of that block (lanes sweep time; any alignment)
#pragma unroll
      for (int q = 0; q < 2; q++) {
        const int t = lane + 32 * q;
        if (t < nb) {
          fdn_cp4(db0 + 4u * (uint32_t)(st * 128 + t), dry + t0 + t);
          fdn_cp4(db0 + 4u * (uint32_t)(st * 128 + 64 + t), dry + a.dry_ch_stride + t0 + t);
        }
      }
    }
    fdn_cp_commit();   // one group per call, empty or not: the wait below counts groups
  };

  const float hz = (float)(1.0 / sqrt(32.0));
  const uint32_t nblk = (a.n + 63u) / 64u;
  auto blen = [&](uint32_t b) { return b < nblk ? (int)((a.n - b * 64u) < 64u ? (a.n - b * 64u) : 64u) : 0; };
  prefetch(0, 0u, blen(0), 0u);
  if (FDN_NST == 3) prefetch(1, 64u, blen(1), 64u);
#pragma unroll 1
  for (uint32_t b = 0; b < nblk; b++) {
    const int st = (int)(b % FDN_NST);
    const uint32_t t0 = b * 64u;
    const int nb = blen(b);
    // the other stage held block b - 1: its rows went back to the rings before the __syncwarp that ended the last iteration. What block
    // b + 1 reads was written at least a whole block ago (every delay >= 192 samples), in program order before this point.
    if (FDN_NST == 2) prefetch((int)((b + 1) % FDN_NST), t0 + 64u, blen(b + 1), (uint32_t)nb);
    fdn_cp_wait<1>();   // all but the newest group: block b has landed (this lane's copies; the __syncwarp below publishes the others')
    __syncwarp();
    if (active) {
      float* rst = rbuf + st * FDN_ROWS;
      const float* db = dbuf + st * 128;
      {  // lane = line: FIR history in front of d[0], and the first new sample (input + the Feedback value carried over)
        const int ro = __float_as_int(tb2[st * 32 + lane].y);
        rst[ro - 2] = f1; rst[ro - 1] = f2;
        rst[lane * FDN_RS] = db[(lane & 1) * 64] + vcarry[lane];   // MultiSplit<2,16>: line l reads input channel l % 2
      }
      __syncwarp();
      const float2* t2 = tb2 + st * 32;
      if (nb == 64 && !(a.flags & 1u)) {
        // full block: lane t evaluates samples t and t + 32 in ONE pass — the per-line weights are loaded once for both, and two independent
        // chains per lane keep the FP32 pipe fed. All taps of the block are read before any new sample is stored.
        float a0[32], a1[32], sl0 = 0.0f, sr0 = 0.0f, sl1 = 0.0f, sr1 = 0.0f;
#pragma unroll
        for (int l = 0; l < 32; l++) {
          const float4 wv = wtab[l];
          const float2 q = t2[l];
          const float* row = rst + __float_as_int(q.y) + lane;
          const float o0 = (wv.x * row[-2] + wv.y * row[-1]) + wv.z * row[0];      // Fir<U3>: accumulate in tap order from the oldest
          const float o1 = (wv.x * row[30] + wv.y * row[31]) + wv.z * row[32];
          a0[l] = o0; a1[l] = o1;
          if (l == 0) { sl0 = o0 * wv.w; sr0 = o0 * q.x; sl1 = o1 * wv.w; sr1 = o1 * q.x; }   // Reduce<U32, Panner, FrameAdd>: left fold
          else { sl0 += o0 * wv.w; sr0 += o0 * q.x; sl1 += o1 * wv.w; sr1 += o1 * q.x; }
        }
        // FrameHadamard<U32> (src/feedback.rs:35-57): in-place butterflies h = 1, 2, 4, 8, 16, then * (1 / sqrt(32)) as f32
#pragma unroll
        for (int h = 1; h < 32; h <<= 1) {
#pragma unroll
          for (int i = 0; i < 32; i += 2 * h) {
#pragma unroll
            for (int j = i; j < i + h; j++) {
              const float x0 = a0[j], y0 = a0[j + h]; a0[j] = x0 + y0; a0[j + h] = x0 - y0;
              const float x1 = a1[j], y1 = a1[j + h]; a1[j] = x1 + y1; a1[j + h] = x1 - y1;
            }
          }
        }
        const float xa0 = db[lane + 1], xb0 = db[64 + lane + 1];                                      // input of sample t + 1
        const float xa1 = db[lane + 33 < 64 ? lane + 33 : 63], xb1 = db[64 + (lane + 33 < 64 ? lane + 33 : 63)];
        sl0 = sl0 * c0; sr0 = sr0 * c1; sl1 = sl1 * c0; sr1 = sr1 * c1;
        if (a.scalar_row >= 0) {
          sl0 = db[lane] + sl0 * scalar; sr0 = db[64 + lane] + sr0 * scalar;
          sl1 = db[lane + 32] + sl1 * scalar; sr1 = db[64 + lane + 32] + sr1 * scalar;
        }
        __syncwarp();   // every lane has read its taps: the rows may now take the new samples
#pragma unroll
        for (int l = 0; l < 32; l++) rst[l * FDN_RS + lane + 1] = ((l & 1) ? xb0 : xa0) + a0[l] * hz;   // Feedback: x.tick(input + value); Delay stores it
        if (lane < 31) {
#pragma unroll
          for (int l = 0; l < 32; l++) rst[l * FDN_RS + lane + 33] = ((l & 1) ? xb1 : xa1) + a1[l] * hz;
        } else {
#pragma unroll
          for (int l = 0; l < 32; l++) vcarry[l] = a1[l] * hz;    // enters the first sample of the next block
        }
        if (a.partial) {   // per-voice rows of the mix-down [V][2][n]: mix_reduce_kernel adds them in voice order
          float* pr = a.partial + ((size_t)v * 2) * a.n + t0 + lane;
          pr[0] = sl0; pr[32] = sl1; pr[a.n] = sr0; pr[a.n + 32] = sr1;
        }
        if (a.out) {
          float* orow = a.out + (size_t)__ldg(a.row_map + v) * a.out_stride + a.out_offset + t0 + lane;
          orow[0] = sl0; orow[32] = sl1; orow[a.out_stride] = sr0; orow[a.out_stride + 32] = sr1;
        }
      } else {
#pragma unroll 1
      for (int h0 = 0; h0 < nb; h0 += 32) {
        const int t = h0 + lane;
        const bool ok = t < nb;
        const int tc = ok ? t : 0;
        float av[32], sl = 0.0f, sr = 0.0f;
#pragma unroll
        for (int l = 0; l < 32; l++) {
          const float4 wv = wtab[l];
          const float2 q = t2[l];
          const float* row = rst + __float_as_int(q.y) + tc;
          const float o = (wv.x * row[-2] + wv.y * row[-1]) + wv.z * row[0];     // Fir<U3>: accumulate in tap order from the oldest
          av[l] = o;
          if (l == 0) { sl = o * wv.w; sr = o * q.x; } else { sl += o * wv.w; sr += o * q.x; }   // Reduce<U32, Panner, FrameAdd>: left fold
        }
        // FrameHadamard<U32> (src/feedback.rs:35-57): in-place butterflies h = 1, 2, 4, 8, 16, then * (1 / sqrt(32)) as f32
#pragma unroll
        for (int h = 1; h < 32; h <<= 1) {
#pragma unroll
          for (int i = 0; i < 32; i += 2 * h) {
#pragma unroll
            for (int j = i; j < i + h; j++) { const float x = av[j], y = av[j + h]; av[j] = x + y; av[j + h] = x - y; }
          }
        }
        const float x0n = db[tc + 1 < 64 ? tc + 1 : 63], x1n = db[64 + (tc + 1 < 64 ? tc + 1 : 63)];   // input of sample t + 1
        sl = sl * c0; sr = sr * c1;
        if (a.scalar_row >= 0) { sl = db[tc] + sl * scalar; sr = db[64 + tc] + sr * scalar; }
        __syncwarp();   // every lane has read its taps of this half: the rows may now take the new samples (slots <= h0 + 32 < first tap of the next half)
        if (ok) {
          if (t + 1 < nb) {
#pragma unroll
            for (int l = 0; l < 32; l++) rst[l * FDN_RS + t + 1] = ((l & 1) ? x1n : x0n) + av[l] * hz;   // Feedback: x.tick(input + value); Delay stores it
          } else {
#pragma unroll
            for (int l = 0; l < 32; l++) vcarry[l] = av[l] * hz;    // enters the first sample of the next block
          }
          if (a.partial) {   // per-voice rows of the mix-down [V][2][n]: mix_reduce_kernel adds them in voice order
            a.partial[((size_t)v * 2) * a.n + t0 + t] = sl; a.partial[((size_t)v * 2 + 1) * a.n + t0 + t] = sr;
          }
          if (a.out) {
            float* orow = a.out + (size_t)__ldg(a.row_map + v) * a.out_stride + a.out_offset + t0 + t;
            orow[0] = sl; orow[a.out_stride] = sr;
          }
        }
      }
      }
      // lane = line again: FIR history for the next block, then the new samples of the line go back to its ring
      {
        const int ro = __float_as_int(tb2[st * 32 + lane].y);
        if (nb >= 3) { f0 = rst[ro + nb - 3]; f1 = rst[ro + nb - 2]; f2 = rst[ro + nb - 1]; }
        else { for (int i = 0; i < nb; i++) { f0 = f1; f1 = f2; f2 = rst[ro + i]; } }
      }
      __syncwarp();
      const bool vec_ok = __all_sync(0xffffffffu, ((idx | (uint32_t)nb) & 3u) == 0u);
      if (vec_ok) {
        // 16-byte stores: lanes sweep (line, chunk of 4 samples); a chunk never straddles the ring end (positions and lp are multiples of 4)
        const uint32_t nch = (uint32_t)nb >> 2;                  // <= 16: half a warp per line, as in the prefetch
        const uint32_t hl = (uint32_t)lane >> 4, k = (uint32_t)lane & 15u;
#pragma unroll 4
        for (uint32_t i = 0; i < 16u; i++) {
          const uint32_t l = 2u * i + hl;
          const uint4 g = geo[l];
          uint32_t pos = g.x + 4u * k; pos -= (pos >= g.z) ? g.z : 0u;
          if (k < nch) *reinterpret_cast<float4*>(vring + g.w + pos) = *reinterpret_cast<const float4*>(rst + l * FDN_RS + 4 * k);
        }
      } else {
        // ragged positions: lanes sweep time, lines are looped (coalesced rows)
#pragma unroll 1
        for (int l = 0; l < 32; l++) {
          const uint4 g = geo[l];
#pragma unroll
          for (int q = 0; q < 2; q++) {
            const int t = lane + 32 * q;
            if (t < nb) { uint32_t pos = g.x + (uint32_t)t; pos -= (pos >= g.z) ? g.z : 0u; vring[g.w + pos] = rst[l * FDN_RS + t]; }
          }
        }
      }
      __syncwarp();   // geo is read by every lane above and advanced by its owner below
      idx += (uint32_t)nb; idx -= (idx >= lp) ? lp : 0u;
      geo[lane].x = idx;
      __syncwarp();
    }
    if (FDN_NST == 3) prefetch((int)((b + 2) % FDN_NST), t0 + 128u, blen(b + 2), 64u);   // (diagnostic three-stage form: distance 2, issued after the block)
  }
  fdn_cp_wait<0>();
  if (active) {
    const uint32_t V = a.V;
    __syncwarp();
    a.state[(size_t)(a.s0 + lane) * V + v] = __float_as_uint(vcarry[lane]);
    a.state[(size_t)(a.s0 + 32 + 4 * lane) * V + v] = idx;
    a.state[(size_t)(a.s0 + 32 + 4 * lane + 1) * V + v] = __float_as_uint(f0);
    a.state[(size_t)(a.s0 + 32 + 4 * lane + 2) * V + v] = __float_as_uint(f1);
    a.state[(size_t)(a.s0 + 32 + 4 * lane + 3) * V + v] = __float_as_uint(f2);
  }
}

}  // namespace fdsp
