// Resident form of the voice-bank kernel for the `AudioUnit::process` call pattern (reference src/audiounit.rs:45, driven one 64-sample
// block at a time by Wave::render src/wave.rs:452-462 or an audio callback): instead of one launch per block — parameters and state
// reloaded, 161 KB of wavetables restaged, a launch and a stream synchronisation on the critical path — ONE launch stays resident with every voice's state in registers and serves blocks on a doorbell:
//
//   host: writes the block's inputs and size into a mapped, pinned control page, then the request's sequence number (the doorbell);
//         spins on `done` in the same page; copies the mix out.
//   GPU : thread 0 of CTA 0 polls the doorbell over PCIe and relays it to a word in device memory that the other CTAs poll; every CTA
//         evaluates the block exactly like bank_kernel (same group structure, tail, CTA mix); the last CTA to finish folds the partial
//         mixes in CTA order into the control page and publishes `done`.
// The kernel leaves by itself when asked (`RT_QUIT`) or after about a second without a request, saving the state words, so any other
// call on the bank simply stops it first (csrc/host/bank.cpp `rt_stop`). All CTAs must be co-resident: the host only uses this form
// for single-class banks whose grid fits the GPU in one wave. Results are bit-identical to process() through the one-launch-per-block path.
#pragma once
#include "bank_kernel.cuh"
#include "rt_args.h"

namespace fdsp {

FDSP_DEV uint32_t rt_ld_sys(const volatile uint32_t* p) { uint32_t v; asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }

template <class G, int NT, bool TB>
__global__ void __launch_bounds__(NT, FDSP_MIN_CTAS) bank_kernel_rt(const BankArgs a, const RtArgs rt) {
  extern __shared__ __align__(16) float tile[];  // [OUT][TS][NT+1]; TB: table data after it
  __shared__ uint32_t s_cmd, s_n, s_last;
  __shared__ float s_in[(G::IN > 0 ? G::IN : 1) * 64];   // the block's shared inputs: fetched from the control page once per CTA, not once per voice
  const uint32_t tid = threadIdx.x;
  const uint32_t vpc = a.vpc ? a.vpc : (uint32_t)NT;
  const uint32_t v = blockIdx.x * vpc + tid;
  const bool active = tid < vpc && v < a.V;
  constexpr int IN = G::IN, OUT = G::OUT;
  constexpr int TS = mix_tile_samples(OUT);
  constexpr bool GROUP = GroupPlan<G>::ok && GroupPlan<G>::code <= FDSP_GROUP_COST && !FDSP_NO_GROUP;
  constexpr int UNROLL = GROUP ? 8 : (Cost<G>::value <= 160 ? 8 : (Cost<G>::value <= 320 ? 4 : (Cost<G>::value <= 640 ? 2 : 1)));
  typename G::R r;
  CtxT<TB> c;
  c.tsm = 0u; c.tsm_kind = -1;
  if (TB) {
    constexpr int KIND = WaveKind<G>::value >= 0 ? WaveKind<G>::value : 0;
    __shared__ __align__(8) unsigned long long mbar;
    float* tsm = tile + mix_tile_floats(OUT, NT);
    const uint32_t bytes = (uint32_t)a.wt[KIND].total * 4u;
    const uint32_t bar = smem_addr(&mbar);
    if (tid == 0) mbar_init(bar, 1);
    __syncthreads();
    if (tid == 0) {
      mbar_expect_tx(bar, bytes);
      const char* src = reinterpret_cast<const char*>(a.wt[KIND].data);
      for (uint32_t o = 0; o < bytes; o += 32768u) bulk_g2s(smem_addr(tsm) + o, src + o, (bytes - o) < 32768u ? (bytes - o) : 32768u, bar);
    }
    mbar_wait(bar, 0);
    c.tsm = smem_addr(tsm); c.tsm_kind = KIND;
  }
  c.wt = a.wt; c.dl = a.dline; c.V = a.V; c.v = v; c.sr = a.sr; c.sd64 = a.sd64; c.sd32 = a.sd32;
  c.rp = a.params; c.rs0 = a.state0; c.ru = a.uniform; c.dl_total = a.dl_floats;
  if (active) {
    Loader l{a.params, a.state, a.uniform, a.V, v, 0u, 0u, 0u, 0u};
    G::load(r, l);
  } else {
    for (int e = 0; e < OUT * TS; e++) tile[e * (NT + 1) + tid] = 0.0f;  // columns of absent voices stay zero
  }
  uint32_t seq = rt.first_seq - 1u;
#pragma unroll 1
  for (;;) {
    // ---- wait for the next request
    if (tid == 0) {
      uint32_t cur = seq, spins = 0;
      if (blockIdx.x == 0) {
        do { cur = rt_ld_sys(&rt.ctl->doorbell); } while (cur == seq && ++spins < RT_POLL_LIMIT_HOST);
        if (cur == seq) cur = RT_QUIT;                                   // idle: leave (the host restarts the kernel with the next block)
        const uint32_t n = cur == RT_QUIT ? 0u : rt_ld_sys(&rt.ctl->size);
        rt.relay[1] = n;
        __threadfence();
        *reinterpret_cast<volatile uint32_t*>(rt.relay) = cur;
        s_n = n;
      } else {
        do { cur = rt_ld_sys(rt.relay); } while (cur == seq && ++spins < RT_POLL_LIMIT_RELAY);
        if (cur == seq) cur = RT_QUIT;
        __threadfence();
        s_n = rt_ld_sys(rt.relay + 1);
      }
      s_cmd = cur;
    }
    __syncthreads();
    const uint32_t cmd = s_cmd;
    const int nb = (int)s_n;
    if (cmd == RT_QUIT) break;
    seq = cmd;
    for (int e = (int)tid; e < IN * 64; e += NT) s_in[e] = (e & 63) < nb ? __ldcv(&rt.ctl->in[e >> 6][e & 63]) : 0.0f;
    __syncthreads();
    // ---- one block, as bank_kernel evaluates it (MODE 2)
    const int nfull = nb & ~7;
    c.n = nb;
#pragma unroll 1
    for (int s0 = 0; s0 < nb; s0 += TS) {
      const int s1 = (s0 + TS) < nb ? (s0 + TS) : nb;
      if (active) {
        const int gend = s1 < nfull ? s1 : nfull;
        c.rem = false;
#pragma unroll 1
        for (int g = s0; g < gend; g += 8) {
          if constexpr (GROUP) {
            Fr8<IN> in8; Fr8<OUT> o8;
#pragma unroll
            for (int k = 0; k < IN; k++) {
#pragma unroll
              for (int j = 0; j < 8; j++) in8.v[k][j] = s_in[k * 64 + g + j];
            }
            c.i = g; c.first = true;
            group_step<G>(r, c, in8, o8);
#pragma unroll
            for (int k = 0; k < OUT; k++) {
#pragma unroll
              for (int j = 0; j < 8; j++) tile[(k * TS + (g - s0) + j) * (NT + 1) + tid] = o8.v[k][j];
            }
          } else {
#pragma unroll(UNROLL)
            for (int j = 0; j < 8; j++) {
              Fr<IN> in; Fr<OUT> o;
#pragma unroll
              for (int k = 0; k < IN; k++) in.v[k] = s_in[k * 64 + g + j];
              c.i = g + j; c.first = (j == 0);
              G::template step<false>(r, c, in, o);
#pragma unroll
              for (int k = 0; k < OUT; k++) tile[(k * TS + (g - s0) + j) * (NT + 1) + tid] = o.v[k];
            }
          }
        }
        if (s1 == nb) {  // end of the block: wrap up the SIMD part, then the (size & 7) tail through the tick path
          G::end_simd(r);
          c.rem = true; c.first = false;
#pragma unroll 1
          for (int i = nfull; i < nb; i++) {
            Fr<IN> in; Fr<OUT> o;
#pragma unroll
            for (int k = 0; k < IN; k++) in.v[k] = s_in[k * 64 + i];
            c.i = i;
            G::template step<false>(r, c, in, o);
#pragma unroll
            for (int k = 0; k < OUT; k++) tile[(k * TS + (i - s0)) * (NT + 1) + tid] = o.v[k];
          }
        }
      }
      // CTA partial mix: the association of bank_kernel (two threads per row, four interleaved accumulators each, low half + high half)
      __syncthreads();
      constexpr int HALF = NT / 2, QN = HALF / 4, ROWS = OUT * TS;
      const int h = (int)(tid & 1u);
      const int c0 = h * HALF + (h * QN) % HALF, c1 = h * HALF + (QN + h * QN) % HALF, c2 = h * HALF + (2 * QN + h * QN) % HALF, c3 = h * HALF + (3 * QN + h * QN) % HALF;
#pragma unroll 1
      for (int eb = (int)(tid >> 5) * 16; eb < ROWS; eb += HALF) {
        const int e = eb + (int)((tid & 31u) >> 1);
        const bool ok = e < ROWS;
        const int k = e / TS, i = e - k * TS;
        const float* row = tile + (ok ? e : 0) * (NT + 1);
        float a0 = row[c0], a1 = row[c1], a2 = row[c2], a3 = row[c3];
#pragma unroll
        for (int q = 1; q < QN; q++) { a0 += row[c0 + q]; a1 += row[c1 + q]; a2 += row[c2 + q]; a3 += row[c3 + q]; }
        const float s = (a0 + a1) + (a2 + a3);
        const float other = __shfl_xor_sync(0xffffffffu, s, 1);
        if (ok && h == 0 && s0 + i < s1) a.partial[((size_t)blockIdx.x * OUT + k) * 64 + s0 + i] = s + other;
      }
      __syncthreads();
    }
    // ---- the last CTA to finish folds the partials in CTA order (= mix_reduce_kernel) into the control page and publishes `done`
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(a.ticket, 1u) == gridDim.x - 1u) ? 1u : 0u;
    __syncthreads();
    if (s_last) {
      __threadfence();
      // CTA-order left fold of the partials (= mix_reduce_kernel, bit for bit). The loads of 8 CTAs are issued together, the adds stay in
      // order. (A version that staged the partials in shared memory first was slower: one CTA cannot keep enough loads in flight to win
      // back the extra pass.)
      for (uint32_t e = tid; e < (uint32_t)OUT * (uint32_t)nb; e += NT) {
        const uint32_t ch = e / (uint32_t)nb, t = e - ch * (uint32_t)nb;
        const float* p0 = a.partial + (size_t)ch * 64 + t;
        float s = __ldcg(p0);
        uint32_t b = 1;
        for (; b + 8 <= gridDim.x; b += 8) {
          float x[8];
#pragma unroll
          for (int u = 0; u < 8; u++) x[u] = __ldcg(p0 + (size_t)(b + u) * OUT * 64);
#pragma unroll
          for (int u = 0; u < 8; u++) s += x[u];
        }
        for (; b < gridDim.x; b++) s += __ldcg(p0 + (size_t)b * OUT * 64);
        rt.ctl->out[ch][t] = s;
      }
      __threadfence_system();
      __syncthreads();
      if (tid == 0) { *a.ticket = 0u; __threadfence(); rt.ctl->done = seq; }
    }
  }
  if (active) {
    Saver s{a.state, a.V, v, 0u};
    G::save(r, s);
  }
  __threadfence();
  __syncthreads();
  if (tid == 0 && atomicAdd(rt.relay + 2, 1u) == gridDim.x - 1u) { rt.relay[2] = 0u; __threadfence_system(); rt.ctl->done = RT_EXITED; }
}

}  // namespace fdsp
