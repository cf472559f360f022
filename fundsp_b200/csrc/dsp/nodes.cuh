// fundsp_b200 device node library: the leaf DSP nodes and structural combinators of the reference's
// hot path (SURVEY.md §8a) as C++ templates that compose into ONE fused per-voice program.
//
// A graph type such as  Pipe<Pipe<Constant<1>,WaveSynth<0,1>>,FixedSvf>  is the device-side analogue of the
// reference's monomorphised `An<Pipe<Pipe<Constant<U1>,WaveSynth<U1>>,FixedSvf<f32,LowpassMode>>>`.
// One thread evaluates one voice: parameters and state live in registers (`R`), per-sample `step`
// carries the recurrences, and the *block* semantics of the reference's `process` path (phase wrap once
// per 64-block, table choice once per 8 samples, tail samples through `tick`, envelope run lengths) are
// reproduced through the block context `Ctx` — see each node's reference citation.
//
// Word layout contract with the host lowering (csrc/host/lower.cpp): per-voice parameter words (P),
// per-voice state words (S) and class-uniform words (U) are consumed in depth-first, left-to-right
// order; `NP/NS/NU` are the totals the host checks against.
#pragma once
#include "libm.cuh"
#include "libm64.cuh"
#include "bank_args.h"

namespace fdsp {



template <int N> struct Fr { float v[N > 0 ? N : 1]; };
// Eight consecutive samples of N channels (channel-major): the device analogue of the reference's f32x8 lane group
// (src/buffer.rs: channel c, sample i lives at slice[(c << 3) + (i >> 3)][i & 7]).
template <int N> struct Fr8 { float v[N > 0 ? N : 1][8]; };

// Block context. `first`: first lane of an 8-sample SIMD group; `rem`: sample belongs to the tail
// (size & 7) that the reference runs through `tick` (src/audionode.rs:110-126); `i`/`n`: index / size of block.
// SM: the wavetables of one waveform kind are staged in shared memory (TMA bulk copy in the kernel prologue).
template <bool SM, bool UH = false> struct CtxT {
  static constexpr bool SMEM_TABLES = SM;
  static constexpr bool UNROLL_HEAVY = UH;   // heavy serial leaves run their 8 steps fully unrolled (the stage-pipelined kernel gives them a warp of their own)
  const WaveTableDev* wt;
  uint32_t tsm;       // shared-space byte address of the staged table data (kind `tsm_kind`)
  int tsm_kind;
  float* dl;          // delay-line storage of this voice class, element (off + pos) * V + v
  uint32_t V, v;
  // what a node needs to put a sub-program back into its construction-time state on the device (Event<X> in a looping sequencer): the class's
  // parameter / reset-image / uniform words and the delay-line floats per voice
  const uint32_t* rp; const uint32_t* rs0; const uint32_t* ru; uint32_t dl_total;
  float sr;           // sample rate as f32
  float sd64;         // (1.0f64 / sr) as f32   (src/oscillator.rs:62-64, src/envelope.rs:290-292)
  float sd32;         // 1.0f32 / (sr as f32)   (src/wavetable.rs:299-302)
  int i, n;
  bool first, rem;
};
typedef CtxT<false> Ctx;

#ifndef FDSP_LDS_VOLATILE
#define FDSP_LDS_VOLATILE 0
#endif
FDSP_DEV float lds_f32(uint32_t addr) {
#ifdef FDSP_HOST_EMUL
  (void)addr; return 0.0f;   // the host emulation never stages tables in shared memory
#else
  float v;
  if (FDSP_LDS_VOLATILE) asm volatile("ld.volatile.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  else asm("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
#endif
}

struct Loader {
  const uint32_t* p; const uint32_t* s; const uint32_t* u; uint32_t V, v;
  uint32_t pi, si, ui, dl;
  FDSP_DEV uint32_t P() { return __ldg(p + (size_t)(pi++) * V + v); }
  FDSP_DEV float Pf() { return __uint_as_float(P()); }
  FDSP_DEV uint32_t S() { return s[(size_t)(si++) * V + v]; }
  FDSP_DEV float Sf() { return __uint_as_float(S()); }
  FDSP_DEV uint32_t U() { return __ldg(u + (ui++)); }
  FDSP_DEV uint32_t D(uint32_t len) { uint32_t o = dl; dl += len; return o; }
};
struct Saver {
  uint32_t* s; uint32_t V, v; uint32_t si;
  FDSP_DEV void S(uint32_t w) { s[(size_t)(si++) * V + v] = w; }
  FDSP_DEV void Sf(float f) { S(__float_as_uint(f)); }
};

#define FDSP_NODE(in_, out_, np_, ns_, nu_) \
  static constexpr int IN = (in_), OUT = (out_), NP = (np_), NS = (ns_), NU = (nu_)

struct Empty {};

// ---------------------------------------------------------------- 8-sample group evaluation
// The block path of the reference evaluates node by node over f32x8 groups, not sample by sample; nodes only interact
// through their buffers, so evaluating X over 8 samples and then Y over the same 8 is exact. On the GPU this is what
// gives one thread instruction-level parallelism: a voice is a serial recurrence, there are fewer voice-warps than
// warp schedulers, so the 8 independent oscillator/table evaluations of a group have to overlap inside one thread.
// A node opts in with `typedef void GroupStep;` + `step8`; everything else runs its per-sample `step` 8 times.
template <class T> struct VoidT { typedef void type; };
template <class Node, class = void> struct HasGroup { static constexpr bool value = false; };
template <class Node> struct HasGroup<Node, typename VoidT<typename Node::GroupStep>::type> { static constexpr bool value = true; };
// `typedef void SteadyGroup;` + `steady8` / `step8_steady`: a heavy leaf whose per-sample "input changed" test can be decided for the whole group
template <class Node, class = void> struct HasSteady { static constexpr bool value = false; };
template <class Node> struct HasSteady<Node, typename VoidT<typename Node::SteadyGroup>::type> { static constexpr bool value = true; };

#ifndef FDSP_ROTATE_COST
#define FDSP_ROTATE_COST 100   // leaves above this static cost are not unrolled over the group (their loop rotates the registers)
#endif
template <class G> struct Cost;   // static per-sample cost estimate of a program (defined with the traits below)

template <class Node, class C> FDSP_DEV void group_step(typename Node::R& r, C& c, const Fr8<Node::IN>& in, Fr8<Node::OUT>& o) {
  if constexpr (HasGroup<Node>::value) {
    Node::step8(r, c, in, o);
  } else if constexpr ((Cost<Node>::value > FDSP_ROTATE_COST) && !C::UNROLL_HEAVY) {
    // Heavy serial leaf (Moog, Rez, Dsf ...): unrolling it 8x only bloats the instruction stream, so its 8 steps run in a real
    // loop. The group registers are ROTATED by one sample per iteration, which keeps every array index static (no local memory).
    Fr8<Node::IN> ri = in;
    Fr8<Node::OUT> ro;
#pragma unroll
    for (int k = 0; k < Node::OUT; k++) {
#pragma unroll
      for (int q = 0; q < 8; q++) ro.v[k][q] = 0.0f;
    }
    const int base = c.i;
#pragma unroll 1
    for (int j = 0; j < 8; j++) {
      Fr<Node::IN> a; Fr<Node::OUT> b;
#pragma unroll
      for (int k = 0; k < Node::IN; k++) a.v[k] = ri.v[k][0];
      c.i = base + j; c.first = (j == 0);
      Node::template step<false>(r, c, a, b);
#pragma unroll
      for (int k = 0; k < Node::IN; k++) {
#pragma unroll
        for (int q = 0; q < 7; q++) ri.v[k][q] = ri.v[k][q + 1];
      }
#pragma unroll
      for (int k = 0; k < Node::OUT; k++) {
#pragma unroll
        for (int q = 0; q < 7; q++) ro.v[k][q] = ro.v[k][q + 1];
        ro.v[k][7] = b.v[k];
      }
    }
    o = ro;
    c.i = base; c.first = true;
  } else {
    if constexpr (HasSteady<Node>::value && C::UNROLL_HEAVY) {
      if (Node::steady8(r, in)) { Node::step8_steady(r, in, o); return; }
    }
    const int base = c.i;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      Fr<Node::IN> a; Fr<Node::OUT> b;
#pragma unroll
      for (int k = 0; k < Node::IN; k++) a.v[k] = in.v[k][j];
      c.i = base + j; c.first = (j == 0);
      Node::template step<false>(r, c, a, b);
#pragma unroll
      for (int k = 0; k < Node::OUT; k++) o.v[k][j] = b.v[k];
    }
    c.i = base; c.first = true;
  }
}
#define FDSP_G8 _Pragma("unroll") for (int j = 0; j < 8; j++)

// ---------------------------------------------------------------- routing (src/audionode.rs:374-722,2800-2837)
template <int N> struct Constant {  // ID 2
  FDSP_NODE(0, N, N, 0, 0);
  struct R { float v[N]; };
  static FDSP_DEV void load(R& r, Loader& l) { for (int c = 0; c < N; c++) r.v[c] = l.Pf(); }
  static FDSP_DEV void save(const R&, Saver&) {}
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<0>&, Fr<N>& o) { for (int c = 0; c < N; c++) o.v[c] = r.v[c]; }
  static FDSP_DEV void end_simd(R&) {}
};
template <int N> struct MultiPass {  // ID 0 (N-channel) / 48 (Pass)
  FDSP_NODE(N, N, 0, 0, 0);
  typedef Empty R;
  static FDSP_DEV void load(R&, Loader&) {}
  static FDSP_DEV void save(const R&, Saver&) {}
  template <bool T, class C> static FDSP_DEV void step(R&, const C&, const Fr<N>& in, Fr<N>& o) { for (int c = 0; c < N; c++) o.v[c] = in.v[c]; }
  static FDSP_DEV void end_simd(R&) {}
};
template <int N> struct Sink {  // ID 1
  FDSP_NODE(N, 0, 0, 0, 0);
  typedef Empty R;
  static FDSP_DEV void load(R&, Loader&) {}
  static FDSP_DEV void save(const R&, Saver&) {}
  template <bool T, class C> static FDSP_DEV void step(R&, const C&, const Fr<N>&, Fr<0>&) {}
  static FDSP_DEV void end_simd(R&) {}
};
template <int M, int N> struct MultiSplit {  // ID 40 / 38
  FDSP_NODE(M, M * N, 0, 0, 0);
  typedef Empty R;
  static FDSP_DEV void load(R&, Loader&) {}
  static FDSP_DEV void save(const R&, Saver&) {}
  template <bool T, class C> static FDSP_DEV void step(R&, const C&, const Fr<M>& in, Fr<M * N>& o) { for (int c = 0; c < M * N; c++) o.v[c] = in.v[c % M]; }
  static FDSP_DEV void end_simd(R&) {}
};
template <int M, int N> struct MultiJoin {  // ID 41 / 39: tick = add then divide; process = scale by 1/N then add
  FDSP_NODE(M * N, M, 0, 0, 0);
  typedef Empty R;
  static FDSP_DEV void load(R&, Loader&) {}
  static FDSP_DEV void save(const R&, Saver&) {}
  template <bool T, class C> static FDSP_DEV void step(R&, const C&, const Fr<M * N>& in, Fr<M>& o) {
    if (T) {
      for (int j = 0; j < M; j++) { float a = in.v[j]; for (int k = 1; k < N; k++) a += in.v[j + k * M]; o.v[j] = a / (float)N; }
    } else {
      const float z = 1.0f / (float)N;
      for (int j = 0; j < M; j++) o.v[j] = in.v[j] * z;
      for (int c = M; c < M * N; c++) o.v[c % M] += in.v[c] * z;
    }
  }
  static FDSP_DEV void end_simd(R&) {}
};
template <int N> struct Reverse {  // ID 45
  FDSP_NODE(N, N, 0, 0, 0);
  typedef Empty R;
  static FDSP_DEV void load(R&, Loader&) {}
  static FDSP_DEV void save(const R&, Saver&) {}
  template <bool T, class C> static FDSP_DEV void step(R&, const C&, const Fr<N>& in, Fr<N>& o) { for (int c = 0; c < N; c++) o.v[c] = in.v[N - 1 - c]; }
  static FDSP_DEV void end_simd(R&) {}
};

// ---------------------------------------------------------------- combinators (src/audionode.rs:724-2800)
template <int K> FDSP_DEV float binop(float x, float y) { return K == 0 ? x + y : (K == 1 ? x - y : x * y); }

template <int K, class X, class Y> struct Binop {  // ID 3: K 0 add, 1 sub, 2 mul
  FDSP_NODE(X::IN + Y::IN, X::OUT, X::NP + Y::NP, X::NS + Y::NS, X::NU + Y::NU);
  struct R { typename X::R x; typename Y::R y; };
  static FDSP_DEV void load(R& r, Loader& l) { X::load(r.x, l); Y::load(r.y, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { X::save(r.x, s); Y::save(r.y, s); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<IN>& in, Fr<OUT>& o) {
    Fr<X::IN> xi; Fr<Y::IN> yi; Fr<X::OUT> a; Fr<Y::OUT> b;
    for (int k = 0; k < X::IN; k++) xi.v[k] = in.v[k];
    for (int k = 0; k < Y::IN; k++) yi.v[k] = in.v[X::IN + k];
    X::template step<T>(r.x, c, xi, a); Y::template step<T>(r.y, c, yi, b);
    for (int k = 0; k < OUT; k++) o.v[k] = binop<K>(a.v[k], b.v[k]);
  }
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C& c, const Fr8<IN>& in, Fr8<OUT>& o) {
    Fr8<X::IN> xi; Fr8<Y::IN> yi; Fr8<Y::OUT> b;
    for (int k = 0; k < X::IN; k++) FDSP_G8 xi.v[k][j] = in.v[k][j];
    for (int k = 0; k < Y::IN; k++) FDSP_G8 yi.v[k][j] = in.v[X::IN + k][j];
    group_step<X>(r.x, c, xi, o); group_step<Y>(r.y, c, yi, b);
    for (int k = 0; k < OUT; k++) FDSP_G8 o.v[k][j] = binop<K>(o.v[k][j], b.v[k][j]);
  }
  static FDSP_DEV void end_simd(R& r) { X::end_simd(r.x); Y::end_simd(r.y); }
};
template <int K, class X> struct Unop {  // ID 4: K 0 neg, 1 +s, 2 -x+s, 3 *s
  FDSP_NODE(X::IN, X::OUT, X::NP + (K == 0 ? 0 : 1), X::NS, X::NU);
  struct R { float s; typename X::R x; };
  static FDSP_DEV void load(R& r, Loader& l) { r.s = (K == 0) ? 0.0f : l.Pf(); X::load(r.x, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { X::save(r.x, s); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<IN>& in, Fr<OUT>& o) {
    X::template step<T>(r.x, c, in, o);
    for (int k = 0; k < OUT; k++) o.v[k] = K == 0 ? -o.v[k] : (K == 1 ? o.v[k] + r.s : (K == 2 ? -o.v[k] + r.s : o.v[k] * r.s));
  }
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C& c, const Fr8<IN>& in, Fr8<OUT>& o) {
    group_step<X>(r.x, c, in, o);
    for (int k = 0; k < OUT; k++) FDSP_G8 o.v[k][j] = K == 0 ? -o.v[k][j] : (K == 1 ? o.v[k][j] + r.s : (K == 2 ? -o.v[k][j] + r.s : o.v[k][j] * r.s));
  }
  static FDSP_DEV void end_simd(R& r) { X::end_simd(r.x); }
};
template <class X, class Y> struct Pipe {  // ID 6
  FDSP_NODE(X::IN, Y::OUT, X::NP + Y::NP, X::NS + Y::NS, X::NU + Y::NU);
  struct R { typename X::R x; typename Y::R y; };
  static FDSP_DEV void load(R& r, Loader& l) { X::load(r.x, l); Y::load(r.y, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { X::save(r.x, s); Y::save(r.y, s); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<IN>& in, Fr<OUT>& o) {
    Fr<X::OUT> t; X::template step<T>(r.x, c, in, t); Y::template step<T>(r.y, c, t, o);
  }
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C& c, const Fr8<IN>& in, Fr8<OUT>& o) {
    Fr8<X::OUT> t; group_step<X>(r.x, c, in, t); group_step<Y>(r.y, c, t, o);
  }
  static FDSP_DEV void end_simd(R& r) { X::end_simd(r.x); Y::end_simd(r.y); }
};
template <class X, class Y> struct Stack {  // ID 7
  FDSP_NODE(X::IN + Y::IN, X::OUT + Y::OUT, X::NP + Y::NP, X::NS + Y::NS, X::NU + Y::NU);
  struct R { typename X::R x; typename Y::R y; };
  static FDSP_DEV void load(R& r, Loader& l) { X::load(r.x, l); Y::load(r.y, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { X::save(r.x, s); Y::save(r.y, s); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<IN>& in, Fr<OUT>& o) {
    Fr<X::IN> xi; Fr<Y::IN> yi; Fr<X::OUT> a; Fr<Y::OUT> b;
    for (int k = 0; k < X::IN; k++) xi.v[k] = in.v[k];
    for (int k = 0; k < Y::IN; k++) yi.v[k] = in.v[X::IN + k];
    X::template step<T>(r.x, c, xi, a); Y::template step<T>(r.y, c, yi, b);
    for (int k = 0; k < X::OUT; k++) o.v[k] = a.v[k];
    for (int k = 0; k < Y::OUT; k++) o.v[X::OUT + k] = b.v[k];
  }
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C& c, const Fr8<IN>& in, Fr8<OUT>& o) {
    Fr8<X::IN> xi; Fr8<Y::IN> yi; Fr8<X::OUT> a; Fr8<Y::OUT> b;
    for (int k = 0; k < X::IN; k++) FDSP_G8 xi.v[k][j] = in.v[k][j];
    for (int k = 0; k < Y::IN; k++) FDSP_G8 yi.v[k][j] = in.v[X::IN + k][j];
    group_step<X>(r.x, c, xi, a); group_step<Y>(r.y, c, yi, b);
    for (int k = 0; k < X::OUT; k++) FDSP_G8 o.v[k][j] = a.v[k][j];
    for (int k = 0; k < Y::OUT; k++) FDSP_G8 o.v[X::OUT + k][j] = b.v[k][j];
  }
  static FDSP_DEV void end_simd(R& r) { X::end_simd(r.x); Y::end_simd(r.y); }
};
template <class X, class Y> struct Branch {  // ID 8
  FDSP_NODE(X::IN, X::OUT + Y::OUT, X::NP + Y::NP, X::NS + Y::NS, X::NU + Y::NU);
  struct R { typename X::R x; typename Y::R y; };
  static FDSP_DEV void load(R& r, Loader& l) { X::load(r.x, l); Y::load(r.y, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { X::save(r.x, s); Y::save(r.y, s); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<IN>& in, Fr<OUT>& o) {
    Fr<X::OUT> a; Fr<Y::OUT> b;
    X::template step<T>(r.x, c, in, a); Y::template step<T>(r.y, c, in, b);
    for (int k = 0; k < X::OUT; k++) o.v[k] = a.v[k];
    for (int k = 0; k < Y::OUT; k++) o.v[X::OUT + k] = b.v[k];
  }
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C& c, const Fr8<IN>& in, Fr8<OUT>& o) {
    Fr8<X::OUT> a; Fr8<Y::OUT> b;
    group_step<X>(r.x, c, in, a); group_step<Y>(r.y, c, in, b);
    for (int k = 0; k < X::OUT; k++) FDSP_G8 o.v[k][j] = a.v[k][j];
    for (int k = 0; k < Y::OUT; k++) FDSP_G8 o.v[X::OUT + k][j] = b.v[k][j];
  }
  static FDSP_DEV void end_simd(R& r) { X::end_simd(r.x); Y::end_simd(r.y); }
};
template <class X, class Y> struct Bus {  // ID 10
  FDSP_NODE(X::IN, X::OUT, X::NP + Y::NP, X::NS + Y::NS, X::NU + Y::NU);
  struct R { typename X::R x; typename Y::R y; };
  static FDSP_DEV void load(R& r, Loader& l) { X::load(r.x, l); Y::load(r.y, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { X::save(r.x, s); Y::save(r.y, s); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<IN>& in, Fr<OUT>& o) {
    Fr<Y::OUT> b;
    X::template step<T>(r.x, c, in, o); Y::template step<T>(r.y, c, in, b);
    for (int k = 0; k < OUT; k++) o.v[k] = o.v[k] + b.v[k];
  }
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C& c, const Fr8<IN>& in, Fr8<OUT>& o) {
    Fr8<Y::OUT> b;
    group_step<X>(r.x, c, in, o); group_step<Y>(r.y, c, in, b);
    for (int k = 0; k < OUT; k++) FDSP_G8 o.v[k][j] = o.v[k][j] + b.v[k][j];
  }
  static FDSP_DEV void end_simd(R& r) { X::end_simd(r.x); Y::end_simd(r.y); }
};
template <class X> struct Thru {  // ID 12
  FDSP_NODE(X::IN, X::IN, X::NP, X::NS, X::NU);
  struct R { typename X::R x; };
  static FDSP_DEV void load(R& r, Loader& l) { X::load(r.x, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { X::save(r.x, s); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<IN>& in, Fr<OUT>& o) {
    Fr<X::OUT> a; X::template step<T>(r.x, c, in, a);
    for (int k = 0; k < IN; k++) o.v[k] = k < X::OUT ? a.v[k < X::OUT ? k : 0] : in.v[k];
  }
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C& c, const Fr8<IN>& in, Fr8<OUT>& o) {
    Fr8<X::OUT> a; group_step<X>(r.x, c, in, a);
    for (int k = 0; k < IN; k++) FDSP_G8 o.v[k][j] = k < X::OUT ? a.v[k < X::OUT ? k : 0][j] : in.v[k][j];
  }
  static FDSP_DEV void end_simd(R& r) { X::end_simd(r.x); }
};
// Indexed combinators over N nodes of one type: KIND = reference node ID (28 bus, 30 stack, 31 reduce, 33 branch, 32 chain)
template <int KIND, int OP, int N, class X> struct Multi {
  static constexpr int IN = (KIND == 30 || KIND == 31) ? X::IN * N : X::IN;
  static constexpr int OUT = (KIND == 30 || KIND == 33) ? X::OUT * N : X::OUT;
  static constexpr int NP = X::NP * N, NS = X::NS * N, NU = X::NU * N;
  struct R { typename X::R x[N]; };
  static FDSP_DEV void load(R& r, Loader& l) {
#pragma unroll
    for (int k = 0; k < N; k++) X::load(r.x[k], l);
  }
  static FDSP_DEV void save(const R& r, Saver& s) {
#pragma unroll
    for (int k = 0; k < N; k++) X::save(r.x[k], s);
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<IN>& in, Fr<OUT>& o) {
    if (KIND == 32) {  // chain
      Fr<X::IN> t; Fr<X::OUT> u;
      for (int q = 0; q < X::IN; q++) t.v[q] = in.v[q];
#pragma unroll
      for (int k = 0; k < N; k++) { X::template step<T>(r.x[k], c, t, u); for (int q = 0; q < X::OUT && q < X::IN; q++) t.v[q] = u.v[q]; }
      for (int q = 0; q < X::OUT; q++) o.v[q] = u.v[q];
      return;
    }
#pragma unroll
    for (int k = 0; k < N; k++) {
      Fr<X::IN> xi; Fr<X::OUT> a;
      for (int q = 0; q < X::IN; q++) xi.v[q] = in.v[((KIND == 30 || KIND == 31) ? k * X::IN : 0) + q];
      X::template step<T>(r.x[k], c, xi, a);
      for (int q = 0; q < X::OUT; q++) {
        if (KIND == 30 || KIND == 33) o.v[k * X::OUT + q] = a.v[q];
        else if (k == 0) o.v[q] = a.v[q];
        else o.v[q] = (KIND == 28) ? o.v[q] + a.v[q] : binop<OP>(o.v[q], a.v[q]);
      }
    }
  }
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C& c, const Fr8<IN>& in, Fr8<OUT>& o) {
    if (KIND == 32) {  // chain
      Fr8<X::IN> t; Fr8<X::OUT> u;
      for (int q = 0; q < X::IN; q++) FDSP_G8 t.v[q][j] = in.v[q][j];
#pragma unroll
      for (int k = 0; k < N; k++) { group_step<X>(r.x[k], c, t, u); for (int q = 0; q < X::OUT && q < X::IN; q++) FDSP_G8 t.v[q][j] = u.v[q][j]; }
      for (int q = 0; q < X::OUT; q++) FDSP_G8 o.v[q][j] = u.v[q][j];
      return;
    }
#pragma unroll
    for (int k = 0; k < N; k++) {
      Fr8<X::IN> xi; Fr8<X::OUT> a;
      for (int q = 0; q < X::IN; q++) FDSP_G8 xi.v[q][j] = in.v[((KIND == 30 || KIND == 31) ? k * X::IN : 0) + q][j];
      group_step<X>(r.x[k], c, xi, a);
      for (int q = 0; q < X::OUT; q++) {
        FDSP_G8 {
          if (KIND == 30 || KIND == 33) o.v[k * X::OUT + q][j] = a.v[q][j];
          else if (k == 0) o.v[q][j] = a.v[q][j];
          else o.v[q][j] = (KIND == 28) ? o.v[q][j] + a.v[q][j] : binop<OP>(o.v[q][j], a.v[q][j]);
        }
      }
    }
  }
  static FDSP_DEV void end_simd(R& r) {
#pragma unroll
    for (int k = 0; k < N; k++) X::end_simd(r.x[k]);
  }
};

// ---------------------------------------------------------------- generators
struct Noise {  // src/noise.rs:170-234, ID 20: counter-based white noise
  FDSP_NODE(0, 1, 0, 1, 0);
  struct R { uint32_t state; };
  static FDSP_DEV void load(R& r, Loader& l) { r.state = l.S(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.S(r.state); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<0>&, Fr<1>& o) {
    r.state += 1u;
    o.v[0] = (float)(hash32x(r.state) >> 8) * (2.0f / 16777215.0f) - 1.0f;
  }
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C&, const Fr8<0>&, Fr8<1>& o) {
    uint32_t h[8];
    FDSP_G8 h[j] = hash32x(r.state + 1u + (uint32_t)j);
    FDSP_G8 o.v[0][j] = (float)(h[j] >> 8) * (2.0f / 16777215.0f) - 1.0f;
    r.state += 8u;
  }
  static FDSP_DEV void end_simd(R&) {}
};
struct Sine {  // src/oscillator.rs:18-102, ID 21
  FDSP_NODE(1, 1, 0, 1, 0);
  struct R { float phase; };
  static FDSP_DEV void load(R& r, Loader& l) { r.phase = l.Sf(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.Sf(r.phase); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<1>& in, Fr<1>& o) {
    float p = r.phase;
    r.phase += in.v[0] * c.sd64;
    if (T || c.rem) {  // tick path :67-72 (libm sinf, wrap every sample)
      r.phase -= floorf(r.phase);
      o.v[0] = m::sinf_(p * TAU_F);
    } else {           // block path :74-86 (wide sin, phase unwrapped inside the block)
      o.v[0] = wide_sinf(p * TAU_F);
    }
  }
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C& c, const Fr8<1>& in, Fr8<1>& o) {  // :74-86, 8 lanes at once
    float p[8];
    FDSP_G8 { p[j] = r.phase * TAU_F; r.phase += in.v[0][j] * c.sd64; }
    wide_sinf8(p, o.v[0]);
  }
  static FDSP_DEV void end_simd(R& r) { r.phase = r.phase - floorf(r.phase); }
};
template <int KIND, int NOUT> struct WaveSynth {  // src/wavetable.rs:244-359, ID 34
  FDSP_NODE(1, NOUT, 0, 2, 0);
  struct R { float phase; int hint; int ti; float w; int o1, o2; int l1, l2; float fsel; int hsel; };  // fsel/hsel: memo of the last select()
  static FDSP_DEV void load(R& r, Loader& l) { r.phase = l.Sf(); r.hint = (int)l.S(); r.ti = r.hint; r.w = 0.0f; r.o1 = r.o2 = 0; r.l1 = r.l2 = 32; r.fsel = __int_as_float(0x7fc00000); r.hsel = -1; }
  static FDSP_DEV void save(const R& r, Saver& s) { s.Sf(r.phase); s.S((uint32_t)r.hint); }
  static FDSP_DEV int table_index(const WaveTableDev& t, int hint, float f) {  // :157-179
    if (f >= __ldg(&t.pitch[hint]) && f <= __ldg(&t.pitch[hint + 1])) return hint;
    int i0 = 0, i1 = t.n - 3;
    while (i0 < i1) {
      int i = (i0 + i1) >> 1;
      if (__ldg(&t.pitch[i]) > f) i1 = i;
      else if (__ldg(&t.pitch[i + 1]) > f) { i0 = i; break; }
      else i0 = i + 1;
    }
    return i0;
  }
  static FDSP_DEV void select(R& r, const WaveTableDev& t, int hint, float freq) {  // read/read_simd :181-212
    float f = fabsf(freq);
    if (f == r.fsel && hint == r.hsel) return;  // pure function of (hint, f): a constant-pitch voice looks the tables up once
    r.fsel = f; r.hsel = hint;
    int ti = table_index(t, hint, f);
    r.ti = ti;
    r.w = clamp01f(delerpf(__ldg(&t.pitch[ti]), __ldg(&t.pitch[ti + 1]), f));
    r.o1 = __ldg(&t.off[ti + 1]); r.l1 = __ldg(&t.len[ti + 1]);
    r.o2 = __ldg(&t.off[ti + 2]); r.l2 = __ldg(&t.len[ti + 2]);
  }
  template <class C> static FDSP_DEV float tap(const C& c, const WaveTableDev& t, int idx) {
    if (C::SMEM_TABLES) { if (c.tsm_kind == KIND) return lds_f32(c.tsm + 4u * (uint32_t)idx); }
    return __ldg(t.data + idx);
  }
  // (int)p and (float)(int)p of a table position p = len * phase on the FP32 pipe, leaving the conversion unit to wide_floorf: the phase
  // lies in [0, 1], or below 0 by a few ulps (wide_floorf's rounding), or is NaN, so |p| < 2^23 and (int)p = (int)|p|. Adding 2^23 rounded
  // toward zero leaves that integer in the low mantissa bits of the sum; the caller masks them to the table (len <= 8192 < 2^23), which also
  // keeps a NaN phase's index inside it (its output is NaN either way).
  static FDSP_DEV int trunc_bits(float p, float& fi) {
    const float t = __fadd_rz(fabsf(p), 8388608.0f);
    fi = t - 8388608.0f;
    return (int)__float_as_uint(t);
  }
  // Tables carry wrap-around guard samples (host device_wavetable): taps i1-1 .. i1+2 modulo len are consecutive floats.
  template <class C> static FDSP_DEV float at(const C& c, const WaveTableDev& t, int off, int len, float phase) {  // :125-155 (i32 index math, truncation)
    float p = (float)len * phase;
    float fi;
    const int i1 = trunc_bits(p, fi);
    float w = p - fi;
    const int b = off + (i1 & (len - 1)) - 1;
    return optimal4x44(tap(c, t, b), tap(c, t, b + 1), tap(c, t, b + 2), tap(c, t, b + 3), w);
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<1>& in, Fr<NOUT>& o) {
    const WaveTableDev& t = c.wt[KIND];
    float ph;
    if (T || c.rem) {  // tick :309-325
      r.phase += in.v[0] * c.sd32;
      r.phase -= floorf(r.phase);
      select(r, t, r.hint, in.v[0]);
      r.hint = r.ti;
      ph = r.phase;
    } else {           // block :327-348: table from lane 0 of each 8-sample group, wide floor
      if (c.first) select(r, t, r.ti, in.v[0]);
      r.phase += in.v[0] * c.sd32;
      ph = r.phase - wide_floorf(r.phase);
    }
    o.v[0] = (1.0f - r.w) * at(c, t, r.o1, r.l1, ph) + r.w * at(c, t, r.o2, r.l2, ph);
    if (NOUT > 1) o.v[NOUT > 1 ? 1 : 0] = ph;
  }
  typedef void GroupStep;
  template <class C> static FDSP_DEV void at8(const C& c, const WaveTableDev& t, int off, int len, const float* ph, float* y) {
    float w[8], a0[8], a1[8], a2[8], a3[8];
    const int mask = len - 1;
    const float flen = (float)len;
    FDSP_G8 {
      const float p = flen * ph[j];
      float fi;
      const int i1 = trunc_bits(p, fi);
      w[j] = p - fi;
      const int b = off + (i1 & mask) - 1;
      a0[j] = tap(c, t, b); a1[j] = tap(c, t, b + 1); a2[j] = tap(c, t, b + 2); a3[j] = tap(c, t, b + 3);
    }
    optimal4x44_8(a0, a1, a2, a3, w, y);
  }
  template <class C> static FDSP_DEV void step8(R& r, C& c, const Fr8<1>& in, Fr8<NOUT>& o) {  // :327-348, one f32x8 group
    const WaveTableDev& t = c.wt[KIND];
    select(r, t, r.ti, in.v[0][0]);
    float ph[8], a[8], b[8];
    FDSP_G8 { r.phase += in.v[0][j] * c.sd32; ph[j] = r.phase - wide_floorf(r.phase); }
    at8(c, t, r.o1, r.l1, ph, a);
    at8(c, t, r.o2, r.l2, ph, b);
    const float u = 1.0f - r.w;
    FDSP_G8 o.v[0][j] = u * a[j] + r.w * b[j];
    if (NOUT > 1) FDSP_G8 o.v[NOUT > 1 ? 1 : 0][j] = ph[j];
  }
  static FDSP_DEV void end_simd(R& r) { r.phase = r.phase - floorf(r.phase); r.hint = r.ti; }
};

// PhaseSynth (src/wavetable.rs:361-433, ID 35): table lookup driven by a phase input; the band is chosen from the phase increment.
// The reference has no block override: every sample takes the scalar `read` (:181-195) on both paths.
template <int KIND> struct PhaseSynth {
  typedef WaveSynth<KIND, 1> W;
  FDSP_NODE(1, 1, 0, 3, 0);
  struct R { typename W::R w; float prev; int ready; };
  static FDSP_DEV void load(R& r, Loader& l) {
    r.prev = l.Sf(); r.ready = (int)l.S(); r.w.hint = (int)l.S();
    r.w.phase = 0.0f; r.w.ti = r.w.hint; r.w.w = 0.0f; r.w.o1 = r.w.o2 = 0; r.w.l1 = r.w.l2 = 32; r.w.fsel = __int_as_float(0x7fc00000); r.w.hsel = -1;
  }
  static FDSP_DEV void save(const R& r, Saver& s) { s.Sf(r.prev); s.S((uint32_t)r.ready); s.S((uint32_t)r.w.hint); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<1>& in, Fr<1>& o) {
    const WaveTableDev& t = c.wt[KIND];
    const float phase = in.v[0] - floorf(in.v[0]);
    float delta = 0.5f;   // first sample: pessimistically Nyquist
    if (r.ready) delta = fminf(fabsf(phase - r.prev), fminf(fabsf(phase - 1.0f - r.prev), fabsf(phase + 1.0f - r.prev)));
    r.ready = 1;
    W::select(r.w, t, r.w.hint, delta * c.sr);
    r.w.hint = r.w.ti;
    r.prev = phase;
    o.v[0] = (1.0f - r.w.w) * W::at(c, t, r.w.o1, r.w.l1, phase) + r.w.w * W::at(c, t, r.w.o2, r.w.l2, phase);
  }
  static FDSP_DEV void end_simd(R&) {}
};

// Mixer<M, N> (src/pan.rs:95-160, ID 84): constant N x M matrix, row i = weights of output i; tick only (0.0 + x0*y0 + x1*y1 ...).
template <int M, int N> struct Mixer {
  FDSP_NODE(M, N, M * N, 0, 0);
  struct R { float m[N][M]; };
  static FDSP_DEV void load(R& r, Loader& l) {
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
      for (int j = 0; j < M; j++) r.m[i][j] = l.Pf();
  }
  static FDSP_DEV void save(const R&, Saver&) {}
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<M>& in, Fr<N>& o) {
#pragma unroll
    for (int i = 0; i < N; i++) {
      float v = 0.0f;
#pragma unroll
      for (int j = 0; j < M; j++) v += in.v[j] * r.m[i][j];
      o.v[i] = v;
    }
  }
  static FDSP_DEV void end_simd(R&) {}
};

// ---------------------------------------------------------------- filters
struct FixedSvf {  // src/svf.rs:857-1031, ID 43 (coefficients computed on the host at set_sample_rate)
  FDSP_NODE(1, 1, 6, 2, 0);
  struct R { float a1, a2, a3, m0, m1, m2, ic1, ic2; };
  static FDSP_DEV void load(R& r, Loader& l) { r.a1 = l.Pf(); r.a2 = l.Pf(); r.a3 = l.Pf(); r.m0 = l.Pf(); r.m1 = l.Pf(); r.m2 = l.Pf(); r.ic1 = l.Sf(); r.ic2 = l.Sf(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.Sf(r.ic1); s.Sf(r.ic2); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<1>& in, Fr<1>& o) {  // :995-1006
    float v0 = in.v[0];
    float v3 = v0 - r.ic2;
    float v1 = r.a1 * r.ic1 + r.a2 * v3;
    float v2 = r.ic2 + r.a2 * r.ic1 + r.a3 * v3;
    r.ic1 = 2.0f * v1 - r.ic1;
    r.ic2 = 2.0f * v2 - r.ic2;
    o.v[0] = r.m0 * v0 + r.m1 * v1 + r.m2 * v2;
  }
  static FDSP_DEV void end_simd(R&) {}
};
// The audio-rate f32 filters keep their coefficients in state next to the controls they were computed from, and `ksr`, the rate they
// were computed at. The reference's set_sample_rate recomputes them from the stored controls (src/svf.rs:823-826, src/biquad.rs:263-266,
// :349-351, :535-538, :745-748, src/filter.rs:58-61, :392-395, src/rez.rs:59-62), and the next sample's change test then compares the
// inputs with those stored controls. So a launch at another rate first recomputes from the stored controls, then runs the usual test.
template <int MODE> struct Svf {  // src/svf.rs:744-855, ID 36 (audio-rate cutoff/Q[/gain] inputs; recompute on change or rate change)
  static constexpr int NI = MODE >= 6 ? 4 : 3;
  FDSP_NODE(NI, 1, 0, 12, 0);
  struct R { float cutoff, q, gain, ksr; SvfCoefs k; float ic1, ic2; };
  static FDSP_DEV void load(R& r, Loader& l) {
    r.cutoff = l.Sf(); r.q = l.Sf(); r.gain = l.Sf(); r.ksr = l.Sf();
    r.k.a1 = l.Sf(); r.k.a2 = l.Sf(); r.k.a3 = l.Sf(); r.k.m0 = l.Sf(); r.k.m1 = l.Sf(); r.k.m2 = l.Sf();
    r.ic1 = l.Sf(); r.ic2 = l.Sf();
  }
  static FDSP_DEV void save(const R& r, Saver& s) {
    s.Sf(r.cutoff); s.Sf(r.q); s.Sf(r.gain); s.Sf(r.ksr);
    s.Sf(r.k.a1); s.Sf(r.k.a2); s.Sf(r.k.a3); s.Sf(r.k.m0); s.Sf(r.k.m1); s.Sf(r.k.m2);
    s.Sf(r.ic1); s.Sf(r.ic2);
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<NI>& in, Fr<1>& o) {
    if (r.ksr != c.sr) { r.ksr = c.sr; r.k = svf_coefs<MODE>(c.sr, r.cutoff, r.q, r.gain); }
    bool ch = in.v[1] != r.cutoff || in.v[2] != r.q;
    if (MODE >= 6) ch = ch || in.v[NI - 1] != r.gain;
    if (ch) { r.cutoff = in.v[1]; r.q = in.v[2]; if (MODE >= 6) r.gain = in.v[NI - 1]; r.k = svf_coefs<MODE>(c.sr, r.cutoff, r.q, r.gain); }
    float v0 = in.v[0];
    float v3 = v0 - r.ic2;
    float v1 = r.k.a1 * r.ic1 + r.k.a2 * v3;
    float v2 = r.ic2 + r.k.a2 * r.ic1 + r.k.a3 * v3;
    r.ic1 = 2.0f * v1 - r.ic1;
    r.ic2 = 2.0f * v2 - r.ic2;
    o.v[0] = r.k.m0 * v0 + r.k.m1 * v1 + r.k.m2 * v2;
  }
  static FDSP_DEV void end_simd(R&) {}
};
struct Morph {  // src/svf.rs:1034-1111, ID 62: (peak SVF(audio, cutoff, q) + morph * audio) / 2
  typedef Svf<4> F;
  FDSP_NODE(4, 1, 0, F::NS, 0);
  typedef F::R R;
  static FDSP_DEV void load(R& r, Loader& l) { F::load(r, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { F::save(r, s); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<4>& in, Fr<1>& o) {
    Fr<3> a; Fr<1> y;
    a.v[0] = in.v[0]; a.v[1] = in.v[1]; a.v[2] = in.v[2];
    F::template step<T>(r, c, a, y);
    o.v[0] = (y.v[0] + in.v[3] * in.v[0]) * 0.5f;
  }
  static FDSP_DEV void end_simd(R&) {}
};
template <int NIN> struct Rez {  // src/rez.rs, ID 75: params = bandpass (and f, fb when the cutoff / q are fixed)
  FDSP_NODE(NIN, 1, NIN == 1 ? 3 : 1, NIN == 1 ? 2 : 7, 0);
  struct R { float bandpass, f, fb, cutoff, q, ksr, buf0, buf1; };
  static FDSP_DEV void load(R& r, Loader& l) {
    r.bandpass = l.Pf();
    if (NIN == 1) { r.f = l.Pf(); r.fb = l.Pf(); r.cutoff = r.q = r.ksr = 0.0f; } else { r.cutoff = l.Sf(); r.q = l.Sf(); r.ksr = l.Sf(); r.f = l.Sf(); r.fb = l.Sf(); }
    r.buf0 = l.Sf(); r.buf1 = l.Sf();
  }
  static FDSP_DEV void save(const R& r, Saver& s) { if (NIN > 1) { s.Sf(r.cutoff); s.Sf(r.q); s.Sf(r.ksr); s.Sf(r.f); s.Sf(r.fb); } s.Sf(r.buf0); s.Sf(r.buf1); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<NIN>& in, Fr<1>& o) {
    if (NIN > 1) {
      const float cu = in.v[NIN > 1 ? 1 : 0], qq = in.v[NIN > 2 ? 2 : 0];
      if (r.ksr != c.sr) { r.ksr = c.sr; r.f = 2.0f * m::sinf_(3.14159274101257324f * r.cutoff / c.sr); r.fb = r.q + r.q / (1.0f - r.f); }
      if (cu != r.cutoff || qq != r.q) { r.cutoff = cu; r.q = qq; r.f = 2.0f * m::sinf_(3.14159274101257324f * cu / c.sr); r.fb = qq + qq / (1.0f - r.f); }
    }
    const float hp = in.v[0] - r.buf0, bp = r.buf0 - r.buf1;
    r.buf0 += r.f * (hp + r.fb * m::tanhf_(bp));
    r.buf1 += r.f * (r.buf0 - r.buf1);
    o.v[0] = r.buf1 - r.bandpass * r.buf0;
  }
  static FDSP_DEV void end_simd(R&) {}
};
struct Biquad {  // src/biquad.rs:130-218, ID 15 (also the fixed ButterLowpass ID 16 / Resonator ID 17): DF1, left-to-right
  FDSP_NODE(1, 1, 5, 4, 0);
  struct R { float a1, a2, b0, b1, b2, x1, x2, y1, y2; };
  static FDSP_DEV void load(R& r, Loader& l) { r.a1 = l.Pf(); r.a2 = l.Pf(); r.b0 = l.Pf(); r.b1 = l.Pf(); r.b2 = l.Pf(); r.x1 = l.Sf(); r.x2 = l.Sf(); r.y1 = l.Sf(); r.y2 = l.Sf(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.Sf(r.x1); s.Sf(r.x2); s.Sf(r.y1); s.Sf(r.y2); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<1>& in, Fr<1>& o) {
    float x0 = in.v[0];
    float y0 = r.b0 * x0 + r.b1 * r.x1 + r.b2 * r.x2 - r.a1 * r.y1 - r.a2 * r.y2;
    r.x2 = r.x1; r.x1 = x0; r.y2 = r.y1; r.y1 = y0;
    o.v[0] = y0;
  }
  static FDSP_DEV void end_simd(R&) {}
};
struct BiquadBank {  // src/biquad_bank.rs:9-117, ID 98: 8 independent DF1 lanes, one per channel
  FDSP_NODE(8, 8, 40, 32, 0);
  struct R { Biquad::R b[8]; };
  static FDSP_DEV void load(R& r, Loader& l) {
#pragma unroll
    for (int k = 0; k < 8; k++) { r.b[k].a1 = l.Pf(); r.b[k].a2 = l.Pf(); r.b[k].b0 = l.Pf(); r.b[k].b1 = l.Pf(); r.b[k].b2 = l.Pf(); }
#pragma unroll
    for (int k = 0; k < 8; k++) { r.b[k].x1 = l.Sf(); r.b[k].x2 = l.Sf(); r.b[k].y1 = l.Sf(); r.b[k].y2 = l.Sf(); }
  }
  static FDSP_DEV void save(const R& r, Saver& s) {
#pragma unroll
    for (int k = 0; k < 8; k++) { s.Sf(r.b[k].x1); s.Sf(r.b[k].x2); s.Sf(r.b[k].y1); s.Sf(r.b[k].y2); }
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<8>& in, Fr<8>& o) {
#pragma unroll
    for (int k = 0; k < 8; k++) { Fr<1> a, b; a.v[0] = in.v[k]; Biquad::step<T>(r.b[k], c, a, b); o.v[k] = b.v[0]; }
  }
  static FDSP_DEV void end_simd(R&) {}
};
// Moog::set_cutoff_q (src/moog.rs:48-57). Out of line: the audio-rate form tests per sample whether (cutoff, q) changed, and an inlined
// sinf + division behind that test put ~400 cold instructions between every two samples of the unrolled ladder (73 KB per 8-sample group:
// instruction-fetch stalls on the recurrence's critical path).
struct MoogCoefs { float p, k, rez; };
FDSP_COLD MoogCoefs moog_coefs(float cutoff, float q, float sr) {
  MoogCoefs o;
  const float cc = 2.0f * cutoff / sr;
  o.p = cc * (1.8f - 0.8f * cc);
  o.k = 2.0f * m::sinf_(cc * 3.14159274101257324f * 0.5f) - 1.0f;
  const float t1 = (1.0f - o.p) * 1.386249f;
  const float t2 = 12.0f + t1 * t1;
  o.rez = q * (t2 + 6.0f * t1) / (t2 - 6.0f * t1);
  return o;
}
template <int NIN> struct Moog {  // src/moog.rs:11-117, ID 60
  FDSP_NODE(NIN, 1, NIN == 1 ? 3 : 0, 8, 0);
  struct R { float p, k, rez, s0, s1, s2, s3, px, ps0, ps1, ps2; float cutoff, q; };
  static FDSP_DEV void load(R& r, Loader& l) {
    if (NIN == 1) { r.p = l.Pf(); r.k = l.Pf(); r.rez = l.Pf(); } else { r.p = r.k = r.rez = 0.0f; }
    r.cutoff = r.q = __uint_as_float(0x7fc00000u);  // NaN: forces the first coefficient computation
    r.s0 = l.Sf(); r.s1 = l.Sf(); r.s2 = l.Sf(); r.s3 = l.Sf(); r.px = l.Sf(); r.ps0 = l.Sf(); r.ps1 = l.Sf(); r.ps2 = l.Sf();
  }
  static FDSP_DEV void save(const R& r, Saver& s) { s.Sf(r.s0); s.Sf(r.s1); s.Sf(r.s2); s.Sf(r.s3); s.Sf(r.px); s.Sf(r.ps0); s.Sf(r.ps1); s.Sf(r.ps2); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<NIN>& in, Fr<1>& o) {
    if (NIN > 1) {
      // :83-85 calls set_cutoff_q (:48-57) every sample; it is a pure function of (cutoff, q, sr), so it is
      // re-evaluated only when an input actually changed (bit-identical result, no sin + divide per sample).
      float cutoff = in.v[NIN > 1 ? 1 : 0], q = in.v[NIN > 2 ? 2 : 0];
      if (!(cutoff == r.cutoff && q == r.q)) {
        r.cutoff = cutoff; r.q = q;
        const MoogCoefs m = moog_coefs(cutoff, q, c.sr);
        r.p = m.p; r.k = m.k; r.rez = m.rez;
      }
    }
    o.v[0] = ladder(r, in.v[0]);
  }
  static FDSP_DEV float ladder(R& r, float in0) {   // :87-98
    float x = -r.rez * r.s3 + in0;
    r.s0 = (x + r.px) * r.p - r.k * r.s0;
    r.s1 = (r.s0 + r.ps0) * r.p - r.k * r.s1;
    r.s2 = (r.s1 + r.ps1) * r.p - r.k * r.s2;
    r.s3 = m::tanhf_((r.s2 + r.ps2) * r.p - r.k * r.s3);
    r.px = x; r.ps0 = r.s0; r.ps1 = r.s1; r.ps2 = r.s2;
    return r.s3;
  }
  // Steady group (group_step, fully unrolled form): when none of the 8 samples changes (cutoff, q) — the normal case — the ladder runs its 8
  // steps as straight-line code, without the "did an input change" test and its branch / reconvergence point between every two samples.
  typedef void SteadyGroup;
  static FDSP_DEV bool steady8(const R& r, const Fr8<NIN>& in) {
    bool same = true;
    if (NIN > 1) {
#pragma unroll
      for (int j = 0; j < 8; j++) same = same && in.v[NIN > 1 ? 1 : 0][j] == r.cutoff && in.v[NIN > 2 ? 2 : 0][j] == r.q;
    }
    return same;
  }
  static FDSP_DEV void step8_steady(R& r, const Fr8<NIN>& in, Fr8<1>& o) {
#pragma unroll
    for (int j = 0; j < 8; j++) o.v[0][j] = ladder(r, in.v[0][j]);
  }
  static FDSP_DEV void end_simd(R&) {}
};
template <int N> struct Fir {  // src/fir.rs:11-89, ID 52: shift register, accumulate from 0.0 in index order
  FDSP_NODE(1, 1, N, N, 0);
  struct R { float w[N], v[N]; };
  static FDSP_DEV void load(R& r, Loader& l) { for (int k = 0; k < N; k++) r.w[k] = l.Pf(); for (int k = 0; k < N; k++) r.v[k] = l.Sf(); }
  static FDSP_DEV void save(const R& r, Saver& s) { for (int k = 0; k < N; k++) s.Sf(r.v[k]); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<1>& in, Fr<1>& o) {
    for (int k = 0; k + 1 < N; k++) r.v[k] = r.v[k + 1];
    r.v[N - 1] = in.v[0];
    float a = 0.0f;
    for (int k = 0; k < N; k++) a += r.w[k] * r.v[k];
    o.v[0] = a;
  }
  static FDSP_DEV void end_simd(R&) {}
};


// ---------------------------------------------------------------- phase oscillators, MLS, impulse
FDSP_DEV float polyblep(float t, float dt) {  // src/oscillator.rs:510-521
  if (t < dt) { float z = t / dt; return z + z - z * z - 1.0f; }
  else if (t > 1.0f - dt) { float z = (t - 1.0f) / dt; return z + z + z * z + 1.0f; }
  return 0.0f;
}
template <int KIND> struct PhaseOsc {  // src/oscillator.rs:440-760: 0 Ramp (ID 94), 1 PolySaw (95), 2 PolySquare (96), 3 PolyPulse (97)
  FDSP_NODE(KIND == 3 ? 2 : 1, 1, 0, 1, 0);
  struct R { float phase; };
  static FDSP_DEV void load(R& r, Loader& l) { r.phase = l.Sf(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.Sf(r.phase); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<IN>& in, Fr<1>& o) {
    const float p = r.phase;
    const float delta = in.v[0] * c.sd64;
    r.phase += delta;
    r.phase -= floorf(r.phase);
    if (KIND == 0) { o.v[0] = p; return; }
    if (KIND == 1) { o.v[0] = 2.0f * p - 1.0f - polyblep(p, delta); return; }
    const float width = KIND == 2 ? 0.5f : in.v[IN - 1];
    const float square = p < width ? 1.0f : -1.0f;
    const float half = p - width;
    o.v[0] = square + polyblep(p, delta) - polyblep(half - floorf(half), delta);
  }
  static FDSP_DEV void end_simd(R&) {}
};
template <int NIN> struct Dsf {  // src/oscillator.rs:104-208, ID 55: params = roughness (clamped), harmonic spacing
  FDSP_NODE(NIN, 1, 2, 1, 0);
  struct R { float roughness, spacing, phase; };
  static FDSP_DEV void load(R& r, Loader& l) { r.roughness = l.Pf(); r.spacing = l.Pf(); r.phase = l.Sf(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.Sf(r.phase); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<NIN>& in, Fr<1>& o) {
    if (NIN > 1) r.roughness = fminf(fmaxf(in.v[NIN > 1 ? 1 : 0], 0.0001f), 0.9999f);   // set_roughness :152-154 (sticky, like the reference field)
    r.phase += in.v[0] * c.sd64;
    r.phase -= floorf(r.phase);
    const float n = floorf(22050.0f / in.v[0] / r.spacing);
    const float f = r.phase * TAU_F, d = r.phase * TAU_F * r.spacing, q = r.roughness;
    o.v[0] = (m::sinf_(f) - q * m::sinf_(f - d) - m::powf_(q, n + 1.0f) * (m::sinf_(f + (n + 1.0f) * d) - q * m::sinf_(f + n * d))) / (1.0f + q * q - 2.0f * q * m::cosf_(d));
  }
  static FDSP_DEV void end_simd(R&) {}
};
template <int KIND> struct Chaos {  // src/oscillator.rs:318-438: KIND 0 Rossler (ID 73), 1 Lorenz (ID 74); input = frequency
  FDSP_NODE(1, 1, 0, 3, 0);
  struct R { float x, y, z; };
  static FDSP_DEV void load(R& r, Loader& l) { r.x = l.Sf(); r.y = l.Sf(); r.z = l.Sf(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.Sf(r.x); s.Sf(r.y); s.Sf(r.z); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<1>& in, Fr<1>& o) {
    if (KIND == 0) {
      const float dx = -r.y - r.z, dy = r.x + 0.15f * r.y, dz = 0.2f + r.z * (r.x - 10.0f), dt = 2.91f * in.v[0] / c.sr;
      r.x += dx * dt; r.y += dy * dt; r.z += dz * dt;
      o.v[0] = r.x * 0.05757f;
    } else {
      const float dx = 10.0f * (r.y - r.x), dy = r.x * (28.0f - r.z) - r.y, dz = r.x * r.y - (8.0f / 3.0f) * r.z, dt = in.v[0] / c.sr;
      r.x += dx * dt; r.y += dy * dt; r.z += dz * dt;
      o.v[0] = r.x * 0.05107f;
    }
  }
  static FDSP_DEV void end_simd(R&) {}
};
struct Mls {  // src/noise.rs:11-148, ID 19: params = feedback polynomial, length mask, n - 1
  FDSP_NODE(0, 1, 3, 1, 0);
  struct R { uint32_t poly, mask, shift, s; };
  static FDSP_DEV void load(R& r, Loader& l) { r.poly = l.P(); r.mask = l.P(); r.shift = l.P(); r.s = l.S(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.S(r.s); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<0>&, Fr<1>& o) {
    const float value = (float)((r.s >> r.shift) & 1u);
    const uint32_t parity = (uint32_t)__popc(r.poly & r.s) & 1u;
    r.s = ((r.s << 1) | parity) & r.mask;
    o.v[0] = value * 2.0f - 1.0f;
  }
  static FDSP_DEV void end_simd(R&) {}
};
template <int N> struct Impulse {  // src/audionode.rs:2839-2873, ID 81
  FDSP_NODE(0, N, 0, 1, 0);
  struct R { float value; };
  static FDSP_DEV void load(R& r, Loader& l) { r.value = l.Sf(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.Sf(r.value); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<0>&, Fr<N>& o) { for (int k = 0; k < N; k++) o.v[k] = r.value; r.value = 0.0f; }
  static FDSP_DEV void end_simd(R&) {}
};

// ---------------------------------------------------------------- interpolated taps (src/delay.rs:141-286, 379-505)
FDSP_DEV float splinef(float y0, float y1, float y2, float y3, float x) {  // src/math.rs:327-333
  return y1 + x * 0.5f * (y2 - y0 + x * (2.0f * y0 - 5.0f * y1 + 4.0f * y2 - y3 + x * (3.0f * (y1 - y2) + y3 - y0)));
}
template <int NT_, int LINEAR> struct Tap {  // Tap<N> ID 50 (Catmull-Rom) / TapLinear<N> ID 54; power-of-two ring in HBM
  FDSP_NODE(NT_ + 1, 1, 2, 1, 1);
  struct R { float lo, hi; uint32_t i, len, off; };
  static FDSP_DEV void load(R& r, Loader& l) { r.lo = l.Pf(); r.hi = l.Pf(); r.len = l.U(); r.off = l.D(r.len); r.i = l.S(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.S(r.i); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<IN>& in, Fr<1>& o) {
    const uint32_t mask = r.len - 1u;
    float* b = c.dl + c.v;
    const size_t V = c.V;
    b[(size_t)(r.off + r.i) * V] = in.v[0];
    float acc = 0.0f;
#pragma unroll
    for (int t = 1; t <= NT_; t++) {
      const float tap = fminf(fmaxf(in.v[t], r.lo), r.hi) * c.sr;
      const uint32_t tf = (uint32_t)tap;
      const uint32_t i1 = (r.i - tf) & mask;
      const float d = tap - (float)tf;
      if (LINEAR) {
        const uint32_t i2 = (i1 - 1u) & mask;
        acc += lerpf(b[(size_t)(r.off + i1) * V], b[(size_t)(r.off + i2) * V], d);
      } else {
        const uint32_t i0 = (i1 + 1u) & mask, i2 = (i1 - 1u) & mask, i3 = (i1 - 2u) & mask;
        acc += splinef(b[(size_t)(r.off + i0) * V], b[(size_t)(r.off + i1) * V], b[(size_t)(r.off + i2) * V], b[(size_t)(r.off + i3) * V], d);
      }
    }
    r.i = (r.i + 1u) & mask;
    o.v[0] = acc;
  }
  static FDSP_DEV void end_simd(R&) {}
};

// ---------------------------------------------------------------- biquads with audio-rate parameters (src/biquad.rs:220-382)
struct ButterLowpass2 {  // ButterLowpass<f32,U2>, ID 16: (audio, cutoff) -> 1, coefficients recomputed when the cutoff input changes
  FDSP_NODE(2, 1, 0, 11, 0);
  static FDSP_DEV void set(Biquad::R& b, const BqCoefs& k) { b.a1 = k.a1; b.a2 = k.a2; b.b0 = k.b0; b.b1 = k.b1; b.b2 = k.b2; }
  struct R { float cutoff, ksr; Biquad::R b; };
  static FDSP_DEV void load(R& r, Loader& l) { r.cutoff = l.Sf(); r.ksr = l.Sf(); r.b.a1 = l.Sf(); r.b.a2 = l.Sf(); r.b.b0 = l.Sf(); r.b.b1 = l.Sf(); r.b.b2 = l.Sf(); r.b.x1 = l.Sf(); r.b.x2 = l.Sf(); r.b.y1 = l.Sf(); r.b.y2 = l.Sf(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.Sf(r.cutoff); s.Sf(r.ksr); s.Sf(r.b.a1); s.Sf(r.b.a2); s.Sf(r.b.b0); s.Sf(r.b.b1); s.Sf(r.b.b2); s.Sf(r.b.x1); s.Sf(r.b.x2); s.Sf(r.b.y1); s.Sf(r.b.y2); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<2>& in, Fr<1>& o) {
    if (r.ksr != c.sr) { r.ksr = c.sr; set(r.b, bq_butter_lowpass(c.sr, r.cutoff)); }
    if (in.v[1] != r.cutoff) { r.cutoff = in.v[1]; set(r.b, bq_butter_lowpass(c.sr, r.cutoff)); }
    Fr<1> a; a.v[0] = in.v[0];
    Biquad::step<T>(r.b, c, a, o);
  }
  static FDSP_DEV void end_simd(R&) {}
};
struct Resonator3 {  // Resonator<f32,U3>, ID 17: (audio, center, q) -> 1
  FDSP_NODE(3, 1, 0, 12, 0);
  struct R { float center, q, ksr; Biquad::R b; };
  static FDSP_DEV void load(R& r, Loader& l) { r.center = l.Sf(); r.q = l.Sf(); r.ksr = l.Sf(); r.b.a1 = l.Sf(); r.b.a2 = l.Sf(); r.b.b0 = l.Sf(); r.b.b1 = l.Sf(); r.b.b2 = l.Sf(); r.b.x1 = l.Sf(); r.b.x2 = l.Sf(); r.b.y1 = l.Sf(); r.b.y2 = l.Sf(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.Sf(r.center); s.Sf(r.q); s.Sf(r.ksr); s.Sf(r.b.a1); s.Sf(r.b.a2); s.Sf(r.b.b0); s.Sf(r.b.b1); s.Sf(r.b.b2); s.Sf(r.b.x1); s.Sf(r.b.x2); s.Sf(r.b.y1); s.Sf(r.b.y2); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<3>& in, Fr<1>& o) {
    if (r.ksr != c.sr) { r.ksr = c.sr; ButterLowpass2::set(r.b, bq_resonator(c.sr, r.center, r.q)); }
    if (in.v[1] != r.center || in.v[2] != r.q) { r.center = in.v[1]; r.q = in.v[2]; ButterLowpass2::set(r.b, bq_resonator(c.sr, r.center, r.q)); }
    Fr<1> a; a.v[0] = in.v[0];
    Biquad::step<T>(r.b, c, a, o);
  }
  static FDSP_DEV void end_simd(R&) {}
};

// ---------------------------------------------------------------- delays / feedback
template <int N> struct Tick {  // src/delay.rs:17-65, ID 9
  FDSP_NODE(N, N, 0, N, 0);
  struct R { float b[N]; };
  static FDSP_DEV void load(R& r, Loader& l) { for (int k = 0; k < N; k++) r.b[k] = l.Sf(); }
  static FDSP_DEV void save(const R& r, Saver& s) { for (int k = 0; k < N; k++) s.Sf(r.b[k]); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<N>& in, Fr<N>& o) { for (int k = 0; k < N; k++) { float t = r.b[k]; r.b[k] = in.v[k]; o.v[k] = t; } }
  static FDSP_DEV void end_simd(R&) {}
};
struct Delay {  // src/delay.rs:67-139, ID 13: ring buffer of round(t*sr)+1 samples in HBM, element (off+pos)*V+v
  FDSP_NODE(1, 1, 0, 1, 1);
  struct R { uint32_t i, len, off; };
  static FDSP_DEV void load(R& r, Loader& l) { r.len = l.U(); r.off = l.D(r.len); r.i = l.S(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.S(r.i); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<1>& in, Fr<1>& o) {
    c.dl[(size_t)(r.off + r.i) * c.V + c.v] = in.v[0];
    r.i += 1u; if (r.i >= r.len) r.i = 0u;
    o.v[0] = c.dl[(size_t)(r.off + r.i) * c.V + c.v];
  }
  static FDSP_DEV void end_simd(R&) {}
};
template <int NIN, class X> struct AllNest {  // src/delay.rs:288-377, ID 83
  FDSP_NODE(NIN, 1, (NIN == 1 ? 1 : 0) + X::NP, 1 + (NIN > 1 ? 1 : 0) + X::NS, X::NU);
  struct R { float eta, z; typename X::R x; };
  static FDSP_DEV void load(R& r, Loader& l) { if (NIN == 1) { r.eta = l.Pf(); r.z = l.Sf(); } else { r.eta = l.Sf(); r.z = l.Sf(); } X::load(r.x, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { if (NIN > 1) s.Sf(r.eta); s.Sf(r.z); X::save(r.x, s); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<NIN>& in, Fr<1>& o) {
    if (NIN > 1) r.eta = in.v[NIN > 1 ? 1 : 0];
    Fr<1> v, y;
    v.v[0] = in.v[0] - r.eta * r.z;
    float out = r.eta * v.v[0] + r.z;
    X::template step<true>(r.x, c, v, y);  // default process = per-sample tick (no block path)
    r.z = y.v[0];
    o.v[0] = out;
  }
  static FDSP_DEV void end_simd(R&) {}
};
template <int N> FDSP_DEV void hadamard(float (&v)[N]) {  // src/feedback.rs:35-57
#pragma unroll
  for (int h = 1; h < N; h *= 2)
#pragma unroll
    for (int i = 0; i < N; i += h * 2)
#pragma unroll
      for (int j = i; j < i + h; j++) { float x = v[j], y = v[j + h]; v[j] = x + y; v[j + h] = x - y; }
  const float z = (float)(1.0 / sqrt((double)N));
#pragma unroll
  for (int i = 0; i < N; i++) v[i] = v[i] * z;
}
template <int HAD, class X> struct Feedback {  // src/feedback.rs:68-178, ID 11: the enclosed graph runs its TICK semantics
  static constexpr int N = X::IN;
  FDSP_NODE(N, N, X::NP, N + X::NS, X::NU);
  struct R { float value[N]; typename X::R x; };
  static FDSP_DEV void load(R& r, Loader& l) { for (int k = 0; k < N; k++) r.value[k] = l.Sf(); X::load(r.x, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { for (int k = 0; k < N; k++) s.Sf(r.value[k]); X::save(r.x, s); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<N>& in, Fr<N>& o) {
    Fr<N> t;
    for (int k = 0; k < N; k++) t.v[k] = in.v[k] + r.value[k];
    X::template step<true>(r.x, c, t, o);
    for (int k = 0; k < N; k++) r.value[k] = o.v[k];
    if (HAD) hadamard<N>(r.value);
  }
  static FDSP_DEV void end_simd(R&) {}
};


template <int HAD, class X, class Y> struct Feedback2 {  // src/feedback.rs:180-314, ID 66: out = x(in + value); value = U(y(out))
  static constexpr int N = X::IN;
  FDSP_NODE(N, N, X::NP + Y::NP, N + X::NS + Y::NS, X::NU + Y::NU);
  struct R { float value[N]; typename X::R x; typename Y::R y; };
  static FDSP_DEV void load(R& r, Loader& l) { for (int k = 0; k < N; k++) r.value[k] = l.Sf(); X::load(r.x, l); Y::load(r.y, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { for (int k = 0; k < N; k++) s.Sf(r.value[k]); X::save(r.x, s); Y::save(r.y, s); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<N>& in, Fr<N>& o) {
    Fr<N> t, u;
    for (int k = 0; k < N; k++) t.v[k] = in.v[k] + r.value[k];
    X::template step<true>(r.x, c, t, o);
    Y::template step<true>(r.y, c, o, u);
    for (int k = 0; k < N; k++) r.value[k] = u.v[k];
    if (HAD) hadamard<N>(r.value);
  }
  static FDSP_DEV void end_simd(R&) {}
};

// ---------------------------------------------------------------- one-pole family (src/filter.rs, F = f32)
// KIND 0 Lowpole (ID 18), 1 Highpole (ID 47), 2 Allpole (ID 46), 3 DCBlock (ID 22); NIN = 2 adds the audio-rate parameter input
// (cutoff: coefficient recomputed when it or the rate changes, :65-70 / :399-404, `ksr` as in Svf; allpole delay: every sample, :315-317).
template <int KIND, int NIN> struct OnePole {
  static constexpr bool KSR = NIN > 1 && KIND != 2;
  FDSP_NODE(NIN, 1, NIN == 1 ? 1 : 0, (KIND == 0 ? 1 : 2) + (NIN > 1 ? 2 : 0) + (KSR ? 1 : 0), 0);
  struct R { float coeff, param, ksr, x1, y1; };
  static FDSP_DEV void load(R& r, Loader& l) {
    if (NIN == 1) { r.coeff = l.Pf(); r.param = 0.0f; } else { r.param = l.Sf(); r.coeff = l.Sf(); }
    r.ksr = KSR ? l.Sf() : 0.0f;
    r.x1 = (KIND == 0) ? 0.0f : l.Sf(); r.y1 = l.Sf();
  }
  static FDSP_DEV void save(const R& r, Saver& s) { if (NIN > 1) { s.Sf(r.param); s.Sf(r.coeff); } if (KSR) s.Sf(r.ksr); if (KIND != 0) s.Sf(r.x1); s.Sf(r.y1); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<NIN>& in, Fr<1>& o) {
    if (NIN > 1) {
      const float p = in.v[NIN > 1 ? 1 : 0];
      if (KIND == 2) r.coeff = onepole_coeff(2, c.sr, p);
      else {
        if (r.ksr != c.sr) { r.ksr = c.sr; r.coeff = onepole_coeff(KIND, c.sr, r.param); }
        if (p != r.param) { r.param = p; r.coeff = onepole_coeff(KIND, c.sr, p); }
      }
    }
    const float x = in.v[0];
    float y0;
    if (KIND == 0) y0 = (1.0f - r.coeff) * x + r.coeff * r.y1;
    else if (KIND == 1) y0 = r.coeff * (r.y1 + x - r.x1);
    else if (KIND == 2) y0 = r.coeff * (x - r.y1) + r.x1;
    else y0 = x - r.x1 + r.coeff * r.y1;
    r.x1 = x; r.y1 = y0;
    o.v[0] = y0;
  }
  static FDSP_DEV void end_simd(R&) {}
};
struct Pinkpass {  // src/filter.rs:178-262, ID 26 (Paul Kellett's pinking filter)
  FDSP_NODE(1, 1, 0, 7, 0);
  struct R { float b[7]; };
  static FDSP_DEV void load(R& r, Loader& l) { for (int k = 0; k < 7; k++) r.b[k] = l.Sf(); }
  static FDSP_DEV void save(const R& r, Saver& s) { for (int k = 0; k < 7; k++) s.Sf(r.b[k]); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<1>& in, Fr<1>& o) {
    const float x = in.v[0];
    r.b[0] = (float)0.99886 * r.b[0] + x * (float)0.0555179;
    r.b[1] = (float)0.99332 * r.b[1] + x * (float)0.0750759;
    r.b[2] = (float)0.96900 * r.b[2] + x * (float)0.1538520;
    r.b[3] = (float)0.86650 * r.b[3] + x * (float)0.3104856;
    r.b[4] = (float)0.55000 * r.b[4] + x * (float)0.5329522;
    r.b[5] = (float)-0.7616 * r.b[5] - x * (float)0.0168980;
    o.v[0] = (r.b[0] + r.b[1] + r.b[2] + r.b[3] + r.b[4] + r.b[5] + r.b[6] + x * (float)0.5362) * (float)0.115830421;
    r.b[6] = x * (float)0.115926;
  }
  static FDSP_DEV void end_simd(R&) {}
};

// ---------------------------------------------------------------- Declick<f32> (src/dynamics.rs:245-315, ID 23)
// smooth5 fade-in over the first `duration` seconds. The block path accumulates the fade phase inside the block and advances the
// time by the whole block at once (process :287-307, which also covers the tail samples); tick recomputes the phase from t.
FDSP_DEV float smooth5f(float x) { return ((x * 6.0f - 15.0f) * x + 10.0f) * x * x * x; }
struct Declick {
  FDSP_NODE(1, 1, 1, 1, 0);
  struct R { float duration, t, phase, phase_d, end_time; int end_index; };
  static FDSP_DEV void load(R& r, Loader& l) { r.duration = l.Pf(); r.t = l.Sf(); r.phase = r.phase_d = r.end_time = 0.0f; r.end_index = 0; }
  static FDSP_DEV void save(const R& r, Saver& s) { s.Sf(r.t); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<1>& in, Fr<1>& o) {
    if (T) {
      if (r.t < r.duration) { const float phase = (r.t - 0.0f) / (r.duration - 0.0f); o.v[0] = in.v[0] * smooth5f(phase); r.t += c.sd64; }
      else o.v[0] = in.v[0];
      return;
    }
    if (c.i == 0) {   // block start: plan the fade for this block
      r.end_index = 0;
      if (r.t < r.duration) {
        r.phase = (r.t - 0.0f) / (r.duration - 0.0f);
        r.phase_d = c.sd64 / r.duration;
        r.end_time = r.t + (float)c.n * c.sd64;
        r.end_index = r.duration < r.end_time ? (int)ceilf((r.duration - r.t) / c.sd64) : c.n;
        r.t = r.end_time;
      }
    }
    if (c.i < r.end_index) { o.v[0] = in.v[0] * smooth5f(r.phase); r.phase += r.phase_d; }
    else o.v[0] = in.v[0];
  }
  static FDSP_DEV void end_simd(R&) {}
};

// ---------------------------------------------------------------- Follow (ID 24) / AFollow (ID 29), src/follow.rs
// Three one-pole smoothers in series; coefficients (host: halfway_coeff) are 1 for the very first sample after a reset.
template <int ASYM> struct Follower {
  FDSP_NODE(1, 1, 2, 5, 0);
  struct R { float ac, rc, anow, rnow, v1, v2, v3; };
  static FDSP_DEV void load(R& r, Loader& l) { r.ac = l.Pf(); r.rc = l.Pf(); r.anow = l.Sf(); r.rnow = l.Sf(); r.v1 = l.Sf(); r.v2 = l.Sf(); r.v3 = l.Sf(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.Sf(r.anow); s.Sf(r.rnow); s.Sf(r.v1); s.Sf(r.v2); s.Sf(r.v3); }
  static FDSP_DEV float pole2(float in, float cur, float a, float rr) { return cur + fmaxf(0.0f, in - cur) * a - fmaxf(0.0f, cur - in) * rr; }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<1>& in, Fr<1>& o) {
    if (ASYM) {
      r.v1 = pole2(in.v[0], r.v1, r.anow, r.rnow); r.v2 = pole2(r.v1, r.v2, r.anow, r.rnow); r.v3 = pole2(r.v2, r.v3, r.anow, r.rnow);
    } else {
      const float k = 1.0f - r.anow;
      r.v1 = r.anow * in.v[0] + k * r.v1; r.v2 = r.anow * r.v1 + k * r.v2; r.v3 = r.anow * r.v2 + k * r.v3;
    }
    r.anow = r.ac; r.rnow = r.rc;
    o.v[0] = r.v3;
  }
  static FDSP_DEV void end_simd(R&) {}
};

// ---------------------------------------------------------------- Shaper<S> (src/shape.rs, ID 42)
// KIND 0 Clip(h), 1 ClipTo(lo, hi), 2 Tanh(h), 3 Softsign(h), 4 Crush(levels), 5 SoftCrush(levels), 6 Atan(h) with p0 = h * PI * 0.5
// (folded on the host, src/shape.rs:97-103); the block path follows Shape::simd (round-to-even, F32x::floor, |x|*h, wide's atan), tail
// and tick follow Shape::shape.
FDSP_DEV float smooth9f(float x) { const float x2 = x * x; return ((((70.0f * x - 315.0f) * x + 540.0f) * x - 420.0f) * x + 126.0f) * x2 * x2 * x; }
template <int KIND> FDSP_DEV float shape_tick(float p0, float p1, float x) {   // Shape::shape (src/shape.rs), per shape kind
  if (KIND == 6) return m::atanf_(x * p0) * (2.0f / PI_F);
  if (KIND == 0) return fminf(fmaxf(x * p0, -1.0f), 1.0f);
  if (KIND == 1) return fminf(fmaxf(x, p0), p1);
  if (KIND == 2) return m::tanhf_(x * p0);
  if (KIND == 3) return (x * p0) / (1.0f + fabsf(x * p0));
  if (KIND == 4) return roundf(x * p0) / p0;
  const float v = x * p0, fl = floorf(v);
  return (fl + smooth9f(v - fl)) / p0;
}
template <int KIND> struct Shaper {
  FDSP_NODE(1, 1, 2, 0, 0);
  struct R { float p0, p1; };
  static FDSP_DEV void load(R& r, Loader& l) { r.p0 = l.Pf(); r.p1 = l.Pf(); }
  static FDSP_DEV void save(const R&, Saver&) {}
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<1>& in, Fr<1>& o) {
    const float x = in.v[0];
    const bool tick = T || c.rem;
    float y;
    if (KIND == 0) y = fminf(fmaxf(x * r.p0, -1.0f), 1.0f);
    else if (KIND == 1) y = fminf(fmaxf(x, r.p0), r.p1);
    else if (KIND == 2) y = m::tanhf_(x * r.p0);
    else if (KIND == 3) y = tick ? (x * r.p0) / (1.0f + fabsf(x * r.p0)) : x * r.p0 / (1.0f + fabsf(x) * r.p0);
    else if (KIND == 4) y = (tick ? roundf(x * r.p0) : wide_roundf(x * r.p0)) / r.p0;
    else if (KIND == 6) y = (tick ? m::atanf_(x * r.p0) : wide_atanf(x * r.p0)) * (2.0f / PI_F);
    else { const float v = x * r.p0, fl = tick ? floorf(v) : wide_floorf(v); y = (fl + smooth9f(v - fl)) / r.p0; }
    o.v[0] = y;
  }
  static FDSP_DEV void end_simd(R&) {}
};
// Shaper<Adaptive<S>> (src/shape.rs:156-200, ID 42): the level estimate `state` follows smoothing * state + (1 - smoothing) * (1e-6 + x^2)
// and the inner shape INNER (0..6 as above) sees x / sqrt(state). Adaptive::simd is the trait default (lane by lane through `shape`), so
// the inner shape takes its tick form on both paths. Words: P smoothing, p0, p1; S state (0.0 after construction, 1e-3 after reset()).
FDSP_DEV float adaptive_level(float smoothing, float state, float x) { return smoothing * state + (1.0f - smoothing) * (1.0e-6f + x * x); }
template <int INNER> struct ShaperAdaptive {
  FDSP_NODE(1, 1, 3, 1, 0);
  struct R { float sm, p0, p1, st; };
  static FDSP_DEV void load(R& r, Loader& l) { r.sm = l.Pf(); r.p0 = l.Pf(); r.p1 = l.Pf(); r.st = l.Sf(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.Sf(r.st); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<1>& in, Fr<1>& o) {
    const float x = in.v[0];
    r.st = adaptive_level(r.sm, r.st, x);
    o.v[0] = shape_tick<INNER>(r.p0, r.p1, x / sqrtf(r.st));
  }
  static FDSP_DEV void end_simd(R&) {}
};
// Nonlinear biquads (src/biquad.rs:494-920): transposed direct form II with a waveshaper in the loop.
//   FB = 1: FbBiquad (ID 88) / FixedFbBiquad (ID 90): feedback is shape(y0);  FB = 0: DirtyBiquad (89) / FixedDirtyBiquad (91):
//   both state updates are shaped, by two clones of the shape (shape1 for s1, then shape2 for s2, src/biquad.rs:711-720, :780-795).
//   MODE 0 resonator, 1 lowpass, 2 highpass, 3 bell; NIN 1 = fixed coefficients, 3 / 4 = audio-rate (center, q[, gain]) with the
//   reference's change test squared(dc) + squared(dq) [+ squared(dg)] != 0. The shape SH is evaluated on its tick path:
//   BqShape<KIND>: a Shaper kind (0..6) with its words p0, p1;
//   BqShapeAdaptive<INNER>: Adaptive around a Shaper kind, words smoothing, p0, p1 and one level estimate per clone. The biquads'
//   set_sample_rate does not reach the shape (:536-539, :745-748), so `smoothing` is the one Adaptive::new computed at 44.1 kHz.
//   A rate change recomputes the audio-rate coefficients at the next sample (`ksr`, as in Svf).
// Words: P shape words [, a1, a2, b0, b1, b2 for NIN 1]; S [center, q, gain, ksr, a1, a2, b0, b1, b2 for NIN > 1], s1, s2, shape1 [, shape2] state.
template <int KIND> struct BqShape {
  static constexpr int NP = 2, NS = 0;
  struct P { float p0, p1; };
  struct S {};
  static FDSP_DEV void load_p(P& p, Loader& l) { p.p0 = l.Pf(); p.p1 = l.Pf(); }
  static FDSP_DEV void load_s(S&, Loader&) {}
  static FDSP_DEV void save_s(const S&, Saver&) {}
  static FDSP_DEV float shape(const P& p, S&, float x) { return shape_tick<KIND>(p.p0, p.p1, x); }
};
template <int INNER> struct BqShapeAdaptive {
  static constexpr int NP = 3, NS = 1;
  struct P { float sm, p0, p1; };
  struct S { float st; };
  static FDSP_DEV void load_p(P& p, Loader& l) { p.sm = l.Pf(); p.p0 = l.Pf(); p.p1 = l.Pf(); }
  static FDSP_DEV void load_s(S& s, Loader& l) { s.st = l.Sf(); }
  static FDSP_DEV void save_s(const S& s, Saver& sv) { sv.Sf(s.st); }
  static FDSP_DEV float shape(const P& p, S& s, float x) { s.st = adaptive_level(p.sm, s.st, x); return shape_tick<INNER>(p.p0, p.p1, x / sqrtf(s.st)); }
};
template <int FB, int MODE, class SH, int NIN> struct NlBiquadT {
  FDSP_NODE(NIN, 1, SH::NP + (NIN == 1 ? 5 : 0), 2 + (NIN > 1 ? 9 : 0) + (FB ? 1 : 2) * SH::NS, 0);
  struct R { typename SH::P sp; BqCoefs k; float center, q, gain, ksr, s1, s2; typename SH::S sh1, sh2; };
  static FDSP_DEV void load(R& r, Loader& l) {
    SH::load_p(r.sp, l);
    if (NIN == 1) { r.k.a1 = l.Pf(); r.k.a2 = l.Pf(); r.k.b0 = l.Pf(); r.k.b1 = l.Pf(); r.k.b2 = l.Pf(); r.center = r.q = r.gain = r.ksr = 0.0f; }
    else { r.center = l.Sf(); r.q = l.Sf(); r.gain = l.Sf(); r.ksr = l.Sf(); r.k.a1 = l.Sf(); r.k.a2 = l.Sf(); r.k.b0 = l.Sf(); r.k.b1 = l.Sf(); r.k.b2 = l.Sf(); }
    r.s1 = l.Sf(); r.s2 = l.Sf();
    SH::load_s(r.sh1, l); if (!FB) SH::load_s(r.sh2, l);
  }
  static FDSP_DEV void save(const R& r, Saver& s) {
    if (NIN > 1) { s.Sf(r.center); s.Sf(r.q); s.Sf(r.gain); s.Sf(r.ksr); s.Sf(r.k.a1); s.Sf(r.k.a2); s.Sf(r.k.b0); s.Sf(r.k.b1); s.Sf(r.k.b2); }
    s.Sf(r.s1); s.Sf(r.s2);
    SH::save_s(r.sh1, s); if (!FB) SH::save_s(r.sh2, s);
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<NIN>& in, Fr<1>& o) {
    if (NIN > 1) {
      const float ce = in.v[NIN > 1 ? 1 : 0], qq = in.v[NIN > 2 ? 2 : 0], gg = NIN > 3 ? in.v[NIN > 3 ? 3 : 0] : r.gain;
      const float dc = ce - r.center, dq = qq - r.q, dg = gg - r.gain;
      const float test = NIN > 3 ? dc * dc + dq * dq + dg * dg : dc * dc + dq * dq;
      if (r.ksr != c.sr) { r.ksr = c.sr; r.k = bq_mode(MODE, c.sr, r.center, r.q, r.gain); }
      if (test != 0.0f) { r.center = ce; r.q = qq; r.gain = gg; r.k = bq_mode(MODE, c.sr, ce, qq, gg); }
    }
    const float x0 = in.v[0];
    const float y0 = r.k.b0 * x0 + r.s1;
    if (FB) {
      const float fb = SH::shape(r.sp, r.sh1, y0);
      r.s1 = r.s2 + r.k.b1 * x0 - fb * r.k.a1;
      r.s2 = r.k.b2 * x0 - fb * r.k.a2;
    } else {
      r.s1 = SH::shape(r.sp, r.sh1, r.s2 + r.k.b1 * x0 - y0 * r.k.a1);
      r.s2 = SH::shape(r.sp, r.sh2, r.k.b2 * x0 - y0 * r.k.a2);
    }
    o.v[0] = y0;
  }
  static FDSP_DEV void end_simd(R&) {}
};
template <int FB, int MODE, int SHAPE, int NIN> struct NlBiquad : NlBiquadT<FB, MODE, BqShape<SHAPE>, NIN> {};
template <int FB, int MODE, int INNER, int NIN> struct NlBiquadAdaptive : NlBiquadT<FB, MODE, BqShapeAdaptive<INNER>, NIN> {};

// ---------------------------------------------------------------- Convolver (src/convolve.rs:9-59, ID 100)
// Direct-form linear convolution with an impulse response shared by the voice class (class-uniform words: K, ring length,
// then h[0..K)); input history in a power-of-two HBM ring per voice. The block path produces 8 outputs per pass over the
// window, so every history sample is loaded once per 8 outputs and meets a sliding register window of 8 coefficients.
// The reference computes the same sum with a partitioned FFT (fft-convolver), so this node is tolerance-, not bit-checked;
// FMA is therefore allowed here, and both paths accumulate in the same order (k ascending), so tick == process exactly.
struct Convolver {
  FDSP_NODE(1, 1, 0, 1, 2);   // NU counts the two header words; the K coefficient words follow them in the uniform block
  struct R { uint32_t K, len, off, i; const uint32_t* h; };
  static FDSP_DEV void load(R& r, Loader& l) { r.K = l.U(); r.len = l.U(); r.h = l.u + l.ui; l.ui += r.K; r.off = l.D(r.len); r.i = l.S(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.S(r.i); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<1>& in, Fr<1>& o) {
    const uint32_t mask = r.len - 1u;
    float* ring = c.dl + (size_t)r.off * c.V + c.v;
    ring[(size_t)r.i * c.V] = in.v[0];
    float acc = 0.0f;
#pragma unroll 4
    for (uint32_t k = 0; k < r.K; k++) acc = __fmaf_rn(__uint_as_float(__ldg(r.h + k)), ring[(size_t)((r.i - k) & mask) * c.V], acc);
    r.i = (r.i + 1u) & mask;
    o.v[0] = acc;
  }
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C& c, const Fr8<1>& in, Fr8<1>& o) {
    const uint32_t mask = r.len - 1u;
    float* ring = c.dl + (size_t)r.off * c.V + c.v;
#pragma unroll
    for (int j = 0; j < 8; j++) ring[(size_t)((r.i + (uint32_t)j) & mask) * c.V] = in.v[0][j];
    // Window position m holds x[t0 + 7 - m] and meets output j with coefficient k = j - 7 + m. The window is walked 8 positions
    // at a time: 8 independent ring loads in flight, then 64 FMAs against the 15 coefficients hw[t] = h[m0 - 7 + t] that
    // this chunk can touch (7 carried over, 8 loaded). acc[j] still accumulates in ascending k, exactly like `step`.
    float acc[8], hw[15];
#pragma unroll
    for (int j = 0; j < 8; j++) acc[j] = 0.0f;
#pragma unroll
    for (int t = 0; t < 15; t++) hw[t] = (t >= 7 && (uint32_t)(t - 7) < r.K) ? __uint_as_float(__ldg(r.h + (t - 7))) : 0.0f;
    const uint32_t last = r.i + 7u, M = r.K + 7u;
#pragma unroll 2
    for (uint32_t m0 = 0; m0 < M; m0 += 8u) {
      float xv[8];
#pragma unroll
      for (int q = 0; q < 8; q++) xv[q] = ring[(size_t)((last - m0 - (uint32_t)q) & mask) * c.V];
#pragma unroll
      for (int q = 0; q < 8; q++) {
#pragma unroll
        for (int j = 0; j < 8; j++) acc[j] = __fmaf_rn(hw[j + q], xv[q], acc[j]);
      }
#pragma unroll
      for (int t = 0; t < 7; t++) hw[t] = hw[t + 8];
#pragma unroll
      for (int t = 7; t < 15; t++) { const uint32_t k = m0 + 1u + (uint32_t)t; hw[t] = k < r.K ? __uint_as_float(__ldg(r.h + k)) : 0.0f; }
    }
#pragma unroll
    for (int j = 0; j < 8; j++) o.v[0][j] = acc[j];
    r.i = (r.i + 8u) & mask;
  }
  static FDSP_DEV void end_simd(R&) {}
};

// ---------------------------------------------------------------- FeedbackUnit (src/feedback.rs:316-481, ID 79)
// Feedback with an integrated delay of `samples` >= 1: a block no longer than the delay runs the inner graph's BLOCK path on
// (input + output delayed by `samples`), a longer block ticks it. Per-channel power-of-two rings in HBM; uniform words:
// samples, ring length. The rings never alias inside a block-mode block (the read position trails the write by >= size).
template <class X> struct FeedbackUnit {
  static constexpr int N = X::IN;
  FDSP_NODE(N, N, X::NP, 1 + X::NS, 2 + X::NU);
  struct R { uint32_t samples, len, off, index; bool block; typename X::R x; };
  static FDSP_DEV void load(R& r, Loader& l) { r.samples = l.U(); r.len = l.U(); r.off = l.D(r.len * (uint32_t)N); r.index = l.S(); r.block = false; X::load(r.x, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.S(r.index); X::save(r.x, s); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<N>& in, Fr<N>& o) {
    const uint32_t mask = r.len - 1u;
    const uint32_t ri = (r.index + r.len - r.samples) & mask;
    Fr<N> t;
#pragma unroll
    for (int k = 0; k < N; k++) t.v[k] = in.v[k] + c.dl[(size_t)(r.off + (uint32_t)k * r.len + ri) * c.V + c.v];
    r.block = !T && (uint32_t)c.n <= r.samples;
    if (r.block) X::template step<false>(r.x, c, t, o); else X::template step<true>(r.x, c, t, o);
#pragma unroll
    for (int k = 0; k < N; k++) c.dl[(size_t)(r.off + (uint32_t)k * r.len + r.index) * c.V + c.v] = o.v[k];
    r.index = (r.index + 1u) & mask;
  }
  static FDSP_DEV void end_simd(R& r) { if (r.block) X::end_simd(r.x); }
};

// ---------------------------------------------------------------- Event<X>: ONE event of a Sequencer (src/sequencer.rs:768-843)
// as a voice. The reference's per-block scheduling arithmetic runs here, per voice, at the start of every block, in f64 like the
// reference: time += sample_duration * size; an event turns active when start_time < block_end - sample_duration / 2, ends when
// end_time <= time + sample_duration / 2; inside a block the unit renders samples [start_index, end_index) with ITS OWN process()
// of end_index - start_index samples (so its 8-sample groups and its tail are relative to start_index); fade-in / fade-out multiply
// the unit's buffer from the block-relative indices of :113-217, the fade value advancing by f32 addition. Nothing here needs the
// host per block, so a sequence renders in long launches. X is a generator (the span() of inputs is not reproduced).
FDSP_DEV float sine_ease_f(float x) {   // src/math.rs:453-458, T = f32
  const float pi = (float)3.141592653589793;
  x = x * (float)(3.141592653589793 * 0.5);
  return 16.0f * x * (pi - x) / ((float)(5.0 * 3.141592653589793 * 3.141592653589793) - 4.0f * x * (pi - x));
}
template <class X> struct Event {
  static constexpr int NO = X::OUT;
  static constexpr int NPE = 13, NSE = 7;   // the event's own parameter / state words, in front of X's
  static constexpr int NOSPLIT = 1 << 30;
  FDSP_NODE(0, NO, NPE + X::NP, NSE + X::NS, X::NU);
  struct R {
    double sr, sd, start, end, fin, fout, time; int ease, status;   // status 0 ready, 1 active, 2 past
    // ReplayMode::Loop (src/sequencer.rs:219-229): lp = loop point in seconds (+inf: no loop); cs / ce = the event's CURRENT start / end, which a
    // wrap shifts back by lp while the event is sounding and the end of the event restores to start / end (the original times, :622-639)
    double lp, cs, ce;
    int s_idx, n_v, nfull_v, fi_end, fo_i, fo_end; float fi_cur, fi_d, fo_cur, fo_d; bool fi_on, fo_on;
    bool whole;   // this block: the event spans it entirely and no fade touches it -> X runs its own 8-sample group form (step8)
    int split;    // loop: index inside this block at which the sequencer wraps (NOSPLIT: it does not)
    bool silent;  // the rest of a block after the wrap is rendered into a scratch buffer by the reference (:845-872 as written): state advances, output stays 0
    typename X::R x;
  };
  static FDSP_DEV double ld64(Loader& l, bool state) {
    const uint32_t lo = state ? l.S() : l.P(), hi = state ? l.S() : l.P();
    return __longlong_as_double((long long)(((unsigned long long)hi << 32) | lo));
  }
  static FDSP_DEV void st64(Saver& s, double v) { const unsigned long long b = (unsigned long long)__double_as_longlong(v); s.S((uint32_t)b); s.S((uint32_t)(b >> 32)); }
  static FDSP_DEV bool looped(const R& r) { return r.lp < 1.0e300; }
  static FDSP_DEV void load(R& r, Loader& l) {
    r.sr = ld64(l, false); r.start = ld64(l, false); r.end = ld64(l, false); r.fin = ld64(l, false); r.fout = ld64(l, false); r.ease = (int)l.P();
    r.lp = ld64(l, false);
    r.sd = 1.0 / r.sr;
    r.time = ld64(l, true); r.status = (int)l.S(); r.cs = ld64(l, true); r.ce = ld64(l, true);
    r.s_idx = r.n_v = r.nfull_v = r.fi_end = r.fo_i = r.fo_end = 0; r.fi_cur = r.fi_d = r.fo_cur = r.fo_d = 0.0f; r.fi_on = r.fo_on = false; r.whole = false;
    r.split = NOSPLIT; r.silent = false;
    X::load(r.x, l);
  }
  static FDSP_DEV void save(const R& r, Saver& s) {
    st64(s, r.time); s.S((uint32_t)r.status); st64(s, r.cs); st64(s, r.ce); X::save(r.x, s);
  }
  static FDSP_DEV int as_index(double x) { return x > 0.0 ? (x < 1.0e9 ? (int)x : 1000000000) : 0; }   // `as usize`, saturating
  // `unit.reset()` of a finished event in a replaying sequencer (:631-633): X back to its construction-time words (the class's reset image),
  // its delay lines cleared. Only looping events get here on the device (ReplayMode::All resets the whole bank from the host).
  template <class C> static FDSP_DEV void reset_x(R& r, const C& c) {
    Loader l{c.rp, c.rs0, c.ru, c.V, c.v, (uint32_t)NPE, (uint32_t)NSE, 0u, 0u};
    X::load(r.x, l);
    for (uint32_t k = 0; k < c.dl_total; k++) c.dl[(size_t)k * c.V + c.v] = 0.0f;
  }
  // Sequencer::process (:768-843) for this event over `n` samples that begin at index `off` of the kernel's block
  template <class C> static FDSP_DEV void plan(R& r, const C& c, int n, int off, bool silent) {
    const bool lo = looped(r);
    const double end_blk = lo ? fmin(r.time + r.sd * (double)n, r.lp) : r.time + r.sd * (double)n;
    if (r.status == 0 && (lo ? r.cs : r.start) < end_blk - r.sd * 0.5) r.status = 1;    // ready_to_active
    const int loop_size = lo ? as_index(round(fmax(0.0, r.lp - r.time) * r.sr)) : n;
    r.n_v = 0; r.s_idx = off; r.nfull_v = 0; r.fi_on = r.fo_on = false; r.whole = false; r.silent = silent;
    if (r.status == 1) {
      const double st = lo ? r.cs : r.start, en = lo ? r.ce : r.end;
      if (en <= r.time + 0.5 * r.sd) {                                                  // end_of_event
        if (lo) { r.cs = r.start; r.ce = r.end; reset_x(r, c); r.status = r.cs >= r.time ? 0 : 2; }
        else r.status = 2;
      } else {
        const int s = st <= r.time ? 0 : as_index(round((st - r.time) * r.sr));
        const int lim = n < loop_size ? n : loop_size;
        const int e0 = en >= end_blk ? lim : as_index(round((en - r.time) * r.sr));
        const int e = en >= end_blk ? lim : (e0 < loop_size ? e0 : loop_size);
        if (e > s) {
          r.s_idx = off + s; r.n_v = e - s; r.nfull_v = (e - s) & ~7;
          const double fe = st + r.fin;
          if (r.fin > 0.0 && fe > r.time) {                                            // fade_in :113-160
            r.fi_on = true;
            r.fi_end = fe >= end_blk ? e : as_index(round((fe - r.time) / r.sd));
            r.fi_cur = (float)(((r.time + (double)s * r.sd) - st) / (fe - st));
            r.fi_d = (float)(r.sd / r.fin);
          }
          const double fs = en - r.fout;
          if (r.fout > 0.0 && fs < end_blk) {                                          // fade_out :162-217
            r.fo_on = true;
            r.fo_i = fs <= r.time ? 0 : as_index(round((fs - r.time) / r.sd));
            r.fo_cur = (float)(((r.time + (double)r.fo_i * r.sd) - fs) / (en - fs));
            r.fo_d = (float)(r.sd / r.fout);
            r.fo_end = e;
          }
        }
      }
    }
    r.whole = r.n_v == n && off == 0 && !silent && !r.fi_on && !r.fo_on;
    r.time = end_blk;
    r.split = loop_size < n ? off + loop_size : NOSPLIT;
  }
  // first sample of a kernel block: plan it; the sample at which the loop wraps: Sequencer::reset in loop mode (:642-683 — sounding events
  // move back by the loop period, past events become ready again, time restarts) and the plan of the rest of the block, which the reference
  // renders into a scratch buffer (a loop is at least 64 samples, so a block wraps at most once)
  template <class C> static FDSP_DEV void at_sample(R& r, const C& c) {
    if (c.i == 0) plan(r, c, c.n, 0, false);
    if (c.i == r.split) {
      const int off = r.split;
      if (r.status == 1) { r.cs -= r.lp; r.ce -= r.lp; } else if (r.status == 2) r.status = 0;
      r.time = 0.0;
      plan(r, c, c.n - off, off, true);
    }
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<0>& in, Fr<NO>& o) {
    if (T) { X::template step<true>(r.x, c, in, o); return; }   // (an event is always the root of a voice: not reached)
    at_sample(r, c);
    step_planned(r, c, in, o);
  }
  template <class C> static FDSP_DEV void step_planned(R& r, const C& c, const Fr<0>& in, Fr<NO>& o) {
    const int b = c.i - r.s_idx;
    if (b >= 0 && b < r.n_v) {
      C c2 = c;
      c2.n = r.n_v; c2.i = b; c2.rem = b >= r.nfull_v; c2.first = !c2.rem && (b & 7) == 0;
      if (b == r.nfull_v && !r.whole) X::end_simd(r.x);           // the unit's own block: SIMD part done, tail through its tick path
      X::template step<false>(r.x, c2, in, o);                    // (a whole block: the kernel's end_simd call reaches X through end_simd below)
      if (b == r.n_v - 1 && r.nfull_v == r.n_v && !r.whole) X::end_simd(r.x); // no tail
      float g = 1.0f; bool scaled = false;
      if (r.fi_on && b < r.fi_end) { g = r.ease == 0 ? sine_ease_f(r.fi_cur) : smooth5f(r.fi_cur); r.fi_cur += r.fi_d; scaled = true; }
      if (scaled) {
#pragma unroll
        for (int k = 0; k < NO; k++) o.v[k] *= g;
      }
      if (r.fo_on && b >= r.fo_i && b < r.fo_end) {
        const float h = r.ease == 0 ? sine_ease_f(1.0f - r.fo_cur) : smooth5f(1.0f - r.fo_cur); r.fo_cur += r.fo_d;
#pragma unroll
        for (int k = 0; k < NO; k++) o.v[k] *= h;
      }
      if (r.silent) {
#pragma unroll
        for (int k = 0; k < NO; k++) o.v[k] = 0.0f;
      }
    } else {
#pragma unroll
      for (int k = 0; k < NO; k++) o.v[k] = 0.0f;
    }
  }
  // Steady state of a note — the block lies inside the event and outside its fades — is X's own group form at full speed; every
  // other block (start, end, fades, silence) takes the per-sample path above. The plan is made by the block's first group.
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C& c, const Fr8<0>& in, Fr8<NO>& o) {
    at_sample(r, c);
    if (r.whole) { group_step<X>(r.x, c, in, o); return; }
    if (r.n_v == 0 && r.split == NOSPLIT) {
#pragma unroll
      for (int k = 0; k < NO; k++) {
#pragma unroll
        for (int j = 0; j < 8; j++) o.v[k][j] = 0.0f;
      }
      return;
    }
    const int base = c.i;
    const bool planned = true;
    (void)planned;
#pragma unroll 1
    for (int j = 0; j < 8; j++) {
      Fr<0> none; Fr<NO> y;
      c.i = base + j; c.first = (j == 0);
      if (j > 0 && c.i == r.split) at_sample(r, c);
      step_planned(r, c, none, y);
#pragma unroll
      for (int k = 0; k < NO; k++) {
#pragma unroll
        for (int q = 0; q < 7; q++) o.v[k][q] = o.v[k][q + 1];
        o.v[k][7] = y.v[k];
      }
    }
    c.i = base; c.first = true;
  }
  static FDSP_DEV void end_simd(R& r) { if (r.whole) X::end_simd(r.x); }
};

// ---------------------------------------------------------------- Oversample<X> (Oversampler ID 51, src/oversample.rs): X at twice
// the sample rate between two 43-tap minimum-phase halfband filters (24-tap polyphase interpolation, 48-tap decimation), the
// reference's arithmetic as written: 8 lane accumulators per filter (`mul_add` = mul, add — the crate's non-FMA form), lanes summed
// ((l0+l2)+(l1+l3)) low + high. The 128-sample rings of every input and output channel live in the class's delay-line storage. In a
// block the inner program runs ITS block path twice over `size` inner samples (one per half of the outer block); with an odd size the
// last outer sample is 0 and the inner program consumes one zero-input sample per half (see oracle/fo_nodes.h Oversampler).
FDSP_DEV float os_tap(int k) {   // HALFBAND_MIN (:344-388); k is a compile-time constant wherever this is called
  const float h[43] = {4.73552339e-02f, 1.81988040e-01f, 3.49148434e-01f, 3.92748135e-01f, 2.18230867e-01f, -5.31842843e-02f, -1.79186566e-01f, -7.34488007e-02f,
                       8.94524103e-02f, 1.00868556e-01f, -2.08681451e-02f, -8.82510989e-02f, -2.07640777e-02f, 6.22587555e-02f, 4.07776255e-02f, -3.52258090e-02f,
                       -4.57407870e-02f, 1.27033444e-02f, 4.14376136e-02f, 3.30799834e-03f, -3.24608206e-02f, -1.27856355e-02f, 2.21659033e-02f, 1.67803711e-02f,
                       -1.27406974e-02f, -1.68177367e-02f, 5.35518220e-03f, 1.44761581e-02f, -3.70651781e-04f, -1.11140183e-02f, -2.40622311e-03f, 7.71596027e-03f,
                       3.48227062e-03f, -4.86763558e-03f, -3.45536353e-03f, 2.79880054e-03f, 2.86736431e-03f, -1.48746153e-03f, -2.11827989e-03f, 7.72684113e-04f,
                       1.44384114e-03f, -4.49807048e-04f, -9.41945265e-04f};
  return h[k];
}
FDSP_DEV float os_reduce8(const float* a) { return ((a[0] + a[2]) + (a[1] + a[3])) + ((a[4] + a[6]) + (a[5] + a[7])); }
template <class X> struct Oversample {
  static constexpr int NI = X::IN, NO = X::OUT, NC = NI < NO ? NI : NO;
  FDSP_NODE(NI, NO, X::NP, 2 + X::NS, X::NU);
  struct R { uint32_t in_idx, out_idx, off; typename X::R x; };
  static FDSP_DEV void load(R& r, Loader& l) { r.in_idx = l.S(); r.out_idx = l.S(); r.off = l.D(128u * (uint32_t)(NI + NO)); X::load(r.x, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.S(r.in_idx); s.S(r.out_idx); X::save(r.x, s); }
  template <class C> static FDSP_DEV float* ring(const R& r, const C& c, int channel) { return c.dl + (size_t)(r.off + (uint32_t)channel * 128u) * c.V + c.v; }
  template <class C> static FDSP_DEV void interpolate(const float* rb, const C& c, uint32_t newest, float& even, float& odd) {   // :12-44
    const uint32_t start = newest + (129u - 24u);
    float ae[8], ao[8];
#pragma unroll
    for (int j = 0; j < 8; j++) { ae[j] = 0.0f; ao[j] = 0.0f; }
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const int k = i * 8 + j;
        const float sm = rb[(size_t)((start + (uint32_t)k) & 0x7fu) * c.V];
        ae[j] = sm * (k < 2 ? 0.0f : os_tap(k < 2 ? 0 : 2 * (k - 2))) + ae[j];
        ao[j] = sm * (k < 3 ? 0.0f : os_tap(k < 3 ? 0 : 2 * (k - 3) + 1)) + ao[j];
      }
    }
    even = os_reduce8(ae) * 2.0f; odd = os_reduce8(ao) * 2.0f;
  }
  template <class C> static FDSP_DEV float decimate(const float* rb, const C& c, uint32_t last) {   // :46-66
    const uint32_t start = last + (129u - 48u);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; j++) acc[j] = 0.0f;
#pragma unroll
    for (int i = 0; i < 6; i++) {
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const int k = i * 8 + j;
        acc[j] = rb[(size_t)((start + (uint32_t)k) & 0x7fu) * c.V] * (k < 5 ? 0.0f : os_tap(k < 5 ? 0 : k - 5)) + acc[j];
      }
    }
    return os_reduce8(acc);
  }
  template <class C> static FDSP_DEV void inner(R& r, const C& c, int idx, int n, const Fr<NI>& in, Fr<NO>& y) {   // one sample of X's own block of n samples
    C c2 = c;
    const int nfull = n & ~7;
    c2.n = n; c2.i = idx; c2.rem = idx >= nfull; c2.first = !c2.rem && (idx & 7) == 0;
    c2.sr = c.sr * 2.0f; c2.sd64 = c.sd64 * 0.5f; c2.sd32 = c.sd32 * 0.5f;   // X runs at twice the rate (exact: powers of two)
    if (idx == nfull) X::end_simd(r.x);
    X::template step<false>(r.x, c2, in, y);
    if (idx == n - 1 && nfull == n) X::end_simd(r.x);
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<NI>& in, Fr<NO>& o) {
    Fr<NI> e, d; Fr<NO> y0, y1;
    const bool live = T || c.i < 2 * (c.n / 2);
    if (!live) {   // the odd tail sample of a block
      if (c.n == 1) {   // process(1): both halves are empty, and each still runs X's process(1) over its one zero inner sample
        Fr<NI> z; Fr<NO> drop;
#pragma unroll
        for (int k = 0; k < NI; k++) z.v[k] = 0.0f;
        inner(r, c, 0, 1, z, drop);
        inner(r, c, 0, 1, z, drop);
      }
#pragma unroll
      for (int k = 0; k < NO; k++) o.v[k] = 0.0f;
      return;
    }
#pragma unroll
    for (int k = 0; k < NI; k++) {
      float* rb = ring(r, c, k);
      rb[(size_t)r.in_idx * c.V] = in.v[k];
      interpolate(rb, c, r.in_idx, e.v[k], d.v[k]);
    }
    r.in_idx = (r.in_idx + 1u) & 0x7fu;
    if (T) {
      C c2 = c; c2.sr = c.sr * 2.0f; c2.sd64 = c.sd64 * 0.5f; c2.sd32 = c.sd32 * 0.5f;
      X::template step<true>(r.x, c2, e, y0); X::template step<true>(r.x, c2, d, y1);
    }
    else {
      const int half = c.n / 2, local = c.i >= half ? c.i - half : c.i;
      inner(r, c, 2 * local, c.n, e, y0);
      inner(r, c, 2 * local + 1, c.n, d, y1);
      if ((c.n & 1) && local == half - 1) {   // process(size) of an odd size: one inner sample more, fed from the zeroed buffer
        Fr<NI> z; Fr<NO> drop;
#pragma unroll
        for (int k = 0; k < NI; k++) z.v[k] = 0.0f;
        inner(r, c, c.n - 1, c.n, z, drop);
      }
    }
    const uint32_t next = (r.out_idx + 1u) & 0x7fu;
#pragma unroll
    for (int k = 0; k < NO; k++) {
      if (T || k < NC) {   // the block path decimates `Inputs` channels (:207)
        float* rb = ring(r, c, NI + k);
        rb[(size_t)r.out_idx * c.V] = y0.v[k];
        rb[(size_t)next * c.V] = y1.v[k];
        o.v[k] = decimate(rb, c, next);
      } else o.v[k] = 0.0f;
    }
    r.out_idx = (r.out_idx + 2u) & 0x7fu;
  }
  static FDSP_DEV void end_simd(R&) {}
};

// ---------------------------------------------------------------- Slot<X> (SlotBackend ID 78, src/slot.rs): a voice whose unit can be
// replaced by another unit OF THE SAME CLASS with a crossfade, without touching the program: two instances of X live in the voice, one
// current, one next; the host writes the next instance's words and arms the fade (fdsp_bank_slot_set), the device runs both through
// the block path, mixes them with the reference's per-block arithmetic (:205-262: phase_left, n, the fade advanced by f32 addition,
// f64 phase) and swaps their roles when the fade is over. The root of a voice only.
template <class X> struct Slot {
  static constexpr int NI = X::IN, NO = X::OUT;
  FDSP_NODE(NI, NO, 5 + 2 * X::NP, 4 + 2 * X::NS, 2 * X::NU);
  struct R {
    double sr, fade_time, fade_phase; int ease, which, has_next;
    int n_f; float fade, fade_d; bool swap_at_end;
    typename X::R u[2];
  };
  static FDSP_DEV double p64(Loader& l, bool state) {
    const uint32_t lo = state ? l.S() : l.P(), hi = state ? l.S() : l.P();
    return __longlong_as_double((long long)(((unsigned long long)hi << 32) | lo));
  }
  static FDSP_DEV void load(R& r, Loader& l) {
    r.sr = p64(l, false); r.fade_time = p64(l, false); r.ease = (int)l.P();
    r.which = (int)l.S(); r.has_next = (int)l.S(); r.fade_phase = p64(l, true);
    r.n_f = 0; r.fade = r.fade_d = 0.0f; r.swap_at_end = false;
    X::load(r.u[0], l); X::load(r.u[1], l);
  }
  static FDSP_DEV void save(const R& r, Saver& s) {
    s.S((uint32_t)r.which); s.S((uint32_t)r.has_next);
    const unsigned long long b = (unsigned long long)__double_as_longlong(r.fade_phase);
    s.S((uint32_t)b); s.S((uint32_t)(b >> 32));
    X::save(r.u[0], s); X::save(r.u[1], s);
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<NI>& in, Fr<NO>& o) {
    if (T) { if (r.which) X::template step<true>(r.u[1], c, in, o); else X::template step<true>(r.u[0], c, in, o); return; }   // (a slot is a root: not reached)
    if (c.i == 0 && r.has_next) {   // the block's crossfade plan
      const double span = r.fade_time * r.sr;
      const double left = (1.0 - r.fade_phase) * span;
      const int phase_left = left > 0.0 ? (left < 1.0e9 ? (int)left : 1000000000) : 0;
      r.n_f = c.n < phase_left ? c.n : phase_left;
      r.fade = (float)r.fade_phase; r.fade_d = (float)(1.0 / span);
      r.swap_at_end = phase_left <= c.n;
    }
    Fr<NO> y;
    if (r.which) X::template step<false>(r.u[1], c, in, o); else X::template step<false>(r.u[0], c, in, o);
    if (r.has_next) {
      if (r.which) X::template step<false>(r.u[0], c, in, y); else X::template step<false>(r.u[1], c, in, y);
      if (c.i < r.n_f) {
        const float e1 = r.ease == 0 ? sine_ease_f(1.0f - r.fade) : smooth5f(1.0f - r.fade);
        const float e2 = r.ease == 0 ? sine_ease_f(r.fade) : smooth5f(r.fade);
#pragma unroll
        for (int k = 0; k < NO; k++) { const float a = o.v[k] * e1; o.v[k] = a + y.v[k] * e2; }
        r.fade += r.fade_d;
      } else {
#pragma unroll
        for (int k = 0; k < NO; k++) o.v[k] = y.v[k];
      }
      if (c.i == c.n - 1) {
        r.fade_phase += (double)r.n_f / (r.fade_time * r.sr);
        if (r.swap_at_end) { r.which ^= 1; r.has_next = 0; r.fade_phase = 0.0; }   // next_phase (no `latest`: the host refuses a set while fading)
      }
    }
  }
  // No replacement pending: the current unit's own group form at full speed. A block with a fade runs both units per sample.
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C& c, const Fr8<NI>& in, Fr8<NO>& o) {
    if (!r.has_next) { if (r.which) group_step<X>(r.u[1], c, in, o); else group_step<X>(r.u[0], c, in, o); return; }
    const int base = c.i;
    Fr8<NI> ri = in;
#pragma unroll 1
    for (int j = 0; j < 8; j++) {
      Fr<NI> a; Fr<NO> y;
#pragma unroll
      for (int k = 0; k < NI; k++) a.v[k] = ri.v[k][0];
      c.i = base + j; c.first = (j == 0);
      step<false>(r, c, a, y);
#pragma unroll
      for (int k = 0; k < NI; k++) {
#pragma unroll
        for (int q = 0; q < 7; q++) ri.v[k][q] = ri.v[k][q + 1];
      }
#pragma unroll
      for (int k = 0; k < NO; k++) {
#pragma unroll
        for (int q = 0; q < 7; q++) o.v[k][q] = o.v[k][q + 1];
        o.v[k][7] = y.v[k];
      }
    }
    c.i = base; c.first = true;
  }
  static FDSP_DEV void end_simd(R& r) { X::end_simd(r.u[0]); X::end_simd(r.u[1]); }
};

// ---------------------------------------------------------------- Xfade<X, Y>: a Net vertex that crossfades from its unit X to a unit Y
// of ANY graph class (Net::crossfade, src/net.rs:480-504; the arithmetic of src/vertex.rs:138-229, all in f32: fade_phase, fade_time and the
// Net's f32 sample rate). While the fade runs both programs are evaluated (each through its own block path, like `unit.process` and
// `next.process`); afterwards the voice is Y alone (`next_phase`). The host builds this class around a RUNNING voice: X's state words and
// delay lines are carried over from the voice's old class (csrc/host/bank.cpp crossfade_voice).
template <class X, class Y> struct Xfade {
  static constexpr int NI = X::IN, NO = X::OUT;
  static_assert(X::IN == Y::IN && X::OUT == Y::OUT, "Net::crossfade: the replacement has the arity of the unit it replaces");
  FDSP_NODE(NI, NO, 3 + X::NP + Y::NP, 2 + X::NS + Y::NS, X::NU + Y::NU);
  struct R {
    float sr, fade_time, fade_phase; int ease, done;
    int n_f; float fade, fade_d; bool swap_at_end;
    typename X::R x; typename Y::R y;
  };
  static FDSP_DEV void load(R& r, Loader& l) {
    r.sr = l.Pf(); r.fade_time = l.Pf(); r.ease = (int)l.P();
    r.done = (int)l.S(); r.fade_phase = l.Sf();
    r.n_f = 0; r.fade = r.fade_d = 0.0f; r.swap_at_end = false;
    X::load(r.x, l); Y::load(r.y, l);
  }
  static FDSP_DEV void save(const R& r, Saver& s) { s.S((uint32_t)r.done); s.Sf(r.fade_phase); X::save(r.x, s); Y::save(r.y, s); }
  static FDSP_DEV float at(int ease, float x) { return ease == 0 ? sine_ease_f(x) : smooth5f(x); }   // Fade::at (src/sequencer.rs:48-55)
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<NI>& in, Fr<NO>& o) {
    if (T) { if (r.done) Y::template step<true>(r.y, c, in, o); else X::template step<true>(r.x, c, in, o); return; }   // (a vertex of a voice bank is a root: not reached)
    if (r.done) { Y::template step<false>(r.y, c, in, o); return; }
    if (c.i == 0) {   // the block's plan, vertex.rs:173-176
      const float left = (1.0f - r.fade_phase) * r.fade_time * r.sr;
      const int phase_left = left > 0.0f ? (left < 1.0e9f ? (int)left : 1000000000) : 0;   // `as usize`, saturating
      r.n_f = c.n < phase_left ? c.n : phase_left;
      r.fade = r.fade_phase; r.fade_d = 1.0f / (r.fade_time * r.sr);
      r.swap_at_end = phase_left <= c.n;
    }
    Fr<NO> y;
    X::template step<false>(r.x, c, in, o);
    Y::template step<false>(r.y, c, in, y);
    if (c.i < r.n_f) {   // x *= at(1 - fade); x += y * at(fade): two passes over the block in the reference, the same f32 fade sequence in both
      const float e1 = at(r.ease, 1.0f - r.fade), e2 = at(r.ease, r.fade);
#pragma unroll
      for (int k = 0; k < NO; k++) { const float a = o.v[k] * e1; o.v[k] = a + y.v[k] * e2; }
      r.fade += r.fade_d;
    } else {
#pragma unroll
      for (int k = 0; k < NO; k++) o.v[k] = y.v[k];
    }
    if (c.i == c.n - 1) {
      r.fade_phase += (float)r.n_f / (r.fade_time * r.sr);
      if (r.swap_at_end) { r.done = 1; r.fade_phase = 0.0f; }   // next_phase: the vertex's unit is Y from the next block on
    }
  }
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C& c, const Fr8<NI>& in, Fr8<NO>& o) {
    if (r.done) { group_step<Y>(r.y, c, in, o); return; }
    const int base = c.i;
    Fr8<NI> ri = in;
#pragma unroll 1
    for (int j = 0; j < 8; j++) {
      Fr<NI> a; Fr<NO> y;
#pragma unroll
      for (int k = 0; k < NI; k++) a.v[k] = ri.v[k][0];
      c.i = base + j; c.first = (j == 0);
      step<false>(r, c, a, y);
#pragma unroll
      for (int k = 0; k < NI; k++) {
#pragma unroll
        for (int q = 0; q < 7; q++) ri.v[k][q] = ri.v[k][q + 1];
      }
#pragma unroll
      for (int k = 0; k < NO; k++) {
#pragma unroll
        for (int q = 0; q < 7; q++) o.v[k][q] = o.v[k][q + 1];
        o.v[k][7] = y.v[k];
      }
    }
    c.i = base; c.first = true;
  }
  static FDSP_DEV void end_simd(R& r) { X::end_simd(r.x); Y::end_simd(r.y); }
};

// ---------------------------------------------------------------- Limiter<N> (ID 25, src/dynamics.rs:56-243): look-ahead limiter.
// A ring of L frames delays the audio; a binary max-tree over the last L amplitudes (ReduceBuffer, updated leaf-to-root per sample)
// gives the window peak, which an asymmetric follower smooths into the gain. Ring and tree live in the class's delay-line storage:
// every voice of a class has the same L and the same ring position, so all tree accesses of a warp are coalesced. Tick-only.
template <int N> struct Limiter {
  FDSP_NODE(N, N, 2, 7, 2);
  struct R { float ac, rc, anow, rnow, v1, v2, v3; uint32_t L, leaf, off, index, filled; };
  static FDSP_DEV void load(R& r, Loader& l) {
    r.L = l.U(); r.leaf = l.U(); r.ac = l.Pf(); r.rc = l.Pf();
    r.index = l.S(); r.filled = l.S(); r.anow = l.Sf(); r.rnow = l.Sf(); r.v1 = l.Sf(); r.v2 = l.Sf(); r.v3 = l.Sf();
    r.off = l.D((uint32_t)N * r.L + r.leaf + r.L + (r.L & 1u));
  }
  static FDSP_DEV void save(const R& r, Saver& s) { s.S(r.index); s.S(r.filled); s.Sf(r.anow); s.Sf(r.rnow); s.Sf(r.v1); s.Sf(r.v2); s.Sf(r.v3); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<N>& in, Fr<N>& o) {
    float* base = c.dl + (size_t)r.off * c.V + c.v;
    float* tree = base + (size_t)((uint32_t)N * r.L) * c.V;
    float amp = 0.0f;
#pragma unroll
    for (int k = 0; k < N; k++) amp = fmaxf(amp, fabsf(in.v[k]));
    uint32_t i = r.leaf + r.index;
    tree[(size_t)i * c.V] = amp;
    float cur = amp;
    while (i > 1u) {   // ReduceBuffer::set :106-114
      cur = fmaxf(cur, tree[(size_t)(i ^ 1u) * c.V]);
      i >>= 1;
      tree[(size_t)i * c.V] = cur;
    }
    const float total = cur;   // = buffer[1]
    if (r.filled < r.L) {      // filling the look-ahead: silence out
#pragma unroll
      for (int k = 0; k < N; k++) { base[(size_t)((uint32_t)k * r.L + r.index) * c.V] = in.v[k]; o.v[k] = 0.0f; }
      r.filled++;
      if (r.filled == r.L) { r.v1 = r.v2 = r.v3 = total; }   // start following from the buffer's peak
    } else {
      const float x = fmaxf(1.0f, total * 1.10f);            // leave some headroom
      r.v1 = Follower<1>::pole2(x, r.v1, r.anow, r.rnow); r.v2 = Follower<1>::pole2(r.v1, r.v2, r.anow, r.rnow); r.v3 = Follower<1>::pole2(r.v2, r.v3, r.anow, r.rnow);
      r.anow = r.ac; r.rnow = r.rc;
      const float g = 1.0f / r.v3;
#pragma unroll
      for (int k = 0; k < N; k++) {
        float* slot = base + (size_t)((uint32_t)k * r.L + r.index) * c.V;
        o.v[k] = *slot * g; *slot = in.v[k];
      }
    }
    r.index++; if (r.index >= r.L) r.index = 0u;
  }
  static FDSP_DEV void end_simd(R&) {}
};

// ---------------------------------------------------------------- MeterNode (ID 61, src/dynamics.rs:316-437), WavePlayer (ID 65,
// src/wave.rs:739-797), Resample<X> (ID 69, src/resample.rs:210-300). All three are tick-only in the reference.
template <int KIND> struct MeterNode {   // KIND 0 Sample, 1 Peak(timescale), 2 Rms(timescale); smoothing computed on the host in f64
  FDSP_NODE(1, 1, 1, 1, 0);
  struct R { float smoothing, state; };
  static FDSP_DEV void load(R& r, Loader& l) { r.smoothing = l.Pf(); r.state = l.Sf(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.Sf(r.state); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<1>& in, Fr<1>& o) {
    const float v = in.v[0];
    if (KIND == 0) { r.state = v; o.v[0] = v; }
    else if (KIND == 1) { r.state = fmaxf(r.state * r.smoothing, fabsf(v)); o.v[0] = r.state; }
    else { r.state = r.state * r.smoothing + (v * v) * (1.0f - r.smoothing); o.v[0] = sqrtf(r.state); }
  }
  static FDSP_DEV void end_simd(R&) {}
};

// ---------------------------------------------------------------- writers of a Shared: Monitor (ID 56, src/dynamics.rs:441-520), Timer (ID 57,
// src/shared.rs:203-250). Each leaves the value the reference would store last in a write-back state word of its own; the host stores
// it into the Shared after the call. Device code never touches the Shared itself.
template <int KIND> struct MonitorShared {   // the audio passes through; MeterNode<KIND>'s arithmetic on the input
  FDSP_NODE(1, 1, 1, 2, 0);
  struct R { typename MeterNode<KIND>::R m; };
  static FDSP_DEV void load(R& r, Loader& l) { MeterNode<KIND>::load(r.m, l); (void)l.S(); }
  // Meter::level: the state, or its square root for Rms (the block path of Meter::Sample ticks only the last sample, which leaves the same state)
  static FDSP_DEV void save(const R& r, Saver& s) { MeterNode<KIND>::save(r.m, s); s.Sf(KIND == 2 ? sqrtf(r.m.state) : r.m.state); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<1>& in, Fr<1>& o) {
    Fr<1> level;
    MeterNode<KIND>::template step<T>(r.m, c, in, level);
    o.v[0] = in.v[0];
  }
  static FDSP_DEV void end_simd(R&) {}
};
struct TimerShared {   // time += size * sample_duration once per block (Timer::process), += sample_duration per tick; stores time as f32
  FDSP_NODE(0, 0, 2, 3, 0);
  struct R { double sd, time; };
  static FDSP_DEV void load(R& r, Loader& l) {
    uint32_t lo = l.P(), hi = l.P(); r.sd = __longlong_as_double((long long)(((unsigned long long)hi << 32) | lo));
    lo = l.S(); hi = l.S(); r.time = __longlong_as_double((long long)(((unsigned long long)hi << 32) | lo));
    (void)l.S();
  }
  static FDSP_DEV void save(const R& r, Saver& s) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(r.time);
    s.S((uint32_t)b); s.S((uint32_t)(b >> 32)); s.Sf((float)r.time);
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<0>&, Fr<0>&) {
    if (T) r.time += r.sd;
    else if (c.i == 0) r.time += (double)c.n * r.sd;
  }
  static FDSP_DEV void end_simd(R&) {}
};

// The wave's samples are class-uniform data (voices playing the same wave share a class); the play region is per voice.
struct WavePlayer {
  FDSP_NODE(0, 1, 2, 1, 1);   // NU counts the length word; the samples follow it in the uniform block
  struct R { uint32_t end, loop, index; const uint32_t* w; };
  static FDSP_DEV void load(R& r, Loader& l) { const uint32_t n = l.U(); r.w = l.u + l.ui; l.ui += n; r.end = l.P(); r.loop = l.P(); r.index = l.S(); }
  static FDSP_DEV void save(const R& r, Saver& s) { s.S(r.index); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<0>&, Fr<1>& o) {
    if (r.index < r.end) {
      o.v[0] = __uint_as_float(__ldg(r.w + r.index));
      r.index++;
      if (r.index == r.end && r.loop != 0xffffffffu) r.index = r.loop;
    } else o.v[0] = 0.0f;
  }
  static FDSP_DEV void end_simd(R&) {}
};

// Variable-speed playback of a generator: the input is the speed (1 = original); the inner node is ticked as far as the cubic needs.
// The 128-frame ring per channel lives in the class's delay-line storage. The read position is f64 like the reference's.
template <class X> struct Resample {
  static constexpr int NO = X::OUT;
  FDSP_NODE(1, NO, X::NP, 3 + X::NS, X::NU);
  struct R { double consumer; uint32_t producer, off; typename X::R x; };
  static FDSP_DEV void load(R& r, Loader& l) {
    const uint32_t lo = l.S(), hi = l.S();
    r.consumer = __longlong_as_double((long long)(((unsigned long long)hi << 32) | lo));
    r.producer = l.S(); r.off = l.D(128u * (uint32_t)NO); X::load(r.x, l);
  }
  static FDSP_DEV void save(const R& r, Saver& s) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(r.consumer);
    s.S((uint32_t)b); s.S((uint32_t)(b >> 32)); s.S(r.producer); X::save(r.x, s);
  }
  static FDSP_DEV float spline(float y0, float y1, float y2, float y3, float x) {   // src/math.rs:360-366, the reference's evaluation order
    return y1 + x * 0.5f * (y2 - y0 + x * (2.0f * y0 - 5.0f * y1 + 4.0f * y2 - y3 + x * (3.0f * (y1 - y2) + y3 - y0)));
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<1>& in, Fr<NO>& o) {
    r.consumer += (double)fmaxf(0.0f, in.v[0]);
    const double d = r.consumer - floor(r.consumer);
    const uint32_t ci = (uint32_t)(unsigned long long)(r.consumer - d);
    float* ring = c.dl + (size_t)r.off * c.V + c.v;
    while (ci + 2u >= r.producer) {
      Fr<0> none; Fr<NO> y;
      X::template step<true>(r.x, c, none, y);
#pragma unroll
      for (int k = 0; k < NO; k++) ring[(size_t)((uint32_t)k * 128u + (r.producer & 0x7fu)) * c.V] = y.v[k];
      r.producer++;
    }
    const float x = (float)d;
#pragma unroll
    for (int k = 0; k < NO; k++) {
      const float* ch = ring + (size_t)((uint32_t)k * 128u) * c.V;
      o.v[k] = spline(ch[(size_t)((ci + 0x7fu) & 0x7fu) * c.V], ch[(size_t)(ci & 0x7fu) * c.V], ch[(size_t)((ci + 1u) & 0x7fu) * c.V], ch[(size_t)((ci + 2u) & 0x7fu) * c.V], x);
    }
  }
  static FDSP_DEV void end_simd(R&) {}
};

// ---------------------------------------------------------------- Reverb<F> (src/reverb.rs:139-279, ID 85: reverb3_stereo)
// Allpass-loop stereo reverb: 4 pre-delay allpasses, then 8 blocks of (delay, 4 allpasses, loop filter, 4 allpasses, loop
// filter) traversed in series; the last block's output is fed back. Tick-only in the reference, so every part runs `step<true>`.
// Word order (host ReverbN::lower): a | feedback | pre[0..3] | per block: delay, ap0[0..3], f0, ap1[0..3], f1.
template <class F> struct Reverb85 {
  typedef AllNest<1, Delay> Sch;
  static constexpr int IN = 2, OUT = 2;
  static constexpr int NP = 1 + 68 * Sch::NP + 8 * Delay::NP + 16 * F::NP;
  static constexpr int NS = 1 + 68 * Sch::NS + 8 * Delay::NS + 16 * F::NS;
  static constexpr int NU = 68 * Sch::NU + 8 * Delay::NU + 16 * F::NU;
  struct Blk { Delay::R delay; typename Sch::R a0[4]; typename F::R f0; typename Sch::R a1[4]; typename F::R f1; };
  struct R { float a, feedback; typename Sch::R pre[4]; Blk b[8]; };
  static FDSP_DEV void load(R& r, Loader& l) {
    r.a = l.Pf(); r.feedback = l.Sf();
    for (int k = 0; k < 4; k++) Sch::load(r.pre[k], l);
    for (int i = 0; i < 8; i++) {
      Delay::load(r.b[i].delay, l);
      for (int k = 0; k < 4; k++) Sch::load(r.b[i].a0[k], l);
      F::load(r.b[i].f0, l);
      for (int k = 0; k < 4; k++) Sch::load(r.b[i].a1[k], l);
      F::load(r.b[i].f1, l);
    }
  }
  static FDSP_DEV void save(const R& r, Saver& s) {
    s.Sf(r.feedback);
    for (int k = 0; k < 4; k++) Sch::save(r.pre[k], s);
    for (int i = 0; i < 8; i++) {
      Delay::save(r.b[i].delay, s);
      for (int k = 0; k < 4; k++) Sch::save(r.b[i].a0[k], s);
      F::save(r.b[i].f0, s);
      for (int k = 0; k < 4; k++) Sch::save(r.b[i].a1[k], s);
      F::save(r.b[i].f1, s);
    }
  }
  template <class N, class C> static FDSP_DEV float mono(typename N::R& r, const C& c, float x) { Fr<1> a, b; a.v[0] = x; N::template step<true>(r, c, a, b); return b.v[0]; }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<2>& in, Fr<2>& o) {  // :244-274
    float v0 = r.feedback, o0 = 0.0f, o1 = 0.0f;
    float in0 = mono<Sch>(r.pre[0], c, in.v[0] * 0.5f); in0 = mono<Sch>(r.pre[1], c, in0);
    float in1 = mono<Sch>(r.pre[2], c, in.v[1] * 0.5f); in1 = mono<Sch>(r.pre[3], c, in1);
#pragma unroll 1
    for (int i = 0; i < 8; i++) {
      Blk& b = r.b[i];
      v0 = mono<Delay>(b.delay, c, v0);
      v0 = mono<Sch>(b.a0[0], c, r.a * v0 + in0); v0 = mono<Sch>(b.a0[1], c, v0); v0 = mono<Sch>(b.a0[2], c, v0); v0 = mono<Sch>(b.a0[3], c, v0);
      v0 = mono<F>(b.f0, c, v0); o0 = v0;
      v0 = mono<Sch>(b.a1[0], c, r.a * v0 + in1); v0 = mono<Sch>(b.a1[1], c, v0); v0 = mono<Sch>(b.a1[2], c, v0); v0 = mono<Sch>(b.a1[3], c, v0);
      v0 = mono<F>(b.f1, c, v0); o1 = v0;
    }
    r.feedback = v0;
    o.v[0] = o0; o.v[1] = o1;
  }
  static FDSP_DEV void end_simd(R&) {}
};

// ---------------------------------------------------------------- panning / envelopes
template <int NIN> struct Panner {  // src/pan.rs:19-91, ID 49
  FDSP_NODE(NIN, 2, NIN == 1 ? 2 : 0, NIN == 1 ? 0 : 2, 0);
  struct R { float lw, rw; };
  static FDSP_DEV void load(R& r, Loader& l) { if (NIN == 1) { r.lw = l.Pf(); r.rw = l.Pf(); } else { r.lw = l.Sf(); r.rw = l.Sf(); } }
  static FDSP_DEV void save(const R& r, Saver& s) { if (NIN > 1) { s.Sf(r.lw); s.Sf(r.rw); } }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<NIN>& in, Fr<2>& o) {
    if (NIN > 1) pan_weights(in.v[NIN > 1 ? 1 : 0], r.lw, r.rw);
    o.v[0] = in.v[0] * r.lw; o.v[1] = in.v[0] * r.rw;
  }
  static FDSP_DEV void end_simd(R&) {}
};
template <int T64> struct FSel { typedef float type; };
template <> struct FSel<1> { typedef double type; };
// Envelope<F, E, R> (src/envelope.rs:14-183, ID 14: `envelope`, `lfo`): a control signal sampled at jittered points ~interval apart
// and interpolated linearly. The closure E lives on the host; its values at the sample points are data here. The points do not depend
// on how the signal is processed (t_1 = t_0 + lerp(0.75, 1.25, rnd1(t_hash)) * interval, t_hash an LCG of the node's hash), so the
// host evaluates the closure at exactly the points the reference would and lowers the K values per output as per-voice words; the
// point arithmetic, interpolation and the block path's run logic (:131-157) are restated here. F = f32 or f64 (T64).
template <int NO, int T64> struct EnvelopeTab {
  typedef typename FSel<T64>::type F;
  static constexpr int TW = T64 ? 2 : 1;   // words per time value
  FDSP_NODE(0, NO, 2 * TW, 3 * TW + 3 + 4 * NO + 3, 1);   // NP counts interval and sample duration; the K * NO table words follow them (K is class-uniform)
  struct R {
    uint32_t K, k; const uint32_t* tab; uint32_t V;
    F interval, sd, t, t0, t1; uint64_t t_hash;
    float v0[NO], v1[NO], value[NO], delta[NO];
    uint32_t run, run_len, seg_end;
  };
  static FDSP_DEV F ldF(Loader& l, bool state) {
    if (T64) { const uint32_t lo = state ? l.S() : l.P(), hi = state ? l.S() : l.P(); return (F)__longlong_as_double((long long)(((unsigned long long)hi << 32) | lo)); }
    return (F)(state ? l.Sf() : l.Pf());
  }
  static FDSP_DEV void stF(Saver& s, F x) {
    if (T64) { const unsigned long long b = (unsigned long long)__double_as_longlong((double)x); s.S((uint32_t)b); s.S((uint32_t)(b >> 32)); }
    else s.Sf((float)x);
  }
  static FDSP_DEV void load(R& r, Loader& l) {
    r.K = l.U(); r.interval = ldF(l, false); r.sd = ldF(l, false);
    r.tab = l.p + (size_t)l.pi * l.V + l.v; r.V = l.V; l.pi += r.K * (uint32_t)NO;
    r.t = ldF(l, true); r.t0 = ldF(l, true); r.t1 = ldF(l, true);
    const uint32_t lo = l.S(), hi = l.S(); r.t_hash = ((uint64_t)hi << 32) | lo;
    r.k = l.S();
#pragma unroll
    for (int c = 0; c < NO; c++) { r.v0[c] = l.Sf(); r.v1[c] = l.Sf(); r.value[c] = l.Sf(); r.delta[c] = l.Sf(); }
    r.run = l.S(); r.run_len = l.S(); r.seg_end = l.S();
  }
  static FDSP_DEV void save(const R& r, Saver& s) {
    stF(s, r.t); stF(s, r.t0); stF(s, r.t1);
    s.S((uint32_t)r.t_hash); s.S((uint32_t)(r.t_hash >> 32)); s.S(r.k);
#pragma unroll
    for (int c = 0; c < NO; c++) { s.Sf(r.v0[c]); s.Sf(r.v1[c]); s.Sf(r.value[c]); s.Sf(r.delta[c]); }
    s.S(r.run); s.S(r.run_len); s.S(r.seg_end);
  }
  static FDSP_DEV void next_segment(R& r) {   // :63-82
    r.t0 = r.t1;
    const F w = (F)rnd1(r.t_hash);
    const F next_interval = ((F)0.75f * ((F)1 - w) + (F)1.25f * w) * r.interval;
    r.t1 = r.t0 + next_interval;
    const uint32_t kk = r.k < r.K ? r.k : r.K - 1u;   // past the sampled horizon the last value holds
    r.k += 1u;
    r.t_hash = r.t_hash * 6364136223846793005ull + 1ull;
    const float u = (float)((r.t - r.t0) / (r.t1 - r.t0));
    const float samples = (float)(next_interval / r.sd);
#pragma unroll
    for (int c = 0; c < NO; c++) {
      r.v0[c] = r.v1[c];
      r.v1[c] = __uint_as_float(__ldg(r.tab + (size_t)(kk * (uint32_t)NO + (uint32_t)c) * r.V));
      r.value[c] = r.v0[c] * (1.0f - u) + r.v1[c] * u;
      r.delta[c] = (r.v1[c] - r.v0[c]) / samples;
    }
  }
  static FDSP_DEV F ceilF(F x) { return T64 ? (F)ceil((double)x) : (F)ceilf((float)x); }
  template <class C> static FDSP_DEV void plan(R& r, const C& c) {   // the while-loop of :135-156 from block index c.i
    for (;;) {
      const long long left = (long long)ceilF((r.t1 - r.t) / r.sd);
      const long long room = (long long)(c.n - c.i);   // > 0: plan runs only with samples left in the block
      const long long loop = left < room ? left : room;
      if (loop <= 0) { next_segment(r); continue; }     // t == t_1 exactly: zero samples, loop_samples == segment_samples_left
      r.run = (uint32_t)loop; r.run_len = r.run; r.seg_end = (loop == left) ? 1u : 0u;
      return;
    }
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<0>&, Fr<NO>& o) {
    if (T) {   // tick :117-126
      if (r.t >= r.t1) next_segment(r);
#pragma unroll
      for (int k = 0; k < NO; k++) { o.v[k] = r.value[k]; r.value[k] += r.delta[k]; }
      r.t += r.sd;
      return;
    }
    if (c.i == 0) { if (r.t >= r.t1) next_segment(r); plan(r, c); }
    else if (r.run == 0u) plan(r, c);
#pragma unroll
    for (int k = 0; k < NO; k++) { o.v[k] = r.value[k]; r.value[k] += r.delta[k]; }
    r.run -= 1u;
    if (r.run == 0u) { r.t += (F)(long long)r.run_len * r.sd; if (r.seg_end) next_segment(r); }
  }
  static FDSP_DEV void end_simd(R&) {}
};

struct AdsrLive {  // src/envelope.rs:185-358 EnvelopeIn<f32,_,U1,f32> (ID 53) + the closure of src/adsr.rs:21-70
  FDSP_NODE(1, 1, 5, 15, 0);
  struct R {
    float attack, decay, sustain, release, interval;
    uint32_t attacked; float attack_start, release_start;
    float t, t0, t1; uint64_t t_hash; float v0, v1, value, delta;
    uint32_t run, run_len, seg_end;  // block-path run bookkeeping (envelope.rs:315-340), see step()
  };
  static FDSP_DEV void load(R& r, Loader& l) {
    r.attack = l.Pf(); r.decay = l.Pf(); r.sustain = l.Pf(); r.release = l.Pf(); r.interval = l.Pf();
    r.attacked = l.S(); r.attack_start = l.Sf(); r.release_start = l.Sf();
    r.t = l.Sf(); r.t0 = l.Sf(); r.t1 = l.Sf();
    uint32_t lo = l.S(), hi = l.S(); r.t_hash = ((uint64_t)hi << 32) | lo;
    r.v0 = l.Sf(); r.v1 = l.Sf(); r.value = l.Sf(); r.delta = l.Sf();
    r.run = l.S(); r.run_len = l.S(); r.seg_end = l.S();
  }
  static FDSP_DEV void save(const R& r, Saver& s) {
    s.S(r.attacked); s.Sf(r.attack_start); s.Sf(r.release_start);
    s.Sf(r.t); s.Sf(r.t0); s.Sf(r.t1);
    s.S((uint32_t)r.t_hash); s.S((uint32_t)(r.t_hash >> 32));
    s.Sf(r.v0); s.Sf(r.v1); s.Sf(r.value); s.Sf(r.delta);
    s.S(r.run); s.S(r.run_len); s.S(r.seg_end);
  }
  static FDSP_DEV float ads(const R& r, float time) {  // adsr.rs:59-70
    if (time < r.attack) return lerpf(0.0f, 1.0f, time / r.attack);
    float decay_time = time - r.attack;
    if (decay_time < r.decay) return lerpf(1.0f, r.sustain, decay_time / r.decay);
    return r.sustain;
  }
  static FDSP_DEV float envelope(R& r, float time, float control) {  // adsr.rs:34-56
    if (r.release_start >= 0.0f && control > 0.0f) { r.attacked = 1u; r.attack_start = time; r.release_start = -1.0f; }
    else if (r.release_start < 0.0f && control <= 0.0f) { r.release_start = time; }
    if (!r.attacked) return 0.0f;
    float a = ads(r, time - r.attack_start);
    if (r.release_start < 0.0f) return a;
    return a * clamp01f(delerpf(r.release_start + r.release, r.release_start, time));
  }
  template <class C> static FDSP_DEV void next_segment(R& r, const C& c, float input) {  // envelope.rs:238-263
    if (r.t0 == 0.0f && r.t1 == 0.0f) { r.v0 = envelope(r, r.t0, input); }
    else { r.t0 = r.t1; r.v0 = r.v1; }
    float next_interval = lerpf(0.75f, 1.25f, (float)rnd1(r.t_hash)) * r.interval;
    r.t1 = r.t0 + next_interval;
    r.v1 = envelope(r, r.t1, input);
    r.t_hash = r.t_hash * 6364136223846793005ull + 1ull;
    float u = delerpf(r.t0, r.t1, r.t);
    r.value = lerpf(r.v0, r.v1, u);
    float samples = next_interval / c.sd64;
    r.delta = (r.v1 - r.v0) / samples;
  }
  // plan the next run of the block path's while-loop (envelope.rs:321-339) starting at block index i
  template <class C> static FDSP_DEV void plan(R& r, const C& c, float input) {
    for (;;) {
      unsigned long long left = (unsigned long long)(long long)ceilf((r.t1 - r.t) / c.sd64);
      unsigned long long room = (unsigned long long)(c.n - c.i);
      unsigned long long loop = left < room ? left : room;
      if (loop == 0ull) { r.t += 0.0f * c.sd64; next_segment(r, c, input); continue; }
      r.run = (uint32_t)loop; r.run_len = r.run; r.seg_end = (loop == left) ? 1u : 0u;
      return;
    }
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<1>& in, Fr<1>& o) {
    if (T) {  // tick :297-305
      if (r.t >= r.t1) next_segment(r, c, in.v[0]);
      o.v[0] = r.value; r.value += r.delta; r.t += c.sd64;
      return;
    }
    if (c.i == 0) { if (r.t >= r.t1) next_segment(r, c, in.v[0]); plan(r, c, in.v[0]); }
    else if (r.run == 0u) { if (r.seg_end) next_segment(r, c, in.v[0]); plan(r, c, in.v[0]); }
    o.v[0] = r.value; r.value += r.delta;
    r.run -= 1u;
    if (r.run == 0u) r.t += (float)r.run_len * c.sd64;
  }
  static FDSP_DEV void end_simd(R&) {}
};

// ---------------------------------------------------------------- closures of the signal: map (ID 5), shape_fn (ID 42), EnvelopeIn (ID 53)
// A closure crosses the C ABI as text; csrc/host/closure.cpp parses it and writes it into the class signature as a tree of the
// expression templates below, so it is compiled like any other node. Everything is f32, evaluated as Rust evaluates the closure:
// each operation individually rounded, no contraction. Literals are f32 bit patterns in the type (class-uniform); captured values
// are per-voice parameter words (Cap<k>), so voices that share a closure text and differ in what they capture form one class.
// `let` bindings are de Bruijn indexed (Var<0> is the innermost), so the spelling of names never reaches the signature.
namespace Ex {
struct Root {   // the closure's arguments: the input frame (or the shaper's scalar), the captures, the envelope's time
  const float* x; const float* c; float t;
  FDSP_HD const Root& root() const { return *this; }
};
template <class P> struct Scope { float v; const P& up; FDSP_HD const Root& root() const { return up.root(); } };
template <int K, class S> FDSP_HD float var(const S& s) { if constexpr (K == 0) return s.v; else return var<K - 1>(s.up); }

FDSP_HD float lerp_(float a, float b, float t) { return a * (1.0f - t) + b * t; }                 // src/math.rs:170-177 (f32 Lerp)
FDSP_HD float exp10_(float x) { return m::expf_(x * (float)2.302585092994045684); }             // src/math.rs:76-78: (x * LN_10 as f32).exp()
FDSP_HD float clamp_m(float x, float lo, float hi) { if (x < lo) x = lo; if (x > hi) x = hi; return x; }   // std f32::clamp: NaN propagates
FDSP_HD float signum_m(float x) { return x != x ? m::fromb(0x7fc00000u) : copysignf(1.0f, x); }   // std f32::signum (fundsp's is copysignf)
FDSP_HD float softexp_(float x) { const float p = fmaxf(x, 0.0f); return p * p + p + 1.0f / (1.0f + p - x); }   // src/math.rs:394-399
FDSP_HD float sqr_hz_(float hz, float t) { float x = t * hz; x = x - floorf(x); return x < 0.5f ? 1.0f : -1.0f; }     // src/math.rs:485-493
FDSP_HD float tri_hz_(float hz, float t) { float x = t * hz - 0.25f; x = x - floorf(x); return fabsf(x - 0.5f) * 4.0f - 1.0f; }   // :507-511

#define FDSP_EX_LEAF(Name, cost_, expr) \
  struct Name { static constexpr int cost = (cost_); template <class S> static FDSP_HD float ev(const S& s) { return (expr); } };
#define FDSP_EX1(Name, cost_, expr) \
  template <class A> struct Name { static constexpr int cost = A::cost + (cost_); \
    template <class S> static FDSP_HD float ev(const S& s) { const float a = A::ev(s); return (expr); } };
#define FDSP_EX2(Name, R_, cost_, expr) \
  template <class A, class B> struct Name { static constexpr int cost = A::cost + B::cost + (cost_); \
    template <class S> static FDSP_HD R_ ev(const S& s) { const auto a = A::ev(s); const auto b = B::ev(s); return (expr); } };
#define FDSP_EX3(Name, cost_, expr) \
  template <class A, class B, class C> struct Name { static constexpr int cost = A::cost + B::cost + C::cost + (cost_); \
    template <class S> static FDSP_HD float ev(const S& s) { const float a = A::ev(s), b = B::ev(s), c = C::ev(s); return (expr); } };

template <int K> struct In { static constexpr int cost = 0; template <class S> static FDSP_HD float ev(const S& s) { return s.root().x[K]; } };
template <int K> struct Cap { static constexpr int cost = 0; template <class S> static FDSP_HD float ev(const S& s) { return s.root().c[K]; } };
template <uint32_t B> struct Lit { static constexpr int cost = 0; template <class S> static FDSP_HD float ev(const S&) { return m::fromb(B); } };
FDSP_EX_LEAF(T, 0, s.root().t)
template <int K> struct Var { static constexpr int cost = 0; template <class S> static FDSP_HD float ev(const S& s) { return var<K>(s); } };
template <int K> struct BVar { static constexpr int cost = 0; template <class S> static FDSP_HD bool ev(const S& s) { return var<K>(s) != 0.0f; } };

FDSP_EX2(Add, float, 1, a + b) FDSP_EX2(Sub, float, 1, a - b) FDSP_EX2(Mul, float, 1, a * b) FDSP_EX2(Div, float, 8, a / b)
FDSP_EX1(Neg, 1, -a)
FDSP_EX2(Lt, bool, 1, a < b) FDSP_EX2(Le, bool, 1, a <= b) FDSP_EX2(Gt, bool, 1, a > b) FDSP_EX2(Ge, bool, 1, a >= b)
FDSP_EX2(Eq, bool, 1, a == b) FDSP_EX2(Ne, bool, 1, a != b)
FDSP_EX2(And, bool, 1, a && b) FDSP_EX2(Or, bool, 1, a || b)
template <class A> struct Not { static constexpr int cost = A::cost + 1; template <class S> static FDSP_HD bool ev(const S& s) { return !A::ev(s); } };
template <class C, class A, class B> struct If {
  static constexpr int cost = C::cost + A::cost + B::cost + 2;
  template <class S> static FDSP_HD auto ev(const S& s) { return C::ev(s) ? A::ev(s) : B::ev(s); }
};
template <class X, class B> struct Let {
  static constexpr int cost = X::cost + B::cost;
  template <class S> static FDSP_HD auto ev(const S& s) { const Scope<S> in{(float)X::ev(s), s}; return B::ev(in); }
};
template <class... Es> struct Out { static constexpr int cost = (0 + ... + Es::cost); };

// exact operations (src/math.rs, Rust core), each as written there
FDSP_EX1(Abs, 1, fabsf(a)) FDSP_EX2(Min, float, 1, fminf(a, b)) FDSP_EX2(Max, float, 1, fmaxf(a, b))
FDSP_EX3(Clamp, 2, fminf(fmaxf(c, a), b))            // clamp(x0, x1, x) = x.max(x0).min(x1)
FDSP_EX3(ClampM, 2, clamp_m(a, b, c))                 // x.clamp(lo, hi)
FDSP_EX1(Clamp01, 2, fminf(fmaxf(a, 0.0f), 1.0f)) FDSP_EX1(Clamp11, 2, fminf(fmaxf(a, -1.0f), 1.0f))
FDSP_EX1(Floor, 1, floorf(a)) FDSP_EX1(Ceil, 1, ceilf(a)) FDSP_EX1(Round, 2, roundf(a)) FDSP_EX1(Sqrt, 8, sqrtf(a))
FDSP_EX1(Signum, 1, copysignf(1.0f, a)) FDSP_EX1(SignumM, 2, signum_m(a))
FDSP_EX3(Lerp, 3, lerp_(a, b, c)) FDSP_EX3(Lerp11, 5, lerp_(a, b, c * 0.5f + 0.5f))
FDSP_EX3(Delerp, 10, (c - a) / (b - a)) FDSP_EX3(Delerp11, 12, (c - a) / (b - a) * 2.0f - 1.0f)
FDSP_EX1(Softsign, 10, a / (1.0f + fabsf(a)))
FDSP_EX1(Softexp, 12, softexp_(a))
FDSP_EX1(Smooth3, 4, (3.0f - 2.0f * a) * a * a)
FDSP_EX1(Smooth5, 6, ((a * 6.0f - 15.0f) * a + 10.0f) * a * a * a)
FDSP_EX1(Smooth7, 8, (a * a) * (a * a) * (35.0f - 84.0f * a + (70.0f - 20.0f * a) * (a * a)))
FDSP_EX1(Smooth9, 10, ((((70.0f * a - 315.0f) * a + 540.0f) * a - 420.0f) * a + 126.0f) * (a * a) * (a * a) * a)
template <class Y0, class Y1, class Y2, class Y3, class X> struct Spline {   // src/math.rs:360-366
  static constexpr int cost = Y0::cost + Y1::cost + Y2::cost + Y3::cost + X::cost + 14;
  template <class S> static FDSP_HD float ev(const S& s) {
    const float y0 = Y0::ev(s), y1 = Y1::ev(s), y2 = Y2::ev(s), y3 = Y3::ev(s), x = X::ev(s);
    return y1 + x * 0.5f * (y2 - y0 + x * (2.0f * y0 - 5.0f * y1 + 4.0f * y2 - y3 + x * (3.0f * (y1 - y2) + y3 - y0)));
  }
};
FDSP_EX2(SqrHz, float, 4, sqr_hz_(a, b)) FDSP_EX2(TriHz, float, 6, tri_hz_(a, b))
FDSP_EX1(BpmHz, 2, a * (1.0f / 60.0f)) FDSP_EX1(Squared, 1, a * a)
// musl restatements (csrc/dsp/libm.cuh): what fundsp's Real / Float traits resolve to for f32, and what the project maps std's
// inherent f32 methods to (DESIGN.md §4)
FDSP_EX1(Sin, 40, m::sinf_(a)) FDSP_EX1(Cos, 40, m::cosf_(a)) FDSP_EX1(Tan, 50, m::tanf_(a)) FDSP_EX1(Tanh, 96, m::tanhf_(a))
FDSP_EX1(Exp, 40, m::expf_(a)) FDSP_EX2(Pow, float, 120, m::powf_(a, b)) FDSP_EX1(Exp10, 41, exp10_(a)) FDSP_EX1(DbAmp, 49, exp10_(a / 20.0f))
FDSP_EX2(SinHz, float, 42, m::sinf_(b * a * TAU_F)) FDSP_EX2(CosHz, float, 42, m::cosf_(b * a * TAU_F))   // sin_hz(hz, t) = sin(t * hz * TAU)
#undef FDSP_EX_LEAF
#undef FDSP_EX1
#undef FDSP_EX2
#undef FDSP_EX3

// Writes the closure's value into o[0..NO): a tuple (the reference's ConstantFrame return) may stand in tail position, under
// `let` and in both arms of an `if`.
template <class X> struct Emit { template <class S> static FDSP_HD void out(const S& s, float* o) { o[0] = X::ev(s); } };
template <class... Es> struct Emit<Out<Es...>> {
  template <class S> static FDSP_HD void out(const S& s, float* o) { int i = 0; ((o[i++] = Es::ev(s)), ...); }
};
template <class X, class B> struct Emit<Let<X, B>> {
  template <class S> static FDSP_HD void out(const S& s, float* o) { const Scope<S> in{(float)X::ev(s), s}; Emit<B>::out(in, o); }
};
template <class C, class A, class B> struct Emit<If<C, A, B>> {
  template <class S> static FDSP_HD void out(const S& s, float* o) { if (C::ev(s)) Emit<A>::out(s, o); else Emit<B>::out(s, o); }
};
}  // namespace Ex

template <int NI, int NO, int NC, class E> struct Map {   // src/audionode.rs:1328-1371, ID 5: no `process` override, so the block path is the tick loop
  FDSP_NODE(NI, NO, NC, 0, 0);
  struct R { float c[NC > 0 ? NC : 1]; };
  static FDSP_DEV void load(R& r, Loader& l) {
#pragma unroll
    for (int k = 0; k < NC; k++) r.c[k] = l.Pf();
  }
  static FDSP_DEV void save(const R&, Saver&) {}
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<NI>& in, Fr<NO>& o) {
    const Ex::Root s{in.v, r.c, 0.0f};
    Ex::Emit<E>::out(s, o.v);
  }
  static FDSP_DEV void end_simd(R&) {}
};
// VarFn<F, R> (src/shared.rs:134-200, ID 70): the closure of the Shared's value. The value is a parameter word the host rewrites between
// calls (Bank::sh_pull), so within one launch value and captures are constant and the closure, evaluated once when the voice is loaded,
// gives what VarFn::process computes for every block of the call.
template <int NO, int NC, class E> struct VarFn {
  FDSP_NODE(0, NO, 1 + NC, 0, 0);
  struct R { float o[NO]; };
  static FDSP_DEV void load(R& r, Loader& l) {
    const float x = l.Pf();
    float c[NC > 0 ? NC : 1];
#pragma unroll
    for (int k = 0; k < NC; k++) c[k] = l.Pf();
    const Ex::Root s{&x, c, 0.0f};
    Ex::Emit<E>::out(s, r.o);
  }
  static FDSP_DEV void save(const R&, Saver&) {}
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<0>&, Fr<NO>& o) {
#pragma unroll
    for (int k = 0; k < NO; k++) o.v[k] = r.o[k];
  }
  static FDSP_DEV void end_simd(R&) {}
};
// Shaper<ShapeFn<S>> (src/shape.rs:33-42, ID 42): ShapeFn::simd is the default per-lane `shape`, so tick and block paths coincide
template <int NC, class E> struct ShaperFn : Map<1, 1, NC, E> {};

// EnvelopeIn<f32, E, I, R> (src/envelope.rs:185-358, ID 53) with the closure E in the type: sampled at jittered points ~interval apart
// with the input frame of the sample where the segment starts, interpolated linearly. Same run structure as AdsrLive above.
template <int NI, int NO, int NC, class E> struct EnvelopeInFn {
  FDSP_NODE(NI, NO, NC + 1, 8 + 4 * NO, 0);
  struct R {
    float c[NC > 0 ? NC : 1]; float interval;
    float t, t0, t1; uint64_t t_hash;
    float v0[NO], v1[NO], value[NO], delta[NO];
    uint32_t run, run_len, seg_end;
  };
  static FDSP_DEV void load(R& r, Loader& l) {
#pragma unroll
    for (int k = 0; k < NC; k++) r.c[k] = l.Pf();
    r.interval = l.Pf();
    r.t = l.Sf(); r.t0 = l.Sf(); r.t1 = l.Sf();
    const uint32_t lo = l.S(), hi = l.S(); r.t_hash = ((uint64_t)hi << 32) | lo;
#pragma unroll
    for (int k = 0; k < NO; k++) { r.v0[k] = l.Sf(); r.v1[k] = l.Sf(); r.value[k] = l.Sf(); r.delta[k] = l.Sf(); }
    r.run = l.S(); r.run_len = l.S(); r.seg_end = l.S();
  }
  static FDSP_DEV void save(const R& r, Saver& s) {
    s.Sf(r.t); s.Sf(r.t0); s.Sf(r.t1);
    s.S((uint32_t)r.t_hash); s.S((uint32_t)(r.t_hash >> 32));
#pragma unroll
    for (int k = 0; k < NO; k++) { s.Sf(r.v0[k]); s.Sf(r.v1[k]); s.Sf(r.value[k]); s.Sf(r.delta[k]); }
    s.S(r.run); s.S(r.run_len); s.S(r.seg_end);
  }
  static FDSP_DEV void call(const R& r, float time, const Fr<NI>& in, float* out) { const Ex::Root s{in.v, r.c, time}; Ex::Emit<E>::out(s, out); }
  template <class C> static FDSP_DEV void next_segment(R& r, const C& c, const Fr<NI>& in) {   // envelope.rs:251-278
    if (r.t0 == 0.0f && r.t1 == 0.0f) call(r, r.t0, in, r.v0);
    else {
      r.t0 = r.t1;
#pragma unroll
      for (int k = 0; k < NO; k++) r.v0[k] = r.v1[k];
    }
    const float next_interval = lerpf(0.75f, 1.25f, (float)rnd1(r.t_hash)) * r.interval;
    r.t1 = r.t0 + next_interval;
    call(r, r.t1, in, r.v1);
    r.t_hash = r.t_hash * 6364136223846793005ull + 1ull;
    const float u = delerpf(r.t0, r.t1, r.t);
    const float samples = next_interval / c.sd64;
#pragma unroll
    for (int k = 0; k < NO; k++) { r.value[k] = lerpf(r.v0[k], r.v1[k], u); r.delta[k] = (r.v1[k] - r.v0[k]) / samples; }
  }
  template <class C> static FDSP_DEV void plan(R& r, const C& c, const Fr<NI>& in) {   // the while-loop of :323-341 from block index c.i
    for (;;) {
      const unsigned long long left = (unsigned long long)(long long)ceilf((r.t1 - r.t) / c.sd64);
      const unsigned long long room = (unsigned long long)(c.n - c.i);
      const unsigned long long loop = left < room ? left : room;
      if (loop == 0ull) { next_segment(r, c, in); continue; }
      r.run = (uint32_t)loop; r.run_len = r.run; r.seg_end = (loop == left) ? 1u : 0u;
      return;
    }
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<NI>& in, Fr<NO>& o) {
    if (T) {   // tick :305-313
      if (r.t >= r.t1) next_segment(r, c, in);
#pragma unroll
      for (int k = 0; k < NO; k++) { o.v[k] = r.value[k]; r.value[k] += r.delta[k]; }
      r.t += c.sd64;
      return;
    }
    // process :315-342: the input is read at the block index where a segment changes
    if (c.i == 0) { if (r.t >= r.t1) next_segment(r, c, in); plan(r, c, in); }
    else if (r.run == 0u) { if (r.seg_end) next_segment(r, c, in); plan(r, c, in); }
#pragma unroll
    for (int k = 0; k < NO; k++) { o.v[k] = r.value[k]; r.value[k] += r.delta[k]; }
    r.run -= 1u;
    if (r.run == 0u) r.t += (float)r.run_len * c.sd64;
  }
  static FDSP_DEV void end_simd(R&) {}
};

// Envelope<f32, E, R> (src/envelope.rs:14-183, ID 14) with the closure E of time in the type. It samples at the same jittered points as
// EnvelopeTab, from the same hash, but evaluates E there instead of reading a table, so nothing holds past a horizon. The host lowers
// reset's t = t_0 = t_1 = 0; E(0), which reset() stores as value_0 = value_1, is evaluated by the first next_segment (t_1 > 0 after it).
// The block path follows process (:139-163): a run ending a segment moves to the next one at once, as the reference does.
template <int NO, int NC, class E> struct EnvelopeFn {
  FDSP_NODE(0, NO, NC + 1, 8 + 4 * NO, 0);
  typedef typename EnvelopeInFn<0, NO, NC, E>::R R;
  static FDSP_DEV void load(R& r, Loader& l) { EnvelopeInFn<0, NO, NC, E>::load(r, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { EnvelopeInFn<0, NO, NC, E>::save(r, s); }
  static FDSP_DEV void call(const R& r, float time, float* out) { const Ex::Root s{nullptr, r.c, time}; Ex::Emit<E>::out(s, out); }
  template <class C> static FDSP_DEV void next_segment(R& r, const C& c) {   // :80-101
    if (r.t0 == 0.0f && r.t1 == 0.0f) call(r, 0.0f, r.v1);                 // reset :114-122
    r.t0 = r.t1;
#pragma unroll
    for (int k = 0; k < NO; k++) r.v0[k] = r.v1[k];
    const float next_interval = lerpf(0.75f, 1.25f, (float)rnd1(r.t_hash)) * r.interval;
    r.t1 = r.t0 + next_interval;
    call(r, r.t1, r.v1);
    r.t_hash = r.t_hash * 6364136223846793005ull + 1ull;
    const float u = delerpf(r.t0, r.t1, r.t);
    const float samples = next_interval / c.sd64;
#pragma unroll
    for (int k = 0; k < NO; k++) { r.value[k] = lerpf(r.v0[k], r.v1[k], u); r.delta[k] = (r.v1[k] - r.v0[k]) / samples; }
  }
  template <class C> static FDSP_DEV void plan(R& r, const C& c) {   // the while-loop of :144-162 from block index c.i
    for (;;) {
      const unsigned long long left = (unsigned long long)(long long)ceilf((r.t1 - r.t) / c.sd64);
      const unsigned long long room = (unsigned long long)(c.n - c.i);
      const unsigned long long loop = left < room ? left : room;
      if (loop == 0ull) { next_segment(r, c); continue; }
      r.run = (uint32_t)loop; r.run_len = r.run; r.seg_end = (loop == left) ? 1u : 0u;
      return;
    }
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<0>&, Fr<NO>& o) {
    if (T) {   // tick :129-137
      if (r.t >= r.t1) next_segment(r, c);
#pragma unroll
      for (int k = 0; k < NO; k++) { o.v[k] = r.value[k]; r.value[k] += r.delta[k]; }
      r.t += c.sd64;
      return;
    }
    if (c.i == 0) { if (r.t >= r.t1) next_segment(r, c); plan(r, c); }
    else if (r.run == 0u) plan(r, c);
#pragma unroll
    for (int k = 0; k < NO; k++) { o.v[k] = r.value[k]; r.value[k] += r.delta[k]; }
    r.run -= 1u;
    if (r.run == 0u) { r.t += (float)r.run_len * c.sd64; if (r.seg_end) next_segment(r, c); }
  }
  static FDSP_DEV void end_simd(R&) {}
};


// ---------------------------------------------------------------- Dag: a whole Net as ONE fused node (src/net.rs:118-146, 1224-1286)
// The reference's Net is a dynamic DAG of boxed units processed vertex by vertex in dependency order, each vertex reading the
// output buffers of its sources. Here the host emits the vertices in a dependency order and encodes every edge in the TYPE:
//   Dag<NIN, NOUT, VList<Vx<Unit0, src...>, Vx<Unit1, src...>, ...>, Outs<src...>>
// one `src` code per unit input / net output: (type << 24) | (vertex << 8) | port with type 0 = zero, 1 = global input `port`,
// 2 = output `port` of an earlier vertex (vertex = position in the list). All vertex outputs of a group live in registers
// (`buf`), so an arbitrary acyclic Net costs what the equivalent static combinator expression would. Block semantics hold
// vertex by vertex (each runs its own group / tick form), exactly like Net::process calling `unit.process` per vertex.
template <class U, int... S> struct Vx {
  typedef U Unit;
  static __host__ __device__ constexpr int src(int i) { constexpr int a[] = {S..., 0}; return a[i]; }
};
template <class... V> struct VList {};
template <int... S> struct Outs { static __host__ __device__ constexpr int src(int i) { constexpr int a[] = {S..., 0}; return a[i]; } };
template <class... V> struct DagState;
template <> struct DagState<> {};
template <class H, class... T> struct DagState<H, T...> { typename H::Unit::R head; DagState<T...> tail; };
template <int NIN, int NOUT, class VL, class OS> struct Dag;
template <int NIN, int NOUT, class... V, class OS> struct Dag<NIN, NOUT, VList<V...>, OS> {
  static constexpr int IN = NIN, OUT = NOUT;
  static constexpr int NP = (0 + ... + V::Unit::NP), NS = (0 + ... + V::Unit::NS), NU = (0 + ... + V::Unit::NU);
  static constexpr int TOT = (0 + ... + V::Unit::OUT);
  static constexpr int TB = TOT > 0 ? TOT : 1;
  typedef DagState<V...> R;
  static __host__ __device__ constexpr int offset(int k) { constexpr int outs[] = {V::Unit::OUT..., 0}; int o = 0; for (int i = 0; i < k; i++) o += outs[i]; return o; }

  static FDSP_DEV void load_(DagState<>&, Loader&) {}
  template <class H, class... T> static FDSP_DEV void load_(DagState<H, T...>& r, Loader& l) { H::Unit::load(r.head, l); load_(r.tail, l); }
  static FDSP_DEV void save_(const DagState<>&, Saver&) {}
  template <class H, class... T> static FDSP_DEV void save_(const DagState<H, T...>& r, Saver& s) { H::Unit::save(r.head, s); save_(r.tail, s); }
  static FDSP_DEV void end_(DagState<>&) {}
  template <class H, class... T> static FDSP_DEV void end_(DagState<H, T...>& r) { H::Unit::end_simd(r.head); end_(r.tail); }
  static FDSP_DEV void load(R& r, Loader& l) { load_(r, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { save_(r, s); }
  static FDSP_DEV void end_simd(R& r) { end_(r); }

  // ---- 8-sample group form
  template <int CODE> static FDSP_DEV void fetch8(const Fr8<NIN>& in, const float (&buf)[TB][8], float (&dst)[8]) {
    constexpr int type = CODE >> 24, node = (CODE >> 8) & 0xffff, port = CODE & 0xff;
    constexpr int row = type == 2 ? offset(node) + port : 0;
#pragma unroll
    for (int j = 0; j < 8; j++) dst[j] = type == 0 ? 0.0f : (type == 1 ? in.v[type == 1 ? port : 0][j] : buf[row][j]);
  }
  template <class H, int I> static FDSP_DEV void gather8(const Fr8<NIN>& in, const float (&buf)[TB][8], Fr8<H::Unit::IN>& a) {
    if constexpr (I < H::Unit::IN) { fetch8<H::src(I)>(in, buf, a.v[I]); gather8<H, I + 1>(in, buf, a); }
  }
  template <int K, class C> static FDSP_DEV void run8(DagState<>&, C&, const Fr8<NIN>&, float (&)[TB][8]) {}
  template <int K, class C, class H, class... T> static FDSP_DEV void run8(DagState<H, T...>& r, C& c, const Fr8<NIN>& in, float (&buf)[TB][8]) {
    Fr8<H::Unit::IN> a; Fr8<H::Unit::OUT> b;
    gather8<H, 0>(in, buf, a);
    group_step<typename H::Unit>(r.head, c, a, b);
    constexpr int base = offset(K);
#pragma unroll
    for (int q = 0; q < H::Unit::OUT; q++) {
#pragma unroll
      for (int j = 0; j < 8; j++) buf[base + q][j] = b.v[q][j];
    }
    run8<K + 1>(r.tail, c, in, buf);
  }
  template <int I> static FDSP_DEV void out8(const Fr8<NIN>& in, const float (&buf)[TB][8], Fr8<NOUT>& o) {
    if constexpr (I < NOUT) { fetch8<OS::src(I)>(in, buf, o.v[I]); out8<I + 1>(in, buf, o); }
  }
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C& c, const Fr8<NIN>& in, Fr8<NOUT>& o) {
    float buf[TB][8];
    run8<0>(r, c, in, buf);
    out8<0>(in, buf, o);
  }

  // ---- per-sample form (tail samples, and Nets inside a Feedback: Net::tick, src/net.rs:1187-1222)
  template <int CODE> static FDSP_DEV float fetch1(const Fr<NIN>& in, const float (&buf)[TB]) {
    constexpr int type = CODE >> 24, node = (CODE >> 8) & 0xffff, port = CODE & 0xff;
    constexpr int row = type == 2 ? offset(node) + port : 0;
    return type == 0 ? 0.0f : (type == 1 ? in.v[type == 1 ? port : 0] : buf[row]);
  }
  template <class H, int I> static FDSP_DEV void gather1(const Fr<NIN>& in, const float (&buf)[TB], Fr<H::Unit::IN>& a) {
    if constexpr (I < H::Unit::IN) { a.v[I] = fetch1<H::src(I)>(in, buf); gather1<H, I + 1>(in, buf, a); }
  }
  template <bool T, int K, class C> static FDSP_DEV void run1(DagState<>&, const C&, const Fr<NIN>&, float (&)[TB]) {}
  template <bool T, int K, class C, class H, class... TT> static FDSP_DEV void run1(DagState<H, TT...>& r, const C& c, const Fr<NIN>& in, float (&buf)[TB]) {
    Fr<H::Unit::IN> a; Fr<H::Unit::OUT> b;
    gather1<H, 0>(in, buf, a);
    H::Unit::template step<T>(r.head, c, a, b);
    constexpr int base = offset(K);
#pragma unroll
    for (int q = 0; q < H::Unit::OUT; q++) buf[base + q] = b.v[q];
    run1<T, K + 1>(r.tail, c, in, buf);
  }
  template <int I> static FDSP_DEV void out1(const Fr<NIN>& in, const float (&buf)[TB], Fr<NOUT>& o) {
    if constexpr (I < NOUT) { o.v[I] = fetch1<OS::src(I)>(in, buf); out1<I + 1>(in, buf, o); }
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<NIN>& in, Fr<NOUT>& o) {
    float buf[TB];
    run1<T, 0>(r, c, in, buf);
    out1<0>(in, buf, o);
  }
};

// ---------------------------------------------------------------- traits
// First wavetable kind used by a graph type (-1: none): decides whether the kernel stages tables in shared memory.
template <class G> struct WaveKind { static constexpr int value = -1; };
template <int K, int N> struct WaveKind<WaveSynth<K, N>> { static constexpr int value = K; };
template <int K> struct WaveKind<PhaseSynth<K>> { static constexpr int value = K; };
template <class X, class Y> struct Wk2 { static constexpr int value = WaveKind<X>::value >= 0 ? WaveKind<X>::value : WaveKind<Y>::value; };
template <int K, class X, class Y> struct WaveKind<Binop<K, X, Y>> : Wk2<X, Y> {};
template <class X, class Y> struct WaveKind<Pipe<X, Y>> : Wk2<X, Y> {};
template <class X, class Y> struct WaveKind<Stack<X, Y>> : Wk2<X, Y> {};
template <class X, class Y> struct WaveKind<Branch<X, Y>> : Wk2<X, Y> {};
template <class X, class Y> struct WaveKind<Bus<X, Y>> : Wk2<X, Y> {};
template <int K, class X> struct WaveKind<Unop<K, X>> : WaveKind<X> {};
template <class X> struct WaveKind<Thru<X>> : WaveKind<X> {};
template <int KIND, int OP, int N, class X> struct WaveKind<Multi<KIND, OP, N, X>> : WaveKind<X> {};
template <int NIN, class X> struct WaveKind<AllNest<NIN, X>> : WaveKind<X> {};
template <int HAD, class X> struct WaveKind<Feedback<HAD, X>> : WaveKind<X> {};
template <int HAD, class X, class Y> struct WaveKind<Feedback2<HAD, X, Y>> : Wk2<X, Y> {};


// ---------------------------------------------------------------- System<X, F> (src/system.rs:47-97, ID 67): `update(x, dt, f)`
// At the start of each of X's blocks (and before each tick) the update point test of System::process / tick: when due, the compiled
// update function f(t, dt, x) (closure text, csrc/host/closure.cpp CL_UPDATE) gives the arguments of its `x.set(..)` statements; the host
// resolved each statement to a target leaf of X (UpdTarget: its kind, the hops to it, which argument writes which of its set values). The
// set values are state words; the target's coefficients are recomputed from them with the function its host set() uses (graph.cpp), so
// the device's coefficients are the reference's bits. They are recomputed too when a launch loads the voice: its words hold the values
// the host lowered, and the sample rate may have changed (FixedSvf::set_sample_rate recomputes from the last-set cutoff). Between update
// points X runs its own block path, 8-sample groups included.
template <int... H> struct UpdAt {};
template <bool B, class T, class F> struct UpdSel { typedef T type; };
template <class T, class F> struct UpdSel<false, T, F> { typedef F type; };
template <class N, class P> struct UpdNav;   // the registers of the leaf at hops P inside N's
template <class N> struct UpdNav<N, UpdAt<>> { typedef N T; static FDSP_DEV typename N::R& get(typename N::R& r) { return r; } };
template <class X, class Y, int H, int... Hs> struct UpdNav2 {   // a binary combinator: hop 0 is X, 1 is Y
  typedef typename UpdNav<typename UpdSel<H == 0, X, Y>::type, UpdAt<Hs...>>::T T;
  template <class RR> static FDSP_DEV typename T::R& get(RR& r) {
    if constexpr (H == 0) return UpdNav<X, UpdAt<Hs...>>::get(r.x); else return UpdNav<Y, UpdAt<Hs...>>::get(r.y);
  }
};
template <class X, class Y, int H, int... Hs> struct UpdNav<Pipe<X, Y>, UpdAt<H, Hs...>> : UpdNav2<X, Y, H, Hs...> {};
template <class X, class Y, int H, int... Hs> struct UpdNav<Stack<X, Y>, UpdAt<H, Hs...>> : UpdNav2<X, Y, H, Hs...> {};
template <class X, class Y, int H, int... Hs> struct UpdNav<Branch<X, Y>, UpdAt<H, Hs...>> : UpdNav2<X, Y, H, Hs...> {};
template <class X, class Y, int H, int... Hs> struct UpdNav<Bus<X, Y>, UpdAt<H, Hs...>> : UpdNav2<X, Y, H, Hs...> {};
template <int K, class X, class Y, int H, int... Hs> struct UpdNav<Binop<K, X, Y>, UpdAt<H, Hs...>> : UpdNav2<X, Y, H, Hs...> {};
template <class X, class P> struct UpdNav1 {   // Unop / Thru: the setting passes through
  typedef typename UpdNav<X, P>::T T;
  template <class RR> static FDSP_DEV typename T::R& get(RR& r) { return UpdNav<X, P>::get(r.x); }
};
template <int K, class X, int H, int... Hs> struct UpdNav<Unop<K, X>, UpdAt<H, Hs...>> : UpdNav1<X, UpdAt<Hs...>> {};
template <class X, int H, int... Hs> struct UpdNav<Thru<X>, UpdAt<H, Hs...>> : UpdNav1<X, UpdAt<Hs...>> {};
template <int KIND, int OP, int N, class X, int H, int... Hs> struct UpdNav<Multi<KIND, OP, N, X>, UpdAt<H, Hs...>> {
  typedef typename UpdNav<X, UpdAt<Hs...>>::T T;
  template <class RR> static FDSP_DEV typename T::R& get(RR& r) { return UpdNav<X, UpdAt<Hs...>>::get(r.x[H]); }
};
// KIND (graph.cpp SystemN): 0 FixedSvf<MODE>, 1 ButterLowpass, 3 Biquad, 4 Lowpole, 5 Highpole, 6 DCBlock, 7 Constant, 8 Panner<U1> (a
// Resonator, 2, takes no setting and is never a target); its set values are sv[OFF..): (cutoff, q, gain), (cutoff), (a1, a2, b0, b1, b2),
// (cutoff), (cutoff), (cutoff), (value), (pan).
// Ak: the update's argument that writes value k (-1: none does).
template <int KIND, int MODE, int OFF, int A0, int A1, int A2, int A3, int A4, class P> struct UpdTarget {
  static FDSP_DEV void take(float* sv, const float* a) {
    if (A0 >= 0) sv[OFF] = a[A0 < 0 ? 0 : A0];
    if (A1 >= 0) sv[OFF + 1] = a[A1 < 0 ? 0 : A1];
    if (A2 >= 0) sv[OFF + 2] = a[A2 < 0 ? 0 : A2];
    if (A3 >= 0) sv[OFF + 3] = a[A3 < 0 ? 0 : A3];
    if (A4 >= 0) sv[OFF + 4] = a[A4 < 0 ? 0 : A4];
  }
  template <class X> static FDSP_DEV void apply(typename X::R& xr, const float* sv, float sr) {
    typedef typename UpdNav<X, P>::T T;
    auto& r = UpdNav<X, P>::get(xr);
    const float* v = sv + OFF;
    if constexpr (KIND == 0) { const SvfCoefs k = svf_coefs<MODE>(sr, v[0], v[1], v[2]); r.a1 = k.a1; r.a2 = k.a2; r.a3 = k.a3; r.m0 = k.m0; r.m1 = k.m1; r.m2 = k.m2; }
    else if constexpr (KIND == 1) { const BqCoefs k = bq_butter_lowpass(sr, v[0]); r.a1 = k.a1; r.a2 = k.a2; r.b0 = k.b0; r.b1 = k.b1; r.b2 = k.b2; }
    else if constexpr (KIND == 3) { r.a1 = v[0]; r.a2 = v[1]; r.b0 = v[2]; r.b1 = v[3]; r.b2 = v[4]; }
    else if constexpr (KIND >= 4 && KIND <= 6) r.coeff = onepole_coeff(KIND == 6 ? 3 : KIND - 4, sr, v[0]);
    else if constexpr (KIND == 7) { for (int c = 0; c < T::OUT; c++) r.v[c] = v[0]; }
    else pan_weights(v[0], r.lw, r.rw);
  }
};
template <class... Tg> struct UpdTargets {
  static FDSP_DEV void take(float* sv, const float* a) { (Tg::take(sv, a), ...); }
  template <class X> static FDSP_DEV void apply(typename X::R& xr, const float* sv, float sr) { (Tg::template apply<X>(xr, sv, sr), ...); }
};
template <class E> struct UpdArity;
template <class... Es> struct UpdArity<Ex::Out<Es...>> { static constexpr int value = sizeof...(Es); };
template <class A, class B> struct UpdArity<Ex::Let<A, B>> : UpdArity<B> {};

template <class X, int NSV, int NC, class E, class TG> struct System {
  static constexpr int NA = UpdArity<E>::value;
  FDSP_NODE(X::IN, X::OUT, 1 + NC + X::NP, 2 + NSV + X::NS, X::NU);
  struct R { float interval, time, dtime; float c[NC > 0 ? NC : 1]; float sv[NSV > 0 ? NSV : 1]; bool fresh; typename X::R x; };
  static FDSP_DEV void load(R& r, Loader& l) {
    r.interval = l.Pf();
#pragma unroll
    for (int k = 0; k < NC; k++) r.c[k] = l.Pf();
    r.time = l.Sf(); r.dtime = l.Sf();
#pragma unroll
    for (int k = 0; k < NSV; k++) r.sv[k] = l.Sf();
    r.fresh = true;
    X::load(r.x, l);
  }
  static FDSP_DEV void save(const R& r, Saver& s) {
    s.Sf(r.time); s.Sf(r.dtime);
#pragma unroll
    for (int k = 0; k < NSV; k++) s.Sf(r.sv[k]);
    X::save(r.x, s);
  }
  // the update point test and the clock (process :74-84 with delta_now = size / sample_rate, tick :61-72 with 1 / sample_rate); the
  // process form's `size > 0` always holds here, since the device runs no empty block
  static FDSP_DEV void advance(R& r, float sr, float delta_now) {
    if (r.fresh) { TG::template apply<X>(r.x, r.sv, sr); r.fresh = false; }
    if (r.dtime >= r.interval || r.time == 0.0f) {
      const float t[2] = {r.time, r.dtime};
      float a[NA];
      const Ex::Root s{t, r.c, 0.0f};
      Ex::Emit<E>::out(s, a);
      TG::take(r.sv, a);
      TG::template apply<X>(r.x, r.sv, sr);
      r.dtime = 0.0f;
    }
    r.time += delta_now;
    r.dtime += delta_now;
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<X::IN>& in, Fr<X::OUT>& o) {
    if (T) advance(r, c.sr, 1.0f / c.sr);
    else if (c.i == 0) advance(r, c.sr, (float)c.n / c.sr);
    X::template step<T>(r.x, c, in, o);
  }
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C& c, const Fr8<X::IN>& in, Fr8<X::OUT>& o) {
    if (c.i == 0) advance(r, c.sr, (float)c.n / c.sr);
    group_step<X>(r.x, c, in, o);
  }
  static FDSP_DEV void end_simd(R& r) { X::end_simd(r.x); }
};

// Rough per-sample instruction cost of a graph type: picks how far the 8-sample group is unrolled (big bodies
// thrash the instruction cache when only one warp runs per scheduler).
template <class G> struct Cost { static constexpr int value = 8; };
template <int K, int N> struct Cost<WaveSynth<K, N>> { static constexpr int value = 100; };
template <int K> struct Cost<PhaseSynth<K>> { static constexpr int value = 110; };
template <int M, int N> struct Cost<Mixer<M, N>> { static constexpr int value = 2 * M * N; };
template <int K> struct Cost<MeterNode<K>> { static constexpr int value = 10; };
template <int K> struct Cost<MonitorShared<K>> { static constexpr int value = 10; };
template <> struct Cost<TimerShared> { static constexpr int value = 4; };
template <> struct Cost<WavePlayer> { static constexpr int value = 12; };
template <int N> struct Cost<Limiter<N>> { static constexpr int value = 150; };
template <int N, int T> struct Cost<EnvelopeTab<N, T>> { static constexpr int value = 120; };
template <> struct Cost<Sine> { static constexpr int value = 40; };
template <> struct Cost<Noise> { static constexpr int value = 16; };
template <> struct Cost<FixedSvf> { static constexpr int value = 20; };
template <int M> struct Cost<Svf<M>> { static constexpr int value = 60; };
template <> struct Cost<Biquad> { static constexpr int value = 12; };
template <> struct Cost<BiquadBank> { static constexpr int value = 96; };
template <int N> struct Cost<Moog<N>> { static constexpr int value = 200; };
template <> struct Cost<AdsrLive> { static constexpr int value = 120; };
template <int NI, int NO, int NC, class E> struct Cost<Map<NI, NO, NC, E>> { static constexpr int value = 2 + E::cost; };
template <int NC, class E> struct Cost<ShaperFn<NC, E>> { static constexpr int value = 2 + E::cost; };
template <int NO, int NC, class E> struct Cost<VarFn<NO, NC, E>> { static constexpr int value = NO; };
template <int NI, int NO, int NC, class E> struct Cost<EnvelopeInFn<NI, NO, NC, E>> { static constexpr int value = 120; };
template <int NO, int NC, class E> struct Cost<EnvelopeFn<NO, NC, E>> { static constexpr int value = 120; };
template <class X, int NSV, int NC, class E, class TG> struct Cost<System<X, NSV, NC, E, TG>> { static constexpr int value = Cost<X>::value + 4; };
template <class X, int NSV, int NC, class E, class TG> struct WaveKind<System<X, NSV, NC, E, TG>> : WaveKind<X> {};
template <> struct Cost<Delay> { static constexpr int value = 12; };
template <int N> struct Cost<Panner<N>> { static constexpr int value = N == 1 ? 2 : 80; };
template <int K, class X, class Y> struct Cost<Binop<K, X, Y>> { static constexpr int value = Cost<X>::value + Cost<Y>::value + 1; };
template <class X, class Y> struct Cost<Pipe<X, Y>> { static constexpr int value = Cost<X>::value + Cost<Y>::value; };
template <class X, class Y> struct Cost<Stack<X, Y>> { static constexpr int value = Cost<X>::value + Cost<Y>::value; };
template <class X, class Y> struct Cost<Branch<X, Y>> { static constexpr int value = Cost<X>::value + Cost<Y>::value; };
template <class X, class Y> struct Cost<Bus<X, Y>> { static constexpr int value = Cost<X>::value + Cost<Y>::value + 1; };
template <int K, class X> struct Cost<Unop<K, X>> { static constexpr int value = Cost<X>::value + 1; };
template <class X> struct Cost<Thru<X>> { static constexpr int value = Cost<X>::value; };
template <int KIND, int OP, int N, class X> struct Cost<Multi<KIND, OP, N, X>> { static constexpr int value = N * Cost<X>::value; };
template <int NIN, class X> struct Cost<AllNest<NIN, X>> { static constexpr int value = Cost<X>::value + 6; };
template <int HAD, class X, class Y> struct Cost<Feedback2<HAD, X, Y>> { static constexpr int value = Cost<X>::value + Cost<Y>::value + (HAD ? 6 * X::IN : X::IN); };
template <int K, int N> struct Cost<OnePole<K, N>> { static constexpr int value = N > 1 ? 40 : 8; };
template <> struct Cost<Pinkpass> { static constexpr int value = 24; };
template <> struct Cost<Declick> { static constexpr int value = 24; };
template <int K> struct Cost<Chaos<K>> { static constexpr int value = 32; };
template <> struct Cost<Morph> { static constexpr int value = 64; };
template <int N> struct Cost<Rez<N>> { static constexpr int value = N > 1 ? 180 : 120; };
template <int A> struct Cost<Follower<A>> { static constexpr int value = 16; };
template <int FB, int M, int S, int N> struct Cost<NlBiquad<FB, M, S, N>> { static constexpr int value = (S == 2 ? 120 : S == 6 ? 60 : 30) * (FB ? 1 : 2) + (N > 1 ? 60 : 0); };
template <int K> struct Cost<Shaper<K>> { static constexpr int value = K == 2 ? 100 : K == 6 ? 40 : 12; };
template <int K> struct Cost<ShaperAdaptive<K>> { static constexpr int value = Cost<Shaper<K>>::value + 20; };
template <int FB, int M, int S, int N> struct Cost<NlBiquadAdaptive<FB, M, S, N>> { static constexpr int value = Cost<NlBiquad<FB, M, S, N>>::value + (FB ? 20 : 40); };
template <> struct Cost<Convolver> { static constexpr int value = 48; };
template <class X> struct WaveKind<Resample<X>> : WaveKind<X> {};
template <class X> struct Cost<Resample<X>> { static constexpr int value = 4 * Cost<X>::value + 120; };
template <class X> struct WaveKind<Event<X>> : WaveKind<X> {};
template <class X> struct Cost<Event<X>> { static constexpr int value = Cost<X>::value + 110; };
template <class X> struct WaveKind<Oversample<X>> : WaveKind<X> {};
template <class X> struct Cost<Oversample<X>> { static constexpr int value = 2 * Cost<X>::value + 150 * (X::IN + X::OUT) + 101; };
template <class X> struct WaveKind<Slot<X>> : WaveKind<X> {};
template <class X> struct Cost<Slot<X>> { static constexpr int value = 2 * Cost<X>::value + 101; };
template <class X, class Y> struct WaveKind<Xfade<X, Y>> { static constexpr int value = WaveKind<X>::value >= 0 ? WaveKind<X>::value : WaveKind<Y>::value; };
template <class X, class Y> struct Cost<Xfade<X, Y>> { static constexpr int value = Cost<X>::value + Cost<Y>::value + 101; };
template <class X> struct WaveKind<FeedbackUnit<X>> : WaveKind<X> {};
template <class X> struct Cost<FeedbackUnit<X>> { static constexpr int value = Cost<X>::value + 12 * X::IN; };
template <class F> struct Cost<Reverb85<F>> { static constexpr int value = 1200 + 16 * Cost<F>::value; };
template <class F> struct WaveKind<Reverb85<F>> : WaveKind<F> {};
template <int N> struct Cost<Dsf<N>> { static constexpr int value = 700; };
template <int NT_, int LIN> struct Cost<Tap<NT_, LIN>> { static constexpr int value = 40 * NT_; };
template <int HAD, class X> struct Cost<Feedback<HAD, X>> { static constexpr int value = Cost<X>::value + (HAD ? 6 * X::IN : X::IN); };


// ---------------------------------------------------------------- prelude64: f64 state (F = f64 in the reference's generic nodes)
// Node inputs and outputs stay f32: each input sample is widened to f64 (`convert`), each output rounded to f32. Every f64 parameter
// or state word takes two u32 words, low word first (as Event's). The sample rate a node uses is its own f64 parameter word, lowered
// from the rate the host node received (a Net hands its units the f32-rounded rate). These classes compile through NVRTC only.
FDSP_DEV double ld64p(Loader& l) { const uint32_t lo = l.P(), hi = l.P(); return __longlong_as_double((long long)(((unsigned long long)hi << 32) | lo)); }
FDSP_DEV double ld64s(Loader& l) { const uint32_t lo = l.S(), hi = l.S(); return __longlong_as_double((long long)(((unsigned long long)hi << 32) | lo)); }
FDSP_DEV void sv64(Saver& s, double v) { const unsigned long long b = (unsigned long long)__double_as_longlong(v); s.S((uint32_t)b); s.S((uint32_t)(b >> 32)); }

struct Sine64 {  // Sine<f64> src/oscillator.rs:18-102, ID 21: f64 phase and sample duration; the output is still sin(phase as f32 * f32::TAU)
  FDSP_NODE(1, 1, 2, 2, 0);
  struct R { double sd, phase; };
  static FDSP_DEV void load(R& r, Loader& l) { r.sd = ld64p(l); r.phase = ld64s(l); }
  static FDSP_DEV void save(const R& r, Saver& s) { sv64(s, r.phase); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C& c, const Fr<1>& in, Fr<1>& o) {
    const double p = r.phase;
    r.phase += (double)in.v[0] * r.sd;
    if (T || c.rem) {  // tick path :67-72
      r.phase -= floor(r.phase);
      o.v[0] = m::sinf_((float)p * TAU_F);
    } else {           // block path :74-86
      o.v[0] = wide_sinf((float)p * TAU_F);
    }
  }
  typedef void GroupStep;
  template <class C> static FDSP_DEV void step8(R& r, C&, const Fr8<1>& in, Fr8<1>& o) {
    float p[8];
    FDSP_G8 { p[j] = (float)r.phase * TAU_F; r.phase += (double)in.v[0][j] * r.sd; }
    wide_sinf8(p, o.v[0]);
  }
  static FDSP_DEV void end_simd(R& r) { r.phase = r.phase - floor(r.phase); }
};
struct Svf64K { double a1, a2, a3, m0, m1, m2; };
FDSP_DEV void svf64_tick(const Svf64K& k, double& ic1, double& ic2, float x, float& y) {   // src/svf.rs:995-1006 with F = f64
  const double v0 = (double)x;
  const double v3 = v0 - ic2;
  const double v1 = k.a1 * ic1 + k.a2 * v3;
  const double v2 = ic2 + k.a2 * ic1 + k.a3 * v3;
  ic1 = 2.0 * v1 - ic1;
  ic2 = 2.0 * v2 - ic2;
  y = (float)(k.m0 * v0 + k.m1 * v1 + k.m2 * v2);
}
struct FixedSvf64 {  // FixedSvf<f64, M> src/svf.rs:857-1031, ID 43: coefficients computed on the host (libm64.cuh)
  FDSP_NODE(1, 1, 12, 4, 0);
  struct R { Svf64K k; double ic1, ic2; };
  static FDSP_DEV void load(R& r, Loader& l) {
    r.k.a1 = ld64p(l); r.k.a2 = ld64p(l); r.k.a3 = ld64p(l); r.k.m0 = ld64p(l); r.k.m1 = ld64p(l); r.k.m2 = ld64p(l);
    r.ic1 = ld64s(l); r.ic2 = ld64s(l);
  }
  static FDSP_DEV void save(const R& r, Saver& s) { sv64(s, r.ic1); sv64(s, r.ic2); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<1>& in, Fr<1>& o) { svf64_tick(r.k, r.ic1, r.ic2, in.v[0], o.v[0]); }
  static FDSP_DEV void end_simd(R&) {}
};
template <int MODE> struct Svf64 {  // Svf<f64, M> src/svf.rs:744-855, ID 36: f64 parameters from the f32 inputs, coefficients recomputed on change
  // `ksr` is the rate the coefficients were computed at: a rate change recomputes them at the next sample, as set_sample_rate's
  // update_frequency does at once (:823-826; the inputs of that sample then decide as usual)
  static constexpr int NI = MODE >= 6 ? 4 : 3;
  FDSP_NODE(NI, 1, 2, 24, 0);
  struct R { double sr, cutoff, q, gain, ksr; Svf64K k; double ic1, ic2; };
  static FDSP_DEV void load(R& r, Loader& l) {
    r.sr = ld64p(l);
    r.cutoff = ld64s(l); r.q = ld64s(l); r.gain = ld64s(l); r.ksr = ld64s(l);
    r.k.a1 = ld64s(l); r.k.a2 = ld64s(l); r.k.a3 = ld64s(l); r.k.m0 = ld64s(l); r.k.m1 = ld64s(l); r.k.m2 = ld64s(l);
    r.ic1 = ld64s(l); r.ic2 = ld64s(l);
  }
  static FDSP_DEV void save(const R& r, Saver& s) {
    sv64(s, r.cutoff); sv64(s, r.q); sv64(s, r.gain); sv64(s, r.ksr);
    sv64(s, r.k.a1); sv64(s, r.k.a2); sv64(s, r.k.a3); sv64(s, r.k.m0); sv64(s, r.k.m1); sv64(s, r.k.m2);
    sv64(s, r.ic1); sv64(s, r.ic2);
  }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<NI>& in, Fr<1>& o) {   // update_inputs :299-313
    const double cu = (double)in.v[1], qq = (double)in.v[2], gg = (double)in.v[NI - 1];
    bool ch = cu != r.cutoff || qq != r.q || r.ksr != r.sr;
    if (MODE >= 6) ch = ch || gg != r.gain;
    if (ch) {
      r.cutoff = cu; r.q = qq; if (MODE >= 6) r.gain = gg; r.ksr = r.sr;
      const SvfCoefs64 k = svf_coefs64<MODE>(r.sr, r.cutoff, r.q, r.gain);
      r.k.a1 = k.a1; r.k.a2 = k.a2; r.k.a3 = k.a3; r.k.m0 = k.m0; r.k.m1 = k.m1; r.k.m2 = k.m2;
    }
    svf64_tick(r.k, r.ic1, r.ic2, in.v[0], o.v[0]);
  }
  static FDSP_DEV void end_simd(R&) {}
};
// ---- biquads with f64 state (src/biquad.rs:130-370, F = f64): DF1, left to right
struct Bq64 { double a1, a2, b0, b1, b2, x1, x2, y1, y2; };
FDSP_DEV void bq64_ld_coefs(Bq64& b, Loader& l, bool state) {
  if (state) { b.a1 = ld64s(l); b.a2 = ld64s(l); b.b0 = ld64s(l); b.b1 = ld64s(l); b.b2 = ld64s(l); }
  else { b.a1 = ld64p(l); b.a2 = ld64p(l); b.b0 = ld64p(l); b.b1 = ld64p(l); b.b2 = ld64p(l); }
}
FDSP_DEV void bq64_ld_state(Bq64& b, Loader& l) { b.x1 = ld64s(l); b.x2 = ld64s(l); b.y1 = ld64s(l); b.y2 = ld64s(l); }
FDSP_DEV void bq64_sv_coefs(const Bq64& b, Saver& s) { sv64(s, b.a1); sv64(s, b.a2); sv64(s, b.b0); sv64(s, b.b1); sv64(s, b.b2); }
FDSP_DEV void bq64_sv_state(const Bq64& b, Saver& s) { sv64(s, b.x1); sv64(s, b.x2); sv64(s, b.y1); sv64(s, b.y2); }
FDSP_DEV void bq64_set(Bq64& b, const BqCoefs64& k) { b.a1 = k.a1; b.a2 = k.a2; b.b0 = k.b0; b.b1 = k.b1; b.b2 = k.b2; }
FDSP_DEV float bq64_tick(Bq64& b, float x) {   // :184-194
  const double x0 = (double)x;
  const double y0 = b.b0 * x0 + b.b1 * b.x1 + b.b2 * b.x2 - b.a1 * b.y1 - b.a2 * b.y2;
  b.x2 = b.x1; b.x1 = x0; b.y2 = b.y1; b.y1 = y0;
  return (float)y0;
}
struct Biquad64 {  // Biquad<f64> ID 15, and the fixed ButterLowpass<f64, U1> ID 16 / Resonator<f64, U1> ID 17 (coefficients from the host)
  FDSP_NODE(1, 1, 10, 8, 0);
  typedef Bq64 R;
  static FDSP_DEV void load(R& r, Loader& l) { bq64_ld_coefs(r, l, false); bq64_ld_state(r, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { bq64_sv_state(r, s); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<1>& in, Fr<1>& o) { o.v[0] = bq64_tick(r, in.v[0]); }
  static FDSP_DEV void end_simd(R&) {}
};
// ButterLowpass<f64, U2> (KIND 0, inputs audio, cutoff) and Resonator<f64, U3> (KIND 1, inputs audio, center, q): coefficients recomputed
// when an input changes (:270-278, :355-366) or the rate did (`ksr`, as in Svf64)
template <int KIND> struct BiquadAudio64 {
  static constexpr int NI = KIND == 0 ? 2 : 3;
  FDSP_NODE(NI, 1, 2, 24, 0);
  struct R { double sr, f, q, ksr; Bq64 b; };
  static FDSP_DEV void load(R& r, Loader& l) { r.sr = ld64p(l); r.f = ld64s(l); r.q = ld64s(l); r.ksr = ld64s(l); bq64_ld_coefs(r.b, l, true); bq64_ld_state(r.b, l); }
  static FDSP_DEV void save(const R& r, Saver& s) { sv64(s, r.f); sv64(s, r.q); sv64(s, r.ksr); bq64_sv_coefs(r.b, s); bq64_sv_state(r.b, s); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<NI>& in, Fr<1>& o) {
    const double f = (double)in.v[1], q = KIND == 0 ? r.q : (double)in.v[NI - 1];
    if (f != r.f || q != r.q || r.ksr != r.sr) {
      r.f = f; r.q = q; r.ksr = r.sr;
      bq64_set(r.b, KIND == 0 ? bq_butter_lowpass64(r.sr, r.f) : bq_resonator64(r.sr, r.f, r.q));
    }
    o.v[0] = bq64_tick(r.b, in.v[0]);
  }
  static FDSP_DEV void end_simd(R&) {}
};
// ---- one-pole family with f64 state (src/filter.rs, F = f64): KIND 0 Lowpole (ID 18), 1 Highpole (ID 47), 2 Allpole (ID 46),
// 3 DCBlock (ID 22); NIN = 2 adds the audio-rate parameter input (cutoff: recomputed on change or after a rate change; allpole delay:
// every sample, :315-317)
template <int KIND, int NIN> struct OnePole64 {
  FDSP_NODE(NIN, 1, 2, (KIND == 0 ? 2 : 4) + (NIN > 1 ? 6 : 0), 0);
  struct R { double sr, coeff, param, ksr, x1, y1; };
  static FDSP_DEV void load(R& r, Loader& l) {
    if (NIN == 1) { r.coeff = ld64p(l); r.sr = r.param = r.ksr = 0.0; } else { r.sr = ld64p(l); r.param = ld64s(l); r.ksr = ld64s(l); r.coeff = ld64s(l); }
    r.x1 = (KIND == 0) ? 0.0 : ld64s(l); r.y1 = ld64s(l);
  }
  static FDSP_DEV void save(const R& r, Saver& s) { if (NIN > 1) { sv64(s, r.param); sv64(s, r.ksr); sv64(s, r.coeff); } if (KIND != 0) sv64(s, r.x1); sv64(s, r.y1); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<NIN>& in, Fr<1>& o) {
    if (NIN > 1) {
      const double p = (double)in.v[NIN > 1 ? 1 : 0];
      if (KIND == 2) r.coeff = onepole_coeff64(2, r.sr, p);
      else if (p != r.param || r.ksr != r.sr) { r.param = p; r.ksr = r.sr; r.coeff = onepole_coeff64(KIND, r.sr, p); }
    }
    const double x = (double)in.v[0];
    double y0;
    if (KIND == 0) y0 = (1.0 - r.coeff) * x + r.coeff * r.y1;
    else if (KIND == 1) y0 = r.coeff * (r.y1 + x - r.x1);
    else if (KIND == 2) y0 = r.coeff * (x - r.y1) + r.x1;
    else y0 = x - r.x1 + r.coeff * r.y1;
    r.x1 = x; r.y1 = y0;
    o.v[0] = (float)y0;
  }
  static FDSP_DEV void end_simd(R&) {}
};
struct Pinkpass64 {  // Pinkpass<f64> src/filter.rs:178-262, ID 26
  FDSP_NODE(1, 1, 0, 14, 0);
  struct R { double b[7]; };
  static FDSP_DEV void load(R& r, Loader& l) { for (int k = 0; k < 7; k++) r.b[k] = ld64s(l); }
  static FDSP_DEV void save(const R& r, Saver& s) { for (int k = 0; k < 7; k++) sv64(s, r.b[k]); }
  template <bool T, class C> static FDSP_DEV void step(R& r, const C&, const Fr<1>& in, Fr<1>& o) {
    const double x = (double)in.v[0];
    r.b[0] = 0.99886 * r.b[0] + x * 0.0555179;
    r.b[1] = 0.99332 * r.b[1] + x * 0.0750759;
    r.b[2] = 0.96900 * r.b[2] + x * 0.1538520;
    r.b[3] = 0.86650 * r.b[3] + x * 0.3104856;
    r.b[4] = 0.55000 * r.b[4] + x * 0.5329522;
    r.b[5] = -0.7616 * r.b[5] - x * 0.0168980;
    o.v[0] = (float)((r.b[0] + r.b[1] + r.b[2] + r.b[3] + r.b[4] + r.b[5] + r.b[6] + x * 0.5362) * 0.115830421);
    r.b[6] = x * 0.115926;
  }
  static FDSP_DEV void end_simd(R&) {}
};
template <> struct Cost<Sine64> { static constexpr int value = 48; };
template <> struct Cost<FixedSvf64> { static constexpr int value = 24; };
template <int M> struct Cost<Svf64<M>> { static constexpr int value = 80; };
template <> struct Cost<Biquad64> { static constexpr int value = 16; };
template <int K> struct Cost<BiquadAudio64<K>> { static constexpr int value = 90; };
template <int K, int N> struct Cost<OnePole64<K, N>> { static constexpr int value = N > 1 ? 60 : 10; };
template <> struct Cost<Pinkpass64> { static constexpr int value = 30; };

// ---- traits of a Dag: sums / first match over its vertices
template <int... X> struct FirstNonNeg { static constexpr int value = -1; };
template <int H, int... T> struct FirstNonNeg<H, T...> { static constexpr int value = H >= 0 ? H : FirstNonNeg<T...>::value; };
template <int NIN, int NOUT, class... V, class OS> struct WaveKind<Dag<NIN, NOUT, VList<V...>, OS>> { static constexpr int value = FirstNonNeg<WaveKind<typename V::Unit>::value...>::value; };
template <int NIN, int NOUT, class... V, class OS> struct Cost<Dag<NIN, NOUT, VList<V...>, OS>> { static constexpr int value = (2 + ... + Cost<typename V::Unit>::value); };

// ---- group-evaluation plan: instructions the 8-sample group form of G unrolls to (per sample), and whether every heavy leaf is
// narrow enough to rotate; the kernel uses the group form when ok && code <= FDSP_GROUP_COST
template <class G> struct GroupPlan {
  static constexpr bool heavy = !HasGroup<G>::value && Cost<G>::value > FDSP_ROTATE_COST;
  static constexpr bool ok = !heavy || (G::IN + G::OUT <= 6);
  static constexpr int code = heavy ? Cost<G>::value / 8 + 2 * (G::IN + G::OUT) : Cost<G>::value;
};
template <class X, class Y> struct Plan2 { static constexpr bool ok = GroupPlan<X>::ok && GroupPlan<Y>::ok; static constexpr int code = GroupPlan<X>::code + GroupPlan<Y>::code + 1; };
template <int K, class X, class Y> struct GroupPlan<Binop<K, X, Y>> : Plan2<X, Y> {};
template <class X, class Y> struct GroupPlan<Pipe<X, Y>> : Plan2<X, Y> {};
template <class X, class Y> struct GroupPlan<Stack<X, Y>> : Plan2<X, Y> {};
template <class X, class Y> struct GroupPlan<Branch<X, Y>> : Plan2<X, Y> {};
template <class X, class Y> struct GroupPlan<Bus<X, Y>> : Plan2<X, Y> {};
template <int K, class X> struct GroupPlan<Unop<K, X>> { static constexpr bool ok = GroupPlan<X>::ok; static constexpr int code = GroupPlan<X>::code + 1; };
template <class X> struct GroupPlan<Thru<X>> : GroupPlan<X> {};
template <int KIND, int OP, int N, class X> struct GroupPlan<Multi<KIND, OP, N, X>> { static constexpr bool ok = GroupPlan<X>::ok; static constexpr int code = N * GroupPlan<X>::code; };

template <class X> struct GroupPlan<Slot<X>> { static constexpr bool ok = GroupPlan<X>::ok; static constexpr int code = GroupPlan<X>::code + 16; };
template <class X, class Y> struct GroupPlan<Xfade<X, Y>> { static constexpr bool ok = GroupPlan<X>::ok && GroupPlan<Y>::ok; static constexpr int code = GroupPlan<X>::code + GroupPlan<Y>::code + 16; };
template <class X, int NSV, int NC, class E, class TG> struct GroupPlan<System<X, NSV, NC, E, TG>> { static constexpr bool ok = GroupPlan<X>::ok; static constexpr int code = GroupPlan<X>::code + 4; };
template <class X> struct GroupPlan<Event<X>> { static constexpr bool ok = GroupPlan<X>::ok; static constexpr int code = GroupPlan<X>::code + 24; };
template <int NIN, int NOUT, class... V, class OS> struct GroupPlan<Dag<NIN, NOUT, VList<V...>, OS>> {
  static constexpr bool ok = (true && ... && GroupPlan<typename V::Unit>::ok);
  static constexpr int code = (2 + ... + GroupPlan<typename V::Unit>::code);
};

}  // namespace fdsp
