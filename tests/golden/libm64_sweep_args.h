// TEST INFRASTRUCTURE: the arguments and the per-chunk hash of the f64 math sweep (sin, cos, tan, exp of csrc/dsp/libm64.cuh), shared by
// the host generator of the expected hashes (tests/golden/gen_libm64_sweep.cpp, which evaluates the ORACLE, oracle/fo_libm64.h) and the
// device probe (tools/probe/libm64_sweep_probe.cu, which evaluates the PRODUCT, compiled by nvcc and by NVRTC). Neither the product's
// nor the oracle's math is in here, only which argument index i stands for.
//
// Every function has the same 514 chunks. Chunk c < 512 (set a, 2^33 arguments): every high word h = i >> 1 of both signs, with the low
// word 0 on even i and a hash of h on odd i. Chunk 512 (set b, 2^24 points): the domain the filters evaluate, x = lo + (hi - lo) t with
// t in [0, 1) spread evenly: tan on [0, pi/2), cos and sin on [0, 2 pi], exp on [-746, 710]. Chunk 513 (set c, NSPECIAL arguments):
//   the high words where rem_pio2 changes branch and the multiples of pi/4 near them, the small-argument cut-offs, and exp's overflow,
//   underflow and reduction cut-offs, each +- 64 ulps; the 2^20 pi/2 threshold of the large reduction (0x413921fb00000000) +- 4096 ulps;
//   the doubles nearest k pi/2 for k = floor(2^e (1 + u)), e = 0, 8, ..., 1000, u uniform (mpmath, 2200 bits), +- 2 ulps;
//   0x7506ac5b262ca1ff, the double nearest a multiple of pi/2 (x mod pi/2 = 4.687e-19), subnormals, zeros, DBL_MIN, DBL_MAX, infinities,
//   NaNs; every one with both signs.
// A chunk's hash is the sum over its i of splitmix64(splitmix64(i) + canon(bits(f(x_i)))) mod 2^64, which does not depend on the order
// of evaluation; canon maps every NaN to 0x7ff8000000000000 and keeps every other pattern (both zeros).
#pragma once
#if defined(__CUDACC__)
#define SWEEP64_HD __host__ __device__ __forceinline__
#else
#define SWEEP64_HD static inline
#endif
#ifndef __CUDACC_RTC__
#include <cstdint>
#include <cstring>
#endif

namespace sweep64 {

enum { SIN, COS, TAN, EXP, NFN };
#define SWEEP64_NAMES {"sin", "cos", "tan", "exp"}
constexpr int CHUNK_LOG2 = 24;
constexpr int CHUNKS = 514, CHUNK_DOMAIN = 512, CHUNK_SPECIAL = 513;

SWEEP64_HD uint64_t splitmix64(uint64_t z) {
  z += 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}
SWEEP64_HD uint64_t canon(uint64_t b) { return (b & 0x7fffffffffffffffull) > 0x7ff0000000000000ull ? 0x7ff8000000000000ull : b; }
SWEEP64_HD uint64_t term(uint64_t i, uint64_t result_bits) { return splitmix64(splitmix64(i) + canon(result_bits)); }
SWEEP64_HD double as_double(uint64_t u) {
#ifdef __CUDA_ARCH__
  return __longlong_as_double((long long)u);
#else
  double x; memcpy(&x, &u, 8); return x;
#endif
}

// set c, as positive patterns; the sign is the lowest bit of the index within the set
constexpr int NCENTER = 34, CENTER_R = 64, THRESHOLD_R = 4096, NKPIO2 = 126, KPIO2_R = 2, NSINGLE = 16;
SWEEP64_HD uint64_t center(int k) {
  const uint64_t C[NCENTER] = {
    // rem_pio2's branch words: the first pattern of the word and of the next one
    0x400f6a7a00000000ull, 0x400f6a7b00000000ull, 0x4002d97c00000000ull, 0x4002d97d00000000ull, 0x4015fdbc00000000ull, 0x4015fdbd00000000ull,
    0x4012d97c00000000ull, 0x4012d97d00000000ull, 0x401c463b00000000ull, 0x401c463c00000000ull, 0x401921fb00000000ull, 0x401921fc00000000ull,
    0x3ff921fb00000000ull, 0x3ff921fc00000000ull, 0x400921fb00000000ull, 0x400921fc00000000ull,
    // the doubles nearest pi/4 (the kernels' limit), pi/2, 3pi/4, pi, 5pi/4, 3pi/2, 7pi/4, 2pi, 9pi/4
    0x3fe921fb54442d18ull, 0x3ff921fb54442d18ull, 0x4002d97c7f3321d2ull, 0x400921fb54442d18ull, 0x400f6a7a2955385eull, 0x4012d97c7f3321d2ull,
    0x4015fdbbe9bba775ull, 0x401921fb54442d18ull, 0x401c463abeccb2bbull,
    // the small-argument cut-offs of sin, cos and tan; exp's 2^-28, ln2 / 2 and 1.5 ln2 cut-offs
    0x3e50000000000000ull, 0x3e46a09e00000000ull, 0x3e40000000000000ull, 0x3e30000100000000ull, 0x3fd62e4300000000ull, 0x3ff0a2b200000000ull,
    // exp: the largest finite result, the smallest subnormal one (as -x), and |x| = 708.39 where the careful tests begin
    0x40862e42fefa39efull, 0x40874910d52d3051ull, 0x4086232b00000000ull};
  return C[k];
}
SWEEP64_HD uint64_t kpio2(int k) {   // the doubles nearest k pi/2, k = floor(2^e (1 + u)) for e = 0, 8, ..., 1000
  const uint64_t K[NKPIO2] = {
    0x3ff921fb54442d18ull, 0x407e23c0660dc214ull, 0x41066148833b6d80ull, 0x41876aeef624a8edull, 0x4202e0f7fc04032full,
    0x42836a4e17d04429ull, 0x42fc099e3baa4ab2ull, 0x437eaea41bb9238eull, 0x43fa8a5fc09039dbull, 0x447ffc2a1299e001ull,
    0x4503cd370f9dac58ull, 0x45874214124754b6ull, 0x45fdccbba1bf81e4ull, 0x468359206d1336f0ull, 0x470829220a3dd50bull,
    0x477f276dfea4b8c3ull, 0x4806970585e90600ull, 0x4887d89a3ffd6dd4ull, 0x48fbeba5da6b2255ull, 0x4983f6a3de2a7cafull,
    0x4a0839eaf454df57ull, 0x4a843163362c008full, 0x4b06da969e0a69a4ull, 0x4b87922033098e6cull, 0x4c02dddb150a29a9ull,
    0x4c87a176f09407b3ull, 0x4cfb8e7029e25712ull, 0x4d87f22a37eaa4e1ull, 0x4e02a9d0e9a7e426ull, 0x4e86e3097af7be63ull,
    0x4f038ed08aaca66bull, 0x4f8539697ce8834cull, 0x500670295b572655ull, 0x50846d4e6ded00e3ull, 0x510829503030d2a4ull,
    0x5183b48d43396577ull, 0x51f9f13a156dd3a7ull, 0x528372ed9f0b5f9eull, 0x530585f2c1137b62ull, 0x5387e7a1ab025504ull,
    0x53fb9415744eda67ull, 0x547a96903e319529ull, 0x5505780db3c578bcull, 0x558257ca74936d45ull, 0x55fedf28ccd7eae6ull,
    0x5688f951c6e61ed0ull, 0x57028465979f2292ull, 0x578301b23800ca4full, 0x58077b784b4dc78cull, 0x5881fa714315769bull,
    0x58fe1958b89ce05aull, 0x5985f9d1e3f7224eull, 0x5a0878d3f996e5abull, 0x5a83c177ff20a573ull, 0x5b06f2463f39cf23ull,
    0x5b7e18d768b7ca22ull, 0x5c08f163ec574f95ull, 0x5c7c7eb010e453f2ull, 0x5cfc1966764672aaull, 0x5d81a668a03148deull,
    0x5dfe2e6aa3b4ad2bull, 0x5e87ce855dc9888eull, 0x5f0144f9eac01e96ull, 0x5f85683594333b92ull, 0x5ffe42a9c915d0bfull,
    0x607c0ad2124d687cull, 0x6103f7d38ae60404ull, 0x618461d954cd3d2bull, 0x61fef4effc28e3bbull, 0x627ceac608286fc3ull,
    0x6302ece2e5feb348ull, 0x637b241770555e39ull, 0x6408afcf8e8a32abull, 0x648113f7cd60d9dbull, 0x65053404efa98242ull,
    0x6581b85a146b391cull, 0x6601962a7bf1a571ull, 0x66882b26c395673cull, 0x670410abe6d69acbull, 0x67822b1686f3bd93ull,
    0x6806bc101f59a834ull, 0x687f9562b2f72d98ull, 0x690157c45bce1061ull, 0x69871915205761c2ull, 0x6a009732b486d779ull,
    0x6a79ad906ba1677bull, 0x6b07fc341344b917ull, 0x6b7a318a69805d68ull, 0x6c07f03afb3253e4ull, 0x6c8387494ae2f8ddull,
    0x6d05b24bb0df3a53ull, 0x6d88860b0a127b85ull, 0x6e090f071dfb7b60ull, 0x6e7a4461a0c2973full, 0x6f06411fc384c842ull,
    0x6f818b49c0baf215ull, 0x7006021a6d43ab4cull, 0x708150bf6ddf6c2cull, 0x7106d85b01d4bcf0ull, 0x718686744e8eeeb1ull,
    0x71fbd165673b6bc0ull, 0x72822cc0c58471b7ull, 0x72fd067163d89463ull, 0x737bb77b69d868f7ull, 0x73fe39a3d2d8b083ull,
    0x747d58f3bc9157f8ull, 0x7508d185555ba5e4ull, 0x7587adbc7c3260f9ull, 0x7606d8ced07c1e56ull, 0x7687b866bf537493ull,
    0x76fa5a7f80d30750ull, 0x778591d2005ad269ull, 0x77fd4943731a7384ull, 0x788450551fbab7e5ull, 0x79043b895488184cull,
    0x798457e82a6003cbull, 0x7a0014797966aff1ull, 0x7a80db77bec1a02full, 0x7b038e677b4a4b72ull, 0x7b83d1bf159339a8ull,
    0x7c05fc1cad8cc9a6ull, 0x7c7a8c8624dcb416ull, 0x7cfd8f6a80a6cdabull, 0x7d8524c7ed644ddaull, 0x7e008b585a78bea8ull,
    0x7e865f7854f348ccull};
  return K[k];
}
SWEEP64_HD uint64_t single(int k) {
  const uint64_t S[NSINGLE] = {0x7506ac5b262ca1ffull, 0x0000000000000000ull, 0x0000000000000001ull, 0x0000000000000002ull,
                               0x000fffffffffffffull, 0x0008000000000000ull, 0x0000000123456789ull, 0x0010000000000000ull,
                               0x7fefffffffffffffull, 0x7feffffffffffffeull, 0x7ff0000000000000ull, 0x7ff8000000000000ull,
                               0x7ff0000000000001ull, 0x7fffffffffffffffull, 0x3ff0000000000000ull, 0x4000000000000000ull};
  return S[k];
}
constexpr int NC_ARGS = NCENTER * (2 * CENTER_R + 1), NT_ARGS = 2 * THRESHOLD_R + 1, NK_ARGS = NKPIO2 * (2 * KPIO2_R + 1);
constexpr int NSPECIAL = 2 * (NC_ARGS + NT_ARGS + NK_ARGS + NSINGLE);

SWEEP64_HD uint32_t chunk_len(int c) { return c == CHUNK_SPECIAL ? (uint32_t)NSPECIAL : (1u << CHUNK_LOG2); }

// bit pattern of the argument of function fn at index i
SWEEP64_HD uint64_t arg_bits(int fn, uint64_t i) {
  const int c = (int)(i >> CHUNK_LOG2);
  if (c < CHUNK_DOMAIN) {
    const uint64_t h = i >> 1;
    return (h << 32) | ((i & 1) ? (splitmix64(h) & 0xffffffffull) : 0ull);
  }
  const uint32_t j = (uint32_t)(i & ((1ull << CHUNK_LOG2) - 1));
  if (c == CHUNK_DOMAIN) {
    const double PI = 3.14159265358979323846;
    const double lo = fn == EXP ? -746.0 : 0.0, hi = fn == EXP ? 710.0 : fn == TAN ? PI / 2.0 : 2.0 * PI;
    const double t = (double)j * 0x1p-24 + (double)(splitmix64(j) >> 40) * 0x1p-48;   // < 1: j / 2^24 plus a hashed fraction of 2^-24
    const double x = lo + (hi - lo) * t;
    uint64_t u;
#ifdef __CUDA_ARCH__
    u = (uint64_t)__double_as_longlong(x);
#else
    memcpy(&u, &x, 8);
#endif
    return u;
  }
  const uint64_t sign = (uint64_t)(j & 1) << 63;
  int k = (int)(j >> 1);
  if (k < NC_ARGS) return sign | (center(k / (2 * CENTER_R + 1)) + (uint64_t)(k % (2 * CENTER_R + 1)) - CENTER_R);
  k -= NC_ARGS;
  if (k < NT_ARGS) return sign | (0x413921fb00000000ull + (uint64_t)k - THRESHOLD_R);
  k -= NT_ARGS;
  if (k < NK_ARGS) return sign | (kpio2(k / (2 * KPIO2_R + 1)) + (uint64_t)(k % (2 * KPIO2_R + 1)) - KPIO2_R);
  k -= NK_ARGS;
  return sign | single(k);
}

}  // namespace sweep64
