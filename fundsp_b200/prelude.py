"""Opcode vocabulary: the hot-path subset of the reference's `prelude32` (src/prelude.rs, F = f32).

Every function returns an `An` expression and cites the reference constructor it mirrors
(file:line relative to the reference crate (SamiPerttu/fundsp v0.23.0)).  Names, argument order and argument meaning follow the
reference; `pass` is spelled `pass_` (Python keyword).  Anything that needs a Rust closure
(`envelope(|t| ..)`, `map`, `shape_fn`) cannot cross a C ABI and is intentionally absent;
`adsr_live` is a closed-form opcode (src/adsr.rs:21-70).
"""
from __future__ import annotations

import math

import numpy as np

from .graph import (An, ArityError, _arity, M_BRANCH, M_BUS, M_CHAIN, M_REDUCE, M_STACK, OP_ADD, OP_MUL, f32, multi)

F = np.float32

# SVF modes (src/svf.rs:26-221)
LOWPASS, HIGHPASS, BANDPASS, NOTCH, PEAK, ALLPASS, BELL, LOWSHELF, HIGHSHELF = range(9)
# global wavetables (src/wavetable.rs:493-623)
SAW, SQUARE, TRIANGLE, ORGAN, SOFT_SAW, HAMMOND = range(6)


def _frame(x):
    return tuple(f32(v) for v in (x if isinstance(x, (tuple, list)) else (x,)))


# ---- src/prelude.rs:189-235
def constant(x):
    v = _frame(x)
    return An("constant", (v,), (), 0, len(v))


dc = constant


def zero():
    return dc(0.0)


def multizero(n):
    return dc((0.0,) * n)


# ---- src/prelude.rs:257-330
def pass_():
    return An("pass", (), (), 1, 1)


def multipass(n):
    return An("multipass", (n,), (), n, n)


def sink():
    return An("sink", (1,), (), 1, 0)


def multisink(n):
    return An("sink", (n,), (), n, 0)


def reverse(n):
    return An("reverse", (n,), (), n, n)


# ---- src/prelude.rs:1675-1715
def split(n):
    return An("split", (n,), (), 1, n)


def multisplit(m, n):
    return An("multisplit", (m, n), (), m, m * n)


def join(n):
    return An("join", (n,), (), n, 1)


def multijoin(m, n):
    return An("multijoin", (m, n), (), m * n, m)


# ---- src/prelude.rs:337-351
def sine():
    return An("sine", (), (), 1, 1)


def sine_hz(f):
    return constant(f) >> sine()


# ---- src/prelude.rs:2003-2089 wavetable oscillators
def _wave(kind):
    return An("wavesynth", (kind, 1), (), 1, 1)


def saw():
    return _wave(SAW)


def square():
    return _wave(SQUARE)


def triangle():
    return _wave(TRIANGLE)


def organ():
    return _wave(ORGAN)


def soft_saw():
    return _wave(SOFT_SAW)


def hammond():
    return _wave(HAMMOND)


def saw_hz(f):
    return constant(f) >> saw()


def square_hz(f):
    return constant(f) >> square()


def triangle_hz(f):
    return constant(f) >> triangle()


def organ_hz(f):
    return constant(f) >> organ()


def soft_saw_hz(f):
    return constant(f) >> soft_saw()


def hammond_hz(f):
    return constant(f) >> hammond()


# ---- src/prelude.rs:808-823
def noise():
    return An("noise", (), (), 0, 1)


white = noise


# ---- src/prelude.rs:2096-2560 Simper SVF family.  `x()` takes parameter inputs, `x_hz` is fixed, `x_q` fixes Q.
def _svf(mode):
    gain_in = mode >= BELL
    return An("svf", (mode, 440.0, 1.0, 1.0), (), 4 if gain_in else 3, 1)


def _svf_hz(mode, f, q, gain=1.0):
    return An("fixed_svf", (mode, f32(f), f32(q), f32(gain)), (), 1, 1)


def _svf_q(mode, q, gain=None):
    n = An("svf", (mode, 440.0, f32(q), 1.0 if gain is None else f32(gain)), (), 3 if gain is None else 4, 1)
    tail = dc(q) if gain is None else dc((q, gain))
    return (multipass(2) | tail) >> n


def lowpass():
    return _svf(LOWPASS)


def lowpass_hz(f, q):
    return _svf_hz(LOWPASS, f, q)


def lowpass_q(q):
    return _svf_q(LOWPASS, q)


def highpass():
    return _svf(HIGHPASS)


def highpass_hz(f, q):
    return _svf_hz(HIGHPASS, f, q)


def highpass_q(q):
    return _svf_q(HIGHPASS, q)


def bandpass():
    return _svf(BANDPASS)


def bandpass_hz(f, q):
    return _svf_hz(BANDPASS, f, q)


def bandpass_q(q):
    return _svf_q(BANDPASS, q)


def notch():
    return _svf(NOTCH)


def notch_hz(f, q):
    return _svf_hz(NOTCH, f, q)


def notch_q(q):
    return _svf_q(NOTCH, q)


def peak():
    return _svf(PEAK)


def peak_hz(f, q):
    return _svf_hz(PEAK, f, q)


def peak_q(q):
    return _svf_q(PEAK, q)


def allpass():
    return _svf(ALLPASS)


def allpass_hz(f, q):
    return _svf_hz(ALLPASS, f, q)


def allpass_q(q):
    return _svf_q(ALLPASS, q)


def bell():
    return _svf(BELL)


def bell_hz(f, q, gain):
    return _svf_hz(BELL, f, q, gain)


def bell_q(q, gain):
    return _svf_q(BELL, q, gain)


def lowshelf():
    return _svf(LOWSHELF)


def lowshelf_hz(f, q, gain):
    return _svf_hz(LOWSHELF, f, q, gain)


def lowshelf_q(q, gain):
    return _svf_q(LOWSHELF, q, gain)


def highshelf():
    return _svf(HIGHSHELF)


def highshelf_hz(f, q, gain):
    return _svf_hz(HIGHSHELF, f, q, gain)


def highshelf_q(q, gain):
    return _svf_q(HIGHSHELF, q, gain)


# ---- src/prelude.rs:441-548, src/prelude32.rs:2711-2713
def biquad(a1, a2, b0, b1, b2):
    return An("biquad", (f32(a1), f32(a2), f32(b0), f32(b1), f32(b2)), (), 1, 1)


def biquad_bank():
    return An("biquad_bank", (), (), 8, 8)


def butterpass():
    return An("butterpass", (440.0, 2), (), 2, 1)


def butterpass_hz(f):
    return An("butterpass", (f32(f), 1), (), 1, 1)


def resonator():
    return An("resonator", (440.0, 1.0, 3), (), 3, 1)


def resonator_hz(center, q):
    return An("resonator", (f32(center), f32(q), 1), (), 1, 1)


# ---- src/prelude.rs:551-568
def moog():
    return An("moog", (1000.0, f32(0.1), 3), (), 3, 1)


def moog_q(q):
    return (multipass(2) | dc(q)) >> An("moog", (1000.0, f32(q), 3), (), 3, 1)


def moog_hz(frequency, q):
    return An("moog", (f32(frequency), f32(q), 1), (), 1, 1)


# ---- src/prelude.rs:855-867
def fir(weights):
    w = _frame(weights)
    return An("fir", (w,), (), 1, 1)


def fir3_weights(gain):
    alpha = (F(gain) + F(1.0)) / F(2.0)
    beta = (F(1.0) - alpha) / F(2.0)
    return (float(beta), float(alpha), float(beta))


def fir3(gain):
    return fir(fir3_weights(gain))


# ---- src/prelude.rs:878-912
def tick():
    return An("tick", (1,), (), 1, 1)


def multitick(n):
    return An("tick", (n,), (), n, n)


def delay(t):
    return An("delay", (float(t),), (), 1, 1)


# ---- src/prelude.rs:1102-1135
def allnest_c(coefficient, x):
    return An("allnest", (f32(coefficient), 1), (x,), 1, 1)


def allnest(x):
    return An("allnest", (0.0, 2), (x,), 2, 1)


# ---- src/prelude.rs:1236-1256
def panner():
    return An("panner", (), (), 2, 2)


def pan(p):
    return An("pan", (f32(p),), (), 1, 2)


# ---- src/prelude.rs:766-775 / src/adsr.rs:21-70
def adsr_live(attack, decay, sustain, release):
    return An("adsr_live", (f32(attack), f32(decay), f32(sustain), f32(release)), (), 1, 1)


# ---- src/prelude.rs:1053-1085, 1336-1364
def feedback(node):
    return An("feedback", (0,), (node,), node.nin, node.nout)


def fdn(node):
    return An("feedback", (1,), (node,), node.nin, node.nout)


# ---- src/prelude.rs:1370-1670 functional forms of the operators and the indexed multi-combinators
def bus(x, y):
    return x & y


def stack(x, y):
    return x | y


def branch(x, y):
    return x ^ y


def pipe(x, y):
    return x >> y


def thru(x):
    return ~x


def product(x, y):
    return x * y


def sum(x, y):  # noqa: A001 (mirrors the reference name)
    return x + y


def busi(n, f):
    return multi(M_BUS, 0, [f(i) for i in range(n)])


def _frac(n, i):
    return f32(i / (n - 1)) if n > 1 else 0.5


def busf(n, f):
    return multi(M_BUS, 0, [f(_frac(n, i)) for i in range(n)])


def stacki(n, f):
    return multi(M_STACK, 0, [f(i) for i in range(n)])


def stackf(n, f):
    return multi(M_STACK, 0, [f(_frac(n, i)) for i in range(n)])


def branchi(n, f):
    return multi(M_BRANCH, 0, [f(i) for i in range(n)])


def branchf(n, f):
    return multi(M_BRANCH, 0, [f(_frac(n, i)) for i in range(n)])


def sumi(n, f):
    return multi(M_REDUCE, OP_ADD, [f(i) for i in range(n)])


def sumf(n, f):
    return multi(M_REDUCE, OP_ADD, [f(_frac(n, i)) for i in range(n)])


def pipei(n, f):
    return multi(M_CHAIN, 0, [f(i) for i in range(n)])


def pipef(n, f):
    return multi(M_CHAIN, 0, [f(_frac(n, i)) for i in range(n)])


# ---- f32 math used by the composites (src/math.rs:170-177, 430-437, 289-291)
def lerp(a, b, t):
    a, b, t = F(a), F(b), F(t)
    return float(a * (F(1.0) - t) + b * t)


def smooth9(x):
    x = F(x)
    x2 = x * x
    return float(((((F(70) * x - F(315)) * x + F(540)) * x - F(420)) * x + F(126)) * x2 * x2 * x)


def db_amp(db):
    return math.exp((db / 20.0) * math.log(10.0))


def xerp(a, b, t):
    """f32 xerp (src/math.rs:236-238) as used for per-voice parameter draws."""
    a, b, t = F(a), F(b), F(t)
    la, lb = np.log(a), np.log(b)
    return float(np.exp(la * (F(1.0) - t) + lb * t))


REVERB_DELAYS = (
    0.073904, 0.052918, 0.066238, 0.066387, 0.037783, 0.080073, 0.050961, 0.075900, 0.043646,
    0.072095, 0.056194, 0.045961, 0.058934, 0.068016, 0.047529, 0.058156, 0.072972, 0.036084,
    0.062715, 0.076377, 0.044339, 0.076725, 0.077884, 0.046126, 0.067741, 0.049800, 0.051709,
    0.082923, 0.070121, 0.079315, 0.055039, 0.081859,
)


# ---- src/prelude.rs:1732-1762
def reverb_stereo(room_size, time, damping):
    a = F(math.pow(db_amp(-60.0), 0.03 * room_size / 10.0 / time))
    w = fir3_weights(f32(1.0) - f32(damping))
    weights = tuple(float(F(x) * a) for x in w)
    line = stacki(32, lambda i: delay(REVERB_DELAYS[i] * room_size / 10.0) >> fir(weights))
    reverb = fdn(line)
    return (multisplit(2, 16) >> reverb
            >> sumf(32, lambda x: pan(lerp(-1.0, 1.0, smooth9(x)))) * dc((1.0 / 16.0, 1.0 / 16.0)))


# ---- src/prelude.rs:1873-1946 reverb4_stereo: two 16-line Hadamard FDNs in series (delay times from the reference's optimiser run)
REVERB4_DELAYS = (
    0.059326634, 0.04778291, 0.06995449, 0.0393001, 0.041604012, 0.06215825, 0.052269846, 0.043227978,
    0.06966107, 0.031615064, 0.068442, 0.037332155, 0.032944717, 0.034493037, 0.06787566, 0.038824916,
    0.068260126, 0.068044715, 0.0688076, 0.066724524, 0.051293883, 0.06023173, 0.040897705, 0.031507637,
    0.060309593, 0.049584292, 0.04532072, 0.056379095, 0.035180368, 0.041291796, 0.046129026, 0.05504605,
)


def reverb4_stereo_delays(delays, time):
    _arity(len(delays) == 32, "reverb4_stereo_delays: 32 delay times")
    d = [F(x) for x in delays]
    a = F(math.pow(db_amp(-60.0), 0.03 * 10.0 / 10.0 / time))
    w = (float(-a / F(4.0)), float(-a / F(2.0)), float(-a / F(4.0)))
    line1 = stacki(16, lambda i: delay(float(d[i])) >> fir(w))
    line2 = stacki(16, lambda i: delay(float(d[16 + i])) >> fir(w))
    return (multisplit(2, 8) >> fdn(line1) >> multijoin(2, 8) >> multisplit(2, 8) >> fdn(line2)
            >> sumf(16, lambda x: pan(lerp(-1.0, 1.0, smooth9(x)))) * dc((1.0 / 4.0, 1.0 / 4.0)))


def reverb4_stereo(room_size, time):
    k = np.maximum(F(room_size), F(15.0)) / F(10.0)   # "the delays sound like garbage below 15 meters"
    return reverb4_stereo_delays([F(x) * k for x in REVERB4_DELAYS], time)


# ---- src/prelude.rs:2606 pulse(), src/wavetable.rs:361 PhaseSynth, src/prelude.rs:2876 rotate(), src/pan.rs:95 Mixer
def pulse():
    return An("pulse", (), (), 2, 1)


def phase_synth(kind):
    return An("phase_synth", (kind,), (), 1, 1)


def rotate(angle, gain):
    return An("rotate", (f32(angle), f32(gain)), (), 2, 2)


def mixer(matrix):
    """matrix[i] = the weights of output i over the inputs (a Frame of Frames in the reference)."""
    rows = [tuple(f32(x) for x in r) for r in matrix]
    _arity(len(rows) > 0 and all(len(r) == len(rows[0]) and len(r) > 0 for r in rows), "mixer: ragged matrix")
    return An("mixer", (len(rows[0]), len(rows), tuple(x for r in rows for x in r)), (), len(rows[0]), len(rows))


# ---- src/prelude.rs:580-612 envelope / lfo: control signals from a closure of time, sampled every ~2 ms and interpolated.
# `f(t)` returns a float or a tuple (one value per output); `outputs` defaults to what f(0.0) returns. The closure runs on the HOST when
# the graph is lowered, at the sample points the reference would use, up to `horizon` seconds (then the last value holds).
# time64=True is `F = f64` (prelude64 / hacker); the default is the f32 time of hacker32.
def envelope(f, outputs=None, horizon=10.0, time64=False, interval=0.002):
    if outputs is None:
        v = f(0.0)
        outputs = len(v) if isinstance(v, (tuple, list)) else 1
    return An("envelope", (float(interval) if time64 else f32(interval), int(outputs), 1 if time64 else 0, f, float(horizon)), (), 0, int(outputs))


def lfo(f, outputs=None, horizon=10.0, time64=False):
    return envelope(f, outputs, horizon, time64)


# ---- src/prelude.rs:2719-2753 flanger / phaser: the delay (phase) closure is a closure of time, so it lowers like `lfo`
def flanger(feedback_amount, minimum_delay, maximum_delay, delay_f, horizon=10.0):
    return pass_() & feedback2((pass_() | lfo(lambda t: f32(delay_f(t)), 1, horizon)) >> tap(minimum_delay, maximum_delay), shape(Tanh(feedback_amount)))


def phaser(feedback_amount, phase_f, horizon=10.0):
    c01 = lambda x: min(1.0, max(0.0, f32(x)))
    return pass_() & feedback((pass_() | lfo(lambda t: lerp(2.0, 20.0, c01(phase_f(t))), 1, horizon))
                              >> pipei(10, lambda i: add((0.0, 0.1)) >> ~allpole()) >> (mul(feedback_amount) | sink()))


def unit(x):   # src/audiounit.rs:430-484 Unit<I, O>: a boxed AudioUnit as a node; transparent to ping, settings and processing
    return x


def monitor(shared=None, meter=None):   # src/dynamics.rs:441-520: the audio passes through; the Shared is host-side (use `meter` to read a level)
    return An("monitor", (), (), 1, 1)


def oversample(node):   # src/prelude.rs:996-1005: run `node` at twice the sample rate between halfband filters
    return An("oversample", (), (node,), node.nin, node.nout)


def white():   # src/prelude.rs: white() is noise()
    return noise()


# ---- src/prelude.rs:1288-1301 look-ahead limiters
def limiter(attack_time, release_time):
    return An("limiter", (1, f32(attack_time), f32(release_time)), (), 1, 1)


def limiter_stereo(attack_time, release_time):
    return An("limiter", (2, f32(attack_time), f32(release_time)), (), 2, 2)


# ---- src/prelude.rs:299 meter(), src/dynamics.rs:316-326 Meter
class Meter:
    """Meter::Sample / Meter::Peak(timescale) / Meter::Rms(timescale)."""
    Sample = (0, 0.0)

    @staticmethod
    def Peak(timescale): return (1, float(timescale))

    @staticmethod
    def Rms(timescale): return (2, float(timescale))


def meter(m):
    return An("meter", (int(m[0]), float(m[1])), (), 1, 1)


# ---- src/prelude.rs:2631-2654 playwave / playwave_at: `wave` is a [channels, length] f32 array (Wave), src/prelude.rs:1034 resample
def playwave_at(wave, channel, start_point, end_point, loop_point=None):
    w = np.ascontiguousarray(np.atleast_2d(np.asarray(wave, np.float32))[channel])
    _arity(0 <= start_point and end_point <= len(w), "playwave: end_point <= wave.length()")
    return An("playwave", (_Samples(w), int(start_point), int(end_point), -1 if loop_point is None else int(loop_point)), (), 0, 1)


def playwave(wave, channel, loop_point=None):
    return playwave_at(wave, channel, 0, np.atleast_2d(np.asarray(wave)).shape[1], loop_point)


class _Samples:
    """A wave channel as an An argument (kept out of repr)."""
    def __init__(self, a): self.a = a
    def __len__(self): return len(self.a)
    def __iter__(self): return iter(self.a)
    def __array__(self, dtype=None, copy=None): return self.a if dtype is None else self.a.astype(dtype)
    def __repr__(self): return f"<wave {len(self.a)}>"


def resample(node):
    _arity(node.nin == 0, "resample: the inner node must be a generator")
    return An("resample", (), (node,), 1, node.nout)


# ---- src/prelude.rs:395-430
def add(x):
    v = _frame(x)
    return multipass(len(v)) + dc(v) if len(v) > 1 else An("multipass", (1,), (), 1, 1) + dc(v)


def sub(x):
    v = _frame(x)
    return An("multipass", (len(v),), (), len(v), len(v)) - dc(v)


def mul(x):
    v = _frame(x)
    return An("multipass", (len(v),), (), len(v), len(v)) * dc(v)


# ---- src/prelude.rs:356-366, 3112-3156 phase oscillators
def ramp():
    return An("phase_osc", (0,), (), 1, 1)


def ramp_hz(f):
    return dc(f) >> ramp()


def poly_saw():
    return An("phase_osc", (1,), (), 1, 1)


def poly_saw_hz(f):
    return dc(f) >> poly_saw()


def poly_square():
    return An("phase_osc", (2,), (), 1, 1)


def poly_square_hz(f):
    return dc(f) >> poly_square()


def poly_pulse():
    return An("phase_osc", (3,), (), 2, 1)


def poly_pulse_hz(f, width):
    return dc((f, width)) >> poly_pulse()


# ---- src/prelude.rs:783-797, 2860-2862
def mls_bits(n):
    return An("mls", (int(n),), (), 0, 1)


def mls():
    return mls_bits(29)


def impulse(n=1):
    return An("impulse", (n,), (), 0, n)


# ---- src/prelude.rs:923-990 interpolated delay taps (delay times in seconds are audio-rate inputs)
def tap(min_delay, max_delay):
    return An("tap", (1, 0, f32(min_delay), f32(max_delay)), (), 2, 1)


def multitap(n, min_delay, max_delay):
    return An("tap", (n, 0, f32(min_delay), f32(max_delay)), (), n + 1, 1)


def tap_linear(min_delay, max_delay):
    return An("tap", (1, 1, f32(min_delay), f32(max_delay)), (), 2, 1)


def multitap_linear(n, min_delay, max_delay):
    return An("tap", (n, 1, f32(min_delay), f32(max_delay)), (), n + 1, 1)


# ---- src/prelude.rs:1074-1085, 1353-1364
def feedback2(node, loopback):
    return An("feedback2", (0,), (node, loopback), node.nin, node.nout)


def fdn2(node, loopback):
    return An("feedback2", (1,), (node, loopback), node.nin, node.nout)


# ---- src/prelude.rs:1948-1978 discrete summation formula oscillators
def dsf_saw():
    return An("dsf", (2, 1.0, 0.5), (), 2, 1)


def dsf_saw_r(roughness):
    return An("dsf", (1, 1.0, f32(roughness)), (), 1, 1)


def dsf_square():
    return An("dsf", (2, 2.0, 0.5), (), 2, 1)


def dsf_square_r(roughness):
    return An("dsf", (1, 2.0, f32(roughness)), (), 1, 1)


# ---- src/prelude.rs:1858-1864 allpass-loop stereo reverb with a user loop filter; src/shared.rs:84 shared control value
def reverb3_stereo(time, diffusion, filt):
    if (filt.nin, filt.nout) != (1, 1):
        raise ArityError("reverb3_stereo: the loop filter must be 1 -> 1")
    return An("reverb3", (float(time), float(diffusion)), (filt,), 2, 2)


def var(value):
    """var(&shared): here the shared value is changed through Setting value (kind 4) / GpuBank.set."""
    return An("var", (f32(value),), (), 0, 1)


def feedback_unit(delay, node):
    """FeedbackUnit::new(delay, Box::new(node)) (src/feedback.rs:347): feedback loop with an integrated delay in seconds."""
    if node.nin != node.nout:
        raise ArityError("feedback_unit: the enclosed node must have as many outputs as inputs")
    return An("feedback_unit", (float(delay),), (node,), node.nin, node.nout)


def convolve(response):
    """convolve(&wave, channel) (src/prelude.rs:3158): `response` = the samples of that channel."""
    return An("convolve", (tuple(f32(x) for x in response),), (), 1, 1)


# ---- src/prelude.rs:462-507, 1160-1175, 1306-1321 (prelude32: F = f32) one-pole filters, pink and brown noise
def lowpole():
    return An("onepole", (0, 440.0, 2), (), 2, 1)


def lowpole_hz(cutoff):
    return An("onepole", (0, f32(cutoff), 1), (), 1, 1)


def highpole():
    return An("onepole", (1, 440.0, 2), (), 2, 1)


def highpole_hz(cutoff):
    return An("onepole", (1, f32(cutoff), 1), (), 1, 1)


def allpole():
    return An("onepole", (2, 1.0, 2), (), 2, 1)


def allpole_delay(delay_in_samples):
    return An("onepole", (2, f32(delay_in_samples), 1), (), 1, 1)


def dcblock_hz(cutoff):
    return An("onepole", (3, f32(cutoff), 1), (), 1, 1)


def dcblock():
    return dcblock_hz(10.0)


def pinkpass():
    return An("onepole", (4, 0.0, 1), (), 1, 1)


def pink():
    return white() >> pinkpass()


def brown():
    return white() >> lowpole_hz(10.0) * dc(13.7)


# ---- src/shape.rs + src/prelude.rs:1207-1223 waveshapers: shape(Tanh(1.5)), shape(Crush(16.0)), clip(), clip_to(lo, hi)
def Clip(hardness=1.0): return ("shape", 0, f32(hardness), 0.0)
def ClipTo(lo, hi): return ("shape", 1, f32(lo), f32(hi))
def Tanh(hardness): return ("shape", 2, f32(hardness), 0.0)
def Softsign(hardness): return ("shape", 3, f32(hardness), 0.0)
def Crush(levels): return ("shape", 4, f32(levels), 0.0)
def SoftCrush(levels): return ("shape", 5, f32(levels), 0.0)


def shape(mode):
    _, kind, p0, p1 = mode
    return An("shaper", (kind, p0, p1), (), 1, 1)


def clip():
    return shape(Clip(1.0))


def clip_to(lo, hi):
    return shape(ClipTo(lo, hi))


# ---- src/prelude.rs:1264-1281 parameter smoothing
def follow(response_time):
    return An("follow", (0, f32(response_time), f32(response_time)), (), 1, 1)


def afollow(attack_time, release_time):
    return An("follow", (1, f32(attack_time), f32(release_time)), (), 1, 1)


# ---- src/prelude.rs:2559-2627 resonant two-pole (Rez) and morphing SVF
def lowrez():
    return An("rez", (0.0, 440.0, 1.0, 3), (), 3, 1)


def lowrez_hz(cutoff, q):
    return An("rez", (0.0, f32(cutoff), f32(q), 1), (), 1, 1)


def lowrez_q(q):
    return (multipass(2) | dc(f32(q))) >> lowrez()


def bandrez():
    return An("rez", (1.0, 440.0, 1.0, 3), (), 3, 1)


def bandrez_hz(center, q):
    return An("rez", (1.0, f32(center), f32(q), 1), (), 1, 1)


def bandrez_q(q):
    return (multipass(2) | dc(f32(q))) >> bandrez()


def morph():
    return An("morph", (440.0, 1.0), (), 4, 1)


def morph_hz(f, q, m):
    return (pass_() | dc((f32(f), f32(q), f32(m)))) >> An("morph", (f32(f), f32(q)), (), 4, 1)


# ---- src/prelude.rs rossler() / lorenz(): chaotic oscillators, input = frequency
def rossler():
    return An("chaos", (0,), (), 1, 1)


def lorenz():
    return An("chaos", (1,), (), 1, 1)


# ---- src/prelude.rs:1180-1189
def declick():
    return An("declick", (f32(0.010),), (), 1, 1)


def declick_s(t):
    return An("declick", (f32(t),), (), 1, 1)


# ---- src/prelude.rs:2900-3110 nonlinear biquads: d* = DirtyBiquad (shaped state), f* = FbBiquad (shaped feedback)
def _nlb(fb, mode, shape_mode, nin, center=440.0, q=1.0, gain=1.0):
    _, kind, p0, p1 = shape_mode
    return An("nl_biquad", (fb, mode, kind, p0, p1, nin, f32(center), f32(q), f32(gain)), (), nin, 1)


def dbell(s): return _nlb(0, 3, s, 4)
def dbell_hz(s, center, q, gain): return _nlb(0, 3, s, 1, center, q, gain)
def fbell(s): return _nlb(1, 3, s, 4)
def fbell_hz(s, center, q, gain): return _nlb(1, 3, s, 1, center, q, gain)
def dhighpass(s): return _nlb(0, 2, s, 3)
def dhighpass_hz(s, cutoff, q): return _nlb(0, 2, s, 1, cutoff, q)
def fhighpass(s): return _nlb(1, 2, s, 3)
def fhighpass_hz(s, cutoff, q): return _nlb(1, 2, s, 1, cutoff, q)
def dlowpass(s): return _nlb(0, 1, s, 3)
def dlowpass_hz(s, cutoff, q): return _nlb(0, 1, s, 1, cutoff, q)
def flowpass(s): return _nlb(1, 1, s, 3)
def flowpass_hz(s, cutoff, q): return _nlb(1, 1, s, 1, cutoff, q)
def dresonator(s): return _nlb(0, 0, s, 3)
def dresonator_hz(s, center, q): return _nlb(0, 0, s, 1, center, q)
def fresonator(s): return _nlb(1, 0, s, 3)
def fresonator_hz(s, center, q): return _nlb(1, 0, s, 1, center, q)
