"""prelude64 filters on the GPU at the edges of their control inputs, bit for bit against the oracle (oracle/fo_prelude64.h), NaN
canonicalized. The audio-rate nodes (Svf<f64, M> in all nine modes, butterpass(), resonator(), lowpole(), highpole(), allpole()) recompute
their coefficients on the device from whatever f32 arrives: zeros of both signs, subnormals, negative values, sr/2 and its neighbours,
cutoffs that land on rem_pio2's branch words, the 2^20 pi/2 threshold of the large trig reduction, values up to 3.4e38, infinities and
NaN. Every voice of a class reads the bank's one input, scaled by its own power of two (exact in f32 unless it overflows), with its own q
and gain (q = 0, q < 0 and gain <= 0 included). The input is a list of segments: after a reset of every voice, 8 samples of an ordinary
value, then 16 of one edge value. A value that makes a voice's state NaN or infinite so spoils only its own segment, and every edge value
meets a live state. The resonator's q follows its center (q = center * k, k = 0 and k < 0 included), so that r = exp(-pi center / (q sr)) stays
inside (0, 1) at any center and its cos(tau center / sr) reaches the output. Each test checks on the oracle's output that the values that
take the large reduction (or exp's overflow and underflow, for the one-poles) were met with a live state: a stated number of finite
output samples at those steps. The host path: fixed *_hz nodes built at huge cutoffs, Setting::center_q_gain on a running bank, and a
rate change to a low rate."""
import ctypes as C
import math

import numpy as np
import pytest

from fundsp_b200.prelude import pass_
from fundsp_b200.prelude64 import *  # noqa: F401,F403
from oracle import OracleUnit, lib as olib

pytestmark = pytest.mark.gpu
F32 = np.float32
LARGE = 2.0 ** 20 * math.pi / 2   # about 1647099.33: from here on the trig functions reduce with the large reduction
EXP_MAX, EXP_MIN = 709.782712893383973096, -745.13321910194110842
P_CENTER_Q_GAIN = 3
MODES = ("lowpass", "highpass", "bandpass", "notch", "peak", "allpass", "bell", "lowshelf", "highshelf")
KINDS = MODES + ("butterpass", "resonator", "lowpole", "highpole", "allpole")
SCALES = (1.0, -1.0, 0.5, 2.0 ** -20, 2.0 ** 40, 1.0, 2.0, 2.0 ** 100)   # one per voice
QS = (0.7, 5.0, 0.0, -0.5, 1e-30, 1e30, 2.0, 0.9)
GAINS = (2.0, 0.5, 0.0, -1.0, 1e-30, 8.0, 1.5, 3.0)
RES_K = (1.3e-3, 2.6e-4, 1.3e-2, 0.0, -1.3e-3, 6.5e-4, 1.3e-3, 1e-30)   # resonator: q = center * k (k = 0: q = 0; k < 0: q < 0)
V = len(SCALES)
WARM, HOLD = 8, 16
SEG = WARM + HOLD


def _f32_neighbours(x, k=3):
    v = np.array([x], F32)
    out = [v[0]]
    lo = hi = v
    for _ in range(k):
        lo, hi = np.nextafter(lo, F32(-np.inf)), np.nextafter(hi, F32(np.inf))
        out += [lo[0], hi[0]]
    return out


def edge_values(sr):
    """The control values, in f32, one segment each."""
    rng = np.random.default_rng(int(sr))
    v = [0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, 300.0, -300.0, -1e4]
    v += _f32_neighbours(sr / 2)
    # cutoffs whose pi f / sr (tan) and tau f / sr (cos) land on rem_pio2's branch words and on the large-reduction threshold
    for w in (0x400f6a7a, 0x4002d97c, 0x4015fdbc, 0x4012d97c, 0x401c463b, 0x401921fb, 0x3ff921fb, 0x400921fb, 0x413921fb):
        arg = np.array([w << 32], np.uint64).view(np.float64)[0]
        v += _f32_neighbours(arg * sr / math.pi, 2) + _f32_neighbours(arg * sr / (2 * math.pi), 2)
    # one-poles: exp(-tau p / sr) past overflow (p < -5.4e6 at 48 kHz) and underflow (p > 5.7e6), and where the careful tests begin
    for arg in (EXP_MAX, EXP_MIN, -708.39641853226410622):
        v += _f32_neighbours(-arg * sr / (2 * math.pi), 2)
    v += [2.52e10, 1.26e10, 6.0e13, 1e20, 3.4028235e38, -3.4028235e38]
    v += list(np.exp(rng.uniform(0.0, 88.7, 24)).astype(F32) * rng.choice([-1.0, 1.0], 24))   # up to 3.4e38, both signs
    v += list(np.exp(rng.uniform(16.0, 60.0, 40)).astype(F32) * rng.choice([-1.0, 1.0], 40))  # mostly past 2^20 pi/2
    v += [np.inf, -np.inf, np.nan]
    return np.array(v, F32)


def schedule(sr):
    ev = edge_values(sr)
    s = np.empty((ev.size, SEG), F32)
    s[:, :WARM] = F32(1000.0)
    s[:, WARM:] = ev[:, None]
    return s


def _node(kind, i):
    ctl = pass_() * dc(SCALES[i])
    x = noise().seed(i)
    if kind in MODES:
        head = x | ctl | dc(QS[i])
        if MODES.index(kind) >= 6:
            head = head | dc(GAINS[i])
        return head >> globals()[kind]()
    if kind == "butterpass":
        return (x | ctl) >> butterpass()
    if kind == "resonator":
        return (x | (ctl >> (pass_() ^ (pass_() * dc(RES_K[i]))))) >> resonator()
    return (x | ctl) >> globals()[kind]()


def _canon(a):   # bit patterns, every NaN as 0x7fc00000
    a = np.asarray(a, np.float32)
    b = a.view(np.uint32).copy()
    b[np.isnan(a)] = 0x7FC00000
    return b


def _same(g, o):
    return np.array_equal(_canon(g), _canon(o))


def _bank(voices, sr):
    from fundsp_b200.bank import GpuBank
    return GpuBank(voices, sample_rate=sr, per_voice=True)


def _controls(s, i):
    """The control value voice i's node sees at every sample, in f32 as on the device and in the oracle."""
    with np.errstate(over="ignore", invalid="ignore"):
        return s * F32(SCALES[i])


def _large_steps(kind, c, sr):
    """Where the node's coefficient function takes the path the test is after: the large trig reduction, or exp past its limits."""
    c = c.astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        if kind in ("lowpole", "highpole"):
            e = -2 * math.pi * c / sr
            return (e > EXP_MAX) | (e < EXP_MIN)
        if kind == "allpole":
            return np.zeros(c.shape, bool)
        a = np.abs((2 * math.pi if kind == "resonator" else math.pi) * c / sr)
        return np.isfinite(a) & (a >= LARGE)


# least number of finite oracle output samples, summed over the voices, at steps that take the large reduction (one-poles: exp's limits);
# the schedule gives 9 000-13 000 in every class at both rates. allpole() computes no trig and no exp.
MIN_LIVE = {"allpole": 0}


@pytest.mark.parametrize("sr", [48000.0, 44100.0])
@pytest.mark.parametrize("kind", KINDS)
def test_audio_rate_edges_match_oracle(kind, sr):
    olib().fo_set_denormal_emulation(0)
    s = schedule(sr)
    b = _bank([_node(kind, i) for i in range(V)], sr)
    assert len(b.classes()) == 1, [c["signature"] for c in b.classes()]
    us = [OracleUnit(_node(kind, i)) for i in range(V)]
    for u in us:
        u.set_sample_rate(sr)
    got = np.zeros((V, s.shape[0], SEG), F32)
    want = np.zeros_like(got)
    for k, seg in enumerate(s):
        b.reset()
        g, _ = b.render_samples(SEG, seg.reshape(1, -1))
        got[:, k] = g[:, 0]
        for i, u in enumerate(us):
            u.reset()
            want[i, k] = u.process_many(SEG, seg.reshape(1, -1))[0]
    live = 0
    for i in range(V):
        bad = np.nonzero((_canon(got[i]) != _canon(want[i])).any(axis=1))[0]
        assert bad.size == 0, (kind, sr, i, f"{bad.size} segments differ, first at edge value {edge_values(sr)[bad[0]]!r}")
        live += int((_large_steps(kind, _controls(s, i), sr) & np.isfinite(want[i])).sum())
    print(f"{kind} at {sr:.0f} Hz: {live} finite samples at large-reduction steps")
    assert live >= MIN_LIVE.get(kind, 5000), (kind, sr, live)


def test_schedule_reaches_the_large_reduction_and_exp_limits():
    for sr in (48000.0, 44100.0):
        s = schedule(sr)
        tan_steps = np.sum([int(_large_steps("lowpass", _controls(s, i), sr).sum()) for i in range(V)])
        cos_steps = np.sum([int(_large_steps("resonator", _controls(s, i), sr).sum()) for i in range(V)])
        assert tan_steps > 2000 and cos_steps > 2000, (tan_steps, cos_steps)
        e = np.concatenate([-2 * math.pi * _controls(s, i).astype(np.float64) / sr for i in range(V)])
        assert (e > EXP_MAX).any() and (e < EXP_MIN).any()
        assert ((e > 708.0) & (e < EXP_MAX)).any() and ((e < -708.4) & (e > EXP_MIN)).any()


NF = 48


def _huge(i):   # cutoffs from 2.52e10 Hz (tan past 2^20 pi/2 at 48 kHz) to 3.4e38, log-spaced with a hashed jitter
    return float(F32(math.exp(math.log(2.52e10) + (math.log(3.4e38) - math.log(2.52e10)) * ((i * 0.618034) % 1.0))))


def _fixed(kind, i):
    f = _huge(i)
    x = noise().seed(i)
    if kind in MODES:
        hz = globals()[f"{kind}_hz"]
        return x >> (hz(f, 0.5 + 0.1 * (i % 7), 2.0) if MODES.index(kind) >= 6 else hz(f, 0.5 + 0.1 * (i % 7)))
    if kind == "butterpass":
        return x >> butterpass_hz(f)
    return x >> resonator_hz(f, f * 1.3e-3)   # q with the center, so that r stays inside (0, 1)


@pytest.mark.parametrize("kind", MODES + ("butterpass", "resonator"))
def test_fixed_nodes_at_huge_cutoffs_and_a_low_rate(kind):
    """Coefficients lowered on the host at cutoffs past the large-reduction threshold, then recomputed after a change to a low rate."""
    olib().fo_set_denormal_emulation(0)
    n = 64
    b = _bank([_fixed(kind, i) for i in range(NF)], 48000.0)
    g1, _ = b.render_samples(n)
    b.set_sample_rate(1000.0)
    b.reset()
    g2, _ = b.render_samples(n)
    live = 0
    for i in range(NF):
        u = OracleUnit(_fixed(kind, i)); u.set_sample_rate(48000.0)
        o1 = u.process_many(n)[0]
        assert _same(g1[i, 0], o1), (kind, i, _huge(i))
        u.set_sample_rate(1000.0)
        u.reset()
        o2 = u.process_many(n)[0]
        assert _same(g2[i, 0], o2), (kind, i, _huge(i), "after the rate change")
        live += int(np.isfinite(o1).sum() + np.isfinite(o2).sum())
    assert live >= NF * n / 2, (kind, live)   # most of the outputs come from live state


def test_center_q_gain_setting_at_edges_on_a_running_bank():
    olib().fo_set_denormal_emulation(0)
    mk = lambda i: noise().seed(i) >> bell_hz(1000.0 + 10.0 * i, 1.0, 2.0)   # noqa: E731
    edges = [(2.52e10, 1.0, 2.0), (3.4e38, 0.7, 0.5), (-5e12, 1.0, 1.0), (0.0, 0.0, 0.0), (24000.0, -1.0, -2.0),
             (float("inf"), 1.0, 1.0), (float("nan"), 1.0, 1.0), (1e-45, 1e30, 1e-30), (7.3e17, 0.7, 1.5), (-9.1e25, 2.0, 0.25)]
    nv = len(edges)
    b = _bank([mk(i) for i in range(nv)], 48000.0)
    us = [OracleUnit(mk(i)) for i in range(nv)]
    for u in us:
        u.set_sample_rate(48000.0)
    g1, _ = b.render_samples(300)
    assert _same(g1[:, 0], np.stack([u.process_many(300)[0] for u in us]))
    for v, vals in enumerate(edges):
        b.set(v, P_CENTER_Q_GAIN, vals)
        us[v].L.fo_set(us[v].h, P_CENTER_Q_GAIN, (C.c_float * 3)(*vals), 3, 0, None, 0)
    g2, _ = b.render_samples(300)
    for v in range(nv):
        assert _same(g2[v, 0], us[v].process_many(300)[0]), (v, edges[v])
