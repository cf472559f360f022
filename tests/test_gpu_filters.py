"""The f32 filter nodes on the device, bit for bit against the oracle (NaN canonicalized) and within the bounds of the f64 models of
tests/filter_model.py (written from the reference's source), where their state and launch structure can go wrong:
- voice counts on both sides of the stage-pipelined kernel's limit, every voice with parameters of its own;
- filters behind a Moog stage cut, in the plain kernel and the staged kernel at widths 32 and 128;
- ragged process() sizes, with and without the resident kernel, then clone and reset;
- Moog's steady 8-sample group path against its per-sample path;
- every audio-rate family at the edges of its control inputs (the f32 counterpart of tests/test_gpu_prelude64_edges.py);
- a rate change on a running bank with held controls, which must recompute the coefficients at the new rate as the reference's
  set_sample_rate does, then clone and reset.
Runs on the CPU mock device too (tests/test_filters_cpu.py)."""
import functools
import math
import os

import numpy as np
import pytest

import filter_model as M
from fundsp_b200.prelude import (Tanh, allpass, allpole, bandpass, bandrez, bell, butterpass, dc, dlowpass, fbell, highpass, highpole,
                                 highshelf, lowpass, lowpole, lowrez, lowshelf, moog, moog_hz, morph, multipass, noise, notch, pass_,
                                 peak, resonator)
from oracle import OracleUnit, lib as olib

pytestmark = pytest.mark.gpu
F32 = np.float32
SR = 48000.0
MOCK = "mock" in os.environ.get("FDSP_B200_LIB", "")
MODES = ("lowpass", "highpass", "bandpass", "notch", "peak", "allpass", "bell", "lowshelf", "highshelf")
# every audio-rate f32 family: name -> (constructor, number of control inputs)
FAM = {m: (globals()[m], 3 if i >= 6 else 2) for i, m in enumerate(MODES)}
FAM.update(morph=(morph, 3), butterpass=(butterpass, 1), resonator=(resonator, 2), lowpole=(lowpole, 1), highpole=(highpole, 1),
           allpole=(allpole, 1), moog=(moog, 2), lowrez=(lowrez, 2), bandrez=(bandrez, 2),
           dlowpass=(lambda: dlowpass(Tanh(0.5)), 2), fbell=(lambda: fbell(Tanh(0.5)), 3))
# the families whose coefficients live in state next to the last control value (all but moog and allpole, which recompute on every
# sample): the ones a rate change on a running bank reaches through their `ksr` word
KSR = tuple(f for f in FAM if f not in ("moog", "allpole"))
MODELLED = tuple(f for f in FAM if f not in ("dlowpass", "fbell"))


@functools.lru_cache(None)
def sms():
    from test_gpu_mix import sms as s
    return s()


def held(fam, i):
    """Voice i's control values: cutoff / center, then q (resonator: bandwidth in Hz; allpole: the delay in samples), then gain or morph."""
    g = (i * 0.6180339887498949) % 1.0
    if fam == "allpole":
        return (0.3 + 2.5 * g,)
    c = 300.0 + 2500.0 * g
    if fam == "butterpass" or fam in ("lowpole", "highpole"):
        return (c,)
    q = 60.0 + 40.0 * g if fam == "resonator" else (0.1 + 0.5 * g if fam == "moog" else 0.6 + 3.0 * g)
    if FAM[fam][1] == 2:
        return (c, q)
    return (c, q, (0.4 + 0.5 * g) if fam == "morph" else (0.3 + 2.5 * g))


def held_voice(fam, i):
    return (noise().seed(i) | dc(tuple(float(F32(v)) for v in held(fam, i)))) >> FAM[fam][0]()


def scales(fam, i):
    """Voice i's factors on the bank's shared control inputs (exact in f32 unless the product overflows)."""
    nc = FAM[fam][1]
    return (2.0 ** ((i % 5) - 2) * (1.0 + (i % 3) / 8.0),) + tuple(1.0 + (i % 4) / 4.0 for _ in range(nc - 1))


def ctl(fam, i):
    nc = FAM[fam][1]
    s = scales(fam, i)
    return (pass_() * dc(s[0])) if nc == 1 else multipass(nc) * dc(s)


def live_voice(fam, i):
    return (noise().seed(i) | ctl(fam, i)) >> FAM[fam][0]()


def cut_moog(i):
    return noise().seed(i) >> moog_hz(900.0 + 7.0 * i, 0.3)


def cut_voice(fam, i):
    """A Moog (the heavy leaf: the stage-pipelined kernel cuts the spine there, and the controls ride beside it as pass-through channels),
    then the family."""
    return (cut_moog(i) | ctl(fam, i)) >> FAM[fam][0]()


def voice_controls(fam, i, inp):
    """The control rows voice i's filter sees, in f32 as on the device."""
    with np.errstate(over="ignore", invalid="ignore"):
        return np.array([inp[k] * F32(s) for k, s in enumerate(scales(fam, i))], F32)


def inputs(fam, n, seed):
    """Shared control rows: a cutoff that moves every sample over a few hundred samples, then holds for whole blocks, then steps at the
    first and the last sample of 64-sample blocks; q and gain that change alone, while the cutoff holds."""
    rng = np.random.default_rng(seed)
    k = np.arange(n)
    c = (900.0 + 600.0 * np.sin(k * (2 * math.pi / 333.0))).astype(F32)
    c[(k // 128) % 3 == 1] = F32(1200.0)
    c[(k % 64 == 0) & ((k // 64) % 4 == 2)] = F32(1700.0)
    c[(k % 64 == 63) & ((k // 64) % 4 == 3)] = F32(400.0)
    if fam == "allpole":
        c = (c / F32(1000.0)).astype(F32)
    rows = [c]
    for j in range(1, FAM[fam][1]):
        v = np.full(n, F32(0.7 if j == 1 else 1.5))
        v[(k // 97) % 2 == 1] = F32(rng.uniform(0.5, 4.0))
        if fam == "resonator":
            v = (v * F32(50.0)).astype(F32)
        if fam == "moog":
            v = (v * F32(0.2)).astype(F32)
        rows.append(v)
    return np.array(rows, F32)


def bank(voices, sr=SR, **kw):
    from fundsp_b200.bank import GpuBank
    olib().fo_set_denormal_emulation(0)
    return GpuBank(voices, sample_rate=sr, per_voice=True, **kw)


def units(voices, sr=SR):
    us = [OracleUnit(v) for v in voices]
    for u in us:
        u.set_sample_rate(sr)
    return us


def canon(a):   # bit patterns, every NaN as 0x7fc00000
    a = np.asarray(a, np.float32)
    b = a.view(np.uint32).copy()
    b[np.isnan(a)] = 0x7FC00000
    return b


def same(g, o):
    return np.array_equal(canon(g), canon(o))


def sampled(V):
    return sorted(set([0, 1, V // 2, V - 2, V - 1] + list(range(3, V, max(1, V // 24))))) if V > 1 else [0]


def noise_of(i, n):
    """Voice i's noise input: the oracle's noise().seed(i) alone."""
    return OracleUnit(noise().seed(i)).process_many(n)[0]


def model_ratio(fam, i, got, x, c, sr, what):
    want, bound = M.run(fam, x, c, sr)
    err = np.abs(np.asarray(got, np.float64) - want)
    assert np.isfinite(got).all(), what
    r = float(np.max(err / np.maximum(bound, 1e-300)))
    assert r <= 1.0, (what, r, int(np.argmax(err / np.maximum(bound, 1e-300))))
    return r


def render_both(b, us, sizes, inp, p0=0):
    """process() in `sizes` on the bank and on the oracle units; returns ([V][1][n] device, oracle)."""
    V = len(us)
    nout = b.outputs() // V
    g, o, p = [], [], p0
    for m in sizes:
        x = inp[:, p:p + m] if inp is not None else None
        g.append(b.process(m, x).reshape(V, nout, m))
        o.append(np.stack([u.process(m, x) for u in us]) if m else np.zeros((V, nout, 0), F32))
        p += m
    return np.concatenate(g, axis=2), np.concatenate(o, axis=2)


# ---------------------------------------------------------------- voice counts
@pytest.mark.parametrize("V", ["1", "33", "sms*32", "sms*32+1"])
@pytest.mark.parametrize("fam", ["lowpass", "bell", "resonator", "highpole", "moog", "lowrez"])
def test_voice_counts(fam, V):
    V = {"sms*32": sms() * 32, "sms*32+1": sms() * 32 + 1}.get(V) or int(V)
    n = 64 * 12 + 37
    inp = inputs(fam, n, V)
    voices = [live_voice(fam, i) for i in range(V)]
    b = bank(voices)
    g, _ = b.render_samples(n, inp)
    vs = sampled(V) if V > 200 else list(range(V))
    o = np.stack([u.process_many(n, inp) for u in units([voices[v] for v in vs])])
    assert same(g[vs], o), (fam, V, int((canon(g[vs]) != canon(o)).sum()))
    worst = max(model_ratio(fam, v, g[v, 0], noise_of(v, n), voice_controls(fam, v, inp), SR, (fam, V, v)) for v in vs[:: max(1, len(vs) // 6)] + [V - 1])
    print(f"{fam} V={V}: worst {worst:.3g} of the bound")


# ---------------------------------------------------------------- stage cuts in every kernel form
@pytest.mark.parametrize("form", ["plain", "staged32", "staged128"])
@pytest.mark.parametrize("fam", ["lowpass", "highshelf", "morph", "butterpass", "resonator", "lowpole", "allpole", "moog", "bandrez", "dlowpass", "fbell"])
def test_filters_behind_a_stage_cut(fam, form, monkeypatch):
    monkeypatch.setenv("FDSP_STAGED", "0" if form == "plain" else "1")
    if form != "plain":
        monkeypatch.setenv("FDSP_STAGED_W", form[len("staged"):])
    V, n = 300, 64 * 9 + 61
    inp = inputs(fam, n, 7)
    voices = [cut_voice(fam, i) for i in range(V)]
    b = bank(voices)
    if not MOCK:
        assert b.classes()[0]["stages"] >= 2, b.classes()
    g, _ = b.render_samples(n, inp)
    vs = sampled(V)
    o = np.stack([u.process_many(n, inp) for u in units([voices[v] for v in vs])])
    assert same(g[vs], o), (fam, form, int((canon(g[vs]) != canon(o)).sum()))
    if fam in MODELLED:
        for v in vs[::6]:
            u = OracleUnit(cut_moog(v)); u.set_sample_rate(SR)
            x = u.process_many(n)[0]
            model_ratio(fam, v, g[v, 0], x, voice_controls(fam, v, inp), SR, (fam, form, v))


# ---------------------------------------------------------------- process() sizes, clone, reset
SIZES = [64, 61, 8, 7, 1, 0, 64, 33, 17, 64, 2, 63, 40, 64, 64, 13, 52, 53, 54, 24, 25, 23, 64, 64]


@pytest.mark.parametrize("rt", ["1", "0"])
@pytest.mark.parametrize("fam", ["notch", "morph", "resonator", "lowpole", "moog", "lowrez", "fbell"])
def test_ragged_process_clone_and_reset(fam, rt, monkeypatch):
    monkeypatch.setenv("FDSP_RT", rt)
    V = 40
    n = sum(SIZES)
    inp = inputs(fam, 3 * n, 11)
    voices = [live_voice(fam, i) for i in range(V)]
    b = bank(voices)
    us = units(voices)
    g1, o1 = render_both(b, us, SIZES, inp)
    assert same(g1, o1), (fam, int((canon(g1) != canon(o1)).sum()))
    c = b.clone()
    a_out, c_out, p = [], [], n
    for m in SIZES:
        a_out.append(b.process(m, inp[:, p:p + m])); c_out.append(c.process(m, inp[:, p:p + m])); p += m
    assert all(same(x, y) for x, y in zip(a_out, c_out))
    if fam in MODELLED:
        full = np.concatenate([g1.reshape(V, -1), np.concatenate(a_out, axis=1)], axis=1)
        for v in (0, 17, V - 1):
            model_ratio(fam, v, full[v], noise_of(v, 2 * n), voice_controls(fam, v, inp[:, :2 * n]), SR, (fam, v))
    b.reset()
    g3, _ = render_both(b, units(voices), SIZES, inp)
    assert same(g3, g1)


# ---------------------------------------------------------------- Moog's steady 8-sample groups
@pytest.mark.parametrize("form", ["plain", "staged32"])
def test_moog_steady_groups_against_the_per_sample_path(form, monkeypatch):
    """Controls that hold for whole 8-sample groups, change at lane 0 or lane 7 of a group, or are NaN (then no group is steady, since
    NaN != NaN): the steady group path and the per-sample path must give the oracle's samples."""
    monkeypatch.setenv("FDSP_STAGED", "0" if form == "plain" else "1")
    V, n = 300, 64 * 8
    k = np.arange(n)
    c = np.full(n, F32(800.0))
    c[(k // 8) % 5 == 1] = F32(1500.0)                       # whole groups
    c[(k % 8 == 0) & ((k // 8) % 7 == 3)] = F32(2100.0)      # lane 0
    c[(k % 8 == 7) & ((k // 8) % 7 == 5)] = F32(300.0)       # lane 7
    c[(k >= 320) & (k < 352)] = F32(np.nan)                  # four groups of NaN
    q = np.full(n, F32(0.2))
    q[(k % 8 == 7) & ((k // 8) % 11 == 4)] = F32(0.45)       # q alone, at lane 7
    inp = np.array([c, q], F32)
    voices = [cut_voice("moog", i) for i in range(V)]
    b = bank(voices)
    g, _ = b.render_samples(n, inp)
    vs = sampled(V)
    o = np.stack([u.process_many(n, inp) for u in units([voices[v] for v in vs])])
    assert same(g[vs], o), (form, int((canon(g[vs]) != canon(o)).sum()))


# ---------------------------------------------------------------- control edges
def _f32_neighbours(x, k=2):
    v = np.array([x], F32)
    out = [v[0]]
    lo = hi = v
    for _ in range(k):
        lo, hi = np.nextafter(lo, F32(-np.inf)), np.nextafter(hi, F32(np.inf))
        out += [lo[0], hi[0]]
    return out


# sinf / cosf / tanf branch words of rem_pio2f (csrc/dsp/libm.cuh), and the large-reduction threshold 2^28 pi/2 (DESIGN §2)
TRIG_WORDS = (0x39800000, 0x3f490fda, 0x4016cbe3, 0x407b53d1, 0x40afeddf, 0x40e231d5, 0x4dc90fdb)
EXPF_LIMITS = (88.72283935546875, -103.97207641601562, -87.33654022216797)   # expf overflow, underflow to 0, the last normal result


def edge_values(fam, sr):
    """Cutoff control values, in f32, one segment each."""
    rng = np.random.default_rng(int(sr))
    v = [0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, -1.1754942e-38, 1e-3, 1.0, 300.0, -300.0, -1e4, 0.49 * sr]
    v += _f32_neighbours(sr / 2)
    for w in TRIG_WORDS:
        a = float(np.array([w], np.uint32).view(F32)[0])
        for mult in (math.pi, 2 * math.pi, math.pi / 2):   # SVF / Rez / butterpass: pi f / sr; resonator: tau f / sr; Moog: pi/2 * 2f/sr
            v += _f32_neighbours(a * sr / mult, 1)
    for arg in EXPF_LIMITS:   # one-poles: expf(-tau p / sr)
        v += _f32_neighbours(-arg * sr / (2 * math.pi), 1)
    v += [2.52e10, 6.0e13, 1e20, 3.4028235e38, -3.4028235e38]
    v += list(np.exp(rng.uniform(0.0, 88.7, 12)).astype(F32) * rng.choice([-1.0, 1.0], 12))
    v += [np.inf, -np.inf, np.nan]
    if fam == "allpole":   # the delay in samples: around the pole at -1 as well
        v += _f32_neighbours(-1.0) + [2.0, 1e-7]
    return np.array(v, F32)


EV = 4   # voices in the edge tests
WARM, HOLD = 8, 16
SEG = WARM + HOLD


def edge_voice(fam, i):
    """Voice i scales the shared cutoff by a power of two (i = 1: -1) and holds its other controls at values of its own."""
    nc = FAM[fam][1]
    s = (1.0, -1.0, 0.5, 2.0 ** 40)[i]
    rest = [(0.7, 5.0, 1e-3, 100.0)[i], (2.0, 0.5, 1e-30, 1e30)[i]]
    if fam == "resonator":
        rest[0] = (50.0, 5.0, 0.0, -30.0)[i]
    if fam == "moog":
        rest[0] = (0.2, 0.9, 0.0, 1.0)[i]
    if fam == "morph":
        rest[1] = (0.5, -1.0, 1.0, 0.0)[i]
    c = pass_() * dc(s)
    if nc > 1:
        c = c | dc(tuple(rest[:nc - 1]))
    return (noise().seed(i) | c) >> FAM[fam][0]()


@pytest.mark.parametrize("sr", [48000.0, 44100.0])
@pytest.mark.parametrize("fam", list(FAM))
def test_audio_rate_edges_match_oracle(fam, sr):
    """After a reset of every voice, WARM samples of an ordinary cutoff, then HOLD of one edge value: every edge value meets a live
    state, and a value that spoils a voice's state spoils only its own segment."""
    ev = edge_values(fam, sr)
    s = np.empty((ev.size, SEG), F32)
    s[:, :WARM] = F32(0.5 if fam == "allpole" else 1000.0)
    s[:, WARM:] = ev[:, None]
    voices = [edge_voice(fam, i) for i in range(EV)]
    b = bank(voices, sr)
    assert len(b.classes()) == 1, [c["signature"] for c in b.classes()]
    us = units(voices, sr)
    for k, seg in enumerate(s):
        b.reset()
        g, _ = b.render_samples(SEG, seg.reshape(1, -1))
        for i, u in enumerate(us):
            u.reset()
            o = u.process_many(SEG, seg.reshape(1, -1))[0]
            assert same(g[i, 0], o), (fam, sr, i, f"edge value {ev[k]!r}", g[i, 0], o)


# ---------------------------------------------------------------- the running rate change
RATES = (48000.0, 8000.0, 96000.0)


@pytest.mark.parametrize("rt", ["1", "0"])
@pytest.mark.parametrize("fam", list(FAM))
def test_rate_change_of_a_running_bank_with_held_controls(fam, rt, monkeypatch):
    """48 kHz, then 8 kHz, then 96 kHz on a running bank whose controls hold (a dc per voice): the reference's set_sample_rate recomputes
    the coefficients from the stored cutoff, q and gain, so the next sample runs at the new rate's coefficients. Then a clone, which must
    follow its source, then a reset."""
    monkeypatch.setenv("FDSP_RT", rt)
    V = 33
    voices = [held_voice(fam, i) for i in range(V)]
    b = bank(voices, RATES[0])
    us = units(voices, RATES[0])
    sizes = [64, 61, 3, 64, 64, 128 - 67]
    for k, sr in enumerate(RATES):
        if k:
            b.set_sample_rate(sr)
            for u in us:
                u.set_sample_rate(sr)
        g, o = render_both(b, us, sizes, None)
        assert same(g, o), (fam, sr, "after the rate change", int((canon(g) != canon(o)).sum()))
    c = b.clone()
    a1, _ = b.render_samples(200)
    c1, _ = c.render_samples(200)
    o1 = np.stack([u.process_many(200) for u in us])
    assert same(a1, o1) and same(c1, o1), (fam, "clone")
    b.reset()
    for u in us:
        u.reset()
    g, o = render_both(b, us, sizes, None)
    assert same(g, o), (fam, "after reset", int((canon(g) != canon(o)).sum()))
    if fam in MODELLED:
        n = sum(sizes)
        for v in (0, V - 1):
            c = np.repeat(np.array(held(fam, v), F32)[:, None], n, axis=1)
            model_ratio(fam, v, g[v, 0], noise_of(v, n), c, RATES[-1], (fam, v, "after reset"))
