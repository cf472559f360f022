"""The oracle's f32 filters against the f64 models of tests/filter_model.py, written from the reference's source, at 48 kHz, 44.1 kHz and
8 kHz (where ordinary cutoffs pass Nyquist): cutoffs from 1e-3 Hz to past sr/2 (tan's negative branch), 0 and negative; q from 0.01 to
100, with runs of 8192 samples at q = 100 and a low cutoff, long enough to ring down into subnormals; bell and shelf gains tiny, 1 and
large; controls that change every sample, q or gain alone, at the first and the last sample of a 64-sample block, a first input equal
to the constructor's value; infinite and NaN controls (there only where the output is not finite); a rate change on a running unit
with held controls, then a reset. The fixed forms too, with biquad() standing for a BiquadBank lane. Negative controls: every mutation of a model misses its
bound by at least 10^3 on some case, and by at least 10x in every family it applies to. tests/test_gpu_filters.py holds the device to the same models and to the oracle, and runs here on
the CPU mock device."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import filter_model as M
from fundsp_b200.prelude import (biquad, butterpass_hz, dc, dcblock_hz, highpole_hz, lowpole_hz, lowrez_hz, moog_hz,
                                 noise, resonator_hz)
from oracle import OracleUnit, lib as olib
from test_gpu_filters import FAM
from test_mock_bank_cpu import ROOT, mock_env  # noqa: F401  (the mock device build, shared with that file)
import fundsp_b200.prelude as P

F32 = np.float32
RATES = (48000.0, 44100.0, 8000.0)
AUDIO = tuple(f for f in FAM if f in M.FAMILIES)   # every audio-rate family the models cover


def noise_of(seed, n):
    return OracleUnit(noise().seed(seed)).process_many(n)[0]


def oracle(graph, sr, n, inp=None):
    olib().fo_set_denormal_emulation(0)
    u = OracleUnit(graph)
    u.set_sample_rate(sr)
    return u.process_many(n, inp)[0]


def comparable(want, bound):
    """The samples where a first-order bound means something: before the bound first exceeds 1e-3 of the signal's scale (a resonant
    Rez near Nyquist amplifies its rounding to the size of the signal, and its linearisation no longer holds), and before an unstable
    filter's output first reaches 1e15 (its f32 state overflows a few samples later, before its output does)."""
    with np.errstate(invalid="ignore", over="ignore"):
        a = np.where(np.isfinite(want), np.abs(want), np.inf)
        rel = np.where(np.isfinite(bound), bound / np.maximum(1.0, a), np.inf)
        return (np.maximum.accumulate(a) < 1e15) & (np.maximum.accumulate(rel) < 1e-3)


def within(fam, got, want, bound, what):
    """max |got - want| / bound over the comparable samples; asserts <= 1."""
    got = np.asarray(got, np.float64)
    ok = comparable(want, bound)
    assert np.isfinite(got[ok]).all(), (what, "not finite where the model is")
    r = np.abs(got[ok] - want[ok]) / bound[ok]
    worst = float(r.max()) if r.size else 0.0
    assert worst <= 1.0, (what, worst, int(np.flatnonzero(ok)[np.argmax(r)]))
    return worst


def miss(got, want, bound):
    ok = comparable(want, bound) & np.isfinite(got)
    return float((np.abs(np.asarray(got, np.float64)[ok] - want[ok]) / bound[ok]).max()) if ok.any() else 0.0


# ---------------------------------------------------------------- held controls over the parameter grid
def cutoffs(sr):
    h = F32(sr / 2)
    return [1e-3, 1.0, 440.0, 1000.0, 3000.0, 0.49 * sr, float(np.nextafter(h, F32(0))), float(h), float(np.nextafter(h, F32(np.inf))),
            0.6 * sr, 0.0, -0.0, -500.0]


QS = (0.01, 0.5, 0.707, 10.0, 100.0)
GAINS = (1e-6, 1.0, 40.0)


def held_cases(fam, sr):
    """(controls, n) for every held case of the family at rate sr."""
    out = []
    for c in cutoffs(sr):
        if fam == "allpole":
            out += [((d,), 256) for d in (0.01, 0.5, 1.0, 3.0, 100.0, 0.0, -0.5)]
            break
        if FAM[fam][1] == 1:
            out.append(((c,), 512))
            continue
        for q in (QS if fam != "moog" else (0.0, 0.1, 0.5, 0.9, 1.0)):
            if fam == "resonator":
                q = q * 100.0   # the bandwidth in Hz
            if FAM[fam][1] == 2:
                out.append(((c, q), 512))
            else:
                for g in (GAINS if fam != "morph" else (-1.0, 0.0, 0.5, 1.0)):
                    out.append(((c, q, g), 256))
    if fam in ("lowpass", "bandpass", "peak", "bell", "notch", "lowrez", "bandrez", "moog"):
        out.append(((100.0, 100.0, 2.0)[:FAM[fam][1]] if fam != "moog" else (100.0, 0.99), 8192))   # ringing into subnormals
    return out


@pytest.mark.parametrize("sr", RATES)
@pytest.mark.parametrize("fam", AUDIO)
def test_held_controls_within_the_model(fam, sr):
    worst, n_cases = 0.0, 0
    for k, (ctl, n) in enumerate(held_cases(fam, sr)):
        ctl = tuple(float(F32(v)) for v in ctl)
        o = oracle((noise().seed(k) | dc(ctl)) >> FAM[fam][0](), sr, n)
        c = np.repeat(np.array(ctl, F32)[:, None], n, axis=1)
        want, bound = M.run(fam, noise_of(k, n), c, sr)
        worst = max(worst, within(fam, o, want, bound, (fam, sr, ctl)))
        n_cases += 1
    print(f"{fam} at {sr:.0f} Hz: {n_cases} cases, worst {worst:.3g} of the bound")


def test_q100_rings_into_subnormals():
    """At q = 100 an impulse into a 1 kHz lowpass at 8 kHz rings for thousands of samples and decays through the subnormal range."""
    n = 8192 * 4
    x = np.zeros(n, F32)
    x[0] = 1.0
    c = np.array([[1000.0] * n, [100.0] * n], F32)
    o = oracle(P.multipass(3) >> P.lowpass(), 8000.0, n, np.vstack([x, c]))
    want, bound = M.run("lowpass", x, c, 8000.0)
    within("lowpass", o, want, bound, "impulse")
    assert (np.abs(o[:8192]) > 1e-3).sum() > 100    # it rings
    sub = (o != 0) & (np.abs(o) < 2.0 ** -126)
    assert sub.sum() > 1000, int(sub.sum())          # and decays through the subnormals, held to the bound there too


# ---------------------------------------------------------------- moving controls
def moving(fam, n, seed):
    """Control rows that change every sample, hold, step at the first and last sample of 64-sample blocks, and change q or gain
    alone; the first sample equals the constructor's value, so the first recompute is skipped."""
    from test_gpu_filters import inputs
    rows = inputs(fam, n, seed)
    first = {"allpole": (1.0,), "moog": (1000.0, 0.1)}.get(fam, (440.0, 1.0, 1.0))
    rows[:, 0] = np.array(first[:rows.shape[0]], F32) if fam != "morph" else np.array([440.0, 1.0, rows[2, 0]], F32)
    return rows


@pytest.mark.parametrize("sr", RATES)
@pytest.mark.parametrize("fam", AUDIO)
def test_moving_controls_within_the_model(fam, sr):
    n = 64 * 24
    c = moving(fam, n, 5)
    if sr == 8000.0 and fam not in ("allpole",):
        c[0] = (c[0] * F32(0.2)).astype(F32)   # below 4 kHz
        c[0, 0] = F32({"moog": 1000.0}.get(fam, 440.0))
    o = oracle((noise().seed(3) | P.multipass(c.shape[0])) >> FAM[fam][0](), sr, n, c)
    want, bound = M.run(fam, noise_of(3, n), c, sr)
    print(f"{fam} at {sr:.0f} Hz, moving controls: worst {within(fam, o, want, bound, (fam, sr)):.3g} of the bound")


@pytest.mark.parametrize("fam", AUDIO)
def test_non_finite_controls(fam):
    """inf, -inf and NaN cutoffs (and q) for 64 samples each after a live stretch: the output is not finite exactly where the model's
    is not (values past f32's range count as not finite)."""
    n = 64 * 7
    c = moving(fam, n, 9)
    for j, v in enumerate((np.inf, -np.inf, np.nan)):
        c[0, 64 * (2 * j + 1):64 * (2 * j + 2)] = F32(v)
    if c.shape[0] > 1:
        c[1, 64 * 6 + 10:64 * 6 + 20] = F32(np.nan)
    o = oracle((noise().seed(4) | P.multipass(c.shape[0])) >> FAM[fam][0](), 48000.0, n, c)
    want, _ = M.run(fam, noise_of(4, n), c, 48000.0)
    with np.errstate(over="ignore"):
        fin = np.isfinite(want.astype(F32))
    assert np.array_equal(np.isfinite(o), fin), (fam, np.flatnonzero(np.isfinite(o) != fin)[:10])


# ---------------------------------------------------------------- rate changes, reset, tick = process
@pytest.mark.parametrize("fam", AUDIO)
def test_rate_change_with_held_controls_then_reset(fam):
    """48 kHz -> 8 kHz -> 44.1 kHz on a running unit whose controls hold, then a reset: the model recomputes from its stored controls."""
    ctl = {"allpole": (0.7,), "moog": (1500.0, 0.4)}.get(fam, (1500.0, 2.0, 3.0) if fam != "morph" else (1500.0, 2.0, 0.5))[:FAM[fam][1]]
    ctl = tuple(float(F32(v)) for v in ctl)
    graph = (noise().seed(6) | dc(ctl)) >> FAM[fam][0]()
    olib().fo_set_denormal_emulation(0)
    u = OracleUnit(graph)
    m = M.Unit(fam, {"allpole": (1.0,), "moog": (1000.0, 0.1, 1.0)}.get(fam, (440.0, 1.0, 1.0)))
    x = noise_of(6, 4 * 300)
    c = np.repeat(np.array(ctl, F32)[:, None], 300, axis=1)
    for k, sr in enumerate((48000.0, 8000.0, 44100.0, None)):
        if sr is None:
            u.reset(); m.reset()
            u2 = OracleUnit((noise().seed(6) | dc(ctl)) >> FAM[fam][0]()); u2.set_sample_rate(44100.0)
            o = u.process_many(300)[0]
            assert np.array_equal(o, u2.process_many(300)[0])   # a reset unit is a new one at the same rate
            xs = x[:300]
        else:
            u.set_sample_rate(sr); m.set_sample_rate(sr)
            o = u.process_many(300)[0]
            xs = x[300 * k:300 * (k + 1)]
        want, bound = m.run(xs, c)
        within(fam, o, want, bound, (fam, sr))


@pytest.mark.parametrize("fam", AUDIO)
def test_tick_equals_process(fam):
    n = 64 * 5 + 13
    c = moving(fam, n, 12)
    g = (noise().seed(2) | P.multipass(c.shape[0])) >> FAM[fam][0]()
    olib().fo_set_denormal_emulation(0)
    a, b = OracleUnit(g), OracleUnit(g)
    a.set_sample_rate(44100.0); b.set_sample_rate(44100.0)
    p = a.process_many(n, c)[0]
    t = np.array([b.tick(c[:, i])[0] for i in range(n)], F32)
    assert np.array_equal(p, t)


# ---------------------------------------------------------------- fixed forms and BiquadBank
def fixed_cases():
    out = []
    for i, mode in enumerate(M.MODES):
        hz = getattr(P, f"{mode}_hz")
        for f, q, g in ((1000.0, 0.707, 4.0), (20.0, 10.0, 0.25), (15000.0, 0.5, 1.0)):
            out.append((mode, (f, q, g), hz(f, q, g) if i >= 6 else hz(f, q)))
    out += [("butterpass", (f,), butterpass_hz(f)) for f in (50.0, 2000.0, 20000.0)]
    out += [("resonator", (f, bw), resonator_hz(f, bw)) for f, bw in ((440.0, 20.0), (5000.0, 300.0))]
    out += [("moog", (f, q), moog_hz(f, q)) for f, q in ((300.0, 0.9), (4000.0, 0.2))]
    out += [(k, (f,), mk(f)) for k, mk in (("lowpole", lowpole_hz), ("highpole", highpole_hz), ("dcblock", dcblock_hz)) for f in (5.0, 3000.0)]
    out += [(k, (f, q), lowrez_hz(f, q)) for k, f, q in (("lowrez", 800.0, 0.9), ("lowrez", 6000.0, 0.3))]
    out += [("biquad", (-1.8, 0.81, 0.01, 0.02, 0.01), biquad(-1.8, 0.81, 0.01, 0.02, 0.01))]
    return out


@pytest.mark.parametrize("sr", RATES)
def test_fixed_forms_within_the_model(sr):
    for k, (fam, params, node) in enumerate(fixed_cases()):
        o = oracle(noise().seed(k) >> node, sr, 2000)
        want, bound = M.run(fam, noise_of(k, 2000), (), sr, params=params, fixed=True)
        within(fam, o, want, bound, (fam, params, sr))


# ---------------------------------------------------------------- the negative controls
MUTATIONS = {
    "swap_a": ("lowpass", "bell", "butterpass", "resonator"),
    "m1_sign": ("highpass", "notch", "peak", "allpass", "bell", "lowshelf", "highshelf", "morph"),
    "cutoff_only": ("lowpass", "bell", "resonator", "lowrez", "morph"),
    "late": ("lowpass", "butterpass", "resonator", "lowpole", "highpole", "lowrez"),
    "stale_rate": ("lowpass", "highshelf", "morph", "butterpass", "resonator", "lowpole", "highpole", "lowrez", "bandrez"),   # not moog(): it recomputes every sample
    "no_ps": ("moog",),
    "rez_fb": ("lowrez", "bandrez"),
}
def mutation_miss(mut, fam):
    """By how much the oracle misses the bound of the model with mutation `mut` (its worst error over the bound)."""
    n = 64 * 12
    c = moving(fam, n, 21)
    if mut == "stale_rate":   # a running unit changes rate with held controls
        ctl = c[:, 5:6].repeat(n, axis=1)
        u = OracleUnit((noise().seed(8) | dc(tuple(float(v) for v in ctl[:, 0]))) >> FAM[fam][0]())
        u.set_sample_rate(48000.0); u.process_many(200)
        u.set_sample_rate(8000.0)
        o = u.process_many(n)[0]
        m = M.Unit(fam, {"moog": (1000.0, 0.1, 1.0)}.get(fam, (440.0, 1.0, 1.0)), mutate=mut)
        m.set_sample_rate(48000.0); m.run(noise_of(8, 200), ctl[:, :200])
        m.set_sample_rate(8000.0)
        want, bound = m.run(noise_of(8, 200 + n)[200:], ctl)
    else:
        o = oracle((noise().seed(8) | P.multipass(c.shape[0])) >> FAM[fam][0](), 48000.0, n, c)
        want, bound = M.run(fam, noise_of(8, n), c, 48000.0, mutate=mut)
    return miss(o, want, bound)


@pytest.mark.parametrize("mut", list(MUTATIONS))
def test_every_mutation_misses_its_bound(mut):
    got = {f: mutation_miss(mut, f) for f in MUTATIONS[mut]}
    print(mut, {f: f"{v:.3g}" for f, v in got.items()})
    assert max(got.values()) >= 1e3 and min(got.values()) >= 10.0, (mut, got)


def test_report_per_family():
    """For every audio-rate family: the worst error-to-bound ratio over the moving controls at the three rates, and the smallest factor
    by which a mutation that applies to it misses its bound. Computed here, so the report does not depend on which tests ran before."""
    worst = {}
    for fam in AUDIO:
        for sr in RATES:
            n = 64 * 24
            c = moving(fam, n, 5)
            if sr == 8000.0 and fam != "allpole":
                c[0] = (c[0] * F32(0.2)).astype(F32)
                c[0, 0] = F32({"moog": 1000.0}.get(fam, 440.0))
            o = oracle((noise().seed(3) | P.multipass(c.shape[0])) >> FAM[fam][0](), sr, n, c)
            want, bound = M.run(fam, noise_of(3, n), c, sr)
            worst[fam] = max(worst.get(fam, 0.0), within(fam, o, want, bound, (fam, sr)))
    misses = {}
    for mut, fams in MUTATIONS.items():
        for fam in fams:
            misses[fam] = min(misses.get(fam, math.inf), mutation_miss(mut, fam))
    assert set(worst) == set(AUDIO) and set(misses) <= set(AUDIO)
    for fam in AUDIO:
        m = f"mutations miss by at least {misses[fam]:.3g}x" if fam in misses else "no mutation applies"
        print(f"{fam:>10}: worst {worst[fam]:.3g} of the bound; {m}")
    assert max(worst.values()) <= 1.0 and min(misses.values()) >= 10.0


# ---------------------------------------------------------------- the GPU file on the mock device
def test_gpu_filters_on_the_mock_device(mock_env):
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_filters.py"), "-m", "gpu", "-q", "-n", "8",
                        "-p", "no:cacheprovider", "--tb=short"], capture_output=True, text=True, env=mock_env, cwd=ROOT, timeout=3000)
    tail = r.stdout[-3000:]
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, tail
