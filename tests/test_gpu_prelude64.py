"""prelude64 graphs on the GPU: Sine<f64>, the nine SVF modes with f64 state, fixed (FixedSvf<f64, M>) and audio-rate (Svf<f64, M>), the
f64 biquads (Biquad, ButterLowpass, Resonator) and the one-pole family (Lowpole, Highpole, Allpole, DCBlock, Pinkpass, pink, brown).
Every case is compared bit for bit with the oracle (oracle/fo_prelude64.h), per voice, over 40 voices that differ in their parameters and
share one class."""
import ctypes as C
import os

import numpy as np
import pytest

from fundsp_b200 import prelude as p32
from fundsp_b200.net import Net
from fundsp_b200.prelude64 import *  # noqa: F401,F403
from fundsp_b200.sequencer import event
from oracle import OracleUnit, lib as olib, oracle_bank_render
import oracle_prelude64  # noqa: F401  (the oracle's prelude64 nodes, registered on OracleBackend)

pytestmark = pytest.mark.gpu
SR = 48000.0
N = 17000 + 13
V = 40
P_CENTER_Q_GAIN = 3


def fv(i, k=0):
    return ((i * 37 + k * 11) % 29) / 29.0


MODES = ("lowpass", "highpass", "bandpass", "notch", "peak", "allpass", "bell", "lowshelf", "highshelf")


def _fixed(m):
    hz = globals()[f"{m}_hz"]
    if MODES.index(m) >= 6:
        return lambda i: noise().seed(i) >> hz(300.0 + 40.0 * i, 0.6 + fv(i), 0.25 + 3.0 * fv(i, 1))
    return lambda i: noise().seed(i) >> hz(300.0 + 40.0 * i, 0.6 + fv(i))


def _audio(m):
    node = globals()[m]

    def mk(i):
        cut = sine_hz(1.5 + fv(i)) * dc(300.0) + dc(800.0 + 10.0 * i)
        q = dc(0.7 + fv(i, 2))
        if MODES.index(m) >= 6:
            return (noise().seed(i) | cut | q | (sine_hz(0.5) * dc(0.5) + dc(1.5 + fv(i)))) >> node()
        return (noise().seed(i) | cut | q) >> node()
    return mk


def _q(m):
    qf = globals()[f"{m}_q"]
    if MODES.index(m) >= 6:
        return lambda i: (noise().seed(i) | (saw_hz(0.7) * dc(400.0) + dc(1000.0 + 7.0 * i))) >> qf(1.0 + fv(i), 2.0 + fv(i, 1))
    return lambda i: (noise().seed(i) | (saw_hz(0.7) * dc(400.0) + dc(1000.0 + 7.0 * i))) >> qf(1.0 + fv(i))


def headline(i):   # saw_hz(f) >> lowpass_hz(fc, q) as written against prelude64 (fc stays below Nyquist at any voice count)
    return saw_hz(55.0 + 0.37 * i) >> lowpass_hz(400.0 + 3.0 * (i % 1000), 0.7 + fv(i))


def _ctl(i, lo, span, rate=1.7):   # a control signal that changes every sample
    return sine_hz(rate + fv(i)) * dc(span) + dc(lo)


FILTERS = {
    "biquad": lambda i: noise().seed(i) >> biquad(-1.6 + 0.01 * i, 0.7 - 0.002 * i, 0.03, 0.06, 0.03),
    "butterpass_hz": lambda i: noise().seed(i) >> butterpass_hz(200.0 + 50.0 * i),
    "butterpass_audio": lambda i: (noise().seed(i) | _ctl(i, 1000.0 + 10.0 * i, 400.0)) >> butterpass(),
    "resonator_hz": lambda i: noise().seed(i) >> resonator_hz(300.0 + 40.0 * i, 5.0 + 10.0 * fv(i)),
    "resonator_audio": lambda i: (noise().seed(i) | _ctl(i, 900.0 + 10.0 * i, 300.0) | (sine_hz(0.3) + dc(4.0 + fv(i)))) >> resonator(),
    "lowpole_hz": lambda i: noise().seed(i) >> lowpole_hz(50.0 + 30.0 * i),
    "lowpole_audio": lambda i: (noise().seed(i) | _ctl(i, 500.0 + 10.0 * i, 300.0)) >> lowpole(),
    "highpole_hz": lambda i: noise().seed(i) >> highpole_hz(20.0 + 30.0 * i),
    "highpole_audio": lambda i: (noise().seed(i) | _ctl(i, 400.0 + 10.0 * i, 300.0)) >> highpole(),
    "allpole_delay": lambda i: noise().seed(i) >> allpole_delay(0.3 + 0.05 * i),
    "allpole_audio": lambda i: (noise().seed(i) | (sine_hz(2.0) * dc(0.2) + dc(0.5 + 0.02 * i))) >> allpole(),
    "dcblock_hz": lambda i: (noise().seed(i) + dc(0.5)) >> dcblock_hz(5.0 + i),
    "dcblock": lambda i: (noise().seed(i) + dc(0.3 + 0.01 * i)) >> dcblock(),
    "pinkpass": lambda i: (noise().seed(i) * dc(0.5 + fv(i))) >> pinkpass(),
    "pink": lambda i: pink() * dc(0.5 + fv(i)),
    "brown": lambda i: brown() * dc(0.5 + fv(i)),
    # constant (dc) control inputs: after a rate change the coefficients are recomputed although no input changes
    "svf_lowpass_dc": lambda i: (noise().seed(i) | dc((700.0 + 10.0 * i, 1.0 + fv(i)))) >> lowpass(),
    "resonator_dc": lambda i: (noise().seed(i) | dc((600.0 + 20.0 * i, 8.0))) >> resonator(),
    "lowpole_dc": lambda i: (noise().seed(i) | dc(100.0 + 5.0 * i)) >> lowpole(),
}


CASES = {
    **FILTERS,
    **{f"svf_{m}_hz": _fixed(m) for m in MODES},
    **{f"svf_{m}_audio": _audio(m) for m in MODES},
    **{f"svf_{m}_q": _q(m) for m in ("lowpass", "bell")},
    "sine_hz": lambda i: sine_hz(110.0 + 17.3 * i),
    "sine_fm": lambda i: (sine_hz(3.0 + fv(i)) * dc(50.0) + dc(440.0 + i)) >> sine(),
    "sine_phase": lambda i: sine_hz(1000.0 + i).phase(fv(i)),
    "headline": headline,
    "lowpass_sub_hertz": lambda i: noise().seed(i) >> lowpass_hz(2.0 + 0.1 * i, 0.7),   # where f64 state matters
    "mixed_precision": lambda i: noise().seed(i) >> p32.lowpass_hz(2000.0 + 10.0 * i, 1.0) >> highpass_hz(20.0 + i, 0.7) >> p32.bell_hz(1000.0, 1.0, 2.0),
    "net_mixed": lambda i: (Net.wrap(sine_hz(220.0 + i).phase(0.1)) >> Net.wrap(p32.lowpass_hz(3000.0, 1.0)) >> Net.wrap(bell_hz(800.0 + i, 2.0, 3.0))).node(),
    "event": lambda i: event(saw_hz(110.0 + i) >> lowpass_hz(900.0 + 5.0 * i, 1.0 + fv(i)), (30.0 + 97.3 * i) / SR, (30.0 + 97.3 * i + 9000.0) / SR, i % 2, 40.0 / SR, 300.0 / SR),
}


def _bank(mk, n_voices=V, sr=SR, **kw):
    from fundsp_b200.bank import GpuBank
    return GpuBank([mk(i) for i in range(n_voices)], sample_rate=sr, **kw)


def _units(mk, sr=SR, n_voices=V):
    us = [OracleUnit(mk(i)) for i in range(n_voices)]
    for u in us:
        u.set_sample_rate(sr)
    return us


@pytest.mark.parametrize("name", sorted(CASES))
def test_prelude64_case_matches_oracle(name):
    olib().fo_set_denormal_emulation(0)
    mk = CASES[name]
    b = _bank(mk, per_voice=True, mix=True)
    g, mx = b.render_samples(N)
    o, omx = oracle_bank_render([mk(i) for i in range(V)], SR, N, mix=True, threads=4)
    assert len(b.classes()) == 1, [c["signature"] for c in b.classes()]
    assert g.shape == o.shape and np.isfinite(g).all() and np.abs(o).max() > 1e-3
    bad = int((g != o).sum())
    assert bad == 0, (name, bad, float(np.abs(g - o).max()), b.classes()[0]["signature"])
    assert np.abs(mx - omx).max() <= 2e-6 * max(1.0, float(np.abs(o).sum(axis=0).max()))


@pytest.mark.parametrize("name", ["svf_bell_hz", "svf_highshelf_audio", "sine_fm", "headline"])
def test_at_44100(name):
    olib().fo_set_denormal_emulation(0)
    mk = CASES[name]
    g, _ = _bank(mk, sr=44100.0, per_voice=True).render_samples(N)
    o, _ = oracle_bank_render([mk(i) for i in range(V)], 44100.0, N, threads=4)
    assert np.array_equal(g, o), int((g != o).sum())


@pytest.mark.parametrize("name", ["sine_fm", "svf_lowpass_audio", "svf_lowshelf_hz", "headline"])
def test_ragged_process_sizes(name):
    olib().fo_set_denormal_emulation(0)
    mk = CASES[name]
    b = _bank(mk, per_voice=True)
    us = _units(mk)
    for k, sz in enumerate([64, 61, 8, 7, 1, 0, 64, 33, 64, 5, 64, 64, 17] * 8):
        got = b.process(sz)
        want = np.concatenate([u.process(sz) for u in us])
        assert np.array_equal(got, want), (k, sz, int((got != want).sum()))


@pytest.mark.parametrize("name", ["svf_peak_audio", "sine_hz", "headline", "svf_lowpass_dc", "resonator_dc", "lowpole_dc", "butterpass_audio"])
def test_reset_clone_and_sample_rate_change(name):
    olib().fo_set_denormal_emulation(0)
    mk = CASES[name]
    b = _bank(mk, per_voice=True)
    g1, _ = b.render_samples(3000)
    c = b.clone()
    g2, _ = b.render_samples(2000)
    gc, _ = c.render_samples(2000)
    assert np.array_equal(g2, gc)
    b.reset()
    g3, _ = b.render_samples(3000)
    b.set_sample_rate(44100.0)                      # mid-stream: the running state continues at the new rate
    g4, _ = b.render_samples(2500)
    for i in range(V):
        u = OracleUnit(mk(i)); u.set_sample_rate(SR)
        assert np.array_equal(g1[i], u.process_many(3000))
        u.reset()
        assert np.array_equal(g3[i], u.process_many(3000))
        u.set_sample_rate(44100.0)
        want = u.process_many(2500)
        assert np.array_equal(g4[i], want), (i, int((g4[i] != want).sum()))


def test_live_center_q_gain_setting():
    """Setting::center_q_gain on running FixedSvf<f64, Bell> voices: F::from_f32 of each value, coefficients recomputed in f64."""
    olib().fo_set_denormal_emulation(0)
    mk = CASES["svf_bell_hz"]
    b = _bank(mk, per_voice=True)
    us = _units(mk)
    n1, n2 = 64 * 30 + 5, 64 * 40 + 3
    g1, _ = b.render_samples(n1)
    assert np.array_equal(g1, np.stack([u.process_many(n1) for u in us]))
    for v in range(0, V, 3):
        vals = (1500.0 + 10.0 * v, 3.0, 0.5 + fv(v))
        b.set(v, P_CENTER_Q_GAIN, vals)
        us[v].L.fo_set(us[v].h, P_CENTER_Q_GAIN, (C.c_float * 3)(*vals), 3, 0, None, 0)
    g2, _ = b.render_samples(n2)
    o2 = np.stack([u.process_many(n2) for u in us])
    assert np.array_equal(g2, o2), int((g2 != o2).sum())
    assert not np.array_equal(g2[0], _bank(mk, n_voices=1, per_voice=True).render_samples(n1 + n2)[0][0, n1:])


def test_headline_sixteen_thousand_voices():
    """16 384 voices of saw_hz >> lowpass_hz in prelude64: one class, sampled rows equal to the oracle, and the mix equal to the exact
    summation-order model of tests/test_gpu_mix.py applied to the rows."""
    if "mock" in os.environ.get("FDSP_B200_LIB", ""):
        pytest.skip("a full-size bank is for the GPU (the CPU mock device walks every voice serially)")
    import test_gpu_mix as MX
    olib().fo_set_denormal_emulation(0)
    n_voices, n = 16384, 4800
    voices = [headline(i) for i in range(n_voices)]
    b = _bank(headline, n_voices, per_voice=True, mix=True)
    assert len(b.classes()) == 1 and b.classes()[0]["signature"].endswith("FixedSvf64>")
    g, mx = b.render_samples(n)
    idx = list(range(0, n_voices, 997)) + [n_voices - 1]
    o, _ = oracle_bank_render([headline(i) for i in idx], SR, n, threads=4)
    assert np.array_equal(g[idx], o)
    classes = MX.bank_classes(b, voices)
    pipe = MX.is_pipelined(classes)
    MX.check_mix(mx, g, classes, MX.launch_segments(n, classes, g.shape[0], g.shape[1], True, pipe), pipe, "prelude64 headline")


@pytest.mark.parametrize("name", ["p64_sine_hz", "p64_lowpass_hz", "p64_bell_hz", "p64_lowpass_swept", "p64_resonator_hz", "p64_lowpole_hz", "p64_pink"])
def test_matches_the_reference_crate(name):
    """Vectors of the real crate (oracle/ref_dump64), when they have been generated: the bank renders them bit for bit."""
    from test_prelude64_cpu import reference_vector
    g, want = reference_vector(name)
    from fundsp_b200.bank import GpuBank
    got, _ = GpuBank([g], per_voice=True, sample_rate=SR).render_samples(want.shape[1])
    assert np.array_equal(got[0], want), (name, int((got[0] != want).sum()))
