"""`update(x, dt, f)` on the GPU: System<X, F> (src/system.rs) with its update function `|t, dt, x| ..` compiled into the voice program.
Every case is compared bit for bit, per voice, with the oracle's System (tests/update_oracle.py), whose update function runs the same
text's arguments through the oracle's closure interpreter and sets the oracle's nodes; the voices differ in their captured values."""
import ctypes as C
import os

import numpy as np
import pytest

from fundsp_b200.capi import FdspError, ERR_UNSUPPORTED
from fundsp_b200.net import Net
from fundsp_b200.prelude import *  # noqa: F401,F403
from fundsp_b200.sequencer import event, slot
from oracle import OracleUnit, lib as olib, oracle_bank_render
from update_oracle import oracle_of

pytestmark = pytest.mark.gpu
SR = 48000.0
N = 17000 + 13
V = 40
MOCK = "mock" in os.environ.get("FDSP_B200_LIB", "")
P_CENTER, P_CENTER_Q = 1, 2


def fv(i, k=0):
    return ((i * 37 + k * 11) % 29) / 29.0


SWEEP = "|t, dt, x| x.set(Setting::center(600.0 + 400.0 * sin_hz(r, t)).right())"
SWEEP_Q = "|t, dt, x| { let u = sin_hz(r, t); x.set(Setting::center_q(800.0 + 500.0 * u, 1.0 + 0.5 * u).right()); }"
SWEEP_QG = "|t, dt: f32, x| { let u = tri_hz(r, t); x.set(Setting::center_q_gain(900.0 + 600.0 * u, 0.8 + 0.2 * u, 1.0 + u).right()) }"
AUDIO = lambda i: saw_hz(110.0 + 3.0 * i)
SVF_MODES = [lambda: lowpass_hz(1000.0, 1.0), lambda: highpass_hz(1000.0, 1.0), lambda: bandpass_hz(1000.0, 1.0), lambda: notch_hz(1000.0, 1.0),
             lambda: peak_hz(1000.0, 1.0), lambda: allpass_hz(1000.0, 1.0), lambda: bell_hz(1000.0, 1.0, 2.0), lambda: lowshelf_hz(1000.0, 1.0, 2.0),
             lambda: highshelf_hz(1000.0, 1.0, 0.5)]

# the Resonator takes no setting (src/biquad.rs:340-387 has no `set`): its two statements are ignored and it keeps its center and q
BUTTER_RESON = ("|t, dt, x| { let u = sin_hz(r, t); x.set(Setting::center(1500.0 + 1000.0 * u).left().right());"
                " x.set(Setting::center_q(700.0 - 300.0 * u, 40.0 + 20.0 * u).right()); x.set(Setting::center(900.0).right()) }")
BUTTER_ONLY = "|t, dt, x| { let u = sin_hz(r, t); x.set(Setting::center(1500.0 + 1000.0 * u).left().right()) }"
SWEEP_AT = "|t, dt, x| {{ let u = sin_hz(r, t); x.set(Setting::center(700.0 + 500.0 * u){a}); x.set(Setting::center(2000.0 - 900.0 * u){b}) }}"

CASES = {
    "svf_center": lambda i: update(AUDIO(i) >> lowpass_hz(1000.0, 1.0), 0.002, SWEEP, r=0.5 + fv(i)),
    **{f"svf_mode{m}_center_q_gain": (lambda m: lambda i: update(AUDIO(i) >> SVF_MODES[m](), 0.003, SWEEP_QG, r=1.0 + fv(i)))(m) for m in range(9)},
    "svf_center_q_dt_below_block": lambda i: update(AUDIO(i) >> bandpass_hz(1000.0, 1.0), 0.0005, SWEEP_Q, r=2.0 + fv(i)),
    "svf_dt_one_block": lambda i: update(AUDIO(i) >> lowpass_hz(1000.0, 1.0), 64.0 / SR, SWEEP, r=3.0 + fv(i)),
    "svf_dt_zero": lambda i: update(AUDIO(i) >> lowpass_hz(1000.0, 1.0), 0.0, SWEEP, r=1.0 + fv(i)),
    "butterpass_resonator": lambda i: update(AUDIO(i) >> butterpass_hz(1000.0) >> resonator_hz(500.0, 50.0), 0.002, BUTTER_RESON, r=0.7 + fv(i)),
    "biquad_coefficients": lambda i: update(AUDIO(i) >> biquad(-1.8, 0.82, 0.005, 0.01, 0.005), 0.002,
                                            "|t, dt, x| { let a = 0.8 + 0.15 * sin_hz(r, t); x.set(Setting::biquad(-2.0 * a, a * a, 0.25 * (1.0 - a) * (1.0 - a), 0.5 * (1.0 - a) * (1.0 - a), 0.25 * (1.0 - a) * (1.0 - a)).right()) }",
                                            r=1.0 + fv(i)),
    "onepoles_index": lambda i: update(AUDIO(i) >> lowpole_hz(500.0) >> highpole_hz(50.0) >> dcblock_hz(10.0), 0.001,
                                       "|t, dt, x| { let u = sin_hz(r, t) * 0.5 + 0.5; x.set(Setting::center(200.0 + 3000.0 * u).index(0).index(1).index(1));"
                                       " x.set(Setting::center(20.0 + 200.0 * u).left().right()); x.set(Setting::center(5.0 + 20.0 * u).index(1)) }",
                                       r=0.3 + fv(i)),
    "dc_value_and_ignored": lambda i: update(dc(1.0) >> (pass_() * sine_hz(220.0 + i)), 0.004,
                                             "|t, dt, x| { x.set(Setting::value(0.5 + 0.5 * sin_hz(r, t)).left()); x.set(Setting::pan(0.3).left()); x.set(Setting::center(1.0).index(7)) }",
                                             r=1.0 + fv(i)),
    "pan": lambda i: update(AUDIO(i) >> pan(0.0), 0.002, "|t, dt, x| x.set(Setting::pan(sin_hz(r, t) + dt).right())", r=0.5 + fv(i)),
    "stack_branch_thru": lambda i: update((AUDIO(i) >> ~lowpass_hz(1000.0, 1.0)) | (AUDIO(i + 1) >> (lowpass_hz(500.0, 1.0) ^ highpass_hz(900.0, 2.0))),
                                          0.002, SWEEP_AT.format(a=".left().right()", b=".right().right().right()"), r=1.0 + fv(i)),
    "bus": lambda i: update(AUDIO(i) >> (lowpass_hz(800.0, 1.0) & bandpass_hz(1500.0, 2.0)), 0.002, SWEEP_AT.format(a=".right().left()", b=".right().right()"),
                            r=0.5 + fv(i)),
    "multi": lambda i: update(AUDIO(i) >> split(3) >> stacki(3, lambda k: lowpass_hz(600.0 + 300.0 * k, 1.0)), 0.002,
                              SWEEP_AT.format(a=".right().index(0)", b=".right().index(2)"), r=0.5 + fv(i)),
    "set_reaching_the_oscillator": lambda i: update(AUDIO(i) >> lowpass_hz(1000.0, 1.0), 0.002,
                                                    "|t, dt, x| { x.set(Setting::center(5.0).left().right()); x.set(Setting::center(700.0 + 300.0 * sin_hz(r, t)).right()) }",
                                                    r=1.0 + fv(i)),
    "in_net": lambda i: (Net.wrap(update(AUDIO(i) >> lowpass_hz(1000.0, 1.0), 0.002, SWEEP, r=0.5 + fv(i))) >> Net.wrap(pass_() * dc(0.5))).node(),
    "in_event": lambda i: event(update(AUDIO(i) >> lowpass_hz(1000.0, 1.0), 0.002, SWEEP, r=0.5 + fv(i)), (30.0 + 97.3 * i) / SR,
                                (30.0 + 97.3 * i + 9000.0) / SR, i % 2, 40.0 / SR, 300.0 / SR),
    "in_slot": lambda i: slot(update(AUDIO(i) >> lowpass_hz(1000.0, 1.0), 0.002, SWEEP, r=0.5 + fv(i))),
    "in_feedback": lambda i: noise().seed(i) * 0.1 >> feedback(update(lowpass_hz(1000.0, 1.0) * 0.9, 0.002,
                                                                      "|t, dt, x| x.set(Setting::center(600.0 + 400.0 * sin_hz(r, t)))", r=1.0 + fv(i))),
    "oversampled": lambda i: AUDIO(i) >> oversample(update(lowpass_hz(1000.0, 1.0), 0.002, "|t, dt, x| x.set(Setting::center(3000.0 + 2500.0 * sin_hz(r, t)))",
                                                           r=2.0 + fv(i))),
}


# what the reference computes, where the oracle's own node would take a setting the reference's ignores (the oracle's Resonator has a set())
ORACLE = {"butterpass_resonator": lambda i: update(AUDIO(i) >> butterpass_hz(1000.0) >> resonator_hz(500.0, 50.0), 0.002, BUTTER_ONLY, r=0.7 + fv(i))}


def expected(name, i):
    """Voice i of case `name` as the oracle builds it."""
    return oracle_of(ORACLE.get(name, CASES[name])(i))


def _bank(mk, n_voices=V, **kw):
    from fundsp_b200.bank import GpuBank
    return GpuBank([mk(i) for i in range(n_voices)], sample_rate=SR, **kw)


def _units(mk, n_voices=V):
    us = [OracleUnit(oracle_of(mk(i))) for i in range(n_voices)]
    for u in us:
        u.set_sample_rate(SR)
    return us


@pytest.mark.parametrize("name", sorted(CASES))
def test_update_case_matches_oracle(name):
    olib().fo_set_denormal_emulation(0)
    mk = CASES[name]
    b = _bank(mk, per_voice=True, mix=True)
    g, mx = b.render_samples(N)
    o, omx = oracle_bank_render([expected(name, i) for i in range(V)], SR, N, mix=True, threads=4)
    sigs = [c["signature"] for c in b.classes()]
    assert len(sigs) == 1 and "System<" in sigs[0], sigs
    assert g.shape == o.shape and np.isfinite(g).all() and np.abs(o).max() > 1e-3
    bad = int((g != o).sum())
    assert bad == 0, (name, bad, float(np.abs(g - o).max()), sigs[0])
    assert np.abs(mx - omx).max() <= 2e-6 * max(1.0, float(np.abs(o).sum(axis=0).max()))


@pytest.mark.parametrize("name", ["svf_center", "svf_center_q_dt_below_block", "in_event"])
def test_ragged_process_sizes(name):
    olib().fo_set_denormal_emulation(0)
    mk = CASES[name]
    b = _bank(mk, per_voice=True)
    us = _units(mk)
    for k, sz in enumerate([1, 7, 63, 64, 1000, 0, 64, 33, 5, 17, 2, 1000, 63, 64, 64] * 6):
        if sz > 64:   # process() takes at most 64 samples (MAX_BUFFER_SIZE); a longer call is a render, 64-sample blocks and the tail
            got = b.render_samples(sz)[0].reshape(-1, sz)
            want = np.concatenate([u.process_many(sz) for u in us])
        else:
            got = b.process(sz)
            want = np.concatenate([u.process(sz) for u in us])
        assert np.array_equal(got, want), (k, sz, int((got != want).sum()))


def test_reset_clone_and_sample_rate_change():
    """Reset and clone keep the last-set values; after a rate change the first block runs with the last-set cutoff at the new rate."""
    olib().fo_set_denormal_emulation(0)
    mk = lambda i: update(AUDIO(i) >> lowpass_hz(1000.0, 1.0), 0.01, SWEEP_Q, r=2.0 + fv(i))
    b = _bank(mk, per_voice=True)
    g1, _ = b.render_samples(3000 + 5)
    c = b.clone()
    g2, _ = b.render_samples(2000)
    gc, _ = c.render_samples(2000)
    assert np.array_equal(g2, gc)
    b.reset()
    g3, _ = b.render_samples(3000 + 5)
    assert np.array_equal(g1, g3)
    b.set_sample_rate(44100.0)
    g4, _ = b.render_samples(2500)
    o3, o4 = [], []
    for i in range(V):
        u = OracleUnit(oracle_of(mk(i))); u.set_sample_rate(SR)
        u.process_many(3000 + 5); u.process_many(2000); u.reset()
        o3.append(u.process_many(3000 + 5))
        u.set_sample_rate(44100.0)
        o4.append(u.process_many(2500))
    assert np.array_equal(g3, np.stack(o3)) and np.array_equal(g4, np.stack(o4)), (int((g4 != np.stack(o4)).sum()))


def test_bank_set_through_the_system():
    """fdsp_bank_set on a voice with `update`: a setting of a target holds until the next update point, one elsewhere at once."""
    olib().fo_set_denormal_emulation(0)
    mk = lambda i: update(AUDIO(i) >> lowpass_hz(1000.0, 1.0) >> highpass_hz(100.0, 1.0), 0.02,
                          "|t, dt, x| x.set(Setting::center(600.0 + 400.0 * sin_hz(r, t)).left().right())", r=1.0 + fv(i))
    b = _bank(mk, per_voice=True)
    us = _units(mk)
    got, want = [], []
    for step, n in enumerate([700, 64 * 5 + 3, 1000, 2000]):
        got.append(b.render_samples(n)[0])
        want.append(np.stack([u.process_many(n) for u in us]))
        for v in range(step % 3, V, 3):
            for kind, vals, addr in [(P_CENTER_Q, (300.0 + v, 2.0), ((1, 0), (1, 1))), (P_CENTER, (150.0 + v,), ((1, 1),))]:
                b.set(v, kind, vals, address=addr)
                us[v].L.fo_set(us[v].h, kind, (C.c_float * len(vals))(*vals), len(vals), 0, (C.c_int64 * 4)(*[w for a in addr for w in a]), len(addr))
    g, o = np.concatenate(got, axis=2), np.concatenate(want, axis=2)
    assert np.array_equal(g, o), int((g != o).sum())


def test_refused_targets_build_no_bank():
    """Nodes that take the setting in the reference but whose coefficients the device does not recompute: the fixed Moog, the audio-rate
    panner, prelude64 filters. (An audio-rate Svf has no set() in the reference: a statement reaching it is ignored, not refused.)"""
    from fundsp_b200 import prelude64
    from fundsp_b200.bank import GpuBank
    for x, text in [(saw_hz(110.0) >> moog_hz(1000.0, 0.5), "|t, dt, x| x.set(Setting::center(500.0).right())"),
                    (saw_hz(110.0) >> (pass_() | dc(0.0)) >> panner(), "|t, dt, x| x.set(Setting::pan(0.5).right())"),
                    (saw_hz(110.0) >> prelude64.lowpass_hz(1000.0, 1.0), "|t, dt, x| x.set(Setting::center(500.0).right())")]:
        with pytest.raises(FdspError) as e:
            GpuBank([update(x, 0.002, text)], sample_rate=SR)
        assert e.value.code == ERR_UNSUPPORTED and "Setting::" in str(e.value) and "which an update function cannot set" in str(e.value), str(e.value)


def test_sixteen_thousand_voices_one_class_mix_model():
    if MOCK:
        pytest.skip("a full-size bank is for the GPU (the CPU mock device walks every voice serially)")
    from test_gpu_mix import render_and_check
    n_voices, n = 16384, 4800
    mk = lambda i: update(saw_hz(55.0 + (i % 500)) >> lowpass_hz(1000.0, 1.0), 0.002, SWEEP, r=0.5 + (i % 61) / 16.0)
    _, _, classes, _, _ = render_and_check([mk(i) for i in range(n_voices)], n, mix_only_too=False, oracle=True,
                                           voices_again=lambda: [oracle_of(mk(i)) for i in range(n_voices)], what="update svf")
    assert len(classes) == 1
