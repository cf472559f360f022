"""The Atan and Adaptive waveshapes on the GPU: shape(Atan(h)), shape(Adaptive(timescale, inner)) for every inner kind, and both in the
four nonlinear biquad families with fixed and audio-rate coefficients. Every case is compared bit for bit with the oracle
(oracle/fo_shapes.h), per voice, over 40 voices that differ in their parameters and share one class."""
import os

import numpy as np
import pytest

from fundsp_b200.net import Net
from fundsp_b200.prelude import *  # noqa: F401,F403
from fundsp_b200.sequencer import event
from oracle import OracleUnit, lib as olib, oracle_bank_render
import oracle_shapes  # noqa: F401  (the oracle's Atan / Adaptive nodes, registered on OracleBackend)

pytestmark = pytest.mark.gpu
SR = 48000.0
N = 17000 + 13
V = 40


def fv(i, k=0):
    return ((i * 37 + k * 11) % 29) / 29.0


INNER = {   # one inner shape per kind, its parameter varying per voice
    0: lambda i: Clip(0.5 + fv(i)), 1: lambda i: ClipTo(-0.4 - 0.3 * fv(i), 0.6), 2: lambda i: Tanh(0.5 + 2.0 * fv(i)),
    3: lambda i: Softsign(1.0 + fv(i)), 4: lambda i: Crush(3.0 + (i % 5)), 5: lambda i: SoftCrush(2.0 + (i % 4)), 6: lambda i: Atan(0.3 + 3.0 * fv(i)),
}


def adaptive(i, kind=2):
    return Adaptive(0.002 + 0.0005 * (i % 7), INNER[kind](i))


def level(i):   # an input whose level changes by orders of magnitude
    return (saw_hz(55.0 + i) * dc(0.02 + 3.0 * fv(i, 1))) + (sine_hz(0.7) * dc(0.5))


# the four families: (fixed builder, audio-rate builder, audio-rate control inputs)
FAMILIES = {
    "resonator": (lambda d, s, i: (dresonator_hz if d else fresonator_hz)(s, 300.0 + 20.0 * i, 2.0 + fv(i)),
                  lambda d, s, i: (noise().seed(i) | (sine_hz(1.5) * dc(200.0) + dc(700.0 + 5.0 * i)) | dc(3.0)) >> (dresonator if d else fresonator)(s)),
    "lowpass": (lambda d, s, i: (dlowpass_hz if d else flowpass_hz)(s, 600.0 + 30.0 * i, 1.5 + fv(i)),
                lambda d, s, i: (noise().seed(i) | (sine_hz(2.0) * dc(300.0) + dc(900.0)) | dc(4.0 + fv(i))) >> (dlowpass if d else flowpass)(s)),
    "highpass": (lambda d, s, i: (dhighpass_hz if d else fhighpass_hz)(s, 200.0 + 10.0 * i, 2.5),
                 lambda d, s, i: (noise().seed(i) | (sine_hz(3.0) * dc(100.0) + dc(400.0)) | (sine_hz(0.5) + dc(3.0))) >> (dhighpass if d else fhighpass)(s)),
    "bell": (lambda d, s, i: (dbell_hz if d else fbell_hz)(s, 1000.0 + 10.0 * i, 2.0, 4.0 + fv(i)),
             lambda d, s, i: (noise().seed(i) | (sine_hz(1.0) * dc(500.0) + dc(1500.0)) | dc(2.0) | (sine_hz(0.3) + dc(3.0))) >> (dbell if d else fbell)(s)),
}


def _biquad_case(fi, fam, ri, rate, si, shp):
    """DirtyBiquad or FbBiquad alternating over the cases, so that each family meets both shapes in both; an Adaptive case has one inner
    kind for all its voices (the kind is part of the class)."""
    dirty, kind = (fi + ri + si) % 2 == 0, (2 * fi + ri) % 7
    fixed, audio = FAMILIES[fam]

    def mk(i):
        s = Atan(0.5 + 4.0 * fv(i)) if shp == "atan" else adaptive(i, kind)
        return (noise().seed(i) * dc(0.5 + fv(i, 2))) >> fixed(dirty, s, i) if rate == "fixed" else audio(dirty, s, i)
    return mk


CASES = {
    "shape_atan": lambda i: level(i) >> shape(Atan(0.3 + 4.0 * fv(i))),
    "shape_atan_in_chain": lambda i: noise().seed(i) >> lowpass_hz(800.0 + 10.0 * i, 1.0) >> shape(Atan(2.0 + fv(i))) >> highpass_hz(100.0, 0.7),
    **{f"shape_adaptive_{k}": (lambda k: lambda i: level(i) >> shape(adaptive(i, k)))(k) for k in range(7)},
    **{f"nlb_{fam}_{rate}_{shp}": _biquad_case(fi, fam, ri, rate, si, shp)
       for fi, fam in enumerate(FAMILIES) for ri, rate in enumerate(("fixed", "audio")) for si, shp in enumerate(("atan", "adaptive"))},
    "net_adaptive": lambda i: ((Net.wrap(level(i)) >> Net.wrap(shape(adaptive(i, 6)))) >> Net.wrap(lowpass_hz(2000.0, 1.0))).node(),
    "event_adaptive": lambda i: event(level(i) >> shape(adaptive(i, 2)), (30.0 + 97.3 * i) / SR, (30.0 + 97.3 * i + 9000.0) / SR, i % 2, 40.0 / SR, 300.0 / SR),
    "moog_then_adaptive": lambda i: noise().seed(i) >> moog_hz(800.0 + 20.0 * i, 0.6) >> shape(adaptive(i, 6)),
}


def _bank(mk, n_voices=V, sr=SR, **kw):
    from fundsp_b200.bank import GpuBank
    return GpuBank([mk(i) for i in range(n_voices)], sample_rate=sr, **kw)


@pytest.mark.parametrize("name", sorted(CASES))
def test_shape_case_matches_oracle(name):
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


@pytest.mark.parametrize("name", ["shape_atan", "shape_adaptive_6", "nlb_bell_fixed_adaptive", "nlb_lowpass_audio_adaptive"])
def test_at_44100(name):
    olib().fo_set_denormal_emulation(0)
    mk = CASES[name]
    g, _ = _bank(mk, sr=44100.0, per_voice=True).render_samples(N)
    o, _ = oracle_bank_render([mk(i) for i in range(V)], 44100.0, N, threads=4)
    assert np.array_equal(g, o), int((g != o).sum())


@pytest.mark.parametrize("name", ["shape_atan", "shape_adaptive_4", "nlb_resonator_audio_adaptive"])
def test_ragged_process_sizes(name):
    olib().fo_set_denormal_emulation(0)
    mk = CASES[name]
    b = _bank(mk, per_voice=True)
    us = [OracleUnit(mk(i)) for i in range(V)]
    for u in us:
        u.set_sample_rate(SR)
    for k, sz in enumerate([64, 61, 8, 7, 1, 0, 64, 33, 64, 5, 64, 64, 17] * 8):
        got = b.process(sz)
        want = np.concatenate([u.process(sz) for u in us])
        assert np.array_equal(got, want), (k, sz, int((got != want).sum()))


@pytest.mark.parametrize("name", ["shape_adaptive_2", "nlb_highpass_fixed_adaptive"])
def test_reset_starts_from_the_reset_level_and_clone_continues(name):
    """A new unit's level estimate starts at 0, a reset one's at 1e-3 (src/shape.rs:173-196): the render after reset() equals the
    oracle's reset units, and differs from the first render."""
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
    o1, o3 = [], []
    for i in range(V):
        u = OracleUnit(mk(i)); u.set_sample_rate(SR)
        o1.append(u.process_many(3000))
        u.reset()
        o3.append(u.process_many(3000))
    assert np.array_equal(g1, np.stack(o1))
    assert np.array_equal(g3, np.stack(o3)), int((g3 != np.stack(o3)).sum())
    assert not np.array_equal(g1, g3)


def test_sixteen_thousand_voices_one_class():
    """16 384 voices of shape(Atan(h)) with per-voice hardness: one class, the launches of the shape(Tanh(h)) bank, and a fixed sample of
    voices equal to the oracle."""
    if "mock" in os.environ.get("FDSP_B200_LIB", ""):
        pytest.skip("a full-size bank is for the GPU (the CPU mock device walks every voice serially)")
    olib().fo_set_denormal_emulation(0)
    n_voices, n = 16384, 4800
    mk = lambda i: saw_hz(50.0 + 0.05 * i).phase(0.0) >> shape(Atan(0.5 + (i % 97) / 32.0))
    ref = lambda i: saw_hz(50.0 + 0.05 * i).phase(0.0) >> shape(Tanh(0.5 + (i % 97) / 32.0))
    b = _bank(mk, n_voices, per_voice=True, mix=True)
    r = _bank(ref, n_voices, per_voice=True, mix=True)
    assert len(b.classes()) == 1
    l0, r0 = b.launch_count(), r.launch_count()
    g, _ = b.render_samples(n)
    r.render_samples(n)
    assert b.launch_count() - l0 == r.launch_count() - r0
    idx = list(range(0, n_voices, 997)) + [n_voices - 1]
    o, _ = oracle_bank_render([mk(i) for i in idx], SR, n, threads=4)
    assert np.array_equal(g[idx], o)


def _close(g, o):
    """The mix bar of DESIGN.md §4: a bank's CTA-level sum associates differently from the sequencer's left fold over its active events."""
    tol = 1e-5 * np.maximum(np.abs(o), 1e-2 * np.abs(o).max())
    return bool(np.all(np.abs(g - o) <= tol))


def test_live_pushes_of_adaptive_events_start_from_a_new_units_state():
    """Sequencer::push into a running 48 kHz sequencer only re-rates the unit (src/sequencer.rs:369): a pushed Adaptive starts from the
    level estimate of a new unit (0.0). The events pushed before the rate was set were reset by Sequencer::set_sample_rate (1e-3). Both
    paths of a live push are taken: a new class (the bank grows) and the slot of a finished event of the same class."""
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.sequencer import Sequencer, Fade, ReplayMode
    from oracle import OracleBackend
    L = olib()
    L.fo_set_denormal_emulation(0)
    unit = lambda a: dc(a) >> shape(Adaptive(0.01, ClipTo(-1e9, 1e9)))          # the first sample shows the starting level estimate
    q = Sequencer(0, 1, ReplayMode.All)
    q.push(0.0, 10.0, Fade.Smooth, 0.0, 0.0, level(3) >> shape(adaptive(3, 6)))  # held through the whole test
    q.push(0.001, 0.004, Fade.Smooth, 0.0, 0.0, unit(0.25))                      # ends early: its slot is reused below
    b = GpuBank.from_sequencer(q, per_voice=False, mix=True, sample_rate=SR)
    u = OracleUnit(q.node()); u.set_sample_rate(SR)
    be = OracleBackend()
    n1 = 64 * 10
    assert _close(b.render_samples(n1)[1], u.process_many(n1))
    t0 = b.time() + 0.001                                                        # a class the bank does not have: the bank grows
    grown = b.push_event(event(dc(0.5) >> shape(Adaptive(0.02, Atan(2.0))), t0, t0 + 0.01, Fade.Smooth, 0.0, 0.0))
    assert grown == 2 and b.voices() == 3
    L.fo_sequencer_push(u.h, t0, t0 + 0.01, 1, 0.0, 0.0, (dc(0.5) >> shape(Adaptive(0.02, Atan(2.0)))).lower(be))
    t1 = b.time() + 0.002                                                        # the finished event's class: its slot is taken
    assert b.push_event(event(unit(0.5), t1, t1 + 0.01, Fade.Smooth, 0.0, 0.0)) == 1
    L.fo_sequencer_push(u.h, t1, t1 + 0.01, 1, 0.0, 0.0, unit(0.5).lower(be))
    n2 = 64 * 20 + 9
    g2, o2 = b.render_samples(n2)[1], u.process_many(n2)
    assert np.abs(o2).max() > 1.0 and _close(g2, o2), float(np.abs(g2 - o2).max())


def test_adaptive_in_a_bank_made_from_a_net():
    """A Net hands its units the f32-rounded rate (fdsp_bank_create_from_net), and Shaper<Adaptive> computes its smoothing from it."""
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.net import voice_net
    olib().fo_set_denormal_emulation(0)
    sr = 48000.1                                                                 # not an f32 value: the unit rate is float32(sr)
    # (fixed phases: a Net pings its units, so hashed initial phases would differ from those of a unit built alone)
    mk = lambda i: ((saw_hz(55.0 + i).phase(0.0) * dc(0.02 + 3.0 * fv(i, 1))) + (sine_hz(0.7).phase(0.25) * dc(0.5))) >> shape(adaptive(i, 6 if i % 2 else 3))
    b = GpuBank.from_net(voice_net([mk(i) for i in range(V)]), per_voice=True, mix=True, sample_rate=sr)
    rows, _ = b.render_samples(N)
    for i in range(V):
        u = OracleUnit(mk(i)); u.set_sample_rate(float(np.float32(sr)))
        want = u.process_many(N)
        assert np.array_equal(rows[i], want), (i, int((rows[i] != want).sum()))


def test_adaptive_events_of_a_looping_sequencer_reset_from_the_reset_image():
    """ReplayMode::Loop at 48 kHz: an event that ends is reset on the device from its class's reset image, so every period after the
    first starts its Adaptive level estimate at 1e-3 (the first period of an event pushed before the rate was set starts at 0.0: a
    looping sequencer's re-rate shifts its events and does not reset them)."""
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.sequencer import Sequencer, Fade, ReplayMode
    olib().fo_set_denormal_emulation(0)
    T = 600 / SR

    def seq():
        q = Sequencer(0, 1, ReplayMode.Loop(T))
        q.push(0.0, 0.4 * T, Fade.Smooth, 0.0, 0.05 * T, dc(0.5) >> shape(Adaptive(0.01, ClipTo(-1e9, 1e9))))
        q.push(0.1 * T, 0.6 * T, Fade.Smooth, 0.05 * T, 0.1 * T, level(1) >> shape(adaptive(1, 6)))
        q.push(0.3 * T, 0.9 * T, Fade.Power, 0.02 * T, 0.03 * T, noise().seed(3) >> dlowpass_hz(adaptive(2, 2), 800.0, 2.0))
        return q
    n = int(3.3 * 600)
    rows, _ = GpuBank.from_sequencer(seq(), per_voice=True, mix=True, sample_rate=SR).render_samples(n)
    for v, ev in enumerate(seq().voices()):
        u = OracleUnit(ev); u.set_sample_rate(SR)
        want = u.process_many(n)
        assert np.abs(want).max() > 1e-3 and np.array_equal(rows[v], want), (v, int((rows[v] != want).sum()))
