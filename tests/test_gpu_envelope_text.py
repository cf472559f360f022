"""Text envelopes on the GPU: `envelope` / `lfo` whose closure `|t| ...` of time is compiled into the voice program (EnvelopeFn) and
evaluated at the reference's sample points, with no horizon. Every case is compared bit for bit with the oracle's Envelope<f32>, which
calls its closure live, here the text run by the oracle's closure interpreter (oracle/fo_closure.h), per voice, over 40 voices that
differ in their captured values; within the callback form's horizon, with the callback form running the same text through the same
interpreter."""
import ctypes as C
import math
import os
import weakref

import numpy as np
import pytest

from fundsp_b200.graph import f32
from fundsp_b200.net import Net
from fundsp_b200.prelude import *  # noqa: F401,F403
from fundsp_b200.sequencer import event, slot
from oracle import OracleBackend, OracleUnit, lib as olib, oracle_bank_render

pytestmark = pytest.mark.gpu
SR = 48000.0
N = 17000 + 13
V = 40
P_INTERVAL = 15   # Parameter::Interval (src/setting.rs)
MOCK = "mock" in os.environ.get("FDSP_B200_LIB", "")


def fv(i, k=0):
    return ((i * 37 + k * 11) % 29) / 29.0


VIBRATO = "|t| 220.0 + depth * sin_hz(rate, t)"
PAN2 = "|t: f32| { let p = tri_hz(rate, t); (sin_hz(110.0 * (1.0 + p * 0.01), t) * 0.5, clamp11(p * width)) }"
SWEEP = "move |t| if t < 0.1 { 300.0 + t * 5000.0 } else { 800.0 + 600.0 * smooth5(clamp01(sqr_hz(rate, t) * 0.5 + 0.5)) * depth }"
FLANGE = "|t| lerp11(0.004, 0.009, sin_hz(rate, t))"
PHASE = "|t| sin_hz(rate, t) * 0.5 + 0.5"
GAIN = "|t| 0.4 + 0.3 * cos_hz(rate, t)"

CASES = {
    "lfo_sine": lambda i: lfo(VIBRATO, depth=20.0 + i, rate=0.5 + fv(i)) >> sine(),
    "envelope2_pan": lambda i: envelope(PAN2, 2, rate=1.0 + 0.25 * fv(i), width=0.5 + 0.5 * fv(i, 1)) >> panner(),
    "lfo_svf_cutoff": lambda i: (noise().seed(i) | lfo(SWEEP, rate=2.0 + 0.1 * (i % 7), depth=fv(i, 2)) | dc(1.0)) >> lowpass(),
    "flanger_text": lambda i: noise().seed(i) >> flanger(0.6, 0.004, 0.009, FLANGE, rate=0.3 + fv(i)),
    "phaser_text": lambda i: (saw_hz(110.0 + 3.0 * i) >> phaser(0.5, PHASE, rate=0.2 + fv(i, 3))),
    "lfo_in_net": lambda i: ((Net.wrap(saw_hz(110.0 + i)) | Net.wrap(lfo(GAIN, rate=1.0 + fv(i)))) >> Net.wrap(pass_() * pass_())).node(),
    "lfo_in_event": lambda i: event(lfo(VIBRATO, depth=10.0, rate=1.0 + fv(i)) >> sine(), (30.0 + 97.3 * i) / SR, (30.0 + 97.3 * i + 9000.0) / SR,
                                    i % 2, 40.0 / SR, 300.0 / SR),
    "lfo_in_slot": lambda i: slot(noise().seed(i) * lfo(GAIN, rate=2.0 + fv(i))),
    "lfo_in_feedback": lambda i: noise().seed(i) >> feedback((pass_() * lfo(GAIN, rate=0.5 + fv(i)) >> lowpass_hz(1500.0, 1.0))),
    "lfo_oversampled": lambda i: saw_hz(220.0 + i) >> oversample(pass_() * lfo(GAIN, rate=3.0 + fv(i)) >> lowpass_hz(2000.0, 1.0)),
}


class ClosureOfTime:
    """A text closure `|t| ...` run by the oracle's interpreter as a callable `f(t) -> float | tuple`. The interpreter's map node of one
    input reads a bare parameter as that input, so an oracle `map` of the same text, ticked with t, evaluates the closure at t."""

    def __init__(self, text, outputs=1, **captures):
        self.L, self.nout = olib(), int(outputs)
        self.h = OracleBackend().b_map(text, 1, self.nout, tuple((str(k), f32(v)) for k, v in captures.items()))
        self._in, self._out = (C.c_float * 1)(), (C.c_float * self.nout)()
        weakref.finalize(self, self.L.fo_free, self.h)

    def __call__(self, t):
        self._in[0] = t
        self.L.fo_tick(self.h, self._in, self._out)
        return self._out[0] if self.nout == 1 else tuple(self._out)


class _TextEnvelopes:
    """The oracle backend, with a text envelope lowered as the oracle's Envelope<f32> whose live closure is the text (ClosureOfTime)."""

    def __init__(self, be):
        self.be = be

    def __getattr__(self, name):
        return getattr(self.be, name)

    def b_envelope_text(self, interval, text, nout, caps):
        return self.be.b_envelope(interval, nout, 0, ClosureOfTime(text, nout, **dict(caps)), math.inf)

    def b_netnode(self, net): return net.lower(self)
    def b_seqnode(self, seq): return seq.lower(self)


class oracle_of:
    """`expr` as the oracle builds it: OracleUnit and oracle_bank_render take it in place of the expression."""

    def __init__(self, expr):
        self.expr = expr

    def lower(self, be):
        return self.expr.lower(_TextEnvelopes(be))


def _bank(mk, n_voices=V, **kw):
    from fundsp_b200.bank import GpuBank
    return GpuBank([mk(i) for i in range(n_voices)], sample_rate=SR, **kw)


@pytest.mark.parametrize("name", sorted(CASES))
def test_text_envelope_case_matches_oracle(name):
    olib().fo_set_denormal_emulation(0)
    mk = CASES[name]
    b = _bank(mk, per_voice=True, mix=True)
    g, mx = b.render_samples(N)
    o, omx = oracle_bank_render([oracle_of(mk(i)) for i in range(V)], SR, N, mix=True, threads=4)
    assert len(b.classes()) == 1, [c["signature"] for c in b.classes()]
    assert "EnvelopeFn<" in b.classes()[0]["signature"]
    assert g.shape == o.shape and np.isfinite(g).all() and np.abs(o).max() > 1e-3
    bad = int((g != o).sum())
    assert bad == 0, (name, bad, float(np.abs(g - o).max()), b.classes()[0]["signature"])
    assert np.abs(mx - omx).max() <= 2e-6 * max(1.0, float(np.abs(o).sum(axis=0).max()))


def test_ragged_process_sizes():
    olib().fo_set_denormal_emulation(0)
    mk = CASES["lfo_svf_cutoff"]
    b = _bank(mk, per_voice=True)
    us = [OracleUnit(oracle_of(mk(i))) for i in range(V)]
    for u in us:
        u.set_sample_rate(SR)
    for k, sz in enumerate([64, 61, 8, 7, 1, 0, 64, 33, 64, 5, 64, 64, 17, 2, 63] * 8):
        got = b.process(sz)
        want = np.concatenate([u.process(sz) for u in us])
        assert np.array_equal(got, want), (k, sz, int((got != want).sum()))


def test_reset_clone_and_sample_rate_change():
    olib().fo_set_denormal_emulation(0)
    mk = CASES["envelope2_pan"]
    b = _bank(mk, per_voice=True)
    g1, _ = b.render_samples(3000)
    c = b.clone()
    g2, _ = b.render_samples(2000)
    gc, _ = c.render_samples(2000)
    assert np.array_equal(g2, gc)
    b.reset()
    g3, _ = b.render_samples(3000)
    assert np.array_equal(g1, g3)
    b.set_sample_rate(44100.0)                      # mid-stream: the running state continues at the new rate
    g4, _ = b.render_samples(2500)
    o4 = []
    for i in range(V):
        u = OracleUnit(oracle_of(mk(i))); u.set_sample_rate(SR)
        assert np.array_equal(g3[i], u.process_many(3000))
        u.set_sample_rate(44100.0)
        o4.append(u.process_many(2500))
    assert np.array_equal(g4, np.stack(o4))


def test_live_interval_setting():
    """Setting::interval on a running Envelope voice (src/envelope.rs:165-170): the next segment uses the new interval."""
    olib().fo_set_denormal_emulation(0)
    mk = lambda i: lfo("|t| t * a + 0.25", a=1.0 + fv(i))
    b = _bank(mk, per_voice=True)
    n1, n2 = 1000 + 7, 4000
    g1, _ = b.render_samples(n1)
    us = [OracleUnit(oracle_of(mk(i))) for i in range(V)]
    o1 = []
    for u in us:
        u.set_sample_rate(SR)
        o1.append(u.process_many(n1))
    assert np.array_equal(g1, np.stack(o1))
    for v in range(0, V, 3):
        iv = 0.0005 + 0.0001 * v
        b.set(v, P_INTERVAL, (iv,))
        us[v].L.fo_set(us[v].h, P_INTERVAL, (C.c_float * 1)(iv), 1, 0, None, 0)
    g2, _ = b.render_samples(n2)
    o2 = np.stack([u.process_many(n2) for u in us])
    assert np.array_equal(g2, o2), int((g2 != o2).sum())
    assert not np.array_equal(np.diff(g2[0]), np.diff(g2[1]))


def test_thirty_seconds_past_the_callback_horizon():
    """A 30 s render: the text form keeps evaluating its closure (equal to the oracle to the last sample), while the callback form with
    its default 10 s horizon holds its last value from then on."""
    if MOCK:
        pytest.skip("a 30 s render is for the GPU (the CPU mock device walks every voice serially)")
    olib().fo_set_denormal_emulation(0)
    nv, n = 8, int(30.0 * SR)
    text = lambda i: lfo("|t| sin_hz(rate, t) * 0.5", rate=0.25 + 0.1 * i)
    g, _ = _bank(text, nv, per_voice=True).render_samples(n)
    o, _ = oracle_bank_render([oracle_of(text(i)) for i in range(nv)], SR, n, threads=4)
    assert np.array_equal(g, o), int((g != o).sum())
    tail = g[:, 0, int(20.0 * SR):]
    assert (tail.max(axis=1) - tail.min(axis=1)).min() > 0.5           # still swinging 20 s in
    fns = [ClosureOfTime("|t| sin_hz(rate, t) * 0.5", rate=0.25 + 0.1 * i) for i in range(nv)]
    cb, _ = _bank(lambda i: lfo(fns[i]), nv, per_voice=True).render_samples(n)
    late = cb[:, 0, int(10.1 * SR):]
    assert (late.max(axis=1) - late.min(axis=1)).max() < 1e-5         # past the horizon the callback form is flat
    h = int(9.9 * SR)
    assert np.array_equal(cb[:, :, :h], g[:, :, :h])


def test_text_form_equals_callback_form_within_the_horizon():
    """Both forms sample at the same points (the same ID 14 hash) and interpolate alike; the callback runs the same text through the
    oracle's interpreter, so within the horizon the rows are the same bits."""
    olib().fo_set_denormal_emulation(0)
    n = 24000 + 17
    texts = [(VIBRATO, 1, dict(depth=20.0, rate=0.7)), (PAN2, 2, dict(rate=1.5, width=0.8)), (SWEEP, 1, dict(rate=2.0, depth=0.6))]
    for text, nout, caps in texts:
        mk = lambda i: envelope(text, nout, **{k: v + 0.01 * i for k, v in caps.items()})
        fns = [ClosureOfTime(text, nout, **{k: v + 0.01 * i for k, v in caps.items()}) for i in range(V)]
        g, _ = _bank(mk, per_voice=True).render_samples(n)
        cb, _ = _bank(lambda i: envelope(fns[i], nout, horizon=1.0), per_voice=True).render_samples(n)
        assert np.abs(g).max() > 1e-3 and np.array_equal(g, cb), (text, int((g != cb).sum()))


def test_sixteen_thousand_voices_one_class_mix_model():
    """16 384 voices of one text with per-voice captures: one class, rows equal to the oracle, and a mix equal to the summation-order
    model of the bank's launches applied to the oracle's rows."""
    if MOCK:
        pytest.skip("a full-size bank is for the GPU (the CPU mock device walks every voice serially)")
    from test_gpu_mix import render_and_check
    n_voices, n = 16384, 4800
    mk = lambda i: lfo("|t| 200.0 + 50.0 * sin_hz(rate, t) + 0.01 * x", rate=0.5 + (i % 61) / 16.0, x=float(i % 1000)) >> sine()
    _, _, classes, _, _ = render_and_check([mk(i) for i in range(n_voices)], n, mix_only_too=False, oracle=True,
                                           voices_again=lambda: [oracle_of(mk(i)) for i in range(n_voices)], what="text lfo >> sine")
    assert len(classes) == 1
