"""Closures of the signal on the GPU: map, shape_fn and the input-dependent envelopes (envelope_in / envelope2 / envelope3), parsed from
their text on the host and compiled into the voice program. Every case is compared bit for bit with the oracle's own closure interpreter
(oracle/fo_closure.h), per voice, over 40 voices that differ in their captured values."""
import ctypes as C
import os

import numpy as np
import pytest

from fundsp_b200.net import Net
from fundsp_b200.prelude import *  # noqa: F401,F403
from fundsp_b200.sequencer import event
from oracle import OracleUnit, lib as olib, oracle_bank_render
import oracle_closure  # noqa: F401  (the oracle's closure nodes, registered on OracleBackend)

pytestmark = pytest.mark.gpu
SR = 48000.0
N = 17000 + 13
V = 40
P_INTERVAL = 15   # Parameter::Interval (src/setting.rs)


def fv(i, k=0):
    return ((i * 37 + k * 11) % 29) / 29.0


MAP2 = "|x: &Frame<f32, U2>| { let a = x[0] * g; let b = x[1] - a; if a > b && !(b == 0.0) { (a, tanh(b * 2.0)) } else { (b * 0.5, a.max(b).clamp(-0.5, 0.75)) } }"
SHAPE = "|x| softsign(x * h) + 0.25 * smooth5(clamp01(x)) - 0.1 * x.abs().sqrt()"
CUTOFF = "|t, x| 900.0 + 700.0 * x * depth + 100.0 * sqr_hz(3.0, t)"
ENV3 = "|t, x, y| (x * y + t, lerp(-1.0, 1.0, clamp01(y)))"
ENV_IN = "|t, i| i[0] * 0.5 + i[1] * i[2] + sin_hz(2.0, t) * k"
NET_MAP = "|x| (x[0] * w + x[1] * (1.0 - w), x[0] - x[1])"

CASES = {
    "map_tuple_let_if": lambda i: (noise().seed(i) | sine_hz(110.0 + i)) >> map_(MAP2, 2, 2, g=0.5 + 0.5 * fv(i)),
    "shape_fn_in_filter_chain": lambda i: noise().seed(i) >> lowpass_hz(800.0 + 10.0 * i, 1.0) >> shape_fn(SHAPE, h=1.0 + 0.1 * i) >> highpass_hz(100.0, 0.7),
    "envelope2_svf_cutoff": lambda i: (noise().seed(i) | (sine_hz(2.0 + 0.1 * (i % 5)) >> envelope2(CUTOFF, depth=fv(i, 1))) | dc(1.0)) >> lowpass(),
    "envelope3": lambda i: (sine_hz(1.0 + 0.1 * i) | dc(0.5 + 0.01 * i)) >> envelope3(ENV3, 2),
    "envelope_in_frame3": lambda i: (noise().seed(i) | sine_hz(3.0) | dc(0.2 + fv(i))) >> envelope_in(ENV_IN, 3, k=0.1 + 0.01 * i),
    "map_in_net": lambda i: ((Net.wrap(saw_hz(110.0 + i)) | Net.wrap(noise().seed(i))) >> Net.wrap(map_(NET_MAP, 2, 2, w=fv(i, 2))) >> Net.wrap(lowpass_hz(1000.0, 1.0) | pass_())).node(),
    "map_in_event": lambda i: event(saw_hz(80.0 + 3.0 * i) >> map_("|x| x[0] * x[0] * a - 0.5", 1, 1, a=1.0 + fv(i)), (30.0 + 97.3 * i) / SR, (30.0 + 97.3 * i + 5000.0) / SR, i % 2, 40.0 / SR, 300.0 / SR),
}


def _bank(mk, n_voices=V, **kw):
    from fundsp_b200.bank import GpuBank
    return GpuBank([mk(i) for i in range(n_voices)], sample_rate=SR, **kw)


@pytest.mark.parametrize("name", sorted(CASES))
def test_closure_case_matches_oracle(name):
    olib().fo_set_denormal_emulation(0)
    mk = CASES[name]
    b = _bank(mk, per_voice=True, mix=True)
    g, mx = b.render_samples(N)
    o, omx = oracle_bank_render([mk(i) for i in range(V)], SR, N, mix=True, threads=4)
    assert len(b.classes()) == 1, [c["signature"] for c in b.classes()]
    assert g.shape == o.shape and np.isfinite(g).all() and np.abs(o).max() > 1e-3
    bad = int((g != o).sum())
    assert bad == 0, (name, bad, float(np.abs(g - o).max()), b.classes()[0]["signature"])
    # the mix of bit-exact rows: the same sum up to the order of the additions
    assert np.abs(mx - omx).max() <= 2e-6 * max(1.0, float(np.abs(o).sum(axis=0).max()))


def test_ragged_process_sizes():
    olib().fo_set_denormal_emulation(0)
    mk = CASES["envelope2_svf_cutoff"]
    b = _bank(mk, per_voice=True)
    us = [OracleUnit(mk(i)) for i in range(V)]
    for u in us:
        u.set_sample_rate(SR)
    for k, sz in enumerate([64, 61, 8, 7, 1, 0, 64, 33, 64, 5, 64, 64, 17] * 8):
        got = b.process(sz)
        want = np.concatenate([u.process(sz) for u in us])
        assert np.array_equal(got, want), (k, sz, int((got != want).sum()))


def test_reset_clone_and_sample_rate_change():
    olib().fo_set_denormal_emulation(0)
    mk = CASES["envelope_in_frame3"]
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
        u = OracleUnit(mk(i)); u.set_sample_rate(SR)
        assert np.array_equal(g3[i], u.process_many(3000))
        u.set_sample_rate(44100.0)
        o4.append(u.process_many(2500))
    assert np.array_equal(g4, np.stack(o4))


def test_live_interval_setting_on_envelope_in():
    """Setting::interval on a running EnvelopeIn voice (src/envelope.rs:344-348): the next segment uses the new interval."""
    olib().fo_set_denormal_emulation(0)
    mk = lambda i: envelope2("|t, x| x * x * a + t", a=1.0 + fv(i))
    b = _bank(mk, per_voice=True)
    n1, n2 = 1000 + 7, 4000
    x = (np.sin(np.arange(n1 + n2) * 0.003) * 0.8).astype(np.float32)[None]
    g1, _ = b.render_samples(n1, x[:, :n1])
    us = [OracleUnit(mk(i)) for i in range(V)]
    o1 = []
    for u in us:
        u.set_sample_rate(SR)
        o1.append(u.process_many(n1, x[:, :n1]))
    assert np.array_equal(g1, np.stack(o1))
    for v in range(0, V, 3):
        iv = 0.0005 + 0.0001 * v
        b.set(v, P_INTERVAL, (iv,))
        us[v].L.fo_set(us[v].h, P_INTERVAL, (C.c_float * 1)(iv), 1, 0, None, 0)
    g2, _ = b.render_samples(n2, x[:, n1:])
    o2 = np.stack([u.process_many(n2, x[:, n1:]) for u in us])
    assert np.array_equal(g2, o2), int((g2 != o2).sum())
    assert not np.array_equal(g2[0], g2[1])


def test_sixteen_thousand_voices_one_class():
    """16 384 voices of one closure text with per-voice captures: one class, the launches of the equivalent built-in bank, and a fixed
    sample of voices equal to the oracle."""
    if "mock" in os.environ.get("FDSP_B200_LIB", ""):
        pytest.skip("a full-size bank is for the GPU (the CPU mock device walks every voice serially)")
    olib().fo_set_denormal_emulation(0)
    n_voices, n = 16384, 4800
    mk = lambda i: saw_hz(50.0 + 0.05 * i).phase(0.0) >> map_("|x| tanh(x[0] * drive)", 1, 1, drive=0.5 + (i % 97) / 32.0)
    ref = lambda i: saw_hz(50.0 + 0.05 * i).phase(0.0) >> shape(Tanh(0.5 + (i % 97) / 32.0))
    b = _bank(mk, n_voices, per_voice=True, mix=True)
    r = _bank(ref, n_voices, per_voice=True, mix=True)
    assert len(b.classes()) == 1
    l0, r0 = b.launch_count(), r.launch_count()
    g, mx = b.render_samples(n)
    gr, mr = r.render_samples(n)
    assert b.launch_count() - l0 == r.launch_count() - r0
    assert np.array_equal(g, gr) and np.array_equal(mx, mr)
    idx = list(range(0, n_voices, 997)) + [n_voices - 1]
    o, _ = oracle_bank_render([mk(i) for i in idx], SR, n, threads=4)
    assert np.array_equal(g[idx], o)
