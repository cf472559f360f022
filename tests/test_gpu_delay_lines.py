"""The delay-line nodes on the device — Tap, TapLinear, Delay, FeedbackUnit — bit for bit against the oracle AND within the bounds of
the f64 models of tests/delay_model.py (written from the reference's source), where the device's layout and launch structure can go
wrong: voice counts on both sides of the stage-pipelined kernel's limit and where bank_grid changes shape, delay lines on both sides of
a stage cut in every kernel form, renders across the time chunk, ragged process() sequences through the resident kernel and one launch
per block, reset, clone, rate changes that change ring lengths, and a delay-line store above 4 GiB. Every voice reads the bank's shared
inputs (x, d) and scales its delay input by its own factor, so a layout or offset error moves one voice's output onto another's.
Runs on the CPU mock device too (tests/test_delay_lines_cpu.py), except the store above 4 GiB."""
import functools
import os

import numpy as np
import pytest

import delay_model as M
from fundsp_b200.prelude import dc, delay, feedback_unit, fir, moog_hz, pass_, tap, tap_linear
from oracle import OracleUnit, lib as olib, oracle_bank_render

pytestmark = pytest.mark.gpu
F32 = np.float32
SR = 48000.0
MOCK = "mock" in os.environ.get("FDSP_B200_LIB", "")
LO, HI = 0.0005, 0.01            # Tap ring: ceil(480) + 11 -> 512 at 48 kHz, 1024 at 96 kHz, 256 at 22.05 kHz
T_DELAY, T_FB = 0.0013, 0.0011   # Delay: 62 / 125 / 29 samples; FeedbackUnit S: 53 / 106 / 24
W = (0.5, 0.3, -0.2)


@functools.lru_cache(None)
def sms():
    from test_gpu_mix import sms as s
    return s()


def scale(i):
    """Per-voice factor on the delay input, different for every voice (a golden-ratio sequence in [0.5, 1.25): over 15 000 voices the
    closest two are still ~1e-5 apart, far above an f32 ulp). d * scale rounds to f32 the same way in numpy as on the device."""
    return float(F32(0.5 + 0.75 * ((i * 0.6180339887498949) % 1.0)))


def inputs(n, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1.0, 1.0, n).astype(F32)
    k = np.arange(n)
    d = (0.5 * (LO + HI) / 0.8 + 0.45 * (HI - LO) / 0.8 * np.sin(k * (2 * np.pi / 1500.0))).astype(F32)   # times scale(i) <= 1.3: past HI
    d[k % 997 < 16] = np.float32(np.nan)
    d[k % 1301 < 16] = F32(0.0)
    return np.vstack([x, d])


def vdelays(d, i):
    return (d * F32(scale(i))).astype(F32)


def tap_cut(i):
    """tap, then a Moog (the heavy leaf: the stage-pipelined kernel cuts the spine there; the tap rides beside it as a pass-through
    channel), then a Delay behind the cut. Outputs: the Moog, the delayed Moog, the tap."""
    return (pass_() | pass_() * dc(scale(i))) >> tap(LO, HI) >> (pass_() ^ pass_()) >> ((moog_hz(900.0 + 7.0 * i, 0.3) >> (pass_() ^ delay(T_DELAY))) | pass_())


def moog_fb(i):
    """The same with a linear tap and a FeedbackUnit behind the Moog. Outputs: the Moog, the FeedbackUnit, the tap."""
    return (pass_() | pass_() * dc(scale(i))) >> tap_linear(LO, HI) >> (pass_() ^ pass_()) >> ((moog_hz(700.0 + 5.0 * i, 0.2) >> (pass_() ^ feedback_unit(T_FB, pass_() * 0.6 >> fir(W)))) | pass_())


def lines(i):   # no Moog: every node resets with the rate (src/delay.rs, src/feedback.rs set_sample_rate). Outputs: tap, Delay(tap), FeedbackUnit(tap)
    return (pass_() | pass_() * dc(scale(i))) >> tap(LO, HI) >> (pass_() ^ delay(T_DELAY) ^ feedback_unit(T_FB, pass_() * 0.6 >> fir(W)))


def bank(mk, V, sr=SR, **kw):
    from fundsp_b200.bank import GpuBank
    olib().fo_set_denormal_emulation(0)
    return GpuBank([mk(i) for i in range(V)], sample_rate=sr, **kw)


def sampled(V):
    return sorted(set([0, 1, V // 2, V - 2, V - 1] + list(range(3, V, max(1, V // 24))))) if V > 1 else [0]


def check_models(mk, rows, inp, voices, sr=SR):
    """rows [V][3][n] of tap_cut / moog_fb / lines voices against the models: the tap row against the Tap model, and the Delay /
    FeedbackUnit rows against their models applied to the row that feeds them (the Moog, or the tap for `lines`). Returns the worst
    error over the bound."""
    x, d = inp
    tap_row, src_row = (0, 0) if mk is lines else (2, 0)
    delay_row = {tap_cut: 1, lines: 1}.get(mk)
    fb_row = {moog_fb: 1, lines: 2}.get(mk)
    worst = 0.0
    for v in voices:
        want, bound = M.tap(x, vdelays(d, v), LO, HI, sr, linear=mk is moog_fb)
        worst = max(worst, ratio(rows[v][tap_row], want, bound, (mk.__name__, v, "tap")))
        src = rows[v][src_row]
        if delay_row is not None:
            assert np.array_equal(rows[v][delay_row], M.delay(src, T_DELAY, sr)[0].astype(F32)), (mk.__name__, v, "delay")
        if fb_row is not None:
            want, bound = M.feedback_unit(src[None], T_FB, sr, (0.6,), W)
            worst = max(worst, ratio(rows[v][fb_row], want[0], bound[0], (mk.__name__, v, "feedback_unit")))
    return worst


def ratio(got, want, bound, what):
    err = np.abs(np.asarray(got, np.float64) - want)
    r = float(np.max(err / np.maximum(bound, 1e-300)))
    assert np.isfinite(got).all() and r <= 1.0, (what, r, int(np.argmax(err / np.maximum(bound, 1e-300))))
    return r


def oracle_rows(mk, voices, n, inp, sr=SR):
    o, _ = oracle_bank_render([mk(i) for i in voices], sr, n, inp, threads=4)
    return o


# ---------------------------------------------------------------- voice counts
@pytest.mark.parametrize("V", ["1", "31", "33", "129", "sms*32", "sms*32+1"])
def test_voice_counts(V):
    V = {"sms*32": sms() * 32, "sms*32+1": sms() * 32 + 1}.get(V) or int(V)
    n = 64 * 30 + 37
    inp = inputs(n, V)
    b = bank(tap_cut, V, per_voice=True)
    if not MOCK:
        assert b.classes()[0]["stages"] >= 2, b.classes()
    g, _ = b.render_samples(n, inp)
    vs = sampled(V) if V > 200 else list(range(V))
    o = oracle_rows(tap_cut, vs, n, inp)
    assert np.array_equal(g[vs], o), (V, int((g[vs] != o).sum()))
    w = check_models(tap_cut, g, inp, vs[:: max(1, len(vs) // 12)] + [V - 1])
    print(f"V={V}: worst {w:.3f} of the bound")


# ---------------------------------------------------------------- stage cuts in every kernel form
@pytest.mark.parametrize("form", ["plain", "staged32", "staged128"])
@pytest.mark.parametrize("mk", [tap_cut, moog_fb], ids=["tap_moog_delay", "moog_feedback_unit"])
def test_delay_lines_on_both_sides_of_a_stage_cut(mk, form, monkeypatch):
    monkeypatch.setenv("FDSP_STAGED", "0" if form == "plain" else "1")
    if form != "plain":
        monkeypatch.setenv("FDSP_STAGED_W", form[len("staged"):])
    V, n = 300, 64 * 21 + 61
    inp = inputs(n, 7)
    b = bank(mk, V, per_voice=True)
    if not MOCK:
        assert b.classes()[0]["stages"] >= 2, b.classes()
    g, _ = b.render_samples(n, inp)
    o = oracle_rows(mk, range(V), n, inp)
    assert np.array_equal(g, o), (form, int((g != o).sum()))
    check_models(mk, g, inp, sampled(V))
    # continuation in the other form: the state words and the delay-line cursors carry over
    monkeypatch.setenv("FDSP_STAGED", "1" if form == "plain" else "0")
    inp2 = inputs(2 * n, 8)
    g2, _ = b.render_samples(n, inp2[:, n:])
    both = np.concatenate([inp[:, :n], inp2[:, n:]], axis=1)
    o2 = oracle_rows(mk, sampled(V), 2 * n, both)
    assert np.array_equal(g2[sampled(V)], o2[:, :, n:])


# ---------------------------------------------------------------- launch and call boundaries
def test_render_across_the_time_chunk():
    V, n = 70, 16384 * 2 + 64 * 3 + 5
    inp = inputs(n, 3)
    b = bank(lines, V, per_voice=True)
    g, _ = b.render_samples(n, inp)
    o = oracle_rows(lines, range(V), n, inp)
    assert np.array_equal(g, o), int((g != o).sum())
    print(f"time chunk: worst {check_models(lines, g, inp, [0, 33, V - 1]):.3f} of the bound")


SIZES = [64, 61, 8, 7, 1, 0, 64, 33, 17, 64, 2, 63, 40, 64, 64, 13, 52, 53, 54, 24, 25, 23, 64, 64]


@pytest.mark.parametrize("rt", ["1", "0"])
def test_ragged_process_reset_and_clone(rt, monkeypatch):
    """process() in ragged sizes around the FeedbackUnit's S (53), through the resident kernel and one launch per block; then a clone
    rendered alternately with its source; then reset, which must reproduce the first calls (the reference zeroes its buffers)."""
    monkeypatch.setenv("FDSP_RT", rt)
    V = 40
    n = sum(SIZES)
    inp = inputs(3 * n, 11)
    b = bank(lines, V, per_voice=True)
    us = [OracleUnit(lines(i)) for i in range(V)]
    for u in us:
        u.set_sample_rate(SR)

    def both(sizes, start, units, bk):
        g, o, p = [], [], start
        for m in sizes:
            g.append(bk.process(m, inp[:, p:p + m]).reshape(V, 3, m))
            o.append(np.stack([u.process(m, inp[:, p:p + m]) for u in units]) if m else np.zeros((V, 3, 0), F32))
            p += m
        return np.concatenate(g, axis=2), np.concatenate(o, axis=2)

    g1, o1 = both(SIZES, 0, us, b)
    assert np.array_equal(g1, o1), int((g1 != o1).sum())
    modes = [M.feedback_block_mode(m, M.feedback_samples(T_FB, SR)) for m in SIZES if m]
    assert any(modes) and not all(modes)
    check_models(lines, g1, inp[:, :n], [0, 17, V - 1])
    c = b.clone()
    a_out, c_out = [], []
    p = n
    for m in SIZES:
        a_out.append(b.process(m, inp[:, p:p + m])); c_out.append(c.process(m, inp[:, p:p + m])); p += m
    assert all(np.array_equal(x, y) for x, y in zip(a_out, c_out))
    full = np.concatenate([g1.reshape(V * 3, -1), np.concatenate(a_out, axis=1)], axis=1).reshape(V, 3, -1)
    check_models(lines, full, inp[:, :2 * n], [0, V - 1])
    b.reset()
    g3 = np.concatenate([b.process(m, inp[:, sum(SIZES[:k]):sum(SIZES[:k]) + m]) for k, m in enumerate(SIZES)], axis=1).reshape(V, 3, -1)
    assert np.array_equal(g3, g1)


# ---------------------------------------------------------------- rate changes
def test_rate_change_changes_ring_lengths():
    """A running bank changes rate: 48 kHz, then 96 kHz (Tap ring 512 -> 1024, Delay 62 -> 125 samples, S 53 -> 106), then 22.05 kHz
    (256; 29; 24). Right after each change (no reset), the Tap and Delay rows equal the oracle and their models: both zero their rings
    with the rate (src/delay.rs set_sample_rate). After a reset, every row equals the oracle and the FeedbackUnit row its model too."""
    V, n = 33, 3000
    b = bank(lines, V, per_voice=True)
    us = [OracleUnit(lines(i)) for i in range(V)]
    for u in us:
        u.set_sample_rate(SR)
    for k, sr in enumerate((48000.0, 96000.0, 22050.0)):
        inp = inputs(n, 20 + k)
        if k:
            b.set_sample_rate(sr)
            for u in us:
                u.set_sample_rate(sr)
        g, _ = b.render_samples(n, inp)
        o = np.stack([u.process_many(n, inp) for u in us])
        # rows 0 and 1 (Tap, Delay: the nodes the reference resets with the rate); the FeedbackUnit's inner Fir keeps its history in the
        # reference, while the bank rebuilds a class whose ring lengths change from its construction-time state (DESIGN §10)
        assert np.array_equal(g[:, :2], o[:, :2]), (sr, "after the rate change", int((g[:, :2] != o[:, :2]).sum()))
        for v in (0, 5, V - 1):
            want, bound = M.tap(inp[0], vdelays(inp[1], v), LO, HI, sr)
            ratio(g[v, 0], want, bound, (sr, v, "tap after the rate change"))
            assert np.array_equal(g[v, 1], M.delay(g[v, 0], T_DELAY, sr)[0].astype(F32)), (sr, v, "delay after the rate change")
        b.reset()
        for u in us:
            u.reset()
        g, _ = b.render_samples(n, inp)
        o = np.stack([u.process_many(n, inp) for u in us])
        assert np.array_equal(g, o), (sr, "after reset", int((g != o).sum()))
        print(f"{sr:.0f} Hz: worst {check_models(lines, g, inp, [0, 5, V - 1], sr=sr):.3f} of the bound")
    assert [M.tap_params(LO, HI, s, False)[3] for s in (48000.0, 96000.0, 22050.0)] == [512, 1024, 256]


# ---------------------------------------------------------------- a delay-line store above 4 GiB
def big(i):
    """Two taps around a 1.5 s Delay (72 001 floats). Each node claims its delay-line floats as the program loads (Loader::D, depth
    first), so the store per voice is [tap 512][Delay 72 001][tap 512] and the second tap's ring starts at 72 513 * V floats: past 4 GiB
    as a whole. Both taps are held to the model, so a misplaced ring of either shows. Inputs (x, d, x, x, d)."""
    return ((pass_() | pass_() * dc(scale(i))) >> tap(LO, HI)) | delay(1.5) | ((pass_() | pass_() * dc(scale(i + 20000))) >> tap(LO, HI))


@pytest.mark.skipif(MOCK, reason="the mock device keeps device memory in host memory: 9 GB with the clone")
def test_delay_line_store_above_4_gib():
    V, n = 15000, 1500
    b = bank(big, V, per_voice=True)
    (c,) = b.classes()
    assert c["delay_floats"] == 512 + 72001 + 512 and (512 + 72001) * V > 2 ** 30, c
    x, d = inputs(n, 31)
    inp = np.vstack([x, d, x, x, d])
    g, _ = b.render_samples(n, inp)
    vs = [0, 1, 4999, 7777, V - 2, V - 1]
    o = oracle_rows(big, vs, n, inp)
    assert np.array_equal(g[vs], o), int((g[vs] != o).sum())
    for v in vs:
        for k, s in ((0, v), (2, v + 20000)):
            want, bound = M.tap(x, vdelays(d, s), LO, HI, SR)
            ratio(g[v, k], want, bound, (v, k))
        assert not g[v, 1].any()   # the Delay's output starts at 72 000 samples
    c2 = b.clone()
    a1, _ = b.render_samples(n, inp)
    c1, _ = c2.render_samples(n, inp)
    assert np.array_equal(a1[vs], c1[vs]) and np.array_equal(a1[V - 1], c1[V - 1])
    del c2
    b.reset()
    g2, _ = b.render_samples(n, inp)
    assert np.array_equal(g2[vs], g[vs])


# ---------------------------------------------------------------- Oversampler
OS_SIZES = [1, 2, 63, 64, 64, 63, 2, 1, 64, 61, 8, 7, 1, 0, 64, 33, 62, 64, 63, 3, 64, 41, 64, 64]


@pytest.mark.parametrize("rt", ["1", "0"])
def test_oversample_over_process_sizes_and_a_render(rt, monkeypatch):
    """oversample(tick() * g) per voice (its 128-sample rings in the delay-line store; the tick makes the zero the odd-size rule feeds
    inward visible) through ragged process() sizes, then a render of 4 000 samples that wraps the rings many times: bit for bit with the
    oracle, and within the model's bound (tests/delay_model.py `oversample`)."""
    from fundsp_b200.prelude import oversample, tick
    monkeypatch.setenv("FDSP_RT", rt)
    V = 40
    gain = lambda i: 0.5 + i / 64.0   # noqa: E731
    mk = lambda i: oversample(tick() * gain(i))   # noqa: E731
    b = bank(mk, V, per_voice=True)
    us = [OracleUnit(mk(i)) for i in range(V)]
    for u in us:
        u.set_sample_rate(SR)
    n1, n2 = sum(OS_SIZES), 4000
    x = inputs(n1 + n2, 41)[0]
    g, o, p = [], [], 0
    for m in OS_SIZES:
        g.append(b.process(m, x[None, p:p + m]).reshape(V, 1, m))
        o.append(np.stack([u.process(m, x[None, p:p + m]) for u in us]) if m else np.zeros((V, 1, 0), F32))
        p += m
    r, _ = b.render_samples(n2, x[None, n1:])
    g = np.concatenate(g + [r], axis=2)
    o = np.concatenate(o + [np.stack([u.process_many(n2, x[None, n1:]) for u in us])], axis=2)
    assert np.array_equal(g, o), int((g != o).sum())
    sizes = OS_SIZES + [64] * (n2 // 64) + [n2 % 64]
    for v in (0, 13, V - 1):
        want, bound = M.oversample(x, sizes, gain=float(F32(gain(v))), inner_delay=1)
        ratio(g[v, 0], want, bound, (v, "oversample"))
