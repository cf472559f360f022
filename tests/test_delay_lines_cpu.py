"""The delay-line nodes of the oracle against the f64 models of tests/delay_model.py, written from the reference's source, at the
edges of their clamps, rings, process() sizes and sample rates: Delay bit for bit, Tap / TapLinear (1, 2, 3, 8 and 32 taps: the
lowering sets no upper bound on N),
FeedbackUnit and Oversampler within the bounds the models derive from their operation counts. Negative controls: every mutation of
a model (a one-sample tap offset, reversed spline taps, round for floor, S +- 1, the odd-size zero left out) misses its bound by at
least 100x. tests/test_gpu_delay_lines.py holds the device to the same models and to the oracle."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import delay_model as M
from fundsp_b200.prelude import delay, feedback_unit, fir, multitap, multitap_linear, oversample, pass_, tick
from oracle import OracleUnit, lib as olib
from test_mock_bank_cpu import ROOT, mock_env  # noqa: F401  (the mock device build, shared with that file)

F32 = np.float32
RATES = (48000.0, 44100.0, 32768.0)
WARM, SEG = 600, 16


def noise(n, seed):
    return np.random.default_rng(seed).uniform(-1.0, 1.0, n).astype(F32)


def ulps(x):
    x = F32(x)
    return [np.nextafter(x, F32(-np.inf)), x, np.nextafter(x, F32(np.inf))]


def tap_edges(mn, mx, sr):
    """Delay inputs in seconds, one per 16-sample segment: below, at and around both clamps, non-finite values, delays whose f32
    product with sr is an exact integer (and one ulp below it), and the one-sample floor."""
    s = F32(sr)
    v = [0.0, -0.0, -0.003, -np.inf, np.inf, 1e30, -1e30, np.nan, 1.0 / sr, 1.00001 / sr]
    v += ulps(mn) + ulps(mx)
    for k in (1, 2, 3, 7, 16, 31, 64, 100, 255):
        d = F32(k / sr)
        for c in (d, np.nextafter(d, F32(0)), np.nextafter(d, F32(1))):
            if F32(c * s) == math.floor(F32(c * s)):   # exactly k samples (or another integer) in f32
                v += [c, np.nextafter(c, F32(0))]
    return np.array(v, F32)


def tap_schedule(mn, mx, sr, ntaps, seed):
    """[ntaps][n] delay inputs: WARM samples at mid range, then the edge segments (tap t sees the edges rotated by t), then a sine that
    sweeps the whole range over hundreds of integer sample boundaries."""
    ev = tap_edges(mn, mx, sr)
    sweep = (0.5 * (mn + mx) + 0.5 * (mx - mn) * 1.02 * np.sin(np.arange(2400) * (2 * math.pi / 700.0))).astype(F32)
    rows = []
    for t in range(ntaps):
        e = np.roll(ev, 3 * t)
        rows.append(np.concatenate([np.full(WARM, F32(0.5 * (mn + mx))), np.repeat(e, SEG), np.roll(sweep, 91 * t)]))
    return np.array(rows, F32)


def oracle_run(expr, sr, inp, sizes=None):
    olib().fo_set_denormal_emulation(0)
    u = OracleUnit(expr)
    u.set_sample_rate(sr)
    inp = np.atleast_2d(np.asarray(inp, F32))
    if sizes is None:
        return u.process_many(inp.shape[1], inp)
    out, p = [], 0
    for m in sizes:
        out.append(u.process(m, inp[:, p:p + m]) if m else np.zeros((u.outputs(), 0), F32))
        p += m
    return np.concatenate(out, axis=1)


def within(got, want, bound, what):
    """max |got - want| / bound (bound 0 means exact); asserts <= 1 and returns the ratio."""
    err = np.abs(np.asarray(got, np.float64) - want)
    assert np.isfinite(got).all(), what
    ratio = float(np.max(np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))))
    assert ratio <= 1.0, (what, ratio, int(np.argmax(err)))
    return ratio


def misses(got, want, bound):
    err = np.abs(np.asarray(got, np.float64) - want)
    return float(np.max(err / np.maximum(bound, 1e-300)))


# ---------------------------------------------------------------- Tap / TapLinear
TAP_CONFIGS = [(0.0005, 0.01), (0.0, 0.004), (0.0, 0.0)]


def pow2_max(sr, extra, k):
    """The largest f32 max delay with ceil(max * sr) + extra == 2^k, and the next f32 up (ceil one more: the ring doubles)."""
    s = F32(sr)
    m = F32((2 ** k - extra) / sr)
    while math.ceil(F32(m * s)) + extra > 2 ** k:
        m = np.nextafter(m, F32(0))
    while math.ceil(F32(np.nextafter(m, F32(1)) * s)) + extra <= 2 ** k:
        m = np.nextafter(m, F32(1))
    up = np.nextafter(m, F32(1))
    assert math.ceil(F32(m * s)) + extra == 2 ** k and math.ceil(F32(up * s)) + extra == 2 ** k + 1
    return float(m), float(up)


def tap_cases(sr):
    out = [(mn, mx) for mn, mx in TAP_CONFIGS]
    for linear, extra in ((0, 11), (1, 2)):
        a, b = pow2_max(sr, extra, 9)
        out += [(0.0001, a), (0.0001, b)]
    return out


@pytest.mark.parametrize("sr", RATES)
@pytest.mark.parametrize("linear", [0, 1])
@pytest.mark.parametrize("ntaps", [1, 2, 3, 8, 32])
def test_tap_matches_model_at_clamp_and_ring_edges(ntaps, linear, sr):
    worst = 0.0
    for j, (mn, mx) in enumerate(tap_cases(sr)):
        d = tap_schedule(mn, mx, sr, ntaps, j)
        x = noise(d.shape[1], 10 + j)
        node = (multitap_linear if linear else multitap)(ntaps, mn, mx)
        got = oracle_run(node, sr, np.vstack([x, d]))[0]
        want, bound = M.tap(x, d, mn, mx, sr, linear=bool(linear))
        worst = max(worst, within(got, want, bound, (mn, mx)))
    print(f"tap N={ntaps} linear={linear} sr={sr:.0f}: worst {worst:.3f} of the bound")


@pytest.mark.parametrize("sr", RATES)
def test_tap_block_path_equals_tick_path_except_taplinear_reading_its_own_group(sr):
    """The reference's process() of Tap / TapLinear, stated literally (tests/delay_model.py `tap_block`, 64-sample blocks as the oracle
    and the bank render them), against its tick path (`tap`), which the oracle and the device follow. Where no lane reads a ring slot
    that a later lane of its own group overwrote, the two are the same f64 values. Tap never aliases (its ring has 3 + SIMD_N slots
    of headroom and a one-sample floor); TapLinear does in exactly the configurations with fewer than 8 spare slots: max = 0 (a ring
    of 2) and max * sr within 8 samples under ring - 2 (the power-of-two edge). There the crate's block output mixes in input samples
    up to 7 samples AHEAD of the sample it is computing; the product keeps the causal tick-path value (DESIGN §10)."""
    for linear in (False, True):
        for j, (mn, mx) in enumerate(tap_cases(sr)):
            d = tap_schedule(mn, mx, sr, 2, j)
            x = noise(d.shape[1], 10 + j)
            n = x.size
            yb, aliased = M.tap_block(x, d, mn, mx, sr, [64] * (n // 64) + [n % 64], linear=linear)
            yt, _ = M.tap(x, d, mn, mx, sr, linear=linear)
            assert np.array_equal(yb[~aliased], yt[~aliased]), (linear, mn, mx)
            ring = M.tap_params(mn, mx, sr, linear)[3]
            spare = ring - 2 - math.ceil(F32(F32(mx) * F32(sr)))
            if not linear or spare >= 8:
                assert not aliased.any(), (linear, mn, mx, ring)
            else:
                assert aliased.any() and np.abs(yb - yt)[aliased].max() > 0.1, (mn, mx, ring)


def test_tap_model_details():
    """The f32 arithmetic the model commits to: the one-sample floor, NaN at lo, the ring lengths at the power-of-two edges."""
    for sr in RATES:
        s, lo, hi, ring = M.tap_params(0.0, 0.0, sr, False)
        assert lo == hi == F32(1.00001) / F32(sr) and ring == 16
        D = M.tap_positions([np.nan, -np.inf, np.inf, 0.0], lo, hi, s)
        assert D[0] == D[1] == D[3] == F32(lo * s) and D[2] == F32(hi * s) and 1.0 < D[0] < 1.0001
        assert M.tap_params(0.0, 0.0, sr, True)[1:3] == (0.0, 0.0)
        for linear, extra in ((False, 11), (True, 2)):
            a, b = pow2_max(sr, extra, 9)
            assert M.tap_params(0.0, a, sr, linear)[3] == 512 and M.tap_params(0.0, b, sr, linear)[3] == 1024


# ---------------------------------------------------------------- Delay
def delay_times(sr):
    """t = 0; t * sr = 1, 63, 64, 65; a half-sample tie (exact in f64 at 32768 Hz: 2^-16 s is half a sample, 2.5 and 3.5 samples
    separate round from rint); one line of about 2 s."""
    ts = [0.0, 1.0 / sr, 63.0 / sr, 64.0 / sr, 65.0 / sr, 2.0 + 3.0 / sr]
    if sr == 32768.0:
        ts += [2.0 ** -16, 2.5 / 32768.0, 3.5 / 32768.0, 64.5 / 32768.0]
    else:
        ts += [2.5 / sr]
    return ts


@pytest.mark.parametrize("sr", RATES)
def test_delay_is_exact(sr):
    for t in delay_times(sr):
        L = M.delay_samples(t, sr)
        n = L + 700
        x = noise(n, L)
        got = oracle_run(delay(t), sr, x)[0]
        want, _ = M.delay(x, t, sr)
        assert np.array_equal(got, want.astype(F32)), (t, L)
    if sr == 32768.0:
        assert [M.delay_samples(t, sr) for t in (2.5 / sr, 3.5 / sr, 2.0 ** -16)] == [3, 4, 1]   # rint would give 2, 4, 0


# ---------------------------------------------------------------- FeedbackUnit
RAGGED = [64, 61, 8, 7, 1, 0, 64, 33, 17, 64, 2, 63, 40, 64, 64, 13]


def fu_sizes(S):
    out = []
    for m in (S - 1, S, S + 1):
        if 1 <= m <= 64:
            out += [m] * 6
    return out + RAGGED * 3


def fu_expr(S, sr, channels, g=(0.6, -0.45), w=(0.5, 0.3, -0.2)):
    d = S / sr
    x0 = pass_() * g[0] >> fir(w)
    return d, feedback_unit(d, x0 if channels == 1 else (x0 | pass_() * g[1]))


@pytest.mark.parametrize("sr", RATES)
@pytest.mark.parametrize("channels", [1, 2])
@pytest.mark.parametrize("S", [1, 2, 63, 64, 65, 240])
def test_feedback_unit_matches_model_in_both_modes(S, channels, sr):
    d, expr = fu_expr(S, sr, channels)
    assert M.feedback_samples(d, sr) == S
    sizes = fu_sizes(S)
    modes = [M.feedback_block_mode(m, S) for m in sizes if m]
    if S < 64:
        assert any(modes) and not all(modes)   # both paths are taken
    n = sum(sizes)
    x = np.vstack([noise(n, 3 + c) for c in range(channels)])
    got = oracle_run(expr, sr, x, sizes)
    want, bound = M.feedback_unit(x, d, sr, (0.6, -0.45), (0.5, 0.3, -0.2))
    worst = within(got, want, bound, (S, channels))
    print(f"feedback_unit S={S} ch={channels} sr={sr:.0f}: worst {worst:.3f} of the bound")


# ---------------------------------------------------------------- Oversampler
OS_SIZES = [1, 2, 63, 64, 64, 63, 2, 1, 64, 64, 61, 8, 7, 1, 0, 64, 33, 62, 64, 63, 3, 64, 64, 64, 64, 41, 64, 64, 64]


def os_exprs():
    return [(1.0, 0, oversample(pass_())), (0.75, 0, oversample(pass_() * 0.75)), (0.75, 1, oversample(tick() * 0.75))]


@pytest.mark.parametrize("sr", RATES)
def test_oversample_matches_model_over_process_sizes(sr):
    sizes = OS_SIZES * 2   # 2 x 1 594 samples: the 128-sample rings wrap many times
    n = sum(sizes)
    x = noise(n, 5)
    for g, dly, expr in os_exprs():
        got = oracle_run(expr, sr, x, sizes)[0]
        want, bound = M.oversample(x, sizes, gain=g, inner_delay=dly)
        worst = within(got, want, bound, (g, dly))
        print(f"oversample g={g} tick={dly} sr={sr:.0f}: worst {worst:.3f} of the bound")
    # renders of 65, 127, 128 and 129 samples: process() takes at most 64 (MAX_BUFFER_SIZE), so these are split into 64-sample blocks
    # and a tail, an odd one after an even one
    for n2 in (65, 127, 128, 129):
        got = oracle_run(oversample(tick() * 0.75), sr, x[:n2])[0]
        want, bound = M.oversample(x, [64] * (n2 // 64) + [n2 % 64], gain=0.75, inner_delay=1)
        within(got, want, bound, n2)


# ---------------------------------------------------------------- negative controls
def test_mutated_models_miss_their_bounds():
    sr = 48000.0
    mn, mx = 0.0005, 0.01
    d = tap_schedule(mn, mx, sr, 2, 0)
    x = noise(d.shape[1], 10)
    for linear, muts in ((False, ("offset", "reverse", "round")), (True, ("offset", "round"))):
        got = oracle_run((multitap_linear if linear else multitap)(2, mn, mx), sr, np.vstack([x, d]))[0]
        _, bound = M.tap(x, d, mn, mx, sr, linear=linear)
        for m in muts:
            want, _ = M.tap(x, d, mn, mx, sr, linear=linear, mutate=m)
            assert misses(got, want, bound) >= 100.0, (linear, m)
    t = 65.0 / sr
    x1 = noise(2000, 1)
    got = oracle_run(delay(t), sr, x1)[0]
    want, _ = M.delay(x1, t, sr, mutate="offset")
    assert np.abs(got - want).max() > 0.1
    for S in (2, 64, 65):
        dd, expr = fu_expr(S, sr, 1)
        sizes = fu_sizes(S)
        xf = noise(sum(sizes), 3)[None]
        got = oracle_run(expr, sr, xf, sizes)
        _, bound = M.feedback_unit(xf, dd, sr, (0.6,), (0.5, 0.3, -0.2))
        for ds in (-1, 1):
            if S + ds >= 1:
                want, _ = M.feedback_unit(xf, dd, sr, (0.6,), (0.5, 0.3, -0.2), mutate_s=ds)
                assert misses(got, want, bound) >= 100.0, (S, ds)
    sizes = OS_SIZES
    xo = noise(sum(sizes), 5)
    got = oracle_run(oversample(tick() * 0.75), sr, xo, sizes)[0]
    _, bound = M.oversample(xo, sizes, gain=0.75, inner_delay=1)
    for m in ("no_zero_feed", "stream"):
        want, _ = M.oversample(xo, sizes, gain=0.75, inner_delay=1, mutate=m)
        assert misses(got, want, bound) >= 100.0, m


# ---------------------------------------------------------------- the GPU file on the CPU mock device
def test_gpu_delay_lines_file_on_the_mock_device(mock_env):
    """tests/test_gpu_delay_lines.py with the host runtime on the mock device: ring lengths, offsets, resets, clones and the regrouping at
    a rate change are host code, checked here against the oracle and the models without a GPU."""
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_delay_lines.py"), "-m", "gpu", "-q", "-n", "4",
                        "-p", "no:cacheprovider", "--tb=short"], capture_output=True, text=True, env=mock_env, cwd=ROOT, timeout=1800)
    tail = r.stdout[-3000:]
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, tail
