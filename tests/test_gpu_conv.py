"""`x >> convolve(h)` against a float64 linear convolution of the same X rows.

A bank of one `Pipe<X, Convolver>` class with a response of FDSP_TC_MINK (32) taps or more runs the tensor-core form
(csrc/dsp/conv_tc_kernel.cuh: X rows with history columns, Toeplitz tiles of h, wgmma with a TMA ring, 3xTF32 split, register
epilogue, history move); shorter responses, FDSP_TC_CONV=0 and the CPU mock device run the direct form (`Convolver::step8`).
Neither form has a bit-exact oracle, so:
  - every voice is compared with the f64 convolution of its own X rows (the oracle's, bit-exact with the GPU's), with a per-voice
    bar: max_t |g - want| <= 1e-5 * max_t |want_v|;
  - responses and inputs whose products are exact (one-hot responses, impulse inputs, power-of-two gains) are compared bit for bit:
    the tensor-core form multiplies by x ~ xh + xl with xh = tf32(x), xl = tf32(x - xh) (same split for h), which numpy computes
    exactly, so any off-by-one in the look-back, the history columns, the window start, the Toeplitz band or the row mapping shows;
  - whenever a case is meant to run the tensor-core form, the launch count says it did (4 launches per 16 384-sample chunk plus one
    for the mix, against 1 or 2 for the direct form), so a silent fall-back to the direct form fails the test.
"""
import os

import numpy as np
import pytest
from scipy.signal import fftconvolve

from fundsp_b200.prelude import convolve, noise, pass_, sine_hz

pytestmark = pytest.mark.gpu
SR = 48000.0
CHUNK = 16384                             # TIME_CHUNK: samples per launch of a long render
N_CROSS = CHUNK + 3 * 64 + 37             # crosses the chunk boundary, ragged last 64-sample tile
MOCK = "mock" in os.environ.get("FDSP_B200_LIB", "")
MOCK_MACS = 3e9                           # the mock device runs the direct form on the CPU: bigger cases are GPU-only


def skip_slow_on_mock(macs):
    if MOCK and macs > MOCK_MACS:
        pytest.skip(f"{macs:.2g} multiply-adds in the direct form on the CPU mock device take minutes; the tensor-core form is GPU-only")


def tc_form(K):
    """Whether a one-class bank with K taps runs the tensor-core form here (bank.cpp tc_conv_wanted)."""
    return not MOCK and K >= 32 and os.environ.get("FDSP_TC_CONV", "1") != "0"


def response(K, seed=None):
    rng = np.random.default_rng(K if seed is None else seed)
    h = rng.uniform(-1, 1, K) * np.exp(-np.arange(K) / max(1.0, K / 3.0))
    return (h / np.abs(h).max()).astype(np.float32)


def tf32(a):
    """FP32 with the low 13 mantissa bits cleared (what the split kernels store)."""
    return (np.ascontiguousarray(a, np.float32).view(np.uint32) & np.uint32(0xffffe000)).view(np.float32)


def split_value(a):
    """xh + xl with xh = tf32(x), xl = tf32(x - xh): the value the tensor-core form multiplies by. The sum is exact in FP32."""
    a = np.asarray(a, np.float32)
    hi = tf32(a)
    return hi + tf32(a - hi)


def exact_value(a, K):
    return split_value(a) if tc_form(K) else np.asarray(a, np.float32)


def conv64(x, h, n):
    """f64 linear convolution of each row of x (.., n) with h, first n samples."""
    x = np.asarray(x, np.float64).reshape(-1, x.shape[-1])[:, :n]
    h = np.asarray(h, np.float64)
    if len(h) * n <= 1 << 22:
        return np.stack([np.convolve(r, h)[:n] for r in x])
    return fftconvolve(x, h[None, :], axes=1)[:, :n]


def oracle_rows(exprs, n):
    """X rows of the voices in front of the convolver, from the CPU oracle (bit-exact with the GPU's voice programs)."""
    from oracle import OracleUnit
    rows = []
    for e in exprs:
        u = OracleUnit(e)
        u.set_sample_rate(SR)
        rows.append(u.process_many(n)[0])
    return np.stack(rows)


def worst_error(g, want):
    """Worst per-voice error relative to that voice's peak; asserts every voice within 1e-5."""
    g = np.asarray(g, np.float64).reshape(want.shape)
    peak = np.abs(want).max(axis=-1)
    err = np.abs(g - want).max(axis=-1)
    assert (peak > 0).all()
    rel = err / peak
    bad = np.nonzero(rel > 1e-5)[0]
    assert len(bad) == 0, (f"{len(bad)} of {len(rel)} voices over 1e-5 of their peak", bad[:8].tolist(), rel[bad[:8]].tolist())
    return float(rel.max())


def tc_launches(lens, mix):
    """Launches the tensor-core form makes for render calls of these lengths (bank.cpp: voice program, split, wgmma tiles and history move
    per chunk, plus the voice-order fold when the bank mixes)."""
    return sum((n + CHUNK - 1) // CHUNK * (4 + (1 if mix else 0)) for n in lens if n > 0)


class Launches:
    """Asserts that the calls made inside the block ran the tensor-core form (skipped where that form does not run)."""

    def __init__(self, bank, lens, mix, K):
        self.b, self.lens, self.mix, self.K = bank, list(lens), mix, K

    def __enter__(self):
        self.l0 = self.b.launch_count()
        return self

    def __exit__(self, *exc):
        if exc[0] is None and tc_form(self.K):
            got, want = self.b.launch_count() - self.l0, tc_launches(self.lens, self.mix)
            assert got == want, f"{got} launches for calls of {self.lens} samples, the tensor-core form makes {want}: it did not run"


def noise_voice(i):
    return noise().seed(i) * (0.5 + 0.003 * (i % 97))


def bank(exprs, **kw):
    from fundsp_b200.bank import GpuBank
    kw.setdefault("per_voice", True)
    return GpuBank(exprs, sample_rate=SR, **kw)


def render_checked(b, n, K, inp=None):
    with Launches(b, [n], b.mode & 2, K):
        return b.render_samples(n, inp)


def left_fold(rows):
    acc = rows[0].copy()
    for r in rows[1:]:
        acc = acc + r
    return acc


# ---- moved from test_gpu_jit.py, now against the f64 convolution per voice as well


@pytest.mark.parametrize("K", [1, 3, 64, 1000])
def test_convolver_matches_linear_convolution(K):
    """Convolver (src/convolve.rs): the reference computes y = x * h with a partitioned FFT (fft-convolver, not vendored), so the
    bar is the tolerance of the path, 1e-5 of the output peak (the reference's own test, test_basic.rs:698-711, uses 1e-4)."""
    from oracle import lib as olib, oracle_bank_render
    olib().fo_set_denormal_emulation(0)
    rng = np.random.default_rng(K)
    h = rng.uniform(-1, 1, K) * np.exp(-np.arange(K) / max(1.0, K / 4.0))
    h = (h / np.abs(h).max()).astype(np.float32)
    V, n = 48, 3000 + 61                       # ragged: the last block has 5 tail samples through the per-sample path
    mk = lambda i: noise().seed(i) * (0.5 + 0.01 * i) >> convolve(h)
    b = bank([mk(i) for i in range(V)])
    g, _ = render_checked(b, n, K)
    o, _ = oracle_bank_render([mk(i) for i in range(V)], SR, n, None, threads=4)
    assert b.classes()[0]["voices"] == V       # one class: the impulse response is shared, class-uniform data
    peak = float(np.abs(o).max())
    assert peak > 0.1 and float(np.abs(g - o).max()) <= 1e-5 * peak, float(np.abs(g - o).max()) / peak
    worst_error(g[:, 0], conv64(oracle_rows([noise().seed(i) * (0.5 + 0.01 * i) for i in range(V)], n), h, n))
    # state carries across calls and process()-sized launches agree with the long render
    b2 = bank([mk(i) for i in range(V)])
    parts = np.concatenate([b2.render_samples(m)[0] for m in (64, 7, 1000, 61, n - 64 - 7 - 1000 - 61)], axis=-1)
    if not tc_form(K):
        assert np.array_equal(parts, g)
    else:   # tensor-core form (K >= 32): how a launch is cut into 64-sample tiles changes the order of the partial sums, not the value
        assert float(np.abs(parts - g).max()) <= 2e-6 * peak, float(np.abs(parts - g).max()) / peak


@pytest.mark.parametrize("K", [64, 257, 1000, 4096])
def test_tensor_core_convolver(K, monkeypatch):
    """`x >> convolve(h)` as Toeplitz GEMM tiles on tensor cores against the f64 linear convolution (what the reference's partitioned
    FFT computes, src/convolve.rs:9-59), every voice within 1e-5 of its own peak, for responses from one tile chunk to 4096 taps;
    partly filled voice tile, ragged last time tile, a render longer than the 16384-sample chunk (history columns), state across calls,
    reset, clone, the voice-order mix, and the direct form as a cross-check."""
    V, n = 150, CHUNK + 128 * 2 + 77
    skip_slow_on_mock(V * n * K)
    h = response(K)
    mk = lambda i: noise_voice(i) >> convolve(h)
    b = bank([mk(i) for i in range(V)], mix=True)
    g, mix = render_checked(b, n, K)
    want = conv64(oracle_rows([noise_voice(i) for i in range(V)], n), h, n)
    print(f"K = {K}: worst per-voice error {worst_error(g[:, 0], want):.3g} of the peak")
    peak = float(np.abs(want).max())
    acc = left_fold(g[:, 0])
    if MOCK:   # (the mock runs the direct form, whose mix is the CTA-level tree)
        assert np.abs(mix[0] - acc).max() <= 1e-5 * np.abs(g).sum(axis=0).max()
    else:
        assert np.array_equal(mix[0], acc)      # the mix is the left fold of the rows in voice order (the reference's index-order sum)
    # continuation / reset / clone
    b.reset()
    c = b.clone()
    p1, _ = b.render_samples(5000); p2, _ = b.render_samples(3000 + 5)
    assert float(np.abs(np.concatenate([p1, p2], axis=-1) - g[..., :8005]).max()) <= 2e-6 * peak
    q1, _ = c.render_samples(5000)
    assert np.array_equal(q1, p1)
    # the direct form (FP32 pipe) on the same voices
    if not MOCK:
        monkeypatch.setenv("FDSP_TC_CONV", "0")
        d, _ = bank([mk(i) for i in range(V)], mix=True).render_samples(2000)
        assert float(np.abs(d - g[..., :2000]).max()) <= 1e-5 * peak
        worst_error(d[:, 0], want[:, :2000])


# ---- 1. exact structure: products that are exact in the 3xTF32 split


def shared_input(n, seed=5):
    return np.random.default_rng(seed).uniform(-1.0, 1.0, (1, n)).astype(np.float32)


def gain_exponents(V):
    return [(v * 7) % 81 - 40 for v in range(V)]     # 2^-40 .. 2^40, every exponent once in 81 voices


@pytest.mark.parametrize("K,d", [(K, d) for K in (32, 33, 35, 100, 1000) for d in sorted({0, 1, 3, 4, 31, 32, K - 1}) if d < K])
def test_one_hot_response_delays_the_input(K, d):
    """h = e_d: every voice's output is its input delayed by d samples, bit for bit (in the tensor-core form, the input as xh + xl)."""
    V, n = (130 if not MOCK else 3), N_CROSS
    h = np.zeros(K, np.float32); h[d] = 1.0
    es = gain_exponents(V)
    b = bank([pass_() * float(2.0 ** e) >> convolve(h) for e in es])
    x = shared_input(n)
    g, _ = render_checked(b, n, K, x)
    xe = exact_value(x[0], K)
    want = np.zeros(n, np.float32); want[d:] = xe[: n - d]
    for v, e in enumerate(es):
        bad = np.nonzero(g[v, 0] != want * np.float32(2.0 ** e))[0]
        assert len(bad) == 0, (v, e, len(bad), bad[:8].tolist())


@pytest.mark.parametrize("K", [33, 1000])
def test_impulse_input_reproduces_the_response(K):
    """An impulse at t reproduces h at t (in the tensor-core form, hh + hl), also when the response straddles the 16384-sample chunk and
    the history move (t = 16383, 16389); between the impulses the bank is reset, so the history columns must be cleared."""
    V = 130 if not MOCK else 3
    h = response(K)
    es = gain_exponents(V)
    b = bank([pass_() * float(2.0 ** e) >> convolve(h) for e in es])
    he = exact_value(h, K)
    for t in (0, 63, 64, 16383, 16389):
        n = t + K + 70
        x = np.zeros((1, n), np.float32); x[0, t] = 1.0
        b.reset()
        g, _ = render_checked(b, n, K, x)
        want = np.zeros(n, np.float32); want[t: t + K] = he
        for v, e in enumerate(es):
            bad = np.nonzero(g[v, 0] != want * np.float32(2.0 ** e))[0]
            assert len(bad) == 0, (t, v, e, len(bad), bad[:8].tolist())


@pytest.mark.parametrize("K", [100, 1000])
def test_power_of_two_gains_scale_exactly(K):
    """The same input at gains 2^e, e in [-40, 40]: rows exactly 2^e times the e = 0 row (any rounding or row mix-up breaks this),
    and each within 1e-5 of its f64 convolution."""
    V, n = 81, N_CROSS
    skip_slow_on_mock(V * n * K)
    h = response(K)
    es = gain_exponents(V)
    b = bank([pass_() * float(2.0 ** e) >> convolve(h) for e in es])
    x = shared_input(n, seed=K)
    g, _ = render_checked(b, n, K, x)
    ref = g[es.index(0), 0]
    for v, e in enumerate(es):
        assert np.array_equal(g[v, 0], ref * np.float32(2.0 ** e)), (v, e)
    worst_error(g[:, 0], conv64(x, h, n) * np.array([2.0 ** e for e in es])[:, None])


# ---- 2. shape sweep against f64


def sweep(V, K):
    skip_slow_on_mock(V * N_CROSS * K)
    h = response(K)
    b = bank([noise_voice(i) >> convolve(h) for i in range(V)])
    g, _ = render_checked(b, N_CROSS, K)
    err = worst_error(g[:, 0], conv64(oracle_rows([noise_voice(i) for i in range(V)], N_CROSS), h, N_CROSS))
    print(f"K = {K}, V = {V}: worst per-voice error {err:.3g} of the peak")


@pytest.mark.parametrize("K", [32, 33, 35, 63, 64, 66, 97, 98, 129, 257, 1000, 4096])
def test_sweep_taps(K):
    """3, 4, 5 and 6 contraction chunks (fewer than, as many as and more than the 4 ring stages), the first wraps of the ring parity,
    K - 1 divisible and not divisible by 4, up to 4096 taps; 129 voices (a second voice tile with one voice)."""
    sweep(129, K)


@pytest.mark.parametrize("K", [66, 1000])
@pytest.mark.parametrize("V", [1, 63, 64, 65, 127, 128, 129, 200])
def test_sweep_voices(V, K):
    """Voice tiles of 128 rows in two warpgroups of 64: an empty second warpgroup, a partial one, a second tile."""
    sweep(V, K)


# ---- 3. call patterns, against the f64 convolution of the whole stream


@pytest.mark.parametrize("K", [100, 1000])
def test_render_call_sizes(K):
    """Calls shorter than one 64-sample tile, than the history (H = 1024 at K = 1000: the history move overlaps itself), one chunk
    exactly and one chunk plus one; odd and even lengths give odd and even row strides (scalar and float2 stores)."""
    sizes = [1, 7, 63, 64, 65, 1000, 16383, 16384, 16385]
    V, n = 130, sum(sizes)
    skip_slow_on_mock(V * n * K)
    h = response(K)
    b = bank([noise_voice(i) >> convolve(h) for i in range(V)])
    parts = []
    for m in sizes:
        parts.append(render_checked(b, m, K)[0])
        assert parts[-1].shape == (V, 1, m)
    g = np.concatenate(parts, axis=-1)
    worst_error(g[:, 0], conv64(oracle_rows([noise_voice(i) for i in range(V)], n), h, n))


def test_process_sizes():
    """AudioUnit::process blocks of 64, 61, 8, 7, 1, 0 and 33 samples, eight times over, with K = 1000: every launch is shorter than the
    1024 history columns, so the history move's source and destination overlap."""
    K, V = 1000, 130
    sizes = [64, 61, 8, 7, 1, 0, 33] * 8
    n = sum(sizes)
    h = response(K)
    b = bank([noise_voice(i) >> convolve(h) for i in range(V)])
    parts = []
    for m in sizes:
        with Launches(b, [m], False, K):
            parts.append(b.process(m))
        assert parts[-1].shape == (V, m)
    g = np.concatenate(parts, axis=-1)
    worst_error(g, conv64(oracle_rows([noise_voice(i) for i in range(V)], n), h, n))


@pytest.mark.parametrize("n", [N_CROSS, N_CROSS + 1])
def test_output_modes(n):
    """Rows only, rows and mix, mix only (rows in an internal buffer): the same rows, and the same mix bit for bit — the voice-order
    left fold of the rows. Odd and even n: odd and even row strides."""
    K, V = 257, 130
    h = response(K)
    mk = lambda: [noise_voice(i) >> convolve(h) for i in range(V)]
    rows, _ = render_checked(bank(mk()), n, K)
    rows2, mix2 = render_checked(bank(mk(), mix=True), n, K)
    _, mix3 = render_checked(bank(mk(), per_voice=False, mix=True), n, K)
    assert np.array_equal(rows, rows2)
    worst_error(rows[:, 0], conv64(oracle_rows([noise_voice(i) for i in range(V)], n), h, n))
    if MOCK:   # (the mock runs the direct form, whose mix is the CTA-level tree)
        assert np.abs(mix2 - mix3).max() <= 1e-6 * np.abs(rows).sum(axis=0).max()
    else:
        assert np.array_equal(mix3, mix2)
        assert np.array_equal(mix3[0], left_fold(rows[:, 0]))


# ---- 4. long responses


@pytest.mark.parametrize("K", [12290, 16384, 48000])
def test_long_responses(K, monkeypatch):
    """Responses past 12 289 taps (history columns beyond 48 KB per row) up to a one-second impulse response at 48 kHz; the direct
    form at 12 290 taps as a cross-check."""
    V, n = 130, CHUNK + 1000
    skip_slow_on_mock(V * n * K)
    h = response(K)
    b = bank([noise_voice(i) >> convolve(h) for i in range(V)])
    g, _ = render_checked(b, n, K)
    x = oracle_rows([noise_voice(i) for i in range(V)], n)
    want = conv64(x, h, n)
    print(f"K = {K}: worst per-voice error {worst_error(g[:, 0], want):.3g} of the peak")
    if K == 12290:
        monkeypatch.setenv("FDSP_TC_CONV", "0")
        d = bank([noise_voice(i) >> convolve(h) for i in range(V)])
        l0 = d.launch_count()
        dg, _ = d.render_samples(2000)
        assert d.launch_count() - l0 == 1       # one voice-program launch: the direct form
        worst_error(dg[:, 0], want[:, :2000])


# ---- 5. banks past 65 535 voices


def test_more_voices_than_grid_y():
    """65 666 voices: more than gridDim.y can count. A strided sample of voices and the last 130 against f64, the mix against the fold."""
    if MOCK:
        pytest.skip("65 666 voices through the direct form on the CPU mock device takes minutes; this is about launch shapes on the GPU")
    K, V, n = 32, 65536 + 130, 256
    h = response(K)
    b = bank([noise_voice(i) >> convolve(h) for i in range(V)], mix=True)
    g, mix = render_checked(b, n, K)
    pick = list(range(0, V - 130, 509)) + list(range(V - 130, V))
    worst_error(g[pick, 0], conv64(oracle_rows([noise_voice(i) for i in pick], n), h, n))
    assert np.array_equal(mix[0], left_fold(g[:, 0]))


# ---- 6. reset, clone, sample rate, growth


def test_reset_clone_and_sample_rate():
    K, V, n = 1000, 130, 20000
    h = response(K)
    mk = lambda: [noise_voice(i) >> convolve(h) for i in range(V)]
    want = conv64(oracle_rows([noise_voice(i) for i in range(V)], 2 * n), h, 2 * n)
    b = bank(mk(), mix=True)
    g, mix = render_checked(b, n, K)
    b.reset()                                  # history columns cleared: the same output as a fresh bank, bit for bit
    g2, mix2 = render_checked(b, n, K)
    assert np.array_equal(g2, g) and np.array_equal(mix2, mix)
    c = b.clone()                              # a clone continues exactly like the original
    p, _ = render_checked(b, 7001, K)
    q, _ = render_checked(c, 7001, K)
    assert np.array_equal(p, q)
    worst_error(np.concatenate([g2, p], axis=-1)[:, 0], want[:, : n + 7001])
    # a new sample rate mid-stream: the response does not depend on it and the history is kept
    s = bank(mk())
    a1, _ = render_checked(s, n, K)
    s.set_sample_rate(44100.0)
    a2, _ = render_checked(s, n, K)
    worst_error(np.concatenate([a1, a2], axis=-1)[:, 0], want)


def test_growth_is_refused():
    """The tensor-core class keeps its X rows in a two-stage layout: add_voice / replace_voice are refused, the bank is rebuilt instead."""
    if MOCK:
        pytest.skip("the mock device runs the direct form, which can grow")
    from fundsp_b200.capi import ERR_UNSUPPORTED, FdspError
    h = response(64)
    b = bank([noise_voice(i) >> convolve(h) for i in range(8)])
    for op in (lambda: b.add_voice(noise_voice(99) >> convolve(h)), lambda: b.replace_voice(3, sine_hz(440.0))):
        with pytest.raises(FdspError) as e:
            op()
        assert e.value.code == ERR_UNSUPPORTED
    g, _ = render_checked(b, 3000, 64)           # the bank is unchanged and still renders
    worst_error(g[:, 0], conv64(oracle_rows([noise_voice(i) for i in range(8)], 3000), h, 3000))


# ---- 7. direct form at the ring-length edge


@pytest.mark.parametrize("K", [24, 25, 56, 57])
def test_direct_form_ring_edge(K, monkeypatch):
    """Convolver::step8 looks K + 7 samples back in a power-of-two ring of at least K + 8: K = 24 / 56 fill a 32 / 64 ring exactly."""
    monkeypatch.setenv("FDSP_TC_CONV", "0")
    V, n = 48, 3000 + 61
    h = response(K)
    b = bank([noise_voice(i) >> convolve(h) for i in range(V)])
    l0 = b.launch_count()
    g, _ = b.render_samples(n)
    if not MOCK:
        assert b.launch_count() - l0 == 1       # one voice-program launch: the direct form
    worst_error(g[:, 0], conv64(oracle_rows([noise_voice(i) for i in range(V)], n), h, n))


# ---- 8. two devices in one process


def test_two_devices_in_one_process():
    """Kernel attributes (the tensor-core form's and the FDN kernel's shared memory) belong to each device: the same banks on device 0
    and device 1 of one process give the same output."""
    if MOCK:
        pytest.skip("needs 2 GPUs, the mock device is one")
    import torch
    ndev = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if ndev < 2:
        pytest.skip(f"needs 2 GPUs, this machine has {ndev}")
    from fundsp_b200 import workloads
    K, V, n = 1000, 130, 5000
    h = response(K)
    outs = []
    for dev in (0, 1):
        b = bank([noise_voice(i) >> convolve(h) for i in range(V)], device=dev)
        g, _ = render_checked(b, n, K)
        f = bank(workloads.build("subtractive", 64), device=dev)
        r, _ = f.render_samples(1280, workloads.gate_signal(1280))
        outs.append((g, r))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
    worst_error(outs[1][0][:, 0], conv64(oracle_rows([noise_voice(i) for i in range(V)], n), h, n))
