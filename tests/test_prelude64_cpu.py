"""prelude64 without a GPU: the product's f64 libm against the oracle's restatement bit for bit and against __float128, oracle pins
(impulse responses against the reference's response() formulas, prelude32 against prelude64, tick against process, Sine<f64>'s
unrounded initial phase), signatures and word layouts, prelude64.py's refusals, NVRTC compilation of every class of
tests/test_gpu_prelude64.py for sm_90a, the device templates on the host emulation against the oracle, and the GPU file itself on the
CPU mock device."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy import signal

from fundsp_b200 import capi
from fundsp_b200 import prelude as p32
from fundsp_b200 import prelude64 as p64
from oracle import OracleUnit, lib as olib
import oracle_prelude64
from test_mock_bank_cpu import ROOT, mock_env  # noqa: F401  (the mock device build, shared with that file)

import test_gpu_prelude64 as G

F32 = np.float32


def sig(g):
    return capi.NodeHandle(g).signature()


# ---- 1. f64 libm: every 97th high word x 4 low words, and 2^24 points over the filters' domains (tan [0, pi/2), cos [0, 2 pi],
# exp [-746, 710]); `libm64_equiv 1 0` walks every high word. Accuracy against libquadmath where it can be linked.
def _build_equiv(tmp_path):
    exe = str(tmp_path / "libm64_equiv")
    src = os.path.join(ROOT, "tests", "cpp", "libm64_equiv.cpp")
    base = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-pthread", "-w"]
    if subprocess.run(base + ["-DFO_QUAD", src, "-o", exe, "-l:libquadmath.so.0"], capture_output=True).returncode == 0:
        return exe, True
    subprocess.check_call(base + [src, "-o", exe])
    return exe, False


def test_product_libm64_equals_oracle_and_quad(tmp_path):
    exe, quad = _build_equiv(tmp_path)
    r = subprocess.run([exe, "97", str(1 << 24)], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and r.stdout.count("bit-identical") == 4 and "specials: ok" in r.stdout, r.stdout
    if quad:
        ulp = {ln.split(":")[0]: float(ln.split("max ulp ")[1].split()[0]) for ln in r.stdout.splitlines() if "max ulp" in ln}
        assert len(ulp) == 4 and max(ulp.values()) <= 1.0, ulp


def test_oracle_libm64_known_values():
    L = oracle_prelude64.lib()
    xs = np.concatenate([np.linspace(-10.0, 10.0, 2001), np.geomspace(1e-9, 1e5, 301)])
    for f, ref in ((L.fo64_sin, np.sin), (L.fo64_cos, np.cos), (L.fo64_tan, np.tan)):
        got = np.array([f(float(x)) for x in xs])
        assert np.all(np.abs(got - ref(xs)) <= 2.0 * np.spacing(np.abs(ref(xs)))), f
    xe = np.linspace(-700.0, 700.0, 3001)
    got = np.array([L.fo64_exp(float(x)) for x in xe])
    assert np.all(np.abs(got - np.exp(xe)) <= 2.0 * np.spacing(np.exp(xe)))


# ---- 2. oracle pins: the real crate cannot run here
def _render(g, x, sr=48000.0):
    olib().fo_set_denormal_emulation(0)
    u = OracleUnit(g)
    u.set_sample_rate(sr)
    return u.process_many(x.shape[-1], x.reshape(1, -1).astype(F32))[0].astype(np.float64)


def _svf_lowpass_truth(f, q, sr, n):
    """src/svf.rs LowpassMode::response as a transfer function in z^-1, evaluated in f64 on a unit impulse."""
    g, k = math.tan(math.pi * f / sr), 1.0 / q
    b = np.array([g * g, 2 * g * g, g * g])
    a = np.array([1 + g * g + g * k, 2 * g * g - 2, 1 + g * g - g * k])
    x = np.zeros(n); x[0] = 1.0
    return signal.lfilter(b, a, x)


def _bell_truth(f, q, gain, sr, n):   # BellMode::response (src/svf.rs, bell)
    A, g = math.sqrt(gain), math.tan(math.pi * f / sr)
    k = 1.0 / (q * A)
    # H(z) = 1 + k (A^2 - 1) * g (z^2 - 1) / D(z), D(z) = (z - 1)^2 + g^2 (z + 1)^2 + g k (z^2 - 1)
    d = np.array([1 + g * g + g * k, 2 * g * g - 2, 1 + g * g - g * k])
    nb = d + k * (A * A - 1) * g * np.array([1.0, 0.0, -1.0])
    x = np.zeros(n); x[0] = 1.0
    return signal.lfilter(nb, d, x)


@pytest.mark.parametrize("f,q", [(5.0, 0.7), (2.0, 0.5)])
def test_impulse_response_where_f64_state_matters(f, q):
    """lowpass_hz at a few Hz and 48 kHz: the f64-state node's impulse response is within a few f32 roundings of the exact response;
    the f32 node misses that bar by more than 100x. Recorded (5 Hz, Q 0.7): prelude64 max error ~1e-11 of the peak, prelude32 ~1e-6."""
    n = 48000
    truth = _svf_lowpass_truth(f, q, 48000.0, n)
    x = np.zeros(n); x[0] = 1.0
    e64 = np.abs(_render(p64.lowpass_hz(f, q), x) - truth).max() / np.abs(truth).max()
    e32 = np.abs(_render(p32.lowpass_hz(f, q), x) - truth).max() / np.abs(truth).max()
    print(f"lowpass_hz({f}, {q}) @ 48 kHz: relative max error prelude64 {e64:.3e}, prelude32 {e32:.3e}")
    assert e64 <= 2.0 ** -23 and e32 >= 100.0 * e64, (e64, e32)


def test_impulse_responses_of_ordinary_settings():
    n = 4096
    x = np.zeros(n); x[0] = 1.0
    for g, truth in ((p64.lowpass_hz(1000.0, 2.0), _svf_lowpass_truth(1000.0, 2.0, 48000.0, n)),
                     (p64.bell_hz(2000.0, 1.5, 4.0), _bell_truth(2000.0, 1.5, 4.0, 48000.0, n))):
        got = _render(g, x)
        assert np.abs(got - truth).max() <= 2.0 ** -23 * np.abs(truth).max(), np.abs(got - truth).max()


@pytest.mark.parametrize("name", ["svf_lowpass_hz", "svf_bell_hz", "svf_highshelf_audio", "svf_notch_audio"])
def test_prelude32_and_prelude64_agree_within_f32_rounding(name):
    """The same filter graph built from prelude (f32 state) and prelude64: outputs differ only by the f32 arithmetic of the former.
    (An oscillator's f32 phase drifts from the f64 one without bound, so Sine is pinned by its first samples below instead.)"""
    mk64 = G.CASES[name]
    olib().fo_set_denormal_emulation(0)
    a = OracleUnit(mk64(5)); a.set_sample_rate(48000.0)
    y64 = a.process_many(8000)[0]
    g32 = _as_prelude32(name, 5)
    b = OracleUnit(g32); b.set_sample_rate(48000.0)
    y32 = b.process_many(8000)[0]
    scale = float(np.abs(y64).max())
    assert scale > 1e-3 and not np.array_equal(y32, y64)
    assert np.abs(y32.astype(np.float64) - y64).max() <= 2e-4 * scale, np.abs(y32.astype(np.float64) - y64).max() / scale


def _as_prelude32(name, i):
    fv = G.fv
    if name == "svf_lowpass_hz":
        return p32.noise().seed(i) >> p32.lowpass_hz(300.0 + 40.0 * i, 0.6 + fv(i))
    if name == "svf_bell_hz":
        return p32.noise().seed(i) >> p32.bell_hz(300.0 + 40.0 * i, 0.6 + fv(i), 0.25 + 3.0 * fv(i, 1))
    if name in ("svf_highshelf_audio", "svf_notch_audio"):
        node = p32.highshelf if "highshelf" in name else p32.notch
        cut = p32.sine_hz(1.5 + fv(i)) * p32.dc(300.0) + p32.dc(800.0 + 10.0 * i)
        q = p32.dc(0.7 + fv(i, 2))
        if "highshelf" in name:
            return (p32.noise().seed(i) | cut | q | (p32.sine_hz(0.5) * p32.dc(0.5) + p32.dc(1.5 + fv(i)))) >> node()
        return (p32.noise().seed(i) | cut | q) >> node()
    raise KeyError(name)


@pytest.mark.parametrize("g", [p64.lowpass_hz(700.0, 3.0), p64.highshelf_hz(700.0, 1.0, 5.0), p64.sine_hz(440.0)], ids=["lowpass", "highshelf", "sine"])
def test_tick_equals_process_for_filters(g):
    """FixedSvf<f64> has no block path of its own: tick and process agree bit for bit. (Sine<f64>'s block path uses wide sin, so
    its tick and process agree only to the two sines' accuracy.)"""
    olib().fo_set_denormal_emulation(0)
    x = (np.sin(np.arange(2000) * 0.37) * 0.8).astype(F32)
    a = OracleUnit(g); a.set_sample_rate(48000.0)
    if g.nin == 0:
        blk = a.process_many(2000)[0]
        a.reset()
        ticks = np.array([a.tick()[0] for _ in range(2000)], F32)
        assert np.abs(blk - ticks).max() <= 1e-6
        return
    blk = a.process_many(2000, x.reshape(1, -1))[0]
    a.reset()
    ticks = np.array([a.tick((float(v),))[0] for v in x], F32)
    assert np.array_equal(blk, ticks)


def _rnd1(x):   # src/math.rs:569-576
    M = (1 << 64) - 1
    x = (x ^ 0x5555555555555555) & M
    x = (x * 0x9e3779b97f4a7c15) & M
    x = ((x ^ (x >> 30)) * 0xbf58476d1ce4e5b9) & M
    x = ((x ^ (x >> 27)) * 0x94d049bb133111eb) & M
    x ^= x >> 31
    return (x >> 11) * (1.0 / 9007199254740992.0)


def test_sine_phase_starts_unrounded_and_advances_in_f64():
    """Sine<f64>::reset sets phase = rnd1(hash) in f64 (src/oscillator.rs:56-61) and tick advances it in f64. The oracle's phase after n
    ticks equals that f64 track exactly and differs from the track that starts from the f32-rounded phase; the product lowers the
    unrounded phase into its state word."""
    sr, f, n = 48000.0, 440.0, 1000
    L = oracle_prelude64.lib()
    for hash_ in (1, 12345, 0xdeadbeefcafef00d):
        p0 = _rnd1(hash_)
        assert float(F32(p0)) != p0
        tracks = []
        for start in (p0, float(F32(p0))):
            p = start
            for _ in range(n):
                p += float(F32(f)) * (1.0 / sr)
                p -= math.floor(p)
            tracks.append(p)
        got = L.fo_sine_f64_phase_after(hash_, sr, f, n)
        assert got == tracks[0] and got != tracks[1], (got, tracks)
        assert L.fo_sine_f64_phase_after(hash_, sr, f, 0) == p0
    h = capi.NodeHandle(p64.sine_hz(f)); h.set_sample_rate(sr)
    phase = float(h.lowering()[1].view(np.float64)[0])
    assert 0.0 < phase < 1.0 and float(F32(phase)) != phase


# ---- reference vectors of the real crate (oracle/ref_dump64 writes tests/golden/ref/manifest64.json); skipped until they exist
REF = os.path.join(ROOT, "tests", "golden", "ref")
MAN64 = os.path.join(REF, "manifest64.json")
PRELUDE64_REF = {   # the graphs of oracle/ref_dump64/src/main.rs
    "p64_sine_hz": lambda: p64.sine_hz(440.0),
    "p64_lowpass_hz": lambda: p64.white().seed(1) >> p64.lowpass_hz(1000.0, 1.0),
    "p64_bell_hz": lambda: p64.white().seed(2) >> p64.bell_hz(2000.0, 2.0, 3.0),
    "p64_lowpass_swept": lambda: (p64.white().seed(3) | (p64.sine_hz(2.0) * 400.0 + 900.0) | p64.dc(2.0)) >> p64.lowpass(),
    "p64_resonator_hz": lambda: p64.white().seed(4) >> p64.resonator_hz(700.0, 20.0),
    "p64_lowpole_hz": lambda: p64.white().seed(5) >> p64.lowpole_hz(2.0),
    "p64_pink": lambda: p64.pink(),
}


def reference_vector(name):
    """(graph, [channels, samples] float32) of a vector of the real crate, or a pytest skip when none were generated."""
    import json
    if not os.path.exists(MAN64):
        pytest.skip("no prelude64 reference vectors: tests/golden/ref/manifest64.json is absent (needs cargo and fundsp 0.23.0: oracle/ref_dump64)")
    v = next((x for x in json.load(open(MAN64))["vectors"] if x["name"] == name), None)
    if v is None:
        pytest.skip(f"{name} is not in manifest64.json")
    return PRELUDE64_REF[name](), np.fromfile(os.path.join(REF, name + ".f32"), "<f4").reshape(v["channels"], v["samples"])


@pytest.mark.parametrize("name", sorted(PRELUDE64_REF))
def test_oracle_matches_the_reference_crate_prelude64(name):
    g, want = reference_vector(name)
    olib().fo_set_denormal_emulation(0)
    u = OracleUnit(g); u.set_sample_rate(48000.0)
    got = u.process_many(want.shape[1])
    assert np.array_equal(got, want), (name, int((got != want).sum()), float(np.abs(got - want).max()))


# ---- 3. signatures, word layouts and refusals
def test_signatures_and_word_layouts():
    assert sig(p64.lowpass_hz(1000.0, 1.0)) == sig(p64.bell_hz(10.0, 2.0, 3.0)) == "FixedSvf64"
    assert sig(p64.bell()) == "Svf64<6>" and sig(p64.lowpass()) == "Svf64<0>"
    assert sig(p64.sine()) == "Sine64" and sig(p64.sine_hz(440.0)) == "Pipe<Constant<1>,Sine64>"
    assert sig(p32.lowpass_hz(1000.0, 1.0)) == "FixedSvf" and sig(p32.sine()) == "Sine"          # the f32 classes are unchanged
    sr = 48000.0
    h = capi.NodeHandle(p64.lowpass_hz(1000.0, 2.0)); h.set_sample_rate(sr)
    P, S, U = h.lowering()
    g, k = math.tan(math.pi * 1000.0 / sr), 0.5
    a1 = 1.0 / (1.0 + g * (g + k))
    assert len(P) == 12 and len(S) == 4 and len(U) == 0 and not S.any()
    assert np.allclose(P.view(np.float64), [a1, g * a1, g * g * a1, 0.0, 0.0, 1.0], rtol=1e-15, atol=0)
    h = capi.NodeHandle(p64.highshelf()); h.set_sample_rate(sr)
    P, S, _ = h.lowering()
    assert P.view(np.float64).tolist() == [sr] and len(S) == 24 and S.view(np.float64)[:4].tolist() == [440.0, 1.0, 1.0, sr]
    # the biquad and one-pole families: f64 word pairs, sample rate (and the rate the coefficients were made at) for the audio-rate forms
    assert sig(p64.biquad(0.1, 0.2, 0.3, 0.4, 0.5)) == sig(p64.resonator_hz(500.0, 3.0)) == sig(p64.butterpass_hz(900.0)) == "Biquad64"
    assert sig(p64.butterpass()) == "BiquadAudio64<0>" and sig(p64.resonator()) == "BiquadAudio64<1>"
    assert sig(p64.lowpole_hz(10.0)) == "OnePole64<0,1>" and sig(p64.allpole()) == "OnePole64<2,2>" and sig(p64.dcblock()) == "OnePole64<3,1>"
    assert sig(p64.pinkpass()) == "Pinkpass64" and sig(p64.pink()) == "Pipe<Noise,Pinkpass64>"
    P, S, _ = capi.NodeHandle(p64.biquad(0.1, 0.2, 0.3, 0.4, 0.5)).lowering()
    assert P.view(np.float64).tolist() == [float(F32(v)) for v in (0.1, 0.2, 0.3, 0.4, 0.5)] and len(S) == 8
    h = capi.NodeHandle(p64.lowpole_hz(10.0)); h.set_sample_rate(sr)
    P, S, _ = h.lowering()
    assert abs(P.view(np.float64)[0] - math.exp(-2 * math.pi * 10.0 / sr)) <= 2e-16
    assert len(S) == 2
    h = capi.NodeHandle(p64.resonator()); h.set_sample_rate(sr)
    P, S, _ = h.lowering()
    assert P.view(np.float64).tolist() == [sr] and len(S) == 24 and S.view(np.float64)[:3].tolist() == [440.0, 1.0, sr]
    h = capi.NodeHandle(p64.sine()); h.set_sample_rate(44100.0)
    P, S, _ = h.lowering()
    assert P.view(np.float64).tolist() == [1.0 / 44100.0] and len(S) == 2


def test_prelude64_refuses_what_it_does_not_lower():
    for name in ("moog_hz", "lowrez_hz", "morph", "follow", "afollow", "declick", "ramp", "poly_saw", "dlowpass_hz", "fbell",
                 "biquad_bank", "envelope_in", "lfo_in", "envelope2", "envelope3"):
        with pytest.raises(NotImplementedError, match="f64"):
            getattr(p64, name)(1.0, 1.0)
    assert p64.saw_hz is p32.saw_hz and p64.noise is p32.noise                   # names without f64 state are prelude's own
    assert p64.envelope(lambda t: t, 1).args[2] == 1                             # f64 time


# ---- 4. NVRTC compiles every class of the GPU file for sm_90a (no GPU needed; into a cache directory of the test's own)
def test_every_gpu_prelude64_class_compiles_with_nvrtc(tmp_path):
    sigs = sorted({sig(mk(i)) for mk in G.CASES.values() for i in (0, 1)})
    code = ("import sys\nfrom fundsp_b200 import capi\nfor s in sys.stdin.read().split('\\n'):\n"
            "    capi.jit_precompile(s, 1, 1 if ('WaveSynth<' in s or 'PhaseSynth<' in s) else 0)\nprint('compiled', capi.jit_cache_stats())\n")
    env = dict(os.environ, FDSP_JIT_CACHE=str(tmp_path))
    r = subprocess.run([sys.executable, "-c", code], input="\n".join(sigs), capture_output=True, text=True, env=env, cwd=ROOT, timeout=1800)
    assert r.returncode == 0 and "compiled" in r.stdout, (r.stdout[-500:], r.stderr[-2000:])
    assert len(os.listdir(tmp_path)) >= len(sigs)


# ---- 5. the device templates on the host emulation, one voice of every GPU case, against the oracle
@pytest.mark.parametrize("name", sorted(G.CASES))
def test_gpu_case_on_host_emulation(name, tmp_path):
    from test_device_emul_cpu import emulate, oracle
    n = 64 * 40 + 61
    mk = G.CASES[name]
    want = oracle(mk(3), n)
    got, s = emulate(mk(3), n, None, str(tmp_path))
    assert np.abs(want).max() > 1e-3, name
    assert np.array_equal(got, want), (name, int((got != want).sum()), float(np.abs(got - want).max()), s)


# ---- 6. the GPU file on the CPU mock device
def test_gpu_prelude64_file_on_the_mock_device(mock_env):
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_prelude64.py"), "-m", "gpu", "-q", "-n", "4",
                        "-p", "no:cacheprovider", "--tb=short"], capture_output=True, text=True, env=mock_env, cwd=ROOT, timeout=1800)
    tail = r.stdout[-3000:]
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, tail
