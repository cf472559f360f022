"""CPU tests of the product's host side (no GPU, no compute calls): the C-ABI library loads and exports
every symbol include/fundsp_b200.h declares; its construction-time logic (ping hashes, settings, arity,
type expressions, wavetables) agrees with the oracle."""
import os

import numpy as np
import pytest

from fundsp_b200 import capi, workloads
from fundsp_b200 import prelude64 as p64
from fundsp_b200.graph import ArityError
from fundsp_b200.prelude import *  # noqa: F401,F403
from oracle import OracleUnit, lib as olib

L = capi.lib()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    syms = capi.header_symbols()
    assert len(syms) >= 60
    for s in syms:
        assert hasattr(L, s), s
    assert set(capi._SIG) == set(syms)
    assert b"sm_90a" in L.fdsp_version()


GRAPHS = [
    lambda: sine_hz(440.0) >> lowpass_hz(1000.0, 1.0),
    lambda: workloads.fm_voice(7),
    lambda: workloads.noise_svf_voice(3),
    lambda: workloads.saw_svf_voice(11),
    lambda: workloads.biquad_bank_unit(2),
    lambda: workloads.subtractive_voice(5),
    lambda: workloads.net_voice(0), lambda: workloads.net_voice(1), lambda: workloads.net_voice(2), lambda: workloads.net_voice(3),
    lambda: noise() | (~zero() >> noise()) | noise() & zero(),
    lambda: (noise() | dc((1000.0, 0.5))) >> moog() | (noise() | dc(800.0)) >> moog_q(0.3),
    lambda: dc((440.0, 880.0)) >> multisplit(2, 5) >> sumi(10, lambda i: saw() * 0.1) | saw_hz(220.0).phase(0.5) * 0.1,
    lambda: (pass_() ^ mul(-4.0) ^ add(-2.0)) >> add(5.0) + sub(3.0) + mul(-4.0),
    lambda: feedback(delay(0.5) * 0.5),
    lambda: dc(1.0) >> adsr_live(0.001, 0.002, 0.5, 0.003),
    lambda: poly_saw_hz(440.0) | poly_square_hz(220.0).phase(0.5) | poly_pulse_hz(110.0, 0.3) | ramp_hz(5.0),
    lambda: mls() | mls_bits(10).seed(3) | (impulse(2) >> join(2)),
    lambda: (noise() | sine_hz(0.5) * 0.004 + 0.005) >> tap(0.001, 0.01) | (noise() | dc((0.002, 0.007))) >> multitap_linear(2, 0.001, 0.01),
    lambda: (noise() | noise()) >> (multipass(2) & 0.25 * reverb3_stereo(2.0, 0.5, lowpass_hz(8000.0, 0.7))) | var(0.5) * noise(),
    lambda: noise() >> feedback_unit(0.01, 0.5 * lowpass_hz(1000.0, 1.0)) | noise() >> feedback_unit(0.001, 0.5 * highpass_hz(1000.0, 1.0)),
    lambda: noise() >> convolve([1.0, 0.9, 0.8]) | noise() >> convolve([0.5, 0.4, 0.3]),
    lambda: pink() | brown().seed(2) | noise() >> dcblock() >> allpole_delay(0.5) >> highpole_hz(500.0) | (noise() | dc(440.0)) >> lowpole(),
    lambda: noise() >> shape(Tanh(2.0)) >> clip() | noise() >> shape(Crush(8.0)) >> shape(SoftCrush(5.0)) >> shape(Softsign(1.5)) >> clip_to(-0.5, 0.5),
    lambda: noise() >> follow(0.002) | noise() >> afollow(0.001, 0.01),
    lambda: (noise() | noise()) >> ((pass_() | dc((2000.0, 5.0, 0.8))) >> morph() | morph_hz(440.0, 1.0, 0.0)) | (noise() | noise()) >> (lowrez_hz(440.0, 0.5) | bandrez_hz(440.0, 0.5)) | (noise() | dc(900.0)) >> lowrez_q(0.3),
    lambda: noise() >> declick() >> declick_s(0.002),
    lambda: noise() >> dbell_hz(Tanh(1.0), 1000.0, 10.0, 2.0) >> flowpass_hz(Clip(1.0), 2000.0, 2.0) | (noise() | dc((800.0, 3.0))) >> dresonator(Softsign(0.5)),
    lambda: dc(220.0) >> lorenz() | dc(110.0) >> rossler() | dc(330.0) >> lorenz(),
    lambda: dc((220.0, 0.3)) >> pulse() | dc((220.0, 0.3)) >> pulse().phase(0.5) | (ramp_hz(50.0) >> phase_synth(3) | noise()) >> rotate(0.3, 0.5) >> mixer([[1.0, 2.0]]),
    lambda: (noise() | noise()) >> reverb4_stereo(25.0, 2.0),
    lambda: __import__('fundsp_b200.sequencer', fromlist=['slot']).slot(saw_hz(110.0) >> lowpass_hz(800.0, 1.0) | noise()),
    lambda: noise() >> oversample(shape(Tanh(2.0)) >> lowpass_hz(5000.0, 1.0)) | oversample(saw_hz(110.0)) | noise() >> oversample(sine_hz(3.0) * pass_()),
    lambda: unit(noise() >> monitor() >> lowpass_hz(500.0, 1.0)) | noise() >> pass_() >> lowpass_hz(500.0, 1.0),     # Monitor hashes as ID 56, not as a Pass
    lambda: noise() >> flanger(0.5, 0.005, 0.010, lambda t: 0.0075, horizon=0.05) | noise() >> phaser(0.5, lambda t: 0.5, horizon=0.05) | white(),
    lambda: lfo(lambda t: 440.0 + t, horizon=0.05) >> sine() | envelope(lambda t: (t, 1.0 - t), horizon=0.05) >> (pass_() * pass_()) | lfo(lambda t: 1.0, horizon=0.02, time64=True) * noise(),
    lambda: noise() >> limiter(0.005, 0.05) | (noise() | noise()) >> limiter_stereo(0.002, 0.02),
    lambda: dc(1.5) >> resample(noise() | sine_hz(440.0)) | dc(0.5) >> resample(playwave(np.linspace(-1, 1, 50, dtype=np.float32)[None, :], 0, 0)) | noise() >> meter(Meter.Rms(0.1)),
    lambda: dc(220.0) >> dsf_saw_r(0.7) | (dc(110.0) | dc(0.4)) >> dsf_square() | dc(440.0) >> dsf_square_r(0.3).phase(0.25),
    lambda: noise() >> feedback2(delay(0.002) * 0.5, lowpass_hz(2000.0, 1.0)) | (noise() | dc(800.0)) >> butterpass() | (noise() | dc((900.0, 8.0))) >> resonator(),
    # closures, the Atan and Adaptive shapes, prelude64 and Shared controls: leaves built by the oracle's fo_closure, fo_shapes,
    # fo_prelude64 and fo_shared units, which its leaf-hash trace sees like those of fundsp_oracle.cpp
    lambda: (noise() | sine_hz(110.0)) >> map_("|x| (x[0] * g, x[1] - x[0])", 2, 2, g=0.5) | noise() >> shape_fn("|x| x * 0.5") >> sine()
            | (noise() | sine_hz(3.0) | dc(0.2)) >> envelope_in("|t, i| i[0] * 0.5 + i[1] * i[2] + sin_hz(2.0, t) * k", 3, k=0.1),
    lambda: noise() >> shape(Atan(2.0)) >> sine() | noise() >> shape(Adaptive(0.01, Tanh(1.0))) | noise() >> fbell_hz(Atan(1.0), 500.0, 50.0, 0.5),
    lambda: dc(440.0) >> p64.sine() | sine_hz(3.0) | noise() >> p64.lowpass_hz(1000.0, 0.7) | (noise() | dc(800.0)) >> p64.butterpass(),
    lambda: var(shared(0.5)) * saw_hz(220.0) | var_fn(shared(0.25), "|x| (x, -x)", 2) | noise() >> monitor(shared(), Meter.Rms(0.1)) | timer(shared()),
]


@pytest.mark.parametrize("k", range(len(GRAPHS)))
def test_host_ping_and_arity_match_oracle(k):
    g = GRAPHS[k]()
    n, o = capi.NodeHandle(g), OracleUnit(g)
    assert (n.inputs(), n.outputs()) == (o.inputs(), o.outputs()) == (g.inputs(), g.outputs())
    assert n.leaf_hashes() == o.leaf_hashes()
    assert n.ping(True, 12345) == o.ping(True, 12345)


def test_arity_errors_are_reported_not_crashes():
    be = capi.GpuBackend()
    a, b = be.b_pass(), be.b_stack(be.b_pass(), be.b_pass())
    with pytest.raises(capi.FdspError) as e:
        be.b_pipe(a, b)  # 1 output >> 2 inputs
    assert e.value.code == capi.ERR_ARITY
    with pytest.raises(ArityError):
        pass_() >> (pass_() | pass_())
    with pytest.raises(capi.FdspError):
        be.b_wavesynth(9, 1)


def test_builder_argument_errors_return_null_with_a_message():
    """Invalid constructor arguments (asserts / type errors in the reference) come back as NULL + fdsp_last_error, never a crash."""
    be = capi.GpuBackend()
    two_in = be.b_stack(be.b_pass(), be.b_pass())
    bad = [
        lambda: be.b_tap(1, 0, 0.02, 0.01),                 # min_delay > max_delay (src/delay.rs:164-165)
        lambda: be.b_mls(0), lambda: be.b_mls(32),          # 1 <= n <= 31 (src/noise.rs:61)
        lambda: be.b_onepole(7, 100.0, 1), lambda: be.b_onepole(3, 100.0, 2), lambda: be.b_onepole(2, 0.0, 1),   # allpole delay must be > 0
        lambda: be.b_shaper(9, 1.0, 0.0), lambda: be.b_chaos(2), lambda: be.b_phase_osc(4), lambda: be.b_dsf(3, 1.0, 0.5),
        lambda: be.b_convolve([]), lambda: be.b_rez(0.0, 440.0, 1.0, 2),
        lambda: be.b_feedback_unit(0.01, be.b_stack(be.b_pass(), be.b_sink(1))),      # inputs != outputs (src/feedback.rs:349)
        lambda: be.b_reverb3(2.0, 0.5, two_in),                                       # loop filter must be 1 -> 1
        lambda: be.b_feedback2(0, be.b_pass(), be.b_stack(be.b_pass(), be.b_pass())), # X and Y arity differ
        lambda: be.b_impulse(0),
        lambda: be.b_meter(3, 0.1), lambda: be.b_meter(1, 0.0), lambda: be.b_playwave([0.0] * 8, 0, 9, -1), lambda: be.b_resample(be.b_pass()),   # end_point <= length; generator only
        lambda: be.b_limiter(0, 0.01, 0.01), lambda: be.b_limiter(1, -1.0, 0.01),
        lambda: be.b_event(0.0, 1.0, 1, 0.0, 0.0, be.b_pass()), lambda: be.b_event(0.0, 1.0, 1, 2.0, 0.0, be.b_noise()), lambda: be.b_event(0.0, 1.0, 3, 0.0, 0.0, be.b_noise()),   # generators only; fade <= duration
        lambda: be.b_envelope(0.0, 1, 0, lambda t: 0.0, 1.0), lambda: be.b_envelope(0.002, 0, 0, lambda t: 0.0, 1.0), lambda: be.b_envelope(1e-9, 1, 0, lambda t: 0.0, 10.0),   # interval > 0; 1..8 outputs; bounded table
        lambda: be.b_oversample(be.b_stack(be.b_pass(), be.b_sink(1))),   # more inputs than outputs
        lambda: be.b_phase_synth(6), lambda: be.b_mixer(0, 2, [1.0]), lambda: be.b_mixer(9, 9, [0.0] * 81),      # tables 0..5; 1 <= M*N <= 64
    ]
    for k, f in enumerate(bad):
        with pytest.raises(capi.FdspError) as e:
            f()
        assert e.value.code in (capi.ERR_ARITY, capi.ERR_ARG), k
        assert len(str(e.value)) > 10


def test_config_graphs_have_aot_programs():
    from ctypes import create_string_buffer
    for name in workloads.WORKLOADS:
        g = workloads.build(name, 1)[0]
        sig = capi.NodeHandle(g).signature()
        assert "Unsupported" not in sig, (name, sig)
    assert capi.NodeHandle(workloads.saw_svf_voice(0)).signature() == "Pipe<Pipe<Constant<1>,WaveSynth<0,1>>,FixedSvf>"
    assert capi.NodeHandle(workloads.fm_voice(0)).signature() == "Pipe<Unop<1,Unop<3,Unop<3,Pipe<Constant<1>,Sine>>>>,Sine>"
    assert create_string_buffer(4) is not None


def test_wavetables_match_oracle():
    O = olib()
    for kind in range(6):
        n = L.fdsp_wavetable_count(kind)
        assert n == O.fo_wavetable_count(kind) == 40
        worst, differing, total = 0.0, 0, 0
        for i in range(n):
            pitch, ln = capi.C.c_float(), capi.C.c_int()
            capi.check(L.fdsp_wavetable_info(kind, i, capi.C.byref(pitch), capi.C.byref(ln)))
            assert pitch.value == O.fo_wavetable_pitch(kind, i) and ln.value == O.fo_wavetable_len(kind, i)
            a = np.ctypeslib.as_array(L.fdsp_wavetable_data(kind, i), (ln.value,))
            b = np.ctypeslib.as_array(O.fo_wavetable_data(kind, i), (ln.value,))
            worst = max(worst, float(np.abs(a - b).max()))
            differing += int((a != b).sum())
            total += ln.value
        # independent builders (radix-2 f64 inverse FFT vs direct f64 DFT): equal to f32 rounding
        assert worst <= 2.4e-7, (kind, worst)
        assert differing <= total // 50, (kind, differing, total)


def test_bank_create_fails_loudly_without_gpu():
    if L.fdsp_device_count() > 0:
        pytest.skip("GPU present")
    from fundsp_b200.bank import GpuBank
    with pytest.raises(capi.FdspError) as e:
        GpuBank([sine_hz(440.0) >> lowpass_hz(1000.0, 1.0)])
    assert "no CPU fallback" in str(e.value)


def test_python_net_algebra_matches_oracle_cpp_algebra():
    """fundsp_b200/net.py (Python mirror of src/net.rs:1447-1832) vs the oracle's own C++ restatement of the same algebra."""
    import oracle as O
    from fundsp_b200.net import Net, balanced_bus
    be = O.OracleBackend()
    OL = O.lib()
    v = [sine_hz(110.0 * (i + 1)) >> lowpass_hz(1000.0, 1.0) >> pan(0.1 * i) for i in range(5)]
    # Python algebra lowered vertex by vertex
    pnet = balanced_bus([Net.wrap(g) for g in v])
    a = O.OracleUnit(pnet.lower(be))
    # oracle C++ algebra: same level-wise pairing with fo_net_combine(op 0 = bus)
    cur = [OL.fo_net_wrap(g.lower(be)) for g in v]
    while len(cur) > 1:
        nxt = [OL.fo_net_combine(0, cur[i], cur[i + 1]) for i in range(0, len(cur) - 1, 2)]
        if len(cur) & 1:
            nxt.append(cur[-1])
        cur = nxt
    b = O.OracleUnit(cur[0])
    assert OL.fo_net_size(a.h) == OL.fo_net_size(b.h) == pnet.size() == 5 + 2 * 4
    ya, yb = a.render(48000.0, 0.02), b.render(48000.0, 0.02)
    assert np.array_equal(ya, yb) and np.abs(ya).max() > 0.1
    # pipe / stack / product
    n1 = (Net.wrap(noise() | noise()) >> Net.wrap(lowpass_hz(500.0, 1.0) | highpass_hz(2000.0, 1.0))) * Net.wrap(dc((0.5, 0.25)))
    c1 = OL.fo_net_combine(5, OL.fo_net_combine(1, OL.fo_net_wrap((noise() | noise()).lower(be)), OL.fo_net_wrap((lowpass_hz(500.0, 1.0) | highpass_hz(2000.0, 1.0)).lower(be))),
                           OL.fo_net_wrap(dc((0.5, 0.25)).lower(be)))
    assert np.array_equal(O.OracleUnit(n1.lower(be)).render(48000.0, 0.01), O.OracleUnit(c1).render(48000.0, 0.01))


def test_product_net_extraction_errors_and_hashes():
    from fundsp_b200.net import Net, voice_net
    be = capi.GpuBackend()
    # a Net with a non-adder, non-voice vertex is not voice-separable: bank creation must say so (even without a GPU the
    # structural check runs first)
    n = Net(0, 1)
    a = n.chain(noise())
    n.chain(lowpass_hz(500.0, 1.0))
    out = capi.C.c_void_p()
    rc = L.fdsp_bank_create_from_net(n.lower(be), 0, capi.OUT_MIX, capi.C.byref(out))
    assert rc == capi.ERR_UNSUPPORTED and b"Net" in L.fdsp_last_error() and a == 0
    h = voice_net([workloads.net_voice(i) for i in range(6)]).lower(be)
    assert L.fdsp_net_size(h) == 6 + 2 * 5
    L.fdsp_node_free(h)


def test_cpp_host_mirror_compiles_and_matches_python_mirror(tmp_path):
    """include/fundsp_b200.hpp: the reference's graph notation for C++ hosts (same operators / precedence / opcode names)."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "host_mirror_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"), os.path.join(root, "tests", "cpp", "host_mirror_test.cpp"),
                           "-o", exe, "-L", os.path.join(root, "fundsp_b200"), "-lfundsp_b200", "-Wl,-rpath," + os.path.join(root, "fundsp_b200")])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    n = capi.NodeHandle(sine_hz(440.0) >> lowpass_hz(1000.0, 1.0))
    assert lines[0] == "sig " + n.signature()
    assert [int(x.split()[1], 16) for x in lines if x.startswith("hash")] == n.leaf_hashes()
    f, m = 220.0, 2.0
    fm = capi.NodeHandle(sine_hz(f) * f * m + f >> sine())
    assert f"fm 0 1 {fm.signature()}" in lines
    assert "bus 0 2" in lines and "stacki 4 4" in lines and any(x.startswith("arity error") for x in lines)
    synth = capi.NodeHandle((poly_saw_hz(110.0) & 0.5 * (dc(55.0) >> dsf_saw_r(0.6))) >> lowrez_hz(900.0, 0.4) >> shape(Tanh(1.5)) >> dcblock()
                            >> (pass_() & 0.3 * feedback_unit(0.02, 0.5 * lowpole_hz(3000.0))) >> pan(0.25)
                            >> (multipass(2) & 0.25 * reverb3_stereo(2.0, 0.5, lowpole_hz(8000.0))))
    assert f"synth 0 2 {synth.signature()}" in lines and "misc 0 8" in lines
    nlb = capi.NodeHandle((noise() >> dlowpass_hz(Tanh(1.0), 1200.0, 2.0)) | ((noise() | dc((900.0, 1.5, 2.0))) >> fbell(Softsign(0.8))) | (noise() >> fresonator_hz(Clip(1.0), 700.0, 4.0)))
    assert f"nlb 0 3 {nlb.signature()}" in lines

    def words_hash(g):
        h = capi.NodeHandle(g)
        P, S, _ = h.lowering()
        x = 1469598103934665603
        for w in list(P) + list(S):
            x = ((x ^ int(w)) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
        return h, f"{x:016x}"
    wide, wh = words_hash(((dc((110.0, 0.3)) >> pulse()) | (noise() >> phase_synth(2))) >> rotate(0.5, 0.8) >> mixer([[0.5, -0.25], [0.125, 1.0], [1.0, 1.0]]))
    assert f"wide 0 3 {wide.signature()} {wh}" in lines
    wv = (np.arange(64, dtype=np.float32) / np.float32(64.0) - np.float32(0.5))[None, :]
    smp, sh = words_hash((dc(0.75) >> resample(playwave(wv, 0, 8))) | (playwave_at(wv, 0, 4, 40) >> meter(Meter.Rms(0.05))) | (noise() >> meter(Meter.Peak(0.1)) >> limiter(0.003, 0.02)))
    assert f"smp 0 3 {smp.signature()} {sh}" in lines
    from fundsp_b200.sequencer import event, Fade
    ev, eh = words_hash(event(saw_hz(220.0) >> lowpass_hz(900.0, 2.0), 0.0125, 0.75, Fade.Power, 0.01, 0.2))
    assert f"event 0 1 {ev.signature()} {eh}" in lines
    assert "vib 0 1 Pipe<EnvelopeTab<1,0>,Sine>" in lines
    r1, h1 = words_hash(reverb_stereo(12.0, 2.5, 0.4))
    r4, h4 = words_hash(reverb4_stereo(20.0, 3.0))
    assert f"reverb_stereo {r1.signature()} {h1}" in lines and f"reverb4_stereo {r4.signature()} {h4}" in lines   # every coefficient, bit for bit


# ---------------------------------------------------------------- the NVRTC translation unit compiles without a GPU
def _nvrtc_available():
    import subprocess, sys
    return subprocess.run([sys.executable, "-c", "import warnings; warnings.simplefilter('ignore'); from cuda import nvrtc"], capture_output=True).returncode == 0


JIT_SAMPLES = [
    lambda: dc(220.0) >> dsf_saw_r(0.7),
    lambda: (noise() | dc((0.002, 0.007))) >> multitap_linear(2, 0.001, 0.01),
    lambda: noise() >> feedback2(delay(0.002) * 0.5, lowpass_hz(2000.0, 1.0)),
    lambda: (noise() | dc((900.0, 8.0))) >> resonator() | mls() | poly_saw_hz(110.0),
    lambda: (noise() | dc((1000.0, 0.5))) >> moog() >> pan(0.25),
]


def test_jit_translation_units_compile_for_sm90a():
    """Same headers and options as csrc/host/jit.cpp (tools/nvrtc_check.py); compile only, nothing runs. In a subprocess:
    the cuda-python bindings must not be imported into the test process (they break a later `import torch`)."""
    import subprocess, sys
    if not _nvrtc_available():
        pytest.skip("cuda-python NVRTC bindings not importable")
    sigs = [capi.NodeHandle(mk()).signature() for mk in JIT_SAMPLES]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "nvrtc_check.py")] + sigs, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-1000:]
    assert r.stdout.count("ok   ") == len(sigs)


def test_wav_files_match_the_reference_layout(tmp_path):
    """Wave::write_wav16 / write_wav32 (src/write.rs:24-116) byte for byte: the expectation is built here with struct + numpy, and
    Python's own `wave` module reads the 16-bit file back."""
    import struct
    import wave as pywave
    rng = np.random.default_rng(9)
    x = rng.uniform(-1.3, 1.3, (2, 1000)).astype(np.float32)
    x[0, :6] = [0.0, 1.0, -1.0, 0.5, -0.5, 3.0e-5]
    sr = 44100.0

    def header(data_len, fmt, ch, rate):
        sb = 2 if fmt == 1 else 4
        return (b"RIFF" + struct.pack("<I", data_len + 36) + b"WAVEfmt " + struct.pack("<IHHIIHH", 16, fmt, ch, rate, rate * ch * sb, ch * sb, sb * 8)
                + b"data" + struct.pack("<I", data_len))
    # 16 bit: round(clamp11(x) * 32767.49) in f32, half away from zero
    s = np.clip(x, np.float32(-1), np.float32(1)) * np.float32(32767.49)
    q = (np.sign(s) * np.floor(np.abs(s) + np.float32(0.5))).astype(np.int16)        # f32 round-half-away (|s| + 0.5 is exact enough below 2**15: checked against np.round for non-ties)
    nt = np.abs(np.abs(s) - np.floor(np.abs(s)) - 0.5) > 1e-3
    assert np.array_equal(q[nt], np.round(s[nt]).astype(np.int16))
    want16 = header(2 * 2 * 1000, 1, 2, 44100) + q.T.astype("<i2").tobytes()
    got16 = capi.encode_wav(x, sr, 16)
    assert got16 == want16
    want32 = header(4 * 2 * 1000, 3, 2, 44100) + x.T.astype("<f4").tobytes()
    assert capi.encode_wav(x, sr, 32) == want32
    p16, p32 = tmp_path / "a16.wav", tmp_path / "a32.wav"
    capi.save_wav(p16, x, sr, 16); capi.save_wav(p32, x, sr, 32)
    assert p16.read_bytes() == want16 and p32.read_bytes() == want32
    with pywave.open(str(p16), "rb") as f:
        assert (f.getnchannels(), f.getsampwidth(), f.getframerate(), f.getnframes()) == (2, 2, 44100, 1000)
        assert np.array_equal(np.frombuffer(f.readframes(1000), "<i2").reshape(1000, 2).T, q)
    y32, r32 = capi.load_wav(p32)
    assert r32 == 44100.0 and np.array_equal(y32, x)                                  # float files round-trip exactly
    y16, _ = capi.load_wav(p16)
    assert np.array_equal(y16, q.astype(np.float32) / np.float32(32768.0))
    assert q[0, 0] == 0 and q[0, 1] == 32767 and q[0, 2] == -32767 and q[0, 5] == 1   # 3e-5 * 32767.49 = 0.98 -> 1
    with pytest.raises(capi.FdspError):
        capi.encode_wav(np.zeros((0, 10), np.float32), sr, 16)                       # assert!(self.channels() > 0)
    with pytest.raises(capi.FdspError):
        capi.load_wav(tmp_path / "missing.wav")


def test_jit_disk_cache_fills_without_a_gpu(tmp_path):
    """csrc/host/jit.cpp keeps compiled units on disk, keyed by the exact compilation; fdsp_jit_precompile fills the cache on a
    machine without a GPU (tools/warm_jit_cache.py does it for the GPU suite's graph classes). Own process: the directory is read once."""
    import subprocess
    import sys
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "from fundsp_b200 import capi\n"
        "sig = 'Pipe<Noise,MeterNode<1>>'\n"
        "capi.jit_precompile(sig, 0); capi.jit_precompile(sig, 1, 0); a = capi.jit_cache_stats()\n"
        "capi.jit_precompile(sig, 0); capi.jit_precompile(sig, 1, 0); b = capi.jit_cache_stats()\n"
        "capi.jit_precompile('Pipe<Pipe<Constant<1>,WaveSynth<0,1>>,FixedSvf>', 1, 1); c = capi.jit_cache_stats()\n"   # ahead-of-time class: nothing to do
        "try:\n    capi.jit_precompile('Pipe<Noise,NoSuchNode>', 1, 0); bad = 'compiled'\nexcept capi.FdspError as e:\n    bad = 'error'\n"
        "print(a, b, c, bad)\n" % os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    env = dict(os.environ, FDSP_JIT_CACHE=str(tmp_path / "cache"))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.strip() == "{'hits': 0, 'nvrtc_runs': 2} {'hits': 2, 'nvrtc_runs': 2} {'hits': 2, 'nvrtc_runs': 2} error", r.stdout
    files = sorted(os.listdir(tmp_path / "cache"))
    assert len(files) == 2 and all(f.endswith(".fdspjit") for f in files)


def test_bench_tables_cover_every_workload():
    """bench.py --workload choices, its names and the workload builders stay in step (no GPU needed to find a missing key)."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    assert set(bench.HEADLINE) == set(workloads.WORKLOADS)
    for w, v in bench.HEADLINE.items():
        assert str(v) in bench.workload_name(w, v) and workloads.WORKLOADS[w][1] == v
        assert bench.gate_for(w, 64) is None or bench.gate_for(w, 64).shape == (1, 64)
