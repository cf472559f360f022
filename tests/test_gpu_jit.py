"""Structural coverage beyond the AOT config graphs: every §8a node family composed in ways the registry does not
list, compiled at bank creation by the NVRTC path from the same device headers, checked bit-for-bit against the oracle."""
import math

import numpy as np
import pytest

from fundsp_b200.graph import An
from fundsp_b200.prelude import *  # noqa: F401,F403
from fundsp_b200.prelude import _svf_hz
from oracle import lib as olib, oracle_bank_render

pytestmark = pytest.mark.gpu
SR = 48000.0


def fv(i, k=0):  # deterministic per-voice variation
    return ((i * 37 + k * 11) % 29) / 29.0


def _diamond(i):
    from fundsp_b200.net import Net
    net = Net(1, 2)
    a = net.push(lowpass_hz(600.0 + 20.0 * i, 1.0)); b = net.push(highpass_hz(300.0, 2.0)); c = net.push(pass_() + pass_())
    net.connect_input(0, a, 0); net.connect_input(0, b, 0); net.connect(a, 0, c, 0); net.connect(b, 0, c, 1)
    net.connect_output(c, 0, 0); net.connect_output(b, 0, 1)
    return net


def _net_ops(i):
    from fundsp_b200.net import Net
    return (Net.wrap(sine_hz(110.0 + i)) | Net.wrap(noise().seed(i))) >> Net.wrap(lowpass_hz(500.0 + 10.0 * i, 1.0) | pass_())


_WAVE = np.random.default_rng(77).uniform(-1.0, 1.0, (2, 1500)).astype(np.float32)   # a two-channel `Wave` for the sampler cases

def _ev(unit, start, end, ease, fade_in, fade_out, loop=0.0):
    from fundsp_b200.sequencer import event
    return event(unit, start, end, ease, fade_in, fade_out, loop=loop)


CASES = {
    "svf_var_lowpass_pan": lambda i: (noise().seed(i) | dc((300.0 + 4000.0 * fv(i), 0.5 + 4.0 * fv(i, 1)))) >> lowpass() >> pan(2.0 * fv(i, 2) - 1.0),
    "svf_var_bell": lambda i: (noise().seed(i) | dc((300.0 + 4000.0 * fv(i), 0.7, 0.5 + 2.0 * fv(i, 1)))) >> bell(),
    "svf_var_highshelf_mod": lambda i: (noise().seed(i) | (sine_hz(3.0 + i % 4) * 500.0 + 2000.0) | dc((1.0, 2.0))) >> highshelf(),
    "svf_fixed_all_modes": lambda i: noise().seed(i) >> pipei(3, lambda k: _svf_hz((i + 3 * k) % 9, 400.0 + 900.0 * k + 50.0 * (i % 7), 0.8 + 0.3 * k, 1.5)),
    "butter_resonator": lambda i: noise().seed(i) >> butterpass_hz(500.0 + 100.0 * (i % 9)) >> resonator_hz(800.0 + 40.0 * i, 5.0 + i % 3),
    "ticks_bus": lambda i: noise().seed(i) >> (pass_() & tick() * 0.5 & (tick() >> tick()) * (0.1 + 0.01 * i)),
    "feedback_delay": lambda i: noise().seed(i) >> feedback(delay(0.001) * (0.3 + 0.02 * (i % 10))),
    "allnest_delay": lambda i: noise().seed(i) >> allnest_c(0.2 + 0.02 * (i % 20), delay(0.0013)) >> fir((0.25, 0.5, 0.25)),
    "split_stacki_join": lambda i: noise().seed(i) >> split(4) >> stacki(4, lambda k: lowpass_hz(300.0 * (k + 1) + 10.0 * i, 1.0)) >> join(4),
    "organ_hammond_bus": lambda i: organ_hz(110.0 + 7.0 * i) & 0.5 * hammond_hz(220.0 + 3.0 * i) & square_hz(55.0 + i) * 0.25 & triangle_hz(330.0 - i) & soft_saw_hz(82.0 + i),
    "panner_audio_rate": lambda i: (noise().seed(i) | sine_hz(0.5 + 0.1 * (i % 5))) >> panner(),
    "moog_var": lambda i: (noise().seed(i) | (sine_hz(2.0) * 400.0 + 1200.0 + 10.0 * i) | dc(0.2 + 0.02 * (i % 20))) >> moog(),
    "moog_q_chain": lambda i: (noise().seed(i) | dc(900.0 + 25.0 * i)) >> moog_q(0.4) >> moog_hz(2000.0, 0.1 + 0.01 * (i % 30)),
    "sumi_sines_ops": lambda i: 1.0 - (-(sumi(3, lambda k: sine_hz(110.0 * (k + 1) + i).phase(0.1 * k)) * 0.3) - 0.25) + 0.125,
    "busi_branchi": lambda i: noise().seed(i) >> branchi(3, lambda k: lowpass_hz(200.0 * (k + 1) + i, 1.0)) >> (pass_() | sink() | pass_()) >> join(2),
    "multisplit_multijoin_thru": lambda i: (noise().seed(i) | noise().seed(i + 1000)) >> multisplit(2, 3) >> multijoin(2, 3) >> ~(join(2) >> lowpass_hz(700.0 + i, 2.0)) >> reverse(2),
    "wavesynth_phase_out": lambda i: dc(100.0 + 9.0 * i) >> An("wavesynth", (0, 2), (), 1, 2),
    "polyblep_oscs": lambda i: poly_saw_hz(110.0 + 13.0 * i) * 0.5 & poly_square_hz(55.0 + 7.0 * i).phase(0.25) * 0.3 & poly_pulse_hz(220.0 + i, 0.1 + 0.02 * (i % 30)) * 0.2 & ramp_hz(3.0 + i),
    "poly_pulse_modulated": lambda i: ((sine_hz(5.0) * 30.0 + 200.0 + 11.0 * i) | (sine_hz(0.5 + 0.1 * (i % 7)) * 0.4 + 0.5)) >> poly_pulse(),
    "mls_impulse": lambda i: mls_bits(5 + i % 20) * 0.5 + mls().seed(i) * 0.25 + (impulse(1) >> lowpass_hz(500.0 + 10.0 * i, 4.0)),
    "tap_spline_mod": lambda i: (noise().seed(i) | (sine_hz(0.7 + 0.1 * (i % 5)) * 0.004 + 0.005)) >> tap(0.0005, 0.01),
    "multitap_linear": lambda i: (noise().seed(i) | dc((0.002 + 0.0001 * i, 0.007)) | (sine_hz(2.0) * 0.001 + 0.003)) >> multitap_linear(3, 0.001, 0.01),
    "feedback2_delay_filter": lambda i: noise().seed(i) >> feedback2(delay(0.002) * (0.3 + 0.01 * (i % 30)), lowpass_hz(1500.0 + 20.0 * i, 1.0)),
    "fdn2_pair": lambda i: (noise().seed(i) | noise().seed(i + 500)) >> fdn2(stacki(2, lambda k: delay(0.001 + 0.0004 * k) * 0.45), stacki(2, lambda k: fir3(0.4 + 0.01 * (i % 20)))),
    "butterpass_audio_rate": lambda i: (noise().seed(i) | (sine_hz(1.0 + 0.2 * (i % 5)) * 300.0 + 900.0)) >> butterpass(),
    "resonator_audio_rate": lambda i: (noise().seed(i) | (sine_hz(0.5) * 200.0 + 700.0 + 5.0 * i) | dc(20.0 + i)) >> resonator(),
    "dsf_saw_fixed_roughness": lambda i: dc(55.0 + 9.0 * i) >> dsf_saw_r(0.3 + 0.015 * (i % 40)),
    "dsf_square_modulated": lambda i: ((sine_hz(4.0) * 20.0 + 110.0 + 7.0 * i) | (sine_hz(0.3 + 0.05 * (i % 9)) * 0.45 + 0.5)) >> dsf_square(),
    "reverb3_lowpass_loop": lambda i: (noise().seed(i) | noise().seed(i + 100)) >> (multipass(2) & 0.25 * reverb3_stereo(1.0 + 0.1 * (i % 10), 0.3 + 0.01 * (i % 40), lowpass_hz(6000.0 + 50.0 * i, 0.7))),
    "var_gain": lambda i: var(0.1 + 0.02 * i) * noise().seed(i) + var(0.5) * sine_hz(100.0 + i),
    "feedback_unit_block_mode": lambda i: noise().seed(i) >> feedback_unit(0.005 + 0.0001 * (i % 20), (0.4 + 0.005 * (i % 40)) * lowpass_hz(1000.0 + 30.0 * i, 1.0)),
    "feedback_unit_tick_mode_sine": lambda i: noise().seed(i) >> feedback_unit(0.0005, 0.5 * (pass_() * sine_hz(3.0 + i))),
    "feedback_unit_stereo": lambda i: (noise().seed(i) | sine_hz(220.0 + i)) >> feedback_unit(0.003, (0.3 * lowpass_hz(900.0 + 10.0 * i, 0.8)) | (0.3 * pass_())),
    "pink_brown_dcblock": lambda i: pink().seed(i) * 0.5 + brown().seed(i + 7) * 0.25 + (noise().seed(i + 9) >> dcblock_hz(20.0 + i) >> allpole_delay(0.2 + 0.03 * (i % 30))),
    "onepoles_audio_rate": lambda i: (noise().seed(i) | (sine_hz(2.0) * 300.0 + 500.0 + 10.0 * i)) >> ~lowpole() >> highpole() | (noise().seed(i + 3) | (sine_hz(1.0 + 0.1 * (i % 7)) * 0.4 + 0.6)) >> allpole(),
    "reverb3_lowpole_loop": lambda i: (noise().seed(i) | noise().seed(i + 100)) >> reverb3_stereo(2.0, 0.5, lowpole_hz(8000.0 - 40.0 * i)),
    "shapers": lambda i: noise().seed(i) * (0.5 + 0.05 * i) >> (shape(Tanh(1.0 + 0.1 * i)) & shape(Softsign(2.0)) & shape(Crush(4.0 + i)) & shape(SoftCrush(3.0 + i)) & clip() & clip_to(-0.3, 0.1 + 0.01 * i)),
    "tanh_in_feedback": lambda i: noise().seed(i) >> feedback(delay(0.001 + 0.0001 * (i % 10)) >> shape(Tanh(1.2)) * 0.9),
    "followers": lambda i: (noise().seed(i) >> follow(0.0005 + 0.0001 * i)) * 4.0 + (square_hz(5.0 + i) >> afollow(0.001 + 0.0002 * (i % 9), 0.01 + 0.001 * (i % 13))),
    "rez_filters": lambda i: noise().seed(i) >> (lowrez_hz(300.0 + 40.0 * i, 0.2 + 0.01 * (i % 50)) & bandrez_hz(900.0 + 20.0 * i, 0.4)) | (noise().seed(i + 50) | (sine_hz(1.5) * 400.0 + 900.0) | dc(0.3 + 0.01 * (i % 30))) >> bandrez(),
    "morph_filter": lambda i: (noise().seed(i) | (sine_hz(0.7) * 500.0 + 1500.0) | dc(1.0 + 0.1 * (i % 20)) | (sine_hz(0.3 + 0.05 * (i % 11)) * 0.9)) >> morph() | noise().seed(i + 9) >> morph_hz(600.0 + 10.0 * i, 2.0, -0.5),
    "declick": lambda i: noise().seed(i) >> declick_s(0.001 + 0.0005 * (i % 20)) | saw_hz(100.0 + i) >> declick(),
    "declick_in_feedback": lambda i: noise().seed(i) >> feedback(delay(0.001) * 0.5 >> declick_s(0.003 + 0.0001 * i)),
    "lorenz_rossler": lambda i: dc(100.0 + 20.0 * i) >> lorenz() | (sine_hz(0.5) * 50.0 + 200.0 + i) >> rossler(),
    "product_fm_feedback": lambda i: (sine_hz(200.0 + i) * sine_hz(3.0 + 0.1 * i)) >> feedback(tick() * 0.25 >> lowpass_hz(2000.0, 0.7)),
}
# Cases added after the last GPU run of the round they were written in: tests/test_gpu_wider.py runs them AFTER the parity tests,
# so that `pytest -x` reaches the BASELINE configurations first. (tests/test_device_emul_cpu.py runs them on the host emulation.)
WIDER = {
    "dag_diamond_net": lambda i: noise().seed(i) >> _diamond(i).node(),
    "dag_net_operators": lambda i: _net_ops(i).node() >> join(2),
    "dag_net_in_feedback": lambda i: noise().seed(i) >> feedback((__import__("fundsp_b200.net", fromlist=["Net"]).Net.wrap(delay(0.001) * 0.5) >> __import__("fundsp_b200.net", fromlist=["Net"]).Net.wrap(lowpole_hz(1500.0 + 10.0 * i))).node()),
    "dirty_biquads": lambda i: noise().seed(i) >> (dbell_hz(Tanh(1.0), 800.0 + 30.0 * i, 10.0, 2.0) & dhighpass_hz(Softsign(1.0), 2000.0, 2.0) & dresonator_hz(Tanh(0.5), 1000.0 + 10.0 * i, 10.0) & dlowpass_hz(Crush(64.0), 1500.0, 2.0)),
    "feedback_biquads": lambda i: noise().seed(i) >> (fbell_hz(Tanh(1.0), 500.0 + 20.0 * i, 50.0, 0.5) & flowpass_hz(Clip(1.0), 2000.0, 2.0) & fresonator_hz(SoftCrush(32.0), 700.0, 20.0) & fhighpass_hz(Softsign(0.2), 2000.0 + 10.0 * i, 2.0)),
    "nl_biquads_audio_rate": lambda i: (noise().seed(i) | (sine_hz(1.0) * 500.0 + 1500.0 + 10.0 * i) | dc(2.0)) >> dlowpass(Tanh(1.0)) | (noise().seed(i + 3) | dc((800.0, 3.0, 2.0 + 0.05 * i))) >> fbell(Softsign(1.0)),
    "pulse_wave": lambda i: ((sine_hz(3.0 + i % 5) * 30.0 + 110.0 + 7.0 * i) | (sine_hz(0.7) * 0.4 + 0.5)) >> pulse() | dc((55.0 + i, 0.1 + 0.02 * (i % 40))) >> pulse().phase(0.25),
    "phase_synth_tables": lambda i: ramp_hz(100.0 + 13.0 * i) >> (phase_synth(SQUARE) & phase_synth(ORGAN) * 0.5) | (sine_hz(50.0 + i) * 0.6) >> phase_synth(SOFT_SAW),
    "rotate_mixer": lambda i: (noise().seed(i) | sine_hz(200.0 + i)) >> rotate(0.1 * i, 0.8) >> mixer([[0.5, -0.25], [0.125 * (i % 8), 1.0], [1.0, 1.0]]),
    "reverb4_short_lines": lambda i: (noise().seed(i) | noise().seed(i + 100)) >> reverb4_stereo_delays([d * (0.15 + 0.002 * (i % 25)) for d in REVERB4_DELAYS], 1.0 + 0.05 * (i % 8)),
    "slot_voices": lambda i: __import__("fundsp_b200.sequencer", fromlist=["slot"]).slot((saw_hz(110.0 + 5.0 * i) >> lowpass_hz(800.0 + 30.0 * i, 1.0 + 0.05 * i)) | noise().seed(i) >> declick_s(0.003)),
    "oversampled_distortion": lambda i: (sine_hz(2000.0 + 150.0 * i) * (1.0 + 0.1 * i) | noise().seed(i)) >> oversample(shape(Tanh(1.0 + 0.05 * i)) | lowpass_hz(4000.0 + 100.0 * i, 1.0)),
    "oversampled_oscillator_mix": lambda i: noise().seed(i) * 0.01 >> oversample(pass_() + (saw_hz(300.0 + 20.0 * i) >> lowpole_hz(5000.0)) * 0.5 >> declick_s(0.002)),
    "flanger_phaser": lambda i: noise().seed(i) >> flanger(0.3 + 0.01 * (i % 40), 0.001, 0.004, lambda t, i=i: 0.0025 + 0.0015 * math.sin((20.0 + i) * t), horizon=0.1) | noise().seed(i + 7) >> phaser(0.2 + 0.01 * (i % 50), lambda t, i=i: 0.5 + 0.5 * math.sin((30.0 + i) * t), horizon=0.1),
    # closures crossing the ABI as host callbacks (envelope / lfo): sampled on the host at the reference's points, interpolated on the device
    "lfo_vibrato": lambda i: lfo(lambda t, i=i: 220.0 + 3.0 * i + (2.0 + 0.1 * i) * math.sin(2.0 * math.pi * (4.0 + 0.1 * i) * t), horizon=0.1) >> sine() | envelope(lambda t, i=i: math.exp(-t * (5.0 + i)), horizon=0.1) * noise().seed(i),
    "envelope_two_outputs_f64": lambda i: envelope(lambda t, i=i: (min(1.0, t * (50.0 + i)), 300.0 + 100.0 * t), horizon=0.1, time64=True) >> (pass_() * (pass_() >> saw())),
    # sequencer events (src/sequencer.rs): per-voice start / end / fades; checked against one-event Sequencers of the oracle
    "events_saw_filter": lambda i: _ev(saw_hz(110.0 + 3.0 * i) >> lowpass_hz(900.0 + 20.0 * i, 2.0), (31.0 + 37.7 * i) / SR, (31.0 + 37.7 * i + 600.3 + 23.1 * i) / SR, 1, (40.5 + i) / SR, (200.0 + 5 * i) / SR),
    "events_power_fades_stereo": lambda i: _ev(sine_hz(300.0 + i) | noise().seed(i), (1.0 + 0.37 * i) * 64.0 / SR, ((1.0 + 0.37 * i) * 64.0 + 700.0 + 11.0 * i) / SR, 0, (100.0 + 3.3 * i) / SR, (300.0 + 2.1 * i) / SR),
    "events_moog_program": lambda i: _ev(saw_hz(80.0 + 4.0 * i) >> moog_hz(700.0 + 30.0 * i, 0.5) >> pan(0.02 * i - 0.4), (17.0 + 9.3 * i) / SR, (17.0 + 9.3 * i + 900.0) / SR, i % 2, (50.0 + i) / SR, (250.0 + 3 * i) / SR),
    # events of a ReplayMode::Loop(777.25 / SR) sequencer: notes that end and restart every period (unit reset on the device, delay line cleared), notes that
    # straddle the loop point, notes longer than a period; the silent block tails behind each wrap are the reference's (src/sequencer.rs:845-872 as written)
    "events_looping": lambda i: _ev(saw_hz(90.0 + 5.0 * i) >> (pass_() & delay(0.0005 + 0.00001 * i)) >> moog_hz(900.0 + 25.0 * i, 0.4), (13.0 + 17.3 * i) / SR,
                                    (13.0 + 17.3 * i + 300.0 + 19.7 * i) / SR, i % 2, (20.5 + i) / SR, (60.0 + 2 * i) / SR, loop=777.25 / SR),
    "events_short_and_late": lambda i: _ev(organ_hz(200.0 + 5.0 * i) >> declick_s(0.002), (i * 50.25) / SR, (i * 50.25 + 1.0 + 9.0 * (i % 13)) / SR, i % 2, 0.0, 0.0) if i % 3 else _ev(organ_hz(200.0 + 5.0 * i) >> declick_s(0.002), 5000.0 / SR, 6000.0 / SR, 1, 0.0, 0.0),
    "limiters": lambda i: noise().seed(i) * (1.0 + 0.2 * i) >> limiter(0.001 + 0.0004 * (i % 2), 0.01) | (noise().seed(i + 50) * (sine_hz(3.0) * 2.0 + 2.5) | sine_hz(300.0 + i) * 4.0) >> limiter_stereo(0.0005, 0.003 + 0.001 * (i % 3)),
    "meters": lambda i: noise().seed(i) * (0.2 + 0.02 * i) >> (meter(Meter.Sample) & meter(Meter.Peak(0.002 + 0.0005 * (i % 9))) & meter(Meter.Rms(0.001 + 0.0003 * (i % 7)))),
    "sampler_regions": lambda i: playwave(_WAVE, i % 2, None if i % 3 else 100 + i) | playwave_at(_WAVE, 0, 10 + i, 400 + 7 * i, 50 + i) * 0.5,
    "sampler_pitched": lambda i: (sine_hz(1.0 + 0.1 * i) * 0.3 + 0.5 + 0.04 * i) >> resample(playwave(_WAVE, 1, 0)) | dc(0.25 + 0.05 * (i % 30)) >> resample(saw_hz(110.0 + i) | noise().seed(i)),
}
GATED = {
    "adsr_noise": lambda i: adsr_live(0.005 + 0.001 * (i % 5), 0.05, 0.5 + 0.01 * (i % 20), 0.1) * noise().seed(i) | ~zero() >> sine_hz(100.0 + i),
}


def run_case(mk, V, n, inp=None):
    from fundsp_b200.bank import GpuBank
    olib().fo_set_denormal_emulation(0)
    b = GpuBank([mk(i) for i in range(V)], per_voice=True, sample_rate=SR)
    g, _ = b.render_samples(n, inp)
    o, _ = oracle_bank_render([mk(i) for i in range(V)], SR, n, inp, threads=4)
    return b, g, o


@pytest.mark.parametrize("name", sorted(CASES))
def test_jit_graph_matches_oracle(name):
    b, g, o = run_case(CASES[name], 40, 2000 + 61)
    assert g.shape == o.shape and np.isfinite(g).all() and np.abs(o).max() > 1e-4
    bad = int((g != o).sum())
    assert bad == 0, (name, bad, float(np.abs(g - o).max()), b.classes()[0]["signature"])


def test_jit_gated_envelope():
    n = 9600 + 7
    gate = np.zeros((1, n), np.float32)
    gate[0, 300:4000] = 1.0
    gate[0, 6000:7000] = 0.7
    b, g, o = run_case(GATED["adsr_noise"], 40, n, gate)
    assert np.abs(o).max() > 0.1
    assert np.array_equal(g, o), (int((g != o).sum()), float(np.abs(g - o).max()))


@pytest.mark.parametrize("K", [1, 3, 64, 1000])
def test_convolver_matches_linear_convolution(K):
    """Convolver (src/convolve.rs): the reference computes y = x * h with a partitioned FFT (fft-convolver, not vendored), so the
    bar is the tolerance of the path, 1e-5 of the output peak (the reference's own test, test_basic.rs:698-711, uses 1e-4)."""
    rng = np.random.default_rng(K)
    h = rng.uniform(-1, 1, K) * np.exp(-np.arange(K) / max(1.0, K / 4.0))
    h = (h / np.abs(h).max()).astype(np.float32)
    V, n = 48, 3000 + 61                       # ragged: the last block has 5 tail samples through the per-sample path
    mk = lambda i: noise().seed(i) * (0.5 + 0.01 * i) >> convolve(h)
    b, g, o = run_case(mk, V, n)
    assert b.classes()[0]["voices"] == V       # one class: the impulse response is shared, class-uniform data
    peak = float(np.abs(o).max())
    assert peak > 0.1 and float(np.abs(g - o).max()) <= 1e-5 * peak, float(np.abs(g - o).max()) / peak
    # state carries across calls and process()-sized launches agree with the long render
    from fundsp_b200.bank import GpuBank
    b2 = GpuBank([mk(i) for i in range(V)], per_voice=True, sample_rate=SR)
    parts = np.concatenate([b2.render_samples(m)[0] for m in (64, 7, 1000, 61, n - 64 - 7 - 1000 - 61)], axis=-1)
    if K < 32:
        assert np.array_equal(parts, g)
    else:   # tensor-core form (K >= 32): how a launch is cut into 64-sample tiles changes the order of the partial sums, not the value
        assert float(np.abs(parts - g).max()) <= 2e-6 * peak, float(np.abs(parts - g).max()) / peak


@pytest.mark.parametrize("K", [64, 257, 1000, 4096])
def test_tensor_core_convolver(K, monkeypatch):
    """`x >> convolve(h)` as Toeplitz GEMM tiles on tensor cores (csrc/dsp/conv_tc_kernel.cuh: wgmma, TMA operand tiles, 3xTF32):
    against the f64 linear convolution (what the reference's partitioned FFT computes, src/convolve.rs:9-59) within 1e-5 of the output
    peak, for responses from one tile chunk to 4096 taps; partly filled voice tile, ragged last time tile, a render longer than the
    16384-sample chunk (history columns), state across calls, reset, clone, the voice-order mix, and the direct form as a cross-check."""
    import os
    from fundsp_b200.bank import GpuBank
    if K > 1000 and "mock" in os.environ.get("FDSP_B200_LIB", ""):
        pytest.skip("4096 taps in the direct form on the CPU mock device takes minutes; the tensor-core form is GPU-only")
    rng = np.random.default_rng(K)
    h = rng.uniform(-1, 1, K) * np.exp(-np.arange(K) / (K / 3.0))
    h = (h / np.abs(h).max()).astype(np.float32)
    V, n = 150, 16384 + 128 * 2 + 77
    mk = lambda i: noise().seed(i) * (0.5 + 0.003 * i) >> convolve(h)
    b = GpuBank([mk(i) for i in range(V)], per_voice=True, mix=True, sample_rate=SR)
    g, mix = b.render_samples(n)
    x = np.stack([oracle_rows(noise().seed(i) * (0.5 + 0.003 * i), n) for i in (0, 77, V - 1)])
    want = np.stack([np.convolve(r.astype(np.float64), h.astype(np.float64))[:n] for r in x])
    peak = float(np.abs(want).max())
    err = float(np.abs(g[[0, 77, V - 1], 0] - want).max())
    assert peak > 0.1 and err <= 1e-5 * peak, err / peak
    acc = g[0, 0].copy()
    for v in range(1, V):
        acc = acc + g[v, 0]
    if "mock" in os.environ.get("FDSP_B200_LIB", ""):   # (the mock runs the direct form, whose mix is the CTA-level tree)
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
    if "mock" not in os.environ.get("FDSP_B200_LIB", ""):
        monkeypatch.setenv("FDSP_TC_CONV", "0")
        d, _ = GpuBank([mk(i) for i in range(V)], per_voice=True, mix=True, sample_rate=SR).render_samples(2000)
        assert float(np.abs(d - g[..., :2000]).max()) <= 1e-5 * peak


def oracle_rows(expr, n):
    from oracle import OracleUnit
    u = OracleUnit(expr); u.set_sample_rate(SR)
    return u.process_many(n)[0]


def test_unsupported_graph_reports_error():
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.capi import ERR_UNSUPPORTED, FdspError
    with pytest.raises(FdspError) as e:
        GpuBank([busi(2, lambda k: noise() if k == 0 else sine_hz(440.0))], per_voice=True)  # busi needs one node type (MultiBus<N, X>)
    assert e.value.code == ERR_UNSUPPORTED
