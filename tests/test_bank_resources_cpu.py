"""Every CUDA resource a bank takes is given back: each bank form is driven through create, render, process() and destroy on the mock
device (tests/test_mock_bank_cpu.py), whose runtime counts the device and pinned allocations, streams and events that are live, and the
count returns to where it started. Repeated rebuilds and repeated process() calls leave it where it is.

The mock never takes the tensor-core convolver or the resident process() kernel, so their buffers are not covered here; the convolver
and process() tests cover them on the GPU."""
import subprocess
import sys

from test_mock_bank_cpu import ROOT, mock_env  # noqa: F401  (the mock device build, shared with that file)

SCRIPT = r'''
import ctypes

import numpy as np
from fundsp_b200 import capi, workloads
from fundsp_b200.bank import GpuBank
from fundsp_b200.net import voice_net
from fundsp_b200.prelude import Meter, delay, lowpass_hz, monitor, noise, pan, pass_, reverb_stereo, saw_hz, sine_hz, timer, var
from fundsp_b200.sequencer import Fade, ReplayMode, Sequencer, event, slot
from fundsp_b200.shared import shared

live = capi.lib().fdsp_mock_live_resources
live.restype = ctypes.c_long
SR = 44100.0
stereo = lambda n: np.stack([np.sin(np.arange(n) * 0.01), np.cos(np.arange(n) * 0.013)]).astype(np.float32)


def run(b):
    inp = stereo(300) if b.inputs() else None
    b.render_samples(300, inp)
    for _ in range(4):
        b.process(64, None if inp is None else inp[:, :64])


def check(name, make, edit=None):
    base = live()
    b = make()
    counts = []
    for r in range(4):   # repeated rebuilds (a sample rate that changes every delay length) and process() calls hold the count
        b.set_sample_rate([48000.0, SR][r % 2])
        run(b)
        counts.append(live())
    assert len(set(counts)) == 1, (name, counts)
    for r in range(3 if edit else 0):
        edit(b, r)
        run(b)
    del b
    assert live() == base, (name, live() - base)
    print(name, "ok")


sat = lambda i: saw_hz(110.0 + 13 * i) >> lowpass_hz(900.0 + 20 * i, 1.0)
check("one class", lambda: GpuBank([sat(i) for i in range(8)], per_voice=True, mix=True, sample_rate=SR))
check("concurrent classes", lambda: GpuBank([[sat(i), sine_hz(200.0 + i), noise().seed(i) >> lowpass_hz(700.0, 1.0)][i % 3] for i in range(9)],
                                            per_voice=True, mix=True, sample_rate=SR))
check("net tree mix", lambda: GpuBank.from_net(voice_net([workloads.net_voice(i) for i in range(6)]), per_voice=False, mix=True, sample_rate=SR))
check("reverb with dry program", lambda: GpuBank([(noise().seed(i) >> pan(0.1 * i - 0.3)) >> reverb_stereo(12.0, 1.5, 0.4) for i in range(3)],
                                                 per_voice=True, mix=True, sample_rate=SR))
check("reverb without dry program", lambda: GpuBank([reverb_stereo(10.0, 1.0 + 0.5 * i, 0.3) for i in range(2)], per_voice=False, mix=True, sample_rate=SR))


def seq(mode):
    q = Sequencer(0, 1, mode)
    q.push(0.0, 0.002, Fade.Smooth, 0.0, 0.001, sine_hz(440.0))
    q.push(0.001, 0.004, Fade.Power, 0.0005, 0.001, noise().seed(3) >> (pass_() & delay(0.0007)) >> lowpass_hz(900.0, 1.0))
    q.push(0.0, 0.0, Fade.Smooth, 0.0, 0.0, sine_hz(330.0))   # finished at once: a free slot for push_event
    return q


check("sequencer events", lambda: GpuBank.from_sequencer(seq(ReplayMode.None_), per_voice=True, mix=True, sample_rate=SR),
      lambda b, r: b.push_event(event(sine_hz(500.0 + r), 0.0, 0.003)) if r else None)
check("looping sequencer", lambda: GpuBank.from_sequencer(seq(ReplayMode.Loop(0.005)), per_voice=True, mix=True, sample_rate=SR))


def slot_edit(b, r):   # the second set lands while the first fade runs: it is parked, and armed when that fade ends
    b.slot_set(1, Fade.Smooth, 0.004, sat(20 + r))
    b.slot_set(1, Fade.Power, 0.002, sat(30 + r))


check("slot with a parked update", lambda: GpuBank([slot(sat(i)) for i in range(4)], per_voice=True, mix=True, sample_rate=SR), slot_edit)


def xfade_edit(b, r):
    b.crossfade_voice(2, Fade.Smooth, 0.004, workloads.net_voice(7 + r))
    b.crossfade_voice(2, Fade.Power, 0.002, workloads.net_voice(11 + r))


check("net crossfade with a parked update", lambda: GpuBank.from_net(voice_net([workloads.net_voice(i) for i in range(5)]), per_voice=True, mix=True,
                                                                     sample_rate=SR), xfade_edit)
a, m, t = shared(0.7), shared(0.0), shared(0.0)
check("shared readers and writers", lambda: GpuBank([(var(a) * saw_hz(150.0 + 7 * i) >> monitor(m, Meter.Rms(0.01)) >> lowpass_hz(800.0, 1.0)) | timer(t)
                                                     for i in range(4)], per_voice=True, mix=True, sample_rate=SR), lambda b, r: a.set(0.1 * r))
check("shared readers", lambda: GpuBank([var(a) * sat(i) for i in range(4)], per_voice=True, mix=True, sample_rate=SR), lambda b, r: a.set(0.2 * r))

dl = lambda i: saw_hz(200.0 + i) >> (pass_() & delay(0.001)) >> lowpass_hz(900.0, 1.0)


def edits(b, r):
    c = b.clone()
    c.render_samples(100)
    del c
    b.reset()
    b.add_voice(sine_hz(300.0 + r))                               # a new class the first time: the classes are regrouped
    b.replace_voice(0, [noise().seed(9) >> lowpass_hz(500.0, 1.0), dl(5)][r % 2])   # into another class
    b.set_sample_rate([48000.0, SR][r % 2])                       # another delay length: the classes are rebuilt


check("clone, reset, add, replace, set_sample_rate", lambda: GpuBank([dl(i) for i in range(4)], per_voice=True, mix=True, sample_rate=SR), edits)
print("resources ok")
'''


def test_every_bank_form_gives_back_what_it_takes(mock_env):
    r = subprocess.run([sys.executable, "-c", SCRIPT], capture_output=True, text=True, env=mock_env, cwd=ROOT, timeout=1800)
    assert r.returncode == 0 and "resources ok" in r.stdout, (r.stdout[-2000:], r.stderr[-3000:])
