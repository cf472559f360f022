"""Cost of `update` on the GPU: a saw into a fixed SVF whose cutoff an update function sets every 2 ms, against the same voice without
`update` and against the audio-rate equivalent, an `lfo` into the audio-rate SVF.

    update:     update(saw_hz(f) >> lowpass_hz(1000.0, 1.0), 0.002, |t, dt, x| x.set(Setting::center(SWEEP).right()))
    plain:      saw_hz(f) >> lowpass_hz(1000.0, 1.0)
    audio-rate: (saw_hz(f) | lfo(|t| SWEEP) | dc(1.0)) >> lowpass()

and two controls that split the cost: `plain-jit`, the plain voice times 1.0, which compiles through NVRTC like the update voice rather
than being the precompiled headline class, and `update-noop`, the update voice whose statement reaches the saw, which ignores it.

SWEEP = 1000.0 + 600.0 * sin_hz(rate, t), with per-voice f and rate. The banks are timed in the same process, alternating, each
rendering --voices voices x --samples samples at 48 kHz from a reset. Prints one line per bank (median, min and max Gsample/s over
--reps runs) and the card's name, power limit and SM clock limit.
Usage: python tools/bench_update.py [--voices 16384] [--samples 48000] [--reps 7]"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SWEEP = "1000.0 + 600.0 * sin_hz(rate, t)"


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout
        return ", ".join(s.strip() for s in out.splitlines()[0].split(","))
    except Exception:  # noqa: BLE001
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voices", type=int, default=16384)
    ap.add_argument("--samples", type=int, default=48000)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    os.environ.setdefault("FDSP_JIT_CACHE", tempfile.mkdtemp(prefix="fdsp_update_bench_"))
    from fundsp_b200 import capi
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.prelude import dc, lfo, lowpass, lowpass_hz, saw_hz, update

    if capi.lib().fdsp_device_count() < 1:
        raise SystemExit("no CUDA device: this script measures the GPU")
    sr, V, n = 48000.0, a.voices, a.samples
    f = lambda i: 55.0 + (i % 500)
    rate = lambda i: 0.5 + (i % 61) / 16.0
    voices = {
        "update": lambda i: update(saw_hz(f(i)) >> lowpass_hz(1000.0, 1.0), 0.002,
                                   f"|t, dt, x| x.set(Setting::center({SWEEP}).right())", rate=rate(i)),
        "plain": lambda i: saw_hz(f(i)) >> lowpass_hz(1000.0, 1.0),
        # controls: the plain voice through the NVRTC path (a unary multiply keeps it off the precompiled headline class), and `update`
        # whose only statement the saw ignores (System's clock and update function, no target)
        "plain-jit": lambda i: saw_hz(f(i)) >> lowpass_hz(1000.0, 1.0) * 1.0,
        "update-noop": lambda i: update(saw_hz(f(i)) >> lowpass_hz(1000.0, 1.0), 0.002,
                                        f"|t, dt, x| x.set(Setting::center({SWEEP}).left().right())", rate=rate(i)),
        "audio-rate": lambda i: (saw_hz(f(i)) | lfo(f"|t| {SWEEP}", rate=rate(i)) | dc(1.0)) >> lowpass(),
    }
    banks = {k: GpuBank([mk(i) for i in range(V)], per_voice=False, mix=True, sample_rate=sr) for k, mk in voices.items()}
    for b in banks.values():                                 # warm-up: module load, staging buffers
        b.render_samples(n)
    rates = {k: [] for k in banks}
    for _ in range(a.reps):
        for k, b in banks.items():
            b.reset()
            t0 = time.perf_counter()
            b.render_samples(n)                              # synchronous: returns after the device work and the copy of the mix
            rates[k].append(V * n / (time.perf_counter() - t0) / 1e9)
    info = gpu_info()
    for k, r in rates.items():
        r = sorted(r)
        print(f"{k:11s} {V} voices x {n} samples: median {r[len(r) // 2]:.2f} Gsample/s (min {r[0]:.2f}, max {r[-1]:.2f}, {a.reps} runs) on {info}")


if __name__ == "__main__":
    main()
