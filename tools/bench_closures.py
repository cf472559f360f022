"""Cost of a closure node against the built-in node that computes the same arithmetic, on the GPU.

A 16 384-voice bank of `saw_hz(f) >> map_("|x| tanh(x[0] * drive)", 1, 1, drive=d)` and one of `saw_hz(f) >> shape(Tanh(d))` are timed
in the same process, alternating, with per-voice f and d and the saw phase fixed at 0 (its default phase is hashed from the node IDs,
which differ: Map is ID 5, Shaper ID 42). Both then run `tanhf_(x * d)` on the same saw, so their mixes must be bit-identical;
the script asserts that. It also reports how long NVRTC takes to compile the closure class from a cold cache (a fresh temporary cache
directory, so nothing is written into the tree). Prints one JSON line with the card's name and power limit.
Usage: python tools/bench_closures.py [--voices 16384] [--samples 48000] [--reps 7]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception:  # noqa: BLE001
        return "unknown", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voices", type=int, default=16384)
    ap.add_argument("--samples", type=int, default=48000)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    cache = tempfile.mkdtemp(prefix="fdsp_closure_bench_")
    os.environ["FDSP_JIT_CACHE"] = cache                     # read by the library when it compiles: every class below starts cold
    from fundsp_b200 import capi
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.prelude import map_, saw_hz, shape, Tanh

    if capi.lib().fdsp_device_count() < 1:
        raise SystemExit("no CUDA device: this script measures the GPU")
    sr, V, n = 48000.0, a.voices, a.samples
    f = lambda i: 50.0 + 0.05 * i
    d = lambda i: 0.5 + (i % 97) / 32.0
    closure = lambda i: saw_hz(f(i)).phase(0.0) >> map_("|x| tanh(x[0] * drive)", 1, 1, drive=d(i))
    builtin = lambda i: saw_hz(f(i)).phase(0.0) >> shape(Tanh(d(i)))
    t0 = time.perf_counter()
    bc = GpuBank([closure(i) for i in range(V)], per_voice=False, mix=True, sample_rate=sr)
    t_closure_bank = time.perf_counter() - t0
    t0 = time.perf_counter()
    bb = GpuBank([builtin(i) for i in range(V)], per_voice=False, mix=True, sample_rate=sr)
    t_builtin_bank = time.perf_counter() - t0
    # NVRTC alone, for one unit of a closure class nothing has compiled yet (another literal: another class)
    sig = capi.NodeHandle(saw_hz(50.0) >> map_("|x| tanh(x[0] * drive * 1.5)", 1, 1, drive=1.0)).signature()
    t0 = time.perf_counter()
    try:
        capi.jit_precompile(sig, 2, 1)
        t_nvrtc = round(time.perf_counter() - t0, 3)
    except capi.FdspError as e:                               # a build without NVRTC (the CPU mock device of tests/)
        t_nvrtc = str(e)

    for b in (bc, bb):                                       # warm-up: module load, staging buffers
        b.render_samples(n)
    rates = {"closure": [], "builtin": []}
    mixes = {}
    for _ in range(a.reps):
        for name, b in (("closure", bc), ("builtin", bb)):
            b.reset()
            t0 = time.perf_counter()
            _, mx = b.render_samples(n)                      # synchronous: returns after the device work and the copy of the mix
            dt = time.perf_counter() - t0
            rates[name].append(V * n / dt / 1e9)
            mixes[name] = mx
    import numpy as np
    assert np.array_equal(mixes["closure"], mixes["builtin"]), "closure and built-in mixes differ"
    name, power = gpu_info()
    med = lambda v: sorted(v)[len(v) // 2]
    print(json.dumps({
        "gpu": name, "power_limit": power, "voices": V, "samples": n, "reps": a.reps,
        "closure_gsamples_per_s": {"median": round(med(rates["closure"]), 3), "min": round(min(rates["closure"]), 3), "max": round(max(rates["closure"]), 3)},
        "builtin_gsamples_per_s": {"median": round(med(rates["builtin"]), 3), "min": round(min(rates["builtin"]), 3), "max": round(max(rates["builtin"]), 3)},
        "mix_bit_identical": True,
        "closure_bank_create_s_cold": round(t_closure_bank, 3), "builtin_bank_create_s_cold": round(t_builtin_bank, 3),
        "closure_nvrtc_compile_s_cold": t_nvrtc, "closure_signature": sig,
    }))


if __name__ == "__main__":
    main()
