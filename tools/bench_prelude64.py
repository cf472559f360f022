"""Throughput of prelude64 (f64 filter state) against prelude32, on the GPU.

Two workloads, `saw_hz(f) >> lowpass_hz(fc, q)` and `noise() >> resonator_hz(center, q)`, each as a 16 384-voice bank built from
`fundsp_b200.prelude` (f32 state) and from `fundsp_b200.prelude64` (f64 state), with per-voice parameters (one class per bank). The four
banks are rendered in the same process, alternating, from a reset each time. The classes compile into a fresh temporary NVRTC cache, removed at the end, so nothing is written
into the tree or left behind. Prints one JSON line with the card's name and power limit.
Usage: python tools/bench_prelude64.py [--voices 16384] [--samples 48000] [--reps 7]"""
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
    with tempfile.TemporaryDirectory(prefix="fdsp_p64_bench_") as cache:   # removed with the compiled modules when the run ends
        os.environ["FDSP_JIT_CACHE"] = cache
        run(a)


def run(a):
    from fundsp_b200 import capi
    from fundsp_b200 import prelude as p32
    from fundsp_b200 import prelude64 as p64
    from fundsp_b200.bank import GpuBank

    if capi.lib().fdsp_device_count() < 1:
        raise SystemExit("no CUDA device: this script measures the GPU")
    sr, V, n = 48000.0, a.voices, a.samples
    work = {"saw_lowpass": lambda P, i: P.saw_hz(50.0 + 0.05 * i).phase(0.0) >> P.lowpass_hz(300.0 + 0.2 * i, 0.7 + (i % 13) / 10.0),
            "noise_resonator": lambda P, i: P.noise().seed(i) >> P.resonator_hz(200.0 + 0.25 * i, 5.0 + (i % 13))}
    banks = {f"{pk}_{wk}": GpuBank([w(P, i) for i in range(V)], per_voice=False, mix=True, sample_rate=sr)
             for wk, w in work.items() for pk, P in (("prelude32", p32), ("prelude64", p64))}
    for b in banks.values():                                 # warm-up: module load, staging buffers
        b.render_samples(n)
    rates = {k: [] for k in banks}
    for _ in range(a.reps):
        for k, b in banks.items():
            b.reset()
            t0 = time.perf_counter()
            b.render_samples(n)                              # synchronous: returns after the device work and the copy of the mix
            rates[k].append(V * n / (time.perf_counter() - t0) / 1e9)
    name, power = gpu_info()
    med = lambda v: sorted(v)[len(v) // 2]
    print(json.dumps({
        "gpu": name, "power_limit": power, "voices": V, "samples": n, "reps": a.reps,
        **{f"{k}_gsamples_per_s": {"median": round(med(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)} for k, v in rates.items()},
        "classes": {k: b.classes()[0]["signature"][-40:] for k, b in banks.items()},
    }))


if __name__ == "__main__":
    main()
