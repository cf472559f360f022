"""Cost of Shared readers on the GPU.

1. Throughput: a 16 384-voice bank of `var(s) * saw_hz(f) >> lowpass_hz(fc, q)` against the same bank with `var(0.5)`, rendered in the
   same process, alternating. Both read the value 0.5, so their mixes must be bit-identical; the script asserts that. The Shared bank's
   cell is set before every render, so each timed call also rewrites the readers' parameter words.
2. Latency: `process(64)` microseconds per call of a 1024-voice bank of the same voice, with a Shared (launch-per-block path, the cell
   set before every call) and with `var(0.5)` (resident process() kernel), alternating in runs of `--calls` calls.
Prints one JSON line with the card's name and power limit. Usage: python tools/bench_shared.py [--voices 16384] [--samples 48000] [--reps 7]
"""
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
    ap.add_argument("--process-voices", type=int, default=1024)
    ap.add_argument("--calls", type=int, default=2000)
    a = ap.parse_args()
    os.environ.setdefault("FDSP_JIT_CACHE", tempfile.mkdtemp(prefix="fdsp_shared_bench_"))   # nothing is compiled into the tree
    import numpy as np
    from fundsp_b200 import capi
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.prelude import lowpass_hz, saw_hz, shared, var

    if capi.lib().fdsp_device_count() < 1:
        raise SystemExit("no CUDA device: this script measures the GPU")
    sr, V, n = 48000.0, a.voices, a.samples
    s = shared(0.5)
    voice = lambda x, i: var(x) * saw_hz(50.0 + 0.05 * i) >> lowpass_hz(400.0 + (i % 61) * 20.0, 0.8 + (i % 7) * 0.1)
    bs = GpuBank([voice(s, i) for i in range(V)], per_voice=False, mix=True, sample_rate=sr)
    bc = GpuBank([voice(0.5, i) for i in range(V)], per_voice=False, mix=True, sample_rate=sr)
    for b in (bs, bc):
        b.render_samples(n)
    rates = {"shared": [], "constant": []}
    mixes = {}
    for _ in range(a.reps):
        for name, b in (("shared", bs), ("constant", bc)):
            b.reset()
            if name == "shared":
                s.set(0.25)
                s.set(0.5)                                    # (changed since the last call: the readers' words are rewritten)
            t0 = time.perf_counter()
            _, mx = b.render_samples(n)                       # synchronous: returns after the device work and the copy of the mix
            rates[name].append(V * n / (time.perf_counter() - t0) / 1e9)
            mixes[name] = mx
    assert np.array_equal(mixes["shared"], mixes["constant"]), "Shared and constant mixes differ"
    del bs, bc

    P = a.process_voices
    ps = GpuBank([voice(s, i) for i in range(P)], per_voice=False, mix=True, sample_rate=sr)
    pc = GpuBank([voice(0.5, i) for i in range(P)], per_voice=False, mix=True, sample_rate=sr)
    lat = {"shared": [], "constant": []}
    for rep in range(a.reps + 1):
        for name, b in (("shared", ps), ("constant", pc)):
            t0 = time.perf_counter()
            for k in range(a.calls):
                if name == "shared":
                    s.set(0.5 + 1e-3 * (k & 1))
                b.process(64)
            if rep:                                           # the first run of each is warm-up (and starts the resident kernel)
                lat[name].append((time.perf_counter() - t0) / a.calls * 1e6)
    del ps, pc
    name, power = gpu_info()
    med = lambda v: sorted(v)[len(v) // 2]
    stat = lambda v, d: {"median": round(med(v), d), "min": round(min(v), d), "max": round(max(v), d)}
    print(json.dumps({
        "gpu": name, "power_limit": power, "voices": V, "samples": n, "reps": a.reps,
        "shared_gsamples_per_s": stat(rates["shared"], 3), "constant_gsamples_per_s": stat(rates["constant"], 3), "mix_bit_identical": True,
        "process_voices": P, "process_calls": a.calls,
        "shared_launch_path_us_per_process64": stat(lat["shared"], 2), "constant_resident_us_per_process64": stat(lat["constant"], 2),
    }))


if __name__ == "__main__":
    main()
