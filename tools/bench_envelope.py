"""Cost of a text envelope against the callback envelope with the same function, on the GPU.

A bank of `lfo(text) >> sine()` and one of `lfo(callback) >> sine()` are timed in the same process, alternating. The closure is a
sawtooth LFO of per-voice rate and depth, arithmetic only:
    |t| { let u = t * rate; 300.0 + depth * (u - floor(u)) }
and the callback computes the same f32 operations in numpy float32, so within the callback's horizon the two mixes must be
bit-identical; the script asserts that. The timed callback bank has a horizon just past the render, the shortest one that covers it.

It also reports what each form costs to build. The text form stores no sampled values: its parameter words are its captures and
interval, at any render length, and it does not call back into Python. The callback form is called once per voice and sample point
up to its horizon, on the host, and stores one parameter word per point; both grow with the horizon. Banks of the callback form at
10 s and 60 s horizons take minutes of Python at 16 384 voices, so they are built with --create-voices voices (default 256); their
parameter bytes for the full bank are those words per voice times --voices, since every voice of the class has the same words.
Prints one JSON line with the card's name and power limit.
Usage: python tools/bench_envelope.py [--voices 16384] [--samples 48000] [--reps 7] [--create-voices 256]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TEXT = "|t| { let u = t * rate; 300.0 + depth * (u - floor(u)) }"


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception:  # noqa: BLE001
        return "unknown", "unknown"


class SawLfo:
    """The numpy float32 form of TEXT for voices 0..V-1. Every voice samples at the same points (they share the node's hash), so the
    values at a point are computed for all voices at once, elementwise, and each voice's callback reads its own."""

    def __init__(self, rate, depth):
        self.rate, self.depth, self.at = np.float32(rate), np.float32(depth), {}

    def values(self, t):
        v = self.at.get(t)
        if v is None:
            u = np.float32(t) * self.rate
            v = self.at[t] = (np.float32(300.0) + self.depth * (u - np.floor(u))).astype(np.float32).tolist()
        return v

    def voice(self, i):
        return lambda t: self.values(t)[i]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voices", type=int, default=16384)
    ap.add_argument("--samples", type=int, default=48000)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--create-voices", type=int, default=256)
    a = ap.parse_args()
    os.environ["FDSP_JIT_CACHE"] = tempfile.mkdtemp(prefix="fdsp_envelope_bench_")   # every class below compiles from a cold cache
    from fundsp_b200 import capi
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.prelude import lfo, sine

    if capi.lib().fdsp_device_count() < 1:
        raise SystemExit("no CUDA device: this script measures the GPU")
    sr, V, n = 48000.0, a.voices, a.samples
    rate = np.array([0.5 + (i % 61) / 16.0 for i in range(V)], np.float32)
    depth = np.array([50.0 + (i % 37) for i in range(V)], np.float32)
    text = lambda i: lfo(TEXT, rate=float(rate[i]), depth=float(depth[i])) >> sine()

    def callback_bank(nv, horizon):
        f = SawLfo(rate[:nv], depth[:nv])
        return GpuBank([lfo(f.voice(i), 1, horizon) >> sine() for i in range(nv)], per_voice=False, mix=True, sample_rate=sr)

    def build(make):
        t0 = time.perf_counter()
        b = make()
        dt = time.perf_counter() - t0
        return b, dt, sum(c["voices"] * c["param_words"] * 4 for c in b.classes()), b.classes()[0]["param_words"]

    mk_text = lambda nv: lambda: GpuBank([text(i) for i in range(nv)], per_voice=False, mix=True, sample_rate=sr)
    bt, t_text_cold, text_bytes, _ = build(mk_text(V))
    _, t_text_warm, _, _ = build(mk_text(V))
    horizon = n / sr * 1.01
    bc, t_cb, cb_bytes, _ = build(lambda: callback_bank(V, horizon))

    for b in (bt, bc):                                       # warm-up: module load, staging buffers
        b.render_samples(n)
    rates = {"text": [], "callback": []}
    mixes = {}
    for _ in range(a.reps):
        for name, b in (("text", bt), ("callback", bc)):
            b.reset()
            t0 = time.perf_counter()
            _, mx = b.render_samples(n)                      # synchronous: returns after the device work and the copy of the mix
            dt = time.perf_counter() - t0
            rates[name].append(V * n / dt / 1e9)
            mixes[name] = mx
    assert np.abs(mixes["text"]).max() > 0.1
    assert np.array_equal(mixes["text"], mixes["callback"]), "text and callback mixes differ within the horizon"
    del bc

    nc = min(a.create_voices, V)
    create = {}
    for hz in (10.0, 60.0):
        _, dt, _, words = build(lambda: callback_bank(nc, hz))
        create[f"callback_horizon_{int(hz)}s"] = {"create_s": round(dt, 3), "create_voices": nc, "param_words_per_voice": words,
                                                  "param_bytes_full_bank": words * 4 * V}
    _, dt, _, words = build(mk_text(nc))
    create["text"] = {"create_s_warm": round(dt, 3), "create_voices": nc, "param_words_per_voice": words, "param_bytes_full_bank": text_bytes}

    name, power = gpu_info()
    med = lambda v: sorted(v)[len(v) // 2]
    stat = lambda v: {"median": round(med(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}
    print(json.dumps({
        "gpu": name, "power_limit": power, "voices": V, "samples": n, "reps": a.reps, "closure": TEXT,
        "text_gsamples_per_s": stat(rates["text"]), "callback_gsamples_per_s": stat(rates["callback"]),
        "mix_bit_identical_within_horizon": True,
        "full_bank": {"text_create_s_cold": round(t_text_cold, 3), "text_create_s_warm": round(t_text_warm, 3), "text_param_bytes": text_bytes,
                      "callback_horizon_s": round(horizon, 4), "callback_create_s": round(t_cb, 3), "callback_param_bytes": cb_bytes},
        "create_by_horizon": create,
    }))


if __name__ == "__main__":
    main()
