"""Cost of setting many voices of a running bank: `set_voices` (one call, one copy, one scatter launch per class) against the loop of
per-voice `set` calls it replaces, on the headline bank (saw_hz(f) >> lowpass_hz(fc, q), --voices voices, mix only).

For each n in --n, every call sets Setting::center_q on voices 0..n-1:
    batch host    host time of one set_voices call (it returns before the device work)
    batch applied host time of set_voices followed by a synchronise of the bank's stream
    batch device  CUDA events on the bank's stream around the call: the copy of the staged words and the scatter launch
    kernel        the scatter kernel alone (set_columns_kernel), from torch.profiler in a pass of its own
    loop          host time of n per-voice set calls (each ends in a synchronise)
and the latency of process(64) alone and with a set_voices(n) call before every process() call. Times are medians over --reps calls.
Prints the card's name, power limit and SM clock limit with the numbers.
Usage: python tools/bench_set_voices.py [--voices 16384] [--n 1 64 1024 16384] [--reps 50]"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
P_CENTER_Q = 2


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout
        return ", ".join(s.strip() for s in out.splitlines()[0].split(","))
    except Exception:  # noqa: BLE001
        return "unknown"


def med(x):
    x = sorted(x)
    return x[len(x) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voices", type=int, default=16384)
    ap.add_argument("--n", type=int, nargs="+", default=[1, 64, 1024, 16384])
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    os.environ.setdefault("FDSP_JIT_CACHE", tempfile.mkdtemp(prefix="fdsp_set_voices_bench_"))
    from fundsp_b200 import capi, workloads
    from fundsp_b200.bank import GpuBank

    if capi.lib().fdsp_device_count() < 1:
        raise SystemExit("no CUDA device: this script measures the GPU")
    import torch

    V = a.voices
    b = GpuBank(workloads.build("saw_svf", V), per_voice=False, mix=True, sample_rate=48000.0)
    L = capi.lib()
    stream = torch.cuda.ExternalStream(L.fdsp_bank_stream(b.h))
    rng = np.random.default_rng(1)
    vals = {n: np.stack([rng.uniform(200, 8000, n), rng.uniform(0.5, 8, n)], 1).astype(np.float32) for n in a.n}
    idx = {n: np.arange(n, dtype=np.uint32) for n in a.n}
    address = ((1, 1),)
    for n in a.n:                                                    # warm-up: staging buffers, the resolved address, module load
        b.set_voices(P_CENTER_Q, vals[n], voices=idx[n], address=address)
    b.render_samples(1024)
    for _ in range(20):
        b.process(64)
    rows = []
    for n in a.n:
        host, applied, dev = [], [], []
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(a.reps):
            L.fdsp_bank_sync(b.h)
            t0 = time.perf_counter()
            b.set_voices(P_CENTER_Q, vals[n], voices=idx[n], address=address)
            host.append(time.perf_counter() - t0)
            L.fdsp_bank_sync(b.h)
            t0 = time.perf_counter()
            b.set_voices(P_CENTER_Q, vals[n], voices=idx[n], address=address)
            L.fdsp_bank_sync(b.h)
            applied.append(time.perf_counter() - t0)
            e0.record(stream)
            b.set_voices(P_CENTER_Q, vals[n], voices=idx[n], address=address)
            e1.record(stream)
            e1.synchronize()
            dev.append(e0.elapsed_time(e1) * 1e-3)
        loop = []
        for _ in range(max(1, min(a.reps, 16384 // n))):
            t0 = time.perf_counter()
            for j in range(n):
                b.set(j, P_CENTER_Q, (float(vals[n][j, 0]), float(vals[n][j, 1])), address=address)
            loop.append(time.perf_counter() - t0)
        plain, batched = [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            b.process(64)
            plain.append(time.perf_counter() - t0)
            b.set_voices(P_CENTER_Q, vals[n], voices=idx[n], address=address)
            t0 = time.perf_counter()
            b.process(64)
            batched.append(time.perf_counter() - t0)
        rows.append((n, med(host), med(applied), med(dev), med(loop), med(plain), med(batched)))
    kernel = {}
    try:
        from torch.profiler import ProfilerActivity, profile
        for n in a.n:
            L.fdsp_bank_sync(b.h)
            with profile(activities=[ProfilerActivity.CUDA]) as p:
                for _ in range(a.reps):
                    b.set_voices(P_CENTER_Q, vals[n], voices=idx[n], address=address)
                L.fdsp_bank_sync(b.h)
            ev = [e for e in p.key_averages() if "set_columns_kernel" in e.key]
            kernel[n] = ev[0].device_time_total / ev[0].count * 1e-6 if ev else None
    except Exception as e:  # noqa: BLE001
        print(f"(kernel time not measured: {e})")
    info = gpu_info()
    print(f"headline bank saw_hz >> lowpass_hz, {V} voices, Setting::center_q on voices 0..n-1, medians of {a.reps} calls, on {info}")
    print(f"{'n':>6} {'batch host':>11} {'batch applied':>14} {'batch device':>13} {'kernel':>9} {'loop':>12} {'loop/applied':>13} "
          f"{'process(64)':>12} {'with batch':>11}")
    for n, h, ap_, d, lo, pl, bt in rows:
        k = kernel.get(n)
        ks = f"{k * 1e6:7.1f}us" if k is not None else "   n/a   "
        print(f"{n:>6} {h * 1e6:9.1f}us {ap_ * 1e6:12.1f}us {d * 1e6:11.1f}us {ks} {lo * 1e6:10.1f}us {lo / ap_:12.1f}x {pl * 1e6:10.1f}us {bt * 1e6:9.1f}us")


if __name__ == "__main__":
    main()
