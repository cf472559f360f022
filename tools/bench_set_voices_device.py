"""Cost of setting many voices from values in GPU memory: `set_voices_device` (the values stay on the device, one kernel per class computes
the coefficients) against `set_voices` (values on the host, lowered there), on the headline bank (saw_hz(f) >> lowpass_hz(fc, q),
--voices voices, mix only), alternating the two calls in one run.

For each n in --n, every call sets Setting::center_q on voices 0..n-1:
    host       host time of one call (both return before the device work)
    applied    host time of the call followed by a synchronise of the bank's stream
    device     CUDA events on the bank's stream around the call
    kernel     the call's kernel alone (set_controls_kernel / set_columns_kernel), from torch.profiler in a pass of its own
Then a block loop of --iters iterations, each: a torch op writes new cutoffs for every voice, set_voices_device, process(64); its time per
iteration against the 1.33 ms a 64-sample block lasts at 48 kHz (and the same loop with the values copied to the host and set_voices).
Times are medians over --reps calls. Prints the card's name, power limit and SM clock limit with the numbers.
Usage: python tools/bench_set_voices_device.py [--voices 16384] [--n 1 64 1024 16384] [--reps 50] [--iters 1000]"""
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
BLOCK_S = 64 / 48000.0


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
    ap.add_argument("--iters", type=int, default=1000)
    a = ap.parse_args()
    os.environ.setdefault("FDSP_JIT_CACHE", tempfile.mkdtemp(prefix="fdsp_set_voices_device_bench_"))
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
    hvals = {n: np.stack([rng.uniform(200, 8000, n), rng.uniform(0.5, 8, n)], 1).astype(np.float32) for n in a.n}
    dvals = {n: torch.from_numpy(hvals[n]).cuda() for n in a.n}
    idx = {n: np.arange(n, dtype=np.uint32) for n in a.n}
    address = ((1, 1),)
    calls = {"set_voices": lambda n: b.set_voices(P_CENTER_Q, hvals[n], voices=idx[n], address=address),
             "set_voices_device": lambda n: b.set_voices_device(P_CENTER_Q, dvals[n], voices=idx[n], address=address)}
    for n in a.n:                                                    # warm-up: staging buffers, the resolved address, tables, module load
        for f in calls.values():
            f(n)
    b.render_samples(1024)
    for _ in range(20):
        b.process(64)
    torch.cuda.synchronize()
    res = {}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for n in a.n:
        t = {k: ([], [], []) for k in calls}
        for _ in range(a.reps):
            for k, f in calls.items():                              # alternating, so that both see the same machine
                host, applied, dev = t[k]
                L.fdsp_bank_sync(b.h); torch.cuda.synchronize()
                t0 = time.perf_counter(); f(n); host.append(time.perf_counter() - t0)
                L.fdsp_bank_sync(b.h); torch.cuda.synchronize()
                t0 = time.perf_counter(); f(n); L.fdsp_bank_sync(b.h); applied.append(time.perf_counter() - t0)
                e0.record(stream); f(n); e1.record(stream); e1.synchronize()
                dev.append(e0.elapsed_time(e1) * 1e-3)
        for k in calls:
            res[(k, n)] = [med(x) for x in t[k]]
    kernel = {}
    try:
        from torch.profiler import ProfilerActivity, profile
        for n in a.n:
            for k, f in calls.items():
                L.fdsp_bank_sync(b.h); torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as p:
                    for _ in range(a.reps):
                        f(n)
                    L.fdsp_bank_sync(b.h)
                name = "set_controls_kernel" if k == "set_voices_device" else "set_columns_kernel"
                ev = [e for e in p.key_averages() if name in e.key]
                kernel[(k, n)] = ev[0].device_time_total / ev[0].count * 1e-6 if ev else None
    except Exception as e:  # noqa: BLE001
        print(f"(kernel time not measured: {e})")
    # the block loop: a torch op computes every voice's cutoff, the bank takes it, one 64-sample block
    base = torch.from_numpy(hvals[max(a.n)][:, 0].copy()).cuda() if max(a.n) == V else torch.full((V,), 1000.0, device="cuda")
    cq = torch.stack([base, torch.full((V,), 2.0, device="cuda")], 1).contiguous()
    loops = {}
    for mode in ("set_voices_device", "set_voices"):
        for it in range(a.iters + 20):
            if it == 20:
                torch.cuda.synchronize(); t0 = time.perf_counter()
            cq[:, 0] = base * (1.0 + 0.5 * np.sin(0.01 * it))
            if mode == "set_voices_device":
                b.set_voices_device(P_CENTER_Q, cq, address=address)
            else:
                b.set_voices(P_CENTER_Q, cq.cpu().numpy(), address=address)
            b.process(64)
        torch.cuda.synchronize()
        loops[mode] = (time.perf_counter() - t0) / a.iters
    info = gpu_info()
    print(f"headline bank saw_hz >> lowpass_hz, {V} voices, Setting::center_q on voices 0..n-1, medians of {a.reps} calls "
          f"(set_voices and set_voices_device alternating), on {info}")
    print(f"{'n':>6} {'call':>18} {'host':>10} {'applied':>10} {'device':>10} {'kernel':>9}")
    for n in a.n:
        for k in calls:
            h, ap_, d = res[(k, n)]
            kt = kernel.get((k, n))
            ks = f"{kt * 1e6:7.1f}us" if kt is not None else "not measured"
            print(f"{n:>6} {k:>18} {h * 1e6:8.1f}us {ap_ * 1e6:8.1f}us {d * 1e6:8.1f}us {ks}")
    for mode, s in loops.items():
        print(f"block loop ({a.iters} x torch op + {mode} of {V} voices + process(64)): {s * 1e6:.1f} us per iteration, "
              f"{100.0 * s / BLOCK_S:.1f}% of the {BLOCK_S * 1e3:.2f} ms block")


if __name__ == "__main__":
    main()
