"""Profiling driver: one workload, device-resident buffers, a few launches (run it under a profiler)."""
import argparse, sys
sys.path.insert(0, "."); sys.path.insert(0, "tests")
import torch
from fundsp_b200 import workloads
from fundsp_b200.bank import GpuBank

ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="saw_svf"); ap.add_argument("--voices", type=int, default=16384)
ap.add_argument("--n", type=int, default=16384); ap.add_argument("--mode", default="voices+mix"); ap.add_argument("--iters", type=int, default=3)
a = ap.parse_args()
pv, mx = "voices" in a.mode, "mix" in a.mode
b = GpuBank(workloads.build(a.workload, a.voices), per_voice=pv, mix=mx, sample_rate=48000.0)
c = b.voice_outputs()
out = torch.empty((a.voices * c, a.n), device="cuda", dtype=torch.float32) if pv else None
mix = torch.empty((c, a.n), device="cuda", dtype=torch.float32) if mx else None
inp = torch.zeros((max(1, b.inputs()), a.n), device="cuda", dtype=torch.float32)
if b.inputs():
    inp[0, 480:a.n // 2] = 1.0
for it in range(a.iters):
    b.render_device(a.n, inp.data_ptr() if b.inputs() else 0, a.n, out.data_ptr() if pv else 0, a.n, mix.data_ptr() if mx else 0, a.n, sync=True)
    print(f"{a.workload} V={a.voices} n={a.n} mode={a.mode}: {b.last_kernel_ms():.3f} ms  {a.voices * a.n / b.last_kernel_ms() / 1e6:.1f} Gsamples/s", flush=True)
