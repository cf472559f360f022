"""Multi-GPU parity (SURVEY.md §8e): real GpuBank shards on >= 2 GPUs, mix-down through the C ABI's NCCL group, against the oracle's
index-order mix. Needs two devices; skipped with the reason on a one-GPU machine."""
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def test_sharded_banks_reduce_to_the_oracle_mix():
    n = _gpus()
    if n < 2:
        pytest.skip(f"needs 2 GPUs, this machine has {n}")
    world = 2 if n < 4 else 4
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1", "--master-port", str(port),
                        os.path.join(ROOT, "tests", "_gpu_group_worker.py")], capture_output=True, text=True, cwd=ROOT, timeout=200)
    assert r.returncode == 0 and r.stdout.count("rank-order ok") == 3 and "MISMATCH" not in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])


def test_group_of_one_is_a_plain_render():
    """nranks = 1 needs no NCCL: render_reduced is render."""
    import numpy as np
    from fundsp_b200 import workloads
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.parallel import BankGroup
    g = BankGroup(1, 0, None, 0)
    b = GpuBank(workloads.build("noise_svf", 50), per_voice=False, mix=True, sample_rate=48000.0)
    a = g.render_reduced(b, 1000)
    b.reset()
    _, m = b.render_samples(1000)
    assert np.array_equal(a, m) and np.abs(m).max() > 0.1
