"""`set_voices_device` without a GPU: tests/test_gpu_set_voices_device.py on the CPU mock device, whose streams run as late as CUDA allows
(in creation order and in reverse), with the values in a host buffer (the mock's device memory is host memory). The device call's checks,
its one launch per class, the order of its stream waits and the host graphs' reconciliation before every call that reads them run with
the host logic that runs on the GPU. A refused call is checked there to launch nothing and to leave the host graphs as they were (a clone,
which is built from them, equals an untouched twin's)."""
import os
import subprocess
import sys

import pytest

from test_mock_bank_cpu import ROOT, mock_env  # noqa: F401  (the mock device build, shared with that file)


@pytest.mark.parametrize("schedule", ["late", "late-reverse"])
def test_gpu_set_voices_device_file_on_the_mock_device(mock_env, schedule):
    env = dict(mock_env, FDSP_MOCK_SCHEDULE=schedule)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_set_voices_device.py"), "-m", "gpu", "-q", "-n", "8",
                        "-p", "no:cacheprovider", "--tb=short"], capture_output=True, text=True, env=env, cwd=ROOT, timeout=2400)
    tail = r.stdout[-3000:]
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, tail
