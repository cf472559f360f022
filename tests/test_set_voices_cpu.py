"""`set_voices` without a GPU: tests/test_gpu_set_voices.py on the CPU mock device, whose streams run as late as CUDA allows (in creation
order and in reverse), so the batch's one copy and its scatter launches are checked against the per-voice loop with the host logic that
runs on the GPU, including the launch count of a call (the copy count is read from a CUDA trace on the GPU)."""
import os
import subprocess
import sys

import pytest

from test_mock_bank_cpu import ROOT, mock_env  # noqa: F401  (the mock device build, shared with that file)


@pytest.mark.parametrize("schedule", ["late", "late-reverse"])
def test_gpu_set_voices_file_on_the_mock_device(mock_env, schedule):
    env = dict(mock_env, FDSP_MOCK_SCHEDULE=schedule)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_set_voices.py"), "-m", "gpu", "-q", "-n", "4",
                        "-p", "no:cacheprovider", "--tb=short"], capture_output=True, text=True, env=env, cwd=ROOT, timeout=1800)
    tail = r.stdout[-3000:]
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, tail
