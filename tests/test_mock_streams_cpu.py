"""The ordering of the bank's device operations, checked without a GPU.

The mock device (tests/cpp/mock/cuda_runtime.h) runs each stream's work as late as CUDA allows: an operation runs only when a synchronise,
an event wait or a synchronous copy forces it, and the legacy stream is not ordered with the bank's non-blocking streams. A missing
dependency between two device operations of the runtime therefore changes a result here, where an eager mock would hide it. This file
checks the mock's rules themselves (tests/cpp/mock_streams_test.cpp) and runs the mock GPU suite a second time with the streams that one
synchronisation forces drained in reverse creation order, so that an operation pair ordered only by luck fails in one of the two runs."""
import os
import subprocess

import pytest

from test_mock_bank_cpu import ROOT, mock_env, run_gpu_suite  # noqa: F401  (the mock device build, shared with that file)

DRIVER = os.path.join(ROOT, "tests", "cpp", "mock_streams_test.cpp")


@pytest.fixture
def reverse_env(mock_env):  # noqa: F811
    return dict(mock_env, FDSP_MOCK_SCHEDULE="late-reverse")


@pytest.mark.parametrize("schedule,order", [("late", "creation"), ("late-reverse", "reverse")])
def test_stream_rules_of_the_mock_device(tmp_path, schedule, order):
    exe = str(tmp_path / "mock_streams_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "tests", "cpp", "mock"), DRIVER, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, env=dict(os.environ, FDSP_MOCK_SCHEDULE=schedule), timeout=60)
    lines = r.stdout.splitlines()
    cases = [ln for ln in lines if ln.endswith(": ok") or ": FAIL" in ln]
    assert r.returncode == 0 and len(cases) >= 25 and all(ln.endswith(": ok") for ln in cases), r.stdout + r.stderr
    assert "schedule: " + order in lines and "live: 0" in lines, r.stdout
    assert "hazard" in r.stderr   # (the negative case of the staging rule reports itself)


def test_gpu_suite_runs_with_streams_drained_in_reverse(reverse_env):
    run_gpu_suite(reverse_env)
