"""The PRODUCT's scalar math (csrc/dsp/libm.cuh: musl / FreeBSD msun restated for host + device, with the branch-free tanhf that sits on the
Moog ladder's recurrence) against the ORACLE's independent restatement (oracle/fo_libm.h), bit for bit over float bit patterns
(tests/cpp/libm_equiv.cpp compiles both for the host). Every 97th of the 2^32 patterns here (44 M arguments per function, about a
second); `libm_equiv 1` walks all of them (2 min on 8 cores; run when libm.cuh changes — last full run: identical for all six functions,
with sinf / cosf / tanf above 2^28 pi/2 in the restated large reduction on both sides). powf_ is compared over the three powf sets of the
scalar-math sweep (tests/golden/libm_sweep_args.h), every pair of them."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_product_libm_equals_oracle_libm(tmp_path):
    exe = str(tmp_path / "libm_equiv")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-pthread", "-w", os.path.join(ROOT, "tests", "cpp", "libm_equiv.cpp"), "-o", exe])
    r = subprocess.run([exe, "97"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.count("bit-identical") == 6, r.stdout


def test_product_powf_equals_oracle_powf(tmp_path):
    exe = str(tmp_path / "libm_equiv_pow")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-pthread", "-w", os.path.join(ROOT, "tests", "cpp", "libm_equiv_pow.cpp"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.count("bit-identical") == 3, r.stdout
    assert r.stdout.count(" 268435456 pairs") == 3, r.stdout
