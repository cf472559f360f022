"""Regenerate tests/golden/libm64_sweep.json: the expected per-chunk hashes of the f64 math sweep, from the oracle's restatement.
Run after a deliberate change to oracle/fo_libm64.h or tests/golden/libm64_sweep_args.h (under 12 minutes on 8 cores):
    python tests/golden/gen_libm64_sweep.py"""
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def build(exe):
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-pthread", "-w", "-I" + os.path.join(ROOT, "oracle"),
                           "-I" + HERE, os.path.join(HERE, "gen_libm64_sweep.cpp"), "-o", exe])


def run(exe, every=1, fns=(), chunks=()):
    extra = [a for k in chunks for a in ("--chunk", str(k))]
    out = subprocess.run([exe, "--every", str(every), *extra, *fns], check=True, capture_output=True, text=True).stdout
    return json.loads(out)


def main():
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "gen_libm64_sweep")
        build(exe)
        res = run(exe)
    fixture = {"chunk_log2": res["chunk_log2"], "functions": res["functions"]}
    with open(os.path.join(HERE, "libm64_sweep.json"), "w") as f:
        json.dump(fixture, f, indent=0)
        f.write("\n")
    print({k: len(v) for k, v in fixture["functions"].items()})


if __name__ == "__main__":
    sys.exit(main())
