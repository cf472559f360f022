"""Regenerate tests/golden/libm_sweep.json: the expected per-chunk hashes of the scalar-math sweep, from the oracle's restatements.
Run after a deliberate change to oracle/fo_libm.h, fo_math.h or fo_shapes.h (about 2 minutes on 8 cores):
    python tests/golden/gen_libm_sweep.py"""
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def build(exe):
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-pthread", "-w", "-I" + os.path.join(ROOT, "oracle"),
                           os.path.join(HERE, "gen_libm_sweep.cpp"), "-o", exe])


def run(exe, every=1, fns=()):
    out = subprocess.run([exe, "--every", str(every), *fns], check=True, capture_output=True, text=True).stdout
    return json.loads(out)


def main():
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "gen_libm_sweep")
        build(exe)
        res = run(exe)
    fixture = {"chunk_log2": res["chunk_log2"], "functions": res["functions"]}
    with open(os.path.join(HERE, "libm_sweep.json"), "w") as f:
        json.dump(fixture, f, indent=0)
        f.write("\n")
    print({k: len(v) for k, v in fixture["functions"].items()})


if __name__ == "__main__":
    sys.exit(main())
