"""Generates tests/golden/halfband_min.json: the 43 coefficients of the reference's minimum-phase halfband filter (`HALFBAND_MIN`,
src/oversample.rs), read out of the crate's source, for the f64 oversampler model of tests/delay_model.py. The decimal strings are kept
as the source writes them, with the f32 each one rounds to (what the crate's `[f32; 43]` holds).
Run: python tests/golden/gen_halfband.py <path to the fundsp crate>
"""
import json
import os
import re
import sys

import numpy as np


def parse(crate):
    src = open(os.path.join(crate, "src", "oversample.rs")).read()
    m = re.search(r"const HALFBAND_MIN_LEN: usize = (\d+);", src)
    n = int(m.group(1))
    body = re.search(r"const HALFBAND_MIN: \[f32; HALFBAND_MIN_LEN\] = \[(.*?)\];", src, re.S).group(1)
    text = re.findall(r"-?\d+\.\d+(?:e[-+]?\d+)?", body)
    assert len(text) == n, (len(text), n)
    return text


def main():
    text = parse(sys.argv[1])
    out = {"source": "fundsp 0.23 src/oversample.rs HALFBAND_MIN", "decimal": text,
           "f32_bits": [int(np.float32(t).view(np.uint32)) for t in text]}
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "halfband_min.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print(f"{len(text)} coefficients -> {path}")


if __name__ == "__main__":
    main()
