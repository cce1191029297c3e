#!/usr/bin/env python
"""Bitwise comparison of two `bench.py --dump-outputs` directories: every .npy of A must exist in B with identical bytes.
Prints one line per file and exits non-zero on any difference.    python tools/compare_outputs.py DIR_A DIR_B"""
import os
import sys

import numpy as np


def main(a, b):
    names = sorted(f for f in os.listdir(a) if f.endswith(".npy"))
    if not names:
        print(f"no .npy files in {a}")
        return 1
    bad = 0
    for f in names:
        pa, pb = os.path.join(a, f), os.path.join(b, f)
        if not os.path.exists(pb):
            print(f"{f}: missing in {b}")
            bad += 1
            continue
        x, y = np.load(pa), np.load(pb)
        same = x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()
        if same:
            print(f"{f}: identical ({x.dtype} {x.shape})")
        else:
            n = int(np.sum(x.view(np.uint8) != y.view(np.uint8))) if x.shape == y.shape and x.dtype == y.dtype else -1
            print(f"{f}: DIFFERENT ({x.dtype} {x.shape} vs {y.dtype} {y.shape}, {n} bytes differ)")
            bad += 1
    return 1 if bad else 0


if __name__ == "__main__":
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    sys.exit(main(sys.argv[1], sys.argv[2]))
