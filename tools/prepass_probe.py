"""Time K1 (model 1, fp64) at 10 000 windows x 200 samples on the bench's synthetic data with and without its special windows.

    python tools/prepass_probe.py [--reps 30] [--rounds 3]

`synth.make_windows(..., special=True)` (what bench.py times) puts 1 % of the windows wholly into the small-|w| Taylor branch of the
scalar pre-pass (CpiV1.h:101), plus a few exact-zero-w and dt = 0 windows; `special=False` has none.  A warp holding one such window
runs both coefficient branches of the pre-pass in every group, so the difference of the two times bounds what removing that
divergence can win.  The two batches alternate run by run, in --rounds rounds of --reps runs each.

Prints ONE JSON line: the card (name, power limit, max SM clock, read in the same run), each round's median ms of both batches, and
the smallest and largest per-round difference of the medians.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from discrete_probe import run_times  # noqa: E402
from scan_probe import gpu_identity  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import subprocess

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("prepass_probe needs a CUDA device")
    from cpi_b200 import preint, synth
    name, power = gpu_identity()
    try:
        sm_clock = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        sm_clock = None
    n, ns = 10_000, 200
    fns = []
    for special in (True, False):
        S, L = synth.make_windows(n, ns, rate=200.0, special=special)
        S = torch.from_numpy(np.ascontiguousarray(S.reshape(-1, 7))).cuda()
        L = torch.from_numpy(L).cuda()
        o = torch.empty((n, 290), dtype=torch.float64, device="cuda")
        fns.append(lambda S=S, L=L, o=o: preint.preintegrate(1, S, L, synth.SIGMAS, 0, ns=ns, out=o))
    rounds = []
    for _ in range(args.rounds):
        ts, tn = run_times(torch, fns, args.reps)
        ms, mn = float(np.median(ts)), float(np.median(tn))
        rounds.append(dict(special_ms=ms, plain_ms=mn, special_minus_plain_ms=ms - mn))
    d = [r["special_minus_plain_ms"] for r in rounds]
    print(json.dumps(dict(gpu=name, power_limit_w=power, max_sm_clock=sm_clock, windows=n, samples=ns, reps=args.reps, rounds=rounds,
                          special_minus_plain_ms=dict(min=min(d), max=max(d)))))


if __name__ == "__main__":
    main()
