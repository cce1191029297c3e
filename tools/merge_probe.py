"""Latency of one long window preintegrated in segments and merged, and throughput of cpi_merge_records against the HBM bound.

    python tools/merge_probe.py [--reps 50]

Prints ONE JSON line:
  gpu / power_limit_w            the card the numbers come from (read in the same run)
  window[N]                      one window of N samples: one-shot cpi_preintegrate_batch latency, and for S segments the latency of
                                 one CSR cpi_preintegrate_batch over the S segments + one cpi_merge_records (CUDA events, median over
                                 --reps), with the merged record's worst relative error against the one-shot record (means / Jacobians
                                 and P, whole-matrix)
  pairs[K]                       K record pairs merged in one call: time, bytes moved (2 x (2320 + 104) read + 2320 written per pair) and
                                 the HBM bound at the H100 SXM data-sheet 3.35 TB/s
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12          # H100 SXM data sheet
BYTES_PER_PAIR = 2 * (2320 + 104) + 2320


def gpu_identity():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvidia-smi query failed: " + r.stderr)
    name, power = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return name, float(power)


def timed(torch, fn, reps):
    """Median ms of fn() over reps, CUDA events around each call (after 3 warm-up calls)."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def rel_errors(got, ref):
    from cpi_b200.capi import REC
    e = {}
    for k in ("R", "alpha", "beta", "J_q", "J_a", "J_b", "H_a", "H_b", "P"):
        a, b = REC[k]
        e[k] = float(np.linalg.norm(got[a:b] - ref[a:b]) / max(np.linalg.norm(ref[a:b]), 1e-300))
    return {"means_jac": max(v for k, v in e.items() if k != "P"), "P": e["P"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("merge_probe needs a CUDA device")
    from cpi_b200 import preint, synth
    name, power = gpu_identity()
    out = dict(gpu=name, power_limit_w=power, reps=args.reps, window={}, pairs={})
    sig = synth.SIGMAS
    for N in (100, 1000, 10000):
        S, L = synth.make_windows(1, N, rate=200.0, first_window=90000, special=False)
        dS, dL = torch.from_numpy(S).cuda(), torch.from_numpy(L).cuda()
        one = preint.preintegrate(1, dS, dL, sig, 0, ns=N)
        row = dict(one_shot_ms=timed(torch, lambda: preint.preintegrate(1, dS, dL, sig, 0, ns=N, out=one), args.reps))
        ref = one.cpu().numpy()[0]
        for nseg in (4, 16, 64):
            cuts = np.linspace(0, N, nseg + 1).round().astype(np.int64)
            off = torch.from_numpy(cuts).cuda()
            dLs = dL.repeat(nseg, 1).contiguous()
            seg = torch.empty((nseg, 290), dtype=torch.float64, device="cuda")
            m = torch.empty((1, 290), dtype=torch.float64, device="cuda")

            def run():
                preint.preintegrate(1, dS, dLs, sig, 0, offsets=off, out=seg)
                preint.merge(1, seg, dLs, group=nseg, out=m)
            ms = timed(torch, run, args.reps)
            row[f"S{nseg}_ms"] = ms
            row[f"S{nseg}_err"] = rel_errors(m.cpu().numpy()[0], ref)
        out["window"][str(N)] = row
    # merge throughput: records tiled from 4096 distinct ones on the device
    S, L = synth.make_windows(4096, 20, rate=200.0, first_window=91000)
    pool = preint.preintegrate(1, torch.from_numpy(S).cuda(), torch.from_numpy(L).cuda(), sig, 0, ns=20)
    dLp = torch.from_numpy(L).cuda()
    for K in (10_000, 1_000_000):
        idx = torch.arange(2 * K, device="cuda") % 4096
        rec, lin = pool[idx].contiguous(), dLp[idx].contiguous()
        o = torch.empty((K, 290), dtype=torch.float64, device="cuda")
        ms = timed(torch, lambda: preint.merge(1, rec, lin, group=2, out=o), args.reps)
        bound_ms = K * BYTES_PER_PAIR / HBM_BPS * 1e3
        out["pairs"][str(K)] = dict(ms=ms, bytes=K * BYTES_PER_PAIR, hbm_bound_ms=bound_ms, frac_of_hbm_bound=bound_ms / ms,
                                    pairs_per_s=K / ms * 1e3)
        del rec, lin, o
    print(json.dumps(out))


if __name__ == "__main__":
    main()
