"""Latency and throughput of cpi_scan_records (the record from a group's first keyframe to every later one).

    python tools/scan_probe.py [--reps 50]

Prints ONE JSON line:
  gpu / power_limit_w            the card the numbers come from (read in the same run)
  chain5k                        the configs[4] chain (4 999 records of 20 samples, one group, each record at its own linearisation
                                 point): one cpi_scan_records call; the dead reckoning it replaces, 4 999 cpi_predict_state_batch
                                 launches one after another (one state each); one cpi_merge_records call on the same group (the last
                                 prefix only).  CUDA events, median over --reps (the sequential chain: over --reps // 10 + 1)
  fixed_lag                      10 000 groups of 30 records (fixed-lag-sized windows) in one call
  bulk                           10^6 records in groups of 64: time, bytes moved (2 424 B read, 2 320 B written per fp64 record) and
                                 the HBM bound at the H100 SXM data-sheet 3.35 TB/s
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12          # H100 SXM data sheet
BYTES_PER_RECORD = (2320 + 104) + 2320


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("scan_probe needs a CUDA device")
    from cpi_b200 import capi, preint, synth
    lib = capi.load()
    name, power = gpu_identity()
    out = dict(gpu=name, power_limit_w=power, reps=args.reps)
    sig = synth.SIGMAS
    # the configs[4] chain as one group
    n = 4999
    S, L = synth.make_windows(n, 20, rate=200.0, first_window=9000)
    dL = torch.from_numpy(L).cuda()
    rec = preint.preintegrate(1, torch.from_numpy(S).cuda(), dL, sig, 0, ns=20)
    o = torch.empty_like(rec)
    ws = torch.empty((int(lib.cpi_scan_records_workspace(1, n)) + 7) // 8, dtype=torch.float64, device="cuda")
    m = torch.empty((1, 290), dtype=torch.float64, device="cuda")
    x0 = torch.from_numpy(synth.make_states(rec[:1].cpu().numpy(), L[:1], 1)[:1]).cuda()
    xs = torch.empty((n + 1, 16), dtype=torch.float64, device="cuda")
    st = torch.cuda.current_stream()

    ptr = lambda t: ctypes.c_void_p(t.data_ptr())

    def sequential():
        xs[0] = x0[0]
        for j in range(n):
            lib.cpi_predict_state_batch(1, 1, ptr(xs[j]), ptr(rec[j]), ptr(dL[j]), ptr(xs[j + 1]), ctypes.c_void_p(st.cuda_stream))
    out["chain5k"] = dict(records=n,
                          scan_ms=timed(torch, lambda: preint.scan(1, rec, dL, group=n, out=o, workspace=ws), args.reps),
                          sequential_predict_ms=timed(torch, sequential, args.reps // 10 + 1),
                          merge_ms=timed(torch, lambda: preint.merge(1, rec, dL, group=n, out=m), args.reps))
    # fixed-lag windows and the bulk rate: records tiled from 4096 distinct ones on the device
    S, L = synth.make_windows(4096, 20, rate=200.0, first_window=91000)
    pool = preint.preintegrate(1, torch.from_numpy(S).cuda(), torch.from_numpy(L).cuda(), sig, 0, ns=20)
    dLp = torch.from_numpy(L).cuda()
    for key, groups, g in (("fixed_lag", 10_000, 30), ("bulk", 15_625, 64)):
        K = groups * g
        idx = torch.arange(K, device="cuda") % 4096
        r, l = pool[idx].contiguous(), dLp[idx].contiguous()
        o = torch.empty_like(r)
        ws = torch.empty((int(lib.cpi_scan_records_workspace(groups, K)) + 7) // 8, dtype=torch.float64, device="cuda")
        ms = timed(torch, lambda: preint.scan(1, r, l, group=g, out=o, workspace=ws), args.reps)
        bound_ms = K * BYTES_PER_RECORD / HBM_BPS * 1e3
        out[key] = dict(groups=groups, group=g, records=K, ms=ms, records_per_s=K / ms * 1e3, bytes=K * BYTES_PER_RECORD,
                        hbm_bound_ms=bound_ms, frac_of_hbm_bound=bound_ms / ms)
        del r, l, o, ws
    print(json.dumps(out))


if __name__ == "__main__":
    main()
