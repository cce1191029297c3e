"""Latency and throughput of cpi_propagate_batch (prediction with covariance).

    python tools/propagate_probe.py [--reps 50]

Prints ONE JSON line:
  gpu / power_limit_w            the card the numbers come from (read in the same run)
  windows10k_m1 / _m2            10 000 windows of 200 samples (model 1 / 2): one propagate call without and with the cross-covariance,
                                 one cpi_predict_state_batch call on the same inputs, the bytes a window moves (cov_k 1 800 B, the
                                 record, state 128 B and lin 104 B in; state 128 B and cov_k1 1 800 B out; cross 1 800 B) and the HBM
                                 bound at the H100 SXM data-sheet 3.35 TB/s
  chain5k                        the configs[4] chain (4 999 records of 20 samples at one linearisation point): cpi_scan_records plus
                                 ONE propagate call with every window anchored at x_0, against 4 999 propagate launches one after
                                 another (each from the previous prediction)
  windows1m_m1 / _m2             10^6 windows (records tiled from 4 096 distinct ones), no cross-covariance
CUDA events, median over --reps (the sequential chain: over --reps // 10 + 1).
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from scan_probe import HBM_BPS, gpu_identity, timed  # noqa: E402

REC_BYTES = {1: 290 * 8, 2: 308 * 8}


def window_bytes(model, cross):
    return 1800 + REC_BYTES[model] + 128 + 104 + 128 + 1800 + (1800 if cross else 0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("propagate_probe needs a CUDA device")
    from cpi_b200 import capi, factor, preint, synth
    lib = capi.load()
    name, power = gpu_identity()
    out = dict(gpu=name, power_limit_w=power, reps=args.reps)
    sig = synth.SIGMAS
    rng = np.random.default_rng(0)

    def covs(n):
        G = rng.normal(size=(n, 15, 15)) * 1e-2
        return torch.from_numpy((G @ G.transpose(0, 2, 1)).reshape(n, 225)).cuda()

    S, L = synth.make_windows(4096, 200, rate=200.0, first_window=93000)
    dL = torch.from_numpy(L).cuda()
    for model in (1, 2):
        pool = preint.preintegrate(model, torch.from_numpy(S).cuda(), dL, sig, 0, ns=200)
        X = torch.from_numpy(synth.make_states(pool.cpu().numpy(), L, model)[:4096]).cuda()
        C = covs(4096)
        for key, n in (("windows10k", 10_000), ("windows1m", 1_000_000)):
            idx = torch.arange(n, device="cuda") % 4096
            r, l, x, c = pool[idx].contiguous(), dL[idx].contiguous(), X[idx].contiguous(), C[idx].contiguous()
            res = dict(windows=n)
            res["propagate_ms"] = timed(torch, lambda: factor.propagate(model, x, c, r, l), args.reps)
            if key == "windows10k":
                res["propagate_cross_ms"] = timed(torch, lambda: factor.propagate(model, x, c, r, l, want_cross=True), args.reps)
                res["predict_ms"] = timed(torch, lambda: factor.predict_state(model, x, r, l), args.reps)
                res["hbm_bound_cross_ms"] = n * window_bytes(model, True) / HBM_BPS * 1e3
            res["bytes_per_window"] = window_bytes(model, False)
            res["hbm_bound_ms"] = n * window_bytes(model, False) / HBM_BPS * 1e3
            res["frac_of_hbm_bound"] = res["hbm_bound_ms"] / res["propagate_ms"]
            res["windows_per_s"] = n / res["propagate_ms"] * 1e3
            out[f"{key}_m{model}"] = res
            del r, l, x, c
            torch.cuda.empty_cache()

    # the configs[4] chain: one anchor, one linearisation point
    n = 4999
    S, L = synth.make_windows(n, 20, rate=200.0, first_window=9000)
    L[:] = L[0]
    dL = torch.from_numpy(L).cuda()
    rec = preint.preintegrate(1, torch.from_numpy(S).cuda(), dL, sig, 0, ns=20)
    o = torch.empty_like(rec)
    ws = torch.empty((int(lib.cpi_scan_records_workspace(1, n)) + 7) // 8, dtype=torch.float64, device="cuda")
    x0 = torch.from_numpy(synth.make_states(rec[:1].cpu().numpy(), L[:1], 1)[:1]).cuda()
    c0 = covs(1)
    anchor = torch.zeros(n, dtype=torch.int64, device="cuda")
    xs = torch.empty((n + 1, 16), dtype=torch.float64, device="cuda")
    cs = torch.empty((n + 1, 225), dtype=torch.float64, device="cuda")
    st = torch.cuda.current_stream()
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())

    def one_shot():
        preint.scan(1, rec, dL, group=n, out=o, workspace=ws)
        factor.propagate(1, x0, c0, o, dL, anchor=anchor)

    def sequential():
        xs[0] = x0[0]; cs[0] = c0[0]
        for j in range(n):
            lib.cpi_propagate_batch(1, 1, ptr(xs[j]), ptr(cs[j]), None, ptr(rec[j]), ptr(dL[j]), ptr(xs[j + 1]), ptr(cs[j + 1]), None,
                                    ctypes.c_void_p(st.cuda_stream))
    out["chain5k"] = dict(records=n, scan_plus_propagate_ms=timed(torch, one_shot, args.reps),
                          sequential_propagate_ms=timed(torch, sequential, args.reps // 10 + 1))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
