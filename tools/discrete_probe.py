"""Time the discrete kernel (CPI_FLAG_DISCRETE, DESIGN.md section 3n) against K1 (model 1) on the same batches.

    python tools/discrete_probe.py [--reps 30]

Prints ONE JSON line:
  gpu / power_limit_w     the card the numbers come from (read in the same run)
  windows10k / 100k       10 000 and 100 000 windows of 200 samples (fp64): median ms of K1 and of the discrete kernel, timed
                          alternately in the same run, windows/s, and the fp64 bound: algorithmic flops per sample (DISCRETE_FLOPS,
                          SURVEY's counting rule) x samples over the H100 SXM data-sheet 34 TFLOP/s, as a share of the measured time
  filter10k               one filter step on 10 000 filters: preintegration + K7 (propagate) + K10 (update), with each propagator
CUDA events, median of the --reps (at least 30) per-run times of each kernel, the two kernels alternating run by run.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from scan_probe import gpu_identity  # noqa: E402

FP64_FLOPS = 34e12            # H100 SXM data sheet, non-tensor fp64
# algorithmic flops per sample (add/sub/mul = 1, FMA = 2, div/sqrt = 1; sin/cos not counted), counted on the kernel's operations:
# front 453 {readings 6, |w_hat| 6, branch scalars 20, Rs / J_r / Phi_tg 105, R' 45, M 27, R^T a 15, means 18, bias Jacobians 207,
# pgg / paa 4} + covariance 1 646 {row theta 355, row v 472, row p 819}
DISCRETE_FLOPS = 453 + 1646
MODEL1_FLOPS = 5800           # SURVEY.md: V1 = 5.8 kflop/sample


def run_times(torch, fns, reps):
    """Per-run ms of every fn over reps runs, CUDA events around each call, the fns alternating run by run (after 3 warm-up rounds)."""
    for _ in range(3):
        for f in fns:
            f()
    torch.cuda.synchronize()
    ts = [[] for _ in fns]
    for _ in range(reps):
        for f, t in zip(fns, ts):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); f(); b.record()
            b.synchronize()
            t.append(a.elapsed_time(b))
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("discrete_probe needs a CUDA device")
    from cpi_b200 import capi, factor, preint, synth
    name, power = gpu_identity()
    out = dict(gpu=name, power_limit_w=power, reps=args.reps, discrete_flops_per_sample=DISCRETE_FLOPS)
    ns = 200
    S0, L0 = synth.make_windows(4096, ns, seed=1)
    for n, key in ((10000, "windows10k"), (100000, "windows100k")):
        reps = np.arange(n) % 4096
        S = torch.from_numpy(np.ascontiguousarray(S0[reps].reshape(-1, 7))).cuda()
        L = torch.from_numpy(np.ascontiguousarray(L0[reps])).cuda()
        o = torch.empty((n, 290), dtype=torch.float64, device="cuda")
        f1 = lambda: preint.preintegrate(1, S, L, synth.SIGMAS, 0, ns=ns, out=o)
        fd = lambda: preint.preintegrate(1, S, L, synth.SIGMAS, capi.FLAG_DISCRETE, ns=ns, out=o)
        t1, td = run_times(torch, (f1, fd), max(args.reps, 30))
        m1, md = float(np.median(t1)), float(np.median(td))
        bound_d = DISCRETE_FLOPS * ns * n / FP64_FLOPS * 1e3
        bound_1 = MODEL1_FLOPS * ns * n / FP64_FLOPS * 1e3
        out[key] = dict(k1_ms=m1, discrete_ms=md, k1_windows_per_s=n / m1 * 1e3, discrete_windows_per_s=n / md * 1e3,
                        discrete_fp64_bound_ms=bound_d, discrete_share_of_fp64_bound=bound_d / md, k1_share_of_fp64_bound=bound_1 / m1)
    # one filter step: preintegrate + propagate (K7) + update (K10)
    n = 10000
    S = torch.from_numpy(np.ascontiguousarray(S0[np.arange(n) % 4096].reshape(-1, 7))).cuda()
    L = torch.from_numpy(np.ascontiguousarray(L0[np.arange(n) % 4096])).cuda()
    X = torch.zeros((n, 16), dtype=torch.float64, device="cuda")
    X[:, 3] = 1.0
    X[:, 4:7], X[:, 10:13] = L[:, 0:3], L[:, 3:6]
    cov = torch.eye(15, dtype=torch.float64, device="cuda").mul(1e-4).reshape(1, 225).repeat(n, 1)
    W = torch.eye(15, dtype=torch.float64, device="cuda").reshape(1, 225).repeat(n, 1)
    def filter_step(fl):
        def f():
            r = preint.preintegrate(1, S, L, synth.SIGMAS, fl, ns=ns)
            x1, c1 = factor.propagate(1, X, cov, r, L)[:2]
            factor.update(x1, c1, W, x1)
        return f
    t1, td = run_times(torch, (filter_step(0), filter_step(capi.FLAG_DISCRETE)), max(args.reps, 30))
    step = dict(k1_ms=float(np.median(t1)), discrete_ms=float(np.median(td)))
    out["filter10k"] = step
    print(json.dumps(out))


if __name__ == "__main__":
    main()
