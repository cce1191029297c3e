"""Latency and throughput of cpi_state_update_batch (the filter's measurement update, kernel K10).

    python tools/update_probe.py [--reps 50]

Prints ONE JSON line:
  gpu / power_limit_w      the card the numbers come from (read in the same run)
  filters10k / filters1m   one update of 10 000 / 10^6 filters (dense random W, a gate per filter), against the HBM bound of the bytes
                           a filter moves: 3 864 in (x 128, Sigma 1 800, W 1 800, x_bar 128, gate 8) and 1 940 out (x+ 128, Sigma+
                           1 800, nis 8, applied 4) at the H100 SXM data-sheet 3.35 TB/s
  filter_step10k           one filter step of 10 000 filters over windows of 200 samples: preintegration (K1), cpi_propagate_batch
                           (K7) and the update (K10), and each part
  chains10k                the same update of 10 000 filters through existing entry points, as single-state chains (the prior
                           Sigma^-1 + W and rhs -W d given): chains_assemble + chains_solve + chains_covariance + retract
CUDA events, median over --reps.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from scan_probe import HBM_BPS, gpu_identity, timed  # noqa: E402

BYTES_IN, BYTES_OUT = 128 + 1800 + 1800 + 128 + 8, 128 + 1800 + 8 + 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("update_probe needs a CUDA device")
    from cpi_b200 import capi, factor, preint, synth
    lib = capi.load()
    name, power = gpu_identity()
    out = dict(gpu=name, power_limit_w=power, reps=args.reps)
    rng = np.random.default_rng(0)
    f64 = dict(dtype=torch.float64, device="cuda")

    def inputs(n):
        m = min(n, 4096)
        G = rng.normal(size=(m, 15, 15))
        S = G @ G.transpose(0, 2, 1) * 1e-4 + np.eye(15) * 1e-6
        H = rng.normal(size=(m, 15, 15))
        W = H @ H.transpose(0, 2, 1) * 1e2
        x = np.zeros((m, 16)); x[:, 3] = 1.0; x[:, 4:] = rng.normal(size=(m, 12)) * 1e-2
        xb = x.copy(); xb[:, 4:] += rng.normal(size=(m, 12)) * 1e-2
        rep = lambda a: torch.from_numpy(np.ascontiguousarray(a.reshape(m, -1))).cuda().repeat((n + m - 1) // m, 1)[:n].contiguous()
        return rep(x), rep(S), rep(W), rep(xb), torch.full((n,), 16.0, **f64)

    def raw(n, x, c, W, xb, g):
        xo, co, nis = torch.empty((n, 16), **f64), torch.empty((n, 225), **f64), torch.empty(n, **f64)
        ap_ = torch.empty(n, dtype=torch.int32, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        p = lambda t: t.data_ptr()
        return lambda: capi.check(lib.cpi_state_update_batch(n, p(x), p(c), p(W), p(xb), p(g), p(xo), p(co), p(nis), p(ap_), st))

    for key, n in (("filters10k", 10_000), ("filters1m", 1_000_000)):
        x, c, W, xb, g = inputs(n)
        ms = timed(torch, raw(n, x, c, W, xb, g), args.reps)
        b = n * (BYTES_IN + BYTES_OUT)
        out[key] = dict(ms=ms, bytes=b, hbm_bound_ms=b / HBM_BPS * 1e3, hbm_fraction=b / HBM_BPS * 1e3 / ms)
        del x, c, W, xb, g
        torch.cuda.empty_cache()

    # one filter step: K1 + K7 + K10 on 10 000 filters over windows of 200 samples
    n, ns = 10_000, 200
    Sw, Lw = synth.make_windows(n, ns, rate=200.0, first_window=93000)
    dS, dL = torch.from_numpy(Sw).cuda(), torch.from_numpy(Lw).cuda()
    rec = preint.preintegrate(1, dS, dL, synth.SIGMAS, 0, ns=ns)
    X = torch.from_numpy(synth.make_states(rec.cpu().numpy(), Lw, 1)[:n]).cuda()
    _, c, W, _, g = inputs(n)
    x1, c1, _ = factor.propagate(1, X, c, rec, dL)
    xb = x1.clone(); xb[:, 13:16] += 0.01
    step = dict(
        k1=timed(torch, lambda: preint.preintegrate(1, dS, dL, synth.SIGMAS, 0, ns=ns), args.reps),
        k7=timed(torch, lambda: factor.propagate(1, X, c, rec, dL), args.reps),
        k10=timed(torch, lambda: factor.update(x1, c1, W, xb, gate=g), args.reps))

    def filter_step():
        r = preint.preintegrate(1, dS, dL, synth.SIGMAS, 0, ns=ns)
        xp, cp, _ = factor.propagate(1, X, c, r, dL)
        factor.update(xp, cp, W, xb, gate=g)
    step["total"] = timed(torch, filter_step, args.reps)
    out["filter_step10k"] = step

    # the same update through the chain entry points, single-state chains
    Si = torch.linalg.inv(c.view(n, 15, 15))
    info = (Si + W.view(n, 15, 15)).reshape(n, 225).contiguous()
    rhs = torch.zeros((n, 15), **f64)
    e0 = torch.empty((0, 225), **f64)
    e1 = torch.empty((0, 15), **f64)
    ws = torch.empty((int(lib.cpi_imu_chains_marginals_workspace(n, n)) + 7) // 8, **f64)

    def chains():
        D, E, r = factor.chains_assemble(e0, e0, e0, e1, e1, 1, 0.0, info, rhs, n_chains=n)
        dx = factor.chains_solve(D, E, r, 1, n_chains=n)
        factor.chains_covariance(D, E, 1, n_chains=n, workspace=ws)
        factor.retract(x1, dx)
    out["chains10k"] = dict(ms=timed(torch, chains, args.reps), k10_ms=step["k10"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
