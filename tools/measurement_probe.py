"""Timing of the attitude-dependent measurements (DESIGN.md section 3l).

    python tools/measurement_probe.py [--reps 50]

Prints ONE JSON line:
  gpu / power_limit_w          the card the numbers come from (read in the same run)
  k12_10k / k12_1m             cpi_imu_measurements_linearize on 10^4 / 10^6 measurements (kinds cycled, 4 measurements per state),
                               against the HBM bound of the bytes a measurement moves: 172 in (kind 4, index 8, state 128, z 24,
                               S 72, aux 24, at most: states are shared) and 1 928 out (info 1 800, rhs 120, f 8) at the H100 SXM
                               data-sheet 3.35 TB/s
  k10_10k / k11_10k            raw kernel calls on 10 000 filters: cpi_state_update_batch with a position fix, and
                               cpi_state_update_measurements_batch with one lever-arm GNSS fix each (the CSR built beforehand)
  lm_priors / lm_lever_arm     ten rounds of chains_lm on 10 000 chains x 30 states with 20 000 position state priors, and with
                               20 000 lever-arm GNSS fixes in their place
CUDA events, median over --reps (chains_lm: over max(--reps // 10, 3)).
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

BYTES_IN, BYTES_OUT = 4 + 8 + 128 + 24 + 72 + 24, 1800 + 120 + 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("measurement_probe needs a CUDA device")
    from cpi_b200 import capi, factor, preint, synth
    lib = capi.load()
    p = factor._tptr
    dev = torch.device("cuda")
    f64 = dict(dtype=torch.float64, device=dev)
    rng = np.random.default_rng(0)
    name, power = gpu_identity()
    out = {"gpu": name, "power_limit_w": power}

    def unit_states(n):
        x = torch.zeros((n, 16), **f64)
        q = torch.randn((n, 4), **f64)
        x[:, 0:4] = q / q.norm(dim=1, keepdim=True)
        x[:, 4:16] = torch.randn((n, 12), **f64)
        return x

    for M, key in ((10_000, "k12_10k"), (1_000_000, "k12_1m")):
        N = M // 4
        X = unit_states(N)
        idx = torch.from_numpy(rng.integers(0, N, M)).to(dev)
        kind = torch.from_numpy((np.arange(M) % 3 + 1).astype(np.int32)).to(dev)
        z, si, aux = torch.randn((M, 3), **f64), torch.randn((M, 9), **f64), torch.randn((M, 3), **f64)
        info, rhs, f = torch.empty((M, 225), **f64), torch.empty((M, 15), **f64), torch.empty(M, **f64)
        ms = timed(torch, lambda: capi.check(lib.cpi_imu_measurements_linearize(M, p(kind), p(idx), p(X), p(z), p(si), p(aux), p(info),
                                                                                 p(rhs), p(f), None)), args.reps)
        bound = M * (BYTES_IN + BYTES_OUT) / HBM_BPS * 1e3
        out[key] = {"ms": ms, "hbm_bound_ms": bound, "share_of_bound": bound / ms}
    n = 10_000
    X = unit_states(n)
    rc = torch.randn((n, 15, 15), **f64)
    C = (rc @ rc.transpose(1, 2) * 1e-4 + torch.eye(15, **f64) * 1e-4).transpose(1, 2).reshape(n, 225).contiguous()
    W = torch.zeros((n, 15, 15), **f64); W[:, 12:15, 12:15] = torch.eye(3, **f64) * 1e4
    W = W.reshape(n, 225).contiguous()
    xb = X.clone(); xb[:, 13:16] += 0.01
    offs = torch.arange(n + 1, dtype=torch.int64, device=dev)
    kind = torch.ones(n, dtype=torch.int32, device=dev)
    z = X[:, 13:16] + 0.01
    si = torch.from_numpy(np.tile(np.eye(3).reshape(9) * 100.0, (n, 1))).to(dev)
    aux = torch.tensor([0.5, 0.2, 1.0], **f64).repeat(n, 1)
    xo, co, nis = torch.empty((n, 16), **f64), torch.empty((n, 225), **f64), torch.empty(n, **f64)
    ap_ = torch.empty(n, dtype=torch.int32, device=dev)
    out["k10_10k_ms"] = timed(torch, lambda: capi.check(lib.cpi_state_update_batch(n, p(X), p(C), p(W), p(xb), None, p(xo), p(co), p(nis),
                                                                                   p(ap_), None)), args.reps)
    out["k11_10k_ms"] = timed(torch, lambda: capi.check(lib.cpi_state_update_measurements_batch(n, p(X), p(C), p(offs), p(kind), p(z), p(si),
                                                                                                p(aux), None, p(xo), p(co), p(nis), p(ap_),
                                                                                                None)), args.reps)
    Cn, S = 10_000, 30
    Sw, L = synth.make_windows(S - 1, 20, rate=200.0, special=False)
    rec = preint.preintegrate_host(1, Sw, L, synth.SIGMAS, 0, ns=20)
    Xc = synth.make_states(rec, L, 1, perturb=False)
    Xa = torch.from_numpy(np.tile(Xc, (Cn, 1))).to(dev)
    R, Ld = torch.from_numpy(np.tile(rec, (Cn, 1))).to(dev), torch.from_numpy(np.tile(L, (Cn, 1))).to(dev)
    info = np.diag(np.repeat([1e4, 1e6, 1e2, 1e4, 1e2], 3))
    prior = (torch.from_numpy(np.tile(info.T.reshape(225), (Cn, 1))).to(dev), None, None, None)
    M = 20_000
    sidx = torch.from_numpy(np.sort(rng.integers(0, Cn * S, M))).to(dev)
    Wp = np.zeros((15, 15)); Wp[12:15, 12:15] = np.eye(3) * 1e4
    sp = (sidx, torch.from_numpy(np.tile(Wp.T.reshape(225), (M, 1))).to(dev), None, None, Xa[sidx].clone())
    lever = torch.tensor([0.5, 0.2, 1.0], **f64).repeat(M, 1)
    mss = (sidx, torch.ones(M, dtype=torch.int32, device=dev), Xa[sidx, 13:16].clone(),
           torch.from_numpy(np.tile(np.eye(3).reshape(9) * 100.0, (M, 1))).to(dev), lever)
    kw = dict(prior=prior, max_rounds=10, check_every=0)
    lr = max(args.reps // 10, 3)
    out["lm_priors_ms"] = timed(torch, lambda: factor.chains_lm(1, Xa, R, Ld, S, state_priors=sp, **kw), lr)
    out["lm_lever_arm_ms"] = timed(torch, lambda: factor.chains_lm(1, Xa, R, Ld, S, measurements=mss, **kw), lr)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
