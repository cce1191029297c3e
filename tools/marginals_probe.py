"""Marginal covariances of many chains (cpi_imu_chains_marginals; DESIGN.md section 3j): time of the selected inversion on one GPU.
Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/marginals_probe.py [--chains 10000] [--states 30] [--reps 11]

Model 1, `chains` chains of `states` keyframes (20-sample windows at 200 Hz) at their dead-reckoned prediction with a 1e8 I prior on
x_0, and the configs[4] chain (5 000 states) with a 1 cm position fix every 50 keyframes.  Cases (CUDA events, median of --reps after
3 warm-up calls):
  covariance           factor.chains_covariance on the assembled undamped system, workspace preallocated
  covariance_cross     the same with the cross blocks
  marginals            the whole factor.chains_marginals (linearisation, assembly with lambda = 0, covariance)
  assemble             one chains_assemble of the same blocks (lambda = 0), for comparison
  solve                one chains_solve of the assembled system, workspace preallocated, for comparison
The byte counts are what the kernels load and store, counted from the level structure (D, E read; the forward phase's Lc, Za, Zb, zb
and reduced systems; the level walk's reads of Lc, Za, Zb, the neighbours' blocks and its writes); `hbm_bound_ms` is that over the
H100 SXM data sheet's 3.35 TB/s."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from scan_probe import gpu_identity, timed  # noqa: E402

HBM = 3.35e12


def covariance_bytes(n, cross):
    """Bytes the isolated forward phase and the level walk load and store for n states (fp64; chain ids and the zero rhs included)."""
    d = 8 * n + 15 * n                                           # k_chain_ids writes, the zero rhs
    m = n
    while m > 1:
        odd, even = m // 2, (m + 1) // 2
        d += odd * (120 + 2 * 225 + 15 + 3 * 225 + 15)           # eliminate: D (lower), E left / right, b -> Lc, Za, Zb, zb
        d += even * (225 + 15 + 3 * 225 + 30 + 2 * 225 + 15)     # reduce: D, b, Zb, Za, Zb, zb -> D', E', b'
        d += odd * (120 + 2 * 225 + 3 * 225 + 225 + 2 * 225)     # level walk: Lc, Za, Zb, two diagonal blocks + N -> Sigma_ii, 2 N
        m = even
    d += 225 * 2                                                 # the root
    if not cross:
        d -= 225 * (n - 1)                                       # level 0's neighbour blocks are not stored
    return 8 * d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=10_000)
    ap.add_argument("--states", type=int, default=30)
    ap.add_argument("--reps", type=int, default=11)
    a = ap.parse_args()
    import torch
    from cpi_b200 import capi, factor, preint, synth
    name, power = gpu_identity()
    C, S = a.chains, a.states
    N = C * S
    dev = torch.device("cuda")
    Sm, L = synth.make_windows(C * (S - 1), 20, rate=200.0, first_window=0, special=False)
    dL = torch.from_numpy(L).cuda()
    rec = preint.preintegrate(1, torch.from_numpy(Sm).cuda(), dL, synth.SIGMAS, 0, ns=20)
    X = torch.empty((C, S, 16), dtype=torch.float64, device=dev)
    X[:, 0] = 0.0; X[:, 0, 3] = 1.0
    X[:, 0, 4:7] = dL.view(C, S - 1, 13)[:, 0, 0:3]; X[:, 0, 10:13] = dL.view(C, S - 1, 13)[:, 0, 3:6]
    for k in range(S - 1):
        X[:, k + 1] = factor.predict_state(1, X[:, k].contiguous(), rec.view(C, S - 1, -1)[:, k].contiguous(), dL.view(C, S - 1, 13)[:, k].contiguous())
    X = X.reshape(N, 16)
    info0 = torch.eye(15, dtype=torch.float64, device=dev).reshape(1, 225).repeat(C, 1) * 1e8
    prior = (info0, None, None, None)
    e, H1, H2 = factor.factor_eval(1, X, rec, dL, *factor._chain_factor_states(C, None, S, C * (S - 1), dev))
    G = factor.factor_hessian(1, rec, e, H1, H2)
    D, E, rhs = factor.chains_assemble(*G[:5], S, 0.0, info0, None)
    ws = torch.empty((int(capi.load().cpi_imu_chains_marginals_workspace(C, N)) + 7) // 8, dtype=torch.float64, device=dev)
    ws_solve = torch.empty((int(capi.load().cpi_imu_chains_solve_workspace(C, N)) + 7) // 8, dtype=torch.float64, device=dev)
    res = {"gpu": name, "power_limit_w": power, "chains": C, "states": S, "reps": a.reps}
    t = {
        "covariance": timed(torch, lambda: factor.chains_covariance(D, E, S, workspace=ws), a.reps),
        "covariance_cross": timed(torch, lambda: factor.chains_covariance(D, E, S, cross=True, workspace=ws), a.reps),
        "marginals": timed(torch, lambda: factor.chains_marginals(1, X, rec, dL, S, prior=prior), a.reps),
        "assemble": timed(torch, lambda: factor.chains_assemble(*G[:5], S, 0.0, info0, None), a.reps),
        "solve": timed(torch, lambda: factor.chains_solve(D, E, rhs, S, workspace=ws_solve), a.reps),
    }
    res["ms"] = t
    for key, cross in (("covariance", False), ("covariance_cross", True)):
        b = covariance_bytes(N, cross)
        res[key + "_bytes"] = b
        res[key + "_hbm_bound_ms"] = b / HBM * 1e3
        res[key + "_hbm_share"] = b / HBM * 1e3 / t[key]
    # the configs[4] chain with a position fix every 50 keyframes
    n = 5000
    rng = np.random.default_rng(1)
    Sm, L = synth.make_windows(n - 1, 20, rate=200.0, first_window=9000, special=False)
    r5 = preint.preintegrate_host(1, Sm, L, synth.SIGMAS, 0, ns=20)
    truth = synth.make_states(r5, L, 1, perturb=False)
    idx = np.arange(50, n, 50, dtype=np.int64)
    W = np.zeros((15, 15)); W[12:15, 12:15] = np.eye(3) / 0.01 ** 2
    lin = truth[idx].copy(); lin[:, 13:16] += rng.normal(0, 0.01, (len(idx), 3))
    sp = (torch.from_numpy(idx).cuda(), torch.from_numpy(np.repeat(W.T.reshape(1, 225), len(idx), axis=0)).cuda(), None, None,
          torch.from_numpy(lin).cuda())
    d5 = [torch.from_numpy(v).cuda() for v in (truth, r5, L)]
    res["chain5k_marginals_ms"] = timed(torch, lambda: factor.chains_marginals(1, *d5, n, prior=(info0[:1], None, None, None), state_priors=sp,
                                                                              cross=True), a.reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
