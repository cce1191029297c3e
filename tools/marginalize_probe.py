"""Latency and throughput of the fixed-lag smoother entry points (cpi_imu_chain_marginalize, cpi_imu_chains_assemble via
factor.chains_lm_step).

    python tools/marginalize_probe.py [--reps 50]

Prints ONE JSON line:
  gpu / power_limit_w      the card the numbers come from (read in the same run)
  marg10k                  10 000 chains of 2 states, each eliminating one (one cpi_imu_chain_marginalize call, with a prior): the
                           bytes a chain moves (one factor's blocks G11 / G12 / G22 / g1 / g2 / f = 5 648 B, the prior in and out
                           2 x 1 928 B) and the HBM bound at the H100 SXM data-sheet 3.35 TB/s
  lm10k                    10 000 chains of 30 states (290 000 model-1 factors): ONE factor.chains_lm_step over all of them, against
                           factor.chain_lm_step called chain by chain -- 100 such calls are timed, `per_chain_ms` is their mean and
                           `chain_by_chain_10k_ms` = 10 000 x that
  head5k                   one chain of 5 000 states whose first 4 999 are eliminated: the sequential depth of K8 (one warp walks
                           the whole head)
CUDA events, median over --reps (head5k and the chain-by-chain loop: over --reps // 10 + 1).
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

BLOCK_BYTES = 3 * 1800 + 2 * 120 + 8          # G11, G12, G22, g1, g2, f of one factor
PRIOR_BYTES = 1800 + 120 + 8                  # info, rhs, f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("marginalize_probe needs a CUDA device")
    from cpi_b200 import capi, factor, preint, synth
    capi.load()
    name, power = gpu_identity()
    out = dict(gpu=name, power_limit_w=power, reps=args.reps)

    # one 29-record chain, tiled: 10 000 chains of 30 states
    n_chains, S = 10_000, 30
    Sm, L = synth.make_windows(S - 1, 20, rate=200.0, first_window=50000, special=False)
    rec = preint.preintegrate_host(1, Sm, L, synth.SIGMAS, 0, ns=20)
    X = synth.make_states(rec, L, 1)
    dR = torch.from_numpy(np.tile(rec, (n_chains, 1))).cuda()
    dL = torch.from_numpy(np.tile(L, (n_chains, 1))).cuda()
    dX = torch.from_numpy(np.tile(X, (n_chains, 1))).cuda()
    info0 = torch.eye(15, dtype=torch.float64, device="cuda").reshape(1, 225) * 1e8
    prior = (info0.repeat(n_chains, 1).contiguous(), torch.zeros((n_chains, 15), dtype=torch.float64, device="cuda"),
             torch.zeros(n_chains, dtype=torch.float64, device="cuda"), dX[::S].contiguous())

    # 10 000 chains eliminating one state each: the first factor of every chain
    first = torch.arange(n_chains, device="cuda") * (S - 1)
    e, H1, H2 = factor.factor_eval(1, dX, dR[first].contiguous(), dL[first].contiguous(), idx_i=first + torch.arange(n_chains, device="cuda"),
                                   idx_j=first + torch.arange(n_chains, device="cuda") + 1)
    G = factor.factor_hessian(1, dR[first].contiguous(), e, H1, H2)
    ms = timed(torch, lambda: factor.chain_marginalize(*G, 2, 1, prior=prior[:3], n_chains=n_chains), args.reps)
    byts = n_chains * (BLOCK_BYTES + 2 * PRIOR_BYTES)
    out["marg10k"] = dict(chains=n_chains, ms=ms, bytes_per_chain=BLOCK_BYTES + 2 * PRIOR_BYTES, hbm_bound_ms=byts / HBM_BPS * 1e3,
                          frac_of_hbm_bound=byts / HBM_BPS * 1e3 / ms)

    # one LM step of 10 000 windows of 30 states, against one chain at a time
    ms_all = timed(torch, lambda: factor.chains_lm_step(1, dX, dR, dL, S, prior=prior), args.reps)
    one = [(dX[c * S:(c + 1) * S], dR[c * (S - 1):(c + 1) * (S - 1)], dL[c * (S - 1):(c + 1) * (S - 1)]) for c in range(100)]

    def chain_by_chain():
        for x, r, l in one:
            factor.chain_lm_step(1, x, r, l)
    ms_100 = timed(torch, chain_by_chain, args.reps // 10 + 1)
    out["lm10k"] = dict(chains=n_chains, states_per_chain=S, chains_lm_step_ms=ms_all, chain_lm_step_calls_timed=100,
                        per_chain_ms=ms_100 / 100, chain_by_chain_10k_ms=ms_100 / 100 * n_chains, speedup=ms_100 / 100 * n_chains / ms_all)

    # a 5 000-state head eliminated in one chain
    nh = 4999
    Sh, Lh = synth.make_windows(nh, 20, rate=200.0, first_window=9000, special=False)
    rech = preint.preintegrate_host(1, Sh, Lh, synth.SIGMAS, 0, ns=20)
    Xh = synth.make_states(rech, Lh, 1)
    dRh = torch.from_numpy(rech).cuda()
    e, H1, H2 = factor.factor_eval(1, torch.from_numpy(Xh).cuda(), dRh, torch.from_numpy(Lh).cuda())
    Gh = factor.factor_hessian(1, dRh, e, H1, H2)
    ph = (info0, torch.zeros((1, 15), dtype=torch.float64, device="cuda"), torch.zeros(1, dtype=torch.float64, device="cuda"))
    ms_h = timed(torch, lambda: factor.chain_marginalize(*Gh, nh + 1, nh, prior=ph), args.reps // 10 + 1)
    out["head5k"] = dict(states=nh + 1, eliminated=nh, ms=ms_h, us_per_eliminated_state=ms_h * 1e3 / nh)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
