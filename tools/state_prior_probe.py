"""Cost and effect of priors on any state (factor.chains_lm with state_priors, cpi_imu_state_priors_fold).

    python tools/state_prior_probe.py [--reps 5]

Prints ONE JSON line:
  gpu / power_limit_w   the card the numbers come from (read in the same run)
  chains10k             10 000 model-1 chains of 30 states (small perturbations, a 1e8 I prior on every first state), run to
                        convergence (check_every 8) without state priors and with a 1 cm position fix on every 10th keyframe:
                        total_ms, rounds, statuses
  chain5k               the configs[4] chain (5 000 states, model 1, small perturbations, a 1e8 I prior on x_0) with a 1 cm position
                        fix every 50 keyframes at lambda_lower = 0: total_ms, rounds, accepted steps, final status and lambda
  fold_us               the fold kernel alone on the 10 000-chain layout with its 20 000 fixes: fold and f-only fold
CUDA events, median over --reps (the fold: over 20 * --reps calls).
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from scan_probe import gpu_identity, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("state_prior_probe needs a CUDA device")
    from cpi_b200 import capi, factor, preint, synth
    capi.load()
    name, power = gpu_identity()
    out = dict(gpu=name, power_limit_w=power, reps=args.reps)
    rng = np.random.default_rng(1)
    dev = dict(dtype=torch.float64, device="cuda")

    def problem(n_chains, S, first_window, every):
        Sm, L = synth.make_windows(n_chains * (S - 1), 20, rate=200.0, first_window=first_window, special=False)
        rec = preint.preintegrate_host(1, Sm, L, synth.SIGMAS, 0, ns=20)
        truth = np.concatenate([synth.make_states(rec[c * (S - 1):(c + 1) * (S - 1)], L[c * (S - 1):(c + 1) * (S - 1)], 1, perturb=False)
                                for c in range(n_chains)]).reshape(n_chains, S, 16)
        X = truth.copy()
        X[:, 1:, 7:10] += rng.normal(0, 1e-3, (n_chains, S - 1, 3)); X[:, 1:, 13:16] += rng.normal(0, 1e-3, (n_chains, S - 1, 3))
        X[:, 1:, 4:7] += rng.normal(0, 1e-5, (n_chains, S - 1, 3))
        dX, dR, dL = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (X.reshape(-1, 16), rec, L))
        prior = ((torch.eye(15, **dev).reshape(1, 225) * 1e8).repeat(n_chains, 1).contiguous(), None, None, dX[::S].contiguous())
        idx = (np.arange(n_chains)[:, None] * S + np.arange(every, S, every)[None, :]).reshape(-1)
        W = np.zeros((15, 15)); W[12:15, 12:15] = np.eye(3) * 1e4                 # 1 cm
        lin = truth.reshape(-1, 16)[idx].copy()
        lin[:, 13:16] += rng.normal(0, 0.01, (len(idx), 3))
        M = len(idx)
        sp = (torch.from_numpy(idx.astype(np.int64)).cuda(), torch.from_numpy(np.tile(W.T.reshape(1, 225), (M, 1))).cuda(), None, None,
              torch.from_numpy(lin).cuda())
        return dX, dR, dL, prior, sp

    def run(n_chains, S, first_window, every, with_sp):
        dX, dR, dL, prior, sp = problem(n_chains, S, first_window, every)
        go = lambda: factor.chains_lm(1, dX, dR, dL, S, prior=prior, state_priors=sp if with_sp else None)
        ms = timed(torch, go, args.reps)
        Xs, cost, lam, st, it, tr = go()
        return dict(chains=n_chains, states_per_chain=S, state_priors=int(sp[0].numel()) if with_sp else 0, total_ms=ms, rounds=int(tr.max()),
                    accepted_steps_max=int(it.max()), statuses=np.bincount(st.cpu().numpy(), minlength=5).tolist(),
                    lambda_min=float(lam.min()), finite=bool(torch.isfinite(Xs).all())), (dX, sp, S)

    plain, _ = run(10_000, 30, 50000, 10, False)
    fixed, (dX, sp, S) = run(10_000, 30, 50000, 10, True)
    out["chains10k"] = dict(without=plain, with_position_fixes=fixed)
    out["chain5k"] = run(1, 5000, 9000, 50, True)[0]
    # the fold alone on the 10 000-chain layout
    N, nf = dX.shape[0], dX.shape[0] - 10_000
    order, sp_off = factor._state_prior_csr(sp[0], N)
    info = sp[1][order].contiguous()
    rhs, f = torch.zeros((info.shape[0], 15), **dev), torch.zeros(info.shape[0], **dev)
    G11, G22 = torch.zeros((nf, 225), **dev), torch.zeros((nf, 225), **dev)
    g1, g2, fk = torch.zeros((nf, 15), **dev), torch.zeros((nf, 15), **dev), torch.zeros(nf, **dev)
    fold = lambda: factor.state_priors_fold(S, sp_off, info, rhs, f, G11=G11, G22=G22, g1=g1, g2=g2, f=fk, n_chains=10_000)
    fonly = lambda: factor.state_priors_fold(S, sp_off, None, None, f, f=fk, n_chains=10_000)
    out["fold_us"] = dict(fold=1e3 * timed(torch, fold, 20 * args.reps), f_only=1e3 * timed(torch, fonly, 20 * args.reps),
                          states=N, priors=int(info.shape[0]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
