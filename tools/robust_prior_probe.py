"""Cost and effect of robust losses on state priors (factor.chains_lm with state_prior_loss, cpi_imu_state_priors_robust).

    python tools/robust_prior_probe.py [--reps 5]

Prints ONE JSON line:
  gpu / power_limit_w   the card the numbers come from (read in the same run)
  chains10k             10 000 model-1 chains of 30 states (small perturbations, a 1e8 I prior on every first state) with a 1 cm
                        position fix on every 10th keyframe, 5 % of the fixes replaced by 5 m outliers, run to convergence
                        (check_every 8) under each loss (gaussian, huber k = 1.345, cauchy k = 2.3849): total_ms, rounds, statuses
                        and the worst position error against the true states
  robust_us             the robust pass alone on those 20 000 priors: the full pass and the f-only pass
CUDA events, median over --reps (the robust pass: over 20 * --reps calls).
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
        raise SystemExit("robust_prior_probe needs a CUDA device")
    from cpi_b200 import capi, factor, preint, synth
    capi.load()
    name, power = gpu_identity()
    out = dict(gpu=name, power_limit_w=power, reps=args.reps)
    rng = np.random.default_rng(1)
    dev = dict(dtype=torch.float64, device="cuda")
    C, S, every = 10_000, 30, 10

    Sm, L = synth.make_windows(C * (S - 1), 20, rate=200.0, first_window=50000, special=False)
    rec = preint.preintegrate_host(1, Sm, L, synth.SIGMAS, 0, ns=20)
    truth = np.concatenate([synth.make_states(rec[c * (S - 1):(c + 1) * (S - 1)], L[c * (S - 1):(c + 1) * (S - 1)], 1, perturb=False)
                            for c in range(C)]).reshape(C, S, 16)
    X = truth.copy()
    X[:, 1:, 7:10] += rng.normal(0, 1e-3, (C, S - 1, 3)); X[:, 1:, 13:16] += rng.normal(0, 1e-3, (C, S - 1, 3))
    X[:, 1:, 4:7] += rng.normal(0, 1e-5, (C, S - 1, 3))
    dX, dR, dL = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (X.reshape(-1, 16), rec, L))
    prior = ((torch.eye(15, **dev).reshape(1, 225) * 1e8).repeat(C, 1).contiguous(), None, None, dX[::S].contiguous())
    idx = (np.arange(C)[:, None] * S + np.arange(every, S, every)[None, :]).reshape(-1)
    M = len(idx)
    W = np.zeros((15, 15)); W[12:15, 12:15] = np.eye(3) * 1e4                 # 1 cm
    lin = truth.reshape(-1, 16)[idx].copy()
    lin[:, 13:16] += rng.normal(0, 0.01, (M, 3))
    n_out = M // 20
    out_q = rng.choice(M, size=n_out, replace=False)
    d = rng.normal(size=(n_out, 3))
    lin[out_q, 13:16] += 5.0 * d / np.linalg.norm(d, axis=1, keepdims=True)    # 5 m outliers
    sp = (torch.from_numpy(idx.astype(np.int64)).cuda(), torch.from_numpy(np.tile(W.T.reshape(1, 225), (M, 1))).cuda(), None, None,
          torch.from_numpy(lin).cuda())
    tp = torch.from_numpy(truth.reshape(-1, 16)[:, 13:16].copy()).cuda()
    runs = {}
    for lname, code, k in (("gaussian", None, 0.0), ("huber", capi.LOSS_HUBER, 1.345), ("cauchy", capi.LOSS_CAUCHY, 2.3849)):
        loss = None if code is None else (torch.full((M,), code, dtype=torch.int32, device="cuda"), torch.full((M,), k, **dev))
        go = lambda: factor.chains_lm(1, dX, dR, dL, S, prior=prior, state_priors=sp, state_prior_loss=loss)
        ms = timed(torch, go, args.reps)
        Xs, cost, lam, st, it, tr = go()
        err = torch.linalg.norm(Xs[:, 13:16] - tp, dim=1)
        runs[lname] = dict(total_ms=ms, rounds=int(tr.max()), accepted_steps_max=int(it.max()),
                           statuses=np.bincount(st.cpu().numpy(), minlength=5).tolist(), worst_position_error_m=float(err.max()),
                           median_position_error_m=float(err.median()), finite=bool(torch.isfinite(Xs).all()))
    out["chains10k"] = dict(chains=C, states_per_chain=S, state_priors=M, outliers=n_out, **runs)
    # the robust pass alone on the moved priors of the initial states
    order, _ = factor._state_prior_csr(sp[0], C * S)
    info = sp[1][order].contiguous()
    rr, ff = factor.prior_at(info, torch.zeros((M, 15), **dev), None, sp[4][order].contiguous(), dX[sp[0][order]].contiguous())
    code, kk = torch.full((M,), capi.LOSS_CAUCHY, dtype=torch.int32, device="cuda"), torch.full((M,), 2.3849, **dev)
    iw, rw, fw = torch.empty_like(info), torch.empty_like(rr), torch.empty_like(ff)
    full = lambda: factor.state_priors_robust(code, kk, info, rr, ff, info_out=iw, rhs_out=rw, f_out=fw)
    fonly = lambda: factor.state_priors_robust(code, kk, None, None, ff, f_out=fw)
    out["robust_us"] = dict(full=1e3 * timed(torch, full, 20 * args.reps), f_only=1e3 * timed(torch, fonly, 20 * args.reps), priors=M,
                            bytes_full=M * (225 + 15 + 1) * 8 * 2 + M * 12)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
