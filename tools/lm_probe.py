"""Latency of Levenberg-Marquardt to convergence over many chains (factor.chains_lm).

    python tools/lm_probe.py [--reps 5]

Prints ONE JSON line:
  gpu / power_limit_w      the card the numbers come from (read in the same run)
  small10k / large10k      10 000 model-1 chains of 30 states, perturbed as in the 64-sequence smoother test (v, p 1e-3, b_g 1e-5),
                           or with v, p 0.1 and attitude 1e-2 rad; a 1e8 I prior on every first state; run to convergence
                           (check_every 8).  total_ms, rounds (the most tries of any chain), ms_per_round split into linearise (eval +
                           information blocks + prior_at), solve (assembly + isolated solve + retract) and cost+update (K9 + prior_at +
                           the LM update), statuses, and a histogram of accepted steps
  chain5k                  the configs[4] chain (5 000 states, model 1) run to convergence the same way
CUDA events, median over --reps for the totals; the per-round split is one round of each phase timed alone.
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
        raise SystemExit("lm_probe needs a CUDA device")
    from cpi_b200 import capi, factor, preint, synth
    capi.load()
    name, power = gpu_identity()
    out = dict(gpu=name, power_limit_w=power, reps=args.reps)
    rng = np.random.default_rng(1)

    def problem(n_chains, S, large, first_window):
        Sm, L = synth.make_windows(n_chains * (S - 1), 20, rate=200.0, first_window=first_window, special=False)
        rec = preint.preintegrate_host(1, Sm, L, synth.SIGMAS, 0, ns=20)
        X = np.concatenate([synth.make_states(rec[c * (S - 1):(c + 1) * (S - 1)], L[c * (S - 1):(c + 1) * (S - 1)], 1, perturb=False)
                            for c in range(n_chains)]).reshape(n_chains, S, 16)
        if large:
            d = np.zeros((n_chains, S - 1, 15))
            d[..., 0:3] = rng.normal(0, 1e-2, d[..., 0:3].shape)
            d[..., 6:9] = rng.normal(0, 0.1, d[..., 6:9].shape); d[..., 12:15] = rng.normal(0, 0.1, d[..., 12:15].shape)
            X[:, 1:] = factor.retract(X[:, 1:].reshape(-1, 16), d.reshape(-1, 15)).reshape(n_chains, S - 1, 16)
        else:
            X[:, 1:, 7:10] += rng.normal(0, 1e-3, (n_chains, S - 1, 3)); X[:, 1:, 13:16] += rng.normal(0, 1e-3, (n_chains, S - 1, 3))
            X[:, 1:, 4:7] += rng.normal(0, 1e-5, (n_chains, S - 1, 3))
        dX, dR, dL = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (X.reshape(-1, 16), rec, L))
        info0 = torch.eye(15, dtype=torch.float64, device="cuda").reshape(1, 225) * 1e8
        prior = (info0.repeat(n_chains, 1).contiguous(), None, None, dX[::S].contiguous())
        return dX, dR, dL, prior

    def run(n_chains, S, large, first_window):
        dX, dR, dL, prior = problem(n_chains, S, large, first_window)
        go = lambda **kw: factor.chains_lm(1, dX, dR, dL, S, prior=prior, **kw)
        ms = timed(torch, go, args.reps)
        Xs, cost, lam, st, it, tr = go()
        rounds = int(tr.max())
        # one round's phases alone, at the initial states
        nf = dR.shape[0]
        ar = torch.arange(nf, device="cuda")
        ii = ar + ar // (S - 1); jj = ii + 1
        lams = torch.full((n_chains,), 1e-5, dtype=torch.float64, device="cuda")
        pz = (prior[0], torch.zeros((n_chains, 15), dtype=torch.float64, device="cuda"), torch.zeros(n_chains, dtype=torch.float64, device="cuda"),
              prior[3])

        def lin():
            e, H1, H2 = factor.factor_eval(1, dX, dR, dL, ii, jj)
            G = factor.factor_hessian(1, dR, e, H1, H2)
            factor.prior_at(pz[0], pz[1], pz[2], pz[3], dX[::S].contiguous())
            return G
        G = lin()

        def solve():
            D, E, rhs, damp = factor.chains_assemble_lm(*G[:5], S, lams, pz[0], pz[1], n_chains=n_chains)
            return factor.retract(dX, factor.chains_solve(D, E, rhs, S, n_chains=n_chains))
        Xn = solve()
        D, E, rhs, damp = factor.chains_assemble_lm(*G[:5], S, lams, pz[0], pz[1], n_chains=n_chains)
        dx = factor.chains_solve(D, E, rhs, S, n_chains=n_chains)
        lib = capi.load()
        ws = torch.empty(int(lib.cpi_imu_chains_lm_workspace(dX.shape[0])) // 8, dtype=torch.float64, device="cuda")
        Xc = dX.clone()
        lam_c, cost_c = lams.clone(), torch.empty_like(lams)
        st_c, it_c, tr_c = (torch.zeros(n_chains, dtype=torch.int32, device="cuda") for _ in range(3))
        prm = capi.LMParams()
        p = factor._tptr

        def update():
            st_c.zero_()                                           # every chain running, as in a round
            fn = factor.factor_cost(1, Xn, dR, dL, ii, jj)
            _, pfn = factor.prior_at(pz[0], pz[1], pz[2], pz[3], Xn[::S].contiguous())
            capi.check(lib.cpi_imu_chains_lm_update(n_chains, None, S, dX.shape[0], __import__("ctypes").byref(prm), p(G[5]), p(pz[2]), p(fn), p(pfn),
                                                    p(rhs), p(D), p(E), p(damp), p(dx), p(Xn), p(Xc), p(lam_c), p(cost_c), p(st_c), p(it_c), p(tr_c),
                                                    None, p(ws), __import__("ctypes").c_void_p(torch.cuda.current_stream().cuda_stream)))
        split = dict(linearise=timed(torch, lin, args.reps), solve=timed(torch, solve, args.reps), cost_update=timed(torch, update, args.reps))
        hist = np.bincount(it.cpu().numpy(), minlength=1)
        return dict(chains=n_chains, states_per_chain=S, total_ms=ms, rounds=rounds, ms_per_round=ms / max(rounds, 1), split_ms_per_round=split,
                    statuses=np.bincount(st.cpu().numpy(), minlength=5).tolist(), accepted_steps_histogram=hist.tolist(),
                    max_tries=rounds, finite=bool(torch.isfinite(Xs).all()))

    out["small10k"] = run(10_000, 30, False, 50000)
    out["large10k"] = run(10_000, 30, True, 50000)
    out["chain5k"] = run(1, 5000, False, 9000)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
