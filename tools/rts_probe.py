"""Time the Rauch-Tung-Striebel smoothers of filter runs (factor.rts_smooth: one K7 pass, then K15; DESIGN.md section 3o;
factor.rts_smooth_scan: the same K7 pass, then the parallel-in-time K16; section 3p).

    python tools/rts_probe.py [--reps 30]

Prints ONE JSON line:
  gpu / power_limit_w      the card the numbers come from (read in the same run)
  runs10k_S10 / _S30       10 000 runs of 10 and 30 keyframes (model 1): median ms of the K7 pass (propagate with want_cross over every
                           transition) and of K15 (the raw C call, with cross), K15's counted bytes and their time at the H100 SXM
                           data-sheet 3.35 TB/s, and chains_marginals on the same chains (with a prior on each first state)
  one_run_S4999            one run of 4 999 keyframes: K15's median ms and ms per keyframe (K15 is sequential over a run's keyframes)
  scan                     K15 against K16 (both raw C calls with cross, on the same K7 outputs) on 1 x 4 999, 1 x 100 000,
                           100 x 1 000, 10 000 x 10 and 10 000 x 30 keyframes: median ms of each, K16's workspace bytes, launches per
                           call, counted bytes and their share of the 3.35 TB/s bound
  crossover                per run count (1, 100, 1 000) the median ms of K15 and K16 over run lengths, and the shortest length
                           from which K16 stays faster
CUDA events, median of --reps (at least 30) runs of each call.
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

from scan_probe import gpu_identity, timed  # noqa: E402

HBM = 3.35e12                  # H100 SXM data sheet, bytes/s


def k15_bytes(n_runs, n_states, cross=True):
    """Bytes K15 moves: per transition it reads x_k, P_k, xb, Pb, C (16 + 4 x 225 ... = 707 doubles) and writes xs_k, Ps_k (+ Xs_k);
    per run it reads and writes the last keyframe (241 doubles each way)."""
    nt = n_states - n_runs
    return 8 * (nt * (16 + 225 + 16 + 225 + 225 + 16 + 225 + (225 if cross else 0)) + n_runs * 2 * (16 + 225))


def k16_bytes(n_runs, n_states, cross=True):
    """Bytes K16 moves: the element kernel reads x_{k+1}, xb, Pb, C, P_k (707 doubles) per transition and P_{S-1} per run and
    writes one element (691 doubles) per keyframe; every scan level reads its elements, the reduce writes one aggregate per chunk,
    the down pass reads the seeds and writes back L and a at level 0 (240 doubles) and the whole element above; the apply kernel
    reads L, a and x_k (+ G_k and Ps_{k+1}) and writes xs_k, Ps_k (+ Xs_k) per transition, and copies each run's last keyframe."""
    ES, C = 691, 16
    nt = n_states - n_runs
    b = nt * 707 + n_runs * 225 + n_states * ES
    n = [n_states]
    while n[-1] > C:
        n.append((n[-1] + C - 1) // C)
    for l in range(len(n)):
        up = n[l + 1] if l + 1 < len(n) else 0
        if l + 1 < len(n):
            b += n[l] * ES + up * ES                                   # reduce
        b += n[l] * ES + up * ES + n[l] * (240 if l == 0 else ES - 1)  # down
    b += nt * (240 + 16 + 16 + 225 + (3 * 225 if cross else 0)) + n_runs * 2 * (16 + 225)
    return 8 * b


def filter_batch(torch, model, n_runs, S, seed=0):
    """n_runs runs of S keyframes: records tiled from 512 synthetic windows, the first state of each run from synth.make_states, and
    every later keyframe's (x, P) propagated by K7 from a random SPD P_0 (a dead-reckoned filter: its posteriors are its predictions)."""
    from cpi_b200 import factor, preint, synth
    base = 512
    Sm, L = synth.make_windows(base, 20, rate=200.0, first_window=seed, special=False)
    rec = preint.preintegrate_host(model, Sm, L, synth.SIGMAS, 0, ns=20)
    X0 = synth.make_states(rec, L, model, perturb=False)
    nt = n_runs * (S - 1)
    sel = np.arange(nt) % base
    dR, dL = torch.from_numpy(rec[sel]).cuda(), torch.from_numpy(L[sel]).cuda()
    rng = np.random.default_rng(seed)
    G = rng.normal(size=(64, 15, 15))
    D = np.repeat([2e-3, 2e-4, 2e-2, 2e-3, 5e-2], 3)
    P0 = D[None, :, None] * (G @ G.transpose(0, 2, 1) / 15 + 0.5 * np.eye(15)) * D[None, None, :]
    P0 = 0.5 * (P0 + P0.transpose(0, 2, 1))
    X = torch.empty((n_runs, S, 16), dtype=torch.float64, device="cuda")
    P = torch.empty((n_runs, S, 225), dtype=torch.float64, device="cuda")
    X[:, 0] = torch.from_numpy(X0[np.arange(n_runs) % base]).cuda()
    P[:, 0] = torch.from_numpy(P0[np.arange(n_runs) % 64].transpose(0, 2, 1).reshape(-1, 225)).cuda()
    r3, l3 = dR.view(n_runs, S - 1, -1), dL.view(n_runs, S - 1, 13)
    for k in range(S - 1):
        x1, c1, _ = factor.propagate(model, X[:, k].contiguous(), P[:, k].contiguous(), r3[:, k].contiguous(), l3[:, k].contiguous())
        X[:, k + 1], P[:, k + 1] = x1, c1
    torch.cuda.synchronize()
    return X.reshape(-1, 16), P.reshape(-1, 225), dR, dL, np.linalg.inv(P0[np.arange(n_runs) % 64])


def measure(torch, model, n_runs, S, reps):
    from cpi_b200 import capi, factor
    X, P, dR, dL, info0 = filter_batch(torch, model, n_runs, S)
    N = n_runs * S
    lib = capi.load()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    idx_i = None
    if n_runs > 1:
        idx_i = (torch.arange(N - n_runs, device="cuda") // (S - 1)) + torch.arange(N - n_runs, device="cuda")
    k7 = lambda: factor.propagate(model, X, P, dR, dL, anchor=idx_i, want_cross=True)
    xp, cp, cr = k7()
    out = [torch.empty_like(X), torch.empty_like(P), torch.empty_like(cr)]
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    k15 = lambda: capi.check(lib.cpi_rts_smooth_batch(n_runs, None, S, N, p(X), p(P), p(xp), p(cp), p(cr), p(out[0]), p(out[1]), p(out[2]), st))
    res = dict(k7_ms=timed(torch, k7, reps), k15_ms=timed(torch, k15, reps), k15_bytes=k15_bytes(n_runs, N))
    res["k15_hbm_bound_ms"] = res["k15_bytes"] / HBM * 1e3
    res["k15_share_of_hbm_bound"] = res["k15_hbm_bound_ms"] / res["k15_ms"]
    res["k15_ms_per_keyframe"] = res["k15_ms"] / max(S - 1, 1)
    if n_runs > 1:
        prior = (torch.from_numpy(info0.transpose(0, 2, 1).reshape(-1, 225).copy()).cuda(), None, None, None)
        res["chains_marginals_ms"] = timed(torch, lambda: factor.chains_marginals(model, X, dR, dL, S, prior=prior), reps)
    del X, P, dR, dL, xp, cp, cr, out
    torch.cuda.empty_cache()
    return res


def k15_k16(torch, model, n_runs, S, reps, X=None, P=None, dR=None, dL=None):
    """Median ms of K15 and K16 (raw C calls with cross) on n_runs runs of S keyframes, with K16's workspace bytes, launches per call
    and counted bytes.  X, P, dR, dL: a batch of runs of at least S keyframes to take the first S of (default: a new batch)."""
    from cpi_b200 import capi, factor
    if X is None:
        X, P, dR, dL, _ = filter_batch(torch, model, n_runs, S)
    else:
        Sm = X.shape[0] // n_runs
        X = X.view(n_runs, Sm, 16)[:, :S].reshape(-1, 16).contiguous()
        P = P.view(n_runs, Sm, 225)[:, :S].reshape(-1, 225).contiguous()
        dR = dR.view(n_runs, Sm - 1, -1)[:, :S - 1].reshape(n_runs * (S - 1), -1).contiguous()
        dL = dL.view(n_runs, Sm - 1, 13)[:, :S - 1].reshape(-1, 13).contiguous()
    N = n_runs * S
    lib = capi.load()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    idx_i = None
    if n_runs > 1:
        idx_i = (torch.arange(N - n_runs, device="cuda") // (S - 1)) + torch.arange(N - n_runs, device="cuda")
    xp, cp, cr = factor.propagate(model, X, P, dR, dL, anchor=idx_i, want_cross=True)
    out = [torch.empty_like(X), torch.empty_like(P), torch.empty_like(cr)]
    ws_bytes = int(lib.cpi_rts_smooth_scan_workspace(n_runs, N))
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    k15 = lambda: capi.check(lib.cpi_rts_smooth_batch(n_runs, None, S, N, p(X), p(P), p(xp), p(cp), p(cr), p(out[0]), p(out[1]), p(out[2]), st))
    k16 = lambda: capi.check(lib.cpi_rts_smooth_scan_batch(n_runs, None, S, N, p(X), p(P), p(xp), p(cp), p(cr), p(out[0]), p(out[1]),
                                                           p(out[2]), p(ws), st))
    before = capi.launch_count()
    k16()
    launches = capi.launch_count() - before
    res = dict(k15_ms=timed(torch, k15, reps), k16_ms=timed(torch, k16, reps), k16_workspace_bytes=ws_bytes, k16_launches=launches,
               k16_bytes=k16_bytes(n_runs, N))
    res["k16_share_of_hbm_bound"] = res["k16_bytes"] / HBM * 1e3 / res["k16_ms"]
    res["k15_over_k16"] = res["k15_ms"] / res["k16_ms"]
    del X, P, dR, dL, xp, cp, cr, out, ws
    torch.cuda.empty_cache()
    return res


def crossover(torch, model, n_runs, lengths, reps):
    """K15 and K16 over run lengths at n_runs runs, and the shortest length from which K16 is faster at every longer one."""
    X, P, dR, dL, _ = filter_batch(torch, model, n_runs, max(lengths))
    rows = {S: k15_k16(torch, model, n_runs, S, reps, X, P, dR, dL) for S in lengths}
    from_S = None
    for S in sorted(lengths, reverse=True):
        if rows[S]["k16_ms"] < rows[S]["k15_ms"]:
            from_S = S
        else:
            break
    return dict(k15_ms={S: r["k15_ms"] for S, r in rows.items()}, k16_ms={S: r["k16_ms"] for S, r in rows.items()}, k16_faster_from=from_S)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    if args.reps < 30:
        raise SystemExit("--reps must be at least 30")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("rts_probe needs a CUDA device")
    name, power = gpu_identity()
    out = dict(gpu=name, power_limit_w=power, reps=args.reps)
    out["runs10k_S10"] = measure(torch, 1, 10_000, 10, args.reps)
    out["runs10k_S30"] = measure(torch, 1, 10_000, 30, args.reps)
    out["one_run_S4999"] = measure(torch, 1, 1, 4999, args.reps)
    out["scan"] = {f"{R}x{S}": k15_k16(torch, 1, R, S, args.reps)
                   for R, S in ((1, 4999), (1, 100_000), (100, 1000), (10_000, 10), (10_000, 30))}
    lengths = [2, 3, 4, 6, 8, 12, 16, 24, 32, 48, 64, 96, 128, 192, 256, 384, 512]
    out["crossover"] = {str(R): crossover(torch, 1, R, lengths, args.reps) for R in (1, 100, 1000)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
