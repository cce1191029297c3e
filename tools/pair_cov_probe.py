"""Time cpi_imu_chains_pair_covariance (DESIGN.md section 3q) with CUDA events, median of 30 calls after warm-up, on synthetic SPD
block-tridiagonal systems: every chain is the information form of a random walk x_{k+1} = F_k x_k + w_k, F_k a random rotation
(Cayley transform of a random skew matrix), Cov(w_k) = I, with a unit prior on its first state.  Far blocks are then of the order of
the diagonal ones (the first and last keyframe of a 30-state chain correlate at about 0.1 to 0.3), and the walk's work does not depend on
the values.  Cases:

  anchor    10 000 chains x 30 states, one pair per chain (first, last keyframe), against the route without the walk: 15 unit-column
            chains_solve calls with the anchor column of every chain at once; the two routes' worst difference is reported relative
            to each block's own largest entry and in the units of the diagonal
  all435    the same batch, all 435 pairs i < j of every chain
  long1e5   10^5 random pairs on one chain of 5 000 states

Each case is split into the forward phase plus Sigma_root (the same call with one pair) and the walk (the rest).  Flops per pair
are counted on the host by replaying the walk's bracket logic: an expansion of one bracket node costs 15 forward substitutions
(15 x 105 FMA + 225 divisions) and 15 x 225 FMA per neighbour of its chain, a node in both brackets 3 375 FMA more, the root
2 x 3 375 FMA; an FMA counts 2 flops.  Prints one JSON line per case, with the card's name and power limit read in the same run."""
import json
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, __file__.rsplit("/tools/", 1)[0])
from cpi_b200 import factor  # noqa: E402


def system(C, S, seed):
    """D [C*S,225], E [C*S-1,225] of C random-walk chains of S states (column-major blocks; exact 0 between chains)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    N = C * S
    I = torch.eye(15, device="cuda", dtype=torch.float64)
    A = torch.randn((N, 15, 15), generator=g, device="cuda", dtype=torch.float64) * 0.1
    Sk = A - A.transpose(1, 2)
    F = torch.linalg.solve(I - Sk, I + Sk)                         # x_{k+1} = F_k x_k + w_k: a rotation
    k = torch.arange(N, device="cuda") % S
    last = (k == S - 1)[:, None, None]
    D = I + torch.where(last, 0 * I, F.transpose(1, 2) @ F)         # prior (first) or the previous step's w, then this step's F^T F
    E = torch.where(last, 0 * I, -F)[:-1]                           # block (k, k+1) = -F_k^T, stored column-major
    return D.reshape(N, 225).contiguous(), E.reshape(N - 1, 225).contiguous()


def timed(fn, reps=30):
    fn(); fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def flops(N, cid, pairs):
    """Counted flops of the walk of each pair (the kernel's bracket logic, no arithmetic)."""
    levels, m = [], N
    while m > 1:
        levels.append(m); m = (m + 1) // 2
    out = []
    for i, j in pairs:
        if cid[i] != cid[j]:
            out.append(0); continue
        a0, live, f = [i, j], [[True, False], [True, False]], 0
        ended = True
        for l, m in enumerate(levels):
            if not any(live[0]) or not any(live[1]):
                ended = False; break
            s = 1 << l
            xs = []
            for q in (0, 1):
                o = 0 if a0[q] & 1 else 1
                x = a0[q] + o
                if live[q][o]:
                    hl = cid[(x - 1) * s] == cid[x * s]
                    hr = x + 1 < m and cid[(x + 1) * s] == cid[x * s]
                    f += 2 * (15 * 105 + 15 * 225 * (hl + hr)) + 225
                    xs.append(x)
                    live[q] = [hl, live[q][1] or hr] if o == 0 else [live[q][0] or hl, hr]
                a0[q] >>= 1
            if len(xs) == 2 and xs[0] == xs[1]:
                f += 2 * 3375
        if ended and live[0][0] and live[1][0]:
            f += 4 * 3375
        out.append(f)
    return np.array(out)


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"
    C, S = 10_000, 30
    D, E = system(C, S, 1)
    N = C * S
    cid = np.repeat(np.arange(C), S)
    ws = torch.empty(int(factor.capi.load().cpi_imu_chains_pair_covariance_workspace(C, N)) // 8 + 1, dtype=torch.float64, device="cuda")
    first = np.arange(C) * S
    cases = {"anchor": np.stack([first, first + S - 1], -1),
             "all435": np.concatenate([np.stack([first + i, first + j], -1) for i in range(S) for j in range(i + 1, S)])}
    one = torch.tensor([[0, S - 1]], dtype=torch.int64, device="cuda")
    t_fwd = timed(lambda: factor.chains_pair_covariance(D, E, S, one, workspace=ws))
    for name, pairs in cases.items():
        dp = torch.from_numpy(pairs).cuda()
        t = timed(lambda: factor.chains_pair_covariance(D, E, S, dp, workspace=ws), reps=30 if name == "anchor" else 10)
        fl = flops(N, cid, pairs[:2000])
        rec = dict(case=name, card=card, chains=C, states=S, pairs=len(pairs), ms=t, forward_and_root_ms=t_fwd, walk_ms=t - t_fwd,
                   flops_per_pair=float(fl.mean()), walk_gflops=float(fl.mean() * len(pairs) / max(t - t_fwd, 1e-9) / 1e6))
        if name == "anchor":
            # the route without the walk: 15 unit-column solves, Sigma_{., last} of every chain
            rhs = [torch.zeros((N, 15), dtype=torch.float64, device="cuda") for _ in range(15)]
            for c in range(15):
                rhs[c].view(C, S, 15)[:, S - 1, c] = 1.0
            sws = torch.empty(int(factor.capi.load().cpi_imu_chains_solve_workspace(C, N)) // 8 + 1, dtype=torch.float64, device="cuda")
            cols = lambda: [factor.chains_solve(D, E, r, S, workspace=sws) for r in rhs]
            rec["solve15_ms"] = timed(cols, reps=30)
            Xs = torch.stack([x.view(C, S, 15)[:, 0] for x in cols()], -1)            # [C, 15 (row), 15 (column)]
            got = factor.chains_pair_covariance(D, E, S, dp, workspace=ws).view(C, 15, 15).transpose(1, 2)   # column-major -> [r, c]
            d0 = torch.diagonal(factor.chains_pair_covariance(D, E, S, torch.from_numpy(np.stack([first, first], -1)).cuda()).view(C, 15, 15),
                                dim1=1, dim2=2)
            dl = torch.diagonal(factor.chains_pair_covariance(D, E, S, torch.from_numpy(np.stack([first + S - 1] * 2, -1)).cuda()).view(C, 15, 15),
                                dim1=1, dim2=2)
            diff = (got - Xs).abs()
            rec["diff_vs_solve15_of_block"] = float((diff.amax(dim=(1, 2)) / Xs.abs().amax(dim=(1, 2))).max())
            rec["diff_vs_solve15_of_diagonal"] = float((diff / torch.sqrt(d0[:, :, None] * dl[:, None, :])).max())
            rec["far_block_of_diagonal"] = float((Xs.abs() / torch.sqrt(d0[:, :, None] * dl[:, None, :])).amax(dim=(1, 2)).min())
        print(json.dumps(rec))
        del dp
        torch.cuda.empty_cache()
    n = 5000
    D, E = system(1, n, 2)
    rng = np.random.default_rng(0)
    pairs = rng.integers(0, n, (100_000, 2))
    dp = torch.from_numpy(pairs).cuda()
    ws = torch.empty(int(factor.capi.load().cpi_imu_chains_pair_covariance_workspace(1, n)) // 8 + 1, dtype=torch.float64, device="cuda")
    t_fwd = timed(lambda: factor.chains_pair_covariance(D, E, n, dp[:1], workspace=ws))
    t = timed(lambda: factor.chains_pair_covariance(D, E, n, dp, workspace=ws))
    fl = flops(n, np.zeros(n, dtype=np.int64), pairs[:2000])
    print(json.dumps(dict(case="long1e5", card=card, chains=1, states=n, pairs=len(pairs), ms=t, forward_and_root_ms=t_fwd, walk_ms=t - t_fwd,
                          flops_per_pair=float(fl.mean()), walk_gflops=float(fl.mean() * len(pairs) / max(t - t_fwd, 1e-9) / 1e6))))


if __name__ == "__main__":
    main()
