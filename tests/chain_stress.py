"""Seeded chain stress batch for the precision tests of the chain marginalisation (K8), the prior move (k_prior_at), the chain
assembly, the block cyclic reduction and the LM model decrease.

numpy only, plus the fp64 oracle that is passed in (it preintegrates the records and evaluates the factors):

  pool         the model-1 records of every ``stress.make_batch()`` window (1 kHz, 20-35 rad/s, gap and 10 000-sample windows
               included) and 20-sample 200 Hz windows; ``spd`` marks the records whose P_meas has a Cholesky factor (the gap
               windows' indefinite ones give NaN blocks, as k_factor_hessian does, and are kept for the isolation checks only)
  chains       chains of consecutive records at perturbed ``synth.make_states`` states, information blocks from the fp64 oracle's
               factors: every length in LENGTHS (each end case of the reduction), 20-sample chains, and one chain at positions
               of 1e6 m.  The 1 023 - 1 025 and 4 999 chains cycle through the whole pool.
  ragged       short chains whose boundaries fall on every residue mod 2^l, l <= 6, single-state chains at the start, at the
               end and back to back
  priors       none, 1e8 I, dense random, 1e12 I and nearly rank-deficient, cycling over the chains
  prior_at     state pairs in every branch of local15: equal quaternion bits, the sign-flipped quaternion, rotations of one ulp,
               1e-300, subnormal, 1e-8, 1, pi -/+ 1e-9 (w of either sign) and pi with w ~ 0 of either sign, positions of 1e6 m

``local_branches`` mirrors the branch decisions of local15 (marginalize.cu): quat_multiply's w < 0 flip, ``same`` and s == 0."""
from __future__ import annotations

import numpy as np

import stress
import test_marginalize as tmg
from cpi_b200 import synth

SEED = 20261018
LENGTHS = tuple(range(1, 10)) + (15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 1023, 1024, 1025, 4999)
PRIORS = ("none", "1e8", "dense", "1e12", "rankdef")
SIGMAS = np.array([0.005, 4e-6, 0.01, 0.0002])


def _threads():
    return synth.usable_cpus()


def pool(o64):
    """dict(records [n,290], lin [n,13], regime [n], spd [n])."""
    S, off, L, tags = stress.make_batch()
    rec = o64.preintegrate(1, S, L, SIGMAS, 0, offsets=off, nthreads=_threads())
    S2, L2 = synth.make_windows(64, 20, rate=200.0, first_window=41000, special=False)
    rec2 = o64.preintegrate(1, S2, L2, SIGMAS, 0, ns=20, nthreads=_threads())
    rec, lin = np.concatenate([rec, rec2]), np.concatenate([L, L2])
    regime = np.concatenate([tags, np.full(len(rec2), "syn20")])
    P = tmg.mat(rec[:, 65:290])
    spd = np.zeros(len(rec), dtype=bool)
    for i in range(len(rec)):
        d = np.diag(P[i])
        if np.all(d > 0) and rec[i, 19] > 0:
            try:
                np.linalg.cholesky(P[i] / np.sqrt(d[:, None] * d[None, :]))
                spd[i] = True
            except np.linalg.LinAlgError:
                pass
    return dict(records=rec, lin=lin, regime=regime, spd=spd)


def chains(o64, pl, lengths, rng, far=(), syn=False, spd_only=True):
    """Chains of the given state counts, concatenated in the C ABI's layout: dict(offsets [C+1], states [N,16], records / lin [N-C],
    G11 / G12 / G22 [N-C,225], g1 / g2 [N-C,15], f [N-C], regime [N-C]).  Chain c in ``far``: positions moved by 1e6 m.  syn: the
    20-sample windows only."""
    ok = pl["spd"] if spd_only else np.ones(len(pl["spd"]), dtype=bool)
    cand = np.flatnonzero(ok & ((pl["regime"] == "syn20") if syn else True))
    Xs, idx = [], []
    for c, S in enumerate(lengths):
        k = S - 1
        if k >= len(cand) // 2:                         # long chains: every record of the pool in turn
            start = int(rng.integers(0, len(cand)))
            ii = cand[(start + np.arange(k)) % len(cand)]
        else:
            ii = cand[rng.integers(0, len(cand), size=k)]
        X = synth.make_states(pl["records"][ii], pl["lin"][ii], 1, seed=SEED + c) if k else synth.make_states(pl["records"][:0], pl["lin"][:1], 1, seed=SEED + c)
        if c in far:
            X[:, 13:16] += 1e6 * np.array([0.6, -0.48, 0.64])
        Xs.append(X); idx.append(ii)
    off = np.r_[0, np.cumsum(lengths)].astype(np.int64)
    ii = np.concatenate(idx).astype(np.int64)
    X = np.concatenate(Xs)
    rec, lin = pl["records"][ii], pl["lin"][ii]
    C = len(lengths)
    chain_of = np.repeat(np.arange(C), np.asarray(lengths) - 1)
    ia = np.arange(len(ii)) + chain_of
    e, H1, H2 = o64.factor_eval(1, X, rec, lin, idx_i=ia, idx_j=ia + 1, nthreads=_threads())
    with np.errstate(divide="ignore", invalid="ignore"):
        G = list(tmg._np_hessian(rec, e, H1, H2))
    G[0], G[2] = 0.5 * (G[0] + G[0].transpose(0, 2, 1)), 0.5 * (G[2] + G[2].transpose(0, 2, 1))   # exactly symmetric, as K3/K4's
    bad = ~pl["spd"][ii]
    out = dict(offsets=off, states=X, records=rec, lin=lin, regime=pl["regime"][ii], G11=tmg.vec(G[0]), G12=tmg.vec(G[1]),
               G22=tmg.vec(G[2]), g1=G[3], g2=G[4], f=G[5])
    for k in ("G11", "G12", "G22", "g1", "g2", "f"):     # k_factor_hessian's NaN where P_meas has no Cholesky factor
        out[k] = np.array(out[k]); out[k][bad] = np.nan
    return out


def concat(lays, head_flags):
    """Layouts one after the other (offsets shifted, factors back to back); "head" marks the chains of layouts flagged 1."""
    out = {}
    for k in ("states", "records", "lin", "regime", "G11", "G12", "G22", "g1", "g2", "f"):
        out[k] = np.concatenate([l[k] for l in lays])
    sizes = np.concatenate([np.diff(l["offsets"]) for l in lays])
    out["offsets"] = np.r_[0, np.cumsum(sizes)].astype(np.int64)
    out["head"] = np.concatenate([np.full(len(l["offsets"]) - 1, bool(h)) for l, h in zip(lays, head_flags)])
    return out


def main_lengths():
    return list(LENGTHS) + [21] * 6 + [40]


def ragged_lengths(rng):
    """Short chains with a boundary on every residue mod 64 (so mod every 2^l, l <= 6), single-state chains first, last and back
    to back."""
    while True:
        sizes = [1] + list(rng.integers(1, 10, size=180)) + [1, 1, 1] + list(rng.integers(1, 10, size=20)) + [1]
        b = np.cumsum(sizes)[:-1]
        if len(set(b % 64)) == 64:
            return sizes


def priors(rng, C, kinds=PRIORS):
    """(info [C,225], rhs [C,15], f [C], kind [C]) cycling over kinds; "none" is zero."""
    info, rhs, f, kind = np.zeros((C, 225)), np.zeros((C, 15)), np.zeros(C), []
    for c in range(C):
        k = kinds[c % len(kinds)]
        kind.append(k)
        if k == "none":
            continue
        if k in ("1e8", "1e12"):
            A = np.eye(15) * float(k)
        elif k == "dense":
            A = tmg.random_prior(rng, scale=(1e-3, 1e-4, 1e-2, 1e-3, 1e-2))[0]
        else:                                           # nearly rank-deficient: one direction held 1e-10 as firmly as the rest
            Q, _ = np.linalg.qr(rng.normal(size=(15, 15)))
            ev = np.full(15, 1e8); ev[0] = 1e-2
            A = (Q * ev) @ Q.T
            A = 0.5 * (A + A.T)
        info[c] = tmg.vec(A[None])[0]
        rhs[c] = rng.normal(size=15) * np.sqrt(np.diag(A)) * 1e-3
        f[c] = rng.uniform(1, 10)
    return info, rhs, f, np.array(kind)


# ---------------------------------------------------------------------------------------------- prior_at

def _qmul_raw(q, p):
    """quat_multiply's product before its w < 0 flip (cpi_common.cuh), batched [n,4]."""
    return np.stack([q[:, 3] * p[:, 0] + q[:, 2] * p[:, 1] - q[:, 1] * p[:, 2] + q[:, 0] * p[:, 3],
                     -q[:, 2] * p[:, 0] + q[:, 3] * p[:, 1] + q[:, 0] * p[:, 2] + q[:, 1] * p[:, 3],
                     q[:, 1] * p[:, 0] - q[:, 0] * p[:, 1] + q[:, 3] * p[:, 2] + q[:, 2] * p[:, 3],
                     -q[:, 0] * p[:, 0] - q[:, 1] * p[:, 1] - q[:, 2] * p[:, 2] + q[:, 3] * p[:, 3]], axis=1)


def local_branches(lin, x):
    """(flip, same, s0) per pair: quat_multiply's w < 0 flip, the equal-bits branch and the s == 0 branch of local15."""
    qi = lin[:, 0:4] * np.array([-1, -1, -1, 1.0])
    t = _qmul_raw(x[:, 0:4], qi)
    flip = t[:, 3] < 0
    t = np.where(flip[:, None], -t, t)
    dq = t / np.sqrt(np.sum(t * t, axis=1, keepdims=True))
    s = np.sqrt(dq[:, 0] * dq[:, 0] + dq[:, 1] * dq[:, 1] + dq[:, 2] * dq[:, 2])
    same = np.all(x[:, 0:4] == lin[:, 0:4], axis=1)
    return flip, same, (s == 0) & ~same


def _unit_q(rng, n):
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[q[:, 3] < 0] *= -1
    return q


def prior_at_batch(rng):
    """dict(lin [n,16], x [n,16], info [n,225], rhs [n,15], f [n], regime [n], identity [n]): every pair twice, with a dense random
    prior and with info = I, rhs = 0 (there rhs' = -delta exactly, so local15's delta is read directly)."""
    lins, xs, tags = [], [], []

    def add(lin, x, tag):
        lins.append(lin); xs.append(x); tags.extend([tag] * len(lin))

    def base(n, q=None):
        L = np.zeros((n, 16)); L[:, 0:4] = _unit_q(rng, n) if q is None else q
        L[:, 4:16] = rng.normal(size=(n, 12))
        X = L.copy(); X[:, 4:16] += rng.normal(size=(n, 12)) * 1e-2
        return L, X

    def rotated(L, X, angle, w_sign=None):
        ax = rng.normal(size=(len(L), 3)); ax /= np.linalg.norm(ax, axis=1, keepdims=True)
        dq = np.concatenate([np.sin(angle / 2) * ax, np.full((len(L), 1), np.cos(angle / 2))], axis=1)
        if w_sign is not None:
            dq[:, 3] = w_sign * np.abs(rng.normal(size=len(L))) * 1e-17
            dq[:, 0:3] = ax * np.sqrt(1 - dq[:, 3:4] ** 2)
        t = _qmul_raw(dq, L[:, 0:4])                      # x = dq (x) q_lin, the rotation of retract, w sign as it falls
        X[:, 0:4] = t / np.linalg.norm(t, axis=1, keepdims=True)
        return X

    L, X = base(16); X[:, 0:4] = L[:, 0:4]; add(L, X, "same")
    L, X = base(16); X[:, 0:4] = -L[:, 0:4]; add(L, X, "flipped")
    L, X = base(16); X[:, 0:4] = L[:, 0:4]
    j = rng.integers(0, 4, 16); X[np.arange(16), j] = np.nextafter(L[np.arange(16), j], 2.0); add(L, X, "ulp")
    for tag, a in (("1e-300", 1e-300), ("subnormal", 1e-310)):
        ident = np.tile([0, 0, 0, 1.0], (16, 1))
        L, X = base(16, ident)
        ax = rng.normal(size=(16, 3)); ax /= np.linalg.norm(ax, axis=1, keepdims=True)
        X[:, 0:3] = ax * a; X[:, 3] = 1.0
        add(L, X, tag)
    for tag, a in (("1e-8", 1e-8), ("1", 1.0), ("pi-1e-9", np.pi - 1e-9), ("pi+1e-9", np.pi + 1e-9)):
        L, X = base(32); add(L, rotated(L, X, a), tag)
    for tag, sg in (("pi+", 1.0), ("pi-", -1.0)):
        L, X = base(48); add(L, rotated(L, X, np.pi, sg), tag)
    L, X = base(24)
    L[:, 13:16] = rng.normal(size=(24, 3)) * 1e6; X[:, 13:16] = L[:, 13:16] + rng.normal(size=(24, 3)) * 1e-6
    add(L, rotated(L, X, 0.1), "far")
    lin, x = np.concatenate(lins), np.concatenate(xs)
    n = len(lin)
    info = np.zeros((2 * n, 225)); rhs = np.zeros((2 * n, 15)); f = np.zeros(2 * n)
    for i in range(n):
        p = tmg.random_prior(rng)
        info[i], rhs[i], f[i] = tmg.vec(p[0][None])[0], p[1], p[2]
        info[n + i] = tmg.vec(np.eye(15)[None])[0]
        f[n + i] = rng.uniform(1, 10)
    tags = np.array(tags)
    return dict(lin=np.concatenate([lin, lin]), x=np.concatenate([x, x]), info=info, rhs=rhs, f=f,
                regime=np.concatenate([tags, tags]), identity=np.r_[np.zeros(n, dtype=bool), np.ones(n, dtype=bool)])


def check_prior_at_coverage(b):
    flip, same, s0 = local_branches(b["lin"], b["x"])
    seen = dict(flip=int(flip.sum()), no_flip=int((~flip).sum()), same=int(same.sum()), s0=int(s0.sum()))
    assert all(v > 0 for v in seen.values()), f"local15 branches not all taken: {seen}"
    return seen
