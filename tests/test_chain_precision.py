"""Precision of the solver side of the IMU chain -- the chain marginalisation (K8, cpi_imu_chain_marginalize), the prior move
(k_prior_at), the chain assembly (k_chain_assemble / _lm), the block cyclic reduction (k_chain_ids, k_bcr_*) and the
LM model decrease (k_lm_terms, k_lm_decide) -- against an extended-precision truth.

The truths are the long-double build of the oracle's dense statements (oracle/cpi_oracle.c: oracle_chain_marginalize, oracle_local /
oracle_prior_at, oracle_chain_solve, oracle_lm_terms).  Inputs: the chain stress batch of tests/chain_stress.py.  Errors are
measured per block, each relative to the size of the terms that cancel into it, never as a whole-matrix or whole-vector norm:
  K8        every 3x3 block of Lambda relative to |G22| + |Z|^T |Z| of the last step, every 3-block of eta likewise, f relative to
            |f_prior| + sum f_k + sum z^T z;
  prior_at  delta per 3-block (delta_theta modulo the antipodal pair where the truth's |w| < 1e-12), rhs' per component relative to
            |rhs| + |info| |delta|, f' relative to |f| + 2 |rhs|^T |delta| + |delta|^T |info| |delta|; delta_theta = 2 dq_v cancels
            from products of unit-quaternion components, so its size counts 2 more (what any fp64 route resolves), and where the
            truth's |w| < 1e-12 rhs' and f' are also compared with the antipodal delta's;
  solve     per chain and per component type (theta, b_g, v, b_a, p) over the chain's states, |dx| / |x_true|;
  LM        the model decrease m_c per chain relative to sum |delta|^T (2 |rhs| + |H| |delta|).
The gate is e_dev <= K max(e_64, floor), K = 8, floor = 1e-15 (parity.gate_errors), with e_64 the larger fp64 error of the routes
named for each quantity: the fp64 oracle recurrence and test_marginalize's plain and Jacobi-scaled numpy recurrences (K8), the fp64 local (prior_at), the fp64 sequential block Cholesky and the fp64
restatement of the reduction in solve.cu's order (solve), the fp64 oracle terms (LM).

CPU tests: the truth agrees with the refined-fp64 truth of test_gpu_parity and with a long-double dense Schur complement, the
long-double local inverts retract, the gate passes the fp64 routes and fails five injected errors that the older flat gates pass.
GPU tests: every kernel on the batch; DESIGN.md section 5 lists the measured worst ratios."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest

import chain_stress as cs
import test_marginalize as tmg
from parity import gate_errors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K, FLOOR = 8.0, 1e-15
COMP = ("theta", "b_g", "v", "b_a", "p")
THETA_SIZE = 2.0


@pytest.fixture(scope="module")
def oracles():
    """(fp64, long double) oracles, rebuilt when older than their source (the entry points used here are newer than the rest)."""
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("long double has no extended precision on this platform")
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "liboracle.so", "liboracle_ld.so"], check=True)
    from oracle import oracle as om
    return om.Oracle(), om.OracleLD()


_cache = {}


def batch(o64):
    """The pool, the main layout (every LENGTHS chain, 20-sample chains, a chain at 1e6 m), the ragged layout, chains with the gap
    records' NaN blocks left in (for the isolation checks), and the K8 layout: the main chains, 20-sample chains and five 1 025-state
    20-sample chains (the long heads)."""
    if "b" not in _cache:
        rng = np.random.default_rng(cs.SEED)
        pl = cs.pool(o64)
        ml = cs.main_lengths()
        main = cs.chains(o64, pl, ml, rng, far=(len(ml) - 1,))
        main["syn"] = cs.chains(o64, pl, [21] * 6, rng, syn=True)
        rl = cs.ragged_lengths(rng)
        ragged = cs.chains(o64, pl, rl, rng)
        nan = cs.chains(o64, pl, [12] * 40, rng, spd_only=False)
        head = cs.chains(o64, pl, [1025] * 5, rng, syn=True)
        _cache["b"] = dict(pool=pl, main=main, ragged=ragged, nan=nan, k8=cs.concat([main, main["syn"], head], [0, 0, 1]), rng=rng)
    return _cache["b"]


def worst_line(label, worst):
    k = max(worst, key=lambda f: worst[f]["ratio"])
    print(f"{label}: worst ratio {worst[k]['ratio']:.3f} ({k})")


def _threads():
    return cs._threads()


# ---------------------------------------------------------------------------------------------- K8

def marg_inputs(b, o64):
    """n_marg per chain of the K8 layout: 0, 1, S - 1 and random (at most 64 on the stress chains longer than 200 states: an
    undamped head of hundreds of those records loses positive definiteness in fp64 itself), and the 20-sample heads of 1 000 and
    1 024 states; priors cycling."""
    if "marg" not in _cache:
        m = b["k8"]
        off = m["offsets"]
        S = np.diff(off)
        rng = np.random.default_rng(cs.SEED + 1)
        nm = np.array([(0, 1, s - 1, int(rng.integers(0, s)))[c % 4] for c, s in enumerate(S)], dtype=np.int64)
        nm = np.minimum(np.maximum(nm, 0), S - 1)
        nm[(S > 200) & (S < 1025)] = np.minimum(nm[(S > 200) & (S < 1025)], 64)
        nm[S == 4999] = 64
        heads = np.flatnonzero(m["head"])
        nm[heads] = np.where(np.arange(len(heads)) % 2 == 0, 1000, 1024)
        pi, pr, pf, kind = cs.priors(rng, len(S))
        _cache["marg"] = (nm, (pi, pr, pf), kind)
    return _cache["marg"]


def k8_errors(got, truth, scale):
    """dict field -> [C]: Lambda blocks "L_IJ" (I <= J), eta blocks "eta_I" and "f", each relative to its cancelling scale."""
    gi, gr, gf = got
    ti, tr, tf = truth
    C = len(tf)
    Gi, Ti, Si = tmg.mat(gi), tmg.mat(ti), tmg.mat(scale[:, :225])
    out = {}

    def rel(num, den):
        return np.where(den > 0, num / np.where(den > 0, den, 1.0), np.where(num > 0, np.inf, 0.0))

    for I in range(5):
        for J in range(I, 5):
            s = (slice(None), slice(3 * I, 3 * I + 3), slice(3 * J, 3 * J + 3))
            out[f"L_{I}{J}"] = rel(np.linalg.norm((Gi[s] - Ti[s]).reshape(C, -1), axis=1), np.linalg.norm(Si[s].reshape(C, -1), axis=1))
        s = slice(3 * I, 3 * I + 3)
        out[f"eta_{I}"] = rel(np.linalg.norm(gr[:, s] - tr[:, s], axis=1), np.linalg.norm(scale[:, 225:240][:, s], axis=1))
    out["f"] = rel(np.abs(gf - tf), scale[:, 240])
    return out


def k8_truths(b, o64, old):
    if "k8" not in _cache:
        m = b["k8"]
        nm, prior, _ = marg_inputs(b, o64)
        blk = [m[k] for k in ("G11", "G12", "G22", "g1", "g2", "f")]
        t = old.chain_marginalize(*blk, nm, prior, chain_offsets=m["offsets"], nthreads=_threads())
        f = o64.chain_marginalize(*blk, nm, prior, chain_offsets=m["offsets"], nthreads=_threads())
        _cache["k8"] = (t, (f, numpy_marginalize(m, nm, prior, False), numpy_marginalize(m, nm, prior, True)))
    return _cache["k8"]


def numpy_marginalize(m, nm, prior, jacobi):
    """The other fp64 routes: test_marginalize.marginalize_ref (LAPACK Cholesky and triangular solves) per chain, plain or on the
    Jacobi-scaled M."""
    off = m["offsets"]
    C = len(off) - 1
    oi, orr, of = np.zeros((C, 225)), np.zeros((C, 15)), np.zeros(C)
    for c in range(C):
        k = int(nm[c])
        if k == 0:
            continue
        sl = slice(int(off[c] - c), int(off[c] - c) + k)
        L, e, fc = tmg.marginalize_ref(tmg.mat(m["G11"][sl]), tmg.mat(m["G12"][sl]), tmg.mat(m["G22"][sl]), m["g1"][sl], m["g2"][sl], m["f"][sl],
                                       k, (tmg.mat(prior[0][c])[0], prior[1][c], prior[2][c]), jacobi=jacobi)
        oi[c], orr[c], of[c] = tmg.vec(L[None])[0], e, fc
    return oi, orr, of


def k8_gate(got, t, f, nm):
    """f: the fp64 routes (the oracle recurrence, numpy's plain and Jacobi-scaled); e_64 per field and chain the largest of their
    errors."""
    sel = nm > 0
    pick = lambda x: tuple(a[sel] for a in x[:3])
    ed = k8_errors(pick(got), pick(t), t[3][sel])
    es = [k8_errors(pick(r), pick(t), t[3][sel]) for r in f]
    e64 = {k: np.max(np.stack([e[k] for e in es]), axis=0) for k in ed}
    return gate_errors(ed, e64, K, FLOOR)


# ---------------------------------------------------------------------------------------------- assembly and solve

DAMPINGS = (("lam0", 0.0, False), ("lamI", 1e-3, False), ("marquardt", 1e-5, True))


def assemble(lay, lams, diag, pinfo, prhs):
    """numpy statement of k_chain_assemble(_lm) in the kernel's order of additions: (D, E, rhs, damp)."""
    off = lay["offsets"]
    C, N = len(off) - 1, int(off[-1])
    c = np.repeat(np.arange(C), np.diff(off))
    k = np.arange(N)
    first, last = k == off[c], k == off[c + 1] - 1
    fr = k - c
    D, rhs = np.zeros((N, 225)), np.zeros((N, 15))
    D[~first] = D[~first] + lay["G22"][fr[~first] - 1]; rhs[~first] = rhs[~first] + lay["g2"][fr[~first] - 1]
    D[~last] = D[~last] + lay["G11"][fr[~last]]; rhs[~last] = rhs[~last] + lay["g1"][fr[~last]]
    if pinfo is not None:
        D[first] = D[first] + pinfo[c[first]]; rhs[first] = rhs[first] + prhs[c[first]]
    lam = np.broadcast_to(np.asarray(lams, dtype=np.float64), (C,))[c]
    d = D[:, ::16]
    a = lam[:, None] * np.clip(d, 1e-6, 1e32) if diag else np.repeat(lam[:, None], 15, axis=1)
    D[:, ::16] = d + a
    E = np.zeros((max(N - 1, 1), 225))
    nl = np.flatnonzero(~last[:N - 1])
    E[nl] = lay["G12"][fr[nl]]
    return D, E[:N - 1], rhs, a


def solve_systems(b, which):
    """(name, lambda (scalar or per chain), Marquardt?, prior info, prior rhs, prior kinds) per damping of one layout."""
    key = ("sys", which)
    if key not in _cache:
        lay = b[which]
        C = len(lay["offsets"]) - 1
        rng = np.random.default_rng(cs.SEED + 2)
        out = []
        for name, lam, diag in DAMPINGS:
            if lam == 0 and which == "main":      # undamped, the long stress chains are singular in fp64 for any elimination order
                continue
            # undamped under the nearly rank-deficient prior a chain is singular to working precision (fp64 errors ~1e-4): that
            # prior is solved damped only
            kinds = cs.PRIORS[1:4] if lam == 0 else cs.PRIORS
            pi, pr, _, kind = cs.priors(rng, C, kinds)
            out.append((name, lam, diag, pi, pr, kind))
        lams = 10.0 ** rng.uniform(-8, 4, C)
        pi, pr, _, kind = cs.priors(rng, C)
        out.append(("per-chain", lams, True, pi, pr, kind))
        _cache[key] = out
    return _cache[key]


def solve_errors(x, xt, off):
    """dict component -> [C]: |dx| / |x_true| over each chain's states."""
    C = len(off) - 1
    out = {}
    for t, name in enumerate(COMP):
        s = slice(3 * t, 3 * t + 3)
        num, den = np.zeros(C), np.zeros(C)
        for c in range(C):
            num[c] = np.linalg.norm(x[off[c]:off[c + 1], s] - xt[off[c]:off[c + 1], s])
            den[c] = np.linalg.norm(xt[off[c]:off[c + 1], s])
        out[name] = np.where(den > 0, num / np.where(den > 0, den, 1.0), np.where(num > 0, np.inf, 0.0))
    return out


def solve_truths(o64, old, key, off, D, E, rhs):
    if key not in _cache:
        t = old.chain_solve(D, E, rhs, 0, chain_offsets=off, nthreads=_threads())
        s = o64.chain_solve(D, E, rhs, 0, chain_offsets=off, nthreads=_threads())
        r = o64.chain_solve(D, E, rhs, 1, chain_offsets=off)
        _cache[key] = (t, s, r)
    return _cache[key]


def solve_gate(x, t, s, r, off):
    ed = solve_errors(x, t, off)
    es, er = solve_errors(s, t, off), solve_errors(r, t, off)
    e64 = {k: np.maximum(es[k], er[k]) for k in es}
    return gate_errors(ed, e64, K, FLOOR)


# ---------------------------------------------------------------------------------------------- prior_at

def prior_errors(rhs_o, f_o, delta, b, t_rhs, t_f, t_delta):
    """dict: delta blocks (identity priors; delta_theta modulo the antipodal pair where the truth's |w| < 1e-12), rhs' per
    component and f', each relative to its scale."""
    info = tmg.mat(b["info"])
    ad = np.abs(t_delta)
    ad[:, 0:3] += THETA_SIZE                               # delta_theta cancels from products of unit quaternion components: size 2
    iad = np.einsum("nrc,nc->nr", np.abs(info), ad)
    out = {}
    sc_r = np.abs(b["rhs"]) + iad
    rel = lambda num, den: np.where(den > 0, num / np.where(den > 0, den, 1.0), np.where(num > 0, np.inf, 0.0))
    idn = b["identity"]
    th = t_delta[:, 0:3]
    nth = np.linalg.norm(th, axis=1, keepdims=True)
    anti = th - 2 * np.pi * th / np.where(nth > 0, nth, 1.0)
    w = np.abs(_dq_w(b))
    da = t_delta.copy(); da[:, 0:3] = anti
    ua = np.einsum("nrc,nc->nr", info, da)
    ra, fa = b["rhs"] - ua, b["f"] - 2 * np.einsum("nr,nr->n", b["rhs"], da) + np.einsum("nr,nr->n", da, ua)
    er = np.abs(rhs_o - t_rhs)
    ef = np.abs(f_o - t_f)
    er = np.where(w[:, None] < 1e-12, np.minimum(er, np.abs(rhs_o - ra)), er)
    ef = np.where(w < 1e-12, np.minimum(ef, np.abs(f_o - fa)), ef)
    out["rhs"] = np.max(rel(er, sc_r), axis=1)
    out["f"] = rel(ef, np.abs(b["f"]) + 2 * np.einsum("nr,nr->n", np.abs(b["rhs"]), ad) + np.einsum("nr,nr->n", ad, iad))
    for I in range(5):
        s = slice(3 * I, 3 * I + 3)
        num = np.linalg.norm(delta[:, s] - t_delta[:, s], axis=1)
        if I == 0:
            num = np.where(w < 1e-12, np.minimum(num, np.linalg.norm(delta[:, s] - anti, axis=1)), num)
        den = np.linalg.norm(t_delta[:, s], axis=1)
        out[f"delta_{I}"] = np.where(idn, rel(num, np.maximum(den, THETA_SIZE) if I == 0 else den), 0.0)
    return out


def _dq_w(b):
    t = cs._qmul_raw(b["x"][:, 0:4], b["lin"][:, 0:4] * np.array([-1, -1, -1, 1.0]))
    return t[:, 3] / np.linalg.norm(t, axis=1)


def prior_batch():
    if "pa" not in _cache:
        b = cs.prior_at_batch(np.random.default_rng(cs.SEED + 3))
        cs.check_prior_at_coverage(b)
        _cache["pa"] = b
    return _cache["pa"]


def prior_truths(o64, old):
    if "pat" not in _cache:
        b = prior_batch()
        args = (b["info"], b["rhs"], b["f"], b["lin"], b["x"])
        t = old.prior_at(*args) + (old.local(b["lin"], b["x"]),)
        f = o64.prior_at(*args) + (o64.local(b["lin"], b["x"]),)
        _cache["pat"] = (t, f)
    return _cache["pat"]


def prior_gate(got, t, f):
    b = prior_batch()
    ed = prior_errors(*got, b, *t)
    e64 = prior_errors(*f, b, *t)
    return gate_errors(ed, e64, K, FLOOR)


# ---------------------------------------------------------------------------------------------- LM

def lm_gate(m_dev, t, f):
    """m per chain relative to its terms' size; e_64 the fp64 oracle's."""
    sc = t[:, 1]
    rel = lambda m: np.where(sc > 0, np.abs(m - t[:, 0]) / np.where(sc > 0, sc, 1.0), np.where(m != t[:, 0], np.inf, 0.0))
    return gate_errors({"m": rel(m_dev)}, {"m": rel(f[:, 0])}, K, FLOOR)


def lm_decide(t, lam, params):
    """k_lm_decide's rule on the long-double sums (tries / iterations from 0): (status, lam, accept, rho, rho bound)."""
    m, cur, nw, moved = t[:, 0], t[:, 2], t[:, 3], t[:, 4] != 0
    rho = (cur - nw) / np.where(m != 0, m, 1.0)
    bound = 16 * 2.0 ** -53 * (np.abs(rho) * t[:, 1] + np.abs(cur) + np.abs(nw)) / np.where(m != 0, np.abs(m), 1e-300)
    st = np.zeros(len(m), dtype=np.int32); lo = lam.copy(); acc = np.zeros(len(m), dtype=bool)
    for c in range(len(m)):
        if not (np.isfinite(cur[c]) and np.isfinite(m[c])):
            st[c] = 4
        elif not moved[c]:
            st[c] = 1
        elif np.isfinite(nw[c]) and m[c] > 0 and rho[c] > params.min_model_fidelity:
            acc[c] = True
            lo[c] = max(lam[c] / params.lambda_factor, params.lambda_lower)
            dec = cur[c] - nw[c]
            if 0.5 * dec <= params.absolute_error_tol or dec <= params.relative_error_tol * cur[c]:
                st[c] = 1
            elif 1 >= params.max_iterations:
                st[c] = 2
        elif lam[c] >= params.lambda_upper:
            st[c] = 3
        else:
            lo[c] = lam[c] * params.lambda_factor
    return st, lo, acc, rho, bound


def lm_inputs(b, o64, old):
    """Inputs of cpi_imu_chains_lm_update on the ragged layout, Marquardt-damped with a lambda per chain: delta = s_c x, x the damped
    step, s_c in (1, 1e-8, 2, 1.999, 0) (near 2, m cancels down to the damping's share; 1e-8: near convergence), candidate costs set
    so that the long-double rho falls on either side of min_model_fidelity, near it and far from it.  dict with the long-double /
    fp64 oracle terms."""
    if "lm" not in _cache:
        lay = b["ragged"]
        off = lay["offsets"]
        C = len(off) - 1
        rng = np.random.default_rng(cs.SEED + 4)
        lams = 10.0 ** rng.uniform(-8, 4, C)
        lams[25] = 1e5                             # a full step rejected at the upper bound: lambda exhausted
        pi, pr, _, _ = cs.priors(rng, C, cs.PRIORS[1:])
        D, E, rhs, damp = assemble(lay, lams, True, pi, pr)
        x = o64.chain_solve(D, E, rhs, 0, chain_offsets=off, nthreads=_threads())
        s = np.array([(1.0, 1e-8, 2.0, 1.999, 0.0)[c % 5] for c in range(C)])
        delta = x * np.repeat(s, np.diff(off))[:, None]
        f_cur = np.abs(lay["f"]); f_new = f_cur.copy()
        pf_cur = rng.uniform(1e3, 1e4, C)
        t0 = old.lm_terms(rhs, D, E, damp, delta, f_cur, f_new, pf_cur, pf_cur, chain_offsets=off, nthreads=_threads())
        rho = np.array([(1.5, -0.5, 1e-3 + 1e-9, 1e-3 - 1e-9, 0.5, 1e-3 * (1 + 1e-15))[c % 6] for c in range(C)])
        pf_new = pf_cur - rho * t0[:, 0]
        t = old.lm_terms(rhs, D, E, damp, delta, f_cur, f_new, pf_cur, pf_new, chain_offsets=off, nthreads=_threads())
        f = o64.lm_terms(rhs, D, E, damp, delta, f_cur, f_new, pf_cur, pf_new, chain_offsets=off, nthreads=_threads())
        _cache["lm"] = dict(off=off, D=D, E=E, rhs=rhs, damp=damp, delta=delta, f_cur=f_cur, f_new=f_new, pf_cur=pf_cur, pf_new=pf_new,
                            lam=lams, t=t, f=f, s=s)
    return _cache["lm"]


# ---------------------------------------------------------------------------------------------------------- CPU

def test_batch_covers_its_regimes(oracles):
    o64, _ = oracles
    b = batch(o64)
    m = b["main"]
    S = np.diff(m["offsets"])
    assert set(cs.LENGTHS) <= set(S)
    assert {"rate1000", "fast", "long", "gaps", "syn20"} <= set(m["regime"]) | set(b["main"]["syn"]["regime"])
    assert np.all(np.isfinite(m["G11"])) and np.all(np.isfinite(b["ragged"]["G11"]))
    assert np.any(np.isnan(b["nan"]["G11"][:, 0])), "no gap window with an indefinite P_meas in the isolation chains"
    assert np.max(np.abs(m["states"][:, 13:16])) > 9e5
    rb = b["ragged"]["offsets"][1:-1]
    for l in range(1, 7):
        assert len(set(rb % 2 ** l)) == 2 ** l, l
    sr = np.diff(b["ragged"]["offsets"])
    assert sr[0] == 1 and sr[-1] == 1 and np.any((sr[:-1] == 1) & (sr[1:] == 1))
    nm, _, kind = marg_inputs(b, o64)
    S8 = np.diff(b["k8"]["offsets"])
    assert set(kind) == set(cs.PRIORS) and 0 in nm and 1 in nm and np.any(nm == S8 - 1) and nm.max() >= 1000
    print("prior_at branches of local15:", cs.check_prior_at_coverage(prior_batch()))


def test_extended_solve_agrees_with_the_refined_truth(oracles):
    """The long-double sequential solve against test_gpu_parity's refined-fp64 truth, per chain and component, within 1e-2 e_64, on
    the chains of 2 .. 130 states of the main layout (lambda I and Marquardt)."""
    from test_gpu_parity import _chain_truth
    o64, old = oracles
    b = batch(o64)
    m = b["main"]
    off = m["offsets"]
    worst = 0.0
    for name, lam, diag, pi, pr, _ in solve_systems(b, "main")[0:2]:
        D, E, rhs, _ = assemble(m, lam, diag, pi, pr)
        t, s, r = solve_truths(o64, old, ("main", name), off, D, E, rhs)
        for c in range(len(off) - 1):
            lo, hi = off[c], off[c + 1]
            if hi - lo < 2 or hi - lo > 130:
                continue
            xr, x64 = _chain_truth(D[lo:hi], E[lo:hi - 1], rhs[lo:hi])
            e_t = solve_errors(t[lo:hi], xr, np.array([0, hi - lo]))
            e64 = solve_errors(x64, xr, np.array([0, hi - lo]))
            for k in COMP:
                if e64[k][0] > 0:
                    worst = max(worst, e_t[k][0] / e64[k][0])
                assert e_t[k][0] <= 1e-2 * max(e64[k][0], 1e-16), (name, c, k, e_t[k][0], e64[k][0])
    print(f"long-double sequential vs refined fp64: worst {worst:.1e} of e_64")


def _ld_solve(A, B):
    """Gauss-Jordan in numpy long double (A square, B columns)."""
    A, B = A.astype(np.longdouble).copy(), B.astype(np.longdouble).copy()
    n = len(A)
    for i in range(n):
        p = A[i, i]
        A[i] /= p; B[i] /= p
        for j in range(n):
            if j != i and A[j, i] != 0:
                g = A[j, i]
                A[j] -= g * A[i]; B[j] -= g * B[i]
    return B


def test_extended_recurrence_is_the_dense_schur_complement(oracles):
    """On chains of 2 .. 6 states with every prior kind: the long-double recurrence and a long-double dense Schur complement of the
    head system (Gauss-Jordan, no pivoting) agree per chain to 1e-14 of the size of the cancelling terms, or to the fp64
    recurrence's distance where that is larger (heads under a 1e12 prior): an algebra slip would be orders of magnitude above."""
    o64, old = oracles
    b = batch(o64)
    lay = b["ragged"]
    off = lay["offsets"]
    rng = np.random.default_rng(7)
    sel = [c for c in range(len(off) - 1) if 2 <= off[c + 1] - off[c] <= 6][:25]
    pi, pr, pf, _ = cs.priors(rng, len(off) - 1)
    nm = np.zeros(len(off) - 1, dtype=np.int64)
    for c in sel:
        nm[c] = off[c + 1] - off[c] - 1
    blk = [lay[k] for k in ("G11", "G12", "G22", "g1", "g2", "f")]
    t = old.chain_marginalize(*blk, nm, (pi, pr, pf), chain_offsets=off)
    f = o64.chain_marginalize(*blk, nm, (pi, pr, pf), chain_offsets=off)
    worst = 0.0
    for c in sel:
        m = int(nm[c]); f0 = int(off[c] - c)
        sl = slice(f0, f0 + m)
        A, bb, F = tmg.dense_head(tmg.mat(lay["G11"][sl]), tmg.mat(lay["G12"][sl]), tmg.mat(lay["G22"][sl]), lay["g1"][sl], lay["g2"][sl],
                                  lay["f"][sl], m, (tmg.mat(pi[c])[0], pr[c], pf[c]))
        A = np.tril(A) + np.tril(A, -1).T
        n = 15 * m
        Y = _ld_solve(A[:n, :n], np.concatenate([A[:n, n:], bb[:n, None]], axis=1))
        S = A[n:, n:].astype(np.longdouble) - A[n:, :n].astype(np.longdouble) @ Y[:, :15]
        eta = bb[n:].astype(np.longdouble) - A[n:, :n].astype(np.longdouble) @ Y[:, 15]
        fm = np.longdouble(F) - bb[:n].astype(np.longdouble) @ Y[:, 15]
        sc = t[3][c]
        dense = (tmg.vec(S.astype(np.float64)[None])[0], eta.astype(np.float64), float(fm))
        err = lambda o: max(np.max(np.abs(o[0][c] - dense[0]) / sc[:225]), np.max(np.abs(o[1][c] - dense[1]) / sc[225:240]),
                            abs(o[2][c] - dense[2]) / sc[240])
        e_ld, e_64 = err(t), err(f)
        worst = max(worst, e_ld / max(e_64, 1e-300))
        assert e_ld <= max(e_64, 1e-14), (c, e_ld, e_64)
    print(f"long-double recurrence vs long-double dense Schur complement: worst {worst:.1e} of the fp64 recurrence's distance")


def test_extended_local_inverts_retract(oracles):
    """retract(x_lin, local(x_lin, x)) = x in every prior_at regime (quaternion up to sign), long double and fp64."""
    o64, old = oracles
    b = prior_batch()
    for o in (old, o64):
        d = o.local(b["lin"], b["x"])
        y = o64.retract(b["lin"], d)
        eq = np.minimum(np.linalg.norm(y[:, 0:4] - b["x"][:, 0:4], axis=1), np.linalg.norm(y[:, 0:4] + b["x"][:, 0:4], axis=1))
        assert eq.max() <= 1e-15, (b["regime"][np.argmax(eq)], eq.max())
        assert np.max(np.abs(y[:, 4:] - b["x"][:, 4:])) <= 1e-9
    same = np.all(b["lin"][:, 0:4] == b["x"][:, 0:4], axis=1)
    assert np.all(old.local(b["lin"], b["x"])[same, 0:3] == 0.0)


def test_gate_passes_the_fp64_routes(oracles):
    o64, old = oracles
    b = batch(o64)
    nm, _, _ = marg_inputs(b, o64)
    t, f = k8_truths(b, o64, old)
    for r in f:
        ratio, worst, bad = k8_gate(r, t, f, nm)
        assert not bad, bad
    for r, name in zip(f[1:], ("plain", "Jacobi-scaled")):
        _, w_one, _ = k8_gate(r, t, f[:1], nm)
        print(f"K8: numpy's {name} fp64 route against the oracle recurrence's e_64 alone: {max(v['ratio'] for v in w_one.values()):.2f}")
    t, f = prior_truths(o64, old)
    assert not prior_gate(f, t, f)[2]
    for which in ("main", "ragged"):
        lay = b[which]
        for name, lam, diag, pi, pr, _ in solve_systems(b, which):
            D, E, rhs, _ = assemble(lay, lam, diag, pi, pr)
            t, s, r = solve_truths(o64, old, (which, name), lay["offsets"], D, E, rhs)
            for x in (s, r):
                _, worst, bad = solve_gate(x, t, s, r, lay["offsets"])
                assert not bad, (which, name, bad)
            _, w_seq, _ = gate_errors(solve_errors(r, t, lay["offsets"]), solve_errors(s, t, lay["offsets"]), K, FLOOR)
            print(which, name, f"fp64 reduction against the sequential e_64 alone: {max(v['ratio'] for v in w_seq.values()):.2f}")
    d = lm_inputs(b, o64, old)
    assert not lm_gate(d["f"][:, 0], d["t"], d["f"])[2]


def test_gate_fails_injected_errors_that_the_old_gates_pass(oracles):
    """One Lambda block rounded to fp32; b_g and b_a of a lambda-I solve scaled by 1 + 1e-7; local without the w < 0 flip at the
    near-pi pairs; m_c with the damping not subtracted; the last step's z^T z dropped from f."""
    o64, old = oracles
    b = batch(o64)
    nm, _, _ = marg_inputs(b, o64)
    t, f = k8_truths(b, o64, old)
    c = int(np.flatnonzero(nm >= 5)[0])
    got = tuple(a.copy() for a in f[0][:3])
    Lm = tmg.mat(got[0][c])[0]
    Lm[9:12, 9:12] = Lm[9:12, 9:12].astype(np.float32).astype(np.float64)
    got[0][c] = tmg.vec(Lm[None])[0]
    bad = k8_gate(got, t, f, nm)[2]
    assert any(x.startswith("L_33") for x in bad), bad
    got = tuple(a.copy() for a in f[0][:3])
    got[2][c] += t[3][c, 241]
    assert any(x.startswith("f") for x in k8_gate(got, t, f, nm)[2])
    # the solve
    lay = b["main"]
    off = lay["offsets"]
    name, lam, diag, pi, pr, _ = solve_systems(b, "main")[0]
    D, E, rhs, _ = assemble(lay, lam, diag, pi, pr)
    t, s, r = solve_truths(o64, old, ("main", name), off, D, E, rhs)
    x = s.copy()
    x[:, 3:6] *= 1 + 1e-7; x[:, 9:12] *= 1 + 1e-7
    bad = solve_gate(x, t, s, r, off)[2]
    assert any(x_.startswith("b_g") for x_ in bad) and any(x_.startswith("b_a") for x_ in bad), bad
    # prior_at: local without the flip
    pb = prior_batch()
    tp, fp = prior_truths(o64, old)
    flip, _, _ = cs.local_branches(pb["lin"], pb["x"])
    raw = cs._qmul_raw(pb["x"][:, 0:4], pb["lin"][:, 0:4] * np.array([-1, -1, -1, 1.0]))
    dq = raw / np.linalg.norm(raw, axis=1, keepdims=True)
    s_ = np.linalg.norm(dq[:, 0:3], axis=1)
    d = fp[2].copy()
    near = flip & np.isin(pb["regime"], ("pi+", "pi-", "pi+1e-9"))
    assert near.sum() > 0
    d[near, 0:3] = (2 * np.arctan2(s_[near], dq[near, 3]) / s_[near])[:, None] * dq[near, 0:3]
    rhs_o = pb["rhs"] - np.einsum("nrc,nc->nr", tmg.mat(pb["info"]), d)
    f_o = pb["f"] - 2 * np.einsum("nr,nr->n", pb["rhs"], d) + np.einsum("nr,nrc,nc->n", d, tmg.mat(pb["info"]), d)
    rhs_o[pb["identity"]] = -d[pb["identity"]]
    bad = prior_gate((rhs_o, f_o, d), tp, fp)[2]
    assert any(x_.startswith("delta_0") for x_ in bad), bad
    # LM: the damping not subtracted
    dl = lm_inputs(b, o64, old)
    m_nd = o64.lm_terms(dl["rhs"], dl["D"], dl["E"], np.zeros_like(dl["damp"]), dl["delta"], dl["f_cur"], dl["f_new"], dl["pf_cur"],
                        dl["pf_new"], chain_offsets=dl["off"])[:, 0]
    assert lm_gate(m_nd, dl["t"], dl["f"])[2]


# ---------------------------------------------------------------------------------------------------------- GPU

def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.gpu
def test_marginalize_against_extended_oracle(cuda, oracles):
    """K8 on the K8 layout (n_marg 0, 1, S - 1, random, heads of 1 000 and 1 024 states; every prior kind): Lambda, eta and f per block;
    Lambda exactly symmetric; m = 0 the prior's bits; NaN in exactly the chains with a non-positive pivot."""
    from cpi_b200 import factor
    torch = cuda
    o64, old = oracles
    b = batch(o64)
    m = b["k8"]
    nm, prior, _ = marg_inputs(b, o64)
    t, f = k8_truths(b, o64, old)
    G = [_dev(torch, m[k]) for k in ("G11", "G12", "G22", "g1", "g2", "f")]
    dp = tuple(_dev(torch, a) for a in prior)
    got = [a.cpu().numpy() for a in factor.chain_marginalize(*G, _dev(torch, m["offsets"]), _dev(torch, nm), prior=dp)]
    Lm = tmg.mat(got[0])
    assert np.array_equal(Lm, Lm.transpose(0, 2, 1))
    z = nm == 0
    assert np.array_equal(got[0][z], prior[0][z]) and np.array_equal(got[1][z], prior[1][z]) and np.array_equal(got[2][z], prior[2][z])
    _, w_one, _ = k8_gate(got, t, f[:1], nm)
    ratio, worst, bad = k8_gate(got, t, f, nm)
    worst_line(f"K8 (Lambda, eta, f per block; oracle-only e_64: {max(v['ratio'] for v in w_one.values()):.2f})", worst)
    assert not bad, bad
    # NaN isolation: chains holding a gap record's NaN block or a negated G11 in their eliminated head
    n = b["nan"]
    Gn = [n[k].copy() for k in ("G11", "G12", "G22", "g1", "g2", "f")]
    Gn[0][5 * 11 + 2] *= -1                                      # chain 5, third factor: a negative pivot
    C = len(n["offsets"]) - 1
    nmn = np.full(C, 11, dtype=np.int64)
    ref = o64.chain_marginalize(*Gn, nmn, None, chain_offsets=n["offsets"])
    got = factor.chain_marginalize(*[_dev(torch, a) for a in Gn], _dev(torch, n["offsets"]), _dev(torch, nmn))
    gi = got[0].cpu().numpy()
    bad_ref = np.isnan(ref[2])
    assert bad_ref[5] and 0 < bad_ref.sum() < C
    assert np.array_equal(np.isnan(gi).any(axis=1), bad_ref) and np.all(np.isnan(gi[bad_ref]))
    print(f"K8 NaN isolation: {int(bad_ref.sum())} of {C} chains non-finite, as the oracle's pivots say")


@pytest.mark.gpu
def test_prior_at_against_extended_oracle(cuda, oracles):
    from cpi_b200 import factor
    torch = cuda
    o64, old = oracles
    pb = prior_batch()
    t, f = prior_truths(o64, old)
    r, fo = factor.prior_at(*[_dev(torch, pb[k]) for k in ("info", "rhs", "f", "lin", "x")])
    r, fo = r.cpu().numpy(), fo.cpu().numpy()
    d = np.where(pb["identity"][:, None], -r, 0.0)
    assert np.array_equal(r[pb["identity"]], -d[pb["identity"]])
    ratio, worst, bad = prior_gate((r, fo, d), t, f)
    worst_line("prior_at (delta, rhs', f')", worst)
    assert not bad, bad


def _check_assembly(got, ref, diag):
    """E, rhs and the damping added bit for bit; D bit for bit except the Marquardt-damped diagonal, within one ulp (fma)."""
    D, E, rhs, damp = tuple(a.cpu().numpy() for a in got[:3]) + ((got[3].cpu().numpy(),) if len(got) > 3 else (None,))
    Dr, Er, rr, ar = ref
    assert np.array_equal(E, Er) and np.array_equal(rhs, rr)
    off = np.ones(225, dtype=bool)
    if diag:
        off[::16] = False
        assert np.all(np.abs(D[:, ~off] - Dr[:, ~off]) <= np.spacing(np.abs(Dr[:, ~off])))
    assert np.array_equal(D[:, off], Dr[:, off])
    if damp is not None:
        assert np.array_equal(damp, ar)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["main", "ragged"])
def test_assembly_and_solve_against_extended_oracle(cuda, oracles, which):
    """Every damping (lambda = 0, lambda I, Marquardt, a lambda per chain through chains_assemble_lm) on both layouts: the assembly
    bit for bit against the numpy statement, chain_solve and chains_solve per chain and component against the long-double
    sequential solve, chains_solve bitwise chain_solve, and (ragged) a non-SPD chain at each boundary residue mod 64 leaves every
    other chain bitwise as it was."""
    from cpi_b200 import factor
    torch = cuda
    o64, old = oracles
    b = batch(o64)
    lay = b[which]
    off = lay["offsets"]
    doff = _dev(torch, off)
    G = [_dev(torch, lay[k]) for k in ("G11", "G12", "G22", "g1", "g2")]
    C = len(off) - 1
    for name, lam, diag, pi, pr, _ in solve_systems(b, which):
        ref = assemble(lay, lam, diag, pi, pr)
        if name == "per-chain":
            got = factor.chains_assemble_lm(*G, doff, _dev(torch, lam), _dev(torch, pi), _dev(torch, pr), diagonal_damping=diag)
        else:
            got = factor.chains_assemble(*G, doff, lam, _dev(torch, pi), _dev(torch, pr), diagonal_damping=diag)
        _check_assembly(got, ref, diag)
        D, E, rhs = got[:3]
        x = factor.chain_solve(D, E, rhs)
        xi = factor.chains_solve(D, E, rhs, doff)
        t, s, r = solve_truths(o64, old, (which, name), off, D.cpu().numpy(), E.cpu().numpy(), rhs.cpu().numpy())
        bads = {}
        for label, xx in (("chain_solve", x), ("chains_solve", xi)):
            xh = xx.cpu().numpy()
            _, w_seq, _ = gate_errors(solve_errors(xh, t, off), solve_errors(s, t, off), K, FLOOR)
            ratio, worst, bads[label] = solve_gate(xh, t, s, r, off)
            worst_line(f"{label} {which} {name} (sequential-only e_64: {max(v['ratio'] for v in w_seq.values()):.2f})", worst)
        same = torch.equal(x, xi)
        assert same and not bads["chain_solve"] and not bads["chains_solve"], (name, "isolated solve bitwise the plain one:", same, bads)
    if which != "ragged":
        return
    healthy = xi.cpu().numpy()
    starts = off[:-1]
    done = set()
    for c in range(C):
        r64 = int(starts[c] % 64)
        if r64 in done:
            continue
        done.add(r64)
        Db = D.clone()
        Db[int(starts[c])] *= -1
        xb = factor.chains_solve(Db, E, rhs, doff).cpu().numpy()
        lo, hi = off[c], off[c + 1]
        assert np.isnan(xb[lo:hi]).any(), c
        assert np.array_equal(np.delete(xb, np.s_[lo:hi], axis=0), np.delete(healthy, np.s_[lo:hi], axis=0)), c
    assert len(done) == 64
    print(f"non-SPD chain at each of the {len(done)} boundary residues mod 64: every other chain bitwise unchanged")


@pytest.mark.gpu
def test_lm_terms_against_extended_oracle(cuda, oracles):
    """cpi_imu_chains_lm_update on prepared inputs: the per-state terms summed per chain against the long-double m_c; the delta != 0
    flag and the factor costs per state exactly; where the long-double rho is farther from min_model_fidelity than its error bound,
    the device's accept / reject, lambda and status equal the long-double decision."""
    from cpi_b200 import capi
    torch = cuda
    o64, old = oracles
    d = lm_inputs(batch(o64), o64, old)
    off = d["off"]
    C, N = len(off) - 1, int(off[-1])
    params = capi.LMParams(absolute_error_tol=0.0, relative_error_tol=0.0, max_iterations=100)
    lib = capi.load()
    X = np.zeros((N, 16)); X[:, 3] = 1.0
    Xn = X.copy(); Xn[:, 4:16] = 1.0
    a = {k: _dev(torch, v) for k, v in d.items() if isinstance(v, np.ndarray) and v.dtype == np.float64}
    dX, dXn, doff = _dev(torch, X), _dev(torch, Xn), _dev(torch, off)
    lam = a["lam"].clone()
    cost = torch.zeros(C, dtype=torch.float64, device="cuda")
    i32 = lambda: torch.zeros(C, dtype=torch.int32, device="cuda")
    status, iters, tries = i32(), i32(), i32()
    ws = torch.empty((int(lib.cpi_imu_chains_lm_workspace(N)) + 7) // 8, dtype=torch.float64, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    capi.check(lib.cpi_imu_chains_lm_update(C, p(doff), 0, N, ctypes.byref(params), p(a["f_cur"]), p(a["pf_cur"]), p(a["f_new"]), p(a["pf_new"]),
                                            p(a["rhs"]), p(a["D"]), p(a["E"]), p(a["damp"]), p(a["delta"]), p(dXn), p(dX), p(lam), p(cost),
                                            p(status), p(iters), p(tries), None, p(ws), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    terms = ws[:4 * N].cpu().numpy().reshape(N, 4)
    k = np.arange(N)
    c_of = np.repeat(np.arange(C), np.diff(off))
    last = k == off[c_of + 1] - 1
    assert np.array_equal(terms[:, 3], (d["delta"] != 0).any(axis=1).astype(np.float64))
    assert np.array_equal(terms[~last, 1], d["f_cur"][(k - c_of)[~last]]) and np.all(terms[last, 1:3] == 0)
    m_dev = np.array([math.fsum(terms[off[c]:off[c + 1], 0]) for c in range(C)])
    ratio, worst, bad = lm_gate(m_dev, d["t"], d["f"])
    worst_line("LM model decrease m_c", worst)
    assert not bad, bad
    st, lo, acc, rho, bound = lm_decide(d["t"], d["lam"], params)
    clear = (np.abs(rho - params.min_model_fidelity) > bound) | (d["t"][:, 4] == 0)
    assert clear.sum() >= C // 2 and (~clear).sum() > 0 and acc[clear].any() and (~acc[clear]).any()
    assert set(st[clear]) >= {0, 1, 3}
    ds, dl = status.cpu().numpy(), lam.cpu().numpy()
    assert np.array_equal(ds[clear], st[clear]) and np.array_equal(dl[clear], lo[clear])
    X_out = dX.cpu().numpy()
    moved = np.repeat(acc, np.diff(off))
    assert np.array_equal(X_out[moved & np.repeat(clear, np.diff(off))], Xn[moved & np.repeat(clear, np.diff(off))])
    print(f"LM decisions: {int(clear.sum())} of {C} chains clear of the fidelity threshold, all equal to the long-double rule")
