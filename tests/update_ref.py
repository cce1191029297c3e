"""numpy statement of the filter's measurement update (cpi_state_update_batch, DESIGN.md section 3k), the loader of its plain-C oracle
(tests/update_oracle.c, compiled on first use into a temporary directory in fp64 and long double) and the stress batch of the
precision gate.  Layouts as include/cpi_b200.h: states [n,16], covariances and informations [n,225] column-major."""
from __future__ import annotations

import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

from test_marginalize import local, mat, vec
from test_propagate import qmul, random_cov

_HERE = os.path.dirname(os.path.abspath(__file__))
CHI2_3_999 = 16.266236196238129          # the 0.999 quantile of chi^2_3


def retract(x, xi):
    """JPLNavState::retract, batched [n,16] (+) [n,15]."""
    x, xi = np.atleast_2d(x), np.atleast_2d(xi)
    th = np.linalg.norm(xi[:, 0:3], axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        dq = np.concatenate([(np.sin(th / 2) / th)[:, None] * xi[:, 0:3], np.cos(th / 2)[:, None]], axis=1)
    dq = np.where(np.isnan(dq).any(axis=1, keepdims=True), np.array([0, 0, 0, 1.0]), dq)
    dq[dq[:, 3] < 0] *= -1
    q = qmul(dq, x[:, 0:4])
    q[q[:, 3] < 0] *= -1
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return np.concatenate([q, x[:, 4:16] + xi[:, 3:15]], axis=1)


def update_ref(x, cov, W, xb):
    """The update in the square-root form of the kernel, batched.  Returns (x+ [n,16], cov+ [n,225], xi [n,15], gamma [n])."""
    S, Wm = mat(cov), mat(W)
    d = local(xb, x)
    L = np.linalg.cholesky(S)
    C = np.linalg.cholesky(np.eye(15) + L.transpose(0, 2, 1) @ Wm @ L)
    u = (L.transpose(0, 2, 1) @ (Wm @ d[:, :, None]))[:, :, 0]
    v = np.linalg.solve(C, u[:, :, None])
    w = np.linalg.solve(C.transpose(0, 2, 1), v)[:, :, 0]
    xi = -(L @ w[:, :, None])[:, :, 0]
    M = np.linalg.solve(C, L.transpose(0, 2, 1)).transpose(0, 2, 1)          # L C^-T
    P = M @ M.transpose(0, 2, 1)
    s = d + xi
    g = np.einsum("ni,nij,nj->n", s, Wm, s) + np.einsum("ni,ni->n", w, w)
    return retract(x, xi), vec(P), xi, g


def update_info(x, cov, W, xb):
    """The same statement in information form, (Sigma^-1 + W)^-1, batched; returns as update_ref."""
    S, Wm = mat(cov), mat(W)
    d = local(xb, x)
    Si = np.linalg.inv(S)
    P = np.linalg.inv(Si + Wm)
    P = 0.5 * (P + P.transpose(0, 2, 1))
    xi = -(P @ (Wm @ d[:, :, None]))[:, :, 0]
    s = d + xi
    g = np.einsum("ni,nij,nj->n", s, Wm, s) + np.einsum("ni,nij,nj->n", xi, Si, xi)
    return retract(x, xi), vec(P), xi, g


def update_kalman(x, cov, W, xb, rows):
    """The textbook Kalman update with H selecting the rows `rows` (W = H^T R^-1 H, R = W[rows, rows]^-1), batched."""
    S, Wm = mat(cov), mat(W)
    d = local(xb, x)
    H = np.eye(15)[list(rows)]
    R = np.linalg.inv(Wm[:, rows][:, :, rows])
    Sy = H @ S @ H.T + R
    K = S @ H.T @ np.linalg.inv(Sy)
    y = -(H @ d.T).T                                               # z - H x = H (x_bar - x) = -H d
    xi = (K @ y[:, :, None])[:, :, 0]
    P = (np.eye(15) - K @ H) @ S
    g = np.einsum("ni,nij,nj->n", y, np.linalg.inv(Sy), y)
    return retract(x, xi), vec(0.5 * (P + P.transpose(0, 2, 1))), xi, g


_LIBS = {}


def oracle(long_double=False):
    """The plain-C statement (tests/update_oracle.c) in fp64 or long double, compiled on first use with oracle/Makefile's flags."""
    key = bool(long_double)
    if key not in _LIBS:
        tmp = tempfile.mkdtemp(prefix="cpi_update_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        out = os.path.join(tmp, f"libupdate{'_ld' if key else ''}.so")
        cmd = [os.environ.get("CC", "gcc"), "-std=c11", "-O2", "-fPIC", "-shared", "-fno-fast-math", "-ffp-contract=off", "-o", out,
               os.path.join(_HERE, "update_oracle.c"), "-lm"] + (["-DCPI_ORACLE_LONG_DOUBLE"] if key else [])
        subprocess.run(cmd, check=True)
        lib = ctypes.CDLL(out)
        P = ctypes.POINTER(ctypes.c_double)
        lib.oracle_state_update.argtypes = [ctypes.c_int64, P, P, P, P, ctypes.c_int, P, P, P, P]
        lib.oracle_state_update.restype = ctypes.c_int
        _LIBS[key] = lib
    return _LIBS[key]


def oracle_update(x, cov, W, xb, order, long_double=False):
    """oracle_state_update: order 0 the square-root form, 1 the information form.  Returns as update_ref."""
    a = [np.ascontiguousarray(v, dtype=np.float64) for v in (x, cov, W, xb)]
    n = a[0].shape[0]
    xo, co, xi, g = np.zeros((n, 16)), np.zeros((n, 225)), np.zeros((n, 15)), np.zeros(n)
    P = lambda v: v.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    assert oracle(long_double).oracle_state_update(n, *[P(v) for v in a], int(order), P(xo), P(co), P(xi), P(g)) == 0
    return xo, co, xi, g


# ---------------------------------------------------------------------------------------------- inputs

def unit_states(rng, n, far=False):
    x = np.zeros((n, 16))
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True); q[q[:, 3] < 0] *= -1
    x[:, 0:4] = q
    x[:, 4:16] = rng.normal(size=(n, 12)) * np.repeat([1e-3, 1.0, 1e-2, 10.0], 3)
    if far:
        x[:, 13:16] += rng.normal(size=(n, 3)) * 1e6
    return x


def info_of(kind, rng, sigma=1e-2):
    """One W [15,15]: 'pos', 'vel', 'att', 'bg', 'ba' (isotropic 1/sigma^2 on that block), 'posvel', 'full' (random PSD of rank 15),
    'rank' (random PSD of rank 5) or 'zero'."""
    W = np.zeros((15, 15))
    blocks = dict(att=0, bg=3, vel=6, ba=9, pos=12)
    if kind in blocks:
        b = blocks[kind]
        G = rng.normal(size=(3, 3)) * 0.2 + np.eye(3)
        W[b:b + 3, b:b + 3] = G @ G.T / sigma ** 2
    elif kind == "posvel":
        W[12:15, 12:15] = np.eye(3) / sigma ** 2
        W[6:9, 6:9] = np.eye(3) / (10 * sigma) ** 2
    elif kind in ("full", "rank"):
        G = rng.normal(size=(15, 15 if kind == "full" else 5))
        W = G @ G.T / sigma ** 2
    W = 0.5 * (W + W.T)
    return W


def rows_of(kind):
    return dict(att=[0, 1, 2], bg=[3, 4, 5], vel=[6, 7, 8], ba=[9, 10, 11], pos=[12, 13, 14], posvel=[6, 7, 8, 12, 13, 14],
                full=list(range(15)))[kind]


def fix_near(rng, x, W, scale=1.0):
    """x_bar = x moved by a draw of N(0, W^+ scale^2) on W's blocks (the attitude by retract): d = local(x_bar, x) is of order scale."""
    n = len(x)
    xb = x.copy()
    for i in range(n):
        Wi = mat(W[i:i + 1])[0]
        ev, U = np.linalg.eigh(Wi)
        pos = ev > ev.max() * 1e-14 if ev.max() > 0 else np.zeros(15, bool)
        e = U[:, pos] @ (rng.normal(size=pos.sum()) / np.sqrt(ev[pos])) * scale
        xb[i] = retract(x[i:i + 1], e[None])[0]
    return xb


def conditioned_cov(rng, n, cond):
    """n random SPD covariances with eigenvalues log-spaced from 1 down to 1/cond, column-major [n,225]."""
    Q, _ = np.linalg.qr(rng.normal(size=(n, 15, 15)))
    ev = np.logspace(0, -np.log10(cond), 15)
    S = Q @ (ev[None, :, None] * Q.transpose(0, 2, 1))
    return vec(0.5 * (S + S.transpose(0, 2, 1)))


def stress_batch(rng, extra_cov=None):
    """dict(x, cov, W, xb, tag): every kind of W (position at 1 mm .. 1 um and 1e-8, entries up to 1e16; velocity, attitude, biases,
    full, rank 5, weak 1e-12, zero) against dead-reckoning-like, random, tight (position sd ~5e-5 m, so that the 1e16 fixes stay below
    the limit) and conditioned covariances, fixes at d = 0, near x and 5 m off, and the quaternion branches of local15
    (chain_stress.prior_at_batch's pairs, x_bar the linearisation point).  Filters whose lambda_max(W Sigma) exceeds SHARPEST are
    left out: the fp64 square-root form's limit (DESIGN.md section 3k)."""
    import chain_stress
    covs = [random_cov(rng, 24), random_cov(rng, 24, scale=(1e-2, 1e-5, 1.0, 1e-3, 10.0)), conditioned_cov(rng, 24, 1e12),
            conditioned_cov(rng, 24, 1e8), random_cov(rng, 24, scale=(2e-6, 2e-8, 2e-5, 2e-6, 5e-5))]
    if extra_cov is not None:
        covs.append(np.asarray(extra_cov))
    covs = np.concatenate(covs)
    kinds = [("pos", 1e-3), ("pos", 1e-6), ("pos", 1e-8), ("vel", 1e-2), ("att", 1e-3), ("bg", 1e-5), ("ba", 1e-3), ("posvel", 1e-2),
             ("full", 1e-2), ("rank", 1e-1), ("full", 1e6), ("zero", 1.0)]
    xs, cs, ws, xbs, tags = [], [], [], [], []
    for k, (kind, sigma) in enumerate(kinds):
        for mode in ("near", "zero_d", "outlier"):
            m = len(covs)
            x = unit_states(rng, m, far=(k % 3 == 2))
            W = vec(np.stack([info_of(kind, rng, sigma) for _ in range(m)]))
            if mode == "near":
                xb = fix_near(rng, x, W)
            elif mode == "zero_d":
                xb = x.copy()
            else:
                xb = x.copy(); xb[:, 13:16] += 5.0 / np.sqrt(3)
            xs.append(x); cs.append(covs); ws.append(W); xbs.append(xb); tags += [f"{kind}@{sigma:g}/{mode}"] * m
    b = chain_stress.prior_at_batch(rng)
    m = len(b["lin"])
    xs.append(b["x"]); xbs.append(b["lin"]); cs.append(random_cov(rng, m))
    # an attitude fix half a turn away is ill-posed (local15's axis flips with the sign of a w of 1e-17): position fixes there
    ws.append(vec(np.stack([info_of("pos" if str(r).startswith("pi") else ("att", "full", "pos")[i % 3], rng, 1e-2)
                            for i, r in enumerate(b["regime"])])))
    tags += [f"branch/{r}" for r in b["regime"]]
    b = dict(x=np.concatenate(xs), cov=np.concatenate(cs), W=np.concatenate(ws), xb=np.concatenate(xbs), tag=np.array(tags))
    keep = sharpness(b["cov"], b["W"]) <= SHARPEST
    return {k: v[keep] for k, v in b.items()}


SHARPEST = 1e12        # the largest eigenvalue of W Sigma the square-root form handles in fp64 (DESIGN.md section 3k)


def sharpness(cov, W):
    """The largest eigenvalue of W Sigma per filter (of L^T W L): how much sharper the fix is than the prior, squared."""
    L = np.linalg.cholesky(mat(cov))
    return np.linalg.eigvalsh(L.transpose(0, 2, 1) @ mat(W) @ L)[:, -1]


def errors(truth, got, x):
    """Per-filter scaled errors of got = (x+, cov+, gamma) against truth (x+, cov+, gamma): cov+ per 3x3 block pair [n,5,5] in
    units of sqrt(truth_ii truth_jj), x+ per component [n,15] as local(x+_true, x+) in the truth's posterior standard deviations,
    gamma [n] relative to max(gamma, 1) (a chi-square value: absolute below 1)."""
    xt, ct, gt = truth
    xg, cg, gg = got
    T, G = mat(ct), mat(cg)
    dg = np.sqrt(np.abs(np.diagonal(T, axis1=1, axis2=2)))
    E = np.abs(G - T) / (dg[:, :, None] * dg[:, None, :])
    eb = E.reshape(-1, 5, 3, 5, 3).max(axis=(2, 4))
    ex = np.abs(local(xt, xg)) / dg
    eg = np.abs(gg - gt) / np.maximum(gt, 1.0)
    return eb, ex, eg
