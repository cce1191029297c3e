"""numpy statement of the Rauch-Tung-Striebel backward recursion of filter runs (cpi_rts_smooth_batch, kernel K15; DESIGN.md section 3o).

Its inputs are K7's outputs: the filter's posterior (x_k, P_k) at every keyframe and, per transition, the prediction (xb_{k+1},
Pb_{k+1}) and the cross C_k = P_k A_k^T that cpi_propagate_batch writes from (x_k, P_k).  Vectorised over runs (the chain layout of
include/cpi_b200.h: run c holds keyframes o[c] .. o[c+1]-1, its transitions stored from o[c] - c) and parameterised by dtype, so that
the same code runs in float64 and in np.longdouble.  numpy.linalg has no long double: the 15x15 Cholesky and the triangular solves
are written out.  Per run, from the last keyframe (copied) backwards:

    G_k = C_k Pb_{k+1}^-1            (Pb_{k+1} = L L^T;  G_k^T = L^-T L^-1 C_k^T)
    d = local(xb_{k+1}, xs_{k+1}),   xs_k = retract(x_k, G_k d)
    Ps_k = P_k + G_k (Ps_{k+1} - Pb_{k+1}) G_k^T      (the lower triangle, mirrored: exactly symmetric)
    Xs_k = G_k Ps_{k+1}

Matrices are [.., 15, 15] (row, column); mat / vec convert the C ABI's column-major [n, 225]."""
from __future__ import annotations

import numpy as np


def mat(a, dtype=None):
    """[n, 225] column-major -> [n, 15, 15]"""
    a = np.asarray(a).reshape(-1, 15, 15).transpose(0, 2, 1)
    return a if dtype is None else a.astype(dtype)


def vec(A):
    """[n, 15, 15] -> [n, 225] column-major"""
    return np.ascontiguousarray(np.asarray(A).transpose(0, 2, 1).reshape(-1, 225))


def qmul(q, p):
    """cpi_common.cuh quat_multiply (JPL), batched [n, 4], in the inputs' dtype."""
    t = np.stack([q[:, 3] * p[:, 0] + q[:, 2] * p[:, 1] - q[:, 1] * p[:, 2] + q[:, 0] * p[:, 3],
                  -q[:, 2] * p[:, 0] + q[:, 3] * p[:, 1] + q[:, 0] * p[:, 2] + q[:, 1] * p[:, 3],
                  q[:, 1] * p[:, 0] - q[:, 0] * p[:, 1] + q[:, 3] * p[:, 2] + q[:, 2] * p[:, 3],
                  -q[:, 0] * p[:, 0] - q[:, 1] * p[:, 1] - q[:, 2] * p[:, 2] + q[:, 3] * p[:, 3]], axis=1)
    t[t[:, 3] < 0] *= -1
    return t / np.sqrt(np.sum(t * t, axis=1, keepdims=True))


def local(base, x):
    """local(x_lin, x), the inverse of JPLNavState::retract, batched [n, 16] -> [n, 15]; exactly 0 at x == x_lin."""
    one = x.dtype.type(1)
    dq = qmul(x[:, 0:4], base[:, 0:4] * np.array([-one, -one, -one, one], dtype=x.dtype))
    s = np.sqrt(np.sum(dq[:, 0:3] * dq[:, 0:3], axis=1))
    with np.errstate(invalid="ignore", divide="ignore"):
        k = np.where(s > 0, 2 * np.arctan2(s, dq[:, 3]) / np.where(s > 0, s, one), 2 * one)
    k[np.all(x[:, 0:4] == base[:, 0:4], axis=1)] = 0
    return np.concatenate([k[:, None] * dq[:, 0:3], x[:, 4:16] - base[:, 4:16]], axis=1)


def retract(x, xi):
    """JPLNavState::retract, batched [n, 16] (+) [n, 15]; xi = 0 gives the identity rotation step (the quaternion renormalised)."""
    one = x.dtype.type(1)
    th = np.sqrt(np.sum(xi[:, 0:3] * xi[:, 0:3], axis=1))
    with np.errstate(invalid="ignore", divide="ignore"):
        dq = np.concatenate([(np.sin(th / 2) / th)[:, None] * xi[:, 0:3], np.cos(th / 2)[:, None]], axis=1)
    dq = np.where(np.isnan(dq).any(axis=1, keepdims=True), np.array([0, 0, 0, one], dtype=x.dtype), dq)
    dq[dq[:, 3] < 0] *= -1
    q = qmul(dq, x[:, 0:4])
    return np.concatenate([q, x[:, 4:16] + xi[:, 3:15]], axis=1)


def cholesky(A):
    """Lower Cholesky factor of a batch [n, 15, 15] in A's dtype; a non-positive pivot gives NaN."""
    n, m = A.shape[0], A.shape[1]
    L = np.zeros_like(A)
    with np.errstate(invalid="ignore"):
        for j in range(m):
            s = A[:, j, j] - np.sum(L[:, j, :j] * L[:, j, :j], axis=1)
            L[:, j, j] = np.sqrt(np.where(s > 0, s, np.nan))
            for i in range(j + 1, m):
                L[:, i, j] = (A[:, i, j] - np.sum(L[:, i, :j] * L[:, j, :j], axis=1)) / L[:, j, j]
    return L


def solve_lower(L, B):
    """L^-1 B for lower triangular L [n, m, m] and B [n, m, r]."""
    Y = np.zeros_like(B)
    for i in range(L.shape[1]):
        Y[:, i] = (B[:, i] - np.einsum("nk,nkr->nr", L[:, i, :i], Y[:, :i])) / L[:, i, i, None]
    return Y


def solve_upper_t(L, B):
    """L^-T B for lower triangular L [n, m, m] and B [n, m, r]."""
    m = L.shape[1]
    Y = np.zeros_like(B)
    for i in range(m - 1, -1, -1):
        Y[:, i] = (B[:, i] - np.einsum("nk,nkr->nr", L[:, i + 1:, i], Y[:, i + 1:])) / L[:, i, i, None]
    return Y


def gain(C, Pb, dtype):
    """G = C Pb^-1 by the Cholesky of Pb: G^T = L^-T L^-1 C^T."""
    L = cholesky(Pb.astype(dtype))
    return solve_upper_t(L, solve_lower(L, np.swapaxes(C.astype(dtype), 1, 2))).swapaxes(1, 2)


def sym_lower(A):
    """A's lower triangle mirrored: exactly symmetric."""
    lo = np.tril(A)
    return lo + np.swapaxes(np.tril(A, -1), 1, 2)


def rts(offsets, x, P, xb, Pb, C, dtype=np.float64, inject=None, mirror=True):
    """The smoothed (xs [N,16], Ps [N,15,15], Xs [N - n_runs,15,15]) of the runs of `offsets` (int array [n_runs+1]) from the posteriors
    x [N,16], P [N,15,15] and K7's xb, Pb, C per transition, all in dtype.  inject: None, or a function (name, value) -> value applied
    to the intermediate values "Pb", "G" and "Ps"; mirror=False forms Ps without mirroring its lower triangle (both only for the
    sensitivity checks of the precision gate)."""
    inj = inject or (lambda name, v: v)
    o = np.asarray(offsets, dtype=np.int64)
    lens = o[1:] - o[:-1]
    x, P, xb, Pb, C = (np.asarray(a).astype(dtype) for a in (x, P, xb, Pb, C))
    xs, Ps = x.copy(), P.copy()
    Xs = np.zeros_like(C)
    for j in range(1, int(lens.max()) if len(lens) else 0):     # step j: keyframe o1 - 1 - j of every run longer than j
        r = np.nonzero(lens > j)[0]
        s = o[r + 1] - 1 - j
        t = s - r
        pb = inj("Pb", Pb[t])
        G = inj("G", gain(C[t], pb, dtype))
        d = local(xb[t], xs[s + 1])
        xs[s] = retract(x[s], np.einsum("nij,nj->ni", G, d))
        ps = inj("Ps", P[s] + G @ (Ps[s + 1] - pb) @ np.swapaxes(G, 1, 2))
        Ps[s] = sym_lower(ps) if mirror else ps
        Xs[t] = G @ Ps[s + 1]
    return xs, Ps, Xs


def errors(truth, got, layout):
    """Scaled errors of got = (xs, Ps, Xs) against truth, in the truth's smoothed standard deviations: per keyframe the worst of Ps
    [N], the components of local(xs_true, xs) [N, 15] (0 for a component of zero variance), and per transition the worst of Xs
    [N - n_runs] (in sqrt(Ps_k,ii Ps_k+1,jj)); a block equal to the truth has error 0 whatever its scale."""
    o = np.asarray(layout, dtype=np.int64)
    xt, Pt, Xt = (np.asarray(a, dtype=np.float64) for a in truth)
    xg, Pg, Xg = (np.asarray(a, dtype=np.float64) for a in got)
    sd = np.sqrt(np.abs(np.diagonal(Pt, axis1=1, axis2=2)))
    with np.errstate(invalid="ignore", divide="ignore"):
        eP = np.nan_to_num(np.abs(Pg - Pt) / (sd[:, :, None] * sd[:, None, :]), nan=np.inf).max(axis=(1, 2))
        eP[np.all(Pg == Pt, axis=(1, 2))] = 0.0
        ex = np.where(sd > 0, np.abs(local(xt, xg)) / np.where(sd > 0, sd, 1.0), 0.0)     # zero variance: checked exactly
        ks = np.concatenate([np.arange(o[c], o[c + 1] - 1) for c in range(len(o) - 1)]).astype(np.int64)
        eX = np.nan_to_num(np.abs(Xg - Xt) / (sd[ks][:, :, None] * sd[ks + 1][:, None, :]), nan=np.inf).max(axis=(1, 2)) if len(ks) else np.zeros(0)
        if len(ks):
            eX[np.all(Xg == Xt, axis=(1, 2))] = 0.0
    return eP, np.nan_to_num(ex, nan=np.inf), eX


def state_floor(truth):
    """[N, 15]: one ulp of the stored smoothed state per component (the quaternion: 2^-52 rad) in the truth's smoothed sd."""
    xt, Pt, _ = truth
    xt = np.asarray(xt, dtype=np.float64)
    sd = np.sqrt(np.abs(np.diagonal(np.asarray(Pt, dtype=np.float64), axis1=1, axis2=2)))
    ulp = np.concatenate([np.full((len(xt), 3), 2.0 ** -52), np.spacing(np.abs(xt[:, 4:16]))], axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(sd > 0, ulp / sd, 0.0)
