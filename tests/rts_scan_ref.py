"""numpy statement of the parallel-in-time Rauch-Tung-Striebel smoother of filter runs (cpi_rts_smooth_scan_batch, kernel K16;
DESIGN.md section 3p).

Inputs are rts_ref's: the filter's posteriors (x_k, P_k) and K7's (xb_{k+1}, Pb_{k+1}, C_k) per transition, in the chain layout.
Per transition k (keyframes k -> k+1):

    G_k  = C_k Pb_{k+1}^-1                       (rts_ref.gain)
    L_k  = P_k - G_k Pb_{k+1} G_k^T              (the lower triangle, mirrored)
    d0_k = local(xb_{k+1}, x_{k+1}),   J_k = diag(Jr^-1(phi), I_12),  phi = d0_k[0:3]

The element of keyframe k is (E, L, B, a) = (G_k, L_k, G_k J_k, G_k d0_k); a run's last keyframe holds (0, P_{S-1}, 0, 0).  Elements
compose as (E_o, L_o, B_o, a_o) o (E_i, L_i, B_i, a_i) = (E_o E_i, L_o + E_o L_i E_o^T, B_o B_i, a_o + B_o a_i), and the suffix
composition at k holds (Ps_k, delta_k); xs_k = retract(x_k, delta_k), Xs_k = G_k Ps_{k+1}, the last keyframe copied.

Two bracketings: `sequential` (the backward recursion, vectorised over runs) and `tree` (a Kogge-Stone scan over the reflected flat
index with the run boundaries applied by selection, vectorised over every keyframe).  Both run in the dtype they are given."""
from __future__ import annotations

import numpy as np

import rts_ref as rr


def jr_inv(phi):
    """Jr^-1(phi) [n, 3, 3] = I + [phi]x / 2 + (1 - (t/2) cot(t/2)) / t^2 [phi]x^2, t = |phi| (the series below 1e-4), in phi's dtype:
    d Log(Exp(phi) Exp(delta)) / d delta at 0, the attitude block of d local(xb, retract(x, delta)) / d delta."""
    one = phi.dtype.type(1)
    t2 = np.sum(phi * phi, axis=1)
    t = np.sqrt(t2)
    with np.errstate(invalid="ignore", divide="ignore"):
        h = t / 2
        k = np.where(t < 1e-4, one / 12 + t2 / 720, (one - h * np.cos(h) / np.sin(h)) / np.where(t2 > 0, t2, one))
    K = np.zeros((len(phi), 3, 3), dtype=phi.dtype)
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -phi[:, 2], phi[:, 1], -phi[:, 0]
    K[:, 1, 0], K[:, 2, 0], K[:, 2, 1] = phi[:, 2], -phi[:, 1], phi[:, 0]
    return np.eye(3, dtype=phi.dtype)[None] + K / 2 + k[:, None, None] * (K @ K)


def elements(offsets, x, P, xb, Pb, C, dtype=np.float64, inject=None, mirror=True):
    """(E, L, B, a, flag) per keyframe in keyframe order ([N,15,15] x 3, [N,15], [N] bool: a run's last keyframe).  inject: None or
    (name, value) -> value on "Pb" and "G"; mirror=False leaves L's upper triangle as computed (sensitivity checks only)."""
    inj = inject or (lambda name, v: v)
    o = np.asarray(offsets, dtype=np.int64)
    x, P, xb, Pb, C = (np.asarray(a).astype(dtype) for a in (x, P, xb, Pb, C))
    N, R = len(x), len(o) - 1
    run = np.repeat(np.arange(R), o[1:] - o[:-1])
    flag = np.zeros(N, dtype=bool)
    flag[o[1:] - 1] = True
    E, B = np.zeros((N, 15, 15), dtype=dtype), np.zeros((N, 15, 15), dtype=dtype)
    L, a = P.copy(), np.zeros((N, 15), dtype=dtype)
    s = np.nonzero(~flag)[0]
    if len(s):
        t = s - run[s]
        pb = inj("Pb", Pb[t])
        G = inj("G", rr.gain(C[t], pb, dtype))
        d0 = rr.local(xb[t], x[s + 1])
        E[s] = G
        Bs = G.copy()
        Bs[:, :, 0:3] = G[:, :, 0:3] @ jr_inv(d0[:, 0:3])
        B[s] = Bs
        a[s] = np.einsum("nij,nj->ni", G, d0)
        Ls = P[s] - G @ pb @ np.swapaxes(G, 1, 2)
        L[s] = rr.sym_lower(Ls) if mirror else Ls
    return E, L, B, a, flag


def compose(o, i, mirror=True):
    """o (outer) composed with i, each (E, L, B, a) batched."""
    Eo, Lo, Bo, ao = o
    Ei, Li, Bi, ai = i
    L = Lo + Eo @ Li @ np.swapaxes(Eo, 1, 2)
    return Eo @ Ei, rr.sym_lower(L) if mirror else L, Bo @ Bi, ao + np.einsum("nij,nj->ni", Bo, ai)


def _outputs(offsets, x, P, el, Ps, delta, dtype):
    o = np.asarray(offsets, dtype=np.int64)
    x, P = np.asarray(x).astype(dtype), np.asarray(P).astype(dtype)
    E, flag = el[0], el[4]
    R = len(o) - 1
    run = np.repeat(np.arange(R), o[1:] - o[:-1])
    xs, Pso = x.copy(), P.copy()
    s = np.nonzero(~flag)[0]
    Xs = np.zeros((len(x) - R, 15, 15), dtype=dtype)
    if len(s):
        xs[s] = rr.retract(x[s], delta[s])
        Pso[s] = Ps[s]
        Xs[s - run[s]] = E[s] @ Ps[s + 1]
    return xs, Pso, Xs


def sequential(offsets, x, P, xb, Pb, C, dtype=np.float64, inject=None, mirror=True):
    """(xs [N,16], Ps [N,15,15], Xs [N - n_runs,15,15]) by the backward recursion Ps_k = L_k + G_k Ps_{k+1} G_k^T (mirrored),
    delta_k = a_k + B_k delta_{k+1}, vectorised over runs."""
    o = np.asarray(offsets, dtype=np.int64)
    lens = o[1:] - o[:-1]
    el = elements(o, x, P, xb, Pb, C, dtype, inject, mirror)
    E, L, B, a, _ = el
    Ps, delta = L.copy(), a.copy()
    for j in range(1, int(lens.max()) if len(lens) else 0):
        r = np.nonzero(lens > j)[0]
        s = o[r + 1] - 1 - j
        _, Ps[s], _, delta[s] = compose((E[s], L[s], B[s], a[s]), (E[s + 1], Ps[s + 1], B[s + 1], delta[s + 1]), mirror)
    return _outputs(o, x, P, el, Ps, delta, dtype)


def tree(offsets, x, P, xb, Pb, C, dtype=np.float64, inject=None, mirror=True, flag_by_product=False):
    """The same outputs by a Kogge-Stone scan over the reflected flat index: at distance d, element p (outer) composes with p - d
    unless a run ends within p's span (selection).  flag_by_product=True instead multiplies the inner element by (1 - flag), which
    lets a NaN run leak into its neighbours (sensitivity checks only)."""
    o = np.asarray(offsets, dtype=np.int64)
    el = elements(o, x, P, xb, Pb, C, dtype, inject, mirror)
    cur = [v[::-1].copy() for v in el[:4]]                  # slot p = keyframe N - 1 - p
    f = el[4][::-1].copy()
    n, d = len(f), 1
    while d < n:
        p = np.arange(d, n)
        outer = tuple(v[p] for v in cur)
        inner = tuple(v[p - d] for v in cur)
        if flag_by_product:
            keep = (~f[p]).astype(dtype)
            inner = tuple(v * keep.reshape((-1,) + (1,) * (v.ndim - 1)) for v in inner)
            new = compose(outer, inner, mirror)
        else:
            new = compose(outer, inner, mirror)
            new = tuple(np.where(f[p].reshape((-1,) + (1,) * (nv.ndim - 1)), ov, nv) for nv, ov in zip(new, outer))
        for v, nv in zip(cur, new):
            v[p] = nv
        f[p] = f[p] | f[p - d]
        d *= 2
    return _outputs(o, x, P, el, cur[1][::-1], cur[3][::-1], dtype)
