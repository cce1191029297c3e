"""numpy statement of the iterated filter update by measurements with robust losses (cpi_state_update_measurements_iterated_batch,
kernel K13, factor.update_measurements_iterated; DESIGN.md section 3m), on the functions of measurement_ref.py.  Layouts as
include/cpi_b200.h: states [n,16], covariances [n,225] column-major, measurements a CSR list per filter."""
from __future__ import annotations

import numpy as np

import measurement_ref as mr
from test_marginalize import local, mat, vec
from update_ref import retract

GAUSSIAN, HUBER, CAUCHY = 0, 1, 2


def weight(code, k, s):
    """The IRLS weight omega(s) of robust_loss (robust_loss.cuh) for whitened squared residuals s [M]."""
    code, k, s = np.broadcast_arrays(np.asarray(code), np.asarray(k, dtype=float), np.asarray(s, dtype=float))
    w = np.ones(s.shape)
    with np.errstate(divide="ignore", invalid="ignore"):
        h = (code == HUBER) & (s > k * k)
        w[h] = k[h] / np.sqrt(s[h])
        c = code == CAUCHY
        w[c] = 1.0 / (1.0 + s[c] / (k[c] * k[c]))
    return w


def _weighted(kind, x, z, si, aux, code, k):
    """(A [m,3,15], b [m,3], omega [m]) of one filter's measurements at its state x [16]."""
    _, A, b = mr.meas_ref(kind, np.repeat(x[None], len(kind), axis=0), z, si, aux)
    return A, b, weight(code, k, np.einsum("ni,ni->n", b, b))


def update_iter_ref(x, cov, offsets, kind, z, si, aux, loss=None, loss_k=None, gate=None, max_iterations=10, tol=1e-9, info=False):
    """K13 per filter in numpy: the square-root steps of the kernel, or (info) the same Gauss-Newton iteration in dense information
    form, delta = -(Sigma^-1 + sum om A^T A)^-1 (Sigma^-1 d + sum om A^T b), Sigma+ = (Sigma^-1 + sum om A^T A)^-1 and
    gamma = sum om |b + A eps_0|^2 + eps_0^T Sigma^-1 eps_0.  Returns (x+ [n,16], cov+ [n,225], gamma [n], status [n], iterations [n],
    x_lin [n,16] the last linearisation point, margin [n]): margin is the smallest |r - 1| over the stopping tests taken, r the step's
    max_k |delta_k| / (tol sqrt(Sigma_kk)), so a filter whose status a rounding could flip has a margin near 0."""
    n = len(x)
    M = len(kind)
    code = np.zeros(M, dtype=np.int32) if loss is None else np.asarray(loss)
    kk = np.zeros(M) if loss_k is None else np.asarray(loss_k, dtype=float)
    xo, co, xl = x.copy(), np.array(cov, dtype=np.float64), x.copy()
    g, st, it, margin = np.zeros(n), np.ones(n, dtype=np.int32), np.zeros(n, dtype=np.int32), np.full(n, np.inf)
    for i in range(n):
        a, e = int(offsets[i]), int(offsets[i + 1])
        if a == e:
            continue
        Sig = mat(cov[i:i + 1])[0]
        L = np.linalg.cholesky(Sig)
        Si = np.linalg.inv(Sig)
        sd = np.sqrt(np.diag(Sig))
        xt = x[i].copy()
        for t in range(max_iterations):
            A, b, om = _weighted(kind[a:e], xt, z[a:e], si[a:e], aux[a:e], code[a:e], kk[a:e])
            d = np.zeros(15) if t == 0 else local(x[i:i + 1], xt[None])[0]
            if info:
                P = np.linalg.inv(Si + np.einsum("j,jki,jkl->il", om, A, A))
                P = 0.5 * (P + P.T)
                delta = -P @ (Si @ d + np.einsum("j,jki,jk->i", om, A, b))
                eps = d + delta
                gw = eps @ Si @ eps
            else:
                sw = np.sqrt(om)[:, None]
                B = sw[:, :, None] * A @ L
                bp = sw * (b - A @ d)
                C = np.linalg.cholesky(np.eye(15) + np.einsum("jki,jkl->il", B, B))
                w = np.linalg.solve(C.T, np.linalg.solve(C, np.einsum("jki,jk->i", B, bp)))
                eps = -L @ w
                delta = eps - d
                Mf = np.linalg.solve(C, L.T).T
                P = Mf @ Mf.T
                gw = w @ w
            if t == 0:
                g[i] = np.sum(om[:, None] * (b + A @ eps) ** 2) + gw
                if gate is not None and g[i] > gate[i]:
                    st[i], it[i] = 0, 1
                    break
            with np.errstate(divide="ignore", invalid="ignore"):
                r = np.max(np.abs(delta) / (tol * sd))
            margin[i] = min(margin[i], abs(r - 1.0))
            xl[i] = xt
            xt = retract(xt[None], delta[None])[0]
            it[i] = t + 1
            if r <= 1.0:
                st[i] = 1
                break
            st[i] = 2
        if st[i] != 0:
            xo[i] = xt
            co[i] = vec(P[None])[0]
    return xo, co, g, st, it, xl, margin


def stationarity(x_hat, cov, x_star, offsets, kind, z, si, aux, loss=None, loss_k=None):
    """Per filter, the gradient g = Sigma^-1 local(x_hat, x*) + sum_j om_j A_j^T b_j of the MAP objective (the prior's Jacobian taken
    as I) at x*, relative to its terms' scale: max |L^T g| over the larger of max |L^T Sigma^-1 local| and max |L^T sum om A^T b|
    (in the prior's standard deviations, Sigma = L L^T)."""
    n = len(x_hat)
    M = len(kind)
    code = np.zeros(M, dtype=np.int32) if loss is None else np.asarray(loss)
    kk = np.zeros(M) if loss_k is None else np.asarray(loss_k, dtype=float)
    out = np.zeros(n)
    for i in range(n):
        a, e = int(offsets[i]), int(offsets[i + 1])
        if a == e:
            continue
        A, b, om = _weighted(kind[a:e], x_star[i], z[a:e], si[a:e], aux[a:e], code[a:e], kk[a:e])
        Sig = mat(cov[i:i + 1])[0]
        L = np.linalg.cholesky(Sig)
        p = L.T @ np.linalg.solve(Sig, local(x_hat[i:i + 1], x_star[i:i + 1])[0])
        m = L.T @ np.einsum("j,jki,jk->i", om, A, b)
        out[i] = np.max(np.abs(p + m)) / max(np.max(np.abs(p)), np.max(np.abs(m)), 1e-300)
    return out


def covariance_at(cov, x_lin, offsets, kind, z, si, aux, loss=None, loss_k=None):
    """The dense (Sigma^-1 + sum_j om_j A_j^T A_j)^-1 [n,225] with A_j and om_j at the linearisation points x_lin."""
    M = len(kind)
    code = np.zeros(M, dtype=np.int32) if loss is None else np.asarray(loss)
    kk = np.zeros(M) if loss_k is None else np.asarray(loss_k, dtype=float)
    out = np.array(cov, dtype=np.float64)
    for i in range(len(x_lin)):
        a, e = int(offsets[i]), int(offsets[i + 1])
        if a == e:
            continue
        A, _, om = _weighted(kind[a:e], x_lin[i], z[a:e], si[a:e], aux[a:e], code[a:e], kk[a:e])
        P = np.linalg.inv(np.linalg.inv(mat(cov[i:i + 1])[0]) + np.einsum("j,jki,jkl->il", om, A, A))
        out[i] = vec((0.5 * (P + P.T))[None])[0]
    return out
