"""numpy statement of the attitude-dependent measurements (cpi_imu_measurements_linearize, kernel K12, and
cpi_state_update_measurements_batch, kernel K11; DESIGN.md section 3l).  Layouts as include/cpi_b200.h: states [n,16], z and aux
[M,3], sqrt_info [M,9] column-major S with Lambda = S^T S, covariances and informations [n,225] column-major."""
from __future__ import annotations

import numpy as np

from test_marginalize import mat, vec
from update_ref import retract

POSITION, VELOCITY_BODY, DIRECTION = 1, 2, 3


def rot(q):
    """quat_2_Rot of JPL quaternions [n,4] (global to IMU), [n,3,3]."""
    q = np.atleast_2d(q)
    v, w = q[:, 0:3], q[:, 3]
    K = skew(v)
    return (2 * w ** 2 - 1)[:, None, None] * np.eye(3) - 2 * w[:, None, None] * K + 2 * v[:, :, None] * v[:, None, :]


def skew(a):
    a = np.atleast_2d(a)
    K = np.zeros((len(a), 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -a[:, 2], a[:, 1], -a[:, 0]
    K[:, 1, 0], K[:, 2, 0], K[:, 2, 1] = a[:, 2], -a[:, 1], a[:, 0]
    return K


def h_of(kind, x, aux):
    """h(x) [M,3] of measurements of `kind` [M] at the states x [M,16] (NaN for an unknown kind)."""
    C = rot(x[:, 0:4])
    kind = np.broadcast_to(kind, (len(x),))
    out = np.full((len(x), 3), np.nan)
    p = kind == POSITION
    out[p] = x[p, 13:16] + np.einsum("nki,nk->ni", C[p], aux[p])
    v = kind == VELOCITY_BODY
    out[v] = np.einsum("nij,nj->ni", C[v], x[v, 7:10])
    d = kind == DIRECTION
    out[d] = np.einsum("nij,nj->ni", C[d], aux[d])
    return out


def jacobian(kind, x, aux):
    """H = dh/dxi [M,3,15] at xi = 0 of h(retract(x, xi)), the analytic blocks of DESIGN.md section 3l."""
    C = rot(x[:, 0:4])
    kind = np.broadcast_to(kind, (len(x),))
    H = np.full((len(x), 3, 15), np.nan)
    for i in range(len(x)):
        Hi = np.zeros((3, 15))
        if kind[i] == POSITION:
            Hi[:, 0:3] = -C[i].T @ skew(aux[i])[0]
            Hi[:, 12:15] = np.eye(3)
        elif kind[i] == VELOCITY_BODY:
            Hi[:, 0:3] = skew(C[i] @ x[i, 7:10])[0]
            Hi[:, 6:9] = C[i]
        elif kind[i] == DIRECTION:
            Hi[:, 0:3] = skew(C[i] @ aux[i])[0]
        else:
            continue
        H[i] = Hi
    return H


def sqrt_mat(si):
    """S [M,3,3] of column-major sqrt_info [M,9]."""
    return np.asarray(si).reshape(-1, 3, 3).transpose(0, 2, 1)


def meas_ref(kind, x, z, si, aux):
    """(r [M,3], A [M,3,15], b [M,3]) of the measurements at the states x [M,16] (x already gathered by state_idx)."""
    r = h_of(kind, x, aux) - z
    S = sqrt_mat(si)
    return r, S @ jacobian(kind, x, aux), np.einsum("nij,nj->ni", S, r)


def linearize_ref(kind, x, z, si, aux):
    """(info [M,225], rhs' [M,15], f' [M]) of K12 at the gathered states x."""
    _, A, b = meas_ref(kind, x, z, si, aux)
    return vec(A.transpose(0, 2, 1) @ A), -np.einsum("nki,nk->ni", A, b), np.einsum("ni,ni->n", b, b)


def update_meas_ref(x, cov, offsets, kind, z, si, aux):
    """K11 in numpy, per filter in the square-root form of the kernel: filter i takes measurements offsets[i] .. offsets[i+1]-1, all
    linearised at x[i].  Returns (x+ [n,16], cov+ [n,225], xi [n,15], gamma [n])."""
    n = len(x)
    xo, co, xis, g = x.copy(), np.array(cov, dtype=np.float64), np.zeros((n, 15)), np.zeros(n)
    for i in range(n):
        a, e = int(offsets[i]), int(offsets[i + 1])
        if a == e:
            continue
        xi_ = np.repeat(x[i:i + 1], e - a, axis=0)
        _, A, b = meas_ref(kind[a:e], xi_, z[a:e], si[a:e], aux[a:e])
        L = np.linalg.cholesky(mat(cov[i:i + 1])[0])
        B = A @ L
        C = np.linalg.cholesky(np.eye(15) + np.einsum("jki,jkl->il", B, B))
        u = np.einsum("jki,jk->i", B, b)
        w = np.linalg.solve(C.T, np.linalg.solve(C, u))
        xi = -L @ w
        M = np.linalg.solve(C, L.T).T
        co[i] = vec((M @ M.T)[None])[0]
        res = b + A @ xi
        g[i] = np.sum(res ** 2) + w @ w
        xis[i] = xi
        xo[i] = retract(x[i:i + 1], xi[None])[0]
    return xo, co, xis, g


def update_meas_info(x, cov, offsets, kind, z, si, aux):
    """The same update in dense information form: Sigma+ = (Sigma^-1 + sum A^T A)^-1, xi = -Sigma+ sum A^T b, gamma =
    sum |b + A xi|^2 + xi^T Sigma^-1 xi.  Returns as update_meas_ref."""
    n = len(x)
    xo, co, xis, g = x.copy(), np.array(cov, dtype=np.float64), np.zeros((n, 15)), np.zeros(n)
    for i in range(n):
        a, e = int(offsets[i]), int(offsets[i + 1])
        if a == e:
            continue
        _, A, b = meas_ref(kind[a:e], np.repeat(x[i:i + 1], e - a, axis=0), z[a:e], si[a:e], aux[a:e])
        Si = np.linalg.inv(mat(cov[i:i + 1])[0])
        P = np.linalg.inv(Si + np.einsum("jki,jkl->il", A, A))
        P = 0.5 * (P + P.T)
        xi = -P @ np.einsum("jki,jk->i", A, b)
        co[i] = vec(P[None])[0]
        g[i] = np.sum((b + A @ xi) ** 2) + xi @ Si @ xi
        xis[i] = xi
        xo[i] = retract(x[i:i + 1], xi[None])[0]
    return xo, co, xis, g


def random_measurements(rng, x, n_meas, kinds=(POSITION, VELOCITY_BODY, DIRECTION), sigma=0.05, near=True):
    """n_meas measurements on the states x [N,16] (state_idx uniform), kinds cycled, lever arms of about a metre, directions of unit
    length, S = R^-1/2 with a random rotation of diag(1/sigma); z = h(x) plus noise of about one sigma (near) or h(x) exactly."""
    N = len(x)
    idx = rng.integers(0, N, size=n_meas).astype(np.int64)
    kind = np.array([kinds[j % len(kinds)] for j in range(n_meas)], dtype=np.int32)
    aux = rng.normal(size=(n_meas, 3))
    aux[kind == DIRECTION] /= np.linalg.norm(aux[kind == DIRECTION], axis=1, keepdims=True)
    Q, _ = np.linalg.qr(rng.normal(size=(n_meas, 3, 3)))
    S = np.diag([1 / sigma] * 3)[None] @ Q.transpose(0, 2, 1) * rng.uniform(0.5, 2.0, size=(n_meas, 1, 1))
    si = S.transpose(0, 2, 1).reshape(n_meas, 9)
    z = h_of(kind, x[idx], aux)
    if near:
        z = z + rng.normal(size=(n_meas, 3)) * sigma
    return idx, kind, z, si, aux
