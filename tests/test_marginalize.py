"""Fixed-lag smoothing of many IMU chains on the device (cpi_imu_chain_marginalize / cpi_imu_prior_at / cpi_imu_chains_assemble,
factor.chain_marginalize / prior_at / chains_assemble / chains_lm_step).

GTSAM is not in the reference tree, so parity with its BatchFixedLagSmoother is UNPINNED.  The truths are the numpy statements
below: ``marginalize_ref`` (the elimination recurrence) and ``local`` (the inverse of JPLNavState::retract).  On the CPU they are
pinned against dense linear algebra and the oracle's retract; the GPU tests compare the kernels with them and check two exact
identities against merged code: the reduced solve equals the full solve, and the marginal information of a chain at its exact
prediction is the inverse of the covariance cpi_propagate_batch carries."""
import ctypes

import numpy as np
import pytest
import scipy.linalg

from cpi_b200 import capi, synth

P = lambda a: ctypes.c_void_p(a.ctypes.data)


def mat(a):
    """[n, 225] column-major -> [n, 15, 15]"""
    return np.asarray(a).reshape(-1, 15, 15).transpose(0, 2, 1)


def vec(A):
    """[n, 15, 15] -> [n, 225] column-major"""
    return np.ascontiguousarray(np.asarray(A).transpose(0, 2, 1).reshape(-1, 225))


def marginalize_ref(G11, G12, G22, g1, g2, f, m, prior=None, jacobi=False):
    """numpy statement of the elimination of the first m states of ONE chain (its factor blocks as [k,15,15] / [k,15] / [k]):
        M = Lam + G11_k = L L^T,  Z = L^-1 G12_k,  z = L^-1 (eta + g1_k);  Lam <- G22_k - Z^T Z,  eta <- g2_k - Z^T z,  f <- f + f_k - z^T z
    jacobi: factor the Jacobi-scaled M (D M D, D = diag(M)^-1/2) -- the same algebra, better conditioned in fp64.
    Returns (Lam [15,15], eta [15], f)."""
    Lam, eta, F = (np.zeros((15, 15)), np.zeros(15), 0.0) if prior is None else (np.array(prior[0], dtype=float), np.array(prior[1], dtype=float), float(prior[2]))
    for k in range(m):
        M, r = Lam + G11[k], eta + g1[k]
        d = 1.0 / np.sqrt(np.diag(M)) if jacobi else np.ones(15)
        L = np.linalg.cholesky(M * d[:, None] * d[None, :])
        Z = scipy.linalg.solve_triangular(L, d[:, None] * G12[k], lower=True)
        z = scipy.linalg.solve_triangular(L, d * r, lower=True)
        Lam, eta, F = G22[k] - Z.T @ Z, g2[k] - Z.T @ z, F + f[k] - z @ z
    return Lam, eta, F


def qmul(q, p):
    """cpi_common.cuh quat_multiply (JPL), batched [n, 4]."""
    t = np.stack([q[:, 3] * p[:, 0] + q[:, 2] * p[:, 1] - q[:, 1] * p[:, 2] + q[:, 0] * p[:, 3],
                  -q[:, 2] * p[:, 0] + q[:, 3] * p[:, 1] + q[:, 0] * p[:, 2] + q[:, 1] * p[:, 3],
                  q[:, 1] * p[:, 0] - q[:, 0] * p[:, 1] + q[:, 3] * p[:, 2] + q[:, 2] * p[:, 3],
                  -q[:, 0] * p[:, 0] - q[:, 1] * p[:, 1] - q[:, 2] * p[:, 2] + q[:, 3] * p[:, 3]], axis=1)
    t[t[:, 3] < 0] *= -1
    return t / np.linalg.norm(t, axis=1, keepdims=True)


def local(base, x):
    """numpy statement of local(x_lin, x), the inverse of JPLNavState::retract, batched [n, 16] -> [n, 15]: the rotation vector of
    q_x (x) q_lin^-1 (w >= 0), differences for the other 12 entries."""
    dq = qmul(x[:, 0:4], base[:, 0:4] * np.array([-1, -1, -1, 1.0]))
    s = np.linalg.norm(dq[:, 0:3], axis=1)
    k = np.where(s > 0, 2 * np.arctan2(s, dq[:, 3]) / np.maximum(s, 1e-300), 2.0)
    k[np.all(x[:, 0:4] == base[:, 0:4], axis=1)] = 0.0
    return np.concatenate([k[:, None] * dq[:, 0:3], x[:, 4:16] - base[:, 4:16]], axis=1)


def prior_at_ref(info, rhs, f, lin, x):
    d = local(lin, x)
    u = np.einsum("nrc,nc->nr", mat(info), d)
    return rhs - u, f - 2 * np.einsum("nr,nr->n", rhs, d) + np.einsum("nr,nr->n", d, u)


def random_factors(rng, k, scale=(1, 1, 1, 1, 1)):
    """k random linearised factors between consecutive 15-dof states (a perturbed random walk x_{k+1} ~ x_k), from random Jacobians
    and residuals with a random SPD noise covariance of standard deviations ~ scale per 3-block: (G11, G12, G22 [k,15,15], g1, g2 [k,15], f [k])."""
    Ds = np.repeat(np.asarray(scale), 3)
    H1 = np.eye(15) + 0.1 * rng.normal(size=(k, 15, 15))
    H2 = -np.eye(15) + 0.1 * rng.normal(size=(k, 15, 15))
    C = rng.normal(size=(k, 15, 15))
    Pm = (C @ C.transpose(0, 2, 1) / 15 + 0.5 * np.eye(15)) * Ds[None, :, None] * Ds[None, None, :]
    W = np.linalg.inv(Pm)
    W = 0.5 * (W + W.transpose(0, 2, 1))
    e = rng.normal(size=(k, 15)) * Ds
    H1t, H2t = H1.transpose(0, 2, 1), H2.transpose(0, 2, 1)
    return (H1t @ W @ H1, H1t @ W @ H2, H2t @ W @ H2, -np.einsum("kij,kj->ki", H1t @ W, e), -np.einsum("kij,kj->ki", H2t @ W, e),
            np.einsum("ki,kij,kj->k", e, W, e))


def random_prior(rng, scale=(1e-2, 1e-3, 1e-1, 1e-2, 1e-1)):
    Ds = np.repeat(np.asarray(scale), 3)
    C = rng.normal(size=(15, 15))
    S = (C @ C.T / 15 + 0.5 * np.eye(15)) * Ds[:, None] * Ds[None, :]
    info = np.linalg.inv(S)
    return 0.5 * (info + info.T), rng.normal(size=15) / Ds, float(rng.uniform(1, 10))


def dense_head(G11, G12, G22, g1, g2, f, n, prior):
    """Dense normal equations (A, b, F) of the chain x_0 .. x_n of the first n factors with the prior on x_0: cost = F - 2 b^T d + d^T A d."""
    A = np.zeros((15 * (n + 1), 15 * (n + 1))); b = np.zeros(15 * (n + 1)); F = prior[2] + np.sum(f[:n])
    A[:15, :15] += prior[0]; b[:15] += prior[1]
    for k in range(n):
        i, j = slice(15 * k, 15 * k + 15), slice(15 * k + 15, 15 * k + 30)
        A[i, i] += G11[k]; A[i, j] += G12[k]; A[j, i] += G12[k].T; A[j, j] += G22[k]
        b[i] += g1[k]; b[j] += g2[k]
    return A, b, F


# ------------------------------------------------------------------------------------------------------------------
# CPU: the numpy statements against dense linear algebra and the oracle, argument checks of the C ABI
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", [0, 1, 2])
def test_recurrence_is_the_schur_complement(seed):
    """On random SPD block-tridiagonal systems: the reduced system with the marginal prior has the full system's solution for the
    states it keeps, inv(Lam_m) is block (m, m) of the inverse of the head system (x_0 .. x_m), and f is the head's minimum cost with x_m = 0."""
    rng = np.random.default_rng(seed)
    n = 12
    G11, G12, G22, g1, g2, f = random_factors(rng, n)
    prior = random_prior(rng, scale=(1, 1, 1, 1, 1))
    A, b, F = dense_head(G11, G12, G22, g1, g2, f, n, prior)
    x = np.linalg.solve(A, b)
    for m in (1, 2, 5, n - 1, n):
        Lam, eta, fm = marginalize_ref(G11, G12, G22, g1, g2, f, m, prior)
        # reduced system: the marginal prior on x_m plus the factors m .. n-1
        Ar, br, _ = dense_head(G11[m:], G12[m:], G22[m:], g1[m:], g2[m:], f[m:], n - m, (Lam, eta, 0.0))
        xr = np.linalg.solve(Ar, br)
        assert np.linalg.norm(xr - x[15 * m:]) <= 1e-9 * np.linalg.norm(x[15 * m:]), m
        # marginal covariance of x_m in the head system
        Ah, bh, Fh = dense_head(G11, G12, G22, g1, g2, f, m, prior)
        Sm = np.linalg.inv(Ah)[15 * m:, 15 * m:]
        Sl = np.linalg.inv(Lam)
        assert np.linalg.norm(Sl - Sm) <= 1e-9 * np.linalg.norm(Sm), m
        # f: min over x_0 .. x_{m-1} of F - 2 b^T d + d^T A d with x_m = 0
        Ae, be = Ah[:15 * m, :15 * m], bh[:15 * m]
        fmin = Fh - be @ np.linalg.solve(Ae, be)
        assert abs(fm - fmin) <= 1e-9 * max(abs(Fh), abs(fmin)), m
        # and the Jacobi-scaled route is the same algebra
        Lj, ej, fj = marginalize_ref(G11, G12, G22, g1, g2, f, m, prior, jacobi=True)
        assert np.linalg.norm(Lj - Lam) <= 1e-9 * np.linalg.norm(Lam) and abs(fj - fm) <= 1e-9 * abs(Fh)
    # m = 0 is the prior itself
    L0, e0, f0 = marginalize_ref(G11, G12, G22, g1, g2, f, 0, prior)
    assert np.array_equal(L0, prior[0]) and np.array_equal(e0, prior[1]) and f0 == prior[2]


def test_local_inverts_retract(oracle):
    """local(x, retract(x, d)) = d and retract(x_lin, local(x_lin, x)) = x through the oracle's JPLNavState::retract."""
    rng = np.random.default_rng(5)
    n = 500
    X = np.zeros((n, 16))
    q = rng.normal(size=(n, 4)); q[:, 3] = np.abs(q[:, 3]); X[:, 0:4] = q / np.linalg.norm(q, axis=1, keepdims=True)
    X[:, 4:16] = rng.normal(size=(n, 12))
    d = rng.normal(size=(n, 15)) * np.r_[np.full(3, 0.5), np.ones(12)]
    d[:10, 0:3] *= 1e-9                                      # tiny rotations
    d[10:20, 0:3] = 0.0
    Y = oracle.retract(X, d)
    assert np.max(np.abs(local(X, Y) - d)) <= 1e-12
    Z = oracle.retract(X, local(X, Y))
    assert np.max(np.abs(Z[:, 0:4] - Y[:, 0:4])) <= 1e-14 and np.max(np.abs(Z[:, 4:] - Y[:, 4:])) <= 1e-12
    assert np.all(local(X, X) == 0.0)


def test_argument_validation_without_gpu():
    lib = capi.load()
    buf = np.zeros(4 * 225)
    p = P(buf)
    offs = np.array([0, 2, 5], dtype=np.int64)
    # cpi_imu_chain_marginalize(n_chains, offs, uniform, n_marg, n_marg_uniform, G11, G12, G22, g1, g2, f, pi, pr, pf, oi, orr, of, stream)
    marg = lambda *a: lib.cpi_imu_chain_marginalize(*a, None)
    good = [p] * 6 + [p, p, p] + [p, p, p]
    assert marg(-1, None, 3, None, 1, *good) == -1 and b"negative" in lib.cpi_last_error()
    assert marg(2, None, 0, None, 0, *good) == -1 and b"chain_uniform" in lib.cpi_last_error()
    assert marg(2, None, 3, None, -1, *good) == -1 and b"negative" in lib.cpi_last_error()
    for m in (3, 4):                                           # n_marg >= S_c
        assert marg(2, None, 3, None, m, *good) == -1 and b"n_marg_uniform" in lib.cpi_last_error()
    for k in range(6):                                         # a factor block missing, f included
        bad = list(good); bad[k] = None
        assert marg(2, None, 3, None, 1, *bad) == -1 and b"null" in lib.cpi_last_error(), k
    bad = list(good); bad[5] = None; bad[11] = None             # f is required even when out_f is NULL: the kernel reads it
    assert marg(2, None, 3, None, 1, *bad) == -1 and b"null" in lib.cpi_last_error()
    for k in (9, 10):                                          # out_info / out_rhs
        bad = list(good); bad[k] = None
        assert marg(2, None, 3, None, 1, *bad) == -1 and b"null" in lib.cpi_last_error(), k
    bad = list(good); bad[7] = None                            # prior_info without prior_rhs
    assert marg(2, None, 3, None, 1, *bad) == -1 and b"both" in lib.cpi_last_error()
    assert marg(0, None, 1, None, 0, *[None] * 12) == 0
    # cpi_imu_prior_at(n, info, rhs, f, lin, x, rhs_out, f_out, stream)
    assert lib.cpi_imu_prior_at(-1, p, p, p, p, p, p, p, None) == -1 and b"negative" in lib.cpi_last_error()
    for k in (0, 1, 3, 4, 5):
        a = [p] * 7; a[k] = None
        assert lib.cpi_imu_prior_at(2, *a, None) == -1 and b"null" in lib.cpi_last_error(), k
    assert lib.cpi_imu_prior_at(0, *[None] * 7, None) == 0
    # cpi_imu_chains_assemble(n_chains, offs, uniform, G11, G12, G22, g1, g2, lambda, damping, pi, pr, D, E, rhs, stream)
    asm = lambda n, o, u, *a, lam=0.0: lib.cpi_imu_chains_assemble(n, o, u, *a[:5], lam, 0, *a[5:], None)
    ga = [p] * 5 + [None, None] + [p, p, p]
    assert asm(-1, None, 2, *ga) == -1 and b"negative" in lib.cpi_last_error()
    assert asm(3, None, 0, *ga) == -1 and b"chain_uniform" in lib.cpi_last_error()
    assert asm(2, P(offs), 0, *ga, lam=-1.0) == -1 and b"lambda" in lib.cpi_last_error()
    for k in (0, 1, 2, 3, 4, 7, 8, 9):                         # G11 .. g2, D, E, rhs
        bad = list(ga); bad[k] = None
        assert asm(2, None, 3, *bad) == -1 and b"null" in lib.cpi_last_error(), k
    assert asm(0, None, 1, *[None] * 10) == 0
    # Python layer
    from cpi_b200 import factor
    with pytest.raises(ValueError):
        factor._chain_layout(0, None, n_states=4)
    with pytest.raises(ValueError):
        factor._chain_layout(3, None, n_states=4)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------

def _chain_blocks(torch, model, nf, first_window, perturb=True):
    """Records, lin, states (x_0 .. x_nf of one long chain) and the device information blocks of its nf factors."""
    from cpi_b200 import factor, preint
    S, L = synth.make_windows(nf, 20, rate=200.0, first_window=first_window, special=False)
    rec = preint.preintegrate_host(model, S, L, synth.SIGMAS, 0, ns=20)
    X = synth.make_states(rec, L, model, perturb=perturb)
    dX, dR, dL = (torch.from_numpy(a).cuda() for a in (X, rec, L))
    e, H1, H2 = factor.factor_eval(model, dX, dR, dL)
    return rec, L, X, factor.factor_hessian(model, dR, e, H1, H2)


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(np.asarray(b)), 1e-300))


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_marginalize_kernel_matches_numpy(cuda, model):
    """K8 on ragged chains of 1..70 states with n_marg from 0 to S-1, with and without a prior, against the numpy statement.  The gate is
    calibrated on the Jacobi-scaled numpy route: the device's worst distance to it within 50x the worst distance of the plain
    (unscaled) fp64 numpy route on the same batch (floor 1e-13)."""
    from cpi_b200 import factor
    torch = cuda
    rng = np.random.default_rng(10 + model)
    sizes = np.r_[1, 2, 70, rng.integers(1, 71, size=45)]
    C = len(sizes)
    offs = np.r_[0, np.cumsum(sizes)].astype(np.int64)
    nf = int(offs[-1] - C)
    _, _, _, blocks = _chain_blocks(torch, model, nf, 7000 + 1000 * model)
    G11, G12, G22, g1, g2, f = blocks
    Gh = [t.cpu().numpy() for t in blocks]
    M11, M12, M22 = mat(Gh[0]), mat(Gh[1]), mat(Gh[2])
    nm = np.array([rng.integers(0, s) for s in sizes], dtype=np.int64)
    nm[0] = 0; nm[2] = 69; nm[3] = 0
    pri = [random_prior(rng, scale=(1e-3, 1e-4, 1e-2, 1e-3, 1e-2)) for _ in range(C)]
    pinfo = np.stack([vec(p[0][None])[0] for p in pri]); prhs = np.stack([p[1] for p in pri]); pf = np.array([p[2] for p in pri])
    d_offs, d_nm = torch.from_numpy(offs).cuda(), torch.from_numpy(nm).cuda()
    dprior = tuple(torch.from_numpy(a).cuda() for a in (pinfo, prhs, pf))
    errs = {k: [] for k in ("info", "rhs", "f")}                   # (device, plain fp64 numpy) distances to the Jacobi-scaled route
    for with_prior in (False, True):
        oi, orr, of = factor.chain_marginalize(G11, G12, G22, g1, g2, f, d_offs, d_nm, prior=dprior if with_prior else None)
        torch.cuda.synchronize()
        oi, orr, of = oi.cpu().numpy(), orr.cpu().numpy(), of.cpu().numpy()
        assert np.array_equal(mat(oi), mat(oi).transpose(0, 2, 1))
        for c in range(C):
            m, f0 = int(nm[c]), int(offs[c] - c)
            if m == 0:                                          # a bitwise copy of the prior (zeros without one)
                if with_prior:
                    assert np.array_equal(oi[c], pinfo[c]) and np.array_equal(orr[c], prhs[c]) and of[c] == pf[c]
                else:
                    assert not np.any(oi[c]) and not np.any(orr[c]) and of[c] == 0.0
                continue
            sl = slice(f0, f0 + m)
            pr = (mat(pinfo[c])[0], prhs[c], pf[c]) if with_prior else None
            args = (M11[sl], M12[sl], M22[sl], Gh[3][sl], Gh[4][sl], Gh[5][sl], m, pr)
            plain, truth = marginalize_ref(*args), marginalize_ref(*args, jacobi=True)
            fscale = abs(truth[2]) + np.sum(Gh[5][sl]) + (pf[c] if with_prior else 0.0)
            for i, (key, got) in enumerate((("info", mat(oi[c])[0]), ("rhs", orr[c]), ("f", of[c]))):
                if key == "f":
                    eg, ep = abs(got - truth[2]) / fscale, abs(plain[2] - truth[2]) / fscale
                else:                                           # relative to the terms that cancel (without a prior the result is exactly 0)
                    sc = max(np.linalg.norm(truth[i]), np.linalg.norm((M22 if key == "info" else Gh[4])[f0 + m - 1]))
                    eg, ep = np.linalg.norm(got - truth[i]) / sc, np.linalg.norm(plain[i] - truth[i]) / sc
                errs[key].append((eg, ep, c, m, with_prior))
    for key, v in errs.items():
        eg, ep = max(v), max(x[1] for x in v)
        print(f"model {model} {key}: device worst {eg[0]:.2e} (chain {eg[2]}, m {eg[3]}, prior {eg[4]}), plain fp64 numpy worst {ep:.2e}")
        assert eg[0] <= 50 * max(ep, 1e-13), (key, eg, ep)       # the fp64 elimination class of this batch
    # uniform layout and counts: the same kernel on 3 chains of 5 states, 2 eliminated each
    sub = slice(0, 12)
    oi, orr, of = factor.chain_marginalize(G11[sub], G12[sub], G22[sub], g1[sub], g2[sub], f[sub], 5, 2)
    oi2, orr2, of2 = factor.chain_marginalize(G11[sub], G12[sub], G22[sub], g1[sub], g2[sub], f[sub], torch.tensor([0, 5, 10, 15], device="cuda"),
                                              torch.full((3,), 2, dtype=torch.int64, device="cuda"))
    assert torch.equal(oi, oi2) and torch.equal(orr, orr2) and torch.equal(of, of2)
    # a non-positive pivot: NaN for that chain only
    bad = G11[sub].clone(); bad[4] = -bad[4]
    oi, orr, of = factor.chain_marginalize(bad, G12[sub], G22[sub], g1[sub], g2[sub], f[sub], 5, 2)
    fin = torch.isfinite(oi).all(dim=1).cpu().numpy()
    assert list(fin) == [True, False, True], fin             # factor 4 is the first factor of chain 1


def assemble_ref(G11, G12, G22, g1, g2, offs, lam, diag, pinfo, prhs):
    """numpy statement of cpi_imu_chains_assemble, summed in the kernel's order (column-major [.,225] blocks in and out)."""
    C, N = len(offs) - 1, int(offs[-1])
    D, E, rhs = np.zeros((N, 225)), np.zeros((max(N - 1, 1), 225)), np.zeros((N, 15))
    for c in range(C):
        lo, hi = int(offs[c]), int(offs[c + 1])
        for k in range(lo, hi):
            fr = k - c
            d, v = np.zeros(225), np.zeros(15)
            if k > lo:
                d, v = d + G22[fr - 1], v + g2[fr - 1]
            if k < hi - 1:
                d, v = d + G11[fr], v + g1[fr]
                E[k] = G12[fr]
            if k == lo:
                d, v = d + pinfo[c], v + prhs[c]
            d[::16] = d[::16] + (lam * np.clip(d[::16], 1e-6, 1e32) if diag else lam)
            D[k], rhs[k] = d, v
    return D, E[:N - 1], rhs


def _check_assembly(got, ref, diag):
    """E and rhs bit for bit; D bit for bit except the diagonally damped diagonal (the device may fuse d + lam * clamp(d) into one fma)."""
    D, E, rhs = (t.cpu().numpy() for t in got)
    Dr, Er, rr = ref
    assert np.array_equal(E, Er) and np.array_equal(rhs, rr)
    off = np.ones(225, dtype=bool)
    if diag:
        off[::16] = False
        assert np.allclose(D[:, ~off], Dr[:, ~off], rtol=5e-16, atol=0)
    assert np.array_equal(D[:, off], Dr[:, off])


def _dense_truth(A, b):
    """Solution of the SPD system by a Jacobi-scaled fp64 solve refined with 80-bit residuals (the truth), and the unrefined solve
    (what a sequential fp64 elimination achieves on this system)."""
    s = 1.0 / np.sqrt(np.diag(A))
    As = A * s[:, None] * s[None, :]
    solve = lambda r: np.linalg.solve(As, r * s) * s
    x64 = solve(b)
    x = x64.astype(np.longdouble)
    Al, bl = A.astype(np.longdouble), b.astype(np.longdouble)
    for _ in range(4):
        x = x + solve((bl - Al @ x).astype(np.float64)).astype(np.longdouble)
    return x.astype(np.float64), x64


@pytest.mark.gpu
def test_reduced_solve_equals_full_solve(cuda):
    """A perturbed chain of 40 keyframes with a 1e8 I prior on x_0, undamped: marginalise m -> prior_at -> chains_assemble -> solve gives
    the full chain's step for the states m .. 39 (full: cpi_imu_chain_assemble + solve).  Gate: both within 50x of a sequential fp64
    dense elimination's distance to the refined truth (floor 1e-13)."""
    from cpi_b200 import factor
    torch = cuda
    nf = 39
    _, _, X, (G11, G12, G22, g1, g2, f) = _chain_blocks(torch, 1, nf, 12000)
    prior = (torch.eye(15, dtype=torch.float64, device="cuda") * 1e8).reshape(1, 225)
    zeros15, zero = torch.zeros((1, 15), dtype=torch.float64, device="cuda"), torch.zeros(1, dtype=torch.float64, device="cuda")
    D, E, rhs = factor.chain_assemble(G11, G12, G22, g1, g2, 0.0, prior, None)
    x_full = factor.chain_solve(D, E, rhs).cpu().numpy()
    Dh, Eh, bh = mat(D.cpu().numpy()), mat(E.cpu().numpy()), rhs.cpu().numpy()
    A = np.zeros((15 * (nf + 1),) * 2)
    for k in range(nf + 1):
        A[15 * k:15 * k + 15, 15 * k:15 * k + 15] = Dh[k]
        if k < nf:
            A[15 * k:15 * k + 15, 15 * k + 15:15 * k + 30] = Eh[k]; A[15 * k + 15:15 * k + 30, 15 * k:15 * k + 15] = Eh[k].T
    xt, x64 = _dense_truth(A, bh.reshape(-1))
    xt, x64 = xt.reshape(-1, 15), x64.reshape(-1, 15)
    dX = torch.from_numpy(X).cuda()
    for m in (1, 7, 20, 38):
        info, r, fm = factor.chain_marginalize(G11, G12, G22, g1, g2, f, nf + 1, m, prior=(prior, zeros15, zero))
        r2, f2 = factor.prior_at(info, r, fm, dX[m:m + 1], dX[m:m + 1])       # the same linearisation point: unchanged
        assert torch.equal(r2, r) and torch.equal(f2, fm)
        sl = slice(m, nf)
        Dr, Er, br = factor.chains_assemble(G11[sl], G12[sl], G22[sl], g1[sl], g2[sl], nf + 1 - m, 0.0, info, r2)
        x_red = factor.chain_solve(Dr, Er, br).cpu().numpy()
        nt = np.linalg.norm(xt[m:])
        e64 = np.linalg.norm(x64[m:] - xt[m:]) / nt
        e_red, e_full = np.linalg.norm(x_red - xt[m:]) / nt, np.linalg.norm(x_full[m:] - xt[m:]) / nt
        print(f"m={m}: reduced {e_red:.2e}, full {e_full:.2e}, sequential fp64 {e64:.2e}, |reduced - full| {np.linalg.norm(x_red - x_full[m:]) / nt:.2e}")
        assert e_red <= 50 * max(e64, 1e-13) and e_full <= 50 * max(e64, 1e-13), (m, e_red, e_full, e64)


@pytest.mark.gpu
def test_marginal_information_is_the_propagated_covariance(cuda):
    """A model-1 chain at its exact prediction (zero residual) with the prior Lam_0 = Sigma_0^-1: inv(Lam_m) equals the Sigma_m of m chained
    cpi_propagate_batch calls from Sigma_0 (exact in linear-Gaussian theory, both routes use the same H1 / H2), and eta = 0 to rounding.
    Gate: 20x the distance between the same two routes computed in numpy from the device's blocks (floor 1e-12)."""
    from cpi_b200 import factor, preint
    torch = cuda
    m = 25
    S, L = synth.make_windows(m, 20, rate=200.0, first_window=15000, special=False)
    L[:] = L[0]
    rec = preint.preintegrate_host(1, S, L, synth.SIGMAS, 0, ns=20)
    x0 = synth.make_states(rec, L, 1, perturb=False)[:1]
    x0[:, 4:7], x0[:, 10:13] = L[:1, 0:3], L[:1, 3:6]
    rng = np.random.default_rng(4)
    C0 = rng.normal(size=(15, 15)) * 1e-3
    Sig0 = C0 @ C0.T + 1e-6 * np.eye(15)
    dR, dL = torch.from_numpy(rec).cuda(), torch.from_numpy(L).cuda()
    xs, cs = [torch.from_numpy(x0).cuda()], [torch.from_numpy(vec(Sig0[None])).cuda()]
    for k in range(m):
        x1, c1, _ = factor.propagate(1, xs[-1], cs[-1], dR[k:k + 1], dL[k:k + 1])
        xs.append(x1); cs.append(c1)
    X = torch.cat(xs)
    e, H1, H2 = factor.factor_eval(1, X, dR, dL)
    G11, G12, G22, g1, g2, f = factor.factor_hessian(1, dR, e, H1, H2)
    Lam0 = np.linalg.inv(Sig0); Lam0 = 0.5 * (Lam0 + Lam0.T)
    prior = (torch.from_numpy(vec(Lam0[None])).cuda(), torch.zeros((1, 15), dtype=torch.float64, device="cuda"),
             torch.zeros(1, dtype=torch.float64, device="cuda"))
    info, eta, _ = factor.chain_marginalize(G11, G12, G22, g1, g2, f, m + 1, m, prior=prior)
    torch.cuda.synchronize()
    Sm = mat(cs[-1].cpu().numpy())[0]
    Lm = mat(info.cpu().numpy())[0]
    d = 1.0 / np.sqrt(np.diag(Sm))
    scaled = lambda A: np.max(np.abs(A * d[:, None] * d[None, :]))
    err = scaled(np.linalg.inv(Lm) - Sm)
    # the same two routes in numpy, from the device's H1 / H2 / blocks
    h1, h2 = mat(H1.cpu().numpy()), mat(H2.cpu().numpy())
    Pm = mat(rec[:, 65:290])
    S_np = Sig0.copy()
    for k in range(m):
        B = np.linalg.inv(h2[k]); A = -B @ h1[k]
        S_np = A @ S_np @ A.T + B @ Pm[k] @ B.T
    Gh = [t.cpu().numpy() for t in (G11, G12, G22, g1, g2, f)]
    L_np, _, _ = marginalize_ref(mat(Gh[0]), mat(Gh[1]), mat(Gh[2]), Gh[3], Gh[4], Gh[5], m, (Lam0, np.zeros(15), 0.0), jacobi=True)
    err_np = scaled(np.linalg.inv(L_np) - S_np)
    shift = np.max(np.abs(np.linalg.solve(Lm, eta.cpu().numpy()[0]) * d))    # the mean the prior implies, in standard deviations
    print(f"inv(Lam_m) vs propagated Sigma_m: device {err:.2e}, numpy {err_np:.2e}; |Lam^-1 eta| / sigma {shift:.2e}")
    assert err <= 20 * max(err_np, 1e-12), (err, err_np)
    assert shift <= 1e-6


@pytest.mark.gpu
def test_prior_at_matches_numpy(cuda):
    from cpi_b200 import factor
    torch = cuda
    rng = np.random.default_rng(8)
    n = 300
    X = np.zeros((n, 16))
    q = rng.normal(size=(n, 4)); q[:, 3] = np.abs(q[:, 3]); X[:, 0:4] = q / np.linalg.norm(q, axis=1, keepdims=True)
    X[:, 4:16] = rng.normal(size=(n, 12))
    from oracle.oracle import Oracle
    Y = Oracle().retract(X, rng.normal(size=(n, 15)) * 1e-2)
    pri = [random_prior(rng) for _ in range(n)]
    info = np.stack([vec(p[0][None])[0] for p in pri]); rhs = np.stack([p[1] for p in pri]); f = np.array([p[2] for p in pri])
    d = [torch.from_numpy(a).cuda() for a in (info, rhs, f, X, Y)]
    r2, f2 = factor.prior_at(*d)
    rr, fr = prior_at_ref(info, rhs, f, X, Y)
    r2, f2 = r2.cpu().numpy(), f2.cpu().numpy()
    scale = np.abs(rhs) + np.abs(rr) + np.einsum("nrc,nc->nr", np.abs(mat(info)), np.abs(local(X, Y)))
    assert np.max(np.abs(r2 - rr) / scale) <= 1e-12
    assert np.max(np.abs(f2 - fr) / (np.abs(f) + np.abs(fr) + 2 * np.abs(np.einsum("nr,nr->n", rhs, local(X, Y))) + 1.0)) <= 1e-10
    # at x = x_lin: bitwise unchanged (rhs and f), also in place
    r3, f3 = factor.prior_at(d[0], d[1], d[2], d[3], d[3])
    assert torch.equal(r3, d[1]) and torch.equal(f3, d[2])


@pytest.mark.gpu
def test_chains_assemble_and_one_solve_for_all_chains(cuda):
    """Both assembly entry points against the numpy statement summed in the kernel's order (bit for bit); one chain: bitwise
    cpi_imu_chain_assemble.  Ragged chains (single-state ones included): E exactly 0 at chain boundaries and the one solve matches
    every chain assembled and solved alone.  A chain that is not SPD poisons its neighbours (NaN * 0)."""
    from cpi_b200 import factor
    torch = cuda
    _, _, _, (G11, G12, G22, g1, g2, f) = _chain_blocks(torch, 1, 300, 20000)
    rng = np.random.default_rng(3)
    pinfo = torch.from_numpy(np.stack([vec(random_prior(rng)[0][None])[0] for _ in range(40)])).cuda()
    prhs = torch.from_numpy(rng.normal(size=(40, 15))).cuda()
    Gh = [t.cpu().numpy() for t in (G11, G12, G22, g1, g2)]
    ph, rh = pinfo.cpu().numpy(), prhs.cpu().numpy()
    for lam, diag in ((0.0, False), (1e-3, False), (1e-5, True)):
        a = factor.chain_assemble(G11[:120], G12[:120], G22[:120], g1[:120], g2[:120], lam, pinfo[0], prhs[0], diagonal_damping=diag)
        b = factor.chains_assemble(G11[:120], G12[:120], G22[:120], g1[:120], g2[:120], 121, lam, pinfo[:1], prhs[:1], diagonal_damping=diag)
        assert all(torch.equal(x, y) for x, y in zip(a, b))
        _check_assembly(a, assemble_ref(*(g[:120] for g in Gh), np.array([0, 121]), lam, diag, ph, rh), diag)
    sizes = np.array([1, 5, 1, 1, 17, 64, 2, 33, 1, 9])
    C = len(sizes)
    offs = np.r_[0, np.cumsum(sizes)].astype(np.int64)
    nf = int(offs[-1] - C)
    sl = slice(0, nf)
    D, E, rhs = factor.chains_assemble(G11[sl], G12[sl], G22[sl], g1[sl], g2[sl], torch.from_numpy(offs).cuda(), 1e-5, pinfo[:C], prhs[:C],
                                       diagonal_damping=True)
    _check_assembly((D, E, rhs), assemble_ref(*(g[sl] for g in Gh), offs, 1e-5, True, ph, rh), True)
    x = factor.chain_solve(D, E, rhs)
    Eh = E.cpu().numpy()
    for c in range(C - 1):
        assert not np.any(Eh[offs[c + 1] - 1]), c
    worst = 0.0
    for c in range(C):
        f0, k = int(offs[c] - c), int(sizes[c] - 1)
        s = slice(f0, f0 + k)
        Da, Ea, ra = factor.chain_assemble(G11[s], G12[s], G22[s], g1[s], g2[s], 1e-5, pinfo[c], prhs[c], diagonal_damping=True)
        assert torch.equal(Da, D[offs[c]:offs[c + 1]]) and torch.equal(ra, rhs[offs[c]:offs[c + 1]]) and torch.equal(Ea, E[offs[c]:offs[c + 1] - 1])
        xa = factor.chain_solve(Da, Ea, ra)
        worst = max(worst, _rel(x[offs[c]:offs[c + 1]].cpu().numpy(), xa.cpu().numpy()))
    print("ragged chains: one solve vs each chain alone, worst relative difference", worst)
    assert worst <= 1e-9                                     # the existing solve gate of a Marquardt-damped chain
    # the NaN caveat: chain 4 not SPD -> NaN there and, through 0 * NaN in the reduction, in other chains
    bad = D.clone(); bad[offs[4] + 3] = -bad[offs[4] + 3]
    xb = factor.chain_solve(bad, E, rhs).cpu().numpy()
    nan_chains = [c for c in range(C) if np.isnan(xb[offs[c]:offs[c + 1]]).any()]
    print("non-SPD chain 4 -> NaN in chains", nan_chains)
    assert 4 in nan_chains and len(nan_chains) > 1


def _np_hessian(rec, e, H1, H2):
    """numpy information blocks (Jacobi-scaled inverse of P_meas)."""
    Pm = mat(rec[:, 65:290])
    d = 1.0 / np.sqrt(np.einsum("kii->ki", Pm))
    W = np.linalg.inv(Pm * d[:, :, None] * d[:, None, :]) * d[:, :, None] * d[:, None, :]
    h1, h2 = mat(H1), mat(H2)
    h1t, h2t = h1.transpose(0, 2, 1), h2.transpose(0, 2, 1)
    return (h1t @ W @ h1, h1t @ W @ h2, h2t @ W @ h2, -np.einsum("kij,kj->ki", h1t @ W, e), -np.einsum("kij,kj->ki", h2t @ W, e),
            np.einsum("ki,kij,kj->k", e, W, e))


def _np_smoother_step(orc, Xw, rec, lin, prior, lam):
    """One chains_lm_step of ONE window in numpy (dense solve), then the marginalisation of its oldest state."""
    n = len(Xw)
    e, H1, H2 = orc.factor_eval(1, Xw, rec, lin)
    G11, G12, G22, g1, g2, f = _np_hessian(rec, e, H1, H2)
    info, rhs, f0, x_lin = prior
    rhs_p, _ = prior_at_ref(vec(info[None]), rhs[None], np.array([f0]), x_lin[None], Xw[:1])
    A, b, _ = dense_head(G11, G12, G22, g1, g2, f, n - 1, (info, rhs_p[0], 0.0))
    dg = np.diag(A).copy()
    A[np.diag_indices_from(A)] += lam * np.clip(dg, 1e-6, 1e32)
    s = 1.0 / np.sqrt(np.diag(A))
    dx = (np.linalg.solve(A * s[:, None] * s[None, :], b * s) * s).reshape(n, 15)
    Xw = orc.retract(Xw, dx)
    e, H1, H2 = orc.factor_eval(1, Xw[:2], rec[:1], lin[:1])
    G = _np_hessian(rec[:1], e, H1, H2)
    rhs_p, f_p = prior_at_ref(vec(info[None]), rhs[None], np.array([f0]), x_lin[None], Xw[:1])
    Lam, eta, fm = marginalize_ref(*G, 1, (info, rhs_p[0], f_p[0]), jacobi=True)
    return Xw[1:], (Lam, eta, fm, Xw[1].copy())


@pytest.mark.gpu
def test_fixed_lag_smoother_of_64_sequences(cuda, oracle):
    """A fixed-lag smoother written with the new entry points: 64 independent sequences of 200 keyframes, lag 30; for every new keyframe
    one chains_lm_step over all windows, then the oldest state of every window is marginalised into its prior.  The same loop in numpy
    (dense solves) on 4 of the sequences must agree with the device: the distance of the final windows in retract coordinates within
    2e-11 of the norm of the window's states (measured on an H100: 1.6e-12).  The distances from the simulated truth (an IMU-only chain:
    the biases are weakly observable, so the estimate drifts from it) and from a full-batch solve of the 200 keyframes are reported,
    not gated."""
    from cpi_b200 import factor, preint
    torch = cuda
    ns, K, W, lam = 64, 200, 30, 1e-5
    S, L = synth.make_windows(ns * (K - 1), 20, rate=200.0, first_window=30000, special=False)
    rec = preint.preintegrate_host(1, S, L, synth.SIGMAS, 0, ns=20).reshape(ns, K - 1, -1)
    L = L.reshape(ns, K - 1, 13)
    rng = np.random.default_rng(21)
    truth = np.stack([synth.make_states(rec[s], L[s], 1, perturb=False) for s in range(ns)])          # [ns, K, 16]
    X0 = truth[:, :W].copy()
    X0[:, 1:, 7:10] += rng.normal(0, 1e-3, (ns, W - 1, 3)); X0[:, 1:, 13:16] += rng.normal(0, 1e-3, (ns, W - 1, 3))
    X0[:, 1:, 4:7] += rng.normal(0, 1e-5, (ns, W - 1, 3))
    dR, dL = torch.from_numpy(rec).cuda(), torch.from_numpy(L).cuda()
    info0 = np.eye(15) * 1e8
    prior = (torch.from_numpy(np.tile(vec(info0[None]), (ns, 1))).cuda(), torch.zeros((ns, 15), dtype=torch.float64, device="cuda"),
             torch.zeros(ns, dtype=torch.float64, device="cuda"), torch.from_numpy(X0[:, 0].copy()).cuda())
    Xw = torch.from_numpy(X0).cuda()
    first = torch.arange(ns, device="cuda") * (W + 1)
    for t in range(W, K):
        xn = factor.predict_state(1, Xw[:, -1].contiguous(), dR[:, t - 1].contiguous(), dL[:, t - 1].contiguous())
        Xw = torch.cat([Xw, xn[:, None]], dim=1)
        states = Xw.reshape(-1, 16).contiguous()
        new, dx, cost = factor.chains_lm_step(1, states, dR[:, t - W:t].reshape(-1, rec.shape[-1]).contiguous(),
                                              dL[:, t - W:t].reshape(-1, 13).contiguous(), W + 1, prior=prior, lam=lam)
        Xw = new.view(ns, W + 1, 16)
        # marginalise the oldest state: the first factor of every window, at the new estimate
        e, H1, H2 = factor.factor_eval(1, Xw.reshape(-1, 16), dR[:, t - W].contiguous(), dL[:, t - W].contiguous(), idx_i=first, idx_j=first + 1)
        G = factor.factor_hessian(1, dR[:, t - W].contiguous(), e, H1, H2)
        r_p, f_p = factor.prior_at(prior[0], prior[1], prior[2], prior[3], Xw[:, 0].contiguous())
        mi, mr, mf = factor.chain_marginalize(*G, 2, 1, prior=(prior[0], r_p, f_p), n_chains=ns)
        prior = (mi, mr, mf, Xw[:, 1].contiguous())
        Xw = Xw[:, 1:].contiguous()
    torch.cuda.synchronize()
    Xg = Xw.cpu().numpy()
    assert np.all(np.isfinite(Xg)) and np.all(np.isfinite(cost.cpu().numpy()))
    worst = 0.0
    for s in (0, 17, 40, 63):
        Xs, pr = X0[s].copy(), (info0, np.zeros(15), 0.0, X0[s, 0].copy())
        for t in range(W, K):
            xn = oracle.predict_state(1, Xs[-1:], rec[s, t - 1:t], L[s, t - 1:t])
            Xs = np.concatenate([Xs, xn])
            Xs, pr = _np_smoother_step(oracle, Xs, rec[s, t - W:t], L[s, t - W:t], pr, lam)
        diff = np.linalg.norm(local(Xs, Xg[s]))
        worst = max(worst, diff / np.linalg.norm(Xs[:, 4:16]))
        print(f"sequence {s}: |device - numpy| {diff:.2e} (retract coordinates), |numpy - simulated truth| {np.linalg.norm(local(truth[s, K - W:], Xs)):.2e}")
    # the full-batch solve of the 200 keyframes, for reference
    Xf = torch.from_numpy(np.concatenate([X0, truth[:, W:]], axis=1)).cuda().reshape(-1, 16)
    pf = (torch.from_numpy(np.tile(vec(info0[None]), (ns, 1))).cuda(), torch.zeros((ns, 15), dtype=torch.float64, device="cuda"),
          torch.zeros(ns, dtype=torch.float64, device="cuda"), torch.from_numpy(X0[:, 0].copy()).cuda())
    for _ in range(4):
        Xf, _, cf = factor.chains_lm_step(1, Xf, dR.reshape(-1, rec.shape[-1]), dL.reshape(-1, 13), K, prior=pf, lam=lam)
    Xf = Xf.view(ns, K, 16)[:, K - W:].cpu().numpy()
    full = max(float(np.max(np.abs(local(Xf[s], Xg[s])))) for s in range(ns))
    print(f"fixed-lag vs numpy: worst relative difference {worst:.2e}; final windows vs a 4-step full-batch solve: max |local| {full:.2e}")
    assert worst <= 2e-11
