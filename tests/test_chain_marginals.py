"""Marginal covariances of many chains by selected inversion of the block cyclic reduction (cpi_imu_chains_marginals,
factor.chains_covariance / chains_marginals; DESIGN.md section 3j).

GTSAM is not in the reference tree, so parity with its Marginals is UNPINNED.  The truths are ``selinv_ref`` (the level walk in
numpy, pinned on the CPU against the dense inverse) and, on the GPU, the dense per-chain inverse of the assembled system refined with
80-bit residuals, K7's propagated covariance (a chain at its exact prediction), K8's marginal prior, and the Monte-Carlo spread of
the smoother's error against the truth.  These systems are short (at most 33 states) or checked only for finite, positive-definite
blocks; tests/test_marginals_precision.py gates every block of the long chains, the chain stress batch and the tiled production
batch per component against the extended-precision oracle (oracle_chain_marginals)."""
import ctypes

import numpy as np
import pytest
import scipy.linalg

from cpi_b200 import capi, synth
from test_chains_lm import make_problem, zero_step_record
from test_marginalize import assemble_ref, mat, random_factors, random_prior, vec
from test_propagate import random_cov
from test_state_priors import _dev, _fix, _meas_priors, _sp_dev

P = lambda a: ctypes.c_void_p(a.ctypes.data)


def selinv_ref(D, E, cid, far=None):
    """numpy statement of the level walk of cpi_imu_chains_marginals on D [n,15,15], E [n-1,15,15] (block (k, k+1)), cid [n] the
    chain of every state: the isolated forward phase (as k_bcr_eliminate_iso / k_bcr_reduce_iso, couplings between chains never
    read), then top-down Sigma_{i,i-1}, Sigma_{i,i+1}, Sigma_{i,i} of every odd node.  Returns (cov [n,15,15], the neighbour
    blocks Sigma_{k,k+1} [n-1,15,15], exactly 0 across chains).  far(stride, N) (None: N^T) is the block the walk reads as
    Sigma_{i+1,i-1} from N = Sigma_{i-1,i+1}: a hook through which tests/test_marginals_precision.py injects a misread."""
    n = len(D)
    Z = np.zeros((15, 15))
    lv, Dl, El, stride, m = [], [np.asarray(d) for d in D], [np.asarray(e) for e in E], 1, n
    while m > 1:
        same = lambda p, q: cid[p * stride] == cid[q * stride]
        Lc, Za, Zb = [], [], []
        for t in range(m // 2):
            i = 2 * t + 1
            L = np.linalg.cholesky(Dl[i])
            Lc.append(L)
            Za.append(scipy.linalg.solve_triangular(L, El[i - 1].T, lower=True) if same(i - 1, i) else Z)
            Zb.append(scipy.linalg.solve_triangular(L, El[i], lower=True) if i + 1 < m and same(i + 1, i) else Z)
        Dn, En = [], []
        for u in range((m + 1) // 2):
            j = 2 * u
            d = Dl[j].copy()
            if j >= 1 and same(j - 1, j):
                d -= Zb[(j - 2) // 2].T @ Zb[(j - 2) // 2]
            if j + 1 < m and same(j + 1, j):
                d -= Za[j // 2].T @ Za[j // 2]
            Dn.append(d)
            if j + 2 < m:
                En.append(-Za[j // 2].T @ Zb[j // 2] if same(j + 2, j) else Z)
        lv.append((m, stride, Lc, Za, Zb))
        Dl, El, stride, m = Dn, En, 2 * stride, (m + 1) // 2
    cov = np.zeros((n, 15, 15))
    cov[0] = np.linalg.inv(Dl[0])
    nin = None
    for m, stride, Lc, Za, Zb in reversed(lv):
        nout = np.zeros((m - 1, 15, 15))
        for t in range(m // 2):
            i = 2 * t + 1
            hl = cid[(i - 1) * stride] == cid[i * stride]
            hr = i + 1 < m and cid[(i + 1) * stride] == cid[i * stride]
            back = lambda B: scipy.linalg.solve_triangular(Lc[t].T, B, lower=False)
            N_t = (nin[t].T if far is None else far(stride, nin[t])) if hl and hr else None
            XL = -back(Za[t] @ cov[(i - 1) * stride] + (Zb[t] @ N_t if hr else 0)) if hl else Z
            XR = -back((Za[t] @ nin[t] if hl else 0) + Zb[t] @ cov[(i + 1) * stride]) if hr else Z
            cov[i * stride] = back(np.linalg.inv(Lc[t]) - Za[t] @ XL.T - Zb[t] @ XR.T)
            nout[i - 1] = XL.T
            if i + 1 < m:
                nout[i] = XR
        nin = nout
    return cov, (nin if nin is not None else np.zeros((0, 15, 15)))


def dense(D, E, lo, hi):
    """The dense matrix of states lo .. hi-1 of tridiag(E^T, D, E) ([.,15,15] blocks)."""
    n = hi - lo
    A = np.zeros((15 * n, 15 * n))
    for k in range(n):
        A[15 * k:15 * k + 15, 15 * k:15 * k + 15] = D[lo + k]
        if k + 1 < n:
            A[15 * k:15 * k + 15, 15 * k + 15:15 * k + 30] = E[lo + k]
            A[15 * k + 15:15 * k + 30, 15 * k:15 * k + 15] = E[lo + k].T
    return A


def inv_truth(A):
    """(truth, plain): the inverse of the SPD A by a Jacobi-scaled fp64 inverse refined with 80-bit residuals, and the plain
    (unscaled) fp64 inverse."""
    s = 1.0 / np.sqrt(np.diag(A))
    Si = np.linalg.inv(A * s[:, None] * s[None, :])
    X = (Si * s[:, None] * s[None, :]).astype(np.longdouble)
    Al, I = A.astype(np.longdouble), np.eye(len(A), dtype=np.longdouble)
    for _ in range(2):
        R = (I - Al @ X).astype(np.float64)
        X = X + ((Si @ (R * s[:, None])) * s[:, None]).astype(np.longdouble)
    return X.astype(np.float64), np.linalg.inv(A)


def scaled(S, T):
    """max |S - T| of the blocks in the units of T's diagonal: |S - T|_ij / sqrt(T_ii T_jj), blocks of the full inverse T."""
    d = 1.0 / np.sqrt(np.diag(T))
    return d, lambda blk, I, J: float(np.max(np.abs(blk - T[15 * I:15 * I + 15, 15 * J:15 * J + 15]) * d[15 * I:15 * I + 15, None]
                                             * d[None, 15 * J:15 * J + 15]))


def random_system(rng, sizes):
    """D, E ([.,15,15]) of ragged SPD chains (random factors, a random prior on every chain's first state, a unit prior on every state
    so that the dense fp64 inverse stays accurate) and cid."""
    sizes = np.asarray(sizes)
    offs = np.r_[0, np.cumsum(sizes)].astype(np.int64)
    C, nf = len(sizes), int(offs[-1] - len(sizes))
    G = random_factors(rng, max(nf, 1))
    pri = [random_prior(rng, scale=(1, 1, 1, 1, 1)) for _ in range(C)]
    D, E, _ = assemble_ref(*(vec(g[:nf]) for g in G[:3]), G[3][:nf], G[4][:nf], offs, 0.0, False, vec(np.stack([p[0] for p in pri])),
                           np.stack([p[1] for p in pri]))
    return mat(D) + np.eye(15), mat(E), offs, np.repeat(np.arange(C), sizes)


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", [0, 1])
def test_level_walk_is_the_dense_inverse(seed):
    """On random SPD block-tridiagonal systems of ragged chains (1 .. 70 states, single-state chains, lengths 2^k and 2^k +- 1) the level
    walk gives the block-tridiagonal part of every chain's dense inverse to 1e-12 in the units of its diagonal, exact zeros across
    chains, and the same bits with NaN couplings between chains."""
    rng = np.random.default_rng(seed)
    sizes = [1, 2, 3, 4, 5, 7, 8, 9, 1, 1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 70, 1, 13]
    sizes = sizes if seed == 0 else list(rng.permutation(sizes))
    D, E, offs, cid = random_system(rng, sizes)
    cov, nb = selinv_ref(D, E, cid)
    worst = 0.0
    for c in range(len(sizes)):
        lo, hi = int(offs[c]), int(offs[c + 1])
        T = np.linalg.inv(dense(D, E, lo, hi))
        _, err = scaled(None, T)
        for k in range(hi - lo):
            worst = max(worst, err(cov[lo + k], k, k))
            if k + 1 < hi - lo:
                worst = max(worst, err(nb[lo + k], k, k + 1))
        if hi < offs[-1]:
            assert not np.any(nb[hi - 1]), c                       # the pair (last of c, first of c+1)
    print(f"seed {seed}: worst block error {worst:.1e} in units of the diagonal")
    assert worst <= 1e-12
    Ep = E.copy()
    Ep[offs[1:-1] - 1] = np.nan                                    # the couplings between chains: never read
    cov_p, nb_p = selinv_ref(D, Ep, cid)
    assert np.array_equal(cov_p, cov) and np.array_equal(nb_p, nb)


def test_argument_validation_without_gpu():
    import torch
    from cpi_b200 import factor
    lib = capi.load()
    buf = np.zeros(8 * 225)
    p = P(buf)
    # cpi_imu_chains_marginals(n_chains, offs, uniform, n_states, D, E, cov, cross, workspace, stream)
    mg = lambda *a: lib.cpi_imu_chains_marginals(*a, None)
    assert mg(-1, None, 2, 4, p, p, p, p, p) == -1 and b"negative" in lib.cpi_last_error()
    assert mg(2, None, 0, 4, p, p, p, p, p) == -1 and b"chain_uniform" in lib.cpi_last_error()
    assert mg(2, None, 2, 5, p, p, p, p, p) == -1 and b"n_states" in lib.cpi_last_error()
    assert mg(3, P(buf), 0, 2, p, p, p, p, p) == -1 and b"n_states" in lib.cpi_last_error()
    for k in (0, 1, 2, 4):                                         # D, E, cov, workspace (cross may be NULL)
        a = [p] * 5; a[k] = None
        assert mg(2, None, 2, 4, *a) == -1 and b"null" in lib.cpi_last_error(), k
    assert mg(0, None, 1, 0, *[None] * 5) == 0
    ws = lib.cpi_imu_chains_marginals_workspace
    assert ws(2, 1) < 0 and ws(-1, 4) < 0 and ws(2, -1) < 0
    for n in (1, 2, 3, 64, 65, 1000):                              # the solve's workspace + a zero rhs + the neighbour blocks
        assert ws(1, n) >= lib.cpi_imu_chains_solve_workspace(1, n) + 15 * 8 * n, n
    # the wrappers, before the device is touched (CPU tensors: shapes and dtypes are checked first)
    f64 = dict(dtype=torch.float64)
    D, E = torch.zeros((4, 225), **f64), torch.zeros((3, 225), **f64)
    cases = [((D.float(), E, 2), "float64"), ((D[:, :224], E, 2), "225"), ((D, E[:2], 2), "225"), ((D, E, 3), "match"),
             ((D, E, torch.tensor([0, 1, 2, 3, 4, 4])), "more chains"), ((D, E, torch.tensor([0, 2, 4])), "CUDA")]
    for args, msg in cases:
        with pytest.raises(ValueError, match=msg):
            factor.chains_covariance(*args)
    with pytest.raises(ValueError, match="n_chains"):
        factor.chains_covariance(D, E, torch.tensor([0, 2, 4]), n_chains=3)
    short = torch.zeros(int(ws(2, 4)) // 8 - 1, **f64)
    with pytest.raises(ValueError, match="workspace"):
        factor.chains_covariance(D, E, 2, workspace=short)
    with pytest.raises(ValueError, match="workspace"):
        factor.chains_covariance(D, E, 2, workspace=short.float())
    with pytest.raises(ValueError, match="CUDA"):                  # a workspace large enough, but on the host
        factor.chains_covariance(D, E, 2, workspace=torch.zeros(int(ws(2, 4)) // 8, **f64))
    X, rec, lin = torch.zeros((6, 16), **f64), torch.zeros((4, 290), **f64), torch.zeros((4, 13), **f64)
    with pytest.raises(ValueError, match="record"):
        factor.chains_marginals(1, X, rec[:3], lin, 3)
    with pytest.raises(ValueError):
        factor.chains_marginals(1, X, rec, lin, 4)
    with pytest.raises(ValueError, match="state_priors"):
        factor.chains_marginals(1, X, rec, lin, 3, state_priors=(torch.zeros(1, dtype=torch.int64), torch.zeros((1, 224), **f64), None, None,
                                                                  torch.zeros((1, 16), **f64)))
    with pytest.raises(ValueError, match="CUDA"):
        factor.chains_marginals(1, X, rec, lin, 3)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------

def _system(torch, model, X, rec, L, offs, pri, sp=None, loss=None):
    """D, E of the system chains_marginals inverts (its linearisation, lambda = 0), as numpy [.,15,15]."""
    from cpi_b200 import factor
    (C, _, _), _, (G11, G12, G22, g1, g2, _), (pi, pr, _) = factor._linearized(model, X, rec, L, offs, pri, None, sp, loss)
    D, E, _ = factor.chains_assemble(G11, G12, G22, g1, g2, offs, 0.0, pi, pr, n_chains=C)
    return D, E


def _prior(torch, C, X, offs, sigma0=None):
    """A chain prior (info, rhs 0, f 0, lin = the first states) on every chain: diag(1e4, 1e6, 1e2, 1e4, 1e2) per 3-block."""
    info = np.repeat(vec(np.diag(np.repeat([1e4, 1e6, 1e2, 1e4, 1e2], 3))[None]), C, axis=0)
    return (_dev(torch, info), _dev(torch, np.zeros((C, 15))), _dev(torch, np.zeros(C)), _dev(torch, X[offs[:-1]]))


def _gate_chains(D, E, offs, cov, cr, label):
    """Every chain's diagonal and cross blocks against the refined dense inverse: the device's worst distance within 50x the plain
    fp64 dense inverse's worst distance on the same batch (floor 1e-13), in units of the truth's diagonal."""
    D, E, cov = mat(D.cpu().numpy()), mat(E.cpu().numpy()), mat(cov.cpu().numpy())
    cr = None if cr is None else mat(cr.cpu().numpy())
    assert np.array_equal(cov, cov.transpose(0, 2, 1))
    ed = ep = 0.0
    for c in range(len(offs) - 1):
        lo, hi = int(offs[c]), int(offs[c + 1])
        T, P64 = inv_truth(dense(D, E, lo, hi))
        _, err = scaled(None, T)
        for k in range(hi - lo):
            blocks = [(cov[lo + k], k, k)] + ([(cr[lo - c + k], k, k + 1)] if cr is not None and k + 1 < hi - lo else [])
            for blk, I, J in blocks:
                ed = max(ed, err(blk, I, J))
                ep = max(ep, err(P64[15 * I:15 * I + 15, 15 * J:15 * J + 15], I, J))
    print(f"{label}: device worst {ed:.2e}, plain fp64 dense inverse worst {ep:.2e} (units of the diagonal)")
    assert ed <= 50 * max(ep, 1e-13), (ed, ep)


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_against_the_dense_inverse(cuda, oracle, model):
    """Ragged chains (single-state ones, 2^k and 2^k +- 1 states) with a chain prior and state priors: chains_covariance on the system
    chains_marginals assembles is chains_marginals bit for bit and lies within the gate of the refined dense inverse of every chain."""
    from cpi_b200 import factor
    torch = cuda
    sizes = [1, 2, 3, 4, 5, 8, 9, 1, 15, 16, 17, 31, 32, 33]
    X, rec, L, offs, pri, _ = make_problem(oracle, model, sizes, 31 + model, with_prior=True)
    rng = np.random.default_rng(model)
    sp = _sp_dev(torch, *_meas_priors(oracle, rng, X, offs, 4, "mixed"))
    dX, dR, dL, d_offs = (_dev(torch, a) for a in (X, rec, L, offs))
    from test_chains_lm import dev_prior
    pr = dev_prior(torch, pri)
    D, E = _system(torch, model, dX, dR, dL, d_offs, pr, sp)
    cov, cr = factor.chains_covariance(D, E, d_offs, cross=True)
    cov2, cr2 = factor.chains_marginals(model, dX, dR, dL, d_offs, prior=pr, state_priors=sp, cross=True)
    assert torch.equal(cov, cov2) and torch.equal(cr, cr2)
    cov3, none = factor.chains_covariance(D, E, d_offs)
    assert torch.equal(cov3, cov) and none is None
    _gate_chains(D, E, offs, cov, cr, f"model {model}, {len(sizes)} ragged chains")


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_chain_at_its_prediction_is_the_propagated_covariance(cuda, model):
    """A chain at its exact prediction with only the prior Sigma_0^-1 on x_0: later factors carry no information on x_k, so
    Sigma_kk is the Sigma_k of k chained cpi_propagate_batch calls and Sigma_{k,k+1} their cross-covariance.  Gate: 20x the distance
    between the same two routes in numpy (propagation and the dense inverse of the device's blocks), floor 1e-12."""
    from cpi_b200 import factor, preint
    torch = cuda
    m = 25
    S, L = synth.make_windows(m, 20, rate=200.0, first_window=15000, special=False)
    L[:] = L[0]
    rec = preint.preintegrate_host(model, S, L, synth.SIGMAS, 0, ns=20)
    x0 = synth.make_states(rec, L, model, perturb=False)[:1]
    x0[:, 4:7], x0[:, 10:13] = L[:1, 0:3], L[:1, 3:6]
    rng = np.random.default_rng(4)
    C0 = rng.normal(size=(15, 15)) * 1e-3
    Sig0 = C0 @ C0.T + 1e-6 * np.eye(15)
    dR, dL = torch.from_numpy(rec).cuda(), torch.from_numpy(L).cuda()
    xs, cs, crs = [torch.from_numpy(x0).cuda()], [torch.from_numpy(vec(Sig0[None])).cuda()], []
    for k in range(m):
        x1, c1, cr1 = factor.propagate(model, xs[-1], cs[-1], dR[k:k + 1], dL[k:k + 1], want_cross=True)
        xs.append(x1); cs.append(c1); crs.append(cr1)
    X = torch.cat(xs)
    e, H1, H2 = factor.factor_eval(model, X, dR, dL)
    G11, G12, G22, g1, g2, f = factor.factor_hessian(model, dR, e, H1, H2)
    Lam0 = np.linalg.inv(Sig0); Lam0 = 0.5 * (Lam0 + Lam0.T)
    D, E, _ = factor.chains_assemble(G11, G12, G22, g1, g2, m + 1, 0.0, torch.from_numpy(vec(Lam0[None])).cuda(), None)
    cov, cr = factor.chains_covariance(D, E, m + 1, cross=True)
    cov, cr = mat(cov.cpu().numpy()), mat(cr.cpu().numpy())
    Sk, Ck = mat(torch.cat(cs).cpu().numpy()), mat(torch.cat(crs).cpu().numpy())
    # numpy: the propagation from the device's H1 / H2 and the refined dense inverse of the device's blocks
    h1, h2, Pm = mat(H1.cpu().numpy()), mat(H2.cpu().numpy()), mat(rec[:, 65:290])
    S_np, C_np = [Sig0], []
    for k in range(m):
        B = np.linalg.inv(h2[k]); A = -B @ h1[k]
        C_np.append(S_np[-1] @ A.T); S_np.append(A @ S_np[-1] @ A.T + B @ Pm[k] @ B.T)
    T, _ = inv_truth(dense(mat(D.cpu().numpy()), mat(E.cpu().numpy()), 0, m + 1))
    err = err_np = 0.0
    d = [1.0 / np.sqrt(np.diag(s)) for s in Sk]
    sc = lambda A, i, j: float(np.max(np.abs(A) * d[i][:, None] * d[j][None, :]))     # in the propagated standard deviations
    for k in range(m + 1):
        err = max(err, sc(cov[k] - Sk[k], k, k))
        err_np = max(err_np, sc(T[15 * k:15 * k + 15, 15 * k:15 * k + 15] - S_np[k], k, k))
        if k < m:
            err = max(err, sc(cr[k] - Ck[k], k, k + 1))
            err_np = max(err_np, sc(T[15 * k:15 * k + 15, 15 * k + 15:15 * k + 30] - C_np[k], k, k + 1))
    print(f"Sigma_kk, Sigma_k,k+1 against the propagated covariance: device {err:.2e}, numpy routes {err_np:.2e}")
    assert err <= 20 * max(err_np, 1e-12), (err, err_np)


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_marginal_prior_keeps_the_marginals(cuda, oracle, model):
    """One chain of 30 states with a chain prior and state priors on inner states: inv(Lam) of K8 with n_marg = S - 1 is
    Sigma_{S-1,S-1}, and the reduced problem (K8's prior at state m, the remaining factors and priors) has the full chain's Sigma_kk for
    every k >= m.  Gate: 50x the plain fp64 dense inverse's distance to the refined truth (floor 1e-13), units of the diagonal."""
    from cpi_b200 import factor
    from test_chains_lm import dev_prior
    torch = cuda
    S = 30
    X, rec, L, offs, pri, _ = make_problem(oracle, model, [S], 41, with_prior=True)
    idx, info, rhs, f, lin = _meas_priors(oracle, np.random.default_rng(5), X, offs, 3, "mixed")
    keep = idx < S - 1
    idx, info, rhs, f, lin = idx[keep], info[keep], rhs[keep], f[keep], lin[keep]
    dX, dR, dL = (_dev(torch, a) for a in (X, rec, L))
    pr = dev_prior(torch, pri)
    sp = _sp_dev(torch, idx, info, rhs, f, lin)
    D, E = _system(torch, model, dX, dR, dL, S, pr, sp)
    cov = mat(factor.chains_marginals(model, dX, dR, dL, S, prior=pr, state_priors=sp)[0].cpu().numpy())
    T, P64 = inv_truth(dense(mat(D.cpu().numpy()), mat(E.cpu().numpy()), 0, S))
    _, err = scaled(None, T)
    e64 = max(err(P64[15 * k:15 * k + 15, 15 * k:15 * k + 15], k, k) for k in range(S))
    gate = 50 * max(e64, 1e-13)
    # K8 at the blocks' linearisation point X: the chain prior and the state priors moved there
    e, H1, H2 = factor.factor_eval(model, dX, dR, dL)
    G = factor.factor_hessian(model, dR, e, H1, H2)
    pr_r, pr_f = factor.prior_at(pr[0], pr[1], pr[2], pr[3], dX[:1])
    sp_r, sp_f = factor.prior_at(sp[1], sp[2], sp[3], sp[4], dX[sp[0]])
    sp_moved = (sp[0], sp[1], sp_r, sp_f, dX[sp[0]].contiguous())
    worst = 0.0
    for m in (1, 6, 21, S - 1):
        Lam, eta, fm = factor.chain_marginalize(*G, S, m, prior=(pr[0], pr_r, pr_f), state_priors=sp_moved)
        if m == S - 1:
            e_last = err(np.linalg.inv(mat(Lam.cpu().numpy())[0]), S - 1, S - 1)
            print(f"inv(Lam) of K8 against the truth: {e_last:.2e}; device Sigma_{{S-1,S-1}}: {err(cov[S - 1], S - 1, S - 1):.2e}")
            assert e_last <= gate and err(cov[S - 1], S - 1, S - 1) <= gate
        rest = idx >= m
        sp_red = _sp_dev(torch, idx[rest] - m, info[rest], rhs[rest], f[rest], lin[rest])
        cr = factor.chains_marginals(model, dX[m:].contiguous(), dR[m:].contiguous(), dL[m:].contiguous(), S - m, prior=(Lam, eta, fm, None),
                                     state_priors=sp_red if rest.any() else None)[0]
        cr = mat(cr.cpu().numpy())
        worst_m = max(err(cr[k - m], k, k) for k in range(m, S))
        worst = max(worst, worst_m)
        print(f"m = {m}: reduced Sigma_kk against the truth, worst {worst_m:.2e}")
    print(f"plain fp64 dense inverse {e64:.2e}")
    assert worst <= gate, (worst, e64)


@pytest.mark.gpu
def test_priors_and_robust_losses(cuda, oracle):
    """All-Gaussian codes and Huber with k above every residual give the Gaussian result bit for bit; Huber and Cauchy (with outlying
    fixes) match the refined dense inverse of the system reweighted at the states, w = k / sqrt(s) or 1 / (1 + s / k^2)."""
    from cpi_b200 import factor
    from test_chains_lm import dev_prior
    from test_marginalize import local
    torch = cuda
    sizes = [3, 12, 1, 20, 9]
    X, rec, L, offs, pri, _ = make_problem(oracle, 1, sizes, 51, with_prior=True)
    rng = np.random.default_rng(6)
    idx, info, rhs, f, lin = _meas_priors(oracle, rng, X, offs, 2, "p", sigma=0.01)
    lin[::3, 13:16] += 0.2                                         # outliers: 20 standard deviations
    M = len(idx)
    dX, dR, dL, d_offs = (_dev(torch, a) for a in (X, rec, L, offs))
    pr = dev_prior(torch, pri)
    sp = _sp_dev(torch, idx, info, None, None, lin)
    base = factor.chains_marginals(1, dX, dR, dL, d_offs, prior=pr, state_priors=sp, cross=True)
    code = lambda c: torch.full((M,), c, dtype=torch.int32, device="cuda")
    for loss in ((code(capi.LOSS_GAUSSIAN), torch.ones(M, dtype=torch.float64, device="cuda")),
                 (code(capi.LOSS_HUBER), torch.full((M,), 1e6, dtype=torch.float64, device="cuda"))):
        got = factor.chains_marginals(1, dX, dR, dL, d_offs, prior=pr, state_priors=sp, state_prior_loss=loss, cross=True)
        assert torch.equal(got[0], base[0]) and torch.equal(got[1], base[1])
    s = np.einsum("ni,nij,nj->n", local(lin, X[idx]), mat(info), local(lin, X[idx]))
    Dp, Ep = _system(torch, 1, dX, dR, dL, d_offs, pr)             # without the state priors
    Dp, Ep = mat(Dp.cpu().numpy()), mat(Ep.cpu().numpy())
    for c, k in ((capi.LOSS_HUBER, 1.0), (capi.LOSS_CAUCHY, 2.0)):
        w = np.where(s <= k * k, 1.0, k / np.sqrt(s)) if c == capi.LOSS_HUBER else 1.0 / (1.0 + s / (k * k))
        assert w.min() < 0.1
        Dw = Dp.copy()
        for i in range(M):
            Dw[idx[i]] += w[i] * mat(info[i])[0]
        cov, cr = factor.chains_marginals(1, dX, dR, dL, d_offs, prior=pr, state_priors=sp, cross=True,
                                          state_prior_loss=(code(c), torch.full((M,), k, dtype=torch.float64, device="cuda")))
        _gate_chains(torch.from_numpy(vec(Dw)), torch.from_numpy(vec(Ep)), offs, cov, cr, f"loss {c}, k {k}")


@pytest.mark.gpu
def test_isolation_and_determinism(cuda, oracle):
    """Ten chains: a zero-step record or a NaN prior in one chain makes that chain's blocks NaN and leaves the other nine bitwise the
    clean run; two calls are bitwise identical; uniform and device-resident layouts give the same bits."""
    from cpi_b200 import factor
    from test_chains_lm import dev_prior
    torch = cuda
    sizes = [5, 9, 12, 7, 16, 3, 8, 11, 6, 10]
    X, rec, L, offs, pri, _ = make_problem(oracle, 1, sizes, 61, with_prior=True)
    idx, info, rhs, f, lin = _meas_priors(oracle, np.random.default_rng(7), X, offs, 3, "p")
    dX, dR, dL, d_offs = (_dev(torch, a) for a in (X, rec, L, offs))
    pr = dev_prior(torch, pri)
    sp = _sp_dev(torch, idx, info, None, None, lin)
    run = lambda R=dR, S=sp: [t.cpu().numpy() for t in factor.chains_marginals(1, dX, R, dL, d_offs, prior=pr, state_priors=S, cross=True)]
    cov0, cr0 = run()
    cov1, cr1 = run()
    assert np.array_equal(cov0, cov1) and np.array_equal(cr0, cr1)
    assert np.all(np.isfinite(cov0)) and np.all(np.isfinite(cr0))
    bad_rec = rec.copy(); bad_rec[int(offs[3] - 3) + 2] = zero_step_record(1)
    info_nan = info.copy(); j = int(np.nonzero(idx >= offs[6])[0][0]); info_nan[j, 0] = np.nan
    for bad, run_bad in ((3, lambda: run(R=_dev(torch, bad_rec))), (6, lambda: run(S=_sp_dev(torch, idx, info_nan, None, None, lin)))):
        cov, cr = run_bad()
        for c in range(len(sizes)):
            s, t = slice(offs[c], offs[c + 1]), slice(offs[c] - c, offs[c + 1] - c - 1)
            if c == bad:
                assert np.isnan(cov[s]).any(axis=1).all() and np.isnan(cr[t]).any(axis=1).all(), c
            else:
                assert np.array_equal(cov[s], cov0[s]) and np.array_equal(cr[t], cr0[t]), (bad, c)
    # uniform layout against the device-resident one
    Xu, ru, Lu, ou, pu, _ = make_problem(oracle, 1, [8] * 6, 62, with_prior=True)
    a = factor.chains_marginals(1, _dev(torch, Xu), _dev(torch, ru), _dev(torch, Lu), 8, prior=dev_prior(torch, pu), cross=True)
    b = factor.chains_marginals(1, _dev(torch, Xu), _dev(torch, ru), _dev(torch, Lu), _dev(torch, ou), prior=dev_prior(torch, pu), cross=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def _smoother_monte_carlo(torch, oracle, model, N, K, seed, noise=None, fixes=(3, 6, 9), sigma_fix=0.01):
    """N realisations of one truth trajectory as chains of K keyframes (20-sample windows at 200 Hz): every realisation has its own IMU
    noise (the reference simulator's white noise and bias walk, as test_propagate._monte_carlo), x_hat_0 drawn from the prior Sigma_0
    and a position fix of sigma_fix drawn from its own sigma on the keyframes `fixes`.  chains_lm to convergence, then chains_marginals
    at the result.  seed draws the configuration (the truth's initial attitude and Sigma_0) and, with noise None, the realisations;
    noise = s draws the realisations from an independent stream [seed, s] instead, for the same configuration.  Returns (errors
    [N, K, 15] of the truth in retract coordinates at the estimate, Sigma_kk [N, K, 15, 15], status)."""
    from cpi_b200 import factor, preint
    rng = np.random.default_rng(seed)
    nz = None if noise is None else np.random.default_rng([seed, noise])

    def draw(size, scale=1.0):
        """A draw of the realisations: the configuration stream makes it in any case, so its later draws stay the seed's."""
        x = rng.normal(0.0, scale, size)
        return x if nz is None else nz.normal(0.0, scale, size)
    ns = 20
    Sw, Lw = synth.make_windows(K - 1, ns, rate=200.0, first_window=81000 + 100 * model, special=False)
    Lw[:] = Lw[0]
    dt = Sw[:, :, 6]                                               # [K-1, ns]
    w_true, a_true = Sw[:, :, 0:3] - Lw[0, 0:3], Sw[:, :, 3:6] - Lw[0, 3:6]
    # the truth's attitude, velocity and position: the noise-free propagation of the bias-free readings
    x_true = np.zeros((K, 16))
    q = rng.normal(size=4); q /= np.linalg.norm(q); q *= np.sign(q[3])
    x_true[0, 0:4], x_true[0, 4:7], x_true[0, 7:10], x_true[0, 10:13], x_true[0, 13:16] = q, Lw[0, 0:3], [1.0, -0.5, 0.2], Lw[0, 3:6], [3.0, 1.0, -2.0]
    for k in range(K - 1):
        lin_t = np.concatenate([x_true[k, 4:7], x_true[k, 10:13], x_true[k, 0:4], synth.GRAVITY])[None]
        clean = np.concatenate([w_true[k] + x_true[k, 4:7], a_true[k] + x_true[k, 10:13], dt[k][:, None]], axis=1)[None]
        x_true[k + 1] = oracle.predict_state(model, x_true[k:k + 1], preint.preintegrate_host(model, clean, lin_t, synth.SIGMAS, 0, ns=ns), lin_t)[0]
    # every realisation: its bias walk (the truth's biases at the keyframes), readings, x_hat_0 and fixes
    sw, swb, sa, sab = synth.SIGMAS
    T = (K - 1) * ns
    sq = np.sqrt(dt.reshape(-1))[None, :, None]
    bw = x_true[0, 4:7] + np.concatenate([np.zeros((N, 1, 3)), np.cumsum(swb * sq * draw((N, T, 3)), axis=1)], axis=1)
    ba = x_true[0, 10:13] + np.concatenate([np.zeros((N, 1, 3)), np.cumsum(sab * sq * draw((N, T, 3)), axis=1)], axis=1)
    samples = np.empty((N, T, 7))
    samples[:, :, 0:3] = w_true.reshape(-1, 3) + bw[:, :T] + sw / sq * draw((N, T, 3))
    samples[:, :, 3:6] = a_true.reshape(-1, 3) + ba[:, :T] + sa / sq * draw((N, T, 3))
    samples[:, :, 6] = dt.reshape(-1)
    truth = np.repeat(x_true[None], N, axis=0)
    truth[:, :, 4:7], truth[:, :, 10:13] = bw[:, ::ns], ba[:, ::ns]
    Sig0 = mat(random_cov(rng, 1)[0])[0]
    delta = draw((N, 15)) @ np.linalg.cholesky(Sig0).T
    xh0 = oracle.retract(truth[:, 0], -delta)                      # truth_0 = retract(x_hat_0, delta)
    # records at x_hat_0's biases and (model 2) the truth's attitude turned by x_hat_0's attitude error
    att = np.zeros((N, 15)); att[:, 0:3] = -delta[:, 0:3]
    lin = np.empty((N, K - 1, 13))
    lin[:, :, 0:3], lin[:, :, 3:6], lin[:, :, 10:13] = xh0[:, None, 4:7], xh0[:, None, 10:13], synth.GRAVITY
    for k in range(K - 1):
        lin[:, k, 6:10] = oracle.retract(truth[:, k], att)[:, 0:4]
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dl = d(lin.reshape(-1, 13))
    rec = preint.preintegrate(model, d(samples.reshape(N * (K - 1), ns, 7)), dl, synth.SIGMAS, 0, ns=ns)
    # initial states: dead reckoning from x_hat_0
    X0 = torch.empty((N, K, 16), dtype=torch.float64, device="cuda")
    X0[:, 0] = d(xh0)
    recK, linK = rec.view(N, K - 1, -1), dl.view(N, K - 1, 13)
    for k in range(K - 1):
        X0[:, k + 1] = factor.predict_state(model, X0[:, k].contiguous(), recK[:, k].contiguous(), linK[:, k].contiguous())
    X0 = X0.reshape(N * K, 16)
    Lam0 = np.linalg.inv(Sig0); Lam0 = 0.5 * (Lam0 + Lam0.T)
    prior = (d(np.repeat(vec(Lam0[None]), N, axis=0)), d(np.zeros((N, 15))), d(np.zeros(N)), d(xh0))
    idx, W, xb = [], [], []
    for k in fixes:
        w, _ = _fix(rng, truth[0, k], sigma_fix)
        fix = truth[:, k].copy(); fix[:, 13:16] += draw((N, 3), sigma_fix)
        idx.append(np.arange(N) * K + k); W.append(np.repeat(vec(w[None]), N, axis=0)); xb.append(fix)
    sp = (d(np.concatenate(idx).astype(np.int64)), d(np.concatenate(W)), None, None, d(np.concatenate(xb)))
    params = capi.LMParams(absolute_error_tol=0.0, relative_error_tol=1e-13, max_iterations=50)
    Xs, _, _, status, _, _ = factor.chains_lm(model, X0, rec, dl, K, prior=prior, state_priors=sp, params=params, max_rounds=100)
    cov, _ = factor.chains_marginals(model, Xs, rec, dl, K, prior=prior, state_priors=sp)
    from test_marginalize import local
    Xe = Xs.cpu().numpy()
    err = local(Xe, truth.reshape(N * K, 16)).reshape(N, K, 15)
    return err, mat(cov.cpu().numpy()).reshape(N, K, 15, 15), status.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_monte_carlo_consistency_of_the_smoother(cuda, oracle, model):
    """N = 30 000 realisations of one configuration (seed 90 + model) as chains of 10 keyframes: three batches of 10 000, the seed's own
    noise stream and two independent ones, pooled.  A 1 cm position fix on keyframes 3, 6 and 9, chains_lm to convergence
    (relative_error_tol 1e-13, absolute 0, at most 50 steps) and chains_marginals at the result: at every keyframe the mean NEES
    e^T Sigma_kk^-1 e of the retract-coordinate error against the truth lies in the two-sided 99.9 % chi^2_15 band for N, and every
    entry of the error's second moment lies within 5 standard errors of the mean Sigma_kk (as test_monte_carlo_consistency).
    DESIGN.md section 3j has every batch's mean NEES: the seed's own model-1 batch alone lies 1.3 % low, just below its band."""
    from scipy.stats import chi2
    n, K, streams = 10_000, 10, (None, 1, 2)
    nees_sum, m2_sum, cov_sum = np.zeros(K), np.zeros((K, 15, 15)), np.zeros((K, 15, 15))
    for s in streams:
        err, cov, status = _smoother_monte_carlo(cuda, oracle, model, n, K, 90 + model, noise=s)
        assert np.all(status != capi.LM_NONFINITE) and np.all(status != capi.LM_RUNNING)
        for k in range(K):
            e, C = err[:, k], cov[:, k]
            nees = np.einsum("ni,ni->n", e, np.linalg.solve(C, e[:, :, None])[:, :, 0])
            print(f"model {model}, noise stream {s}, keyframe {k}: mean NEES of the batch {nees.mean():.3f}")
            nees_sum[k] += nees.sum(); m2_sum[k] += e.T @ e; cov_sum[k] += C.sum(axis=0)
    N = n * len(streams)
    lo, hi = chi2.ppf([0.0005, 0.9995], 15 * N) / N
    worst_z, outside = 0.0, []
    for k in range(K):
        M, Cm = m2_sum[k] / N, cov_sum[k] / N
        se = np.sqrt((np.outer(np.diag(Cm), np.diag(Cm)) + Cm ** 2) / N)
        z = float(np.max(np.abs((M - Cm) / se)))
        worst_z = max(worst_z, z)
        print(f"model {model}, keyframe {k}: mean NEES {nees_sum[k] / N:.3f} over {N} (band [{lo:.3f}, {hi:.3f}]), worst |z| {z:.1f}")
        if not lo <= nees_sum[k] / N <= hi:
            outside.append((k, float(nees_sum[k] / N)))
    assert not outside, outside
    assert worst_z <= 5.0, worst_z


@pytest.mark.gpu
def test_scale(cuda, oracle):
    """10 000 chains x 30 states and the 5 000-state configs[4] chain with a position fix every 50 keyframes: every block finite, every
    diagonal block positive definite."""
    from cpi_b200 import factor, preint
    torch = cuda
    C, S = 10_000, 30
    Sm, L = synth.make_windows(C * (S - 1), 20, rate=200.0, first_window=0, special=False)
    rec = preint.preintegrate(1, _dev(torch, Sm), _dev(torch, L), synth.SIGMAS, 0, ns=20)
    dL = _dev(torch, L)
    X = torch.empty((C, S, 16), dtype=torch.float64, device="cuda")
    X[:, 0] = 0.0; X[:, 0, 3] = 1.0; X[:, 0, 4:7] = dL.view(C, S - 1, 13)[:, 0, 0:3]; X[:, 0, 10:13] = dL.view(C, S - 1, 13)[:, 0, 3:6]
    for k in range(S - 1):
        X[:, k + 1] = factor.predict_state(1, X[:, k].contiguous(), rec.view(C, S - 1, -1)[:, k].contiguous(), dL.view(C, S - 1, 13)[:, k].contiguous())
    X = X.reshape(C * S, 16)
    info0 = torch.eye(15, dtype=torch.float64, device="cuda").reshape(1, 225).repeat(C, 1) * 1e8
    cov, cr = factor.chains_marginals(1, X, rec, dL, S, prior=(info0, None, None, None), cross=True)
    assert bool(torch.isfinite(cov).all()) and bool(torch.isfinite(cr).all())
    assert bool((torch.linalg.cholesky_ex(cov.view(-1, 15, 15))[1] == 0).all())
    n = 5000
    rng = np.random.default_rng(1)
    Sm, L = synth.make_windows(n - 1, 20, rate=200.0, first_window=9000, special=False)
    rec = preint.preintegrate_host(1, Sm, L, synth.SIGMAS, 0, ns=20)
    truth = synth.make_states(rec, L, 1, perturb=False)
    idx = np.arange(50, n, 50, dtype=np.int64)
    fx = [_fix(rng, truth[k]) for k in idx]
    M = len(idx)
    sp = _sp_dev(torch, idx, np.stack([vec(w[None])[0] for w, _ in fx]), None, None, np.stack([xb for _, xb in fx]))
    dX = _dev(torch, truth)
    cov, cr = factor.chains_marginals(1, dX, _dev(torch, rec), _dev(torch, L), n, prior=(info0[:1], None, None, None), state_priors=sp, cross=True)
    assert bool(torch.isfinite(cov).all()) and bool(torch.isfinite(cr).all())
    assert bool((torch.linalg.cholesky_ex(cov.view(-1, 15, 15))[1] == 0).all())
    sd = torch.sqrt(torch.diagonal(cov.view(-1, 15, 15), dim1=1, dim2=2)).cpu().numpy()
    print(f"5 000-state chain, fixes every 50: position sigma min {sd[:, 12:15].min():.2e} max {sd[:, 12:15].max():.2e} m, M = {M} fixes")
