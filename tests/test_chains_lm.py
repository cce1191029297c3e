"""Levenberg-Marquardt of many IMU chains on the device (cpi_imu_factor_cost_batch, cpi_imu_chains_assemble_lm, cpi_imu_chains_solve,
cpi_imu_chains_lm_update, factor.chains_lm).

GTSAM is not in the reference tree, so parity with its LevenbergMarquardtOptimizer is UNPINNED.  The reference is ``np_lm`` below: the
rule of include/cpi_b200.h written in numpy, with the oracle's evaluateError and retract, the information blocks of test_marginalize and
dense Jacobi-scaled solves."""
import ctypes

import numpy as np
import pytest

from cpi_b200 import capi, synth
from test_marginalize import _np_hessian, dense_head, local, marginalize_ref, mat, prior_at_ref, vec

P = lambda a: ctypes.c_void_p(a.ctypes.data)
RD = {1: 290, 2: 308}
DEFAULTS = dict(lambda_factor=10.0, lambda_lower=0.0, lambda_upper=1e5, min_model_fidelity=1e-3, absolute_error_tol=1e-5,
                relative_error_tol=1e-5, max_iterations=100)


# ------------------------------------------------------------------------------------------------------------------
# numpy statement of the rule
# ------------------------------------------------------------------------------------------------------------------

def np_cost(orc, model, X, rec, lin):
    """Per-factor e^T P^-1 e of one chain (chain indexing)."""
    if len(rec) == 0:
        return np.zeros(0)
    e, _, _ = orc.factor_eval(model, X, rec, lin)
    Pm = mat(rec[:, 65:290])
    d = 1.0 / np.sqrt(np.einsum("kii->ki", Pm))
    W = np.linalg.inv(Pm * d[:, :, None] * d[:, None, :]) * d[:, :, None] * d[:, None, :]
    return np.einsum("ki,kij,kj->k", e, W, e)


def np_lm(orc, model, X, rec, lin, prior=None, lam=1e-5, p=DEFAULTS, max_rounds=200):
    """LM of ONE chain: X [S,16], rec / lin its S-1 factors, prior (info [15,15], rhs [15], f, lin0 [16]) or None.
    Returns (X, cost, lam, status, iterations, tries, trace) with trace = [(accepted, rho, dec, cost_cur)] per round."""
    S = len(X)
    X = X.copy()
    status, it, tries, cost, trace = 0, 0, 0, 0.0, []

    def prior_terms(Xs):
        if prior is None:
            return np.zeros((15, 15)), np.zeros(15), 0.0
        info, rhs, f0, lin0 = prior
        r, f = prior_at_ref(vec(info[None]), rhs[None], np.array([f0]), lin0[None], Xs[:1])
        return info, r[0], f[0]

    while status == 0 and tries < max_rounds:
        if S > 1:
            e, H1, H2 = orc.factor_eval(model, X, rec, lin)
            G = _np_hessian(rec, e, H1, H2)
        else:
            G = (np.zeros((0, 15, 15)),) * 3 + (np.zeros((0, 15)),) * 2 + (np.zeros(0),)
        pi, pr, pf = prior_terms(X)
        A, b, _ = dense_head(G[0], G[1], G[2], G[3], G[4], G[5], S - 1, (pi, pr, 0.0))
        cur = float(np.sum(G[5]) + pf)
        Ad = A.copy()
        Ad[np.diag_indices_from(A)] += lam * np.clip(np.diag(A), 1e-6, 1e32)
        s = 1.0 / np.sqrt(np.diag(Ad))
        dx = np.linalg.solve(Ad * s[:, None] * s[None, :], b * s) * s
        Xn = orc.retract(X, dx.reshape(S, 15))
        new = float(np.sum(np_cost(orc, model, Xn, rec, lin)) + prior_terms(Xn)[2])
        m = float(dx @ (2 * b - A @ dx))
        tries += 1
        rho = (cur - new) / m if m != 0 else np.nan
        acc = False
        if not (np.isfinite(cur) and np.isfinite(m)):
            status = 4
        elif not np.any(dx):
            status = 1
        elif np.isfinite(new) and m > 0 and rho > p["min_model_fidelity"]:
            acc = True
            it += 1
            lam = max(lam / p["lambda_factor"], p["lambda_lower"])
            dec = cur - new
            if 0.5 * dec <= p["absolute_error_tol"] or dec <= p["relative_error_tol"] * cur:
                status = 1
            elif it >= p["max_iterations"]:
                status = 2
            X = Xn
        elif lam >= p["lambda_upper"]:
            status = 3
        else:
            lam = lam * p["lambda_factor"]
        cost = new if acc else cur
        trace.append((acc, rho, cur - new, cur))
    return X, cost, lam, status, it, tries, trace


def well_posed(trace, p=DEFAULTS):
    """No decision of the trace within rounding of its threshold: rho 1e-6 from min_model_fidelity, the decrease 1e-4 (relative) from
    the tolerances."""
    for acc, rho, dec, cur in trace:
        if np.isfinite(rho):
            assert abs(rho - p["min_model_fidelity"]) > 1e-6, rho
        if acc:
            assert abs(0.5 * dec - p["absolute_error_tol"]) > 1e-4 * p["absolute_error_tol"], dec
            assert abs(dec - p["relative_error_tol"] * cur) > 1e-4 * p["relative_error_tol"] * cur, (dec, cur)


# ------------------------------------------------------------------------------------------------------------------
# problems
# ------------------------------------------------------------------------------------------------------------------

def zero_step_record(model):
    """The record of a window with zero steps: R = I, q = identity, everything else 0 (P_meas = 0: not positive definite)."""
    r = np.zeros(RD[model])
    r[3] = 1.0
    r[4:13] = np.eye(3).reshape(-1)
    return r


def perturb(orc, rng, X, large):
    """Small: v, p 1e-3, b_g 1e-5 (the smoother test's); large: v, p 0.1, attitude 1e-2 rad.  The first state is left as it is."""
    X = X.copy()
    n = len(X) - 1
    if n <= 0:
        return X
    if large:
        d = np.zeros((n, 15))
        d[:, 0:3] = rng.normal(0, 1e-2, (n, 3))
        d[:, 6:9] = rng.normal(0, 0.1, (n, 3)); d[:, 12:15] = rng.normal(0, 0.1, (n, 3))
        X[1:] = orc.retract(X[1:], d)
    else:
        X[1:, 7:10] += rng.normal(0, 1e-3, (n, 3)); X[1:, 13:16] += rng.normal(0, 1e-3, (n, 3))
        X[1:, 4:7] += rng.normal(0, 1e-5, (n, 3))
    return X


def make_problem(orc, model, sizes, seed, large=False, with_prior=False, first_window=40000):
    """Ragged chains: (X [N,16], rec [nf,RD], lin [nf,13], offs, priors list or None, per-chain (X, rec, lin))."""
    rng = np.random.default_rng(seed)
    sizes = np.asarray(sizes)
    offs = np.r_[0, np.cumsum(sizes)].astype(np.int64)
    nf = int(offs[-1] - len(sizes))
    S, L = synth.make_windows(max(nf, 1), 20, rate=200.0, first_window=first_window, special=False)
    rec = orc.preintegrate(model, S, L, synth.SIGMAS, 0, ns=20, nthreads=synth.usable_cpus())[:nf]
    L = L[:nf]
    Xs, per, priors = [], [], []
    for c, s in enumerate(sizes):
        f0 = int(offs[c] - c)
        r, l = rec[f0:f0 + s - 1], L[f0:f0 + s - 1]
        if s > 1:
            X = synth.make_states(r, l, model, perturb=False)
        else:
            X = np.zeros((1, 16)); X[0, 3] = 1.0
        X = perturb(orc, rng, X, large)
        Xs.append(X); per.append((X, r, l))
        if with_prior:
            info = np.diag(np.repeat([1e4, 1e6, 1e2, 1e4, 1e2], 3))
            priors.append((info, rng.normal(size=15) * 0.1, 0.5, orc.retract(X[:1], rng.normal(0, 1e-3, (1, 15)))[0]))
    return np.concatenate(Xs), rec, L, offs, (priors if with_prior else None), per


def dev_prior(torch, priors):
    if priors is None:
        return None
    return tuple(torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (np.stack([vec(p[0][None])[0] for p in priors]),
                                                                            np.stack([p[1] for p in priors]), np.array([p[2] for p in priors]),
                                                                            np.stack([p[3] for p in priors])))


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------

def test_argument_validation_without_gpu():
    lib = capi.load()
    buf = np.zeros(8 * 225)
    p = P(buf)
    # cpi_imu_factor_cost_batch(model, n, states, idx_i, idx_j, records, lin, f, stream)
    cost = lambda *a: lib.cpi_imu_factor_cost_batch(*a, None)
    assert cost(3, 2, p, None, None, p, p, p) == -1 and b"model" in lib.cpi_last_error()
    assert cost(1, -1, p, None, None, p, p, p) == -1 and b"negative" in lib.cpi_last_error()
    for k in (0, 3, 4, 5):
        a = [p, None, None, p, p, p]; a[k] = None
        assert cost(1, 2, *a) == -1 and b"null" in lib.cpi_last_error(), k
    assert cost(1, 2, p, p, None, p, p, p) == -1 and b"both" in lib.cpi_last_error()
    assert cost(1, 0, *[None] * 6) == 0
    # cpi_imu_chains_assemble_lm(n_chains, offs, uniform, G11, G12, G22, g1, g2, lambda, damping, pi, pr, D, E, rhs, damp, stream)
    asm = lambda n, o, u, *a: lib.cpi_imu_chains_assemble_lm(n, o, u, *a[:6], 1, *a[6:], None)
    ga = [p] * 6 + [None, None] + [p, p, p, p]
    assert asm(-1, None, 2, *ga) == -1 and b"negative" in lib.cpi_last_error()
    assert asm(3, None, 0, *ga) == -1 and b"chain_uniform" in lib.cpi_last_error()
    bad = list(ga); bad[5] = None                              # the lambda array missing
    assert asm(2, None, 3, *bad) == -1 and b"lambda" in lib.cpi_last_error()
    for k in (0, 1, 2, 3, 4, 8, 9, 10):                        # G11 .. g2, D, E, rhs
        bad = list(ga); bad[k] = None
        assert asm(2, None, 3, *bad) == -1 and b"null" in lib.cpi_last_error(), k
    assert asm(0, None, 1, *[None] * 12) == 0
    # cpi_imu_chains_solve(n_chains, offs, uniform, n_states, D, E, rhs, x, workspace, stream)
    sol = lambda *a: lib.cpi_imu_chains_solve(*a, None)
    assert sol(-1, None, 2, 4, p, p, p, p, p) == -1 and b"negative" in lib.cpi_last_error()
    assert sol(2, None, 0, 4, p, p, p, p, p) == -1 and b"chain_uniform" in lib.cpi_last_error()
    assert sol(2, None, 2, 5, p, p, p, p, p) == -1 and b"n_states" in lib.cpi_last_error()
    assert sol(3, P(buf), 0, 2, p, p, p, p, p) == -1 and b"n_states" in lib.cpi_last_error()
    for k in range(5):
        a = [p] * 5; a[k] = None
        assert sol(2, None, 2, 4, *a) == -1 and b"null" in lib.cpi_last_error(), k
    assert lib.cpi_imu_chains_solve_workspace(2, 1) < 0 and lib.cpi_imu_chains_solve_workspace(2, 4) > 0
    # cpi_imu_chains_lm_update(n_chains, offs, uniform, n_states, params, f_cur, pf_cur, f_new, pf_new, rhs, D, E, damp, delta, states_new,
    #                          states, lambda, cost, status, iterations, tries, any_running, workspace, stream)
    prm = capi.LMParams()
    upd = lambda n, o, u, N, pr, *a: lib.cpi_imu_chains_lm_update(n, o, u, N, ctypes.byref(pr) if pr is not None else None, *a, None)
    ua = [p, None, p, None] + [p] * 7 + [p] * 5 + [None, p]
    assert upd(-1, None, 3, 6, prm, *ua) == -1 and b"negative" in lib.cpi_last_error()
    assert upd(2, None, 3, 5, prm, *ua) == -1 and b"n_states" in lib.cpi_last_error()
    assert upd(2, None, 3, 6, None, *ua) == -1 and b"params" in lib.cpi_last_error()
    for field, val in (("lambda_factor", 1.0), ("lambda_factor", float("nan")), ("lambda_lower", -1.0), ("lambda_upper", -0.5),
                       ("min_model_fidelity", -1e-3), ("min_model_fidelity", 1.0), ("absolute_error_tol", -1e-5),
                       ("relative_error_tol", -1e-5), ("relative_error_tol", float("nan")), ("max_iterations", 0)):
        bad = capi.LMParams(); setattr(bad, field, val)
        assert upd(2, None, 3, 6, bad, *ua) == -1 and field.encode() in lib.cpi_last_error(), (field, val)
    for k in [0, 2] + list(range(4, 16)) + [17]:               # every required array (f, rhs .. tries, workspace)
        bad = list(ua); bad[k] = None
        assert upd(2, None, 3, 6, prm, *bad) == -1 and b"null" in lib.cpi_last_error(), k
    bad = list(ua); bad[1] = p                                 # a current prior constant without the candidate's
    assert upd(2, None, 3, 6, prm, *bad) == -1 and b"both" in lib.cpi_last_error()
    assert upd(0, None, 1, 0, prm, *[None] * 18) == 0
    # Python layer
    from cpi_b200 import factor
    with pytest.raises(ValueError):
        factor._chain_layout(3, None, n_states=4)


def test_numpy_rule_on_the_cpu(oracle):
    """The numpy statement itself: it converges, its decisions are well posed, and model 2 with large perturbations rejects steps."""
    for model, large in ((1, False), (2, True)):
        X, rec, L, offs, pri, per = make_problem(oracle, model, [1, 6, 25], 5, large=large, with_prior=True)
        for c, (Xc, r, l) in enumerate(per):
            out = np_lm(oracle, model, Xc, r, l, pri[c])
            well_posed(out[6])
            assert out[3] == 1, out[3:6]
            if large and len(Xc) > 6:
                assert out[5] >= out[4] + 2, out[3:6]


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------

def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_factor_cost_is_the_hessian_f(cuda, oracle, model):
    """K9 on the factor stress batch: bitwise k_factor_hessian's f at the same states (NaN on the same factors: those whose P_meas is
    not positive definite, the zero-step record among them), finite elsewhere; idx and chain indexing give the same bits."""
    import factor_stress as fs
    from cpi_b200 import factor
    torch = cuda
    b = fs.factor_batch(oracle, model, np.array([0.005, 4e-6, 0.01, 0.0002]))
    X, rec, lin, ii, jj = (_dev(torch, b[k]) for k in ("states", "records", "lin", "idx_i", "idx_j"))
    e, H1, H2 = factor.factor_eval(model, X, rec, lin, ii, jj)
    f_h = factor.factor_hessian(model, rec, e, H1, H2)[5].cpu().numpy()
    f_c = factor.factor_cost(model, X, rec, lin, ii, jj).cpu().numpy()
    nan = np.isnan(f_h)
    print(f"model {model}: {len(f_h)} factors, {int(nan.sum())} with P_meas not positive definite")
    assert 0 < nan.sum() < 0.1 * len(f_h)
    assert np.array_equal(np.isnan(f_c), nan) and np.all(np.isfinite(f_c[~nan]))
    assert np.all(nan[b["records"][:, 19] == 0.0])                # the zero-step record
    same = np.array_equal(f_c[~nan], f_h[~nan])
    rel = np.max(np.abs(f_c[~nan] - f_h[~nan]) / np.maximum(np.abs(f_h[~nan]), 1e-300))
    print(f"model {model}: K9 f bitwise the Hessian kernel's: {same} (max relative difference {rel:.1e})")
    assert same
    # chain indexing: states x_K^0, x_K1^0, x_K^1, ... and every other factor
    n = len(b["idx_i"])
    st = np.empty((2 * n, 16)); st[0::2] = b["states"][b["idx_i"]]; st[1::2] = b["states"][b["idx_j"]]
    rc = np.repeat(b["records"], 2, axis=0)[:2 * n - 1]; ln = np.repeat(b["lin"], 2, axis=0)[:2 * n - 1]
    f_chain = factor.factor_cost(model, _dev(torch, st), _dev(torch, rc), _dev(torch, ln)).cpu().numpy()[0::2]
    assert np.array_equal(f_chain, f_c, equal_nan=True)


def _blocks(torch, model, nf, first_window):
    from cpi_b200 import factor, preint
    S, L = synth.make_windows(nf, 20, rate=200.0, first_window=first_window, special=False)
    rec = preint.preintegrate_host(model, S, L, synth.SIGMAS, 0, ns=20)
    X = synth.make_states(rec, L, model)
    dX, dR, dL = (_dev(torch, a) for a in (X, rec, L))
    e, H1, H2 = factor.factor_eval(model, dX, dR, dL)
    return factor.factor_hessian(model, dR, e, H1, H2)


@pytest.mark.gpu
def test_per_chain_assembly_and_isolated_solve(cuda):
    """Per-chain lambda: equal lambdas give bitwise chains_assemble, distinct ones give every chain bitwise its own chain_assemble; damp
    is the added diagonal.  Isolated solve: bitwise chain_solve on SPD input; with chain 4 not SPD, NaN in chain 4 only and every other
    chain bitwise its healthy solution."""
    from cpi_b200 import factor
    torch = cuda
    G11, G12, G22, g1, g2, f = _blocks(torch, 1, 300, 20000)
    sizes = np.array([1, 5, 1, 1, 17, 64, 2, 33, 1, 9])
    C = len(sizes)
    offs = np.r_[0, np.cumsum(sizes)].astype(np.int64)
    nf = int(offs[-1] - C)
    sl = slice(0, nf)
    G = [t[sl] for t in (G11, G12, G22, g1, g2)]
    rng = np.random.default_rng(3)
    pinfo = _dev(torch, np.stack([vec(np.diag(rng.uniform(1e2, 1e6, 15))[None])[0] for _ in range(C)]))
    prhs = _dev(torch, rng.normal(size=(C, 15)))
    d_offs = _dev(torch, offs)
    for diag in (False, True):
        ref = factor.chains_assemble(*G, d_offs, 1e-3, pinfo, prhs, diagonal_damping=diag)
        got = factor.chains_assemble_lm(*G, d_offs, torch.full((C,), 1e-3, dtype=torch.float64, device="cuda"), pinfo, prhs, diagonal_damping=diag)
        assert all(torch.equal(a, b) for a, b in zip(ref, got[:3]))
        und = torch.diagonal(factor.chains_assemble(*G, d_offs, 0.0, pinfo, prhs, diagonal_damping=diag)[0].view(-1, 15, 15), dim1=1, dim2=2)
        want = 1e-3 * und.clamp(1e-6, 1e32) if diag else torch.full_like(und, 1e-3)
        assert torch.equal(want, got[3])                           # the added diagonal: lambda * clamp(undamped diagonal) or lambda
    lams = torch.from_numpy(10.0 ** rng.uniform(-6, 2, C)).cuda()
    D, E, rhs, damp = factor.chains_assemble_lm(*G, d_offs, lams, pinfo, prhs, diagonal_damping=True)
    for c in range(C):
        f0, k = int(offs[c] - c), int(sizes[c] - 1)
        s = slice(f0, f0 + k)
        Da, Ea, ra = factor.chain_assemble(G11[s], G12[s], G22[s], g1[s], g2[s], float(lams[c]), pinfo[c], prhs[c], diagonal_damping=True)
        lo, hi = int(offs[c]), int(offs[c + 1])
        assert torch.equal(Da, D[lo:hi]) and torch.equal(ra, rhs[lo:hi]) and torch.equal(Ea, E[lo:hi - 1]), c
    x_plain = factor.chain_solve(D, E, rhs)
    x_iso = factor.chains_solve(D, E, rhs, d_offs)
    assert torch.equal(x_plain, x_iso)
    # uniform layout: the same bits
    Du, Eu, ru, _ = factor.chains_assemble_lm(*(t[:4 * 6] for t in (G11, G12, G22, g1, g2)), 7, lams[:4], n_chains=4)
    assert torch.equal(factor.chains_solve(Du, Eu, ru, 7), factor.chain_solve(Du, Eu, ru))
    bad = D.clone(); bad[offs[4] + 3] = -bad[offs[4] + 3]
    xb = factor.chains_solve(bad, E, rhs, d_offs).cpu().numpy()
    xh = x_iso.cpu().numpy()
    for c in range(C):
        part = slice(offs[c], offs[c + 1])
        if c == 4:
            assert np.isnan(xb[part]).any()
        else:
            assert np.array_equal(xb[part], xh[part]), c


def _device_run(torch, model, X, rec, L, offs, pri, lam=1e-5, **kw):
    from cpi_b200 import factor
    out = factor.chains_lm(model, _dev(torch, X), _dev(torch, rec), _dev(torch, L), _dev(torch, offs), prior=dev_prior(torch, pri), lam=lam, **kw)
    return [t.cpu().numpy() for t in out]


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_first_round_is_chains_lm_step(cuda, oracle, model):
    from cpi_b200 import factor
    torch = cuda
    X, rec, L, offs, pri, _ = make_problem(oracle, model, [1, 4, 9, 2, 30, 17], 7, large=False, with_prior=True)
    Xs, cost, lam, st, it, tr = _device_run(torch, model, X, rec, L, offs, pri, max_rounds=1, check_every=0)
    new, _, _ = factor.chains_lm_step(model, _dev(torch, X), _dev(torch, rec), _dev(torch, L), _dev(torch, offs), prior=dev_prior(torch, pri))
    new = new.cpu().numpy()
    acc = it == 1
    assert acc.sum() >= 3
    for c in np.flatnonzero(acc):
        assert np.array_equal(Xs[offs[c]:offs[c + 1]], new[offs[c]:offs[c + 1]]), c


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_lm_matches_numpy(cuda, oracle, model):
    """About 40 ragged chains of 1-60 states, with and without priors, small and large perturbations: every chain's accept / reject
    sequence, final lambda, status and counters identical to the numpy statement; final states within a relative distance in retract
    coordinates; cost never above the initial cost.  Measured on an H100: 1.0e-10 (model 1), 3.5e-8 (model 2, whose chains reject up to
    53 times and several of which end lambda-exhausted, where the system is at its worst conditioning); gated at about 10x and 5x."""
    torch = cuda
    rng = np.random.default_rng(30 + model)
    sizes = np.r_[1, 60, rng.integers(1, 61, size=38)]
    worst, rejects = 0.0, 0
    for case, (large, with_prior) in enumerate(((False, False), (False, True), (True, False), (True, True))):
        X, rec, L, offs, pri, per = make_problem(oracle, model, sizes, 100 * model + case, large=large, with_prior=with_prior,
                                                 first_window=60000 + 5000 * case)
        ref = [np_lm(oracle, model, Xc, r, l, None if pri is None else pri[c]) for c, (Xc, r, l) in enumerate(per)]
        for o in ref:
            well_posed(o[6])
        R = max(o[5] for o in ref)
        seq = []                                                   # iterations after 1 .. R rounds
        for r in range(1, R + 1):
            seq.append(_device_run(torch, model, X, rec, L, offs, pri, max_rounds=r, check_every=0))
        Xs, cost, lam, st, it, tr = _device_run(torch, model, X, rec, L, offs, pri)
        for c, o in enumerate(ref):
            dev_acc = [bool(seq[r][4][c] > (seq[r - 1][4][c] if r else 0)) for r in range(o[5])]
            assert dev_acc == [t[0] for t in o[6]], (case, c, dev_acc, o[6])
            assert (lam[c], st[c], it[c], tr[c]) == (o[2], o[3], o[4], o[5]), (case, c, (lam[c], st[c], it[c], tr[c]), o[2:6])
            rejects = max(rejects, o[5] - o[4])
            Xd = Xs[offs[c]:offs[c + 1]]
            worst = max(worst, np.linalg.norm(local(o[0], Xd)) / max(np.linalg.norm(o[0][:, 4:16]), 1e-300))
            assert cost[c] <= ref[c][6][0][3] * (1 + 1e-12)
        print(f"model {model} case {case}: rounds {R}, statuses {np.bincount(st, minlength=5)}")
    print(f"model {model}: worst final-state distance to numpy (retract coordinates, relative) {worst:.2e}; most rejections {rejects}")
    if model == 2:                                             # model 1 accepts every step of these problems
        assert rejects >= 2
    assert worst <= (1e-9 if model == 1 else 2e-7)


@pytest.mark.gpu
def test_frozen_isolated_deterministic(cuda, oracle):
    """Single-state chains without a prior start converged: zero steps, states bitwise.  A zero-step record in one chain of 10: that
    chain ends non-finite with its input states, the other nine bitwise the run with the healthy record.  Two identical calls: the
    same bits."""
    torch = cuda
    sizes = [5, 1, 12, 20, 8, 1, 30, 3, 16, 9]
    X, rec, L, offs, _, _ = make_problem(oracle, 1, sizes, 11, large=True)
    a = _device_run(torch, 1, X, rec, L, offs, None)
    b = _device_run(torch, 1, X, rec, L, offs, None)
    assert all(np.array_equal(u, v) for u, v in zip(a, b))
    Xs, cost, lam, st, it, tr = a
    for c in (1, 5):
        assert st[c] == capi.LM_CONVERGED and it[c] == 0 and tr[c] == 1
        assert np.array_equal(Xs[offs[c]:offs[c + 1]], X[offs[c]:offs[c + 1]])
    assert np.all(st == capi.LM_CONVERGED) and np.all(it[[0, 2, 3]] > 0)
    bad = rec.copy()
    bad[int(offs[3] - 3) + 4] = zero_step_record(1)
    Xb, cb, lb, sb, ib, tb = _device_run(torch, 1, X, bad, L, offs, None)
    assert sb[3] == capi.LM_NONFINITE and ib[3] == 0
    assert np.array_equal(Xb[offs[3]:offs[4]], X[offs[3]:offs[4]])
    for c in range(len(sizes)):
        if c == 3:
            continue
        part = slice(offs[c], offs[c + 1])
        assert np.array_equal(Xb[part], Xs[part]) and cb[c] == cost[c] and lb[c] == lam[c] and sb[c] == st[c] and ib[c] == it[c], c


def _np_smoother_lm(orc, Xw, rec, lin, prior, lam):
    """One chains_lm of ONE window in numpy, then the marginalisation of its oldest state."""
    info, rhs, f0, x_lin = prior
    Xw = np_lm(orc, 1, Xw, rec, lin, (info, rhs, f0, x_lin), lam)[0]
    e, H1, H2 = orc.factor_eval(1, Xw[:2], rec[:1], lin[:1])
    G = _np_hessian(rec[:1], e, H1, H2)
    rhs_p, f_p = prior_at_ref(vec(info[None]), rhs[None], np.array([f0]), x_lin[None], Xw[:1])
    Lam, eta, fm = marginalize_ref(*G, 1, (info, rhs_p[0], f_p[0]), jacobi=True)
    return Xw[1:], (Lam, eta, fm, Xw[1].copy())


@pytest.mark.gpu
def test_fixed_lag_smoother_with_lm(cuda, oracle):
    """The fixed-lag loop of test_fixed_lag_smoother_of_64_sequences with chains_lm in place of one step: 16 sequences of 80 keyframes,
    lag 20; the same loop in numpy on 3 sequences agrees in retract coordinates."""
    from cpi_b200 import factor, preint
    torch = cuda
    ns, K, W, lam = 16, 80, 20, 1e-5
    S, L = synth.make_windows(ns * (K - 1), 20, rate=200.0, first_window=70000, special=False)
    rec = preint.preintegrate_host(1, S, L, synth.SIGMAS, 0, ns=20).reshape(ns, K - 1, -1)
    L = L.reshape(ns, K - 1, 13)
    rng = np.random.default_rng(22)
    truth = np.stack([synth.make_states(rec[s], L[s], 1, perturb=False) for s in range(ns)])
    X0 = truth[:, :W].copy()
    X0[:, 1:, 7:10] += rng.normal(0, 1e-3, (ns, W - 1, 3)); X0[:, 1:, 13:16] += rng.normal(0, 1e-3, (ns, W - 1, 3))
    X0[:, 1:, 4:7] += rng.normal(0, 1e-5, (ns, W - 1, 3))
    dR, dL = _dev(torch, rec), _dev(torch, L)
    info0 = np.eye(15) * 1e8
    prior = (_dev(torch, np.tile(vec(info0[None]), (ns, 1))), torch.zeros((ns, 15), dtype=torch.float64, device="cuda"),
             torch.zeros(ns, dtype=torch.float64, device="cuda"), _dev(torch, X0[:, 0].copy()))
    Xw = _dev(torch, X0)
    first = torch.arange(ns, device="cuda") * (W + 1)
    for t in range(W, K):
        xn = factor.predict_state(1, Xw[:, -1].contiguous(), dR[:, t - 1].contiguous(), dL[:, t - 1].contiguous())
        Xw = torch.cat([Xw, xn[:, None]], dim=1)
        new, cost, _, st, _, _ = factor.chains_lm(1, Xw.reshape(-1, 16).contiguous(), dR[:, t - W:t].reshape(-1, rec.shape[-1]).contiguous(),
                                                  dL[:, t - W:t].reshape(-1, 13).contiguous(), W + 1, prior=prior, lam=lam)
        Xw = new.view(ns, W + 1, 16)
        e, H1, H2 = factor.factor_eval(1, Xw.reshape(-1, 16), dR[:, t - W].contiguous(), dL[:, t - W].contiguous(), idx_i=first, idx_j=first + 1)
        G = factor.factor_hessian(1, dR[:, t - W].contiguous(), e, H1, H2)
        r_p, f_p = factor.prior_at(prior[0], prior[1], prior[2], prior[3], Xw[:, 0].contiguous())
        mi, mr, mf = factor.chain_marginalize(*G, 2, 1, prior=(prior[0], r_p, f_p), n_chains=ns)
        prior = (mi, mr, mf, Xw[:, 1].contiguous())
        Xw = Xw[:, 1:].contiguous()
    Xg = Xw.cpu().numpy()
    assert np.all(np.isfinite(Xg)) and np.all(st.cpu().numpy() == capi.LM_CONVERGED)
    worst = 0.0
    for s in (0, 7, 15):
        Xs, pr = X0[s].copy(), (info0, np.zeros(15), 0.0, X0[s, 0].copy())
        for t in range(W, K):
            Xs = np.concatenate([Xs, oracle.predict_state(1, Xs[-1:], rec[s, t - 1:t], L[s, t - 1:t])])
            Xs, pr = _np_smoother_lm(oracle, Xs, rec[s, t - W:t], L[s, t - W:t], pr, lam)
        worst = max(worst, np.linalg.norm(local(Xs, Xg[s])) / np.linalg.norm(Xs[:, 4:16]))
    print(f"fixed-lag smoother with LM vs numpy: worst relative difference {worst:.2e} (retract coordinates)")
    assert worst <= 1e-9
