"""Robust (Huber, Cauchy) losses on state priors (cpi_imu_state_priors_robust, factor.state_priors_robust and the state_prior_loss
argument of factor.chains_lm_step / chains_lm / chain_marginalize; DESIGN.md section 3h).

GTSAM's noiseModel::Robust is not in the reference tree, so parity is UNPINNED.  The reference is ``np_loss`` below: the cost
c(s) = 2 rho(sqrt s) of a whitened squared residual s and its IRLS weight w(s) = dc/ds.  A robust prior enters the system as
(w W, w rhs', c(s)) at the states it is linearised at; the GPU tests compare the kernel with that per prior, and the solver entry
points with numpy statements of the whole reweighted system."""
import ctypes

import numpy as np
import pytest

from cpi_b200 import capi, synth
from test_chains_lm import DEFAULTS, dev_prior, make_problem, np_cost, well_posed
from test_marginalize import _dense_truth, _np_hessian, local, marginalize_ref, mat, prior_at_ref, random_prior, vec
from test_state_priors import (_chain_idx, _dev, _meas_priors, _np_system, _per_chain_sps, _sp_dev, csr, dense_chain, fold_ref,
                               random_layout)

P = lambda a: ctypes.c_void_p(a.ctypes.data)
HUBER_K, CAUCHY_K = 1.345, 2.3849          # GTSAM's 95 %-efficiency thresholds


# ------------------------------------------------------------------------------------------------------------------
# numpy statements
# ------------------------------------------------------------------------------------------------------------------

def np_loss(code, k, s):
    """(w, c) of whitened squared residuals s under loss codes `code` with thresholds k (arrays, broadcast): the header's table.
    An unknown code or k outside 0 < k^2 < inf gives NaN."""
    code, k, s = (np.asarray(a) for a in np.broadcast_arrays(code, k, s))
    s = s.astype(np.float64)
    w, c = np.full(s.shape, np.nan), np.full(s.shape, np.nan)
    with np.errstate(all="ignore"):
        k2 = k * k
        ok = (k > 0) & (k2 > 0) & np.isfinite(k2)
        g = code == capi.LOSS_GAUSSIAN
        w[g], c[g] = 1.0, s[g]
        hi = (code == capi.LOSS_HUBER) & ok & (s <= k2)
        w[hi], c[hi] = 1.0, s[hi]
        ho = (code == capi.LOSS_HUBER) & ok & ~(s <= k2)
        r = np.sqrt(s[ho])
        w[ho], c[ho] = k[ho] / r, 2.0 * k[ho] * r - k2[ho]
        ca = (code == capi.LOSS_CAUCHY) & ok
        u = s[ca] / k2[ca]
        w[ca], c[ca] = 1.0 / (1.0 + u), k2[ca] * np.log1p(u)
        big = np.zeros(s.shape, bool)
        big[ca] = np.isinf(u)                                      # k < 1 and finite s above k^2 DBL_MAX: u overflows
        w[big], c[big] = k2[big] / s[big], k2[big] * (np.log(s[big]) - np.log(k2[big]))
    return w, c


def robust_ref(code, k, info, rhs, f):
    """The kernel's statement: (w info, w rhs, c(f)) per prior; a weight of 1 copies."""
    w, c = np_loss(code, k, f)
    one = (w == 1.0)
    return (np.where(one[:, None], info, w[:, None] * info), np.where(one[:, None], rhs, w[:, None] * rhs), c)


def np_system_rb(orc, model, Xc, r, l, prior, sps, blocks=None):
    """_np_system of test_state_priors.py with robust state priors (local index, info, rhs, f, lin, code, k): each moved to its
    state, then reweighted there, (w W, w rhs', c(s))."""
    A, b, cost = _np_system(orc, model, Xc, r, l, prior, [], blocks=blocks)
    for q, info, rhs, f, lin, code, k in sps:
        rr, ff = prior_at_ref(info[None], rhs[None], np.array([f]), lin[None], Xc[q:q + 1])
        w, c = np_loss(code, k, ff)
        s = slice(15 * q, 15 * q + 15)
        A[s, s] += w[0] * mat(info)[0]; b[s] += w[0] * rr[0]; cost += c[0]
    return A, b, cost


def np_cost_rb(orc, model, Xc, r, l, prior, sps):
    c = float(np.sum(np_cost(orc, model, Xc, r, l)))
    if prior is not None:
        c += prior_at_ref(vec(prior[0][None]), prior[1][None], np.array([prior[2]]), prior[3][None], Xc[:1])[1][0]
    for q, info, rhs, f, lin, code, k in sps:
        ff = prior_at_ref(info[None], rhs[None], np.array([f]), lin[None], Xc[q:q + 1])[1]
        c += np_loss(code, k, ff)[1][0]
    return c


def np_lm_rb(orc, model, X, rec, lin, prior, sps, lam=1e-5, p=DEFAULTS, max_rounds=200):
    """np_lm_sp of test_state_priors.py on the reweighted system: the same LM rule, the weights recomputed every round."""
    S = len(X)
    X = X.copy()
    status, it, tries, cost, trace = 0, 0, 0, 0.0, []
    while status == 0 and tries < max_rounds:
        A, b, cur = np_system_rb(orc, model, X, rec, lin, prior, sps)
        Ad = A.copy()
        Ad[np.diag_indices_from(A)] += lam * np.clip(np.diag(A), 1e-6, 1e32)
        s = 1.0 / np.sqrt(np.diag(Ad))
        dx = np.linalg.solve(Ad * s[:, None] * s[None, :], b * s) * s
        Xn = orc.retract(X, dx.reshape(S, 15))
        new = np_cost_rb(orc, model, Xn, rec, lin, prior, sps)
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


def per_chain_rb(offs, idx, info, rhs, f, lin, code, k):
    sps = _per_chain_sps(offs, idx, info, rhs, f, lin)
    pos = [0] * (len(offs) - 1)
    out = [[] for _ in sps]
    for q in range(len(idx)):                                      # _per_chain_sps keeps the input order within a chain
        c = int(np.searchsorted(offs, idx[q], side="right") - 1)
        out[c].append(sps[c][pos[c]] + (int(code[q]), float(k[q])))
        pos[c] += 1
    return out


def mixed_losses(M):
    """Codes cycling Gaussian, Huber, Cauchy, with GTSAM's thresholds."""
    code = (np.arange(M) % 3).astype(np.int32)
    k = np.where(code == capi.LOSS_HUBER, HUBER_K, np.where(code == capi.LOSS_CAUCHY, CAUCHY_K, 0.0))
    return code, k


def add_outliers(sp, every, offset):
    """Every `every`-th measurement moved by `offset` metres in position and metres per second in velocity."""
    lin = sp[4].copy()
    lin[::every, 7:10] += offset
    lin[::every, 13:16] += offset
    return sp[:4] + (lin,)


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("code,k", [(capi.LOSS_HUBER, 0.5), (capi.LOSS_HUBER, HUBER_K), (capi.LOSS_HUBER, 10.0), (capi.LOSS_CAUCHY, 0.5),
                                    (capi.LOSS_CAUCHY, CAUCHY_K), (capi.LOSS_CAUCHY, 10.0)])
def test_weight_is_the_derivative_of_the_cost(code, k):
    s = np.logspace(-4, 6, 301) * 1.0137                           # no point within the difference step of a Huber threshold k^2
    w, c = np_loss(code, k, s)
    h = 1e-5 * s
    cd = (np_loss(code, k, s + h)[1] - np_loss(code, k, s - h)[1]) / (2 * h)
    assert np.all(np.abs(cd - w) <= 1e-7 * np.maximum(w, 1e-300) + 1e-9), np.max(np.abs(cd - w) / w)
    assert np.all(w > 0) and np.all(w <= 1) and np.all(c <= s * (1 + 1e-15))         # robust: never above the Gaussian cost
    g = np_loss(capi.LOSS_GAUSSIAN, np.nan, s)
    assert np.array_equal(g[0], np.ones_like(s)) and np.array_equal(g[1], s)


def test_huber_is_continuous_at_the_threshold_and_cauchy_tends_to_gaussian():
    for k in (0.1, HUBER_K, 3.0, 1e3):
        k2 = k * k
        lo, hi = np_loss(1, k, k2 * (1 - 1e-12)), np_loss(1, k, k2 * (1 + 1e-12))
        at = np_loss(1, k, k2)
        assert at[0][()] == 1.0 and at[1][()] == k2
        assert abs(lo[0] - hi[0]) <= 1e-11 and abs(lo[1] - hi[1]) <= 1e-11 * k2
    s = np.logspace(-3, 3, 61)
    for k in (1e3, 1e5, 1e7):
        w, c = np_loss(2, k, s)
        assert np.all(np.abs(c - s) <= s * s / (k * k) + 4e-16 * s) and np.all(np.abs(1 - w) <= s / (k * k) + 2.3e-16)
    for code, k in ((3, 1.0), (-1, 1.0), (1, 0.0), (1, -1.0), (2, np.nan), (2, np.inf), (1, 1e200), (2, 1e-200)):
        w, c = np_loss(code, k, 2.0)
        assert np.isnan(w) and np.isnan(c), (code, k)


@pytest.mark.parametrize("seed", [0, 1])
def test_reweighted_dense_system_is_the_fold_of_weighted_priors(seed):
    """Ragged chains with measurement priors of mixed losses (inliers and outliers) moved to random states: the dense system with
    every prior reweighted on its own state equals the numpy fold of the weighted priors (robust_ref, then fold_ref)."""
    rng = np.random.default_rng(seed)
    sizes = np.r_[1, 2, 9, 1, rng.integers(1, 10, size=12)]
    offs, blocks, chain_prior = random_layout(rng, sizes)
    N = int(offs[-1])
    X = np.zeros((N, 16)); X[:, 3] = 1.0; X[:, 4:16] = rng.normal(size=(N, 12))
    idx = rng.integers(0, N, size=3 * N)
    M = len(idx)
    W = [random_prior(rng, scale=(1e-1, 1e-2, 1e-2, 1e-1, 1e-2))[0] for _ in range(M)]
    info = vec(np.stack(W))
    lin = X[idx].copy()
    lin[:, 4:16] += rng.normal(size=(M, 12)) * np.where(rng.random(M) < 0.3, 1.0, 1e-3)[:, None]   # 30 % outliers
    code = rng.integers(0, 3, size=M).astype(np.int32)
    k = rng.uniform(0.5, 3.0, size=M)
    rr, ff = prior_at_ref(info, np.zeros((M, 15)), np.zeros(M), lin, X[idx])
    w, c = np_loss(code, k, ff)
    assert np.any(w < 1e-2) and np.any((code == 1) & (w == 1.0)) and np.any((code == 2) & (w > 0.9))
    iw, rw, cw = robust_ref(code, k, info, rr, ff)
    order, sp_off = csr(idx, N)
    G11, G12, G22, g1, g2, fk = blocks
    (F11, F22, fg1, fg2, ffk), (fpi, fpr, fpf) = fold_ref(offs, sp_off, iw[order], rw[order], cw[order], (G11, G22, g1, g2, fk), chain_prior)
    for ch in range(len(sizes)):
        lo, hi, f0 = int(offs[ch]), int(offs[ch + 1]), int(offs[ch] - ch)
        s = slice(f0, f0 + hi - lo - 1)
        A, b, F = dense_chain(F11[s], G12[s], F22[s], fg1[s], fg2[s], ffk[s], (fpi[ch], fpr[ch], fpf[ch]))
        pr = (mat(chain_prior[0][ch:ch + 1])[0], chain_prior[1][ch], chain_prior[2][ch], None)
        A0, b0, F0 = _np_system(None, 1, X[lo:hi], None, None, None, [], blocks=[g[s] for g in blocks])
        A0[:15, :15] += pr[0]; b0[:15] += pr[1]; F0 += pr[2]
        sps = [(int(idx[q] - lo), info[q], np.zeros(15), 0.0, lin[q], int(code[q]), float(k[q])) for q in np.flatnonzero((idx >= lo) & (idx < hi))]
        for q, inf_q, _, _, lin_q, cq, kq in sps:
            r1, f1 = prior_at_ref(inf_q[None], np.zeros((1, 15)), np.zeros(1), lin_q[None], X[lo + q:lo + q + 1])
            wq, cq_ = np_loss(cq, kq, f1)
            sl = slice(15 * q, 15 * q + 15)
            A0[sl, sl] += wq[0] * mat(inf_q)[0]; b0[sl] += wq[0] * r1[0]; F0 += cq_[0]
        sc = np.abs(A0).max()
        assert np.allclose(A, A0, rtol=0, atol=1e-14 * sc), ch
        assert np.allclose(b, b0, rtol=1e-13, atol=1e-13 * max(np.abs(b0).max(), 1.0)), ch
        assert abs(F - F0) <= 1e-13 * (abs(F0) + np.abs(fk).sum() + np.abs(cw).sum()), ch


def test_argument_validation_without_gpu():
    import torch
    from cpi_b200 import factor
    lib = capi.load()
    buf = np.zeros(8 * 225)
    ib = np.zeros(8, dtype=np.int32)
    p, pi = P(buf), P(ib)
    # cpi_imu_state_priors_robust(n, loss, loss_k, info, rhs, f, info_out, rhs_out, f_out, stream)
    rob = lambda n, *a: lib.cpi_imu_state_priors_robust(n, *a, None)
    ga = [pi, p, p, p, p, p, p, p]
    assert rob(-1, *ga) == -1 and b"negative" in lib.cpi_last_error()
    assert rob((1 << 31) + 1, *ga) == -1 and b"too many" in lib.cpi_last_error()
    for j in (0, 1, 4, 7):
        bad = list(ga); bad[j] = None
        assert rob(2, *bad) == -1 and b"null" in lib.cpi_last_error(), j
    for j in (5, 6):
        bad = list(ga); bad[j] = None
        assert rob(2, *bad) == -1 and b"both" in lib.cpi_last_error(), j
    for j in (2, 3):
        bad = list(ga); bad[j] = None
        assert rob(2, *bad) == -1 and b"info / rhs" in lib.cpi_last_error(), j
    assert rob(0, *[None] * 8) == 0
    # the Python layer raises before the device is touched
    N = 12
    X, rec, lin = torch.zeros(N, 16, dtype=torch.float64), torch.zeros(N - 3, 290, dtype=torch.float64), torch.zeros(N - 3, 13, dtype=torch.float64)
    G = [torch.zeros(N - 3, k, dtype=torch.float64) for k in (225, 225, 225, 15, 15, 1)]
    sp = (torch.tensor([0, 5], dtype=torch.int64), torch.zeros(2, 225, dtype=torch.float64), None, torch.zeros(2, dtype=torch.float64),
          torch.zeros(2, 16, dtype=torch.float64))
    code, k = torch.tensor([1, 2], dtype=torch.int32), torch.tensor([1.345, 2.3849], dtype=torch.float64)
    calls = (lambda sp, l: factor.chains_lm_step(1, X, rec, lin, 4, state_priors=sp, state_prior_loss=l),
             lambda sp, l: factor.chains_lm(1, X, rec, lin, 4, state_priors=sp, state_prior_loss=l),
             lambda sp, l: factor.chain_marginalize(*G, 4, 1, state_priors=sp, state_prior_loss=l))
    rhs1 = torch.zeros(2, 15, dtype=torch.float64); rhs1[1, 3] = 1.0
    f1 = torch.tensor([0.0, 0.5], dtype=torch.float64)
    for j, call in enumerate(calls):
        cases = [(sp, (code,), ValueError, "state_prior_loss is"), (None, (code, k), ValueError, "needs state_priors"),
                 (sp, (code.long(), k), ValueError, "int32"), (sp, (code.double(), k), ValueError, "int32"),
                 (sp, (code, k.float()), ValueError, "float64"), (sp, (code[:1], k), ValueError, "one code"),
                 (sp, (code, k[:1]), ValueError, "one threshold"), (sp, (code.reshape(2, 1), k), ValueError, "1-d"),
                 (sp, (torch.tensor([1, 3], dtype=torch.int32), k), ValueError, "loss codes"),
                 (sp, (torch.tensor([-1, 0], dtype=torch.int32), k), ValueError, "loss codes"),
                 (sp, (code, torch.tensor([0.0, 1.0], dtype=torch.float64)), ValueError, "threshold k"),
                 (sp, (code, torch.tensor([1.0, -2.0], dtype=torch.float64)), ValueError, "threshold k"),
                 (sp, (code, torch.tensor([float("nan"), 1.0], dtype=torch.float64)), ValueError, "threshold k"),
                 (sp, (code, torch.tensor([1.0, float("inf")], dtype=torch.float64)), ValueError, "threshold k"),
                 (sp, (code, torch.tensor([1.0, 1e200], dtype=torch.float64)), ValueError, "threshold k"),
                 (sp, (code, k), ValueError, "CUDA")]
        if j < 2:                                                  # a robust prior in LM must be a measurement prior
            cases += [((sp[0], sp[1], rhs1, None, sp[4]), (code, k), ValueError, "measurement prior"),
                      ((sp[0], sp[1], None, f1, sp[4]), (code, k), ValueError, "measurement prior")]
        else:                                                      # chain_marginalize takes them moved, with f' = s
            cases += [((sp[0], sp[1], rhs1, None, sp[4]), (code, k), ValueError, "f must be given")]
        for s_, l_, exc, msg in cases:
            with pytest.raises(exc, match=msg):
                call(s_, l_)
    # a Gaussian code with any k, and a Gaussian prior with a nonzero rhs, pass the value checks (then meet the device check)
    for call in calls[:2]:
        with pytest.raises(ValueError, match="CUDA"):
            call((sp[0], sp[1], rhs1, f1, sp[4]), (torch.tensor([0, 0], dtype=torch.int32), torch.tensor([float("nan"), -1.0], dtype=torch.float64)))


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------

def _ulps(got, want):
    with np.errstate(all="ignore"):
        d = np.abs(got - want) / np.spacing(np.abs(want))
    return np.where(got == want, 0.0, d)


@pytest.mark.gpu
def test_kernel_against_numpy(cuda):
    """Per prior: Gaussian and Huber inliers are bitwise copies, Huber outliers and Cauchy within a few ulp of numpy (sqrt, log1p);
    the f-only pass writes the full pass's f bit for bit, in place as well; two runs give the same bits; invalid codes and k give NaN."""
    from cpi_b200 import factor
    torch = cuda
    rng = np.random.default_rng(3)
    M = 5003
    W = vec(np.stack([random_prior(rng)[0] for _ in range(64)]))
    info = W[rng.integers(0, 64, size=M)] * rng.uniform(0.5, 2.0, size=(M, 1))
    rhs = rng.normal(size=(M, 15)) * 10.0
    s = 10.0 ** rng.uniform(-6, 7, size=M)
    code = rng.integers(0, 3, size=M).astype(np.int32)
    k = rng.uniform(0.3, 5.0, size=M)
    s[:50] = k[:50] ** 2                                            # exactly at the Huber threshold: an inlier
    s[50:60] = 0.0
    code[-8:] = [3, -1, 1, 1, 2, 2, 1, 2]                           # invalid codes and thresholds: NaN
    k[-6:] = [0.0, -1.0, np.nan, np.inf, 1e200, 1e-200]
    d = lambda a: _dev(torch, a)
    ri, rr, rc = robust_ref(code, k, info, rhs, s)
    outs = []
    for _ in range(2):
        io, ro, fo = factor.state_priors_robust(d(code), d(k), d(info), d(rhs), d(s))
        outs.append([t.cpu().numpy() for t in (io, ro, fo)])
    for a, b in zip(outs[0], outs[1]):
        assert np.array_equal(a, b, equal_nan=True)
    io, ro, fo = outs[0]
    w, _ = np_loss(code, k, s)
    copy = w == 1.0
    assert copy.sum() > M // 3 and np.any((code == 1) & copy) and np.any((code == 1) & ~copy)
    assert np.array_equal(io[copy], info[copy]) and np.array_equal(ro[copy], rhs[copy]) and np.array_equal(fo[copy], rc[copy])
    bad = np.isnan(w)
    assert np.array_equal(np.flatnonzero(bad), np.arange(M - 8, M))
    assert np.all(np.isnan(fo[bad])) and np.all(np.isnan(io[bad])) and np.all(np.isnan(ro[bad]))
    rest = ~copy & ~bad
    ui, ur, uf = _ulps(io[rest], ri[rest]).max(), _ulps(ro[rest], rr[rest]).max(), _ulps(fo[rest], rc[rest]).max()
    print(f"robust kernel vs numpy: worst {ui:.1f} / {ur:.1f} / {uf:.1f} ulp (info / rhs / cost) over {rest.sum()} reweighted priors")
    assert max(ui, ur, uf) <= 4.0
    # the f-only pass, and the full pass in place (rhs_out = rhs, f_out = f)
    _, _, f_only = factor.state_priors_robust(d(code), d(k), None, None, d(s))
    assert np.array_equal(f_only.cpu().numpy(), fo, equal_nan=True)
    tr, tf = d(rhs), d(s)
    io2, ro2, fo2 = factor.state_priors_robust(d(code), d(k), d(info), tr, tf, rhs_out=tr, f_out=tf)
    assert ro2.data_ptr() == tr.data_ptr() and fo2.data_ptr() == tf.data_ptr()
    assert all(np.array_equal(a.cpu().numpy(), b, equal_nan=True) for a, b in zip((io2, ro2, fo2), (io, ro, fo)))


def _moved(torch, sp, X):
    """The measurement priors of sp moved to the states X (for chain_marginalize): (idx, info, rhs', f', x)."""
    from cpi_b200 import factor
    idx, info, rhs, f, lin = sp
    x = X[idx]
    rr, ff = factor.prior_at(_dev(torch, info), _dev(torch, rhs), _dev(torch, f), _dev(torch, lin), _dev(torch, x))
    return (_dev(torch, idx), _dev(torch, info), rr, ff, _dev(torch, x))


@pytest.mark.gpu
def test_no_loss_gaussian_codes_and_huber_inliers_are_bitwise_the_plain_calls(cuda, oracle):
    from cpi_b200 import factor
    torch = cuda
    rng = np.random.default_rng(17)
    X, rec, L, offs, pri, _ = make_problem(oracle, 1, [1, 4, 9, 2, 30, 17], 7, with_prior=True)
    sp = _meas_priors(oracle, rng, X, offs, 3, "mixed")
    M = len(sp[0])
    a = (_dev(torch, X), _dev(torch, rec), _dev(torch, L), _dev(torch, offs))
    losses = [None, (np.zeros(M, dtype=np.int32), rng.normal(size=M)), (np.ones(M, dtype=np.int32), np.full(M, 1e6))]
    dl = lambda l: None if l is None else (_dev(torch, l[0]), _dev(torch, l[1]))
    for fn in (factor.chains_lm_step, factor.chains_lm):
        ref = fn(1, *a, prior=dev_prior(torch, pri), state_priors=_sp_dev(torch, *sp))
        for l in losses:
            got = fn(1, *a, prior=dev_prior(torch, pri), state_priors=_sp_dev(torch, *sp), state_prior_loss=dl(l))
            what = (fn.__name__, None if l is None else int(l[0][0]))
            assert all(torch.equal(u, v) for u, v in zip(ref, got)), what
    nm = _dev(torch, np.array([0, 2, 5, 1, 29, 3]))
    e, H1, H2 = factor.factor_eval(1, a[0], a[1], a[2], *_chain_idx(torch, offs))
    G = factor.factor_hessian(1, a[1], e, H1, H2)
    pr = dev_prior(torch, pri)[:3]
    msp = _moved(torch, sp, X)
    ref = factor.chain_marginalize(*G, a[3], nm, prior=pr, state_priors=msp)
    for l in losses:
        got = factor.chain_marginalize(*G, a[3], nm, prior=pr, state_priors=msp, state_prior_loss=dl(l))
        assert all(torch.equal(u, v) for u, v in zip(ref, got))


def _device_lm(torch, model, X, rec, L, offs, pri, sp, loss, **kw):
    from cpi_b200 import factor
    out = factor.chains_lm(model, _dev(torch, X), _dev(torch, rec), _dev(torch, L), _dev(torch, offs), prior=dev_prior(torch, pri),
                           state_priors=None if sp is None else _sp_dev(torch, *sp),
                           state_prior_loss=None if loss is None else (_dev(torch, loss[0]), _dev(torch, loss[1])), **kw)
    return [t.cpu().numpy() for t in out]


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_lm_matches_numpy(cuda, oracle, model):
    """chains_lm with Gaussian, Huber and Cauchy position, velocity and full fixes on ragged chains, every 5th fix an outlier,
    against np_lm_rb: identical accept / reject sequences, final lambda, status and counters (no rho within 1e-6 of the threshold),
    final states at the gates of test_state_priors.py::test_lm_matches_numpy."""
    torch = cuda
    rng = np.random.default_rng(90 + model)
    sizes = np.r_[1, 25, rng.integers(1, 26, size=10)]
    worst, n_out = 0.0, 0
    for case, (kind, large, offset) in enumerate((("p", False, 0.2), ("mixed", True, 0.5))):
        X, rec, L, offs, pri, per = make_problem(oracle, model, sizes, 300 * model + case, large=large, with_prior=True,
                                                 first_window=70000 + 5000 * case)
        sp = add_outliers(_meas_priors(oracle, rng, X, offs, 3, kind), 5, offset)
        loss = mixed_losses(len(sp[0]))
        sps = per_chain_rb(offs, *sp, *loss)
        ref = [np_lm_rb(oracle, model, Xc, r, l, pri[c], sps[c]) for c, (Xc, r, l) in enumerate(per)]
        for o in ref:
            well_posed(o[6])
        R = max(o[5] for o in ref)
        seq = [_device_lm(torch, model, X, rec, L, offs, pri, sp, loss, max_rounds=r, check_every=0) for r in range(1, R + 1)]
        Xs, cost, lam, st, it, tr = _device_lm(torch, model, X, rec, L, offs, pri, sp, loss)
        for c, o in enumerate(ref):
            dev_acc = [bool(seq[r][4][c] > (seq[r - 1][4][c] if r else 0)) for r in range(o[5])]
            assert dev_acc == [t[0] for t in o[6]], (case, c, dev_acc, o[6])
            assert (lam[c], st[c], it[c], tr[c]) == (o[2], o[3], o[4], o[5]), (case, c, (lam[c], st[c], it[c], tr[c]), o[2:6])
            Xd = Xs[offs[c]:offs[c + 1]]
            worst = max(worst, np.linalg.norm(local(o[0], Xd)) / max(np.linalg.norm(o[0][:, 4:16]), 1e-300))
            n_out += sum(1 for q in sps[c] if np_loss(q[5], q[6], prior_at_ref(q[1][None], q[2][None], np.array([q[3]]), q[4][None],
                                                                                o[0][q[0]:q[0] + 1])[1])[0][0] < 0.1)
        print(f"model {model} case {kind}: rounds {R}, statuses {np.bincount(st, minlength=5)}")
    print(f"model {model}: {n_out} priors end with weight < 0.1; worst final-state distance to numpy (retract coordinates, relative) {worst:.2e}")
    assert n_out > 0
    assert worst <= (1e-9 if model == 1 else 2e-7)


def _outlier_problem(rng, n_chains, S, every, first_window):
    """Model-1 chains of S states (small perturbations) with a 1 cm position fix every `every`-th keyframe."""
    from cpi_b200 import preint
    Sm, L = synth.make_windows(n_chains * (S - 1), 20, rate=200.0, first_window=first_window, special=False)
    rec = preint.preintegrate_host(1, Sm, L, synth.SIGMAS, 0, ns=20)
    truth = np.concatenate([synth.make_states(rec[c * (S - 1):(c + 1) * (S - 1)], L[c * (S - 1):(c + 1) * (S - 1)], 1, perturb=False)
                            for c in range(n_chains)])
    X = truth.copy().reshape(n_chains, S, 16)
    X[:, 1:, 7:10] += rng.normal(0, 1e-3, (n_chains, S - 1, 3)); X[:, 1:, 13:16] += rng.normal(0, 1e-3, (n_chains, S - 1, 3))
    X[:, 1:, 4:7] += rng.normal(0, 1e-5, (n_chains, S - 1, 3))
    idx = (np.arange(n_chains)[:, None] * S + np.arange(every, S, every)[None, :]).reshape(-1)
    Wm = np.zeros((15, 15)); Wm[12:15, 12:15] = np.eye(3) * 1e4
    lin = truth[idx].copy()
    lin[:, 13:16] += rng.normal(0, 0.01, (len(idx), 3))
    M = len(idx)
    return X.reshape(-1, 16), rec, L, truth, (idx.astype(np.int64), np.tile(vec(Wm[None]), (M, 1)), np.zeros((M, 15)), np.zeros(M), lin)


@pytest.mark.gpu
def test_outlier_rejection(cuda):
    """40 chains of 30 states with a 1 cm position fix every 5th keyframe; in every other chain the fix on keyframe 15 is replaced by
    a 5 m outlier (a whitened residual of 500).  Under each loss the outlier's pull is the worst position shift from the run of the
    same loss without that fix.  Its weight is about 2.7e-3 under Huber (k = 1.345) and 2.3e-5 under Cauchy (k = 2.3849), so the
    pull shrinks by about those factors against the Gaussian run: gated at 2e-2 and 1e-3.  LM runs to tight tolerances, so that
    where each run stops is far below the pulls compared."""
    from cpi_b200 import factor
    torch = cuda
    rng = np.random.default_rng(12)
    params = capi.LMParams(absolute_error_tol=0.0, relative_error_tol=1e-13)
    C, S = 40, 30
    X, rec, L, truth, sp = _outlier_problem(rng, C, S, 5, 61000)
    q_out = np.flatnonzero(np.isin(sp[0], np.arange(0, C, 2) * S + 15))
    assert len(q_out) == C // 2
    bad = sp[4].copy()
    bad[q_out, 13:16] += 5.0 / np.sqrt(3.0)
    keep = np.setdiff1d(np.arange(len(sp[0])), q_out)
    dX, dR, dL = _dev(torch, X), _dev(torch, rec), _dev(torch, L)
    prior = (torch.eye(15, dtype=torch.float64, device="cuda").reshape(1, 225).repeat(C, 1) * 1e8, None, None, dX[::S].clone())

    def run(sel, lin, code, k):
        M = len(sel)
        s_ = (sp[0][sel], sp[1][sel], sp[2][sel], sp[3][sel], lin[sel])
        loss = None if code is None else (_dev(torch, np.full(M, code, dtype=np.int32)), _dev(torch, np.full(M, k)))
        Xs, cost, lam, st, it, tr = factor.chains_lm(1, dX, dR, dL, S, prior=prior, params=params, state_priors=_sp_dev(torch, *s_),
                                                     state_prior_loss=loss)
        st = st.cpu().numpy()
        assert np.all(st != capi.LM_NONFINITE), st
        return Xs.cpu().numpy().reshape(C, S, 16)

    shift, outs = {}, {}
    all_q = np.arange(len(sp[0]))
    for name, code, k in (("gaussian", None, 0.0), ("huber", capi.LOSS_HUBER, HUBER_K), ("cauchy", capi.LOSS_CAUCHY, CAUCHY_K)):
        clean = run(keep, sp[4], code, k)
        dirty = run(all_q, bad, code, k)
        d = np.linalg.norm(dirty[::2, :, 13:16] - clean[::2, :, 13:16], axis=2)
        shift[name] = float(d.max())
        outs[name] = dirty
        assert np.linalg.norm(dirty[1::2, :, 13:16] - clean[1::2, :, 13:16], axis=2).max() == 0.0     # chains without the outlier
    xo = outs["gaussian"].reshape(-1, 16)[sp[0][q_out]]
    rh, rc = shift["huber"] / shift["gaussian"], shift["cauchy"] / shift["gaussian"]
    print(f"outlier pull (worst position shift): gaussian {shift['gaussian']:.3e} m, huber {shift['huber']:.3e} m (ratio {rh:.2e}), "
          f"cauchy {shift['cauchy']:.3e} m (ratio {rc:.2e}); gaussian residual at the outlier "
          f"{np.linalg.norm(xo[:, 13:16] - bad[q_out, 13:16], axis=1).max():.3f} m")
    assert shift["gaussian"] > 1e-4
    assert rh <= 2e-2 and rc <= 1e-3


@pytest.mark.gpu
def test_marginalize_with_robust_priors(cuda, oracle):
    """K8 with robust priors on eliminated heads equals marginalize_ref with them reweighted at the blocks' point (weights frozen
    there); the reduced solve plus the remaining (reweighted) priors equals the full solve's tail."""
    from cpi_b200 import factor
    torch = cuda
    rng = np.random.default_rng(78)
    sizes = np.r_[2, 9, 1, 30, rng.integers(1, 31, size=20)]
    X, rec, L, offs, _, _ = make_problem(oracle, 1, sizes, 10, first_window=91000)
    C, N = len(sizes), int(offs[-1])
    nm = np.array([rng.integers(0, s) for s in sizes], dtype=np.int64)
    nm[0] = 1; nm[1] = 8
    dX, dR, dL, dO = (_dev(torch, a) for a in (X, rec, L, offs))
    e, H1, H2 = factor.factor_eval(1, dX, dR, dL, *_chain_idx(torch, offs))
    G = factor.factor_hessian(1, dR, e, H1, H2)
    Gh = [t.cpu().numpy() for t in G]

    def moved_meas(idx, Xs):
        """Measurement priors on idx, moved to Xs[idx]: (info W, rhs' = -W delta, f' = delta^T W delta), every 4th an outlier (the
        codes of mixed_losses cycle with period 3, so the outliers meet every loss)."""
        M = len(idx)
        W = vec(np.stack([random_prior(rng, scale=(1e-2, 1e-3, 1e-2, 1e-3, 1e-2))[0] for _ in range(M)]))
        dlt = rng.normal(size=(M, 15)) * np.repeat([1e-2, 1e-3, 1e-2, 1e-3, 1e-2], 3) * np.where(np.arange(M) % 4 == 1, 30.0, 0.5)[:, None]
        u = np.einsum("nrc,nc->nr", mat(W), dlt)
        return W, -u, np.einsum("nr,nr->n", dlt, u), Xs[idx]

    idx = np.r_[offs[:-1], rng.integers(0, N, size=3 * C)].astype(np.int64)
    info, rhs, f, lin = moved_meas(idx, X)
    code, k = mixed_losses(len(idx))
    w, cst = np_loss(code, k, f)
    assert np.any(w < 0.1) and np.any(w == 1.0)
    pri = [random_prior(rng, scale=(1e-3, 1e-4, 1e-2, 1e-3, 1e-2)) for _ in range(C)]
    pinfo = np.stack([vec(p[0][None])[0] for p in pri]); prhs = np.stack([p[1] for p in pri]); pf = np.array([p[2] for p in pri])
    oi, orr, of = (t.cpu().numpy() for t in factor.chain_marginalize(*G, dO, _dev(torch, nm), prior=tuple(_dev(torch, a) for a in (pinfo, prhs, pf)),
                                                                      state_priors=_sp_dev(torch, idx, info, rhs, f, lin),
                                                                      state_prior_loss=(_dev(torch, code), _dev(torch, k))))
    errs = []
    for c in range(C):
        m, f0, lo = int(nm[c]), int(offs[c] - c), int(offs[c])
        if m == 0:
            assert np.array_equal(oi[c], pinfo[c]) and np.array_equal(orr[c], prhs[c]) and of[c] == pf[c]
            continue
        sl = slice(f0, f0 + m)
        M11, fg1, ff = mat(Gh[0][sl]).copy(), Gh[3][sl].copy(), Gh[5][sl].copy()
        for q in np.flatnonzero((idx >= lo) & (idx < lo + m)):
            M11[idx[q] - lo] += w[q] * mat(info[q])[0]; fg1[idx[q] - lo] += w[q] * rhs[q]; ff[idx[q] - lo] += cst[q]
        args = (M11, mat(Gh[1][sl]), mat(Gh[2][sl]), fg1, Gh[4][sl], ff, m, (mat(pinfo[c])[0], prhs[c], pf[c]))
        plain, truth = marginalize_ref(*args), marginalize_ref(*args, jacobi=True)
        sc = max(np.linalg.norm(truth[0]), np.linalg.norm(mat(Gh[2])[f0 + m - 1]))
        errs.append((np.linalg.norm(mat(oi[c])[0] - truth[0]) / sc, np.linalg.norm(plain[0] - truth[0]) / sc))
        sc = max(np.linalg.norm(truth[1]), np.linalg.norm(Gh[4][f0 + m - 1]))
        errs.append((np.linalg.norm(orr[c] - truth[1]) / sc, np.linalg.norm(plain[1] - truth[1]) / sc))
        fs = abs(truth[2]) + np.sum(np.abs(ff)) + abs(pf[c])
        errs.append((abs(of[c] - truth[2]) / fs, abs(plain[2] - truth[2]) / fs))
    eg, ep = max(x[0] for x in errs), max(x[1] for x in errs)
    print(f"K8 with robust state priors: device worst {eg:.2e}, plain fp64 numpy worst {ep:.2e}")
    assert eg <= 50 * max(ep, 1e-13)
    # the reduced solve: chain 3 (30 states), a 1e8 I prior on x_0, robust priors on eliminated and kept states (the last among them)
    nf = 29
    G1 = [t[offs[3] - 3:offs[3] - 3 + nf] for t in G]
    Xc = X[offs[3]:offs[4]]
    kidx = np.array([2, 5, 5, 11, 20, 29, 29], dtype=np.int64)
    kinfo, krhs, kf, klin = moved_meas(kidx, Xc)
    kcode = np.array([1, 2, 0, 2, 1, 2, 1], dtype=np.int32)
    kk = np.where(kcode == 1, HUBER_K, CAUCHY_K)
    d = lambda a: _dev(torch, a)
    prior = (torch.eye(15, dtype=torch.float64, device="cuda") * 1e8).reshape(1, 225)
    z15, z1 = torch.zeros((1, 15), dtype=torch.float64, device="cuda"), torch.zeros(1, dtype=torch.float64, device="cuda")
    full = [t.clone() for t in G1]
    order, sp_off = csr(kidx, nf + 1)
    wi, wr, wf = factor.state_priors_robust(d(kcode[order]), d(kk[order]), d(kinfo[order]), d(krhs[order]), d(kf[order]))
    factor.state_priors_fold(nf + 1, d(sp_off), wi, wr, wf, G11=full[0], G22=full[2], g1=full[3], g2=full[4], f=full[5], n_chains=1)
    D, E, b = factor.chains_assemble(*full[:5], nf + 1, 0.0, prior, z15)
    x_full = factor.chain_solve(D, E, b).cpu().numpy()
    Dh, Eh, bh = mat(D.cpu().numpy()), mat(E.cpu().numpy()), b.cpu().numpy()
    A = np.zeros((15 * (nf + 1),) * 2)
    for q in range(nf + 1):
        A[15 * q:15 * q + 15, 15 * q:15 * q + 15] = Dh[q]
        if q < nf:
            A[15 * q:15 * q + 15, 15 * q + 15:15 * q + 30] = Eh[q]; A[15 * q + 15:15 * q + 30, 15 * q:15 * q + 15] = Eh[q].T
    xt, x64 = (v.reshape(-1, 15) for v in _dense_truth(A, bh.reshape(-1)))
    sp_all = _sp_dev(torch, kidx, kinfo, krhs, kf, klin)
    for m in (1, 6, 21, 29):
        info_m, r_m, f_m = factor.chain_marginalize(*G1, nf + 1, m, prior=(prior, z15, z1), state_priors=sp_all,
                                                    state_prior_loss=(d(kcode), d(kk)))
        sl = slice(m, nf)
        red = [t[sl].clone() for t in G1]
        keep = kidx >= m
        order, sp_off = csr(kidx[keep] - m, nf + 1 - m)
        wi, wr, wf = factor.state_priors_robust(d(kcode[keep][order]), d(kk[keep][order]), d(kinfo[keep][order]), d(krhs[keep][order]),
                                                d(kf[keep][order]))
        pi_m = info_m.clone()
        factor.state_priors_fold(nf + 1 - m, d(sp_off), wi, wr, wf, G11=red[0] if m < nf else None, G22=red[2] if m < nf else None,
                                 g1=red[3] if m < nf else None, g2=red[4] if m < nf else None, f=red[5] if m < nf else None,
                                 prior_info=pi_m, prior_rhs=r_m, prior_f=f_m, n_chains=1)
        Dr, Er, br = factor.chains_assemble(*red[:5], nf + 1 - m, 0.0, pi_m, r_m, n_chains=1)
        x_red = factor.chain_solve(Dr, Er, br).cpu().numpy()
        nt = np.linalg.norm(xt[m:])
        e64 = np.linalg.norm(x64[m:] - xt[m:]) / nt
        e_red, e_full = np.linalg.norm(x_red - xt[m:]) / nt, np.linalg.norm(x_full[m:] - xt[m:]) / nt
        print(f"m={m}: reduced {e_red:.2e}, full {e_full:.2e}, sequential fp64 {e64:.2e}")
        assert e_red <= 50 * max(e64, 1e-13) and e_full <= 50 * max(e64, 1e-13), (m, e_red, e_full, e64)


@pytest.mark.gpu
@pytest.mark.parametrize("poison", ["code", "k"])
def test_invalid_loss_on_the_device_is_isolated(cuda, oracle, monkeypatch, poison):
    """An unknown loss code or a NaN threshold that reaches the device (the entry's value checks bypassed) in chain 3 of 10 ends that
    chain NONFINITE with its input states; the other nine are bitwise the clean run."""
    from cpi_b200 import factor
    torch = cuda
    rng = np.random.default_rng(8)
    sizes = [5, 1, 12, 20, 8, 1, 30, 3, 16, 9]
    X, rec, L, offs, pri, _ = make_problem(oracle, 1, sizes, 11, large=True, with_prior=True)
    sp = add_outliers(_meas_priors(oracle, rng, X, offs, 3, "p"), 4, 0.3)
    loss = mixed_losses(len(sp[0]))
    clean = _device_lm(torch, 1, X, rec, L, offs, pri, sp, loss)
    q = int(np.flatnonzero((sp[0] >= offs[3]) & (sp[0] < offs[4]))[0])
    code, k = loss[0].copy(), loss[1].copy()
    if poison == "code":
        code[q] = 7
    else:
        code[q], k[q] = capi.LOSS_CAUCHY, np.nan
    monkeypatch.setattr(factor, "_loss_flags", lambda c, *a: [torch.zeros((), dtype=torch.bool, device=c.device)] * 3)
    Xb, cb, lb, sb, ib, tb = _device_lm(torch, 1, X, rec, L, offs, pri, sp, (code, k))
    assert sb[3] == capi.LM_NONFINITE and ib[3] == 0
    assert np.array_equal(Xb[offs[3]:offs[4]], X[offs[3]:offs[4]])
    Xs, cost, lam, st, it, tr = clean
    assert not np.any(st == capi.LM_NONFINITE)
    for c in range(len(sizes)):
        if c == 3:
            continue
        part = slice(offs[c], offs[c + 1])
        assert np.array_equal(Xb[part], Xs[part]) and cb[c] == cost[c] and lb[c] == lam[c] and sb[c] == st[c] and ib[c] == it[c], c


@pytest.mark.gpu
def test_fixed_lag_smoother_with_cauchy_fixes(cuda, oracle):
    """test_state_priors.py::test_fixed_lag_smoother_with_position_fixes with Cauchy fixes (k = 2.3849), every 7th fix a 1 m outlier:
    chains_lm reweights them every round; the oldest state's fix is moved to the states it is marginalised at and enters K8 with its
    weight frozen there.  The same loop in numpy on 3 sequences agrees in retract coordinates."""
    from cpi_b200 import factor, preint
    torch = cuda
    ns, K, W, lam = 8, 50, 12, 1e-5
    S, L = synth.make_windows(ns * (K - 1), 20, rate=200.0, first_window=96000, special=False)
    rec = preint.preintegrate_host(1, S, L, synth.SIGMAS, 0, ns=20).reshape(ns, K - 1, -1)
    L = L.reshape(ns, K - 1, 13)
    rng = np.random.default_rng(24)
    truth = np.stack([synth.make_states(rec[s], L[s], 1, perturb=False) for s in range(ns)])
    fixes, n = {}, 0
    for s in range(ns):
        for k in range(5, K, 5):
            Wm = np.zeros((15, 15)); Wm[12:15, 12:15] = np.eye(3) * 1e4
            xb = truth[s, k].copy(); xb[13:16] += rng.normal(0, 0.01, 3)
            if n % 7 == 3:
                xb[13:16] += 1.0 / np.sqrt(3.0)
            fixes[(s, k)] = (Wm, xb)
            n += 1
    X0 = truth[:, :W].copy()
    X0[:, 1:, 7:10] += rng.normal(0, 1e-3, (ns, W - 1, 3)); X0[:, 1:, 13:16] += rng.normal(0, 1e-3, (ns, W - 1, 3))
    X0[:, 1:, 4:7] += rng.normal(0, 1e-5, (ns, W - 1, 3))
    dR, dL = _dev(torch, rec), _dev(torch, L)
    info0 = np.eye(15) * 1e8
    prior = (_dev(torch, np.tile(vec(info0[None]), (ns, 1))), torch.zeros((ns, 15), dtype=torch.float64, device="cuda"),
             torch.zeros(ns, dtype=torch.float64, device="cuda"), _dev(torch, X0[:, 0].copy()))
    Xw = _dev(torch, X0)
    first = torch.arange(ns, device="cuda") * (W + 1)
    cauchy = lambda M: (torch.full((M,), capi.LOSS_CAUCHY, dtype=torch.int32, device="cuda"),
                        torch.full((M,), CAUCHY_K, dtype=torch.float64, device="cuda"))

    def window_fixes(t0, n):
        idx, info, lin = [], [], []
        for s in range(ns):
            for j in range(n):
                if (s, t0 + j) in fixes:
                    Wm, xb = fixes[(s, t0 + j)]
                    idx.append(s * (W + 1) + j); info.append(vec(Wm[None])[0]); lin.append(xb)
        M = len(idx)
        return np.array(idx, dtype=np.int64), np.array(info).reshape(M, 225), np.zeros((M, 15)), np.zeros(M), np.array(lin).reshape(M, 16)

    for t in range(W, K):
        xn = factor.predict_state(1, Xw[:, -1].contiguous(), dR[:, t - 1].contiguous(), dL[:, t - 1].contiguous())
        Xw = torch.cat([Xw, xn[:, None]], dim=1)
        t0 = t - W
        sp = window_fixes(t0, W + 1)
        new, cost, _, st, _, _ = factor.chains_lm(1, Xw.reshape(-1, 16).contiguous(), dR[:, t0:t].reshape(-1, rec.shape[-1]).contiguous(),
                                                  dL[:, t0:t].reshape(-1, 13).contiguous(), W + 1, prior=prior, lam=lam,
                                                  state_priors=_sp_dev(torch, *sp), state_prior_loss=cauchy(len(sp[0])))
        Xw = new.view(ns, W + 1, 16)
        e, H1, H2 = factor.factor_eval(1, Xw.reshape(-1, 16), dR[:, t0].contiguous(), dL[:, t0].contiguous(), idx_i=first, idx_j=first + 1)
        G = factor.factor_hessian(1, dR[:, t0].contiguous(), e, H1, H2)
        r_p, f_p = factor.prior_at(prior[0], prior[1], prior[2], prior[3], Xw[:, 0].contiguous())
        i0, f_info, f_rhs, f_f, f_lin = window_fixes(t0, 1)
        sidx = torch.from_numpy(i0 // (W + 1) * 2).cuda()
        x_at = Xw.reshape(-1, 16)[torch.from_numpy(i0).cuda()]
        rr, ff = factor.prior_at(_dev(torch, f_info), _dev(torch, f_rhs), _dev(torch, f_f), _dev(torch, f_lin), x_at)
        mi, mr, mf = factor.chain_marginalize(*G, 2, 1, prior=(prior[0], r_p, f_p), n_chains=ns,
                                              state_priors=(sidx, _dev(torch, f_info), rr, ff, x_at), state_prior_loss=cauchy(len(i0)))
        prior = (mi, mr, mf, Xw[:, 1].contiguous())
        Xw = Xw[:, 1:].contiguous()
    Xg = Xw.cpu().numpy()
    assert np.all(np.isfinite(Xg)) and np.all(st.cpu().numpy() == capi.LM_CONVERGED)
    worst = 0.0
    for s in (0, 3, 7):
        Xs, pr = X0[s].copy(), (info0, np.zeros(15), 0.0, X0[s, 0].copy())
        for t in range(W, K):
            Xs = np.concatenate([Xs, oracle.predict_state(1, Xs[-1:], rec[s, t - 1:t], L[s, t - 1:t])])
            t0 = t - W
            sps = [(j, vec(fixes[(s, t0 + j)][0][None])[0], np.zeros(15), 0.0, fixes[(s, t0 + j)][1], capi.LOSS_CAUCHY, CAUCHY_K)
                   for j in range(W + 1) if (s, t0 + j) in fixes]
            Xs = np_lm_rb(oracle, 1, Xs, rec[s, t0:t], L[s, t0:t], pr, sps, lam)[0]
            info, rhs, f0, x_lin = pr
            e, H1, H2 = oracle.factor_eval(1, Xs[:2], rec[s, t0:t0 + 1], L[s, t0:t0 + 1])
            G = [g.copy() for g in _np_hessian(rec[s, t0:t0 + 1], e, H1, H2)]
            rhs_p, f_p = prior_at_ref(vec(info[None]), rhs[None], np.array([f0]), x_lin[None], Xs[:1])
            if sps and sps[0][0] == 0:
                _, fi, frhs, ff0, fl, _, _ = sps[0]
                rr, fq = prior_at_ref(fi[None], frhs[None], np.array([ff0]), fl[None], Xs[:1])
                wq, cq = np_loss(capi.LOSS_CAUCHY, CAUCHY_K, fq)
                G[0][0] = G[0][0] + wq[0] * mat(fi)[0]; G[3][0] = G[3][0] + wq[0] * rr[0]; G[5][0] = G[5][0] + cq[0]
            Lam, eta, fm = marginalize_ref(*G, 1, (info, rhs_p[0], f_p[0]), jacobi=True)
            pr = (Lam, eta, fm, Xs[1].copy())
            Xs = Xs[1:]
        worst = max(worst, np.linalg.norm(local(Xs, Xg[s])) / np.linalg.norm(Xs[:, 4:16]))
    print(f"fixed-lag smoother with Cauchy fixes and outliers vs numpy: worst relative difference {worst:.2e} (retract coordinates)")
    assert worst <= 1e-9
