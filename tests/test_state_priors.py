"""Priors on any state of many IMU chains (cpi_imu_state_priors_fold, factor.state_priors_fold and the state_priors argument of
factor.chains_lm_step / chains_lm / chain_marginalize; DESIGN.md section 3g).

GTSAM is not in the reference tree, so parity with its PriorFactor is UNPINNED.  The reference is ``fold_ref`` below, the fold rule in
numpy: on the CPU it is pinned against the dense normal equations with every prior added on its own state; the GPU tests compare the
kernel with it bit for bit and the solver entry points with numpy statements of the whole system."""
import ctypes

import numpy as np
import pytest

from cpi_b200 import capi, synth
from test_chains_lm import DEFAULTS, dev_prior, make_problem, np_cost, well_posed
from test_marginalize import (_dense_truth, _np_hessian, dense_head, local, marginalize_ref, mat, prior_at_ref, random_factors,
                              random_prior, vec)

P = lambda a: ctypes.c_void_p(a.ctypes.data)


# ------------------------------------------------------------------------------------------------------------------
# numpy statements
# ------------------------------------------------------------------------------------------------------------------

def csr(idx, N):
    """The stable sort of the priors by state and the per-state CSR offsets [N+1]."""
    order = np.argsort(idx, kind="stable")
    return order, np.searchsorted(idx[order], np.arange(N + 1), side="left").astype(np.int64)


def fold_ref(offs, sp_off, info, rhs, f, blocks, chain_prior, f_only=False):
    """The fold rule, priors already sorted by state (info [M,225], rhs [M,15], f [M] or None), added one after the other in CSR order
    into copies of blocks = (G11, G22 [nf,225], g1, g2 [nf,15], f [nf]) and chain_prior = (info [C,225], rhs [C,15], f [C]).
    f_only: only f is added (into blocks[4] / chain_prior[2])."""
    G11, G22, g1, g2, fk = (None if a is None else np.array(a, dtype=np.float64) for a in blocks)
    pi, pr, pf = (None if a is None else np.array(a, dtype=np.float64) for a in chain_prior)
    C = len(offs) - 1
    for c in range(C):
        lo, hi = int(offs[c]), int(offs[c + 1])
        for k in range(lo, hi):
            if k < hi - 1:
                I, r, fs, j = G11, g1, fk, k - c
            elif hi - lo >= 2:
                I, r, fs, j = G22, g2, fk, k - 1 - c
            else:
                I, r, fs, j = pi, pr, pf, c
            for q in range(int(sp_off[k]), int(sp_off[k + 1])):
                if not f_only:
                    I[j] = I[j] + info[q]
                    r[j] = r[j] + rhs[q]
                if f is not None and fs is not None:
                    fs[j] = fs[j] + f[q]
    return (G11, G22, g1, g2, fk), (pi, pr, pf)


def dense_chain(G11, G12, G22, g1, g2, f, prior):
    """Dense (A, b, F) of one chain from [k,225]-form blocks and a prior (info [225], rhs [15], f) on its first state."""
    n = len(G11)
    return dense_head(mat(G11), mat(G12), mat(G22), g1, g2, f, n, (mat(prior[0])[0], prior[1], prior[2]))


def random_layout(rng, sizes):
    offs = np.r_[0, np.cumsum(sizes)].astype(np.int64)
    C, N = len(sizes), int(offs[-1])
    G = random_factors(rng, N - C)
    blocks = (vec(G[0]), vec(G[1]), vec(G[2]), G[3], G[4], G[5])
    pri = [random_prior(rng) for _ in range(C)]
    chain_prior = (np.stack([vec(p[0][None])[0] for p in pri]), np.stack([p[1] for p in pri]), np.array([p[2] for p in pri]))
    return offs, blocks, chain_prior


def random_state_priors(rng, offs, extra=()):
    """Priors on the first, a middle and the last state of every chain, two on some states, plus `extra` states; shuffled."""
    idx = []
    for c in range(len(offs) - 1):
        lo, hi = int(offs[c]), int(offs[c + 1])
        idx += [lo, hi - 1, (lo + hi) // 2]
        if c % 3 == 0:
            idx.append(hi - 1)
    idx = np.array(idx + list(extra), dtype=np.int64)
    rng.shuffle(idx)
    pr = [random_prior(rng, scale=(1e-1, 1e-2, 1.0, 1e-1, 1.0)) for _ in idx]
    return idx, np.stack([vec(p[0][None])[0] for p in pr]), np.stack([p[1] for p in pr]), np.array([p[2] for p in pr])


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", [0, 1])
def test_fold_is_the_dense_system_with_priors_on_their_states(seed):
    """Ragged chains of 1-9 states (single-state chains among them), priors on first, middle and last states and several on one
    state: the dense system of the folded blocks equals the dense system of the IMU factors plus every prior on its own state."""
    rng = np.random.default_rng(seed)
    sizes = np.r_[1, 2, 9, 1, rng.integers(1, 10, size=12)]
    offs, blocks, chain_prior = random_layout(rng, sizes)
    idx, info, rhs, f = random_state_priors(rng, offs)
    order, sp_off = csr(idx, int(offs[-1]))
    G11, G12, G22, g1, g2, fk = blocks
    (F11, F22, fg1, fg2, ff), (fpi, fpr, fpf) = fold_ref(offs, sp_off, info[order], rhs[order], f[order], (G11, G22, g1, g2, fk), chain_prior)
    assert np.array_equal(G12, blocks[1])
    for c in range(len(sizes)):
        lo, hi, f0 = int(offs[c]), int(offs[c + 1]), int(offs[c] - c)
        s = slice(f0, f0 + hi - lo - 1)
        A, b, F = dense_chain(F11[s], G12[s], F22[s], fg1[s], fg2[s], ff[s], (fpi[c], fpr[c], fpf[c]))
        A0, b0, F0 = dense_chain(G11[s], G12[s], G22[s], g1[s], g2[s], fk[s], (chain_prior[0][c], chain_prior[1][c], chain_prior[2][c]))
        for q in np.flatnonzero((idx >= lo) & (idx < hi)):
            k = slice(15 * (idx[q] - lo), 15 * (idx[q] - lo) + 15)
            A0[k, k] += mat(info[q])[0]; b0[k] += rhs[q]; F0 += f[q]
        sc = np.abs(A0).max()
        assert np.allclose(A, A0, rtol=0, atol=1e-14 * sc) and np.allclose(b, b0, rtol=1e-13, atol=1e-13 * np.abs(b0).max()), c
        assert abs(F - F0) <= 1e-13 * (abs(F0) + np.abs(f).sum()), c


def test_argument_validation_without_gpu():
    import torch
    from cpi_b200 import factor
    lib = capi.load()
    buf = np.zeros(8 * 225)
    p = P(buf)
    # cpi_imu_state_priors_fold(n_chains, offs, uniform, sp_offsets, sp_info, sp_rhs, sp_f, G11, G22, g1, g2, f, pi, pr, pf, stream)
    fold = lambda n, o, u, *a: lib.cpi_imu_state_priors_fold(n, o, u, *a, None)
    ga = [p, p, p, p] + [p] * 5 + [p, p, p]
    assert fold(-1, None, 3, *ga) == -1 and b"negative" in lib.cpi_last_error()
    assert fold(2, None, 0, *ga) == -1 and b"chain_uniform" in lib.cpi_last_error()
    bad = list(ga); bad[0] = None
    assert fold(2, None, 3, *bad) == -1 and b"sp_offsets" in lib.cpi_last_error()
    bad = list(ga); bad[2] = None
    assert fold(2, None, 3, *bad) == -1 and b"both" in lib.cpi_last_error()
    bad = list(ga); bad[1] = bad[2] = bad[3] = None
    assert fold(2, None, 3, *bad) == -1 and b"sp_f" in lib.cpi_last_error()
    for k in (9, 10, 11):                                          # single-state chains need the chain-prior targets
        bad = list(ga); bad[k] = None
        assert fold(2, None, 1, *bad) == -1 and b"single-state" in lib.cpi_last_error(), k
    assert fold(0, None, 1, *[None] * 12) == 0
    # the Python layer raises before the device is touched
    N = 12
    X, rec, lin = torch.zeros(N, 16, dtype=torch.float64), torch.zeros(N - 3, 290, dtype=torch.float64), torch.zeros(N - 3, 13, dtype=torch.float64)
    G = [torch.zeros(N - 3, k, dtype=torch.float64) for k in (225, 225, 225, 15, 15, 1)]
    good = lambda M=2: (torch.tensor([0, 5][:M], dtype=torch.int64), torch.zeros(M, 225, dtype=torch.float64), None, None,
                        torch.zeros(M, 16, dtype=torch.float64))
    calls = (lambda sp: factor.chains_lm_step(1, X, rec, lin, 4, state_priors=sp), lambda sp: factor.chains_lm(1, X, rec, lin, 4, state_priors=sp),
             lambda sp: factor.chain_marginalize(*G, 4, 1, state_priors=sp))
    for call in calls:
        i, info, r, f, l = good()
        for bad, exc, msg in (((i, info), ValueError, "state_priors is"), ((i.int(), info, r, f, l), ValueError, "int64"),
                              ((i.double(), info, r, f, l), ValueError, "int64"), ((i, info[:, :200], r, f, l), ValueError, "info"),
                              ((i, info, torch.zeros(2, 14, dtype=torch.float64), f, l), ValueError, "rhs"),
                              ((i, info, r, torch.zeros(3, dtype=torch.float64), l), ValueError, "f"), ((i, info, r, f, l[:1]), ValueError, "lin"),
                              ((i, info.float(), r, f, l), ValueError, "float64"),
                              ((torch.tensor([0, 12]), info, r, f, l), IndexError, "out of range"),
                              ((torch.tensor([-1, 3]), info, r, f, l), IndexError, "out of range"),
                              ((i, info, r, f, l), ValueError, "CUDA")):
            with pytest.raises(exc, match=msg):
                call(bad)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------

def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _host(t):
    return None if t is None else t.cpu().numpy()


@pytest.mark.gpu
def test_fold_kernel_is_bitwise_the_numpy_fold(cuda):
    """The kernel against fold_ref in CSR order: ragged (device-resident offsets) and uniform layouts, single-state chains, the fold
    and the f-only fold; two calls give the same bits."""
    from cpi_b200 import factor
    torch = cuda
    rng = np.random.default_rng(5)
    for sizes in (np.r_[1, 2, 9, 1, 40, rng.integers(1, 70, size=60)], np.full(50, 7), np.full(13, 1)):
        offs, blocks, chain_prior = random_layout(rng, sizes)
        idx, info, rhs, f = random_state_priors(rng, offs, extra=rng.integers(0, offs[-1], size=40))
        N = int(offs[-1])
        order, sp_off = csr(idx, N)
        info, rhs, f = info[order], rhs[order], f[order]
        G11, G12, G22, g1, g2, fk = blocks
        layouts = [_dev(torch, offs)] + ([int(sizes[0])] if np.all(sizes == sizes[0]) else [])
        for layout in layouts:
            for f_only in (False, True):
                ref_b, ref_p = fold_ref(offs, sp_off, info, rhs, f, (G11, G22, g1, g2, fk), chain_prior, f_only=f_only)
                outs = []
                for _ in range(2):
                    tb = [_dev(torch, a) for a in (G11, G22, g1, g2, fk)]
                    tp = [_dev(torch, a) for a in chain_prior]
                    factor.state_priors_fold(layout, _dev(torch, sp_off), None if f_only else _dev(torch, info), None if f_only else _dev(torch, rhs),
                                             _dev(torch, f), *tb, *tp, n_chains=len(sizes))
                    outs.append([_host(t) for t in tb + tp])
                for a, b in zip(outs[0], outs[1]):
                    assert np.array_equal(a, b)
                for got, want in zip(outs[0], list(ref_b) + list(ref_p)):
                    assert np.array_equal(got, want), (sizes[:4], f_only)


def _sp_dev(torch, idx, info, rhs, f, lin):
    return (_dev(torch, np.asarray(idx, dtype=np.int64)), _dev(torch, info), None if rhs is None else _dev(torch, rhs),
            None if f is None else _dev(torch, f), _dev(torch, lin))


def _meas_priors(orc, rng, X, offs, every, kind, truth=None, sigma=0.01):
    """Measurement priors (info W, rhs 0, f 0, lin x_bar) every `every`-th state of each chain from its second: kind 'p' (position),
    'v' (velocity), 'mixed' (alternately position, velocity and a full 15-dof prior).  x_bar: truth (or X) with noise."""
    idx, info, lin = [], [], []
    base = X if truth is None else truth
    for c in range(len(offs) - 1):
        for j, k in enumerate(range(int(offs[c]) + 1, int(offs[c + 1]), every)):
            kk = kind if kind != "mixed" else ("p", "v", "full")[(c + j) % 3]
            W = np.zeros((15, 15))
            if kk == "p":
                W[12:15, 12:15] = np.eye(3) / sigma ** 2
            elif kk == "v":
                W[6:9, 6:9] = np.eye(3) / sigma ** 2
            else:
                W = np.diag(np.repeat([1e4, 1e6, 1e2, 1e4, 1e2], 3))
            xb = base[k].copy()
            xb[13:16] += rng.normal(0, sigma, 3)
            idx.append(k); info.append(vec(W[None])[0]); lin.append(xb)
    M = len(idx)
    return np.array(idx, dtype=np.int64), np.array(info).reshape(M, 225), np.zeros((M, 15)), np.zeros(M), np.array(lin).reshape(M, 16)


@pytest.mark.gpu
def test_no_priors_and_empty_list_are_bitwise_the_plain_calls(cuda, oracle):
    from cpi_b200 import factor
    torch = cuda
    X, rec, L, offs, pri, _ = make_problem(oracle, 1, [1, 4, 9, 2, 30, 17], 7, with_prior=True)
    a = (_dev(torch, X), _dev(torch, rec), _dev(torch, L), _dev(torch, offs))
    empty = (torch.zeros(0, dtype=torch.int64, device="cuda"), torch.zeros((0, 225), dtype=torch.float64, device="cuda"), None, None,
             torch.zeros((0, 16), dtype=torch.float64, device="cuda"))
    for fn in (factor.chains_lm_step, factor.chains_lm):
        ref = fn(1, *a, prior=dev_prior(torch, pri))
        for sp in (None, empty):
            got = fn(1, *a, prior=dev_prior(torch, pri), state_priors=sp)
            assert all(torch.equal(u, v) for u, v in zip(ref, got)), fn.__name__
    nm = _dev(torch, np.array([0, 2, 5, 1, 29, 3]))
    e, H1, H2 = factor.factor_eval(1, a[0], a[1], a[2], *_chain_idx(torch, offs))
    G = factor.factor_hessian(1, a[1], e, H1, H2)
    pr = dev_prior(torch, pri)[:3]
    ref = factor.chain_marginalize(*G, a[3], nm, prior=pr)
    for sp in (None, empty):
        got = factor.chain_marginalize(*G, a[3], nm, prior=pr, state_priors=sp)
        assert all(torch.equal(u, v) for u, v in zip(ref, got))


def _chain_idx(torch, offs):
    C = len(offs) - 1
    cof = np.repeat(np.arange(C), np.diff(offs) - 1)
    ii = np.arange(len(cof)) + cof
    return _dev(torch, ii), _dev(torch, ii + 1)


def _np_system(orc, model, Xc, r, l, prior, sps, blocks=None):
    """Dense (A, b, cost) of one chain at Xc: IMU factors (numpy blocks, or the given [k,225]-form ones), the chain prior moved to
    Xc[0], the state priors (local index, info [225], rhs, f, lin) moved to their states."""
    S = len(Xc)
    if blocks is not None:
        G = (mat(blocks[0]), mat(blocks[1]), mat(blocks[2]), blocks[3], blocks[4], blocks[5])
    elif S > 1:
        e, H1, H2 = orc.factor_eval(model, Xc, r, l)
        G = _np_hessian(r, e, H1, H2)
    else:
        G = (np.zeros((0, 15, 15)),) * 3 + (np.zeros((0, 15)),) * 2 + (np.zeros(0),)
    if prior is None:
        pi, pr, pf = np.zeros((15, 15)), np.zeros(15), 0.0
    else:
        rr, ff = prior_at_ref(vec(prior[0][None]), prior[1][None], np.array([prior[2]]), prior[3][None], Xc[:1])
        pi, pr, pf = prior[0], rr[0], ff[0]
    A, b, _ = dense_head(G[0], G[1], G[2], G[3], G[4], G[5], S - 1, (pi, pr, 0.0))
    cost = float(np.sum(G[5]) + pf)
    for k, info, rhs, f, lin in sps:
        rr, ff = prior_at_ref(info[None], rhs[None], np.array([f]), lin[None], Xc[k:k + 1])
        s = slice(15 * k, 15 * k + 15)
        A[s, s] += mat(info)[0]; b[s] += rr[0]; cost += ff[0]
    return A, b, cost


def _np_sp_cost(orc, model, Xc, r, l, prior, sps):
    c = float(np.sum(np_cost(orc, model, Xc, r, l)))
    if prior is not None:
        c += prior_at_ref(vec(prior[0][None]), prior[1][None], np.array([prior[2]]), prior[3][None], Xc[:1])[1][0]
    for k, info, rhs, f, lin in sps:
        c += prior_at_ref(info[None], rhs[None], np.array([f]), lin[None], Xc[k:k + 1])[1][0]
    return c


def np_lm_sp(orc, model, X, rec, lin, prior, sps, lam=1e-5, p=DEFAULTS, max_rounds=200):
    """test_chains_lm.np_lm with state priors: the same rule on the dense system of _np_system."""
    S = len(X)
    X = X.copy()
    status, it, tries, cost, trace = 0, 0, 0, 0.0, []
    while status == 0 and tries < max_rounds:
        A, b, cur = _np_system(orc, model, X, rec, lin, prior, sps)
        Ad = A.copy()
        Ad[np.diag_indices_from(A)] += lam * np.clip(np.diag(A), 1e-6, 1e32)
        s = 1.0 / np.sqrt(np.diag(Ad))
        dx = np.linalg.solve(Ad * s[:, None] * s[None, :], b * s) * s
        Xn = orc.retract(X, dx.reshape(S, 15))
        new = _np_sp_cost(orc, model, Xn, rec, lin, prior, sps)
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


def _per_chain_sps(offs, idx, info, rhs, f, lin):
    out = [[] for _ in range(len(offs) - 1)]
    for q in range(len(idx)):
        c = int(np.searchsorted(offs, idx[q], side="right") - 1)
        out[c].append((int(idx[q] - offs[c]), info[q], rhs[q], f[q], lin[q]))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_lm_step_matches_dense_gauss_newton(cuda, oracle, model):
    """chains_lm_step with state priors (position, velocity, full; single-state chains carrying priors, without a chain prior on
    some) against the dense damped step of the same system: within 50x the distance of a plain fp64 dense solve to the refined truth
    (floor 1e-13), the chain solves' gate of test_marginalize.py; the cost before the step to 1e-12."""
    from cpi_b200 import factor
    torch = cuda
    rng = np.random.default_rng(40 + model)
    sizes = [1, 4, 9, 2, 30, 17, 1, 12]
    for with_prior in (True, False):
        X, rec, L, offs, pri, per = make_problem(oracle, model, sizes, 3 + model, large=True, with_prior=with_prior)
        idx, info, rhs, f, lin = _meas_priors(oracle, rng, X, offs, 3, "mixed")
        idx = np.r_[idx, 0, int(offs[6]), int(offs[6])]               # single-state chains 0 and 6, two priors on one of them
        extra = np.diag(np.repeat([1e4, 1e6, 1e2, 1e4, 1e2], 3))
        info = np.r_[info, np.tile(vec(extra[None]), (3, 1))]
        rhs = np.r_[rhs, rng.normal(size=(3, 15))]; f = np.r_[f, [0.5, 1.0, 2.0]]
        lin = np.r_[lin, X[[0, offs[6], offs[6]]]]
        lin[-3:, 13:16] += 0.01
        if not with_prior:                                          # every chain anchored: a full prior on each first state
            firsts = offs[:-1]
            idx = np.r_[idx, firsts]; info = np.r_[info, np.tile(vec(extra[None]), (len(firsts), 1))]
            rhs = np.r_[rhs, np.zeros((len(firsts), 15))]; f = np.r_[f, np.zeros(len(firsts))]; lin = np.r_[lin, X[firsts]]
        lam = 1e-5
        dX, dR, dL = _dev(torch, X), _dev(torch, rec), _dev(torch, L)
        new, dx, cost = factor.chains_lm_step(model, dX, dR, dL, _dev(torch, offs), prior=dev_prior(torch, pri), lam=lam,
                                              state_priors=_sp_dev(torch, idx, info, rhs, f, lin))
        dx, cost = dx.cpu().numpy(), cost.cpu().numpy()
        e, H1, H2 = factor.factor_eval(model, dX, dR, dL, *_chain_idx(torch, offs))   # the device's own blocks: the solve is what is compared
        Gh = [t.cpu().numpy() for t in factor.factor_hessian(model, dR, e, H1, H2)]
        sps = _per_chain_sps(offs, idx, info, rhs, f, lin)
        for c, (Xc, r, l) in enumerate(per):
            f0, S = int(offs[c] - c), len(Xc)
            blk = [g[f0:f0 + S - 1] for g in Gh]
            A, b, cur = _np_system(oracle, model, Xc, r, l, None if pri is None else pri[c], sps[c], blocks=blk)
            A[np.diag_indices_from(A)] += lam * np.clip(np.diag(A), 1e-6, 1e32)
            xt, x64 = _dense_truth(A, b)
            dd = dx[offs[c]:offs[c + 1]].reshape(-1)
            nt = np.linalg.norm(xt)
            e_dev, e64 = np.linalg.norm(dd - xt) / nt, np.linalg.norm(x64 - xt) / nt
            assert e_dev <= 50 * max(e64, 1e-13), (with_prior, c, e_dev, e64)
            assert abs(cost[c] - cur) <= 1e-10 * max(abs(cur), 1.0), (with_prior, c, cost[c], cur)


def _device_lm(torch, model, X, rec, L, offs, pri, sp, **kw):
    from cpi_b200 import factor
    out = factor.chains_lm(model, _dev(torch, X), _dev(torch, rec), _dev(torch, L), _dev(torch, offs), prior=dev_prior(torch, pri),
                           state_priors=None if sp is None else _sp_dev(torch, *sp), **kw)
    return [t.cpu().numpy() for t in out]


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_lm_matches_numpy(cuda, oracle, model):
    """chains_lm with position, velocity and mixed state priors on ragged chains against np_lm_sp: identical accept / reject
    sequences, final lambda, status and counters (no rho within 1e-6 of the threshold), final states close in retract coordinates."""
    torch = cuda
    rng = np.random.default_rng(60 + model)
    sizes = np.r_[1, 25, rng.integers(1, 26, size=10)]
    worst = 0.0
    for case, (kind, large, with_prior) in enumerate((("p", False, True), ("v", True, True), ("mixed", True, False))):
        X, rec, L, offs, pri, per = make_problem(oracle, model, sizes, 200 * model + case, large=large, with_prior=with_prior,
                                                 first_window=80000 + 5000 * case)
        sp = _meas_priors(oracle, rng, X, offs, 4, kind)
        if not with_prior:                                          # anchor every chain on its first state through a state prior
            firsts = offs[:-1]
            W = vec(np.diag(np.repeat([1e4, 1e6, 1e2, 1e4, 1e2], 3))[None])
            sp = (np.r_[sp[0], firsts], np.r_[sp[1], np.tile(W, (len(firsts), 1))], np.r_[sp[2], np.zeros((len(firsts), 15))],
                  np.r_[sp[3], np.zeros(len(firsts))], np.r_[sp[4], X[firsts]])
        sps = _per_chain_sps(offs, *sp)
        ref = [np_lm_sp(oracle, model, Xc, r, l, None if pri is None else pri[c], sps[c]) for c, (Xc, r, l) in enumerate(per)]
        for o in ref:
            well_posed(o[6])
        R = max(o[5] for o in ref)
        seq = [_device_lm(torch, model, X, rec, L, offs, pri, sp, max_rounds=r, check_every=0) for r in range(1, R + 1)]
        Xs, cost, lam, st, it, tr = _device_lm(torch, model, X, rec, L, offs, pri, sp)
        for c, o in enumerate(ref):
            dev_acc = [bool(seq[r][4][c] > (seq[r - 1][4][c] if r else 0)) for r in range(o[5])]
            assert dev_acc == [t[0] for t in o[6]], (case, c, dev_acc, o[6])
            assert (lam[c], st[c], it[c], tr[c]) == (o[2], o[3], o[4], o[5]), (case, c, (lam[c], st[c], it[c], tr[c]), o[2:6])
            Xd = Xs[offs[c]:offs[c + 1]]
            worst = max(worst, np.linalg.norm(local(o[0], Xd)) / max(np.linalg.norm(o[0][:, 4:16]), 1e-300))
            assert cost[c] <= o[6][0][3] * (1 + 1e-12)
        print(f"model {model} case {kind}: rounds {R}, statuses {np.bincount(st, minlength=5)}")
    print(f"model {model}: worst final-state distance to numpy (retract coordinates, relative) {worst:.2e}")
    assert worst <= (1e-9 if model == 1 else 2e-7)


@pytest.mark.gpu
def test_marginalize_with_state_priors(cuda, oracle):
    """K8 with priors on eliminated states equals marginalize_ref with them added to G11 / g1 / f; priors on kept states (the last
    state with m = S_c - 1 among them) are not folded.  The reduced solve plus the remaining priors equals the full solve's tail."""
    from cpi_b200 import factor
    torch = cuda
    rng = np.random.default_rng(77)
    sizes = np.r_[2, 9, 1, 30, rng.integers(1, 31, size=20)]
    X, rec, L, offs, _, _ = make_problem(oracle, 1, sizes, 9, first_window=90000)
    C, N = len(sizes), int(offs[-1])
    nm = np.array([rng.integers(0, s) for s in sizes], dtype=np.int64)
    nm[0] = 1; nm[1] = 8                                            # m = S_c - 1: the last state is kept and carries priors
    dX, dR, dL, dO = (_dev(torch, a) for a in (X, rec, L, offs))
    e, H1, H2 = factor.factor_eval(1, dX, dR, dL, *_chain_idx(torch, offs))
    G = factor.factor_hessian(1, dR, e, H1, H2)
    Gh = [t.cpu().numpy() for t in G]
    idx, info, rhs, f = random_state_priors(rng, offs, extra=offs[:-1])
    lin = X[idx]
    pri = [random_prior(rng, scale=(1e-3, 1e-4, 1e-2, 1e-3, 1e-2)) for _ in range(C)]
    pinfo = np.stack([vec(p[0][None])[0] for p in pri]); prhs = np.stack([p[1] for p in pri]); pf = np.array([p[2] for p in pri])
    oi, orr, of = (t.cpu().numpy() for t in factor.chain_marginalize(*G, dO, _dev(torch, nm), prior=tuple(_dev(torch, a) for a in (pinfo, prhs, pf)),
                                                                      state_priors=_sp_dev(torch, idx, info, rhs, f, lin)))
    errs = []
    for c in range(C):
        m, f0, lo = int(nm[c]), int(offs[c] - c), int(offs[c])
        if m == 0:
            assert np.array_equal(oi[c], pinfo[c]) and np.array_equal(orr[c], prhs[c]) and of[c] == pf[c]
            continue
        sl = slice(f0, f0 + m)
        M11, fg1, ff = mat(Gh[0][sl]).copy(), Gh[3][sl].copy(), Gh[5][sl].copy()
        for q in np.flatnonzero((idx >= lo) & (idx < lo + m)):
            M11[idx[q] - lo] += mat(info[q])[0]; fg1[idx[q] - lo] += rhs[q]; ff[idx[q] - lo] += f[q]
        args = (M11, mat(Gh[1][sl]), mat(Gh[2][sl]), fg1, Gh[4][sl], ff, m, (mat(pinfo[c])[0], prhs[c], pf[c]))
        plain, truth = marginalize_ref(*args), marginalize_ref(*args, jacobi=True)
        sc = max(np.linalg.norm(truth[0]), np.linalg.norm(mat(Gh[2])[f0 + m - 1]))
        errs.append((np.linalg.norm(mat(oi[c])[0] - truth[0]) / sc, np.linalg.norm(plain[0] - truth[0]) / sc, c))
        sc = max(np.linalg.norm(truth[1]), np.linalg.norm(Gh[4][f0 + m - 1]))
        errs.append((np.linalg.norm(orr[c] - truth[1]) / sc, np.linalg.norm(plain[1] - truth[1]) / sc, c))
        fs = abs(truth[2]) + np.sum(np.abs(ff)) + abs(pf[c])
        errs.append((abs(of[c] - truth[2]) / fs, abs(plain[2] - truth[2]) / fs, c))
    eg, ep = max(x[0] for x in errs), max(x[1] for x in errs)
    print(f"K8 with state priors: device worst {eg:.2e}, plain fp64 numpy worst {ep:.2e}")
    assert eg <= 50 * max(ep, 1e-13)
    # the reduced solve: one chain of 40 states, a 1e8 I prior on x_0, priors on eliminated and kept states (the last among them)
    nf = 29
    G1 = [t[offs[3] - 3:offs[3] - 3 + nf] for t in G]               # chain 3 (30 states)
    Xc = X[offs[3]:offs[4]]
    kidx = np.array([2, 5, 5, 11, 20, 29, 29], dtype=np.int64)
    kp = [random_prior(rng, scale=(1e-2, 1e-3, 1e-1, 1e-2, 1e-1)) for _ in kidx]
    kinfo, krhs, kf = np.stack([vec(p[0][None])[0] for p in kp]), np.stack([p[1] for p in kp]), np.array([p[2] for p in kp])
    prior = (torch.eye(15, dtype=torch.float64, device="cuda") * 1e8).reshape(1, 225)
    z15, z1 = torch.zeros((1, 15), dtype=torch.float64, device="cuda"), torch.zeros(1, dtype=torch.float64, device="cuda")
    full = [t.clone() for t in G1]
    order, sp_off = csr(kidx, nf + 1)
    factor.state_priors_fold(nf + 1, _dev(torch, sp_off), _dev(torch, kinfo[order]), _dev(torch, krhs[order]), _dev(torch, kf[order]),
                             G11=full[0], G22=full[2], g1=full[3], g2=full[4], f=full[5], n_chains=1)
    D, E, b = factor.chains_assemble(*full[:5], nf + 1, 0.0, prior, z15)
    x_full = factor.chain_solve(D, E, b).cpu().numpy()
    Dh, Eh, bh = mat(D.cpu().numpy()), mat(E.cpu().numpy()), b.cpu().numpy()
    A = np.zeros((15 * (nf + 1),) * 2)
    for k in range(nf + 1):
        A[15 * k:15 * k + 15, 15 * k:15 * k + 15] = Dh[k]
        if k < nf:
            A[15 * k:15 * k + 15, 15 * k + 15:15 * k + 30] = Eh[k]; A[15 * k + 15:15 * k + 30, 15 * k:15 * k + 15] = Eh[k].T
    xt, x64 = (v.reshape(-1, 15) for v in _dense_truth(A, bh.reshape(-1)))
    sp_all = _sp_dev(torch, kidx, kinfo, krhs, kf, Xc[kidx])
    for m in (1, 6, 21, 29):
        info_m, r_m, f_m = factor.chain_marginalize(*G1, nf + 1, m, prior=(prior, z15, z1), state_priors=sp_all)
        sl = slice(m, nf)
        red = [t[sl].clone() for t in G1]
        keep = kidx >= m
        order, sp_off = csr(kidx[keep] - m, nf + 1 - m)
        pi_m = info_m.clone()
        factor.state_priors_fold(nf + 1 - m, _dev(torch, sp_off), _dev(torch, kinfo[keep][order]), _dev(torch, krhs[keep][order]),
                                 _dev(torch, kf[keep][order]), G11=red[0] if m < nf else None, G22=red[2] if m < nf else None,
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
def test_nan_prior_is_isolated(cuda, oracle):
    """A state prior with NaN info in chain 3 of 10 ends that chain NONFINITE with its input states; the other nine are bitwise the
    clean run."""
    torch = cuda
    rng = np.random.default_rng(8)
    sizes = [5, 1, 12, 20, 8, 1, 30, 3, 16, 9]
    X, rec, L, offs, pri, _ = make_problem(oracle, 1, sizes, 11, large=True, with_prior=True)
    sp = _meas_priors(oracle, rng, X, offs, 3, "p")
    clean = _device_lm(torch, 1, X, rec, L, offs, pri, sp)
    q = int(np.flatnonzero((sp[0] >= offs[3]) & (sp[0] < offs[4]))[0])
    bad = list(sp); bad[1] = sp[1].copy(); bad[1][q, 200] = np.nan
    Xb, cb, lb, sb, ib, tb = _device_lm(torch, 1, X, rec, L, offs, pri, bad)
    assert sb[3] == capi.LM_NONFINITE and ib[3] == 0
    assert np.array_equal(Xb[offs[3]:offs[4]], X[offs[3]:offs[4]])
    Xs, cost, lam, st, it, tr = clean
    assert np.all(st == capi.LM_CONVERGED)
    for c in range(len(sizes)):
        if c == 3:
            continue
        part = slice(offs[c], offs[c + 1])
        assert np.array_equal(Xb[part], Xs[part]) and cb[c] == cost[c] and lb[c] == lam[c] and sb[c] == st[c] and ib[c] == it[c], c


def _fix(rng, truth_k, sigma=0.01):
    W = np.zeros((15, 15)); W[12:15, 12:15] = np.eye(3) / sigma ** 2
    xb = truth_k.copy(); xb[13:16] += rng.normal(0, sigma, 3)
    return W, xb


@pytest.mark.gpu
def test_fixed_lag_smoother_with_position_fixes(cuda, oracle):
    """The fixed-lag loop of test_fixed_lag_smoother_with_lm with a position fix on every 5th keyframe: 8 sequences of 50 keyframes,
    lag 12; each window's fixes go to chains_lm, the oldest state's fix (moved to the current states) into the marginalisation.  The
    same loop in numpy on 3 sequences agrees in retract coordinates."""
    from cpi_b200 import factor, preint
    torch = cuda
    ns, K, W, lam = 8, 50, 12, 1e-5
    S, L = synth.make_windows(ns * (K - 1), 20, rate=200.0, first_window=95000, special=False)
    rec = preint.preintegrate_host(1, S, L, synth.SIGMAS, 0, ns=20).reshape(ns, K - 1, -1)
    L = L.reshape(ns, K - 1, 13)
    rng = np.random.default_rng(23)
    truth = np.stack([synth.make_states(rec[s], L[s], 1, perturb=False) for s in range(ns)])
    fixes = {}
    for s in range(ns):
        for k in range(5, K, 5):
            fixes[(s, k)] = _fix(rng, truth[s, k])
    X0 = truth[:, :W].copy()
    X0[:, 1:, 7:10] += rng.normal(0, 1e-3, (ns, W - 1, 3)); X0[:, 1:, 13:16] += rng.normal(0, 1e-3, (ns, W - 1, 3))
    X0[:, 1:, 4:7] += rng.normal(0, 1e-5, (ns, W - 1, 3))
    dR, dL = _dev(torch, rec), _dev(torch, L)
    info0 = np.eye(15) * 1e8
    prior = (_dev(torch, np.tile(vec(info0[None]), (ns, 1))), torch.zeros((ns, 15), dtype=torch.float64, device="cuda"),
             torch.zeros(ns, dtype=torch.float64, device="cuda"), _dev(torch, X0[:, 0].copy()))
    Xw = _dev(torch, X0)
    first = torch.arange(ns, device="cuda") * (W + 1)

    def window_fixes(t0, n):                                       # the fixes on keyframes t0 .. t0 + n - 1 of every window (W + 1 states)
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
                                                  state_priors=_sp_dev(torch, *sp))
        Xw = new.view(ns, W + 1, 16)
        e, H1, H2 = factor.factor_eval(1, Xw.reshape(-1, 16), dR[:, t0].contiguous(), dL[:, t0].contiguous(), idx_i=first, idx_j=first + 1)
        G = factor.factor_hessian(1, dR[:, t0].contiguous(), e, H1, H2)
        r_p, f_p = factor.prior_at(prior[0], prior[1], prior[2], prior[3], Xw[:, 0].contiguous())
        i0, f_info, f_rhs, f_f, f_lin = window_fixes(t0, 1)            # the oldest state's fix, moved to the states it is marginalised at
        sidx = torch.from_numpy(i0 // (W + 1) * 2).cuda()
        x_at = Xw.reshape(-1, 16)[torch.from_numpy(i0).cuda()]
        rr, ff = factor.prior_at(_dev(torch, f_info), _dev(torch, f_rhs), _dev(torch, f_f), _dev(torch, f_lin), x_at)
        mi, mr, mf = factor.chain_marginalize(*G, 2, 1, prior=(prior[0], r_p, f_p), n_chains=ns,
                                              state_priors=(sidx, _dev(torch, f_info), rr, ff, x_at))
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
            sps = [(j, vec(fixes[(s, t0 + j)][0][None])[0], np.zeros(15), 0.0, fixes[(s, t0 + j)][1]) for j in range(W + 1) if (s, t0 + j) in fixes]
            Xs = np_lm_sp(oracle, 1, Xs, rec[s, t0:t], L[s, t0:t], pr, sps, lam)[0]
            info, rhs, f0, x_lin = pr
            e, H1, H2 = oracle.factor_eval(1, Xs[:2], rec[s, t0:t0 + 1], L[s, t0:t0 + 1])
            G = [g.copy() for g in _np_hessian(rec[s, t0:t0 + 1], e, H1, H2)]
            rhs_p, f_p = prior_at_ref(vec(info[None]), rhs[None], np.array([f0]), x_lin[None], Xs[:1])
            if sps and sps[0][0] == 0:
                _, fi, frhs, ff0, fl = sps[0]
                rr, fq = prior_at_ref(fi[None], frhs[None], np.array([ff0]), fl[None], Xs[:1])
                G[0][0] = G[0][0] + mat(fi)[0]; G[3][0] = G[3][0] + rr[0]; G[5][0] = G[5][0] + fq[0]
            Lam, eta, fm = marginalize_ref(*G, 1, (info, rhs_p[0], f_p[0]), jacobi=True)
            pr = (Lam, eta, fm, Xs[1].copy())
            Xs = Xs[1:]
        worst = max(worst, np.linalg.norm(local(Xs, Xg[s])) / np.linalg.norm(Xs[:, 4:16]))
    print(f"fixed-lag smoother with position fixes vs numpy: worst relative difference {worst:.2e} (retract coordinates)")
    assert worst <= 1e-9


@pytest.mark.gpu
def test_long_chain_with_position_fixes(cuda):
    """The configs[4]-style chain (5 000 states, model 1, a 1e8 I prior on x_0, small perturbations) with a 1 cm position fix every
    50 keyframes, lambda_lower = 0 (the default).  Without fixes it ends NONFINITE (DESIGN.md section 3f); it must not end NONFINITE
    with them.  Prints its final status and counters."""
    from cpi_b200 import factor, preint
    torch = cuda
    n = 5000
    rng = np.random.default_rng(1)
    Sm, L = synth.make_windows(n - 1, 20, rate=200.0, first_window=9000, special=False)
    rec = preint.preintegrate_host(1, Sm, L, synth.SIGMAS, 0, ns=20)
    truth = synth.make_states(rec, L, 1, perturb=False)
    X = truth.copy()
    X[1:, 7:10] += rng.normal(0, 1e-3, (n - 1, 3)); X[1:, 13:16] += rng.normal(0, 1e-3, (n - 1, 3)); X[1:, 4:7] += rng.normal(0, 1e-5, (n - 1, 3))
    idx = np.arange(50, n, 50, dtype=np.int64)
    fx = [_fix(rng, truth[k]) for k in idx]
    M = len(idx)
    sp = (idx, np.stack([vec(w[None])[0] for w, _ in fx]), np.zeros((M, 15)), np.zeros(M), np.stack([xb for _, xb in fx]))
    info0 = torch.eye(15, dtype=torch.float64, device="cuda").reshape(1, 225) * 1e8
    dX = _dev(torch, X)
    Xs, cost, lam, st, it, tr = factor.chains_lm(1, dX, _dev(torch, rec), _dev(torch, L), n, prior=(info0, None, None, dX[:1].clone()),
                                              state_priors=_sp_dev(torch, *sp))
    st, it, tr = int(st[0]), int(it[0]), int(tr[0])
    print(f"5 000-state chain with a position fix every 50 keyframes: status {st}, {it} accepted steps in {tr} rounds, lambda {float(lam[0]):.1e}, "
          f"cost {float(cost[0]):.6e}")
    assert st != capi.LM_NONFINITE and bool(torch.isfinite(Xs).all())
