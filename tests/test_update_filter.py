"""The filter that cpi_propagate_batch (K7) and cpi_state_update_batch (K10) make, against the smoother of the chain entry points
(DESIGN.md section 3k): the linear-Gaussian identity filter = smoother at the newest state, and the filter's Monte-Carlo consistency
on the configuration of test_chain_marginals.test_monte_carlo_consistency_of_the_smoother."""
from __future__ import annotations

import numpy as np
import pytest

from cpi_b200 import capi, synth
from test_chain_marginals import _system, dense, inv_truth
from test_marginalize import local, mat, vec
from test_propagate import random_cov
from test_state_priors import _fix


def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_filter_is_the_smoother_at_the_newest_state(cuda, model):
    """A chain at its exact prediction from x_0 with the prior Sigma_0 and 1 cm position fixes placed exactly at the predicted states
    of keyframes 5, 10, 15 and 20 (d = 0), so both estimators linearise at the same points.  The filter runs K7 + K10 keyframe by
    keyframe; its Sigma_k is the marginal of the last state of the chain truncated at k, all truncations in one ragged
    chains_marginals call.  Gate: 20x the distance between the same two routes in numpy (propagation and update from the device's
    Jacobians, and the refined dense inverse of the device's blocks), floor 1e-12, in the filter's standard deviations."""
    from cpi_b200 import factor, preint
    torch = cuda
    m, fixes = 25, (5, 10, 15, 20)
    S, L = synth.make_windows(m, 20, rate=200.0, first_window=15000 + model, special=False)
    L[:] = L[0]
    rec = preint.preintegrate_host(model, S, L, synth.SIGMAS, 0, ns=20)
    x0 = synth.make_states(rec, L, model, perturb=False)[:1]
    x0[:, 4:7], x0[:, 10:13] = L[:1, 0:3], L[:1, 3:6]
    rng = np.random.default_rng(6 + model)
    Sig0 = mat(random_cov(rng, 1))[0]
    Wp = np.zeros((15, 15)); Wp[12:15, 12:15] = np.eye(3) / 0.01 ** 2
    dR, dL = _dev(torch, rec), _dev(torch, L)
    # the filter
    xs, cs = [_dev(torch, x0)], [_dev(torch, vec(Sig0[None]))]
    for k in range(m):
        x1, c1, _ = factor.propagate(model, xs[-1], cs[-1], dR[k:k + 1], dL[k:k + 1])
        if k + 1 in fixes:
            x1, c1, nis, applied = factor.update(x1, c1, _dev(torch, vec(Wp[None])), x1.clone())
            assert float(nis[0]) == 0.0 and int(applied[0]) == 1
        xs.append(x1); cs.append(c1)
    X = torch.cat(xs)
    Sf = mat(torch.cat(cs).cpu().numpy())
    # every truncation 0..k as one chain of a ragged batch; the fixes as state priors at the predicted states
    Xn, recn = X.cpu().numpy(), rec
    Xr = np.concatenate([Xn[:k + 1] for k in range(m + 1)])
    Rr = np.concatenate([recn[:k] for k in range(m + 1)])
    Lr = np.concatenate([L[:k] for k in range(m + 1)])
    offs = np.concatenate([[0], np.cumsum(np.arange(1, m + 2))]).astype(np.int64)
    idx = np.array([offs[c] + j for c in range(m + 1) for j in fixes if j <= c], dtype=np.int64)
    Lam0 = np.linalg.inv(Sig0); Lam0 = 0.5 * (Lam0 + Lam0.T)
    C = m + 1
    prior = (_dev(torch, np.repeat(vec(Lam0[None]), C, axis=0)), _dev(torch, np.zeros((C, 15))), _dev(torch, np.zeros(C)),
             _dev(torch, Xr[offs[:-1]]))
    sp = (_dev(torch, idx), _dev(torch, np.repeat(vec(Wp[None]), len(idx), axis=0)), None, None, _dev(torch, Xr[idx]))
    d_offs = _dev(torch, offs)
    cov, _ = factor.chains_marginals(model, _dev(torch, Xr), _dev(torch, Rr), _dev(torch, Lr), d_offs, prior=prior, state_priors=sp)
    cov = mat(cov.cpu().numpy())
    # numpy: the filter from the device's Jacobians, and the refined dense inverse of the device's blocks
    e, H1, H2 = factor.factor_eval(model, X, dR, dL)
    h1, h2, Pm = mat(H1.cpu().numpy()), mat(H2.cpu().numpy()), mat(rec[:, 65:290])
    S_np = [Sig0]
    for k in range(m):
        B = np.linalg.inv(h2[k]); A = -B @ h1[k]
        P = A @ S_np[-1] @ A.T + B @ Pm[k] @ B.T
        if k + 1 in fixes:
            P = np.linalg.inv(np.linalg.inv(P) + Wp)
        S_np.append(0.5 * (P + P.T))
    D, E = _system(torch, model, _dev(torch, Xr), _dev(torch, Rr), _dev(torch, Lr), d_offs, prior, sp)
    D, E = mat(D.cpu().numpy()), mat(E.cpu().numpy())
    err = err_np = 0.0
    for k in range(m + 1):
        lo, hi = int(offs[k]), int(offs[k + 1])
        T, _ = inv_truth(dense(D, E, lo, hi))
        d = 1.0 / np.sqrt(np.diag(Sf[k]))
        sc = lambda A: float(np.max(np.abs(A) * d[:, None] * d[None, :]))
        err = max(err, sc(cov[hi - 1] - Sf[k]))
        err_np = max(err_np, sc(T[-15:, -15:] - S_np[k]))
    print(f"model {model}: filter Sigma_k against the last marginal of the chain truncated at k: device {err:.2e}, numpy routes {err_np:.2e}")
    assert err <= 20 * max(err_np, 1e-12), (err, err_np)


def _filter_and_smoother(torch, oracle, model, N, K, seed, noise=None, fixes=(3, 6, 9), sigma_fix=0.01):
    """The realisations of test_chain_marginals._smoother_monte_carlo (the same configuration and draws, restated here because the
    filter needs its records and fixes), smoothed as there and filtered: from x_hat_0 with Sigma_0, cpi_propagate_batch over every
    record and cpi_state_update_batch with the fix at each fixed keyframe.  Returns (filter errors [N, K, 15] of the truth in retract
    coordinates at the filter's estimate, the filter's Sigma [N, K, 15, 15], the smoother's estimate at the last keyframe [N, 16] and
    its Sigma there [N, 15, 15], the filter's estimate there [N, 16], smoother status)."""
    from cpi_b200 import factor, preint
    from test_propagate import random_cov as rc
    rng = np.random.default_rng(seed)
    nz = None if noise is None else np.random.default_rng([seed, noise])

    def draw(size, scale=1.0):
        x = rng.normal(0.0, scale, size)
        return x if nz is None else nz.normal(0.0, scale, size)
    ns = 20
    Sw, Lw = synth.make_windows(K - 1, ns, rate=200.0, first_window=81000 + 100 * model, special=False)
    Lw[:] = Lw[0]
    dt = Sw[:, :, 6]
    w_true, a_true = Sw[:, :, 0:3] - Lw[0, 0:3], Sw[:, :, 3:6] - Lw[0, 3:6]
    x_true = np.zeros((K, 16))
    q = rng.normal(size=4); q /= np.linalg.norm(q); q *= np.sign(q[3])
    x_true[0, 0:4], x_true[0, 4:7], x_true[0, 7:10], x_true[0, 10:13], x_true[0, 13:16] = q, Lw[0, 0:3], [1.0, -0.5, 0.2], Lw[0, 3:6], [3.0, 1.0, -2.0]
    for k in range(K - 1):
        lin_t = np.concatenate([x_true[k, 4:7], x_true[k, 10:13], x_true[k, 0:4], synth.GRAVITY])[None]
        clean = np.concatenate([w_true[k] + x_true[k, 4:7], a_true[k] + x_true[k, 10:13], dt[k][:, None]], axis=1)[None]
        x_true[k + 1] = oracle.predict_state(model, x_true[k:k + 1], preint.preintegrate_host(model, clean, lin_t, synth.SIGMAS, 0, ns=ns), lin_t)[0]
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
    Sig0 = mat(rc(rng, 1)[0])[0]
    delta = draw((N, 15)) @ np.linalg.cholesky(Sig0).T
    xh0 = oracle.retract(truth[:, 0], -delta)
    att = np.zeros((N, 15)); att[:, 0:3] = -delta[:, 0:3]
    lin = np.empty((N, K - 1, 13))
    lin[:, :, 0:3], lin[:, :, 3:6], lin[:, :, 10:13] = xh0[:, None, 4:7], xh0[:, None, 10:13], synth.GRAVITY
    for k in range(K - 1):
        lin[:, k, 6:10] = oracle.retract(truth[:, k], att)[:, 0:4]
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dl = d(lin.reshape(-1, 13))
    rec = preint.preintegrate(model, d(samples.reshape(N * (K - 1), ns, 7)), dl, synth.SIGMAS, 0, ns=ns)
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
    Xs, cov = Xs.cpu().numpy().reshape(N, K, 16), mat(cov.cpu().numpy()).reshape(N, K, 15, 15)
    # the filter
    x, c = d(xh0), d(np.repeat(vec(Sig0[None]), N, axis=0))
    xf, cf = [x], [c]
    for k in range(K - 1):
        x, c, _ = factor.propagate(model, x, c, recK[:, k].contiguous(), linK[:, k].contiguous())
        if k + 1 in fixes:
            j = fixes.index(k + 1)
            x, c, _, applied = factor.update(x, c, d(W[j]), d(xb[j]))
            assert bool((applied == 1).all())
        xf.append(x); cf.append(c)
    Xf = torch.stack(xf, dim=1).cpu().numpy()
    Cf = mat(torch.stack(cf, dim=1).cpu().numpy().reshape(-1, 225)).reshape(N, K, 15, 15)
    err = local(Xf.reshape(N * K, 16), truth.reshape(N * K, 16)).reshape(N, K, 15)
    return err, Cf, Xs[:, K - 1], cov[:, K - 1], Xf[:, K - 1], status.cpu().numpy()


# The filter's distance to the smoother at the last keyframe, in the smoother's marginal standard deviations (worst component over
# the 30 000 realisations): model 1 measured 0.062 on one H100 80GB HBM3 at 700 W (DESIGN.md section 3k); the gate is 4 times that.
FILTER_SMOOTHER_BOUND = 0.25


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, pytest.param(2, marks=pytest.mark.xfail(strict=True, reason=(
    "model 2's filter is not consistent on this configuration: its mean NEES leaves the band from keyframe 4 and reaches 17.5 at "
    "keyframe 9, and it lies 0.9 marginal sd from the smoother on average at the last keyframe (DESIGN.md section 3k)")))])
def test_monte_carlo_consistency_of_the_filter(cuda, oracle, model):
    """The realisations of test_monte_carlo_consistency_of_the_smoother (N = 30 000: seed 90 + model, its own noise stream and two
    independent ones), filtered with K7 + K10 from x_hat_0 and Sigma_0 with the same 1 cm fixes on keyframes 3, 6 and 9: at every
    keyframe the filter's mean NEES lies in the two-sided 99.9 % chi^2_15 band for N and every entry of the error's second moment lies
    within 5 standard errors of the mean Sigma_k.  At the last keyframe the filter and the smoother estimate the same state; their
    distance in the smoother's marginal standard deviations is gated at FILTER_SMOOTHER_BOUND.  Model 2 fails both (a finding, kept
    as a strict expected failure so that a fix shows: DESIGN.md section 3k)."""
    from scipy.stats import chi2
    n, K, streams = 10_000, 10, (None, 1, 2)
    nees_sum, m2_sum, cov_sum = np.zeros(K), np.zeros((K, 15, 15)), np.zeros((K, 15, 15))
    dist, dist_mean = 0.0, 0.0
    for s in streams:
        err, cov, xs, cs, xf, status = _filter_and_smoother(cuda, oracle, model, n, K, 90 + model, noise=s)
        assert np.all(status != capi.LM_NONFINITE) and np.all(status != capi.LM_RUNNING)
        for k in range(K):
            e, C = err[:, k], cov[:, k]
            nees = np.einsum("ni,ni->n", e, np.linalg.solve(C, e[:, :, None])[:, :, 0])
            print(f"model {model}, noise stream {s}, keyframe {k}: filter's mean NEES of the batch {nees.mean():.3f}")
            nees_sum[k] += nees.sum(); m2_sum[k] += e.T @ e; cov_sum[k] += C.sum(axis=0)
        z = np.abs(local(xs, xf)) / np.sqrt(np.diagonal(cs, axis1=1, axis2=2))
        dist = max(dist, float(z.max())); dist_mean += float(z.max(axis=1).sum())
    N = n * len(streams)
    lo, hi = chi2.ppf([0.0005, 0.9995], 15 * N) / N
    worst_z, outside = 0.0, []
    for k in range(K):
        M, Cm = m2_sum[k] / N, cov_sum[k] / N
        se = np.sqrt((np.outer(np.diag(Cm), np.diag(Cm)) + Cm ** 2) / N)
        z = float(np.max(np.abs((M - Cm) / se)))
        worst_z = max(worst_z, z)
        print(f"model {model}, keyframe {k}: filter's mean NEES {nees_sum[k] / N:.3f} over {N} (band [{lo:.3f}, {hi:.3f}]), worst |z| {z:.1f}")
        if not lo <= nees_sum[k] / N <= hi:
            outside.append((k, float(nees_sum[k] / N)))
    print(f"model {model}: filter - smoother at the last keyframe, in the smoother's marginal sd: worst {dist:.3e}, "
          f"mean of the per-realisation worst {dist_mean / N:.3e}")
    assert not outside, outside
    assert worst_z <= 5.0, worst_z
    assert dist <= FILTER_SMOOTHER_BOUND, (dist, FILTER_SMOOTHER_BOUND)
