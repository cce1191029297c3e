"""The filter's update by attitude-dependent measurements (cpi_state_update_measurements_batch, kernel K11,
factor.update_measurements; DESIGN.md section 3l) against its numpy statement tests/measurement_ref.py (update_meas_ref, tied on the
CPU to the information form and the Kalman gain in tests/test_measurements.py) and against K10."""
import numpy as np
import pytest

import measurement_ref as mr
from cpi_b200 import capi, synth
from test_marginalize import local, mat, vec
from test_measurements import _filters, realisations
from test_propagate import random_cov
from update_ref import errors

LEVER = np.array([0.5, 0.2, 1.0])                                     # the GNSS antenna in the IMU frame, metres


def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _run(torch, x, cov, owner, kind, z, si, aux, gate=None):
    from cpi_b200 import factor
    g = _dev(torch, gate) if isinstance(gate, np.ndarray) else gate
    ms = (_dev(torch, owner.astype(np.int64)), _dev(torch, kind), _dev(torch, z), _dev(torch, si), _dev(torch, aux))
    out = factor.update_measurements(_dev(torch, x), _dev(torch, cov), ms, gate=g)
    torch.cuda.synchronize()
    return tuple(t.cpu().numpy() for t in out)


@pytest.mark.gpu
def test_kernel_is_the_statement(cuda):
    """0 to 4 measurements of every kind per filter (owners shuffled: the wrapper sorts them): every field within 20x the distance
    between the square-root and the information statements (floor 1e-13); cov+ exactly symmetric; a filter without measurements
    bitwise its inputs with gamma = 0 and applied = 1; two runs give the same bits."""
    torch = cuda
    rng = np.random.default_rng(70)
    counts = rng.integers(0, 5, size=400)
    x, cov, off, owner, kind, z, si, aux = _filters(rng, len(counts), counts)
    perm = rng.permutation(len(owner))
    got = _run(torch, x, cov, owner[perm], kind[perm], z[perm], si[perm], aux[perm])
    again = _run(torch, x, cov, owner[perm], kind[perm], z[perm], si[perm], aux[perm])
    assert all(np.array_equal(a, b) for a, b in zip(got, again))
    assert np.array_equal(mat(got[1]), mat(got[1]).transpose(0, 2, 1)) and np.all(got[3] == 1)
    none = counts == 0
    assert np.array_equal(got[0][none], x[none]) and np.array_equal(got[1][none], cov[none]) and np.all(got[2][none] == 0)
    r = mr.update_meas_ref(x, cov, off, kind, z, si, aux)
    i = mr.update_meas_info(x, cov, off, kind, z, si, aux)
    some = ~none
    eb, ex, eg = errors((r[0][some], r[1][some], r[3][some]), (got[0][some], got[1][some], got[2][some]), x[some])
    nb, nx, ng = errors((r[0][some], r[1][some], r[3][some]), (i[0][some], i[1][some], i[3][some]), x[some])
    print(f"K11 vs update_meas_ref: cov {eb.max():.1e}, state {ex.max():.1e}, gamma {eg.max():.1e}; "
          f"information form: {nb.max():.1e}, {nx.max():.1e}, {ng.max():.1e}")
    assert eb.max() <= 20 * max(nb.max(), 1e-13) and ex.max() <= 20 * max(nx.max(), 1e-13) and eg.max() <= 20 * max(ng.max(), 1e-13)


@pytest.mark.gpu
def test_gating_and_isolation(cuda):
    """A gate skips exactly the filters with gamma > gate (bitwise copies, applied = 0) and leaves the others bitwise the ungated
    run; +inf is bitwise no gate.  A non-SPD cov or a NaN in z in one filter leaves every other filter bitwise the clean run."""
    torch = cuda
    rng = np.random.default_rng(71)
    counts = rng.integers(1, 4, size=64)
    x, cov, off, owner, kind, z, si, aux = _filters(rng, len(counts), counts)
    z[::5] += 1.0                                                    # 20-sigma outliers in some filters
    free = _run(torch, x, cov, owner, kind, z, si, aux)
    inf = _run(torch, x, cov, owner, kind, z, si, aux, gate=float("inf"))
    assert all(np.array_equal(a, b) for a, b in zip(free, inf))
    gate = np.full(len(counts), 16.0)
    xo, co, g, a = _run(torch, x, cov, owner, kind, z, si, aux, gate=gate)
    skip = a == 0
    assert skip.any() and (~skip).any() and np.array_equal(skip, free[2] > gate) and np.array_equal(g, free[2])
    assert np.array_equal(xo[skip], x[skip]) and np.array_equal(co[skip], cov[skip])
    assert np.array_equal(xo[~skip], free[0][~skip]) and np.array_equal(co[~skip], free[1][~skip])
    f = 7
    j = int(off[f])
    for what in ("cov", "z"):
        c2, z2, k2 = cov.copy(), z.copy(), kind.copy()
        if what == "cov":
            S = mat(c2[f:f + 1])[0]; S[3, 3] = -1.0; c2[f] = vec(S[None])[0]
        else:
            z2[j, 1] = np.nan
        got = _run(torch, x, c2, owner, k2, z2, si, aux)
        keep = np.arange(len(counts)) != f
        assert all(np.array_equal(u[keep], v[keep]) for u, v in zip(got, free)), what
        assert np.isnan(got[2][f]) and np.isnan(got[0][f]).any(), what


@pytest.mark.gpu
def test_position_without_lever_arm_is_k10(cuda):
    """One POSITION measurement with aux = 0 per filter equals K10's update by the state fix (W = S^T S on p, x_bar = x with p = z)
    to rounding: 1e-12 in the posterior's standard deviations, gamma to 1e-12."""
    from cpi_b200 import factor
    torch = cuda
    rng = np.random.default_rng(72)
    n = 200
    x, cov, off, owner, kind, z, si, aux = _filters(rng, n, np.ones(n, dtype=np.int64), kinds=(mr.POSITION,))
    aux[:] = 0.0
    got = _run(torch, x, cov, owner, kind, z, si, aux)
    S = mr.sqrt_mat(si)
    W = np.zeros((n, 15, 15)); W[:, 12:15, 12:15] = S.transpose(0, 2, 1) @ S
    xb = x.copy(); xb[:, 13:16] = z
    k10 = [t.cpu().numpy() for t in factor.update(_dev(torch, x), _dev(torch, cov), _dev(torch, vec(W)), _dev(torch, xb))]
    sd = np.sqrt(np.diagonal(mat(k10[1]), axis1=1, axis2=2))
    ex = np.max(np.abs(local(k10[0], got[0])) / sd)
    ec = np.max(np.abs(mat(got[1]) - mat(k10[1])) / (sd[:, :, None] * sd[:, None, :]))
    eg = np.max(np.abs(got[2] - k10[2]) / np.maximum(k10[2], 1.0))
    print(f"K11 vs K10: state {ex:.1e}, cov {ec:.1e}, gamma {eg:.1e}")
    assert ex <= 1e-12 and ec <= 1e-12 and eg <= 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_filter_is_the_smoother_at_the_newest_state(cuda, model):
    """test_update_filter.test_filter_is_the_smoother_at_the_newest_state with measurements in place of the fixes, each taken exactly
    at the predicted state (r = 0): a lever-arm GNSS fix at keyframe 5, a body-velocity fix at 10, two directions at 15, lever-arm
    GNSS and body velocity together at 20.  The filter runs K7 + K11; its Sigma_k is the last marginal of the chain truncated at k
    with the measurements (chains_marginals, K12).  Gate: 20x the distance between the same two routes in numpy (propagation and
    the information-form update from the device's Jacobians and measurement_ref, and the refined dense inverse of the device's
    blocks), floor 1e-12, in the filter's standard deviations."""
    from cpi_b200 import factor, preint
    from test_chain_marginals import _system, dense, inv_truth
    torch = cuda
    m = 25
    plan = {5: [(mr.POSITION, LEVER)], 10: [(mr.VELOCITY_BODY, np.zeros(3))],
            15: [(mr.DIRECTION, np.array([0.0, 0.0, 1.0])), (mr.DIRECTION, np.array([0.6, 0.8, 0.0]))],
            20: [(mr.POSITION, LEVER), (mr.VELOCITY_BODY, np.zeros(3))]}
    S, L = synth.make_windows(m, 20, rate=200.0, first_window=15000 + model, special=False)
    L[:] = L[0]
    rec = preint.preintegrate_host(model, S, L, synth.SIGMAS, 0, ns=20)
    x0 = synth.make_states(rec, L, model, perturb=False)[:1]
    x0[:, 4:7], x0[:, 10:13] = L[:1, 0:3], L[:1, 3:6]
    rng = np.random.default_rng(6 + model)
    Sig0 = mat(random_cov(rng, 1))[0]
    si = (np.eye(3) / 0.01).reshape(9)
    dR, dL = _dev(torch, rec), _dev(torch, L)
    xs, cs, meas = [_dev(torch, x0)], [_dev(torch, vec(Sig0[None]))], {}
    for k in range(m):
        x1, c1, _ = factor.propagate(model, xs[-1], cs[-1], dR[k:k + 1], dL[k:k + 1])
        if k + 1 in plan:
            xn = x1.cpu().numpy()
            kind = np.array([q for q, _ in plan[k + 1]], dtype=np.int32)
            aux = np.array([a for _, a in plan[k + 1]])
            z = mr.h_of(kind, np.repeat(xn, len(kind), axis=0), aux)
            meas[k + 1] = (kind, z, aux)
            ms = (np.zeros(len(kind), dtype=np.int64), kind, z, np.tile(si, (len(kind), 1)), aux)
            x1, c1, nis, applied = factor.update_measurements(x1, c1, tuple(_dev(torch, a) for a in ms))
            assert float(nis[0]) <= 1e-20 and int(applied[0]) == 1
        xs.append(x1); cs.append(c1)
    X = torch.cat(xs)
    Sf = mat(torch.cat(cs).cpu().numpy())
    Xn = X.cpu().numpy()
    Xr = np.concatenate([Xn[:k + 1] for k in range(m + 1)])
    Rr = np.concatenate([rec[:k] for k in range(m + 1)])
    Lr = np.concatenate([L[:k] for k in range(m + 1)])
    offs = np.concatenate([[0], np.cumsum(np.arange(1, m + 2))]).astype(np.int64)
    rows = [(offs[c] + j, meas[j]) for c in range(m + 1) for j in sorted(plan) if j <= c]
    idx = np.concatenate([np.full(len(q[0]), i, dtype=np.int64) for i, q in rows])
    kind = np.concatenate([q[0] for _, q in rows]); z = np.concatenate([q[1] for _, q in rows]); aux = np.concatenate([q[2] for _, q in rows])
    ms_all = tuple(_dev(torch, a) for a in (idx, kind, z, np.tile(si, (len(idx), 1)), aux))
    Lam0 = np.linalg.inv(Sig0); Lam0 = 0.5 * (Lam0 + Lam0.T)
    C = m + 1
    prior = (_dev(torch, np.repeat(vec(Lam0[None]), C, axis=0)), _dev(torch, np.zeros((C, 15))), _dev(torch, np.zeros(C)),
             _dev(torch, Xr[offs[:-1]]))
    d_offs, dXr = _dev(torch, offs), _dev(torch, Xr)
    cov, _ = factor.chains_marginals(model, dXr, _dev(torch, Rr), _dev(torch, Lr), d_offs, prior=prior, measurements=ms_all)
    cov = mat(cov.cpu().numpy())
    e, H1, H2 = factor.factor_eval(model, X, dR, dL)
    h1, h2, Pm = mat(H1.cpu().numpy()), mat(H2.cpu().numpy()), mat(rec[:, 65:290])
    S_np = [Sig0]
    for k in range(m):
        B = np.linalg.inv(h2[k]); A = -B @ h1[k]
        P = A @ S_np[-1] @ A.T + B @ Pm[k] @ B.T
        if k + 1 in plan:
            kk, zz, aa = meas[k + 1]
            _, Am, _ = mr.meas_ref(kk, np.repeat(Xn[k + 1:k + 2], len(kk), axis=0), zz, np.tile(si, (len(kk), 1)), aa)
            P = np.linalg.inv(np.linalg.inv(P) + np.einsum("jki,jkl->il", Am, Am))
        S_np.append(0.5 * (P + P.T))
    sp = factor.measurements_linearize(dXr, ms_all)[3]
    D, E = _system(torch, model, dXr, _dev(torch, Rr), _dev(torch, Lr), d_offs, prior, sp)
    D, E = mat(D.cpu().numpy()), mat(E.cpu().numpy())
    err = err_np = 0.0
    for k in range(m + 1):
        lo, hi = int(offs[k]), int(offs[k + 1])
        T, _ = inv_truth(dense(D, E, lo, hi))
        d = 1.0 / np.sqrt(np.diag(Sf[k]))
        sc = lambda A: float(np.max(np.abs(A) * d[:, None] * d[None, :]))
        err = max(err, sc(cov[hi - 1] - Sf[k]))
        err_np = max(err_np, sc(T[-15:, -15:] - S_np[k]))
    print(f"model {model}: K11 filter Sigma_k against the last marginal of the truncated chain with measurements: device {err:.2e}, "
          f"numpy routes {err_np:.2e}")
    assert err <= 20 * max(err_np, 1e-12), (err, err_np)


def _gnss_velocity(rng, truth, keyframes, sigma_p=0.01, sigma_v=0.05, lever=LEVER):
    """Lever-arm GNSS (sigma_p) and body-velocity (sigma_v) measurements of the realisations truth [N,K,16] at `keyframes`, with
    noise: (state_idx into the N*K states, kind, z, sqrt_info, aux), and the GNSS rows."""
    N, K = truth.shape[:2]
    idx, kind, aux, si = [], [], [], []
    for k in keyframes:
        for q, s in ((mr.POSITION, sigma_p), (mr.VELOCITY_BODY, sigma_v)):
            idx.append(np.arange(N) * K + k); kind.append(np.full(N, q, dtype=np.int32))
            aux.append(np.tile(lever if q == mr.POSITION else np.zeros(3), (N, 1))); si.append(np.tile((np.eye(3) / s).reshape(9), (N, 1)))
    idx, kind, aux, si = np.concatenate(idx).astype(np.int64), np.concatenate(kind), np.concatenate(aux), np.concatenate(si)
    X = truth.reshape(N * K, 16)
    sig = np.where(kind == mr.POSITION, sigma_p, sigma_v)[:, None]
    z = mr.h_of(kind, X[idx], aux) + rng.normal(size=(len(idx), 3)) * sig
    return (idx, kind, z, si, aux), kind == mr.POSITION


def _smooth(torch, model, r, K, ms, loss=None):
    from cpi_b200 import factor
    params = capi.LMParams(absolute_error_tol=0.0, relative_error_tol=1e-13, max_iterations=50)
    dms = tuple(_dev(torch, a) for a in ms)
    Xs, _, _, st, _, _ = factor.chains_lm(model, r["X0"], r["rec"], r["lin"], K, prior=r["prior"], measurements=dms, measurement_loss=loss,
                                          params=params, max_rounds=100)
    return Xs, st.cpu().numpy(), dms


@pytest.mark.gpu
def test_lever_arm_gnss_value(cuda, oracle):
    """Lever-arm GNSS fixes (l = (0.5, 0.2, 1.0) m, 1 cm sigma) and body-velocity fixes on every keyframe of 200 synthetic chains:
    solved with POSITION and the true lever arm, every position and attitude error lies within 6 of the smoother's marginal standard
    deviations; treated as plain position fixes of the IMU (aux = 0) the worst error exceeds 20 of them."""
    from cpi_b200 import factor
    torch = cuda
    N, K = 200, 10
    r = realisations(torch, oracle, 1, N, K, 100)
    truth = r["truth"]
    ms, _ = _gnss_velocity(np.random.default_rng(101), truth, range(K))
    out = []
    for aux in (ms[4], np.zeros_like(ms[4])):
        m2 = (ms[0], ms[1], ms[2], ms[3], aux)
        Xs, st, dms = _smooth(torch, 1, r, K, m2)
        assert np.all(st != capi.LM_NONFINITE)
        cov, _ = factor.chains_marginals(1, Xs, r["rec"], r["lin"], K, prior=r["prior"], measurements=dms)
        sd = np.sqrt(np.diagonal(mat(cov.cpu().numpy()), axis1=1, axis2=2))
        e = np.abs(local(Xs.cpu().numpy(), truth.reshape(N * K, 16))) / sd
        out.append((float(e[:, 12:15].max()), float(e[:, 0:3].max())))
    print(f"lever-arm GNSS: worst position / attitude error {out[0][0]:.2f} / {out[0][1]:.2f} sd with the lever arm, "
          f"{out[1][0]:.1f} / {out[1][1]:.1f} sd as plain position fixes")
    assert max(out[0]) <= 6.0 and max(out[1]) >= 20.0, out


@pytest.mark.gpu
def test_robust_lever_arm_gnss_with_outliers(cuda, oracle):
    """The fixes of test_lever_arm_gnss_value with 5 % of the GNSS fixes moved 5 m: chains_lm converges (no chain non-finite or still
    running) with Gaussian, Huber and Cauchy losses on the GNSS rows (k = 3), and the robust losses' RMS position error is below
    the Gaussian one."""
    torch = cuda
    N, K = 200, 10
    r = realisations(torch, oracle, 1, N, K, 110)
    truth = r["truth"]
    rng = np.random.default_rng(111)
    ms, gnss = _gnss_velocity(rng, truth, range(K))
    out = gnss & (rng.random(len(gnss)) < 0.05)
    ms[2][out] += 5.0 / np.sqrt(3)
    rms = {}
    for name, code in (("gaussian", capi.LOSS_GAUSSIAN), ("huber", capi.LOSS_HUBER), ("cauchy", capi.LOSS_CAUCHY)):
        codes = np.where(gnss, code, capi.LOSS_GAUSSIAN).astype(np.int32)
        loss = (_dev(torch, codes), _dev(torch, np.full(len(codes), 3.0)))
        Xs, st, _ = _smooth(torch, 1, r, K, ms, loss)
        assert np.all(st != capi.LM_NONFINITE) and np.all(st != capi.LM_RUNNING), name
        e = local(Xs.cpu().numpy(), truth.reshape(N * K, 16))[:, 12:15]
        rms[name] = float(np.sqrt(np.mean(e ** 2)))
    print(f"{int(out.sum())} outlying GNSS fixes of {int(gnss.sum())}: RMS position error " + ", ".join(f"{k} {v * 100:.2f} cm" for k, v in rms.items()))
    assert rms["huber"] < rms["gaussian"] and rms["cauchy"] < rms["gaussian"]


@pytest.mark.gpu
def test_monte_carlo_consistency_with_measurements(cuda, oracle):
    """Model 1, 10 000 realisations of 10 keyframes (test_update_filter's configuration) with lever-arm GNSS (1 cm) and body-velocity
    (5 cm/s) fixes on keyframes 3, 6 and 9: at every keyframe the mean NEES of the smoother (chains_lm + chains_marginals with
    measurements, K12) and of the filter (K7 + K11) lies in the two-sided 99.9 % chi^2_15 band for N."""
    from scipy.stats import chi2

    from cpi_b200 import factor
    torch = cuda
    N, K, fixes = 10_000, 10, (3, 6, 9)
    r = realisations(torch, oracle, 1, N, K, 120)
    truth = r["truth"]
    ms, _ = _gnss_velocity(np.random.default_rng(121), truth, fixes)
    Xs, st, dms = _smooth(torch, 1, r, K, ms)
    assert np.all(st != capi.LM_NONFINITE) and np.all(st != capi.LM_RUNNING)
    cov, _ = factor.chains_marginals(1, Xs, r["rec"], r["lin"], K, prior=r["prior"], measurements=dms)
    es = local(Xs.cpu().numpy(), truth.reshape(N * K, 16)).reshape(N, K, 15)
    Cs = mat(cov.cpu().numpy()).reshape(N, K, 15, 15)
    # the filter: the measurements of keyframe k, indexed by filter
    x, c = _dev(torch, r["xh0"]), _dev(torch, np.repeat(vec(r["Sig0"][None]), N, axis=0))
    xf, cf = [x], [c]
    for k in range(K - 1):
        x, c, _ = factor.propagate(1, x, c, r["recK"][:, k].contiguous(), r["linK"][:, k].contiguous())
        if k + 1 in fixes:
            sel = ms[0] % K == k + 1
            mk = (ms[0][sel] // K, ms[1][sel], ms[2][sel], ms[3][sel], ms[4][sel])
            x, c, _, applied = factor.update_measurements(x, c, tuple(_dev(torch, a) for a in mk))
            assert bool((applied == 1).all())
        xf.append(x); cf.append(c)
    Xf = torch.stack(xf, dim=1).cpu().numpy()
    Cf = mat(torch.stack(cf, dim=1).cpu().numpy().reshape(-1, 225)).reshape(N, K, 15, 15)
    ef = local(Xf.reshape(N * K, 16), truth.reshape(N * K, 16)).reshape(N, K, 15)
    lo, hi = chi2.ppf([0.0005, 0.9995], 15 * N) / N
    outside = []
    for name, e, C in (("smoother", es, Cs), ("filter", ef, Cf)):
        for k in range(K):
            nees = float(np.mean(np.einsum("ni,ni->n", e[:, k], np.linalg.solve(C[:, k], e[:, k, :, None])[:, :, 0])))
            print(f"{name}, keyframe {k}: mean NEES {nees:.3f} (band [{lo:.3f}, {hi:.3f}])")
            if not lo <= nees <= hi:
                outside.append((name, k, nees))
    assert not outside, outside
