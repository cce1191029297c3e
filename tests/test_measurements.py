"""Attitude-dependent measurements on any keyframe of many IMU chains: lever-arm position, body-frame velocity and known directions
(cpi_imu_measurements_linearize, kernel K12; factor.measurements_linearize and the measurements argument of chains_lm_step /
chains_lm / chains_marginals; DESIGN.md section 3l).

GTSAM is not in the reference tree, so parity with its GPSFactor and attitude factors is UNPINNED.  The reference is
tests/measurement_ref.py: on the CPU its Jacobians are pinned against central differences through the oracle's retract, and the GPU
tests tie the kernel and the solver entry points to it."""
import ctypes

import numpy as np
import pytest

import measurement_ref as mr
from cpi_b200 import capi, synth
from test_chains_lm import make_problem
from test_marginalize import _dense_truth, local, mat, prior_at_ref, vec
from test_robust_priors import robust_ref
from test_state_priors import _chain_idx, _np_system
from update_ref import unit_states

P = lambda a: ctypes.c_void_p(a.ctypes.data)
KINDS = (mr.POSITION, mr.VELOCITY_BODY, mr.DIRECTION)


def _states(rng, n):
    x = unit_states(rng, n)
    x[:, 7:10] = rng.normal(size=(n, 3)) * 5.0
    return x


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", KINDS)
def test_jacobian_is_the_central_difference_through_retract(oracle, kind):
    """H of every kind equals the central difference of h(retract(x, xi)) through the oracle's retract, at random states with
    rotations up to half a turn: within 1e-8 of the entries' scale."""
    rng = np.random.default_rng(kind)
    n = 16
    x = _states(rng, n)
    aux = rng.normal(size=(n, 3))
    H = mr.jacobian(np.full(n, kind), x, aux)
    eps = 1e-6
    for c in range(15):
        d = np.zeros((n, 15)); d[:, c] = eps
        hp = mr.h_of(np.full(n, kind), oracle.retract(x, d), aux)
        hm = mr.h_of(np.full(n, kind), oracle.retract(x, -d), aux)
        fd = (hp - hm) / (2 * eps)
        scale = max(1.0, np.abs(H).max())
        assert np.max(np.abs(fd - H[:, :, c])) <= 1e-8 * scale, (kind, c, np.max(np.abs(fd - H[:, :, c])))


def test_unknown_kind_gives_nan():
    rng = np.random.default_rng(1)
    x = _states(rng, 2)
    r, A, b = mr.meas_ref(np.array([0, 4]), x, np.zeros((2, 3)), np.tile(np.eye(3).reshape(9), (2, 1)), np.zeros((2, 3)))
    assert np.isnan(r).all() and np.isnan(A).all() and np.isnan(b).all()


def test_position_without_lever_arm_is_a_state_prior():
    """POSITION with aux = 0 is the state prior (W = S^T S on the p block, x_bar = x with p = z): the same (info, rhs', f')."""
    rng = np.random.default_rng(2)
    n = 12
    x = _states(rng, n)
    idx, kind, z, si, aux = mr.random_measurements(rng, x, n, kinds=(mr.POSITION,))
    aux[:] = 0.0
    info, rhs, f = mr.linearize_ref(kind, x[idx], z, si, aux)
    S = mr.sqrt_mat(si)
    W = np.zeros((n, 15, 15)); W[:, 12:15, 12:15] = S.transpose(0, 2, 1) @ S
    xb = x[idx].copy(); xb[:, 13:16] = z
    r2, f2 = prior_at_ref(vec(W), np.zeros((n, 15)), np.zeros(n), xb, x[idx])
    assert np.allclose(info, vec(W), rtol=1e-13, atol=1e-13 * np.abs(info).max())
    assert np.allclose(rhs, r2, rtol=1e-12, atol=1e-12 * np.abs(r2).max()) and np.allclose(f, f2, rtol=1e-12)


def _filters(rng, n, counts, kinds=KINDS, sigma=0.05):
    from test_propagate import random_cov
    x, cov = _states(rng, n), random_cov(rng, n)
    offsets = np.r_[0, np.cumsum(counts)].astype(np.int64)
    M = int(offsets[-1])
    owner = np.repeat(np.arange(n), counts)
    _, kind, z, si, aux = mr.random_measurements(rng, x[owner] if M else x, M, kinds=kinds, sigma=sigma)
    if M:
        z = mr.h_of(kind, x[owner], aux) + rng.normal(size=(M, 3)) * 0.5 * sigma
    return x, cov, offsets, owner, kind, z, si, aux


def test_filter_statement_is_the_information_form_and_the_kalman_gain():
    """update_meas_ref equals the dense information form; for one measurement with invertible Lambda its gain, covariance and gamma
    are the textbook Kalman update's, gamma = r^T (H Sigma H^T + Lambda^-1)^-1 r; two measurements in one call equal their combined
    information form; a singular S (non-holonomic rows) works."""
    rng = np.random.default_rng(3)
    counts = np.array([1, 1, 1, 2, 3, 0, 4, 2])
    x, cov, off, owner, kind, z, si, aux = _filters(rng, len(counts), counts)
    si[3] = (np.diag([0.0, 20.0, 20.0]) @ mr.sqrt_mat(si[3:4])[0]).T.reshape(9)       # lateral and vertical rows only
    r = mr.update_meas_ref(x, cov, off, kind, z, si, aux)
    i = mr.update_meas_info(x, cov, off, kind, z, si, aux)
    for a, b in zip(r[1:], i[1:]):
        assert np.allclose(a, b, rtol=1e-9, atol=1e-9 * np.abs(b).max())
    for f in range(3):                                                 # single measurements: the Kalman form
        j = int(off[f])
        rr, A, b = mr.meas_ref(kind[j:j + 1], x[f:f + 1], z[j:j + 1], si[j:j + 1], aux[j:j + 1])
        S = mr.sqrt_mat(si[j:j + 1])[0]
        H = np.linalg.solve(S, A[0])
        Sig = mat(cov[f:f + 1])[0]
        Sy = H @ Sig @ H.T + np.linalg.inv(S.T @ S)
        K = Sig @ H.T @ np.linalg.inv(Sy)
        assert np.allclose(r[2][f], -K @ rr[0], rtol=1e-9, atol=1e-12)
        assert np.allclose(mat(r[1][f:f + 1])[0], (np.eye(15) - K @ H) @ Sig, rtol=1e-8, atol=1e-12 * np.abs(Sig).max())
        assert abs(r[3][f] - rr[0] @ np.linalg.solve(Sy, rr[0])) <= 1e-9 * max(1.0, r[3][f])
    assert r[3][5] == 0 and np.array_equal(r[1][5], cov[5]) and np.array_equal(r[0][5], x[5])


def test_argument_validation_without_gpu():
    """The C ABI rejects bad counts, NULL pointers and aliased outputs before the device; the wrappers reject shapes, dtypes, index
    range, kind codes and loss values before the device."""
    import torch

    from cpi_b200 import factor
    lib = capi.load()
    buf = [np.zeros(8 * 225) for _ in range(12)]
    p = [P(b) for b in buf]
    lin = lambda n, *a: lib.cpi_imu_measurements_linearize(n, *a, None)
    ok = p[0:7] + [p[7], p[8]]
    assert lin(-1, *ok) == -1 and b"negative" in lib.cpi_last_error()
    assert lin(0, *[None] * 9) == 0
    for k in range(7):
        bad = list(ok); bad[k] = None
        assert lin(2, *bad) == -1 and b"null" in lib.cpi_last_error(), k
    bad = list(ok); bad[7] = None
    assert lin(2, *bad) == -1 and b"both" in lib.cpi_last_error()
    bad = list(ok); bad[8] = p[6]
    assert lin(2, *bad) == -1 and b"overlap" in lib.cpi_last_error()
    bad = list(ok); bad[7] = p[8]
    assert lin(2, *bad) == -1 and b"overlap" in lib.cpi_last_error()
    upd = lambda n, *a: lib.cpi_state_update_measurements_batch(n, *a, None)
    ok = p[0:8] + [p[8], p[9], p[10], None]
    assert upd(-1, *ok) == -1 and b"negative" in lib.cpi_last_error()
    assert upd(0, *[None] * 12) == 0
    for k in (0, 1, 2, 3, 4, 5, 6, 8, 9):
        bad = list(ok); bad[k] = None
        assert upd(2, *bad) == -1 and b"null" in lib.cpi_last_error(), k
    bad = list(ok); bad[9] = p[1]
    assert upd(2, *bad) == -1 and b"overlap" in lib.cpi_last_error()
    bad = list(ok); bad[10] = p[9]
    assert upd(2, *bad) == -1 and b"overlap" in lib.cpi_last_error()
    # the Python layer
    N = 12
    X, rec, lin_ = torch.zeros(N, 16, dtype=torch.float64), torch.zeros(N - 3, 290, dtype=torch.float64), torch.zeros(N - 3, 13, dtype=torch.float64)
    f64 = dict(dtype=torch.float64)
    good = lambda: (torch.tensor([0, 5]), torch.tensor([1, 3], dtype=torch.int32), torch.zeros(2, 3, **f64), torch.zeros(2, 9, **f64),
                    torch.zeros(2, 3, **f64))
    calls = (lambda m, l=None: factor.chains_lm_step(1, X, rec, lin_, 4, measurements=m, measurement_loss=l),
             lambda m, l=None: factor.chains_lm(1, X, rec, lin_, 4, measurements=m, measurement_loss=l),
             lambda m, l=None: factor.chains_marginals(1, X, rec, lin_, 4, measurements=m, measurement_loss=l),
             lambda m, l=None: factor.measurements_linearize(X, m))
    for call in calls:
        i, k, z, s, a = good()
        for bad, exc, msg in (((i, k), ValueError, "measurements is"), ((i.int(), k, z, s, a), ValueError, "int64"),
                              ((i, k.long(), z, s, a), ValueError, "int32"), ((i, k[:1], z, s, a), ValueError, "kind"),
                              ((i, k, z[:, :2], s, a), ValueError, "z"), ((i, k, z, s[:, :8], a), ValueError, "sqrt_info"),
                              ((i, k, z, s, a.float()), ValueError, "float64"),
                              ((torch.tensor([0, 12]), k, z, s, a), IndexError, "out of range"),
                              ((torch.tensor([-1, 3]), k, z, s, a), IndexError, "out of range"),
                              ((i, torch.tensor([0, 1], dtype=torch.int32), z, s, a), ValueError, "kind codes"),
                              ((i, torch.tensor([1, 4], dtype=torch.int32), z, s, a), ValueError, "kind codes"),
                              ((i, k, z, s, a), ValueError, "CUDA")):
            with pytest.raises(exc, match=msg):
                call(bad)
    for call in calls[:3]:
        for loss, msg in (((torch.tensor([0, 1], dtype=torch.int32),), "measurement_loss is"),
                          ((torch.tensor([0, 3], dtype=torch.int32), torch.ones(2, **f64)), "loss codes"),
                          ((torch.tensor([1, 1], dtype=torch.int32), torch.tensor([1.0, 0.0], **f64)), "threshold"),
                          ((torch.tensor([1, 1]), torch.ones(2, **f64)), "int32")):
            with pytest.raises(ValueError, match=msg):
                call(good(), loss)
        with pytest.raises(ValueError, match="needs measurements"):
            call(None, (torch.tensor([0, 1], dtype=torch.int32), torch.ones(2, **f64)))
    xs, cs = torch.zeros(4, 16, **f64), torch.zeros(4, 225, **f64)
    with pytest.raises(ValueError, match="CUDA"):
        factor.update_measurements(xs, cs, good())
    with pytest.raises(ValueError, match="tensor"):
        factor.update_measurements(xs.numpy(), cs, good())


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------

def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ms_dev(torch, ms):
    return tuple(_dev(torch, a) for a in ms)


@pytest.mark.gpu
def test_kernel_is_the_statement(cuda):
    """K12 against linearize_ref for every kind (and an unknown one, NaN) at random states: every field within 1e-13 of the scale it
    is formed at; info exactly symmetric; the f-only pass bitwise the full pass's f; two runs give the same bits.  K12's
    extended-precision gate on the measurement stress batch is tests/test_measurements_precision.py."""
    from cpi_b200 import factor
    torch = cuda
    rng = np.random.default_rng(20)
    x = _states(rng, 300)
    ms = list(mr.random_measurements(rng, x, 5000))
    dX, dms = _dev(torch, x), _ms_dev(torch, ms)
    clean = factor.measurements_linearize(dX, dms)
    ms[1][77] = 9                                                    # the wrapper refuses unknown kinds: the C ABI takes them
    idx, kind, z, si, aux = dms = _ms_dev(torch, ms)
    lib = capi.load()
    p = factor._tptr
    M = len(ms[0])

    def k12(full):
        info, rhs, f = torch.empty((M, 225), dtype=torch.float64, device="cuda"), torch.empty((M, 15), dtype=torch.float64, device="cuda"), \
            torch.empty(M, dtype=torch.float64, device="cuda")
        capi.check(lib.cpi_imu_measurements_linearize(M, p(kind), p(idx), p(dX), p(z), p(si), p(aux), p(info) if full else None,
                                                      p(rhs) if full else None, p(f), None))
        return info, rhs, f
    keep = torch.arange(M, device="cuda") != 77
    info, rhs, f = k12(True)
    again, f_only = k12(True), k12(False)[2]
    torch.cuda.synchronize()
    got = [t.cpu().numpy() for t in (info, rhs, f)]
    assert all(torch.equal(a[keep], b[keep]) and bool(torch.isnan(b[~keep]).all()) for a, b in zip((info, rhs, f), again))
    assert torch.equal(f_only[keep], f[keep]) and bool(torch.isnan(f_only[77]))
    assert all(torch.equal(a[keep], b[keep]) for a, b in zip((info, rhs, f), clean[:3]))
    assert torch.equal(clean[3][1], clean[0]) and torch.equal(clean[3][4], dX[idx])
    I = mat(got[0])
    bad = np.zeros(len(f), bool); bad[77] = True
    assert np.isnan(got[0][77]).all() and np.isnan(got[1][77]).all() and np.isnan(got[2][77])
    assert np.array_equal(I[~bad], I[~bad].transpose(0, 2, 1))
    want = mr.linearize_ref(ms[1], x[ms[0]], ms[2], ms[3], ms[4])
    # r = h - z is formed at the scale of |h| + |z| (metres of position against a residual of centimetres): rhs' and f' are
    # measured against |A| (|S| (|h| + |z|)) and (|S| (|h| + |z|))^2, info against its own largest entry
    good = ~bad
    hz = np.abs(mr.h_of(ms[1][good], x[ms[0]][good], ms[4][good])).max(axis=1) + np.abs(ms[2][good]).max(axis=1)
    sb = np.abs(ms[3][good]).max(axis=1) * hz
    sa = np.sqrt(np.abs(want[0][good]).max(axis=1))
    worst = 0.0
    for g, w, sc in zip(got, want, (sa * sa, sa * sb, sb * sb)):
        g, w = g[good].reshape(len(sc), -1), w[good].reshape(len(sc), -1)
        worst = max(worst, float(np.max(np.abs(g - w) / sc[:, None])))
    print(f"K12 against the numpy statement: worst {worst:.1e} of the scale each field is formed at")
    assert worst <= 1e-13


def realisations(torch, oracle, model, N, K, seed, clean=False):
    """N realisations of one K-keyframe trajectory (the construction of test_update_filter._filter_and_smoother): the truth by
    predict_state from clean IMU samples, samples with white noise and bias random walks (clean: none, so the records are exact at
    the truth), records preintegrated at x_hat_0's biases, the dead-reckoned initial states and the prior (Sigma_0^-1 at x_hat_0 =
    the truth perturbed by a draw of Sigma_0; clean: x_hat_0 = the truth).  Returns dict(truth [N,K,16], Sig0, xh0 [N,16], and the
    device tensors rec, lin, recK, linK, X0 [N*K,16], prior)."""
    from cpi_b200 import factor, preint
    from test_propagate import random_cov as rc
    rng = np.random.default_rng(seed)
    draw = (lambda size, scale=1.0: np.zeros(size)) if clean else (lambda size, scale=1.0: rng.normal(0.0, scale, size))
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
        clean_k = np.concatenate([w_true[k] + x_true[k, 4:7], a_true[k] + x_true[k, 10:13], dt[k][:, None]], axis=1)[None]
        x_true[k + 1] = oracle.predict_state(model, x_true[k:k + 1], preint.preintegrate_host(model, clean_k, lin_t, synth.SIGMAS, 0, ns=ns), lin_t)[0]
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
    dl = _dev(torch, lin.reshape(-1, 13))
    rec = preint.preintegrate(model, _dev(torch, samples.reshape(N * (K - 1), ns, 7)), dl, synth.SIGMAS, 0, ns=ns)
    X0 = torch.empty((N, K, 16), dtype=torch.float64, device="cuda")
    X0[:, 0] = _dev(torch, xh0)
    recK, linK = rec.view(N, K - 1, -1), dl.view(N, K - 1, 13)
    for k in range(K - 1):
        X0[:, k + 1] = factor.predict_state(model, X0[:, k].contiguous(), recK[:, k].contiguous(), linK[:, k].contiguous())
    Lam0 = np.linalg.inv(Sig0); Lam0 = 0.5 * (Lam0 + Lam0.T)
    prior = (_dev(torch, np.repeat(vec(Lam0[None]), N, axis=0)), _dev(torch, np.zeros((N, 15))), _dev(torch, np.zeros(N)), _dev(torch, xh0))
    return dict(truth=truth, Sig0=Sig0, xh0=xh0, rec=rec, lin=dl, recK=recK, linK=linK, X0=X0.reshape(N * K, 16), prior=prior)


def _exact_measurements(rng, truth, kinds, sigma=0.01):
    """One measurement of each kind in `kinds` on every state, noise-free (z = h(truth)); two directions per state for DIRECTION."""
    N = len(truth)
    idx, kind, aux = [], [], []
    for k in kinds:
        reps = 2 if k == mr.DIRECTION else 1
        for _ in range(reps):
            idx.append(np.arange(N)); kind.append(np.full(N, k, dtype=np.int32))
            a = rng.normal(size=(N, 3)) * (0.8 if k == mr.POSITION else 1.0)
            aux.append(a / np.linalg.norm(a, axis=1, keepdims=True) if k == mr.DIRECTION else a)
    idx, kind, aux = np.concatenate(idx).astype(np.int64), np.concatenate(kind), np.concatenate(aux)
    M = len(idx)
    si = np.tile((np.eye(3) / sigma).reshape(9), (M, 1))
    return idx, kind, mr.h_of(kind, truth[idx], aux), si, aux


def _rotate(oracle, rng, X, angle):
    d = np.zeros((len(X), 15))
    ax = rng.normal(size=(len(X), 3)); ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    d[:, 0:3] = angle * ax
    d[:, 12:15] = rng.normal(size=(len(X), 3)) * 0.1
    return oracle.retract(X, d)


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_lm_recovers_the_truth_from_exact_measurements(cuda, oracle, model):
    """Chains whose records are exact at the truth (noise-free IMU samples, records preintegrated at the true biases), a prior at the
    truth, and noise-free lever-arm position, body-velocity and direction measurements on every keyframe, started 0.3 rad off in
    attitude (and 0.1 m in position): chains_lm returns to the truth within 1e-11 in retract coordinates, per component (measured at
    most 5.7e-13 on an H100); with all three
    kinds, and with lever-arm position or body velocity next to the directions."""
    from cpi_b200 import factor
    torch = cuda
    N, K = 6, 12
    r = realisations(torch, oracle, model, N, K, 30 + model, clean=True)
    truth = r["truth"].reshape(N * K, 16)
    rng = np.random.default_rng(31 + model)
    params = capi.LMParams(absolute_error_tol=0.0, relative_error_tol=1e-14, max_iterations=100)
    for kinds in (KINDS, (mr.POSITION, mr.DIRECTION), (mr.VELOCITY_BODY, mr.DIRECTION)):
        ms = _exact_measurements(rng, truth, kinds)
        out = factor.chains_lm(model, _dev(torch, _rotate(oracle, rng, truth, 0.3)), r["rec"], r["lin"], K, prior=r["prior"],
                               measurements=_ms_dev(torch, ms), params=params)
        Xs, st = out[0].cpu().numpy(), out[3].cpu().numpy()
        err = np.abs(local(truth, Xs)).max()
        print(f"model {model} kinds {kinds}: from 0.3 rad, {err:.1e} off the truth, statuses {np.bincount(st, minlength=5)}")
        assert np.all(st != capi.LM_NONFINITE) and err <= 1e-11, (kinds, err)


@pytest.mark.gpu
@pytest.mark.parametrize("loss", [None, capi.LOSS_HUBER, capi.LOSS_CAUCHY])
def test_lm_step_is_the_dense_gauss_newton_step(cuda, oracle, loss):
    """One chains_lm_step with measurements (and state priors, and a robust loss on the measurements) equals the dense damped step
    of the numpy system with every measurement linearised by linearize_ref and reweighted by the IRLS statement: within 50x the
    distance of a plain fp64 dense solve to the refined truth (floor 1e-13); the cost before the step to 1e-10."""
    from cpi_b200 import factor
    torch = cuda
    rng = np.random.default_rng(40)
    sizes = [1, 4, 9, 2, 17, 1, 12]
    model = 1
    X, rec, L, offs, prior, per = make_problem(oracle, model, sizes, 41, large=True, with_prior=True)
    ms = mr.random_measurements(rng, X, 60, sigma=0.05)
    M = len(ms[0])
    code = None if loss is None else np.full(M, loss, dtype=np.int32)
    kk = np.full(M, 1.5)
    lam = 1e-5
    dX, dR, dL = _dev(torch, X), _dev(torch, rec), _dev(torch, L)
    from test_chains_lm import dev_prior
    new, dx, cost = factor.chains_lm_step(model, dX, dR, dL, _dev(torch, offs), prior=dev_prior(torch, prior), lam=lam,
                                          measurements=_ms_dev(torch, ms),
                                          measurement_loss=None if loss is None else (_dev(torch, code), _dev(torch, kk)))
    dx, cost = dx.cpu().numpy(), cost.cpu().numpy()
    e, H1, H2 = factor.factor_eval(model, dX, dR, dL, *_chain_idx(torch, offs))
    Gh = [t.cpu().numpy() for t in factor.factor_hessian(model, dR, e, H1, H2)]
    info, rhs, f = mr.linearize_ref(ms[1], X[ms[0]], ms[2], ms[3], ms[4])
    if loss is not None:
        info, rhs, f = robust_ref(code, kk, info, rhs, f)
    for c, (Xc, r, l) in enumerate(per):
        f0, S = int(offs[c] - c), len(Xc)
        sel = np.flatnonzero((ms[0] >= offs[c]) & (ms[0] < offs[c + 1]))
        sps = [(int(ms[0][q] - offs[c]), info[q], rhs[q], f[q], X[ms[0][q]]) for q in sel]
        A, b, cur = _np_system(oracle, model, Xc, r, l, prior[c], sps, blocks=[g[f0:f0 + S - 1] for g in Gh])
        A[np.diag_indices_from(A)] += lam * np.clip(np.diag(A), 1e-6, 1e32)
        xt, x64 = _dense_truth(A, b)
        dd = dx[offs[c]:offs[c + 1]].reshape(-1)
        nt = np.linalg.norm(xt)
        e_dev, e64 = np.linalg.norm(dd - xt) / nt, np.linalg.norm(x64 - xt) / nt
        assert e_dev <= 50 * max(e64, 1e-13), (c, e_dev, e64)
        assert abs(cost[c] - cur) <= 1e-10 * max(abs(cur), 1.0), (c, cost[c], cur)


@pytest.mark.gpu
def test_no_measurements_is_bitwise_the_plain_calls(cuda, oracle):
    """measurements=None and an empty list give bitwise the results of the calls without the argument."""
    from cpi_b200 import factor
    from test_chains_lm import dev_prior
    torch = cuda
    X, rec, L, offs, pri, _ = make_problem(oracle, 1, [1, 4, 9, 2, 30, 17], 7, with_prior=True)
    a = (_dev(torch, X), _dev(torch, rec), _dev(torch, L), _dev(torch, offs))
    i64 = dict(dtype=torch.int64, device="cuda")
    f64 = dict(dtype=torch.float64, device="cuda")
    empty = (torch.zeros(0, **i64), torch.zeros(0, dtype=torch.int32, device="cuda"), torch.zeros((0, 3), **f64), torch.zeros((0, 9), **f64),
             torch.zeros((0, 3), **f64))
    for fn in (factor.chains_lm_step, factor.chains_lm, factor.chains_marginals):
        ref = fn(1, *a, prior=dev_prior(torch, pri))
        for ms in (None, empty):
            got = fn(1, *a, prior=dev_prior(torch, pri), measurements=ms)
            assert all((u is None and v is None) or torch.equal(u, v) for u, v in zip(ref, got)), fn.__name__


@pytest.mark.gpu
def test_position_without_lever_arm_is_the_state_prior_route(cuda, oracle):
    """chains_lm with POSITION measurements at aux = 0 and with the same fixes as state priors (W = S^T S on p, x_bar = the state with
    p = z): the same statuses and final states to rounding (1e-13 of the position scale; measured 6.9e-15); chains_marginals to 1e-14
    relative (measured bitwise: both routes fold the same S^T S)."""
    from cpi_b200 import factor
    from test_chains_lm import dev_prior
    torch = cuda
    rng = np.random.default_rng(50)
    X, rec, L, offs, pri, _ = make_problem(oracle, 1, [1, 8, 15, 3, 25], 51, with_prior=True)
    ms = list(mr.random_measurements(rng, X, 40, kinds=(mr.POSITION,), sigma=0.02))
    ms[4][:] = 0.0
    S = mr.sqrt_mat(ms[3])
    W = np.zeros((40, 15, 15)); W[:, 12:15, 12:15] = S.transpose(0, 2, 1) @ S
    xb = X[ms[0]].copy(); xb[:, 13:16] = ms[2]
    sp = (_dev(torch, ms[0]), _dev(torch, vec(W)), None, None, _dev(torch, xb))
    a = (_dev(torch, X), _dev(torch, rec), _dev(torch, L), _dev(torch, offs))
    r1 = factor.chains_lm(1, *a, prior=dev_prior(torch, pri), measurements=_ms_dev(torch, ms))
    r2 = factor.chains_lm(1, *a, prior=dev_prior(torch, pri), state_priors=sp)
    X1, X2 = r1[0].cpu().numpy(), r2[0].cpu().numpy()
    assert torch.equal(r1[3], r2[3])
    err = np.abs(local(X2, X1)).max() / max(1.0, np.abs(X2[:, 13:16]).max())
    c1, _ = factor.chains_marginals(1, r1[0], a[1], a[2], a[3], prior=dev_prior(torch, pri), measurements=_ms_dev(torch, ms))
    c2, _ = factor.chains_marginals(1, r1[0], a[1], a[2], a[3], prior=dev_prior(torch, pri),
                                    state_priors=(sp[0], sp[1], None, None, _dev(torch, np.c_[X1[ms[0]][:, :13], ms[2]])))
    c1, c2 = c1.cpu().numpy(), c2.cpu().numpy()
    ec = np.max(np.abs(c1 - c2)) / np.abs(c2).max()
    print(f"measurements vs state priors: states {err:.1e}, marginals {ec:.1e}")
    assert err <= 1e-13 and ec <= 1e-14


@pytest.mark.gpu
def test_marginals_and_marginalisation_take_the_linearised_blocks(cuda, oracle):
    """chains_marginals with measurements equals chains_marginals with measurements_linearize's state priors at the same states
    (the same blocks, folded the same way), and chain_marginalize with those state priors equals the Schur complement of the numpy
    blocks with the measurements of eliminated states added to G11 / g1 / f."""
    from cpi_b200 import factor
    from test_chains_lm import dev_prior
    from test_marginalize import marginalize_ref
    torch = cuda
    rng = np.random.default_rng(60)
    sizes = [6, 9, 12]
    X, rec, L, offs, pri, _ = make_problem(oracle, 1, sizes, 61, with_prior=True)
    ms = mr.random_measurements(rng, X, 30)
    a = (_dev(torch, X), _dev(torch, rec), _dev(torch, L), _dev(torch, offs))
    dms = _ms_dev(torch, ms)
    info, rhs, f, sp = factor.measurements_linearize(a[0], dms)
    c1, x1 = factor.chains_marginals(1, *a, prior=dev_prior(torch, pri), measurements=dms, cross=True)
    c2, x2 = factor.chains_marginals(1, *a, prior=dev_prior(torch, pri), state_priors=sp, cross=True)
    assert torch.allclose(c1, c2, rtol=1e-12, atol=0) and torch.allclose(x1, x2, rtol=1e-12, atol=1e-12 * float(x2.abs().max()))
    e, H1, H2 = factor.factor_eval(1, a[0], a[1], a[2], *_chain_idx(torch, offs))
    G = factor.factor_hessian(1, a[1], e, H1, H2)
    m = 3
    pr = dev_prior(torch, pri)[:3]
    got = [t.cpu().numpy() for t in factor.chain_marginalize(*G, a[3], m, prior=pr, state_priors=sp)]
    Gh = [t.cpu().numpy() for t in G]
    inf_, rhs_, f_ = (t.cpu().numpy() for t in (info, rhs, f))
    for c in range(len(sizes)):
        f0 = int(offs[c] - c)
        blk = [g[f0:f0 + sizes[c] - 1].copy() for g in Gh]
        for q in np.flatnonzero((ms[0] >= offs[c]) & (ms[0] < offs[c] + m)):
            k = int(ms[0][q] - offs[c])
            blk[0][k] += inf_[q]; blk[3][k] += rhs_[q]; blk[5][k] += f_[q]
        want = marginalize_ref(mat(blk[0]), mat(blk[1]), mat(blk[2]), blk[3], blk[4], blk[5], m, prior=pri[c][:3], jacobi=True)
        sc = np.abs(want[0]).max()
        assert np.allclose(mat(got[0][c:c + 1])[0], want[0], rtol=0, atol=1e-8 * sc), c
        assert np.allclose(got[1][c], want[1], rtol=0, atol=1e-8 * np.abs(want[1]).max()), c


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_marginals_are_the_dense_inverse_of_the_numpy_system(cuda, oracle, model):
    """chains_marginals with measurements (ragged chains, single-state ones among them, a chain prior) against the refined dense
    inverse of the system assembled in numpy: the oracle's factors, the prior moved by prior_at_ref and every measurement
    linearised by linearize_ref on its state.  Diagonal and cross blocks within 50x the plain fp64 dense inverse's distance to the
    refined one (floor 1e-13), in units of the truth's diagonal: the gate of test_chain_marginals.py."""
    from cpi_b200 import factor
    from test_chain_marginals import inv_truth, scaled
    from test_chains_lm import dev_prior
    torch = cuda
    rng = np.random.default_rng(80 + model)
    sizes = [1, 5, 9, 2, 16, 1, 12]
    X, rec, L, offs, pri, per = make_problem(oracle, model, sizes, 81 + model, with_prior=True)
    ms = mr.random_measurements(rng, X, 50, sigma=0.05)
    cov, cr = factor.chains_marginals(model, _dev(torch, X), _dev(torch, rec), _dev(torch, L), _dev(torch, offs), prior=dev_prior(torch, pri),
                                      measurements=_ms_dev(torch, ms), cross=True)
    cov, cr = mat(cov.cpu().numpy()), mat(cr.cpu().numpy())
    assert np.array_equal(cov, cov.transpose(0, 2, 1))
    info, rhs, f = mr.linearize_ref(ms[1], X[ms[0]], ms[2], ms[3], ms[4])
    ed = ep = 0.0
    for c, (Xc, r, l) in enumerate(per):
        lo, hi = int(offs[c]), int(offs[c + 1])
        sel = np.flatnonzero((ms[0] >= lo) & (ms[0] < hi))
        sps = [(int(ms[0][q] - lo), info[q], rhs[q], f[q], X[ms[0][q]]) for q in sel]
        A, _, _ = _np_system(oracle, model, Xc, r, l, pri[c], sps)
        T, P64 = inv_truth(A)
        _, err = scaled(None, T)
        for k in range(hi - lo):
            blocks = [(cov[lo + k], k, k)] + ([(cr[lo - c + k], k, k + 1)] if k + 1 < hi - lo else [])
            for blk, I, J in blocks:
                ed = max(ed, err(blk, I, J))
                ep = max(ep, err(P64[15 * I:15 * I + 15, 15 * J:15 * J + 15], I, J))
    print(f"model {model}: chains_marginals with measurements against the numpy system's refined inverse: device {ed:.2e}, "
          f"plain fp64 dense inverse {ep:.2e} (units of the diagonal)")
    assert ed <= 50 * max(ep, 1e-13), (ed, ep)
