"""The iterated filter update by attitude-dependent measurements with Huber and Cauchy losses
(cpi_state_update_measurements_iterated_batch, kernel K13, factor.update_measurements_iterated; DESIGN.md section 3m) against its
numpy statement tests/update_iter_ref.py, against K11 and against the smoother's library calls on single-state chains, and its value
over K11 for a filter with a poor heading and for outlying GNSS fixes."""
import ctypes

import numpy as np
import pytest

import measurement_ref as mr
import update_iter_ref as ir
from cpi_b200 import capi
from test_marginalize import local, mat, vec
from test_measurements import _filters
from update_ref import errors, retract

LEVER = np.array([0.5, 0.2, 1.0])                                     # the GNSS antenna in the IMU frame, metres
P = lambda a: ctypes.c_void_p(a.ctypes.data)


def _losses(rng, M):
    """A mix of Gaussian, Huber and Cauchy codes with thresholds between 0.5 and 2 standard deviations."""
    return rng.integers(0, 3, size=M).astype(np.int32), rng.uniform(0.5, 2.0, size=M)


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------

def test_one_iteration_is_the_k11_statement():
    """At max_iterations = 1 with Gaussian losses the statement is update_meas_ref (K11's statement) to rounding, in both forms."""
    rng = np.random.default_rng(1)
    counts = np.array([1, 2, 3, 4, 0, 2, 1, 3])
    x, cov, off, owner, kind, z, si, aux = _filters(rng, len(counts), counts)
    k11 = mr.update_meas_ref(x, cov, off, kind, z, si, aux)
    for info in (False, True):
        r = ir.update_iter_ref(x, cov, off, kind, z, si, aux, max_iterations=1, tol=np.inf, info=info)
        eb, ex, eg = errors((k11[0], k11[1], k11[3]), (r[0], r[1], r[2]), x)
        assert eb.max() <= 1e-10 and ex.max() <= 1e-10 and eg.max() <= 1e-10, (info, eb.max(), ex.max(), eg.max())
        assert np.array_equal(r[3], np.ones(len(counts))) and np.array_equal(r[4], np.minimum(counts, 1))


def test_convergence_is_stationary_with_the_dense_covariance():
    """At convergence (tol = 1e-13) with a loss mix and outliers: the gradient Sigma^-1 local(x_hat, x*) + sum om A^T b vanishes relative
    to its terms' scale, and Sigma+ is the dense (Sigma^-1 + sum om A^T A)^-1 at the last linearisation."""
    rng = np.random.default_rng(2)
    counts = rng.integers(1, 5, size=24)
    x, cov, off, owner, kind, z, si, aux = _filters(rng, len(counts), counts)
    z[::4] += 0.3
    code, k = _losses(rng, len(kind))
    r = ir.update_iter_ref(x, cov, off, kind, z, si, aux, code, k, max_iterations=60, tol=1e-13)
    grad = ir.stationarity(x, cov, r[0], off, kind, z, si, aux, code, k)
    dense = ir.covariance_at(cov, r[5], off, kind, z, si, aux, code, k)
    sd = np.sqrt(np.diagonal(mat(dense), axis1=1, axis2=2))
    ec = np.max(np.abs(mat(r[1]) - mat(dense)) / (sd[:, :, None] * sd[:, None, :]))
    print(f"statement at convergence: {int((r[3] == 1).sum())} of {len(counts)} converged, iterations up to {r[4].max()}, "
          f"gradient {grad.max():.1e}, Sigma+ against the dense inverse {ec:.1e}")
    assert np.all(r[3] == 1) and grad.max() <= 1e-8 and ec <= 1e-10


def test_argument_validation_without_gpu():
    """The C ABI rejects a negative count, max_iterations < 1, a NaN or negative tol, one of loss / loss_k alone, NULL required pointers
    and aliased outputs before any CUDA call; n = 0 is a no-op.  The wrapper rejects max_iterations, tol and host tensors first."""
    import torch

    from cpi_b200 import factor
    lib = capi.load()
    buf = [np.zeros(8 * 225) for _ in range(16)]
    p = [P(b) for b in buf]
    upd = lambda n, *a, mi=3, tol=1e-9: lib.cpi_state_update_measurements_iterated_batch(n, *a[:10], mi, tol, *a[10:], None)
    ok = p[0:7] + [None, None, None] + [p[8], p[9], p[10], p[11], p[12]]
    assert upd(-1, *ok) == -1 and b"negative" in lib.cpi_last_error()
    assert upd(0, *[None] * 15) == 0
    for mi in (0, -2):
        assert upd(2, *ok, mi=mi) == -1 and b"max_iterations" in lib.cpi_last_error()
    for tol in (float("nan"), -1e-9):
        assert upd(2, *ok, tol=tol) == -1 and b"tol" in lib.cpi_last_error()
    for k in (7, 8):
        bad = list(ok); bad[k] = p[13]
        assert upd(2, *bad) == -1 and b"both" in lib.cpi_last_error(), k
    for k in (0, 1, 2, 3, 4, 5, 6, 10, 11):
        bad = list(ok); bad[k] = None
        assert upd(2, *bad) == -1 and b"null" in lib.cpi_last_error(), k
    bad = list(ok); bad[7], bad[8] = p[13], p[14]
    bad[12] = p[14]
    assert upd(2, *bad) == -1 and b"overlap" in lib.cpi_last_error()
    bad = list(ok); bad[11] = p[8]
    assert upd(2, *bad) == -1 and b"overlap" in lib.cpi_last_error()
    bad = list(ok); bad[14] = p[11]
    assert upd(2, *bad) == -1 and b"overlap" in lib.cpi_last_error()
    f64 = dict(dtype=torch.float64)
    xs, cs = torch.zeros(4, 16, **f64), torch.zeros(4, 225, **f64)
    ms = (torch.tensor([0, 3]), torch.tensor([1, 3], dtype=torch.int32), torch.zeros(2, 3, **f64), torch.zeros(2, 9, **f64),
          torch.zeros(2, 3, **f64))
    for mi in (0, 2.0, True, None):
        with pytest.raises(ValueError, match="max_iterations"):
            factor.update_measurements_iterated(xs, cs, ms, max_iterations=mi)
    for tol in (float("nan"), -1.0, None, "1e-9"):
        with pytest.raises(ValueError, match="tol"):
            factor.update_measurements_iterated(xs, cs, ms, tol=tol)
    with pytest.raises(ValueError, match="CUDA"):
        factor.update_measurements_iterated(xs, cs, ms)
    with pytest.raises(ValueError, match="tensor"):
        factor.update_measurements_iterated(xs.numpy(), cs, ms)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------

def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _run(torch, x, cov, owner, kind, z, si, aux, loss=None, gate=None, max_iterations=10, tol=1e-9):
    from cpi_b200 import factor
    g = _dev(torch, gate) if isinstance(gate, np.ndarray) else gate
    ms = (_dev(torch, owner.astype(np.int64)), _dev(torch, kind), _dev(torch, z), _dev(torch, si), _dev(torch, aux))
    lo = None if loss is None else (_dev(torch, loss[0].astype(np.int32)), _dev(torch, loss[1]))
    out = factor.update_measurements_iterated(_dev(torch, x), _dev(torch, cov), ms, gate=g, measurement_loss=lo,
                                              max_iterations=max_iterations, tol=tol)
    torch.cuda.synchronize()
    return tuple(t.cpu().numpy() for t in out)


def _k11(torch, x, cov, owner, kind, z, si, aux, gate=None):
    from cpi_b200 import factor
    g = _dev(torch, gate) if isinstance(gate, np.ndarray) else gate
    ms = (_dev(torch, owner.astype(np.int64)), _dev(torch, kind), _dev(torch, z), _dev(torch, si), _dev(torch, aux))
    out = factor.update_measurements(_dev(torch, x), _dev(torch, cov), ms, gate=g)
    torch.cuda.synchronize()
    return tuple(t.cpu().numpy() for t in out)


def _mixed(seed, n=400):
    """n filters with 0 to 4 measurements of every kind, some 6-sigma outliers and a loss mix."""
    rng = np.random.default_rng(seed)
    counts = rng.integers(0, 5, size=n)
    x, cov, off, owner, kind, z, si, aux = _filters(rng, n, counts)
    z[::7] += 0.3
    return rng, counts, x, cov, off, owner, kind, z, si, aux, _losses(rng, len(kind))


@pytest.mark.gpu
def test_kernel_is_the_statement(cuda):
    """400 filters, 0 to 4 measurements of every kind, Gaussian, Huber and Cauchy losses, owners shuffled.  tol = 0 with 1, 3 and 8
    iterations: every field within 20x the distance between the square-root and the information statements (floor 1e-13), and the
    same iteration counts.  tol = 1e-9: status and iterations equal the statement's on every filter whose stopping tests all lie
    further than 1e-6 (relative) from the threshold.  K13's extended-precision gate on the measurement stress batch is
    tests/test_measurements_precision.py."""
    torch = cuda
    rng, counts, x, cov, off, owner, kind, z, si, aux, loss = _mixed(40)
    perm = rng.permutation(len(owner))
    sh = lambda *a: tuple(t[perm] for t in a)
    some = counts > 0
    for T in (1, 3, 8):
        got = _run(torch, x, cov, *sh(owner, kind, z, si, aux), loss=sh(*loss), max_iterations=T, tol=0.0)
        r = ir.update_iter_ref(x, cov, off, kind, z, si, aux, *loss, max_iterations=T, tol=0.0)
        i = ir.update_iter_ref(x, cov, off, kind, z, si, aux, *loss, max_iterations=T, tol=0.0, info=True)
        eb, ex, eg = errors((r[0][some], r[1][some], r[2][some]), (got[0][some], got[1][some], got[2][some]), x[some])
        nb, nx, ng = errors((r[0][some], r[1][some], r[2][some]), (i[0][some], i[1][some], i[2][some]), x[some])
        print(f"K13 at {T} iterations vs update_iter_ref: cov {eb.max():.1e}, state {ex.max():.1e}, gamma {eg.max():.1e}; "
              f"information form: {nb.max():.1e}, {nx.max():.1e}, {ng.max():.1e}")
        assert eb.max() <= 20 * max(nb.max(), 1e-13) and ex.max() <= 20 * max(nx.max(), 1e-13) and eg.max() <= 20 * max(ng.max(), 1e-13)
        assert np.array_equal(got[4], r[4]) and np.array_equal(got[3], r[3]), T
    got = _run(torch, x, cov, *sh(owner, kind, z, si, aux), loss=sh(*loss), max_iterations=10, tol=1e-9)
    r = ir.update_iter_ref(x, cov, off, kind, z, si, aux, *loss, max_iterations=10, tol=1e-9)
    clear = r[6] > 1e-6
    print(f"tol 1e-9: {int((~clear).sum())} of {len(counts)} filters excluded (a stopping test within 1e-6 of the threshold); "
          f"status counts {np.bincount(got[3], minlength=3).tolist()}, iterations up to {got[4].max()}")
    assert np.array_equal(got[3][clear], r[3][clear]) and np.array_equal(got[4][clear], r[4][clear])


@pytest.mark.gpu
def test_one_iteration_is_k11(cuda):
    """max_iterations = 1, tol = +inf and no loss against K11 on the same inputs.  K13 performs K11's operations in K11's order, but
    ptxas contracts the unfused products of the retraction differently in the two kernels, so the states are not bitwise K11's: every
    field lies within K11's numpy gate, 20x the distance between the square-root and the information statements (floor 1e-13).
    Status 1 and one iteration on every filter with measurements, none on the others."""
    torch = cuda
    rng, counts, x, cov, off, owner, kind, z, si, aux, _ = _mixed(41)
    got = _run(torch, x, cov, owner, kind, z, si, aux, max_iterations=1, tol=float("inf"))
    k11 = _k11(torch, x, cov, owner, kind, z, si, aux)
    some = counts > 0
    differ = [int(np.sum(np.any(a.reshape(len(a), -1) != b.reshape(len(b), -1), axis=1))) for a, b in zip(got[:3], k11[:3])]
    r = mr.update_meas_ref(x, cov, off, kind, z, si, aux)
    i = mr.update_meas_info(x, cov, off, kind, z, si, aux)
    eb, ex, eg = errors((k11[0][some], k11[1][some], k11[2][some]), (got[0][some], got[1][some], got[2][some]), x[some])
    nb, nx, ng = errors((r[0][some], r[1][some], r[3][some]), (i[0][some], i[1][some], i[3][some]), x[some])
    print(f"K13 at one iteration against K11: {differ} of {int(some.sum())} filters differ in state / cov / gamma; cov {eb.max():.1e}, "
          f"state {ex.max():.1e}, gamma {eg.max():.1e}; information form: {nb.max():.1e}, {nx.max():.1e}, {ng.max():.1e}")
    assert eb.max() <= 20 * max(nb.max(), 1e-13) and ex.max() <= 20 * max(nx.max(), 1e-13) and eg.max() <= 20 * max(ng.max(), 1e-13)
    assert np.array_equal(got[0][~some], k11[0][~some]) and np.array_equal(got[1][~some], k11[1][~some])
    assert np.all(got[3] == 1) and np.array_equal(got[4], np.minimum(counts, 1))


@pytest.mark.gpu
def test_loss_equivalences(cuda):
    """Every code LOSS_GAUSSIAN is bitwise measurement_loss = None; Huber with k above every whitened residual at every iterate
    (weight exactly 1) is bitwise the Gaussian run."""
    torch = cuda
    rng, counts, x, cov, off, owner, kind, z, si, aux, _ = _mixed(42)
    M = len(kind)
    free = _run(torch, x, cov, owner, kind, z, si, aux, max_iterations=5, tol=1e-12)
    gauss = _run(torch, x, cov, owner, kind, z, si, aux, loss=(np.zeros(M, np.int32), np.zeros(M)), max_iterations=5, tol=1e-12)
    huber = _run(torch, x, cov, owner, kind, z, si, aux, loss=(np.ones(M, np.int32), np.full(M, 1e4)), max_iterations=5, tol=1e-12)
    assert all(np.array_equal(a, b) for a, b in zip(free, gauss))
    assert all(np.array_equal(a, b) for a, b in zip(free, huber))


@pytest.mark.gpu
def test_gating_isolation_cap_and_determinism(cuda):
    """The gate skips exactly the filters with nis > gate (bitwise copies, status 0) and leaves the others bitwise the ungated run; a
    non-SPD cov or a NaN in z in one filter of ten leaves the other nine bitwise the clean run; a filter stopped by the cap reports
    status 2; two runs give the same bits and Sigma+ is exactly symmetric."""
    torch = cuda
    rng, counts, x, cov, off, owner, kind, z, si, aux, loss = _mixed(43, n=64)
    z[::5] += 1.0
    free = _run(torch, x, cov, owner, kind, z, si, aux, loss=loss)
    again = _run(torch, x, cov, owner, kind, z, si, aux, loss=loss)
    assert all(np.array_equal(a, b) for a, b in zip(free, again))
    assert np.array_equal(mat(free[1]), mat(free[1]).transpose(0, 2, 1))
    gate = np.full(len(counts), 16.0)
    xo, co, g, st, it = _run(torch, x, cov, owner, kind, z, si, aux, loss=loss, gate=gate)
    skip = st == 0
    assert skip.any() and (~skip).any() and np.array_equal(skip, free[2] > gate) and np.array_equal(g, free[2])
    assert np.array_equal(xo[skip], x[skip]) and np.array_equal(co[skip], cov[skip]) and np.all(it[skip] == 1)
    assert all(np.array_equal(u[~skip], v[~skip]) for u, v in zip((xo, co, st, it), (free[0], free[1], free[3], free[4])))
    capped = _run(torch, x, cov, owner, kind, z, si, aux, loss=loss, max_iterations=2, tol=1e-15)
    assert np.all(capped[3][counts > 0] == 2) and np.all(capped[4][counts > 0] == 2)
    m = int(off[10])
    x10, c10 = x[:10], cov[:10]
    o10, k10, z10, s10, a10, l10 = owner[:m], kind[:m], z[:m], si[:m], aux[:m], (loss[0][:m], loss[1][:m])
    clean = _run(torch, x10, c10, o10, k10, z10, s10, a10, loss=l10)
    f = int(np.flatnonzero(counts[:10] > 0)[0])
    j = int(off[f])
    for what in ("cov", "z"):
        c2, z2 = c10.copy(), z10.copy()
        if what == "cov":
            S = mat(c2[f:f + 1])[0]; S[3, 3] = -1.0; c2[f] = vec(S[None])[0]
        else:
            z2[j, 1] = np.nan
        got = _run(torch, x10, c2, o10, k10, z2, s10, a10, loss=l10)
        keep = np.arange(10) != f
        assert all(np.array_equal(u[keep], v[keep]) for u, v in zip(got, clean)), what
        assert np.isnan(got[0][f]).any() and got[3][f] == 2, what


def _single_state_steps(torch, x, cov, off, owner, kind, z, si, aux, loss, T):
    """T Gauss-Newton steps at lambda = 0 through the smoother's library calls on single-state chains: the prior (Sigma^-1, x_hat) a
    state prior moved to the iterate by prior_at, the measurements linearised there by measurements_linearize and reweighted by
    state_priors_robust, both folded onto the chain prior, then chains_assemble, chains_solve and retract.  Sigma+ is chains_covariance
    of the last linearisation's system.  Returns (x_T, Sigma+)."""
    from cpi_b200 import factor
    n = len(x)
    Si = np.linalg.inv(mat(cov)); Si = 0.5 * (Si + Si.transpose(0, 2, 1))
    f64 = dict(dtype=torch.float64, device="cuda")
    dSi, dxh = _dev(torch, vec(Si)), _dev(torch, x)
    ms = (_dev(torch, owner.astype(np.int64)), _dev(torch, kind), _dev(torch, z), _dev(torch, si), _dev(torch, aux))
    dl = (_dev(torch, loss[0].astype(np.int32)), _dev(torch, loss[1]))
    offs, sp_off = torch.arange(n + 1, dtype=torch.int64, device="cuda"), _dev(torch, off)
    e0, e1 = torch.empty((0, 225), **f64), torch.empty((0, 15), **f64)
    X = dxh.clone()
    for _ in range(T):
        pr, pf = factor.prior_at(dSi, torch.zeros((n, 15), **f64), torch.zeros(n, **f64), dxh, X)
        info, rhs, f, _ = factor.measurements_linearize(X, ms)
        iw, rw, fw = factor.state_priors_robust(dl[0], dl[1], info, rhs, f)
        pi = dSi.clone()
        factor.state_priors_fold(offs, sp_off, iw, rw, fw, prior_info=pi, prior_rhs=pr, prior_f=pf)
        D, E, r = factor.chains_assemble(e0, e0, e0, e1, e1, 1, 0.0, pi, pr, n_chains=n)
        X = factor.retract(X, factor.chains_solve(D, E, r, 1, n_chains=n))
    c, _ = factor.chains_covariance(D, E, 1, n_chains=n)
    torch.cuda.synchronize()
    return X.cpu().numpy(), c.cpu().numpy()


@pytest.mark.gpu
def test_against_the_smoother_library_calls(cuda):
    """Single-state chains iterated step by step at lambda = 0 through the smoother's library calls (with the loss mix): the states and
    Sigma+ after 1 and 4 steps agree with K13 within 20x the distance between the square-root and the information statements, floor
    1e-12, in the posterior's standard deviations."""
    torch = cuda
    rng = np.random.default_rng(44)
    counts = rng.integers(1, 5, size=96)
    x, cov, off, owner, kind, z, si, aux = _filters(rng, len(counts), counts)
    z[::7] += 0.3
    loss = _losses(rng, len(kind))
    for T in (1, 4):
        got = _run(torch, x, cov, owner, kind, z, si, aux, loss=loss, max_iterations=T, tol=0.0)
        xl, cl = _single_state_steps(torch, x, cov, off, owner, kind, z, si, aux, loss, T)
        r = ir.update_iter_ref(x, cov, off, kind, z, si, aux, *loss, max_iterations=T, tol=0.0)
        i = ir.update_iter_ref(x, cov, off, kind, z, si, aux, *loss, max_iterations=T, tol=0.0, info=True)
        sd = np.sqrt(np.diagonal(mat(r[1]), axis1=1, axis2=2))
        dg = sd[:, :, None] * sd[:, None, :]
        ex = float(np.max(np.abs(local(xl, got[0])) / sd))
        ex_np = float(np.max(np.abs(local(i[0], r[0])) / sd))
        ec = float(np.max(np.abs(mat(cl) - mat(got[1])) / dg))
        ec_np = float(np.max(np.abs(mat(i[1]) - mat(r[1])) / dg))
        print(f"{T} steps: K13 vs the library calls: state {ex:.1e} (numpy routes {ex_np:.1e}), Sigma+ {ec:.1e} (numpy routes {ec_np:.1e})")
        assert ex <= 20 * max(ex_np, 1e-12) and ec <= 20 * max(ec_np, 1e-12)


def _poor_heading(seed, N):
    """N filters whose prior has about 0.3 rad of yaw standard deviation (0.05 rad in roll and pitch, global frame), and truths drawn
    from it, x = retract(x_hat, delta), delta ~ N(0, Sigma).  Each takes one update of three measurements of its truth: lever-arm GNSS
    (l = LEVER, 1 cm), a magnetometer direction and the gravity direction (0.01 each).  Returns (x_hat, cov, truth, off, owner, kind,
    z, si, aux)."""
    rng = np.random.default_rng(seed)
    xh = np.zeros((N, 16))
    q = rng.normal(size=(N, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True); q[q[:, 3] < 0] *= -1
    xh[:, 0:4] = q
    xh[:, 4:16] = rng.normal(size=(N, 12)) * np.repeat([1e-3, 1.0, 1e-2, 10.0], 3)
    C = mr.rot(q)
    Sig = np.zeros((N, 15, 15))
    Sig[:, 0:3, 0:3] = C @ np.diag([0.05 ** 2, 0.05 ** 2, 0.3 ** 2]) @ C.transpose(0, 2, 1)
    for b, s in ((1, 1e-3), (2, 0.1), (3, 1e-2), (4, 0.1)):
        Sig[:, 3 * b:3 * b + 3, 3 * b:3 * b + 3] = np.eye(3) * s * s
    Sig = 0.5 * (Sig + Sig.transpose(0, 2, 1))
    truth = retract(xh, np.einsum("nij,nj->ni", np.linalg.cholesky(Sig), rng.normal(size=(N, 15))))
    mag = np.array([0.5, 0.0, 0.866]); mag /= np.linalg.norm(mag)
    kind = np.tile(np.array([mr.POSITION, mr.DIRECTION, mr.DIRECTION], dtype=np.int32), N)
    aux = np.tile(np.stack([LEVER, mag, np.array([0.0, 0.0, 1.0])]), (N, 1))
    owner = np.repeat(np.arange(N), 3)
    sig = np.tile([0.01, 0.01, 0.01], N)[:, None]
    si = (np.eye(3)[None] / sig[:, :, None]).transpose(0, 2, 1).reshape(-1, 9)
    z = mr.h_of(kind, truth[owner], aux) + rng.normal(size=(3 * N, 3)) * sig
    off = np.arange(N + 1, dtype=np.int64) * 3
    return xh, vec(Sig), truth, off, owner, kind, z, si, aux


def _nees(x, cov, truth):
    e = local(x, truth)
    return float(np.mean(np.einsum("ni,ni->n", e, np.linalg.solve(mat(cov), e[:, :, None])[:, :, 0])))


@pytest.mark.gpu
def test_poor_heading_value(cuda):
    """10 000 filters with about 0.3 rad of prior yaw standard deviation, one update by lever-arm GNSS, a magnetometer and gravity:
    K13 (tol 1e-10, cap 20) converges on every filter and its mean NEES lies in the two-sided 99.9 % chi^2_15 band for N; K11's lies
    above it (its single linearisation drops theta^2/2 of the lever arm and of the directions)."""
    from scipy.stats import chi2
    torch = cuda
    N = 10_000
    xh, cov, truth, off, owner, kind, z, si, aux = _poor_heading(90, N)
    xo, co, g, st, it = _run(torch, xh, cov, owner, kind, z, si, aux, max_iterations=20, tol=1e-10)
    k11 = _k11(torch, xh, cov, owner, kind, z, si, aux)
    lo, hi = chi2.ppf([0.0005, 0.9995], 15 * N) / N
    n13, n11 = _nees(xo, co, truth), _nees(k11[0], k11[1], truth)
    print(f"poor heading, {N} filters: K13 mean NEES {n13:.3f} ({int((st == 1).sum())} converged, iterations "
          f"{np.bincount(it).tolist()}), K11 mean NEES {n11:.3f}, band [{lo:.3f}, {hi:.3f}]")
    assert np.all(st == 1)
    assert lo <= n13 <= hi and n11 > hi


@pytest.mark.gpu
def test_outlying_gnss_value(cuda):
    """test_poor_heading_value's filters with 5 % of the GNSS fixes moved by 5 m: the RMS position error of K13 with Huber and with
    Cauchy losses (k = 3) on the GNSS rows lies below that of K13 with Gaussian losses.  The chi^2-gated K11's is printed beside them."""
    from scipy.stats import chi2
    torch = cuda
    N = 10_000
    xh, cov, truth, off, owner, kind, z, si, aux = _poor_heading(91, N)
    rng = np.random.default_rng(92)
    gnss = kind == mr.POSITION
    out = gnss & (rng.random(len(kind)) < 0.05)
    z[out] += 5.0 / np.sqrt(3)
    rms, info = {}, {}
    for name, code in (("gaussian", capi.LOSS_GAUSSIAN), ("huber", capi.LOSS_HUBER), ("cauchy", capi.LOSS_CAUCHY)):
        codes = np.where(gnss, code, capi.LOSS_GAUSSIAN).astype(np.int32)
        xo, co, g, st, it = _run(torch, xh, cov, owner, kind, z, si, aux, loss=(codes, np.full(len(codes), 3.0)), max_iterations=20,
                                 tol=1e-10)
        rms[name] = float(np.sqrt(np.mean(local(xo, truth)[:, 12:15] ** 2)))
        info[name] = np.bincount(st, minlength=3).tolist()
    k11 = _k11(torch, xh, cov, owner, kind, z, si, aux, gate=np.full(N, chi2.ppf(0.999, 9)))
    rms["gated K11"] = float(np.sqrt(np.mean(local(k11[0], truth)[:, 12:15] ** 2)))
    print(f"{int(out.sum())} outlying GNSS fixes of {N}: RMS position error " + ", ".join(f"{k} {v * 100:.2f} cm" for k, v in rms.items())
          + f"; K13 status counts {info}; K11 gated {int((k11[3] == 0).sum())}")
    assert rms["huber"] < rms["gaussian"] and rms["cauchy"] < rms["gaussian"]


@pytest.mark.gpu
def test_wrapper_validation_on_the_device(cuda):
    """factor.update_measurements_iterated rejects bad losses, a gate of the wrong length and NaN gates before any launch; an empty
    batch and filters without measurements launch nothing or are copied with status 1 and 0 iterations."""
    from cpi_b200 import factor
    torch = cuda
    f64 = dict(dtype=torch.float64, device="cuda")
    x, c = torch.zeros(4, 16, **f64), torch.zeros(4, 225, **f64)
    ms = (torch.tensor([0, 3], device="cuda"), torch.tensor([1, 3], dtype=torch.int32, device="cuda"), torch.zeros(2, 3, **f64),
          torch.zeros(2, 9, **f64), torch.zeros(2, 3, **f64))
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")
    before = capi.launch_count()
    for loss, msg in (((i32([0, 1]),), "measurement_loss is"), ((i32([0, 3]), torch.ones(2, **f64)), "loss codes"),
                      ((i32([1, 2]), torch.tensor([1.0, 0.0], **f64)), "threshold"),
                      ((i32([2, 2]), torch.tensor([1.0, float("inf")], **f64)), "threshold"),
                      ((torch.tensor([0, 1], device="cuda"), torch.ones(2, **f64)), "int32")):
        with pytest.raises(ValueError, match=msg):
            factor.update_measurements_iterated(x, c, ms, measurement_loss=loss)
    with pytest.raises(ValueError, match="needs measurements"):
        factor.update_measurements_iterated(x, c, None, measurement_loss=(i32([0, 1]), torch.ones(2, **f64)))
    with pytest.raises(ValueError, match="one entry per filter"):
        factor.update_measurements_iterated(x, c, ms, gate=torch.ones(3, **f64))
    for gate in (float("nan"), torch.tensor([1.0, float("nan"), 1.0, 1.0], **f64)):
        with pytest.raises(ValueError, match="NaN"):
            factor.update_measurements_iterated(x, c, ms, gate=gate)
    e = torch.empty((0, 16), **f64)
    out = factor.update_measurements_iterated(e, torch.empty((0, 225), **f64), None)
    assert capi.launch_count() == before and out[0].shape == (0, 16)
    rng = np.random.default_rng(45)
    xs, cs = _dev(torch, rng.normal(size=(4, 16))), _dev(torch, rng.normal(size=(4, 225)))
    xo, co, nis, st, it = factor.update_measurements_iterated(xs, cs, None)
    assert torch.equal(xo, xs) and torch.equal(co, cs) and bool((nis == 0).all()) and bool((st == 1).all()) and bool((it == 0).all())
