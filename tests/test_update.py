"""The filter's measurement update by direct state fixes (cpi_state_update_batch, kernel K10, factor.update; DESIGN.md section 3k).

The numpy statement is tests/update_ref.py's update_ref (the square-root form of the kernel); the CPU tests tie it to the dense
information form, the textbook Kalman gain and the plain-C oracle, and the GPU tests tie the kernel to it and to the existing
propagate, marginals and LM entry points.  The extended-precision gate is tests/test_update_precision.py."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest
from scipy.stats import binom

import update_ref as ur
from test_marginalize import local, mat, vec
from test_propagate import random_cov
from update_ref import CHI2_3_999, info_of, rows_of, unit_states, update_info, update_kalman, update_ref


def _case(seed, kind, n=16, sigma=0.05, scale=1.0):
    rng = np.random.default_rng(seed)
    x = unit_states(rng, n)
    cov = random_cov(rng, n)
    W = vec(np.stack([info_of(kind, rng, sigma) for _ in range(n)]))
    return x, cov, W, ur.fix_near(rng, x, W, scale)


def _close(a, b, tol):
    return np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-300 + np.max(np.abs(b)))) <= tol


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["full", "pos", "vel", "att", "posvel"])
def test_statement_is_the_information_form_and_the_kalman_gain(kind):
    """update_ref equals the dense information form (Sigma^-1 + W)^-1 and, for a W of whole blocks, the textbook Kalman update with
    H selecting them: xi, Sigma+ and gamma, on well-conditioned inputs."""
    x, cov, W, xb = _case(1, kind)
    r = update_ref(x, cov, W, xb)
    i = update_info(x, cov, W, xb)
    k = update_kalman(x, cov, W, xb, rows_of(kind))
    for o in (i, k):
        assert _close(r[2], o[2], 1e-9) and _close(r[1], o[1], 1e-9) and _close(r[3], o[3], 1e-9)
    assert np.array_equal(mat(r[1]), mat(r[1]).transpose(0, 2, 1))


def test_gamma_is_the_normalised_innovation_squared():
    """gamma = d^T (Sigma + W^-1)^-1 d for an invertible W."""
    x, cov, W, xb = _case(2, "full")
    _, _, _, g = update_ref(x, cov, W, xb)
    d = local(xb, x)
    Sy = mat(cov) + np.linalg.inv(mat(W))
    assert _close(g, np.einsum("ni,nij,nj->n", d, np.linalg.inv(Sy), d), 1e-9)


def test_two_sequential_fixes_are_one_combined_fix():
    """A position fix then a velocity fix (the second at the first's result) equal one fix with both blocks: both are exact under
    the identity Jacobian, so the information adds.  The attitude is uncorrelated with the rest here: an attitude correction would
    compose by retract, which adds rotations only to first order."""
    rng = np.random.default_rng(3)
    n = 16
    x, S = unit_states(rng, n), mat(random_cov(rng, n)).copy()
    S[:, 0:3, 3:], S[:, 3:, 0:3] = 0.0, 0.0
    cov = vec(S)
    Wp, Wv = (vec(np.stack([info_of(k, rng, 0.05) for _ in range(n)])) for k in ("pos", "vel"))
    xb = ur.fix_near(rng, x, Wp + Wv)
    xb[:, 0:4] = x[:, 0:4]                                           # an attitude-free fix: local is a difference on its blocks
    x1, c1, _, g1 = update_ref(x, cov, Wp, xb)
    x2, c2, _, g2 = update_ref(x1, c1, Wv, xb)
    x3, c3, _, _ = update_ref(x, cov, Wp + Wv, xb)
    assert _close(c2, c3, 1e-10)
    assert np.max(np.abs(local(x3, x2)) / np.sqrt(np.diagonal(mat(c3), axis1=1, axis2=2))) <= 1e-9


def test_zero_information_leaves_the_state():
    """W = 0: xi = 0 and gamma = 0 exactly, and x+ = retract(x, 0): the other 12 entries bit for bit, the quaternion renormalised
    as retract does (within an ulp).  The numpy statement and the oracle; the kernel in test_zero_information_and_nothing_to_do."""
    rng = np.random.default_rng(4)
    x, cov = unit_states(rng, 8), random_cov(rng, 8)
    W, xb = np.zeros((8, 225)), unit_states(rng, 8)
    for xo, co, xi, g in (update_ref(x, cov, W, xb), ur.oracle_update(x, cov, W, xb, 0), ur.oracle_update(x, cov, W, xb, 1)):
        assert np.all(xi == 0) and np.all(g == 0)
        assert np.array_equal(xo[:, 4:], x[:, 4:]) and np.max(np.abs(xo[:, 0:4] - x[:, 0:4])) <= 2.3e-16


@pytest.mark.parametrize("order", [0, 1])
def test_oracles_are_the_statement(order):
    """oracle_state_update in fp64 and in long double, both orders, equals update_ref on well-conditioned inputs."""
    for kind in ("full", "pos", "att", "rank"):
        x, cov, W, xb = _case(5, kind)
        r = update_ref(x, cov, W, xb)
        for ld in (False, True):
            o = ur.oracle_update(x, cov, W, xb, order, long_double=ld)
            assert _close(o[1], r[1], 1e-9) and _close(o[2], r[2], 1e-9) and _close(o[3], r[3], 1e-9)
            assert np.max(np.abs(o[0] - r[0])) <= 1e-12


def test_argument_validation_without_gpu():
    """The C ABI rejects a negative count, NULL required pointers and outputs equal to inputs before any CUDA call; n = 0 is a no-op."""
    from cpi_b200 import capi
    lib = capi.load()
    a = np.zeros((1, 225))
    p = lambda v: ctypes.c_void_p(v.ctypes.data)
    b, c, o1, o2 = (np.zeros((1, 225)) for _ in range(4))
    ok = [p(a), p(b), p(c), p(b), None, p(o1), p(o2), None, None]
    assert lib.cpi_state_update_batch(-1, *ok, None) != 0 and "negative" in lib.cpi_last_error().decode()
    assert lib.cpi_state_update_batch(0, *([None] * 9), None) == 0
    for k in (0, 1, 2, 3, 5, 6):
        args = list(ok); args[k] = None
        assert lib.cpi_state_update_batch(1, *args, None) != 0
        assert "null" in lib.cpi_last_error().decode()
    args = list(ok); args[5] = p(a)
    assert lib.cpi_state_update_batch(1, *args, None) != 0 and "overlap" in lib.cpi_last_error().decode()
    args = list(ok); args[6] = p(o1)
    assert lib.cpi_state_update_batch(1, *args, None) != 0 and "overlap" in lib.cpi_last_error().decode()


def test_wrapper_validation_without_gpu():
    """factor.update rejects host tensors, wrong dtypes and shapes before the device is touched."""
    import torch

    from cpi_b200 import factor
    f64 = dict(dtype=torch.float64)
    x, c, w, xb = torch.zeros(4, 16, **f64), torch.zeros(4, 225, **f64), torch.zeros(4, 225, **f64), torch.zeros(4, 16, **f64)
    with pytest.raises(ValueError, match="CUDA"):
        factor.update(x, c, w, xb)
    with pytest.raises(ValueError, match="tensor"):
        factor.update(x.numpy(), c, w, xb)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------

def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _run(torch, x, cov, W, xb, gate=None):
    from cpi_b200 import factor
    g = _dev(torch, gate) if isinstance(gate, np.ndarray) else gate
    out = factor.update(_dev(torch, x), _dev(torch, cov), _dev(torch, W), _dev(torch, xb), gate=g)
    torch.cuda.synchronize()
    return tuple(t.cpu().numpy() for t in out)


def _k7_covariances(torch, model, n, steps, seed):
    """Covariances after `steps` chained cpi_propagate_batch calls of n filters (dead reckoning, 20-sample windows at 200 Hz) and the
    propagated states: [steps, n, 225], [steps, n, 16]."""
    from cpi_b200 import factor, preint, synth
    S, L = synth.make_windows(steps, 20, rate=200.0, first_window=3000 + seed, special=False)
    L[:] = L[0]
    rec = preint.preintegrate_host(model, S, L, synth.SIGMAS, 0, ns=20)
    x0 = synth.make_states(rec, L, model, perturb=False)[:1]
    x0[:, 4:7], x0[:, 10:13] = L[:1, 0:3], L[:1, 3:6]
    rng = np.random.default_rng(seed)
    xs = [_dev(torch, np.repeat(x0, n, axis=0))]
    cs = [_dev(torch, random_cov(rng, n, scale=(1e-3, 1e-5, 1e-2, 1e-4, 1e-2)))]
    dR, dL = _dev(torch, rec), _dev(torch, L)
    for k in range(steps):
        x1, c1, _ = factor.propagate(model, xs[-1], cs[-1], dR[k:k + 1].expand(n, -1).contiguous(), dL[k:k + 1].expand(n, -1).contiguous())
        xs.append(x1); cs.append(c1)
    torch.cuda.synchronize()
    return np.stack([c.cpu().numpy() for c in cs[1:]]), np.stack([x.cpu().numpy() for x in xs[1:]])


@pytest.mark.gpu
def test_kernel_is_the_statement(cuda):
    """Random and K7-propagated covariances with every kind of W: cov+ exactly symmetric, every field within a few ulp-scaled units of
    update_ref (the distance between update_ref and the information form, times 20, floor 1e-13), and two runs give the same bits."""
    torch = cuda
    rng = np.random.default_rng(11)
    covs, xs = _k7_covariances(torch, 1, 8, 40, 11)
    cov = np.concatenate([random_cov(rng, 48), covs[[9, 19, 39]].reshape(-1, 225)])
    n = len(cov)
    x = np.concatenate([unit_states(rng, 48), xs[[9, 19, 39]].reshape(-1, 16)])
    kinds = ["full", "pos", "vel", "att", "bg", "ba", "posvel", "rank"]
    W = vec(np.stack([info_of(kinds[i % len(kinds)], rng, 0.05) for i in range(n)]))
    xb = ur.fix_near(rng, x, W)
    got = _run(torch, x, cov, W, xb)
    again = _run(torch, x, cov, W, xb)
    assert all(np.array_equal(a, b) for a, b in zip(got, again))
    assert np.array_equal(mat(got[1]), mat(got[1]).transpose(0, 2, 1))
    assert np.all(got[3] == 1)
    r = update_ref(x, cov, W, xb)
    i = update_info(x, cov, W, xb)
    eb, ex, eg = ur.errors((r[0], r[1], r[3]), (got[0], got[1], got[2]), x)
    nb, nx, ng = ur.errors((r[0], r[1], r[3]), (i[0], i[1], i[3]), x)
    print(f"kernel vs update_ref: cov {eb.max():.1e}, state {ex.max():.1e}, gamma {eg.max():.1e}; "
          f"information form vs update_ref: {nb.max():.1e}, {nx.max():.1e}, {ng.max():.1e}")
    assert eb.max() <= 20 * max(nb.max(), 1e-13) and ex.max() <= 20 * max(nx.max(), 1e-13) and eg.max() <= 20 * max(ng.max(), 1e-13)


@pytest.mark.gpu
def test_zero_information_and_nothing_to_do(cuda):
    """W = 0 gives gamma = 0 and x+ = retract(x, 0) on the device: the other 12 entries bit for bit, the quaternion renormalised
    (within an ulp of x's); n = 0 launches nothing."""
    from cpi_b200 import capi, factor
    torch = cuda
    rng = np.random.default_rng(12)
    x, cov = unit_states(rng, 9), random_cov(rng, 9)
    xo, co, g, a = _run(torch, x, cov, np.zeros((9, 225)), unit_states(rng, 9))
    assert np.array_equal(xo[:, 4:], x[:, 4:]) and np.max(np.abs(xo[:, 0:4] - x[:, 0:4])) <= 2.3e-16
    assert np.all(g == 0) and np.all(a == 1)
    before = capi.launch_count()
    e = torch.empty((0, 16), dtype=torch.float64, device="cuda")
    out = factor.update(e, torch.empty((0, 225), dtype=torch.float64, device="cuda"), torch.empty((0, 225), dtype=torch.float64, device="cuda"), e)
    assert capi.launch_count() == before and out[0].shape == (0, 16)


@pytest.mark.gpu
def test_wrapper_validation_on_the_device(cuda):
    """factor.update rejects wrong lengths, dtypes, a gate of the wrong length and NaN gates; +inf is accepted."""
    from cpi_b200 import factor
    torch = cuda
    f64 = dict(dtype=torch.float64, device="cuda")
    x, c, w, xb = torch.zeros(4, 16, **f64), torch.zeros(4, 225, **f64), torch.zeros(4, 225, **f64), torch.zeros(4, 16, **f64)
    with pytest.raises(ValueError, match="meas_info"):
        factor.update(x, c, w[:3], xb)
    with pytest.raises(ValueError, match="float64"):
        factor.update(x, c.float(), w, xb)
    with pytest.raises(ValueError, match="one entry per filter"):
        factor.update(x, c, w, xb, gate=torch.ones(3, **f64))
    with pytest.raises(ValueError, match="NaN"):
        factor.update(x, c, w, xb, gate=float("nan"))
    with pytest.raises(ValueError, match="NaN"):
        factor.update(x, c, w, xb, gate=torch.tensor([1.0, float("nan"), 1.0, 1.0], **f64))
    with pytest.raises(ValueError, match="CUDA"):
        factor.update(x, c, w, xb, gate=torch.ones(4, dtype=torch.float64))


@pytest.mark.gpu
def test_gating(cuda):
    """Skipped filters are bitwise their inputs with applied = 0; gate = +inf is bitwise the NULL gate.  20 000 1 cm position fixes
    with 5 % replaced by 5 m outliers, gated at the chi^2_3 0.999 quantile: every outlier is rejected, and the rejected inliers lie
    within the two-sided 1e-6 binomial bound of their expected 0.1 %."""
    torch = cuda
    rng = np.random.default_rng(13)
    n = 20_000
    x, cov = unit_states(rng, n), random_cov(rng, n)
    Wp = np.zeros((15, 15)); Wp[12:15, 12:15] = np.eye(3) / 0.01 ** 2
    W = np.repeat(vec(Wp[None]), n, axis=0)
    S = mat(cov)
    # inliers: x_bar drawn from the predicted measurement distribution, so gamma ~ chi^2_3 exactly
    Sy = S[:, 12:15, 12:15] + np.eye(3) * 0.01 ** 2
    xb = x.copy()
    xb[:, 13:16] += np.einsum("nij,nj->ni", np.linalg.cholesky(Sy), rng.normal(size=(n, 3)))
    out = rng.random(n) < 0.05
    xb[out, 13:16] = x[out, 13:16] + 5.0 / np.sqrt(3)
    free = _run(torch, x, cov, W, xb)
    inf = _run(torch, x, cov, W, xb, gate=float("inf"))
    assert all(np.array_equal(a, b) for a, b in zip(free, inf)) and np.all(inf[3] == 1)
    xo, co, g, a = _run(torch, x, cov, W, xb, gate=np.full(n, CHI2_3_999))
    assert np.array_equal(g, free[2])
    skip = a == 0
    assert np.array_equal(skip, g > CHI2_3_999)
    assert np.array_equal(xo[skip], x[skip]) and np.array_equal(co[skip], cov[skip])
    assert np.array_equal(xo[~skip], free[0][~skip]) and np.array_equal(co[~skip], free[1][~skip])
    n_in, rej_in = int((~out).sum()), int((skip & ~out).sum())
    lo, hi = binom.ppf([5e-7, 1 - 5e-7], n_in, 1e-3)
    print(f"gating: {int(out.sum())} outliers (gamma >= {g[out].min():.3g}) all rejected; {rej_in} of {n_in} inliers rejected "
          f"(expected {1e-3 * n_in:.1f}, bound [{lo:.0f}, {hi:.0f}])")
    assert np.all(skip[out]) and lo <= rej_in <= hi


@pytest.mark.gpu
def test_isolation(cuda):
    """A cov that is not SPD, or a NaN in W or x_bar, in one filter of ten leaves the other nine bitwise the clean run; the faulty
    filter's fix is applied (NaN gamma is not > gate) and its NaN shows."""
    torch = cuda
    rng = np.random.default_rng(14)
    x, cov = unit_states(rng, 10), random_cov(rng, 10)
    W = vec(np.stack([info_of("full", rng, 0.05) for _ in range(10)]))
    xb = ur.fix_near(rng, x, W)
    gate = np.full(10, 1e300)
    clean = _run(torch, x, cov, W, xb, gate)
    for what in ("cov", "W", "xb"):
        c2, W2, xb2 = cov.copy(), W.copy(), xb.copy()
        if what == "cov":
            S = mat(c2[4:5])[0]; S[3, 3] = -1.0; c2[4] = vec(S[None])[0]
        elif what == "W":
            W2[4, 17] = np.nan
        else:
            xb2[4, 14] = np.nan
        got = _run(torch, x, c2, W2, xb2, gate)
        keep = np.arange(10) != 4
        assert all(np.array_equal(a[keep], b[keep]) for a, b in zip(got, clean)), what
        assert np.isnan(got[2][4]) and got[3][4] == 1 and np.isnan(got[0][4]).any(), what
        if what != "xb":
            assert np.isnan(got[1][4]).all(), what


def _single_state_routes(torch, x, cov, W, xb):
    """x+ and Sigma+ through the chain entry points on single-state chains, the chain prior Sigma^-1 at x and the fix a state prior.
    Sigma+ is chains_marginals.  chains_lm_step refuses a batch of single-state chains only (no factor: its cost sum is handed an
    empty factor-cost array, checked here), so x+ is its steps called one by one: prior_at, state_priors_fold onto the chain prior,
    chains_assemble at lambda = 0, chains_solve and retract."""
    from cpi_b200 import capi, factor
    n = len(x)
    Si = np.linalg.inv(mat(cov)); Si = 0.5 * (Si + Si.transpose(0, 2, 1))
    f64 = dict(dtype=torch.float64, device="cuda")
    dW, dX, dxb = _dev(torch, W), _dev(torch, x), _dev(torch, xb)
    prior = (_dev(torch, vec(Si)), torch.zeros((n, 15), **f64), torch.zeros(n, **f64), dX)
    sp = (torch.arange(n, dtype=torch.int64, device="cuda"), dW, None, None, dxb)
    rec, lin = torch.empty((0, 290), **f64), torch.empty((0, 13), **f64)
    c1, _ = factor.chains_marginals(1, dX, rec, lin, 1, prior=prior, state_priors=sp)
    with pytest.raises(capi.CpiError, match="null pointer"):
        factor.chains_lm_step(1, dX, rec, lin, 1, prior=prior, lam=0.0, diagonal_damping=False, state_priors=sp)
    rhs, f = factor.prior_at(dW, torch.zeros((n, 15), **f64), torch.zeros(n, **f64), dxb, dX)
    pi, pr, pf = prior[0].clone(), torch.zeros((n, 15), **f64), torch.zeros(n, **f64)
    offs = torch.arange(n + 1, dtype=torch.int64, device="cuda")
    factor.state_priors_fold(offs, offs, dW, rhs, f, prior_info=pi, prior_rhs=pr, prior_f=pf)
    e0, e1 = torch.empty((0, 225), **f64), torch.empty((0, 15), **f64)
    D, E, r = factor.chains_assemble(e0, e0, e0, e1, e1, 1, 0.0, pi, pr, n_chains=n)
    x1 = factor.retract(dX, factor.chains_solve(D, E, r, 1, n_chains=n))
    torch.cuda.synchronize()
    return x1.cpu().numpy(), c1.cpu().numpy()


@pytest.mark.gpu
def test_against_the_chain_entry_points(cuda):
    """Single-state chains with the prior Sigma^-1 linearised at x and the fix as a state prior: the Gauss-Newton step at lambda = 0
    gives x+ and chains_marginals gives Sigma+, both within 20x the distance between the same two routes in numpy (the information form
    and the square-root form), floor 1e-12."""
    torch = cuda
    rng = np.random.default_rng(15)
    n = 64
    x, cov = unit_states(rng, n), random_cov(rng, n)
    kinds = ["full", "pos", "vel", "posvel", "ba", "rank"]
    W = vec(np.stack([info_of(kinds[i % len(kinds)], rng, 0.05) for i in range(n)]))
    xb = ur.fix_near(rng, x, W)
    xb[:, 0:4] = x[:, 0:4]
    got = _run(torch, x, cov, W, xb)
    xl, cl = _single_state_routes(torch, x, cov, W, xb)
    r, i = update_ref(x, cov, W, xb), update_info(x, cov, W, xb)
    sd = np.sqrt(np.diagonal(mat(r[1]), axis1=1, axis2=2))
    ex = float(np.max(np.abs(local(xl, got[0])) / sd))
    ex_np = float(np.max(np.abs(local(i[0], r[0])) / sd))
    dg = sd[:, :, None] * sd[:, None, :]
    ec = float(np.max(np.abs(mat(cl) - mat(got[1])) / dg))
    ec_np = float(np.max(np.abs(mat(i[1]) - mat(r[1])) / dg))
    print(f"update vs chains_lm_step: {ex:.1e} (numpy routes {ex_np:.1e}); vs chains_marginals: {ec:.1e} (numpy routes {ec_np:.1e})")
    assert ex <= 20 * max(ex_np, 1e-12) and ec <= 20 * max(ec_np, 1e-12)
