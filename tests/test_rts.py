"""Rauch-Tung-Striebel smoothing of filter runs (cpi_rts_smooth_batch, kernel K15, factor.rts_smooth; DESIGN.md section 3o).

CPU: the numpy statement (tests/rts_ref.py) against the dense inverse of linear-Gaussian chains in float64 and long double, its edge
cases, the argument checks of the C ABI and the binding, and the sensitivity of the precision gate.
GPU: the smoother of a filter run at its exact prediction is chains_marginals; K15 against the statement in long double on filter
runs of every update kernel; exact properties; the stream contract; Monte-Carlo consistency.

The precision gate: errors in the truth's smoothed standard deviations, per run and per output block (Ps_k, each component of
local(xs_true, xs_k), Xs_k), with e_64 the fp64 statement's worst error in the run's group (family):
    e_dev <= 8 max(e_64, floor, 1e-15),   floor = one ulp of the stored smoothed state component (0 for Ps and Xs),
and Ps exactly symmetric.  Keyframes with P_k = 0 (exact anchors) are checked exactly instead."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest

import rts_ref as rr
from cpi_b200 import capi, synth
from test_chain_marginals import inv_truth

K_GATE, FLOOR = 8.0, 1e-15


# ------------------------------------------------------------------------------------------------------------------
# the gate
# ------------------------------------------------------------------------------------------------------------------

def _err(truth, got, offs):
    """[N, 17] per keyframe: Ps, the 15 state components, and Xs of the transition leaving it (0 for a run's last keyframe)."""
    eP, ex, eX = rr.errors(truth, got, offs)
    o = np.asarray(offs, dtype=np.int64)
    ks = np.concatenate([np.arange(o[c], o[c + 1] - 1) for c in range(len(o) - 1)]).astype(np.int64)
    eXk = np.zeros(len(eP))
    eXk[ks] = eX
    return np.concatenate([eP[:, None], ex, eXk[:, None]], axis=1)


def gate(offs, inputs, got, groups, long_truth=None):
    """(worst ratio e_dev / (K_GATE max(e_64, floor, FLOOR)), its keyframe and column) of got = (xs, Ps, Xs) on the runs of offs with
    the statement's inputs (x, P, xb, Pb, C); groups [n_runs] labels the families e_64 is pooled over.  inf if Ps is not exactly
    symmetric."""
    o = np.asarray(offs, dtype=np.int64)
    truth = long_truth if long_truth is not None else rr.rts(o, *inputs, dtype=np.longdouble)
    f64 = rr.rts(o, *inputs, dtype=np.float64)
    e_dev, e_64 = _err(truth, got, o), _err(truth, f64, o)
    run_of = np.repeat(np.arange(len(o) - 1), o[1:] - o[:-1])
    g = np.asarray(groups)[run_of]
    pooled = np.zeros_like(e_64)
    for lab in np.unique(g):
        pooled[g == lab] = e_64[g == lab].max(axis=0)
    floor = np.zeros_like(e_64)
    floor[:, 1:16] = rr.state_floor(truth)
    ratio = e_dev / (K_GATE * np.maximum(np.maximum(pooled, floor), FLOOR))
    Ps = np.asarray(got[1])
    if not np.array_equal(Ps, np.swapaxes(Ps, 1, 2)):
        return np.inf, -1, -1
    i = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
    return float(ratio[i]), int(i[0]), int(i[1])


# ------------------------------------------------------------------------------------------------------------------
# CPU: linear-Gaussian chains in numpy
# ------------------------------------------------------------------------------------------------------------------

def _spd(rng, n, scale):
    G = rng.normal(size=(n, 15, 15))
    C = G @ G.transpose(0, 2, 1) / 15 + 0.3 * np.eye(15)
    D = np.repeat(np.asarray(scale), 3)
    C = D[None, :, None] * C * D[None, None, :]
    return 0.5 * (C + C.transpose(0, 2, 1))


def _unit_states(rng, n):
    x = np.zeros((n, 16))
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True); q[q[:, 3] < 0] *= -1
    x[:, 0:4], x[:, 4:16] = q, rng.normal(size=(n, 12))
    return x


def linear_runs(rng, lengths, fix_every=3, anchor=False):
    """Random linear-Gaussian runs: x_{k+1} = A_k x_k + B_k w_k with w_k ~ N(0, Pm_k), a random prior P_0 (0 with anchor), and a
    random fix W on every fix_every-th keyframe.  Returns (offsets, the statement's inputs (x, P, xb, Pb, C) as K7 would write them
    for a filter that fixes with W, the information matrix of every run as (dense [15 S, 15 S] per run))."""
    o = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    N, R = int(o[-1]), len(lengths)
    x = _unit_states(rng, N)
    P = np.zeros((N, 15, 15))
    xb, Pb, Cr = np.zeros((N - R, 16)), np.zeros((N - R, 15, 15)), np.zeros((N - R, 15, 15))
    infos = []
    for c, S in enumerate(lengths):
        s0, t0 = int(o[c]), int(o[c] - c)
        P0 = np.zeros((15, 15)) if anchor else _spd(rng, 1, (1e-2, 1e-3, 1e-1, 1e-2, 1.0))[0]
        Lam = np.zeros((15 * S, 15 * S))
        Lam[:15, :15] = np.linalg.inv(P0) if not anchor else 0.0
        P[s0] = P0
        for k in range(S - 1):
            A = np.eye(15) + 0.03 * rng.normal(size=(15, 15))
            B = np.eye(15) + 0.05 * rng.normal(size=(15, 15))
            Q = B @ _spd(rng, 1, (1e-3, 1e-4, 1e-2, 1e-3, 1e-2))[0] @ B.T
            Q = 0.5 * (Q + Q.T)
            t, s = t0 + k, s0 + k
            Pb[t] = A @ P[s] @ A.T + Q
            Pb[t] = 0.5 * (Pb[t] + Pb[t].T)
            Cr[t] = P[s] @ A.T
            xb[t] = x[s + 1] if k % 2 else rr.retract(x[s + 1:s + 2], rng.normal(size=(1, 15)) * 1e-3)[0]
            Qi = np.linalg.inv(Q)
            a, b = 15 * k, 15 * k + 15
            Lam[a:b, a:b] += A.T @ Qi @ A
            Lam[a:b, b:b + 15] -= A.T @ Qi
            Lam[b:b + 15, a:b] -= Qi @ A
            Lam[b:b + 15, b:b + 15] += Qi
            if (k + 1) % fix_every == 0:
                W = _spd(rng, 1, (10.0, 100.0, 1.0, 10.0, 1.0))[0]
                Lam[b:b + 15, b:b + 15] += W
                Pn = np.linalg.inv(np.linalg.inv(Pb[t]) + W)
                P[s + 1] = 0.5 * (Pn + Pn.T)
            else:
                P[s + 1] = Pb[t]
        infos.append(Lam)
    return o, (x, P, xb, Pb, Cr), infos


def _scaled(A, sa, sb):
    return float(np.max(np.abs(A) / (sa[:, None] * sb[None, :])))


@pytest.mark.parametrize("dtype", [np.float64, np.longdouble])
def test_statement_is_the_dense_inverse(dtype):
    """The statement's Ps_k and Xs_k are the diagonal and next-to-diagonal blocks of the inverse of each linear-Gaussian run's
    information matrix (prior, transition factors with noise B Pm B^T and the fixes), in the smoothed standard deviations."""
    rng = np.random.default_rng(31)
    o, inputs, infos = linear_runs(rng, [1, 2, 5, 12, 30])
    xs, Ps, Xs = rr.rts(o, *inputs, dtype=dtype)
    worst = 0.0
    for c, Lam in enumerate(infos):
        s0, S = int(o[c]), int(o[c + 1] - o[c])
        T, _ = inv_truth(Lam)
        for k in range(S):
            sd = np.sqrt(np.diag(T[15 * k:15 * k + 15, 15 * k:15 * k + 15]))
            worst = max(worst, _scaled(np.asarray(Ps[s0 + k], dtype=np.float64) - T[15 * k:15 * k + 15, 15 * k:15 * k + 15], sd, sd))
            if k + 1 < S:
                sd1 = np.sqrt(np.diag(T[15 * k + 15:15 * k + 30, 15 * k + 15:15 * k + 30]))
                worst = max(worst, _scaled(np.asarray(Xs[s0 - c + k], dtype=np.float64) - T[15 * k:15 * k + 15, 15 * k + 15:15 * k + 30],
                                           sd, sd1))
    print(f"{np.dtype(dtype).name}: worst distance to the dense inverse {worst:.2e} smoothed sd")
    assert worst < 1e-8, worst                                         # the inputs' own fp64 inversions: 7.6e-10 in both dtypes
    assert np.array_equal(Ps, np.swapaxes(Ps, 1, 2))


def test_statement_edge_cases():
    """The last keyframe is copied bit for bit; one-keyframe runs are copied; P_k = 0 gives G = 0, Ps_k = 0 and xs_k = retract(x_k, 0)
    (the linear entries bitwise, the quaternion within an ulp); xs_{k+1} == xb_{k+1} gives d = 0 exactly."""
    rng = np.random.default_rng(32)
    o, (x, P, xb, Pb, C), _ = linear_runs(rng, [1, 4, 1, 6], anchor=True)
    xs, Ps, Xs = rr.rts(o, x, P, xb, Pb, C)
    for c in range(len(o) - 1):
        last = int(o[c + 1]) - 1
        assert np.array_equal(xs[last], x[last]) and np.array_equal(Ps[last], P[last])
        s0 = int(o[c])
        if o[c + 1] - o[c] > 1:                                       # the anchor: P_0 = 0
            assert not np.any(Ps[s0]) and not np.any(Xs[s0 - c])
            assert np.array_equal(xs[s0, 4:16], x[s0, 4:16])
            assert np.max(np.abs(xs[s0, 0:4] - x[s0, 0:4])) <= 2.0 ** -52
    # d = 0: run 1's last prediction equal to its (copied) last keyframe
    xb1 = xb.copy()
    last, t = int(o[2]) - 1, int(o[2]) - 2 - 1                        # run 1's transitions are stored from o[1] - 1
    xb1[t] = x[last]
    assert not np.any(rr.local(xb1[[t]], x[[last]]))
    xs1, _, _ = rr.rts(o, x, P, xb1, Pb, C)
    assert np.array_equal(xs1[last - 1], rr.retract(x[[last - 1]], np.zeros((1, 15)))[0])


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def test_argument_validation_without_gpu():
    """cpi_rts_smooth_batch rejects bad arguments with CPI_EINVAL before any CUDA call, and n_runs = 0 launches nothing; the binding
    rejects shapes, dtypes, layouts and host tensors before touching the device."""
    import torch
    from cpi_b200 import factor
    lib = capi.load()
    bufs = [np.zeros(16 * 225) for _ in range(9)]
    p = [_p(b) for b in bufs]
    # cpi_rts_smooth_batch(n_runs, offs, uniform, n_states, states, cov, pred_states, pred_cov, cross, states_out, cov_out, cross_out, stream)
    rts = lambda *a: lib.cpi_rts_smooth_batch(*a, None)
    before = capi.launch_count()
    assert rts(-1, None, 2, 4, *p) == -1 and b"negative" in lib.cpi_last_error()
    assert rts(2, None, 0, 4, *p) == -1 and b"uniform" in lib.cpi_last_error()
    assert rts(2, None, 2, 5, *p) == -1 and b"n_states" in lib.cpi_last_error()
    assert rts(3, p[0], 0, 2, *p[1:]) == -1 and b"n_states" in lib.cpi_last_error()
    for k in range(7):                                                 # states .. cov_out (cross_out may be NULL)
        a = list(p[1:]); a[k] = None
        assert rts(2, None, 2, 4, *a) == -1 and b"null" in lib.cpi_last_error(), k
    for o in range(5, 8):                                              # an output equal to an input
        for i in range(5):
            a = list(p[1:]); a[o] = a[i]
            assert rts(2, None, 2, 4, *a) == -1 and b"overlap inputs" in lib.cpi_last_error(), (o, i)
    a = list(p[1:]); a[5] = p[0]
    assert rts(2, p[0], 0, 4, *a) == -1 and b"overlap inputs" in lib.cpi_last_error()
    for o1, o2 in ((5, 6), (5, 7), (6, 7)):
        a = list(p[1:]); a[o2] = a[o1]
        assert rts(2, None, 2, 4, *a) == -1 and b"overlap each other" in lib.cpi_last_error()
    assert rts(0, None, 1, 0, *[None] * 8) == 0
    assert capi.launch_count() == before
    # the binding
    f64 = dict(dtype=torch.float64)
    X, C, rec, lin = torch.zeros((6, 16), **f64), torch.zeros((6, 225), **f64), torch.zeros((4, 290), **f64), torch.zeros((4, 13), **f64)
    with pytest.raises(ValueError, match="model"):
        factor.rts_smooth(3, X, C, rec, lin, 3)
    with pytest.raises(ValueError, match="CUDA"):
        factor.rts_smooth(1, X, C, rec, lin, 3)
    with pytest.raises(ValueError, match="tensor"):
        factor.rts_smooth(1, X.numpy(), C, rec, lin, 3)


@pytest.mark.parametrize("inject", ["Pb-fp32", "G-scaled", "no-mirror"])
def test_gate_is_sensitive(inject):
    """Three injected errors in the fp64 statement fail the precision gate that the clean fp64 statement passes: Pb rounded to fp32,
    G scaled by 1 + 1e-7, Ps formed without mirroring its lower triangle."""
    rng = np.random.default_rng(33)
    o, inputs, _ = linear_runs(rng, [3, 8, 20])
    groups = np.zeros(len(o) - 1)
    truth = rr.rts(o, *inputs, dtype=np.longdouble)
    clean = rr.rts(o, *inputs)
    assert gate(o, inputs, clean, groups, truth)[0] <= 1.0 / K_GATE + 1e-12
    f = {"Pb-fp32": lambda n, v: v.astype(np.float32).astype(np.float64) if n == "Pb" else v,
         "G-scaled": lambda n, v: v * (1 + 1e-7) if n == "G" else v,
         "no-mirror": None}[inject]
    bad = rr.rts(o, *inputs, inject=f, mirror=inject != "no-mirror")
    ratio = gate(o, inputs, bad, groups, truth)
    print(f"{inject}: worst ratio {ratio[0]:.3g} at keyframe {ratio[1]}, column {ratio[2]}")
    assert ratio[0] > 1.0, ratio


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------

def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_smoother_of_the_filter_is_the_chain_smoother(cuda, model):
    """The configuration of test_update_filter.test_filter_is_the_smoother_at_the_newest_state: a chain at its exact prediction from
    x_0 with Sigma_0, 1 cm position fixes placed at the predicted states of keyframes 5, 10, 15 and 20 (d = 0), filtered with K7 + K10
    and smoothed by rts_smooth(cross=True).  Ps_k is chains_marginals' Sigma_kk at every keyframe and Xs_k its cross slot (one
    untruncated chain); the gate is 20x the distance between the same two routes in numpy (the filter and the statement from the
    device's Jacobians, and the refined dense inverse of the device's blocks), floor 1e-12, in the smoothed standard deviations.  The
    smoothed means are the filtered ones to rounding: bitwise at the last two keyframes, the quaternion within a few ulps and every
    component within 1e-12 smoothed sd (an ulp of attitude, from the renormalisation, reaches the other entries through G)."""
    from cpi_b200 import factor, preint
    from test_chain_marginals import _system, dense
    from test_propagate import random_cov
    torch = cuda
    m, fixes = 25, (5, 10, 15, 20)
    S, L = synth.make_windows(m, 20, rate=200.0, first_window=15000 + model, special=False)
    L[:] = L[0]
    rec = preint.preintegrate_host(model, S, L, synth.SIGMAS, 0, ns=20)
    x0 = synth.make_states(rec, L, model, perturb=False)[:1]
    x0[:, 4:7], x0[:, 10:13] = L[:1, 0:3], L[:1, 3:6]
    rng = np.random.default_rng(6 + model)
    Sig0 = rr.mat(random_cov(rng, 1))[0]
    Wp = np.zeros((15, 15)); Wp[12:15, 12:15] = np.eye(3) / 0.01 ** 2
    dR, dL = _dev(torch, rec), _dev(torch, L)
    xs, cs = [_dev(torch, x0)], [_dev(torch, rr.vec(Sig0[None]))]
    for k in range(m):
        x1, c1, _ = factor.propagate(model, xs[-1], cs[-1], dR[k:k + 1], dL[k:k + 1])
        if k + 1 in fixes:
            x1, c1, nis, applied = factor.update(x1, c1, _dev(torch, rr.vec(Wp[None])), x1.clone())
            assert float(nis[0]) == 0.0 and int(applied[0]) == 1
        xs.append(x1); cs.append(c1)
    X, Cf = torch.cat(xs), torch.cat(cs)
    Xs, Ps, Xc = factor.rts_smooth(model, X, Cf, dR, dL, m + 1, cross=True)
    Xn, Ps, Xc = X.cpu().numpy(), rr.mat(Ps.cpu().numpy()), rr.mat(Xc.cpu().numpy())
    Lam0 = np.linalg.inv(Sig0); Lam0 = 0.5 * (Lam0 + Lam0.T)
    idx = np.array(fixes, dtype=np.int64)
    prior = (_dev(torch, rr.vec(Lam0[None])), _dev(torch, np.zeros((1, 15))), _dev(torch, np.zeros(1)), _dev(torch, Xn[:1]))
    sp = (_dev(torch, idx), _dev(torch, np.repeat(rr.vec(Wp[None]), len(idx), axis=0)), None, None, _dev(torch, Xn[idx]))
    cov, cr = factor.chains_marginals(model, X, dR, dL, m + 1, prior=prior, state_priors=sp, cross=True)
    cov, cr = rr.mat(cov.cpu().numpy()), rr.mat(cr.cpu().numpy())
    # numpy: the filter and the statement from the device's Jacobians, and the refined dense inverse of the device's blocks
    e, H1, H2 = factor.factor_eval(model, X, dR, dL)
    h1, h2, Pm = rr.mat(H1.cpu().numpy()), rr.mat(H2.cpu().numpy()), rr.mat(rec[:, 65:290])
    P_np, Pb_np, C_np = [Sig0], [], []
    for k in range(m):
        B = np.linalg.inv(h2[k]); A = -B @ h1[k]
        Pb = A @ P_np[-1] @ A.T + B @ Pm[k] @ B.T
        Pb = 0.5 * (Pb + Pb.T)
        Pb_np.append(Pb); C_np.append(P_np[-1] @ A.T)
        P = np.linalg.inv(np.linalg.inv(Pb) + Wp) if k + 1 in fixes else Pb
        P_np.append(0.5 * (P + P.T))
    o = np.array([0, m + 1])
    _, Ps_np, Xc_np = rr.rts(o, Xn, np.array(P_np), Xn[1:], np.array(Pb_np), np.array(C_np))
    D, E = _system(torch, model, X, dR, dL, m + 1, prior, sp)
    T, _ = inv_truth(dense(rr.mat(D.cpu().numpy()), rr.mat(E.cpu().numpy()), 0, m + 1))
    sd = [np.sqrt(np.diag(p)) for p in Ps]
    err = err_np = 0.0
    for k in range(m + 1):
        blk = T[15 * k:15 * k + 15, 15 * k:15 * k + 15]
        err = max(err, _scaled(cov[k] - Ps[k], sd[k], sd[k]))
        err_np = max(err_np, _scaled(blk - Ps_np[k], sd[k], sd[k]))
        if k < m:
            err = max(err, _scaled(cr[k] - Xc[k], sd[k], sd[k + 1]))
            err_np = max(err_np, _scaled(T[15 * k:15 * k + 15, 15 * k + 15:15 * k + 30] - Xc_np[k], sd[k], sd[k + 1]))
    Xsn = Xs.cpu().numpy()
    ulps = np.max(np.abs(Xsn[:, 4:16] - Xn[:, 4:16]) / np.spacing(np.abs(Xn[:, 4:16])))
    dq = float(np.max(np.abs(Xsn[:, 0:4] - Xn[:, 0:4])))
    dsd = float(np.max(np.abs(rr.local(Xn, Xsn)) / np.sqrt(np.diagonal(Ps, axis1=1, axis2=2))))
    print(f"model {model}: RTS against chains_marginals: device {err:.2e}, numpy routes {err_np:.2e}; means: linear entries within "
          f"{ulps:.0f} ulp, quaternion within {dq:.1e}, {dsd:.1e} smoothed sd")
    assert err <= 20 * max(err_np, 1e-12), (err, err_np)
    # d is exactly 0 but where K10's retract(x, 0) renormalised a quaternion; that ulp of attitude reaches the other entries through G
    assert np.array_equal(Xsn[m, 4:16], Xn[m, 4:16]) and np.array_equal(Xsn[m - 1, 4:16], Xn[m - 1, 4:16])
    assert dq <= 4 * 2.0 ** -52 and dsd <= 1e-12, (dq, dsd)


def filter_runs(torch, model, lengths, seed, update=None, every=3, anchor=False, sharp=False, dead=False, keep_k7=False):
    """Filter runs on the device: run c of lengths[c] keyframes from x_0 (a state of synth.make_states) and a random Sigma_0 (0 with
    anchor), propagated by K7 over synthetic records and updated on every `every`-th keyframe by `update`: "k10" (a position fix of
    1 cm, or with sharp of lambda_max(W Sigma) up to 1e12), "k11" (one measurement of each kind), "k13-huber" / "k13-cauchy" (the
    same, iterated with a loss), or None.  Returns (offsets, states [N,16], cov [N,225], records, lin) as device tensors, and with
    keep_k7 the forward pass's own K7 outputs per transition (predicted states, covariances, cross)."""
    from cpi_b200 import factor, preint
    from measurement_ref import h_of, random_measurements
    from test_propagate import random_cov
    rng = np.random.default_rng(seed)
    lengths = np.asarray(lengths, dtype=np.int64)
    o = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    R, N = len(lengths), int(o[-1])
    nt = N - R
    Sm, L = synth.make_windows(nt, 20, rate=200.0, first_window=1000 * seed, special=False)
    rec = preint.preintegrate_host(model, Sm, L, synth.SIGMAS, 0, ns=20)
    chain = synth.make_states(rec, L, model, perturb=False)
    X = torch.empty((N, 16), dtype=torch.float64, device="cuda")
    P = torch.empty((N, 225), dtype=torch.float64, device="cuda")
    first = _dev(torch, o[:-1])
    X[first] = _dev(torch, chain[o[:-1] - np.arange(R)])
    P[first] = _dev(torch, np.zeros((R, 225)) if anchor else random_cov(rng, R) * (1e-2 if dead else 1.0))
    dR, dL = _dev(torch, rec), _dev(torch, L)
    K7 = (torch.empty((nt, 16), dtype=torch.float64, device="cuda"), torch.empty((nt, 225), dtype=torch.float64, device="cuda"),
          torch.empty((nt, 225), dtype=torch.float64, device="cuda"))
    for j in range(int(lengths.max()) - 1):
        r = np.nonzero(lengths > j + 1)[0]
        s, t = o[r] + j, o[r] - r + j
        ds, dt = _dev(torch, s), _dev(torch, t)
        x1, c1, cr = factor.propagate(model, X[ds], P[ds], dR[dt], dL[dt], want_cross=True)
        K7[0][dt], K7[1][dt], K7[2][dt] = x1, c1, cr
        if update is not None and (j + 1) % every == 0:
            n = len(r)
            if update == "k10":
                W = np.zeros((n, 15, 15)); W[:, 12:15, 12:15] = np.eye(3) / 0.01 ** 2
                if sharp:
                    Spp = rr.mat(c1.cpu().numpy())[:, 12:15, 12:15]
                    lam = np.linalg.eigvalsh(Spp)[:, -1]
                    W[:, 12:15, 12:15] = np.eye(3)[None] * (10.0 ** rng.uniform(0, 12, n) / lam)[:, None, None]
                xb = x1.cpu().numpy().copy()
                xb[:, 13:16] += rng.normal(size=(n, 3)) * 0.01
                x1, c1, _, _ = factor.update(x1, c1, _dev(torch, rr.vec(W)), _dev(torch, xb))
            else:
                xn = x1.cpu().numpy()
                idx, kind, z, si, aux = random_measurements(rng, xn, 3 * n)
                idx = np.repeat(np.arange(n), 3).astype(np.int64)
                z = h_of(kind, xn[idx], aux) + rng.normal(size=(3 * n, 3)) * 0.05
                z[::7] += 5.0                                             # outliers for the losses
                ms = tuple(_dev(torch, a) for a in (idx, kind, z, si, aux))
                if update == "k11":
                    x1, c1, _, _ = factor.update_measurements(x1, c1, ms)
                else:
                    code = capi.LOSS_HUBER if update == "k13-huber" else capi.LOSS_CAUCHY
                    loss = (_dev(torch, np.full(3 * n, code, dtype=np.int32)), _dev(torch, np.full(3 * n, 1.5)))
                    x1, c1, _, _, _ = factor.update_measurements_iterated(x1, c1, ms, measurement_loss=loss, max_iterations=5)
        X[ds + 1], P[ds + 1] = x1, c1
    return (o, X, P, dR, dL, K7) if keep_k7 else (o, X, P, dR, dL)


def _k7(torch, model, o, X, P, dR, dL):
    """The statement's inputs from the device: the posteriors and K7's outputs over every transition (as rts_smooth computes them)."""
    from cpi_b200 import factor
    R = len(o) - 1
    idx_i = _dev(torch, np.concatenate([np.arange(o[c], o[c + 1] - 1) for c in range(R)]).astype(np.int64))
    xp, cp, cr = factor.propagate(model, X, P, dR, dL, anchor=idx_i if R > 1 else None, want_cross=True)
    return (X.cpu().numpy(), rr.mat(P.cpu().numpy()), xp.cpu().numpy(), rr.mat(cp.cpu().numpy()), rr.mat(cr.cpu().numpy())), (xp, cp, cr)


FAMILIES = {
    "friendly": dict(lengths=[10] * 64, update="k10"),
    "dead-reckoned": dict(lengths=[600] * 4, dead=True),
    "sharp": dict(lengths=[12] * 64, update="k10", sharp=True, every=2),
    "anchor": dict(lengths=[10] * 32, update="k10", anchor=True),
    "k11": dict(lengths=[10] * 48, update="k11"),
    "k13-huber": dict(lengths=[10] * 48, update="k13-huber"),
    "k13-cauchy": dict(lengths=[10] * 48, update="k13-cauchy"),
    "ragged": dict(lengths=list(np.arange(4000) % 64 + 1), update="k10", every=4),
}


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_against_the_long_double_statement(cuda, model):
    """K15 (through rts_smooth) against the statement in long double on the K7 outputs the binding computes, per run and output
    block, at K_GATE max(e_64 of the family, floor).  Families: friendly runs, 600 dead-reckoned keyframes, fixes up to
    lambda_max(W Sigma) = 1e12, an exact first anchor (checked exactly there), K11 and K13 (Huber, Cauchy) posteriors, and ragged
    lengths 1 .. 64 over 4 000 runs (more than one wave, every warp slot of a CTA)."""
    from cpi_b200 import factor
    torch = cuda
    worst = {}
    for i, (name, fam) in enumerate(FAMILIES.items()):
        o, X, P, dR, dL = filter_runs(torch, model, seed=100 * model + i, **fam)
        inputs, _ = _k7(torch, model, o, X, P, dR, dL)
        xs, Ps, Xc = factor.rts_smooth(model, X, P, dR, dL, _dev(torch, o), cross=True)
        got = (xs.cpu().numpy(), rr.mat(Ps.cpu().numpy()), rr.mat(Xc.cpu().numpy()))
        assert all(np.all(np.isfinite(a)) for a in got), name
        if fam.get("anchor"):                                         # P_0 = 0: G = 0, Ps = 0, Xs = 0, xs = retract(x, 0)
            s0 = o[:-1]
            x = inputs[0]
            assert not np.any(got[1][s0]) and not np.any(got[2][s0 - np.arange(len(s0))])
            assert np.array_equal(got[0][s0, 4:16], x[s0, 4:16])
            assert np.max(np.abs(got[0][s0, 0:4] - x[s0, 0:4])) <= 2.0 ** -52
        r, k, col = gate(o, inputs, got, np.zeros(len(o) - 1))
        worst[name] = r
        print(f"model {model}, {name}: worst ratio {r:.3g} (keyframe {k}, column {col})")
    print(f"model {model}: worst ratio over the families {max(worst.values()):.3g}")
    assert max(worst.values()) <= 1.0, worst


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_exact_properties(cuda, model):
    """rts_smooth is bitwise K15 fed through the C ABI with the forward filter's own stored K7 outputs; repeated runs give the same
    bits; Ps is exactly symmetric; the uniform layout and the offsets tensor give the same bits; a run whose Pb is not SPD (P_0 = 0 and
    a record with P_meas = 0) is NaN alone and its CTA mates are bitwise the clean result."""
    from cpi_b200 import factor
    torch = cuda
    o, X, P, dR, dL, K7 = filter_runs(torch, model, [7] * 11, seed=300 + model, update="k11", keep_k7=True)
    do = _dev(torch, o)
    xs, Ps, Xc = factor.rts_smooth(model, X, P, dR, dL, do, cross=True)
    got = [a.cpu().numpy() for a in (xs, Ps, Xc)]
    out = [torch.empty_like(a) for a in (xs, Ps, Xc)]
    lib = capi.load()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    capi.check(lib.cpi_rts_smooth_batch(len(o) - 1, p(do), 0, int(o[-1]), p(X), p(P), p(K7[0]), p(K7[1]), p(K7[2]), p(out[0]), p(out[1]),
                                        p(out[2]), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    for a, b in zip(got, out):
        assert np.array_equal(a, b.cpu().numpy())
    for _ in range(3):
        again = [a.cpu().numpy() for a in factor.rts_smooth(model, X, P, dR, dL, do, cross=True)]
        assert all(np.array_equal(a, b) for a, b in zip(got, again))
    M = rr.mat(got[1])
    assert np.array_equal(M, M.transpose(0, 2, 1))
    uni = [a.cpu().numpy() for a in factor.rts_smooth(model, X, P, dR, dL, 7, cross=True)]
    assert all(np.array_equal(a, b) for a, b in zip(got, uni))
    no_cross = factor.rts_smooth(model, X, P, dR, dL, do)
    assert no_cross[2] is None and np.array_equal(no_cross[0].cpu().numpy(), got[0]) and np.array_equal(no_cross[1].cpu().numpy(), got[1])
    # NaN isolation: run 5 (a CTA mate of runs 4, 6 and 7) with P_0 = 0 and a record without noise
    c = 5
    P2, R2 = P.clone(), dR.clone()
    P2[int(o[c])] = 0.0
    R2[int(o[c]) - c, capi.REC["P"][0]:capi.REC["P"][1]] = 0.0
    bad = [a.cpu().numpy() for a in factor.rts_smooth(model, X, P2, R2, dL, do, cross=True)]
    s0, t0 = int(o[c]), int(o[c]) - c
    assert np.all(np.isnan(bad[1][s0])) and np.all(np.isnan(bad[2][t0]))
    keep_s = np.ones(len(got[0]), dtype=bool); keep_s[s0] = False
    keep_t = np.ones(len(got[2]), dtype=bool); keep_t[t0] = False
    assert np.array_equal(bad[1][keep_s], got[1][keep_s]) and np.array_equal(bad[0][keep_s], got[0][keep_s])
    assert np.array_equal(bad[2][keep_t], got[2][keep_t])
    # one-keyframe runs are copied, and so is every run's last keyframe
    o1, X1, P1, dR1, dL1 = filter_runs(torch, model, [1, 3, 1, 1, 4], seed=310 + model, update="k10", every=2)
    s1 = [a.cpu().numpy() for a in factor.rts_smooth(model, X1, P1, dR1, dL1, _dev(torch, o1))[:2]]
    last = o1[1:] - 1
    assert np.array_equal(s1[0][last], X1.cpu().numpy()[last]) and np.array_equal(s1[1][last], P1.cpu().numpy()[last])


@pytest.fixture(scope="module")
def stream_base(cuda):
    import test_streams as ts
    b = ts.base(cuda)
    b["cov11"] = _dev(cuda, np.tile((np.eye(15) * 1e-2).reshape(1, 225), (11, 1)) + 1e-4)
    return b


@pytest.fixture(scope="module")
def spin_rate(cuda):
    """torch.cuda._sleep's spin rate, measured once (as test_streams.cycles_per_ms)."""
    torch = cuda
    torch.cuda._sleep(1000)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    torch.cuda._sleep(20_000_000)
    b.record()
    b.synchronize()
    return 20_000_000 / a.elapsed_time(b)


def _rts_case(cross, nc):
    from cpi_b200 import factor
    import test_streams as ts
    make = lambda B, I: dict(X=I.v(B["Xr"]), c=I.v(B["cov11"]), r=I.v(B["rec"]), l=I.v(B["lin"]), o=I.v(B["offs"]))
    call = lambda a, st: factor.rts_smooth(ts.MODEL, a["X"], a["c"], a["r"], a["l"], a["o"], cross=cross, stream=st)
    return (make, call, False, nc)


@pytest.mark.gpu
@pytest.mark.parametrize("cross", [False, True])
@pytest.mark.parametrize("nc", [False, True])
def test_stream_contract(cuda, stream_base, spin_rate, monkeypatch, cross, nc):
    """The procedure of test_streams.test_stream_contract on rts_smooth over the ragged layout (runs of 4, 1 and 6 keyframes), with
    and without cross, contiguous and not: dry and wet stream-order checks, bitwise under a held caller or side stream, and the call
    returns with its stream still busy."""
    import stream_check as sc
    import test_streams as ts
    torch = cuda
    B, entry = stream_base, _rts_case(cross, nc)
    name = f"rts_smooth-cross{int(cross)}-nc{int(nc)}"
    torch.cuda.synchronize()
    for ambient in (False, True):
        S = torch.cuda.Stream()
        ck = sc.Checker(dry=True)
        with ck.active(name, monkeypatch):
            out = ts._one(torch, B, entry, S, ambient=S if ambient else None)
        torch.cuda.synchronize()
        del out
        assert not ck.errors, "\n".join(str(e) for e in ck.errors)
    S = torch.cuda.Stream()
    ck = sc.Checker(dry=False)
    with ck.active(name, monkeypatch):
        out = ts._one(torch, B, entry, S)
    torch.cuda.synchronize()
    del out
    assert not ck.errors, "\n".join(str(e) for e in ck.errors)
    make, call, _, _ = entry
    a = make(B, ts.Inputs(nc))
    torch.cuda.synchronize()
    want = ts._bytes(call(a, None))
    torch.cuda.synchronize()
    for hold in ("C", "S"):
        S = torch.cuda.Stream()
        got = ts._bytes(ts._one(torch, B, entry, S, hold=hold, cycles=int(20 * spin_rate)))
        torch.cuda.synchronize()
        assert got == want, f"{name}: held {hold} changes the result"
    S = torch.cuda.Stream()
    a = make(B, ts.Inputs(nc))
    S.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(S):
        torch.cuda._sleep(int(200 * spin_rate))
    out = call(a, S)
    busy = not S.query()
    torch.cuda.synchronize()
    del out
    assert busy, f"{name} synchronised with its stream"


def _realisations(torch, oracle, model, N, K, seed, noise=None, fixes=(3, 6, 9), sigma_fix=0.01):
    """The realisations of test_update_filter._filter_and_smoother (the same configuration and draws), restated to keep what the
    smoother of the filter needs: the truth [N, K, 16], the filter's posteriors at every keyframe (device [N K, 16], [N K, 225]), the
    records and lin (device), and chains_lm's estimate and chains_marginals' Sigma at every keyframe ([N, K, 16], [N, K, 15, 15])."""
    from cpi_b200 import factor, preint
    from test_marginalize import vec
    from test_propagate import random_cov as rc
    from test_state_priors import _fix
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
    Sig0 = rr.mat(rc(rng, 1)[0])[0]
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
    assert np.all(status.cpu().numpy() != capi.LM_NONFINITE) and np.all(status.cpu().numpy() != capi.LM_RUNNING)
    cov, _ = factor.chains_marginals(model, Xs, rec, dl, K, prior=prior, state_priors=sp)
    Xs, cov = Xs.cpu().numpy().reshape(N, K, 16), rr.mat(cov.cpu().numpy()).reshape(N, K, 15, 15)
    x, c = d(xh0), d(np.repeat(vec(Sig0[None]), N, axis=0))
    xf, cf = [x], [c]
    for k in range(K - 1):
        x, c, _ = factor.propagate(model, x, c, recK[:, k].contiguous(), linK[:, k].contiguous())
        if k + 1 in fixes:
            j = fixes.index(k + 1)
            x, c, _, applied = factor.update(x, c, d(W[j]), d(xb[j]))
            assert bool((applied == 1).all())
        xf.append(x); cf.append(c)
    Xf = torch.stack(xf, dim=1).reshape(N * K, 16)
    Cf = torch.stack(cf, dim=1).reshape(N * K, 225)
    return truth, Xf, Cf, rec, dl, Xs, cov


# The RTS smoother's distance to chains_lm's estimate at every keyframe, in chains_marginals' standard deviations (worst component over
# the 30 000 realisations of model 1): measured 0.062 on one H100 80GB HBM3 at 700 W (DESIGN.md section 3o); the gate is 4 times that.
RTS_SMOOTHER_BOUND = 0.25


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, pytest.param(2, marks=pytest.mark.xfail(strict=True, reason=(
    "model 2's filter is not consistent on this configuration (DESIGN.md section 3k), and its smoother inherits that: the smoothed "
    "mean NEES is 15.9 at keyframe 0, 15.1 at keyframe 5 and 17.5 at keyframe 9 over 30 000 realisations, and the estimate lies up "
    "to 3.9 marginal sd from chains_lm's (0.45 on average) (DESIGN.md section 3o)")))])
def test_monte_carlo_consistency_of_the_smoother_of_the_filter(cuda, oracle, model):
    """The realisations of test_update_filter.test_monte_carlo_consistency_of_the_filter (N = 30 000: seed 90 + model, three noise
    streams; K = 10; 1 cm fixes on keyframes 3, 6 and 9), filtered with K7 + K10 keeping every keyframe's posterior, then smoothed by
    rts_smooth: at every keyframe the smoothed mean NEES lies in the two-sided 99.9 % chi^2_15 band for N and every entry of the
    error's second moment lies within 5 standard errors of the mean Ps_k.  The distance to chains_lm's estimate at every keyframe, in
    chains_marginals' standard deviations, is gated at RTS_SMOOTHER_BOUND.  Model 2 fails as its filter does (a finding, kept as a
    strict expected failure so that a fix shows: DESIGN.md section 3o)."""
    from scipy.stats import chi2
    from cpi_b200 import factor
    from test_marginalize import local
    n, K, streams = 10_000, 10, (None, 1, 2)
    nees_sum, m2_sum, cov_sum = np.zeros(K), np.zeros((K, 15, 15)), np.zeros((K, 15, 15))
    dist, dist_mean = 0.0, 0.0
    for s in streams:
        truth, Xf, Cf, rec, dl, Xlm, Clm = _realisations(cuda, oracle, model, n, K, 90 + model, noise=s)
        xs, cs, _ = factor.rts_smooth(model, Xf, Cf, rec, dl, K)
        xs, cs = xs.cpu().numpy().reshape(n, K, 16), rr.mat(cs.cpu().numpy()).reshape(n, K, 15, 15)
        err = local(xs.reshape(-1, 16), truth.reshape(-1, 16)).reshape(n, K, 15)
        for k in range(K):
            e, C = err[:, k], cs[:, k]
            nees = np.einsum("ni,ni->n", e, np.linalg.solve(C, e[:, :, None])[:, :, 0])
            nees_sum[k] += nees.sum(); m2_sum[k] += e.T @ e; cov_sum[k] += C.sum(axis=0)
        z = np.abs(local(Xlm.reshape(-1, 16), xs.reshape(-1, 16))) / np.sqrt(np.diagonal(Clm.reshape(-1, 15, 15), axis1=1, axis2=2))
        dist = max(dist, float(z.max())); dist_mean += float(z.max(axis=1).sum())
    N = n * len(streams)
    lo, hi = chi2.ppf([0.0005, 0.9995], 15 * N) / N
    worst_z, outside = 0.0, []
    for k in range(K):
        M, Cm = m2_sum[k] / N, cov_sum[k] / N
        se = np.sqrt((np.outer(np.diag(Cm), np.diag(Cm)) + Cm ** 2) / N)
        z = float(np.max(np.abs((M - Cm) / se)))
        worst_z = max(worst_z, z)
        print(f"model {model}, keyframe {k}: smoothed mean NEES {nees_sum[k] / N:.3f} over {N} (band [{lo:.3f}, {hi:.3f}]), worst |z| {z:.1f}")
        if not lo <= nees_sum[k] / N <= hi:
            outside.append((k, float(nees_sum[k] / N)))
    print(f"model {model}: RTS - chains_lm at every keyframe, in the smoother's marginal sd: worst {dist:.3e}, "
          f"mean of the per-keyframe worst {dist_mean / (N * K):.3e}")
    assert not outside, outside
    assert worst_z <= 5.0, worst_z
    assert dist <= RTS_SMOOTHER_BOUND, (dist, RTS_SMOOTHER_BOUND)
