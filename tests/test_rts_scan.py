"""Parallel-in-time Rauch-Tung-Striebel smoothing of filter runs (cpi_rts_smooth_scan_batch, kernel K16, factor.rts_smooth_scan;
DESIGN.md section 3p).

CPU: the numpy statement (tests/rts_scan_ref.py): J_k against central differences, its two bracketings against each other, its
covariances against dense inverses and K15's statement, its means' second-order distance to K15's, the exact d0 = 0 identity, the
argument checks of the C ABI and the binding, and the sensitivity of the precision gate.
GPU: K16 against the statement in long double on filter runs of every update kernel and on long and chunk-boundary layouts, against
K15 on the same inputs, the identity with chains_marginals, exact properties, the stream contract and Monte-Carlo consistency.

The precision gate is test_rts's: errors in the truth's smoothed standard deviations, per run and per output block, at
8 max(e_64, floor, 1e-15), with e_64 the larger worst error of the fp64 statement in its two bracketings (sequential and a pairwise
tree), pooled over the family, and Ps exactly symmetric."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest

import rts_ref as rr
import rts_scan_ref as sr
from cpi_b200 import capi, synth
from test_chain_marginals import inv_truth
from test_rts import (FAMILIES, _dev, _err, _k7, _scaled, filter_runs, linear_runs, spin_rate, stream_base)  # noqa: F401

K_GATE, FLOOR = 8.0, 1e-15


def gate(offs, inputs, got, groups, truth=None, cols=None):
    """(worst ratio e_dev / (K_GATE max(e_64, floor, FLOOR)), its keyframe and column) of got = (xs, Ps, Xs); e_64 is the worse of
    the fp64 statement's sequential and tree bracketings, pooled over groups [n_runs].  Keyframes whose truth is not finite are
    skipped (and must be NaN in got); cols restricts the columns of test_rts._err (0: Ps, 1..15: the state, 16: Xs).  inf if Ps is not exactly
    symmetric."""
    o = np.asarray(offs, dtype=np.int64)
    truth = truth if truth is not None else sr.sequential(o, *inputs, dtype=np.longdouble)
    e_dev = _err(truth, got, o)
    e_64 = np.maximum(_err(truth, sr.sequential(o, *inputs), o), _err(truth, sr.tree(o, *inputs), o))
    run_of = np.repeat(np.arange(len(o) - 1), o[1:] - o[:-1])
    skip = ~np.all(np.isfinite(np.asarray(truth[1], dtype=np.float64)), axis=(1, 2))
    assert np.all(np.isnan(np.asarray(got[1])[skip]))
    g = np.asarray(groups)[run_of]
    pooled = np.zeros_like(e_64)
    for lab in np.unique(g):
        m = (g == lab) & ~skip
        if m.any():
            pooled[g == lab] = e_64[m].max(axis=0)
    floor = np.zeros_like(e_64)
    floor[:, 1:16] = rr.state_floor(truth)
    with np.errstate(invalid="ignore"):
        ratio = e_dev / (K_GATE * np.maximum(np.maximum(pooled, floor), FLOOR))
    ratio[skip] = 0.0
    if cols is not None:
        ratio = ratio[:, cols]
    Ps = np.asarray(got[1])
    if not np.array_equal(Ps[~skip], np.swapaxes(Ps[~skip], 1, 2)):
        return np.inf, -1, -1
    i = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
    return float(ratio[i]), int(i[0]), int(i[1])


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------

def test_jacobian_against_central_differences():
    """J_k = d local(xb, retract(x, delta)) / d delta at 0 is diag(Jr^-1(phi), I_12), phi the rotation of local(xb, x), against
    central differences through the statement's retract and local, at random states and rotations up to pi - 1e-3."""
    rng = np.random.default_rng(41)
    worst = 0.0
    for th in list(rng.uniform(0.0, 3.0, 12)) + [1e-6, 0.0, np.pi - 1e-2, np.pi - 1e-3]:
        x = np.zeros((1, 16))
        q = rng.normal(size=4); q /= np.linalg.norm(q); q *= np.sign(q[3])
        x[0, 0:4], x[0, 4:16] = q, rng.normal(size=12)
        phi = rng.normal(size=3); phi *= th / np.linalg.norm(phi)
        xb = rr.retract(x, np.concatenate([-phi, rng.normal(size=12)])[None])
        d0 = rr.local(xb, x)[0]
        J = np.zeros((15, 15))
        h = 1e-6
        for i in range(15):
            e = np.zeros((1, 15)); e[0, i] = h
            J[:, i] = (rr.local(xb, rr.retract(x, e))[0] - rr.local(xb, rr.retract(x, -e))[0]) / (2 * h)
        want = np.eye(15)
        want[0:3, 0:3] = sr.jr_inv(d0[None, 0:3])[0]
        worst = max(worst, float(np.max(np.abs(J - want))))
    print(f"J against central differences: worst {worst:.2e}")
    assert worst < 1e-8, worst
    assert np.array_equal(sr.jr_inv(np.zeros((1, 3)))[0], np.eye(3))


def test_bracketings_agree_in_long_double():
    """The sequential recursion and the Kogge-Stone tree of the element compositions agree to long-double rounding, on ragged runs
    whose elements are far from commuting."""
    rng = np.random.default_rng(42)
    o, inputs, _ = linear_runs(rng, [1, 2, 5, 12, 30, 17, 33])
    a = sr.sequential(o, *inputs, dtype=np.longdouble)
    b = sr.tree(o, *inputs, dtype=np.longdouble)
    rel = max(float(np.max(np.abs(u - v)) / max(np.max(np.abs(u)), 1e-300)) for u, v in zip(a, b))
    print(f"sequential against tree in long double: {rel:.2e} relative")
    assert rel < 1e-16, rel


@pytest.mark.parametrize("dtype", [np.float64, np.longdouble])
def test_covariances_are_the_dense_inverse_and_k15s(dtype):
    """Ps_k and Xs_k are the blocks of the inverse of each linear-Gaussian run's information matrix (as test_rts), and equal K15's
    statement to long-double rounding."""
    rng = np.random.default_rng(31)
    o, inputs, infos = linear_runs(rng, [1, 2, 5, 12, 30])
    xs, Ps, Xs = sr.tree(o, *inputs, dtype=dtype)
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
    assert worst < 1e-8, worst
    assert np.array_equal(Ps, np.swapaxes(Ps, 1, 2))
    if dtype is np.longdouble:
        _, Pk, Xk = rr.rts(o, *inputs, dtype=np.longdouble)
        assert float(np.max(np.abs(Pk - Ps))) < 1e-17 * float(np.max(np.abs(Pk)))
        assert float(np.max(np.abs(Xk - Xs))) < 1e-17 * float(np.max(np.abs(Xk)))


def _with_corrections(rng, o, inputs, h):
    """inputs with xb_{k+1} = retract(x_{k+1}, -h u_k), u_k fixed random directions (h = 0: xb_{k+1} = x_{k+1}): the filter's
    correction d0_k = O(h)."""
    x, P, xb, Pb, C = inputs
    R = len(o) - 1
    s = np.concatenate([np.arange(o[c], o[c + 1] - 1) for c in range(R)]).astype(np.int64)
    u = np.random.default_rng(7).normal(size=(len(s), 15)) * np.array([1e-1] * 3 + [1.0] * 12)
    xb = rr.retract(x[s + 1], -h * u) if h else x[s + 1].copy()
    return x, P, xb, Pb, C


def test_means_identity_and_second_order():
    """Every d0 = 0 gives delta = 0 exactly (the linear entries copied, the quaternion renormalised within an ulp).  With d0 = O(h)
    the means differ from K15's statement by O(|phi| |delta|^2) = O(h^3): second order in delta, and local(xb, retract(x, delta)) is
    linear in the 12 linear entries and has no delta^2 term at phi = 0 (Baker-Campbell-Hausdorff), so halving h cuts the difference
    by about 8.  Every difference is far above the long-double floor, and the last transition of every run is K15's expression
    exactly."""
    rng = np.random.default_rng(43)
    o, inputs, _ = linear_runs(rng, [2, 5, 12, 30])
    x, P, xb, Pb, C = _with_corrections(rng, o, inputs, 0.0)
    assert not np.any(rr.local(xb, x[np.concatenate([np.arange(o[c] + 1, o[c + 1]) for c in range(len(o) - 1)])]))
    xs, _, _ = sr.tree(o, x, P, xb, Pb, C)
    assert np.array_equal(xs[:, 4:16], x[:, 4:16])
    assert np.max(np.abs(xs[:, 0:4] - x[:, 0:4])) <= 2.0 ** -52
    diffs = []
    for h in (4e-2, 2e-2, 1e-2):
        inp = _with_corrections(rng, o, inputs, h)
        a = sr.sequential(o, *inp, dtype=np.longdouble)[0]
        b = rr.rts(o, *inp, dtype=np.longdouble)[0]
        d = np.abs(np.asarray(rr.local(a, b), dtype=np.float64))
        last = o[1:] - 2                                               # the last transition: the same expression
        assert float(np.max(d[last])) < 1e-15
        diffs.append(float(np.max(d)))
    ratios = [diffs[i] / diffs[i + 1] for i in range(2)]
    print(f"means: max |local(K16, K15)| {diffs}, ratios {ratios}")
    assert min(diffs) > 1e-10
    assert all(7.0 < r < 9.0 for r in ratios), ratios


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def test_argument_validation_without_gpu():
    """cpi_rts_smooth_scan_batch rejects bad arguments with CPI_EINVAL before any CUDA call (those of cpi_rts_smooth_batch, a NULL
    workspace when a run has a transition, a workspace equal to an input or output), n_runs = 0 launches nothing; the workspace
    function rejects negative counts and n_states < n_runs; the binding rejects models, host tensors and non-tensors."""
    import torch
    from cpi_b200 import factor
    lib = capi.load()
    bufs = [np.zeros(16 * 225) for _ in range(11)]
    p = [_p(b) for b in bufs]
    rts = lambda *a: lib.cpi_rts_smooth_scan_batch(*a, None)
    before = capi.launch_count()
    assert lib.cpi_rts_smooth_scan_workspace(-1, 4) == -1 and lib.cpi_rts_smooth_scan_workspace(2, -1) == -1
    assert lib.cpi_rts_smooth_scan_workspace(3, 2) == -1 and lib.cpi_rts_smooth_scan_workspace(3, 3) == 0
    assert lib.cpi_rts_smooth_scan_workspace(1, 2) == 2 * 691 * 8
    assert lib.cpi_rts_smooth_scan_workspace(1, 17) == (17 + 2) * 691 * 8
    assert rts(-1, None, 2, 4, *p[1:11]) == -1 and b"negative" in lib.cpi_last_error()
    assert rts(2, None, 0, 4, *p[1:11]) == -1 and b"uniform" in lib.cpi_last_error()
    assert rts(2, None, 2, 5, *p[1:11]) == -1 and b"n_states" in lib.cpi_last_error()
    assert rts(3, p[0], 0, 2, *p[1:11]) == -1 and b"n_states" in lib.cpi_last_error()
    for k in list(range(7)) + [8]:                                     # states .. cov_out, workspace (cross_out may be NULL)
        a = list(p[1:11]); a[k] = None
        assert rts(2, None, 2, 4, *a) == -1 and b"null" in lib.cpi_last_error(), k
    for o in (5, 6, 7, 8):                                             # an output or the workspace equal to an input
        for i in range(5):
            a = list(p[1:11]); a[o] = a[i]
            assert rts(2, None, 2, 4, *a) == -1 and b"overlap inputs" in lib.cpi_last_error(), (o, i)
    for o1, o2 in ((5, 6), (5, 7), (6, 7), (5, 8), (6, 8), (7, 8)):
        a = list(p[1:11]); a[o2] = a[o1]
        assert rts(2, None, 2, 4, *a) == -1 and b"overlap each other" in lib.cpi_last_error(), (o1, o2)
    assert rts(0, None, 1, 0, *[None] * 10) == 0
    assert capi.launch_count() == before
    f64 = dict(dtype=torch.float64)
    X, C, rec, lin = torch.zeros((6, 16), **f64), torch.zeros((6, 225), **f64), torch.zeros((4, 290), **f64), torch.zeros((4, 13), **f64)
    with pytest.raises(ValueError, match="model"):
        factor.rts_smooth_scan(3, X, C, rec, lin, 3)
    with pytest.raises(ValueError, match="CUDA"):
        factor.rts_smooth_scan(1, X, C, rec, lin, 3)
    with pytest.raises(ValueError, match="tensor"):
        factor.rts_smooth_scan(1, X.numpy(), C, rec, lin, 3)


@pytest.mark.parametrize("inject", ["Pb-fp32", "G-scaled", "no-mirror", "flag-by-product"])
def test_gate_is_sensitive(inject):
    """Four injected errors in the fp64 statement fail the gate that the clean tree passes: Pb rounded to fp32, G scaled by
    1 + 1e-7, L and the compositions without the mirror, and run boundaries applied by multiplying by 0 (a run whose Pb is not SPD
    then leaks NaN into its neighbours)."""
    rng = np.random.default_rng(33)
    o, inputs, _ = linear_runs(rng, [3, 8, 20, 5, 9])
    x, P, xb, Pb, C = inputs
    if inject == "flag-by-product":                                   # run 3: Pb not SPD
        Pb = Pb.copy()
        Pb[int(o[3]) - 3] = -np.eye(15)
        inputs = (x, P, xb, Pb, C)
    groups = np.zeros(len(o) - 1)
    truth = sr.sequential(o, *inputs, dtype=np.longdouble)
    assert gate(o, inputs, sr.tree(o, *inputs), groups, truth)[0] <= 1.0 / K_GATE + 1e-12
    f = {"Pb-fp32": lambda n, v: v.astype(np.float32).astype(np.float64) if n == "Pb" else v,
         "G-scaled": lambda n, v: v * (1 + 1e-7) if n == "G" else v}.get(inject)
    bad = sr.tree(o, *inputs, inject=f, mirror=inject != "no-mirror", flag_by_product=inject == "flag-by-product")
    ratio = gate(o, inputs, bad, groups, truth)
    print(f"{inject}: worst ratio {ratio[0]:.3g} at keyframe {ratio[1]}, column {ratio[2]}")
    assert ratio[0] > 1.0, ratio


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------

CH = 16                                                                # K16's chunk
SCAN_FAMILIES = dict(FAMILIES, **{
    "one-4999": dict(lengths=[4999], update="k10", every=50),
    "three-20000": dict(lengths=[20000] * 3, update="k10", every=400),
    "chunk-edges": dict(lengths=[CH - 1, CH, CH + 1, CH * CH - 1, CH * CH, CH * CH + 1, 1, CH * CH * CH + 1], update="k10", every=5),
})


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_against_the_long_double_statement(cuda, model):
    """K16 (through rts_smooth_scan) against the statement in long double on the K7 outputs the binding computes, per run and
    output block: test_rts's families, one run of 4 999, three runs of 20 000 and lengths at the chunk and level edges.  K15 on the
    same inputs: its covariances and cross within the same gate, and the distance of its means reported."""
    from cpi_b200 import factor
    torch = cuda
    worst, worst_k15, mean_dist = {}, {}, {}
    for i, (name, fam) in enumerate(SCAN_FAMILIES.items()):
        o, X, P, dR, dL = filter_runs(torch, model, seed=500 + 100 * model + i, **fam)
        inputs, _ = _k7(torch, model, o, X, P, dR, dL)
        do = _dev(torch, o)
        xs, Ps, Xc = factor.rts_smooth_scan(model, X, P, dR, dL, do, cross=True)
        got = (xs.cpu().numpy(), rr.mat(Ps.cpu().numpy()), rr.mat(Xc.cpu().numpy()))
        assert all(np.all(np.isfinite(a)) for a in got), name
        truth = sr.sequential(o, *inputs, dtype=np.longdouble)
        r, k, col = gate(o, inputs, got, np.zeros(len(o) - 1), truth)
        worst[name] = r
        ks, Pk, Xk = factor.rts_smooth(model, X, P, dR, dL, do, cross=True)
        k15 = (ks.cpu().numpy(), rr.mat(Pk.cpu().numpy()), rr.mat(Xk.cpu().numpy()))
        worst_k15[name] = gate(o, inputs, k15, np.zeros(len(o) - 1), truth, cols=[0, 16])[0]
        sd = np.sqrt(np.diagonal(got[1], axis1=1, axis2=2))
        with np.errstate(invalid="ignore", divide="ignore"):
            mean_dist[name] = float(np.max(np.where(sd > 0, np.abs(rr.local(got[0], k15[0])) / np.where(sd > 0, sd, 1.0), 0.0)))
        print(f"model {model}, {name}: worst ratio {r:.3g} (keyframe {k}, column {col}); K15's covariances {worst_k15[name]:.3g}; "
              f"K15's means at {mean_dist[name]:.3e} smoothed sd")
    print(f"model {model}: worst ratio over the families {max(worst.values()):.3g}, K15 {max(worst_k15.values()):.3g}, "
          f"means {max(mean_dist.values()):.3e} sd")
    assert max(worst.values()) <= 1.0, worst
    assert max(worst_k15.values()) <= 1.0, worst_k15
    assert max(mean_dist.values()) <= SCAN_K15_MEANS_BOUND, mean_dist


# The distance between K16's and K15's smoothed means over the families above, in K16's smoothed standard deviations (worst
# component, both models): measured 0.057 (model 1, K11 posteriors) on one H100 80GB HBM3 (DESIGN.md section 3p); the gate is 4
# times that.
SCAN_K15_MEANS_BOUND = 0.23


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_smoother_of_the_filter_is_the_chain_smoother(cuda, monkeypatch, model):
    """test_rts's chain at its exact prediction with 1 cm fixes (d = 0 up to K10's renormalised quaternion), smoothed by
    rts_smooth_scan: Ps and Xs are chains_marginals' within test_rts's 20x-numpy gate and the means are the filtered ones within
    1e-12 smoothed sd (test_rts's own checks); after the last fix, where every d0 is exactly 0, the linear entries are bitwise the
    filtered ones and the quaternions within an ulp."""
    import test_rts
    from cpi_b200 import factor
    seen = {}

    def scan(model_, X, Cf, dR, dL, offs, cross=False, **kw):
        out = factor.rts_smooth_scan(model_, X, Cf, dR, dL, offs, cross=cross, **kw)
        seen.update(X=X.cpu().numpy(), xs=out[0].cpu().numpy())
        return out
    monkeypatch.setattr(factor, "rts_smooth", scan)
    test_rts.test_smoother_of_the_filter_is_the_chain_smoother(cuda, model)
    X, xs = seen["X"], seen["xs"]
    assert np.array_equal(xs[20:, 4:16], X[20:, 4:16])
    assert np.max(np.abs(xs[:, 0:4] - X[:, 0:4])) <= 4 * 2.0 ** -52


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_exact_properties(cuda, model):
    """rts_smooth_scan is bitwise K16 through the C ABI with the forward filter's own K7 outputs; repeated runs give the same bits;
    Ps is exactly symmetric; the uniform layout and the offsets tensor give the same bits; dead-reckoned runs (every d0 = 0) keep
    their linear entries bitwise and their quaternions within an ulp; a run whose Pb is not SPD is NaN alone and every other run,
    its chunk mates included, is bitwise the clean result; one-keyframe runs and last keyframes are copied."""
    from cpi_b200 import factor
    torch = cuda
    o, X, P, dR, dL, K7 = filter_runs(torch, model, [7] * 11, seed=700 + model, update="k11", keep_k7=True)
    do = _dev(torch, o)
    xs, Ps, Xc = factor.rts_smooth_scan(model, X, P, dR, dL, do, cross=True)
    got = [a.cpu().numpy() for a in (xs, Ps, Xc)]
    out = [torch.empty_like(a) for a in (xs, Ps, Xc)]
    lib = capi.load()
    N, R = int(o[-1]), len(o) - 1
    ws = torch.empty(int(lib.cpi_rts_smooth_scan_workspace(R, N)), dtype=torch.uint8, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    capi.check(lib.cpi_rts_smooth_scan_batch(R, p(do), 0, N, p(X), p(P), p(K7[0]), p(K7[1]), p(K7[2]), p(out[0]), p(out[1]), p(out[2]),
                                             p(ws), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    for a, b in zip(got, out):
        assert np.array_equal(a, b.cpu().numpy())
    for _ in range(3):
        again = [a.cpu().numpy() for a in factor.rts_smooth_scan(model, X, P, dR, dL, do, cross=True)]
        assert all(np.array_equal(a, b) for a, b in zip(got, again))
    M = rr.mat(got[1])
    assert np.array_equal(M, M.transpose(0, 2, 1))
    uni = [a.cpu().numpy() for a in factor.rts_smooth_scan(model, X, P, dR, dL, 7, cross=True)]
    assert all(np.array_equal(a, b) for a, b in zip(got, uni))
    no_cross = factor.rts_smooth_scan(model, X, P, dR, dL, do)
    assert no_cross[2] is None and np.array_equal(no_cross[0].cpu().numpy(), got[0]) and np.array_equal(no_cross[1].cpu().numpy(), got[1])
    # NaN isolation: run 5 (keyframes 35 .. 41, sharing 16-element chunks with runs 3, 4 and 6) with P_0 = 0 and a noiseless record
    c = 5
    P2, R2 = P.clone(), dR.clone()
    P2[int(o[c])] = 0.0
    R2[int(o[c]) - c, capi.REC["P"][0]:capi.REC["P"][1]] = 0.0
    bad = [a.cpu().numpy() for a in factor.rts_smooth_scan(model, X, P2, R2, dL, do, cross=True)]
    s0, t0 = int(o[c]), int(o[c]) - c
    assert np.all(np.isnan(bad[1][s0])) and np.all(np.isnan(bad[2][t0]))
    keep_s = np.ones(N, dtype=bool); keep_s[o[c]:o[c + 1]] = False
    keep_t = np.ones(N - R, dtype=bool); keep_t[o[c] - c:o[c + 1] - c - 1] = False
    for a, b, k in ((bad[0], got[0], keep_s), (bad[1], got[1], keep_s), (bad[2], got[2], keep_t)):
        assert np.array_equal(a[k], b[k])
    # every d0 = 0: dead-reckoned runs
    o3, X3, P3, dR3, dL3 = filter_runs(torch, model, [40, 3, 17], seed=720 + model, dead=True)
    x3 = X3.cpu().numpy()
    s3 = factor.rts_smooth_scan(model, X3, P3, dR3, dL3, _dev(torch, o3))[0].cpu().numpy()
    assert np.array_equal(s3[:, 4:16], x3[:, 4:16])
    assert np.max(np.abs(s3[:, 0:4] - x3[:, 0:4])) <= 2.0 ** -52
    # one-keyframe runs are copied, and so is every run's last keyframe
    o1, X1, P1, dR1, dL1 = filter_runs(torch, model, [1, 3, 1, 1, 4], seed=710 + model, update="k10", every=2)
    s1 = [a.cpu().numpy() for a in factor.rts_smooth_scan(model, X1, P1, dR1, dL1, _dev(torch, o1))[:2]]
    last = o1[1:] - 1
    assert np.array_equal(s1[0][last], X1.cpu().numpy()[last]) and np.array_equal(s1[1][last], P1.cpu().numpy()[last])
    o0 = np.arange(4, dtype=np.int64)                                  # only one-keyframe runs: no workspace, copies
    e = torch.empty((0, dR1.shape[1]), dtype=torch.float64, device="cuda")
    s0_ = factor.rts_smooth_scan(model, X1[:3], P1[:3], e, torch.empty((0, 13), dtype=torch.float64, device="cuda"), _dev(torch, o0))
    assert torch.equal(s0_[0], X1[:3]) and torch.equal(s0_[1], P1[:3])


def _scan_case(cross, nc):
    from cpi_b200 import factor
    import test_streams as ts
    make = lambda B, I: dict(X=I.v(B["Xr"]), c=I.v(B["cov11"]), r=I.v(B["rec"]), l=I.v(B["lin"]), o=I.v(B["offs"]))
    call = lambda a, st: factor.rts_smooth_scan(ts.MODEL, a["X"], a["c"], a["r"], a["l"], a["o"], cross=cross, stream=st)
    return (make, call, False, nc)


@pytest.mark.gpu
@pytest.mark.parametrize("cross", [False, True])
@pytest.mark.parametrize("nc", [False, True])
def test_stream_contract(cuda, stream_base, spin_rate, monkeypatch, cross, nc):
    """test_rts's stream procedure on rts_smooth_scan over the ragged layout (runs of 4, 1 and 6 keyframes), with and without cross,
    contiguous and not: dry and wet stream-order checks, bitwise under a held caller or side stream, and the call returns with its
    stream still busy."""
    import test_rts
    monkeypatch.setattr(test_rts, "_rts_case", _scan_case)
    test_rts.test_stream_contract(cuda, stream_base, spin_rate, monkeypatch, cross, nc)


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, pytest.param(2, marks=pytest.mark.xfail(strict=True, reason=(
    "model 2's filter is not consistent on this configuration (DESIGN.md section 3k), and K16 inherits that as K15 does: the "
    "smoothed mean NEES is 15.9 at keyframe 0, 15.1 at keyframe 5 and 17.5 at keyframe 9 over 30 000 realisations, and the estimate "
    "lies up to 3.9 marginal sd from chains_lm's (0.45 on average) (DESIGN.md section 3p)")))])
def test_monte_carlo_consistency(cuda, oracle, monkeypatch, model):
    """test_rts's Monte-Carlo consistency test (30 000 realisations, 1 cm fixes on keyframes 3, 6 and 9) smoothed by
    rts_smooth_scan: the smoothed mean NEES in the 99.9 % chi^2_15 band at every keyframe, the error's second moment within 5
    standard errors of the mean Ps_k, and the distance to chains_lm's estimate within test_rts's RTS_SMOOTHER_BOUND."""
    import test_rts
    from cpi_b200 import factor
    monkeypatch.setattr(factor, "rts_smooth", factor.rts_smooth_scan)
    test_rts.test_monte_carlo_consistency_of_the_smoother_of_the_filter(cuda, oracle, model)
