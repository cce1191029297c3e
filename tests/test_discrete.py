"""Discrete (Forster) preintegration into model-1 records, CPI_FLAG_DISCRETE (include/cpi_b200.h, DESIGN.md section 3n).

Parity with GTSAM is unpinned: ``discrete_ref`` is the specification.  The CPU tests pin the statement's conventions (bias
Jacobians by central differences, first-order convergence to model 1 under step splitting, composition, edge cases) and the
rejections of the C ABI and the wrappers; the GPU tests gate the kernel against the statement."""
import ctypes

import numpy as np
import pytest

import discrete_ref as dr
from cpi_b200 import capi, synth
from parity import REC, conditioned_gate

P = lambda a: ctypes.c_void_p(a.ctypes.data)
SIG = synth.SIGMAS
FL = capi.FLAG_DISCRETE


def _windows(n, ns, seed=11, rate=200.0):
    S, L = synth.make_windows(n, ns, rate=rate, seed=seed)
    return S, L


def _special(S, L):
    """(Taylor-branch, exact-zero w_hat, dt = 0 step) window masks of a synth batch."""
    wh = S[:, :, 0:3] - L[:, None, 0:3]
    mag = np.linalg.norm(wh, axis=2)
    return np.all(mag < dr.SMALL_W, axis=1) & np.any(mag > 0, axis=1), np.all(mag == 0, axis=1), np.any(S[:, :, 6] == 0, axis=1)


def _pick(S, L, n_ord=12):
    """Ordinary windows plus every special window of the batch."""
    small, zero, dz = _special(S, L)
    idx = np.concatenate([np.arange(n_ord), np.where(small | zero | dz)[0]])
    return S[idx], L[idx], small[idx], zero[idx]


# ------------------------------------------------------------------------------------------------------------------
# CPU: the statement's conventions
# ------------------------------------------------------------------------------------------------------------------

def test_bias_jacobians_are_central_differences():
    """J_q, J_a, J_b, H_a, H_b of the statement are the derivatives of its R, alpha, beta with respect to lin's biases, in the
    convention R(b + d) = Exp(J_q d_w) R(b), alpha/beta(b + d) = alpha/beta + J d_w + H d_a."""
    S, L = _windows(1500, 30)
    S, L, small, zero = _pick(S, L)
    assert small.any() and zero.any()
    n, ns = L.shape[0], S.shape[1]
    ld = np.longdouble
    run = lambda Lx: dr.preintegrate(S.reshape(-1, 7), Lx, SIG, ns=ns, dtype=ld)
    r0 = run(L)
    h = 1e-6
    for k in range(6):
        Lp, Lm = L.astype(ld).copy(), L.astype(ld).copy()
        Lp[:, k] += h; Lm[:, k] -= h
        rp, rm = run(Lp), run(Lm)
        Rp = rp[:, 4:13].reshape(n, 3, 3).transpose(0, 2, 1); Rm = rm[:, 4:13].reshape(n, 3, 3).transpose(0, 2, 1)
        D = Rp @ Rm.transpose(0, 2, 1)
        dth = np.stack([D[:, 2, 1] - D[:, 1, 2], D[:, 0, 2] - D[:, 2, 0], D[:, 1, 0] - D[:, 0, 1]], axis=1) / 2 / (2 * h)
        dal = (rp[:, 13:16] - rm[:, 13:16]) / (2 * h)
        dbe = (rp[:, 16:19] - rm[:, 16:19]) / (2 * h)
        col = lambda f: r0[:, REC[f][0]:REC[f][1]].reshape(n, 3, 3).transpose(0, 2, 1)[:, :, k % 3]
        pairs = [("J_q", dth), ("J_a", dal), ("J_b", dbe)] if k < 3 else [("H_a", dal), ("H_b", dbe)]
        if k >= 3:
            assert np.all(np.abs(dth) < 1e-12)
        for f, fd in pairs:
            J = col(f).astype(np.float64); fd = fd.astype(np.float64)
            scale = np.maximum(np.linalg.norm(J, axis=1), 1e-300)
            err = np.linalg.norm(J - fd, axis=1) / scale
            assert err.max() < 1e-7, (f, k, err.max(), int(np.argmax(err)))


def _split(S, m):
    """Every step of every window cut into m equal sub-steps with the same readings."""
    Sm = np.repeat(S, m, axis=1)
    Sm[:, :, 6] = Sm[:, :, 6] / m
    return Sm


BLOCKS = ("th", "bg", "v", "ba", "p")
FIRST_ORDER = ("alpha", "beta", "J_a", "J_b", "H_a", "H_b")


def _pblocks(rec):
    n = rec.shape[0]
    Pm = rec[:, 65:290].reshape(n, 15, 15).transpose(0, 2, 1)
    return {f"P_{BLOCKS[I]}{BLOCKS[J]}": Pm[:, 3 * I:3 * I + 3, 3 * J:3 * J + 3] for I in range(5) for J in range(I + 1)}


def test_converges_to_model_1_at_first_order(oracle):
    """Model 1 is exact for piecewise-constant readings, so splitting every step into m sub-steps leaves its record unchanged
    (P up to RK4 truncation).  The discrete record's distance to it falls as 1/m for the means, J_a, J_b, H_a, H_b and the P blocks
    of the v and p rows; the other P blocks are at rounding or fall at least as fast; R, q and J_q agree to rounding at every m."""
    S, L = _windows(24, 40, seed=5)
    small, zero, dz = _special(S, L)
    S, L = S[~(small | zero | dz)], L[~(small | zero | dz)]
    n, ns = L.shape[0], S.shape[1]
    ref = oracle.preintegrate(1, S.reshape(-1, 7), L, SIG, 0, ns=ns)
    refP = _pblocks(ref)
    dist = {}
    for m in (1, 2, 4, 8, 16):
        d = dr.preintegrate(_split(S, m).reshape(-1, 7), L, SIG, ns=ns * m)
        for f in ("R", "q", "J_q"):
            a, b = REC[f]
            assert np.abs(d[:, a:b] - ref[:, a:b]).max() < 1e-13 * max(1.0, np.abs(ref[:, a:b]).max()), (f, m)
        for f in FIRST_ORDER:
            a, b = REC[f]
            dist.setdefault(f, []).append(np.linalg.norm(d[:, a:b] - ref[:, a:b]) / np.linalg.norm(ref[:, a:b]))
        for k, blk in _pblocks(d).items():
            dist.setdefault(k, []).append(np.linalg.norm(blk - refP[k]) / max(np.linalg.norm(refP[k]), 1e-300))
    floor = 1e-12                        # relative distance at which a block counts as agreeing to rounding
    report = {}
    for k, ds in dist.items():
        ratios = [ds[i] / ds[i + 1] if ds[i + 1] > 0 else np.inf for i in range(len(ds) - 1)]
        report[k] = (ds[0], ratios)
        first = k in FIRST_ORDER or (k.startswith("P_") and k[2] in "vp")      # the v and p rows
        if first:
            assert min(ds) > floor, (k, ds)          # every first-order field is checked by its ratios, never waved through
            assert all(1.8 <= r <= 2.2 for r in ratios), (k, ds, ratios)
        else:
            assert all(ds[i + 1] <= floor or r >= 1.8 for i, r in enumerate(ratios)), (k, ds, ratios)
    print({k: (f"{v[0]:.2e}", [round(r, 3) for r in v[1]]) for k, v in report.items()})


def test_zero_rate_windows_agree_with_model_1(oracle):
    """With exact-zero w_hat the rotation is constant and Euler steps integrate constant readings exactly."""
    S, L = _windows(3000, 30, seed=3)
    small, zero, dz = _special(S, L)
    S, L = S[zero & ~dz], L[zero & ~dz]
    assert L.shape[0] > 0
    ref = oracle.preintegrate(1, S.reshape(-1, 7), L, SIG, 0, ns=S.shape[1])
    d = dr.preintegrate(S.reshape(-1, 7), L, SIG, ns=S.shape[1])
    for f in ("R", "q", "J_q", "alpha", "beta", "H_a", "H_b", "DT"):
        a, b = REC[f]
        assert np.abs(d[:, a:b] - ref[:, a:b]).max() <= 1e-13 * max(1.0, np.abs(ref[:, a:b]).max()), f


def test_statement_composes_bitwise():
    """The statement over a whole window equals the statement continued over its parts, bit for bit in float64."""
    S, L = _windows(40, 50, seed=7)
    one = dr.preintegrate(S.reshape(-1, 7), L, SIG, ns=50)
    for cut in (1, 17, 49):
        a = dr.preintegrate(S[:, :cut].reshape(-1, 7), L, SIG, ns=cut)
        b = dr.preintegrate(S[:, cut:].reshape(-1, 7), L, SIG, ns=50 - cut, init=a)
        assert np.array_equal(b, one), cut


def test_zero_dt_step_and_empty_window():
    S, L = _windows(8, 20, seed=9)
    base = dr.preintegrate(S.reshape(-1, 7), L, SIG, ns=20)
    Z = np.concatenate([S[:, :7], S[:, 7:8] * np.array([1, 1, 1, 1, 1, 1, 0]), S[:, 7:]], axis=1)
    assert np.array_equal(dr.preintegrate(Z.reshape(-1, 7), L, SIG, ns=21), base)
    off = np.zeros(9, dtype=np.int64)
    e = dr.preintegrate(np.zeros((0, 7)), L, SIG, offsets=off)
    zero = np.zeros(290); zero[3] = 1.0; zero[[4, 8, 12]] = 1.0
    assert np.array_equal(e, np.broadcast_to(zero, e.shape))


def test_rejections_before_the_device():
    """Model 2 and dtype 32 with CPI_FLAG_DISCRETE are CPI_EINVAL before any CUDA call, in the C ABI and in the wrappers."""
    from cpi_b200 import factor, preint
    lib = capi.load()
    buf = np.zeros(4096)
    for fn in (lib.cpi_preintegrate_batch, lib.cpi_preintegrate_batch_continue):
        rc = fn(2, 64, 1, None, 1, P(buf), P(buf), P(buf), FL, P(buf), None)
        assert rc == -1 and b"model must be 1" in lib.cpi_last_error()
        rc = fn(1, 32, 1, None, 1, P(buf), P(buf), P(buf), FL, P(buf), None)
        assert rc == -1 and b"fp64 only" in lib.cpi_last_error()
    rc = lib.cpi_preintegrate_batch_host(2, 64, 1, None, 1, P(buf), P(buf), P(buf), FL, P(buf))
    assert rc == -1 and b"model must be 1" in lib.cpi_last_error()
    rc = lib.cpi_preintegrate_batch_host(1, 32, 1, None, 1, P(buf), P(buf), P(buf), FL, P(buf))
    assert rc == -1 and b"fp64 only" in lib.cpi_last_error()
    rc = lib.cpi_imu_records_relinearize(2, 1, P(buf), None, None, 1, P(buf), P(buf), FL, 0.0, 0.0, 0.0, P(buf), P(buf), None, None,
                                         P(buf), None)
    assert rc == -1 and b"model must be 1" in lib.cpi_last_error()
    S, L = _windows(2, 4)
    with pytest.raises(ValueError, match="model must be 1"):
        preint.preintegrate_host(2, S, L, SIG, FL)
    with pytest.raises(ValueError, match="fp64"):
        preint.preintegrate_host(1, S.astype(np.float32), L.astype(np.float32), SIG, FL)
    with pytest.raises(ValueError, match="model must be 1"):
        factor.relinearize_records(2, None, None, None, None, None, SIG, flags=FL, tol_bw=0.0, tol_ba=0.0)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the kernel against the statement
# ------------------------------------------------------------------------------------------------------------------

def _csr_batch(n, seed, lmax=400, avg=False):
    """CSR windows of lengths 1 .. lmax (plus empty ones) cut from synth streams, with the synth special windows."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, lmax + 1, size=n)
    lens[:4] = [1, 2, lmax, 0]
    S, L = synth.make_windows(n, lmax + 1, seed=seed)
    e = 1 if avg else 0
    wins = [S[i, :lens[i] + e] if lens[i] else S[i, :0] for i in range(n)]
    off = np.zeros(n + 1, dtype=np.int64); off[1:] = np.cumsum([len(w) for w in wins])
    return np.ascontiguousarray(np.concatenate(wins).reshape(-1, 7)), L, off


def _dev(cuda, *a):
    return [None if x is None else cuda.from_numpy(np.ascontiguousarray(x)).cuda() for x in a]


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["uniform", "csr", "uniform_avg", "csr_avg", "special"])
def test_kernel_precision_gate(cuda, layout):
    """Every field and every P block per window within 8 x the fp64 statement's own error against its long-double run (DESIGN.md
    section 5's rule, floor 1e-15)."""
    from cpi_b200 import preint
    flags = FL | (capi.FLAG_IMU_AVG if layout.endswith("avg") else 0)
    avg = 1 if flags & capi.FLAG_IMU_AVG else 0
    if layout.startswith("csr"):
        S, L, off = _csr_batch(160, 21, avg=bool(avg))
        ns = None
    else:
        n = 3000 if layout == "special" else 200
        S, L = synth.make_windows(n, 120, seed=23, imu_avg=bool(avg))
        if layout == "special":
            small, zero, dz = _special(S[:, :120], L)
            keep = np.where(small | zero | dz)[0]
            assert small[keep].any() and zero[keep].any() and dz[keep].any()
            S, L = S[keep], L[keep]
        off, ns = None, 120
        S = S.reshape(-1, 7)
    d_S, d_L, d_off = _dev(cuda, S, L, off)
    got = preint.preintegrate(1, d_S, d_L, SIG, flags, offsets=d_off, ns=ns).cpu().numpy()
    o64 = dr.preintegrate(S, L, SIG, flags, offsets=off, ns=ns)
    ld = dr.preintegrate(S, L, SIG, flags, offsets=off, ns=ns, dtype=np.longdouble)
    ratio, worst, bad = conditioned_gate(got, o64, ld, 1, K=8, floor=1e-15)
    print(layout, "worst ratio", max(w["ratio"] for w in worst.values()), max(worst, key=lambda k: worst[k]["ratio"]))
    assert not bad, bad[:5]


@pytest.mark.gpu
def test_continuation_host_and_repeat_are_bitwise(cuda):
    """Continuing at random split points, the host entry point and a second run all give the one-shot record's bits."""
    from cpi_b200 import preint
    S, L, off = _csr_batch(300, 31)
    d_S, d_L, d_off = _dev(cuda, S, L, off)
    one = preint.preintegrate(1, d_S, d_L, SIG, FL, offsets=d_off).cpu().numpy()
    again = preint.preintegrate(1, d_S, d_L, SIG, FL, offsets=d_off).cpu().numpy()
    assert np.array_equal(one, again)
    assert np.array_equal(preint.preintegrate_host(1, S, L, SIG, FL, offsets=off), one)
    rng = np.random.default_rng(3)
    lens = np.diff(off)
    cut = np.array([rng.integers(0, l + 1) for l in lens])
    off_a = np.zeros_like(off); off_a[1:] = np.cumsum(cut)
    off_b = np.zeros_like(off); off_b[1:] = np.cumsum(lens - cut)
    Sa = np.concatenate([S[off[i]:off[i] + cut[i]] for i in range(len(lens))])
    Sb = np.concatenate([S[off[i] + cut[i]:off[i + 1]] for i in range(len(lens))])
    rec = preint.preintegrate(1, *_dev(cuda, Sa, L), SIG, FL, offsets=_dev(cuda, off_a)[0])
    preint.preintegrate(1, *_dev(cuda, Sb, L), SIG, FL, offsets=_dev(cuda, off_b)[0], continue_records=rec)
    assert np.array_equal(rec.cpu().numpy(), one)
    lib = capi.load()
    r = rec.clone()
    rc = lib.cpi_preintegrate_batch_continue(1, 64, r.shape[0], ctypes.c_void_p(d_off.data_ptr()), 0, ctypes.c_void_p(d_S.data_ptr()),
                                             ctypes.c_void_p(d_L.data_ptr()), P(np.ascontiguousarray(SIG)), FL | capi.FLAG_IMU_AVG,
                                             ctypes.c_void_p(r.data_ptr()), None)
    assert rc == -1 and b"continuation" in lib.cpi_last_error()


@pytest.mark.gpu
def test_same_rotation_as_model_1(cuda):
    """R, q, J_q and DT come out of model 1's own rotation chain: they match K1's records to rounding."""
    from cpi_b200 import preint
    S, L = synth.make_windows(2000, 200, seed=41)
    d_S, d_L = _dev(cuda, S.reshape(-1, 7), L)
    d = preint.preintegrate(1, d_S, d_L, SIG, FL, ns=200).cpu().numpy()
    k1 = preint.preintegrate(1, d_S, d_L, SIG, 0, ns=200).cpu().numpy()
    for f in ("R", "q", "J_q", "DT"):
        a, b = REC[f]
        err = np.abs(d[:, a:b] - k1[:, a:b]).max()
        print(f, err)
        assert err < 1e-12 * max(1.0, np.abs(k1[:, a:b]).max()), (f, err)


@pytest.mark.gpu
def test_relinearize_repreintegrates_discretely(cuda):
    """relinearize_records(flags=FLAG_DISCRETE) writes, for every selected window, the record preintegrate gives at the new lin, bitwise;
    unselected records keep their bits."""
    import torch
    from cpi_b200 import factor, preint
    nf, ns = 64, 50
    S, L = synth.make_windows(nf, ns, seed=51)
    d_S, d_L = _dev(cuda, S.reshape(-1, 7), L)
    rec = preint.preintegrate(1, d_S, d_L, SIG, FL, ns=ns)
    rng = np.random.default_rng(5)
    X = np.zeros((nf + 1, 16)); X[:, 3] = 1.0
    X[:nf, 4:7] = L[:, 0:3]; X[:nf, 10:13] = L[:, 3:6]
    moved = rng.random(nf) < 0.4
    X[:nf][moved, 4:7] += 0.01
    states = torch.from_numpy(X).cuda()
    rec0 = rec.clone()
    n, mask = factor.relinearize_records(1, states, rec, d_L, nf + 1, d_S, SIG, ns=ns, flags=FL, tol_bw=2e-3, tol_ba=2e-2)
    mask = mask.cpu().numpy().astype(bool)
    assert n == moved.sum() and np.array_equal(mask, moved)
    want = preint.preintegrate(1, d_S, d_L, SIG, FL, ns=ns).cpu().numpy()      # d_L now holds the new points
    got = rec.cpu().numpy()
    assert np.array_equal(got[mask], want[mask])
    assert np.array_equal(got[~mask], rec0.cpu().numpy()[~mask])


@pytest.mark.gpu
def test_merge_and_scan_of_discrete_segments(cuda):
    """Euler steps compose exactly: merging / scanning discrete segment records gives the one-shot discrete record's means and
    Jacobians to rounding.  The distance on P is reported."""
    from cpi_b200 import preint
    ng, seg, ns = 50, 4, 40
    S, L = synth.make_windows(ng, seg * ns, seed=61)
    d_one = preint.preintegrate(1, *_dev(cuda, S.reshape(-1, 7), L), SIG, FL, ns=seg * ns).cpu().numpy()
    Sseg = S.reshape(ng * seg, ns, 7)
    Lseg = np.repeat(L, seg, axis=0)
    d_S, d_L = _dev(cuda, Sseg.reshape(-1, 7), Lseg)
    segs = preint.preintegrate(1, d_S, d_L, SIG, FL, ns=ns)
    merged = preint.merge(1, segs, d_L, group=seg).cpu().numpy()
    scanned = preint.scan(1, segs, d_L, group=seg).cpu().numpy()[seg - 1::seg]
    for name, r in (("merge", merged), ("scan", scanned)):
        for f in ("R", "alpha", "beta", "J_q", "J_a", "J_b", "H_a", "H_b", "DT"):
            a, b = REC[f]
            e = np.abs(r[:, a:b] - d_one[:, a:b]).max() / max(np.abs(d_one[:, a:b]).max(), 1e-300)
            assert e < 1e-12, (name, f, e)
        eP = np.linalg.norm(r[:, 65:] - d_one[:, 65:], axis=1) / np.linalg.norm(d_one[:, 65:], axis=1)
        print(name, "P relative distance to the one-shot record: max", eP.max())


# ------------------------------------------------------------------------------------------------------------------
# GPU: the smoother on discrete records (the shape of test_chain_marginals._smoother_monte_carlo, with the truth's propagator
# and the records' propagator chosen separately)
# ------------------------------------------------------------------------------------------------------------------

def _monte_carlo(torch, oracle, truth_flags, rec_flags, N, K, seed, noise=None, rate=200.0, fixes=(3, 6, 9), sigma_fix=0.01):
    """N realisations of one truth trajectory as chains of K keyframes (20-sample windows at `rate`).  The truth is the noise-free
    propagation of the bias-free readings with the propagator of `truth_flags` (0: model 1, FLAG_DISCRETE: the discrete recursion);
    each realisation has its own white noise and bias walk, x_hat_0 drawn from the prior and a position fix on the keyframes `fixes`.
    For every entry of rec_flags the same realisations are preintegrated with those flags, chains_lm runs to convergence and
    chains_marginals at the result.  Returns {flags: (errors [N, K, 15] in retract coordinates at the estimate, Sigma_kk, status)}."""
    from cpi_b200 import factor, preint
    from test_marginalize import local, mat, vec
    from test_propagate import random_cov
    from test_state_priors import _fix
    rng = np.random.default_rng(seed)
    nz = None if noise is None else np.random.default_rng([seed, noise])

    def draw(size, scale=1.0):
        x = rng.normal(0.0, scale, size)
        return x if nz is None else nz.normal(0.0, scale, size)
    ns = 20
    Sw, Lw = synth.make_windows(K - 1, ns, rate=rate, first_window=81000, special=False)
    Lw[:] = Lw[0]
    dt = Sw[:, :, 6]
    w_true, a_true = Sw[:, :, 0:3] - Lw[0, 0:3], Sw[:, :, 3:6] - Lw[0, 3:6]
    x_true = np.zeros((K, 16))
    q = rng.normal(size=4); q /= np.linalg.norm(q); q *= np.sign(q[3])
    x_true[0, 0:4], x_true[0, 4:7], x_true[0, 7:10], x_true[0, 10:13], x_true[0, 13:16] = q, Lw[0, 0:3], [1.0, -0.5, 0.2], Lw[0, 3:6], [3.0, 1.0, -2.0]
    for k in range(K - 1):
        lin_t = np.concatenate([x_true[k, 4:7], x_true[k, 10:13], x_true[k, 0:4], synth.GRAVITY])[None]
        clean = np.concatenate([w_true[k] + x_true[k, 4:7], a_true[k] + x_true[k, 10:13], dt[k][:, None]], axis=1)[None]
        x_true[k + 1] = oracle.predict_state(1, x_true[k:k + 1], preint.preintegrate_host(1, clean, lin_t, SIG, truth_flags, ns=ns), lin_t)[0]
    sw, swb, sa, sab = SIG
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
    Sig0 = mat(random_cov(rng, 1)[0])[0]
    delta = draw((N, 15)) @ np.linalg.cholesky(Sig0).T
    xh0 = oracle.retract(truth[:, 0], -delta)
    lin = np.zeros((N, K - 1, 13))
    lin[:, :, 0:3], lin[:, :, 3:6], lin[:, :, 10:13] = xh0[:, None, 4:7], xh0[:, None, 10:13], synth.GRAVITY
    lin[:, :, 9] = 1.0
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dl, dS = d(lin.reshape(-1, 13)), d(samples.reshape(N * (K - 1), ns, 7))
    Lam0 = np.linalg.inv(Sig0); Lam0 = 0.5 * (Lam0 + Lam0.T)
    prior = (d(np.repeat(vec(Lam0[None]), N, axis=0)), d(np.zeros((N, 15))), d(np.zeros(N)), d(xh0))
    idx, W, xb = [], [], []
    for k in fixes:
        w, _ = _fix(rng, truth[0, k], sigma_fix)
        fix = truth[:, k].copy(); fix[:, 13:16] += draw((N, 3), sigma_fix)
        idx.append(np.arange(N) * K + k); W.append(np.repeat(vec(w[None]), N, axis=0)); xb.append(fix)
    sp = (d(np.concatenate(idx).astype(np.int64)), d(np.concatenate(W)), None, None, d(np.concatenate(xb)))
    params = capi.LMParams(absolute_error_tol=0.0, relative_error_tol=1e-13, max_iterations=50)
    out = {}
    for fl in rec_flags:
        rec = preint.preintegrate(1, dS, dl, SIG, fl, ns=ns)
        X0 = torch.empty((N, K, 16), dtype=torch.float64, device="cuda")
        X0[:, 0] = d(xh0)
        recK, linK = rec.view(N, K - 1, -1), dl.view(N, K - 1, 13)
        for k in range(K - 1):
            X0[:, k + 1] = factor.predict_state(1, X0[:, k].contiguous(), recK[:, k].contiguous(), linK[:, k].contiguous())
        X0 = X0.reshape(N * K, 16)
        Xs, _, _, status, _, _ = factor.chains_lm(1, X0, rec, dl, K, prior=prior, state_priors=sp, params=params, max_rounds=100)
        cov, _ = factor.chains_marginals(1, Xs, rec, dl, K, prior=prior, state_priors=sp)
        err = local(Xs.cpu().numpy(), truth.reshape(N * K, 16)).reshape(N, K, 15)
        out[fl] = (err, mat(cov.cpu().numpy()).reshape(N, K, 15, 15), status.cpu().numpy())
    return out


def _nees(err, cov):
    """[N, K] NEES e^T Sigma_kk^-1 e per realisation and keyframe."""
    return np.einsum("nki,nki->nk", err, np.linalg.solve(cov, err[..., None])[..., 0])


@pytest.mark.gpu
def test_monte_carlo_consistency_on_discrete_truth(cuda, oracle):
    """P_meas is right for its own model: with the truth generated by the discrete recursion, chains_lm + chains_marginals on discrete
    records keep the mean NEES at every keyframe inside the two-sided 99.9 % chi^2_15 band, pooled over 30 000 realisations (three
    batches of 10 000: the seed's own noise stream and two independent ones) of chains of 10 keyframes with 1 cm position fixes on
    keyframes 3, 6 and 9.  This is the check that reaches the dt^2 terms of Phi and Q, which step splitting cannot pin."""
    from scipy.stats import chi2
    n, K, streams = 10_000, 10, (None, 1, 2)
    nees_sum = np.zeros(K)
    for s in streams:
        err, cov, status = _monte_carlo(cuda, oracle, FL, (FL,), n, K, 95, noise=s)[FL]
        assert np.all(status != capi.LM_NONFINITE) and np.all(status != capi.LM_RUNNING)
        nees_sum += _nees(err, cov).sum(axis=0)
    N = n * len(streams)
    lo, hi = chi2.ppf([0.0005, 0.9995], 15 * N) / N
    mean = nees_sum / N
    print("discrete truth, discrete records: mean NEES per keyframe", np.round(mean, 3).tolist(), f"band [{lo:.3f}, {hi:.3f}]")
    assert np.all((lo <= mean) & (mean <= hi)), (mean, lo, hi)


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [200.0, 50.0])
def test_model_1_against_discrete_records(cuda, oracle, rate):
    """The reference's comparison: the truth that is exact for model 1, the same 10 000 noisy realisations, model-1 records against
    discrete records.  Reports the mean NEES per keyframe (with its standard error) and the RMS attitude, velocity and position
    errors of both (DESIGN.md section 3n).  The one gate is on the gap, which is many standard errors wide at both rates: the
    discrete records' mean NEES exceeds model 1's at every keyframe by more than 10 standard errors of the paired difference
    (measured on an H100: 20 to 33 at 200 Hz, 69 to 209 at 50 Hz)."""
    from scipy.stats import chi2
    n, K = 10_000, 10
    res = _monte_carlo(cuda, oracle, 0, (0, FL), n, K, 96, rate=rate)
    lo, hi = chi2.ppf([0.0005, 0.9995], 15 * n) / n
    diff = _nees(*res[FL][:2]) - _nees(*res[0][:2])
    z = diff.mean(axis=0) / (diff.std(axis=0) / np.sqrt(n))
    print(f"{rate:g} Hz: discrete minus model-1 mean NEES per keyframe, in standard errors of the paired difference", np.round(z, 1).tolist())
    assert np.all(z > 10.0), z
    for fl, name in ((0, "model 1"), (FL, "discrete")):
        err, cov, status = res[fl]
        assert np.all(status != capi.LM_NONFINITE) and np.all(status != capi.LM_RUNNING)
        nees = _nees(err, cov)
        rms = lambda sl: np.sqrt(np.mean(np.sum(err[:, :, sl] ** 2, axis=2)))
        print(f"{rate:g} Hz, {name} records: mean NEES per keyframe {np.round(nees.mean(axis=0), 3).tolist()} "
              f"(s.e. {np.round(nees.std(axis=0) / np.sqrt(n), 3).tolist()}), band [{lo:.3f}, {hi:.3f}]; RMS attitude "
              f"{rms(slice(0, 3)):.3e} rad, velocity {rms(slice(6, 9)):.3e} m/s, position {rms(slice(12, 15)):.3e} m")
