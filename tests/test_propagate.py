"""Prediction with covariance (cpi_propagate_batch / _host, factor.propagate / propagate_host).

The truth is ``propagate_ref`` below, a numpy statement of the formula built from the oracle's ``predict_state`` and ``factor_eval``:
A = -H2^-1 H1, B = H2^-1, cov_k1 = A cov_k A^T + B P_meas B^T, cross = cov_k A^T.  On the CPU it is pinned against a central finite
difference of the implicit map x_k -> x_k1 defined by the factor's residual e(x_k, x_k1) = 0.  The GPU tests compare the kernel
with it, check known answers, composition with the merge and the scan, and what P_meas claims to be: the covariance of the
preintegration error under the reference simulator's noise model (a Monte Carlo NEES test)."""
import ctypes

import numpy as np
import pytest

from cpi_b200 import capi, synth

RD = {1: 290, 2: 308}
P = lambda a: ctypes.c_void_p(a.ctypes.data)
BLK = [slice(3 * k, 3 * k + 3) for k in range(5)]


def mat(a):
    """[n, 225] column-major -> [n, 15, 15]"""
    return np.asarray(a).reshape(-1, 15, 15).transpose(0, 2, 1)


def propagate_ref(orc, model, X, Sig, rec, lin):
    """numpy statement: (x_k1, A, B, cov_k1, cross), every matrix [n, 15, 15]."""
    n = len(X)
    Xh = orc.predict_state(model, X, rec, lin)
    st = np.empty((2 * n, 16)); st[0::2] = X; st[1::2] = Xh
    _, H1, H2 = orc.factor_eval(model, st, rec, lin, np.arange(0, 2 * n, 2), np.arange(1, 2 * n, 2))
    H1, H2 = mat(H1), mat(H2)
    B = np.zeros((n, 15, 15))
    B[:, 0:3, 0:3] = np.linalg.inv(H2[:, 0:3, 0:3])
    B[:, 3:6, 3:6] = B[:, 9:12, 9:12] = np.eye(3)
    B[:, 6:9, 6:9] = H2[:, 6:9, 6:9].transpose(0, 2, 1)           # Rk^-1 = Rk^T
    B[:, 12:15, 12:15] = H2[:, 12:15, 12:15].transpose(0, 2, 1)
    A = -B @ H1
    S = mat(Sig)
    Pm = mat(rec[:, 65:290])
    At = A.transpose(0, 2, 1)
    return Xh, A, B, A @ S @ At + B @ Pm @ B.transpose(0, 2, 1), S @ At


def block_errors(got, ref, rows_scale, cols_scale):
    """Worst 3x3-block error of [n,15,15] arrays, each block relative to sqrt(|rows_scale_II| |cols_scale_JJ|) (Frobenius norms of the
    diagonal blocks: the natural scale of a covariance block, finite for structurally zero ones).  Returns (worst, (I, J))."""
    worst, at = 0.0, None
    for I in range(5):
        for J in range(5):
            num = np.linalg.norm(got[:, BLK[I], BLK[J]] - ref[:, BLK[I], BLK[J]], axis=(1, 2))
            den = np.sqrt(np.linalg.norm(rows_scale[:, BLK[I], BLK[I]], axis=(1, 2)) * np.linalg.norm(cols_scale[:, BLK[J], BLK[J]], axis=(1, 2)))
            e = float(np.max(num / np.maximum(den, 1e-300)))
            if e > worst:
                worst, at = e, (I, J)
    return worst, at


def random_cov(rng, n, scale=(2e-3, 2e-4, 2e-2, 2e-3, 5e-2)):
    """n random SPD 15x15 covariances, exactly symmetric, column-major [n, 225]; standard deviations about `scale` per block."""
    D = np.repeat(np.asarray(scale), 3)
    G = rng.normal(size=(n, 15, 15))
    C = G @ G.transpose(0, 2, 1) / 15 + 0.5 * np.eye(15)
    C = D[None, :, None] * C * D[None, None, :]
    C = 0.5 * (C + C.transpose(0, 2, 1))
    return np.ascontiguousarray(C.transpose(0, 2, 1).reshape(n, 225))


def qmul(q, p):
    """cpi_common.cuh quat_multiply (JPL), batched [n, 4]."""
    t = np.stack([q[:, 3] * p[:, 0] + q[:, 2] * p[:, 1] - q[:, 1] * p[:, 2] + q[:, 0] * p[:, 3],
                  -q[:, 2] * p[:, 0] + q[:, 3] * p[:, 1] + q[:, 0] * p[:, 2] + q[:, 1] * p[:, 3],
                  q[:, 1] * p[:, 0] - q[:, 0] * p[:, 1] + q[:, 3] * p[:, 2] + q[:, 2] * p[:, 3],
                  -q[:, 0] * p[:, 0] - q[:, 1] * p[:, 1] - q[:, 2] * p[:, 2] + q[:, 3] * p[:, 3]], axis=1)
    t[t[:, 3] < 0] *= -1
    return t / np.linalg.norm(t, axis=1, keepdims=True)


def local(base, x):
    """Retract coordinates of x at base: x = JPLNavState::retract(base, d), batched [n, 16] -> [n, 15]."""
    qi = base[:, 0:4] * np.array([-1, -1, -1, 1.0])
    dq = qmul(x[:, 0:4], qi)
    s = np.linalg.norm(dq[:, 0:3], axis=1)
    f = np.where(s > 0, 2 * np.arctan2(s, dq[:, 3]) / np.maximum(s, 1e-300), 2.0)
    return np.concatenate([f[:, None] * dq[:, 0:3], x[:, 4:16] - base[:, 4:16]], axis=1)


def anchors_at_lin(rec, L, model):
    """Anchor states of a chain through the records, with biases at the linearisation point (and q_K = q_lin in model 2), so that
    the factor's residual vanishes at the prediction."""
    X = synth.make_states(rec, L, model)[:len(rec)]
    X[:, 4:7], X[:, 10:13] = L[:, 0:3], L[:, 3:6]
    if model == 2:
        X[:, 0:4] = L[:, 6:10]
    return X


# ------------------------------------------------------------------------------------------------------------------
# CPU: argument checks of the C ABI, and the numpy statement against the implicit map
# ------------------------------------------------------------------------------------------------------------------

def test_propagate_argument_validation_without_gpu():
    lib = capi.load()
    x, c, r, l = np.zeros(2 * 16), np.zeros(2 * 225), np.zeros(2 * 308), np.zeros(2 * 13)
    x1, c1, cr = np.zeros(2 * 16), np.zeros(2 * 225), np.zeros(2 * 225)
    calls = (lambda m, n, *a, na=2: lib.cpi_propagate_batch(m, n, *a, None),
             lambda m, n, xs, cs, an, *a, na=2: lib.cpi_propagate_batch_host(m, n, na, xs, cs, an, *a))
    args = [P(x), P(c), None, P(r), P(l), P(x1), P(c1), P(cr)]
    for fn in calls:
        for model in (0, 3):
            assert fn(model, 2, *args) == -1 and b"model" in lib.cpi_last_error()
        assert fn(1, -1, *args) == -1 and b"negative" in lib.cpi_last_error()
        for k in (0, 1, 3, 4, 5, 6):                                 # states_k, cov_k, records, lin, states_k1, cov_k1
            bad = list(args); bad[k] = None
            assert fn(1, 2, *bad) == -1 and b"null" in lib.cpi_last_error(), k
        for k, o in ((5, P(x)), (6, P(c)), (7, P(r)), (7, P(x1))):  # an output aliasing an input or another output
            bad = list(args); bad[k] = o
            assert fn(2, 2, *bad) == -1 and b"overlap" in lib.cpi_last_error(), k
        assert fn(1, 0, *[None] * 8) == 0
    host = calls[1]
    assert host(1, 2, *args, na=-1) == -1 and b"negative" in lib.cpi_last_error()
    assert host(1, 2, *args, na=1) == -1 and b"n_anchors" in lib.cpi_last_error()
    for bad in ([0, 2], [-1, 0], [1, 1 << 40]):
        an = np.array(bad, dtype=np.int64)
        a2 = list(args); a2[2] = P(an)
        assert host(1, 2, *a2) == -1 and b"out of range" in lib.cpi_last_error(), bad
    # Python layer
    from cpi_b200 import factor
    with pytest.raises(ValueError):
        factor.propagate_host(1, x.reshape(2, 16), c.reshape(2, 225), r[:290].reshape(1, 290), l.reshape(2, 13))
    with pytest.raises(ValueError):
        factor.propagate_host(1, x.reshape(2, 16), c.reshape(2, 225), r[:580].reshape(2, 290), l.reshape(2, 13), anchor=[0])
    with pytest.raises(capi.CpiError, match="out of range"):
        factor.propagate_host(1, x.reshape(2, 16), c.reshape(2, 225), r[:580].reshape(2, 290), l.reshape(2, 13), anchor=[0, 2])


def implicit_state(orc, model, xk, rec, lin, x0, iters=8):
    """x_k1 with e(x_k, x_k1) = 0: Newton on the oracle's residual, stepping through retract."""
    x = x0.copy()
    for _ in range(iters):
        e, _, H2 = orc.factor_eval(model, np.stack([xk, x]), rec[None], lin[None])
        x = orc.retract(x[None], -np.linalg.solve(mat(H2)[0], e[0])[None])[0]
    return x


@pytest.mark.parametrize("model", [1, 2])
def test_formula_matches_the_implicit_map(oracle, model):
    """A = -H2^-1 H1 of the numpy statement equals a central finite difference of x_k -> x_k1 (Newton on e(x_k, x_k1) = 0, x_k
    perturbed through retract by +-h = 1e-5 per tangent coordinate) to 1e-6 per 3x3 block, relative to max(|A_IJ|, 1); and A, B
    have the structure of DESIGN.md section 3d: zero blocks exactly zero, the bias rows exactly [0 I 0 0 0] / [0 0 0 I 0], B block
    diagonal, and the v / p identity and DT I blocks equal to them to the orthogonality of R(q_k) (<= 1e-14)."""
    n, h = 4, 1e-5
    S, L = synth.make_windows(n, 200, rate=200.0, first_window=66000, special=False)
    rec = oracle.preintegrate(model, S, L, synth.SIGMAS, 0, ns=200)
    X = anchors_at_lin(rec, L, model)
    Xh, A, B, _, _ = propagate_ref(oracle, model, X, random_cov(np.random.default_rng(1), n), rec, L)
    worst = 0.0
    for w in range(n):
        x1 = implicit_state(oracle, model, X[w], rec[w], L[w], Xh[w])
        assert np.max(np.abs(local(Xh[w:w + 1], x1[None]))) < 1e-12          # the prediction solves e = 0
        Afd = np.zeros((15, 15))
        for c in range(15):
            d = np.zeros(15); d[c] = h
            xp = implicit_state(oracle, model, oracle.retract(X[w:w + 1], d[None])[0], rec[w], L[w], x1)
            xm = implicit_state(oracle, model, oracle.retract(X[w:w + 1], -d[None])[0], rec[w], L[w], x1)
            Afd[:, c] = (local(x1[None], xp[None])[0] - local(x1[None], xm[None])[0]) / (2 * h)
        for I in range(5):
            for J in range(5):
                blk = A[w, BLK[I], BLK[J]]
                worst = max(worst, np.linalg.norm(Afd[BLK[I], BLK[J]] - blk) / max(np.linalg.norm(blk), 1.0))
    print(f"model {model}: worst block of A against the finite difference {worst:.1e}")
    assert worst <= 1e-6
    I3, Z3 = np.eye(3), np.zeros((3, 3))
    for w in range(n):
        a = lambda I, J: A[w, BLK[I], BLK[J]]
        for I, J in ((0, 2), (0, 3), (0, 4), (2, 4)):
            assert np.all(a(I, J) == 0), (I, J)
        for I, want in ((1, 1), (3, 3)):
            for J in range(5):
                assert np.array_equal(a(I, J), I3 if J == want else Z3), (I, J)
        dt = rec[w, 19]
        for I, J, want in ((2, 2, I3), (4, 4, I3), (4, 2, dt * I3)):
            assert np.max(np.abs(a(I, J) - want)) <= 1e-14, (I, J)
        for I in range(5):
            for J in range(5):
                if I != J:
                    assert np.all(B[w, BLK[I], BLK[J]] == 0)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------

def _inputs(model, which, orc):
    """(X, Sig, rec, L): stress-batch windows (tests/stress.py) or configs-style windows (synth, 200 samples at 200 Hz), with anchor
    states off the linearisation point (make_states perturbs them) and random anchor covariances."""
    import stress
    from cpi_b200 import preint
    if which == "stress":
        S, off, L, _ = stress.make_batch(n_long=0)
        rec = preint.preintegrate_host(model, S, L, synth.SIGMAS, 0, offsets=off)
    else:
        S, L = synth.make_windows(2000, 200, rate=200.0, first_window=67000)
        rec = preint.preintegrate_host(model, S, L, synth.SIGMAS, 0, ns=200)
    X = synth.make_states(rec, L, model)[:len(rec)]
    return X, random_cov(np.random.default_rng(2), len(rec)), rec, L


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_kernel_matches_numpy_statement(cuda, oracle, model):
    """Stress-batch and configs-style windows: cov_k1 and cross against the numpy statement per 3x3 block (<= 1e-12, relative to the
    diagonal blocks' scale), cov_k1 exactly symmetric, states_k1 bit for bit cpi_predict_state_batch."""
    from cpi_b200 import factor
    torch = cuda
    for which in ("stress", "configs"):
        X, Sig, rec, L = _inputs(model, which, oracle)
        d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        x1, c1, cr = factor.propagate(model, d(X), d(Sig), d(rec), d(L), want_cross=True)
        pred = factor.predict_state(model, d(X), d(rec), d(L))
        torch.cuda.synchronize()
        x1, c1, cr, pred = (t.cpu().numpy() for t in (x1, c1, cr, pred))
        assert np.array_equal(x1, pred), "states_k1 differs from cpi_predict_state_batch"
        C1, CR = mat(c1), mat(cr)
        assert np.array_equal(C1, C1.transpose(0, 2, 1)), "cov_k1 not exactly symmetric"
        Xh, A, B, S1, C = propagate_ref(oracle, model, X, Sig, rec, L)
        e1, at1 = block_errors(C1, S1, S1, S1)
        e2, at2 = block_errors(CR, C, mat(Sig), S1)
        print(f"model {model} {which} ({len(X)} windows): cov_k1 worst block {e1:.1e} at {at1}, cross {e2:.1e} at {at2}, "
              f"states vs oracle {np.max(np.abs(x1 - Xh) / np.maximum(1, np.abs(Xh))):.1e}")
        assert e1 <= 1e-12 and e2 <= 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_known_answers(cuda, oracle, model):
    """cov_k = 0 gives B P B^T (and a zero cross-covariance); the zero-step record leaves cov_k unchanged to rounding; host and device
    paths are bitwise equal on a multi-wave batch (60 000 windows) with a ragged anchor array."""
    from cpi_b200 import factor, preint
    torch = cuda
    S, L = synth.make_windows(512, 30, rate=200.0, first_window=68000)
    rec = preint.preintegrate_host(model, S, L, synth.SIGMAS, 0, ns=30)
    X = synth.make_states(rec, L, model)[:512]
    _, _, B, _, _ = propagate_ref(oracle, model, X, np.zeros((512, 225)), rec, L)
    BPB = B @ mat(rec[:, 65:290]) @ B.transpose(0, 2, 1)
    _, c1, cr = factor.propagate_host(model, X, np.zeros((512, 225)), rec, L, want_cross=True)
    e, at = block_errors(mat(c1), BPB, BPB, BPB)
    print(f"model {model}: cov_k = 0 against B P B^T {e:.1e} at {at}")
    assert e <= 1e-12 and np.all(cr == 0)

    zero = np.zeros((512, RD[model])); zero[:, 3] = 1.0; zero[:, 4:13] = np.eye(3).reshape(-1)
    Sig = random_cov(np.random.default_rng(3), 512)
    x1, c1, _ = factor.propagate_host(model, X, Sig, zero, L)
    e, at = block_errors(mat(c1), mat(Sig), mat(Sig), mat(Sig))
    print(f"model {model}: zero-step record {e:.1e} at {at}")
    assert e <= 1e-14

    rng = np.random.default_rng(4)
    n, m = 60_000, 700
    idx = rng.integers(0, 512, size=n)
    anchor = rng.integers(0, m, size=n)
    Xa, Sa = np.repeat(X, 2, axis=0)[:m], random_cov(rng, m)
    h = factor.propagate_host(model, Xa, Sa, rec[idx], L[idx], anchor=anchor, want_cross=True)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    g = factor.propagate(model, d(Xa), d(Sa), d(rec[idx]), d(L[idx]), anchor=d(anchor), want_cross=True)
    torch.cuda.synchronize()
    for a, b in zip(h, g):
        assert np.array_equal(a, b.cpu().numpy())
    ref = propagate_ref(oracle, model, Xa[anchor[:2000]], Sa[anchor[:2000]], rec[idx[:2000]], L[idx[:2000]])
    assert block_errors(mat(h[1][:2000]), ref[3], ref[3], ref[3])[0] <= 1e-12


@pytest.mark.gpu
def test_composition_with_merge_and_scan(cuda, oracle):
    """Model 1.  Propagating k -> m, then m -> j from the prediction, agrees with one propagation through the cpi_merge_records
    record of k -> j (<= 1e-10 per block, the merge's P tolerance).  A 300-keyframe chain: cpi_scan_records then ONE propagate call
    with anchor = 0 agrees with 300 sequential propagate calls; the gate is 10x what the same two routes differ by in numpy (the
    oracle's statement step by step against the numpy prefix fold of test_scan.py)."""
    from cpi_b200 import factor, preint
    from test_scan import prefix_folds
    torch = cuda
    # k -> m -> j: two halves of 200-sample windows, one linearisation point each
    n = 256
    S, L = synth.make_windows(n, 200, rate=200.0, first_window=69000, special=False)
    off = np.arange(2 * n + 1, dtype=np.int64) * 100
    L2 = np.repeat(L, 2, axis=0)
    halves = preint.preintegrate_host(1, S.reshape(-1, 7), L2, synth.SIGMAS, 0, offsets=off)
    merged = preint.merge_host(1, halves, L2, group=2)
    X = anchors_at_lin(merged, L, 1)
    Sig = random_cov(np.random.default_rng(5), n)
    xm, cm, _ = factor.propagate_host(1, X, Sig, halves[0::2], L)
    xj, cj, _ = factor.propagate_host(1, xm, cm, halves[1::2], L)
    xJ, cJ, _ = factor.propagate_host(1, X, Sig, merged, L)
    e, at = block_errors(mat(cj), mat(cJ), mat(cJ), mat(cJ))
    print(f"k -> m -> j against the merged record: worst block {e:.1e} at {at}, states {np.max(np.abs(xj - xJ) / np.maximum(1, np.abs(xJ))):.1e}")
    assert e <= 1e-10

    # the chain: one linearisation point per chain, anchors at it
    k, chains = 300, 2
    S, L = synth.make_windows(chains * k, 20, rate=200.0, first_window=65000, special=False)
    L = np.repeat(L[::k], k, axis=0)
    rec = preint.preintegrate_host(1, S, L, synth.SIGMAS, 0, ns=20)
    out = preint.scan_host(1, rec, L, group=k)
    X0 = anchors_at_lin(rec[::k], L[::k], 1)
    S0 = random_cov(np.random.default_rng(6), chains)
    seq_x, seq_c = X0, S0
    seq, num_seq = [], []
    nx, nc = X0, S0
    for j in range(k):
        seq_x, seq_c, _ = factor.propagate_host(1, seq_x, seq_c, rec[j::k], L[j::k])
        seq.append(seq_c)
        nx, _, _, ncm, _ = propagate_ref(oracle, 1, nx, nc, rec[j::k], L[j::k])
        nc = ncm.transpose(0, 2, 1).reshape(chains, 225)
        num_seq.append(ncm)
    seq = mat(np.stack(seq, axis=1).reshape(-1, 225))                  # [chain * k + j]
    num_seq = np.stack(num_seq, axis=1).reshape(-1, 15, 15)
    anchor = np.repeat(np.arange(chains), k)
    _, one, _ = factor.propagate_host(1, X0, S0, out, L, anchor=anchor)
    fold = np.concatenate([np.stack([r for _, r in sorted(prefix_folds(rec[c * k:(c + 1) * k], L[c * k:(c + 1) * k]).items())])
                           for c in range(chains)])
    num_one = propagate_ref(oracle, 1, X0[anchor], S0[anchor], fold, L)[3]
    cal, cat = block_errors(num_one, num_seq, num_seq, num_seq)
    e, at = block_errors(mat(one), seq, seq, seq)
    print(f"chain of {k}: scan + one propagate against {k} sequential calls: worst block {e:.1e} at {at}; "
          f"numpy routes differ by {cal:.1e} at {cat}")
    assert e <= max(10 * cal, 1e-12)


def _monte_carlo(torch, oracle, model, S, L, N, seed):
    """N realisations of one window under the reference simulator's noise model (synth.py: w_m = w + b + sigma/sqrt(dt) n,
    b += sigma_b sqrt(dt) n, likewise for a), an anchor drawn from cov_k, every realisation preintegrated at its anchor's biases
    (and, model 2, orientation) and propagated.  The truth is the noise-free discrete propagation from the true anchor: the window's
    readings minus its bias, preintegrated exactly, with the realisation's own bias walk for the biases at k+1.
    Returns (errors [N, 15] in retract coordinates at the prediction, cov_k1 [N, 15, 15])."""
    from cpi_b200 import factor, preint
    rng = np.random.default_rng(seed)
    ns, dt = S.shape[0], S[:, 6]
    w_true, a_true = S[:, 0:3] - L[0:3], S[:, 3:6] - L[3:6]
    x_true = np.zeros(16)
    q = rng.normal(size=4); q /= np.linalg.norm(q); q *= np.sign(q[3])
    x_true[0:4], x_true[4:7], x_true[7:10], x_true[10:13], x_true[13:16] = q, L[0:3], [1.0, -0.5, 0.2], L[3:6], [3.0, 1.0, -2.0]
    Sig = random_cov(rng, 1)[0]
    delta = rng.normal(size=(N, 15)) @ np.linalg.cholesky(mat(Sig)[0]).T
    xh = oracle.retract(np.repeat(x_true[None], N, axis=0), -delta)       # x_true = retract(x_hat, delta) exactly
    sw, swb, sa, sab = synth.SIGMAS
    sq = np.sqrt(dt)[None, :, None]
    bw = x_true[4:7] + np.concatenate([np.zeros((N, 1, 3)), np.cumsum(swb * sq * rng.normal(size=(N, ns, 3)), axis=1)], axis=1)
    ba = x_true[10:13] + np.concatenate([np.zeros((N, 1, 3)), np.cumsum(sab * sq * rng.normal(size=(N, ns, 3)), axis=1)], axis=1)
    samples = np.empty((N, ns, 7))
    samples[:, :, 0:3] = w_true + bw[:, :ns] + sw / sq * rng.normal(size=(N, ns, 3))
    samples[:, :, 3:6] = a_true + ba[:, :ns] + sa / sq * rng.normal(size=(N, ns, 3))
    samples[:, :, 6] = dt
    lin = np.empty((N, 13))
    lin[:, 0:3], lin[:, 3:6], lin[:, 6:10], lin[:, 10:13] = xh[:, 4:7], xh[:, 10:13], xh[:, 0:4], synth.GRAVITY
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dl = d(lin)
    rec = preint.preintegrate(model, d(samples), dl, synth.SIGMAS, 0, ns=ns)
    x1, c1, _ = factor.propagate(model, d(xh), d(np.repeat(Sig[None], N, axis=0)), rec, dl)
    # truth: the bias-free readings at the true anchor's linearisation point
    lin_t = np.concatenate([x_true[4:7], x_true[10:13], x_true[0:4], synth.GRAVITY])[None]
    clean = np.concatenate([w_true + x_true[4:7], a_true + x_true[10:13], dt[:, None]], axis=1)[None]
    rec_t = preint.preintegrate_host(model, clean, lin_t, synth.SIGMAS, 0, ns=ns)
    truth = np.repeat(oracle.predict_state(model, x_true[None], rec_t, lin_t), N, axis=0)
    truth[:, 4:7], truth[:, 10:13] = bw[:, ns], ba[:, ns]
    torch.cuda.synchronize()
    x1, c1 = x1.cpu().numpy(), mat(c1.cpu().numpy())
    return local(x1, truth), c1


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_monte_carlo_consistency(cuda, oracle, model):
    """N = 20 000 realisations of a 200-sample 200 Hz window and of a 1 s window at 400 Hz: the mean NEES e^T cov_k1^-1 e of the
    retract-coordinate error lies in the two-sided 99.9 % chi^2_15 band for N, and every entry of the second moment of e lies within
    5 standard errors of the mean cov_k1 (standard error of entry ij: sqrt((S_ii S_jj + S_ij^2) / N))."""
    from scipy.stats import chi2
    N = 20_000
    S1, L1 = synth.make_windows(1, 200, rate=200.0, first_window=71000, special=False)
    S2, L2 = synth.make_windows(1, 400, rate=400.0, first_window=72000, special=False)
    S2[0, :, 6] = 1.0 / 400.0
    lo, hi = chi2.ppf([0.0005, 0.9995], 15 * N) / N
    for name, S, L, seed in (("200 samples at 200 Hz", S1[0], L1[0], 7), ("1 s at 400 Hz", S2[0], L2[0], 8)):
        e, C = _monte_carlo(cuda, oracle, model, S, L, N, seed + 10 * model)
        nees = np.einsum("ni,ni->n", e, np.linalg.solve(C, e[:, :, None])[:, :, 0])
        M = e.T @ e / N
        Cm = C.mean(axis=0)
        se = np.sqrt((np.outer(np.diag(Cm), np.diag(Cm)) + Cm ** 2) / N)
        z = (M - Cm) / se
        zb = [[float(np.max(np.abs(z[BLK[I], BLK[J]]))) for J in range(5)] for I in range(5)]
        print(f"model {model}, {name}: mean NEES {nees.mean():.3f} (band [{lo:.3f}, {hi:.3f}]), worst |z| per block row "
              + " ".join(f"{max(r):.1f}" for r in zb))
        assert lo <= nees.mean() <= hi, nees.mean()
        assert np.max(np.abs(z)) <= 5.0
