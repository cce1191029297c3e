"""The chain-side kernels at the sizes where their launches leave the first grid-stride pass or fold several CTA totals per scan
thread (tests/chain_scale.py, DESIGN.md section 5): the state-prior fold over >= 3 passes, the isolated solve beyond the first pass
of k_chain_ids, chains_lm, chains_lm_step and K8 on about 300 000 states of tiled chain copies, re-preintegration with more than
two passes of the gather and scatter and every per-CTA selection pattern; and two
documented claims at their edges, ties of the selection rule at the tolerance (section 3i) and the robust losses at s = k^2,
subnormal, huge and non-finite s (section 3h)."""
import fractions

import numpy as np
import pytest

from chain_scale import (LM_LENGTHS, SMS, TILE, bcr_modulus, bcr_pattern, chain_ids_pass, check_fold, check_lm_batch, check_relin,
                         contracted, fold_batch, fold_pass, lm_batch, np_norm2, relin_copy_pass, relin_plan, solve_layout, tie_cases)
from cpi_b200 import capi, synth
from test_relinearize import TOL, new_lin, np_select, sq_norms, windows
from test_chains_lm import make_problem, well_posed
from test_marginalize import local
from test_robust_priors import CAUCHY_K, HUBER_K, _moved, add_outliers, mixed_losses, np_loss, np_lm_rb, per_chain_rb
from test_state_priors import _chain_idx, _dev, _host, _meas_priors, _sp_dev, csr, fold_ref, random_layout

DBL_MAX = np.finfo(np.float64).max


# ------------------------------------------------------------------------------------------------------------------
# numpy statements
# ------------------------------------------------------------------------------------------------------------------

def fold_ref_vec(offs, sp_off, info, rhs, f, blocks, chain_prior, f_only=False):
    """fold_ref of test_state_priors.py vectorised over the states: round r adds the r-th prior of every target at once, so each
    target still receives its priors one after the other in CSR order (the f of a chain's last factor: the left state's first)."""
    G11, G22, g1, g2, fk = (np.array(a, dtype=np.float64) for a in blocks)
    pi, pr, pf = (np.array(a, dtype=np.float64) for a in chain_prior)
    N, C = int(offs[-1]), len(offs) - 1
    cnt = np.diff(sp_off)
    chain = np.repeat(np.arange(C), np.diff(offs))
    k = np.arange(N)
    lo, hi = offs[chain], offs[chain + 1]
    kind = np.where(k < hi - 1, 0, np.where(hi - lo >= 2, 1, 2))
    tgt = np.where(kind == 0, k - chain, np.where(kind == 1, k - 1 - chain, chain))
    st = np.repeat(k, cnt)
    pos = np.arange(len(st)) - sp_off[st]
    if not f_only:
        for r in range(int(pos.max(initial=-1)) + 1):
            q = np.flatnonzero(pos == r)
            for kd, I, R in ((0, G11, g1), (1, G22, g2), (2, pi, pr)):
                qq = q[kind[st[q]] == kd]
                j = tgt[st[qq]]
                I[j] = I[j] + info[qq]
                R[j] = R[j] + rhs[qq]
    if f is not None:
        fpos = pos + np.where(kind[st] == 1, cnt[np.maximum(st - 1, 0)], 0)
        for r in range(int(fpos.max(initial=-1)) + 1):
            q = np.flatnonzero(fpos == r)
            for kd, F in ((0, fk), (1, fk), (2, pf)):
                qq = q[kind[st[q]] == kd]
                j = tgt[st[qq]]
                F[j] = F[j] + f[qq]
    return (G11, G22, g1, g2, fk), (pi, pr, pf)


def ld_loss(code, k, s):
    """(w, c) of one prior in long double; the threshold is k2 = k*k in fp64, as the kernel compares it."""
    L = np.longdouble
    k2d = np.float64(k) * np.float64(k)
    sl, kl, k2 = L(s), L(k), L(k2d)
    if code == capi.LOSS_GAUSSIAN:
        return L(1), sl
    if code == capi.LOSS_HUBER:
        if s <= k2d:
            return L(1), sl
        r = np.sqrt(sl)
        return kl / r, 2 * kl * r - k2
    u = sl / k2
    return 1 / (1 + u), k2 * np.log1p(u)


def edge_inputs():
    """(code, k, s): for Huber and Cauchy at k = 0.5, GTSAM's k and 10, and Gaussian: s = k^2 and its neighbours, 0, subnormal,
    1e-300, 1, 1e300, DBL_MAX, inf, NaN; with k = 0.5 also 1e308 and 5e307, where s / k^2 overflows."""
    rows = []
    for code, ks in ((capi.LOSS_HUBER, (0.5, HUBER_K, 10.0)), (capi.LOSS_CAUCHY, (0.5, CAUCHY_K, 10.0)), (capi.LOSS_GAUSSIAN, (0.0,))):
        for k in ks:
            k2 = k * k
            ss = [k2, np.nextafter(k2, 0.0), np.nextafter(k2, np.inf), 0.0, 3e-310, 1e-300, 1.0, 1e300, DBL_MAX, np.inf, np.nan]
            if k < 1:
                ss += [1e308, 5e307]
            rows += [(code, k, s) for s in ss]
    code, k, s = (np.array(a) for a in zip(*rows))
    return code.astype(np.int32), k.astype(np.float64), s.astype(np.float64)


def _ulps(got, want):
    with np.errstate(all="ignore"):
        return np.where(got == want, 0.0, np.abs(got - want) / np.spacing(np.abs(want)))


def cost_ulps(code, k, s, got, want):
    """ulps of a cost from the long-double value.  Where a Cauchy u = s/k^2 is subnormal, its rounding is absolute (up to 2^-1075)
    and k^2 scales it back: that bound, k^2 2^-1075, is taken off first.  Of the edge inputs only the Cauchy ones at s = 3e-310 take
    it; at k = 10 the cost is 7 ulp from the long-double value (the bound is 50 ulp there), in numpy as on the device (DESIGN.md
    section 3h).  Everywhere else the gate is the plain 2 ulp."""
    k2 = k * k
    with np.errstate(all="ignore"):
        slack = k2 / 2 * 2.0 ** -1074 if code == capi.LOSS_CAUCHY and s / k2 < np.finfo(np.float64).tiny else 0.0
        return 0.0 if got == want else max(abs(got - want) - slack, 0.0) / np.spacing(abs(want))


def _sms(torch):
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------

def test_builders_cover_the_second_paths_at_both_sm_counts():
    offs, counts = fold_batch()
    check_fold(offs, counts, SMS)
    for s in SMS:
        assert -(-int(offs[-1]) // fold_pass(s, len(offs) - 1)) >= 3
    offs, N = solve_layout(7)
    for s in SMS:
        B = chain_ids_pass(s, N)
        assert N > 2 * B
        c = int(np.searchsorted(offs, B, side="right") - 1)
        assert offs[c] < B - 1 and offs[c + 1] > B + 1
    sel = relin_plan()
    check_relin(sel)
    assert all(sel.sum() > 2 * relin_copy_pass(s, len(sel)) for s in SMS)


def test_bcr_pattern_depends_on_the_offset_mod_m():
    """The solve's level pattern of a chain of L <= 64 states depends only on its offset mod M(L), a power of two dividing TILE;
    offsets o and o + 1 give different patterns for L >= 2, so copies at the wrong residue would not be checked against their own
    arithmetic.  The LM batch's builder places every copy of a class at congruent offsets."""
    want = {1: 1, 2: 2, 3: 4, 4: 4, 5: 8, 6: 8, 8: 8, 9: 16, 12: 16, 16: 16, 17: 32, 30: 32, 31: 32, 32: 32, 33: 64, 64: 64}
    for L in range(1, 65):
        M = bcr_modulus(L)
        assert TILE % M == 0 and (L not in want or M == want[L]), (L, M)
        assert all(bcr_pattern(o, L) == bcr_pattern(o % M, L) for o in range(0, 4 * TILE))
        if L >= 2:
            assert all(bcr_pattern(o, L) != bcr_pattern(o + 1, L) for o in range(TILE))
    src, offs, cls, nan_at = lm_batch()
    check_lm_batch(np.asarray(LM_LENGTHS), src, offs, cls, nan_at, SMS)


def test_vectorised_fold_is_bitwise_the_loop_fold():
    rng = np.random.default_rng(4)
    sizes = np.r_[1, 2, 9, 1, 2, rng.integers(1, 12, size=40)]
    offs, blocks, chain_prior = random_layout(rng, sizes)
    N = int(offs[-1])
    idx = np.repeat(np.arange(N), rng.choice([0, 1, 2, 5], size=N))
    rng.shuffle(idx)
    M = len(idx)
    info, rhs, f = rng.normal(size=(M, 225)), rng.normal(size=(M, 15)), rng.normal(size=M) * 10.0 ** rng.integers(-8, 8, size=M)
    order, sp_off = csr(idx, N)
    G11, G12, G22, g1, g2, fk = blocks
    for f_only in (False, True):
        a = fold_ref(offs, sp_off, info[order], rhs[order], f[order], (G11, G22, g1, g2, fk), chain_prior, f_only=f_only)
        b = fold_ref_vec(offs, sp_off, info[order], rhs[order], f[order], (G11, G22, g1, g2, fk), chain_prior, f_only=f_only)
        for x, y in zip(a[0] + a[1], b[0] + b[1]):
            assert np.array_equal(x, y)


@pytest.mark.parametrize("tol", [TOL[0], TOL[1]])
def test_tie_cases(tol):
    """Every `at` vector has numpy's (x^2 + y^2) + z^2 exactly tol*tol and every `above` vector its successor; at least 8 of each
    give another sum when contracted into FMAs (either order), checked with exact rationals."""
    T = tol * tol
    at, above = tie_cases(tol, 10, 1)
    assert np.all(np_norm2(at) == T) and np.all(np_norm2(above) == np.nextafter(T, np.inf))
    F = fractions.Fraction
    for v in np.r_[at, above]:                                     # numpy's sum is the rule's: each operation rounded once
        x2, y2, z2 = (float(F(c) * F(c)) for c in v)
        assert float(F(float(F(x2) + F(y2))) + F(z2)) == np_norm2(v)
    flip_at = sum(all(c > T for c in contracted(*v)) for v in at)
    flip_above = sum(all(c <= T for c in contracted(*v)) for v in above)
    assert flip_at >= 8 and flip_above >= 8
    assert not np_select(1, _tie_states(at)[0], _tie_states(at)[1], tol, tol).any()
    assert np_select(1, _tie_states(above)[0], _tie_states(above)[1], tol, tol).all()


def _tie_states(v):
    """States i and lin with b_g - lin_bw = b_a - lin_ba = v exactly."""
    n = len(v)
    X, lin = np.zeros((n, 16)), np.zeros((n, 13))
    X[:, 3] = 1.0; lin[:, 9] = 1.0
    X[:, 4:7] = v; X[:, 10:13] = v
    return X, lin


def test_robust_loss_reference_and_the_overflow():
    """np_loss against the long-double statement on the edge inputs: w within 1 ulp and c within 2 ulp wherever finite, the same
    infinities and NaNs; at s / k^2 overflowing (Cauchy, k = 0.5, s = 1e308) the cost is k^2 ln(1 + s/k^2) = 177.6, where
    k^2 log1p(s/k^2) in fp64 gives inf."""
    code, k, s = edge_inputs()
    w, c = np_loss(code, k, s)
    for i in range(len(s)):
        wl, cl = ld_loss(code[i], k[i], s[i])
        wl, cl = np.float64(wl), np.float64(cl)
        if np.isnan(s[i]):
            assert np.isnan(c[i]), i
            continue
        assert (np.isinf(cl) and c[i] == cl) or cost_ulps(code[i], k[i], s[i], c[i], cl) <= 2.0, (code[i], k[i], s[i], c[i], cl)
        assert w[i] == wl or _ulps(w[i], wl) <= 1.0, (code[i], k[i], s[i], w[i], wl)
    with np.errstate(over="ignore"):
        assert np.isinf(0.25 * np.log1p(1e308 / 0.25))
    w1, c1 = np_loss(capi.LOSS_CAUCHY, 0.5, 1e308)
    assert abs(c1 - 0.25 * (np.log(1e308) + np.log(4.0))) <= 1e-13 * c1 and 177.0 < c1 < 178.0 and w1 == 0.25 / 1e308


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_fold_over_three_passes_is_bitwise_the_numpy_fold(cuda):
    """The fold on device offsets over >= 3 grid-stride passes on this device, chains straddling each boundary (the last factor's
    f written from both passes among them), single-state chains beside it and 0, 1 and 5 priors on its states: the fold and the
    f-only fold bitwise fold_ref."""
    from cpi_b200 import factor
    torch = cuda
    sms = _sms(torch)
    offs, counts = fold_batch(extra_sms=(sms,))
    check_fold(offs, counts, (sms,))
    rng = np.random.default_rng(11)
    N, C = int(offs[-1]), len(offs) - 1
    nf = N - C
    blocks = (rng.normal(size=(nf, 225)), rng.normal(size=(nf, 225)), rng.normal(size=(nf, 15)), rng.normal(size=(nf, 15)),
              rng.normal(size=nf))
    chain_prior = (rng.normal(size=(C, 225)), rng.normal(size=(C, 15)), rng.normal(size=C))
    sp_off = np.r_[0, np.cumsum(counts)].astype(np.int64)
    M = int(sp_off[-1])
    info, rhs, f = rng.normal(size=(M, 225)), rng.normal(size=(M, 15)), rng.normal(size=M)
    for f_only in (False, True):
        ref_b, ref_p = fold_ref_vec(offs, sp_off, info, rhs, f, blocks, chain_prior, f_only=f_only)
        tb, tp = [_dev(torch, a) for a in blocks], [_dev(torch, a) for a in chain_prior]
        factor.state_priors_fold(_dev(torch, offs), _dev(torch, sp_off), None if f_only else _dev(torch, info),
                                 None if f_only else _dev(torch, rhs), _dev(torch, f), *tb, *tp)
        for got, want in zip(tb + tp, list(ref_b) + list(ref_p)):
            assert np.array_equal(_host(got), want), f_only


@pytest.mark.gpu
def test_chains_solve_beyond_the_first_chain_ids_pass(cuda):
    """N = 2 cap + 1234 states (cap = sms * 2048, the states of one k_chain_ids pass) in chains of 1 .. 40 states: chains_solve is
    bitwise chain_solve.  With one chain beyond the first pass and the one straddling its end made indefinite, NaN falls in exactly
    those two chains and every other chain is bitwise the clean run."""
    from cpi_b200 import factor
    torch = cuda
    sms = _sms(torch)
    offs, N = solve_layout(7, tuple(dict.fromkeys(SMS + (sms,))))
    B = chain_ids_pass(sms, N)
    assert N > 2 * B
    f64 = dict(dtype=torch.float64, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(7)
    nb = 4096                                                      # diagonally dominant blocks: every chain SPD
    Db = torch.rand((nb, 15, 15), generator=g, **f64) * 0.02 - 0.01
    Db = Db + Db.transpose(1, 2) + 3.0 * torch.eye(15, **f64)
    Eb = (torch.rand((nb, 225), generator=g, **f64) - 0.5) * 0.1
    pick = lambda n: torch.randint(0, nb, (n,), generator=g, device="cuda")
    D = Db.reshape(nb, 225)[pick(N)]
    E = Eb[pick(N - 1)]
    E[_dev(torch, offs[1:-1] - 1)] = 0.0
    b = torch.randn((N, 15), generator=g, **f64)
    do = _dev(torch, offs)
    ws = torch.empty((int(capi.load().cpi_imu_chains_solve_workspace(len(offs) - 1, N)) + 7) // 8, **f64)
    x_iso = factor.chains_solve(D, E, b, do, workspace=ws).cpu().numpy()
    x_plain = factor.chain_solve(D, E, b, workspace=ws).cpu().numpy()
    assert np.all(np.isfinite(x_iso)) and np.array_equal(x_iso, x_plain)
    cA = int(np.searchsorted(offs, B + 5000, side="right"))       # a chain of >= 2 states wholly beyond the first pass
    while offs[cA + 1] - offs[cA] < 2:
        cA += 1
    cB = int(np.searchsorted(offs, B, side="right") - 1)          # the chain straddling its end
    assert offs[cB] < B - 1 and offs[cB + 1] > B + 1 and offs[cA] > B
    D[int(offs[cA]) + 1] = -torch.eye(15, **f64).reshape(225)
    D[B + 1] = -torch.eye(15, **f64).reshape(225)
    x_bad = factor.chains_solve(D, E, b, do, workspace=ws).cpu().numpy()
    nan_chain = np.add.reduceat(np.isnan(x_bad).any(axis=1), offs[:-1]) > 0
    assert np.array_equal(np.flatnonzero(nan_chain), sorted([cA, cB]))
    keep = np.repeat(~nan_chain, np.diff(offs))
    assert np.array_equal(x_bad[keep], x_iso[keep])


def _relin_case(rng, model, flags, sel, first_window):
    """Ragged windows of 0 .. 24 samples (empty ones included) on one chain of n + 1 states; the factors of `sel` drift past a
    tolerance (b_g or b_a, 1.5 .. 4 tolerances), the others stay within 0.1 .. 0.6 of both; model 2 keeps q_i = q_lin."""
    n = len(sel)
    S, off, L = windows(rng, n, 24, flags, True, first_window)
    X = np.zeros((n + 1, 16))
    X[:, 3] = 1.0
    X[:, 7:10] = rng.normal(size=(n + 1, 3)); X[:, 13:16] = rng.normal(size=(n + 1, 3))
    X[:n, 0:4] = L[:, 6:10]
    which = rng.integers(0, 2, n)
    for col, lcol, tol, j in ((4, 0, TOL[0], 0), (10, 3, TOL[1], 1)):
        u = rng.normal(size=(n, 3))
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        mag = np.where(sel & (which == j), rng.uniform(1.5, 4.0, n), rng.uniform(0.1, 0.6, n)) * tol
        X[:n, col:col + 3] = L[:, lcol:lcol + 3] + u * mag[:, None]
    for v, t in zip(sq_norms(model, X[:n], L), TOL):
        if v is not None:
            assert np.all(np.abs(v - t * t) > 1e-9 * t * t)
    assert np.array_equal(np_select(model, X[:n], L, *TOL), sel)
    return S, off, L, X


@pytest.mark.gpu
@pytest.mark.parametrize("model,flags", [(1, 0), (1, capi.FLAG_IMU_AVG), (2, 0)])
def test_relinearize_at_scale(cuda, model, flags):
    """70 201 ragged factors whose selection empties whole scan-thread ranges, runs across them, CTAs with one selected factor at
    thread 0 or 255, full CTAs and the partial last CTA's last factor, and selects more than two gather / scatter passes: mask, count
    and lin as np_select and new_lin, unselected slots keep their bits, selected records bitwise a preintegrate call over the whole
    batch at the new lin, two calls the same bits."""
    from cpi_b200 import factor, preint
    torch = cuda
    sel = relin_plan()
    assert sel.sum() > 2 * relin_copy_pass(_sms(torch), len(sel))
    rng = np.random.default_rng(40 + model + flags)
    S, off, L, X = _relin_case(rng, model, flags, sel, 300000)
    n = len(sel)
    dS, doff = _dev(torch, S), _dev(torch, off)
    rec0 = preint.preintegrate(model, dS, _dev(torch, L), synth.SIGMAS, flags, offsets=doff)
    runs = []
    for _ in range(2):
        dR, dL = rec0.clone(), _dev(torch, L)
        cnt, mask = factor.relinearize_records(model, _dev(torch, X), dR, dL, n + 1, dS, synth.SIGMAS, doff, None, flags,
                                               tol_bw=TOL[0], tol_ba=TOL[1], tol_theta=TOL[2])
        runs.append((cnt, mask.cpu().numpy().astype(bool), dR.cpu().numpy(), dL.cpu().numpy()))
    cnt, mask, rec, lin = runs[0]
    assert cnt == sel.sum() and np.array_equal(mask, sel)
    r0 = rec0.cpu().numpy()
    assert np.array_equal(rec[~sel], r0[~sel]) and np.array_equal(lin[~sel], L[~sel])
    assert np.array_equal(lin[sel], new_lin(model, X[:n][sel], L[sel]))
    full = preint.preintegrate(model, dS, _dev(torch, lin), synth.SIGMAS, flags, offsets=doff).cpu().numpy()
    assert np.array_equal(rec[sel], full[sel])
    assert runs[1][0] == cnt and all(np.array_equal(a, b) for a, b in zip(runs[0][1:], runs[1][1:]))


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_selection_ties_on_the_device(cuda, model):
    """b_g and b_a exactly at tol (not selected) and one ulp above (selected), half of them vectors whose FMA-contracted squared
    norm falls on the other side, spread over 4 CTAs: the mask is numpy's."""
    from cpi_b200 import factor, preint
    torch = cuda
    n, ns = 1024, 4
    rng = np.random.default_rng(60 + model)
    Sm, L = synth.make_windows(n, ns, rate=200.0, first_window=400000)
    L[:, 0:6] = 0.0
    X = np.zeros((n + 1, 16))
    X[:, 3] = 1.0
    X[:n, 0:4] = L[:, 6:10]
    want = np.zeros(n, bool)
    slots = rng.permutation(n)
    used = 0
    for col, tol, seed in ((4, TOL[0], 1), (10, TOL[1], 2)):
        at, above = tie_cases(tol, 10, seed)
        for v, sel in ((at, False), (above, True)):
            q = slots[used:used + len(v)]
            used += len(v)
            X[q, col:col + 3] = v
            want[q] = sel
    assert np.array_equal(np_select(model, X[:n], L, TOL[0], TOL[1], np.inf), want)
    dR = preint.preintegrate(model, _dev(torch, Sm.reshape(-1, 7)), _dev(torch, L), synth.SIGMAS, 0, ns=ns)
    cnt, mask = factor.relinearize_records(model, _dev(torch, X), dR, _dev(torch, L), n + 1, _dev(torch, Sm.reshape(-1, 7)), synth.SIGMAS,
                                           None, ns, 0, tol_bw=TOL[0], tol_ba=TOL[1], tol_theta=np.inf)
    assert np.array_equal(mask.cpu().numpy().astype(bool), want) and cnt == want.sum()


@pytest.mark.gpu
def test_robust_loss_edges_on_the_device(cuda):
    """The robust kernel on the edge inputs, info and rhs all ones so that the outputs carry w: Gaussian priors and Huber inliers
    (s <= k^2, s = k^2 included) copied bitwise, w bitwise numpy's, c within 2 ulp of the long-double value where that is finite
    (inf where it is inf, NaN for NaN s); s / k^2 overflowing gives the finite cost."""
    from cpi_b200 import factor
    torch = cuda
    code, k, s = edge_inputs()
    M = len(s)
    io, ro, fo = (t.cpu().numpy() for t in factor.state_priors_robust(_dev(torch, code), _dev(torch, k), _dev(torch, np.ones((M, 225))),
                                                                       _dev(torch, np.ones((M, 15))), _dev(torch, s)))
    w_np, _ = np_loss(code, k, s)
    assert np.array_equal(io, np.repeat(io[:, :1], 225, axis=1), equal_nan=True) and np.array_equal(ro, io[:, :15], equal_nan=True)
    w = io[:, 0]
    assert np.array_equal(w, w_np, equal_nan=True)
    inlier = (code == capi.LOSS_GAUSSIAN) | ((code == capi.LOSS_HUBER) & (s <= k * k))
    assert inlier.sum() >= 3 * 5 + 11 and np.array_equal(fo[inlier], s[inlier], equal_nan=True) and np.all(w[inlier] == 1.0)
    worst = 0.0
    for i in range(M):
        wl, cl = (np.float64(v) for v in ld_loss(code[i], k[i], s[i]))
        if np.isnan(s[i]):
            assert np.isnan(fo[i]), i
        elif np.isinf(cl):
            assert fo[i] == cl, (code[i], k[i], s[i], fo[i])
        else:
            u = cost_ulps(code[i], k[i], s[i], fo[i], cl)
            worst = max(worst, u)
            assert u <= 2.0, (code[i], k[i], s[i], fo[i], cl, u)
    over = (code == capi.LOSS_CAUCHY) & (k < 1) & (s >= 5e307) & np.isfinite(s)
    assert over.sum() == 3 and np.all(np.isfinite(fo[over])) and np.all(fo[over] < 178.0)
    print(f"robust losses at the edges: {M} inputs, worst cost {worst:.2f} ulp from long double")


def _lm_tiled(oracle, model, sms):
    """The LM batch of chain_scale.lm_batch for one model: 40 distinct chains of make_problem (every other with a zero chain prior),
    position, velocity and full measurement fixes every third state under Gaussian, Huber and Cauchy losses, every fifth an
    outlier; tiled copies bit for bit; the NaN copies' fixes at NaN.  Returns the distinct problem, the tiling and the tiled
    arrays."""
    lengths = np.asarray(LM_LENGTHS)
    rng = np.random.default_rng(80 + model)
    X, rec, L, offs, pri, per = make_problem(oracle, model, lengths, 500 + model, large=True, with_prior=True, first_window=120000)
    for c in range(1, len(lengths), 2):
        pri[c] = (np.zeros((15, 15)), np.zeros(15), 0.0, pri[c][3])
    sp = add_outliers(_meas_priors(oracle, rng, X, offs, 3, "mixed"), 5, 0.5)
    loss = mixed_losses(len(sp[0]))
    src, toffs, cls, nan_at = lm_batch(lengths, tuple(dict.fromkeys(SMS + (sms,))))
    sidx = np.concatenate([np.arange(offs[c], offs[c + 1]) for c in src])
    fidx = np.concatenate([np.arange(offs[c] - c, offs[c + 1] - c - 1) for c in src])
    chain_of = np.searchsorted(offs, sp[0], side="right") - 1
    mine = [np.flatnonzero(chain_of == c) for c in range(len(lengths))]
    q = np.concatenate([mine[c] for c in src])
    qi = np.concatenate([toffs[i] + sp[0][mine[c]] - offs[c] for i, c in enumerate(src)]).astype(np.int64)
    lin_t = sp[4][q].copy()
    for i in nan_at:
        lin_t[np.isin(qi, np.arange(toffs[i], toffs[i + 1]))] = np.nan
    PI = np.stack([p[0].reshape(225, order="F") for p in pri])
    tiled = dict(X=X[sidx], rec=rec[fidx], L=L[fidx], offs=toffs,
                 prior=(PI[src], np.stack([p[1] for p in pri])[src], np.array([p[2] for p in pri])[src], np.stack([p[3] for p in pri])[src]),
                 sp=(qi, sp[1][q], sp[2][q], sp[3][q], lin_t), sp_clean=(qi, sp[1][q], sp[2][q], sp[3][q], sp[4][q]),
                 loss=(loss[0][q], loss[1][q]))
    return (X, rec, L, offs, pri, per, sp, loss), (src, cls, nan_at), tiled


def _same_per_class(arrs_per_copy, cls, skip):
    """Every copy bitwise the first copy of its class (copies in `skip` left out)."""
    first = {}
    for i, k in enumerate(cls):
        if i in skip:
            continue
        j = first.setdefault(int(k), i)
        for a in arrs_per_copy:
            assert np.array_equal(a(i), a(j)), (i, j)


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_chains_lm_on_the_tiled_batch(cuda, oracle, model):
    """chains_lm on about 300 000 states, 14 000 chains: every copy bitwise its class's first copy in states, cost, lambda, status,
    iterations and tries, and chains_lm_step likewise in its step and cost; the copies beyond the first k_chain_ids pass of this
    device take np_lm_rb's accept or reject in each of the first 16 rounds and end at its lambda, status and counters, their states at the gates of
    test_robust_priors.py; the NaN copies end non-finite and the chains beside them are bitwise their classes."""
    from cpi_b200 import factor
    torch = cuda
    sms = _sms(torch)
    (X, rec, L, offs, pri, per, sp, loss), (src, cls, nan_at), t = _lm_tiled(oracle, model, sms)
    toffs = t["offs"]
    d = lambda a: _dev(torch, a)
    args = (d(t["X"]), d(t["rec"]), d(t["L"]), d(toffs))
    kw = dict(prior=tuple(d(a) for a in t["prior"]), state_priors=_sp_dev(torch, *t["sp"]), state_prior_loss=tuple(d(a) for a in t["loss"]))
    sps = per_chain_rb(offs, *sp, *loss)
    ref = [np_lm_rb(oracle, model, Xc, r, l, pri[c], sps[c]) for c, (Xc, r, l) in enumerate(per)]
    for o in ref:
        well_posed(o[6])
    Xs, cost, lam, st, it, tr = (a.cpu().numpy() for a in factor.chains_lm(model, *args, **kw))
    seg = lambda A: (lambda i: A[toffs[i]:toffs[i + 1]])
    per_c = lambda A: (lambda i: A[i])
    skip = set(nan_at)
    _same_per_class([seg(Xs), per_c(cost), per_c(lam), per_c(st), per_c(it), per_c(tr)], cls, skip)
    for i in nan_at:
        assert st[i] == capi.LM_NONFINITE and st[i - 1] != capi.LM_NONFINITE and st[i + 1] != capi.LM_NONFINITE
    assert np.sum(st == capi.LM_NONFINITE) == len(nan_at)
    kw_clean = dict(kw, state_priors=_sp_dev(torch, *t["sp_clean"]))   # one solve over all chains: a NaN chain would reach them all
    Xn, dx, c0 = (a.cpu().numpy() for a in factor.chains_lm_step(model, *args, **kw_clean))
    assert np.all(np.isfinite(dx))
    _same_per_class([seg(Xn), seg(dx), per_c(c0)], cls, skip)
    B1 = chain_ids_pass(sms, int(toffs[-1]))
    beyond = np.flatnonzero((toffs[:-1] > B1) & ~np.isin(np.arange(len(src)), nan_at))
    assert set(src[beyond]) == set(range(len(per)))
    R = min(max(o[5] for o in ref), 16)                            # rounds checked decision by decision (each a run of r rounds)
    prev = np.zeros(len(src), np.int32)
    worst = 0.0
    for r in range(1, R + 1):
        it_r = factor.chains_lm(model, *args, max_rounds=r, check_every=0, **kw)[4].cpu().numpy()
        for i in beyond:
            o = ref[src[i]]
            if r <= o[5]:
                assert bool(it_r[i] > prev[i]) == o[6][r - 1][0], (r, i, src[i])
        prev = it_r
    for i in beyond:
        o = ref[src[i]]
        assert (lam[i], st[i], it[i], tr[i]) == (o[2], o[3], o[4], o[5]), (i, src[i])
        worst = max(worst, np.linalg.norm(local(o[0], seg(Xs)(i))) / max(np.linalg.norm(o[0][:, 4:16]), 1e-300))
    print(f"model {model}: {len(src)} chains, {int(toffs[-1])} states, {len(set(cls))} classes, {R} rounds; {len(beyond)} copies beyond "
          f"state {B1} against numpy, worst final-state distance {worst:.2e}")
    assert worst <= (1e-9 if model == 1 else 2e-7)


@pytest.mark.gpu
def test_chain_marginalize_on_the_tiled_batch(cuda, oracle):
    """K8 on the tiled batch (model 1) with a per-chain n_marg, the chain priors and the moved Gaussian and robust state priors:
    every chain's (info, rhs, f) bitwise chain_marginalize of that chain alone (a single-state chain: its prior as given)."""
    from cpi_b200 import factor
    torch = cuda
    (X, rec, L, offs, pri, per, sp, loss), (src, cls, nan_at), t = _lm_tiled(oracle, 1, _sms(torch))
    toffs = t["offs"]
    lengths = np.asarray(LM_LENGTHS)
    qi, info, rhs, f, _ = t["sp"]
    lin = t["X"][qi]                                               # moved to the tiled states: finite everywhere
    rng = np.random.default_rng(5)
    nm_c = np.array([rng.integers(0, n) for n in lengths], dtype=np.int64)
    nm = nm_c[src]
    d = lambda a: _dev(torch, a)
    dX = d(t["X"])
    e, H1, H2 = factor.factor_eval(1, dX, d(t["rec"]), d(t["L"]), *_chain_idx(torch, toffs))
    G = factor.factor_hessian(1, d(t["rec"]), e, H1, H2)
    msp = _moved(torch, (qi, info, rhs, f, lin), t["X"])
    pr = tuple(d(a) for a in t["prior"][:3])
    out = [a.cpu().numpy() for a in factor.chain_marginalize(*G, d(toffs), d(nm), prior=pr, state_priors=msp,
                                                            state_prior_loss=tuple(d(a) for a in t["loss"]))]
    first = {}
    for i, c in enumerate(src):
        first.setdefault(int(c), i)
    for c, i in first.items():
        lo, hi = int(toffs[i]), int(toffs[i + 1])
        if hi - lo == 1:                                           # nothing to eliminate: the chain prior as given
            for j in np.flatnonzero(src == c):
                assert all(np.array_equal(o[j], a[j]) for o, a in zip(out, t["prior"][:3])), (c, j)
            continue
        f0 = lo - i
        Gc = [g[f0:f0 + hi - lo - 1] for g in G]
        q = np.flatnonzero((qi >= lo) & (qi < hi))
        alone = factor.chain_marginalize(*Gc, d(np.array([0, hi - lo], dtype=np.int64)), d(nm_c[c:c + 1]),
                                         prior=tuple(a[i:i + 1] for a in pr),
                                         state_priors=(d(qi[q] - lo),) + tuple(a[d(q)] for a in msp[1:]),
                                         state_prior_loss=(d(t["loss"][0][q]), d(t["loss"][1][q])))
        alone = [a.cpu().numpy()[0] for a in alone]
        for j in np.flatnonzero(src == c):
            assert all(np.array_equal(o[j], a) for o, a in zip(out, alone)), (c, j)
