"""Precision of the chain marginals -- the selected inversion of the block cyclic reduction (k_bcr_selinv_root, k_bcr_selinv_iso;
cpi_imu_chains_marginals, factor.chains_covariance / chains_marginals; DESIGN.md section 3j) -- against an extended-precision truth.

The truth is the long-double build of oracle_chain_marginals (oracle/cpi_oracle.c) in its sequential route: per chain the block
Cholesky M_k = D_k - U_{k-1}^T U_{k-1} = L_k L_k^T, U_k = L_k^-1 E_k, then Sigma_{n-1} = M_{n-1}^-1, Sigma_{k,k+1} = -L_k^-T U_k
Sigma_{k+1,k+1}, Sigma_kk = L_k^-T (L_k^-1 - U_k Sigma_{k,k+1}^T).  Its other route (order 1) is the kernels' own: the isolated forward
phase on a zero right-hand side and the top-down level walk in solve.cu's order.

Errors are measured per chain, per block kind (Sigma_kk, Sigma_{k,k+1}) and per 3x3 component pair of (theta, b_g, v, b_a, p)^2, never
as a whole-matrix norm: each field is the largest |dSigma|_ij / sqrt(T_ii T_jj) over the chain's states, T the truth's diagonal
blocks (for Sigma_{k,k+1}: T_ii of state k, T_jj of state k+1).  The gate is e_dev <= K max(e_64, floor), K = 8, floor = 1e-15
(parity.gate_errors), e_64 the larger error of the two fp64 routes of the oracle (sequential and the kernels' order).

Inputs: the chain stress batch of tests/test_chain_precision.py (every damping of its solve gate; undamped on the ragged layout
only, since the long undamped stress chains are singular in fp64), single chains of 2^k and 2^k +- 1 states up to k = 13, the
5 000-state chain of test_chain_marginals.test_scale (both models), and the tiled production batch of tests/chain_scale.lm_batch.

CPU tests: the long-double routes against a long-double dense inverse and the refined inverse (short chains), against each other, the kernels'
route against test_chain_marginals.selinv_ref, the gate passing both fp64 routes and failing three injected errors."""
import time

import numpy as np
import pytest

import chain_stress as cs
import test_chain_marginals as tcm
from chain_scale import TILE, chain_ids_pass, SMS
from parity import gate_errors
from test_chain_precision import _dev, _ld_solve, _threads, assemble, batch, oracles, solve_systems, worst_line  # noqa: F401
from test_marginalize import mat, vec

K, FLOOR = 8.0, 1e-15
COMP = ("theta", "b_g", "v", "b_a", "p")
FIELDS_KK = [(I, J) for I in range(5) for J in range(I, 5)]      # Sigma_kk is symmetric
FIELDS_X = [(I, J) for I in range(5) for J in range(5)]

_cache = {}


# ---------------------------------------------------------------------------------------------- the error measure and gate

def _blocks(A):
    """[n, 15, 15] -> [n, 5, 5]: the largest entry of every 3x3 component block."""
    return A.reshape(-1, 5, 3, 5, 3).max(axis=(2, 4))


def marg_errors(got, truth, off):
    """dict field -> [C]: "Skk I.J" (I <= J) and "Sx I.J" (Sigma_{k,k+1}), per chain the largest |dSigma|_ij / sqrt(T_ii T_jj) over its
    states.  got, truth: (cov [N,225], cross [N-C,225]) in the slots of cpi_imu_chains_marginals.  A NaN in got is a NaN error."""
    off = np.asarray(off)
    C, N = len(off) - 1, int(off[-1])
    cov, cross = got
    tc, tx = truth
    d = 1.0 / np.sqrt(tc[:, ::16])                                # the truth's diagonal, [N, 15]
    ek = _blocks(np.abs(mat(cov) - mat(tc)) * d[:, :, None] * d[:, None, :])
    per_k = np.maximum.reduceat(ek, off[:-1], axis=0)
    per_x = np.zeros((C, 5, 5))
    xo = off - np.arange(C + 1)
    has = np.diff(xo) > 0
    if has.any():
        chain = np.repeat(np.arange(C), np.diff(off))
        left = np.flatnonzero(chain[:-1] == chain[1:])
        ex = _blocks(np.abs(mat(cross) - mat(tx)) * d[left][:, :, None] * d[left + 1][:, None, :])
        per_x[has] = np.maximum.reduceat(ex, xo[:-1][has], axis=0)
    out = {f"Skk {COMP[I]}.{COMP[J]}": per_k[:, I, J] for I, J in FIELDS_KK}
    out.update({f"Sx {COMP[I]}.{COMP[J]}": per_x[:, I, J] for I, J in FIELDS_X})
    return out


def marg_gate(got, t, s, r, off):
    """(ratio, worst, failures) of got against the long-double truth t; e_64 the larger error of the fp64 routes s (sequential) and r
    (the kernels' order)."""
    ed = marg_errors(got, t, off)
    es, er = marg_errors(s, t, off), marg_errors(r, t, off)
    return gate_errors(ed, {k: np.maximum(es[k], er[k]) for k in es}, K, FLOOR)


def marg_truths(o64, old, key, off, D, E):
    """(t, s, r): the long-double sequential truth, the fp64 sequential route and the fp64 route in the kernels' order."""
    if key not in _cache:
        kw = dict(chain_offsets=off)
        t = old.chain_marginals(D, E, 0, nthreads=_threads(), **kw)
        s = o64.chain_marginals(D, E, 0, nthreads=_threads(), **kw)
        r = o64.chain_marginals(D, E, 1, **kw)
        _cache[key] = (t, s, r)
    return _cache[key]


def systems(b, which):
    """(name, D, E) of every damping of test_chain_precision's solve gate on one layout, assembled by its numpy statement."""
    key = ("sys", which)
    if key not in _cache:
        lay = b[which]
        _cache[key] = [(name, *assemble(lay, lam, diag, pi, pr)[:2]) for name, lam, diag, pi, pr, _ in solve_systems(b, which)]
    return _cache[key]


def _worst(worst):
    k = max(worst, key=lambda f: worst[f]["ratio"])
    return worst[k]["ratio"], k


def _chain_err(got, T, n):
    """The largest block error of one chain's (cov, cross) against its dense inverse T, in the units of T's diagonal."""
    d = 1.0 / np.sqrt(np.diag(T).astype(np.float64))
    cov, cross = mat(got[0]), mat(got[1])
    e = 0.0
    for k in range(n):
        blk = [(cov[k], k, k)] + ([(cross[k], k, k + 1)] if k + 1 < n else [])
        for B, I, J in blk:
            Tb = T[15 * I:15 * I + 15, 15 * J:15 * J + 15]
            e = max(e, float(np.max(np.abs(B - Tb) * d[15 * I:15 * I + 15, None] * d[None, 15 * J:15 * J + 15])))
    return e


# ---------------------------------------------------------------------------------------------------------- CPU

def test_extended_marginals_are_the_dense_inverse(oracles):
    """On chains of 2 .. 6 states of the ragged layout under every damping and every prior kind: the long-double sequential route
    matches a long-double dense Gauss-Jordan inverse (no pivoting) to 1e-14 in the units of the diagonal, or to the fp64 route's
    distance where that is larger (the 1e12 and nearly rank-deficient priors): an algebra slip would be orders of magnitude above."""
    o64, old = oracles
    b = batch(o64)
    off = b["ragged"]["offsets"]
    sel = [c for c in range(len(off) - 1) if 2 <= off[c + 1] - off[c] <= 6]
    worst, n = 0.0, 0
    for name, D, E in systems(b, "ragged"):
        t, s, _ = marg_truths(o64, old, ("ragged", name), off, D, E)
        for c in sel[:40]:
            lo, hi = int(off[c]), int(off[c + 1])
            A = tcm.dense(mat(D), mat(E), lo, hi)
            A = np.tril(A) + np.tril(A, -1).T
            T = _ld_solve(A, np.eye(len(A)))
            xs = slice(lo - c, hi - c - 1)
            e_ld = _chain_err((t[0][lo:hi], t[1][xs]), T, hi - lo)
            e_64 = _chain_err((s[0][lo:hi], s[1][xs]), T, hi - lo)
            worst = max(worst, e_ld / max(e_64, 1e-300))
            assert e_ld <= max(e_64, 1e-14), (name, c, e_ld, e_64)
            n += 1
    print(f"long-double sequential route vs long-double dense inverse, {n} chains: worst {worst:.1e} of the fp64 route's distance")


def test_extended_marginals_agree_with_the_refined_inverse(oracles):
    """The long-double sequential route against test_chain_marginals.inv_truth (a Jacobi-scaled fp64 inverse refined twice with 80-bit
    residuals) on the chains of 2 .. 33 states of the main layout that carry a chain prior (lambda I and Marquardt): per chain and field
    within 1e-2 of e_64, the fp64 routes' error against the same truth, plus the two outputs' fp64 rounding (2.3e-16 in the units of
    the diagonal).  Without a prior, lambda I = 1e-3 alone holds the gauge (condition ~1e11) and two refinement steps leave inv_truth
    itself at a third of e_64; the long-double dense inverse gates those chains."""
    o64, old = oracles
    b = batch(o64)
    off = b["main"]["offsets"]
    worst = 0.0
    for (name, D, E), sysp in zip(systems(b, "main")[0:2], solve_systems(b, "main")[0:2]):
        kinds = sysp[5]
        t, s, r = marg_truths(o64, old, ("main", name), off, D, E)
        Dm, Em = mat(D), mat(E)
        for c in range(len(off) - 1):
            lo, hi = int(off[c]), int(off[c + 1])
            if hi - lo < 2 or hi - lo > 33 or kinds[c] == "none":
                continue
            R, _ = tcm.inv_truth(tcm.dense(Dm, Em, lo, hi))
            tr = (vec(np.stack([R[15 * k:15 * k + 15, 15 * k:15 * k + 15] for k in range(hi - lo)])),
                  vec(np.stack([R[15 * k:15 * k + 15, 15 * k + 15:15 * k + 30] for k in range(hi - lo - 1)])))
            one = np.array([0, hi - lo])
            pick = lambda x: (x[0][lo:hi], x[1][lo - c:hi - c - 1])
            e_t = marg_errors(pick(t), tr, one)
            es, er = marg_errors(pick(s), tr, one), marg_errors(pick(r), tr, one)
            for k in e_t:
                e64 = max(es[k][0], er[k][0])
                worst = max(worst, e_t[k][0] / max(e64, 1e-16))
                assert e_t[k][0] <= 1e-2 * e64 + 2.3e-16, (name, c, k, e_t[k][0], e64)
    print(f"long-double sequential route vs the refined fp64 inverse: worst {worst:.1e} of e_64")


def test_the_two_extended_routes_agree(oracles):
    """The long-double route in the kernels' order against the long-double sequential route on every layout and damping: per chain
    and field within 1e-2 of e_64 plus the two outputs' fp64 rounding (2.3e-16 in the units of the diagonal)."""
    o64, old = oracles
    b = batch(o64)
    for which in ("main", "ragged"):
        off = b[which]["offsets"]
        for name, D, E in systems(b, which):
            t, s, r = marg_truths(o64, old, (which, name), off, D, E)
            t1 = old.chain_marginals(D, E, 1, chain_offsets=off)
            e1 = marg_errors(t1, t, off)
            es, er = marg_errors(s, t, off), marg_errors(r, t, off)
            worst = 0.0
            for k in e1:
                e64 = np.maximum(es[k], er[k])
                worst = max(worst, float(np.max(e1[k] / np.maximum(e64, 1e-16))))
                assert np.all(e1[k] <= 1e-2 * e64 + 2.3e-16), (which, name, k)
            print(f"{which} {name}: the long-double routes agree to {worst:.1e} of e_64")


def test_kernel_order_route_is_the_numpy_level_walk(oracles):
    """The fp64 route in the kernels' order against test_chain_marginals.selinv_ref on random ragged systems (1 .. 70 states): equal to
    rounding (1e-13 in the units of the diagonal), exact zeros where selinv_ref has them.  On the ragged stress layout, a chain made
    indefinite gets NaN in every one of its blocks and leaves every other chain bitwise as it was."""
    o64, _ = oracles
    rng = np.random.default_rng(3)
    sizes = [1, 2, 3, 4, 5, 7, 8, 9, 1, 1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 70, 1, 13]
    D, E, offs, cid = tcm.random_system(rng, sizes)
    cov, nb = tcm.selinv_ref(D, E, cid)
    c1, x1 = o64.chain_marginals(vec(D), vec(E), 1, chain_offsets=offs)
    same = cid[:-1] == cid[1:]
    d = 1.0 / np.sqrt(np.einsum("nii->ni", cov))
    e_k = np.max(np.abs(mat(c1) - cov) * d[:, :, None] * d[:, None, :])
    k = np.flatnonzero(same)
    e_x = np.max(np.abs(mat(x1) - nb[k]) * d[k][:, :, None] * d[k + 1][:, None, :])
    print(f"kernels' order (fp64 oracle) vs selinv_ref: {e_k:.1e} (Sigma_kk), {e_x:.1e} (Sigma_k,k+1)")
    assert e_k <= 1e-13 and e_x <= 1e-13
    assert np.array_equal(mat(x1) == 0, nb[k] == 0)
    b = batch(o64)
    off = b["ragged"]["offsets"]
    name, D, E = systems(b, "ragged")[1]
    clean = o64.chain_marginals(D, E, 1, chain_offsets=off)
    for c in (0, 7, 100):
        Db = D.copy()
        Db[int(off[c])] *= -1
        bad = o64.chain_marginals(Db, E, 1, chain_offsets=off)
        _check_nan_chain(bad, clean, off, c)


def _check_nan_chain(bad, clean, off, c):
    """Every Sigma_kk and cross slot of chain c holds a NaN; every other chain is bitwise `clean`."""
    lo, hi = int(off[c]), int(off[c + 1])
    xs = np.s_[lo - c:hi - c - 1]
    assert np.isnan(bad[0][lo:hi]).any(axis=1).all() and np.isnan(bad[1][xs]).any(axis=1).all(), c
    assert np.array_equal(np.delete(bad[0], np.s_[lo:hi], axis=0), np.delete(clean[0], np.s_[lo:hi], axis=0)), c
    assert np.array_equal(np.delete(bad[1], xs, axis=0), np.delete(clean[1], xs, axis=0)), c


def test_gate_passes_the_fp64_routes(oracles):
    o64, old = oracles
    b = batch(o64)
    for which in ("main", "ragged"):
        off = b[which]["offsets"]
        for name, D, E in systems(b, which):
            t, s, r = marg_truths(o64, old, (which, name), off, D, E)
            for x in (s, r):
                assert not marg_gate(x, t, s, r, off)[2], (which, name)
            _, w_seq, _ = gate_errors(marg_errors(r, t, off), marg_errors(s, t, off), K, FLOOR)
            print(which, name, "fp64 kernels' order against the sequential route's e_64 alone: %.2f (%s)" % _worst(w_seq))


def _old_gates_catch(got, D, E, off, short=33):
    """Whether the criteria of test_chain_marginals.py catch got: on the chains of at most `short` states, the device's worst block
    error against the refined dense inverse above 50x the plain fp64 inverse's (floor 1e-13) (_gate_chains); on every chain, a
    non-finite block or a diagonal block that is not positive definite (test_scale)."""
    cov, cross = got
    if not (np.all(np.isfinite(cov)) and np.all(np.isfinite(cross))):
        return True
    if np.any(np.linalg.eigvalsh(0.5 * (mat(cov) + mat(cov).transpose(0, 2, 1)))[:, 0] <= 0):
        return True
    Dm, Em = mat(D), mat(E)
    ed = ep = 0.0
    for c in range(len(off) - 1):
        lo, hi = int(off[c]), int(off[c + 1])
        if hi - lo > short:
            continue
        T, P64 = tcm.inv_truth(tcm.dense(Dm, Em, lo, hi))
        ed = max(ed, _chain_err((cov[lo:hi], cross[lo - c:hi - c - 1]), T, hi - lo))
        n = hi - lo
        p = (vec(np.stack([P64[15 * k:15 * k + 15, 15 * k:15 * k + 15] for k in range(n)])),
             vec(np.stack([P64[15 * k:15 * k + 15, 15 * k + 15:15 * k + 30] for k in range(n - 1)])) if n > 1 else np.zeros((0, 225)))
        ep = max(ep, _chain_err(p, T, n))
    return ed > 50 * max(ep, 1e-13)


def test_gate_fails_injected_errors(oracles):
    """One Sigma_kk 3x3 block rounded to fp32; the b_a rows of Sigma_{k,k+1} scaled by 1 + 1e-7; a level walk (selinv_ref's hook) that
    reads Sigma_{i+1,i-1} untransposed at strides >= 64 only.  Each fails the gate; how many the criteria of test_chain_marginals.py
    catch is printed."""
    o64, old = oracles
    b = batch(o64)
    off = b["main"]["offsets"]
    name, D, E = systems(b, "main")[0]
    t, s, r = marg_truths(o64, old, ("main", name), off, D, E)
    caught = []
    # one Sigma_kk block (b_a, b_a) rounded to fp32, in the chain of >= 5 states where the fp64 routes are most accurate
    es, er = marg_errors(s, t, off)["Skk b_a.b_a"], marg_errors(r, t, off)["Skk b_a.b_a"]
    c = int(np.argmin(np.where(np.diff(off) >= 5, np.maximum(es, er), np.inf)))
    k = int(off[c]) + 2
    got = (s[0].copy(), s[1].copy())
    S = mat(got[0][k:k + 1])[0].copy()
    S[9:12, 9:12] = S[9:12, 9:12].astype(np.float32).astype(np.float64)
    got[0][k] = vec(S[None])[0]
    bad = marg_gate(got, t, s, r, off)[2]
    assert any(x.startswith("Skk b_a.b_a") for x in bad), bad
    caught.append(("fp32 Sigma_kk block", _old_gates_catch(got, D, E, off)))
    # the b_a rows of every Sigma_{k,k+1} scaled by 1 + 1e-7
    X = mat(s[1]).copy()
    X[:, 9:12, :] *= 1 + 1e-7
    got = (s[0], vec(X))
    bad = marg_gate(got, t, s, r, off)[2]
    assert any(x.startswith("Sx b_a.") for x in bad), bad
    caught.append(("b_a rows of Sigma_k,k+1 x (1 + 1e-7)", _old_gates_catch(got, D, E, off)))
    # Sigma_{i+1,i-1} read untransposed at strides >= 64: chains of more than 128 states only
    chain = np.repeat(np.arange(len(off) - 1), np.diff(off))
    far = lambda stride, N: N if stride >= 64 else N.T
    cov, nb = tcm.selinv_ref(mat(D), mat(E), chain, far=far)
    got = (vec(cov), vec(nb[chain[:-1] == chain[1:]]))
    ratio, worst, bad = marg_gate(got, t, s, r, off)
    assert bad, worst
    hit = {int(i) for k_ in ratio for i in np.flatnonzero(~(ratio[k_] <= 1))}
    assert hit and all(off[i + 1] - off[i] > 128 for i in hit), sorted(hit)
    caught.append(("Sigma_i+1,i-1 untransposed at stride >= 64", _old_gates_catch(got, D, E, off)))
    print("injected errors the criteria of test_chain_marginals.py catch:", ", ".join(f"{n}: {'yes' if y else 'no'}" for n, y in caught))


# ---------------------------------------------------------------------------------------------------------- GPU

def _cov(factor, torch, D, E, off, cross=True):
    """chains_covariance on host arrays (off: offsets [C+1] or an int, the uniform layout); numpy (cov, cross)."""
    o = _dev(torch, off) if isinstance(off, np.ndarray) else int(off)
    cv, cr = factor.chains_covariance(_dev(torch, D), _dev(torch, E.reshape(-1, 225)), o, cross=cross)
    return cv.cpu().numpy(), (None if cr is None else cr.cpu().numpy())


def _symmetric(cov):
    return np.array_equal(mat(cov), mat(cov).transpose(0, 2, 1))


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["main", "ragged"])
def test_stress_batch_against_extended_oracle(cuda, oracles, which):
    """chains_covariance on every damping of the solve gate (undamped on ragged only): Sigma_kk and Sigma_{k,k+1} per chain and field
    against the long-double truth; Sigma_kk exactly symmetric; cov the same bits with and without cross; the uniform and
    device-offset layouts the same bits on the main layout's six 21-state chains; (ragged) a chain made indefinite at each boundary
    residue mod 64 gets NaN in every one of its blocks and leaves every other chain bitwise the clean run."""
    from cpi_b200 import factor
    torch = cuda
    o64, old = oracles
    b = batch(o64)
    off = b[which]["offsets"]
    t0 = time.time()
    for name, D, E in systems(b, which):
        t, s, r = marg_truths(o64, old, (which, name), off, D, E)
        got = _cov(factor, torch, D, E, off)
        assert _symmetric(got[0])
        assert np.array_equal(_cov(factor, torch, D, E, off, cross=False)[0], got[0])
        _, w_seq, _ = gate_errors(marg_errors(r, t, off), marg_errors(s, t, off), K, FLOOR)
        ratio, worst, bad = marg_gate(got, t, s, r, off)
        worst_line(f"marginals {which} {name} (fp64 kernels' order on the sequential e_64 alone: {_worst(w_seq)[0]:.2f})", worst)
        assert not bad, (name, bad)
    if which == "main":
        S = np.diff(off)
        c0 = int(np.flatnonzero(S == 21)[0])
        assert np.all(S[c0:c0 + 6] == 21)
        lo, hi = int(off[c0]), int(off[c0 + 6])
        Ds, Es = D[lo:hi], E[lo:hi - 1]
        u = _cov(factor, torch, Ds, Es, 21)
        o = _cov(factor, torch, Ds, Es, off[c0:c0 + 7] - lo)
        assert np.array_equal(u[0], o[0]) and np.array_equal(u[1], o[1])
        return
    clean = got
    done = set()
    for c in range(len(off) - 1):
        r64 = int(off[c] % 64)
        if r64 in done:
            continue
        done.add(r64)
        Db = D.copy()
        Db[int(off[c])] *= -1
        _check_nan_chain(_cov(factor, torch, Db, E, off), clean, off, c)
    assert len(done) == 64
    print(f"chain made indefinite at each of the {len(done)} boundary residues mod 64: NaN in it alone; {time.time() - t0:.1f} s")


def _stress_chain(o64, lengths, seed):
    """Single SPD chains of the stress pool's records, lambda I = 1e-3 and a 1e8 or dense chain prior: [(D, E)] per length."""
    b = batch(o64)
    rng = np.random.default_rng(seed)
    lay = cs.chains(o64, b["pool"], list(lengths), rng)
    pi, pr, _, _ = cs.priors(rng, len(lengths), ("1e8", "dense"))
    D, E, _, _ = assemble(lay, 1e-3, False, pi, pr)
    off = lay["offsets"]
    return [(D[off[c]:off[c + 1]], E[off[c]:off[c + 1] - 1]) for c in range(len(lengths))]


@pytest.mark.gpu
def test_edges_against_extended_oracle(cuda, oracles):
    """One state (the root alone, cross requested and empty); all single-state chains (N = C = 37, cross with zero rows, uniform and
    device offsets); one chain of 2^k and 2^k +- 1 states for k up to 13 (8 193 states): each against the oracle."""
    from cpi_b200 import factor
    torch = cuda
    o64, old = oracles
    lengths = sorted({n for k in range(1, 14) for n in (2 ** k - 1, 2 ** k, 2 ** k + 1)})
    sys_ = _stress_chain(o64, [1] * 37 + lengths, 11)
    D1 = np.concatenate([d for d, _ in sys_[:37]])
    gated = []
    for label, D, E, off in [("one state", D1[:1], np.zeros((0, 225)), np.array([0, 1])),
                             ("37 single-state chains", D1, np.zeros((36, 225)), np.arange(38))] + \
                            [(f"one chain of {len(d)}", d, e, np.array([0, len(d)])) for d, e in sys_[37:]]:
        t, s, r = marg_truths(o64, old, ("edge", label), off, D, E)
        got = _cov(factor, torch, D, E, off)
        assert got[1].shape == (len(D) - len(off) + 1, 225) and _symmetric(got[0])
        u = _cov(factor, torch, D, E, len(D) // (len(off) - 1))
        assert np.array_equal(u[0], got[0]) and np.array_equal(u[1], got[1])
        ratio, worst, bad = marg_gate(got, t, s, r, off)
        gated.append((label, *_worst(worst)))
        assert not bad, (label, bad)
    w = max(gated, key=lambda g: g[1])
    print(f"edges: {len(gated)} systems, worst ratio {w[1]:.3f} ({w[0]}, {w[2]})")


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_5000_state_chain_against_extended_oracle(cuda, oracles, model):
    """The 5 000-state chain of test_chain_marginals.test_scale (undamped, a 1e8 prior on x_0, a position fix every 50 keyframes) in
    both models: chains_marginals bitwise chains_covariance of the system it assembles, gated per field against the oracle.  Its
    odd nodes read the level-(l+1) neighbour block on levels 1 .. 11."""
    from cpi_b200 import factor, preint, synth
    from test_state_priors import _fix, _sp_dev
    torch = cuda
    o64, old = oracles
    n = 5000
    rng = np.random.default_rng(1)
    Sm, L = synth.make_windows(n - 1, 20, rate=200.0, first_window=9000, special=False)
    rec = preint.preintegrate_host(model, Sm, L, synth.SIGMAS, 0, ns=20)
    truth = synth.make_states(rec, L, model, perturb=False)
    idx = np.arange(50, n, 50, dtype=np.int64)
    fx = [_fix(rng, truth[k]) for k in idx]
    sp = _sp_dev(torch, idx, np.stack([vec(w[None])[0] for w, _ in fx]), None, None, np.stack([xb for _, xb in fx]))
    info0 = torch.eye(15, dtype=torch.float64, device="cuda").reshape(1, 225) * 1e8
    dX, dR, dL = _dev(torch, truth), _dev(torch, rec), _dev(torch, L)
    Dd, Ed = tcm._system(torch, model, dX, dR, dL, n, (info0, None, None, None), sp)
    cv, cr = factor.chains_marginals(model, dX, dR, dL, n, prior=(info0, None, None, None), state_priors=sp, cross=True)
    cv2, cr2 = factor.chains_covariance(Dd, Ed, n, cross=True)
    assert torch.equal(cv, cv2) and torch.equal(cr, cr2)
    D, E = Dd.cpu().numpy(), Ed.cpu().numpy()
    off = np.array([0, n])
    t, s, r = marg_truths(o64, old, ("5000", model), off, D, E)
    assert np.all(np.isfinite(t[0])) and np.all(np.isfinite(t[1]))
    got = (cv.cpu().numpy(), cr.cpu().numpy())
    ratio, worst, bad = marg_gate(got, t, s, r, off)
    worst_line(f"marginals, 5 000-state chain, model {model}", worst)
    assert not bad, bad


WEAK = np.diag(np.repeat([1e4, 1e6, 1e2, 1e4, 1e2], 3)) * 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_tiled_batch_against_extended_oracle(cuda, oracles, model):
    """chains_marginals with cross on the tiled batch of chain_scale.lm_batch (about 300 000 states, 14 000 chains; Gaussian, Huber
    and Cauchy state priors; copies beyond every k_chain_ids pass boundary of 132 and 114 SMs and of this device).  The chains with a
    zero chain prior get a weak one (1e-6 of make_problem's), so that every class's system has a positive long-double
    factorisation, which is asserted.

    The selected inversion runs the solve's forward phase and walks the same levels back, so bcr_pattern's argument holds unchanged:
    a chain's arithmetic depends on its offset only mod M(L), which divides TILE, and every copy of a class must be bitwise its first
    copy.  Each class is gated per field against the oracle on its system placed at offset TILE + its residue behind single-state
    pad chains with D = I, where the oracle's route in the kernels' order walks the device's levels.  With the NaN fixes, NaN falls in
    exactly the NaN copies and every other chain is bitwise its class."""
    from cpi_b200 import factor
    from test_chain_scale import _lm_tiled, _same_per_class, _sms
    from test_state_priors import _sp_dev
    torch = cuda
    o64, old = oracles
    sms = _sms(torch)
    t0 = time.time()
    (_, _, _, _, _, _, _, _), (src, cls, nan_at), t = _lm_tiled(o64, model, sms)
    toffs = t["offs"]
    C, N = len(src), int(toffs[-1])
    for s_ in tuple(dict.fromkeys(SMS + (sms,))):
        assert any(toffs[i] > chain_ids_pass(s_, N) for i in range(C)), s_
    PI = t["prior"][0].copy()
    zero = ~PI.any(axis=1)
    PI[zero] = vec(WEAK[None])[0]
    d = lambda a: _dev(torch, a)
    args = (d(t["X"]), d(t["rec"]), d(t["L"]), d(toffs))
    pr = (d(PI),) + tuple(d(a) for a in t["prior"][1:])
    loss = tuple(d(a) for a in t["loss"])
    cv, cr = factor.chains_marginals(model, *args, prior=pr, state_priors=_sp_dev(torch, *t["sp_clean"]), state_prior_loss=loss, cross=True)
    Dd, Ed = tcm._system(torch, model, *args, pr, _sp_dev(torch, *t["sp_clean"]), loss)
    cov, cross = cv.cpu().numpy(), cr.cpu().numpy()
    assert np.all(np.isfinite(cov)) and np.all(np.isfinite(cross)) and _symmetric(cov)
    seg = lambda A: (lambda i: A[toffs[i]:toffs[i + 1]])
    segx = lambda A: (lambda i: A[toffs[i] - i:toffs[i + 1] - i - 1])
    _same_per_class([seg(cov), segx(cross)], cls, set())
    # every class against the oracle, placed at TILE + its residue behind single-state chains with D = I
    first = {}
    for i, k in enumerate(cls):
        first.setdefault(int(k), i)
    eye = vec(np.eye(15)[None])[0]
    ed, e64 = {}, {}
    for k, i in first.items():
        lo, hi = int(toffs[i]), int(toffs[i + 1])
        n, P = hi - lo, TILE + lo % TILE
        D = np.concatenate([np.repeat(eye[None], P, axis=0), Dd[lo:hi].cpu().numpy()])
        E = np.concatenate([np.zeros((P, 225)), Ed[lo:hi - 1].cpu().numpy()])
        off = np.r_[np.arange(P + 1), P + n].astype(np.int64)
        tt, ss, rr = (o.chain_marginals(D, E, order, chain_offsets=off, nthreads=1)
                      for o, order in ((old, 0), (o64, 0), (o64, 1)))
        assert np.all(np.isfinite(tt[0])) and np.all(np.isfinite(tt[1])), ("no positive long-double factorisation", k, n)
        one = np.array([0, n])
        pick = lambda x: (x[0][P:], x[1])
        e_d = marg_errors((cov[lo:hi], cross[lo - i:hi - i - 1]), pick(tt), one)
        es, er = marg_errors(pick(ss), pick(tt), one), marg_errors(pick(rr), pick(tt), one)
        for f in e_d:
            ed.setdefault(f, []).append(e_d[f][0])
            e64.setdefault(f, []).append(max(es[f][0], er[f][0]))
    ratio, worst, bad = gate_errors({f: np.array(v) for f, v in ed.items()}, {f: np.array(v) for f, v in e64.items()}, K, FLOOR)
    worst_line(f"marginals, tiled batch, model {model}: {C} chains, {N} states, {len(first)} classes", worst)
    assert not bad, bad
    # the NaN fixes: NaN in exactly the NaN copies, every other chain bitwise its class (the clean run)
    bv, bc = (a.cpu().numpy() for a in factor.chains_marginals(model, *args, prior=pr, state_priors=_sp_dev(torch, *t["sp"]),
                                                                 state_prior_loss=loss, cross=True))
    nan_chain = np.add.reduceat(np.isnan(bv).any(axis=1), toffs[:-1]) > 0
    assert np.array_equal(np.flatnonzero(nan_chain), sorted(nan_at))
    keep = np.repeat(~nan_chain, np.diff(toffs))
    keepx = np.repeat(~nan_chain, np.diff(toffs) - 1)
    assert np.array_equal(bv[keep], cov[keep]) and np.array_equal(bc[keepx], cross[keepx])
    print(f"tiled batch, model {model}: {len(nan_at)} NaN copies alone non-finite; {time.time() - t0:.1f} s")
