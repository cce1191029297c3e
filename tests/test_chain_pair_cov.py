"""Any blocks Sigma_ij of the inverse of many chains by a walk up the block-cyclic-reduction levels (cpi_imu_chains_pair_covariance,
factor.chains_pair_covariance / chains_pair_marginals; DESIGN.md section 3q).

GTSAM is not in the reference tree, so parity with its jointMarginalCovariance is UNPINNED.  The truths are pair_cov_ref.walk (the
walk in numpy, pinned on the CPU against the dense inverse and test_chain_marginals.selinv_ref) and, on the GPU, the long-double
sequential block-Cholesky route of pair_cov_ref.sequential, chains_covariance, and the Monte-Carlo spread of the smoother's relative
error against the truth.

The gate is the rule of test_marginals_precision.marg_gate on pairs: per chain and per 3x3 component pair of (theta, b_g, v, b_a, p)^2,
the largest |dSigma_ij| / sqrt(T_ii T_jj) over the chain's pairs (T the truth's diagonal blocks) within K = 8 times e_64, the larger
error of the fp64 routes (the sequential route, the walk in the kernel's level order and, on the GPU on chains of at most 40 states,
the plain fp64 dense inverse), floor 1e-15.  The stress batch pools the chains of one length into one group."""
import ctypes

import numpy as np
import pytest

import pair_cov_ref as pcr
import test_chain_marginals as tcm
from parity import gate_errors
from test_chain_precision import batch, oracles  # noqa: F401
from test_marginalize import mat, vec
from test_marginals_precision import COMP, systems
from test_streams import B, Inputs, _F, _kw, _lm_args, _system, cycles_per_ms  # noqa: F401
import test_streams as ts

K, FLOOR = 8.0, 1e-15
LD = np.longdouble
P = lambda a: ctypes.c_void_p(a.ctypes.data)


# ---------------------------------------------------------------------------------------------- the error measure and gate

def pair_errors(got, truth, dii, djj, group):
    """dict "I.J" -> [G]: per group the largest |got - truth|_ab / sqrt(T_aa T_bb) of the 3x3 block (I, J) over the group's pairs.
    got, truth [q,15,15]; dii, djj [q,15] the truth's diagonals of Sigma_ii and Sigma_jj; group [q] in 0 .. G-1.  NaN in got: NaN."""
    e = np.abs(got.astype(np.float64) - truth.astype(np.float64)) / np.sqrt(dii[:, :, None] * djj[:, None, :])
    e = e.reshape(-1, 5, 3, 5, 3).max(axis=(2, 4))
    G = int(group.max()) + 1
    out = {}
    for I in range(5):
        for J in range(5):
            v = np.full(G, 0.0)
            np.maximum.at(v, group, e[:, I, J])
            v[np.bincount(group, weights=np.isnan(e[:, I, J]), minlength=G) > 0] = np.nan
            out[f"{COMP[I]}.{COMP[J]}"] = v
    return out


def pair_gate(got, truth, routes, dii, djj, group):
    """(ratio, worst, failures) of got against the truth; e_64 the larger error of the fp64 routes."""
    ed = pair_errors(got, truth, dii, djj, group)
    es = [pair_errors(r, truth, dii, djj, group) for r in routes]
    return gate_errors(ed, {k: np.maximum.reduce([e[k] for e in es]) for k in ed}, K, FLOOR)


def chain_truths(D, E, off, pairs, ld=True):
    """The sequential route's Sigma_ij [q,15,15] and the diagonals of Sigma_ii, Sigma_jj for global pairs [q,2] of the layout off
    (pairs within one chain), in long double (ld) or fp64."""
    Dm, Em = mat(D).astype(LD if ld else np.float64), mat(E).astype(LD if ld else np.float64)
    chain = np.searchsorted(off, pairs[:, 0], side="right") - 1
    out = np.zeros((len(pairs), 15, 15), dtype=Dm.dtype)
    dii, djj = np.zeros((len(pairs), 15)), np.zeros((len(pairs), 15))
    for c in np.unique(chain):
        lo, hi = int(off[c]), int(off[c + 1])
        G, Skk = pcr.sequential(Dm[lo:hi], Em[lo:hi - 1])
        sel = np.flatnonzero(chain == c)
        loc = pairs[sel] - lo
        out[sel] = pcr.sequential_pairs(G, Skk, loc)
        d = np.einsum("kii->ki", Skk).astype(np.float64)
        dii[sel], djj[sel] = d[loc[:, 0]], d[loc[:, 1]]
    return out, dii, djj, chain


def walk_pairs(fw, pairs, drop=None):
    return np.array([pcr.walk(fw, int(i), int(j), drop) for i, j in pairs]).reshape(-1, 15, 15)


def all_pairs(off, max_len=None):
    """Every pair (i, j) (both orders, i = j included) within every chain of at most max_len states."""
    out = []
    for c in range(len(off) - 1):
        lo, hi = int(off[c]), int(off[c + 1])
        if max_len is None or hi - lo <= max_len:
            k = np.arange(lo, hi)
            out.append(np.stack(np.meshgrid(k, k, indexing="ij"), -1).reshape(-1, 2))
    return np.concatenate(out).astype(np.int64)


def cid_of(off):
    return np.repeat(np.arange(len(off) - 1), np.diff(off))


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", [0, 1])
def test_walk_is_the_dense_inverse(seed):
    """On random SPD systems of ragged chains (1 .. 70 states, chain boundaries at odd and even states) the walk gives every block
    of every chain's dense inverse (i = j, i < j, i > j) to 1e-12 in the units of its diagonal, exact 0 across chains and the same bits
    with NaN couplings between chains; neither bracket ever holds more than two nodes (asserted inside walk).  In long double it
    gives the same blocks to 1e-12 too, and the transposed pair the transposed block."""
    rng = np.random.default_rng(seed)
    sizes = [1, 2, 3, 4, 5, 7, 8, 9, 1, 1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 70, 1, 13]
    sizes = sizes if seed == 0 else list(rng.permutation(sizes))
    D, E, offs, cid = tcm.random_system(rng, sizes)
    assert len(set(offs[1:-1] % 2)) == 2
    fw = pcr.forward(D, E, cid)
    worst = 0.0
    for c in range(len(sizes)):
        lo, hi = int(offs[c]), int(offs[c + 1])
        T = np.linalg.inv(tcm.dense(D, E, lo, hi))
        _, err = tcm.scaled(None, T)
        ks = range(hi - lo) if hi - lo <= 33 else sorted({0, 1, 2, 17, 31, 32, 33, hi - lo - 2, hi - lo - 1})
        for a in ks:
            for b in ks:
                worst = max(worst, err(pcr.walk(fw, lo + a, lo + b), a, b))
    print(f"seed {seed}: worst block error {worst:.1e} in units of the diagonal")
    assert worst <= 1e-12
    # across chains: exact 0; NaN couplings between chains are never read
    for a, b in ((0, int(offs[5])), (int(offs[-2]), int(offs[3]) + 1)):
        assert not pcr.walk(fw, a, b).any()
    Ep = E.copy()
    Ep[offs[1:-1] - 1] = np.nan
    fwp = pcr.forward(D, Ep, cid)
    pairs = [(int(offs[13]) + 3, int(offs[13]) + 29), (int(offs[19]) + 60, int(offs[19])), (5, 5)]
    for i, j in pairs:
        assert np.array_equal(pcr.walk(fwp, i, j), pcr.walk(fw, i, j))
    fwl = pcr.forward(D.astype(LD), E.astype(LD), cid)
    c = sizes.index(70)
    lo = int(offs[c])
    T = np.linalg.inv(tcm.dense(D, E, lo, lo + 70))
    _, err = tcm.scaled(None, T)
    for a, b in ((0, 69), (69, 0), (5, 40), (33, 33)):
        X = pcr.walk(fwl, lo + a, lo + b)
        assert X.dtype == LD and err(X.astype(np.float64), a, b) <= 1e-12
        assert np.array_equal(pcr.walk(fwl, lo + b, lo + a), X.T) or a == b


def test_walk_is_selinv_ref():
    """(k, k) and (k, k+1) of the walk are test_chain_marginals.selinv_ref's cov and neighbour blocks to rounding (1e-13 in the
    units of the diagonal)."""
    rng = np.random.default_rng(7)
    sizes = [1, 2, 3, 9, 16, 17, 33, 1, 40]
    D, E, offs, cid = tcm.random_system(rng, sizes)
    cov, nb = tcm.selinv_ref(D, E, cid)
    fw = pcr.forward(D, E, cid)
    d = 1.0 / np.sqrt(np.einsum("nii->ni", cov))
    worst = 0.0
    for k in range(len(D)):
        worst = max(worst, np.max(np.abs(pcr.walk(fw, k, k) - cov[k]) * d[k][:, None] * d[k][None, :]))
        if k + 1 < len(D) and cid[k] == cid[k + 1]:
            worst = max(worst, np.max(np.abs(pcr.walk(fw, k, k + 1) - nb[k]) * d[k][:, None] * d[k + 1][None, :]))
    print(f"walk vs selinv_ref: {worst:.1e}")
    assert worst <= 1e-13


def test_argument_validation_without_gpu():
    import torch
    from cpi_b200 import capi, factor
    lib = capi.load()
    buf, b2, b3, b4 = (np.zeros(8 * 225) for _ in range(4))
    p, q, r, o = P(buf), P(b2), P(b3), P(b4)
    # (n_chains, offs, uniform, n_states, D, E, n_pairs, pair_i, pair_j, out, workspace, stream)
    pc = lambda *a: lib.cpi_imu_chains_pair_covariance(*a, None)
    assert pc(-1, None, 2, 4, p, p, 1, q, q, o, r) == -1 and b"negative" in lib.cpi_last_error()
    assert pc(2, None, 0, 4, p, p, 1, q, q, o, r) == -1 and b"chain_uniform" in lib.cpi_last_error()
    assert pc(2, None, 2, 5, p, p, 1, q, q, o, r) == -1 and b"n_states" in lib.cpi_last_error()
    assert pc(2, None, 2, 4, p, p, -1, q, q, o, r) == -1 and b"n_pairs" in lib.cpi_last_error()
    for k in (0, 1, 3, 4, 5, 6):                                   # D, E, pair_i, pair_j, out, workspace
        a = [p, p, 1, q, q, o, r]; a[k] = None
        assert pc(2, None, 2, 4, *a) == -1 and b"null" in lib.cpi_last_error(), k
    for k in (0, 1, 3, 4, 6):                                      # out equal to D, E, pair_i, pair_j or the workspace
        a = [p, P(b2), 1, P(b3), q, o, P(np.zeros(8))]; a[5] = a[k]
        assert pc(2, None, 2, 4, *a) == -1 and b"overlap" in lib.cpi_last_error(), k
    assert pc(0, None, 1, 0, None, None, 1, q, q, o, r) == -1 and b"state" in lib.cpi_last_error()
    assert pc(2, None, 2, 4, None, None, 0, None, None, None, None) == 0
    assert pc(0, None, 1, 0, *[None] * 2, 0, *[None] * 4) == 0
    ws = lib.cpi_imu_chains_pair_covariance_workspace
    assert ws(2, 1) < 0 and ws(-1, 4) < 0 and ws(2, -1) < 0
    for n in (1, 2, 3, 64, 65, 1000):                              # the selected inversion's workspace and Sigma_root
        assert ws(1, n) == lib.cpi_imu_chains_marginals_workspace(1, n) + 225 * 8, n
    # the bindings, before the device is touched
    f64 = dict(dtype=torch.float64)
    D, E = torch.zeros((4, 225), **f64), torch.zeros((3, 225), **f64)
    pr = np.array([[0, 1], [3, 3]])
    cases = [((D.float(), E, 2, pr), "float64"), ((D[:, :224], E, 2, pr), "225"), ((D, E, 3, pr), "match"),
             ((D, E, torch.tensor([0, 1, 2, 3, 4, 4]), pr), "more chains"), ((D, E, 2, np.array([[0, 4]])), "index"),
             ((D, E, 2, np.array([[-1, 0]])), "index"), ((D, E, 2, np.array([0, 1])), r"\[q,2\]"), ((D, E, 2, pr.astype(float)), "integer"),
             ((D, E, 2, torch.tensor([[0, 1]])), "CUDA"), ((D, E, 2, pr), "CUDA")]
    for args, msg in cases:
        with pytest.raises(ValueError, match=msg):
            factor.chains_pair_covariance(*args)
    short = torch.zeros(int(ws(2, 4)) // 8 - 1, **f64)
    with pytest.raises(ValueError, match="cpi_imu_chains_pair_covariance_workspace"):
        factor.chains_pair_covariance(D, E, 2, pr, workspace=short)
    X, rec, lin = torch.zeros((6, 16), **f64), torch.zeros((4, 290), **f64), torch.zeros((4, 13), **f64)
    with pytest.raises(ValueError, match="record"):
        factor.chains_pair_marginals(1, X, rec[:3], lin, 3, pr)
    with pytest.raises(ValueError, match="CUDA"):
        factor.chains_pair_marginals(1, X, rec, lin, 3, pr)


def test_gate_fails_injected_errors():
    """On a random ragged system the gate passes the two fp64 routes and fails four injected errors: Sigma_ij transposed, Sigma_ij
    zeroed for |i - j| >= 2, one Sigma_kk rounded to fp32, and a single K+ dropped at one level."""
    rng = np.random.default_rng(11)
    sizes = [3, 9, 17, 33, 40, 1, 24]
    D, E, offs, cid = tcm.random_system(rng, sizes)
    pairs = all_pairs(offs)
    t, dii, djj, grp = chain_truths(vec(D), vec(E), offs, pairs)
    s, _, _, _ = chain_truths(vec(D), vec(E), offs, pairs, ld=False)
    fw = pcr.forward(D, E, cid)
    w = walk_pairs(fw, pairs)
    routes = (s, w)
    for x in routes:
        assert not pair_gate(x, t, routes, dii, djj, grp)[2]
    far = np.abs(pairs[:, 0] - pairs[:, 1]) >= 2
    bad = [("transposed", w.transpose(0, 2, 1)), ("zero far", np.where(far[:, None, None], 0.0, w))]
    f32 = w.copy()
    k = int(np.flatnonzero((pairs[:, 0] == offs[4] + 3) & (pairs[:, 1] == offs[4] + 3))[0])
    f32[k] = f32[k].astype(np.float32)
    bad.append(("fp32 block", f32))
    x0 = int(offs[3]) + 10                                         # one odd node of level 0 in the 33-state chain
    assert x0 % 2 == 1
    bad.append(("K+ dropped", walk_pairs(fw, pairs, drop=lambda lv, x, right: lv == 0 and x == x0 and right)))
    for name, got in bad:
        assert pair_gate(got, t, routes, dii, djj, grp)[2], name


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------

def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _pc(torch, D, E, off, pairs):
    from cpi_b200 import factor
    o = _dev(torch, off) if isinstance(off, np.ndarray) else int(off)
    return mat(factor.chains_pair_covariance(_dev(torch, D), _dev(torch, np.asarray(E).reshape(-1, 225)), o, pairs).cpu().numpy())


def _gate_routes(D, E, off, pairs, got, label, by_length=False):
    """got against the long-double sequential route; e_64 from the fp64 routes: the sequential route, the walk in the kernel's
    levels and, on chains of at most 40 states, the plain fp64 dense inverse.  Groups: chains, or (by_length) the chains of one
    length pooled."""
    t, dii, djj, grp = chain_truths(D, E, off, pairs)
    s, _, _, _ = chain_truths(D, E, off, pairs, ld=False)
    w = walk_pairs(pcr.forward(mat(D), mat(E), cid_of(off)), pairs)
    dn = s.copy()
    for c in np.unique(grp):
        lo, hi = int(off[c]), int(off[c + 1])
        if hi - lo <= 40:
            T = np.linalg.inv(tcm.dense(mat(D), mat(E), lo, hi))
            for k in np.flatnonzero(grp == c):
                a, b = pairs[k] - lo
                dn[k] = T[15 * a:15 * a + 15, 15 * b:15 * b + 15]
    if by_length:
        grp = np.unique(np.diff(off)[grp], return_inverse=True)[1]
    ratio, worst, bad = pair_gate(got, t, (s, w, dn), dii, djj, grp)
    k = max(worst, key=lambda f: worst[f]["ratio"])
    print(f"{label}: {len(pairs)} pairs, worst ratio {worst[k]['ratio']:.3f} ({k})")
    assert not bad, (label, bad)
    return worst[k]["ratio"]


@pytest.mark.gpu
def test_stress_batch_against_extended_oracle(cuda, oracles):
    """Every damping of the ragged stress layout (chains of 1 .. 9 states, a boundary on every residue mod 64) and the main layout's
    first system: every pair of the chains of at most 40 states and 400 sampled pairs of the longer ones, per field against the
    long-double sequential route, the chains of one length pooled into one group (the ragged layout's 200 short chains would
    otherwise make 200 groups of a few pairs each, whose e_64 can fall to a few ulps by chance).  Sigma_ii exactly symmetric."""
    torch = cuda
    o64, _ = oracles
    b = batch(o64)
    rng = np.random.default_rng(5)
    worst = []
    for which, sel in (("ragged", slice(None)), ("main", slice(0, 1))):
        off = b[which]["offsets"]
        pairs = all_pairs(off, 40)
        long_ = [c for c in range(len(off) - 1) if off[c + 1] - off[c] > 40]
        if long_:
            c = rng.choice(long_, 400)
            lo, n = off[c], off[c + 1] - off[c]
            pairs = np.concatenate([pairs, np.stack([lo + rng.integers(0, n), lo + rng.integers(0, n)], -1)])
        for name, D, E in systems(b, which)[sel]:
            got = _pc(torch, D, E, off, pairs)
            same = pairs[:, 0] == pairs[:, 1]
            assert np.array_equal(got[same], got[same].transpose(0, 2, 1))
            worst.append(_gate_routes(D, E, off, pairs, got, f"pairs {which} {name}", by_length=True))
    print(f"stress batch: worst ratio {max(worst):.3f}")


def _scale_problem(torch, model=1):
    """The 10 000 x 30 batch and the 5 000-state chain of test_chain_marginals.test_scale: (D, E) of each, on the device."""
    from cpi_b200 import factor, preint, synth
    from test_state_priors import _fix, _sp_dev
    C, S = 10_000, 30
    Sm, L = synth.make_windows(C * (S - 1), 20, rate=200.0, first_window=0, special=False)
    rec = preint.preintegrate(model, _dev(torch, Sm), _dev(torch, L), synth.SIGMAS, 0, ns=20)
    dL = _dev(torch, L)
    X = torch.empty((C, S, 16), dtype=torch.float64, device="cuda")
    X[:, 0] = 0.0; X[:, 0, 3] = 1.0; X[:, 0, 4:7] = dL.view(C, S - 1, 13)[:, 0, 0:3]; X[:, 0, 10:13] = dL.view(C, S - 1, 13)[:, 0, 3:6]
    for k in range(S - 1):
        X[:, k + 1] = factor.predict_state(model, X[:, k].contiguous(), rec.view(C, S - 1, -1)[:, k].contiguous(),
                                           dL.view(C, S - 1, 13)[:, k].contiguous())
    X = X.reshape(C * S, 16)
    info0 = torch.eye(15, dtype=torch.float64, device="cuda").reshape(1, 225).repeat(C, 1) * 1e8
    tiled = tcm._system(torch, model, X, rec, dL, S, (info0, None, None, None))
    n = 5000
    rng = np.random.default_rng(1)
    Sm, L = synth.make_windows(n - 1, 20, rate=200.0, first_window=9000, special=False)
    rec = preint.preintegrate_host(model, Sm, L, synth.SIGMAS, 0, ns=20)
    truth = synth.make_states(rec, L, model, perturb=False)
    idx = np.arange(50, n, 50, dtype=np.int64)
    fx = [_fix(rng, truth[k]) for k in idx]
    sp = _sp_dev(torch, idx, np.stack([vec(w[None])[0] for w, _ in fx]), None, None, np.stack([xb for _, xb in fx]))
    long_ = tcm._system(torch, model, _dev(torch, truth), _dev(torch, rec), _dev(torch, L), n, (info0[:1], None, None, None), sp)
    return tiled, long_


@pytest.mark.gpu
def test_production_scale_against_extended_oracle(cuda):
    """The 10 000 x 30 batch with four pairs per chain (spans 1, 2, 7 and 29: 40 000 pairs, many grid-stride passes) and the 5 000-state
    chain with pairs spanning 1, 2, 7, 29 and 4 999 keyframes: 60 sampled chains and every long pair against the long-double
    sequential route; every block finite; each pair's bits the same in a call of its own."""
    from cpi_b200 import factor
    torch = cuda
    (Dt, Et), (Dl, El) = _scale_problem(torch)
    C, S = 10_000, 30
    first = np.arange(C) * S
    spans = [(3, 4), (10, 12), (20, 27), (0, 29)]
    pairs = np.concatenate([np.stack([first + a, first + b], -1) for a, b in spans])
    pairs[1::2] = pairs[1::2, ::-1]
    got = mat(factor.chains_pair_covariance(Dt, Et, S, _dev(torch, pairs)).cpu().numpy())
    assert np.all(np.isfinite(got))
    rng = np.random.default_rng(3)
    c0 = 4321                                                      # 60 consecutive chains, gated as a layout of their own
    pick = np.flatnonzero((pairs[:, 0] // S >= c0) & (pairs[:, 0] // S < c0 + 60))
    D, E = Dt.cpu().numpy()[c0 * S:(c0 + 60) * S], Et.cpu().numpy()[c0 * S:(c0 + 60) * S - 1]
    _gate_routes(D, E, np.arange(61, dtype=np.int64) * S, pairs[pick] - c0 * S, got[pick], "10 000 x 30, 60 chains gated")
    one = mat(factor.chains_pair_covariance(Dt, Et, S, _dev(torch, pairs[pick[:7]])).cpu().numpy())
    assert np.array_equal(one, got[pick[:7]])
    n = 5000
    lp = np.array([[0, 1], [4998, 4999], [100, 102], [2501, 2499], [777, 784], [4000, 4029], [29, 0], [0, 4999], [4999, 0], [1234, 1234]])
    lp = np.concatenate([lp, rng.integers(0, n, (20, 2))])
    got = _pc(torch, Dl.cpu().numpy(), El.cpu().numpy(), np.array([0, n]), lp)
    assert np.all(np.isfinite(got))
    _gate_routes(Dl.cpu().numpy(), El.cpu().numpy(), np.array([0, n]), lp, got, "5 000-state chain")


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_agrees_with_chains_covariance(cuda, oracle, model):
    """Ragged chains with a chain prior and state priors: chains_pair_marginals is chains_pair_covariance of the system it assembles
    bit for bit; its (k, k) and (k, k+1) lie within the gate of test_chain_marginals._gate_chains of the refined dense inverse, as
    chains_covariance's cov and cross do, and (k, k) is exactly symmetric."""
    from cpi_b200 import factor
    from test_chains_lm import dev_prior, make_problem
    from test_state_priors import _dev as sdev, _meas_priors, _sp_dev
    torch = cuda
    sizes = [1, 2, 3, 4, 5, 8, 9, 1, 15, 16, 17, 31, 32, 33]
    X, rec, L, offs, pri, _ = make_problem(oracle, model, sizes, 31 + model, with_prior=True)
    sp = _sp_dev(torch, *_meas_priors(oracle, np.random.default_rng(model), X, offs, 4, "mixed"))
    dX, dR, dL, d_offs = (sdev(torch, a) for a in (X, rec, L, offs))
    pr = dev_prior(torch, pri)
    D, E = tcm._system(torch, model, dX, dR, dL, d_offs, pr, sp)
    N, C = len(X), len(sizes)
    k = np.arange(N)
    nb = k[:-1][cid_of(offs)[:-1] == cid_of(offs)[1:]]
    pairs = np.concatenate([np.stack([k, k], -1), np.stack([nb, nb + 1], -1)])
    got = factor.chains_pair_marginals(model, dX, dR, dL, d_offs, _dev(torch, pairs), prior=pr, state_priors=sp)
    assert torch.equal(got, factor.chains_pair_covariance(D, E, d_offs, pairs))
    cov, cr = factor.chains_covariance(D, E, d_offs, cross=True)
    g = mat(got.cpu().numpy())
    assert np.array_equal(g[:N], g[:N].transpose(0, 2, 1))        # (k, k) exactly symmetric
    tcm._gate_chains(D, E, offs, got[:N].contiguous(), got[N:].contiguous(), f"pair route, model {model}")
    tcm._gate_chains(D, E, offs, cov, cr, f"selected inversion, model {model}")
    # the two routes against each other, in the units of the diagonal, within section 3j's gate: 50x the plain fp64 dense inverse's
    # distance to the refined truth (floor 1e-13)
    Dm, Em, cv, cx = mat(D.cpu().numpy()), mat(E.cpu().numpy()), mat(cov.cpu().numpy()), mat(cr.cpu().numpy())
    d = 1.0 / np.sqrt(np.einsum("kii->ki", cv))
    diff = max(float(np.max(np.abs(g[:N] - cv) * d[:, :, None] * d[:, None, :])),
               float(np.max(np.abs(g[N:] - cx) * d[nb][:, :, None] * d[nb + 1][:, None, :])))
    ep = 0.0
    for c in range(C):
        lo, hi = int(offs[c]), int(offs[c + 1])
        T, P64 = tcm.inv_truth(tcm.dense(Dm, Em, lo, hi))
        _, err = tcm.scaled(None, T)
        ep = max([ep] + [err(P64[15 * a:15 * a + 15, 15 * b:15 * b + 15], a, b) for a in range(hi - lo) for b in range(a, min(a + 2, hi - lo))])
    print(f"model {model}: pair route vs chains_covariance {diff:.1e} of the diagonal, gate {50 * max(ep, 1e-13):.1e}")
    assert diff <= 50 * max(ep, 1e-13), (diff, ep)


@pytest.mark.gpu
def test_isolation_and_determinism(cuda, oracle):
    """Ten chains: a chain made indefinite gets NaN in its own pairs only, every other pair is bitwise the clean run; pairs across
    chains are exact 0; indices outside [0, N) give NaN blocks; a pair's bits do not depend on the other pairs of the call or their
    order; two runs are bitwise equal."""
    from cpi_b200 import factor
    torch = cuda
    rng = np.random.default_rng(9)
    sizes = [5, 9, 12, 7, 16, 3, 8, 11, 6, 10]
    D, E, offs, cid = tcm.random_system(rng, sizes)
    D, E = vec(D), vec(E)
    N = len(D)
    pairs = np.concatenate([all_pairs(offs), rng.integers(0, N, (500, 2))])
    run = lambda Dx=D, p=pairs: _pc(torch, Dx, E, offs, p)
    clean = run()
    assert np.array_equal(run(), clean) and np.all(np.isfinite(clean))
    cross = cid[pairs[:, 0]] != cid[pairs[:, 1]]
    assert cross.sum() > 100 and not clean[cross].any()
    for bad in (3, 6):
        Db = D.copy()
        Db[int(offs[bad]) + 1] *= -1
        got = run(Db)
        mine = (cid[pairs[:, 0]] == bad) & (cid[pairs[:, 1]] == bad)
        assert np.isnan(got[mine]).any(axis=(1, 2)).all()
        assert np.array_equal(got[~mine], clean[~mine])
    perm = rng.permutation(len(pairs))[: len(pairs) // 3]
    assert np.array_equal(run(p=pairs[perm]), clean[perm])
    oob = np.array([[-1, 0], [0, N], [N + 5, -7], [3, 3]], dtype=np.int64)
    got = mat(factor.chains_pair_covariance(_dev(torch, D), _dev(torch, E), _dev(torch, offs), _dev(torch, oob)).cpu().numpy())
    assert np.isnan(got[:3]).all() and np.array_equal(got[3], clean[np.flatnonzero((pairs == [3, 3]).all(1))[0]])


# ---- the stream contract (the procedure of test_streams.test_stream_contract)
def _torch():
    import torch
    return torch


PAIRS_R = np.array([[0, 3], [3, 0], [4, 4], [5, 10], [0, 5], [2, 2], [10, 6]], dtype=np.int64)
CASES = {
    "chains_pair_covariance-offsets-noncontig": (
        lambda B, I: dict(sys=I.vs(_system(B, B["offs"])[:2]), o=I.v(B["offs"]), p=I.v(_dev(_torch(), PAIRS_R))),
        lambda a, st: _F().chains_pair_covariance(*a["sys"], a["o"], a["p"], stream=st), False, True),
    "chains_pair_covariance-uniform-numpy-workspace": (
        lambda B, I: dict(sys=tuple(I.f(t) for t in _system(B, 3)[:2]),
                          ws=_torch().empty(1 << 16, dtype=_torch().float64, device="cuda")),
        lambda a, st: _F().chains_pair_covariance(*a["sys"], 3, np.array([[0, 2], [11, 9], [4, 4], [0, 11]]), workspace=a["ws"], stream=st),
        True, False),                                              # numpy pairs: a blocking upload, as retract's numpy path
    "chains_pair_marginals-offsets-priors-measurements": (
        lambda B, I: dict(_lm_args(B, I), p=I.v(_dev(_torch(), PAIRS_R))),
        lambda a, st: _F().chains_pair_marginals(ts.MODEL, a["X"], a["r"], a["l"], a["o"], a["p"], a["prior"], stream=st, **_kw(a)),
        True, True),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_stream_contract(cuda, B, cycles_per_ms, monkeypatch, name):
    monkeypatch.setitem(ts.CASES, name, CASES[name])
    ts.test_stream_contract(cuda, B, cycles_per_ms, monkeypatch, name)


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_monte_carlo_relative_error(cuda, oracle, model, monkeypatch):
    """The realisations of test_chain_marginals._smoother_monte_carlo (30 000: three batches of 10 000 chains of 10 keyframes, fixes
    on keyframes 3, 6, 9), with chains_pair_marginals at the same estimates: the relative error e_j - e_i (in the tangent space at
    the estimate) has covariance Sigma_ii + Sigma_jj - Sigma_ij - Sigma_ij^T, and its mean NEES lies in the two-sided 99.9 % chi^2_15
    band for (0, 9), (2, 7) and (4, 5).  With Sigma_ij set to 0 it leaves the band."""
    from scipy.stats import chi2
    from cpi_b200 import factor
    n, K, streams = 10_000, 10, (None, 1, 2)
    sel = [(0, 9), (2, 7), (4, 5)]
    seen = {}
    orig = factor.chains_marginals

    def spy(model_, X, rec, lin, S, **kw):
        seen["pc"] = factor.chains_pair_marginals(model_, X, rec, lin, S, pairs, prior=kw.get("prior"), state_priors=kw.get("state_priors"))
        return orig(model_, X, rec, lin, S, **kw)
    base = np.arange(n)[:, None] * K
    pairs = np.concatenate([np.concatenate([base + i, base + j], 1) for i, j in sel] +
                           [np.concatenate([base + i, base + i], 1) for i, _ in sel] +
                           [np.concatenate([base + j, base + j], 1) for _, j in sel]).astype(np.int64)
    monkeypatch.setattr(factor, "chains_marginals", spy)
    sums, sums0 = np.zeros(len(sel)), np.zeros(len(sel))
    for s in streams:
        err, _, _ = tcm._smoother_monte_carlo(cuda, oracle, model, n, K, 90 + model, noise=s)
        pc = mat(seen.pop("pc").cpu().numpy()).reshape(3, len(sel), n, 15, 15)
        for q, (i, j) in enumerate(sel):
            d = err[:, j] - err[:, i]
            Sij, Sii, Sjj = pc[0, q], pc[1, q], pc[2, q]
            for Cm, acc in ((Sii + Sjj - Sij - Sij.transpose(0, 2, 1), sums), (Sii + Sjj, sums0)):
                acc[q] += np.einsum("ni,ni->", d, np.linalg.solve(Cm, d[:, :, None])[:, :, 0])
    N = n * len(streams)
    lo, hi = chi2.ppf([0.0005, 0.9995], 15 * N) / N
    for q, (i, j) in enumerate(sel):
        print(f"model {model}, ({i}, {j}): mean relative NEES {sums[q] / N:.3f}, with Sigma_ij = 0 {sums0[q] / N:.3f} (band [{lo:.3f}, {hi:.3f}])")
    assert all(lo <= v / N <= hi for v in sums), sums / N
    assert all(not lo <= v / N <= hi for v in sums0), sums0 / N
