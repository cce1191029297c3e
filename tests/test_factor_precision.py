"""Precision of the factor, prediction, retraction and information-form kernels against an extended-precision truth.

Inputs: the factor stress batch of tests/factor_stress.py (records of every preintegration regime from the fp64 oracle, state
pairs in tagged regimes, shuffled / repeated / reversed indices) and its retraction batch.  Truths, all computed in long double:
  * K3/K4 evaluateError, k_predict, k_retract: oracle/liboracle_ld.so (factor_eval, predict_state, retract);
  * K7 cov_k1 = A Sigma_k A^T + B P_meas B^T: test_propagate's statement with the long-double oracle and np.longdouble products;
  * k_factor_hessian / k_factor_whiten: a vectorised np.longdouble Cholesky of P_meas and forward substitution (R_w, the upper
    Cholesky factor of P^-1 with positive diagonal, is unique, so the whitened blocks compare block by block).
e_64 is the same computation in fp64 (the fp64 oracle; for the information form the larger error of LAPACK and of the kernels'
operation order, see info_gate; K7's statement at the x_k1 the kernel predicted), and the gate is parity.conditioned_gate's rule
e_dev <= K max(e_64, floor), K = 8, floor = 1e-15, as in test_precision.py.  Fields: e per 3-block, every structurally non-zero 3x3
block of H1 / H2 (structural zeros must be exact zeros), predicted and retracted states per component group (q up to sign only
where the truth's |w| < 1e-12), and every 3x3 block / 3-block of G11, G12, G22, A1, A2, g1, g2, b and f.

A residual that is nearly zero is ill-conditioned relative to itself, so e and the two H1 blocks built from pa / pb are measured
relative to the size of the terms that cancel into them (e_theta: 2, the scale of 2 q_r; e_p: |p_K1| + |p_K| + |v_K| DT
(+ |g| DT^2 / 2) + |J_a dbg| + |H_a dba| + |alpha| (+ |O_a dtheta_k|), e_v alike); predicted / retracted v and p likewise.  The
information blocks are measured relative to |Y|^T |Y| and |R_w| |H| (info_errors), K7's cov_k1 blocks relative to
sqrt(|C_II| |C_JJ|), the scale of a covariance block.

P_meas of some gap windows is indefinite (RK4 truncation over 0.1-0.5 s steps, not rounding: both oracles agree), and the zero-step
record has P = 0.  There the unpivoted Cholesky of k_factor_hessian / k_factor_whiten meets a non-positive pivot: those factors
must give NaN f and b, and every other factor of the batch and of the same 4-warp CTA must pass the gate.

Constants calibrated on one H100 80GB HBM3 (700 W power limit); DESIGN.md section 5 lists the measured worst ratios."""
import os
import subprocess

import numpy as np
import pytest

import factor_stress as fs
from parity import gate_errors, scaled_errors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIGMAS = np.array([0.005, 4e-6, 0.01, 0.0002])
K, FLOOR = 8.0, 1e-15
H1_BLOCKS = ((0, 0), (2, 0), (4, 0), (0, 1), (1, 1), (2, 1), (4, 1), (2, 2), (4, 2), (2, 3), (3, 3), (4, 3), (4, 4))
H2_BLOCKS = ((0, 0), (1, 1), (2, 2), (3, 3), (4, 4))
B3 = [slice(3 * k, 3 * k + 3) for k in range(5)]
LD = np.longdouble


@pytest.fixture(scope="session")
def oracle_ld():
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("long double has no extended precision on this platform")
    from oracle import oracle as om
    if not os.path.exists(om.OracleLD.path):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "liboracle_ld.so"], check=True)
    return om.OracleLD()


def _threads():
    from cpi_b200.synth import usable_cpus
    return usable_cpus()


def mat(a):
    """[n, 225] column-major -> [n, 15, 15]"""
    return np.asarray(a).reshape(-1, 15, 15).transpose(0, 2, 1)


def flat(M):
    """[n, 15, 15] -> [n, 225] column-major"""
    return np.ascontiguousarray(np.asarray(M).transpose(0, 2, 1).reshape(-1, 225))


# ---------------------------------------------------------------------------------------------- error fields

def _norm(a):
    return np.linalg.norm(a, axis=-1)


def residual_scales(model, b):
    """Per factor, the size of the terms that cancel into each 3-block of e and into H1's (v, theta) / (p, theta) blocks."""
    X, r, l = b["states"], b["records"], b["lin"]
    xi, xj = X[b["idx_i"]], X[b["idx_j"]]
    dT = r[:, 19]; g = _norm(l[:, 10:13]) if model == 1 else 0.0
    dbg, dba = xi[:, 4:7] - l[:, 0:3], xi[:, 10:13] - l[:, 3:6]
    mv = lambda a, v: _norm(np.einsum("nij,nj->ni", fs.rec33(r, a), v))
    sv = _norm(xj[:, 7:10]) + _norm(xi[:, 7:10]) + g * dT
    sp = _norm(xj[:, 13:16]) + _norm(xi[:, 13:16]) + _norm(xi[:, 7:10]) * dT + 0.5 * g * dT * dT
    s = dict(e_th=np.full(len(r), 2.0), e_bg=_norm(xj[:, 4:7]) + _norm(xi[:, 4:7]), e_ba=_norm(xj[:, 10:13]) + _norm(xi[:, 10:13]),
             e_v=sv + mv(38, dbg) + mv(56, dba) + _norm(r[:, 16:19]), e_p=sp + mv(29, dbg) + mv(47, dba) + _norm(r[:, 13:16]),
             H1_20=np.sqrt(2) * sv, H1_40=np.sqrt(2) * sp)
    if model == 2:
        dth = 2 * fs.front(X, b["idx_i"], b["idx_j"], r, l)["q_kR"][:, 0:3]
        s["e_v"] = s["e_v"] + mv(299, dth); s["e_p"] = s["e_p"] + mv(290, dth)
        s["H1_20"] = s["H1_20"] + np.sqrt(3) * _norm(r[:, 299:308]); s["H1_40"] = s["H1_40"] + np.sqrt(3) * _norm(r[:, 290:299])
    return s


def factor_errors(got, truth, scales):
    """(e, H1, H2) against the truth: dict field -> [n]."""
    e, H1, H2 = got; te, tH1, tH2 = truth
    out = {}
    for k, name in enumerate(("e_th", "e_bg", "e_v", "e_ba", "e_p")):
        out[name] = scaled_errors(e[:, 3 * k:3 * k + 3], te[:, 3 * k:3 * k + 3], scales[name])
    for tag, G, T, blocks in (("H1", H1, tH1, H1_BLOCKS), ("H2", H2, tH2, H2_BLOCKS)):
        if G is None:
            continue
        Gm, Tm = mat(G), mat(T)
        for I, J in blocks:
            out[f"{tag}_{I}{J}"] = scaled_errors(Gm[:, B3[I], B3[J]], Tm[:, B3[I], B3[J]], scales.get(f"{tag}_{I}{J}"))
    return out


def structural_zeros_exact(H, blocks):
    Hm = mat(H)
    for I in range(5):
        for J in range(5):
            if (I, J) not in blocks:
                assert np.all(Hm[:, B3[I], B3[J]] == 0.0), f"structural zero block ({I},{J}) is not exactly zero"


def state_errors(got, truth, scale_v=None, scale_p=None, scale_b=None):
    """Per component group of [n,16] states: q (up to sign where the truth's |w| < 1e-12), bg, v, ba, p."""
    sf = np.abs(truth[:, 3]) < 1e-12
    out = dict(q=scaled_errors(got[:, 0:4], truth[:, 0:4], sign_free=sf))
    for name, a, s in (("bg", 4, scale_b), ("v", 7, scale_v), ("ba", 10, scale_b), ("p", 13, scale_p)):
        sc = s[name] if isinstance(s, dict) else s
        out[name] = scaled_errors(got[:, a:a + 3], truth[:, a:a + 3], sc)
    return out


def predict_scales(model, XK, rec, lin):
    g = _norm(lin[:, 10:13]) if model == 1 else 0.0
    dt = rec[:, 19]
    return (_norm(XK[:, 7:10]) + g * dt + _norm(rec[:, 16:19]),
            _norm(XK[:, 13:16]) + _norm(XK[:, 7:10]) * dt + 0.5 * g * dt * dt + _norm(rec[:, 13:16]))


def retract_scales(X, xi):
    return {name: _norm(X[:, a:a + 3]) + _norm(xi[:, a - 1:a + 2]) for name, a in (("bg", 4), ("v", 7), ("ba", 10), ("p", 13))}


def report(label, ratio, tags, regimes):
    rows = []
    for reg in regimes:
        sel = tags == reg
        if sel.any() and ratio:
            k = max(ratio, key=lambda f: np.max(ratio[f][sel]))
            rows.append(f"{reg}={np.max(ratio[k][sel]):.2f}({k})")
    print(label, " ".join(rows))


# ---------------------------------------------------------------------------------------------- long-double statements

def chol(P):
    """Vectorised unpivoted Cholesky of [n,15,15] (any float dtype): (L lower, ok [n]: every pivot > 0)."""
    A = np.array(P, copy=True)
    n = A.shape[0]
    L = np.zeros_like(A)
    ok = np.ones(n, dtype=bool)
    for k in range(15):
        d = A[:, k, k]
        ok &= d > 0
        s = np.sqrt(np.where(d > 0, d, 1))
        L[:, k, k] = s
        L[:, k + 1:, k] = A[:, k + 1:, k] / s[:, None]
        A[:, k + 1:, k + 1:] -= L[:, k + 1:, k, None] * L[:, None, k + 1:, k]
    return L, ok


def fwd(L, B):
    """L^-1 B for lower-triangular L [n,15,15] and B [n,15,m]."""
    Y = np.zeros(B.shape, dtype=L.dtype)
    for i in range(15):
        Y[:, i] = (B[:, i] - np.sum(L[:, i, :i, None] * Y[:, :i], axis=1)) / L[:, i, i, None]
    return Y


def info_stmt(rec, e, H1, H2, dtype):
    """The statement of k_factor_hessian and k_factor_whiten in ``dtype`` with the kernels' operation order (right-looking
    Cholesky, forward substitution, R_w from the Cholesky factor of L^-T L^-1): (dict of blocks, ok [n]: every pivot > 0)."""
    P = mat(rec[:, 65:290]).astype(dtype)
    L, ok = chol(P)
    L[~ok] = np.eye(15)
    B = np.concatenate([mat(H1), mat(H2), np.asarray(e)[:, :, None]], axis=2).astype(dtype)
    Y = fwd(L, B)
    G = Y.transpose(0, 2, 1) @ Y
    Linv = fwd(L, np.broadcast_to(np.eye(15, dtype=dtype), P.shape).copy())
    C, ok2 = chol(Linv.transpose(0, 2, 1) @ Linv)
    ok &= ok2
    A = C.transpose(0, 2, 1) @ B
    absY, absB = np.abs(Y), np.abs(B)
    size = _info_fields(absY.transpose(0, 2, 1) @ absY, np.abs(C.transpose(0, 2, 1)) @ absB)
    return _info_fields(G, A), ok, size


def info_64(rec, e, H1, H2, ok):
    """The same statement in fp64 through LAPACK, factor by factor (rows not ok: NaN)."""
    import scipy.linalg as sl
    n = len(rec)
    G = np.full((n, 31, 31), np.nan); A = np.full((n, 15, 31), np.nan)
    P = mat(rec[:, 65:290])
    B = np.concatenate([mat(H1), mat(H2), np.asarray(e)[:, :, None]], axis=2)
    for i in np.flatnonzero(ok):
        L = np.linalg.cholesky(P[i])
        Y = sl.solve_triangular(L, B[i], lower=True)
        G[i] = Y.T @ Y
        M = sl.solve_triangular(L, np.eye(15), lower=True)
        A[i] = np.linalg.cholesky(M.T @ M).T @ B[i]
    return _info_fields(G, A)


def _info_fields(G, A):
    return dict(G11=G[:, 0:15, 0:15], G12=G[:, 0:15, 15:30], G22=G[:, 15:30, 15:30], g1=-G[:, 0:15, 30], g2=-G[:, 15:30, 30],
                f=G[:, 30, 30], A1=A[:, :, 0:15], A2=A[:, :, 15:30], b=-A[:, :, 30])


def info_errors(got, truth, size, sel):
    """Every 3x3 block / 3-block, relative to the Frobenius norm of the same block of ``size`` (|Y|^T |Y| and |R_w| |H|: the
    terms summed into it, as for the residual)."""
    out = {}
    sz = lambda k, *ix: np.linalg.norm(size[k][sel][(slice(None),) + ix].astype(np.float64).reshape(int(sel.sum()), -1), axis=1)
    for k in ("G11", "G12", "G22", "A1", "A2"):
        for I in range(5):
            for J in range(5):
                out[f"{k}_{I}{J}"] = scaled_errors(got[k][sel][:, B3[I], B3[J]], truth[k][sel][:, B3[I], B3[J]], sz(k, B3[I], B3[J]))
    for k in ("g1", "g2", "b"):
        for I in range(5):
            out[f"{k}_{I}"] = scaled_errors(got[k][sel][:, B3[I]], truth[k][sel][:, B3[I]], sz(k, B3[I]))
    out["f"] = scaled_errors(got["f"][sel][:, None], truth["f"][sel][:, None], sz("f"))
    return out


def device_info(G11, G12, G22, g1, g2, f, A1, A2, b):
    return dict(G11=mat(G11), G12=mat(G12), G22=mat(G22), g1=g1, g2=g2, f=f, A1=mat(A1), A2=mat(A2), b=b)


def random_cov(rng, n, scale=(2e-3, 2e-4, 2e-2, 2e-3, 5e-2)):
    """n random SPD 15x15 covariances, exactly symmetric, [n, 15, 15]."""
    D = np.repeat(np.asarray(scale), 3)
    G = rng.normal(size=(n, 15, 15))
    C = G @ G.transpose(0, 2, 1) / 15 + 0.5 * np.eye(15)
    C = D[None, :, None] * C * D[None, None, :]
    return 0.5 * (C + C.transpose(0, 2, 1))


def propagate_stmt(orc, model, X, Xh, Sig, rec, lin, dtype):
    """cov_k1 = A Sigma A^T + B P B^T, A = -H2^-1 H1, B = H2^-1 at (x_k, x_k1), products in ``dtype``."""
    n = len(X)
    st = np.empty((2 * n, 16)); st[0::2] = X; st[1::2] = Xh
    _, H1, H2 = orc.factor_eval(model, st, rec, lin, np.arange(0, 2 * n, 2), np.arange(1, 2 * n, 2))
    H1, H2 = mat(H1).astype(dtype), mat(H2).astype(dtype)
    B = np.zeros((n, 15, 15), dtype=dtype)
    # Q = w I + [v x] (top-left block of H2, q_r = [v w]): Q^-1 = (w^2 I - w [v x] + v v^T) / (w |q|^2)
    w = H2[:, 0, 0]
    v = np.stack([H2[:, 2, 1], H2[:, 0, 2], H2[:, 1, 0]], axis=1)
    K_ = H2[:, 0:3, 0:3] - w[:, None, None] * np.eye(3, dtype=dtype)
    B[:, 0:3, 0:3] = (w[:, None, None] ** 2 * np.eye(3, dtype=dtype) - w[:, None, None] * K_ + v[:, :, None] * v[:, None, :]) / (
        w * (w * w + np.sum(v * v, axis=1)))[:, None, None]
    B[:, 3:6, 3:6] = B[:, 9:12, 9:12] = np.eye(3, dtype=dtype)
    B[:, 6:9, 6:9] = H2[:, 6:9, 6:9].transpose(0, 2, 1)
    B[:, 12:15, 12:15] = H2[:, 12:15, 12:15].transpose(0, 2, 1)
    A = -B @ H1
    S = Sig.astype(dtype)
    Pm = mat(rec[:, 65:290]).astype(dtype)
    return A @ S @ A.transpose(0, 2, 1) + B @ Pm @ B.transpose(0, 2, 1)


def cov_errors(got, truth):
    out = {}
    T = truth.astype(np.float64)
    d = [np.linalg.norm(T[:, B3[I], B3[I]].reshape(len(T), -1), axis=1) for I in range(5)]
    for I in range(5):
        for J in range(I, 5):
            out[f"C_{I}{J}"] = scaled_errors(got[:, B3[I], B3[J]], truth[:, B3[I], B3[J]], np.sqrt(d[I] * d[J]))
    return out


# ---------------------------------------------------------------------------------------------- the batch and its truths

_cache = {}


def batch(oracle, oracle_ld, model):
    """Factor batch of one model with the fp64 and long-double outputs of factor_eval and predict_state (cached per session)."""
    if model not in _cache:
        b = fs.factor_batch(oracle, model, SIGMAS)
        args = (model, b["states"], b["records"], b["lin"], b["idx_i"], b["idx_j"])
        b["o64"] = oracle.factor_eval(*args, nthreads=_threads())
        b["truth"] = oracle_ld.factor_eval(*args, nthreads=_threads())
        b["scales"] = residual_scales(model, b)
        XK = b["states"][b["idx_i"]]
        b["XK"] = XK
        b["pred64"] = oracle.predict_state(model, XK, b["records"], b["lin"])
        b["pred_ld"] = oracle_ld.predict_state(model, XK, b["records"], b["lin"])
        b["pred_scales"] = predict_scales(model, XK, b["records"], b["lin"])
        te, tH1, tH2 = b["truth"]
        b["info_ld"], b["pd"], b["info_size"] = info_stmt(b["records"], te, tH1, tH2, LD)
        b["info_64"] = info_64(b["records"], te, tH1, tH2, b["pd"])
        b["info_64k"] = info_stmt(b["records"], te, tH1, tH2, np.float64)[0]
        _cache[model] = b
    return _cache[model]


def factor_gate(b, got):
    ed = factor_errors(got, b["truth"], b["scales"])
    e64 = factor_errors(b["o64"], b["truth"], b["scales"])
    return gate_errors(ed, {k: e64[k] for k in ed}, K, FLOOR)


def predict_gate(b, got):
    sv, sp = b["pred_scales"]
    ed = state_errors(got, b["pred_ld"], sv, sp)
    e64 = state_errors(b["pred64"], b["pred_ld"], sv, sp)
    return gate_errors(ed, e64, K, FLOOR)


@pytest.fixture(scope="module")
def rbatch(oracle, oracle_ld):
    r = fs.retract_batch()
    r["o64"] = oracle.retract(r["states"], r["xi"])
    r["truth"] = oracle_ld.retract(r["states"], r["xi"])
    r["scales"] = retract_scales(r["states"], r["xi"])
    return r


def retract_gate(r, got):
    ed = state_errors(got, r["truth"], r["scales"], r["scales"], r["scales"])
    e64 = state_errors(r["o64"], r["truth"], r["scales"], r["scales"], r["scales"])
    return gate_errors(ed, e64, K, FLOOR)


def info_gate(b, got):
    """e_64 is the larger error of the two fp64 routes, LAPACK and the kernels' order, and every block is measured relative to the
    terms summed into it.  Measured on the H100: against LAPACK alone and relative to each block's own norm the device was 24x
    the fp64 error on f of a ``far`` factor; with the kernels' order added, 1.3x the bound on g1 of a ``far`` factor, whose e is
    large and whose g1 cancels (g1 = -Y1^T y_e)."""
    sel = b["pd"]
    args = (b["info_ld"], b["info_size"], sel)
    ed = info_errors(got, *args)
    ea, eb = info_errors(b["info_64"], *args), info_errors(b["info_64k"], *args)
    return gate_errors(ed, {k: np.fmax(ea[k], eb[k]) for k in ea}, K, FLOOR)


# ---------------------------------------------------------------------------------------------------------- CPU

@pytest.mark.parametrize("model", [1, 2])
def test_extended_oracle_meets_the_golden_factor_gates(oracle, oracle_ld, golden, model):
    """The long-double factor_eval / retract meet the golden gates of test_gpu_parity (1e-12 of max(1, max|ref|), 1e-14 on the
    retracted states), and its predict_state the 1e-11 gate against the fp64 restatement."""
    F = golden["factor"]
    X, rec, lin = F[f"m{model}/states"], F[f"m{model}/records"], F[f"m{model}/lin"]
    for idx, suffix in ((None, ""), ((F[f"m{model}/idx_i"], F[f"m{model}/idx_j"]), "_idx")):
        got = oracle_ld.factor_eval(model, X, rec, lin, *(idx or (None, None)))
        for g, key in zip(got, ("e", "H1", "H2")):
            ref = F[f"m{model}/{key}{suffix}"]
            assert np.max(np.abs(g - ref)) <= 1e-12 * max(1.0, np.max(np.abs(ref))), key
            assert np.array_equal(g == 0, ref == 0) or key == "e"
    assert np.max(np.abs(oracle_ld.retract(X, F[f"m{model}/xi"]) - F[f"m{model}/retracted"])) <= 1e-14
    pl, p64 = oracle_ld.predict_state(model, X[:-1], rec, lin), oracle.predict_state(model, X[:-1], rec, lin)
    assert np.max(np.abs(pl - p64)) <= 1e-11 * np.max(np.abs(X))


@pytest.mark.parametrize("model", [1, 2])
def test_extended_oracle_agrees_with_fp64_on_the_chain(oracle, oracle_ld, model):
    """On the benign chain regime the two builds agree to 1e-13 in every field (the scale-relative errors above)."""
    b = batch(oracle, oracle_ld, model)
    sel = b["tags"] == "chain"
    e64 = factor_errors(b["o64"], b["truth"], b["scales"])
    e64.update({f"pred_{k}": v for k, v in state_errors(b["pred64"], b["pred_ld"], *b["pred_scales"]).items()})
    worst = {k: float(v[sel].max()) for k, v in e64.items()}
    print(model, "fp64 vs long double on the chain", {k: f"{v:.0e}" for k, v in worst.items() if v > 1e-15})
    assert max(worst.values()) <= 1e-13, worst


@pytest.mark.parametrize("model", [1, 2])
def test_builder_covers_every_branch(oracle, model):
    b = fs.factor_batch(oracle, model, SIGMAS)
    print(model, b["coverage"])
    assert all(v > 0 for v in b["coverage"].values())
    assert set(np.unique(b["tags"])) == set(fs.FREGIMES)
    print(fs.retract_batch()["coverage"])


@pytest.mark.parametrize("model", [1, 2])
def test_gate_passes_the_fp64_oracle(oracle, oracle_ld, model):
    b = batch(oracle, oracle_ld, model)
    for name, (ratio, worst, bad) in (("factor_eval", factor_gate(b, b["o64"])), ("predict", predict_gate(b, b["pred64"])),
                                      ("hessian/whiten", info_gate(b, b["info_64"]))):
        assert not bad, (name, bad)
    structural_zeros_exact(b["truth"][1], H1_BLOCKS); structural_zeros_exact(b["truth"][2], H2_BLOCKS)
    # the indefinite P_meas of the gap windows (and the zero-step record) are what the kernels' Cholesky fails on
    n_bad = int((~b["pd"]).sum())
    assert 0 < n_bad < 0.1 * len(b["pd"])
    print(model, "factors whose P_meas is not positive definite in long double:", n_bad)


def test_gate_passes_the_fp64_retract(rbatch):
    ratio, worst, bad = retract_gate(rbatch, rbatch["o64"])
    assert not bad, bad


def _must_fail(result):
    _, _, bad = result
    assert bad, "the gate missed an injected error"
    return bad


def test_gate_fails_one_element_rounded_to_fp32(oracle, oracle_ld):
    """Every element of e, H1 and the predicted state of one factor per regime.  The factor is the regime's one with the smallest
    position scale: where |p| is 1e4 m or more (the chain after its long windows, ``large``) fp64 itself resolves e_p only to about
    1e-12 absolute, so a float rounding of a small e_p is within what the gate must allow."""
    b = batch(oracle, oracle_ld, 1)
    for reg in ("chain", "near_pi", "bias_far", "zero_bias", "large"):
        sel = np.flatnonzero(b["tags"] == reg)
        i = int(sel[np.argmin(b["scales"]["e_p"][sel])])
        for arr, cols in ((0, range(15)), (1, np.flatnonzero(b["o64"][1][i]))):
            for c in cols:
                got = [a.copy() for a in b["o64"]]
                v = got[arr][i, c]
                if np.float64(np.float32(v)) == v:
                    continue
                got[arr][i, c] = np.float32(v)
                _must_fail(factor_gate(b, got))
        for c in range(16):
            got = b["pred64"].copy()
            v = got[i, c]
            if np.float64(np.float32(v)) == v:
                continue
            got[i, c] = np.float32(v)
            _must_fail(predict_gate(b, got))


def test_gate_fails_a_1e_10_change_of_e_theta_that_the_flat_gate_passes(oracle, oracle_ld):
    b = batch(oracle, oracle_ld, 1)
    i = int(np.flatnonzero(b["tags"] == "chain")[7])
    got = [a.copy() for a in b["o64"]]
    got[0][i, 0:3] *= 1 + 1e-10
    ref = b["o64"][0]
    assert np.max(np.abs(got[0] - ref)) <= 1e-11 * max(1.0, np.max(np.abs(ref)))    # test_factor_chain_5k_and_predict's gate
    bad = _must_fail(factor_gate(b, got))
    assert any(x.startswith("e_th") for x in bad), bad


def test_gate_fails_one_G11_block_scaled_by_1e_11(oracle, oracle_ld):
    b = batch(oracle, oracle_ld, 1)
    i = int(np.flatnonzero(b["pd"] & (b["tags"] == "chain"))[5])
    for I, J in ((0, 0), (1, 3), (4, 4)):
        got = dict(b["info_64"]); got["G11"] = got["G11"].copy()
        got["G11"][i, B3[I], B3[J]] *= 1 + 1e-11
        bad = _must_fail(info_gate(b, got))
        assert any(x.startswith(f"G11_{I}{J}") for x in bad), bad


# ---------------------------------------------------------------------------------------------------------- GPU

def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _interleaved(b):
    """The batch in chain indexing: states x_K^0, x_K1^0, x_K^1, x_K1^1, ...; factor 2f is factor f, factor 2f+1 links x_K1^f to
    x_K^(f+1) with record f (evaluated, not used)."""
    X = b["states"]
    n = len(b["idx_i"])
    st = np.empty((2 * n, 16)); st[0::2] = X[b["idx_i"]]; st[1::2] = X[b["idx_j"]]
    rec = np.repeat(b["records"], 2, axis=0)[:2 * n - 1]
    lin = np.repeat(b["lin"], 2, axis=0)[:2 * n - 1]
    return st, rec, lin


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_factor_eval_against_extended_oracle(cuda, oracle, oracle_ld, model):
    """K3/K4 through the device and host entry points, idx and chain indexing: the conditioned gate on every field, structural
    zeros exact, and the same bits through every route (each lane computes its factor alone)."""
    from cpi_b200 import factor
    torch = cuda
    b = batch(oracle, oracle_ld, model)
    X, rec, lin, ii, jj = b["states"], b["records"], b["lin"], b["idx_i"], b["idx_j"]
    dX, drec, dlin, dii, djj = (_dev(torch, a) for a in (X, rec, lin, ii, jj))
    got = [t.cpu().numpy() for t in factor.factor_eval(model, dX, drec, dlin, dii, djj)]
    ratio, worst, bad = factor_gate(b, got)
    report(f"m{model} factor_eval", ratio, b["tags"], fs.FREGIMES)
    assert not bad, bad
    structural_zeros_exact(got[1], H1_BLOCKS); structural_zeros_exact(got[2], H2_BLOCKS)
    host = factor.factor_eval_host(model, X, rec, lin, ii, jj)
    st, rc, ln = _interleaved(b)
    chain_h = factor.factor_eval_host(model, st, rc, ln)
    chain_d = [t.cpu().numpy() for t in factor.factor_eval(model, _dev(torch, st), _dev(torch, rc), _dev(torch, ln))]
    for route in (host, [a[0::2] for a in chain_h], [a[0::2] for a in chain_d]):
        for a, g in zip(route, got):
            assert np.array_equal(a, g)
    # partial CTAs: batches of 1, 7, 8, 9 factors give the rows of the full batch
    for m in (1, 7, 8, 9):
        sub = factor.factor_eval_host(model, X, rec[:m], lin[:m], ii[:m], jj[:m])
        for a, g in zip(sub, got):
            assert np.array_equal(a, g[:m])


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_factor_eval_want_flags_and_misaligned_outputs(cuda, oracle, oracle_ld, model):
    """All four want_H1 / want_H2 combinations give the same e (and the same H when asked for); outputs written through views
    offset by one double (copy_out's scalar path) are bit-identical, and the doubles either side of each view stay untouched."""
    from cpi_b200 import factor
    torch = cuda
    b = batch(oracle, oracle_ld, model)
    args = [_dev(torch, a) for a in (b["states"], b["records"], b["lin"], b["idx_i"], b["idx_j"])]
    ref = [t.cpu().numpy() for t in factor.factor_eval(model, *args)]
    for w1 in (False, True):
        for w2 in (False, True):
            e, H1, H2 = factor.factor_eval(model, *args, want_H1=w1, want_H2=w2)
            assert np.array_equal(e.cpu().numpy(), ref[0]) and (H1 is None) != w1 and (H2 is None) != w2
            if w1:
                assert np.array_equal(H1.cpu().numpy(), ref[1])
            if w2:
                assert np.array_equal(H2.cpu().numpy(), ref[2])
    n = len(b["idx_i"])
    SENT = -1.2345678e300
    bufs, views = [], []
    for width in (15, 225, 225):
        buf = torch.full((n * width + 3,), SENT, dtype=torch.float64, device="cuda")
        bufs.append(buf); views.append(buf[1:1 + n * width].view(n, width))
    assert all(v.data_ptr() % 16 == 8 for v in views)
    factor.factor_eval(model, *args, out=tuple(views))
    torch.cuda.synchronize()
    for buf, v, r in zip(bufs, views, ref):
        h = buf.cpu().numpy()
        assert h[0] == SENT and np.all(h[-2:] == SENT)
        assert np.array_equal(v.cpu().numpy(), r)


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_predict_and_retract_against_extended_oracle(cuda, oracle, oracle_ld, rbatch, model):
    from cpi_b200 import factor
    b = batch(oracle, oracle_ld, model)
    got = factor.predict_state(model, b["XK"], b["records"], b["lin"])
    ratio, worst, bad = predict_gate(b, got)
    report(f"m{model} predict", ratio, b["tags"], fs.FREGIMES)
    assert not bad, bad
    got = factor.retract(rbatch["states"], rbatch["xi"])
    ratio, worst, bad = retract_gate(rbatch, got)
    report("retract", ratio, rbatch["tags"], [name for name, _ in fs.RETRACT_ANGLES] + ["1e-12 on 1e6"])
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_propagate_against_extended_statement(cuda, oracle, oracle_ld, model):
    """K7 on the factor pairs' x_K: states_k1 bit for bit k_predict's, cov_k1 against the long-double statement at that x_k1."""
    from cpi_b200 import factor
    torch = cuda
    b = batch(oracle, oracle_ld, model)
    XK, rec, lin = b["XK"], b["records"], b["lin"]
    Sig = random_cov(np.random.default_rng(model), len(XK))
    x1, c1, _ = factor.propagate(model, _dev(torch, XK), _dev(torch, flat(Sig)), _dev(torch, rec), _dev(torch, lin))
    x1, c1 = x1.cpu().numpy(), mat(c1.cpu().numpy())
    assert np.array_equal(x1, factor.predict_state(model, XK, rec, lin))
    # H1 / H2 at the kernel's own x_k1 (gated above against the truth of predict_state): with |p| up to 1e6 m an ulp of the
    # predicted position is 1e-14 of pa, which the (v, theta) / (p, theta) blocks inherit whichever code rounded it
    t = propagate_stmt(oracle_ld, model, XK, x1, Sig, rec, lin, LD)
    c64 = propagate_stmt(oracle, model, XK, x1, Sig, rec, lin, np.float64)
    ratio, worst, bad = gate_errors(cov_errors(c1, t), cov_errors(c64, t), K, FLOOR)
    report(f"m{model} propagate", ratio, b["tags"], fs.FREGIMES)
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_information_form_against_extended_statement(cuda, oracle, oracle_ld, model):
    """k_factor_hessian and k_factor_whiten on the long-double e / H1 / H2: every block gated where P_meas is positive definite;
    where it is not (indefinite gap windows, the zero-step record) f and b are NaN, and the other factors of the same CTA finite."""
    from cpi_b200 import factor
    b = batch(oracle, oracle_ld, model)
    rec = b["records"]
    e, H1, H2 = b["truth"]
    hs = factor.factor_hessian(model, rec, e, H1, H2)
    wh = factor.factor_whiten(model, rec, e, H1, H2)
    got = device_info(*hs, *wh)
    pd = b["pd"]
    bad_rows = np.flatnonzero(~pd)
    assert np.all(np.isnan(got["f"][bad_rows])) and np.all(np.isnan(got["b"][bad_rows]))
    cta = np.unique(bad_rows // 4)
    mates = np.setdiff1d(np.concatenate([4 * cta + k for k in range(4)]), bad_rows)
    mates = mates[mates < len(pd)]
    print(model, "non-PD factors", len(bad_rows), "their CTA mates", len(mates))
    assert len(mates) > 0
    for k, v in got.items():
        assert np.all(np.isfinite(v[pd])), k
    ratio, worst, bad = info_gate(b, got)
    report(f"m{model} hessian/whiten", ratio, b["tags"][pd], fs.FREGIMES)
    assert not bad, bad
    for k in ratio:
        assert np.all(ratio[k][np.searchsorted(np.flatnonzero(pd), mates)] <= 1.0)
