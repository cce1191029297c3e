"""Extended-precision gate of the filter's time update (cpi_propagate_batch, kernel K7; DESIGN.md sections 3d and 5) on the propagation
stress batch of tests/propagate_stress.py, over chained runs of thousands of keyframes, in filter runs alternating with K11 and K13,
and at production scale (K7, and the filter's update K10 past one wave).

The truth is oracle/cpi_oracle.c's oracle_propagate in long double, order 0: x_k1 kept unrounded, H1 / H2 the dense Jacobians of
evaluateError at (x_k, x_k1), B = H2^-1 by a pivoted Gauss-Jordan inverse and dense products.  It shares no algebra with the kernel
(order 1 restates the kernel's sparse route).  e_64 is the larger error, in the window's group (its tag), of the fp64 orders 0 and 1,
each built plain (-ffp-contract=off) and fma-contracted, pooled over every block of a field.  Every window satisfies
    e_dev <= 8 max(e_64, floor, 1e-15).
Fields: Sigma_k1 per 3x3 block pair relative to sqrt(|Sigma_k1,II| |Sigma_k1,JJ|); the cross-covariance C = Sigma_k A^T per 3x3 block
relative to sqrt(|Sigma_k,II| |Sigma_k1,JJ|); x_k1 in retract coordinates local(x_true, x) in the truth's standard deviations, with
the one-ulp floor of test_update_precision._floor (x_k1 is stored in fp64: no route does better than half an ulp); a component
whose truth sd is 0 (Sigma_k = 0 through a record with a zero block of P_meas) is measured in its own units.

Departures from the plain per-entry measure, and why:
  * e_64 pools the two orders: the long-double orders themselves differ by up to 2.2x the fp64 error of a window (measured on this
    batch), because order 0 inverts Rk while order 1 (and the kernel) uses Rk^T, and Rk of a quaternion that is unit only to fp64
    is orthogonal only to 1e-16.
  * e_64 pools the blocks of a field within a group: which block pair a rounding lands in differs from route to route.
  * the contracted builds are in e_64 because the kernel contracts to fma (as in test_measurements_precision)."""
from __future__ import annotations

import atexit
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import propagate_stress as ps
from parity import scaled_errors
from test_update_precision import FLOOR, K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B3 = [slice(3 * k, 3 * k + 3) for k in range(5)]
UPPER = [(I, J) for I in range(5) for J in range(I, 5)]
_CACHE = {}


def mat(a):
    return np.asarray(a).reshape(-1, 15, 15).transpose(0, 2, 1)


def _threads():
    from cpi_b200.synth import usable_cpus
    return usable_cpus()


# ---------------------------------------------------------------------------------------------- the statements

def _oracle(kind):
    """'fp64', 'ld' (oracle/Makefile's builds) or 'fma' (fp64, -ffp-contract=fast and -mfma where the host has it, in a temporary
    directory), as oracle.Oracle objects."""
    if kind not in _CACHE:
        from oracle import oracle as om
        import update_ref as ur
        if kind == "fma":
            tmp = tempfile.mkdtemp(prefix="cpi_oracle_fma_")
            atexit.register(shutil.rmtree, tmp, True)
            out = os.path.join(tmp, "liboracle_fma.so")
            src = os.path.join(ROOT, "oracle", "cpi_oracle.c")
            subprocess.run([os.environ.get("CC", "gcc"), "-std=c11", "-O2", "-fPIC", "-shared", "-fno-fast-math", "-ffp-contract=fast",
                            *(["-mfma"] if ur._host_fma() else []), "-pthread", "-o", out, src, "-lm"], check=True)
            cls = type("OracleFMA", (om.Oracle,), dict(path=out))
        else:
            cls = om.OracleLD if kind == "ld" else om.Oracle
            if not os.path.exists(cls.path):
                subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-s", os.path.basename(cls.path)], check=True)
        _CACHE[kind] = cls()
    return _CACHE[kind]


FP64 = (("fp64", 0), ("fp64", 1), ("fma", 0), ("fma", 1))


def batch(model):
    """The stress batch of one model with the truth and the four fp64 routes (cached per session)."""
    key = ("batch", model)
    if key not in _CACHE:
        if np.finfo(np.longdouble).nmant < 63:
            pytest.skip("long double has no extended precision on this platform")
        b = ps.stress_batch(_oracle("fp64"), model)
        args = (model, b["x"], b["cov"], b["records"], b["lin"])
        b["truth"] = _oracle("ld").propagate(*args, order=0, nthreads=_threads())
        b["fp64"] = [_oracle(k).propagate(*args, order=o, nthreads=_threads()) for k, o in FP64]
        _CACHE[key] = b
    return _CACHE[key]


# ---------------------------------------------------------------------------------------------- the measure

def errors(b, got, truth):
    """[n, 15 + 25 + 15]: Sigma_k1 per upper block pair, C per block, x_k1 per component (retract coordinates in the truth's sd)."""
    tx, tc, tr = truth
    T, S0 = mat(tc), mat(b["cov"])
    G, GC, TC = mat(got[1]), mat(got[2]), mat(tr)
    dT = [np.linalg.norm(T[:, B3[I], B3[I]], axis=(1, 2)) for I in range(5)]
    d0 = [np.linalg.norm(S0[:, B3[I], B3[I]], axis=(1, 2)) for I in range(5)]
    es = [scaled_errors(G[:, B3[I], B3[J]], T[:, B3[I], B3[J]], np.sqrt(dT[I] * dT[J])) for I, J in UPPER]
    ec = [scaled_errors(GC[:, B3[I], B3[J]], TC[:, B3[I], B3[J]], np.sqrt(d0[I] * dT[J])) for I in range(5) for J in range(5)]
    sd = np.sqrt(np.abs(np.diagonal(T, axis1=1, axis2=2)))
    dx = np.abs(_oracle("ld").local(tx, got[0]))
    ex = dx / np.where(sd > 0, sd, 1.0)                 # a component the truth holds exactly (sd 0): in its own units
    return np.concatenate([np.stack(es, 1), np.stack(ec, 1), ex], axis=1)


POOL = np.r_[np.zeros(15, int), np.ones(25, int), 2 + np.repeat(np.arange(5), 3)]       # Sigma_k1 | C | x_k1 per 3-block
NAMES = [f"S[{I},{J}]" for I, J in UPPER] + [f"C[{I},{J}]" for I in range(5) for J in range(5)] + [f"x[{k}]" for k in range(15)]


def floor(truth):
    """[n, 55]: one ulp of the stored x_k1 per component in the truth's sd (0 for the covariances)."""
    tx, tc, _ = truth
    sd = np.sqrt(np.abs(np.diagonal(mat(tc), axis1=1, axis2=2)))
    ulp = np.concatenate([np.full((len(tx), 3), 2.0 ** -52), np.spacing(np.abs(tx[:, 4:16]))], axis=1)
    return np.concatenate([np.zeros((len(tx), 40)), ulp / np.where(sd > 0, sd, 1.0)], axis=1)


def e64_of(tags, errs):
    """[n, 55]: the worst error of every fp64 route in the window's group, pooled over the blocks of a field."""
    out = np.zeros_like(errs[0])
    for e in errs:
        assert np.all(np.isfinite(e)), "an fp64 route is not finite on the batch"
        e = np.stack([e[:, POOL == POOL[c]].max(axis=1) for c in range(e.shape[1])], axis=1)
        for t in np.unique(tags):
            g = tags == t
            out[g] = np.maximum(out[g], e[g].max(axis=0))
    return out


def gate(b, got, sel=None):
    """(worst ratio, its group and field, per-group worst ratio dict) of got = (x_k1, cov_k1, cross) over the windows sel."""
    if "e64" not in b:
        b["e64"] = e64_of(b["tag"], [errors(b, o, b["truth"]) for o in b["fp64"]])
        b["floor"] = floor(b["truth"])
    sel = np.ones(len(b["x"]), bool) if sel is None else sel
    ed = errors(b, got, b["truth"])
    r = np.where(np.isnan(ed), np.inf, ed / (K * np.maximum(np.maximum(b["e64"], b["floor"]), FLOOR)))[sel]
    i, j = np.unravel_index(int(np.argmax(r)), r.shape)
    tags = b["tag"][sel]
    fam = np.array([t.split("/")[2] for t in tags])
    per = {f: float(r[fam == f].max()) for f in np.unique(fam)}
    return float(r[i, j]), f"{tags[i]} {NAMES[j]}", per


# ---------------------------------------------------------------------------------------------------------- CPU

@pytest.mark.parametrize("model", [1, 2])
def test_long_double_orders_agree(model):
    """The long-double orders agree to 1e-14 of the block scales (measured 4.1e-15 and 2.9e-15: Rk^-1 against Rk^T, see the module docstring,
    and the mirrored upper triangle of a merged P_meas that is symmetric only to rounding); order 0 agrees with
    test_propagate.propagate_ref on the long-double Jacobians to 1e-12 (an fp64 numpy statement: measured 1.4e-13); its A (the
    cross-covariance of Sigma_k = I) agrees with the central difference of the implicit map to 1e-6."""
    from test_propagate import implicit_state, local, propagate_ref
    b = batch(model)
    ld = _oracle("ld")
    o1 = ld.propagate(model, b["x"], b["cov"], b["records"], b["lin"], order=1, nthreads=_threads())
    e = errors(b, o1, b["truth"])[:, :40]
    print(f"model {model}: long-double orders differ by {e.max():.1e} of the block scales")
    assert e.max() <= 1e-14
    assert np.array_equal(o1[0], b["truth"][0])
    pick = np.flatnonzero(np.char.startswith(b["tag"], "stress/bias_off/random"))[:64]
    _, _, _, S1, C = propagate_ref(ld, model, b["x"][pick], b["cov"][pick], b["records"][pick], b["lin"][pick])
    T = mat(b["truth"][1][pick])
    d = np.sqrt(np.abs(np.diagonal(T, axis1=1, axis2=2)))
    assert np.max(np.abs(S1 - T) / (d[:, :, None] * d[:, None, :])) <= 1e-12
    w, h = int(np.flatnonzero(np.char.startswith(b["tag"], "stress/at_lin/random"))[3]), 1e-5   # there x_k1 solves e = 0
    x, rec, lin = b["x"][w], b["records"][w], b["lin"][w]
    At = mat(ld.propagate(model, x[None], np.eye(15).reshape(1, 225), rec[None], lin[None])[2])[0]
    x1 = implicit_state(ld, model, x, rec, lin, b["truth"][0][w])
    Afd = np.zeros((15, 15))
    for c in range(15):
        dd = np.zeros(15); dd[c] = h
        xp = implicit_state(ld, model, ld.retract(x[None], dd[None])[0], rec, lin, x1)
        xm = implicit_state(ld, model, ld.retract(x[None], -dd[None])[0], rec, lin, x1)
        Afd[:, c] = (local(x1[None], xp[None])[0] - local(x1[None], xm[None])[0]) / (2 * h)
    worst = max(np.linalg.norm(Afd[B3[I], B3[J]] - At.T[B3[I], B3[J]]) / max(np.linalg.norm(At.T[B3[I], B3[J]]), 1.0)
                for I in range(5) for J in range(5))
    assert worst <= 1e-6, worst


@pytest.mark.parametrize("model", [1, 2])
def test_batch_covers_the_families(model):
    """Every anchor and covariance family in every record family (merged and scan: model 1 only, K5 and K6 take model 1), q_n's flip
    both ways, |J_q dbg| past 3 rad and the dead-reckoned block scales (asserted by the builder)."""
    b = batch(model)
    parts = np.array([t.split("/") for t in b["tag"]])
    rfams = {"stress", "gaps", "edge"} | ({"merged", "scan"} if model == 1 else set())
    assert set(parts[:, 0]) == rfams
    for r in rfams:
        sel = parts[:, 0] == r
        assert set(parts[sel, 1]) == set(ps.ANCHORS) and set(parts[sel, 2]) == set(ps.COVS)
    print(f"model {model}: {len(b['x'])} windows, coverage {b['coverage']}")


def _table_row(b, model, got, w):
    """Whether the criteria of test_propagate (1e-12 per block against its fp64 numpy statement, cov_k1 and cross) and of
    test_factor_precision (Sigma_k1 only, gated against its long-double statement) catch got on the windows w."""
    from test_factor_precision import cov_errors, propagate_stmt
    from test_propagate import block_errors, propagate_ref
    from parity import gate_errors
    o, ld = _oracle("fp64"), _oracle("ld")
    x, S, r, L = b["x"][w], b["cov"][w], b["records"][w], b["lin"][w]
    _, _, _, S1, C = propagate_ref(o, model, x, S, r, L)
    G, GC = mat(got[1][w]), mat(got[2][w])
    tp = block_errors(G, S1, S1, S1)[0] > 1e-12 or block_errors(GC, C, mat(S), S1)[0] > 1e-12
    x1 = got[0][w]
    t = propagate_stmt(ld, model, x, x1, mat(S), r, L, np.longdouble)
    c64 = propagate_stmt(o, model, x, x1, mat(S), r, L, np.float64)
    tf = bool(gate_errors(cov_errors(G, t), cov_errors(c64, t), 8.0, 1e-15)[2])
    return tp, tf


def test_gate_passes_fp64_and_fails_injected_errors():
    """Both fp64 orders, plain and contracted, pass the gate on both models; four injected errors fail it (model 1, one window each),
    and the table says which the criteria of test_propagate / test_factor_precision catch."""
    for model in (1, 2):
        b = batch(model)
        for (k, o), out in zip(FP64, b["fp64"]):
            r, where, _ = gate(b, out)
            print(f"model {model} fp64 {k} order {o}: worst ratio {r:.3f} ({where})")
            assert r <= 1.0, (k, o, where)
    b = batch(1)
    base = b["fp64"][1]
    w = int(np.flatnonzero(np.char.startswith(b["tag"], "stress/bias_off/random"))[5])
    inj = {}
    c = base[2].copy(); M = mat(c[w:w + 1])[0]; M[B3[4], B3[2]] = M[B3[4], B3[2]].astype(np.float32)
    c[w] = M.T.reshape(225); inj["C: one block rounded to fp32"] = (base[0], base[1], c)
    c = base[2].copy(); c[w] = mat(c[w:w + 1])[0].reshape(225); inj["C written as A Sigma (untransposed)"] = (base[0], base[1], c)
    s = base[1].copy(); M = mat(s[w:w + 1])[0]; M[B3[3], B3[3]] *= 1 + 1e-9
    s[w] = M.T.reshape(225); inj["Sigma_k1 (b_a, b_a) x (1 + 1e-9)"] = (base[0], s, base[2])
    A = mat(_oracle("fp64").propagate(1, b["x"][w:w + 1], np.eye(15).reshape(1, 225), b["records"][w:w + 1], b["lin"][w:w + 1])[2])[0].T
    A2 = A.copy(); A2[B3[4], B3[2]] -= b["records"][w, 19] * np.eye(3)
    S0 = mat(b["cov"][w:w + 1])[0]
    s = base[1].copy(); c = base[2].copy()
    s[w] = (mat(s[w:w + 1])[0] + A2 @ S0 @ A2.T - A @ S0 @ A.T).T.reshape(225)
    c[w] = (S0 @ A2.T).T.reshape(225)
    inj["A without its DT I block"] = (base[0], s, c)
    rows = []
    for name, got in inj.items():
        r, where, _ = gate(b, got)
        tp, tf = _table_row(b, 1, got, np.array([w]))
        rows.append(f"| {name} | {r:.3g} | {'yes' if tp else 'no'} | {'yes' if tf else 'no'} |")
        assert r > 1.0, (name, r)
    print("\n| injected error | ratio | test_propagate | test_factor_precision |\n|---|---|---|---|\n" + "\n".join(rows))


# ---------------------------------------------------------------------------------------------------------- GPU

def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _k7(torch, model, b, anchor=None, want_cross=True, X=None, S=None):
    from cpi_b200 import factor
    out = factor.propagate(model, _dev(torch, b["x"] if X is None else X), _dev(torch, b["cov"] if S is None else S),
                           _dev(torch, b["records"]), _dev(torch, b["lin"]), anchor=None if anchor is None else _dev(torch, anchor),
                           want_cross=want_cross)
    torch.cuda.synchronize()
    return tuple(None if t is None else t.cpu().numpy() for t in out)


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_batch_against_extended_precision(cuda, model):
    """Sigma_k1, C and x_k1 of every window within the gate; and exactly: Sigma_k1 symmetric, want_cross leaves Sigma_k1's bits,
    states_k1 bitwise predict_state's, anchor=None and anchor=arange(n) the same bits, host and device entries the same bits, and
    Sigma_k = 0 gives C exactly 0."""
    from cpi_b200 import factor
    torch = cuda
    b = batch(model)
    got = _k7(torch, model, b)
    r, where, per = gate(b, got)
    print(f"model {model}: {len(b['x'])} windows, worst ratio {r:.3f} ({where}); per covariance family "
          + " ".join(f"{k}={v:.2f}" for k, v in per.items()))
    assert r <= 1.0, where
    C1 = mat(got[1])
    assert np.array_equal(C1, C1.transpose(0, 2, 1))
    nc = _k7(torch, model, b, want_cross=False)
    assert np.array_equal(nc[0], got[0]) and np.array_equal(nc[1], got[1]) and nc[2] is None
    pred = factor.predict_state(model, _dev(torch, b["x"]), _dev(torch, b["records"]), _dev(torch, b["lin"])).cpu().numpy()
    assert np.array_equal(got[0], pred)
    ar = _k7(torch, model, b, anchor=np.arange(len(b["x"]), dtype=np.int64))
    assert all(np.array_equal(u, v, equal_nan=True) for u, v in zip(got, ar))
    h = factor.propagate_host(model, b["x"], b["cov"], b["records"], b["lin"], want_cross=True)
    assert all(np.array_equal(u, v, equal_nan=True) for u, v in zip(got, h))
    zero = np.char.endswith(b["tag"], "/zero")
    assert np.all(got[2][zero] == 0.0)


def nan_pattern(i, j):
    """Which entries of Sigma_k1 and C [15, 15] the kernel's order makes NaN from a NaN in Sigma_k(i, j) (and its mirror): N = A Sigma
    column by column, row r of Sigma_k1 from A applied to row r of N, the upper triangle mirrored, C = N^T.  a_apply reads its whole
    input into every row of A's structure (0 x NaN is NaN), so A's pattern is its 3x3 block structure with the DT I, I and bias
    identity blocks diagonal."""
    P = np.zeros((15, 15), bool)
    blk = lambda I, J: P.__setitem__((B3[I], B3[J]), True)
    for I, J in ((0, 0), (0, 1), (2, 0), (2, 1), (2, 3), (4, 0), (4, 1), (4, 3)):
        blk(I, J)
    for I, J in ((1, 1), (2, 2), (3, 3), (4, 2), (4, 4)):
        P[B3[I], B3[J]] |= np.eye(3, dtype=bool)
    S = np.zeros((15, 15), bool); S[i, j] = S[j, i] = True
    N = (P.astype(int) @ S.astype(int)) > 0
    R = (N.astype(int) @ P.T.astype(int)) > 0                # row r, column c: from N(r, :) through A's row c
    up = np.triu(np.ones((15, 15), bool))
    S1 = np.where(up, R, R.T)
    return S1, N.T


@pytest.mark.gpu
def test_nan_in_one_window_is_confined(cuda):
    """A ragged anchor array (2 000 windows reading 301 anchors, each anchor read by windows in several warps and CTAs): a NaN in one
    anchor's Sigma_k and one in another window's record.  Every window reading other anchors (and not the bad record) is bitwise the
    clean run, the bad record's three CTA mates included; every window sharing the bad anchor is NaN in exactly the entries
    nan_pattern predicts."""
    torch = cuda
    b = batch(1)
    rng = np.random.default_rng(7)
    m, n = 301, 2000
    ai = rng.choice(len(b["x"]), m, replace=False)
    X, S = b["x"][ai], b["cov"][ai].copy()
    anchor = rng.integers(0, m, n).astype(np.int64)
    wi = rng.choice(len(b["x"]), n, replace=False)
    sub = dict(x=X, cov=S, records=b["records"][wi].copy(), lin=b["lin"][wi])
    bad_a = int(anchor[10])
    cta_clean = np.flatnonzero(np.all((anchor != bad_a).reshape(-1, 4), axis=1))
    bad_w = int(4 * cta_clean[len(cta_clean) // 2] + 1)                # a window whose three CTA mates read other anchors
    share = anchor == bad_a
    assert len(np.unique(np.flatnonzero(share) // 4)) >= 2
    clean = _k7(torch, 1, sub, anchor=anchor)
    i, j = 13, 7                                                      # (p, v): an off-diagonal entry
    sub["cov"][bad_a, i + 15 * j] = sub["cov"][bad_a, j + 15 * i] = np.nan
    sub["records"][bad_w, 13] = np.nan                              # alpha: x_k1, H1 and through them Sigma_k1
    dirty = _k7(torch, 1, sub, anchor=anchor)
    keep = ~share; keep[bad_w] = False
    mates = [w for w in range(4 * (bad_w // 4), 4 * (bad_w // 4) + 4) if w != bad_w]
    assert keep[mates].all()
    assert all(np.array_equal(u[keep], v[keep]) for u, v in zip(clean, dirty))
    assert all(np.all(~np.isnan(v[keep])) for v in dirty)
    p1, pc = nan_pattern(i, j)
    for k in np.flatnonzero(share):
        assert np.array_equal(np.isnan(mat(dirty[1][k])[0]), p1) and np.array_equal(np.isnan(mat(dirty[2][k])[0]), pc)
        assert np.array_equal(dirty[0][k], clean[0][k])
    assert np.isnan(dirty[0][bad_w, 13]) and np.any(np.isnan(dirty[1][bad_w]))


# ---------------------------------------------------------------------------------------------- chained runs

STEPS = 4999


def _chain_gate(truth_S, e64s, got_S):
    """Worst ratio of the chained covariances [C, 225] (Sigma per upper block pair, pooled over pairs) to K max(e_64, FLOOR)."""
    def err(S):
        T, G = mat(truth_S), mat(S)
        d = [np.linalg.norm(T[:, B3[I], B3[I]], axis=(1, 2)) for I in range(5)]
        return np.stack([scaled_errors(G[:, B3[I], B3[J]], T[:, B3[I], B3[J]], np.sqrt(d[I] * d[J])) for I, J in UPPER], 1)
    e64 = max(float(err(S).max()) for S in e64s)
    return float(err(got_S).max() / (K * max(e64, FLOOR))), e64


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_dead_reckoning_chain(cuda, model):
    """4 999 keyframes of dead reckoning from one anchor per chain (3 chains), one K7 call per keyframe.  The covariance after the
    last keyframe is gated along the device's own trajectory: the long-double chain of oracle_propagate_chain from the device's
    states; e_64 the four fp64 chains along the same trajectory.  The final state is gated against the long-double chain's own
    prediction, e_64 the fp64 chains' own predictions, in the truth's sd with the one-ulp floor.  Model 1: the same through K6 (the
    scan of each chain) and one anchored K7 call, against the long-double sequential chain at keyframes 50, 600 and 4 999."""
    from cpi_b200 import factor, preint
    torch = cuda
    o = _oracle("fp64")
    C = 3
    rec, L = ps.chain_records(o, model, C, STEPS, 73000 + 10 * model)
    X0 = ps.anchors_at_lin(rec[::STEPS], L[::STEPS], model)
    S0 = ps.ur.random_cov(np.random.default_rng(9), C)
    R, Lr = rec.reshape(C, STEPS, -1), L.reshape(C, STEPS, 13)
    dR, dL = _dev(torch, R.transpose(1, 0, 2)), _dev(torch, Lr.transpose(1, 0, 2))
    x, S = _dev(torch, X0), _dev(torch, S0)
    path = torch.empty((STEPS + 1, C, 16), dtype=torch.float64, device="cuda")
    path[0] = x
    for k in range(STEPS):
        x, S, _ = factor.propagate(model, x, S, dR[k], dL[k])
        path[k + 1] = x
    torch.cuda.synchronize()
    path, S, x = path.transpose(0, 1).cpu().numpy(), S.cpu().numpy(), x.cpu().numpy()
    ld = _oracle("ld")
    _, tS = ld.propagate_chain(model, X0, S0, R, Lr, STEPS, order=0, path=path, nthreads=_threads())
    e64s = [_oracle(k).propagate_chain(model, X0, S0, R, Lr, STEPS, order=od, path=path, nthreads=_threads())[1] for k, od in FP64]
    r, e64 = _chain_gate(tS, e64s, S)
    print(f"model {model}: {STEPS} keyframes along the device's trajectory: Sigma ratio {r:.3f} (e_64 {e64:.1e})")
    assert r <= 1.0
    tx, tS2 = ld.propagate_chain(model, X0, S0, R, Lr, STEPS, order=0, nthreads=_threads())
    sd = np.sqrt(np.diagonal(mat(tS2), axis1=1, axis2=2))
    ex = lambda xx: np.abs(ld.local(tx, xx)) / sd
    fl = np.concatenate([np.full((C, 3), 2.0 ** -52), np.spacing(np.abs(tx[:, 4:16]))], axis=1) / sd
    e64x = np.max([ex(_oracle(k).propagate_chain(model, X0, S0, R, Lr, STEPS, order=od, nthreads=_threads())[0]) for k, od in FP64], axis=0)
    rr = ex(x) / (K * np.maximum(np.maximum(e64x, fl), FLOOR))
    rx = float(np.max(rr))
    c, k = np.unravel_index(int(np.argmax(rr)), rr.shape)
    routes = " ".join(f"{ex(_oracle(n).propagate_chain(model, X0, S0, R, Lr, STEPS, order=od, nthreads=_threads())[0])[c, k] / fl[c, k]:.1f}"
                      for n, od in FP64)
    print(f"model {model}: final state ratio {rx:.3f} at chain {c} component {k}: device {ex(x)[c, k] / fl[c, k]:.1f} ulp, "
          f"fp64 routes {routes} ulp of the stored component; sd {sd[c, k]:.2e}")
    assert rx <= 1.0
    if model != 1:
        return
    scan = preint.scan(1, _dev(torch, rec), _dev(torch, L), group=STEPS)
    anchor = np.repeat(np.arange(C), STEPS).astype(np.int64)
    _, one, _ = factor.propagate(1, _dev(torch, X0), _dev(torch, S0), scan, _dev(torch, L), anchor=_dev(torch, anchor))
    torch.cuda.synchronize()
    one = one.cpu().numpy().reshape(C, STEPS, 225)
    scan64 = o.scan_records(rec, L, group=STEPS, nthreads=_threads())
    for k in (50, 600, STEPS):
        _, tk = ld.propagate_chain(1, X0, S0, R[:, :k], Lr[:, :k], k, order=0, nthreads=_threads())
        e64s = [_oracle(n).propagate_chain(1, X0, S0, R[:, :k], Lr[:, :k], k, order=od, nthreads=_threads())[1] for n, od in FP64]
        e64s += [_oracle(n).propagate(1, X0, S0, scan64.reshape(C, STEPS, -1)[:, k - 1], Lr[:, k - 1], order=od, want_cross=False)[1]
                 for n, od in FP64]
        r, e64 = _chain_gate(tk, e64s, one[:, k - 1])
        print(f"K6 + one K7 at keyframe {k}: ratio {r:.3f} (e_64 {e64:.1e})")
        assert r <= 1.0


# ---------------------------------------------------------------------------------------------- production scale

PWARPS = 4                                                           # windows (warps) per CTA of k_propagate


def _same_bits(torch, out, cls, first):
    ref = out.index_select(0, first.index_select(0, cls))
    return torch.equal(out.view(torch.int64), ref.view(torch.int64))


def placement(n, C, sms):
    """K7's launch geometry: ceil(n / 4) CTAs of 4 windows and no grid-stride loop.  With window p a copy of class p mod C (C odd),
    returns whether every class sits at every warp slot mod 4, has a copy in the first, the middle and the last `sms` CTAs (with
    4 sms >= C windows, each such run of CTAs holds every class), and whether the last CTA is partial."""
    p = np.arange(n)
    cls = p % C
    slots = np.zeros((C, PWARPS), bool); slots[cls, p % PWARPS] = True
    cta = p // PWARPS
    n_cta = -(-n // PWARPS)
    first = np.zeros(C, bool); first[cls[cta < sms]] = True
    last = np.zeros(C, bool); last[cls[cta >= n_cta - sms]] = True
    mid = np.zeros(C, bool); mid[cls[(cta >= n_cta // 2) & (cta < n_cta // 2 + sms)]] = True
    return bool(slots.all()), bool(first.all() and mid.all() and last.all()), n % PWARPS != 0


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_k7_at_scale(cuda, model):
    """1.25 * 2^20 + 3 windows (byte offsets into the 225-double outputs past 2^31, the last CTA partial), window p a copy of class
    p mod C of 455 windows spread over the batch (C odd and at most 4 x 114: every class at every warp slot mod 4 and in the first,
    a middle and the last SM-count CTAs, for 132 and 114 SMs and this device's count); anchors are the classes' states, shared by
    copies in every CTA.  With and without cross: every copy bitwise its class's first copy; the first copies pass the batch's
    gate."""
    torch = cuda
    b = batch(model)
    sel = np.unique(np.linspace(0, len(b["x"]) - 1, 455).astype(np.int64))
    C, n = len(sel), 5 * 2 ** 18 + 3
    assert C % 2 == 1 and n * 225 * 8 > 2 ** 31
    sms_here = torch.cuda.get_device_properties(0).multi_processor_count
    for sms in (132, 114, sms_here):
        assert placement(n, C, sms) == (True, True, True), sms
    from cpi_b200 import factor
    torch.cuda.reset_peak_memory_stats()
    d = lambda a: _dev(torch, a)
    cls = torch.arange(n, device="cuda") % C
    rec, lin = d(b["records"][sel]).index_select(0, cls), d(b["lin"][sel]).index_select(0, cls)
    X, S = d(b["x"][sel]), d(b["cov"][sel])
    first = torch.arange(C, device="cuda")
    x1, c1, cr = factor.propagate(model, X, S, rec, lin, anchor=cls, want_cross=True)
    torch.cuda.synchronize()
    assert all(_same_bits(torch, a, cls, first) for a in (x1, c1, cr))
    got = tuple(a[:C].cpu().numpy() for a in (x1, c1, cr))
    del x1, c1, cr
    y1, s1, none = factor.propagate(model, X, S, rec, lin, anchor=cls, want_cross=False)
    torch.cuda.synchronize()
    assert none is None and _same_bits(torch, s1, cls, first)
    assert np.array_equal(s1[:C].cpu().numpy(), got[1]) and np.array_equal(y1[:C].cpu().numpy(), got[0])
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    del y1, s1, rec, lin
    mask = np.zeros(len(b["x"]), bool); mask[sel] = True
    full = tuple(np.zeros((len(b["x"]),) + a.shape[1:]) for a in got)
    for f, g in zip(full, got):
        f[sel] = g
    r, where, _ = gate(b, full, mask)
    print(f"model {model}: K7 at scale, {n} windows of {C} classes ({sms_here} SMs here): copies bitwise their classes; classes' "
          f"worst ratio {r:.3f} ({where}); peak device memory {peak:.1f} GiB")
    assert r <= 1.0
    assert peak < 16.0


@pytest.mark.gpu
def test_k10_at_scale(cuda):
    """K10 (cpi_state_update_batch) on 10^6 filters, filter p a copy of class p mod C: the classes are K10's stress batch
    (update_ref.stress_batch) with this batch's dead-reckoned K7 covariances of both models as an extra family, C odd (every class at
    every warp slot mod 4).  Filters with p mod 3 = 0 are gated at 16, the rest at +inf, so gated and applied filters share CTAs and
    every class has copies of both kinds (C mod 3 != 0).  Every copy is bitwise its class's first copy of the same gate; a gated copy
    that was not applied is bitwise its input, an applied one bitwise the ungated copy; the ungated first copies pass
    test_update_precision's gate."""
    import update_ref as ur
    from test_update_precision import gate as k10_gate
    from cpi_b200 import factor
    torch = cuda
    extra = np.concatenate([batch(m)["cov"][np.char.endswith(batch(m)["tag"], f"/at_lin/dr{k}")][:8] for m in (1, 2) for k in (600, 5000)])
    b = ur.stress_batch(np.random.default_rng(20261017), extra_cov=extra)
    keep = np.ones(len(b["x"]), bool)
    while keep.sum() % 2 == 0 or keep.sum() % 3 == 0:
        keep[np.flatnonzero(keep)[-1]] = False
    b = {k: v[keep] for k, v in b.items()}
    C, n = len(b["x"]), 10 ** 6
    d = lambda a: _dev(torch, a)
    torch.cuda.reset_peak_memory_stats()
    cls = torch.arange(n, device="cuda") % C
    X, S, W, XB = (d(b[k]).index_select(0, cls) for k in ("x", "cov", "W", "xb"))
    p = torch.arange(n, device="cuda")
    gated = p % 3 == 0
    g = torch.where(gated, torch.full((n,), 16.0, dtype=torch.float64, device="cuda"),
                    torch.full((n,), float("inf"), dtype=torch.float64, device="cuda"))
    x1, c1, nis, applied = factor.update(X, S, W, XB, gate=g)
    torch.cuda.synchronize()
    # the first copy of class c with the same gate: p = c + j C for the smallest j with (c + j C) mod 3 matching
    c = torch.arange(C, device="cuda")
    first_open = torch.where(c % 3 != 0, c, c + C)
    first_gated = torch.stack([c + j * C for j in range(3)], 1)
    first_gated = first_gated.gather(1, (first_gated % 3 == 0).int().argmax(1, keepdim=True))[:, 0]
    ref = torch.where(gated, first_gated.index_select(0, cls), first_open.index_select(0, cls))
    bits = lambda t: t.contiguous().view(torch.int64) if t.dtype == torch.float64 else t
    for t in (x1, c1, nis, applied):
        assert torch.equal(bits(t), bits(t.index_select(0, ref)))
    skipped = gated & (applied == 0)
    assert int(skipped.sum()) > 0 and int((gated & (applied == 1)).sum()) > 0
    assert torch.equal(bits(x1[skipped]), bits(X[skipped])) and torch.equal(bits(c1[skipped]), bits(S[skipped]))
    ag = gated & (applied == 1)
    open_ref = first_open.index_select(0, cls[ag])
    assert torch.equal(bits(c1[ag]), bits(c1.index_select(0, open_ref))) and torch.equal(bits(x1[ag]), bits(x1.index_select(0, open_ref)))
    fo = first_open
    got = (x1[fo].cpu().numpy(), c1[fo].cpu().numpy(), nis[fo].cpu().numpy())
    assert bool((applied[fo] == 1).all())
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    del X, S, W, XB, x1, c1, nis, applied
    r, name, _ = k10_gate(b, got)
    print(f"K10 at scale: {n} filters of {C} classes, {int(gated.sum())} gated at 16 ({int(skipped.sum())} not applied): copies bitwise "
          f"their classes; classes' worst ratio {r:.3f} ({name}); peak device memory {peak:.1f} GiB")
    assert r <= 1.0, (name, r)


FILTER_STEPS = 600


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_k7_in_a_filter_run(cuda, model):
    """600 keyframes of 16 filters each in three runs: K7 alternating with K11, with K13 under Huber and with K13 under Cauchy losses,
    lever-arm GNSS (1 m lever arm, 5 cm) every 3rd keyframe and a magnetometer (unit field, 0.01) every 5th, the fixes drawn about the
    predicted state at 1 sigma.  Every K7 step of every filter is gated as a window of the batch is, against the long-double step from
    the device's own input state and covariance (so rounding does not compound in the truth), e_64 the four fp64 routes from the same
    inputs, pooled within a run and the kind of the step before it (prediction or update)."""
    import measurement_ref as mr
    from cpi_b200 import capi, factor
    torch = cuda
    o = _oracle("fp64")
    F, runs = 16, ("k11", "huber", "cauchy")
    N = F * len(runs)
    rec, L = ps.chain_records(o, model, N, FILTER_STEPS, 81000 + 10 * model)
    R, Lr = rec.reshape(N, FILTER_STEPS, -1), L.reshape(N, FILTER_STEPS, 13)
    X = ps.anchors_at_lin(R[:, 0], Lr[:, 0], model)
    S = ps.ur.random_cov(np.random.default_rng(11), N)
    rng = np.random.default_rng(12)
    d = lambda a: _dev(torch, a)
    x, s = d(X), d(S)
    ins_x, ins_s, outs, tags = [], [], [], []
    prev = "pred"
    for k in range(FILTER_STEPS):
        ins_x.append(x.cpu().numpy()); ins_s.append(s.cpu().numpy())
        x1, s1, c1 = factor.propagate(model, x, s, d(R[:, k]), d(Lr[:, k]), want_cross=True)
        outs.append(tuple(t.cpu().numpy() for t in (x1, s1, c1)))
        tags += [f"filter/{r}/{prev}" for r in np.repeat(runs, F)]
        kinds = ([mr.POSITION] if k % 3 == 2 else []) + ([mr.DIRECTION] if k % 5 == 4 else [])
        x, s, prev = x1, s1, "pred"
        if not kinds:
            continue
        xp = outs[-1][0]
        idx, kind, z, si, aux = [], [], [], [], []
        for kd in kinds:
            a = rng.normal(size=(N, 3))
            a = a / np.linalg.norm(a, axis=1, keepdims=True)                # 1 m lever arm, unit field
            sig = 0.05 if kd == mr.POSITION else 0.01
            h = mr.h_of(np.full(N, kd, np.int32), xp, a)
            idx.append(np.arange(N)); kind.append(np.full(N, kd, np.int32)); aux.append(a)
            z.append(h + sig * rng.normal(size=(N, 3))); si.append(np.tile((np.eye(3) / sig).reshape(9), (N, 1)))
        meas = (d(np.concatenate(idx).astype(np.int64)), d(np.concatenate(kind)), d(np.concatenate(z)), d(np.concatenate(si)),
                d(np.concatenate(aux)))
        m = len(kinds) * N
        loss = np.where(np.tile(np.repeat(np.arange(3), F), len(kinds)) == 1, capi.LOSS_HUBER, capi.LOSS_CAUCHY).astype(np.int32)
        lk = np.full(m, 2.0)
        xa, sa, _, _ = factor.update_measurements(x1, s1, meas)
        xb, sb, *_ = factor.update_measurements_iterated(x1, s1, meas, measurement_loss=(d(loss), d(lk)), max_iterations=10, tol=1e-9)
        k11 = torch.arange(N, device="cuda") < F
        x = torch.where(k11[:, None], xa, xb)
        s = torch.where(k11[:, None], sa, sb)
        prev = "update"
    torch.cuda.synchronize()
    b = dict(x=np.concatenate(ins_x), cov=np.concatenate(ins_s), records=R.transpose(1, 0, 2).reshape(-1, R.shape[2]),
             lin=Lr.transpose(1, 0, 2).reshape(-1, 13), tag=np.array(tags))
    args = (model, b["x"], b["cov"], b["records"], b["lin"])
    b["truth"] = _oracle("ld").propagate(*args, order=0, nthreads=_threads())
    b["fp64"] = [_oracle(kk).propagate(*args, order=od, nthreads=_threads()) for kk, od in FP64]
    got = tuple(np.concatenate([u[i] for u in outs]) for i in range(3))
    r, where, _ = gate(b, got)
    updated = mat(b["cov"][np.char.endswith(b["tag"], "/update")])
    print(f"model {model}: K7 in {len(runs)} filter runs of {FILTER_STEPS} keyframes ({len(b['x'])} steps, "
          f"{int(np.char.endswith(b['tag'], '/update').sum())} after an update, their position sd down to "
          f"{np.sqrt(updated[:, 12, 12].min()):.1e} m): worst ratio {r:.3f} ({where})")
    assert r <= 1.0, where
