"""Precision of the record merge (K5, cpi_merge_records) and scan (K6, cpi_scan_records) kernels against an extended-precision truth.

The truth is the long-double build of the oracle's dense statement of the composition (oracle/cpi_oracle.c: oracle_merge_records,
oracle_scan_records, the left fold of every group with full 15x15 Phi~ and T).  Inputs: the record stress batch of
tests/record_stress.py (stress windows cut into segments at moved linearisation points, independent records of every regime in
random groups, and the group lengths where the kernels' CTA widths, chunks and levels change).  Per record: q (up to sign only
where the truth's |w| < 1e-12, so a missing w < 0 flip fails; its e_64 is the larger of q's and R's), R, alpha, beta, DT, J_q, J_a, J_b, H_a, H_b and every 3x3 block
of P, each relative to its own norm; the gate is e_dev <= K max(e_64, floor), K = 8, floor = 1e-15 (parity.gate_errors).  e_64
is the larger fp64 error of two bracketings: the oracle's fp64 left fold, and the kernel's own order of merges restated with
the fp64 oracle's pair merge (record_stress.merge_bracketing / scan_bracketing).  fp32 storage: the truth is the long-double
fold of the float-rounded inputs and the bound gains one output rounding, 2^-24: every operation is fp64.

CPU tests: the long-double fold of a window's segments is its long-double one-shot record; the fp64 fold is test_merge.fold; the
gate passes the fp64 fold and fails four injected errors that the flat 1e-12 gate of test_merge passes.  GPU tests: K5 and K6
through the device and host entry points, uniform and CSR layouts, fp64 and fp32, and one group of 5 000 and one of 10^5
records; DESIGN.md section 5 lists the measured worst ratios."""
import os
import subprocess

import numpy as np
import pytest

import record_stress as rs
import test_merge as tm
from parity import REC, field_errors, scaled_errors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIGMAS = np.array([0.005, 4e-6, 0.01, 0.0002])
K, FLOOR = 8.0, 1e-15
U32 = 2.0 ** -24


@pytest.fixture(scope="module")
def oracles():
    """(fp64, long double) oracles.  make rebuilds a library older than its source: the session ``oracle`` fixture only builds
    a missing one, and the entry points used here are newer than the rest of the library."""
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("long double has no extended precision on this platform")
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "liboracle.so", "liboracle_ld.so"], check=True)
    from oracle import oracle as om
    return om.Oracle(), om.OracleLD()


def _threads():
    return rs._threads()


# ---------------------------------------------------------------------------------------------- errors and the gate

def record_errors(got, truth):
    """dict field -> [n] relative error per record (parity.field_errors' fields and P blocks, DT, and q compared up to sign only
    where the truth's w is below 1e-12)."""
    got = np.asarray(got, dtype=np.float64)
    e = field_errors(got, truth, 1)
    e["q"] = scaled_errors(got[:, 0:4], truth[:, 0:4], sign_free=np.abs(truth[:, 3]) < 1e-12)
    e["DT"] = scaled_errors(got[:, 19:20], truth[:, 19:20])
    return e


def gate(got, truth, o64s, allowance=0.0):
    """e_dev <= K max(e_64, FLOOR) + allowance, e_64 the larger error of the fp64 computations o64s.  Returns (ratio, worst, bad)."""
    got = np.asarray(got, dtype=np.float64)
    assert np.all(np.isfinite(got)), "non-finite output"
    ed = record_errors(got, truth)
    e64 = [record_errors(o, truth) for o in o64s]
    ratio, worst, bad = {}, {}, []
    for k in ed:
        # q is rot_2_quat of R in every code: it carries R's error, whichever of the two the fp64 computations got luckier on
        m = np.max(np.stack([e[j] for e in e64 for j in ((k, "R") if k == "q" else (k,))]), axis=0)
        bound = K * np.maximum(m, FLOOR) + allowance
        r = np.where(np.isnan(ed[k]), np.inf, ed[k] / bound)
        ratio[k] = r
        i = int(np.argmax(r)) if len(r) else 0
        worst[k] = float(r[i]) if len(r) else 0.0
        if len(r) and not r[i] <= 1.0:
            bad.append(f"{k}: record {i} e_dev {ed[k][i]:.3e} e_64 {m[i]:.3e} bound {bound[i]:.3e}")
    return ratio, worst, bad


def worst_line(label, worst):
    k = max(worst, key=worst.get)
    print(f"{label}: worst ratio {worst[k]:.3f} ({k});", " ".join(f"{f}={v:.2f}" for f, v in worst.items() if v >= 0.05))


def assert_structure(out):
    P_ = np.asarray(out, dtype=np.float64)[:, 65:290].reshape(-1, 15, 15)
    assert np.array_equal(P_, P_.transpose(0, 2, 1)), "P not exactly symmetric"
    assert np.all(P_[:, 0:6, 9:12] == 0), "structural zeros of P"


# ---------------------------------------------------------------------------------------------- the batch and its truths

_cache = {}


def seg_batch(o64):
    if "seg" not in _cache:
        _cache["seg"] = rs.segment_batch(o64, SIGMAS)
    return _cache["seg"]


def ind_batch(o64):
    if "ind" not in _cache:
        pool, plin = rs.independent_pool(o64, SIGMAS)
        rec, lin, off = rs.random_groups(np.random.default_rng(rs.SEED + 1), pool, plin, 240)
        _cache["ind"] = dict(pool=pool, pool_lin=plin, records=rec, lin=lin, offsets=off)
    return _cache["ind"]


def merge_cases(o64):
    """(name, records, lin, offsets, group): the segment groups, the independent groups, every uniform width and the ragged lengths."""
    seg, ind = seg_batch(o64), ind_batch(o64)
    rng = np.random.default_rng(rs.SEED + 2)
    pool, plin = ind["pool"], ind["pool_lin"]
    cases = [("segments", seg["records"], seg["lin"], seg["offsets"], None),
             ("independent", ind["records"], ind["lin"], ind["offsets"], None)]
    for w in rs.MERGE_WIDTHS:
        idx = rng.integers(0, len(pool), size=12 * w)
        cases.append((f"uniform {w}", pool[idx], plin[idx], None, w))
    lens = np.r_[rs.MERGE_RAGGED, rs.MERGE_RAGGED[::-1]]
    off = np.zeros(len(lens) + 1, dtype=np.int64); off[0] = 2; off[1:] = 2 + np.cumsum(lens)
    idx = rng.integers(0, len(pool), size=int(off[-1]) + 1)
    cases.append(("ragged", pool[idx], plin[idx], off, None))
    return cases


def scan_cases(o64):
    seg, ind = seg_batch(o64), ind_batch(o64)
    rng = np.random.default_rng(rs.SEED + 3)
    pool, plin = ind["pool"], ind["pool_lin"]
    off = rs.scan_layout(rng)
    idx = rng.integers(0, len(pool), size=int(off[-1]) + 2)
    return [("segments", seg["records"], seg["lin"], seg["offsets"], None),
            ("independent", ind["records"], ind["lin"], ind["offsets"], None),
            ("uniform 33", pool[idx[:33 * 40]], plin[idx[:33 * 40]], None, 33),
            ("lengths", pool[idx], plin[idx], off, None)]


def truths(kind, o64, old, name, rec, lin, off, grp, dtype):
    """(long-double fold, fp64 fold, fp64 kernel bracketing) of one case, inputs rounded to ``dtype`` first (cached)."""
    key = (kind, name, np.dtype(dtype).name)
    if key not in _cache:
        r, l = rec.astype(dtype).astype(np.float64), lin.astype(dtype).astype(np.float64)
        fn = "merge_records" if kind == "merge" else "scan_records"
        t = getattr(old, fn)(r, l, off, grp, nthreads=_threads())
        f = getattr(o64, fn)(r, l, off, grp, nthreads=_threads())
        b = (rs.merge_bracketing if kind == "merge" else rs.scan_bracketing)(o64, r, l, off, grp)
        _cache[key] = (t, f, b)
    return _cache[key]


# ---------------------------------------------------------------------------------------------------------- CPU

def test_batch_covers_its_regimes(oracles):
    o64, old = oracles
    seg = seg_batch(o64)
    assert set(seg["regime"]) == set(rs.stress.REGIMES) and set(seg["offset"]) == set(rs.OFFSETS)
    assert set(seg["S"]) == set(rs.SEGMENTS)
    n_steps = np.diff(seg["seg_offsets"])
    assert np.any(n_steps == 0) and np.any(n_steps == 1)
    # zero-step records inside a group: a 1-sample segment holding a dt = 0 sample
    first = np.zeros(len(n_steps), dtype=bool); first[seg["offsets"][:-1]] = True
    zero_dt = (seg["records"][:, 19] == 0) & (n_steps == 1)
    assert np.any(zero_dt & ~first)
    big = seg["angle"]
    print("|J_q db_w| of the moved segments: max", f"{big.max():.4f}", "closest to pi", f"{np.min(np.abs(big - np.pi)):.1e}")
    assert 2.9 <= big.max() <= np.pi + 1e-3 and np.min(np.abs(big - np.pi)) <= 1e-3
    # every rot_2_quat case and both sides of its flip in the truth's merged R
    seen = {}
    for name, rec, lin, off, grp in merge_cases(o64)[:2]:
        t = truths("merge", o64, old, name, rec, lin, off, grp, np.float64)[0]
        many = np.diff(off) >= 2
        case, flip = rs.r2q_branches(t[many])
        for c, label in enumerate(rs.fs.R2Q_CASES):
            seen[label] = seen.get(label, 0) + int(np.sum(case == c))
        seen["flip"] = seen.get("flip", 0) + int(flip.sum()); seen["no flip"] = seen.get("no flip", 0) + int((~flip).sum())
    print("rot_2_quat branches of the merged R:", seen)
    assert all(v > 0 for v in seen.values()), seen


def test_extended_fold_of_segments_is_the_one_shot_record(oracles):
    """Long double: a window's segments preintegrated and folded give its one-shot record.  The means and Jacobians compose exactly,
    so they agree to the rounding of the fp64-stored segment records (measured: worst 5.3e-16 relative, on R); P differs by the RK4 truncation of the
    transitions the merge replaces (worst 2.5e-5 per block outside the gap and fast regimes; reported there)."""
    o64, old = oracles
    seg = seg_batch(o64)
    sel = np.isin(seg["offset"], ("zero", "qg"))
    segrec = old.preintegrate(1, seg["samples"], seg["lin"], SIGMAS, 0, offsets=seg["seg_offsets"], nthreads=_threads())
    folded = old.merge_records(segrec, seg["lin"], seg["offsets"], nthreads=_threads())[sel]
    one = old.preintegrate(1, seg["win_samples"], seg["win_lin"], SIGMAS, 0, offsets=seg["win_offsets"], nthreads=_threads())[sel]
    e = record_errors(folded, one)
    worst = {k: float(v.max()) for k, v in e.items()}
    print("long-double fold vs one-shot:", {k: f"{v:.1e}" for k, v in worst.items()})
    for k in ("R", "alpha", "beta", "J_q", "J_a", "J_b", "H_a", "H_b", "q", "DT"):
        assert worst[k] <= 2e-15, (k, worst[k])
    tags = seg["regime"][sel]
    ordinary = ~np.isin(tags, ("gaps", "fast"))
    Pw = np.max(np.stack([v for k, v in e.items() if k.startswith("P_")]), axis=0)
    print("P block gap to the one-shot: ordinary", f"{Pw[ordinary].max():.1e}", "gaps / fast", f"{Pw[~ordinary].max():.1e}")
    assert Pw[ordinary].max() <= 1e-4


def test_fp64_fold_is_the_numpy_fold(oracles):
    o64, _ = oracles
    ind = ind_batch(o64)
    rec, lin, off = ind["records"], ind["lin"], ind["offsets"]
    got = o64.merge_records(rec, lin, off)
    ref = np.stack([tm.fold(rec[off[g]:off[g + 1]], lin[off[g]:off[g + 1]]) for g in range(len(off) - 1)])
    e = record_errors(got, ref)
    worst = {k: float(v.max()) for k, v in e.items()}
    print("fp64 C fold vs numpy fold:", {k: f"{v:.0e}" for k, v in worst.items()})
    # test_merge.merge2 conjugates Phi2 by T^T, the oracle by T^-1 (the transform that composes): they differ by the orthogonality
    # defect of the stored rotations in the v and p blocks of P (1e-12 after the 10 000-sample windows)
    R = rec[:, 4:13].reshape(-1, 3, 3)
    defect = float(np.max(np.linalg.norm(R.transpose(0, 2, 1) @ R - np.eye(3), axis=(1, 2))))
    for k, v in worst.items():
        assert v <= (1e-12 if not k.startswith("P_") else 10 * defect + 1e-13), (k, v, defect)
    assert np.all(got[:, 65:290].reshape(-1, 15, 15)[:, 0:6, 9:12] == 0), "structural zeros of P"


@pytest.mark.parametrize("kind", ["merge", "scan"])
def test_gate_passes_fp64_and_the_kernels_bracketing(oracles, kind):
    """The fp64 fold passes; so does the fp64 restatement of the kernel's bracketing, and the ratio against the fold alone is
    printed (how much the bracketing calibration of e_64 is needed on these inputs)."""
    o64, old = oracles
    for name, rec, lin, off, grp in (merge_cases if kind == "merge" else scan_cases)(o64):
        t, f, b = truths(kind, o64, old, name, rec, lin, off, grp, np.float64)
        rows = slice(None) if kind == "merge" else _rows(len(rec), off)
        assert not gate(f[rows], t[rows], [f[rows]])[2]
        _, w_fold, _ = gate(b[rows], t[rows], [f[rows]])
        _, w_both, bad = gate(b[rows], t[rows], [f[rows], b[rows]])
        assert not bad, (name, bad)
        print(kind, name, f"bracketing against the fold's e_64: {max(w_fold.values()):.2f}")


def _rows(n, off):
    rows = np.zeros(n, dtype=bool)
    if off is None:
        rows[:] = True
    else:
        rows[off[0]:off[-1]] = True
    return rows


def _must_fail(got, t, f, field):
    _, _, bad = gate(got, t, [f])
    assert bad, "the gate missed an injected error"
    assert any(x.startswith(field) for x in bad), bad


def _setP(rec, I, fn):
    P = rec[:, 65:290].reshape(-1, 15, 15).transpose(0, 2, 1).copy()
    P[:, 3 * I:3 * I + 3, 3 * I:3 * I + 3] = fn(P[:, 3 * I:3 * I + 3, 3 * I:3 * I + 3])
    rec[:, 65:290] = P.transpose(0, 2, 1).reshape(-1, 225)


def test_gate_fails_injected_errors_that_the_flat_gate_passes(oracles):
    """Four injected errors in the fp64 fold of the segment groups: P_bg,bg rounded to fp32, P_ba,ba scaled by 1 + 1e-9, the move to
    the first lin skipped where only b_a differs, and q without its w < 0 flip.  The first two pass test_merge's whole-matrix
    1e-12 gate, the third its 1e-12 gate on everything but alpha and beta."""
    o64, old = oracles
    seg = seg_batch(o64)
    rec, lin, off = seg["records"], seg["lin"], seg["offsets"]
    t, f, _ = truths("merge", o64, old, "segments", rec, lin, off, None, np.float64)
    many = np.flatnonzero((np.diff(off) >= 2) & (seg["offset"] == "zero") & (t[:, 19] > 0))
    g = int(many[np.argmax(np.diff(off)[many])])
    for I, fn, field in ((1, lambda B: B.astype(np.float32).astype(np.float64), "P_11"), (3, lambda B: B * (1 + 1e-9), "P_33")):
        got = f.copy()
        sub = got[g:g + 1]; _setP(sub, I, fn); got[g] = sub[0]
        assert tm.field_errors(got[g:g + 1], f[g:g + 1])["P"] <= 1e-12
        _must_fail(got, t, f, field)
    # the move skipped where only b_a differs from the first lin (a kernel testing db_w alone)
    first = np.repeat(off[:-1], np.diff(off))
    only_a = np.all(lin[:, 0:3] == lin[first, 0:3], axis=1) & np.any(lin[:, 3:6] != lin[first, 3:6], axis=1)
    assert only_a.sum() > 10
    lin_b = lin.copy(); lin_b[only_a, 3:6] = lin[first[only_a], 3:6]
    got = o64.merge_records(rec, lin_b, off, nthreads=_threads())
    bad = gate(got, t, [f])[2]
    assert bad and any(x.startswith(("alpha", "beta")) for x in bad), bad
    # q without its flip
    _, flip = rs.r2q_branches(f)
    assert flip.sum() > 0
    got = f.copy(); got[flip, 0:4] *= -1
    _must_fail(got, t, f, "q")


def test_q_lin_and_gravity_do_not_enter(oracles):
    """lin[6:13] of the later records leaves the fold bit-identical (a model-1 record does not depend on them)."""
    o64, _ = oracles
    seg = seg_batch(o64)
    rec, lin, off = seg["records"], seg["lin"], seg["offsets"]
    first = np.repeat(off[:-1], np.diff(off))
    lin_r = lin.copy(); lin_r[:, 6:13] = lin[first, 6:13]
    assert not np.array_equal(lin_r, lin)
    assert np.array_equal(o64.merge_records(rec, lin, off), o64.merge_records(rec, lin_r, off))


# ---------------------------------------------------------------------------------------------------------- GPU

def _run(torch, kind, path, rec, lin, off, grp):
    from cpi_b200 import preint
    if path == "host":
        return (preint.merge_host if kind == "merge" else preint.scan_host)(1, rec, lin, group_offsets=off, group=grp)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    out = (preint.merge if kind == "merge" else preint.scan)(1, d(rec), d(lin), group_offsets=None if off is None else d(off), group=grp)
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kind", ["merge", "scan"])
def test_kernel_against_extended_oracle(cuda, oracles, kind, dtype):
    """Every case through the device and the host entry point (same bits), held to the conditioned gate; scan: out[lo] is
    records[lo] bit for bit.  P exactly symmetric with its structural zeros exact."""
    o64, old = oracles
    allow = 0.0 if dtype == np.float64 else U32
    for name, rec, lin, off, grp in (merge_cases if kind == "merge" else scan_cases)(o64):
        t, f, b = truths(kind, o64, old, name, rec, lin, off, grp, dtype)
        r, l = rec.astype(dtype), lin.astype(dtype)
        got = _run(cuda, kind, "device", r, l, off, grp)
        host = _run(cuda, kind, "host", r, l, off, grp)
        assert got.dtype == dtype and np.array_equal(host, got), name
        rows = slice(None) if kind == "merge" else _rows(len(rec), off)
        if kind == "scan":
            starts = np.arange(0, len(rec), grp) if off is None else np.unique(off[:-1][np.diff(off) > 0])
            assert np.array_equal(got[starts], r[starts])
        assert_structure(got[rows])
        _, w_fold, _ = gate(got[rows], t[rows], [f[rows]], allow)
        ratio, worst, bad = gate(got[rows], t[rows], [f[rows], b[rows]], allow)
        worst_line(f"{kind} {np.dtype(dtype).name} {name} (fold-only e_64: {max(w_fold.values()):.2f})", worst)
        assert not bad, (name, bad)


@pytest.mark.gpu
def test_long_groups(cuda, oracles):
    """One group of 5 000 consecutive 20-sample records and one of 10^5 (those records tiled, each at its own lin), through both
    kernels.  Scan: every prefix."""
    o64, old = oracles
    rec5, lin5 = rs.chain_records(o64, SIGMAS)
    rng = np.random.default_rng(rs.SEED + 4)
    big = np.arange(100_000) % len(rec5)
    for n, rec, lin in ((5000, rec5, lin5), (100_000, rec5[big], lin5[rng.integers(0, len(rec5), size=len(big))])):
        for kind in ("merge", "scan"):
            t, f, b = truths(kind, o64, old, f"long {n}", rec, lin, None, n, np.float64)
            got = _run(cuda, kind, "device", rec, lin, None, n)
            if kind == "merge":
                assert np.array_equal(_run(cuda, kind, "host", rec, lin, None, n), got)
            assert_structure(got)
            _, w_fold, _ = gate(got, t, [f])
            ratio, worst, bad = gate(got, t, [f, b])
            worst_line(f"{kind} long {n} (fold-only e_64: {max(w_fold.values()):.2f})", worst)
            assert not bad, (n, kind, bad)
