"""Inclusive scan of consecutive model-1 records within groups (cpi_scan_records / _host, preint.scan / scan_host).

The truth is the numpy left fold of test_merge.py taken at every prefix: out[i] of group lo .. hi-1 is fold(records[lo .. i]).  The
GPU tests compare the kernel with those prefix folds, with the merge kernel, with the device one-shot preintegration of every prefix
window and with the oracle, and check the dead reckoning of a chain from one anchor state."""
import ctypes

import numpy as np
import pytest

from cpi_b200 import capi, synth
from parity import compare_records, fp32_errors, window_band
from test_merge import (FIELDS, _pack, _random_cuts, _record_pool, _unpack, field_errors, merge2, relinearise, split_windows,
                        with_ref_DT)

RD = 290
CHUNK = 32                      # records per chunk of the kernel (scan.cu C)
P = lambda a: ctypes.c_void_p(a.ctypes.data)


def prefix_folds(records, lins, at=None):
    """fold(records[0 .. i]) for every i (or for i in `at`), incrementally: every later record moved to lins[0], composed in order."""
    want = set(range(len(records))) if at is None else set(int(i) for i in at)
    out = {}
    if len(records) == 0:
        return out
    acc = _unpack(records[0])
    if 0 in want:
        out[0] = records[0].copy()
    for i in range(1, len(records)):
        acc = merge2(acc, relinearise(records[i], lins[i], lins[0]))
        if i in want:
            out[i] = _pack(acc)
    return out


def scan_ref(rec, lin, off):
    ref = np.zeros_like(rec)
    for g in range(len(off) - 1):
        lo, hi = off[g], off[g + 1]
        for i, r in prefix_folds(rec[lo:hi], lin[lo:hi]).items():
            ref[lo + i] = r
    return ref


def assert_structure(out):
    P_ = np.asarray(out, dtype=np.float64)[:, 65:290].reshape(-1, 15, 15)
    assert np.all(np.isfinite(out))
    assert np.array_equal(P_, P_.transpose(0, 2, 1)), "P not exactly symmetric"
    assert np.all(P_[:, 0:6, 9:12] == 0), "structural zeros of P"


# ------------------------------------------------------------------------------------------------------------------
# CPU: argument checks of the C ABI (no device needed)
# ------------------------------------------------------------------------------------------------------------------

def test_scan_argument_validation_without_gpu():
    lib = capi.load()
    buf = np.zeros(4 * RD); lin = np.zeros(4 * 13); out = np.zeros(4 * RD); ws = np.zeros(64)
    for fn, extra in ((lib.cpi_scan_records, (P(ws), None)), (lib.cpi_scan_records_host, ())):
        rc = fn(2, 64, 2, None, 2, P(buf), P(lin), P(out), *extra)
        assert rc == -1 and b"model 2" in lib.cpi_last_error() and b"scanned" in lib.cpi_last_error()
        rc = fn(3, 64, 2, None, 2, P(buf), P(lin), P(out), *extra)
        assert rc == -1 and b"model" in lib.cpi_last_error()
        rc = fn(1, 16, 2, None, 2, P(buf), P(lin), P(out), *extra)
        assert rc == -1 and b"dtype" in lib.cpi_last_error()
        rc = fn(1, 64, -1, None, 2, P(buf), P(lin), P(out), *extra)
        assert rc == -1 and b"negative" in lib.cpi_last_error()
        rc = fn(1, 64, 2, None, -2, P(buf), P(lin), P(out), *extra)
        assert rc == -1 and b"negative" in lib.cpi_last_error()
        for args in ((None, P(lin), P(out)), (P(buf), None, P(out)), (P(buf), P(lin), None)):
            rc = fn(1, 64, 2, None, 2, *args, *extra)
            assert rc == -1 and b"null" in lib.cpi_last_error()
        assert fn(1, 64, 0, None, 2, None, None, None, *([None, None] if extra else [])) == 0
        assert fn(1, 32, 0, None, 0, None, None, None, *([None, None] if extra else [])) == 0
        rc = fn(1, 64, 2, None, 2, P(buf), P(lin), P(buf), *extra)
        assert rc == -1 and b"overlap" in lib.cpi_last_error()
    # the device entry point needs its workspace, and checks the uniform layout's whole extent for overlap
    rc = lib.cpi_scan_records(1, 64, 2, None, 2, P(buf), P(lin), P(out), None, None)
    assert rc == -1 and b"workspace" in lib.cpi_last_error()
    rc = lib.cpi_scan_records(1, 64, 2, None, 2, P(buf), P(lin), ctypes.c_void_p(buf.ctypes.data + 8 * RD), P(ws), None)
    assert rc == -1 and b"overlap" in lib.cpi_last_error()
    # host offsets: decreasing, negative start, past any possible record count
    for offs, word in (([0, 3, 2, 4], b"non-decreasing"), ([-1, 1, 2, 4], b"out of range"), ([0, 1, 2, 1 << 61], b"out of range")):
        o = np.array(offs, dtype=np.int64)
        rc = lib.cpi_scan_records_host(1, 64, 3, P(o), 0, P(buf), P(lin), P(out))
        assert rc == -1 and word in lib.cpi_last_error(), (offs, lib.cpi_last_error())
    # workspace: explicit, grows with the record count, never zero
    assert lib.cpi_scan_records_workspace(-1, 4) == -1 and lib.cpi_scan_records_workspace(1, -4) == -1
    sizes = [lib.cpi_scan_records_workspace(1, n) for n in (0, 1, CHUNK, CHUNK + 1, 10 ** 4, 10 ** 6)]
    assert sizes[0] > 0 and sizes == sorted(sizes)
    assert sizes[3] == 8 * 291 * 2 and sizes[5] >= 8 * 291 * (10 ** 6 // CHUNK)
    # Python layer: layout errors are caught before the library is called
    from cpi_b200 import preint
    with pytest.raises(ValueError):
        preint.scan_host(1, buf.reshape(4, RD), lin.reshape(4, 13))
    with pytest.raises(ValueError):
        preint.scan_host(1, buf.reshape(4, RD), lin.reshape(4, 13), group=3)
    with pytest.raises(ValueError):
        preint.scan_host(1, buf.reshape(4, RD), lin.reshape(4, 13), group=0)
    with pytest.raises(capi.CpiError, match="model 2"):
        preint.scan_host(2, np.zeros((2, 308)), np.zeros((2, 13)), group=2)
    got = preint.scan_host(1, np.zeros((0, RD)), np.zeros((0, 13)), group_offsets=np.zeros(1, dtype=np.int64))
    assert got.shape == (0, RD)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_scan_matches_numpy_prefix_folds(cuda):
    """Ragged groups around the chunk size (0, 1, 2, C-1, C, C+1, 2C+1 and random), at one linearisation point per group or a different
    one per record, starting after a few records outside every group: every out[i] is the numpy prefix fold to <= 1e-12 per field,
    and the rows outside every group are left as they were."""
    from cpi_b200 import preint
    torch = cuda
    pool, Lp = _record_pool()
    rng = np.random.default_rng(5)
    lens = np.r_[[0, 1, 2, CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK + 1, 0, 0], rng.integers(0, 80, size=40)]
    head = 3
    off = np.zeros(len(lens) + 1, dtype=np.int64); off[0] = head; off[1:] = head + np.cumsum(lens)
    n = int(off[-1])
    idx = rng.integers(0, len(pool), size=n)
    rec = pool[idx]; lin = Lp[rng.integers(0, len(pool), size=n)].copy()
    for g in range(0, len(lens), 2):                    # even groups: one linearisation point for the whole group
        lin[off[g]:off[g + 1]] = lin[off[g]]
    ref = scan_ref(rec, lin, off)
    sentinel = torch.full((n, RD), 7.0, dtype=torch.float64, device="cuda")
    d = preint.scan(1, torch.from_numpy(rec).cuda(), torch.from_numpy(lin).cuda(), group_offsets=torch.from_numpy(off).cuda(),
                    out=sentinel)
    torch.cuda.synchronize()
    d = d.cpu().numpy()
    assert np.all(d[:head] == 7.0)
    err = field_errors(d[head:], ref[head:])
    print({k: f"{v:.1e}" for k, v in err.items()})
    for k in FIELDS + ("q", "DT", "P"):
        assert err[k] <= 1e-12, (k, err[k])
    assert_structure(d[head:])
    host = preint.scan_host(1, rec, lin, group_offsets=off)
    assert np.array_equal(host[head:], d[head:]) and np.all(host[:head] == 0)


@pytest.mark.gpu
def test_long_groups_spread_over_many_ctas(cuda):
    """One group of 5 000 records and one of 10^5 (tiled from the pool, each at a different linearisation point): sampled prefixes (the
    first, around chunk edges of every level, the last) against the numpy fold.  Observed on one H100 80GB HBM3 (700 W): means,
    Jacobians, q and DT <= 4.2e-14 and 1.5e-13; P 7.1e-11 at 5 000 and 3.5e-8 at 10^5 records.  P is ill-conditioned in the
    bracketing over such chains: the numpy fold and a numpy pairwise tree of the same records differ by 1.9e-10 and 5.3e-8 on P.
    The P gate is about 5x the observed value at each length."""
    from cpi_b200 import preint
    torch = cuda
    pool, Lp = _record_pool(n=2048, first_window=74000)
    for n, seed, tol_P in ((5000, 6, 5e-10), (100_000, 7, 2e-7)):
        rng = np.random.default_rng(seed)
        rec = pool[np.arange(n) % len(pool)]; lin = Lp[rng.integers(0, len(pool), size=n)]
        edges = [e + k for e in (CHUNK, CHUNK ** 2, CHUNK ** 3) for k in (-1, 0, 1) if e + k < n]
        at = np.unique(np.r_[0, 1, 2, edges, rng.integers(0, n, size=8), n - 2, n - 1])
        d = preint.scan(1, torch.from_numpy(rec).cuda(), torch.from_numpy(lin).cuda(), group=n)
        torch.cuda.synchronize()
        d = d.cpu().numpy()
        assert_structure(d)
        ref = prefix_folds(rec, lin, at)
        err = field_errors(d[at], np.stack([ref[i] for i in at]))
        print(n, {k: f"{v:.1e}" for k, v in err.items()})
        for k in FIELDS + ("q", "DT"):
            assert err[k] <= 1e-12, (n, k, err[k])
        assert err["P"] <= tol_P, (n, err["P"])


@pytest.mark.gpu
def test_last_element_is_the_merge_and_first_a_copy(cuda):
    """out[hi-1] is cpi_merge_records of the group to <= 1e-12 per field; out[lo] is records[lo] bit for bit (fp64 and fp32).  (fp32
    records are not compared with the merge: float-rounded rotations are orthogonal only to ~1e-7, so two bracketings of them differ
    by more than the output rounding.)"""
    from cpi_b200 import preint
    pool, Lp = _record_pool(n=1024, first_window=75000)
    rng = np.random.default_rng(9)
    lens = np.r_[[1, 2, CHUNK, CHUNK + 1, 300], rng.integers(1, 120, size=60)]
    off = np.zeros(len(lens) + 1, dtype=np.int64); off[1:] = np.cumsum(lens)
    idx = rng.integers(0, len(pool), size=int(off[-1]))
    rec, lin = pool[idx], Lp[rng.integers(0, len(pool), size=len(idx))]
    for dt in (np.float64, np.float32):
        r, l = rec.astype(dt), lin.astype(dt)
        s = preint.scan_host(1, r, l, group_offsets=off)
        m = preint.merge_host(1, r, l, group_offsets=off) if dt is np.float64 else None
        assert s.dtype == dt and np.array_equal(s[off[:-1]], r[off[:-1]])
        if dt is np.float64:
            err = field_errors(s[off[1:] - 1], m)
            print({k: f"{v:.1e}" for k, v in err.items()})
            for k in FIELDS + ("q", "DT", "P"):
                assert err[k] <= 1e-12, (k, err[k])


@pytest.mark.gpu
def test_split_window_prefixes_match_one_shot_and_oracle(cuda, oracle):
    """Windows of 200 samples (incl. the forced small_w / zero-w_hat / dt = 0 windows) cut into S segments (incl. segments of 0 and 1
    samples), one CSR preintegration of the segments, one scan: every prefix against the device one-shot preintegration of the same
    prefix window (1e-12 on the means and Jacobians; P within the RK4 truncation, as the merge's split test) and, on a selection,
    against the oracle's prefix records under the standard gates."""
    from cpi_b200 import preint
    torch = cuda
    n, ns = 1000, 200
    S, L = synth.make_windows(n, ns, rate=200.0, first_window=64000)
    mag = np.linalg.norm(S[:, :, 0:3] - L[:, None, 0:3], axis=2)
    special = np.where((mag.max(axis=1) < 0.0088) | (S[:, :, 6].min(axis=1) == 0))[0]
    assert len(special) >= 3
    sel = np.unique(np.r_[0:16, n - 8:n, special[:16]])
    rng = np.random.default_rng(10)
    for nseg in (3, 8, 40):
        cuts = _random_cuts(rng, n, ns, nseg)
        Sx, off, Ls, _ = split_windows(S, L, cuts)
        dLs = torch.from_numpy(Ls).cuda()
        seg = preint.preintegrate(1, torch.from_numpy(Sx).cuda(), dLs, synth.SIGMAS, 0, offsets=torch.from_numpy(off).cuda())
        got = preint.scan(1, seg, dLs, group=nseg)
        # the prefix windows: window w's samples 0 .. bound_j, one CSR one-shot call
        bounds = np.concatenate([np.r_[c, ns] for c in cuts])                       # end sample of every prefix
        win = np.repeat(np.arange(n), nseg)
        poff = np.zeros(n * nseg + 1, dtype=np.int64); poff[1:] = np.cumsum(bounds)
        Sp = np.concatenate([S[w, :b] for w, b in zip(win, bounds)]).reshape(-1, 7)
        one = preint.preintegrate(1, torch.from_numpy(Sp).cuda(), dLs, synth.SIGMAS, 0, offsets=torch.from_numpy(poff).cuda())
        torch.cuda.synchronize()
        got, one = got.cpu().numpy(), one.cpu().numpy()
        err = field_errors(got, one)
        for k in FIELDS + ("q",):
            assert err[k] <= 1e-12, (nseg, k, err[k])
        assert err["P"] <= 1e-7, (nseg, err["P"])
        assert np.all(np.abs(got[:, 19] - one[:, 19]) <= 1e-14 * np.abs(one[:, 19]))
        assert_structure(got)
        rows = (sel[:, None] * nseg + np.arange(nseg)[None, :]).reshape(-1)
        Sr = np.concatenate([S[win[r], :bounds[r]] for r in rows]).reshape(-1, 7)
        roff = np.zeros(len(rows) + 1, dtype=np.int64); roff[1:] = np.cumsum(bounds[rows])
        ref = oracle.preintegrate(1, Sr, Ls[rows], synth.SIGMAS, 0, offsets=roff, nthreads=8)
        band = window_band(Sr, roff, Ls[rows])
        worst = compare_records(with_ref_DT(got[rows], ref), ref, 1, in_band=band, has_steps=bounds[rows] > 0)
        print(f"S={nseg}: vs oracle", {k: f"{v:.1e}" for k, v in worst.items()}, "vs one-shot", {k: f"{v:.1e}" for k, v in err.items()})


@pytest.mark.gpu
def test_dead_reckoning_from_one_anchor(cuda):
    """Chains of 300 keyframes of 20 samples (as the configs[4] chain) at one linearisation point: predict_state(x_0, out[j]) for every
    j in one launch equals the sequential predict_state chain to <= 1e-12, and the factor between x_0 and that state, built from
    out[j], has a zero residual (<= 1e-11)."""
    from cpi_b200 import factor, preint
    n_chains, k = 3, 300
    S, L = synth.make_windows(n_chains * k, 20, rate=200.0, first_window=65000, special=False)
    L = np.repeat(L[::k], k, axis=0)                    # one linearisation point per chain
    rec = preint.preintegrate_host(1, S, L, synth.SIGMAS, 0, ns=20)
    out = preint.scan_host(1, rec, L, group=k)
    X = synth.make_states(rec[::k], L[::k], 1)[:n_chains]
    X[:, 4:7], X[:, 10:13] = L[::k, 0:3], L[::k, 3:6]    # biases at the linearisation point: the factor's bias-correction terms vanish
    X[:, 13:16] = 0.0                                   # positions at the origin
    seq = np.empty((n_chains, k, 16))
    x = X
    for j in range(k):
        x = factor.predict_state(1, x, rec[j::k], L[j::k])
        seq[:, j] = x
    x0 = np.repeat(X, k, axis=0)
    xs = factor.predict_state(1, x0, out, L)
    ref = seq.reshape(-1, 16)
    per = np.max(np.abs(xs - ref) / np.maximum(1.0, np.abs(ref)), axis=0)
    err = per.max()
    print("predict", err, "per state entry", " ".join(f"{v:.1e}" for v in per))
    assert err <= 1e-12
    st = np.empty((2 * len(xs), 16)); st[0::2] = x0; st[1::2] = xs
    e, _, _ = factor.factor_eval_host(1, st, out, L, np.arange(0, len(st), 2), np.arange(1, len(st), 2))
    print("residual", np.max(np.abs(e)))
    assert np.max(np.abs(e)) <= 1e-11


@pytest.mark.gpu
def test_fp32_storage(cuda):
    """Float records scan in fp64 arithmetic: the result is the fp64 scan of the same float-rounded records, rounded once."""
    from cpi_b200 import preint
    pool, Lp = _record_pool(n=2000, first_window=76000)
    rng = np.random.default_rng(11)
    lens = rng.integers(0, 70, size=300)
    off = np.zeros(len(lens) + 1, dtype=np.int64); off[1:] = np.cumsum(lens)
    idx = rng.integers(0, len(pool), size=int(off[-1]))
    r32, l32 = pool[idx].astype(np.float32), Lp[idx].astype(np.float32)
    got = preint.scan_host(1, r32, l32, group_offsets=off)
    ref = preint.scan_host(1, r32.astype(np.float64), l32.astype(np.float64), group_offsets=off)
    assert got.dtype == np.float32
    worst = fp32_errors(got, ref)
    print({k: f"{v:.1e}" for k, v in worst.items()})
    for k, v in worst.items():
        assert v <= 1.2e-7, (k, v)           # 2 x the single float rounding of the output (2^-24 = 6e-8), the merge's bound
    assert_structure(got)


@pytest.mark.gpu
def test_layouts_and_multiwave_host_path(cuda):
    """Uniform and CSR layouts give the same bits; a batch of > 1 GB of records (ragged groups of 0 .. 60) gives the same bits through
    the host and the device entry points, and sampled groups match the numpy prefix folds.  A uniform call of n records takes
    2 ceil(log32 n) - 1 launches (here 5)."""
    from cpi_b200 import preint
    torch = cuda
    pool, Lp = _record_pool(n=4096, ns=20, first_window=77000)
    n = 5000
    rec, lin = torch.from_numpy(pool[np.arange(n * 5) % 4096]).cuda(), torch.from_numpy(Lp[np.arange(n * 5) % 4096]).cuda()
    before = capi.launch_count()
    u = preint.scan(1, rec[:n], lin[:n], group=1000)
    assert capi.launch_count() - before == 5
    c = preint.scan(1, rec[:n], lin[:n], group_offsets=torch.arange(0, n + 1, 1000, device="cuda"))
    torch.cuda.synchronize()
    assert torch.equal(u, c)
    del rec, lin, u, c
    rng = np.random.default_rng(12)
    lens = rng.integers(0, 61, size=15000); lens[:3] = [0, 1, 60]
    off = np.zeros(len(lens) + 1, dtype=np.int64); off[1:] = np.cumsum(lens)
    tot = int(off[-1])
    rec, lin = pool[np.arange(tot) % 4096], Lp[np.arange(tot) % 4096].copy()
    for g in range(0, len(lens), 3):
        lin[off[g]:off[g + 1]] = lin[off[g]]
    assert rec.nbytes > 1e9
    d = preint.scan(1, torch.from_numpy(rec).cuda(), torch.from_numpy(lin).cuda(), group_offsets=torch.from_numpy(off).cuda())
    torch.cuda.synchronize()
    d = d.cpu().numpy()
    host = preint.scan_host(1, rec, lin, group_offsets=off)
    assert np.array_equal(host, d)
    sel = np.unique(np.r_[0:8, len(lens) // 2:len(lens) // 2 + 8, len(lens) - 8:len(lens), np.arange(0, len(lens), 997)])
    rows = np.concatenate([np.arange(off[g], off[g + 1]) for g in sel])
    ref = np.concatenate([np.stack([r for _, r in sorted(prefix_folds(rec[off[g]:off[g + 1]], lin[off[g]:off[g + 1]]).items())])
                          for g in sel if off[g + 1] > off[g]])
    err = field_errors(d[rows], ref)
    print(len(sel), {k: f"{v:.1e}" for k, v in err.items()})
    for k in FIELDS + ("q", "DT", "P"):
        assert err[k] <= 1e-12, (k, err[k])
    assert_structure(d[rows])
