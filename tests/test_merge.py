"""Merging consecutive model-1 records (cpi_merge_records / _host, preint.merge / merge_host, CpiV1.mergeWith).

The truth for the merge formulas is ``fold`` below: a dense numpy left fold of the composition rules of DESIGN.md "Merging
records", itself checked against the oracle's one-shot records on the CPU.  The GPU tests compare the kernel with that fold, with
the device one-shot preintegration of the same windows, with the oracle and with the golden records of the reference."""
import ctypes

import numpy as np
import pytest

from cpi_b200 import capi, synth
from parity import REC, compare_records, fp32_errors, window_band

RD = 290
P = lambda a: ctypes.c_void_p(a.ctypes.data)


# ------------------------------------------------------------------------------------------------------------------
# numpy restatement of the merge (row-major 3x3 matrices; records are column-major)
# ------------------------------------------------------------------------------------------------------------------

def _skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def _exp_so3(w):
    th = np.linalg.norm(w)
    if th == 0:
        return np.eye(3)
    K = _skew(w)
    return np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th ** 2 * (K @ K)


def _rot_2_quat(R):
    """cpi_common.cuh rot_2_quat (JPL, q = [x y z w], w >= 0)."""
    T = np.trace(R)
    q = np.zeros(4)
    r00, r11, r22 = R[0, 0], R[1, 1], R[2, 2]
    if r00 >= T and r00 >= r11 and r00 >= r22:
        q[0] = np.sqrt((1 + 2 * r00 - T) / 4); s = 1 / (4 * q[0])
        q[1], q[2], q[3] = s * (R[0, 1] + R[1, 0]), s * (R[0, 2] + R[2, 0]), s * (R[1, 2] - R[2, 1])
    elif r11 >= T and r11 >= r00 and r11 >= r22:
        q[1] = np.sqrt((1 + 2 * r11 - T) / 4); s = 1 / (4 * q[1])
        q[0], q[2], q[3] = s * (R[0, 1] + R[1, 0]), s * (R[1, 2] + R[2, 1]), s * (R[2, 0] - R[0, 2])
    elif r22 >= T and r22 >= r00 and r22 >= r11:
        q[2] = np.sqrt((1 + 2 * r22 - T) / 4); s = 1 / (4 * q[2])
        q[0], q[1], q[3] = s * (R[0, 2] + R[2, 0]), s * (R[1, 2] + R[2, 1]), s * (R[0, 1] - R[1, 0])
    else:
        q[3] = np.sqrt((1 + T) / 4); s = 1 / (4 * q[3])
        q[0], q[1], q[2] = s * (R[1, 2] - R[2, 1]), s * (R[2, 0] - R[0, 2]), s * (R[0, 1] - R[1, 0])
    if q[3] < 0:
        q = -q
    return q / np.linalg.norm(q)


def _unpack(r):
    m = lambda name: r[REC[name][0]:REC[name][1]].reshape(3, 3, order="F").copy()
    return dict(R=m("R"), a=r[13:16].copy(), b=r[16:19].copy(), DT=float(r[19]), Jq=m("J_q"), Ja=m("J_a"), Jb=m("J_b"), Ha=m("H_a"),
                Hb=m("H_b"), P=r[65:290].reshape(15, 15, order="F").copy())


def _pack(d):
    r = np.zeros(RD)
    r[0:4] = _rot_2_quat(d["R"]); r[4:13] = d["R"].reshape(-1, order="F"); r[13:16] = d["a"]; r[16:19] = d["b"]; r[19] = d["DT"]
    for name, k in (("J_q", "Jq"), ("J_a", "Ja"), ("J_b", "Jb"), ("H_a", "Ha"), ("H_b", "Hb")):
        r[REC[name][0]:REC[name][1]] = d[k].reshape(-1, order="F")
    r[65:290] = d["P"].reshape(-1, order="F")
    return r


def zero_record():
    r = np.zeros(RD); r[3] = 1.0; r[4:13] = np.eye(3).reshape(-1)
    return r


def relinearise(r, lin_k, lin_0):
    """Record r (preintegrated at lin_k) moved to lin_0 to first order; Jacobians and P unchanged."""
    d = _unpack(r)
    dbw, dba = lin_0[0:3] - lin_k[0:3], lin_0[3:6] - lin_k[3:6]
    d["R"] = _exp_so3(d["Jq"] @ dbw) @ d["R"]
    d["a"] = d["a"] + d["Ja"] @ dbw + d["Ha"] @ dba
    d["b"] = d["b"] + d["Jb"] @ dbw + d["Hb"] @ dba
    return d


def merge2(d1, d2):
    """k -> m (+) m -> j, both at one linearisation point; dense 15x15 products for P."""
    R1, R2, dt2 = d1["R"], d2["R"], d2["DT"]
    I3, Z3 = np.eye(3), np.zeros((3, 3))
    out = dict(R=R2 @ R1, DT=d1["DT"] + dt2, b=d1["b"] + R1.T @ d2["b"], a=d1["a"] + d1["b"] * dt2 + R1.T @ d2["a"],
               Jq=R2 @ d1["Jq"] + d2["Jq"], Hb=d1["Hb"] + R1.T @ d2["Hb"], Ha=d1["Ha"] + d1["Hb"] * dt2 + R1.T @ d2["Ha"],
               Jb=d1["Jb"] + R1.T @ (_skew(d2["b"]) @ d1["Jq"] + d2["Jb"]),
               Ja=d1["Ja"] + d1["Jb"] * dt2 + R1.T @ (_skew(d2["a"]) @ d1["Jq"] + d2["Ja"]))
    Phi2 = np.block([[R2, -d2["Jq"], Z3, Z3, Z3],
                     [Z3, I3, Z3, Z3, Z3],
                     [-_skew(d2["b"]), d2["Jb"], I3, d2["Hb"], Z3],
                     [Z3, Z3, Z3, I3, Z3],
                     [-_skew(d2["a"]), d2["Ja"], dt2 * I3, d2["Ha"], I3]])
    T = np.zeros((15, 15))
    for k, B in enumerate((I3, I3, R1.T, I3, R1.T)):
        T[3 * k:3 * k + 3, 3 * k:3 * k + 3] = B
    Phi = T @ Phi2 @ T.T
    out["P"] = Phi @ d1["P"] @ Phi.T + T @ d2["P"] @ T.T
    return out


def fold(records, lins):
    """Left fold of a group: every later record moved to the first one's linearisation point, then composed in order."""
    if len(records) == 0:
        return zero_record()
    if len(records) == 1:
        return records[0].copy()
    acc = _unpack(records[0])
    for r, l in zip(records[1:], lins[1:]):
        acc = merge2(acc, relinearise(r, l, lins[0]))
    return _pack(acc)


FIELDS = ("R", "alpha", "beta", "J_q", "J_a", "J_b", "H_a", "H_b")


def field_errors(got, ref):
    """Worst relative (Frobenius, per record) error of every field; q up to sign; P whole-matrix."""
    got = np.asarray(got, dtype=np.float64); ref = np.asarray(ref, dtype=np.float64)
    out = {}
    for k in FIELDS + ("P", "DT"):
        a, b = REC[k]
        num = np.linalg.norm(got[:, a:b] - ref[:, a:b], axis=1); den = np.maximum(np.linalg.norm(ref[:, a:b], axis=1), 1e-300)
        out[k] = float(np.max(num / den))
    eq = np.minimum(np.linalg.norm(got[:, 0:4] - ref[:, 0:4], axis=1), np.linalg.norm(got[:, 0:4] + ref[:, 0:4], axis=1))
    out["q"] = float(np.max(eq))
    return out


def with_ref_DT(got, ref, tol=1e-14):
    """DT of a merged record is a sum of segment sums: it may differ from the one-shot's sequential sum in the last bits, more than
    compare_records' 2-ulp DT gate allows.  Check it here at tol and hand compare_records a copy carrying the reference DT."""
    got = np.array(got, copy=True)
    assert np.all(np.abs(got[:, 19] - ref[:, 19]) <= tol * np.abs(ref[:, 19])), "DT"
    got[:, 19] = ref[:, 19]
    return got


def split_windows(S, L, cuts):
    """Windows S[n, ns, 7] cut at cuts[w] (sorted, in [0, ns]) -> CSR segments (entries, offsets) and lin per segment."""
    n, ns = S.shape[0], S.shape[1]
    bounds = [np.concatenate([[0], c, [ns]]) for c in cuts]
    lens = np.concatenate([np.diff(b) for b in bounds])
    off = np.zeros(len(lens) + 1, dtype=np.int64); off[1:] = np.cumsum(lens)
    nseg = len(bounds[0]) - 1
    return np.ascontiguousarray(S.reshape(-1, 7)), off, np.repeat(L, nseg, axis=0), nseg


# ------------------------------------------------------------------------------------------------------------------
# CPU: argument checks of the C ABI (no device needed) and the numpy restatement against the oracle
# ------------------------------------------------------------------------------------------------------------------

def test_merge_argument_validation_without_gpu():
    lib = capi.load()
    buf = np.zeros(4 * RD); lin = np.zeros(4 * 13); out = np.zeros(4 * RD)
    for fn, extra in ((lib.cpi_merge_records, (None,)), (lib.cpi_merge_records_host, ())):
        rc = fn(2, 64, 2, None, 2, P(buf), P(lin), P(out), *extra)
        assert rc == -1 and b"model 2" in lib.cpi_last_error()
        rc = fn(3, 64, 2, None, 2, P(buf), P(lin), P(out), *extra)
        assert rc == -1 and b"model" in lib.cpi_last_error()
        rc = fn(1, 16, 2, None, 2, P(buf), P(lin), P(out), *extra)
        assert rc == -1 and b"dtype" in lib.cpi_last_error()
        rc = fn(1, 64, -1, None, 2, P(buf), P(lin), P(out), *extra)
        assert rc == -1 and b"negative" in lib.cpi_last_error()
        rc = fn(1, 64, 2, None, -2, P(buf), P(lin), P(out), *extra)
        assert rc == -1 and b"negative" in lib.cpi_last_error()
        # NULL pointers with n_groups > 0
        for args in ((None, P(lin), P(out)), (P(buf), None, P(out)), (P(buf), P(lin), None)):
            rc = fn(1, 64, 2, None, 2, *args, *extra)
            assert rc == -1 and b"null" in lib.cpi_last_error()
        # n_groups = 0 is a no-op, whatever the pointers
        assert fn(1, 64, 0, None, 2, None, None, None, *extra) == 0
        assert fn(1, 32, 0, None, 0, None, None, None, *extra) == 0
        # out must not alias records
        rc = fn(1, 64, 2, None, 2, P(buf), P(lin), P(buf), *extra)
        assert rc == -1 and b"overlap" in lib.cpi_last_error()
    # host offsets: decreasing, negative start, past any possible record count
    for offs, word in (([0, 3, 2, 4], b"non-decreasing"), ([-1, 1, 2, 4], b"out of range"), ([0, 1, 2, 1 << 61], b"out of range")):
        o = np.array(offs, dtype=np.int64)
        rc = lib.cpi_merge_records_host(1, 64, 3, P(o), 0, P(buf), P(lin), P(out))
        assert rc == -1 and word in lib.cpi_last_error(), (offs, lib.cpi_last_error())
    # Python layer: layout errors are caught before the library is called
    from cpi_b200 import preint
    with pytest.raises(ValueError):
        preint.merge_host(1, buf.reshape(4, RD), lin.reshape(4, 13))
    with pytest.raises(ValueError):
        preint.merge_host(1, buf.reshape(4, RD), lin.reshape(4, 13), group=3)
    with pytest.raises(capi.CpiError, match="model 2"):
        preint.merge_host(2, np.zeros((2, 308)), np.zeros((2, 13)), group=2)
    assert preint.merge_host(1, np.zeros((0, RD)), np.zeros((0, 13)), group_offsets=np.zeros(1, dtype=np.int64)).shape == (0, RD)


def test_numpy_fold_matches_oracle_one_shot(oracle):
    """The composition rules, on the CPU: windows preintegrated by the oracle in segments and folded in numpy give the oracle's one-shot
    record (means and Jacobians to rounding, P to the RK4 truncation); a lin offset on the later segments leaves a second-order error."""
    n, ns = 6, 200
    S, L = synth.make_windows(n, ns, rate=200.0, first_window=880, special=False)
    one = oracle.preintegrate(1, S, L, synth.SIGMAS, 0, ns=ns)
    cuts = [np.array([83]), np.array([20, 20, 21, 150])]
    for c in cuts:
        Sx, off, Ls, nseg = split_windows(S, L, [c] * n)
        seg = oracle.preintegrate(1, Sx, Ls, synth.SIGMAS, 0, offsets=off)
        got = np.stack([fold(seg[w * nseg:(w + 1) * nseg], Ls[w * nseg:(w + 1) * nseg]) for w in range(n)])
        err = field_errors(got, one)
        print(len(c), {k: f"{v:.1e}" for k, v in err.items()})
        assert max(err[k] for k in FIELDS) <= 1e-13 and err["q"] <= 1e-13 and err["P"] <= 1e-8 and err["DT"] <= 1e-14
    # bias mismatch: second order in the offset for the means
    errs = []
    for scale in (1.0, 0.5):
        Sx, off, Ls, nseg = split_windows(S, L, [np.array([83])] * n)
        Lm = Ls.copy()
        Lm[1::2, 0:3] += scale * np.array([2e-3, -1e-3, 1.5e-3]); Lm[1::2, 3:6] += scale * np.array([2e-2, 1e-2, -1e-2])
        seg = oracle.preintegrate(1, Sx, Lm, synth.SIGMAS, 0, offsets=off)
        got = np.stack([fold(seg[2 * w:2 * w + 2], Lm[2 * w:2 * w + 2]) for w in range(n)])
        errs.append(field_errors(got, one))
    for k in ("R", "alpha", "beta"):
        assert 3.0 <= errs[0][k] / errs[1][k] <= 5.0, (k, errs[0][k], errs[1][k])


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------

def _device_split_merge(torch, S, L, cuts, csr_groups):
    """Preintegrate the segments in one CSR call and merge per window in one call; returns (merged, segment records) on the host."""
    from cpi_b200 import preint
    Sx, off, Ls, nseg = split_windows(S, L, cuts)
    dLs = torch.from_numpy(Ls).cuda()
    seg = preint.preintegrate(1, torch.from_numpy(Sx).cuda(), dLs, synth.SIGMAS, 0, offsets=torch.from_numpy(off).cuda())
    if csr_groups:
        goff = torch.arange(0, S.shape[0] * nseg + 1, nseg, dtype=torch.int64, device="cuda")
        m = preint.merge(1, seg, dLs, group_offsets=goff)
    else:
        m = preint.merge(1, seg, dLs, group=nseg)
    torch.cuda.synchronize()
    return m.cpu().numpy(), seg.cpu().numpy(), Ls


def _random_cuts(rng, n, ns, nseg):
    cuts = np.sort(rng.integers(0, ns + 1, size=(n, nseg - 1)), axis=1)
    cuts[0] = np.r_[np.zeros(nseg - 2, dtype=np.int64), [1]] if nseg > 2 else [0]          # empty segments, then a 1-sample one
    cuts[1] = np.r_[[ns - 1], np.full(nseg - 2, ns)] if nseg > 2 else [ns]                   # a 1-sample segment, then empty ones
    if nseg > 3:
        cuts[2, :3] = [10, 11, 11]                                                            # 1 sample, 0 samples
    return np.sort(cuts, axis=1)


@pytest.mark.gpu
def test_split_and_merge_matches_oracle_and_one_shot(cuda, oracle):
    """~2000 windows of 200 samples (incl. the forced small_w / zero-w_hat / dt = 0 windows) cut into S segments (incl. segments of 0
    and 1 samples), one CSR preintegration of the segments, one merge call: against the oracle's whole-window records (standard gates)
    and the device one-shot (1e-12 on the means and Jacobians; P within the RK4 truncation of the window)."""
    from cpi_b200 import preint
    torch = cuda
    n, ns = 2000, 200
    S, L = synth.make_windows(n, ns, rate=200.0, first_window=60000)
    one = preint.preintegrate(1, torch.from_numpy(S).cuda(), torch.from_numpy(L).cuda(), synth.SIGMAS, 0, ns=ns)
    torch.cuda.synchronize()
    one = one.cpu().numpy()
    mag = np.linalg.norm(S[:, :, 0:3] - L[:, None, 0:3], axis=2)
    special = np.where((mag.max(axis=1) < 0.0088) | (S[:, :, 6].min(axis=1) == 0))[0]
    assert len(special) >= 3
    sel = np.unique(np.r_[0:48, n - 16:n, special[:40]])
    ref = oracle.preintegrate(1, S[sel], L[sel], synth.SIGMAS, 0, ns=ns, nthreads=8)
    band = window_band(S[sel].reshape(-1, 7), np.arange(len(sel) + 1, dtype=np.int64) * ns, L[sel])
    rng = np.random.default_rng(8)
    for nseg in (2, 3, 8, 64):
        got, _, _ = _device_split_merge(torch, S, L, _random_cuts(rng, n, ns, nseg), csr_groups=nseg in (3, 64))
        worst = compare_records(with_ref_DT(got[sel], ref), ref, 1, in_band=band)
        err = field_errors(got, one)
        print(f"S={nseg}: vs oracle", {k: f"{v:.1e}" for k, v in worst.items()}, "vs one-shot", {k: f"{v:.1e}" for k, v in err.items()})
        for k in FIELDS + ("q", "DT"):
            assert err[k] <= 1e-12, (nseg, k, err[k])
        assert err["P"] <= 1e-7, (nseg, err["P"])
        P_ = got[:, 65:290].reshape(n, 15, 15)
        assert np.array_equal(P_, P_.transpose(0, 2, 1)) and np.all(P_[:, 0:6, 9:12] == 0)


def _golden_split(S, off, avg):
    """Every golden window split at its middle sample; imu_avg: each segment's trailing entry = the next segment's first entry."""
    segs = []
    for i in range(len(off) - 1):
        s = S[off[i]:off[i + 1]]
        m = len(s) // 2
        if not avg:
            segs += [s[:m], s[m:]]
        else:
            segs += [np.concatenate([s[:m], s[m:m + 1]]) if m > 0 else s[:0], np.concatenate([s[m:], s[-1:]]) if len(s) else s[:0]]
    o = np.zeros(len(segs) + 1, dtype=np.int64); o[1:] = np.cumsum([len(x) for x in segs])
    return np.concatenate(segs).reshape(-1, 7), o


@pytest.mark.gpu
@pytest.mark.parametrize("name", ("real100", "real200", "real400", "cam200"))
def test_golden_windows_split_and_merged(cuda, golden, name):
    from cpi_b200 import preint
    G = golden["preint"]
    S, off, lin = G[f"{name}/samples"], G[f"{name}/offsets"], G[f"{name}/lin"]
    steps = np.diff(off)
    Ls = np.repeat(lin, 2, axis=0)
    for flags in (0, 1):
        Sg, og = _golden_split(S, off, bool(flags))
        seg = preint.preintegrate_host(1, Sg, Ls, G["sigmas"], flags, offsets=og)
        got = preint.merge_host(1, seg, Ls, group=2)
        ref = G[f"{name}/records_m1_f{flags}"]
        worst = compare_records(with_ref_DT(got, ref), ref, 1, in_band=window_band(S, off, lin), has_steps=steps > 0)
        print(name, flags, {k: f"{v:.1e}" for k, v in worst.items()})


def _record_pool(n=512, ns=30, first_window=70000):
    """Real records of ragged windows (0..ns samples, so some are zero-step records) and their lin."""
    from cpi_b200 import preint
    S, L = synth.make_windows(n, ns, rate=200.0, first_window=first_window)
    rng = np.random.default_rng(first_window)
    lens = rng.integers(0, ns + 1, size=n); lens[:3] = [0, 1, ns]
    off = np.zeros(n + 1, dtype=np.int64); off[1:] = np.cumsum(lens)
    Sx = np.concatenate([S[i, :lens[i]] for i in range(n)])
    return preint.preintegrate_host(1, Sx, L, synth.SIGMAS, 0, offsets=off), L


@pytest.mark.gpu
def test_formula_pinning_against_numpy_fold(cuda):
    """Random groups of 1..70 records, at one linearisation point per group or at a different one per record: the device result is the
    numpy left fold of the formulas to <= 1e-12 per field (the device reduces by a pairwise tree)."""
    from cpi_b200 import preint
    pool, Lp = _record_pool()
    rng = np.random.default_rng(3)
    lens = rng.integers(1, 71, size=60); lens[:4] = [1, 2, 17, 70]
    idx = rng.integers(0, len(pool), size=lens.sum())
    rec = pool[idx]
    lin = Lp[idx].copy()
    off = np.zeros(len(lens) + 1, dtype=np.int64); off[1:] = np.cumsum(lens)
    for g in range(0, len(lens), 2):                    # even groups: one linearisation point for the whole group
        lin[off[g]:off[g + 1]] = lin[off[g]]
    got = preint.merge_host(1, rec, lin, group_offsets=off)
    ref = np.stack([fold(rec[off[g]:off[g + 1]], lin[off[g]:off[g + 1]]) for g in range(len(lens))])
    err = field_errors(got, ref)
    print({k: f"{v:.1e}" for k, v in err.items()})
    for k in FIELDS + ("q", "DT", "P"):
        assert err[k] <= 1e-12, (k, err[k])
    # uniform groups of every width the launcher distinguishes, through the device entry point
    torch = cuda
    for w in (2, 3, 5, 9, 33):
        n = 40
        r = pool[rng.integers(0, len(pool), size=n * w)]; l = Lp[rng.integers(0, len(pool), size=n * w)]
        d = preint.merge(1, torch.from_numpy(r).cuda(), torch.from_numpy(l).cuda(), group=w)
        torch.cuda.synchronize()
        ref = np.stack([fold(r[g * w:(g + 1) * w], l[g * w:(g + 1) * w]) for g in range(n)])
        err = field_errors(d.cpu().numpy(), ref)
        assert max(err.values()) <= 1e-12, (w, err)


@pytest.mark.gpu
def test_identity_and_associativity(cuda):
    from cpi_b200 import preint
    pool, Lp = _record_pool(n=64, first_window=71000)
    r = pool[10:12]; Z = zero_record()
    lin = np.repeat(Lp[10:11], 2, axis=0)
    for pair, keep in (((Z, r[0]), r[0]), ((r[1], Z), r[1])):
        got = preint.merge_host(1, np.stack(pair), lin, group=2)[0]
        assert np.array_equal(got, keep)
    # a group of one is a bitwise copy (also in fp32), an empty group is the zero-step record
    off = np.array([0, 1, 1, 2], dtype=np.int64)
    got = preint.merge_host(1, r, Lp[10:12], group_offsets=off)
    assert np.array_equal(got[0], r[0]) and np.array_equal(got[1], Z) and np.array_equal(got[2], r[1])
    r32 = r.astype(np.float32)
    got = preint.merge_host(1, r32, Lp[10:12].astype(np.float32), group=1)
    assert got.dtype == np.float32 and np.array_equal(got, r32)
    # one merge of a group of 8 == three calls merging pairs of pairs
    r8, l8 = pool[20:28], np.repeat(Lp[20:21], 8, axis=0)
    one = preint.merge_host(1, r8, l8, group=8)
    a = preint.merge_host(1, r8, l8, group=2)
    b = preint.merge_host(1, a, l8[:4], group=2)
    c = preint.merge_host(1, b, l8[:2], group=2)
    err = field_errors(c, one)
    print({k: f"{v:.1e}" for k, v in err.items()})
    assert max(err.values()) <= 1e-12, err


@pytest.mark.gpu
def test_bias_mismatch_is_second_order(cuda):
    """Second segment preintegrated at lin + db: the merge moves it back to first order, so the R / alpha / beta errors against the one-shot
    record at the first lin shrink by 4 when db halves; db = 0 is the equal-lin merge (1e-12 of the one-shot)."""
    from cpi_b200 import preint
    torch = cuda
    n, ns = 400, 200
    S, L = synth.make_windows(n, ns, rate=200.0, first_window=62000, special=False)
    one = preint.preintegrate_host(1, S, L, synth.SIGMAS, 0, ns=ns)
    Sx, off, Ls, nseg = split_windows(S, L, [np.array([83])] * n)
    errs = []
    for scale in (1.0, 0.5, 0.0):
        Lm = Ls.copy()
        Lm[1::2, 0:3] += scale * np.array([2e-3, -1e-3, 1.5e-3]); Lm[1::2, 3:6] += scale * np.array([2e-2, 1e-2, -1e-2])
        dL = torch.from_numpy(Lm).cuda()
        seg = preint.preintegrate(1, torch.from_numpy(Sx).cuda(), dL, synth.SIGMAS, 0, offsets=torch.from_numpy(off).cuda())
        got = preint.merge(1, seg, dL, group=2)
        torch.cuda.synchronize()
        errs.append(field_errors(got.cpu().numpy(), one))
    print({k: (f"{errs[0][k]:.2e}", f"{errs[1][k]:.2e}") for k in ("R", "alpha", "beta")})
    for k in ("R", "alpha", "beta"):
        assert 3.0 <= errs[0][k] / errs[1][k] <= 5.0, (k, errs[0][k], errs[1][k])
    assert max(errs[2][k] for k in FIELDS) <= 1e-12 and errs[2]["P"] <= 1e-7


@pytest.mark.gpu
def test_factor_side_of_a_merged_record(cuda):
    """predict(x_k, merged) == predict(predict(x_k, r1), r2); the merged factor between x_k and that x_k+2 has a zero residual."""
    from cpi_b200 import factor, preint
    n, ns = 300, 120
    S, L = synth.make_windows(n, ns, rate=200.0, first_window=63000, special=False)
    Sx, off, Ls, nseg = split_windows(S, L, [np.array([50])] * n)
    seg = preint.preintegrate_host(1, Sx, Ls, synth.SIGMAS, 0, offsets=off)
    merged = preint.merge_host(1, seg, Ls, group=2)
    X = synth.make_states(merged, L, 1)[:n]
    X[:, 4:7], X[:, 10:13] = L[:, 0:3], L[:, 3:6]       # biases at the linearisation point: the factor's bias-correction terms vanish
    X[:, 13:16] = 0.0                                   # positions at the origin (the chain drifts to ~1e4 m, whose rounding would dominate)
    x1 =factor.predict_state(1, X, seg[0::2], L)
    x2 = factor.predict_state(1, x1, seg[1::2], L)
    xm = factor.predict_state(1, X, merged, L)
    err = np.max(np.abs(xm - x2) / np.maximum(1.0, np.abs(x2)))
    print("predict", err)
    assert err <= 1e-12
    st = np.empty((2 * n, 16)); st[0::2] = X; st[1::2] = xm
    e, _, _ = factor.factor_eval_host(1, st, merged, L, np.arange(0, 2 * n, 2), np.arange(1, 2 * n, 2))
    print("residual", np.max(np.abs(e)))
    assert np.max(np.abs(e)) <= 1e-11


@pytest.mark.gpu
def test_fp32_storage(cuda):
    """Float records merge in fp64 arithmetic: the result is the fp64 merge of the same float-rounded records, rounded once."""
    from cpi_b200 import preint
    pool, Lp = _record_pool(n=2000, first_window=72000)
    rng = np.random.default_rng(4)
    lens = rng.integers(0, 20, size=500)
    off = np.zeros(501, dtype=np.int64); off[1:] = np.cumsum(lens)
    idx = rng.integers(0, len(pool), size=lens.sum())
    r32, l32 = pool[idx].astype(np.float32), Lp[idx].astype(np.float32)
    got = preint.merge_host(1, r32, l32, group_offsets=off)
    ref = preint.merge_host(1, r32.astype(np.float64), l32.astype(np.float64), group_offsets=off)
    assert got.dtype == np.float32 and np.all(np.isfinite(got))
    worst = fp32_errors(got, ref)
    print({k: f"{v:.1e}" for k, v in worst.items()})
    for k, v in worst.items():
        assert v <= 1.2e-7, (k, v)           # 2 x the single float rounding of the output (2^-24 = 6e-8), the observed bound
    g = got.astype(np.float64)[:, 65:290].reshape(-1, 15, 15)
    assert np.array_equal(g, g.transpose(0, 2, 1)) and np.all(g[:, 0:6, 9:12] == 0)


@pytest.mark.gpu
def test_multiwave_ragged_groups_and_host_path(cuda):
    """20k groups of 0..40 records (~0.9 GB of input tiled from 4096 distinct records), more than one wave of CTAs: sampled groups
    against the numpy fold, and the host entry point bit for bit against the device one."""
    from cpi_b200 import preint
    torch = cuda
    pool, Lp = _record_pool(n=4096, ns=20, first_window=73000)
    rng = np.random.default_rng(20)
    n = 20000
    lens = rng.integers(0, 41, size=n); lens[:4] = [0, 1, 40, 2]
    off = np.zeros(n + 1, dtype=np.int64); off[1:] = np.cumsum(lens)
    tot = int(off[-1])
    idx = np.arange(tot) % len(pool)
    rec = pool[idx]; lin = Lp[idx]
    for g in range(0, n, 3):                            # every third group at one linearisation point
        lin[off[g]:off[g + 1]] = lin[off[g]]
    assert rec.nbytes > 800e6
    d = preint.merge(1, torch.from_numpy(rec).cuda(), torch.from_numpy(lin).cuda(), group_offsets=torch.from_numpy(off).cuda())
    torch.cuda.synchronize()
    d = d.cpu().numpy()
    sel = np.unique(np.r_[0:64, n // 2:n // 2 + 64, n - 64:n, np.arange(0, n, 401), np.where(lens == 40)[0][:10]])
    ref = np.stack([fold(rec[off[g]:off[g + 1]], lin[off[g]:off[g + 1]]) for g in sel])
    err = field_errors(d[sel], ref)
    print(len(sel), {k: f"{v:.1e}" for k, v in err.items()})
    for k in FIELDS + ("q", "DT", "P"):
        assert err[k] <= 1e-12, (k, err[k])
    assert np.all(np.isfinite(d))
    host = preint.merge_host(1, rec, lin, group_offsets=off)
    assert np.array_equal(host, d)


@pytest.mark.gpu
def test_cpiv1_merge_with(cuda, golden):
    """CpiV1.mergeWith on finalised objects == the batch call on their records."""
    from cpi_b200.preint import CpiV1
    G = golden["preint"]
    S, off, lin = G["cam200/samples"], G["cam200/offsets"], G["cam200/lin"]
    sg = G["sigmas"]
    w = int(np.argmax(np.diff(off)))
    s = S[off[w]:off[w + 1]]
    m = len(s) // 2
    objs = []
    for part, l in ((s[:m], lin[w]), (s[m:], lin[w] + np.r_[1e-4, 0, 0, 0, 1e-3, 0, np.zeros(7)])):
        c = CpiV1(*sg)
        c.setLinearizationPoints(l[0:3], l[3:6], l[6:10], l[10:13])
        t = 0.0
        for row in part:
            c.feed_IMU(t, t + row[6], row[0:3], row[3:6])
            t += row[6]
        objs.append(c.finalize())
    a, b = objs
    from cpi_b200 import preint
    ref = preint.merge_host(1, np.stack([a.record(), b.record()]), np.stack([a._lin(), b._lin()]), group=2)[0]
    a.mergeWith(b)
    assert np.array_equal(a.record(), ref)
    assert np.array_equal(a.R_k2tau, ref[4:13].reshape(3, 3, order="F")) and a.DT == ref[19]
    assert np.array_equal(a.P_meas, ref[65:290].reshape(15, 15, order="F"))
