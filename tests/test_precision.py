"""Precision of the preintegration kernels against an extended-precision truth, regime by regime.

The truth is oracle/liboracle_ld.so: the plain-C restatement computed in long double (64-bit mantissa), with the reference's
small_w and dt == 0 branches taken on the fp64 values, so it is the same piecewise function the reference evaluates.  Against
it, each record field and each 3x3 block of P gets two relative errors per window: e_dev of the kernel, e_64 of the fp64
oracle.  The gate (parity.conditioned_gate) is e_dev <= K max(e_64, floor) + allowance: a kernel may be as inaccurate as the
fp64 computation is on that window (ill-conditioned windows: the small_w band, the threshold, large theta, long windows), times
K, and otherwise within K * floor of the truth.

CPU tests: the extended oracle is pinned to the golden records and to the fp64 oracle; the gate passes the fp64 oracle's own
records (default and analytic mode) and fails each of four injected subtle errors.  GPU tests: the stress batch (tests/stress.py)
through the device entry point, the host entry point, a continuation cut at ring / trio boundaries, imu_avg on the round-1
kernels and model 2 with analytic Jacobians (with and without imu_avg, device and host entry), models 1 and 2, fp64 and fp32.  Constants calibrated on one H100 80GB HBM3 (700 W power limit); DESIGN.md section 5 lists the measured worst ratios."""
import os
import subprocess

import numpy as np
import pytest

import stress
from parity import REC, compare_records, conditioned_gate, field_errors, imu_avg_inputs, window_band

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIGMAS = np.array([0.005, 4e-6, 0.01, 0.0002])
GOLDEN_CASES = ("cam200", "real200", "real100", "real400", "synth200", "edge")
MODES = [(1, 0), (1, 1), (2, 0), (2, 1), (2, 2), (2, 3)]

# fp64: worst measured e_dev / max(e_64, 1e-15) over every field, regime and path is 4.1 (P_22 of a gaps window, model 2,
# imu_avg); K = 8 keeps a 2x margin.  Injecting 1e-11 into one P block or one fp32 rounding anywhere fails it.
K64, FLOOR64 = 8.0, 1e-15
# fp32 storage variant: means and Jacobians are fp64 arithmetic rounded to float on output (2^-24 per element; a continuation
# call re-reads the rounded record, so a cut window carries up to four roundings).  P runs its RK4 in fp32: 1e-6 (the P
# contract) + 2e-11 per step, plus the window's fp64 conditioning carried to fp32 (2^29 e_64, the ratio of the unit
# roundoffs).  The round-1 imu_avg kernels keep the whole state in fp32: 4e-6 on the means, P 2e-5 + 5e-8 per step.
K32 = 8.0
U32 = 2.0 ** -24
COND32 = 2.0 ** 29
# Model 2 with analytic Jacobians runs on the round-1 kernels too, but keeps R, alpha, beta and the Jacobian state in fp64 (only
# the P tile and its stage slots are float): the output rounding on means and Jacobians, the round-1 allowance on P.
FP32_ALLOW = dict(device=(U32, 1e-6, 2e-11), host=(U32, 1e-6, 2e-11), cont=(4 * U32, 1e-6, 2e-11), avg=(4e-6, 2e-5, 5e-8),
                  ana=(U32, 2e-5, 5e-8), ana_avg=(U32, 2e-5, 5e-8))
# (model 2) flags of each path; "ana" / "ana_avg" are model 2 with CPI_FLAG_ANALYTIC_JACOBIANS (state_transition_jacobians = False)
PATH_FLAGS = dict(device=0, host=0, cont=0, avg=1, ana=2, ana_avg=3)


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


def gate(model, dtype, path, got, o64, truth, steps):
    """The gate of one (dtype, path) combination; returns (ratio, worst, failures) of parity.conditioned_gate."""
    if dtype == np.float64:
        return conditioned_gate(got, o64, truth, model, K64, FLOOR64)
    out, p0, p1 = FP32_ALLOW[path]
    e64 = field_errors(o64, truth, model)
    allow = {k: (p0 + p1 * steps + COND32 * e64[k]) if k.startswith("P_") else out for k in e64}
    return conditioned_gate(got, o64, truth, model, K32, FLOOR64, allowance=allow)


def report(label, ratio, tags):
    """Worst ratio per regime (and the field that sets it), printed for calibration."""
    rows = []
    for reg in stress.REGIMES:
        sel = tags == reg
        if sel.any():
            k = max(ratio, key=lambda f: ratio[f][sel].max())
            rows.append(f"{reg}={ratio[k][sel].max():.2f}({k})")
    print(label, " ".join(rows))


# ---------------------------------------------------------------------------------------------------------- CPU

# alpha, J_a, J_b, H_a and O_a come from the closed-form coefficients f1, f2, df1..df4 (CpiV1.h:196-238), which cancel like
# theta^3 .. theta^6 at small theta = |w_hat| dt: in fp64 they lose digits on every window, not only in the small_w band
# (1e-8 on J_a of ordinary cam200 windows; DESIGN.md section 5).  The other fields are well conditioned.
CLOSED_FORM_FIELDS = ("alpha", "J_a", "J_b", "H_a", "O_a")


@pytest.mark.parametrize("name", GOLDEN_CASES)
@pytest.mark.parametrize("model,flags", MODES)
def test_extended_oracle_matches_golden(oracle, oracle_ld, golden, name, model, flags):
    """The long-double build meets the north-star gates against the reference's own golden records (J_a at the band gate on
    every window: the golden J_a itself is only as good as fp64 makes it), and the golden records are as far from it as the
    fp64 oracle is (the conditioned gate, with the golden records in the device's place)."""
    G = golden["preint"]
    S, off = G[f"{name}/samples"], G[f"{name}/offsets"]
    if flags & 1:
        S, off = imu_avg_inputs(S, off)
    lin = G[f"{name}/lin"]
    ref = G[f"{name}/records_m{model}_f{flags}"]
    got = oracle_ld.preintegrate(model, S, lin, G["sigmas"], flags, offsets=off, nthreads=_threads())
    steps = np.diff(off) - (1 if flags & 1 else 0)
    # DT: the truth's sum of dt is exact to long double, the reference's is a running fp64 sum (a few ulps apart)
    assert np.all(np.abs(got[:, 19] - ref[:, 19]) <= 4e-16 * np.maximum(steps, 1) * np.abs(ref[:, 19]))
    got[:, 19] = ref[:, 19]
    compare_records(got, ref, model, in_band=np.ones(len(steps), dtype=bool), has_steps=steps > 0)
    if name != "edge":      # "edge" has a window ON the small_w threshold, where the reference's build takes the other branch
        o64 = oracle.preintegrate(model, S, lin, G["sigmas"], flags, offsets=off, nthreads=_threads())
        _, worst, bad = conditioned_gate(ref, o64, got, model, K64, FLOOR64)
        assert not bad, bad


@pytest.mark.parametrize("model,flags", MODES)
def test_extended_oracle_agrees_with_fp64_outside_the_band(oracle, oracle_ld, golden, model, flags):
    """On the golden inputs, windows that stay out of the ill-conditioned band agree with the fp64 oracle to 1e-13 in every
    well-conditioned field and every P block (the two builds compute the same function); the closed-form fields to 1e-7."""
    G = golden["preint"]
    worst = {}
    for name in GOLDEN_CASES:
        S, off = G[f"{name}/samples"], G[f"{name}/offsets"]
        if flags & 1:
            S, off = imu_avg_inputs(S, off)
        lin = G[f"{name}/lin"]
        a = oracle.preintegrate(model, S, lin, G["sigmas"], flags, offsets=off, nthreads=_threads())
        b = oracle_ld.preintegrate(model, S, lin, G["sigmas"], flags, offsets=off, nthreads=_threads())
        keep = ~window_band(S, off, lin)
        for k, e in field_errors(a[keep], b[keep], model).items():
            assert e.max() <= (1e-7 if k in CLOSED_FORM_FIELDS else 1e-13), (name, k, float(e.max()))
            worst[k] = max(worst.get(k, 0.0), float(e.max()))
    print(model, flags, "worst fp64 vs long double outside the band", {k: f"{v:.0e}" for k, v in worst.items() if v > 1e-14})


@pytest.fixture(scope="module")
def stress_cpu(oracle, oracle_ld):
    """Model 1 stress batch without the long windows, with both oracles."""
    S, off, L, tags = stress.make_batch(n_long=0)
    a = oracle.preintegrate(1, S, L, SIGMAS, 0, offsets=off, nthreads=_threads())
    b = oracle_ld.preintegrate(1, S, L, SIGMAS, 0, offsets=off, nthreads=_threads())
    return S, off, L, tags, a, b


def test_gate_passes_the_fp64_oracle(stress_cpu):
    S, off, L, tags, o64, truth = stress_cpu
    ratio, worst, bad = gate(1, np.float64, "device", o64, o64, truth, np.diff(off))
    assert not bad, bad
    report("fp64 oracle as device", ratio, tags)


def _must_fail(rec, o64, truth, off):
    _, _, bad = gate(1, np.float64, "device", rec, o64, truth, np.diff(off))
    assert bad, "the gate missed an injected error"
    return bad


def test_gate_fails_one_element_rounded_to_fp32(stress_cpu):
    S, off, L, tags, o64, truth = stress_cpu
    i = int(np.flatnonzero(tags == "rate200")[3])
    cols = [c for c in range(0, 65) if c != 19] + [65 + 1 + 15 * 1, 65 + 6 + 15 * 12]   # every mean / Jacobian element (not DT), two of P
    for col in cols:
        rec = o64.copy()
        v = rec[i, col]
        if np.float64(np.float32(v)) == v:
            continue
        rec[i, col] = np.float32(v)
        _must_fail(rec, o64, truth, off)


def test_gate_fails_one_P_block_scaled_by_1e_11(stress_cpu):
    S, off, L, tags, o64, truth = stress_cpu
    i = int(np.flatnonzero(tags == "rate200")[5])
    for I, J in ((0, 0), (2, 2), (1, 4), (4, 4)):
        rec = o64.copy()
        P = rec[i, 65:290].reshape(15, 15, order="F").copy()
        P[3 * I:3 * I + 3, 3 * J:3 * J + 3] *= 1 + 1e-11
        P[3 * J:3 * J + 3, 3 * I:3 * I + 3] = P[3 * I:3 * I + 3, 3 * J:3 * J + 3].T
        rec[i, 65:290] = P.reshape(-1, order="F")
        bad = _must_fail(rec, o64, truth, off)
        assert any(b.startswith(f"P_{min(I, J)}{max(I, J)}") for b in bad), bad


def test_gate_fails_a_J_a_column_perturbation_in_a_band_window(stress_cpu):
    """A band window where the fp64 computation of J_a is good to better than 1e-9: a 1e-7 relative change of one J_a column
    passes the north-star gate (flat 1e-6 in the band) and fails the conditioned gate."""
    S, off, L, tags, o64, truth = stress_cpu
    band = np.flatnonzero(tags == "band")
    e64 = field_errors(o64[band], truth[band], 1)["J_a"]
    i = int(band[np.argmin(e64)])
    assert e64.min() < 1e-7 / K64 / 4
    rec = o64.copy()
    J = rec[i, 29:38].reshape(3, 3, order="F")
    J[:, 1] += 1e-7 * np.linalg.norm(J) * np.array([1.0, -0.5, 0.25])
    rec[i, 29:38] = J.reshape(-1, order="F")
    compare_records(rec[i:i + 1], o64[i:i + 1], 1, in_band=np.array([True]))
    bad = _must_fail(rec, o64, truth, off)
    assert any(b.startswith("J_a") for b in bad), bad


@pytest.fixture(scope="module")
def stress_cpu_ana(oracle, oracle_ld):
    """Model 2 with analytic Jacobians on the stress batch without the long windows, with both oracles."""
    S, off, L, tags = stress.make_batch(n_long=0)
    a = oracle.preintegrate(2, S, L, SIGMAS, 2, offsets=off, nthreads=_threads())
    b = oracle_ld.preintegrate(2, S, L, SIGMAS, 2, offsets=off, nthreads=_threads())
    return S, off, L, tags, a, b


@pytest.mark.parametrize("field", ["O_a", "O_b"])
def test_gate_fails_one_analytic_O_element_rounded_to_fp32(stress_cpu_ana, field):
    """Analytic mode: the fp64 oracle passes the gate; one element of O_a or O_b rounded to fp32, where the rounding is below the
    north-star 1e-9 of the field (compare_records passes it), fails it."""
    S, off, L, tags, o64, truth = stress_cpu_ana
    _, _, bad = gate(2, np.float64, "device", o64, o64, truth, np.diff(off))
    assert not bad, bad
    a, b = REC[field]
    O = o64[:, a:b]
    d = np.abs(O.astype(np.float32).astype(np.float64) - O) / np.maximum(np.linalg.norm(O, axis=1, keepdims=True), 1e-300)
    d[d >= 5e-10] = 0.0                                              # keep it under the north-star gate
    i, j = np.unravel_index(int(np.argmax(d)), d.shape)
    assert d[i, j] > 1e-12
    rec = o64.copy()
    rec[i, a + j] = np.float32(rec[i, a + j])
    compare_records(rec[i:i + 1], o64[i:i + 1], 2, in_band=window_band(S, off, L)[i:i + 1])
    _, _, bad = gate(2, np.float64, "device", rec, o64, truth, np.diff(off))
    assert any(x.startswith(field) for x in bad), bad


# ---------------------------------------------------------------------------------------------------------- GPU

@pytest.fixture(scope="module")
def stress_batch():
    return stress.make_batch()


_truth_cache = {}


def _oracles(oracle, oracle_ld, model, dtype, flags, S, off, L):
    key = (model, np.dtype(dtype).name, flags)
    if key not in _truth_cache:
        Sx, Lx = S.astype(dtype).astype(np.float64), L.astype(dtype).astype(np.float64)
        if flags & 1:
            Sx, off = imu_avg_inputs(Sx, off)
        _truth_cache[key] = tuple(o.preintegrate(model, Sx, Lx, SIGMAS, flags, offsets=off, nthreads=_threads()) for o in (oracle, oracle_ld))
    return _truth_cache[key]


def _run_path(torch, preint, model, path, Sx, Lx, off, flags=0):
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    if flags & 1:
        Sx, off = imu_avg_inputs(Sx, off)
    if path == "host":
        return preint.preintegrate_host(model, Sx, Lx, SIGMAS, flags, offsets=off)
    if path == "cont":
        SA, oa, SB, ob = stress.split_for_continuation(Sx, off)
        out = preint.preintegrate(model, d(SA), d(Lx), SIGMAS, flags, offsets=d(oa))
        out = preint.preintegrate(model, d(SB), d(Lx), SIGMAS, flags, offsets=d(ob), continue_records=out)
    else:
        out = preint.preintegrate(model, d(Sx), d(Lx), SIGMAS, flags, offsets=d(off))
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["device", "host", "cont", "avg", "ana", "ana_avg"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("model", [1, 2])
def test_kernels_against_extended_oracle(cuda, oracle, oracle_ld, stress_batch, model, dtype, path):
    """Every stress regime through one entry point, held to the conditioned gate.  fp32: inputs rounded to float, both oracles
    run on the rounded inputs.  ana / ana_avg (model 2 with analytic Jacobians, without and with imu_avg): the device and the host
    entry, which give the same bits; model 1 is always analytic, so there the flag is dropped and the record is the one without it,
    bit for bit."""
    from cpi_b200 import preint
    S, off, L, tags = stress_batch
    Sx, Lx = S.astype(dtype), L.astype(dtype)
    flags = PATH_FLAGS[path] if model == 2 or not path.startswith("ana") else PATH_FLAGS[path] & 1
    entry = "host" if path == "host" else ("cont" if path == "cont" else "device")
    got = _run_path(cuda, preint, model, entry, Sx, Lx, off, flags)
    if path.startswith("ana"):
        host = _run_path(cuda, preint, model, "host", Sx, Lx, off, PATH_FLAGS[path])
        assert np.array_equal(host, got), "host and device entry differ"
        dev = _run_path(cuda, preint, model, "device", Sx, Lx, off, PATH_FLAGS[path])
        assert np.array_equal(dev, got), "the analytic flag changes the record"
    assert got.dtype == dtype
    P = got[:, 65:290].reshape(-1, 15, 15)
    assert np.array_equal(P, P.transpose(0, 2, 1)), "P is not exactly symmetric"
    o64, truth = _oracles(oracle, oracle_ld, model, dtype, flags, S, off, L)
    steps = np.maximum(np.diff(off), 1)
    gpath = path if model == 2 or not path.startswith("ana") else ("avg" if flags & 1 else "device")
    ratio, worst, bad = gate(model, dtype, gpath, got, o64, truth, steps)
    report(f"m{model} {np.dtype(dtype).name} {path}", ratio, tags)
    if dtype == np.float32:
        eP = np.max(np.stack([e for k, e in field_errors(got, truth, model).items() if k.startswith("P_")]), axis=0)
        ordinary = ~np.isin(tags, ("gaps", "threshold", "band", "fast"))
        print("  fp32 e_P against length:", {n: f"{eP[ordinary & (steps == n)].max():.1e}" for n in (2000, 10000) if np.any(steps == n)},
              "<=300:", f"{eP[ordinary & (steps <= 300)].max():.1e}", "gaps:", f"{eP[tags == 'gaps'].max():.1e}", "fast:", f"{eP[tags == 'fast'].max():.1e}")
    assert not bad, bad
