"""CPU tests of the host-side logic and of the C-ABI boundary (no compute calls: there is no GPU here)."""
import ctypes
import os
import re

import numpy as np
import pytest

from cpi_b200 import capi, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_and_binding_agree():
    """Every function declared in include/cpi_b200.h is bound in capi.SYMBOLS and vice versa."""
    hdr = open(os.path.join(ROOT, "include", "cpi_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(cpi_[a-z_0-9]+)\s*\(", hdr))
    assert declared == set(capi.SYMBOLS), declared ^ set(capi.SYMBOLS)
    consts = dict(re.findall(r"#define\s+(CPI_[A-Z0-9_]+)\s+(-?\d+)", hdr))
    assert int(consts["CPI_REC_V1_DOUBLES"]) == capi.REC_DOUBLES[1] and int(consts["CPI_REC_V2_DOUBLES"]) == capi.REC_DOUBLES[2]
    for name, key in (("q", "Q"), ("R", "R"), ("alpha", "ALPHA"), ("beta", "BETA"), ("DT", "DT"), ("J_q", "JQ"), ("J_a", "JA"), ("J_b", "JB"),
                      ("H_a", "HA"), ("H_b", "HB"), ("P", "P"), ("O_a", "OA"), ("O_b", "OB")):
        assert capi.REC[name][0] == int(consts["CPI_REC_" + key])


def test_library_loads_and_exports_every_symbol():
    """The built shared object loads (libcudart resolves without a GPU) and exports the whole ABI."""
    if not os.path.exists(capi.LIB_PATH):
        pytest.fail(f"{capi.LIB_PATH} not built: run `python __graft_entry__.py`")
    lib = capi.load()
    for name in capi.SYMBOLS:
        assert hasattr(lib, name), name
    assert lib.cpi_record_doubles(1) == 290 and lib.cpi_record_doubles(2) == 308 and lib.cpi_record_doubles(3) < 0
    assert b"sm_90a" in lib.cpi_version()


def test_argument_validation_without_gpu():
    """Bad arguments are rejected before any CUDA call, with a message."""
    lib = capi.load()
    rc = lib.cpi_preintegrate_batch(3, 64, 1, None, 1, None, None, None, 0, None, None)
    assert rc == -1 and b"model" in lib.cpi_last_error()
    rc = lib.cpi_preintegrate_batch(1, 16, 1, None, 1, None, None, None, 0, None, None)
    assert rc == -1 and b"dtype" in lib.cpi_last_error()
    assert lib.cpi_preintegrate_batch(1, 32, 0, None, 1, None, None, None, 0, None, None) == 0
    rc = lib.cpi_preintegrate_batch(1, 64, -5, None, 1, None, None, None, 0, None, None)
    assert rc == -1
    assert lib.cpi_preintegrate_batch(1, 64, 0, None, 1, None, None, None, 0, None, None) == 0      # empty batch is a no-op
    import numpy as np
    bad = np.array([0, 5, 3, 9], dtype=np.int64); buf = np.zeros(64)
    P = lambda a: ctypes.c_void_p(a.ctypes.data)
    rc = lib.cpi_preintegrate_batch_host(1, 64, 3, P(bad), 0, P(buf), P(buf), P(buf), 0, P(buf))
    assert rc == -1 and b"non-decreasing" in lib.cpi_last_error()
    rc = lib.cpi_imu_factor_eval_batch(1, 4, None, None, None, None, None, None, None, None, None)
    assert rc == -1 and b"null" in lib.cpi_last_error()


def test_missing_extension_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(capi, "_lib", None)
    monkeypatch.setattr(capi, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(ImportError, match="no CPU fallback"):
        capi.load()


def test_product_package_never_imports_oracle():
    pkg = os.path.join(ROOT, "cpi_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle|liboracle|libcpi_ref|#include\s+\".*oracle", src, flags=re.M), f


def test_synth_is_partition_independent():
    S, L = synth.make_windows(64, 20, first_window=1000)
    S2, L2 = synth.make_windows(20, 20, first_window=1030)
    assert np.array_equal(S[30:50], S2) and np.array_equal(L[30:50], L2)
    # bench batch stays out of the ill-conditioned band except for forced small / zero windows
    mag = np.linalg.norm(S[:, :, 0:3] - L[:, None, 0:3], axis=2)
    assert not np.any((mag >= 0.008726646) & (mag < 0.05))


def test_cut_windows_replays_reference_driver(golden):
    """cpi_cut_windows (C ABI, host) == the reference's driver loop.  The golden cam200 windows were cut by the REFERENCE's loop itself
    (oracle/ref_shim.cpp:ref_replay_run: std::deque handling, feed_IMU arguments and erase order of GraphSolver_IMU.cpp:50-69, message
    order of SimulationLoader.cpp:214-290), not by the product: bit-for-bit, incl. the partial tail step, the imu_times[0] rewrite and
    the initialisation phase that drops the first imuWait readings (GraphSolver.cpp:264, 357)."""
    G = golden["preint"]
    t, w, a = synth.parse_imu_dat(os.path.join(ROOT, "tests", "golden", "imu_200hz_run00_head.dat"))
    S, off = synth.cut_windows(t, w, a, G["cam200/cam_times"])
    assert np.array_equal(off, G["cam200/offsets"]) and np.array_equal(S, G["cam200/samples"])
    dts = np.array([S[off[i]:off[i + 1], 6].sum() for i in range(len(off) - 1)])
    cam = G["cam200/cam_times"]
    assert np.allclose(dts[1:], np.diff(cam), atol=1e-9)        # every window spans exactly camera-to-camera
    assert abs(S[off[-2]:off[-1], 6][-1] - 0.0023) < 1e-9       # the last window ends with a partial step
    Si, offi = synth.cut_windows(t, w, a, cam, imu_wait=300)
    assert np.array_equal(offi, G["cam200_init300/offsets"]) and np.array_equal(Si, G["cam200_init300/samples"]) and 0 < len(offi) < len(off)
    # error behaviour: unsorted stamps are rejected
    import pytest as _pt
    from cpi_b200.capi import CpiError
    with _pt.raises(CpiError):
        synth.cut_windows(t[::-1], w, a, cam)


def test_cut_windows_matches_reference_driver_on_random_streams(reference):
    """cpi_cut_windows against the reference's own driver loop (oracle/_ref: ref_replay_run) on random streams the shipped datasets never
    contain: jittered and duplicated IMU stamps (dt = 0 steps), camera frames before the first IMU reading, on an IMU stamp exactly,
    several frames inside one IMU interval, frames beyond the last reading, with and without the initialisation phase.  Bit for bit."""
    rng = np.random.default_rng(20260924)
    for case in range(40):
        n = int(rng.integers(5, 400))
        dt = rng.choice([0.0025, 0.005, 0.01]) * (1.0 + 0.3 * rng.standard_normal(n).clip(-2, 2))
        dt[rng.random(n) < 0.05] = 0.0                                   # duplicated stamps
        t = 10.0 + np.cumsum(np.abs(dt))
        w = rng.standard_normal((n, 3)); a = rng.standard_normal((n, 3)) + [0, 0, 9.8]
        nc = int(rng.integers(1, 40))
        cam = np.sort(rng.uniform(t[0] - 0.05, t[-1] + 0.05, nc))
        k = rng.integers(0, n, size=max(1, nc // 4))
        cam[rng.integers(0, nc, size=len(k))] = t[k]                      # frames exactly on an IMU stamp
        cam = np.sort(cam)
        if case % 5 == 0 and nc > 3:
            cam[1] = cam[0]                                               # two frames with the same stamp
        for wait in (0, 3, int(rng.integers(2, 60))):
            lin = np.zeros((nc, 13)); lin[:, 9] = 1.0; lin[:, 12] = 9.8
            Sr, offr, _ = reference.replay_run(1, t, w, a, cam, lin, synth.SIGMAS, imu_wait=wait)
            S, off = synth.cut_windows(t, w, a, cam, imu_wait=wait)
            assert np.array_equal(off, offr), (case, wait)
            assert np.array_equal(S, Sr), (case, wait)


def test_preint_staging_layout():
    from cpi_b200.preint import CpiV1, CpiV2
    c = CpiV1(0.005, 4e-6, 0.01, 0.0002)
    c.setLinearizationPoints([1, 2, 3], [4, 5, 6], [0, 0, 0, 1], [0, 0, 9.8])
    c.feed_IMU(1.0, 1.005, [1, 0, 0], [0, 0, 9.8], [2, 0, 0], [0, 0, 9.7])
    c.feed_IMU(1.005, 1.015, [2, 0, 0], [0, 0, 9.7])
    E = c._entries()
    assert E.shape == (2, 7) and np.allclose(E[:, 6], [0.005, 0.010]) and E[1, 0] == 2
    assert np.array_equal(c._lin(), [1, 2, 3, 4, 5, 6, 0, 0, 0, 1, 0, 0, 9.8])
    with pytest.raises(RuntimeError, match="finalize"):
        _ = c.alpha_tau
    c2 = CpiV2(0.005, 4e-6, 0.01, 0.0002, True)
    c2.state_transition_jacobians = False
    c2.feed_IMU(0.0, 0.005, [1, 0, 0], [0, 0, 9.8], [3, 0, 0], [0, 0, 9.0])
    E = c2._entries()
    assert E.shape == (3, 7) and E[1, 0] == 3 and E[1, 6] == 0 and c2._flags() == 3
