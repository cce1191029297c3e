#!/usr/bin/env python
"""Generate the committed golden fixtures from the UNMODIFIED reference (oracle/_ref/libcpi_ref.so).

Needs the rpng/cpi checkout (CPI_REFERENCE, by default /root/reference) for the datasets and for building oracle/_ref:
    make -C oracle ref && python tests/golden/make_golden.py
Writes
    tests/golden/imu_200hz_run00_head.dat   first 700 lines of GAZEBO_FREQ_200/rawdata_00/imu_data_meas.dat (input fixture)
    tests/golden/preint_golden.npz          inputs + reference CpiV1/CpiV2 records for every case below
    tests/golden/factor_golden.npz          states/records/lin + reference evaluateError e, H1, H2 (both models)
The reference ships no tests or golden vectors of its own (SURVEY.md section 4), so these are produced by running it.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.oracle import Reference, FLAG_IMU_AVG, FLAG_ANALYTIC_JACOBIANS  # noqa: E402
from cpi_b200 import synth  # noqa: E402

REF = os.path.join(os.environ.get("CPI_REFERENCE", "/root/reference"), "cpi_simulation")
HERE = os.path.dirname(os.path.abspath(__file__))


def csr(windows):
    offsets = np.zeros(len(windows) + 1, dtype=np.int64)
    for i, w in enumerate(windows):
        offsets[i + 1] = offsets[i] + len(w)
    S = np.concatenate([np.asarray(w, dtype=np.float64).reshape(-1, 7) for w in windows]) if windows else np.zeros((0, 7))
    return np.ascontiguousarray(S), offsets


def rand_lin(rng, n, identity_q=False):
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True); q[q[:, 3] < 0] *= -1
    if identity_q:
        q[:] = [0, 0, 0, 1]
    return np.concatenate([rng.normal(0, 1e-3, (n, 3)), rng.normal(0, 1e-2, (n, 3)), q, np.tile(synth.GRAVITY, (n, 1))], axis=1)


def stream(path):
    t, w, a = synth.parse_imu_dat(path)
    dt = np.diff(t)
    return np.concatenate([w[:-1], a[:-1], dt[:, None]], axis=1)


def main():
    R = Reference()
    rng = np.random.default_rng(20260924)
    cases = {}

    # ---- 1. camera-cut (ragged, ~20 steps) windows from the head of 200 Hz run 00: the reference's own usage
    src = f"{REF}/GAZEBO_FREQ_200/rawdata_00/imu_data_meas.dat"
    head = "".join(open(src).readlines()[:700])
    with open(os.path.join(HERE, "imu_200hz_run00_head.dat"), "w") as f:
        f.write(head)
    t, w, a = synth.parse_imu_dat(os.path.join(HERE, "imu_200hz_run00_head.dat"))
    cam = np.array([float(l.split()[-1]) for l in open(f"{REF}/GAZEBO_FREQ_200/rawdata_00/camera_data_meas.dat")]) * 1e-3
    cam = cam[(cam > t[0]) & (cam < t[-1])]
    cam = np.concatenate([cam[:25], [cam[25] + 0.0023]])     # last update falls between IMU stamps: partial tail step
    # the windows are cut by the REFERENCE's own driver loop (oracle/ref_shim.cpp:ref_replay_run -- std::deque handling, feed_IMU
    # arguments and erase order of GraphSolver_IMU.cpp:50-69), not by the product's cutter: cpi_cut_windows is tested against this
    lin_cam = rand_lin(rng, len(cam))
    S, off, _ = R.replay_run(1, t, w, a, cam, lin_cam, synth.SIGMAS, 0, imu_wait=0)
    assert len(off) - 1 == len(cam)
    cases["cam200"] = dict(samples=S, offsets=off, lin=lin_cam, cam_times=cam)
    # a second cut of the same stream WITH the reference's initialisation phase (imuWait queued readings, GraphSolver.cpp:264, 357)
    S_i, off_i, _ = R.replay_run(1, t, w, a, cam, lin_cam, synth.SIGMAS, 0, imu_wait=300)
    extra_init = dict(samples=S_i, offsets=off_i)

    # ---- 2. long windows cut at stride from the real streams
    for rate, ns, nwin in ((200, 200, 8), (100, 100, 4), (400, 400, 4)):
        st = stream(f"{REF}/GAZEBO_FREQ_{rate}/rawdata_0{rate // 100 % 10}/imu_data_meas.dat")
        starts = np.linspace(50, len(st) - ns - 1, nwin).astype(int)
        S, off = csr([st[s:s + ns] for s in starts])
        cases[f"real{rate}"] = dict(samples=S, offsets=off, lin=rand_lin(rng, nwin))

    # ---- 3. synthetic generator windows (bench distribution)
    S3, L3 = synth.make_windows(12, 200, rate=200.0)
    S, off = csr(list(S3))
    cases["synth200"] = dict(samples=S, offsets=off, lin=L3)

    # ---- 4. edge cases the datasets never hit
    base = S3[0].copy(); lin0 = L3[0].copy()
    bw = lin0[0:3]
    edge, elin = [], []

    def add(win, lin=lin0):
        edge.append(np.asarray(win)); elin.append(np.asarray(lin))

    wh = base[:, 0:3] - bw
    n = np.linalg.norm(wh, axis=1, keepdims=True)
    x = base.copy(); x[:, 0:3] = wh / n * np.linspace(1e-4, 0.008, len(x))[:, None] + bw; add(x)          # small_w branch (CpiV1.h:101)
    x = base.copy(); x[:, 0:3] = bw; add(x)                                                                 # w_hat == 0 exactly
    x = base.copy(); x[57, 6] = 0.0; x[58, 6] = 0.0; add(x)                                                 # dt == 0 steps (CpiV1.h:72)
    x = base.copy(); x[:, 0:3] = wh / n * np.linspace(0.0088, 0.049, len(x))[:, None] + bw; add(x)          # ill-conditioned band
    x = base.copy(); x[:, 0:3] = wh / n * 0.008726646 + bw; add(x)                                          # at the threshold
    add(np.zeros((0, 7)))                                                                                   # empty window
    add(base[:1])                                                                                           # single step
    x = base.copy(); x[:, 0:3] = wh * 4.0 + bw; add(x)                                                      # fast rotation (~10 rad/s)
    x = base[:50].copy(); x[:, 6] = 0.05; add(x)                                                            # long steps (20 Hz)
    x = base.copy(); add(x, np.concatenate([np.zeros(6), [0, 0, 0, 1], [0, 0, 0]]))                         # zero biases, g = 0
    x = base.copy(); x[:, 0:3] = 0.0; x[:, 3:6] = [0, 0, 9.8]; add(x, np.concatenate([np.zeros(6), [0, 0, 0, 1], synth.GRAVITY]))  # at rest
    S, off = csr(edge)
    cases["edge"] = dict(samples=S, offsets=off, lin=np.array(elin))

    out = {}
    for name, c in cases.items():
        for k, v in c.items():
            out[f"{name}/{k}"] = v
        n = len(c["offsets"]) - 1
        for model in (1, 2):
            for flags in ((0, FLAG_IMU_AVG) if model == 1 else (0, FLAG_IMU_AVG, FLAG_ANALYTIC_JACOBIANS, FLAG_IMU_AVG | FLAG_ANALYTIC_JACOBIANS)):
                S, off = c["samples"], c["offsets"]
                if flags & FLAG_IMU_AVG:
                    # imu_avg consumes one trailing entry per window: re-cut so that every window keeps >= 0 steps
                    # (not stored: tests/parity.py:imu_avg_inputs rebuilds this layout)
                    wins = [S[off[i]:off[i + 1]] for i in range(n)]
                    wins = [np.concatenate([w_, w_[-1:]]) if len(w_) else w_ for w_ in wins]
                    S, off = csr(wins)
                out[f"{name}/records_m{model}_f{flags}"] = R.preintegrate(model, S, c["lin"], synth.SIGMAS, flags, offsets=off)
    out["sigmas"] = synth.SIGMAS
    out["cam200_init300/samples"] = extra_init["samples"]; out["cam200_init300/offsets"] = extra_init["offsets"]
    np.savez_compressed(os.path.join(HERE, "preint_golden.npz"), **out)
    print("preint cases:", {k: len(v["offsets"]) - 1 for k, v in cases.items()})

    # ---- factor evaluation goldens: a perturbed chain over the synthetic + real200 records, both models
    fout = {}
    for model in (1, 2):
        Sx = np.concatenate([cases["synth200"]["samples"], cases["real200"]["samples"]])
        offx = np.concatenate([cases["synth200"]["offsets"], cases["real200"]["offsets"][1:] + cases["synth200"]["offsets"][-1]])
        linx = np.concatenate([cases["synth200"]["lin"], cases["real200"]["lin"]])
        rec = R.preintegrate(model, Sx, linx, synth.SIGMAS, 0, offsets=offx)
        X = synth.make_states(rec, linx, model)
        e, H1, H2 = R.factor_eval(model, X, rec, linx)
        # also non-chain index pairs
        ii = rng.integers(0, len(X), size=len(rec)); jj = rng.integers(0, len(X), size=len(rec))
        e2, H12, H22 = R.factor_eval(model, X, rec, linx, ii, jj)
        xi = rng.normal(0, 1e-2, (len(X), 15)); xi[0, 0:3] = 0.0
        fout.update({f"m{model}/states": X, f"m{model}/records": rec, f"m{model}/lin": linx, f"m{model}/e": e, f"m{model}/H1": H1,
                     f"m{model}/H2": H2, f"m{model}/idx_i": ii, f"m{model}/idx_j": jj, f"m{model}/e_idx": e2, f"m{model}/H1_idx": H12,
                     f"m{model}/H2_idx": H22, f"m{model}/xi": xi, f"m{model}/retracted": R.retract(X, xi)})
    np.savez_compressed(os.path.join(HERE, "factor_golden.npz"), **fout)
    for f in ("preint_golden.npz", "factor_golden.npz", "imu_200hz_run00_head.dat"):
        print(f, os.path.getsize(os.path.join(HERE, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()
