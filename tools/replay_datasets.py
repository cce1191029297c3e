#!/usr/bin/env python
"""Replay every camera frame of the reference's shipped Monte-Carlo runs (50 runs x {100, 200, 400} Hz) through the product path --
cpi_cut_windows (host window builder) + K1 / K2 on the GPU -- and compare EVERY window with the unmodified reference driven by its own
driver loop (oracle/ref_shim.cpp:ref_replay_run).  SURVEY.md 8f rank 3.

    python tools/pack_datasets.py                       (where an rpng/cpi checkout exists)
    python tools/replay_datasets.py                     (GPU: needs tests/golden/_datasets/*.npz and oracle/_ref/libcpi_ref.so)

Prints a JSON report on its last line: per rate and model the number of windows, whether the cut is bit-identical to the
reference's, the worst error per record field, and the windows/s of the real-data batch.  The linearisation points (biases, q_k,
gravity) come from a seeded generator: the reference takes them from its state estimate, which needs the vision factors (GTSAM)."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
IMU_WAIT = {100: 300, 200: 900, 400: 2300}           # launch/synthetic_test.launch:31-33


def main():
    import torch
    from cpi_b200 import preint, synth
    from oracle.oracle import Reference
    from parity import compare_records, window_band
    R = Reference()
    rng = np.random.default_rng(20260924)
    report = {"what": "all camera frames of the shipped runs; reference = unmodified CpiV1/CpiV2 driven by ref_replay_run", "rates": {}}
    for rate in (100, 200, 400):
        path = os.path.join(ROOT, "tests", "golden", "_datasets", f"replay_{rate}.npz")
        if not os.path.exists(path):
            print("missing", path, file=sys.stderr); continue
        D = np.load(path)
        runs = sorted({k.split("/")[0] for k in D.files})
        Ss, offs, lins, refs = [], [0], [], {1: [], 2: []}
        cut_identical, t_cut, t_ref = True, 0.0, 0.0
        for r in runs:
            imu, cam = D[f"{r}/imu"], D[f"{r}/cam"]
            t, w, a = imu[:, 6], imu[:, 0:3], imu[:, 3:6]
            t0 = time.perf_counter()
            S, off = synth.cut_windows(t, w, a, cam, imu_wait=IMU_WAIT[rate])
            t_cut += time.perf_counter() - t0
            nw = len(off) - 1
            lin = np.zeros((len(cam), 13))
            lin[:, 0:3] = rng.normal(0, 1e-3, (len(cam), 3)); lin[:, 3:6] = rng.normal(0, 1e-2, (len(cam), 3))
            q = rng.normal(0, 1, (len(cam), 4)); q /= np.linalg.norm(q, axis=1, keepdims=True); q[q[:, 3] < 0] *= -1
            lin[:, 6:10] = q; lin[:, 10:13] = synth.GRAVITY
            t0 = time.perf_counter()
            for model in (1, 2):
                Sr, offr, rec = R.replay_run(model, t, w, a, cam, lin, synth.SIGMAS, 0, imu_wait=IMU_WAIT[rate])
                cut_identical &= bool(np.array_equal(Sr, S) and np.array_equal(offr, off))
                refs[model].append(rec)
            t_ref += time.perf_counter() - t0
            Ss.append(S); offs += list(off[1:] + offs[-1]); lins.append(lin[:nw])
        S = np.concatenate(Ss); off = np.array(offs, dtype=np.int64); L = np.concatenate(lins)
        n = len(off) - 1
        entry = {"runs": len(runs), "windows": int(n), "entries": int(len(S)), "steps_per_window_mean": float(len(S) / max(n, 1)),
                 "cut_bit_identical_to_reference_loop": cut_identical, "cut_windows_per_s_host": n / t_cut,
                 "reference_cpu_windows_per_s_1thread_both_models": 2 * n / t_ref}
        band = window_band(S, off, L)
        dS, dL, dO = torch.from_numpy(S).cuda(), torch.from_numpy(L).cuda(), torch.from_numpy(off).cuda()
        for model in (1, 2):
            got = preint.preintegrate(model, dS, dL, synth.SIGMAS, 0, offsets=dO)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                preint.preintegrate(model, dS, dL, synth.SIGMAS, 0, offsets=dO, out=got)
            e1.record(); torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 5
            ref = np.concatenate(refs[model])
            worst = compare_records(got.cpu().numpy(), ref, model, in_band=band)      # asserts the north_star gates window by window
            host = preint.preintegrate_host(model, S, L, synth.SIGMAS, 0, offsets=off)
            entry[f"model{model}"] = {"worst": {k: float(f"{v:.3e}") for k, v in worst.items()}, "kernel_ms": ms, "windows_per_s": n / (ms * 1e-3),
                                      "host_entry_bitwise_equal": bool(np.array_equal(host, got.cpu().numpy())), "windows_in_ill_conditioned_band": int(band.sum())}
            print(rate, model, n, entry[f"model{model}"], file=sys.stderr)
        report["rates"][str(rate)] = entry
    print(json.dumps(report))


if __name__ == "__main__":
    main()
