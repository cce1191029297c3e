#!/usr/bin/env python
"""Parity report at scale: the CUDA path (through the C ABI) against the UNMODIFIED reference compiled in place
(oracle/_ref/libcpi_ref.so, all host threads) on the bench distribution.  Writes one JSON object to stdout.
Run:  python tools/parity_report.py > parity.json"""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np
from cpi_b200 import preint, factor, synth
from oracle.oracle import Reference
from parity import REC, window_band

R = Reference()
cores = synth.usable_cpus()
FIELDS = ["R", "alpha", "beta", "J_q", "J_a", "J_b", "H_a", "H_b", "P"]


def field_errors(got, ref, model, band):
    out = {}
    names = FIELDS + (["O_a", "O_b"] if model == 2 else [])
    for k in names:
        a, b = REC[k]
        num = np.linalg.norm(got[:, a:b] - ref[:, a:b], axis=1)
        den = np.maximum(np.linalg.norm(ref[:, a:b], axis=1), 1e-300)
        rel = num / den if k != "R" else num            # dR: absolute Frobenius (north_star gate)
        if k == "J_a":
            out["J_a (no sample in the ill-conditioned band)"] = float(rel[~band].max()) if (~band).any() else None
            out["J_a (band |w| in [0.0087,0.05))"] = float(rel[band].max()) if band.any() else None
        else:
            out[k] = float(rel.max())
    # P: worst 3x3 block, relative to the block's own norm; structural zeros exact
    Pg = got[:, 65:290].reshape(-1, 15, 15); Pr = ref[:, 65:290].reshape(-1, 15, 15)
    worst = 0.0
    for I in range(5):
        for J in range(5):
            bg, br = Pg[:, 3 * J:3 * J + 3, 3 * I:3 * I + 3], Pr[:, 3 * J:3 * J + 3, 3 * I:3 * I + 3]
            nr = np.linalg.norm(br.reshape(len(br), -1), axis=1)
            if np.all(nr == 0):
                assert np.all(bg == 0)
                continue
            worst = max(worst, float((np.linalg.norm((bg - br).reshape(len(br), -1), axis=1) / np.maximum(nr, 1e-300)).max()))
    out["P worst 3x3 block"] = worst
    out["P exactly symmetric"] = bool(np.array_equal(Pg, Pg.transpose(0, 2, 1)))
    return out


report = {"reference": "oracle/_ref/libcpi_ref.so (unmodified rpng/cpi headers, compiled in place)", "host_threads": cores, "cases": []}
for model, n, ns, rate, flags in ((1, 10000, 200, 200.0, 0), (2, 3000, 400, 400.0, 0), (1, 2000, 200, 200.0, 1), (2, 2000, 200, 200.0, 2)):
    S, L = synth.make_windows(n, ns, rate=rate, imu_avg=bool(flags & 1))
    t0 = time.time(); ref = R.preintegrate(model, S, L, synth.SIGMAS, flags, ns=ns, nthreads=cores); t_ref = time.time() - t0
    got = preint.preintegrate_host(model, S, L, synth.SIGMAS, flags, ns=ns)
    off = np.arange(n + 1, dtype=np.int64) * S.shape[1]
    band = window_band(S.reshape(-1, 7), off, L)
    report["cases"].append({"model": model, "flags": flags, "windows": n, "samples": ns, "reference_seconds": round(t_ref, 2),
                            "worst_error_over_all_windows": field_errors(got, ref, model, band)})
# fp32-storage variant against the fp64 reference on the same float-rounded inputs
S, L = synth.make_windows(4000, 200)
S32, L32 = S.astype(np.float32), L.astype(np.float32)
ref = R.preintegrate(1, S32.astype(np.float64), L32.astype(np.float64), synth.SIGMAS, 0, ns=200, nthreads=cores)
got = preint.preintegrate_host(1, S32, L32, synth.SIGMAS, 0, ns=200).astype(np.float64)
report["cases"].append({"model": 1, "dtype": "fp32 storage (fp32 RK4 stages, fp64-accumulated state)", "windows": 4000, "samples": 200,
                        "worst_error_over_all_windows": field_errors(got, ref, 1, window_band(S.reshape(-1, 7), np.arange(4001, dtype=np.int64) * 200, L))})
# full-size multi-wave batches (BASELINE configs[2] / configs[3] shapes): a strided + tail sample of windows against the reference
import torch
for tag, model, n, ns, rate, dt in (("configs[2] 100k x 400 model 2 fp64", 2, 100_000, 400, 400.0, np.float64), ("configs[3] per-GPU share 125k x 200 model 1 fp32 storage", 1, 125_000, 200, 200.0, np.float32),
                                   ("125k x 200 model 1 fp64", 1, 125_000, 200, 200.0, np.float64)):
    nd = 12_500
    S, L = synth.make_windows(nd, ns, rate=rate, first_window=70_000)
    Sx, Lx = S.astype(dt), L.astype(dt)
    reps = n // nd
    dS = torch.from_numpy(Sx).cuda().repeat(reps, 1, 1).contiguous(); dL = torch.from_numpy(Lx).cuda().repeat(reps, 1).contiguous()
    got = preint.preintegrate(model, dS, dL, synth.SIGMAS, 0, ns=ns)
    torch.cuda.synchronize()
    sel = np.unique(np.r_[0:80, n // 2:n // 2 + 80, n - 200:n, np.arange(0, n, 997)])
    g = got[torch.from_numpy(sel).cuda()].cpu().numpy().astype(np.float64)
    src = sel % nd
    ref = R.preintegrate(model, Sx[src].astype(np.float64), Lx[src].astype(np.float64), synth.SIGMAS, 0, ns=ns, nthreads=cores)
    off = np.arange(len(sel) + 1, dtype=np.int64) * ns
    report["cases"].append({"what": tag, "windows_in_batch": n, "windows_compared": int(len(sel)), "inputs": f"{nd} distinct windows tiled x{reps} on the device",
                            "worst_error_over_compared_windows": field_errors(g, ref, model, window_band(S[src].reshape(-1, 7), off, L[src]))})
    del dS, dL, got
# factor evaluation, 5k chain, both models
for model in (1, 2):
    S, L = synth.make_windows(4999, 20, first_window=9000)
    rec = preint.preintegrate_host(model, S, L, synth.SIGMAS, 0, ns=20)
    X = synth.make_states(rec, L, model)
    e, H1, H2 = factor.factor_eval_host(model, X, rec, L)
    er, H1r, H2r = R.factor_eval(model, X, rec, L, nthreads=cores)
    report["cases"].append({"kernel": f"ImuFactorCPIv{model}::evaluateError", "factors": 4999,
                            "max_abs_error": {"e": float(np.abs(e - er).max()), "H1": float(np.abs(H1 - H1r).max()), "H2": float(np.abs(H2 - H2r).max())},
                            "structural_zeros_exact": bool(np.array_equal(H1 == 0, H1r == 0) and np.array_equal(H2 == 0, H2r == 0))})
print(json.dumps(report, indent=1))
