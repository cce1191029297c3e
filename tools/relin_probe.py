"""Re-preintegration of drifted windows (cpi_imu_records_relinearize; DESIGN.md section 3i): cost of the call and value of the
relinearising loop, on one GPU.  Prints one JSON line.

    python tools/relin_probe.py [--chains 10000] [--states 30] [--ns 200] [--reps 5]
    python tools/relin_probe.py --table        # CPU only: the first-order model's error against the bias offset (oracle)

Model 1, chains of `states` keyframes with `ns`-sample windows (10 000 x 30 x 200: 290 000 windows).  Cases: the whole call with
0 %, 1 %, 10 % and 100 % of the factors selected (CUDA events, median of --reps; the lin the call rewrites is restored before each
call, outside the timed window); its split into selection + compaction, gather, K1 and scatter (torch.profiler kernel times, median
of --reps calls); preint.preintegrate of every window as the reference; then chains_lm alone against the loop chains_lm ->
relinearize_records -> chains_lm (tests/test_relinearize.py's problem: b_g = 5e-2 rad/s, b_a = 0.2 m/s^2, a prior on x_0, a 1 cm
position fix every 5th keyframe): rounds, time, worst error against the truth in retract coordinates."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from scan_probe import gpu_identity, timed  # noqa: E402

TOL = (2e-3, 2e-2, 1e-2)


def first_order_table():
    """Worst |e| of the factor residual at states consistent with a bias b*, records at lin = 0 against records at b*, for 200-sample
    windows: the plain-C oracle on the CPU (computed, not timed).  Per (model, |db_w|, |db_a|): the worst rotation, velocity and
    position residual entries over 64 windows."""
    from cpi_b200 import synth
    from oracle.oracle import Oracle
    orc = Oracle()
    n, ns = 64, 200
    S, L = synth.make_windows(n, ns, rate=200.0, first_window=5000, special=False)
    Sf = S.reshape(-1, 7)
    rng = np.random.default_rng(1)
    dirs = rng.normal(size=(n, 6))
    dirs[:, 0:3] /= np.linalg.norm(dirs[:, 0:3], axis=1, keepdims=True)
    dirs[:, 3:6] /= np.linalg.norm(dirs[:, 3:6], axis=1, keepdims=True)
    rows = []
    for model in (1, 2):
        for bw, ba in ((1e-3, 1e-2), (1e-2, 1e-2), (1e-2, 1e-1), (3e-2, 1e-1), (1e-1, 1e-1), (1e-1, 1.0)):
            Lt = L.copy()
            Lt[:, 0:3], Lt[:, 3:6] = bw * dirs[:, 0:3], ba * dirs[:, 3:6]
            e_row = {"rot": 0.0, "vel": 0.0, "pos": 0.0}
            for k in range(n):
                r = orc.preintegrate(model, Sf[k * ns:(k + 1) * ns], Lt[k:k + 1], synth.SIGMAS, 0, ns=ns)
                X = synth.make_states(r, Lt[k:k + 1], model, perturb=False)
                Lk = Lt[k:k + 1].copy()
                Lk[0, 6:10] = X[0, 0:4]
                r = orc.preintegrate(model, Sf[k * ns:(k + 1) * ns], Lk, synth.SIGMAS, 0, ns=ns)
                X = synth.make_states(r, Lk, model, perturb=False)
                L0 = Lk.copy()
                L0[0, 0:6] = 0.0
                r0 = orc.preintegrate(model, Sf[k * ns:(k + 1) * ns], L0, synth.SIGMAS, 0, ns=ns)
                e = orc.factor_eval(model, X, r0, L0)[0][0]
                e_row["rot"] = max(e_row["rot"], float(np.abs(e[0:3]).max()))
                e_row["vel"] = max(e_row["vel"], float(np.abs(e[6:9]).max()))
                e_row["pos"] = max(e_row["pos"], float(np.abs(e[12:15]).max()))
            rows.append(dict(model=model, db_w=bw, db_a=ba, **e_row))
    return rows


def kernel_split(torch, fn, reps):
    """Median per-call device time (ms) of the call's kernels, grouped: selection + compaction, gather, K1, scatter."""
    from torch.profiler import ProfilerActivity, profile
    groups = {"select_compact": ("k_relin_select", "k_relin_scan_blocks", "k_relin_compact"), "gather": ("k_relin_gather",),
              "k1": ("k_preintegrate",), "scatter": ("k_relin_scatter",)}
    per = {g: [] for g in groups}
    for _ in range(reps):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        tot = {g: 0.0 for g in groups}
        for ev in prof.events():
            if ev.device_type.name != "CUDA":
                continue
            for g, names in groups.items():
                if any(nm in ev.name for nm in names):
                    tot[g] += ev.device_time / 1e3 if hasattr(ev, "device_time") else ev.cuda_time / 1e3
        for g in groups:
            per[g].append(tot[g])
    return {g: float(np.median(v)) for g, v in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=10000)
    ap.add_argument("--states", type=int, default=30)
    ap.add_argument("--ns", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--unique-chains", type=int, default=128, help="chains of distinct windows; the rest repeat them")
    ap.add_argument("--table", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.table:
        print(json.dumps({"first_order_error": first_order_table()}))
        return
    import torch
    from cpi_b200 import capi, factor, preint, synth
    from test_relinearize import run_value, value_problem
    assert torch.cuda.is_available(), "relin_probe needs a CUDA device"
    name, power = gpu_identity()
    capi.load()
    C, S, ns = a.chains, a.states, a.ns
    nf = C * (S - 1)
    X, truth, Sf, lin0, prior, sps = value_problem(1, C, S, ns, seed=7, unique_chains=a.unique_chains)
    dS = torch.from_numpy(Sf).cuda()
    dX = torch.from_numpy(truth).cuda()
    idx_i = np.delete(np.arange(C * S), np.arange(S - 1, C * S, S))
    base = lin0.copy()
    base[:, 0:3], base[:, 3:6] = truth[idx_i, 4:7], truth[idx_i, 10:13]
    dR = preint.preintegrate(1, dS, torch.from_numpy(base).cuda(), synth.SIGMAS, 0, ns=ns)
    ws = torch.empty((int(capi.load().cpi_imu_records_relinearize_workspace(1, nf, Sf.shape[0])) + 7) // 8, dtype=torch.float64, device="cuda")
    rng = np.random.default_rng(3)
    res = {"gpu": name, "power_limit_w": power, "chains": C, "states": S, "ns": ns, "windows": nf, "reps": a.reps,
           "workspace_gb": ws.numel() * 8 / 1e9, "call_ms": {}, "selected": {}}
    for frac in (0.0, 0.01, 0.1, 1.0):
        lin = base.copy()
        pick = rng.random(nf) < frac if frac < 1.0 else np.ones(nf, bool)
        lin[pick, 0] += 1.0                           # a bias far outside the tolerance: those factors are selected
        dl0 = torch.from_numpy(lin).cuda()
        dl = dl0.clone()
        counts = []

        def call():
            dl.copy_(dl0)
            st = torch.cuda.current_stream()
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record(st)
            n, _ = factor.relinearize_records(1, dX, dR, dl, S, dS, synth.SIGMAS, None, ns, 0, tol_bw=TOL[0], tol_ba=TOL[1], workspace=ws)
            ev1.record(st)
            ev1.synchronize()
            counts.append(n)
            return ev0.elapsed_time(ev1)
        for _ in range(2):
            call()
        ts = [call() for _ in range(a.reps)]
        res["call_ms"][f"{frac:g}"] = float(np.median(ts))
        res["selected"][f"{frac:g}"] = int(counts[-1])
        if frac in (0.1, 1.0):
            res[f"split_ms_{frac:g}"] = kernel_split(torch, call, a.reps)
    dl = torch.from_numpy(base).cuda()
    out = torch.empty_like(dR)
    res["preintegrate_all_ms"] = timed(torch, lambda: preint.preintegrate(1, dS, dl, synth.SIGMAS, 0, ns=ns, out=out), a.reps)
    del ws, dR, out
    torch.cuda.empty_cache()
    for relin in (False, True):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        Xf, lf, passes, rounds, n_last, err = run_value(torch, 1, X, truth, Sf, lin0, prior, sps, S, ns, TOL, relin=relin)
        torch.cuda.synchronize()
        res["loop" if relin else "lm_alone"] = {"passes": passes, "rounds": rounds, "ms": 1e3 * (time.perf_counter() - t0),
                                                "worst_error": err, "last_count": n_last}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
