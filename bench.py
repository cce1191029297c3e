#!/usr/bin/env python
"""bench.py -- IMU windows/sec of the batched closed-form preintegration hot path (BASELINE.json metric).

    python bench.py --gpus N --steps K --warmup W [--impl reference] [--workload v1_10k_200|v2_100k_400] [--dump-outputs DIR]

One "step" = one pass of the hot path over one batch of synthetic IMU windows (cpi_b200/synth.py, seed 20260924).
Default workload = BASELINE.json configs[1]: 10 000 windows x 200 samples, CPI model 1 (mean + Jacobians + covariance),
fp64, per GPU.  With N > 1 every rank preintegrates its own 10k-window shard (weak scaling, windows are independent) and
the step ends with ONE NCCL all-gather of the result records, the kernel having written its shard straight into its
slice of the gather buffer -- both through the product's C ABI (cpi_preintegrate_batch_sharded, cpi_b200.shard.Communicator):
the all-gather runs on the communicator's own stream, so step i's collective overlaps step i+1's kernel (two gather buffers).  Timing: W untimed warm-up steps, then K steps between barrier + synchronize, CUDA events on
the launching stream, max over ranks.  Inputs rotate over several distinct resident batches whose total size exceeds
the 50 MB L2 of an H100, so no step finds its samples in cache.

The default run appends a "configs" array to the same JSON line: short measurements of the other BASELINE configs
(configs[2] v2 100k x 400, configs[3] fp32 125k per GPU, configs[4] the 5k factor chain, configs[0] single window).

Extra keys: roofline (dominant kernel vs the H100 SXM data-sheet fp64 / fp32 and HBM3 peaks), cpu_baseline (the
reference's own CPU implementation timed on this box's host cores, rank 0, N = 1), e2e (same metric through the C-ABI
host entry point with pinned HOST buffers: H2D + kernel + D2H inside the timed region), clocks, gpu_launches.
`--impl reference` times the reference's CPU path (oracle/_ref when it was compiled, else the oracle port) on all host
threads on a bounded sample of the same workload.

`--dump-outputs DIR` writes, after the timed steps, what the last timed step computed (the records of the preintegration
workloads, e / H1 / H2 of the factor workloads) as DIR/<name>.npy, at most 64 MB in all: larger outputs are reduced to a fixed,
seeded sample of rows, whose indices are written as DIR/rows.npy.  Inputs depend only on the arguments, so two builds can
be compared output for output.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

WORKLOADS = {
    # name: (model, windows per GPU, samples per window, rate Hz, algorithmic flops/sample, bytes/window in+out)  SURVEY 8(d)
    "v1_10k_200": dict(model=1, n=10_000, ns=200, rate=200.0, flops_per_sample=5.8e3, bytes_per_window=13_624,
                       desc="configs[1]: 10k-window batch x 200 samples, CPI v1 mean+covariance, fp64"),
    "v2_100k_400": dict(model=2, n=100_000, ns=400, rate=400.0, flops_per_sample=15.0e3, bytes_per_window=24_968,
                        desc="configs[2]: 100k-window batch x 400 samples, CPI v2, fp64"),
    # configs[0]: the reference's own CPU-runnable case (one window, 100 samples); for the GPU arm this is pure launch latency
    "v1_single_100": dict(model=1, n=1, ns=100, rate=200.0, flops_per_sample=5.8e3, bytes_per_window=8_024, single=True,
                          desc="configs[0]: single CPI v1 window, 100 IMU samples @ 200 Hz, fp64"),
    # throughput regime of the headline kernel (not a BASELINE config): 125k windows = the per-GPU share of configs[3], in fp64
    "v1_125k_200": dict(model=1, n=125_000, ns=200, rate=200.0, flops_per_sample=5.8e3, bytes_per_window=13_624,
                        desc="125k-window batch x 200 samples, CPI v1, fp64 (large-batch regime of the configs[1] kernel)"),
    # configs[3] is quoted on 8 GPUs: 1M windows = 125k per GPU (weak-scaling unit); fp32-storage variant (DESIGN.md 3a)
    "v1_1m_200_fp32": dict(model=1, n=125_000, ns=200, rate=200.0, flops_per_sample=5.8e3, bytes_per_window=6_812, fp32=True,
                           desc="configs[3]: 1M-window batch x 200 samples, CPI v1, fp32 storage, 125k windows per GPU + NCCL all-gather"),
    # configs[4]: the factor-evaluation kernel K3 over a 5k-keyframe chain (factors/s, HBM-write bound)
    "factor_5k": dict(model=1, n=4_999, ns=20, rate=200.0, factor=True,
                      desc="configs[4]: 5k-keyframe chain, batched ImuFactorCPIv1 residual + H1 + H2 (4 999 factors per step)"),
    # bandwidth regime of K3 (not a BASELINE config): 1M factors = 4.5 GB of output per launch against the HBM write roofline
    "factor_1m": dict(model=1, n=1_000_000, ns=20, rate=200.0, factor=True, distinct=20_000,
                      desc="1M-factor chain, batched ImuFactorCPIv1 residual + H1 + H2 (bandwidth regime of the configs[4] kernel)"),
}
# Roofline denominators: NVIDIA's H100 SXM data sheet (cards allowed 700 W; a card with a lower power limit clocks lower, and the
# "clocks" key of the result line shows what the run got).  Non-tensor fp64 and fp32, since no kernel of this path uses tensor cores.
DFMA_PEAK_TFLOPS = 34.0
FFMA_PEAK_TFLOPS = 67.0
HBM_PEAK_GBS = 3350.0
PEAK_SOURCE = "H100 SXM data sheet (700 W), not measured"
DUMP_LIMIT_BYTES = 64 << 20


def dump_outputs(dirname, tensors):
    """Write {name: tensor} as dirname/<name>.npy (float32 / float64), at most DUMP_LIMIT_BYTES in all.  Tensors share their leading
    dimension; if they do not fit, the same fixed, seeded sample of rows is selected on the device from each (only those rows are
    copied to the host) and its indices are written as rows.npy."""
    import torch
    os.makedirs(dirname, exist_ok=True)
    tensors = {k: v.detach().to(torch.float32 if v.dtype == torch.float32 else torch.float64) for k, v in tensors.items()}
    rows = next(iter(tensors.values())).shape[0]
    row_bytes = sum(v.numel() // max(v.shape[0], 1) * v.element_size() for v in tensors.values())
    out = {}
    if rows * row_bytes > DUMP_LIMIT_BYTES:
        keep = DUMP_LIMIT_BYTES // (row_bytes + 8)
        idx = np.sort(np.random.default_rng(20260924).choice(rows, size=keep, replace=False))
        tensors = {k: v.index_select(0, torch.from_numpy(idx).to(v.device)) for k, v in tensors.items()}
        out["rows"] = idx.astype(np.float64)
    out.update({k: v.cpu().numpy() for k, v in tensors.items()})
    for k, v in out.items():
        np.save(os.path.join(dirname, f"{k}.npy"), np.ascontiguousarray(v))


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index=0):
        self.index = index; self.rows = []; self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "50", "-i", str(self.index)],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True); self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append((time.time(), line.strip()))

    def stop(self, t0, t1):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.12)
        self.proc.terminate()
        sm, mx, reasons = [], None, set()
        for ts, line in self.rows:
            f = [x.strip() for x in line.split(",")]
            if len(f) < 9:
                continue
            try:
                clk, mx = float(f[1]), float(f[2])
            except ValueError:
                continue
            if t0 - 0.05 <= ts <= t1 + 0.05:
                sm.append(clk)
                for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                    if v.lower().startswith("active"):
                        reasons.add(name)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": mx, "reasons": sorted(reasons), "samples": len(sm)}


def cpu_arm(wl, sample_windows, nthreads=None):
    """The reference's own CPU implementation of the path on the host cores: (value windows/s, kind, cores, sample)."""
    from oracle.oracle import Oracle, Reference
    from cpi_b200 import synth
    if Reference.available():
        impl, kind = Reference(), "reference"
    else:
        if not os.path.exists(Oracle.path):
            subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "liboracle.so"], check=True)
        impl, kind = Oracle(), "port"
    cores = nthreads or synth.usable_cpus()        # scheduler affinity capped by the cgroup quota: the threads we can actually run
    S, L = synth.make_windows(sample_windows, wl["ns"], rate=wl["rate"])
    impl.preintegrate(wl["model"], S[:cores], L[:cores], synth.SIGMAS, 0, ns=wl["ns"], nthreads=cores)   # warm
    t0 = time.perf_counter()
    impl.preintegrate(wl["model"], S, L, synth.SIGMAS, 0, ns=wl["ns"], nthreads=cores)
    dt = time.perf_counter() - t0
    return sample_windows / dt, kind, cores, dt


def config_dict(wl, world, note=None):
    """The SAME dict on both arms (the driver compares them): the workload, not how an arm samples it."""
    n, ns, model = wl["n"], wl["ns"], wl["model"]
    f32 = bool(wl.get("fp32"))
    es = 4 if f32 else 8
    if wl.get("factor"):
        return {"workload": wl["desc"], "factors_per_step": n, "model": f"ImuFactorCPIv{model}", "parallelism": "rank 0 only (the solver lives there)",
                "l2": "192 MB buffer written between timed launches (outside the event pair) > 50 MB L2"}
    bytes_in = n * ns * 7 * es + n * 13 * es
    nb = 2 if bytes_in > 300e6 else min(8, max(2, int(np.ceil(300e6 / bytes_in))))
    return {"workload": wl["desc"], "windows_per_gpu": n, "samples_per_window": ns, "model": f"CpiV{model}",
            "parallelism": f"window-sharded x{world}" + (", one NCCL all-gather of records per step (overlapped with the next step's kernel)" if world > 1 else ""),
            "l2": f"{nb} rotating resident input batches = {nb * bytes_in / 1e6:.0f} MB > 50 MB L2"}


def run_reference(args, wl):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    from cpi_b200 import synth
    cores = synth.usable_cpus()
    if wl.get("single"):
        # SURVEY 8(d) config 1: one window, reference CpiV1 on ONE thread, median of >= 1000 repeats
        from oracle.oracle import Oracle, Reference
        impl, kind = (Reference(), "reference") if Reference.available() else (Oracle(), "port")
        S, L = synth.make_windows(1, wl["ns"], rate=wl["rate"], special=False)
        ts = []
        for _ in range(1200):
            t0 = time.perf_counter(); impl.preintegrate(wl["model"], S, L, synth.SIGMAS, 0, ns=wl["ns"], nthreads=1); ts.append(time.perf_counter() - t0)
        ms = 1e3 * float(np.median(ts[200:]))
        print(json.dumps({"impl": "reference", "metric": "imu_windows_per_sec", "value": 1e3 / ms, "unit": "windows/s", "n_gpus": args.gpus, "steps": 1000, "warmup": 200,
                          "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
                          "config": config_dict(wl, args.gpus),
                          "cpu_baseline": {"value": 1e3 / ms, "unit": "windows/s", "cores": 1, "kind": kind, "sample": "1 window x 100 samples, median of 1000 repeats (includes ~3 us of ctypes call overhead)"},
                          "e2e": {"value": 1e3 / ms, "unit": "windows/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}), flush=True)
        return
    # bounded sample: calibrate on a small run, then size each step for ~5 s of CPU work (all usable host threads)
    v0, kind, cores, _ = cpu_arm(wl, max(2 * cores, 64))
    sample = int(min(wl["n"], max(cores, v0 * 5.0)))
    times = []
    for i in range(args.warmup + args.steps):
        v, kind, cores, dt = cpu_arm(wl, sample)
        if i >= args.warmup:
            times.append(dt)
    ms = 1e3 * float(np.mean(times))
    value = sample / (ms * 1e-3)
    line = {"impl": "reference", "metric": "imu_windows_per_sec", "value": value, "unit": "windows/s", "n_gpus": args.gpus, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32 storage + f32 covariance RK4, f64 rotations/coefficients/means" if wl.get("fp32") else "f64",
            "data": "synthetic", "config": config_dict(wl, args.gpus),
            "cpu_baseline": {"value": value, "unit": "windows/s", "cores": cores, "cores_online": os.cpu_count(), "kind": kind,
                             "sample": f"{sample} windows x {wl['ns']} samples per step, {'oracle/_ref (unmodified reference, std::thread over windows)' if kind == 'reference' else 'oracle C port'}"
                                       + (" -- the reference is double-only: the fp64 path on the same inputs" if wl.get("fp32") else "")},
            "e2e": {"value": value, "unit": "windows/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


def run_factor(args, wl, emit=True, cpu=True, dump=None):
    """configs[4]: K3 (ImuFactorCPIv1::evaluateError batched) over a 5k-keyframe chain.  HBM-write bound: 4 496 algorithmic
    bytes per factor (776 in, 3 720 out); at 5k factors the launch is ~10 us, i.e. launch-latency sized."""
    from cpi_b200 import synth
    from oracle.oracle import Oracle, Reference
    model, n, ns = wl["model"], wl["n"], wl["ns"]
    nd = min(n, wl.get("distinct", n))
    S, L = synth.make_windows(nd, ns, rate=wl["rate"], first_window=9000)
    if nd < n:      # tile a distinct block (host generation is ~0.1 ms per 20-sample window)
        reps = (n + nd - 1) // nd
        S = np.tile(S, (reps, 1, 1))[:n]; L = np.tile(L, (reps, 1))[:n]
    if args.impl == "reference":
        if int(os.environ.get("RANK", "0")) != 0:
            return
        impl, kind = (Reference(), "reference") if Reference.available() else (Oracle(), "port")
        cores = synth.usable_cpus()
        rec = impl.preintegrate(model, S, L, synth.SIGMAS, 0, ns=ns, nthreads=cores)
        X = synth.make_states(rec, L, model)
        ts = []
        for i in range(args.warmup + args.steps):
            t0 = time.perf_counter(); impl.factor_eval(model, X, rec, L, nthreads=cores); ts.append(time.perf_counter() - t0)
        ms = 1e3 * float(np.mean(ts[args.warmup:])); v = n / (ms * 1e-3)
        print(json.dumps({"impl": "reference", "metric": "imu_factors_per_sec", "value": v, "unit": "factors/s", "n_gpus": args.gpus, "steps": args.steps,
                          "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
                          "config": config_dict(wl, args.gpus), "cpu_baseline": {"value": v, "unit": "factors/s", "cores": cores, "kind": kind, "sample": f"{n} factors per step"},
                          "e2e": {"value": v, "unit": "factors/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}), flush=True)
        return
    import torch
    from cpi_b200 import capi, factor, preint
    lib = capi.load()
    rec = preint.preintegrate_host(model, S, L, synth.SIGMAS, 0, ns=ns)
    X = synth.make_states(rec, L, model)
    dX, dR, dL = (torch.from_numpy(a).cuda() for a in (X, rec, L))
    outs = (torch.empty((n, 15), dtype=torch.float64, device="cuda"), torch.empty((n, 225), dtype=torch.float64, device="cuda"),
            torch.empty((n, 225), dtype=torch.float64, device="cuda"))
    flush = torch.empty(192 << 20, dtype=torch.uint8, device="cuda")      # > 50 MB L2: written between timed launches
    big = n > 100_000
    stream = torch.cuda.current_stream()
    t_settle = time.perf_counter()
    while time.perf_counter() - t_settle < 0.15:
        factor.factor_eval(model, dX, dR, dL, out=outs); torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    for i in range(args.warmup):
        flush.zero_(); factor.factor_eval(model, dX, dR, dL, out=outs)
    launches0 = capi.launch_count()
    torch.cuda.synchronize()
    for i in range(args.steps):
        flush.zero_()                                                       # L2 flush, outside the per-launch event pair
        evs[i][0].record(stream); factor.factor_eval(model, dX, dR, dL, out=outs); evs[i][1].record(stream)
    torch.cuda.synchronize()
    launches = capi.launch_count() - launches0
    ms = float(np.mean([a.elapsed_time(b) for a, b in evs]))
    if dump:
        dump_outputs(dump, dict(zip(("e", "H1", "H2"), outs)))
    ach = 4496.0 * n / (ms * 1e-3) * 1e-9
    hX, hR, hL = (torch.from_numpy(a).pin_memory() for a in (X, rec, L))
    hE, hH1, hH2 = (torch.empty(sh, dtype=torch.float64).pin_memory() for sh in ((n, 15), (n, 225), (n, 225)))
    import ctypes
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    def host_step():
        capi.check(lib.cpi_imu_factor_eval_batch_host(model, n, n + 1, P(hX), None, None, P(hR), P(hL), P(hE), P(hH1), P(hH2)))
    for _ in range(1 if big else 3):
        host_step()
    ke = 2 if big else 10
    per_call = []
    t0 = time.perf_counter()
    for _ in range(ke):
        t1 = time.perf_counter(); host_step(); per_call.append((time.perf_counter() - t1) * 1e3)
    e2e_ms = (time.perf_counter() - t0) * 1e3 / ke
    out = {"metric": "imu_factors_per_sec", "value": n / (ms * 1e-3), "unit": "factors/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms,
           "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
           "config": config_dict(wl, 1), "gpu_launches": int(launches), "kernel_ms": ms,
           "roofline": {"bound": "hbm", "achieved": ach, "peak": HBM_PEAK_GBS, "unit": "GB/s", "frac": ach / HBM_PEAK_GBS, "peak_source": PEAK_SOURCE,
                        "note": "4 496 algorithmic B/factor; at 5k factors (22 MB) the launch is latency-sized: 22 MB at peak would take 6.7 us; the 1M-factor workload shows the bandwidth regime"},
           "e2e": {"value": n / (e2e_ms * 1e-3), "unit": "factors/s", "ms_per_step": e2e_ms, "h2d_bytes_per_step": int((hX.numel() + hR.numel() + hL.numel()) * 8),
                   "d2h_bytes_per_step": int((hE.numel() + hH1.numel() + hH2.numel()) * 8), "api": "cpi_imu_factor_eval_batch_host",
                   "ms_per_call": [round(t, 3) for t in per_call]}}
    # one Levenberg-Marquardt step of the IMU-only chain entirely on device: eval -> information blocks -> block-tridiagonal
    # assembly -> block-cyclic-reduction Cholesky solve -> retract (SURVEY 8f rank 1; parity unpinned: GTSAM is not in the tree)
    if hasattr(factor, "chain_lm_step") and not big:
        try:
            factor.chain_lm_step(model, dX, dR, dL); torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            for _ in range(5):
                factor.chain_lm_step(model, dX, dR, dL)
            b.record(stream); torch.cuda.synchronize()
            out["lm_step"] = {"ms": a.elapsed_time(b) / 5, "what": "eval + Hessian blocks + assemble + block-tridiagonal solve + retract, all on device", "keyframes": n + 1}
        except Exception as ex:     # noqa: BLE001 -- reported, never hidden
            out["lm_step"] = {"error": repr(ex)}
    if cpu and not args.no_cpu_baseline:
        impl, kind = (Reference(), "reference") if Reference.available() else (Oracle(), "port")
        cores = synth.usable_cpus()
        impl.factor_eval(model, X, rec, L, nthreads=cores)
        t0 = time.perf_counter()
        for _ in range(5):
            impl.factor_eval(model, X, rec, L, nthreads=cores)
        dt = (time.perf_counter() - t0) / 5
        out["cpu_baseline"] = {"value": n / dt, "unit": "factors/s", "cores": cores, "kind": kind, "sample": f"{n} factors x 5 repeats, reference evaluateError with H1 and H2"}
    if emit:
        print(json.dumps(out), flush=True)
    return out


class Ctx:
    """Process-wide state shared by the measurements of one bench run."""
    def __init__(self):
        import torch
        import torch.distributed as dist
        from cpi_b200 import capi
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.rank = int(os.environ.get("RANK", "0"))
        local = int(os.environ.get("LOCAL_RANK", "0"))
        if self.world > 1:
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            torch.cuda.set_device(local)
            import datetime
            dist.init_process_group("nccl", device_id=torch.device("cuda", local), timeout=datetime.timedelta(seconds=180))
        else:
            torch.cuda.set_device(0)
        capi.load()
        self.dev = torch.device("cuda", torch.cuda.current_device())
        # pinned host buffers belong on the GPU's NUMA node (a remote node costs ~25 % of the H2D rate on these boxes).  N > 1: the rank binds
        # itself for good; N = 1: only while it allocates them (measure_preint), so that the CPU-baseline leg keeps every usable core
        self.numa = None
        self.affinity0 = os.sched_getaffinity(0)
        if self.world > 1:
            self.numa = self.pin_to_gpu_numa_node(torch)
        self.comm = None
        if self.world > 1:
            from cpi_b200 import shard
            self.comm = shard.Communicator()      # the product's NCCL communicator (C ABI)


def _pin_to_gpu_numa_node(self, torch):
    """Bind this process (and therefore the pinned host buffers it allocates next, first-touch) to the CPUs of its GPU's NUMA node, so that
    H2D does not cross the socket interconnect and eight ranks do not push their traffic through one socket.  Best effort: silently
    skipped when sysfs does not say."""
    try:
        pr = torch.cuda.get_device_properties(self.dev)
        bdf = f"{pr.pci_domain_id:04x}:{pr.pci_bus_id:02x}:{pr.pci_device_id:02x}.0"
        base = f"/sys/bus/pci/devices/{bdf}"
        node = int(open(f"{base}/numa_node").read())
        cpus = set()
        for part in open(f"{base}/local_cpulist").read().strip().split(","):
            a, _, b = part.partition("-")
            cpus.update(range(int(a), int(b or a) + 1))
        cpus &= os.sched_getaffinity(0)
        if node >= 0 and cpus:
            os.sched_setaffinity(0, cpus)
            return {"node": node, "cpus": len(cpus)}
    except Exception:      # noqa: BLE001
        pass
    return None


Ctx.pin_to_gpu_numa_node = _pin_to_gpu_numa_node


def measure_preint(ctx, name, args, steps, warmup, distinct=None, e2e=True, cpu=False, clocks=True, dump=None):
    """One workload of the preintegration path on this process' GPU (all ranks call it together).  `distinct`: generate only
    that many distinct windows on the host and tile them on the device (host generation is ~0.5 ms per window; the kernel does not
    care, and the resident set still exceeds L2) -- the headline workload always uses all-distinct windows."""
    import gc
    import torch
    import torch.distributed as dist
    from cpi_b200 import capi, preint, synth
    wl = WORKLOADS[name]
    world, rank, dev = ctx.world, ctx.rank, ctx.dev
    model, n, ns = wl["model"], wl["n"], wl["ns"]
    rd = capi.REC_DOUBLES[model]
    f32 = bool(wl.get("fp32"))
    tdt, es = (torch.float32, 4) if f32 else (torch.float64, 8)
    nd = n if not distinct else min(n, distinct)
    reps = (n + nd - 1) // nd

    # ---- resident inputs: NB distinct batches, NB * bytes > L2
    bytes_in = n * ns * 7 * es + n * 13 * es
    NB = 2 if bytes_in > 300e6 else min(8, max(2, int(np.ceil(300e6 / bytes_in))))
    batches = []
    for b in range(NB):
        S, L = synth.make_windows(nd, ns, rate=wl["rate"], first_window=(rank * NB + b) * n)
        dS, dL = torch.from_numpy(S).to(tdt).to(dev), torch.from_numpy(L).to(tdt).to(dev)
        if reps > 1:
            dS = dS.repeat(reps, 1, 1)[:n].contiguous(); dL = dL.repeat(reps, 1)[:n].contiguous()
        batches.append((dS, dL))
    del S, L      # NB: dropping a 112 MB numpy array is a ~12 ms munmap on the host -- must not happen inside the timed loop
    # rank r's kernel writes gathers[k][r] in place; two buffers in rotation, so that step i's exchange overlaps step i+1's kernel
    NG = 2 if world > 1 else 1
    gathers = [torch.empty((world, n, rd), dtype=tdt, device=dev) for _ in range(NG)]
    stream = torch.cuda.current_stream()
    exchange = None
    if world > 1:
        torch.cuda.synchronize()             # nothing of torch's own NCCL group in flight while the product communicator runs collectives
        pushed = [ctx.comm.register(g) for g in gathers]
        smfree = ctx.comm.lib.cpi_comm_sm_free_barriers(ctx.comm.handle) == 1
        exchange = ("copy-engine peer copies of every rank's slice into CUDA-IPC mappings of the peers' gather buffers, barriers = "
                    + ("copy-engine flag writes + cuStreamWaitValue32 (no SM)" if smfree else "two 1-element NCCL all-reduces")
                    if all(pushed) else "ncclAllGather (CPI_B200_GATHER=nccl, or the buffers could not be exported with CUDA IPC)")

    def step(i):
        dS, dL = batches[i % NB]
        if world > 1:
            ctx.comm.step(model, dS, dL, synth.SIGMAS, 0, gathers[i % NG], ns=ns, stream=stream)
        else:
            preint.preintegrate(model, dS, dL, synth.SIGMAS, 0, ns=ns, out=gathers[0][0], stream=stream)

    # everything host-side (events, clock sampler) is set up BEFORE the warm-up so that the GPU goes from the warm-up
    # steps straight into the timed region without an idle gap (see DESIGN.md "measurement notes").
    sampler = ClockSampler(torch.cuda.current_device()) if (rank == 0 and clocks and not args.no_clocks) else None
    if sampler:
        sampler.start(); time.sleep(0.3)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    kev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for e in [ev0, ev1] + [x for pair in kev for x in pair]:
        e.record(stream)                     # force the lazy cudaEventCreate now
    # clock settle: the part idles at 120 MHz while the host generates inputs and needs ~20 ms of work (with a ~13 ms
    # P-state stall in it, measured) to reach its load clocks; keep it busy for >= 150 ms before the W warm-up steps
    # (kernel only: this loop is time-bounded, so ranks may run different numbers of iterations -- no collective may be in it)
    t_settle = time.perf_counter()
    while time.perf_counter() - t_settle < 0.15:
        preint.preintegrate(model, batches[0][0], batches[0][1], synth.SIGMAS, 0, ns=ns, out=gathers[0][rank], stream=stream)
        torch.cuda.synchronize()
    for i in range(warmup):
        step(i)
    if world > 1:
        ctx.comm.wait(stream)
    launches0 = capi.launch_count()
    gc.collect(); gc.disable()        # no collector pauses inside the timed region
    # Two NCCL communicators (the product's and torch's) must never have collectives in flight at the same time on the same devices
    # (their kernels could start in different orders on different ranks and wait for each other): drain the device BEFORE the barrier.
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    t0 = time.time()
    ev0.record(stream)
    for i in range(steps):
        kev[i][0].record(stream)
        step(warmup + i)
        kev[i][1].record(stream)          # the all-gather is on the communicator's stream: this pair brackets the kernel alone
    if world > 1:
        ctx.comm.wait(stream)             # the timed region ends when the LAST all-gather has landed
    ev1.record(stream)
    torch.cuda.synchronize()
    t1 = time.time()
    if world > 1:
        dist.barrier()
    launches = capi.launch_count() - launches0
    gc.enable()
    if dump and rank == 0:
        last = gathers[(warmup + steps - 1) % NG]
        dump_outputs(dump, {"records": last.reshape(world * n, rd) if world > 1 else last[0]})
    clk = sampler.stop(t0, t1) if sampler else None
    total_ms = ev0.elapsed_time(ev1)
    kern_ms = float(np.mean([a.elapsed_time(b) for a, b in kev]))
    if os.environ.get("CPI_BENCH_DEBUG"):
        print("kernel ms:", [round(a.elapsed_time(b), 3) for a, b in kev], file=sys.stderr)
    if world > 1:
        t = torch.tensor([total_ms], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        total_ms = float(t.item())
    ms_per_step = total_ms / steps
    value = world * n / (ms_per_step * 1e-3)

    flops = wl["flops_per_sample"] * ns * n          # algorithmic flops per launch (SURVEY 8d contract)
    ach_tf = flops / (kern_ms * 1e-3) * 1e-12
    ach_gbs = wl["bytes_per_window"] * n / (kern_ms * 1e-3) * 1e-9
    cfg = config_dict(wl, world)
    if reps > 1:
        cfg["inputs"] = f"{nd} distinct synthetic windows per batch, tiled x{reps} on the device"
    out = {"metric": "imu_windows_per_sec", "value": value, "unit": "windows/s", "n_gpus": world, "steps": steps, "warmup": warmup,
           "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
           "dtype": "f32 storage + f32 covariance RK4, f64 rotations/coefficients/means" if f32 else "f64", "data": "synthetic",
           "config": cfg, "gpu_launches": int(launches), "kernel_ms": kern_ms, **({"exchange": exchange} if exchange else {}),
           "roofline": {"bound": "fp32+fp64 CUDA cores" if f32 else "fp64", "achieved": ach_tf, "peak": FFMA_PEAK_TFLOPS if f32 else DFMA_PEAK_TFLOPS, "unit": "TFLOP/s",
                        "frac": ach_tf / (FFMA_PEAK_TFLOPS if f32 else DFMA_PEAK_TFLOPS),
                        "peak_source": PEAK_SOURCE,
                        **({"contract_vs_executed": "model 2 applies RK4 directly to the consumed Discrete_J_b columns (Phi never formed) and executes fewer "
                                                    "fp64 operations than the survey's 15 k flop/sample contract, so this contract fraction can exceed what the pipe does"}
                           if model == 2 else {}),
                        "note": "CUDA-core FMA bound, not HBM/tensor (85 flop/B); achieved = algorithmic flops (5.8 kflop/sample v1, 15 v2; SURVEY 8d) / "
                                "CUDA-event kernel time (the executed fp64 instruction count is below that contract for v2 -- see DESIGN.md)",
                        "hbm": {"achieved": ach_gbs, "peak": HBM_PEAK_GBS, "unit": "GB/s", "frac": ach_gbs / HBM_PEAK_GBS, "peak_source": PEAK_SOURCE}},
           "clocks": clk}

    # ---- e2e through the C-ABI host entry point, pinned host buffers, H2D + kernel + D2H inside the timed region
    if e2e and not args.no_e2e:
        import ctypes
        S, L = synth.make_windows(nd, ns, rate=wl["rate"], first_window=rank * n)
        hS = torch.from_numpy(S).to(tdt); hL = torch.from_numpy(L).to(tdt)
        if reps > 1:
            hS = hS.repeat(reps, 1, 1)[:n].contiguous(); hL = hL.repeat(reps, 1)[:n].contiguous()
        if world == 1:
            ctx.numa = ctx.pin_to_gpu_numa_node(torch)
        hS = hS.pin_memory(); hL = hL.pin_memory()
        hO = torch.empty((n, rd), dtype=tdt).pin_memory()
        hO.zero_()
        if world == 1:
            os.sched_setaffinity(0, ctx.affinity0)
        del S, L
        sig = np.ascontiguousarray(synth.SIGMAS)
        lib = capi.load()

        def host_step():
            capi.check(lib.cpi_preintegrate_batch_host(model, 8 * es, n, None, ns, ctypes.c_void_p(hS.data_ptr()), ctypes.c_void_p(hL.data_ptr()),
                                                       ctypes.c_void_p(sig.ctypes.data), 0, ctypes.c_void_p(hO.data_ptr())))
        for _ in range(3):
            host_step()
        torch.cuda.synchronize()
        # the floor of this box: a plain pinned cudaMemcpyAsync of the same input bytes (H2D) and output bytes (D2H), back to back
        dprobe = torch.empty_like(hS, device=dev); oprobe = torch.empty((n, rd), dtype=tdt, device=dev)
        for _ in range(2):
            dprobe.copy_(hS, non_blocking=True); hO.copy_(oprobe, non_blocking=True)
        torch.cuda.synchronize()
        tp0 = time.perf_counter()
        for _ in range(5):
            dprobe.copy_(hS, non_blocking=True)
        torch.cuda.synchronize()
        h2d_ms = (time.perf_counter() - tp0) * 1e3 / 5
        tp0 = time.perf_counter()
        for _ in range(5):
            hO.copy_(oprobe, non_blocking=True)
        torch.cuda.synchronize()
        d2h_ms = (time.perf_counter() - tp0) * 1e3 / 5
        del dprobe, oprobe
        if world > 1:
            dist.barrier()
        ke = max(3, min(steps, 10))
        t0 = time.perf_counter()
        for _ in range(ke):
            host_step()
        torch.cuda.synchronize()
        e2e_ms = (time.perf_counter() - t0) * 1e3 / ke
        if world > 1:
            t = torch.tensor([e2e_ms], device=dev, dtype=torch.float64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            e2e_ms = float(t.item())
        out["e2e"] = {"value": world * n / (e2e_ms * 1e-3), "unit": "windows/s", "ms_per_step": e2e_ms,
                      "h2d_bytes_per_step": int(hS.numel() * es + hL.numel() * es), "d2h_bytes_per_step": int(hO.numel() * es),
                      "api": "cpi_preintegrate_batch_host (C ABI, pinned host buffers)",
                      "pcie_floor": {"h2d_ms": h2d_ms, "h2d_gbs": hS.numel() * es / h2d_ms * 1e-6, "d2h_ms": d2h_ms,
                                     "note": "plain pinned cudaMemcpyAsync of the same bytes on this box, measured in this run; the copies run full duplex, so H2D alone is the floor of the host path"}}
        if ctx.numa:
            out["e2e"]["host_numa"] = f"pinned host buffers allocated on the NUMA node of the rank's GPU (rank 0: node {ctx.numa['node']}, {ctx.numa['cpus']} cpus)"
        del hS, hL, hO
    if world > 1:
        # CUDA IPC: every rank drops its mappings of the peers' gather buffers, the ranks meet, and only then are the buffers freed
        torch.cuda.synchronize()
        ctx.comm.unregister()
        dist.barrier()
        torch.cuda.synchronize()
    del batches, gathers
    torch.cuda.empty_cache()

    if cpu and rank == 0 and world == 1 and not args.no_cpu_baseline:
        cores = synth.usable_cpus()
        v0, kind, cores, _ = cpu_arm(wl, max(2 * cores, 64))
        sample = int(min(wl["n"], max(cores, v0 * 10.0)))
        v, kind, cores, dt = cpu_arm(wl, sample)
        out["cpu_baseline"] = {"value": v, "unit": "windows/s", "cores": cores, "cores_online": os.cpu_count(), "kind": kind,
                               "sample": f"{sample} windows x {ns} samples of the same synthetic workload, {dt:.1f} s, "
                                         + ("unmodified reference headers (oracle/_ref), std::thread over windows" if kind == "reference" else "oracle C port")}
    return out


def measure_single(ctx, args, wl, steps=50, dump=None):
    """configs[0]: ONE 100-sample window -- for the GPU arm this is launch latency (one CTA, three lanes)."""
    import torch
    from cpi_b200 import preint, synth
    S, L = synth.make_windows(1, wl["ns"], rate=wl["rate"], special=False)
    dS, dL = torch.from_numpy(S).cuda(), torch.from_numpy(L).cuda()
    out = torch.empty((1, 290), dtype=torch.float64, device="cuda")
    stream = torch.cuda.current_stream()
    for _ in range(20):
        preint.preintegrate(1, dS, dL, synth.SIGMAS, 0, ns=wl["ns"], out=out, stream=stream)
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for a, b in evs:
        a.record(stream); preint.preintegrate(1, dS, dL, synth.SIGMAS, 0, ns=wl["ns"], out=out, stream=stream); b.record(stream)
    torch.cuda.synchronize()
    ms = float(np.median([a.elapsed_time(b) for a, b in evs]))
    if dump:
        dump_outputs(dump, {"records": out})
    hS, hL = S.copy(), L.copy()
    for _ in range(5):
        preint.preintegrate_host(1, hS, hL, synth.SIGMAS, 0, ns=wl["ns"])
    t0 = time.perf_counter()
    for _ in range(50):
        preint.preintegrate_host(1, hS, hL, synth.SIGMAS, 0, ns=wl["ns"])
    e2e_ms = (time.perf_counter() - t0) * 1e3 / 50
    return {"metric": "imu_windows_per_sec", "value": 1e3 / ms, "unit": "windows/s", "kernel_ms": ms, "config": config_dict(wl, 1),
            "roofline": {"frac": None, "note": "one window is a chain of 100 dependent samples on three lanes: pure latency, no roofline applies"},
            "e2e": {"value": 1e3 / e2e_ms, "unit": "windows/s", "ms_per_step": e2e_ms, "h2d_bytes_per_step": 100 * 56 + 104, "d2h_bytes_per_step": 2320}}


def compact(name, r):
    """Entry of the "configs" array: the numbers the judge asked for, not the whole line."""
    if r is None:
        return None
    keep = {k: r.get(k) for k in ("metric", "value", "unit", "n_gpus", "steps", "ms_per_step", "kernel_ms", "dtype", "gpu_launches", "lm_step") if k in r}
    keep["name"] = name
    keep["workload"] = r["config"]["workload"]
    if "inputs" in r["config"]:
        keep["inputs"] = r["config"]["inputs"]
    rf = r.get("roofline") or {}
    keep["roofline"] = {k: rf.get(k) for k in ("bound", "achieved", "peak", "unit", "frac") if k in rf}
    if "e2e" in r:
        keep["e2e"] = r["e2e"]
    return keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default="v1_10k_200", choices=list(WORKLOADS))
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-configs", action="store_true", help="skip the short runs of the other BASELINE configs appended to the default line")
    ap.add_argument("--distinct", type=int, default=0, help="generate only this many distinct windows on the host and tile them on the device (0 = all distinct)")
    ap.add_argument("--no-clocks", action="store_true", help="debug: do not poll nvidia-smi during the timed region")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last timed step computed as DIR/<name>.npy (at most 64 MB in all)")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be >= 1")
    if args.dump_outputs and args.impl != "ours":
        ap.error("--dump-outputs records the GPU path (--impl ours)")
    wl = WORKLOADS[args.workload]
    args.warmup = max(args.warmup, 3) if args.impl == "ours" else args.warmup
    if args.impl == "reference":
        return run_factor(args, wl) if wl.get("factor") else run_reference(args, wl)

    ctx = Ctx()
    if wl.get("factor"):
        if ctx.rank == 0:
            run_factor(args, wl, dump=args.dump_outputs)
        return
    if wl.get("single"):
        if ctx.rank == 0:
            r = measure_single(ctx, args, wl, steps=args.steps, dump=args.dump_outputs)
            r.update({"n_gpus": 1, "steps": args.steps, "warmup": 20, "ms_per_step": r["kernel_ms"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
                      "dtype": "f64", "data": "synthetic", "gpu_launches": args.steps})
            print(json.dumps(r), flush=True)
        return
    out = measure_preint(ctx, args.workload, args, args.steps, args.warmup, distinct=args.distinct or None, e2e=True, cpu=True, dump=args.dump_outputs)

    # ---- the other BASELINE configs, short runs, appended to the default line so that the driver's record carries them
    if args.workload == "v1_10k_200" and not args.no_configs:
        extra = []
        k = max(3, min(args.steps, 10))
        for name, distinct in (("v2_100k_400", 5_000), ("v1_1m_200_fp32", 5_000)):
            try:
                extra.append(compact(name, measure_preint(ctx, name, args, k, 3, distinct=distinct, e2e=(ctx.world == 1), cpu=False, clocks=False)))
            except Exception as ex:     # noqa: BLE001 -- reported in the line, never hidden
                extra.append({"name": name, "error": repr(ex)})
        if ctx.rank == 0:
            class A: pass
            fa = A(); fa.__dict__.update(vars(args)); fa.steps = 20; fa.warmup = 3
            for name, fn in (("factor_5k", lambda: run_factor(fa, WORKLOADS["factor_5k"], emit=False, cpu=False)),
                             ("v1_single_100", lambda: measure_single(ctx, args, WORKLOADS["v1_single_100"]))):
                try:
                    extra.append(compact(name, fn()))
                except Exception as ex:     # noqa: BLE001
                    extra.append({"name": name, "error": repr(ex)})
        out["configs"] = extra
    if ctx.rank == 0:
        print(json.dumps(out), flush=True)
    if ctx.world > 1:
        import torch.distributed as dist
        if ctx.comm:
            ctx.comm.close()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
