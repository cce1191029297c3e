#!/usr/bin/env python
"""In-process A/B of the host entry point's schedules (CPI_B200_HOST_WAVE = "G,S[,H]") on BASELINE configs[1], next to the raw PCIe
numbers of the box: one plain pinned H2D of the same bytes, and the same bytes as strided 2-D tile copies:
    python tools/host_pipeline_probe.py > host_probe.json"""
import ctypes, json, os, statistics, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from cpi_b200 import capi, synth

SPECS = sys.argv[1].split(";") if len(sys.argv) > 1 else ["0,0", "1,8,60", "1,4,60", "2,8,50", "4,8,40", "4,4,40", "14,8", "6,4", "8,2", "1,8,70", "2,8,70"]
n, ns = 10000, 200
dev = torch.device("cuda", 0)
torch.cuda.set_device(0)
lib = capi.load()
# pinned buffers on the GPU's NUMA node
numa = None
try:
    pr = torch.cuda.get_device_properties(dev)
    base = f"/sys/bus/pci/devices/{pr.pci_domain_id:04x}:{pr.pci_bus_id:02x}:{pr.pci_device_id:02x}.0"
    cpus = set()
    for part in open(f"{base}/local_cpulist").read().strip().split(","):
        a, _, b = part.partition("-"); cpus.update(range(int(a), int(b or a) + 1))
    cpus &= os.sched_getaffinity(0)
    if cpus:
        os.sched_setaffinity(0, cpus); numa = {"node": int(open(f"{base}/numa_node").read()), "cpus": len(cpus)}
except Exception as ex:      # noqa: BLE001
    numa = {"error": str(ex)}
S, L = synth.make_windows(2500, ns)
hS = torch.from_numpy(S).repeat(4, 1, 1).contiguous().pin_memory(); hL = torch.from_numpy(L).repeat(4, 1).contiguous().pin_memory()
hO = torch.empty((n, 290), dtype=torch.float64).pin_memory()
sig = np.ascontiguousarray(synth.SIGMAS)
out = {"numa": numa, "bytes_in": hS.numel() * 8}

# ---- raw copies
rt = ctypes.CDLL("libcudart.so.12")
rt.cudaMemcpy2DAsync.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p]
rt.cudaMemcpyAsync.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p]
dS = torch.empty_like(hS, device=dev)
st = torch.cuda.Stream()
def timed(fn, reps=7):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize(); t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)
def copy1d():
    rt.cudaMemcpyAsync(dS.data_ptr(), hS.data_ptr(), hS.numel() * 8, 1, st.cuda_stream)
out["h2d_1d_ms"] = timed(copy1d)
def copy2d(G, Sg):
    def f():
        wg = n // G; seg = ns // Sg
        for g in range(G):
            for s in range(Sg):
                rt.cudaMemcpy2DAsync(dS.data_ptr() + (g * wg * ns + wg * s * seg) * 56, seg * 56, hS.data_ptr() + (g * wg * ns + s * seg) * 56, ns * 56, seg * 56, wg, 1, st.cuda_stream)
    return f
for G, Sg in ((1, 8), (4, 8), (14, 8), (14, 4), (1, 2), (32, 8)):
    out[f"h2d_2d_G{G}_S{Sg}_ms"] = timed(copy2d(G, Sg))
del dS

def step():
    capi.check(lib.cpi_preintegrate_batch_host(1, 64, n, None, ns, ctypes.c_void_p(hS.data_ptr()), ctypes.c_void_p(hL.data_ptr()), ctypes.c_void_p(sig.ctypes.data), 0,
                                               ctypes.c_void_p(hO.data_ptr())))
res = {s: {"total": [], "submit": []} for s in SPECS}
sub, tot = ctypes.c_double(), ctypes.c_double()
for rnd in range(4):
    for spec in SPECS:
        os.environ["CPI_B200_HOST_WAVE"] = spec
        step(); step()
        for _ in range(8):
            t0 = time.perf_counter(); step(); dt = (time.perf_counter() - t0) * 1e3
            lib.cpi_host_last_timing(ctypes.byref(sub), ctypes.byref(tot))
            res[spec]["total"].append(dt); res[spec]["submit"].append(sub.value)
out["schedules"] = {s: {"e2e_ms_median": round(statistics.median(v["total"]), 4), "e2e_ms_min": round(min(v["total"]), 4), "submit_ms_median": round(statistics.median(v["submit"]), 4)}
                    for s, v in res.items()}
print(json.dumps(out, indent=1))
