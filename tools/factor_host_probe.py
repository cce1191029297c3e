import sys, os, time, ctypes
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from cpi_b200 import capi, synth, preint, factor
lib = capi.load()
n = 4999
S, L = synth.make_windows(n, 20, rate=200.0, first_window=9000)
rec = preint.preintegrate_host(1, S, L, synth.SIGMAS, 0, ns=20)
X = synth.make_states(rec, L, 1)
def run(tag):
    hX, hR, hL = (torch.from_numpy(a).pin_memory() for a in (X, rec, L))
    hE, hH1, hH2 = (torch.empty(sh, dtype=torch.float64).pin_memory() for sh in ((n, 15), (n, 225), (n, 225)))
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    ts = []
    for i in range(12):
        t0 = time.perf_counter()
        capi.check(lib.cpi_imu_factor_eval_batch_host(1, n, n + 1, P(hX), None, None, P(hR), P(hL), P(hE), P(hH1), P(hH2)))
        ts.append((time.perf_counter() - t0) * 1e3)
    print(tag, " ".join(f"{t:.2f}" for t in ts), "pinned:", hX.is_pinned(), hH1.is_pinned(), flush=True)
run("fresh")
# a big preintegration through the host entry first (as bench's configs do), then again
S2, L2 = synth.make_windows(2500, 200)
hS = torch.from_numpy(S2).repeat(4, 1, 1).contiguous().pin_memory(); hL2 = torch.from_numpy(L2).repeat(4, 1).contiguous().pin_memory(); hO = torch.empty((10000, 290), dtype=torch.float64).pin_memory()
sig = np.ascontiguousarray(synth.SIGMAS)
for _ in range(3):
    capi.check(lib.cpi_preintegrate_batch_host(1, 64, 10000, None, 200, ctypes.c_void_p(hS.data_ptr()), ctypes.c_void_p(hL2.data_ptr()), ctypes.c_void_p(sig.ctypes.data), 0, ctypes.c_void_p(hO.data_ptr())))
run("after big host preint")
del hS, hL2, hO
run("after freeing pinned")
