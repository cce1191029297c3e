"""Timing of the iterated filter update by measurements (K13, DESIGN.md section 3m) against the single update K11.

    python tools/update_iterated_probe.py [--reps 50]

Prints ONE JSON line:
  gpu / power_limit_w          the card the numbers come from (read in the same run)
  k11_10k_ms                   cpi_state_update_measurements_batch on 10 000 filters, one lever-arm GNSS and one direction each
  k13_1_10k_ms                 cpi_state_update_measurements_iterated_batch on the same filters, one iteration (tol = +inf)
  k13_3_10k_ms / k13_10_10k_ms  the same at exactly 3 and 10 iterations (tol = 0)
  k13_3_1m                     10^6 such filters at 3 iterations, against the HBM bound of the bytes a filter moves once: 2 184 in
                               (state 128, cov 1 800, offset 8, two measurements of kind 4, z 24, S 72, aux 24) and 1 944 out (state
                               128, cov 1 800, nis 8, status 4, iterations 4) at the H100 SXM data-sheet 3.35 TB/s
The CSR and the inputs are built beforehand; every call is one raw kernel launch.  CUDA events, median over --reps.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from scan_probe import HBM_BPS, gpu_identity, timed  # noqa: E402

BYTES_IN, BYTES_OUT = 128 + 1800 + 8 + 2 * (4 + 24 + 72 + 24), 128 + 1800 + 8 + 4 + 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("update_iterated_probe needs a CUDA device")
    from cpi_b200 import capi, factor
    lib = capi.load()
    p = factor._tptr
    dev = torch.device("cuda")
    f64 = dict(dtype=torch.float64, device=dev)
    name, power = gpu_identity()
    out = {"gpu": name, "power_limit_w": power}

    def filters(n):
        """n filters near a unit attitude with a lever-arm GNSS fix (1 cm) and a direction (0.01) each, 2 cm and 0.02 off."""
        X = torch.zeros((n, 16), **f64)
        q = torch.randn((n, 4), **f64)
        X[:, 0:4] = q / q.norm(dim=1, keepdim=True)
        X[:, 4:16] = torch.randn((n, 12), **f64)
        rc = torch.randn((n, 15, 15), **f64)
        C = (rc @ rc.transpose(1, 2) * 1e-4 + torch.eye(15, **f64) * 1e-4).transpose(1, 2).reshape(n, 225).contiguous()
        offs = torch.arange(n + 1, dtype=torch.int64, device=dev) * 2
        kind = torch.tensor([capi.MEAS_POSITION, capi.MEAS_DIRECTION], dtype=torch.int32, device=dev).repeat(n)
        aux = torch.tensor([[0.5, 0.2, 1.0], [0.6, 0.0, 0.8]], **f64).repeat(n, 1)
        z = torch.randn((2 * n, 3), **f64) * 0.02
        z[0::2] += X[:, 13:16]
        si = torch.from_numpy(np.tile(np.eye(3).reshape(9) * 100.0, (2 * n, 1))).to(dev)
        outs = (torch.empty((n, 16), **f64), torch.empty((n, 225), **f64), torch.empty(n, **f64),
                torch.empty(n, dtype=torch.int32, device=dev), torch.empty(n, dtype=torch.int32, device=dev))
        return X, C, offs, kind, z, si, aux, outs

    def k13(n, F, iters, tol):
        X, C, offs, kind, z, si, aux, (xo, co, nis, st, it) = F
        return lambda: capi.check(lib.cpi_state_update_measurements_iterated_batch(n, p(X), p(C), p(offs), p(kind), p(z), p(si), p(aux),
                                                                                    None, None, None, iters, tol, p(xo), p(co), p(nis),
                                                                                    p(st), p(it), None))

    n = 10_000
    F = filters(n)
    X, C, offs, kind, z, si, aux, (xo, co, nis, st, it) = F
    out["k11_10k_ms"] = timed(torch, lambda: capi.check(lib.cpi_state_update_measurements_batch(n, p(X), p(C), p(offs), p(kind), p(z), p(si),
                                                                                                p(aux), None, p(xo), p(co), p(nis), p(st),
                                                                                                None)), args.reps)
    out["k13_1_10k_ms"] = timed(torch, k13(n, F, 1, float("inf")), args.reps)
    out["k13_3_10k_ms"] = timed(torch, k13(n, F, 3, 0.0), args.reps)
    out["k13_10_10k_ms"] = timed(torch, k13(n, F, 10, 0.0), args.reps)
    torch.cuda.synchronize()
    out["k13_iterations_10k"] = sorted(set(it.cpu().tolist()))
    del F, X, C, offs, kind, z, si, aux, xo, co, nis, st, it
    n = 1_000_000
    F = filters(n)
    ms = timed(torch, k13(n, F, 3, 0.0), args.reps)
    bound = n * (BYTES_IN + BYTES_OUT) / HBM_BPS * 1e3
    out["k13_3_1m"] = {"ms": ms, "hbm_bound_ms": bound, "share_of_bound": bound / ms}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
