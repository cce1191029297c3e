"""Scalar pre-pass of the tri-lane preintegration kernels (models 1 and 2, fp64 and fp32): the branch-free pre-pass gives, bit for
bit, the records of a launch that computes every group's scalar sets with the IEEE operations (CPI_B200_TRI_IEEE_PREPASS=1).
The batch mixes, inside one warp, small-|w| (Taylor) windows with closed-form ones, an exactly zero w_hat, dt = 0 steps and windows of
0, 1, 2, 4 and 5 samples (group and staging-ring edges); another warp holds inputs outside the fast primitives' domains (subnormal
and huge dt, |w dt| beyond the sincos fast path, NaN), which that warp recomputes with the IEEE operations; the records are then
continued by a second call."""
import os

import numpy as np
import pytest
import torch

from cpi_b200 import capi, preint, synth

pytestmark = pytest.mark.gpu

N = 37                                   # ten windows per warp: warps 0..2 full, warp 3 partly empty
NS = 40


def _batch(first_window, fp32):
    S, L = synth.make_windows(N, NS, first_window=first_window, special=False)
    bw = L[:, 0:3]
    lens = np.full(N, NS, dtype=np.int64)
    # warp 0: every step kind the fast pre-pass handles, side by side
    for w in (1, 5):                                              # whole window in the Taylor branch, next to closed-form windows
        S[w, :, 0:3] = bw[w] + 1e-3 * (S[w, :, 0:3] - bw[w]) / np.linalg.norm(S[w, :, 0:3] - bw[w], axis=1, keepdims=True)
    S[2, :, 0:3] = bw[2]                                          # w_hat exactly 0
    S[6, 3:9, 0:3] = bw[6] + 1e-4                                 # a few Taylor steps inside a closed-form window
    S[0, [0, 4, 17], 6] = 0.0                                     # dt = 0 steps
    lens[3], lens[4], lens[7], lens[8], lens[9] = 4, 5, 0, 1, 2
    # warp 1: inputs outside the fast primitives' domains
    S[10, 5, 6] = 1e-40 if fp32 else 5e-320                       # subnormal dt
    S[11, 7, 6] = 1e30 if fp32 else 1e300                         # huge dt
    S[12, 2:4, 0] = 1e12                                          # |w dt| >= 2^31: Payne-Hanek reduction in sincos
    S[13, 9, 1] = np.nan
    S[14, 11, 6] = np.nan
    # warp 2: one out-of-domain group in an otherwise ordinary warp
    S[23, 20, 2] = 1e12
    flat = [np.full((1, 7), 0.5)] + [S[i, :lens[i]] for i in range(N)]
    off = np.zeros(N + 1, dtype=np.int64)
    off[0] = 1
    off[1:] = 1 + np.cumsum(lens)
    return np.concatenate(flat), L, off


def _launch(ieee, model, S, L, off, tdt, init=None):
    rd = capi.REC_DOUBLES[model]
    n = L.shape[0]
    out = torch.zeros((n, rd), dtype=tdt, device="cuda")
    if init is not None:
        out.copy_(torch.from_numpy(init))
    prev = os.environ.get("CPI_B200_TRI_IEEE_PREPASS")
    os.environ["CPI_B200_TRI_IEEE_PREPASS"] = "1" if ieee else "0"
    try:
        args = (model, torch.from_numpy(S).to(tdt).cuda(), torch.from_numpy(L).to(tdt).cuda(), synth.SIGMAS, 0)
        offsets = torch.from_numpy(off).cuda()
        if init is None:
            preint.preintegrate(*args, offsets=offsets, out=out)
        else:
            preint.preintegrate(*args, offsets=offsets, continue_records=out)
        torch.cuda.synchronize()
    finally:
        if prev is None:
            del os.environ["CPI_B200_TRI_IEEE_PREPASS"]
        else:
            os.environ["CPI_B200_TRI_IEEE_PREPASS"] = prev
    return out.cpu().numpy()


def _same_bits(a, b):
    assert a.dtype == b.dtype and a.shape == b.shape
    diff = np.nonzero(a.view(np.uint8) != b.view(np.uint8))[0]
    assert diff.size == 0, f"{diff.size} bytes differ, first in window {diff[0] // (a.itemsize * a.shape[1])}"


@pytest.mark.parametrize("model", [1, 2])
@pytest.mark.parametrize("fp32", [False, True])
def test_branch_free_prepass_matches_ieee_prepass(cuda, model, fp32):
    tdt = torch.float32 if fp32 else torch.float64
    S, L, off = _batch(0, fp32)
    ref = _launch(True, model, S, L, off, tdt)
    assert np.all(np.isfinite(ref[:10]))                         # warp 0 holds no absurd input
    _same_bits(_launch(False, model, S, L, off, tdt), ref)

    S2, _, off2 = _batch(1000, fp32)                              # continuation from those records
    ref2 = _launch(True, model, S2, L, off2, tdt, init=ref)
    _same_bits(_launch(False, model, S2, L, off2, tdt, init=ref), ref2)
