"""Sample staging and record write of the tri-lane preintegration kernels (models 1 and 2, fp64 and fp32): the TMA-staged sample
stream, the tail samples that the pre-pass copies into the staging ring and the record written through shared memory give, bit for
bit, the records of a launch that stages nothing by TMA and reads every sample from global memory (CPI_B200_TRI_NO_TMA=1).
The windows are ragged (lengths that are not multiples of 3 or of a TMA chunk, empty and one-sample windows), start at odd sample
offsets (misaligned TMA sources), leave the last one-warp CTA partly empty, are written to output slices that are not 16-byte
aligned, and are continued by a second call."""
import os

import numpy as np
import pytest
import torch

from cpi_b200 import capi, preint, synth

pytestmark = pytest.mark.gpu

N = 37                                   # ten windows per CTA: the last CTA holds seven
SENTINEL = 12345.0


def _windows(n, lens, first_window, lead):
    """Samples of n windows of the given lengths, packed after `lead` unused samples, and their CSR offsets."""
    S, L = synth.make_windows(n, int(max(lens)), first_window=first_window)
    flat = [np.full((lead, 7), 0.5)] + [S[i, :lens[i]] for i in range(n)]
    off = np.zeros(n + 1, dtype=np.int64)
    off[0] = lead
    off[1:] = lead + np.cumsum(lens)
    return np.concatenate(flat), L, off


def _launch(no_tma, model, S, L, off, out_shift, tdt, init=None):
    """Records of one call written into a sentinel-filled buffer at element offset out_shift; the sentinel must survive around them."""
    rd = capi.REC_DOUBLES[model]
    n = L.shape[0]
    buf = torch.full((out_shift + n * rd + 7,), SENTINEL, dtype=tdt, device="cuda")
    out = buf[out_shift:out_shift + n * rd].view(n, rd)
    if init is not None:
        out.copy_(torch.from_numpy(init).to(tdt))
    prev = os.environ.get("CPI_B200_TRI_NO_TMA")
    os.environ["CPI_B200_TRI_NO_TMA"] = "1" if no_tma else "0"
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
            del os.environ["CPI_B200_TRI_NO_TMA"]
        else:
            os.environ["CPI_B200_TRI_NO_TMA"] = prev
    b = buf.cpu().numpy()
    assert np.all(b[:out_shift] == SENTINEL) and np.all(b[out_shift + n * rd:] == SENTINEL), "written outside the records"
    return b[out_shift:out_shift + n * rd].reshape(n, rd).copy()


def _same_bits(a, b):
    assert a.dtype == b.dtype and a.shape == b.shape
    diff = np.nonzero(a.view(np.uint8) != b.view(np.uint8))[0]
    assert diff.size == 0, f"{diff.size} bytes differ, first in window {diff[0] // (a.itemsize * a.shape[1])}"


@pytest.mark.parametrize("model", [1, 2])
@pytest.mark.parametrize("fp32", [False, True])
def test_staged_stream_and_record_write_match_global_loads(cuda, model, fp32):
    tdt = torch.float32 if fp32 else torch.float64
    lens = np.array([(7 * i + 1) % 23 + (40 if i % 5 == 0 else 0) for i in range(N)], dtype=np.int64)
    lens[3], lens[4], lens[N - 1] = 0, 1, 2
    S, L, off = _windows(N, lens, 0, lead=1)
    ref = _launch(True, model, S, L, off, 0, tdt)
    assert np.all(np.isfinite(ref))
    for out_shift in (0, 1, 3):                                     # 16-byte stores, and the element-store fallback
        _same_bits(_launch(False, model, S, L, off, out_shift, tdt), ref)

    # continuation from those records, with windows that now start at an even offset and have other lengths
    lens2 = np.array([(5 * i + 2) % 17 for i in range(N)], dtype=np.int64)
    S2, _, off2 = _windows(N, lens2, 1000, lead=2)
    ref2 = _launch(True, model, S2, L, off2, 0, tdt, init=ref)
    for out_shift in (0, 1):
        _same_bits(_launch(False, model, S2, L, off2, out_shift, tdt, init=ref), ref2)
