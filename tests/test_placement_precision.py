"""A window's record does not depend on where the batch puts it, and trailing null steps change nothing.

Placement (tests/placement_stress.py): the 424 stress windows copied into every thread slot the preintegration kernels index by
position -- lanes 16-31 and every warp of a full round-1 CTA, every trio slot of the tri-lane kernel, quiet warps and warps
that run to 10 000 samples, both 16-byte phases in fp64 and all four TMA shifts in fp32 -- in one CSR batch of sms * 128 + r
windows, so the round-1 kernels run at their tile capacity S with a full wave and a partial last CTA.  All six (model, flags)
modes, fp64 and fp32:
  * every copy is bitwise the record of the same window in the plain stress-batch run (round-1 CTAs of 4 windows there);
    empty windows give the fresh-object record;
  * the distinct windows pass the conditioned gate of tests/test_precision.py with its constants;
  * the host entry (over 16 MB and >= 8 x SMs windows: the chunked pipeline) is bitwise the device call.

Null steps: every stress window except the long ones padded to 300 entries with copies of its last entry at dt = 0 (before
the imu_avg layout is formed, so the last real step reads the same trailing reading).  The reference skips dt == 0
(CpiV1.h:72-74), so the device record is bitwise the unpadded one.  Tiled so that the fp64 default modes take the host
entry's wavefront schedule: windows that travel whole are bitwise, the others (sample segments through continuation kernels)
pass the conditioned gate."""
import os
import subprocess

import numpy as np
import pytest

import placement_stress
import stress
import test_precision as tp
from parity import imu_avg_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GATE_PATH = {0: "device", 1: "avg", 2: "ana", 3: "ana_avg"}
NS_PAD = 300
PAD_TILES = 30          # 12 630 windows x 300 samples = 212 MB in fp64: the wavefront takes the tail of the batch, not all of it
SEG_BYTES = {1: 231e3, 2: 344e3}     # capi.cu, cpi_preintegrate_batch_host: bytes per sample of the wavefront group


@pytest.fixture(scope="session")
def oracle_ld():
    if np.finfo(np.longdouble).nmant < 63:
        pytest.skip("long double has no extended precision on this platform")
    from oracle import oracle as om
    if not os.path.exists(om.OracleLD.path):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "liboracle_ld.so"], check=True)
    return om.OracleLD()


def fresh_record(model, dtype):
    """The record of an object that was never fed: q = (0, 0, 0, 1) (JPL), R = I, everything else zero."""
    rec = np.zeros(308 if model == 2 else 290, dtype=dtype)
    rec[3] = 1.0
    rec[4:13] = np.eye(3).reshape(-1)
    return rec


def padded_batch(S, off, L, tags):
    """(samples [n * 300, 7], lin, distinct window per row): every window but the long ones, padded to NS_PAD entries at dt = 0 and
    tiled PAD_TILES times.  An empty window is padded with zero readings."""
    keep = np.flatnonzero(tags != "long")
    P = np.zeros((len(keep), NS_PAD, 7))
    for j, i in enumerate(keep):
        w = S[off[i]:off[i + 1]]
        P[j, :len(w)] = w
        if len(w):
            P[j, len(w):] = w[-1]
            P[j, len(w):, 6] = 0.0
    idx = np.tile(keep, PAD_TILES)
    return np.ascontiguousarray(np.tile(P.reshape(-1, 7), (PAD_TILES, 1))), np.ascontiguousarray(L[idx]), idx


def wave_head(model, n, in_bytes, ns, sms):
    """Windows [0, head) of a uniform fp64 default-mode batch travel whole through the host entry, the rest as the wavefront
    (capi.cu, cpi_preintegrate_batch_host: one group of 4 segments sized by SEG_BYTES, ten-window CTAs)."""
    wpb = min(-(-n // sms), 10)
    blocks = -(-n // wpb)
    frac = ns * SEG_BYTES[model] / in_bytes
    H = 0 if frac >= 1.0 else min(int(100.0 * (1.0 - frac)), 95)
    return blocks * H // 100 * wpb


# ---------------------------------------------------------------------------------------------------------- CPU

@pytest.mark.parametrize("sms", [132, 114])
def test_placement_batch_covers_every_slot(sms):
    S, off, L, idx = placement_stress.make_placement_batch(sms)        # asserts the coverage
    S0, off0, L0, tags = stress.make_batch()
    assert len(idx) == sms * 128 + placement_stress.pick_r(sms)
    for g in (0, len(idx) // 2, len(idx) - 1):
        w = idx[g]
        assert np.array_equal(S[off[g]:off[g + 1]], S0[off0[w]:off0[w + 1]]) and np.array_equal(L[g], L0[w])
    print(sms, "SMs:", len(idx), "windows,", len(S), "samples, copies per window", np.bincount(idx).min(), "-", np.bincount(idx).max())


def test_padded_batch_is_the_same_function(oracle):
    """The fp64 oracle gives the padded windows (and imu_avg's layout of them) the unpadded records bit for bit, and an empty
    window the fresh record."""
    S, off, L, tags = stress.make_batch(n_long=0)
    P, LP, idx = padded_batch(S, off, L, tags)
    k = len(np.flatnonzero(tags != "long"))
    for model, flags in tp.MODES:
        Sx, ox = (imu_avg_inputs(S, off) if flags & 1 else (S, off))
        plain = oracle.preintegrate(model, Sx, L, tp.SIGMAS, flags, offsets=ox, nthreads=tp._threads())
        Px = imu_avg_inputs(P[:k * NS_PAD], np.arange(k + 1) * NS_PAD)[0] if flags & 1 else P[:k * NS_PAD]
        pad = oracle.preintegrate(model, Px, LP[:k], tp.SIGMAS, flags, ns=NS_PAD, nthreads=tp._threads())
        assert np.array_equal(pad, plain[idx[:k]]), (model, flags)
        assert np.array_equal(plain[np.diff(off) == 0], np.broadcast_to(fresh_record(model, np.float64), plain[np.diff(off) == 0].shape))


# ---------------------------------------------------------------------------------------------------------- GPU

@pytest.fixture(scope="module")
def stress_batch():
    return stress.make_batch()


@pytest.fixture(scope="module")
def placement(cuda):
    sms = cuda.cuda.get_device_properties(0).multi_processor_count
    return sms, placement_stress.make_placement_batch(sms)


def _dev(torch, preint, model, flags, Sx, Lx, off=None, ns=None):
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    out = preint.preintegrate(model, d(Sx), d(Lx), tp.SIGMAS, flags, offsets=None if off is None else d(off), ns=ns)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _layout(S, off, flags):
    return imu_avg_inputs(S, off) if flags & 1 else (S, off)


def _first_mismatch(got, want, idx):
    bad = np.flatnonzero(~np.all(got == want, axis=1))
    if not len(bad):
        return None
    g = int(bad[0])
    slots = ", ".join(f"S={S}: CTA {g // S} thread {g % S}" for S in placement_stress.ROUND1_S)
    return f"{len(bad)} of {len(got)} differ; first at position {g} (stress window {idx[g]}; trio slot {g % 10}; {slots})"


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("model,flags", tp.MODES)
def test_every_slot_gives_the_same_bits(cuda, oracle, oracle_ld, placement, stress_batch, model, flags, dtype):
    from cpi_b200 import preint
    sms, (PS, Poff, PL, idx) = placement
    S, off, L, tags = stress_batch
    Sx, ox = _layout(S.astype(dtype), off, flags)
    plain = _dev(cuda, preint, model, flags, Sx, L.astype(dtype), ox)
    PSx, Pox = _layout(PS.astype(dtype), Poff, flags)
    got = _dev(cuda, preint, model, flags, PSx, PL.astype(dtype), Pox)
    msg = _first_mismatch(got, plain[idx], idx)
    assert msg is None, msg
    empty = np.diff(off) == 0
    assert np.array_equal(plain[empty], np.broadcast_to(fresh_record(model, dtype), plain[empty].shape))
    # the distinct windows (their first copies) through the conditioned gate
    first = np.unique(idx, return_index=True)[1]
    o64, truth = tp._oracles(oracle, oracle_ld, model, dtype, flags, S, off, L)
    ratio, worst, bad = tp.gate(model, dtype, GATE_PATH[flags], got[first], o64, truth, np.maximum(np.diff(off), 1))
    tp.report(f"placement m{model} f{flags} {np.dtype(dtype).name}", ratio, tags)
    assert not bad, bad
    # the host entry cuts the batch into chunks of whole CTAs: the same bits
    assert PSx.nbytes >= 16 << 20 and len(idx) >= 8 * sms
    host = preint.preintegrate_host(model, PSx, PL.astype(dtype), tp.SIGMAS, flags, offsets=Pox)
    msg = _first_mismatch(host, got, idx)
    assert msg is None, "host entry: " + msg


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("model,flags", tp.MODES)
def test_null_steps_change_no_bit(cuda, oracle, oracle_ld, stress_batch, model, flags, dtype):
    from cpi_b200 import preint
    S, off, L, tags = stress_batch
    sms = cuda.cuda.get_device_properties(0).multi_processor_count
    Sx, ox = _layout(S.astype(dtype), off, flags)
    plain = _dev(cuda, preint, model, flags, Sx, L.astype(dtype), ox)
    P, LP, idx = padded_batch(S, off, L, tags)
    n = len(idx)
    Px = P.astype(dtype)
    if flags & 1:
        Px = imu_avg_inputs(Px, np.arange(n + 1) * NS_PAD)[0]
    LPx = LP.astype(dtype)
    got = _dev(cuda, preint, model, flags, Px, LPx, ns=NS_PAD)
    msg = _first_mismatch(got, plain[idx], idx)
    assert msg is None, msg
    host = preint.preintegrate_host(model, Px, LPx, tp.SIGMAS, flags, ns=NS_PAD)
    wave = dtype == np.float64 and not flags
    head = wave_head(model, n, Px.nbytes, NS_PAD, sms) if wave else n
    assert n >= 8 * sms and Px.nbytes >= 16 << 20 and (not wave or 0 < head < n), (n, head)
    msg = _first_mismatch(host[:head], got[:head], idx)
    assert msg is None, "host entry: " + msg
    if head < n:        # the wavefront: sample segments through continuation kernels, held to the gate
        o64, truth = tp._oracles(oracle, oracle_ld, model, dtype, flags, S, off, L)
        t = idx[head:]
        ratio, worst, bad = tp.gate(model, dtype, "cont", host[head:], o64[t], truth[t], np.maximum(np.diff(off), 1)[t])
        tp.report(f"null steps wavefront m{model} ({n - head} windows)", ratio, tags[t])
        assert not bad, bad
