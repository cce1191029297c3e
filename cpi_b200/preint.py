"""Host-side mirror of the reference preintegrator interface (cpi/CpiBase.h, cpi/CpiV1.h, cpi/CpiV2.h) on top of the
C ABI, plus the batch entry points the kernels are built for.

Reference surface kept (same names, argument meaning, public result fields):

    CpiV1(sigma_w, sigma_wb, sigma_a, sigma_ab, imu_avg_=False)            CpiV1.h:53
    .setLinearizationPoints(b_w_lin, b_a_lin, q_k_lin=0, grav=0)           CpiBase.h:73
    .feed_IMU(t_0, t_1, w_m_0, a_m_0, w_m_1=0, a_m_1=0)                    CpiBase.h:86
    fields  DT alpha_tau beta_tau q_k2tau R_k2tau J_q J_a J_b H_a H_b P_meas (O_a O_b, state_transition_jacobians)

One honest difference (SURVEY.md section 8b): the reference updates its fields eagerly inside every feed_IMU; here
feed_IMU only appends the step to a host staging list and the fields are populated by ``finalize()`` (one window) or by
``flush([cpi, ...])`` (many windows, ONE kernel launch) -- the call a maintainer adds after the feed loop at
solvers/GraphSolver_IMU.cpp:69 / :124.  Reading a result field before that raises.

Nothing here computes on the CPU: every result comes out of libcpi_b200.so.  The device entry points keep the stream contract of
cpi_b200.factor: a call with ``stream=S`` runs wholly on S, and the caller orders its inputs before and its consumers after.
"""
from __future__ import annotations

import ctypes

import numpy as np

from . import capi
from .capi import FLAG_ANALYTIC_JACOBIANS, FLAG_IMU_AVG, REC, REC_DOUBLES
from .factor import _launch, _on, _tptr

_RESULT_FIELDS = ("DT", "alpha_tau", "beta_tau", "q_k2tau", "R_k2tau", "J_q", "J_a", "J_b", "H_a", "H_b", "P_meas", "O_a", "O_b")


def _ptr(a):
    return None if a is None else ctypes.c_void_p(a.ctypes.data)


# ------------------------------------------------------------------------------------------------------------------
# batch entry points
# ------------------------------------------------------------------------------------------------------------------

def preintegrate_host(model, samples, lin, sigmas, flags=0, offsets=None, ns=None, dtype=None):
    """HOST numpy in, HOST numpy out, through ``cpi_preintegrate_batch_host`` (H2D + kernel + D2H inside the call).

    samples: (entries, 7) [wx wy wz ax ay az dt];  lin: (n, 13);  offsets: int64 (n+1) or None with uniform ``ns``.
    dtype: np.float64 (default) or np.float32 = the fp32-storage variant (float samples / lin / records; DESIGN.md section 3a).
    Returns records (n, 290|308) in that dtype."""
    lib = capi.load()
    if dtype is None:
        dtype = np.float32 if getattr(samples, "dtype", None) == np.float32 else np.float64
    dtype = np.dtype(dtype)
    if dtype not in (np.dtype(np.float64), np.dtype(np.float32)):
        raise ValueError("dtype must be float64 or float32")
    capi.check_discrete(model, 8 * dtype.itemsize, flags)
    samples = np.ascontiguousarray(samples, dtype=dtype).reshape(-1, 7)
    lin = np.ascontiguousarray(lin, dtype=dtype).reshape(-1, 13)
    sig = np.ascontiguousarray(sigmas, dtype=np.float64)
    n = lin.shape[0]
    avg = 1 if flags & FLAG_IMU_AVG else 0
    if offsets is not None:
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        if offsets.shape[0] != n + 1:
            raise ValueError("offsets must have n_windows + 1 entries")
        if n and offsets[-1] > samples.shape[0]:
            raise ValueError("offsets run past the sample array")
        ns = 0
    else:
        if ns is None:
            ns = samples.shape[0] // max(n, 1) - avg
        if samples.shape[0] < n * (ns + avg):
            raise ValueError("sample array shorter than n_windows * (ns + imu_avg)")
    out = np.empty((n, REC_DOUBLES[model]), dtype=dtype)
    capi.check(lib.cpi_preintegrate_batch_host(model, 8 * dtype.itemsize, n, _ptr(offsets), int(ns), _ptr(samples), _ptr(lin), _ptr(sig),
                                               int(flags), _ptr(out)))
    return out


def preintegrate(model, samples, lin, sigmas, flags=0, offsets=None, ns=None, out=None, stream=None, continue_records=None):
    """DEVICE torch tensors in/out (float64 -- or float32 for the fp32-storage variant --, contiguous, all on the current
    CUDA device); enqueues on ``stream`` (a torch.cuda.Stream; default: torch's current stream) and does not synchronise.
    ``continue_records``: records of an earlier call, updated IN PLACE with the new samples (cpi_preintegrate_batch_continue -- the batched
    form of calling feed_IMU again on existing objects) and returned."""
    import torch

    lib = capi.load()
    if not (samples.is_cuda and lin.is_cuda):
        raise ValueError("preintegrate() takes CUDA tensors; use preintegrate_host() for host arrays")
    if samples.dtype not in (torch.float64, torch.float32) or lin.dtype != samples.dtype:
        raise ValueError("samples and lin must both be float64 or both float32")
    tdt = samples.dtype
    dev = samples.device
    capi.check_discrete(model, 64 if tdt == torch.float64 else 32, flags)
    if continue_records is not None:
        if out is not None:
            raise ValueError("give either out or continue_records")
        out = continue_records
    for name, t in (("lin", lin), ("offsets", offsets), ("out", out)):
        if t is not None and t.device != dev:
            raise ValueError(f"{name} lives on {t.device}, samples on {dev}: all tensors of one call must be on the same CUDA device")
    n = lin.numel() // 13
    avg = 1 if flags & FLAG_IMU_AVG else 0
    if offsets is not None:
        if offsets.dtype != torch.int64 or offsets.numel() != n + 1:
            raise ValueError("offsets must be int64 with n_windows + 1 entries")
        ns = 0
    else:
        if ns is None:
            ns = (samples.numel() // 7) // max(n, 1) - avg
        if samples.numel() // 7 < n * (ns + avg):
            raise ValueError("sample tensor shorter than n_windows * (ns + imu_avg)")
    if out is not None and (out.numel() < n * REC_DOUBLES[model] or not out.is_contiguous() or out.dtype != tdt):
        raise ValueError("out must be a contiguous tensor of n_windows * record_doubles in the input dtype")
    sig = np.ascontiguousarray(sigmas, dtype=np.float64)
    with _on(dev, stream):
        samples, lin = samples.contiguous(), lin.contiguous()
        offsets = None if offsets is None else offsets.contiguous()
        if out is None:
            out = torch.empty((n, REC_DOUBLES[model]), dtype=tdt, device=lin.device)
        _launch(lib.cpi_preintegrate_batch if continue_records is None else lib.cpi_preintegrate_batch_continue, dev, stream, model,
                64 if tdt == torch.float64 else 32, n, _tptr(offsets), int(ns), _tptr(samples), _tptr(lin), _ptr(sig), int(flags), _tptr(out))
    return out


def _merge_layout(n_rec, group_offsets, group, n_offsets):
    """(n_groups, uniform) of a merge call; group_offsets has n_offsets entries (or is None)."""
    if (group_offsets is None) == (group is None):
        raise ValueError("give exactly one of group_offsets (CSR, n_groups + 1 entries) and group (uniform group length)")
    if group_offsets is not None:
        return n_offsets - 1, 0
    group = int(group)
    if group < 1:
        raise ValueError("group must be >= 1 (use group_offsets for empty groups)")
    if n_rec % group:
        raise ValueError(f"{n_rec} records do not split into groups of {group}")
    return n_rec // group, group


def _record_layout(records, lin, group_offsets, group):
    """(n_groups, uniform) of a device merge or scan call, after the checks of lin and group_offsets; copies nothing."""
    import torch

    n_rec = records.numel() // REC_DOUBLES[1]
    if lin.numel() != 13 * n_rec:
        raise ValueError("lin must hold one linearisation point per record")
    if group_offsets is not None and group_offsets.dtype != torch.int64:
        raise ValueError("group_offsets must be int64")
    return _merge_layout(n_rec, group_offsets, group, 0 if group_offsets is None else group_offsets.numel())


def merge_host(model, records, lin, group_offsets=None, group=None):
    """Merge consecutive records (``cpi_merge_records_host``): HOST numpy in and out.  records (n, 290) float64 or float32, lin (n, 13)
    in the same dtype, one linearisation point per record; either ``group_offsets`` (int64, n_groups + 1: group g is records
    offsets[g] .. offsets[g+1]-1, in time order) or ``group`` (groups of that many consecutive records).  Returns one record per group,
    at the linearisation point of the group's first record."""
    lib = capi.load()
    records = np.asarray(records)
    dtype = np.dtype(np.float32) if records.dtype == np.float32 else np.dtype(np.float64)
    records = np.ascontiguousarray(records, dtype=dtype).reshape(-1, REC_DOUBLES.get(model, REC_DOUBLES[1]))   # the library rejects model 2
    lin = np.ascontiguousarray(lin, dtype=dtype).reshape(-1, 13)
    if lin.shape[0] != records.shape[0]:
        raise ValueError("lin must hold one linearisation point per record")
    offs = None if group_offsets is None else np.ascontiguousarray(group_offsets, dtype=np.int64)
    n, uniform = _merge_layout(records.shape[0], offs, group, 0 if offs is None else offs.shape[0])
    if offs is not None and offs.shape[0] and offs[-1] > records.shape[0]:
        raise ValueError("group_offsets run past the record array")
    out = np.empty((max(n, 0), records.shape[1]), dtype=dtype)
    capi.check(lib.cpi_merge_records_host(model, 8 * dtype.itemsize, n, _ptr(offs), uniform, _ptr(records), _ptr(lin), _ptr(out)))
    return out


def merge(model, records, lin, group_offsets=None, group=None, out=None, stream=None):
    """Merge consecutive records on the device (``cpi_merge_records``): CUDA tensors (float64, or float32 records and lin), contiguous,
    on one device; enqueues on ``stream`` (default: torch's current stream) and does not synchronise.  Layout as ``merge_host``;
    ``group_offsets`` is an int64 CUDA tensor.  Returns ``out`` (n_groups, 290), which must not overlap ``records``."""
    import torch

    lib = capi.load()
    if not (records.is_cuda and lin.is_cuda):
        raise ValueError("merge() takes CUDA tensors; use merge_host() for host arrays")
    if records.dtype not in (torch.float64, torch.float32) or lin.dtype != records.dtype:
        raise ValueError("records and lin must both be float64 or both float32")
    dev = records.device
    for name, t in (("lin", lin), ("group_offsets", group_offsets), ("out", out)):
        if t is not None and t.device != dev:
            raise ValueError(f"{name} lives on {t.device}, records on {dev}: all tensors of one call must be on the same CUDA device")
    rd = REC_DOUBLES[1]
    n, uniform = _record_layout(records, lin, group_offsets, group)
    if out is not None and (out.numel() < n * rd or not out.is_contiguous() or out.dtype != records.dtype):
        raise ValueError("out must be a contiguous tensor of n_groups * 290 elements in the records' dtype")
    with _on(dev, stream):
        records, lin = records.contiguous(), lin.contiguous()
        group_offsets = None if group_offsets is None else group_offsets.contiguous()
        if out is None:
            out = torch.empty((max(n, 0), rd), dtype=records.dtype, device=dev)
        _launch(lib.cpi_merge_records, dev, stream, model, 64 if records.dtype == torch.float64 else 32, n, _tptr(group_offsets), uniform,
                _tptr(records), _tptr(lin), _tptr(out))
    return out


def scan_host(model, records, lin, group_offsets=None, group=None):
    """Inclusive scan of consecutive records within groups (``cpi_scan_records_host``): HOST numpy in and out, arguments as
    ``merge_host``.  Returns an array shaped like ``records``: row i of group g (lo <= i < hi) is the record of records lo .. i, at the
    linearisation point of record lo (row hi - 1 is the group's ``merge_host`` result up to rounding, row lo a copy of record lo).
    Rows outside every group are zero."""
    lib = capi.load()
    records = np.asarray(records)
    dtype = np.dtype(np.float32) if records.dtype == np.float32 else np.dtype(np.float64)
    records = np.ascontiguousarray(records, dtype=dtype).reshape(-1, REC_DOUBLES.get(model, REC_DOUBLES[1]))   # the library rejects model 2
    lin = np.ascontiguousarray(lin, dtype=dtype).reshape(-1, 13)
    if lin.shape[0] != records.shape[0]:
        raise ValueError("lin must hold one linearisation point per record")
    offs = None if group_offsets is None else np.ascontiguousarray(group_offsets, dtype=np.int64)
    n, uniform = _merge_layout(records.shape[0], offs, group, 0 if offs is None else offs.shape[0])
    if offs is not None and offs.shape[0] and offs[-1] > records.shape[0]:
        raise ValueError("group_offsets run past the record array")
    out = np.zeros_like(records)
    capi.check(lib.cpi_scan_records_host(model, 8 * dtype.itemsize, n, _ptr(offs), uniform, _ptr(records), _ptr(lin), _ptr(out)))
    return out


def scan(model, records, lin, group_offsets=None, group=None, out=None, stream=None, workspace=None):
    """Inclusive scan of consecutive records within groups on the device (``cpi_scan_records``): CUDA tensors as ``merge``; enqueues on
    ``stream`` (default: torch's current stream) and does not synchronise.  Layout and result as ``scan_host``; ``out`` (shaped like
    ``records``, default zeros) must not overlap ``records``, and only its rows inside a group are written.  ``workspace``: a CUDA tensor
    of at least ``cpi_scan_records_workspace`` bytes, allocated here when absent or too small; pass one to keep the call
    allocation-free."""
    import torch

    lib = capi.load()
    if not (records.is_cuda and lin.is_cuda):
        raise ValueError("scan() takes CUDA tensors; use scan_host() for host arrays")
    if records.dtype not in (torch.float64, torch.float32) or lin.dtype != records.dtype:
        raise ValueError("records and lin must both be float64 or both float32")
    dev = records.device
    for name, t in (("lin", lin), ("group_offsets", group_offsets), ("out", out), ("workspace", workspace)):
        if t is not None and t.device != dev:
            raise ValueError(f"{name} lives on {t.device}, records on {dev}: all tensors of one call must be on the same CUDA device")
    rd = REC_DOUBLES[1]
    n, uniform = _record_layout(records, lin, group_offsets, group)
    n_rec = records.numel() // rd
    if out is not None and (out.numel() < n_rec * rd or not out.is_contiguous() or out.dtype != records.dtype):
        raise ValueError("out must be a contiguous tensor of n_records * 290 elements in the records' dtype")
    nbytes = int(lib.cpi_scan_records_workspace(max(n, 0), n_rec))
    with _on(dev, stream):                                           # the zero fill of out before the scan that writes inside it
        records, lin = records.contiguous(), lin.contiguous()
        group_offsets = None if group_offsets is None else group_offsets.contiguous()
        if out is None:
            out = torch.zeros((n_rec, rd), dtype=records.dtype, device=dev)
        if workspace is None or workspace.numel() * workspace.element_size() < nbytes or not workspace.is_contiguous():
            workspace = torch.empty((nbytes + 7) // 8, dtype=torch.float64, device=dev)
        _launch(lib.cpi_scan_records, dev, stream, model, 64 if records.dtype == torch.float64 else 32, n, _tptr(group_offsets), uniform,
                _tptr(records), _tptr(lin), _tptr(out), _tptr(workspace))
    return out


# ------------------------------------------------------------------------------------------------------------------
# reference-shaped objects
# ------------------------------------------------------------------------------------------------------------------

class CpiBase:
    """cpi/CpiBase.h:40-145.  ``model`` is fixed by the subclass."""
    model = 0

    def __init__(self, sigma_w, sigma_wb, sigma_a, sigma_ab, imu_avg_=False):
        self._sigmas = np.array([sigma_w, sigma_wb, sigma_a, sigma_ab], dtype=np.float64)
        self.imu_avg = bool(imu_avg_)
        # Q_c, CpiBase.h:54-57
        self.Q_c = np.diag(np.repeat(self._sigmas ** 2, 3))
        self.b_w_lin = np.zeros(3); self.b_a_lin = np.zeros(3); self.q_k_lin = np.zeros(4); self.grav = np.zeros(3)
        self._steps = []        # (w0[3], a0[3], dt, w1[3], a1[3])
        self._result = None

    def setLinearizationPoints(self, b_w_lin_, b_a_lin_, q_k_lin_=None, grav_=None):
        self.b_w_lin = np.asarray(b_w_lin_, dtype=np.float64).reshape(3).copy()
        self.b_a_lin = np.asarray(b_a_lin_, dtype=np.float64).reshape(3).copy()
        self.q_k_lin = np.zeros(4) if q_k_lin_ is None else np.asarray(q_k_lin_, dtype=np.float64).reshape(4).copy()
        self.grav = np.zeros(3) if grav_ is None else np.asarray(grav_, dtype=np.float64).reshape(3).copy()

    def feed_IMU(self, t_0, t_1, w_m_0, a_m_0, w_m_1=None, a_m_1=None):
        z = np.zeros(3)
        self._steps.append((np.asarray(w_m_0, dtype=np.float64).reshape(3), np.asarray(a_m_0, dtype=np.float64).reshape(3),
                            float(t_1) - float(t_0),
                            z if w_m_1 is None else np.asarray(w_m_1, dtype=np.float64).reshape(3),
                            z if a_m_1 is None else np.asarray(a_m_1, dtype=np.float64).reshape(3)))
        self._result = None

    # ---- staging -> batch layout
    def _flags(self):
        f = FLAG_IMU_AVG if self.imu_avg else 0
        if self.model == 2 and not getattr(self, "state_transition_jacobians", True):
            f |= FLAG_ANALYTIC_JACOBIANS
        return f

    def _entries(self):
        n = len(self._steps)
        if not self.imu_avg:
            S = np.zeros((n, 7))
            for i, (w0, a0, dt, _, _) in enumerate(self._steps):
                S[i, 0:3], S[i, 3:6], S[i, 6] = w0, a0, dt
            return S
        # imu_avg: step i needs its own (w_m_1, a_m_1); lay every step out as  (w0,a0,dt) (w1,a1,dt=0)  -- the dt = 0
        # entry is a no-op step (CpiV1.h:72-74) whose only role is to be the "_1" reading of the step before it.
        S = np.zeros((2 * n + 1, 7))
        for i, (w0, a0, dt, w1, a1) in enumerate(self._steps):
            S[2 * i, 0:3], S[2 * i, 3:6], S[2 * i, 6] = w0, a0, dt
            S[2 * i + 1, 0:3], S[2 * i + 1, 3:6] = w1, a1
        if n:
            S[2 * n, 0:6] = S[2 * n - 1, 0:6]
        return S

    def _lin(self):
        return np.concatenate([self.b_w_lin, self.b_a_lin, self.q_k_lin, self.grav])

    def _adopt(self, rec):
        def m(name, shape):
            a, b = REC[name]
            return rec[a:b].reshape(shape, order="F").copy()
        self._result = dict(DT=float(rec[19]), alpha_tau=m("alpha", 3), beta_tau=m("beta", 3), q_k2tau=m("q", 4), R_k2tau=m("R", (3, 3)),
                            J_q=m("J_q", (3, 3)), J_a=m("J_a", (3, 3)), J_b=m("J_b", (3, 3)), H_a=m("H_a", (3, 3)), H_b=m("H_b", (3, 3)),
                            P_meas=m("P", (15, 15)))
        if self.model == 2:
            self._result.update(O_a=m("O_a", (3, 3)), O_b=m("O_b", (3, 3)))
        self._record = rec.copy()

    def finalize(self):
        """Run the kernel for this one window and populate the public result fields."""
        flush([self])
        return self

    def record(self):
        """The raw result record (include/cpi_b200.h layout) -- what the factor constructors consume."""
        if self._result is None:
            raise RuntimeError("call finalize() / flush() after the last feed_IMU before reading results")
        return self._record

    def __getattr__(self, name):
        if name in _RESULT_FIELDS:
            res = self.__dict__.get("_result")
            if res is None:
                raise RuntimeError(f"{name} is not available yet: call finalize() / flush() after the last feed_IMU "
                                   f"(results are produced by one batched GPU launch, not per sample)")
            if name in res:
                return res[name]
        raise AttributeError(name)


class CpiV1(CpiBase):
    """Model 1, piecewise-constant measurement (cpi/CpiV1.h:41)."""
    model = 1

    def mergeWith(self, later):
        """Extend this finalised window by the finalised window that follows it (GTSAM's mergeWith), in place: the fields become those
        of the combined interval, at this object's linearisation point (``later`` is moved to it to first order).  The staged steps
        are concatenated too, so a later ``finalize()`` re-preintegrates the combined window from its samples."""
        if not isinstance(later, CpiV1):
            raise TypeError("mergeWith takes a CpiV1")
        rec = merge_host(1, np.stack([self.record(), later.record()]), np.stack([self._lin(), later._lin()]), group=2)
        self._steps = self._steps + later._steps
        self._adopt(rec[0])
        return self


class CpiV2(CpiBase):
    """Model 2, piecewise-constant local acceleration (cpi/CpiV2.h:41)."""
    model = 2

    def __init__(self, sigma_w, sigma_wb, sigma_a, sigma_ab, imu_avg_=False):
        super().__init__(sigma_w, sigma_wb, sigma_a, sigma_ab, imu_avg_)
        self.state_transition_jacobians = True     # CpiV2.h:58


def flush(cpis):
    """Preintegrate many staged objects at once.  Objects that share (model, flags, sigmas) go out in ONE launch."""
    groups = {}
    for c in cpis:
        groups.setdefault((c.model, c._flags(), tuple(c._sigmas)), []).append(c)
    for (model, flags, sig), members in groups.items():
        ent = [c._entries() for c in members]
        offsets = np.zeros(len(members) + 1, dtype=np.int64)
        offsets[1:] = np.cumsum([e.shape[0] for e in ent])
        S = np.concatenate(ent) if ent else np.zeros((0, 7))
        L = np.stack([c._lin() for c in members])
        rec = preintegrate_host(model, S, L, np.array(sig), flags, offsets=offsets)
        for c, r in zip(members, rec):
            c._adopt(r)
