"""Host-side mirror of the GTSAM-side plug-ins of the hot path, on top of the C ABI:

    JPLNavState                      gtsam/JPLNavState.h:59-151   (value layout q, bg, v, ba, p; retract)
    ImuFactorCPIv1 / ImuFactorCPIv2  gtsam/ImuFactorCPIv1.h:55, gtsam/ImuFactorCPIv2.h:55   (ctor argument order kept)
        .evaluateError(state_i, state_j, H1=False, H2=False)      gtsam/ImuFactorCPIv1.cpp:37, ImuFactorCPIv2.cpp:38

and the batch entry points (``factor_eval``, ``predict_state``, ``retract``, ``propagate``, ``update``).  The residual and Jacobians are UNWHITENED,
exactly what evaluateError returns; GTSAM's Gaussian::Covariance(P_meas) whitening is outside the reference tree.
All arithmetic happens in libcpi_b200.so on the GPU.

Streams (DESIGN.md section 5x): a device binding's call with ``stream=S`` is the same call with ``stream=None`` made inside
``torch.cuda.stream(S)``: its allocations, copies, fills, sorts, host reads and launches all go on S, and its temporaries return to
S's pool.  The caller orders the inputs before the call (``S.wait_stream(C)`` for inputs made on stream C), orders the consumers of
the results after it (``C.wait_stream(S)``, or ``record_stream``), and keeps to the same rule for any ``out=`` or ``workspace=`` it
passes.
"""
from __future__ import annotations

import contextlib
import ctypes
import math

import numpy as np

from . import capi
from .capi import FLAG_IMU_AVG, LOSS_CAUCHY, LOSS_GAUSSIAN, REC, REC_DOUBLES


def _ptr(a):
    return None if a is None else ctypes.c_void_p(a.ctypes.data)


class _TensorPtr(ctypes.c_void_p):
    """A tensor's data pointer that keeps the tensor alive: an argument written _tptr(x.contiguous()) holds its copy until the call
    it is passed to returns, so the copy cannot go back to the pool, and be handed to the next argument's copy, before the launch."""


def _tptr(t):
    if t is None:
        return None
    p = _TensorPtr(t.data_ptr())
    p.tensor = t
    return p


def _stream(dev, stream):
    """The handle of stream, or of dev's current stream when it is None."""
    import torch

    return ctypes.c_void_p((stream if stream is not None else torch.cuda.current_stream(dev)).cuda_stream)


@contextlib.contextmanager
def _on(dev, stream):
    """dev current and stream (None: dev's current stream) torch's current stream.  A binding runs its whole body under it, from its
    first allocation to its last launch or host read, so that a call with stream=S is the call with stream=None made inside
    torch.cuda.stream(S): its copies, fills, sorts and launches go on S, and its temporaries return to S's pool.  A dev that is not a
    CUDA device enters nothing, so that the binding's own checks reject its tensors."""
    import torch

    if torch.device(dev if not isinstance(dev, int) else f"cuda:{dev}").type != "cuda":
        yield
        return
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        yield


def _launch(fn, dev, stream, *args):
    """fn(*args, stream handle) with dev current: the library launches on the current device, so a call on another device's tensors
    makes theirs current for the call.  stream: a stream of dev, or None for dev's current stream."""
    import torch

    with torch.cuda.device(dev):
        capi.check(fn(*args, _stream(dev, stream)))


def _staged(run, stream, *arrays):
    """run(*arrays) on device tensors; numpy arrays are staged to the current device as float64 and run's results (a tensor or a
    tuple of them) copied back to numpy, the copies on ``stream`` (default: the current stream) with the launch."""
    import torch

    if not isinstance(arrays[0], np.ndarray):
        return run(*arrays)
    with _on(torch.cuda.current_device(), stream):
        out = run(*(torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda() for a in arrays))
        return tuple(t.cpu().numpy() for t in out) if isinstance(out, tuple) else out.cpu().numpy()


def factor_eval_host(model, states, records, lin, idx_i=None, idx_j=None, want_H1=True, want_H2=True):
    """HOST numpy in/out through ``cpi_imu_factor_eval_batch_host``.  Returns (e[n,15], H1[n,225]|None, H2[n,225]|None);
    H blocks are column-major 15x15 (reshape(15,15,order='F'))."""
    lib = capi.load()
    states = np.ascontiguousarray(states, dtype=np.float64).reshape(-1, 16)
    records = np.ascontiguousarray(records, dtype=np.float64).reshape(-1, REC_DOUBLES[model])
    lin = np.ascontiguousarray(lin, dtype=np.float64).reshape(-1, 13)
    n = records.shape[0]
    if lin.shape[0] != n:
        raise ValueError("one linearisation point per factor required")
    if (idx_i is None) != (idx_j is None):
        raise ValueError("idx_i and idx_j must both be given or both be None")
    if idx_i is not None:
        idx_i = np.ascontiguousarray(idx_i, dtype=np.int64); idx_j = np.ascontiguousarray(idx_j, dtype=np.int64)
        if idx_i.shape[0] != n or idx_j.shape[0] != n:
            raise ValueError("index arrays must have one entry per factor")
        if n and (min(idx_i.min(), idx_j.min()) < 0 or max(idx_i.max(), idx_j.max()) >= states.shape[0]):
            raise IndexError("state index out of range")
    elif states.shape[0] < n + 1:
        raise ValueError("chain indexing needs n_factors + 1 states")
    e = np.empty((n, 15)); H1 = np.empty((n, 225)) if want_H1 else None; H2 = np.empty((n, 225)) if want_H2 else None
    capi.check(lib.cpi_imu_factor_eval_batch_host(model, n, states.shape[0], _ptr(states), _ptr(idx_i), _ptr(idx_j), _ptr(records), _ptr(lin),
                                                  _ptr(e), _ptr(H1), _ptr(H2)))
    return e, H1, H2


def _factor_indices(n, dev, states, lin, idx_i, idx_j):
    """The checks factor_eval and factor_cost share: states, lin, idx_i and idx_j (both or neither; int64, one entry per factor of
    the n) CUDA tensors on dev.  Returns (idx_i, idx_j) contiguous."""
    import torch

    for name, t in (("states", states), ("lin", lin), ("idx_i", idx_i), ("idx_j", idx_j)):
        if t is not None and (not t.is_cuda or t.device != dev):
            raise ValueError(f"{name} must be a CUDA tensor on {dev}")
    if (idx_i is None) != (idx_j is None):
        raise ValueError("idx_i and idx_j must both be given or both be None")
    if idx_i is None:
        return None, None
    if idx_i.dtype != torch.int64 or idx_j.dtype != torch.int64 or idx_i.numel() != n or idx_j.numel() != n:
        raise ValueError("idx_i / idx_j must be int64 tensors with one entry per factor")
    return idx_i.contiguous(), idx_j.contiguous()


def factor_eval(model, states, records, lin, idx_i=None, idx_j=None, want_H1=True, want_H2=True, out=None, stream=None):
    """DEVICE torch tensors (float64 / int64, contiguous).  Enqueues on ``stream`` (default: torch's current stream)."""
    import torch

    lib = capi.load()
    n = records.numel() // REC_DOUBLES[model]
    dev = records.device
    with _on(dev, stream):
        idx_i, idx_j = _factor_indices(n, dev, states, lin, idx_i, idx_j)
        if out is None:
            e = torch.empty((n, 15), dtype=torch.float64, device=dev)
            H1 = torch.empty((n, 225), dtype=torch.float64, device=dev) if want_H1 else None
            H2 = torch.empty((n, 225), dtype=torch.float64, device=dev) if want_H2 else None
        else:
            e, H1, H2 = out
        _launch(lib.cpi_imu_factor_eval_batch, dev, stream, model, n, _tptr(states.contiguous()), _tptr(idx_i), _tptr(idx_j),
                _tptr(records.contiguous()), _tptr(lin.contiguous()), _tptr(e), _tptr(H1), _tptr(H2))
    return e, H1, H2


def factor_hessian(model, records, e, H1, H2, stream=None):
    """Information-form linearisation (cpi_imu_factor_hessian_batch): returns (G11, G12, G22 [n,225 col-major], g1, g2 [n,15], f [n]).
    Device tensors in/out, or numpy (staged through torch).  Parity vs GTSAM unpinned (GTSAM is not in the reference tree)."""
    return _from_residuals(capi.load().cpi_imu_factor_hessian_batch, model, records, e, H1, H2, stream, (225,), (225,), (225,), (15,), (15,), ())


def factor_whiten(model, records, e, H1, H2, stream=None):
    """Explicitly whitened form (cpi_imu_factor_whiten_batch): A1 = R_w H1, A2 = R_w H2 [n,225 col-major], b = -R_w e [n,15], with
    R_w the upper Cholesky factor of P_meas^-1 (GTSAM's Gaussian::Covariance).  Device tensors in/out, or numpy.  Parity unpinned."""
    return _from_residuals(capi.load().cpi_imu_factor_whiten_batch, model, records, e, H1, H2, stream, (225,), (225,), (15,))


def _from_residuals(fn, model, records, e, H1, H2, stream, *shapes):
    """fn(model, n, records, e, H1, H2, outputs...) of factor_hessian / factor_whiten into new outputs [n, *shape] per shape."""
    import torch

    def run(records, e, H1, H2):
        dev = records.device
        _check_f64(dev, records=records, e=e, H1=H1, H2=H2)
        n = records.numel() // REC_DOUBLES[model]
        with _on(dev, stream):
            out = tuple(torch.empty((n, *shape), dtype=torch.float64, device=dev) for shape in shapes)
            _launch(fn, dev, stream, model, n, _tptr(records.contiguous()), _tptr(e.contiguous()), _tptr(H1.contiguous()),
                    _tptr(H2.contiguous()), *(_tptr(t) for t in out))
        return out
    return _staged(run, stream, records, e, H1, H2)


def chain_assemble(G11, G12, G22, g1, g2, lam=0.0, prior_info0=None, prior_rhs0=None, stream=None, diagonal_damping=False):
    """Block-tridiagonal normal equations of the chain x_0 .. x_n from the per-factor information blocks: chains_assemble on one
    chain of n + 1 states (the kernel cpi_imu_chain_assemble launches).  Device tensors.  Damping: lam * I, or with diagonal_damping
    lam * clamp(diag, 1e-6, 1e32) (GTSAM's LevenbergMarquardtParams::diagonalDamping).  Returns (D [n+1,225], E [n,225], rhs [n+1,15])."""
    return chains_assemble(G11, G12, G22, g1, g2, G11.shape[0] + 1, lam, prior_info0, prior_rhs0, diagonal_damping, n_chains=1, stream=stream)


def chain_solve(D, E, rhs, stream=None, workspace=None):
    """x = A^-1 rhs for the SPD block-tridiagonal A = tridiag(E^T, D, E) by block cyclic reduction on the device (cpi_imu_chain_solve):
    chains_solve with every state in one chain, so the NaN of a non-SPD part spreads into the rest through its zero couplings."""
    import torch

    lib = capi.load()
    dev = D.device
    _check_f64(dev, D=D, E=E, rhs=rhs, workspace=workspace)
    n = D.shape[0]
    nbytes = int(lib.cpi_imu_chain_solve_workspace(n))
    with _on(dev, stream):
        x = torch.empty((n, 15), dtype=torch.float64, device=dev)
        if workspace is None or workspace.numel() * 8 < nbytes:
            workspace = torch.empty((nbytes + 7) // 8, dtype=torch.float64, device=dev)
        _launch(lib.cpi_imu_chain_solve, dev, stream, n, _tptr(D), _tptr(E), _tptr(rhs), _tptr(x), _tptr(workspace))
    return x


def _check_f64(dev, **tensors):
    import torch

    for name, t in tensors.items():
        if t is None:
            continue
        if not t.is_cuda or t.device != dev:
            raise ValueError(f"{name} must be a CUDA tensor on {dev}")
        if t.dtype != torch.float64:
            raise ValueError(f"{name} must be float64")


def _chain_layout(chain_offsets, dev, n_factors=None, n_states=None, n_chains=None):
    """(n_chains, offsets tensor or None, states per chain) of a chain layout: a device int64 tensor [n_chains+1] of state offsets
    (offsets[0] = 0, every chain non-empty), or an int, the states per chain, with the chain count taken from n_chains, n_states or
    n_factors (each chain of S states has S - 1 factors)."""
    import torch

    if isinstance(chain_offsets, torch.Tensor):
        if not chain_offsets.is_cuda or chain_offsets.device != dev or chain_offsets.dtype != torch.int64 or chain_offsets.dim() != 1:
            raise ValueError(f"chain_offsets must be a 1-d int64 CUDA tensor on {dev}")
        if chain_offsets.numel() < 1:
            raise ValueError("chain_offsets needs n_chains + 1 entries")
        return chain_offsets.numel() - 1, chain_offsets.contiguous(), 0
    S = int(chain_offsets)
    if S < 1:
        raise ValueError("a chain holds at least one state")
    if n_chains is None:
        if n_states is not None:
            n_chains = n_states // S
        elif S > 1:
            n_chains = n_factors // (S - 1)
        else:
            raise ValueError("single-state chains hold no factor: pass n_chains")
    if (n_states is not None and n_states != n_chains * S) or (n_factors is not None and n_factors != n_chains * (S - 1)):
        raise ValueError(f"{n_chains} chains of {S} states do not match the given states / factors")
    return int(n_chains), None, S


def _chain_factor_states(C, offs, S, nf, dev):
    """(idx_i, idx_j) of the nf factors of a chain layout (chain c's factors stored back to back from index offsets[c] - c; factor
    k links states idx_i[k] and idx_i[k] + 1), or (None, None) for one chain: the kernels' own chain indexing."""
    import torch

    if C <= 1:
        return None, None
    ar = torch.arange(nf, dtype=torch.int64, device=dev)
    if offs is not None:
        chain_of = torch.repeat_interleave(torch.arange(C, dtype=torch.int64, device=dev), offs[1:] - offs[:-1] - 1, output_size=nf)
    else:
        chain_of = ar // (S - 1) if S > 1 else ar
    idx_i = ar + chain_of
    return idx_i, idx_i + 1


def chains_assemble(G11, G12, G22, g1, g2, chain_offsets, lam=0.0, prior_info=None, prior_rhs=None, diagonal_damping=False, n_chains=None,
                    stream=None):
    """Block-tridiagonal normal equations of many independent chains at once (cpi_imu_chains_assemble).  chain_offsets: device int64
    [n_chains+1] state offsets, or an int (states per chain; n_chains is then taken from the factor count unless given).  Chain c's
    factors are stored back to back from index offsets[c] - c.  prior_info [n_chains,225] / prior_rhs [n_chains,15] (each may be None) go
    on every chain's first state; damping as chain_assemble.  E is exactly 0 at chain boundaries, so chain_solve(D, E, rhs) solves every
    chain at once -- provided every chain is SPD (a NaN pivot spreads into the neighbouring chains).
    Returns (D [N,225], E [N-1,225], rhs [N,15]) for the N = n_factors + n_chains states."""
    return _assemble(G11, G12, G22, g1, g2, chain_offsets, lam, prior_info, prior_rhs, diagonal_damping, n_chains, stream, per_chain=False)


def _assemble(G11, G12, G22, g1, g2, chain_offsets, lam, prior_info, prior_rhs, diagonal_damping, n_chains, stream, per_chain):
    """chains_assemble (lam a scalar), or with per_chain chains_assemble_lm (lam a device float64 [n_chains]; damp returned too)."""
    import torch

    dev = G11.device
    _check_f64(dev, G11=G11, G12=G12, G22=G22, g1=g1, g2=g2, prior_info=prior_info, prior_rhs=prior_rhs, lam=lam if per_chain else None)
    nf = G11.numel() // 225
    with _on(dev, stream):
        C, offs, S = _chain_layout(chain_offsets, dev, n_factors=nf, n_chains=n_chains)
        if any(t.numel() != k * nf for t, k in ((G11, 225), (G12, 225), (G22, 225), (g1, 15), (g2, 15))):
            raise ValueError("G11 / G12 / G22 need 225 doubles and g1 / g2 15 per factor")
        if per_chain and (lam is None or lam.numel() != C):
            raise ValueError("lam needs one float64 CUDA entry per chain")
        if (prior_info is not None and prior_info.numel() != 225 * C) or (prior_rhs is not None and prior_rhs.numel() != 15 * C):
            raise ValueError("prior_info needs 225 doubles and prior_rhs 15 per chain")
        N = nf + C
        out = (torch.empty((N, 225), dtype=torch.float64, device=dev), torch.empty((max(N - 1, 1), 225), dtype=torch.float64, device=dev),
               torch.empty((N, 15), dtype=torch.float64, device=dev)) + ((torch.empty((N, 15), dtype=torch.float64, device=dev),) if per_chain else ())
        lib = capi.load()
        c = lambda t: None if t is None else t.contiguous()
        _launch(lib.cpi_imu_chains_assemble_lm if per_chain else lib.cpi_imu_chains_assemble, dev, stream, C, _tptr(offs), S, _tptr(c(G11)),
                _tptr(c(G12)), _tptr(c(G22)), _tptr(c(g1)), _tptr(c(g2)), _tptr(c(lam)) if per_chain else float(lam), int(bool(diagonal_damping)),
                _tptr(c(prior_info)), _tptr(c(prior_rhs)), *(_tptr(t) for t in out))
    return (out[0], out[1][:N - 1]) + out[2:]


def _loss_flags(code, k, rhs, f, measurement):
    """The value checks of state_prior_loss as 0-d bool tensors, for the entry's one host read: a code outside {0, 1, 2}, a robust
    prior whose k does not satisfy 0 < k^2 < inf, and (measurement) a robust prior with a nonzero rhs or f."""
    import torch

    robust = code != LOSS_GAUSSIAN
    k2 = k * k
    flags = [((code < LOSS_GAUSSIAN) | (code > LOSS_CAUCHY)).any(), (robust & ~((k > 0) & (k2 > 0) & torch.isfinite(k2))).any()]
    if measurement:
        nz = torch.zeros_like(robust)
        if rhs is not None:
            nz = nz | (rhs.reshape(code.numel(), 15) != 0).any(dim=1)
        if f is not None:
            nz = nz | (f.reshape(code.numel()) != 0)
        flags.append((robust & nz).any())
    return flags


def _state_priors(state_priors, N, dev, offs=None, S=0, loss=None, measurement=True):
    """Validated state priors (state_idx [M] int64, info [M,225], rhs [M,15] | None, f [M] | None, lin [M,16]) on N states: returns
    (idx, info, rhs (zeros if None), f or None, lin, single, loss) with single whether a chain of one state carries a prior, or None
    for state_priors None or M = 0.  loss: state_prior_loss, (code [M] int32, k [M] float64) or None, returned as given.  Checks
    shapes and dtypes, then 0 <= state_idx < N and the loss values (the one host read), then the device.  measurement: a robust prior
    must have rhs and f None or zero (chain_marginalize takes them moved, and skips that check)."""
    import torch

    if state_priors is None:
        if loss is not None:
            raise ValueError("state_prior_loss needs state_priors")
        return None
    if not isinstance(state_priors, (tuple, list)) or len(state_priors) != 5:
        raise ValueError("state_priors is (state_idx [M], info [M,225], rhs [M,15] or None, f [M] or None, lin [M,16])")
    idx, info, rhs, f, lin = state_priors
    if not isinstance(idx, torch.Tensor) or idx.dtype != torch.int64 or idx.dim() != 1:
        raise ValueError("state_priors: state_idx must be a 1-d int64 tensor")
    M = idx.numel()
    for name, t, k in (("info", info, 225), ("rhs", rhs, 15), ("f", f, 1), ("lin", lin, 16)):
        if t is None and name in ("rhs", "f"):
            continue
        if not isinstance(t, torch.Tensor) or t.dtype != torch.float64:
            raise ValueError(f"state_priors: {name} must be a float64 tensor")
        if t.numel() != k * M or t.dim() < 1 or t.shape[0] != M:
            raise ValueError(f"state_priors: {name} needs {k} doubles for each of the {M} priors")
    if loss is not None:
        if not isinstance(loss, (tuple, list)) or len(loss) != 2:
            raise ValueError("state_prior_loss is (loss [M] int32, loss_k [M] float64)")
        code, lk = loss
        if not isinstance(code, torch.Tensor) or code.dtype != torch.int32 or code.dim() != 1 or code.numel() != M:
            raise ValueError(f"state_prior_loss: loss must be a 1-d int32 tensor with one code for each of the {M} priors")
        if not isinstance(lk, torch.Tensor) or lk.dtype != torch.float64 or lk.dim() != 1 or lk.numel() != M:
            raise ValueError(f"state_prior_loss: loss_k must be a 1-d float64 tensor with one threshold for each of the {M} priors")
        if code.device != idx.device or lk.device != idx.device:
            raise ValueError("state_prior_loss: loss and loss_k must be on the device of state_idx")
    if M:
        flags = [((idx < 0) | (idx >= N)).any()]
        if offs is not None and idx.device == offs.device:         # a chain of one state carrying a prior: the chain prior is its target
            c = (torch.searchsorted(offs, idx.clamp(0, max(N - 1, 0)), right=True) - 1).clamp(0, offs.numel() - 2)
            flags.append(((offs[c + 1] - offs[c]) == 1).any())
        else:
            flags.append(torch.zeros((), dtype=torch.bool, device=idx.device))
        if loss is not None:
            flags += _loss_flags(code, lk, rhs, f, measurement)
        flags = torch.stack(flags).tolist()
        if flags[0]:
            raise IndexError(f"state_priors: state_idx out of range [0, {N})")
        if loss is not None:
            if flags[2]:
                raise ValueError("state_prior_loss: loss codes are 0 (Gaussian), 1 (Huber) and 2 (Cauchy)")
            if flags[3]:
                raise ValueError("state_prior_loss: a Huber or Cauchy prior needs a threshold k with 0 < k^2 < inf")
            if measurement and flags[4]:
                raise ValueError("state_prior_loss: a Huber or Cauchy prior must be a measurement prior (rhs and f None or zero)")
    if not idx.is_cuda or idx.device != dev:
        raise ValueError(f"state_priors: state_idx must be a CUDA tensor on {dev}")
    _check_f64(dev, state_prior_info=info, state_prior_rhs=rhs, state_prior_f=f, state_prior_lin=lin)
    if M == 0:
        return None
    single = bool(flags[1]) if offs is not None else S == 1
    rhs = torch.zeros((M, 15), dtype=torch.float64, device=dev) if rhs is None else rhs
    return (idx, info.reshape(M, 225), rhs.reshape(M, 15), None if f is None else f.reshape(M), lin.reshape(M, 16), single,
            None if loss is None else (code.contiguous(), lk.contiguous()))


def _measurements(measurements, N, dev, offs=None, S=0, loss=None):
    """Validated measurements (state_idx [M] int64, kind [M] int32 capi.MEAS_*, z [M,3], sqrt_info [M,9], aux [M,3]; DESIGN.md
    section 3l) on N states: returns (idx, kind, z, sqrt_info, aux, single, loss) as _state_priors does, or None for measurements None
    or M = 0.  loss: measurement_loss, (code [M] int32, k [M] float64) with the semantics of state_prior_loss, or None.  Checks shapes
    and dtypes, then 0 <= state_idx < N, the kind codes and the loss values (one host read), then the device."""
    import torch

    from .capi import MEAS_DIRECTION, MEAS_POSITION

    if measurements is None:
        if loss is not None:
            raise ValueError("measurement_loss needs measurements")
        return None
    if not isinstance(measurements, (tuple, list)) or len(measurements) != 5:
        raise ValueError("measurements is (state_idx [M] int64, kind [M] int32, z [M,3], sqrt_info [M,9], aux [M,3])")
    idx, kind, z, si, aux = measurements
    if not isinstance(idx, torch.Tensor) or idx.dtype != torch.int64 or idx.dim() != 1:
        raise ValueError("measurements: state_idx must be a 1-d int64 tensor")
    M = idx.numel()
    if not isinstance(kind, torch.Tensor) or kind.dtype != torch.int32 or kind.dim() != 1 or kind.numel() != M:
        raise ValueError(f"measurements: kind must be a 1-d int32 tensor with one code for each of the {M} measurements")
    for name, t, k in (("z", z, 3), ("sqrt_info", si, 9), ("aux", aux, 3)):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.float64:
            raise ValueError(f"measurements: {name} must be a float64 tensor")
        if t.numel() != k * M or t.dim() < 1 or t.shape[0] != M:
            raise ValueError(f"measurements: {name} needs {k} doubles for each of the {M} measurements")
    if loss is not None:
        if not isinstance(loss, (tuple, list)) or len(loss) != 2:
            raise ValueError("measurement_loss is (loss [M] int32, loss_k [M] float64)")
        code, lk = loss
        if not isinstance(code, torch.Tensor) or code.dtype != torch.int32 or code.dim() != 1 or code.numel() != M:
            raise ValueError(f"measurement_loss: loss must be a 1-d int32 tensor with one code for each of the {M} measurements")
        if not isinstance(lk, torch.Tensor) or lk.dtype != torch.float64 or lk.dim() != 1 or lk.numel() != M:
            raise ValueError(f"measurement_loss: loss_k must be a 1-d float64 tensor with one threshold for each of the {M} measurements")
        if code.device != idx.device or lk.device != idx.device:
            raise ValueError("measurement_loss: loss and loss_k must be on the device of state_idx")
    if kind.device != idx.device:
        raise ValueError("measurements: kind must be on the device of state_idx")
    single = S == 1
    if M:
        flags = [((idx < 0) | (idx >= N)).any(), ((kind < MEAS_POSITION) | (kind > MEAS_DIRECTION)).any()]
        if offs is not None and idx.device == offs.device:         # a chain of one state carrying a measurement
            c = (torch.searchsorted(offs, idx.clamp(0, max(N - 1, 0)), right=True) - 1).clamp(0, offs.numel() - 2)
            flags.append(((offs[c + 1] - offs[c]) == 1).any())
        else:
            flags.append(torch.zeros((), dtype=torch.bool, device=idx.device))
        if loss is not None:
            flags += _loss_flags(code, lk, None, None, False)
        flags = torch.stack(flags).tolist()
        if flags[0]:
            raise IndexError(f"measurements: state_idx out of range [0, {N})")
        if flags[1]:
            raise ValueError("measurements: kind codes are 1 (position), 2 (body-frame velocity) and 3 (direction)")
        if loss is not None:
            if flags[3]:
                raise ValueError("measurement_loss: loss codes are 0 (Gaussian), 1 (Huber) and 2 (Cauchy)")
            if flags[4]:
                raise ValueError("measurement_loss: a Huber or Cauchy measurement needs a threshold k with 0 < k^2 < inf")
        if offs is not None:
            single = bool(flags[2])
    if not idx.is_cuda or idx.device != dev:
        raise ValueError(f"measurements: state_idx must be a CUDA tensor on {dev}")
    _check_f64(dev, z=z, sqrt_info=si, aux=aux)
    if M == 0:
        return None
    return (idx, kind.contiguous(), z.reshape(M, 3), si.reshape(M, 9), aux.reshape(M, 3), single,
            None if loss is None else (code.contiguous(), lk.contiguous()))


def _state_prior_csr(key, N):
    """(order, sp_offsets [N+1]): the stable sort of the priors by key and the CSR of the keys below N (the priors of state k are
    order[sp_offsets[k] .. sp_offsets[k+1]-1])."""
    import torch

    key_s, order = torch.sort(key, stable=True)
    return order, torch.searchsorted(key_s, torch.arange(N + 1, dtype=torch.int64, device=key.device))


class _StatePriors:
    """The state priors of one call (the tuple of _state_priors) in the order the fold adds them: sorted stably by key (default:
    their state), with the CSR of the keys below N, on the chain layout (C, offs, S), and the buffers their moved and reweighted
    copies go to.  Its methods launch on the stream handle sp, with the priors' device current."""

    def __init__(self, sp, N, layout, key=None):
        import torch

        idx, info, rhs, f, lin, single, loss = sp
        order = self._sorted(idx, N, layout, key, single, loss)
        self.info, self.rhs, self.lin = info[order].contiguous(), rhs[order].contiguous(), lin[order].contiguous()
        self.f = None if f is None else f[order].contiguous()
        f64 = dict(dtype=torch.float64, device=idx.device)
        self.x, self.r, self.fm = torch.empty((self.M, 16), **f64), torch.empty((self.M, 15), **f64), torch.empty(self.M, **f64)
        self._weighted()

    def _sorted(self, idx, N, layout, key, single, loss):
        """What the fold reads of every source: the stable sort by key (default: the state) and its CSR, the layout, the count, the
        single-state flag and the loss in that order.  Returns the order; sets idx sorted."""
        order, self.sp_off = _state_prior_csr(idx if key is None else key, N)
        self.C, self.offs, self.S = layout
        self.M, self.single, self.idx = idx.numel(), single, idx[order]
        self.loss = None if loss is None else (loss[0][order].contiguous(), loss[1][order].contiguous())
        return order

    def _weighted(self):
        """The info the fold reads: self.info, or a buffer for the weighted info under a loss."""
        import torch

        self.iw = self.info if self.loss is None else torch.empty((self.M, 225), dtype=torch.float64, device=self.info.device)

    def fold(self, lib, sp, rhs, f, G11=None, G22=None, g1=None, g2=None, f_out=None, pi=None, pr=None, pf=None):
        """Reweight the priors (info, rhs, f) in place under their loss (s = f) and fold them into the targets; rhs None: f alone."""
        p = _tptr
        info, iw = (None, None) if rhs is None else (self.info, self.iw)
        if self.loss is not None:
            capi.check(lib.cpi_imu_state_priors_robust(self.M, p(self.loss[0]), p(self.loss[1]), p(info), p(rhs), p(f), p(iw), p(rhs), p(f), sp))
        capi.check(lib.cpi_imu_state_priors_fold(self.C, p(self.offs), self.S, p(self.sp_off), p(iw), p(rhs), p(f), p(G11), p(G22), p(g1),
                                                 p(g2), p(f_out), p(pi), p(pr), p(pf), sp))

    def at(self, lib, sp, X, cost_only=False, **targets):
        """Move the priors to the states X [N,16] (prior_at), reweight them there and fold them into the targets; cost_only: their
        cost alone."""
        import torch

        p = _tptr
        torch.index_select(X, 0, self.idx, out=self.x)
        capi.check(lib.cpi_imu_prior_at(self.M, p(self.info), p(self.rhs), p(self.f), p(self.lin), p(self.x), p(self.r), p(self.fm), sp))
        self.fold(lib, sp, None if cost_only else self.r, self.fm, **targets)


class _Measurements(_StatePriors):
    """The measurements of one call (the tuple of _measurements) sorted stably by state, with their CSR, on the chain layout: the
    state priors' fold, with the blocks linearised by cpi_imu_measurements_linearize at every call of `at` (DESIGN.md section 3l)."""

    def __init__(self, ms, N, layout):
        import torch

        idx, kind, z, si, aux, single, loss = ms
        order = self._sorted(idx, N, layout, None, single, loss)
        self.idx, self.kind = self.idx.contiguous(), kind[order].contiguous()
        self.z, self.si, self.aux = z[order].contiguous(), si[order].contiguous(), aux[order].contiguous()
        M, f64 = self.M, dict(dtype=torch.float64, device=idx.device)
        self.info, self.r, self.fm = torch.empty((M, 225), **f64), torch.empty((M, 15), **f64), torch.empty(M, **f64)
        self._weighted()

    def at(self, lib, sp, X, cost_only=False, **targets):
        """Linearise the measurements at the states X [N,16] (the f-only pass for cost_only), reweight and fold them as state priors."""
        p = _tptr
        info, r = (None, None) if cost_only else (self.info, self.r)
        capi.check(lib.cpi_imu_measurements_linearize(self.M, p(self.kind), p(self.idx), p(X), p(self.z), p(self.si), p(self.aux), p(info),
                                                      p(r), p(self.fm), sp))
        self.fold(lib, sp, r, self.fm, **targets)


def _folds(sp, ms, N, layout):
    """The fold sources of one call: the state priors, then the measurements (each None or validated); an empty list for neither.
    Folded one after the other, the measurements of a state are added after its priors."""
    return ([] if sp is None else [_StatePriors(sp, N, layout)]) + ([] if ms is None else [_Measurements(ms, N, layout)])


def measurements_linearize(states, measurements, stream=None):
    """The measurements (state_idx [M] int64, kind [M] int32 capi.MEAS_*, z [M,3], sqrt_info [M,9], aux [M,3]) linearised at the
    states [N,16] (cpi_imu_measurements_linearize, kernel K12; DESIGN.md section 3l) into moved prior blocks: info = A^T A [M,225]
    (exactly symmetric), rhs' = -A^T b [M,15], f' = b^T b [M].  Validated like state_priors (one host read).  Returns (info, rhs, f,
    state_priors) with state_priors = (state_idx, info, rhs, f, states[state_idx]): what chain_marginalize takes, as given at the
    blocks' linearisation point, to marginalise a lag window's measurements on eliminated states."""
    import torch

    if not isinstance(states, torch.Tensor):
        raise ValueError("states must be a tensor")
    if measurements is None:
        raise ValueError("measurements_linearize needs measurements")
    dev = states.device
    N = states.numel() // 16
    if states.numel() != 16 * N:
        raise ValueError(f"states must hold 16 doubles per state (got {states.numel()} doubles)")
    idx = measurements[0]
    f64 = dict(dtype=torch.float64, device=dev)
    with _on(dev, stream):                                           # the check's host read, buffers, copies and the launch
        ms = _measurements(measurements, N, dev)
        _check_f64(dev, states=states)
        M = idx.numel()
        info, rhs, f =torch.empty((M, 225), **f64), torch.empty((M, 15), **f64), torch.empty(M, **f64)
        X = states.reshape(N, 16).contiguous()
        if ms is not None:
            kind, z, si, aux = (t.contiguous() for t in ms[1:5])
            _launch(capi.load().cpi_imu_measurements_linearize, dev, stream, M, _tptr(kind), _tptr(idx.contiguous()), _tptr(X), _tptr(z),
                    _tptr(si), _tptr(aux), _tptr(info), _tptr(rhs), _tptr(f))
        lin = X.index_select(0, idx)
    return info, rhs, f, (idx, info, rhs, f, lin)


def state_priors_fold(chain_offsets, sp_offsets, sp_info, sp_rhs, sp_f, G11=None, G22=None, g1=None, g2=None, f=None, prior_info=None,
                      prior_rhs=None, prior_f=None, n_chains=None, stream=None):
    """Add already-moved state priors IN PLACE into the factor blocks and chain priors (cpi_imu_state_priors_fold): a prior on state k
    of chain c goes to G11 / g1 / f of factor k - c, on a chain's last state to G22 / g2 / f of factor k - 1 - c, on a chain's only state
    to the chain prior.  sp_offsets: device int64 [N+1] CSR over the states (priors sorted by state, added in that order); sp_info
    [M,225] / sp_rhs [M,15]: both or None (None: the f-only fold of sp_f [M]); a target that is None receives nothing.  Chain layout as
    chains_assemble (the state count N is sp_offsets' length - 1)."""
    import torch

    dev = sp_offsets.device
    if not sp_offsets.is_cuda or sp_offsets.dtype != torch.int64 or sp_offsets.dim() != 1 or sp_offsets.numel() < 1:
        raise ValueError("sp_offsets must be a 1-d int64 CUDA tensor of n_states + 1 entries")
    _check_f64(dev, sp_info=sp_info, sp_rhs=sp_rhs, sp_f=sp_f, G11=G11, G22=G22, g1=g1, g2=g2, f=f, prior_info=prior_info,
               prior_rhs=prior_rhs, prior_f=prior_f)
    N = sp_offsets.numel() - 1
    for t in (G11, G22, g1, g2, f, prior_info, prior_rhs, prior_f):
        if t is not None and not t.is_contiguous():
            raise ValueError("the fold writes in place: its targets must be contiguous")
    with _on(dev, stream):
        C, offs, S = _chain_layout(chain_offsets, dev, n_states=N, n_chains=n_chains)
        c = lambda t: None if t is None else t.contiguous()
        _launch(capi.load().cpi_imu_state_priors_fold, dev, stream, C, _tptr(offs), S, _tptr(sp_offsets.contiguous()), _tptr(c(sp_info)),
                _tptr(c(sp_rhs)), _tptr(c(sp_f)), _tptr(G11), _tptr(G22), _tptr(g1), _tptr(g2), _tptr(f), _tptr(prior_info), _tptr(prior_rhs),
                _tptr(prior_f))


def state_priors_robust(loss, loss_k, info, rhs, f, info_out=None, rhs_out=None, f_out=None, stream=None):
    """Robust (Huber / Cauchy) reweighting of moved measurement priors (cpi_imu_state_priors_robust; include/cpi_b200.h, DESIGN.md
    section 3h): with s = f, (info, rhs, f) -> (w(s) info, w(s) rhs, c(s)) per prior.  loss: device int32 [M] (capi.LOSS_*); loss_k:
    float64 [M] (thresholds in standard deviations); info [M,225] / rhs [M,15]: both or None (None: the f-only pass); f [M] the moved
    f' = s.  Outputs are allocated where None (rhs_out may be rhs, f_out may be f).  Returns (info_out, rhs_out, f_out), the first two
    None for the f-only pass."""
    import torch

    dev = f.device
    _check_f64(dev, loss_k=loss_k, info=info, rhs=rhs, f=f, info_out=info_out, rhs_out=rhs_out, f_out=f_out)
    M = f.numel()
    if not loss.is_cuda or loss.device != dev or loss.dtype != torch.int32 or loss.numel() != M or loss_k.numel() != M:
        raise ValueError(f"loss must be an int32 CUDA tensor on {dev} and loss_k float64, one entry per prior")
    if (info is None) != (rhs is None):
        raise ValueError("info and rhs must both be given or both be None")
    if info is not None and (info.numel() != 225 * M or rhs.numel() != 15 * M):
        raise ValueError("info needs 225 doubles and rhs 15 per prior")
    for t in (info_out, rhs_out, f_out):
        if t is not None and not t.is_contiguous():
            raise ValueError("the outputs must be contiguous")
    with _on(dev, stream):
        if info is not None:
            info_out = torch.empty((M, 225), dtype=torch.float64, device=dev) if info_out is None else info_out
            rhs_out = torch.empty((M, 15), dtype=torch.float64, device=dev) if rhs_out is None else rhs_out
        else:
            info_out = rhs_out = None
        f_out = torch.empty(M, dtype=torch.float64, device=dev) if f_out is None else f_out
        c = lambda t: None if t is None else t.contiguous()
        _launch(capi.load().cpi_imu_state_priors_robust, dev, stream, M, _tptr(loss.contiguous()), _tptr(loss_k.contiguous()), _tptr(c(info)),
                _tptr(c(rhs)), _tptr(f.contiguous()), _tptr(info_out), _tptr(rhs_out), _tptr(f_out))
    return info_out, rhs_out, f_out


def chain_marginalize(G11, G12, G22, g1, g2, f, chain_offsets, n_marg, prior=None, n_chains=None, stream=None, state_priors=None,
                      state_prior_loss=None):
    """Eliminate the first n_marg states of every chain into a dense prior on the first state it keeps (cpi_imu_chain_marginalize,
    kernel K8): the Schur complement a fixed-lag smoother keeps of the states that leave its window, at the linearisation point of the
    blocks, undamped.  Blocks as factor_hessian returns them (chain layout as chains_assemble); n_marg: int or device int64 [n_chains]
    (0 <= n_marg < states of the chain); prior: (info [n_chains,225], rhs [n_chains,15], f [n_chains]) on every chain's first state, or
    None.  state_priors: as chains_lm_step, taken as given at the blocks' linearisation point; only those on eliminated states
    (state_idx < offsets[c] + n_marg[c]) are folded, into copies of G11 / g1 / f, so a prior on a kept state is left to the caller.
    state_prior_loss: as chains_lm_step; a robust prior is given moved, (W, rhs', f') with f' = s, and enters with its weight frozen
    at the blocks' linearisation point (state_priors_robust before the fold; f must then be given).
    Returns the prior on state offsets[c] + n_marg[c]: (info [n_chains,225] exactly symmetric, rhs [n_chains,15], f [n_chains])."""
    import torch

    dev = G11.device
    nf = G11.numel() // 225
    with _on(dev, stream):
        C, offs, S = _chain_layout(chain_offsets, dev, n_factors=nf, n_chains=n_chains)
        if state_prior_loss is not None and state_priors is not None and len(state_priors) == 5 and state_priors[3] is None:
            raise ValueError("state_prior_loss: chain_marginalize takes the priors moved, and a robust prior's f' is its s: f must be given")
        sp = _state_priors(state_priors, nf + C, dev, loss=state_prior_loss, measurement=False)
        _check_f64(dev, G11=G11, G12=G12, G22=G22, g1=g1, g2=g2, f=f)
        if any(t.numel() != k * nf for t, k in ((G11, 225), (G12, 225), (G22, 225), (g1, 15), (g2, 15), (f, 1))):
            raise ValueError("G11 / G12 / G22 need 225 doubles, g1 / g2 15 and f 1 per factor")
        pi = pr = pf = None
        if prior is not None:
            pi, pr, pf = prior
            _check_f64(dev, prior_info=pi, prior_rhs=pr, prior_f=pf)
            if pi.numel() != 225 * C or pr.numel() != 15 * C or (pf is not None and pf.numel() != C):
                raise ValueError("the prior needs info [n_chains,225], rhs [n_chains,15] and f [n_chains]")
            pi, pr, pf = pi.contiguous(), pr.contiguous(), (None if pf is None else pf.contiguous())
        if isinstance(n_marg, torch.Tensor):
            if not n_marg.is_cuda or n_marg.device != dev or n_marg.dtype != torch.int64 or n_marg.numel() != C:
                raise ValueError(f"n_marg must be an int64 CUDA tensor on {dev} with one entry per chain")
            nm, nmu = n_marg.contiguous(), 0
        else:
            nm, nmu = None, int(n_marg)
        lib = capi.load()
        if sp is not None:                                           # eliminated states are never last: their priors land in G11 / g1 / f
            idx = sp[0]
            if offs is not None:
                c = (torch.searchsorted(offs, idx, right=True) - 1).clamp(0, C - 1)
                head = offs[c]
            else:
                c = idx // S
                head = c * S
            head = head + (nm[c] if nm is not None else nmu)
            sps = _StatePriors(sp, nf + C, (C, offs, S), key=torch.where(idx < head, idx, idx + nf + C))
            G11, g1, f = G11.contiguous().clone(), g1.contiguous().clone(), f.contiguous().clone()
            # the weights frozen at the blocks' point (s = the given f')
            sps.fold(lib, _stream(dev, stream), sps.rhs, sps.f, G11=G11, g1=g1, f_out=f)
        info = torch.empty((C, 225), dtype=torch.float64, device=dev)
        rhs = torch.empty((C, 15), dtype=torch.float64, device=dev)
        fo = torch.empty((C,), dtype=torch.float64, device=dev)
        _launch(lib.cpi_imu_chain_marginalize, dev, stream, C, _tptr(offs), S, _tptr(nm), nmu, _tptr(G11.contiguous()), _tptr(G12.contiguous()),
                _tptr(G22.contiguous()), _tptr(g1.contiguous()), _tptr(g2.contiguous()), _tptr(f.contiguous()), _tptr(pi), _tptr(pr), _tptr(pf),
                _tptr(info), _tptr(rhs), _tptr(fo))
    return info, rhs, fo


def prior_at(info, rhs, f, lin_states, states, stream=None):
    """A prior (info [n,225], rhs [n,15], f [n] or None) linearised at lin_states [n,16], moved to the states [n,16]
    (cpi_imu_prior_at): delta = local(lin, x) (the inverse of retract), rhs' = rhs - info delta, f' = f - 2 rhs^T delta + delta^T info delta;
    info is unchanged (the Jacobian of local taken as I, as GTSAM's LinearContainerFactor does).  Returns (rhs' [n,15], f' [n])."""
    import torch

    dev, n = _prior_at_checks(info, rhs, f, lin_states, states)
    with _on(dev, stream):
        rhs_out = torch.empty((n, 15), dtype=torch.float64, device=dev)
        f_out = torch.empty((n,), dtype=torch.float64, device=dev)
        _launch(capi.load().cpi_imu_prior_at, dev, stream, n, _tptr(info.contiguous()), _tptr(rhs.contiguous()),
                _tptr(None if f is None else f.contiguous()), _tptr(lin_states.contiguous()), _tptr(states.contiguous()), _tptr(rhs_out), _tptr(f_out))
    return rhs_out, f_out


def _prior_at_checks(info, rhs, f, lin_states, states):
    """prior_at's argument checks; returns (device, n)."""
    dev = info.device
    _check_f64(dev, info=info, rhs=rhs, f=f, lin_states=lin_states, states=states)
    n = info.numel() // 225
    if info.numel() != 225 * n or rhs.numel() != 15 * n or (f is not None and f.numel() != n) or lin_states.numel() != 16 * n or states.numel() != 16 * n:
        raise ValueError("prior_at needs info [n,225], rhs [n,15], f [n], lin_states and states [n,16]")
    return dev, n


def chains_lm_step(model, states, records, lin, chain_offsets, prior=None, lam=1e-5, diagonal_damping=True, stream=None, state_priors=None,
                   state_prior_loss=None, measurements=None, measurement_loss=None):
    """One damped Gauss-Newton step of many independent IMU-only chains at once (a fixed-lag smoother's windows), on the device:
    evaluateError -> information blocks -> prior_at (every chain's prior moved to its current first state) -> chains_assemble ->
    ONE block-cyclic-reduction solve over all chains -> retract.  states [N,16]; records / lin: the N - n_chains factors, chain c's
    stored back to back from index offsets[c] - c; chain_offsets as chains_assemble (device int64 [n_chains+1], or states per chain);
    prior: (info [n_chains,225], rhs [n_chains,15], f [n_chains], lin_states [n_chains,16]) or None.  lin_states = None: the prior is
    linearised at the chains' current first states, so it is used as given without prior_at (rhs and f may then be None: zero).
    state_priors: priors on any states, (state_idx [M] int64, info [M,225], rhs [M,15] or None, f [M] or None, lin [M,16]) or None
    (include/cpi_b200.h, DESIGN.md section 3g): moved to the states by prior_at and folded into the blocks (state_priors_fold).
    state_prior_loss: (loss [M] int32 capi.LOSS_*, loss_k [M] float64) aligned with state_priors, or None (DESIGN.md section 3h): a
    Huber or Cauchy prior (a measurement prior: rhs and f None or zero) is reweighted at the states (state_priors_robust) before the
    fold and costs c(s).
    measurements: (state_idx [M] int64, kind [M] int32 capi.MEAS_*, z [M,3], sqrt_info [M,9], aux [M,3]) or None (DESIGN.md section
    3l): linearised at the states (measurements_linearize) and folded after the state priors; measurement_loss as state_prior_loss.
    Returns (new_states, delta [N,15], cost per chain before the step [n_chains] = sum of e^T P^-1 e + the moved priors' f' + the
    measurements' whitened squared residuals)."""
    import torch

    with _on(states.device, stream):                                 # the one-chain cost and the sum with pf_c on `stream` too
        (C, offs, S), X, (G11, G12, G22, g1, g2, f), (pi_a, pr_c, pf_c) = _linearized(model, states, records, lin, chain_offsets, prior,
                                                                                      stream, state_priors, state_prior_loss,
                                                                                      measurements, measurement_loss)
        D, E, rhs = chains_assemble(G11, G12, G22, g1, g2, chain_offsets, lam, pi_a, pr_c, diagonal_damping=diagonal_damping, n_chains=C,
                                    stream=stream)
        dx = chain_solve(D, E, rhs, stream=stream)
        dev, lib, f64 = X.device, capi.load(), dict(dtype=torch.float64, device=X.device)
        # per-chain cost: one chain sums like chain_lm_step always has; many chains sum their factors' f in a fixed order
        # (cpi_imu_chains_cost_sum: an atomic scatter-add would give different bits from run to run)
        if C == 1:
            cost = f.sum().reshape(1)
        else:
            cost = torch.empty(C, **f64)
            _launch(lib.cpi_imu_chains_cost_sum, dev, stream, C, _tptr(offs), S, _tptr(f), _tptr(cost))
        if pf_c is not None:
            cost = cost + pf_c
        return retract(X, dx, stream=stream), dx, cost


def _linearized(model, states, records, lin, chain_offsets, prior, stream, state_priors, state_prior_loss, measurements=None,
                measurement_loss=None):
    """What chains_lm_step and chains_marginals do before the assembly: the layout and argument checks, the state priors (their one
    host read), the factors' state indices, the buffers and one _linearize at the states.  Returns ((C, offs, S), X [N,16], the
    blocks (G11, G12, G22, g1, g2, f) with the state priors folded in, and the chain prior as the assembly and the cost read it:
    (info, rhs, f), each possibly None).  Its callers run it under _on(dev, stream): every buffer, copy, sort and launch goes on
    `stream`."""
    import torch

    dev = states.device
    N = states.numel() // 16
    C, offs, S = _chain_layout(chain_offsets, dev, n_states=N)
    nf = N - C
    if records.numel() != REC_DOUBLES[model] * nf:
        raise ValueError(f"{C} chains over {N} states hold {nf} factors: one record each")
    sp = _state_priors(state_priors, N, dev, offs, S, loss=state_prior_loss)
    ms = _measurements(measurements, N, dev, offs, S, loss=measurement_loss)
    idx_i, idx_j = _factor_indices(nf, records.device, states, lin, *_chain_factor_states(C, offs, S, nf, dev))
    f64 = dict(dtype=torch.float64, device=dev)
    c = lambda t: None if t is None else t.contiguous()
    pi, pr, pf, lin0 = (None,) * 4 if prior is None else map(c, prior)
    single = (sp is not None and sp[5]) or (ms is not None and ms[5])
    first, x0, pr_c, pf_c = None, None, pr, pf
    if lin0 is not None:
        first = offs[:-1] if offs is not None else torch.arange(C, dtype=torch.int64, device=dev) * S
        x0, pr_c, pf_c = torch.empty((C, 16), **f64), torch.empty((C, 15), **f64), torch.empty(C, **f64)
        _prior_at_checks(pi, pr, pf, lin0, x0)
    elif single:                                                     # the chain prior receives priors: fold into copies (zeros without one)
        pr_c, pf_c = (torch.zeros((C, 15), **f64) if pr is None else pr.clone()), (torch.zeros(C, **f64) if pf is None else pf.clone())
    _check_f64(dev, prior_info=pi, prior_rhs=pr, prior_f=pf)
    if single and pi is None:
        pi = torch.zeros((C, 225), **f64)
    pi_r = torch.empty((C, 225), **f64) if single else None
    X = states.reshape(N, 16).contiguous()
    e, H1, H2 = torch.empty((nf, 15), **f64), torch.empty((nf, 225), **f64), torch.empty((nf, 225), **f64)
    G11, G12, G22 = (torch.empty((nf, 225), **f64) for _ in range(3))
    g1, g2, f = torch.empty((nf, 15), **f64), torch.empty((nf, 15), **f64), torch.empty(nf, **f64)
    folds = _folds(sp, ms, N, (C, offs, S))
    lib = capi.load()
    _linearize(lib, _stream(dev, stream), model, X, records.contiguous(), lin.contiguous(), idx_i, idx_j, (e, H1, H2, G11, G12, G22, g1, g2, f),
               (pi, pr, pf, lin0, first), (x0, pr_c, pf_c), folds, pi_r)
    return (C, offs, S), X, (G11, G12, G22, g1, g2, f), (pi_r if single else pi, pr_c, pf_c)


def _linearize(lib, sp, model, X, records, lin, idx_i, idx_j, blocks, prior, moved, folds, pi_r):
    """The linearisation at the states X [N,16] that chains_lm_step and every round of chains_lm share, on the stream handle sp:
    eval and the information blocks into blocks = (e, H1, H2, G11, G12, G22, g1, g2, f); the chain prior (pi, pr, pf, lin0, first)
    moved to X[first] into moved = (x0, pr_c, pf_c) unless lin0 is None; the fold sources (_folds: state priors, measurements)
    linearised or moved to X, reweighted and folded into the blocks and, on single-state chains, into pi_r (a copy of pi), pr_c and
    pf_c."""
    import torch

    p = _tptr
    e, H1, H2, G11, G12, G22, g1, g2, f = blocks
    pi, pr, pf, lin0, first = prior
    x0, pr_c, pf_c = moved
    if f.numel():
        capi.check(lib.cpi_imu_factor_eval_batch(model, f.numel(), p(X), p(idx_i), p(idx_j), p(records), p(lin), p(e), p(H1), p(H2), sp))
        capi.check(lib.cpi_imu_factor_hessian_batch(model, f.numel(), p(records), p(e), p(H1), p(H2), p(G11), p(G12), p(G22), p(g1), p(g2),
                                                    p(f), sp))
    if lin0 is not None:
        torch.index_select(X, 0, first, out=x0)
        capi.check(lib.cpi_imu_prior_at(x0.shape[0], p(pi), p(pr), p(pf), p(lin0), p(x0), p(pr_c), p(pf_c), sp))
    single = any(s.single for s in folds)
    if single:
        pi_r.copy_(pi)
    for s in folds:
        s.at(lib, sp, X, G11=G11, G22=G22, g1=g1, g2=g2, f_out=f, pi=pi_r, pr=pr_c if single else None, pf=pf_c if single else None)


_PRIOR = {}


def chain_lm_step(model, states, records, lin, lam=1e-5, prior_sigma=1e-4, stream=None, diagonal_damping=True):
    """One damped Gauss-Newton (Levenberg-Marquardt) step of an IMU-only chain, entirely on the device:
    evaluateError for every factor -> information blocks -> block-tridiagonal assembly (prior 1/prior_sigma^2 on x_0: the
    reference initialises with cov = 1e-8 I, GraphSolver.cpp:331; Marquardt damping lam * diag by default, lam = GTSAM's lambdaInitial:
    an undamped IMU-only chain of thousands of keyframes is numerically singular in fp64) -> block-cyclic-reduction solve -> JPLNavState::retract.
    chains_lm_step on one chain, with the prior linearised at the current x_0 (no rhs, no constant: nothing to move).
    Returns (new_states, delta, cost = sum e^T P^-1 e before the step)."""
    import torch

    dev = states.device
    with _on(dev, stream):
        key = (dev, prior_sigma)
        if key not in _PRIOR:
            _PRIOR[key] = (torch.eye(15, dtype=torch.float64, device=dev) / (prior_sigma * prior_sigma)).reshape(1, 225).contiguous()
        new_states, dx, cost = chains_lm_step(model, states, records, lin, states.numel() // 16, (_PRIOR[key], None, None, None), lam=lam,
                                              diagonal_damping=diagonal_damping, stream=stream)
    return new_states, dx, cost[0]


def factor_cost(model, states, records, lin, idx_i=None, idx_j=None, out=None, stream=None):
    """Whitened cost f = e^T P_meas^-1 e of every factor at the states (cpi_imu_factor_cost_batch, kernel K9): factor_hessian's f
    without evaluating or writing e and the blocks; NaN where P_meas is not positive definite.  Indexing as factor_eval.
    Device tensors; returns f [n]."""
    import torch

    import torch

    n = records.numel() // REC_DOUBLES[model]
    dev = records.device
    with _on(dev, stream):
        idx_i, idx_j = _factor_indices(n, dev, states, lin, idx_i, idx_j)
        f = torch.empty((n,), dtype=torch.float64, device=dev) if out is None else out
        _launch(capi.load().cpi_imu_factor_cost_batch, dev, stream, model, n, _tptr(states.contiguous()), _tptr(idx_i), _tptr(idx_j),
                _tptr(records.contiguous()), _tptr(lin.contiguous()), _tptr(f))
    return f


def chains_assemble_lm(G11, G12, G22, g1, g2, chain_offsets, lam, prior_info=None, prior_rhs=None, diagonal_damping=True, n_chains=None,
                       stream=None):
    """chains_assemble with one lambda per chain (cpi_imu_chains_assemble_lm): lam is a device float64 [n_chains].
    Returns (D [N,225], E [N-1,225], rhs [N,15], damp [N,15]) -- damp the diagonal the damping added."""
    return _assemble(G11, G12, G22, g1, g2, chain_offsets, lam, prior_info, prior_rhs, diagonal_damping, n_chains, stream, per_chain=True)


def chains_solve(D, E, rhs, chain_offsets, n_chains=None, workspace=None, stream=None):
    """x = A^-1 rhs by block cyclic reduction with every coupling between two chains structurally absent (cpi_imu_chains_solve): a
    chain that is not SPD gets NaN and leaves every other chain as it is; on SPD input bitwise chain_solve.  chain_offsets as
    chains_assemble."""
    import torch

    dev = D.device
    N = D.numel() // 225
    with _on(dev, stream):
        C, offs, S = _chain_layout(chain_offsets, dev, n_states=N, n_chains=n_chains)
        lib = capi.load()
        x = torch.empty((N, 15), dtype=torch.float64, device=dev)
        nbytes = int(lib.cpi_imu_chains_solve_workspace(C, N))
        if workspace is None or workspace.numel() * 8 < nbytes:
            workspace = torch.empty((nbytes + 7) // 8, dtype=torch.float64, device=dev)
        _launch(lib.cpi_imu_chains_solve, dev, stream, C, _tptr(offs), S, N, _tptr(D.contiguous()), _tptr(E.contiguous()), _tptr(rhs.contiguous()),
                _tptr(x), _tptr(workspace))
    return x


def chains_covariance(D, E, chain_offsets, cross=False, n_chains=None, workspace=None, stream=None):
    """The diagonal blocks and the blocks next to them of A^-1, A = tridiag(E^T, D, E) the system chains_solve solves, by selected
    inversion of its block cyclic reduction (cpi_imu_chains_marginals; DESIGN.md section 3j).  D [N,225], E [N-1,225] as chains_assemble
    returns them; chain_offsets as chains_assemble.  Every coupling between two chains is structurally absent: a chain that is not SPD
    gets NaN blocks and leaves every other chain as it is.  workspace: a float64 CUDA tensor of at least
    cpi_imu_chains_marginals_workspace bytes, or None (allocated).  The call inverts whatever system it is given: marginal covariances
    need the undamped system at the estimate (chains_marginals).  Returns (cov [N,225] with cov[k] = (A^-1)_{k,k}, exactly symmetric;
    with cross, [N - n_chains, 225] with chain c's slot o[c] - c + j = (A^-1)_{o[c]+j, o[c]+j+1}, the factors' order; else None)."""
    import torch

    N = _inverse_checks(D, E, chain_offsets, n_chains, workspace)
    lib = capi.load()
    dev = D.device
    with _on(dev, stream):
        C, offs, S = _chain_layout(chain_offsets, dev, n_states=N, n_chains=n_chains)
        workspace = _inverse_workspace(lib, "cpi_imu_chains_marginals_workspace", C, N, dev, D, E, workspace)
        cov = torch.empty((N, 225), dtype=torch.float64, device=dev)
        cr = torch.empty((N - C, 225), dtype=torch.float64, device=dev) if cross else None
        _launch(lib.cpi_imu_chains_marginals, dev, stream, C, _tptr(offs), S, N, _tptr(D.contiguous()), _tptr(None if E is None else E.contiguous()),
                _tptr(cov), _tptr(cr), _tptr(workspace))
    return cov, cr


def _inverse_checks(D, E, chain_offsets, n_chains, workspace):
    """The host-side checks of chains_covariance and chains_pair_covariance on the system and its layout; returns N."""
    import torch

    for name, t in (("D", D), ("E", E), ("workspace", workspace)):
        if t is not None and (not isinstance(t, torch.Tensor) or t.dtype != torch.float64):
            raise ValueError(f"{name} must be a float64 tensor")
    N = D.numel() // 225
    if N < 1 or D.numel() != 225 * N or (E.numel() if E is not None else 0) != 225 * (N - 1):
        raise ValueError("D needs 225 doubles per state (at least one) and E 225 per state but the last")
    if isinstance(chain_offsets, torch.Tensor) and chain_offsets.numel() - 1 > N:
        raise ValueError(f"chain_offsets has {chain_offsets.numel()} entries: more chains than the {N} states")
    if isinstance(chain_offsets, torch.Tensor) and n_chains is not None and n_chains != chain_offsets.numel() - 1:
        raise ValueError(f"chain_offsets has {chain_offsets.numel()} entries, not n_chains + 1 = {n_chains + 1}")
    return N


def _inverse_workspace(lib, ws_name, C, N, dev, D, E, workspace):
    """The workspace of C chains over N states that the C ABI's ws_name sizes: the caller's, checked, or a new one; D, E and the
    workspace checked to be float64 tensors on dev."""
    import torch

    nbytes = int(getattr(lib, ws_name)(C, N))
    if nbytes < 0:
        raise ValueError(f"{C} chains over {N} states: every chain holds a state")
    if workspace is not None and (workspace.numel() * 8 < nbytes or not workspace.is_contiguous()):
        raise ValueError(f"workspace needs {nbytes} contiguous bytes ({ws_name}), got {workspace.numel() * 8}")
    _check_f64(dev, D=D, E=E, workspace=workspace)
    if workspace is None:
        workspace = torch.empty((nbytes + 7) // 8, dtype=torch.float64, device=dev)
    return workspace


def chains_pair_covariance(D, E, chain_offsets, pairs, n_chains=None, workspace=None, stream=None):
    """Any blocks of A^-1, A = tridiag(E^T, D, E) the system chains_covariance inverts (cpi_imu_chains_pair_covariance; DESIGN.md
    section 3q): GTSAM's Marginals::jointMarginalCovariance for pairs of keyframes.  D, E, chain_offsets, n_chains and the workspace
    (cpi_imu_chains_pair_covariance_workspace bytes) as chains_covariance.  pairs: int64 [q,2] of global state indices (i, j), a CUDA
    tensor on D's device (an index outside [0, N) gives a NaN block) or numpy (range-checked here, then copied to the device from
    pageable memory: the call then waits for `stream`, as the numpy paths of retract and predict_state do).  Returns [q,225]: row p is
    (A^-1)_{i,j}, column-major; (A^-1)_{j,i} is its transpose, a pair (i, i) is exactly symmetric, a pair of states in different chains
    is exactly 0.  GTSAM's 30x30 joint of keyframes {i, j} is the pairs (i, i), (j, j), (i, j)."""
    import torch

    N = _inverse_checks(D, E, chain_offsets, n_chains, workspace)
    dev = D.device
    if isinstance(pairs, torch.Tensor):
        if not pairs.is_cuda or pairs.device != dev or pairs.dtype != torch.int64 or pairs.dim() != 2 or pairs.shape[1] != 2:
            raise ValueError(f"pairs must be an int64 CUDA tensor [q,2] on {dev}, or numpy")
    else:
        pairs = np.asarray(pairs)
        if pairs.dtype.kind not in "iu" or pairs.ndim != 2 or pairs.shape[1] != 2:
            raise ValueError("pairs must be integer [q,2]")
        if pairs.size and (pairs.min() < 0 or pairs.max() >= N):
            raise ValueError(f"pairs index the states 0 .. {N - 1}")
    lib = capi.load()
    with _on(dev, stream):
        C, offs, S = _chain_layout(chain_offsets, dev, n_states=N, n_chains=n_chains)
        workspace = _inverse_workspace(lib, "cpi_imu_chains_pair_covariance_workspace", C, N, dev, D, E, workspace)
        if not isinstance(pairs, torch.Tensor):
            pairs = torch.from_numpy(np.ascontiguousarray(pairs, dtype=np.int64)).to(dev)
        q = pairs.shape[0]
        out = torch.empty((q, 225), dtype=torch.float64, device=dev)
        _launch(lib.cpi_imu_chains_pair_covariance, dev, stream, C, _tptr(offs), S, N, _tptr(D.contiguous()),
                _tptr(None if E is None else E.contiguous()), q, _tptr(pairs[:, 0].contiguous()), _tptr(pairs[:, 1].contiguous()), _tptr(out),
                _tptr(workspace))
    return out


def _marginal_system(model, states, records, lin, chain_offsets, prior, stream, state_priors, state_prior_loss, measurements,
                     measurement_loss):
    """What chains_marginals and chains_pair_marginals invert: the linearisation of chains_lm_step at `states`, assembled with
    lambda = 0.  Returns (n_chains, D, E).  Its callers run it under _on(dev, stream)."""
    (C, _, _), _, (G11, G12, G22, g1, g2, _), (pi_a, pr_c, _) = _linearized(model, states, records, lin, chain_offsets, prior, stream,
                                                                            state_priors, state_prior_loss, measurements, measurement_loss)
    D, E, _ = chains_assemble(G11, G12, G22, g1, g2, chain_offsets, 0.0, pi_a, pr_c, n_chains=C, stream=stream)
    return C, D, E


def chains_marginals(model, states, records, lin, chain_offsets, prior=None, state_priors=None, state_prior_loss=None, cross=False, stream=None,
                     measurements=None, measurement_loss=None):
    """Marginal covariances of every keyframe of many IMU chains at the states (GTSAM's Marginals / BatchFixedLagSmoother::
    marginalCovariance; DESIGN.md section 3j): the linearisation of chains_lm_step at `states` (the chain prior moved there by prior_at,
    the state priors folded in, robust weights frozen at `states` as GTSAM linearises a robust factor for Marginals), assembled with
    lambda = 0, then chains_covariance.  Arguments as chains_lm_step; call it at an estimate (chains_lm's result).  Long IMU-only chains
    without priors on later states are numerically singular in fp64: their covariances are meaningless.  Returns (cov [N,225],
    cross [N - n_chains,225] or None) as chains_covariance, in the tangent space of retract at the states."""
    with _on(states.device, stream):
        C, D, E = _marginal_system(model, states, records, lin, chain_offsets, prior, stream, state_priors, state_prior_loss, measurements,
                                   measurement_loss)
        return chains_covariance(D, E, chain_offsets, cross=cross, n_chains=C, stream=stream)


def chains_pair_marginals(model, states, records, lin, chain_offsets, pairs, prior=None, state_priors=None, state_prior_loss=None,
                          measurements=None, measurement_loss=None, stream=None):
    """Joint marginal covariances of pairs of keyframes of many IMU chains at the states (GTSAM's Marginals::jointMarginalCovariance;
    DESIGN.md section 3q): the system chains_marginals inverts, then chains_pair_covariance on `pairs` (int64 [q,2] of global state
    indices, a CUDA tensor or numpy; numpy pairs make the call wait for `stream`, as in chains_pair_covariance).  Arguments otherwise
    as chains_marginals.  Returns [q,225] as chains_pair_covariance, in the tangent spaces of retract at the states."""
    with _on(states.device, stream):
        C, D, E = _marginal_system(model, states, records, lin, chain_offsets, prior, stream, state_priors, state_prior_loss, measurements,
                                   measurement_loss)
        return chains_pair_covariance(D, E, chain_offsets, pairs, n_chains=C, stream=stream)


def chains_lm(model, states, records, lin, chain_offsets, prior=None, lam=1e-5, diagonal_damping=True, params=None, max_rounds=200, check_every=8,
              stream=None, state_priors=None, state_prior_loss=None, measurements=None, measurement_loss=None):
    """Levenberg-Marquardt of many independent IMU-only chains at once, to convergence, on the device (GTSAM's
    LevenbergMarquardtOptimizer rule per chain: include/cpi_b200.h, DESIGN.md section 3f).  Arguments as chains_lm_step; lam: the
    initial lambda of every chain; params: capi.LMParams (None: GTSAM's defaults).  A prior without a linearisation point is taken as
    linearised at the initial first states.  Per round: eval -> information blocks -> prior_at -> chains_assemble_lm (lambda per chain)
    -> chains_solve (chains isolated) -> retract -> factor_cost + prior_at at the candidate -> cpi_imu_chains_lm_update.  No host
    synchronisation inside the loop except one 4-byte "any chain running" read every check_every rounds (0: max_rounds rounds, fully
    asynchronous).  state_priors as chains_lm_step: every round moves them to the current states after the information blocks and
    folds them in (state_priors_fold), and folds their f' at the candidate into its cost.  state_prior_loss as chains_lm_step: the
    robust priors are reweighted at every round's states before the fold (the weighted info goes to a buffer of the call; the given
    info is constant), and their cost c(s) at the candidate goes into its cost.  measurements / measurement_loss as chains_lm_step:
    every round linearises them at its states after the state priors, and the candidate's cost takes their f-only pass there.  Returns (states [N,16], cost [C] at them,
    lam [C], status [C] int32 (capi.LM_*), iterations [C] (accepted steps), tries [C] (rounds the chain ran)), all int32 counters."""
    import torch

    lib = capi.load()
    dev = states.device
    N = states.numel() // 16
    with _on(dev, stream):
        C, offs, S = _chain_layout(chain_offsets, dev, n_states=N)
        sps = _state_priors(state_priors, N, dev, offs, S, loss=state_prior_loss)
        ms = _measurements(measurements, N, dev, offs, S, loss=measurement_loss)
        _check_f64(dev, states=states, records=records, lin=lin)
        nf = N - C
        if records.numel() != REC_DOUBLES[model] * nf or lin.numel() != 13 * nf:
            raise ValueError(f"{C} chains over {N} states hold {nf} factors: one record and one linearisation point each")
        params = capi.LMParams() if params is None else params
        if max_rounds < 0 or check_every < 0:
            raise ValueError("max_rounds and check_every must be >= 0")
        f64 = dict(dtype=torch.float64, device=dev)
        i32 = dict(dtype=torch.int32, device=dev)
        X = states.reshape(N, 16).clone()
        records, lin = records.contiguous(), lin.contiguous()
        idx_i, idx_j = _chain_factor_states(C, offs, S, nf, dev)
        first = offs[:-1] if offs is not None else torch.arange(C, dtype=torch.int64, device=dev) * S
        pi = pr = pf = lin0 = None
        if prior is not None:
            pi, pr, pf, lin0 = prior
            _check_f64(dev, prior_info=pi, prior_rhs=pr, prior_f=pf, prior_lin=lin0)
            pi = pi.contiguous()
            pr = torch.zeros((C, 15), **f64) if pr is None else pr.contiguous()
            pf = torch.zeros(C, **f64) if pf is None else pf.contiguous()
            lin0 = X.index_select(0, first) if lin0 is None else lin0.contiguous()
        use_prior = prior is not None
        folds = _folds(sps, ms, N, (C, offs, S))
        single = any(s.single for s in folds)
        if folds:
            if single and not use_prior:                             # a chain of one state carries priors: a zero chain prior receives them
                pi, pr, pf, lin0 = torch.zeros((C, 225), **f64), torch.zeros((C, 15), **f64), torch.zeros(C, **f64), X.index_select(0, first)
                use_prior = True
        pi_r = torch.empty((C, 225), **f64) if single else None      # the chain prior's info with the round's priors folded in
        lam_t = torch.full((C,), float(lam), **f64)
        cost = torch.zeros(C, **f64)
        status, iters, tries = torch.zeros(C, **i32), torch.zeros(C, **i32), torch.zeros(C, **i32)
        flag = torch.zeros(1, **i32)
        # round buffers, allocated once
        e, H1, H2 = torch.empty((nf, 15), **f64), torch.empty((nf, 225), **f64), torch.empty((nf, 225), **f64)
        G11, G12, G22 = (torch.empty((nf, 225), **f64) for _ in range(3))
        g1, g2, f_cur, f_new = torch.empty((nf, 15), **f64), torch.empty((nf, 15), **f64), torch.empty(nf, **f64), torch.empty(nf, **f64)
        D, E, rhs, damp = torch.empty((N, 225), **f64), torch.empty((max(N - 1, 1), 225), **f64), torch.empty((N, 15), **f64), torch.empty((N, 15), **f64)
        dx, Xn, x0 = torch.empty((N, 15), **f64), torch.empty((N, 16), **f64), torch.empty((C, 16), **f64)
        pr_c, pf_c, pr_n, pf_n = torch.empty((C, 15), **f64), torch.empty(C, **f64), torch.empty((C, 15), **f64), torch.empty(C, **f64)
        ws_solve = torch.empty((int(lib.cpi_imu_chains_solve_workspace(C, N)) + 7) // 8, **f64)
        ws_lm = torch.empty((int(lib.cpi_imu_chains_lm_workspace(N)) + 7) // 8, **f64)
        p = _tptr
        blocks, chain_prior, moved = (e, H1, H2, G11, G12, G22, g1, g2, f_cur), (pi, pr, pf, lin0, first), (x0, pr_c, pf_c)
        sp = _stream(dev, stream)
        for r in range(max_rounds):
            check = check_every > 0 and (r + 1) % check_every == 0
            _linearize(lib, sp, model, X, records, lin, idx_i, idx_j, blocks, chain_prior, moved, folds, pi_r)
            capi.check(lib.cpi_imu_chains_assemble_lm(C, p(offs), S, p(G11), p(G12), p(G22), p(g1), p(g2), p(lam_t), int(bool(diagonal_damping)),
                                                      p(pi_r if single else pi), p(pr_c if use_prior else None), p(D), p(E), p(rhs), p(damp), sp))
            capi.check(lib.cpi_imu_chains_solve(C, p(offs), S, N, p(D), p(E), p(rhs), p(dx), p(ws_solve), sp))
            capi.check(lib.cpi_retract_batch(N, p(X), p(dx), p(Xn), sp))
            if nf:
                capi.check(lib.cpi_imu_factor_cost_batch(model, nf, p(Xn), p(idx_i), p(idx_j), p(records), p(lin), p(f_new), sp))
            if use_prior:
                torch.index_select(Xn, 0, first, out=x0)
                capi.check(lib.cpi_imu_prior_at(C, p(pi), p(pr), p(pf), p(lin0), p(x0), p(pr_n), p(pf_n), sp))
            for s in folds:                                      # the state priors' and measurements' cost at the candidate
                s.at(lib, sp, Xn, cost_only=True, f_out=f_new, pf=pf_n if single else None)
            if check:
                flag.zero_()
            capi.check(lib.cpi_imu_chains_lm_update(C, p(offs), S, N, ctypes.byref(params), p(f_cur), p(pf_c if use_prior else None),
                                                    p(f_new), p(pf_n if use_prior else None), p(rhs), p(D), p(E), p(damp), p(dx), p(Xn),
                                                    p(X), p(lam_t), p(cost), p(status), p(iters), p(tries), p(flag if check else None),
                                                    p(ws_lm), sp))
            if check and int(flag.item()) == 0:
                break
    return X, cost, lam_t, status, iters, tries


def relinearize_records(model, states, records, lin, chain_offsets, samples, sigmas, sample_offsets=None, ns=None, flags=0, *, tol_bw, tol_ba,
                        tol_theta=math.inf, stream=None, workspace=None):
    """Re-preintegrate, on the device, the windows whose state bias left the records' linearisation point
    (cpi_imu_records_relinearize; include/cpi_b200.h, DESIGN.md section 3i).  Between solves:
    chains_lm -> relinearize_records -> if n > 0: chains_lm again from the new states.
    states [N,16], records / lin: the factors of the chain layout (chain_offsets as chains_lm; factor k reads the bias of its state
    i); samples / sample_offsets / ns / sigmas / flags: the windows as preint.preintegrate took them (sample_offsets a device int64
    tensor [n_factors + 1], or None with ns steps per window).  tol_bw (rad/s), tol_ba (m/s^2), tol_theta (rad, model 2 only):
    >= 0, math.inf disables a test.  A selected factor gets lin = [bg_i, ba_i, q_i (model 2; model 1 keeps its q), grav] and the
    record of its window at that point; the others keep their bits.  records and lin are updated IN PLACE (both contiguous float64).
    workspace: a CUDA tensor of at least cpi_imu_records_relinearize_workspace bytes, allocated here when absent or too small.
    One host synchronisation (the count).  Returns (n_relinearized, mask [n_factors] int32 device tensor)."""
    import torch

    lib = capi.load()
    if model not in (1, 2):
        raise ValueError(f"model must be 1 or 2 (got {model})")
    capi.check_discrete(model, 64, flags)
    for name, t in (("tol_bw", tol_bw), ("tol_ba", tol_ba), ("tol_theta", tol_theta)):
        if not float(t) >= 0.0:
            raise ValueError(f"{name} must be >= 0 (math.inf disables the test; got {t})")
    dev = states.device
    for name, t in (("states", states), ("records", records), ("lin", lin), ("samples", samples)):
        if t.dtype != torch.float64:
            raise ValueError(f"{name} must be float64")
    N = states.numel() // 16
    with _on(dev, stream):
        C, offs, S = _chain_layout(chain_offsets, dev, n_states=N)
        nf = N - C
        if records.numel() != REC_DOUBLES[model] * nf or lin.numel() != 13 * nf:
            raise ValueError(f"{C} chains over {N} states hold {nf} factors: one record ({REC_DOUBLES[model]} doubles) and one linearisation "
                             f"point (13) each")
        if not records.is_contiguous() or not lin.is_contiguous():
            raise ValueError("records and lin are updated in place: they must be contiguous")
        n_ent = samples.numel() // 7
        avg = 1 if flags & FLAG_IMU_AVG else 0
        if sample_offsets is not None:
            if sample_offsets.dtype != torch.int64 or sample_offsets.numel() != nf + 1:
                raise ValueError(f"sample_offsets must be an int64 tensor with n_factors + 1 = {nf + 1} entries")
            sample_offsets, ns = sample_offsets.contiguous(), 0
        else:
            if ns is None or int(ns) < 0:
                raise ValueError("give sample_offsets, or ns >= 0 steps per window")
            ns = int(ns)
            if n_ent < nf * (ns + avg):
                raise ValueError("sample tensor shorter than n_factors * (ns + imu_avg)")
        _check_f64(dev, states=states, records=records, lin=lin, samples=samples)
        if sample_offsets is not None and (not sample_offsets.is_cuda or sample_offsets.device != dev):
            raise ValueError(f"sample_offsets must be a CUDA tensor on {dev}")
        idx_i, _ = _chain_factor_states(C, offs, S, nf, dev)
        nbytes = int(lib.cpi_imu_records_relinearize_workspace(model, nf, n_ent))
        if nbytes < 0:
            capi.check(nbytes)
        if workspace is None or workspace.numel() * workspace.element_size() < nbytes or not workspace.is_contiguous():
            workspace = torch.empty((nbytes + 7) // 8, dtype=torch.float64, device=dev)
        mask = torch.zeros(nf, dtype=torch.int32, device=dev)
        sig = np.ascontiguousarray(sigmas, dtype=np.float64)
        if sig.shape != (4,):
            raise ValueError("sigmas must be the four sigmas (sigma_w, sigma_wb, sigma_a, sigma_ab)")
        count = ctypes.c_int64(0)
        _launch(lib.cpi_imu_records_relinearize, dev, stream, model, nf, _tptr(states.contiguous()), _tptr(idx_i), _tptr(sample_offsets), ns,
                _tptr(samples.contiguous()), _ptr(sig), int(flags), float(tol_bw), float(tol_ba), float(tol_theta), _tptr(lin), _tptr(records),
                _tptr(mask), ctypes.byref(count), _tptr(workspace))
    return int(count.value), mask


def predict_state(model, states_k, records, lin, stream=None):
    """getpredictedstate_v1/_v2 (solvers/GraphSolver_IMU.cpp:263-307), batched.  Device tensors, or numpy (staged via torch)."""
    import torch

    lib = capi.load()

    def run(states_k, records, lin):
        dev = states_k.device
        _check_f64(dev, states_k=states_k, records=records, lin=lin)
        n = states_k.numel() // 16
        with _on(dev, stream):
            out = torch.empty((n, 16), dtype=torch.float64, device=dev)
            _launch(lib.cpi_predict_state_batch, dev, stream, model, n, _tptr(states_k.contiguous()), _tptr(records.contiguous()),
                    _tptr(lin.contiguous()), _tptr(out))
        return out
    return _staged(run, stream, states_k, records, lin)


def propagate(model, states_k, cov_k, records, lin, anchor=None, want_cross=False, stream=None):
    """Prediction with covariance (cpi_propagate_batch): x_k1 = predict_state(x_k, record), cov_k1 = A cov_k A^T + B P_meas B^T with
    A = -H2^-1 H1, B = H2^-1 the factor Jacobians at (x_k, x_k1); cross = cov_k A^T.  DEVICE float64 tensors: states_k [m,16],
    cov_k [m,225] (column-major 15x15), records [n,RD], lin [n,13], anchor int64 [n] or None (window i starts from entry anchor[i],
    None: from entry i).  Enqueues on ``stream`` (default: torch's current stream) without synchronising.
    Returns (states_k1 [n,16], cov_k1 [n,225], cross [n,225] or None)."""
    import torch

    lib = capi.load()
    n = records.numel() // REC_DOUBLES[model]
    dev = records.device
    for name, t in (("states_k", states_k), ("cov_k", cov_k), ("lin", lin), ("anchor", anchor)):
        if t is not None and (not t.is_cuda or t.device != dev):
            raise ValueError(f"{name} must be a CUDA tensor on {dev}")
    for name, t in (("states_k", states_k), ("cov_k", cov_k), ("records", records), ("lin", lin)):
        if t.dtype != torch.float64:
            raise ValueError(f"{name} must be float64")
    m = states_k.numel() // 16
    if cov_k.numel() != 225 * m or lin.numel() != 13 * n:
        raise ValueError("cov_k needs 225 doubles per anchor state and lin 13 per record")
    if anchor is None:
        if m < n:
            raise ValueError("without an anchor array window i starts from entry i: states_k needs one entry per record")
    else:
        if anchor.dtype != torch.int64 or anchor.numel() != n:
            raise ValueError("anchor must be an int64 tensor with one entry per record")
    with _on(dev, stream):
        anchor = None if anchor is None else anchor.contiguous()
        x1 = torch.empty((n, 16), dtype=torch.float64, device=dev)
        c1 = torch.empty((n, 225), dtype=torch.float64, device=dev)
        cr = torch.empty((n, 225), dtype=torch.float64, device=dev) if want_cross else None
        _launch(lib.cpi_propagate_batch, dev, stream, model, n, _tptr(states_k.contiguous()), _tptr(cov_k.contiguous()), _tptr(anchor),
                _tptr(records.contiguous()), _tptr(lin.contiguous()), _tptr(x1), _tptr(c1), _tptr(cr))
    return x1, c1, cr


def propagate_host(model, states_k, cov_k, records, lin, anchor=None, want_cross=False):
    """HOST numpy in/out through ``cpi_propagate_batch_host`` (synchronous); arguments and results as ``propagate``."""
    lib = capi.load()
    states_k = np.ascontiguousarray(states_k, dtype=np.float64).reshape(-1, 16)
    cov_k = np.ascontiguousarray(cov_k, dtype=np.float64).reshape(-1, 225)
    records = np.ascontiguousarray(records, dtype=np.float64).reshape(-1, REC_DOUBLES[model])
    lin = np.ascontiguousarray(lin, dtype=np.float64).reshape(-1, 13)
    n, m = records.shape[0], states_k.shape[0]
    if lin.shape[0] != n or cov_k.shape[0] != m:
        raise ValueError("one linearisation point per record and one covariance per anchor state required")
    if anchor is not None:
        anchor = np.ascontiguousarray(anchor, dtype=np.int64)
        if anchor.shape != (n,):
            raise ValueError("anchor must have one entry per record")
    x1 = np.empty((n, 16)); c1 = np.empty((n, 225)); cr = np.empty((n, 225)) if want_cross else None
    capi.check(lib.cpi_propagate_batch_host(model, n, m, _ptr(states_k), _ptr(cov_k), _ptr(anchor), _ptr(records), _ptr(lin),
                                            _ptr(x1), _ptr(c1), _ptr(cr)))
    return x1, c1, cr


def retract(states, xi, stream=None):
    """JPLNavState::retract (gtsam/JPLNavState.cpp:37-71), batched."""
    import torch

    lib = capi.load()

    def run(states, xi):
        dev = states.device
        _check_f64(dev, states=states, xi=xi)
        n = states.numel() // 16
        with _on(dev, stream):
            out = torch.empty((n, 16), dtype=torch.float64, device=dev)
            _launch(lib.cpi_retract_batch, dev, stream, n, _tptr(states.contiguous()), _tptr(xi.contiguous()), _tptr(out))
        return out
    return _staged(run, stream, states, xi)


def update(states, cov, meas_info, meas_states, gate=None, stream=None):
    """Measurement update of n filters by direct state fixes, with chi-square gating (cpi_state_update_batch, kernel K10; DESIGN.md
    section 3k): the update step of the filter that ``propagate`` predicts.  DEVICE float64 tensors: states [n,16], cov [n,225] (SPD,
    column-major, the tangent space of retract), meas_info [n,225] (W, PSD, zero outside the blocks it measures), meas_states [n,16]
    (x_bar, the fix in the convention of the state priors: residual local(x_bar, x), Jacobian taken as I).  With d = local(x_bar, x):
        xi = -(cov^-1 + W)^-1 W d,   cov+ = (cov^-1 + W)^-1,   x+ = retract(x, xi),   nis = (d+xi)^T W (d+xi) + xi^T cov^-1 xi
    computed in square-root form.  gate: None (every fix applied), a float, or a float64 CUDA tensor [n]; the fix of filter i is
    skipped when nis[i] > gate[i] (its state and cov are copied bit for bit).  NaN gates are rejected, +inf is allowed.  Enqueues on
    ``stream`` (default: torch's current stream); a float gate is filled on that stream.  A tensor gate is checked for NaN with one
    host read, which synchronises with ``stream``; a float gate or None does not synchronise.
    Returns (states [n,16], cov [n,225] exactly symmetric, nis [n], applied [n] int32 0/1)."""
    import torch

    dev, n = _filter_checks(states, cov, gate, "update")
    for name, t in (("meas_info", meas_info), ("meas_states", meas_states)):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"{name} must be a tensor")
    _check_f64(dev, meas_info=meas_info, meas_states=meas_states)
    if meas_info.numel() != 225 * n or meas_states.numel() != 16 * n:
        raise ValueError("update needs meas_info [n,225] and meas_states [n,16]")
    f64 = dict(dtype=torch.float64, device=dev)
    with _on(dev, stream):                                           # the gate's check and fill are ordered with the launch
        gate = _filter_gate(gate, n, f64)
        x1, c1, nis = torch.empty((n, 16), **f64), torch.empty((n, 225), **f64), torch.empty(n, **f64)
        applied = torch.empty(n, dtype=torch.int32, device=dev)
        if n:
            _launch(capi.load().cpi_state_update_batch, dev, stream, n, _tptr(states.contiguous()), _tptr(cov.contiguous()),
                    _tptr(meas_info.contiguous()), _tptr(meas_states.contiguous()), _tptr(gate), _tptr(x1), _tptr(c1), _tptr(nis),
                    _tptr(applied))
    return x1, c1, nis, applied


def update_measurements(states, cov, measurements, gate=None, stream=None):
    """Measurement update of n filters by the measurements of DESIGN.md section 3l (cpi_state_update_measurements_batch, kernel K11):
    GNSS at a lever arm, body-frame velocity and known directions, linearised at the predicted states.  states [n,16], cov [n,225] as
    ``update``; measurements as chains_lm_step's, (state_idx [M] int64, kind [M] int32 capi.MEAS_*, z [M,3], sqrt_info [M,9], aux
    [M,3]), with state_idx indexing the FILTERS: every measurement of a filter is applied in one update, stably sorted by filter.  With
    A_j, b_j the whitened rows at x, Sigma = L L^T, B_j = A_j L and C = chol(I + sum B_j^T B_j):
        w = -C^-T C^-1 sum B_j^T b_j,  xi = L w,  cov+ = M M^T with M = L C^-T,  x+ = retract(x, xi),  nis = sum |b_j + A_j xi|^2 + |w|^2
    A filter without measurements is copied bit for bit with nis = 0 and applied = 1.  gate as ``update``.  The measurements are
    validated like state_priors (one host read for the filter indices and kind codes).
    Returns (states [n,16], cov [n,225] exactly symmetric, nis [n], applied [n] int32 0/1)."""
    import torch

    dev, n = _filter_checks(states, cov, gate, "update_measurements")
    f64 = dict(dtype=torch.float64, device=dev)
    with _on(dev, stream):                                           # the checks' host reads, the gate's fill and the sort too
        ms = _measurements(measurements, n, dev)
        gate = _filter_gate(gate, n, f64)
        offsets, kind, z, si, aux, _ = _filter_csr(ms, n, f64)
        x1, c1, nis = torch.empty((n, 16), **f64), torch.empty((n, 225), **f64), torch.empty(n, **f64)
        applied = torch.empty(n, dtype=torch.int32, device=dev)
        if n:
            _launch(capi.load().cpi_state_update_measurements_batch, dev, stream, n, _tptr(states.contiguous()), _tptr(cov.contiguous()),
                    _tptr(offsets), _tptr(kind), _tptr(z), _tptr(si), _tptr(aux), _tptr(gate), _tptr(x1), _tptr(c1), _tptr(nis),
                    _tptr(applied))
    return x1, c1, nis, applied


def update_measurements_iterated(states, cov, measurements, gate=None, measurement_loss=None, max_iterations=10, tol=1e-9, stream=None):
    """The iterated EKF update of n filters by the measurements of ``update_measurements``, with Huber and Cauchy losses
    (cpi_state_update_measurements_iterated_batch, kernel K13; DESIGN.md section 3m): Gauss-Newton on the one-step MAP problem
    |L^-1 local(x, x')|^2 + sum_j rho_j(|b_j(x')|^2) (Sigma = cov = L L^T, the prior's Jacobian taken as I), relinearising every
    measurement at each iterate and reweighting it by IRLS.  From x_0 = x, with d_t = local(x, x_t), A_j, b_j at x_t and om_j the
    IRLS weight of |b_j|^2:
        B_j = sqrt(om_j) A_j L,  b'_j = sqrt(om_j) (b_j - A_j d_t),  C = chol(I + sum B_j^T B_j),  w = C^-T C^-1 sum B_j^T b'_j,
        delta = -L w - d_t,  x_{t+1} = retract(x_t, delta)
    until max_k |delta_k| <= tol sqrt(cov_kk) (status 1) or max_iterations linearisations (status 2).  cov+ = M M^T with M = L C^-T of
    the last linearisation (exactly symmetric); nis is gamma of the first linearisation, sum_j om_j |b_j + A_j eps_0|^2 + |w_0|^2 with
    eps_0 = -L w_0 (K11's gamma without a loss), and the gate compares it before iterating: a gated filter is copied bit for bit with
    status 0.  A filter without measurements is copied bit for bit with nis 0, status 1 and 0 iterations.  tol = +inf takes one
    iteration (update_measurements without a loss, to rounding); tol = 0 takes max_iterations unless a step is exactly zero.
    states, cov, measurements and gate as ``update_measurements``; measurement_loss as chains_lm_step's, (loss [M] int32 capi.LOSS_*,
    loss_k [M] float64) or None (every measurement Gaussian), validated with the measurements' one host read.  max_iterations: int
    >= 1; tol: float >= 0 (+inf allowed), in the prior's standard deviations.
    Returns (states [n,16], cov [n,225], nis [n], status [n] int32 0 gated / 1 converged / 2 stopped at max_iterations,
    iterations [n] int32 linearisations)."""
    import torch

    if isinstance(max_iterations, bool) or not isinstance(max_iterations, (int, np.integer)) or not 1 <= max_iterations < 2 ** 31:
        raise ValueError(f"max_iterations must be an int >= 1 (got {max_iterations!r})")
    if not isinstance(tol, (int, float, np.floating)) or isinstance(tol, bool) or not float(tol) >= 0.0:
        raise ValueError(f"tol must be a float >= 0 (+inf: one iteration; got {tol!r})")
    dev, n = _filter_checks(states, cov, gate, "update_measurements_iterated")
    f64 = dict(dtype=torch.float64, device=dev)
    with _on(dev, stream):                                           # the checks' host reads, the gate's fill and the sort too
        ms = _measurements(measurements, n, dev, loss=measurement_loss)
        gate = _filter_gate(gate, n, f64)
        offsets, kind, z, si, aux, loss = _filter_csr(ms, n, f64)
        x1, c1, nis = torch.empty((n, 16), **f64), torch.empty((n, 225), **f64), torch.empty(n, **f64)
        status, iters = torch.empty(n, dtype=torch.int32, device=dev), torch.empty(n, dtype=torch.int32, device=dev)
        if n:
            _launch(capi.load().cpi_state_update_measurements_iterated_batch, dev, stream, n, _tptr(states.contiguous()),
                    _tptr(cov.contiguous()), _tptr(offsets), _tptr(kind), _tptr(z), _tptr(si), _tptr(aux), _tptr(loss[0]), _tptr(loss[1]),
                    _tptr(gate), int(max_iterations), float(tol), _tptr(x1), _tptr(c1), _tptr(nis), _tptr(status), _tptr(iters))
    return x1, c1, nis, status, iters


def rts_smooth(model, states, cov, records, lin, run_offsets, cross=False, n_runs=None, stream=None):
    """Fixed-interval (Rauch-Tung-Striebel) smoothing of many filter runs from the filter's own posteriors (cpi_rts_smooth_batch,
    kernel K15; DESIGN.md section 3o).  Runs use the chain layout of chains_marginals: run_offsets is a device int64 tensor [n_runs+1]
    of keyframe offsets or an int, the keyframes per run (n_runs as chains_covariance's n_chains); run c's transitions are stored back
    to back from index offsets[c] - c.  DEVICE float64 tensors: states [N,16] and cov [N,225] (column-major) the filter's posterior
    (x_k, P_k) at every keyframe, the prediction itself where no update was applied; records [N - n_runs, RD] and lin
    [N - n_runs, 13] per transition.  The records and lin must be the ones the filter propagated with.  One propagate(...,
    want_cross=True) call over every transition recomputes the predictions (xb_{k+1}, Pb_{k+1}) and the cross C_k = P_k A_k^T; K7 is
    deterministic, so they are bitwise the forward pass's own.  That pass allocates 3 728 B per transition (16 + 225 + 225 doubles).
    Then, per run from its last keyframe (copied bit for bit) backwards:
        G = C_k Pb_{k+1}^-1,  xs_k = retract(x_k, G local(xb_{k+1}, xs_{k+1})),  Ps_k = P_k + G (Ps_{k+1} - Pb_{k+1}) G^T,
        Xs_k = G Ps_{k+1}
    A Pb_{k+1} that is not SPD gives NaN for that run only.  Enqueues on ``stream`` (default: torch's current stream) without
    synchronising.  Returns (states_s [N,16], cov_s [N,225] exactly symmetric, cross_s [N - n_runs,225] with Xs_k in transition k's
    slot, the slots and orientation of chains_covariance's cross, or None)."""
    return _rts_smooth(False, model, states, cov, records, lin, run_offsets, cross, n_runs, stream)


def rts_smooth_scan(model, states, cov, records, lin, run_offsets, cross=False, n_runs=None, stream=None):
    """rts_smooth's smoothing, parallel in time (cpi_rts_smooth_scan_batch, kernel K16; DESIGN.md section 3p): the same arguments,
    checks, K7 pass and return values, then a segmented associative scan over every keyframe of every run instead of one warp
    walking each run, so that one long run spreads over the whole device.  Covariances and cross are rts_smooth's up to
    reassociation; the means follow the backward recursion linearised at the filtered states,
        xs_k = retract(x_k, delta_k),  delta_k = G_k d0_k + G_k J_k delta_{k+1},  d0_k = local(xb_{k+1}, x_{k+1}),
    which agrees with rts_smooth's to second order in delta (the parallel extended RTS smoother of Sarkka and Garcia-Fernandez).
    Faster than rts_smooth on few long runs, slower on many short ones (DESIGN.md section 3p has the crossover).  Allocates the
    workspace (cpi_rts_smooth_scan_workspace bytes: about 5.5 KB per keyframe) on the stream's device.  Enqueues on ``stream``
    (default: torch's current stream) without synchronising.  Returns (states_s [N,16], cov_s [N,225] exactly symmetric, cross_s
    [N - n_runs,225] or None)."""
    return _rts_smooth(True, model, states, cov, records, lin, run_offsets, cross, n_runs, stream)


def _rts_smooth(scan, model, states, cov, records, lin, run_offsets, cross, n_runs, stream):
    """rts_smooth (K15) or, scan True, rts_smooth_scan (K16): the checks, the run layout, the K7 pass, the outputs, the scan's
    workspace and the launch."""
    import torch

    name = "rts_smooth_scan" if scan else "rts_smooth"
    if model not in (1, 2):
        raise ValueError(f"model must be 1 or 2 (got {model!r})")
    for what, t in (("states", states), ("cov", cov), ("records", records), ("lin", lin)):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"{what} must be a tensor")
    if not states.is_cuda:
        raise ValueError("states must be a CUDA tensor")
    dev = states.device
    _check_f64(dev, states=states, cov=cov, records=records, lin=lin)
    N = states.numel() // 16
    if N < 1 or states.numel() != 16 * N or cov.numel() != 225 * N:
        raise ValueError(f"{name} needs states [N,16] and cov [N,225] with at least one keyframe")
    if isinstance(run_offsets, torch.Tensor):
        if run_offsets.numel() - 1 > N:
            raise ValueError(f"run_offsets has {run_offsets.numel()} entries: more runs than the {N} keyframes")
        if n_runs is not None and n_runs != run_offsets.numel() - 1:
            raise ValueError(f"run_offsets has {run_offsets.numel()} entries, not n_runs + 1 = {n_runs + 1}")
    with _on(dev, stream):
        C, offs, S = _chain_layout(run_offsets, dev, n_states=N, n_chains=n_runs)
        nt = N - C
        if C < 1 or nt < 0:
            raise ValueError(f"{C} runs over {N} keyframes: every run holds a keyframe")
        if records.numel() != nt * REC_DOUBLES[model] or lin.numel() != 13 * nt:
            raise ValueError(f"{N - C} transitions need records [{nt},{REC_DOUBLES[model]}] and lin [{nt},13]")
        states, cov = states.contiguous(), cov.contiguous()
        lib = capi.load()
        if nt:
            idx_i, _ = _chain_factor_states(C, offs, S, nt, dev)
            xp, cp, cr = propagate(model, states, cov, records, lin, anchor=idx_i, want_cross=True, stream=stream)
            ws = torch.empty(int(lib.cpi_rts_smooth_scan_workspace(C, N)), dtype=torch.uint8, device=dev) if scan else None
        else:
            xp = cp = cr = ws = None
        f64 = dict(dtype=torch.float64, device=dev)
        xs, cs = torch.empty((N, 16), **f64), torch.empty((N, 225), **f64)
        xc = torch.empty((nt, 225), **f64) if cross else None
        args = (C, _tptr(offs), S, N, _tptr(states), _tptr(cov), _tptr(xp), _tptr(cp), _tptr(cr), _tptr(xs), _tptr(cs), _tptr(xc))
        if scan:
            _launch(lib.cpi_rts_smooth_scan_batch, dev, stream, *args, _tptr(ws))
        else:
            _launch(lib.cpi_rts_smooth_batch, dev, stream, *args)
    return xs, cs, xc


def _filter_checks(states, cov, gate, name):
    """The host checks of the filter updates by measurements: states [n,16] and cov [n,225] float64 CUDA tensors on one device, and a
    gate that is None, a number other than NaN, or a float64 tensor [n] on that device.  Returns (device, n)."""
    import torch

    for what, t in (("states", states), ("cov", cov)):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"{what} must be a tensor")
    if not states.is_cuda:
        raise ValueError("states must be a CUDA tensor")
    dev = states.device
    _check_f64(dev, states=states, cov=cov)
    n = states.numel() // 16
    if states.numel() != 16 * n or cov.numel() != 225 * n:
        raise ValueError(f"{name} needs states [n,16] and cov [n,225]")
    if isinstance(gate, torch.Tensor):
        _check_f64(dev, gate=gate)
        if gate.numel() != n:
            raise ValueError(f"gate needs one entry per filter ({n}), got {gate.numel()}")
    elif gate is not None and math.isnan(float(gate)):
        raise ValueError("gate must not be NaN (+inf applies every update)")
    return dev, n


def _filter_gate(gate, n, f64):
    """The gate as the kernels read it, on the current stream: a tensor gate checked for NaN (one host read), a number filled in."""
    import torch

    if isinstance(gate, torch.Tensor):
        gate = gate.contiguous()
        if bool(torch.isnan(gate).any()):
            raise ValueError("gate must not be NaN (+inf applies every update)")
    elif gate is not None:
        gate = torch.full((n,), float(gate), **f64)
    return gate


def _filter_csr(ms, n, f64):
    """The validated measurements ms (_measurements) of n filters as the kernels read them, on the current stream: (offsets [n+1],
    kind, z, sqrt_info, aux, (loss, loss_k)) sorted stably by filter, the loss permuted alike ((None, None) without one).  Without
    measurements every filter is copied: offsets are zero and one row keeps the pointers valid."""
    import torch

    if ms is None:
        dev = f64["device"]
        return (torch.zeros(n + 1, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros((1, 3), **f64),
                torch.zeros((1, 9), **f64), torch.zeros((1, 3), **f64), (None, None))
    order, offsets = _state_prior_csr(ms[0], n)
    kind, z, si, aux = (t[order].contiguous() for t in ms[1:5])
    loss = (None, None) if ms[6] is None else tuple(t[order].contiguous() for t in ms[6])
    return offsets, kind, z, si, aux, loss


class JPLNavState:
    """gtsam/JPLNavState.h:59-151: [q_GtoI(4, JPL xyzw), biasg(3), v_IinG(3), biasa(3), p_IinG(3)], dimension 15."""
    dimension = 15

    def __init__(self, q=(0, 0, 0, 1), bg=(0, 0, 0), v=(0, 0, 0), ba=(0, 0, 0), p=(0, 0, 0)):
        self._x = np.concatenate([np.asarray(a, dtype=np.float64).reshape(-1) for a in (q, bg, v, ba, p)])
        assert self._x.shape == (16,)

    @classmethod
    def from_vector(cls, x):
        x = np.asarray(x, dtype=np.float64).reshape(16)
        return cls(x[0:4], x[4:7], x[7:10], x[10:13], x[13:16])

    def vector(self): return self._x.copy()
    def q(self): return self._x[0:4].copy()
    def bg(self): return self._x[4:7].copy()
    def v(self): return self._x[7:10].copy()
    def ba(self): return self._x[10:13].copy()
    def p(self): return self._x[13:16].copy()

    def retract(self, xi):
        return JPLNavState.from_vector(retract(self._x[None], np.asarray(xi, dtype=np.float64).reshape(1, 15))[0])

    def equals(self, other, tol=1e-8):
        return bool(np.all(np.abs(self._x - other._x) <= tol))


class _ImuFactorCPI:
    model = 0

    def _pack(self, covariance, deltatime, grav, alpha, beta, q_KtoK1, q_K_lin, ba_lin, bg_lin, J_q, J_beta, J_alpha, H_beta, H_alpha,
              O_beta=None, O_alpha=None):
        rec = np.zeros(REC_DOUBLES[self.model])

        def put(name, a):
            lo, hi = REC[name]
            rec[lo:hi] = np.asarray(a, dtype=np.float64).reshape(-1, order="F")
        put("q", q_KtoK1); put("alpha", alpha); put("beta", beta); rec[19] = float(deltatime)
        put("J_q", J_q); put("J_a", J_alpha); put("J_b", J_beta); put("H_a", H_alpha); put("H_b", H_beta); put("P", covariance)
        if self.model == 2:
            put("O_a", O_alpha); put("O_b", O_beta)
        self._rec = rec
        self._lin = np.concatenate([np.asarray(bg_lin, dtype=np.float64).reshape(3), np.asarray(ba_lin, dtype=np.float64).reshape(3),
                                    np.asarray(q_K_lin, dtype=np.float64).reshape(4), np.asarray(grav, dtype=np.float64).reshape(3)])

    # accessors of the reference class (ImuFactorCPIv1.h:104-134)
    def dt(self): return float(self._rec[19])
    def m_alpha(self): return self._rec[13:16].copy()
    def m_beta(self): return self._rec[16:19].copy()
    def m_q(self): return self._rec[0:4].copy()
    def m_balin(self): return self._lin[3:6].copy()
    def m_bglin(self): return self._lin[0:3].copy()
    def gravity(self): return self._lin[10:13].copy()
    def key1(self): return self._keys[0]
    def key2(self): return self._keys[1]

    def evaluateError(self, state_i, state_j, H1=False, H2=False):
        """Returns the 15-vector error; with H1/H2 truthy returns (error, H1, H2) with 15x15 arrays (None if not asked)."""
        X = np.stack([state_i.vector(), state_j.vector()])
        e, h1, h2 = factor_eval_host(self.model, X, self._rec[None], self._lin[None], want_H1=bool(H1), want_H2=bool(H2))
        if not (H1 or H2):
            return e[0]
        return (e[0], h1[0].reshape(15, 15, order="F") if H1 else None, h2[0].reshape(15, 15, order="F") if H2 else None)

    def equals(self, other, tol=1e-9):
        return type(other) is type(self) and self._keys == other._keys and bool(
            np.all(np.abs(self._rec - other._rec) <= tol) and np.all(np.abs(self._lin - other._lin) <= tol))


class ImuFactorCPIv1(_ImuFactorCPI):
    """gtsam/ImuFactorCPIv1.h:78-82 -- argument order kept (note J_beta before J_alpha, H_beta before H_alpha)."""
    model = 1

    def __init__(self, state_i, state_j, covariance, deltatime, grav, alpha, beta, q_KtoK1, ba_lin, bg_lin, J_q, J_beta, J_alpha,
                 H_beta, H_alpha):
        self._keys = (state_i, state_j)
        self._pack(covariance, deltatime, grav, alpha, beta, q_KtoK1, np.array([0, 0, 0, 1.0]), ba_lin, bg_lin, J_q, J_beta, J_alpha,
                   H_beta, H_alpha)


class ImuFactorCPIv2(_ImuFactorCPI):
    """gtsam/ImuFactorCPIv2.h:82-86 (adds q_K_lin, O_beta, O_alpha)."""
    model = 2

    def __init__(self, state_i, state_j, covariance, deltatime, grav, alpha, beta, q_KtoK1, q_K_lin, ba_lin, bg_lin, J_q, J_beta,
                 J_alpha, H_beta, H_alpha, O_beta, O_alpha):
        self._keys = (state_i, state_j)
        self._pack(covariance, deltatime, grav, alpha, beta, q_KtoK1, q_K_lin, ba_lin, bg_lin, J_q, J_beta, J_alpha, H_beta, H_alpha,
                   O_beta, O_alpha)

    def m_qklin(self): return self._lin[6:10].copy()
