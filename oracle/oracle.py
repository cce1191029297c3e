"""TEST INFRASTRUCTURE ONLY: ctypes loaders for the CPU checkers.

  * ``Oracle()``    -> oracle/liboracle.so       (plain-C restatement, oracle/cpi_oracle.c)
  * ``OracleLD()``  -> oracle/liboracle_ld.so    (the same source in long double arithmetic)
  * ``Reference()`` -> oracle/_ref/libcpi_ref.so (the UNMODIFIED reference compiled in place by oracle/ref_shim.cpp;
                       built only where an rpng/cpi checkout is given: make -C oracle ref REF=...)

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / ``--impl reference`` leg may import this module.
The product package ``cpi_b200`` never does.  Both classes expose the same numpy-level methods.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_P = ctypes.POINTER(ctypes.c_double)
_PI = ctypes.POINTER(ctypes.c_int64)

REC_DOUBLES = {1: 290, 2: 308}
FLAG_IMU_AVG = 1
FLAG_ANALYTIC_JACOBIANS = 2


def build(force: bool = False) -> None:
    """Compile liboracle.so (always possible) and _ref/libcpi_ref.so (only if the reference tree is present)."""
    args = ["make", "-C", _HERE, "-s"]
    if force:
        args.append("-B")
    subprocess.run(args + ["liboracle.so"], check=True)
    subprocess.run(args + ["ref"], check=True)


def _d(a):
    return a.ctypes.data_as(_P)


def _i(a):
    return None if a is None else a.ctypes.data_as(_PI)


class _Base:
    prefix = ""
    path = ""

    def __init__(self):
        if not os.path.exists(self.path):
            raise FileNotFoundError(self.path)
        self.lib = ctypes.CDLL(self.path)
        f = getattr(self.lib, self.prefix + "cpi_preintegrate")
        f.argtypes = [ctypes.c_int, ctypes.c_int64, _PI, ctypes.c_int64, _P, _P, _P, ctypes.c_int, _P, ctypes.c_int]
        f.restype = ctypes.c_int
        self._pre = f
        f = getattr(self.lib, self.prefix + "imu_factor_eval")
        f.argtypes = [ctypes.c_int, ctypes.c_int64, _P, _PI, _PI, _P, _P, _P, _P, _P, ctypes.c_int]
        f.restype = ctypes.c_int
        self._fac = f
        f = getattr(self.lib, self.prefix + "retract")
        f.argtypes = [ctypes.c_int64, _P, _P, _P]
        self._ret = f
        for name, n_in in (("rot_2_quat", 1), ("quat_2_Rot", 1), ("quat_multiply", 2), ("Exp", 1)):
            g = getattr(self.lib, self.prefix + name)
            g.argtypes = [_P] * (n_in + 1)
            g.restype = None

    # ---- batch entry points (same meaning as include/cpi_b200.h, host numpy arrays) ----
    def preintegrate(self, model, samples, lin, sigmas, flags=0, offsets=None, ns=None, nthreads=1):
        samples = np.ascontiguousarray(samples, dtype=np.float64).reshape(-1, 7)
        lin = np.ascontiguousarray(lin, dtype=np.float64).reshape(-1, 13)
        sigmas = np.ascontiguousarray(sigmas, dtype=np.float64)
        n = lin.shape[0]
        if offsets is not None:
            offsets = np.ascontiguousarray(offsets, dtype=np.int64)
            assert offsets.shape[0] == n + 1
            ns = 0
        else:
            extra = 1 if flags & FLAG_IMU_AVG else 0
            if ns is None:
                ns = samples.shape[0] // max(n, 1) - extra
            assert samples.shape[0] >= n * (ns + extra)
        out = np.zeros((n, REC_DOUBLES[model]))
        rc = self._pre(model, n, _i(offsets), int(ns), _d(samples), _d(lin), _d(sigmas), int(flags), _d(out), int(nthreads))
        assert rc == 0
        return out

    def factor_eval(self, model, states, records, lin, idx_i=None, idx_j=None, nthreads=1):
        states = np.ascontiguousarray(states, dtype=np.float64).reshape(-1, 16)
        records = np.ascontiguousarray(records, dtype=np.float64).reshape(-1, REC_DOUBLES[model])
        lin = np.ascontiguousarray(lin, dtype=np.float64).reshape(-1, 13)
        n = records.shape[0]
        if idx_i is not None:
            idx_i = np.ascontiguousarray(idx_i, dtype=np.int64)
            idx_j = np.ascontiguousarray(idx_j, dtype=np.int64)
        e = np.zeros((n, 15)); H1 = np.zeros((n, 225)); H2 = np.zeros((n, 225))
        rc = self._fac(model, n, _d(states), _i(idx_i), _i(idx_j), _d(records), _d(lin), _d(e), _d(H1), _d(H2), int(nthreads))
        assert rc == 0
        return e, H1, H2

    def retract(self, states, xi):
        states = np.ascontiguousarray(states, dtype=np.float64).reshape(-1, 16)
        xi = np.ascontiguousarray(xi, dtype=np.float64).reshape(-1, 15)
        out = np.zeros_like(states)
        self._ret(states.shape[0], _d(states), _d(xi), _d(out))
        return out

    # ---- quat_ops helpers (3x3 as column-major flat [9]) ----
    def _call(self, name, nout, *ins):
        ins = [np.ascontiguousarray(a, dtype=np.float64) for a in ins]
        out = np.zeros(nout)
        getattr(self.lib, self.prefix + name)(*[_d(a) for a in ins], _d(out))
        return out

    def rot_2_quat(self, R): return self._call("rot_2_quat", 4, R)
    def quat_2_Rot(self, q): return self._call("quat_2_Rot", 9, q)
    def quat_multiply(self, q, p): return self._call("quat_multiply", 4, q, p)
    def Exp(self, w): return self._call("Exp", 9, w)


class Oracle(_Base):
    prefix = "oracle_"
    path = os.path.join(_HERE, "liboracle.so")

    def __init__(self):
        super().__init__()
        f = self.lib.oracle_predict_state
        f.argtypes = [ctypes.c_int, ctypes.c_int64, _P, _P, _P, _P]
        self._pred = f

    def predict_state(self, model, states_k, records, lin):
        states_k = np.ascontiguousarray(states_k, dtype=np.float64).reshape(-1, 16)
        records = np.ascontiguousarray(records, dtype=np.float64).reshape(-1, REC_DOUBLES[model])
        lin = np.ascontiguousarray(lin, dtype=np.float64).reshape(-1, 13)
        out = np.zeros_like(states_k)
        self._pred(model, states_k.shape[0], _d(states_k), _d(records), _d(lin), _d(out))
        return out

    # ---- model-1 record composition (merge / scan).  Bound on first use, so that a library built before these entry points
    # existed still serves everything above.
    def _rec_fn(self, name, argtypes):
        f = getattr(self.lib, name, None)
        if f is None:
            # dlopen hands back the image this process already mapped for the same path, even after a rebuild: load the file
            # on disk under another name if it has the symbol
            import shutil
            import tempfile
            tmp = os.path.join(tempfile.mkdtemp(prefix="cpi_oracle_"), os.path.basename(self.path))
            shutil.copyfile(self.path, tmp)
            lib = ctypes.CDLL(tmp)
            f = getattr(lib, name, None)
            if f is None:
                raise AttributeError(f"{self.path} has no {name}: rebuild it (make -C oracle)")
            self.lib = lib
        f.argtypes = argtypes
        f.restype = ctypes.c_int
        return f

    @staticmethod
    def _groups(n_rec, group_offsets, group):
        if group_offsets is not None:
            offs = np.ascontiguousarray(group_offsets, dtype=np.int64)
            assert offs.ndim == 1 and offs.shape[0] >= 1 and offs[-1] <= n_rec
            return offs.shape[0] - 1, offs, 0
        assert group is not None and group >= 1 and n_rec % group == 0
        return n_rec // group, None, int(group)

    def merge_pair(self, a, b, nthreads=1):
        """out[i] = a[i] (+) b[i]: two consecutive model-1 records at one linearisation point."""
        f = self._rec_fn("oracle_merge_pair", [ctypes.c_int64, _P, _P, _P, ctypes.c_int])
        a = np.ascontiguousarray(a, dtype=np.float64).reshape(-1, REC_DOUBLES[1])
        b = np.ascontiguousarray(b, dtype=np.float64).reshape(-1, REC_DOUBLES[1])
        assert a.shape == b.shape
        out = np.zeros_like(a)
        assert f(a.shape[0], _d(a), _d(b), _d(out), int(nthreads)) == 0
        return out

    def relinearise(self, records, lin, lin0):
        """records[i], preintegrated at lin[i], moved to lin0[i] to first order (q, Jacobians and P unchanged)."""
        f = self._rec_fn("oracle_relinearise_records", [ctypes.c_int64, _P, _P, _P, _P])
        records = np.ascontiguousarray(records, dtype=np.float64).reshape(-1, REC_DOUBLES[1])
        lin = np.ascontiguousarray(lin, dtype=np.float64).reshape(-1, 13)
        lin0 = np.ascontiguousarray(lin0, dtype=np.float64).reshape(-1, 13)
        out = np.zeros_like(records)
        assert f(records.shape[0], _d(records), _d(lin), _d(lin0), _d(out)) == 0
        return out

    def _fold(self, name, records, lin, group_offsets, group, nthreads, scan):
        f = self._rec_fn(name, [ctypes.c_int64, _PI, ctypes.c_int64, _P, _P, _P, ctypes.c_int])
        records = np.ascontiguousarray(records, dtype=np.float64).reshape(-1, REC_DOUBLES[1])
        lin = np.ascontiguousarray(lin, dtype=np.float64).reshape(-1, 13)
        assert lin.shape[0] == records.shape[0]
        n, offs, uniform = self._groups(records.shape[0], group_offsets, group)
        out = np.zeros_like(records) if scan else np.zeros((n, REC_DOUBLES[1]))
        assert f(n, _i(offs), uniform, _d(records), _d(lin), _d(out), int(nthreads)) == 0
        return out

    def merge_records(self, records, lin, group_offsets=None, group=None, nthreads=1):
        """The left fold of every group (layout as cpi_merge_records_host): one record per group."""
        return self._fold("oracle_merge_records", records, lin, group_offsets, group, nthreads, False)

    def scan_records(self, records, lin, group_offsets=None, group=None, nthreads=1):
        """Every prefix of the left fold of every group (layout as cpi_scan_records_host); rows outside every group are zero."""
        return self._fold("oracle_scan_records", records, lin, group_offsets, group, nthreads, True)

    # ---- the solver side of a chain (K8, k_prior_at, the block-tridiagonal solve, the LM model decrease).  Layouts as
    # include/cpi_b200.h: chain_offsets [n_chains+1] int64, or chains of `uniform` states with n_chains given.
    @staticmethod
    def _chains(chain_offsets, uniform, n_chains):
        if chain_offsets is not None:
            offs = np.ascontiguousarray(chain_offsets, dtype=np.int64)
            return offs.shape[0] - 1, offs, 0, int(offs[-1])
        assert uniform is not None and uniform >= 1 and n_chains is not None
        return int(n_chains), None, int(uniform), int(n_chains) * int(uniform)

    def chain_marginalize(self, G11, G12, G22, g1, g2, f, n_marg, prior=None, chain_offsets=None, uniform=None, n_chains=None, nthreads=1):
        """K8's recurrence per chain: returns (info [C,225], rhs [C,15], f [C], scale [C,242]) -- scale: the size of the terms that cancel
        into info and rhs in the last step, of f over all steps, and the last step's z^T z.  n_marg: int or [C] int64."""
        fn = self._rec_fn("oracle_chain_marginalize", [ctypes.c_int64, _PI, ctypes.c_int64, _PI, ctypes.c_int64] + [_P] * 12 + [_P, ctypes.c_int])
        C, offs, u, _ = self._chains(chain_offsets, uniform, n_chains)
        blk = [np.ascontiguousarray(a, dtype=np.float64) for a in (G11, G12, G22, g1, g2, f)]
        nm, nmu = (None, int(n_marg)) if np.isscalar(n_marg) else (np.ascontiguousarray(n_marg, dtype=np.int64), 0)
        pr = [None] * 3 if prior is None else [np.ascontiguousarray(a, dtype=np.float64) for a in prior]
        oi, orr, of, sc = np.zeros((C, 225)), np.zeros((C, 15)), np.zeros(C), np.zeros((C, 242))
        dp = lambda a: None if a is None else _d(a)
        assert fn(C, _i(offs), u, _i(nm), nmu, *[_d(a) for a in blk], *[dp(a) for a in pr], _d(oi), _d(orr), _d(of), _d(sc), int(nthreads)) == 0
        return oi, orr, of, sc

    def chain_solve(self, D, E, b, order, chain_offsets=None, uniform=None, n_chains=None, nthreads=1):
        """x [N,15] of tridiag(E^T, D, E) x = b: order 0 sequential block Cholesky per chain, 1 the block cyclic reduction of solve.cu."""
        fn = self._rec_fn("oracle_chain_solve", [ctypes.c_int64, _PI, ctypes.c_int64, _P, _P, _P, _P, ctypes.c_int, ctypes.c_int])
        C, offs, u, N = self._chains(chain_offsets, uniform, n_chains)
        D = np.ascontiguousarray(D, dtype=np.float64).reshape(N, 225)
        E = np.ascontiguousarray(E, dtype=np.float64).reshape(-1, 225)
        if E.shape[0] < max(N - 1, 1):
            E = np.concatenate([E, np.zeros((max(N - 1, 1) - E.shape[0], 225))])
        b = np.ascontiguousarray(b, dtype=np.float64).reshape(N, 15)
        x = np.zeros((N, 15))
        assert fn(C, _i(offs), u, _d(D), _d(E), _d(b), _d(x), int(order), int(nthreads)) == 0
        return x

    def chain_marginals(self, D, E, order, chain_offsets=None, uniform=None, n_chains=None, nthreads=1):
        """(cov [N,225], cross [N-C,225]): Sigma_kk of every state and Sigma_{k,k+1} of every pair of neighbours in a chain (slot k - c,
        as cpi_imu_chains_marginals) of tridiag(E^T, D, E): order 0 a sequential block Cholesky and backward recurrence per chain, 1 the
        isolated block cyclic reduction and level walk of solve.cu.  NaN for a chain with a pivot that is not positive."""
        fn = self._rec_fn("oracle_chain_marginals", [ctypes.c_int64, _PI, ctypes.c_int64, _P, _P, _P, _P, ctypes.c_int, ctypes.c_int])
        C, offs, u, N = self._chains(chain_offsets, uniform, n_chains)
        D = np.ascontiguousarray(D, dtype=np.float64).reshape(N, 225)
        E = np.ascontiguousarray(E, dtype=np.float64).reshape(-1, 225)
        if E.shape[0] < max(N - 1, 1):
            E = np.concatenate([E, np.zeros((max(N - 1, 1) - E.shape[0], 225))])
        cov, cross = np.zeros((N, 225)), np.zeros((max(N - C, 0), 225))
        assert fn(C, _i(offs), u, _d(D), _d(E), _d(cov), _d(cross) if len(cross) else None, int(order), int(nthreads)) == 0
        return cov, cross

    def lm_terms(self, rhs, D, E, damp, delta, f_cur, f_new, pf_cur=None, pf_new=None, chain_offsets=None, uniform=None, n_chains=None, nthreads=1):
        """Per chain [C,5]: (model decrease m, sum |delta|^T (2|rhs| + |H||delta|), current cost, candidate cost, delta != 0)."""
        fn = self._rec_fn("oracle_lm_terms", [ctypes.c_int64, _PI, ctypes.c_int64] + [_P] * 10 + [ctypes.c_int])
        C, offs, u, N = self._chains(chain_offsets, uniform, n_chains)
        a = [np.ascontiguousarray(x, dtype=np.float64) for x in (rhs, D, E, damp, delta, f_cur)]
        pc = None if pf_cur is None else np.ascontiguousarray(pf_cur, dtype=np.float64)
        fnw = np.ascontiguousarray(f_new, dtype=np.float64)
        pn = None if pf_new is None else np.ascontiguousarray(pf_new, dtype=np.float64)
        dp = lambda x: None if x is None else _d(x)
        out = np.zeros((C, 5))
        assert fn(C, _i(offs), u, *[_d(x) for x in a], dp(pc), _d(fnw), dp(pn), _d(out), int(nthreads)) == 0
        return out

    # ---- K7, the covariance propagation (DESIGN.md 3d)
    def propagate(self, model, states_k, cov_k, records, lin, order=0, anchor=None, want_cross=True, nthreads=1):
        """(x_k1 [n,16], cov_k1 [n,225], cross [n,225] or None) of cpi_propagate_batch_host: order 0 the dense statement (a pivoted
        inverse of H2, dense products), 1 the sparse route of propagate.cu."""
        fn = self._rec_fn("oracle_propagate", [ctypes.c_int, ctypes.c_int64, _P, _P, _PI, _P, _P, ctypes.c_int, _P, _P, _P, ctypes.c_int])
        X = np.ascontiguousarray(states_k, dtype=np.float64).reshape(-1, 16)
        S = np.ascontiguousarray(cov_k, dtype=np.float64).reshape(-1, 225)
        rec = np.ascontiguousarray(records, dtype=np.float64).reshape(-1, REC_DOUBLES[model])
        lin = np.ascontiguousarray(lin, dtype=np.float64).reshape(-1, 13)
        n = rec.shape[0]
        an = np.arange(n, dtype=np.int64) if anchor is None else np.ascontiguousarray(anchor, dtype=np.int64)
        assert an.shape == (n,) and lin.shape[0] == n and (n == 0 or (an.min() >= 0 and an.max() < len(X) and len(S) == len(X)))
        x1, c1 = np.zeros((n, 16)), np.zeros((n, 225))
        cr = np.zeros((n, 225)) if want_cross else None

        assert fn(model, n, _d(X), _d(S), _i(an), _d(rec), _d(lin), int(order), _d(x1), _d(c1), None if cr is None else _d(cr),
                  int(nthreads)) == 0
        return x1, c1, cr

    def propagate_chain(self, model, states0, cov0, records, lin, steps, order=0, path=None, nthreads=1):
        """(x [C,16], cov [C,225]) after `steps` windows of K7 per chain (records / lin chain-major [C * steps]), held in working
        precision between steps; path [C * (steps + 1), 16]: the states each step starts from (default: the statement's own)."""
        fn = self._rec_fn("oracle_propagate_chain", [ctypes.c_int, ctypes.c_int64, ctypes.c_int64, _P, _P, _P, _P, _P, ctypes.c_int,
                                                      _P, _P, ctypes.c_int])
        X = np.ascontiguousarray(states0, dtype=np.float64).reshape(-1, 16)
        S = np.ascontiguousarray(cov0, dtype=np.float64).reshape(-1, 225)
        C = X.shape[0]
        rec = np.ascontiguousarray(records, dtype=np.float64).reshape(C, steps, REC_DOUBLES[model])
        lin = np.ascontiguousarray(lin, dtype=np.float64).reshape(C, steps, 13)
        pth = None if path is None else np.ascontiguousarray(path, dtype=np.float64).reshape(C, steps + 1, 16)
        xo, co = np.zeros((C, 16)), np.zeros((C, 225))

        assert fn(model, C, int(steps), _d(X), _d(S), None if pth is None else _d(pth), _d(rec), _d(lin), int(order), _d(xo), _d(co),
                  int(nthreads)) == 0
        return xo, co

    def local(self, lin, x):
        """local(x_lin, x) [n,15], the inverse of retract."""
        fn = self._rec_fn("oracle_local", [ctypes.c_int64, _P, _P, _P])
        lin = np.ascontiguousarray(lin, dtype=np.float64).reshape(-1, 16)
        x = np.ascontiguousarray(x, dtype=np.float64).reshape(-1, 16)
        d = np.zeros((lin.shape[0], 15))
        assert fn(lin.shape[0], _d(lin), _d(x), _d(d)) == 0
        return d

    def prior_at(self, info, rhs, f, lin, x):
        """cpi_imu_prior_at: (rhs' [n,15], f' [n])."""
        fn = self._rec_fn("oracle_prior_at", [ctypes.c_int64] + [_P] * 7)
        info = np.ascontiguousarray(info, dtype=np.float64).reshape(-1, 225)
        n = info.shape[0]
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (rhs, f, lin, x)]
        ro, fo = np.zeros((n, 15)), np.zeros(n)
        assert fn(n, _d(info), *[_d(v) for v in a], _d(ro), _d(fo)) == 0
        return ro, fo


class OracleLD(Oracle):
    """The same restatement computed in long double (oracle/liboracle_ld.so): double in, double out, about 1e-19 working
    precision on x86-64.  The truth of the precision tests; its small_w / dt == 0 branches follow the fp64 code."""
    path = os.path.join(_HERE, "liboracle_ld.so")


class Reference(_Base):
    prefix = "ref_"
    path = os.path.join(_HERE, "_ref", "libcpi_ref.so")

    @classmethod
    def available(cls) -> bool:
        return os.path.exists(cls.path)

    def replay_run(self, model, t, w, a, cam_t, lin, sigmas, flags=0, imu_wait=0):
        """ref_replay_run (oracle/ref_shim.cpp): the reference DRIVER over one dataset run with its own deque handling.
        Returns (samples fed [total,7], offsets[nwin+1], records[nwin, rd])."""
        f = self.lib.ref_replay_run
        f.argtypes = [ctypes.c_int, ctypes.c_int64, _P, _P, _P, ctypes.c_int64, _P, ctypes.c_int64, _P, _P, ctypes.c_int, ctypes.c_int64, _P, _PI, _P]
        f.restype = ctypes.c_int64
        t = np.ascontiguousarray(t, dtype=np.float64); w = np.ascontiguousarray(w, dtype=np.float64); a = np.ascontiguousarray(a, dtype=np.float64)
        cam_t = np.ascontiguousarray(cam_t, dtype=np.float64); lin = np.ascontiguousarray(lin, dtype=np.float64)
        sig = np.ascontiguousarray(sigmas, dtype=np.float64)
        rd = 290 if model == 1 else 308
        cap = len(t) + len(cam_t) + 1
        S = np.zeros((cap, 7)); off = np.zeros(len(cam_t) + 1, dtype=np.int64); rec = np.zeros((len(cam_t), rd))
        assert lin.shape[0] >= len(cam_t)
        nw = f(model, len(t), _d(t), _d(w), _d(a), len(cam_t), _d(cam_t), int(imu_wait), _d(lin), _d(sig), flags, cap, _d(S), _i(off), _d(rec))
        if nw < 0:
            raise RuntimeError("ref_replay_run failed")
        return S[:off[nw]].copy(), off[:nw + 1].copy(), rec[:nw].copy()

    def hardware_threads(self) -> int:
        return int(self.lib.ref_hardware_threads())
