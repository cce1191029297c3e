"""Extended-precision gate of the filter's measurement update (cpi_state_update_batch, kernel K10; DESIGN.md section 3k).

The truth is tests/update_oracle.c in long double, square-root order.  Errors are taken per filter: every 3x3 block pair of Sigma+ (in
units of sqrt(truth_ii truth_jj)), every component of x+ in retract coordinates (local(x+_true, x+) in the truth's posterior standard
deviations) and gamma (relative to max(gamma, 1)).  They are gated within every group of the stress batch (one tag: one kind of fix
and residual against every covariance), as tests/parity.py gates per row: e_64 is the larger worst fp64 error in the group of the
oracle's two orders, the square-root form and the information form (Sigma^-1 + W)^-1, and every filter must satisfy
    e_dev <= 8 max(e_64, floor, 1e-15).
floor is zero except for x+, where it is one ulp of the stored component of x+ (the quaternion: 2^-52 rad) in the same units: x+ is
x + xi rounded to fp64, so an xi that differs from the oracle's in its last bits (the kernel contracts to fma, the oracle is built
with -ffp-contract=off) moves x+ by one ulp, and no fp64 route can do better than half of one.

Excluded on purpose: fixes with lambda_max(W Sigma) > SHARPEST = 1e12 (tests/update_ref.py).  The square-root form's C = I + L^T W L
has that condition number; beyond it the fp64 forms lose digits in proportion and near 1e17 the Cholesky of C fails (DESIGN.md
section 3k).  W entries of 1e16 stay in the batch, against covariances tight enough to keep lambda_max below the limit."""
from __future__ import annotations

import numpy as np
import pytest

import update_ref as ur

K, FLOOR = 8.0, 1e-15


def _errors(truth, got, x):
    eb, ex, eg = ur.errors(truth, got, x)
    return np.concatenate([eb.reshape(len(eb), -1), ex, eg[:, None]], axis=1)


def _floor(truth):
    """[n, 41]: one ulp of the stored x+ per component, in the truth's posterior standard deviations (0 for Sigma+ and gamma)."""
    tx, tc, _ = truth
    sd = np.sqrt(np.abs(np.diagonal(ur.mat(tc), axis1=1, axis2=2)))
    ulp = np.concatenate([np.full((len(tx), 3), 2.0 ** -52), np.spacing(np.abs(tx[:, 4:16]))], axis=1)
    return np.concatenate([np.zeros((len(tx), 25)), ulp / sd, np.zeros((len(tx), 1))], axis=1)


def _names():
    blk = "att bg v ba p".split()
    return [f"cov[{a},{b}]" for a in blk for b in blk] + [f"x+[{k}]" for k in range(15)] + ["gamma"]


def gate(b, got):
    """(worst ratio e_dev / (K max(e_64, floor, FLOOR)) over the filters and categories, its group and category, that filter's error
    in ulps of the floor where it has one) of got = (x+, cov+, gamma) on the batch b; truth and e_64 from the oracle."""
    x, cov, W, xb = b["x"], b["cov"], b["W"], b["xb"]
    tx, tc, _, tg = ur.oracle_update(x, cov, W, xb, 0, long_double=True)
    truth = (tx, tc, tg)
    ok = np.isfinite(tg) & np.all(np.isfinite(tc), axis=1)
    assert ok.all(), f"the truth is not finite for {int((~ok).sum())} filters"
    fl = _floor(truth)
    e64 = np.zeros_like(fl)
    for order in (0, 1):
        o = ur.oracle_update(x, cov, W, xb, order)
        e = _errors(truth, (o[0], o[1], o[3]), x)
        assert np.all(np.isfinite(e)), f"fp64 order {order} is not finite on the batch"
        for t in np.unique(b["tag"]):
            g = b["tag"] == t
            e64[g] = np.maximum(e64[g], e[g].max(axis=0))
    ed = _errors(truth, got, x)
    r = np.where(np.isnan(ed), np.inf, ed / (K * np.maximum(np.maximum(e64, fl), FLOOR)))
    i, j = np.unravel_index(int(np.argmax(r)), r.shape)
    ulps = float(ed[i, j] / fl[i, j]) if fl[i, j] > 0 else None
    return float(r[i, j]), f"{b['tag'][i]} {_names()[j]}", ulps


def _batch():
    return ur.stress_batch(np.random.default_rng(20261017))


def test_long_double_orders_agree_and_cover_the_branches():
    """The two long-double orders agree where the information matrix Sigma^-1 + W is well enough conditioned for the information
    form in long double (condition number below 1e6: to 1e-7), and the batch takes every quaternion branch of local15.  Beyond that
    only the square-root order is a truth: the information form loses digits with the condition number, in long double as in fp64."""
    import chain_stress
    b = _batch()
    a = ur.oracle_update(b["x"], b["cov"], b["W"], b["xb"], 0, long_double=True)
    c = ur.oracle_update(b["x"], b["cov"], b["W"], b["xb"], 1, long_double=True)
    eb, ex, eg = ur.errors((a[0], a[1], a[3]), (c[0], c[1], c[3]), b["x"])
    kappa = np.linalg.cond(np.linalg.inv(ur.mat(b["cov"])) + ur.mat(b["W"]))
    ok = kappa < 1e6
    worst = max(eb.reshape(len(eb), -1)[ok].max(), ex[ok].max(), eg[ok].max())
    print(f"long double orders on {int(ok.sum())} of {len(ok)} filters with condition < 1e6: worst {worst:.1e}; "
          f"over all: cov {eb.max():.1e}, x+ {ex.max():.1e}, gamma {eg.max():.1e}")
    assert ok.sum() > len(ok) // 4 and worst <= 1e-7
    sel = np.char.startswith(b["tag"], "branch/")
    flip, same, s0 = chain_stress.local_branches(b["xb"][sel], b["x"][sel])
    assert flip.any() and (~flip).any() and same.any() and s0.any()


def test_gate_passes_fp64_and_fails_injected_errors():
    """Both fp64 orders pass the gate; it fails Sigma+ of one filter rounded to fp32, one position of x+ moved by 1e-5 posterior
    standard deviations, and one gamma scaled by 1 + 1e-7 (one filter of the group of well-conditioned 1 cm full fixes)."""
    b = _batch()
    for order in (0, 1):
        o = ur.oracle_update(b["x"], b["cov"], b["W"], b["xb"], order)
        r, name, _ = gate(b, (o[0], o[1], o[3]))
        print(f"fp64 order {order}: worst ratio {r:.2f} ({name})")
        assert r <= 1.0
    o = ur.oracle_update(b["x"], b["cov"], b["W"], b["xb"], 0)
    i = int(np.flatnonzero(b["tag"] == "full@0.01/near")[0])
    c = o[1].copy(); c[i] = c[i].astype(np.float32).astype(np.float64)
    assert gate(b, (o[0], c, o[3]))[0] > 1.0
    x = o[0].copy(); x[i, 13] += 1e-5 * np.sqrt(ur.mat(o[1][i:i + 1])[0, 12, 12])
    assert gate(b, (x, o[1], o[3]))[0] > 1.0
    g = o[3].copy(); g[i] *= 1 + 1e-7
    assert gate(b, (o[0], o[1], g))[0] > 1.0


@pytest.mark.gpu
def test_kernel_against_extended_precision(cuda):
    """The stress batch plus covariances of K7 chains dead-reckoned for 600 keyframes (both models; position blocks up to ~1e5, bias
    blocks down to ~1e-9): every filter of the kernel passes the gate in every category."""
    from test_update import _k7_covariances, _run
    torch = cuda
    extra = []
    for model in (1, 2):
        covs, _ = _k7_covariances(torch, model, 4, 600, 40 + model)
        extra.append(covs[[49, 199, 599]].reshape(-1, 225))
        S = ur.mat(covs[599])
        print(f"model {model}: K7 covariance after 600 keyframes, diagonal {np.diagonal(S, axis1=1, axis2=2).min():.1e} .. "
              f"{np.diagonal(S, axis1=1, axis2=2).max():.1e}")
    b = ur.stress_batch(np.random.default_rng(20261017), extra_cov=np.concatenate(extra))
    got = _run(torch, b["x"], b["cov"], b["W"], b["xb"])
    assert np.all(got[3] == 1)
    r, name, ulps = gate(b, (got[0], got[1], got[2]))
    print(f"kernel on {len(b['x'])} filters: worst ratio to the bound {r:.2f} ({name})"
          + ("" if ulps is None else f", {ulps:.2f} ulp of the stored x+"))
    assert r <= 1.0, (name, r)
