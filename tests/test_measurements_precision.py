"""Extended-precision gate of the measurement linearisation (cpi_imu_measurements_linearize, K12; DESIGN.md section 3l), the filter's
update by measurements (cpi_state_update_measurements_batch, K11) and the iterated update with robust losses
(cpi_state_update_measurements_iterated_batch, K13; section 3m), on the measurement stress batch of tests/measurement_stress.py.

The truth is tests/update_oracle.c in long double, square-root order (K12: order 0, A = S H).  K11 and K13 are measured as K10 is in
tests/test_update_precision.py: errors per filter of every 3x3 block pair of Sigma+, every component of x+ in the truth's posterior
standard deviations and gamma relative to max(gamma, 1); e_64 the larger worst error in the group (tag) of the oracle's two fp64 orders,
the square-root form and the information form, for K11 and K13 each built without and with fma contraction; every filter satisfies e_dev <= 8 max(e_64, floor, 1e-15) with the one-ulp floor on
x+.  K12 is measured per measurement in units of the scale each field is formed at (info against its largest entry, f' against
(|S| (|h| + |z|))^2, rhs' against the geometric mean: r = h - z is formed at the scale of |h| + |z|); e_64 of the two fp64 orders
(A^T A and H^T (S^T S) H), pooled over the entries of each field: where z = h the fp64 r is zero in some components by luck, and a
per-entry e_64 would then be far below the rounding of r.  Its floor is one ulp of the stored truth in the same units, not 1e-15: the units are the first-order
rounding bound of r, so 1e-15 of them is about ten ulps of the largest term and would hide an r formed as S h - S z.

The contracted builds are in e_64 for K11 and K13 because the kernels contract to fma and the two uncontracted orders do not span
the rounding that follows: on this batch the contracted order-0 build of the same C lies up to 12x (Sigma+ of K13) and 4x (gamma
of K11) beyond 8 e_64 of the uncontracted orders, in groups that the kernels also exceed by similar factors.  They are the plain-C
statement with the kernels' kind of rounding, not their order of operations.  e_64 is pooled over the block pairs of Sigma+ (and
the components of each block of x+): entries that the update shrinks by its sharpness lambda carry a relative error near eps lambda
on every route, and which pair that cancellation lands in differs from route to route (a 1024-long list of 300 m/s body velocities
puts 1e-9 into one pair on one route and another pair on the next).  gamma has a floor too: what one ulp of h moves it by
(gamma_floor), as x+ has one ulp of itself.

K13 is compared after the same number of linearisations as the kernel took (the oracle's forced count), so a status that a rounding
flips near the threshold does not change what is compared; status and iterations are compared with the free oracle where its
stopping margin exceeds 1e-6.

Excluded on purpose: filters whose lambda_max(L^T sum_j om_j A_j^T A_j L) exceeds update_ref.SHARPEST at any linearisation the
long-double oracle visits (DESIGN.md section 3k: the fp64 square-root form's limit)."""
from __future__ import annotations

import numpy as np
import pytest

import measurement_ref as mr
import measurement_stress as ms
import update_iter_ref as ir
import update_ref as ur
from test_update_precision import FLOOR, K, _errors, _floor, _names

_CACHE = {}



def _batch():
    if "b" not in _CACHE:
        _CACHE["b"] = ms.stress_batch()
    return _CACHE["b"]


def _args(b):
    return b["x"], b["cov"], b["offsets"], b["kind"], b["z"], b["sqrt_info"], b["aux"]


# ---------------------------------------------------------------------------------------------- the gates

def _per_tag_max(e, tags):
    out = np.zeros_like(e)
    for t in np.unique(tags):
        g = tags == t
        out[g] = e[g].max(axis=0)
    return out


def _group(tags, drop):
    """The gate's groups: the tags (kind/variant/mode/cov/S/state) without their parts at the positions drop."""
    return np.array(["/".join(p for k, p in enumerate(t.split("/")) if k not in drop) for t in tags])


_POOL = np.r_[np.zeros(25, int), 25 + np.repeat(np.arange(5) * 3, 3), 40]          # Sigma+ | x+ per block | gamma


def gamma_floor(b, gamma):
    """[n]: what one ulp of h moves gamma by, relative to max(gamma, 1): 2 eps sum_j |b_j| sb_j at x_hat, sb_j = |S_j| (|h_j| + |z_j|).
    r = h - z is formed in fp64 at the scale of |h| + |z|, and where it cancels (a residual of centimetres on metres) no fp64 route
    can give gamma more digits than that; the uncontracted orders can share one rounding of h and agree with the truth by luck."""
    own = ms.owners(b)
    _, _, bb = mr.meas_ref(b["kind"], b["x"][own], b["z"], b["sqrt_info"], b["aux"])
    t = 2.0 ** -52 * 2 * np.linalg.norm(bb, axis=1) * _k12_units(b)
    return np.bincount(own, weights=np.nan_to_num(t, nan=np.inf, posinf=np.inf), minlength=len(b["x"])) / np.maximum(np.abs(gamma), 1.0)


def e64_filters(tags, x, truth, fp64s, ok):
    """[n, 41]: per filter (zero outside ok) the worst fp64 error of fp64s in its group (its tag without the residual mode), pooled
    over the block pairs of Sigma+ and over the three components of each block of x+."""
    t = tuple(a[ok] for a in truth)
    out = np.zeros((len(ok), 41))
    groups = _group(tags[ok], (2,))
    for o in fp64s:
        e = _errors(t, tuple(a[ok] for a in o), x[ok])
        assert np.all(np.isfinite(e)), "an fp64 order is not finite on the batch"
        e = np.stack([e[:, _POOL == _POOL[c]].max(axis=1) for c in range(41)], axis=1)
        out[ok] = np.maximum(out[ok], _per_tag_max(e, groups))
    return out


def gate_filters(tags, x, truth, fp64s, got, ok, gfloor=None, e64=None):
    """(worst ratio e_dev / (K max(e_64, floor, FLOOR)), its tag and category) over the filters ok of got = (x+, cov+, gamma) against
    truth; e_64 that of e64_filters, or the given [n, 41] e64; gfloor [n] the floor of gamma (gamma_floor)."""
    t = tuple(a[ok] for a in truth)
    fl = _floor(t)
    if gfloor is not None:
        fl[:, -1] = gfloor[ok]
    e64 = (e64_filters(tags, x, truth, fp64s, ok) if e64 is None else e64)[ok]
    ed = _errors(t, tuple(a[ok] for a in got), x[ok])
    r = np.where(np.isnan(ed), np.inf, ed / (K * np.maximum(np.maximum(e64, fl), FLOOR)))
    i, j = np.unravel_index(int(np.argmax(r)), r.shape)
    return float(r[i, j]), f"{tags[ok][i]} {_names()[j]}"


def _k12_units(b):
    """Per measurement sb = |S| (|h| + |z|), the scale r = h - z and b are formed at (_k12_errors forms the scales of the fields)."""
    own = ms.owners(b)
    h = mr.h_of(b["kind"], b["x"][own], b["aux"])
    sb = np.abs(b["sqrt_info"]).max(axis=1) * (np.abs(h).max(axis=1) + np.abs(b["z"]).max(axis=1))
    return sb


def _k12_errors(truth, got, sb):
    info, rhs, f = truth
    sa = np.sqrt(np.abs(info).max(axis=1))
    tiny = np.finfo(np.float64).tiny
    units = [np.maximum(u, tiny)[:, None] for u in (sa * sa, sa * sb, sb * sb)]
    e = np.concatenate([np.abs(g.reshape(len(sb), -1) - w.reshape(len(sb), -1)) / u for g, w, u in zip(got, truth, units)], axis=1)
    fl = np.concatenate([np.spacing(np.abs(w.reshape(len(sb), -1))) / u for w, u in zip(truth, units)], axis=1)
    return e, fl


def gate_k12(b, got, truth=None, fp64s=None):
    """(worst ratio, tag and field) of K12's got = (info, rhs, f) over the batch's measurements."""
    own = ms.owners(b)
    if truth is None:
        truth = ur.oracle_linearize(b["kind"], own, b["x"], b["z"], b["sqrt_info"], b["aux"], 0, long_double=True)
    if fp64s is None:
        fp64s = [ur.oracle_linearize(b["kind"], own, b["x"], b["z"], b["sqrt_info"], b["aux"], o) for o in (0, 1)]
    sb = _k12_units(b)
    tags = _group(b["tag"][own], (2, 3))                                         # K12 reads neither the mode nor Sigma
    fields = np.r_[np.zeros(225, int), np.ones(15, int), 2]
    e64 = None
    for o in fp64s:
        e, fl = _k12_errors(truth, o, sb)
        assert np.all(np.isfinite(e))
        e = np.stack([e[:, fields == k].max(axis=1) for k in range(3)], axis=1)[:, fields]       # pooled over each field's entries
        e64 = _per_tag_max(e, tags) if e64 is None else np.maximum(e64, _per_tag_max(e, tags))
    ed, fl = _k12_errors(truth, got, sb)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(ed == 0, 0.0, np.where(np.isnan(ed), np.inf, ed / (K * np.maximum(e64, fl))))
    i, j = np.unravel_index(int(np.argmax(r)), r.shape)
    field = f"info[{j % 15},{j // 15}]" if j < 225 else (f"rhs[{j - 225}]" if j < 240 else "f")
    return float(r[i, j]), f"{tags[i]} {field}"


def k11_reference(b):
    """(truth, [fp64 order 0, order 1, both contracted], ok, gamma floor): the oracle's K11 in long double and fp64, ok the filters
    under SHARPEST with a finite truth."""
    a = _args(b)
    t = ur.oracle_update_meas(*a, 0, long_double=True)
    f = [ur.oracle_update_meas(*a, o, contract=c) for c in (False, True) for o in (0, 1)]
    ok = t[3] <= ur.SHARPEST
    bad = ok & ~(np.isfinite(t[2]) & np.all(np.isfinite(t[1]), axis=1) & np.all(np.isfinite(t[0]), axis=1))
    assert not bad.any(), f"the truth is not finite for {int(bad.sum())} filters under SHARPEST"
    return (t[0], t[1], t[2]), [(o[0], o[1], o[2]) for o in f], ok, gamma_floor(b, t[2])


def k13_reference(b, force, max_iterations, tol, gate=None):
    """As k11_reference, and the long-double outputs, for K13 forced to `force` linearisations per filter; ok also needs every
    visited linearisation under SHARPEST."""
    a = _args(b)
    kw = dict(loss=b["loss"], loss_k=b["loss_k"], gate=gate, max_iterations=max_iterations, tol=tol, force=force)
    t = ur.oracle_update_iter(*a, 0, long_double=True, **kw)
    f = [ur.oracle_update_iter(*a, o, contract=c, **kw) for c in (False, True) for o in (0, 1)]
    ok = t[7] <= ur.SHARPEST
    bad = ok & ~(np.isfinite(t[2]) & np.all(np.isfinite(t[1]), axis=1) & np.all(np.isfinite(t[0]), axis=1))
    assert not bad.any(), f"the truth is not finite for {int(bad.sum())} filters under SHARPEST"
    return (t[0], t[1], t[2]), [(o[0], o[1], o[2]) for o in f], ok, gamma_floor(b, t[2]), t


def _numpy_style_catches(truth, fp64s, got, x, ok):
    """Whether the criterion of the existing statement tests rejects got: its error against the fp64 square-root statement above
    20 max(the distance between the fp64 square-root and information statements, 1e-13), over the whole batch."""
    r0 = tuple(a[ok] for a in fp64s[0])
    eb, ex, eg = ur.errors(r0, tuple(a[ok] for a in got), x[ok])
    nb, nx, ng = ur.errors(r0, tuple(a[ok] for a in fp64s[1]), x[ok])
    return not (eb.max() <= 20 * max(nb.max(), 1e-13) and ex.max() <= 20 * max(nx.max(), 1e-13) and eg.max() <= 20 * max(ng.max(), 1e-13))


# ---------------------------------------------------------------------------------------------- CPU

def test_batch_reaches_the_edges():
    """Every list length survives the exclusions in some group, every kind variant and S family is gated, and the edge groups
    (Huber at s = k^2, Cauchy past its overflow) take the branches they are named for."""
    b = _batch()
    ok = k11_reference(b)[2]
    ok13 = k13_reference(b, None, 10, 1e-9)[2]
    for m in ms.LENGTHS + ms.LONG:
        assert (ok & (b["length"] == m)).any() and (ok13 & (b["length"] == m)).any(), m
    for v in ms.VARIANTS:
        assert (ok & np.char.startswith(b["tag"], v)).any(), v
    for fam in ms.S_FAMILIES:
        assert (ok & (b["s_family"] == fam)).any(), fam
    own = ms.owners(b)
    x0 = b["x"][own]
    _, _, bb = mr.meas_ref(b["kind"], x0, b["z"], b["sqrt_info"], b["aux"])
    s = np.einsum("ni,ni->n", bb, bb)
    hub = b["tag"][own] == "edge/huber_s=k2"
    assert np.all(s[hub] == b["loss_k"][hub] ** 2)
    cau = b["tag"][own] == "edge/cauchy_overflow"
    assert np.all(np.isinf(s[cau] / b["loss_k"][cau] ** 2)) and np.all(np.isfinite(s[cau]))
    assert ok13[b["tag"] == "edge/cauchy_overflow"].all() and not ok[b["tag"] == "edge/cauchy_overflow"].any()
    print(f"{len(b['x'])} filters, {len(b['kind'])} measurements; K11 gates {int(ok.sum())}, K13 {int(ok13.sum())}")


def test_weight_matches_the_long_double_loss():
    """update_iter_ref.weight (used by update_iter_ref's statement, stationarity and covariance_at) equals the long-double IRLS weight
    on test_chain_scale.edge_inputs to one ulp, the Cauchy overflow branch (omega = k^2/s, not 0) included."""
    from test_chain_scale import _ulps, edge_inputs, ld_loss
    code, k, s = edge_inputs()
    w = ir.weight(code, k, s)
    for i in range(len(s)):
        wl = np.float64(ld_loss(code[i], k[i], s[i])[0])
        if np.isnan(s[i]):
            continue
        if code[i] == ir.CAUCHY and np.isinf(s[i] / (k[i] * k[i])) and np.isfinite(s[i]):
            wl = np.float64(np.longdouble(k[i] * k[i]) / np.longdouble(s[i]))
            assert w[i] > 0, (k[i], s[i])
        assert w[i] == wl or _ulps(w[i], wl) <= 1.0, (code[i], k[i], s[i], w[i], wl)


def test_long_double_orders_agree_and_cover_the_branches():
    """The two long-double orders of K12, K11 and K13 agree where the problem is well conditioned (K11, K13: condition of
    Sigma^-1 + sum A^T A below 1e6, to 1e-10; K12 to 1e-12 of its scales), and K13's (x_hat, x_lin) pairs take the flip and the
    no-flip branches of local15, the same-bits branch and the s = 0 branch."""
    import chain_stress
    b = _batch()
    own = ms.owners(b)
    a = [ur.oracle_linearize(b["kind"], own, b["x"], b["z"], b["sqrt_info"], b["aux"], o, long_double=True) for o in (0, 1)]
    e, _ = _k12_errors(a[0], a[1], _k12_units(b))
    assert e.max() <= 1e-12, e.max()
    t0 = ur.oracle_update_meas(*_args(b), 0, long_double=True)
    t1 = ur.oracle_update_meas(*_args(b), 1, long_double=True)
    ok = (t0[3] <= ur.SHARPEST) & (b["length"] > 0)
    P = np.linalg.inv(ur.mat(t0[1][ok]))
    well = np.linalg.cond(P) < 1e6
    eb, ex, eg = ur.errors(tuple(v[ok][well] for v in (t0[0], t0[1], t0[2])), tuple(v[ok][well] for v in (t1[0], t1[1], t1[2])), b["x"][ok][well])
    worst = max(eb.max(), ex.max(), eg.max())
    print(f"K11 long double orders on {int(well.sum())} of {int(ok.sum())} filters with condition < 1e6: worst {worst:.1e}")
    assert well.sum() >= 100 and worst <= 1e-10
    kw = dict(loss=b["loss"], loss_k=b["loss_k"], max_iterations=3, tol=0.0)
    i0 = ur.oracle_update_iter(*_args(b), 0, long_double=True, **kw)
    i1 = ur.oracle_update_iter(*_args(b), 1, long_double=True, **kw)
    ok = (i0[7] <= ur.SHARPEST) & (b["length"] > 0)
    well = np.linalg.cond(np.linalg.inv(ur.mat(i0[1][ok]))) < 1e6
    eb, ex, eg = ur.errors(tuple(v[ok][well] for v in (i0[0], i0[1], i0[2])), tuple(v[ok][well] for v in (i1[0], i1[1], i1[2])), b["x"][ok][well])
    worst = max(eb.max(), ex.max(), eg.max())
    print(f"K13 (3 iterations) long double orders on {int(well.sum())} of {int(ok.sum())} filters: worst {worst:.1e}")
    assert well.sum() >= 100 and worst <= 1e-10
    t = ur.oracle_update_iter(*_args(b), 0, long_double=True, loss=b["loss"], loss_k=b["loss_k"], max_iterations=10, tol=1e-9)
    some = b["length"] > 0
    flip, same, s0 = chain_stress.local_branches(b["x"][some], t[5][some])
    fb = b["tag"][some] == "branch/flip"
    print(f"local15 branches on (x_hat, x_lin): flip {int(flip.sum())} (branch group {int(flip[fb].sum())} of {int(fb.sum())}), "
          f"same {int(same.sum())}, s = 0 {int(s0.sum())}")
    assert flip.any() and (~flip & ~same).any() and same.any() and flip[fb].any() and s0[b["tag"][some] == "branch/s0"].all()


def test_gate_passes_fp64_and_fails_injected_errors():
    """Both fp64 orders pass the gate of each kernel.  The gate fails, and the criterion of the existing statement tests is reported
    beside it for: K12 one info entry rounded to fp32, f' of a far lever-arm-free position measurement formed as |S h - S z|^2; K11
    Sigma+ of one filter rounded to fp32, gamma x (1 + 1e-7), the last measurement of a 1024-long list dropped; K13 Sigma+ of the
    first linearisation with the state of the last, IRLS weights frozen at x_hat."""
    b = _batch()
    own = ms.owners(b)
    caught = {}
    # K12
    truth = ur.oracle_linearize(b["kind"], own, b["x"], b["z"], b["sqrt_info"], b["aux"], 0, long_double=True)
    fp = [ur.oracle_linearize(b["kind"], own, b["x"], b["z"], b["sqrt_info"], b["aux"], o) for o in (0, 1)]
    for o in (0, 1):
        r, name = gate_k12(b, fp[o], truth, fp)
        print(f"K12 fp64 order {o}: worst ratio {r:.2f} ({name})")
        assert r <= 1.0
    j = int(np.flatnonzero((b["tag"][own] == "pos/l1/near/random/S1e-2/unit") | (b["tag"][own] == "pos/l1/near/random/S1e-2/slow"))[0])
    info = fp[0][0].copy(); info[j, 12 * 15 + 1] = np.float32(info[j, 12 * 15 + 1])
    caught["K12 info entry in fp32"] = gate_k12(b, (info, fp[0][1], fp[0][2]), truth, fp)[0]
    far = np.flatnonzero(np.char.startswith(b["tag"][own], "pos/l0/near/") & (b["state"][own] == "far") & (b["s_family"][own] == "1e-2"))
    j = int(far[0])
    S = mr.sqrt_mat(b["sqrt_info"][j:j + 1])[0]
    h = mr.h_of(b["kind"][j:j + 1], b["x"][own[j]:own[j] + 1], b["aux"][j:j + 1])[0]
    f = fp[0][2].copy(); f[j] = np.sum((S @ h - S @ b["z"][j]) ** 2)
    caught["K12 f' as |S h - S z|^2"] = gate_k12(b, (fp[0][0], fp[0][1], f), truth, fp)[0]
    sb = _k12_units(b)
    for name, got in (("K12 info entry in fp32", (info, fp[0][1], fp[0][2])), ("K12 f' as |S h - S z|^2", (fp[0][0], fp[0][1], f))):
        old = _k12_errors(fp[0], got, sb)[0].max() > 1e-13                # test_measurements' 1e-13 of the scales, against fp64
        print(f"{name}: the existing statement test's criterion {'catches' if old else 'misses'} it")
    # K11
    t, f64, ok, gf = k11_reference(b)
    for o in (0, 1):
        r, name = gate_filters(b["tag"], b["x"], t, f64, f64[o], ok, gf)
        print(f"K11 fp64 order {o}: worst ratio {r:.2f} ({name})")
        assert r <= 1.0
    i = int(np.flatnonzero(np.char.startswith(b["tag"], "pos/l1/near/random/S1e-2/") & ok & (b["length"] > 0) & (b["state"] != "far"))[0])
    c = f64[0][1].copy(); c[i] = c[i].astype(np.float32)
    inj = {"K11 Sigma+ in fp32": (f64[0][0], c, f64[0][2])}
    g = f64[0][2].copy(); g[i] *= 1 + 1e-7
    inj["K11 gamma x (1 + 1e-7)"] = (f64[0][0], f64[0][1], g)
    i = int(np.flatnonzero(ok & (b["length"] == 1024) & (np.char.find(b["tag"], "/near/") > 0) & (b["s_family"] != "zero"))[0])
    si = b["sqrt_info"].copy(); si[b["offsets"][i + 1] - 1] = 0.0                 # S = 0: the measurement drops out
    d = ur.oracle_update_meas(b["x"], b["cov"], b["offsets"], b["kind"], b["z"], si, b["aux"], 0)
    inj["K11 last of 1024 dropped"] = (d[0], d[1], d[2])
    for name, got in inj.items():
        caught[name] = gate_filters(b["tag"], b["x"], t, f64, got, ok, gf)[0]
        print(f"{name}: the existing statement tests' criterion {'catches' if _numpy_style_catches(t, f64, got, b['x'], ok) else 'misses'} it")
    # K13 at tol 0, cap 3
    t, f64, ok, gf, _ = k13_reference(b, None, 3, 0.0)
    for o in (0, 1):
        r, name = gate_filters(b["tag"], b["x"], t, f64, f64[o], ok, gf)
        print(f"K13 fp64 order {o}: worst ratio {r:.2f} ({name})")
        assert r <= 1.0
    first = ur.oracle_update_iter(*_args(b), 0, loss=b["loss"], loss_k=b["loss_k"], max_iterations=1, tol=0.0)
    inj = {"K13 Sigma+ of the first linearisation": (f64[0][0], first[1], f64[0][2])}
    x0 = b["x"][own]
    _, _, b0 = mr.meas_ref(b["kind"], x0, b["z"], b["sqrt_info"], b["aux"])
    om = ir.weight(b["loss"], b["loss_k"], np.einsum("ni,ni->n", b0, b0))
    fr = ur.oracle_update_iter(b["x"], b["cov"], b["offsets"], b["kind"], b["z"], b["sqrt_info"] * np.sqrt(om)[:, None], b["aux"], 0,
                               max_iterations=3, tol=0.0)
    inj["K13 IRLS weights frozen at x_hat"] = (fr[0], fr[1], fr[2])
    for name, got in inj.items():
        caught[name] = gate_filters(b["tag"], b["x"], t, f64, got, ok, gf)[0]
        print(f"{name}: the existing statement tests' criterion {'catches' if _numpy_style_catches(t, f64, got, b['x'], ok) else 'misses'} it")
    for name, r in caught.items():
        print(f"injected {name}: ratio {r:.3g}")
    assert all(r > 1.0 for r in caught.values()), caught


# ---------------------------------------------------------------------------------------------- GPU

def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def gpu_batch(cuda):
    """The stress batch with K7 covariances after 50, 200 and 600 keyframes of both models as one more covariance family."""
    from test_update import _k7_covariances
    extra = []
    for model in (1, 2):
        covs, _ = _k7_covariances(cuda, model, 4, 600, 40 + model)
        extra.append(covs[[49, 199, 599]].reshape(-1, 225))
    return ms.stress_batch(extra_cov=np.concatenate(extra))


def _k12(torch, b, full=True):
    from cpi_b200 import capi, factor
    lib, p = capi.load(), factor._tptr
    M = len(b["kind"])
    f64 = dict(dtype=torch.float64, device="cuda")
    d = [_dev(torch, a) for a in (b["kind"], ms.owners(b), b["x"], b["z"], b["sqrt_info"], b["aux"])]
    info, rhs, f = torch.empty((M, 225), **f64), torch.empty((M, 15), **f64), torch.empty(M, **f64)
    capi.check(lib.cpi_imu_measurements_linearize(M, *[p(t) for t in d], p(info) if full else None, p(rhs) if full else None, p(f), None))
    torch.cuda.synchronize()
    return info.cpu().numpy(), rhs.cpu().numpy(), f.cpu().numpy()


def _ms(torch, b):
    return tuple(_dev(torch, a) for a in (ms.owners(b), b["kind"], b["z"], b["sqrt_info"], b["aux"]))


def _k11(torch, b, gate=None):
    from cpi_b200 import factor
    g = _dev(torch, gate) if isinstance(gate, np.ndarray) else gate
    out = factor.update_measurements(_dev(torch, b["x"]), _dev(torch, b["cov"]), _ms(torch, b), gate=g)
    torch.cuda.synchronize()
    return tuple(t.cpu().numpy() for t in out)


def _k13(torch, b, max_iterations, tol, gate=None):
    from cpi_b200 import factor
    g = _dev(torch, gate) if isinstance(gate, np.ndarray) else gate
    out = factor.update_measurements_iterated(_dev(torch, b["x"]), _dev(torch, b["cov"]), _ms(torch, b), gate=g,
                                              measurement_loss=(_dev(torch, b["loss"]), _dev(torch, b["loss_k"])),
                                              max_iterations=max_iterations, tol=tol)
    torch.cuda.synchronize()
    return tuple(t.cpu().numpy() for t in out)


@pytest.mark.gpu
def test_k12_against_extended_precision(cuda, gpu_batch):
    """Every measurement of K12 passes the gate; info exactly symmetric; the f-only pass bitwise the full pass's f."""
    b = gpu_batch
    got = _k12(cuda, b)
    f_only = _k12(cuda, b, full=False)[2]
    I = ur.mat(got[0])
    assert np.array_equal(I, I.transpose(0, 2, 1)) and np.array_equal(f_only, got[2])
    r, name = gate_k12(b, got)
    print(f"K12 on {len(b['kind'])} measurements: worst ratio to the bound {r:.3f} ({name})")
    assert r <= 1.0, (name, r)


@pytest.mark.gpu
def test_k11_against_extended_precision(cuda, gpu_batch):
    """Every filter of K11 under the limit passes the gate; Sigma+ exactly symmetric; filters without measurements and gated filters
    (gate 16) bitwise their inputs, the others bitwise the ungated run."""
    b = gpu_batch
    got = _k11(cuda, b)
    assert np.array_equal(ur.mat(got[1]), ur.mat(got[1]).transpose(0, 2, 1), equal_nan=True) and np.all(got[3] == 1)
    none = b["length"] == 0
    assert np.array_equal(got[0][none], b["x"][none]) and np.array_equal(got[1][none], b["cov"][none]) and np.all(got[2][none] == 0)
    t, f64, ok, gf = k11_reference(b)
    r, name = gate_filters(b["tag"], b["x"], t, f64, got[:3], ok, gf)
    print(f"K11 on {int(ok.sum())} of {len(ok)} filters: worst ratio to the bound {r:.3f} ({name})")
    assert r <= 1.0, (name, r)
    xo, co, g, a = _k11(cuda, b, gate=np.full(len(b["x"]), 16.0))
    skip = a == 0
    assert skip.any() and np.array_equal(g, got[2], equal_nan=True)
    assert np.array_equal(xo[skip], b["x"][skip]) and np.array_equal(co[skip], b["cov"][skip])
    assert np.array_equal(xo[~skip], got[0][~skip], equal_nan=True) and np.array_equal(co[~skip], got[1][~skip], equal_nan=True)


RUNS = ((3, 0.0), (10, 1e-9))


def _k13_gates(b, outs):
    """Gate K13's outputs outs[(cap, tol)] = (x+, cov+, gamma, status, iterations) of the batch b for both RUNS against the oracle
    forced to the kernel's iteration counts (e_64 the larger of the two runs': the fp64 error scale is the filter's problem's, not the
    stopping point's), and its status and iterations against the free oracle where fp64 decides them."""
    runs = {}
    for cap, tol in RUNS:
        got = outs[cap, tol]
        t, f64, ok, gf, _ = k13_reference(b, got[4].astype(np.int32), cap, tol)
        runs[cap, tol] = (got, t, f64, ok, gf, e64_filters(b["tag"], b["x"], t, f64, ok))
    e64 = np.maximum(*[v[5] for v in runs.values()])
    for (cap, tol), (got, t, f64, ok, gf, _) in runs.items():
        r, name = gate_filters(b["tag"], b["x"], t, f64, got[:3], ok, gf, e64)
        kw = dict(loss=b["loss"], loss_k=b["loss_k"], max_iterations=cap, tol=tol)
        free = ur.oracle_update_iter(*_args(b), 0, long_double=True, **kw)
        fp = [ur.oracle_update_iter(*_args(b), o, contract=c, **kw) for c in (False, True) for o in (0, 1)]
        if tol > 0:
            # the issue's criterion (margin above 1e-6) narrowed to where every fp64 statement stops as the truth does: an
            # ill-conditioned filter's fp64 path drifts from the long-double one by far more than 1e-6 in r
            decided = ok & (free[6] > 1e-6)
            for o in fp:
                decided &= (o[3] == free[3]) & (o[4] == free[4])
        else:
            # at tol = 0 there is no margin (any step that rounds to zero stops); the count is decided where the truth and every
            # fp64 statement take all cap linearisations
            decided = ok & (free[4] == cap)
            for o in fp:
                decided &= o[4] == cap
        differ = decided & ((got[3] != free[3]) | (got[4] != free[4]))
        print(f"K13 cap {cap}, tol {tol:g}, on {int(ok.sum())} of {len(ok)} filters: worst ratio to the bound {r:.3f} ({name}); "
              f"iterations {np.bincount(got[4]).tolist()}; status and iterations decided in fp64 on {int(decided.sum())}, "
              f"the kernel's differ on {int(differ.sum())} {list(zip(b['tag'][differ][:5], got[4][differ][:5], free[4][differ][:5]))}")
        assert r <= 1.0, (name, r)
        assert decided.sum() > len(ok) // 2 and not differ.any()


@pytest.mark.gpu
def test_k13_against_extended_precision(cuda, gpu_batch):
    """K13 at tol 0 with cap 3 and at tol 1e-9 with cap 10, against the oracle forced to the kernel's iteration counts: every filter
    under the limit passes the gate (e_64 the larger of the two runs'); Sigma+ exactly symmetric; status and iterations those of the
    free oracle wherever fp64 decides them (_k13_gates); gated filters (gate 16) and filters without measurements bitwise their inputs; at tol = +inf Sigma+ and
    gamma bitwise K11's."""
    b = gpu_batch
    none = b["length"] == 0
    outs = {}
    for cap, tol in RUNS:
        got = outs[cap, tol] = _k13(cuda, b, cap, tol)
        assert np.array_equal(ur.mat(got[1]), ur.mat(got[1]).transpose(0, 2, 1), equal_nan=True)
        assert np.array_equal(got[0][none], b["x"][none]) and np.array_equal(got[1][none], b["cov"][none]) and np.all(got[4][none] == 0)
    _k13_gates(b, outs)
    k11 = _k11(cuda, b)
    gauss = dict(b); gauss["loss"] = np.zeros_like(b["loss"])
    one = _k13(cuda, gauss, 1, float("inf"))
    assert np.array_equal(one[1], k11[1], equal_nan=True) and np.array_equal(one[2], k11[2], equal_nan=True)
    free = _k13(cuda, b, 10, 1e-9)
    xo, co, g, st, it = _k13(cuda, b, 10, 1e-9, gate=np.full(len(b["x"]), 16.0))
    skip = st == 0
    assert skip.any() and np.array_equal(g, free[2], equal_nan=True) and np.all(it[skip] == 1)
    assert np.array_equal(xo[skip], b["x"][skip]) and np.array_equal(co[skip], b["cov"][skip])
    assert all(np.array_equal(u[~skip], v[~skip], equal_nan=True) for u, v in zip((xo, co, st, it), (free[0], free[1], free[3], free[4])))


@pytest.mark.gpu
def test_nan_in_one_filter_is_confined(cuda, gpu_batch):
    """A NaN in z of one measurement of one 33-long list leaves every other measurement of K12 and every other filter of K11 and
    K13 bitwise the clean run."""
    b = gpu_batch
    i = int(np.flatnonzero((b["length"] == 33) & np.char.startswith(b["tag"], "dir/unit/near"))[0])
    bad = dict(b); bad["z"] = b["z"].copy()
    j = int(b["offsets"][i]) + 16
    bad["z"][j, 1] = np.nan
    keep = np.arange(len(b["x"])) != i
    mk = np.arange(len(b["kind"])) != j
    clean, dirty = _k12(cuda, b), _k12(cuda, bad)
    assert all(np.array_equal(u[mk], v[mk]) for u, v in zip(clean, dirty))
    for run in (lambda q: _k11(cuda, q), lambda q: _k13(cuda, q, 10, 1e-9)):
        clean, dirty = run(b), run(bad)
        assert all(np.array_equal(u[keep], v[keep], equal_nan=True) for u, v in zip(clean, dirty))
        assert np.isnan(dirty[2][i])


# ---------------------------------------------------------------------------------------------- production scale
# The batch's distinct cases (classes) tiled to production sizes on the device; every copy is compared bitwise with its class's first
# copy on the device (host memory stays bounded); the first copies are the batch itself and are gated against the oracle.

def _same_bits(torch, out, cls, first):
    """Whether every row of out [n, ...] is bitwise the row first[cls] (NaNs compared by their bits)."""
    ref = out.index_select(0, first.index_select(0, cls))
    return torch.equal(out.contiguous().view(torch.int64 if out.dtype == torch.float64 else out.dtype), ref.contiguous().view(
        torch.int64 if out.dtype == torch.float64 else out.dtype))


@pytest.mark.gpu
def test_k12_at_scale(cuda, gpu_batch):
    """2^20 + 37 measurements (the last warp partial) on 128 copies of the batch's states (about 2e5): measurement p is class
    p mod C, so the copies of a class sit at several lane and warp residues mod 64 (MWARPS = 2) and every residue hosts copies.  The
    full and the f-only pass: every copy bitwise its class's first copy; the first copies (the batch) pass the gate."""
    from cpi_b200 import capi, factor
    torch = cuda
    b = gpu_batch
    own = ms.owners(b)
    C, N, R = len(own), len(b["x"]), 128
    n = 2 ** 20 + 37
    p = np.arange(n)
    res = p % 64
    per_class = np.bincount(p % C, minlength=C)
    assert per_class.min() >= 2 and len(np.unique(res)) == 64 and n % 64 != 0
    assert C % 64 != 0                                               # copies j and j + C of a class: two residues at least
    d = lambda a: _dev(torch, a)
    cls = torch.arange(n, device="cuda") % C
    idx = ((torch.arange(n, device="cuda") // C) % R) * N + d(own).index_select(0, cls)
    X = d(b["x"]).repeat(R, 1)
    kind, z, si, aux = (d(b[k]).index_select(0, cls).contiguous() for k in ("kind", "z", "sqrt_info", "aux"))
    lib, tp = capi.load(), factor._tptr
    f64 = dict(dtype=torch.float64, device="cuda")
    info, rhs, f, f_only = torch.empty((n, 225), **f64), torch.empty((n, 15), **f64), torch.empty(n, **f64), torch.empty(n, **f64)
    capi.check(lib.cpi_imu_measurements_linearize(n, tp(kind), tp(idx), tp(X), tp(z), tp(si), tp(aux), tp(info), tp(rhs), tp(f), None))
    capi.check(lib.cpi_imu_measurements_linearize(n, tp(kind), tp(idx), tp(X), tp(z), tp(si), tp(aux), None, None, tp(f_only), None))
    torch.cuda.synchronize()
    first = torch.arange(C, device="cuda")
    assert all(_same_bits(torch, a, cls, first) for a in (info, rhs, f))
    assert torch.equal(f_only.view(torch.int64), f.view(torch.int64))
    got = tuple(a[:C].cpu().numpy() for a in (info, rhs, f))
    del info, rhs, f, f_only, X, kind, z, si, aux
    r, name = gate_k12(b, got)
    print(f"K12 at scale: {n} measurements, {C} classes on {R * N} states: copies bitwise their classes; classes' worst ratio "
          f"{r:.3f} ({name})")
    assert r <= 1.0, (name, r)


def _tiled_filters(torch, b, n):
    """The filters of b (an odd count C) tiled to n on the device, filter p a copy of class p mod C: (cls, x, cov, offsets, kind, z,
    sqrt_info, aux, loss, loss_k) as device tensors."""
    d = lambda a: _dev(torch, a)
    C = len(b["x"])
    cls = torch.arange(n, device="cuda") % C
    ln = d(b["length"]).index_select(0, cls)
    toff = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    toff[1:] = torch.cumsum(ln, 0)
    Mt = int(toff[-1])
    start = d(b["offsets"][:-1]).index_select(0, cls)
    g = torch.repeat_interleave(start - toff[:-1], ln, output_size=Mt) + torch.arange(Mt, device="cuda")
    cols = tuple(d(b[k]).index_select(0, g).contiguous() for k in ("kind", "z", "sqrt_info", "aux", "loss", "loss_k"))
    del g
    return (cls, d(b["x"]).index_select(0, cls).contiguous(), d(b["cov"]).index_select(0, cls).contiguous(), toff) + cols


def _odd_classes(b):
    """The batch without its last filter when its count is even: an odd class count puts the copies of every class at every warp
    slot mod UWARPS = 4."""
    keep = np.ones(len(b["x"]), bool)
    if len(keep) % 2 == 0:
        keep[-1] = False
    return ms.select(b, keep)


@pytest.mark.gpu
def test_k11_and_k13_at_scale(cuda, gpu_batch):
    """10^6 filters, filter p a copy of class p mod C (C odd: every class at every warp slot mod 4), CSR lists starting at every residue
    mod 64 and the 1024-long lists included (about 7e7 measurements).  K11, and K13 at tol 0 with cap 3 and at tol 1e-9 with cap 10:
    every copy bitwise its class's first copy in every output; the first copies (the batch) pass the gates of the batch tests."""
    torch = cuda
    from cpi_b200 import capi, factor
    b = _odd_classes(gpu_batch)
    C, n = len(b["x"]), 10 ** 6
    cls, x, cov, off, kind, z, si, aux, loss, loss_k = _tiled_filters(torch, b, n)
    assert C % 2 == 1 and len(torch.unique(off[:-1] % 64)) == 64
    assert int((torch.diff(off) == 1024).sum()) >= n // C
    lib, tp = capi.load(), factor._tptr
    f64 = dict(dtype=torch.float64, device="cuda")
    first = torch.arange(C, device="cuda")
    xo, co, nis = torch.empty((n, 16), **f64), torch.empty((n, 225), **f64), torch.empty(n, **f64)
    a1, a2 = torch.empty(n, dtype=torch.int32, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda")
    capi.check(lib.cpi_state_update_measurements_batch(n, tp(x), tp(cov), tp(off), tp(kind), tp(z), tp(si), tp(aux), None, tp(xo),
                                                       tp(co), tp(nis), tp(a1), None))
    torch.cuda.synchronize()
    assert all(_same_bits(torch, a, cls, first) for a in (xo, co, nis, a1))
    got = tuple(a[:C].cpu().numpy() for a in (xo, co, nis, a1))
    t, f64s, ok, gf = k11_reference(b)
    r, name = gate_filters(b["tag"], b["x"], t, f64s, got[:3], ok, gf)
    print(f"K11 at scale: {n} filters, {int(off[-1])} measurements, {C} classes: copies bitwise their classes; classes' worst ratio "
          f"{r:.3f} ({name})")
    assert r <= 1.0, (name, r)
    outs = {}
    for cap, tol in RUNS:
        capi.check(lib.cpi_state_update_measurements_iterated_batch(n, tp(x), tp(cov), tp(off), tp(kind), tp(z), tp(si), tp(aux), tp(loss),
                                                                    tp(loss_k), None, cap, tol, tp(xo), tp(co), tp(nis), tp(a1), tp(a2),
                                                                    None))
        torch.cuda.synchronize()
        assert all(_same_bits(torch, a, cls, first) for a in (xo, co, nis, a1, a2)), (cap, tol)
        outs[cap, tol] = tuple(a[:C].cpu().numpy() for a in (xo, co, nis, a1, a2))
    _k13_gates(b, outs)


@pytest.mark.gpu
@pytest.mark.parametrize("model", [1, 2])
def test_chain_measurement_fold_at_scale(cuda, oracle, model):
    """chains_lm_step with measurements on every state of chain_scale.lm_batch's tiled layout (about 3e5 states, chains straddling
    every fold_pass boundary for 132 and 114 SMs and this device's count), with Gaussian, Huber and Cauchy measurement losses: every
    copy bitwise its class's first copy in its step and cost; each distinct chain's first copy within
    test_measurements.test_lm_step_is_the_dense_gauss_newton_step's bound of the dense damped step of the numpy system."""
    from chain_scale import LM_LENGTHS, SMS, lm_batch
    from cpi_b200 import capi, factor
    from test_chain_scale import _same_per_class, _sms
    from test_chains_lm import dev_prior, make_problem
    from test_marginalize import _dense_truth, vec
    from test_robust_priors import robust_ref
    from test_state_priors import _chain_idx, _np_system
    torch = cuda
    d = lambda a: _dev(torch, a)
    lengths = np.asarray(LM_LENGTHS)
    rng = np.random.default_rng(90 + model)
    X, rec, L, offs, pri, per = make_problem(oracle, model, lengths, 600 + model, large=True, with_prior=True, first_window=130000)
    Nd = len(X)
    mm = mr.random_measurements(rng, X, Nd, sigma=0.05)
    mm = (np.arange(Nd, dtype=np.int64),) + tuple(mm[1:])                      # one measurement on every state
    mm = (mm[0], mm[1], mr.h_of(mm[1], X, mm[4]) + rng.normal(size=(Nd, 3)) * 0.05, mm[3], mm[4])
    src, toffs, cls, _ = lm_batch(lengths, tuple(dict.fromkeys(SMS + (_sms(torch),))))
    sidx = np.concatenate([np.arange(offs[c], offs[c + 1]) for c in src])
    fidx = np.concatenate([np.arange(offs[c] - c, offs[c + 1] - c - 1) for c in src])
    tms = (np.arange(len(sidx), dtype=np.int64),) + tuple(a[sidx] for a in mm[1:])
    PI = np.stack([vec(p[0][None])[0] for p in pri])
    tprior = tuple(d(a) for a in (PI[src], np.stack([p[1] for p in pri])[src], np.array([p[2] for p in pri])[src],
                                  np.stack([p[3] for p in pri])[src]))
    dX, dR, dL = d(X), d(rec), d(L)
    e, H1, H2 = factor.factor_eval(model, dX, dR, dL, *_chain_idx(torch, offs))
    Gh = [t.cpu().numpy() for t in factor.factor_hessian(model, dR, e, H1, H2)]
    firsts = {}
    for i, c in enumerate(src):
        firsts.setdefault(int(c), i)
    lam, worst = 1e-5, 0.0
    for loss in (None, capi.LOSS_HUBER, capi.LOSS_CAUCHY):
        code = None if loss is None else np.full(Nd, loss, dtype=np.int32)
        kk = np.full(Nd, 1.5)
        tl = None if loss is None else (d(code[sidx]), d(kk[sidx]))
        new, dx, cost = factor.chains_lm_step(model, d(X[sidx]), d(rec[fidx]), d(L[fidx]), d(toffs), prior=tprior, lam=lam,
                                              measurements=tuple(d(a) for a in tms), measurement_loss=tl)
        dx, cost = dx.cpu().numpy(), cost.cpu().numpy()
        _same_per_class([lambda i: dx[toffs[i]:toffs[i + 1]], lambda i: cost[i]], cls, set())
        info, rhs, f = mr.linearize_ref(mm[1], X[mm[0]], mm[2], mm[3], mm[4])
        if loss is not None:
            info, rhs, f = robust_ref(code, kk, info, rhs, f)
        for c, (Xc, r, l) in enumerate(per):
            f0, S = int(offs[c] - c), len(Xc)
            sps = [(int(q - offs[c]), info[q], rhs[q], f[q], X[q]) for q in range(offs[c], offs[c + 1])]
            A, bb, cur = _np_system(oracle, model, Xc, r, l, pri[c], sps, blocks=[g[f0:f0 + S - 1] for g in Gh])
            A[np.diag_indices_from(A)] += lam * np.clip(np.diag(A), 1e-6, 1e32)
            xt, x64 = _dense_truth(A, bb)
            i = firsts[c]
            dd = dx[toffs[i]:toffs[i + 1]].reshape(-1)
            nt = np.linalg.norm(xt)
            e_dev, e64 = np.linalg.norm(dd - xt) / nt, np.linalg.norm(x64 - xt) / nt
            worst = max(worst, e_dev / (50 * max(e64, 1e-13)))
            assert e_dev <= 50 * max(e64, 1e-13), (loss, c, e_dev, e64)
            assert abs(cost[i] - cur) <= 1e-10 * max(abs(cur), 1.0), (loss, c, cost[i], cur)
    print(f"model {model}: chains_lm_step with measurements on {len(sidx)} states, {len(src)} chains: copies bitwise their classes; "
          f"worst ratio to the dense step's bound {worst:.3f}")

