"""Seeded factor stress batch for the precision tests of the factor, prediction, retraction and information-form kernels.

numpy only, plus the fp64 oracle that is passed in: the records are ``stress.make_batch()`` (every preintegration regime, the
2 000 / 10 000-sample windows included) run through the fp64 oracle, so a factor gate measures the factor kernels alone.  Two
constructed records are appended: the zero-step record (an empty window: R = I, DT = 0, P = 0) and a window with g = 0.

State pairs (x_K, x_K1), tagged by regime:

  chain       the perturbed chain of cpi_b200.synth.make_states through every record, in order
  far         independent random states from a small pool: relative rotations up to pi, states shared between factors
  near_pi     x_K1 built so that the residual rotation q_r is 1e-3 .. 1e-7 rad short of pi (q_r's w near 0)
  bias_far    |J_q dbg| from 0 to 3 rad on the long windows, dbg <= 0.1 rad/s, along x, y, z and random axes (every
              rot_2_quat case of q_b)
  zero_bias   biases exactly at the linearisation point (Exp_so3's th == 0 branch), half of them at the exact prediction
  large       positions 1e3 .. 1e6 m, 100 m/s, the 50 s window: cancellation in pa / pb; half at the exact prediction
  same_state  idx_i == idx_j
  q_far_lin   q_K far from the linearisation point's q_lin (model 2: q_kR = q_K q_lin^-1 takes its w < 0 flip)

The factors are shuffled and so is the storage order of the states, so idx_i / idx_j are in no order, repeat, and run backwards
(idx_i > idx_j) about half the time.  The factor count is not a multiple of the 8 factors of a K3 CTA.

``coverage`` is a numpy mirror of the branch decisions of K3 (cpi_common.cuh: rot_2_quat's four cases for q_b, the w < 0 flip of
quat_multiply for q_n, q_rm, q_r, q_m, q_kR); ``retract_coverage`` that of k_retract (the flip of dq and its 0/0 NaN branch).  The
builders fail if a branch is never taken, or never skipped."""
from __future__ import annotations

import numpy as np

import stress

SEED = 20261016
RD = {1: 290, 2: 308}
FREGIMES = ("chain", "far", "near_pi", "bias_far", "zero_bias", "large", "same_state", "q_far_lin")
R2Q_CASES = ("x", "y", "z", "trace")
FLIPS = ("q_n", "q_rm", "q_r", "q_m", "q_kR")


# ---------------------------------------------------------------------------------------------- numpy mirror (fp64)

def qmul(q, p):
    """quat_multiply of cpi_common.cuh, batched [n, 4]: (JPL q (x) p with w >= 0, normalised, flip taken [n] bool)."""
    t = np.stack([q[:, 3] * p[:, 0] + q[:, 2] * p[:, 1] - q[:, 1] * p[:, 2] + q[:, 0] * p[:, 3],
                  -q[:, 2] * p[:, 0] + q[:, 3] * p[:, 1] + q[:, 0] * p[:, 2] + q[:, 1] * p[:, 3],
                  q[:, 1] * p[:, 0] - q[:, 0] * p[:, 1] + q[:, 3] * p[:, 2] + q[:, 2] * p[:, 3],
                  -q[:, 0] * p[:, 0] - q[:, 1] * p[:, 1] - q[:, 2] * p[:, 2] + q[:, 3] * p[:, 3]], axis=1)
    flip = t[:, 3] < 0
    t[flip] *= -1
    return t / np.linalg.norm(t, axis=1, keepdims=True), flip


def qinv(q):
    return q * np.array([-1.0, -1.0, -1.0, 1.0])


def skew(v):
    z = np.zeros(len(v))
    return np.stack([np.stack([z, -v[:, 2], v[:, 1]], 1), np.stack([v[:, 2], z, -v[:, 0]], 1), np.stack([-v[:, 1], v[:, 0], z], 1)], 1)


def exp_so3(w):
    """Exp_so3 [n,3] -> [n,3,3]; identity where |w| == 0 in fp64."""
    th = np.sqrt(np.sum(w * w, axis=1))
    nz = th > 0
    ts = np.where(nz, th, 1.0)
    a = np.where(nz, np.sin(ts) / ts, 0.0)[:, None, None]
    b = np.where(nz, (1 - np.cos(ts)) / ts ** 2, 0.0)[:, None, None]
    K = skew(w)
    return np.eye(3) + a * K + b * (K @ K)


def rot_2_quat(R):
    """rot_2_quat [n,3,3] -> (q [n,4], case index [n] into R2Q_CASES)."""
    r00, r11, r22 = R[:, 0, 0], R[:, 1, 1], R[:, 2, 2]
    T = r00 + r11 + r22
    cx = (r00 >= T) & (r00 >= r11) & (r00 >= r22)
    cy = ~cx & (r11 >= T) & (r11 >= r00) & (r11 >= r22)
    cz = ~cx & ~cy & (r22 >= T) & (r22 >= r00) & (r22 >= r11)
    case = np.where(cx, 0, np.where(cy, 1, np.where(cz, 2, 3)))
    q = np.zeros((len(R), 4))
    with np.errstate(divide="ignore", invalid="ignore"):
        s = np.sqrt(np.maximum(1 + 2 * r00 - T, 0) / 4); d = 1 / (4 * s)
        qx = np.stack([s, d * (R[:, 0, 1] + R[:, 1, 0]), d * (R[:, 0, 2] + R[:, 2, 0]), d * (R[:, 1, 2] - R[:, 2, 1])], 1)
        s = np.sqrt(np.maximum(1 + 2 * r11 - T, 0) / 4); d = 1 / (4 * s)
        qy = np.stack([d * (R[:, 0, 1] + R[:, 1, 0]), s, d * (R[:, 1, 2] + R[:, 2, 1]), d * (R[:, 2, 0] - R[:, 0, 2])], 1)
        s = np.sqrt(np.maximum(1 + 2 * r22 - T, 0) / 4); d = 1 / (4 * s)
        qz = np.stack([d * (R[:, 0, 2] + R[:, 2, 0]), d * (R[:, 1, 2] + R[:, 2, 1]), s, d * (R[:, 0, 1] - R[:, 1, 0])], 1)
        s = np.sqrt(np.maximum(1 + T, 0) / 4); d = 1 / (4 * s)
        qw = np.stack([d * (R[:, 1, 2] - R[:, 2, 1]), d * (R[:, 2, 0] - R[:, 0, 2]), d * (R[:, 0, 1] - R[:, 1, 0]), s], 1)
    for c, qc in enumerate((qx, qy, qz, qw)):
        q[case == c] = qc[case == c]
    q[q[:, 3] < 0] *= -1
    return q / np.linalg.norm(q, axis=1, keepdims=True), case


def rec33(records, a):
    """record 3x3 block at column a (column-major) -> [n,3,3]"""
    return records[:, a:a + 9].reshape(-1, 3, 3).transpose(0, 2, 1)


def front(states, idx_i, idx_j, records, lin):
    """The quaternion chain of evaluateError in fp64: dict of q_b, q_n, q_rm, q_r, q_m, q_kR, the rot_2_quat case of q_b and the
    flip flags (model-2 q_kR; its flags are meaningful for model 2 only)."""
    xi, xj = states[idx_i], states[idx_j]
    dbg = xi[:, 4:7] - lin[:, 0:3]
    t3 = -np.einsum("nij,nj->ni", rec33(records, 20), dbg)
    q_b, case = rot_2_quat(exp_so3(t3))
    q_n, f_n = qmul(xj[:, 0:4], qinv(xi[:, 0:4]))
    q_rm, f_rm = qmul(q_n, qinv(records[:, 0:4]))
    q_r, f_r = qmul(q_rm, q_b)
    q_m, f_m = qmul(qinv(q_b), records[:, 0:4])
    q_kR, f_kR = qmul(xi[:, 0:4], qinv(lin[:, 6:10]))
    return dict(q_b=q_b, q_n=q_n, q_rm=q_rm, q_r=q_r, q_m=q_m, q_kR=q_kR, case=case, t3=t3,
                flip=dict(q_n=f_n, q_rm=f_rm, q_r=f_r, q_m=f_m, q_kR=f_kR))


def coverage(model, states, idx_i, idx_j, records, lin):
    """Counts of every branch of K3's quaternion chain: {"q_b:x": ..., "q_r:flip": ..., "q_r:no flip": ...}."""
    fr = front(states, idx_i, idx_j, records, lin)
    out = {f"q_b:{c}": int(np.sum(fr["case"] == k)) for k, c in enumerate(R2Q_CASES)}
    for name in FLIPS:
        if name == "q_kR" and model == 1:
            continue
        f = fr["flip"][name]
        out[f"{name}:flip"] = int(f.sum()); out[f"{name}:no flip"] = int((~f).sum())
    return out


def retract_branches(xi):
    """k_retract's branches in fp64: (flip of dq taken [n], 0/0 NaN branch taken [n])."""
    n2 = np.sum(xi[:, 0:3] ** 2, axis=1)
    nrm = np.sqrt(n2)
    with np.errstate(divide="ignore", invalid="ignore"):
        nan = np.isnan(np.sin(nrm / 2) / nrm)
    return (np.cos(nrm / 2) < 0) & ~nan, nan


def retract_coverage(xi):
    flip, nan = retract_branches(xi)
    return {"flip": int(flip.sum()), "no flip": int((~flip & ~nan).sum()), "nan": int(nan.sum())}


# ---------------------------------------------------------------------------------------------- builders

def _rand_q(rng, n):
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[q[:, 3] < 0] *= -1
    return q


def _perturb(rng, X, th=1e-2, v=1e-1, p=1e-1, b=1e-3):
    """make_states' perturbation: rotate q by a random angle ~th, add noise to biases, v and p."""
    X = X.copy()
    if th > 0:
        d = rng.normal(0, th, (len(X), 3))
        n = np.linalg.norm(d, axis=1, keepdims=True)
        dq = np.concatenate([np.sin(n / 2) / n * d, np.cos(n / 2)], axis=1)
        X[:, 0:4], _ = qmul(dq, X[:, 0:4])
    X[:, 4:7] += rng.normal(0, b, (len(X), 3)); X[:, 10:13] += rng.normal(0, b, (len(X), 3))
    X[:, 7:10] += rng.normal(0, v, (len(X), 3)); X[:, 13:16] += rng.normal(0, p, (len(X), 3))
    return X


def _random_states(rng, n, lin=None):
    X = np.zeros((n, 16))
    X[:, 0:4] = _rand_q(rng, n)
    X[:, 4:7] = rng.normal(0, 1e-2, (n, 3)) + (0 if lin is None else lin[:, 0:3])
    X[:, 7:10] = rng.normal(0, 3.0, (n, 3))
    X[:, 10:13] = rng.normal(0, 1e-1, (n, 3)) + (0 if lin is None else lin[:, 3:6])
    X[:, 13:16] = rng.normal(0, 10.0, (n, 3))
    return X


def records(oracle, model, sigmas):
    """(records [n,RD], lin [n,13]): the stress batch through the fp64 oracle, plus a zero-step and a g = 0 record."""
    S, off, L, _ = stress.make_batch()
    rng = np.random.default_rng(SEED)
    g0 = stress._window(rng, 150, 1 / 200.0)
    lin_g0 = stress._lin(rng, 0.0)
    g0[:, 0:3] += lin_g0[0:3]; g0[:, 3:6] += lin_g0[3:6]
    wins, lins = [g0], [stress._lin(rng), lin_g0]
    # 50 s of slow rotation: the smallest singular value of J_q is >= 30 s, so |J_q dbg| reaches 3 rad in any direction with
    # |dbg| <= 0.1 rad/s.  The second turns by 2.5 rad about one axis, so that q_b^-1 q_meas can take its w < 0 flip.
    for w_hat in (None, 0.05 * stress._unit(rng, 1)[0]):
        lin = stress._lin(rng)
        w = stress._window(rng, 10000, 1 / 200.0, w_scale=0.002, w_hat=w_hat)
        w[:, 0:3] += lin[0:3]; w[:, 3:6] += lin[3:6]
        wins.append(w); lins.append(lin)
    lens = [0] + [len(w) for w in wins]                              # an empty window first
    S = np.concatenate([S] + wins)
    off = np.concatenate([off, off[-1] + np.cumsum(lens)])
    L = np.concatenate([L, np.stack(lins)])
    from cpi_b200.synth import usable_cpus
    rec = oracle.preintegrate(model, S, L, sigmas, 0, offsets=off, nthreads=usable_cpus())
    assert rec[-4, 19] == 0.0 and np.all(rec[-4, 65:290] == 0.0) and np.all(L[-3, 10:13] == 0.0)
    return rec, L


def factor_batch(oracle, model, sigmas, seed=SEED):
    """The factor stress batch of one model: dict(states [M,16], idx_i, idx_j [n] int64, records [n,RD], lin [n,13], tags [n]).
    Asserts that every branch of ``coverage`` is taken and skipped at least once."""
    from cpi_b200.synth import make_states
    rec, L = records(oracle, model, sigmas)
    nr = len(rec)
    rng = np.random.default_rng(seed + model)
    dt = rec[:, 19]
    long_ = np.flatnonzero(dt >= 9.0)
    pred = lambda X, r: oracle.predict_state(model, X, rec[r], L[r])
    S_list, pairs, rsel, tags = [], [], [], []

    def add(tag, XK, XK1, r, same=False):
        base = sum(len(s) for s in S_list)
        m = len(XK)
        if same:
            S_list.append(XK); a = base + np.arange(m); b = a
        else:
            S_list.append(np.concatenate([XK, XK1])); a = base + np.arange(m); b = a + m
        pairs.append(np.stack([a, b], 1)); rsel.append(np.asarray(r)); tags.extend([tag] * m)

    # chain: every record, in order
    Xc = make_states(rec, L, model, seed=seed)
    base = 0
    S_list.append(Xc); pairs.append(np.stack([np.arange(nr), np.arange(1, nr + 1)], 1)); rsel.append(np.arange(nr)); tags.extend(["chain"] * nr)
    # far: a pool of 48 random states, 240 random pairs (states shared between factors)
    pool = _random_states(rng, 48)
    base = sum(len(s) for s in S_list)
    S_list.append(pool)
    a = rng.integers(0, 48, 240); b = (a + rng.integers(1, 48, 240)) % 48
    pairs.append(np.stack([base + a, base + b], 1)); rsel.append(rng.integers(0, nr, 240)); tags.extend(["far"] * 240)
    # near_pi: q_K1 = q_r q_b^-1 q_meas q_K with q_r a rotation by pi - eps
    m = 120
    r = rng.integers(0, nr, m)
    XK = _random_states(rng, m, L[r])
    XK[:, 4:7] = L[r, 0:3] + rng.normal(0, 1e-3, (m, 3))
    fr = front(np.concatenate([XK, XK]), np.arange(m), np.arange(m, 2 * m), rec[r], L[r])
    eps = 10.0 ** rng.uniform(-7, -3, m)
    u = rng.normal(size=(m, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
    q_t = np.concatenate([u * np.cos(eps / 2)[:, None], np.sin(eps / 2)[:, None]], axis=1)
    q1, _ = qmul(q_t, qinv(fr["q_b"])); q1, _ = qmul(q1, rec[r, 0:4]); q1, _ = qmul(q1, XK[:, 0:4])
    XK1 = _perturb(rng, pred(XK, r), th=0.0)
    XK1[:, 0:4] = q1
    add("near_pi", XK, XK1, r)
    # bias_far: |J_q dbg| in [0, 3] rad on the long windows
    m = 150
    r = long_[np.arange(m) % len(long_)]
    Jq = rec33(rec[r], 20)
    smin = np.linalg.svd(Jq, compute_uv=False)[:, -1]
    frac = rng.uniform(0, 1, m)
    frac[:len(long_)], frac[len(long_):2 * len(long_)] = 1e-3, 1.0       # both ends on every long window
    th = frac * np.minimum(3.0, 0.1 * smin)
    ax = np.concatenate([np.eye(3), rng.normal(size=(1, 3))])[np.arange(m) % 4]
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    ax *= rng.choice([-1.0, 1.0], (m, 1))
    dbg = -np.linalg.solve(Jq, (th[:, None] * ax)[..., None])[..., 0]
    XK = _random_states(rng, m, L[r])
    XK[:, 4:7] = L[r, 0:3] + dbg
    add("bias_far", XK, _perturb(rng, pred(XK, r)), r)
    # zero_bias: dbg = dba = 0 exactly; half at the exact prediction
    m = 80
    r = rng.integers(0, nr, m)
    XK = _random_states(rng, m, L[r])
    XK[:, 4:7] = L[r, 0:3]; XK[:, 10:13] = L[r, 3:6]
    XK1 = pred(XK, r)
    XK1[m // 2:] = _perturb(rng, XK1[m // 2:])
    add("zero_bias", XK, XK1, r)
    # large: |p| 1e3 .. 1e6 m, |v| = 100 m/s, long windows (DT up to 50 s); half at the exact prediction
    m = 64
    r = long_[np.arange(m) % len(long_)]
    XK = _random_states(rng, m, L[r])
    d = rng.normal(size=(m, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    XK[:, 13:16] = d * 10.0 ** rng.uniform(3, 6, (m, 1))
    d = rng.normal(size=(m, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    XK[:, 7:10] = 100.0 * d
    XK1 = pred(XK, r)
    XK1[m // 2:] = _perturb(rng, XK1[m // 2:])
    add("large", XK, XK1, r)
    # same_state
    m = 40
    r = rng.integers(0, nr, m)
    add("same_state", _random_states(rng, m, L[r]), None, r, same=True)
    # q_far_lin: q_K random, so q_K q_lin^-1 is anywhere
    m = 80
    r = rng.integers(0, nr, m)
    XK = _random_states(rng, m, L[r])
    add("q_far_lin", XK, _perturb(rng, pred(XK, r)), r)

    X = np.concatenate(S_list)
    P = np.concatenate(pairs)
    R = np.concatenate(rsel)
    T = np.array(tags)
    if len(P) % 8 == 0:                       # keep the last K3 CTA partial
        P, R, T = P[:-1], R[:-1], T[:-1]
    # shuffle the factors and the storage order of the states
    fperm = rng.permutation(len(P))
    sperm = rng.permutation(len(X))
    where = np.empty(len(X), dtype=np.int64); where[sperm] = np.arange(len(X))
    P, R, T = P[fperm], R[fperm], T[fperm]
    out = dict(states=np.ascontiguousarray(X[sperm]), idx_i=where[P[:, 0]], idx_j=where[P[:, 1]],
               records=np.ascontiguousarray(rec[R]), lin=np.ascontiguousarray(L[R]), tags=T)
    # the regimes do what they claim
    f = front(out["states"], out["idx_i"], out["idx_j"], out["records"], out["lin"])
    npi = T == "near_pi"
    ang = np.pi - 2 * np.arctan2(np.linalg.norm(f["q_r"][npi, 0:3], axis=1), f["q_r"][npi, 3])
    assert np.all((ang > 0.9e-7) & (ang < 1.1e-3)), (ang.min(), ang.max())
    tb = np.linalg.norm(f["t3"][T == "bias_far"], axis=1)
    assert tb.max() > 2.9 and tb.min() < 0.1 and np.all(tb <= 3.0 + 1e-9)
    assert np.all(f["t3"][T == "zero_bias"] == 0.0)
    assert np.array_equal(out["idx_i"][T == "same_state"], out["idx_j"][T == "same_state"])
    assert np.any(out["idx_i"] > out["idx_j"]) and len(np.unique(out["idx_i"])) < len(out["idx_i"])
    assert len(P) % 8 != 0
    cov = coverage(model, out["states"], out["idx_i"], out["idx_j"], out["records"], out["lin"])
    missing = [k for k, v in cov.items() if v == 0]
    assert not missing, ("branches never taken", missing, cov)
    out["coverage"] = cov
    return out


RETRACT_ANGLES = (("0", 0.0), ("1e-300", 1e-300), ("subnormal", 5e-324), ("1e-8", 1e-8), ("pi-1e-9", np.pi - 1e-9), ("pi", np.pi),
                  ("pi+1e-9", np.pi + 1e-9), ("2pi-1e-9", 2 * np.pi - 1e-9), ("2pi+1e-9", 2 * np.pi + 1e-9), ("50", 50.0))


def retract_batch(seed=SEED):
    """dict(states [n,16], xi [n,15], tags [n]): every |dtheta| of RETRACT_ANGLES along the axes and random directions, from
    random states; plus position / velocity / bias increments of 1e-12 on values around 1e6.  Asserts the flip and the NaN
    branch of k_retract are each taken and skipped."""
    rng = np.random.default_rng(seed + 7)
    X, XI, tags = [], [], []
    for name, a in RETRACT_ANGLES:
        u = np.concatenate([np.eye(3), -np.eye(3), rng.normal(size=(10, 3))])
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        m = len(u)
        xi = np.zeros((m, 15))
        xi[:, 0:3] = u * a if a >= 1e-300 else np.where(np.abs(u) == np.abs(u).max(axis=1, keepdims=True), np.sign(u) * a, 0.0)
        xi[:, 3:15] = rng.normal(0, 1e-2, (m, 12))
        X.append(_random_states(rng, m)); XI.append(xi); tags.extend([name] * m)
    m = 24
    Xb = _random_states(rng, m)
    Xb[:, 4:16] = rng.choice([-1.0, 1.0], (m, 12)) * 1e6 * rng.uniform(0.5, 2.0, (m, 12))
    xi = np.zeros((m, 15))
    xi[:, 0:3] = rng.normal(0, 1e-3, (m, 3))
    xi[:, 3:15] = rng.choice([-1e-12, 1e-12], (m, 12))
    X.append(Xb); XI.append(xi); tags.extend(["1e-12 on 1e6"] * m)
    out = dict(states=np.concatenate(X), xi=np.concatenate(XI), tags=np.array(tags))
    cov = retract_coverage(out["xi"])
    assert all(v > 0 for v in cov.values()), cov
    out["coverage"] = cov
    return out
