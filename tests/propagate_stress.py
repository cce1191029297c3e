"""The propagation stress batch: K7 (cpi_propagate_batch) on the records, anchor states and covariances a filter feeds it.

Every window is one case of the cross product record family x anchor family x covariance family, tagged
"record/anchor/cov" (the gate's group).  Records come from the fp64 oracle:
  stress     tests/stress.py's windows: 100 Hz - 1 kHz, 20-35 rad/s, 16 g, dR through pi, the small_w / closed-form band
  gaps       its gap windows (steps of 0.1-0.5 s), whose P_meas is indefinite (DESIGN.md section 5)
  edge       the zero-step record, g = 0 and two 50 s slow-rotation windows (with bias_off, |J_q dbg| of 3 rad)
  merged     model 1: cpi_merge_records of groups of a 300-keyframe chain (K5)
  scan       model 1: prefixes of that chain's scan (K6), every one from the chain's first linearisation point
Anchors: at the linearisation point (at_lin); biases off it (bias_off); q_K far from q_lin (q_far: model 2's q_kR takes its
w < 0 flip); positions of 1e6 m at 300 m/s (far); quaternions that are exactly unit in fp64 (unit_q, where the closed-form Rk^-1 =
Rk^T is exact, see test_propagate_precision).  Covariances (COVS): random_cov, zero, tight (position sd 5e-5 m), condition 1e8 and
1e12, rank-deficient PSD, dead-reckoned by the fp64 statement of K7 after 50, 200, 600 and 5000 keyframes, and posteriors of K10,
K11 and K13 (Huber and Cauchy losses, from K11's batch) from their stress batches."""
from __future__ import annotations

import numpy as np

import factor_stress as fs
import update_ref as ur
from cpi_b200 import synth

SIGMAS = np.array([0.005, 4e-6, 0.01, 0.0002])
SEED = 20261017
DR_STEPS = (50, 200, 600, 5000)
COVS = ("random", "zero", "tight", "cond1e8", "cond1e12", "rank5") + tuple(f"dr{k}" for k in DR_STEPS) + ("k10post", "k11post", "k13post")
ANCHORS = ("at_lin", "bias_off", "q_far", "far", "unit_q")
# after 600 and 5000 keyframes: the smallest position block norm and the largest b_g block norm of the dead-reckoned covariances
# (asserted; measured at least 5.6e4 and 3e8, and at most 2.1e-9 and 1.5e-8)
DR_SCALE = {600: (1e4, 1e-8), 5000: (1e8, 3e-8)}


def mat(a):
    return np.asarray(a).reshape(-1, 15, 15).transpose(0, 2, 1)


def vec(M):
    return np.ascontiguousarray(np.asarray(M).transpose(0, 2, 1).reshape(-1, 225))


def chain_records(oracle, model, n_chains, steps, first_window):
    """(records [n_chains * steps, RD], lin) of n_chains keyframe chains of 20 samples at 200 Hz, one linearisation point per chain."""
    S, L = synth.make_windows(n_chains * steps, 20, rate=200.0, first_window=first_window, special=False)
    L = np.repeat(L[::steps], steps, axis=0)
    return oracle.preintegrate(model, S, L, SIGMAS, 0, ns=20, nthreads=_threads()), L


def _threads():
    return synth.usable_cpus()


def dead_reckoned(oracle, model, rng, n):
    """{steps: [n, 225]}: a random covariance with b_g and b_a sd of 1e-5 propagated through 5000 keyframes of 0.1 s (fp64 statement
    of K7, the kernel's order), read after each of DR_STEPS, from anchors at the linearisation point."""
    rec, L = chain_records(oracle, model, n, max(DR_STEPS), 61000 + 10 * model)
    X = anchors_at_lin(rec[::max(DR_STEPS)], L[::max(DR_STEPS)], model)
    out, S, done = {}, ur.random_cov(rng, n, scale=(2e-3, 1e-5, 2e-2, 1e-5, 5e-2)), 0
    K = max(DR_STEPS)
    rec, L = rec.reshape(n, K, -1), L.reshape(n, K, 13)
    for k in DR_STEPS:
        X, S = oracle.propagate_chain(model, X, S, rec[:, done:k], L[:, done:k], k - done, order=1, nthreads=_threads())
        out[k], done = S, k
    return out


def anchors_at_lin(rec, L, model):
    X = synth.make_states(rec, L, model)[:len(rec)]
    X[:, 4:7], X[:, 10:13] = L[:, 0:3], L[:, 3:6]
    if model == 2:
        X[:, 0:4] = L[:, 6:10]
    return X


def posteriors(rng, n):
    """{"k10post", "k11post", "k13post": [n,225]}: finite posteriors of the fp64 K10, K11 and K13 statements on their stress batches
    (K13 with the batch's Huber and Cauchy losses)."""
    import measurement_stress as ms
    b = ur.stress_batch(rng)
    _, c, _, _ = ur.oracle_update(b["x"], b["cov"], b["W"], b["xb"], 0)
    c = c[np.all(np.isfinite(c), axis=1)]
    m = ms.stress_batch()
    _, c2, _, _ = ur.oracle_update_meas(m["x"], m["cov"], m["offsets"], m["kind"], m["z"], m["sqrt_info"], m["aux"], 0)
    c2 = c2[np.all(np.isfinite(c2), axis=1)]
    c3 = ur.oracle_update_iter(m["x"], m["cov"], m["offsets"], m["kind"], m["z"], m["sqrt_info"], m["aux"], 0, loss=m["loss"],
                               loss_k=m["loss_k"], max_iterations=10, tol=1e-9)[1]
    c3 = c3[np.all(np.isfinite(c3), axis=1)]
    return {k: v[rng.choice(len(v), n, replace=False)] for k, v in (("k10post", c), ("k11post", c2), ("k13post", c3))}


def covariances(oracle, model, rng, n=24):
    """{family: [n, 225]} for every family of COVS."""
    G = rng.normal(size=(n, 15, 5)) * np.repeat([2e-3, 2e-4, 2e-2, 2e-3, 5e-2], 3)[None, :, None]
    R = G @ G.transpose(0, 2, 1)
    out = dict(random=ur.random_cov(rng, n), zero=np.zeros((n, 225)), tight=ur.random_cov(rng, n, scale=(2e-6, 2e-8, 2e-5, 2e-6, 5e-5)),
               cond1e8=ur.conditioned_cov(rng, n, 1e8), cond1e12=ur.conditioned_cov(rng, n, 1e12), rank5=vec(0.5 * (R + R.transpose(0, 2, 1))))
    out.update({f"dr{k}": v for k, v in dead_reckoned(oracle, model, rng, n).items()})
    out.update(posteriors(rng, n))
    return out


def _anchor(rng, fam, rec, L, model):
    X = anchors_at_lin(rec, L, model)
    n = len(X)
    if fam == "bias_off":
        dbg = rng.normal(size=(n, 3)) * 0.03
        slow = rec[:, 19] >= 9.0                                     # the 50 s windows: |J_q dbg| set to 3 rad
        jq = np.linalg.norm(np.einsum("nij,nj->ni", fs.rec33(rec[slow], 20), dbg[slow]), axis=1)
        dbg[slow] *= (3.0 / jq)[:, None]
        X[:, 4:7] += dbg
        X[:, 10:13] += rng.normal(size=(n, 3)) * 0.05
    elif fam == "q_far":
        X[:, 0:4] = fs._rand_q(rng, n)
        X[:, 4:7] += rng.normal(size=(n, 3)) * 1e-3
    elif fam == "far":
        X[:, 13:16] = rng.normal(size=(n, 3)) * 1e6
        v = rng.normal(size=(n, 3))
        X[:, 7:10] = 300.0 * v / np.linalg.norm(v, axis=1, keepdims=True)
    elif fam == "unit_q":
        X[:, 0:4] = np.eye(4)[rng.integers(0, 4, n)]
    return X


def records(oracle, model):
    """(records, lin, family [n])."""
    import stress
    rec, L = fs.records(oracle, model, SIGMAS)
    _, _, _, reg = stress.make_batch()
    fam = np.array(["gaps" if r == "gaps" else "stress" for r in reg] + ["edge"] * (len(rec) - len(reg)))
    if model == 1:
        cr, cl = chain_records(oracle, 1, 2, 300, 64000)
        merged = oracle.merge_records(cr, cl, group_offsets=np.array([0, 7, 40, 300, 301, 420, 600]), nthreads=_threads())
        scan = oracle.scan_records(cr, cl, group=300, nthreads=_threads())
        pick = np.r_[0:300:13, 299, 300:600:17, 599]
        rec = np.concatenate([rec, merged, scan[pick]])
        L = np.concatenate([L, cl[[0, 7, 40, 300, 301, 420]], cl[pick]])
        fam = np.concatenate([fam, ["merged"] * len(merged), ["scan"] * len(pick)])
    return rec, L, fam


def stress_batch(oracle, model, seed=SEED):
    """dict(x [n,16], cov [n,225], records [n,RD], lin [n,13], tag [n]) of one model: every record against every anchor family and
    every covariance family (the member of the family cycles with the window).  Asserts its coverage: both branches of the w < 0 flip
    of q_n, every anchor and covariance family, the block scales of the dead-reckoned covariances, |J_q dbg| of 3 rad."""
    rng = np.random.default_rng(seed + model)
    rec, L, rfam = records(oracle, model)
    covs = covariances(oracle, model, rng)
    xs, cs, rs, ls, tags = [], [], [], [], []
    n = len(rec)
    for a in ANCHORS:
        X = _anchor(rng, a, rec, L, model)
        for k, c in enumerate(COVS):
            pool = covs[c]
            xs.append(X); rs.append(rec); ls.append(L)
            cs.append(pool[(np.arange(n) + k) % len(pool)])
            tags += [f"{f}/{a}/{c}" for f in rfam]
    b = dict(x=np.concatenate(xs), cov=np.concatenate(cs), records=np.concatenate(rs), lin=np.concatenate(ls), tag=np.array(tags))
    b["coverage"] = coverage(oracle, model, b, covs)
    return b


def coverage(oracle, model, b, covs):
    X, rec, L = b["x"], b["records"], b["lin"]
    n = len(X)
    Xh = oracle.predict_state(model, X, rec, L)
    cov = fs.coverage(model, np.concatenate([X, Xh]), np.arange(n), np.arange(n, 2 * n), rec, L)
    # q_n takes both branches.  q_r cannot flip at a prediction: there q_rm = q_n q_meas^-1 is the identity to rounding, so q_r
    # is q_b, whose w >= 0 (rot_2_quat); it could only flip at |J_q dbg| = pi, where Q = w I + [v x] is singular
    assert cov["q_n:flip"] > 0 and cov["q_n:no flip"] > 0, cov
    assert cov["q_r:flip"] == 0, cov
    jq = np.linalg.norm(np.einsum("nij,nj->ni", fs.rec33(rec, 20), X[:, 4:7] - L[:, 0:3]), axis=1)
    assert jq.max() >= 2.99, jq.max()
    parts = np.array([t.split("/") for t in b["tag"]])
    for k, fams in ((1, ANCHORS), (2, COVS)):
        assert set(parts[:, k]) == set(fams)
    for k, (pos, bias) in DR_SCALE.items():
        C = mat(covs[f"dr{k}"])
        assert np.linalg.norm(C[:, 12:15, 12:15], axis=(1, 2)).min() >= pos
        assert np.linalg.norm(C[:, 3:6, 3:6], axis=(1, 2)).max() <= bias
    return dict(cov, jq=float(jq.max()))
