"""The measurement stress batch of the extended-precision gate of K12, K11 and K13 (tests/test_measurements_precision.py; DESIGN.md
sections 3l and 3m).  Per kind variant x residual mode x covariance family the filters cycle through the lengths of their measurement
lists, the families of S and the state variants; the tag (the gate's group) names all five but the length.  S family and state scale
belong in the group: sigma from 1 m to 1e-6 m and positions of 10 m and 1e6 m move fp64's error by orders of magnitude, and a group
holding both would let its worst member's error cover the others.  Layouts as include/cpi_b200.h."""
from __future__ import annotations

import numpy as np

import measurement_ref as mr
import update_ref as ur
from test_marginalize import mat, vec
from test_propagate import random_cov
from update_ref import retract, unit_states

LENGTHS = (0, 1, 2, 3, 31, 32, 33)
LONG = (255, 1024)                       # only in the random and tight covariance families, to bound the oracle's time
S_FAMILIES = ("1", "1e-2", "1e-4", "1e-6", "aniso", "rank2", "rank1", "zero")
SIGMA = {"1": 1.0, "1e-2": 1e-2, "1e-4": 1e-4, "1e-6": 1e-6, "aniso": 1e-4, "rank2": 1e-2, "rank1": 1e-2, "zero": 1.0}
VARIANTS = ("pos/l0", "pos/l1", "pos/l100", "vel/v0", "vel/v1", "vel/v300", "vel/nhc", "dir/unit", "dir/5e-5", "dir/9.81", "dir/axis")
MODES = ("exact", "near", "outlier")
COVS = ("random", "dr", "tight", "c1e8", "c1e12")
STATES = ("unit", "far", "slow")


def _cov(rng, fam, n):
    if fam == "random":
        return random_cov(rng, n)
    if fam == "dr":
        return random_cov(rng, n, scale=(1e-2, 1e-5, 1.0, 1e-3, 10.0))
    if fam == "tight":
        return random_cov(rng, n, scale=(2e-6, 2e-8, 2e-5, 2e-6, 5e-5))
    return ur.conditioned_cov(rng, n, {"c1e8": 1e8, "c1e12": 1e12}[fam])


def _s(rng, fam, m):
    """[m, 9] column-major S of the family: isotropic 1/sigma in a random rotation, anisotropic (sigma 1e-4, 1e-1, 1e2: condition
    1e6), rank 2, rank 1 or zero."""
    Q, _ = np.linalg.qr(rng.normal(size=(m, 3, 3)))
    d = {"aniso": [1e4, 10.0, 1e-2], "rank2": [1e2, 1e2, 0.0], "rank1": [1e2, 0.0, 0.0], "zero": [0.0, 0.0, 0.0]}.get(fam)
    d = np.full(3, 1.0 / SIGMA[fam]) if d is None else np.array(d)
    S = d[None, :, None] * Q.transpose(0, 2, 1)
    return S.transpose(0, 2, 1).reshape(m, 9)


def _state(rng, variant, sv):
    x = unit_states(rng, 1)[0]
    if sv == "far":
        x[13:16] += rng.normal(size=3) * 1e6
    speed = {"vel/v0": 0.0, "vel/v1": 1.0, "vel/v300": 300.0}.get(variant, 5.0 if sv != "slow" else 1.0)
    v = rng.normal(size=3)
    x[7:10] = v / np.linalg.norm(v) * speed
    return x


def _measurements(rng, variant, x, m, fam):
    kind = {"pos": mr.POSITION, "vel": mr.VELOCITY_BODY, "dir": mr.DIRECTION}[variant[:3]]
    kind = np.full(m, kind, dtype=np.int32)
    si = _s(rng, fam, m)
    aux = rng.normal(size=(m, 3))
    aux /= np.linalg.norm(aux, axis=1, keepdims=True)
    if variant.startswith("pos"):
        aux *= {"pos/l0": 0.0, "pos/l1": 1.0, "pos/l100": 100.0}[variant]
    elif variant == "vel/nhc":
        si = np.tile(np.diag([0.0, 20.0, 20.0]).T.reshape(9), (m, 1))          # lateral and vertical body rows only
    elif variant == "dir/5e-5":
        aux *= 5e-5
    elif variant == "dir/9.81":
        aux *= 9.81
    elif variant == "dir/axis":
        q = x[0:3]
        aux = np.tile(q / np.linalg.norm(q), (m, 1)) * rng.uniform(0.5, 2.0, size=(m, 1))
    return kind, si, aux


def _pin(rng, kind, x, si, aux, mode, sigma):
    z = mr.h_of(kind, np.repeat(x[None], len(kind), axis=0), aux)
    if mode != "exact":
        z = z + rng.normal(size=z.shape) * sigma * (1000.0 if mode == "outlier" else 1.0)
    return z


def _losses(rng, m):
    """Gaussian, Huber and Cauchy cycled, k log-uniform from 1e-10 to 1e4."""
    return (np.arange(m) % 3).astype(np.int32), 10.0 ** rng.uniform(-10, 4, size=m)


def _edges(rng):
    """Filters of one exactly known POSITION residual (aux = 0, S = I, r = (3, 0, 0), so s = 9 on every route): Huber with k = 3 at
    s = k^2 exactly; and Cauchy with k = 1e-10 and S = 1e140 I, r = 1e5 m: s = 1e290 > k^2 DBL_MAX, the overflow branch."""
    out = []
    for tag, scale, code, k, r in (("edge/huber_s=k2", 1.0, 1, 3.0, 3.0), ("edge/cauchy_overflow", 1e140, 2, 1e-10, 1e5)):
        for i in range(4):
            x = unit_states(rng, 1)[0]
            x[0:4] = [0.0, 0.0, 0.0, 1.0]
            x[13:16] = [10.0, 20.0, 30.0]
            z = x[13:16][None] - np.array([[r, 0.0, 0.0]])
            out.append((tag, x, _cov(rng, "random", 1)[0], np.array([mr.POSITION], np.int32), z, (np.eye(3) * scale).reshape(1, 9),
                        np.zeros((1, 3)), (np.array([code], np.int32), np.array([k]))))
    return out


def _flip_branch(rng, n=16):
    """Filters with a large attitude prior (sd 1.2 rad) and two tight DIRECTION measurements of a truth 2.5 to 3 rad away from x_hat,
    so that Gauss-Newton carries x_t past the point where local15(x_hat, x_t) takes quat_multiply's flip."""
    out = []
    for i in range(n):
        x = unit_states(rng, 1)[0]
        ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
        truth = retract(x[None], np.concatenate([ax * rng.uniform(2.5, 3.0), np.zeros(12)])[None])[0]
        Sig = mat(random_cov(rng, 1))[0]
        Sig[0:3, :] = 0.0; Sig[:, 0:3] = 0.0; Sig[0:3, 0:3] = np.eye(3) * 1.2 ** 2
        kind = np.full(2, mr.DIRECTION, np.int32)
        aux = np.array([[0.0, 0.0, 1.0], [0.6, 0.8, 0.0]])
        z = mr.h_of(kind, np.repeat(truth[None], 2, axis=0), aux)
        out.append(("branch/flip", x, vec(Sig[None])[0], kind, z, np.tile((np.eye(3) / 0.01).reshape(9), (2, 1)), aux,
                    (np.zeros(2, np.int32), np.zeros(2))))
    return out


def _same_rotation(rng, n=8):
    """Filters whose x_hat has a quaternion of w < 0 with exactly unit norm (components +-1/2), an attitude decoupled from the rest of
    Sigma and one lever-arm-free POSITION fix: the step leaves the attitude exactly (H_theta = 0), the retraction flips the sign, and
    the next linearisation point is -x_hat's quaternion bit for bit: local15(x_hat, x_t) takes its s = 0 branch."""
    out = []
    for i in range(n):
        x = unit_states(rng, 1)[0]
        x[0:4] = 0.5 * np.array([1.0 if (i >> k) & 1 else -1.0 for k in range(3)] + [-1.0])
        Sig = mat(random_cov(rng, 1))[0]
        Sig[0:3, 3:] = 0.0; Sig[3:, 0:3] = 0.0
        z = x[13:16][None] + rng.normal(size=(1, 3)) * 0.05
        out.append(("branch/s0", x, vec(Sig[None])[0], np.array([mr.POSITION], np.int32), z, (np.eye(3) / 0.05).reshape(1, 9),
                    np.zeros((1, 3)), (np.zeros(1, np.int32), np.zeros(1))))
    return out


def stress_batch(seed=20261017, extra_cov=None):
    """dict(x [n,16], cov [n,225], offsets [n+1], kind, z, sqrt_info, aux, loss, loss_k [M], tag [n], length [n], s_family [n],
    state [n]).  extra_cov (K7 covariances, GPU only) adds one covariance family "k7"."""
    rng = np.random.default_rng(seed)
    rows = []
    covs = COVS + (("k7",) if extra_cov is not None else ())
    for vi, variant in enumerate(VARIANTS):
        for mode in MODES:
            for ci, fam in enumerate(covs):
                lengths = LENGTHS + (LONG if fam in ("random", "tight") else ())
                cs = np.asarray(extra_cov)[rng.integers(0, len(extra_cov), len(lengths))] if fam == "k7" else _cov(rng, fam, len(lengths))
                for i, m in enumerate(lengths):
                    sf = S_FAMILIES[(i + vi + ci) % len(S_FAMILIES)]
                    sv = STATES[(i + ci) % len(STATES)]
                    x = _state(rng, variant, sv)
                    kind, si, aux = _measurements(rng, variant, x, m, sf)
                    z = _pin(rng, kind, x, si, aux, mode, SIGMA[sf])
                    rows.append((f"{variant}/{mode}/{fam}/S{sf}/{sv}", x, cs[i], kind, z, si, aux, _losses(rng, m), m, sf, sv))
    for r in _edges(rng) + _flip_branch(rng) + _same_rotation(rng):
        rows.append(r + (len(r[3]), "edge", "unit"))
    counts = np.array([len(r[3]) for r in rows])
    return dict(x=np.stack([r[1] for r in rows]), cov=np.stack([r[2] for r in rows]),
                offsets=np.r_[0, np.cumsum(counts)].astype(np.int64),
                kind=np.concatenate([r[3] for r in rows]).astype(np.int32), z=np.concatenate([r[4] for r in rows]).reshape(-1, 3),
                sqrt_info=np.concatenate([r[5] for r in rows]).reshape(-1, 9), aux=np.concatenate([r[6] for r in rows]).reshape(-1, 3),
                loss=np.concatenate([r[7][0] for r in rows]).astype(np.int32), loss_k=np.concatenate([r[7][1] for r in rows]),
                tag=np.array([r[0] for r in rows]), length=counts, s_family=np.array([r[9] for r in rows]),
                state=np.array([r[10] for r in rows]))


def owners(b):
    """The filter index of every measurement of the batch b."""
    return np.repeat(np.arange(len(b["x"])), np.diff(b["offsets"])).astype(np.int64)


def select(b, keep):
    """The filters keep [n] bool of the batch b with their measurements."""
    own = owners(b)
    mk = keep[own]
    out = {k: b[k][keep] for k in ("x", "cov", "tag", "length", "s_family", "state")}
    out.update({k: b[k][mk] for k in ("kind", "z", "sqrt_info", "aux", "loss", "loss_k")})
    out["offsets"] = np.r_[0, np.cumsum(b["length"][keep])].astype(np.int64)
    return out
