"""Seeded record stress batch for the precision tests of the record merge (K5) and scan (K6) kernels.

numpy only, plus the fp64 oracle that is passed in (it preintegrates the records):

  segments     every window of ``stress.make_batch()`` (every preintegration regime, the 2 000 / 10 000-sample windows
               included) cut into S segments, S cycling through SEGMENTS with the window; segments of 0 and 1 samples, and cuts
               at the dt = 0 samples (a 1-sample segment holding one is a zero-step record mid-group).  One group per window.
               The group's later segments are preintegrated at linearisation points moved by one of OFFSETS (cycling with the
               window, out of step with S):
                 zero    the first segment's lin (no move)
                 ba      only b_a moved
                 bw      only b_w moved
                 tiny    b_w and b_a moved by 1e-12
                 large   b_w moved so that |J_q db_w| is 0.5 .. 3 rad, and within 1e-3 of pi; the segment's gyro readings move
                         with its b_w, so its record (and J_q) is the one at the first lin and the angle is what was asked
                 qg      only lin[6:13] (q_lin, gravity) moved: a model-1 record does not depend on them, nor may its merge
  independent  the records of ``factor_stress.records`` (every stress regime, the zero-step record, g = 0, 50 s of slow rotation,
               gap windows whose P is indefinite) in random groups of 1 .. 12 records, each at its own lin

``r2q_branches`` mirrors the branch decisions of rot_2_quat (cpi_common.cuh): the four cases and the w < 0 flip.

``merge_bracketing`` and ``scan_bracketing`` restate the order in which K5 and K6 combine records (K5: chunked pairwise trees
in 2W shared-memory slots; K6: a segmented reduce-then-scan in chunks of 32, Brent-Kung inside a chunk) with the fp64 oracle's
pair merge, one vectorised call per tree level: the fp64 error of the kernels' own bracketing."""
from __future__ import annotations

import numpy as np

import factor_stress as fs
import stress

SEED = 20261017
RD = 290
SEGMENTS = (2, 3, 8, 40)
OFFSETS = ("zero", "ba", "bw", "tiny", "large", "qg")
SCAN_C = 32                     # records per chunk of K6 (scan.cu C)


def _threads():
    from cpi_b200.synth import usable_cpus
    return usable_cpus()


def zero_record():
    r = np.zeros(RD); r[3] = 1.0; r[4:13] = np.eye(3).reshape(-1)
    return r


# ---------------------------------------------------------------------------------------------- segmented stress windows

def _cuts(rng, L, S, zero_dt):
    """S - 1 sorted cut positions in [0, L]: a 0-sample and a 1-sample segment where S allows, and cuts either side of a
    dt = 0 sample."""
    c = list(rng.integers(0, L + 1, size=S - 1))
    k = 0
    if len(zero_dt) and S >= 2:
        p = int(zero_dt[rng.integers(0, len(zero_dt))])
        c[k] = p; k += 1
        if S >= 3:
            c[k] = p + 1; k += 1
    if S - 1 - k >= 2:
        a = int(rng.integers(0, L + 1)); c[k] = c[k + 1] = a; k += 2          # an empty segment
    if S - 1 - k >= 2 and L >= 1:
        a = int(rng.integers(0, L)); c[k], c[k + 1] = a, a + 1; k += 2       # a 1-sample segment
    return np.sort(np.asarray(c, dtype=np.int64))


def segment_batch(oracle, sigmas, seed=SEED):
    """dict(records [n,290], lin [n,13], offsets [g+1] (one group per window), regime [g], offset [g] (OFFSETS), S [g],
    samples / seg_offsets (the segments' CSR samples, after the "large" shift), win_samples / win_offsets / win_lin (the
    whole windows, for a one-shot record), angle [n] (|J_q db_w| of every record against its group's first lin))."""
    S_, off, L, tags = stress.make_batch()
    rng = np.random.default_rng(seed)
    nw = len(off) - 1
    segs, seg_lin, goff, offset_tag, nseg = [], [], [0], [], []
    for w in range(nw):
        s = S_[off[w]:off[w + 1]]
        S = SEGMENTS[w % len(SEGMENTS)]
        b = np.concatenate([[0], _cuts(rng, len(s), S, np.flatnonzero(s[:, 6] == 0.0)), [len(s)]])
        tag = OFFSETS[(w // len(SEGMENTS) + w) % len(OFFSETS)]
        for k in range(S):
            segs.append(s[b[k]:b[k + 1]].copy())
            lk = L[w].copy()
            if k > 0:
                if tag == "ba":
                    lk[3:6] += rng.normal(0, 0.05, 3)
                elif tag == "bw":
                    lk[0:3] += rng.normal(0, 2e-3, 3)
                elif tag == "tiny":
                    lk[0:6] += rng.choice([-1e-12, 1e-12], 6)
                elif tag == "qg":
                    q = rng.normal(size=4); q /= np.linalg.norm(q)
                    lk[6:10] = q if q[3] >= 0 else -q
                    lk[10:13] = stress._unit(rng, 1)[0] * rng.uniform(0, 30.0)
            seg_lin.append(lk)
        goff.append(goff[-1] + S); offset_tag.append(tag); nseg.append(S)
    lens = np.array([len(x) for x in segs])
    soff = np.zeros(len(segs) + 1, dtype=np.int64); soff[1:] = np.cumsum(lens)
    Sx = np.concatenate(segs).reshape(-1, 7)
    lin = np.stack(seg_lin)
    goff = np.asarray(goff, dtype=np.int64); offset_tag = np.array(offset_tag)
    first = np.repeat(goff[:-1], np.diff(goff))
    # "large": J_q of each later segment at the first lin (its gyro readings move with b_w, so that is its J_q), then the move
    rec0 = oracle.preintegrate(1, Sx, lin, sigmas, 0, offsets=soff, nthreads=_threads())
    targets = np.array([3.0, np.pi - 5e-4, np.pi + 5e-4, np.pi - 1e-3, 2.0, 0.5])
    t = 0
    for g in np.flatnonzero(offset_tag == "large"):
        for k in range(goff[g] + 1, goff[g + 1]):
            Jq = rec0[k, 20:29].reshape(3, 3, order="F")
            sv = np.linalg.svd(Jq, compute_uv=False)
            if sv[-1] < 1e-2:                   # shorter than about 10 ms: |db_w| would exceed ~300 rad/s
                continue
            u = stress._unit(rng, 1)[0]
            d = np.linalg.solve(Jq, targets[t % len(targets)] * u)      # J_q db_w = target u with db_w = lin_0 - lin_k = d
            t += 1
            lin[k, 0:3] = lin[first[k], 0:3] - d
            Sx[soff[k]:soff[k + 1], 0:3] -= d
    rec = oracle.preintegrate(1, Sx, lin, sigmas, 0, offsets=soff, nthreads=_threads())
    dbw = lin[first, 0:3] - lin[:, 0:3]
    angle = np.linalg.norm(np.einsum("nij,nj->ni", fs.rec33(rec, 20), dbw), axis=1)
    return dict(records=rec, lin=lin, offsets=goff, regime=np.asarray(tags), offset=offset_tag, S=np.array(nseg),
                samples=Sx, seg_offsets=soff, win_samples=S_, win_offsets=off, win_lin=L, angle=angle)


# ---------------------------------------------------------------------------------------------- independent records

def independent_pool(oracle, sigmas):
    """(records, lin) of factor_stress: every preintegration regime, zero-step, g = 0, 50 s slow rotation."""
    return fs.records(oracle, 1, sigmas)


def random_groups(rng, pool, lins, n_groups, lo=1, hi=12):
    """n_groups groups of lo .. hi random pool records, each at its own lin: (records, lin, offsets)."""
    lens = rng.integers(lo, hi + 1, size=n_groups)
    idx = rng.integers(0, len(pool), size=int(lens.sum()))
    off = np.zeros(n_groups + 1, dtype=np.int64); off[1:] = np.cumsum(lens)
    return np.ascontiguousarray(pool[idx]), np.ascontiguousarray(lins[idx]), off


def r2q_branches(records):
    """rot_2_quat of every record's R: (case index into factor_stress.R2Q_CASES [n], w < 0 before the flip [n])."""
    R = fs.rec33(records, 4)
    r00, r11, r22 = R[:, 0, 0], R[:, 1, 1], R[:, 2, 2]
    T = r00 + r11 + r22
    cx = (r00 >= T) & (r00 >= r11) & (r00 >= r22)
    cy = ~cx & (r11 >= T) & (r11 >= r00) & (r11 >= r22)
    cz = ~cx & ~cy & (r22 >= T) & (r22 >= r00) & (r22 >= r11)
    case = np.where(cx, 0, np.where(cy, 1, np.where(cz, 2, 3)))
    # the sign of w before the flip: its numerator over a positive 4 q_case
    num = np.select([cx, cy, cz], [R[:, 1, 2] - R[:, 2, 1], R[:, 2, 0] - R[:, 0, 2], R[:, 0, 1] - R[:, 1, 0]], 1.0)
    return case, num < 0


# ---------------------------------------------------------------------------------------------- lengths

MERGE_WIDTHS = (1, 2, 3, 4, 5, 8, 9, 16, 17, 33)
MERGE_RAGGED = (0, 1, 7, 8, 9, 15, 16, 57)
SCAN_LENGTHS = (0, 1, 2, 31, 32, 33, 1023, 1024, 1025, SCAN_C ** 3 + 1)


def scan_layout(rng, head=3):
    """CSR offsets of SCAN_LENGTHS in random order with empty groups at the start, the middle and the end, offsets[0] = head."""
    lens = list(rng.permutation(SCAN_LENGTHS))
    lens = [0, 0] + lens[:5] + [0] + lens[5:] + [0, 0]
    off = np.zeros(len(lens) + 1, dtype=np.int64); off[0] = head; off[1:] = head + np.cumsum(lens)
    return off


def chain_records(oracle, sigmas, n=5000, first_window=90000):
    """n consecutive 20-sample windows at 200 Hz (the configs[4] chain's keyframe spacing), each at its own lin."""
    from cpi_b200 import synth
    S, L = synth.make_windows(n, 20, rate=200.0, first_window=first_window, special=False)
    return oracle.preintegrate(1, S, L, sigmas, 0, ns=20, nthreads=_threads()), L


# ---------------------------------------------------------------------------------------------- the kernels' bracketing in fp64

def _relinearised(oracle, rec, lin, starts):
    """Every record moved to the lin of its group's first record (starts [n]: that record's index)."""
    return oracle.relinearise(rec, lin, lin[starts])


def _group_starts(n, offsets, uniform):
    i = np.arange(n)
    if offsets is None:
        return i - i % uniform
    g = np.searchsorted(offsets, i, side="right") - 1
    return offsets[np.clip(g, 0, len(offsets) - 1)]


def merge_bracketing(oracle, rec, lin, offsets=None, group=None):
    """K5's order of operations in fp64: one record per group.  Uniform groups of u records run in 2W slots with W = 1, 2, 4, 8 for
    u <= 2, 4, 8, more (merge.cu merge_launch), CSR groups with W = 4; each chunk's pairwise tree runs over the running result in slot
    0 and the records that fill the other slots."""
    nt = _threads()
    n_rec = len(rec)
    if offsets is None:
        offsets = np.arange(0, n_rec + 1, group, dtype=np.int64)
        W = 1 if group <= 2 else 2 if group <= 4 else 4 if group <= 8 else 8
        starts = _group_starts(n_rec, None, group)
    else:
        W = 4
        starts = _group_starts(n_rec, offsets, None)
        starts[:offsets[0]] = np.arange(offsets[0])
    C = 2 * W
    E = _relinearised(oracle, rec, lin, starts) if n_rec else rec
    lens = np.diff(offsets)
    out = np.empty((len(lens), RD))
    for m in np.unique(lens):
        gs = np.flatnonzero(lens == m)
        if m == 0:
            out[gs] = zero_record()
            continue
        X = E[offsets[gs][:, None] + np.arange(m)[None, :]]                    # [G, m, RD]
        slots = np.empty((len(gs), C, RD))
        occ, nxt = 0, 0
        while nxt < m:
            take = min(m - nxt, C - occ)
            slots[:, occ:occ + take] = X[:, nxt:nxt + take]
            occ += take; nxt += take
            s = 1
            while s < occ:
                a = np.arange(0, occ - s, 2 * s); b = a + s
                slots[:, a] = oracle.merge_pair(slots[:, a].reshape(-1, RD), slots[:, b].reshape(-1, RD), nt).reshape(len(gs), len(a), RD)
                s *= 2
            occ = 1
        out[gs] = slots[:, 0]
    return out


def _seg_step(oracle, X, F, c, i, j, right):
    """K6's seg_merge on slots (c, i) (the earlier) and (c, j) of X [nch, slots, RD], flags F [nch, slots]."""
    if len(c) == 0:
        return
    fi, fj = F[c, i].copy(), F[c, j].copy()
    m = ~fj
    if m.any():
        r = oracle.merge_pair(X[c[m], i[m]], X[c[m], j[m]], _threads())
        if right:
            X[c[m], j[m]] = r
        else:
            X[c[m], i[m]] = r
    if not right and (~m).any():
        X[c[~m], i[~m]] = X[c[~m], j[~m]]
    if right:
        F[c, j] = fi | fj
    else:
        F[c, i] = fi | fj


def _chunks(E, Fl):
    n = len(E)
    nch = (n + SCAN_C - 1) // SCAN_C
    X = np.zeros((nch, SCAN_C + 1, RD)); F = np.zeros((nch, SCAN_C + 1), dtype=bool)
    idx = np.arange(n)
    X[idx // SCAN_C, idx % SCAN_C] = E; F[idx // SCAN_C, idx % SCAN_C] = Fl
    m = np.minimum(SCAN_C, n - SCAN_C * np.arange(nch))
    return X, F, m


def _pairs(m, pattern):
    """(chunk, i, j) of one step over chunks of sizes m: pattern(mc) -> (i, j) arrays for a chunk of mc elements."""
    cs, iis, jjs = [], [], []
    for c, mc in enumerate(m):
        i, j = pattern(int(mc))
        cs.append(np.full(len(i), c)); iis.append(i); jjs.append(j)
    return np.concatenate(cs).astype(np.int64), np.concatenate(iis).astype(np.int64), np.concatenate(jjs).astype(np.int64)


def _reduce(oracle, E, Fl):
    X, F, m = _chunks(E, Fl)
    s = 1
    while s < SCAN_C:
        a = lambda mc, s=s: (np.arange(0, max(mc - s, 0), 2 * s), np.arange(0, max(mc - s, 0), 2 * s) + s)
        _seg_step(oracle, X, F, *_pairs(m, a), right=False)
        s *= 2
    return X[:, 0].copy(), F[:, 0].copy()


def _down(oracle, E, Fl, seeds):
    X, F, m = _chunks(E, Fl)
    if seeds is not None and len(m) > 1:
        SA, SF = seeds
        X[1:, SCAN_C] = SA[:-1]; F[1:, SCAN_C] = SF[:-1]
        c = np.arange(1, len(m))
        _seg_step(oracle, X, F, c, np.full(len(c), SCAN_C), np.zeros(len(c), dtype=np.int64), right=True)
    d = 1
    while d < SCAN_C:                                                   # up-sweep: slot k <- slot k-d (+) slot k
        up = lambda mc, d=d: (np.arange(2 * d - 1, mc, 2 * d) - d, np.arange(2 * d - 1, mc, 2 * d))
        _seg_step(oracle, X, F, *_pairs(m, up), right=True)
        d *= 2
    d = SCAN_C // 4
    while d >= 1:                                                       # down-sweep: slot k+d <- slot k (+) slot k+d
        dn = lambda mc, d=d: (np.arange(2 * d - 1, max(mc - d, 0), 2 * d), np.arange(2 * d - 1, max(mc - d, 0), 2 * d) + d)
        _seg_step(oracle, X, F, *_pairs(m, dn), right=True)
        d //= 2
    idx = np.arange(len(E))
    return X[idx // SCAN_C, idx % SCAN_C], F[idx // SCAN_C, idx % SCAN_C]


def _scan_level(oracle, E, Fl):
    if len(E) <= SCAN_C:
        return _down(oracle, E, Fl, None)
    agg = _reduce(oracle, E, Fl)
    return _down(oracle, E, Fl, _scan_level(oracle, *agg))


def scan_bracketing(oracle, rec, lin, offsets=None, group=None):
    """K6's order of operations in fp64, shaped like rec (rows outside every group zero): the records of all groups form one
    segmented scan (an element is a record and its group-start flag), reduced chunk by chunk up to a level of at most 32
    elements and rescanned down, each chunk seeded with the scanned aggregate of the chunk before."""
    n_rec = len(rec)
    out = np.zeros_like(rec)
    if offsets is None:
        b0, b1 = 0, n_rec
        starts = _group_starts(n_rec, None, group)
    else:
        b0, b1 = int(offsets[0]), int(offsets[-1])
        starts = _group_starts(n_rec, offsets, None)
    if b1 <= b0:
        return out
    i = np.arange(b0, b1)
    E = _relinearised(oracle, rec[b0:b1], lin[b0:b1], starts[b0:b1] - b0)
    out[b0:b1] = _scan_level(oracle, E, starts[b0:b1] == i)[0]
    return out
