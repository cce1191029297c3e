"""Placement batch for the preintegration kernels: every stress window (tests/stress.py) copied into every thread slot that a
kernel indexes by position, in one CSR batch.

numpy only.  A window's record must not depend on where the batch puts it.  The kernels index shared memory, TMA staging and
mbarriers by thread, so each slot class is worth reaching:

  round 1 (k_preintegrate, one lane per window; imu_avg and model 2 with analytic Jacobians): with n = sms * 128 + r windows,
      ceil(n / sms) exceeds every tile capacity S, so the CTA holds S windows (72 / 80 / 112 / 128 for model 2 fp64, model 1
      fp64, model 2 fp32, model 1 fp32), the grid is at least one full wave plus a partial last CTA.  For each S, every
      window sits at a thread of 16-31 and in every later warp of the CTA.  Threads 0 and S - 1 have one slot per CTA, fewer
      than there are windows: they hold as many distinct windows as there are CTAs (less SLACK), of every regime.  The
      partial last CTA of each S holds distinct windows of every regime.
  tri-lane (ten windows per warp): every window sits in each of the ten trio slots, once in a warp whose nine neighbours all
      have <= 13 samples (the warp stops early) and once in a warp that holds the 10 000-sample window (its neighbours run
      thousands of null steps after their last sample).
  start alignment: every non-empty window starts at each offset mod 4, so at both 16-byte phases in fp64 and at all four
      `shift` values of the TMA staging in fp32.

The 10 000-sample window appears in ~50 warps, all at the front of the batch, so that they share the first wave of every
kernel; the 2 000-sample windows appear about twenty times.  make_placement_batch() asserts the coverage."""
from __future__ import annotations

import numpy as np

import stress

ROUND1_S = (72, 80, 112, 128)        # windows per CTA of k_preintegrate at capacity (preintegrate.cu, Tile<MODEL, T>::S)
TRI = 10                             # windows per warp of the tri-lane kernel (preintegrate_tri.cu, TRI_WPW)
SHORT = 13                           # neighbours of a "quiet" warp have at most this many samples
SLACK = 16                           # one-slot-per-CTA classes may repeat this many windows (blocks A and B place by warp, not by CTA)
FRONT = 4500                         # every copy of the 10 000-sample window lies before this position (inside the first wave)
R_CANDIDATES = range(21, 128, 2)


def round1_classes(S, tid):
    """Slot classes of thread tid of a CTA of S windows: thread 0, a thread of 16-31, warp k >= 1, thread S - 1."""
    out = []
    if tid == 0:
        out.append("t0")
    if 16 <= tid < 32:
        out.append("t16")
    if tid >= 32:
        out.append(f"w{tid // 32}")
    if tid == S - 1:
        out.append("last")
    return out


def _all_round1_classes(S):
    return ["t0", "t16"] + [f"w{k}" for k in range(1, (S + 31) // 32)] + ["last"]


def pick_r(sms):
    """The smallest odd r < 128 such that r is not a multiple of 10 or of any S and the partial last CTA of every S (and the
    last tri-lane warp) is partial and holds at least one window of each regime."""
    for r in R_CANDIDATES:
        n = sms * 128 + r
        if r % 10 and n % 10 and all(r % S and n % S >= len(stress.REGIMES) for S in ROUND1_S):
            return r
    raise AssertionError(f"no remainder fits {sms} SMs")


class _Columns:
    """Requirement columns: (S, class) of round 1, the trio slot, the start offset mod 4, the quiet warp, the 10k warp."""

    def __init__(self):
        names = [(S, c) for S in ROUND1_S for c in _all_round1_classes(S)]
        names += [("slot", k) for k in range(TRI)] + [("phase", k) for k in range(4)] + [("quiet",), ("big",)]
        self.names = names
        self.index = {nm: i for i, nm in enumerate(names)}

    def at(self, g, start):
        cols = [self.index[(S, c)] for S in ROUND1_S for c in round1_classes(S, g % S)]
        cols.append(self.index[("slot", g % TRI)])
        cols.append(self.index[("phase", start % 4)])
        return cols


def _layout(lens, tags, sms):
    """Distinct window index per position (the placement order)."""
    m = len(lens)
    r = pick_r(sms)
    n = sms * 128 + r
    big = int(np.flatnonzero(lens == 10000)[0])
    long_ = lens >= 2000
    short = [int(w) for w in np.flatnonzero(lens <= SHORT)]
    C = _Columns()
    need = np.ones((m, len(C.names)), dtype=bool)
    need[lens == 0, C.index[("phase", 0)]:C.index[("phase", 3)] + 1] = False     # an empty window reads nothing
    order, start = [], 0

    def place(w, extra=()):
        nonlocal start
        cols = C.at(len(order), start) + [C.index[e] for e in extra]
        need[w, cols] = False
        order.append(w)
        start += int(lens[w])

    # block A: warps holding the 10k window (at slot k % 10 of the k-th such warp) and nine others, every window in turn
    others = [w for w in range(m) if w != big]
    groups = [others[i:i + TRI - 1] for i in range(0, len(others), TRI - 1)]
    groups[-1] = groups[-1] + others[:TRI - 1 - len(groups[-1])]
    for k, grp in enumerate(groups):
        slot = k % TRI
        for w in grp[:slot] + [big] + grp[slot:]:
            place(w, [("big",)])
    # block B: quiet warps.  Each longer window with nine short neighbours (the 10k one first, next to block A), then the short
    # windows ten at a time
    sc = 0
    for k, w in enumerate([big] + [w for w in range(m) if lens[w] > SHORT and w != big]):
        nb = [short[(sc + j) % len(short)] for j in range(TRI - 1)]
        sc += TRI - 1
        slot = k % TRI
        for x in nb[:slot] + [w] + nb[slot:]:
            place(x, [("quiet",)])
    for i in range(0, len(short), TRI):
        for j in range(TRI):
            place(short[(i + j) % len(short)], [("quiet",)])
    # the last positions: the partial last CTA of every S holds distinct windows, the very last ones one of each regime
    tail = max(n % S for S in ROUND1_S)
    reps = [int(np.flatnonzero((tags == reg) & (lens < 10000))[0]) for reg in stress.REGIMES]
    # block C: greedily the window that meets the most open requirements at this position; fillers are ordinary windows in turn
    copies = np.bincount(np.asarray(order), minlength=m)
    in_tail = set()
    filler = np.flatnonzero(~long_)
    while len(order) < n:
        g = len(order)
        if g >= n - len(reps):
            w = reps[g - (n - len(reps))]
        else:
            cols = C.at(g, start)
            score = need[:, cols].sum(axis=1).astype(np.int64)
            if g >= FRONT:
                score[big] = -1
            if g >= n - tail:
                score[list(in_tail | set(reps))] = -1
            best = score.max()
            if g < FRONT and np.any(score[long_] > 0):        # the long windows first, while they still share the first wave
                w = int(np.flatnonzero(long_)[np.argmax(score[long_])])
            elif best > 0:
                cand = np.flatnonzero(score == best)
                cand = cand[np.lexsort((copies[cand], long_[cand]))]
                w = int(cand[0])
            else:
                pool = filler if g < n - tail else np.array([x for x in filler if score[x] >= 0])
                w = int(pool[np.argmin(copies[pool])])
        if g >= n - tail:
            in_tail.add(w)
        place(w)
        copies[w] += 1
    return np.asarray(order, dtype=np.int64), r


def coverage(idx, lens, tags, sms):
    """Assert the placement coverage of the module docstring for the order idx (distinct window per position)."""
    n, m = len(idx), len(lens)
    r = n - sms * 128
    assert 0 < r < 128 and r % 10 and n % TRI, (n, r)
    off = np.zeros(n + 1, dtype=np.int64)
    off[1:] = np.cumsum(lens[idx])
    pos = np.arange(n)
    assert set(idx.tolist()) == set(range(m)), "a stress window is missing"
    for S in ROUND1_S:
        assert r % S and n % S, (S, n)
        assert -(-n // sms) > S, "the round-1 kernel would not run at capacity"
        tid = pos % S
        for c in _all_round1_classes(S):
            hit = np.zeros(m, dtype=bool)
            sel = [g for g in range(S) if c in round1_classes(S, g)]
            at = np.isin(tid, sel)
            hit[idx[at]] = True
            if c in ("t0", "last"):      # one slot per CTA: fewer slots than windows, so as many distinct windows as slots, every regime
                assert hit.sum() >= min(at.sum(), m) - SLACK and set(tags[hit]) == set(stress.REGIMES), \
                    f"S = {S}: {hit.sum()} distinct windows in {at.sum()} slots of class {c}"
            else:
                assert hit.all(), f"S = {S}: windows {np.flatnonzero(~hit)[:8]} never at slot class {c}"
        last = idx[n - n % S:]
        assert len(set(last.tolist())) == len(last), f"S = {S}: the partial last CTA repeats a window"
        assert set(tags[last]) == set(stress.REGIMES), f"S = {S}: the partial last CTA misses a regime"
    for k in range(TRI):
        assert set(idx[pos % TRI == k].tolist()) == set(range(m)), f"a window never sits in trio slot {k}"
    warps = np.arange(0, n - n % TRI, TRI)
    W = idx[warps[:, None] + np.arange(TRI)]
    quiet = (lens[W] <= SHORT).sum(axis=1)
    for w in range(m):
        rows = np.flatnonzero((W == w).any(axis=1))
        assert np.any(quiet[rows] - (lens[w] <= SHORT) >= TRI - 1), f"window {w} never has nine short neighbours"
        assert np.any((lens[W[rows]] == 10000).any(axis=1)), f"window {w} never shares a warp with the 10 000-sample window"
        ph = set((off[:-1][idx == w] % 4).tolist())
        assert lens[w] == 0 or ph == {0, 1, 2, 3}, f"window {w} starts only at offsets {ph} mod 4"
    counts = np.bincount(idx, minlength=m)
    assert counts[lens == 10000].max() <= 60 and counts[lens == 2000].max() <= 24, counts[lens >= 2000]
    assert np.all(np.flatnonzero(idx == np.flatnonzero(lens == 10000)[0]) < min(FRONT, sms * min(ROUND1_S))), \
        "a 10 000-sample copy is outside the first wave"
    return counts


def make_placement_batch(sms, seed=stress.SEED):
    """(samples[N,7], offsets[n+1], lin[n,13], idx[n]) with n = sms * 128 + r: position g holds stress window idx[g] of
    stress.make_batch(seed) (same samples and linearisation point)."""
    S0, off0, L0, tags = stress.make_batch(seed)
    lens = np.diff(off0)
    idx, _ = _layout(lens, tags, sms)
    coverage(idx, lens, tags, sms)
    off = np.zeros(len(idx) + 1, dtype=np.int64)
    off[1:] = np.cumsum(lens[idx])
    src = np.concatenate([np.arange(off0[w], off0[w + 1]) for w in idx])
    samples = np.ascontiguousarray(S0[src])
    assert samples.nbytes // 2 >= 16 << 20, "the fp32 batch must take the chunked host pipeline"
    return samples, off, np.ascontiguousarray(L0[idx]), idx
