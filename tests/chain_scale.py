"""Layouts at the sizes where the chain-side kernels leave their first grid-stride pass (tests/test_chain_scale.py, DESIGN.md
section 5).  CPU only, like placement_stress.py.

The launch geometry of each kernel is restated as a function of the SM count; every builder asserts that its batch reaches the
second path for 132 SMs (H100 SXM) and 114 (H100 PCIe), and the GPU tests assert it again for the device they run on."""
import fractions

import numpy as np

SMS = (132, 114)


# ------------------------------------------------------------------------------------------------------------------
# launch geometry
# ------------------------------------------------------------------------------------------------------------------

def fold_pass(sms, n_chains):
    """States per grid-stride pass of k_state_prior_fold on device offsets: max(sms * 32, ceil(C / 4)) CTAs of 4 warps, one warp
    per state (state_priors.cu, state_priors_fold_launch)."""
    return 4 * max(sms * 32, (n_chains + 3) // 4)


def chain_ids_pass(sms, n_states):
    """States per grid-stride pass of k_chain_ids: min(ceil(N / 256), sms * 8) CTAs of 256 threads (solve.cu, chains_solve_launch)."""
    return 256 * min((n_states + 255) // 256, sms * 8)


def relin_scan_per(n_factors):
    """(CTAs of 256 factors, CTA totals each of the 256 threads of k_relin_scan_blocks folds) (relinearize.cu, k_relin_scan_blocks)."""
    nb = (n_factors + 255) // 256
    return nb, (nb + 255) // 256


def relin_copy_pass(sms, n_sel):
    """Windows per grid-stride pass of k_relin_gather / k_relin_scatter: min(ceil(n / 8), sms * 8) CTAs of 8 warps
    (relinearize.cu, relin_gather_launch / relin_scatter_launch)."""
    return 8 * min((n_sel + 7) // 8, sms * 8)


def _boundaries(pass_size, n):
    return list(range(pass_size, n, pass_size))


def _layout_with(rng, N, max_len, inside=(), single=()):
    """Chain offsets over N states, chain lengths 1 .. max_len, except that no chain starts inside each (lo, hi) of `inside` (so
    one chain holds lo-1 .. hi) and that every state of `single` is a chain of its own."""
    cut = np.zeros(N + 1, bool)
    cut[0] = cut[N] = True
    pos = 0
    while pos < N:
        pos += int(rng.integers(1, max_len + 1))
        cut[min(pos, N)] = True
    for lo, hi in inside:
        cut[lo:hi + 1] = False
    for k in single:
        cut[k] = cut[k + 1] = True
    return np.flatnonzero(cut).astype(np.int64)


def _chain_of(offs, k):
    return int(np.searchsorted(offs, k, side="right") - 1)


# ------------------------------------------------------------------------------------------------------------------
# the fold: >= 3 grid-stride passes, chains and prior counts at the pass boundaries
# ------------------------------------------------------------------------------------------------------------------

FOLD_STATES = 4 * 16896 + 1200


def fold_batch(seed=0, extra_sms=()):
    """(offs [C+1], priors per state [N]) of FOLD_STATES states.  At every pass boundary B of every SM count: the chains alternate
    between one whose last factor straddles B (state B-1 its second to last, B its last: the f that the left state's warp writes
    takes priors from both passes), one holding B-4 .. B+4, and single-state chains at B-1 and B.  States B-3 .. B+2 carry 5, 0, 1,
    5, 1, 0 priors, the others 0 or 1 (one in three)."""
    rng = np.random.default_rng(seed)
    N = FOLD_STATES
    sms_all = tuple(dict.fromkeys(tuple(SMS) + tuple(extra_sms)))
    kind = {}                                                      # boundary -> kind, cycling over each SM count's boundaries
    for s in sms_all:                                              # (about 4 400 chains: a pass is sms * 128 states)
        for j, B in enumerate(_boundaries(fold_pass(s, 1), N)):
            kind.setdefault(B, j % 3)
    inside, single = [], []
    for B, kd in kind.items():
        if kd == 0:                                                # a chain ending at B from B-4 or before, a single state at B+1
            inside.append((B - 3, B))
            single.append(B + 1)
        elif kd == 1:
            inside.append((B - 3, B + 4))
        else:
            single += [B - 1, B]
    offs = _layout_with(rng, N, 30, inside, single)
    counts = (rng.random(N) < 1 / 3).astype(np.int64)
    for B in kind:
        counts[B - 3:B + 3] = [5, 0, 1, 5, 1, 0]
    check_fold(offs, counts, sms_all)
    return offs, counts


def check_fold(offs, counts, sms_list):
    N, C = int(offs[-1]), len(offs) - 1
    assert np.all(np.diff(offs) >= 1)
    for s in sms_list:
        P = fold_pass(s, C)
        assert -(-N // P) >= 3, (s, P)
        kinds = set()
        for B in _boundaries(P, N):
            c = _chain_of(offs, B)
            lo, hi = int(offs[c]), int(offs[c + 1])
            here = {k for k, ok in (("b2", hi == B + 1 and lo <= B - 1), ("inside", lo < B - 1 and hi > B + 1),
                                    ("single", hi - lo == 1 and offs[c - 1] == B - 1)) if ok}
            assert len(here) == 1, (s, B, here)                    # one of the three layouts at every boundary
            kinds |= here
            assert set(counts[B - 3:B + 3].tolist()) == {0, 1, 5}
        assert kinds == {"b2", "inside", "single"}, (s, kinds)


# ------------------------------------------------------------------------------------------------------------------
# the isolated solve: k_chain_ids over two full passes and a partial third
# ------------------------------------------------------------------------------------------------------------------

def solve_states(sms_list=SMS):
    """N = 2 cap + 1234 for the largest cap = sms * 8 * 256 of the SM counts: at least three passes of k_chain_ids for each."""
    N = 2 * max(chain_ids_pass(s, 1 << 40) for s in sms_list) + 1234
    for s in sms_list:
        assert -(-N // chain_ids_pass(s, N)) >= 3, s
    return N


def solve_layout(seed, sms_list=SMS):
    """(offs, N): chains of 1 .. 40 states, one straddling every pass boundary of k_chain_ids of every SM count (three states on
    each side)."""
    rng = np.random.default_rng(seed)
    N = solve_states(sms_list)
    bounds = sorted({b for s in sms_list for b in _boundaries(chain_ids_pass(s, N), N)})
    offs = _layout_with(rng, N, 40, [(B - 2, B + 3) for B in bounds])
    for B in bounds:
        c = _chain_of(offs, B)
        assert offs[c] < B - 1 and offs[c + 1] > B + 1
    return offs, N


# ------------------------------------------------------------------------------------------------------------------
# re-preintegration: the selection laid out per CTA of 256 factors
# ------------------------------------------------------------------------------------------------------------------

RELIN_FACTORS = 274 * 256 + 57                                     # 275 CTAs, the last partial: 2 CTA totals per scan thread


def relin_plan(seed=0):
    """The selection mask of RELIN_FACTORS factors, per CTA of 256: CTAs 8..13 empty (the whole ranges of scan threads 4..6),
    CTAs 21..24 empty (a run across the ranges of threads 10..12), CTAs whose only selected factor is at thread 0 and others at
    thread 255, full CTAs, the partial last CTA with its last factor selected, the rest about half selected."""
    rng = np.random.default_rng(seed)
    n = RELIN_FACTORS
    nb, per = relin_scan_per(n)
    sel = rng.random(n) < 0.5
    cta = lambda b: slice(256 * b, min(256 * (b + 1), n))
    for b in list(range(8, 14)) + list(range(21, 25)) + [60, 61, 62]:
        sel[cta(b)] = False
    for b in (30, 31, 90, 200):                                    # only thread 0
        sel[cta(b)] = False; sel[256 * b] = True
    for b in (32, 91, 201, 202):                                   # only thread 255
        sel[cta(b)] = False; sel[256 * b + 255] = True
    for b in (40, 41, 100, 150, 273):
        sel[cta(b)] = True
    sel[-1] = True
    check_relin(sel)
    return sel


def check_relin(sel):
    n = len(sel)
    nb, per = relin_scan_per(n)
    assert per >= 2 and n % 256 and sel[-1]
    blk = np.array([sel[256 * b:256 * (b + 1)].sum() for b in range(nb)])
    full = np.array([min(256, n - 256 * b) for b in range(nb)])
    ranges = [(t * per, min(t * per + per, nb)) for t in range(256) if t * per < nb]
    assert any(blk[lo:hi].sum() == 0 for lo, hi in ranges)                                    # a scan thread with nothing
    assert any(blk[b] == 0 and blk[b + 1] == 0 and (b + 1) % per == 0 for b in range(nb - 1))  # an empty run across two ranges
    one = [b for b in range(nb) if blk[b] == 1]
    assert any(sel[256 * b] for b in one) and any(sel[256 * b + 255] for b in one if 256 * b + 255 < n)
    assert np.any(blk == full)
    for s in SMS:
        assert sel.sum() > 2 * relin_copy_pass(s, 1 << 40), s


# ------------------------------------------------------------------------------------------------------------------
# ties of the selection rule's squared norms
# ------------------------------------------------------------------------------------------------------------------

def _fma(a, b, c):
    """fma(a, b, c) rounded once, from exact rationals."""
    return float(fractions.Fraction(a) * fractions.Fraction(b) + fractions.Fraction(c))


def contracted(x, y, z):
    """The two ways nvcc may contract x*x + y*y + z*z: fma(z, z, fma(x, x, y*y)) and fma(z, z, fma(y, y, x*x))."""
    return _fma(z, z, _fma(x, x, y * y)), _fma(z, z, _fma(y, y, x * x))


def np_norm2(v):
    """numpy's (x^2 + y^2) + z^2, the rule's order."""
    v = np.asarray(v, dtype=np.float64)
    return (v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1]) + v[..., 2] * v[..., 2]


def tie_cases(tol, n_each, seed):
    """(at, above): 3-vectors whose numpy squared norm is exactly tol*tol (not selected), and exactly its successor (selected).
    Each list holds n_each vectors whose contracted sums, both ways, fall on the other side of the rule (above tol*tol for `at`,
    at or below it for `above`), then n_each whose contracted sums agree with numpy."""
    rng = np.random.default_rng(seed)
    T = tol * tol
    targets = (T, np.nextafter(T, np.inf))
    out = [([], []), ([], [])]                                     # [target][sensitive, plain]
    while any(len(lst) < n_each for pair in out for lst in pair):
        m = 20000
        d = rng.normal(size=(m, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        v = d * tol
        for t_i, tgt in enumerate(targets):
            p = v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]
            z0 = np.sqrt(np.maximum(tgt - p, 0.0))
            for step in (0, 1, -1, 2, -2):
                z = z0.copy()
                for _ in range(abs(step)):
                    z = np.nextafter(z, np.inf if step > 0 else -np.inf)
                w = np.c_[v[:, 0], v[:, 1], z]
                hit = np.flatnonzero(np_norm2(w) == tgt)
                # long double (64-bit significand) estimates of both contractions pick the candidates the exact check confirms
                L = w[hit].astype(np.longdouble)
                f2 = lambda a, b, c: (a * b + c).astype(np.float64).astype(np.longdouble)
                est = [f2(L[:, 2], L[:, 2], f2(L[:, 0], L[:, 0], (L[:, 1] * L[:, 1]).astype(np.float64))),
                       f2(L[:, 2], L[:, 2], f2(L[:, 1], L[:, 1], (L[:, 0] * L[:, 0]).astype(np.float64)))]
                odd = (est[0] != tgt) | (est[1] != tgt)
                for q in np.r_[hit[odd], hit[~odd][:n_each]]:
                    x, y, zz = (float(a) for a in w[q])
                    c = contracted(x, y, zz)
                    flips = all(ci > T for ci in c) if t_i == 0 else all(ci <= T for ci in c)
                    same = all(ci == tgt for ci in c)
                    lst = out[t_i][0] if flips else (out[t_i][1] if same else None)
                    if lst is not None and len(lst) < n_each:
                        lst.append((x, y, zz))
    return [np.array(a + b) for a, b in out]


# ------------------------------------------------------------------------------------------------------------------
# block cyclic reduction: the level pattern of a chain, and the tiled LM batch
# ------------------------------------------------------------------------------------------------------------------

def bcr_pattern(o, L):
    """What the isolated solve does to a chain of L states at global offset o, level by level until the chain has one node left: per
    surviving state, (odd: eliminated at this level, has_left, has_right).  Level l keeps the states k with k mod 2^l = 0, and node
    k >> l is odd or even (solve.cu, chains_solve_launch)."""
    out, nodes, lev = [], list(range(o, o + L)), 0
    while len(nodes) > 1:
        out.append(tuple(((k >> lev) & 1, i > 0, i < len(nodes) - 1) for i, k in enumerate(nodes)))
        nodes = [k for k in nodes if not (k >> lev) & 1]
        lev += 1
    return tuple(out)


def bcr_modulus(L, span=256):
    """The smallest M with bcr_pattern(o, L) = bcr_pattern(o + M, L) for every offset o below span."""
    P = [bcr_pattern(o, L) for o in range(2 * span)]
    return next(m for m in range(1, span) if all(P[o] == P[o + m] for o in range(span)))


TILE = 64                                                          # every bcr_modulus of a length <= 64 divides it
LM_LENGTHS = [1, 2, 3, 5, 8, 16, 17, 30, 31, 32, 33, 64] * 3 + [4, 6, 9, 12]


def lm_batch(lengths=LM_LENGTHS, sms_list=SMS, n_states=300_000, seed=0):
    """Copies of the distinct chains `lengths` tiled to at least n_states states: returns (src [n] distinct chain of each copy, offs
    [n+1], cls [n] class id, nan_copy).  Copies of a class start at offsets congruent mod TILE, so that the solve does the same
    arithmetic to each.  Three blocks of all distinct chains (three orders, the long ones twice), each padded with single-state chains to a multiple of TILE,
    fill the batch at TILE-aligned offsets.  At every fold-pass and k_chain_ids boundary of every SM count sits either a chain of
    >= 2 states straddling it (the chains taking turns; at every other one the chain's last state is the first of the next pass) or
    a pair of single-state chains, one on each side.  One copy beyond every k_chain_ids boundary, between two block copies, is the
    NaN chain."""
    rng = np.random.default_rng(seed)
    lengths = np.asarray(lengths)
    D = len(lengths)
    orders = [np.r_[1:D, 0], rng.permutation(D), rng.permutation(D)]
    one = int(np.flatnonzero(lengths == 1)[0])
    extra = list(np.flatnonzero(lengths >= 30))                    # the long chains twice: about 23 states per chain on average
    blocks = []
    for od in orders:
        b = list(od) + extra
        gap = (-int(lengths[b].sum())) % TILE
        for c in np.argsort(-lengths, kind="stable"):              # pad to a multiple of TILE with distinct chains, longest first
            if lengths[c] <= gap:
                b.append(int(c)); gap -= int(lengths[c])
        blocks.append(b)
    orders = [list(b) for b in blocks]
    bounds = {}
    for s in sms_list:
        for j, B in enumerate(range(s * 128, n_states, s * 128)):      # fold passes (asserted below: fewer than s * 128 chains)
            bounds.setdefault(B, j % 2)
    ids = sorted({B for s in sms_list for B in range(chain_ids_pass(s, 1 << 40), n_states, chain_ids_pass(s, 1 << 40))})
    multi = [c for c in range(D) if lengths[c] >= 2]
    by_len = [int(c) for c in np.argsort(-lengths, kind="stable")]
    src, start = [], []
    pos, nb, turn = 0, 0, 0
    events = sorted(bounds)

    def put(c):
        nonlocal pos
        src.append(int(c)); start.append(pos); pos += int(lengths[c])

    def fill_to(target):                                           # whole blocks while they fit, then single-state chains
        nonlocal nb
        while pos % TILE:
            put(one)
        while pos + sum(lengths[blocks[nb % 3]]) <= target:
            for c in blocks[nb % 3]:
                put(c)
            nb += 1
        while pos < target:                                        # the rest with the longest distinct chains that fit
            put(next(c for c in by_len if lengths[c] <= target - pos))

    nan_at = []
    for B in events:
        kind = bounds[B]
        if B in ids:                                               # the NaN chain, between two block copies, then its boundary
            fill_to(B - 3 * TILE - 16)
            fill_to(pos + TILE - pos % TILE if pos % TILE else pos)
            for c in blocks[nb % 3]:
                put(c)
            nb += 1
        if kind == 0 or B in ids:
            c = multi[turn % len(multi)]
            turn += 1
            L = int(lengths[c])
            lead = L - 1 if turn % 2 else L // 2
            fill_to(B - lead)
            put(c)
        else:
            fill_to(B - 1)
            put(one); put(one)
    fill_to(n_states)
    while pos % TILE:
        put(one)
    for c in blocks[nb % 3]:                                       # the batch ends with a block copy
        put(c)
    src = np.array(src)
    offs = np.r_[start, pos].astype(np.int64)
    key = {}
    cls = np.array([key.setdefault((int(c), int(o) % TILE), len(key)) for c, o in zip(src, offs[:-1])])
    for B in ids:                                                  # the NaN copy: the second copy of a long block chain past B
        cand = [i for i in range(1, len(src) - 1) if offs[i] > B + 2 * TILE and lengths[src[i]] >= 3 and src[i - 1] != one and src[i + 1] != one]
        nan_at.append(cand[0])
    check_lm_batch(lengths, src, offs, cls, nan_at, sms_list)
    return src, offs, cls, nan_at


def check_lm_batch(lengths, src, offs, cls, nan_at, sms_list):
    n, N = len(src), int(offs[-1])
    D = len(lengths)
    assert np.array_equal(np.diff(offs), lengths[src])
    for c, o in zip(src, offs[:-1]):                               # copies of a class start at congruent offsets
        assert bcr_pattern(int(o), int(lengths[c])) == bcr_pattern(int(o) % TILE + TILE, int(lengths[c]))
    for c in range(D):
        mine = np.flatnonzero(src == c)
        assert len(set(cls[mine])) >= 2 or lengths[c] == 1, c  # several residue classes
        assert set(mine % 4) == {0, 1, 2, 3}, c                  # every warp slot of the per-chain kernels
    assert lengths[src[0]] > 1 and lengths[src[-1]] > 1 and src[0] != src[-1]
    for s in sms_list:
        P = fold_pass(s, n)
        assert n < s * 128 and -(-N // P) >= 3, s
        for c in range(D):                                         # copies in the first, second and last fold pass
            st = offs[:-1][src == c]
            assert {0, 1, (N - 1) // P} <= set((st // P).tolist()), (s, c)
        B1 = chain_ids_pass(s, N)
        assert N > B1
        for c in range(D):
            assert np.any(offs[:-1][src == c] > B1), (s, c)       # copies beyond the first pass of k_chain_ids
        kinds = set()
        for B in list(range(P, N, P)) + [B1]:
            i = int(np.searchsorted(offs, B, side="right") - 1)
            lo, hi = int(offs[i]), int(offs[i + 1])
            if lo < B:
                kinds.add("b2" if hi == B + 1 else "straddle")
            else:
                assert hi - lo == 1 and offs[i - 1] == B - 1, (s, B)  # a single-state chain on each side
                kinds.add("single")
        assert kinds == {"b2", "straddle", "single"}, (s, kinds)
        i = int(np.searchsorted(offs, B1, side="right") - 1)
        assert offs[i] < B1 < offs[i + 1], s                       # a chain straddles the k_chain_ids boundary
    for q in nan_at:
        assert 0 < q < n - 1 and lengths[src[q]] >= 3
