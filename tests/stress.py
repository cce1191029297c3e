"""Seeded stress batch for the precision tests: the regimes where preintegration kernels go wrong, in one CSR batch.

numpy only.  The readings need not come from a physical trajectory (the preintegrator takes any w_m / a_m / dt), so each
regime draws them directly:

  rate100 / rate200 / rate400 / rate1000   smooth motion, |w| up to ~4 rad/s, 20-300 samples
  fast         |w| 20-35 rad/s (gyro full scale), |a| up to 16 g, 100-1000 Hz
  gaps         steps of 0.1-0.5 s among 200 Hz steps, |w| up to 10 rad/s (theta > pi in one step)
  through_pi   constant rotation about x, y, z or a random axis through a total angle of ~2 pi (every rot_2_quat case)
  bias_off     readings 0.1 rad/s and 1 m/s^2 away from the linearisation point
  grav         random q_k_lin, gravity of any direction and size, zero included (model 2 removes it per step)
  alternating  |w_hat| alternating between the small_w Taylor branch and the closed form inside one window
  threshold    |w_hat| exactly at the small_w threshold and one ulp either side (single-axis, so the norm is exact)
  band         |w_hat| in the ill-conditioned band [small_w, 0.05)
  short        lengths 0-13 with dt = 0 at the first / last sample and where the TMA ring (6 fp64 / 12 fp32 samples,
               chunks of 2 / 4) and the per-trio pre-pass (3 samples) wrap
  long         one-shot windows of 2 000 and 10 000 samples

Every window has its own linearisation point (random q_k_lin and gravity outside ``grav`` too).  Window lengths are
mixed, so window starts fall at every alignment for both dtypes, and the window count is not a multiple of the 10
windows a warp takes."""
from __future__ import annotations

import numpy as np

SMALL_W = 0.008726646
SEED = 20261015
G = 9.80665
REGIMES = ("rate100", "rate200", "rate400", "rate1000", "fast", "gaps", "through_pi", "bias_off", "grav", "alternating",
           "threshold", "band", "short", "long")
RING_POS = (2, 3, 4, 5, 6, 8, 11, 12)       # chunk (2 / 4), trio (3) and ring (6 / 12) boundaries


def _unit(rng, n):
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _smooth(rng, L, t, scale, lo=0.3):
    """L x 3 smooth random signal of magnitude ~scale."""
    c = _unit(rng, 1)[0] * scale * rng.uniform(lo, 1.0)
    A = rng.normal(size=3) * scale * 0.3
    f = rng.uniform(0.2, 3.0, 3); ph = rng.uniform(0, 2 * np.pi, 3)
    return c + A * np.sin(2 * np.pi * f * t[:, None] + ph)


def _window(rng, L, dt, w_scale=2.0, a_scale=12.0, w_hat=None):
    """One window [L, 7] with readings relative to the bias b_w (returned w_hat is added to b_w by the caller)."""
    dt = np.broadcast_to(np.asarray(dt, dtype=np.float64), (L,)).copy()
    t = np.cumsum(dt) - dt
    S = np.zeros((L, 7))
    S[:, 0:3] = _smooth(rng, L, t, w_scale) if w_hat is None else w_hat
    S[:, 3:6] = _smooth(rng, L, t, a_scale, lo=0.0) + rng.normal(0, 0.05, (L, 3))
    S[:, 6] = dt
    return S


def _lin(rng, grav_mag=G):
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    if q[3] < 0:
        q = -q
    return np.concatenate([rng.normal(0, 1e-3, 3), rng.normal(0, 1e-2, 3), q, _unit(rng, 1)[0] * grav_mag])


def _regime(rng, name, n_long):
    """List of (samples[L,7] with w relative to b_w, lin[13], offset of the true bias from lin or None)."""
    out = []
    add = lambda S, lin=None: out.append((S, _lin(rng) if lin is None else lin))
    if name.startswith("rate"):
        rate = float(name[4:])
        for _ in range(32):
            add(_window(rng, int(rng.integers(20, 301)), 1.0 / rate, w_scale=4.0))
    elif name == "fast":
        for _ in range(32):
            rate = rng.choice([100.0, 200.0, 400.0, 1000.0])
            S = _window(rng, int(rng.integers(20, 201)), 1.0 / rate, w_scale=1.0, a_scale=16 * G)
            w = S[:, 0:3]
            S[:, 0:3] = w / np.linalg.norm(w, axis=1, keepdims=True) * rng.uniform(20.0, 35.0, (len(S), 1))
            add(S)
    elif name == "gaps":
        for _ in range(24):
            L = int(rng.integers(10, 120))
            dt = np.full(L, 1 / 200.0)
            k = rng.choice(L, size=max(1, L // 20), replace=False)
            dt[k] = rng.uniform(0.1, 0.5, len(k))
            add(_window(rng, L, dt, w_scale=10.0))
    elif name == "through_pi":
        axes = [np.eye(3)[0], np.eye(3)[1], np.eye(3)[2]] + list(_unit(rng, 21))
        for i, ax in enumerate(axes):
            L = int(rng.integers(40, 160))
            sign = 1.0 if i % 2 == 0 else -1.0
            rate = 2 * np.pi * rng.uniform(0.9, 1.1) / (L / 200.0)
            add(_window(rng, L, 1 / 200.0, w_hat=sign * rate * ax + rng.normal(0, 1e-3, (L, 3))))
    elif name == "bias_off":
        for _ in range(24):
            lin = _lin(rng)
            S = _window(rng, int(rng.integers(20, 201)), 1 / 200.0)
            S[:, 0:3] += _unit(rng, 1)[0] * 0.1          # the true bias is 0.1 rad/s and 1 m/s^2 away from lin
            S[:, 3:6] += _unit(rng, 1)[0] * 1.0
            add(S, lin)
    elif name == "grav":
        for i in range(24):
            mag = (0.0, G, rng.uniform(0, 30.0))[i % 3]
            add(_window(rng, int(rng.integers(20, 201)), 1 / 200.0), _lin(rng, mag))
    elif name == "alternating":
        for _ in range(24):
            L = int(rng.integers(20, 201))
            d = _unit(rng, L)
            m = np.where(np.arange(L) % 2 == 0, rng.uniform(1e-4, 0.008, L), rng.uniform(0.06, 3.0, L))
            add(_window(rng, L, 1 / 200.0, w_hat=d * m[:, None]))
    elif name == "threshold":
        for i in range(24):
            L = int(rng.integers(20, 121))
            m = np.array([np.nextafter(SMALL_W, 0.0), SMALL_W, np.nextafter(SMALL_W, 1.0)])[rng.integers(0, 3, L)]
            w = np.zeros((L, 3)); w[np.arange(L), rng.integers(0, 3, L)] = m * rng.choice([-1.0, 1.0], L)
            lin = _lin(rng); lin[0:3] = 0.0                  # b_w = 0: w_hat = w_m exactly, |w_hat| = |component| exactly
            add(_window(rng, L, 1 / 200.0, w_hat=w), lin)
    elif name == "band":
        for _ in range(24):
            L = int(rng.integers(20, 201))
            add(_window(rng, L, 1 / 200.0, w_hat=_unit(rng, L) * rng.uniform(SMALL_W * 1.0001, 0.05, (L, 1))))
    elif name == "short":
        for L in range(14):
            places = [None, 0, L - 1] + [p for p in RING_POS if p < L]
            for p in (places if L else [None]):
                S = _window(rng, L, rng.choice([1 / 200.0, 1 / 400.0]))
                if p is not None and L:
                    S[p, 6] = 0.0
                add(S)
    elif name == "long":
        for L in (2000, 2000, 10000)[:n_long]:
            add(_window(rng, L, 1 / 200.0, w_scale=2.0))
    else:
        raise ValueError(name)
    return out


def split_for_continuation(samples, offsets):
    """Cut every window in two at a chunk / trio / ring boundary (cycling through RING_POS; some windows at 0 or at their end,
    so one of the two calls gets no samples).  Returns (first samples, first offsets, rest samples, rest offsets)."""
    n = len(offsets) - 1
    lens = np.diff(offsets)
    choice = np.array(list(RING_POS) + [0, 10 ** 9])
    cut = np.minimum(choice[np.arange(n) % len(choice)], lens)
    A = [samples[offsets[i]:offsets[i] + cut[i]] for i in range(n)]
    B = [samples[offsets[i] + cut[i]:offsets[i + 1]] for i in range(n)]
    oa = np.zeros(n + 1, dtype=np.int64); oa[1:] = np.cumsum(cut)
    ob = np.zeros(n + 1, dtype=np.int64); ob[1:] = np.cumsum(lens - cut)
    cat = lambda L: np.ascontiguousarray(np.concatenate(L).reshape(-1, 7))
    return cat(A), oa, cat(B), ob


def make_batch(seed=SEED, regimes=REGIMES, n_long=3):
    """(samples[N,7], offsets[n+1] int64, lin[n,13], regime[n] str).  The readings are w_hat + b_w where b_w is the window's
    linearisation point, so each regime's |w_hat| is what the kernel sees."""
    rng = np.random.default_rng(seed)
    wins, lins, tags = [], [], []
    for name in regimes:
        for S, lin in _regime(rng, name, n_long):
            S = S.copy()
            S[:, 0:3] += lin[0:3]
            S[:, 3:6] += lin[3:6]
            wins.append(S); lins.append(lin); tags.append(name)
    if len(wins) % 10 == 0:                           # keep the last warp of windows partial
        S, lin = _regime(rng, "rate200", 0)[0]
        S = S.copy(); S[:, 0:3] += lin[0:3]; S[:, 3:6] += lin[3:6]
        wins.append(S); lins.append(lin); tags.append("rate200")
    off = np.zeros(len(wins) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(w) for w in wins])
    return np.ascontiguousarray(np.concatenate(wins)), off, np.ascontiguousarray(np.stack(lins)), np.array(tags)
