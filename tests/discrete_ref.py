"""numpy statement of discrete (Forster) preintegration into a model-1 record (CPI_FLAG_DISCRETE, DESIGN.md section 3n).

Vectorised over windows and parameterised by dtype, so that the same code runs in float64 and in np.longdouble.  Per step, with
w_hat = w - b_w_lin, a_hat = a - b_a_lin (the mean of the step's two ends with imu_avg), Rs = Exp(-[w_hat dt]x) and J_r(w_hat dt)
in model 1's closed forms and small-w branch, and R = R_k2tau at the step's start:

    R' = Rs R   beta' = beta + R^T a_hat dt   alpha' = alpha + beta dt + 1/2 R^T a_hat dt^2
    J_q' = Rs J_q + J_r dt   J_b' = J_b + R^T[a_hat]x J_q dt   J_a' = J_a + J_b dt + 1/2 R^T[a_hat]x J_q dt^2
    H_b' = H_b - R^T dt      H_a' = H_a + H_b dt - 1/2 R^T dt^2
    P' = Phi P Phi^T + Q  (record order theta, b_g, v, b_a, p), stored exactly symmetric."""
import numpy as np

SMALL_W = 0.008726646
TH, BG, V, BA, PP = (slice(0, 3), slice(3, 6), slice(6, 9), slice(9, 12), slice(12, 15))


def skew(v):
    o = np.zeros(v.shape[:-1] + (3, 3), dtype=v.dtype)
    o[..., 0, 1], o[..., 0, 2], o[..., 1, 2] = -v[..., 2], v[..., 1], -v[..., 0]
    o[..., 1, 0], o[..., 2, 0], o[..., 2, 1] = v[..., 2], -v[..., 1], v[..., 0]
    return o


def step_factors(wh, dt):
    """(Rs, J_r) of model 1's closed forms: Rs = I - a W + b W^2, J_r = I - c1 dt W + c2 dt^2 W^2, W = [w_hat x]."""
    dtype = wh.dtype
    mag = np.sqrt((wh[:, 0] * wh[:, 0] + wh[:, 1] * wh[:, 1]) + wh[:, 2] * wh[:, 2])
    th = mag * dt
    small = mag < SMALL_W
    one = dtype.type(1)
    with np.errstate(divide="ignore", invalid="ignore"):
        im = np.where(small, 0, one / np.where(small, one, mag))
        ith = np.where(small, 0, one / np.where(small, one, th))
    sn, cs = np.sin(th), np.cos(th)
    a = np.where(small, dt, sn * im)
    b = np.where(small, dt * dt * dtype.type(0.5), (one - cs) * (im * im))
    c1 = np.where(small, dtype.type(0.5), (one - cs) * (ith * ith))
    c2 = np.where(small, one / 6, (th - sn) * (ith * ith * ith))
    W = skew(wh)
    W2 = W @ W
    I = np.eye(3, dtype=dtype)
    Rs = I - a[:, None, None] * W + b[:, None, None] * W2
    Jr = I - (c1 * dt)[:, None, None] * W + (c2 * dt * dt)[:, None, None] * W2
    return Rs, Jr


def rot_2_quat(R):
    """JPL [x y z w] of a batch of rotations (quat_ops.h rot_2_quat, the kernels' branch order)."""
    q = np.zeros(R.shape[:-2] + (4,), dtype=R.dtype)
    for n in range(R.shape[0]):
        r = R[n]
        T = r[0, 0] + r[1, 1] + r[2, 2]
        if r[0, 0] >= T and r[0, 0] >= r[1, 1] and r[0, 0] >= r[2, 2]:
            x = np.sqrt((1 + 2 * r[0, 0] - T) / 4); s = 1 / (4 * x)
            v = [x, s * (r[0, 1] + r[1, 0]), s * (r[0, 2] + r[2, 0]), s * (r[1, 2] - r[2, 1])]
        elif r[1, 1] >= T and r[1, 1] >= r[0, 0] and r[1, 1] >= r[2, 2]:
            y = np.sqrt((1 + 2 * r[1, 1] - T) / 4); s = 1 / (4 * y)
            v = [s * (r[0, 1] + r[1, 0]), y, s * (r[1, 2] + r[2, 1]), s * (r[2, 0] - r[0, 2])]
        elif r[2, 2] >= T and r[2, 2] >= r[0, 0] and r[2, 2] >= r[1, 1]:
            z = np.sqrt((1 + 2 * r[2, 2] - T) / 4); s = 1 / (4 * z)
            v = [s * (r[0, 2] + r[2, 0]), s * (r[1, 2] + r[2, 1]), z, s * (r[0, 1] - r[1, 0])]
        else:
            w = np.sqrt((1 + T) / 4); s = 1 / (4 * w)
            v = [s * (r[1, 2] - r[2, 1]), s * (r[2, 0] - r[0, 2]), s * (r[0, 1] - r[1, 0]), w]
        v = np.array(v, dtype=R.dtype)
        if v[3] < 0:
            v = -v
        q[n] = v / np.sqrt(np.sum(v * v))
    return q


class State:
    """The whole state of the recursion for n windows (everything a model-1 record holds)."""

    def __init__(self, n, dtype=np.float64, records=None):
        dt_ = np.dtype(dtype)
        if records is None:
            self.R = np.broadcast_to(np.eye(3, dtype=dt_), (n, 3, 3)).copy()
            self.al, self.be, self.DT = np.zeros((n, 3), dt_), np.zeros((n, 3), dt_), np.zeros(n, dt_)
            self.Jq, self.Ja, self.Jb, self.Ha, self.Hb = (np.zeros((n, 3, 3), dt_) for _ in range(5))
            self.P = np.zeros((n, 15, 15), dt_)
        else:
            r = np.asarray(records).astype(dt_)
            m = lambda o: r[:, o:o + 9].reshape(-1, 3, 3).transpose(0, 2, 1).copy()   # column-major 3x3
            self.R, self.Jq, self.Ja, self.Jb, self.Ha, self.Hb = m(4), m(20), m(29), m(38), m(47), m(56)
            self.al, self.be, self.DT = r[:, 13:16].copy(), r[:, 16:19].copy(), r[:, 19].copy()
            self.P = r[:, 65:290].reshape(-1, 15, 15).transpose(0, 2, 1).copy()

    def step(self, m, wh, ah, dt, sig2):
        """Advance the windows selected by boolean mask m by one step of bias-corrected readings wh, ah (n,3) and length dt (n,)."""
        if not m.any():
            return
        dtype = self.R.dtype
        self.DT[m] = self.DT[m] + dt[m]
        m = m & (dt != 0)
        if not m.any():
            return
        dt = dt[m]
        wh, ah = wh[m], ah[m]
        R, Jq, Jb, Hb, be = self.R[m], self.Jq[m], self.Jb[m], self.Hb[m], self.be[m]
        Rs, Jr = step_factors(wh, dt)
        RT = R.transpose(0, 2, 1)
        RtA = RT @ skew(ah)
        d1, d2 = dt[:, None], (dt * dt * dtype.type(0.5))[:, None]
        d3, d4 = d1[..., None], d2[..., None]
        Rta = np.einsum("nij,nj->ni", RT, ah)
        self.R[m] = Rs @ R
        self.be[m] = be + Rta * d1
        self.al[m] = (self.al[m] + be * d1) + Rta * d2
        self.Jq[m] = Rs @ Jq + Jr * d3
        self.Jb[m] = Jb + (RtA @ Jq) * d3
        self.Ja[m] = (self.Ja[m] + Jb * d3) + (RtA @ Jq) * d4
        self.Hb[m] = Hb - RT * d3
        self.Ha[m] = (self.Ha[m] + Hb * d3) - RT * d4
        k = int(m.sum())
        I = np.eye(3, dtype=dtype)
        Phi = np.broadcast_to(np.eye(15, dtype=dtype), (k, 15, 15)).copy()
        Phi[:, TH, TH] = Rs
        Phi[:, TH, BG] = -Jr * d3
        Phi[:, V, TH] = -RtA * d3
        Phi[:, V, BA] = -RT * d3
        Phi[:, PP, TH] = -RtA * d4
        Phi[:, PP, V] = I * d3
        Phi[:, PP, BA] = -RT * d4
        q_w, q_wb, q_a, q_ab = sig2
        Q = np.zeros((k, 15, 15), dtype=dtype)
        Q[:, TH, TH] = (q_w * dt)[:, None, None] * (Jr @ Jr.transpose(0, 2, 1))
        Q[:, BG, BG] = (q_wb * dt)[:, None, None] * I
        Q[:, V, V] = (q_a * dt)[:, None, None] * I
        Q[:, V, PP] = Q[:, PP, V] = (q_a * dt * dt * dtype.type(0.5))[:, None, None] * I
        Q[:, PP, PP] = (q_a * dt * dt * dt * dtype.type(0.25))[:, None, None] * I
        Q[:, BA, BA] = (q_ab * dt)[:, None, None] * I
        Pn = Phi @ self.P[m] @ Phi.transpose(0, 2, 1) + Q
        up = np.triu(Pn)
        self.P[m] = up + np.triu(Pn, 1).transpose(0, 2, 1)

    def records(self):
        n = self.R.shape[0]
        rec = np.zeros((n, 290), dtype=self.R.dtype)
        cm = lambda M: M.transpose(0, 2, 1).reshape(n, 9)
        rec[:, 0:4] = rot_2_quat(self.R)
        rec[:, 4:13], rec[:, 20:29], rec[:, 29:38], rec[:, 38:47] = cm(self.R), cm(self.Jq), cm(self.Ja), cm(self.Jb)
        rec[:, 47:56], rec[:, 56:65] = cm(self.Ha), cm(self.Hb)
        rec[:, 13:16], rec[:, 16:19], rec[:, 19] = self.al, self.be, self.DT
        rec[:, 65:290] = self.P.transpose(0, 2, 1).reshape(n, 225)
        return rec


def preintegrate(samples, lin, sigmas, flags=0, offsets=None, ns=None, dtype=np.float64, init=None):
    """Discrete records (n, 290) in `dtype` for the layout of cpi_preintegrate_batch (samples (entries, 7); offsets (n+1) or uniform
    ns).  flags: CPI_FLAG_IMU_AVG (1) averages the step's two ends.  init: records to continue from (the _continue entry point)."""
    dtype = np.dtype(dtype)
    avg = 1 if flags & 1 else 0
    S = np.asarray(samples, dtype=np.float64).reshape(-1, 7).astype(dtype)
    L = np.asarray(lin, dtype=np.float64).reshape(-1, 13).astype(dtype)
    n = L.shape[0]
    if offsets is None:
        if ns is None:
            ns = S.shape[0] // max(n, 1) - avg
        start = np.arange(n, dtype=np.int64) * (ns + avg)
        nsteps = np.full(n, ns, dtype=np.int64)
    else:
        offsets = np.asarray(offsets, dtype=np.int64)
        start = offsets[:-1]
        nsteps = np.maximum(offsets[1:] - offsets[:-1] - avg, 0)
    sig2 = tuple(dtype.type(s) * dtype.type(s) for s in np.asarray(sigmas, dtype=np.float64))
    st = State(n, dtype, init)
    for i in range(int(nsteps.max()) if n else 0):
        m = i < nsteps
        idx = np.where(m, start + i, 0)
        s0 = S[idx]
        wh, ah, dt = s0[:, 0:3] - L[:, 0:3], s0[:, 3:6] - L[:, 3:6], s0[:, 6]
        if avg:
            s1 = S[np.where(m, start + i + 1, 0)]
            wh = (wh + (s1[:, 0:3] - L[:, 0:3])) * dtype.type(0.5)
            ah = (ah + (s1[:, 3:6] - L[:, 3:6])) * dtype.type(0.5)
        st.step(m, wh, ah, dt, sig2)
    return st.records()
