"""Parity gates of SURVEY.md section 8(d), shared by the CPU (oracle) and GPU (CUDA) tests.

north_star tolerances: <= 1e-9 relative on dR / alpha / beta, <= 1e-6 on P.  Jacobian gates proposed by the survey:
1e-9 relative Frobenius, except J_a for windows that touch the ill-conditioned band |w_hat| in [0.0087, 0.05) rad/s,
where the reference's own closed forms are only determined to ~1e-8 (gate 1e-6 there).

conditioned_gate: the tighter, conditioning-aware gate against the long-double oracle (DESIGN.md section 5)."""
import numpy as np

REC = dict(q=(0, 4), R=(4, 13), alpha=(13, 16), beta=(16, 19), DT=(19, 20), J_q=(20, 29), J_a=(29, 38), J_b=(38, 47),
           H_a=(47, 56), H_b=(56, 65), P=(65, 290), O_a=(290, 299), O_b=(299, 308))
SMALL_W = 0.008726646


def window_band(samples, offsets, lin):
    """True per window if any sample has |w_hat| in the ill-conditioned band [SMALL_W, 0.05)."""
    n = len(offsets) - 1
    out = np.zeros(n, dtype=bool)
    for i in range(n):
        s = samples[offsets[i]:offsets[i + 1]]
        if len(s):
            m = np.linalg.norm(s[:, 0:3] - lin[i, 0:3], axis=1)
            out[i] = bool(np.any((m >= SMALL_W) & (m < 0.05) & (s[:, 6] != 0)))
    return out


def imu_avg_inputs(samples, offsets):
    """The imu_avg form of a CSR batch: imu_avg consumes one trailing entry per window, so every non-empty window repeats its last
    entry (tests/golden/make_golden.py ran the reference on exactly this layout)."""
    n = len(offsets) - 1
    wins = [samples[offsets[i]:offsets[i + 1]] for i in range(n)]
    wins = [np.concatenate([w, w[-1:]]) if len(w) else w for w in wins]
    off = np.zeros(n + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(w) for w in wins])
    return np.ascontiguousarray(np.concatenate(wins).reshape(-1, 7)), off


def rel(a, b, floor=1e-300):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), floor))


def compare_records(got, ref, model, in_band=None, tol_mean=1e-9, tol_P=1e-6, tol_J=1e-9, tol_Ja_band=1e-6, has_steps=None):
    """Assert the gates window by window; returns a dict of the worst error per field (for reporting)."""
    got = np.asarray(got); ref = np.asarray(ref)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    n = got.shape[0]
    worst = {}

    def upd(k, v):
        worst[k] = max(worst.get(k, 0.0), float(v))

    for i in range(n):
        g, r = got[i], ref[i]
        assert np.all(np.isfinite(g)), f"window {i}: non-finite output"
        assert g[19] == r[19] or abs(g[19] - r[19]) <= 4e-16 * abs(r[19]), f"window {i}: DT {g[19]} vs {r[19]}"
        eR = np.linalg.norm(g[4:13] - r[4:13]); upd("R", eR)
        assert eR <= tol_mean, f"window {i}: dR Frobenius {eR:.3e}"
        if has_steps is None or has_steps[i]:
            eq = min(np.linalg.norm(g[0:4] - r[0:4]), np.linalg.norm(g[0:4] + r[0:4])); upd("q", eq)
            assert eq <= tol_mean, f"window {i}: q {eq:.3e}"
        for name in ("alpha", "beta"):
            a, b = REC[name]
            e = np.linalg.norm(g[a:b] - r[a:b]) / max(np.linalg.norm(r[a:b]), 1e-9); upd(name, e)
            assert e <= tol_mean, f"window {i}: {name} rel {e:.3e}"
        names = ["J_q", "J_b", "H_a", "H_b"] + (["O_a", "O_b"] if model == 2 else [])
        for name in names:
            a, b = REC[name]
            e = np.linalg.norm(g[a:b] - r[a:b]) / max(np.linalg.norm(r[a:b]), 1e-12); upd(name, e)
            assert e <= tol_J, f"window {i}: {name} rel {e:.3e}"
        a, b = REC["J_a"]
        e = np.linalg.norm(g[a:b] - r[a:b]) / max(np.linalg.norm(r[a:b]), 1e-12)
        band = bool(in_band[i]) if in_band is not None else False
        upd("J_a_band" if band else "J_a", e)
        assert e <= (tol_Ja_band if band else tol_J), f"window {i}: J_a rel {e:.3e} (band={band})"
        Pg = g[65:290].reshape(15, 15, order="F"); Pr = r[65:290].reshape(15, 15, order="F")
        eP = np.linalg.norm(Pg - Pr) / max(np.linalg.norm(Pr), 1e-300); upd("P", eP)
        assert eP <= tol_P, f"window {i}: P rel {eP:.3e}"
        assert np.array_equal(Pg, Pg.T), f"window {i}: P not exactly symmetric"
        for I in range(5):
            for J in range(5):
                bg_, br_ = Pg[3 * I:3 * I + 3, 3 * J:3 * J + 3], Pr[3 * I:3 * I + 3, 3 * J:3 * J + 3]
                nr = np.linalg.norm(br_)
                if nr == 0.0:
                    assert np.all(bg_ == 0.0), f"window {i}: structurally-zero P block ({I},{J}) is not zero"
                else:
                    eb = np.linalg.norm(bg_ - br_)
                    upd("P_block", eb / nr)
                    assert eb <= tol_P * nr + 1e-17, f"window {i}: P block ({I},{J}) err {eb:.3e} vs norm {nr:.3e}"
    return worst


GATE_FIELDS = ("q", "R", "alpha", "beta", "J_q", "J_a", "J_b", "H_a", "H_b", "O_a", "O_b")


def field_errors(got, truth, model):
    """Relative Frobenius error per window of every gated field (q up to sign) and of each 3x3 block of P: a dict
    name -> [n] array, P blocks as "P_IJ".  Where the truth is exactly zero the error is 0 if got is exactly zero too and
    inf otherwise, so a structural zero that is not exactly zero fails any gate."""
    g = np.asarray(got, dtype=np.float64); t = np.asarray(truth, dtype=np.float64)
    n = t.shape[0]

    def rel_rows(d, r):
        num = np.linalg.norm(d.reshape(n, -1), axis=1); den = np.linalg.norm(r.reshape(n, -1), axis=1)
        return np.where(den > 0, num / np.where(den > 0, den, 1.0), np.where(num > 0, np.inf, 0.0))

    out = {}
    for name in GATE_FIELDS:
        if model == 1 and name in ("O_a", "O_b"):
            continue
        a, b = REC[name]
        d = g[:, a:b] - t[:, a:b]
        if name == "q":
            d = np.where(np.linalg.norm(d, axis=1, keepdims=True) <= np.linalg.norm(g[:, a:b] + t[:, a:b], axis=1, keepdims=True), d, g[:, a:b] + t[:, a:b])
        out[name] = rel_rows(d, t[:, a:b])
    Pg = g[:, 65:290].reshape(n, 15, 15).transpose(0, 2, 1); Pt = t[:, 65:290].reshape(n, 15, 15).transpose(0, 2, 1)
    for I in range(5):
        for J in range(I, 5):
            sl = (slice(None), slice(3 * I, 3 * I + 3), slice(3 * J, 3 * J + 3))
            out[f"P_{I}{J}"] = rel_rows(Pg[sl] - Pt[sl], Pt[sl])
    return out


def conditioned_gate(got, o64, truth, model, K, floor, allowance=None):
    """The conditioning-aware gate: for every window and every field of ``field_errors``,
        e_dev <= K * max(e_64, floor) + allowance,
    with e_dev the error of ``got`` against ``truth`` (the long-double oracle) and e_64 that of the fp64 oracle ``o64``: a
    kernel may be as inaccurate as the fp64 reference computation is on that window, times K, and never worse than
    K * floor where that computation is exact.  ``allowance`` (dict field -> scalar or [n] array) adds a fixed error budget,
    e.g. the output rounding and the RK4 accumulation of the fp32 variant ("P" covers every P block).  Returns
    (ratio, worst, failures): per field the [n] array e_dev / (K max(e_64, floor) + allowance), the worst e_dev / e_64 /
    ratio per field for reporting, and one message per field whose worst ratio exceeds 1."""
    g = np.asarray(got, dtype=np.float64)
    n = g.shape[0]
    assert np.all(np.isfinite(g)), "non-finite output"
    ed, e64 = field_errors(g, truth, model), field_errors(o64, truth, model)
    allowance = allowance or {}
    ratio, worst, bad = {}, {}, []
    for k in ed:
        bound = K * np.maximum(e64[k], floor) + allowance.get(k, allowance.get("P", 0.0) if k.startswith("P_") else 0.0)
        r = ed[k] / bound
        ratio[k] = r
        i = int(np.argmax(r))
        worst[k] = dict(e_dev=float(ed[k].max()), e_64=float(e64[k].max()), ratio=float(r[i]))
        if not r[i] <= 1.0:
            bad.append(f"{k}: window {i} e_dev {ed[k][i]:.3e} e_64 {e64[k][i]:.3e} bound {np.broadcast_to(bound, (n,))[i]:.3e}")
    return ratio, worst, bad


def scaled_errors(got, truth, scale=None, sign_free=None):
    """Per row [n, ...]: ||got - truth|| / scale, with scale = ||truth|| by default or an [n] array (the size of the terms that
    cancel into the value).  Where the scale is 0 the error is 0 if got equals truth exactly and inf otherwise.  sign_free: [n] bool,
    rows compared up to sign (a quaternion whose w is near 0)."""
    g = np.asarray(got, dtype=np.float64); t = np.asarray(truth, dtype=np.float64)
    n = t.shape[0]
    g = g.reshape(n, -1); t = t.reshape(n, -1)
    num = np.linalg.norm(g - t, axis=1)
    if sign_free is not None:
        num = np.where(sign_free, np.minimum(num, np.linalg.norm(g + t, axis=1)), num)
    den = np.linalg.norm(t, axis=1) if scale is None else np.broadcast_to(np.asarray(scale, dtype=np.float64), (n,))
    return np.where(den > 0, num / np.where(den > 0, den, 1.0), np.where(num > 0, np.inf, 0.0))


def gate_errors(ed, e64, K, floor):
    """The rule of ``conditioned_gate`` on precomputed per-field error arrays (dicts name -> [n]): e_dev <= K max(e_64, floor).
    Returns (ratio, worst, failures) as conditioned_gate does; a non-finite e_dev fails."""
    ratio, worst, bad = {}, {}, []
    for k in ed:
        bound = K * np.maximum(e64[k], floor)
        r = np.where(np.isnan(ed[k]), np.inf, ed[k] / bound)
        ratio[k] = r
        i = int(np.argmax(r))
        worst[k] = dict(e_dev=float(np.max(ed[k])), e_64=float(np.max(e64[k])), ratio=float(r[i]))
        if not r[i] <= 1.0:
            bad.append(f"{k}: row {i} e_dev {ed[k][i]:.3e} e_64 {e64[k][i]:.3e} bound {bound[i]:.3e}")
    return ratio, worst, bad


def fp32_errors(got, ref):
    """Worst relative error per record field of the fp32-storage variant against the fp64 oracle run on the same float-rounded
    inputs, plus the worst 3x3 block of P (relative to that block's norm; blocks that are exactly zero in the reference must
    be exactly zero).  No fp32 reference exists (the reference is double-only): these are reported, and gated at 2x observed."""
    g = np.asarray(got, dtype=np.float64); r = np.asarray(ref)
    worst = {}
    fields = dict(R=(4, 13), alpha=(13, 16), beta=(16, 19), J_q=(20, 29), J_a=(29, 38), J_b=(38, 47), H_a=(47, 56), H_b=(56, 65), P=(65, 290))
    if g.shape[1] > 290:
        fields.update(O_a=(290, 299), O_b=(299, 308))
    for name, (a, b) in fields.items():
        num = np.linalg.norm(g[:, a:b] - r[:, a:b], axis=1); den = np.maximum(np.linalg.norm(r[:, a:b], axis=1), 1e-30)
        worst[name] = float(np.max(num / den))
    n = g.shape[0]
    Pg = g[:, 65:290].reshape(n, 15, 15).transpose(0, 2, 1); Pr = r[:, 65:290].reshape(n, 15, 15).transpose(0, 2, 1)
    wb = 0.0
    for I in range(5):
        for J in range(5):
            bg_, br_ = Pg[:, 3 * I:3 * I + 3, 3 * J:3 * J + 3], Pr[:, 3 * I:3 * I + 3, 3 * J:3 * J + 3]
            nr = np.linalg.norm(br_.reshape(n, -1), axis=1)
            z = nr == 0.0
            assert np.all(bg_[z] == 0.0), f"structurally-zero P block ({I},{J}) is not zero"
            if np.any(~z):
                eb = np.linalg.norm((bg_ - br_).reshape(n, -1), axis=1)[~z] / nr[~z]
                wb = max(wb, float(eb.max()))
    worst["P_block"] = wb
    return worst
