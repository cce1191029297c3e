"""numpy statement of the robust losses of robust_loss.cuh (DESIGN.md section 3h): the cost and IRLS weight of whitened squared
residuals, shared by the state-prior and the measurement references.  Codes as include/cpi_b200.h's CPI_LOSS_*."""
import numpy as np

GAUSSIAN, HUBER, CAUCHY = 0, 1, 2


def np_loss(code, k, s):
    """(w, c) of whitened squared residuals s under loss codes `code` with thresholds k (arrays, broadcast): the header's table.
    An unknown code or k outside 0 < k^2 < inf gives NaN."""
    code, k, s = (np.asarray(a) for a in np.broadcast_arrays(code, k, s))
    s = s.astype(np.float64)
    w, c = np.full(s.shape, np.nan), np.full(s.shape, np.nan)
    with np.errstate(all="ignore"):
        k2 = k * k
        ok = (k > 0) & (k2 > 0) & np.isfinite(k2)
        g = code == GAUSSIAN
        w[g], c[g] = 1.0, s[g]
        hi = (code == HUBER) & ok & (s <= k2)
        w[hi], c[hi] = 1.0, s[hi]
        ho = (code == HUBER) & ok & ~(s <= k2)
        r = np.sqrt(s[ho])
        w[ho], c[ho] = k[ho] / r, 2.0 * k[ho] * r - k2[ho]
        ca = (code == CAUCHY) & ok
        u = s[ca] / k2[ca]
        w[ca], c[ca] = 1.0 / (1.0 + u), k2[ca] * np.log1p(u)
        big = np.zeros(s.shape, bool)
        big[ca] = np.isinf(u)                                      # k < 1 and finite s above k^2 DBL_MAX: u overflows
        w[big], c[big] = k2[big] / s[big], k2[big] * (np.log(s[big]) - np.log(k2[big]))
    return w, c
