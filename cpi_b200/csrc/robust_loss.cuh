// The robust losses of DESIGN.md section 3h, shared by the prior reweighting k_state_prior_robust (state_priors.cu) and the iterated
// filter update K13 (update.cu), so that the losses are stated once.
#pragma once
#include <math_constants.h>

#include "cpi_common.cuh"

namespace cpi {

// cost c(s) and IRLS weight w(s) = dc/ds of a whitened squared residual s under loss `code` with threshold k (standard deviations).
// A Huber inlier (s <= k^2) is the Gaussian prior itself: w = 1, c = s.  An unknown code, or k outside 0 < k^2 < inf, gives NaN.
// Cauchy with k < 1 and a finite s above k^2 DBL_MAX overflows u = s/k^2: then c = k^2 (log s - log k^2) and w = k^2/s, which differ
// from k^2 log1p(u) and 1/(1+u) by the dropped k^2/s < 1e-308 (relative).
CPI_DEV void robust_loss(int code, double k, double s, double& w, double& c) {
    if (code == CPI_LOSS_GAUSSIAN) { w = 1.0; c = s; return; }
    const double k2 = k * k;
    if (!(k > 0.0 && k2 > 0.0 && k2 < CUDART_INF) || (code != CPI_LOSS_HUBER && code != CPI_LOSS_CAUCHY)) {
        w = c = CUDART_NAN;
        return;
    }
    if (code == CPI_LOSS_HUBER) {
        if (s <= k2) { w = 1.0; c = s; return; }
        const double r = sqrt(s);
        w = k / r;
        c = 2.0 * k * r - k2;
    } else {
        const double u = s / k2;
        if (isinf(u)) {
            w = k2 / s;
            c = k2 * (log(s) - log(k2));
        } else {
            w = 1.0 / (1.0 + u);
            c = k2 * log1p(u);
        }
    }
}

}  // namespace cpi
