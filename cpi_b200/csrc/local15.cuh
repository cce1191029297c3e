// local(x_lin, x), the inverse of JPLNavState::retract, shared by k_prior_at (marginalize.cu) and the relinearisation selection
// (relinearize.cu).
#pragma once
#include "cpi_common.cuh"

namespace cpi {

// local(x_lin, x): the delta with x = JPLNavState::retract(x_lin, delta) -- the rotation vector of q_x (x) q_lin^-1 (w >= 0, JPL),
// the other 12 entries are differences.  Exactly 0 at x == x_lin.
CPI_DEV void local15(const double* xl, const double* x, double* d) {
    const double qi[4] = {-xl[0], -xl[1], -xl[2], xl[3]};
    double dq[4];
    quat_multiply(x, qi, dq);
    const double s = sqrt(dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2]);
    const bool same = x[0] == xl[0] && x[1] == xl[1] && x[2] == xl[2] && x[3] == xl[3];
    const double k = same ? 0.0 : (s > 0.0 ? 2.0 * atan2(s, dq[3]) / s : 2.0);
#pragma unroll
    for (int j = 0; j < 3; j++) d[j] = k * dq[j];
#pragma unroll
    for (int j = 0; j < 12; j++) d[3 + j] = x[4 + j] - xl[4 + j];
}

}  // namespace cpi
