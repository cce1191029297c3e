// Measurements of one state that depend on its attitude (DESIGN.md section 3l), shared by the linearisation K12 (measurements.cu)
// and the filter update K11 (update.cu), so that the model is stated once.  JPL quaternion, C = quat_2_Rot(q) (global to IMU),
// tangent order [dtheta, b_g, v, b_a, p] and retract q+ = dq (x) q, so C+ ~ (I - [dtheta]x) C.  With r = h(x) - z:
//   CPI_MEAS_POSITION       h = p + C^T aux   H_theta = -C^T [aux]x   H_p = I      (aux: lever arm in the IMU frame)
//   CPI_MEAS_VELOCITY_BODY  h = C v           H_theta = [C v]x        H_v = C
//   CPI_MEAS_DIRECTION      h = C aux         H_theta = [C aux]x                   (aux: a known vector in the global frame)
// Whitened with the column-major S (Lambda = S^T S): A = S H (3x15), b = S r.  An unknown kind gives NaN in every entry of A and b.
#pragma once
#include <math_constants.h>

#include "cpi_common.cuh"

namespace cpi {

// b = S r and A = S H (row-major 3x15) of measurement (kind, z[3], s[9] column-major, aux[3]) at the state x[16]
CPI_DEV void meas_linearize(int kind, const double* x, const double* z, const double* s, const double* aux, double* b, double* A) {
    double R[9], h[3], Hq[9], Hv[9];
    quat_2_Rot(x, R);
    const bool pos = kind == CPI_MEAS_POSITION, vel = kind == CPI_MEAS_VELOCITY_BODY, dir = kind == CPI_MEAS_DIRECTION;
    const double zc = pos || vel || dir ? 0.0 : CUDART_NAN;      // the structurally zero entries (NaN for an unknown kind)
    if (pos) {
        double K[9] = {0.0, -aux[2], aux[1], aux[2], 0.0, -aux[0], -aux[1], aux[0], 0.0};
        mvT33(R, aux, h);
#pragma unroll
        for (int i = 0; i < 3; i++) h[i] += x[13 + i];
        mulT33(R, K, Hq);
#pragma unroll
        for (int k = 0; k < 9; k++) { Hq[k] = -Hq[k]; Hv[k] = 0.0; }
    } else {
        mv33(R, vel ? x + 7 : aux, h);
        const double Kh[9] = {0.0, -h[2], h[1], h[2], 0.0, -h[0], -h[1], h[0], 0.0};
#pragma unroll
        for (int k = 0; k < 9; k++) { Hq[k] = dir || vel ? Kh[k] : CUDART_NAN; Hv[k] = vel ? R[k] : zc; }
    }
    double r[3];
#pragma unroll
    for (int i = 0; i < 3; i++) r[i] = h[i] - z[i] + zc;
#pragma unroll
    for (int i = 0; i < 3; i++) {
        b[i] = fma(s[i + 6], r[2], fma(s[i + 3], r[1], s[i] * r[0]));
#pragma unroll
        for (int c = 0; c < 3; c++) {
            A[i * 15 + c] = fma(s[i + 6], Hq[6 + c], fma(s[i + 3], Hq[3 + c], s[i] * Hq[c]));
            A[i * 15 + 3 + c] = zc;
            A[i * 15 + 6 + c] = fma(s[i + 6], Hv[6 + c], fma(s[i + 3], Hv[3 + c], s[i] * Hv[c]));
            A[i * 15 + 9 + c] = zc;
            A[i * 15 + 12 + c] = pos ? s[i + 3 * c] : zc;
        }
    }
}

}  // namespace cpi
