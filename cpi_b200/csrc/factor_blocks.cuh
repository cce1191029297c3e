// Per-window pieces of ImuFactorCPIv1/v2::evaluateError (gtsam/ImuFactorCPIv1.cpp:37-208, ImuFactorCPIv2.cpp:38-212) and of
// getpredictedstate_v1/_v2 (solvers/GraphSolver_IMU.cpp:263-307), force-inlined register code.  The 3x3 helpers and predict_state
// are shared by factor.cu (K3/K4, k_predict) and propagate.cu (K7), so K7's predicted state is k_predict's bit for bit.
// factor_front and h1_theta_blocks restate, operation for operation, the quaternion chain and theta-column blocks that k_factor_eval
// computes in place; K3 keeps its own copy because calling them from it changes its instruction schedule (DESIGN.md section 3d).
#pragma once

#include "cpi_common.cuh"

namespace cpi {

// w*I - [v x]  (sign = -1)   or   w*I + [v x]  (sign = +1),  row-major
CPI_DEV void quat_mat(const double* q, double sign, double* M) {
    M[0] = q[3];            M[1] = -sign * q[2];   M[2] = sign * q[1];
    M[3] = sign * q[2];     M[4] = q[3];           M[5] = -sign * q[0];
    M[6] = -sign * q[1];    M[7] = sign * q[0];    M[8] = q[3];
}
CPI_DEV void skew(const double* v, double* M) {
    M[0] = 0.0; M[1] = -v[2]; M[2] = v[1]; M[3] = v[2]; M[4] = 0.0; M[5] = -v[0]; M[6] = -v[1]; M[7] = v[0]; M[8] = 0.0;
}
// record 3x3 (column-major in global memory) -> row-major registers
CPI_DEV void ldrec33(const double* r, double* M) {
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) M[3 * i + j] = __ldg(r + i + 3 * j);
}

// getpredictedstate_v1/_v2: o = the state x_{k+1} predicted from x = x_k, record r and linearisation point l
template <int MODEL>
CPI_DEV void predict_state(const double* x, const double* r, const double* l, double* o) {
    const double q[4] = {x[0], x[1], x[2], x[3]}, qm[4] = {r[0], r[1], r[2], r[3]}, qi[4] = {-x[0], -x[1], -x[2], x[3]};
    const double dt = r[CPI_REC_DT];
    double qn[4], Rinv[9], rb[3], ra[3];
    quat_multiply(qm, q, qn);
    quat_2_Rot(qi, Rinv);
    const double be[3] = {r[CPI_REC_BETA], r[CPI_REC_BETA + 1], r[CPI_REC_BETA + 2]}, al[3] = {r[CPI_REC_ALPHA], r[CPI_REC_ALPHA + 1], r[CPI_REC_ALPHA + 2]};
    mv33(Rinv, be, rb); mv33(Rinv, al, ra);
#pragma unroll
    for (int k = 0; k < 4; k++) o[k] = qn[k];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const double v = x[7 + k], g = l[10 + k];
        o[4 + k] = x[4 + k]; o[10 + k] = x[10 + k];
        if (MODEL == 1) { o[7 + k] = v - g * dt + rb[k]; o[13 + k] = x[13 + k] + v * dt - 0.5 * g * (dt * dt) + ra[k]; }
        else { o[7 + k] = v + rb[k]; o[13 + k] = x[13 + k] + v * dt + ra[k]; }
    }
}

// The quaternion chain and frame quantities of evaluateError (:57-72; v2 :68-74) for states x_K, x_K1:
//   q_b = rot_2_quat(Exp(-J_q dbg)),  q_n = q_K1 q_K^-1,  q_rm = q_n q_meas^-1,  q_r = q_rm q_b,  q_m = q_b^-1 q_meas,
//   q_kR = q_K q_lin^-1 (model 2; identity in model 1),  Rk = R(q_K),  Rpa = Rk pa,  Rpb = Rk pb
template <int MODEL>
CPI_DEV void factor_front(const double* qK, const double* qK1, const double* vK, const double* vK1, const double* pK, const double* pK1,
                          const double* dbg, const double* q_lin, const double* grav, const double* q_meas, double dT, const double* Jq,
                          double* q_n, double* q_m, double* q_rm, double* q_r, double* q_kR, double* dthk, double* Rk, double* Rpa,
                          double* Rpb) {
    double t3[3], ExpB[9], q_b[4], qi[4], pa[3], pb[3];
    mv33(Jq, dbg, t3);
    t3[0] = -t3[0]; t3[1] = -t3[1]; t3[2] = -t3[2];
    Exp_so3(t3, ExpB);
    rot_2_quat(ExpB, q_b);
    qi[0] = -qK[0]; qi[1] = -qK[1]; qi[2] = -qK[2]; qi[3] = qK[3];
    quat_multiply(qK1, qi, q_n);                                                     // :61
    qi[0] = -q_meas[0]; qi[1] = -q_meas[1]; qi[2] = -q_meas[2]; qi[3] = q_meas[3];
    quat_multiply(q_n, qi, q_rm);                                                    // :62
    quat_multiply(q_rm, q_b, q_r);                                                   // :63
    qi[0] = -q_b[0]; qi[1] = -q_b[1]; qi[2] = -q_b[2]; qi[3] = q_b[3];
    quat_multiply(qi, q_meas, q_m);                                                  // :64

    q_kR[0] = 0; q_kR[1] = 0; q_kR[2] = 0; q_kR[3] = 1; dthk[0] = 0; dthk[1] = 0; dthk[2] = 0;
    if (MODEL == 2) {                                                                // v2 :68-69
        qi[0] = -q_lin[0]; qi[1] = -q_lin[1]; qi[2] = -q_lin[2]; qi[3] = q_lin[3];
        quat_multiply(qK, qi, q_kR);
        dthk[0] = 2.0 * q_kR[0]; dthk[1] = 2.0 * q_kR[1]; dthk[2] = 2.0 * q_kR[2];
    }

    quat_2_Rot(qK, Rk);
#pragma unroll
    for (int k = 0; k < 3; k++) {
        if (MODEL == 1) {                                                            // v1 :70, :72
            pa[k] = pK1[k] - pK[k] - vK[k] * dT + 0.5 * grav[k] * (dT * dT);
            pb[k] = vK1[k] - vK[k] + grav[k] * dT;
        } else {                                                                     // v2 :72, :74
            pa[k] = pK1[k] - pK[k] - vK[k] * dT;
            pb[k] = vK1[k] - vK[k];
        }
    }
    mv33(Rk, pa, Rpa); mv33(Rk, pb, Rpb);
}

// The theta-column blocks of H1 = d e / d x_K (:109-119; v2 :115-119), row-major: (theta, theta), (v, theta), (p, theta) and
// (theta, b_g).  The other non-zero blocks of H1 are -I, -J_b, -J_a, -Rk, -DT Rk, -H_b, -H_a (:121-143).
template <int MODEL>
CPI_DEV void h1_theta_blocks(const double* q_n, const double* q_m, const double* q_rm, const double* q_kR, const double* Rpa,
                             const double* Rpb, const double* Jq, const double* Oal, const double* Obe, double* Htt, double* Hvt,
                             double* Hpt, double* Htb) {
    double A[9], Bm[9], AB[9];
    quat_mat(q_n, -1.0, A); quat_mat(q_m, -1.0, Bm); mul33(A, Bm, AB);
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) Htt[3 * i + j] = -(AB[3 * i + j] + q_n[i] * q_m[j]);
    skew(Rpb, Hvt);
    if (MODEL == 2) { double qm[9], t[9]; quat_mat(q_kR, +1.0, qm); mul33(Obe, qm, t);
#pragma unroll
        for (int k = 0; k < 9; k++) Hvt[k] -= t[k]; }
    skew(Rpa, Hpt);
    if (MODEL == 2) { double qm[9], t[9]; quat_mat(q_kR, +1.0, qm); mul33(Oal, qm, t);
#pragma unroll
        for (int k = 0; k < 9; k++) Hpt[k] -= t[k]; }
    quat_mat(q_rm, -1.0, A); mul33(A, Jq, Htb);
}

}  // namespace cpi
