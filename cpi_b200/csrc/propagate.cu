// K7: covariance propagation through preintegrated records.  For window i with anchor state x_k, covariance Sigma_k, record r and
// linearisation point l (DESIGN.md "Propagating the covariance"):
//   x_k1    = getpredictedstate(x_k, r, l)                        (bit for bit what k_predict writes)
//   H1, H2  = d e / d x_k, d e / d x_k1 of ImuFactorCPIv1/v2 at (x_k, x_k1)   (the blocks k_factor_eval writes)
//   A = -H2^-1 H1,  B = H2^-1,  Sigma_k1 = A Sigma_k A^T + B P_meas B^T,  C = Sigma_k A^T  (cross-covariance)
// H2 = blockdiag(Q, I, Rk, I, Rk) with Q = quat_mat(q_r, +1), so H2^-1 is closed-form: Q^-1 = (w^2 I - w [v x] + v v^T) / (w |q|^2)
// for q_r = [v w], and Rk^-1 = Rk^T.  A is the identity except for its theta, v and p block rows (state order [theta, b_g, v, b_a, p]):
//   theta: [ -Q^-1 H1_tt   -Q^-1 H1_tb   0       0           0 ]
//   v:     [ -Rk^T H1_vt    Rk^T J_b     I       Rk^T H_b    0 ]
//   p:     [ -Rk^T H1_pt    Rk^T J_a     DT I    Rk^T H_a    I ]
// the sparsity of the merge's Phi~ (record_merge.cuh), so A x costs seven 3x3 products, and B P B^T has the shape of T P2 T^T there.
//
// One warp per window.  Lanes 0..8 each build the prediction and the factor's quaternion chain (redundantly: it is one dependent
// chain either way) and then one coefficient block each; Sigma_k and P_meas are staged in shared memory with coalesced loads.  Lane
// j < 15 applies A to column j of Sigma_k (N = A Sigma_k), then lane i < 15 applies A to row i of N and adds row i of B P B^T; only
// the upper triangle is computed and it is mirrored, so Sigma_k1 is exactly symmetric.  C = N^T (= Sigma_k A^T for a symmetric
// Sigma_k) comes for free.  Results leave through shared memory with coalesced stores.
#include "cpi_common.cuh"
#include "cpi_kernels.h"
#include "factor_blocks.cuh"

namespace cpi {

constexpr int PWARPS = 4;                        // windows (warps) per CTA
// per-warp shared scratch (doubles): Sigma (then Sigma_k1), N = A Sigma, P_meas, coefficient blocks
constexpr int CF_TT = 0, CF_TB = 9, CF_VT = 18, CF_PT = 27, CF_VB = 36, CF_VA = 45, CF_PB = 54, CF_PA = 63, CF_QI = 72, CF_RK = 81, CF_DT = 90;
constexpr int SM_S = 0, SM_N = 225, SM_P = 450, SM_CF = 675, SM_WARP = 768;

// x <- A x for a 15-vector x, in place (p rows first: they read v; then v; theta last)
CPI_DEV void a_apply(double* x, const double* cf) {
    const double dt = cf[CF_DT];
#pragma unroll
    for (int i = 0; i < 3; i++) {
        double tp = x[12 + i] + dt * x[6 + i];
#pragma unroll
        for (int j = 0; j < 3; j++) tp += cf[CF_PT + 3 * i + j] * x[j] + cf[CF_PB + 3 * i + j] * x[3 + j] + cf[CF_PA + 3 * i + j] * x[9 + j];
        x[12 + i] = tp;
    }
#pragma unroll
    for (int i = 0; i < 3; i++) {
        double tv = x[6 + i];
#pragma unroll
        for (int j = 0; j < 3; j++) tv += cf[CF_VT + 3 * i + j] * x[j] + cf[CF_VB + 3 * i + j] * x[3 + j] + cf[CF_VA + 3 * i + j] * x[9 + j];
        x[6 + i] = tv;
    }
    double t0[3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
        t0[i] = 0.0;
#pragma unroll
        for (int j = 0; j < 3; j++) t0[i] += cf[CF_TT + 3 * i + j] * x[j] + cf[CF_TB + 3 * i + j] * x[3 + j];
    }
    x[0] = t0[0]; x[1] = t0[1]; x[2] = t0[2];
}

template <int MODEL>
__global__ void __launch_bounds__(PWARPS * 32) k_propagate(const PropagateParams p) {
    __shared__ double smem[PWARPS * SM_WARP];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * PWARPS + warp;
    if (i >= p.n) return;
    constexpr int RD = (MODEL == 1) ? CPI_REC_V1_DOUBLES : CPI_REC_V2_DOUBLES;
    double* S = smem + warp * SM_WARP + SM_S;
    double* N = smem + warp * SM_WARP + SM_N;
    double* Pm = smem + warp * SM_WARP + SM_P;
    double* cf = smem + warp * SM_WARP + SM_CF;
    const int64_t a = p.anchor ? p.anchor[i] : i;
    const double* x = p.states + a * CPI_STATE_DOUBLES;
    const double* r = p.records + i * (int64_t)RD;
    const double* l = p.lin + i * CPI_LIN_DOUBLES;
    {
        const double* sg = p.cov + a * 225;
        for (int e = lane; e < 225; e += 32) { S[e] = __ldg(sg + e); Pm[e] = __ldg(r + CPI_REC_P + e); }
    }

    if (lane < 9) {
        double xh[16];
        predict_state<MODEL>(x, r, l, xh);
        const double qK[4] = {x[0], x[1], x[2], x[3]}, vK[3] = {x[7], x[8], x[9]}, pK[3] = {x[13], x[14], x[15]};
        const double dbg[3] = {x[4] - __ldg(l), x[5] - __ldg(l + 1), x[6] - __ldg(l + 2)};
        const double q_lin[4] = {__ldg(l + 6), __ldg(l + 7), __ldg(l + 8), __ldg(l + 9)};
        const double grav[3] = {__ldg(l + 10), __ldg(l + 11), __ldg(l + 12)};
        const double q_meas[4] = {__ldg(r), __ldg(r + 1), __ldg(r + 2), __ldg(r + 3)};
        const double dT = __ldg(r + CPI_REC_DT);
        double Jq[9], Oal[9], Obe[9];
        ldrec33(r + CPI_REC_JQ, Jq);
        if (MODEL == 2) { ldrec33(r + CPI_REC_OA, Oal); ldrec33(r + CPI_REC_OB, Obe); }
        double q_n[4], q_m[4], q_rm[4], q_r[4], q_kR[4], dthk[3], Rk[9], Rpa[3], Rpb[3];
        factor_front<MODEL>(qK, xh, vK, xh + 7, pK, xh + 13, dbg, q_lin, grav, q_meas, dT, Jq, q_n, q_m, q_rm, q_r, q_kR, dthk, Rk, Rpa, Rpb);
        double Htt[9], Hvt[9], Hpt[9], Htb[9];
        h1_theta_blocks<MODEL>(q_n, q_m, q_rm, q_kR, Rpa, Rpb, Jq, Oal, Obe, Htt, Hvt, Hpt, Htb);
        // Q^-1 for Q = w I + [v x]:  (w I + K)(w^2 I - w K + v v^T) = w (w^2 + |v|^2) I,  since K^2 = v v^T - |v|^2 I and K v = 0
        double Qi[9];
        {
            const double w = q_r[3], v[3] = {q_r[0], q_r[1], q_r[2]};
            const double d = 1.0 / (w * (w * w + v[0] * v[0] + v[1] * v[1] + v[2] * v[2]));
            double K[9];
            skew(v, K);
#pragma unroll
            for (int u = 0; u < 3; u++)
#pragma unroll
                for (int c = 0; c < 3; c++) Qi[3 * u + c] = ((u == c ? w * w : 0.0) - w * K[3 * u + c] + v[u] * v[c]) * d;
        }
        if (lane < 8) {
            // lane -> block: 0 theta,theta  1 theta,b_g  2 v,theta  3 p,theta  (-H2^-1 H1 blocks);  4 v,b_g  5 v,b_a  6 p,b_g  7 p,b_a
            // (H1 there is -J_b, -H_b, -J_a, -H_a, so the block is +Rk^T times the record's)
            double X[9], L[9], Cb[9];
            if (lane >= 4) ldrec33(r + (lane == 4 ? CPI_REC_JB : lane == 5 ? CPI_REC_HB : lane == 6 ? CPI_REC_JA : CPI_REC_HA), X);
#pragma unroll
            for (int e = 0; e < 9; e++) {
                if (lane < 4) X[e] = lane == 0 ? Htt[e] : lane == 1 ? Htb[e] : lane == 2 ? Hvt[e] : Hpt[e];
                L[e] = lane < 2 ? Qi[e] : Rk[3 * (e % 3) + e / 3];
            }
            mul33(L, X, Cb);
            const double s = lane < 4 ? -1.0 : 1.0;
            const int off = lane == 0 ? CF_TT : lane == 1 ? CF_TB : lane == 2 ? CF_VT : lane == 3 ? CF_PT
                          : lane == 4 ? CF_VB : lane == 5 ? CF_VA : lane == 6 ? CF_PB : CF_PA;
#pragma unroll
            for (int e = 0; e < 9; e++) cf[off + e] = s * Cb[e];
        } else {
#pragma unroll
            for (int e = 0; e < 9; e++) { cf[CF_QI + e] = Qi[e]; cf[CF_RK + e] = Rk[e]; }
            cf[CF_DT] = dT;
            double* o = p.states_k1 + i * CPI_STATE_DOUBLES;
#pragma unroll
            for (int k = 0; k < 16; k++) o[k] = xh[k];
        }
    }
    __syncwarp();

    double v[15];
    if (lane < 15) {                                                  // N(:, j) = A Sigma(:, j)
#pragma unroll
        for (int k = 0; k < 15; k++) v[k] = S[k + 15 * lane];
        a_apply(v, cf);
#pragma unroll
        for (int k = 0; k < 15; k++) N[k + 15 * lane] = v[k];
    }
    __syncwarp();
    if (lane < 15) {                                                  // Sigma_k1(i, :) = (A N(i, :)^T)^T + (B P B^T)(i, :), j >= i
        const int I = lane / 3, ii = lane - 3 * I;
#pragma unroll
        for (int k = 0; k < 15; k++) v[k] = N[lane + 15 * k];
        a_apply(v, cf);
        const double* Qi = cf + CF_QI;
        const double* Rk = cf + CF_RK;
        double bi[3];                                                 // row ii of B_I: Q^-1, I or Rk^T
#pragma unroll
        for (int c = 0; c < 3; c++) bi[c] = I == 0 ? Qi[3 * ii + c] : (I == 2 || I == 4) ? Rk[3 * c + ii] : (c == ii ? 1.0 : 0.0);
#pragma unroll
        for (int J = 0; J < 5; J++) {
            double t[3], s[3];
#pragma unroll
            for (int m = 0; m < 3; m++) {
                const int k = 3 * J + m;
                t[m] = bi[0] * Pm[3 * I + 15 * k] + bi[1] * Pm[3 * I + 1 + 15 * k] + bi[2] * Pm[3 * I + 2 + 15 * k];
            }
#pragma unroll
            for (int m = 0; m < 3; m++) {                             // ... B_J^T on the right
                if (J == 0) s[m] = t[0] * Qi[3 * m] + t[1] * Qi[3 * m + 1] + t[2] * Qi[3 * m + 2];
                else if (J == 2 || J == 4) s[m] = t[0] * Rk[m] + t[1] * Rk[3 + m] + t[2] * Rk[6 + m];
                else s[m] = t[m];
            }
#pragma unroll
            for (int m = 0; m < 3; m++) {
                const int j = 3 * J + m;
                if (j >= lane) { const double y = v[j] + s[m]; S[lane + 15 * j] = y; S[j + 15 * lane] = y; }
            }
        }
    }
    __syncwarp();
    double* o = p.cov_k1 + i * 225;
    for (int e = lane; e < 225; e += 32) o[e] = S[e];
    if (p.cross) {
        double* c = p.cross + i * 225;
        for (int e = lane; e < 225; e += 32) c[e] = N[e / 15 + 15 * (e % 15)];      // C = N^T
    }
}

cudaError_t propagate_launch(int model, const PropagateParams& p, cudaStream_t st) {
    if (p.n == 0) return cudaSuccess;
    const int64_t grid = (p.n + PWARPS - 1) / PWARPS;
    if (model == 1) k_propagate<1><<<(unsigned)grid, PWARPS * 32, 0, st>>>(p);
    else k_propagate<2><<<(unsigned)grid, PWARPS * 32, 0, st>>>(p);
    return cudaGetLastError();
}

}  // namespace cpi
