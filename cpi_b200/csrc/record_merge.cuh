// The composition of two consecutive model-1 records, shared by K5 (merge.cu) and K6 (scan.cu).
//
// Record 1 covers k -> m, record 2 covers m -> j, both at the same bias linearisation point; the merged record k -> j is
// (DESIGN.md "Merging records"; blocks 3x3, [x] the skew matrix):
//   R = R2 R1,  DT = DT1 + DT2,  q = rot_2_quat(R)
//   beta = b1 + R1^T b2,  alpha = a1 + b1 DT2 + R1^T a2
//   J_q = R2 J_q1 + J_q2,  H_b = H_b1 + R1^T H_b2,  H_a = H_a1 + H_b1 DT2 + R1^T H_a2
//   J_b = J_b1 + R1^T([b2] J_q1 + J_b2),  J_a = J_a1 + J_b1 DT2 + R1^T([a2] J_q1 + J_a2)
//   P = Phi~ P1 Phi~^T + T P2 T^T,  T = blockdiag(I, I, R1^T, I, R1^T),  Phi~ = T Phi2 T^T  (state order [theta, b_g, v, b_a, p])
// Phi~ is the identity except for its theta, v and p block rows:
//   theta: [ R2   -J_q2  0  0  0 ]     v: [ -R1^T[b2]  R1^T J_b2  I      R1^T H_b2  0 ]     p: [ -R1^T[a2]  R1^T J_a2  DT2 I  R1^T H_a2  I ]
// so Phi~ x costs 7 3x3 products, not a dense 15x15 one.  A record whose linearisation point differs from the group's first is first
// moved to it to first order (R <- Exp(J_q db_w) R, alpha += J_a db_w + H_a db_a, beta += J_b db_w + H_b db_a; Jacobians and P
// as they are), so that every merge composes records at one point and any bracketing equals a left fold up to rounding.
//
// Inside a merge, lane j < 15 applies Phi~ to column j of P1 (M = Phi~ P1), then lane i < 15 applies it to row i of M and adds row i
// of T P2 T^T; only the upper triangle is written, mirrored, so P is exactly symmetric, and the structurally zero blocks P_theta,ba
// and P_bg,ba stay exactly zero (Phi~ maps them from exact zeros).
#pragma once

#include "cpi_common.cuh"

namespace cpi {
namespace rec1 {

constexpr int RD = CPI_REC_V1_DOUBLES;
constexpr int HEAD = CPI_REC_P;                 // fields q .. H_b: the record before P
// per-warp scratch: Phi~ coefficient blocks Xb Yb Zb Xa Ya Za (row-major), the merged head fields, M = Phi~ P1 (column-major)
constexpr int SC_COEF = 0, SC_HEAD = 54, SC_M = SC_HEAD + HEAD, SCR = SC_M + 225;

// 3x3 record block (column-major in memory) <-> row-major registers
CPI_DEV void ld33(const double* r, double* M) {
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) M[3 * i + j] = r[i + 3 * j];
}
CPI_DEV void st33(double* r, const double* M) {
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) r[i + 3 * j] = M[3 * i + j];
}
// A [v]x  for row-major A:  row i of A [v]x = (row_i(A) x v)^T
CPI_DEV void mul_skew(const double* A, const double* v, double* C) {
#pragma unroll
    for (int i = 0; i < 3; i++) cross(A + 3 * i, v, C + 3 * i);
}

// Move a record (fp64, shared memory) from its own linearisation point to the group's first one, to first order.
CPI_DEV void relinearise(double* r, const double* dbw, const double* dba) {
    double Jq[9], Ja[9], Jb[9], Ha[9], Hb[9], R[9], E[9], Rn[9], t[3], u[3], w[3];
    ld33(r + CPI_REC_JQ, Jq); ld33(r + CPI_REC_JA, Ja); ld33(r + CPI_REC_JB, Jb); ld33(r + CPI_REC_HA, Ha); ld33(r + CPI_REC_HB, Hb);
    ld33(r + CPI_REC_R, R);
    mv33(Jq, dbw, t);
    Exp_so3(t, E);                                   // R(q_b^-1 (x) q_meas), q_b = rot_2_quat(Exp(-J_q db_w)): factor.cu
    mul33(E, R, Rn);
    st33(r + CPI_REC_R, Rn);
    mv33(Ja, dbw, u); mv33(Ha, dba, w);
#pragma unroll
    for (int i = 0; i < 3; i++) r[CPI_REC_ALPHA + i] += u[i] + w[i];
    mv33(Jb, dbw, u); mv33(Hb, dba, w);
#pragma unroll
    for (int i = 0; i < 3; i++) r[CPI_REC_BETA + i] += u[i] + w[i];
}

// x <- Phi~ x for a 15-vector x, in place (p rows first: they read v; then v; theta last); B = record 2 (R2, J_q2, DT2),
// cf = the six coefficient blocks (row-major)
CPI_DEV void phi_apply(double* x, const double* B, const double* cf) {
    const double dt2 = B[CPI_REC_DT];
#pragma unroll
    for (int i = 0; i < 3; i++) {
        double tp = x[12 + i] + dt2 * x[6 + i];
#pragma unroll
        for (int j = 0; j < 3; j++) tp += cf[27 + 3 * i + j] * x[j] + cf[36 + 3 * i + j] * x[3 + j] + cf[45 + 3 * i + j] * x[9 + j];
        x[12 + i] = tp;
    }
#pragma unroll
    for (int i = 0; i < 3; i++) {
        double tv = x[6 + i];
#pragma unroll
        for (int j = 0; j < 3; j++) tv += cf[0 + 3 * i + j] * x[j] + cf[9 + 3 * i + j] * x[3 + j] + cf[18 + 3 * i + j] * x[9 + j];
        x[6 + i] = tv;
    }
    double t0[3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
        t0[i] = 0.0;
#pragma unroll
        for (int j = 0; j < 3; j++) t0[i] += B[CPI_REC_R + i + 3 * j] * x[j] - B[CPI_REC_JQ + i + 3 * j] * x[3 + j];
    }
    x[0] = t0[0]; x[1] = t0[1]; x[2] = t0[2];
}

// A (+) B for two fp64 records in shared memory (A the earlier interval), computed by one warp; sc = that warp's scratch.  The result
// replaces A (kRight = false: A <- A (+) B) or B (kRight = true: B <- A (+) B); the arithmetic, and so every bit, is the same.
template <bool kRight>
CPI_DEV void merge_pair(double* A, double* B, double* sc, int lane) {
    double* cf = sc + SC_COEF;
    double* hd = sc + SC_HEAD;
    double* M = sc + SC_M;
    if (lane < 15) {
        double R1[9], b2[3], X[9], C[9], D[9];
        ld33(A + CPI_REC_R, R1);
        if (lane < 6) {                                                   // Phi~ coefficient blocks
            const int k = lane % 3;                                       // 0: [.] term, 1: J term, 2: H term
            const int v = lane < 3 ? CPI_REC_BETA : CPI_REC_ALPHA;
            if (k == 0) {
                b2[0] = B[v]; b2[1] = B[v + 1]; b2[2] = B[v + 2];
                double RT[9];
#pragma unroll
                for (int i = 0; i < 3; i++)
#pragma unroll
                    for (int j = 0; j < 3; j++) RT[3 * i + j] = -R1[3 * j + i];
                mul_skew(RT, b2, C);                                      // -R1^T [b2]
            } else {
                ld33(B + (lane == 1 ? CPI_REC_JB : lane == 2 ? CPI_REC_HB : lane == 4 ? CPI_REC_JA : CPI_REC_HA), X);
                mulT33(R1, X, C);
            }
#pragma unroll
            for (int e = 0; e < 9; e++) cf[9 * lane + e] = C[e];
        } else if (lane == 6) {                                           // R, q, DT
            ld33(B + CPI_REC_R, X);
            mul33(X, R1, C);
            double q[4];
            rot_2_quat(C, q);
            st33(hd + CPI_REC_R, C);
            hd[CPI_REC_Q] = q[0]; hd[CPI_REC_Q + 1] = q[1]; hd[CPI_REC_Q + 2] = q[2]; hd[CPI_REC_Q + 3] = q[3];
            hd[CPI_REC_DT] = A[CPI_REC_DT] + B[CPI_REC_DT];
        } else if (lane == 7) {                                           // alpha, beta
            const double dt2 = B[CPI_REC_DT];
            double a2[3] = {B[CPI_REC_ALPHA], B[CPI_REC_ALPHA + 1], B[CPI_REC_ALPHA + 2]}, ra[3], rb[3];
            b2[0] = B[CPI_REC_BETA]; b2[1] = B[CPI_REC_BETA + 1]; b2[2] = B[CPI_REC_BETA + 2];
            mvT33(R1, a2, ra); mvT33(R1, b2, rb);
#pragma unroll
            for (int i = 0; i < 3; i++) {
                hd[CPI_REC_BETA + i] = A[CPI_REC_BETA + i] + rb[i];
                hd[CPI_REC_ALPHA + i] = A[CPI_REC_ALPHA + i] + A[CPI_REC_BETA + i] * dt2 + ra[i];
            }
        } else if (lane == 8) {                                           // J_q = R2 J_q1 + J_q2
            ld33(B + CPI_REC_R, X); ld33(A + CPI_REC_JQ, D);
            mul33(X, D, C);
            ld33(B + CPI_REC_JQ, X);
#pragma unroll
            for (int e = 0; e < 9; e++) C[e] += X[e];
            st33(hd + CPI_REC_JQ, C);
        } else if (lane == 9 || lane == 10) {                             // H_b = H_b1 + R1^T H_b2 ;  H_a = H_a1 + H_b1 DT2 + R1^T H_a2
            const double dt2 = lane == 10 ? B[CPI_REC_DT] : 0.0;
            const int f = lane == 9 ? CPI_REC_HB : CPI_REC_HA;
            ld33(B + f, X);
            mulT33(R1, X, C);
            ld33(A + f, X); ld33(A + CPI_REC_HB, D);
#pragma unroll
            for (int e = 0; e < 9; e++) C[e] = lane == 10 ? X[e] + D[e] * dt2 + C[e] : X[e] + C[e];
            st33(hd + f, C);
        } else if (lane == 11 || lane == 12) {  // J_b = J_b1 + R1^T([b2] J_q1 + J_b2) ;  J_a = J_a1 + J_b1 DT2 + R1^T([a2] J_q1 + J_a2)
            const bool a = lane == 12;
            const int v = a ? CPI_REC_ALPHA : CPI_REC_BETA, f = a ? CPI_REC_JA : CPI_REC_JB;
            const double dt2 = a ? B[CPI_REC_DT] : 0.0;
            b2[0] = B[v]; b2[1] = B[v + 1]; b2[2] = B[v + 2];
            ld33(A + CPI_REC_JQ, D);
#pragma unroll
            for (int j = 0; j < 3; j++) {                                 // column j of [v] J_q1 = v x (column j of J_q1)
                const double c[3] = {D[j], D[3 + j], D[6 + j]};
                double o[3];
                cross(b2, c, o);
                X[j] = o[0]; X[3 + j] = o[1]; X[6 + j] = o[2];
            }
            ld33(B + f, D);
#pragma unroll
            for (int e = 0; e < 9; e++) X[e] += D[e];
            mulT33(R1, X, C);
            ld33(A + f, X); ld33(A + CPI_REC_JB, D);
#pragma unroll
            for (int e = 0; e < 9; e++) C[e] = a ? X[e] + D[e] * dt2 + C[e] : X[e] + C[e];
            st33(hd + f, C);
        }
    }
    __syncwarp();
    double x[15];
    if (lane < 15) {                                                      // M(:, j) = Phi~ P1(:, j)
        const double* p = A + CPI_REC_P + 15 * lane;
#pragma unroll
        for (int k = 0; k < 15; k++) x[k] = p[k];
        phi_apply(x, B, cf);
#pragma unroll
        for (int k = 0; k < 15; k++) M[k + 15 * lane] = x[k];
    }
    __syncwarp();
    if (lane < 15) {                                                      // P(i, :) = (Phi~ M(i, :)^T)^T + (T P2 T^T)(i, :)
        const int i = lane, I = i / 3, ii = i - 3 * I;
#pragma unroll
        for (int k = 0; k < 15; k++) x[k] = M[i + 15 * k];
        // B's P is still read below, so a result for B is first written over M, once every lane holds its row of M
        if (kRight) __syncwarp(0x7fff);
        phi_apply(x, B, cf);
        const double* P2 = B + CPI_REC_P;
        const double* R1 = A + CPI_REC_R;                                 // R1(m, c) = R1[m + 3 c]
        const bool rot_row = I == 2 || I == 4;                            // row i of T_I P2 = R1^T rows (v, p) or P2's own row
        double* P = kRight ? M : A + CPI_REC_P;
#pragma unroll
        for (int J = 0; J < 5; J++) {
            double r[3];
#pragma unroll
            for (int m = 0; m < 3; m++) {
                const int k = 3 * J + m;
                r[m] = rot_row ? R1[3 * ii] * P2[3 * I + 15 * k] + R1[3 * ii + 1] * P2[3 * I + 1 + 15 * k] + R1[3 * ii + 2] * P2[3 * I + 2 + 15 * k]
                               : P2[i + 15 * k];
            }
            if (J == 2 || J == 4) {                                       // ... T_J^T = R1 on the right
                const double s0 = r[0], s1 = r[1], s2 = r[2];
#pragma unroll
                for (int c = 0; c < 3; c++) r[c] = s0 * R1[3 * c] + s1 * R1[1 + 3 * c] + s2 * R1[2 + 3 * c];
            }
#pragma unroll
            for (int m = 0; m < 3; m++) {
                const int j = 3 * J + m;
                if (j >= i) { const double v = x[j] + r[m]; P[i + 15 * j] = v; P[j + 15 * i] = v; }
            }
        }
    }
    __syncwarp();
    double* dst = kRight ? B : A;
    for (int e = lane; e < HEAD; e += 32) dst[e] = hd[e];
    if (kRight)
        for (int e = lane; e < 225; e += 32) dst[CPI_REC_P + e] = M[e];
    __syncwarp();
}

}  // namespace rec1
}  // namespace cpi
