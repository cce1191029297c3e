/*
 * TEST INFRASTRUCTURE ONLY -- the product path (cpi_b200/) never loads, links or calls this file.
 *
 * Plain-C, dense, literal CPU restatement of the hot path of rpng/cpi (paths relative to
 * /root/reference/cpi_compare/src).  Every function cites the reference lines it follows.  It deliberately does
 * NOT use the block-sparse formulation of the CUDA kernels: the 15x15 / 21x21 products are full dense loops, the
 * way Eigen evaluates them, so that it is an independent check of the kernels' algebra.
 *
 * Parity status: PINNED.  tests/test_oracle.py checks this file against (a) oracle/_ref/libcpi_ref.so = the
 * unmodified reference compiled in place (oracle/ref_shim.cpp) when that library is present, and (b) the committed
 * golden vectors under tests/golden/ that were generated from that library by tests/golden/make_golden.py.
 *
 * Build: oracle/Makefile (gcc -O2 -ffp-contract=off: no FMA contraction, to stay close to the reference's SSE2 code).
 *
 * Precision-generic: all arithmetic is in `real`.  liboracle.so builds it as double (the restatement above);
 * liboracle_ld.so builds the same source with -DCPI_ORACLE_LONG_DOUBLE (x86-64 x87 extended precision, 64-bit mantissa) as
 * the high-precision truth the precision tests measure the kernels and the fp64 build against.  Inputs and outputs are
 * double in both builds.  The two branch decisions of the reference (small_w and dt == 0) are taken on the values the fp64
 * code sees, so the extended build evaluates the same piecewise function, only more accurately.
 */
#include "cpi_oracle.h"
#include "../include/cpi_b200.h"
#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include <tgmath.h>

#ifdef CPI_ORACLE_LONG_DOUBLE
typedef long double real;
#else
typedef double real;
#endif

/* ------------------------------------------------------------------ small dense helpers (column-major) ---------- */
#define E(M, ld, i, j) ((M)[(i) + (j) * (ld)])

static void load(real* dst, const double* src, int n) { for (int i = 0; i < n; i++) dst[i] = src[i]; }
static void store(double* dst, const real* src, int n) { for (int i = 0; i < n; i++) dst[i] = (double)src[i]; }
static void mat_zero(real* A, int n) { memset(A, 0, sizeof *A * (size_t)n); }
static void mat_eye(real* A, int n) { mat_zero(A, n * n); for (int i = 0; i < n; i++) E(A, n, i, i) = 1.0; }
/* C(m x n) = A(m x k) * B(k x n) */
static void gemm(int m, int n, int k, const real* A, const real* B, real* C) {
    for (int j = 0; j < n; j++) for (int i = 0; i < m; i++) {
        real s = 0.0;
        for (int l = 0; l < k; l++) s += E(A, m, i, l) * E(B, k, l, j);
        E(C, m, i, j) = s;
    }
}
/* C(m x n) = A(m x k) * B(n x k)^T */
static void gemm_nt(int m, int n, int k, const real* A, const real* B, real* C) {
    for (int j = 0; j < n; j++) for (int i = 0; i < m; i++) {
        real s = 0.0;
        for (int l = 0; l < k; l++) s += E(A, m, i, l) * E(B, n, j, l);
        E(C, m, i, j) = s;
    }
}
static void transpose(int m, int n, const real* A, real* At) {
    for (int i = 0; i < m; i++) for (int j = 0; j < n; j++) E(At, n, j, i) = E(A, m, i, j);
}
/* dst block (r0,c0) of size br x bc in a matrix with leading dim ld  <-  s * B */
static void set_block(real* M, int ld, int r0, int c0, int br, int bc, const real* B, real s) {
    for (int j = 0; j < bc; j++) for (int i = 0; i < br; i++) E(M, ld, r0 + i, c0 + j) = s * E(B, br, i, j);
}
static void get_block(const real* M, int ld, int r0, int c0, int br, int bc, real* B) {
    for (int j = 0; j < bc; j++) for (int i = 0; i < br; i++) E(B, br, i, j) = E(M, ld, r0 + i, c0 + j);
}
static void m3_mul(const real* A, const real* B, real* C) { real T[9]; gemm(3, 3, 3, A, B, T); memcpy(C, T, sizeof T); }
static void m3_vec(const real* A, const real* v, real* o) {
    real t[3];
    for (int i = 0; i < 3; i++) t[i] = E(A, 3, i, 0) * v[0] + E(A, 3, i, 1) * v[1] + E(A, 3, i, 2) * v[2];
    o[0] = t[0]; o[1] = t[1]; o[2] = t[2];
}
static real norm3(const real* v) { return sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }
static real norm4(const real* v) { return sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3]); }

/* ------------------------------------------------------------------ utils/quat_ops.h ----------------------------- */

/* skew_x, quat_ops.h:92-98 */
static void skew_x(const real* w, real* M) {
    E(M, 3, 0, 0) = 0;     E(M, 3, 0, 1) = -w[2]; E(M, 3, 0, 2) = w[1];
    E(M, 3, 1, 0) = w[2];  E(M, 3, 1, 1) = 0;     E(M, 3, 1, 2) = -w[0];
    E(M, 3, 2, 0) = -w[1]; E(M, 3, 2, 1) = w[0];  E(M, 3, 2, 2) = 0;
}

/* rot_2_quat, quat_ops.h:45-86 : four-case largest-diagonal extraction, force w >= 0, normalise */
static void rot_2_quat(const real* rot, real* q) {
    real r00 = E(rot, 3, 0, 0), r11 = E(rot, 3, 1, 1), r22 = E(rot, 3, 2, 2);
    real T = r00 + r11 + r22;
    if (r00 >= T && r00 >= r11 && r00 >= r22) {
        q[0] = sqrt((1 + (2 * r00) - T) / 4);
        q[1] = (1 / (4 * q[0])) * (E(rot, 3, 0, 1) + E(rot, 3, 1, 0));
        q[2] = (1 / (4 * q[0])) * (E(rot, 3, 0, 2) + E(rot, 3, 2, 0));
        q[3] = (1 / (4 * q[0])) * (E(rot, 3, 1, 2) - E(rot, 3, 2, 1));
    } else if (r11 >= T && r11 >= r00 && r11 >= r22) {
        q[1] = sqrt((1 + (2 * r11) - T) / 4);
        q[0] = (1 / (4 * q[1])) * (E(rot, 3, 0, 1) + E(rot, 3, 1, 0));
        q[2] = (1 / (4 * q[1])) * (E(rot, 3, 1, 2) + E(rot, 3, 2, 1));
        q[3] = (1 / (4 * q[1])) * (E(rot, 3, 2, 0) - E(rot, 3, 0, 2));
    } else if (r22 >= T && r22 >= r00 && r22 >= r11) {
        q[2] = sqrt((1 + (2 * r22) - T) / 4);
        q[0] = (1 / (4 * q[2])) * (E(rot, 3, 0, 2) + E(rot, 3, 2, 0));
        q[1] = (1 / (4 * q[2])) * (E(rot, 3, 1, 2) + E(rot, 3, 2, 1));
        q[3] = (1 / (4 * q[2])) * (E(rot, 3, 0, 1) - E(rot, 3, 1, 0));
    } else {
        q[3] = sqrt((1 + T) / 4);
        q[0] = (1 / (4 * q[3])) * (E(rot, 3, 1, 2) - E(rot, 3, 2, 1));
        q[1] = (1 / (4 * q[3])) * (E(rot, 3, 2, 0) - E(rot, 3, 0, 2));
        q[2] = (1 / (4 * q[3])) * (E(rot, 3, 0, 1) - E(rot, 3, 1, 0));
    }
    if (q[3] < 0) { for (int i = 0; i < 4; i++) q[i] = -q[i]; }
    real n = norm4(q);
    for (int i = 0; i < 4; i++) q[i] = q[i] / n;
}

/* quat_2_Rot, quat_ops.h:104-109 : (2 q4^2 - 1) I - 2 q4 [q_v x] + 2 q_v q_v^T */
static void quat_2_Rot(const real* q, real* R) {
    real qx[9]; skew_x(q, qx);
    real s = 2 * pow(q[3], 2) - 1;
    for (int j = 0; j < 3; j++) for (int i = 0; i < 3; i++)
        E(R, 3, i, j) = s * (i == j ? 1.0 : 0.0) - 2 * q[3] * E(qx, 3, i, j) + 2 * q[i] * q[j];
}

/* quat_multiply, quat_ops.h:115-128 : JPL product q (x) p, force w >= 0, normalise */
static void quat_multiply(const real* q, const real* p, real* out) {
    real Qm[16], qx[9], t[4];
    skew_x(q, qx);
    for (int j = 0; j < 3; j++) for (int i = 0; i < 3; i++) E(Qm, 4, i, j) = q[3] * (i == j ? 1.0 : 0.0) - E(qx, 3, i, j);
    for (int i = 0; i < 3; i++) { E(Qm, 4, i, 3) = q[i]; E(Qm, 4, 3, i) = -q[i]; }
    E(Qm, 4, 3, 3) = q[3];
    gemm(4, 1, 4, Qm, p, t);
    if (t[3] < 0) { for (int i = 0; i < 4; i++) t[i] *= -1; }
    real n = norm4(t);
    for (int i = 0; i < 4; i++) out[i] = t[i] / n;
}

/* Exp, quat_ops.h:145-162 : I + sin(th)/th [w x] + (1-cos th)/th^2 [w x]^2 ; identity iff th == 0 */
static void Exp(const real* w, real* R) {
    real wx[9], wx2[9];
    skew_x(w, wx);
    real th = norm3(w);
    if (th == 0) { mat_eye(R, 3); return; }
    gemm(3, 3, 3, wx, wx, wx2);
    real a = sin(th) / th, b = (1 - cos(th)) / pow(th, 2);
    for (int k = 0; k < 9; k++) R[k] = (k % 4 == 0 ? 1.0 : 0.0) + a * wx[k] + b * wx2[k];
}

void oracle_rot_2_quat(const double* R, double* q) { real r[9], o[4]; load(r, R, 9); rot_2_quat(r, o); store(q, o, 4); }
void oracle_quat_2_Rot(const double* q, double* R) { real a[4], o[9]; load(a, q, 4); quat_2_Rot(a, o); store(R, o, 9); }
void oracle_quat_multiply(const double* q, const double* p, double* out) {
    real a[4], b[4], o[4]; load(a, q, 4); load(b, p, 4); quat_multiply(a, b, o); store(out, o, 4);
}
void oracle_Exp(const double* w, double* R) { real a[3], o[9]; load(a, w, 3); Exp(a, o); store(R, o, 9); }

/* Inv, quat_ops.h:190-197 */
static void quat_inv(const real* q, real* o) { o[0] = -q[0]; o[1] = -q[1]; o[2] = -q[2]; o[3] = q[3]; }

/* ------------------------------------------------------------------ cpi/CpiBase.h -------------------------------- */

typedef struct {
    int imu_avg, stj;                        /* CpiBase.h:95, CpiV2.h:58 */
    real DT, alpha[3], beta[3], q[4], R[9];  /* CpiBase.h:99-103 */
    real J_q[9], J_a[9], J_b[9], H_a[9], H_b[9];  /* :106-110 */
    real O_a[9], O_b[9];                     /* CpiV2.h:62-63 */
    real b_w[3], b_a[3], q_lin[4], grav[3];  /* CpiBase.h:113-118 */
    real Qc[144];                            /* :121 */
    real P[225];                             /* :124 */
    real Pbig[441], D[441];                  /* CpiV2.h:46-49 */
} cpi_t;

/* ctor CpiBase.h:52-66 + setLinearizationPoints :73-80 + member initialisers :99-124 */
static void cpi_init(cpi_t* c, const double* sig, const double* lin, int imu_avg, int stj) {
    memset(c, 0, sizeof *c);
    c->imu_avg = imu_avg; c->stj = stj;
    for (int b = 0; b < 4; b++) for (int i = 0; i < 3; i++) E(c->Qc, 12, 3 * b + i, 3 * b + i) = pow((real)sig[b], 2);
    mat_eye(c->R, 3);
    c->q[3] = 1.0;                 /* uninitialised in the reference; see include/cpi_b200.h */
    mat_eye(c->D, 21);             /* CpiV2.h:49 */
    load(c->b_w, lin, 3); load(c->b_a, lin + 3, 3); load(c->q_lin, lin + 6, 4); load(c->grav, lin + 10, 3);
}

/* The reference's branch test |w_hat| < small_w (CpiV1.h:101), always evaluated in double exactly as the fp64 code does
 * (w_hat = w_m_0 - b_w, averaged with w_m_1 - b_w under imu_avg; the same in both models). */
static int small_w_branch(const double* w_m_0, const double* w_m_1, const real* b_w, int imu_avg) {
    double w[3];
    for (int i = 0; i < 3; i++) {
        w[i] = w_m_0[i] - (double)b_w[i];
        if (imu_avg) { w[i] += w_m_1[i] - (double)b_w[i]; w[i] = 0.5 * w[i]; }
    }
    double mag_w = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    return mag_w < 0.008726646;
}

/* Closed-form scalars shared by both models.  CpiV1.h:132-142 & 196-238  ==  CpiV2.h:158-168 & 231-274 */
typedef struct { real f1, f2, f3, f4, df1, df2, df3, df4; } coef_t;
static void coefficients(int small_w, real dt, real mag_w, real w_dt, real s, real c, coef_t* k) {
    if (small_w) {
        k->f1 = -(pow(dt, 3) / 3); k->f2 = (pow(dt, 4) / 8); k->f3 = -(pow(dt, 2) / 2); k->f4 = (pow(dt, 3) / 6);
        k->df1 = -(pow(dt, 5) / 15); k->df2 = (pow(dt, 6) / 72); k->df3 = -(pow(dt, 4) / 12); k->df4 = (pow(dt, 5) / 60);
    } else {
        k->f1 = (w_dt * c - s) / (pow(mag_w, 3));
        k->f2 = (pow(w_dt, 2) - 2 * c - 2 * w_dt * s + 2) / (2 * pow(mag_w, 4));
        k->f3 = -(1 - c) / pow(mag_w, 2);
        k->f4 = (w_dt - s) / pow(mag_w, 3);
        k->df1 = (pow(w_dt, 2) * s - 3 * s + 3 * w_dt * c) / pow(mag_w, 5);
        k->df2 = (pow(w_dt, 2) - 4 * c - 4 * w_dt * s + pow(w_dt, 2) * c + 4) / (pow(mag_w, 6));
        k->df3 = (2 * (c - 1) + w_dt * s) / (pow(mag_w, 4));
        k->df4 = (2 * w_dt + w_dt * c - 3 * s) / (pow(mag_w, 5));
    }
}

/* I - a*W + b*W2  (the three rotation expressions CpiV1.h:119-120, 267-268; CpiV2.h:138-139, 321-322) */
static void rot_from(real a, real b, const real* W, const real* W2, real* R) {
    for (int k = 0; k < 9; k++) R[k] = (k % 4 == 0 ? 1.0 : 0.0) - a * W[k] + b * W2[k];
}

/* Dense Lyapunov right-hand side  F P + P F^T + G Qc G^T  for n = 15 or 21  (CpiV1.h:291, CpiV2.h:348) */
static void lyap_rhs(int n, const real* F, const real* G, const real* Qc, const real* P, real* out) {
    real FP[441], PFt[441], GQ[21 * 12], GQGt[441];
    gemm(n, n, n, F, P, FP);
    gemm_nt(n, n, n, P, F, PFt);
    gemm(n, 12, 12, G, Qc, GQ);
    gemm_nt(n, n, 12, GQ, G, GQGt);
    for (int k = 0; k < n * n; k++) out[k] = FP[k] + PFt[k] + GQGt[k];
}

/* F and G for one RK4 stage.  CpiV1.h:276-288 (n=15); CpiV2.h:330-344 (n=21, with the two gravity blocks) */
static void build_FG(int n, const real* w_x, const real* a_x, const real* Rstar, const real* R_old,
                     const real* RGk, const real* grav, real* F, real* G) {
    real RsT[9], t[9], eye[9];
    mat_zero(F, n * n); mat_zero(G, n * 12); mat_eye(eye, 3);
    transpose(3, 3, Rstar, RsT);
    set_block(F, n, 0, 0, 3, 3, w_x, -1.0);
    set_block(F, n, 0, 3, 3, 3, eye, -1.0);
    gemm(3, 3, 3, RsT, a_x, t); set_block(F, n, 6, 0, 3, 3, t, -1.0);
    set_block(F, n, 6, 9, 3, 3, RsT, -1.0);
    set_block(F, n, 12, 6, 3, 3, eye, 1.0);
    if (n == 21) {
        real g_k[3], g_tau[3], sk[9], t2[9];
        m3_vec(RGk, grav, g_k);                       /* R_G_to_k * grav */
        m3_vec(R_old, g_k, g_tau);                    /* R_k2tau * R_G_to_k * grav  (always the OLD R_k2tau) */
        skew_x(g_tau, sk); gemm(3, 3, 3, RsT, sk, t); set_block(F, n, 6, 15, 3, 3, t, -1.0);        /* CpiV2.h:335 */
        skew_x(g_k, sk); gemm(3, 3, 3, RsT, R_old, t2); gemm(3, 3, 3, t2, sk, t); set_block(F, n, 6, 18, 3, 3, t, -1.0); /* :336 */
    }
    set_block(G, n, 0, 0, 3, 3, eye, -1.0);
    set_block(G, n, 3, 3, 3, 3, eye, 1.0);
    set_block(G, n, 6, 6, 3, 3, RsT, -1.0);
    set_block(G, n, 9, 9, 3, 3, eye, 1.0);
}

/* The analytic mean / bias-Jacobian part that the two models share textually.
 * model 1: CpiV1.h:119-259.  model 2: CpiV2.h:138-305 (adds O_a/O_b and the gravity terms, incl. the sign slip at :296-297).
 * Outputs R1 (= R_k2tau1) and leaves c->R untouched (the caller commits it after the covariance, CpiV1.h:357). */
static void means_and_jacobians(cpi_t* c, int model, real dt, const real* w_hat, real* a_hat,
                                const double* a_m_1, real mag_w, real w_dt, int small_w, real sin_wt, real cos_wt,
                                const real* w_x, const real* w_tx, const real* w_x_2, real* R1) {
    real eye[9], Rstep[9], R1T[9];
    mat_eye(eye, 3);
    real dt_2 = pow(dt, 2);
    if (small_w) rot_from(dt, pow(dt, 2) / 2, w_x, w_x_2, Rstep);
    else rot_from(sin_wt / mag_w, (1.0 - cos_wt) / (pow(mag_w, 2.0)), w_x, w_x_2, Rstep);
    gemm(3, 3, 3, Rstep, c->R, R1);
    transpose(3, 3, R1, R1T);

    real RGk[9], g_k[3] = {0, 0, 0}, g_tau[3] = {0, 0, 0};
    if (model == 2) {
        quat_2_Rot(c->q_lin, RGk);
        if (c->imu_avg) {            /* CpiV2.h:146-149 : average the LOCAL acceleration using the NEW rotation */
            real t[3], u[3];
            m3_vec(RGk, c->grav, t); m3_vec(R1, t, u);
            for (int i = 0; i < 3; i++) { a_hat[i] += a_m_1[i] - c->b_a[i] - u[i]; a_hat[i] = 0.5 * a_hat[i]; }
        }
        m3_vec(RGk, c->grav, g_k);   /* :202 */
        m3_vec(c->R, g_k, g_tau);    /* :277 */
    }

    coef_t k; coefficients(small_w, dt, mag_w, w_dt, sin_wt, cos_wt, &k);
    real alpha_arg[9], Beta_arg[9], H_al[9], H_be[9], t3[3];
    for (int i = 0; i < 9; i++) {
        alpha_arg[i] = ((dt_2 / 2.0) * eye[i] + k.f1 * w_x[i] + k.f2 * w_x_2[i]);
        Beta_arg[i] = (dt * eye[i] + k.f3 * w_x[i] + k.f4 * w_x_2[i]);
    }
    gemm(3, 3, 3, R1T, alpha_arg, H_al);
    gemm(3, 3, 3, R1T, Beta_arg, H_be);
    m3_vec(H_al, a_hat, t3);
    for (int i = 0; i < 3; i++) c->alpha[i] += c->beta[i] * dt + t3[i];     /* old beta */
    m3_vec(H_be, a_hat, t3);
    for (int i = 0; i < 3; i++) c->beta[i] += t3[i];

    /* right Jacobian and J_q */
    real J_r[9], wtx2[9], J_save[9], t9[9];
    gemm(3, 3, 3, w_tx, w_tx, wtx2);
    if (small_w) for (int i = 0; i < 9; i++) J_r[i] = eye[i] - .5 * w_tx[i] + ((real)1 / 6) * wtx2[i];
    else for (int i = 0; i < 9; i++)
        J_r[i] = eye[i] - ((1 - cos_wt) / (pow((w_dt), 2.0))) * w_tx[i] + ((w_dt - sin_wt) / (pow(w_dt, 3.0))) * wtx2[i];
    memcpy(J_save, c->J_q, sizeof J_save);
    gemm(3, 3, 3, Rstep, c->J_q, t9);
    for (int i = 0; i < 9; i++) c->J_q[i] = t9[i] + J_r[i] * dt;

    for (int i = 0; i < 9; i++) c->H_a[i] -= H_al[i];
    for (int i = 0; i < 9; i++) c->H_a[i] += dt * c->H_b[i];      /* old H_b */
    for (int i = 0; i < 9; i++) c->H_b[i] -= H_be[i];

    if (model == 2) {                /* CpiV2.h:203-205 */
        real sk[9], t1[9], t2[9];
        skew_x(g_k, sk);
        for (int i = 0; i < 9; i++) c->O_a[i] += dt * c->O_b[i];
        gemm(3, 3, 3, H_al, c->R, t1); gemm(3, 3, 3, t1, sk, t2);
        for (int i = 0; i < 9; i++) c->O_a[i] += -t2[i];
        gemm(3, 3, 3, H_be, c->R, t1); gemm(3, 3, 3, t1, sk, t2);
        for (int i = 0; i < 9; i++) c->O_b[i] += -t2[i];
    }

    for (int i = 0; i < 9; i++) c->J_a[i] += c->J_b[i] * dt;      /* old J_b */
    for (int col = 0; col < 3; col++) {
        real e[3] = {0, 0, 0}, ex[9], Jq_e[3], sk[9], dR[9], inner[9], exw[9], wex[9], M[9], v[3];
        e[col] = 1.0; skew_x(e, ex);
        m3_vec(c->J_q, e, Jq_e);                /* NEW J_q */
        skew_x(Jq_e, sk); gemm(3, 3, 3, R1T, sk, dR);
        for (int i = 0; i < 9; i++) dR[i] = -dR[i];
        gemm(3, 3, 3, ex, w_x, exw); gemm(3, 3, 3, w_x, ex, wex);
        real wi = w_hat[col];
        /* J_a column */
        for (int i = 0; i < 9; i++) inner[i] = (wi * k.df1) * w_x[i] - k.f1 * ex[i] + (wi * k.df2) * w_x_2[i] - k.f2 * (exw[i] + wex[i]);
        gemm(3, 3, 3, dR, alpha_arg, M); gemm(3, 3, 3, R1T, inner, t9);
        for (int i = 0; i < 9; i++) M[i] += t9[i];
        m3_vec(M, a_hat, v);
        if (model == 2) {
            real Js_e[3], sk2[9], t1[9], u[3];
            m3_vec(J_save, e, Js_e); skew_x(Js_e, sk2); gemm(3, 3, 3, H_al, sk2, t1); m3_vec(t1, g_tau, u);
            for (int i = 0; i < 3; i++) v[i] = v[i] - u[i];                          /* CpiV2.h:285, 289, 293 */
        }
        for (int i = 0; i < 3; i++) E(c->J_a, 3, i, col) += v[i];
        /* J_b column */
        for (int i = 0; i < 9; i++) inner[i] = (wi * k.df3) * w_x[i] - k.f3 * ex[i] + (wi * k.df4) * w_x_2[i] - k.f4 * (exw[i] + wex[i]);
        gemm(3, 3, 3, dR, Beta_arg, M); gemm(3, 3, 3, R1T, inner, t9);
        for (int i = 0; i < 9; i++) M[i] += t9[i];
        m3_vec(M, a_hat, v);
        if (model == 2) {
            real Js_e[3], sk2[9], t1[9], u[3];
            m3_vec(J_save, e, Js_e); skew_x(Js_e, sk2); gemm(3, 3, 3, H_be, sk2, t1); m3_vec(t1, g_tau, u);
            /* CpiV2.h:296-297 reads "a_hat-\n-H_be*..." : a double minus, i.e. PLUS, for column 0 only */
            for (int i = 0; i < 3; i++) v[i] = (col == 0) ? v[i] + u[i] : v[i] - u[i];
        }
        for (int i = 0; i < 3; i++) E(c->J_b, 3, i, col) += v[i];
    }
}

/* CpiV1::feed_IMU, CpiV1.h:62-361 */
static void feed_imu_v1(cpi_t* c, real dt, const double* w_m_0, const double* a_m_0, const double* w_m_1, const double* a_m_1) {
    c->DT += dt;                                             /* :69 */
    if (dt == 0) return;                                     /* :72-74 */
    real w_hat[3], a_hat[3], w_hatdt[3];
    for (int i = 0; i < 3; i++) { w_hat[i] = w_m_0[i] - c->b_w[i]; a_hat[i] = a_m_0[i] - c->b_a[i]; }
    if (c->imu_avg) for (int i = 0; i < 3; i++) {            /* :81-86 */
        w_hat[i] += w_m_1[i] - c->b_w[i]; w_hat[i] = 0.5 * w_hat[i];
        a_hat[i] += a_m_1[i] - c->b_a[i]; a_hat[i] = .5 * a_hat[i];
    }
    for (int i = 0; i < 3; i++) w_hatdt[i] = w_hat[i] * dt;
    real mag_w = norm3(w_hat), w_dt = mag_w * dt;
    int small_w = small_w_branch(w_m_0, w_m_1, c->b_w, c->imu_avg);   /* :101 */
    real cos_wt = cos(w_dt), sin_wt = sin(w_dt);
    real w_x[9], a_x[9], w_tx[9], w_x_2[9], R1[9];
    skew_x(w_hat, w_x); skew_x(a_hat, a_x); skew_x(w_hatdt, w_tx); gemm(3, 3, 3, w_x, w_x, w_x_2);

    means_and_jacobians(c, 1, dt, w_hat, a_hat, a_m_1, mag_w, w_dt, small_w, sin_wt, cos_wt, w_x, w_tx, w_x_2, R1);

    /* covariance, RK4 on the Lyapunov ODE, :267-353 */
    real R_mid[9], t9[9];
    if (small_w) rot_from(.5 * dt, pow(.5 * dt, 2) / 2, w_x, w_x_2, t9);
    else rot_from(sin(mag_w * .5 * dt) / mag_w, (1.0 - cos(mag_w * .5 * dt)) / (pow(mag_w, 2.0)), w_x, w_x_2, t9);
    gemm(3, 3, 3, t9, c->R, R_mid);

    real F[225], G[180], k1[225], k2[225], k3[225], k4[225], Ps[225];
    build_FG(15, w_x, a_x, c->R, 0, 0, 0, F, G);  lyap_rhs(15, F, G, c->Qc, c->P, k1);
    build_FG(15, w_x, a_x, R_mid, 0, 0, 0, F, G);
    for (int i = 0; i < 225; i++) Ps[i] = c->P[i] + k1[i] * dt / 2.0;
    lyap_rhs(15, F, G, c->Qc, Ps, k2);
    for (int i = 0; i < 225; i++) Ps[i] = c->P[i] + k2[i] * dt / 2.0;
    lyap_rhs(15, F, G, c->Qc, Ps, k3);
    build_FG(15, w_x, a_x, R1, 0, 0, 0, F, G);
    for (int i = 0; i < 225; i++) Ps[i] = c->P[i] + k3[i] * dt;
    lyap_rhs(15, F, G, c->Qc, Ps, k4);
    for (int i = 0; i < 225; i++) c->P[i] += (dt / 6.0) * (k1[i] + 2.0 * k2[i] + 2.0 * k3[i] + k4[i]);
    transpose(15, 15, c->P, Ps);
    for (int i = 0; i < 225; i++) c->P[i] = 0.5 * (c->P[i] + Ps[i]);         /* :353 */

    memcpy(c->R, R1, sizeof c->R);                                            /* :357 */
    rot_2_quat(c->R, c->q);                                            /* :358 */
}

/* CpiV2::feed_IMU, CpiV2.h:84-467 */
static void feed_imu_v2(cpi_t* c, real dt, const double* w_m_0, const double* a_m_0, const double* w_m_1, const double* a_m_1) {
    c->DT += dt;
    if (dt == 0) return;
    real RGk[9], w_hat[3], a_hat[3], w_hatdt[3], t3[3], u3[3];
    quat_2_Rot(c->q_lin, RGk);
    m3_vec(RGk, c->grav, t3); m3_vec(c->R, t3, u3);          /* R_k2tau*quat_2_Rot(q_k_lin)*grav, :99 */
    for (int i = 0; i < 3; i++) { w_hat[i] = w_m_0[i] - c->b_w[i]; a_hat[i] = a_m_0[i] - c->b_a[i] - u3[i]; }
    if (c->imu_avg) for (int i = 0; i < 3; i++) { w_hat[i] += w_m_1[i] - c->b_w[i]; w_hat[i] = 0.5 * w_hat[i]; }
    for (int i = 0; i < 3; i++) w_hatdt[i] = w_hat[i] * dt;
    real mag_w = norm3(w_hat), w_dt = mag_w * dt;
    int small_w = small_w_branch(w_m_0, w_m_1, c->b_w, c->imu_avg);
    real cos_wt = cos(w_dt), sin_wt = sin(w_dt);
    real w_x[9], a_x[9], w_tx[9], w_x_2[9], R1[9];
    skew_x(w_hat, w_x); skew_x(w_hatdt, w_tx); gemm(3, 3, 3, w_x, w_x, w_x_2);

    means_and_jacobians(c, 2, dt, w_hat, a_hat, a_m_1, mag_w, w_dt, small_w, sin_wt, cos_wt, w_x, w_tx, w_x_2, R1);
    skew_x(a_hat, a_x);                                      /* :150 (after the optional averaging) */

    real dt_mid = dt / 2.0, w_dt_mid = mag_w * dt_mid, R_mid[9], t9[9];
    if (small_w) rot_from(dt_mid, pow(dt_mid, 2) / 2, w_x, w_x_2, t9);
    else rot_from(sin(w_dt_mid) / mag_w, (1.0 - cos(w_dt_mid)) / (pow(mag_w, 2.0)), w_x, w_x_2, t9);
    gemm(3, 3, 3, t9, c->R, R_mid);

    enum { N = 21, NN = 441 };
    real F1[NN], F2[NN], F4[NN], G[N * 12], I21[NN];
    real Pd1[NN], Pd2[NN], Pd3[NN], Pd4[NN], Ph1[NN], Ph2[NN], Ph3[NN], Ph4[NN], Ps[NN], Phs[NN];
    mat_eye(I21, N);
    /* k1 :330-348 */
    build_FG(N, w_x, a_x, c->R, c->R, RGk, c->grav, F1, G);
    memcpy(Ph1, F1, sizeof Ph1);
    lyap_rhs(N, F1, G, c->Qc, c->Pbig, Pd1);
    /* k2 :354-374 */
    build_FG(N, w_x, a_x, R_mid, c->R, RGk, c->grav, F2, G);
    for (int i = 0; i < NN; i++) { Phs[i] = I21[i] + Ph1[i] * dt_mid; Ps[i] = c->Pbig[i] + Pd1[i] * dt_mid; }
    gemm(N, N, N, F2, Phs, Ph2);
    lyap_rhs(N, F2, G, c->Qc, Ps, Pd2);
    /* k3 :381-388 */
    for (int i = 0; i < NN; i++) { Phs[i] = I21[i] + Ph2[i] * dt_mid; Ps[i] = c->Pbig[i] + Pd2[i] * dt_mid; }
    gemm(N, N, N, F2, Phs, Ph3);
    lyap_rhs(N, F2, G, c->Qc, Ps, Pd3);
    /* k4 :394-414 */
    build_FG(N, w_x, a_x, R1, c->R, RGk, c->grav, F4, G);
    for (int i = 0; i < NN; i++) { Phs[i] = I21[i] + Ph3[i] * dt; Ps[i] = c->Pbig[i] + Pd3[i] * dt; }
    gemm(N, N, N, F4, Phs, Ph4);
    lyap_rhs(N, F4, G, c->Qc, Ps, Pd4);
    /* combine :421-426 */
    real Phi[NN];
    for (int i = 0; i < NN; i++) c->Pbig[i] += (dt / 6.0) * (Pd1[i] + 2.0 * Pd2[i] + 2.0 * Pd3[i] + Pd4[i]);
    transpose(N, N, c->Pbig, Ps);
    for (int i = 0; i < NN; i++) c->Pbig[i] = 0.5 * (c->Pbig[i] + Ps[i]);
    for (int i = 0; i < NN; i++) Phi[i] = I21[i] + (dt / 6.0) * (Ph1[i] + 2.0 * Ph2[i] + 2.0 * Ph3[i] + Ph4[i]);
    /* clone + marginalise :436-446 */
    real B[NN], T1[NN], T2[NN];
    mat_eye(B, N);
    for (int i = 0; i < 3; i++) { E(B, N, 15 + i, 15 + i) = 0.0; E(B, N, 15 + i, i) = 1.0; }
    gemm(N, N, N, B, c->Pbig, T1); gemm_nt(N, N, N, T1, B, T2);
    transpose(N, N, T2, T1);
    for (int i = 0; i < NN; i++) c->Pbig[i] = 0.5 * (T2[i] + T1[i]);
    gemm(N, N, N, Phi, c->D, T1); gemm(N, N, N, B, T1, T2);     /* B_k * Phi * Discrete_J_b */
    memcpy(c->D, T2, sizeof T2);
    get_block(c->Pbig, N, 0, 0, 15, 15, c->P);
    if (c->stj) {                                               /* :450-458 */
        get_block(c->D, N, 0, 3, 3, 3, c->J_q); for (int i = 0; i < 9; i++) c->J_q[i] = -c->J_q[i];
        get_block(c->D, N, 12, 3, 3, 3, c->J_a); get_block(c->D, N, 6, 3, 3, 3, c->J_b);
        get_block(c->D, N, 12, 9, 3, 3, c->H_a); get_block(c->D, N, 6, 9, 3, 3, c->H_b);
        get_block(c->D, N, 12, 18, 3, 3, c->O_a); get_block(c->D, N, 6, 18, 3, 3, c->O_b);
    }
    memcpy(c->R, R1, sizeof c->R);
    rot_2_quat(c->R, c->q);
}

static void window(int model, const double* s, int64_t entries, const double* lin, const double* sig, int flags, double* rec) {
    int avg = (flags & CPI_FLAG_IMU_AVG) != 0;
    int64_t steps = avg ? (entries > 0 ? entries - 1 : 0) : entries;
    cpi_t* c = (cpi_t*)malloc(sizeof(cpi_t));
    cpi_init(c, sig, lin, avg, (flags & CPI_FLAG_ANALYTIC_JACOBIANS) == 0);
    for (int64_t i = 0; i < steps; i++) {       /* driver loop: GraphSolver_IMU.cpp:50-69 */
        const double* e0 = s + i * CPI_SAMPLE_DOUBLES;
        const double* e1 = avg ? e0 + CPI_SAMPLE_DOUBLES : e0;
        if (model == 1) feed_imu_v1(c, e0[6], e0, e0 + 3, e1, e1 + 3);
        else feed_imu_v2(c, e0[6], e0, e0 + 3, e1, e1 + 3);
    }
    store(rec + CPI_REC_Q, c->q, 4); store(rec + CPI_REC_R, c->R, 9);
    store(rec + CPI_REC_ALPHA, c->alpha, 3); store(rec + CPI_REC_BETA, c->beta, 3);
    rec[CPI_REC_DT] = (double)c->DT;
    store(rec + CPI_REC_JQ, c->J_q, 9); store(rec + CPI_REC_JA, c->J_a, 9); store(rec + CPI_REC_JB, c->J_b, 9);
    store(rec + CPI_REC_HA, c->H_a, 9); store(rec + CPI_REC_HB, c->H_b, 9);
    store(rec + CPI_REC_P, c->P, 225);
    if (model == 2) { store(rec + CPI_REC_OA, c->O_a, 9); store(rec + CPI_REC_OB, c->O_b, 9); }
    free(c);
}

/* ------------------------------------------------------------------ gtsam/ImuFactorCPIv1.cpp, ImuFactorCPIv2.cpp -- */

/* w*I - skew(v) (sign = -1) or w*I + skew(v) (sign = +1) */
static void quat_mat(const real* q, real sign, real* M) {
    real sk[9]; skew_x(q, sk);
    for (int i = 0; i < 9; i++) M[i] = q[3] * (i % 4 == 0 ? 1.0 : 0.0) + sign * sk[i];
}

/* ImuFactorCPIv1::evaluateError (ImuFactorCPIv1.cpp:37-208); model 2: ImuFactorCPIv2.cpp:38-212 */
/* on states held in `real` (propagate_one keeps x_k1 unrounded); the entry below loads double states */
static void factor_eval_r(int model, const real* xi, const real* xj, const double* r_in, const double* l_in,
                          real* err, real* Hi, real* Hj) {
    real r[CPI_REC_V2_DOUBLES], l[CPI_LIN_DOUBLES];
    load(l, l_in, CPI_LIN_DOUBLES);
    load(r, r_in, model == 1 ? CPI_REC_V1_DOUBLES : CPI_REC_V2_DOUBLES);
    const real *q_GtoK = xi, *bg_K = xi + 4, *v_K = xi + 7, *ba_K = xi + 10, *p_K = xi + 13;
    const real *q_GtoK1 = xj, *bg_K1 = xj + 4, *v_K1 = xj + 7, *ba_K1 = xj + 10, *p_K1 = xj + 13;
    const real *bg_lin = l, *ba_lin = l + 3, *q_K_lin = l + 6, *grav = l + 10;
    const real *q_KtoK1 = r + CPI_REC_Q, *alpha = r + CPI_REC_ALPHA, *beta = r + CPI_REC_BETA;
    const real *J_q = r + CPI_REC_JQ, *J_alpha = r + CPI_REC_JA, *J_beta = r + CPI_REC_JB;
    const real *H_alpha = r + CPI_REC_HA, *H_beta = r + CPI_REC_HB;
    const real *O_alpha = r + CPI_REC_OA, *O_beta = r + CPI_REC_OB;
    real deltatime = r[CPI_REC_DT];

    real dbg[3], dba[3], t3[3], ExpB[9], q_b[4], qi[4], q_n[4], q_rminus[4], q_r[4], q_m[4];
    for (int i = 0; i < 3; i++) { dbg[i] = bg_K[i] - bg_lin[i]; dba[i] = ba_K[i] - ba_lin[i]; }
    m3_vec(J_q, dbg, t3); for (int i = 0; i < 3; i++) t3[i] = -t3[i];
    Exp(t3, ExpB); rot_2_quat(ExpB, q_b);                       /* :57-58 */
    quat_inv(q_GtoK, qi); quat_multiply(q_GtoK1, qi, q_n);             /* :61 */
    quat_inv(q_KtoK1, qi); quat_multiply(q_n, qi, q_rminus);           /* :62 */
    quat_multiply(q_rminus, q_b, q_r);                                 /* :63 */
    quat_inv(q_b, qi); quat_multiply(qi, q_KtoK1, q_m);                /* :64 */

    real q_kR[4] = {0, 0, 0, 1}, dthk[3] = {0, 0, 0};
    if (model == 2) {                                                         /* v2 :68-69 */
        quat_inv(q_K_lin, qi); quat_multiply(q_GtoK, qi, q_kR);
        for (int i = 0; i < 3; i++) dthk[i] = 2 * q_kR[i];
    }
    real Rk[9], pa[3], pb[3], alphahat[3], betahat[3], u[3], w[3], o[3];
    quat_2_Rot(q_GtoK, Rk);
    for (int i = 0; i < 3; i++) {
        if (model == 1) {                                                     /* v1 :70, :72 */
            pa[i] = p_K1[i] - p_K[i] - v_K[i] * deltatime + 0.5 * grav[i] * pow(deltatime, 2);
            pb[i] = v_K1[i] - v_K[i] + grav[i] * deltatime;
        } else {                                                              /* v2 :72, :74 */
            pa[i] = p_K1[i] - p_K[i] - v_K[i] * deltatime;
            pb[i] = v_K1[i] - v_K[i];
        }
    }
    m3_vec(Rk, pa, alphahat); m3_vec(J_alpha, dbg, u); m3_vec(H_alpha, dba, w);
    if (model == 2) m3_vec(O_alpha, dthk, o); else o[0] = o[1] = o[2] = 0;
    for (int i = 0; i < 3; i++) alphahat[i] = model == 2 ? alphahat[i] - u[i] - w[i] - o[i] : alphahat[i] - u[i] - w[i];
    m3_vec(Rk, pb, betahat); m3_vec(J_beta, dbg, u); m3_vec(H_beta, dba, w);
    if (model == 2) m3_vec(O_beta, dthk, o);
    for (int i = 0; i < 3; i++) betahat[i] = model == 2 ? betahat[i] - u[i] - w[i] - o[i] : betahat[i] - u[i] - w[i];

    for (int i = 0; i < 3; i++) {                                             /* :84-88 */
        err[i] = 2 * q_r[i];
        err[3 + i] = bg_K1[i] - bg_K[i];
        err[6 + i] = betahat[i] - beta[i];
        err[9 + i] = ba_K1[i] - ba_K[i];
        err[12 + i] = alphahat[i] - alpha[i];
    }
    real eye[9]; mat_eye(eye, 3);
    if (Hi) {                                                                 /* :98-154 */
        real A[9], Bm[9], AB[9], blk[9], sk[9], v3[3];
        mat_zero(Hi, 225);
        quat_mat(q_n, -1.0, A); quat_mat(q_m, -1.0, Bm); gemm(3, 3, 3, A, Bm, AB);
        for (int j = 0; j < 3; j++) for (int i = 0; i < 3; i++) E(blk, 3, i, j) = -(E(AB, 3, i, j) + q_n[i] * q_m[j]);
        set_block(Hi, 15, 0, 0, 3, 3, blk, 1.0);                              /* :109-111 */
        m3_vec(Rk, pb, v3); skew_x(v3, sk);
        if (model == 2) { real qm[9], t[9]; quat_mat(q_kR, +1.0, qm); gemm(3, 3, 3, O_beta, qm, t); for (int i = 0; i < 9; i++) sk[i] -= t[i]; }
        set_block(Hi, 15, 6, 0, 3, 3, sk, 1.0);                               /* :113 / v2 :115-116 */
        m3_vec(Rk, pa, v3); skew_x(v3, sk);
        if (model == 2) { real qm[9], t[9]; quat_mat(q_kR, +1.0, qm); gemm(3, 3, 3, O_alpha, qm, t); for (int i = 0; i < 9; i++) sk[i] -= t[i]; }
        set_block(Hi, 15, 12, 0, 3, 3, sk, 1.0);                              /* :115 / v2 :118-119 */
        quat_mat(q_rminus, -1.0, A); gemm(3, 3, 3, A, J_q, blk);
        set_block(Hi, 15, 0, 3, 3, 3, blk, 1.0);                              /* :119 */
        set_block(Hi, 15, 3, 3, 3, 3, eye, -1.0);                             /* :121 */
        set_block(Hi, 15, 6, 3, 3, 3, J_beta, -1.0);                          /* :123 */
        set_block(Hi, 15, 12, 3, 3, 3, J_alpha, -1.0);                        /* :125 */
        set_block(Hi, 15, 6, 6, 3, 3, Rk, -1.0);                              /* :129 */
        set_block(Hi, 15, 12, 6, 3, 3, Rk, -deltatime);                       /* :131 */
        set_block(Hi, 15, 6, 9, 3, 3, H_beta, -1.0);                          /* :135 */
        set_block(Hi, 15, 9, 9, 3, 3, eye, -1.0);                             /* :137 */
        set_block(Hi, 15, 12, 9, 3, 3, H_alpha, -1.0);                        /* :139 */
        set_block(Hi, 15, 12, 12, 3, 3, Rk, -1.0);                            /* :143 */
    }
    if (Hj) {                                                                 /* :158-198 */
        real A[9];
        mat_zero(Hj, 225);
        quat_mat(q_r, +1.0, A); set_block(Hj, 15, 0, 0, 3, 3, A, 1.0);        /* :169 */
        set_block(Hj, 15, 3, 3, 3, 3, eye, 1.0);
        set_block(Hj, 15, 6, 6, 3, 3, Rk, 1.0);
        set_block(Hj, 15, 9, 9, 3, 3, eye, 1.0);
        set_block(Hj, 15, 12, 12, 3, 3, Rk, 1.0);
    }
}

static void factor_eval(int model, const double* xi_in, const double* xj_in, const double* r_in, const double* l_in,
                        double* err_out, double* H1, double* H2) {
    real xi[CPI_STATE_DOUBLES], xj[CPI_STATE_DOUBLES], err[15], Hi[225], Hj[225];
    load(xi, xi_in, CPI_STATE_DOUBLES); load(xj, xj_in, CPI_STATE_DOUBLES);
    factor_eval_r(model, xi, xj, r_in, l_in, err, H1 ? Hi : 0, H2 ? Hj : 0);
    if (H1) store(H1, Hi, 225);
    if (H2) store(H2, Hj, 225);
    store(err_out, err, 15);
}

/* getpredictedstate_v1 / _v2, solvers/GraphSolver_IMU.cpp:263-307 */
static void predict_state_r(int model, const real* x, const double* r_in, const double* l_in, real* o) {
    real r[CPI_REC_V2_DOUBLES], l[CPI_LIN_DOUBLES];
    load(l, l_in, CPI_LIN_DOUBLES); load(r, r_in, model == 1 ? CPI_REC_V1_DOUBLES : CPI_REC_V2_DOUBLES);
    const real *q_GtoK = x, *bg_K = x + 4, *v_K = x + 7, *ba_K = x + 10, *p_K = x + 13, *grav = l + 10;
    real dt = r[CPI_REC_DT], qi[4], Rinv[9], rb[3], ra[3];
    quat_multiply(r + CPI_REC_Q, q_GtoK, o);
    quat_inv(q_GtoK, qi); quat_2_Rot(qi, Rinv);
    m3_vec(Rinv, r + CPI_REC_BETA, rb); m3_vec(Rinv, r + CPI_REC_ALPHA, ra);
    for (int i = 0; i < 3; i++) {
        o[4 + i] = bg_K[i]; o[10 + i] = ba_K[i];
        if (model == 1) {
            o[7 + i] = v_K[i] - grav[i] * dt + rb[i];
            o[13 + i] = p_K[i] + v_K[i] * dt - 0.5 * grav[i] * pow(dt, 2) + ra[i];
        } else {
            o[7 + i] = v_K[i] + rb[i];
            o[13 + i] = p_K[i] + v_K[i] * dt + ra[i];
        }
    }
}

static void predict_state(int model, const double* x_in, const double* r_in, const double* l_in, double* o_out) {
    real x[CPI_STATE_DOUBLES], o[CPI_STATE_DOUBLES];
    load(x, x_in, CPI_STATE_DOUBLES);
    predict_state_r(model, x, r_in, l_in, o);
    store(o_out, o, CPI_STATE_DOUBLES);
}

/* JPLNavState::retract, gtsam/JPLNavState.cpp:37-71 */
static void retract(const double* x_in, const double* xi_in, double* o_out) {
    real x[CPI_STATE_DOUBLES], xi[15], o[CPI_STATE_DOUBLES];
    load(x, x_in, CPI_STATE_DOUBLES); load(xi, xi_in, 15);
    real n = norm3(xi), dq[4];
    for (int i = 0; i < 3; i++) dq[i] = ((sin(n / 2) / n)) * xi[i];
    dq[3] = cos(n / 2);
    real nn = norm4(dq);
    for (int i = 0; i < 4; i++) dq[i] = dq[i] / nn;
    if (dq[3] < 0) for (int i = 0; i < 4; i++) dq[i] = -dq[i];
    if (isnan(norm4(dq))) { dq[0] = dq[1] = dq[2] = 0; dq[3] = 1.0; }
    quat_multiply(dq, x, o);
    for (int i = 0; i < 12; i++) o[4 + i] = x[4 + i] + xi[3 + i];
    store(o_out, o, CPI_STATE_DOUBLES);
}

/* ------------------------------------------------------------------ K7: covariance propagation (DESIGN.md 3d) ----- */
/* Not a reference routine: a statement of cpi_propagate_batch, x_k1 = predict_state(x_k), H1 / H2 the dense Jacobians of
 * factor_eval at (x_k, x_k1), A = -H2^-1 H1, B = H2^-1, Sigma_k1 = A Sigma_k A^T + B P_meas B^T, C = Sigma_k A^T.  x_k1 stays in
 * `real`, so the long-double build forms the Jacobians at the unrounded prediction.  order 0 is independent of the kernel's algebra:
 * B by a pivoted Gauss-Jordan inverse of the dense H2 and every product a dense 15x15 one.  order 1 restates propagate.cu: the
 * closed-form Q^-1 and Rk^T, the sparse theta / v / p rows of A with their exact I and DT I blocks, N = A Sigma_k column by column,
 * Sigma_k1 row by row from N with its upper triangle mirrored, C = N^T. */

/* Inv = M^-1 (n x n, column-major) by Gauss-Jordan elimination with partial pivoting; 0 where a pivot is exactly zero */
static int gj_inverse(int n, const real* M, real* Inv) {
    real A[225];
    memcpy(A, M, sizeof *A * (size_t)(n * n));
    mat_eye(Inv, n);
    for (int c = 0; c < n; c++) {
        int p = c;
        for (int i = c + 1; i < n; i++) if (fabs(E(A, n, i, c)) > fabs(E(A, n, p, c))) p = i;
        if (E(A, n, p, c) == 0) return 0;
        if (p != c)
            for (int j = 0; j < n; j++) {
                real t = E(A, n, p, j); E(A, n, p, j) = E(A, n, c, j); E(A, n, c, j) = t;
                t = E(Inv, n, p, j); E(Inv, n, p, j) = E(Inv, n, c, j); E(Inv, n, c, j) = t;
            }
        const real d = E(A, n, c, c);
        for (int j = 0; j < n; j++) { E(A, n, c, j) /= d; E(Inv, n, c, j) /= d; }
        for (int i = 0; i < n; i++) {
            const real f = E(A, n, i, c);
            if (i == c || f == 0) continue;
            for (int j = 0; j < n; j++) { E(A, n, i, j) -= f * E(A, n, c, j); E(Inv, n, i, j) -= f * E(Inv, n, c, j); }
        }
    }
    return 1;
}

/* the 3x3 coefficient blocks of A's theta, v and p rows (propagate.cu's cf), (i, j) = E(blk, 3, i, j) */
typedef struct { real tt[9], tb[9], vt[9], vb[9], va[9], pt[9], pb[9], pa[9], dt; } arows_t;

/* x <- A x in place, propagate.cu a_apply's order: p rows first (they read v), then v, theta last */
static void a_apply_r(real* x, const arows_t* a) {
    for (int i = 0; i < 3; i++) {
        real tp = x[12 + i] + a->dt * x[6 + i];
        for (int j = 0; j < 3; j++) tp += E(a->pt, 3, i, j) * x[j] + E(a->pb, 3, i, j) * x[3 + j] + E(a->pa, 3, i, j) * x[9 + j];
        x[12 + i] = tp;
    }
    for (int i = 0; i < 3; i++) {
        real tv = x[6 + i];
        for (int j = 0; j < 3; j++) tv += E(a->vt, 3, i, j) * x[j] + E(a->vb, 3, i, j) * x[3 + j] + E(a->va, 3, i, j) * x[9 + j];
        x[6 + i] = tv;
    }
    real t0[3];
    for (int i = 0; i < 3; i++) {
        t0[i] = 0;
        for (int j = 0; j < 3; j++) t0[i] += E(a->tt, 3, i, j) * x[j] + E(a->tb, 3, i, j) * x[3 + j];
    }
    x[0] = t0[0]; x[1] = t0[1]; x[2] = t0[2];
}

/* one window: x (16) and S (225, column-major) in, x1, S1 and C (may be NULL) out, all in `real` */
static void propagate_one(int model, const real* x, const real* S, const double* r_in, const double* l_in, int order, real* x1,
                          real* S1, real* C) {
    real e[15], H1[225], H2[225], Pm[225], B[225], A[225], T[225], U[225];
    predict_state_r(model, x, r_in, l_in, x1);
    factor_eval_r(model, x, x1, r_in, l_in, e, H1, H2);
    load(Pm, r_in + CPI_REC_P, 225);
    if (order == 0) {
        if (!gj_inverse(15, H2, B)) for (int k = 0; k < 225; k++) B[k] = NAN;
        gemm(15, 15, 15, B, H1, A);
        for (int k = 0; k < 225; k++) A[k] = -A[k];
        gemm(15, 15, 15, A, S, T);
        gemm_nt(15, 15, 15, T, A, S1);
        gemm(15, 15, 15, B, Pm, T);
        gemm_nt(15, 15, 15, T, B, U);
        for (int k = 0; k < 225; k++) S1[k] += U[k];
        if (C) gemm_nt(15, 15, 15, S, A, C);
        return;
    }
    /* Q = w I + [v x] is H2's (theta, theta) block: Q^-1 = (w^2 I - w [v x] + v v^T) / (w |q_r|^2); Rk its (v, v) block */
    const real w = E(H2, 15, 0, 0), v[3] = {E(H2, 15, 2, 1), E(H2, 15, 0, 2), E(H2, 15, 1, 0)};
    const real d = 1 / (w * (w * w + v[0] * v[0] + v[1] * v[1] + v[2] * v[2]));
    real K[9], Qi[9], Rt[9], Rk[9], blk[9];
    skew_x(v, K);
    for (int c = 0; c < 3; c++) for (int u = 0; u < 3; u++) E(Qi, 3, u, c) = ((u == c ? w * w : 0) - w * E(K, 3, u, c) + v[u] * v[c]) * d;
    get_block(H2, 15, 6, 6, 3, 3, Rk);
    transpose(3, 3, Rk, Rt);
    arows_t a;
    a.dt = r_in[CPI_REC_DT];
    /* -H2_II^-1 H1_IJ: the theta row through Q^-1, the v and p rows through Rk^T */
    struct { real* dst; const real* L; int r0, c0; } rows[8] = {
        {a.tt, Qi, 0, 0}, {a.tb, Qi, 0, 1}, {a.vt, Rt, 2, 0}, {a.vb, Rt, 2, 1}, {a.va, Rt, 2, 3},
        {a.pt, Rt, 4, 0}, {a.pb, Rt, 4, 1}, {a.pa, Rt, 4, 3}};
    for (int k = 0; k < 8; k++) {
        get_block(H1, 15, 3 * rows[k].r0, 3 * rows[k].c0, 3, 3, blk);
        m3_mul(rows[k].L, blk, rows[k].dst);
        for (int q = 0; q < 9; q++) rows[k].dst[q] = -rows[k].dst[q];
    }
    real N[225], col[15];
    for (int j = 0; j < 15; j++) {                                           /* N(:, j) = A S(:, j) */
        for (int k = 0; k < 15; k++) col[k] = E(S, 15, k, j);
        a_apply_r(col, &a);
        for (int k = 0; k < 15; k++) E(N, 15, k, j) = col[k];
    }
    for (int i = 0; i < 15; i++) {                                           /* S1(i, j >= i) = (A N(i, :)^T)_j + (B P B^T)(i, j) */
        const int bI = i / 3, ii = i - 3 * bI;
        for (int k = 0; k < 15; k++) col[k] = E(N, 15, i, k);
        a_apply_r(col, &a);
        real bi[3];                                                          /* row ii of B_I: Q^-1, I or Rk^T */
        for (int c = 0; c < 3; c++) bi[c] = bI == 0 ? E(Qi, 3, ii, c) : (bI == 2 || bI == 4) ? E(Rt, 3, ii, c) : (c == ii ? 1 : 0);
        for (int bJ = 0; bJ < 5; bJ++) {
            real t[3], s[3];
            for (int m = 0; m < 3; m++) {
                const int k = 3 * bJ + m;
                t[m] = bi[0] * E(Pm, 15, 3 * bI, k) + bi[1] * E(Pm, 15, 3 * bI + 1, k) + bi[2] * E(Pm, 15, 3 * bI + 2, k);
            }
            for (int m = 0; m < 3; m++) {                                    /* ... B_J^T on the right */
                if (bJ == 0) s[m] = t[0] * E(Qi, 3, m, 0) + t[1] * E(Qi, 3, m, 1) + t[2] * E(Qi, 3, m, 2);
                else if (bJ == 2 || bJ == 4) s[m] = t[0] * E(Rt, 3, m, 0) + t[1] * E(Rt, 3, m, 1) + t[2] * E(Rt, 3, m, 2);
                else s[m] = t[m];
            }
            for (int m = 0; m < 3; m++) {
                const int j = 3 * bJ + m;
                if (j >= i) { const real y = col[j] + s[m]; E(S1, 15, i, j) = y; E(S1, 15, j, i) = y; }
            }
        }
    }
    if (C) transpose(15, 15, N, C);
}

/* the two entries below: windows (chains) [lo, hi) of one job per thread */
typedef struct {
    int model, order, t, nt; int64_t n, steps;
    const double *states, *cov, *path, *records, *lin; const int64_t* anchor;
    double *states_out, *cov_out, *cross;
} pjob_t;

static void* pworker(void* arg) {
    const pjob_t* j = (const pjob_t*)arg;
    const int rd = j->model == 1 ? CPI_REC_V1_DOUBLES : CPI_REC_V2_DOUBLES;
    const int64_t lo = j->n * j->t / j->nt, hi = j->n * (j->t + 1) / j->nt;
    for (int64_t i = lo; i < hi; i++) {
        real x[CPI_STATE_DOUBLES], S[225], x1[CPI_STATE_DOUBLES], S1[225], C[225];
        if (j->steps == 0) {                                                 /* oracle_propagate: window i */
            const int64_t a = j->anchor ? j->anchor[i] : i;
            load(x, j->states + a * CPI_STATE_DOUBLES, CPI_STATE_DOUBLES);
            load(S, j->cov + a * 225, 225);
            propagate_one(j->model, x, S, j->records + i * (int64_t)rd, j->lin + i * CPI_LIN_DOUBLES, j->order, x1, S1, j->cross ? C : 0);
            store(j->states_out + i * CPI_STATE_DOUBLES, x1, CPI_STATE_DOUBLES);
            store(j->cov_out + i * 225, S1, 225);
            if (j->cross) store(j->cross + i * 225, C, 225);
            continue;
        }
        load(x, j->states + i * CPI_STATE_DOUBLES, CPI_STATE_DOUBLES);       /* oracle_propagate_chain: chain i */
        load(S, j->cov + i * 225, 225);
        for (int64_t k = 0; k < j->steps; k++) {
            const int64_t w = i * j->steps + k;
            if (j->path) load(x, j->path + (i * (j->steps + 1) + k) * CPI_STATE_DOUBLES, CPI_STATE_DOUBLES);
            propagate_one(j->model, x, S, j->records + w * (int64_t)rd, j->lin + w * CPI_LIN_DOUBLES, j->order, x1, S1, 0);
            memcpy(x, x1, sizeof x); memcpy(S, S1, sizeof S);
        }
        store(j->states_out + i * CPI_STATE_DOUBLES, x, CPI_STATE_DOUBLES);
        store(j->cov_out + i * 225, S, 225);
    }
    return 0;
}

static void prun(pjob_t* proto, int nthreads) {
    if (nthreads < 1) nthreads = 1;
    if (nthreads > 256) nthreads = 256;
    pjob_t jobs[256]; pthread_t th[256];
    for (int t = 0; t < nthreads; t++) { jobs[t] = *proto; jobs[t].t = t; jobs[t].nt = nthreads; }
    if (nthreads == 1) { pworker(&jobs[0]); return; }
    for (int t = 0; t < nthreads; t++) pthread_create(&th[t], 0, pworker, &jobs[t]);
    for (int t = 0; t < nthreads; t++) pthread_join(th[t], 0);
}

int oracle_propagate(int model, int64_t n, const double* states_k, const double* cov_k, const int64_t* anchor, const double* records,
                     const double* lin, int order, double* states_k1, double* cov_k1, double* cross, int nthreads) {
    if ((model != 1 && model != 2) || (order != 0 && order != 1)) return -1;
    pjob_t j; memset(&j, 0, sizeof j);
    j.model = model; j.order = order; j.n = n; j.states = states_k; j.cov = cov_k; j.anchor = anchor; j.records = records; j.lin = lin;
    j.states_out = states_k1; j.cov_out = cov_k1; j.cross = cross;
    prun(&j, nthreads);
    return 0;
}

/* `steps` windows of K7 per chain (records and lin chain-major, [n_chains * steps]), the state and covariance held in `real`
 * between steps.  path (may be NULL) [n_chains * (steps + 1), 16]: step k starts from path's state k of the chain instead of the
 * statement's own prediction, so that the covariance recursion can follow a given (the device's) trajectory. */
int oracle_propagate_chain(int model, int64_t n_chains, int64_t steps, const double* states0, const double* cov0, const double* path,
                           const double* records, const double* lin, int order, double* states_out, double* cov_out, int nthreads) {
    if ((model != 1 && model != 2) || (order != 0 && order != 1) || steps < 1) return -1;
    pjob_t j; memset(&j, 0, sizeof j);
    j.model = model; j.order = order; j.n = n_chains; j.steps = steps; j.states = states0; j.cov = cov0; j.path = path;
    j.records = records; j.lin = lin; j.states_out = states_out; j.cov_out = cov_out;
    prun(&j, nthreads);
    return 0;
}

/* ------------------------------------------------------------------ merging model-1 records (DESIGN.md 3b, 3c) ---- */
/* Not a reference routine: a dense, literal statement of the composition of two consecutive model-1 records, with the full
 * 15x15 Phi~ and T and dense products (as tests/test_merge.py's numpy merge2 writes it), so that it checks the kernels' sparse
 * lane algebra (cpi_b200/csrc/record_merge.cuh) instead of repeating it.  A record is the [290] layout of include/cpi_b200.h
 * held in `real`; 3x3 blocks are column-major, as everywhere in this file. */
enum { RD1 = CPI_REC_V1_DOUBLES };

static void rec_zero(real* r) {
    mat_zero(r, RD1);
    r[CPI_REC_Q + 3] = 1.0;
    mat_eye(r + CPI_REC_R, 3);
}

/* Move a record from its linearisation point lin_k to lin_0, to first order: R <- Exp(J_q db_w) R, alpha += J_a db_w + H_a db_a,
 * beta += J_b db_w + H_b db_a, with db = lin_0 - lin_k from the double values; nothing moves when all six differences are 0.
 * q, the Jacobians and P are left as they are (the merge recomputes q from R). */
static void rec_relinearise(real* r, const double* lin0, const double* link) {
    real dbw[3], dba[3], t[3], Ex[9], Rn[9], u[3], w[3];
    int moved = 0;
    for (int i = 0; i < 3; i++) {
        dbw[i] = (real)lin0[i] - (real)link[i];
        dba[i] = (real)lin0[3 + i] - (real)link[3 + i];
        moved |= dbw[i] != 0 || dba[i] != 0;
    }
    if (!moved) return;
    m3_vec(r + CPI_REC_JQ, dbw, t);
    Exp(t, Ex);
    gemm(3, 3, 3, Ex, r + CPI_REC_R, Rn);
    memcpy(r + CPI_REC_R, Rn, sizeof Rn);
    m3_vec(r + CPI_REC_JA, dbw, u); m3_vec(r + CPI_REC_HA, dba, w);
    for (int i = 0; i < 3; i++) r[CPI_REC_ALPHA + i] += u[i] + w[i];
    m3_vec(r + CPI_REC_JB, dbw, u); m3_vec(r + CPI_REC_HB, dba, w);
    for (int i = 0; i < 3; i++) r[CPI_REC_BETA + i] += u[i] + w[i];
}

/* A^-1 of a 3x3 matrix: adjugate over determinant */
static void m3_inv(const real* A, real* Ai) {
    real c[9];
    for (int j = 0; j < 3; j++) for (int i = 0; i < 3; i++) {
        int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        E(c, 3, i, j) = E(A, 3, i1, j1) * E(A, 3, i2, j2) - E(A, 3, i1, j2) * E(A, 3, i2, j1);   /* cofactor (i, j) */
    }
    real det = E(A, 3, 0, 0) * E(c, 3, 0, 0) + E(A, 3, 0, 1) * E(c, 3, 0, 1) + E(A, 3, 0, 2) * E(c, 3, 0, 2);
    for (int j = 0; j < 3; j++) for (int i = 0; i < 3; i++) E(Ai, 3, i, j) = E(c, 3, j, i) / det;
}

/* out = A (+) B: A covers k -> m, B covers m -> j, both at one linearisation point.  out may not alias A or B. */
static void rec_merge(const real* A, const real* B, real* out) {
    const real *R1 = A + CPI_REC_R, *R2 = B + CPI_REC_R;
    const real dt2 = B[CPI_REC_DT];
    real R1T[9], sk[9], t9[9], u9[9], t3[3], eye[9];
    mat_eye(eye, 3);
    transpose(3, 3, R1, R1T);
    mat_zero(out, RD1);
    gemm(3, 3, 3, R2, R1, out + CPI_REC_R);                                          /* R = R2 R1 */
    out[CPI_REC_DT] = A[CPI_REC_DT] + dt2;
    m3_vec(R1T, B + CPI_REC_BETA, t3);                                               /* beta = b1 + R1^T b2 */
    for (int i = 0; i < 3; i++) out[CPI_REC_BETA + i] = A[CPI_REC_BETA + i] + t3[i];
    m3_vec(R1T, B + CPI_REC_ALPHA, t3);                                              /* alpha = a1 + b1 DT2 + R1^T a2 */
    for (int i = 0; i < 3; i++) out[CPI_REC_ALPHA + i] = A[CPI_REC_ALPHA + i] + A[CPI_REC_BETA + i] * dt2 + t3[i];
    gemm(3, 3, 3, R2, A + CPI_REC_JQ, t9);                                           /* J_q = R2 J_q1 + J_q2 */
    for (int e = 0; e < 9; e++) out[CPI_REC_JQ + e] = t9[e] + B[CPI_REC_JQ + e];
    gemm(3, 3, 3, R1T, B + CPI_REC_HB, t9);                                          /* H_b = H_b1 + R1^T H_b2 */
    for (int e = 0; e < 9; e++) out[CPI_REC_HB + e] = A[CPI_REC_HB + e] + t9[e];
    gemm(3, 3, 3, R1T, B + CPI_REC_HA, t9);                                          /* H_a = H_a1 + H_b1 DT2 + R1^T H_a2 */
    for (int e = 0; e < 9; e++) out[CPI_REC_HA + e] = A[CPI_REC_HA + e] + A[CPI_REC_HB + e] * dt2 + t9[e];
    skew_x(B + CPI_REC_BETA, sk); gemm(3, 3, 3, sk, A + CPI_REC_JQ, u9);             /* J_b = J_b1 + R1^T([b2] J_q1 + J_b2) */
    for (int e = 0; e < 9; e++) u9[e] += B[CPI_REC_JB + e];
    gemm(3, 3, 3, R1T, u9, t9);
    for (int e = 0; e < 9; e++) out[CPI_REC_JB + e] = A[CPI_REC_JB + e] + t9[e];
    skew_x(B + CPI_REC_ALPHA, sk); gemm(3, 3, 3, sk, A + CPI_REC_JQ, u9);            /* J_a = J_a1 + J_b1 DT2 + R1^T([a2] J_q1 + J_a2) */
    for (int e = 0; e < 9; e++) u9[e] += B[CPI_REC_JA + e];
    gemm(3, 3, 3, R1T, u9, t9);
    for (int e = 0; e < 9; e++) out[CPI_REC_JA + e] = A[CPI_REC_JA + e] + A[CPI_REC_JB + e] * dt2 + t9[e];

    /* Phi2 over [theta, b_g, v, b_a, p], T = blockdiag(I, I, R1^T, I, R1^T) (window 2's v and p error states are in frame m),
     * Phi~ = T Phi2 T^-1, P = Phi~ P1 Phi~^T + T P2 T^T.  T^-1 = T^T for an orthogonal R1; a stored R1 is orthogonal only to its
     * rounding (2^-24 in fp32 storage), and the similarity transform is the one that composes: Phi~ x = T Phi2 (T^-1 x). */
    real Phi2[225], T[225], Ti[225], X[225], Phi[225], Y[225], R1Ti[9];
    m3_inv(R1T, R1Ti);
    mat_eye(Phi2, 15);
    set_block(Phi2, 15, 0, 0, 3, 3, R2, 1.0);
    set_block(Phi2, 15, 0, 3, 3, 3, B + CPI_REC_JQ, -1.0);
    skew_x(B + CPI_REC_BETA, sk); set_block(Phi2, 15, 6, 0, 3, 3, sk, -1.0);
    set_block(Phi2, 15, 6, 3, 3, 3, B + CPI_REC_JB, 1.0);
    set_block(Phi2, 15, 6, 9, 3, 3, B + CPI_REC_HB, 1.0);
    skew_x(B + CPI_REC_ALPHA, sk); set_block(Phi2, 15, 12, 0, 3, 3, sk, -1.0);
    set_block(Phi2, 15, 12, 3, 3, 3, B + CPI_REC_JA, 1.0);
    set_block(Phi2, 15, 12, 6, 3, 3, eye, dt2);
    set_block(Phi2, 15, 12, 9, 3, 3, B + CPI_REC_HA, 1.0);
    mat_eye(T, 15);
    set_block(T, 15, 6, 6, 3, 3, R1T, 1.0);
    set_block(T, 15, 12, 12, 3, 3, R1T, 1.0);
    mat_eye(Ti, 15);
    set_block(Ti, 15, 6, 6, 3, 3, R1Ti, 1.0);
    set_block(Ti, 15, 12, 12, 3, 3, R1Ti, 1.0);
    gemm(15, 15, 15, T, Phi2, X); gemm(15, 15, 15, X, Ti, Phi);
    gemm(15, 15, 15, Phi, A + CPI_REC_P, X); gemm_nt(15, 15, 15, X, Phi, Y);
    gemm(15, 15, 15, T, B + CPI_REC_P, X); gemm_nt(15, 15, 15, X, T, Phi2);
    for (int e = 0; e < 225; e++) out[CPI_REC_P + e] = Y[e] + Phi2[e];
    rot_2_quat(out + CPI_REC_R, out + CPI_REC_Q);
}

/* The left fold of records lo .. hi-1 (global indices into rec / lin), every later record first moved to lin[lo]; merged: the
 * fold (an empty group gives the zero-step record, a group of one a copy), prefix: every prefix fold at its record's row. */
static void fold_group(const double* rec, const double* lin, int64_t lo, int64_t hi, double* merged, double* prefix) {
    if (hi <= lo) {
        if (merged) { real z[RD1]; rec_zero(z); store(merged, z, RD1); }
        return;
    }
    real* acc = (real*)malloc(3 * RD1 * sizeof(real));
    real *nx = acc + RD1, *tmp = acc + 2 * RD1;
    load(acc, rec + lo * RD1, RD1);
    if (prefix) store(prefix + lo * RD1, acc, RD1);
    for (int64_t k = lo + 1; k < hi; k++) {
        load(nx, rec + k * RD1, RD1);
        rec_relinearise(nx, lin + lo * CPI_LIN_DOUBLES, lin + k * CPI_LIN_DOUBLES);
        rec_merge(acc, nx, tmp);
        memcpy(acc, tmp, RD1 * sizeof(real));
        if (prefix) store(prefix + k * RD1, acc, RD1);
    }
    if (merged) store(merged, acc, RD1);
    free(acc);
}

typedef struct {
    int kind, t, nt; int64_t n;                  /* kind 0: pairs, 1: relinearise, 2: merge groups, 3: scan groups */
    const int64_t* offsets; int64_t uniform;
    const double *a, *b, *lin, *lin0;
    double* out;
} rjob_t;

static void* rworker(void* arg) {
    rjob_t* j = (rjob_t*)arg;
    int64_t lo = j->n * j->t / j->nt, hi = j->n * (j->t + 1) / j->nt;
    real* x = (real*)malloc(3 * RD1 * sizeof(real));
    for (int64_t i = lo; i < hi; i++) {
        if (j->kind == 0) {
            load(x, j->a + i * RD1, RD1); load(x + RD1, j->b + i * RD1, RD1);
            rec_merge(x, x + RD1, x + 2 * RD1);
            store(j->out + i * RD1, x + 2 * RD1, RD1);
        } else if (j->kind == 1) {
            load(x, j->a + i * RD1, RD1);
            rec_relinearise(x, j->lin0 + i * CPI_LIN_DOUBLES, j->lin + i * CPI_LIN_DOUBLES);
            store(j->out + i * RD1, x, RD1);
        } else {
            int64_t g0 = j->offsets ? j->offsets[i] : i * j->uniform, g1 = j->offsets ? j->offsets[i + 1] : g0 + j->uniform;
            if (j->kind == 2) fold_group(j->a, j->lin, g0, g1, j->out + i * RD1, 0);
            else fold_group(j->a, j->lin, g0, g1, 0, j->out);
        }
    }
    free(x);
    return 0;
}

static void rrun(rjob_t* proto, int nthreads) {
    if (nthreads < 1) nthreads = 1;
    if (nthreads > 256) nthreads = 256;
    rjob_t jobs[256]; pthread_t th[256];
    for (int t = 0; t < nthreads; t++) { jobs[t] = *proto; jobs[t].t = t; jobs[t].nt = nthreads; }
    if (nthreads == 1) { rworker(&jobs[0]); return; }
    for (int t = 0; t < nthreads; t++) pthread_create(&th[t], 0, rworker, &jobs[t]);
    for (int t = 0; t < nthreads; t++) pthread_join(th[t], 0);
}

int oracle_merge_pair(int64_t n, const double* a, const double* b, double* out, int nthreads) {
    rjob_t j; memset(&j, 0, sizeof j);
    j.kind = 0; j.n = n; j.a = a; j.b = b; j.out = out;
    rrun(&j, nthreads);
    return 0;
}

int oracle_relinearise_records(int64_t n, const double* records, const double* lin, const double* lin0, double* out) {
    rjob_t j; memset(&j, 0, sizeof j);
    j.kind = 1; j.n = n; j.a = records; j.lin = lin; j.lin0 = lin0; j.out = out;
    rrun(&j, 1);
    return 0;
}

static int group_job(int kind, int64_t n_groups, const int64_t* offsets, int64_t uniform, const double* records, const double* lin,
                     double* out, int nthreads) {
    if (n_groups < 0 || (!offsets && uniform < 0)) return -1;
    rjob_t j; memset(&j, 0, sizeof j);
    j.kind = kind; j.n = n_groups; j.offsets = offsets; j.uniform = uniform; j.a = records; j.lin = lin; j.out = out;
    rrun(&j, nthreads);
    return 0;
}

int oracle_merge_records(int64_t n_groups, const int64_t* offsets, int64_t uniform, const double* records, const double* lin,
                         double* out, int nthreads) {
    return group_job(2, n_groups, offsets, uniform, records, lin, out, nthreads);
}

int oracle_scan_records(int64_t n_groups, const int64_t* offsets, int64_t uniform, const double* records, const double* lin,
                        double* out, int nthreads) {
    return group_job(3, n_groups, offsets, uniform, records, lin, out, nthreads);
}

/* ------------------------------------------------------------------ the solver side of a chain (DESIGN.md 3e, 3f) -- */
/* Not reference routines: dense, literal statements of the chain marginalisation (K8), the prior move (k_prior_at), the SPD
 * block-tridiagonal solve and the LM model decrease, so that they check the kernels' lane algebra instead of repeating it.
 * 15x15 blocks are column-major [225] as in include/cpi_b200.h; symmetric inputs are read from their lower triangle, as the kernels
 * read them.  The chain layouts are those of the C ABI: CSR state offsets, or chains of `uniform` states when offsets is NULL;
 * chain c's factors are stored back to back from index offsets[c] - c. */
enum { B15 = 225 };

static void sym_lower(real* dst, const double* src) {
    for (int j = 0; j < 15; j++) for (int i = j; i < 15; i++) E(dst, 15, i, j) = E(dst, 15, j, i) = src[i + 15 * j];
}

/* A = L L^T in place (L lower, the upper triangle zeroed).  Returns 0 at the first pivot that is not positive. */
static int chol15(real* A) {
    for (int j = 0; j < 15; j++) {
        real d = E(A, 15, j, j);
        for (int k = 0; k < j; k++) d -= E(A, 15, j, k) * E(A, 15, j, k);
        if (!(d > 0)) return 0;
        d = sqrt(d);
        E(A, 15, j, j) = d;
        for (int i = j + 1; i < 15; i++) {
            real s = E(A, 15, i, j);
            for (int k = 0; k < j; k++) s -= E(A, 15, i, k) * E(A, 15, j, k);
            E(A, 15, i, j) = s / d;
        }
        for (int i = 0; i < j; i++) E(A, 15, i, j) = 0;
    }
    return 1;
}
/* B (15 x n) <- L^-1 B */
static void fwd_n(const real* L, real* B, int n) {
    for (int c = 0; c < n; c++) for (int i = 0; i < 15; i++) {
        real s = E(B, 15, i, c);
        for (int k = 0; k < i; k++) s -= E(L, 15, i, k) * E(B, 15, k, c);
        E(B, 15, i, c) = s / E(L, 15, i, i);
    }
}
/* v <- L^-T v */
static void bwd_1(const real* L, real* v) {
    for (int i = 14; i >= 0; i--) {
        real s = v[i];
        for (int k = i + 1; k < 15; k++) s -= E(L, 15, k, i) * v[k];
        v[i] = s / E(L, 15, i, i);
    }
}
/* v <- L^-T v column by column, as warp_bwd15 (chol15.cuh): x_i = v_i / L_ii, then v_j -= L_ij x_i for j < i */
static void bwd_col(const real* L, real* v) {
    for (int i = 14; i >= 0; i--) {
        v[i] = v[i] / E(L, 15, i, i);
        for (int j = 0; j < i; j++) v[j] -= E(L, 15, i, j) * v[i];
    }
}
static void fill_nan(double* p, int64_t n) { for (int64_t i = 0; i < n; i++) p[i] = NAN; }

/* K8 for one chain: states lo .. hi-1, factors from fo.  Lam, eta, f start at the prior (0 without one); for k < m:
 *   M = Lam + G11_k = L L^T,  [Z z] = L^-1 [G12_k  eta + g1_k],  Lam <- G22_k - Z^T Z,  eta <- g2_k - Z^T z,  f <- f + f_k - z^T z.
 * m out of [0, hi - lo) or a pivot that is not positive: NaN.  m = 0: the prior's bits.  sc (may be NULL) [242]: the size of the
 * terms that cancel into the result, |G22| + |Z|^T |Z| and |g2| + |Z|^T |z| of the last step, |f_prior| + sum |f_k| + sum z^T z, and the
 * last step's z^T z. */
static void marg_chain(int64_t c, int64_t lo, int64_t hi, int64_t m, const double* G11, const double* G12, const double* G22, const double* g1,
                       const double* g2, const double* fk, const double* pi, const double* pr, const double* pf, double* oi, double* orr,
                       double* of, double* sc) {
    if (!(m >= 0 && m < hi - lo)) {
        fill_nan(oi, B15); fill_nan(orr, 15); fill_nan(of, 1); if (sc) fill_nan(sc, 242);
        return;
    }
    if (m == 0) {
        for (int t = 0; t < B15; t++) oi[t] = pi ? pi[c * B15 + t] : 0.0;
        for (int t = 0; t < 15; t++) orr[t] = pr ? pr[c * 15 + t] : 0.0;
        *of = pf ? pf[c] : 0.0;
        if (sc) { for (int t = 0; t < B15; t++) sc[t] = fabs(oi[t]); for (int t = 0; t < 15; t++) sc[B15 + t] = fabs(orr[t]); sc[240] = fabs(*of); sc[241] = 0; }
        return;
    }
    real Lam[B15], eta[15], F, M[B15], Z[15 * 16], A[B15], fs;
    if (pi) sym_lower(Lam, pi + c * B15); else mat_zero(Lam, B15);
    for (int t = 0; t < 15; t++) eta[t] = pr ? pr[c * 15 + t] : 0.0;
    F = pf ? pf[c] : 0.0;
    fs = fabs(F);
    const int64_t f0 = lo - c;
    for (int64_t k = 0; k < m; k++) {
        const int64_t fi = f0 + k;
        sym_lower(A, G11 + fi * B15);
        for (int t = 0; t < B15; t++) M[t] = Lam[t] + A[t];
        if (!chol15(M)) {
            fill_nan(oi, B15); fill_nan(orr, 15); fill_nan(of, 1); if (sc) fill_nan(sc, 242);
            return;
        }
        load(Z, G12 + fi * B15, B15);
        for (int r = 0; r < 15; r++) Z[B15 + r] = eta[r] + g1[fi * 15 + r];
        fwd_n(M, Z, 16);
        sym_lower(A, G22 + fi * B15);
        real zz = 0;
        for (int q = 0; q < 15; q++) zz += Z[B15 + q] * Z[B15 + q];
        for (int j = 0; j < 15; j++) {
            for (int i = 0; i < 15; i++) {
                real s = 0;
                for (int q = 0; q < 15; q++) s += E(Z, 15, q, i) * E(Z, 15, q, j);
                E(Lam, 15, i, j) = E(A, 15, i, j) - s;
            }
            real s = 0;
            for (int q = 0; q < 15; q++) s += E(Z, 15, q, j) * Z[B15 + q];
            eta[j] = (real)g2[fi * 15 + j] - s;
        }
        F = F + (real)fk[fi] - zz;
        fs += fabs((real)fk[fi]) + zz;
        if (sc && k == m - 1) {
            for (int j = 0; j < 15; j++) {
                for (int i = 0; i < 15; i++) {
                    real s = fabs(E(A, 15, i, j));
                    for (int q = 0; q < 15; q++) s += fabs(E(Z, 15, q, i)) * fabs(E(Z, 15, q, j));
                    sc[i + 15 * j] = (double)s;
                }
                real s = fabs((real)g2[fi * 15 + j]);
                for (int q = 0; q < 15; q++) s += fabs(E(Z, 15, q, j)) * fabs(Z[B15 + q]);
                sc[B15 + j] = (double)s;
            }
            sc[241] = (double)zz;
        }
    }
    store(oi, Lam, B15); store(orr, eta, 15); *of = (double)F;
    if (sc) sc[240] = (double)fs;
}

/* The sequential block Cholesky of one chain's rows lo .. hi-1 of A = tridiag(E^T, D, E), x_lo -> x_{hi-1}, then back:
 *   M_k = D_k - U_{k-1}^T U_{k-1} = L_k L_k^T,  U_k = L_k^-1 E_k,  y_k = L_k^-1 (b_k - U_{k-1}^T y_{k-1});  x_k = L_k^-T (y_k - U_k x_{k+1}).
 * A pivot that is not positive: NaN for the chain. */
static void seq_chain(int64_t lo, int64_t hi, const double* D, const double* Eb, const double* b, double* x) {
    const int64_t n = hi - lo;
    real* L = (real*)malloc((size_t)n * 2 * B15 * sizeof(real));
    real* U = L + n * B15;
    real* y = (real*)malloc((size_t)n * 15 * sizeof(real));
    int ok = 1;
    for (int64_t k = 0; k < n && ok; k++) {
        real* Lk = L + k * B15;
        sym_lower(Lk, D + (lo + k) * B15);
        for (int r = 0; r < 15; r++) y[k * 15 + r] = b[(lo + k) * 15 + r];
        if (k > 0) {
            const real* Up = U + (k - 1) * B15;
            for (int j = 0; j < 15; j++) {
                for (int i = 0; i < 15; i++) {
                    real s = 0;
                    for (int q = 0; q < 15; q++) s += E(Up, 15, q, i) * E(Up, 15, q, j);
                    E(Lk, 15, i, j) -= s;
                }
                real s = 0;
                for (int q = 0; q < 15; q++) s += E(Up, 15, q, j) * y[(k - 1) * 15 + q];
                y[k * 15 + j] -= s;
            }
        }
        ok = chol15(Lk);
        if (!ok) break;
        fwd_n(Lk, y + k * 15, 1);
        if (k + 1 < n) { load(U + k * B15, Eb + (lo + k) * B15, B15); fwd_n(Lk, U + k * B15, 15); }
    }
    if (!ok) {
        fill_nan(x + lo * 15, n * 15);
    } else {
        for (int64_t k = n - 1; k >= 0; k--) {
            real v[15];
            for (int r = 0; r < 15; r++) v[r] = y[k * 15 + r];
            if (k + 1 < n) {
                const real* Uk = U + k * B15;
                for (int r = 0; r < 15; r++) { real s = 0; for (int q = 0; q < 15; q++) s += E(Uk, 15, r, q) * y[(k + 1) * 15 + q]; v[r] -= s; }
            }
            bwd_1(L + k * B15, v);
            for (int r = 0; r < 15; r++) y[k * 15 + r] = v[r];        /* y now holds x_k */
        }
        store(x + lo * 15, y, n * 15);
    }
    free(L); free(y);
}

/* One level of the block cyclic reduction (rows 0 .. m-1), in the order of solve.cu's forward phase:
 * odd node i: D_i = Lc Lc^T, Za = Lc^-1 E_{i-1}^T, Zb = Lc^-1 E_i (0 for the last node), zb = Lc^-1 b_i; even node j -> node j/2 of the
 * next level: D' = D_j - Zb_{j-1}^T Zb_{j-1} - Za_{j+1}^T Za_{j+1}, b' = b_j - Zb_{j-1}^T zb_{j-1} - Za_{j+1}^T zb_{j+1},
 * E' = -Za_{j+1}^T Zb_{j+1}.  Blocks held full (D symmetric); products are subtracted one at a time in the kernels' order.
 * cid (may be NULL: every coupling used as given) [m]: the chain of every node.  With it, as k_bcr_eliminate_iso / k_bcr_reduce_iso, a
 * coupling between two chains is not read and its Za, Zb or E' is exact 0, so that a NaN stays inside its chain.  The buffer at Lc
 * (free it) also holds xn [even, 15] for the next level's solution. */
typedef struct { real *Lc, *Za, *Zb, *zb, *Dn, *En, *bn, *xn; } bcr_t;
#define SAME(p, q) (!cid || cid[p] == cid[q])
static void bcr_forward(int64_t m, const int64_t* cid, const real* D, const real* Eb, const real* b, bcr_t* v) {
    const int64_t odd = m / 2, even = (m + 1) / 2;
    real* Lc = (real*)malloc((size_t)(odd * (3 * B15 + 15) + even * (2 * B15 + 30)) * sizeof(real));
    real *Za = Lc + odd * B15, *Zb = Za + odd * B15, *zb = Zb + odd * B15;
    real *Dn = zb + odd * 15, *En = Dn + even * B15, *bn = En + even * B15, *xn = bn + even * 15;
    for (int64_t t = 0; t < odd; t++) {
        const int64_t i = 2 * t + 1;
        const int hl = SAME(i - 1, i), hr = i + 1 < m && SAME(i + 1, i);
        real* L = Lc + t * B15;
        memcpy(L, D + i * B15, B15 * sizeof(real));
        int ok = chol15(L);
        if (hl) transpose(15, 15, Eb + (i - 1) * B15, Za + t * B15); else mat_zero(Za + t * B15, B15);
        if (hr) memcpy(Zb + t * B15, Eb + i * B15, B15 * sizeof(real)); else mat_zero(Zb + t * B15, B15);
        memcpy(zb + t * 15, b + i * 15, 15 * sizeof(real));
        if (!ok) for (int e = 0; e < B15; e++) L[e] = NAN;
        fwd_n(L, Za + t * B15, 15); fwd_n(L, Zb + t * B15, 15); fwd_n(L, zb + t * 15, 1);
        if (cid && !hl) mat_zero(Za + t * B15, B15);
        if (cid && !hr) mat_zero(Zb + t * B15, B15);
    }
    for (int64_t u = 0; u < even; u++) {
        const int64_t j = 2 * u;
        real *Dj = Dn + u * B15, *bj = bn + u * 15, *Ej = En + u * B15;
        memcpy(Dj, D + j * B15, B15 * sizeof(real));
        memcpy(bj, b + j * 15, 15 * sizeof(real));
        mat_zero(Ej, B15);
        const int hasL = j >= 1 && SAME(j - 1, j), hasR = j + 1 < m && SAME(j + 1, j), linkRR = j + 2 < m && SAME(j + 2, j);
        const real *ZbL = hasL ? Zb + ((j - 2) / 2) * B15 : 0, *zbL = hasL ? zb + ((j - 2) / 2) * 15 : 0;
        const real *ZaR = hasR ? Za + (j / 2) * B15 : 0, *ZbR = linkRR ? Zb + (j / 2) * B15 : 0, *zbR = hasR ? zb + (j / 2) * 15 : 0;
        for (int c2 = 0; c2 < 15; c2++) {                       /* the products subtracted one by one, interleaved, as k_bcr_reduce_iso */
            for (int r = 0; r < 15; r++) {
                real d = E(Dj, 15, r, c2), e = 0;
                for (int q = 0; q < 15; q++) {
                    if (ZbL) d -= E(ZbL, 15, q, r) * E(ZbL, 15, q, c2);
                    if (ZaR) d -= E(ZaR, 15, q, r) * E(ZaR, 15, q, c2);
                    if (ZaR && ZbR) e -= E(ZaR, 15, q, r) * E(ZbR, 15, q, c2);
                }
                E(Dj, 15, r, c2) = d;
                E(Ej, 15, r, c2) = e;
            }
            real v = bj[c2];
            for (int q = 0; q < 15; q++) {
                if (ZbL) v -= E(ZbL, 15, q, c2) * zbL[q];
                if (ZaR) v -= E(ZaR, 15, q, c2) * zbR[q];
            }
            bj[c2] = v;
        }
    }
    v->Lc = Lc; v->Za = Za; v->Zb = Zb; v->zb = zb; v->Dn = Dn; v->En = En; v->bn = bn; v->xn = xn;
}
#undef SAME

/* The block cyclic reduction of the whole system (rows 0 .. m-1, couplings as given), level by level in the order of solve.cu: the
 * forward phase of bcr_forward, one node: x = D^-1 b, back: Lc^T x_i = zb - Za x_{i-1} - Zb x_{i+1}, L^-T column by column as
 * warp_bwd15 does. */
static void bcr_level(int64_t m, const real* D, const real* Eb, const real* b, real* x) {
    if (m == 1) {
        real L[B15], v[15];
        memcpy(L, D, sizeof L);
        if (!chol15(L)) { for (int r = 0; r < 15; r++) x[r] = NAN; return; }
        memcpy(v, b, sizeof v);
        fwd_n(L, v, 1); bwd_col(L, v);
        memcpy(x, v, sizeof v);
        return;
    }
    const int64_t odd = m / 2, even = (m + 1) / 2;
    bcr_t lv;
    bcr_forward(m, 0, D, Eb, b, &lv);
    bcr_level(even, lv.Dn, lv.En, lv.bn, lv.xn);
    for (int64_t u = 0; u < even; u++) memcpy(x + 2 * u * 15, lv.xn + u * 15, 15 * sizeof(real));
    for (int64_t t = 0; t < odd; t++) {
        const int64_t i = 2 * t + 1;
        real v[15];
        for (int r = 0; r < 15; r++) {
            real s = lv.zb[t * 15 + r];
            for (int q = 0; q < 15; q++) {
                s -= E(lv.Za + t * B15, 15, r, q) * x[(i - 1) * 15 + q];
                if (i + 1 < m) s -= E(lv.Zb + t * B15, 15, r, q) * x[(i + 1) * 15 + q];
            }
            v[r] = s;
        }
        bwd_col(lv.Lc + t * B15, v);
        memcpy(x + i * 15, v, sizeof v);
    }
    free(lv.Lc);
}

/* S = L^-T L^-1 (the inverse of L L^T), column c solved as k_bcr_selinv_root's lane c, its lower triangle mirrored */
static void chol_inverse(const real* L, real* S) {
    for (int c = 0; c < 15; c++) {
        real y[15];
        for (int r = 0; r < 15; r++) y[r] = r == c;
        fwd_n(L, y, 1); bwd_1(L, y);
        for (int r = c; r < 15; r++) E(S, 15, r, c) = E(S, 15, c, r) = y[r];
    }
}

/* The selected inversion of one level in the order of cpi_imu_chains_marginals (DESIGN.md 3j): the isolated forward phase of
 * bcr_forward on a zero right-hand side, the next level's blocks, then per odd node i (neighbours: nodes t, t+1 of the next level)
 *   Sigma_{i,i-1} = -Lc^-T (Za Sigma_{i-1,i-1} + Zb Sigma_{i+1,i-1}),   Sigma_{i,i+1} = -Lc^-T (Za Sigma_{i-1,i+1} + Zb Sigma_{i+1,i+1}),
 *   Sigma_{i,i}   =  Lc^-T (Lc^-1 - Za Sigma_{i,i-1}^T - Zb Sigma_{i,i+1}^T)   (lower triangle mirrored),
 * a term with a neighbour of another chain left out, as k_bcr_selinv_iso.  cid [m]: the chain of every node.  Out: cov [m] and the
 * neighbour blocks nb [m-1] (Sigma_{k,k+1}; exact 0 between chains).  One node: cov = D^-1, NaN if its pivot is not positive. */
static void bcr_selinv(int64_t m, const int64_t* cid, const real* D, const real* Eb, real* cov, real* nb) {
    if (m == 1) {
        real L[B15];
        memcpy(L, D, sizeof L);
        if (chol15(L)) chol_inverse(L, cov); else for (int e = 0; e < B15; e++) cov[e] = NAN;
        return;
    }
    const int64_t odd = m / 2, even = (m + 1) / 2;
    real* z = (real*)calloc((size_t)m * 15, sizeof(real));
    bcr_t lv;
    bcr_forward(m, cid, D, Eb, z, &lv);
    free(z);
    int64_t* cn = (int64_t*)malloc((size_t)even * sizeof(int64_t));
    real* covn = (real*)malloc((size_t)(2 * even) * B15 * sizeof(real));
    real* nbn = covn + even * B15;
    for (int64_t u = 0; u < even; u++) cn[u] = cid[2 * u];
    bcr_selinv(even, cn, lv.Dn, lv.En, covn, nbn);
    for (int64_t u = 0; u < even; u++) memcpy(cov + 2 * u * B15, covn + u * B15, B15 * sizeof(real));
    for (int64_t t = 0; t < odd; t++) {
        const int64_t i = 2 * t + 1;
        const int hl = cid[i - 1] == cid[i], hr = i + 1 < m && cid[i + 1] == cid[i];
        const real *L = lv.Lc + t * B15, *A = lv.Za + t * B15, *B = lv.Zb + t * B15;
        const real *XLi = covn + t * B15, *XRi = hr ? covn + (t + 1) * B15 : 0, *N = hl && hr ? nbn + t * B15 : 0;
        real XL[B15], XR[B15], y[15];
        mat_zero(XL, B15); mat_zero(XR, B15);
        for (int c = 0; c < 15; c++) {
            if (hl) {                                               /* column c of Sigma_{i,i-1}; Sigma_{i+1,i-1} = N^T */
                for (int r = 0; r < 15; r++) {
                    real s = 0;
                    for (int q = 0; q < 15; q++) s += E(A, 15, r, q) * E(XLi, 15, q, c);
                    if (hr) for (int q = 0; q < 15; q++) s += E(B, 15, r, q) * E(N, 15, c, q);
                    y[r] = s;
                }
                bwd_1(L, y);
                for (int r = 0; r < 15; r++) E(XL, 15, r, c) = -y[r];
            }
            if (hr) {                                               /* column c of Sigma_{i,i+1} */
                for (int r = 0; r < 15; r++) {
                    real s = 0;
                    if (hl) for (int q = 0; q < 15; q++) s += E(A, 15, r, q) * E(N, 15, q, c);
                    for (int q = 0; q < 15; q++) s += E(B, 15, r, q) * E(XRi, 15, q, c);
                    y[r] = s;
                }
                bwd_1(L, y);
                for (int r = 0; r < 15; r++) E(XR, 15, r, c) = -y[r];
            }
        }
        real* S = cov + i * B15;
        for (int c = 0; c < 15; c++) {
            for (int r = 0; r < 15; r++) y[r] = r == c;
            fwd_n(L, y, 1);
            for (int r = 0; r < 15; r++) {
                real s = y[r];
                if (hl) for (int q = 0; q < 15; q++) s -= E(A, 15, r, q) * E(XL, 15, c, q);
                if (hr) for (int q = 0; q < 15; q++) s -= E(B, 15, r, q) * E(XR, 15, c, q);
                y[r] = s;
            }
            bwd_1(L, y);
            for (int r = c; r < 15; r++) E(S, 15, r, c) = E(S, 15, c, r) = y[r];
        }
        transpose(15, 15, XL, nb + (i - 1) * B15);                 /* Sigma_{i-1,i} = Sigma_{i,i-1}^T */
        if (i + 1 < m) memcpy(nb + i * B15, XR, sizeof XR);
    }
    free(cn); free(covn); free(lv.Lc);
}

/* The selected inversion of one chain (rows lo .. hi-1), sequentially: the block Cholesky of seq_chain, M_k = D_k - U_{k-1}^T U_{k-1}
 * = L_k L_k^T, U_k = L_k^-1 E_k, then backwards Sigma_{n-1} = M_{n-1}^-1, Sigma_{k,k+1} = -L_k^-T U_k Sigma_{k+1,k+1},
 * Sigma_kk = L_k^-T (L_k^-1 - U_k Sigma_{k,k+1}^T) (lower triangle mirrored).  cov [n], cross [n-1] (may be NULL); a pivot that is not
 * positive: NaN for the chain. */
static void seq_marginals(int64_t lo, int64_t hi, const double* D, const double* Eb, double* cov, double* cross) {
    const int64_t n = hi - lo;
    real* L = (real*)malloc((size_t)n * 2 * B15 * sizeof(real));
    real* U = L + n * B15;
    int ok = 1;
    for (int64_t k = 0; k < n && ok; k++) {
        real* Lk = L + k * B15;
        sym_lower(Lk, D + (lo + k) * B15);
        if (k > 0) {
            const real* Up = U + (k - 1) * B15;
            for (int j = 0; j < 15; j++)
                for (int i = 0; i < 15; i++) {
                    real s = 0;
                    for (int q = 0; q < 15; q++) s += E(Up, 15, q, i) * E(Up, 15, q, j);
                    E(Lk, 15, i, j) -= s;
                }
        }
        ok = chol15(Lk);
        if (ok && k + 1 < n) { load(U + k * B15, Eb + (lo + k) * B15, B15); fwd_n(Lk, U + k * B15, 15); }
    }
    if (!ok) {
        fill_nan(cov + lo * B15, n * B15);
        if (cross) fill_nan(cross, (n - 1) * B15);
        free(L);
        return;
    }
    real S[B15], Sn[B15], X[B15], y[15];
    chol_inverse(L + (n - 1) * B15, Sn);
    store(cov + (hi - 1) * B15, Sn, B15);
    for (int64_t k = n - 2; k >= 0; k--) {
        const real *Lk = L + k * B15, *Uk = U + k * B15;
        for (int c = 0; c < 15; c++) {                              /* X = Sigma_{k,k+1} = -L_k^-T U_k Sigma_{k+1,k+1} */
            for (int r = 0; r < 15; r++) {
                real s = 0;
                for (int q = 0; q < 15; q++) s += E(Uk, 15, r, q) * E(Sn, 15, q, c);
                y[r] = s;
            }
            bwd_1(Lk, y);
            for (int r = 0; r < 15; r++) E(X, 15, r, c) = -y[r];
        }
        for (int c = 0; c < 15; c++) {
            for (int r = 0; r < 15; r++) y[r] = r == c;
            fwd_n(Lk, y, 1);
            for (int r = 0; r < 15; r++) {
                real s = y[r];
                for (int q = 0; q < 15; q++) s -= E(Uk, 15, r, q) * E(X, 15, c, q);
                y[r] = s;
            }
            bwd_1(Lk, y);
            for (int r = c; r < 15; r++) E(S, 15, r, c) = E(S, 15, c, r) = y[r];
        }
        store(cov + (lo + k) * B15, S, B15);
        if (cross) store(cross + k * B15, X, B15);
        memcpy(Sn, S, sizeof S);
    }
    free(L);
}

/* the LM model decrease of one chain (k_lm_terms + k_lm_decide's sums): out[5] = (m, the size of its terms, cur, new, moved)
 *   m = sum_k delta_k^T (2 rhs_k - (H delta)_k),  H = tridiag(E^T, D - diag(damp), E) of the chain,  size = sum_k |delta_k|^T (2 |rhs_k| + |H| |delta|),
 *   cur / new = the chain's factor costs + the prior's, moved = 1 if any delta != 0. */
static void lm_chain(int64_t c, int64_t lo, int64_t hi, const double* rhs, const double* D, const double* Eb, const double* damp, const double* delta,
                     const double* f_cur, const double* pf_cur, const double* f_new, const double* pf_new, double* out) {
    real m = 0, sz = 0, cur = pf_cur ? pf_cur[c] : 0.0, nw = pf_new ? pf_new[c] : 0.0;
    int moved = 0;
    for (int64_t k = lo; k < hi; k++) {
        for (int r = 0; r < 15; r++) {
            real hd = 0, ha = 0;
            for (int q = 0; q < 15; q++) {
                real h = D[k * B15 + r + 15 * q] - (q == r ? (real)damp[k * 15 + r] : 0);
                hd += h * delta[k * 15 + q]; ha += fabs(h) * fabs((real)delta[k * 15 + q]);
                if (k > lo) { real e = Eb[(k - 1) * B15 + q + 15 * r]; hd += e * delta[(k - 1) * 15 + q]; ha += fabs(e) * fabs((real)delta[(k - 1) * 15 + q]); }
                if (k + 1 < hi) { real e = Eb[k * B15 + r + 15 * q]; hd += e * delta[(k + 1) * 15 + q]; ha += fabs(e) * fabs((real)delta[(k + 1) * 15 + q]); }
            }
            const real d = delta[k * 15 + r];
            m += d * (2 * (real)rhs[k * 15 + r] - hd);
            sz += fabs(d) * (2 * fabs((real)rhs[k * 15 + r]) + ha);
            moved |= delta[k * 15 + r] != 0.0;
        }
        if (k + 1 < hi) { cur += f_cur[k - c]; nw += f_new[k - c]; }
    }
    out[0] = (double)m; out[1] = (double)sz; out[2] = (double)cur; out[3] = (double)nw; out[4] = moved;
}

typedef struct {
    int kind, t, nt; int64_t n;                  /* kind 0: marginalise, 1: sequential solve, 2: LM terms, 3: marginals */
    const int64_t *offsets, *n_marg; int64_t uniform, marg_uniform;
    const double *G11, *G12, *G22, *g1, *g2, *f, *pi, *pr, *pf;
    const double *D, *E, *b, *damp, *delta, *f_cur, *pf_cur, *f_new, *pf_new;
    double *oi, *orr, *of, *sc, *x, *cov, *cross;
} cjob_t;

static void* cworker(void* arg) {
    cjob_t* j = (cjob_t*)arg;
    for (int64_t c = j->t; c < j->n; c += j->nt) {             /* interleaved: chain lengths vary by orders of magnitude */
        const int64_t lo = j->offsets ? j->offsets[c] : c * j->uniform, hi = j->offsets ? j->offsets[c + 1] : lo + j->uniform;
        if (j->kind == 0)
            marg_chain(c, lo, hi, j->n_marg ? j->n_marg[c] : j->marg_uniform, j->G11, j->G12, j->G22, j->g1, j->g2, j->f, j->pi, j->pr, j->pf,
                       j->oi + c * B15, j->orr + c * 15, j->of + c, j->sc ? j->sc + c * 242 : 0);
        else if (j->kind == 1)
            seq_chain(lo, hi, j->D, j->E, j->b, j->x);
        else if (j->kind == 3)
            seq_marginals(lo, hi, j->D, j->E, j->cov, j->cross ? j->cross + (lo - c) * B15 : 0);
        else
            lm_chain(c, lo, hi, j->b, j->D, j->E, j->damp, j->delta, j->f_cur, j->pf_cur, j->f_new, j->pf_new, j->x + c * 5);
    }
    return 0;
}

static void crun(cjob_t* proto, int nthreads) {
    if (nthreads < 1) nthreads = 1;
    if (nthreads > 256) nthreads = 256;
    cjob_t jobs[256]; pthread_t th[256];
    for (int t = 0; t < nthreads; t++) { jobs[t] = *proto; jobs[t].t = t; jobs[t].nt = nthreads; }
    if (nthreads == 1) { cworker(&jobs[0]); return; }
    for (int t = 0; t < nthreads; t++) pthread_create(&th[t], 0, cworker, &jobs[t]);
    for (int t = 0; t < nthreads; t++) pthread_join(th[t], 0);
}

int oracle_chain_marginalize(int64_t n_chains, const int64_t* offsets, int64_t uniform, const int64_t* n_marg, int64_t marg_uniform,
                             const double* G11, const double* G12, const double* G22, const double* g1, const double* g2, const double* f,
                             const double* prior_info, const double* prior_rhs, const double* prior_f, double* out_info, double* out_rhs,
                             double* out_f, double* scale, int nthreads) {
    if (n_chains < 0 || (!offsets && uniform < 1)) return -1;
    cjob_t j; memset(&j, 0, sizeof j);
    j.kind = 0; j.n = n_chains; j.offsets = offsets; j.uniform = uniform; j.n_marg = n_marg; j.marg_uniform = marg_uniform;
    j.G11 = G11; j.G12 = G12; j.G22 = G22; j.g1 = g1; j.g2 = g2; j.f = f; j.pi = prior_info; j.pr = prior_rhs; j.pf = prior_f;
    j.oi = out_info; j.orr = out_rhs; j.of = out_f; j.sc = scale;
    crun(&j, nthreads);
    return 0;
}

int oracle_chain_solve(int64_t n_chains, const int64_t* offsets, int64_t uniform, const double* D, const double* E, const double* b, double* x,
                       int order, int nthreads) {
    if (n_chains < 0 || (!offsets && uniform < 1) || (order != 0 && order != 1)) return -1;
    const int64_t n = offsets ? offsets[n_chains] : n_chains * uniform;
    if (n == 0) return 0;
    if (order == 0) {
        cjob_t j; memset(&j, 0, sizeof j);
        j.kind = 1; j.n = n_chains; j.offsets = offsets; j.uniform = uniform; j.D = D; j.E = E; j.b = b; j.x = x;
        crun(&j, nthreads);
        return 0;
    }
    real* Dl = (real*)malloc((size_t)n * (2 * B15 + 30) * sizeof(real));
    real *El = Dl + n * B15, *bl = El + n * B15, *xl = bl + n * 15;
    for (int64_t k = 0; k < n; k++) {
        sym_lower(Dl + k * B15, D + k * B15);
        if (k + 1 < n) load(El + k * B15, E + k * B15, B15); else mat_zero(El + k * B15, B15);
        load(bl + k * 15, b + k * 15, 15);
    }
    bcr_level(n, Dl, El, bl, xl);
    store(x, xl, n * 15);
    free(Dl);
    return 0;
}

int oracle_chain_marginals(int64_t n_chains, const int64_t* offsets, int64_t uniform, const double* D, const double* E, double* cov,
                           double* cross, int order, int nthreads) {
    if (n_chains < 0 || (!offsets && uniform < 1) || (order != 0 && order != 1)) return -1;
    const int64_t n = offsets ? offsets[n_chains] : n_chains * uniform;
    if (n == 0) return 0;
    if (order == 0) {
        cjob_t j; memset(&j, 0, sizeof j);
        j.kind = 3; j.n = n_chains; j.offsets = offsets; j.uniform = uniform; j.D = D; j.E = E; j.cov = cov; j.cross = cross;
        crun(&j, nthreads);
        return 0;
    }
    real* Dl = (real*)malloc((size_t)n * 4 * B15 * sizeof(real));
    real *El = Dl + n * B15, *cl = El + n * B15, *nl = cl + n * B15;
    int64_t* cid = (int64_t*)malloc((size_t)n * sizeof(int64_t));
    for (int64_t c = 0; c < n_chains; c++) {
        const int64_t lo = offsets ? offsets[c] : c * uniform, hi = offsets ? offsets[c + 1] : lo + uniform;
        for (int64_t k = lo; k < hi; k++) cid[k] = c;
    }
    for (int64_t k = 0; k < n; k++) {
        sym_lower(Dl + k * B15, D + k * B15);
        if (k + 1 < n) load(El + k * B15, E + k * B15, B15); else mat_zero(El + k * B15, B15);
    }
    bcr_selinv(n, cid, Dl, El, cl, nl);
    store(cov, cl, n * B15);
    if (cross)
        for (int64_t k = 0; k + 1 < n; k++)
            if (cid[k] == cid[k + 1]) store(cross + (k - cid[k]) * B15, nl + k * B15, B15);
    free(Dl); free(cid);
    return 0;
}

int oracle_lm_terms(int64_t n_chains, const int64_t* offsets, int64_t uniform, const double* rhs, const double* D, const double* E,
                    const double* damp, const double* delta, const double* f_cur, const double* pf_cur, const double* f_new,
                    const double* pf_new, double* out, int nthreads) {
    if (n_chains < 0 || (!offsets && uniform < 1)) return -1;
    cjob_t j; memset(&j, 0, sizeof j);
    j.kind = 2; j.n = n_chains; j.offsets = offsets; j.uniform = uniform; j.b = rhs; j.D = D; j.E = E; j.damp = damp; j.delta = delta;
    j.f_cur = f_cur; j.pf_cur = pf_cur; j.f_new = f_new; j.pf_new = pf_new; j.x = out;
    crun(&j, nthreads);
    return 0;
}

/* local(x_lin, x): the delta with x = retract(x_lin, delta): the rotation vector of dq = q_x (x) q_lin^-1 (quat_multiply: w >= 0,
 * normalised), 2 atan2(|v|, w) v / |v|, exactly 0 when the two quaternions have the same bits and 2 v where |v| = 0; the other 12
 * entries are differences.  The `same` test is on the double inputs, so both builds take the same branch. */
static void local_state(const double* xl_in, const double* x_in, real* d) {
    real xl[CPI_STATE_DOUBLES], x[CPI_STATE_DOUBLES], qi[4], dq[4];
    load(xl, xl_in, CPI_STATE_DOUBLES); load(x, x_in, CPI_STATE_DOUBLES);
    quat_inv(xl, qi);
    quat_multiply(x, qi, dq);
    const real s = norm3(dq);
    const int same = x_in[0] == xl_in[0] && x_in[1] == xl_in[1] && x_in[2] == xl_in[2] && x_in[3] == xl_in[3];
    const real k = same ? 0 : (s > 0 ? 2 * atan2(s, dq[3]) / s : 2);
    for (int j = 0; j < 3; j++) d[j] = k * dq[j];
    for (int j = 0; j < 12; j++) d[3 + j] = x[4 + j] - xl[4 + j];
}

int oracle_local(int64_t n, const double* lin, const double* x, double* delta) {
    for (int64_t i = 0; i < n; i++) {
        real d[15];
        local_state(lin + i * CPI_STATE_DOUBLES, x + i * CPI_STATE_DOUBLES, d);
        store(delta + i * 15, d, 15);
    }
    return 0;
}

/* k_prior_at: delta = local(lin, x), rhs' = rhs - info delta, f' = f - 2 rhs^T delta + delta^T info delta (info read in full) */
int oracle_prior_at(int64_t n, const double* info, const double* rhs, const double* f, const double* lin, const double* x, double* rhs_out,
                    double* f_out) {
    for (int64_t i = 0; i < n; i++) {
        real d[15], u[15], fo = f ? f[i] : 0.0;
        local_state(lin + i * CPI_STATE_DOUBLES, x + i * CPI_STATE_DOUBLES, d);
        for (int r = 0; r < 15; r++) { real s = 0; for (int q = 0; q < 15; q++) s += info[i * B15 + r + 15 * q] * d[q]; u[r] = s; }
        for (int r = 0; r < 15; r++) {
            fo += d[r] * (u[r] - 2 * (real)rhs[i * 15 + r]);
            rhs_out[i * 15 + r] = (double)((real)rhs[i * 15 + r] - u[r]);
        }
        if (f_out) f_out[i] = (double)fo;
    }
    return 0;
}

/* ------------------------------------------------------------------ batch drivers -------------------------------- */
typedef struct {
    int kind, model, flags, t, nt; int64_t n;
    const int64_t *offsets, *idx_i, *idx_j; int64_t ns;
    const double *samples, *lin, *sig, *states, *records;
    double *out, *e, *H1, *H2;
} job_t;

static void* worker(void* arg) {
    job_t* j = (job_t*)arg;
    int64_t lo = j->n * j->t / j->nt, hi = j->n * (j->t + 1) / j->nt;
    int rd = j->model == 1 ? CPI_REC_V1_DOUBLES : CPI_REC_V2_DOUBLES;
    int avg = (j->flags & CPI_FLAG_IMU_AVG) != 0;
    for (int64_t w = lo; w < hi; w++) {
        if (j->kind == 0) {
            int64_t o0 = j->offsets ? j->offsets[w] : w * (j->ns + avg);
            int64_t o1 = j->offsets ? j->offsets[w + 1] : o0 + j->ns + avg;
            window(j->model, j->samples + o0 * CPI_SAMPLE_DOUBLES, o1 - o0, j->lin + w * CPI_LIN_DOUBLES, j->sig, j->flags, j->out + w * (int64_t)rd);
        } else {
            int64_t a = j->idx_i ? j->idx_i[w] : w, b = j->idx_j ? j->idx_j[w] : w + 1;
            factor_eval(j->model, j->states + a * CPI_STATE_DOUBLES, j->states + b * CPI_STATE_DOUBLES,
                        j->records + w * (int64_t)rd, j->lin + w * CPI_LIN_DOUBLES, j->e + w * 15,
                        j->H1 ? j->H1 + w * 225 : 0, j->H2 ? j->H2 + w * 225 : 0);
        }
    }
    return 0;
}

static void run(job_t* proto, int nthreads) {
    if (nthreads < 1) nthreads = 1;
    if (nthreads > 256) nthreads = 256;
    job_t jobs[256]; pthread_t th[256];
    for (int t = 0; t < nthreads; t++) { jobs[t] = *proto; jobs[t].t = t; jobs[t].nt = nthreads; }
    if (nthreads == 1) { worker(&jobs[0]); return; }
    for (int t = 0; t < nthreads; t++) pthread_create(&th[t], 0, worker, &jobs[t]);
    for (int t = 0; t < nthreads; t++) pthread_join(th[t], 0);
}

int oracle_cpi_preintegrate(int model, int64_t n_windows, const int64_t* offsets, int64_t ns_uniform,
                            const double* samples, const double* lin, const double* sigmas, int flags,
                            double* out, int nthreads) {
    if (model != 1 && model != 2) return -1;
    job_t j; memset(&j, 0, sizeof j);
    j.kind = 0; j.model = model; j.flags = flags; j.n = n_windows; j.offsets = offsets; j.ns = ns_uniform;
    j.samples = samples; j.lin = lin; j.sig = sigmas; j.out = out;
    run(&j, nthreads);
    return 0;
}

int oracle_imu_factor_eval(int model, int64_t n, const double* states, const int64_t* idx_i, const int64_t* idx_j,
                           const double* records, const double* lin, double* e, double* H1, double* H2, int nthreads) {
    if (model != 1 && model != 2) return -1;
    job_t j; memset(&j, 0, sizeof j);
    j.kind = 1; j.model = model; j.n = n; j.states = states; j.idx_i = idx_i; j.idx_j = idx_j;
    j.records = records; j.lin = lin; j.e = e; j.H1 = H1; j.H2 = H2;
    run(&j, nthreads);
    return 0;
}

int oracle_predict_state(int model, int64_t n, const double* states_k, const double* records, const double* lin, double* states_k1) {
    if (model != 1 && model != 2) return -1;
    int rd = model == 1 ? CPI_REC_V1_DOUBLES : CPI_REC_V2_DOUBLES;
    for (int64_t i = 0; i < n; i++)
        predict_state(model, states_k + i * CPI_STATE_DOUBLES, records + i * (int64_t)rd, lin + i * CPI_LIN_DOUBLES, states_k1 + i * CPI_STATE_DOUBLES);
    return 0;
}

int oracle_retract(int64_t n, const double* states, const double* xi, double* out) {
    for (int64_t i = 0; i < n; i++) retract(states + i * CPI_STATE_DOUBLES, xi + i * 15, out + i * CPI_STATE_DOUBLES);
    return 0;
}
