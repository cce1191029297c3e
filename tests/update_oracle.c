/* TEST INFRASTRUCTURE ONLY.  CPU restatement (plain C, dense, literal) of cpi_state_update_batch (DESIGN.md section 3k), built by
 * tests/update_ref.py in fp64 and, with -DCPI_ORACLE_LONG_DOUBLE, in long double (the flags of oracle/Makefile).  Host pointers;
 * layouts as include/cpi_b200.h.  No gating: the caller compares gamma with its gate.
 *
 *   oracle_state_update(n, states, cov, W, x_bar, order, states_out, cov_out, xi, nis)
 *     d = local(x_bar, x),  xi = -(S^-1 + W)^-1 W d,  S+ = (S^-1 + W)^-1,  x+ = retract(x, xi),
 *     gamma = (d+xi)^T W (d+xi) + xi^T S^-1 xi
 *   order 0: the square-root form of the kernel: S = L L^T, C = chol(I + L^T W L), u = L^T W d, v = C^-1 u, w = C^-T v, xi = -L w,
 *            S+ = M M^T with M = L C^-T, gamma = (d+xi)^T W (d+xi) + w^T w
 *   order 1: the information form: S^-1 = L^-T L^-1, P = S^-1 + W = R R^T, S+ = P^-1, xi = -P^-1 W d, gamma with xi^T S^-1 xi
 *   A Cholesky pivot that is not positive gives NaN outputs for that filter. */
#include <tgmath.h>
#include <stdint.h>
#include <string.h>

#ifdef CPI_ORACLE_LONG_DOUBLE
typedef long double real;
#else
typedef double real;
#endif

#define E(M, i, j) ((M)[(i) + 15 * (j)])

static void quat_multiply(const real* q, const real* p, real* o) {
    real t[4];
    t[0] = q[3] * p[0] + q[2] * p[1] - q[1] * p[2] + q[0] * p[3];
    t[1] = -q[2] * p[0] + q[3] * p[1] + q[0] * p[2] + q[1] * p[3];
    t[2] = q[1] * p[0] - q[0] * p[1] + q[3] * p[2] + q[2] * p[3];
    t[3] = -q[0] * p[0] - q[1] * p[1] - q[2] * p[2] + q[3] * p[3];
    if (t[3] < 0) for (int k = 0; k < 4; k++) t[k] = -t[k];
    const real n = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2] + t[3] * t[3]);
    for (int k = 0; k < 4; k++) o[k] = t[k] / n;
}

/* local(x_lin, x): as oracle/cpi_oracle.c local_state (the `same` test on the double inputs, so both builds take one branch) */
static void local_state(const double* xl_in, const double* x_in, real* d) {
    real xl[16], x[16], qi[4], dq[4];
    for (int k = 0; k < 16; k++) { xl[k] = xl_in[k]; x[k] = x_in[k]; }
    qi[0] = -xl[0]; qi[1] = -xl[1]; qi[2] = -xl[2]; qi[3] = xl[3];
    quat_multiply(x, qi, dq);
    const real s = sqrt(dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2]);
    const int same = x_in[0] == xl_in[0] && x_in[1] == xl_in[1] && x_in[2] == xl_in[2] && x_in[3] == xl_in[3];
    const real k = same ? 0 : (s > 0 ? 2 * atan2(s, dq[3]) / s : 2);
    for (int j = 0; j < 3; j++) d[j] = k * dq[j];
    for (int j = 0; j < 12; j++) d[3 + j] = x[4 + j] - xl[4 + j];
}

/* JPLNavState::retract, as oracle/cpi_oracle.c retract, on a `real` xi */
static void retract(const double* x_in, const real* xi, double* o_out) {
    real x[16], dq[4], o[16];
    for (int k = 0; k < 16; k++) x[k] = x_in[k];
    const real n = sqrt(xi[0] * xi[0] + xi[1] * xi[1] + xi[2] * xi[2]);
    for (int i = 0; i < 3; i++) dq[i] = (sin(n / 2) / n) * xi[i];
    dq[3] = cos(n / 2);
    real nn = sqrt(dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2] + dq[3] * dq[3]);
    for (int i = 0; i < 4; i++) dq[i] = dq[i] / nn;
    if (dq[3] < 0) for (int i = 0; i < 4; i++) dq[i] = -dq[i];
    nn = sqrt(dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2] + dq[3] * dq[3]);
    if (isnan(nn)) { dq[0] = dq[1] = dq[2] = 0; dq[3] = 1; }
    quat_multiply(dq, x, o);
    for (int i = 0; i < 12; i++) o[4 + i] = x[4 + i] + xi[3 + i];
    for (int k = 0; k < 16; k++) o_out[k] = (double)o[k];
}

/* A = L L^T in place from A's lower triangle (the upper triangle zeroed); 0 at the first pivot that is not positive */
static int chol15(real* A) {
    for (int j = 0; j < 15; j++) {
        real d = E(A, j, j);
        for (int k = 0; k < j; k++) d -= E(A, j, k) * E(A, j, k);
        if (!(d > 0)) return 0;
        d = sqrt(d);
        E(A, j, j) = d;
        for (int i = j + 1; i < 15; i++) {
            real s = E(A, i, j);
            for (int k = 0; k < j; k++) s -= E(A, i, k) * E(A, j, k);
            E(A, i, j) = s / d;
        }
        for (int i = 0; i < j; i++) E(A, i, j) = 0;
    }
    return 1;
}
static void fwd(const real* L, real* v) {           /* v <- L^-1 v */
    for (int i = 0; i < 15; i++) { real s = v[i]; for (int k = 0; k < i; k++) s -= E(L, i, k) * v[k]; v[i] = s / E(L, i, i); }
}
static void bwd(const real* L, real* v) {           /* v <- L^-T v */
    for (int i = 14; i >= 0; i--) { real s = v[i]; for (int k = i + 1; k < 15; k++) s -= E(L, k, i) * v[k]; v[i] = s / E(L, i, i); }
}
static void matvec(const real* A, const real* x, real* y) {
    for (int i = 0; i < 15; i++) { real s = 0; for (int k = 0; k < 15; k++) s += E(A, i, k) * x[k]; y[i] = s; }
}
static real quad(const real* A, const real* x) {
    real y[15], s = 0;
    matvec(A, x, y);
    for (int i = 0; i < 15; i++) s += x[i] * y[i];
    return s;
}

static void update_one(const double* x, const double* cov, const double* w_in, const double* xb, int order, double* x_out, double* c_out,
                       double* xi_out, double* nis) {
    real L[225], W[225], d[15], Wd[15], xi[15], S[225], g2 = 0;
    for (int e = 0; e < 225; e++) { L[e] = cov[e]; W[e] = w_in[e]; }
    local_state(xb, x, d);
    matvec(W, d, Wd);
    int ok = chol15(L);
    if (order == 0) {
        real B[225], C[225], M[225];
        for (int j = 0; j < 15; j++) {                /* B(:, j) = W L(:, j) */
            real col[15];
            for (int k = 0; k < 15; k++) col[k] = E(L, k, j);
            matvec(W, col, &B[15 * j]);
        }
        for (int i = 0; i < 15; i++)                  /* C = I + L^T (W L) */
            for (int j = 0; j < 15; j++) {
                real s = i == j;
                for (int k = 0; k < 15; k++) s += E(L, k, i) * E(B, k, j);
                E(C, i, j) = s;
            }
        ok = ok && chol15(C);
        real w[15];
        for (int i = 0; i < 15; i++) { real s = 0; for (int k = 0; k < 15; k++) s += E(L, k, i) * Wd[k]; w[i] = s; }
        fwd(C, w); bwd(C, w);
        for (int i = 0; i < 15; i++) { real s = 0; for (int k = 0; k < 15; k++) s += E(L, i, k) * w[k]; xi[i] = -s; g2 += w[i] * w[i]; }
        for (int i = 0; i < 15; i++) {                /* row i of M: C^-1 L(i, :)^T */
            real r[15];
            for (int k = 0; k < 15; k++) r[k] = E(L, i, k);
            fwd(C, r);
            for (int k = 0; k < 15; k++) E(M, i, k) = r[k];
        }
        for (int i = 0; i < 15; i++)
            for (int j = 0; j <= i; j++) {
                real s = 0;
                for (int k = 0; k < 15; k++) s += E(M, i, k) * E(M, j, k);
                E(S, i, j) = E(S, j, i) = s;
            }
    } else {
        real Si[225], P[225];
        for (int c = 0; c < 15; c++) {                /* S^-1 = L^-T L^-1, column by column */
            real y[15];
            for (int r = 0; r < 15; r++) y[r] = r == c;
            fwd(L, y); bwd(L, y);
            for (int r = 0; r < 15; r++) E(Si, r, c) = y[r];
        }
        for (int i = 0; i < 15; i++)
            for (int j = 0; j <= i; j++) E(P, i, j) = E(P, j, i) = 0.5 * (E(Si, i, j) + E(Si, j, i)) + 0.5 * (E(W, i, j) + E(W, j, i));
        ok = ok && chol15(P);
        for (int c = 0; c < 15; c++) {
            real y[15];
            for (int r = 0; r < 15; r++) y[r] = r == c;
            fwd(P, y); bwd(P, y);
            for (int r = c; r < 15; r++) E(S, r, c) = E(S, c, r) = y[r];
        }
        for (int i = 0; i < 15; i++) xi[i] = -Wd[i];
        fwd(P, xi); bwd(P, xi);
        g2 = quad(Si, xi);
    }
    real s[15];
    for (int i = 0; i < 15; i++) s[i] = d[i] + xi[i];
    const real g = quad(W, s) + g2;
    if (!ok) {
        for (int k = 0; k < 16; k++) x_out[k] = NAN;
        for (int e = 0; e < 225; e++) c_out[e] = NAN;
        for (int k = 0; k < 15; k++) xi_out[k] = NAN;
        *nis = NAN;
        return;
    }
    retract(x, xi, x_out);
    for (int e = 0; e < 225; e++) c_out[e] = (double)S[e];
    for (int k = 0; k < 15; k++) xi_out[k] = (double)xi[k];
    *nis = (double)g;
}

int oracle_state_update(int64_t n, const double* states, const double* cov, const double* W, const double* x_bar, int order,
                        double* states_out, double* cov_out, double* xi, double* nis) {
    if (order != 0 && order != 1) return 1;
    for (int64_t i = 0; i < n; i++)
        update_one(states + 16 * i, cov + 225 * i, W + 225 * i, x_bar + 16 * i, order, states_out + 16 * i, cov_out + 225 * i, xi + 15 * i,
                   nis + i);
    return 0;
}
