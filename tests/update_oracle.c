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
 *   A Cholesky pivot that is not positive gives NaN outputs for that filter.
 *
 *   oracle_measurements_linearize(m, kind, state_idx, states, z, sqrt_info, aux, order, info, rhs, f)       (K12, DESIGN.md section 3l)
 *     r = h(x) - z, A = S H, b = S r.  order 0: info = A^T A, rhs' = -A^T b, f' = b^T b;  order 1: info = H^T (S^T S) H,
 *     rhs' = -H^T S^T (S r), f' = |S r|^2.  An unknown kind gives NaN in every entry.  Order 1 sums the products of h in the reverse
 *     order (here and in the filter updates), so that the two fp64 orders also differ in the rounding of r = h - z.
 *   oracle_state_update_measurements(n, states, cov, offsets, kind, z, sqrt_info, aux, order, states_out, cov_out, nis, sharp)   (K11)
 *     order 0: B_j = A_j L, C = chol(I + sum_j B_j^T B_j), w = C^-T C^-1 sum_j B_j^T b_j, xi = -L w, Sigma+ = M M^T with M = L C^-T,
 *              gamma = sum_j |b_j + A_j xi|^2 + |w|^2 (a sum of squares)
 *     order 1: P = Sigma^-1 + sum_j A_j^T A_j, Sigma+ = P^-1, xi = -P^-1 sum_j A_j^T b_j, gamma = sum_j |b_j + A_j xi|^2 + xi^T Sigma^-1 xi
 *     A filter without measurements is copied with gamma = 0.  sharp: lambda_max(L^T sum_j A_j^T A_j L), by power iteration.
 *   oracle_state_update_measurements_iterated(n, ..., loss, loss_k, gate, max_iter, tol, force, order, states_out, cov_out, nis,
 *                                             status, iterations, margin, x_lin, sharp)                            (K13, section 3m)
 *     Gauss-Newton from x_0 = x_hat with IRLS weights om_j = robust_loss'(|b_j(x_t)|^2), d_t = local(x_hat, x_t):
 *     order 0: B_j = sqrt(om_j) A_j L, b'_j = sqrt(om_j) (b_j - A_j d_t), w = C^-T C^-1 sum B_j^T b'_j, delta = -L w - d_t
 *     order 1: P = Sigma^-1 + sum om_j A_j^T A_j, delta = -P^-1 (Sigma^-1 d_t + sum om_j A_j^T b_j)
 *     x_{t+1} = retract(x_t, delta) until max_k |delta_k| <= tol sqrt(Sigma_kk) (status 1) or max_iter linearisations (status 2); with
 *     force[i] > 0 exactly force[i] linearisations, the status that of the last test.  gamma of the first linearisation, gated as K13
 *     (status 0: the inputs, one linearisation).  margin: the smallest |r - 1| over the tests taken, r = max_k |delta_k| / (tol sd_k)
 *     (+inf unless 0 < tol < inf); x_lin the last linearisation point; sharp the largest lambda_max over the linearisations. */
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

/* ---------------------------------------------------------------------------------------------- measurements (section 3l) */

enum { MEAS_POSITION = 1, MEAS_VELOCITY_BODY = 2, MEAS_DIRECTION = 3, LOSS_GAUSSIAN = 0, LOSS_HUBER = 1, LOSS_CAUCHY = 2 };

/* C = quat_2_Rot(q) = (2 w^2 - 1) I - 2 w [v]x + 2 v v^T, row-major (global to IMU, JPL) */
static void quat_2_Rot(const real* q, real* C) {
    const real v[3] = {q[0], q[1], q[2]}, w = q[3];
    const real K[9] = {0, -v[2], v[1], v[2], 0, -v[0], -v[1], v[0], 0};
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) C[3 * i + j] = (i == j ? 2 * w * w - 1 : 0) - 2 * w * K[3 * i + j] + 2 * v[i] * v[j];
}

static void skew(const real* a, real* K) {
    K[0] = 0; K[1] = -a[2]; K[2] = a[1]; K[3] = a[2]; K[4] = 0; K[5] = -a[0]; K[6] = -a[1]; K[7] = a[0]; K[8] = 0;
}

/* r = h(x) - z and H (row-major 3x15) of one measurement; 0 for an unknown kind.  alt sums the products of h in the reverse order, so that the two orders of the oracle round r = h - z differently (as the kernel's
 * fma chains round it differently again) */
static int meas_hr(int kind, const double* x_in, const double* z, const double* aux_in, int alt, real* r, real* H) {
    real x[16], a[3], C[9], h[3], K[9];
    for (int k = 0; k < 16; k++) x[k] = x_in[k];
    for (int k = 0; k < 3; k++) a[k] = aux_in[k];
    for (int k = 0; k < 45; k++) H[k] = 0;
    quat_2_Rot(x, C);
    if (kind == MEAS_POSITION) {                      /* h = p + C^T aux, H_theta = -C^T [aux]x, H_p = I */
        skew(a, K);
        for (int i = 0; i < 3; i++) {
            real t = 0;
            for (int k = 0; k < 3; k++) t += C[3 * (alt ? 2 - k : k) + i] * a[alt ? 2 - k : k];
            h[i] = alt ? t + x[13 + i] : x[13 + i] + t;
            for (int j = 0; j < 3; j++) {
                real t = 0;
                for (int k = 0; k < 3; k++) t += C[3 * k + i] * K[3 * k + j];
                H[15 * i + j] = -t;
            }
            H[15 * i + 12 + i] = 1;
        }
    } else if (kind == MEAS_VELOCITY_BODY || kind == MEAS_DIRECTION) {   /* h = C v (H_v = C) or C aux; H_theta = [h]x */
        const real* u = kind == MEAS_VELOCITY_BODY ? x + 7 : a;
        for (int i = 0; i < 3; i++) { h[i] = 0; for (int k = 0; k < 3; k++) h[i] += C[3 * i + (alt ? 2 - k : k)] * u[alt ? 2 - k : k]; }
        skew(h, K);
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) {
                H[15 * i + j] = K[3 * i + j];
                if (kind == MEAS_VELOCITY_BODY) H[15 * i + 6 + j] = C[3 * i + j];
            }
    } else {
        return 0;
    }
    for (int i = 0; i < 3; i++) r[i] = h[i] - z[i];
    return 1;
}

/* b = S r and A = S H (S column-major); NaN for an unknown kind */
static void meas_ab(int kind, const double* x, const double* z, const double* s, const double* aux, int alt, real* b, real* A) {
    real r[3], H[45];
    if (!meas_hr(kind, x, z, aux, alt, r, H)) {
        for (int k = 0; k < 3; k++) b[k] = NAN;
        for (int k = 0; k < 45; k++) A[k] = NAN;
        return;
    }
    for (int i = 0; i < 3; i++) {
        b[i] = 0;
        for (int k = 0; k < 3; k++) b[i] += (real)s[i + 3 * k] * r[k];
        for (int c = 0; c < 15; c++) {
            real t = 0;
            for (int k = 0; k < 3; k++) t += (real)s[i + 3 * k] * H[15 * k + c];
            A[15 * i + c] = t;
        }
    }
}

int oracle_measurements_linearize(int64_t m, const int32_t* kind, const int64_t* state_idx, const double* states, const double* z,
                                  const double* sqrt_info, const double* aux, int order, double* info, double* rhs, double* f) {
    if (order != 0 && order != 1) return 1;
    for (int64_t j = 0; j < m; j++) {
        const double* x = states + 16 * state_idx[j];
        const double *zj = z + 3 * j, *s = sqrt_info + 9 * j, *aj = aux + 3 * j;
        real Q[225], g[15], ff = 0;
        if (order == 0) {
            real A[45], b[3];
            meas_ab(kind[j], x, zj, s, aj, 0, b, A);
            for (int r = 0; r < 15; r++) {
                for (int c = 0; c < 15; c++) { real t = 0; for (int k = 0; k < 3; k++) t += A[15 * k + r] * A[15 * k + c]; E(Q, r, c) = t; }
                real t = 0;
                for (int k = 0; k < 3; k++) t += A[15 * k + r] * b[k];
                g[r] = -t;
            }
            for (int k = 0; k < 3; k++) ff += b[k] * b[k];
        } else {
            real r3[3], H[45], Lam[9], Sr[3], StSr[3];
            const int ok = meas_hr(kind[j], x, zj, aj, 1, r3, H);
            for (int a = 0; a < 3; a++)
                for (int c = 0; c < 3; c++) { real t = 0; for (int k = 0; k < 3; k++) t += (real)s[k + 3 * a] * s[k + 3 * c]; Lam[3 * a + c] = t; }
            for (int a = 0; a < 3; a++) { Sr[a] = 0; for (int k = 0; k < 3; k++) Sr[a] += (real)s[a + 3 * k] * r3[k]; }
            for (int a = 0; a < 3; a++) { StSr[a] = 0; for (int k = 0; k < 3; k++) StSr[a] += (real)s[k + 3 * a] * Sr[k]; }
            for (int r = 0; r < 15; r++) {
                for (int c = 0; c < 15; c++) {
                    real t = 0;
                    for (int a = 0; a < 3; a++)
                        for (int k = 0; k < 3; k++) t += H[15 * a + r] * Lam[3 * a + k] * H[15 * k + c];
                    E(Q, r, c) = t;
                }
                real t = 0;
                for (int a = 0; a < 3; a++) t += H[15 * a + r] * StSr[a];
                g[r] = -t;
            }
            for (int k = 0; k < 3; k++) ff += Sr[k] * Sr[k];
            if (!ok) {
                for (int e = 0; e < 225; e++) Q[e] = NAN;
                for (int k = 0; k < 15; k++) g[k] = NAN;
                ff = NAN;
            }
        }
        for (int e = 0; e < 225; e++) info[225 * j + e] = (double)Q[e];
        for (int k = 0; k < 15; k++) rhs[15 * j + k] = (double)g[k];
        f[j] = (double)ff;
    }
    return 0;
}

/* the IRLS weight of robust_loss (robust_loss.cuh), with its Cauchy overflow branch; NaN for an unknown code or k outside
 * 0 < k^2 < inf (k^2 formed in fp64, as the kernel compares it) */
static real robust_weight(int code, double k, real s) {
    if (code == LOSS_GAUSSIAN) return 1;
    const double k2d = k * k;
    if (!(k > 0 && k2d > 0 && k2d < INFINITY) || (code != LOSS_HUBER && code != LOSS_CAUCHY)) return NAN;
    const real k2 = k2d;
    if (code == LOSS_HUBER) return s <= k2 ? (real)1 : (real)k / sqrt(s);
    const double u = (double)s / k2d;
    if (isinf(u)) return k2 / s;                   /* k < 1, s > k^2 DBL_MAX: 1/(1+u) to the dropped k^2/s */
    return 1 / (1 + s / k2);
}

/* lambda_max of a symmetric PSD 15x15 (column-major), power iteration from the ones vector */
static real lambda_max(const real* G) {
    real v[15], y[15], lam = 0;
    for (int k = 0; k < 15; k++) v[k] = 1;
    for (int it = 0; it < 60; it++) {
        matvec(G, v, y);
        real n = 0, q = 0;
        for (int k = 0; k < 15; k++) { n += y[k] * y[k]; q += v[k] * y[k]; }
        real vv = 0;
        for (int k = 0; k < 15; k++) vv += v[k] * v[k];
        lam = q / vv;
        n = sqrt(n);
        if (!(n > 0)) return 0;
        for (int k = 0; k < 15; k++) v[k] = y[k] / n;
    }
    return lam;
}

/* One linearisation of filter i's measurements j0..j1-1 at xt with weights and d (d = 0: K11): the step delta and, when want_cov,
 * Sigma+ and the terms of gamma.  L the Cholesky factor of Sigma, Si = Sigma^-1 (order 1).  Returns 0 at a pivot that is not positive. */
static int linearisation(int order, const real* L, const real* Si, const double* xt, const real* d, int64_t j0, int64_t j1,
                         const int32_t* kind, const double* z, const double* sq, const double* aux, const int32_t* loss,
                         const double* loss_k, real* delta, real* eps, real* S, real* gw, real* sharp) {
    real G[225], u[15], LtGL[225];
    int ok = 1;
    for (int e = 0; e < 225; e++) G[e] = 0;
    for (int k = 0; k < 15; k++) u[k] = 0;
    for (int64_t j = j0; j < j1; j++) {                 /* G = sum om A^T A, u = sum om A^T (b - A d) */
        real A[45], b[3], e[3], s = 0;
        meas_ab(kind[j], xt, z + 3 * j, sq + 9 * j, aux + 3 * j, order, b, A);
        for (int k = 0; k < 3; k++) s += b[k] * b[k];
        const real om = loss ? robust_weight(loss[j], loss_k[j], s) : 1;
        for (int k = 0; k < 3; k++) { e[k] = b[k]; for (int c = 0; c < 15; c++) e[k] -= A[15 * k + c] * d[c]; }
        if (order == 0) {                               /* the square-root form: B = sqrt(om) A L, b' = sqrt(om) e */
            const real sw = sqrt(om);
            real B[45];
            for (int k = 0; k < 3; k++) {
                for (int c = 0; c < 15; c++) { real t = 0; for (int q = c; q < 15; q++) t += A[15 * k + q] * E(L, q, c); B[15 * k + c] = sw * t; }
                e[k] *= sw;
            }
            for (int r = 0; r < 15; r++) {
                for (int c = 0; c < 15; c++) for (int k = 0; k < 3; k++) E(G, r, c) += B[15 * k + r] * B[15 * k + c];
                for (int k = 0; k < 3; k++) u[r] += B[15 * k + r] * e[k];
            }
        } else {
            for (int r = 0; r < 15; r++) {
                for (int c = 0; c < 15; c++) for (int k = 0; k < 3; k++) E(G, r, c) += om * A[15 * k + r] * A[15 * k + c];
                for (int k = 0; k < 3; k++) u[r] += om * A[15 * k + r] * b[k];
            }
        }
    }
    if (order == 0) {
        for (int e = 0; e < 225; e++) LtGL[e] = G[e];
        *sharp = lambda_max(LtGL);
        real C[225], w[15], M[225];
        for (int e = 0; e < 225; e++) C[e] = G[e];
        for (int k = 0; k < 15; k++) E(C, k, k) += 1;
        ok = chol15(C);
        for (int k = 0; k < 15; k++) w[k] = u[k];
        fwd(C, w); bwd(C, w);
        *gw = 0;
        for (int i = 0; i < 15; i++) { real t = 0; for (int k = 0; k <= i; k++) t += E(L, i, k) * w[k]; eps[i] = -t; *gw += w[i] * w[i]; }
        for (int i = 0; i < 15; i++) delta[i] = eps[i] - d[i];
        for (int i = 0; i < 15; i++) {                  /* row i of M: C^-1 L(i, :)^T */
            real r[15];
            for (int k = 0; k < 15; k++) r[k] = E(L, i, k);
            fwd(C, r);
            for (int k = 0; k < 15; k++) E(M, i, k) = r[k];
        }
        for (int i = 0; i < 15; i++)
            for (int j = 0; j <= i; j++) { real t = 0; for (int k = 0; k < 15; k++) t += E(M, i, k) * E(M, j, k); E(S, i, j) = E(S, j, i) = t; }
    } else {
        real P[225], y[15];
        for (int i = 0; i < 15; i++)                    /* L^T G L for the sharpness */
            for (int j = 0; j < 15; j++) {
                real t = 0;
                for (int a = i; a < 15; a++) for (int b = j; b < 15; b++) t += E(L, a, i) * E(G, a, b) * E(L, b, j);
                E(LtGL, i, j) = t;
            }
        *sharp = lambda_max(LtGL);
        for (int i = 0; i < 15; i++)
            for (int j = 0; j <= i; j++) E(P, i, j) = E(P, j, i) = 0.5 * (E(Si, i, j) + E(Si, j, i)) + 0.5 * (E(G, i, j) + E(G, j, i));
        ok = chol15(P);
        for (int c = 0; c < 15; c++) {
            real v[15];
            for (int r = 0; r < 15; r++) v[r] = r == c;
            fwd(P, v); bwd(P, v);
            for (int r = c; r < 15; r++) E(S, r, c) = E(S, c, r) = v[r];
        }
        matvec(Si, d, y);
        for (int i = 0; i < 15; i++) delta[i] = -(y[i] + u[i]);
        fwd(P, delta); bwd(P, delta);
        for (int i = 0; i < 15; i++) eps[i] = d[i] + delta[i];
        *gw = quad(Si, eps);
    }
    return ok;
}

/* gamma's measurement term sum_j om_j |b_j + A_j eps|^2 at x */
static real gamma_meas(int order, const double* x, const real* eps, int64_t j0, int64_t j1, const int32_t* kind, const double* z,
                       const double* sq, const double* aux, const int32_t* loss, const double* loss_k) {
    real g = 0;
    for (int64_t j = j0; j < j1; j++) {
        real A[45], b[3], s = 0, t = 0;
        meas_ab(kind[j], x, z + 3 * j, sq + 9 * j, aux + 3 * j, order, b, A);
        for (int k = 0; k < 3; k++) s += b[k] * b[k];
        const real om = loss ? robust_weight(loss[j], loss_k[j], s) : 1;
        for (int k = 0; k < 3; k++) { real e = b[k]; for (int c = 0; c < 15; c++) e += A[15 * k + c] * eps[c]; t += e * e; }
        g += om * t;
    }
    return g;
}

int oracle_state_update_measurements_iterated(int64_t n, const double* states, const double* cov, const int64_t* offsets,
                                              const int32_t* kind, const double* z, const double* sqrt_info, const double* aux,
                                              const int32_t* loss, const double* loss_k, const double* gate, int max_iter, double tol,
                                              const int32_t* force, int order, double* states_out, double* cov_out, double* nis,
                                              int32_t* status, int32_t* iterations, double* margin, double* x_lin, double* sharp) {
    if ((order != 0 && order != 1) || max_iter < 1) return 1;
    for (int64_t i = 0; i < n; i++) {
        const double* x = states + 16 * i;
        const double* cv = cov + 225 * i;
        double *xo = states_out + 16 * i, *co = cov_out + 225 * i, *xl = x_lin + 16 * i;
        const int64_t j0 = offsets[i], j1 = offsets[i + 1];
        memcpy(xo, x, 16 * sizeof(double)); memcpy(xl, x, 16 * sizeof(double)); memcpy(co, cv, 225 * sizeof(double));
        nis[i] = 0; status[i] = 1; iterations[i] = 0; margin[i] = INFINITY; sharp[i] = 0;
        if (j0 >= j1) continue;
        real L[225], Si[225], S[225], d[15], delta[15], eps[15], gw, sh, mg = INFINITY;
        for (int e = 0; e < 225; e++) L[e] = cv[e];
        int ok = chol15(L);
        for (int c = 0; c < 15; c++) {                  /* Sigma^-1 = L^-T L^-1 */
            real y[15];
            for (int r = 0; r < 15; r++) y[r] = r == c;
            fwd(L, y); bwd(L, y);
            for (int r = 0; r < 15; r++) E(Si, r, c) = y[r];
        }
        double xt[16], xn[16];
        memcpy(xt, x, sizeof xt);
        const int cap = force && force[i] > 0 ? force[i] : max_iter;
        int t = 0, st = 2;
        real g = 0, shmax = 0;
        for (; t < cap; t++) {
            if (t == 0) for (int k = 0; k < 15; k++) d[k] = 0;
            else local_state(x, xt, d);
            ok = linearisation(order, L, Si, xt, d, j0, j1, kind, z, sqrt_info, aux, loss, loss_k, delta, eps, S, &gw, &sh) && ok;
            if (!(sh <= shmax)) shmax = sh;
            if (t == 0) {
                g = gamma_meas(order, x, eps, j0, j1, kind, z, sqrt_info, aux, loss, loss_k) + gw;
                if (gate && g > gate[i]) { st = 0; t = 1; break; }
            }
            int conv = 1;
            real rmax = 0;
            for (int k = 0; k < 15; k++) {
                const real sd = sqrt((real)cv[16 * k]);
                conv = conv && fabs(delta[k]) <= (real)tol * sd;
                const real r = fabs(delta[k]) / sd;
                if (!(r <= rmax)) rmax = r;
            }
            if (tol > 0 && tol < INFINITY) { const real m = fabs(rmax / (real)tol - 1); if (!(m >= mg)) mg = m; }
            memcpy(xl, xt, sizeof xt);
            retract(xt, delta, xn);
            memcpy(xt, xn, sizeof xt);
            st = conv ? 1 : 2;
            if (conv && !(force && force[i] > 0)) { t++; break; }
        }
        nis[i] = (double)g; status[i] = st; iterations[i] = t; margin[i] = (double)mg; sharp[i] = (double)shmax;
        if (!ok) {
            for (int k = 0; k < 16; k++) xo[k] = NAN;
            for (int e = 0; e < 225; e++) co[e] = NAN;
            nis[i] = NAN;
            continue;
        }
        if (st == 0) continue;
        memcpy(xo, xt, sizeof xt);
        for (int e = 0; e < 225; e++) co[e] = (double)S[e];
    }
    return 0;
}

int oracle_state_update_measurements(int64_t n, const double* states, const double* cov, const int64_t* offsets, const int32_t* kind,
                                     const double* z, const double* sqrt_info, const double* aux, int order, double* states_out,
                                     double* cov_out, double* nis, double* sharp) {
    int32_t st, it;
    double mg, xl[16];
    if (order != 0 && order != 1) return 1;
    for (int64_t i = 0; i < n; i++)                     /* one linearisation at x without a loss: K11 */
        oracle_state_update_measurements_iterated(1, states + 16 * i, cov + 225 * i, offsets + i, kind, z, sqrt_info, aux, NULL, NULL, NULL,
                                                  1, INFINITY, NULL, order, states_out + 16 * i, cov_out + 225 * i, nis + i, &st, &it,
                                                  &mg, xl, sharp + i);
    return 0;
}

int oracle_state_update(int64_t n, const double* states, const double* cov, const double* W, const double* x_bar, int order,
                        double* states_out, double* cov_out, double* xi, double* nis) {
    if (order != 0 && order != 1) return 1;
    for (int64_t i = 0; i < n; i++)
        update_one(states + 16 * i, cov + 225 * i, W + 225 * i, x_bar + 16 * i, order, states_out + 16 * i, cov_out + 225 * i, xi + 15 * i,
                   nis + i);
    return 0;
}
