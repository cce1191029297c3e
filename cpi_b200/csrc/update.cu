// K10: EKF measurement update of many filters by direct state fixes, with chi-square gating (DESIGN.md section 3k).  Filter i has
// the state x (16 doubles) and the error covariance Sigma (15x15, in the tangent space of retract); the fix is (W, x_bar) in the
// convention of the state priors: d = local(x_bar, x), Jacobian taken as I.  In square-root form (Sigma^-1 is never formed):
//   Sigma = L L^T,  C = chol(I + L^T W L),  u = L^T W d,  v = C^-1 u,  w = C^-T v,
//   xi = -L w,  Sigma+ = M M^T with M = L C^-T,  gamma = (d + xi)^T W (d + xi) + w^T w,  x+ = retract(x, xi)
// gamma > gate[i] skips the fix: x and Sigma are copied bit for bit.
//
// One warp per filter.  Sigma and W are staged in shared memory (row-major, pitch 16) with coalesced loads; d, u, v and w live in
// the spare column 15 of the pitch-16 buffers.  Lane c < 15 forms column c of L^T W L from column c of L, lane 15 forms u from d in
// the same pass.  After the warp's Cholesky of C, lane i < 15 solves row i of M while lane 15 solves for v; the warp solves for w
// with shuffles (warp_bwd15).  Then lane i < 15 forms row i of Sigma+ left of the diagonal and mirrors it, so Sigma+ is exactly
// symmetric, while lane 15 forms xi, gamma and the retraction.  No atomics: the same bits on every run.
#include "chol15.cuh"
#include "cpi_kernels.h"
#include "local15.cuh"
#include "measurement.cuh"
#include "robust_loss.cuh"

namespace cpi {

constexpr int UWARPS = 4;                        // filters (warps) per CTA
constexpr int UP = 240;                          // one 15x15 matrix, row-major with pitch 16

// JPLNavState::retract: the arithmetic of k_retract (factor.cu), kept as a local copy so that k_retract's code is untouched
CPI_DEV void retract_state(const double* x, const double* d, double* o) {
    const double nrm = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    double s, c;
    sincos(nrm / 2.0, &s, &c);
    double dq[4] = {(s / nrm) * d[0], (s / nrm) * d[1], (s / nrm) * d[2], c};
    double nn = sqrt(dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2] + dq[3] * dq[3]);
#pragma unroll
    for (int k = 0; k < 4; k++) dq[k] /= nn;
    if (dq[3] < 0) { dq[0] = -dq[0]; dq[1] = -dq[1]; dq[2] = -dq[2]; dq[3] = -dq[3]; }
    nn = sqrt(dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2] + dq[3] * dq[3]);
    if (isnan(nn)) { dq[0] = dq[1] = dq[2] = 0.0; dq[3] = 1.0; }
    const double q[4] = {x[0], x[1], x[2], x[3]};
    double qn[4];
    quat_multiply(dq, q, qn);
#pragma unroll
    for (int k = 0; k < 4; k++) o[k] = qn[k];
#pragma unroll
    for (int k = 0; k < 12; k++) o[4 + k] = x[4 + k] + d[3 + k];
}

__global__ void __launch_bounds__(UWARPS * 32) k_state_update(int64_t n, const double* states, const double* cov, const double* meas_info,
                                                             const double* meas_states, const double* gate, double* states_out,
                                                             double* cov_out, double* nis, int32_t* applied) {
    __shared__ double smem[UWARPS][4 * UP];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * UWARPS + warp;
    if (i >= n) return;
    double* L = smem[warp];                       // Sigma, then its Cholesky factor (lower triangle)
    double* W = L + UP;                           // the fix's information
    double* C = W + UP;                           // I + L^T W L (column 15: u), its Cholesky factor, then Sigma+
    double* M = C + UP;                           // L C^-T
    const double* sg = cov + i * 225;
    const double* wg = meas_info + i * 225;
    for (int e = lane; e < 225; e += 32) {        // column-major (r, c) -> row-major pitch 16
        const int r = e % 15, c = e / 15;
        L[r * 16 + c] = __ldg(sg + e);
        W[r * 16 + c] = __ldg(wg + e);
    }
    const double* x = states + i * CPI_STATE_DOUBLES;
    if (lane == 15) {                             // d = local(x_bar, x) in the spare column 15 of W
        double d[15];
        local15(meas_states + i * CPI_STATE_DOUBLES, x, d);
#pragma unroll
        for (int r = 0; r < 15; r++) W[r * 16 + 15] = d[r];
    }
    __syncwarp();
    warp_chol15(L, lane);

    if (lane < 16) {                              // column lane of L^T W L (lane 15: u = L^T W d)
        double y[15];                             // W a, a = column lane of L (lane 15: d), column by column
#pragma unroll
        for (int r = 0; r < 15; r++) y[r] = 0.0;
#pragma unroll
        for (int k = 0; k < 15; k++) {
            const double a = lane == 15 ? W[k * 16 + 15] : (k >= lane ? L[k * 16 + lane] : 0.0);
#pragma unroll
            for (int r = 0; r < 15; r++) y[r] = fma(W[r * 16 + k], a, y[r]);
        }
#pragma unroll
        for (int r = 0; r < 15; r++) {
            double t = 0.0;
#pragma unroll
            for (int k = r; k < 15; k++) t = fma(L[k * 16 + r], y[k], t);
            C[r * 16 + lane] = r == lane ? t + 1.0 : t;
        }
    }
    __syncwarp();
    warp_chol15(C, lane);                         // eigenvalues >= 1 for a PSD W; column 15 is not touched

    if (lane < 15) {                              // row lane of M: (C^-1 L^T)(:, lane) = C^-1 L(lane, :)^T
        double y[15];
#pragma unroll
        for (int k = 0; k < 15; k++) y[k] = k <= lane ? L[lane * 16 + k] : 0.0;
        fwd15(C, y);
#pragma unroll
        for (int k = 0; k < 15; k++) M[lane * 16 + k] = y[k];
    } else if (lane == 15) {                      // v = C^-1 u, in place of u
        double v[15];
#pragma unroll
        for (int k = 0; k < 15; k++) v[k] = C[k * 16 + 15];
        fwd15(C, v);
#pragma unroll
        for (int k = 0; k < 15; k++) C[k * 16 + 15] = v[k];
    }
    __syncwarp();
    {                                             // w = C^-T v = -L^-1 xi, lane k holds w_k; into the spare column 15 of M
        const double wk = warp_bwd15(C, lane < 15 ? C[lane * 16 + 15] : 0.0, lane);
        if (lane < 15) M[lane * 16 + 15] = wk;
    }
    __syncwarp();
    double g = 0.0;
    if (lane < 15) {                              // Sigma+(lane, j) = M(lane, :) M(j, :)^T, j <= lane, mirrored
        double y[15];
#pragma unroll
        for (int k = 0; k < 15; k++) y[k] = M[lane * 16 + k];
        for (int j = 0; j <= lane; j++) {
            double t = 0.0;
#pragma unroll
            for (int k = 0; k < 15; k++) t = fma(y[k], M[j * 16 + k], t);
            C[lane * 16 + j] = t;
            C[j * 16 + lane] = t;
        }
    } else if (lane == 15) {
        double w[15], g2 = 0.0;
#pragma unroll
        for (int k = 0; k < 15; k++) { w[k] = M[k * 16 + 15]; g2 = fma(w[k], w[k], g2); }
#pragma unroll
        for (int r = 14; r >= 0; r--) {           // xi = -L w in place (row r reads w[0..r])
            double t = 0.0;
#pragma unroll
            for (int k = 0; k <= r; k++) t = fma(L[r * 16 + k], w[k], t);
            w[r] = -t;
        }
        double g1 = 0.0;
#pragma unroll
        for (int r = 0; r < 15; r++) {            // (d + xi)^T W (d + xi)
            double t = 0.0;
#pragma unroll
            for (int k = 0; k < 15; k++) t = fma(W[r * 16 + k], W[k * 16 + 15] + w[k], t);
            g1 = fma(W[r * 16 + 15] + w[r], t, g1);
        }
        g = g1 + g2;
        const bool on = !(gate && g > __ldg(gate + i));
        double xo[16];
        if (on) retract_state(x, w, xo);
        else
#pragma unroll
            for (int k = 0; k < 16; k++) xo[k] = x[k];
        double* o = states_out + i * CPI_STATE_DOUBLES;
#pragma unroll
        for (int k = 0; k < 16; k++) o[k] = xo[k];
        if (nis) nis[i] = g;
        if (applied) applied[i] = on ? 1 : 0;
    }
    g = __shfl_sync(0xffffffffu, g, 15);
    const bool on = !(gate && g > __ldg(gate + i));
    __syncwarp();
    double* co = cov_out + i * 225;
    if (on)
        for (int e = lane; e < 225; e += 32) co[e] = C[(e % 15) * 16 + e / 15];
    else
        for (int e = lane; e < 225; e += 32) co[e] = __ldg(sg + e);
}

cudaError_t state_update_launch(int64_t n, const double* states, const double* cov, const double* meas_info, const double* meas_states,
                                const double* gate, double* states_out, double* cov_out, double* nis, int32_t* applied, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const int64_t grid = (n + UWARPS - 1) / UWARPS;
    k_state_update<<<(unsigned)grid, UWARPS * 32, 0, st>>>(n, states, cov, meas_info, meas_states, gate, states_out, cov_out, nis, applied);
    return cudaGetLastError();
}

// K11: the same update by the measurements of DESIGN.md section 3l (measurement.cuh), filter i's being meas_offsets[i] ..
// meas_offsets[i+1]-1, all linearised at x.  With B_j = A_j L, the accumulation replaces K10's L^T W L and u:
//   C = chol(I + sum_j B_j^T B_j),  u = sum_j B_j^T b_j,  w = C^-T C^-1 u,  xi = -L w,  Sigma+ = M M^T with M = L C^-T,
//   gamma = sum_j |b_j + A_j xi|^2 + |w|^2      (a sum of squares: no cancellation for sharp measurements)
// Per measurement, lane 0 stages A_j and b_j in the (not yet used) M buffer, lane c < 15 forms column c of B_j and lane 15 copies
// b_j beside it, then lane c < 16 adds column c of B_j^T [B_j b_j] to its registers: lane c's column of the Gram matrix and lane r's
// row are the same fma chain of commuted products.  From the Cholesky of C on, K10's steps; lane 15 relinearises each measurement
// at x for gamma.  A filter without measurements is copied bit for bit with gamma = 0 and applied = 1.
__global__ void __launch_bounds__(UWARPS * 32) k_state_update_meas(int64_t n, const double* states, const double* cov, const int64_t* meas_offsets,
                                                                  const int32_t* kind, const double* z, const double* sqrt_info, const double* aux,
                                                                  const double* gate, double* states_out, double* cov_out, double* nis,
                                                                  int32_t* applied) {
    __shared__ double smem[UWARPS][3 * UP];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * UWARPS + warp;
    if (i >= n) return;
    const double* sg = cov + i * 225;
    const double* x = states + i * CPI_STATE_DOUBLES;
    double* co = cov_out + i * 225;
    const int64_t j0 = __ldg(meas_offsets + i), j1 = __ldg(meas_offsets + i + 1);
    if (j0 >= j1) {                               // nothing to apply
        for (int e = lane; e < 225; e += 32) co[e] = __ldg(sg + e);
        if (lane < CPI_STATE_DOUBLES) states_out[i * CPI_STATE_DOUBLES + lane] = x[lane];
        if (lane == 0) {
            if (nis) nis[i] = 0.0;
            if (applied) applied[i] = 1;
        }
        return;
    }
    double* L = smem[warp];                       // Sigma, then its Cholesky factor (lower triangle)
    double* C = L + UP;                           // I + sum B^T B (column 15: u), its Cholesky factor, then Sigma+
    double* M = C + UP;                           // A_j, b_j (row-major 3x15, then 3) and B_j | b_j (3 rows, pitch 16); then L C^-T
    double* B = M + 48;
    for (int e = lane; e < 225; e += 32) L[(e % 15) * 16 + e / 15] = __ldg(sg + e);
    __syncwarp();
    warp_chol15(L, lane);

    double y[15];                                 // lane c < 15: column c of sum B^T B; lane 15: u
#pragma unroll
    for (int r = 0; r < 15; r++) y[r] = 0.0;
    for (int64_t j = j0; j < j1; j++) {
        if (lane == 0) meas_linearize(__ldg(kind + j), x, z + j * 3, sqrt_info + j * 9, aux + j * 3, M + 45, M);
        __syncwarp();
        if (lane < 15) {                          // B_j(k, lane) = sum_{m >= lane} A_j(k, m) L(m, lane)
#pragma unroll
            for (int k = 0; k < 3; k++) {
                double t = 0.0;
#pragma unroll
                for (int m = 0; m < 15; m++) t = m >= lane ? fma(M[k * 15 + m], L[m * 16 + lane], t) : t;
                B[k * 16 + lane] = t;
            }
        } else if (lane == 15) {
#pragma unroll
            for (int k = 0; k < 3; k++) B[k * 16 + 15] = M[45 + k];
        }
        __syncwarp();
        if (lane < 16) {
#pragma unroll
            for (int r = 0; r < 15; r++) y[r] = fma(B[32 + r], B[32 + lane], fma(B[16 + r], B[16 + lane], fma(B[r], B[lane], y[r])));
        }
        __syncwarp();
    }
    if (lane < 16) {
#pragma unroll
        for (int r = 0; r < 15; r++) C[r * 16 + lane] = r == lane ? y[r] + 1.0 : y[r];
    }
    __syncwarp();
    warp_chol15(C, lane);                         // eigenvalues >= 1; column 15 is not touched

    if (lane < 15) {                              // row lane of M = L C^-T
        double t[15];
#pragma unroll
        for (int k = 0; k < 15; k++) t[k] = k <= lane ? L[lane * 16 + k] : 0.0;
        fwd15(C, t);
#pragma unroll
        for (int k = 0; k < 15; k++) M[lane * 16 + k] = t[k];
    } else if (lane == 15) {                      // v = C^-1 u, in place of u
        double v[15];
#pragma unroll
        for (int k = 0; k < 15; k++) v[k] = C[k * 16 + 15];
        fwd15(C, v);
#pragma unroll
        for (int k = 0; k < 15; k++) C[k * 16 + 15] = v[k];
    }
    __syncwarp();
    {                                             // w = C^-T v, lane k holds w_k; into the spare column 15 of M
        const double wk = warp_bwd15(C, lane < 15 ? C[lane * 16 + 15] : 0.0, lane);
        if (lane < 15) M[lane * 16 + 15] = wk;
    }
    __syncwarp();
    double g = 0.0;
    if (lane < 15) {                              // Sigma+(lane, j) = M(lane, :) M(j, :)^T, j <= lane, mirrored
        double t[15];
#pragma unroll
        for (int k = 0; k < 15; k++) t[k] = M[lane * 16 + k];
        for (int j = 0; j <= lane; j++) {
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < 15; k++) s = fma(t[k], M[j * 16 + k], s);
            C[lane * 16 + j] = s;
            C[j * 16 + lane] = s;
        }
    } else if (lane == 15) {
        double w[15], g2 = 0.0;
#pragma unroll
        for (int k = 0; k < 15; k++) { w[k] = M[k * 16 + 15]; g2 = fma(w[k], w[k], g2); }
#pragma unroll
        for (int r = 14; r >= 0; r--) {           // xi = -L w in place (row r reads w[0..r])
            double t = 0.0;
#pragma unroll
            for (int k = 0; k <= r; k++) t = fma(L[r * 16 + k], w[k], t);
            w[r] = -t;
        }
        double g1 = 0.0;
        for (int64_t j = j0; j < j1; j++) {       // |b_j + A_j xi|^2
            double A[45], b[3];
            meas_linearize(__ldg(kind + j), x, z + j * 3, sqrt_info + j * 9, aux + j * 3, b, A);
#pragma unroll
            for (int k = 0; k < 3; k++) {
                double e = b[k];
#pragma unroll
                for (int c = 0; c < 15; c++) e = fma(A[k * 15 + c], w[c], e);
                g1 = fma(e, e, g1);
            }
        }
        g = g1 + g2;
        const bool on = !(gate && g > __ldg(gate + i));
        double xo[16];
        if (on) retract_state(x, w, xo);
        else
#pragma unroll
            for (int k = 0; k < 16; k++) xo[k] = x[k];
        double* o = states_out + i * CPI_STATE_DOUBLES;
#pragma unroll
        for (int k = 0; k < 16; k++) o[k] = xo[k];
        if (nis) nis[i] = g;
        if (applied) applied[i] = on ? 1 : 0;
    }
    g = __shfl_sync(0xffffffffu, g, 15);
    const bool on = !(gate && g > __ldg(gate + i));
    __syncwarp();
    if (on)
        for (int e = lane; e < 225; e += 32) co[e] = C[(e % 15) * 16 + e / 15];
    else
        for (int e = lane; e < 225; e += 32) co[e] = __ldg(sg + e);
}

cudaError_t state_update_meas_launch(int64_t n, const double* states, const double* cov, const int64_t* meas_offsets, const int32_t* kind,
                                     const double* z, const double* sqrt_info, const double* aux, const double* gate, double* states_out,
                                     double* cov_out, double* nis, int32_t* applied, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const int64_t grid = (n + UWARPS - 1) / UWARPS;
    k_state_update_meas<<<(unsigned)grid, UWARPS * 32, 0, st>>>(n, states, cov, meas_offsets, kind, z, sqrt_info, aux, gate, states_out,
                                                                cov_out, nis, applied);
    return cudaGetLastError();
}

// K13: the iterated update (DESIGN.md section 3m): Gauss-Newton on the one-step MAP problem
//   |L^-1 local(x_hat, x)|^2 + sum_j rho_j(|b_j(x)|^2)        (the prior's Jacobian taken as I, section 3g's convention)
// from x_0 = x_hat, relinearising the measurements at every iterate x_t and reweighting them by IRLS (robust_loss, section 3h):
//   d_t = local(x_hat, x_t),  A_j, b_j at x_t,  om_j = omega(|b_j|^2),  B_j = sqrt(om_j) A_j L,  b'_j = sqrt(om_j) (b_j - A_j d_t),
//   C = chol(I + sum_j B_j^T B_j),  w = C^-T C^-1 sum_j B_j^T b'_j,  eps = -L w,  delta = eps - d_t,  x_{t+1} = retract(x_t, delta)
// until max_k |delta_k| <= tol sqrt(Sigma_kk) (status 1) or max_iter linearisations (status 2).  Sigma+ = M M^T, M = L C^-T, from the
// last C; gamma = sum_j om_j |b_j + A_j eps_0|^2 + |w_0|^2 of the first linearisation is gated before the first step is taken
// (gamma > gate[i]: bit-for-bit copies, status 0, one linearisation).  At t = 0 (d_0 = 0 exactly, weights 1 without a loss) K13
// performs K11's operations in K11's order: Sigma+ and gamma are bitwise K11's, the state to rounding (ptxas contracts the
// retraction's unfused products differently in the two kernels; DESIGN.md section 3m).
// K11's buffers and steps: L is factored once; x_t, d_t and w live in 48 extra doubles per warp.  Lane 0 stages the weighted A_j and
// b'_j (folding -A_j d_t into column 15); lane 15 takes the step, the stopping test and the retraction, and broadcasts the decision.
// M and Sigma+ are formed once, after the loop.  No atomics: the same bits on every run.
__global__ void __launch_bounds__(UWARPS * 32) k_state_update_meas_iter(int64_t n, const double* states, const double* cov,
                                                                       const int64_t* meas_offsets, const int32_t* kind, const double* z,
                                                                       const double* sqrt_info, const double* aux, const int32_t* loss,
                                                                       const double* loss_k, const double* gate, int max_iter, double tol,
                                                                       double* states_out, double* cov_out, double* nis, int32_t* status,
                                                                       int32_t* iterations) {
    __shared__ double smem[UWARPS][3 * UP + 48];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * UWARPS + warp;
    if (i >= n) return;
    const double* sg = cov + i * 225;
    const double* x = states + i * CPI_STATE_DOUBLES;                // x_hat
    double* co = cov_out + i * 225;
    const int64_t j0 = __ldg(meas_offsets + i), j1 = __ldg(meas_offsets + i + 1);
    if (j0 >= j1) {                               // nothing to apply
        for (int e = lane; e < 225; e += 32) co[e] = __ldg(sg + e);
        if (lane < CPI_STATE_DOUBLES) states_out[i * CPI_STATE_DOUBLES + lane] = x[lane];
        if (lane == 0) {
            if (nis) nis[i] = 0.0;
            if (status) status[i] = 1;
            if (iterations) iterations[i] = 0;
        }
        return;
    }
    double* L = smem[warp];                       // Sigma, then its Cholesky factor (lower triangle)
    double* C = L + UP;                           // I + sum B^T B (column 15: u), its Cholesky factor; after the loop Sigma+
    double* M = C + UP;                           // weighted A_j, b'_j (row-major 3x15, then 3) and B_j | b'_j (3 rows, pitch 16); then L C^-T
    double* B = M + 48;
    double* X = M + UP;                           // x_t
    double* D = X + 16;                           // d_t
    double* W = D + 16;                           // w
    for (int e = lane; e < 225; e += 32) L[(e % 15) * 16 + e / 15] = __ldg(sg + e);
    if (lane < CPI_STATE_DOUBLES) X[lane] = x[lane];
    __syncwarp();
    warp_chol15(L, lane);

    double g = 0.0;
    int t = 0, st;                                // st: -1 go on, 0 gated, 1 converged, 2 stopped at max_iter
    do {
        if (lane == 15 && t > 0) {
            double d[15];
            local15(x, X, d);
#pragma unroll
            for (int r = 0; r < 15; r++) D[r] = d[r];
        }
        __syncwarp();
        double y[15];                             // lane c < 15: column c of sum B^T B; lane 15: u
#pragma unroll
        for (int r = 0; r < 15; r++) y[r] = 0.0;
        for (int64_t j = j0; j < j1; j++) {
            if (lane == 0) {
                meas_linearize(__ldg(kind + j), X, z + j * 3, sqrt_info + j * 9, aux + j * 3, M + 45, M);
                double om, c;
                robust_loss(loss ? __ldg(loss + j) : CPI_LOSS_GAUSSIAN, loss ? __ldg(loss_k + j) : 0.0,
                            fma(M[47], M[47], fma(M[46], M[46], M[45] * M[45])), om, c);
                if (t > 0)                        // b_j - A_j d_t (d_0 = 0)
#pragma unroll
                    for (int k = 0; k < 3; k++) {
                        double e = M[45 + k];
#pragma unroll
                        for (int m = 0; m < 15; m++) e = fma(-M[k * 15 + m], D[m], e);
                        M[45 + k] = e;
                    }
                if (om != 1.0) {
                    const double sw = sqrt(om);
#pragma unroll
                    for (int k = 0; k < 48; k++) M[k] *= sw;
                }
            }
            __syncwarp();
            if (lane < 15) {                      // B_j(k, lane) = sum_{m >= lane} A_j(k, m) L(m, lane)
#pragma unroll
                for (int k = 0; k < 3; k++) {
                    double s = 0.0;
#pragma unroll
                    for (int m = 0; m < 15; m++) s = m >= lane ? fma(M[k * 15 + m], L[m * 16 + lane], s) : s;
                    B[k * 16 + lane] = s;
                }
            } else if (lane == 15) {
#pragma unroll
                for (int k = 0; k < 3; k++) B[k * 16 + 15] = M[45 + k];
            }
            __syncwarp();
            if (lane < 16) {
#pragma unroll
                for (int r = 0; r < 15; r++) y[r] = fma(B[32 + r], B[32 + lane], fma(B[16 + r], B[16 + lane], fma(B[r], B[lane], y[r])));
            }
            __syncwarp();
        }
        if (lane < 16) {
#pragma unroll
            for (int r = 0; r < 15; r++) C[r * 16 + lane] = r == lane ? y[r] + 1.0 : y[r];
        }
        __syncwarp();
        warp_chol15(C, lane);                     // eigenvalues >= 1; column 15 is not touched
        if (lane == 15) {                         // v = C^-1 u, in place of u
            double v[15];
#pragma unroll
            for (int k = 0; k < 15; k++) v[k] = C[k * 16 + 15];
            fwd15(C, v);
#pragma unroll
            for (int k = 0; k < 15; k++) C[k * 16 + 15] = v[k];
        }
        __syncwarp();
        {                                         // w = C^-T v, lane k holds w_k
            const double wk = warp_bwd15(C, lane < 15 ? C[lane * 16 + 15] : 0.0, lane);
            if (lane < 15) W[lane] = wk;
        }
        __syncwarp();
        st = -1;
        if (lane == 15) {
            double w[15], g2 = 0.0;
#pragma unroll
            for (int k = 0; k < 15; k++) { w[k] = W[k]; g2 = fma(w[k], w[k], g2); }
#pragma unroll
            for (int r = 14; r >= 0; r--) {       // eps = -L w in place (row r reads w[0..r])
                double s = 0.0;
#pragma unroll
                for (int k = 0; k <= r; k++) s = fma(L[r * 16 + k], w[k], s);
                w[r] = -s;
            }
            if (t == 0) {                         // gamma: sum om_j |b_j + A_j eps_0|^2 + |w_0|^2 at x_hat
                double g1 = 0.0;
                for (int64_t j = j0; j < j1; j++) {
                    double A[45], b[3], om, c;
                    meas_linearize(__ldg(kind + j), x, z + j * 3, sqrt_info + j * 9, aux + j * 3, b, A);
                    robust_loss(loss ? __ldg(loss + j) : CPI_LOSS_GAUSSIAN, loss ? __ldg(loss_k + j) : 0.0,
                                fma(b[2], b[2], fma(b[1], b[1], b[0] * b[0])), om, c);
#pragma unroll
                    for (int k = 0; k < 3; k++) {
                        double e = b[k];
#pragma unroll
                        for (int q = 0; q < 15; q++) e = fma(A[k * 15 + q], w[q], e);
                        g1 = fma(om * e, e, g1);
                    }
                }
                g = g1 + g2;
                if (gate && g > __ldg(gate + i)) st = 0;
            } else {                              // delta = eps - d_t
#pragma unroll
                for (int k = 0; k < 15; k++) w[k] -= D[k];
            }
            if (st != 0) {
                bool conv = true;
#pragma unroll
                for (int k = 0; k < 15; k++) conv = conv && fabs(w[k]) <= tol * sqrt(__ldg(sg + k * 16));
                double xo[16];
                retract_state(X, w, xo);
#pragma unroll
                for (int k = 0; k < 16; k++) X[k] = xo[k];
                st = conv ? 1 : (t + 1 >= max_iter ? 2 : -1);
            }
        }
        st = __shfl_sync(0xffffffffu, st, 15);
        t++;
        __syncwarp();
    } while (st < 0);

    if (st == 0) {                                // gated: the inputs
        for (int e = lane; e < 225; e += 32) co[e] = __ldg(sg + e);
        if (lane < CPI_STATE_DOUBLES) states_out[i * CPI_STATE_DOUBLES + lane] = x[lane];
    } else {
        if (lane < 15) {                          // row lane of M = L C^-T, from the last C
            double r[15];
#pragma unroll
            for (int k = 0; k < 15; k++) r[k] = k <= lane ? L[lane * 16 + k] : 0.0;
            fwd15(C, r);
#pragma unroll
            for (int k = 0; k < 15; k++) M[lane * 16 + k] = r[k];
        }
        __syncwarp();
        if (lane < 15) {                          // Sigma+(lane, j) = M(lane, :) M(j, :)^T, j <= lane, mirrored
            double r[15];
#pragma unroll
            for (int k = 0; k < 15; k++) r[k] = M[lane * 16 + k];
            for (int j = 0; j <= lane; j++) {
                double s = 0.0;
#pragma unroll
                for (int k = 0; k < 15; k++) s = fma(r[k], M[j * 16 + k], s);
                C[lane * 16 + j] = s;
                C[j * 16 + lane] = s;
            }
        }
        __syncwarp();
        for (int e = lane; e < 225; e += 32) co[e] = C[(e % 15) * 16 + e / 15];
        if (lane < CPI_STATE_DOUBLES) states_out[i * CPI_STATE_DOUBLES + lane] = X[lane];
    }
    if (lane == 15) {
        if (nis) nis[i] = g;
        if (status) status[i] = st;
        if (iterations) iterations[i] = t;
    }
}

cudaError_t state_update_meas_iter_launch(int64_t n, const double* states, const double* cov, const int64_t* meas_offsets, const int32_t* kind,
                                          const double* z, const double* sqrt_info, const double* aux, const int32_t* loss, const double* loss_k,
                                          const double* gate, int max_iter, double tol, double* states_out, double* cov_out, double* nis,
                                          int32_t* status, int32_t* iterations, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const int64_t grid = (n + UWARPS - 1) / UWARPS;
    k_state_update_meas_iter<<<(unsigned)grid, UWARPS * 32, 0, st>>>(n, states, cov, meas_offsets, kind, z, sqrt_info, aux, loss, loss_k, gate,
                                                                     max_iter, tol, states_out, cov_out, nis, status, iterations);
    return cudaGetLastError();
}

}  // namespace cpi
