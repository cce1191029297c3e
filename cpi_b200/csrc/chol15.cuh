// Warp-level 15x15 helpers shared by the chain solve (solve.cu) and the chain marginalisation (marginalize.cu).
// The matrix lives in shared memory, row-major with pitch 16.
#pragma once
#include "cpi_common.cuh"

namespace cpi {

// in-place lower Cholesky; a non-positive pivot gives NaN (GTSAM throws there)
CPI_DEV void warp_chol15(double* L, int lane) {
    for (int k = 0; k < 15; k++) {
        const double d = sqrt(L[k * 16 + k]);
        __syncwarp();
        if (lane == 0) L[k * 16 + k] = d;
        if (lane > k && lane < 15) L[lane * 16 + k] = L[lane * 16 + k] / d;
        __syncwarp();
        for (int t = lane; t < 120; t += 32) {
            int i = 0, acc = 0;
            while (acc + i + 1 <= t) { acc += i + 1; i++; }      // t -> (i, j) in the lower triangle incl. diagonal
            const int j = t - acc;
            if (j > k && i > k) L[i * 16 + j] -= L[i * 16 + k] * L[j * 16 + k];
        }
        __syncwarp();
    }
}
// y = L^-1 b  for a per-lane right-hand side held in registers (b -> y in place)
CPI_DEV void fwd15(const double* L, double* y) {
#pragma unroll
    for (int i = 0; i < 15; i++) {
        double t = y[i];
#pragma unroll
        for (int k = 0; k < i; k++) t = fma(-L[i * 16 + k], y[k], t);
        y[i] = t / L[i * 16 + i];
    }
}
// y = L^-T b  for a per-lane right-hand side held in registers (b -> y in place)
CPI_DEV void bwd15(const double* L, double* y) {
#pragma unroll
    for (int i = 14; i >= 0; i--) {
        double t = y[i];
#pragma unroll
        for (int k = i + 1; k < 15; k++) t = fma(-L[k * 16 + i], y[k], t);
        y[i] = t / L[i * 16 + i];
    }
}
// x = L^-T r : lane k (< 15) passes r_k and receives x_k; column-oriented backward substitution with shuffles
CPI_DEV double warp_bwd15(const double* L, double r, int lane) {
    double x = 0.0;
    for (int k = 14; k >= 0; k--) {
        const double xk = __shfl_sync(0xffffffffu, r, k) / L[k * 16 + k];
        if (lane == k) x = xk;
        if (lane < k) r = fma(-L[k * 16 + lane], xk, r);          // (L^T)[lane, k] = L[k, lane]
    }
    return x;
}

}  // namespace cpi
