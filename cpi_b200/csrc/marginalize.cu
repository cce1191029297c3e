// The fixed-lag smoother side of the IMU chain (BatchFixedLagSmoother, solvers/GraphSolver.h:93-97, GraphSolver.cpp:202-203):
//   k_chain_marginalize  (K8) eliminates the leading states of many chains into a dense linear prior on the first state each chain
//                        keeps: the Schur complement GTSAM stores as a LinearContainerFactor, at the linearisation point of the blocks.
//                        One warp per chain, sequential over the eliminated factors:
//                            M = Lambda + G11_k,  r = eta + g1_k,  M = L L^T,  Z = L^-1 G12_k,  z = L^-1 r
//                            Lambda <- G22_k - Z^T Z,   eta <- g2_k - Z^T z,   f <- f + f_k - z^T z
//                        Lambda sits in shared memory (pitch 16, lower triangle), lanes 0..15 run the 15 + 1 forward substitutions,
//                        the 136 entries of [Z z]^T [Z z] are split over the lanes.
//   k_prior_at           moves such a prior to other states: delta = local(x_lin, x), rhs' = rhs - info delta,
//                        f' = f - 2 rhs^T delta + delta^T info delta (info unchanged; the Jacobian of local is taken as I, as
//                        LinearContainerFactor does).
// GTSAM is not part of the reference tree: PARITY UNPINNED -- validated against numpy statements (tests/test_marginalize.py).
#include <math_constants.h>

#include "cpi_common.cuh"
#include "cpi_kernels.h"
#include "chol15.cuh"
#include "local15.cuh"

namespace cpi {

__global__ void __launch_bounds__(128) k_chain_marginalize(int64_t n_chains, const int64_t* offs, int64_t uniform, const int64_t* n_marg,
                                                           int64_t marg_uniform, const double* G11, const double* G12, const double* G22,
                                                           const double* g1, const double* g2, const double* fk, const double* prior_info,
                                                           const double* prior_rhs, const double* prior_f, double* out_info, double* out_rhs,
                                                           double* out_f) {
    __shared__ double sL[4][15 * 16];          // Lambda (lower triangle), then M = Lambda + G11_k and its Cholesky factor
    __shared__ double sZ[4][15 * 16];          // [Z z] = L^-1 [G12_k r]: row q, column j at q * 16 + j (column 15 = z)
    __shared__ double sE[4][16];               // eta
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t c = (int64_t)blockIdx.x * 4 + wib;
    if (c >= n_chains) return;
    const int64_t lo = offs ? offs[c] : c * uniform, hi = offs ? offs[c + 1] : lo + uniform;
    const int64_t m = n_marg ? n_marg[c] : marg_uniform;
    double* oI = out_info + c * 225;
    double* oR = out_rhs + c * 15;
    if (!(m >= 0 && m < hi - lo)) {            // a device-resident count out of range: NaN for this chain only
        for (int t = lane; t < 225; t += 32) oI[t] = CUDART_NAN;
        if (lane < 15) oR[lane] = CUDART_NAN;
        if (lane == 0 && out_f) out_f[c] = CUDART_NAN;
        return;
    }
    if (m == 0) {                              // nothing eliminated: the input prior, bit for bit (zeros without one)
        for (int t = lane; t < 225; t += 32) oI[t] = prior_info ? prior_info[c * 225 + t] : 0.0;
        if (lane < 15) oR[lane] = prior_rhs ? prior_rhs[c * 15 + lane] : 0.0;
        if (lane == 0 && out_f) out_f[c] = prior_f ? prior_f[c] : 0.0;
        return;
    }
    double *L = sL[wib], *Z = sZ[wib], *eta = sE[wib];
    for (int t = lane; t < 225; t += 32) { const int r = t % 15, q = t / 15; if (r >= q) L[r * 16 + q] = prior_info ? prior_info[c * 225 + t] : 0.0; }
    if (lane < 15) eta[lane] = prior_rhs ? prior_rhs[c * 15 + lane] : 0.0;
    double f = prior_f ? prior_f[c] : 0.0;     // every lane keeps the same value
    for (int64_t k = 0; k < m; k++) {
        const int64_t fi = lo - c + k;         // factor k of the chain links its states k and k+1
        const double* A = G11 + fi * 225;
        __syncwarp();
        for (int t = lane; t < 225; t += 32) { const int r = t % 15, q = t / 15; if (r >= q) L[r * 16 + q] += A[t]; }
        __syncwarp();
        warp_chol15(L, lane);
        if (lane < 16) {
            double y[15];
            if (lane < 15) {
#pragma unroll
                for (int r = 0; r < 15; r++) y[r] = G12[fi * 225 + r + 15 * lane];        // column `lane` of G12
            } else {
#pragma unroll
                for (int r = 0; r < 15; r++) y[r] = eta[r] + g1[fi * 15 + r];
            }
            fwd15(L, y);
#pragma unroll
            for (int r = 0; r < 15; r++) Z[r * 16 + lane] = y[r];
        }
        __syncwarp();
        // entries (i, j), j <= i < 16, of [Z z]^T [Z z] except (15, 15): i < 15 -> Lambda, i == 15 -> eta
        for (int t = lane; t < 135; t += 32) {
            int i = 0, acc = 0;
            while (acc + i + 1 <= t) { acc += i + 1; i++; }
            const int j = t - acc;
            double s = 0.0;
#pragma unroll
            for (int q = 0; q < 15; q++) s = fma(Z[q * 16 + i], Z[q * 16 + j], s);
            if (i < 15) L[i * 16 + j] = G22[fi * 225 + i + 15 * j] - s;
            else eta[j] = g2[fi * 15 + j] - s;
        }
        double zz = 0.0;
#pragma unroll
        for (int q = 0; q < 15; q++) zz = fma(Z[q * 16 + 15], Z[q * 16 + 15], zz);
        f = f + fk[fi] - zz;
    }
    __syncwarp();
    for (int t = lane; t < 225; t += 32) {     // exactly symmetric: the lower triangle, mirrored
        const int r = t % 15, q = t / 15;
        oI[t] = r >= q ? L[r * 16 + q] : L[q * 16 + r];
    }
    if (lane < 15) oR[lane] = eta[lane];
    if (lane == 0 && out_f) out_f[c] = f;
}

// one warp per prior: every lane forms delta, lane r < 15 row r of info * delta
__global__ void __launch_bounds__(128) k_prior_at(int64_t n, const double* info, const double* rhs, const double* f, const double* lin,
                                                  const double* x, double* rhs_out, double* f_out) {
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * 4 + wib;
    if (i >= n) return;
    double d[15];
    local15(lin + i * CPI_STATE_DOUBLES, x + i * CPI_STATE_DOUBLES, d);
    double part = 0.0;                                             // delta_r (2 rhs_r - (info delta)_r): terms of 2 rhs^T delta - delta^T info delta
    if (lane < 15) {
        double u = 0.0;
#pragma unroll
        for (int q = 0; q < 15; q++) u = fma(info[i * 225 + lane + 15 * q], d[q], u);
        const double r = rhs[i * 15 + lane];
        double dl = 0.0;
#pragma unroll
        for (int q = 0; q < 15; q++) if (q == lane) dl = d[q];
        part = dl * (2.0 * r - u);
        rhs_out[i * 15 + lane] = r - u;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (lane == 0 && f_out) f_out[i] = (f ? f[i] : 0.0) - part;
}

cudaError_t marginalize_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, const int64_t* n_marg, int64_t marg_uniform,
                               const double* G11, const double* G12, const double* G22, const double* g1, const double* g2, const double* f,
                               const double* prior_info, const double* prior_rhs, const double* prior_f, double* out_info, double* out_rhs,
                               double* out_f, cudaStream_t st) {
    k_chain_marginalize<<<(int)((n_chains + 3) / 4), 128, 0, st>>>(n_chains, offs, uniform, n_marg, marg_uniform, G11, G12, G22, g1, g2, f,
                                                                   prior_info, prior_rhs, prior_f, out_info, out_rhs, out_f);
    return cudaGetLastError();
}

cudaError_t prior_at_launch(int64_t n, const double* info, const double* rhs, const double* f, const double* lin, const double* x,
                            double* rhs_out, double* f_out, cudaStream_t st) {
    k_prior_at<<<(int)((n + 3) / 4), 128, 0, st>>>(n, info, rhs, f, lin, x, rhs_out, f_out);
    return cudaGetLastError();
}

}  // namespace cpi
