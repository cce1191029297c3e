// The step GTSAM performs after evaluateError, for an IMU-only chain, entirely on the device (SURVEY.md 8f rank 1):
//   k_factor_whiten   A = R_w [H1 H2], b = -R_w e  with the factor's noise model noiseModel::Gaussian::Covariance(P_meas)
//                     (gtsam/ImuFactorCPIv1.h:82, ImuFactorCPIv2.h:86): R_w = upper Cholesky factor of P_meas^-1, R_w^T R_w = P_meas^-1
//   k_chain_assemble  scatter-add of the per-factor information blocks into the block-tridiagonal normal equations of the chain
//                     x_0 - x_1 - ... - x_n  (what BatchFixedLagSmoother::update assembles, solvers/GraphSolver.cpp:202-203)
//   block cyclic reduction: a Cholesky-based solve of that SPD block-tridiagonal system (15x15 blocks) in log2(n) parallel levels
//                     instead of a 5 000-step sequential block recurrence: odd nodes are eliminated (one warp per node: Cholesky of the
//                     diagonal block + 31 forward substitutions), even nodes receive the Schur complements (one warp per node).
// GTSAM is not part of the reference tree (bitbucket gtborg/gtsam @ c21186c): PARITY UNPINNED -- validated against dense / banded
// CPU solves of the same system (tests/test_gpu_parity.py).
#include "cpi_common.cuh"
#include "cpi_kernels.h"
#include "chol15.cuh"

namespace cpi {

// ---- explicitly whitened Jacobian form --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_factor_whiten(int64_t n, int rd, const double* records, const double* e, const double* H1, const double* H2,
                                                       double* A1, double* A2, double* bw) {
    __shared__ double sL[4][15 * 16], sM[4][15 * 16], sR[4][15 * 16];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t f = (int64_t)blockIdx.x * 4 + wib;
    if (f >= n) return;
    double *L = sL[wib], *M = sM[wib], *R = sR[wib];
    const double* P = records + f * (int64_t)rd + CPI_REC_P;
    for (int k = lane; k < 225; k += 32) { const int r = k % 15, c = k / 15; if (r >= c) L[r * 16 + c] = __ldg(P + k); }
    __syncwarp();
    warp_chol15(L, lane);                                          // P = L L^T
    // M = L^-1 (lane c: column c of the inverse), then information = M^T M
    if (lane < 15) {
        double y[15];
#pragma unroll
        for (int i = 0; i < 15; i++) y[i] = (i == lane) ? 1.0 : 0.0;
        fwd15(L, y);
#pragma unroll
        for (int i = 0; i < 15; i++) M[i * 16 + lane] = y[i];
    }
    __syncwarp();
    for (int t = lane; t < 225; t += 32) {                         // lower triangle of P^-1 = M^T M into R (to be factored in place)
        const int i = t / 15, j = t % 15;
        if (j <= i) {
            double s = 0.0;
            for (int k = i; k < 15; k++) s = fma(M[k * 16 + i], M[k * 16 + j], s);     // M is lower triangular: rows >= max(i, j)
            R[i * 16 + j] = s;
        }
    }
    __syncwarp();
    warp_chol15(R, lane);                                          // P^-1 = C C^T  ->  R_w = C^T (upper), R_w^T R_w = P^-1
    // A = R_w H:  (R_w H)[i, c] = sum_{k >= i} C[k, i] H[k, c];  lanes 0..14 -> columns of H1, 15..29 -> H2, 30 -> -e
    if (lane < 31) {
        const double* src = lane < 15 ? H1 + f * 225 + 15 * lane : (lane < 30 ? H2 + f * 225 + 15 * (lane - 15) : e + f * 15);
        double h[15];
#pragma unroll
        for (int i = 0; i < 15; i++) h[i] = __ldg(src + i);
        double* dst = lane < 15 ? A1 + f * 225 + 15 * lane : (lane < 30 ? A2 + f * 225 + 15 * (lane - 15) : bw + f * 15);
        const double sgn = lane < 30 ? 1.0 : -1.0;
#pragma unroll
        for (int i = 0; i < 15; i++) {
            double s = 0.0;
#pragma unroll
            for (int k = i; k < 15; k++) s = fma(R[k * 16 + i], h[k], s);
            dst[i] = sgn * s;
        }
    }
}

// ---- chain assembly ---------------------------------------------------------------------------------------------------------------
// Many independent chains in one block-tridiagonal system.  Chain c holds states o[c] .. o[c+1]-1 of the concatenated states
// (o = offs, or o[c] = c * uniform); its factors are stored back to back from index o[c] - c, so state k of chain c is linked to
// state k+1 by factor k - c.  One chain (o = {0, nf+1}) is the chain x_0 - ... - x_nf with factor f linking states f and f+1.
//   D[k] = G22[k-1-c] (k not first) + G11[k-c] (k not last) (+ prior_info[c] on the chain's first state) + damping
//   E[k] = G12[k-c] (block (k, k+1)), exactly 0 where k is the last state of its chain,   rhs[k] = g2[k-1-c] + g1[k-c] (+ prior_rhs[c])
// Damping as in GTSAM's LevenbergMarquardtParams: lambda I, or with diagonalDamping lambda * clamp(diag, minDiagonal 1e-6, maxDiagonal 1e32).
// Grid-stride over the states: the state count o[n_chains] of a device-resident layout is read here, not on the host.
// PER_CHAIN: lambda is lams[c] per chain, and damp (may be NULL) receives the diagonal the damping added, [N, 15]
// (cpi_imu_chains_assemble_lm, lm.cu); otherwise the scalar lambda.
template <bool PER_CHAIN>
CPI_DEV void chain_assemble_body(int64_t n_chains, const int64_t* offs, int64_t uniform, const double* G11, const double* G12, const double* G22,
                                 const double* g1, const double* g2, double lambda, const double* lams, int diagonal_damping,
                                 const double* prior_info, const double* prior_rhs, double* D, double* E, double* rhs, double* damp) {
    const int64_t ns = offs ? offs[n_chains] : n_chains * uniform;
    for (int64_t k = blockIdx.x; k < ns; k += gridDim.x) {
        int64_t c, lo, hi;
        if (offs) {                                                // the chain holding k: last c with o[c] <= k (chains are non-empty)
            int64_t a = 0, b = n_chains - 1;
            while (a < b) { const int64_t mid = (a + b + 1) >> 1; if (offs[mid] <= k) a = mid; else b = mid - 1; }
            c = a; lo = offs[c]; hi = offs[c + 1];
        } else {
            c = k / uniform; lo = c * uniform; hi = lo + uniform;
        }
        const bool first = k == lo, last = k == hi - 1;
        const int64_t fr = k - c;                                  // the factor to the right of state k (if k is not last)
        const double lam = PER_CHAIN ? lams[c] : lambda;
        for (int t = threadIdx.x; t < 225; t += blockDim.x) {
            double d = 0.0;
            if (!first) d += G22[(fr - 1) * 225 + t];
            if (!last) d += G11[fr * 225 + t];
            if (k + 1 < ns) E[k * 225 + t] = last ? 0.0 : G12[fr * 225 + t];
            if (first && prior_info) d += prior_info[c * 225 + t];
            if (t % 16 == 0) {                                     // t = r + 15 c: diagonal when r == c  <=>  t % 16 == 0
                const double a = diagonal_damping ? lam * fmin(fmax(d, 1e-6), 1e32) : lam;
                if (PER_CHAIN && damp) damp[k * 15 + t / 16] = a;
                d += a;
            }
            D[k * 225 + t] = d;
        }
        for (int t = threadIdx.x; t < 15; t += blockDim.x) {
            double v = 0.0;
            if (!first) v += g2[(fr - 1) * 15 + t];
            if (!last) v += g1[fr * 15 + t];
            if (first && prior_rhs) v += prior_rhs[c * 15 + t];
            rhs[k * 15 + t] = v;
        }
    }
}

__global__ void k_chain_assemble(int64_t n_chains, const int64_t* offs, int64_t uniform, const double* G11, const double* G12, const double* G22,
                                 const double* g1, const double* g2, double lambda, int diagonal_damping, const double* prior_info,
                                 const double* prior_rhs, double* D, double* E, double* rhs) {
    chain_assemble_body<false>(n_chains, offs, uniform, G11, G12, G22, g1, g2, lambda, nullptr, diagonal_damping, prior_info, prior_rhs, D, E, rhs,
                               nullptr);
}

__global__ void k_chain_assemble_lm(int64_t n_chains, const int64_t* offs, int64_t uniform, const double* G11, const double* G12, const double* G22,
                                    const double* g1, const double* g2, const double* lams, int diagonal_damping, const double* prior_info,
                                    const double* prior_rhs, double* D, double* E, double* rhs, double* damp) {
    chain_assemble_body<true>(n_chains, offs, uniform, G11, G12, G22, g1, g2, 0.0, lams, diagonal_damping, prior_info, prior_rhs, D, E, rhs, damp);
}

// ---- block cyclic reduction ---------------------------------------------------------------------------------------------------------
// Level with m nodes: row i reads  E[i-1]^T x_{i-1} + D[i] x_i + E[i] x_{i+1} = b[i].
// ISO (cpi_imu_chains_solve): node i of the level sits at original state i * stride, cid[] holds each original state's chain, and a
// coupling between nodes of different chains is structurally absent: not loaded, not multiplied, written as exact 0.  With finite
// input those couplings are exact zeros anyway, so the ISO kernels give the plain kernels' bits; a NaN stays inside its chain.
#define CPI_SAME(p, q) (!ISO || cid[(p) * stride] == cid[(q) * stride])
#define SAME(p, q) (cid[(p) * stride] == cid[(q) * stride])

// Odd node i = 2t+1:  D_i = Lc Lc^T,  Za = Lc^-1 E[i-1]^T,  Zb = Lc^-1 E[i] (if i+1 < m),  zb = Lc^-1 b_i      (kept for the back-substitution)
template <bool ISO>
CPI_DEV void bcr_eliminate(int64_t m, int64_t stride, const int64_t* cid, const double* D, const double* E, const double* b, double* Lc, double* Za,
                           double* Zb, double* zb) {
    __shared__ double sL[4][15 * 16];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t t = (int64_t)blockIdx.x * 4 + wib;
    const int64_t i = 2 * t + 1;
    if (i >= m) return;
    double* L = sL[wib];
    for (int k = lane; k < 225; k += 32) { const int r = k % 15, c = k / 15; if (r >= c) L[r * 16 + c] = D[i * 225 + k]; }
    __syncwarp();
    warp_chol15(L, lane);
    for (int k = lane; k < 225; k += 32) { const int r = k % 15, c = k / 15; Lc[t * 225 + k] = (r >= c) ? L[r * 16 + c] : 0.0; }
    const bool has_left = CPI_SAME(i - 1, i);
    const bool has_right = i + 1 < m && CPI_SAME(i + 1, i);
    if (lane < 31) {
        double y[15];
        if (lane < 15) {
#pragma unroll
            for (int r = 0; r < 15; r++) y[r] = has_left ? E[(i - 1) * 225 + lane + 15 * r] : 0.0;      // column `lane` of E[i-1]^T = row `lane` of E[i-1]
        } else if (lane < 30) {
#pragma unroll
            for (int r = 0; r < 15; r++) y[r] = has_right ? E[i * 225 + r + 15 * (lane - 15)] : 0.0;
        } else {
#pragma unroll
            for (int r = 0; r < 15; r++) y[r] = b[i * 15 + r];
        }
        fwd15(L, y);
        double* dst = lane < 15 ? Za + t * 225 + 15 * lane : (lane < 30 ? Zb + t * 225 + 15 * (lane - 15) : zb + t * 15);
        if (ISO && ((lane < 15 && !has_left) || (lane >= 15 && lane < 30 && !has_right))) {
#pragma unroll
            for (int r = 0; r < 15; r++) y[r] = 0.0;
        }
#pragma unroll
        for (int r = 0; r < 15; r++) dst[r] = y[r];
    }
}

// Even node j = 2u -> node u of the next level:
//   D' = D_j - Zb_{j-1}^T Zb_{j-1} - Za_{j+1}^T Za_{j+1},   b' = b_j - Zb_{j-1}^T zb_{j-1} - Za_{j+1}^T zb_{j+1},   E' = -Za_{j+1}^T Zb_{j+1}  (couples x_j and x_{j+2})
CPI_DEV void bcr_reduce_iso(int64_t m, int64_t stride, const int64_t* cid, const double* D, const double* b, const double* Za, const double* Zb,
                        const double* zb, double* Dn, double* En, double* bn) {
    __shared__ double sZ[4][4][225 + 15];      // [warp][ZbL | ZaR | ZbR | (zbL, zbR)]
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t u = (int64_t)blockIdx.x * 4 + wib;
    const int64_t j = 2 * u;
    if (j >= m) return;
    const bool hasL = j >= 1 && SAME(j - 1, j), hasR = j + 1 < m && SAME(j + 1, j), hasRR = j + 2 < m;
    const bool linkRR = hasRR && SAME(j + 2, j);                   // x_j and x_{j+2} in one chain (then x_{j+1} too)
    const int64_t tl = (j - 2) / 2, tr = j / 2;                     // odd-node slots of j-1 and j+1
    double *ZbL = sZ[wib][0], *ZaR = sZ[wib][1], *ZbR = sZ[wib][2], *zz = sZ[wib][3];
    for (int k = lane; k < 225; k += 32) {
        ZbL[k] = hasL ? Zb[tl * 225 + k] : 0.0;
        ZaR[k] = hasR ? Za[tr * 225 + k] : 0.0;
        ZbR[k] = linkRR ? Zb[tr * 225 + k] : 0.0;
    }
    if (lane < 15) { zz[lane] = hasL ? zb[tl * 15 + lane] : 0.0; zz[15 + lane] = hasR ? zb[tr * 15 + lane] : 0.0; }
    __syncwarp();
    for (int k = lane; k < 225; k += 32) {
        const int r = k % 15, c = k / 15;                          // column-major 15x15; Z matrices are column-major: Z[q + 15 col]
        double d = D[j * 225 + k], en = 0.0;
#pragma unroll
        for (int q = 0; q < 15; q++) {
            d = fma(-ZbL[q + 15 * r], ZbL[q + 15 * c], d);
            d = fma(-ZaR[q + 15 * r], ZaR[q + 15 * c], d);
            en = fma(-ZaR[q + 15 * r], ZbR[q + 15 * c], en);
        }
        Dn[u * 225 + k] = d;
        if (hasRR) En[u * 225 + k] = linkRR ? en : 0.0;
    }
    if (lane < 15) {
        double v = b[j * 15 + lane];
#pragma unroll
        for (int q = 0; q < 15; q++) { v = fma(-ZbL[q + 15 * lane], zz[q], v); v = fma(-ZaR[q + 15 * lane], zz[15 + q], v); }
        bn[u * 15 + lane] = v;
    }
}

__global__ void __launch_bounds__(128) k_bcr_eliminate(int64_t m, const double* D, const double* E, const double* b, double* Lc, double* Za, double* Zb, double* zb) {
    bcr_eliminate<false>(m, 0, nullptr, D, E, b, Lc, Za, Zb, zb);
}
// (k_bcr_reduce keeps its own copy of the body: through bcr_reduce<false> its register allocation changes)
__global__ void __launch_bounds__(128) k_bcr_reduce(int64_t m, const double* D, const double* b, const double* Za, const double* Zb, const double* zb,
                                                    double* Dn, double* En, double* bn) {
    __shared__ double sZ[4][4][225 + 15];      // [warp][ZbL | ZaR | ZbR | (zbL, zbR)]
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t u = (int64_t)blockIdx.x * 4 + wib;
    const int64_t j = 2 * u;
    if (j >= m) return;
    const bool hasL = j >= 1, hasR = j + 1 < m, hasRR = j + 2 < m;
    const int64_t tl = (j - 2) / 2, tr = j / 2;                     // odd-node slots of j-1 and j+1
    double *ZbL = sZ[wib][0], *ZaR = sZ[wib][1], *ZbR = sZ[wib][2], *zz = sZ[wib][3];
    for (int k = lane; k < 225; k += 32) {
        ZbL[k] = hasL ? Zb[tl * 225 + k] : 0.0;
        ZaR[k] = hasR ? Za[tr * 225 + k] : 0.0;
        ZbR[k] = hasRR ? Zb[tr * 225 + k] : 0.0;
    }
    if (lane < 15) { zz[lane] = hasL ? zb[tl * 15 + lane] : 0.0; zz[15 + lane] = hasR ? zb[tr * 15 + lane] : 0.0; }
    __syncwarp();
    for (int k = lane; k < 225; k += 32) {
        const int r = k % 15, c = k / 15;                          // column-major 15x15; Z matrices are column-major: Z[q + 15 col]
        double d = D[j * 225 + k], en = 0.0;
#pragma unroll
        for (int q = 0; q < 15; q++) {
            d = fma(-ZbL[q + 15 * r], ZbL[q + 15 * c], d);
            d = fma(-ZaR[q + 15 * r], ZaR[q + 15 * c], d);
            en = fma(-ZaR[q + 15 * r], ZbR[q + 15 * c], en);
        }
        Dn[u * 225 + k] = d;
        if (hasRR) En[u * 225 + k] = en;
    }
    if (lane < 15) {
        double v = b[j * 15 + lane];
#pragma unroll
        for (int q = 0; q < 15; q++) { v = fma(-ZbL[q + 15 * lane], zz[q], v); v = fma(-ZaR[q + 15 * lane], zz[15 + q], v); }
        bn[u * 15 + lane] = v;
    }
}
__global__ void __launch_bounds__(128) k_bcr_eliminate_iso(int64_t m, int64_t stride, const int64_t* cid, const double* D, const double* E, const double* b,
                                                           double* Lc, double* Za, double* Zb, double* zb) {
    bcr_eliminate<true>(m, stride, cid, D, E, b, Lc, Za, Zb, zb);
}
__global__ void __launch_bounds__(128) k_bcr_reduce_iso(int64_t m, int64_t stride, const int64_t* cid, const double* D, const double* b, const double* Za,
                                                        const double* Zb, const double* zb, double* Dn, double* En, double* bn) {
    bcr_reduce_iso(m, stride, cid, D, b, Za, Zb, zb, Dn, En, bn);
}

// last level (one node): x = D^-1 b
__global__ void k_bcr_root(const double* D, const double* b, double* x, int64_t stride) {
    __shared__ double L[15 * 16];
    const int lane = threadIdx.x;
    for (int k = lane; k < 225; k += 32) { const int r = k % 15, c = k / 15; if (r >= c) L[r * 16 + c] = D[k]; }
    __syncwarp();
    warp_chol15(L, lane);
    double y[15];
#pragma unroll
    for (int r = 0; r < 15; r++) y[r] = b[r];
    fwd15(L, y);                                                   // every lane redundantly (15 x 15 / 2 fma)
    double r = 0.0;
#pragma unroll
    for (int q = 0; q < 15; q++) if (lane == q) r = y[q];
    const double xv = warp_bwd15(L, r, lane);
    if (lane < 15) x[lane] = xv;
    (void)stride;
}

// odd node i = 2t+1 of a level whose nodes sit at original indices i * stride:  Lc^T x_i = zb - Za x_{i-1} - Zb x_{i+1}
template <bool ISO>
CPI_DEV void bcr_backsub(int64_t m, int64_t stride, const int64_t* cid, const double* Lc, const double* Za, const double* Zb, const double* zb, double* x) {
    __shared__ double sL[4][15 * 16];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t t = (int64_t)blockIdx.x * 4 + wib;
    const int64_t i = 2 * t + 1;
    if (i >= m) return;
    double* L = sL[wib];
    for (int k = lane; k < 225; k += 32) { const int r = k % 15, c = k / 15; if (r >= c) L[r * 16 + c] = Lc[t * 225 + k]; }
    __syncwarp();
    const bool has_left = CPI_SAME(i - 1, i);
    const bool has_right = i + 1 < m && CPI_SAME(i + 1, i);
    double r = 0.0;
    if (lane < 15) {
        r = zb[t * 15 + lane];
        const double* xl = x + (i - 1) * stride * 15;
        const double* xr = x + (i + 1) * stride * 15;
#pragma unroll
        for (int q = 0; q < 15; q++) {
            if (has_left) r = fma(-Za[t * 225 + lane + 15 * q], xl[q], r);
            if (has_right) r = fma(-Zb[t * 225 + lane + 15 * q], xr[q], r);
        }
    }
    const double xv = warp_bwd15(L, r, lane);
    if (lane < 15) x[i * stride * 15 + lane] = xv;
}
#undef CPI_SAME
#undef SAME

__global__ void __launch_bounds__(128) k_bcr_backsub(int64_t m, int64_t stride, const double* Lc, const double* Za, const double* Zb, const double* zb, double* x) {
    bcr_backsub<false>(m, stride, nullptr, Lc, Za, Zb, zb, x);
}
__global__ void __launch_bounds__(128) k_bcr_backsub_iso(int64_t m, int64_t stride, const int64_t* cid, const double* Lc, const double* Za, const double* Zb,
                                                         const double* zb, double* x) {
    bcr_backsub<true>(m, stride, cid, Lc, Za, Zb, zb, x);
}

// the chain of every state, for the ISO kernels (grid-stride; a device-resident layout is searched per state)
__global__ void k_chain_ids(int64_t n_chains, const int64_t* offs, int64_t uniform, int64_t n_states, int64_t* cid) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n_states; k += (int64_t)gridDim.x * blockDim.x) {
        int64_t c;
        if (offs) {
            int64_t a = 0, b = n_chains - 1;
            while (a < b) { const int64_t mid = (a + b + 1) >> 1; if (offs[mid] <= k) a = mid; else b = mid - 1; }
            c = a;
        } else {
            c = k / uniform;
        }
        cid[k] = c;
    }
}

// ---- launchers ----------------------------------------------------------------------------------------------------------------------
cudaError_t whiten_launch(int rd, int64_t n, const double* records, const double* e, const double* H1, const double* H2, double* A1, double* A2, double* b, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    k_factor_whiten<<<(int)((n + 3) / 4), 128, 0, st>>>(n, rd, records, e, H1, H2, A1, A2, b);
    return cudaGetLastError();
}

cudaError_t chains_assemble_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, const double* G11, const double* G12, const double* G22,
                                   const double* g1, const double* g2, double lambda, int diagonal_damping, const double* prior_info,
                                   const double* prior_rhs, double* D, double* E, double* rhs, int sms, cudaStream_t st) {
    // uniform layout: one CTA per state (capped); device offsets: enough CTAs to fill the device, each striding over the states
    const int64_t ns = offs ? (int64_t)sms * 16 : n_chains * uniform;
    const int grid = (int)(ns < 2147483647 ? ns : 2147483647);
    k_chain_assemble<<<grid, 128, 0, st>>>(n_chains, offs, uniform, G11, G12, G22, g1, g2, lambda, diagonal_damping, prior_info, prior_rhs, D, E, rhs);
    return cudaGetLastError();
}

cudaError_t chains_assemble_lm_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, const double* G11, const double* G12, const double* G22,
                                      const double* g1, const double* g2, const double* lams, int diagonal_damping, const double* prior_info,
                                      const double* prior_rhs, double* D, double* E, double* rhs, double* damp, int sms, cudaStream_t st) {
    const int64_t ns = offs ? (int64_t)sms * 16 : n_chains * uniform;
    const int grid = (int)(ns < 2147483647 ? ns : 2147483647);
    k_chain_assemble_lm<<<grid, 128, 0, st>>>(n_chains, offs, uniform, G11, G12, G22, g1, g2, lams, diagonal_damping, prior_info, prior_rhs, D, E, rhs, damp);
    return cudaGetLastError();
}

// workspace layout: for every level l >= 1 the reduced system (D, E, b), for every level l >= 0 the eliminated nodes (Lc, Za, Zb, zb)
static int64_t bcr_doubles(int64_t m) {
    int64_t tot = 0;
    while (m > 1) {
        const int64_t odd = m / 2, even = (m + 1) / 2;
        tot += odd * (3 * 225 + 15);            // Lc, Za, Zb, zb of this level's odd nodes
        tot += even * (2 * 225 + 15);           // D, E, b of the next level
        m = even;
    }
    return tot + 16;
}
int64_t chain_solve_workspace_bytes(int64_t n_states) { return bcr_doubles(n_states) * 8; }
// the isolated solve: the same, followed by the chain id of every state
int64_t chains_solve_workspace_bytes(int64_t n_states) { return bcr_doubles(n_states) * 8 + n_states * 8; }

cudaError_t chains_solve_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, int64_t n_states, const double* D, const double* E, const double* b,
                                double* x, double* ws, int sms, cudaStream_t st, int* launches) {
    int64_t* cid = reinterpret_cast<int64_t*>(ws + bcr_doubles(n_states));
    const int64_t blocks = (n_states + 255) / 256, cap = (int64_t)sms * 8;
    k_chain_ids<<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>(n_chains, offs, uniform, n_states, cid);
    const cudaError_t e = chain_solve_launch(n_states, D, E, b, x, ws, st, launches, cid);
    if (launches) *launches += 1;
    return e;
}

cudaError_t chain_solve_launch(int64_t n_states, const double* D, const double* E, const double* b, double* x, double* ws, cudaStream_t st, int* launches,
                               const int64_t* cid) {
    struct Level { int64_t m; const double *D, *E, *b; double *Lc, *Za, *Zb, *zb; };
    Level lv[64];
    int nl = 0;
    int64_t m = n_states;
    const double *cD = D, *cE = E, *cb = b;
    double* p = ws;
    int nk = 0;
    while (m > 1) {
        const int64_t odd = m / 2, even = (m + 1) / 2;
        Level& L = lv[nl++];
        L.m = m; L.D = cD; L.E = cE; L.b = cb;
        L.Lc = p; p += odd * 225; L.Za = p; p += odd * 225; L.Zb = p; p += odd * 225; L.zb = p; p += odd * 15;
        double* nD = p; p += even * 225; double* nE = p; p += even * 225; double* nb = p; p += even * 15;
        const int64_t stride = (int64_t)1 << (nl - 1);              // level nl - 1: node i is original state i * 2^(nl-1)
        if (cid) {
            k_bcr_eliminate_iso<<<(int)((odd + 3) / 4), 128, 0, st>>>(m, stride, cid, cD, cE, cb, L.Lc, L.Za, L.Zb, L.zb);
            k_bcr_reduce_iso<<<(int)((even + 3) / 4), 128, 0, st>>>(m, stride, cid, cD, cb, L.Za, L.Zb, L.zb, nD, nE, nb);
        } else {
            k_bcr_eliminate<<<(int)((odd + 3) / 4), 128, 0, st>>>(m, cD, cE, cb, L.Lc, L.Za, L.Zb, L.zb);
            k_bcr_reduce<<<(int)((even + 3) / 4), 128, 0, st>>>(m, cD, cb, L.Za, L.Zb, L.zb, nD, nE, nb);
        }
        nk += 2;
        cD = nD; cE = nE; cb = nb; m = even;
    }
    k_bcr_root<<<1, 32, 0, st>>>(cD, cb, x, 1);
    nk++;
    int64_t stride = (int64_t)1 << nl;
    for (int l = nl - 1; l >= 0; l--) {
        stride >>= 1;
        const int64_t odd = lv[l].m / 2;
        if (cid) k_bcr_backsub_iso<<<(int)((odd + 3) / 4), 128, 0, st>>>(lv[l].m, stride, cid, lv[l].Lc, lv[l].Za, lv[l].Zb, lv[l].zb, x);
        else k_bcr_backsub<<<(int)((odd + 3) / 4), 128, 0, st>>>(lv[l].m, stride, lv[l].Lc, lv[l].Za, lv[l].Zb, lv[l].zb, x);
        nk++;
    }
    if (launches) *launches = nk;
    return cudaGetLastError();
}

}  // namespace cpi
