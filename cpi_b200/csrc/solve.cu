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
// Level with m nodes: row i reads  E[i-1]^T x_{i-1} + D[i] x_i + E[i] x_{i+1} = b[i].  Node i of the level sits at original state
// i * stride, and cid[] holds each original state's chain.  The coupling of two nodes is used only when both share a chain: otherwise
// it is not loaded, not multiplied, and written as exact 0, so a NaN stays inside its chain.
#define SAME(p, q) (cid[(p) * stride] == cid[(q) * stride])

// Odd node i = 2t+1:  D_i = Lc Lc^T,  Za = Lc^-1 E[i-1]^T,  Zb = Lc^-1 E[i] (if i+1 < m),  zb = Lc^-1 b_i      (kept for the back-substitution)
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
    const bool has_left = SAME(i - 1, i);
    const bool has_right = i + 1 < m && SAME(i + 1, i);
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
        if ((lane < 15 && !has_left) || (lane >= 15 && lane < 30 && !has_right)) {
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

__global__ void __launch_bounds__(128) k_bcr_eliminate_iso(int64_t m, int64_t stride, const int64_t* cid, const double* D, const double* E, const double* b,
                                                           double* Lc, double* Za, double* Zb, double* zb) {
    bcr_eliminate(m, stride, cid, D, E, b, Lc, Za, Zb, zb);
}
__global__ void __launch_bounds__(128) k_bcr_reduce_iso(int64_t m, int64_t stride, const int64_t* cid, const double* D, const double* b, const double* Za,
                                                        const double* Zb, const double* zb, double* Dn, double* En, double* bn) {
    bcr_reduce_iso(m, stride, cid, D, b, Za, Zb, zb, Dn, En, bn);
}

// last level (one node): x = D^-1 b
__global__ void k_bcr_root(const double* D, const double* b, double* x) {
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
}

// odd node i = 2t+1 of a level whose nodes sit at original indices i * stride:  Lc^T x_i = zb - Za x_{i-1} - Zb x_{i+1}
CPI_DEV void bcr_backsub(int64_t m, int64_t stride, const int64_t* cid, const double* Lc, const double* Za, const double* Zb, const double* zb, double* x) {
    __shared__ double sL[4][15 * 16];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t t = (int64_t)blockIdx.x * 4 + wib;
    const int64_t i = 2 * t + 1;
    if (i >= m) return;
    double* L = sL[wib];
    for (int k = lane; k < 225; k += 32) { const int r = k % 15, c = k / 15; if (r >= c) L[r * 16 + c] = Lc[t * 225 + k]; }
    __syncwarp();
    const bool has_left = SAME(i - 1, i);
    const bool has_right = i + 1 < m && SAME(i + 1, i);
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
#undef SAME

__global__ void __launch_bounds__(128) k_bcr_backsub_iso(int64_t m, int64_t stride, const int64_t* cid, const double* Lc, const double* Za, const double* Zb,
                                                         const double* zb, double* x) {
    bcr_backsub(m, stride, cid, Lc, Za, Zb, zb, x);
}

// the chain of every state, for the level kernels (grid-stride; a device-resident layout is searched per state)
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

// ---- selected inversion: the block-tridiagonal part of the inverse (cpi_imu_chains_marginals) -----------------------------------------
// Level l+1's system is the Schur complement of level l's on its even nodes, so its inverse is the full inverse on the states level l+1
// keeps.  Top-down over the levels of the forward phase, odd node i = 2t+1 of level l (nodes at original states i * stride), whose
// neighbours i-1, i+1 are nodes t, t+1 of level l+1 with known blocks (diagonal ones in cov at their original state, Sigma_{i-1,i+1} in
// Nin[t]):
//   Sigma_{i,i-1} = -Lc^-T (Za Sigma_{i-1,i-1} + Zb Sigma_{i+1,i-1}),   Sigma_{i,i+1} = -Lc^-T (Za Sigma_{i-1,i+1} + Zb Sigma_{i+1,i+1}),
//   Sigma_{i,i}   =  Lc^-T (Lc^-1 - Za Sigma_{i,i-1}^T - Zb Sigma_{i,i+1}^T)
// Isolated as the solve: a neighbour of another chain is not loaded and not multiplied, and its coupling is written as exact 0.

// the root (one node): cov = D^-1, the lower triangle of column `lane` by lane `lane`, mirrored
__global__ void k_bcr_selinv_root(const double* D, double* cov) {
    __shared__ double L[15 * 16];
    const int lane = threadIdx.x;
    for (int k = lane; k < 225; k += 32) { const int r = k % 15, c = k / 15; if (r >= c) L[r * 16 + c] = D[k]; }
    __syncwarp();
    warp_chol15(L, lane);
    if (lane < 15) {
        double y[15];
#pragma unroll
        for (int r = 0; r < 15; r++) y[r] = (r == lane) ? 1.0 : 0.0;
        fwd15(L, y);
        __syncwarp(0x7fffu);                                       // L is reloaded for the backward pass: 120 entries held live would spill
        bwd15(L, y);
#pragma unroll
        for (int r = 0; r < 15; r++) if (r >= lane) { cov[r + 15 * lane] = y[r]; cov[lane + 15 * r] = y[r]; }
    }
}

// One warp per odd node of a level.  Writes Sigma_ii to cov[i * stride] and the level's neighbour blocks Sigma_{k,k+1} of the pairs
// (i-1, i) and (i, i+1): to Nout slot k (levels >= 1; exact 0 across chains) or, with Nout NULL (level 0), to cross slot k - cid[k]
// (factor order; pairs across chains have no slot; cross may be NULL).  Nin is read only for two neighbours of i's chain.
__global__ void __launch_bounds__(128) k_bcr_selinv_iso(int64_t m, int64_t stride, const int64_t* cid, const double* Lc, const double* Za,
                                                        const double* Zb, const double* Nin, double* cov, double* Nout, double* cross) {
    __shared__ double sL[4][15 * 16];
    __shared__ double sM[4][5][225];           // [warp][Za | Zb | Sigma_{i-1,i-1} -> Sigma_{i,i-1} | Sigma_{i-1,i+1} | Sigma_{i+1,i+1} -> Sigma_{i,i+1}]
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t t = (int64_t)blockIdx.x * 4 + wib;
    const int64_t i = 2 * t + 1;
    if (i >= m) return;
    const int64_t ci = cid[i * stride];
    const bool has_left = cid[(i - 1) * stride] == ci;
    const bool has_right = i + 1 < m && cid[(i + 1) * stride] == ci;
    double *L = sL[wib], *A = sM[wib][0], *B = sM[wib][1], *XL = sM[wib][2], *N = sM[wib][3], *XR = sM[wib][4];
    for (int k = lane; k < 225; k += 32) {
        const int r = k % 15, c = k / 15;
        if (r >= c) L[r * 16 + c] = Lc[t * 225 + k];
        if (has_left) { A[k] = Za[t * 225 + k]; XL[k] = cov[(i - 1) * stride * 225 + k]; }
        if (has_right) { B[k] = Zb[t * 225 + k]; XR[k] = cov[(i + 1) * stride * 225 + k]; }
        if (has_left && has_right) N[k] = Nin[t * 225 + k];
    }
    __syncwarp();
    // lanes 0..14: column c of Sigma_{i,i-1}; lanes 15..29: column c of Sigma_{i,i+1}  (Sigma_{i+1,i-1} = N^T)
    const int c = lane % 15;
    const bool right = lane >= 15;
    const bool active = lane < 30 && (right ? has_right : has_left);
    double y[15];
#pragma unroll
    for (int r = 0; r < 15; r++) y[r] = 0.0;
    if (active) {
        if (has_left) {
#pragma unroll
            for (int q = 0; q < 15; q++) {
                const double v = right ? N[q + 15 * c] : XL[q + 15 * c];
#pragma unroll
                for (int r = 0; r < 15; r++) y[r] = fma(A[r + 15 * q], v, y[r]);
            }
        }
        if (has_right) {
#pragma unroll
            for (int q = 0; q < 15; q++) {
                const double v = right ? XR[q + 15 * c] : N[c + 15 * q];
#pragma unroll
                for (int r = 0; r < 15; r++) y[r] = fma(B[r + 15 * q], v, y[r]);
            }
        }
        bwd15(L, y);
    }
    __syncwarp();
    if (active) {
        double* X = right ? XR : XL;
#pragma unroll
        for (int r = 0; r < 15; r++) X[r + 15 * c] = -y[r];
    }
    __syncwarp();
    // the level's neighbour blocks: Sigma_{i-1,i} = Sigma_{i,i-1}^T in slot i-1, Sigma_{i,i+1} in slot i
    for (int k = lane; k < 225; k += 32) {
        const int r = k % 15, cc = k / 15;
        if (Nout) {
            Nout[(i - 1) * 225 + k] = has_left ? XL[cc + 15 * r] : 0.0;
            if (i + 1 < m) Nout[i * 225 + k] = has_right ? XR[k] : 0.0;
        } else if (cross) {
            if (has_left) cross[(i - 1 - ci) * 225 + k] = XL[cc + 15 * r];
            if (has_right) cross[(i - ci) * 225 + k] = XR[k];
        }
    }
    // Sigma_ii: column `lane` of Lc^-T (Lc^-1 - Za Sigma_{i,i-1}^T - Zb Sigma_{i,i+1}^T), its lower triangle mirrored
    if (lane < 15) {
#pragma unroll
        for (int r = 0; r < 15; r++) y[r] = (r == lane) ? 1.0 : 0.0;
        fwd15(L, y);
        __syncwarp(0x7fffu);                                       // as in k_bcr_selinv_root
        if (has_left) {
#pragma unroll
            for (int q = 0; q < 15; q++) {
                const double v = XL[lane + 15 * q];
#pragma unroll
                for (int r = 0; r < 15; r++) y[r] = fma(-A[r + 15 * q], v, y[r]);
            }
        }
        if (has_right) {
#pragma unroll
            for (int q = 0; q < 15; q++) {
                const double v = XR[lane + 15 * q];
#pragma unroll
                for (int r = 0; r < 15; r++) y[r] = fma(-B[r + 15 * q], v, y[r]);
            }
        }
        bwd15(L, y);
        double* S = cov + i * stride * 225;
#pragma unroll
        for (int r = 0; r < 15; r++) if (r >= lane) { S[r + 15 * lane] = y[r]; S[lane + 15 * r] = y[r]; }
    }
}

// ---- pair covariances: any block Sigma_ij of the inverse (cpi_imu_chains_pair_covariance) --------------------------------------------
// Odd node x of level l is, given the level's other nodes, x = K- x_{x-1} + K+ x_{x+1} + w with K- = -Lc^-T Za, K+ = -Lc^-T Zb and
// Cov(w) = Lc^-T Lc^-1 (a neighbour of another chain has no term).  Sigma_ij = R + sum_{a in A, b in B} C_a Sigma_ab D_b^T starts at
// A = {i}, B = {j}, C = D = I, R = 0; each level replaces every node of A and B it eliminates by its neighbours (C_nbr += C_x K-/+),
// adding C_x Lc^-T Lc^-1 D_x^T to R first where x is in both; at the root R += C_0 Sigma_root D_0^T.  A holds the level's nodes that
// bracket i, so at most two, level-local a0 and a0 + 1 with a0 = i >> l (likewise B); exactly one of them is odd.  A chain other than
// chain 0 never reaches the root: its brackets empty out at some level, and the walk stops there.
struct PairWalk { int nl; int64_t m[64]; const double *Lc[64], *Za[64], *Zb[64]; };

// One warp per pair, grid-stride over the pairs.  Lanes 0..14 hold rows of side A's matrices (i), lanes 15..29 those of side B (j).
__global__ void __launch_bounds__(64) k_bcr_pair_cov(PairWalk w, int64_t n_states, const int64_t* cid, const double* root, int64_t n_pairs,
                                                     const int64_t* pi, const int64_t* pj, double* out) {
    __shared__ double sL[2][2][15 * 16];       // [warp][side] Lc of the side's eliminated node
    __shared__ double sZ[2][2][2][225];        // [warp][side][Za | Zb] (column-major), Sigma_root in [warp][0][0] at the end
    __shared__ double sC[2][2][2][225];        // [warp][side][slot] C (side A) or D (side B) of bracket node a0 + slot, row-major
    __shared__ double sR[2][225];              // [warp] R, row-major
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int s = lane >= 15, r = lane - 15 * s; // lane < 30: side s, row r
    double* R = sR[wib];
    for (int64_t p = (int64_t)blockIdx.x * 2 + wib; p < n_pairs; p += (int64_t)gridDim.x * 2) {
        const int64_t i = pi[p], j = pj[p];
        double* o = out + p * 225;
        if (i < 0 || i >= n_states || j < 0 || j >= n_states || cid[i] != cid[j]) {
            const double v = (i < 0 || i >= n_states || j < 0 || j >= n_states) ? __longlong_as_double(0x7ff8000000000000ll) : 0.0;
            for (int k = lane; k < 225; k += 32) o[k] = v;
            continue;
        }
        int64_t a0[2] = {i, j};
        bool live[2][2] = {{true, false}, {true, false}};
        for (int k = lane; k < 225; k += 32) {
            const double e = (k % 16 == 0) ? 1.0 : 0.0;            // k = r * 15 + c is diagonal when k % 16 == 0
            sC[wib][0][0][k] = e; sC[wib][1][0][k] = e; R[k] = 0.0;
        }
        int l = 0;
        for (; l < w.nl; l++) {
            if (!(live[0][0] || live[0][1]) || !(live[1][0] || live[1][1])) break;
            const int64_t m = w.m[l], stride = (int64_t)1 << l;
            int os[2];
            int64_t x[2];
            bool ex[2], hl[2], hr[2];
#pragma unroll
            for (int q = 0; q < 2; q++) {
                os[q] = (a0[q] & 1) ? 0 : 1;                          // the slot holding the level's odd bracket node
                x[q] = a0[q] + os[q];
                ex[q] = live[q][os[q]];
                const int64_t cx = ex[q] ? cid[x[q] * stride] : 0;
                hl[q] = ex[q] && cid[(x[q] - 1) * stride] == cx;
                hr[q] = ex[q] && x[q] + 1 < m && cid[(x[q] + 1) * stride] == cx;
            }
            __syncwarp();
#pragma unroll
            for (int q = 0; q < 2; q++) {
                if (!ex[q]) continue;
                const int64_t t = x[q] >> 1;
                for (int k = lane; k < 225; k += 32) {
                    const int rr = k % 15, cc = k / 15;
                    if (rr >= cc) sL[wib][q][rr * 16 + cc] = w.Lc[l][t * 225 + k];
                    if (hl[q]) sZ[wib][q][0][k] = w.Za[l][t * 225 + k];
                    if (hr[q]) sZ[wib][q][1][k] = w.Zb[l][t * 225 + k];
                }
            }
            __syncwarp();
            // row r of Y = C_x Lc^-T (Lc Y^T = C_x^T), kept in place of C_x for the shared-node term
            const int os_s = s ? os[1] : os[0];                        // this lane's side, selected without a local-memory index
            const bool act = lane < 30 && (s ? ex[1] : ex[0]);
            const bool hl_s = s ? hl[1] : hl[0], hr_s = s ? hr[1] : hr[0];
            const bool live_s[2] = {s ? live[1][0] : live[0][0], s ? live[1][1] : live[0][1]};
            double* Cx = sC[wib][s][os_s];
            double y[15];
            if (act) {
#pragma unroll
                for (int q = 0; q < 15; q++) y[q] = Cx[r * 15 + q];
                fwd15(sL[wib][s], y);
#pragma unroll
                for (int q = 0; q < 15; q++) Cx[r * 15 + q] = y[q];
            }
            __syncwarp();
            if (ex[0] && ex[1] && x[0] == x[1]) {                  // x in A and B: R += Y_A Y_B^T
                const double *YA = sC[wib][0][os[0]], *YB = sC[wib][1][os[1]];
                for (int k = lane; k < 225; k += 32) {
                    const int rr = k / 15, cc = k % 15;
                    double v = R[k];
#pragma unroll
                    for (int q = 0; q < 15; q++) v = fma(YA[rr * 15 + q], YB[cc * 15 + q], v);
                    R[k] = v;
                }
            }
            __syncwarp();
            // the neighbours: slot 0 (node a0 or a0 - 1) takes -Y Za, slot 1 (node a0 + 1 or a0 + 2) takes -Y Zb; the slot that held x is
            // replaced, the other accumulated into
            if (act) {
#pragma unroll
                for (int q = 0; q < 2; q++) {
                    if (!(q ? hr_s : hl_s)) continue;
                    const double* Z = sZ[wib][s][q];
                    double* dst = sC[wib][s][q] + r * 15;
                    const bool acc = q != os_s && live_s[q];
#pragma unroll
                    for (int c = 0; c < 15; c++) {
                        double v = acc ? dst[c] : 0.0;
#pragma unroll
                        for (int k = 0; k < 15; k++) v = fma(-y[k], Z[k + 15 * c], v);
                        dst[c] = v;
                    }
                }
            }
#pragma unroll
            for (int q = 0; q < 2; q++) {
                if (ex[q]) {
                    live[q][0] = os[q] == 0 ? hl[q] : (live[q][0] || hl[q]);
                    live[q][1] = os[q] == 1 ? hr[q] : (live[q][1] || hr[q]);
                }
                a0[q] >>= 1;
            }
            __syncwarp();
        }
        if (l == w.nl && live[0][0] && live[1][0]) {               // both brackets reached the root (node 0): R += C_0 Sigma_root D_0^T
            double* S = sZ[wib][0][0];
            for (int k = lane; k < 225; k += 32) S[k] = root[k];
            __syncwarp();
            if (lane < 15) {
                const double *CA = sC[wib][0][0], *CB = sC[wib][1][0];
                double t[15];
#pragma unroll
                for (int c = 0; c < 15; c++) {
                    double v = 0.0;
#pragma unroll
                    for (int q = 0; q < 15; q++) v = fma(CA[lane * 15 + q], S[q + 15 * c], v);
                    t[c] = v;
                }
#pragma unroll
                for (int c = 0; c < 15; c++) {
                    double v = R[lane * 15 + c];
#pragma unroll
                    for (int q = 0; q < 15; q++) v = fma(t[q], CB[c * 15 + q], v);
                    R[lane * 15 + c] = v;
                }
            }
        }
        __syncwarp();
        for (int k = lane; k < 225; k += 32) {                      // column-major; Sigma_ii as its lower triangle mirrored
            const int rr = k % 15, cc = k / 15;
            o[k] = (i == j && rr < cc) ? R[rr + 15 * cc] : R[rr * 15 + cc];
        }
        __syncwarp();
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

// The workspace of the block cyclic reduction, level by level: level l has m nodes (node i is original state i * 2^l); the workspace
// holds, for l = 0, 1, ..., the eliminated odd nodes' Lc, Za, Zb, zb, then the next level's reduced system D, E, b.  The last level
// (one node) is the root.  Offsets in doubles.
struct BcrLevel { int64_t m, Lc, Za, Zb, zb, D, E, b; };
// fills lv[0 .. nl) and returns nl (at most 63: m < 2^63); *end: the doubles the levels take
static int bcr_levels(int64_t m, BcrLevel* lv, int64_t* end) {
    int nl = 0;
    int64_t p = 0;
    while (m > 1) {
        const int64_t odd = m / 2, even = (m + 1) / 2;
        BcrLevel& L = lv[nl++];
        L.m = m;
        L.Lc = p; p += odd * 225; L.Za = p; p += odd * 225; L.Zb = p; p += odd * 225; L.zb = p; p += odd * 15;
        L.D = p; p += even * 225; L.E = p; p += even * 225; L.b = p; p += even * 15;
        m = even;
    }
    *end = p;
    return nl;
}
static int64_t bcr_doubles(int64_t m) {
    BcrLevel lv[64];
    int64_t end;
    bcr_levels(m, lv, &end);
    return end + 16;
}
// The forward phase (elimination and reduction of every level) on the level table; the root's system is left at level nl's D, b.
static void bcr_forward(const BcrLevel* lv, int nl, const double* D, const double* E, const double* b, double* ws, const int64_t* cid,
                        cudaStream_t st) {
    for (int l = 0; l < nl; l++) {
        const BcrLevel& L = lv[l];
        const double *cD = l ? ws + lv[l - 1].D : D, *cE = l ? ws + lv[l - 1].E : E, *cb = l ? ws + lv[l - 1].b : b;
        const int64_t odd = L.m / 2, even = (L.m + 1) / 2;
        const int64_t stride = (int64_t)1 << l;
        k_bcr_eliminate_iso<<<(int)((odd + 3) / 4), 128, 0, st>>>(L.m, stride, cid, cD, cE, cb, ws + L.Lc, ws + L.Za, ws + L.Zb, ws + L.zb);
        k_bcr_reduce_iso<<<(int)((even + 3) / 4), 128, 0, st>>>(L.m, stride, cid, cD, cb, ws + L.Za, ws + L.Zb, ws + L.zb, ws + L.D, ws + L.E, ws + L.b);
    }
}
// What follows the levels (offsets in doubles): the solve's chain id of every state (int64), then the selected inversion's
// zero right-hand side [n_states, 15] for the forward phase and the neighbour blocks Sigma_{k,k+1} of every level l >= 1 with two nodes
// or more (m_l - 1 blocks each, level order), then the pair covariances' Sigma_root (225).  solve_end / selinv_end / pair_end: the doubles
// the solve / the selected inversion / the pair covariances take.
struct BcrTail { int64_t cid, solve_end, b0, nbr[64], selinv_end, root, pair_end; };
static BcrTail bcr_tail(int64_t n_states, const BcrLevel* lv, int nl) {
    BcrTail t;
    t.cid = bcr_doubles(n_states);
    t.solve_end = t.b0 = t.cid + n_states;
    int64_t p = t.b0 + n_states * 15;
    for (int l = 0; l < 64; l++) t.nbr[l] = -1;
    for (int l = 1; l < nl; l++) { t.nbr[l] = p; p += (lv[l].m - 1) * 225; }
    t.selinv_end = t.root = p;
    t.pair_end = t.root + 225;
    return t;
}
static BcrTail bcr_tail(int64_t n_states) {
    BcrLevel lv[64];
    int64_t end;
    const int nl = bcr_levels(n_states, lv, &end);
    return bcr_tail(n_states, lv, nl);
}

// the solve's workspace: the levels, then the chain id of every state
int64_t chains_solve_workspace_bytes(int64_t n_states) { return bcr_tail(n_states).solve_end * 8; }

// The chain ids, the forward phase, the root and the back-substitution levels.  One state has no level: nothing reads the chain ids
// and the workspace is not touched (it may be NULL).
cudaError_t chains_solve_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, int64_t n_states, const double* D, const double* E, const double* b,
                                double* x, double* ws, int sms, cudaStream_t st, int* launches) {
    BcrLevel lv[64];
    int64_t end;
    const int nl = bcr_levels(n_states, lv, &end);
    int64_t* cid = nullptr;
    if (n_states > 1) {
        cid = reinterpret_cast<int64_t*>(ws + bcr_tail(n_states, lv, nl).cid);
        const int64_t blocks = (n_states + 255) / 256, cap = (int64_t)sms * 8;
        k_chain_ids<<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>(n_chains, offs, uniform, n_states, cid);
    }
    bcr_forward(lv, nl, D, E, b, ws, cid, st);
    k_bcr_root<<<1, 32, 0, st>>>(nl ? ws + lv[nl - 1].D : D, nl ? ws + lv[nl - 1].b : b, x);
    for (int l = nl - 1; l >= 0; l--) {
        const int64_t stride = (int64_t)1 << l, odd = lv[l].m / 2;
        k_bcr_backsub_iso<<<(int)((odd + 3) / 4), 128, 0, st>>>(lv[l].m, stride, cid, ws + lv[l].Lc, ws + lv[l].Za, ws + lv[l].Zb, ws + lv[l].zb, x);
    }
    if (launches) *launches = 3 * nl + 1 + (n_states > 1);
    return cudaGetLastError();
}

// the selected inversion's workspace: the levels, then the tail of bcr_tail
int64_t chains_marginals_workspace_bytes(int64_t n_states) { return bcr_tail(n_states).selinv_end * 8; }

cudaError_t chains_marginals_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, int64_t n_states, const double* D, const double* E,
                                    double* cov, double* cross, double* ws, int sms, cudaStream_t st, int* launches) {
    BcrLevel lv[64];
    int64_t end;
    const int nl = bcr_levels(n_states, lv, &end);
    const BcrTail tail = bcr_tail(n_states, lv, nl);
    int64_t* cid = reinterpret_cast<int64_t*>(ws + tail.cid);
    double* b0 = ws + tail.b0;
    double* nbr[65];                                                // level l's neighbour blocks (l >= 1; NULL: none)
    for (int l = 0; l < 65; l++) nbr[l] = l < 64 && tail.nbr[l] >= 0 ? ws + tail.nbr[l] : nullptr;
    cudaError_t e = cudaMemsetAsync(b0, 0, (size_t)n_states * 15 * 8, st);
    if (e != cudaSuccess) return e;
    const int64_t blocks = (n_states + 255) / 256, cap = (int64_t)sms * 8;
    k_chain_ids<<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>(n_chains, offs, uniform, n_states, cid);
    bcr_forward(lv, nl, D, E, b0, ws, cid, st);
    k_bcr_selinv_root<<<1, 32, 0, st>>>(nl ? ws + lv[nl - 1].D : D, cov);
    for (int l = nl - 1; l >= 0; l--) {
        const int64_t odd = lv[l].m / 2;
        k_bcr_selinv_iso<<<(int)((odd + 3) / 4), 128, 0, st>>>(lv[l].m, (int64_t)1 << l, cid, ws + lv[l].Lc, ws + lv[l].Za, ws + lv[l].Zb,
                                                               nbr[l + 1], cov, nbr[l], l ? nullptr : cross);
    }
    if (launches) *launches = 3 * nl + 2;
    return cudaGetLastError();
}

// the pair covariances' workspace: the selected inversion's, then Sigma_root
int64_t chains_pair_cov_workspace_bytes(int64_t n_states) { return bcr_tail(n_states).pair_end * 8; }

// The chain ids, the forward phase on a zero right-hand side (as chains_marginals_launch), Sigma_root, then one walk per pair.
cudaError_t chains_pair_cov_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, int64_t n_states, const double* D, const double* E,
                                   int64_t n_pairs, const int64_t* pi, const int64_t* pj, double* out, double* ws, int sms, cudaStream_t st,
                                   int* launches) {
    if (launches) *launches = 0;
    if (n_pairs == 0) return cudaSuccess;
    BcrLevel lv[64];
    int64_t end;
    const int nl = bcr_levels(n_states, lv, &end);
    const BcrTail tail = bcr_tail(n_states, lv, nl);
    int64_t* cid = reinterpret_cast<int64_t*>(ws + tail.cid);
    double* b0 = ws + tail.b0;
    cudaError_t e = cudaMemsetAsync(b0, 0, (size_t)n_states * 15 * 8, st);
    if (e != cudaSuccess) return e;
    const int64_t blocks = (n_states + 255) / 256, cap = (int64_t)sms * 8;
    k_chain_ids<<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>(n_chains, offs, uniform, n_states, cid);
    bcr_forward(lv, nl, D, E, b0, ws, cid, st);
    k_bcr_selinv_root<<<1, 32, 0, st>>>(nl ? ws + lv[nl - 1].D : D, ws + tail.root);
    PairWalk w;
    w.nl = nl;
    for (int l = 0; l < nl; l++) { w.m[l] = lv[l].m; w.Lc[l] = ws + lv[l].Lc; w.Za[l] = ws + lv[l].Za; w.Zb[l] = ws + lv[l].Zb; }
    // one pass of resident CTAs (five per SM on sm_90: 40 080 B of static shared memory each), striding over the pairs
    int per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_bcr_pair_cov, 64, 0);
    if (e != cudaSuccess) return e;
    const int64_t ctas = (n_pairs + 1) / 2, pcap = (int64_t)sms * (per_sm > 0 ? per_sm : 1);
    k_bcr_pair_cov<<<(int)(ctas < pcap ? ctas : pcap), 64, 0, st>>>(w, n_states, cid, ws + tail.root, n_pairs, pi, pj, out);
    if (launches) *launches = 2 * nl + 3;
    return cudaGetLastError();
}

}  // namespace cpi
