// K3 / K4: batched ImuFactorCPIv1::evaluateError (gtsam/ImuFactorCPIv1.cpp:37-208) and
// ImuFactorCPIv2::evaluateError (gtsam/ImuFactorCPIv2.cpp:38-212); plus the two tiny callers either side of the
// factor: GraphSolver::getpredictedstate_v1/_v2 (solvers/GraphSolver_IMU.cpp:263-307) and JPLNavState::retract
// (gtsam/JPLNavState.cpp:37-71).
//
// The factor kernel is OUTPUT-WRITE bound (4 496 B / 4 672 B of algorithmic traffic per factor, ~0.5 kflop): one lane
// computes one factor's residual and 3x3 blocks, deposits the dense 15 + 225 + 225 doubles into a shared-memory tile,
// and the whole CTA then streams the tile to HBM with fully coalesced 8-byte stores (the e / H1 / H2 arrays of the
// CTA's 32 consecutive factors are three contiguous ranges).
#include "cpi_common.cuh"
#include "cpi_kernels.h"
#include "factor_blocks.cuh"

namespace cpi {

// Factors per block and threads per block.  The compute phase is one lane per factor and latency-bound (~2 k dependent instructions), so
// what matters is how many CTAs an SM can hold while others stream out: 8 factors x 64 threads = 30 KB of tile at 168 registers ->
// 6 CTAs per SM (round 1: 16 x 128 threads at 255 registers -> 2 per SM).  625 CTAs for a 5k chain: all resident in one wave.
constexpr int FPB = 8;
constexpr int FTHREADS = 64;
// resident CTAs per SM the register allocation aims at: 6 (168 registers, ~400 B of spills) measured faster than 4 (255, none): 789 vs 671 M factors/s at 1M
constexpr int K3_MIN_BLOCKS = 6;
constexpr int FTILE = 15 + 225 + 225;   // doubles per factor in the staging tile


// write a row-major 3x3 (scaled) into a column-major 15x15 tile at block (r0, c0)
CPI_DEV void put33(double* H, int r0, int c0, const double* M, double s) {
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) H[(r0 + i) + 15 * (c0 + j)] = s * M[3 * i + j];
}
CPI_DEV void putI(double* H, int r0, int c0, double s) {
#pragma unroll
    for (int i = 0; i < 3; i++) H[(r0 + i) + 15 * (c0 + i)] = s;
}

template <int MODEL>
__global__ void __launch_bounds__(FTHREADS, K3_MIN_BLOCKS) k_factor_eval(const FactorParams p) {
    extern __shared__ double tile[];
    const int tid = threadIdx.x;
    const int64_t f0 = (int64_t)blockIdx.x * FPB;
    const int nf = (int)((p.n - f0) < FPB ? (p.n - f0) : FPB);
    const bool wantH1 = p.H1 != nullptr, wantH2 = p.H2 != nullptr;

    // Three sub-tiles laid out exactly like the CTA's three contiguous output ranges (e: FPB x 15, H1 / H2: FPB x 225), so that the
    // stream-out is a straight 16-byte-vector copy.  Zero them cooperatively (most of H1/H2 is structural zero).
    double* tE = tile;
    double* tH1 = tile + FPB * 15;
    double* tH2 = tH1 + FPB * 225;
    {
        double2* t2 = reinterpret_cast<double2*>(tile);
        for (int k = tid; k < FPB * FTILE / 2; k += blockDim.x) t2[k] = make_double2(0.0, 0.0);
    }
    __syncthreads();

    if (tid < nf) {
        const int64_t f = f0 + tid;
        constexpr int RD = (MODEL == 1) ? CPI_REC_V1_DOUBLES : CPI_REC_V2_DOUBLES;
        const int64_t ia = p.idx_i ? p.idx_i[f] : f, ib = p.idx_j ? p.idx_j[f] : f + 1;
        const double* xi = p.states + ia * CPI_STATE_DOUBLES;
        const double* xj = p.states + ib * CPI_STATE_DOUBLES;
        const double* r = p.records + f * (int64_t)RD;
        const double* l = p.lin + f * CPI_LIN_DOUBLES;
        double* E = tE + tid * 15;
        double* H1 = tH1 + tid * 225;
        double* H2 = tH2 + tid * 225;

        double qK[4], qK1[4], bgK[3], bgK1[3], vK[3], vK1[3], baK[3], baK1[3], pK[3], pK1[3];
#pragma unroll
        for (int k = 0; k < 4; k++) { qK[k] = __ldg(xi + k); qK1[k] = __ldg(xj + k); }
#pragma unroll
        for (int k = 0; k < 3; k++) {
            bgK[k] = __ldg(xi + 4 + k); vK[k] = __ldg(xi + 7 + k); baK[k] = __ldg(xi + 10 + k); pK[k] = __ldg(xi + 13 + k);
            bgK1[k] = __ldg(xj + 4 + k); vK1[k] = __ldg(xj + 7 + k); baK1[k] = __ldg(xj + 10 + k); pK1[k] = __ldg(xj + 13 + k);
        }
        const double bg_lin[3] = {__ldg(l), __ldg(l + 1), __ldg(l + 2)}, ba_lin[3] = {__ldg(l + 3), __ldg(l + 4), __ldg(l + 5)};
        const double q_lin[4] = {__ldg(l + 6), __ldg(l + 7), __ldg(l + 8), __ldg(l + 9)};
        const double grav[3] = {__ldg(l + 10), __ldg(l + 11), __ldg(l + 12)};
        const double q_meas[4] = {__ldg(r), __ldg(r + 1), __ldg(r + 2), __ldg(r + 3)};
        const double alpha[3] = {__ldg(r + CPI_REC_ALPHA), __ldg(r + CPI_REC_ALPHA + 1), __ldg(r + CPI_REC_ALPHA + 2)};
        const double beta[3] = {__ldg(r + CPI_REC_BETA), __ldg(r + CPI_REC_BETA + 1), __ldg(r + CPI_REC_BETA + 2)};
        const double dT = __ldg(r + CPI_REC_DT);
        double Jq[9], Jal[9], Jbe[9], Hal[9], Hbe[9], Oal[9], Obe[9];
        ldrec33(r + CPI_REC_JQ, Jq); ldrec33(r + CPI_REC_JA, Jal); ldrec33(r + CPI_REC_JB, Jbe);
        ldrec33(r + CPI_REC_HA, Hal); ldrec33(r + CPI_REC_HB, Hbe);
        if (MODEL == 2) { ldrec33(r + CPI_REC_OA, Oal); ldrec33(r + CPI_REC_OB, Obe); }

        const double dbg[3] = {bgK[0] - bg_lin[0], bgK[1] - bg_lin[1], bgK[2] - bg_lin[2]};
        const double dba[3] = {baK[0] - ba_lin[0], baK[1] - ba_lin[1], baK[2] - ba_lin[2]};

        // q_b = rot_2_quat(Exp(-J_q (bg_K - bg_lin)))                                   :57-58
        double t3[3], ExpB[9], q_b[4], qi[4], q_n[4], q_rm[4], q_r[4], q_m[4];
        mv33(Jq, dbg, t3);
        t3[0] = -t3[0]; t3[1] = -t3[1]; t3[2] = -t3[2];
        Exp_so3(t3, ExpB);
        rot_2_quat(ExpB, q_b);
        qi[0] = -qK[0]; qi[1] = -qK[1]; qi[2] = -qK[2]; qi[3] = qK[3];
        quat_multiply(qK1, qi, q_n);                                                     // :61
        qi[0] = -q_meas[0]; qi[1] = -q_meas[1]; qi[2] = -q_meas[2]; qi[3] = q_meas[3];
        quat_multiply(q_n, qi, q_rm);                                                    // :62
        quat_multiply(q_rm, q_b, q_r);                                                   // :63
        qi[0] = -q_b[0]; qi[1] = -q_b[1]; qi[2] = -q_b[2]; qi[3] = q_b[3];
        quat_multiply(qi, q_meas, q_m);                                                  // :64

        double q_kR[4] = {0, 0, 0, 1}, dthk[3] = {0, 0, 0};
        if (MODEL == 2) {                                                                // v2 :68-69
            qi[0] = -q_lin[0]; qi[1] = -q_lin[1]; qi[2] = -q_lin[2]; qi[3] = q_lin[3];
            quat_multiply(qK, qi, q_kR);
            dthk[0] = 2.0 * q_kR[0]; dthk[1] = 2.0 * q_kR[1]; dthk[2] = 2.0 * q_kR[2];
        }

        double Rk[9], pa[3], pb[3], Rpa[3], Rpb[3], ah[3], bh[3], u[3], w[3];
        quat_2_Rot(qK, Rk);
#pragma unroll
        for (int k = 0; k < 3; k++) {
            if (MODEL == 1) {                                                            // v1 :70, :72
                pa[k] = pK1[k] - pK[k] - vK[k] * dT + 0.5 * grav[k] * (dT * dT);
                pb[k] = vK1[k] - vK[k] + grav[k] * dT;
            } else {                                                                     // v2 :72, :74
                pa[k] = pK1[k] - pK[k] - vK[k] * dT;
                pb[k] = vK1[k] - vK[k];
            }
        }
        mv33(Rk, pa, Rpa); mv33(Rk, pb, Rpb);
        mv33(Jal, dbg, u); mv33(Hal, dba, w);
#pragma unroll
        for (int k = 0; k < 3; k++) ah[k] = Rpa[k] - u[k] - w[k];
        mv33(Jbe, dbg, u); mv33(Hbe, dba, w);
#pragma unroll
        for (int k = 0; k < 3; k++) bh[k] = Rpb[k] - u[k] - w[k];
        if (MODEL == 2) {
            mv33(Oal, dthk, u); mv33(Obe, dthk, w);
#pragma unroll
            for (int k = 0; k < 3; k++) { ah[k] -= u[k]; bh[k] -= w[k]; }
        }
#pragma unroll
        for (int k = 0; k < 3; k++) {                                                    // :84-88
            E[k] = 2.0 * q_r[k];
            E[3 + k] = bgK1[k] - bgK[k];
            E[6 + k] = bh[k] - beta[k];
            E[9 + k] = baK1[k] - baK[k];
            E[12 + k] = ah[k] - alpha[k];
        }

        if (wantH1) {                                                                    // :98-154
            double A[9], Bm[9], AB[9], blk[9], sk[9];
            quat_mat(q_n, -1.0, A); quat_mat(q_m, -1.0, Bm); mul33(A, Bm, AB);
#pragma unroll
            for (int i = 0; i < 3; i++)
#pragma unroll
                for (int j = 0; j < 3; j++) blk[3 * i + j] = -(AB[3 * i + j] + q_n[i] * q_m[j]);
            put33(H1, 0, 0, blk, 1.0);                                                   // :109-111
            skew(Rpb, sk);
            if (MODEL == 2) { double qm[9], t[9]; quat_mat(q_kR, +1.0, qm); mul33(Obe, qm, t);
#pragma unroll
                for (int k = 0; k < 9; k++) sk[k] -= t[k]; }
            put33(H1, 6, 0, sk, 1.0);                                                    // :113 / v2 :115-116
            skew(Rpa, sk);
            if (MODEL == 2) { double qm[9], t[9]; quat_mat(q_kR, +1.0, qm); mul33(Oal, qm, t);
#pragma unroll
                for (int k = 0; k < 9; k++) sk[k] -= t[k]; }
            put33(H1, 12, 0, sk, 1.0);                                                   // :115 / v2 :118-119
            quat_mat(q_rm, -1.0, A); mul33(A, Jq, blk);
            put33(H1, 0, 3, blk, 1.0);                                                   // :119
            putI(H1, 3, 3, -1.0);                                                        // :121
            put33(H1, 6, 3, Jbe, -1.0);                                                  // :123
            put33(H1, 12, 3, Jal, -1.0);                                                 // :125
            put33(H1, 6, 6, Rk, -1.0);                                                   // :129
            put33(H1, 12, 6, Rk, -dT);                                                   // :131
            put33(H1, 6, 9, Hbe, -1.0);                                                  // :135
            putI(H1, 9, 9, -1.0);                                                        // :137
            put33(H1, 12, 9, Hal, -1.0);                                                 // :139
            put33(H1, 12, 12, Rk, -1.0);                                                 // :143
        }
        if (wantH2) {                                                                    // :158-198
            double A[9];
            quat_mat(q_r, +1.0, A);
            put33(H2, 0, 0, A, 1.0);                                                     // :169
            putI(H2, 3, 3, 1.0);
            put33(H2, 6, 6, Rk, 1.0);
            putI(H2, 9, 9, 1.0);
            put33(H2, 12, 12, Rk, 1.0);
        }
    }
    __syncthreads();

    // coalesced stream-out: three contiguous ranges per CTA, 16 bytes per lane (f0 is a multiple of FPB = 8, so every range starts
    // 16-byte aligned when the caller's arrays are; the last element of an odd-length range goes out as a single double)
    auto copy_out = [&](double* dst, const double* src, int n) {
        if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
            double2* d2 = reinterpret_cast<double2*>(dst);
            const double2* s2 = reinterpret_cast<const double2*>(src);
            for (int k = tid; k < n / 2; k += blockDim.x) d2[k] = s2[k];
            if ((n & 1) && tid == 0) dst[n - 1] = src[n - 1];
        } else {
            for (int k = tid; k < n; k += blockDim.x) dst[k] = src[k];
        }
    };
    copy_out(p.e + f0 * 15, tE, nf * 15);
    if (wantH1) copy_out(p.H1 + f0 * 225, tH1, nf * 225);
    if (wantH2) copy_out(p.H2 + f0 * 225, tH2, nf * 225);
}

// ---- getpredictedstate_v1/_v2 (GraphSolver_IMU.cpp:263-307): one thread per window -------------------------------------
template <int MODEL>
__global__ void k_predict(int64_t n, const double* states, const double* records, const double* lin, double* out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    constexpr int RD = (MODEL == 1) ? CPI_REC_V1_DOUBLES : CPI_REC_V2_DOUBLES;
    const double* x = states + i * CPI_STATE_DOUBLES;
    const double* r = records + i * (int64_t)RD;
    const double* l = lin + i * CPI_LIN_DOUBLES;
    predict_state<MODEL>(x, r, l, out + i * CPI_STATE_DOUBLES);
}

// ---- JPLNavState::retract (JPLNavState.cpp:37-71) -----------------------------------------------------------------------
__global__ void k_retract(int64_t n, const double* states, const double* xi, double* out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    retract_state(states + i * CPI_STATE_DOUBLES, xi + i * 15, out + i * CPI_STATE_DOUBLES);
}

// ---- information-form linearisation of the IMU factors ("next" row 1 of SURVEY.md 8f) -------------------------------------
// What GTSAM does right after evaluateError: whiten with the factor's Gaussian noise model (noiseModel::Gaussian::Covariance(P_meas),
// gtsam/ImuFactorCPIv1.h:82) and accumulate the normal equations.  With Sigma = L L^T and Y = L^-1 [H1 H2 e]:
//     G_ij = H_i^T Sigma^-1 H_j = Y_i^T Y_j,   g_i = -H_i^T Sigma^-1 e = -Y_i^T y_e,   f = e^T Sigma^-1 e = y_e^T y_e
// (the HessianFactor convention: G, g = A^T b with A = R H, b = -R e; independent of which square root R of Sigma^-1 is used).
// One warp per factor: Cholesky of the 15x15 covariance in shared memory, then lane c forward-substitutes column c of the 31
// right-hand sides, then lane c forms row c of Y^T Y from broadcast reads of Y.
__global__ void __launch_bounds__(128) k_factor_hessian(int64_t n, int rd, const double* records, const double* e, const double* H1, const double* H2,
                                                        double* G11, double* G12, double* G22, double* g1, double* g2, double* fq) {
    __shared__ double sL[4][15 * 16];      // lower Cholesky factor, row-major with pitch 16
    __shared__ double sY[4][15 * 32];      // Y, row i pitch 32
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t f = (int64_t)blockIdx.x * 4 + wib;
    if (f >= n) return;
    double* L = sL[wib];
    double* Y = sY[wib];
    const double* P = records + f * (int64_t)rd + CPI_REC_P;
    for (int k = lane; k < 225; k += 32) { const int r = k % 15, c = k / 15; if (r >= c) L[r * 16 + c] = __ldg(P + k); }   // lower triangle (P symmetric)
    __syncwarp();
    // right-looking Cholesky; a non-positive pivot (covariance not positive definite, e.g. a zero-step window) gives NaN outputs
    for (int k = 0; k < 15; k++) {
        const double d = sqrt(L[k * 16 + k]);
        __syncwarp();
        if (lane == 0) L[k * 16 + k] = d;
        if (lane > k && lane < 15) L[lane * 16 + k] = L[lane * 16 + k] / d;
        __syncwarp();
        // trailing update: pairs (i, j) with k < j <= i < 15 out of the 120 lower-triangle entries
        for (int t = lane; t < 120; t += 32) {
            int i = 0, acc = 0;
            while (acc + i + 1 <= t) { acc += i + 1; i++; }      // t -> (i, j) in the lower triangle incl. diagonal
            const int j = t - acc;
            if (j > k && i > k) L[i * 16 + j] -= L[i * 16 + k] * L[j * 16 + k];
        }
        __syncwarp();
    }
    // forward substitution, one right-hand side per lane: columns of H1 (0..14), H2 (15..29), e (30)
    double y[15];
    if (lane < 31) {
        const double* b = lane < 15 ? H1 + f * 225 + 15 * lane : (lane < 30 ? H2 + f * 225 + 15 * (lane - 15) : e + f * 15);
#pragma unroll
        for (int i = 0; i < 15; i++) {
            double t = __ldg(b + i);
#pragma unroll
            for (int k = 0; k < i; k++) t = fma(-L[i * 16 + k], y[k], t);
            y[i] = t / L[i * 16 + i];
            Y[i * 32 + lane] = y[i];
        }
    }
    __syncwarp();
    if (lane < 31) {
        double g[31];
#pragma unroll
        for (int c = 0; c < 31; c++) {
            double t = 0.0;
#pragma unroll
            for (int i = 0; i < 15; i++) t = fma(y[i], Y[i * 32 + c], t);
            g[c] = t;
        }
        if (lane < 15) {
#pragma unroll
            for (int r = 0; r < 15; r++) G11[f * 225 + r + 15 * lane] = g[r];                 // column `lane` of H1^T W H1
        } else if (lane < 30) {
#pragma unroll
            for (int r = 0; r < 15; r++) { G12[f * 225 + r + 15 * (lane - 15)] = g[r]; G22[f * 225 + r + 15 * (lane - 15)] = g[15 + r]; }
        } else {
#pragma unroll
            for (int r = 0; r < 15; r++) { g1[f * 15 + r] = -g[r]; g2[f * 15 + r] = -g[15 + r]; }
            fq[f] = g[30];
        }
    }
}

// ---- launchers -------------------------------------------------------------------------------------------------------
cudaError_t factor_launch(int model, const FactorParams& p, cudaStream_t st) {
    if (p.n == 0) return cudaSuccess;
    const size_t smem = (size_t)FPB * FTILE * sizeof(double);
    const int grid = (int)((p.n + FPB - 1) / FPB);
    // the opt-in attribute is sticky per device context: set it once per device, not per launch
    static bool configured[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 64 || !configured[dev]) {
        cudaError_t e = cudaFuncSetAttribute(k_factor_eval<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k_factor_eval<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        if (dev < 64) configured[dev] = true;
    }
    if (model == 1) k_factor_eval<1><<<grid, FTHREADS, smem, st>>>(p);
    else k_factor_eval<2><<<grid, FTHREADS, smem, st>>>(p);
    return cudaGetLastError();
}

cudaError_t predict_launch(int model, int64_t n, const double* states, const double* records, const double* lin, double* out, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const int grid = (int)((n + 127) / 128);
    if (model == 1) k_predict<1><<<grid, 128, 0, st>>>(n, states, records, lin, out);
    else k_predict<2><<<grid, 128, 0, st>>>(n, states, records, lin, out);
    return cudaGetLastError();
}

cudaError_t hessian_launch(int rd, int64_t n, const double* records, const double* e, const double* H1, const double* H2,
                           double* G11, double* G12, double* G22, double* g1, double* g2, double* f, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    k_factor_hessian<<<(int)((n + 3) / 4), 128, 0, st>>>(n, rd, records, e, H1, H2, G11, G12, G22, g1, g2, f);
    return cudaGetLastError();
}

cudaError_t retract_launch(int64_t n, const double* states, const double* xi, double* out, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    k_retract<<<(int)((n + 127) / 128), 128, 0, st>>>(n, states, xi, out);
    return cudaGetLastError();
}

}  // namespace cpi
