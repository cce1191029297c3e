// Levenberg-Marquardt over many IMU chains on the device (DESIGN.md section 3f): the pieces a round needs besides the linearisation,
// the per-chain-damped assembly (k_chain_assemble_lm) and the isolated solve (k_bcr_*_iso) of solve.cu.
//   k_factor_cost (K9)  the whitened cost f = e^T P_meas^-1 e of each factor at given states: evaluateError's residual without
//                       Jacobians, the warp Cholesky of P_meas and one forward substitution -- k_factor_hessian's f without its blocks.
//   k_lm_terms          per state k: the model decrease term delta_k^T (2 rhs_k - (H delta)_k) of the UNDAMPED system (H delta from
//                       D minus the damping the assembly added, and E), whether delta_k is non-zero, and the current / candidate cost of
//                       the factor to the right of k.  One warp per state.
//   k_lm_decide         per chain: the sums of its states' terms in a fixed order (strided per thread, then a shuffle tree, then the
//                       four warps in order: no atomics, the same bits on every run), GTSAM's accept / reject rule, and the candidate
//                       states copied into the accepted chains.  One CTA per chain.
// GTSAM is not part of the reference tree: PARITY UNPINNED -- the numpy statement of tests/test_chains_lm.py is the reference.
#include <math_constants.h>

#include "cpi_common.cuh"
#include "cpi_kernels.h"
#include "chol15.cuh"
#include "factor_blocks.cuh"
#include "../../include/cpi_b200.h"

namespace cpi {

// One warp per factor (4 per CTA, as k_factor_hessian).  The Cholesky and the substitution are k_factor_hessian's operations in its
// order, and the residual is K3's, so f is k_factor_hessian's f at the same states; a non-positive pivot gives NaN.
template <int MODEL>
__global__ void __launch_bounds__(128) k_factor_cost(int64_t n, const double* states, const int64_t* idx_i, const int64_t* idx_j,
                                                     const double* records, const double* lin, double* fq) {
    __shared__ double sL[4][15 * 16];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t f = (int64_t)blockIdx.x * 4 + wib;
    if (f >= n) return;
    constexpr int RD = (MODEL == 1) ? CPI_REC_V1_DOUBLES : CPI_REC_V2_DOUBLES;
    double* L = sL[wib];
    const double* r = records + f * (int64_t)RD;
    for (int k = lane; k < 225; k += 32) { const int rr = k % 15, c = k / 15; if (rr >= c) L[rr * 16 + c] = __ldg(r + CPI_REC_P + k); }
    __syncwarp();
    warp_chol15(L, lane);
    if (lane != 0) return;
    const int64_t ia = idx_i ? idx_i[f] : f, ib = idx_j ? idx_j[f] : f + 1;
    const double* xi = states + ia * CPI_STATE_DOUBLES;
    const double* xj = states + ib * CPI_STATE_DOUBLES;
    const double* l = lin + f * CPI_LIN_DOUBLES;
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
    double q_n[4], q_m[4], q_rm[4], q_r[4], q_kR[4], dthk[3], Rk[9], Rpa[3], Rpb[3];
    factor_front<MODEL>(qK, qK1, vK, vK1, pK, pK1, dbg, q_lin, grav, q_meas, dT, Jq, q_n, q_m, q_rm, q_r, q_kR, dthk, Rk, Rpa, Rpb);
    // the residual, as K3 forms it (ImuFactorCPIv1.cpp:84-88)
    double ah[3], bh[3], u[3], w[3], y[15];
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
    for (int k = 0; k < 3; k++) {
        y[k] = 2.0 * q_r[k];
        y[3 + k] = bgK1[k] - bgK[k];
        y[6 + k] = bh[k] - beta[k];
        y[9 + k] = baK1[k] - baK[k];
        y[12 + k] = ah[k] - alpha[k];
    }
    fwd15(L, y);
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 15; i++) s = fma(y[i], y[i], s);
    fq[f] = s;
}

// the chain holding state k (last c with o[c] <= k), and its state range
CPI_DEV int64_t chain_of(int64_t k, int64_t n_chains, const int64_t* offs, int64_t uniform, int64_t& lo, int64_t& hi) {
    if (offs) {
        int64_t a = 0, b = n_chains - 1;
        while (a < b) { const int64_t mid = (a + b + 1) >> 1; if (offs[mid] <= k) a = mid; else b = mid - 1; }
        lo = offs[a]; hi = offs[a + 1];
        return a;
    }
    const int64_t c = k / uniform;
    lo = c * uniform; hi = lo + uniform;
    return c;
}

// terms[k] = (delta_k^T (2 rhs_k - (H delta)_k), f_cur of the factor right of k (0 if k is last), f_new of it, delta_k != 0)
__global__ void __launch_bounds__(128) k_lm_terms(int64_t n_states, int64_t n_chains, const int64_t* offs, int64_t uniform, const double* f_cur,
                                                  const double* f_new, const double* rhs, const double* D, const double* E, const double* damp,
                                                  const double* delta, double* terms) {
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t k = (int64_t)blockIdx.x * 4 + wib;
    if (k >= n_states) return;
    int64_t lo, hi;
    const int64_t c = chain_of(k, n_chains, offs, uniform, lo, hi);
    const bool first = k == lo, last = k == hi - 1;
    double part = 0.0;
    bool nz = false;
    if (lane < 15) {
        const double* Dk = D + k * 225;
        const double* dk = delta + k * 15;
        double hd = 0.0;                                           // row `lane` of H delta: (D_k - damp_k) delta_k + E_{k-1}^T delta_{k-1} + E_k delta_{k+1}
#pragma unroll
        for (int q = 0; q < 15; q++) hd = fma(q == lane ? Dk[lane + 15 * q] - damp[k * 15 + lane] : Dk[lane + 15 * q], dk[q], hd);
        if (!first) {
            const double* Ep = E + (k - 1) * 225;
#pragma unroll
            for (int q = 0; q < 15; q++) hd = fma(Ep[q + 15 * lane], delta[(k - 1) * 15 + q], hd);
        }
        if (!last) {
            const double* En = E + k * 225;
#pragma unroll
            for (int q = 0; q < 15; q++) hd = fma(En[lane + 15 * q], delta[(k + 1) * 15 + q], hd);
        }
        const double d = dk[lane];
        part = d * (2.0 * rhs[k * 15 + lane] - hd);
        nz = d != 0.0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    nz = __any_sync(0xffffffffu, nz);
    if (lane == 0) {
        double* t = terms + k * 4;
        t[0] = part;
        t[1] = last ? 0.0 : f_cur[k - c];
        t[2] = last ? 0.0 : f_new[k - c];
        t[3] = nz ? 1.0 : 0.0;
    }
}

__global__ void __launch_bounds__(128) k_lm_decide(int64_t n_chains, const int64_t* offs, int64_t uniform, cpi_lm_params p, const double* pf_cur,
                                                   const double* pf_new, const double* terms, const double* states_new, double* states,
                                                   double* lam, double* cost, int32_t* status, int32_t* iterations, int32_t* tries,
                                                   int32_t* any_running) {
    __shared__ double sw[4][4];
    __shared__ int accept;
    const int64_t c = blockIdx.x;
    if (status[c] != CPI_LM_RUNNING) return;                       // frozen: never touched again
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t lo = offs ? offs[c] : c * uniform, hi = offs ? offs[c + 1] : lo + uniform;
    double s[4] = {0.0, 0.0, 0.0, 0.0};
    for (int64_t k = lo + threadIdx.x; k < hi; k += blockDim.x)
#pragma unroll
        for (int j = 0; j < 4; j++) s[j] += terms[k * 4 + j];
#pragma unroll
    for (int j = 0; j < 4; j++)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s[j] += __shfl_xor_sync(0xffffffffu, s[j], o);
    if (lane == 0)
#pragma unroll
        for (int j = 0; j < 4; j++) sw[wib][j] = s[j];
    __syncthreads();
    if (threadIdx.x == 0) {
        const double m = ((sw[0][0] + sw[1][0]) + sw[2][0]) + sw[3][0];
        const double cur = (((sw[0][1] + sw[1][1]) + sw[2][1]) + sw[3][1]) + (pf_cur ? pf_cur[c] : 0.0);
        const double nw = (((sw[0][2] + sw[1][2]) + sw[2][2]) + sw[3][2]) + (pf_new ? pf_new[c] : 0.0);
        const bool moved = (((sw[0][3] + sw[1][3]) + sw[2][3]) + sw[3][3]) != 0.0;
        double l = lam[c];
        int st = CPI_LM_RUNNING, acc = 0;
        const int tr = tries[c] + 1;
        int it = iterations[c];
        if (!isfinite(cur) || !isfinite(m)) {
            st = CPI_LM_NONFINITE;
        } else if (!moved) {                                       // delta = 0 exactly: nothing left to do
            st = CPI_LM_CONVERGED;
        } else if (isfinite(nw) && m > 0.0 && (cur - nw) / m > p.min_model_fidelity) {
            acc = 1;
            it += 1;
            l = fmax(l / p.lambda_factor, p.lambda_lower);
            const double dec = cur - nw;                           // twice GTSAM's error: the tolerances apply to half of it
            if (0.5 * dec <= p.absolute_error_tol || dec <= p.relative_error_tol * cur) st = CPI_LM_CONVERGED;
            else if (it >= p.max_iterations) st = CPI_LM_MAX_ITERATIONS;
        } else if (l >= p.lambda_upper) {
            st = CPI_LM_LAMBDA_EXHAUSTED;
        } else {
            l = l * p.lambda_factor;
        }
        lam[c] = l;
        cost[c] = acc ? nw : cur;
        status[c] = st;
        iterations[c] = it;
        tries[c] = tr;
        if (st == CPI_LM_RUNNING && any_running) *any_running = 1;
        accept = acc;
    }
    __syncthreads();
    if (accept)
        for (int64_t t = lo * CPI_STATE_DOUBLES + threadIdx.x; t < hi * CPI_STATE_DOUBLES; t += blockDim.x) states[t] = states_new[t];
}

// ---- launchers ----------------------------------------------------------------------------------------------------------------------
cudaError_t factor_cost_launch(int model, int64_t n, const double* states, const int64_t* idx_i, const int64_t* idx_j, const double* records,
                               const double* lin, double* f, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const int grid = (int)((n + 3) / 4);
    if (model == 1) k_factor_cost<1><<<grid, 128, 0, st>>>(n, states, idx_i, idx_j, records, lin, f);
    else k_factor_cost<2><<<grid, 128, 0, st>>>(n, states, idx_i, idx_j, records, lin, f);
    return cudaGetLastError();
}

int64_t lm_workspace_bytes(int64_t n_states) { return n_states * 4 * 8; }

cudaError_t lm_update_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, int64_t n_states, const cpi_lm_params& p, const double* f_cur,
                             const double* pf_cur, const double* f_new, const double* pf_new, const double* rhs, const double* D, const double* E,
                             const double* damp, const double* delta, const double* states_new, double* states, double* lam, double* cost,
                             int32_t* status, int32_t* iterations, int32_t* tries, int32_t* any_running, double* ws, cudaStream_t st) {
    k_lm_terms<<<(int)((n_states + 3) / 4), 128, 0, st>>>(n_states, n_chains, offs, uniform, f_cur, f_new, rhs, D, E, damp, delta, ws);
    k_lm_decide<<<(int)n_chains, 128, 0, st>>>(n_chains, offs, uniform, p, pf_cur, pf_new, ws, states_new, states, lam, cost, status, iterations, tries,
                                               any_running);
    return cudaGetLastError();
}

}  // namespace cpi
