// Gaussian priors on any state of many IMU chains (DESIGN.md section 3g): GTSAM's PriorFactor / the reference's JPLNavStatePrior on
// any keyframe, not only on a chain's first state.
//   k_state_prior_fold  adds the already-moved priors (info, rhs', f') of every state into ONE block the existing kernels read, so the
//                       assembly, both solves, K8 and the LM decision see them without a change:
//                           state k not the last of its chain        -> G11, g1, f of the factor to its right (index k - c)
//                           last state of a chain of >= 2 states     -> G22, g2, f of the factor to its left  (index k - 1 - c)
//                           the only state of its chain              -> the chain prior (info, rhs, f) of chain c
//                       One warp per state (grid-stride), lanes over the 225 + 15 + 1 entries; the priors of state k are the CSR
//                       range sp_offsets[k] .. sp_offsets[k+1]-1 and are added one after the other in that order: additions only, no
//                       atomics, the same bits on every run.  Each 15x15 block and rhs segment receives the priors of exactly one
//                       state; the f of a chain's last factor receives those of its two states, added by one warp, the left state's first.
//   k_state_prior_robust  reweights moved MEASUREMENT priors (rhs = 0, f = 0 before prior_at, so f' = s = delta^T W delta) by a robust
//                       loss (DESIGN.md section 3h): (info, rhs', f') -> (w info, w rhs', c(s)) with c = 2 rho(sqrt s) and the IRLS
//                       weight w = dc/ds of GTSAM's noiseModel::Robust (Huber, Cauchy).  One warp per prior (grid-stride), one lane
//                       computes s, w and c and broadcasts them, the lanes scale the 225 + 15 entries.  A weight of exactly 1 copies.
// GTSAM is not part of the reference tree: PARITY UNPINNED -- the numpy statement of tests/test_state_priors.py is the reference (and
// that of tests/test_robust_priors.py for the losses).
#include <math_constants.h>

#include <algorithm>

#include "cpi_common.cuh"
#include "cpi_kernels.h"
#include "robust_loss.cuh"

namespace cpi {

__global__ void __launch_bounds__(128) k_state_prior_fold(int64_t n_chains, const int64_t* offs, int64_t uniform, const int64_t* sp_offsets,
                                                          const double* sp_info, const double* sp_rhs, const double* sp_f, double* G11, double* G22,
                                                          double* g1, double* g2, double* f, double* prior_info, double* prior_rhs, double* prior_f) {
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t ns = offs ? offs[n_chains] : n_chains * uniform;
    for (int64_t k = (int64_t)blockIdx.x * 4 + wib; k < ns; k += (int64_t)gridDim.x * 4) {
        const int64_t a = sp_offsets[k], b = sp_offsets[k + 1];
        const int64_t b2 = k + 1 < ns ? sp_offsets[k + 2] : b;     // the next state's priors end (its f may land in the same f as k's)
        if (a >= b && b >= b2) continue;                           // nothing on this state or the next (the whole warp moves on)
        int64_t c, lo, hi;
        if (offs) {                                                // the chain holding k: last c with o[c] <= k (chains are non-empty)
            int64_t u = 0, v = n_chains - 1;
            while (u < v) { const int64_t mid = (u + v + 1) >> 1; if (offs[mid] <= k) u = mid; else v = mid - 1; }
            c = u; lo = offs[u]; hi = offs[u + 1];
        } else {
            c = k / uniform; lo = c * uniform; hi = lo + uniform;
        }
        // the target block; a NULL target receives nothing.  The f of a chain's last factor takes the priors of both its states: the
        // warp of the left state adds its own, then the last state's, so that one warp writes it.
        double *I, *r, *fs;
        int64_t fe = b;                                            // the f terms added: a .. fe-1
        if (k < hi - 1) {
            const int64_t fi = k - c;
            I = G11 ? G11 + fi * 225 : nullptr; r = g1 ? g1 + fi * 15 : nullptr; fs = f ? f + fi : nullptr;
            if (k == hi - 2) fe = b2;
        } else if (hi - lo >= 2) {
            const int64_t fi = k - 1 - c;
            I = G22 ? G22 + fi * 225 : nullptr; r = g2 ? g2 + fi * 15 : nullptr; fs = nullptr;
        } else {
            I = prior_info ? prior_info + c * 225 : nullptr; r = prior_rhs ? prior_rhs + c * 15 : nullptr; fs = prior_f ? prior_f + c : nullptr;
        }
        if (sp_info && I && a < b)
            for (int t = lane; t < 225; t += 32) {
                double s = I[t];
                for (int64_t j = a; j < b; j++) s = s + sp_info[j * 225 + t];
                I[t] = s;
            }
        if (sp_rhs && r && lane < 15 && a < b) {
            double s = r[lane];
            for (int64_t j = a; j < b; j++) s = s + sp_rhs[j * 15 + lane];
            r[lane] = s;
        }
        if (sp_f && fs && lane == 31 && a < fe) {
            double s = *fs;
            for (int64_t j = a; j < fe; j++) s = s + sp_f[j];
            *fs = s;
        }
    }
}

cudaError_t state_priors_fold_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, const int64_t* sp_offsets, const double* sp_info,
                                     const double* sp_rhs, const double* sp_f, double* G11, double* G22, double* g1, double* g2, double* f,
                                     double* prior_info, double* prior_rhs, double* prior_f, int sms, cudaStream_t st) {
    // uniform layout: one warp per state.  A device-resident layout's state count is not known here: at least one warp per chain and
    // 32 CTAs per SM, grid-striding over the states
    int64_t grid = offs ? std::max<int64_t>((int64_t)sms * 32, (n_chains + 3) / 4) : (n_chains * uniform + 3) / 4;
    grid = std::min<int64_t>(grid, 0x7fffffff);
    if (grid < 1) return cudaSuccess;
    k_state_prior_fold<<<(int)grid, 128, 0, st>>>(n_chains, offs, uniform, sp_offsets, sp_info, sp_rhs, sp_f, G11, G22, g1, g2, f, prior_info,
                                                  prior_rhs, prior_f);
    return cudaGetLastError();
}

__global__ void __launch_bounds__(128) k_state_prior_robust(int64_t n, const int32_t* loss, const double* loss_k, const double* info,
                                                            const double* rhs, const double* f, double* info_out, double* rhs_out, double* f_out) {
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t i = (int64_t)blockIdx.x * 4 + wib; i < n; i += (int64_t)gridDim.x * 4) {
        double w = 0.0, c = 0.0;
        if (lane == 0) robust_loss(loss[i], loss_k[i], f[i], w, c);
        w = __shfl_sync(0xffffffffu, w, 0);
        c = __shfl_sync(0xffffffffu, c, 0);
        if (info_out) {                                            // rhs_out may alias rhs: each lane reads its entry before writing it
            for (int t = lane; t < 225; t += 32) {
                const double v = info[i * 225 + t];
                info_out[i * 225 + t] = w == 1.0 ? v : w * v;
            }
            if (lane < 15) {
                const double v = rhs[i * 15 + lane];
                rhs_out[i * 15 + lane] = w == 1.0 ? v : w * v;
            }
        }
        if (lane == 0) f_out[i] = c;                               // f_out may alias f: lane 0 read f[i] above
    }
}

cudaError_t state_priors_robust_launch(int64_t n, const int32_t* loss, const double* loss_k, const double* info, const double* rhs,
                                       const double* f, double* info_out, double* rhs_out, double* f_out, cudaStream_t st) {
    const int64_t grid = std::min<int64_t>((n + 3) / 4, 0x7fffffff);
    if (grid < 1) return cudaSuccess;
    k_state_prior_robust<<<(int)grid, 128, 0, st>>>(n, loss, loss_k, info, rhs, f, info_out, rhs_out, f_out);
    return cudaGetLastError();
}

}  // namespace cpi
