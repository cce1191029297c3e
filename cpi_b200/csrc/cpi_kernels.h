// Kernel parameter blocks and host-side launchers shared by capi.cu and the kernel translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/cpi_b200.h"

namespace cpi {

struct PropagateParams {
    int64_t n;
    const double* states;     // anchor states (CPI_STATE_DOUBLES each)
    const double* cov;        // anchor covariances (225 each, column-major)
    const int64_t* anchor;    // may be null: window i starts from entry i
    const double* records;
    const double* lin;
    double* states_k1;
    double* cov_k1;
    double* cross;            // may be null
};

struct PreintParams {
    int64_t n_windows;
    const int64_t* offsets;   // device, may be null (uniform windows)
    int64_t ns_uniform;
    const void* samples;      // device, double (dtype 64) or float (dtype 32)
    const void* lin;          // device
    void* out;                // device
    const void* init;         // device, may be null: records holding the state to CONTINUE from (may alias `out`); tri-lane kernels only
    double q_w, q_wb, q_a, q_ab;   // sigma^2  (CpiBase.h:54-57)
    int wpb;                  // windows per block; 0 on entry = let preint_launch choose (one wave if possible)
};

struct FactorParams {
    int64_t n;
    const double* states;
    const int64_t* idx_i;
    const int64_t* idx_j;
    const double* records;
    const double* lin;
    double* e;
    double* H1;
    double* H2;
};

int preint_pick_wpb(int model, int dtype, int64_t n_windows, int num_sms);
int preint_cap(int model, int dtype, int flags, int num_sms);
// tri-lane kernels (preintegrate_tri.cu)
bool preint_tri_supported(int model, int flags);
int preint_tri_cap(int model, int dtype);
cudaError_t preint_launch_tri(int model, int dtype, const PreintParams& p, int num_sms, cudaStream_t st);
cudaError_t preint_launch(int model, int dtype, int flags, const PreintParams& p0, int num_sms, int max_smem_bytes, cudaStream_t st, int* launches);
cudaError_t factor_launch(int model, const FactorParams& p, cudaStream_t st);
cudaError_t predict_launch(int model, int64_t n, const double* states, const double* records, const double* lin, double* out, cudaStream_t st);
cudaError_t hessian_launch(int rd, int64_t n, const double* records, const double* e, const double* H1, const double* H2,
                           double* G11, double* G12, double* G22, double* g1, double* g2, double* f, cudaStream_t st);
cudaError_t whiten_launch(int rd, int64_t n, const double* records, const double* e, const double* H1, const double* H2, double* A1, double* A2, double* b, cudaStream_t st);
// solve.cu: block-tridiagonal normal equations of n_chains chains (offs: device int64[n_chains+1], or NULL and `uniform` states per chain)
cudaError_t chains_assemble_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, const double* G11, const double* G12, const double* G22,
                                   const double* g1, const double* g2, double lambda, int diagonal_damping, const double* prior_info,
                                   const double* prior_rhs, double* D, double* E, double* rhs, int sms, cudaStream_t st);
// the per-chain-lambda assembly, and the solve with couplings between chains never loaded (cpi_imu_chains_assemble_lm /
// cpi_imu_chains_solve; cpi_imu_chain_solve is its one-chain case)
cudaError_t chains_assemble_lm_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, const double* G11, const double* G12, const double* G22,
                                      const double* g1, const double* g2, const double* lams, int diagonal_damping, const double* prior_info,
                                      const double* prior_rhs, double* D, double* E, double* rhs, double* damp, int sms, cudaStream_t st);
int64_t chains_solve_workspace_bytes(int64_t n_states);
cudaError_t chains_solve_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, int64_t n_states, const double* D, const double* E, const double* b,
                                double* x, double* ws, int sms, cudaStream_t st, int* launches);
// the diagonal and neighbour blocks of the inverse by selected inversion of the isolated solve's levels (cpi_imu_chains_marginals)
int64_t chains_marginals_workspace_bytes(int64_t n_states);
cudaError_t chains_marginals_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, int64_t n_states, const double* D, const double* E,
                                    double* cov, double* cross, double* ws, int sms, cudaStream_t st, int* launches);
// merge.cu: one merged model-1 record per group (dtype 64 or 32)
cudaError_t merge_launch(int dtype, int64_t n_groups, const int64_t* offsets, int64_t uniform, const void* records, const void* lin,
                         void* out, cudaStream_t st);
// scan.cu: inclusive scan of model-1 records within groups, one record per input record (dtype 64 or 32); n_bound >= the record count
int64_t scan_workspace_bytes(int64_t n_records);
cudaError_t scan_launch(int dtype, int64_t n_groups, const int64_t* offsets, int64_t uniform, int64_t n_bound, const void* records,
                        const void* lin, void* out, void* workspace, int sms, cudaStream_t st, int* launches);
// propagate.cu: prediction and covariance propagation through one record per window (fp64)
cudaError_t propagate_launch(int model, const PropagateParams& p, cudaStream_t st);
// marginalize.cu: elimination of the leading states of every chain into a prior (K8), and a prior moved to other states
cudaError_t marginalize_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, const int64_t* n_marg, int64_t marg_uniform,
                               const double* G11, const double* G12, const double* G22, const double* g1, const double* g2, const double* f,
                               const double* prior_info, const double* prior_rhs, const double* prior_f, double* out_info, double* out_rhs,
                               double* out_f, cudaStream_t st);
cudaError_t prior_at_launch(int64_t n, const double* info, const double* rhs, const double* f, const double* lin, const double* x,
                            double* rhs_out, double* f_out, cudaStream_t st);
// lm.cu: the factor cost (K9) and the per-chain Levenberg-Marquardt decision
cudaError_t factor_cost_launch(int model, int64_t n, const double* states, const int64_t* idx_i, const int64_t* idx_j, const double* records,
                               const double* lin, double* f, cudaStream_t st);
cudaError_t chains_cost_sum_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, const double* f, double* cost, cudaStream_t st);
int64_t lm_workspace_bytes(int64_t n_states);
cudaError_t lm_update_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, int64_t n_states, const cpi_lm_params& p, const double* f_cur,
                             const double* pf_cur, const double* f_new, const double* pf_new, const double* rhs, const double* D, const double* E,
                             const double* damp, const double* delta, const double* states_new, double* states, double* lam, double* cost,
                             int32_t* status, int32_t* iterations, int32_t* tries, int32_t* any_running, double* ws, cudaStream_t st);
// state_priors.cu: priors on any state folded into the factor blocks / chain priors (sp_info, sp_rhs NULL: the f-only fold)
cudaError_t state_priors_fold_launch(int64_t n_chains, const int64_t* offs, int64_t uniform, const int64_t* sp_offsets, const double* sp_info,
                                     const double* sp_rhs, const double* sp_f, double* G11, double* G22, double* g1, double* g2, double* f,
                                     double* prior_info, double* prior_rhs, double* prior_f, int sms, cudaStream_t st);
// state_priors.cu: robust (Huber / Cauchy) reweighting of moved measurement priors (info_out, rhs_out NULL: the f-only pass)
cudaError_t state_priors_robust_launch(int64_t n, const int32_t* loss, const double* loss_k, const double* info, const double* rhs,
                                       const double* f, double* info_out, double* rhs_out, double* f_out, cudaStream_t st);
cudaError_t retract_launch(int64_t n, const double* states, const double* xi, double* out, cudaStream_t st);
// update.cu: the filter's measurement update by direct state fixes, with chi-square gating (K10; gate, nis, applied may be NULL)
cudaError_t state_update_launch(int64_t n, const double* states, const double* cov, const double* meas_info, const double* meas_states,
                                const double* gate, double* states_out, double* cov_out, double* nis, int32_t* applied, cudaStream_t st);
// update.cu: the same update by attitude-dependent measurements, a CSR list per filter (K11; gate, nis, applied may be NULL)
cudaError_t state_update_meas_launch(int64_t n, const double* states, const double* cov, const int64_t* meas_offsets, const int32_t* kind,
                                     const double* z, const double* sqrt_info, const double* aux, const double* gate, double* states_out,
                                     double* cov_out, double* nis, int32_t* applied, cudaStream_t st);
// update.cu: the iterated update by the same measurements, with robust losses (K13; loss / loss_k, gate, nis, status, iterations may be NULL)
cudaError_t state_update_meas_iter_launch(int64_t n, const double* states, const double* cov, const int64_t* meas_offsets, const int32_t* kind,
                                          const double* z, const double* sqrt_info, const double* aux, const int32_t* loss, const double* loss_k,
                                          const double* gate, int max_iter, double tol, double* states_out, double* cov_out, double* nis,
                                          int32_t* status, int32_t* iterations, cudaStream_t st);
// measurements.cu: measurements linearised into moved prior blocks (K12; info, rhs NULL: the f-only pass)
cudaError_t measurements_linearize_launch(int64_t n, const int32_t* kind, const int64_t* state_idx, const double* states, const double* z,
                                          const double* sqrt_info, const double* aux, double* info, double* rhs, double* f, cudaStream_t st);
// relinearize.cu: selection, stable compaction, gather and scatter around the K1/K2 launch of cpi_imu_records_relinearize
struct RelinWorkspace {
    double* crec;             // compact records [n][rd]
    double* clin;             // compact linearisation points [n][13]
    int64_t* idx;             // the selected factors, in factor order
    int64_t* coff;            // compact CSR sample offsets [n + 1]
    int32_t* flag;            // per factor 0/1
    long long* blk;           // per CTA of the selection: {selected, entries}
    long long* pre;           // their exclusive prefixes, then the grand totals {selected, entries} the host reads
    double* csamp;            // compact samples (16-byte aligned), last
    int64_t head_bytes;       // bytes before csamp
};
RelinWorkspace relin_workspace(void* ws, int rd, int64_t n);
int64_t relin_workspace_bytes(int rd, int64_t n, int64_t n_entries);
int64_t relin_total_offset(int64_t n);   // index into `pre` of the grand totals
cudaError_t relin_select_launch(int model, int64_t n, const double* states, const int64_t* idx_i, const int64_t* offs, int64_t ent_uniform,
                                const double* lin, double tw2, double ta2, double tt2, int32_t* mask, const RelinWorkspace& w, cudaStream_t st);
cudaError_t relin_gather_launch(int64_t n_sel, const int64_t* offs, int64_t ent_uniform, const double* samples, const RelinWorkspace& w,
                                int sms, cudaStream_t st);
cudaError_t relin_scatter_launch(int64_t n_sel, int rd, const RelinWorkspace& w, double* records, double* lin, int sms, cudaStream_t st);

}  // namespace cpi
