/* TEST INFRASTRUCTURE ONLY.  CPU restatement (plain C, dense, literal) of the reference's hot path.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may load this.
 * Layouts: include/cpi_b200.h.  All pointers are HOST pointers. */
#ifndef CPI_ORACLE_H
#define CPI_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

int oracle_cpi_preintegrate(int model, int64_t n_windows, const int64_t* offsets, int64_t ns_uniform,
                            const double* samples, const double* lin, const double* sigmas, int flags,
                            double* out, int nthreads);
int oracle_imu_factor_eval(int model, int64_t n, const double* states, const int64_t* idx_i, const int64_t* idx_j,
                           const double* records, const double* lin, double* e, double* H1, double* H2, int nthreads);
int oracle_predict_state(int model, int64_t n, const double* states_k, const double* records, const double* lin,
                         double* states_k1);
int oracle_retract(int64_t n, const double* states, const double* xi, double* out);

/* Model-1 record composition (DESIGN.md 3b, 3c), dense.  merge_pair: out[i] = a[i] (+) b[i], both at one linearisation point.
 * relinearise_records: out[i] = records[i] moved from lin[i] to lin0[i] to first order.  merge_records / scan_records: the left
 * fold of every group (CSR offsets, or groups of `uniform` records when offsets is NULL), every later record moved to the
 * group's first linearisation point; merge writes one record per group (empty group: the zero-step record), scan writes every
 * prefix fold at its record's row of out (shaped like records; rows outside every group are not written). */
int oracle_merge_pair(int64_t n, const double* a, const double* b, double* out, int nthreads);
int oracle_relinearise_records(int64_t n, const double* records, const double* lin, const double* lin0, double* out);
int oracle_merge_records(int64_t n_groups, const int64_t* offsets, int64_t uniform, const double* records, const double* lin,
                         double* out, int nthreads);
int oracle_scan_records(int64_t n_groups, const int64_t* offsets, int64_t uniform, const double* records, const double* lin,
                        double* out, int nthreads);

/* The solver side of a chain (DESIGN.md 3e, 3f), dense.  Chain layouts as the C ABI (CSR state offsets, or chains of `uniform`
 * states when offsets is NULL).  chain_marginalize: K8's recurrence with a plain 15x15 Cholesky, NaN rule and m = 0 copy as
 * cpi_imu_chain_marginalize; scale (may be NULL) [n_chains, 242]: per chain the size of the terms that cancel into info (225), rhs
 * (15) and f (1), and the last step's z^T z.  chain_solve: x = A^-1 b of the SPD block-tridiagonal system, order 0 a sequential block
 * Cholesky per chain, order 1 the block cyclic reduction of the whole system in the order of solve.cu.  chain_marginals: the
 * selected inversion of the same system, cov [N, 225] = Sigma_kk and cross [N - n_chains, 225] = Sigma_{k,k+1} in the slots of
 * cpi_imu_chains_marginals (cross may be NULL), order 0 a sequential block Cholesky and backward recurrence per chain, order 1 the
 * isolated block cyclic reduction and top-down level walk of solve.cu (DESIGN.md 3j); NaN for a chain with a pivot that is not
 * positive.  lm_terms: out [n_chains, 5] =
 * (model decrease, the size of its terms, current cost, candidate cost, delta != 0).  local / prior_at: the inverse of retract and
 * cpi_imu_prior_at. */
int oracle_chain_marginalize(int64_t n_chains, const int64_t* offsets, int64_t uniform, const int64_t* n_marg, int64_t marg_uniform,
                             const double* G11, const double* G12, const double* G22, const double* g1, const double* g2, const double* f,
                             const double* prior_info, const double* prior_rhs, const double* prior_f, double* out_info, double* out_rhs,
                             double* out_f, double* scale, int nthreads);
int oracle_chain_solve(int64_t n_chains, const int64_t* offsets, int64_t uniform, const double* D, const double* E, const double* b, double* x,
                       int order, int nthreads);
int oracle_chain_marginals(int64_t n_chains, const int64_t* offsets, int64_t uniform, const double* D, const double* E, double* cov,
                           double* cross, int order, int nthreads);
int oracle_lm_terms(int64_t n_chains, const int64_t* offsets, int64_t uniform, const double* rhs, const double* D, const double* E,
                    const double* damp, const double* delta, const double* f_cur, const double* pf_cur, const double* f_new,
                    const double* pf_new, double* out, int nthreads);
int oracle_local(int64_t n, const double* lin, const double* x, double* delta);
int oracle_prior_at(int64_t n, const double* info, const double* rhs, const double* f, const double* lin, const double* x, double* rhs_out,
                    double* f_out);

/* K7 (DESIGN.md 3d): x_k1, Sigma_k1 = A Sigma_k A^T + B P_meas B^T and cross = Sigma_k A^T (may be NULL) of window i from the state
 * and covariance of anchor[i] (anchor NULL: i); order 0 dense (a pivoted inverse of H2), 1 propagate.cu's sparse route.
 * propagate_chain: `steps` windows per chain, state and covariance held in working precision between steps; path (may be NULL)
 * [n_chains * (steps + 1), 16] the states each step starts from.  Both split their windows (chains) over nthreads threads. */
int oracle_propagate(int model, int64_t n, const double* states_k, const double* cov_k, const int64_t* anchor, const double* records,
                     const double* lin, int order, double* states_k1, double* cov_k1, double* cross, int nthreads);
int oracle_propagate_chain(int model, int64_t n_chains, int64_t steps, const double* states0, const double* cov0, const double* path,
                           const double* records, const double* lin, int order, double* states_out, double* cov_out, int nthreads);

/* quat_ops.h helpers (col-major 3x3) */
void oracle_rot_2_quat(const double* R, double* q);
void oracle_quat_2_Rot(const double* q, double* R);
void oracle_quat_multiply(const double* q, const double* p, double* out);
void oracle_Exp(const double* w, double* R);

#ifdef __cplusplus
}
#endif
#endif
