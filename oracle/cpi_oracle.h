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

/* quat_ops.h helpers (col-major 3x3) */
void oracle_rot_2_quat(const double* R, double* q);
void oracle_quat_2_Rot(const double* q, double* R);
void oracle_quat_multiply(const double* q, const double* p, double* out);
void oracle_Exp(const double* w, double* R);

#ifdef __cplusplus
}
#endif
#endif
