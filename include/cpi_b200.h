/*
 * cpi_b200.h -- C ABI of libcpi_b200.so: batched closed-form IMU preintegration (CPI) on H100 (sm_90a).
 *
 * This is the drop-in boundary for the ONE hot path of rpng/cpi (reference tree paths are relative to
 * /root/reference/cpi_compare/src):
 *
 *   cpi_preintegrate_batch*    replaces the per-sample loop  CpiV1::feed_IMU  (cpi/CpiV1.h:62-361) and
 *                              CpiV2::feed_IMU (cpi/CpiV2.h:84-467) as driven, once per factor, by
 *                              GraphSolver::createimufactor_cpi_v1/_v2 (solvers/GraphSolver_IMU.cpp:43-75, 97-130),
 *                              for MANY windows at once.  Its per-window output record is exactly the set of public
 *                              CpiBase fields the caller reads afterwards (cpi/CpiBase.h:99-124, cpi/CpiV2.h:62-63).
 *   cpi_imu_factor_eval_batch* replaces ImuFactorCPIv1::evaluateError (gtsam/ImuFactorCPIv1.cpp:37-208) and
 *                              ImuFactorCPIv2::evaluateError (gtsam/ImuFactorCPIv2.cpp:38-212): unwhitened 15-d
 *                              residual and the two 15x15 Jacobians, for many factors at once.
 *   cpi_imu_factor_hessian_batch  the step GTSAM performs next: information-form blocks H^T P^-1 H, -H^T P^-1 e per factor.
 *   cpi_predict_state_batch*   replaces GraphSolver::getpredictedstate_v1/_v2 (solvers/GraphSolver_IMU.cpp:263-307).
 *   cpi_retract_batch*         replaces JPLNavState::retract (gtsam/JPLNavState.cpp:37-71).
 *
 * Conventions (all identical to the reference):  fp64; matrices COLUMN-major (Eigen default); JPL quaternion
 * [x y z w]; 15-d error-state order [dtheta(0:3), b_g(3:6), v/beta(6:9), b_a(9:12), p/alpha(12:15)]
 * (cpi/CpiV1.h:277-281, gtsam/ImuFactorCPIv1.cpp:80-88).
 *
 * Functions without the _host suffix take DEVICE pointers and enqueue on `stream` (a cudaStream_t passed as
 * void*; NULL = legacy default stream) without synchronising.  *_host variants take HOST pointers (pinned or pageable),
 * copy through device buffers owned by the library -- big batches in a 4-deep H2D / kernel / D2H pipeline -- and return
 * after the results are in the caller's buffers.
 * Every function returns CPI_OK (0) or a negative CPI_E* code; cpi_last_error() gives the message of the last
 * failure on the calling thread.  (The reference has no error convention for this path: feed_IMU returns void and
 * never checks its inputs -- CpiBase.h:86.)  No function falls back to a CPU implementation.
 */
#ifndef CPI_B200_H
#define CPI_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- layouts -------------------------------------------------------------------------------------------------- */

/* One IMU entry: [wx wy wz ax ay az dt] ; dt = t_{i+1} - t_i (seconds) is the length of the step that STARTS at this
 * entry, i.e. feed_IMU(t_i, t_i + dt, w_i, a_i, w_{i+1}, a_{i+1}).  The reference's line format "wx wy wz ax ay az
 * <unused> t_ms" (sim/SimParser.h:148-175) maps to this after differencing the time stamps. */
#define CPI_SAMPLE_DOUBLES 7
/* Per-window linearisation point = arguments of CpiBase::setLinearizationPoints (cpi/CpiBase.h:73-80):
 * [b_w_lin(3) b_a_lin(3) q_k_lin(4, JPL xyzw) grav(3)].  Model 1 ignores q_k_lin for preintegration; grav is only
 * carried to the factor (GraphSolver_IMU.cpp:74). */
#define CPI_LIN_DOUBLES 13
/* JPLNavState value (gtsam/JPLNavState.h:62-66): [q_GtoI(4) b_g(3) v_IinG(3) b_a(3) p_IinG(3)] */
#define CPI_STATE_DOUBLES 16

/* Per-window result record, doubles.  Field order = order the factor constructors consume them
 * (gtsam/ImuFactorCPIv1.h:78-81, gtsam/ImuFactorCPIv2.h:82-85). */
#define CPI_REC_Q      0    /* q_k2tau  [4]  rot_2_quat(R_k2tau)            CpiBase.h:102 */
#define CPI_REC_R      4    /* R_k2tau  [9]  col-major                      CpiBase.h:103 */
#define CPI_REC_ALPHA  13   /* alpha_tau[3]                                 CpiBase.h:100 */
#define CPI_REC_BETA   16   /* beta_tau [3]                                 CpiBase.h:101 */
#define CPI_REC_DT     19   /* DT                                           CpiBase.h:99  */
#define CPI_REC_JQ     20   /* J_q [9]  d(theta)/d(b_w)                     CpiBase.h:106 */
#define CPI_REC_JA     29   /* J_a [9]  d(alpha)/d(b_w)                     CpiBase.h:107 */
#define CPI_REC_JB     38   /* J_b [9]  d(beta)/d(b_w)                      CpiBase.h:108 */
#define CPI_REC_HA     47   /* H_a [9]  d(alpha)/d(b_a)                     CpiBase.h:109 */
#define CPI_REC_HB     56   /* H_b [9]  d(beta)/d(b_a)                      CpiBase.h:110 */
#define CPI_REC_P      65   /* P_meas [225] col-major 15x15                 CpiBase.h:124 */
#define CPI_REC_V1_DOUBLES 290
#define CPI_REC_OA     290  /* O_a [9]  d(alpha)/d(theta_k_lin)  (model 2)  CpiV2.h:62 */
#define CPI_REC_OB     299  /* O_b [9]  d(beta)/d(theta_k_lin)   (model 2)  CpiV2.h:63 */
#define CPI_REC_V2_DOUBLES 308

/* flags */
#define CPI_FLAG_IMU_AVG             1  /* CpiBase::imu_avg = true (CpiBase.h:95); each window then carries ONE extra
                                           trailing entry whose (w,a) are the "_1" arguments of the last step */
#define CPI_FLAG_ANALYTIC_JACOBIANS  2  /* model 2 only: state_transition_jacobians = false (CpiV2.h:58); default
                                           (flag clear) is the reference's default/true path (GraphSolver_IMU.cpp:100) */

/* error codes */
#define CPI_OK          0
#define CPI_EINVAL     -1   /* bad argument (NULL pointer, unknown model/dtype, negative count) */
#define CPI_ECUDA      -2   /* a CUDA runtime call failed; see cpi_last_error() */
#define CPI_ENODEVICE  -3   /* no CUDA device / not an sm_90 device */
#define CPI_ENOMEM     -4

/* ---- preintegration ---------------------------------------------------------------------------------------------- */

/*
 * Preintegrate n_windows independent windows.
 *   model          1 (CpiV1) or 2 (CpiV2)
 *   dtype          64 (fp64; samples/lin/records are double) or 32 (fp32 storage: float samples/lin/records,
 *                  see DESIGN.md for the mixed-precision rule)
 *   sample_offsets device int64[n_windows+1], entry index (not bytes) of each window's first entry in `samples`;
 *                  or NULL for uniform windows of `ns_uniform` steps laid out back to back.
 *                  Window w has  steps = offsets[w+1]-offsets[w]  (minus 1 if CPI_FLAG_IMU_AVG).  Device-resident offsets cannot
 *                  be validated by this entry point: a decreasing pair yields a zero-step window (the _host variant checks
 *                  its host copy and returns CPI_EINVAL instead).
 *   samples        device, CPI_SAMPLE_DOUBLES per entry.  The kernels stage every window's stream with 128-byte TMA bulk reads that
 *                  start at the 16-byte boundary at or below the window's first entry: `samples` must be 16-byte aligned (any
 *                  cudaMalloc / torch allocation is), so that no read begins before the buffer; reads never extend past the
 *                  last entry of the buffer (the tail of every window is read with plain loads).
 *   lin            device, CPI_LIN_DOUBLES per window
 *   sigmas         HOST double[4] = {sigma_w, sigma_wb, sigma_a, sigma_ab}  (CpiBase ctor, CpiBase.h:52-57)
 *   out_records    device, CPI_REC_V1_DOUBLES (model 1) or CPI_REC_V2_DOUBLES (model 2) per window
 * A window with zero steps yields the reference's freshly constructed object: R = I, everything else 0
 * (q_k2tau is uninitialised in the reference, CpiBase.h:102; this library writes [0 0 0 1]).
 */
int cpi_preintegrate_batch(int model, int dtype, int64_t n_windows,
                           const int64_t* sample_offsets, int64_t ns_uniform,
                           const void* samples, const void* lin, const double* sigmas, int flags,
                           void* out_records, void* stream);

/*
 * Continue n_windows preintegrations with MORE samples: `records` (device) holds, per window, the record left by an earlier
 * cpi_preintegrate_batch / _continue call and is updated in place -- the batched form of calling feed_IMU again on existing CpiV1 /
 * CpiV2 objects (feed_IMU accumulates into the object's fields, CpiBase.h:86, 99-124; every one of them is in the record).
 * `samples` / `sample_offsets` / `ns_uniform` describe the NEW samples only; lin, sigmas, flags must be those of the first call.
 * fp64: agrees with the one-shot call to rounding (~1e-15 relative; P_pp is re-split symmetrically).  dtype 32 continues from the
 * float-rounded record (the one-shot call carries the covariance state in fp64).  Default modes only (no CPI_FLAG_IMU_AVG, model 2
 * without CPI_FLAG_ANALYTIC_JACOBIANS): CPI_EINVAL otherwise.
 */
int cpi_preintegrate_batch_continue(int model, int dtype, int64_t n_windows,
                                    const int64_t* sample_offsets, int64_t ns_uniform,
                                    const void* samples, const void* lin, const double* sigmas, int flags,
                                    void* records, void* stream);

/* Same with HOST buffers: H2D + kernel + D2H, synchronous, through device buffers owned by the library; batches above 16 MB are
 * pipelined in up to 16 whole-window chunks (copy-in of chunk k+1 under the kernel of chunk k, copy-out under the next kernel); with a
 * uniform layout in the default fp64 modes the LAST windows of the batch (as many as take about one sample chain to transfer) travel
 * sample-major instead -- four strided segment copies, each followed by a continuation kernel over those windows -- so that their
 * chains of dependent samples run while the samples are still arriving and only a quarter of one chain is left behind the last byte
 * (results agree with the device entry point to rounding, ~1e-15; CPI_B200_HOST_WAVE="groups,segments[,head %]" overrides).  sample_offsets
 * is a HOST array.  The copies are cudaMemcpyAsync straight from / to the caller's buffers: PINNED buffers (cudaHostAlloc, or
 * cpi_host_register below) overlap with the kernels; pageable buffers are legal but the CUDA driver stages them synchronously, so
 * the pipeline degrades to copy-then-compute.  Calls from several host threads serialise on the library's scratch buffers. */
int cpi_preintegrate_batch_host(int model, int dtype, int64_t n_windows,
                                const int64_t* sample_offsets, int64_t ns_uniform,
                                const void* samples, const void* lin, const double* sigmas, int flags,
                                void* out_records);

/* Diagnostics of the last cpi_preintegrate_batch_host call of this process: host time until everything was enqueued, and until the
 * streams were drained (milliseconds).  Either pointer may be NULL. */
int cpi_host_last_timing(double* submit_ms, double* total_ms);

/* Pin / unpin a caller-owned host buffer for the *_host entry points (cudaHostRegister / cudaHostUnregister), for C callers that do
 * not link the CUDA runtime themselves.  Registering is expensive (~ms per 100 MB): do it once per buffer, not per call. */
int cpi_host_register(void* ptr, size_t bytes);
int cpi_host_unregister(void* ptr);

/* ---- merging records ------------------------------------------------------------------------------------------- */

/*
 * Merge consecutive model-1 records: the record of the interval k -> j from the records of k -> m and m -> j, what GTSAM's
 * PreintegratedImuMeasurements::mergeWith does.  Used to combine two IMU factors into one when the keyframe between them is dropped,
 * and to preintegrate ONE long window in parallel: cut it into S segments, preintegrate them as S windows of one CSR
 * cpi_preintegrate_batch call, merge each group of S records here (DESIGN.md "Merging records").
 *   model          1.  Model 2 returns CPI_EINVAL (its gravity removal depends on q_k_lin, which a merge would have to re-linearise).
 *   dtype          64, or 32 for float records and lin (the arithmetic is fp64 either way)
 *   group_offsets  device int64[n_groups+1] (the _host variant: HOST): group g is records group_offsets[g] .. group_offsets[g+1]-1,
 *                  in time order; or NULL for groups of `group_uniform` consecutive records.  Device-resident offsets cannot be
 *                  validated by this entry point: a decreasing pair yields an empty group (the _host variant returns CPI_EINVAL).
 *   records        device, CPI_REC_V1_DOUBLES per record
 *   lin            device, CPI_LIN_DOUBLES per RECORD: the linearisation point each record was preintegrated at
 *   out_records    device, one record per group; must not overlap `records`
 * The merged record is expressed at the linearisation point of the group's first record: every later record is first moved there
 * to first order (R <- Exp(J_q db_w) R, alpha/beta += J db_w + H db_a; its Jacobians and P are used as they are, as mergeWith does).
 * At equal linearisation points the means and the bias Jacobians are exact compositions (~1e-15 of the one-shot record) and P
 * agrees with the one-shot RK4 to its truncation error (~1e-10 relative).  An empty group yields the zero-step record (R = I,
 * q = [0 0 0 1], everything else 0); a group of one yields a bitwise copy of its record.  Long groups are merged as a pairwise tree
 * (logarithmic depth); one kernel launch per call.
 */
int cpi_merge_records(int model, int dtype, int64_t n_groups, const int64_t* group_offsets, int64_t group_uniform,
                      const void* records, const void* lin, void* out_records, void* stream);

/* Same with HOST buffers (H2D + kernel + D2H through device buffers owned by the library, synchronous).  group_offsets is a HOST
 * array, checked before anything reaches the device: non-decreasing, group_offsets[0] >= 0, group_offsets[n_groups] records in
 * `records` and `lin`. */
int cpi_merge_records_host(int model, int dtype, int64_t n_groups, const int64_t* group_offsets, int64_t group_uniform,
                           const void* records, const void* lin, void* out_records);

/*
 * Inclusive scan of consecutive model-1 records within groups: the record from a group's first keyframe to EVERY later boundary.
 * Used for dead reckoning of a chain from one anchor (cpi_predict_state_batch of the anchor state with every scanned record gives
 * every keyframe's state in one launch), and for records at intermediate times of a long window (cut it into S segments,
 * preintegrate them as one CSR batch, scan: a record at every segment boundary, computed in parallel).
 *   model, dtype, group_offsets, group_uniform, records, lin   as cpi_merge_records
 *   out_records    device, one record per INPUT record, indexed like `records`: for record i of group g (lo <= i < hi), out[i] is the
 *                  record of records lo .. i, at the linearisation point of record lo (every record moved there as the merge does it).
 *                  out[hi-1] is the group's cpi_merge_records result up to rounding; out[lo] is a bitwise copy of records[lo].  An
 *                  empty group writes nothing, and entries outside every group (before group_offsets[0]) are left untouched.  Must
 *                  not overlap `records`.
 *   workspace      device, cpi_scan_records_workspace(n_groups, n_records) bytes, n_records >= the records the groups span
 *                  (group_offsets[n_groups] - group_offsets[0], or n_groups * group_uniform).  Never NULL.
 * A segmented reduce-then-scan over chunks of 32 records: every group, however long, is spread over many CTAs, at a depth
 * logarithmic in the merges (DESIGN.md "Scanning records").  Allocates nothing and does not synchronise; about 2 log32(n) + 1
 * kernel launches for n records (device offsets: the bound of the records that fit in device memory, the levels the data does not
 * reach returning at once).
 */
int64_t cpi_scan_records_workspace(int64_t n_groups, int64_t n_records);
int cpi_scan_records(int model, int dtype, int64_t n_groups, const int64_t* group_offsets, int64_t group_uniform,
                     const void* records, const void* lin, void* out_records, void* workspace, void* stream);

/* Same with HOST buffers (H2D + kernels + D2H through device buffers owned by the library, synchronous); group_offsets is a HOST
 * array, checked as in cpi_merge_records_host. */
int cpi_scan_records_host(int model, int dtype, int64_t n_groups, const int64_t* group_offsets, int64_t group_uniform,
                          const void* records, const void* lin, void* out_records);

/* ---- factor evaluation ------------------------------------------------------------------------------------------- */

/*
 * Evaluate n IMU factors.  Factor f links states[idx_i[f]] -> states[idx_j[f]] (idx arrays may be NULL: then
 * idx_i[f] = f, idx_j[f] = f+1, the reference's chain X(k),X(k+1) -- GraphSolver_IMU.cpp:74) and uses
 * records[f] / lin[f] (the window's record and linearisation point, i.e. the factor's constructor arguments).
 *   e   device double[n*15]            residual  [2*q_r(0:3); bg_j-bg_i; betahat-beta; ba_j-ba_i; alphahat-alpha]
 *   H1  device double[n*225] col-major d e / d x_i   (may be NULL)
 *   H2  device double[n*225] col-major d e / d x_j   (may be NULL)
 * Unwhitened, exactly what evaluateError returns; the Gaussian::Covariance(P_meas) whitening lives in GTSAM.
 */
int cpi_imu_factor_eval_batch(int model, int64_t n_factors,
                              const double* states, const int64_t* idx_i, const int64_t* idx_j,
                              const double* records, const double* lin,
                              double* e, double* H1, double* H2, void* stream);

int cpi_imu_factor_eval_batch_host(int model, int64_t n_factors, int64_t n_states,
                                   const double* states, const int64_t* idx_i, const int64_t* idx_j,
                                   const double* records, const double* lin,
                                   double* e, double* H1, double* H2);

/*
 * Information-form linearisation of n factors (device pointers), the step GTSAM performs right after evaluateError with
 * the factor's noise model noiseModel::Gaussian::Covariance(P_meas) (gtsam/ImuFactorCPIv1.h:82, ImuFactorCPIv2.h:86):
 *     G11 = H1^T P^-1 H1, G12 = H1^T P^-1 H2, G22 = H2^T P^-1 H2  (15x15 column-major each),
 *     g1 = -H1^T P^-1 e, g2 = -H2^T P^-1 e  (15 each),  f = e^T P^-1 e      [HessianFactor convention: G, g = A^T b, f = b^T b]
 * P = records[f].P_meas; e / H1 / H2 as produced by cpi_imu_factor_eval_batch.  A factor whose covariance is not positive
 * definite (e.g. a zero-step window) gets NaN outputs (GTSAM throws there).  GTSAM itself is not in the reference tree
 * (bitbucket gtborg/gtsam @ c21186c), so this entry point is validated against a dense CPU solve only: PARITY UNPINNED.
 */
int cpi_imu_factor_hessian_batch(int model, int64_t n_factors, const double* records,
                                 const double* e, const double* H1, const double* H2,
                                 double* G11, double* G12, double* G22, double* g1, double* g2, double* f, void* stream);

/*
 * The explicitly whitened Jacobian form GTSAM's NoiseModelFactor::linearize produces with Gaussian::Covariance(P_meas):
 *     A1 = R_w H1,  A2 = R_w H2  (15x15 column-major each),  b = -R_w e  (15),   R_w = upper Cholesky factor of P_meas^-1.
 * PARITY UNPINNED (GTSAM is not in the reference tree); validated against numpy: A^T A = H^T P^-1 H, R_w upper triangular.
 */
int cpi_imu_factor_whiten_batch(int model, int64_t n_factors, const double* records,
                                const double* e, const double* H1, const double* H2,
                                double* A1, double* A2, double* b, void* stream);

/*
 * IMU-only chain x_0 - x_1 - ... - x_n (factor f links states f and f+1): what the smoother assembles and solves after the
 * linearisation (solvers/GraphSolver.cpp:202-203), on the device.
 *   cpi_imu_chain_assemble   scatter-add of the blocks of cpi_imu_factor_hessian_batch into the block-tridiagonal normal equations:
 *       D[k] (n+1 blocks 15x15) = G22[k-1] + G11[k] (+ prior_info0 on x_0) + damping,  E[k] (n blocks, block (k,k+1)) = G12[k],
 *       rhs[k] (15) = g2[k-1] + g1[k] (+ prior_rhs0).  prior_* may be NULL.  Damping as in GTSAM's LevenbergMarquardtParams:
 *       lambda I (diagonal_damping = 0, GTSAM's default) or lambda * clamp(diag D[k], 1e-6, 1e32) (diagonal_damping = 1, Marquardt).
 *       NOTE: an IMU-only chain anchored by one prior is numerically singular in fp64 beyond a few hundred keyframes with
 *       undamped / lambda-I normal equations (the drift modes carry ~1e-16 of the largest eigenvalue) -- for ANY elimination order;
 *       diagonal damping (or the camera factors of the real graph) restores a well-posed system (DESIGN.md section 5); so do priors
 *       on later states (position fixes: cpi_imu_state_priors_fold, DESIGN.md section 3g).
 *   cpi_imu_chain_solve      x = (that SPD block-tridiagonal matrix)^-1 rhs by block cyclic reduction (Cholesky on the 15x15 pivots):
 *       cpi_imu_chains_solve on one chain of n_states states, ~3 log2(n) + 2 kernel launches instead of an n-step sequential block
 *       recurrence.  `workspace`: device buffer of cpi_imu_chain_solve_workspace(n_states) bytes; with n_states = 1, E and the
 *       workspace may be NULL.  The step is then applied with cpi_retract_batch.
 * All pointers are DEVICE pointers.  PARITY UNPINNED; validated against banded / dense CPU solves of the same system.
 */
int cpi_imu_chain_assemble(int64_t n_factors, const double* G11, const double* G12, const double* G22,
                           const double* g1, const double* g2, double lambda, int diagonal_damping,
                           const double* prior_info0, const double* prior_rhs0,
                           double* D, double* E, double* rhs, void* stream);
int64_t cpi_imu_chain_solve_workspace(int64_t n_states);
int cpi_imu_chain_solve(int64_t n_states, const double* D, const double* E, const double* rhs,
                        double* x, void* workspace, void* stream);

/*
 * Many independent chains, and the fixed-lag smoother's marginalisation (BatchFixedLagSmoother, solvers/GraphSolver.h:93-97):
 * DESIGN.md section 3e.  fp64, DEVICE pointers, asynchronous on `stream`, no allocation.  Models 1 and 2 alike (only the
 * information blocks of cpi_imu_factor_hessian_batch are read).  PARITY UNPINNED (GTSAM is not in the reference tree); the numpy
 * statements of tests/test_marginalize.py are the references.
 *
 * Chain layout: chain_offsets = device int64[n_chains+1] with chain_offsets[0] = 0, chain c holding the states o[c] .. o[c+1]-1
 * of the concatenated states (at least one state each), or chain_offsets = NULL and chain_uniform (>= 1) states per chain.  Chain c
 * has S_c - 1 factors, stored back to back from factor index o[c] - c: its factor k links states o[c]+k and o[c]+k+1 (n_states -
 * n_chains factors in all).  A prior on a chain is (info[225] column-major, rhs[15], f), one of each per chain, in the HessianFactor
 * convention: cost = 1/2 (f - 2 rhs^T delta + delta^T info delta).  A device-resident layout cannot be inspected by these entry points.
 *
 *   cpi_imu_chain_marginalize   eliminates the first m = n_marg[c] states of every chain (n_marg: device int64[n_chains], or NULL
 *       and n_marg_uniform; 0 <= m < S_c) into a prior on state o[c] + m, at the linearisation point of the blocks, undamped:
 *           Lambda, eta, f = the prior (or 0); for each eliminated factor k:  M = Lambda + G11_k = L L^T,  Z = L^-1 G12_k,
 *           z = L^-1 (eta + g1_k);  Lambda <- G22_k - Z^T Z,  eta <- g2_k - Z^T z,  f <- f + f_k - z^T z
 *       out_info is exactly symmetric.  m = 0 copies the prior bit for bit (zeros without one).  A non-positive pivot, or a
 *       device-resident m out of range, gives NaN for that chain only.  G11 / G12 / G22 / g1 / g2 / f (the factors' constants) are
 *       all required whenever a factor may be read (n_marg given, or n_marg_uniform > 0); prior_info / prior_rhs: both or neither;
 *       prior_f, out_f may be NULL.  One warp per chain, sequential over its m factors: a long head (thousands of states) runs at
 *       sequential depth.
 *   cpi_imu_prior_at            the prior moved to the states x (one per prior): delta = local(lin_states, x), the exact inverse of
 *       cpi_retract_batch (rotation vector of q_x (x) q_lin^-1, JPL, w >= 0; differences for the other 12 entries; exactly 0 at
 *       x == lin_states), rhs_out = rhs - info delta, f_out = f - 2 rhs^T delta + delta^T info delta, info unchanged.  The Jacobian
 *       of local is taken as the identity, as LinearContainerFactor does (UNPINNED).  f, f_out may be NULL; rhs_out may be rhs.
 *   cpi_imu_chains_assemble     one block-tridiagonal system over all states: as cpi_imu_chain_assemble per chain (same damping),
 *       prior c on chain c's first state (prior_info / prior_rhs may be NULL), E exactly 0 at chain boundaries, E = n_states - 1
 *       blocks.  cpi_imu_chain_assemble is its n_chains = 1 case.  cpi_imu_chain_solve(n_states, D, E, rhs, ...) then solves every
 *       chain at once as one chain: the zero couplings keep the chains exactly decoupled -- PROVIDED EVERY CHAIN IS SPD: a NaN pivot
 *       of one chain spreads into its neighbours through 0 * NaN in the reduction (cpi_imu_chains_solve keeps it in its chain).
 */
int cpi_imu_chain_marginalize(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform,
                              const int64_t* n_marg, int64_t n_marg_uniform,
                              const double* G11, const double* G12, const double* G22, const double* g1, const double* g2, const double* f,
                              const double* prior_info, const double* prior_rhs, const double* prior_f,
                              double* out_info, double* out_rhs, double* out_f, void* stream);
int cpi_imu_prior_at(int64_t n, const double* info, const double* rhs, const double* f,
                     const double* lin_states, const double* states, double* rhs_out, double* f_out, void* stream);
int cpi_imu_chains_assemble(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform,
                            const double* G11, const double* G12, const double* G22, const double* g1, const double* g2,
                            double lambda, int diagonal_damping, const double* prior_info, const double* prior_rhs,
                            double* D, double* E, double* rhs, void* stream);

/*
 * Levenberg-Marquardt over many chains (DESIGN.md section 3f): the optimiser of BatchFixedLagSmoother (GraphSolver.cpp:202-203), run
 * for every chain at once with its own lambda and stopping state.  Chain layout and priors as above; fp64, DEVICE pointers,
 * asynchronous on `stream`, no allocation.  PARITY UNPINNED (GTSAM is not in the reference tree); the numpy statement of
 * tests/test_chains_lm.py is the reference.  Costs follow factor.chains_lm_step: cost = sum_k f_k + f'_prior, twice GTSAM's error.
 *
 * The rule (GTSAM's LevenbergMarquardtOptimizer with its defaults, useFixedLambdaFactor): one round, for every chain still RUNNING:
 *   linearise at x_c (cost_cur = sum f + the prior's f' moved to x_c); assemble with lambda_c; solve; retract to the candidate x~_c;
 *   cost_new at x~_c (cpi_imu_factor_cost_batch + cpi_imu_prior_at); model decrease m_c = sum_k delta_k^T (2 rhs_k - (H delta)_k) of the
 *   UNDAMPED system.  Then
 *     cost_cur or m_c not finite                        -> NONFINITE (the chain keeps its last accepted states)
 *     delta = 0 exactly                                 -> CONVERGED
 *     cost_new finite, m_c > 0, rho = (cost_cur - cost_new) / m_c > min_model_fidelity
 *                                                       -> accept: x_c = x~_c, lambda_c = max(lambda_c / lambda_factor, lambda_lower),
 *                                                          iterations += 1; CONVERGED if (cost_cur - cost_new) / 2 <= absolute_error_tol
 *                                                          or cost_cur - cost_new <= relative_error_tol * cost_cur, else MAX_ITERATIONS
 *                                                          once iterations = max_iterations
 *     otherwise                                         -> reject: LAMBDA_EXHAUSTED if lambda_c >= lambda_upper, else lambda_c *= lambda_factor
 *   and tries += 1 in every case.  A chain that is not RUNNING is never touched again (states, lambda, cost bitwise frozen).
 *
 *   cpi_imu_factor_cost_batch    (K9) f = e^T P_meas^-1 e of n factors at the states (indexing as cpi_imu_factor_eval_batch): the
 *       residual of evaluateError and one Cholesky + forward substitution, no e / H written; bitwise cpi_imu_factor_hessian_batch's f.
 *       A factor whose P_meas is not positive definite gets NaN.
 *   cpi_imu_chains_cost_sum      cost[c] = the sum of f (device double[n_states - n_chains], one per factor, chains back to back) over
 *       chain c's factors, in a fixed order (no atomics: the same bits on every run).  Layout as cpi_imu_chains_assemble.
 *   cpi_imu_chains_assemble_lm   cpi_imu_chains_assemble with lambda[n_chains] (device) per chain; damp (device double[n_states*15],
 *       may be NULL) receives the diagonal the damping added.
 *   cpi_imu_chains_solve         block cyclic reduction over n_states = the layout's state count, with every coupling between two
 *       chains structurally absent (not loaded, not multiplied, written as exact 0): a NaN stays in its chain, and on SPD input the
 *       result is cpi_imu_chain_solve's (all states one chain) bit for bit.  workspace: cpi_imu_chains_solve_workspace(n_chains, n_states)
 *       bytes.
 *   cpi_imu_chains_lm_update     the decision above for every RUNNING chain: f_cur / f_new per factor, prior_f_cur / prior_f_new per chain
 *       (NULL: no prior), rhs / D / E / damp / delta of the round, states_new the candidate states; writes lambda, cost, status,
 *       iterations, tries, copies states_new into `states` for the accepted chains, and sets *any_running = 1 (may be NULL; the caller
 *       zeroes it) if a chain is still RUNNING.  Per-chain sums in a fixed order (no atomics).  workspace: cpi_imu_chains_lm_workspace
 *       (n_states) bytes.  Parameters are checked on the host: lambda_factor > 1, 0 <= lambda_lower <= lambda_upper, tolerances >= 0,
 *       0 <= min_model_fidelity < 1, max_iterations >= 1; CPI_EINVAL otherwise, before the device is touched.
 */
#define CPI_LM_RUNNING           0
#define CPI_LM_CONVERGED         1
#define CPI_LM_MAX_ITERATIONS    2
#define CPI_LM_LAMBDA_EXHAUSTED  3
#define CPI_LM_NONFINITE         4
typedef struct cpi_lm_params {
    double lambda_factor;        /* 10    */
    double lambda_lower;         /* 0     */
    double lambda_upper;         /* 1e5   */
    double min_model_fidelity;   /* 1e-3  */
    double absolute_error_tol;   /* 1e-5  (on GTSAM's error, half the cost) */
    double relative_error_tol;   /* 1e-5  */
    int64_t max_iterations;      /* 100   */
} cpi_lm_params;
int cpi_imu_factor_cost_batch(int model, int64_t n_factors, const double* states, const int64_t* idx_i, const int64_t* idx_j,
                              const double* records, const double* lin, double* f, void* stream);
int cpi_imu_chains_cost_sum(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform, const double* f, double* cost, void* stream);
int cpi_imu_chains_assemble_lm(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform,
                               const double* G11, const double* G12, const double* G22, const double* g1, const double* g2,
                               const double* lambda, int diagonal_damping, const double* prior_info, const double* prior_rhs,
                               double* D, double* E, double* rhs, double* damp, void* stream);
int64_t cpi_imu_chains_solve_workspace(int64_t n_chains, int64_t n_states);
int cpi_imu_chains_solve(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform, int64_t n_states,
                         const double* D, const double* E, const double* rhs, double* x, void* workspace, void* stream);
int64_t cpi_imu_chains_lm_workspace(int64_t n_states);
int cpi_imu_chains_lm_update(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform, int64_t n_states,
                             const cpi_lm_params* params, const double* f_cur, const double* prior_f_cur, const double* f_new,
                             const double* prior_f_new, const double* rhs, const double* D, const double* E, const double* damp,
                             const double* delta, const double* states_new, double* states, double* lambda, double* cost,
                             int32_t* status, int32_t* iterations, int32_t* tries, int32_t* any_running, void* workspace, void* stream);

/*
 * Priors on any state of many chains (DESIGN.md section 3g): GTSAM's PriorFactor / the reference's JPLNavStatePrior on any keyframe --
 * absolute position or attitude fixes, zero-velocity updates, anchors every N keyframes.  fp64, DEVICE pointers, asynchronous on
 * `stream`, no allocation.  PARITY UNPINNED (the convention is the library's own); tests/test_state_priors.py holds the numpy statement.
 *
 * A state prior i is (s_i, info_i[225] column-major, rhs_i[15], f_i, lin_i[16]) in the convention of the chain prior above: s_i indexes
 * the concatenated states of the chain layout, cost = 1/2 (f - 2 rhs^T delta + delta^T info delta) with delta = local(lin_i, x_{s_i}).
 * It is moved to the current states by cpi_imu_prior_at (n = the number of state priors), Jacobian of local taken as the identity.
 * A measurement x_bar with information W is (info = W, rhs = 0, f = 0, lin = x_bar): cost delta^T W delta.  A partial measurement
 * (position only, velocity only) uses a PSD W that is zero outside its blocks.  Limits:
 *   - lin_i must be a finite state with a unit quaternion even where W is zero: delta is formed in full, and 0 * NaN poisons.
 *   - With the identity Jacobian, a strong ATTITUDE prior with a large residual converges to a point off the true optimum by second
 *     order in that residual.  Position, velocity and bias priors are exact (local is a difference there).
 *
 *   cpi_imu_state_priors_fold   adds the moved priors (sp_info, sp_rhs = rhs', sp_f = f') IN PLACE into blocks the assembly, the
 *       solves, K8 and the LM decision already read.  For a prior on state k of chain c (states o[c] .. o[c+1]-1):
 *           k not the chain's last state                 -> G11, g1, f of the factor to its right (index k - c)
 *           k the last state of a chain of >= 2 states   -> G22, g2, f of the factor to its left  (index k - 1 - c)
 *           k the only state of its chain                -> the chain prior prior_info, prior_rhs, prior_f of chain c
 *       Each 15x15 block and rhs segment receives the priors of one state; the f of a chain's last factor receives those of its
 *       two states (the left state's first, one warp adding both).  The priors are sorted by state: sp_offsets (device int64
 *       [n_states+1], CSR) gives state k the priors sp_offsets[k] .. sp_offsets[k+1]-1, added one after the other in that order
 *       (no atomics: the same bits on every run).  Folded before the assembly, a prior sits in diag(D) before the damping, where
 *       Marquardt's diagonal damping and the model decrease of cpi_imu_chains_lm_update see it.  K8 eliminates states that are never
 *       the last of their chain, so the priors of eliminated states land in exactly the G11 blocks it consumes.
 *       sp_info / sp_rhs: both or neither; neither is the f-only fold (sp_f into f / prior_f only: the candidate's cost in LM).
 *       sp_f may be NULL.  A NULL target receives nothing: pass it only where no prior can land (for example G22 / g2 when no prior
 *       sits on a chain's last state); with chain_uniform = 1 the chain-prior targets are required.  The chain is found by binary
 *       search on a device-resident layout, which is never read on the host.
 */
int cpi_imu_state_priors_fold(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform, const int64_t* sp_offsets,
                              const double* sp_info, const double* sp_rhs, const double* sp_f, double* G11, double* G22, double* g1,
                              double* g2, double* f, double* prior_info, double* prior_rhs, double* prior_f, void* stream);

/*
 * Robust losses on state priors (DESIGN.md section 3h): GTSAM's noiseModel::Robust (Huber, Cauchy) around a prior's noise model, so
 * that an outlying fix (GNSS multipath, a false zero-velocity detection, a bad anchor) pulls with a bounded or vanishing weight
 * instead of quadratically.  fp64, DEVICE pointers, asynchronous on `stream`, no allocation.  PARITY UNPINNED; tests/test_robust_priors.py
 * holds the numpy statement.
 *
 * A robust prior must be a MEASUREMENT prior (rhs = 0, f = 0): after cpi_imu_prior_at its f' is s = delta^T W delta, the whitened
 * squared residual.  A prior with a nonzero rhs or f (a marginal prior, for example) has no residual to robustify.  With the library's
 * cost convention (a Gaussian prior costs s, twice GTSAM's error) a robust prior costs c(s) = 2 rho(sqrt s), rho GTSAM's mEstimator
 * residual, and enters the linear system with the IRLS weight w(s) = dc/ds (what noiseModel::Robust::WhitenSystem applies):
 *     CPI_LOSS_GAUSSIAN   c = s                                            w = 1
 *     CPI_LOSS_HUBER, k   c = s if s <= k^2, else 2 k sqrt(s) - k^2        w = 1 if s <= k^2, else k / sqrt(s)
 *     CPI_LOSS_CAUCHY, k  c = k^2 log1p(s / k^2)                           w = 1 / (1 + s / k^2)
 * k is in whitened units (standard deviations); it must satisfy 0 < k^2 < inf, and is ignored for CPI_LOSS_GAUSSIAN.  A Gaussian prior
 * and a Huber inlier are copied bit for bit.  An unknown code or an invalid k gives NaN weight and cost for that prior (its chain
 * then ends CPI_LM_NONFINITE in LM; no other prior is touched).
 *
 *   cpi_imu_state_priors_robust   (info, rhs, f) -> (w info, w rhs, c(s)) with s = f, per prior: info / rhs / f as cpi_imu_prior_at
 *       leaves them (rhs', f').  loss: int32 [n], loss_k: double [n].  info_out / rhs_out: both or neither; neither is the f-only pass
 *       (the candidate's cost in LM).  rhs_out may alias rhs and f_out may alias f; info_out receives the weighted info, so the
 *       caller's info stays constant.  One warp per prior, no atomics: the same bits on every run.  Then cpi_imu_state_priors_fold
 *       adds the weighted priors unchanged.  In LM the weight is recomputed at the states of every round; in marginalisation it is
 *       frozen at the blocks' linearisation point, as GTSAM linearises a robust factor it marginalises.
 */
#define CPI_LOSS_GAUSSIAN        0
#define CPI_LOSS_HUBER           1
#define CPI_LOSS_CAUCHY          2
int cpi_imu_state_priors_robust(int64_t n, const int32_t* loss, const double* loss_k, const double* info, const double* rhs, const double* f,
                                double* info_out, double* rhs_out, double* f_out, void* stream);

/*
 * Measurements of one state that depend on its attitude (DESIGN.md section 3l): a GNSS antenna at a lever arm, body-frame velocity
 * (odometer, DVL, non-holonomic constraint), a known global direction seen in the body frame (magnetometer, gravity at rest).  They
 * enter the solver as moved state priors relinearised at every round, so their Jacobian is exact where a state prior's is taken as I.
 * fp64, DEVICE pointers, asynchronous on `stream`, no allocation.  PARITY UNPINNED (GTSAM's GPSFactor with a lever arm and Pose3
 * attitude factors are the nearest); tests/measurement_ref.py holds the numpy statement.
 *
 * Measurement i is (state_idx[i], kind[i], z[3i..], sqrt_info[9i..] the column-major S with Lambda = S^T S, aux[3i..]) on the state
 * x = states[state_idx[i]] (JPL quaternion, C = C(q) global to IMU, tangent [dtheta, b_g, v, b_a, p] of cpi_retract_batch):
 *     CPI_MEAS_POSITION       h = p + C^T aux    H_theta = -C^T [aux]x   H_p = I     aux: the lever arm in the IMU frame (0: position)
 *     CPI_MEAS_VELOCITY_BODY  h = C v            H_theta = [C v]x        H_v = C     aux: not read
 *     CPI_MEAS_DIRECTION      h = C aux          H_theta = [C aux]x                  aux: the known vector in the global frame
 * r = h(x) - z, whitened A = S H (3x15) and b = S r.  S may be singular (a non-holonomic constraint weighs the lateral and vertical
 * axes only).  An unknown kind gives NaN blocks for that measurement only (its chain ends CPI_LM_NONFINITE in LM).
 *
 *   cpi_imu_measurements_linearize   (info, rhs', f') per measurement in the convention of the state priors (cost f - 2 rhs^T xi +
 *       xi^T info xi at xi = 0 the given state): info = A^T A (device double[n*225], column-major, exactly symmetric), rhs' = -A^T b
 *       (double[n*15]), f' = b^T b (double[n]), the whitened squared residual s that cpi_imu_state_priors_robust reads.  info and rhs:
 *       both or neither; neither is the f-only pass (LM's candidate cost), whose f is bitwise the full pass's.  Then
 *       cpi_imu_state_priors_robust and cpi_imu_state_priors_fold take the blocks unchanged.  Lane-parallel stores, no atomics: the
 *       same bits on every run.  state_idx (device int64) is not checked: indices must lie in the states array.
 *   CPI_EINVAL for n < 0, n > 2^31, a NULL required pointer, or an output equal to an input or another output.  n = 0 launches nothing.
 */
#define CPI_MEAS_POSITION        1
#define CPI_MEAS_VELOCITY_BODY   2
#define CPI_MEAS_DIRECTION       3
int cpi_imu_measurements_linearize(int64_t n, const int32_t* kind, const int64_t* state_idx, const double* states, const double* z,
                                   const double* sqrt_info, const double* aux, double* info /* or NULL */, double* rhs /* or NULL */,
                                   double* f, void* stream);

/*
 * Marginal covariances of many chains (DESIGN.md section 3j): what GTSAM's Marginals / BatchFixedLagSmoother::marginalCovariance give
 * for every keyframe of a window, for every chain at once.  fp64, DEVICE pointers, asynchronous on `stream`, no allocation.  PARITY
 * UNPINNED; tests/test_chain_marginals.py holds the numpy statement of the level walk.
 *
 *   cpi_imu_chains_marginals   the diagonal blocks and the blocks next to them of A^-1, A = tridiag(E^T, D, E) the system of
 *       cpi_imu_chains_solve (same layout, same validation, same error codes): cov[k] = (A^-1)_{k,k} (device double[n_states*225],
 *       column-major, exactly symmetric) and, unless cross is NULL, cross[o[c] - c + j] = (A^-1)_{o[c]+j, o[c]+j+1} for j < S_c - 1
 *       (device double[(n_states - n_chains)*225], the factors' order).  Selected inversion of the block cyclic reduction: the forward
 *       phase of cpi_imu_chains_solve on a zero right-hand side, then one launch per level top-down (3 log2(n_states) + 2 launches in
 *       all).  Every coupling between two chains is structurally absent: a chain that is not SPD gets NaN blocks, and only that chain.
 *       workspace: cpi_imu_chains_marginals_workspace(n_chains, n_states) bytes.
 *   The call inverts whatever system it is given.  A marginal covariance needs the UNDAMPED system (lambda = 0) at the estimate:
 *   factor.chains_marginals assembles it.  Long IMU-only chains without priors on later states are numerically singular in fp64
 *   (DESIGN.md sections 3e, 3f): their covariances are meaningless (finite or not), as is any fp64 inverse of that system.
 */
int64_t cpi_imu_chains_marginals_workspace(int64_t n_chains, int64_t n_states);
int cpi_imu_chains_marginals(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform, int64_t n_states,
                             const double* D, const double* E, double* cov, double* cross, void* workspace, void* stream);

/*
 * Re-preintegration of the windows whose bias estimate left the records' linearisation point (DESIGN.md section 3i): the
 * re-integration VINS-Mono and OKVIS run between solves, on the device.  A factor corrects its record to the bias of its state i
 * only to first order (J_q, J_a, J_b, H_a, H_b; model 2 also O_a, O_b in the orientation), which limits accuracy once the
 * estimate is 1e-2 .. 1e-1 rad/s from `lin`.  Intended use, between solves: chains_lm -> relinearize -> if any: chains_lm again.
 * fp64, DEVICE pointers except sigmas and n_relinearized, no allocation.  PARITY UNPINNED (the rule is the library's own);
 * tests/test_relinearize.py holds the numpy statement.
 *
 *   n_factors        factor k has records[k] and lin[k] and reads the bias of state idx_i[k] (idx_i NULL: state k, as
 *                    cpi_imu_factor_eval_batch); device indices are not checked
 *   sample_offsets / ns_uniform / samples / sigmas / flags
 *                    factor k's window in the layout of cpi_preintegrate_batch, and the sigmas and flags the records were
 *                    preintegrated with (every combination cpi_preintegrate_batch accepts; an imu_avg window's trailing entry is in
 *                    its range)
 *   tol_bw, tol_ba, tol_theta   rad/s, m/s^2, rad; each >= 0, +inf disables that test; tol_theta is read by model 2 only
 * Factor k is SELECTED when  |bg_i - lin_bw|^2 > tol_bw^2  or  |ba_i - lin_ba|^2 > tol_ba^2  or (model 2)  |theta|^2 > tol_theta^2,
 * theta the rotation part of local(lin_q, q_i) (cpi_imu_prior_at's local); squared norms summed x, y, z in that order in fp64,
 * without contraction.  A NaN in what the rule reads (the state's biases, model 2 its quaternion) leaves the factor unselected, so
 * a chain that LM ended non-finite keeps its records.  For a selected factor
 *     lin[k]     <- [bg_i, ba_i, q_lin', grav]   q_lin' = q_i (model 2), unchanged (model 1); gravity is never changed
 *     records[k] <- the record cpi_preintegrate_batch gives for the window at the new lin, with the same sigmas and flags
 * Unselected records and lin entries are not written.  relinearized (device int32 [n_factors], may be NULL) receives the 0/1 mask,
 * *n_relinearized (host, may be NULL) the count.
 *
 * Launches: selection (one thread per factor), a scan of the per-CTA totals, the stable compaction (integer sums, no atomics: the
 * same bits on every run); then ONE 16-byte device-to-host read of the selected windows and entries and a synchronise of
 * `stream`, the call's only host synchronisation (the re-preintegration's grid depends on it); with none selected nothing more is
 * launched.  Otherwise: a gather of the selected windows' samples into a compact 16-byte aligned CSR batch, the unchanged K1/K2
 * launch of cpi_preintegrate_batch on it, a scatter of the records and lin back into their slots.
 *
 * workspace   device, 16-byte aligned, cpi_imu_records_relinearize_workspace(model, n_factors, n_entries) bytes with n_entries >=
 *             every entry a window of the call spans: the worst case, every window selected.  That is 8 RD + 124 bytes per factor
 *             (2 444 for model 1, 2 588 for model 2; RD the record doubles), 32 bytes per 256 factors, 56 bytes per entry, and at most
 *             136 bytes more (alignment and the totals).  The compact samples dominate: 10 000 chains x 30 states x 200 samples need about 3.3 GB.
 *
 * Out of scope: fp32-storage records; records built by cpi_merge_records or cpi_scan_records (re-integration is one-shot over the
 * window's full sample range, so the result differs from a merged record by the RK4 truncation of DESIGN.md section 3b); a cap on
 * the windows re-integrated per call; relinearising inside an LM round (it would change the cost between the linearisation and the
 * acceptance test).
 */
int64_t cpi_imu_records_relinearize_workspace(int model, int64_t n_factors, int64_t n_entries);
int cpi_imu_records_relinearize(int model, int64_t n_factors, const double* states, const int64_t* idx_i,
                                const int64_t* sample_offsets, int64_t ns_uniform, const double* samples,
                                const double* sigmas /* host[4] */, int flags,
                                double tol_bw, double tol_ba, double tol_theta,
                                double* lin /* in/out */, double* records /* in/out */,
                                int32_t* relinearized /* device [n_factors] 0/1, may be NULL */,
                                int64_t* n_relinearized /* host, may be NULL */,
                                void* workspace, void* stream);

/* ---- callers either side of the factor ("next" rows) ----------------------------------------------------------------- */

/* x_{k+1} prediction from x_k and a record: getpredictedstate_v1/_v2 (GraphSolver_IMU.cpp:263-307).
 * states_k / states_k1: device, CPI_STATE_DOUBLES per window. */
int cpi_predict_state_batch(int model, int64_t n, const double* states_k, const double* records, const double* lin,
                            double* states_k1, void* stream);

/*
 * Prediction with covariance: the state x_{k+1} predicted from an anchor x_k and a record, and its 15x15 error covariance, for
 * n windows at once.  Errors live in the tangent space of JPLNavState::retract (cpi_retract_batch; the factor Jacobians' convention).
 * With H1, H2 the Jacobians cpi_imu_factor_eval_batch gives at (x_k, x_{k+1}):
 *     A = -H2^-1 H1,  B = H2^-1,  cov_k1 = A cov_k A^T + B P_meas B^T,  cross = (A cov_k)^T  (= cov_k A^T, the x_k - x_{k+1} block)
 * the linearisation of e(x_k, x_{k+1}) = 0 with the factor's own noise model (covariance P_meas).  One step of an EKF / MSCKF
 * propagation, or, with every window anchored at one state and the records of cpi_scan_records, dead reckoning of a whole chain with
 * its uncertainty in one launch (DESIGN.md "Propagating the covariance").
 *   model      1 or 2 (fp64)
 *   states_k   device, CPI_STATE_DOUBLES per anchor entry;  cov_k  device, 225 doubles (column-major 15x15) per anchor entry,
 *              symmetric (it is read whole)
 *   anchor     device int64[n], or NULL: window i starts from entry anchor[i] of states_k / cov_k (NULL: entry i).  Device-resident
 *              indices cannot be validated by this entry point (the _host variant checks them)
 *   records    device, one record per window;  lin  device, CPI_LIN_DOUBLES per window
 *   states_k1  device, CPI_STATE_DOUBLES per window: bit for bit what cpi_predict_state_batch writes for the same inputs
 *   cov_k1     device, 225 per window, exactly symmetric
 *   cross      device, 225 per window, or NULL
 * Outputs must not overlap inputs.  One kernel launch; does not synchronise.
 */
int cpi_propagate_batch(int model, int64_t n, const double* states_k, const double* cov_k, const int64_t* anchor,
                        const double* records, const double* lin, double* states_k1, double* cov_k1, double* cross, void* stream);

/* Same with HOST buffers (H2D + kernel + D2H through device buffers owned by the library, synchronous).  states_k / cov_k hold
 * n_anchors entries; anchor (HOST, may be NULL: then n_anchors >= n) is checked against n_anchors before anything reaches the device. */
int cpi_propagate_batch_host(int model, int64_t n, int64_t n_anchors, const double* states_k, const double* cov_k,
                             const int64_t* anchor, const double* records, const double* lin,
                             double* states_k1, double* cov_k1, double* cross);

/* JPLNavState::retract (JPLNavState.cpp:37-71): states_out[i] = states[i] (+) xi[i], xi = 15 doubles each. */
int cpi_retract_batch(int64_t n, const double* states, const double* xi, double* states_out, void* stream);

/*
 * Measurement update of n filters by direct state fixes, with chi-square gating (DESIGN.md section 3k): the update step of the filter
 * that cpi_propagate_batch predicts.  fp64, DEVICE pointers, asynchronous on `stream`, one kernel launch, no allocation, no host
 * synchronisation.  PARITY UNPINNED (there is no reference filter); tests/update_ref.py holds the numpy statement.
 *
 * Filter i has the state x = states[i] (CPI_STATE_DOUBLES) and the error covariance S = cov[i] (225, column-major, SPD; the tangent
 * space of cpi_retract_batch, as cpi_propagate_batch).  The fix is (W = meas_info[i], x_bar = meas_states[i]) in the convention of the
 * state priors above: W PSD column-major 15x15, zero outside the blocks it measures; residual delta = local(x_bar, x') at the updated
 * state, Jacobian taken as I.  With d = local(x_bar, x) and x' = retract(x, xi) the update minimises xi^T S^-1 xi + (d+xi)^T W (d+xi):
 *     xi = -(S^-1 + W)^-1 W d,   S+ = (S^-1 + W)^-1,   x+ = retract(x, xi),
 *     gamma = (d+xi)^T W (d+xi) + xi^T S^-1 xi      (= d^T (S + W^-1)^-1 d for an invertible W: the normalised innovation squared)
 * computed in square-root form, S^-1 never formed (S's blocks span about ten orders of magnitude):
 *     S = L L^T,  C = chol(I + L^T W L),  u = L^T W d,  v = C^-1 u,  xi = -L C^-T v,  S+ = M M^T with M = L C^-T,
 *     gamma = (d+xi)^T W (d+xi) + |C^-T v|^2.
 *   gate      device double[n], or NULL (every fix applied).  The fix is SKIPPED when gamma > gate[i]: states_out[i] and cov_out[i] are
 *             then bit-for-bit copies of the inputs, applied[i] = 0.  A NaN gamma is not > gate: it is applied, and its NaN shows in
 *             that filter's outputs.  +inf applies every finite gamma: the outputs are bitwise those of a NULL gate.  gamma does not
 *             depend on the gate: a chi-square quantile for the rank of W is the usual threshold.
 *   states_out / cov_out   device, as states / cov; cov_out exactly symmetric (lower triangle computed and mirrored)
 *   nis       device double[n] (gamma, also for a skipped fix), or NULL;   applied  device int32[n] 0/1, or NULL
 * One fix per filter per call: fixes that arrive together on disjoint blocks (position and velocity) form one (W, x_bar); a second
 * fix on the same block is a second call.  Position, velocity and bias fixes are exact under the identity Jacobian; an attitude fix
 * carries the second-order limit of the state priors.  x_bar must be a finite state with a unit quaternion even where W is zero.
 * Sharpness: I + L^T W L has the condition number 1 + lambda_max(W S); in fp64 its Cholesky loses digits as that grows, and a pivot
 * that is not positive (NaN outputs) appears near 1e17, a fix some 3e8 times sharper than the prior in standard deviations.  The
 * precision gate covers lambda_max(W S) <= 1e12.
 * A cov that is not SPD, or a NaN in W, gives NaN outputs for that filter only (one warp per filter).  A NaN in x_bar or x gives a
 * NaN state and gamma (cov_out does not depend on d).  CPI_EINVAL for n < 0, a NULL required pointer, or an output equal to an input
 * or to another output; outputs must not overlap inputs.  n = 0 launches nothing.
 */
int cpi_state_update_batch(int64_t n, const double* states, const double* cov, const double* meas_info, const double* meas_states,
                           const double* gate, double* states_out, double* cov_out, double* nis, int32_t* applied, void* stream);

/*
 * The same update by the measurements of cpi_imu_measurements_linearize (DESIGN.md section 3l; kinds CPI_MEAS_*): the filter's
 * update by GNSS at a lever arm, body-frame velocity and known directions.  fp64, DEVICE pointers, asynchronous on `stream`, one
 * kernel launch, no allocation, no host synchronisation.  PARITY UNPINNED; tests/measurement_ref.py holds the numpy statement.
 *
 * Filter i (states[i], cov[i] as cpi_state_update_batch) takes measurements meas_offsets[i] .. meas_offsets[i+1]-1 (device int64
 * [n+1], CSR, non-decreasing, not checked) of kind / z / sqrt_info / aux (as cpi_imu_measurements_linearize, without state_idx), all
 * linearised at x = states[i] (one EKF step).  With A_j, b_j their whitened rows at x, in square-root form:
 *     Sigma = L L^T,  B_j = A_j L,  C = chol(I + sum_j B_j^T B_j),  w = -C^-T C^-1 sum_j B_j^T b_j,  xi = L w,
 *     Sigma+ = M M^T with M = L C^-T (exactly symmetric),  x+ = retract(x, xi),  gamma = sum_j |b_j + A_j xi|^2 + |w|^2
 * gamma is the normalised innovation squared r^T (H Sigma H^T + Lambda^-1)^-1 r for invertible Lambda, summed as squares.
 *   gate      as cpi_state_update_batch: gamma > gate[i] skips the update (bit-for-bit copies, applied[i] = 0)
 *   nis, applied   as cpi_state_update_batch
 * A filter without measurements is copied bit for bit with gamma = 0 and applied = 1.  Sharpness: I + sum B^T B has the condition
 * number 1 + lambda_max(W Sigma), W = sum_j A_j^T A_j, with K10's limit (pivots fail near 1e17).  A cov that is not SPD, or a NaN in a
 * measurement's S or kind, gives NaN outputs for that filter only; a NaN in z a NaN state and gamma (cov_out does not depend on z).
 * CPI_EINVAL for n < 0, a NULL required pointer, or an output equal to an input or another output.  n = 0 launches nothing.
 */
int cpi_state_update_measurements_batch(int64_t n, const double* states, const double* cov, const int64_t* meas_offsets,
                                        const int32_t* kind, const double* z, const double* sqrt_info, const double* aux,
                                        const double* gate, double* states_out, double* cov_out, double* nis, int32_t* applied,
                                        void* stream);

/*
 * The iterated update by the same measurements, with robust losses (DESIGN.md section 3m): the iterated EKF, for filters that start
 * or recover with a poor attitude, where the single linearisation of cpi_state_update_measurements_batch lands away from the posterior
 * mode and reports a covariance taken at the wrong attitude.  fp64, DEVICE pointers, asynchronous on `stream`, one kernel launch, no
 * allocation, no host synchronisation.  PARITY UNPINNED; tests/update_iter_ref.py holds the numpy statement.
 *
 * Filter i (states[i] = x_hat, cov[i] = Sigma = L L^T, measurements meas_offsets[i] .. meas_offsets[i+1]-1 as
 * cpi_state_update_measurements_batch) runs undamped Gauss-Newton on  |L^-1 local(x_hat, x)|^2 + sum_j rho_j(|b_j(x)|^2)  with the
 * prior's Jacobian taken as I (the state priors' convention): the iterates of cpi_imu_chains_* on a single-state chain at lambda = 0.
 * rho_j is measurement j's loss (loss[j], loss_k[j] as cpi_imu_state_priors_robust) and om_j its IRLS weight at |b_j|^2.  From
 * x_0 = x_hat, for t = 0, 1, ...:
 *     d_t = local(x_hat, x_t) (0 at t = 0),  A_j, b_j at x_t,  B_j = sqrt(om_j) A_j L,  b'_j = sqrt(om_j) (b_j - A_j d_t),
 *     C = chol(I + sum_j B_j^T B_j),  w = C^-T C^-1 sum_j B_j^T b'_j,  eps = -L w,  delta = eps - d_t,  x_{t+1} = retract(x_t, delta)
 * stopping when max_k |delta_k| <= tol sqrt(Sigma_kk) (the step in prior standard deviations) or after max_iterations linearisations.
 *   states_out  x_T, the last iterate;   cov_out  M M^T with M = L C^-T of the last linearisation, its weights frozen (exactly symmetric)
 *   nis       gamma = sum_j om_j |b_j + A_j eps_0|^2 + |w_0|^2 of the FIRST linearisation (weights at x_hat); K11's gamma without a loss
 *   gate      device double[n] or NULL: gamma > gate[i] is decided before iterating and skips the update (bit-for-bit copies, status 0);
 *             a NaN gamma is not gated
 *   status    device int32[n] or NULL: 0 gated, 1 converged, 2 stopped at max_iterations without meeting tol
 *   iterations  device int32[n] or NULL: the linearisations taken (1 for a gated filter)
 *   loss, loss_k  device int32[M] CPI_LOSS_* and double[M] thresholds, both or neither (neither: every measurement Gaussian)
 * A filter without measurements is copied bit for bit with gamma = 0, status 1 and 0 iterations.  tol = +inf takes exactly one
 * iteration, cpi_state_update_measurements_batch without a loss (to rounding); tol = 0 takes exactly max_iterations unless a step is exactly
 * zero.  A cov that is not SPD, or a NaN in a measurement, gives NaN outputs for that filter only (it stops with status 2).
 * CPI_EINVAL for n < 0, max_iterations < 1, a NaN or negative tol, only one of loss / loss_k, a NULL required pointer, or an output
 * equal to an input or another output.  n = 0 launches nothing.
 */
int cpi_state_update_measurements_iterated_batch(int64_t n, const double* states, const double* cov, const int64_t* meas_offsets,
                                                 const int32_t* kind, const double* z, const double* sqrt_info, const double* aux,
                                                 const int32_t* loss /* or NULL */, const double* loss_k /* or NULL */,
                                                 const double* gate, int max_iterations, double tol, double* states_out, double* cov_out,
                                                 double* nis, int32_t* status, int32_t* iterations, void* stream);

/* ---- window builder (host) ------------------------------------------------------------------------------------------------------ */

/*
 * Cut one IMU stream into the windows the reference preintegrates, one per update (camera) time: the loop of
 * GraphSolver::createimufactor_cpi_v1/_v2 (solvers/GraphSolver_IMU.cpp:50-69, 105-124) incl. the partial tail step and the
 * rewrite of the front stamp, fed as SimulationLoader::execute_publishing delivers the messages (sim/SimulationLoader.cpp:214-290:
 * the IMU reading first at equal stamps) and initialised as GraphSolver::trytoinitalize does (solvers/GraphSolver.cpp:264, 357: the
 * first update that finds >= imu_wait queued readings emits no window and keeps only the newest reading; imu_wait = 0: no such phase).
 *   t[n_imu] seconds (non-decreasing), w / a [n_imu * 3], update_times[n_updates] (non-decreasing) -- all HOST arrays
 *   samples   HOST, capacity cap_entries entries of CPI_SAMPLE_DOUBLES (may be NULL to count only)
 *   offsets   HOST int64[n_updates + 1]; window k is entries offsets[k] .. offsets[k+1]-1 (CSR layout of cpi_preintegrate_batch)
 * Returns the number of windows (<= n_updates) or a negative CPI_E* code; *n_entries receives the number of entries.
 */
int64_t cpi_cut_windows(int64_t n_imu, const double* t, const double* w, const double* a,
                        int64_t n_updates, const double* update_times, int64_t imu_wait,
                        int64_t cap_entries, double* samples, int64_t* offsets, int64_t* n_entries);

/* ---- multi-GPU: one process per GPU, window batches sharded over the ranks ------------------------------------------------ */

/*
 * Windows share nothing but the four sigmas (the reference constructs a fresh preintegrator per factor,
 * solvers/GraphSolver_IMU.cpp:43), so a batch shards contiguously: rank r preintegrates its n_local windows and the only
 * exchange is ONE in-place all-gather of the fixed-size records (NCCL, or copy-engine peer copies for registered buffers), after which every rank -- in particular rank 0, where
 * the solver lives -- holds all world * n_local records in window order.  NCCL is bound at run time (dlopen libnccl.so.2).
 *
 *   cpi_comm_unique_id   rank 0: 128-byte NCCL id to hand to the other ranks (any out-of-band channel)
 *   cpi_comm_create      collective over all ranks, on the CURRENT device of each process
 *   cpi_preintegrate_batch_sharded
 *        enqueues the kernel for this rank's n_local windows on `stream`, writing records straight into slice `rank` of
 *        gather_records (device, world * n_local records: no pack kernel), then the all-gather on the communicator's own
 *        stream behind an event.  Returns without synchronising: the next batch's kernel (into ANOTHER gather buffer)
 *        overlaps the collective.  Re-using a gather buffer orders the new kernel behind that buffer's previous all-gather.
 *        n_local must be the same on every rank (pad a short last shard with zero-step windows).
 *   cpi_comm_register    collective, optional, once per gather buffer (same buffers in the same order on every rank): exports the buffer
 *        with CUDA IPC and maps the peers' buffers, after which cpi_preintegrate_batch_sharded exchanges the records by COPY-ENGINE
 *        copies of every rank's slice into the peers' buffers over NVLink instead of an ncclAllGather kernel, bracketed by two barriers
 *        that are SM-free as well (4-byte copy-engine writes into the peers' flag words + cuStreamWaitValue32; one-element NCCL
 *        all-reduces where stream memory operations are unavailable): nothing is taken from, or has to wait for, the preintegration
 *        kernel that runs beside the exchange.  *peer_copies (may be NULL)
 *        tells whether that path is active; it is not when any rank could not export / import (e.g. memory from a VMM / async pool) --
 *        the buffer then simply keeps the NCCL path.
 *   cpi_comm_unregister  drops the registration of one buffer (NULL: of all) and closes the peer mappings nothing refers to any more.
 *        EVERY rank must have unregistered a buffer before ANY rank frees it (freeing memory a peer still has mapped is undefined in
 *        CUDA IPC): unregister, synchronise the ranks, then free.
 *   cpi_comm_wait        makes `stream` wait for the most recently enqueued exchange (call before consuming the records)
 * The usual NCCL rule applies: collectives of ANOTHER communicator on the same devices (e.g. an MPI / torch.distributed NCCL group)
 * must not be in flight at the same time as this communicator's all-gathers -- synchronise the device between the two.
 */
#define CPI_COMM_ID_BYTES 128
typedef struct cpi_comm cpi_comm;
int cpi_comm_unique_id(void* id_out);
int cpi_comm_create(const void* id, int rank, int world, cpi_comm** out);
int cpi_comm_destroy(cpi_comm* comm);
int cpi_comm_rank(const cpi_comm* comm);
int cpi_comm_world(const cpi_comm* comm);
int cpi_comm_sm_free_barriers(const cpi_comm* comm);   /* 1: the peer-copy exchange synchronises with copy-engine flag writes + stream wait-value ops; 0: with NCCL all-reduces */
int cpi_comm_register(cpi_comm* comm, void* gather_records, size_t bytes, int* peer_copies);
int cpi_comm_unregister(cpi_comm* comm, void* gather_records);
int cpi_preintegrate_batch_sharded(cpi_comm* comm, int model, int dtype, int64_t n_local,
                                   const int64_t* sample_offsets, int64_t ns_uniform,
                                   const void* samples, const void* lin, const double* sigmas, int flags,
                                   void* gather_records, void* stream);
int cpi_comm_wait(cpi_comm* comm, void* stream);

/* ---- misc ----------------------------------------------------------------------------------------------------------- */

const char* cpi_last_error(void);
const char* cpi_version(void);
int cpi_record_doubles(int model);          /* 290 or 308; CPI_EINVAL otherwise */
int cpi_device_count(void);                 /* number of usable sm_90 devices, or negative error */
/* number of kernel launches issued by this library on the calling process since load (for bench.py's gpu_launches) */
int64_t cpi_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* CPI_B200_H */
