// TEST INFRASTRUCTURE ONLY -- never linked into or called by the product path (cpi_b200/).
//
// C-ABI wrapper around the UNMODIFIED reference, compiled in place from an rpng/cpi checkout (make ref REF=...; no source is copied):
//   cpi_compare/src/cpi/{CpiBase,CpiV1,CpiV2}.h, utils/quat_ops.h        (header-only, Eigen 3.2.10 vendored in the reference)
//   cpi_compare/src/gtsam/{ImuFactorCPIv1,ImuFactorCPIv2,JPLNavState}.cpp (against oracle/gtsam_stub/, see stub_core.h)
// Output: oracle/_ref/libcpi_ref.so (git-ignored).
// Uses the batch layouts of include/cpi_b200.h so that tests can compare buffers directly.
//
// The driving loop mirrors GraphSolver::createimufactor_cpi_v1/_v2 (solvers/GraphSolver_IMU.cpp:43-75, 97-130):
// construct, setLinearizationPoints, feed_IMU per step, read the public fields.
#include <deque>
#include <mutex>
#include <thread>
#include <vector>
#include <cstdint>
#include <cstring>

#include "cpi/CpiV1.h"
#include "cpi/CpiV2.h"
#include "gtsam/ImuFactorCPIv1.h"
#include "gtsam/ImuFactorCPIv2.h"
#include "../include/cpi_b200.h"

namespace {

typedef Eigen::Matrix<double, 3, 1> V3;
typedef Eigen::Matrix<double, 4, 1> V4;
typedef Eigen::Matrix<double, 3, 3> M3;

inline void put3x3(double* dst, const M3& m) { std::memcpy(dst, m.data(), 9 * sizeof(double)); }  // col-major

template <class CPI>
void fill_common(const CPI& c, double* r) {
    for (int k = 0; k < 4; k++) r[CPI_REC_Q + k] = c.q_k2tau(k);
    put3x3(r + CPI_REC_R, c.R_k2tau);
    for (int k = 0; k < 3; k++) { r[CPI_REC_ALPHA + k] = c.alpha_tau(k); r[CPI_REC_BETA + k] = c.beta_tau(k); }
    r[CPI_REC_DT] = c.DT;
    put3x3(r + CPI_REC_JQ, c.J_q); put3x3(r + CPI_REC_JA, c.J_a); put3x3(r + CPI_REC_JB, c.J_b);
    put3x3(r + CPI_REC_HA, c.H_a); put3x3(r + CPI_REC_HB, c.H_b);
    std::memcpy(r + CPI_REC_P, c.P_meas.data(), 225 * sizeof(double));
}

template <class CPI>
void feed_all(CPI& cpi, const double* s, int64_t steps, bool avg) {
    for (int64_t i = 0; i < steps; i++) {
        const double* e0 = s + i * CPI_SAMPLE_DOUBLES;
        const double* e1 = avg ? e0 + CPI_SAMPLE_DOUBLES : e0;
        V3 w0(e0[0], e0[1], e0[2]), a0(e0[3], e0[4], e0[5]);
        V3 w1(e1[0], e1[1], e1[2]), a1(e1[3], e1[4], e1[5]);
        cpi.feed_IMU(0.0, e0[6], w0, a0, w1, a1);   // delta_t = t_1 - t_0 = dt exactly
    }
}

void one_window(int model, const double* s, int64_t entries, const double* lin, const double* sig, int flags, double* rec) {
    const bool avg = (flags & CPI_FLAG_IMU_AVG) != 0;
    const int64_t steps = avg ? (entries > 0 ? entries - 1 : 0) : entries;
    V3 bw(lin[0], lin[1], lin[2]), ba(lin[3], lin[4], lin[5]), g(lin[10], lin[11], lin[12]);
    V4 q(lin[6], lin[7], lin[8], lin[9]);
    if (model == 1) {
        CpiV1 cpi(sig[0], sig[1], sig[2], sig[3], avg);
        cpi.q_k2tau << 0, 0, 0, 1;   // uninitialised in the reference (CpiBase.h:102); only visible for 0-step windows
        cpi.setLinearizationPoints(bw, ba, q, g);
        feed_all(cpi, s, steps, avg);
        fill_common(cpi, rec);
    } else {
        CpiV2 cpi(sig[0], sig[1], sig[2], sig[3], avg);
        cpi.q_k2tau << 0, 0, 0, 1;
        cpi.setLinearizationPoints(bw, ba, q, g);
        cpi.state_transition_jacobians = (flags & CPI_FLAG_ANALYTIC_JACOBIANS) == 0;
        feed_all(cpi, s, steps, avg);
        fill_common(cpi, rec);
        put3x3(rec + CPI_REC_OA, cpi.O_a); put3x3(rec + CPI_REC_OB, cpi.O_b);
    }
}

M3 get3x3(const double* p) { M3 m; std::memcpy(m.data(), p, 9 * sizeof(double)); return m; }

gtsam::JPLNavState get_state(const double* s) {
    return gtsam::JPLNavState(V4(s[0], s[1], s[2], s[3]), V3(s[4], s[5], s[6]), V3(s[7], s[8], s[9]),
                              V3(s[10], s[11], s[12]), V3(s[13], s[14], s[15]));
}
void put_state(double* s, const gtsam::JPLNavState& x) {
    for (int k = 0; k < 4; k++) s[k] = x.q()(k);
    for (int k = 0; k < 3; k++) { s[4 + k] = x.bg()(k); s[7 + k] = x.v()(k); s[10 + k] = x.ba()(k); s[13 + k] = x.p()(k); }
}

template <class F>
void run_threads(int64_t n, int nthreads, F f) {
    if (nthreads <= 1 || n < 2) { for (int64_t i = 0; i < n; i++) f(i); return; }
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; t++) {
        int64_t lo = n * t / nthreads, hi = n * (t + 1) / nthreads;
        th.emplace_back([=] { for (int64_t i = lo; i < hi; i++) f(i); });
    }
    for (auto& t : th) t.join();
}

}  // namespace

extern "C" {

// Host pointers everywhere.  Same argument meaning as cpi_preintegrate_batch_host (+ nthreads).
int ref_cpi_preintegrate(int model, int64_t n_windows, const int64_t* offsets, int64_t ns_uniform,
                         const double* samples, const double* lin, const double* sigmas, int flags,
                         double* out, int nthreads) {
    if (model != 1 && model != 2) return -1;
    const int rd = model == 1 ? CPI_REC_V1_DOUBLES : CPI_REC_V2_DOUBLES;
    const bool avg = (flags & CPI_FLAG_IMU_AVG) != 0;
    run_threads(n_windows, nthreads, [=](int64_t w) {
        int64_t o0 = offsets ? offsets[w] : w * (ns_uniform + (avg ? 1 : 0));
        int64_t o1 = offsets ? offsets[w + 1] : o0 + ns_uniform + (avg ? 1 : 0);
        one_window(model, samples + o0 * CPI_SAMPLE_DOUBLES, o1 - o0, lin + w * CPI_LIN_DOUBLES, sigmas, flags,
                   out + w * (int64_t)rd);
    });
    return 0;
}

// ImuFactorCPIv1/v2::evaluateError through the reference's own constructor + method.
int ref_imu_factor_eval(int model, int64_t n, const double* states, const int64_t* idx_i, const int64_t* idx_j,
                        const double* records, const double* lin, double* e, double* H1, double* H2, int nthreads) {
    if (model != 1 && model != 2) return -1;
    const int rd = model == 1 ? CPI_REC_V1_DOUBLES : CPI_REC_V2_DOUBLES;
    run_threads(n, nthreads, [=](int64_t f) {
        const double* r = records + f * (int64_t)rd;
        const double* l = lin + f * CPI_LIN_DOUBLES;
        int64_t i = idx_i ? idx_i[f] : f, j = idx_j ? idx_j[f] : f + 1;
        Eigen::Matrix<double, 15, 15> P; std::memcpy(P.data(), r + CPI_REC_P, 225 * sizeof(double));
        V3 grav(l[10], l[11], l[12]), alpha(r[CPI_REC_ALPHA], r[CPI_REC_ALPHA + 1], r[CPI_REC_ALPHA + 2]),
           beta(r[CPI_REC_BETA], r[CPI_REC_BETA + 1], r[CPI_REC_BETA + 2]);
        V4 qm(r[0], r[1], r[2], r[3]), qlin(l[6], l[7], l[8], l[9]);
        V3 bw(l[0], l[1], l[2]), ba(l[3], l[4], l[5]);
        gtsam::JPLNavState xi = get_state(states + i * CPI_STATE_DOUBLES), xj = get_state(states + j * CPI_STATE_DOUBLES);
        gtsam::Matrix h1, h2;
        gtsam::Vector err;
        // argument order exactly as at GraphSolver_IMU.cpp:74-75 / :129-130  (J_q, J_b, J_a, H_b, H_a [, O_b, O_a])
        if (model == 1) {
            gtsam::ImuFactorCPIv1 fac(i, j, P, r[CPI_REC_DT], grav, alpha, beta, qm, ba, bw, get3x3(r + CPI_REC_JQ),
                                      get3x3(r + CPI_REC_JB), get3x3(r + CPI_REC_JA), get3x3(r + CPI_REC_HB), get3x3(r + CPI_REC_HA));
            err = fac.evaluateError(xi, xj, boost::optional<gtsam::Matrix&>(h1), boost::optional<gtsam::Matrix&>(h2));
        } else {
            gtsam::ImuFactorCPIv2 fac(i, j, P, r[CPI_REC_DT], grav, alpha, beta, qm, qlin, ba, bw, get3x3(r + CPI_REC_JQ),
                                      get3x3(r + CPI_REC_JB), get3x3(r + CPI_REC_JA), get3x3(r + CPI_REC_HB), get3x3(r + CPI_REC_HA),
                                      get3x3(r + CPI_REC_OB), get3x3(r + CPI_REC_OA));
            err = fac.evaluateError(xi, xj, boost::optional<gtsam::Matrix&>(h1), boost::optional<gtsam::Matrix&>(h2));
        }
        std::memcpy(e + f * 15, err.data(), 15 * sizeof(double));
        if (H1) std::memcpy(H1 + f * 225, h1.data(), 225 * sizeof(double));
        if (H2) std::memcpy(H2 + f * 225, h2.data(), 225 * sizeof(double));
    });
    return 0;
}

// JPLNavState::retract through the reference's own TU.
int ref_retract(int64_t n, const double* states, const double* xi, double* out) {
    for (int64_t i = 0; i < n; i++) {
        Eigen::Matrix<double, 15, 1> d; std::memcpy(d.data(), xi + i * 15, 15 * sizeof(double));
        put_state(out + i * CPI_STATE_DOUBLES, get_state(states + i * CPI_STATE_DOUBLES).retract(d));
    }
    return 0;
}

// quat_ops.h helpers, for unit-pinning the restatement
void ref_rot_2_quat(const double* R_colmajor, double* q) { V4 r = rot_2_quat(get3x3(R_colmajor)); std::memcpy(q, r.data(), 32); }
void ref_quat_2_Rot(const double* q, double* R_colmajor) { M3 r = quat_2_Rot(V4(q[0], q[1], q[2], q[3])); put3x3(R_colmajor, r); }
void ref_quat_multiply(const double* q, const double* p, double* out) {
    V4 r = quat_multiply(V4(q[0], q[1], q[2], q[3]), V4(p[0], p[1], p[2], p[3])); std::memcpy(out, r.data(), 32);
}
void ref_Exp(const double* w, double* R_colmajor) { M3 r = Exp(V3(w[0], w[1], w[2])); put3x3(R_colmajor, r); }

int ref_hardware_threads(void) { return (int)std::thread::hardware_concurrency(); }

// Replay of the reference DRIVER over one dataset run, with std::deque containers handled exactly as the reference handles them:
//   GraphSolver::addmeasurement_imu (solvers/GraphSolver.cpp:58-69): push_back as readings arrive;
//   SimulationLoader::execute_publishing (sim/SimulationLoader.cpp:214-290): at equal stamps the IMU reading is delivered before the camera;
//   GraphSolver::addmeasurement_uv (solvers/GraphSolver.cpp:85-119): size() < 2 -> return; not initialised -> trytoinitalize;
//   GraphSolver::trytoinitalize (solvers/GraphSolver.cpp:264, 357): needs >= imuWait queued readings, then erase(begin, end-1);
//   GraphSolver::createimufactor_cpi_v1/_v2 (solvers/GraphSolver_IMU.cpp:43-75, 97-130): the two loops below, on the reference's
//   own CpiV1 / CpiV2 objects, fed with the reference's own arguments (t_0, t_1, w_0, a_0, w_1, a_1).
// The vision half of the solver cannot be built here (GTSAM), so the linearisation points -- which the reference takes from its state
// estimate -- are an input (lin, one per camera frame); preintegration does not depend on where they came from.
// Outputs: the entries the reference fed, in the CSR layout of include/cpi_b200.h (what cpi_cut_windows must reproduce bit for bit),
// and the reference's records for them.  Returns the number of windows, or -1 if out_samples is too small.
int64_t ref_replay_run(int model, int64_t n_imu, const double* t, const double* w, const double* a, int64_t n_cam, const double* cam_t,
                       int64_t imu_wait, const double* lin, const double* sig, int flags, int64_t cap_entries, double* out_samples,
                       int64_t* out_offsets, double* out_records) {
    if (model != 1 && model != 2) return -1;
    const int rd = model == 1 ? CPI_REC_V1_DOUBLES : CPI_REC_V2_DOUBLES;
    std::deque<double> imu_times;
    std::deque<V3, Eigen::aligned_allocator<V3> > imu_linaccs, imu_angvel;
    bool systeminitalized = imu_wait == 0;
    int64_t next_imu = 0, nwin = 0, ne = 0;
    out_offsets[0] = 0;
    bool overflow = false;
    auto record = [&](double t0, double t1, const V3& w0, const V3& a0) {
        if (ne < cap_entries) {
            double* s = out_samples + ne * CPI_SAMPLE_DOUBLES;
            s[0] = w0(0); s[1] = w0(1); s[2] = w0(2); s[3] = a0(0); s[4] = a0(1); s[5] = a0(2); s[6] = t1 - t0;   // feed_IMU: delta_t = t_1 - t_0
        } else overflow = true;
        ne++;
    };
    for (int64_t c = 0; c < n_cam; c++) {
        const double updatetime = cam_t[c];
        while (next_imu < n_imu && t[next_imu] <= updatetime) {                  // addmeasurement_imu, IMU first at equal stamps
            imu_times.push_back(t[next_imu]);
            imu_linaccs.push_back(V3(a[3 * next_imu], a[3 * next_imu + 1], a[3 * next_imu + 2]));
            imu_angvel.push_back(V3(w[3 * next_imu], w[3 * next_imu + 1], w[3 * next_imu + 2]));
            next_imu++;
        }
        if (imu_times.size() < 2) continue;                                       // GraphSolver.cpp:85
        if (!systeminitalized) {                                                  // GraphSolver.cpp:264, 357
            if (imu_times.size() < (size_t)imu_wait) continue;
            imu_times.erase(imu_times.begin(), imu_times.end() - 1);
            imu_linaccs.erase(imu_linaccs.begin(), imu_linaccs.end() - 1);
            imu_angvel.erase(imu_angvel.begin(), imu_angvel.end() - 1);
            systeminitalized = true;
            continue;
        }
        const double* l = lin + nwin * CPI_LIN_DOUBLES;
        V3 bw(l[0], l[1], l[2]), ba(l[3], l[4], l[5]), g(l[10], l[11], l[12]);
        V4 q(l[6], l[7], l[8], l[9]);
        double* rec = out_records + nwin * (int64_t)rd;
        // GraphSolver_IMU.cpp:43-75 (model 1) / 97-130 (model 2): same statements, same containers
#define CPI_REPLAY_LOOP(cpi)                                                                                                              \
        while (imu_times.size() > 1 && imu_times.at(1) <= updatetime) {                                                                    \
            double dt = imu_times.at(1) - imu_times.at(0);                                                                                 \
            if (dt >= 0) {                                                                                                                 \
                cpi.feed_IMU(imu_times.at(0), imu_times.at(1), imu_angvel.at(0), imu_linaccs.at(0), imu_angvel.at(1), imu_linaccs.at(1)); \
                record(imu_times.at(0), imu_times.at(1), imu_angvel.at(0), imu_linaccs.at(0));                                            \
            }                                                                                                                              \
            imu_angvel.erase(imu_angvel.begin());                                                                                          \
            imu_linaccs.erase(imu_linaccs.begin());                                                                                        \
            imu_times.erase(imu_times.begin());                                                                                            \
        }                                                                                                                                  \
        double dt_f = updatetime - imu_times.at(0);                                                                                        \
        if (dt_f > 0) {                                                                                                                    \
            cpi.feed_IMU(imu_times.at(0), updatetime, imu_angvel.at(0), imu_linaccs.at(0), imu_angvel.at(0), imu_linaccs.at(0));          \
            record(imu_times.at(0), updatetime, imu_angvel.at(0), imu_linaccs.at(0));                                                     \
            imu_times.at(0) = updatetime;                                                                                                  \
        }
        if (model == 1) {
            CpiV1 cpi(sig[0], sig[1], sig[2], sig[3]);
            cpi.q_k2tau << 0, 0, 0, 1;
            cpi.setLinearizationPoints(bw, ba, q, g);
            cpi.imu_avg = false;
            CPI_REPLAY_LOOP(cpi)
            fill_common(cpi, rec);
        } else {
            CpiV2 cpi(sig[0], sig[1], sig[2], sig[3]);
            cpi.q_k2tau << 0, 0, 0, 1;
            cpi.setLinearizationPoints(bw, ba, q, g);
            cpi.imu_avg = false;
            cpi.state_transition_jacobians = (flags & CPI_FLAG_ANALYTIC_JACOBIANS) == 0;     // GraphSolver_IMU.cpp:100 sets true
            CPI_REPLAY_LOOP(cpi)
            fill_common(cpi, rec);
            put3x3(rec + CPI_REC_OA, cpi.O_a); put3x3(rec + CPI_REC_OB, cpi.O_b);
        }
#undef CPI_REPLAY_LOOP
        out_offsets[++nwin] = ne;
    }
    return overflow ? -1 : nwin;
}

}  // extern "C"
