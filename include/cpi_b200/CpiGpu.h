/*
 * CpiGpu.h -- C++ drop-in preintegrators for the reference tree (rpng/cpi), backed by libcpi_b200.so.
 *
 * Lives next to the reference's own headers: it includes the reference's cpi/CpiBase.h (and therefore Eigen) and derives
 * from CpiBase, so GraphSolver::createimufactor_cpi_v1/_v2 (solvers/GraphSolver_IMU.cpp:34-134) keeps compiling with
 *     CpiV1  ->  CpiV1Gpu        CpiV2  ->  CpiV2Gpu
 * plus ONE added line after the feed loop (before the public fields are read at :74 / :129):   cpi.finalize();
 * or, to build many factors with one kernel launch,   cpi_b200::flush({&cpi_a, &cpi_b, ...});
 *
 * Same constructor, setLinearizationPoints() (inherited), feed_IMU() signature (CpiBase.h:86-88), same public result
 * fields (CpiBase.h:95-124; CpiV2.h:58-63 for state_transition_jacobians / O_a / O_b).  feed_IMU only stages the step
 * on the host; all arithmetic happens in the CUDA kernels behind the C ABI (include/cpi_b200.h).  There is no CPU path:
 * finalize() throws std::runtime_error if the library reports an error.
 */
#ifndef CPI_B200_CPIGPU_H
#define CPI_B200_CPIGPU_H

#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "cpi/CpiBase.h"
#include "cpi_b200.h"

namespace cpi_b200 {

class CpiGpuBase : public CpiBase {
public:
    CpiGpuBase(int model, double sigma_w, double sigma_wb, double sigma_a, double sigma_ab, bool imu_avg_)
        : CpiBase(sigma_w, sigma_wb, sigma_a, sigma_ab, imu_avg_), model_(model) {
        sig_[0] = sigma_w; sig_[1] = sigma_wb; sig_[2] = sigma_a; sig_[3] = sigma_ab;
        q_k2tau << 0, 0, 0, 1;
    }

    // CpiBase.h:86 -- same signature; stages (w0, a0, dt [, w1, a1]) on the host
    void feed_IMU(double t_0, double t_1, Eigen::Matrix<double, 3, 1> w_m_0, Eigen::Matrix<double, 3, 1> a_m_0,
                  Eigen::Matrix<double, 3, 1> w_m_1 = Eigen::Matrix<double, 3, 1>::Zero(),
                  Eigen::Matrix<double, 3, 1> a_m_1 = Eigen::Matrix<double, 3, 1>::Zero()) {
        const double e[7] = {w_m_0(0), w_m_0(1), w_m_0(2), a_m_0(0), a_m_0(1), a_m_0(2), t_1 - t_0};
        steps_.insert(steps_.end(), e, e + 7);
        const double n[6] = {w_m_1(0), w_m_1(1), w_m_1(2), a_m_1(0), a_m_1(1), a_m_1(2)};
        next_.insert(next_.end(), n, n + 6);
    }

    // Runs the kernel for this window and fills the inherited public fields.
    void finalize() { std::vector<CpiGpuBase*> one(1, this); flush(one); }

    static void flush(const std::vector<CpiGpuBase*>& objs) {
        // group by (model, flags, sigmas): one launch per group
        std::vector<char> done(objs.size(), 0);
        for (size_t a = 0; a < objs.size(); a++) {
            if (done[a]) continue;
            std::vector<CpiGpuBase*> grp;
            for (size_t b = a; b < objs.size(); b++)
                if (!done[b] && objs[b]->model_ == objs[a]->model_ && objs[b]->flags() == objs[a]->flags() &&
                    std::memcmp(objs[b]->sig_, objs[a]->sig_, sizeof(double) * 4) == 0) { grp.push_back(objs[b]); done[b] = 1; }
            run_group(grp);
        }
    }

protected:
    virtual int flags() const { return imu_avg ? CPI_FLAG_IMU_AVG : 0; }
    virtual void adopt_extra(const double*) {}

    // the public result fields in the record layout (include/cpi_b200.h), and the linearisation point
    void pack_v1(double* r) const {
        Eigen::Map<Eigen::Matrix<double, 4, 1> >(r + CPI_REC_Q) = q_k2tau;
        Eigen::Map<Eigen::Matrix<double, 3, 3> >(r + CPI_REC_R) = R_k2tau;
        Eigen::Map<Eigen::Matrix<double, 3, 1> >(r + CPI_REC_ALPHA) = alpha_tau;
        Eigen::Map<Eigen::Matrix<double, 3, 1> >(r + CPI_REC_BETA) = beta_tau;
        r[CPI_REC_DT] = DT;
        Eigen::Map<Eigen::Matrix<double, 3, 3> >(r + CPI_REC_JQ) = J_q;
        Eigen::Map<Eigen::Matrix<double, 3, 3> >(r + CPI_REC_JA) = J_a;
        Eigen::Map<Eigen::Matrix<double, 3, 3> >(r + CPI_REC_JB) = J_b;
        Eigen::Map<Eigen::Matrix<double, 3, 3> >(r + CPI_REC_HA) = H_a;
        Eigen::Map<Eigen::Matrix<double, 3, 3> >(r + CPI_REC_HB) = H_b;
        Eigen::Map<Eigen::Matrix<double, 15, 15> >(r + CPI_REC_P) = P_meas;
    }
    void pack_lin(double* l) const {
        const double v[13] = {b_w_lin(0), b_w_lin(1), b_w_lin(2), b_a_lin(0), b_a_lin(1), b_a_lin(2),
                              q_k_lin(0), q_k_lin(1), q_k_lin(2), q_k_lin(3), grav(0), grav(1), grav(2)};
        std::memcpy(l, v, sizeof v);
    }
    // k -> m (this) (+) m -> j (later): merged on the device, the fields re-adopted; the staged steps are concatenated
    void merge_v1(const CpiGpuBase& later) {
        std::vector<double> rec(2 * (size_t)CPI_REC_V1_DOUBLES), lin(2 * (size_t)CPI_LIN_DOUBLES), out(CPI_REC_V1_DOUBLES);
        pack_v1(rec.data()); later.pack_v1(rec.data() + CPI_REC_V1_DOUBLES);
        pack_lin(lin.data()); later.pack_lin(lin.data() + CPI_LIN_DOUBLES);
        const int rc = cpi_merge_records_host(1, 64, 1, nullptr, 2, rec.data(), lin.data(), out.data());
        if (rc != CPI_OK) throw std::runtime_error(std::string("cpi_b200: ") + cpi_last_error());
        steps_.insert(steps_.end(), later.steps_.begin(), later.steps_.end());
        next_.insert(next_.end(), later.next_.begin(), later.next_.end());
        adopt(out.data());
    }

private:
    int model_;
    double sig_[4];
    std::vector<double> steps_, next_;

    // entries in the batch layout (include/cpi_b200.h).  imu_avg: every step is followed by a dt = 0 entry carrying its
    // (w_m_1, a_m_1) -- a no-op step (CpiV1.h:72-74) that only serves as the "_1" reading of the step before it.
    void entries(std::vector<double>& out) const {
        const size_t n = steps_.size() / 7;
        if (!imu_avg) { out.insert(out.end(), steps_.begin(), steps_.end()); return; }
        for (size_t i = 0; i < n; i++) {
            out.insert(out.end(), steps_.begin() + 7 * i, steps_.begin() + 7 * i + 7);
            out.insert(out.end(), next_.begin() + 6 * i, next_.begin() + 6 * i + 6);
            out.push_back(0.0);
        }
        for (int k = 0; k < 7; k++) out.push_back(n ? out[out.size() - 7] : 0.0);   // trailing entry
    }

    static void run_group(const std::vector<CpiGpuBase*>& g) {
        const int model = g[0]->model_, fl = g[0]->flags();
        const int rd = cpi_record_doubles(model);
        std::vector<double> S, L, out(g.size() * (size_t)rd);
        std::vector<int64_t> off(1, 0);
        for (size_t i = 0; i < g.size(); i++) {
            g[i]->entries(S);
            off.push_back((int64_t)(S.size() / 7));
            const CpiGpuBase* c = g[i];
            const double l[13] = {c->b_w_lin(0), c->b_w_lin(1), c->b_w_lin(2), c->b_a_lin(0), c->b_a_lin(1), c->b_a_lin(2),
                                  c->q_k_lin(0), c->q_k_lin(1), c->q_k_lin(2), c->q_k_lin(3), c->grav(0), c->grav(1), c->grav(2)};
            L.insert(L.end(), l, l + 13);
        }
        if (S.empty()) S.push_back(0.0);
        const int rc = cpi_preintegrate_batch_host(model, 64, (int64_t)g.size(), off.data(), 0, S.data(), L.data(), g[0]->sig_, fl, out.data());
        if (rc != CPI_OK) throw std::runtime_error(std::string("cpi_b200: ") + cpi_last_error());
        for (size_t i = 0; i < g.size(); i++) g[i]->adopt(out.data() + i * (size_t)rd);
    }

    void adopt(const double* r) {
        q_k2tau = Eigen::Map<const Eigen::Matrix<double, 4, 1> >(r + CPI_REC_Q);
        R_k2tau = Eigen::Map<const Eigen::Matrix<double, 3, 3> >(r + CPI_REC_R);
        alpha_tau = Eigen::Map<const Eigen::Matrix<double, 3, 1> >(r + CPI_REC_ALPHA);
        beta_tau = Eigen::Map<const Eigen::Matrix<double, 3, 1> >(r + CPI_REC_BETA);
        DT = r[CPI_REC_DT];
        J_q = Eigen::Map<const Eigen::Matrix<double, 3, 3> >(r + CPI_REC_JQ);
        J_a = Eigen::Map<const Eigen::Matrix<double, 3, 3> >(r + CPI_REC_JA);
        J_b = Eigen::Map<const Eigen::Matrix<double, 3, 3> >(r + CPI_REC_JB);
        H_a = Eigen::Map<const Eigen::Matrix<double, 3, 3> >(r + CPI_REC_HA);
        H_b = Eigen::Map<const Eigen::Matrix<double, 3, 3> >(r + CPI_REC_HB);
        P_meas = Eigen::Map<const Eigen::Matrix<double, 15, 15> >(r + CPI_REC_P);
        adopt_extra(r);
    }
};

/// Drop-in for CpiV1 (cpi/CpiV1.h:41)
class CpiV1Gpu : public CpiGpuBase {
public:
    CpiV1Gpu(double sigma_w, double sigma_wb, double sigma_a, double sigma_ab, bool imu_avg_ = false)
        : CpiGpuBase(1, sigma_w, sigma_wb, sigma_a, sigma_ab, imu_avg_) {}

    /// Extend this finalised window by the finalised window that follows it (GTSAM's mergeWith), in place, at this object's
    /// linearisation point (`later` is moved to it to first order).  Throws std::runtime_error if the library reports an error.
    void mergeWith(const CpiV1Gpu& later) { merge_v1(later); }
};

/// Drop-in for CpiV2 (cpi/CpiV2.h:41)
class CpiV2Gpu : public CpiGpuBase {
public:
    bool state_transition_jacobians = true;                                         // CpiV2.h:58
    Eigen::Matrix<double, 3, 3> O_a = Eigen::Matrix<double, 3, 3>::Zero();          // CpiV2.h:62
    Eigen::Matrix<double, 3, 3> O_b = Eigen::Matrix<double, 3, 3>::Zero();          // CpiV2.h:63
    CpiV2Gpu(double sigma_w, double sigma_wb, double sigma_a, double sigma_ab, bool imu_avg_ = false)
        : CpiGpuBase(2, sigma_w, sigma_wb, sigma_a, sigma_ab, imu_avg_) {}

protected:
    int flags() const override { return (imu_avg ? CPI_FLAG_IMU_AVG : 0) | (state_transition_jacobians ? 0 : CPI_FLAG_ANALYTIC_JACOBIANS); }
    void adopt_extra(const double* r) override {
        O_a = Eigen::Map<const Eigen::Matrix<double, 3, 3> >(r + CPI_REC_OA);
        O_b = Eigen::Map<const Eigen::Matrix<double, 3, 3> >(r + CPI_REC_OB);
    }
};

inline void flush(const std::vector<CpiGpuBase*>& objs) { CpiGpuBase::flush(objs); }

}  // namespace cpi_b200
#endif
