// Test driver for include/cpi_b200/ImuFactorGpu.h: the reference's own ImuFactorCPIv1 / ImuFactorCPIv2 (gtsam/ImuFactorCPIv1.cpp,
// ImuFactorCPIv2.cpp, JPLNavState.cpp compiled UNMODIFIED, in place from an rpng/cpi checkout, against oracle/gtsam_stub) and the drop-in
// ImuFactorCPIv1Gpu / ImuFactorCPIv2Gpu live in ONE binary, are constructed from the same arguments (the public fields of a
// reference CpiV1 / CpiV2 after its feed loop, exactly as GraphSolver_IMU.cpp:74-75 / :129-130 does) and evaluated on the same
// states; e, H1, H2 are compared per factor, once through the per-factor path and once through the graph-level batch.
// Built only where an rpng/cpi checkout is given (make -C tests/cpp REF=...).
#include <cmath>
#include <cstdio>
#include <map>
#include <random>
#include <vector>

#include "cpi/CpiV1.h"
#include "cpi/CpiV2.h"
#include "ImuFactorCPIv1.h"
#include "ImuFactorCPIv2.h"
#include "cpi_b200/ImuFactorGpu.h"

using namespace gtsam;

static std::mt19937_64 g(20260924);
static std::normal_distribution<double> N(0, 1);
static Eigen::Vector3d rnd3(double s) { return s * Eigen::Vector3d(N(g), N(g), N(g)); }
static Eigen::Matrix<double, 4, 1> rndq() { Eigen::Matrix<double, 4, 1> q(N(g), N(g), N(g), N(g)); q.normalize(); if (q(3) < 0) q = -q; return q; }

template <class CPI> static void feed(CPI& c, int steps) {
    double t = 10.0;
    Eigen::Vector3d w(0.4, -0.3, 0.7), a(0.2, -0.1, 9.7);
    for (int i = 0; i < steps; i++) {
        w += rnd3(0.05); a += rnd3(0.1);
        c.feed_IMU(t, t + 0.005, w, a, w, a);
        t += 0.005;
    }
}

static double maxabs(const gtsam::Matrix& a, const gtsam::Matrix& b) { return (a - b).cwiseAbs().maxCoeff(); }

template <class REF, class GPU> static int compare(const std::vector<REF>& rf, const std::vector<GPU>& gf, const std::map<Key, JPLNavState>& val, const char* name) {
    double worst = 0, scale = 0;
    int zero_mismatch = 0;
    for (int pass = 0; pass < 2; pass++) {
        if (pass == 1) {
            std::vector<const GPU*> ptrs;
            for (size_t i = 0; i < gf.size(); i++) ptrs.push_back(&gf[i]);
            cpi_b200::ImuFactorBatch<GPU>::evaluate(ptrs, val);
        }
        for (size_t i = 0; i < rf.size(); i++) {
            const JPLNavState &xi = val.at(rf[i].key1()), &xj = val.at(rf[i].key2());
            gtsam::Matrix H1r, H2r, H1g, H2g;
            gtsam::Vector er = rf[i].evaluateError(xi, xj, H1r, H2r);
            gtsam::Vector eg = gf[i].evaluateError(xi, xj, H1g, H2g);
            gtsam::Vector eg0 = gf[i].evaluateError(xi, xj);                 // without Jacobians
            worst = std::max(worst, std::max(maxabs(er, eg), std::max(maxabs(H1r, H1g), maxabs(H2r, H2g))));
            worst = std::max(worst, maxabs(eg, eg0));
            scale = std::max(scale, std::max(H1r.cwiseAbs().maxCoeff(), H2r.cwiseAbs().maxCoeff()));
            for (int r = 0; r < 15; r++) for (int c = 0; c < 15; c++) {
                if ((H1r(r, c) == 0.0) != (H1g(r, c) == 0.0)) zero_mismatch++;
                if ((H2r(r, c) == 0.0) != (H2g(r, c) == 0.0)) zero_mismatch++;
            }
        }
    }
    // a factor evaluated at OTHER states than the parked batch row must not serve the stale row
    JPLNavState moved(rndq(), rnd3(1e-3), rnd3(1.0), rnd3(1e-2), rnd3(1.0));
    gtsam::Matrix Hr, Hg;
    double stale = maxabs(rf[0].evaluateError(moved, val.at(rf[0].key2()), Hr), gf[0].evaluateError(moved, val.at(gf[0].key2()), Hg));
    worst = std::max(worst, std::max(stale, maxabs(Hr, Hg)));
    std::printf("%s: %zu factors, worst |diff| %.3e (max |H| %.3e), structural-zero mismatches %d\n", name, rf.size(), worst, scale, zero_mismatch);
    return (worst <= 1e-12 * std::max(1.0, scale) && zero_mismatch == 0) ? 0 : 1;
}

int main() {
    const int n = 48;
    const Eigen::Vector3d grav(0, 0, 9.8);
    std::map<Key, JPLNavState> val;
    for (int k = 0; k <= n; k++) val[(Key)k] = JPLNavState(rndq(), rnd3(1e-3), rnd3(1.0), rnd3(1e-2), rnd3(2.0));
    std::vector<ImuFactorCPIv1> r1; std::vector<ImuFactorCPIv1Gpu> g1;
    std::vector<ImuFactorCPIv2> r2; std::vector<ImuFactorCPIv2Gpu> g2;
    for (int k = 0; k < n; k++) {
        Eigen::Vector3d bw = rnd3(1e-3), ba = rnd3(1e-2);
        Eigen::Matrix<double, 4, 1> qlin = val[(Key)k].q();
        CpiV1 c1(0.005, 4e-6, 0.01, 0.0002, false);
        c1.setLinearizationPoints(bw, ba);
        feed(c1, 20 + k % 7);
        // GraphSolver_IMU.cpp:74-75
        r1.push_back(ImuFactorCPIv1((Key)k, (Key)(k + 1), c1.P_meas, c1.DT, grav, c1.alpha_tau, c1.beta_tau, c1.q_k2tau, c1.b_a_lin, c1.b_w_lin, c1.J_q, c1.J_b, c1.J_a, c1.H_b, c1.H_a));
        g1.push_back(ImuFactorCPIv1Gpu((Key)k, (Key)(k + 1), c1.P_meas, c1.DT, grav, c1.alpha_tau, c1.beta_tau, c1.q_k2tau, c1.b_a_lin, c1.b_w_lin, c1.J_q, c1.J_b, c1.J_a, c1.H_b, c1.H_a));
        CpiV2 c2(0.005, 4e-6, 0.01, 0.0002, false);
        c2.setLinearizationPoints(bw, ba, qlin, grav);
        feed(c2, 20 + k % 5);
        // GraphSolver_IMU.cpp:129-130
        r2.push_back(ImuFactorCPIv2((Key)k, (Key)(k + 1), c2.P_meas, c2.DT, grav, c2.alpha_tau, c2.beta_tau, c2.q_k2tau, c2.q_k_lin, c2.b_a_lin, c2.b_w_lin, c2.J_q, c2.J_b, c2.J_a, c2.H_b, c2.H_a, c2.O_b, c2.O_a));
        g2.push_back(ImuFactorCPIv2Gpu((Key)k, (Key)(k + 1), c2.P_meas, c2.DT, grav, c2.alpha_tau, c2.beta_tau, c2.q_k2tau, c2.q_k_lin, c2.b_a_lin, c2.b_w_lin, c2.J_q, c2.J_b, c2.J_a, c2.H_b, c2.H_a, c2.O_b, c2.O_a));
    }
    int bad = 0;
    bad += compare(r1, g1, val, "ImuFactorCPIv1Gpu");
    bad += compare(r2, g2, val, "ImuFactorCPIv2Gpu");
    // equals(): same measurement -> true; another factor -> false  (ImuFactorCPIv1.h:164-182)
    bad += g1[0].equals(g1[0]) && !g1[0].equals(g1[1]) && g2[3].equals(g2[3]) && !g2[3].equals(g2[4]) ? 0 : 1;
    std::printf(bad ? "FACTOR FACADE FAIL\n" : "FACTOR FACADE OK\n");
    return bad;
}
