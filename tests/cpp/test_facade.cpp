// Test driver for include/cpi_b200/CpiGpu.h: runs the SAME feed loop (solvers/GraphSolver_IMU.cpp:43-75 shape) through the
// reference's CpiV1/CpiV2 (compiled in place from an rpng/cpi checkout) and through CpiV1Gpu/CpiV2Gpu, and compares the public
// fields.  Built only where an rpng/cpi checkout is given (make -C tests/cpp REF=...).
#include <cmath>
#include <cstdio>
#include <random>

#include "cpi/CpiV1.h"
#include "cpi/CpiV2.h"
#include "cpi_b200/CpiGpu.h"

template <class A, class B> static double rel(const A& a, const B& b) { return (a - b).norm() / std::max(b.norm(), 1e-300); }

// state_transition_jacobians (CpiV2.h:58) and the O_a / O_b outputs (CpiV2.h:62-63) exist on model 2 only
template <class C> static void set_stj(C&, bool) {}
static void set_stj(CpiV2& c, bool v) { c.state_transition_jacobians = v; }
static void set_stj(cpi_b200::CpiV2Gpu& c, bool v) { c.state_transition_jacobians = v; }
template <class A, class B> static double extra(const A&, const B&) { return 0.0; }
static double extra(const cpi_b200::CpiV2Gpu& g, const CpiV2& r) { return std::max(rel(g.O_a, r.O_a), rel(g.O_b, r.O_b)); }

template <class REF, class GPU> static int run(const char* name, bool avg, bool stj, unsigned seed) {
    std::mt19937_64 g(seed);
    std::normal_distribution<double> N(0, 1);
    REF ref(0.005, 4e-6, 0.01, 0.0002, avg);
    GPU gpu(0.005, 4e-6, 0.01, 0.0002, avg);
    Eigen::Vector3d bw(1e-3 * N(g), 1e-3 * N(g), 1e-3 * N(g)), ba(1e-2 * N(g), 1e-2 * N(g), 1e-2 * N(g)), grav(0, 0, 9.8);
    Eigen::Vector4d q(N(g), N(g), N(g), N(g)); q.normalize(); if (q(3) < 0) q = -q;
    ref.setLinearizationPoints(bw, ba, q, grav);
    gpu.setLinearizationPoints(bw, ba, q, grav);
    set_stj(ref, stj); set_stj(gpu, stj);
    double t = 1275.0;
    Eigen::Vector3d w0(0.3, -0.5, 0.8), a0(0.1, -0.2, 9.7);
    for (int i = 0; i < 60; i++) {
        Eigen::Vector3d w1 = w0 + 0.05 * Eigen::Vector3d(N(g), N(g), N(g)), a1 = a0 + 0.1 * Eigen::Vector3d(N(g), N(g), N(g));
        double t1 = t + ((i % 17 == 3) ? 0.010 : 0.005);
        ref.feed_IMU(t, t1, w0, a0, w1, a1);
        gpu.feed_IMU(t, t1, w0, a0, w1, a1);
        t = t1; w0 = w1; a0 = a1;
    }
    gpu.finalize();
    double e = 0;
    e = std::max(e, rel(gpu.R_k2tau, ref.R_k2tau)); e = std::max(e, rel(gpu.alpha_tau, ref.alpha_tau)); e = std::max(e, rel(gpu.beta_tau, ref.beta_tau));
    e = std::max(e, rel(gpu.q_k2tau, ref.q_k2tau)); e = std::max(e, rel(gpu.J_q, ref.J_q)); e = std::max(e, rel(gpu.J_a, ref.J_a));
    e = std::max(e, rel(gpu.J_b, ref.J_b)); e = std::max(e, rel(gpu.H_a, ref.H_a)); e = std::max(e, rel(gpu.H_b, ref.H_b));
    e = std::max(e, rel(gpu.P_meas, ref.P_meas)); e = std::max(e, std::fabs(gpu.DT - ref.DT));
    e = std::max(e, extra(gpu, ref));
    std::printf("%s avg=%d stj=%d: worst relative field error %.3e\n", name, (int)avg, (int)stj, e);
    return e < 1e-9 ? 0 : 1;
}

struct V2Ref : CpiV2 { V2Ref(double a, double b, double c, double d, bool e) : CpiV2(a, b, c, d, e) {} };

int main() {
    int bad = 0;
    bad += run<CpiV1, cpi_b200::CpiV1Gpu>("CpiV1Gpu", false, true, 1);
    bad += run<CpiV1, cpi_b200::CpiV1Gpu>("CpiV1Gpu", true, true, 2);
    bad += run<CpiV2, cpi_b200::CpiV2Gpu>("CpiV2Gpu", false, true, 3);
    bad += run<CpiV2, cpi_b200::CpiV2Gpu>("CpiV2Gpu", true, true, 4);
    bad += run<CpiV2, cpi_b200::CpiV2Gpu>("CpiV2Gpu", false, false, 5);      // analytic-Jacobian mode (incl. the reference's sign slip, CpiV2.h:296-297)
    bad += run<CpiV2, cpi_b200::CpiV2Gpu>("CpiV2Gpu", true, false, 6);
    std::printf(bad ? "FACADE FAIL\n" : "FACADE OK\n");
    return bad;
}
