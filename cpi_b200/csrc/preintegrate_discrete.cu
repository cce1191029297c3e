// K14: discrete (Forster) preintegration into model-1 records, CPI_FLAG_DISCRETE (DESIGN.md section 3n), for H100 (sm_90a).
//
// Per step: the rotation and J_q chains of model 1 (same closed forms and small-w branch), first-order (Euler) means and
// bias Jacobians at the step's start rotation, and the covariance  P' = Phi P Phi^T + Q  with Forster's Phi and Q
// (TRO 2017, eqs. 62-63) in CpiV1's error convention, record order [theta, b_g, v, b_a, p].  Phi is the identity except
//     Phi_tt = Rs   Phi_tg = -J_r dt   Phi_vt = M dt   Phi_va = B dt   Phi_pt = M dt^2/2   Phi_pv = I dt   Phi_pa = B dt^2/2
// with Rs = Exp(-[w_hat dt]x), M = -R^T [a_hat x], B = -R^T.  P keeps model 1's structure: P_bg,bg = pgg I, P_ba,ba = paa I and
// P_theta,ba = P_bg,ba = 0 identically, so the tile is the same 90 unique entries as `k_preintegrate`'s.
//
// Mapping: one lane per window, like `k_preintegrate` (preintegrate.cu): the per-sample chain is one sparse  Phi P Phi^T  (no stage values),
// and every block product is a short register chain.  The covariance tile is ping-ponged in shared memory in [entry][window]
// order (conflict-free: lane == window), the Jacobian state sits beside it; R, alpha, beta, DT, pgg, paa stay in registers.
// The record holds the whole state of the recursion, so continuing from a record is bitwise the one-shot result.
#include "cpi_common.cuh"
#include "cpi_kernels.h"

namespace cpi {
namespace {

enum : int {
    TT = 0, TG = 6, VT = 15, VG = 24, VV = 33, VA = 39, PT = 48, PG = 57, PV = 66, PA = 75, PP = 84, NP = 90,   // tile (sym: TT, VV, PP)
    J_Q = 0, J_A = 9, J_B = 18, H_A = 27, H_B = 36, NJ = 45                                                        // Jacobian state
};
constexpr int S = 96;                                       // windows per CTA (tile stride)
constexpr size_t SMEM = (size_t)(NJ + 2 * NP) * S * sizeof(double);
static_assert(SMEM <= 232448, "tile exceeds 227 KB");

#define SMD(buf, idx) (buf)[(idx) * S]

CPI_DEV void ld(const double* b, int off, double* x) {
#pragma unroll
    for (int k = 0; k < 9; k++) x[k] = SMD(b, off + k);
}
CPI_DEV void ldS(const double* b, int off, double* x) {        // packed symmetric -> full
    const double a0 = SMD(b, off), a1 = SMD(b, off + 1), a2 = SMD(b, off + 2), a3 = SMD(b, off + 3), a4 = SMD(b, off + 4), a5 = SMD(b, off + 5);
    x[0] = a0; x[1] = a1; x[2] = a2; x[3] = a1; x[4] = a3; x[5] = a4; x[6] = a2; x[7] = a4; x[8] = a5;
}
CPI_DEV void st(double* b, int off, const double* x) {
#pragma unroll
    for (int k = 0; k < 9; k++) SMD(b, off + k) = x[k];
}
// C += A B
CPI_DEV void amm(const double* A, const double* B, double* C) {
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++)
#pragma unroll
            for (int m = 0; m < 3; m++) C[3 * i + j] = fma(A[3 * i + m], B[3 * m + j], C[3 * i + j]);
}
// C += A B^T
CPI_DEV void ammT(const double* A, const double* B, double* C) {
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++)
#pragma unroll
            for (int m = 0; m < 3; m++) C[3 * i + j] = fma(A[3 * i + m], B[3 * j + m], C[3 * i + j]);
}
// C = A + s B
CPI_DEV void axpy(const double* A, double s, const double* B, double* C) {
#pragma unroll
    for (int k = 0; k < 9; k++) C[k] = fma(s, B[k], A[k]);
}
// packed upper triangle of C (+ d I), C symmetric in exact arithmetic
CPI_DEV void stS(double* b, int off, const double* C, double d) {
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = i; j < 3; j++) SMD(b, off + sym3(i, j)) = C[3 * i + j] + (i == j ? d : 0.0);
}

// One Phi P Phi^T + Q step: reads the old tile Po, writes the new tile Pn.  Rows are processed block by block; X = Phi P.
CPI_DEV void cov_step(const double* Po, double* Pn, const double* Rs, const double* Jt, const double* M, const double* B, double pgg,
                      double paa, double dt, double hdt2, const double* Jr, double q_w, double q_a) {
    {   // ---- row theta:  X_tt = Rs P_tt + Jt P_gt,  X_tg = Rs P_tg + pgg Jt
        double tt[9], tg[9], xtt[9], xtg[9];
        ldS(Po, TT, tt); ld(Po, TG, tg);
#pragma unroll
        for (int k = 0; k < 9; k++) { xtt[k] = 0.0; xtg[k] = pgg * Jt[k]; }
        amm(Rs, tt, xtt); ammT(Jt, tg, xtt);           // Jt P_gt = Jt P_tg^T
        amm(Rs, tg, xtg);
        st(Pn, TG, xtg);
        double n[9];
#pragma unroll
        for (int k = 0; k < 9; k++) n[k] = 0.0;
        ammT(xtt, Rs, n); ammT(xtg, Jt, n);
        double jj[9];
#pragma unroll
        for (int k = 0; k < 9; k++) jj[k] = 0.0;
        ammT(Jr, Jr, jj);
        const double qw = q_w * dt;
#pragma unroll
        for (int k = 0; k < 9; k++) n[k] = fma(qw, jj[k], n[k]);
        stS(Pn, TT, n, 0.0);
    }
    {   // ---- row v:  X_vt = P_vt + Vt P_tt,  X_vg = P_vg + Vt P_tg,  X_vv = P_vv + Vt P_tv + Va P_av,  X_va = P_va + paa Va
        double Vt[9], Va[9], xvt[9], xvg[9], xva[9];
#pragma unroll
        for (int k = 0; k < 9; k++) { Vt[k] = M[k] * dt; Va[k] = B[k] * dt; }
        {
            double tt[9], tg[9];
            ld(Po, VT, xvt); ld(Po, VG, xvg); ldS(Po, TT, tt); ld(Po, TG, tg);
            amm(Vt, tt, xvt); amm(Vt, tg, xvg);
        }
        ld(Po, VA, xva);
#pragma unroll
        for (int k = 0; k < 9; k++) xva[k] = fma(paa, Va[k], xva[k]);
        st(Pn, VG, xvg); st(Pn, VA, xva);
        {   // P'_vt = X_vt Rs^T + X_vg Jt^T
            double n[9];
#pragma unroll
            for (int k = 0; k < 9; k++) n[k] = 0.0;
            ammT(xvt, Rs, n); ammT(xvg, Jt, n);
            st(Pn, VT, n);
        }
        {   // P'_vv = X_vv + X_vt Vt^T + X_va Va^T + q_a dt I
            double x[9], vt[9], va[9];
            ldS(Po, VV, x); ld(Po, VT, vt); ld(Po, VA, va);
            ammT(Vt, vt, x); ammT(Va, va, x);
            ammT(xvt, Vt, x); ammT(xva, Va, x);
            stS(Pn, VV, x, q_a * dt);
        }
    }
    {   // ---- row p:  X_pK = P_pK + Pt P_tK + dt P_vK + Pa P_aK
        double Pt[9], Pa[9], xpt[9], xpg[9], xpa[9];
#pragma unroll
        for (int k = 0; k < 9; k++) { Pt[k] = M[k] * hdt2; Pa[k] = B[k] * hdt2; }
        {
            double a[9];
            ld(Po, PT, xpt); ldS(Po, TT, a); amm(Pt, a, xpt); ld(Po, VT, a); axpy(xpt, dt, a, xpt);
            ld(Po, PG, xpg); ld(Po, TG, a); amm(Pt, a, xpg); ld(Po, VG, a); axpy(xpg, dt, a, xpg);
            ld(Po, PA, xpa); ld(Po, VA, a); axpy(xpa, dt, a, xpa);
#pragma unroll
            for (int k = 0; k < 9; k++) xpa[k] = fma(paa, Pa[k], xpa[k]);
        }
        st(Pn, PG, xpg); st(Pn, PA, xpa);
        {   // P'_pt = X_pt Rs^T + X_pg Jt^T
            double n[9];
#pragma unroll
            for (int k = 0; k < 9; k++) n[k] = 0.0;
            ammT(xpt, Rs, n); ammT(xpg, Jt, n);
            st(Pn, PT, n);
        }
        double xpv[9];
        {   // X_pv = P_pv + Pt P_tv + dt P_vv + Pa P_av;  P'_pv = X_pv + X_pt Vt^T + X_pa Va^T + q_a dt^2/2 I
            double a[9];
            ld(Po, PV, xpv); ld(Po, VT, a); ammT(Pt, a, xpv); ldS(Po, VV, a); axpy(xpv, dt, a, xpv); ld(Po, VA, a); ammT(Pa, a, xpv);
            double n[9], Vt[9], Va[9];
#pragma unroll
            for (int k = 0; k < 9; k++) { n[k] = xpv[k]; Vt[k] = M[k] * dt; Va[k] = B[k] * dt; }
            ammT(xpt, Vt, n); ammT(xpa, Va, n);
            const double q = q_a * hdt2;
#pragma unroll
            for (int k = 0; k < 9; k += 4) n[k] += q;
            st(Pn, PV, n);
        }
        {   // X_pp = P_pp + Pt P_tp + dt P_vp + Pa P_ap;  P'_pp = X_pp + X_pt Pt^T + dt X_pv + X_pa Pa^T + q_a dt^3/4 I
            double x[9], a[9];
            ldS(Po, PP, x); ld(Po, PT, a); ammT(Pt, a, x); ld(Po, PV, a);
#pragma unroll
            for (int i = 0; i < 3; i++)
#pragma unroll
                for (int j = 0; j < 3; j++) x[3 * i + j] = fma(dt, a[3 * j + i], x[3 * i + j]);
            ld(Po, PA, a); ammT(Pa, a, x);
            ammT(xpt, Pt, x); axpy(x, dt, xpv, x); ammT(xpa, Pa, x);
            stS(Pn, PP, x, q_a * (hdt2 * dt) * 0.5);
        }
    }
}

}  // namespace

__global__ void __launch_bounds__(S, 1) k_preintegrate_discrete(const PreintParams p, int avg) {
    extern __shared__ __align__(16) double smem_d[];
    const int tid = threadIdx.x;
    const int64_t win = (int64_t)blockIdx.x * p.wpb + tid;
    if (tid >= p.wpb || win >= p.n_windows) return;
    double* Jt_ = smem_d + tid;                              // Jacobian state
    double* P = smem_d + (size_t)NJ * S + tid;               // covariance tile (ping-pongs with Pn every step)
    double* Pn = P + (size_t)NP * S;

    const double* lin = reinterpret_cast<const double*>(p.lin) + win * CPI_LIN_DOUBLES;
    const double bw[3] = {lin[0], lin[1], lin[2]}, ba[3] = {lin[3], lin[4], lin[5]};
    int64_t o0, nsteps;
    if (p.offsets) { o0 = p.offsets[win]; nsteps = p.offsets[win + 1] - o0 - avg; }
    else { o0 = win * (p.ns_uniform + avg); nsteps = p.ns_uniform; }
    if (nsteps < 0) nsteps = 0;
    const double* sp = reinterpret_cast<const double*>(p.samples) + o0 * CPI_SAMPLE_DOUBLES;

    // ---- state: the zero-step record, or the record to continue from
    double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    double alpha[3] = {0, 0, 0}, beta[3] = {0, 0, 0}, DT = 0.0, pgg = 0.0, paa = 0.0;
    if (p.init) {
        const double* rin = reinterpret_cast<const double*>(p.init) + win * (int64_t)CPI_REC_V1_DOUBLES;
        const double* Pm = rin + CPI_REC_P;
        auto g = [&](int r, int c) { return Pm[r + 15 * c]; };
        DT = rin[CPI_REC_DT]; pgg = g(3, 3); paa = g(9, 9);
#pragma unroll
        for (int e = 0; e < 3; e++) { alpha[e] = rin[CPI_REC_ALPHA + e]; beta[e] = rin[CPI_REC_BETA + e]; }
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) {
                const int e = 3 * i + j, c = i + 3 * j;
                R[e] = rin[CPI_REC_R + c];
                SMD(Jt_, J_Q + e) = rin[CPI_REC_JQ + c]; SMD(Jt_, J_A + e) = rin[CPI_REC_JA + c]; SMD(Jt_, J_B + e) = rin[CPI_REC_JB + c];
                SMD(Jt_, H_A + e) = rin[CPI_REC_HA + c]; SMD(Jt_, H_B + e) = rin[CPI_REC_HB + c];
                SMD(P, TG + e) = g(i, 3 + j); SMD(P, VT + e) = g(6 + i, j); SMD(P, VG + e) = g(6 + i, 3 + j); SMD(P, VA + e) = g(6 + i, 9 + j);
                SMD(P, PT + e) = g(12 + i, j); SMD(P, PG + e) = g(12 + i, 3 + j); SMD(P, PV + e) = g(12 + i, 6 + j); SMD(P, PA + e) = g(12 + i, 9 + j);
                if (i <= j) { SMD(P, TT + sym3(i, j)) = g(i, j); SMD(P, VV + sym3(i, j)) = g(6 + i, 6 + j); SMD(P, PP + sym3(i, j)) = g(12 + i, 12 + j); }
            }
    } else {
#pragma unroll 1
        for (int e = 0; e < NP; e++) SMD(P, e) = 0.0;
#pragma unroll 1
        for (int e = 0; e < NJ; e++) SMD(Jt_, e) = 0.0;
    }

#pragma unroll 1
    for (int64_t it = 0; it < nsteps; it++) {
        const double* s = sp + it * CPI_SAMPLE_DOUBLES;
        const double dt = __ldg(s + 6);
        DT += dt;
        if (dt == 0.0) continue;                         // CpiV1.h:72-74
        double wh[3], ah[3];
#pragma unroll
        for (int e = 0; e < 3; e++) { wh[e] = __ldg(s + e) - bw[e]; ah[e] = __ldg(s + 3 + e) - ba[e]; }
        if (avg) {
#pragma unroll
            for (int e = 0; e < 3; e++) {
                wh[e] += __ldg(s + CPI_SAMPLE_DOUBLES + e) - bw[e]; wh[e] = 0.5 * wh[e];
                ah[e] += __ldg(s + CPI_SAMPLE_DOUBLES + 3 + e) - ba[e]; ah[e] = 0.5 * ah[e];
            }
        }
        // ---- model 1's closed forms (preintegrate.cu front_step; CpiV1.h:101-124, 162-167)
        const double mag = sqrt(wh[0] * wh[0] + wh[1] * wh[1] + wh[2] * wh[2]);
        const double th = mag * dt;
        const bool small_w = mag < 0.008726646;
        double sn, cs_;
        sincos(th, &sn, &cs_);
        const double im = small_w ? 0.0 : 1.0 / mag, im2 = im * im;
        const double a1 = small_w ? dt : sn * im, b1 = small_w ? (dt * dt) * 0.5 : (1.0 - cs_) * im2;
        const double ith = small_w ? 0.0 : 1.0 / th;
        const double c1 = small_w ? 0.5 : (1.0 - cs_) * (ith * ith), c2 = small_w ? (1.0 / 6.0) : (th - sn) * (ith * ith * ith);
        const double ca = c1 * dt, cb = c2 * dt * dt;
        const double W2[9] = {-(wh[1] * wh[1] + wh[2] * wh[2]), wh[0] * wh[1], wh[0] * wh[2],
                              wh[0] * wh[1], -(wh[0] * wh[0] + wh[2] * wh[2]), wh[1] * wh[2],
                              wh[0] * wh[2], wh[1] * wh[2], -(wh[0] * wh[0] + wh[1] * wh[1])};
        const double Wm[9] = {0.0, -wh[2], wh[1], wh[2], 0.0, -wh[0], -wh[1], wh[0], 0.0};
        double Rs[9], Jr[9], Jt[9], M[9], B[9];
#pragma unroll
        for (int e = 0; e < 9; e++) {
            const double d = (e % 4 == 0) ? 1.0 : 0.0;
            Rs[e] = d + (-a1 * Wm[e] + b1 * W2[e]);      // rot_apply's D = I - a W + b W^2
            Jr[e] = d - ca * Wm[e] + cb * W2[e];
            Jt[e] = -(Jr[e] * dt);
        }
        {
            double r2[9];
            mul33(Rs, R, r2);
            // M = -R^T [a_hat x] (rows: a_hat x column i of R), B = -R^T, both at the step's start rotation
#pragma unroll
            for (int i = 0; i < 3; i++) {
                const double r[3] = {R[i], R[3 + i], R[6 + i]};
                cross(ah, r, &M[3 * i]);
#pragma unroll
                for (int j = 0; j < 3; j++) B[3 * i + j] = -R[3 * j + i];
            }
            // ---- means:  beta' = beta + R^T a dt,  alpha' = alpha + beta dt + R^T a dt^2/2
            const double hdt2 = (dt * dt) * 0.5;
            double ra[3];
            mvT33(R, ah, ra);
#pragma unroll
            for (int e = 0; e < 3; e++) { alpha[e] = (alpha[e] + beta[e] * dt) + ra[e] * hdt2; beta[e] = beta[e] + ra[e] * dt; }
            // ---- bias Jacobians (old J_q, J_b, H_b):  R^T [a x] J_q = -M J_q
            {
                double jq[9], mj[9], jn[9];
                ld(Jt_, J_Q, jq);
#pragma unroll
                for (int k = 0; k < 9; k++) { mj[k] = 0.0; jn[k] = Jr[k] * dt; }
                amm(M, jq, mj);
                amm(Rs, jq, jn);
                st(Jt_, J_Q, jn);
#pragma unroll
                for (int k = 0; k < 9; k++) {
                    const double jb = SMD(Jt_, J_B + k), hb = SMD(Jt_, H_B + k);
                    SMD(Jt_, J_A + k) = (SMD(Jt_, J_A + k) + jb * dt) - mj[k] * hdt2;
                    SMD(Jt_, J_B + k) = jb - mj[k] * dt;
                    SMD(Jt_, H_A + k) = (SMD(Jt_, H_A + k) + hb * dt) + B[k] * hdt2;
                    SMD(Jt_, H_B + k) = hb + B[k] * dt;
                }
            }
            // ---- covariance
            cov_step(P, Pn, Rs, Jt, M, B, pgg, paa, dt, hdt2, Jr, p.q_w, p.q_a);
            { double* t = P; P = Pn; Pn = t; }
            pgg += p.q_wb * dt;
            paa += p.q_ab * dt;
#pragma unroll
            for (int e = 0; e < 9; e++) R[e] = r2[e];
        }
    }

    // ---- write the record (column-major 3x3 / 15x15, include/cpi_b200.h); every symmetric pair from one value
    double* rec = reinterpret_cast<double*>(p.out) + win * (int64_t)CPI_REC_V1_DOUBLES;
    {
        double q[4];
        rot_2_quat(R, q);
        rec[CPI_REC_Q] = q[0]; rec[CPI_REC_Q + 1] = q[1]; rec[CPI_REC_Q + 2] = q[2]; rec[CPI_REC_Q + 3] = q[3];
    }
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) {
            const int e = 3 * i + j, c = i + 3 * j;
            rec[CPI_REC_R + c] = R[e];
            rec[CPI_REC_JQ + c] = SMD(Jt_, J_Q + e); rec[CPI_REC_JA + c] = SMD(Jt_, J_A + e); rec[CPI_REC_JB + c] = SMD(Jt_, J_B + e);
            rec[CPI_REC_HA + c] = SMD(Jt_, H_A + e); rec[CPI_REC_HB + c] = SMD(Jt_, H_B + e);
        }
#pragma unroll
    for (int e = 0; e < 3; e++) { rec[CPI_REC_ALPHA + e] = alpha[e]; rec[CPI_REC_BETA + e] = beta[e]; }
    rec[CPI_REC_DT] = DT;
    double* Pm = rec + CPI_REC_P;
    auto put = [&](int r, int c, double v) { Pm[r + 15 * c] = v; };
#pragma unroll 1
    for (int i = 0; i < 3; i++)
#pragma unroll 1
        for (int j = 0; j < 3; j++) {
            const int sidx = sym3(i, j);
            put(i, j, SMD(P, TT + sidx));            put(6 + i, 6 + j, SMD(P, VV + sidx));      put(12 + i, 12 + j, SMD(P, PP + sidx));
            put(3 + i, 3 + j, i == j ? pgg : 0.0);   put(9 + i, 9 + j, i == j ? paa : 0.0);
            put(i, 9 + j, 0.0); put(9 + j, i, 0.0); put(3 + i, 9 + j, 0.0); put(9 + j, 3 + i, 0.0);
            double v;
            v = SMD(P, TG + 3 * i + j); put(i, 3 + j, v);      put(3 + j, i, v);
            v = SMD(P, VT + 3 * i + j); put(6 + i, j, v);      put(j, 6 + i, v);
            v = SMD(P, VG + 3 * i + j); put(6 + i, 3 + j, v);  put(3 + j, 6 + i, v);
            v = SMD(P, VA + 3 * i + j); put(6 + i, 9 + j, v);  put(9 + j, 6 + i, v);
            v = SMD(P, PT + 3 * i + j); put(12 + i, j, v);     put(j, 12 + i, v);
            v = SMD(P, PG + 3 * i + j); put(12 + i, 3 + j, v); put(3 + j, 12 + i, v);
            v = SMD(P, PV + 3 * i + j); put(12 + i, 6 + j, v); put(6 + j, 12 + i, v);
            v = SMD(P, PA + 3 * i + j); put(12 + i, 9 + j, v); put(9 + j, 12 + i, v);
        }
}

#undef SMD

int preint_discrete_cap() { return S; }

cudaError_t preint_launch_discrete(int flags, const PreintParams& p0, int num_sms, cudaStream_t st) {
    PreintParams p = p0;
    if (p.n_windows == 0) return cudaSuccess;
    // windows per CTA: spread a small batch over all SMs in one wave, else the tile's capacity
    if (p.wpb <= 0 || p.wpb > S) {
        const int64_t need = (p.n_windows + num_sms - 1) / num_sms;
        p.wpb = need < 1 ? 1 : (need > S ? S : (int)need);
    }
    static bool configured[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 64 || !configured[dev]) {
        cudaError_t e = cudaFuncSetAttribute(k_preintegrate_discrete, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM);
        if (e != cudaSuccess) return e;
        if (dev < 64) configured[dev] = true;
    }
    const int block = (p.wpb + 31) / 32 * 32;
    const int grid = (int)((p.n_windows + p.wpb - 1) / p.wpb);
    k_preintegrate_discrete<<<grid, block, SMEM, st>>>(p, (flags & CPI_FLAG_IMU_AVG) ? 1 : 0);
    return cudaGetLastError();
}

}  // namespace cpi
