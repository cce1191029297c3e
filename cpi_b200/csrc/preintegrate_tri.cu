// K1 / K2, "tri-lane" mapping: THREE LANES PER WINDOW, ten windows per warp, the per-window state distributed over the
// three lanes' REGISTERS and exchanged with warp shuffles.  CpiV1::feed_IMU (cpi/CpiV1.h:62-361) and CpiV2::feed_IMU
// (cpi/CpiV2.h:84-467, state_transition_jacobians = true) of rpng/cpi.  Default kernels for the non-imu_avg modes; the
// lane-per-window kernels of preintegrate.cu serve imu_avg and model 2's analytic-Jacobian mode.
//
// Why three: every quantity on the path is a 3-vector or a 3x3 block, and every equation is equivariant under a CYCLIC
// relabelling of the three axes (a proper rotation: cross products keep their form).  Lane c of a window works in the
// frame whose axes are (c, c+1, c+2) and owns COLUMN 0 of every 3x3 block IN ITS OWN FRAME -- i.e. original column c,
// stored in the order (c, c+1, c+2).  All three lanes therefore execute the same instructions on "column 0", register
// indices are static everywhere, and fetching a neighbour's column is two or three SHFLs with a fixed index permutation
// (gather_cols).  Window-uniform inputs (w_hat, a_hat, the rotations) are simply read / gathered in rotated order.
//
// Covariance blocks are stored in the orientation that makes the Lyapunov right-hand side column-local
// (P_dot = F P + P F^T; column c of F_IK P_KJ needs only column c of P_KJ, column c of P_IK F_JK^T needs all of P_IK
// unless F_JK is the identity):
//     TG = P_theta,bg   TT = P_theta,theta   GV = P_bg,v   TV = P_theta,v   AV = P_ba,v   VV = P_v,v
//     TP = P_theta,p    GP = P_bg,p          AP = P_ba,p   VP = P_v,p       PP = P_p,p
// With this choice only FOUR quantities per RK4 stage cross lanes: the full TG and TT stage values (needed by GV, TV)
// and one row of the symmetric VV / PP right-hand sides: 13 doubles per stage per lane instead of the 943 shared-memory
// operations per sample of the lane-per-window layout, and the covariance tile no longer lives in shared memory at
// all (residency is register-bound, not smem-bound).  The four RK4 stages are the reference's (CpiV1.h:272-353).
//
// Issue rates the mapping rests on (tools/microbench.cu): SHFL.b32 = 1 warp-instr/clk/SM, LDS.64 = 1 warp-instr/clk/SM on the
// same MIO pipe, DFMA = 2 warp-instr/clk/SM, and SHFL overlaps with DFMA.
#include <cstdlib>
#include "cpi_common.cuh"
#include "cpi_kernels.h"
#include "tma.cuh"

namespace cpi {

constexpr int TRI_WPW = 10;                 // windows per warp (lanes 30, 31 idle)
// CTA = ONE warp = ten windows.  Nothing in the kernel is shared between warps, so one-warp CTAs cost nothing and buy (a) even
// distribution by the hardware block scheduler (10 000 windows = 1 000 CTAs over 132 SMs: 7 or 8 per SM, one wave), (b) kernels of
// different streams co-residing on an SM, which is what lets the host entry point pipeline a batch in many small chunks, and (c) a
// finer tail on multi-wave batches.  Up to 8 CTAs per SM: 255 registers x 32 lanes x 8 = the register file; shared memory per CTA is
// kept under 220 KB / 8 for every instantiation (model 1 fp64: 21 KB, model 2 fp64: 24 KB).
template <int MODEL, class T> struct TriNT { static constexpr int NT = 32; };
constexpr int TRI_NBUF = 3;                 // 128-byte chunk buffers per window (TMA ring)
constexpr int TRI_BUF_STRIDE = TRI_NBUF * 128 + 16;   // bytes of sample staging per window, + 16 B pad (bank spread; 16-B aligned for TMA)
// doubles per window of pre-pass scalars: 3 samples x 16 (model 1: 15 used) or 3 x 10 (model 2: 9 used), padded for bank spread
// (strides are multiples of 2 doubles so that the sets can be moved with 16-byte accesses: 50 / 34 doubles = a 4-bank shift per window)
template <int MODEL> struct TriSC { static constexpr int PER = (MODEL == 1) ? 16 : 10, STRIDE = (MODEL == 1) ? 50 : 34; };

template <class T> CPI_DEV T shf(T v, int src) { return __shfl_sync(0xffffffffu, v, src); }

// columns 1 and 2 (own frame) of a block whose column 0 each lane of the trio holds:  X1[k] = next.V[(k+2)%3], X2[k] = prev.V[(k+1)%3]
template <class T> CPI_DEV void gather_cols(const T* V, int nx, int pv, T* X1, T* X2) {
    X1[0] = shf(V[2], nx); X1[1] = shf(V[0], nx); X1[2] = shf(V[1], nx);
    X2[0] = shf(V[1], pv); X2[1] = shf(V[2], pv); X2[2] = shf(V[0], pv);
}

// ---- per-model layout --------------------------------------------------------------------------------------------------
// RK4 stage values handed from the (theta|v)-column group to the p-column group through LANE-PRIVATE shared memory
// slots, [entry][thread]: TV, GV (model 2: + CV) for the four stages.
template <int MODEL> struct TriL {
    static constexpr int NSL = (MODEL == 1 ? 6 : 9) * 4 + (MODEL == 1 ? 0 : 9);   // TV, GV (+ CV) for the four stages; model 2: + TG(start) columns 1, 2 and TT(start) 11, 21, 22
    // front state parked in lane-private smem during the covariance step: bw, ba, alpha, beta, then
    //   model 1: J_q, J_a, J_b, H_a, H_b (own columns)      model 2: g_k and the own columns of the 7 non-trivial Discrete_J_b blocks
    static constexpr int NFS = (MODEL == 1) ? 23 : 32;
};
enum : int { FS_BW = 0, FS_BA = 3, FS_AL = 6, FS_BE = 7, FS_JQ = 8, FS_JA = 11, FS_JB = 14, FS_HA = 17, FS_HB = 20,
             FS_GK = 8, FS_DTG = 11, FS_DVG = 14, FS_DPG = 17, FS_DVA = 20, FS_DPA = 23, FS_DVL = 26, FS_DPL = 29 };
template <int MODEL, class T> struct TriSmem {
    static constexpr int NT = TriNT<MODEL, T>::NT;
    static constexpr int WPB = TRI_WPW * NT / 32;                     // window slots per CTA
    static constexpr size_t off_fs = (size_t)TriL<MODEL>::NSL * NT * sizeof(T);
    static constexpr size_t off_sc = off_fs + (size_t)TriL<MODEL>::NFS * NT * 8;
    // scalar sets: one slot per window + one dummy slot per warp for the two idle lanes
    static constexpr size_t off_buf = (off_sc + (size_t)(WPB + NT / 32) * TriSC<MODEL>::STRIDE * 8 + 127) / 128 * 128;
    static constexpr size_t off_bar = off_buf + (size_t)WPB * TRI_BUF_STRIDE;
    static constexpr size_t bytes = off_bar + (size_t)WPB * 8 * TRI_NBUF;
};
static_assert(TriSmem<1, double>::bytes <= 28160 - 1024 && TriSmem<1, float>::bytes <= 28160 - 1024 && TriSmem<2, double>::bytes <= 28160 - 1024 &&
              TriSmem<2, float>::bytes <= 28160 - 1024,
              "8 CTAs per SM need <= 220 KB / 8 of shared memory each (incl. 1 KB the system reserves per CTA)");

#define SLT(e) sl[(e) * NT]
#define FST(e) fs[(e) * NT]
#define CN(s) ((s) < 2 ? hdt : dt)                       /* x_{s+2} = x_1 + CN(s) k_{s+1}:  dt/2, dt/2, dt   (CpiV1.h:312, 323, 344) */
#define KSUM(ks, k, s) ((s) == 0 ? (k) : ((s) == 3 ? (ks) + (k) : fma(T(2), (k), (ks))))   /* ((k1 + 2 k2) + 2 k3) + k4  (CpiV1.h:352) */
#define CPI_FENCE() asm volatile("" ::: "memory")

// -(R^T u): element i = -(column i of R) . u      (R row-major 3x3)
template <class T> CPI_DEV void negRt(const T* R, const T* u, T* o) {
#pragma unroll
    for (int i = 0; i < 3; i++) o[i] = -(R[i] * u[0] + R[3 + i] * u[1] + R[6 + i] * u[2]);
}

// Covariance state of one lane (column 0 of each block in the lane's frame).  Held in fp64 also by the fp32-storage variant: the
// four RK4 stages run in T, but the state is ACCUMULATED in double (P += dt/6 * ksum), so 200 steps do not random-walk the
// state's 24-bit rounding (worst 3x3 block of P vs the fp64 oracle: 1.9e-6 with a float state, ~1e-7 with a double one).
template <class T> struct TriP {
    double TG[3], TT[3], GV[3], TV[3], AV[3], VV[3], TP[3], GP[3], AP[3], VP[3], PP[3];
};

// One RK4 step of the covariance (model 1: CpiV1.h:272-353).  w, ah: estimated readings; R, Rm, R1: old / mid / new
// rotation (row-major, lane frame); pgg, paa: the scalar diagonal blocks P_bg,bg and P_ba,ba at the start of the step.
template <int MODEL, int NT, class T>
CPI_DEV void tri_cov_step(TriP<T>& P, T* sl, const T* w, const T* ah, const T* gt, const T* R, const T* Rm, const T* R1, T pgg, T paa, T dt, T dt6,
                          T q_w, T q_wb, T q_a, T q_ab, int nx, int pv) {
    const T hdt = dt * T(0.5);
    constexpr int NS = (MODEL == 1) ? 6 : 9;              // slot entries per stage: TV, GV (+ CV)
    constexpr int SL_CV = 6;
    constexpr bool PARK = MODEL == 2 && sizeof(T) == 8;   // model 2 fp64: halves the register spills (ptxas: 200 -> 116 B of spill stores per sample)
    // Model 2 (CpiV2.h:326-443): the clone rows c of P_big are re-initialised from the theta rows at every step (B_k), so within a
    // step  P_cg = TG(start), P_cc = TT(start), P_ca = 0  are constant and only three transient blocks evolve:
    //     TC = P_theta,c  (starts as TT):  TC' = -W TC - TG(start)^T            [needs nothing cross-lane; TV and CV need all of it]
    //     CV = P_c,v      (starts as TV):  CV' = TC^T A_s^T + TT(start) C_s^T
    //     CP = P_c,p      (starts as TP):  CP' = CV                            [recomputed from CV's stage values]
    // and the v rows gain  C_s P_c,J  with  C_s = -R_s^T [g_tau x]  (CpiV2.h:335).
    {   // ---- group 1a: TG, TT, GV, TV, stage by stage (self-contained: needs only w, the rotations and a_hat)
        T xTG[3], xTT[3], xGV[3], xTV[3], xTC[3], xCV[3];
        T sTG[3], sTT[3], sGV[3], sTV[3];
        T G1s[3], G2s[3], tts[3];                             // model 2: TG(start) columns 1, 2 and TT(start) entries 11, 21, 22
        T oTG[3], oTT[3], oGV[3], oTV[3];                     // start-of-step values in the arithmetic type
#pragma unroll
        for (int e = 0; e < 3; e++) { oTG[e] = (T)P.TG[e]; oTT[e] = (T)P.TT[e]; oGV[e] = (T)P.GV[e]; oTV[e] = (T)P.TV[e]; }
#pragma unroll
        for (int e = 0; e < 3; e++) { xTG[e] = oTG[e]; xTT[e] = oTT[e]; xGV[e] = oGV[e]; xTV[e] = oTV[e]; xTC[e] = oTT[e]; xCV[e] = oTV[e]; }
#pragma unroll
        for (int s = 0; s < 4; s++) {
            const T* Rs = (s == 0) ? R : (s == 3 ? R1 : Rm);
            const T rc[3] = {Rs[0], Rs[3], Rs[6]};            // column 0 of R_s
            T a0[3];
            cross(ah, rc, a0);                                // row 0 of A_s = -R_s^T [a x]  (row i = a x r_i)
            // cross-lane: full TG_s, the three missing entries of the symmetric TT_s
            T TG1[3], TG2[3];
            gather_cols(xTG, nx, pv, TG1, TG2);
            const T t11 = shf(xTT[0], nx), t21 = shf(xTT[1], nx), t22 = shf(xTT[0], pv);
            // stage values the later groups need
#pragma unroll
            for (int e = 0; e < 3; e++) { SLT(s * NS + e) = xTV[e]; SLT(s * NS + 3 + e) = xGV[e]; if (MODEL == 2) SLT(s * NS + SL_CV + e) = xCV[e]; }
            const T pg_s = (s == 0) ? pgg : fma(q_wb, (s == 3 ? dt : hdt), pgg);
            T kTG[3], kTT[3], kGV[3], kTV[3];
            T c0[3], TC1[3], TC2[3];
            if (MODEL == 2) {
                cross(gt, rc, c0);                            // row 0 of C_s = -R_s^T [g_tau x]
                if (s == 0) {
#pragma unroll
                    for (int e = 0; e < 3; e++) { G1s[e] = TG1[e]; G2s[e] = TG2[e]; }
                    tts[0] = t11; tts[1] = t21; tts[2] = t22;
                    if (PARK) {                               // constant over the step: parked in lane-private slots rather than held in 18 registers
#pragma unroll
                        for (int e = 0; e < 3; e++) { SLT(4 * NS + e) = TG1[e]; SLT(4 * NS + 3 + e) = TG2[e]; }
                        SLT(4 * NS + 6) = t11; SLT(4 * NS + 7) = t21; SLT(4 * NS + 8) = t22;
                    }
                    TC1[0] = xTT[1]; TC1[1] = t11; TC1[2] = t21; TC2[0] = xTT[2]; TC2[1] = t21; TC2[2] = t22;   // TC(start) = TT(start), symmetric
                } else {
                    gather_cols(xTC, nx, pv, TC1, TC2);
                    if (PARK) {
#pragma unroll
                        for (int e = 0; e < 3; e++) { G1s[e] = SLT(4 * NS + e); G2s[e] = SLT(4 * NS + 3 + e); tts[e] = SLT(4 * NS + 6 + e); }
                    }
                }
            }
            // TG:  -W x - pgg_s I
            cross(xTG, w, kTG);
            kTG[0] -= pg_s;
            // TT:  N + N^T + q_w I,  N = -W TT - TG^T  ->  N[:,0] = TT_0 x w - row0(TG),  N[0,j] = (TT_j x w)[0] - TG[j,0]
            {
                T n0[3];
                cross(xTT, w, n0);
                n0[0] -= xTG[0]; n0[1] -= TG1[0]; n0[2] -= TG2[0];
                const T n01 = (t11 * w[2] - t21 * w[1]) - xTG[1];     // TT_1 = (TT01, TT11, TT21)
                const T n02 = (t21 * w[2] - t22 * w[1]) - xTG[2];     // TT_2 = (TT02, TT12, TT22)
                kTT[0] = n0[0] + n0[0] + q_w; kTT[1] = n0[1] + n01; kTT[2] = n0[2] + n02;
            }
            // GV:  TG^T A_s[0,:]^T  -> element i = (column i of TG) . a0
            kGV[0] = xTG[0] * a0[0] + xTG[1] * a0[1] + xTG[2] * a0[2];
            kGV[1] = TG1[0] * a0[0] + TG1[1] * a0[1] + TG1[2] * a0[2];
            kGV[2] = TG2[0] * a0[0] + TG2[1] * a0[1] + TG2[2] * a0[2];
            // TV:  -W TV - GV + TT A_s[0,:]^T
            cross(xTV, w, kTV);
            kTV[0] = fma(xTT[2], a0[2], fma(xTT[1], a0[1], fma(xTT[0], a0[0], kTV[0] - xGV[0])));      // one accumulation chain per entry
            kTV[1] = fma(t21, a0[2], fma(t11, a0[1], fma(xTT[1], a0[0], kTV[1] - xGV[1])));
            kTV[2] = fma(t22, a0[2], fma(t21, a0[1], fma(xTT[2], a0[0], kTV[2] - xGV[2])));
            T kTC[3], kCV[3];
            if (MODEL == 2) {
                // GV += TG(start)^T C_s[0,:]^T ;  TV += TC C_s[0,:]^T
                kGV[0] += oTG[0] * c0[0] + oTG[1] * c0[1] + oTG[2] * c0[2];
                kGV[1] += G1s[0] * c0[0] + G1s[1] * c0[1] + G1s[2] * c0[2];
                kGV[2] += G2s[0] * c0[0] + G2s[1] * c0[1] + G2s[2] * c0[2];
#pragma unroll
                for (int e = 0; e < 3; e++) kTV[e] = fma(TC2[e], c0[2], fma(TC1[e], c0[1], fma(xTC[e], c0[0], kTV[e])));
                // TC:  -W TC - TG(start)^T  (column 0: minus row 0 of TG(start))
                cross(xTC, w, kTC);
                kTC[0] -= oTG[0]; kTC[1] -= G1s[0]; kTC[2] -= G2s[0];
                // CV:  TC^T A_s[0,:]^T + TT(start) C_s[0,:]^T
                kCV[0] = (xTC[0] * a0[0] + xTC[1] * a0[1] + xTC[2] * a0[2]) + (oTT[0] * c0[0] + oTT[1] * c0[1] + oTT[2] * c0[2]);
                kCV[1] = (TC1[0] * a0[0] + TC1[1] * a0[1] + TC1[2] * a0[2]) + (oTT[1] * c0[0] + tts[0] * c0[1] + tts[1] * c0[2]);
                kCV[2] = (TC2[0] * a0[0] + TC2[1] * a0[1] + TC2[2] * a0[2]) + (oTT[2] * c0[0] + tts[1] * c0[1] + tts[2] * c0[2]);
            }
#pragma unroll
            for (int e = 0; e < 3; e++) {
                sTG[e] = KSUM(sTG[e], kTG[e], s); sTT[e] = KSUM(sTT[e], kTT[e], s); sGV[e] = KSUM(sGV[e], kGV[e], s); sTV[e] = KSUM(sTV[e], kTV[e], s);
                if (s < 3) {
                    xTG[e] = fma(kTG[e], CN(s), oTG[e]); xTT[e] = fma(kTT[e], CN(s), oTT[e]); xGV[e] = fma(kGV[e], CN(s), oGV[e]);
                    xTV[e] = fma(kTV[e], CN(s), oTV[e]);
                    if (MODEL == 2) { xTC[e] = fma(kTC[e], CN(s), oTT[e]); xCV[e] = fma(kCV[e], CN(s), oTV[e]); }
                }
            }
        }
#pragma unroll
        for (int e = 0; e < 3; e++) {
            P.TG[e] = fma((double)dt6, (double)sTG[e], P.TG[e]); P.TT[e] = fma((double)dt6, (double)sTT[e], P.TT[e]);
            P.GV[e] = fma((double)dt6, (double)sGV[e], P.GV[e]); P.TV[e] = fma((double)dt6, (double)sTV[e], P.TV[e]);
        }
    }
    CPI_FENCE();
    {   // ---- groups 1b + 2 fused: AV, VV, TP, GP, AP, VP, PP in ONE stage loop (AV / VV never go through the slots)
        T xAV[3], xVV[3], sAV[3], sVV[3], oAV[3], oVV[3];
        T xTP[3], xGP[3], xAP[3], xVP[3], oTP[3], oGP[3], oAP[3], oVP[3];
        T sTP[3], sGP[3], sAP[3], sVP[3], sPP[3];
#pragma unroll
        for (int e = 0; e < 3; e++) {
            oAV[e] = (T)P.AV[e]; oVV[e] = (T)P.VV[e]; xAV[e] = oAV[e]; xVV[e] = oVV[e];
            oTP[e] = (T)P.TP[e]; oGP[e] = (T)P.GP[e]; oAP[e] = (T)P.AP[e]; oVP[e] = (T)P.VP[e];
            xTP[e] = oTP[e]; xGP[e] = oGP[e]; xAP[e] = oAP[e]; xVP[e] = oVP[e];
        }
#pragma unroll
        for (int s = 0; s < 4; s++) {
            const T* Rs = (s == 0) ? R : (s == 3 ? R1 : Rm);
            const T rc[3] = {Rs[0], Rs[3], Rs[6]};
            T tv[3], gv[3], cv[3];
#pragma unroll
            for (int e = 0; e < 3; e++) { tv[e] = SLT(s * NS + e); gv[e] = SLT(s * NS + 3 + e); if (MODEL == 2) cv[e] = SLT(s * NS + SL_CV + e); }
            const T pa_s = (s == 0) ? paa : fma(q_ab, (s == 3 ? dt : hdt), paa);
            T kAV[3], kVV[3], kTP[3], kVP[3];
#pragma unroll
            for (int e = 0; e < 3; e++) kAV[e] = -(pa_s * rc[e]);
            {   // VV:  M + M^T + q_a I,  M[:,0] = -R_s^T (a x TV_0 + AV_0 (+ g_tau x CV_0))
                T u[3], m0[3];
                cross(ah, tv, u);
#pragma unroll
                for (int e = 0; e < 3; e++) u[e] += xAV[e];
                if (MODEL == 2) {
                    T u2[3];
                    cross(gt, cv, u2);
#pragma unroll
                    for (int e = 0; e < 3; e++) u[e] += u2[e];
                }
                negRt(Rs, u, m0);
                const T m01 = shf(m0[2], nx), m02 = shf(m0[1], pv);
                kVV[0] = m0[0] + m0[0] + q_a; kVV[1] = m0[1] + m01; kVV[2] = m0[2] + m02;
            }
            // TP:  -W TP - GP + TV
            cross(xTP, w, kTP);
#pragma unroll
            for (int e = 0; e < 3; e++) kTP[e] = (kTP[e] - xGP[e]) + tv[e];
            {   // VP:  A_s TP_0 + B_s AP_0 (+ C_s CP_0) + VV_0
                T u[3];
                cross(ah, xTP, u);
#pragma unroll
                for (int e = 0; e < 3; e++) u[e] += xAP[e];
                if (MODEL == 2) {
                    T cp[3], u2[3];
#pragma unroll
                    for (int e = 0; e < 3; e++) cp[e] = (s == 0) ? oTP[e] : fma((T)SLT((s - 1) * NS + SL_CV + e), CN(s - 1), oTP[e]);
                    cross(gt, cp, u2);
#pragma unroll
                    for (int e = 0; e < 3; e++) u[e] += u2[e];
                }
#pragma unroll
                for (int e = 0; e < 3; e++) kVP[e] = fma(-Rs[6 + e], u[2], fma(-Rs[3 + e], u[1], fma(-Rs[e], u[0], xVV[e])));
            }
            // PP' = VP + VP^T has no dependants: only the own-column integral of VP is accumulated here (P.PP holds Q = int VP[:,0]);
            // the transpose is added ONCE per window, when the record is written (PP = Q + Q^T), instead of one exchange per stage
#pragma unroll
            for (int e = 0; e < 3; e++) {
                sTP[e] = KSUM(sTP[e], kTP[e], s); sGP[e] = KSUM(sGP[e], gv[e], s); sAP[e] = KSUM(sAP[e], xAV[e], s);
                sVP[e] = KSUM(sVP[e], kVP[e], s); sPP[e] = KSUM(sPP[e], xVP[e], s);
                sAV[e] = KSUM(sAV[e], kAV[e], s); sVV[e] = KSUM(sVV[e], kVV[e], s);
                if (s < 3) {
                    xTP[e] = fma(kTP[e], CN(s), oTP[e]); xGP[e] = fma(gv[e], CN(s), oGP[e]); xAP[e] = fma(xAV[e], CN(s), oAP[e]);
                    xVP[e] = fma(kVP[e], CN(s), oVP[e]);
                    xAV[e] = fma(kAV[e], CN(s), oAV[e]); xVV[e] = fma(kVV[e], CN(s), oVV[e]);
                }
            }
        }
#pragma unroll
        for (int e = 0; e < 3; e++) {
            P.AV[e] = fma((double)dt6, (double)sAV[e], P.AV[e]); P.VV[e] = fma((double)dt6, (double)sVV[e], P.VV[e]);
            P.TP[e] = fma((double)dt6, (double)sTP[e], P.TP[e]); P.GP[e] = fma((double)dt6, (double)sGP[e], P.GP[e]);
            P.AP[e] = fma((double)dt6, (double)sAP[e], P.AP[e]); P.VP[e] = fma((double)dt6, (double)sVP[e], P.VP[e]);
            P.PP[e] = fma((double)dt6, (double)sPP[e], P.PP[e]);
        }
    }
    CPI_FENCE();
}

// D v  with  D = I - a [w x] + b [w x]^2 :   v - a (w x v) + b (w x (w x v));  second result with (a2, b2) on the same cross products
CPI_DEV void rot_col2(double a, double b, double a2, double b2, const double* w, const double* v, double* o, double* o2) {
    double t[3], u[3];
    cross(w, v, t);
    cross(w, t, u);
#pragma unroll
    for (int e = 0; e < 3; e++) { o[e] = (v[e] - a * t[e]) + b * u[e]; o2[e] = (v[e] - a2 * t[e]) + b2 * u[e]; }
}
CPI_DEV void rot_col(double a, double b, const double* w, const double* v, double* o) {
    double t[3], u[3];
    cross(w, v, t);
    cross(w, t, u);
#pragma unroll
    for (int e = 0; e < 3; e++) o[e] = (v[e] - a * t[e]) + b * u[e];
}

// Scalars of one sample that depend on the raw sample and the bias only -- NOT on the recurrence (CpiV1.h:97-142, 162-164, 196-238):
// rotation coefficients of the full and the half step, f1..f4, and (model 1) the d f/d|w| terms and the right-Jacobian coefficients.
// Profiling-only builds (never shipped; tools/phase_builds.sh): the two phases the north_star wants measured separately.
//   CPI_TRI_PHASE_LOAD  the TMA sample stream alone (stage, wait, read; no arithmetic)  -> achieved HBM GB/s of the sample-load phase
//   CPI_TRI_PHASE_COV   the covariance RK4 alone on constant inputs (no fetch, no front)   -> fp64 FLOP/s of the covariance phase
#if defined(CPI_TRI_PHASE_LOAD)
constexpr bool kLoadOnly = true, kCovOnly = false;
#elif defined(CPI_TRI_PHASE_COV)
constexpr bool kLoadOnly = false, kCovOnly = true;
#else
constexpr bool kLoadOnly = false, kCovOnly = false;
#endif

enum : int { SC_A1 = 0, SC_B1, SC_A2, SC_B2, SC_F1, SC_F2, SC_F3, SC_F4, SC_DT6, SC_D1, SC_D2, SC_D3, SC_D4, SC_CA, SC_CB, SC_N };

template <int MODEL, class T>
__global__ void __launch_bounds__((TriNT<MODEL, T>::NT), 1) k_preintegrate_tri(const PreintParams p) {
    using SM_ = TriSmem<MODEL, T>;
    constexpr int NT = SM_::NT;
    constexpr int CH = 8 / (int)sizeof(T) * 2;            // samples per TMA chunk: 2 (fp64) or 4 (fp32) = 112 B in one aligned 128-B fetch
    constexpr int EPC = 128 / (int)sizeof(T);             // elements per chunk buffer
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const bool lane_ok = lane < 3 * TRI_WPW;
    const int trio = lane_ok ? lane / 3 : 0;
    const int c = lane_ok ? lane - 3 * trio : 0;          // axis offset of this lane's frame
    const int i0 = c, i1 = (c + 1) % 3, i2 = (c + 2) % 3; // original index of frame axis 0, 1, 2
    const int nx = lane_ok ? 3 * trio + i1 : lane, pv = lane_ok ? 3 * trio + i2 : lane;
    const int wslot = wid * TRI_WPW + trio;
    const int64_t win = (int64_t)blockIdx.x * p.wpb + wslot;
    const bool active = lane_ok && wslot < p.wpb && win < p.n_windows;
    if (wid * TRI_WPW >= p.wpb || (int64_t)blockIdx.x * p.wpb + wid * TRI_WPW >= p.n_windows) return;   // whole warp idle (warp-uniform)

    T* sl = reinterpret_cast<T*>(smem_raw) + threadIdx.x;
    double* fs = reinterpret_cast<double*>(smem_raw + SM_::off_fs) + threadIdx.x;
    // per-window scalar sets of the current 3 samples (the two idle lanes of a warp get a dummy slot of their own)
    double* sc = reinterpret_cast<double*>(smem_raw + SM_::off_sc) + (size_t)(lane_ok ? wslot : SM_::WPB + wid) * TriSC<MODEL>::STRIDE;
    const T* buf = reinterpret_cast<const T*>(smem_raw + SM_::off_buf + (size_t)wslot * TRI_BUF_STRIDE);
    const uint32_t buf0 = smem_u32(buf);
    const uint32_t bar0 = smem_u32(smem_raw + SM_::off_bar + (size_t)wslot * (8 * TRI_NBUF));

    // ---- per-window constants (setLinearizationPoints, CpiBase.h:73-80), in the lane frame
    int64_t o0 = 0;
    int nsteps = 0;
#pragma unroll
    for (int e = 0; e < TriL<MODEL>::NFS; e++) FST(e) = 0.0;
    double bwo[3] = {0, 0, 0};                                       // gyro bias in the ORIGINAL axis order (|w_hat| is summed in that order)
    if (active) {
        const T* lin = reinterpret_cast<const T*>(p.lin) + win * CPI_LIN_DOUBLES;
        bwo[0] = (double)lin[0]; bwo[1] = (double)lin[1]; bwo[2] = (double)lin[2];
        FST(FS_BW) = (double)lin[i0]; FST(FS_BW + 1) = (double)lin[i1]; FST(FS_BW + 2) = (double)lin[i2];
        FST(FS_BA) = (double)lin[3 + i0]; FST(FS_BA + 1) = (double)lin[3 + i1]; FST(FS_BA + 2) = (double)lin[3 + i2];
        if (MODEL == 2) {                                            // g_k = quat_2_Rot(q_k_lin) * grav  (CpiV2.h:99, 202, 315), rotated into the lane frame
            const double q[4] = {(double)lin[6], (double)lin[7], (double)lin[8], (double)lin[9]}, g[3] = {(double)lin[10], (double)lin[11], (double)lin[12]};
            double RG[9], gk[3];
            quat_2_Rot(q, RG);
            mv33(RG, g, gk);
            FST(FS_GK) = c == 0 ? gk[0] : (c == 1 ? gk[1] : gk[2]);
            FST(FS_GK + 1) = c == 0 ? gk[1] : (c == 1 ? gk[2] : gk[0]);
            FST(FS_GK + 2) = c == 0 ? gk[2] : (c == 1 ? gk[0] : gk[1]);
        }
        int64_t ns64;
        if (p.offsets) { o0 = p.offsets[win]; ns64 = p.offsets[win + 1] - o0; }
        else { o0 = win * p.ns_uniform; ns64 = p.ns_uniform; }
        nsteps = ns64 < 0 ? 0 : (ns64 > 2147483000 ? 2147483000 : (int)ns64);
    }
    const T* sp = reinterpret_cast<const T*>(p.samples) + o0 * CPI_SAMPLE_DOUBLES;
    const int wmax = __reduce_max_sync(0xffffffffu, nsteps);

    // ---- TMA pipeline: lane 0 of the trio stages the window's stream through a ring of TRI_NBUF 128-byte chunk buffers.  Chunk k
    // (samples CH k .. CH k + CH - 1, fetched as ONE aligned 128-byte transaction that also absorbs the misalignment of the
    // window start) lives in buffer k % NBUF, completes phase k / NBUF of barrier k % NBUF.  The last samples of a window are
    // read with plain loads: an aligned 128-byte fetch there could run past the caller's buffer.
    const int shift = (int)(((uintptr_t)sp & 15) / sizeof(T));      // misalignment of the window start w.r.t. 16 bytes, in elements
    const int n_tma = nsteps > 0 ? (nsteps - 1) / CH : 0;           // chunks with at least one more sample after them
    const int n_tma_samples = n_tma * CH;
    int next_issue = 0;
    if (active && c == 0) {
#pragma unroll
        for (int k = 0; k < TRI_NBUF; k++) mbar_init(bar0 + 8 * k, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        fence_proxy_async();
#pragma unroll
        for (int k = 0; k < TRI_NBUF; k++)
            if (k < n_tma) {
                mbar_arrive_expect_tx(bar0 + 8 * k, 128);
                bulk_g2s(buf0 + 128 * k, sp + 7 * CH * k - shift, 128, bar0 + 8 * k);
            }
        next_issue = TRI_NBUF;
    }
    __syncwarp();                                                    // barrier init visible to the trio before anyone polls

    // pointer to sample `is` of this window: staged copy (after waiting for its chunk) or global memory (tail); null steps return nullptr
    auto sample_ptr = [&](int is, bool& from_smem) -> const T* {
        from_smem = is < n_tma_samples;
        if (from_smem) {
            const int k = is / CH, b = k % TRI_NBUF;
            mbar_wait(bar0 + 8 * b, (uint32_t)((k / TRI_NBUF) & 1));
            return buf + b * EPC + shift + 7 * (is % CH);
        }
        return sp + (int64_t)is * CPI_SAMPLE_DOUBLES;
    };

    // ---- state (CpiBase.h:99-124 initialisers), lane frame
    double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};                       // full old rotation, row-major
    double DT = 0.0, pgg = 0.0, paa = 0.0;
    TriP<T> P;
#pragma unroll
    for (int e = 0; e < 3; e++) P.TG[e] = P.TT[e] = P.GV[e] = P.TV[e] = P.AV[e] = P.VV[e] = P.TP[e] = P.GP[e] = P.AP[e] = P.VP[e] = P.PP[e] = 0.0;

    // ---- continuation: resume from the state a previous call left in a record (the batched form of calling feed_IMU again on an existing
    // CpiV1 / CpiV2 object, CpiBase.h:86 -- every field of the object is in the record; model 2's clone rows are re-initialised at every
    // step, CpiV2.h:436-443, so P_meas is all of the covariance state).  The mirror image of the record write at the end of the kernel.
    if (p.init != nullptr && active) {
        constexpr int RDI = (MODEL == 1) ? CPI_REC_V1_DOUBLES : CPI_REC_V2_DOUBLES;
        const T* rin = reinterpret_cast<const T*>(p.init) + win * (int64_t)RDI;
        const int ri[3] = {i0, i1, i2};
        DT = (double)rin[CPI_REC_DT];
        FST(FS_AL) = (double)rin[CPI_REC_ALPHA + c]; FST(FS_BE) = (double)rin[CPI_REC_BETA + c];
        const T* Pm = rin + CPI_REC_P;
        pgg = (double)Pm[3 + 15 * 3]; paa = (double)Pm[9 + 15 * 9];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const int r = ri[k];
#pragma unroll
            for (int j = 0; j < 3; j++) R[3 * k + j] = (double)rin[CPI_REC_R + r + 3 * ri[j]];     // lane frame: (row, col) = (ri[k], ri[j]) of the column-major record
            if (MODEL == 1) {
                FST(FS_JQ + k) = (double)rin[CPI_REC_JQ + r + 3 * c]; FST(FS_JA + k) = (double)rin[CPI_REC_JA + r + 3 * c]; FST(FS_JB + k) = (double)rin[CPI_REC_JB + r + 3 * c];
                FST(FS_HA + k) = (double)rin[CPI_REC_HA + r + 3 * c]; FST(FS_HB + k) = (double)rin[CPI_REC_HB + r + 3 * c];
            } else {
                FST(FS_DTG + k) = -(double)rin[CPI_REC_JQ + r + 3 * c]; FST(FS_DPG + k) = (double)rin[CPI_REC_JA + r + 3 * c]; FST(FS_DVG + k) = (double)rin[CPI_REC_JB + r + 3 * c];
                FST(FS_DPA + k) = (double)rin[CPI_REC_HA + r + 3 * c]; FST(FS_DVA + k) = (double)rin[CPI_REC_HB + r + 3 * c];
                FST(FS_DPL + k) = (double)rin[CPI_REC_OA + r + 3 * c]; FST(FS_DVL + k) = (double)rin[CPI_REC_OB + r + 3 * c];
            }
            auto blk = [&](int I, int J) { return (double)Pm[(3 * I + r) + 15 * (3 * J + c)]; };
            P.TT[k] = blk(0, 0); P.VV[k] = blk(2, 2);
            P.PP[k] = 0.5 * blk(4, 4);                           // PP is carried as Q with PP = Q + Q^T: the symmetric half is a valid Q
            P.TG[k] = blk(0, 1); P.GV[k] = blk(1, 2); P.TV[k] = blk(0, 2); P.AV[k] = blk(3, 2);
            P.TP[k] = blk(0, 4); P.GP[k] = blk(1, 4); P.AP[k] = blk(3, 4); P.VP[k] = blk(2, 4);
        }
    }

#pragma unroll 1
    for (int it0 = 0; it0 < wmax; it0 += 3) {
        // ================= pre-pass: lane c evaluates the recurrence-free scalars of sample it0 + c =================
        // (one sincos pair, one reciprocal and the closed-form coefficient functions per LANE instead of per lane and sample)
        {
            const int is = it0 + c;
            double w0 = 0.0, w1 = 0.0, w2 = 0.0, dt = 0.0;
            if (is < nsteps && !kCovOnly) {
                bool sm_;
                const T* src = sample_ptr(is, sm_);
                if (sm_) { w0 = (double)src[0]; w1 = (double)src[1]; w2 = (double)src[2]; dt = (double)src[6]; }
                else { w0 = (double)__ldg(src); w1 = (double)__ldg(src + 1); w2 = (double)__ldg(src + 2); dt = (double)__ldg(src + 6); }
            }
            w0 -= bwo[0]; w1 -= bwo[1]; w2 -= bwo[2];                // CpiV1.h:77-79
            const double mag = sqrt(w0 * w0 + w1 * w1 + w2 * w2);
            const double th = mag * dt;
            // dt == 0 is the reference's silent no-op (CpiV1.h:72-74).  With every scalar below equal to zero the step body is exactly
            // that (D = I, all increments 0), so null steps -- finished windows, idle lanes, dt = 0 samples -- need no branch around
            // the shuffles of the body, and they skip the divisions here (a zero operand would send the whole warp through the
            // slow path of the fp64 division routine).
            const bool null_step = dt == 0.0;
            const bool small_w = mag < 0.008726646;                  // CpiV1.h:101
            double v[SC_N];
#pragma unroll
            for (int e = 0; e < SC_N; e++) v[e] = 0.0;
            if (kLoadOnly || kCovOnly) v[SC_A1] = w0 + w1 + w2 + dt;
            else if (!null_step) {
                const double hd = 0.5 * dt, dt2 = dt * dt, dt3 = dt2 * dt;
                v[SC_DT6] = dt / 6.0;                                // CpiV1.h:352
                if (small_w) {                                       // Taylor forms: CpiV1.h:119-120, 132-136, 162-164, 196-216, 267-268
                    v[SC_A1] = dt; v[SC_B1] = dt2 * 0.5; v[SC_A2] = hd; v[SC_B2] = (hd * hd) * 0.5;
                    v[SC_F1] = -(dt3 / 3.0); v[SC_F2] = (dt2 * dt2) / 8.0; v[SC_F3] = -(dt2 / 2.0); v[SC_F4] = dt3 / 6.0;
                    if (MODEL == 1) {
                        v[SC_D1] = -(dt3 * dt2 / 15.0); v[SC_D2] = (dt3 * dt3) / 72.0; v[SC_D3] = -(dt2 * dt2 / 12.0); v[SC_D4] = (dt3 * dt2) / 60.0;
                        v[SC_CA] = 0.5 * dt; v[SC_CB] = (1.0 / 6.0) * dt * dt;
                    }
                } else {
                    double sn, cs_, sh, ch;
                    sincos(th, &sn, &cs_);
                    sincos(mag * 0.5 * dt, &sh, &ch);
                    const double im = 1.0 / mag;                     // one reciprocal instead of ~16 divisions
                    const double im2 = im * im, im3 = im2 * im, im4 = im2 * im2, th2 = th * th;
                    v[SC_A1] = sn * im; v[SC_B1] = (1.0 - cs_) * im2;                                   // CpiV1.h:119-120
                    v[SC_A2] = sh * im; v[SC_B2] = (1.0 - ch) * im2;                                    // CpiV1.h:267-268
                    v[SC_F1] = (th * cs_ - sn) * im3;                                                   // CpiV1.h:138-141
                    v[SC_F2] = (th2 - 2.0 * cs_ - 2.0 * th * sn + 2.0) * (0.5 * im4);
                    v[SC_F3] = -(1.0 - cs_) * im2;
                    v[SC_F4] = (th - sn) * im3;
                    if (MODEL == 1) {
                        v[SC_D1] = (th2 * sn - 3.0 * sn + 3.0 * th * cs_) * (im4 * im);                 // CpiV1.h:218-234
                        v[SC_D2] = (th2 - 4.0 * cs_ - 4.0 * th * sn + th2 * cs_ + 4.0) * (im4 * im2);
                        v[SC_D3] = (2.0 * (cs_ - 1.0) + th * sn) * im4;
                        v[SC_D4] = (2.0 * th + th * cs_ - 3.0 * sn) * (im4 * im);
                        const double ith = 1.0 / th;                 // right Jacobian of w dt (CpiV1.h:162-164): w_tx = dt W, w_tx^2 = dt^2 W2
                        v[SC_CA] = ((1.0 - cs_) * (ith * ith)) * dt; v[SC_CB] = ((th - sn) * (ith * ith * ith)) * dt * dt;
                    }
                }
            }
            constexpr int NSC = (MODEL == 1) ? (int)SC_N : (int)SC_D1;
#pragma unroll
            for (int e = 0; e < (NSC + 1) / 2; e++)           // 16-byte stores
                reinterpret_cast<double2*>(sc + c * TriSC<MODEL>::PER)[e] = make_double2(v[2 * e], 2 * e + 1 < SC_N ? v[2 * e + 1] : 0.0);
        }
        __syncwarp();

#pragma unroll 1
        for (int j = 0; j < 3; j++) {
            const int it = it0 + j;
            if (it >= wmax) break;                                   // warp-uniform
            // ---- fetch entry `it` in the lane frame; finished windows run a NULL step
            double wm[3] = {0, 0, 0}, am[3] = {0, 0, 0}, dt = 0.0;
            if (kCovOnly) { wm[0] = 0.1; wm[1] = -0.2; wm[2] = 0.3; am[0] = 0.1; am[1] = 0.2; am[2] = 9.8; dt = 0.005; }
            else if (it < nsteps) {
                bool sm_;
                const T* src = sample_ptr(it, sm_);
                if (sm_) {
                    wm[0] = (double)src[i0]; wm[1] = (double)src[i1]; wm[2] = (double)src[i2];
                    am[0] = (double)src[3 + i0]; am[1] = (double)src[3 + i1]; am[2] = (double)src[3 + i2];
                    dt = (double)src[6];
                } else {
                    wm[0] = (double)__ldg(src + i0); wm[1] = (double)__ldg(src + i1); wm[2] = (double)__ldg(src + i2);
                    am[0] = (double)__ldg(src + 3 + i0); am[1] = (double)__ldg(src + 3 + i1); am[2] = (double)__ldg(src + 3 + i2);
                    dt = (double)__ldg(src + 6);
                }
            }
            DT += dt;                                                // CpiV1.h:69 (before the dt == 0 return)
            if (kLoadOnly) { DT += wm[0] + wm[1] + wm[2] + am[0] + am[1] + am[2]; continue; }
            double scj[SC_N];                                        // this sample's scalar set, 16-byte loads (same address in the trio: broadcast)
            {
                constexpr int NLD = (MODEL == 1) ? (int)SC_N : (int)SC_D1;
                const double2* s2 = reinterpret_cast<const double2*>(sc + j * TriSC<MODEL>::PER);
#pragma unroll
                for (int e = 0; e < (NLD + 1) / 2; e++) { const double2 t2 = s2[e]; scj[2 * e] = t2.x; if (2 * e + 1 < SC_N) scj[2 * e + 1] = t2.y; }
            }
            const double a1 = scj[SC_A1], b1 = scj[SC_B1], a2 = scj[SC_A2], b2 = scj[SC_B2];
            const double f1 = scj[SC_F1], f2 = scj[SC_F2], f3 = scj[SC_F3], f4 = scj[SC_F4], dt6 = kCovOnly ? dt / 6.0 : scj[SC_DT6];

            // ---- estimated readings (CpiV1.h:77-86)
            const double wh[3] = {wm[0] - FST(FS_BW), wm[1] - FST(FS_BW + 1), wm[2] - FST(FS_BW + 2)};
            double ah[3] = {am[0] - FST(FS_BA), am[1] - FST(FS_BA + 1), am[2] - FST(FS_BA + 2)};
            double g_tau[3] = {0.0, 0.0, 0.0};
            if (MODEL == 2) {                                        // a_hat = a_m - b_a - R_k2tau R_G2k g  with the OLD rotation (CpiV2.h:99)
                const double gk[3] = {FST(FS_GK), FST(FS_GK + 1), FST(FS_GK + 2)};
                mv33(R, gk, g_tau);
                ah[0] -= g_tau[0]; ah[1] -= g_tau[1]; ah[2] -= g_tau[2];
            }

            // ---- relative rotation: own column of the new and the mid-point rotation (CpiV1.h:119-124, 267-269), then the full matrices
            double R1[9], Rm[9];
            if (kCovOnly) {
#pragma unroll
                for (int e = 0; e < 9; e++) { R1[e] = R[e]; Rm[e] = R[e]; }
            } else {
                const double rc[3] = {R[0], R[3], R[6]};
                double r1c[3], rmc[3], X1[3], X2[3];
                rot_col2(a1, b1, a2, b2, wh, rc, r1c, rmc);
                gather_cols(r1c, nx, pv, X1, X2);
#pragma unroll
                for (int e = 0; e < 3; e++) { R1[3 * e] = r1c[e]; R1[3 * e + 1] = X1[e]; R1[3 * e + 2] = X2[e]; }
                gather_cols(rmc, nx, pv, X1, X2);
#pragma unroll
                for (int e = 0; e < 3; e++) { Rm[3 * e] = rmc[e]; Rm[3 * e + 1] = X1[e]; Rm[3 * e + 2] = X2[e]; }
            }

            if (!kCovOnly) {
            // ---- means (CpiV1.h:145-154):  alpha += beta dt + R1^T alpha_arg a ;  beta += R1^T beta_arg a   (old beta); this lane owns element c
            const double hdt2 = (dt * dt) * 0.5;
            double Wa[3], W2a[3], ua[3], ub[3];
            cross(wh, ah, Wa);                                       // W a
            cross(wh, Wa, W2a);                                      // W^2 a
#pragma unroll
            for (int e = 0; e < 3; e++) {
                ua[e] = hdt2 * ah[e] + f1 * Wa[e] + f2 * W2a[e];     // alpha_arg * a_hat   (CpiV1.h:145)
                ub[e] = dt * ah[e] + f3 * Wa[e] + f4 * W2a[e];       // beta_arg * a_hat    (CpiV1.h:146)
            }
            {
                const double be = FST(FS_BE);
                FST(FS_AL) = FST(FS_AL) + be * dt + (R1[0] * ua[0] + R1[3] * ua[1] + R1[6] * ua[2]);
                FST(FS_BE) = be + (R1[0] * ub[0] + R1[3] * ub[1] + R1[6] * ub[2]);
            }

            if (MODEL == 1) {
                // ---- analytic bias Jacobians, own column (CpiV1.h:162-259)
                const double d1 = scj[SC_D1], d2 = scj[SC_D2], d3 = scj[SC_D3], d4 = scj[SC_D4], ca = scj[SC_CA], cb = scj[SC_CB];
                // [w x] and [w x]^2, column 0:  W[:,0] = (0, w2, -w1),  W2[:,0] = (-(w1^2 + w2^2), w0 w1, w0 w2)
                const double Wc[3] = {0.0, wh[2], -wh[1]};
                const double W2c[3] = {-(wh[1] * wh[1] + wh[2] * wh[2]), wh[0] * wh[1], wh[0] * wh[2]};
                double aargc[3], bargc[3], Hal[3], Hbe[3], Jq[3], Ja[3], Jb[3], Ha[3], Hb[3];
#pragma unroll
                for (int e = 0; e < 3; e++) { Jq[e] = FST(FS_JQ + e); Ja[e] = FST(FS_JA + e); Jb[e] = FST(FS_JB + e); Ha[e] = FST(FS_HA + e); Hb[e] = FST(FS_HB + e); }
#pragma unroll
                for (int e = 0; e < 3; e++) {
                    aargc[e] = ((e == 0) ? hdt2 : 0.0) + f1 * Wc[e] + f2 * W2c[e];
                    bargc[e] = ((e == 0) ? dt : 0.0) + f3 * Wc[e] + f4 * W2c[e];
                }
                mvT33(R1, aargc, Hal);                               // column of R_tau12k * alpha_arg
                mvT33(R1, bargc, Hbe);
                {
                    double t3[3];
                    rot_col(a1, b1, wh, Jq, t3);                     // R_tau2tau1 * J_q
#pragma unroll
                    for (int e = 0; e < 3; e++) { Jq[e] = t3[e] + (((e == 0) ? 1.0 : 0.0) - ca * Wc[e] + cb * W2c[e]) * dt; FST(FS_JQ + e) = Jq[e]; }   // CpiV1.h:167
                }
#pragma unroll
                for (int e = 0; e < 3; e++) {                        // CpiV1.h:170-172 (old H_b)
                    FST(FS_HA + e) = (Ha[e] - Hal[e]) + dt * Hb[e];
                    FST(FS_HB + e) = Hb[e] - Hbe[e];
                }
                {
                    // column 0 of the frame: e_0 x a = (0, -a2, a1)
                    const double exa[3] = {0.0, -ah[2], ah[1]}, exWa[3] = {0.0, -Wa[2], Wa[1]};
                    double Wexa[3], c1v[3], c2v[3], va_[3], vb_[3], oa3[3], ob3[3];
                    cross(wh, exa, Wexa);
                    cross(Jq, ua, c1v);                              // [J_q e_i x] (alpha_arg a), NEW J_q
                    cross(Jq, ub, c2v);
                    const double wi = wh[0];
#pragma unroll
                    for (int e = 0; e < 3; e++) {
                        va_[e] = -c1v[e] + (wi * d1) * Wa[e] - f1 * exa[e] + (wi * d2) * W2a[e] - f2 * (exWa[e] + Wexa[e]);
                        vb_[e] = -c2v[e] + (wi * d3) * Wa[e] - f3 * exa[e] + (wi * d4) * W2a[e] - f4 * (exWa[e] + Wexa[e]);
                    }
                    mvT33(R1, va_, oa3);
                    mvT33(R1, vb_, ob3);
#pragma unroll
                    for (int r = 0; r < 3; r++) {                    // J_a += J_b dt (old J_b, CpiV1.h:241) then the column terms
                        FST(FS_JA + r) = (Ja[r] + Jb[r] * dt) + oa3[r];
                        FST(FS_JB + r) = Jb[r] + ob3[r];
                    }
                }
            }
            if (MODEL == 2) {
                // ---- Discrete_J_b <- B_k Phi Discrete_J_b on the consumed columns (CpiV2.h:347-426, 443).  Phi is RK4 on Phi' = F Phi, a
                // LINEAR map, so it is applied directly to this lane's own columns (bg_c, ba_c, l_c) of Discrete_J_b: same four stages,
                // no Phi ever formed, nothing crosses lanes.  Rows: theta' = -W theta - e_c (bg column only); v' = A_s theta + C_s theta(start)
                // (the clone rows equal the theta rows at the start of every step, B_k) + B_s e_c (ba column) + L_s e_c (l column); p' = v.
                const double hdt = 0.5 * dt;
                double xt[3], xv[3], st[3], sv[3], sp_[3], gxt0[3];
                const double Dtg[3] = {FST(FS_DTG), FST(FS_DTG + 1), FST(FS_DTG + 2)}, Dvg[3] = {FST(FS_DVG), FST(FS_DVG + 1), FST(FS_DVG + 2)};
                cross(g_tau, Dtg, gxt0);                             // g_tau x theta(start): the C_s term is -R_s^T of this
#pragma unroll
                for (int e = 0; e < 3; e++) { xt[e] = Dtg[e]; xv[e] = Dvg[e]; }
#pragma unroll
                for (int s = 0; s < 4; s++) {
                    const double* Rs = (s == 0) ? R : (s == 3 ? R1 : Rm);
                    const double cn = (s < 2) ? hdt : dt;
                    double kt[3], u[3], kv[3];
                    cross(xt, wh, kt);
                    kt[0] -= 1.0;
                    cross(ah, xt, u);
#pragma unroll
                    for (int e = 0; e < 3; e++) u[e] += gxt0[e];
                    negRt(Rs, u, kv);
#pragma unroll
                    for (int e = 0; e < 3; e++) {
                        st[e] = (s == 0) ? kt[e] : (s == 3 ? st[e] + kt[e] : st[e] + 2.0 * kt[e]);
                        sv[e] = (s == 0) ? kv[e] : (s == 3 ? sv[e] + kv[e] : sv[e] + 2.0 * kv[e]);
                        sp_[e] = (s == 0) ? xv[e] : (s == 3 ? sp_[e] + xv[e] : sp_[e] + 2.0 * xv[e]);
                        if (s < 3) { xt[e] = Dtg[e] + cn * kt[e]; xv[e] = Dvg[e] + cn * kv[e]; }
                    }
                }
#pragma unroll
                for (int e = 0; e < 3; e++) {
                    FST(FS_DTG + e) = Dtg[e] + dt6 * st[e];
                    FST(FS_DVG + e) = Dvg[e] + dt6 * sv[e];
                    FST(FS_DPG + e) = FST(FS_DPG + e) + dt6 * sp_[e];
                }
                // ba and l columns: v' = B_s e_c = -(row 0 of R_s),  v' = L_s e_c = -R_s^T (R_old [g_k x] e_c)  (CpiV2.h:336); p' = v
                const double gk[3] = {FST(FS_GK), FST(FS_GK + 1), FST(FS_GK + 2)};
                const double sk0[3] = {0.0, gk[2], -gk[1]};          // [g_k x] e_0
                double y[3], l0[3], lm[3], l1[3];
                mv33(R, sk0, y);
                negRt(R, y, l0); negRt(Rm, y, lm); negRt(R1, y, l1);
                const double Ppv = dt6 * (1.0 + 2.0 + 2.0 + 1.0);
#pragma unroll
                for (int e = 0; e < 3; e++) {
                    const double b0 = -R[e], bm = -Rm[e], b1_ = -R1[e];
                    const double dva = FST(FS_DVA + e), dvl = FST(FS_DVL + e);
                    FST(FS_DPA + e) = dt6 * (2.0 * (b0 * hdt) + 2.0 * (bm * hdt) + bm * dt) + Ppv * dva + FST(FS_DPA + e);
                    FST(FS_DVA + e) = dt6 * (b0 + 2.0 * bm + 2.0 * bm + b1_) + dva;
                    FST(FS_DPL + e) = dt6 * (2.0 * (l0[e] * hdt) + 2.0 * (lm[e] * hdt) + lm[e] * dt) + Ppv * dvl + FST(FS_DPL + e);
                    FST(FS_DVL + e) = dt6 * (l0[e] + 2.0 * lm[e] + 2.0 * lm[e] + l1[e]) + dvl;
                }
            }
            }
            CPI_FENCE();

            // ---- covariance RK4 (CpiV1.h:272-353)
            {
                T w_[3], a_[3], g_[3], R_[9], Rm_[9], R1_[9];
#pragma unroll
                for (int e = 0; e < 3; e++) { w_[e] = (T)wh[e]; a_[e] = (T)ah[e]; g_[e] = (T)g_tau[e]; }
#pragma unroll
                for (int e = 0; e < 9; e++) { R_[e] = (T)R[e]; Rm_[e] = (T)Rm[e]; R1_[e] = (T)R1[e]; }
                tri_cov_step<MODEL, NT, T>(P, sl, w_, a_, g_, R_, Rm_, R1_, (T)pgg, (T)paa, (T)dt, (T)dt6, (T)p.q_w, (T)p.q_wb, (T)p.q_a, (T)p.q_ab, nx, pv);
                pgg += dt6 * (p.q_wb + 2.0 * p.q_wb + 2.0 * p.q_wb + p.q_wb);
                paa += dt6 * (p.q_ab + 2.0 * p.q_ab + 2.0 * p.q_ab + p.q_ab);
            }
#pragma unroll
            for (int e = 0; e < 9; e++) R[e] = R1[e];                // CpiV1.h:357
        }
        __syncwarp();                                                // all lanes are done with this group's scalar sets and staged samples
        // ---- refill: every chunk whose samples all lie before it0 + 3 has been consumed by the three lanes
        if (c == 0 && next_issue < n_tma) {
            const int consumed = (it0 + 3) / CH;
            while (next_issue < n_tma && next_issue - TRI_NBUF < consumed) {
                const int b = next_issue % TRI_NBUF;
                fence_proxy_async();
                mbar_arrive_expect_tx(bar0 + 8 * b, 128);
                bulk_g2s(buf0 + 128 * b, sp + 7 * CH * next_issue - shift, 128, bar0 + 8 * b);
                next_issue++;
            }
        }
    }

    // ---- write the record (column-major 3x3 / 15x15, include/cpi_b200.h).  Lane c writes original column c (rows c, c+1, c+2).
    // symmetric diagonal blocks: average the two independently rounded copies of each off-diagonal entry (the reference
    // symmetrises every step, CpiV1.h:353)
    double sTT[3], sVV[3], sPP[3];
    sTT[0] = P.TT[0]; sTT[1] = 0.5 * (P.TT[1] + shf(P.TT[2], nx)); sTT[2] = 0.5 * (P.TT[2] + shf(P.TT[1], pv));
    sVV[0] = P.VV[0]; sVV[1] = 0.5 * (P.VV[1] + shf(P.VV[2], nx)); sVV[2] = 0.5 * (P.VV[2] + shf(P.VV[1], pv));
    sPP[0] = P.PP[0] + P.PP[0]; sPP[1] = P.PP[1] + shf(P.PP[2], nx); sPP[2] = P.PP[2] + shf(P.PP[1], pv);     // PP = Q + Q^T (exactly symmetric: a + b == b + a)
    if (!active) return;
    constexpr int RD = (MODEL == 1) ? CPI_REC_V1_DOUBLES : CPI_REC_V2_DOUBLES;
    T* rec = reinterpret_cast<T*>(p.out) + win * (int64_t)RD;
    const int ri[3] = {i0, i1, i2};
    if (c == 0) {                                                    // lane 0's frame is the original frame
        double q[4];
        rot_2_quat(R, q);                                            // CpiV1.h:358 (only the last one is ever consumed)
        rec[CPI_REC_Q] = (T)q[0]; rec[CPI_REC_Q + 1] = (T)q[1]; rec[CPI_REC_Q + 2] = (T)q[2]; rec[CPI_REC_Q + 3] = (T)q[3];
        rec[CPI_REC_DT] = (T)DT;
    }
    rec[CPI_REC_ALPHA + c] = (T)FST(FS_AL); rec[CPI_REC_BETA + c] = (T)FST(FS_BE);
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const int r = ri[k];
        rec[CPI_REC_R + r + 3 * c] = (T)R[3 * k];
        if (MODEL == 1) {
            rec[CPI_REC_JQ + r + 3 * c] = (T)FST(FS_JQ + k); rec[CPI_REC_JA + r + 3 * c] = (T)FST(FS_JA + k); rec[CPI_REC_JB + r + 3 * c] = (T)FST(FS_JB + k);
            rec[CPI_REC_HA + r + 3 * c] = (T)FST(FS_HA + k); rec[CPI_REC_HB + r + 3 * c] = (T)FST(FS_HB + k);
        } else {   // read-out of Discrete_J_b (CpiV2.h:450-458): J_q = -D[theta,bg], J_a = D[p,bg], J_b = D[v,bg], H_a = D[p,ba], H_b = D[v,ba], O_a = D[p,l], O_b = D[v,l]
            rec[CPI_REC_JQ + r + 3 * c] = (T)(-FST(FS_DTG + k)); rec[CPI_REC_JA + r + 3 * c] = (T)FST(FS_DPG + k); rec[CPI_REC_JB + r + 3 * c] = (T)FST(FS_DVG + k);
            rec[CPI_REC_HA + r + 3 * c] = (T)FST(FS_DPA + k); rec[CPI_REC_HB + r + 3 * c] = (T)FST(FS_DVA + k);
            rec[CPI_REC_OA + r + 3 * c] = (T)FST(FS_DPL + k); rec[CPI_REC_OB + r + 3 * c] = (T)FST(FS_DVL + k);
        }
    }
    // P_meas, full 15x15: block (I,J), I,J in {theta=0, bg=1, v=2, ba=3, p=4}; every off-diagonal block is written twice
    T* Pm = rec + CPI_REC_P;
    auto put2 = [&](int I, int J, int r, T v) { Pm[(3 * I + r) + 15 * (3 * J + c)] = v; Pm[(3 * J + c) + 15 * (3 * I + r)] = v; };
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const int r = ri[k];
        put2(0, 0, r, (T)sTT[k]); put2(2, 2, r, (T)sVV[k]); put2(4, 4, r, (T)sPP[k]);
        put2(0, 1, r, (T)P.TG[k]); put2(1, 2, r, (T)P.GV[k]); put2(0, 2, r, (T)P.TV[k]); put2(3, 2, r, (T)P.AV[k]);
        put2(0, 4, r, (T)P.TP[k]); put2(1, 4, r, (T)P.GP[k]); put2(3, 4, r, (T)P.AP[k]); put2(2, 4, r, (T)P.VP[k]);
        put2(1, 1, r, r == c ? (T)pgg : T(0)); put2(3, 3, r, r == c ? (T)paa : T(0));
        put2(0, 3, r, T(0)); put2(1, 3, r, T(0));                    // P_theta,ba = P_bg,ba = 0 identically
    }
}

#undef SLT
#undef FST
#undef CN
#undef KSUM

template <int MODEL, class T>
static cudaError_t launch_tri_one(const PreintParams& p0, int num_sms, cudaStream_t st) {
    PreintParams p = p0;
    auto kern = k_preintegrate_tri<MODEL, T>;
    constexpr int smem = (int)TriSmem<MODEL, T>::bytes;
    static bool configured[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 64 || !configured[dev]) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return e;
        if (dev < 64) configured[dev] = true;
    }
    (void)num_sms;
    constexpr int WPB = TriSmem<MODEL, T>::WPB;      // ten windows per one-warp CTA; the block scheduler spreads the CTAs over the SMs
    p.wpb = WPB;
    const int grid = (int)((p.n_windows + p.wpb - 1) / p.wpb);
    kern<<<grid, TriSmem<MODEL, T>::NT, smem, st>>>(p);
    return cudaGetLastError();
}

int preint_tri_cap(int model, int dtype) {
    if (model == 1) return dtype == 32 ? TriSmem<1, float>::WPB : TriSmem<1, double>::WPB;
    return dtype == 32 ? TriSmem<2, float>::WPB : TriSmem<2, double>::WPB;
}
bool preint_tri_supported(int model, int flags) {
    if (flags & CPI_FLAG_IMU_AVG) return false;
    return model == 1 || (model == 2 && !(flags & CPI_FLAG_ANALYTIC_JACOBIANS));
}

cudaError_t preint_launch_tri(int model, int dtype, const PreintParams& p, int num_sms, cudaStream_t st) {
    if (model == 1) return dtype == 32 ? launch_tri_one<1, float>(p, num_sms, st) : launch_tri_one<1, double>(p, num_sms, st);
    if (model == 2) return dtype == 32 ? launch_tri_one<2, float>(p, num_sms, st) : launch_tri_one<2, double>(p, num_sms, st);
    return cudaErrorInvalidValue;
}

}  // namespace cpi
