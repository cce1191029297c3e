// K1 / K2: batched closed-form IMU preintegration, CpiV1::feed_IMU (cpi/CpiV1.h:62-361) and CpiV2::feed_IMU
// (cpi/CpiV2.h:84-467) of rpng/cpi, for H100 (sm_90a).  See DESIGN.md for the derivation.
//
// Mapping: ONE LANE PER WINDOW, a warp advances 32 independent windows in lock-step.  A single warp per SMSP keeps the
// DFMA pipe busy at ILP >= 4, whereas every cross-lane double costs as much as 4 DFMA (SHFL / LDS bandwidth is 16
// doubles/clk/SM vs 64 DFMA/clk/SM; tools/microbench.cu measures both).  So the window recurrence is kept free of cross-lane traffic; the per-window state that does not fit
// the register file -- the 90 unique non-trivial entries of the 15x15 covariance (ping-pong copy), the RK4 stage values
// other blocks depend on and the Jacobian state -- lives in shared memory in [entry][window] order (conflict-free:
// lane == window; base + immediate addressing because the window stride is a compile-time constant).
//
// One kernel, k_preintegrate: one warp does everything for its 32 windows.  It serves the modes the tri-lane kernels
// (preintegrate_tri.cu) do not: imu_avg, and model 2 with analytic Jacobians.
//
// Arithmetic: the reference integrates  Pdot = F P + P F^T + G Qc G^T  with RK4, F evaluated at R_old / R_mid / R_mid /
// R_new.  The same four stages are replicated here, but on the 3x3 block structure of F (five non-zero blocks), with P
// symmetric (15 unique blocks, two of them identically zero, two of them scalar multiples of I):
//     rows theta:  (FP)_tJ = -W P_tJ - P_gJ          W = [w_hat x]
//     rows v:      (FP)_vJ =  A P_tJ + B P_aJ (+ C P_cJ, model 2)     A = -R*^T [a_hat x],  B = -R*^T,  C = -R*^T [g_tau x]
//     rows p:      (FP)_pJ =  P_vJ
// Model 2's 21x21 system reduces to the same 15x15 tile plus three transient 3x3 blocks (clone rows c) per step: the
// theta_klin rows/cols of P_big are identically zero and the clone rows are re-initialised from the theta rows every
// step (B_k, CpiV2.h:436-443).  Its Jacobians are read out of the compounded transition Discrete_J_b; only 7 of its
// 3x3 blocks are ever non-trivial in the 9 consumed columns, and Phi's RK4 has closed block forms (the "Discrete_J_b" sections of k_preintegrate).
#include "cpi_common.cuh"
#include "cpi_kernels.h"
#include "tma.cuh"

namespace cpi {

// ---- shared-memory tile layout (units: doubles per window; element e of window w lives at tile[e * S + w]) ----------
enum : int {
    TT = 0,   // P_theta,theta  sym 6
    TG = 6,   // P_theta,bg     9   (i = theta row, j = bg col)
    VT = 15,  // P_v,theta      9
    VG = 24,  // P_v,bg         9
    VV = 33,  // P_v,v          sym 6
    VA = 39,  // P_v,ba         9
    PT = 48,  // P_p,theta      9
    PG = 57,  // P_p,bg         9
    PV = 66,  // P_p,v          9
    PA = 75,  // P_p,ba         9
    PP = 84,  // P_p,p          sym 6
    NP = 90,  // P_bg,bg = pgg*I and P_ba,ba = paa*I are scalars in registers; P_theta,ba = P_bg,ba = 0 identically
    // model 2, default mode: the non-trivial blocks of Discrete_J_b in the consumed columns (bg, ba, theta_klin)
    D_TG = 0, D_VG = 9, D_PG = 18, D_VA = 27, D_PA = 36, D_VL = 45, D_PL = 54, ND = 63,
    // analytic Jacobian state (model 1; model 2 with CPI_FLAG_ANALYTIC_JACOBIANS): same 63-double region
    J_Q = 0, J_A = 9, J_B = 18, H_A = 27, H_B = 36, O_A = 45, O_B = 54
};

// Per-model tile description.  S (window stride == max windows per CTA) is a compile-time constant so that every
// shared-memory access is [base + immediate]; it is chosen as large as 227 KB allow.
//   [0, 90)    covariance tile, buffer a   } ping-pong: a sample reads the old tile and writes the new one, because a
//   [90, 180)  covariance tile, buffer b   } block's old value is still the stage-1 input of blocks processed after it
//   [180, ..)  RK4 stage-value slots (stage values 2..4 of the blocks that later blocks depend on; slots are re-used as
//              soon as the last dependant has run -- see rk4_cascade)
//   then       Jacobian state (45 / 63 doubles)
enum : int { SLOT_A = 0, SLOT_B = 27, SLOT_C = 54, SLOT_D = 81 /*18*/, SLOT_E = 99 /*model 2*/ };
template <int MODEL, class T> struct Tile;
template <> struct Tile<1, double> { static constexpr int NSLOT = 99, NJ = 45, S = 80; };
template <> struct Tile<2, double> { static constexpr int NSLOT = 126, NJ = ND, S = 72; };
// fp32 storage (dtype 32): the covariance tile and its stage slots are float, the Jacobian state stays double
template <> struct Tile<1, float> { static constexpr int NSLOT = 99, NJ = 45, S = 128; };
template <> struct Tile<2, float> { static constexpr int NSLOT = 126, NJ = ND, S = 112; };
// byte layout of the dynamic shared memory:  [J: NJ doubles x S] [P a | P b | slots : T x S each element] [2 x 128 B staging per window] [2 mbarriers per window]
template <int MODEL, class T> __host__ __device__ constexpr size_t tile_off_T() { return (size_t)Tile<MODEL, T>::NJ * Tile<MODEL, T>::S * 8; }
template <int MODEL, class T> __host__ __device__ constexpr size_t tile_off_buf() {
    return tile_off_T<MODEL, T>() + (size_t)(2 * NP + Tile<MODEL, T>::NSLOT) * Tile<MODEL, T>::S * sizeof(T);
}
template <int MODEL, class T> __host__ __device__ constexpr size_t tile_off_bar() { return tile_off_buf<MODEL, T>() + (size_t)Tile<MODEL, T>::S * 256; }
template <int MODEL, class T> __host__ __device__ constexpr size_t tile_bytes() { return tile_off_bar<MODEL, T>() + (size_t)Tile<MODEL, T>::S * 16; }
static_assert(tile_bytes<1, double>() <= 232448 && tile_bytes<2, double>() <= 232448 && tile_bytes<1, float>() <= 232448 &&
              tile_bytes<2, float>() <= 232448, "tile exceeds 227 KB");
static_assert(tile_off_T<1, float>() % 16 == 0 && tile_off_T<2, float>() % 16 == 0 && tile_off_buf<1, float>() % 16 == 0 &&
              tile_off_buf<2, float>() % 16 == 0 && tile_off_buf<1, double>() % 16 == 0 && tile_off_buf<2, double>() % 16 == 0,
              "cp.async.bulk destinations must be 16-byte aligned");

// ---- block loaders ----------------------------------------------------------------------------------------------------
#define SM(buf, idx) (buf)[(idx) * S]

template <int S, class TP, class TX> CPI_DEV void ld9(const TP* b, int off, TX* x) {
#pragma unroll
    for (int k = 0; k < 9; k++) x[k] = SM(b, off + k);
}
template <int S, class TP, class TX> CPI_DEV void ldsym(const TP* b, int off, TX* x) {   // packed sym -> full row-major 3x3
    const TX a0 = SM(b, off), a1 = SM(b, off + 1), a2 = SM(b, off + 2), a3 = SM(b, off + 3), a4 = SM(b, off + 4), a5 = SM(b, off + 5);
    x[0] = a0; x[1] = a1; x[2] = a2; x[3] = a1; x[4] = a3; x[5] = a4; x[6] = a2; x[7] = a4; x[8] = a5;
}

// =====================================================================================================================
// Covariance: the reference's RK4 on  Pdot = F P + P F^T + G Qc G^T  (CpiV1.h:272-353; CpiV2.h:326-422), block-serial.
//
// F is block lower-triangular in the order (bg, ba | theta | v | p): theta-row blocks depend only on bg/theta blocks,
// v-row blocks on theta/ba/v blocks, p-row blocks on v/p blocks.  RK4 on a triangular system can therefore be run ONE
// 3x3 BLOCK AT A TIME -- all four stages of a block in registers, given the four stage values of the blocks it depends
// on -- with exactly the arithmetic of the stage-by-stage form.  Compared with sweeping the whole tile once per stage
// this removes the accumulator array and about half of the shared-memory traffic.  Order and slot reuse (model 1):
//     tg->A  tt->B  vg->C(+pg)  vt->A  pt->B  va->C(+pa)  vv->D  pv->A  pp
// model 2 adds the transient clone-row blocks ct (->A, before vt which then goes to E) and cv (->B, after vt); the p-row
// transient cp is recomputed from cv's stage values, like pg from vg and pa from va.
// Stage s (0..3) of a block lives in the OLD tile (s == 0) or in its slot at (s-1)*n.
#define CPI_SECTION() asm volatile("" ::: "memory")
#define CN(s) ((s) < 2 ? hdt : dt)                       /* x_{s+2} = x_1 + CN(s) k_{s+1}:  dt/2, dt/2, dt   (CpiV1.h:312, 323, 344) */
#define RS(s) ((s) == 0 ? R : ((s) == 3 ? R1 : Rm))       /* F evaluated at R_old, R_mid, R_mid, R_new */
#define KSUM(ks, k, s) ((s) == 0 ? (k) : ((s) == 3 ? (ks) + (k) : fma(T(2), (k), (ks))))   /* ((k1 + 2 k2) + 2 k3) + k4  (CpiV1.h:352) */

template <int S, class TP, class TX> CPI_DEV void st9(TP* b, int off, const TX* x) {
#pragma unroll
    for (int e = 0; e < 9; e++) SM(b, off + e) = x[e];
}
template <int S, class T> CPI_DEV void ldst9(const T* Po, int off, const T* sl, int slot, int s, T* x) {
    if (s == 0) ld9<S>(Po, off, x); else ld9<S>(sl, slot + (s - 1) * 9, x);
}
template <int S, class T> CPI_DEV void ldstsym(const T* Po, int off, const T* sl, int slot, int s, T* x) {
    if (s == 0) ldsym<S>(Po, off, x); else ldsym<S>(sl, slot + (s - 1) * 6, x);
}
template <class T> CPI_DEV void sym_expand(const T* a, T* x) { x[0] = a[0]; x[1] = a[1]; x[2] = a[2]; x[3] = a[1]; x[4] = a[3]; x[5] = a[4]; x[6] = a[2]; x[7] = a[4]; x[8] = a[5]; }

// rows of  -R^T [a x] : row i = a cross r_i  with r_i = column i of R (R row-major)
template <class T> CPI_DEV void make_A(const T* R, const T* a, T* A) {
#pragma unroll
    for (int i = 0; i < 3; i++) {
        const T r[3] = {R[i], R[3 + i], R[6 + i]};
        cross(a, r, &A[3 * i]);
    }
}
template <class T> CPI_DEV void make_B(const T* R, T* B) {   // -R^T
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) B[3 * i + j] = -R[3 * j + i];
}


template <int MODEL, int S, class T>
CPI_DEV void rk4_cascade(const T* Po, T* Pn, T* sl, const double* w_, const double* ah_, const double* gt_,
                         const double* R_, const double* Rm_, const double* R1_, double pgg_, double paa_, double dt_,
                         double q_w_, double q_wb_, double q_a_, double q_ab_) {
    // operands in the tile's arithmetic type (no-op copies for T = double)
    T w[3], ah[3], gt[3], R[9], Rm[9], R1[9];
#pragma unroll
    for (int e = 0; e < 3; e++) { w[e] = (T)w_[e]; ah[e] = (T)ah_[e]; gt[e] = (T)gt_[e]; }
#pragma unroll
    for (int e = 0; e < 9; e++) { R[e] = (T)R_[e]; Rm[e] = (T)Rm_[e]; R1[e] = (T)R1_[e]; }
    const T pgg = (T)pgg_, paa = (T)paa_, dt = (T)dt_, q_w = (T)q_w_, q_wb = (T)q_wb_, q_a = (T)q_a_, q_ab = (T)q_ab_;
    const T hdt = dt * T(0.5), dt6 = (T)(dt_ / 6.0);
    constexpr int SL_TG = SLOT_A, SL_TT = SLOT_B, SL_VG = SLOT_C, SL_CT = SLOT_A, SL_CV = SLOT_B, SL_VA = SLOT_C, SL_VV = SLOT_D;
    constexpr int SL_VT = (MODEL == 1) ? SLOT_A : SLOT_E, SL_PT = (MODEL == 1) ? SLOT_B : SLOT_A, SL_PV = (MODEL == 1) ? SLOT_A : SLOT_E;

    {   // ---- tg:  k = -W x - pgg_s I        (-W c = c cross w, column-wise)
        T x1[9], x[9], ks[9], k[9];
        ld9<S>(Po, TG, x1);
#pragma unroll
        for (int e = 0; e < 9; e++) x[e] = x1[e];
#pragma unroll
        for (int s = 0; s < 4; s++) {
            const T pg_s = (s == 0) ? pgg : fma(q_wb, (s == 3 ? dt : hdt), pgg);
#pragma unroll
            for (int j = 0; j < 3; j++) {
                const T col[3] = {x[j], x[3 + j], x[6 + j]};
                T c3[3];
                cross(col, w, c3);
#pragma unroll
                for (int i = 0; i < 3; i++) k[3 * i + j] = c3[i] - (i == j ? pg_s : T(0));
            }
#pragma unroll
            for (int e = 0; e < 9; e++) ks[e] = KSUM(ks[e], k[e], s);
            if (s < 3) {
#pragma unroll
                for (int e = 0; e < 9; e++) x[e] = fma(k[e], CN(s), x1[e]);
                st9<S>(sl, SL_TG + s * 9, x);
            }
        }
#pragma unroll
        for (int e = 0; e < 9; e++) SM(Pn, TG + e) = fma(dt6, ks[e], x1[e]);
    }
    CPI_SECTION();
    {   // ---- tt:  k = M + M^T + q_w I,  M = -W x - P_tg^T
        T a1[6], a[6], ks[6], x[9], M[9], tg[9];
#pragma unroll
        for (int e = 0; e < 6; e++) a[e] = a1[e] = SM(Po, TT + e);
#pragma unroll
        for (int s = 0; s < 4; s++) {
            sym_expand(a, x);
            ldst9<S>(Po, TG, sl, SL_TG, s, tg);
#pragma unroll
            for (int j = 0; j < 3; j++) {
                const T col[3] = {x[j], x[3 + j], x[6 + j]};
                T c3[3];
                cross(col, w, c3);
#pragma unroll
                for (int i = 0; i < 3; i++) M[3 * i + j] = c3[i] - tg[3 * j + i];
            }
#pragma unroll
            for (int i = 0; i < 3; i++)
#pragma unroll
                for (int j = i; j < 3; j++) {
                    const T kk = M[3 * i + j] + M[3 * j + i] + (i == j ? q_w : T(0));
                    ks[sym3(i, j)] = KSUM(ks[sym3(i, j)], kk, s);
                    if (s < 3) { a[sym3(i, j)] = fma(kk, CN(s), a1[sym3(i, j)]); SM(sl, SL_TT + s * 6 + sym3(i, j)) = a[sym3(i, j)]; }
                }
        }
#pragma unroll
        for (int e = 0; e < 6; e++) SM(Pn, TT + e) = fma(dt6, ks[e], a1[e]);
    }
    CPI_SECTION();
    {   // ---- vg:  k = A_s P_tg,s (+ C_s P_cg, P_cg = P_tg at step start)    and pg:  k = P_vg,s  (pure integral of vg's stage values)
        T x1[9], x[9], ks[9], k[9], pg1[9], pgs[9], tg[9], A[9], C[9], cg[9];
        ld9<S>(Po, VG, x1); ld9<S>(Po, PG, pg1);
        if (MODEL == 2) ld9<S>(Po, TG, cg);
#pragma unroll
        for (int e = 0; e < 9; e++) x[e] = x1[e];
#pragma unroll
        for (int s = 0; s < 4; s++) {
            if (s != 2) { make_A(RS(s), ah, A); if (MODEL == 2) make_A(RS(s), gt, C); }
            ldst9<S>(Po, TG, sl, SL_TG, s, tg);
#pragma unroll
            for (int i = 0; i < 3; i++)
#pragma unroll
                for (int j = 0; j < 3; j++) {
                    T t = T(0);
#pragma unroll
                    for (int m = 0; m < 3; m++) t = fma(A[3 * i + m], tg[3 * m + j], t);
                    if (MODEL == 2) {
#pragma unroll
                        for (int m = 0; m < 3; m++) t = fma(C[3 * i + m], cg[3 * m + j], t);
                    }
                    k[3 * i + j] = t;
                }
#pragma unroll
            for (int e = 0; e < 9; e++) { ks[e] = KSUM(ks[e], k[e], s); pgs[e] = KSUM(pgs[e], x[e], s); }
            if (s < 3) {
#pragma unroll
                for (int e = 0; e < 9; e++) x[e] = fma(k[e], CN(s), x1[e]);
                st9<S>(sl, SL_VG + s * 9, x);
            }
        }
#pragma unroll
        for (int e = 0; e < 9; e++) { SM(Pn, VG + e) = fma(dt6, ks[e], x1[e]); SM(Pn, PG + e) = fma(dt6, pgs[e], pg1[e]); }
    }
    CPI_SECTION();
    if (MODEL == 2) {
        // ---- ct (transient clone rows x theta; starts as P_tt, CpiV2.h:436-441):  k = x W - P_cg ;  only its stage values matter
        T x1[9], x[9], cg[9];
        ldsym<S>(Po, TT, x1); ld9<S>(Po, TG, cg);
#pragma unroll
        for (int e = 0; e < 9; e++) x[e] = x1[e];
#pragma unroll
        for (int s = 0; s < 3; s++) {
            T k[9];
#pragma unroll
            for (int i = 0; i < 3; i++) {
                T c3[3];
                cross(&x[3 * i], w, c3);
#pragma unroll
                for (int j = 0; j < 3; j++) k[3 * i + j] = c3[j] - cg[3 * i + j];
            }
#pragma unroll
            for (int e = 0; e < 9; e++) x[e] = fma(k[e], CN(s), x1[e]);
            st9<S>(sl, SL_CT + s * 9, x);
        }
        CPI_SECTION();
    }
    {   // ---- vt:  k = A_s P_tt,s + x W - P_vg,s (+ C_s P_ct,s)
        T x1[9], x[9], ks[9], k[9], tt[9], vg[9], A[9], C[9], ct[9];
        ld9<S>(Po, VT, x1);
#pragma unroll
        for (int e = 0; e < 9; e++) x[e] = x1[e];
#pragma unroll
        for (int s = 0; s < 4; s++) {
            if (s != 2) { make_A(RS(s), ah, A); if (MODEL == 2) make_A(RS(s), gt, C); }
            ldstsym<S>(Po, TT, sl, SL_TT, s, tt);
            ldst9<S>(Po, VG, sl, SL_VG, s, vg);
            if (MODEL == 2) { if (s == 0) ldsym<S>(Po, TT, ct); else ld9<S>(sl, SL_CT + (s - 1) * 9, ct); }
#pragma unroll
            for (int i = 0; i < 3; i++) {
                T c3[3];
                cross(&x[3 * i], w, c3);
#pragma unroll
                for (int j = 0; j < 3; j++) {
                    T t = c3[j] - vg[3 * i + j];
#pragma unroll
                    for (int m = 0; m < 3; m++) t = fma(A[3 * i + m], tt[3 * m + j], t);
                    if (MODEL == 2) {
#pragma unroll
                        for (int m = 0; m < 3; m++) t = fma(C[3 * i + m], ct[3 * m + j], t);
                    }
                    k[3 * i + j] = t;
                }
            }
#pragma unroll
            for (int e = 0; e < 9; e++) ks[e] = KSUM(ks[e], k[e], s);
            if (s < 3) {
#pragma unroll
                for (int e = 0; e < 9; e++) x[e] = fma(k[e], CN(s), x1[e]);
                st9<S>(sl, SL_VT + s * 9, x);
            }
        }
#pragma unroll
        for (int e = 0; e < 9; e++) SM(Pn, VT + e) = fma(dt6, ks[e], x1[e]);
    }
    CPI_SECTION();
    if (MODEL == 2) {
        // ---- cv (transient; starts as P_theta,v = P_vt^T):  k = P_ct,s A_s^T + P_cc C_s^T,  P_cc = P_tt at step start
        T x1[9], cc[9], A[9], C[9];
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) x1[3 * i + j] = SM(Po, VT + 3 * j + i);
        ldsym<S>(Po, TT, cc);
#pragma unroll
        for (int s = 0; s < 3; s++) {
            T ct[9], x[9];
            if (s != 2) { make_A(RS(s), ah, A); make_A(RS(s), gt, C); }
            if (s == 0) ldsym<S>(Po, TT, ct); else ld9<S>(sl, SL_CT + (s - 1) * 9, ct);
#pragma unroll
            for (int i = 0; i < 3; i++)
#pragma unroll
                for (int j = 0; j < 3; j++) {
                    T t = T(0);
#pragma unroll
                    for (int m = 0; m < 3; m++) t = fma(ct[3 * i + m], A[3 * j + m], t);
#pragma unroll
                    for (int m = 0; m < 3; m++) t = fma(cc[3 * i + m], C[3 * j + m], t);
                    x[3 * i + j] = fma(t, CN(s), x1[3 * i + j]);
                }
            st9<S>(sl, SL_CV + s * 9, x);
        }
        CPI_SECTION();
    }
    {   // ---- pt:  k = P_vt,s + x W - P_pg,s ;  P_pg,s = P_pg + CN(s-1) P_vg,s-1  (recomputed, not stored)
        T x1[9], x[9], ks[9], k[9], vt[9], pg1[9], pg[9], vgp[9];
        ld9<S>(Po, PT, x1); ld9<S>(Po, PG, pg1);
#pragma unroll
        for (int e = 0; e < 9; e++) { x[e] = x1[e]; pg[e] = pg1[e]; }
#pragma unroll
        for (int s = 0; s < 4; s++) {
            ldst9<S>(Po, VT, sl, SL_VT, s, vt);
            if (s > 0) {
                ldst9<S>(Po, VG, sl, SL_VG, s - 1, vgp);
#pragma unroll
                for (int e = 0; e < 9; e++) pg[e] = fma(vgp[e], CN(s - 1), pg1[e]);
            }
#pragma unroll
            for (int i = 0; i < 3; i++) {
                T c3[3];
                cross(&x[3 * i], w, c3);
#pragma unroll
                for (int j = 0; j < 3; j++) k[3 * i + j] = vt[3 * i + j] + c3[j] - pg[3 * i + j];
            }
#pragma unroll
            for (int e = 0; e < 9; e++) ks[e] = KSUM(ks[e], k[e], s);
            if (s < 3) {
#pragma unroll
                for (int e = 0; e < 9; e++) x[e] = fma(k[e], CN(s), x1[e]);
                st9<S>(sl, SL_PT + s * 9, x);
            }
        }
#pragma unroll
        for (int e = 0; e < 9; e++) SM(Pn, PT + e) = fma(dt6, ks[e], x1[e]);
    }
    CPI_SECTION();
    {   // ---- va:  k = paa_s B_s      and pa:  k = P_va,s
        T x1[9], x[9], ks[9], pa1[9], pas[9], B[9];
        ld9<S>(Po, VA, x1); ld9<S>(Po, PA, pa1);
#pragma unroll
        for (int e = 0; e < 9; e++) x[e] = x1[e];
#pragma unroll
        for (int s = 0; s < 4; s++) {
            const T pa_s = (s == 0) ? paa : fma(q_ab, (s == 3 ? dt : hdt), paa);
            if (s != 2) make_B(RS(s), B);
#pragma unroll
            for (int e = 0; e < 9; e++) {
                const T kk = pa_s * B[e];
                ks[e] = KSUM(ks[e], kk, s);
                pas[e] = KSUM(pas[e], x[e], s);
                if (s < 3) x[e] = fma(kk, CN(s), x1[e]);
            }
            if (s < 3) st9<S>(sl, SL_VA + s * 9, x);
        }
#pragma unroll
        for (int e = 0; e < 9; e++) { SM(Pn, VA + e) = fma(dt6, ks[e], x1[e]); SM(Pn, PA + e) = fma(dt6, pas[e], pa1[e]); }
    }
    CPI_SECTION();
    {   // ---- vv:  k = M + M^T + q_a I,  M = A_s P_vt,s^T + B_s P_va,s^T (+ C_s P_cv,s),  B_s = -R_s^T used straight from R_s.
        //      Terms are accumulated in fenced passes so that only one operand pair is live at a time.
        T a1[6], ks[6], M[9];
#pragma unroll
        for (int e = 0; e < 6; e++) a1[e] = SM(Po, VV + e);
#pragma unroll
        for (int s = 0; s < 4; s++) {
            {
                T A[9], vt[9];
                make_A(RS(s), ah, A);
                ldst9<S>(Po, VT, sl, SL_VT, s, vt);
#pragma unroll
                for (int i = 0; i < 3; i++)
#pragma unroll
                    for (int j = 0; j < 3; j++) M[3 * i + j] = A[3 * i] * vt[3 * j] + A[3 * i + 1] * vt[3 * j + 1] + A[3 * i + 2] * vt[3 * j + 2];
            }
            CPI_SECTION();
            {
                T va[9];
                const T* Rs = RS(s);
                ldst9<S>(Po, VA, sl, SL_VA, s, va);
#pragma unroll
                for (int i = 0; i < 3; i++)
#pragma unroll
                    for (int j = 0; j < 3; j++)
#pragma unroll
                        for (int m = 0; m < 3; m++) M[3 * i + j] = fma(-Rs[3 * m + i], va[3 * j + m], M[3 * i + j]);
            }
            if (MODEL == 2) {
                CPI_SECTION();
                T C[9], cv[9];
                make_A(RS(s), gt, C);
                if (s == 0) {
#pragma unroll
                    for (int i = 0; i < 3; i++)
#pragma unroll
                        for (int j = 0; j < 3; j++) cv[3 * i + j] = SM(Po, VT + 3 * j + i);      // P_theta,v = P_vt^T
                } else ld9<S>(sl, SL_CV + (s - 1) * 9, cv);
#pragma unroll
                for (int i = 0; i < 3; i++)
#pragma unroll
                    for (int j = 0; j < 3; j++)
#pragma unroll
                        for (int m = 0; m < 3; m++) M[3 * i + j] = fma(C[3 * i + m], cv[3 * m + j], M[3 * i + j]);
            }
#pragma unroll
            for (int i = 0; i < 3; i++)
#pragma unroll
                for (int j = i; j < 3; j++) {
                    const T kk = M[3 * i + j] + M[3 * j + i] + (i == j ? q_a : T(0));
                    ks[sym3(i, j)] = KSUM(ks[sym3(i, j)], kk, s);
                    if (s < 3) SM(sl, SL_VV + s * 6 + sym3(i, j)) = fma(kk, CN(s), a1[sym3(i, j)]);
                }
            CPI_SECTION();
        }
#pragma unroll
        for (int e = 0; e < 6; e++) SM(Pn, VV + e) = fma(dt6, ks[e], a1[e]);
    }
    CPI_SECTION();
    {   // ---- pv:  k = P_vv,s + P_pt,s A_s^T + P_pa,s B_s^T (+ P_cp,s^T C_s^T);  P_pa,s = P_pa + CN(s-1) P_va,s-1 and
        //      P_cp,s = P_pt^T + CN(s-1) P_cv,s-1 are recomputed from the va / cv stage values instead of being stored
        T x1[9], ks[9], k[9];
        ld9<S>(Po, PV, x1);
#pragma unroll
        for (int s = 0; s < 4; s++) {
            {
                T A[9], pt[9];
                ldstsym<S>(Po, VV, sl, SL_VV, s, k);
                make_A(RS(s), ah, A);
                ldst9<S>(Po, PT, sl, SL_PT, s, pt);
#pragma unroll
                for (int i = 0; i < 3; i++)
#pragma unroll
                    for (int j = 0; j < 3; j++)
#pragma unroll
                        for (int m = 0; m < 3; m++) k[3 * i + j] = fma(pt[3 * i + m], A[3 * j + m], k[3 * i + j]);
            }
            CPI_SECTION();
            {
                T pa[9];
                const T* Rs = RS(s);
                ld9<S>(Po, PA, pa);
                if (s > 0) {
                    T prev[9];
                    ldst9<S>(Po, VA, sl, SL_VA, s - 1, prev);
#pragma unroll
                    for (int e = 0; e < 9; e++) pa[e] = fma(prev[e], CN(s - 1), pa[e]);
                }
#pragma unroll
                for (int i = 0; i < 3; i++)
#pragma unroll
                    for (int j = 0; j < 3; j++)
#pragma unroll
                        for (int m = 0; m < 3; m++) k[3 * i + j] = fma(pa[3 * i + m], -Rs[3 * m + j], k[3 * i + j]);
            }
            if (MODEL == 2) {
                CPI_SECTION();
                T C[9], cp[9];
                make_A(RS(s), gt, C);
#pragma unroll
                for (int i = 0; i < 3; i++)
#pragma unroll
                    for (int j = 0; j < 3; j++) cp[3 * i + j] = SM(Po, PT + 3 * j + i);     // P_theta,p = P_pt^T
                if (s > 0) {
                    T prev[9];
                    if (s == 1) {
#pragma unroll
                        for (int i = 0; i < 3; i++)
#pragma unroll
                            for (int j = 0; j < 3; j++) prev[3 * i + j] = SM(Po, VT + 3 * j + i);     // cv stage 1 = P_vt^T
                    } else ld9<S>(sl, SL_CV + (s - 2) * 9, prev);
#pragma unroll
                    for (int e = 0; e < 9; e++) cp[e] = fma(prev[e], CN(s - 1), cp[e]);
                }
#pragma unroll
                for (int i = 0; i < 3; i++)
#pragma unroll
                    for (int j = 0; j < 3; j++)
#pragma unroll
                        for (int m = 0; m < 3; m++) k[3 * i + j] = fma(cp[3 * m + i], C[3 * j + m], k[3 * i + j]);
            }
#pragma unroll
            for (int e = 0; e < 9; e++) {
                ks[e] = KSUM(ks[e], k[e], s);
                if (s < 3) SM(sl, SL_PV + s * 9 + e) = fma(k[e], CN(s), x1[e]);
            }
            CPI_SECTION();
        }
#pragma unroll
        for (int e = 0; e < 9; e++) SM(Pn, PV + e) = fma(dt6, ks[e], x1[e]);
    }
    CPI_SECTION();
    {   // ---- pp:  k = P_pv,s + P_pv,s^T
        T a1[6], ks[6], pv[9];
#pragma unroll
        for (int e = 0; e < 6; e++) a1[e] = SM(Po, PP + e);
#pragma unroll
        for (int s = 0; s < 4; s++) {
            ldst9<S>(Po, PV, sl, SL_PV, s, pv);
#pragma unroll
            for (int i = 0; i < 3; i++)
#pragma unroll
                for (int j = i; j < 3; j++) ks[sym3(i, j)] = KSUM(ks[sym3(i, j)], pv[3 * i + j] + pv[3 * j + i], s);
        }
#pragma unroll
        for (int e = 0; e < 6; e++) SM(Pn, PP + e) = fma(dt6, ks[e], a1[e]);
    }
    CPI_SECTION();
}
#undef CN
#undef RS
#undef KSUM

// I - a W + b W2 applied to R:  out = (I - a [w x] + b [w x]^2) R
CPI_DEV void rot_apply(double a, double b, const double* w, const double* R, double* out) {
    const double w00 = -(w[1] * w[1] + w[2] * w[2]), w11 = -(w[0] * w[0] + w[2] * w[2]), w22 = -(w[0] * w[0] + w[1] * w[1]);
    const double w01 = w[0] * w[1], w02 = w[0] * w[2], w12 = w[1] * w[2];
    double D[9];
    D[0] = 1.0 + b * w00;      D[1] = a * w[2] + b * w01; D[2] = -a * w[1] + b * w02;
    D[3] = -a * w[2] + b * w01; D[4] = 1.0 + b * w11;     D[5] = a * w[0] + b * w12;
    D[6] = a * w[1] + b * w02;  D[7] = -a * w[0] + b * w12; D[8] = 1.0 + b * w22;
    mul33(D, R, out);
}

// =====================================================================================================================
// Per-sample "front" work: estimated readings, rotation chain (new and mid-point rotation), closed-form means and the
// analytic bias Jacobians (CpiV1.h:77-259; CpiV2.h:98-305).  Everything the covariance step needs comes out as
// (wh, ah, g_tau, Rm, R1); R (old rotation) is NOT committed here.  Jacobian state lives in the tile (Jt).
template <int MODEL, bool AVG, bool ANALYTIC, int S>
CPI_DEV void front_step(const double* s0, const double* nx, const double* bw, const double* ba, const double* g_k, const double* R,
                        double* alpha, double* beta, double* Jt, double* wh, double* ah, double* g_tau, double* Rm, double* R1) {
    const double dt = s0[6];
    // ---- estimated readings (CpiV1.h:77-86; CpiV2.h:98-106)
    wh[0] = s0[0] - bw[0]; wh[1] = s0[1] - bw[1]; wh[2] = s0[2] - bw[2];
    ah[0] = s0[3] - ba[0]; ah[1] = s0[4] - ba[1]; ah[2] = s0[5] - ba[2];
    g_tau[0] = g_tau[1] = g_tau[2] = 0.0;
    if (MODEL == 2) {
        mv33(R, g_k, g_tau);                         // R_k2tau * R_G_to_k * grav  (old R)
        ah[0] -= g_tau[0]; ah[1] -= g_tau[1]; ah[2] -= g_tau[2];
    }
    if (AVG) {
#pragma unroll
        for (int e = 0; e < 3; e++) { wh[e] += nx[e] - bw[e]; wh[e] = 0.5 * wh[e]; }
        if (MODEL == 1) {
#pragma unroll
            for (int e = 0; e < 3; e++) { ah[e] += nx[3 + e] - ba[e]; ah[e] = 0.5 * ah[e]; }
        }
    }
    const double mag2 = wh[0] * wh[0] + wh[1] * wh[1] + wh[2] * wh[2];
    const double mag = sqrt(mag2);
    const double th = mag * dt;
    const bool small_w = mag < 0.008726646;          // CpiV1.h:101
    double sn, cs_, sh, ch;
    sincos(th, &sn, &cs_);
    sincos(mag * 0.5 * dt, &sh, &ch);
    // one reciprocal instead of ~16 divisions (each an ~40-instruction subroutine); never used when small_w
    const double im = small_w ? 0.0 : 1.0 / mag;
    const double im2 = im * im;

    // ---- relative rotation, new and mid rotation (CpiV1.h:119-124, 267-269)
    const double a1 = small_w ? dt : sn * im, b1 = small_w ? (dt * dt) * 0.5 : (1.0 - cs_) * im2;
    rot_apply(a1, b1, wh, R, R1);
    {
        const double hd = 0.5 * dt;
        const double a2 = small_w ? hd : sh * im, b2 = small_w ? (hd * hd) * 0.5 : (1.0 - ch) * im2;
        rot_apply(a2, b2, wh, R, Rm);
    }
    if (MODEL == 2 && AVG) {                         // CpiV2.h:146-149: average the LOCAL acceleration with the NEW rotation
        double g1[3];
        mv33(R1, g_k, g1);
#pragma unroll
        for (int e = 0; e < 3; e++) { ah[e] += nx[3 + e] - ba[e] - g1[e]; ah[e] = 0.5 * ah[e]; }
    }

    // ---- closed-form coefficients (CpiV1.h:132-142, 196-238 == CpiV2.h:158-168, 231-274)
    double f1, f2, f3, f4, d1, d2, d3, d4;
    {
        const double dt2 = dt * dt, dt3 = dt2 * dt;
        if (small_w) {
            f1 = -(dt3 / 3.0); f2 = (dt2 * dt2) / 8.0; f3 = -(dt2 / 2.0); f4 = dt3 / 6.0;
            d1 = -(dt3 * dt2 / 15.0); d2 = (dt3 * dt3) / 72.0; d3 = -(dt2 * dt2 / 12.0); d4 = (dt3 * dt2) / 60.0;
        } else {
            const double im3 = im2 * im, im4 = im2 * im2, th2 = th * th;
            f1 = (th * cs_ - sn) * im3;
            f2 = (th2 - 2.0 * cs_ - 2.0 * th * sn + 2.0) * (0.5 * im4);
            f3 = -(1.0 - cs_) * im2;
            f4 = (th - sn) * im3;
            if (MODEL == 1 || ANALYTIC) {
                d1 = (th2 * sn - 3.0 * sn + 3.0 * th * cs_) * (im4 * im);
                d2 = (th2 - 4.0 * cs_ - 4.0 * th * sn + th2 * cs_ + 4.0) * (im4 * im2);
                d3 = (2.0 * (cs_ - 1.0) + th * sn) * im4;
                d4 = (2.0 * th + th * cs_ - 3.0 * sn) * (im4 * im);
            }
        }
    }

    // W and W^2 entries
    const double W2[9] = {-(wh[1] * wh[1] + wh[2] * wh[2]), wh[0] * wh[1], wh[0] * wh[2],
                          wh[0] * wh[1], -(wh[0] * wh[0] + wh[2] * wh[2]), wh[1] * wh[2],
                          wh[0] * wh[2], wh[1] * wh[2], -(wh[0] * wh[0] + wh[1] * wh[1])};
    const double Wm[9] = {0.0, -wh[2], wh[1], wh[2], 0.0, -wh[0], -wh[1], wh[0], 0.0};
    double aarg[9], barg[9], Hal[9], Hbe[9];
    {
        const double hdt2 = (dt * dt) * 0.5;
#pragma unroll
        for (int e = 0; e < 9; e++) {
            aarg[e] = ((e % 4 == 0) ? hdt2 : 0.0) + f1 * Wm[e] + f2 * W2[e];     // CpiV1.h:145
            barg[e] = ((e % 4 == 0) ? dt : 0.0) + f3 * Wm[e] + f4 * W2[e];       // CpiV1.h:146
        }
    }
    mulT33(R1, aarg, Hal);                            // R_tau12k * alpha_arg
    mulT33(R1, barg, Hbe);
    {
        double t3[3];
        mv33(Hal, ah, t3);
#pragma unroll
        for (int e = 0; e < 3; e++) alpha[e] += beta[e] * dt + t3[e];   // CpiV1.h:153 (old beta)
        mv33(Hbe, ah, t3);
#pragma unroll
        for (int e = 0; e < 3; e++) beta[e] += t3[e];                   // CpiV1.h:154
    }

    if (MODEL == 1 || ANALYTIC) {
        // ---- analytic bias Jacobians (CpiV1.h:162-259; CpiV2.h:188-305); state lives in the tile, not in registers
        double Jq[9], Jsave[9];
        ld9<S>(Jt, J_Q, Jq);
#pragma unroll
        for (int e = 0; e < 9; e++) Jsave[e] = Jq[e];
        {
            const double ith = small_w ? 0.0 : 1.0 / th;
            const double c1 = small_w ? 0.5 : (1.0 - cs_) * (ith * ith), c2 = small_w ? (1.0 / 6.0) : (th - sn) * (ith * ith * ith);
            double t9[9];
            rot_apply(a1, b1, wh, Jsave, t9);         // R_tau2tau1 * J_q
            const double ca = c1 * dt, cb = c2 * dt * dt;   // w_tx = dt*W, w_tx^2 = dt^2 W2
#pragma unroll
            for (int e = 0; e < 9; e++) {
                Jq[e] = t9[e] + (((e % 4 == 0) ? 1.0 : 0.0) - ca * Wm[e] + cb * W2[e]) * dt;   // CpiV1.h:167
                SM(Jt, J_Q + e) = Jq[e];
            }
        }
#pragma unroll
        for (int e = 0; e < 9; e++) {                  // CpiV1.h:170-172 (old H_b)
            const double hb = SM(Jt, H_B + e);
            SM(Jt, H_A + e) = (SM(Jt, H_A + e) - Hal[e]) + dt * hb;
            SM(Jt, H_B + e) = hb - Hbe[e];
        }
        if (MODEL == 2) {                              // CpiV2.h:203-205
            const double sk[9] = {0.0, -g_k[2], g_k[1], g_k[2], 0.0, -g_k[0], -g_k[1], g_k[0], 0.0};
            double t1[9], t2[9], t4[9];
            mul33(R, sk, t1);
            mul33(Hal, t1, t2);
            mul33(Hbe, t1, t4);
#pragma unroll
            for (int e = 0; e < 9; e++) {
                const double ob = SM(Jt, O_B + e);
                SM(Jt, O_A + e) = (SM(Jt, O_A + e) + dt * ob) + -t2[e];
                SM(Jt, O_B + e) = ob + -t4[e];
            }
        }
        // vectors shared by the three columns
        double ua[3], ub[3], Wa[3], W2a[3];
        mv33(aarg, ah, ua); mv33(barg, ah, ub);
        cross(wh, ah, Wa);                             // W a = w x a
        cross(wh, Wa, W2a);                            // W^2 a
#pragma unroll
        for (int col = 0; col < 3; col++) {
            const double e3[3] = {col == 0 ? 1.0 : 0.0, col == 1 ? 1.0 : 0.0, col == 2 ? 1.0 : 0.0};
            const double jc[3] = {Jq[col], Jq[3 + col], Jq[6 + col]};   // NEW J_q e_i
            double exa[3], exWa[3], Wexa[3], c1v[3], c2v[3], va_[3], vb_[3], oa3[3], ob3[3];
            cross(e3, ah, exa);                        // e_ix a
            cross(e3, Wa, exWa);                       // e_ix W a
            cross(wh, exa, Wexa);                      // W e_ix a
            cross(jc, ua, c1v);                        // [J_q e_i x] (alpha_arg a)
            cross(jc, ub, c2v);
            const double wi = wh[col];
#pragma unroll
            for (int e = 0; e < 3; e++) {
                va_[e] = -c1v[e] + (wi * d1) * Wa[e] - f1 * exa[e] + (wi * d2) * W2a[e] - f2 * (exWa[e] + Wexa[e]);
                vb_[e] = -c2v[e] + (wi * d3) * Wa[e] - f3 * exa[e] + (wi * d4) * W2a[e] - f4 * (exWa[e] + Wexa[e]);
            }
            mvT33(R1, va_, oa3);
            mvT33(R1, vb_, ob3);
            if (MODEL == 2) {                          // - H_al [J_save e_i x] g_tau (CpiV2.h:285-293); J_b column 0 carries
                const double js[3] = {Jsave[col], Jsave[3 + col], Jsave[6 + col]};   // the reference's "- -" = plus (:296-297)
                double cg[3], u[3];
                cross(js, g_tau, cg);
                mv33(Hal, cg, u);
                oa3[0] -= u[0]; oa3[1] -= u[1]; oa3[2] -= u[2];
                mv33(Hbe, cg, u);
                if (col == 0) { ob3[0] += u[0]; ob3[1] += u[1]; ob3[2] += u[2]; }
                else { ob3[0] -= u[0]; ob3[1] -= u[1]; ob3[2] -= u[2]; }
            }
#pragma unroll
            for (int r = 0; r < 3; r++) {              // J_a += J_b*dt (old J_b, CpiV1.h:241) then the column terms
                const double jb = SM(Jt, J_B + 3 * r + col);
                SM(Jt, J_A + 3 * r + col) = (SM(Jt, J_A + 3 * r + col) + jb * dt) + oa3[r];
                SM(Jt, J_B + 3 * r + col) = jb + ob3[r];
            }
        }
    }

}

// =====================================================================================================================
// Sample stream: per-window contiguous entries of 7 doubles.  Without imu_avg it is staged with 1-D TMA bulk copies
// (cp.async.bulk -> SASS UBLKCP): every lane owns two 128-byte line buffers and two mbarriers and keeps two chunks of
// two samples (112 B, fetched as ONE aligned 128-byte transaction that also covers the 8-byte misalignment of odd
// window offsets) in flight ahead of the arithmetic.  The last chunk of a window is read with plain loads because the
// aligned 128-byte fetch could run past the end of the caller's buffer there.
template <int MODEL, bool AVG, bool ANALYTIC, class T>
__global__ void __launch_bounds__(128, 1) k_preintegrate(const PreintParams p) {
    using TL = Tile<MODEL, T>;
    constexpr int S = TL::S;
    constexpr int CH = 8 / (int)sizeof(T) * 2;           // samples per TMA chunk: 2 (fp64, 2 x 56 B) or 4 (fp32, 4 x 28 B) = 112 B
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int tid = threadIdx.x;
    const int64_t win = (int64_t)blockIdx.x * p.wpb + tid;
    if (tid >= p.wpb || win >= p.n_windows) return;

    double* Jt = reinterpret_cast<double*>(smem_raw) + tid;                       // analytic Jacobians, or Discrete_J_b blocks (model 2 default)
    T* P = reinterpret_cast<T*>(smem_raw + tile_off_T<MODEL, T>()) + tid;         // current covariance tile (ping-pongs with Pn every step)
    T* Pn = P + (size_t)NP * S;
    T* sl = P + (size_t)2 * NP * S;                                               // RK4 stage-value slots
    const T* buf = reinterpret_cast<const T*>(smem_raw + tile_off_buf<MODEL, T>() + (size_t)tid * 256);
    const uint32_t buf0 = smem_u32(buf);
    const uint32_t bar0 = smem_u32(smem_raw + tile_off_bar<MODEL, T>() + (size_t)tid * 16);

    // ---- per-window constants (setLinearizationPoints, CpiBase.h:73-80)
    const T* lin = reinterpret_cast<const T*>(p.lin) + win * CPI_LIN_DOUBLES;
    const double bw[3] = {(double)lin[0], (double)lin[1], (double)lin[2]}, ba[3] = {(double)lin[3], (double)lin[4], (double)lin[5]};
    double g_k[3] = {0, 0, 0};
    if (MODEL == 2) {
        const double q[4] = {(double)lin[6], (double)lin[7], (double)lin[8], (double)lin[9]}, g[3] = {(double)lin[10], (double)lin[11], (double)lin[12]};
        double RG[9];
        quat_2_Rot(q, RG);
        mv33(RG, g, g_k);                                // quat_2_Rot(q_k_lin) * grav   (CpiV2.h:99, 202, 315)
    }
    int64_t o0, nsteps;
    if (p.offsets) { o0 = p.offsets[win]; nsteps = p.offsets[win + 1] - o0 - (AVG ? 1 : 0); }
    else { o0 = win * (p.ns_uniform + (AVG ? 1 : 0)); nsteps = p.ns_uniform; }
    if (nsteps < 0) nsteps = 0;
    const T* sp = reinterpret_cast<const T*>(p.samples) + o0 * CPI_SAMPLE_DOUBLES;

    // ---- TMA pipeline set-up
    const int shift = (int)(((uintptr_t)sp & 15) / sizeof(T));   // misalignment of the window start w.r.t. 16 bytes, in elements
    const int64_t n_tma = AVG ? 0 : (nsteps > 0 ? (nsteps - 1) / CH : 0);   // chunks with at least one more sample after them
    if (!AVG) {
        mbar_init(bar0, 1); mbar_init(bar0 + 8, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        fence_proxy_async();
#pragma unroll
        for (int c = 0; c < 2; c++)
            if (c < n_tma) {
                mbar_arrive_expect_tx(bar0 + 8 * c, 128);
                bulk_g2s(buf0 + 128 * c, sp + 7 * CH * c - shift, 128, bar0 + 8 * c);
            }
    }

    // ---- state (CpiBase.h:99-124 initialisers)
    double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    double alpha[3] = {0, 0, 0}, beta[3] = {0, 0, 0}, DT = 0.0;
    double pgg = 0.0, paa = 0.0;
#pragma unroll 1
    for (int e = 0; e < NP; e++) SM(P, e) = T(0);
#pragma unroll 1
    for (int e = 0; e < TL::NJ; e++) SM(Jt, e) = 0.0;

#pragma unroll 1
    for (int64_t it = 0; it < nsteps; it++) {
        // ---- fetch entry `it` (and, for imu_avg, the (w, a) of entry it+1)
        double s0[7], nx[6];
        if (!AVG && it < CH * n_tma) {
            const int64_t c = it / CH;
            const int b = (int)(c & 1), j = (int)(it % CH);
            if (j == 0) mbar_wait(bar0 + 8 * b, (uint32_t)((c >> 1) & 1));
            const T* src = buf + b * (128 / (int)sizeof(T)) + shift + 7 * j;
#pragma unroll
            for (int e = 0; e < 7; e++) s0[e] = (double)src[e];
            if (j == CH - 1 && c + 2 < n_tma) {
                fence_proxy_async();                     // generic-proxy reads of this buffer are done; hand it to the async proxy
                mbar_arrive_expect_tx(bar0 + 8 * b, 128);
                bulk_g2s(buf0 + 128 * b, sp + 7 * CH * (c + 2) - shift, 128, bar0 + 8 * b);
            }
        } else {
#pragma unroll
            for (int e = 0; e < 7; e++) s0[e] = (double)__ldg(sp + it * CPI_SAMPLE_DOUBLES + e);
            if (AVG) {
#pragma unroll
                for (int e = 0; e < 6; e++) nx[e] = (double)__ldg(sp + (it + 1) * CPI_SAMPLE_DOUBLES + e);
            }
        }
        const double dt = s0[6];
        DT += dt;                                        // CpiV1.h:69
        if (dt == 0.0) continue;                         // CpiV1.h:72-74

        double wh[3], ah[3], g_tau[3], Rm[9], R1[9];
        front_step<MODEL, AVG, ANALYTIC, S>(s0, nx, bw, ba, g_k, R, alpha, beta, Jt, wh, ah, g_tau, Rm, R1);

        // ---- covariance: the reference's RK4, block-serial on the block-triangular Lyapunov operator (rk4_cascade)
        const double hdt = dt * 0.5, dt6 = dt / 6.0;
        rk4_cascade<MODEL, S, T>(P, Pn, sl, wh, ah, g_tau, R, Rm, R1, pgg, paa, dt, p.q_w, p.q_wb, p.q_a, p.q_ab);
        { T* t = P; P = Pn; Pn = t; }
        pgg += dt6 * (p.q_wb + 2.0 * p.q_wb + 2.0 * p.q_wb + p.q_wb);
        paa += dt6 * (p.q_ab + 2.0 * p.q_ab + 2.0 * p.q_ab + p.q_ab);

        if (MODEL == 2 && !ANALYTIC) {
            // ---- Discrete_J_b <- B_k * Phi * Discrete_J_b restricted to the consumed columns (CpiV2.h:347-426, 443).
            // Phi's RK4 (Phi_dot = F Phi, Phi(0) = I) in block form; stage matrices F1 (R_old), F2 = F3 (R_mid), F4 (R_new).
            //   row theta:  X' = -W X (- I for the bg column)
            //   row v:      k_s = A_s X_theta,s  (+ the direct blocks B_s, C_s, L_s for the identity rows of Phi)
            //   row p:      k_s = (row v stage VALUE)_s = {0, hdt k_1, hdt k_2, dt k_3}
            // Phi_v,X = dt/6 (k1 + 2k2 + 2k3 + k4),  Phi_p,X = dt/6 (2 hdt k1 + 2 hdt k2 + dt k3),  Phi_p,v = dt I.
            // Done in fenced sections that park the theta-row stage values in the (now free) RK4 slots, so that the
            // register allocator never sees more than ~60 live doubles.
            const double Ppv = dt6 * (1.0 + 2.0 + 2.0 + 1.0);
            {   // section 1: theta row.  X_tt,s -> slot A, X_tg,s -> slot B (s = 1..3);  D_tg' -> slot C (committed last)
                double xtt[9], xtg[9], stt[9], stg[9], k1[9], k2[9];
#pragma unroll
                for (int e = 0; e < 9; e++) { xtt[e] = (e % 4 == 0) ? 1.0 : 0.0; xtg[e] = 0.0; }
#pragma unroll
                for (int st = 0; st < 4; st++) {
#pragma unroll
                    for (int j = 0; j < 3; j++) {
                        const double col[3] = {xtt[j], xtt[3 + j], xtt[6 + j]}, col2[3] = {xtg[j], xtg[3 + j], xtg[6 + j]};
                        double c3[3];
                        cross(col, wh, c3);
                        k1[j] = c3[0]; k1[3 + j] = c3[1]; k1[6 + j] = c3[2];
                        cross(col2, wh, c3);
                        k2[j] = c3[0] - (j == 0 ? 1.0 : 0.0); k2[3 + j] = c3[1] - (j == 1 ? 1.0 : 0.0); k2[6 + j] = c3[2] - (j == 2 ? 1.0 : 0.0);
                    }
#pragma unroll
                    for (int e = 0; e < 9; e++) {
                        stt[e] = (st == 0) ? k1[e] : (st == 3 ? stt[e] + k1[e] : stt[e] + 2.0 * k1[e]);
                        stg[e] = (st == 0) ? k2[e] : (st == 3 ? stg[e] + k2[e] : stg[e] + 2.0 * k2[e]);
                    }
                    if (st < 3) {
                        const double cstep = (st == 2) ? dt : hdt;
#pragma unroll
                        for (int e = 0; e < 9; e++) {
                            xtt[e] = ((e % 4 == 0) ? 1.0 : 0.0) + k1[e] * cstep;
                            xtg[e] = k2[e] * cstep;
                            SM(sl, SLOT_A + st * 9 + e) = (T)xtt[e];
                            SM(sl, SLOT_B + st * 9 + e) = (T)xtg[e];
                        }
                    }
                }
                double Dtg[9], n1[9];
                ld9<S>(Jt, D_TG, Dtg);
#pragma unroll
                for (int e = 0; e < 9; e++) { stt[e] = ((e % 4 == 0) ? 1.0 : 0.0) + dt6 * stt[e]; stg[e] = dt6 * stg[e]; }   // Phi_tt, Phi_tg
                mul33(stt, Dtg, n1);
#pragma unroll
                for (int e = 0; e < 9; e++) SM(sl, SLOT_C + e) = (T)(n1[e] + stg[e]);
            }
            CPI_SECTION();
            {   // section 2: bg column of rows v and p
                double swt[9], sut[9], swg[9], sug[9], A[9], X[9], k[9];
#pragma unroll
                for (int st = 0; st < 4; st++) {
                    if (st != 2) make_A(st == 0 ? R : (st == 3 ? R1 : Rm), ah, A);
                    // theta-theta column:  k = A_s X_tt,s   (X_tt,1 = I)
                    if (st == 0) {
#pragma unroll
                        for (int e = 0; e < 9; e++) k[e] = A[e];
                    } else { ld9<S>(sl, SLOT_A + (st - 1) * 9, X); mul33(A, X, k); }
#pragma unroll
                    for (int e = 0; e < 9; e++) {
                        swt[e] = (st == 0) ? k[e] : (st == 3 ? swt[e] + k[e] : swt[e] + 2.0 * k[e]);
                        if (st < 3) sut[e] = (st == 0) ? 2.0 * (k[e] * hdt) : (st == 1 ? sut[e] + 2.0 * (k[e] * hdt) : sut[e] + k[e] * dt);
                    }
                    // theta-bg column:  k = A_s X_tg,s   (X_tg,1 = 0)
                    if (st == 0) {
#pragma unroll
                        for (int e = 0; e < 9; e++) { swg[e] = 0.0; sug[e] = 2.0 * (0.0 * hdt); }
                    } else {
                        ld9<S>(sl, SLOT_B + (st - 1) * 9, X); mul33(A, X, k);
#pragma unroll
                        for (int e = 0; e < 9; e++) {
                            swg[e] = (st == 3) ? swg[e] + k[e] : swg[e] + 2.0 * k[e];
                            if (st < 3) sug[e] = (st == 1) ? sug[e] + 2.0 * (k[e] * hdt) : sug[e] + k[e] * dt;
                        }
                    }
                }
                double Pv[9], Pp[9];
                {   // clone-column direct blocks  C_s = -R_s^T [g_tau x]  (three distinct values)
                    double C0[9], Cm[9], C1[9];
                    make_A(R, g_tau, C0); make_A(Rm, g_tau, Cm); make_A(R1, g_tau, C1);
#pragma unroll
                    for (int e = 0; e < 9; e++) {
                        const double swc = C0[e] + 2.0 * Cm[e] + 2.0 * Cm[e] + C1[e];
                        const double suc = 2.0 * (C0[e] * hdt) + 2.0 * (Cm[e] * hdt) + Cm[e] * dt;
                        Pv[e] = dt6 * swt[e] + dt6 * swc;            // Phi_v,theta + Phi_v,c
                        Pp[e] = dt6 * sut[e] + dt6 * suc;            // Phi_p,theta + Phi_p,c
                    }
                }
                double Dtg[9], Dvg[9], Dpg[9], n2[9], n3[9];
                ld9<S>(Jt, D_TG, Dtg); ld9<S>(Jt, D_VG, Dvg); ld9<S>(Jt, D_PG, Dpg);
                mul33(Pv, Dtg, n2); mul33(Pp, Dtg, n3);
#pragma unroll
                for (int e = 0; e < 9; e++) {
                    SM(Jt, D_PG + e) = n3[e] + dt6 * sug[e] + Ppv * Dvg[e] + Dpg[e];
                    SM(Jt, D_VG + e) = n2[e] + dt6 * swg[e] + Dvg[e];
                }
            }
            CPI_SECTION();
            {   // section 3: ba and theta_klin columns (direct blocks):  Phi_v,a = dt/6 (B1 + 2 Bm + 2 Bm + B4),  Phi_v,l likewise with
                // L_s = -R_s^T R_old [g_k x]  (CpiV2.h:336)
                const double sk[9] = {0.0, -g_k[2], g_k[1], g_k[2], 0.0, -g_k[0], -g_k[1], g_k[0], 0.0};
                double RS[9], L0[9], Lm[9], L1[9];
                mul33(R, sk, RS);
                mulT33(R, RS, L0); mulT33(Rm, RS, Lm); mulT33(R1, RS, L1);
#pragma unroll
                for (int i = 0; i < 3; i++)
#pragma unroll
                    for (int j = 0; j < 3; j++) {
                        const int e = 3 * i + j;
                        const double b0 = -R[3 * j + i], bm = -Rm[3 * j + i], b1 = -R1[3 * j + i];
                        const double Pva = dt6 * (b0 + 2.0 * bm + 2.0 * bm + b1);
                        const double Ppa = dt6 * (2.0 * (b0 * hdt) + 2.0 * (bm * hdt) + bm * dt);
                        const double l0 = -L0[e], lm = -Lm[e], l1 = -L1[e];
                        const double Pvl = dt6 * (l0 + 2.0 * lm + 2.0 * lm + l1);
                        const double Ppl = dt6 * (2.0 * (l0 * hdt) + 2.0 * (lm * hdt) + lm * dt);
                        const double dva = SM(Jt, D_VA + e), dvl = SM(Jt, D_VL + e);
                        SM(Jt, D_PA + e) = Ppa + Ppv * dva + SM(Jt, D_PA + e);
                        SM(Jt, D_VA + e) = Pva + dva;
                        SM(Jt, D_PL + e) = Ppl + Ppv * dvl + SM(Jt, D_PL + e);
                        SM(Jt, D_VL + e) = Pvl + dvl;
                    }
                // commit D_tg' (parked in slot C by section 1; sections 2 needed the old value)
#pragma unroll
                for (int e = 0; e < 9; e++) SM(Jt, D_TG + e) = (double)SM(sl, SLOT_C + e);
            }
            CPI_SECTION();
        }

        // ---- commit rotation (CpiV1.h:357)
#pragma unroll
        for (int e = 0; e < 9; e++) R[e] = R1[e];
    }

    // ---- write the record (column-major 3x3 / 15x15, include/cpi_b200.h)
    constexpr int RD = (MODEL == 1) ? CPI_REC_V1_DOUBLES : CPI_REC_V2_DOUBLES;
    T* rec = reinterpret_cast<T*>(p.out) + win * (int64_t)RD;
    {
        double q[4];
        rot_2_quat(R, q);                                  // CpiV1.h:358 (only the last one is ever consumed)
        rec[CPI_REC_Q] = (T)q[0]; rec[CPI_REC_Q + 1] = (T)q[1]; rec[CPI_REC_Q + 2] = (T)q[2]; rec[CPI_REC_Q + 3] = (T)q[3];
    }
    {
        // Jacobian blocks: analytic state, or the read-out of Discrete_J_b (CpiV2.h:450-458: J_q = -D[theta,bg], J_a = D[p,bg],
        // J_b = D[v,bg], H_a = D[p,ba], H_b = D[v,ba], O_a = D[p,l], O_b = D[v,l])
        constexpr bool DJ = (MODEL == 2 && !ANALYTIC);
        constexpr int oJq = DJ ? D_TG : J_Q, oJa = DJ ? D_PG : J_A, oJb = DJ ? D_VG : J_B, oHa = DJ ? D_PA : H_A, oHb = DJ ? D_VA : H_B,
                      oOa = DJ ? D_PL : O_A, oOb = DJ ? D_VL : O_B;
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) {
                rec[CPI_REC_R + i + 3 * j] = (T)(R[3 * i + j]);
                rec[CPI_REC_JQ + i + 3 * j] = (T)(DJ ? -SM(Jt, oJq + 3 * i + j) : SM(Jt, oJq + 3 * i + j));
                rec[CPI_REC_JA + i + 3 * j] = (T)(SM(Jt, oJa + 3 * i + j));
                rec[CPI_REC_JB + i + 3 * j] = (T)(SM(Jt, oJb + 3 * i + j));
                rec[CPI_REC_HA + i + 3 * j] = (T)(SM(Jt, oHa + 3 * i + j));
                rec[CPI_REC_HB + i + 3 * j] = (T)(SM(Jt, oHb + 3 * i + j));
                if (MODEL == 2) { rec[CPI_REC_OA + i + 3 * j] = (T)(SM(Jt, oOa + 3 * i + j)); rec[CPI_REC_OB + i + 3 * j] = (T)(SM(Jt, oOb + 3 * i + j)); }
            }
    }
#pragma unroll
    for (int e = 0; e < 3; e++) { rec[CPI_REC_ALPHA + e] = (T)alpha[e]; rec[CPI_REC_BETA + e] = (T)beta[e]; }
    rec[CPI_REC_DT] = (T)DT;
    // P_meas, full 15x15: block (I,J), I,J in {theta=0,bg=1,v=2,ba=3,p=4}
    T* Pm = rec + CPI_REC_P;
    auto put = [&](int r, int c, T v) { Pm[r + 15 * c] = v; };
#pragma unroll 1
    for (int i = 0; i < 3; i++)
#pragma unroll 1
        for (int j = 0; j < 3; j++) {
            const int sidx = sym3(i, j);
            put(i, j, SM(P, TT + sidx));            put(6 + i, 6 + j, SM(P, VV + sidx));      put(12 + i, 12 + j, SM(P, PP + sidx));
            put(3 + i, 3 + j, i == j ? (T)pgg : T(0));  put(9 + i, 9 + j, i == j ? (T)paa : T(0));
            put(i, 9 + j, T(0)); put(9 + j, i, T(0)); put(3 + i, 9 + j, T(0)); put(9 + j, 3 + i, T(0));
            T v;
            v = SM(P, TG + 3 * i + j); put(i, 3 + j, v);      put(3 + j, i, v);
            v = SM(P, VT + 3 * i + j); put(6 + i, j, v);      put(j, 6 + i, v);
            v = SM(P, VG + 3 * i + j); put(6 + i, 3 + j, v);  put(3 + j, 6 + i, v);
            v = SM(P, VA + 3 * i + j); put(6 + i, 9 + j, v);  put(9 + j, 6 + i, v);
            v = SM(P, PT + 3 * i + j); put(12 + i, j, v);     put(j, 12 + i, v);
            v = SM(P, PG + 3 * i + j); put(12 + i, 3 + j, v); put(3 + j, 12 + i, v);
            v = SM(P, PV + 3 * i + j); put(12 + i, 6 + j, v); put(6 + j, 12 + i, v);
            v = SM(P, PA + 3 * i + j); put(12 + i, 9 + j, v); put(9 + j, 12 + i, v);
        }
}

// ---- host-side launcher (called from capi.cu) --------------------------------------------------------------------------
template <int MODEL, bool AVG, bool ANALYTIC, class T>
static cudaError_t launch_one(const PreintParams& p, int grid, int block, cudaStream_t st) {
    auto kern = k_preintegrate<MODEL, AVG, ANALYTIC, T>;
    static bool configured[64] = {false};     // per instantiation and device; the attribute is sticky per device context
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 64 || !configured[dev]) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tile_bytes<MODEL, T>());
        if (e != cudaSuccess) return e;
        if (dev < 64) configured[dev] = true;
    }
    kern<<<grid, block, tile_bytes<MODEL, T>(), st>>>(p);
    return cudaGetLastError();
}

// Windows per block.  Small batches: spread over all SMs in ONE wave (a second wave would double the latency of a
// latency-bound launch).  Large batches: the tile's compile-time capacity S.
int preint_pick_wpb(int model, int dtype, int64_t n_windows, int num_sms) {
    const int cap = dtype == 32 ? (model == 1 ? Tile<1, float>::S : Tile<2, float>::S) : (model == 1 ? Tile<1, double>::S : Tile<2, double>::S);
    const int64_t need = (n_windows + num_sms - 1) / num_sms;
    if (need <= cap) return (int)(need < 1 ? 1 : need);
    return cap;
}

int preint_cap(int model, int dtype, int flags, int num_sms) {
    if (flags & CPI_FLAG_DISCRETE) return preint_discrete_cap();
    if (preint_tri_supported(model, flags)) return preint_tri_cap(model, dtype);
    return preint_pick_wpb(model, dtype, (int64_t)1 << 40, num_sms);
}

// Only the modes the tri-lane kernels do not serve get here: imu_avg, and model 2 with analytic Jacobians.
template <class T>
static cudaError_t launch_typed(int model, int flags, const PreintParams& p, int grid, int block, cudaStream_t st) {
    const bool avg = flags & CPI_FLAG_IMU_AVG, ana = flags & CPI_FLAG_ANALYTIC_JACOBIANS;
    if (model == 1) return launch_one<1, true, false, T>(p, grid, block, st);
    if (!ana) return launch_one<2, true, false, T>(p, grid, block, st);
    return avg ? launch_one<2, true, true, T>(p, grid, block, st) : launch_one<2, false, true, T>(p, grid, block, st);
}

cudaError_t preint_launch(int model, int dtype, int flags, const PreintParams& p0, int num_sms, int max_smem_bytes, cudaStream_t st, int* launches) {
    PreintParams p = p0;
    if (p.n_windows == 0) return cudaSuccess;
    if (max_smem_bytes < 232448) return cudaErrorInvalidConfiguration;
    if (flags & CPI_FLAG_DISCRETE) {
        if (launches) *launches = 1;
        return preint_launch_discrete(flags, p, num_sms, st);
    }
    if (preint_tri_supported(model, flags)) {
        if (launches) *launches = 1;
        return preint_launch_tri(model, dtype, p, num_sms, st);
    }
    if (p.init) return cudaErrorNotSupported;      // continuation exists for the tri-lane modes only
    { const int cap = preint_pick_wpb(model, dtype, (int64_t)1 << 40, num_sms);
      if (p.wpb <= 0 || p.wpb > cap) p.wpb = preint_pick_wpb(model, dtype, p.n_windows, num_sms); }
    const int block = (p.wpb + 31) / 32 * 32;
    const int grid = (int)((p.n_windows + p.wpb - 1) / p.wpb);
    cudaError_t e = dtype == 32 ? launch_typed<float>(model, flags, p, grid, block, st) : launch_typed<double>(model, flags, p, grid, block, st);
    if (launches) *launches = 1;
    return e;
}

}  // namespace cpi
