// The Rauch-Tung-Striebel smoothers of filter runs: K15 (k_rts_smooth, after K16's kernels) walks each run with one warp; K16
// scans every keyframe in parallel.  Both form the gain with rts_gain.
//
// K16: parallel-in-time Rauch-Tung-Striebel smoothing of filter runs (cpi_rts_smooth_scan_batch, include/cpi_b200.h; DESIGN.md
// section 3p).  The inputs and outputs are K15's; the latency grows with the log of a run's length instead of the length.
//
// Per transition k of a run (keyframes k -> k+1), from the filter's (x_k, P_k) and K7's (xb_{k+1}, Pb_{k+1}, C_k):
//   G_k = C_k Pb_{k+1}^-1 (rts_gain: K15's arithmetic),  L_k = P_k - G_k Pb_{k+1} G_k^T,  d0_k = local(xb_{k+1}, x_{k+1}),
//   J_k = d local(xb_{k+1}, retract(x_{k+1}, delta)) / d delta at 0 = diag(Jr^-1(phi), I_12), phi the rotation of d0_k
// The element of keyframe k is (E, L, B, a) = (G_k, L_k, G_k J_k, G_k d0_k); a run's last keyframe holds (0, P_{S-1}, 0, 0) and a
// segment flag.  Elements compose as
//   (E_o, L_o, B_o, a_o) o (E_i, L_i, B_i, a_i) = (E_o E_i, L_o + E_o L_i E_o^T, B_o B_i, a_o + B_o a_i)
// (o the outer element, nearer its run's start), and the suffix composition at k holds Ps_k (K15's covariance recursion
// Ps_k = L_k + G_k Ps_{k+1} G_k^T, reassociated) and delta_k, the means' recursion linearised at the filtered states
// (delta_k = G_k d0_k + G_k J_k delta_{k+1}); xs_k = retract(x_k, delta_k) and Xs_k = G_k Ps_{k+1}.
//
// Mapping: element kernel (one warp per keyframe, grid-stride), a segmented reverse scan, apply kernel (one warp per keyframe).  The
// scan is K6's skeleton (scan.cu) on a reflected index: keyframe s sits in workspace slot n - 1 - s, so a run's last keyframe starts
// its segment and the scan runs forward.  (fa, a) (+) (fb, b) = (fa | fb, fb ? b : b o a) applies the segment flag by selection, so a
// NaN run never reaches its neighbours.  Level 0 is the elements; level l + 1 holds one aggregate per chunk of C elements of level l,
// up to the first level of at most C (the top, scanned by one CTA).  Up: pairwise tree per chunk; down: Brent-Kung per chunk, seeded
// with the scanned aggregate of the chunk before.  Level 0's down pass writes back only L and a, so the apply kernel still finds G_k.
// No atomics and a fixed bracketing: every run gives the same bits.  The host launches the levels of n_states, which it knows; device
// offsets are read by the element and apply kernels only.
#include <cuda_runtime.h>
#include <stdint.h>

#include "chol15.cuh"
#include "cpi_kernels.h"
#include "local15.cuh"

namespace cpi {
namespace {

constexpr int C = 16;                 // elements per chunk: slots 0 .. C-1, slot C holds the seed
constexpr int W = 8;                  // warps per CTA of the scan
constexpr int OE = 0, OB = 225, OL = 450, OA = 675, OF = 690;   // element: E, B, L (row-major 15x15), a, flag (1.0 or 0.0)
constexpr int ES = 691;
constexpr size_t SMEM = sizeof(double) * ((C + 1) * ES + W * 225);
constexpr int EW = 4;                 // warps (runs for K15, keyframes for K16's element and apply kernels) per CTA
constexpr int RP = 240;               // one 15x15 matrix, row-major with pitch 16

// The smoother gain G = C Pb^-1 by one warp, never an explicit inverse: L holds Pb on entry and its Cholesky factor on return (lower
// triangle), G holds C on entry and G on return.  Lane i < 15 solves row i of G from row i of C (Pb symmetric: G(i,:)^T = L^-T L^-1
// C(i,:)^T) by two per-lane triangular solves; lane 15 runs spare() meanwhile.  A Pb that is not SPD gives NaN.  The caller syncs the
// warp before reading G.
template <class Spare>
CPI_DEV void rts_gain(double* L, double* G, int lane, Spare spare) {
    warp_chol15(L, lane);
    if (lane < 15) {
        double g[15];
#pragma unroll
        for (int k = 0; k < 15; k++) g[k] = G[lane * 16 + k];
        fwd15(L, g);
#pragma unroll
        for (int k = 0; k < 15; k++) G[lane * 16 + k] = g[k];
    }
    __syncwarp();                             // L reloaded for the backward solve: the two solves do not hold it in registers
    if (lane < 15) {
        double g[15];
#pragma unroll
        for (int k = 0; k < 15; k++) g[k] = G[lane * 16 + k];
        bwd15(L, g);
#pragma unroll
        for (int k = 0; k < 15; k++) G[lane * 16 + k] = g[k];
    } else if (lane == 15) {
        spare();
    }
}

// run c holding keyframe s (runs non-empty), and the run's last keyframe
CPI_DEV int64_t run_of(int64_t n_runs, const int64_t* offs, int64_t uniform, int64_t s, int64_t& last) {
    if (!offs) {
        const int64_t c = s / uniform;
        last = c * uniform + uniform - 1;
        return c;
    }
    int64_t lo = 0, hi = n_runs;
    while (hi - lo > 1) {
        const int64_t m = (lo + hi) / 2;
        if (__ldg(offs + m) <= s) lo = m; else hi = m;
    }
    last = __ldg(offs + lo + 1) - 1;
    return lo;
}

// Jr^-1(phi) (row-major 3x3) = I + [phi]x / 2 + (1 - (t/2) cot(t/2)) / t^2 [phi]x^2, t = |phi| (the series below 1e-4)
CPI_DEV void jr_inv(const double* p, double* J) {
    const double t2 = p[0] * p[0] + p[1] * p[1] + p[2] * p[2], t = sqrt(t2);
    double k;
    if (t < 1e-4) {
        k = 1.0 / 12.0 + t2 / 720.0;
    } else {
        double s, c;
        sincos(0.5 * t, &s, &c);
        k = (1.0 - 0.5 * t * c / s) / t2;
    }
    const double K[9] = {0.0, -p[2], p[1], p[2], 0.0, -p[0], -p[1], p[0], 0.0};
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) {
            const double kk = K[3 * i] * K[j] + K[3 * i + 1] * K[3 + j] + K[3 * i + 2] * K[6 + j];
            J[3 * i + j] = (i == j ? 1.0 : 0.0) + 0.5 * K[3 * i + j] + k * kk;
        }
}

__global__ void __launch_bounds__(EW * 32) k_rts_elements(int64_t n_runs, const int64_t* offs, int64_t uniform, int64_t n,
                                                          const double* states, const double* cov, const double* pred_states,
                                                          const double* pred_cov, const double* cross, double* ws) {
    __shared__ double smem[EW][4 * RP + 32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* Pb = smem[warp];
    double* L = Pb + RP;
    double* G = L + RP;
    double* T = G + RP;                           // G Pb
    double* V = T + RP;                           // d0 (15), Jr^-1 (9)
    for (int64_t s = (int64_t)blockIdx.x * EW + warp; s < n; s += (int64_t)gridDim.x * EW) {
        int64_t last;
        const int64_t c = run_of(n_runs, offs, uniform, s, last);
        double* el = ws + (n - 1 - s) * ES;
        if (s == last) {                          // (0, P_{S-1}, 0, 0), a segment start
            const double* sg = cov + s * 225;
            for (int e = lane; e < 225; e += 32) {
                el[OE + e] = 0.0;
                el[OB + e] = 0.0;
                el[OL + (e % 15) * 15 + e / 15] = __ldg(sg + e);
            }
            if (lane < 15) el[OA + lane] = 0.0;
            if (lane == 0) el[OF] = 1.0;
            continue;
        }
        const int64_t t = s - c;
        const double* pg = pred_cov + t * 225;
        const double* cg = cross + t * 225;
        for (int e = lane; e < 225; e += 32) {    // column-major (r, c) -> row-major pitch 16
            const int r = e % 15, q = e / 15;
            const double p = __ldg(pg + e);
            Pb[r * 16 + q] = p;
            L[r * 16 + q] = p;
            G[r * 16 + q] = __ldg(cg + e);
        }
        __syncwarp();
        rts_gain(L, G, lane, [&] {                // d0 = local(xb_{k+1}, x_{k+1}) and Jr^-1 of its rotation
            double xb[16], x1[16], d[15];
#pragma unroll
            for (int k = 0; k < 16; k++) { xb[k] = __ldg(pred_states + t * CPI_STATE_DOUBLES + k); x1[k] = __ldg(states + (s + 1) * CPI_STATE_DOUBLES + k); }
            local15(xb, x1, d);
#pragma unroll
            for (int k = 0; k < 15; k++) V[k] = d[k];
            jr_inv(d, V + 15);
        });
        __syncwarp();
        if (lane < 15) {                          // row lane of E = G, B = G J, a = G d0 and T = G Pb
            const double* g = G + lane * 16;
            double a = 0.0;
#pragma unroll
            for (int m = 0; m < 15; m++) a = fma(g[m], V[m], a);
            el[OA + lane] = a;
#pragma unroll
            for (int j = 0; j < 15; j++) {
                el[OE + lane * 15 + j] = g[j];
                double b = g[j];
                if (j < 3) b = fma(g[0], V[15 + j], fma(g[1], V[18 + j], g[2] * V[21 + j]));
                el[OB + lane * 15 + j] = b;
            }
#pragma unroll 1
            for (int j = 0; j < 15; j++) {
                double v = 0.0;
#pragma unroll
                for (int m = 0; m < 15; m++) v = fma(g[m], Pb[m * 16 + j], v);
                T[lane * 16 + j] = v;
            }
        }
        __syncwarp();
        if (lane < 15) {                          // L(lane, j) = P_k(lane, j) - T(lane, :) G(j, :)^T, j <= lane, mirrored
            const double* sg = cov + s * 225;
            for (int j = 0; j <= lane; j++) {
                double v = 0.0;
#pragma unroll
                for (int m = 0; m < 15; m++) v = fma(T[lane * 16 + m], G[j * 16 + m], v);
                v = __ldg(sg + j * 15 + lane) - v;
                el[OL + lane * 15 + j] = v;
                el[OL + j * 15 + lane] = v;
            }
        } else if (lane == 15) {
            el[OF] = 0.0;
        }
        __syncwarp();
    }
}

// dst <- o (outer) composed with i (inner), by one warp; every input is read before dst is written.  sc: the warp's 225 doubles.
CPI_DEV void compose(const double* o, const double* i, double* dst, double* sc, int lane) {
    double e[8], b[8], l[4], a = 0.0;
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const int x = lane + 32 * r;
        if (x < 225) {
            const int row = x / 15, col = x - 15 * (x / 15);
            double ve = 0.0, vb = 0.0, vt = 0.0;
#pragma unroll
            for (int m = 0; m < 15; m++) {
                const double eo = o[OE + row * 15 + m];
                ve = fma(eo, i[OE + m * 15 + col], ve);
                vb = fma(o[OB + row * 15 + m], i[OB + m * 15 + col], vb);
                vt = fma(eo, i[OL + m * 15 + col], vt);
            }
            e[r] = ve;
            b[r] = vb;
            sc[x] = vt;                           // T = E_o L_i
        }
    }
    if (lane < 15) {
        double v = 0.0;
#pragma unroll
        for (int m = 0; m < 15; m++) v = fma(o[OB + lane * 15 + m], i[OA + m], v);
        a = o[OA + lane] + v;
    }
    __syncwarp();
#pragma unroll
    for (int r = 0; r < 4; r++) {                 // the lower triangle of L_o + T E_o^T
        const int x = lane + 32 * r;
        if (x < 120) {
            const int row = (int)((sqrt(8.0 * x + 1.0) - 1.0) * 0.5), col = x - row * (row + 1) / 2;
            double v = 0.0;
#pragma unroll
            for (int m = 0; m < 15; m++) v = fma(sc[row * 15 + m], o[OE + col * 15 + m], v);
            l[r] = o[OL + row * 15 + col] + v;
        }
    }
    __syncwarp();
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const int x = lane + 32 * r;
        if (x < 225) { dst[OE + x] = e[r]; dst[OB + x] = b[r]; }
    }
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const int x = lane + 32 * r;
        if (x < 120) {
            const int row = (int)((sqrt(8.0 * x + 1.0) - 1.0) * 0.5), col = x - row * (row + 1) / 2;
            dst[OL + row * 15 + col] = l[r];
            dst[OL + col * 15 + row] = l[r];
        }
    }
    if (lane < 15) dst[OA + lane] = a;
    __syncwarp();
}

// slot i (+) slot j (i the earlier in scan order, j the outer element) under the segmented operator, by one warp; the result replaces
// slot j (kRight) or slot i
template <bool kRight>
__device__ void seg_merge(double* slot, int i, int j, double* sc, int lane) {
    double* si = slot + i * ES;
    double* sj = slot + j * ES;
    const double fi = si[OF], fj = sj[OF];
    __syncwarp();
    if (fj == 0.0) {
        compose(sj, si, kRight ? sj : si, sc, lane);
    } else if (!kRight) {                                                 // a run ends at j: the result is slot j as it is
        for (int e = lane; e < ES; e += 32) si[e] = sj[e];
        __syncwarp();
    }
    if (lane == 0) (kRight ? sj : si)[OF] = (fi != 0.0 || fj != 0.0) ? 1.0 : 0.0;
    __syncwarp();
}

CPI_DEV void stage(const double* src, int m, double* slot) {
    for (int e = threadIdx.x; e < m * ES; e += 32 * W) slot[e] = src[e];
    __syncthreads();
}

// level l below the top: n elements at ws + pos, one aggregate per chunk to ws + pos_up
__global__ void __launch_bounds__(32 * W, 2) k_rts_scan_reduce(double* ws, int64_t n, int64_t pos, int64_t pos_up) {
    extern __shared__ double smem[];
    double* slot = smem;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double* sc = smem + (C + 1) * ES + warp * 225;
    const int64_t nch = (n + C - 1) / C;
    for (int64_t c = blockIdx.x; c < nch; c += gridDim.x) {
        const int m = (int)(n - c * C < C ? n - c * C : C);
        stage(ws + pos + c * C * ES, m, slot);
        for (int s = 1; s < m; s *= 2) {
            for (int k = warp; 2 * s * k + s < m; k += W) seg_merge<false>(slot, 2 * s * k, 2 * s * k + s, sc, lane);
            __syncthreads();
        }
        double* dst = ws + pos_up + c * ES;
        for (int e = tid; e < ES; e += 32 * W) dst[e] = slot[e];
        __syncthreads();
    }
}

// level l: inclusive scan of every chunk, seeded with the scanned aggregate of the chunk before (at ws + pos_up; the top level, at
// most C elements, is one chunk).  Level 0 writes back L and a, higher levels the whole element but its flag.
__global__ void __launch_bounds__(32 * W, 2) k_rts_scan_down(double* ws, int64_t n, int64_t pos, int64_t pos_up, int level0) {
    extern __shared__ double smem[];
    double* slot = smem;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double* sc = smem + (C + 1) * ES + warp * 225;
    const int64_t nch = (n + C - 1) / C;
    for (int64_t c = blockIdx.x; c < nch; c += gridDim.x) {
        const int m = (int)(n - c * C < C ? n - c * C : C);
        stage(ws + pos + c * C * ES, m, slot);
        if (c > 0) {
            const double* src = ws + pos_up + (c - 1) * ES;
            for (int e = tid; e < ES; e += 32 * W) slot[C * ES + e] = src[e];
            __syncthreads();
            if (warp == 0) seg_merge<true>(slot, C, 0, sc, lane);
            __syncthreads();
        }
        for (int d = 1; d < C; d *= 2) {                                  // up-sweep
            for (int k = (warp + 1) * 2 * d - 1; k < m; k += W * 2 * d) seg_merge<true>(slot, k - d, k, sc, lane);
            __syncthreads();
        }
        for (int d = C / 4; d >= 1; d /= 2) {                             // down-sweep
            for (int k = (warp + 1) * 2 * d - 1; k + d < m; k += W * 2 * d) seg_merge<true>(slot, k, k + d, sc, lane);
            __syncthreads();
        }
        double* dst = ws + pos + c * C * ES;
        for (int e = tid; e < m * ES; e += 32 * W) {
            const int k = e % ES;
            if (level0 ? k >= OL && k < OF : k != OF) dst[e] = slot[e];
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(EW * 32) k_rts_apply(int64_t n_runs, const int64_t* offs, int64_t uniform, int64_t n,
                                                       const double* states, const double* cov, const double* ws, double* states_out,
                                                       double* cov_out, double* cross_out) {
    __shared__ double smem[EW][2 * RP];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* G = smem[warp];
    double* P1 = G + RP;                          // Ps_{k+1}
    for (int64_t s = (int64_t)blockIdx.x * EW + warp; s < n; s += (int64_t)gridDim.x * EW) {
        int64_t last;
        const int64_t c = run_of(n_runs, offs, uniform, s, last);
        const double* sg = cov + s * 225;
        double* co = cov_out + s * 225;
        if (s == last) {                          // copied bit for bit
            for (int e = lane; e < 225; e += 32) co[e] = __ldg(sg + e);
            if (lane < CPI_STATE_DOUBLES) states_out[s * CPI_STATE_DOUBLES + lane] = __ldg(states + s * CPI_STATE_DOUBLES + lane);
            continue;
        }
        const double* el = ws + (n - 1 - s) * ES;
        for (int e = lane; e < 225; e += 32) co[e] = el[OL + (e % 15) * 15 + e / 15];
        if (lane == 0) {                          // xs_k = retract(x_k, delta_k)
            double x[16], d[15], xo[16];
#pragma unroll
            for (int k = 0; k < 16; k++) x[k] = __ldg(states + s * CPI_STATE_DOUBLES + k);
#pragma unroll
            for (int k = 0; k < 15; k++) d[k] = el[OA + k];
            retract_state(x, d, xo);
#pragma unroll
            for (int k = 0; k < 16; k++) states_out[s * CPI_STATE_DOUBLES + k] = xo[k];
        }
        if (cross_out) {                          // Xs_k = G_k Ps_{k+1}, column-major in transition k's slot
            const double* el1 = el - ES;          // keyframe s + 1
            for (int e = lane; e < 225; e += 32) {
                G[(e / 15) * 16 + e % 15] = el[OE + e];
                P1[(e / 15) * 16 + e % 15] = el1[OL + e];
            }
            __syncwarp();
            double* xo = cross_out + (s - c) * 225;
            for (int e = lane; e < 225; e += 32) {
                const int r = e % 15, q = e / 15;
                double v = 0.0;
#pragma unroll
                for (int m = 0; m < 15; m++) v = fma(G[r * 16 + m], P1[m * 16 + q], v);
                xo[e] = v;
            }
            __syncwarp();
        }
    }
}

// element counts of the scan's levels: level 0 has n, level l + 1 one per chunk of level l, up to the first of at most C
int levels_of(int64_t n, int64_t* count) {
    int l = 0;
    count[0] = n;
    while (count[l] > C) {
        count[l + 1] = (count[l] + C - 1) / C;
        l++;
    }
    return l;
}

}  // namespace

// K15: Rauch-Tung-Striebel smoothing of filter runs (DESIGN.md section 3o).  Run c holds keyframes o[c] .. o[c+1]-1 with the
// filter's posteriors (x_k, P_k); its transitions are stored from o[c] - c, transition k carrying K7's prediction (xb_{k+1},
// Pb_{k+1}) and cross C_k = P_k A_k^T from (x_k, P_k).  From the last keyframe (copied bit for bit) backwards:
//   G = C_k Pb^-1 (Pb = L L^T),  d = local(xb_{k+1}, xs_{k+1}),  xs_k = retract(x_k, G d),
//   Ps_k = P_k + G (Ps_{k+1} - Pb) G^T,  Xs_k = G Ps_{k+1}  (the smoothed (x_k, x_{k+1}) block)
// One warp per run, sequential over its keyframes; xs_{k+1} and Ps_{k+1} are carried in shared memory.  Lane i < 15 solves row i
// of G from row i of C_k with L (two per-lane triangular solves) while lane 15 forms d, then row i of T = G (Ps_{k+1} - Pb), row i
// of Xs_k and (G d)_i; after a sync it forms row i of Ps_k left of the diagonal and mirrors it, so Ps_k is exactly symmetric, while
// lane 15 retracts.  A Pb that is not SPD gives NaN from that keyframe back, in that run only.  No atomics: the same bits on every run.
__global__ void __launch_bounds__(EW * 32) k_rts_smooth(int64_t n_runs, const int64_t* offs, int64_t uniform, const double* states,
                                                       const double* cov, const double* pred_states, const double* pred_cov,
                                                       const double* cross, double* states_out, double* cov_out, double* cross_out) {
    __shared__ double smem[EW][5 * RP + 64];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t c = (int64_t)blockIdx.x * EW + warp;
    if (c >= n_runs) return;
    double* Pb = smem[warp];                      // Pb_{k+1}
    double* L = Pb + RP;                          // its Cholesky factor (lower triangle)
    double* G = L + RP;                           // C_k, then G row by row
    double* Ps = G + RP;                          // Ps_{k+1}, then Ps_k
    double* Pk = Ps + RP;                         // P_k
    double* XS = Pk + RP;                         // xs_{k+1}, then xs_k
    double* XK = XS + 16;                         // x_k
    double* XB = XK + 16;                         // xb_{k+1}
    double* GD = XB + 16;                         // G d
    const int64_t o0 = offs ? __ldg(offs + c) : c * uniform;
    const int64_t o1 = offs ? __ldg(offs + c + 1) : o0 + uniform;
    const int64_t last = o1 - 1, t0 = o0 - c;     // the run's last keyframe and its first transition
    {                                             // the last keyframe: copied, and carried
        const double* sg = cov + last * 225;
        double* co = cov_out + last * 225;
        for (int e = lane; e < 225; e += 32) {
            const double v = __ldg(sg + e);
            co[e] = v;
            Ps[(e % 15) * 16 + e / 15] = v;
        }
        if (lane < CPI_STATE_DOUBLES) {
            const double v = __ldg(states + last * CPI_STATE_DOUBLES + lane);
            states_out[last * CPI_STATE_DOUBLES + lane] = v;
            XS[lane] = v;
        }
    }
    for (int64_t s = last - 1; s >= o0; s--) {
        const int64_t t = t0 + (s - o0);
        const double* pg = pred_cov + t * 225;
        const double* cg = cross + t * 225;
        const double* sg = cov + s * 225;
        for (int e = lane; e < 225; e += 32) {    // column-major (r, c) -> row-major pitch 16
            const int r = e % 15, q = e / 15;
            const double p = __ldg(pg + e);
            Pb[r * 16 + q] = p;
            L[r * 16 + q] = p;
            G[r * 16 + q] = __ldg(cg + e);
            Pk[r * 16 + q] = __ldg(sg + e);
        }
        if (lane < CPI_STATE_DOUBLES) {
            XK[lane] = __ldg(states + s * CPI_STATE_DOUBLES + lane);
            XB[lane] = __ldg(pred_states + t * CPI_STATE_DOUBLES + lane);
        }
        __syncwarp();
        rts_gain(L, G, lane, [&] {                // d = local(xb_{k+1}, xs_{k+1}) in the spare column 15 of G
            double d[15];
            local15(XB, XS, d);
#pragma unroll
            for (int r = 0; r < 15; r++) G[r * 16 + 15] = d[r];
        });
        __syncwarp();
        if (lane < 15) {                          // row lane of T = G (Ps_{k+1} - Pb) into L (free after the solves), of Xs_k, and (G d)_lane
            const double* g = G + lane * 16;
            double gd = 0.0;
#pragma unroll
            for (int m = 0; m < 15; m++) gd = fma(g[m], G[m * 16 + 15], gd);
            GD[lane] = gd;
            double tr[15];
#pragma unroll
            for (int j = 0; j < 15; j++) tr[j] = 0.0;
#pragma unroll 1
            for (int m = 0; m < 15; m++) {
                const double gm = g[m];
#pragma unroll
                for (int j = 0; j < 15; j++) tr[j] = fma(gm, Ps[m * 16 + j] - Pb[m * 16 + j], tr[j]);
            }
#pragma unroll
            for (int j = 0; j < 15; j++) L[lane * 16 + j] = tr[j];
            if (cross_out) {                      // Xs_k(lane, j) = G(lane, :) Ps_{k+1}(:, j), column-major: coalesced over lanes
                double* xo = cross_out + t * 225;
#pragma unroll 1
                for (int j = 0; j < 15; j++) {
                    double x = 0.0;
#pragma unroll
                    for (int m = 0; m < 15; m++) x = fma(g[m], Ps[m * 16 + j], x);
                    xo[lane + 15 * j] = x;
                }
            }
        }
        __syncwarp();
        if (lane < 15) {                          // Ps_k(lane, j) = P_k(lane, j) + T(lane, :) G(j, :)^T, j <= lane, mirrored
            double tr[15];
#pragma unroll
            for (int m = 0; m < 15; m++) tr[m] = L[lane * 16 + m];
            for (int j = 0; j <= lane; j++) {
                double v = 0.0;
#pragma unroll
                for (int m = 0; m < 15; m++) v = fma(tr[m], G[j * 16 + m], v);
                v += Pk[lane * 16 + j];
                Ps[lane * 16 + j] = v;
                Ps[j * 16 + lane] = v;
            }
        } else if (lane == 15) {                  // xs_k = retract(x_k, G d)
            double xo[16];
            retract_state(XK, GD, xo);
            double* o = states_out + s * CPI_STATE_DOUBLES;
#pragma unroll
            for (int k = 0; k < 16; k++) { XS[k] = xo[k]; o[k] = xo[k]; }
        }
        __syncwarp();
        double* co = cov_out + s * 225;
        for (int e = lane; e < 225; e += 32) co[e] = Ps[(e % 15) * 16 + e / 15];
        __syncwarp();
    }
}

cudaError_t rts_smooth_launch(int64_t n_runs, const int64_t* offs, int64_t uniform, const double* states, const double* cov,
                              const double* pred_states, const double* pred_cov, const double* cross, double* states_out, double* cov_out,
                              double* cross_out, cudaStream_t st) {
    if (n_runs == 0) return cudaSuccess;
    const int64_t grid = (n_runs + EW - 1) / EW;
    k_rts_smooth<<<(unsigned)grid, EW * 32, 0, st>>>(n_runs, offs, uniform, states, cov, pred_states, pred_cov, cross, states_out,
                                                    cov_out, cross_out);
    return cudaGetLastError();
}

int64_t rts_scan_workspace_bytes(int64_t n_states) {
    int64_t count[64], elems = 0;
    const int top = levels_of(n_states, count);
    for (int l = 0; l <= top; l++) elems += count[l];
    return elems * ES * (int64_t)sizeof(double);
}

cudaError_t rts_scan_launch(int64_t n_runs, const int64_t* offs, int64_t uniform, int64_t n, const double* states, const double* cov,
                            const double* pred_states, const double* pred_cov, const double* cross, double* states_out, double* cov_out,
                            double* cross_out, void* workspace, int sms, cudaStream_t st, int* launches) {
    if (n_runs == 0) return cudaSuccess;
    cudaError_t e;
    auto wgrid = [&](int64_t items, int per, int64_t cap) { const int64_t g = (items + per - 1) / per; return (unsigned)(g < cap ? (g > 0 ? g : 1) : cap); };
    if (n > n_runs) {                             // a transition exists
        double* ws = (double*)workspace;
        if ((e = cudaFuncSetAttribute(k_rts_scan_reduce, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM)) != cudaSuccess) return e;
        if ((e = cudaFuncSetAttribute(k_rts_scan_down, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM)) != cudaSuccess) return e;
        k_rts_elements<<<wgrid(n, EW, 16 * (int64_t)sms), EW * 32, 0, st>>>(n_runs, offs, uniform, n, states, cov, pred_states, pred_cov,
                                                                             cross, ws);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        ++*launches;
        int64_t count[64], pos[64];
        const int top = levels_of(n, count);
        pos[0] = 0;
        for (int l = 0; l < top; l++) pos[l + 1] = pos[l] + count[l] * ES;
        for (int l = 0; l < top; l++) {
            k_rts_scan_reduce<<<wgrid(count[l], C, 2 * (int64_t)sms), 32 * W, SMEM, st>>>(ws, count[l], pos[l], pos[l + 1]);
            if ((e = cudaGetLastError()) != cudaSuccess) return e;
            ++*launches;
        }
        for (int l = top; l >= 0; l--) {
            k_rts_scan_down<<<wgrid(count[l], C, 2 * (int64_t)sms), 32 * W, SMEM, st>>>(ws, count[l], pos[l], l < top ? pos[l + 1] : 0,
                                                                                        l == 0);
            if ((e = cudaGetLastError()) != cudaSuccess) return e;
            ++*launches;
        }
    }
    k_rts_apply<<<wgrid(n, EW, 16 * (int64_t)sms), EW * 32, 0, st>>>(n_runs, offs, uniform, n, states, cov, (const double*)workspace,
                                                                      states_out, cov_out, cross_out);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    ++*launches;
    return cudaSuccess;
}

}  // namespace cpi
