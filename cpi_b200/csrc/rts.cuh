// Pieces of the Rauch-Tung-Striebel smoother shared by K15 (update.cu: sequential, one warp per run) and the parallel-in-time
// smoother (rts_scan.cu): the retraction of the filter's states and the gain G = C Pb^-1.  Matrices live in shared memory,
// row-major with pitch 16.
#pragma once
#include "chol15.cuh"

namespace cpi {

// JPLNavState::retract: the arithmetic of k_retract (factor.cu), kept as a local copy so that k_retract's code is untouched
CPI_DEV void retract_state(const double* x, const double* d, double* o) {
    const double nrm = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    double s, c;
    sincos(nrm / 2.0, &s, &c);
    double dq[4] = {(s / nrm) * d[0], (s / nrm) * d[1], (s / nrm) * d[2], c};
    double nn = sqrt(dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2] + dq[3] * dq[3]);
#pragma unroll
    for (int k = 0; k < 4; k++) dq[k] /= nn;
    if (dq[3] < 0) { dq[0] = -dq[0]; dq[1] = -dq[1]; dq[2] = -dq[2]; dq[3] = -dq[3]; }
    nn = sqrt(dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2] + dq[3] * dq[3]);
    if (isnan(nn)) { dq[0] = dq[1] = dq[2] = 0.0; dq[3] = 1.0; }
    const double q[4] = {x[0], x[1], x[2], x[3]};
    double qn[4];
    quat_multiply(dq, q, qn);
#pragma unroll
    for (int k = 0; k < 4; k++) o[k] = qn[k];
#pragma unroll
    for (int k = 0; k < 12; k++) o[4 + k] = x[4 + k] + d[3 + k];
}

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

}  // namespace cpi
