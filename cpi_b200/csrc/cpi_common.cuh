// Shared device helpers for the CPI kernels (sm_90a).  All small-matrix code works on register arrays with
// compile-time indices so that nothing is spilled to local memory by dynamic indexing.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/cpi_b200.h"

namespace cpi {

#define CPI_DEV __device__ __forceinline__

// 3x3 blocks are ROW-major in registers: M[3*i+j] = M(i,j).  Records (global memory) are column-major like Eigen.

// x cross w.   Note  (-[w]x) c = c x w  (acts on a column)   and   r^T [w]x = (r x w)^T  (acts on a row).
template <class T> CPI_DEV void cross(const T* x, const T* w, T* o) {
    o[0] = x[1] * w[2] - x[2] * w[1];
    o[1] = x[2] * w[0] - x[0] * w[2];
    o[2] = x[0] * w[1] - x[1] * w[0];
}
// C = A * B
template <class T> CPI_DEV void mul33(const T* A, const T* B, T* C) {
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
// C = A^T * B
template <class T> CPI_DEV void mulT33(const T* A, const T* B, T* C) {
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) C[3 * i + j] = A[i] * B[j] + A[3 + i] * B[3 + j] + A[6 + i] * B[6 + j];
}
// o = A * v
template <class T> CPI_DEV void mv33(const T* A, const T* v, T* o) {
#pragma unroll
    for (int i = 0; i < 3; i++) o[i] = A[3 * i] * v[0] + A[3 * i + 1] * v[1] + A[3 * i + 2] * v[2];
}
// o = A^T * v
template <class T> CPI_DEV void mvT33(const T* A, const T* v, T* o) {
#pragma unroll
    for (int i = 0; i < 3; i++) o[i] = A[i] * v[0] + A[3 + i] * v[1] + A[6 + i] * v[2];
}

// index of (i,j) in a packed symmetric 3x3 [00 01 02 11 12 22]
__host__ __device__ constexpr int sym3(int i, int j) {
    return (i <= j) ? (i == 0 ? j : (i == 1 ? 2 + j : 5)) : (j == 0 ? i : (j == 1 ? 2 + i : 5));
}

// JPL quaternion helpers (utils/quat_ops.h), q = [x y z w]
CPI_DEV void quat_2_Rot(const double* q, double* R) {          // quat_ops.h:104-109
    const double s = 2.0 * q[3] * q[3] - 1.0, t = 2.0 * q[3];
    // (2 q4^2 - 1) I - 2 q4 [qv x] + 2 qv qv^T ;   [v x] = [[0,-v2,v1],[v2,0,-v0],[-v1,v0,0]]
    R[0] = s + 2.0 * q[0] * q[0];            R[1] = t * q[2] + 2.0 * q[0] * q[1];     R[2] = -t * q[1] + 2.0 * q[0] * q[2];
    R[3] = -t * q[2] + 2.0 * q[1] * q[0];    R[4] = s + 2.0 * q[1] * q[1];            R[5] = t * q[0] + 2.0 * q[1] * q[2];
    R[6] = t * q[1] + 2.0 * q[2] * q[0];     R[7] = -t * q[0] + 2.0 * q[2] * q[1];    R[8] = s + 2.0 * q[2] * q[2];
}

CPI_DEV void rot_2_quat(const double* R, double* q) {          // quat_ops.h:45-86 (R row-major here)
    const double r00 = R[0], r11 = R[4], r22 = R[8];
    const double T = r00 + r11 + r22;
    if (r00 >= T && r00 >= r11 && r00 >= r22) {
        q[0] = sqrt((1.0 + 2.0 * r00 - T) / 4.0);
        const double s = 1.0 / (4.0 * q[0]);
        q[1] = s * (R[1] + R[3]); q[2] = s * (R[2] + R[6]); q[3] = s * (R[5] - R[7]);
    } else if (r11 >= T && r11 >= r00 && r11 >= r22) {
        q[1] = sqrt((1.0 + 2.0 * r11 - T) / 4.0);
        const double s = 1.0 / (4.0 * q[1]);
        q[0] = s * (R[1] + R[3]); q[2] = s * (R[5] + R[7]); q[3] = s * (R[6] - R[2]);
    } else if (r22 >= T && r22 >= r00 && r22 >= r11) {
        q[2] = sqrt((1.0 + 2.0 * r22 - T) / 4.0);
        const double s = 1.0 / (4.0 * q[2]);
        q[0] = s * (R[2] + R[6]); q[1] = s * (R[5] + R[7]); q[3] = s * (R[1] - R[3]);
    } else {
        q[3] = sqrt((1.0 + T) / 4.0);
        const double s = 1.0 / (4.0 * q[3]);
        q[0] = s * (R[5] - R[7]); q[1] = s * (R[6] - R[2]); q[2] = s * (R[1] - R[3]);
    }
    if (q[3] < 0) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}

CPI_DEV void quat_multiply(const double* q, const double* p, double* o) {   // quat_ops.h:115-128
    double t[4];
    // Qm = [ q4 I - [qv x] , qv ; -qv^T , q4 ]
    t[0] = q[3] * p[0] + q[2] * p[1] - q[1] * p[2] + q[0] * p[3];
    t[1] = -q[2] * p[0] + q[3] * p[1] + q[0] * p[2] + q[1] * p[3];
    t[2] = q[1] * p[0] - q[0] * p[1] + q[3] * p[2] + q[2] * p[3];
    t[3] = -q[0] * p[0] - q[1] * p[1] - q[2] * p[2] + q[3] * p[3];
    if (t[3] < 0) { t[0] = -t[0]; t[1] = -t[1]; t[2] = -t[2]; t[3] = -t[3]; }
    const double n = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2] + t[3] * t[3]);
    o[0] = t[0] / n; o[1] = t[1] / n; o[2] = t[2] / n; o[3] = t[3] / n;
}

// JPLNavState::retract (gtsam/JPLNavState.cpp:37-71): o = x retracted by the tangent step d (15 doubles)
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
    if (isnan(nn)) { dq[0] = dq[1] = dq[2] = 0.0; dq[3] = 1.0; }                       // :53-55 (dtheta == 0 -> 0/0)
    const double q[4] = {x[0], x[1], x[2], x[3]};
    double qn[4];
    quat_multiply(dq, q, qn);
#pragma unroll
    for (int k = 0; k < 4; k++) o[k] = qn[k];
#pragma unroll
    for (int k = 0; k < 12; k++) o[4 + k] = x[4 + k] + d[3 + k];
}

CPI_DEV void Exp_so3(const double* w, double* R) {            // quat_ops.h:145-162
    const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
    const double th = sqrt(th2);
    if (th == 0) { R[0] = R[4] = R[8] = 1.0; R[1] = R[2] = R[3] = R[5] = R[6] = R[7] = 0.0; return; }
    double s, c; sincos(th, &s, &c);
    const double a = s / th, b = (1.0 - c) / (th * th);
    // I + a [w x] + b [w x]^2
    R[0] = 1.0 - b * (w[1] * w[1] + w[2] * w[2]); R[1] = -a * w[2] + b * w[0] * w[1];           R[2] = a * w[1] + b * w[0] * w[2];
    R[3] = a * w[2] + b * w[0] * w[1];            R[4] = 1.0 - b * (w[0] * w[0] + w[2] * w[2]); R[5] = -a * w[0] + b * w[1] * w[2];
    R[6] = -a * w[1] + b * w[0] * w[2];           R[7] = a * w[0] + b * w[1] * w[2];            R[8] = 1.0 - b * (w[0] * w[0] + w[1] * w[1]);
}

}  // namespace cpi
