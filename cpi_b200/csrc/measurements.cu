// K12: the linearisation of measurements on any state of many chains into the moved prior blocks the solver already reads
// (DESIGN.md section 3l).  Measurement i on state s_i: A = S H and b = S r at x_{s_i} (measurement.cuh), then
//   info = A^T A,   rhs' = -A^T b,   f' = b^T b  (= s, the whitened squared residual the robust losses read)
// in the convention of the state priors (cost f - 2 rhs^T xi + xi^T info xi).  Lane m of a warp linearises measurement base + m and
// stages A and b in shared memory; the warp then writes the 225 + 15 entries of each of its 32 measurements with coalesced stores.
// info(r, c) and info(c, r) are the same fma chain of commuted products, so info is exactly symmetric.  f is written before the
// branch on `info`, by the same instructions in the full and the f-only pass.  No atomics: the same bits on every run.
#include <algorithm>

#include "cpi_kernels.h"
#include "measurement.cuh"

namespace cpi {

constexpr int MWARPS = 2;                        // warps per CTA
constexpr int MP = 49;                           // A (45), b (3) per measurement, odd pitch: conflict-free staging

__global__ void __launch_bounds__(MWARPS * 32) k_meas_linearize(int64_t n, const int32_t* kind, const int64_t* state_idx, const double* states,
                                                               const double* z, const double* sqrt_info, const double* aux, double* info,
                                                               double* rhs, double* f) {
    __shared__ double smem[MWARPS][32 * MP];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t base = ((int64_t)blockIdx.x * MWARPS + warp) * 32;
    if (base >= n) return;
    const int64_t i = base + lane;
    double* st = smem[warp] + lane * MP;
    if (i < n) {
        double A[45], b[3];
        meas_linearize(__ldg(kind + i), states + __ldg(state_idx + i) * CPI_STATE_DOUBLES, z + i * 3, sqrt_info + i * 9, aux + i * 3, b, A);
        f[i] = fma(b[2], b[2], fma(b[1], b[1], b[0] * b[0]));
        if (info) {
#pragma unroll
            for (int k = 0; k < 45; k++) st[k] = A[k];
#pragma unroll
            for (int k = 0; k < 3; k++) st[45 + k] = b[k];
        }
    }
    if (!info) return;
    __syncwarp();
    const int m = (int)std::min<int64_t>(32, n - base);
    for (int j = 0; j < m; j++) {
        const double* a = smem[warp] + j * MP;
        double* o = info + (base + j) * 225;
        for (int t = lane; t < 225; t += 32) {
            const int r = t % 15, c = t / 15;
            o[t] = fma(a[30 + r], a[30 + c], fma(a[15 + r], a[15 + c], a[r] * a[c]));
        }
        if (lane < 15) rhs[(base + j) * 15 + lane] = -fma(a[30 + lane], a[47], fma(a[15 + lane], a[46], a[lane] * a[45]));
    }
}

cudaError_t measurements_linearize_launch(int64_t n, const int32_t* kind, const int64_t* state_idx, const double* states, const double* z,
                                          const double* sqrt_info, const double* aux, double* info, double* rhs, double* f, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const int64_t grid = (n + MWARPS * 32 - 1) / (MWARPS * 32);
    k_meas_linearize<<<(unsigned)grid, MWARPS * 32, 0, st>>>(n, kind, state_idx, states, z, sqrt_info, aux, info, rhs, f);
    return cudaGetLastError();
}

}  // namespace cpi
