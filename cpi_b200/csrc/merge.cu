// K5: merge consecutive model-1 records (cpi_merge_records, include/cpi_b200.h).
//
// The composition of two records and the move to the group's linearisation point are in record_merge.cuh.
//
// Mapping: one CTA of W warps per group.  The group's records are staged in fp64 in 2W shared-memory slots and reduced by a pairwise
// tree (one warp per merge, log2(2W) levels); a group longer than 2W is taken in chunks, each chunk's tree running over the running
// result in slot 0 followed by 2W - 1 new records.
// fp32 storage (dtype 32): records and lin are float in memory, every operation is fp64.
#include <cuda_runtime.h>
#include <stdint.h>

#include "cpi_common.cuh"
#include "cpi_kernels.h"
#include "record_merge.cuh"

namespace cpi {
namespace {

using namespace rec1;

template <class T, int W>
__global__ void __launch_bounds__(32 * W) k_merge_records(int64_t n_groups, const int64_t* __restrict__ offsets, int64_t uniform,
                                                          const T* __restrict__ rec, const T* __restrict__ lin, T* __restrict__ out) {
    constexpr int C = 2 * W;
    extern __shared__ double smem[];
    double* slot = smem;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double* sc = smem + C * RD + warp * SCR;
    const int64_t g = blockIdx.x;
    int64_t lo, hi;
    if (offsets) { lo = offsets[g]; hi = offsets[g + 1]; } else { lo = g * uniform; hi = lo + uniform; }
    T* o = out + g * (int64_t)RD;
    if (hi <= lo) {                                                       // empty group: the zero-step record
        for (int e = tid; e < RD; e += 32 * W)
            o[e] = (T)((e == CPI_REC_Q + 3 || e == CPI_REC_R || e == CPI_REC_R + 4 || e == CPI_REC_R + 8) ? 1.0 : 0.0);
        return;
    }
    int n = 0;                                                            // occupied slots
    for (int64_t next = lo; next < hi;) {
        const int take = (int)(hi - next < C - n ? hi - next : C - n);
        const T* src = rec + next * (int64_t)RD;
        for (int e = tid; e < take * RD; e += 32 * W) slot[n * RD + e] = (double)src[e];
        __syncthreads();
        for (int s = tid; s < take; s += 32 * W) {
            if (next + s == lo) continue;
            const T* l0 = lin + lo * (int64_t)CPI_LIN_DOUBLES;
            const T* lk = lin + (next + s) * (int64_t)CPI_LIN_DOUBLES;
            const double dbw[3] = {(double)l0[0] - (double)lk[0], (double)l0[1] - (double)lk[1], (double)l0[2] - (double)lk[2]};
            const double dba[3] = {(double)l0[3] - (double)lk[3], (double)l0[4] - (double)lk[4], (double)l0[5] - (double)lk[5]};
            if (dbw[0] != 0.0 || dbw[1] != 0.0 || dbw[2] != 0.0 || dba[0] != 0.0 || dba[1] != 0.0 || dba[2] != 0.0)
                relinearise(slot + (n + s) * RD, dbw, dba);
        }
        __syncthreads();
        n += take; next += take;
        for (int stride = 1; stride < n; stride *= 2) {                   // pairwise tree: slot a <- slot a (+) slot a + stride
            for (int m = warp; 2 * stride * m + stride < n; m += W)
                merge_pair<false>(slot + 2 * stride * m * RD, slot + (2 * stride * m + stride) * RD, sc, lane);
            __syncthreads();
        }
        n = 1;
    }
    for (int e = tid; e < RD; e += 32 * W) o[e] = (T)slot[e];
}

template <class T, int W>
cudaError_t launch_w(int64_t n_groups, const int64_t* offsets, int64_t uniform, const void* rec, const void* lin, void* out, cudaStream_t st) {
    const size_t smem = sizeof(double) * (size_t)(2 * W * RD + W * SCR);
    cudaError_t e = cudaFuncSetAttribute(k_merge_records<T, W>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    k_merge_records<T, W><<<(unsigned)n_groups, 32 * W, smem, st>>>(n_groups, offsets, uniform, (const T*)rec, (const T*)lin, (T*)out);
    return cudaGetLastError();
}

template <class T>
cudaError_t launch_t(int w, int64_t n_groups, const int64_t* offsets, int64_t uniform, const void* rec, const void* lin, void* out, cudaStream_t st) {
    switch (w) {
        case 1: return launch_w<T, 1>(n_groups, offsets, uniform, rec, lin, out, st);
        case 2: return launch_w<T, 2>(n_groups, offsets, uniform, rec, lin, out, st);
        case 4: return launch_w<T, 4>(n_groups, offsets, uniform, rec, lin, out, st);
        default: return launch_w<T, 8>(n_groups, offsets, uniform, rec, lin, out, st);
    }
}

}  // namespace

cudaError_t merge_launch(int dtype, int64_t n_groups, const int64_t* offsets, int64_t uniform, const void* records, const void* lin,
                         void* out, cudaStream_t st) {
    // warps per CTA: uniform groups get the smallest CTA whose 2W slots hold the whole group (pairs: one warp; 8 warps at most), ragged
    // groups 4 warps (8 slots; a longer group folds 7 more records per chunk).  The group lengths of device offsets are not read here.
    int w = 4;
    if (!offsets) w = uniform <= 2 ? 1 : uniform <= 4 ? 2 : uniform <= 8 ? 4 : 8;
    return dtype == 32 ? launch_t<float>(w, n_groups, offsets, uniform, records, lin, out, st)
                       : launch_t<double>(w, n_groups, offsets, uniform, records, lin, out, st);
}

}  // namespace cpi
