// K6: inclusive scan of consecutive model-1 records within groups (cpi_scan_records, include/cpi_b200.h): out[i] = the record of
// records lo .. i of i's group, every record first moved to the linearisation point of record lo (the composition: record_merge.cuh).
//
// Mapping: a segmented reduce-then-scan over the flat record index, in chunks of C records, restarting at every group start.  An
// element is a record and a flag "a group starts here"; (fa, a) (+) (fb, b) = (fa | fb, fb ? b : a (+) b) is associative, so the
// groups of one call are one scan.  Level 0 is the records; level l + 1 holds one aggregate per chunk of level l (workspace), up to
// the first level of at most C elements (the top):
//   up    (k_scan_reduce, one launch per level below the top): each chunk reduced by a pairwise tree, slot a <- slot a (+) slot a + s;
//   top   (k_scan_down at the top level): one CTA scans it;
//   down  (k_scan_down, top - 1 .. 0): each chunk rescanned, its first element seeded with the scanned aggregate of the chunk before.
// A chunk's scan is a Brent-Kung up-sweep / down-sweep over C shared-memory slots (slot k <- slot k - d (+) slot k, then slot k + d <-
// slot k (+) slot k + d), one warp per merge.  Depth: about 3 log2(C) merges per level and log_C(n) levels.  Device offsets are not
// read on the host, so it launches the levels of a bound on the record count (device memory / record size; the uniform layout's
// exact count), and the kernels of levels the data does not reach return at once; a top level longer than C (never at the bound)
// is scanned chunk after chunk by its one CTA.
// fp32 storage (dtype 32): records and lin are float in memory, every operation is fp64; the workspace is fp64.
#include <cuda_runtime.h>
#include <stdint.h>

#include "cpi_common.cuh"
#include "cpi_kernels.h"
#include "record_merge.cuh"

namespace cpi {
namespace {

using namespace rec1;

constexpr int C = 32;                 // elements per chunk: shared-memory slots 0 .. C-1, slot C holds the carry
constexpr int W = 4;                  // warps per CTA (214 / 244 registers a thread, ~88 KB of shared memory: two CTAs per SM)
constexpr int ES = RD + 1;            // workspace element: an aggregate record and its group-start flag (1.0 or 0.0)
constexpr size_t SMEM = sizeof(double) * ((C + 1) * RD + W * SCR) + sizeof(int) * (C + 1);

struct ScanArgs {
    int64_t n_groups;
    const int64_t* offsets;           // device CSR, or nullptr for groups of `uniform` records
    int64_t uniform;
    const void* rec;
    const void* lin;
    void* out;
    double* ws;
    int levels;                       // levels above 0 the host launches; the top is at most this one
};

// Level l of the scan: n elements (l >= 1: at ws + pos), its aggregates at ws + pos_up, and the top level.
struct Level { int64_t n, pos, pos_up; int top; };
CPI_DEV Level level(int64_t n0, int l, int levels) {
    Level r{0, 0, 0, 0};
    int64_t n = n0, pos = 0;
    for (int k = 0;; k++) {
        if (k == l) { r.n = n; r.pos = pos; }
        if (k == l + 1) r.pos_up = pos;
        if (n <= C || k == levels) { r.top = k; return r; }
        if (k > 0) pos += n * ES;
        n = (n + C - 1) / C;
    }
}

// first record b0 and record count n0 of the flat range the groups cover
CPI_DEV void extent(const ScanArgs& a, int64_t& b0, int64_t& n0) {
    if (a.offsets) { b0 = a.offsets[0]; n0 = a.offsets[a.n_groups] - b0; } else { b0 = 0; n0 = a.n_groups * a.uniform; }
    if (n0 < 0) n0 = 0;
}

// first record of the group holding record f (b0 <= f < b0 + n0): the last g with offsets[g] <= f is f's group (empty groups before
// it share its offset).  Unvalidated device offsets cannot send it below b0 or above f.
CPI_DEV int64_t group_start(const ScanArgs& a, int64_t f) {
    if (!a.offsets) return f - f % a.uniform;
    int64_t lo = 0, hi = a.n_groups;
    while (hi - lo > 1) {
        const int64_t m = (lo + hi) / 2;
        if (a.offsets[m] <= f) lo = m; else hi = m;
    }
    const int64_t s = a.offsets[lo];
    return s <= f ? s : f;
}

// Stage elements first .. first + m - 1 of level l in slots 0 .. m-1 with their flags.  Level 0 elements are the input records, each
// moved to the linearisation point of its group's first record, as the merge does it.
template <class T>
__device__ void stage(const ScanArgs& a, int l, const Level& L, int64_t b0, int64_t first, int m, double* slot, int* fl) {
    const int tid = threadIdx.x;
    if (l == 0) {
        const T* src = (const T*)a.rec + (b0 + first) * (int64_t)RD;
        for (int e = tid; e < m * RD; e += 32 * W) slot[e] = (double)src[e];
        __syncthreads();
        for (int s = tid; s < m; s += 32 * W) {
            const int64_t f = b0 + first + s, lo = group_start(a, f);
            fl[s] = f == lo;
            if (f == lo) continue;
            const T* l0 = (const T*)a.lin + lo * (int64_t)CPI_LIN_DOUBLES;
            const T* lk = (const T*)a.lin + f * (int64_t)CPI_LIN_DOUBLES;
            const double dbw[3] = {(double)l0[0] - (double)lk[0], (double)l0[1] - (double)lk[1], (double)l0[2] - (double)lk[2]};
            const double dba[3] = {(double)l0[3] - (double)lk[3], (double)l0[4] - (double)lk[4], (double)l0[5] - (double)lk[5]};
            if (dbw[0] != 0.0 || dbw[1] != 0.0 || dbw[2] != 0.0 || dba[0] != 0.0 || dba[1] != 0.0 || dba[2] != 0.0)
                relinearise(slot + s * RD, dbw, dba);
        }
    } else {
        const double* src = a.ws + L.pos + first * ES;
        for (int e = tid; e < m * ES; e += 32 * W) {
            const int s = e / ES, k = e - s * ES;
            if (k < RD) slot[s * RD + k] = src[e]; else fl[s] = src[e] != 0.0;
        }
    }
    __syncthreads();
}

// slot i (+) slot j (i the earlier) under the segmented operator, by one warp; the result replaces slot j (kRight) or slot i
template <bool kRight>
__device__ void seg_merge(double* slot, int* fl, int i, int j, double* sc, int lane) {
    const int fi = fl[i], fj = fl[j];
    __syncwarp();
    if (!fj) {
        merge_pair<kRight>(slot + i * RD, slot + j * RD, sc, lane);
    } else if (!kRight) {                                                 // a group starts at j: the result is slot j as it is
        for (int e = lane; e < RD; e += 32) slot[i * RD + e] = slot[j * RD + e];
        __syncwarp();
    }
    if (lane == 0) fl[kRight ? j : i] = fi | fj;
    __syncwarp();
}

// level l < top: one aggregate per chunk into level l + 1
template <class T>
__global__ void __launch_bounds__(32 * W) k_scan_reduce(ScanArgs a, int l) {
    extern __shared__ double smem[];
    double* slot = smem;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double* sc = smem + (C + 1) * RD + warp * SCR;
    int* fl = (int*)(smem + (C + 1) * RD + W * SCR);
    int64_t b0, n0;
    extent(a, b0, n0);
    const Level L = level(n0, l, a.levels);
    if (l >= L.top) return;
    const int64_t nch = (L.n + C - 1) / C;
    for (int64_t c = blockIdx.x; c < nch; c += gridDim.x) {
        const int m = (int)(L.n - c * C < C ? L.n - c * C : C);
        stage<T>(a, l, L, b0, c * C, m, slot, fl);
        for (int s = 1; s < m; s *= 2) {
            for (int k = warp; 2 * s * k + s < m; k += W) seg_merge<false>(slot, fl, 2 * s * k, 2 * s * k + s, sc, lane);
            __syncthreads();
        }
        double* dst = a.ws + L.pos_up + c * ES;
        for (int e = tid; e < ES; e += 32 * W) dst[e] = e < RD ? slot[e] : (double)fl[0];
        __syncthreads();
    }
}

// level l <= top: inclusive scan of every chunk, seeded with the scanned aggregate of the chunk before (level l + 1); the top level is
// scanned by CTA 0 alone, each chunk seeded with the last element of the one before.  Level 0 writes out, higher levels themselves.
template <class T>
__global__ void __launch_bounds__(32 * W) k_scan_down(ScanArgs a, int l) {
    extern __shared__ double smem[];
    double* slot = smem;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double* sc = smem + (C + 1) * RD + warp * SCR;
    int* fl = (int*)(smem + (C + 1) * RD + W * SCR);
    int64_t b0, n0;
    extent(a, b0, n0);
    const Level L = level(n0, l, a.levels);
    const bool top = l == L.top;
    if (l > L.top || (top && blockIdx.x > 0)) return;
    const int64_t nch = (L.n + C - 1) / C;
    for (int64_t c = blockIdx.x; c < nch; c += top ? 1 : gridDim.x) {
        const int m = (int)(L.n - c * C < C ? L.n - c * C : C);
        stage<T>(a, l, L, b0, c * C, m, slot, fl);
        if (c > 0) {
            if (!top) {
                const double* src = a.ws + L.pos_up + (c - 1) * ES;
                for (int e = tid; e < RD; e += 32 * W) slot[C * RD + e] = src[e];
                if (tid == 0) fl[C] = src[RD] != 0.0;
                __syncthreads();
            }
            if (warp == 0) seg_merge<true>(slot, fl, C, 0, sc, lane);
            __syncthreads();
        }
        for (int d = 1; d < C; d *= 2) {                                  // up-sweep
            for (int k = (warp + 1) * 2 * d - 1; k < m; k += W * 2 * d) seg_merge<true>(slot, fl, k - d, k, sc, lane);
            __syncthreads();
        }
        for (int d = C / 4; d >= 1; d /= 2) {                             // down-sweep
            for (int k = (warp + 1) * 2 * d - 1; k + d < m; k += W * 2 * d) seg_merge<true>(slot, fl, k, k + d, sc, lane);
            __syncthreads();
        }
        if (l == 0) {
            T* dst = (T*)a.out + (b0 + c * C) * (int64_t)RD;
            for (int e = tid; e < m * RD; e += 32 * W) dst[e] = (T)slot[e];
        } else {
            double* dst = a.ws + L.pos + c * C * ES;
            for (int e = tid; e < m * ES; e += 32 * W) {
                const int s = e / ES, k = e - s * ES;
                if (k < RD) dst[e] = slot[s * RD + k];
            }
        }
        if (top) {                                                        // carry into the next chunk of the top level
            for (int e = tid; e < RD; e += 32 * W) slot[C * RD + e] = slot[(m - 1) * RD + e];
            if (tid == 0) fl[C] = fl[m - 1];
        }
        __syncthreads();
    }
}

// levels above 0 needed for n records
int levels_for(int64_t n) {
    int l = 0;
    for (; n > C; n = (n + C - 1) / C) l++;
    return l;
}

template <class T>
cudaError_t launch_t(const ScanArgs& a, int64_t n_bound, int sms, cudaStream_t st, int* launches) {
    cudaError_t e = cudaFuncSetAttribute(k_scan_reduce<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_scan_down<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM);
    if (e != cudaSuccess) return e;
    // CTAs for level l: its chunk count at the bound, at most two per SM (grid-stride beyond)
    auto grid = [&](int l) {
        int64_t n = n_bound;
        for (int k = 0; k <= l; k++) n = (n + C - 1) / C;
        return (unsigned)(n < 2 * (int64_t)sms ? (n > 0 ? n : 1) : 2 * sms);
    };
    for (int l = 0; l < a.levels; l++) {
        k_scan_reduce<T><<<grid(l), 32 * W, SMEM, st>>>(a, l);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        ++*launches;
    }
    for (int l = a.levels; l >= 0; l--) {
        k_scan_down<T><<<grid(l), 32 * W, SMEM, st>>>(a, l);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        ++*launches;
    }
    return cudaSuccess;
}

}  // namespace

int64_t scan_workspace_bytes(int64_t n_records) {
    int64_t elems = 0;
    for (int64_t n = n_records; n > C;) {
        n = (n + C - 1) / C;
        elems += n;
    }
    return elems > 0 ? elems * ES * (int64_t)sizeof(double) : 8;
}

cudaError_t scan_launch(int dtype, int64_t n_groups, const int64_t* offsets, int64_t uniform, int64_t n_bound, const void* records,
                        const void* lin, void* out, void* workspace, int sms, cudaStream_t st, int* launches) {
    ScanArgs a{n_groups, offsets, uniform, records, lin, out, (double*)workspace, levels_for(n_bound)};
    return dtype == 32 ? launch_t<float>(a, n_bound, sms, st, launches) : launch_t<double>(a, n_bound, sms, st, launches);
}

}  // namespace cpi
