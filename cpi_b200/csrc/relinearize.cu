// Re-preintegration of the windows whose state bias left the records' linearisation point (cpi_imu_records_relinearize,
// include/cpi_b200.h; DESIGN.md section 3i).  The kernels around the unchanged K1/K2 launch:
//   k_relin_select       one thread per factor: the selection rule, the mask, and per CTA the number of selected factors and
//                        of their sample entries
//   k_relin_scan_blocks  one CTA: exclusive prefixes of the per-CTA totals, and the grand totals the host reads
//   k_relin_compact      one thread per factor: the stable compaction (block scan + the CTA's prefix) into the selected factors'
//                        indices, compact CSR offsets and new linearisation points
//   k_relin_gather       one warp per selected window, grid-stride: its sample range into the compact, 16-byte aligned buffer
//   k_relin_scatter      one warp per selected window, grid-stride: the compact record and lin back into the factor's slots
// Integer sums only, no atomics: the same bits on every run.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "cpi_common.cuh"
#include "cpi_kernels.h"
#include "local15.cuh"

namespace cpi {

namespace {
constexpr int RELIN_TPB = 256;          // factors per CTA of the select and compact kernels
constexpr int RELIN_SCAN_TPB = 256;

struct Pair { long long sel, ent; };
struct PairSum { __device__ Pair operator()(const Pair& a, const Pair& b) const { return {a.sel + b.sel, a.ent + b.ent}; } };

int64_t align16(int64_t b) { return (b + 15) & ~(int64_t)15; }
int64_t relin_blocks(int64_t n) { return (n + RELIN_TPB - 1) / RELIN_TPB; }

// fp64 squared norm of a 3-vector, summed x, y, z in that order, without contraction (the rule's bits do not depend on the compiler)
CPI_DEV double norm2_3(double x, double y, double z) { return __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)); }

// the window's sample entries [*lo, *lo + return)
CPI_DEV int64_t window_range(int64_t k, const int64_t* offs, int64_t ent_uniform, int64_t* lo) {
    if (offs) { *lo = offs[k]; const int64_t c = offs[k + 1] - offs[k]; return c > 0 ? c : 0; }
    *lo = k * ent_uniform;
    return ent_uniform;
}
}  // namespace

// per-call view of the workspace: every region 16-byte aligned, the compact samples last so that the regions before them depend
// on the factor count only
RelinWorkspace relin_workspace(void* ws, int rd, int64_t n) {
    int64_t off[8], b = 0;
    const int64_t sizes[7] = {n * rd * 8, n * CPI_LIN_DOUBLES * 8, n * 8, (n + 1) * 8, n * 4, relin_blocks(n) * 16, (relin_blocks(n) + 1) * 16};
    for (int r = 0; r < 7; r++) { off[r] = b; b += align16(sizes[r]); }
    off[7] = b;
    char* p = (char*)ws;
    RelinWorkspace w;
    w.crec = (double*)(p + off[0]); w.clin = (double*)(p + off[1]); w.idx = (int64_t*)(p + off[2]); w.coff = (int64_t*)(p + off[3]);
    w.flag = (int32_t*)(p + off[4]); w.blk = (long long*)(p + off[5]); w.pre = (long long*)(p + off[6]); w.csamp = (double*)(p + off[7]);
    w.head_bytes = off[7];
    return w;
}

int64_t relin_total_offset(int64_t n) { return 2 * relin_blocks(n); }

int64_t relin_workspace_bytes(int rd, int64_t n, int64_t n_entries) {
    return relin_workspace(nullptr, rd, n).head_bytes + n_entries * CPI_SAMPLE_DOUBLES * 8;
}

__global__ void __launch_bounds__(RELIN_TPB) k_relin_select(int64_t n, int model, const double* __restrict__ states,
                                                            const int64_t* __restrict__ idx_i, const int64_t* __restrict__ offs,
                                                            int64_t ent_uniform, const double* __restrict__ lin, double tw2, double ta2,
                                                            double tt2, int32_t* __restrict__ flag, int32_t* __restrict__ mask,
                                                            long long* __restrict__ blk) {
    using Reduce = cub::BlockReduce<Pair, RELIN_TPB>;
    __shared__ typename Reduce::TempStorage tmp;
    const int64_t k = (int64_t)blockIdx.x * RELIN_TPB + threadIdx.x;
    Pair v{0, 0};
    if (k < n) {
        const double* x = states + (idx_i ? idx_i[k] : k) * CPI_STATE_DOUBLES;
        const double* l = lin + k * CPI_LIN_DOUBLES;
        const double dw2 = norm2_3(x[4] - l[0], x[5] - l[1], x[6] - l[2]);
        const double da2 = norm2_3(x[10] - l[3], x[11] - l[4], x[12] - l[5]);
        bool sel = dw2 > tw2 || da2 > ta2;
        bool nan = dw2 != dw2 || da2 != da2;
        if (model == 2) {                         // the rotation part of local(q_lin, q_i), as k_prior_at forms it
            double xl[CPI_STATE_DOUBLES] = {l[6], l[7], l[8], l[9]}, d[15];
            local15(xl, x, d);
            const double th2 = norm2_3(d[0], d[1], d[2]);
            sel = sel || th2 > tt2;
            nan = nan || th2 != th2;
        }
        sel = sel && !nan;                        // a NaN in what the rule reads leaves the factor unselected
        int64_t lo;
        v = {sel ? 1 : 0, sel ? window_range(k, offs, ent_uniform, &lo) : 0};
        flag[k] = sel;
        if (mask) mask[k] = sel;
    }
    const Pair t = Reduce(tmp).Reduce(v, PairSum());
    if (threadIdx.x == 0) { blk[2 * blockIdx.x] = t.sel; blk[2 * blockIdx.x + 1] = t.ent; }
}

// pre[b] = totals of CTAs 0 .. b-1 (pre[nb] = the grand totals the host reads); coff[n_selected] = the selected entries
__global__ void __launch_bounds__(RELIN_SCAN_TPB) k_relin_scan_blocks(int64_t nb, const long long* __restrict__ blk,
                                                                      long long* __restrict__ pre, int64_t* __restrict__ coff) {
    using Scan = cub::BlockScan<Pair, RELIN_SCAN_TPB>;
    __shared__ typename Scan::TempStorage tmp;
    const int64_t per = (nb + RELIN_SCAN_TPB - 1) / RELIN_SCAN_TPB;
    const int64_t lo = threadIdx.x * per, hi = lo + per < nb ? lo + per : nb;
    Pair s{0, 0};
    for (int64_t b = lo; b < hi; b++) { s.sel += blk[2 * b]; s.ent += blk[2 * b + 1]; }
    Pair run, total;
    Scan(tmp).ExclusiveScan(s, run, Pair{0, 0}, PairSum(), total);
    for (int64_t b = lo; b < hi; b++) {
        pre[2 * b] = run.sel; pre[2 * b + 1] = run.ent;
        run.sel += blk[2 * b]; run.ent += blk[2 * b + 1];
    }
    if (threadIdx.x == 0) { pre[2 * nb] = total.sel; pre[2 * nb + 1] = total.ent; coff[total.sel] = total.ent; }
}

__global__ void __launch_bounds__(RELIN_TPB) k_relin_compact(int64_t n, int model, const double* __restrict__ states,
                                                             const int64_t* __restrict__ idx_i, const int64_t* __restrict__ offs,
                                                             int64_t ent_uniform, const double* __restrict__ lin,
                                                             const int32_t* __restrict__ flag, const long long* __restrict__ pre,
                                                             int64_t* __restrict__ idx, int64_t* __restrict__ coff, double* __restrict__ clin) {
    using Scan = cub::BlockScan<Pair, RELIN_TPB>;
    __shared__ typename Scan::TempStorage tmp;
    const int64_t b = blockIdx.x;
    if (pre[2 * b + 2] == pre[2 * b]) return;     // nothing selected in this CTA (uniform across it)
    const int64_t k = b * RELIN_TPB + threadIdx.x;
    const bool sel = k < n && flag[k];
    int64_t lo = 0;
    Pair v{sel ? 1 : 0, sel ? window_range(k, offs, ent_uniform, &lo) : 0}, ex;
    Scan(tmp).ExclusiveScan(v, ex, Pair{0, 0}, PairSum());
    if (!sel) return;
    const int64_t j = pre[2 * b] + ex.sel;
    idx[j] = k;
    coff[j] = pre[2 * b + 1] + ex.ent;
    const double* x = states + (idx_i ? idx_i[k] : k) * CPI_STATE_DOUBLES;
    const double* l = lin + k * CPI_LIN_DOUBLES;
    double* o = clin + j * CPI_LIN_DOUBLES;
#pragma unroll
    for (int t = 0; t < 3; t++) { o[t] = x[4 + t]; o[3 + t] = x[10 + t]; o[10 + t] = l[10 + t]; }
#pragma unroll
    for (int t = 0; t < 4; t++) o[6 + t] = model == 2 ? x[t] : l[6 + t];
}

// count doubles from s to d, one warp; 16-byte vectors where both sides share the 16-byte phase
CPI_DEV void warp_copy(const double* __restrict__ s, double* __restrict__ d, int64_t count, int lane) {
    if ((((uintptr_t)s ^ (uintptr_t)d) & 15) == 0) {
        const int64_t head = ((uintptr_t)s & 15) ? (count > 0 ? 1 : 0) : 0;
        if (lane == 0 && head) d[0] = s[0];
        const int64_t nv = (count - head) / 2;
        const double2* s2 = (const double2*)(s + head);
        double2* d2 = (double2*)(d + head);
        for (int64_t t = lane; t < nv; t += 32) d2[t] = __ldg(s2 + t);
        const int64_t tail = head + 2 * nv;
        if (lane == 0 && tail < count) d[tail] = s[tail];
    } else {
        for (int64_t t = lane; t < count; t += 32) d[t] = __ldg(s + t);
    }
}

__global__ void __launch_bounds__(256) k_relin_gather(int64_t n_sel, const int64_t* __restrict__ idx, const int64_t* __restrict__ offs,
                                                      int64_t ent_uniform, const double* __restrict__ samples,
                                                      const int64_t* __restrict__ coff, double* __restrict__ csamp) {
    const int lane = threadIdx.x & 31;
    const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t j = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); j < n_sel; j += nw) {
        int64_t lo;
        window_range(idx[j], offs, ent_uniform, &lo);
        const int64_t d0 = coff[j];
        warp_copy(samples + lo * CPI_SAMPLE_DOUBLES, csamp + d0 * CPI_SAMPLE_DOUBLES, (coff[j + 1] - d0) * CPI_SAMPLE_DOUBLES, lane);
    }
}

__global__ void __launch_bounds__(256) k_relin_scatter(int64_t n_sel, int rd, const int64_t* __restrict__ idx, const double* __restrict__ crec,
                                                       const double* __restrict__ clin, double* __restrict__ records, double* __restrict__ lin) {
    const int lane = threadIdx.x & 31;
    const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t j = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); j < n_sel; j += nw) {
        const int64_t k = idx[j];
        warp_copy(crec + j * rd, records + k * rd, rd, lane);
        if (lane < CPI_LIN_DOUBLES) lin[k * CPI_LIN_DOUBLES + lane] = clin[j * CPI_LIN_DOUBLES + lane];
    }
}

cudaError_t relin_select_launch(int model, int64_t n, const double* states, const int64_t* idx_i, const int64_t* offs, int64_t ent_uniform,
                                const double* lin, double tw2, double ta2, double tt2, int32_t* mask, const RelinWorkspace& w, cudaStream_t st) {
    const int64_t nb = relin_blocks(n);
    k_relin_select<<<(unsigned)nb, RELIN_TPB, 0, st>>>(n, model, states, idx_i, offs, ent_uniform, lin, tw2, ta2, tt2, w.flag, mask, w.blk);
    k_relin_scan_blocks<<<1, RELIN_SCAN_TPB, 0, st>>>(nb, w.blk, w.pre, w.coff);
    k_relin_compact<<<(unsigned)nb, RELIN_TPB, 0, st>>>(n, model, states, idx_i, offs, ent_uniform, lin, w.flag, w.pre, w.idx, w.coff, w.clin);
    return cudaGetLastError();
}

cudaError_t relin_gather_launch(int64_t n_sel, const int64_t* offs, int64_t ent_uniform, const double* samples, const RelinWorkspace& w,
                                int sms, cudaStream_t st) {
    const int64_t want = (n_sel + 7) / 8, cap = (int64_t)sms * 8;
    k_relin_gather<<<(unsigned)(want < cap ? want : cap), 256, 0, st>>>(n_sel, w.idx, offs, ent_uniform, samples, w.coff, w.csamp);
    return cudaGetLastError();
}

cudaError_t relin_scatter_launch(int64_t n_sel, int rd, const RelinWorkspace& w, double* records, double* lin, int sms, cudaStream_t st) {
    const int64_t want = (n_sel + 7) / 8, cap = (int64_t)sms * 8;
    k_relin_scatter<<<(unsigned)(want < cap ? want : cap), 256, 0, st>>>(n_sel, rd, w.idx, w.crec, w.clin, records, lin);
    return cudaGetLastError();
}

}  // namespace cpi
