// extern "C" boundary of libcpi_b200.so (declared in include/cpi_b200.h).  Plain pointers and sizes only.
#include <atomic>
#include <chrono>
#include <cstdlib>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <mutex>
#include <optional>
#include <string>

#include "cpi_common.cuh"
#include "cpi_kernels.h"


namespace {

thread_local std::string g_err;
std::atomic<int64_t> g_launches{0};
}  // namespace
namespace cpi {
int capi_fail(int code, const char* fmt, ...) {      // the per-thread error slot, shared with the other translation units of the C ABI
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    g_err = buf;
    return code;
}
}  // namespace cpi
namespace {
constexpr auto fail = cpi::capi_fail;
#define CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail(CPI_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)

struct DevInfo { int sms = 0; int max_smem = 0; size_t mem = 0; bool ok = false; };
int device_info(DevInfo& d) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return fail(CPI_ENODEVICE, "no CUDA device: %s", cudaGetErrorString(e));
    static std::mutex mu;
    static DevInfo cache[64];
    std::lock_guard<std::mutex> lk(mu);
    if (dev < 64 && cache[dev].ok) { d = cache[dev]; return CPI_OK; }
    int major = 0, minor = 0;
    CU(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    CU(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
    if (major != 9 || minor != 0) return fail(CPI_ENODEVICE, "device %d is sm_%d%d, this library is built for sm_90a (H100) only", dev, major, minor);
    CU(cudaDeviceGetAttribute(&d.sms, cudaDevAttrMultiProcessorCount, dev));
    CU(cudaDeviceGetAttribute(&d.max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    size_t free_mem = 0;
    CU(cudaMemGetInfo(&free_mem, &d.mem));
    d.ok = true;
    if (dev < 64) cache[dev] = d;
    return CPI_OK;
}

// grow-only scratch buffers for the *_host entry points (per process; guarded by one mutex: host calls serialise)
struct Scratch {
    static constexpr int NBUF = 8, NSTREAM = 8;
    void* dev[NBUF] = {nullptr}; size_t dev_sz[NBUF] = {0};
    cudaStream_t stream = nullptr;            // copy-in / general stream
    cudaStream_t work[NSTREAM] = {nullptr};   // one per pipeline chunk (kernel + copy-out)
    cudaEvent_t ev[NSTREAM] = {nullptr};
    int device = -1;
};
std::mutex g_scratch_mu;
double g_host_submit_ms = 0.0, g_host_total_ms = 0.0;   // last cpi_preintegrate_batch_host call: time to enqueue everything / until drained
Scratch g_scratch;

int scratch_prepare() {
    int dev = 0;
    CU(cudaGetDevice(&dev));
    if (g_scratch.device != dev) {
        // buffers belong to the device they were allocated on; drop them if the caller switched device
        for (int i = 0; i < Scratch::NBUF; i++) { if (g_scratch.dev[i]) cudaFree(g_scratch.dev[i]); g_scratch.dev[i] = nullptr; g_scratch.dev_sz[i] = 0; }
        if (g_scratch.stream) { cudaStreamDestroy(g_scratch.stream); g_scratch.stream = nullptr; }
        for (int i = 0; i < Scratch::NSTREAM; i++) {
            if (g_scratch.work[i]) { cudaStreamDestroy(g_scratch.work[i]); g_scratch.work[i] = nullptr; }
            if (g_scratch.ev[i]) { cudaEventDestroy(g_scratch.ev[i]); g_scratch.ev[i] = nullptr; }
        }
        g_scratch.device = dev;
    }
    if (!g_scratch.stream) CU(cudaStreamCreateWithFlags(&g_scratch.stream, cudaStreamNonBlocking));
    for (int i = 0; i < Scratch::NSTREAM; i++) {
        if (!g_scratch.work[i]) CU(cudaStreamCreateWithFlags(&g_scratch.work[i], cudaStreamNonBlocking));
        if (!g_scratch.ev[i]) CU(cudaEventCreateWithFlags(&g_scratch.ev[i], cudaEventDisableTiming));
    }
    return CPI_OK;
}

// What every *_host entry point does around its kernels.  start() checks the device, takes the scratch lock and prepares the
// scratch; buf() hands out the next free grow-only scratch buffer; copy_stream() and work_stream() hand out the streams and record
// which ones the call used.  Those streams are drained on every exit, because async copies from / into the caller's buffers must
// not outlive the call: finish(rc) drains them and returns rc, or the first synchronisation error when rc is CPI_OK; on an early
// (error) return the destructor drains them.
class HostCall {
public:
    DevInfo dev;
    int start() {
        if (int rc = device_info(dev)) return rc;
        lk_ = std::unique_lock<std::mutex>(g_scratch_mu);
        return scratch_prepare();
    }
    int buf(size_t bytes, void** out) {
        if (next_ == Scratch::NBUF) return fail(CPI_ENOMEM, "a host call has at most %d scratch buffers", Scratch::NBUF);
        const int slot = next_++;
        if (bytes == 0) bytes = 8;
        if (g_scratch.dev_sz[slot] < bytes) {
            if (g_scratch.dev[slot]) CU(cudaFree(g_scratch.dev[slot]));
            g_scratch.dev[slot] = nullptr; g_scratch.dev_sz[slot] = 0;
            cudaError_t e = cudaMalloc(&g_scratch.dev[slot], bytes);
            if (e != cudaSuccess) return fail(CPI_ENOMEM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
            g_scratch.dev_sz[slot] = bytes;
        }
        *out = g_scratch.dev[slot];
        return CPI_OK;
    }
    // a buf() filled from the caller's host buffer on the copy stream
    int upload(const void* src, size_t bytes, void** out) {
        if (int rc = buf(bytes, out)) return rc;
        if (bytes > 0) CU(cudaMemcpyAsync(*out, src, bytes, cudaMemcpyHostToDevice, copy_stream()));
        return CPI_OK;
    }
    cudaStream_t copy_stream() { used_ |= 1u << Scratch::NSTREAM; return g_scratch.stream; }
    // pipeline work stream k (round robin), ordered after everything enqueued on the copy stream so far
    int work_stream(int64_t k, cudaStream_t* out) {
        const int si = (int)(k % Scratch::NSTREAM);
        used_ |= 1u << si | 1u << Scratch::NSTREAM;
        CU(cudaEventRecord(g_scratch.ev[si], g_scratch.stream));
        CU(cudaStreamWaitEvent(g_scratch.work[si], g_scratch.ev[si], 0));
        *out = g_scratch.work[si];
        return CPI_OK;
    }
    int finish(int rc) {
        for (int k = 0; k <= Scratch::NSTREAM; k++) {            // the work streams, then the copy stream
            if (!(used_ >> k & 1)) continue;
            cudaError_t e = cudaStreamSynchronize(k < Scratch::NSTREAM ? g_scratch.work[k] : g_scratch.stream);
            if (e != cudaSuccess && rc == CPI_OK) rc = fail(CPI_ECUDA, "cudaStreamSynchronize failed: %s", cudaGetErrorString(e));
        }
        used_ = 0;
        return rc;
    }
    ~HostCall() { finish(CPI_ECUDA); }      // an early return has already reported its error; a drain error does not replace it

private:
    std::unique_lock<std::mutex> lk_;
    int next_ = 0;
    unsigned used_ = 0;                     // bit k: work stream k; bit NSTREAM: the copy stream
};

// outputs (NULL ones skipped) must differ from every input and from each other
int check_aliasing(std::initializer_list<const void*> ins, std::initializer_list<const void*> outs) {
    for (const void* o : outs)
        for (const void* q : ins)
            if (o && o == q) return fail(CPI_EINVAL, "outputs must not overlap inputs");
    for (auto a = outs.begin(); a != outs.end(); ++a)
        for (auto b = a + 1; b != outs.end(); ++b)
            if (*a && *a == *b) return fail(CPI_EINVAL, "outputs must not overlap each other");
    return CPI_OK;
}

bool bytes_overlap(const void* a, size_t a_bytes, const void* b, size_t b_bytes) {
    return (const char*)a < (const char*)b + b_bytes && (const char*)b < (const char*)a + a_bytes;
}

// CPI_FLAG_DISCRETE produces model-1 records in fp64 only
int check_discrete(int model, int dtype, int flags) {
    if (!(flags & CPI_FLAG_DISCRETE)) return CPI_OK;
    if (model != 1) return fail(CPI_EINVAL, "CPI_FLAG_DISCRETE produces model-1 records: model must be 1 (got %d)", model);
    if (dtype != 64) return fail(CPI_EINVAL, "CPI_FLAG_DISCRETE is fp64 only: dtype must be 64 (got %d)", dtype);
    return CPI_OK;
}

int preintegrate_dev(int model, int dtype, int64_t n_windows, const int64_t* sample_offsets, int64_t ns_uniform,
                            const void* samples, const void* lin, const double* sigmas, int flags, void* out_records, void* stream, int wpb,
                            const void* init_records = nullptr) {
    if (model != 1 && model != 2) return fail(CPI_EINVAL, "model must be 1 or 2 (got %d)", model);
    if (dtype != 64 && dtype != 32) return fail(CPI_EINVAL, "dtype must be 64 or 32 (got %d)", dtype);
    if (int rc = check_discrete(model, dtype, flags)) return rc;
    if (n_windows < 0 || (!sample_offsets && ns_uniform < 0)) return fail(CPI_EINVAL, "negative count");
    if (n_windows >= 2147483647) return fail(CPI_EINVAL, "too many windows (%lld; at most 2^31 - 2 per call)", (long long)n_windows);
    if (n_windows == 0) return CPI_OK;
    if (!lin || !sigmas || !out_records) return fail(CPI_EINVAL, "null pointer argument");
    // device-resident CSR offsets cannot be inspected here: a NULL samples pointer is only rejected when the layout is uniform and
    // non-empty (an all-empty CSR shard legitimately has no sample buffer)
    if (!samples && !sample_offsets && ns_uniform > 0) return fail(CPI_EINVAL, "samples is null");
    if (model == 1 && (flags & CPI_FLAG_ANALYTIC_JACOBIANS)) flags &= ~CPI_FLAG_ANALYTIC_JACOBIANS;   // model 1 is always analytic
    DevInfo d;
    int rc = device_info(d);
    if (rc) return rc;
    cpi::PreintParams p;
    p.n_windows = n_windows; p.offsets = sample_offsets; p.ns_uniform = ns_uniform;
    p.samples = samples; p.lin = lin; p.out = out_records; p.init = init_records;
    if (init_records && !cpi::preint_tri_supported(model, flags) && (flags & (CPI_FLAG_DISCRETE | CPI_FLAG_IMU_AVG)) != CPI_FLAG_DISCRETE)
        return fail(CPI_EINVAL, "continuation is implemented for the default modes and the discrete mode only (no imu_avg, model 2 with "
                                "state_transition_jacobians)");
    p.q_w = sigmas[0] * sigmas[0]; p.q_wb = sigmas[1] * sigmas[1]; p.q_a = sigmas[2] * sigmas[2]; p.q_ab = sigmas[3] * sigmas[3];
    p.wpb = wpb;
    int launches = 0;
    CU(cpi::preint_launch(model, dtype, flags, p, d.sms, d.max_smem, (cudaStream_t)stream, &launches));
    g_launches += launches;
    return CPI_OK;
}

}  // namespace

extern "C" {

const char* cpi_last_error(void) { return g_err.c_str(); }
const char* cpi_version(void) { return "cpi_b200 0.3 (sm_90a)"; }
int cpi_record_doubles(int model) { return model == 1 ? CPI_REC_V1_DOUBLES : (model == 2 ? CPI_REC_V2_DOUBLES : CPI_EINVAL); }
int64_t cpi_launch_count(void) { return g_launches.load(); }

int cpi_device_count(void) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) return fail(CPI_ENODEVICE, "cudaGetDeviceCount: %s", cudaGetErrorString(e));
    int ok = 0;
    for (int i = 0; i < n; i++) {
        int major = 0, minor = 0;
        if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, i) == cudaSuccess &&
            cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, i) == cudaSuccess && major == 9 && minor == 0) ok++;
    }
    return ok;
}

int cpi_preintegrate_batch(int model, int dtype, int64_t n_windows, const int64_t* sample_offsets, int64_t ns_uniform,
                           const void* samples, const void* lin, const double* sigmas, int flags, void* out_records, void* stream) {
    return preintegrate_dev(model, dtype, n_windows, sample_offsets, ns_uniform, samples, lin, sigmas, flags, out_records, stream, 0);
}

int cpi_preintegrate_batch_continue(int model, int dtype, int64_t n_windows, const int64_t* sample_offsets, int64_t ns_uniform,
                                    const void* samples, const void* lin, const double* sigmas, int flags, void* records, void* stream) {
    return preintegrate_dev(model, dtype, n_windows, sample_offsets, ns_uniform, samples, lin, sigmas, flags, records, stream, 0, records);
}

int64_t cpi_imu_records_relinearize_workspace(int model, int64_t n_factors, int64_t n_entries) {
    if (model != 1 && model != 2) return fail(CPI_EINVAL, "model must be 1 or 2 (got %d)", model);
    if (n_factors < 0 || n_entries < 0) return fail(CPI_EINVAL, "negative count");
    if (n_factors >= 2147483647 || n_entries > ((int64_t)1 << 56)) return fail(CPI_EINVAL, "count out of range");
    return cpi::relin_workspace_bytes(cpi_record_doubles(model), n_factors, n_entries);
}

int cpi_imu_records_relinearize(int model, int64_t n_factors, const double* states, const int64_t* idx_i, const int64_t* sample_offsets,
                                int64_t ns_uniform, const double* samples, const double* sigmas, int flags, double tol_bw, double tol_ba,
                                double tol_theta, double* lin, double* records, int32_t* relinearized, int64_t* n_relinearized,
                                void* workspace, void* stream) {
    if (n_relinearized) *n_relinearized = 0;
    if (model != 1 && model != 2) return fail(CPI_EINVAL, "model must be 1 or 2 (got %d)", model);
    if (int rc = check_discrete(model, 64, flags)) return rc;
    if (n_factors < 0 || (!sample_offsets && ns_uniform < 0)) return fail(CPI_EINVAL, "negative count");
    if (n_factors >= 2147483647) return fail(CPI_EINVAL, "too many factors (%lld; at most 2^31 - 2 per call)", (long long)n_factors);
    const double tols[3] = {tol_bw, tol_ba, tol_theta};
    const char* names[3] = {"tol_bw", "tol_ba", "tol_theta"};
    for (int t = 0; t < 3; t++)
        if (!(tols[t] >= 0.0)) return fail(CPI_EINVAL, "%s must be >= 0 (+inf disables the test; got %g)", names[t], tols[t]);
    if (n_factors == 0) return CPI_OK;
    if (!states || !lin || !records || !sigmas) return fail(CPI_EINVAL, "null pointer argument (states / lin / records / sigmas)");
    if (!workspace) return fail(CPI_EINVAL, "null pointer argument (workspace: cpi_imu_records_relinearize_workspace bytes)");
    if ((uintptr_t)workspace & 15) return fail(CPI_EINVAL, "workspace must be 16-byte aligned");
    const int64_t ent_uniform = ns_uniform + ((flags & CPI_FLAG_IMU_AVG) ? 1 : 0);
    if (!samples && !sample_offsets && ent_uniform > 0) return fail(CPI_EINVAL, "samples is null");
    DevInfo d;
    int rc = device_info(d);
    if (rc) return rc;
    const int rd = cpi_record_doubles(model);
    cudaStream_t st = (cudaStream_t)stream;
    const cpi::RelinWorkspace w = cpi::relin_workspace(workspace, rd, n_factors);
    CU(cpi::relin_select_launch(model, n_factors, states, idx_i, sample_offsets, ent_uniform, lin, tol_bw * tol_bw, tol_ba * tol_ba,
                                tol_theta * tol_theta, relinearized, w, st));
    g_launches += 3;
    // the call's one host synchronisation: the re-preintegration's grid depends on the count, and so does the caller's next step
    long long tot[2] = {0, 0};
    CU(cudaMemcpyAsync(tot, w.pre + cpi::relin_total_offset(n_factors), sizeof tot, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (n_relinearized) *n_relinearized = tot[0];
    if (tot[0] == 0) return CPI_OK;
    CU(cpi::relin_gather_launch(tot[0], sample_offsets, ent_uniform, samples, w, d.sms, st));
    g_launches += 1;
    rc = preintegrate_dev(model, 64, tot[0], w.coff, 0, w.csamp, w.clin, sigmas, flags, w.crec, stream, 0);
    if (rc) return rc;
    CU(cpi::relin_scatter_launch(tot[0], rd, w, records, lin, d.sms, st));
    g_launches += 1;
    return CPI_OK;
}

int cpi_preintegrate_batch_host(int model, int dtype, int64_t n_windows, const int64_t* sample_offsets, int64_t ns_uniform,
                                const void* samples, const void* lin, const double* sigmas, int flags, void* out_records) {
    if (model != 1 && model != 2) return fail(CPI_EINVAL, "model must be 1 or 2 (got %d)", model);
    if (dtype != 64 && dtype != 32) return fail(CPI_EINVAL, "dtype must be 64 or 32 (got %d)", dtype);
    if (int rc = check_discrete(model, dtype, flags)) return rc;
    if (n_windows < 0) return fail(CPI_EINVAL, "negative count");
    if (n_windows == 0) return CPI_OK;
    if (!lin || !sigmas || !out_records) return fail(CPI_EINVAL, "null pointer argument");
    const int avg = (flags & CPI_FLAG_IMU_AVG) ? 1 : 0;
    const int64_t ent_w = ns_uniform + avg;
    const int64_t entries = sample_offsets ? sample_offsets[n_windows] : n_windows * ent_w;
    if (entries > 0 && !samples) return fail(CPI_EINVAL, "samples is null");
    if (sample_offsets) {                       // the host copy of the CSR layout can be validated before anything reaches the device
        if (sample_offsets[0] < 0) return fail(CPI_EINVAL, "sample_offsets[0] is negative");
        for (int64_t w = 0; w < n_windows; w++)
            if (sample_offsets[w + 1] < sample_offsets[w])     // an empty window is legal (also with imu_avg: it simply has no step)
                return fail(CPI_EINVAL, "sample_offsets must be non-decreasing (window %lld)", (long long)w);
    } else if (ns_uniform < 0) return fail(CPI_EINVAL, "negative count");
    const int rd = cpi_record_doubles(model);
    const size_t es = dtype == 32 ? 4 : 8;
    HostCall h;
    int rc = h.start();
    if (rc) return rc;
    const DevInfo& d = h.dev;
    void *d_s, *d_l, *d_o, *d_off = nullptr;
    if ((rc = h.buf((size_t)entries * CPI_SAMPLE_DOUBLES * es + 16, &d_s))) return rc;
    if ((rc = h.buf((size_t)n_windows * CPI_LIN_DOUBLES * es, &d_l))) return rc;
    if ((rc = h.buf((size_t)n_windows * rd * es, &d_o))) return rc;
    if (sample_offsets && (rc = h.buf((size_t)(n_windows + 1) * 8, &d_off))) return rc;

    // Chunked pipeline: H2D of chunk k+1 runs under the kernel of chunk k, D2H of chunk k under the kernel of chunk k+1.  The
    // default kernels are one-warp CTAs, so chunk kernels of different streams co-reside on the SMs and a batch can be cut into
    // many small chunks.  The lane-per-window kernels (imu_avg / analytic modes) are launched with the windows-per-block the WHOLE
    // batch would use, so that a chunk occupies only its share of the SMs.
    //
    // Wavefront schedule (uniform layout, fp64, default modes).  A window is a chain of ns DEPENDENT samples (a few microseconds each,
    // whatever the occupancy), so a chunk that travels whole finishes ~ns sample latencies after it arrived, however small it is: for
    // 200-sample windows a sizeable fraction of the PCIe time of the whole 10k-window batch.  Instead the batch
    // is cut into G window groups x S sample segments, and the (group, segment) tiles are sent along ANTI-DIAGONALS: tile (g, s) is a
    // strided copy (cudaMemcpy2DAsync: rows = windows of the group, row = samples [s ns/S, (s+1) ns/S)) followed, on the group's stream,
    // by a CONTINUATION kernel over the group (cpi_preintegrate_batch_continue).  Every group's chain then runs WHILE its samples
    // arrive, S other groups keep the SMs busy in between, groups finish (and copy out) one after the other, and what is left behind
    // the last byte is one segment of one group + that group's D2H.  fp64 only: a float record would round the fp64-accumulated
    // covariance state at every segment.
    const size_t in_bytes = (size_t)entries * CPI_SAMPLE_DOUBLES * es;
    const int cap = cpi::preint_cap(model, dtype, flags, d.sms);     // windows per CTA of the kernel preint_launch will select
    const bool small_ctas = cap <= 16;
    const bool big = in_bytes >= ((size_t)16 << 20) && n_windows >= 8 * (int64_t)d.sms;
    int nchunk = 1;
    if (big) {
        nchunk = small_ctas ? (int)(in_bytes >> 23) : 4;             // ~8 MB of samples per chunk
        if (nchunk < 4) nchunk = 4;
        if (nchunk > 16) nchunk = 16;
    }
    if (const char* e = getenv("CPI_B200_HOST_CHUNKS")) { int v = atoi(e); if (v >= 1 && v <= 64) nchunk = v; }   // A/B measurements
    int64_t need = (n_windows + d.sms - 1) / d.sms;
    const int wpb = (int)(need < cap ? (need < 1 ? 1 : need) : cap);
    const int64_t blocks = (n_windows + wpb - 1) / wpb;
    // wavefront geometry: the first wave_H % of the windows travel as whole-window chunks, the rest as G groups x S segments.
    // Defaults (tools/host_pipeline_probe.py compares geometries): every copy costs a few microseconds of dead
    // time on the copy engine, so few large tiles beat a fine wavefront -- ONE group of 4 segments, sized so that its transfer lasts
    // about as long as its sample chain (ns x ~4.6 us incl. the per-segment record reload, x ~50 GB/s of PCIe; model 2 chains are
    // ~1.5x longer), behind whole-window chunks for everything before it.
    int wave_G = 0, wave_S = 0, wave_H = 0;
    if (big) {
        wave_G = 1;
        wave_S = (int)(ns_uniform / 8 < 4 ? ns_uniform / 8 : 4);
        const double tail_bytes = (double)ns_uniform * (model == 1 ? 231e3 : 344e3);
        const double frac = tail_bytes / (double)in_bytes;
        wave_H = frac >= 1.0 ? 0 : (int)(100.0 * (1.0 - frac));
        if (wave_H > 95) wave_H = 95;
    }
    if (const char* e = getenv("CPI_B200_HOST_WAVE")) {              // "G,S[,H]": A/B measurements and tests ("0,0" = whole-window chunks only)
        int a_ = 0, b_ = 0, c_ = 0;
        const int nf = sscanf(e, "%d,%d,%d", &a_, &b_, &c_);
        if (nf >= 2 && a_ >= 0 && a_ <= 256 && b_ >= 0 && b_ <= 64 && c_ >= 0 && c_ < 100) { wave_G = a_; wave_S = b_; wave_H = nf == 3 ? c_ : 0; }
    }
    const bool wave = dtype == 64 && !sample_offsets && !avg && small_ctas && cpi::preint_tri_supported(model, flags) &&
                      wave_G >= 1 && wave_S >= 2 && ns_uniform >= 2 * (int64_t)wave_S;
    const int64_t head_blocks = wave ? blocks * wave_H / 100 : blocks;
    const int64_t head_hi = wave ? head_blocks * wpb : n_windows;    // windows [0, head_hi) travel whole, [head_hi, n) as the wavefront
    if (wave && head_blocks > 0) { nchunk = (int)((int64_t)nchunk * wave_H / 100); if (nchunk < 1) nchunk = 1; }
    const int64_t blocks_per_chunk = (head_blocks + nchunk - 1) / nchunk > 0 ? (head_blocks + nchunk - 1) / nchunk : 1;
    const auto t_start = std::chrono::steady_clock::now();
    int used = 0;                                                    // streams handed out so far (round robin)
    cudaStream_t s_in = h.copy_stream();
    rc = [&]() -> int {
        if (sample_offsets) CU(cudaMemcpyAsync(d_off, sample_offsets, (size_t)(n_windows + 1) * 8, cudaMemcpyHostToDevice, s_in));
        for (int k = 0; k < nchunk; k++) {
            const int64_t lo = (int64_t)k * blocks_per_chunk * wpb;
            if (lo >= head_hi) break;
            const int64_t hi = (lo + blocks_per_chunk * wpb < head_hi) ? lo + blocks_per_chunk * wpb : head_hi;
            used = k + 1;
            const int64_t e_lo = sample_offsets ? sample_offsets[lo] : lo * ent_w, e_hi = sample_offsets ? sample_offsets[hi] : hi * ent_w;
            CU(cudaMemcpyAsync((char*)d_l + (size_t)lo * CPI_LIN_DOUBLES * es, (const char*)lin + (size_t)lo * CPI_LIN_DOUBLES * es,
                               (size_t)(hi - lo) * CPI_LIN_DOUBLES * es, cudaMemcpyHostToDevice, s_in));
            if (e_hi > e_lo)
                CU(cudaMemcpyAsync((char*)d_s + (size_t)e_lo * CPI_SAMPLE_DOUBLES * es, (const char*)samples + (size_t)e_lo * CPI_SAMPLE_DOUBLES * es,
                                   (size_t)(e_hi - e_lo) * CPI_SAMPLE_DOUBLES * es, cudaMemcpyHostToDevice, s_in));
            cudaStream_t sk = nullptr;
            if (int r = h.work_stream(k, &sk)) return r;
            // offsets are absolute entry indices, so CSR chunks keep the global sample base; uniform chunks shift it
            const void* s_base = sample_offsets ? d_s : (const void*)((const char*)d_s + (size_t)e_lo * CPI_SAMPLE_DOUBLES * es);
            if (int r = preintegrate_dev(model, dtype, hi - lo, sample_offsets ? (const int64_t*)d_off + lo : nullptr, ns_uniform, s_base,
                                         (const char*)d_l + (size_t)lo * CPI_LIN_DOUBLES * es, sigmas, flags, (char*)d_o + (size_t)lo * rd * es, sk, wpb))
                return r;
            CU(cudaMemcpyAsync((char*)out_records + (size_t)lo * rd * es, (const char*)d_o + (size_t)lo * rd * es, (size_t)(hi - lo) * rd * es,
                               cudaMemcpyDeviceToHost, sk));
        }
        if (wave && head_hi < n_windows) {
            const size_t sb = (size_t)CPI_SAMPLE_DOUBLES * es;            // bytes per sample
            const int64_t wblocks = blocks - head_blocks;
            const int64_t bpg = (wblocks + wave_G - 1) / wave_G;          // blocks per group
            const int64_t G = (wblocks + bpg - 1) / bpg;
            const int64_t seg_len = (ns_uniform + wave_S - 1) / wave_S;
            const int64_t S = (ns_uniform + seg_len - 1) / seg_len;
            for (int64_t t = 0; t < G + S - 1; t++) {
                for (int64_t g = t - S + 1 > 0 ? t - S + 1 : 0; g <= t && g < G; g++) {      // oldest group (latest segment) first
                    const int64_t sidx = t - g, s0 = sidx * seg_len;
                    const int64_t len = s0 + seg_len <= ns_uniform ? seg_len : ns_uniform - s0;
                    const int64_t lo = head_hi + g * bpg * wpb, hi = (lo + bpg * wpb < n_windows) ? lo + bpg * wpb : n_windows, ng = hi - lo;
                    char* d_lg = (char*)d_l + (size_t)lo * CPI_LIN_DOUBLES * es;
                    char* d_og = (char*)d_o + (size_t)lo * rd * es;
                    if (sidx == 0)
                        CU(cudaMemcpyAsync(d_lg, (const char*)lin + (size_t)lo * CPI_LIN_DOUBLES * es, (size_t)ng * CPI_LIN_DOUBLES * es, cudaMemcpyHostToDevice, s_in));
                    // the tiles of a group are compact ([window][len]) and together fill the group's share of the device sample buffer
                    char* d_seg = (char*)d_s + ((size_t)lo * ns_uniform + (size_t)ng * s0) * sb;
                    CU(cudaMemcpy2DAsync(d_seg, (size_t)len * sb, (const char*)samples + ((size_t)lo * ns_uniform + (size_t)s0) * sb, (size_t)ns_uniform * sb,
                                         (size_t)len * sb, (size_t)ng, cudaMemcpyHostToDevice, s_in));
                    cudaStream_t sk = nullptr;
                    if (int r = h.work_stream(used + g, &sk)) return r;
                    if (int r = preintegrate_dev(model, dtype, ng, nullptr, len, d_seg, d_lg, sigmas, flags, d_og, sk, wpb, sidx > 0 ? d_og : nullptr))
                        return r;
                    if (sidx == S - 1)
                        CU(cudaMemcpyAsync((char*)out_records + (size_t)lo * rd * es, d_og, (size_t)ng * rd * es, cudaMemcpyDeviceToHost, sk));
                }
            }
        }
        return CPI_OK;
    }();
    g_host_submit_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_start).count();
    rc = h.finish(rc);
    g_host_total_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_start).count();
    return rc;
}

int cpi_host_last_timing(double* submit_ms, double* total_ms) {
    if (submit_ms) *submit_ms = g_host_submit_ms;
    if (total_ms) *total_ms = g_host_total_ms;
    return CPI_OK;
}

int cpi_host_register(void* ptr, size_t bytes) {
    if (!ptr || bytes == 0) return fail(CPI_EINVAL, "null pointer argument");
    CU(cudaHostRegister(ptr, bytes, cudaHostRegisterDefault));
    return CPI_OK;
}
int cpi_host_unregister(void* ptr) {
    if (!ptr) return fail(CPI_EINVAL, "null pointer argument");
    CU(cudaHostUnregister(ptr));
    return CPI_OK;
}

int cpi_imu_factor_eval_batch(int model, int64_t n_factors, const double* states, const int64_t* idx_i, const int64_t* idx_j,
                              const double* records, const double* lin, double* e, double* H1, double* H2, void* stream) {
    if (model != 1 && model != 2) return fail(CPI_EINVAL, "model must be 1 or 2 (got %d)", model);
    if (n_factors < 0) return fail(CPI_EINVAL, "negative count");
    if (n_factors == 0) return CPI_OK;
    if (!states || !records || !lin || !e) return fail(CPI_EINVAL, "null pointer argument");
    if ((idx_i == nullptr) != (idx_j == nullptr)) return fail(CPI_EINVAL, "idx_i and idx_j must both be given or both be null");
    DevInfo d;
    int rc = device_info(d);
    if (rc) return rc;
    cpi::FactorParams p{n_factors, states, idx_i, idx_j, records, lin, e, H1, H2};
    CU(cpi::factor_launch(model, p, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int cpi_imu_factor_eval_batch_host(int model, int64_t n_factors, int64_t n_states, const double* states, const int64_t* idx_i,
                                   const int64_t* idx_j, const double* records, const double* lin, double* e, double* H1, double* H2) {
    if (model != 1 && model != 2) return fail(CPI_EINVAL, "model must be 1 or 2 (got %d)", model);
    if (n_factors < 0 || n_states < 0) return fail(CPI_EINVAL, "negative count");
    if (n_factors == 0) return CPI_OK;
    if (!states || !records || !lin || !e) return fail(CPI_EINVAL, "null pointer argument");
    if (!idx_i && n_states < n_factors + 1) return fail(CPI_EINVAL, "chain indexing needs n_states >= n_factors + 1");
    if ((idx_i == nullptr) != (idx_j == nullptr)) return fail(CPI_EINVAL, "idx_i and idx_j must both be given or both be null");
    if (idx_i)
        for (int64_t f = 0; f < n_factors; f++)
            if (idx_i[f] < 0 || idx_i[f] >= n_states || idx_j[f] < 0 || idx_j[f] >= n_states)
                return fail(CPI_EINVAL, "factor %lld: state index out of range [0, %lld)", (long long)f, (long long)n_states);
    const int rd = cpi_record_doubles(model);
    HostCall h;
    int rc = h.start();
    if (rc) return rc;
    void *d_x, *d_r, *d_l, *d_e, *d_h1 = nullptr, *d_h2 = nullptr, *d_i = nullptr, *d_j = nullptr;
    if (idx_i && (rc = h.upload(idx_i, (size_t)n_factors * 8, &d_i))) return rc;
    if (idx_i && (rc = h.upload(idx_j, (size_t)n_factors * 8, &d_j))) return rc;
    if ((rc = h.upload(states, (size_t)n_states * CPI_STATE_DOUBLES * 8, &d_x))) return rc;
    if ((rc = h.upload(lin, (size_t)n_factors * CPI_LIN_DOUBLES * 8, &d_l))) return rc;
    if ((rc = h.upload(records, (size_t)n_factors * rd * 8, &d_r))) return rc;
    if ((rc = h.buf((size_t)n_factors * 15 * 8, &d_e))) return rc;
    if (H1 && (rc = h.buf((size_t)n_factors * 225 * 8, &d_h1))) return rc;
    if (H2 && (rc = h.buf((size_t)n_factors * 225 * 8, &d_h2))) return rc;
    cudaStream_t st = h.copy_stream();
    rc = cpi_imu_factor_eval_batch(model, n_factors, (const double*)d_x, (const int64_t*)d_i, (const int64_t*)d_j, (const double*)d_r,
                                   (const double*)d_l, (double*)d_e, (double*)d_h1, (double*)d_h2, st);
    if (rc) return rc;
    CU(cudaMemcpyAsync(e, d_e, (size_t)n_factors * 15 * 8, cudaMemcpyDeviceToHost, st));
    if (H1) CU(cudaMemcpyAsync(H1, d_h1, (size_t)n_factors * 225 * 8, cudaMemcpyDeviceToHost, st));
    if (H2) CU(cudaMemcpyAsync(H2, d_h2, (size_t)n_factors * 225 * 8, cudaMemcpyDeviceToHost, st));
    return h.finish(CPI_OK);
}

int cpi_imu_factor_hessian_batch(int model, int64_t n_factors, const double* records, const double* e, const double* H1, const double* H2,
                                 double* G11, double* G12, double* G22, double* g1, double* g2, double* f, void* stream) {
    if (model != 1 && model != 2) return fail(CPI_EINVAL, "model must be 1 or 2 (got %d)", model);
    if (n_factors < 0) return fail(CPI_EINVAL, "negative count");
    if (n_factors == 0) return CPI_OK;
    if (!records || !e || !H1 || !H2 || !G11 || !G12 || !G22 || !g1 || !g2 || !f) return fail(CPI_EINVAL, "null pointer argument");
    DevInfo d;
    int rc = device_info(d);
    if (rc) return rc;
    CU(cpi::hessian_launch(cpi_record_doubles(model), n_factors, records, e, H1, H2, G11, G12, G22, g1, g2, f, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int cpi_imu_factor_whiten_batch(int model, int64_t n_factors, const double* records, const double* e, const double* H1, const double* H2,
                                double* A1, double* A2, double* b, void* stream) {
    if (model != 1 && model != 2) return fail(CPI_EINVAL, "model must be 1 or 2 (got %d)", model);
    if (n_factors < 0) return fail(CPI_EINVAL, "negative count");
    if (n_factors == 0) return CPI_OK;
    if (!records || !e || !H1 || !H2 || !A1 || !A2 || !b) return fail(CPI_EINVAL, "null pointer argument");
    DevInfo d;
    int rc = device_info(d);
    if (rc) return rc;
    CU(cpi::whiten_launch(cpi_record_doubles(model), n_factors, records, e, H1, H2, A1, A2, b, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int cpi_imu_chain_assemble(int64_t n_factors, const double* G11, const double* G12, const double* G22, const double* g1, const double* g2, double lambda,
                           int diagonal_damping, const double* prior_info0, const double* prior_rhs0, double* D, double* E, double* rhs, void* stream) {
    if (n_factors < 0) return fail(CPI_EINVAL, "negative count");
    if (n_factors > 0 && (!G11 || !G12 || !G22 || !g1 || !g2 || !E)) return fail(CPI_EINVAL, "null pointer argument");
    if (!D || !rhs) return fail(CPI_EINVAL, "null pointer argument");
    if (n_factors >= 2147483647) return fail(CPI_EINVAL, "chain too long");
    if (!(lambda >= 0.0)) return fail(CPI_EINVAL, "lambda must be >= 0 (got %g)", lambda);
    DevInfo d;
    int rc = device_info(d);
    if (rc) return rc;
    CU(cpi::chains_assemble_launch(1, nullptr, n_factors + 1, G11, G12, G22, g1, g2, lambda, diagonal_damping != 0, prior_info0, prior_rhs0, D, E, rhs,
                                   d.sms, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

}  // extern "C"

namespace {
// the chain layout shared by the many-chain entry points: chain_offsets (device, not inspected here) or chain_uniform >= 1 states per chain;
// n_states, where the entry point takes it, is the layout's state count
int chain_layout_check(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform, std::optional<int64_t> n_states = std::nullopt) {
    if (n_chains < 0) return fail(CPI_EINVAL, "negative count");
    if (n_chains > ((int64_t)1 << 31)) return fail(CPI_EINVAL, "too many chains (%lld; at most 2^31 per call)", (long long)n_chains);
    if (!chain_offsets && chain_uniform < 1) return fail(CPI_EINVAL, "chain_uniform must be >= 1 state per chain (got %lld)", (long long)chain_uniform);
    if (!chain_offsets && n_chains > 0 && chain_uniform > ((int64_t)1 << 40) / n_chains)
        return fail(CPI_EINVAL, "chain_uniform out of range: %lld x %lld states", (long long)n_chains, (long long)chain_uniform);
    if (!n_states) return CPI_OK;
    if (*n_states < n_chains) return fail(CPI_EINVAL, "n_states (%lld) below n_chains (%lld): every chain holds a state", (long long)*n_states,
                                          (long long)n_chains);
    if (!chain_offsets && *n_states != n_chains * chain_uniform)
        return fail(CPI_EINVAL, "n_states (%lld) must be n_chains x chain_uniform (%lld)", (long long)*n_states, (long long)(n_chains * chain_uniform));
    return CPI_OK;
}
}  // namespace

extern "C" {

int cpi_imu_chains_assemble(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform, const double* G11, const double* G12,
                            const double* G22, const double* g1, const double* g2, double lambda, int diagonal_damping,
                            const double* prior_info, const double* prior_rhs, double* D, double* E, double* rhs, void* stream) {
    int rc = chain_layout_check(n_chains, chain_offsets, chain_uniform);
    if (rc || n_chains == 0) return rc;
    const bool any_factor = chain_offsets || chain_uniform > 1;   // a device layout may hold factors
    if (!D || !rhs) return fail(CPI_EINVAL, "null pointer argument (D / rhs)");
    if (any_factor && (!G11 || !G12 || !G22 || !g1 || !g2)) return fail(CPI_EINVAL, "null pointer argument (G11 / G12 / G22 / g1 / g2)");
    if ((chain_offsets || n_chains * chain_uniform > 1) && !E) return fail(CPI_EINVAL, "null pointer argument (E)");
    if (!(lambda >= 0.0)) return fail(CPI_EINVAL, "lambda must be >= 0 (got %g)", lambda);
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    CU(cpi::chains_assemble_launch(n_chains, chain_offsets, chain_uniform, G11, G12, G22, g1, g2, lambda, diagonal_damping != 0, prior_info, prior_rhs,
                                   D, E, rhs, d.sms, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int cpi_imu_factor_cost_batch(int model, int64_t n_factors, const double* states, const int64_t* idx_i, const int64_t* idx_j,
                              const double* records, const double* lin, double* f, void* stream) {
    if (model != 1 && model != 2) return fail(CPI_EINVAL, "model must be 1 or 2 (got %d)", model);
    if (n_factors < 0) return fail(CPI_EINVAL, "negative count");
    if (n_factors == 0) return CPI_OK;
    if (n_factors >= ((int64_t)1 << 33)) return fail(CPI_EINVAL, "too many factors (%lld)", (long long)n_factors);
    if (!states || !records || !lin || !f) return fail(CPI_EINVAL, "null pointer argument");
    if ((idx_i == nullptr) != (idx_j == nullptr)) return fail(CPI_EINVAL, "idx_i and idx_j must both be given or both be null");
    DevInfo d;
    int rc = device_info(d);
    if (rc) return rc;
    CU(cpi::factor_cost_launch(model, n_factors, states, idx_i, idx_j, records, lin, f, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int cpi_imu_chains_cost_sum(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform, const double* f, double* cost, void* stream) {
    if (n_chains < 0) return fail(CPI_EINVAL, "negative count");
    if (n_chains == 0) return CPI_OK;
    if (!chain_offsets && chain_uniform < 1) return fail(CPI_EINVAL, "chain_uniform must be >= 1 without chain_offsets");
    if (!f || !cost) return fail(CPI_EINVAL, "null pointer argument");
    CU(cpi::chains_cost_sum_launch(n_chains, chain_offsets, chain_offsets ? 0 : chain_uniform, f, cost, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int cpi_imu_chains_assemble_lm(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform, const double* G11, const double* G12,
                               const double* G22, const double* g1, const double* g2, const double* lambda, int diagonal_damping,
                               const double* prior_info, const double* prior_rhs, double* D, double* E, double* rhs, double* damp, void* stream) {
    int rc = chain_layout_check(n_chains, chain_offsets, chain_uniform);
    if (rc || n_chains == 0) return rc;
    const bool any_factor = chain_offsets || chain_uniform > 1;
    if (!lambda) return fail(CPI_EINVAL, "null pointer argument (lambda: one per chain)");
    if (!D || !rhs) return fail(CPI_EINVAL, "null pointer argument (D / rhs)");
    if (any_factor && (!G11 || !G12 || !G22 || !g1 || !g2)) return fail(CPI_EINVAL, "null pointer argument (G11 / G12 / G22 / g1 / g2)");
    if ((chain_offsets || n_chains * chain_uniform > 1) && !E) return fail(CPI_EINVAL, "null pointer argument (E)");
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    CU(cpi::chains_assemble_lm_launch(n_chains, chain_offsets, chain_uniform, G11, G12, G22, g1, g2, lambda, diagonal_damping != 0, prior_info,
                                      prior_rhs, D, E, rhs, damp, d.sms, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int64_t cpi_imu_chains_solve_workspace(int64_t n_chains, int64_t n_states) {
    if (n_chains < 0 || n_states < 0 || n_states < n_chains) return (int64_t)CPI_EINVAL;
    return cpi::chains_solve_workspace_bytes(n_states);
}

int cpi_imu_chains_solve(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform, int64_t n_states, const double* D, const double* E,
                         const double* rhs, double* x, void* workspace, void* stream) {
    int rc = chain_layout_check(n_chains, chain_offsets, chain_uniform, n_states);
    if (rc) return rc;
    if (n_chains == 0) return CPI_OK;
    if (!D || !rhs || !x || !workspace || (n_states > 1 && !E)) return fail(CPI_EINVAL, "null pointer argument");
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    int launches = 0;
    CU(cpi::chains_solve_launch(n_chains, chain_offsets, chain_uniform, n_states, D, E, rhs, x, (double*)workspace, d.sms, (cudaStream_t)stream,
                                &launches));
    g_launches += launches;
    return CPI_OK;
}

int64_t cpi_imu_chains_marginals_workspace(int64_t n_chains, int64_t n_states) {
    if (n_chains < 0 || n_states < 0 || n_states < n_chains) return (int64_t)CPI_EINVAL;
    return cpi::chains_marginals_workspace_bytes(n_states);
}

int cpi_imu_chains_marginals(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform, int64_t n_states, const double* D, const double* E,
                             double* cov, double* cross, void* workspace, void* stream) {
    int rc = chain_layout_check(n_chains, chain_offsets, chain_uniform, n_states);
    if (rc) return rc;
    if (n_chains == 0) return CPI_OK;
    if (!D || !cov || !workspace || (n_states > 1 && !E)) return fail(CPI_EINVAL, "null pointer argument");
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    int launches = 0;
    CU(cpi::chains_marginals_launch(n_chains, chain_offsets, chain_uniform, n_states, D, E, cov, cross, (double*)workspace, d.sms, (cudaStream_t)stream,
                                    &launches));
    g_launches += launches;
    return CPI_OK;
}

int64_t cpi_imu_chains_pair_covariance_workspace(int64_t n_chains, int64_t n_states) {
    if (n_chains < 0 || n_states < 0 || n_states < n_chains) return (int64_t)CPI_EINVAL;
    return cpi::chains_pair_cov_workspace_bytes(n_states);
}

int cpi_imu_chains_pair_covariance(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform, int64_t n_states, const double* D,
                                   const double* E, int64_t n_pairs, const int64_t* pair_i, const int64_t* pair_j, double* out, void* workspace,
                                   void* stream) {
    int rc = chain_layout_check(n_chains, chain_offsets, chain_uniform, n_states);
    if (rc) return rc;
    if (n_pairs < 0) return fail(CPI_EINVAL, "negative count (n_pairs)");
    if (n_pairs == 0) return CPI_OK;
    if (n_chains == 0) return fail(CPI_EINVAL, "n_pairs > 0 needs at least one state");
    if (!D || !workspace || (n_states > 1 && !E) || !pair_i || !pair_j || !out) return fail(CPI_EINVAL, "null pointer argument");
    if ((rc = check_aliasing({D, E, pair_i, pair_j, workspace}, {out}))) return rc;
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    int launches = 0;
    CU(cpi::chains_pair_cov_launch(n_chains, chain_offsets, chain_uniform, n_states, D, E, n_pairs, pair_i, pair_j, out, (double*)workspace, d.sms,
                                   (cudaStream_t)stream, &launches));
    g_launches += launches;
    return CPI_OK;
}

int64_t cpi_imu_chains_lm_workspace(int64_t n_states) { return n_states < 0 ? (int64_t)CPI_EINVAL : cpi::lm_workspace_bytes(n_states); }

int cpi_imu_chains_lm_update(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform, int64_t n_states, const cpi_lm_params* params,
                             const double* f_cur, const double* prior_f_cur, const double* f_new, const double* prior_f_new, const double* rhs,
                             const double* D, const double* E, const double* damp, const double* delta, const double* states_new, double* states,
                             double* lambda, double* cost, int32_t* status, int32_t* iterations, int32_t* tries, int32_t* any_running,
                             void* workspace, void* stream) {
    int rc = chain_layout_check(n_chains, chain_offsets, chain_uniform, n_states);
    if (rc) return rc;
    if (!params) return fail(CPI_EINVAL, "null pointer argument (params)");
    const cpi_lm_params& p = *params;
    if (!(p.lambda_factor > 1.0)) return fail(CPI_EINVAL, "lambda_factor must be > 1 (got %g)", p.lambda_factor);
    if (!(p.lambda_lower >= 0.0)) return fail(CPI_EINVAL, "lambda_lower must be >= 0 (got %g)", p.lambda_lower);
    if (!(p.lambda_upper >= p.lambda_lower)) return fail(CPI_EINVAL, "lambda_upper (%g) must be >= lambda_lower (%g)", p.lambda_upper, p.lambda_lower);
    if (!(p.min_model_fidelity >= 0.0 && p.min_model_fidelity < 1.0))
        return fail(CPI_EINVAL, "min_model_fidelity must be in [0, 1) (got %g)", p.min_model_fidelity);
    if (!(p.absolute_error_tol >= 0.0)) return fail(CPI_EINVAL, "absolute_error_tol must be >= 0 (got %g)", p.absolute_error_tol);
    if (!(p.relative_error_tol >= 0.0)) return fail(CPI_EINVAL, "relative_error_tol must be >= 0 (got %g)", p.relative_error_tol);
    if (p.max_iterations < 1 || p.max_iterations > 2147483647)
        return fail(CPI_EINVAL, "max_iterations must be in [1, 2^31) (got %lld)", (long long)p.max_iterations);
    if (n_chains == 0) return CPI_OK;
    if (n_states > n_chains && (!f_cur || !f_new || !E)) return fail(CPI_EINVAL, "null pointer argument (f_cur / f_new / E)");
    if (!rhs || !D || !damp || !delta || !states_new || !states || !workspace)
        return fail(CPI_EINVAL, "null pointer argument (rhs / D / damp / delta / states_new / states / workspace)");
    if (!lambda || !cost || !status || !iterations || !tries) return fail(CPI_EINVAL, "null pointer argument (lambda / cost / status / iterations / tries)");
    if ((prior_f_cur == nullptr) != (prior_f_new == nullptr)) return fail(CPI_EINVAL, "prior_f_cur and prior_f_new must both be given or both be null");
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    CU(cpi::lm_update_launch(n_chains, chain_offsets, chain_uniform, n_states, p, f_cur, prior_f_cur, f_new, prior_f_new, rhs, D, E, damp, delta,
                             states_new, states, lambda, cost, status, iterations, tries, any_running, (double*)workspace, (cudaStream_t)stream));
    g_launches += 2;
    return CPI_OK;
}

int cpi_imu_chain_marginalize(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform, const int64_t* n_marg, int64_t n_marg_uniform,
                              const double* G11, const double* G12, const double* G22, const double* g1, const double* g2, const double* f,
                              const double* prior_info, const double* prior_rhs, const double* prior_f,
                              double* out_info, double* out_rhs, double* out_f, void* stream) {
    int rc = chain_layout_check(n_chains, chain_offsets, chain_uniform);
    if (rc || n_chains == 0) return rc;
    if (!n_marg && n_marg_uniform < 0) return fail(CPI_EINVAL, "negative count (n_marg_uniform)");
    if (!n_marg && !chain_offsets && n_marg_uniform >= chain_uniform)
        return fail(CPI_EINVAL, "n_marg_uniform (%lld) must be < the states per chain (%lld): a chain keeps at least one state",
                    (long long)n_marg_uniform, (long long)chain_uniform);
    if (!out_info || !out_rhs) return fail(CPI_EINVAL, "null pointer argument (out_info / out_rhs)");
    if ((prior_info == nullptr) != (prior_rhs == nullptr)) return fail(CPI_EINVAL, "prior_info and prior_rhs must both be given or both be null");
    const bool any_factor = n_marg || n_marg_uniform > 0;
    if (any_factor && (!G11 || !G12 || !G22 || !g1 || !g2 || !f)) return fail(CPI_EINVAL, "null pointer argument (G11 / G12 / G22 / g1 / g2 / f)");
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    CU(cpi::marginalize_launch(n_chains, chain_offsets, chain_uniform, n_marg, n_marg_uniform, G11, G12, G22, g1, g2, f, prior_info, prior_rhs, prior_f,
                               out_info, out_rhs, out_f, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int cpi_imu_prior_at(int64_t n, const double* info, const double* rhs, const double* f, const double* lin_states, const double* states,
                     double* rhs_out, double* f_out, void* stream) {
    if (n < 0) return fail(CPI_EINVAL, "negative count");
    if (n == 0) return CPI_OK;
    if (n > ((int64_t)1 << 31)) return fail(CPI_EINVAL, "too many priors (%lld; at most 2^31 per call)", (long long)n);
    if (!info || !rhs || !lin_states || !states || !rhs_out) return fail(CPI_EINVAL, "null pointer argument");
    DevInfo d;
    int rc = device_info(d);
    if (rc) return rc;
    CU(cpi::prior_at_launch(n, info, rhs, f, lin_states, states, rhs_out, f_out, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int cpi_imu_state_priors_fold(int64_t n_chains, const int64_t* chain_offsets, int64_t chain_uniform, const int64_t* sp_offsets,
                              const double* sp_info, const double* sp_rhs, const double* sp_f, double* G11, double* G22, double* g1,
                              double* g2, double* f, double* prior_info, double* prior_rhs, double* prior_f, void* stream) {
    int rc = chain_layout_check(n_chains, chain_offsets, chain_uniform);
    if (rc || n_chains == 0) return rc;
    if (!sp_offsets) return fail(CPI_EINVAL, "null pointer argument (sp_offsets)");
    if ((sp_info == nullptr) != (sp_rhs == nullptr)) return fail(CPI_EINVAL, "sp_info and sp_rhs must both be given or both be null");
    if (!sp_info && !sp_f) return fail(CPI_EINVAL, "null pointer argument (sp_f: the f-only fold needs the priors' constants)");
    if (!chain_offsets && chain_uniform == 1) {                    // every state is a chain of its own: everything lands on the chain priors
        if (sp_info && (!prior_info || !prior_rhs)) return fail(CPI_EINVAL, "null pointer argument (prior_info / prior_rhs: single-state chains)");
        if (sp_f && !prior_f) return fail(CPI_EINVAL, "null pointer argument (prior_f: single-state chains)");
    }
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    CU(cpi::state_priors_fold_launch(n_chains, chain_offsets, chain_uniform, sp_offsets, sp_info, sp_rhs, sp_f, G11, G22, g1, g2, f, prior_info,
                                     prior_rhs, prior_f, d.sms, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int cpi_imu_state_priors_robust(int64_t n, const int32_t* loss, const double* loss_k, const double* info, const double* rhs, const double* f,
                                double* info_out, double* rhs_out, double* f_out, void* stream) {
    if (n < 0) return fail(CPI_EINVAL, "negative count");
    if (n == 0) return CPI_OK;
    if (n > ((int64_t)1 << 31)) return fail(CPI_EINVAL, "too many priors (%lld; at most 2^31 per call)", (long long)n);
    if (!loss || !loss_k || !f || !f_out) return fail(CPI_EINVAL, "null pointer argument (loss / loss_k / f / f_out)");
    if ((info_out == nullptr) != (rhs_out == nullptr)) return fail(CPI_EINVAL, "info_out and rhs_out must both be given or both be null");
    if (info_out && (!info || !rhs)) return fail(CPI_EINVAL, "null pointer argument (info / rhs: the full pass reads them)");
    DevInfo d;
    int rc = device_info(d);
    if (rc) return rc;
    CU(cpi::state_priors_robust_launch(n, loss, loss_k, info, rhs, f, info_out, rhs_out, f_out, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int64_t cpi_imu_chain_solve_workspace(int64_t n_states) { return n_states < 0 ? (int64_t)CPI_EINVAL : cpi::chains_solve_workspace_bytes(n_states); }

int cpi_imu_chain_solve(int64_t n_states, const double* D, const double* E, const double* rhs, double* x, void* workspace, void* stream) {
    if (n_states < 0) return fail(CPI_EINVAL, "negative count");
    if (n_states == 0) return CPI_OK;
    if (!D || !rhs || !x || (n_states > 1 && (!E || !workspace))) return fail(CPI_EINVAL, "null pointer argument");
    DevInfo d;
    int rc = device_info(d);
    if (rc) return rc;
    int launches = 0;
    CU(cpi::chains_solve_launch(1, nullptr, n_states, n_states, D, E, rhs, x, (double*)workspace, d.sms, (cudaStream_t)stream, &launches));
    g_launches += launches;
    return CPI_OK;
}

int cpi_predict_state_batch(int model, int64_t n, const double* states_k, const double* records, const double* lin, double* states_k1, void* stream) {
    if (model != 1 && model != 2) return fail(CPI_EINVAL, "model must be 1 or 2 (got %d)", model);
    if (n < 0) return fail(CPI_EINVAL, "negative count");
    if (n == 0) return CPI_OK;
    if (!states_k || !records || !lin || !states_k1) return fail(CPI_EINVAL, "null pointer argument");
    DevInfo d;
    int rc = device_info(d);
    if (rc) return rc;
    CU(cpi::predict_launch(model, n, states_k, records, lin, states_k1, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

}  // extern "C"

namespace {
// argument checks shared by the merge and scan entry points (no CUDA call); `what` names the operation ("merged" / "scanned")
int merge_check(int model, int dtype, int64_t n_groups, const int64_t* group_offsets, int64_t group_uniform, const char* what = "merged") {
    if (model == 2)
        return fail(CPI_EINVAL, "model 2 records cannot be %s: their gravity removal depends on q_k_lin, which a merge would have to "
                                "re-linearise (only model 1 is supported)", what);
    if (model != 1) return fail(CPI_EINVAL, "model must be 1 (got %d)", model);
    if (dtype != 64 && dtype != 32) return fail(CPI_EINVAL, "dtype must be 64 or 32 (got %d)", dtype);
    if (n_groups < 0 || (!group_offsets && group_uniform < 0)) return fail(CPI_EINVAL, "negative count");
    if (n_groups > 2147483647) return fail(CPI_EINVAL, "too many groups (%lld; at most 2^31 - 1 per call)", (long long)n_groups);
    return CPI_OK;
}

// the host copy of a CSR layout (or the uniform one) is validated before anything reaches the device; *n_rec = records it spans
int host_layout_check(int dtype, int64_t n_groups, const int64_t* group_offsets, int64_t group_uniform, int64_t* n_rec) {
    const size_t es = dtype == 32 ? 4 : 8;
    const int64_t max_records = (int64_t)(((uint64_t)1 << 62) / ((uint64_t)CPI_REC_V1_DOUBLES * es));
    if (group_offsets) {
        if (group_offsets[0] < 0) return fail(CPI_EINVAL, "group_offsets out of range: group_offsets[0] = %lld is negative", (long long)group_offsets[0]);
        for (int64_t g = 0; g < n_groups; g++)
            if (group_offsets[g + 1] < group_offsets[g])
                return fail(CPI_EINVAL, "group_offsets must be non-decreasing (group %lld)", (long long)g);
        if (group_offsets[n_groups] > max_records)
            return fail(CPI_EINVAL, "group_offsets out of range: %lld records", (long long)group_offsets[n_groups]);
    } else if (group_uniform > max_records / n_groups) {
        return fail(CPI_EINVAL, "group_uniform out of range: %lld x %lld records", (long long)n_groups, (long long)group_uniform);
    }
    *n_rec = group_offsets ? group_offsets[n_groups] : n_groups * group_uniform;
    return CPI_OK;
}
}  // namespace

extern "C" {

int cpi_merge_records(int model, int dtype, int64_t n_groups, const int64_t* group_offsets, int64_t group_uniform,
                      const void* records, const void* lin, void* out_records, void* stream) {
    int rc = merge_check(model, dtype, n_groups, group_offsets, group_uniform);
    if (rc || n_groups == 0) return rc;
    if (!out_records) return fail(CPI_EINVAL, "null pointer argument (out_records)");
    if ((!records || !lin) && (group_offsets || group_uniform > 0)) return fail(CPI_EINVAL, "null pointer argument (records / lin)");
    const size_t rb = (size_t)CPI_REC_V1_DOUBLES * (dtype == 32 ? 4 : 8);
    // equal pointers always overlap; the uniform layout's extent is known, so check its whole range
    if (out_records == records ||
        (!group_offsets && records && bytes_overlap(records, (size_t)n_groups * group_uniform * rb, out_records, (size_t)n_groups * rb)))
        return fail(CPI_EINVAL, "out_records must not overlap records");
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    CU(cpi::merge_launch(dtype, n_groups, group_offsets, group_uniform, records, lin, out_records, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int cpi_merge_records_host(int model, int dtype, int64_t n_groups, const int64_t* group_offsets, int64_t group_uniform,
                           const void* records, const void* lin, void* out_records) {
    int rc = merge_check(model, dtype, n_groups, group_offsets, group_uniform);
    if (rc || n_groups == 0) return rc;
    if (!out_records) return fail(CPI_EINVAL, "null pointer argument (out_records)");
    const size_t es = dtype == 32 ? 4 : 8;
    int64_t n_rec = 0;
    if ((rc = host_layout_check(dtype, n_groups, group_offsets, group_uniform, &n_rec))) return rc;
    if (n_rec > 0 && (!records || !lin)) return fail(CPI_EINVAL, "null pointer argument (records / lin)");
    if (n_rec > 0 && out_records == records) return fail(CPI_EINVAL, "out_records must not overlap records");
    HostCall h;
    if ((rc = h.start())) return rc;
    const size_t rb = (size_t)CPI_REC_V1_DOUBLES * es;
    void *d_r, *d_l, *d_o, *d_off = nullptr;
    if (group_offsets && (rc = h.upload(group_offsets, (size_t)(n_groups + 1) * 8, &d_off))) return rc;
    if ((rc = h.upload(records, (size_t)n_rec * rb, &d_r))) return rc;
    if ((rc = h.upload(lin, (size_t)n_rec * CPI_LIN_DOUBLES * es, &d_l))) return rc;
    if ((rc = h.buf((size_t)n_groups * rb, &d_o))) return rc;
    cudaStream_t st = h.copy_stream();
    if ((rc = cpi_merge_records(model, dtype, n_groups, (const int64_t*)d_off, group_uniform, d_r, d_l, d_o, st))) return rc;
    CU(cudaMemcpyAsync(out_records, d_o, (size_t)n_groups * rb, cudaMemcpyDeviceToHost, st));
    return h.finish(CPI_OK);
}

int64_t cpi_scan_records_workspace(int64_t n_groups, int64_t n_records) {
    if (n_groups < 0 || n_records < 0) return fail(CPI_EINVAL, "negative count");
    return cpi::scan_workspace_bytes(n_records);
}

int cpi_scan_records(int model, int dtype, int64_t n_groups, const int64_t* group_offsets, int64_t group_uniform,
                     const void* records, const void* lin, void* out_records, void* workspace, void* stream) {
    int rc = merge_check(model, dtype, n_groups, group_offsets, group_uniform, "scanned");
    if (rc || n_groups == 0) return rc;
    if (!out_records) return fail(CPI_EINVAL, "null pointer argument (out_records)");
    if (!workspace) return fail(CPI_EINVAL, "null pointer argument (workspace: cpi_scan_records_workspace bytes)");
    if ((!records || !lin) && (group_offsets || group_uniform > 0)) return fail(CPI_EINVAL, "null pointer argument (records / lin)");
    const size_t rb = (size_t)CPI_REC_V1_DOUBLES * (dtype == 32 ? 4 : 8), bytes = (size_t)n_groups * group_uniform * rb;
    // equal pointers always overlap; the uniform layout's extent is known, so check its whole range
    if (out_records == records || (!group_offsets && records && bytes_overlap(records, bytes, out_records, bytes)))
        return fail(CPI_EINVAL, "out_records must not overlap records");
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    // device offsets are not read here: the records of one call fit in device memory, which bounds their count
    const int64_t n_bound = group_offsets ? (int64_t)(d.mem / rb) : n_groups * group_uniform;
    int launches = 0;
    cudaError_t e = cpi::scan_launch(dtype, n_groups, group_offsets, group_uniform, n_bound, records, lin, out_records, workspace, d.sms,
                                     (cudaStream_t)stream, &launches);
    g_launches += launches;
    CU(e);
    return CPI_OK;
}

int cpi_scan_records_host(int model, int dtype, int64_t n_groups, const int64_t* group_offsets, int64_t group_uniform,
                          const void* records, const void* lin, void* out_records) {
    int rc = merge_check(model, dtype, n_groups, group_offsets, group_uniform, "scanned");
    if (rc || n_groups == 0) return rc;
    if (!out_records) return fail(CPI_EINVAL, "null pointer argument (out_records)");
    const size_t es = dtype == 32 ? 4 : 8;
    int64_t n_end = 0;
    if ((rc = host_layout_check(dtype, n_groups, group_offsets, group_uniform, &n_end))) return rc;
    const int64_t b0 = group_offsets ? group_offsets[0] : 0, n_rec = n_end - b0;
    if (n_rec > 0 && (!records || !lin)) return fail(CPI_EINVAL, "null pointer argument (records / lin)");
    if (n_rec > 0 && out_records == records) return fail(CPI_EINVAL, "out_records must not overlap records");
    if (n_rec == 0) return CPI_OK;             // only empty groups: nothing to write
    const size_t rb = (size_t)CPI_REC_V1_DOUBLES * es, lb = (size_t)CPI_LIN_DOUBLES * es;
    // the device copies start at record b0; the offsets are shifted to match (declared before the host call, which drains the copy
    // out of it before it is freed)
    std::string shifted;
    if (group_offsets) {
        shifted.resize((size_t)(n_groups + 1) * 8);
        int64_t* so = (int64_t*)&shifted[0];
        for (int64_t g = 0; g <= n_groups; g++) so[g] = group_offsets[g] - b0;
    }
    HostCall h;
    if ((rc = h.start())) return rc;
    void *d_r, *d_l, *d_o, *d_ws, *d_off = nullptr;
    if (group_offsets && (rc = h.upload(shifted.data(), (size_t)(n_groups + 1) * 8, &d_off))) return rc;
    if ((rc = h.upload((const char*)records + (size_t)b0 * rb, (size_t)n_rec * rb, &d_r))) return rc;
    if ((rc = h.upload((const char*)lin + (size_t)b0 * lb, (size_t)n_rec * lb, &d_l))) return rc;
    if ((rc = h.buf((size_t)n_rec * rb, &d_o))) return rc;
    if ((rc = h.buf((size_t)cpi::scan_workspace_bytes(n_rec), &d_ws))) return rc;
    cudaStream_t st = h.copy_stream();
    if ((rc = cpi_scan_records(model, dtype, n_groups, (const int64_t*)d_off, group_uniform, d_r, d_l, d_o, d_ws, st))) return rc;
    CU(cudaMemcpyAsync((char*)out_records + (size_t)b0 * rb, d_o, (size_t)n_rec * rb, cudaMemcpyDeviceToHost, st));
    return h.finish(CPI_OK);
}

}  // extern "C"

namespace {
// argument checks shared by the two propagation entry points (no CUDA call)
int propagate_check(int model, int64_t n, const double* states_k, const double* cov_k, const double* records, const double* lin,
                    const double* states_k1, const double* cov_k1, const double* cross) {
    if (model != 1 && model != 2) return fail(CPI_EINVAL, "model must be 1 or 2 (got %d)", model);
    if (n < 0) return fail(CPI_EINVAL, "negative count");
    if (n == 0) return CPI_OK;
    if (!states_k || !cov_k || !records || !lin || !states_k1 || !cov_k1) return fail(CPI_EINVAL, "null pointer argument");
    return check_aliasing({states_k, cov_k, records, lin}, {states_k1, cov_k1, cross});
}

// argument checks shared by the two smoother entry points (no CUDA call); scan: the parallel smoother, which needs the workspace
int rts_check(bool scan, int64_t n_runs, const int64_t* run_offsets, int64_t run_uniform, int64_t n_states, const double* states,
              const double* cov, const double* pred_states, const double* pred_cov, const double* cross, const double* states_out,
              const double* cov_out, const double* cross_out, const void* workspace) {
    int rc = chain_layout_check(n_runs, run_offsets, run_uniform, n_states);
    if (rc || n_runs == 0) return rc;
    const bool any_step = n_states > n_runs;                       // a transition exists
    if (!states || !cov || !states_out || !cov_out || (any_step && (!pred_states || !pred_cov || !cross)))
        return fail(CPI_EINVAL, "null pointer argument");
    if (scan && any_step && !workspace) return fail(CPI_EINVAL, "null pointer argument (workspace: cpi_rts_smooth_scan_workspace bytes)");
    return check_aliasing({run_offsets, states, cov, pred_states, pred_cov, cross}, {states_out, cov_out, cross_out, workspace});
}
}  // namespace

extern "C" {

int cpi_propagate_batch(int model, int64_t n, const double* states_k, const double* cov_k, const int64_t* anchor, const double* records,
                        const double* lin, double* states_k1, double* cov_k1, double* cross, void* stream) {
    int rc = propagate_check(model, n, states_k, cov_k, records, lin, states_k1, cov_k1, cross);
    if (rc || n == 0) return rc;
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    cpi::PropagateParams p{n, states_k, cov_k, anchor, records, lin, states_k1, cov_k1, cross};
    CU(cpi::propagate_launch(model, p, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int cpi_propagate_batch_host(int model, int64_t n, int64_t n_anchors, const double* states_k, const double* cov_k, const int64_t* anchor,
                             const double* records, const double* lin, double* states_k1, double* cov_k1, double* cross) {
    if (n_anchors < 0) return fail(CPI_EINVAL, "negative count");
    int rc = propagate_check(model, n, states_k, cov_k, records, lin, states_k1, cov_k1, cross);
    if (rc || n == 0) return rc;
    if (!anchor && n_anchors < n) return fail(CPI_EINVAL, "without an anchor array window i starts from entry i: n_anchors must be >= n");
    if (anchor)
        for (int64_t i = 0; i < n; i++)
            if (anchor[i] < 0 || anchor[i] >= n_anchors)
                return fail(CPI_EINVAL, "window %lld: anchor index %lld out of range [0, %lld)", (long long)i, (long long)anchor[i], (long long)n_anchors);
    const int64_t na = anchor ? n_anchors : n;           // anchor entries the windows read
    const size_t rb = (size_t)cpi_record_doubles(model) * 8;
    HostCall h;
    if ((rc = h.start())) return rc;
    void *d_x, *d_c, *d_r, *d_l, *d_a = nullptr, *d_x1, *d_c1, *d_cr = nullptr;
    if ((rc = h.upload(states_k, (size_t)na * CPI_STATE_DOUBLES * 8, &d_x))) return rc;
    if ((rc = h.upload(cov_k, (size_t)na * 225 * 8, &d_c))) return rc;
    if ((rc = h.upload(records, (size_t)n * rb, &d_r))) return rc;
    if ((rc = h.upload(lin, (size_t)n * CPI_LIN_DOUBLES * 8, &d_l))) return rc;
    if (anchor && (rc = h.upload(anchor, (size_t)n * 8, &d_a))) return rc;
    if ((rc = h.buf((size_t)n * CPI_STATE_DOUBLES * 8, &d_x1))) return rc;
    if ((rc = h.buf((size_t)n * 225 * 8, &d_c1))) return rc;
    if (cross && (rc = h.buf((size_t)n * 225 * 8, &d_cr))) return rc;
    cudaStream_t st = h.copy_stream();
    rc = cpi_propagate_batch(model, n, (const double*)d_x, (const double*)d_c, (const int64_t*)d_a, (const double*)d_r, (const double*)d_l,
                             (double*)d_x1, (double*)d_c1, (double*)d_cr, st);
    if (rc) return rc;
    CU(cudaMemcpyAsync(states_k1, d_x1, (size_t)n * CPI_STATE_DOUBLES * 8, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(cov_k1, d_c1, (size_t)n * 225 * 8, cudaMemcpyDeviceToHost, st));
    if (cross) CU(cudaMemcpyAsync(cross, d_cr, (size_t)n * 225 * 8, cudaMemcpyDeviceToHost, st));
    return h.finish(CPI_OK);
}

int cpi_retract_batch(int64_t n, const double* states, const double* xi, double* states_out, void* stream) {
    if (n < 0) return fail(CPI_EINVAL, "negative count");
    if (n == 0) return CPI_OK;
    if (!states || !xi || !states_out) return fail(CPI_EINVAL, "null pointer argument");
    DevInfo d;
    int rc = device_info(d);
    if (rc) return rc;
    CU(cpi::retract_launch(n, states, xi, states_out, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int cpi_state_update_batch(int64_t n, const double* states, const double* cov, const double* meas_info, const double* meas_states,
                           const double* gate, double* states_out, double* cov_out, double* nis, int32_t* applied, void* stream) {
    if (n < 0) return fail(CPI_EINVAL, "negative count");
    if (n == 0) return CPI_OK;
    if (!states || !cov || !meas_info || !meas_states || !states_out || !cov_out) return fail(CPI_EINVAL, "null pointer argument");
    int rc = check_aliasing({states, cov, meas_info, meas_states, gate}, {states_out, cov_out, nis, applied});
    if (rc) return rc;
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    CU(cpi::state_update_launch(n, states, cov, meas_info, meas_states, gate, states_out, cov_out, nis, applied, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int cpi_state_update_measurements_batch(int64_t n, const double* states, const double* cov, const int64_t* meas_offsets, const int32_t* kind,
                                        const double* z, const double* sqrt_info, const double* aux, const double* gate, double* states_out,
                                        double* cov_out, double* nis, int32_t* applied, void* stream) {
    if (n < 0) return fail(CPI_EINVAL, "negative count");
    if (n == 0) return CPI_OK;
    if (!states || !cov || !meas_offsets || !kind || !z || !sqrt_info || !aux || !states_out || !cov_out)
        return fail(CPI_EINVAL, "null pointer argument");
    int rc = check_aliasing({states, cov, meas_offsets, kind, z, sqrt_info, aux, gate}, {states_out, cov_out, nis, applied});
    if (rc) return rc;
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    CU(cpi::state_update_meas_launch(n, states, cov, meas_offsets, kind, z, sqrt_info, aux, gate, states_out, cov_out, nis, applied,
                                     (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int cpi_state_update_measurements_iterated_batch(int64_t n, const double* states, const double* cov, const int64_t* meas_offsets,
                                                 const int32_t* kind, const double* z, const double* sqrt_info, const double* aux,
                                                 const int32_t* loss, const double* loss_k, const double* gate, int max_iterations, double tol,
                                                 double* states_out, double* cov_out, double* nis, int32_t* status, int32_t* iterations,
                                                 void* stream) {
    if (n < 0) return fail(CPI_EINVAL, "negative count");
    if (max_iterations < 1) return fail(CPI_EINVAL, "max_iterations must be >= 1 (got %d)", max_iterations);
    if (!(tol >= 0.0)) return fail(CPI_EINVAL, "tol must be >= 0 (+inf: one iteration; got %g)", tol);
    if ((loss == nullptr) != (loss_k == nullptr)) return fail(CPI_EINVAL, "loss and loss_k must both be given or both be null");
    if (n == 0) return CPI_OK;
    if (!states || !cov || !meas_offsets || !kind || !z || !sqrt_info || !aux || !states_out || !cov_out)
        return fail(CPI_EINVAL, "null pointer argument");
    int rc = check_aliasing({states, cov, meas_offsets, kind, z, sqrt_info, aux, loss, loss_k, gate},
                            {states_out, cov_out, nis, status, iterations});
    if (rc) return rc;
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    CU(cpi::state_update_meas_iter_launch(n, states, cov, meas_offsets, kind, z, sqrt_info, aux, loss, loss_k, gate, max_iterations, tol,
                                          states_out, cov_out, nis, status, iterations, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int cpi_rts_smooth_batch(int64_t n_runs, const int64_t* run_offsets, int64_t run_uniform, int64_t n_states, const double* states,
                         const double* cov, const double* pred_states, const double* pred_cov, const double* cross, double* states_out,
                         double* cov_out, double* cross_out, void* stream) {
    int rc = rts_check(false, n_runs, run_offsets, run_uniform, n_states, states, cov, pred_states, pred_cov, cross, states_out, cov_out,
                       cross_out, nullptr);
    if (rc || n_runs == 0) return rc;
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    CU(cpi::rts_smooth_launch(n_runs, run_offsets, run_offsets ? 0 : run_uniform, states, cov, pred_states, pred_cov, cross, states_out, cov_out,
                              cross_out, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

int64_t cpi_rts_smooth_scan_workspace(int64_t n_runs, int64_t n_states) {
    if (n_runs < 0 || n_states < 0) return fail(CPI_EINVAL, "negative count");
    if (n_states < n_runs) return fail(CPI_EINVAL, "n_states (%lld) < n_runs (%lld): every run holds a keyframe", (long long)n_states,
                                       (long long)n_runs);
    return n_states > n_runs ? cpi::rts_scan_workspace_bytes(n_states) : 0;
}

int cpi_rts_smooth_scan_batch(int64_t n_runs, const int64_t* run_offsets, int64_t run_uniform, int64_t n_states, const double* states,
                              const double* cov, const double* pred_states, const double* pred_cov, const double* cross, double* states_out,
                              double* cov_out, double* cross_out, void* workspace, void* stream) {
    int rc = rts_check(true, n_runs, run_offsets, run_uniform, n_states, states, cov, pred_states, pred_cov, cross, states_out, cov_out,
                       cross_out, workspace);
    if (rc || n_runs == 0) return rc;
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    int launches = 0;
    cudaError_t e = cpi::rts_scan_launch(n_runs, run_offsets, run_offsets ? 0 : run_uniform, n_states, states, cov, pred_states, pred_cov,
                                         cross, states_out, cov_out, cross_out, workspace, d.sms, (cudaStream_t)stream, &launches);
    g_launches += launches;
    CU(e);
    return CPI_OK;
}

int cpi_imu_measurements_linearize(int64_t n, const int32_t* kind, const int64_t* state_idx, const double* states, const double* z,
                                   const double* sqrt_info, const double* aux, double* info, double* rhs, double* f, void* stream) {
    if (n < 0) return fail(CPI_EINVAL, "negative count");
    if (n == 0) return CPI_OK;
    if (n > ((int64_t)1 << 31)) return fail(CPI_EINVAL, "too many measurements (%lld; at most 2^31 per call)", (long long)n);
    if (!kind || !state_idx || !states || !z || !sqrt_info || !aux || !f) return fail(CPI_EINVAL, "null pointer argument");
    if ((info == nullptr) != (rhs == nullptr)) return fail(CPI_EINVAL, "info and rhs must both be given or both be null");
    int rc = check_aliasing({kind, state_idx, states, z, sqrt_info, aux}, {info, rhs, f});
    if (rc) return rc;
    DevInfo d;
    if ((rc = device_info(d))) return rc;
    CU(cpi::measurements_linearize_launch(n, kind, state_idx, states, z, sqrt_info, aux, info, rhs, f, (cudaStream_t)stream));
    g_launches += 1;
    return CPI_OK;
}

}  // extern "C"
