// Multi-GPU entry points of libcpi_b200.so (declared in include/cpi_b200.h): one process per GPU, window batches sharded
// contiguously over the ranks, ONE in-place all-gather of the fixed-size result records per batch (SURVEY.md 8e; the
// reference builds one preintegrator per factor on one CPU thread, solvers/GraphSolver_IMU.cpp:43 -- windows share nothing).
//
// The preintegration kernel writes this rank's records straight into its slice of the caller's gather buffer; the exchange runs
// on the communicator's OWN stream behind an event, so that the next batch's kernel (into a second gather buffer) overlaps it.
//
// Two exchange paths:
//   PUSH (gather buffers registered with cpi_comm_register): every rank copies its slice into the peers' gather buffers over
//        NVLink with the COPY ENGINES (cudaMemcpyAsync into CUDA-IPC mappings of the peers' buffers), bracketed by two one-element
//        NCCL all-reduces that act as barriers ("every rank has released this buffer" before, "every slice has landed" after).
//        No SM is involved in moving the records.  This matters because the preintegration kernel of configs[1] is a ONE-WAVE
//        kernel (1 000 one-warp CTAs on the 1 056 slots of 132 SMs): an NCCL all-gather kernel running beside it takes whole SMs
//        (one NCCL CTA ~ 7 of an SM's 8 slots) and pushes part of the grid into a second wave.
//   NCCL (unregistered buffers, or CUDA IPC unavailable for them): ncclAllGather on the communicator's stream, with the
//        communicator limited to CPI_B200_NCCL_MAX_CTAS (default 16) CTAs so that the kernel beside it still fits one wave.
//
// NCCL and the CUDA driver are bound at run time (dlopen "libnccl.so.2" / "libcuda.so.1": the copies torch already mapped when
// called from Python), so single-GPU users of the library need neither at link time.
#include <dlfcn.h>
#include <nccl.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include "cpi_common.cuh"
#include "cpi_kernels.h"

extern "C" int cpi_preintegrate_batch(int model, int dtype, int64_t n_windows, const int64_t* sample_offsets, int64_t ns_uniform, const void* samples,
                                      const void* lin, const double* sigmas, int flags, void* out_records, void* stream);
extern "C" int cpi_record_doubles(int model);

namespace cpi { int capi_fail(int code, const char* fmt, ...); }

namespace {

struct NcclApi {
    void* h = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommInitRankConfig)(ncclComm_t*, int, ncclUniqueId, int, ncclConfig_t*) = nullptr;      // optional
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    ncclResult_t (*GetVersion)(int*) = nullptr;
};
NcclApi g_nccl;
std::mutex g_nccl_mu;
// cuMemGetAddressRange_v2(CUdeviceptr* base, size_t* size, CUdeviceptr ptr): the allocation a pointer lives in (for the IPC handle)
typedef int (*cuMemGetAddressRange_t)(unsigned long long*, size_t*, unsigned long long);
cuMemGetAddressRange_t g_addr_range = nullptr;
// cuStreamWriteValue32_v2 / cuStreamWaitValue32_v2(CUstream, CUdeviceptr, cuuint32_t value, unsigned flags): stream-ordered flag write / wait, no SM
typedef int (*cuStreamOp32_t)(cudaStream_t, unsigned long long, unsigned int, unsigned int);
cuStreamOp32_t g_write32 = nullptr, g_wait32 = nullptr;

int nccl_load() {
    std::lock_guard<std::mutex> lk(g_nccl_mu);
    if (g_nccl.h) return CPI_OK;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return cpi::capi_fail(CPI_ENODEVICE, "NCCL not found (dlopen libnccl.so.2): %s", dlerror());
    NcclApi a;
    a.h = h;
#define SYM(field, name) *(void**)(&a.field) = dlsym(h, name); if (!a.field) return cpi::capi_fail(CPI_ENODEVICE, "NCCL symbol %s missing", name)
    SYM(GetUniqueId, "ncclGetUniqueId"); SYM(CommInitRank, "ncclCommInitRank"); SYM(CommDestroy, "ncclCommDestroy");
    SYM(AllGather, "ncclAllGather"); SYM(AllReduce, "ncclAllReduce"); SYM(GetErrorString, "ncclGetErrorString"); SYM(GetVersion, "ncclGetVersion");
#undef SYM
    *(void**)(&a.CommInitRankConfig) = dlsym(h, "ncclCommInitRankConfig");
    if (void* cu = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL)) {
        *(void**)(&g_addr_range) = dlsym(cu, "cuMemGetAddressRange_v2");
        if (!g_addr_range) *(void**)(&g_addr_range) = dlsym(cu, "cuMemGetAddressRange");
        *(void**)(&g_write32) = dlsym(cu, "cuStreamWriteValue32_v2");
        *(void**)(&g_wait32) = dlsym(cu, "cuStreamWaitValue32_v2");
    }
    g_nccl = a;
    return CPI_OK;
}
#define NC(call) do { ncclResult_t r_ = (call); if (r_ != ncclSuccess) return cpi::capi_fail(CPI_ECUDA, "%s failed: %s", #call, g_nccl.GetErrorString(r_)); } while (0)
#define CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return cpi::capi_fail(CPI_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)

constexpr int MAX_WORLD = 64;
struct IpcMsg {                       // what every rank tells the others about a gather buffer it registers
    cudaIpcMemHandle_t handle;        // of the allocation the buffer lives in
    uint64_t offset;                  // of the buffer inside that allocation
    uint64_t bytes;
    int32_t ok;                       // 0: this rank could not export the buffer -> everybody uses the NCCL path for it
    int32_t pad;
};
static_assert(sizeof(IpcMsg) == 88, "IpcMsg layout");
struct OpenedAlloc { int peer; cudaIpcMemHandle_t handle; void* base; int refs; };
struct Registered { void* local = nullptr; size_t bytes = 0; bool push = false; char* peer[MAX_WORLD] = {nullptr}; void* peer_base[MAX_WORLD] = {nullptr}; };

}  // namespace

struct cpi_comm {
    ncclComm_t comm = nullptr;
    int rank = 0, world = 1, device = 0;
    cudaStream_t stream = nullptr;            // communication stream (barriers, NCCL all-gather)
    static constexpr int NCOPY = 4;           // peer copies are spread over several streams = several copy engines: one engine moves
    cudaStream_t copy[NCOPY] = {nullptr};     // ~200 GB/s over NVLink (measured at N = 8: 7 x 23 MB in ~0.8 ms on one stream)
    cudaEvent_t released = nullptr;           // barrier 1 done (comm stream)
    cudaEvent_t copied[NCOPY] = {nullptr};    // this rank's copies on copy stream j done
    cudaEvent_t entry = nullptr;              // recorded on the caller's stream when the call is entered
    cudaEvent_t kernel_done = nullptr;        // recorded on the caller's stream after the kernel
    static constexpr int NBUF = 4;
    void* buf[NBUF] = {nullptr};              // gather buffers seen recently ...
    cudaEvent_t gathered[NBUF] = {nullptr};   // ... and the event recorded behind their last exchange
    int last = -1;
    int* d_bar = nullptr;                     // two ints: source / sink of the barrier all-reduces
    // SM-free barriers: flags[kind][rank] of every rank, written by the peers with 4-byte copy-engine copies and awaited with stream
    // wait-value operations.  An NCCL barrier kernel would have to find SM resources next to a kernel that fills the machine in one wave:
    // it starts only when that kernel drains, and the next kernel on the same gather buffer waits for it (~90 us per step at N = 8).
    uint32_t* flags = nullptr;                // [2][MAX_WORLD] flags + [2] staging words
    uint32_t* peer_flags[64] = {nullptr};     // the peers' flag arrays (CUDA IPC)
    void* peer_flags_base[64] = {nullptr};
    uint32_t seq[2] = {0, 0};
    bool ce_barrier = false;
    std::vector<Registered> regs;             // cpi_comm_register
    std::vector<OpenedAlloc> opened;          // peer allocations mapped with cudaIpcOpenMemHandle (one mapping per allocation)
};

namespace {
// barrier over all ranks on stream s: returns when EVERY rank's stream s has reached its matching call
int comm_barrier(cpi_comm* c, int kind, cudaStream_t s) {
    if (!c->ce_barrier) {
        NC(g_nccl.AllReduce(c->d_bar, c->d_bar + 1, 1, ncclInt, ncclMax, c->comm, s));
        return CPI_OK;
    }
    const uint32_t v = ++c->seq[kind];
    uint32_t* stage = c->flags + 2 * MAX_WORLD + kind;
    if (g_write32(s, (unsigned long long)(uintptr_t)stage, v, 0) != 0) return cpi::capi_fail(CPI_ECUDA, "cuStreamWriteValue32 failed");
    for (int k = 1; k < c->world; k++) {
        const int p = (c->rank + k) % c->world;
        CU(cudaMemcpyAsync(c->peer_flags[p] + kind * MAX_WORLD + c->rank, stage, sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
    }
    for (int k = 1; k < c->world; k++) {
        const int p = (c->rank + k) % c->world;
        if (g_wait32(s, (unsigned long long)(uintptr_t)(c->flags + kind * MAX_WORLD + p), v, 0 /* CU_STREAM_WAIT_VALUE_GEQ */) != 0)
            return cpi::capi_fail(CPI_ECUDA, "cuStreamWaitValue32 failed");
    }
    return CPI_OK;
}
}  // namespace

extern "C" {

int cpi_comm_unique_id(void* id_out) {
    if (!id_out) return cpi::capi_fail(CPI_EINVAL, "null pointer argument");
    int rc = nccl_load();
    if (rc) return rc;
    static_assert(sizeof(ncclUniqueId) == CPI_COMM_ID_BYTES, "ncclUniqueId size");
    ncclUniqueId id;
    NC(g_nccl.GetUniqueId(&id));
    memcpy(id_out, &id, sizeof id);
    return CPI_OK;
}

int cpi_comm_create(const void* id_in, int rank, int world, cpi_comm** out) {
    if (!id_in || !out) return cpi::capi_fail(CPI_EINVAL, "null pointer argument");
    if (world < 1 || world > MAX_WORLD || rank < 0 || rank >= world) return cpi::capi_fail(CPI_EINVAL, "bad rank %d / world %d", rank, world);
    int rc = nccl_load();
    if (rc) return rc;
    cpi_comm* c = new cpi_comm;
    c->rank = rank; c->world = world;
    CU(cudaGetDevice(&c->device));
    ncclUniqueId id;
    memcpy(&id, id_in, sizeof id);
    // cap the CTAs NCCL may use: its all-gather runs BESIDE a one-wave kernel (see the header of this file)
    int max_ctas = 16;
    if (const char* e = getenv("CPI_B200_NCCL_MAX_CTAS")) { const int v = atoi(e); if (v >= 0 && v <= 64) max_ctas = v; }
    if (g_nccl.CommInitRankConfig && max_ctas > 0) {
        ncclConfig_t cfg = NCCL_CONFIG_INITIALIZER;
        cfg.minCTAs = 1; cfg.maxCTAs = max_ctas;
        NC(g_nccl.CommInitRankConfig(&c->comm, world, id, rank, &cfg));
    } else {
        NC(g_nccl.CommInitRank(&c->comm, world, id, rank));
    }
    // highest priority: when batch i's exchange and batch i+1's kernel become runnable together, the exchange goes first
    int prio_least = 0, prio_greatest = 0;
    CU(cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest));
    CU(cudaStreamCreateWithPriority(&c->stream, cudaStreamNonBlocking, prio_greatest));
    CU(cudaEventCreateWithFlags(&c->entry, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&c->released, cudaEventDisableTiming));
    for (int j = 0; j < cpi_comm::NCOPY; j++) {
        CU(cudaStreamCreateWithPriority(&c->copy[j], cudaStreamNonBlocking, prio_greatest));
        CU(cudaEventCreateWithFlags(&c->copied[j], cudaEventDisableTiming));
    }
    CU(cudaEventCreateWithFlags(&c->kernel_done, cudaEventDisableTiming));
    for (int i = 0; i < cpi_comm::NBUF; i++) CU(cudaEventCreateWithFlags(&c->gathered[i], cudaEventDisableTiming));
    CU(cudaMalloc(&c->d_bar, 2 * sizeof(int)));
    CU(cudaMemset(c->d_bar, 0, 2 * sizeof(int)));
    // SM-free barriers (optional: falls back to one-element NCCL all-reduces when anything below is unavailable on ANY rank)
    if (world > 1) {
        const size_t fbytes = (2 * MAX_WORLD + 2) * sizeof(uint32_t);
        CU(cudaMalloc(&c->flags, fbytes));
        CU(cudaMemset(c->flags, 0, fbytes));
        IpcMsg mine;
        memset(&mine, 0, sizeof mine);
        static const bool nccl_barrier = getenv("CPI_B200_BARRIER") && !strcmp(getenv("CPI_B200_BARRIER"), "nccl");
        if (g_write32 && g_wait32 && !nccl_barrier && cudaIpcGetMemHandle(&mine.handle, c->flags) == cudaSuccess) {
            // self-test of the stream memory operations on this device
            uint32_t* stage = c->flags + 2 * MAX_WORLD;
            if (g_write32(c->stream, (unsigned long long)(uintptr_t)stage, 7u, 0) == 0 &&
                g_wait32(c->stream, (unsigned long long)(uintptr_t)stage, 7u, 0) == 0 && cudaStreamSynchronize(c->stream) == cudaSuccess) mine.ok = 1;
            CU(cudaMemsetAsync(stage, 0, 2 * sizeof(uint32_t), c->stream));
        }
        cudaGetLastError();
        std::vector<IpcMsg> all(world);
        void* d_x = nullptr;
        CU(cudaMalloc(&d_x, sizeof(IpcMsg) * world));
        CU(cudaMemcpyAsync((char*)d_x + sizeof(IpcMsg) * rank, &mine, sizeof mine, cudaMemcpyHostToDevice, c->stream));
        NC(g_nccl.AllGather((char*)d_x + sizeof(IpcMsg) * rank, d_x, sizeof(IpcMsg), ncclChar, c->comm, c->stream));
        CU(cudaMemcpyAsync(all.data(), d_x, sizeof(IpcMsg) * world, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        CU(cudaFree(d_x));
        int ok = 1;
        for (int p = 0; p < world; p++) ok = ok && all[p].ok == 1;
        if (ok) {
            for (int p = 0; p < world && ok; p++) {
                if (p == rank) { c->peer_flags[p] = c->flags; continue; }
                void* base = nullptr;
                if (cudaIpcOpenMemHandle(&base, all[p].handle, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = 0; break; }
                c->peer_flags_base[p] = base;
                c->peer_flags[p] = (uint32_t*)base;
            }
        }
        int agreed = 0;
        CU(cudaMemcpyAsync(c->d_bar, &ok, sizeof(int), cudaMemcpyHostToDevice, c->stream));
        NC(g_nccl.AllReduce(c->d_bar, c->d_bar + 1, 1, ncclInt, ncclMin, c->comm, c->stream));
        CU(cudaMemcpyAsync(&agreed, c->d_bar + 1, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        CU(cudaMemsetAsync(c->d_bar, 0, 2 * sizeof(int), c->stream));
        CU(cudaStreamSynchronize(c->stream));
        c->ce_barrier = agreed == 1;
    }
    *out = c;
    return CPI_OK;
}

int cpi_comm_destroy(cpi_comm* c) {
    if (!c) return CPI_OK;
    if (c->stream) cudaStreamSynchronize(c->stream);
    for (int j = 0; j < cpi_comm::NCOPY; j++) {
        if (c->copy[j]) { cudaStreamSynchronize(c->copy[j]); cudaStreamDestroy(c->copy[j]); }
        if (c->copied[j]) cudaEventDestroy(c->copied[j]);
    }
    if (c->released) cudaEventDestroy(c->released);
    for (auto& o : c->opened) cudaIpcCloseMemHandle(o.base);
    if (c->comm) g_nccl.CommDestroy(c->comm);
    if (c->stream) cudaStreamDestroy(c->stream);
    if (c->entry) cudaEventDestroy(c->entry);
    if (c->kernel_done) cudaEventDestroy(c->kernel_done);
    for (int i = 0; i < cpi_comm::NBUF; i++) if (c->gathered[i]) cudaEventDestroy(c->gathered[i]);
    if (c->d_bar) cudaFree(c->d_bar);
    for (int p = 0; p < MAX_WORLD; p++) if (c->peer_flags_base[p]) cudaIpcCloseMemHandle(c->peer_flags_base[p]);
    if (c->flags) cudaFree(c->flags);
    delete c;
    return CPI_OK;
}

int cpi_comm_rank(const cpi_comm* c) { return c ? c->rank : CPI_EINVAL; }
int cpi_comm_world(const cpi_comm* c) { return c ? c->world : CPI_EINVAL; }
int cpi_comm_sm_free_barriers(const cpi_comm* c) { return c ? (c->ce_barrier ? 1 : 0) : CPI_EINVAL; }

int cpi_comm_register(cpi_comm* c, void* gather_records, size_t bytes, int* peer_copies) {
    if (peer_copies) *peer_copies = 0;
    if (!c || !gather_records || bytes == 0) return cpi::capi_fail(CPI_EINVAL, "null pointer argument");
    int dev = 0;
    CU(cudaGetDevice(&dev));
    if (dev != c->device) return cpi::capi_fail(CPI_EINVAL, "communicator was created on device %d, current device is %d", c->device, dev);
    for (auto& r : c->regs) if (r.local == gather_records && r.bytes == bytes) { if (peer_copies) *peer_copies = r.push; return CPI_OK; }      // already registered
    Registered reg;
    reg.local = gather_records; reg.bytes = bytes;
    if (c->world == 1) { c->regs.push_back(reg); return CPI_OK; }
    // 1. export: IPC handle of the allocation + offset of the buffer inside it
    IpcMsg mine;
    memset(&mine, 0, sizeof mine);
    mine.bytes = bytes;
    static const bool no_push = getenv("CPI_B200_GATHER") && !strcmp(getenv("CPI_B200_GATHER"), "nccl");
    if (g_addr_range && !no_push) {
        unsigned long long base = 0; size_t asz = 0;
        if (g_addr_range(&base, &asz, (unsigned long long)(uintptr_t)gather_records) == 0 && base != 0 &&
            (unsigned long long)(uintptr_t)gather_records + bytes <= base + asz &&
            cudaIpcGetMemHandle(&mine.handle, (void*)(uintptr_t)base) == cudaSuccess) {
            mine.offset = (uint64_t)((unsigned long long)(uintptr_t)gather_records - base);
            mine.ok = 1;
        }
        cudaGetLastError();                                           // an export failure is not an error of this call: the buffer takes the NCCL path
    }
    // 2. exchange (collective): every rank learns every handle, and whether EVERY rank could export
    std::vector<IpcMsg> all(c->world);
    void* d_x = nullptr;
    CU(cudaMalloc(&d_x, sizeof(IpcMsg) * c->world));
    CU(cudaMemcpyAsync((char*)d_x + sizeof(IpcMsg) * c->rank, &mine, sizeof mine, cudaMemcpyHostToDevice, c->stream));
    NC(g_nccl.AllGather((char*)d_x + sizeof(IpcMsg) * c->rank, d_x, sizeof(IpcMsg), ncclChar, c->comm, c->stream));
    CU(cudaMemcpyAsync(all.data(), d_x, sizeof(IpcMsg) * c->world, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    CU(cudaFree(d_x));
    bool ok = true;
    for (int p = 0; p < c->world; p++) ok = ok && all[p].ok == 1 && all[p].bytes == bytes;
    // 3. import the peers' allocations (one mapping per allocation and process)
    int imported = ok ? 1 : 0;
    if (ok) {
        for (int p = 0; p < c->world && imported; p++) {
            if (p == c->rank) { reg.peer[p] = (char*)gather_records; continue; }
            void* base = nullptr;
            for (auto& o : c->opened) if (o.peer == p && !memcmp(&o.handle, &all[p].handle, sizeof(cudaIpcMemHandle_t))) base = o.base;
            if (!base) {
                if (cudaIpcOpenMemHandle(&base, all[p].handle, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); imported = 0; break; }
                c->opened.push_back(OpenedAlloc{p, all[p].handle, base, 0});
            }
            for (auto& o : c->opened) if (o.base == base) o.refs++;
            reg.peer_base[p] = base;
            reg.peer[p] = (char*)base + all[p].offset;
        }
    }
    // 4. agree (collective): the push path is used only if EVERY rank imported every peer -- the choice of path must never differ between ranks
    int agreed = 0;
    CU(cudaMemcpyAsync(c->d_bar, &imported, sizeof(int), cudaMemcpyHostToDevice, c->stream));
    NC(g_nccl.AllReduce(c->d_bar, c->d_bar + 1, 1, ncclInt, ncclMin, c->comm, c->stream));
    CU(cudaMemcpyAsync(&agreed, c->d_bar + 1, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemsetAsync(c->d_bar, 0, 2 * sizeof(int), c->stream));
    CU(cudaStreamSynchronize(c->stream));
    reg.push = agreed == 1;
    c->regs.push_back(reg);
    if (peer_copies) *peer_copies = reg.push ? 1 : 0;
    return CPI_OK;
}

int cpi_comm_unregister(cpi_comm* c, void* gather_records) {
    if (!c) return cpi::capi_fail(CPI_EINVAL, "null pointer argument");
    for (int j = 0; j < cpi_comm::NCOPY; j++) CU(cudaStreamSynchronize(c->copy[j]));
    CU(cudaStreamSynchronize(c->stream));                             // no exchange of this communicator in flight
    for (size_t i = 0; i < c->regs.size();) {
        if (gather_records && c->regs[i].local != gather_records) { i++; continue; }
        for (int p = 0; p < c->world; p++)
            if (c->regs[i].peer_base[p])
                for (auto& o : c->opened) if (o.base == c->regs[i].peer_base[p]) o.refs--;
        for (int k = 0; k < cpi_comm::NBUF; k++) if (c->buf[k] == c->regs[i].local) c->buf[k] = nullptr;
        c->regs.erase(c->regs.begin() + i);
    }
    for (size_t i = 0; i < c->opened.size();) {
        if (c->opened[i].refs <= 0) { cudaIpcCloseMemHandle(c->opened[i].base); c->opened.erase(c->opened.begin() + i); }
        else i++;
    }
    return CPI_OK;
}

int cpi_preintegrate_batch_sharded(cpi_comm* c, int model, int dtype, int64_t n_local, const int64_t* sample_offsets, int64_t ns_uniform,
                                   const void* samples, const void* lin, const double* sigmas, int flags, void* gather_records, void* stream) {
    if (!c || !gather_records) return cpi::capi_fail(CPI_EINVAL, "null pointer argument");
    if (n_local < 0) return cpi::capi_fail(CPI_EINVAL, "negative count");
    const int rd = cpi_record_doubles(model);
    if (rd < 0) return cpi::capi_fail(CPI_EINVAL, "model must be 1 or 2 (got %d)", model);
    if (dtype != 64 && dtype != 32) return cpi::capi_fail(CPI_EINVAL, "dtype must be 64 or 32 (got %d)", dtype);
    int dev = 0;
    CU(cudaGetDevice(&dev));
    if (dev != c->device) return cpi::capi_fail(CPI_EINVAL, "communicator was created on device %d, current device is %d", c->device, dev);
    const size_t slice = (size_t)n_local * rd * (dtype == 32 ? 4 : 8);
    cudaStream_t st = (cudaStream_t)stream;
    const Registered* reg = nullptr;
    for (auto& r : c->regs) if (r.local == gather_records && r.push && slice * c->world <= r.bytes) reg = &r;
    // this gather buffer may still be the source / destination of an earlier exchange: order the kernel behind it
    int slot = -1;
    for (int i = 0; i < cpi_comm::NBUF; i++) if (c->buf[i] == gather_records) slot = i;
    if (slot >= 0) CU(cudaStreamWaitEvent(st, c->gathered[slot], 0));
    else { slot = (c->last + 1) % cpi_comm::NBUF; c->buf[slot] = gather_records; }
    if (reg && c->world > 1 && slice > 0) {
        // barrier 1, under the kernel: the peers may write into this buffer once EVERY rank's stream has reached this call
        // (whatever the caller enqueued before it -- e.g. the consumer of the buffer's previous contents -- is then done)
        CU(cudaEventRecord(c->entry, st));
        CU(cudaStreamWaitEvent(c->stream, c->entry, 0));
        { const int brc = comm_barrier(c, 0, c->stream); if (brc) return brc; }
        CU(cudaEventRecord(c->released, c->stream));
    }
    int rc = cpi_preintegrate_batch(model, dtype, n_local, sample_offsets, ns_uniform, samples, lin, sigmas, flags,
                                    (char*)gather_records + (size_t)c->rank * slice, stream);
    if (rc) return rc;
    if (c->world > 1) {
        CU(cudaEventRecord(c->kernel_done, st));
        if (slice > 0 && reg) {
            const char* src = (const char*)gather_records + (size_t)c->rank * slice;
            const int nstreams = c->world - 1 < cpi_comm::NCOPY ? c->world - 1 : cpi_comm::NCOPY;
            for (int j = 0; j < nstreams; j++) {
                CU(cudaStreamWaitEvent(c->copy[j], c->released, 0));       // the peers have released the buffer (barrier 1) ...
                CU(cudaStreamWaitEvent(c->copy[j], c->kernel_done, 0));    // ... and this rank's slice is complete
            }
            for (int k = 1; k < c->world; k++) {                     // start with the next rank: at any moment every rank targets a different peer
                const int p = (c->rank + k) % c->world;
                CU(cudaMemcpyAsync(reg->peer[p] + (size_t)c->rank * slice, src, slice, cudaMemcpyDeviceToDevice, c->copy[(k - 1) % nstreams]));
            }
            for (int j = 0; j < nstreams; j++) {
                CU(cudaEventRecord(c->copied[j], c->copy[j]));
                CU(cudaStreamWaitEvent(c->stream, c->copied[j], 0));
            }
            // barrier 2: every rank's copies (ordered before its contribution) have landed
            { const int brc = comm_barrier(c, 1, c->stream); if (brc) return brc; }
        } else if (slice > 0) {
            CU(cudaStreamWaitEvent(c->stream, c->kernel_done, 0));
            NC(g_nccl.AllGather((const char*)gather_records + (size_t)c->rank * slice, gather_records, slice, ncclChar, c->comm, c->stream));
        }
        CU(cudaEventRecord(c->gathered[slot], c->stream));
    } else {
        CU(cudaEventRecord(c->gathered[slot], st));
    }
    c->last = slot;
    return CPI_OK;
}

int cpi_comm_wait(cpi_comm* c, void* stream) {
    if (!c) return cpi::capi_fail(CPI_EINVAL, "null pointer argument");
    if (c->last >= 0) CU(cudaStreamWaitEvent((cudaStream_t)stream, c->gathered[c->last], 0));
    return CPI_OK;
}

}  // extern "C"
