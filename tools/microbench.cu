// Micro-benchmarks that size the design of the preintegration kernels on H100 (sm_90a).
// Not part of the product path.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o microbench microbench.cu
//
// Measures (all on the current device, CUDA-event timed, after warm-up):
//   1. fp64 DFMA peak (all SMs saturated)           -> roofline denominator for K1/K2 ("of measured")
//   2. fp32 FFMA peak                                -> denominator for the fp32 variant
//   3. DFMA issue rate of ONE warp per SMSP vs ILP   -> what a thread-per-window mapping can reach at low occupancy
//   4. shared-memory LDS.64 / LDS.128 bandwidth per SM
//   5. SHFL throughput per SM
//   6. sincos(double) cost per call
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

template <int ILP>
__global__ void k_dfma(double* out, int iters, double a, double b) {
    double x[ILP];
#pragma unroll
    for (int i = 0; i < ILP; i++) x[i] = threadIdx.x * 1e-3 + i;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) x[i] = fma(x[i], a, b);
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < ILP; i++) s += x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int ILP>
__global__ void k_ffma(float* out, int iters, float a, float b) {
    float x[ILP];
#pragma unroll
    for (int i = 0; i < ILP; i++) x[i] = threadIdx.x * 1e-3f + i;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < ILP; i++) x[i] = fmaf(x[i], a, b);
    }
    float s = 0;
#pragma unroll
    for (int i = 0; i < ILP; i++) s += x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int W>  // W = 1: LDS.64, W = 2: LDS.128.  The address rotates with the iteration so that nothing can be hoisted.
__global__ void k_lds(double* out, int iters) {
    extern __shared__ double sm[];
    const int n = blockDim.x * W * 8;
    for (int i = threadIdx.x; i < n; i += blockDim.x) sm[i] = i;
    __syncthreads();
    double s = 0;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int row = (j + it) & 7;
            if (W == 1) {
                s += sm[row * blockDim.x + threadIdx.x];
            } else {
                double2 v = reinterpret_cast<double2*>(sm)[row * blockDim.x + threadIdx.x];
                s += v.x + v.y;
            }
        }
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// SHFL.IDX of 32-bit values, 8 independent chains per thread, source lane = a per-lane table (like the trio gathers of the
// tri-lane kernels: lane 3w+c reads 3w+(c+1)%3)
__global__ void k_shfl(double* out, int iters) {
    int v[8];
    const int lane = threadIdx.x & 31;
    const int src = lane < 30 ? (lane / 3) * 3 + (lane % 3 + 1) % 3 : lane;
#pragma unroll
    for (int i = 0; i < 8; i++) v[i] = threadIdx.x + i;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < 8; i++) v[i] = __shfl_sync(0xffffffffu, v[i], src) + 1;
    }
    int s = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) s += v[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// Mixed: per iteration NF dependent-free DFMA (8 chains) + NS double shuffles (2 SHFL each) + NL LDS.64 -- do the pipes overlap?
template <int NF, int NS, int NL>
__global__ void k_mix(double* out, int iters, double a, double b) {
    extern __shared__ double sm[];
    for (int i = threadIdx.x; i < blockDim.x * 8; i += blockDim.x) sm[i] = i * 1e-9;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int src = lane < 30 ? (lane / 3) * 3 + (lane % 3 + 1) % 3 : lane;
    double x[8], y[4] = {1, 2, 3, 4}, l = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) x[i] = threadIdx.x * 1e-3 + i;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int r = 0; r < (NF > NS ? (NF > NL ? NF : NL) : (NS > NL ? NS : NL)); r++) {
            if (r < NF) x[r & 7] = fma(x[r & 7], a, b);
            if (r < NS) y[r & 3] = __shfl_sync(0xffffffffu, y[r & 3], src);
            if (r < NL) l += sm[((r + it) & 7) * blockDim.x + threadIdx.x];
        }
    }
    double s = l;
#pragma unroll
    for (int i = 0; i < 8; i++) s += x[i];
#pragma unroll
    for (int i = 0; i < 4; i++) s += y[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void k_sincos(double* out, int iters, double x0) {
    double x = x0 + threadIdx.x * 1e-4, acc = 0;
    for (int it = 0; it < iters; it++) {
        double s, c;
        sincos(x, &s, &c);
        acc += s * c;
        x += 1e-3;
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

__global__ void k_rcp(double* out, int iters, double x0) {
    double x = x0 + threadIdx.x * 1e-4, acc = 0;
    for (int it = 0; it < iters; it++) { acc += 1.0 / x; x += 1e-3; }
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

template <typename F>
float time_ms(F launch, int reps = 5) {
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    launch(); launch();
    CK(cudaDeviceSynchronize());
    float best = 1e30f;
    for (int r = 0; r < reps; r++) {
        CK(cudaEventRecord(e0));
        launch();
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
        if (ms < best) best = ms;
    }
    CK(cudaGetLastError());
    return best;
}

int main() {
    cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
    int sms = p.multiProcessorCount;
    int clk_khz = 0; cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
    printf("{\"device\": \"%s\", \"sms\": %d, \"clock_khz_attr\": %d}\n", p.name, sms, clk_khz);
    double* out; CK(cudaMalloc(&out, sizeof(double) * 1024 * 1024 * 4));

    // 1. DFMA peak: 8 blocks per SM x 256 threads, ILP 8
    {
        const int iters = 20000, blocks = sms * 8, thr = 256;
        float ms = time_ms([&] { k_dfma<8><<<blocks, thr>>>(out, iters, 1.0000001, 1e-9); });
        double flops = 2.0 * 8 * (double)iters * blocks * thr;
        printf("{\"test\": \"dfma_peak\", \"ms\": %.3f, \"tflops\": %.3f}\n", ms, flops / ms * 1e-9);
        // sustained: ~2 s loop
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        int n = (int)(2000.0 / ms) + 1;
        cudaEventRecord(e0);
        for (int i = 0; i < n; i++) k_dfma<8><<<blocks, thr>>>(out, iters, 1.0000001, 1e-9);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        float tot; cudaEventElapsedTime(&tot, e0, e1);
        printf("{\"test\": \"dfma_sustained\", \"ms_total\": %.1f, \"tflops\": %.3f}\n", tot, flops * n / tot * 1e-9);
    }
    // 2. FFMA peak
    {
        const int iters = 40000, blocks = sms * 8, thr = 256;
        float ms = time_ms([&] { k_ffma<8><<<blocks, thr>>>((float*)out, iters, 1.0000001f, 1e-9f); });
        double flops = 2.0 * 8 * (double)iters * blocks * thr;
        printf("{\"test\": \"ffma_peak\", \"ms\": %.3f, \"tflops\": %.3f}\n", ms, flops / ms * 1e-9);
    }
    // 3. one warp per SMSP (4 warps/SM in one block), vary ILP; and 1,2,4,8,16 warps per SM at ILP 8
#define RUN_ILP(I) { const int iters = 20000; \
        float ms = time_ms([&] { k_dfma<I><<<sms, 128>>>(out, iters, 1.0000001, 1e-9); }); \
        double per = ms * 1e-3 / ((double)iters * I); \
        printf("{\"test\": \"dfma_1warp_per_smsp\", \"ilp\": %d, \"ns_per_warp_dfma\": %.4f, \"tflops\": %.3f}\n", I, per * 1e9, 2.0 * I * iters * sms * 128 / ms * 1e-9); }
    RUN_ILP(1) RUN_ILP(2) RUN_ILP(4) RUN_ILP(8) RUN_ILP(16)
    for (int thr = 32; thr <= 1024; thr *= 2) {
        const int iters = 20000;
        float ms = time_ms([&] { k_dfma<8><<<sms, thr>>>(out, iters, 1.0000001, 1e-9); });
        printf("{\"test\": \"dfma_threads_per_sm\", \"threads\": %d, \"ilp\": 8, \"tflops\": %.3f}\n", thr, 2.0 * 8 * iters * sms * thr / ms * 1e-9);
    }
    // 4. LDS bandwidth per SM (dynamic smem > 48 KB needs the opt-in attribute: the round-1 run died here)
    CK(cudaFuncSetAttribute(k_lds<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CK(cudaFuncSetAttribute(k_lds<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    for (int thr = 64; thr <= 1024; thr *= 2) {
        const int iters = 20000;
        float ms1 = time_ms([&] { k_lds<1><<<sms, thr, thr * 8 * 8>>>(out, iters); });
        float ms2 = time_ms([&] { k_lds<2><<<sms, thr, thr * 16 * 8>>>(out, iters); });
        double b1 = 8.0 * 8 * iters * thr, b2 = 16.0 * 8 * iters * thr;  // bytes per SM
        printf("{\"test\": \"lds\", \"threads\": %d, \"lds64_GBps_per_sm\": %.1f, \"lds64_B_per_clk_per_sm\": %.1f, \"lds128_GBps_per_sm\": %.1f, \"lds128_B_per_clk_per_sm\": %.1f}\n",
               thr, b1 / ms1 * 1e-6, b1 / ms1 * 1e-6 / (clk_khz * 1e-6), b2 / ms2 * 1e-6, b2 / ms2 * 1e-6 / (clk_khz * 1e-6));
    }
    // 5. SHFL.b32 throughput (a double costs two)
    for (int thr = 128; thr <= 1024; thr *= 2) {
        const int iters = 20000;
        float ms = time_ms([&] { k_shfl<<<sms, thr>>>(out, iters); });
        double lanes = 8.0 * iters * thr;
        printf("{\"test\": \"shfl_b32\", \"threads\": %d, \"Glanes_per_s_per_sm\": %.2f, \"lanes_per_clk_per_sm\": %.2f}\n", thr, lanes / ms * 1e-6, lanes / ms * 1e-6 / (clk_khz * 1e-6));
    }
    // 5b. pipe overlap at 512 threads/SM (4 warps per SMSP): time per iteration-warp in clocks for DFMA only, SHFL only, LDS only and mixes
#define RUN_MIX(NF, NS, NL) { const int iters = 5000, thr = 512; \
        float ms = time_ms([&] { k_mix<NF, NS, NL><<<sms, thr, thr * 64>>>(out, iters, 1.0000001, 1e-9); }); \
        printf("{\"test\": \"mix\", \"threads\": %d, \"dfma\": %d, \"shfl_b32\": %d, \"lds64\": %d, \"clk_per_iter_per_sm\": %.1f}\n", thr, NF, NS, NL, ms * 1e-3 * clk_khz * 1e3 / iters); }
    RUN_MIX(32, 0, 0) RUN_MIX(0, 16, 0) RUN_MIX(0, 0, 16) RUN_MIX(32, 16, 0) RUN_MIX(32, 0, 16) RUN_MIX(0, 16, 16) RUN_MIX(32, 16, 16) RUN_MIX(32, 8, 8) RUN_MIX(32, 32, 0)
    // 6. sincos(double), 1/x (double)
    for (int thr = 128; thr <= 1024; thr *= 4) {
        const int iters = 4000;
        float ms = time_ms([&] { k_sincos<<<sms, thr>>>(out, iters, 0.01); });
        printf("{\"test\": \"sincos_f64\", \"threads\": %d, \"clk_per_warp_call_per_smsp\": %.1f, \"Gcalls_per_s\": %.3f}\n", thr, ms * 1e-3 * clk_khz * 1e3 / iters / (thr / 128.0), (double)iters * thr * sms / ms * 1e-6);
        float ms2 = time_ms([&] { k_rcp<<<sms, thr>>>(out, iters, 0.01); });
        printf("{\"test\": \"rcp_f64\", \"threads\": %d, \"clk_per_warp_call_per_smsp\": %.1f}\n", thr, ms2 * 1e-3 * clk_khz * 1e3 / iters / (thr / 128.0));
    }
    return 0;
}
