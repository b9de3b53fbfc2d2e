// FP64 roofline microbenchmarks for sm_90a (H100): the denominators of every "fraction of FP64 peak" in this repo.
//
//   dfma_tput   dependent-free DFMA streams (8 chains per thread, full occupancy)  -> TFLOP/s (2 flop per FMA)
//   dadd_tput   idem with DADD (1 flop each)
//   dfma_lat    one dependent DFMA chain in one warp                               -> cycles per DFMA
//   dmma_tput   mma.sync.aligned.m8n8k4.f64 streams (4 accumulator tiles per warp) -> TFLOP/s (2*8*8*4 flop each)
//   dmma_lat    one dependent DMMA chain in one warp                               -> cycles per DMMA
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/bin/fp64_peak tools/fp64_peak.cu
// Run (GPU box): tools/bin/fp64_peak > gpurun_out/fp64_peak.json
#include <cstdio>
#include <cstdlib>
#include <vector>

#include <cuda_runtime.h>

#define CK(x)                                                                                                          \
    do {                                                                                                               \
        cudaError_t e_ = (x);                                                                                          \
        if (e_ != cudaSuccess) {                                                                                       \
            std::fprintf(stderr, "CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__);              \
            std::exit(1);                                                                                              \
        }                                                                                                              \
    } while (0)

constexpr int ITERS = 4096;

__global__ void k_dfma_tput(double *out, double a, double b)
{
    double c0 = threadIdx.x, c1 = c0 + 1, c2 = c0 + 2, c3 = c0 + 3, c4 = c0 + 4, c5 = c0 + 5, c6 = c0 + 6, c7 = c0 + 7;
#pragma unroll 4
    for (int i = 0; i < ITERS; ++i) {
        c0 = fma(c0, a, b);
        c1 = fma(c1, a, b);
        c2 = fma(c2, a, b);
        c3 = fma(c3, a, b);
        c4 = fma(c4, a, b);
        c5 = fma(c5, a, b);
        c6 = fma(c6, a, b);
        c7 = fma(c7, a, b);
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = ((c0 + c1) + (c2 + c3)) + ((c4 + c5) + (c6 + c7));
}

__global__ void k_dadd_tput(double *out, double b)
{
    double c0 = threadIdx.x, c1 = c0 + 1, c2 = c0 + 2, c3 = c0 + 3, c4 = c0 + 4, c5 = c0 + 5, c6 = c0 + 6, c7 = c0 + 7;
#pragma unroll 4
    for (int i = 0; i < ITERS; ++i) {
        c0 = __dadd_rn(c0, b);
        c1 = __dadd_rn(c1, b);
        c2 = __dadd_rn(c2, b);
        c3 = __dadd_rn(c3, b);
        c4 = __dadd_rn(c4, b);
        c5 = __dadd_rn(c5, b);
        c6 = __dadd_rn(c6, b);
        c7 = __dadd_rn(c7, b);
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = ((c0 + c1) + (c2 + c3)) + ((c4 + c5) + (c6 + c7));
}

__global__ void k_dfma_lat(double *out, long long *cycles, double a, double b)
{
    double c = threadIdx.x;
    const long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < ITERS; ++i) {
        c = fma(c, a, b);
    }
    const long long t1 = clock64();
    out[threadIdx.x] = c;
    if (threadIdx.x == 0) {
        *cycles = t1 - t0;
    }
}

__device__ __forceinline__ void dmma(double &d0, double &d1, double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(d0), "+d"(d1)
                 : "d"(a), "d"(b));
}

__global__ void k_dmma_tput(double *out, double a, double b)
{
    double c[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        c[i] = threadIdx.x + i;
    }
#pragma unroll 2
    for (int i = 0; i < ITERS; ++i) {
        dmma(c[0], c[1], a, b);
        dmma(c[2], c[3], a, b);
        dmma(c[4], c[5], a, b);
        dmma(c[6], c[7], a, b);
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = ((c[0] + c[1]) + (c[2] + c[3])) + ((c[4] + c[5]) + (c[6] + c[7]));
}

__global__ void k_dmma_lat(double *out, long long *cycles, double a, double b)
{
    double c0 = threadIdx.x, c1 = 1.;
    const long long t0 = clock64();
#pragma unroll 8
    for (int i = 0; i < ITERS; ++i) {
        dmma(c0, c1, a, b);
    }
    const long long t1 = clock64();
    out[threadIdx.x] = c0 + c1;
    if (threadIdx.x == 0) {
        *cycles = t1 - t0;
    }
}

template <typename F>
double time_ms(F &&launch, int reps = 5)
{
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    launch();
    CK(cudaDeviceSynchronize());
    double best = 1e30;
    for (int r = 0; r < reps; ++r) {
        CK(cudaEventRecord(e0));
        launch();
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        best = ms < best ? ms : best;
    }
    return best;
}

int main()
{
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    const int sms = prop.multiProcessorCount;
    const int threads = 512, blocks = sms * 4;
    double *out;
    long long *cyc;
    CK(cudaMalloc(&out, sizeof(double) * threads * blocks));
    CK(cudaMalloc(&cyc, sizeof(long long)));
    const double total_threads = static_cast<double>(threads) * blocks;

    const double ms_fma = time_ms([&] { k_dfma_tput<<<blocks, threads>>>(out, 1.0000001, 1e-9); });
    const double ms_add = time_ms([&] { k_dadd_tput<<<blocks, threads>>>(out, 1e-9); });
    const double ms_mma = time_ms([&] { k_dmma_tput<<<blocks, threads>>>(out, 1.0000001, 1e-9); });
    long long c_fma = 0, c_mma = 0;
    k_dfma_lat<<<1, 32>>>(out, cyc, 1.0000001, 1e-9);
    CK(cudaMemcpy(&c_fma, cyc, sizeof(c_fma), cudaMemcpyDeviceToHost));
    k_dmma_lat<<<1, 32>>>(out, cyc, 1.0000001, 1e-9);
    CK(cudaMemcpy(&c_mma, cyc, sizeof(c_mma), cudaMemcpyDeviceToHost));

    const double tf_fma = total_threads * ITERS * 8. * 2. / (ms_fma * 1e-3) / 1e12;
    const double tf_add = total_threads * ITERS * 8. * 1. / (ms_add * 1e-3) / 1e12;
    // One warp-wide DMMA = 8*8*4 FMA = 512 flop; 4 per iteration per warp.
    const double tf_mma = (total_threads / 32.) * ITERS * 4. * 512. / (ms_mma * 1e-3) / 1e12;
    int clk_khz = 0;
    CK(cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0));
    std::printf("{\"gpu\": \"%s\", \"sms\": %d, \"sm_clock_max_mhz\": %.0f, \"dfma_tflops\": %.3f, \"dadd_tflops\": %.3f, "
                "\"dmma_m8n8k4_tflops\": %.3f, \"dfma_latency_cycles\": %.2f, \"dmma_latency_cycles\": %.2f, "
                "\"dfma_per_clk_per_sm_at_max_clock\": %.1f}\n",
                prop.name, sms, clk_khz / 1e3, tf_fma, tf_add, tf_mma, static_cast<double>(c_fma) / ITERS,
                static_cast<double>(c_mma) / ITERS, tf_fma * 1e12 / 2. / sms / (clk_khz * 1e3));
    return 0;
}
