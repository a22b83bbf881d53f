// microbenchmark: scatter-add of 32-byte rows to random table rows: (a) 2 x red.global.add.v4.f32 per row (lane pairs),
// (b) one cp.reduce.async.bulk (TMA) per row from shared memory.
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/micro/tma_reduce tools/micro/tma_reduce.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ uint32_t rnd(uint32_t x) { x ^= x >> 16; x *= 0x85EBCA6Bu; x ^= x >> 13; x *= 0xC2B2AE35u; x ^= x >> 16; return x; }

__global__ void k_red(float* table, uint32_t rows, int iters) {
    const uint32_t gt = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t pair = gt >> 1, half = gt & 1;
    for (int i = 0; i < iters; ++i) {
        const uint32_t r = rnd(pair * 977u + i) % rows;
        float* p = table + (size_t)r * 8 + 4 * half;
        asm volatile("red.global.add.v4.f32 [%0], {%1,%1,%1,%1};" ::"l"(p), "f"(1.0f) : "memory");
    }
}
__global__ void k_tma(float* table, uint32_t rows, int iters) {
    extern __shared__ __align__(128) float sm[];
    const uint32_t gt = blockIdx.x * blockDim.x + threadIdx.x;
    float* my = sm + threadIdx.x * 8;                       // 32-byte row per thread
    for (int q = 0; q < 8; ++q) my[q] = 1.0f;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const uint32_t saddr = (uint32_t)__cvta_generic_to_shared(my);
    for (int i = 0; i < iters; ++i) {
        const uint32_t r = rnd(gt * 977u + i) % rows;
        float* p = table + (size_t)r * 8;
        asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], 32;" ::"l"(p), "r"(saddr) : "memory");
        if ((i & 15) == 15) { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
    }
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}
int main() {
    const uint32_t rows = 86000; float* t; cudaMalloc(&t, (size_t)rows * 32); cudaMemset(t, 0, (size_t)rows * 32);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1); float ms;
    int sms = 0, khz = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    const double hz = khz * 1e3;
    const int blocks = sms * 4, thr = 256, iters = 256;
    for (int rep = 0; rep < 2; ++rep) {
        cudaEventRecord(e0); k_red<<<blocks, thr>>>(t, rows, iters); cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
        double nrows = (double)blocks * thr / 2 * iters;
        printf("red.v4 x2 per row : %.3f ms  %.2f Grows/s  (%.2f rows/clk/SM at the maximum SM clock)\n", ms, nrows / ms / 1e6, nrows / (ms * 1e-3) / sms / hz);
        cudaEventRecord(e0); k_tma<<<blocks, thr, thr * 32>>>(t, rows, iters / 2); cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
        nrows = (double)blocks * thr * (iters / 2);
        printf("TMA bulk reduce   : %.3f ms  %.2f Grows/s  (%.2f rows/clk/SM)  err=%s\n", ms, nrows / ms / 1e6, nrows / (ms * 1e-3) / sms / hz, cudaGetErrorString(cudaGetLastError()));
    }
    float h[8]; cudaMemcpy(h, t, 32, cudaMemcpyDeviceToHost); printf("row0 = %g %g ... (sanity)\n", h[0], h[7]);
    return 0;
}
