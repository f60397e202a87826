// Microbenchmark: peak FP64 FMA and FP64 tensor (mma.sync.m8n8k4.f64) throughput on this GPU.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/mb_fp64 tools/microbench_fp64.cu
#include <cstdio>
#include <cuda_runtime.h>

__global__ void dfma_kernel(double *out, int iters) {
    double a[16], x = 1.0000001 + threadIdx.x * 1e-9, y = 0.9999999;
#pragma unroll
    for (int i = 0; i < 16; i++) a[i] = i * 0.1;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < 16; i++) a[i] = fma(a[i], x, y);
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) s += a[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void dmma_kernel(double *out, int iters) {
    double c[8][2];
#pragma unroll
    for (int i = 0; i < 8; i++) { c[i][0] = 0; c[i][1] = 0; }
    double a = 1.0 + threadIdx.x * 1e-6, b = 1e-3;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < 8; i++)
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(c[i][0]), "+d"(c[i][1]) : "d"(a), "d"(b));
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) s += c[i][0] + c[i][1];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    printf("device %s sms=%d clock=%d kHz\n", p.name, p.multiProcessorCount, p.clockRate);
    double *out; cudaMalloc(&out, 148 * 8 * 1024 * sizeof(double));
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int threads : {256, 512, 1024}) {
        int blocks = p.multiProcessorCount * (2048 / threads);
        int iters = 20000;
        dfma_kernel<<<blocks, threads>>>(out, 100);
        cudaEventRecord(e0); dfma_kernel<<<blocks, threads>>>(out, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        double fl = 2.0 * 16 * iters * (double)blocks * threads;
        printf("DFMA threads/blk=%d: %.2f TFLOP/s (%.3f ms)\n", threads, fl / ms / 1e9, ms);
        dmma_kernel<<<blocks, threads>>>(out, 100);
        cudaEventRecord(e0); dmma_kernel<<<blocks, threads>>>(out, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1);
        fl = 2.0 * 8 * 8 * 4 * 8 * iters * (double)blocks * (threads / 32);
        printf("DMMA m8n8k4 threads/blk=%d: %.2f TFLOP/s (%.3f ms)\n", threads, fl / ms / 1e9, ms);
    }
    printf("%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
