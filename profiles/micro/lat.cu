// Latency micro-benchmarks for the primitives the path-QP kernel is built from (sm_90a, H100).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o profiles/micro/lat profiles/micro/lat.cu
#include <cstdio>
#include <cuda_runtime.h>
#define N_IT 4096
__global__ void k_dfma(double *out, long long *cyc, double a, double b) {
    double x = out[threadIdx.x];
    long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N_IT; ++i) x = fma(x, a, b);
    long long t1 = clock64();
    out[threadIdx.x] = x;
    if (threadIdx.x == 0) cyc[0] = (t1 - t0);
}
__global__ void k_dfma4(double *out, long long *cyc, double a, double b) {   // 4 independent chains
    double x0 = out[threadIdx.x], x1 = x0 + 1, x2 = x0 + 2, x3 = x0 + 3;
    long long t0 = clock64();
#pragma unroll 4
    for (int i = 0; i < N_IT; ++i) { x0 = fma(x0, a, b); x1 = fma(x1, a, b); x2 = fma(x2, a, b); x3 = fma(x3, a, b); }
    long long t1 = clock64();
    out[threadIdx.x] = x0 + x1 + x2 + x3;
    if (threadIdx.x == 0) cyc[1] = (t1 - t0);
}
__global__ void k_clamp(double *out, long long *cyc, double lo, double hi, double a) {
    double x = out[threadIdx.x];
    long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N_IT; ++i) x = fmin(fmax(x * a, lo), hi);
    long long t1 = clock64();
    out[threadIdx.x] = x;
    if (threadIdx.x == 0) cyc[2] = (t1 - t0);
}
__global__ void k_ffma(float *out, long long *cyc, float a, float b) {
    float x = out[threadIdx.x];
    long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N_IT; ++i) x = fmaf(x, a, b);
    long long t1 = clock64();
    out[threadIdx.x] = x;
    if (threadIdx.x == 0) cyc[3] = (t1 - t0);
}
__global__ void k_lds(double *out, long long *cyc) {      // pointer chase in shared memory (doubles hold indices)
    extern __shared__ double sm[];
    for (int i = threadIdx.x; i < 4096; i += blockDim.x) sm[i] = (double)((i + 33) % 4096);
    __syncthreads();
    int idx = threadIdx.x;
    long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N_IT; ++i) idx = (int)sm[idx];
    long long t1 = clock64();
    out[threadIdx.x] = idx;
    if (threadIdx.x == 0) cyc[4] = (t1 - t0);
}
__global__ void k_bar(double *out, long long *cyc) {
    long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N_IT; ++i) __syncthreads();
    long long t1 = clock64();
    if (threadIdx.x == 0) cyc[5] = (t1 - t0);
    out[threadIdx.x] = 0;
}
__global__ void k_local(double *out, long long *cyc, int stride) {   // dynamically indexed local array -> LDL chain
    extern __shared__ double sm[];
    double loc[64];
    for (int i = 0; i < 64; ++i) loc[i] = (double)((i * stride + 7) & 63);
    int idx = threadIdx.x & 63;
    long long t0 = clock64();
#pragma unroll 4
    for (int i = 0; i < 1024; ++i) idx = (int)loc[idx];
    long long t1 = clock64();
    out[threadIdx.x] = idx + sm[0];
    if (threadIdx.x == 0) cyc[6] = (t1 - t0);
}
__global__ void k_dfma_tp(double *out, long long *cyc, double a, double b) {   // throughput: 8 indep chains, many warps
    double x[8];
    for (int j = 0; j < 8; ++j) x[j] = out[threadIdx.x] + j;
    long long t0 = clock64();
    for (int i = 0; i < 1024; ++i) {
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = fma(x[j], a, b);
    }
    long long t1 = clock64();
    double s = 0;
    for (int j = 0; j < 8; ++j) s += x[j];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0 && blockIdx.x == 0) cyc[7] = (t1 - t0);
}
int main() {
    double *out; long long *cyc; float *outf;
    cudaMalloc(&out, 1 << 20); cudaMalloc(&outf, 1 << 16); cudaMalloc(&cyc, 64 * 8);
    cudaMemset(out, 0, 1 << 20); cudaMemset(outf, 0, 1 << 16); cudaMemset(cyc, 0, 64 * 8);
    k_dfma<<<1, 32>>>(out, cyc, 0.999, 0.001);
    k_dfma4<<<1, 32>>>(out, cyc, 0.999, 0.001);
    k_clamp<<<1, 32>>>(out, cyc, -1.0, 1.0, 0.999);
    k_ffma<<<1, 32>>>(outf, cyc, 0.999f, 0.001f);
    k_lds<<<1, 32, 4096 * 8>>>(out, cyc);
    k_bar<<<1, 128>>>(out, cyc);
    cudaFuncSetAttribute(k_local, cudaFuncAttributeMaxDynamicSharedMemorySize, 110 * 1024);
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    k_local<<<2 * sms, 128, 110 * 1024>>>(out, cyc, 5);
    k_dfma_tp<<<sms, 512>>>(out, cyc, 0.999, 0.001);
    long long h[8];
    cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
    printf("dependent DFMA        : %.2f cycles/op\n", (double)h[0] / N_IT);
    printf("4 indep DFMA chains   : %.2f cycles/iter (4 ops)\n", (double)h[1] / N_IT);
    printf("dmul+fmax+fmin chain  : %.2f cycles/iter\n", (double)h[2] / N_IT);
    printf("dependent FFMA        : %.2f cycles/op\n", (double)h[3] / N_IT);
    printf("LDS.64 pointer chase  : %.2f cycles/load (incl. cvt)\n", (double)h[4] / N_IT);
    printf("__syncthreads 4 warps : %.2f cycles\n", (double)h[5] / N_IT);
    printf("LDL chase, 110KB smem/CTA x2: %.2f cycles/load (incl. cvt)\n", (double)h[6] / 1024);
    printf("DFMA throughput 16 warps/SM: %.3f cycles per warp-DFMA per SM-subpartition  (8192 dfma/warp in %lld cyc)\n", (double)h[7] / 8192.0 / 4.0, h[7]);
    return 0;
}
