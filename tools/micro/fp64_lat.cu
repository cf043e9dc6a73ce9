// Micro-benchmark: latency / issue interval of the vector fp64 instructions the panel kernel's serial chains use.
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k_lat(double* out, long long* cyc, double seed) {
    double x = seed + threadIdx.x * 1e-9, y = 1.0000001, z = 0.25;
    long long t0, t1;
    const int N = 256;
    int s = 0;
    // dependent DFMA
    t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N; ++i) x = fma(x, y, z);
    t1 = clock64(); if (threadIdx.x == 0 && blockIdx.x == 0) cyc[s] = t1 - t0; ++s;
    // dependent DMUL
    t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N; ++i) x = x * y;
    t1 = clock64(); if (threadIdx.x == 0 && blockIdx.x == 0) cyc[s] = t1 - t0; ++s;
    // dependent DADD
    t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N; ++i) x = x + z;
    t1 = clock64(); if (threadIdx.x == 0 && blockIdx.x == 0) cyc[s] = t1 - t0; ++s;
    // dependent rsqrt
    x = fabs(x) + 1.0;
    t0 = clock64();
#pragma unroll 8
    for (int i = 0; i < N; ++i) x = rsqrt(x) + 1.0;
    t1 = clock64(); if (threadIdx.x == 0 && blockIdx.x == 0) cyc[s] = t1 - t0; ++s;
    // dependent division
    t0 = clock64();
#pragma unroll 8
    for (int i = 0; i < N; ++i) x = 1.0 / x + 1.0;
    t1 = clock64(); if (threadIdx.x == 0 && blockIdx.x == 0) cyc[s] = t1 - t0; ++s;
    // dependent sqrt
    t0 = clock64();
#pragma unroll 8
    for (int i = 0; i < N; ++i) x = sqrt(x) + 1.0;
    t1 = clock64(); if (threadIdx.x == 0 && blockIdx.x == 0) cyc[s] = t1 - t0; ++s;
    // dependent 64-bit shuffle
    t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N; ++i) x = __shfl_sync(0xffffffffu, x, (i + 1) & 31);
    t1 = clock64(); if (threadIdx.x == 0 && blockIdx.x == 0) cyc[s] = t1 - t0; ++s;
    // independent DFMA (8 chains)
    double a[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) a[u] = x + u;
    t0 = clock64();
#pragma unroll 4
    for (int i = 0; i < N; ++i) {
#pragma unroll
        for (int u = 0; u < 8; ++u) a[u] = fma(a[u], y, z);
    }
    t1 = clock64(); if (threadIdx.x == 0 && blockIdx.x == 0) cyc[s] = t1 - t0; ++s;
#pragma unroll
    for (int u = 0; u < 8; ++u) x += a[u];
    // approximate reciprocal: MUFU.RCP64H + 2 Newton steps
    t0 = clock64();
#pragma unroll 8
    for (int i = 0; i < N; ++i) {
        double r;
        asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
        double e = fma(-x, r, 1.0); r = fma(r, e, r);
        e = fma(-x, r, 1.0); r = fma(r, e, r);
        x = r + 1.0;
    }
    t1 = clock64(); if (threadIdx.x == 0 && blockIdx.x == 0) cyc[s] = t1 - t0; ++s;
    out[blockIdx.x * blockDim.x + threadIdx.x] = x;
}
int main() {
    double* out; long long* cyc;
    cudaMalloc(&out, 8 * 132 * 1024); cudaMalloc(&cyc, 8 * 64);
    const char* names[] = {"dep DFMA", "dep DMUL", "dep DADD", "dep rsqrt+add", "dep div+add", "dep sqrt+add", "dep shfl64", "8 indep DFMA chains (per 8 ops)", "dep rcp.approx+2 Newton+add"};
    for (int threads : {32, 128, 512}) {
        for (int rep = 0; rep < 2; ++rep) k_lat<<<132, threads>>>(out, cyc, 1.5);
        cudaDeviceSynchronize();
        long long h[16]; cudaMemcpy(h, cyc, sizeof(long long) * 9, cudaMemcpyDeviceToHost);
        printf("threads per CTA = %d (one CTA per SM)\n", threads);
        for (int s = 0; s < 9; ++s) printf("  %-36s %8.1f cycles per iteration\n", names[s], h[s] / 256.0);
    }
    printf("%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
