// fp64 tensor pipe (DMMA.8x8x4) issue-rate microbenchmark for sm_90a:
//   mode 0: registers only, ILP independent accumulators per warp, W warps per CTA, one CTA per SM
//   mode 1: the gemm_cvy inner step (4 A + 4 B fragment LDS.64, then 16 DMMA), fragments loaded right before use
//   mode 2: the same with the next k-step's fragments loaded before the current step's DMMAs (software pipelined)
//   mode 3: 64x32 warp tile (8 A + 4 B fragments, 32 DMMA per k-step), software pipelined
// build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o build/dmma_rate tools/micro/dmma_rate.cu
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
template <int ILP>
__global__ void k_reg(int iters, double* out) {
    double acc[ILP][2];
    for (int i = 0; i < ILP; ++i) acc[i][0] = acc[i][1] = 0.0;
    double a = threadIdx.x * 1e-3, b = 1.0 + threadIdx.x * 1e-4;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < ILP; ++i) dmma(acc[i][0], acc[i][1], a, b);
    }
    double s = 0.0;
    for (int i = 0; i < ILP; ++i) s += acc[i][0] + acc[i][1];
    if (s == 12345.678) out[0] = s;
}
constexpr int LDA = 68, LDB = 36;
template <int MI, bool PIPE>
__global__ void k_lds(int iters, double* out) {
    extern __shared__ double sm[];
    double* sA = sm;                    // [32 k][LDA]  (A stored [k][row], rows 0..63)
    double* sB = sm + 32 * LDA;         // [32 n][LDB]  (B stored [n][k])
    for (int i = threadIdx.x; i < 32 * LDA + 32 * LDB; i += blockDim.x) sm[i] = 1e-3 * (i % 97);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const double* a0 = sA + (lane & 3) * LDA + (lane >> 2);
    const double* b0 = sB + (lane >> 2) * LDB + (lane & 3);
    double acc[MI][4][2];
    for (int i = 0; i < MI; ++i) for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
    double af[MI], bf[4], an[MI], bn[4];
    if (PIPE) {
#pragma unroll
        for (int i = 0; i < MI; ++i) af[i] = a0[i * 8];
#pragma unroll
        for (int j = 0; j < 4; ++j) bf[j] = b0[j * 8 * LDB];
    }
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
            if (PIPE) {
                const int kn = (kk + 1) & 7;
#pragma unroll
                for (int i = 0; i < MI; ++i) an[i] = a0[kn * 4 * LDA + i * 8];
#pragma unroll
                for (int j = 0; j < 4; ++j) bn[j] = b0[j * 8 * LDB + kn * 4];
            } else {
#pragma unroll
                for (int i = 0; i < MI; ++i) af[i] = a0[kk * 4 * LDA + i * 8];
#pragma unroll
                for (int j = 0; j < 4; ++j) bf[j] = b0[j * 8 * LDB + kk * 4];
            }
#pragma unroll
            for (int i = 0; i < MI; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) dmma(acc[i][j][0], acc[i][j][1], af[i], bf[j]);
            if (PIPE) {
#pragma unroll
                for (int i = 0; i < MI; ++i) af[i] = an[i];
#pragma unroll
                for (int j = 0; j < 4; ++j) bf[j] = bn[j];
            }
        }
    }
    double s = 0.0;
    for (int i = 0; i < MI; ++i) for (int j = 0; j < 4; ++j) s += acc[i][j][0] + acc[i][j][1];
    if (s == 12345.678) out[0] = s;
}
template <typename F>
static float timeit(F f) {
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    f(); cudaDeviceSynchronize();
    cudaEventRecord(e0); f(); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1); return ms;
}
int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    const int sms = p.multiProcessorCount; int khz = 0; cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    double* out; cudaMalloc(&out, 8);
    printf("%s, %d SMs, %.0f MHz nominal\n", p.name, sms, khz / 1e3);
    const int iters = 20000;
    auto report = [&](const char* what, int warps, double dmmas_per_warp, float ms) {
        const double tot = dmmas_per_warp * warps * sms;
        printf("%-34s warps/SM %2d: %7.3f ms  %6.2f TFLOP/s  %.3f DMMA/clk/SM (at nominal clock)\n", what, warps, ms, tot * 512 / ms / 1e9,
               tot / sms / (ms * 1e-3 * khz * 1e3));
    };
    for (int w : {4, 8, 16, 32}) {
        report("regs ILP 1", w, (double)iters * 1, timeit([&] { k_reg<1><<<sms, w * 32>>>(iters, out); }));
        report("regs ILP 2", w, (double)iters * 2, timeit([&] { k_reg<2><<<sms, w * 32>>>(iters, out); }));
        report("regs ILP 4", w, (double)iters * 4, timeit([&] { k_reg<4><<<sms, w * 32>>>(iters, out); }));
        report("regs ILP 16", w, (double)iters * 16, timeit([&] { k_reg<16><<<sms, w * 32>>>(iters, out); }));
    }
    const size_t smem = (32 * LDA + 32 * LDB) * 8;
    const int it2 = 2000;
    for (int w : {4, 8, 16}) {
        report("32x32 tile, LDS before use", w, (double)it2 * 8 * 16, timeit([&] { k_lds<4, false><<<sms, w * 32, smem>>>(it2, out); }));
        report("32x32 tile, LDS pipelined", w, (double)it2 * 8 * 16, timeit([&] { k_lds<4, true><<<sms, w * 32, smem>>>(it2, out); }));
        report("64x32 tile, LDS before use", w, (double)it2 * 8 * 32, timeit([&] { k_lds<8, false><<<sms, w * 32, smem>>>(it2, out); }));
        report("64x32 tile, LDS pipelined", w, (double)it2 * 8 * 32, timeit([&] { k_lds<8, true><<<sms, w * 32, smem>>>(it2, out); }));
    }
    return 0;
}
