// fp64 tensor pipe issue-rate microbenchmark for sm_90a (DMMA.8x8x4, DMMA.16x8x4, DMMA.16x8x8, DMMA.16x8x16):
//   layout check: one m16n8k8 and one m16n8k16 product against a host reference (the fragment tables of dmma16())
//   regs: registers only, ILP independent accumulators per warp, W warps per CTA, one CTA per SM, per MMA shape
//   8x8x4 32x32 / 64x32 tile: the m8n8k4 inner step (4 or 8 A + 4 B fragment LDS.64 per k4, then 16 or 32 DMMA),
//         fragments loaded right before use or one k-step ahead (software pipelined)
//   16x8xK 32x32 tile: the same 32x32 warp tile as 2 (m16) x 4 (n8) MMAs per k-step of K, fragments read from the
//         LD = 68 / 36 layouts of the bulk GEMMs with the per-register address pattern gid * LD + tig
// build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o build/dmma_rate tools/micro/dmma_rate.cu
#include <cstdio>
#include <cmath>
#include <cuda_runtime.h>
__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
// D(16x8) += A(16xK) B(Kx8):  a[i] = A[gid + 8 (i&1)][tig + 4 (i>>1)],  b[i] = B[tig + 4 i][gid],  c[i] = C[gid + 8 (i>>1)][2 tig + (i&1)]
template <int K>
__device__ __forceinline__ void dmma16(double (&c)[4], const double (&a)[K / 2], const double (&b)[K / 4]) {
    if constexpr (K == 4)
        asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
    else if constexpr (K == 8)
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
    else
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, "
                     "{%0,%1,%2,%3};"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                       "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}
// one 16 x 8 product A (16 x K, row-major) * B (K x 8, row-major) with the fragment tables above
template <int K>
__global__ void k_layout(const double* A, const double* B, double* C) {
    const int lane = threadIdx.x, gid = lane >> 2, tig = lane & 3;
    double a[K / 2], b[K / 4], c[4] = {0.0, 0.0, 0.0, 0.0};
    for (int i = 0; i < K / 2; ++i) a[i] = A[(gid + 8 * (i & 1)) * K + tig + 4 * (i >> 1)];
    for (int i = 0; i < K / 4; ++i) b[i] = B[(tig + 4 * i) * 8 + gid];
    dmma16<K>(c, a, b);
    for (int i = 0; i < 4; ++i) C[(gid + 8 * (i >> 1)) * 8 + 2 * tig + (i & 1)] = c[i];
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
template <int K, int ILP>
__global__ void k_reg16(int iters, double* out) {
    double acc[ILP][4];
    for (int i = 0; i < ILP; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.0;
    double a[K / 2], b[K / 4];
    for (int i = 0; i < K / 2; ++i) a[i] = (threadIdx.x + i) * 1e-3;
    for (int i = 0; i < K / 4; ++i) b[i] = 1.0 + (threadIdx.x + i) * 1e-4;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < ILP; ++i) dmma16<K>(acc[i], a, b);
    }
    double s = 0.0;
    for (int i = 0; i < ILP; ++i) s += acc[i][0] + acc[i][1] + acc[i][2] + acc[i][3];
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
// 32x32 warp tile as 2 x 4 m16n8kK MMAs per k-step, 32 k per iteration; A stored [k][row] (LD 68), B stored [n][k] (LD 36)
template <int K, bool PIPE>
__global__ void k_lds16(int iters, double* out) {
    extern __shared__ double sm[];
    double* sA = sm;
    double* sB = sm + 32 * LDA;
    for (int i = threadIdx.x; i < 32 * LDA + 32 * LDB; i += blockDim.x) sm[i] = 1e-3 * (i % 97);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const double* a0 = sA + (lane & 3) * LDA + (lane >> 2);
    const double* b0 = sB + (lane >> 2) * LDB + (lane & 3);
    constexpr int KS = 32 / K;
    double acc[2][4][4];
    for (int i = 0; i < 2; ++i) for (int j = 0; j < 4; ++j) for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.0;
    double af[2][K / 2], bf[4][K / 4];
    auto load = [&](int kk) {
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int r = 0; r < K / 2; ++r) af[i][r] = a0[(kk * K + 4 * (r >> 1)) * LDA + 16 * i + 8 * (r & 1)];
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int r = 0; r < K / 4; ++r) bf[j][r] = b0[j * 8 * LDB + kk * K + 4 * r];
    };
    if (PIPE) load(0);
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int kk = 0; kk < KS; ++kk) {
            if (!PIPE) load(kk);
            double ac[2][K / 2], bc[4][K / 4];
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int r = 0; r < K / 2; ++r) ac[i][r] = af[i][r];
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int r = 0; r < K / 4; ++r) bc[j][r] = bf[j][r];
            if (PIPE) load((kk + 1) % KS);
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) dmma16<K>(acc[i][j], ac[i], bc[j]);
        }
    }
    double s = 0.0;
    for (int i = 0; i < 2; ++i) for (int j = 0; j < 4; ++j) for (int e = 0; e < 4; ++e) s += acc[i][j][e];
    if (s == 12345.678) out[0] = s;
}
// -1 when the launch is refused (too many registers for the block size at 16 or 32 warps)
template <typename F>
static float timeit(F f) {
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    f();
    if (cudaGetLastError() != cudaSuccess) return -1.0f;
    cudaDeviceSynchronize();
    cudaEventRecord(e0); f(); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1); return ms;
}
template <int K>
static void layout_check(double* dbuf) {
    double A[16 * K], B[K * 8], C[16 * 8], R[16 * 8];
    for (int i = 0; i < 16 * K; ++i) A[i] = (double)((i * 7) % 13 - 6);
    for (int i = 0; i < K * 8; ++i) B[i] = (double)((i * 5) % 11 - 5);
    for (int r = 0; r < 16; ++r)
        for (int c = 0; c < 8; ++c) {
            double s = 0.0;
            for (int k = 0; k < K; ++k) s += A[r * K + k] * B[k * 8 + c];
            R[r * 8 + c] = s;
        }
    cudaMemcpy(dbuf, A, sizeof A, cudaMemcpyHostToDevice);
    cudaMemcpy(dbuf + 16 * K, B, sizeof B, cudaMemcpyHostToDevice);
    k_layout<K><<<1, 32>>>(dbuf, dbuf + 16 * K, dbuf + 32 * K);
    cudaMemcpy(C, dbuf + 32 * K, sizeof C, cudaMemcpyDeviceToHost);
    int bad = 0;
    for (int i = 0; i < 16 * 8; ++i) bad += C[i] != R[i];   // small integers: exact
    printf("layout check m16n8k%d: %s (%d of 128 entries differ)\n", K, bad ? "FAIL" : "ok", bad);
}
int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    const int sms = p.multiProcessorCount; int khz = 0; cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    double* out; cudaMalloc(&out, 8);
    double* dbuf; cudaMalloc(&dbuf, 1024 * 8);
    printf("%s, %d SMs, %.0f MHz nominal\n", p.name, sms, khz / 1e3);
    layout_check<8>(dbuf);
    layout_check<16>(dbuf);
    const int iters = 20000;
    // flop_per_mma: 512 for 8x8x4, 16 * 8 * K * 2 for 16x8xK; the last column counts 8x8x4-equivalents per clock
    auto report = [&](const char* what, int warps, double mmas_per_warp, double flop_per_mma, float ms) {
        if (ms < 0) { printf("%-34s warps/SM %2d: not launched (registers)\n", what, warps); return; }
        const double tot = mmas_per_warp * warps * sms;
        printf("%-34s warps/SM %2d: %7.3f ms  %6.2f TFLOP/s  %.3f DMMA.8x8x4-equiv/clk/SM (at nominal clock)\n", what, warps, ms,
               tot * flop_per_mma / ms / 1e9, tot * flop_per_mma / 512 / sms / (ms * 1e-3 * khz * 1e3));
    };
    // the same flop per warp in every register-only mode (20000 x 16 DMMA.8x8x4)
    auto reg16 = [&](const char* what, int w, auto kern, int k, int ilp) {
        const int it = iters * 16 * 512 / (ilp * 256 * k);
        report(what, w, (double)it * ilp, 256.0 * k, timeit([&] { kern<<<sms, w * 32>>>(it, out); }));
    };
    for (int w : {4, 8, 16, 32}) {
        report("regs 8x8x4 ILP 1", w, (double)iters * 1, 512, timeit([&] { k_reg<1><<<sms, w * 32>>>(iters, out); }));
        report("regs 8x8x4 ILP 4", w, (double)iters * 4, 512, timeit([&] { k_reg<4><<<sms, w * 32>>>(iters, out); }));
        report("regs 8x8x4 ILP 16", w, (double)iters * 16, 512, timeit([&] { k_reg<16><<<sms, w * 32>>>(iters, out); }));
        reg16("regs 16x8x4 ILP 4", w, k_reg16<4, 4>, 4, 4);
        reg16("regs 16x8x4 ILP 8", w, k_reg16<4, 8>, 4, 8);
        reg16("regs 16x8x8 ILP 4", w, k_reg16<8, 4>, 8, 4);
        reg16("regs 16x8x8 ILP 8", w, k_reg16<8, 8>, 8, 8);
        reg16("regs 16x8x16 ILP 4", w, k_reg16<16, 4>, 16, 4);
        reg16("regs 16x8x16 ILP 8", w, k_reg16<16, 8>, 16, 8);
    }
    const size_t smem = (32 * LDA + 32 * LDB) * 8;
    const int it2 = 2000;
    for (int w : {4, 8, 16}) {
        report("8x8x4 32x32 tile, LDS before use", w, (double)it2 * 8 * 16, 512, timeit([&] { k_lds<4, false><<<sms, w * 32, smem>>>(it2, out); }));
        report("8x8x4 32x32 tile, LDS pipelined", w, (double)it2 * 8 * 16, 512, timeit([&] { k_lds<4, true><<<sms, w * 32, smem>>>(it2, out); }));
        report("8x8x4 64x32 tile, LDS pipelined", w, (double)it2 * 8 * 32, 512, timeit([&] { k_lds<8, true><<<sms, w * 32, smem>>>(it2, out); }));
        report("16x8x8 32x32 tile, LDS before use", w, (double)it2 * 4 * 8, 2048, timeit([&] { k_lds16<8, false><<<sms, w * 32, smem>>>(it2, out); }));
        report("16x8x8 32x32 tile, LDS pipelined", w, (double)it2 * 4 * 8, 2048, timeit([&] { k_lds16<8, true><<<sms, w * 32, smem>>>(it2, out); }));
        report("16x8x16 32x32 tile, LDS before use", w, (double)it2 * 2 * 8, 4096, timeit([&] { k_lds16<16, false><<<sms, w * 32, smem>>>(it2, out); }));
        report("16x8x16 32x32 tile, LDS pipelined", w, (double)it2 * 2 * 8, 4096, timeit([&] { k_lds16<16, true><<<sms, w * 32, smem>>>(it2, out); }));
    }
    return 0;
}
