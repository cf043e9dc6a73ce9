// L2 -> shared-memory delivery rate of TMA bulk copies on sm_90a, in the stage shape of k_gemm_cvy_p: one CTA per SM streams
// 53 248 B stages (two 17 408 B V slices + one 18 432 B Y block) out of a 24 MB buffer that stays resident in L2, with
// 1, 2 or 3 stages in flight per CTA, completion counted on mbarriers (complete_tx).  Nothing reads the stages: this is the
// rate at which L2 can fill shared memory, the ceiling of a GEMM fed this way.
//   unicast     : clusters of 1, each CTA fetches its whole stage
//   mc-V        : clusters of 2, each CTA fetches one V slice multicast to both plus its own Y block (k_gemm_cvy_p's pattern)
//   mc-half     : clusters of 2, each CTA fetches half of the stage multicast to both
// A CTA reuses a ring slot once both CTAs of its cluster have seen the slot's previous stage land (an empty barrier with one
// arrival per CTA), as the GEMM does.  Reported per mode: TB/s delivered into shared memory (summed over CTAs) and TB/s read
// from L2 (a multicast copy is read once), from CUDA events around the kernel, median of 5 launches.
// build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o build/l2_rate tools/micro/l2_rate.cu
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>

#define CK(x)                                                                                   \
    do {                                                                                        \
        cudaError_t e_ = (x);                                                                   \
        if (e_ != cudaSuccess) {                                                                \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
            exit(1);                                                                            \
        }                                                                                       \
    } while (0)

constexpr uint32_t VB = 32 * 68 * 8, YB = 64 * 36 * 8, STAGE = 2 * VB + YB;   // 17 408, 18 432, 53 248 B
constexpr size_t BUF = 24u << 20;
enum Mode { UNICAST = 0, MC_V = 1, MC_HALF = 2 };

__device__ __forceinline__ uint32_t su32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(su32(bar)), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void arrive_remote(uint64_t* bar, uint32_t cta) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(su32(bar)), "r"(cta));
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(r) : "memory");
}
__device__ __forceinline__ void copy(void* dst, const char* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(su32(dst)), "l"(src),
                 "r"(bytes), "r"(su32(bar)) : "memory");
}
__device__ __forceinline__ void copy_mc(void* dst, const char* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;" ::"r"(
                     su32(dst)), "l"(src), "r"(bytes), "r"(su32(bar)), "h"((uint16_t)3) : "memory");
}
__device__ __forceinline__ void csync() { asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory"); }

// one thread per CTA issues everything; the launch's cluster size is 1 (UNICAST) or 2
__global__ void k_stream(const char* buf, int iters, int depth, int mode) {
    extern __shared__ __align__(128) unsigned char smem[];
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + 3 * STAGE);
    uint64_t* empty = full + 3;
    uint32_t rank, csize;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(csize));
    if (threadIdx.x == 0) {
        for (int s = 0; s < depth; ++s) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(su32(&full[s])));
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(su32(&empty[s])), "r"(csize));
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    csync();
    if (threadIdx.x == 0) {
        const size_t nslots = BUF / STAGE;
        for (int i = 0; i < iters; ++i) {
            const int s = i % depth;
            if (i >= depth) {
                const uint32_t ph = ((i - depth) / depth) & 1;
                wait(&full[s], ph);   // this CTA's copy of the slot's previous stage has landed
                asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(su32(&empty[s])) : "memory");
                if (csize == 2) arrive_remote(&empty[s], rank ^ 1);
                wait(&empty[s], ph);  // ... and the peer's
            }
            const uint32_t tx = (mode == MC_V) ? 2 * VB + YB : STAGE;
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(su32(&full[s])), "r"(tx) : "memory");
            unsigned char* d = smem + (size_t)s * STAGE;
            const char* src = buf + ((size_t)(blockIdx.x / csize) * 7 + i) % nslots * STAGE;   // both CTAs of a cluster: same stage
            if (mode == UNICAST) {
                copy(d, src, VB, &full[s]);
                copy(d + VB, src + VB, VB, &full[s]);
                copy(d + 2 * VB, src + 2 * VB + (size_t)rank * YB, YB, &full[s]);
            } else if (mode == MC_V) {
                copy_mc(d + rank * VB, src + rank * VB, VB, &full[s]);
                copy(d + 2 * VB, src + 2 * VB + (size_t)rank * YB, YB, &full[s]);   // own Y: the neighbour stage's bytes
            } else {
                copy_mc(d + rank * (STAGE / 2), src + rank * (STAGE / 2), STAGE / 2, &full[s]);
            }
        }
        for (int i = max(iters - depth, 0); i < iters; ++i) wait(&full[i % depth], (i / depth) & 1);
    }
    csync();   // no CTA leaves while its peer may still multicast into it
}

int main(int argc, char** argv) {
    const int iters = argc > 1 ? atoi(argv[1]) : 20000;
    cudaDeviceProp p;
    CK(cudaGetDeviceProperties(&p, 0));
    char info[256] = "nvidia-smi unavailable";
    if (FILE* f = popen("nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader -i 0 2>/dev/null", "r")) {
        if (!fgets(info, sizeof info, f)) snprintf(info, sizeof info, "nvidia-smi gave nothing");
        pclose(f);
    }
    printf("GPU: %s (%d SMs); nvidia-smi: %s", p.name, p.multiProcessorCount, info);
    char* buf;
    CK(cudaMalloc(&buf, BUF + STAGE));
    CK(cudaMemset(buf, 1, BUF + STAGE));
    const size_t smem = 3 * STAGE + 6 * 8;
    CK(cudaFuncSetAttribute(k_stream, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    const char* names[] = {"unicast", "mc-V", "mc-half"};
    printf("%-8s %5s %5s %12s %12s %10s\n", "mode", "depth", "CTAs", "smem TB/s", "L2 rd TB/s", "ms");
    for (int mode = 0; mode < 3; ++mode)
        for (int depth = 1; depth <= 3; ++depth) {
            const int csize = mode == UNICAST ? 1 : 2;
            const int ctas = p.multiProcessorCount / csize * csize;
            cudaLaunchConfig_t cfg = {};
            cudaLaunchAttribute attr[1];
            attr[0].id = cudaLaunchAttributeClusterDimension;
            attr[0].val.clusterDim.x = csize;
            attr[0].val.clusterDim.y = attr[0].val.clusterDim.z = 1;
            cfg.gridDim = dim3(ctas);
            cfg.blockDim = dim3(32);
            cfg.dynamicSmemBytes = smem;
            cfg.attrs = attr;
            cfg.numAttrs = 1;
            CK(cudaLaunchKernelEx(&cfg, k_stream, (const char*)buf, iters / 10, depth, mode));   // warm-up
            CK(cudaDeviceSynchronize());
            std::vector<float> ms;
            for (int r = 0; r < 5; ++r) {
                CK(cudaEventRecord(e0));
                CK(cudaLaunchKernelEx(&cfg, k_stream, (const char*)buf, iters, depth, mode));
                CK(cudaEventRecord(e1));
                CK(cudaEventSynchronize(e1));
                float t;
                CK(cudaEventElapsedTime(&t, e0, e1));
                ms.push_back(t);
            }
            std::sort(ms.begin(), ms.end());
            const double t = ms[2] * 1e-3;
            const double delivered = (double)ctas * iters * STAGE;
            const double per_cta_read = mode == UNICAST ? STAGE : mode == MC_V ? VB + YB : STAGE / 2;
            const double l2 = (double)ctas * iters * per_cta_read;
            printf("%-8s %5d %5d %12.2f %12.2f %10.3f\n", names[mode], depth, ctas, delivered / t / 1e12, l2 / t / 1e12, ms[2]);
        }
    CK(cudaFree(buf));
    return 0;
}
