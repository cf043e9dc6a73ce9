// dhqr_api.cu — context, workspace, panel/update drivers and the C-ABI of libdhqr.so.
// See include/dhqr.h for the contract; each entry point names the reference method it replaces
// (S:n = line n of the reference's src/DistributedHouseholderQR.jl).
#include "../../include/dhqr.h"

#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include <algorithm>
#include <memory>
#include <type_traits>
#include <utility>
#include <vector>

#include "dhqr_kernels.cuh"
#include "dhqr_wide.cuh"
#include "dhqr_complex.cuh"
#include "dhqr_qrcp.cuh"
#include "dhqr_append.cuh"
#include "dhqr_batched.cuh"

using namespace dhqr;

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static int set_err(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
#define CU(call)                                                                                         \
    do {                                                                                                 \
        cudaError_t e_ = (call);                                                                         \
        if (e_ != cudaSuccess)                                                                           \
            return set_err(1000 + (int)e_, "%s failed at %s:%d: %s", #call, __FILE__, __LINE__, cudaGetErrorString(e_)); \
    } while (0)
#define TRY(call)          \
    do {                   \
        int rc_ = (call);  \
        if (rc_) return rc_; \
    } while (0)

// ------------------------------------------------------------------------------------------------
// NCCL, loaded lazily so that single-GPU use needs no NCCL at all
// ------------------------------------------------------------------------------------------------
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;
enum { ncclFloat64 = 8, ncclInt64 = 4, ncclSum = 0 };
struct NcclApi {
    void* lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*Broadcast)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Send)(const void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
static NcclApi g_nccl;
static int load_nccl() {
    if (g_nccl.lib) return 0;
    // DHQR_NCCL_LIBRARY names the library to use.  It is opened privately (RTLD_LOCAL), so its symbols never take the place
    // of those of a libnccl.so.2 the process already has (torch's), and the library resolves its ten entry points in it alone.
    const char* path = getenv("DHQR_NCCL_LIBRARY");
    if (path && *path) {
        g_nccl.lib = dlopen(path, RTLD_NOW | RTLD_LOCAL);
        if (!g_nccl.lib) return set_err(2001, "cannot dlopen DHQR_NCCL_LIBRARY=%s: %s", path, dlerror());
    }
    // Otherwise an already-loaded libnccl.so.2 (e.g. the one bundled with torch) is reused by soname.
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* nm : names) {
        if (g_nccl.lib) break;
        g_nccl.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
    }
    if (!g_nccl.lib) return set_err(2001, "cannot dlopen libnccl.so.2: %s", dlerror());
#define SYM(field, name)                                                       \
    *(void**)(&g_nccl.field) = dlsym(g_nccl.lib, name);                        \
    if (!g_nccl.field) return set_err(2002, "libnccl lacks symbol %s", name);
    SYM(GetUniqueId, "ncclGetUniqueId")
    SYM(CommInitRank, "ncclCommInitRank")
    SYM(CommDestroy, "ncclCommDestroy")
    SYM(Broadcast, "ncclBroadcast")
    SYM(AllGather, "ncclAllGather")
    SYM(Send, "ncclSend")
    SYM(Recv, "ncclRecv")
    SYM(GroupStart, "ncclGroupStart")
    SYM(GroupEnd, "ncclGroupEnd")
    SYM(GetErrorString, "ncclGetErrorString")
#undef SYM
    return 0;
}
#define NC(call)                                                                                              \
    do {                                                                                                      \
        ncclResult_t r_ = (call);                                                                             \
        if (r_ != 0) return set_err(3000 + (int)r_, "%s failed at %s:%d: %s", #call, __FILE__, __LINE__, g_nccl.GetErrorString(r_)); \
    } while (0)

// ------------------------------------------------------------------------------------------------
// context
// ------------------------------------------------------------------------------------------------
static inline int64_t rup(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

// Owns one device allocation of n elements of T and frees it with its owner.  Converts to the raw pointer (null when empty),
// which is what kernels and the CUDA API take.
template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    DevBuf() = default;
    DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p, o.p); std::swap(n, o.n); return *this; }
    ~DevBuf() { release(); }
    operator T*() const { return p; }
    cudaError_t release() {
        T* q = p;
        p = nullptr;
        n = 0;
        return q ? cudaFree(q) : cudaSuccess;
    }
    // `need` elements, contents undefined
    int alloc(size_t need) {
        CU(release());
        CU(cudaMalloc((void**)&p, need * sizeof(T)));
        n = need;
        return 0;
    }
    // Grows to at least `need` elements.  The zero fill goes on `st`, the stream of the call that needs the buffer: a synchronous
    // cudaMemset would run on the legacy default stream, which a non-blocking caller stream is not ordered after.
    int ensure(size_t need, cudaStream_t st) {
        if (n >= need && p) return 0;
        CU(release());
        CU(cudaMalloc((void**)&p, need * sizeof(T)));
        CU(cudaMemsetAsync(p, 0, need * sizeof(T), st));
        n = need;
        return 0;
    }
};

// Owns one CUDA stream or event and destroys it with its owner.  Converts to the raw handle (null when empty).
template <typename H, cudaError_t (*Destroy)(H)>
struct Owned {
    H h = nullptr;
    Owned() = default;
    Owned(Owned&& o) noexcept : h(o.h) { o.h = nullptr; }
    Owned& operator=(Owned&& o) noexcept { std::swap(h, o.h); return *this; }
    ~Owned() { reset(); }
    operator H() const { return h; }
    void reset() {
        if (h) Destroy(h);
        h = nullptr;
    }
};
struct Stream : Owned<cudaStream_t, cudaStreamDestroy> {
    cudaError_t create() { reset(); return cudaStreamCreateWithFlags(&h, cudaStreamNonBlocking); }
    cudaError_t create(int priority) { reset(); return cudaStreamCreateWithPriority(&h, cudaStreamNonBlocking, priority); }
};
struct Event : Owned<cudaEvent_t, cudaEventDestroy> {
    cudaError_t create(unsigned flags) { reset(); return cudaEventCreateWithFlags(&h, flags); }
};

struct dhqr_context {
    int device = 0, sms = 0;
    int rank = 0, nranks = 1;
    ncclComm_t comm = nullptr;
    // options
    int nb = 128, panel_ctas = 0, sync = 0;
    // workspace
    // three V buffers (panels k, k+1 and the one being broadcast live at the same time under look-ahead) and two
    // workspace sets (set 0: trailing update on the caller's stream; set 1: panel chain on the high-priority stream)
    DevBuf<double> vpk2[6];                                             // packed V [chunk][128][68]; [3..5]: catch-up of late column chunks (host entry)
    struct WSet {
        DevBuf<double> wpart;                                           // gemm_vta partials
        DevBuf<double> wsum;                                            // reduced Wext
        DevBuf<double> ypk;                                             // packed Y = -T'W
        DevBuf<double> linv;                                            // [128*128]
    } ws[6];                                                            // [2]: the chain's second apply (columns of panel k+2) on its own stream; [3..5]: catch-up (host entry)
    DevBuf<double> linv_all;                                            // T' of every outer panel of the factorisation in flight (look-ahead): slot k = panel k
    double* tslot(int k) const { return linv_all.p + (size_t)k * 128 * 128; }
    DevBuf<double> gram_all;                                            // G = V_b' V_a of each panel pair (slot = first panel of the pair)
    double* gslot(int k) const { return gram_all.p + (size_t)k * 128 * 128; }
    DevBuf<double> vpkb[3];                                             // V of the second panel of a pair, ring as vpk2[0..2]
    int64_t pair_units = 0;                                             // statistics: panel pairs applied as one 256-wide block
    Stream hp_stream;                                                   // stream of the panel chain (high priority)
    Stream comm_stream;                                                 // collectives of the look-ahead schedule (high priority)
    Stream aux_stream;                                                  // small side kernels of the wide chain (Rt = R2 R1, k_trecon), high priority
    Event ev_aux[4];
    Stream hp2_stream;                                                  // the chain's second apply (V_k -> columns of panel k+2), high priority
    int host_trace = 0;                                                 // option: print a stage timeline of dhqr_qr_host_f64 to stderr
    int lookahead = 1;
    int la_trace = 0;                                                   // keep timing events of the look-ahead schedule
    std::vector<float> la_times;                                        // [k][3]: panel k done (hp), next k signalled (st), bulk k done (st), ms since start
    // option chain_wait_trace (look-ahead schedule): CUDA events right before and after every launch on hp, hp2 and aux, and
    // the CwtScope stamps of the same launch, so that the time a launch was ready but had no SM can be told from its run time
    int chain_wait_trace = 0;
    DevBuf<unsigned long long> cwt_stamps;                              // [CWT_MAX][2]: first CTA start, last warp end (%globaltimer ns)
    int cwt_unit = 0;                                                   // unit of the look-ahead step being enqueued
    struct CwtRec { int unit, stream, cls; Event e0, e1; };
    std::vector<CwtRec> cwt_recs;
    std::vector<double> cwt_rows;                                       // [launch][6]: unit, stream, class, event span, stamp span, wait (ms)
    DevBuf<unsigned long long> cells;                                   // panel exchange cells [IB+1][MAXG+1][IB][2]
    uint32_t ll_epoch = 0;
    DevBuf<unsigned long long> cells2;                                  // exchange cells of the panel kernel's fast path
    DevBuf<int> fast_stats;                                             // [2] fast / fallback panel counters
    int panel_fast = 1;
    int bs_wave = 1;                                                    // back-substitution as one wavefront launch per right-hand side
    int bs_wave_max_ctas = 0;                                           // co-residency limit of k_backsolve_wave on this device
    int fs_wave_max_ctas = 0;                                           // ... and of k_forwardsolve_wave
    DevBuf<unsigned long long> bs_cells;                                // x cells of the wavefronts ([block][32][2 words])
    size_t bs_blocks() const { return bs_cells.n / 64; }
    uint32_t bs_epoch = 0;
    int unblocked_wave = 1;                                             // nb = 1, m <= 8192: the column loop as one persistent launch
    DevBuf<unsigned int> uw_flags; unsigned int uw_epoch = 0;
    int fuse_house = 1;                                                 // nb = 1: next reflector formed inside the apply kernel (one launch per column)
    int cvy_persist = 4;                                                // 128-wide gemm_cvy: consecutive tiles per CTA (0: one tile per CTA); 4 is fastest on an H100 at one CTA per SM
    DevBuf<long long> panel_trace;                                      // optional k_panel clock stamps (option "panel_trace")
    // 128-column panel chain (dhqr_wide.cuh)
    int wide_panel = 1;                                                 // option: factor full aligned outer panels with CholeskyQR2 + reconstruction
    DevBuf<WideCtl> wctl;                                               // device control words (first refused panel, guards of the panel in flight)
    DevBuf<double> wbuf;                                                // R1, R2, X2, Rt, Y3 (plain 128x128) + XL, XL3 (rmul operand layout)
    int64_t wide_panels = 0, wide_redone = 0;                           // statistics: panels factored by the wide chain / factorisations restarted
    double wide_kappa = 1000.0;                                         // guard on ||D R1^{-1}||_F of the first Cholesky factor (option "wide_kappa")
    DevBuf<long long> wstamps;                                          // clock64 stamps of the single-CTA kernels (option "wide_trace")
    int wide_trace = 0;
    DevBuf<unsigned long long> gtr_rows;                                // option "gemm_trace": [GTR_MAX_CTAS][GTR_WORDS] bulk-GEMM buckets
    size_t gtr_used = 0;                                                // rows handed to traced launches since the option was set
    size_t gtr_dropped = 0;                                             // launches left untraced for want of rows
    int gemm_trace = 0;
    // Q'b / Qb with one right-hand side: T' of every local panel (computed before the sweep), per-CTA partials of V'b, y, ticket
    DevBuf<double> qt_T;
    DevBuf<double> qt_part;
    DevBuf<unsigned int> qt_ticket;
    int qt_vec = 1;                                                     // option: use it (0: the GEMM-shaped block update also for one right-hand side)
    DevBuf<double> v1;                                                  // unblocked path: v
    DevBuf<double> xbuf;                                                // back-substitution output
    DevBuf<double> xfer;                                                // a right-hand-side block packed for the rank-to-rank hand-over
    // pivoted factorisation (dhqr_qrcp.cuh): vn1, vn2, F, the column in flight and the partials of both reductions; renorm
    // flags; scalars of the reflector in flight, the pivot ticket and the renorm counter
    DevBuf<double> qp_buf;
    DevBuf<int> qp_flag;
    DevBuf<QrcpCtl> qp_ctl;
    DevBuf<double> hostA;                                               // device staging for _host_ entry points
    DevBuf<double> hostB;
    DevBuf<int64_t> d_i64;                                              // small int64 scratch (partition exchange)
    int64_t launches = 0;
    Stream copy_stream;                      // compute stream of the _host_ entry points
    Stream d2h_stream;                       // drains finished panels to the host while the factorisation continues
    Stream h2d_stream;                       // uploads the later column chunks while the first ones are being factored
    Stream cu_stream[3];                     // catch-up: reflectors of finished panels applied to a column chunk that arrived late (chunks alternate)
    // dhqr_qr_host_f64 -> look-ahead driver: column chunks still on their way to the device.  Chunk j = global columns [c0, c1),
    // usable once `ev` has fired, joins the trailing matrix at step `join` (after a catch-up with the reflectors of panels < join)
    struct UpChunk { int64_t c0, c1; cudaEvent_t ev; int join; };
    std::vector<UpChunk> up_chunks;
    int host_chunk = 512;                    // option: columns per upload chunk (0: one upload, no overlap)
    int host_first = 0;                      // option: columns of the first upload (0: three panels)
    int host_h2d_gbs = 50, host_tflops = 27; // option: what the join-step planner assumes about the link and the device
    int host_chain_us = 300;                 // option: ... and about the duration of a step of the schedule while the window is narrow
    int host_cu_streams = 3;                 // option: catch-up streams in use (1..3)
    std::vector<Event> panel_events;
    // set by dhqr_qr_host_f64: finished columns are copied back as soon as their panel is final
    double* mirror_host = nullptr;
    int64_t mirror_lda = 0;
    // kernel attribute state
    bool attrs_set = false;
    // per-kernel-class CUDA-event profiling (option "profile")
    int profile = 0;
    struct ProfRec { int slot; Event e0, e1; };
    struct ProfSlot { const char* name; double ms = 0.0; int64_t count = 0; double work = 0.0; };
    std::vector<ProfRec> prof_pending;
    std::vector<ProfSlot> prof_slots;
};

static constexpr int NBMAX = 128;
static constexpr int CWT_MAX = 8192;   // traced launches per factorisation (option chain_wait_trace)
static constexpr size_t GTR_MAX_CTAS = (size_t)1 << 17;   // traced CTAs of k_gemm_vta / k_gemm_cvy_p (option gemm_trace), 8 MB
static constexpr int MAXCTAS_FACTOR = 3;

// gemm tile configurations
static constexpr int G1_BN = 64, G1_NPW = 2;                // gemm_vta<128>: 128 x 64 tile, 8 MMA + 2 TMA warps
static constexpr int G1S_BN = 128, G1S_NPW = 4;             // gemm_vta<32> : 32 x 128 tile, 4 MMA + 4 TMA warps
static constexpr int G2_BM = 128, G2_BN = YT;               // gemm_cvy: 128 x 64 tile, 8 MMA + 1 TMA warps

static size_t smem_g1(int nbp, int bn) { return (size_t)2 * (nbp + bn) * LD1 * 8 + 4 * 8; }
static size_t smem_g2() { return (size_t)2 * (2 * KC * LD1 + G2_BN * LDK) * 8 + 4 * 8; }
// the operand ring, the C tile, 2 barriers per stage + cfull, cdone and the gate word: 226 KB (one CTA per SM)
static size_t smem_g2p() { return (size_t)(CVYP_STAGES * (2 * KC * LD1 + G2_BN * LDK) + G2_BN * LDCT) * 8 + (2 * CVYP_STAGES + 3) * 8; }
static size_t smem_tinv(int nbp) { return ((size_t)nbp * (nbp + 1) + 4 * 32 * 33 + (nbp == 128 ? 64 * 65 : 0)) * 8; }
static size_t smem_ymake(int nbp) { return ((size_t)nbp * nbp + YCOLS * nbp) * 8; }

#define K_G1_128 k_gemm_vta<128, G1_BN, 4, 2, G1_NPW>
#define K_G1_32 k_gemm_vta<32, G1S_BN, 1, 4, G1S_NPW>
#define K_G1_128T k_gemm_vta_traced<128, G1_BN, 4, 2, G1_NPW>
#define K_G1_32T k_gemm_vta_traced<32, G1S_BN, 1, 4, G1S_NPW>

static int set_attrs(dhqr_context* c) {
    if (c->attrs_set) return 0;
    CU(cudaFuncSetAttribute(K_G1_128, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_g1(128, G1_BN)));
    CU(cudaFuncSetAttribute(K_G1_32, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_g1(32, G1S_BN)));
    CU(cudaFuncSetAttribute(K_G1_128T, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_g1(128, G1_BN)));
    CU(cudaFuncSetAttribute(K_G1_32T, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_g1(32, G1S_BN)));
    CU(cudaFuncSetAttribute(k_gemm_cvy, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_g2()));
    CU(cudaFuncSetAttribute(k_gemm_cvy, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    CU(cudaFuncSetAttribute(k_gemm_cvy_p, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_g2p()));
    CU(cudaFuncSetAttribute(k_gemm_cvy_p, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    CU(cudaFuncSetAttribute(k_gemm_cvy_p_traced, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_g2p()));
    CU(cudaFuncSetAttribute(k_gemm_cvy_p_traced, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    CU(cudaFuncSetAttribute(k_gram_sym, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_GRAM_SYM));
    CU(cudaFuncSetAttribute(k_pack_gram, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_GRAM_SYM));
    CU(cudaFuncSetAttribute(k_tinv<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_tinv(128)));
    CU(cudaFuncSetAttribute(k_tinv<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_tinv(32)));
    CU(cudaFuncSetAttribute(k_ymake<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_ymake(128)));
    CU(cudaFuncSetAttribute(k_ymake<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_ymake(32)));
    CU(cudaFuncSetAttribute(k_tinv<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_tinv(128)));
    CU(cudaFuncSetAttribute(k_ymake<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_ymake(128)));
    CU(cudaFuncSetAttribute(k_ymake2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_YMAKE2));
    CU(cudaFuncSetAttribute(k_panel, cudaFuncAttributeMaxDynamicSharedMemorySize, 184 * 1024));
    CU(cudaFuncSetAttribute(k_tp_panel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 184 * 1024));
    CU(cudaFuncSetAttribute(k_tp_panel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 184 * 1024));
    CU(cudaFuncSetAttribute(k_chol128, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_WIDE1));
    CU(cudaFuncSetAttribute(k_hr128, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_WIDE1));
    CU(cudaFuncSetAttribute(k_vpk_rmul, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_RMUL));
    CU(cudaFuncSetAttribute(k_trimm128, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_TRIMM));
    CU(cudaFuncSetAttribute(k_trimm_z, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_TRIMM));
    CU(cudaFuncSetAttribute(k_trecon, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_TRECON));
    CU(cudaFuncSetAttribute(k_apply1_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    c->attrs_set = true;
    return 0;
}

static int prof_slot(dhqr_context* c, const char* name) {
    for (size_t i = 0; i < c->prof_slots.size(); ++i)
        if (!strcmp(c->prof_slots[i].name, name)) return (int)i;
    dhqr_context::ProfSlot s;
    s.name = name;
    c->prof_slots.push_back(s);
    return (int)c->prof_slots.size() - 1;
}

// chain_wait_trace: where a launch's kernel leaves its stamps (null: the launch is not traced)
using CwtSlot = unsigned long long*;

// Every kernel launch goes through here.  `enqueue(cwt)` launches on `st`: a <<<>>> launch returns nothing (its error is read
// here, with cudaGetLastError), a launch through the runtime API returns its error.  Kernels without a CwtScope ignore the stamp
// slot `cwt`.  Around the launch go the CUDA-event brackets of option chain_wait_trace (on the chain's streams) and of option
// "profile" (class `what`, credited with `work`); the launch is counted, and under option "sync" waited for.  A failed launch
// leaves no bracket behind.
template <typename Enqueue>
static int launch(dhqr_context* c, cudaStream_t st, const char* what, double work, Enqueue&& enqueue) {
    Event cw0, cw1, pf0, pf1;
    CwtSlot cwt = nullptr;
    const int cws = st == c->hp_stream ? 0 : st == c->hp2_stream ? 1 : st == c->aux_stream ? 2 : -1;
    if (c->chain_wait_trace && c->cwt_stamps && c->cwt_recs.size() < (size_t)CWT_MAX && cws >= 0 && cw0.create(cudaEventDefault) == cudaSuccess) {
        cudaEventRecord(cw0, st);
        cwt = c->cwt_stamps + 2 * c->cwt_recs.size();
    }
    if (c->profile && pf0.create(cudaEventDefault) == cudaSuccess) cudaEventRecord(pf0, st);
    cudaError_t e = cudaSuccess;
    if constexpr (std::is_void_v<decltype(enqueue(cwt))>) enqueue(cwt);
    else e = enqueue(cwt);
    c->launches++;
    if (cw0) { cw1.create(cudaEventDefault); cudaEventRecord(cw1, st); }
    if (pf0) { pf1.create(cudaEventDefault); cudaEventRecord(pf1, st); }
    const cudaError_t e2 = cudaGetLastError();
    if (e == cudaSuccess) e = e2;
    if (e != cudaSuccess) return set_err(1000 + (int)e, "launch of %s failed: %s", what, cudaGetErrorString(e));
    if (cw0) c->cwt_recs.push_back({c->cwt_unit, cws, prof_slot(c, what), std::move(cw0), std::move(cw1)});
    if (pf0) {
        const int s = prof_slot(c, what);
        c->prof_pending.push_back({s, std::move(pf0), std::move(pf1)});
        c->prof_slots[s].work += work;
    }
    if (c->sync) {
        e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) return set_err(1000 + (int)e, "%s failed: %s", what, cudaGetErrorString(e));
    }
    return 0;
}

// gemm_trace: the rows of a launch of `ctas` CTAs of k_gemm_vta or k_gemm_cvy_p (null: the option is off or the rows ran out)
static unsigned long long* gtr_slot(dhqr_context* c, size_t ctas) {
    if (!c->gemm_trace) return nullptr;
    if (c->gtr_used + ctas > GTR_MAX_CTAS) {
        c->gtr_dropped++;
        return nullptr;
    }
    unsigned long long* p = c->gtr_rows.p + GTR_WORDS * c->gtr_used;
    c->gtr_used += ctas;
    return p;
}

// Every column of `p` starts 16 B aligned (bulk copies legal): `p` itself is, and the leading dimension is even.
static bool bulk_ok(const void* p, int64_t ld) { return ((uintptr_t)p & 15) == 0 && (ld & 1) == 0; }

static constexpr int64_t WPART_TILES = 2304;   // capacity of the partial buffer in 128 x 64 tiles (151 MB per set)

// npanels: outer panels of the factorisation about to run (T' slots of the look-ahead schedule); catchup: also size the fourth
// V buffer / workspace set (dhqr_qr_host_f64 only)
static int ensure_workspace(dhqr_context* c, cudaStream_t st, int64_t m, int64_t n_local_max, int64_t npanels = 0, bool catchup = false) {
    TRY(set_attrs(c));
    const size_t vpk_elems = (size_t)((rup(m, 128) + 128) / KC1) * VPK_CHUNK;
    for (int b = 0; b < 3; ++b) TRY(c->vpk2[b].ensure(vpk_elems, st));
    for (int b = 0; b < 3; ++b) TRY(c->vpkb[b].ensure(vpk_elems, st));
    if (catchup) for (int b = 3; b < 3 + c->host_cu_streams; ++b) TRY(c->vpk2[b].ensure(vpk_elems, st));
    TRY(c->linv_all.ensure((size_t)std::max<int64_t>(npanels, 4) * NBMAX * NBMAX, st));
    TRY(c->gram_all.ensure((size_t)std::max<int64_t>(npanels, 4) * NBMAX * NBMAX, st));
    const int64_t tiles_max = (n_local_max + NBMAX + G1_BN - 1) / G1_BN + 1;
    for (int b = 0; b < (catchup ? 3 + c->host_cu_streams : 3); ++b) {
        auto& w = c->ws[b];
        // set 2 only ever updates the <= 128 columns of one panel: a quarter of the split-K partial buffer is plenty
        TRY(w.wpart.ensure((size_t)(b != 2 ? std::max(WPART_TILES, tiles_max) : WPART_TILES / 4) * NBMAX * G1_BN, st));
        // sets 0-2 also hold W and Y of a panel pair: W_a and W_b side by side, 8 k-chunks of Y per column tile
        const size_t pairx = b < 3 ? 2 : 1;
        TRY(w.wsum.ensure(pairx * NBMAX * (rup(n_local_max + NBMAX, 128) + 128), st));
        TRY(w.ypk.ensure(pairx * (NBMAX / KC) * YT * LDK * ((n_local_max + YT - 1) / YT + 2), st));
        TRY(w.linv.ensure((size_t)NBMAX * NBMAX, st));
    }
    if (!c->cells2) {
        const size_t words = (2 * (size_t)(PANEL_MAXG + 1) * (IB * (IB + 1) / 2) + IB * IB + 2 * IB) * 2;
        TRY(c->cells2.ensure(words, st));
        TRY(c->fast_stats.ensure(2, st));
        c->ll_epoch = 0;
    }
    if (!c->cells) { TRY(c->cells.ensure((size_t)IB * (PANEL_MAXG + 2) * IB * 2, st)); c->ll_epoch = 0; }
    if (!c->wctl) {
        TRY(c->wctl.ensure(1, st));
        // initial state {W_NOFAIL, 0}, in the caller's stream order
        TRY(launch(c, st, "k_wide_reset", 0.0, [&](CwtSlot) { k_wide_reset<<<1, 32, 0, st>>>(c->wctl); }));
        TRY(c->wbuf.ensure((size_t)5 * WP * WP + 3 * XL_ELEMS, st));
        TRY(c->wstamps.ensure(32, st));
    }
    TRY(c->v1.ensure((size_t)2 * rup(m + 4, 2), st));
    TRY(c->xbuf.ensure(1, st));
    return 0;
}

// ------------------------------------------------------------------------------------------------
// block-reflector application  C <- (I - V T' V') C  on window rows >= row_lo
//   V: nbp columns of the packed V buffer starting at Vcols (window row 0), T from the Gram matrix.
// ------------------------------------------------------------------------------------------------
// splits over the row chunks: fill whole waves of SMs
static int pick_splits(int tiles, int nchunks, int sms, int64_t cap_tiles) {
    tiles = std::max(tiles, 1);
    int smax = std::max(1, std::min(nchunks / 4, (MAXCTAS_FACTOR * sms) / tiles));
    smax = std::max(smax, std::min(1 + (sms + tiles - 1) / tiles, std::max(1, nchunks / 2)));
    smax = (int)std::min<int64_t>(smax, std::max<int64_t>(1, cap_tiles / tiles));
    int best = 1;
    double beste = 0.0;
    for (int s = 1; s <= smax; ++s) {
        const int ctas = tiles * s;
        const double e = (double)ctas / ((double)sms * ((ctas + sms - 1) / sms));
        if (e > beste + 1e-9) { beste = e; best = s; }
    }
    return best;
}

// The kb columns (mp rows) of a Householder block at A -> the first `width` packed columns of vpk, the block's row 0 at window row
// vtop, zero-filled to vrows rows (k_pack; tril: the block is stored in place in A, zeros above its diagonal)
static int pack_v(dhqr_context* c, cudaStream_t st, const double* A, int64_t lda, int64_t mp, int kb, int tril, double* vpk, int64_t vtop,
                  int64_t vrows, int width) {
    const dim3 grid((unsigned)std::min<int64_t>((vrows / 4 + 255) / 256, 4 * c->sms), width);
    return launch(c, st, "k_pack", 0.0, [&](CwtSlot) { k_pack<<<grid, 256, 0, st>>>(A, lda, mp, kb, tril, vpk, 0, vtop, vrows); });
}

// Partials of W = V' B -> w.wpart.  V = packed columns [voff, voff + nbp) of vpk, through the 32- or the 128-column kernel as nbp
// asks; nv > 0: W starts with the nv columns of V'V itself (for T), then come the ncols columns of B (`rows` rows).
static int launch_vta_partials(dhqr_context* c, cudaStream_t st, const double* vpk, dhqr_context::WSet& w, int voff, int nbp, int nv,
                               const double* B, int64_t ldb, int64_t rows, int ncols, const char* what, int* nsplit_out,
                               int64_t* pstride_out, int reserve = 0) {
    const bool small = (nbp <= 32);
    const int NBPK = small ? 32 : 128;          // kernel instantiation
    const int bn = small ? G1S_BN : G1_BN;
    const int tiles = (nv + ncols + bn - 1) / bn;
    const int nchunks = (int)((rows + KC1 - 1) / KC1);
    const int nsplit = pick_splits(tiles, nchunks, c->sms, (int64_t)(w.wpart.n / ((size_t)bn * NBPK)) - (int64_t)reserve * tiles);
    const int64_t pstride = (int64_t)tiles * bn * NBPK;
    if ((size_t)(pstride * (nsplit + reserve)) > w.wpart.n) return set_err(4001, "internal: W partial workspace too small");
    GemmVtaArgs g1;
    g1.vpk = vpk; g1.voff = voff; g1.nv = nv;
    g1.A = B; g1.lda = ldb; g1.rows = rows; g1.na = ncols; g1.nchunks = nchunks;
    g1.a_aligned = bulk_ok(B, ldb);
    g1.Wp = w.wpart; g1.pstride = pstride;
    *nsplit_out = nsplit;
    *pstride_out = pstride;
    return launch(c, st, what, 2.0 * (double)rows * nbp * ((double)ncols + nv), [&](CwtSlot cwt) {
        g1.cwt = cwt;
        g1.gtr = gtr_slot(c, (size_t)tiles * nsplit);
        const dim3 grid(tiles, nsplit);
        if (small) (g1.gtr ? K_G1_32T : K_G1_32)<<<grid, (1 * 4 + G1S_NPW) * 32, smem_g1(32, G1S_BN), st>>>(g1);
        else (g1.gtr ? K_G1_128T : K_G1_128)<<<grid, (4 * 2 + G1_NPW) * 32, smem_g1(128, G1_BN), st>>>(g1);
    });
}

// k_wreduce: one thread per element, at most eight CTAs per SM
static unsigned wreduce_grid(const dhqr_context* c, int64_t nelem) { return (unsigned)std::min<int64_t>((nelem + 255) / 256, 8 * c->sms); }

static int launch_cvy(dhqr_context* c, cudaStream_t st, const double* vpk, int voff, int nbp, const double* ypk, int64_t rows,
                      int64_t row_lo, double* C, int64_t ldc, int ncols, int gate);

// block-reflector application  C <- (I - V T' V') C  on window rows >= row_lo
//   V = packed columns [voff, voff + nbp) of `vpk` (columns beyond the live ones are zero); T from the
//   Gram matrix; `w` = the workspace set of the calling chain.
static int apply_block_reflector(dhqr_context* c, cudaStream_t st, const double* vpk, dhqr_context::WSet& w, int voff, int nbp,
                                 int64_t rows, int64_t row_lo, double* C, int64_t ldc, int ncols, bool reuse_T = false,
                                 double* linv_io = nullptr, int gate = 0, int trans = 0) {
    double* linv = linv_io ? linv_io : w.linv;   // where T' is written (or read from, with reuse_T)
    // reuse_T: w.linv already holds T' of this V (same chain, previous call) -> skip the Gram block and k_tinv
    if (ncols <= 0 || rows <= 0) return 0;
    const bool small = (nbp <= 32);
    const int NBPK = small ? 32 : 128;          // kernel instantiation
    const int nv = reuse_T ? 0 : NBPK;
    const int next = nv + ncols;
    if ((size_t)next * NBPK > w.wsum.n) return set_err(4003, "internal: W workspace too small");
    int nsplit = 0;
    int64_t pstride = 0;
    TRY(launch_vta_partials(c, st, vpk, w, voff, nbp, nv, C, ldc, rows, ncols, small ? "k_gemm_vta32" : "k_gemm_vta128", &nsplit,
                            &pstride));
    const int ygrid = (ncols + YCOLS - 1) / YCOLS;
    if (small && !reuse_T) {
        TRY(launch(c, st, "k_mid32", 0.0, [&](CwtSlot) {
            k_mid32<><<<ygrid, 512, 0, st>>>(w.wpart, pstride, nsplit, ncols, w.ypk, linv, trans);
        }));
    } else {
        const int64_t nelem = (int64_t)next * NBPK;
        TRY(launch(c, st, "k_wreduce", 0.0, [&](CwtSlot cwt) {
            k_wreduce<<<wreduce_grid(c, nelem), 256, 0, st>>>(w.wpart, pstride, nsplit, nelem, w.wsum, cwt);
        }));
        if (!reuse_T) {
            TRY(launch(c, st, small ? "k_tinv32" : "k_tinv128", 0.0, [&](CwtSlot cwt) {
                if (small) k_tinv<32><<<1, 512, smem_tinv(32), st>>>(w.wsum, linv, 0, cwt);
                else k_tinv<128><<<1, 512, smem_tinv(128), st>>>(w.wsum, linv, 0, cwt);
            }));
        }
        TRY(launch(c, st, small ? "k_ymake32" : "k_ymake128", 0.0, [&](CwtSlot cwt) {
            if (small) k_ymake<32><<<ygrid, 256, smem_ymake(32), st>>>(w.wsum, nv, ncols, linv, w.ypk, trans, cwt);
            else k_ymake<128><<<ygrid, 256, smem_ymake(128), st>>>(w.wsum, nv, ncols, linv, w.ypk, trans, cwt);
        }));
    }
    return launch_cvy(c, st, vpk, voff, nbp, w.ypk, rows, row_lo, C, ldc, ncols, gate);
}

// The arguments of C += V Y that come from C and the schedule: the 128 x 64 tiles over C, how many of them one CTA of the
// persistent variant walks through, whether C moves by bulk copies, and the gate of the speculative panel chain
static GemmCvyArgs cvy_args(const dhqr_context* c, double* C, int64_t ldc, int64_t rows, int ncols, int gate) {
    GemmCvyArgs g2;
    g2.C = C; g2.ldc = ldc; g2.rows = rows; g2.ncols = ncols;
    g2.tiles_m = (int)((rows + G2_BM - 1) / G2_BM); g2.tiles_n = (ncols + G2_BN - 1) / G2_BN;
    g2.tiles_per_cta = std::max(c->cvy_persist, 1);   // cvy_persist = 0: one tile per CTA
    g2.c_bulk = bulk_ok(C, ldc);
    g2.ctl = c->wctl; g2.gate = gate;
    return g2;
}

// k_gemm_cvy_p: one CTA pair per `tiles_per_cta` consecutive pair-tiles (a row tile by two adjacent column tiles)
static unsigned cvy_p_grid(const GemmCvyArgs& g2) {
    const int npairs = g2.tiles_m * ((g2.tiles_n + 1) / 2);
    const int clusters = (npairs + g2.tiles_per_cta - 1) / g2.tiles_per_cta;
    return clusters * CVYP_CLUSTER;
}

// C += V Y on window rows >= row_lo, Y packed in the ypk layout (nbp <= 32: one k-chunk per column tile; else NBMAX / KC):
// the second half of a block-reflector application, also fed a Y made elsewhere (the pivoted factorisation's -F')
static int launch_cvy(dhqr_context* c, cudaStream_t st, const double* vpk, int voff, int nbp, const double* ypk, int64_t rows,
                      int64_t row_lo, double* C, int64_t ldc, int ncols, int gate) {
    const bool small = (nbp <= 32);
    const int NBPK = small ? 32 : 128;
    GemmCvyArgs g2 = cvy_args(c, C, ldc, rows, ncols, gate);
    g2.row_lo = row_lo;
    g2.vpk = vpk; g2.voff = voff; g2.ypk = ypk;
    g2.nkq = small ? 1 : (int)(rup(nbp, KC) / KC); g2.nkq_alloc = NBPK / KC;
    g2.nks = 4; g2.vpk2 = nullptr;
    return launch(c, st, small ? "k_gemm_cvy32" : "k_gemm_cvy128", 2.0 * (double)rows * (small ? 32 : nbp) * (double)ncols,
                  [&](CwtSlot cwt) {
                      g2.cwt = cwt;
                      g2.gtr = g2.nkq == 4 ? gtr_slot(c, cvy_p_grid(g2)) : nullptr;
                      if (g2.nkq == 4) (g2.gtr ? k_gemm_cvy_p_traced : k_gemm_cvy_p)<<<cvy_p_grid(g2), CVYP_THREADS, smem_g2p(), st>>>(g2);
                      else k_gemm_cvy<<<dim3(g2.tiles_m, g2.tiles_n), 9 * 32, smem_g2(), st>>>(g2);
                  });
}

// W = V' C for one 128-column block -> Ws (128 x ncols, col-major), T' reused
static int block_w(dhqr_context* c, cudaStream_t st, const double* vpk, dhqr_context::WSet& w, const double* C, int64_t ldc, int64_t rows,
                   int ncols, double* Ws) {
    int nsplit = 0;
    int64_t pstride = 0;
    TRY(launch_vta_partials(c, st, vpk, w, 0, NBMAX, 0, C, ldc, rows, ncols, "k_gemm_vta128", &nsplit, &pstride));
    const int64_t nelem = (int64_t)ncols * NBMAX;
    return launch(c, st, "k_wreduce", 0.0, [&](CwtSlot cwt) {
        k_wreduce<<<wreduce_grid(c, nelem), 256, 0, st>>>(w.wpart, pstride, nsplit, nelem, Ws, cwt);
    });
}

// G = V_b' V_a of a panel pair (a = panel at column ca, b = the next 128 columns) into gout.  Below row ca + 128 the columns of
// panel a in A hold V_a (the panel is final once factored), so the product runs against A with the existing W kernel.
static int form_pair_gram(dhqr_context* c, cudaStream_t st, const double* vpk_b, dhqr_context::WSet& w, const double* A, int64_t lda,
                          int64_t col0, int64_t ca, int64_t m, double* gout) {
    int nsplit = 0;
    int64_t pstride = 0;
    TRY(launch_vta_partials(c, st, vpk_b, w, 0, NBMAX, 0, A + (ca - col0) * lda + ca + WP, lda, m - ca - WP, WP, "k_gram_pair", &nsplit,
                            &pstride));
    return launch(c, st, "k_wreduce", 0.0, [&](CwtSlot cwt) {
        k_wreduce4<<<(WP * WP * 4) / 256, 256, 0, st>>>(w.wpart, pstride, nsplit, (int64_t)WP * WP, gout, cwt);
    });
}

// Two 128-column blocks a then b in one pass over C:  C <- (I - V_b T_b' V_b')(I - V_a T_a' V_a') C,  i.e.  C += [V_a V_b] [Y_a; Y_b]
// with K = 256 (k_ymake2).  C = `rows` rows of a's window (starting at a's pivot row); V_b's window starts 128 rows lower.
// T_a', T_b' and G = V_b' V_a come from their slots.  Skipped on the device when a panel below `gate` was refused.
static int apply_pair(dhqr_context* c, cudaStream_t st, const double* vpa, const double* vpb, dhqr_context::WSet& w, int64_t rows,
                      double* C, int64_t ldc, int ncols, const double* Ta, const double* Tb, const double* G, int gate) {
    if (ncols <= 0) return 0;
    if ((size_t)2 * ncols * NBMAX > w.wsum.n) return set_err(4003, "internal: W workspace too small");
    double* Wa = w.wsum, *Wb = w.wsum + (size_t)ncols * NBMAX;
    TRY(block_w(c, st, vpa, w, C, ldc, rows, ncols, Wa));
    TRY(block_w(c, st, vpb, w, C + WP, ldc, rows - WP, ncols, Wb));
    TRY(launch(c, st, "k_ymake2", 0.0, [&](CwtSlot cwt) {
        k_ymake2<<<(ncols + YCOLS - 1) / YCOLS, 256, SMEM_YMAKE2, st>>>(Wa, Wb, ncols, Ta, Tb, G, w.ypk, cwt);
    }));
    GemmCvyArgs g2 = cvy_args(c, C, ldc, rows, ncols, gate);
    g2.row_lo = 0;
    g2.vpk = vpa; g2.voff = 0; g2.vpk2 = vpb; g2.ypk = w.ypk;
    g2.nkq = 8; g2.nkq_alloc = 8; g2.nks = 8;
    return launch(c, st, "k_gemm_cvy256", 2.0 * ((double)rows * WP + (double)(rows - WP) * WP) * (double)ncols, [&](CwtSlot cwt) {
        g2.cwt = cwt;
        g2.gtr = gtr_slot(c, cvy_p_grid(g2));
        (g2.gtr ? k_gemm_cvy_p_traced : k_gemm_cvy_p)<<<cvy_p_grid(g2), CVYP_THREADS, smem_g2p(), st>>>(g2);
    });
}

// Reset thresholds of the launch tags.  Tags are 32-bit and compared for equality with what a cell holds, so no tag may pass
// 2^32 - 1 before its counter is reset.
//   ll_epoch (k_panel, k_tp_panel): a launch starts at ll_epoch <= LL_EPOCH_MAX and uses tags up to ll_epoch + IB + 3 (k_panel's
//     fast path: ftag + 2 = epoch + IB + 3; k_tp_panel: epoch + IB), at most 0xF0000023 < 2^32 - 1; it then advances the
//     counter by IB + 8.
//   bs_epoch (k_backsolve_wave, k_forwardsolve_wave) and uw_epoch (k_unblocked_wave): one tag per launch, ++epoch after a reset
//     check at WAVE_EPOCH_MAX, so at most 0xFFFFFFF1 < 2^32 - 1.
static constexpr uint32_t LL_EPOCH_MAX = 0xF0000000u;
static constexpr uint32_t WAVE_EPOCH_MAX = 0xFFFFFFF0u;

// tag space of the exchange cells nearly used up: start over with clean cells (k_panel, k_tp_panel)
static int ll_epoch_check(dhqr_context* c, cudaStream_t st) {
    if (c->ll_epoch > LL_EPOCH_MAX) {
        CU(cudaMemsetAsync(c->cells, 0, sizeof(unsigned long long) * (size_t)IB * (PANEL_MAXG + 2) * IB * 2, st));
        CU(cudaMemsetAsync(c->cells2, 0, sizeof(unsigned long long) * (2 * (size_t)(PANEL_MAXG + 1) * (IB * (IB + 1) / 2) + IB * IB + 2 * IB) * 2, st));
        c->ll_epoch = 0;
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------
// cooperative panel launch: factor mp x ncols (<= IB) at P, V block -> vout columns
// ------------------------------------------------------------------------------------------------
static int launch_panel(dhqr_context* c, cudaStream_t st, double* vpk, double* P, int64_t ldp, int64_t mp, int ncols,
                        double* alpha, int voff, int64_t vtop, int64_t vrows, int gate = 0) {
    int gmax = c->panel_ctas > 0 ? c->panel_ctas : (c->lookahead ? 64 : c->sms);
    gmax = std::min(std::min(gmax, c->sms), PANEL_MAXG);
    int64_t rpc = std::max<int64_t>((mp + gmax - 1) / gmax, 64);
    rpc = rup(rpc, 8);
    while ((size_t)IB * ((size_t)rpc + 4) * 8 > 184 * 1024 && gmax < std::min(c->sms, PANEL_MAXG)) {   // slab too big: use more CTAs
        gmax = std::min(gmax * 2, std::min(c->sms, PANEL_MAXG));
        rpc = rup(std::max<int64_t>((mp + gmax - 1) / gmax, 64), 8);
    }
    const int G = (int)((mp + rpc - 1) / rpc);
    const int lds = (int)rpc + 4;   // rpc is a multiple of 8 -> lds == 4 mod 8
    const size_t smem = (size_t)IB * lds * 8;
    if (smem > 184 * 1024) return set_err(-2, "m too large for the resident panel kernel (%lld rows per CTA)", (long long)rpc);
    TRY(ll_epoch_check(c, st));
    PanelArgs a;
    a.P = P; a.ldp = ldp; a.mp = mp; a.ncols = ncols; a.alpha = alpha;
    a.vpk = vpk; a.voff = voff; a.vtop = vtop; a.vrows = vrows;
    a.rows_per_cta = (int)rpc; a.lds = lds;
    a.cells = c->cells; a.epoch = c->ll_epoch; a.trace = c->panel_trace;
    a.cells2 = c->cells2; a.fast = c->panel_fast; a.fast_stats = c->fast_stats;
    a.ctl = c->wctl; a.gate = gate;
    void* args[] = {&a};
    return launch(c, st, "k_panel", 16.0 * (double)mp * ncols, [&](CwtSlot) {   // work = bytes: panel read once + written once
        const cudaError_t e = cudaLaunchCooperativeKernel((void*)k_panel, dim3(G), dim3(PANEL_THREADS), args, smem, st);
        if (e == cudaSuccess) c->ll_epoch += IB + 8;   // the launch has used the tags up to here
        return e;
    });
}

// ------------------------------------------------------------------------------------------------
// partition bookkeeping: global list of panels (owner, first global column, width)
// ------------------------------------------------------------------------------------------------
struct Panel { int owner; int64_t c; int kb; };

static int gather_partition(dhqr_context* c, cudaStream_t st, int64_t col0, int64_t n_local, std::vector<int64_t>& col0s,
                            std::vector<int64_t>& nls) {
    col0s.assign(c->nranks, 0);
    nls.assign(c->nranks, 0);
    if (c->nranks == 1) { col0s[0] = col0; nls[0] = n_local; return 0; }
    int64_t mine[2] = {col0, n_local};
    CU(cudaMemcpyAsync(c->d_i64, mine, sizeof(mine), cudaMemcpyHostToDevice, st));
    NC(g_nccl.AllGather(c->d_i64, c->d_i64 + 2, 2, ncclInt64, c->comm, st));
    std::vector<int64_t> all(2 * c->nranks);
    CU(cudaMemcpyAsync(all.data(), c->d_i64 + 2, sizeof(int64_t) * 2 * c->nranks, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    for (int r = 0; r < c->nranks; ++r) { col0s[r] = all[2 * r]; nls[r] = all[2 * r + 1]; }
    return 0;
}

static int check_partition(const std::vector<int64_t>& col0s, const std::vector<int64_t>& nls, int64_t n_global) {
    // DArray (1,P) grid: contiguous, ascending with rank (S:19, test/runtests.jl:71)
    int64_t next = 0;
    for (size_t r = 0; r < col0s.size(); ++r) {
        if (col0s[r] != next || nls[r] < 0) return set_err(-4, "column blocks must be contiguous and ascending with rank (rank %zu: col0=%lld, expected %lld)", r, (long long)col0s[r], (long long)next);
        next += nls[r];
    }
    if (next != n_global) return set_err(-3, "column blocks cover %lld columns, n_global=%lld", (long long)next, (long long)n_global);
    return 0;
}

static void build_panels(const std::vector<int64_t>& col0s, const std::vector<int64_t>& nls, int nb, std::vector<Panel>& out) {
    out.clear();
    for (size_t r = 0; r < col0s.size(); ++r)
        for (int64_t o = 0; o < nls[r]; o += nb) out.push_back({(int)r, col0s[r] + o, (int)std::min<int64_t>(nb, nls[r] - o)});
}

// ------------------------------------------------------------------------------------------------
// argument checks: the storage contract of include/dhqr.h
// ------------------------------------------------------------------------------------------------
// An entry point lists its arguments in order: require() for a scalar rule, operand() for a pointer with its extent.  The first
// failing check sets the error, minus the argument's 1-based position, and turns every later check into a no-op; the entry point
// returns that code (a Check converts to it) before anything is enqueued.  The success path neither allocates nor formats.
enum : unsigned {
    NEED = 1,       // a null pointer is an error (the entry point passes it when the operand is not empty)
    ALIGN = 2,      // the pointer must be aligned for its element type, even when the operand is empty
    DISJOINT = 4,   // the operand must not overlap any operand listed before it
    OR_SAME = 8,    // ... unless it is that operand itself, with the same leading dimension (form_q's Q == A)
};
static unsigned when(bool cond, unsigned rules) { return cond ? rules : 0u; }

// rows x cols elements, leading dimension ld; `batch` of them `stride` elements apart (the stride counts when batch > 1)
struct Extent { int64_t rows, cols, ld; bool has_ld; int64_t batch, stride; };
static Extent mat(int64_t rows, int64_t cols, int64_t ld, int64_t batch = 1, int64_t stride = 0) {
    return {rows, cols, ld, true, batch, stride};
}
static Extent vec(int64_t n, int64_t batch = 1, int64_t stride = 0) { return {n, 1, n, false, batch, stride}; }

class Check {
  public:
    // argument 1: a null handle, or one of several ranks when the entry point is single-GPU (`single_gpu` names what it serves)
    explicit Check(const dhqr_context* c, const char* single_gpu = nullptr) {
        if (!c) fail(1, "null handle");
        else if (single_gpu && c->nranks != 1) fail(1, "%s is single-GPU (the handle has %d ranks)", single_gpu, c->nranks);
    }
    operator int() const { return rc_; }

    template <typename... A>
    Check& require(bool ok, int pos, const char* fmt, A... args) {
        if (!rc_ && !ok) fail(pos, fmt, args...);
        return *this;
    }

    // Pointer argument `pos` to elements of type T; a matrix's leading dimension is argument pos + 1, and the stride (batch > 1)
    // the argument after the last of these.  Checks null, alignment, ld, stride, then overlap with the operands listed before.
    template <typename T>
    Check& operand(int pos, const char* name, const void* p, const Extent& e, unsigned rules) {
        if (rc_) return *this;
        if ((rules & NEED) && !p) return fail(pos, "null %s", name);
        // The complex kernels move whole double2 elements.  The C-ABI takes void*, and an 8 B aligned ComplexF64 pointer is legal C
        // (double _Complex, Julia's ComplexF64, a reinterpreted view of a Float64 vector): refuse it here instead of faulting.
        if ((rules & ALIGN) && (uintptr_t)p % alignof(T)) {
            if (std::is_same<T, double2>::value)
                return fail(pos, "%s is not 16-byte aligned (ComplexF64 data needs the alignment of double2)", name);
            return fail(pos, "%s must be %d B aligned", name, (int)alignof(T));
        }
        if (e.has_ld && e.ld < std::max<int64_t>(1, e.rows))
            return fail(pos + 1, "the leading dimension of %s is %lld < max(1, rows = %lld)", name, (long long)e.ld, (long long)e.rows);
        if (e.batch > 1 && (__int128)e.stride < (__int128)e.ld * e.cols)
            return fail(pos + (e.has_ld ? 2 : 1), "the stride of %s is %lld < %lld (%s)", name, (long long)e.stride,
                        (long long)(e.ld * e.cols), e.has_ld ? "leading dimension x columns" : "its length");
        const Span s = {name, (uintptr_t)p, span(e, sizeof(T)), e.ld};
        for (int i = 0; i < nseen_ && (rules & DISJOINT); ++i) {
            const Span& q = seen_[i];
            if (s.bytes && q.bytes && s.p < q.p + q.bytes && q.p < s.p + s.bytes && !((rules & OR_SAME) && s.p == q.p && s.ld == q.ld))
                return fail(pos, (rules & OR_SAME) ? "%s overlaps %s without being it (with the same leading dimension)" : "%s overlaps %s",
                            name, q.name);
        }
        if (nseen_ < MAXOPS) seen_[nseen_++] = s;
        return *this;
    }

  private:
    static constexpr int MAXOPS = 8;   // the batched downdate has seven
    struct Span { const char* name; uintptr_t p; size_t bytes; int64_t ld; };
    int rc_ = 0;
    int nseen_ = 0;
    Span seen_[MAXOPS];

    template <typename... A>
    Check& fail(int pos, const char* fmt, A... args) {
        rc_ = set_err(-pos, fmt, args...);
        return *this;
    }
    // Bytes from the first element to one past the last; 0 when the operand is empty.  A negative stride counts as 0, and the span
    // is clamped, so that an absurd stride or leading dimension cannot wrap the interval test.
    static size_t span(const Extent& e, size_t esz) {
        if (e.batch <= 0 || e.rows <= 0 || e.cols <= 0) return 0;
        const __int128 n = (__int128)(e.batch - 1) * std::max<int64_t>(e.stride, 0) + (__int128)(e.cols - 1) * e.ld + e.rows;
        const __int128 bytes = n * (__int128)esz, cap = (__int128)1 << 61;
        return (size_t)(bytes > cap ? cap : bytes);
    }
};

// arguments 2-5 of the column-block entry points: the m x n_global matrix and this rank's columns [col0, col0 + n_local)
static void column_block(Check& a, int64_t m, int64_t n_global, int64_t col0, int64_t n_local) {
    a.require(m >= 0, 2, "m < 0");
    a.require(n_global >= 0 && n_global <= m, 3, "need 0 <= n_global <= m (reference asserts full column rank shapes)");
    a.require(col0 >= 0 && col0 <= n_global, 4, "col0 out of range");
    a.require(n_local >= 0 && col0 + n_local <= n_global, 5, "n_local out of range");
}

// the profile class of a launch: the Float64 kernel's name or the ComplexF64 one's
template <typename T>
static const char* kname(const char* f64, const char* c64) { return std::is_same<T, double>::value ? f64 : c64; }

// ------------------------------------------------------------------------------------------------
// qr!: blocked driver  (S:113-148, S:198-213)
// ------------------------------------------------------------------------------------------------
struct PanelGeom { int64_t r0, rows, vrows; int nbp; };
static PanelGeom panel_geom(const Panel& p, int64_t m) {
    PanelGeom g;
    g.r0 = p.c & ~(int64_t)31;              // window start: 32-row aligned for the TMA chunks
    g.rows = m - g.r0;                       // valid window rows
    g.vrows = rup(g.rows, 128);
    g.nbp = (int)rup(p.kb, IB);
    return g;
}

// factor one outer panel on stream st: inner panels of IB columns + updates inside the outer panel; V -> vpk
// (the 32-column chain: one cooperative launch per inner panel, S:127-135 column by column in the worst case)
static int factor_outer_panel_narrow(dhqr_context* c, cudaStream_t st, double* vpk, dhqr_context::WSet& w, const Panel& p, int64_t m,
                                     int64_t col0, double* A, int64_t lda, double* alpha, int step) {
    const PanelGeom g = panel_geom(p, m);
    for (int o = 0; o < p.kb; o += IB) {
        const int ib = std::min(IB, p.kb - o);
        const int64_t cs = p.c + o;                                   // global column == pivot row
        double* P = A + (cs - col0) * lda + cs;
        TRY(launch_panel(c, st, vpk, P, lda, m - cs, ib, alpha + cs, o, cs - g.r0, g.vrows, step));
        const int rem = p.kb - (o + ib);
        if (rem > 0)   // update the rest of the outer panel with this sub-panel's reflectors
            TRY(apply_block_reflector(c, st, vpk, w, o, IB, g.rows, cs - g.r0, A + (cs + ib - col0) * lda + g.r0, lda, rem, false,
                                      nullptr, step));
    }
    if (g.nbp > IB && g.nbp < NBMAX) {   // zero the V columns the 128-wide kernels read beyond nbp
        TRY(launch(c, st, "k_vpk_zero_cols", 0.0, [&](CwtSlot) {
            k_vpk_zero_cols<<<2 * c->sms, 256, 0, st>>>(vpk, g.vrows / KC1, g.nbp, NBMAX);
        }));
    }
    return 0;
}

// The split of a panel's Gram matrix over CTAs: k_gram_sym, k_pack_gram and the Gram mode of k_vpk_rmul all run on this many
// CTAs, so that they sum the same chunks in the same order.
static int panel_gram_split(dhqr_context* c, const dhqr_context::WSet& w, int64_t rows, int* nchunks_out, int* nsplit_out) {
    const int nchunks = (int)((rows + KC1 - 1) / KC1);
    const int cps = std::max(1, (nchunks + c->sms - 1) / c->sms);                           // chunks per CTA: whole waves of equal CTAs
    const int nsplit = (nchunks + cps - 1) / cps;
    if ((size_t)nsplit * WP * WP > w.wpart.n) return set_err(4001, "internal: W partial workspace too small");
    *nchunks_out = nchunks;
    *nsplit_out = nsplit;
    return 0;
}

// Partial Gram matrices of the packed panel in `vpk` (window rows `rows`) -> w.wpart; returns the number of partials and their stride.
static int launch_panel_gram(dhqr_context* c, cudaStream_t st, const double* vpk, dhqr_context::WSet& w, int64_t rows, int* nsplit_out,
                             int64_t* pstride_out) {
    const int64_t pstride = (int64_t)WP * WP;
    int nchunks, nsplit;
    TRY(panel_gram_split(c, w, rows, &nchunks, &nsplit));
    GramSymArgs g;
    g.vpk = vpk; g.nchunks = nchunks; g.Wp = w.wpart; g.pstride = pstride;
    *nsplit_out = nsplit;
    *pstride_out = pstride;
    return launch(c, st, "k_gram128", 2.0 * (double)rows * WP * WP, [&](CwtSlot) {
        k_gram_sym<<<nsplit, (GS_MMA_WARPS + 1) * 32, SMEM_GRAM_SYM, st>>>(g);
    });
}

// the 128-column chain (dhqr_wide.cuh): CholeskyQR2 + Householder reconstruction of a full aligned outer panel
static bool wide_eligible(const dhqr_context* c, const Panel& p, int64_t m, int nb) {
    return c->wide_panel && nb == WP && p.kb == WP && (p.c & 31) == 0 && m - p.c >= WP;
}
static int factor_outer_panel_wide(dhqr_context* c, cudaStream_t st, double* vpk, dhqr_context::WSet& w, const Panel& p, int64_t m,
                                   int64_t col0, double* A, int64_t lda, double* alpha, int step, double* linv_out) {
    const PanelGeom g = panel_geom(p, m);       // r0 == p.c: the window starts at the pivot row
    double* P = A + (p.c - col0) * lda + p.c;
    double* R1 = c->wbuf, *R2 = R1 + WP * WP, *Rt = R2 + WP * WP, *Rr = Rt + WP * WP, *MT = Rr + WP * WP;
    double* Z1 = MT + WP * WP, *Z2 = Z1 + XL_ELEMS, *Z23 = Z2 + XL_ELEMS;
    double* vflag = vpk + KC1;                  // padding row 64 of packed column 0: travels with the V buffer
    const int nq = (int)(g.vrows / KC1);
    long long* stamps = c->wide_trace ? c->wstamps.p : nullptr;
    // Gram matrices of the panel: partials over the window rows, split over CTAs as launch_panel_gram splits them
    int nchunks = 0, nsplit = 0;
    const int64_t pstride = (int64_t)WP * WP;
    TRY(panel_gram_split(c, w, g.rows, &nchunks, &nsplit));
    RmulArgs r;
    r.vpk = vpk; r.ctl = c->wctl; r.step = step; r.P = nullptr; r.ldp = lda; r.mp = g.rows;
    r.Wp = nullptr; r.nchunks = nchunks; r.pstride = pstride;
    auto rmul = [&](int q0, int n, const double* Z, double* Pout, bool with_gram) -> int {
        if (n <= 0) return 0;
        r.q0 = q0; r.nq = n; r.ZL = Z; r.P = Pout; r.Wp = with_gram ? w.wpart.p : nullptr;
        const double work = 2.0 * 64.0 * n * WP * 80.0 + (with_gram ? 2.0 * (double)g.rows * WP * WP : 0.0);
        return launch(c, st, with_gram ? "k_rmul_gram" : "k_vpk_rmul", work, [&](CwtSlot cwt) {
            r.cwt = cwt;
            k_vpk_rmul<<<with_gram ? nsplit : std::min(n, c->sms), 256, SMEM_RMUL, st>>>(r);
        });
    };
    // pack + first Gram: the chunks go from the caller's matrix into the Gram kernel's tiles, and from there to vpk
    PackGramArgs pg;
    pg.P = P; pg.ldp = lda; pg.rows = g.rows; pg.p_bulk = bulk_ok(P, lda);
    pg.vpk = vpk; pg.nq = nq; pg.nchunks = nchunks; pg.Wp = w.wpart; pg.pstride = pstride;
    TRY(launch(c, st, "k_gram128", 2.0 * (double)g.rows * WP * WP, [&](CwtSlot cwt) {
        pg.cwt = cwt;
        k_pack_gram<<<nsplit, (GS_MMA_WARPS + PG_PROD_WARPS) * 32, SMEM_GRAM_SYM, st>>>(pg);
    }));
    TRY(launch(c, st, "k_wreduce", 0.0, [&](CwtSlot cwt) {
        k_wreduce4<<<(WP * WP * 4) / 256, 256, 0, st>>>(w.wpart, pstride, nsplit, (int64_t)WP * WP, w.wsum, cwt);
    }));
    TRY(launch(c, st, "k_chol128", 0.0, [&](CwtSlot cwt) {
        k_chol128<<<1, 512, SMEM_WIDE1, st>>>(w.wsum, R1, Z1, c->wctl, step, vflag, c->wide_kappa, stamps, cwt);
    }));
    TRY(rmul(0, nq, Z1, nullptr, true));    // Q1, and the partials of the second Gram matrix Q1'Q1
    TRY(launch(c, st, "k_gram2_finish", 0.0, [&](CwtSlot cwt) {
        k_gram2_finish<<<256, 256, 0, st>>>(w.wpart, pstride, nsplit, w.wsum, R2, Z2, c->wctl, step, vflag, cwt);
    }));
    // Two small kernels sit beside the chain, not in it (their own high-priority stream, unless the per-launch profile or the
    // debug sync asks for plain stream order): Rt = R2 R1 overlaps the solve of the top chunks, k_trecon the last pass
    cudaStream_t sx = (!c->profile && !c->sync) ? c->aux_stream : st;
    if (sx != st) { CU(cudaEventRecord(c->ev_aux[0], st)); CU(cudaStreamWaitEvent(sx, c->ev_aux[0], 0)); }
    TRY(launch(c, sx, "k_trimm128", 0.0, [&](CwtSlot cwt) { k_trimm128<<<10, 256, SMEM_TRIMM, sx>>>(R2, R1, Rt, c->wctl, step, cwt); }));
    if (sx != st) CU(cudaEventRecord(c->ev_aux[1], sx));
    TRY(rmul(0, 2, Z2, nullptr, false));
    if (sx != st) CU(cudaStreamWaitEvent(st, c->ev_aux[1], 0));
    TRY(launch(c, st, "k_hr128", 0.0, [&](CwtSlot cwt) {
        k_hr128<<<1, 512, SMEM_WIDE1, st>>>(vpk, Rt, P, lda, alpha + p.c, Rr, MT, c->wctl, step, stamps ? stamps + 16 : nullptr, cwt);
    }));
    if (linv_out) {     // T' of the panel from the reconstruction: the owner's next block update needs neither V'V nor k_tinv
        if (sx != st) { CU(cudaEventRecord(c->ev_aux[2], st)); CU(cudaStreamWaitEvent(sx, c->ev_aux[2], 0)); }
        TRY(launch(c, sx, "k_trecon", 0.0, [&](CwtSlot cwt) {
            k_trecon<<<4, 256, SMEM_TRECON, sx>>>(vpk, MT, linv_out, c->wctl, step, cwt);
        }));
        if (sx != st) CU(cudaEventRecord(c->ev_aux[3], sx));
    }
    TRY(launch(c, st, "k_trimm_z", 0.0, [&](CwtSlot cwt) { k_trimm_z<<<10, 256, SMEM_TRIMM, st>>>(Rr, R2, Z23, c->wctl, step, cwt); }));
    TRY(rmul(2, nq - 2, Z23, P, false));
    if (linv_out && sx != st) CU(cudaStreamWaitEvent(st, c->ev_aux[3], 0));   // T' is part of the panel's result
    c->wide_panels++;
    return 0;
}

static int factor_outer_panel(dhqr_context* c, cudaStream_t st, double* vpk, dhqr_context::WSet& w, const Panel& p, int64_t m,
                              int64_t col0, double* A, int64_t lda, double* alpha, int step, bool wide, double* linv_out = nullptr) {
    if (c->wctl) {   // clear the guards of the previous panel and the verdict that travels with this V buffer
        TRY(launch(c, st, "k_wide_begin", 0.0, [&](CwtSlot cwt) { k_wide_begin<<<1, 32, 0, st>>>(c->wctl, vpk + KC1, cwt); }));
    }
    if (wide) return factor_outer_panel_wide(c, st, vpk, w, p, m, col0, A, lda, alpha, step, linv_out);
    return factor_outer_panel_narrow(c, st, vpk, w, p, m, col0, A, lda, alpha, step);
}

static int mirror_panel_to_host(dhqr_context* c, cudaStream_t st, const Panel& p, int64_t m, int64_t col0, const double* A,
                                int64_t lda) {
    if (!c->mirror_host) return 0;   // host entry point only: this panel's columns are final -> start their D2H now
    Event ev;
    CU(ev.create(cudaEventDisableTiming));
    CU(cudaEventRecord(ev, st));
    CU(cudaStreamWaitEvent(c->d2h_stream, ev, 0));
    c->panel_events.push_back(std::move(ev));
    CU(cudaMemcpy2DAsync(c->mirror_host + p.c * c->mirror_lda, (size_t)c->mirror_lda * 8, A + (p.c - col0) * lda, (size_t)lda * 8,
                         (size_t)m * 8, (size_t)p.kb, cudaMemcpyDeviceToHost, c->d2h_stream));
    return 0;
}

// Which panels go through the 128-column chain: those at or beyond `wide_from` that are full and aligned.
struct Plan { int kstart; int wide_from; int nb; };
static bool plan_wide(const dhqr_context* c, const Plan& pl, const std::vector<Panel>& panels, int k, int64_t m) {
    return k >= pl.wide_from && wide_eligible(c, panels[k], m, pl.nb);
}

// Unit of work of the drivers: one panel, or a pair of panels (a, a + 1) whose trailing update is one 256-wide block (apply_pair),
// so the bulk update reads and writes C once per 256 reflectors.  A pair needs one rank, both panels through the 128-column
// chain (nb = 128), and not the windowed first pass of the host entry, whose catch-ups apply one panel at a time.
struct Unit { int a; int np; };
static void build_units(const dhqr_context* c, const Plan& pl, const std::vector<Panel>& panels, int64_t m, bool windowed,
                        std::vector<Unit>& units) {
    units.clear();
    const bool pairs = c->nranks == 1 && !windowed;
    for (int k = pl.kstart; k < (int)panels.size();) {
        const bool two = pairs && k + 1 < (int)panels.size() && plan_wide(c, pl, panels, k, m) && plan_wide(c, pl, panels, k + 1, m);
        units.push_back({k, two ? 2 : 1});
        k += two ? 2 : 1;
    }
}

// Factor the panels of unit u into va (and vb): a pair factors a, applies V_a to the columns of b (K = 128, T'_a from its slot),
// factors b and forms G = V_b' V_a.  T' of a single panel goes to linv_single, of a pair's panels to their slots.  Returns in
// *ownT whether T' of the unit is known on this rank.
static int factor_unit(dhqr_context* c, cudaStream_t st, const Unit& u, double* va, double* vb, dhqr_context::WSet& w,
                       const std::vector<Panel>& panels, const Plan& pl, int64_t m, int64_t col0, double* A, int64_t lda, double* alpha,
                       double* linv_single, bool* ownT) {
    const int a = u.a;
    const Panel& pa = panels[a];
    if (u.np == 1) {
        const bool wide = plan_wide(c, pl, panels, a, m);
        TRY(factor_outer_panel(c, st, va, w, pa, m, col0, A, lda, alpha, a, wide, linv_single));
        TRY(mirror_panel_to_host(c, st, pa, m, col0, A, lda));
        *ownT = wide;
        return 0;
    }
    const Panel& pb = panels[a + 1];
    const PanelGeom ga = panel_geom(pa, m);
    TRY(factor_outer_panel(c, st, va, w, pa, m, col0, A, lda, alpha, a, true, c->tslot(a)));
    TRY(mirror_panel_to_host(c, st, pa, m, col0, A, lda));
    TRY(apply_block_reflector(c, st, va, w, 0, WP, ga.rows, 0, A + (pb.c - col0) * lda + ga.r0, lda, WP, true, c->tslot(a), a + 1));
    TRY(factor_outer_panel(c, st, vb, w, pb, m, col0, A, lda, alpha, a + 1, true, c->tslot(a + 1)));
    TRY(mirror_panel_to_host(c, st, pb, m, col0, A, lda));
    TRY(form_pair_gram(c, st, vb, w, A, lda, col0, pa.c, m, c->gslot(a)));
    c->pair_units++;
    *ownT = true;
    return 0;
}

// single stream, one unit after the other (options lookahead = 0, sync, profile; any number of ranks)
static int qr_blocked_serial(dhqr_context* c, cudaStream_t st, int64_t m, int64_t col0, int64_t nl, double* A, int64_t lda,
                             double* alpha, const std::vector<Panel>& panels, const Plan& pl, const std::vector<Unit>& units) {
    const int64_t lend = col0 + nl;
    double* vpk = c->vpk2[0];
    auto& w = c->ws[0];
    for (const Unit& u : units) {
        const int k = u.a;
        const Panel& p = panels[k];
        const PanelGeom g = panel_geom(p, m);
        bool haveT = false;
        if (c->rank == p.owner) TRY(factor_unit(c, st, u, vpk, c->vpkb[0], w, panels, pl, m, col0, A, lda, alpha, w.linv, &haveT));
        if (u.np == 2) {
            const int64_t t0 = panels[k + 1].c + WP;
            if (t0 < lend)
                TRY(apply_pair(c, st, vpk, c->vpkb[0], w, g.rows, A + (t0 - col0) * lda + g.r0, lda, (int)(lend - t0), c->tslot(k),
                               c->tslot(k + 1), c->gslot(k), k + 2));
            continue;
        }
        if (c->nranks > 1) {
            // C2 (S:141-143): the owner's reflectors go to every rank, once per panel instead of once per column
            NC(g_nccl.Broadcast(vpk, vpk, (size_t)(g.vrows / KC1) * VPK_CHUNK, ncclFloat64, p.owner, c->comm, st));
            NC(g_nccl.Broadcast(alpha + p.c, alpha + p.c, (size_t)p.kb, ncclFloat64, p.owner, c->comm, st));
            TRY(launch(c, st, "k_wide_note", 0.0, [&](CwtSlot) { k_wide_note<<<1, 32, 0, st>>>(c->wctl, vpk + KC1, k); }));
        }
        // trailing update of the local columns right of the panel (S:198-213 for nb columns at once)
        const int64_t t0 = std::max(p.c + p.kb, col0);
        if (t0 < lend)
            TRY(apply_block_reflector(c, st, vpk, w, 0, g.nbp, g.rows, p.c - g.r0, A + (t0 - col0) * lda + g.r0, lda, (int)(lend - t0),
                                      haveT, nullptr, k + 1));
    }
    return 0;
}

// The events of one run of the look-ahead schedule: per unit (hp: created by the unit's publish, with several ranks only), per
// upload chunk that joined (caught: its catch-up is done), and the fork from the caller's stream.  They are destroyed with their
// owner: once recorded and waited on, the work they order is already enqueued.  Unless dismissed, the owner first makes the
// caller's stream wait for every internal stream of the schedule, so that on an error return it neither runs ahead of nor
// returns before work already queued there.
struct LookaheadEvents {
    dhqr_context* c;
    cudaStream_t st;
    std::vector<Event> panel, next, bulk, a2, hp, caught;
    Event fork;
    bool join = true;
    LookaheadEvents(dhqr_context* c_, cudaStream_t st_, int K) : c(c_), st(st_), panel(K), next(K), bulk(K), a2(K), hp(K) {}
    void dismiss() { join = false; }
    ~LookaheadEvents() {
        Event done;
        if (join && done.create(cudaEventDisableTiming) == cudaSuccess) {
            for (cudaStream_t s : {c->hp_stream.h, c->comm_stream.h, c->hp2_stream.h, c->cu_stream[0].h, c->cu_stream[1].h, c->cu_stream[2].h}) {
                cudaEventRecord(done, s);
                cudaStreamWaitEvent(st, done, 0);
            }
        }
    }
};

// chain_wait_trace, before a look-ahead factorisation: forget the launches of the previous one and reset the stamps in stream
// order, starts to ~0 (atomicMin), ends to 0 (atomicMax)
static int cwt_reset(dhqr_context* c, cudaStream_t st) {
    if (!c->chain_wait_trace || !c->cwt_stamps) return 0;
    c->cwt_recs.clear();
    c->cwt_rows.clear();
    c->cwt_unit = 0;
    if (cudaMemset2DAsync(c->cwt_stamps, 16, 0xFF, 8, CWT_MAX, st) != cudaSuccess ||
        cudaMemset2DAsync(c->cwt_stamps + 1, 16, 0, 8, CWT_MAX, st) != cudaSuccess) return set_err(1002, "chain_wait_trace reset failed");
    return 0;
}

// chain_wait_trace, after it: one row per traced launch (unit, stream, class, event span, stamp span, wait; ms)
static int cwt_collect(dhqr_context* c, cudaStream_t st) {
    if (!c->chain_wait_trace || !c->cwt_stamps) return 0;
    for (cudaStream_t s : {st, c->hp_stream.h, c->hp2_stream.h, c->aux_stream.h}) cudaStreamSynchronize(s);
    std::vector<unsigned long long> t(2 * c->cwt_recs.size());
    if (!t.empty() && cudaMemcpy(t.data(), c->cwt_stamps, t.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost) != cudaSuccess)
        return set_err(1002, "chain_wait_trace read-back failed");
    for (size_t i = 0; i < c->cwt_recs.size(); ++i) {
        const auto& r = c->cwt_recs[i];
        float span = 0.f;
        cudaEventElapsedTime(&span, r.e0, r.e1);
        const bool stamped = t[2 * i] != ~0ull && t[2 * i + 1] >= t[2 * i];   // kernels without a CwtScope: -1
        const double run = stamped ? (double)(t[2 * i + 1] - t[2 * i]) * 1e-6 : -1.0;
        const double row[6] = {(double)r.unit, (double)r.stream, (double)r.cls, (double)span, run, stamped ? span - run : -1.0};
        c->cwt_rows.insert(c->cwt_rows.end(), row, row + 6);
    }
    return 0;
}

// la_trace, after a look-ahead factorisation: la_times, and under host_trace the stage timeline of the pipelined host entry on
// stderr (ms since the first chunk was on the device).  joinedAt: the step at which each upload chunk joined.
static void la_collect(dhqr_context* c, cudaStream_t st, const LookaheadEvents& ev, const std::vector<Panel>& panels, const Plan& pl,
                       const std::vector<Unit>& units, const std::vector<int>& joinedAt) {
    if (!c->la_trace) return;
    cudaStreamSynchronize(st);
    cudaStreamSynchronize(c->hp_stream);
    c->la_times.assign(panels.size() * 3, 0.f);
    for (size_t k = 0; k < units.size(); ++k)
        for (int q = units[k].a; q < units[k].a + units[k].np; ++q) {
            cudaEventElapsedTime(&c->la_times[3 * q + 0], ev.fork, ev.panel[k]);
            cudaEventElapsedTime(&c->la_times[3 * q + 1], ev.fork, ev.next[k]);
            cudaEventElapsedTime(&c->la_times[3 * q + 2], ev.fork, ev.bulk[k]);
        }
    if (!c->host_trace) return;
    for (size_t j = 0; j < ev.caught.size(); ++j) {
        float tu = -1.f, tc = -1.f;
        cudaEventSynchronize(ev.caught[j]);
        cudaEventElapsedTime(&tu, ev.fork, c->up_chunks[j].ev);
        cudaEventElapsedTime(&tc, ev.fork, ev.caught[j]);
        fprintf(stderr, "[dhqr host] chunk at column %5lld: uploaded %7.2f ms, joins at step %2d (planned %2d), caught up %7.2f ms\n",
                (long long)c->up_chunks[j].c0, tu, joinedAt[j], c->up_chunks[j].join, tc);
    }
    for (int k = pl.kstart; k < (int)panels.size(); ++k)
        fprintf(stderr, "[dhqr host] step %2d: panel %7.2f  T' %7.2f  bulk %7.2f ms\n", k, c->la_times[3 * k], c->la_times[3 * k + 1],
                c->la_times[3 * k + 2]);
}

// look-ahead: the panel chain (latency bound) runs on a high-priority stream ahead of the bulk trailing update, which stays on
// the caller's stream.  SPMD over ranks: the owner of a panel factors it, the packed V block is broadcast on the high-priority
// stream (the only stream that issues collectives), every rank updates its own columns.
//   hp step k: wait next[k-1];  owner(k+1): apply V_k -> columns of panel k+1, factor panel k+1 (V -> vpk[(k+1)%3]);
//              broadcast vpk[(k+1)%3] + alpha slice;  signal panel[k+1]                                    set 1
//   st step k: wait panel[k];   (a) apply V_k -> local columns of panel k+2, signal next[k];
//                               (b) apply V_k -> local columns right of panel k+2 (T reused)                set 0
// Every column block receives every V exactly once and in order; the panel chain only depends on the small
// (a) parts, i.e. it has two bulk updates of slack.  Three V buffers: V_{k+2} replaces V_{k-1}, whose last
// reader (b)_{k-1} precedes (a)_k on st (hence the wait on next[k-1] on every rank before the broadcast).
// k counts units (build_units): "panel k" above is unit k, a single panel or a pair whose updates run with K = 256; a pair's
// second V buffer (vpkb) and G slot follow the same ring rule.  la_times stays per panel (both panels of a pair get the pair's).
static int qr_blocked_lookahead(dhqr_context* c, cudaStream_t st, int64_t m, int64_t col0, int64_t nl, double* A, int64_t lda,
                                double* alpha, const std::vector<Panel>& panels, const Plan& pl, const std::vector<Unit>& units) {
    const int64_t lend = col0 + nl;
    const int K = (int)units.size(), K0 = 0;
    auto P = [&](int k) -> const Panel& { return panels[units[k].a]; };                              // first panel of unit k
    auto uend = [&](int k) { const Panel& q = panels[units[k].a + units[k].np - 1]; return q.c + q.kb; };
    cudaStream_t hp = c->hp_stream;
    LookaheadEvents ev(c, st, K);
    auto& evPanel = ev.panel, &evNext = ev.next, &evBulk = ev.bulk, &evA2 = ev.a2, &evHp = ev.hp, &evCatch = ev.caught;
    std::vector<char> haveA2(K, 0);
    const unsigned evflags = c->la_trace ? cudaEventDefault : cudaEventDisableTiming;
    for (int k = K0; k < K; ++k) {
        CU(evA2[k].create(cudaEventDisableTiming));
        CU(evPanel[k].create(evflags));
        CU(evNext[k].create(evflags));
        CU(evBulk[k].create(evflags));
    }
    // local intersection of the global column range [a, b) -> pointer + count
    auto clip = [&](int64_t a, int64_t b, int64_t& lo, int64_t& hi) { lo = std::max(a, col0); hi = std::min(b, lend); return hi > lo; };
    // publish panel k (already factored on its owner into vpk[k%3]) to every rank.  The collectives run on their own stream:
    // the owner's chain goes on with panel k+1 (it has V_k already) while V_k travels; the other ranks pick it up through
    // evPanel[k].  The comm stream first waits for everything queued on hp so far: on the owner that is the factorisation of
    // panel k, on every rank the last reads of the ring slot's previous occupant V_{k-3}.
    cudaStream_t cs = c->comm_stream;
    auto publish = [&](int k) -> int {
        if (c->nranks > 1) {
            const PanelGeom g = panel_geom(P(k), m);
            double* v = c->vpk2[k % 3];
            CU(evHp[k].create(cudaEventDisableTiming));
            CU(cudaEventRecord(evHp[k], hp));
            CU(cudaStreamWaitEvent(cs, evHp[k], 0));
            NC(g_nccl.Broadcast(v, v, (size_t)(g.vrows / KC1) * VPK_CHUNK, ncclFloat64, P(k).owner, c->comm, cs));
            NC(g_nccl.Broadcast(alpha + P(k).c, alpha + P(k).c, (size_t)P(k).kb, ncclFloat64, P(k).owner, c->comm, cs));
            // the owner's verdict on the panel arrived with the buffer
            TRY(launch(c, cs, "k_wide_note", 0.0, [&](CwtSlot) { k_wide_note<<<1, 32, 0, cs>>>(c->wctl, v + KC1, units[k].a); }));
            CU(cudaEventRecord(evPanel[k], cs));
        } else {
            CU(cudaEventRecord(evPanel[k], hp));
        }
        return 0;
    };
    // V_k is usable on stream s: the owner has it once its own chain got there (hp order / evHp), the others once it arrived
    auto wait_panel = [&](cudaStream_t s, int k) {
        if (c->nranks > 1 && c->rank == P(k).owner) {
            if (s != hp) cudaStreamWaitEvent(s, evHp[k], 0);
        } else {
            cudaStreamWaitEvent(s, evPanel[k], 0);
        }
    };
    // Host entry (dhqr_qr_host_f64, one rank, first pass): columns [wend, lend) are still on their way to the device in chunks
    // (c->up_chunks).  The schedule runs on the window [col0, wend); a chunk joins at the step its plan names - at the latest
    // while it still lies right of panel k+2 - after a CATCH-UP on its own stream: the reflectors of panels < k, re-packed from
    // the factored columns, applied to the chunk with the T' kept in the per-panel slots.  Same reflectors in the same order on
    // every column, only the time at which a column receives them changes.
    const bool windowed = !c->up_chunks.empty() && c->nranks == 1 && pl.kstart == 0;   // then every unit is one panel
    int64_t wend = windowed ? std::min(lend, c->up_chunks.front().c0) : lend;
    size_t upnext = 0;
    std::vector<char> haveTslot(K, 0);
    auto catch_up = [&](const dhqr_context::UpChunk& u, int lane, int k, cudaEvent_t done) -> int {
        cudaStream_t cu = c->cu_stream[lane];
        double* vpk_cu = c->vpk2[3 + lane];
        auto& ws_cu = c->ws[3 + lane];
        cudaStreamWaitEvent(cu, u.ev, 0);
        for (int q = K0; q < k; ++q) {
            const Panel& pq = P(q);
            const PanelGeom gq = panel_geom(pq, m);
            cudaStreamWaitEvent(cu, evPanel[q], 0);                   // V_q is final in A ...
            cudaStreamWaitEvent(cu, evNext[q], 0);                    // ... and T'_q sits in its slot
            TRY(pack_v(c, cu, A + (pq.c - col0) * lda + pq.c, lda, m - pq.c, pq.kb, 1, vpk_cu, pq.c - gq.r0, gq.vrows,
                       gq.nbp <= IB ? IB : NBMAX));
            TRY(apply_block_reflector(c, cu, vpk_cu, ws_cu, 0, gq.nbp, gq.rows, pq.c - gq.r0, A + (u.c0 - col0) * lda + gq.r0, lda,
                                      (int)(u.c1 - u.c0), haveTslot[q] != 0, c->tslot(units[q].a), units[q].a + 1));
        }
        cudaEventRecord(done, cu);
        return 0;
    };
    std::vector<int> joinedAt;                                    // step at which each upload chunk joined (host_trace)
    TRY(cwt_reset(c, st));
    if (ev.fork.create(evflags) != cudaSuccess) return set_err(1001, "event create failed");
    cudaEventRecord(ev.fork, st);
    cudaStreamWaitEvent(hp, ev.fork, 0);                          // hp starts after everything already queued on st
    std::vector<char> ownT(K, 0);       // T'_k already sits in the ring slot on this rank (wide panel factored here, k_trecon)
    if (c->rank == P(K0).owner) {
        bool wide = false;
        TRY(factor_unit(c, hp, units[K0], c->vpk2[K0 % 3], c->vpkb[K0 % 3], c->ws[1], panels, pl, m, col0, A, lda, alpha,
                        c->tslot(units[K0].a), &wide));
        if (wide) { ownT[K0] = 1; cudaEventRecord(evNext[K0], hp); }
    }
    TRY(publish(K0));
    for (int k = K0; k < K; ++k) {
        const Panel& p = P(k);
        const PanelGeom g = panel_geom(p, m);
        const double* vk = c->vpk2[k % 3];
        c->cwt_unit = k + 1;   // chain launches of this step end with unit k + 1 factored (unit 0: before the loop)
        const int pk = units[k].a;                                                   // first panel of the unit
        const int64_t t0 = uend(k);                                                  // first trailing column
        const int64_t t1 = k + 1 < K ? uend(k + 1) : t0;                             // end of unit k+1
        const int64_t t2 = k + 2 < K ? uend(k + 2) : t1;                             // end of unit k+2
        // V_k (one panel, or both panels of a pair: K = 256, T' and G from their slots) -> local columns [lo, hi) on stream s
        auto apply_k = [&](cudaStream_t s, dhqr_context::WSet& w, int64_t lo, int64_t hi, bool haveT, double* linv_io) -> int {
            double* C = A + (lo - col0) * lda + g.r0;
            if (units[k].np == 2)
                return apply_pair(c, s, vk, c->vpkb[k % 3], w, g.rows, C, lda, (int)(hi - lo), c->tslot(pk), c->tslot(pk + 1),
                                  c->gslot(pk), pk + 2);
            return apply_block_reflector(c, s, vk, w, 0, g.nbp, g.rows, p.c - g.r0, C, lda, (int)(hi - lo), haveT, linv_io, pk + 1);
        };
        int64_t lo, hi;
        // chunks that join the window at this step: planned, or forced because step k+1 would reach into them
        const int64_t wold = wend;
        const size_t up0 = upnext;
        if (windowed) {
            const int64_t t3 = k + 3 < K ? uend(k + 3) : lend;                         // end of unit k+3
            while (upnext < c->up_chunks.size() && (c->up_chunks[upnext].join <= k || c->up_chunks[upnext].c0 < t3)) {
                const auto& u = c->up_chunks[upnext];
                if (u.c0 < t2 || u.c0 != wend) return set_err(4005, "internal: upload chunk %d joins too late (step %d)", (int)upnext, k);
                Event done;
                if (done.create(evflags) != cudaSuccess) return set_err(1001, "event create failed");
                evCatch.push_back(std::move(done));
                joinedAt.push_back(k);
                TRY(catch_up(u, (int)(upnext % (size_t)c->host_cu_streams), k, evCatch.back()));
                wend = u.c1;
                ++upnext;
            }
            if (wend < t2) return set_err(4005, "internal: window ends at %lld before panel %d", (long long)wend, k + 2);
        }
        double* lk = c->tslot(pk);
        bool haveT = ownT[k];                                        // T'_k in lk (this rank)
        bool hp2_gate = false;                                       // evA2[k] already marks where hp2 may start on hp
        if (k + 1 < K) {
            // vpk[(k+1)%3] was last read by the bulk update k-2 (and, on the owner of panel k-2, by its broadcast)
            if (k - 2 >= K0) {
                cudaStreamWaitEvent(hp, evBulk[k - 2], 0);
                if (haveA2[k - 2]) cudaStreamWaitEvent(hp, evA2[k - 2], 0);
                if (c->nranks > 1) cudaStreamWaitEvent(hp, evPanel[k - 2], 0);
            }
            if (c->rank == P(k + 1).owner) {
                wait_panel(hp, k);
                if (k - 1 >= K0 && haveA2[k - 1]) cudaStreamWaitEvent(hp, evA2[k - 1], 0);   // V_{k-1} reached these columns
                if (clip(t0, t1, lo, hi)) {
                    const bool hadT = haveT;
                    TRY(apply_k(hp, c->ws[1], lo, hi, haveT, lk));
                    haveT = true;
                    if (!hadT) cudaEventRecord(evNext[k], hp);       // T'_k is in the ring: the bulk update may start
                }
                // hp2 needs nothing of the factorisation of unit k+1 below: it neither touches nor gates on its columns
                cudaEventRecord(evA2[k], hp);
                hp2_gate = true;
                bool widen = false;
                TRY(factor_unit(c, hp, units[k + 1], c->vpk2[(k + 1) % 3], c->vpkb[(k + 1) % 3], c->ws[1], panels, pl, m, col0, A, lda,
                                alpha, c->tslot(units[k + 1].a), &widen));
                if (widen) { ownT[k + 1] = 1; cudaEventRecord(evNext[k + 1], hp); }
            }
            TRY(publish(k + 1));
        }
        // columns of panel k+2: their V_0..V_{k-1} come from the bulk updates up to k-1.  This apply is off the chain's
        // stream and overlaps the factorisation of panel k+1; the chain picks it up through evA2[k] before it applies
        // V_{k+1} to the same columns.
        if (clip(t1, t2, lo, hi)) {
            cudaStream_t s2 = c->hp2_stream;
            if (!hp2_gate) cudaEventRecord(evA2[k], hp);             // (used as a scratch event first: order s2 behind hp's
            cudaStreamWaitEvent(s2, evA2[k], 0);                     //  work up to T'_k, not behind the factorisation of k+1)
            if (k - 1 >= K0) cudaStreamWaitEvent(s2, evBulk[k - 1], 0);
            wait_panel(s2, k);
            const bool hadT = haveT;
            TRY(apply_k(s2, c->ws[2], lo, hi, haveT, lk));
            haveT = true;
            if (!hadT) cudaEventRecord(evNext[k], s2);               // T'_k came from this apply
            cudaEventRecord(evA2[k], s2);
            haveA2[k] = true;
        }
        if (!haveT) cudaEventRecord(evNext[k], hp);                  // keep the event defined (timeline tracing)
        wait_panel(st, k);
        if (clip(t2, std::min(lend, wold), lo, hi)) {
            if (haveT) cudaStreamWaitEvent(st, evNext[k], 0);
            TRY(apply_k(st, c->ws[0], lo, hi, haveT, haveT ? lk : nullptr));
        }
        for (size_t j = up0; j < upnext; ++j) {                      // the chunks that joined at this step, each behind its catch-up
            const auto& u = c->up_chunks[j];
            cudaStreamWaitEvent(st, evCatch[j], 0);
            if (haveT) cudaStreamWaitEvent(st, evNext[k], 0);
            TRY(apply_k(st, c->ws[0], u.c0, u.c1, haveT, haveT ? lk : nullptr));
        }
        haveTslot[k] = haveT;
        cudaEventRecord(evBulk[k], st);
    }
    cudaStreamWaitEvent(st, evPanel[K - 1], 0);                    // join: alpha and the last panel come from hp / the comm stream
    if (c->nranks > 1) {
        cudaEventRecord(evHp[K - 1], hp);                          // (re-recorded: everything queued on hp)
        cudaStreamWaitEvent(st, evHp[K - 1], 0);
    }
    TRY(cwt_collect(c, st));
    la_collect(c, st, ev, panels, pl, units, joinedAt);
    ev.dismiss();
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_err(1000 + (int)e, "look-ahead enqueue failed: %s", cudaGetErrorString(e));
    return 0;
}

// largest row count the resident 32-column panel kernel can take on this device (slab of rows in shared memory)
static int64_t narrow_panel_max_rows(const dhqr_context* c) {
    const int gmax = std::min(c->sms, PANEL_MAXG);
    const int64_t rpc = ((184 * 1024) / (IB * 8) - 4) & ~(int64_t)7;
    return rpc * gmax;
}

static int qr_blocked(dhqr_context* c, cudaStream_t st, int64_t m, int64_t n, int64_t col0, int64_t nl, double* A,
                      int64_t lda, double* alpha, int nb) {
    std::vector<int64_t> col0s, nls;
    TRY(gather_partition(c, st, col0, nl, col0s, nls));
    TRY(check_partition(col0s, nls, n));
    int64_t nlmax = 0;
    for (auto v : nls) nlmax = std::max(nlmax, v);
    std::vector<Panel> panels;
    build_panels(col0s, nls, nb, panels);
    TRY(ensure_workspace(c, st, m, nlmax, (int64_t)panels.size(), !c->up_chunks.empty()));
    if (panels.empty()) return 0;
    // rank-uniform precondition, checked on every rank BEFORE the first collective: a panel that neither chain can take
    // would otherwise fail on its owner only and leave the other ranks inside ncclBroadcast
    Plan pl = {0, 0, nb};
    for (int k = 0; k < (int)panels.size(); ++k)
        if (m - panels[k].c > narrow_panel_max_rows(c))
            return set_err(-2, "m too large for the resident panel kernel (%lld rows; limit %lld)", (long long)(m - panels[k].c),
                           (long long)narrow_panel_max_rows(c));
    const bool la = c->lookahead && panels.size() > 1 && !c->sync && !c->profile;
    for (;;) {
        bool any_wide = false;
        for (int k = pl.kstart; k < (int)panels.size(); ++k) any_wide |= plan_wide(c, pl, panels, k, m);
        TRY(launch(c, st, "k_wide_reset", 0.0, [&](CwtSlot) { k_wide_reset<<<1, 32, 0, st>>>(c->wctl); }));
        const bool use_la = la && (int)panels.size() - pl.kstart > 1;
        if (!use_la && !c->up_chunks.empty()) {   // the serial schedule knows nothing about columns still in flight: wait for them
            for (const auto& u : c->up_chunks) CU(cudaStreamWaitEvent(st, u.ev, 0));
            c->up_chunks.clear();
        }
        std::vector<Unit> units;
        build_units(c, pl, panels, m, use_la && !c->up_chunks.empty() && pl.kstart == 0, units);
        const int rc = use_la ? qr_blocked_lookahead(c, st, m, col0, nl, A, lda, alpha, panels, pl, units)
                              : qr_blocked_serial(c, st, m, col0, nl, A, lda, alpha, panels, pl, units);
        c->up_chunks.clear();                     // every chunk has joined (or the pass failed): a restart sees the whole matrix
        if (rc || !any_wide) return rc;
        // The wide chain is speculative: its guards are evaluated on the device.  One synchronisation per factorisation to
        // learn whether a panel was refused; if so, everything from that panel on was skipped on the device and is redone
        // here, that panel with the 32-column chain (same result on every rank: the verdict travels with the V buffer).
        int fail = W_NOFAIL;
        CU(cudaMemcpyAsync(&fail, &c->wctl.p->fail_step, sizeof(int), cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        if (fail == W_NOFAIL) return 0;
        if (fail < pl.kstart || fail >= (int)panels.size()) return set_err(4004, "internal: bad restart index %d", fail);
        c->wide_redone++;
        for (const Unit& u : units)
            if (u.np == 2 && u.a + 1 == fail) {
                // the refused panel is the second of a pair: V_a reached b's columns (inner apply), but not the columns right of b,
                // whose merged update was skipped.  Apply V_a alone there (re-packed from A, T'_a from its slot) before redoing b.
                const Panel& pa = panels[u.a];
                const PanelGeom ga = panel_geom(pa, m);
                const int64_t t0 = panels[fail].c + panels[fail].kb;
                if (t0 >= col0 + nl) break;
                TRY(pack_v(c, st, A + (pa.c - col0) * lda + pa.c, lda, m - pa.c, pa.kb, 1, c->vpk2[0], 0, ga.vrows, NBMAX));
                TRY(apply_block_reflector(c, st, c->vpk2[0], c->ws[0], 0, WP, ga.rows, 0, A + (t0 - col0) * lda + ga.r0, lda,
                                          (int)(col0 + nl - t0), true, c->tslot(u.a), 0));
            }
        pl.kstart = fail;
        pl.wide_from = fail + 1;
    }
}

// qr!: unblocked driver (nb == 1): one reflector per step, as the reference does it (S:127-144)
static int qr_unblocked(dhqr_context* c, cudaStream_t st, int64_t m, int64_t n, int64_t col0, int64_t nl, double* A,
                        int64_t lda, double* alpha) {
    std::vector<int64_t> col0s, nls;
    TRY(gather_partition(c, st, col0, nl, col0s, nls));
    TRY(check_partition(col0s, nls, n));
    TRY(ensure_workspace(c, st, m, nl));
    const int64_t lend = col0 + nl;
    if (c->nranks == 1 && n > 0 && m <= (int64_t)UW_MAXI * UW_THREADS && c->unblocked_wave && !c->profile && !c->sync) {
        // single GPU, short columns: the whole column loop as one persistent cooperative launch (k_unblocked_wave)
        if (c->uw_flags.n < (size_t)n) {
            TRY(c->uw_flags.ensure((size_t)n + 64, st));
            c->uw_epoch = 0;
        }
        if (c->uw_epoch > WAVE_EPOCH_MAX) { CU(cudaMemsetAsync(c->uw_flags, 0, sizeof(unsigned int) * c->uw_flags.n, st)); c->uw_epoch = 0; }
        const unsigned int tag = ++c->uw_epoch;
        int nn = (int)n;
        unsigned int* flags = c->uw_flags;
        void* args[] = {&A, &lda, &m, &nn, &alpha, &flags, (void*)&tag};
        const int G = (int)std::min<int64_t>(c->sms, n);
        return launch(c, st, "k_unblocked_wave", 16.0 * (double)m * n * n / 2, [&](CwtSlot) {
            return cudaLaunchCooperativeKernel((void*)k_unblocked_wave, dim3(G), dim3(UW_THREADS), args, 0, st);
        });
    }
    if (c->nranks == 1 && n > 0 && (size_t)((m + 2) & ~(int64_t)1) * 8 * (A1_CW + 1) <= 200 * 1024 && c->fuse_house) {
        // single GPU, the column tile fits in shared memory: one launch per column step (the next reflector is formed by the
        // CTA that has just updated its column, k_apply1_tma), two v buffers alternating between steps
        const int64_t voff = rup(m + 4, 2);
        TRY(launch(c, st, "k_house1", 0.0, [&](CwtSlot) { k_house1<<<1, 1024, 0, st>>>(A, m, alpha, c->v1); }));
        for (int64_t j = 0; j + 1 < n; ++j) {
            const int lead = (int)(j & 1);
            const int64_t lenw = m - j + lead, lenp = (lenw + 1) & ~(int64_t)1;
            const int nc = (int)(n - j - 1);
            double* C = A + (j + 1) * lda + (j - lead);
            const int aligned = bulk_ok(C, lda);
            double* vcur = c->v1 + (j & 1) * voff, *vnext = c->v1 + ((j + 1) & 1) * voff;
            cudaLaunchConfig_t cfg = {};
            cfg.gridDim = dim3((nc + A1_CW - 1) / A1_CW);
            cfg.blockDim = dim3(A1_THREADS);
            cfg.dynamicSmemBytes = (size_t)lenp * 8 * (A1_CW + 1);
            cfg.stream = st;
            cudaLaunchAttribute at[1];
            at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
            at[0].val.programmaticStreamSerializationAllowed = c->profile ? 0 : 1;   // event brackets want plain stream order
            cfg.attrs = at;
            cfg.numAttrs = 1;
            const double* vc = vcur;
            const int64_t ldc = lda;
            TRY(launch(c, st, "k_apply1_tma", 16.0 * (double)(m - j) * nc, [&](CwtSlot) {
                return cudaLaunchKernelEx(&cfg, k_apply1_tma, vc, lenw, C, ldc, nc, aligned, vnext, alpha + j + 1, lead);
            }));
        }
        return 0;
    }
    for (int owner = 0; owner < c->nranks; ++owner) {
        for (int64_t j = col0s[owner]; j < col0s[owner] + nls[owner]; ++j) {
            const int lead = (int)(j & 1);          // window starts on an even row so TMA sources stay 16B aligned
            const int64_t len = m - j;
            if (c->rank == owner) {
                if (lead) CU(cudaMemsetAsync(c->v1, 0, sizeof(double), st));
                TRY(launch(c, st, "k_house1", 0.0, [&](CwtSlot) {
                    k_house1<<<1, 1024, 0, st>>>(A + (j - col0) * lda + j, len, alpha + j, c->v1 + lead);
                }));
            }
            if (c->nranks > 1) {
                NC(g_nccl.Broadcast(c->v1, c->v1, (size_t)(len + lead + 1), ncclFloat64, owner, c->comm, st));
                NC(g_nccl.Broadcast(alpha + j, alpha + j, 1, ncclFloat64, owner, c->comm, st));
            }
            const int64_t t0 = std::max(j + 1, col0);
            if (t0 >= lend) continue;
            const int nc = (int)(lend - t0);
            double* C = A + (t0 - col0) * lda + (j - lead);
            const int64_t lenw = len + lead;
            const int64_t lenp = (lenw + 1) & ~(int64_t)1;
            const size_t smem = (size_t)lenp * 8 * (A1_CW + 1);
            if (smem <= 200 * 1024) {
                const int aligned = bulk_ok(C, lda);
                TRY(launch(c, st, "k_apply1_tma", 0.0, [&](CwtSlot) {
                    k_apply1_tma<<<(nc + A1_CW - 1) / A1_CW, A1_THREADS, smem, st>>>(c->v1, lenw, C, lda, nc, aligned, nullptr, nullptr, lead);
                }));
            } else {
                TRY(launch(c, st, "k_apply1_direct", 0.0, [&](CwtSlot) {
                    k_apply1_direct<<<std::min(nc, 8 * c->sms), A1_THREADS, 0, st>>>(c->v1, lenw, C, lda, nc);
                }));
            }
        }
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------
// solve phases
// ------------------------------------------------------------------------------------------------
// Q'b on the local reflectors: panels of <= 128 reflectors, each applied as a block reflector
// built from V alone (T recomputed from V'V), so only (A, alpha) are needed, like the reference.
static int apply_qt_local(dhqr_context* c, cudaStream_t st, int64_t m, int64_t col0, int64_t nl, const double* A,
                          int64_t lda, double* b, int64_t ldb, int nrhs, int notrans = 0) {
    // notrans: b <- Q b = H_1 (H_2 (... H_n b)): the panels in reverse order, each as I - V T V' (T instead of T')
    if (nl <= 0) return 0;
    const int64_t ofirst = notrans ? ((nl - 1) / NBMAX) * NBMAX : 0, ostep = notrans ? -(int64_t)NBMAX : NBMAX;
    for (int64_t o = ofirst; o >= 0 && o < nl; o += ostep) {
        const int kb = (int)std::min<int64_t>(NBMAX, nl - o);
        const int64_t cs = col0 + o;
        const int64_t r0 = cs & ~(int64_t)31;
        const int64_t rows = m - r0, vrows = rup(rows, 128);
        const int nbp = kb <= IB ? IB : NBMAX;
        TRY(pack_v(c, st, A + o * lda + cs, lda, m - cs, kb, 1, c->vpk2[0], cs - r0, vrows, nbp));
        TRY(apply_block_reflector(c, st, c->vpk2[0], c->ws[0], 0, nbp, rows, cs - r0, b + r0, ldb, nrhs, false, nullptr, 0, notrans));
    }
    return 0;
}

// One right-hand side: T' of every local panel first (independent of b, so with several ranks every rank does this while b is
// still with its predecessors), then the sweep with two GEMV-shaped launches per panel (k_qt_dot, k_qt_axpy).
static constexpr int QT_MAXG = 1024;
static int qt_prepare(dhqr_context* c, cudaStream_t st, int64_t m, int64_t col0, int64_t nl, const double* A, int64_t lda) {
    const int npl = (int)((nl + NBMAX - 1) / NBMAX);
    if (npl <= 0) return 0;
    TRY(c->qt_T.ensure((size_t)npl * NBMAX * NBMAX, st));
    if (!c->qt_part) {
        TRY(c->qt_part.alloc((size_t)(QT_MAXG + 1) * WP));     // last row: y
        TRY(c->qt_ticket.ensure(1, st));
    }
    auto& w = c->ws[0];
    if ((size_t)npl * NBMAX * NBMAX > w.wsum.n) return set_err(4006, "internal: Gram workspace too small");
    for (int p = 0; p < npl; ++p) {
        const int64_t o = (int64_t)p * NBMAX, cs = col0 + o, r0 = cs & ~(int64_t)31;
        const int kb = (int)std::min<int64_t>(NBMAX, nl - o);
        const int64_t rows = m - r0, vrows = rup(rows, 128);
        TRY(pack_v(c, st, A + o * lda + cs, lda, m - cs, kb, 1, c->vpk2[0], cs - r0, vrows, NBMAX));
        int nsplit = 0;
        int64_t pstride = 0;
        TRY(launch_panel_gram(c, st, c->vpk2[0], w, rows, &nsplit, &pstride));
        TRY(launch(c, st, "k_wreduce4", 0.0, [&](CwtSlot) {
            k_wreduce4<<<(WP * WP * 4) / 256, 256, 0, st>>>(w.wpart, pstride, nsplit, (int64_t)WP * WP, w.wsum + (size_t)p * WP * WP);
        }));
    }
    return launch(c, st, "k_tinv128", 0.0, [&](CwtSlot) {
        k_tinv<128><<<npl, 512, smem_tinv(128), st>>>(w.wsum, c->qt_T, (int64_t)WP * WP);
    });
}

static int apply_qt_local_vec(dhqr_context* c, cudaStream_t st, int64_t m, int64_t col0, int64_t nl, const double* A, int64_t lda,
                              double* b, int notrans) {
    const int npl = (int)((nl + NBMAX - 1) / NBMAX);
    for (int q = 0; q < npl; ++q) {
        const int p = notrans ? npl - 1 - q : q;
        const int64_t o = (int64_t)p * NBMAX, cs = col0 + o;
        QtArgs a;
        a.V = A + o * lda + cs; a.lda = lda; a.mp = m - cs; a.kb = (int)std::min<int64_t>(NBMAX, nl - o);
        a.b = b + cs; a.Linv = c->qt_T + (size_t)p * NBMAX * NBMAX;
        a.part = c->qt_part; a.y = c->qt_part + (size_t)QT_MAXG * WP; a.ticket = c->qt_ticket; a.trans = notrans;
        int64_t rpc = rup(std::max<int64_t>((a.mp + c->sms - 1) / c->sms, 64), 32);                // one CTA per SM
        rpc = std::min<int64_t>(rpc, QT_MAXROWS);
        const int64_t G = (a.mp + rpc - 1) / rpc;
        if (G > QT_MAXG) return set_err(4007, "internal: too many k_qt_dot CTAs");                  // callers check m first
        a.rows_per_cta = (int)rpc;
        TRY(launch(c, st, "k_qt_dot", 8.0 * (double)a.mp * a.kb, [&](CwtSlot) { k_qt_dot<<<(unsigned)G, QT_THREADS, 0, st>>>(a); }));
        TRY(launch(c, st, "k_qt_axpy", 8.0 * (double)a.mp * a.kb, [&](CwtSlot) {
            k_qt_axpy<<<(unsigned)((a.mp + QT_AROWS - 1) / QT_AROWS), QT_ATHREADS, 0, st>>>(a);
        }));
    }
    return 0;
}
static bool qt_vec_ok(const dhqr_context* c, int64_t m, int nrhs) { return c->qt_vec && nrhs == 1 && m <= (int64_t)QT_MAXG * QT_MAXROWS; }

// Set-up shared by both wavefront substitutions: the x cells for nl local unknowns (zeroed in stream order when they grow)
// and the co-residency limit of each wave kernel on this device.
static int wave_prepare(dhqr_context* c, cudaStream_t st, int64_t nl) {
    if (c->bs_blocks() < (size_t)(nl + 31) / 32 + 1) {
        TRY(c->bs_cells.ensure(((size_t)(nl + 31) / 32 + 64) * 64, st));
        c->bs_epoch = 0;
    }
    if (!c->bs_wave_max_ctas) {
        int per_sm = 0;
        CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_backsolve_wave, BW_THREADS, 0));
        c->bs_wave_max_ctas = std::max(1, per_sm * c->sms);
        CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_forwardsolve_wave, BW_THREADS, 0));
        c->fs_wave_max_ctas = std::max(1, per_sm * c->sms);
    }
    return 0;
}

// Tag of the next wave launch; the cells are cleared before the 32-bit tag could come round to a value they still hold.
static int wave_tag(dhqr_context* c, cudaStream_t st, uint32_t* tag) {
    if (c->bs_epoch > WAVE_EPOCH_MAX) {
        CU(cudaMemsetAsync(c->bs_cells, 0, c->bs_cells.n * sizeof(unsigned long long), st));
        c->bs_epoch = 0;
    }
    *tag = ++c->bs_epoch;
    return 0;
}

// x <- R^{-1} y by blocks of BS_BLK columns, last to first (S:260: i = n:-1:1), one k_backsolve_step launch per block: the
// fallback of backsolve_local and every ComplexF64 back-substitution.  y[0:col0 + nl] is overwritten on the way.
template <typename T>
static int backsolve_steps(dhqr_context* c, cudaStream_t st, int64_t col0, int64_t nl, const T* A, int64_t lda, const T* alpha, T* y,
                           int64_t ldy, int nrhs, T* x, int64_t ldx) {
    for (int64_t o = ((nl - 1) / BS_BLK) * BS_BLK; o >= 0; o -= BS_BLK) {
        const int bs = (int)std::min<int64_t>(BS_BLK, nl - o);
        const int64_t c0 = col0 + o;
        const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((c0 + 255) / 256, 2 * c->sms));
        TRY(launch(c, st, kname<T>("k_backsolve_step", "k_backsolve_step_c"), 0.0, [&](CwtSlot) {
            k_backsolve_step<T><<<grid, 256, 0, st>>>(A + o * lda, lda, alpha, y, ldy, nrhs, x, ldx, c0, bs);
        }));
    }
    return 0;
}

static int backsolve_local(dhqr_context* c, cudaStream_t st, int64_t col0, int64_t nl, const double* A, int64_t lda,
                           const double* alpha, double* y, int64_t ldy, int nrhs, double* x, int64_t ldx) {
    if (nl <= 0) return 0;
    // one launch per right-hand side: a wavefront over 32-row strips (k_backsolve_wave); needs every CTA resident at once
    const int64_t nbk = (nl + 31) / 32, nlow = (col0 + 31) / 32;
    if (c->bs_wave && nbk + nlow <= c->bs_wave_max_ctas && nbk <= (int64_t)c->bs_blocks()) {
        for (int rhs = 0; rhs < nrhs; ++rhs) {
            uint32_t tag;
            TRY(wave_tag(c, st, &tag));
            TRY(launch(c, st, "k_backsolve_wave", 0.0, [&](CwtSlot) {
                k_backsolve_wave<<<(unsigned)(nbk + nlow), BW_THREADS, 0, st>>>(A, lda, alpha, y + (int64_t)rhs * ldy, x + (int64_t)rhs * ldx,
                                                                              col0, nl, c->bs_cells, tag);
            }));
        }
        return 0;
    }
    return backsolve_steps(c, st, col0, nl, A, lda, alpha, y, ldy, nrhs, x, ldx);
}

// x (n x nrhs, leading dimension n) <- R^{-1} y[0:n] on one GPU, n > 0: backsolve_local for Float64, the steps for ComplexF64
template <typename T>
static int backsolve_single(dhqr_context* c, cudaStream_t st, int64_t n, const T* A, int64_t lda, const T* alpha, T* y, int64_t ldy,
                            int nrhs, T* x) {
    if constexpr (std::is_same<T, double>::value) {
        TRY(wave_prepare(c, st, n));
        return backsolve_local(c, st, 0, n, A, lda, alpha, y, ldy, nrhs, x, n);
    } else {
        return backsolve_steps(c, st, 0, n, A, lda, alpha, y, ldy, nrhs, x, n);
    }
}

// y[0:n] <- R^{-H} y[0:n] on one GPU, through c->xbuf.  Float64: the wavefront of k_forwardsolve_wave (first strip to last) when
// every CTA fits on the device at once.  Otherwise (or with "bs_wave" = 0), and always for ComplexF64: blocks of BS_BLK columns,
// first to last, one k_forwardsolve_step each.  Every CTA of a step reads the block's y, so z goes to xbuf and is copied back at
// the end, as in the back-substitution.
template <typename T>
static int forwardsolve_local(dhqr_context* c, cudaStream_t st, int64_t n, const T* A, int64_t lda, const T* alpha, T* y, int64_t ldy,
                              int nrhs) {
    if (n <= 0 || nrhs <= 0) return 0;
    constexpr int w = sizeof(T) / sizeof(double);
    TRY(c->xbuf.ensure((size_t)w * n * nrhs, st));
    T* x = (T*)c->xbuf.p;
    const int64_t ldx = n, nbk = (n + 31) / 32;
    bool wave = false;
    if constexpr (std::is_same<T, double>::value) {
        TRY(wave_prepare(c, st, n));
        wave = c->bs_wave && nbk <= c->fs_wave_max_ctas && nbk <= (int64_t)c->bs_blocks();
        if (wave) {
            for (int rhs = 0; rhs < nrhs; ++rhs) {
                uint32_t tag;
                TRY(wave_tag(c, st, &tag));
                TRY(launch(c, st, "k_forwardsolve_wave", 0.0, [&](CwtSlot) {
                    k_forwardsolve_wave<<<(unsigned)nbk, BW_THREADS, 0, st>>>(A, lda, alpha, y + (int64_t)rhs * ldy, x + (int64_t)rhs * ldx,
                                                                             n, c->bs_cells, tag);
                }));
            }
        }
    }
    if (!wave) {
        for (int64_t c0 = 0; c0 < n; c0 += BS_BLK) {
            const int bs = (int)std::min<int64_t>(BS_BLK, n - c0);
            const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n - c0 - bs + 7) / 8, 4 * c->sms));
            TRY(launch(c, st, kname<T>("k_forwardsolve_step", "k_forwardsolve_step_c"), 0.0, [&](CwtSlot) {
                k_forwardsolve_step<T><<<grid, 256, 0, st>>>(A, lda, alpha, y, ldy, nrhs, x, ldx, c0, bs, n);
            }));
        }
    }
    CU(cudaMemcpy2DAsync(y, (size_t)ldy * sizeof(T), x, (size_t)ldx * sizeof(T), (size_t)n * sizeof(T), nrhs, cudaMemcpyDeviceToDevice, st));
    return 0;
}

// V^ of a complex panel (64 complex reflectors, 128 real vectors) into vpk2[0]
static int pack_complex_panel(dhqr_context* c, cudaStream_t st, const double2* P, int64_t lda, int64_t mpc, int kb, int64_t vrows) {
    dim3 grid((unsigned)std::min<int64_t>((vrows + 255) / 256, 4 * c->sms), NBMAX);
    return launch(c, st, "k_pack_c", 0.0, [&](CwtSlot) { k_pack_c<<<grid, 256, 0, st>>>(P, lda, mpc, kb, c->vpk2[0], 0, vrows); });
}

// b <- Q^H b (notrans = 0) or b <- Q b = H_1 ... H_n b (notrans = 1) with the first n reflectors of a single-GPU factorisation,
// n > 0.  Float64: the one-vector sweep (qt_vec_ok) or the 128-column panels of apply_qt_local.
static int apply_q_local(dhqr_context* c, cudaStream_t st, int64_t m, int64_t n, const double* A, int64_t lda, double* b, int64_t ldb,
                         int nrhs, int notrans) {
    TRY(ensure_workspace(c, st, m, std::max<int64_t>(n, nrhs)));
    if (qt_vec_ok(c, m, nrhs)) {
        TRY(qt_prepare(c, st, m, 0, n, A, lda));
        return apply_qt_local_vec(c, st, m, 0, n, A, lda, b, notrans);
    }
    return apply_qt_local(c, st, m, 0, n, A, lda, b, ldb, nrhs, notrans);
}

// ComplexF64 (S:232-242): panel by panel, last to first for Q b, each as the real block reflector of its 128 vectors [v_r, v_i]
// on the real view of b (I - V T' V' for Q^H b, I - V T V' for Q b)
static int apply_q_local(dhqr_context* c, cudaStream_t st, int64_t m, int64_t n, const double2* A, int64_t lda, double2* b, int64_t ldb,
                         int nrhs, int notrans) {
    TRY(ensure_workspace(c, st, 2 * m, std::max<int64_t>(n, nrhs)));
    const int64_t last = ((n - 1) / CPW) * CPW;
    for (int64_t p = 0; p <= last; p += CPW) {
        const int64_t c0 = notrans ? last - p : p;
        const int kb = (int)std::min<int64_t>(CPW, n - c0);
        const int64_t mpc = m - c0, rows = 2 * mpc, vrows = rup(rows, 128);
        TRY(pack_complex_panel(c, st, A + c0 * lda + c0, lda, mpc, kb, vrows));
        TRY(apply_block_reflector(c, st, c->vpk2[0], c->ws[0], 0, NBMAX, rows, 0, (double*)(b + c0), 2 * ldb, nrhs, false, nullptr, 0,
                                  notrans));
    }
    return 0;
}

// The minimum-norm solution of A^H y = c, y = Q [R^{-H} c; 0], in place on b[0:m] (c = b[0:n]): forward substitution on rows
// [0, n), zero rows [n, m), then b <- H_1 ... H_n b.  The body of dhqr_solve_adj_*, also the second stage of dhqr_solve_cod_*.
template <typename T>
static int solve_adj_local(dhqr_context* c, cudaStream_t st, int64_t m, int64_t n, const T* A, int64_t lda, const T* alpha, T* b,
                           int64_t ldb, int nrhs) {
    TRY(forwardsolve_local(c, st, n, A, lda, alpha, b, ldb, nrhs));
    if (m > n) CU(cudaMemset2DAsync(b + n, (size_t)ldb * sizeof(T), 0, (size_t)(m - n) * sizeof(T), nrhs, st));   // n = 0: y = 0, as in ?gels
    if (n == 0) return 0;
    return apply_q_local(c, st, m, n, A, lda, b, ldb, nrhs, 1);
}

// ------------------------------------------------------------------------------------------------
// C-ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

int dhqr_version(void) { return DHQR_VERSION; }
const char* dhqr_last_error(void) { return g_err; }

// A new context on `device` in *out; on failure *out stays empty and nothing is left behind.
static int create_context(std::unique_ptr<dhqr_context>& out, int device) {
    int ndev = 0;
    CU(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return set_err(-2, "device %d out of range (%d devices)", device, ndev);
    CU(cudaSetDevice(device));
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device));
    // sm_90a code runs on compute capability 9.0 only (architecture-specific features do not carry forward)
    if (prop.major != 9 || prop.minor != 0) return set_err(5001, "libdhqr is built for sm_90a only; device %d is sm_%d%d", device, prop.major, prop.minor);
    auto c = std::make_unique<dhqr_context>();
    c->device = device;
    c->sms = prop.multiProcessorCount;
    TRY(c->d_i64.alloc((size_t)2 * 1025));
    CU(c->copy_stream.create());
    CU(c->d2h_stream.create());
    CU(c->h2d_stream.create());
    for (int i = 0; i < 3; ++i) CU(c->cu_stream[i].create());
    {
        int lo = 0, hi = 0;
        CU(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        CU(c->hp_stream.create(hi));
        CU(c->comm_stream.create(hi));
        CU(c->hp2_stream.create(hi));
        CU(c->aux_stream.create(hi));
        for (int i = 0; i < 4; ++i) CU(c->ev_aux[i].create(cudaEventDisableTiming));
    }
    // the batched kernels size their shared memory per shape; set here so that no batched call does anything but enqueue
    const int optin = (int)prop.sharedMemPerBlockOptin;
    CU(cudaFuncSetAttribute(k_qr_batched, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
    CU(cudaFuncSetAttribute(k_apply_batched<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
    CU(cudaFuncSetAttribute(k_apply_batched<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
    CU(cudaFuncSetAttribute(k_apply_batched<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
    CU(cudaFuncSetAttribute(k_tp_batched<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
    CU(cudaFuncSetAttribute(k_tp_batched<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
    CU(cudaFuncSetAttribute(k_backsolve_batched, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
    out = std::move(c);
    return 0;
}

int dhqr_create(dhqr_handle* h, int device) {
    if (!h) return set_err(-1, "null handle pointer");
    std::unique_ptr<dhqr_context> c;
    TRY(create_context(c, device));
    *h = c.release();
    return 0;
}

int dhqr_nccl_unique_id(void* out) {
    if (!out) return set_err(-1, "null output");
    TRY(load_nccl());
    ncclUniqueId id;
    NC(g_nccl.GetUniqueId(&id));
    memcpy(out, &id, sizeof(id));
    return 0;
}

int dhqr_create_dist(dhqr_handle* h, int device, const void* unique_id, int rank, int nranks) {
    if (nranks < 1 || nranks > 1024) return set_err(-5, "nranks out of range");
    if (rank < 0 || rank >= nranks) return set_err(-4, "rank out of range");
    if (nranks > 1 && !unique_id) return set_err(-3, "null unique id");
    if (!h) return set_err(-1, "null handle pointer");
    if (nranks > 1) TRY(load_nccl());
    std::unique_ptr<dhqr_context> c;
    TRY(create_context(c, device));
    c->rank = rank;
    c->nranks = nranks;
    if (nranks > 1) {
        ncclUniqueId id;
        memcpy(&id, unique_id, sizeof(id));
        NC(g_nccl.CommInitRank(&c->comm, nranks, id, rank));
    }
    *h = c.release();
    return 0;
}

int dhqr_destroy(dhqr_handle c) {
    if (!c) return 0;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    if (c->comm) g_nccl.CommDestroy(c->comm);   // before the buffers it may still reference are freed
    delete c;
    return 0;
}

int dhqr_set_option(dhqr_handle c, const char* key, int64_t value) {
    if (!c) return set_err(-1, "null handle");
    if (!key) return set_err(-2, "null key");
    if (!strcmp(key, "nb")) {
        if (value < 32 || value > 128 || value % 32) return set_err(-3, "nb must be a multiple of 32 in [32,128]");
        c->nb = (int)value;
    } else if (!strcmp(key, "panel_ctas")) {
        if (value < 0) return set_err(-3, "panel_ctas < 0");
        c->panel_ctas = (int)value;
    } else if (!strcmp(key, "sync")) {
        c->sync = value ? 1 : 0;
    } else if (!strcmp(key, "profile")) {
        c->profile = value ? 1 : 0;
    } else if (!strcmp(key, "lookahead")) {
        c->lookahead = value ? 1 : 0;
    } else if (!strcmp(key, "host_trace")) {
        c->host_trace = value ? 1 : 0;
    } else if (!strcmp(key, "host_chunk")) {
        if (value < 0 || value % 128) return set_err(-3, "host_chunk must be a non-negative multiple of 128");
        c->host_chunk = (int)value;
    } else if (!strcmp(key, "host_first")) {
        if (value < 0) return set_err(-3, "host_first < 0");
        c->host_first = (int)value;
    } else if (!strcmp(key, "host_h2d_gbs")) {
        if (value < 1) return set_err(-3, "host_h2d_gbs < 1");
        c->host_h2d_gbs = (int)value;
    } else if (!strcmp(key, "host_chain_us")) {
        if (value < 1) return set_err(-3, "host_chain_us < 1");
        c->host_chain_us = (int)value;
    } else if (!strcmp(key, "host_cu_streams")) {
        if (value < 1 || value > 3) return set_err(-3, "host_cu_streams must be 1, 2 or 3");
        c->host_cu_streams = (int)value;
    } else if (!strcmp(key, "host_tflops")) {
        if (value < 1) return set_err(-3, "host_tflops < 1");
        c->host_tflops = (int)value;
    } else if (!strcmp(key, "qt_vec")) {
        c->qt_vec = value ? 1 : 0;
    } else if (!strcmp(key, "bs_wave")) {
        c->bs_wave = value ? 1 : 0;
    } else if (!strcmp(key, "unblocked_wave")) {
        c->unblocked_wave = value ? 1 : 0;
    } else if (!strcmp(key, "fuse_house")) {
        c->fuse_house = value ? 1 : 0;
    } else if (!strcmp(key, "cvy_persist")) {
        if (value < 0 || value > 1 << 20) return set_err(-3, "cvy_persist out of range");
        c->cvy_persist = (int)value;
    } else if (!strcmp(key, "la_trace")) {
        c->la_trace = value ? 1 : 0;
    } else if (!strcmp(key, "chain_wait_trace")) {
        if (value && !c->cwt_stamps) TRY(c->cwt_stamps.alloc((size_t)2 * CWT_MAX));
        c->chain_wait_trace = value ? 1 : 0;
    } else if (!strcmp(key, "panel_fast")) {
        c->panel_fast = value ? 1 : 0;
    } else if (!strcmp(key, "wide_panel")) {
        c->wide_panel = value ? 1 : 0;
    } else if (!strcmp(key, "wide_kappa")) {
        if (value < 1) return set_err(-3, "wide_kappa < 1");
        c->wide_kappa = (double)value;
    } else if (!strcmp(key, "wide_trace")) {
        c->wide_trace = value ? 1 : 0;
    } else if (!strcmp(key, "gemm_trace")) {
        // 1: start over with zero rows (no stream here: the fill is complete before the call returns); 0: stop tracing, keep the rows
        if (value) {
            CU(cudaSetDevice(c->device));
            if (!c->gtr_rows) TRY(c->gtr_rows.alloc(GTR_MAX_CTAS * GTR_WORDS));
            CU(cudaMemset(c->gtr_rows.p, 0, GTR_MAX_CTAS * GTR_WORDS * sizeof(unsigned long long)));
            CU(cudaStreamSynchronize(cudaStreamLegacy));
            c->gtr_used = c->gtr_dropped = 0;
        }
        c->gemm_trace = value ? 1 : 0;
    } else if (!strcmp(key, "epoch_near_wrap")) {
        // test hook: the tag counters two launches short of their reset (never backwards, so no tag a cell holds comes back);
        // a counter whose buffer is allocated later starts over at 0 with it
        if (value != 1) return set_err(-3, "epoch_near_wrap takes the value 1");
        c->ll_epoch = std::max(c->ll_epoch, LL_EPOCH_MAX - 2 * (IB + 8) + 1);
        c->bs_epoch = std::max(c->bs_epoch, WAVE_EPOCH_MAX - 1);
        c->uw_epoch = std::max(c->uw_epoch, WAVE_EPOCH_MAX - 1);
    } else if (!strcmp(key, "panel_trace")) {
        if (value && !c->panel_trace) {
            // no stream here: the fill is complete before the call returns, so every later call sees it
            TRY(c->panel_trace.ensure((size_t)PANEL_MAXG * IB * 8, cudaStreamLegacy));
            CU(cudaStreamSynchronize(cudaStreamLegacy));
        } else if (!value && c->panel_trace) {
            CU(c->panel_trace.release());
        }
    } else {
        return set_err(-2, "unknown option '%s'", key);
    }
    return 0;
}

int dhqr_get_option(dhqr_handle c, const char* key, int64_t* value) {
    if (!c) return set_err(-1, "null handle");
    if (!key) return set_err(-2, "null key");
    if (!value) return set_err(-3, "null value");
    if (!strcmp(key, "nb")) *value = c->nb;
    else if (!strcmp(key, "panel_ctas")) *value = c->panel_ctas;
    else if (!strcmp(key, "sync")) *value = c->sync;
    else if (!strcmp(key, "profile")) *value = c->profile;
    else if (!strcmp(key, "lookahead")) *value = c->lookahead;
    else if (!strcmp(key, "panel_fast")) *value = c->panel_fast;
    else if (!strcmp(key, "wide_panel")) *value = c->wide_panel;
    else if (!strcmp(key, "cvy_persist")) *value = c->cvy_persist;
    else if (!strcmp(key, "qt_vec")) *value = c->qt_vec;
    else if (!strcmp(key, "bs_wave")) *value = c->bs_wave;
    else if (!strcmp(key, "unblocked_wave")) *value = c->unblocked_wave;
    else if (!strcmp(key, "fuse_house")) *value = c->fuse_house;
    else if (!strcmp(key, "host_chunk")) *value = c->host_chunk;
    else if (!strcmp(key, "wide_panels")) *value = c->wide_panels;
    else if (!strcmp(key, "wide_redone")) *value = c->wide_redone;
    else if (!strcmp(key, "pair_units")) *value = c->pair_units;
    else if (!strcmp(key, "qrcp_renorms")) {
        unsigned long long r = 0;
        if (c->qp_ctl) CU(cudaMemcpy(&r, &c->qp_ctl.p->renorms, sizeof(r), cudaMemcpyDeviceToHost));
        *value = (int64_t)r;
    }
    else if (!strcmp(key, "panels_fast") || !strcmp(key, "panels_fallback")) {
        int st2[2] = {0, 0};
        if (c->fast_stats) CU(cudaMemcpy(st2, c->fast_stats, sizeof(st2), cudaMemcpyDeviceToHost));
        *value = st2[!strcmp(key, "panels_fallback") ? 1 : 0];
    }
    else if (!strcmp(key, "sms")) *value = c->sms;
    else if (!strcmp(key, "append_max_rows")) *value = narrow_panel_max_rows(c);
    else if (!strcmp(key, "batch_max_elems")) *value = BQ_MAX_ELEMS;
    else if (!strcmp(key, "batch_update_max_cols")) *value = BQ_UPD_MAX_COLS;
    else if (!strcmp(key, "rank")) *value = c->rank;
    else if (!strcmp(key, "nranks")) *value = c->nranks;
    else return set_err(-2, "unknown option '%s'", key);
    return 0;
}

int dhqr_launch_count(dhqr_handle c, int64_t* count) {
    if (!c) return set_err(-1, "null handle");
    if (!count) return set_err(-2, "null count");
    *count = c->launches;
    return 0;
}

static int prof_drain(dhqr_context* c) {
    for (auto& r : c->prof_pending) {
        float ms = 0.f;
        CU(cudaEventSynchronize(r.e1));
        CU(cudaEventElapsedTime(&ms, r.e0, r.e1));
        c->prof_slots[r.slot].ms += ms;
        c->prof_slots[r.slot].count += 1;
    }
    c->prof_pending.clear();
    return 0;
}

int dhqr_profile_reset(dhqr_handle c) {
    if (!c) return set_err(-1, "null handle");
    TRY(prof_drain(c));
    for (auto& s : c->prof_slots) { s.ms = 0.0; s.count = 0; s.work = 0.0; }
    return 0;
}

int dhqr_profile_get(dhqr_handle c, int index, char* name, int name_len, double* ms, int64_t* count, double* work) {
    if (!c) return set_err(-1, "null handle");
    TRY(prof_drain(c));
    if (index < 0 || index >= (int)c->prof_slots.size()) return set_err(-2, "index out of range");
    const auto& s = c->prof_slots[index];
    if (name && name_len > 0) { strncpy(name, s.name, name_len - 1); name[name_len - 1] = 0; }
    if (ms) *ms = s.ms;
    if (count) *count = s.count;
    if (work) *work = s.work;
    return 0;
}

int dhqr_qr_f64(dhqr_handle c, int64_t m, int64_t n_global, int64_t col0, int64_t n_local, double* dA, int64_t lda,
                double* d_alpha, int nb, void* stream) {
    Check a(c);
    column_block(a, m, n_global, col0, n_local);
    a.operand<double>(6, "A", dA, mat(m, n_local, lda), when(n_local > 0, NEED));
    a.operand<double>(8, "alpha", d_alpha, vec(n_global), when(n_global > 0, NEED));
    a.require(nb == 0 || nb == 1 || (nb >= 32 && nb <= 128 && nb % 32 == 0), 9, "nb must be 0, 1 or a multiple of 32 in [32,128]");
    TRY(a);
    if (nb == 0) nb = c->nb;
    if (n_global == 0) return 0;
    CU(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    if (nb == 1) return qr_unblocked(c, st, m, n_global, col0, n_local, dA, lda, d_alpha);
    return qr_blocked(c, st, m, n_global, col0, n_local, dA, lda, d_alpha, nb);
}

// The rows x nrhs block of b as one contiguous message for the rank-to-rank hand-over.  With ldb > rows and nrhs > 1 the rows
// between its columns are the caller's padding, which must neither travel nor be overwritten by another rank's: the block is
// then packed into handle workspace (*msg = c->xfer) and unpacked after.  Otherwise *msg = b.
static int rhs_message(dhqr_context* c, cudaStream_t st, double* b, int64_t ldb, int64_t rows, int nrhs, double** msg) {
    *msg = b;
    if (ldb == rows || nrhs == 1) return 0;
    TRY(c->xfer.ensure((size_t)rows * nrhs, st));
    *msg = c->xfer;
    return 0;
}
static int rhs_copy(cudaStream_t st, double* dst, int64_t lddst, const double* src, int64_t ldsrc, int64_t rows, int nrhs) {
    if (dst == src) return 0;
    CU(cudaMemcpy2DAsync(dst, (size_t)lddst * 8, src, (size_t)ldsrc * 8, (size_t)rows * 8, nrhs, cudaMemcpyDeviceToDevice, st));
    return 0;
}

// b <- Q^H b (notrans = 0) or b <- Q b (notrans = 1).  The owners act on b one after the other and b travels rank to rank: in rank
// order for Q^H b (C3, S:227-229), in reverse rank order for Q b = H_1 ... H_n b.  The last owner to act broadcasts the result.
static int apply_q_dist(dhqr_context* c, int64_t m, int64_t n_global, int64_t col0, int64_t n_local, const double* dA, int64_t lda,
                        double* d_b, int64_t ldb, int nrhs, void* stream, int notrans) {
    Check a(c);
    column_block(a, m, n_global, col0, n_local);
    a.operand<double>(6, "A", dA, mat(m, n_local, lda), when(n_local > 0, NEED));
    a.operand<double>(8, "b", d_b, mat(m, nrhs, ldb), when(nrhs > 0, NEED));
    a.require(nrhs >= 0, 10, "nrhs < 0");
    TRY(a);
    if (n_global == 0 || nrhs == 0) return 0;
    CU(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<int64_t> col0s, nls;
    TRY(gather_partition(c, st, col0, n_local, col0s, nls));
    TRY(check_partition(col0s, nls, n_global));
    TRY(ensure_workspace(c, st, m, std::max<int64_t>(n_local, nrhs)));
    const int step = notrans ? -1 : 1, first = notrans ? c->nranks - 1 : 0, last = notrans ? 0 : c->nranks - 1;
    const size_t cnt = (size_t)m * nrhs;
    double* msg = d_b;
    if (c->nranks > 1) TRY(rhs_message(c, st, d_b, ldb, m, nrhs, &msg));
    const bool vec = qt_vec_ok(c, m, nrhs);
    if (vec) TRY(qt_prepare(c, st, m, col0, n_local, dA, lda));
    if (c->nranks > 1 && c->rank != first) {
        NC(g_nccl.Recv(msg, cnt, ncclFloat64, c->rank - step, c->comm, st));
        TRY(rhs_copy(st, d_b, ldb, msg, m, m, nrhs));
    }
    if (vec) TRY(apply_qt_local_vec(c, st, m, col0, n_local, dA, lda, d_b, notrans));
    else TRY(apply_qt_local(c, st, m, col0, n_local, dA, lda, d_b, ldb, nrhs, notrans));
    if (c->nranks > 1) {
        TRY(rhs_copy(st, msg, m, d_b, ldb, m, nrhs));
        if (c->rank != last) NC(g_nccl.Send(msg, cnt, ncclFloat64, c->rank + step, c->comm, st));
        NC(g_nccl.Broadcast(msg, msg, cnt, ncclFloat64, last, c->comm, st));
        if (c->rank != last) TRY(rhs_copy(st, d_b, ldb, msg, m, m, nrhs));
    }
    return 0;
}

int dhqr_apply_qt_f64(dhqr_handle c, int64_t m, int64_t n_global, int64_t col0, int64_t n_local, const double* dA,
                      int64_t lda, double* d_b, int64_t ldb, int nrhs, void* stream) {
    return apply_q_dist(c, m, n_global, col0, n_local, dA, lda, d_b, ldb, nrhs, stream, 0);
}

int dhqr_apply_q_f64(dhqr_handle c, int64_t m, int64_t n_global, int64_t col0, int64_t n_local, const double* dA,
                     int64_t lda, double* d_b, int64_t ldb, int nrhs, void* stream) {
    return apply_q_dist(c, m, n_global, col0, n_local, dA, lda, d_b, ldb, nrhs, stream, 1);
}

int dhqr_backsolve_f64(dhqr_handle c, int64_t m, int64_t n_global, int64_t col0, int64_t n_local, const double* dA,
                       int64_t lda, const double* d_alpha, double* d_b, int64_t ldb, int nrhs, void* stream) {
    Check a(c);
    column_block(a, m, n_global, col0, n_local);
    a.operand<double>(6, "A", dA, mat(m, n_local, lda), when(n_local > 0, NEED));
    a.operand<double>(8, "alpha", d_alpha, vec(n_global), when(n_global > 0, NEED));
    a.operand<double>(9, "b", d_b, mat(m, nrhs, ldb), when(nrhs > 0, NEED));
    a.require(nrhs >= 0, 11, "nrhs < 0");
    TRY(a);
    if (n_global == 0 || nrhs == 0) return 0;
    CU(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<int64_t> col0s, nls;
    TRY(gather_partition(c, st, col0, n_local, col0s, nls));
    TRY(check_partition(col0s, nls, n_global));
    TRY(c->xbuf.ensure((size_t)n_global * nrhs, st));
    TRY(wave_prepare(c, st, n_local));
    // C4 (S:260-267), column oriented: the last owner solves its block of unknowns and removes their
    // contribution from the rows above; the partially reduced right-hand side then moves one rank down.
    const size_t cnt = (size_t)n_global * nrhs;
    double* msg = d_b;
    if (c->nranks > 1) TRY(rhs_message(c, st, d_b, ldb, n_global, nrhs, &msg));
    if (c->nranks > 1 && c->rank + 1 < c->nranks) {
        NC(g_nccl.Recv(msg, cnt, ncclFloat64, c->rank + 1, c->comm, st));
        NC(g_nccl.Recv(c->xbuf, (size_t)n_global * nrhs, ncclFloat64, c->rank + 1, c->comm, st));
        TRY(rhs_copy(st, d_b, ldb, msg, n_global, n_global, nrhs));
    }
    TRY(backsolve_local(c, st, col0, n_local, dA, lda, d_alpha, d_b, ldb, nrhs, c->xbuf, n_global));
    if (c->nranks > 1) {
        if (c->rank > 0) {
            TRY(rhs_copy(st, msg, n_global, d_b, ldb, n_global, nrhs));
            NC(g_nccl.Send(msg, cnt, ncclFloat64, c->rank - 1, c->comm, st));
            NC(g_nccl.Send(c->xbuf, (size_t)n_global * nrhs, ncclFloat64, c->rank - 1, c->comm, st));
        }
        NC(g_nccl.Broadcast(c->xbuf, c->xbuf, (size_t)n_global * nrhs, ncclFloat64, 0, c->comm, st));
    }
    CU(cudaMemcpy2DAsync(d_b, (size_t)ldb * 8, c->xbuf, (size_t)n_global * 8, (size_t)n_global * 8, nrhs,
                         cudaMemcpyDeviceToDevice, st));
    return 0;
}

int dhqr_solve_f64(dhqr_handle c, int64_t m, int64_t n_global, int64_t col0, int64_t n_local, const double* dA,
                   int64_t lda, const double* d_alpha, double* d_b, int64_t ldb, int nrhs, void* stream) {
    // Every argument before Q'b runs.  b, ldb and nrhs keep the codes of dhqr_apply_qt_f64, which reports them in its numbering.
    Check a(c);
    column_block(a, m, n_global, col0, n_local);
    a.operand<double>(6, "A", dA, mat(m, n_local, lda), when(n_local > 0, NEED));
    a.operand<double>(8, "alpha", d_alpha, vec(n_global), when(n_global > 0, NEED));
    a.operand<double>(8, "b", d_b, mat(m, nrhs, ldb), when(nrhs > 0, NEED));
    a.require(nrhs >= 0, 10, "nrhs < 0");
    TRY(a);
    TRY(dhqr_apply_qt_f64(c, m, n_global, col0, n_local, dA, lda, d_b, ldb, nrhs, stream));   // S:288
    return dhqr_backsolve_f64(c, m, n_global, col0, n_local, dA, lda, d_alpha, d_b, ldb, nrhs, stream);   // S:291
}

// ---- ComplexF64 (S:9, S:51-59, S:162-196; test/runtests.jl:43) -------------------------------------------------------
// Panels of 64 complex columns: complex column-by-column panel, then the trailing update as the REAL block reflector of the
// 128 vectors [v_r, v_i] on the real view of the matrix (dhqr_complex.cuh).  Single GPU.
static const char* const C64_PATH = "the ComplexF64 path";
static const char* const C64_BLOCK = "the ComplexF64 path is single-GPU (col0 = 0, n_local = n_global)";

static int qr_c64_local(dhqr_context* c, cudaStream_t st, int64_t m, int64_t n, double2* A, int64_t lda, double2* alpha);

int dhqr_qr_c64(dhqr_handle c, int64_t m, int64_t n_global, int64_t col0, int64_t n_local, void* dA, int64_t lda, void* d_alpha,
                void* stream) {
    Check a(c, C64_PATH);
    column_block(a, m, n_global, col0, n_local);
    a.require(col0 == 0 && n_local == n_global, 1, C64_BLOCK);
    a.operand<double2>(6, "A", dA, mat(m, n_local, lda), when(n_local > 0, NEED) | ALIGN);
    a.operand<double2>(8, "alpha", d_alpha, vec(n_global), when(n_global > 0, NEED) | ALIGN);
    TRY(a);
    if (n_global == 0) return 0;
    CU(cudaSetDevice(c->device));
    return qr_c64_local(c, (cudaStream_t)stream, m, n_global, (double2*)dA, lda, (double2*)d_alpha);
}

// the body of dhqr_qr_c64 (n > 0), also the second factorisation of dhqr_cod_c64
static int qr_c64_local(dhqr_context* c, cudaStream_t st, int64_t m, int64_t n, double2* A, int64_t lda, double2* alpha) {
    TRY(ensure_workspace(c, st, 2 * m, n));
    for (int64_t c0 = 0; c0 < n; c0 += CPW) {
        const int kb = (int)std::min<int64_t>(CPW, n - c0);
        double2* P = A + c0 * lda + c0;
        const int64_t mpc = m - c0;
        for (int j = 0; j < kb; ++j) {                       // S:127-144 restricted to the panel
            double2* col = P + (int64_t)j * lda + j;
            TRY(launch(c, st, "k_house1_c", 0.0, [&](CwtSlot) { k_house1_c<<<1, 1024, 0, st>>>(col, mpc - j, alpha + c0 + j); }));
            if (j + 1 < kb) {
                TRY(launch(c, st, "k_apply1_c", 0.0, [&](CwtSlot) {
                    k_apply1_c<<<kb - j - 1, 256, 0, st>>>(col, mpc - j, col + lda, lda, kb - j - 1);
                }));
            }
        }
        const int64_t t0 = c0 + kb;
        if (t0 < n) {                                        // S:198-213 for the columns right of the panel, blocked
            const int64_t rows = 2 * mpc, vrows = rup(rows, 128);
            TRY(pack_complex_panel(c, st, P, lda, mpc, kb, vrows));
            TRY(apply_block_reflector(c, st, c->vpk2[0], c->ws[0], 0, NBMAX, rows, 0, (double*)(A + t0 * lda + c0), 2 * lda, (int)(n - t0)));
        }
    }
    return 0;
}

int dhqr_apply_qt_c64(dhqr_handle c, int64_t m, int64_t n_global, int64_t col0, int64_t n_local, const void* dA, int64_t lda,
                      void* d_b, int64_t ldb, int nrhs, void* stream) {
    Check a(c, C64_PATH);
    column_block(a, m, n_global, col0, n_local);
    a.require(col0 == 0 && n_local == n_global, 1, C64_BLOCK);
    a.operand<double2>(6, "A", dA, mat(m, n_local, lda), when(n_local > 0, NEED) | ALIGN);
    a.operand<double2>(8, "b", d_b, mat(m, nrhs, ldb), when(nrhs > 0, NEED) | ALIGN);
    a.require(nrhs >= 0, 10, "nrhs < 0");
    TRY(a);
    if (n_global == 0 || nrhs == 0) return 0;
    CU(cudaSetDevice(c->device));
    return apply_q_local(c, (cudaStream_t)stream, m, n_global, (const double2*)dA, lda, (double2*)d_b, ldb, nrhs, 0);
}

int dhqr_backsolve_c64(dhqr_handle c, int64_t m, int64_t n_global, int64_t col0, int64_t n_local, const void* dA, int64_t lda,
                       const void* d_alpha, void* d_b, int64_t ldb, int nrhs, void* stream) {
    Check a(c, C64_PATH);
    column_block(a, m, n_global, col0, n_local);
    a.require(col0 == 0 && n_local == n_global, 1, C64_BLOCK);
    a.operand<double2>(6, "A", dA, mat(m, n_local, lda), when(n_local > 0, NEED) | ALIGN);
    a.operand<double2>(8, "alpha", d_alpha, vec(n_global), when(n_global > 0, NEED) | ALIGN);
    a.operand<double2>(9, "b", d_b, mat(m, nrhs, ldb), when(nrhs > 0, NEED) | ALIGN);
    a.require(nrhs >= 0, 11, "nrhs < 0");
    TRY(a);
    if (n_global == 0 || nrhs == 0) return 0;
    CU(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t n = n_global;
    TRY(c->xbuf.ensure((size_t)2 * n * nrhs, st));
    double2* x = (double2*)c->xbuf.p;
    TRY(backsolve_single(c, st, n, (const double2*)dA, lda, (const double2*)d_alpha, (double2*)d_b, ldb, nrhs, x));
    CU(cudaMemcpy2DAsync(d_b, (size_t)ldb * 16, x, (size_t)n * 16, (size_t)n * 16, nrhs, cudaMemcpyDeviceToDevice, st));
    return 0;
}

int dhqr_solve_c64(dhqr_handle c, int64_t m, int64_t n_global, int64_t col0, int64_t n_local, const void* dA, int64_t lda,
                   const void* d_alpha, void* d_b, int64_t ldb, int nrhs, void* stream) {
    Check a(c, C64_PATH);                                                                       // every argument, before Q'b runs
    column_block(a, m, n_global, col0, n_local);
    a.require(col0 == 0 && n_local == n_global, 1, C64_BLOCK);
    a.operand<double2>(6, "A", dA, mat(m, n_local, lda), when(n_local > 0, NEED) | ALIGN);
    a.operand<double2>(8, "alpha", d_alpha, vec(n_global), when(n_global > 0, NEED) | ALIGN);
    a.operand<double2>(9, "b", d_b, mat(m, nrhs, ldb), when(nrhs > 0, NEED) | ALIGN);
    a.require(nrhs >= 0, 11, "nrhs < 0");
    TRY(a);
    TRY(dhqr_apply_qt_c64(c, m, n_global, col0, n_local, dA, lda, d_b, ldb, nrhs, stream));                   // S:288
    return dhqr_backsolve_c64(c, m, n_global, col0, n_local, dA, lda, d_alpha, d_b, ldb, nrhs, stream);       // S:291
}

// ---- explicit thin Q (LAPACK orgqr / ungqr) ---------------------------------------------------------------------------------
// Q <- H_1 ... H_n [I_n; 0], accumulated backwards over panels p = last .. 0 with columns [cs, cs + kb): pack V_p from A, make the
// panel's columns of Q those of the identity (all m rows, which also clears R's rows when Q is A), then apply I - V_p T_p V_p'
// (T, not T') to rows >= cs, columns [cs, n) of Q.  Columns left of cs are still unit vectors with zeros in rows >= cs, so the
// panel leaves them alone: 2mn^2 - 2n^3/3 flops instead of the 4mn^2 - 2n^3 of Q applied to [I; 0].  V_p is packed before its
// columns are overwritten, so in place and out of place are the same sweep.
static int eye_cols(dhqr_context* c, cudaStream_t st, void* Q, bool cplx, int64_t ldq, int64_t m, int64_t c0, int kb) {
    const dim3 grid((unsigned)std::min<int64_t>((m + 255) / 256, 64), kb);
    return launch(c, st, cplx ? "k_eye_cols_c" : "k_eye_cols", 0.0, [&](CwtSlot) {
        if (cplx) k_eye_cols<double2><<<grid, 256, 0, st>>>((double2*)Q, ldq, m, c0);
        else k_eye_cols<double><<<grid, 256, 0, st>>>((double*)Q, ldq, m, c0);
    });
}

int dhqr_form_q_f64(dhqr_handle c, int64_t m, int64_t n, const double* dA, int64_t lda, double* dQ, int64_t ldq, void* stream) {
    Check a(c, "form_q");                                        // Float64 pointers are not checked for alignment here
    a.require(m >= 0, 2, "m < 0");
    a.require(n >= 0 && n <= m, 3, "need 0 <= n <= m");
    a.operand<double>(4, "A", dA, mat(m, n, lda), when(n > 0, NEED));
    a.operand<double>(6, "Q", dQ, mat(m, n, ldq), when(n > 0, NEED) | DISJOINT | OR_SAME);
    TRY(a);
    if (n == 0) return 0;
    CU(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    TRY(ensure_workspace(c, st, m, n));
    TRY(qt_prepare(c, st, m, 0, n, dA, lda));                    // T' of every panel, from A before the sweep writes anything
    for (int64_t p = (n - 1) / NBMAX; p >= 0; --p) {
        const int64_t cs = p * NBMAX, rows = m - cs, vrows = rup(rows, 128);   // cs is 128-aligned: the window starts at row cs
        const int kb = (int)std::min<int64_t>(NBMAX, n - cs);
        TRY(pack_v(c, st, dA + cs * lda + cs, lda, rows, kb, 1, c->vpk2[0], 0, vrows, NBMAX));
        TRY(eye_cols(c, st, dQ, false, ldq, m, cs, kb));
        TRY(apply_block_reflector(c, st, c->vpk2[0], c->ws[0], 0, NBMAX, rows, 0, dQ + cs * ldq + cs, ldq, (int)(n - cs), true,
                                  c->qt_T + (size_t)p * NBMAX * NBMAX, 0, 1));
    }
    return 0;
}

// ComplexF64: the same sweep over 64-column complex panels on the real view of Q (2m x n, leading dimension 2 ldq), each panel the
// real block reflector of its 128 vectors [v_r, v_i] (dhqr_complex.cuh); T from the Gram block of the update itself.
int dhqr_form_q_c64(dhqr_handle c, int64_t m, int64_t n, const void* dA, int64_t lda, void* dQ, int64_t ldq, void* stream) {
    Check a(c, "form_q");
    a.require(m >= 0, 2, "m < 0");
    a.require(n >= 0 && n <= m, 3, "need 0 <= n <= m");
    a.operand<double2>(4, "A", dA, mat(m, n, lda), when(n > 0, NEED) | ALIGN);
    a.operand<double2>(6, "Q", dQ, mat(m, n, ldq), when(n > 0, NEED) | ALIGN | DISJOINT | OR_SAME);
    TRY(a);
    if (n == 0) return 0;
    CU(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    TRY(ensure_workspace(c, st, 2 * m, n));
    const double2* A = (const double2*)dA;
    double2* Q = (double2*)dQ;
    for (int64_t c0 = ((n - 1) / CPW) * CPW; c0 >= 0; c0 -= CPW) {
        const int kb = (int)std::min<int64_t>(CPW, n - c0);
        const int64_t mpc = m - c0, rows = 2 * mpc, vrows = rup(rows, 128);
        TRY(pack_complex_panel(c, st, A + c0 * lda + c0, lda, mpc, kb, vrows));
        TRY(eye_cols(c, st, Q, true, ldq, m, c0, kb));
        TRY(apply_block_reflector(c, st, c->vpk2[0], c->ws[0], 0, NBMAX, rows, 0, (double*)(Q + c0 * ldq + c0), 2 * ldq, (int)(n - c0),
                                  false, nullptr, 0, 1));
    }
    return 0;
}

// ---- solves with the adjoint (LAPACK ?gels, TRANS = 'C') ------------------------------------------------------------------
// forwardsolve: b[0:n] <- R^{-H} b[0:n].  solve_adj: the minimum-norm solution of A^H y = c (solve_adj_local).  Single GPU.
// Templates and overloads over the element type, which C linkage does not allow, sit in extern "C++" blocks; the dhqr_* functions
// keep the C linkage of their declarations in dhqr.h.
extern "C++" {

// dhqr_forwardsolve_* (forward) and dhqr_solve_adj_*: the same arguments
template <typename T>
static int adjoint_solve(dhqr_context* c, int64_t m, int64_t n, const void* dA, int64_t lda, const void* d_alpha, void* d_b, int64_t ldb,
                         int nrhs, void* stream, bool forward) {
    const unsigned align = when(std::is_same<T, double2>::value, ALIGN);   // Float64 pointers are not checked for alignment here
    Check a(c, "the adjoint solve");
    a.require(m >= 0, 2, "m < 0");
    a.require(n >= 0 && n <= m, 3, "need 0 <= n <= m");
    a.operand<T>(4, "A", dA, mat(m, n, lda), when(n > 0, NEED) | align);
    a.operand<T>(6, "alpha", d_alpha, vec(n), when(n > 0, NEED) | align);
    a.operand<T>(7, "b", d_b, mat(m, nrhs, ldb), when(nrhs > 0, NEED) | align);
    a.require(nrhs >= 0, 9, "nrhs < 0");
    TRY(a);
    if ((forward ? n : m) == 0 || nrhs == 0) return 0;
    CU(cudaSetDevice(c->device));
    if (forward) return forwardsolve_local(c, (cudaStream_t)stream, n, (const T*)dA, lda, (const T*)d_alpha, (T*)d_b, ldb, nrhs);
    return solve_adj_local(c, (cudaStream_t)stream, m, n, (const T*)dA, lda, (const T*)d_alpha, (T*)d_b, ldb, nrhs);
}

}  // extern "C++"

int dhqr_forwardsolve_f64(dhqr_handle c, int64_t m, int64_t n, const double* dA, int64_t lda, const double* d_alpha, double* d_b,
                          int64_t ldb, int nrhs, void* stream) {
    return adjoint_solve<double>(c, m, n, dA, lda, d_alpha, d_b, ldb, nrhs, stream, true);
}

int dhqr_forwardsolve_c64(dhqr_handle c, int64_t m, int64_t n, const void* dA, int64_t lda, const void* d_alpha, void* d_b,
                          int64_t ldb, int nrhs, void* stream) {
    return adjoint_solve<double2>(c, m, n, dA, lda, d_alpha, d_b, ldb, nrhs, stream, true);
}

int dhqr_solve_adj_f64(dhqr_handle c, int64_t m, int64_t n, const double* dA, int64_t lda, const double* d_alpha, double* d_b,
                       int64_t ldb, int nrhs, void* stream) {
    return adjoint_solve<double>(c, m, n, dA, lda, d_alpha, d_b, ldb, nrhs, stream, false);
}

int dhqr_solve_adj_c64(dhqr_handle c, int64_t m, int64_t n, const void* dA, int64_t lda, const void* d_alpha, void* d_b, int64_t ldb,
                       int nrhs, void* stream) {
    return adjoint_solve<double2>(c, m, n, dA, lda, d_alpha, d_b, ldb, nrhs, stream, false);
}

// ---- QR with column pivoting (LAPACK ?geqp3 / ?laqps, dhqr_qrcp.cuh), Float64 and ComplexF64 ---------------------------------
// Panels of QP_NB columns, four launches per column, then the trailing update A[k0+32:, k0+32:] -= V F^H (qrcp_update).  A column
// whose norm downdate fails LAPACK's tol3z test is renormed exactly inside the panel, before the next pivot is chosen, instead of
// ending the panel early: every panel has its static width and the host never needs a device value, so the driver is one static
// loop and the call does not synchronise.  Single GPU, n <= m, no row limit.  T = double or double2; the workspace is sized in
// doubles, and every section of it that holds T is aligned for T.
extern "C++" {   // as for the adjoint solves above

// A[c1:, c1:] -= V F' on the window starting at row k0 (a multiple of 32), rows >= c1 only: the 32-wide C += V Y with Y = -F'
static int qrcp_update(dhqr_context* c, cudaStream_t st, int64_t m, int64_t n, int64_t k0, int kb, double* A, int64_t lda,
                       const double* F, int64_t ldf) {
    const int64_t c1 = k0 + kb, wrows = m - k0, vrows = rup(wrows, 128);
    const int ncols = (int)(n - c1);
    TRY(pack_v(c, st, A + k0 * lda + k0, lda, wrows, kb, 1, c->vpk2[0], 0, vrows, QP_NB));
    const int64_t ytot = (int64_t)((ncols + YT - 1) / YT) * YT * LDK;
    TRY(launch(c, st, "k_qrcp_ypack", 0.0, [&](CwtSlot) {
        k_qrcp_ypack<<<(unsigned)((ytot + 255) / 256), 256, 0, st>>>(F, ldf, c1, ncols, kb, c->ws[0].ypk);
    }));
    return launch_cvy(c, st, c->vpk2[0], 0, QP_NB, c->ws[0].ypk, wrows, kb, A + c1 * lda + k0, lda, ncols, 0);
}

// A[c1:, c1:] -= V F^H on the real view of the window starting at complex row k0, real rows >= 2 kb only: the real C += V^ Y^
// through the 128-instantiation (64 real vectors: two k-chunks)
static int qrcp_update(dhqr_context* c, cudaStream_t st, int64_t m, int64_t n, int64_t k0, int kb, double2* A, int64_t lda,
                       const double2* F, int64_t ldf) {
    const int64_t c1 = k0 + kb, mpc = m - k0, wrows = 2 * mpc, vrows = rup(wrows, 128);
    const int ncols = (int)(n - c1);
    TRY(launch(c, st, "k_pack_c", 0.0, [&](CwtSlot) {
        k_pack_c<<<dim3((unsigned)std::min<int64_t>((vrows + 255) / 256, 4 * c->sms), 2 * QP_NB), 256, 0, st>>>(
            A + k0 * lda + k0, lda, mpc, kb, c->vpk2[0], 0, vrows);
    }));
    const int64_t ytot = (int64_t)((ncols + YT - 1) / YT) * QPC_NKQ * YT * LDK;
    TRY(launch(c, st, "k_qrcp_ypack_c", 0.0, [&](CwtSlot) {
        k_qrcp_ypack_c<<<(unsigned)((ytot + 255) / 256), 256, 0, st>>>(F, ldf, c1, ncols, kb, c->ws[0].ypk);
    }));
    return launch_cvy(c, st, c->vpk2[0], 0, 2 * QP_NB, c->ws[0].ypk, wrows, 2 * kb, (double*)(A + c1 * lda + k0), 2 * lda, ncols, 0);
}

template <typename T>
static int qrcp_local(dhqr_context* c, cudaStream_t st, int64_t m, int64_t n, T* A, int64_t lda, T* alpha, int64_t* jpvt) {
    constexpr int w = sizeof(T) / sizeof(double);                                      // doubles per element
    TRY(ensure_workspace(c, st, w * m, n));
    const int64_t p1 = (m + QP_PROWS - 1) / QP_PROWS;                                    // k_qrcp_pivot CTAs
    const int64_t smax = std::max<int64_t>(1, std::min<int64_t>((m + QP_THREADS - 1) / QP_THREADS, 8 * c->sms));
    // in doubles: vn1, vn2 (real); F, x, the pivot partials (real, padded to keep what follows aligned for T) and the GEMV partials
    const size_t need = (size_t)2 * n + (size_t)w * QP_NB * n + (size_t)w * m + (size_t)rup(p1, w) + (size_t)w * smax * n;
    TRY(c->qp_buf.ensure(need, st));
    TRY(c->qp_flag.ensure((size_t)n, st));
    TRY(c->qp_ctl.ensure(1, st));
    QrcpArgs<T> a;
    a.A = A; a.lda = lda; a.m = m; a.n = n; a.alpha = alpha; a.jpvt = jpvt; a.flag = c->qp_flag; a.ctl = c->qp_ctl;
    a.vn1 = c->qp_buf; a.vn2 = a.vn1 + n; a.F = (T*)(a.vn2 + n); a.ldf = n; a.x = a.F + (size_t)QP_NB * n;
    a.part1 = (double*)(a.x + m); a.part2 = (T*)(a.part1 + rup(p1, w)); a.ldp = n;
    TRY(launch(c, st, kname<T>("k_qrcp_init", "k_qrcp_init_c"), (double)sizeof(T) * (double)m * n, [&](CwtSlot) {
        k_qrcp_init<T><<<(unsigned)n, QP_THREADS, 0, st>>>(A, lda, m, a.vn1, a.vn2, jpvt, c->qp_flag);
    }));
    for (int64_t k0 = 0; k0 < n; k0 += QP_NB) {
        const int kb = (int)std::min<int64_t>(QP_NB, n - k0);
        const int tiles = (int)((n - k0 + QP_GCOLS<T> - 1) / QP_GCOLS<T>);
        for (int jj = 0; jj < kb; ++jj) {
            const int64_t j = k0 + jj, rows = m - j;
            a.j = j; a.k0 = k0; a.jj = jj;
            TRY(launch(c, st, kname<T>("k_qrcp_pivot", "k_qrcp_pivot_c"),
                       32.0 * (double)m + (double)sizeof(T) * (double)rows * (jj + 1) + 8.0 * (double)(n - j), [&](CwtSlot) {
                k_qrcp_pivot<<<(unsigned)p1, QP_THREADS, 0, st>>>(a);
            }));
            // row splits: about eight CTAs per SM in all, at least QP_THREADS rows each
            const int64_t s = std::max<int64_t>(1, std::min<int64_t>((rows + QP_THREADS - 1) / QP_THREADS,
                                                                     (8 * (int64_t)c->sms + tiles - 1) / tiles));
            a.split_rows = rup((rows + s - 1) / s, QP_THREADS);
            a.nsplit = (int)((rows + a.split_rows - 1) / a.split_rows);
            TRY(launch(c, st, kname<T>("k_qrcp_gemv", "k_qrcp_gemv_c"), (double)sizeof(T) * (double)rows * (double)(n - k0), [&](CwtSlot) {
                k_qrcp_gemv<<<dim3((unsigned)tiles, (unsigned)a.nsplit), QP_THREADS, 0, st>>>(a);
            }));
            if (j + 1 >= n) continue;
            TRY(launch(c, st, kname<T>("k_qrcp_finish", "k_qrcp_finish_c"), 0.0, [&](CwtSlot) {
                k_qrcp_finish<<<(unsigned)((n - j - 1 + QP_THREADS - 1) / QP_THREADS), QP_THREADS, 0, st>>>(a);
            }));
            TRY(launch(c, st, kname<T>("k_qrcp_renorm", "k_qrcp_renorm_c"), 0.0, [&](CwtSlot) {
                k_qrcp_renorm<<<(unsigned)std::min<int64_t>(n - j - 1, 2 * (int64_t)c->sms), QP_THREADS, 0, st>>>(a);
            }));
        }
        if (k0 + kb >= n) break;
        TRY(qrcp_update(c, st, m, n, k0, kb, A, lda, a.F, a.ldf));
    }
    return 0;
}

template <typename T>
static int qrcp_factor(dhqr_context* c, int64_t m, int64_t n, void* dA, int64_t lda, void* d_alpha, int64_t* d_jpvt, void* stream) {
    Check a(c, "the pivoted factorisation");
    a.require(m >= 0, 2, "m < 0");
    a.require(n >= 0 && n <= m, 3, "need 0 <= n <= m");
    a.operand<T>(4, "A", dA, mat(m, n, lda), when(n > 0, NEED) | ALIGN);
    a.operand<T>(6, "alpha", d_alpha, vec(n), when(n > 0, NEED) | ALIGN);
    a.operand<int64_t>(7, "jpvt", d_jpvt, vec(n), when(n > 0, NEED) | ALIGN);
    TRY(a);
    if (n == 0) return 0;
    CU(cudaSetDevice(c->device));
    return qrcp_local(c, (cudaStream_t)stream, m, n, (T*)dA, lda, (T*)d_alpha, d_jpvt);
}

// b[jpvt[i]] = z[i] for i < rank, 0 for rank <= i < n, on every right-hand side; jpvt entries outside [0, n) are skipped
template <typename T>
static int qrcp_scatter(dhqr_context* c, cudaStream_t st, int64_t n, int64_t rank, const T* z, int64_t ldz, const int64_t* d_jpvt,
                        T* d_b, int64_t ldb, int nrhs) {
    for (int r0 = 0; r0 < nrhs; r0 += 65535) {
        const int nr = std::min(nrhs - r0, 65535);
        TRY(launch(c, st, kname<T>("k_qrcp_scatter", "k_qrcp_scatter_c"), 0.0, [&](CwtSlot) {
            k_qrcp_scatter<T><<<dim3((unsigned)((n + 255) / 256), (unsigned)nr), 256, 0, st>>>(z + (size_t)r0 * ldz, ldz, d_jpvt, n, rank,
                                                                                            d_b + (size_t)r0 * ldb, ldb);
        }));
    }
    return 0;
}

template <typename T>
static int qrcp_solve(dhqr_context* c, int64_t m, int64_t n, int64_t rank, const void* dA, int64_t lda, const void* d_alpha,
                      const int64_t* d_jpvt, void* d_b, int64_t ldb, int nrhs, void* stream) {
    Check a(c, "the pivoted solve");
    a.require(m >= 0, 2, "m < 0");
    a.require(n >= 0 && n <= m, 3, "need 0 <= n <= m");
    a.require(rank >= 0 && rank <= n, 4, "need 0 <= rank <= n");
    a.operand<T>(5, "A", dA, mat(m, n, lda), when(n > 0, NEED) | ALIGN);
    a.operand<T>(7, "alpha", d_alpha, vec(n), when(n > 0, NEED) | ALIGN);
    a.operand<int64_t>(8, "jpvt", d_jpvt, vec(n), when(n > 0, NEED) | ALIGN);
    a.operand<T>(9, "b", d_b, mat(m, nrhs, ldb), when(nrhs > 0, NEED) | ALIGN);
    a.require(nrhs >= 0, 11, "nrhs < 0");
    TRY(a);
    if (n == 0 || nrhs == 0) return 0;
    CU(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    constexpr int w = sizeof(T) / sizeof(double);
    TRY(ensure_workspace(c, st, w * m, std::max<int64_t>(n, nrhs)));
    TRY(c->xbuf.ensure((size_t)w * n * nrhs, st));
    const T* A = (const T*)dA;
    T* b = (T*)d_b;
    T* z = (T*)c->xbuf.p;
    if (rank > 0) {
        TRY(apply_q_local(c, st, m, rank, A, lda, b, ldb, nrhs, 0));                 // (Q^H b)[0:rank]
        TRY(backsolve_single(c, st, rank, A, lda, (const T*)d_alpha, b, ldb, nrhs, z));   // z = R11^{-1} b[0:rank]
    }
    return qrcp_scatter(c, st, n, rank, z, rank, d_jpvt, b, ldb, nrhs);
}

}  // extern "C++"

int dhqr_qrcp_f64(dhqr_handle c, int64_t m, int64_t n, double* dA, int64_t lda, double* d_alpha, int64_t* d_jpvt, void* stream) {
    return qrcp_factor<double>(c, m, n, dA, lda, d_alpha, d_jpvt, stream);
}

int dhqr_qrcp_c64(dhqr_handle c, int64_t m, int64_t n, void* dA, int64_t lda, void* d_alpha, int64_t* d_jpvt, void* stream) {
    return qrcp_factor<double2>(c, m, n, dA, lda, d_alpha, d_jpvt, stream);
}

int dhqr_solve_qrcp_f64(dhqr_handle c, int64_t m, int64_t n, int64_t rank, const double* dA, int64_t lda, const double* d_alpha,
                        const int64_t* d_jpvt, double* d_b, int64_t ldb, int nrhs, void* stream) {
    return qrcp_solve<double>(c, m, n, rank, dA, lda, d_alpha, d_jpvt, d_b, ldb, nrhs, stream);
}

int dhqr_solve_qrcp_c64(dhqr_handle c, int64_t m, int64_t n, int64_t rank, const void* dA, int64_t lda, const void* d_alpha,
                        const int64_t* d_jpvt, void* d_b, int64_t ldb, int nrhs, void* stream) {
    return qrcp_solve<double2>(c, m, n, rank, dA, lda, d_alpha, d_jpvt, d_b, ldb, nrhs, stream);
}

// ---- complete orthogonal decomposition on the pivoted QR (DESIGN §2.8, §2.9) ------------------------------------------------
// A P = Q R at rank r: R_r = R[0:r, 0:n] (r x n, upper trapezoidal), and its adjoint factored by the unpivoted QR, R_r^H = Z [U; 0],
// gives A P ~ Q1 [U^H 0] Z^H.  The minimum-norm solution of the rank-r problem is x = P Z [U^{-H} (Q^H b)[0:r]; 0], and the step
// after Q^H b is exactly the minimum-norm solution of R_r y = c that dhqr_solve_adj_* computes from the factorisation (F, gamma) of
// R_r^H.
extern "C++" {   // as for the pivoted QR above

// (F, gamma) <- the unpivoted factorisation of R_r^H (n x rank) in place
static int qr_rrh(dhqr_context* c, cudaStream_t st, int64_t n, int64_t rank, double* F, int64_t ldf, double* gamma) {
    return qr_blocked(c, st, n, rank, 0, rank, F, ldf, gamma, c->nb);     // what dhqr_qr_f64 runs for nb = 0
}

static int qr_rrh(dhqr_context* c, cudaStream_t st, int64_t n, int64_t rank, double2* F, int64_t ldf, double2* gamma) {
    return qr_c64_local(c, st, n, rank, F, ldf, gamma);                  // the body of dhqr_qr_c64
}

template <typename T>
static int cod_factor(dhqr_context* c, int64_t m, int64_t n, int64_t rank, const void* dA, int64_t lda, const void* d_alpha, void* dF,
                      int64_t ldf, void* d_gamma, void* stream) {
    Check a(c, "the complete orthogonal decomposition");
    a.require(m >= 0, 2, "m < 0");
    a.require(n >= 0 && n <= m, 3, "need 0 <= n <= m");
    TRY(a);
    if (std::is_same<T, double>::value)   // R_r' has n rows and goes through the unpivoted path; the ComplexF64 one has no row limit
        a.require(n <= narrow_panel_max_rows(c), 3, "n = %lld exceeds the row limit of the unpivoted factorisation (%lld)", (long long)n,
                  (long long)narrow_panel_max_rows(c));
    a.require(rank >= 0 && rank <= n, 4, "need 0 <= rank <= n");
    a.operand<T>(5, "A", dA, mat(m, n, lda), when(n > 0, NEED) | ALIGN);
    a.operand<T>(7, "alpha", d_alpha, vec(n), when(n > 0, NEED) | ALIGN);
    a.operand<T>(8, "F", dF, mat(n, rank, ldf), when(rank > 0, NEED) | ALIGN | DISJOINT);     // F and gamma are written
    a.operand<T>(10, "gamma", d_gamma, vec(rank), when(rank > 0, NEED) | ALIGN | DISJOINT);
    TRY(a);
    if (n == 0 || rank == 0) return 0;
    CU(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    TRY(launch(c, st, kname<T>("k_cod_pack", "k_cod_pack_c"), (double)sizeof(T) * (double)n * rank, [&](CwtSlot) {
        k_cod_pack<T><<<dim3((unsigned)((n + CP_TILE - 1) / CP_TILE), (unsigned)((rank + CP_TILE - 1) / CP_TILE)), dim3(CP_TILE, CP_ROWS), 0,
                        st>>>((const T*)dA, lda, (const T*)d_alpha, n, rank, (T*)dF, ldf);
    }));
    return qr_rrh(c, st, n, rank, (T*)dF, ldf, (T*)d_gamma);
}

template <typename T>
static int cod_solve(dhqr_context* c, int64_t m, int64_t n, int64_t rank, const void* dA, int64_t lda, const int64_t* d_jpvt,
                     const void* dF, int64_t ldf, const void* d_gamma, void* d_b, int64_t ldb, int nrhs, void* stream) {
    Check a(c, "the complete orthogonal decomposition");
    a.require(m >= 0, 2, "m < 0");
    a.require(n >= 0 && n <= m, 3, "need 0 <= n <= m");
    a.require(rank >= 0 && rank <= n, 4, "need 0 <= rank <= n");
    a.operand<T>(5, "A", dA, mat(m, n, lda), when(n > 0, NEED) | ALIGN);
    a.operand<int64_t>(7, "jpvt", d_jpvt, vec(n), when(n > 0, NEED) | ALIGN);
    a.operand<T>(8, "F", dF, mat(n, rank, ldf), when(rank > 0, NEED) | ALIGN);
    a.operand<T>(10, "gamma", d_gamma, vec(rank), when(rank > 0, NEED) | ALIGN);
    a.operand<T>(11, "b", d_b, mat(m, nrhs, ldb), when(nrhs > 0, NEED) | ALIGN);
    a.require(nrhs >= 0, 13, "nrhs < 0");
    TRY(a);
    if (n == 0 || nrhs == 0) return 0;
    CU(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    constexpr int w = sizeof(T) / sizeof(double);
    TRY(ensure_workspace(c, st, w * m, std::max<int64_t>(n, nrhs)));
    TRY(c->xbuf.ensure((size_t)w * n * nrhs, st));
    T* b = (T*)d_b;
    T* z = (T*)c->xbuf.p;
    if (rank > 0) {
        TRY(apply_q_local(c, st, m, rank, (const T*)dA, lda, b, ldb, nrhs, 0));
        // b[0:n] <- Z [U^{-H} b[0:rank]; 0] from the factorisation (F, gamma) of R_r^H, rows n..m-1 of b untouched; then into xbuf,
        // which the scatter reads while it writes b
        TRY(solve_adj_local(c, st, n, rank, (const T*)dF, ldf, (const T*)d_gamma, b, ldb, nrhs));
        CU(cudaMemcpy2DAsync(z, (size_t)n * sizeof(T), b, (size_t)ldb * sizeof(T), (size_t)n * sizeof(T), nrhs, cudaMemcpyDeviceToDevice, st));
    }
    return qrcp_scatter(c, st, n, rank > 0 ? n : 0, z, n, d_jpvt, b, ldb, nrhs);
}

}  // extern "C++"

int dhqr_cod_f64(dhqr_handle c, int64_t m, int64_t n, int64_t rank, const double* dA, int64_t lda, const double* d_alpha, double* dF,
                 int64_t ldf, double* d_gamma, void* stream) {
    return cod_factor<double>(c, m, n, rank, dA, lda, d_alpha, dF, ldf, d_gamma, stream);
}

int dhqr_cod_c64(dhqr_handle c, int64_t m, int64_t n, int64_t rank, const void* dA, int64_t lda, const void* d_alpha, void* dF,
                 int64_t ldf, void* d_gamma, void* stream) {
    return cod_factor<double2>(c, m, n, rank, dA, lda, d_alpha, dF, ldf, d_gamma, stream);
}

int dhqr_solve_cod_f64(dhqr_handle c, int64_t m, int64_t n, int64_t rank, const double* dA, int64_t lda, const int64_t* d_jpvt,
                       const double* dF, int64_t ldf, const double* d_gamma, double* d_b, int64_t ldb, int nrhs, void* stream) {
    return cod_solve<double>(c, m, n, rank, dA, lda, d_jpvt, dF, ldf, d_gamma, d_b, ldb, nrhs, stream);
}

int dhqr_solve_cod_c64(dhqr_handle c, int64_t m, int64_t n, int64_t rank, const void* dA, int64_t lda, const int64_t* d_jpvt,
                       const void* dF, int64_t ldf, const void* d_gamma, void* d_b, int64_t ldb, int nrhs, void* stream) {
    return cod_solve<double2>(c, m, n, rank, dA, lda, d_jpvt, dF, ldf, d_gamma, d_b, ldb, nrhs, stream);
}

// ---- triangular-pentagonal QR: fold new rows into a factorisation (LAPACK dtpqrt / dtpmqrt), DESIGN §2.10, or delete rows (§2.11) -
// One block reflector of the structured update, on the stacked operand [X; C]: X = the block's kb rows of R (or of c), C = k rows of B
// (or of e).  V~ = [diag(vtop); V2] with V2 = packed columns [voff, voff + nbp) of vpk.  The existing sequence of
// apply_block_reflector on C with V = V2, plus the vtop rows in two places: diag(vtop) X as one more split-K partial of W (so the
// fixed-order reduction adds it), and X += diag(vtop) Y after Y is formed.  T comes from V2'V2 unchanged: off the diagonal it equals
// V~'V~, and T' is built from the strict triangle alone.  trans = 1: Q~ instead of Q~'.
// hyp (the downdate, §2.11): Theta = I - V~ T' V~'J with T^{-1} = I - striu(V2'V2); the W partial is -diag(vtop) X, so the reduced
// W is -(V~'J [X; C]), and Y = +T'W.  The launches are the append's, one for one.
static int tp_block_update(dhqr_context* c, cudaStream_t st, const double* vpk, int voff, int nbp, int kb, const double* vtop, int64_t k,
                           double* C, int64_t ldc, double* X, int64_t ldx, int ncols, int trans, bool hyp) {
    if (ncols <= 0 || k <= 0) return 0;
    auto& w = c->ws[0];
    const bool small = (nbp <= 32);
    const int NBPK = small ? 32 : 128;
    const int next = NBPK + ncols;
    if ((size_t)next * NBPK > w.wsum.n) return set_err(4003, "internal: W workspace too small");
    int nsplit = 0;
    int64_t pstride = 0;
    TRY(launch_vta_partials(c, st, vpk, w, voff, nbp, NBPK, C, ldc, k, ncols, small ? "k_gemm_vta32" : "k_gemm_vta128", &nsplit,
                            &pstride, 1));
    const int64_t nelem = (int64_t)next * NBPK;
    TRY(launch(c, st, "k_tp_wpart", 8.0 * (double)kb * ncols, [&](CwtSlot) {
        double* const wp = w.wpart.p + (size_t)nsplit * pstride;
        if (hyp) k_tp_wpart<true><<<wreduce_grid(c, nelem), 256, 0, st>>>(wp, NBPK, NBPK, ncols, vtop, kb, X, ldx);
        else k_tp_wpart<false><<<wreduce_grid(c, nelem), 256, 0, st>>>(wp, NBPK, NBPK, ncols, vtop, kb, X, ldx);
    }));
    ++nsplit;
    const int ygrid = (ncols + YCOLS - 1) / YCOLS;
    if (small) {
        TRY(launch(c, st, "k_mid32", 0.0, [&](CwtSlot) {
            if (hyp) k_mid32<true><<<ygrid, 512, 0, st>>>(w.wpart, pstride, nsplit, ncols, w.ypk, w.linv, trans);
            else k_mid32<false><<<ygrid, 512, 0, st>>>(w.wpart, pstride, nsplit, ncols, w.ypk, w.linv, trans);
        }));
    } else {
        TRY(launch(c, st, "k_wreduce", 0.0, [&](CwtSlot cwt) {
            k_wreduce<<<wreduce_grid(c, nelem), 256, 0, st>>>(w.wpart, pstride, nsplit, nelem, w.wsum, cwt);
        }));
        TRY(launch(c, st, "k_tinv128", 0.0, [&](CwtSlot cwt) {
            if (hyp) k_tinv<128, true><<<1, 512, smem_tinv(128), st>>>(w.wsum, w.linv, 0, cwt);
            else k_tinv<128, false><<<1, 512, smem_tinv(128), st>>>(w.wsum, w.linv, 0, cwt);
        }));
        TRY(launch(c, st, "k_ymake128", 0.0, [&](CwtSlot cwt) {
            if (hyp) k_ymake<128, true><<<ygrid, 256, smem_ymake(128), st>>>(w.wsum, NBPK, ncols, w.linv, w.ypk, trans, cwt);
            else k_ymake<128, false><<<ygrid, 256, smem_ymake(128), st>>>(w.wsum, NBPK, ncols, w.linv, w.ypk, trans, cwt);
        }));
    }
    TRY(launch_cvy(c, st, vpk, voff, nbp, w.ypk, k, 0, C, ldc, ncols, 0));
    const int64_t nx = (int64_t)kb * ncols;
    return launch(c, st, "k_tp_rows", 16.0 * (double)nx, [&](CwtSlot) {
        k_tp_rows<<<(unsigned)std::min<int64_t>((nx + 255) / 256, 8 * c->sms), 256, 0, st>>>(X, ldx, ncols, vtop, kb, w.ypk, NBPK / KC);
    });
}

// Workspace of both structured calls: the usual sets for k rows and `cols` W columns, and room for the extra W partial.
static int tp_workspace(dhqr_context* c, cudaStream_t st, int64_t k, int64_t cols) {
    TRY(ensure_workspace(c, st, k, cols));
    const int64_t tiles = (NBMAX + cols + G1_BN - 1) / G1_BN;
    return c->ws[0].wpart.ensure((size_t)std::max<int64_t>(2 * tiles, WPART_TILES) * NBMAX * G1_BN, st);
}

static int launch_tp_panel(dhqr_context* c, cudaStream_t st, double* B, int64_t ldb, int64_t k, double* R, int64_t ldr, double* alpha,
                           double* vtop, int ncols, int voff, int64_t vrows, int64_t* info, int64_t col0) {
    const int gmax = std::min(c->sms, PANEL_MAXG);
    const int64_t rpc = rup(std::max<int64_t>((k + gmax - 1) / gmax, 64), 8);
    const int G = (int)((k + rpc - 1) / rpc);
    const int lds = (int)rpc + 4;
    const size_t smem = (size_t)IB * lds * 8;
    if (smem > 184 * 1024) return set_err(-3, "k too large for the resident panel kernel (%lld rows per CTA)", (long long)rpc);
    TRY(ll_epoch_check(c, st));
    TpPanelArgs a;
    a.B = B; a.ldb = ldb; a.k = k; a.R = R; a.ldr = ldr; a.alpha = alpha; a.vtop = vtop; a.ncols = ncols;
    a.vpk = c->vpk2[0]; a.voff = voff; a.vrows = vrows; a.rows_per_cta = (int)rpc; a.lds = lds;
    a.cells = c->cells; a.epoch = c->ll_epoch; a.info = info; a.col0 = col0;
    void* args[] = {&a};
    void* const kern = info ? (void*)k_tp_panel<true> : (void*)k_tp_panel<false>;
    return launch(c, st, "k_tp_panel", 16.0 * (double)k * ncols, [&](CwtSlot) {   // work = bytes: the B panel read once + written once
        const cudaError_t e = cudaLaunchCooperativeKernel(kern, dim3(G), dim3(PANEL_THREADS), args, smem, st);
        if (e == cudaSuccess) c->ll_epoch += IB + 8;
        return e;
    });
}

// Outer panels of 128 columns, each four 32-column k_tp_panel launches with the 32-wide update of the rest of the outer panel after
// each, then the 128-wide update of the trailing columns.  Row i of R changes only under reflector i, so each launch reads R as the
// caller passed it.  info != nullptr: the downdate (hyperbolic reflectors, §2.11), which first zero-fills *info in stream order.
static int qr_append_local(dhqr_context* c, cudaStream_t st, int64_t n, int64_t k, double* R, int64_t ldr, double* alpha, double* B,
                           int64_t ldb, double* vtop, int64_t* info) {
    TRY(tp_workspace(c, st, k, n));
    const bool hyp = info != nullptr;
    if (hyp) CU(cudaMemsetAsync(info, 0, sizeof(int64_t), st));
    const int64_t vrows = rup(k, 128);
    for (int64_t k0 = 0; k0 < n; k0 += NBMAX) {
        const int kb = (int)std::min<int64_t>(NBMAX, n - k0);
        for (int o = 0; o < kb; o += IB) {
            const int ib = std::min(IB, kb - o);
            const int64_t cs = k0 + o;
            TRY(launch_tp_panel(c, st, B + cs * ldb, ldb, k, R + cs * ldr + cs, ldr, alpha + cs, vtop + cs, ib, o, vrows, info, cs));
            const int rem = kb - o - ib;
            if (rem > 0)
                TRY(tp_block_update(c, st, c->vpk2[0], o, IB, ib, vtop + cs, k, B + (cs + ib) * ldb, ldb, R + (cs + ib) * ldr + cs, ldr,
                                    rem, 0, hyp));
        }
        const int64_t trail = n - k0 - kb;
        if (trail > 0)
            TRY(tp_block_update(c, st, c->vpk2[0], 0, NBMAX, kb, vtop + k0, k, B + (k0 + kb) * ldb, ldb, R + (k0 + kb) * ldr + k0, ldr,
                                (int)trail, 0, hyp));
    }
    return 0;
}

// [c; e] <- Q~' [c; e] (blocks first to last) or Q~ [c; e] (trans = 1, last to first); V2 packed from B, T recomputed from V2.
// hyp: [c; e] <- Theta [c; e] of the downdate (trans = 0).
static int apply_append_local(dhqr_context* c, cudaStream_t st, int64_t n, int64_t k, const double* B, int64_t ldb, const double* vtop,
                              double* dc, int64_t ldc, double* de, int64_t lde, int nrhs, int trans, bool hyp) {
    TRY(tp_workspace(c, st, k, std::max<int64_t>(n, nrhs)));
    const int64_t vrows = rup(k, 128);
    const int64_t ofirst = trans ? ((n - 1) / NBMAX) * NBMAX : 0, ostep = trans ? -(int64_t)NBMAX : NBMAX;
    for (int64_t o = ofirst; o >= 0 && o < n; o += ostep) {
        const int kb = (int)std::min<int64_t>(NBMAX, n - o);
        const int nbp = kb <= IB ? IB : NBMAX;
        TRY(pack_v(c, st, B + o * ldb, ldb, k, kb, 0, c->vpk2[0], 0, vrows, nbp));
        TRY(tp_block_update(c, st, c->vpk2[0], 0, nbp, kb, vtop + o, k, de, lde, dc + o, ldc, nrhs, trans, hyp));
    }
    return 0;
}

// k is capped by the panel kernel's slab capacity
static const char* const TP_ROWS = "k = %lld exceeds the rows one %s can take on this device (%lld): split the block";

// dhqr_qr_append_f64 (d_info == nullptr, the rows are B) and dhqr_qr_downdate_f64 (the rows are Z): the same checks and driver
static int qr_tp(dhqr_context* c, int64_t n, int64_t k, double* dR, int64_t ldr, double* d_alpha, double* dB, int64_t ldb, double* d_vtop,
                 int64_t* d_info, bool hyp, void* stream) {
    const bool work = n > 0 && k > 0;
    Check a(c, hyp ? "deleting rows" : "appending rows");
    a.require(n >= 0, 2, "n < 0");
    a.require(k >= 0, 3, "k < 0");
    TRY(a);
    a.require(k <= narrow_panel_max_rows(c), 3, TP_ROWS, (long long)k, hyp ? "downdate" : "append", (long long)narrow_panel_max_rows(c));
    a.operand<double>(4, "R", dR, mat(n, n, ldr), when(n > 0, NEED) | ALIGN);
    a.operand<double>(6, "alpha", d_alpha, vec(n), when(n > 0, NEED) | ALIGN);
    a.operand<double>(7, hyp ? "Z" : "B", dB, mat(k, n, ldb), when(work, NEED) | ALIGN | DISJOINT);
    a.operand<double>(9, "vtop", d_vtop, vec(n), when(n > 0, NEED) | ALIGN | when(k > 0, DISJOINT));
    if (hyp) a.operand<int64_t>(10, "info", d_info, vec(1), when(work, NEED | DISJOINT) | ALIGN);
    TRY(a);
    if (!work) return 0;
    CU(cudaSetDevice(c->device));
    return qr_append_local(c, (cudaStream_t)stream, n, k, dR, ldr, d_alpha, dB, ldb, d_vtop, hyp ? d_info : nullptr);
}

int dhqr_qr_append_f64(dhqr_handle c, int64_t n, int64_t k, double* dR, int64_t ldr, double* d_alpha, double* dB, int64_t ldb,
                       double* d_vtop, void* stream) {
    return qr_tp(c, n, k, dR, ldr, d_alpha, dB, ldb, d_vtop, nullptr, false, stream);
}

int dhqr_qr_downdate_f64(dhqr_handle c, int64_t n, int64_t k, double* dR, int64_t ldr, double* d_alpha, double* dZ, int64_t ldz,
                         double* d_vtop, int64_t* d_info, void* stream) {
    return qr_tp(c, n, k, dR, ldr, d_alpha, dZ, ldz, d_vtop, d_info, true, stream);
}

// the three applies: Q~' (trans = 0), Q~ (trans = 1) of the append, Theta of the downdate (hyp, trans = 0); the rows are B or Z
static int apply_append(dhqr_context* c, int64_t n, int64_t k, const double* dB, int64_t ldb, const double* d_vtop, double* d_c,
                        int64_t ldc, double* d_e, int64_t lde, int nrhs, void* stream, int trans, bool hyp = false) {
    Check a(c, hyp ? "deleting rows" : "appending rows");
    a.require(n >= 0, 2, "n < 0");
    a.require(k >= 0, 3, "k < 0");
    TRY(a);
    a.require(k <= narrow_panel_max_rows(c), 3, TP_ROWS, (long long)k, hyp ? "downdate" : "append", (long long)narrow_panel_max_rows(c));
    a.operand<double>(4, hyp ? "Z" : "B", dB, mat(k, n, ldb), when(n > 0 && k > 0, NEED) | ALIGN);
    a.operand<double>(6, "vtop", d_vtop, vec(n), when(n > 0, NEED) | ALIGN);
    a.operand<double>(7, "c", d_c, mat(n, nrhs, ldc), when(n > 0 && nrhs > 0, NEED) | ALIGN | DISJOINT);
    a.operand<double>(9, "e", d_e, mat(k, nrhs, lde), when(k > 0 && nrhs > 0, NEED) | ALIGN | DISJOINT);
    a.require(nrhs >= 0, 11, "nrhs < 0");
    TRY(a);
    if (n == 0 || k == 0 || nrhs == 0) return 0;
    CU(cudaSetDevice(c->device));
    return apply_append_local(c, (cudaStream_t)stream, n, k, dB, ldb, d_vtop, d_c, ldc, d_e, lde, nrhs, trans, hyp);
}

int dhqr_apply_qt_append_f64(dhqr_handle c, int64_t n, int64_t k, const double* dB, int64_t ldb, const double* d_vtop, double* d_c,
                             int64_t ldc, double* d_e, int64_t lde, int nrhs, void* stream) {
    return apply_append(c, n, k, dB, ldb, d_vtop, d_c, ldc, d_e, lde, nrhs, stream, 0);
}

int dhqr_apply_q_append_f64(dhqr_handle c, int64_t n, int64_t k, const double* dB, int64_t ldb, const double* d_vtop, double* d_c,
                            int64_t ldc, double* d_e, int64_t lde, int nrhs, void* stream) {
    return apply_append(c, n, k, dB, ldb, d_vtop, d_c, ldc, d_e, lde, nrhs, stream, 1);
}

int dhqr_apply_downdate_f64(dhqr_handle c, int64_t n, int64_t k, const double* dZ, int64_t ldz, const double* d_vtop, double* d_c,
                            int64_t ldc, double* d_e, int64_t lde, int nrhs, void* stream) {
    return apply_append(c, n, k, dZ, ldz, d_vtop, d_c, ldc, d_e, lde, nrhs, stream, 0, true);
}

// ---- batched QR of many small problems (DESIGN §2.12) -----------------------------------------------------------------------
extern "C++" {   // as for the pivoted QR above
template <typename Kernel, typename... Args>
static int launch_batched(dhqr_context* c, cudaStream_t st, const char* what, double work, Kernel kern, const BatchedGeom& g,
                          int64_t batch, int ny, size_t smem, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(batch * g.cs), (unsigned)ny);
    cfg.blockDim = dim3(g.threads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = (unsigned)g.cs;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    return launch(c, st, what, work, [&](CwtSlot) { return cudaLaunchKernelEx(&cfg, kern, args...); });
}
}   // extern "C++"

int dhqr_qr_batched_f64(dhqr_handle c, int64_t m, int64_t n, int64_t batch, double* dA, int64_t lda, int64_t stride_a,
                        double* d_alpha, int64_t stride_alpha, void* stream) {
    Check a(c, "the batched QR");
    a.require(m >= 0, 2, "m < 0");
    a.require(n >= 0 && n <= m, 3, "need 0 <= n <= m");
    a.require(n == 0 || m <= BQ_MAX_ELEMS / n, 3, "m * n exceeds batch_max_elems (%lld): factor a problem this large with dhqr_qr_f64",
              (long long)BQ_MAX_ELEMS);
    a.require(batch >= 0, 4, "batch < 0");
    TRY(a);
    a.require(batch * batched_geom(m, n).cs <= INT32_MAX, 4, "batch too large for one grid (batch x CTAs per problem > 2^31 - 1)");
    a.operand<double>(5, "A", dA, mat(m, n, lda, batch, stride_a), when(batch > 0 && n > 0, NEED) | ALIGN);
    a.operand<double>(8, "alpha", d_alpha, vec(n, batch, stride_alpha), when(batch > 0 && n > 0, NEED) | ALIGN | DISJOINT);
    TRY(a);
    if (batch == 0 || n == 0) return 0;
    CU(cudaSetDevice(c->device));
    const BatchedGeom g = batched_geom(m, n);
    const double flops = (double)batch * (2.0 * m * n * n - 2.0 * n * n * n / 3.0);
    return launch_batched(c, (cudaStream_t)stream, "k_qr_batched", flops, k_qr_batched, g, batch, 1, smem_qr_batched(g, n), dA, lda,
                          stride_a, d_alpha, stride_alpha, (int)m, (int)n, g.rpc);
}

// dhqr_apply_qt_batched_f64 (trans), dhqr_apply_q_batched_f64 and dhqr_solve_batched_f64 (solve: alpha is arguments 8-9, and
// every later argument index moves up by 2)
static int apply_batched(dhqr_context* c, int64_t m, int64_t n, int64_t batch, const double* dA, int64_t lda, int64_t stride_a,
                         const double* d_alpha, int64_t stride_alpha, double* d_b, int64_t ldb, int64_t stride_b, int nrhs, void* stream,
                         bool trans, bool solve) {
    Check a(c, "the batched QR");
    a.require(m >= 0, 2, "m < 0");
    a.require(n >= 0 && n <= m, 3, "need 0 <= n <= m");
    a.require(n == 0 || m <= BQ_MAX_ELEMS / n, 3, "m * n exceeds batch_max_elems (%lld): factor a problem this large with dhqr_qr_f64",
              (long long)BQ_MAX_ELEMS);
    a.require(batch >= 0, 4, "batch < 0");
    TRY(a);
    a.require(batch * batched_geom(m, n).cs <= INT32_MAX, 4, "batch too large for one grid (batch x CTAs per problem > 2^31 - 1)");
    a.operand<double>(5, "A", dA, mat(m, n, lda, batch, stride_a), when(batch > 0 && n > 0, NEED) | ALIGN);
    const int o = solve ? 2 : 0;
    if (solve) a.operand<double>(8, "alpha", d_alpha, vec(n, batch, stride_alpha), when(batch > 0 && n > 0, NEED) | ALIGN | DISJOINT);
    a.operand<double>(8 + o, "b", d_b, mat(m, nrhs, ldb, batch, stride_b), when(batch > 0 && n > 0 && nrhs > 0, NEED) | ALIGN | DISJOINT);
    a.require(nrhs >= 0, 11 + o, "nrhs < 0");
    TRY(a);
    if (batch == 0 || n == 0 || nrhs == 0) return 0;
    CU(cudaSetDevice(c->device));
    const BatchedGeom g = batched_geom(m, n);
    const int kc = batched_kc(g, n, nrhs);
    const int ny = (int)std::min<int64_t>((nrhs + kc - 1) / kc, 65535);
    const size_t smem = smem_apply_batched(g, n, kc, solve);
    const double flops = (double)batch * nrhs * (4.0 * m * n - 2.0 * n * n + (solve ? (double)n * n : 0.0));
    cudaStream_t st = (cudaStream_t)stream;
    if (solve)
        return launch_batched(c, st, "k_solve_batched", flops, k_apply_batched<true, true>, g, batch, ny, smem, dA, lda, stride_a, d_alpha,
                              stride_alpha, d_b, ldb, stride_b, (int)m, (int)n, nrhs, g.rpc, kc);
    return launch_batched(c, st, trans ? "k_apply_qt_batched" : "k_apply_q_batched", flops,
                          trans ? k_apply_batched<true, false> : k_apply_batched<false, false>, g, batch, ny, smem, dA, lda, stride_a,
                          (const double*)nullptr, (int64_t)0, d_b, ldb, stride_b, (int)m, (int)n, nrhs, g.rpc, kc);
}

int dhqr_apply_qt_batched_f64(dhqr_handle c, int64_t m, int64_t n, int64_t batch, const double* dA, int64_t lda, int64_t stride_a,
                              double* d_b, int64_t ldb, int64_t stride_b, int nrhs, void* stream) {
    return apply_batched(c, m, n, batch, dA, lda, stride_a, nullptr, 0, d_b, ldb, stride_b, nrhs, stream, true, false);
}

int dhqr_apply_q_batched_f64(dhqr_handle c, int64_t m, int64_t n, int64_t batch, const double* dA, int64_t lda, int64_t stride_a,
                             double* d_b, int64_t ldb, int64_t stride_b, int nrhs, void* stream) {
    return apply_batched(c, m, n, batch, dA, lda, stride_a, nullptr, 0, d_b, ldb, stride_b, nrhs, stream, false, false);
}

int dhqr_solve_batched_f64(dhqr_handle c, int64_t m, int64_t n, int64_t batch, const double* dA, int64_t lda, int64_t stride_a,
                           const double* d_alpha, int64_t stride_alpha, double* d_b, int64_t ldb, int64_t stride_b, int nrhs,
                           void* stream) {
    return apply_batched(c, m, n, batch, dA, lda, stride_a, d_alpha, stride_alpha, d_b, ldb, stride_b, nrhs, stream, true, true);
}

// ---- batched append and downdate, batched back-substitution (DESIGN §2.13) ----------------------------------------------------
// dhqr_qr_append_batched_f64 (hyp = false, the rows are B) and dhqr_qr_downdate_batched_f64 (the rows are Z, d_info is argument 22)
static int tp_batched(dhqr_context* c, int64_t n, int64_t k, int64_t batch, double* dR, int64_t ldr, int64_t stride_r, double* d_alpha,
                      int64_t stride_alpha, double* dB, int64_t ldb, int64_t stride_b, double* d_vtop, int64_t stride_vtop, double* d_c,
                      int64_t ldc, int64_t stride_c, double* d_e, int64_t lde, int64_t stride_e, int nrhs, int64_t* d_info, bool hyp,
                      void* stream) {
    const int64_t ncol = n + std::max(nrhs, 0);
    const bool work = batch > 0 && n > 0 && k > 0, rhs = work && nrhs > 0;
    Check a(c, hyp ? "the batched downdate" : "the batched append");
    a.require(n >= 0, 2, "n < 0");
    a.require(k >= 0, 3, "k < 0");
    a.require(ncol <= BQ_UPD_MAX_COLS, 3, "n + nrhs = %lld exceeds batch_update_max_cols (%d)", (long long)ncol, BQ_UPD_MAX_COLS);
    a.require(ncol == 0 || k <= BQ_MAX_ELEMS / ncol, 3, "k * (n + nrhs) exceeds batch_max_elems (%lld): split the block",
              (long long)BQ_MAX_ELEMS);
    a.require(batch >= 0, 4, "batch < 0");
    TRY(a);
    a.require(batch * batched_geom(k, ncol).cs <= INT32_MAX, 4, "batch too large for one grid (batch x CTAs per problem > 2^31 - 1)");
    a.operand<double>(5, "R", dR, mat(n, n, ldr, batch, stride_r), when(batch > 0 && n > 0, NEED) | ALIGN);
    a.operand<double>(8, "alpha", d_alpha, vec(n, batch, stride_alpha), when(batch > 0 && n > 0, NEED) | ALIGN | DISJOINT);
    a.operand<double>(10, hyp ? "Z" : "B", dB, mat(k, n, ldb, batch, stride_b), when(work, NEED) | ALIGN | DISJOINT);
    a.operand<double>(13, "vtop", d_vtop, vec(n, batch, stride_vtop), when(work, NEED | DISJOINT) | ALIGN);
    if (nrhs > 0) {
        a.operand<double>(15, "c", d_c, mat(n, nrhs, ldc, batch, stride_c), when(rhs, NEED | DISJOINT) | ALIGN);
        a.operand<double>(18, "e", d_e, mat(k, nrhs, lde, batch, stride_e), when(rhs, NEED | DISJOINT) | ALIGN);
    }
    a.require(nrhs >= 0, 21, "nrhs < 0");
    if (hyp) a.operand<int64_t>(22, "info", d_info, vec(batch), when(work, NEED | DISJOINT) | ALIGN);
    TRY(a);
    if (!work) return 0;
    CU(cudaSetDevice(c->device));
    const BatchedGeom g = batched_geom(k, ncol);
    const double flops = (double)batch * (4.0 * k + 6.0) * n * (ncol - (n + 1) / 2.0);
    return launch_batched(c, (cudaStream_t)stream, hyp ? "k_downdate_batched" : "k_append_batched", flops,
                          hyp ? k_tp_batched<true> : k_tp_batched<false>, g, batch, 1, smem_tp_batched(g, ncol), dR, ldr, stride_r,
                          d_alpha, stride_alpha, dB, ldb, stride_b, d_vtop, stride_vtop, rhs ? d_c : nullptr, ldc, stride_c,
                          rhs ? d_e : nullptr, lde, stride_e, hyp ? d_info : nullptr, (int)n, (int)k, nrhs, g.rpc);
}

int dhqr_qr_append_batched_f64(dhqr_handle c, int64_t n, int64_t k, int64_t batch, double* dR, int64_t ldr, int64_t stride_r,
                               double* d_alpha, int64_t stride_alpha, double* dB, int64_t ldb, int64_t stride_b, double* d_vtop,
                               int64_t stride_vtop, double* d_c, int64_t ldc, int64_t stride_c, double* d_e, int64_t lde, int64_t stride_e,
                               int nrhs, void* stream) {
    return tp_batched(c, n, k, batch, dR, ldr, stride_r, d_alpha, stride_alpha, dB, ldb, stride_b, d_vtop, stride_vtop, d_c, ldc, stride_c,
                      d_e, lde, stride_e, nrhs, nullptr, false, stream);
}

int dhqr_qr_downdate_batched_f64(dhqr_handle c, int64_t n, int64_t k, int64_t batch, double* dR, int64_t ldr, int64_t stride_r,
                                 double* d_alpha, int64_t stride_alpha, double* dZ, int64_t ldz, int64_t stride_z, double* d_vtop,
                                 int64_t stride_vtop, double* d_c, int64_t ldc, int64_t stride_c, double* d_e, int64_t lde,
                                 int64_t stride_e, int nrhs, int64_t* d_info, void* stream) {
    return tp_batched(c, n, k, batch, dR, ldr, stride_r, d_alpha, stride_alpha, dZ, ldz, stride_z, d_vtop, stride_vtop, d_c, ldc, stride_c,
                      d_e, lde, stride_e, nrhs, d_info, true, stream);
}

int dhqr_backsolve_batched_f64(dhqr_handle c, int64_t n, int64_t batch, const double* dR, int64_t ldr, int64_t stride_r,
                               const double* d_alpha, int64_t stride_alpha, double* d_b, int64_t ldb, int64_t stride_b, int nrhs,
                               void* stream) {
    Check a(c, "the batched back-substitution");
    a.require(n >= 0, 2, "n < 0");
    a.require(n <= BQ_UPD_MAX_COLS, 2, "n = %lld exceeds batch_update_max_cols (%d)", (long long)n, BQ_UPD_MAX_COLS);
    a.require(batch >= 0, 3, "batch < 0");
    a.require(batch <= INT32_MAX, 3, "batch too large for one grid (> 2^31 - 1)");
    a.operand<double>(4, "R", dR, mat(n, n, ldr, batch, stride_r), when(batch > 0 && n > 0, NEED) | ALIGN);
    a.operand<double>(7, "alpha", d_alpha, vec(n, batch, stride_alpha), when(batch > 0 && n > 0, NEED) | ALIGN);
    a.operand<double>(9, "b", d_b, mat(n, nrhs, ldb, batch, stride_b), when(batch > 0 && n > 0 && nrhs > 0, NEED) | ALIGN | DISJOINT);
    a.require(nrhs >= 0, 12, "nrhs < 0");
    TRY(a);
    if (batch == 0 || n == 0 || nrhs == 0) return 0;
    CU(cudaSetDevice(c->device));
    const int kc = (int)std::min<int64_t>({(int64_t)BQ_KC, BQ_SLAB / n, (int64_t)nrhs});
    const int ny = (int)std::min<int64_t>((nrhs + kc - 1) / kc, 65535);
    BatchedGeom g;
    g.cs = 1;
    g.rpc = (int)n;
    g.threads = 32 * (int)std::min<int64_t>(std::max<int64_t>((n + 31) / 32, 1), 8);
    return launch_batched(c, (cudaStream_t)stream, "k_backsolve_batched", (double)batch * nrhs * n * n, k_backsolve_batched, g, batch, ny,
                          (size_t)kc * n * 8, dR, ldr, stride_r, d_alpha, stride_alpha, d_b, ldb, stride_b, (int)n, nrhs, kc);
}

// ---- host-buffer entry points --------------------------------------------------------------------
// Plan of the chunked upload of dhqr_qr_host_f64: chunk boundaries B (multiples of nb; B[0] = 0, B.back() = n) and, for every
// chunk after the first, the step of the look-ahead schedule at which it joins the trailing matrix.  A chunk joins as soon as
// the model says it has arrived (earlier = less catch-up work), at the latest one step before the panel chain reaches into it.
// The model has two parameters (options host_h2d_gbs, host_tflops); a wrong guess costs idle time, never correctness: the
// driver orders every use of a chunk behind its upload event and forces a join that the plan names too late.
struct UploadModel { int chunk, first, h2d_gbs, tflops, chain_us; };
static void plan_upload(const UploadModel* c, int64_t m, int64_t n, int nb, std::vector<int64_t>& B, std::vector<int>& join) {
    B.assign(1, 0);
    join.assign(1, 0);
    // the schedule starts on panels 0..2: the first (exposed) upload is those three panels unless option host_first asks for more;
    // the second chunk ends where a first chunk of 1.5 chunks would have, so that the later boundaries do not move
    const int64_t chunk = rup(c->chunk, nb), second = std::max(rup(chunk + chunk / 2, nb), 3 * (int64_t)nb);
    const int64_t first = c->first > 0 ? std::min(std::max(rup(c->first, nb), 3 * (int64_t)nb), second) : 3 * (int64_t)nb;
    if (c->chunk <= 0 || m < n || n < second + chunk) { B.push_back(n); return; }
    B.push_back(first);
    if (second > first) B.push_back(second);
    while (B.back() < n) B.push_back(std::min(n, B.back() + chunk));
    if (n - B[B.size() - 2] < chunk / 2) B.erase(B.end() - 2);           // no sliver at the end
    const int nch = (int)B.size() - 1, K = (int)((n + nb - 1) / nb);
    const double U = 1e9 * c->h2d_gbs, R = 1e12 * c->tflops, chain = 1e-6 * c->chain_us;
    auto tup = [&](int j) { return (double)B[j + 1] * (double)m * 8.0 / U; };
    join.assign(nch, 0);
    double T = tup(0);
    int64_t wend = B[1];
    int nxt = 1;
    for (int k = 0; k < K; ++k) {
        while (nxt < nch && (B[nxt] < std::min<int64_t>(n, (int64_t)nb * (k + 4)) || tup(nxt) <= T)) {
            T = std::max(T, tup(nxt));                        // (the catch-up runs beside the schedule on its own stream)
            join[nxt] = k;
            wend = B[nxt + 1];
            ++nxt;
        }
        T += std::max(chain, 4.0 * (double)(m - (int64_t)nb * k) * nb * (double)std::max<int64_t>(0, wend - (int64_t)nb * (k + 1)) / R);
    }
}

int dhqr_plan_host_upload(int64_t m, int64_t n, int nb, int chunk, int first, int h2d_gbs, int tflops, int chain_us, int cap,
                          int64_t* bounds, int* join, int* nchunks) {
    if (m < 0) return set_err(-1, "m < 0");
    if (n < 0 || n > m) return set_err(-2, "need 0 <= n <= m");
    if (nb < 32 || nb > 128 || nb % 32) return set_err(-3, "nb must be a multiple of 32 in [32,128]");
    if (chunk < 0 || first < 0) return set_err(chunk < 0 ? -4 : -5, "negative width");
    if (h2d_gbs < 1 || tflops < 1 || chain_us < 1) return set_err(h2d_gbs < 1 ? -6 : (tflops < 1 ? -7 : -8), "model parameters must be positive");
    if (!bounds || !join || !nchunks) return set_err(!bounds ? -10 : (!join ? -11 : -12), "null output");
    const UploadModel um = {chunk, first, h2d_gbs, tflops, chain_us};
    std::vector<int64_t> B;
    std::vector<int> J;
    plan_upload(&um, m, n, nb, B, J);
    const int nch = (int)B.size() - 1;
    if (cap < nch + 1) return set_err(-9, "cap too small: %d chunks", nch);
    for (int j = 0; j <= nch; ++j) bounds[j] = B[j];
    for (int j = 0; j < nch; ++j) join[j] = J[j];
    *nchunks = nch;
    return 0;
}

int dhqr_qr_host_f64(dhqr_handle c, int64_t m, int64_t n, double* hA, int64_t lda, double* h_alpha, int nb) {
    Check a(c, "the host entry");   // hA, lda and h_alpha keep the codes of dA_local, lda and d_alpha of dhqr_qr_f64
    column_block(a, m, n, 0, n);
    a.operand<double>(6, "A", hA, mat(m, n, lda), when(n > 0, NEED));
    a.operand<double>(6, "alpha", h_alpha, vec(n), when(n > 0, NEED));
    a.require(nb == 0 || nb == 1 || (nb >= 32 && nb <= 128 && nb % 32 == 0), 9, "nb must be 0, 1 or a multiple of 32 in [32,128]");
    TRY(a);
    if (n == 0) return 0;
    CU(cudaSetDevice(c->device));
    const int64_t ldd = rup(m, 32);                       // padded device leading dimension (aligned TMA sources)
    const bool blocked = (nb != 1);
    const int nbe = nb == 0 ? c->nb : nb;
    // The matrix goes up in column chunks.  Only the first upload is exposed: the factorisation starts on it, every later chunk
    // travels while the device works and joins the trailing matrix through a catch-up (qr_blocked_lookahead); finished panels
    // stream back while later panels are factored.  One factorisation, the same reflectors as with the matrix resident.
    std::vector<int64_t> B;
    std::vector<int> join;
    const UploadModel um = {c->host_chunk, c->host_first, c->host_h2d_gbs, c->host_tflops, c->host_chain_us};
    if (blocked) plan_upload(&um, m, n, nbe, B, join);
    else { B = {0, n}; join = {0}; }
    const int nch = (int)B.size() - 1;
    cudaStream_t st = c->copy_stream;
    TRY(c->hostA.ensure((size_t)ldd * n + (size_t)n, st));
    // everything sized once, before the pipeline starts: growing a buffer later would synchronise the device
    TRY(ensure_workspace(c, st, m, n, blocked ? (n + nbe - 1) / nbe + 1 : 0, nch > 1));
    double* dA = c->hostA;
    double* dal = c->hostA + (size_t)ldd * n;
    std::vector<Event> evUp;
    struct timespec ts0;
    clock_gettime(CLOCK_MONOTONIC, &ts0);
    auto stamp = [&](const char* what, bool sync_all) {
        if (!c->host_trace) return;
        if (sync_all) { cudaStreamSynchronize(st); }
        struct timespec ts;
        clock_gettime(CLOCK_MONOTONIC, &ts);
        fprintf(stderr, "[dhqr host] %-34s %8.2f ms\n", what, (ts.tv_sec - ts0.tv_sec) * 1e3 + (ts.tv_nsec - ts0.tv_nsec) * 1e-6);
    };
    if (c->host_trace) {
        fprintf(stderr, "[dhqr host] upload chunks (first column : join step):");
        for (int j = 0; j < nch; ++j) fprintf(stderr, " %lld:%d", (long long)B[j], join[j]);
        fprintf(stderr, "\n");
    }
    c->up_chunks.clear();
    // The pipeline returns at its first failure, possibly with work still queued; the tail below runs after it either way.
    const int rc = [&]() -> int {
        if (cudaMemcpy2DAsync(dA, (size_t)ldd * 8, hA, (size_t)lda * 8, (size_t)m * 8, (size_t)B[1], cudaMemcpyHostToDevice, st) != cudaSuccess)
            return set_err(1001, "H2D failed");
        if (nch > 1) {
            // the later chunks go up one after the other BEHIND the first (concurrent uploads would share the link and delay the
            // start of the factorisation), on their own stream
            evUp.emplace_back();
            if (evUp.back().create(cudaEventDisableTiming) != cudaSuccess) return set_err(1001, "event create failed");
            cudaEventRecord(evUp.back(), st);
            cudaStreamWaitEvent(c->h2d_stream, evUp.back(), 0);
            for (int j = 1; j < nch; ++j) {
                evUp.emplace_back();
                if (evUp.back().create(c->host_trace ? cudaEventDefault : cudaEventDisableTiming) != cudaSuccess)
                    return set_err(1001, "event create failed");
                if (cudaMemcpy2DAsync(dA + B[j] * ldd, (size_t)ldd * 8, hA + B[j] * lda, (size_t)lda * 8, (size_t)m * 8, (size_t)(B[j + 1] - B[j]),
                                      cudaMemcpyHostToDevice, c->h2d_stream) != cudaSuccess)
                    return set_err(1001, "H2D failed");
                cudaEventRecord(evUp.back(), c->h2d_stream);
                c->up_chunks.push_back({B[j], B[j + 1], evUp.back(), join[j]});
            }
        }
        stamp("first chunk uploaded", true);
        if (blocked) { c->mirror_host = hA; c->mirror_lda = lda; }   // finished panels stream back while later panels are factored
        const int la_trace_keep = c->la_trace;
        if (c->host_trace) c->la_trace = 1;
        const int rq = dhqr_qr_f64(c, m, n, 0, n, dA, ldd, dal, nb, st);
        c->la_trace = la_trace_keep;
        c->mirror_host = nullptr;
        TRY(rq);
        stamp("factored", true);
        if (!blocked && cudaMemcpy2DAsync(hA, (size_t)lda * 8, dA, (size_t)ldd * 8, (size_t)m * 8, (size_t)n, cudaMemcpyDeviceToHost, st) != cudaSuccess)
            return set_err(1001, "D2H failed");
        if (cudaMemcpyAsync(h_alpha, dal, (size_t)n * 8, cudaMemcpyDeviceToHost, st) != cudaSuccess) return set_err(1001, "D2H failed");
        return 0;
    }();
    c->mirror_host = nullptr;
    c->up_chunks.clear();
    const cudaError_t e0 = cudaStreamSynchronize(c->h2d_stream), e1 = cudaStreamSynchronize(st), e2 = cudaStreamSynchronize(c->d2h_stream);
    cudaError_t e3 = cudaSuccess;
    for (int i = 0; i < 3; ++i) { const cudaError_t e4 = cudaStreamSynchronize(c->cu_stream[i]); if (e3 == cudaSuccess) e3 = e4; }
    stamp("everything back on the host", false);
    c->panel_events.clear();
    if (rc) return rc;
    if (e0 != cudaSuccess) return set_err(1000 + (int)e0, "qr_host H2D: %s", cudaGetErrorString(e0));
    if (e1 != cudaSuccess) return set_err(1000 + (int)e1, "qr_host: %s", cudaGetErrorString(e1));
    if (e2 != cudaSuccess) return set_err(1000 + (int)e2, "qr_host D2H: %s", cudaGetErrorString(e2));
    if (e3 != cudaSuccess) return set_err(1000 + (int)e3, "qr_host catch-up: %s", cudaGetErrorString(e3));
    return 0;
}

int dhqr_ldiv_host_f64(dhqr_handle c, int64_t m, int64_t n, const double* hA, int64_t lda, const double* h_alpha,
                       const double* h_b, double* h_x) {
    Check a(c, "the host entry");   // hA, lda and h_alpha keep the codes of dA_local, lda and d_alpha of dhqr_qr_f64
    column_block(a, m, n, 0, n);
    a.operand<double>(6, "A", hA, mat(m, n, lda), when(n > 0, NEED));
    a.operand<double>(6, "alpha", h_alpha, vec(n), when(n > 0, NEED));
    a.operand<double>(7, "b", h_b, vec(m), when(m > 0, NEED));
    a.operand<double>(8, "x", h_x, vec(n), when(n > 0, NEED));
    TRY(a);
    if (n == 0) return 0;
    CU(cudaSetDevice(c->device));
    const int64_t ldd = rup(m, 32);
    cudaStream_t st = c->copy_stream;
    TRY(c->hostA.ensure((size_t)ldd * n + (size_t)n, st));
    TRY(c->hostB.ensure((size_t)ldd, st));
    double* dA = c->hostA;
    double* dal = c->hostA + (size_t)ldd * n;
    CU(cudaMemcpy2DAsync(dA, (size_t)ldd * 8, hA, (size_t)lda * 8, (size_t)m * 8, (size_t)n, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(dal, h_alpha, (size_t)n * 8, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(c->hostB, h_b, (size_t)m * 8, cudaMemcpyHostToDevice, st));   // S:318: b itself is never touched
    TRY(dhqr_solve_f64(c, m, n, 0, n, dA, ldd, dal, c->hostB, ldd, 1, st));
    CU(cudaMemcpyAsync(h_x, c->hostB, (size_t)n * 8, cudaMemcpyDeviceToHost, st));     // S:320
    CU(cudaStreamSynchronize(st));
    return 0;
}

// ---- primitives ---------------------------------------------------------------------------------
extern "C++" {   // as for the adjoint solves above

template <typename T>
static int partialdot(dhqr_context* c, const void* d_a, const void* d_b, int64_t i0, int64_t i1, void* d_out, void* stream) {
    const unsigned rules = NEED | when(std::is_same<T, double2>::value, ALIGN);   // Float64 pointers are not checked for alignment here
    Check a(c);
    a.operand<T>(2, "a", d_a, vec(i1), rules);
    a.operand<T>(3, "b", d_b, vec(i1), rules);
    a.require(i0 >= 0, 4, "i0 < 0");
    a.require(i1 >= i0, 5, "i1 < i0");
    a.operand<T>(6, "out", d_out, vec(1), rules);
    TRY(a);
    CU(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    return launch(c, st, kname<T>("k_partialdot", "k_partialdot_c"), 0.0, [&](CwtSlot) {
        // k_partialdot_c sums its block in its own order, so the kernels stay one per type
        if constexpr (std::is_same<T, double>::value) k_partialdot<<<1, 1024, 0, st>>>((const T*)d_a, (const T*)d_b, i0, i1, (T*)d_out);
        else k_partialdot_c<<<1, 1024, 0, st>>>((const T*)d_a, (const T*)d_b, i0, i1, (T*)d_out);
    });
}

}  // extern "C++"

int dhqr_partialdot_f64(dhqr_handle c, const double* d_a, const double* d_b, int64_t i0, int64_t i1, double* d_out,
                        void* stream) {
    return partialdot<double>(c, d_a, d_b, i0, i1, d_out, stream);
}

int dhqr_partialdot_c64(dhqr_handle c, const void* d_a, const void* d_b, int64_t i0, int64_t i1, void* d_out, void* stream) {
    return partialdot<double2>(c, d_a, d_b, i0, i1, d_out, stream);
}

int dhqr_fill_uniform_f64(dhqr_handle c, uint64_t seed, int64_t i0, int64_t j0, int64_t m, int64_t n, double* dA,
                          int64_t lda, void* stream) {
    Check a(c);
    a.require(m >= 0, 5, "m < 0");
    a.require(n >= 0, 6, "n < 0");
    TRY(a);
    if (m == 0 || n == 0) return 0;
    TRY(a.operand<double>(7, "A", dA, mat(m, n, lda), NEED));
    CU(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid((unsigned)std::min<int64_t>((m + 255) / 256, 1024), (unsigned)std::min<int64_t>(n, 4096));
    return launch(c, st, "k_fill_uniform", 0.0, [&](CwtSlot) { k_fill_uniform<<<grid, 256, 0, st>>>(seed, i0, j0, m, n, dA, lda); });
}

// ---- kernel-level hooks ---------------------------------------------------------------------------
int dhqr_k_block_reflector_f64(dhqr_handle c, int64_t rows, int nbp, const double* dV, int64_t ldv, int64_t row_lo,
                               int ncols, double* dC, int64_t ldc, double* d_linv_out, void* stream) {
    if (!c) return set_err(-1, "null handle");
    if (rows <= 0) return set_err(-2, "rows <= 0");
    if (nbp < 1 || nbp > 128) return set_err(-3, "nbp out of range");
    if (!dV) return set_err(-4, "null V");
    if (ldv < rows) return set_err(-5, "ldv < rows");
    if (!dC) return set_err(-8, "null C");
    CU(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    TRY(ensure_workspace(c, st, rows, ncols));
    const int nbk = nbp <= IB ? IB : NBMAX;
    const int64_t vrows = rup(rows, 128);
    TRY(pack_v(c, st, dV, ldv, rows, nbp, 0, c->vpk2[0], 0, vrows, nbk));
    TRY(apply_block_reflector(c, st, c->vpk2[0], c->ws[0], 0, nbk, rows, row_lo, dC, ldc, ncols));
    if (d_linv_out) CU(cudaMemcpyAsync(d_linv_out, c->ws[0].linv, sizeof(double) * (size_t)nbk * nbk, cudaMemcpyDeviceToDevice, st));
    return 0;
}

int dhqr_debug_copy_f64(dhqr_handle c, const char* which, double* d_dst, int64_t nelems, void* stream) {
    if (!c) return set_err(-1, "null handle");
    if (!which) return set_err(-2, "null name");
    if (!d_dst) return set_err(-3, "null destination");
    if (!strcmp(which, "la_times")) {   // host-side list: converted to doubles and copied to the device buffer
        std::vector<double> t(c->la_times.begin(), c->la_times.end());
        if ((size_t)nelems < t.size()) return set_err(-4, "need %zu elements", t.size());
        CU(cudaMemcpy(d_dst, t.data(), t.size() * sizeof(double), cudaMemcpyHostToDevice));
        return 0;
    }
    if (!strcmp(which, "epochs")) {   // the tag counters ll_epoch, bs_epoch, uw_epoch (exact in a double)
        const double t[3] = {(double)c->ll_epoch, (double)c->bs_epoch, (double)c->uw_epoch};
        if (nelems < 3) return set_err(-4, "need 3 elements");
        CU(cudaMemcpy(d_dst, t, sizeof(t), cudaMemcpyHostToDevice));
        return 0;
    }
    if (!strcmp(which, "chain_wait")) {   // [0] = launches of the last look-ahead factorisation, then 6 doubles per launch
        std::vector<double> t(1, (double)(c->cwt_rows.size() / 6));
        t.insert(t.end(), c->cwt_rows.begin(), c->cwt_rows.end());
        if ((size_t)nelems < t.size()) return set_err(-4, "need %zu elements", t.size());
        CU(cudaMemcpy(d_dst, t.data(), t.size() * sizeof(double), cudaMemcpyHostToDevice));
        return 0;
    }
    if (!strcmp(which, "gemm_trace")) {   // [0] = rows, [1] = launches left untraced, then GTR_WORDS doubles per CTA
        std::vector<unsigned long long> rows(c->gtr_used * GTR_WORDS);
        if (!rows.empty()) CU(cudaMemcpy(rows.data(), c->gtr_rows.p, rows.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        std::vector<double> t = {(double)c->gtr_used, (double)c->gtr_dropped};
        t.insert(t.end(), rows.begin(), rows.end());
        if ((size_t)nelems < t.size()) return set_err(-4, "need %zu elements", t.size());
        CU(cudaMemcpy(d_dst, t.data(), t.size() * sizeof(double), cudaMemcpyHostToDevice));
        return 0;
    }
    const double* src = nullptr;
    size_t have = 0;
    if (!strcmp(which, "wpart")) { src = c->ws[0].wpart; have = c->ws[0].wpart.n; }
    else if (!strcmp(which, "wsum")) { src = c->ws[0].wsum; have = c->ws[0].wsum.n; }
    else if (!strcmp(which, "ypk")) { src = c->ws[0].ypk; have = c->ws[0].ypk.n; }
    else if (!strcmp(which, "linv")) { src = c->ws[0].linv; have = (size_t)NBMAX * NBMAX; }
    else if (!strcmp(which, "vpk")) { src = c->vpk2[0]; have = c->vpk2[0].n; }
    else if (!strcmp(which, "wstamps")) { src = (const double*)c->wstamps.p; have = c->wstamps.n; }
    else if (!strcmp(which, "wide")) { src = c->wbuf; have = c->wbuf.n; }
    else if (!strcmp(which, "panel_trace")) { src = (const double*)c->panel_trace.p; have = c->panel_trace.n; }
    else return set_err(-2, "unknown buffer '%s'", which);
    if (nelems < 0 || (size_t)nelems > have) return set_err(-4, "nelems out of range (have %zu)", have);
    CU(cudaMemcpyAsync(d_dst, src, sizeof(double) * (size_t)nelems, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return 0;
}

int dhqr_k_panel_f64(dhqr_handle c, int64_t rows, int ncols, double* dP, int64_t ldp, double* d_alpha, void* stream) {
    if (!c) return set_err(-1, "null handle");
    if (rows <= 0) return set_err(-2, "rows <= 0");
    if (ncols < 1 || ncols > IB || ncols > rows) return set_err(-3, "ncols out of range");
    if (!dP) return set_err(-4, "null panel");
    if (ldp < rows) return set_err(-5, "ldp < rows");
    if (!d_alpha) return set_err(-6, "null alpha");
    CU(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    TRY(ensure_workspace(c, st, rows, ncols));
    return launch_panel(c, st, c->vpk2[0], dP, ldp, rows, ncols, d_alpha, 0, 0, rup(rows, 128));
}

int dhqr_k_wide_panel_f64(dhqr_handle c, int64_t rows, double* dP, int64_t ldp, double* d_alpha, int* refused, void* stream) {
    if (!c) return set_err(-1, "null handle");
    if (rows < WP) return set_err(-2, "rows < 128");
    if (!dP) return set_err(-3, "null panel");
    if (ldp < rows) return set_err(-4, "ldp < rows");
    if (!d_alpha) return set_err(-5, "null alpha");
    if (!refused) return set_err(-6, "null result");
    CU(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    TRY(ensure_workspace(c, st, rows, WP));
    TRY(launch(c, st, "k_wide_reset", 0.0, [&](CwtSlot) { k_wide_reset<<<1, 32, 0, st>>>(c->wctl); }));
    const Panel p = {0, 0, WP};
    TRY(factor_outer_panel(c, st, c->vpk2[0], c->ws[0], p, rows, 0, dP, ldp, d_alpha, 0, true, c->ws[0].linv));
    WideCtl host;
    CU(cudaMemcpyAsync(&host, c->wctl, sizeof(host), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    *refused = host.status != 0 || host.fail_step != W_NOFAIL;
    return 0;
}

}  // extern "C"
