// nccl_loopback.cpp — a stand-in for NCCL whose ranks share one CUDA device, each rank in its own process (test infrastructure).
//
// libdhqr resolves ten NCCL entry points (load_nccl in dhqr_api.cu; DHQR_NCCL_LIBRARY selects the library).  This file exports
// exactly those, so that the multi-rank path (column blocks over ranks, V broadcasts, the hand-over of b) runs on one GPU.
// Real NCCL refuses two ranks on one device.
//
//   - The unique id names a control file in $DHQR_LOOPBACK_DIR.  Every rank maps it (MAP_SHARED); rank 0 unlinks it once every
//     rank has attached.
//   - Each rank exports a staging buffer (cudaIpcGetMemHandle) of NSLOT slots per receiver, plus interprocess events: "filled"
//     (the sender recorded it after writing a slot) and "drained" (the receiver recorded it after reading one).  A message goes
//     in slot-sized pieces: cudaMemcpyAsync into the sender's slot and out of it into the receiver's buffer, on the caller's
//     streams.
//   - A rank calls cudaStreamWaitEvent on a peer's event only after that peer has posted (in the control file) that the event is
//     recorded, so the transport never holds up the device.  Only the host waits, and every wait gives up after
//     $DHQR_LOOPBACK_TIMEOUT seconds (default 60) with ncclSystemError naming the rank, the call and the operation.
//   - Every call posts (sequence number, op, count, type, root or peer).  Collectives are compared with the same collective on
//     every other rank, a Send with the matching Recv; a mismatch returns ncclInvalidUsage and names both sides.  NCCL would
//     hang or move the wrong bytes instead.
//   - Data types 4 (int64) and 8 (float64); anything else returns ncclInvalidArgument.
#include <cuda_runtime.h>
#include <fcntl.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <time.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>

namespace {

enum { ncclSuccess = 0, ncclUnhandledCudaError = 1, ncclSystemError = 2, ncclInternalError = 3, ncclInvalidArgument = 4,
       ncclInvalidUsage = 5 };
enum Op { OP_NONE = 0, OP_BCAST = 1, OP_ALLGATHER = 2, OP_SEND = 3, OP_RECV = 4 };
const char* op_name(int op) {
    switch (op) {
        case OP_BCAST: return "Broadcast";
        case OP_ALLGATHER: return "AllGather";
        case OP_SEND: return "Send";
        case OP_RECV: return "Recv";
        default: return "none";
    }
}

constexpr int MAXR = 8;                      // ranks per communicator
constexpr int NSLOT = 2;                     // staging slots per (sender, receiver) channel
constexpr size_t SLOT = (size_t)1 << 21;     // 2 MiB: a 2048-row V buffer of the library already goes in several pieces
constexpr int LOG = 64;                      // posted calls kept per sequence

struct Desc { int64_t seq; int64_t count; int32_t op, type, root, peer; };

struct RankArea {
    std::atomic<int> ready;                                 // the handles below are valid
    cudaIpcMemHandle_t mem;
    cudaIpcEventHandle_t filled[MAXR][NSLOT];               // recorded after filling slot s of the channel to receiver r
    cudaIpcEventHandle_t drained[MAXR][NSLOT];              // recorded after reading slot s of sender r's channel to this rank
    std::atomic<int64_t> fill_gen[MAXR][NSLOT];             // generation of the piece last posted as filled
    std::atomic<int64_t> drain_gen[MAXR][NSLOT];            // generation of the piece last posted as drained
    std::atomic<int64_t> ncoll;                             // collectives posted
    Desc coll[LOG];
    std::atomic<int64_t> nsend[MAXR], nrecv[MAXR];          // sends to / receives from rank r posted
    Desc send[MAXR][LOG], recv[MAXR][LOG];
    Desc cur;                                               // the call in progress (for error texts only)
    std::atomic<int64_t> calls;
};
struct Shared {
    std::atomic<int> attached, opened, finished;
    int nranks;
    RankArea r[MAXR];
};

struct Comm {
    int rank = 0, nranks = 1, device = 0;
    Shared* sh = nullptr;
    char* buf = nullptr;                                    // this rank's staging buffer
    char* peer_buf[MAXR] = {};
    cudaEvent_t filled[MAXR][NSLOT] = {}, drained[MAXR][NSLOT] = {};
    cudaEvent_t peer_filled[MAXR][NSLOT] = {}, peer_drained[MAXR][NSLOT] = {};   // [peer][slot] of the channel with this rank
    int64_t sent_pieces[MAXR] = {}, recv_pieces[MAXR] = {}; // pieces moved per channel
    int64_t ncoll = 0, nsend[MAXR] = {}, nrecv[MAXR] = {}, calls = 0;
    Desc cur{};
};

thread_local char g_msg[1024] = "";
int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_msg, sizeof(g_msg), fmt, ap);
    va_end(ap);
    return code;
}

double timeout_s() {
    const char* t = getenv("DHQR_LOOPBACK_TIMEOUT");
    const double v = t ? atof(t) : 0.0;
    return v > 0 ? v : 60.0;
}
double now_s() {
    timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec + 1e-9 * ts.tv_nsec;
}

const char* describe(const Desc& d, char* out, size_t n) {
    if (d.op == OP_NONE) snprintf(out, n, "no call");
    else if (d.op == OP_SEND || d.op == OP_RECV)
        snprintf(out, n, "call #%lld %s(count %lld, type %d, peer %d)", (long long)d.seq, op_name(d.op), (long long)d.count, d.type, d.peer);
    else snprintf(out, n, "call #%lld %s(count %lld, type %d, root %d)", (long long)d.seq, op_name(d.op), (long long)d.count, d.type, d.root);
    return out;
}

// Waits on the host until pred() holds; on timeout fails with a text naming this rank's call, what it waited for and the peer's call.
template <typename P>
int wait_for(Comm* c, int peer, const char* what, P pred) {
    const double t0 = now_s(), tmax = timeout_s();
    for (long spin = 0; !pred(); ++spin) {
        if (spin > 1000) {
            if (now_s() - t0 > tmax) {
                char a[160], b[160];
                Desc pd = c->sh->r[peer].cur;
                return fail(ncclSystemError, "loopback: rank %d, %s: timed out after %.0f s waiting for rank %d (%s); rank %d is in %s",
                            c->rank, describe(c->cur, a, sizeof(a)), tmax, peer, what, peer, describe(pd, b, sizeof(b)));
            }
            usleep(spin > 100000 ? 200 : 20);
        }
    }
    return ncclSuccess;
}

#define CK(call)                                                                                                           \
    do {                                                                                                                   \
        cudaError_t e_ = (call);                                                                                           \
        if (e_ != cudaSuccess) return fail(ncclUnhandledCudaError, "loopback: rank %d: %s failed: %s", c->rank, #call,     \
                                           cudaGetErrorString(e_));                                                         \
    } while (0)
#define RET(call)              \
    do {                       \
        int r_ = (call);       \
        if (r_) return r_;     \
    } while (0)

int elem_size(int type) { return (type == 4 || type == 8) ? 8 : 0; }

int begin(Comm* c, int op, size_t count, int type, int root, int peer) {
    c->cur = {c->calls++, (int64_t)count, op, type, root, peer};
    c->sh->r[c->rank].cur = c->cur;
    c->sh->r[c->rank].calls.store(c->calls);
    if (!elem_size(type)) return fail(ncclInvalidArgument, "loopback: rank %d: data type %d is not supported (4 and 8 are)", c->rank, type);
    return ncclSuccess;
}

bool same(const Desc& a, const Desc& b) { return a.count == b.count && a.type == b.type && a.root == b.root; }

int mismatch(Comm* c, int peer, const Desc& mine, const Desc& theirs, const char* kind) {
    char a[160], b[160];
    return fail(ncclInvalidUsage, "loopback: %s mismatch: rank %d is in %s, rank %d in %s", kind, c->rank, describe(mine, a, sizeof(a)),
                peer, describe(theirs, b, sizeof(b)));
}

// every rank posts collective #k and compares it with the same collective on every other rank
int check_collective(Comm* c) {
    RankArea& me = c->sh->r[c->rank];
    const int64_t k = c->ncoll++;
    Desc d = c->cur;
    me.coll[k % LOG] = d;
    me.ncoll.store(k + 1);
    for (int p = 0; p < c->nranks; ++p) {
        if (p == c->rank) continue;
        RankArea& pa = c->sh->r[p];
        RET(wait_for(c, p, "its next collective", [&] { return pa.ncoll.load() > k; }));
        const Desc t = pa.coll[k % LOG];
        if (t.op != d.op || !same(t, d)) return mismatch(c, p, d, t, "collective");
    }
    return ncclSuccess;
}

// Send #k from this rank to `peer` against Recv #k of `peer` from this rank (or the other way round)
int check_p2p(Comm* c, int peer, bool sending) {
    RankArea& me = c->sh->r[c->rank];
    RankArea& pa = c->sh->r[peer];
    const int64_t k = sending ? c->nsend[peer]++ : c->nrecv[peer]++;
    Desc d = c->cur;
    Desc t{};
    if (sending) {
        me.send[peer][k % LOG] = d;
        me.nsend[peer].store(k + 1);
        RET(wait_for(c, peer, "the matching Recv", [&] { return pa.nrecv[c->rank].load() > k; }));
        t = pa.recv[c->rank][k % LOG];
    } else {
        me.recv[peer][k % LOG] = d;
        me.nrecv[peer].store(k + 1);
        RET(wait_for(c, peer, "the matching Send", [&] { return pa.nsend[c->rank].load() > k; }));
        t = pa.send[c->rank][k % LOG];
    }
    if (t.count != d.count || t.type != d.type) return mismatch(c, peer, d, t, "send/receive");
    return ncclSuccess;
}

// one piece of a message into the channel to `to`, after its previous occupant was read
int put_piece(Comm* c, int to, const char* src, size_t bytes, cudaStream_t st) {
    const int64_t k = c->sent_pieces[to]++;
    const int s = (int)(k % NSLOT);
    const int64_t g = k / NSLOT + 1;
    if (g > 1) {
        RankArea& pa = c->sh->r[to];
        RET(wait_for(c, to, "a staging slot to be read", [&] { return pa.drain_gen[c->rank][s].load() >= g - 1; }));
        CK(cudaStreamWaitEvent(st, c->peer_drained[to][s], 0));
    }
    CK(cudaMemcpyAsync(c->buf + ((size_t)to * NSLOT + s) * SLOT, src, bytes, cudaMemcpyDeviceToDevice, st));
    CK(cudaEventRecord(c->filled[to][s], st));
    c->sh->r[c->rank].fill_gen[to][s].store(g);
    return ncclSuccess;
}

// one piece of a message out of the channel from `from`
int get_piece(Comm* c, int from, char* dst, size_t bytes, cudaStream_t st) {
    const int64_t k = c->recv_pieces[from]++;
    const int s = (int)(k % NSLOT);
    const int64_t g = k / NSLOT + 1;
    RankArea& pa = c->sh->r[from];
    RET(wait_for(c, from, "a staging slot to be filled", [&] { return pa.fill_gen[c->rank][s].load() >= g; }));
    CK(cudaStreamWaitEvent(st, c->peer_filled[from][s], 0));
    CK(cudaMemcpyAsync(dst, c->peer_buf[from] + ((size_t)c->rank * NSLOT + s) * SLOT, bytes, cudaMemcpyDeviceToDevice, st));
    CK(cudaEventRecord(c->drained[from][s], st));
    c->sh->r[c->rank].drain_gen[from][s].store(g);
    return ncclSuccess;
}

int set_device(Comm* c) {
    int d = -1;
    CK(cudaGetDevice(&d));
    if (d != c->device) return fail(ncclInvalidUsage, "loopback: rank %d: called on device %d, communicator is on %d", c->rank, d, c->device);
    return ncclSuccess;
}

}  // namespace

extern "C" {

typedef struct { char internal[128]; } ncclUniqueId;
typedef Comm* ncclComm_t;

const char* ncclGetErrorString(int result) {
    if (g_msg[0]) return g_msg;
    switch (result) {
        case ncclSuccess: return "no error";
        case ncclUnhandledCudaError: return "unhandled cuda error";
        case ncclSystemError: return "system error";
        case ncclInvalidArgument: return "invalid argument";
        case ncclInvalidUsage: return "invalid usage";
        default: return "internal error";
    }
}

int ncclGroupStart() { return ncclSuccess; }
int ncclGroupEnd() { return ncclSuccess; }

int ncclGetUniqueId(ncclUniqueId* id) {
    g_msg[0] = 0;
    const char* dir = getenv("DHQR_LOOPBACK_DIR");
    if (!id) return fail(ncclInvalidArgument, "loopback: null unique id");
    if (!dir || !*dir) return fail(ncclSystemError, "loopback: DHQR_LOOPBACK_DIR is not set");
    static std::atomic<int> serial{0};
    memset(id, 0, sizeof(*id));
    timespec ts;
    clock_gettime(CLOCK_REALTIME, &ts);
    snprintf(id->internal, sizeof(id->internal), "dhqr-loopback-%d-%d-%lx", (int)getpid(), serial++, (long)ts.tv_nsec);
    char path[4096];
    snprintf(path, sizeof(path), "%s/%s", dir, id->internal);
    const int fd = open(path, O_RDWR | O_CREAT | O_EXCL, 0600);
    if (fd < 0) return fail(ncclSystemError, "loopback: cannot create %s", path);
    const int rc = ftruncate(fd, sizeof(Shared));   // zero-filled: every counter starts at 0
    close(fd);
    if (rc) { unlink(path); return fail(ncclSystemError, "loopback: cannot size %s", path); }
    return ncclSuccess;
}

int ncclCommInitRank(ncclComm_t* out, int nranks, ncclUniqueId id, int rank) {
    g_msg[0] = 0;
    if (!out || nranks < 1 || nranks > MAXR || rank < 0 || rank >= nranks)
        return fail(ncclInvalidArgument, "loopback: rank %d of %d (at most %d ranks)", rank, nranks, MAXR);
    const char* dir = getenv("DHQR_LOOPBACK_DIR");
    if (!dir || !*dir) return fail(ncclSystemError, "loopback: DHQR_LOOPBACK_DIR is not set");
    id.internal[sizeof(id.internal) - 1] = 0;
    char path[4096];
    snprintf(path, sizeof(path), "%s/%s", dir, id.internal);
    const int fd = open(path, O_RDWR);
    if (fd < 0) return fail(ncclSystemError, "loopback: rank %d cannot open the control file %s", rank, path);
    void* p = mmap(nullptr, sizeof(Shared), PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    close(fd);
    if (p == MAP_FAILED) return fail(ncclSystemError, "loopback: rank %d cannot map %s", rank, path);
    Comm* c = new Comm();
    c->rank = rank;
    c->nranks = nranks;
    c->sh = (Shared*)p;
    c->cur = {0, 0, OP_NONE, 0, 0, 0};
    CK(cudaGetDevice(&c->device));
    RankArea& me = c->sh->r[rank];
    CK(cudaMalloc((void**)&c->buf, (size_t)MAXR * NSLOT * SLOT));
    CK(cudaIpcGetMemHandle(&me.mem, c->buf));
    for (int r = 0; r < MAXR; ++r)
        for (int s = 0; s < NSLOT; ++s) {
            CK(cudaEventCreateWithFlags(&c->filled[r][s], cudaEventInterprocess | cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&c->drained[r][s], cudaEventInterprocess | cudaEventDisableTiming));
            CK(cudaIpcGetEventHandle(&me.filled[r][s], c->filled[r][s]));
            CK(cudaIpcGetEventHandle(&me.drained[r][s], c->drained[r][s]));
        }
    me.ready.store(1);
    c->sh->attached.fetch_add(1);
    for (int q = 0; q < nranks; ++q) {
        if (q == rank) continue;
        RankArea& pa = c->sh->r[q];
        RET(wait_for(c, q, "CommInitRank", [&] { return pa.ready.load() == 1; }));
        cudaError_t e = cudaIpcOpenMemHandle((void**)&c->peer_buf[q], pa.mem, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess)
            return fail(ncclSystemError, "loopback: rank %d: cudaIpcOpenMemHandle of rank %d's staging buffer failed: %s", rank, q,
                        cudaGetErrorString(e));
        for (int s = 0; s < NSLOT; ++s) {
            CK(cudaIpcOpenEventHandle(&c->peer_filled[q][s], pa.filled[rank][s]));
            CK(cudaIpcOpenEventHandle(&c->peer_drained[q][s], pa.drained[rank][s]));
        }
    }
    c->sh->opened.fetch_add(1);
    if (rank == 0) {   // once every rank has the file mapped, nothing needs its name: nothing is left behind
        RET(wait_for(c, nranks > 1 ? 1 : 0, "every rank to attach", [&] { return c->sh->opened.load() == nranks; }));
        unlink(path);
    }
    *out = c;
    return ncclSuccess;
}

int ncclCommDestroy(ncclComm_t c) {
    g_msg[0] = 0;
    if (!c) return ncclSuccess;
    int rc = ncclSuccess;
    // a peer may still be reading this rank's slots: every rank drains its device work, then the buffers go
    cudaDeviceSynchronize();
    c->sh->finished.fetch_add(1);
    for (int q = 0; q < c->nranks && !rc; ++q)
        if (q != c->rank) rc = wait_for(c, q, "CommDestroy", [&] { return c->sh->finished.load() >= c->nranks; });
    for (int q = 0; q < c->nranks; ++q) {
        if (q == c->rank) continue;
        if (c->peer_buf[q]) cudaIpcCloseMemHandle(c->peer_buf[q]);
        for (int s = 0; s < NSLOT; ++s) {
            if (c->peer_filled[q][s]) cudaEventDestroy(c->peer_filled[q][s]);
            if (c->peer_drained[q][s]) cudaEventDestroy(c->peer_drained[q][s]);
        }
    }
    for (int r = 0; r < MAXR; ++r)
        for (int s = 0; s < NSLOT; ++s) {
            if (c->filled[r][s]) cudaEventDestroy(c->filled[r][s]);
            if (c->drained[r][s]) cudaEventDestroy(c->drained[r][s]);
        }
    cudaFree(c->buf);
    munmap(c->sh, sizeof(Shared));
    delete c;
    return rc;
}

int ncclBroadcast(const void* sendbuff, void* recvbuff, size_t count, int datatype, int root, ncclComm_t c, cudaStream_t st) {
    g_msg[0] = 0;
    if (!c) return fail(ncclInvalidArgument, "loopback: null communicator");
    RET(begin(c, OP_BCAST, count, datatype, root, -1));
    if (root < 0 || root >= c->nranks) return fail(ncclInvalidArgument, "loopback: rank %d: Broadcast root %d", c->rank, root);
    RET(set_device(c));
    RET(check_collective(c));
    const size_t bytes = count * elem_size(datatype);
    if (c->rank == root) {
        if (sendbuff != recvbuff && bytes) CK(cudaMemcpyAsync(recvbuff, sendbuff, bytes, cudaMemcpyDeviceToDevice, st));
        for (size_t off = 0; off < bytes; off += SLOT)
            for (int q = 0; q < c->nranks; ++q)
                if (q != root) RET(put_piece(c, q, (const char*)sendbuff + off, std::min(SLOT, bytes - off), st));
    } else {
        for (size_t off = 0; off < bytes; off += SLOT) RET(get_piece(c, root, (char*)recvbuff + off, std::min(SLOT, bytes - off), st));
    }
    return ncclSuccess;
}

int ncclAllGather(const void* sendbuff, void* recvbuff, size_t count, int datatype, ncclComm_t c, cudaStream_t st) {
    g_msg[0] = 0;
    if (!c) return fail(ncclInvalidArgument, "loopback: null communicator");
    RET(begin(c, OP_ALLGATHER, count, datatype, -1, -1));
    RET(set_device(c));
    RET(check_collective(c));
    const size_t bytes = count * elem_size(datatype);
    char* out = (char*)recvbuff;
    if (bytes && (const char*)sendbuff != out + c->rank * bytes)
        CK(cudaMemcpyAsync(out + c->rank * bytes, sendbuff, bytes, cudaMemcpyDeviceToDevice, st));
    // piece by piece: every rank fills piece i for all peers before it reads piece i from them, so no ring waits on another
    for (size_t off = 0; off < bytes; off += SLOT) {
        const size_t len = std::min(SLOT, bytes - off);
        for (int q = 0; q < c->nranks; ++q)
            if (q != c->rank) RET(put_piece(c, q, (const char*)sendbuff + off, len, st));
        for (int q = 0; q < c->nranks; ++q)
            if (q != c->rank) RET(get_piece(c, q, out + q * bytes + off, len, st));
    }
    return ncclSuccess;
}

int ncclSend(const void* sendbuff, size_t count, int datatype, int peer, ncclComm_t c, cudaStream_t st) {
    g_msg[0] = 0;
    if (!c) return fail(ncclInvalidArgument, "loopback: null communicator");
    RET(begin(c, OP_SEND, count, datatype, -1, peer));
    if (peer < 0 || peer >= c->nranks || peer == c->rank) return fail(ncclInvalidArgument, "loopback: rank %d: Send to rank %d", c->rank, peer);
    RET(set_device(c));
    RET(check_p2p(c, peer, true));
    const size_t bytes = count * elem_size(datatype);
    for (size_t off = 0; off < bytes; off += SLOT) RET(put_piece(c, peer, (const char*)sendbuff + off, std::min(SLOT, bytes - off), st));
    return ncclSuccess;
}

int ncclRecv(void* recvbuff, size_t count, int datatype, int peer, ncclComm_t c, cudaStream_t st) {
    g_msg[0] = 0;
    if (!c) return fail(ncclInvalidArgument, "loopback: null communicator");
    RET(begin(c, OP_RECV, count, datatype, -1, peer));
    if (peer < 0 || peer >= c->nranks || peer == c->rank) return fail(ncclInvalidArgument, "loopback: rank %d: Recv from rank %d", c->rank, peer);
    RET(set_device(c));
    RET(check_p2p(c, peer, false));
    const size_t bytes = count * elem_size(datatype);
    for (size_t off = 0; off < bytes; off += SLOT) RET(get_piece(c, peer, (char*)recvbuff + off, std::min(SLOT, bytes - off), st));
    return ncclSuccess;
}

}  // extern "C"
