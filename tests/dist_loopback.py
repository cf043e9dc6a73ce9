"""The multi-rank path on one GPU: P rank processes on cuda:0 that talk through tests/nccl_loopback.cpp, a stand-in for NCCL built
on CUDA IPC (test infrastructure for test_gpu_dist_loopback.py).

``build()`` compiles the stand-in with nvcc into a temporary directory; ``run(P, job, outdir, lib)`` spawns P ranks (the
``spawn`` start method, one process each: processes on one device are time-sliced, so each rank has the whole device while it
runs, as it would alone), ships the unique id through a gloo process group and the unchanged ``init_distributed(device=0)``,
runs one job (every case of one configuration) and returns each rank's results.  A hard timeout applies, and on any exit every
child is terminated and joined.  A device that refuses a second context or cudaIpcOpenMemHandle makes the caller skip.

The jobs below run on every rank.  They write ``rank{r}.npz`` under ``outdir``: arrays keyed "<case>/<what>".
"""
import os
import shutil
import subprocess
import tempfile
import time
import traceback

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SLOT_DOUBLES = (1 << 21) // 8                      # staging slot of the stand-in, in 8-byte elements
SKIP_MARKERS = ("cudaIpcOpenMemHandle", "busy or unavailable", "CUDA-capable device", "all CUDA-capable devices are busy")


def build():
    """(directory, path of libnccl_loopback.so); the caller removes the directory once the runs are done."""
    out = tempfile.mkdtemp(prefix="nccl_loopback_")
    so = os.path.join(out, "libnccl_loopback.so")
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    nvcc = nvcc if os.path.exists(nvcc) else (shutil.which("nvcc") or "nvcc")
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fPIC",
                           "-cudart", "shared", "-o", so, os.path.join(HERE, "nccl_loopback.cpp")])
    return out, so


def _worker(rank, P, job, outdir, env, args):
    os.environ.update(env)
    try:
        import torch
        import torch.distributed as dist
        try:
            torch.cuda.set_device(0)
            torch.zeros(1, device="cuda:0")
        except RuntimeError as e:
            with open(os.path.join(outdir, f"skip{rank}.txt"), "w") as fh:
                fh.write(f"rank {rank}: a second CUDA context on device 0 failed: {e}")
            return
        dist.init_process_group("gloo", init_method="file://" + os.path.join(outdir, "pg_store"), rank=rank, world_size=P)
        try:
            res = JOBS[job](rank, P, *args)
        finally:
            dist.destroy_process_group()
        np.savez(os.path.join(outdir, f"rank{rank}.npz"), **res)
    except BaseException as e:                      # noqa: BLE001 - reported by the parent
        text = traceback.format_exc()
        name = "skip" if any(s in str(e) for s in SKIP_MARKERS) else "err"
        with open(os.path.join(outdir, f"{name}{rank}.txt"), "w") as fh:
            fh.write(f"rank {rank}: {text}")
        raise SystemExit(1)


class Skip(Exception):
    pass


def run(P, job, outdir, lib, args=(), timeout=900.0):
    """Runs ``job`` on P ranks; returns a list of per-rank dicts.  Raises Skip(reason) or AssertionError."""
    import multiprocessing as mp
    os.makedirs(outdir, exist_ok=True)
    env = {"DHQR_NCCL_LIBRARY": lib, "DHQR_LOOPBACK_DIR": outdir, "DHQR_LOOPBACK_TIMEOUT": "60",
           "OMP_NUM_THREADS": "4", "OMP_WAIT_POLICY": "PASSIVE"}
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_worker, args=(r, P, job, outdir, env, args)) for r in range(P)]
    t0 = time.monotonic()
    timed_out = False
    try:
        for p in procs:
            p.start()
        failed_at = None
        while any(p.is_alive() for p in procs):
            now = time.monotonic()
            if failed_at is None and any(p.exitcode not in (None, 0) for p in procs):
                failed_at = now                      # the others get a moment to report their side, then they go
            if now - t0 > timeout or (failed_at is not None and now - failed_at > 5.0):
                timed_out = failed_at is None
                break
            time.sleep(0.1)
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
        for p in procs:
            p.join(10)
            if p.is_alive():
                p.kill()
                p.join()
    skips = [open(os.path.join(outdir, f)).read() for f in sorted(os.listdir(outdir)) if f.startswith("skip")]
    errs = [open(os.path.join(outdir, f)).read() for f in sorted(os.listdir(outdir)) if f.startswith("err")]
    if skips:
        raise Skip(skips[0].strip().splitlines()[-1])
    assert not timed_out, f"job {job} on {P} ranks did not finish within {timeout:.0f} s; " + "\n".join(errs)
    assert not errs, f"job {job} on {P} ranks failed:\n" + "\n".join(errs)
    codes = [p.exitcode for p in procs]
    assert codes == [0] * P, f"job {job} on {P} ranks: exit codes {codes}"
    out = []
    for r in range(P):
        with np.load(os.path.join(outdir, f"rank{r}.npz")) as z:
            out.append({k: z[k] for k in z.files})
    return out


# ---------------------------------------------------------------------------------------------------------------------
# jobs (run on every rank)
# ---------------------------------------------------------------------------------------------------------------------
import ctypes as _C


class _UniqueId(_C.Structure):
    _fields_ = [("internal", _C.c_char * 128)]


def _nccl(lib):
    C = _C
    L = C.CDLL(lib)
    vp, sz, ci = C.c_void_p, C.c_size_t, C.c_int
    L.ncclGetUniqueId.argtypes = [C.POINTER(_UniqueId)]
    L.ncclCommInitRank.argtypes = [C.POINTER(vp), ci, _UniqueId, ci]
    L.ncclCommDestroy.argtypes = [vp]
    L.ncclBroadcast.argtypes = [vp, vp, sz, ci, ci, vp, vp]
    L.ncclAllGather.argtypes = [vp, vp, sz, ci, vp, vp]
    L.ncclSend.argtypes = [vp, sz, ci, ci, vp, vp]
    L.ncclRecv.argtypes = [vp, sz, ci, ci, vp, vp]
    L.ncclGetErrorString.restype = C.c_char_p
    return L


def transport(rank, P, lib):
    """Bitwise transfers of the stand-in itself: Broadcast from every root in place and out of place, AllGather, Send/Recv
    between every ordered pair, at 1 element, odd sizes and sizes over one and over three staging slots, both data types, on a
    non-blocking stream.  Then the refusals: an unsupported data type and two ranks that disagree on a count."""
    import ctypes as C
    import torch
    import torch.distributed as dist
    L = _nccl(lib)
    uid = _UniqueId()
    if rank == 0:
        assert L.ncclGetUniqueId(C.byref(uid)) == 0, L.ncclGetErrorString(0)
    obj = [bytes(_C.string_at(C.addressof(uid), 128))]
    dist.broadcast_object_list(obj, src=0)
    uid = _UniqueId.from_buffer_copy(obj[0])
    comm = C.c_void_p()
    rc = L.ncclCommInitRank(C.byref(comm), P, uid, rank)
    assert rc == 0, L.ncclGetErrorString(rc).decode()
    st = torch.cuda.Stream(device=0)
    sp = C.c_void_p(st.cuda_stream)
    dev = "cuda:0"

    def data(seed, count):
        g = torch.Generator().manual_seed(seed)
        return torch.randint(-2 ** 62, 2 ** 62, (count,), generator=g, dtype=torch.int64)

    def ok(rc):
        assert rc == 0, L.ncclGetErrorString(rc).decode()

    sizes = [1, 7, 1001, SLOT_DOUBLES + 3, 3 * SLOT_DOUBLES + 5]
    checks = 0
    for ti, typ in enumerate((8, 4)):
        for si, count in enumerate(sizes):
            for root in range(P):
                for inplace in (True, False):
                    seed = 1000 * ti + 100 * si + 10 * root + inplace
                    want = data(seed, count)
                    with torch.cuda.stream(st):
                        src = want.to(dev) if rank == root else torch.full((count,), -1, dtype=torch.int64, device=dev)
                        dst = src if inplace else torch.full((count,), -2, dtype=torch.int64, device=dev)
                        ok(L.ncclBroadcast(src.data_ptr(), dst.data_ptr(), count, typ, root, comm, sp))
                    st.synchronize()
                    assert torch.equal(dst.cpu(), want), f"Broadcast type {typ} count {count} root {root} inplace {inplace}"
                    checks += 1
            with torch.cuda.stream(st):
                mine = data(7000 + 100 * si + rank, count).to(dev)
                out = torch.full((P * count,), -3, dtype=torch.int64, device=dev)
                ok(L.ncclAllGather(mine.data_ptr(), out.data_ptr(), count, typ, comm, sp))
            st.synchronize()
            assert torch.equal(out.cpu(), torch.cat([data(7000 + 100 * si + q, count) for q in range(P)])), f"AllGather {count}"
            checks += 1
            for s in range(P):
                for r in range(P):
                    if s == r or rank not in (s, r):
                        continue
                    want = data(9000 + 100 * si + 10 * s + r, count)
                    with torch.cuda.stream(st):
                        if rank == s:
                            buf = want.to(dev)
                            ok(L.ncclSend(buf.data_ptr(), count, typ, r, comm, sp))
                        else:
                            buf = torch.full((count,), -4, dtype=torch.int64, device=dev)
                            ok(L.ncclRecv(buf.data_ptr(), count, typ, s, comm, sp))
                    st.synchronize()
                    assert torch.equal(buf.cpu(), want), f"Send {s} -> {r} count {count}"
                    checks += 1
    x = torch.zeros(16, dtype=torch.int64, device=dev)
    rc_type = L.ncclBroadcast(x.data_ptr(), x.data_ptr(), 16, 7, 0, comm, sp)        # float16 / anything but 4 and 8
    rc_count = L.ncclBroadcast(x.data_ptr(), x.data_ptr(), 10 + rank, 8, 0, comm, sp)  # ranks disagree on the count
    text = L.ncclGetErrorString(rc_count).decode()
    torch.cuda.synchronize()
    ok(L.ncclCommDestroy(comm))
    return {"checks": np.array(checks), "rc_type": np.array(rc_type), "rc_count": np.array(rc_count), "text": np.array(text)}


def _init(P):
    import dhqr_b200 as D
    h = D.init_distributed(device=0)
    assert h.nranks == P
    return D, h


def _local(D, A, bounds, rank):
    import torch
    c0, c1 = bounds[rank], bounds[rank + 1]
    Al = D.colmajor_empty(A.shape[0], c1 - c0, "cuda:0")
    if c1 > c0:
        Al.copy_(torch.from_numpy(np.ascontiguousarray(A[:, c0:c1])))
    return D.ColumnBlockMatrix(Al, A.shape[1], c0, D.default_handle(0)), Al


def _factor_case(D, h, rank, out, key, A, bounds, nb, opts, solve, b):
    """qr! on the column block of this rank, then Q'b (qt_vec 1 and 0), Qb and x (bs_wave 1 and 0) for one right-hand side."""
    import torch
    from ext_rule import COUNTERS, counters, options
    with options(h, **opts):
        c0 = counters(h)
        Ad, Al = _local(D, A, bounds, rank)
        st = D.qr_(Ad, nb=nb)
        torch.cuda.synchronize()
        c1 = counters(h)
        out[key + "/H"] = Al.cpu().numpy()
        out[key + "/alpha"] = st.α.cpu().numpy()
        out[key + "/counters"] = np.array([c1[k] - c0[k] for k in COUNTERS])
        if not solve:
            return
        bd = torch.from_numpy(b.copy()).cuda()
        for qv in (1, 0):
            with options(h, qt_vec=qv):
                out[f"{key}/qtb{qv}"] = D.apply_qt_(bd.clone(), Ad).cpu().numpy()
        out[key + "/qb"] = D.apply_q_(bd.clone(), Ad).cpu().numpy()
        for bw in (1, 0):
            with options(h, bs_wave=bw):
                out[f"{key}/x{bw}"] = D.ldiv(st, bd).cpu().numpy()


def matrix(rank, P, cases):
    """cases: (key, family, m, n, bounds, nb, opts, solve, stream) with stream "default" or "side" (a low-priority
    non-blocking stream)."""
    import torch
    import matrix_families as F
    D, h = _init(P)
    out = {}
    for key, family, m, n, bounds, nb, opts, solve, stream in cases:
        A = F.make(family, m, n)
        b = F.rhs(m, 4)[:, 0]
        if stream == "side":
            s = torch.cuda.Stream(device=0, priority=0)
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                _factor_case(D, h, rank, out, key, A, bounds, nb, opts, solve, b)
            s.synchronize()
        else:
            _factor_case(D, h, rank, out, key, A, bounds, nb, opts, solve, b)
    D.shutdown_distributed()
    return out


def pad_payload(rank, m, ldb, nrhs):
    """The bits of a column-major (ldb, nrhs) block whose padding rows m..ldb-1 hold NaNs with a payload naming the rank, the
    column and the row."""
    bits = np.zeros((nrhs, ldb), dtype=np.uint64)
    col = np.arange(nrhs, dtype=np.uint64)[:, None]
    row = np.arange(ldb, dtype=np.uint64)[None, :]
    nan = np.uint64(0x7FF8000000000000) | (np.uint64(rank + 1) << np.uint64(40)) | (col << np.uint64(16)) | row
    bits[:, m:] = nan[:, m:]
    return bits


def rhs_blocks(rank, P, family, m, n, bounds, widths):
    """Q'b, Qb and the least-squares solve of (m, k) blocks with ldb = m + 5 whose padding rows hold rank-specific NaNs."""
    import torch
    import matrix_families as F
    D, h = _init(P)
    out = {}
    A = F.make(family, m, n)
    Ad, Al = _local(D, A, bounds, rank)
    st = D.qr_(Ad)
    for k in widths:
        B = F.rhs(m, 4)[:, 1:] if k == 3 else F.rhs(m, k)
        ldb = m + 5
        for what in ("qtb", "qb", "x"):
            bits = pad_payload(rank, m, ldb, k)
            full = bits.view(np.float64).copy()
            full[:, :m] = B.T
            base = torch.from_numpy(full).cuda()
            blk = base.t()[:m, :]
            if what == "qtb":
                D.apply_qt_(blk, Ad)
            elif what == "qb":
                D.apply_q_(blk, Ad)
            else:
                D.solve_householder_(blk, Ad, st.α)
            got = base.cpu().numpy()
            out[f"k{k}/{what}"] = np.ascontiguousarray(got[:, :m].T)
            out[f"k{k}/{what}_pad_ok"] = np.array(np.array_equal(got.view(np.uint64)[:, m:], bits[:, m:]))
    D.shutdown_distributed()
    return out


def restart(rank, P, m, n, dup, bounds_list):
    """test_gpu_dist.py's refused panel: column `dup` nearly equals column dup - 30, so the wide chain refuses its panel on the
    owner's device; every rank must learn it from the broadcast V buffer and redo the panel.  Once per partition."""
    import torch
    D, h = _init(P)
    out = {}
    for i, bounds in enumerate(bounds_list):
        c0, nl = bounds[rank], bounds[rank + 1] - bounds[rank]
        Al = D.colmajor_empty(m, nl, "cuda:0")
        D.fill_uniform_(Al, 0, 0, c0, h)
        if c0 <= dup < c0 + nl:
            noise = D.colmajor_empty(m, 1, "cuda:0")
            D.fill_uniform_(noise, 13, 0, 0, h)
            Al[:, dup - c0] = Al[:, dup - 30 - c0] + 1e-11 * noise[:, 0]
        r0 = h.get_option("wide_redone")
        H = D.qr_(D.ColumnBlockMatrix(Al, n, c0, h))
        torch.cuda.synchronize()
        out[f"{i}/redone"] = np.array(h.get_option("wide_redone") - r0)
        out[f"{i}/H"] = Al.cpu().numpy()
        out[f"{i}/alpha"] = H.α.cpu().numpy()
    D.shutdown_distributed()
    return out


def errors(rank, P):
    """Rank-uniform refusals, each followed by a valid call on the same handle; then the single-rank entry points, which must
    refuse a multi-rank handle with -1 and enqueue nothing."""
    import torch
    import dhqr_b200 as D
    import matrix_families as F
    D, h = _init(P)
    out = {}
    err = D._lib.DhqrError

    def code(fn):
        try:
            fn()
        except err as e:
            return e.code
        return 0

    def valid(tag):
        A = F.make("normal", 512, 256)
        Ad, Al = _local(D, A, D.splits(P, 256), rank)
        st = D.qr_(Ad)
        torch.cuda.synchronize()
        out[tag + "/H"] = Al.cpu().numpy()
        out[tag + "/alpha"] = st.α.cpu().numpy()

    lim = 728 * min(h.get_option("sms"), 160)
    big = D.colmajor_empty(lim + 1, 32, "cuda:0")
    D.fill_uniform_(big, 0, 0, 32 * rank, h)
    out["rows/code"] = np.array(code(lambda: D.qr_(D.ColumnBlockMatrix(big, 32 * P, 32 * rank, h))))
    del big
    valid("rows")
    n = 1024
    c0, nl = (0, 600) if rank == 0 else (500 + 524 * (rank - 1), 524)   # rank 1 starts inside rank 0's block
    n = max(n, c0 + nl)
    Al = D.colmajor_empty(2048, nl, "cuda:0")
    D.fill_uniform_(Al, 0, 0, c0, h)
    out["overlap/code"] = np.array(code(lambda: D.qr_(D.ColumnBlockMatrix(Al, n, c0, h))))
    valid("overlap")
    # single-rank entry points
    A = D.colmajor_empty(64, 32, "cuda:0")
    D.fill_uniform_(A, 0, 0, 0, h)
    alpha = torch.ones(32, dtype=torch.float64, device="cuda:0")
    b = torch.ones(64, dtype=torch.float64, device="cuda:0")
    p = torch.arange(32, dtype=torch.int64, device="cuda:0")
    Ah = np.asfortranarray(np.random.default_rng(0).random((64, 32)))
    Ac = torch.ones((64, 32), dtype=torch.complex128, device="cuda:0").t().contiguous().t()
    ac = torch.ones(32, dtype=torch.complex128, device="cuda:0")
    bc = torch.ones(64, dtype=torch.complex128, device="cuda:0")
    calls = {
        "form_q": lambda: D.form_q(A, handle=h),
        "forwardsolve": lambda: D.forwardsolve_(b.clone(), A, alpha, handle=h),
        "solve_adj": lambda: D.solve_adjoint_(b.clone(), A, alpha, handle=h),
        "qrcp": lambda: D.qrcp_(A.clone(), handle=h),
        "solve_qrcp": lambda: D.solve_qrcp_(b.clone(), A, alpha, p, 32, handle=h),
        "qr_host": lambda: D.qr_(Ah.copy(order="F"), handle=h),
        "ldiv_host": lambda: D.ldiv(D.DistributedHouseholderQRStruct(Ah.copy(order="F"), np.ones(32), h), np.ones(64)),
        "qr_c64": lambda: D.householder_(Ac.clone(), ac.clone(), handle=h),
        "apply_qt_c64": lambda: D.apply_qt_(bc.clone(), Ac, handle=h),
        "solve_c64": lambda: D.solve_householder_(bc.clone(), Ac, ac, handle=h),
        "backsolve_c64": lambda: D.backsolve_(bc.clone(), Ac, ac, handle=h),
        "form_q_c64": lambda: D.form_q(Ac, handle=h),
    }
    for name, fn in calls.items():
        l0 = h.launch_count()
        out[f"single/{name}"] = np.array([code(fn), h.launch_count() - l0])
    torch.cuda.synchronize()
    D.shutdown_distributed()
    return out


JOBS = {"transport": transport, "matrix": matrix, "rhs_blocks": rhs_blocks, "restart": restart, "errors": errors}
