"""GPU diagnostic battery: every kernel of libdhqr.so checked in isolation against torch fp64 / the CPU
oracle, then the full qr!/\\ path, then quick timings.  Prints one line per check and writes
build/diag.json.  Run under `timeout` on an H100: python tools/gpu_diag.py [--quick]"""
import json, os, sys, time, traceback
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import ctypes as C
import numpy as np
import torch
import dhqr_b200 as D
import dhqr_oracle as O

res = []
def say(*a):
    print(*a, flush=True)

def check(name, fn):
    say(f"[run ] {name}")
    t = time.time()
    try:
        out = fn()
        torch.cuda.synchronize()
        ok = bool(out.pop("ok")) if isinstance(out, dict) and "ok" in out else True
        res.append({"name": name, "ok": ok, "t": time.time() - t, **(out or {})})
        say(f"[{'PASS' if ok else 'FAIL'}] {name} {out} ({time.time()-t:.2f}s)")
    except Exception as e:
        res.append({"name": name, "ok": False, "err": repr(e)})
        say(f"[EXC ] {name}: {e!r}")
        traceback.print_exc()

dev = torch.device("cuda:0")
h = D.default_handle(0)
h.set_option("sync", 1)
co = O.COracle()
sp = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
vp = lambda t: C.c_void_p(t.data_ptr())

def t_fill():
    A = D.colmajor_empty(257, 33, dev)
    D.fill_uniform_(A, 7, 3, 5)
    ref = O.np_uniform(7, 257, 33, 3, 5)
    return {"ok": bool((A.cpu().numpy() == ref).all())}
check("fill_uniform bit-exact", t_fill)

def t_pdot():
    a = torch.rand(1000, dtype=torch.float64, device=dev); b = torch.rand(1000, dtype=torch.float64, device=dev)
    worst = 0.0
    for i0 in (0, 1, 17, 999):
        got = D.partialdot(a, b, range(i0, 1000)); ref = float(a[i0:] @ b[i0:])
        worst = max(worst, abs(got - ref) / max(abs(ref), 1e-300))
    return {"ok": worst < 1e-13, "rel": worst}
check("partialdot", t_pdot)

def block_reflector_case(rows, nbp, ncols, row_lo, ld_extra=0, seed=0):
    g = torch.Generator(device="cpu"); g.manual_seed(seed)
    # a genuine Householder block (|v|^2 = 2): V = tril of the oracle's factorisation of a random panel
    Hp, _ = O.np_qr(O.np_uniform(seed + 11, rows - row_lo, nbp))
    V = torch.zeros(rows, nbp, dtype=torch.float64)
    V[row_lo:] = torch.from_numpy(np.tril(Hp))
    Cm = torch.rand(rows, ncols, dtype=torch.float64, generator=g)
    dV = D.to_colmajor(V, dev)
    dC = D.colmajor_empty(rows, ncols, dev, lda=rows + ld_extra); dC.copy_(Cm)
    nbk = 32 if nbp <= 32 else 128
    dL = torch.zeros(nbk * nbk, dtype=torch.float64, device=dev)
    D._lib.call("dhqr_k_block_reflector_f64", h.raw, rows, nbp, vp(dV), rows, row_lo, ncols, vp(dC), rows + ld_extra, vp(dL), sp())
    torch.cuda.synchronize()
    Vd = V.to(dev); Cd = Cm.to(dev)
    S = Vd.T @ Vd
    L = torch.eye(nbp, dtype=torch.float64, device=dev) + torch.tril(S, -1)
    Linv = torch.linalg.inv(L)
    Y = -Linv @ (Vd.T @ Cd)
    Cexp = Cd + Vd @ Y
    Cexp[:row_lo] = Cd[:row_lo]
    Lg = dL.view(nbk, nbk).T[:nbp, :nbp]      # stored column-major
    eL = float((Lg - Linv).abs().max())
    eC = float((dC - Cexp).abs().max() / Cexp.abs().max())
    return {"ok": eL < 1e-9 and eC < 1e-12, "errLinv": eL, "errC": eC}

for (rows, nbp, ncols, row_lo, ex) in [(256, 32, 64, 0, 0), (1000, 32, 100, 0, 0), (1000, 32, 96, 7, 0), (999, 32, 33, 0, 0),
                                        (999, 32, 33, 0, 1), (512, 128, 128, 0, 0), (4100, 128, 300, 0, 0), (4100, 100, 300, 5, 0),
                                        (4099, 128, 77, 0, 0), (4099, 64, 77, 3, 1), (33000, 128, 1000, 0, 0)]:
    check(f"block_reflector rows={rows} nbp={nbp} ncols={ncols} row_lo={row_lo} ldx={ex}",
          lambda: block_reflector_case(rows, nbp, ncols, row_lo, ex))

def panel_case(rows, ncols, seed=1):
    A = O.np_uniform(seed, rows, ncols)
    Href, aref = O.np_qr(A)
    dP = D.to_colmajor(A, dev)
    dal = torch.zeros(ncols, dtype=torch.float64, device=dev)
    D._lib.call("dhqr_k_panel_f64", h.raw, rows, ncols, vp(dP), rows, vp(dal), sp())
    torch.cuda.synchronize()
    eH = float(np.abs(dP.cpu().numpy() - Href).max()); ea = float(np.abs(dal.cpu().numpy() - aref).max() / np.abs(aref).max())
    return {"ok": eH < 1e-11 and ea < 1e-12, "errH": eH, "errAlpha": ea}

for (rows, ncols) in [(64, 32), (40, 32), (32, 32), (300, 32), (300, 7), (5000, 32), (33000, 32), (65536, 32)]:
    check(f"panel rows={rows} ncols={ncols}", lambda: panel_case(rows, ncols))

def qr_case(m, n, nb=0, seed=0, solve=True):
    A0 = co.fill_uniform(seed, m, n)
    Href = A0.copy(order="F"); Href, aref = co.qr(Href)
    dA = D.colmajor_empty(m, n, dev); D.fill_uniform_(dA, seed)
    H = D.qr_(dA, nb=nb)
    torch.cuda.synchronize()
    Hg = dA.cpu().numpy(); ag = H.α.cpu().numpy()
    out = {"errH": float(np.abs(Hg - Href).max()), "errAlpha": float(np.abs(ag - aref).max() / np.abs(aref).max()),
           "resid": O.qr_residual(A0, np.asfortranarray(Hg), ag)}
    ok = out["errH"] < 1e-10 and out["errAlpha"] < 1e-12 and out["resid"] < 1e-13
    if solve:
        b = O.np_uniform(seed + 1, m, 1)[:, 0].copy()
        x = D.ldiv(H, torch.from_numpy(b).to(dev)).cpu().numpy()
        xr = co.ldiv(Href, aref, b)
        qtb = D.apply_qt_(torch.from_numpy(b).to(dev), dA).cpu().numpy()
        qtr = co.apply_qt(Href, b)
        out["errQtb"] = float(np.linalg.norm(qtb - qtr) / np.linalg.norm(b))
        out["errX"] = float(np.abs(x - xr).max() / np.abs(xr).max())
        out["neq"] = O.normal_eq_residual(A0, x, b); out["neq_lapack"] = O.normal_eq_residual(A0, O.lapack_lstsq(A0, b), b)
        ok = ok and out["errQtb"] < 1e-12 and out["neq"] < 8 * out["neq_lapack"]
    out["ok"] = ok
    return out

for (m, n, nb) in [(110, 100, 0), (64, 64, 0), (1024, 128, 0), (1024, 128, 1), (1000, 37, 0), (1001, 37, 0), (2200, 2000, 0),
                   (2200, 2000, 64), (4400, 4000, 0), (8192, 1024, 0), (8192, 1024, 1)]:
    check(f"qr m={m} n={n} nb={nb}", lambda: qr_case(m, n, nb))

def host_case(m, n):
    A0 = co.fill_uniform(3, m, n)
    Href = A0.copy(order="F"); Href, aref = co.qr(Href)
    A = A0.copy(order="F")
    H = D.qr_(A)
    b = O.np_uniform(4, m, 1)[:, 0].copy()
    x = D.ldiv(H, b); xr = co.ldiv(Href, aref, b)
    return {"ok": np.abs(A - Href).max() < 1e-10 and np.abs(x - xr).max() / np.abs(xr).max() < 1e-9,
            "errH": float(np.abs(A - Href).max()), "errX": float(np.abs(x - xr).max() / np.abs(xr).max())}
check("host path 1024x128", lambda: host_case(1024, 128))
check("host path 1001x37", lambda: host_case(1001, 37))

# ---- timings (sync option off) ----
h.set_option("sync", 0)
def time_qr(m, n, nb=0, reps=3):
    dA = D.colmajor_empty(m, n, dev); al = torch.zeros(n, dtype=torch.float64, device=dev)
    ts = []
    for r in range(reps + 1):
        D.fill_uniform_(dA, 0)
        torch.cuda.synchronize()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        l0 = h.launch_count()
        e0.record(); D.householder_(dA, al, nb); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
        nl = h.launch_count() - l0
    t = min(ts[1:]); fl = 2.0 * m * n * n - 2.0 / 3.0 * n ** 3
    return {"ms": t, "all_ms": ts, "gflops": fl / t / 1e6, "launches": nl}
if "--quick" not in sys.argv:
    for (m, n, nb) in [(8192, 1024, 0), (8192, 1024, 1), (32768, 4096, 0), (32768, 4096, 64)]:
        check(f"time qr m={m} n={n} nb={nb}", lambda: time_qr(m, n, nb))
    def big_resid():
        m, n = 32768, 4096
        dA = D.colmajor_empty(m, n, dev); D.fill_uniform_(dA, 0)
        H = D.qr_(dA)
        # ||QR - A|| / ||A|| on the GPU with torch (size-independent property)
        R = torch.zeros(m, n, dtype=torch.float64, device=dev)
        R[:n] = torch.triu(dA[:n], 1) + torch.diag(H.α)
        for k in range(((n - 1) // 128) * 128, -1, -128):
            V = torch.tril(dA[k:, k:k + 128])
            S = V.T @ V
            Tinv = torch.eye(128, dtype=torch.float64, device=dev) + torch.triu(S, 1)
            R[k:] -= V @ torch.linalg.solve_triangular(Tinv, V.T @ R[k:], upper=True)
        A0 = D.colmajor_empty(m, n, dev); D.fill_uniform_(A0, 0)
        r = float(torch.linalg.norm(R - A0) / torch.linalg.norm(A0))
        return {"ok": r < 1e-13, "resid": r}
    check("resid 32768x4096", big_resid)
    def dgemm_peak():
        n = 8192
        a = torch.rand(n, n, dtype=torch.float64, device=dev); b = torch.rand(n, n, dtype=torch.float64, device=dev)
        torch.matmul(a, b); torch.cuda.synchronize()
        best = 1e9
        for _ in range(5):
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record(); torch.matmul(a, b); e1.record(); torch.cuda.synchronize()
            best = min(best, e0.elapsed_time(e1))
        return {"ms": best, "tflops": 2.0 * n ** 3 / best / 1e9}
    check("cuBLAS dgemm 8192^3 (fp64 peak denominator)", dgemm_peak)
    def geqrf_time():
        m, n = 32768, 4096
        a = torch.rand(m, n, dtype=torch.float64, device=dev)
        torch.geqrf(a); torch.cuda.synchronize()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); torch.geqrf(a); e1.record(); torch.cuda.synchronize()
        t = e0.elapsed_time(e1)
        return {"ms": t, "gflops": (2.0 * m * n * n - 2.0 / 3.0 * n ** 3) / t / 1e6}
    check("cuSOLVER geqrf 32768x4096 (comparator)", geqrf_time)

os.makedirs("build", exist_ok=True)
json.dump(res, open("build/diag.json", "w"), indent=1)
nfail = sum(1 for r in res if not r["ok"])
say(f"SUMMARY: {len(res) - nfail} passed, {nfail} failed")
