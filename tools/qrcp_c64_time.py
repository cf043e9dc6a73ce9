"""Time the ComplexF64 pivoted factorisation (qrcp_ on complex128) against qr_ on the same device-resident matrices and against the
Float64 qrcp_ at the same shape, in alternated rounds; cod_ and solve_cod_ at rank n and n/2; the per-class profile of the complex
qrcp_ with the GEMV class's rate from algorithmic bytes; cuBLAS ZGEMV (A^H v in torch) at the step-0 shape in the same run;
launches per column; one host scipy.linalg.qr(pivoting=True).

    python tools/qrcp_c64_time.py [--rounds 3] [--shapes 8192x1024,16384x2048] [--host] [--out build/qrcp_c64_time.json]

The GPU's name, power limit and max SM clock are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import dhqr_b200 as D  # noqa: E402

QP_NB = 32


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError as e:
        return f"nvidia-smi unavailable: {e}"


def ev_time(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def timed(fn, src, dst):
    dst.copy_(src)
    return ev_time(lambda: fn(dst))


def gemv_bytes(m, n):
    """Algorithmic bytes of the complex F-column GEMV: A[j:, k0(j):n] read once per column j, 16 B per element."""
    return sum(16.0 * (m - j) * (n - (j // QP_NB) * QP_NB) for j in range(n))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default="8192x1024,16384x2048")
    ap.add_argument("--out", default="")
    ap.add_argument("--host", action="store_true", help="also time scipy.linalg.qr(pivoting=True) on complex input at the first shape")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("qrcp_c64_time.py needs a GPU")
    h = D.default_handle(0)
    res = {"gpu": gpu_info(), "shapes": {}}
    for shp in args.shapes.split(","):
        m, n = map(int, shp.split("x"))
        re_, im_ = D.colmajor_empty(m, n, "cuda:0"), D.colmajor_empty(m, n, "cuda:0")
        D.fill_uniform_(re_, 1)
        D.fill_uniform_(im_, 2)
        src = D.colmajor_empty(m, n, "cuda:0", dtype=torch.complex128)
        src.copy_(torch.complex(re_ - 0.5, im_ - 0.5))
        srcf = re_.sub_(0.5)
        dst = D.colmajor_empty(m, n, "cuda:0", dtype=torch.complex128)
        dstf = D.colmajor_empty(m, n, "cuda:0")
        fq = lambda A: D.qrcp_(A, handle=h)
        fr = lambda A: D.qr_(A, handle=h)
        timed(fq, src, dst), timed(fr, src, dst), timed(fq, srcf, dstf)              # warm-up: workspace, modules
        l0 = h.launch_count()
        timed(fq, src, dst)
        launches = h.launch_count() - l0
        tq, tr, tf = [], [], []
        for _ in range(args.rounds):
            tq.append(timed(fq, src, dst))
            tr.append(timed(fr, src, dst))
            tf.append(timed(fq, srcf, dstf))
        # cod_ and solve_cod_ at rank n and n/2 on the complex factorisation
        dst.copy_(src)
        st = D.qrcp_(dst, handle=h)
        b0 = D.colmajor_empty(m, 1, "cuda:0", dtype=torch.complex128)
        b0.copy_(src[:, :1] * 0.5 + 1.0)
        b = b0.clone()
        cod = {}
        for r in (n, n // 2):
            D.cod_(st.A, st.α, r, handle=h)
            Fd, gd = D.cod_(st.A, st.α, r, handle=h)
            tc = [ev_time(lambda: D.cod_(st.A, st.α, r, handle=h)) for _ in range(args.rounds)]
            ts = []
            for _ in range(args.rounds + 1):
                b.copy_(b0)
                ts.append(ev_time(lambda: D.solve_cod_(b, st.A, st.p, Fd, gd, r, handle=h)))
            cod[r] = {"cod_ms": tc, "solve_cod_ms": ts[1:]}
        h.set_option("profile", 1)
        h.profile_reset()
        timed(fq, src, dst)
        prof = h.profile()
        h.set_option("profile", 0)
        h.profile_reset()
        g = prof.get("k_qrcp_gemv_c", {"ms": float("nan"), "work": 0.0})
        # cuBLAS ZGEMV at the step-0 shape: A[0:, 1:]^H v
        A1, v = src[:, 1:], src[:, 0].contiguous()
        for _ in range(3):
            A1.mH @ v
        torch.cuda.synchronize()
        gemv_ms = ev_time(lambda: [A1.mH @ v for _ in range(20)]) / 20
        r = {"qrcp_c64_ms": tq, "qr_c64_ms": tr, "qrcp_f64_ms": tf, "launches": launches, "launches_per_column": launches / n,
             "cod": cod,
             "profile": {k: {"ms": round(v_["ms"], 3), "count": v_["count"], "work": v_["work"]} for k, v_ in prof.items()},
             "gemv_c_bytes": gemv_bytes(m, n), "gemv_c_GBps": g["work"] / (g["ms"] * 1e6) if g["ms"] else None,
             "cublas_zgemv_ms": gemv_ms, "cublas_zgemv_GBps": 16.0 * m * (n - 1) / (gemv_ms * 1e6)}
        r["gemv_c_vs_cublas"] = r["gemv_c_GBps"] / r["cublas_zgemv_GBps"] if r["gemv_c_GBps"] else None
        res["shapes"][shp] = r
        print(shp, json.dumps({k: v_ for k, v_ in r.items() if k != "profile"}), flush=True)
        print("  profile:", json.dumps(r["profile"]), flush=True)
    if args.host:
        import scipy.linalg
        m, n = map(int, args.shapes.split(",")[0].split("x"))
        g = np.random.default_rng(1)
        a = np.asfortranarray(g.random((m, n)) - 0.5 + 1j * (g.random((m, n)) - 0.5))
        t0 = time.perf_counter()
        scipy.linalg.qr(a, mode="r", pivoting=True)
        res["scipy_host_s"] = time.perf_counter() - t0
        print("scipy.linalg.qr(pivoting=True) complex", f"{m}x{n}", res["scipy_host_s"], "s", flush=True)
    res["gpu_after"] = gpu_info()
    print(res["gpu"])
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
