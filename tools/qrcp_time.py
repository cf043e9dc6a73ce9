"""Time the pivoted factorisation (qrcp_) against qr_ on the same device-resident matrices, with the per-class profile of qrcp_,
cuBLAS GEMV at the shape of the first F column, launches per column and one host scipy.linalg.qr(pivoting=True).

    python tools/qrcp_time.py [--rounds 3] [--shapes 16384x2048,32768x4096] [--host] [--out build/qrcp_time.json]

Rounds alternate qrcp_ and qr_; the GPU's name, power limit and max SM clock are read in the same run.
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


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError as e:
        return f"nvidia-smi unavailable: {e}"


def timed(fn, src, dst):
    dst.copy_(src)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn(dst)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default="16384x2048,32768x4096")
    ap.add_argument("--out", default="")
    ap.add_argument("--host", action="store_true", help="also time scipy.linalg.qr(pivoting=True) at the first shape")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("qrcp_time.py needs a GPU")
    h = D.default_handle(0)
    res = {"gpu": gpu_info(), "shapes": {}}
    for shp in args.shapes.split(","):
        m, n = map(int, shp.split("x"))
        src = D.colmajor_empty(m, n, "cuda:0")
        D.fill_uniform_(src, 1)
        src.sub_(0.5)
        dst = D.colmajor_empty(m, n, "cuda:0")
        fq = lambda A: D.qrcp_(A, handle=h)
        fr = lambda A: D.qr_(A, handle=h)
        timed(fq, src, dst), timed(fr, src, dst)                      # warm-up: workspace, modules
        l0 = h.launch_count()
        timed(fq, src, dst)
        launches = h.launch_count() - l0
        tq, tr = [], []
        for _ in range(args.rounds):
            tq.append(timed(fq, src, dst))
            tr.append(timed(fr, src, dst))
        h.set_option("profile", 1)
        h.profile_reset()
        timed(fq, src, dst)
        prof = h.profile()
        h.set_option("profile", 0)
        h.profile_reset()
        g = prof.get("k_qrcp_gemv", {"ms": float("nan"), "work": 0.0})
        # cuBLAS GEMV at the step-0 shape: A[0:, 1:]' v
        A1, v = src[:, 1:], src[:, 0].contiguous()
        for _ in range(3):
            torch.mv(A1.T, v)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            torch.mv(A1.T, v)
        e1.record()
        e1.synchronize()
        gemv_ms = e0.elapsed_time(e1) / 20
        floor_bytes = sum(8.0 * (m - j) * (n - j - 1) for j in range(n))          # A[j:, j+1:] read once per column
        r = {"qrcp_ms": tq, "qr_ms": tr, "launches": launches, "launches_per_column": launches / n,
             "profile": {k: {"ms": round(v_["ms"], 3), "count": v_["count"], "work": v_["work"]} for k, v_ in prof.items()},
             "fcol_GBps": g["work"] / (g["ms"] * 1e6) if g["ms"] else None,
             "cublas_gemv_ms": gemv_ms, "cublas_gemv_GBps": 8.0 * m * (n - 1) / (gemv_ms * 1e6),
             "fcol_floor_bytes": floor_bytes}
        r["fcol_floor_ms_at_measured_rate"] = floor_bytes / (r["fcol_GBps"] * 1e6) if r["fcol_GBps"] else None
        res["shapes"][shp] = r
        print(shp, json.dumps({k: v_ for k, v_ in r.items() if k != "profile"}), flush=True)
        print("  profile:", json.dumps(r["profile"]), flush=True)
    if args.host:
        import scipy.linalg
        m, n = map(int, args.shapes.split(",")[0].split("x"))
        a = np.asfortranarray(np.random.default_rng(1).random((m, n)) - 0.5)
        t0 = time.perf_counter()
        scipy.linalg.qr(a, mode="r", pivoting=True)
        res["scipy_host_s"] = time.perf_counter() - t0
        print("scipy.linalg.qr(pivoting=True)", f"{m}x{n}", res["scipy_host_s"], "s", flush=True)
    res["gpu_after"] = gpu_info()
    print(res["gpu"])
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
