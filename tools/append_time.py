"""Time folding new rows into a factorisation (dhqr_qr_append_f64, DESIGN §2.10) against factoring the stacked matrix again, and the
streaming least-squares solve of a system taller than qr_'s row limit.

    python tools/append_time.py [--rounds 3] [--json OUT] [--skip-stream]

Appends: n in {1024, 4096}, k in {64, 512, 4096, 32768}, R the triangle of a 32768 x n factorisation, B uniform random.  Beside each,
in the same run: dhqr_qr_f64 and torch.linalg.qr on the stacked (32768 + k) x n matrix.  Reported: CUDA-event median of `rounds`
calls (inputs refilled outside the timed region), TFLOP/s of the append's 2 k n^2 flops, launches per append.  Stream: 1048576 x
1024 in blocks of 65536 rows from pinned host memory through StreamingLeastSquares, wall time to the solution on the device, beside
torch.linalg.lstsq on the device-resident matrix.  The GPU's name, power limit and max SM clock are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import dhqr_b200 as D  # noqa: E402


def gpu_info():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        info["nvidia-smi"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["nvidia-smi"] = f"unavailable ({e})"
    return info


def timed(fn, prep):
    ts = []
    for _ in range(ROUNDS):
        prep()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def append_case(h, m0, n, k):
    S0 = D.colmajor_empty(m0 + k, n, "cuda")
    D.fill_uniform_(S0, 1, handle=h)
    A = S0[:m0].clone()
    st = D.qr_(A, handle=h)
    R0, a0 = A[:n].clone(), st.α.clone()
    B = D.colmajor_empty(k, n, "cuda")
    S = D.colmajor_empty(m0 + k, n, "cuda")
    Ad = D.colmajor_empty(n, n, "cuda")
    al = torch.empty_like(a0)
    Srow = S0.contiguous()

    def prep_append():
        Ad.copy_(R0)
        al.copy_(a0)
        B.copy_(S0[m0:])

    l0 = h.launch_count()
    prep_append()
    D.append_rows_((Ad, al), B, handle=h)
    launches = h.launch_count() - l0
    out = {"n": n, "k": k, "launches": launches}
    out["append_ms"] = timed(lambda: D.append_rows_((Ad, al), B, handle=h), prep_append)
    out["append_tflops"] = 2.0 * k * n * n / (out["append_ms"] * 1e-3) / 1e12
    out["qr_stacked_ms"] = timed(lambda: D.qr_(S, handle=h), lambda: S.copy_(S0))
    out["torch_qr_stacked_ms"] = timed(lambda: torch.linalg.qr(Srow, mode="r"), lambda: None)
    del S0, A, B, S, Srow
    torch.cuda.empty_cache()
    return out


def stream_case(h, m, n, blk):
    ls_ms, lstsq_ms = [], []
    Ah = torch.empty((m // blk, blk, n), dtype=torch.float64).pin_memory()
    bh = torch.empty((m // blk, blk, 1), dtype=torch.float64).pin_memory()
    g = torch.Generator().manual_seed(0)
    for i in range(m // blk):
        Ah[i].copy_(torch.rand((blk, n), generator=g, dtype=torch.float64))
        bh[i].copy_(torch.rand((blk, 1), generator=g, dtype=torch.float64))
    for _ in range(ROUNDS):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ls = D.StreamingLeastSquares(n, 1, device=0, handle=h)
        for i in range(m // blk):
            ls.add(Ah[i], bh[i])
        x = ls.solve()
        torch.cuda.synchronize()
        ls_ms.append((time.perf_counter() - t0) * 1e3)
    Ad = Ah.reshape(m, n).to("cuda")
    bd = bh.reshape(m, 1).to("cuda")
    for _ in range(ROUNDS):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        xl = torch.linalg.lstsq(Ad, bd).solution
        torch.cuda.synchronize()
        lstsq_ms.append((time.perf_counter() - t0) * 1e3)
    dx = float((x - xl[:, 0]).norm() / xl.norm())
    return {"m": m, "n": n, "block": blk, "stream_ms": float(np.median(ls_ms)), "torch_lstsq_ms": float(np.median(lstsq_ms)),
            "rel_diff_x": dx, "residual": float(ls.residual_norm()[0])}


def main():
    global ROUNDS
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    ap.add_argument("--skip-stream", action="store_true")
    args = ap.parse_args()
    ROUNDS = args.rounds
    h = D.Handle(0)
    res = {"gpu": gpu_info(), "append": []}
    print(json.dumps(res["gpu"]), flush=True)
    for n in (1024, 4096):
        for k in (64, 512, 4096, 32768):
            r = append_case(h, 32768, n, k)
            res["append"].append(r)
            print(f"n={n:5d} k={k:6d}: append {r['append_ms']:8.2f} ms ({r['append_tflops']:5.2f} TFLOP/s, {r['launches']} launches)"
                  f"  qr_ stacked {r['qr_stacked_ms']:8.2f} ms  torch.linalg.qr stacked {r['torch_qr_stacked_ms']:8.2f} ms", flush=True)
    if not args.skip_stream:
        r = stream_case(h, 1 << 20, 1024, 65536)
        res["stream"] = r
        print(f"stream {r['m']} x {r['n']} in blocks of {r['block']} from pinned host memory: {r['stream_ms']:.1f} ms; "
              f"torch.linalg.lstsq on the device {r['torch_lstsq_ms']:.1f} ms; |dx|/|x| {r['rel_diff_x']:.2e}", flush=True)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)
    h.close()


ROUNDS = 3
if __name__ == "__main__":
    main()
