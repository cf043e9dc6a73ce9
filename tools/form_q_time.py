"""Time the explicit thin Q (form_q) against the two ways to get it without it, on device-resident inputs factored once.

    python tools/form_q_time.py [--rounds 7] [--json OUT]

Float64 32768 x 4096 and ComplexF64 8192 x 2048.  Each round runs, one after the other:
  form_q      dhqr_form_q_* (the structured backward sweep)
  apply_q     dhqr_apply_q_f64 on an explicit [I; 0] (Float64 only; the identity is refilled outside the timed region)
  cusolver    torch.linalg.householder_product on the LAPACK form of the same reflectors (u_j = v_j / v_jj, tau_j = |v_jj|^2,
              converted once outside the timed region)
Reported: CUDA-event median / min / max per method, TFLOP/s from 2mn^2 - 2n^3/3 (x4 real flops per complex one), max |dQ|
between the results, and the GPU's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import dhqr_b200 as D  # noqa: E402


def gpu_info():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["nvidia-smi"] = out
    except (OSError, subprocess.SubprocessError) as e:
        info["nvidia-smi"] = f"unavailable ({e})"
    return info


def timed(fn, prep=None):
    if prep is not None:
        prep()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1), out


def run_case(h, m, n, cplx, rounds):
    dt = torch.complex128 if cplx else torch.float64
    g = torch.Generator(device="cuda").manual_seed(1)
    A = D.colmajor_empty(m, n, "cuda", dtype=dt)
    if cplx:
        A.copy_(torch.complex(torch.rand(m, n, dtype=torch.float64, device="cuda", generator=g),
                              torch.rand(m, n, dtype=torch.float64, device="cuda", generator=g)))
    else:
        A.copy_(torch.rand(m, n, dtype=torch.float64, device="cuda", generator=g))
    D.qr_(A, handle=h)
    d = torch.diagonal(A)
    U = torch.tril(A, -1) / d + torch.eye(m, n, dtype=dt, device="cuda")
    tau = (d.abs() ** 2).to(dt)
    Q = D.colmajor_empty(m, n, "cuda", dtype=dt)
    eye = torch.eye(m, n, dtype=dt, device="cuda")
    E = D.colmajor_empty(m, n, "cuda", dtype=dt)
    methods = {"form_q": (lambda: D.form_q(A, out=Q, handle=h), None),
               "cusolver": (lambda: torch.linalg.householder_product(U, tau), None)}
    if not cplx:
        methods["apply_q"] = (lambda: D.apply_q_(E, A, handle=h), lambda: E.copy_(eye))
    times = {k: [] for k in methods}
    outs = {}
    for k, (fn, prep) in methods.items():              # warm-up: workspace, module loads, cuSOLVER's own setup
        timed(fn, prep)
    for _ in range(rounds):
        for k, (fn, prep) in methods.items():
            ms, outs[k] = timed(fn, prep)
            times[k].append(ms)
    flops = (2.0 * m * n * n - 2.0 * n ** 3 / 3.0) * (4.0 if cplx else 1.0)
    res = {"shape": f"{m}x{n}", "dtype": "ComplexF64" if cplx else "Float64", "rounds": rounds, "flops": flops, "methods": {}}
    for k, t in times.items():
        med = float(np.median(t))
        res["methods"][k] = {"median_ms": med, "min_ms": float(min(t)), "max_ms": float(max(t)), "tflops": flops / med / 1e9}
    keys = list(outs)
    res["max_abs_dQ"] = {f"{a} vs {b}": float((outs[a] - outs[b]).abs().max()) for i, a in enumerate(keys) for b in keys[i + 1:]}
    del A, U, tau, Q, E, eye, outs
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("form_q_time.py needs a CUDA device")
    h = D.Handle(0)
    out = {"gpu": gpu_info(), "cases": [run_case(h, 32768, 4096, False, args.rounds), run_case(h, 8192, 2048, True, args.rounds)]}
    torch.cuda.synchronize()
    h.close()
    print(f"GPU: {out['gpu']['name']} ({out['gpu']['nvidia-smi']})")
    for c in out["cases"]:
        print(f"{c['dtype']} {c['shape']}, {c['rounds']} alternated rounds, {c['flops']:.3e} flops")
        for k, r in c["methods"].items():
            print(f"  {k:9s} median {r['median_ms']:8.2f} ms  (min {r['min_ms']:.2f}, max {r['max_ms']:.2f})  {r['tflops']:6.2f} TFLOP/s")
        for k, v in c["max_abs_dQ"].items():
            print(f"  max|dQ| {k}: {v:.2e}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
