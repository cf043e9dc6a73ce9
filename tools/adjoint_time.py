"""Time the solves with the adjoint against the back-substitution and against torch's routes, on a factorisation computed once.

    python tools/adjoint_time.py [--rounds 9] [--json OUT]

Float64 32768 x 4096 and ComplexF64 8192 x 2048, one right-hand side unless named.  Each round runs, one after the other:
  fwd_wave / bwd_wave   forwardsolve_ / backsolve_ with "bs_wave" = 1 (Float64 only: the complex solves have no wavefront)
  fwd_step / bwd_step   the same with "bs_wave" = 0 (the per-block launches)
  solve_adj_1 / _16     solve_adjoint_ (y = Q [R^{-H} c; 0]) with 1 and 16 right-hand sides
  torch_form_q          torch.linalg.solve_triangular on R (formed once outside the timed region), form_q, Q @ z
  torch_ormqr           solve_triangular on R from torch.geqrf (factored once outside), then torch.ormqr on [z; 0]
Right-hand sides are refilled outside the timed region.  Reported: CUDA-event median / min / max per method, max |dy| between
the routes to y, the ratio fwd_wave / bwd_wave, and the GPU's name, power limit and max SM clock read in the same run.
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
    rnd = lambda *s: torch.rand(*s, dtype=torch.float64, device="cuda", generator=g)
    A0 = D.colmajor_empty(m, n, "cuda", dtype=dt)
    A0.copy_(torch.complex(rnd(m, n), rnd(m, n)) if cplx else rnd(m, n))
    A = A0.clone()
    H = D.qr_(A, handle=h)
    alpha = H.α
    R = D.form_r(A, alpha)
    a_t, tau = torch.geqrf(A0)
    R_t = torch.triu(a_t[:n])
    del A0
    c1 = (torch.complex(rnd(n), rnd(n)) if cplx else rnd(n)) - 0.5
    c16 = D.colmajor_empty(n, 16, "cuda", dtype=dt)
    c16.copy_((torch.complex(rnd(n, 16), rnd(n, 16)) if cplx else rnd(n, 16)) - 0.5)
    b1 = torch.zeros(m, dtype=dt, device="cuda")
    b16 = D.colmajor_empty(m, 16, "cuda", dtype=dt)
    Y = torch.zeros(m, 1, dtype=dt, device="cuda")

    def fill1():
        b1.zero_()
        b1[:n] = c1

    def fill16():
        b16.zero_()
        b16[:n] = c16

    def wave(v, fill):
        return lambda: (h.set_option("bs_wave", v), fill())

    def form_q_route():
        z = torch.linalg.solve_triangular(R.mH, c1[:, None], upper=False)
        return (D.form_q(A, handle=h) @ z)[:, 0]

    def ormqr_route():
        Y[:n] = torch.linalg.solve_triangular(R_t.mH, c1[:, None], upper=False)
        Y[n:] = 0
        return torch.ormqr(a_t, tau, Y, left=True, transpose=False)[:, 0]

    methods = {}
    if not cplx:
        methods["fwd_wave"] = (lambda: D.forwardsolve_(b1, A, alpha, handle=h), wave(1, fill1))
        methods["bwd_wave"] = (lambda: D.backsolve_(b1, A, alpha, handle=h), wave(1, fill1))
    methods["fwd_step"] = (lambda: D.forwardsolve_(b1, A, alpha, handle=h), wave(0, fill1))
    methods["bwd_step"] = (lambda: D.backsolve_(b1, A, alpha, handle=h), wave(0, fill1))
    methods["solve_adj_1"] = (lambda: D.solve_adjoint_(b1, A, alpha, handle=h).clone(), wave(1, fill1))
    methods["solve_adj_16"] = (lambda: D.solve_adjoint_(b16, A, alpha, handle=h), wave(1, fill16))
    methods["torch_form_q"] = (form_q_route, None)
    methods["torch_ormqr"] = (ormqr_route, None)
    times = {k: [] for k in methods}
    outs = {}
    for k, (fn, prep) in methods.items():              # warm-up: workspace, module loads, cuSOLVER's own set-up
        timed(fn, prep)
    for _ in range(rounds):
        for k, (fn, prep) in methods.items():
            ms, out = timed(fn, prep)
            times[k].append(ms)
            if k in ("solve_adj_1", "torch_form_q", "torch_ormqr"):
                outs[k] = out.clone()
    h.set_option("bs_wave", 1)
    res = {"shape": f"{m}x{n}", "dtype": "ComplexF64" if cplx else "Float64", "rounds": rounds, "methods": {}}
    for k, t in times.items():
        res["methods"][k] = {"median_ms": float(np.median(t)), "min_ms": float(min(t)), "max_ms": float(max(t))}
    keys = list(outs)
    res["max_abs_dy"] = {f"{a} vs {b}": float((outs[a] - outs[b]).abs().max()) for i, a in enumerate(keys) for b in keys[i + 1:]}
    if not cplx:
        res["fwd_over_bwd_wave"] = res["methods"]["fwd_wave"]["median_ms"] / res["methods"]["bwd_wave"]["median_ms"]
    del A, H, alpha, R, a_t, tau, R_t, b1, b16, Y, outs
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("adjoint_time.py needs a CUDA device")
    h = D.Handle(0)
    out = {"gpu": gpu_info(), "cases": [run_case(h, 32768, 4096, False, args.rounds), run_case(h, 8192, 2048, True, args.rounds)]}
    torch.cuda.synchronize()
    h.close()
    print(f"GPU: {out['gpu']['name']} ({out['gpu']['nvidia-smi']})")
    for c in out["cases"]:
        print(f"{c['dtype']} {c['shape']}, {c['rounds']} alternated rounds")
        for k, r in c["methods"].items():
            print(f"  {k:13s} median {r['median_ms']:8.3f} ms  (min {r['min_ms']:.3f}, max {r['max_ms']:.3f})")
        for k, v in c["max_abs_dy"].items():
            print(f"  max|dy| {k}: {v:.2e}")
        if "fwd_over_bwd_wave" in c:
            print(f"  fwd_wave / bwd_wave = {c['fwd_over_bwd_wave']:.2f}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
