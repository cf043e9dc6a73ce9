"""Time the complete orthogonal decomposition on the pivoted QR (DESIGN §2.8) against the pivoted factorisation it follows and the
basic solution it replaces.

    python tools/cod_time.py [--rounds 5] [--json OUT]

Float64 32768 x 4096 and 16384 x 2048 (uniform random, so the rank is chosen, not revealed), at ranks n, n - 96, n / 2 and 128.
Each round runs, one after the other: qrcp_ on a fresh copy of the matrix; then for every rank cod_, solve_cod_ and solve_qrcp_
with 1 and 16 right-hand sides (refilled outside the timed region).  Reported: CUDA-event median / min / max per method, cod_ as a
share of qrcp_, a per-class profile of one cod_ at every rank (option "profile", in a pass of its own), and the GPU's name, power
limit and max SM clock read in the same run.
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
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1), out


def run_case(h, m, n, rounds):
    ranks = [n, n - 96, n // 2, 128]
    A0 = D.colmajor_empty(m, n, "cuda")
    D.fill_uniform_(A0, 1, handle=h)
    A = A0.clone()
    B1, B16 = D.colmajor_empty(m, 1, "cuda"), D.colmajor_empty(m, 16, "cuda")
    D.fill_uniform_(B1, 2, handle=h)
    D.fill_uniform_(B16, 3, handle=h)
    b1, b16 = B1[:, 0].clone(), B16.clone()
    st = {}

    def factor():
        st["s"] = D.qrcp_(A, handle=h)

    def refill_a():
        A.copy_(A0)

    methods = {"qrcp": (factor, refill_a)}
    fac = {}
    for r in ranks:
        methods[f"cod_r{r}"] = (lambda r=r: fac.__setitem__(r, D.cod_(st["s"].A, st["s"].α, r, handle=h)), None)
        for k, b, B in ((1, b1, B1[:, 0]), (16, b16, B16)):
            fill = (lambda b=b, B=B: b.copy_(B))
            methods[f"solve_cod_r{r}_nrhs{k}"] = (lambda r=r, b=b: D.solve_cod_(b, st["s"].A, st["s"].p, *fac[r], r, handle=h), fill)
            methods[f"solve_qrcp_r{r}_nrhs{k}"] = (lambda r=r, b=b: D.solve_qrcp_(b, st["s"].A, st["s"].α, st["s"].p, r, handle=h), fill)
    times = {k: [] for k in methods}
    for k, (fn, prep) in methods.items():              # warm-up: workspace growth, module loads
        timed(fn, prep)
    for _ in range(rounds):
        for k, (fn, prep) in methods.items():
            ms, _ = timed(fn, prep)
            times[k].append(ms)
    res = {"shape": f"{m}x{n}", "rounds": rounds, "ranks": ranks, "methods": {}}
    for k, t in times.items():
        res["methods"][k] = {"median_ms": float(np.median(t)), "min_ms": float(min(t)), "max_ms": float(max(t))}
    q = res["methods"]["qrcp"]["median_ms"]
    res["cod_over_qrcp"] = {f"r{r}": res["methods"][f"cod_r{r}"]["median_ms"] / q for r in ranks}
    # per-class profile of one cod_ at every rank, in a pass of its own (the brackets serialise the schedule)
    res["cod_profile"] = {}
    h.set_option("profile", 1)
    try:
        for r in ranks:
            torch.cuda.synchronize()
            h.profile_reset()
            D.cod_(st["s"].A, st["s"].α, r, handle=h)
            torch.cuda.synchronize()
            prof = h.profile()
            res["cod_profile"][f"r{r}"] = {k: {"ms": v["ms"], "count": v["count"]} for k, v in prof.items() if v["count"]}
    finally:
        h.set_option("profile", 0)
        h.profile_reset()
    res["wide_panels"], res["wide_redone"] = h.get_option("wide_panels"), h.get_option("wide_redone")
    del A, A0, B1, B16, b1, b16, st, fac
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("cod_time.py needs a GPU")
    h = D.Handle(0)
    out = {"gpu": gpu_info(), "cases": []}
    try:
        for m, n in ((32768, 4096), (16384, 2048)):
            out["cases"].append(run_case(h, m, n, args.rounds))
    finally:
        h.close()
    out["gpu_after"] = gpu_info()
    text = json.dumps(out, indent=1)
    print(text)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
