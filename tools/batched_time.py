"""Time the batched QR and its fused least-squares solve (dhqr_qr_batched_f64, dhqr_solve_batched_f64; DESIGN §2.12) against
torch.geqrf and torch.linalg.lstsq(driver="gels") on the same batch, and against a loop of dhqr_qr_f64 over single problems.

    python tools/batched_time.py [--rounds 5] [--json OUT]

Shapes (batch x (m x n)): 100 000 x (8 x 4), 10 000 x (64 x 16), 10 000 x (256 x 32), 2 000 x (128 x 128), 1 000 x (1024 x 24),
200 x (4096 x 48): from tiny problems on one CTA to the cluster of 8.  Each round times every method once, in turn (interleaved
rounds), with the inputs refilled outside the timed region; reported are the CUDA-event medians over the rounds.  The dhqr_qr_f64
loop runs over the first 100 problems (nb = 0, the blocked path, and nb = 1, the column loop) and is scaled to the whole batch;
it is labelled as such.  Rates: TFLOP/s of 2 m n^2 - 2 n^3 / 3 per problem, and HBM GB/s of 16 m n bytes per problem (A read
and written once) against the data sheet's 3.35 TB/s; the nearer bound is named.  The GPU's name, power limit and max SM clock
are read in the same run.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dhqr_b200 as D  # noqa: E402
from append_time import gpu_info  # noqa: E402

SHAPES = ((100_000, 8, 4), (10_000, 64, 16), (10_000, 256, 32), (2_000, 128, 128), (1_000, 1024, 24), (200, 4096, 48))
LOOP = 100
HBM_GBS = 3350.0
FP64_TFLOPS = 34.0     # H100 SXM data sheet, FP64 on CUDA cores, where the batched kernels compute (tensor cores: 67)


def event_ms(fn, prep):
    prep()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def case(h, nb, m, n, rounds):
    g = torch.Generator(device="cuda").manual_seed(m * 7 + n)
    M = torch.randn(nb, m, n, device="cuda", dtype=torch.float64, generator=g)
    bb = torch.randn(nb, m, 1, device="cuda", dtype=torch.float64, generator=g)
    A = D.colmajor_empty_batched(nb, m, n, "cuda")
    Ms = M.clone()                                          # torch's own (row-major batch) copy, refilled per round
    b = D.colmajor_empty_batched(nb, m, 1, "cuda")
    A.copy_(M)
    st = D.qr_batched_(A, handle=h)
    F0, al = A.clone(), st.α
    singles = [D.colmajor_empty(m, n, "cuda") for _ in range(LOOP)]
    alphas = torch.empty(LOOP, n, dtype=torch.float64, device="cuda")

    def prep_qr():
        A.copy_(M)

    def prep_solve():
        A.copy_(F0)
        b.copy_(bb)

    def prep_torch():
        Ms.copy_(M)

    def prep_loop():
        for i in range(LOOP):
            singles[i].copy_(M[i])

    def loop(nbk):
        def run():
            for i in range(LOOP):
                D.householder_(singles[i], alphas[i], nb=nbk, handle=h)
        return run

    l0 = h.launch_count()
    D.qr_batched_(A, handle=h)
    launches_qr = h.launch_count() - l0
    methods = {
        "qr_batched": (lambda: D.qr_batched_(A, handle=h), prep_qr),
        "solve_batched": (lambda: D.solve_batched_(b, A, al, handle=h), prep_solve),
        "torch.geqrf": (lambda: torch.geqrf(Ms), prep_torch),
        "torch.lstsq_gels": (lambda: torch.linalg.lstsq(Ms, bb, driver="gels"), prep_torch),
        f"qr_f64 nb=0 loop x{LOOP}": (loop(0), prep_loop),
        f"qr_f64 nb=1 loop x{LOOP}": (loop(1), prep_loop),
    }
    for fn, prep in methods.values():                       # warm-up: module load, library algorithm choice, workspace
        event_ms(fn, prep)
    times = {k: [] for k in methods}
    for _ in range(rounds):
        for k, (fn, prep) in methods.items():
            times[k].append(event_ms(fn, prep))
    med = {k: float(np.median(v)) for k, v in times.items()}
    for k in list(med):
        if "loop" in k:
            med[k + " scaled to batch"] = med[k] * nb / LOOP
    flops = nb * (2.0 * m * n * n - 2.0 * n ** 3 / 3.0)
    bytes_ = nb * 16.0 * m * n
    t = med["qr_batched"] * 1e-3
    tf, gbs = flops / t / 1e12, bytes_ / t / 1e9
    return {"batch": nb, "m": m, "n": n, "ms": med, "launches_qr_batched": launches_qr,
            "qr_batched_tflops": tf, "qr_batched_hbm_gbs": gbs, "hbm_share": gbs / HBM_GBS, "fp64_share": tf / FP64_TFLOPS,
            "nearer_bound": "HBM" if bytes_ / (HBM_GBS * 1e9) > flops / (FP64_TFLOPS * 1e12) else "FP64"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("batched_time.py needs a GPU: it times CUDA kernels and has nothing to measure without one")
    h = D.Handle(0)
    out = {"gpu": gpu_info(), "rounds": args.rounds, "cases": []}
    print(json.dumps(out["gpu"]))
    for nb, m, n in SHAPES:
        r = case(h, nb, m, n, args.rounds)
        out["cases"].append(r)
        ms = "  ".join(f"{k} {v:.3f}" for k, v in r["ms"].items())
        print(f"{nb} x ({m} x {n}): {ms} ms | qr_batched {r['qr_batched_tflops']:.2f} TFLOP/s, {r['qr_batched_hbm_gbs']:.0f} GB/s "
              f"({100 * r['hbm_share']:.1f} % of 3.35 TB/s); nearer bound {r['nearer_bound']}", flush=True)
        torch.cuda.empty_cache()
    torch.cuda.synchronize()
    h.close()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
