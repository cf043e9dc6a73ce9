"""Time one slide of a rolling least-squares window over many independent problems (BatchedStreamingLeastSquares: add the newest k
rows, remove the oldest k, solve; DESIGN §2.13) against refactoring every window from scratch.

    python tools/rolling_time.py [--rounds 5] [--json OUT]

Workloads (batch x (n unknowns, window w rows, step k rows)): 100 000 x (4, 64, 1), 10 000 x (8, 256, 1), 1 000 x (32, 1024, 16) and
200 x (128, 4096, 64), on both sides of the expected crossover (the update pays 2 n column steps of k rows per slide, a refactor
n column steps of w rows).  Methods, each timed with CUDA events around one whole slide, in interleaved rounds after a warm-up
slide; reported are the medians over the rounds:
  rolling update       BatchedStreamingLeastSquares.add + .remove + .solve (three library launches and their torch copies)
  qr_batched refactor  the window copied into column-major storage, qr_batched_ and solve_batched_ (only where w n fits
                       batch_max_elems; the last workload is above it)
  torch.lstsq_gels     torch.linalg.lstsq(driver="gels") on the (batch, w, n) windows
  StreamingLeastSquares loop  the single-problem solver's slide looped over the first 100 problems (its remove reads the downdate
                       status, one synchronisation per problem), scaled to the batch and labelled as such
Every method slides over the same seeded row stream, so all solve the same windows.  The GPU's name, power limit and max SM clock
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

WORKLOADS = ((100_000, 4, 64, 1), (10_000, 8, 256, 1), (1_000, 32, 1024, 16), (200, 128, 4096, 64))
LOOP = 100


def timed(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def case(h, nb, n, w, k, rounds):
    slides = rounds + 1
    g = torch.Generator(device="cuda").manual_seed(n * 1000 + w)
    T = w + k * slides
    A = torch.randn(nb, T, n, dtype=torch.float64, device="cuda", generator=g)
    b = torch.randn(nb, T, dtype=torch.float64, device="cuda", generator=g)
    fits = w * n <= h.get_option("batch_max_elems")
    ls = D.BatchedStreamingLeastSquares(nb, n, handle=h)
    ls.add(A[:, :w], b[:, :w])
    singles = []
    for i in range(LOOP):
        s = D.StreamingLeastSquares(n, handle=h)
        s.add(A[i, :w], b[i, :w])
        singles.append(s)
    Aw = D.colmajor_empty_batched(nb, w, n, "cuda") if fits else None
    bw = D.colmajor_empty_batched(nb, w, 1, "cuda") if fits else None
    state = {"s": 0}

    def window(s):
        return slice(k * (s + 1), w + k * (s + 1))

    def rolling():
        s = state["s"]
        lo, hi = k * s, w + k * s
        ls.add(A[:, hi:hi + k], b[:, hi:hi + k])
        ls.remove(A[:, lo:lo + k], b[:, lo:lo + k])
        return ls.solve()

    def refactor():
        r = window(state["s"])
        Aw.copy_(A[:, r])
        bw.copy_(b[:, r, None])
        st = D.qr_batched_(Aw, handle=h)
        D.solve_batched_(bw, Aw, st.α, handle=h)
        return bw[:, :n, 0]

    def gels():
        r = window(state["s"])
        return torch.linalg.lstsq(A[:, r], b[:, r, None], driver="gels").solution[..., 0]

    def loop():
        s = state["s"]
        lo, hi = k * s, w + k * s
        for i, sl in enumerate(singles):
            sl.add(A[i, hi:hi + k], b[i, hi:hi + k])
            sl.remove(A[i, lo:lo + k], b[i, lo:lo + k])
            sl.solve()

    methods = {"rolling update": rolling, "torch.lstsq_gels": gels, f"StreamingLeastSquares loop x{LOOP}": loop}
    if fits:
        methods["qr_batched refactor"] = refactor
    times = {key: [] for key in methods}
    worst = 0.0
    for s in range(slides):                 # slide 0 is the warm-up; every method moves over the same windows
        state["s"] = s
        for key, fn in methods.items():
            t = timed(fn)
            if s > 0:
                times[key].append(t)
        x = ls.solve()
        xl = gels()
        worst = max(worst, ((x - xl).norm(dim=1) / xl.norm(dim=1)).max().item())
    med = {key: float(np.median(v)) for key, v in times.items()}
    med[f"StreamingLeastSquares loop x{LOOP} scaled to batch"] = med[f"StreamingLeastSquares loop x{LOOP}"] * nb / LOOP
    l0 = h.launch_count()
    ls.add(A[:, :k], b[:, :k])
    ls.remove(A[:, :k], b[:, :k])
    ls.solve()
    return {"batch": nb, "n": n, "w": w, "k": k, "ms": med, "refactor_fits": fits, "launches_per_slide": h.launch_count() - l0,
            "rolling_vs_lstsq_max_rel": worst}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rolling_time.py needs a GPU: it times CUDA kernels and has nothing to measure without one")
    h = D.Handle(0)
    out = {"gpu": gpu_info(), "rounds": args.rounds, "cases": []}
    print(json.dumps(out["gpu"]))
    for nb, n, w, k in WORKLOADS:
        r = case(h, nb, n, w, k, args.rounds)
        out["cases"].append(r)
        ms = "  ".join(f"{key} {v:.3f}" for key, v in r["ms"].items())
        print(f"{nb} x (n {n}, w {w}, k {k}): {ms} ms | launches per slide {r['launches_per_slide']}, "
              f"max rel |x - x_gels| {r['rolling_vs_lstsq_max_rel']:.1e}", flush=True)
        torch.cuda.empty_cache()
    torch.cuda.synchronize()
    h.close()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
